"""The blocked trailing-update schedule of the tiled Cholesky (covins_b200/csrc/cholesky.cu, TilePlan::build).

CPU: a host-only harness (tests/cpp/tile_plan_dump.cu, compiled with nvcc, run without a GPU) dumps the launch lists of a
plan.  For every mask the blocked plan must execute exactly the (target tile, panel) products of the width-1 plan (the
same plan built with a one-rank owner map), each once, in the same kernel class (the critical chain's tile product or a
DMMA tile GEMM), and every target tile must receive its panels in increasing order.

GPU: the dense solve against LAPACK at sizes that put block boundaries everywhere and on block-sparse patterns."""
import os
import subprocess
from collections import Counter

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
T = 128


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("tile_plan") / "tile_plan_dump")
    subprocess.check_call([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-std=c++17", "--expt-relaxed-constexpr",
                           "-o", exe, os.path.join(ROOT, "tests", "cpp", "tile_plan_dump.cu"),
                           os.path.join(ROOT, "covins_b200", "csrc", "cholesky.cu")])
    return exe


def _plan(exe, tmp, mask, group=None, owner=None, rank=0):
    nt = len(mask)
    hdr = [nt, group is not None, owner is not None, rank]
    parts = [np.array(hdr, np.int32), np.tril(mask).astype(np.int32).ravel()]
    if group is not None:
        parts.append(np.asarray(group, np.int32))
    if owner is not None:
        parts.append(np.asarray(owner, np.int32))
    fin, fout = os.path.join(tmp, "in.bin"), os.path.join(tmp, "out.bin")
    np.concatenate(parts).tofile(fin)
    subprocess.check_call([exe, fin, fout])
    raw, pos, sec = np.fromfile(fout, np.int32), 0, []
    while pos < len(raw):
        n = raw[pos]
        sec.append(raw[pos + 1:pos + 1 + n])
        pos += 1 + n
    names = ["col_ptr", "row_idx", "pair_ptr", "pair_i", "pair_j", "pair_mask", "pair_k0", "pair_split", "blk_end", "b", "flops"]
    p = dict(zip(names, sec))
    p["nt"] = nt
    return p


def _structure(mask):
    """tile structure of L (symbolic right-looking elimination) → bool [nt, nt], lower"""
    L = np.tril(np.asarray(mask, bool)) | np.eye(len(mask), dtype=bool)
    for k in range(len(L)):
        rows = np.nonzero(L[k + 1:, k])[0] + k + 1
        L[np.ix_(rows, rows)] = True
    return np.tril(L)


def _products(p):
    """plan order of the (i, j, k, class) products: column by column, the update lists (the pair at their head, a
    diagonal tile, is applied before the chain's product), then the chain's S(k+1,k+1) -= L(k+1,k) L(k+1,k)^T"""
    out = []
    for k in range(p["nt"]):
        rows = p["row_idx"][p["col_ptr"][k]:p["col_ptr"][k + 1]]
        for q in range(p["pair_ptr"][k], p["pair_ptr"][k + 1]):
            i, j, m = int(p["pair_i"][q]), int(p["pair_j"][q]), int(p["pair_mask"][q])
            assert m > 0
            for b in range(32):
                if m >> b & 1:
                    out.append((i, j, int(p["pair_k0"][k]) + b, "dmma"))
        if len(rows) and rows[0] == k + 1:
            out.append((k + 1, k + 1, k, "chain"))
    return out


def _check(exe, tmp, mask, group=None):
    L = _structure(mask)
    nt = len(L)
    blk = _plan(exe, tmp, mask, group)
    ref = _plan(exe, tmp, mask, group, owner=[0] * nt)        # one-rank owner map: width 1 everywhere
    b = int(blk["b"][0])
    assert (ref["blk_end"] == np.arange(1, nt + 1)).all() and (ref["pair_k0"] == np.arange(nt)).all()
    assert (ref["pair_mask"] == 1).all()
    pb, pr = _products(blk), _products(ref)
    # every product of the width-1 plan exactly once, in the same kernel class; both equal the symbolic structure's
    assert Counter(pb) == Counter(pr)
    assert max(Counter(pb).values(), default=1) == 1
    want = {(i, j, k) for k in range(nt) for j in range(k + 1, nt) for i in range(j, nt) if L[i, k] and L[j, k]}
    assert {x[:3] for x in pb} == want
    assert all((c == "chain") == (i == j == k + 1) for i, j, k, c in pb)
    assert int(blk["flops"][0]) == int(ref["flops"][0]) == len(want) + int(L.sum()) - nt
    # panels of each target tile in increasing order
    last = {}
    for i, j, k, _ in pb:
        assert last.get((i, j), -1) < k, (i, j, k)
        last[(i, j)] = k
    # blocks: runs of at most b main-sequence columns; column groups width 1
    end = blk["blk_end"]
    for k in range(nt):
        assert k < end[k] <= min(k + b, nt)
        if group is not None and group[k] >= 0:
            assert end[k] == k + 1
    # the work stream's part of a list (listed first) is the next block's columns, the first of them first
    for k in range(nt):
        lo, hi, na = blk["pair_ptr"][k], blk["pair_ptr"][k + 1], blk["pair_split"][k]
        js = blk["pair_j"][lo:hi]
        assert (np.diff(js) >= 0).all()
        if group is not None and group[k] >= 0:
            assert na == hi - lo
        elif end[k] == k + 1:
            nxt = end[end[k]] if end[k] < nt else nt
            assert (js[:na] < nxt).all() and (js[na:] >= nxt).all()
        else:
            assert na == hi - lo and (js > k).all() and (js < end[k]).all()
    return blk


def _random_mask(rng, nt, density):
    m = rng.random((nt, nt)) < density
    return np.tril(m | m.T) | np.eye(nt, dtype=bool)


@pytest.mark.parametrize("nt", [1, 2, 3, 5, 6, 7, 8, 9, 12])
def test_plan_dense(harness, tmp_path, nt):
    p = _check(harness, str(tmp_path), np.ones((nt, nt), bool))
    if nt >= 2 and int(p["b"][0]) > 1:
        assert (p["blk_end"] != np.arange(1, nt + 1)).any()


@pytest.mark.parametrize("nt,bw", [(10, 1), (11, 2), (16, 3)])
def test_plan_banded(harness, tmp_path, nt, bw):
    i, j = np.indices((nt, nt))
    _check(harness, str(tmp_path), (i - j >= 0) & (i - j <= bw))


def test_plan_arrow(harness, tmp_path):
    nt = 11
    m = np.eye(nt, dtype=bool)
    m[-2:, :] = True
    _check(harness, str(tmp_path), m)


def test_plan_missing_next_panel_tile(harness, tmp_path):
    """(k+1,k) is a zero tile of L for several k, some of them at a block's last column (no chain product there); column 1
    has no rows at all while column 0 does"""
    nt = 10
    m = np.eye(nt, dtype=bool)
    for i, j in [(2, 0), (3, 0), (5, 3), (6, 3), (6, 5), (8, 5), (9, 8), (9, 6), (7, 4)]:
        m[i, j] = True
    L = _structure(m)
    assert not L[1, 0] and not L[4, 3] and not L[2:, 1].any() and L[2:, 0].any()
    _check(harness, str(tmp_path), m)


@pytest.mark.parametrize("seed", range(8))
def test_plan_random_block_sparse(harness, tmp_path, seed):
    rng = np.random.default_rng(seed)
    nt = int(rng.integers(6, 24))
    _check(harness, str(tmp_path), _random_mask(rng, nt, float(rng.uniform(0.05, 0.3))))


def test_plan_column_groups(harness, tmp_path):
    """IMU-chain-like groups first (each group a band of its own, coupled to the trailing pose columns), then the main
    sequence; and a group column in the middle of the main sequence"""
    rng = np.random.default_rng(3)
    sizes, nt_main = [3, 2, 4], 9
    nt = sum(sizes) + nt_main
    m = np.eye(nt, dtype=bool)
    group, c = [-1] * nt, 0
    for g, s in enumerate(sizes):
        for t in range(c, c + s):
            group[t] = g
            if t > c:
                m[t, t - 1] = True
            m[sum(sizes) + rng.integers(0, nt_main, 2), t] = True
        c += s
    m[sum(sizes):, sum(sizes):] |= np.tril(rng.random((nt_main, nt_main)) < 0.4)
    _check(harness, str(tmp_path), m, group)
    group2 = [-1] * nt
    group2[sum(sizes) + 3] = 0
    _check(harness, str(tmp_path), m, group2)


def test_plan_distributed_is_width_one(harness, tmp_path):
    rng = np.random.default_rng(5)
    nt = 12
    m = _random_mask(rng, nt, 0.3)
    owner = [(k // 2) % 2 for k in range(nt)]
    both = [_plan(harness, str(tmp_path), m, owner=owner, rank=r) for r in range(2)]
    ref = _plan(harness, str(tmp_path), m, owner=[0] * nt)
    for r, p in enumerate(both):
        assert (p["blk_end"] == np.arange(1, nt + 1)).all() and (p["pair_mask"] == 1).all()
        assert all(owner[j] == r for j in p["pair_j"])
    # the ranks' lists partition the one-rank lists (every update applied by the owner of its target column)
    got = Counter(x for p in both for x in _products(p) if x[3] == "dmma")
    assert got == Counter(x for x in _products(ref) if x[3] == "dmma")


def _rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-12)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [5 * T - 3, 6 * T, 7 * T, 8 * T + 1, 9 * T - 64])
def test_dense_solve_block_boundaries(ctx, n):
    from covins_b200 import optimization as O
    rng = np.random.default_rng(n)
    M = rng.normal(size=(n, n))
    A = M @ M.T + n * np.eye(n)
    b = rng.normal(size=n)
    x, _ = O.dense_cholesky_solve(ctx, A, b)
    assert _rel(x, np.linalg.solve(A, b)) < 1e-10


@pytest.mark.gpu
@pytest.mark.parametrize("pattern", ["banded", "arrow", "gaps", "random0", "random1"])
def test_dense_solve_block_sparse(ctx, pattern):
    from covins_b200 import optimization as O
    rng = np.random.default_rng(len(pattern))
    nt = 9
    if pattern == "banded":
        i, j = np.indices((nt, nt))
        tm = (i - j >= 0) & (i - j <= 2)
    elif pattern == "arrow":
        tm = np.eye(nt, dtype=bool)
        tm[-2:, :] = True
    elif pattern == "gaps":
        tm = np.eye(nt, dtype=bool)
        for i, j in [(2, 0), (3, 0), (5, 3), (6, 3), (6, 5), (8, 5), (8, 6), (7, 4)]:
            tm[i, j] = True
    else:
        tm = _random_mask(np.random.default_rng(int(pattern[-1])), nt, 0.25)
    tm = np.tril(tm | tm.T)
    n = nt * T - 17
    A = np.zeros((nt * T, nt * T))
    for i, j in zip(*np.nonzero(tm)):
        blk = rng.normal(size=(T, T)) * 0.02
        A[i * T:(i + 1) * T, j * T:(j + 1) * T] = blk
        A[j * T:(j + 1) * T, i * T:(i + 1) * T] = blk.T
    A = A[:n, :n] + (nt * T * 0.1 + 4.0) * np.eye(n)
    A = 0.5 * (A + A.T)
    b = rng.normal(size=n)
    x, _ = O.dense_cholesky_solve(ctx, A, b)
    assert _rel(x, np.linalg.solve(A, b)) < 1e-10
