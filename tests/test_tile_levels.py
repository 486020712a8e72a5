"""The level schedule of the tiled Cholesky's column groups (TilePlan::h_lvl_*, covins_b200/csrc/cholesky.cu).

The engine lays a column group's tiles out in nested-dissection order (position p of a chain at level = trailing one bits
of p, the chains interleaved level by level).  The plan cuts the group columns into levels of independent columns, and
factor() / solve() run each level as a few batched launches.

CPU: a host-only harness (tests/cpp/tile_plan_levels_dump.cu) dumps the level data of a plan built on BA-like masks
(IMU chains of 1-40 tiles, then a dense pose part) and PGO-like masks (chain interiors, then a border).  The levels must be
independent, their merged update lists must hold exactly the width-1 plan's (target, panel) products of the group
columns, each once, and a chain of n tiles must take ceil(log2(n + 1)) levels.

The engine's layout function (cvb_chol::nd_layout) is checked on the IMU chains of the C1 and C2 maps.

GPU: factor + solve through tests/cpp/chol_harness.cu on the same kind of masks, and on one whose level is split at the
32-column cap: bitwise the width-1 plan's L, tile inverses and x, and the backward-error bound of
tests/test_cholesky_kernels.py."""
import math
import os
import subprocess
import zlib

import numpy as np
import pytest

from test_cholesky_kernels import LD, T, _bound, _factor, _matrix, _same_bits, _within, gamma, h, harness  # noqa: F401
from test_tile_plan import _structure

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


@pytest.fixture(scope="module")
def levels_exe(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("tile_levels") / "tile_plan_levels_dump")
    subprocess.check_call([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-std=c++17", "--expt-relaxed-constexpr",
                           "-o", exe, os.path.join(ROOT, "tests", "cpp", "tile_plan_levels_dump.cu"),
                           os.path.join(ROOT, "covins_b200", "csrc", "cholesky.cu")])
    return exe


NAMES = ["col_ptr", "row_idx", "pair_ptr", "pair_i", "pair_j", "pair_mask", "pair_k0", "lvl_ptr", "lvl_pair_ptr",
         "lvl_pair_i", "lvl_pair_j", "lvl_pair_k0", "lvl_pair_mask", "lvl_trsm_ptr", "lvl_trsm_tile", "lvl_trsm_col",
         "lvl_fwd_ptr", "lvl_fwd_idx", "lvl_bwd_ptr", "lvl_bwd_idx", "col_base", "rowc_ptr", "rowc_idx"]


def _levels(exe, tmp, mask, group):
    nt = len(mask)
    fin, fout = os.path.join(tmp, "lin.bin"), os.path.join(tmp, "lout.bin")
    np.concatenate([np.array([nt, 1, 0, 0], np.int32), np.tril(mask).astype(np.int32).ravel(),
                    np.asarray(group, np.int32)]).tofile(fin)
    subprocess.check_call([exe, fin, fout])
    raw, pos, sec = np.fromfile(fout, np.int32), 0, []
    while pos < len(raw):
        n = raw[pos]
        sec.append(raw[pos + 1:pos + 1 + n])
        pos += 1 + n
    p = dict(zip(NAMES, sec))
    p["nt"] = nt
    return p


def _nd_order(sizes):
    """tile position of every (chain, p): level by level (trailing one bits of p), inside a level chain by chain"""
    lv = lambda p: (~p & (p + 1)).bit_length() - 1   # noqa: E731
    order = sorted(((lv(p), g, p) for g, n in enumerate(sizes) for p in range(n)))
    return {(g, p): t for t, (_, g, p) in enumerate(order)}


def _ba_mask(sizes, n_pose=2, seed=0):
    """IMU chains (band: p couples to p + 1, every tile to its chain's n_pose pose tiles), then the dense pose part"""
    pos = _nd_order(sizes)
    n_sb = len(pos)
    nt = n_sb + n_pose * len(sizes)
    m, group = np.eye(nt, dtype=bool), [-1] * nt
    for (g, p), t in pos.items():
        group[t] = g
        if p + 1 < sizes[g]:
            a, b = t, pos[(g, p + 1)]
            m[max(a, b), min(a, b)] = True
        m[n_sb + n_pose * g:n_sb + n_pose * (g + 1), t] = True
    m[n_sb:, n_sb:] = np.tril(np.ones((nt - n_sb, nt - n_sb), bool))
    return m, group


def _pgo_mask(sizes):
    """chain interiors (band of 1 tile), each coupled at its two ends to its own border tile; the border tiles coupled
    to each other (loop edges)"""
    pos = _nd_order(sizes)
    n_in = len(pos)
    nt = n_in + len(sizes)
    m, group = np.eye(nt, dtype=bool), [-1] * nt
    for (g, p), t in pos.items():
        group[t] = g
        if p + 1 < sizes[g]:
            a, b = t, pos[(g, p + 1)]
            m[max(a, b), min(a, b)] = True
        if p in (0, sizes[g] - 1):
            m[n_in + g, t] = True
    m[n_in:, n_in:] = np.tril(np.ones((len(sizes), len(sizes)), bool))
    return m, group


def _cap_mask(n_leaf, n_pose=2):
    """one group of n_leaf independent tiles, every one coupled to the same n_pose pose tiles: a level of more than 32
    columns whose panels all reach the same targets, so the level builder has to split it"""
    nt = n_leaf + n_pose
    m, group = np.eye(nt, dtype=bool), [0] * n_leaf + [-1] * n_pose
    m[n_leaf:, :n_leaf] = True
    m[n_leaf:, n_leaf:] = np.tril(np.ones((n_pose, n_pose), bool))
    return m, group


PLAN_CASES = {
    "ba_one_chain_1": _ba_mask([1]),
    "ba_one_chain_2": _ba_mask([2]),
    "ba_one_chain_7": _ba_mask([7]),
    "ba_one_chain_29": _ba_mask([29]),
    "ba_one_chain_40": _ba_mask([40]),
    "ba_chains_5x29": _ba_mask([29] * 5),
    "ba_chains_mixed": _ba_mask([40, 1, 13, 2, 31, 8]),
    "pgo_chains": _pgo_mask([20, 7, 33]),
    "pgo_one_chain": _pgo_mask([16]),
    "ba_one_chain_70": _ba_mask([70]),
    "cap_leaves_34": _cap_mask(34),
    "cap_leaves_65": _cap_mask(65),
}


@pytest.mark.parametrize("case", list(PLAN_CASES))
def test_levels_plan(levels_exe, tmp_path, case):
    mask, group = PLAN_CASES[case]
    nt = len(mask)
    L = _structure(mask)
    p = _levels(levels_exe, str(tmp_path), mask, group)
    lp = p["lvl_ptr"]
    assert lp[0] == 0 and lp[-1] == nt and (np.diff(lp) > 0).all()
    got, want = [], []
    n_levels = {}
    for l in range(len(lp) - 1):
        c0, c1 = int(lp[l]), int(lp[l + 1])
        cols = range(c0, c1)
        if group[c0] < 0:
            assert c1 == c0 + 1, f"level {l}: main-sequence column {c0} not alone"
            assert p["lvl_pair_ptr"][l + 1] == p["lvl_pair_ptr"][l] and p["lvl_trsm_ptr"][l + 1] == p["lvl_trsm_ptr"][l]
            continue
        for g in {group[k] for k in cols}:
            n_levels[g] = n_levels.get(g, 0) + 1
        # independent: no column of the level has a row tile inside the level
        for k in cols:
            assert group[k] >= 0
            assert not L[k, c0:k].any(), f"level {l}: column {k} depends on an earlier column of its level"
        # merged list: one entry per target, panels inside the level, 32 mask bits
        seen = set()
        for q in range(p["lvl_pair_ptr"][l], p["lvl_pair_ptr"][l + 1]):
            i, j, k0, m = (int(p[x][q]) for x in ("lvl_pair_i", "lvl_pair_j", "lvl_pair_k0", "lvl_pair_mask"))
            assert (i, j) not in seen and i >= j and m & 1 and c0 <= k0
            seen.add((i, j))
            for b in range(32):
                if m >> b & 1:
                    assert k0 + b < c1
                    got.append((i, j, k0 + b))
        # the width-1 lists of the level's columns (group columns: panel k alone), minus the chain's product
        for k in cols:
            for q in range(p["pair_ptr"][k], p["pair_ptr"][k + 1]):
                assert p["pair_k0"][k] == k and p["pair_mask"][q] == 1
                want.append((int(p["pair_i"][q]), int(p["pair_j"][q]), k))
        # trsm list: every panel tile of the level's columns but the chain's tile (k + 1, k)
        tr = {(int(t), int(c)) for t, c in zip(p["lvl_trsm_tile"][p["lvl_trsm_ptr"][l]:p["lvl_trsm_ptr"][l + 1]],
                                              p["lvl_trsm_col"][p["lvl_trsm_ptr"][l]:p["lvl_trsm_ptr"][l + 1]])}
        tr_want = set()
        for k in cols:
            rows = np.nonzero(L[k + 1:, k])[0] + k + 1
            for a, i in enumerate(rows):
                if not (a == 0 and i == k + 1):
                    tr_want.add((int(p["col_base"][k]) + 1 + a, k))
        assert tr == tr_want
        # solve targets
        fwd = sorted({int(i) for k in cols for i in np.nonzero(L[k + 1:, k])[0] + k + 1})
        bwd = sorted({int(i) for k in cols for i in np.nonzero(L[k, :k])[0]})
        assert list(p["lvl_fwd_idx"][p["lvl_fwd_ptr"][l]:p["lvl_fwd_ptr"][l + 1]]) == fwd
        assert list(p["lvl_bwd_idx"][p["lvl_bwd_ptr"][l]:p["lvl_bwd_ptr"][l + 1]]) == bwd
    assert len(got) == len(set(got)), "a (target, panel) product listed twice"
    assert sorted(got) == sorted(want)
    # every product of the group columns is in some width-1 list or is the chain's (k + 1, k + 1) product
    for k in range(nt):
        if group[k] < 0:
            continue
        rows = np.nonzero(L[k + 1:, k])[0] + k + 1
        prods = {(int(i), int(j), k) for a, i in enumerate(rows) for j in rows[:a + 1]}
        prods.discard((k + 1, k + 1, k))
        assert prods == {x for x in want if x[2] == k}
    if case.startswith("cap_leaves"):   # 32 columns per level at most: ceil(n / 32) runs of independent leaves
        assert n_levels[0] == math.ceil((len(group) - 2) / 32)
    elif case == "ba_one_chain_70":     # level 0 (35 columns sharing the pose rows) is split at the cap
        assert lp[1] == 32 and n_levels[0] <= math.ceil(math.log2(70 + 1)) + 1
    elif case.startswith("ba_one_chain") or case.startswith("pgo_one_chain"):
        n = sum(1 for g in group if g == 0)
        assert n_levels[0] == math.ceil(math.log2(n + 1))
    else:
        for g in set(x for x in group if x >= 0):
            n = sum(1 for x in group if x == g)
            assert n_levels[g] <= math.ceil(math.log2(n + 1))


def _layout(exe, tmp, sizes, bw):
    fin, fout = os.path.join(tmp, "yin.bin"), os.path.join(tmp, "yout.bin")
    np.array([bw, len(sizes)] + list(sizes), np.int32).tofile(fin)
    subprocess.check_call([exe, "layout", fin, fout])
    raw = np.fromfile(fout, np.int32)
    n = raw[0]
    return raw[1:1 + n], raw[2 + n:]


@pytest.mark.parametrize("config", ["C1", "C2"])
def test_engine_layout(levels_exe, tmp_path, config):
    """the engine's column-group layout (cvb_chol::nd_layout) on the IMU chains of a synthetic map: whole blocks per tile
    (14 speed-bias blocks, or 21 poses for a pose-graph chain interior), and the plan of the resulting structure — IMU
    couplings between the speed-bias tiles, each chain's speed-bias tiles coupled to its own pose tiles, a dense pose part —
    takes at most ceil(log2(tiles + 1)) levels per chain"""
    from covins_b200 import synth_map
    p = synth_map.make_config(config)
    K, ii, jj = int(p["K"]), p["imu_i"].astype(int), p["imu_j"].astype(int)
    parent = list(range(K))

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x
    for a, b in zip(ii, jj):
        ra, rb = find(a), find(b)
        if ra != rb:
            parent[max(ra, rb)] = min(ra, rb)
    chains = {}
    for k in range(K):
        chains.setdefault(find(k), []).append(k)
    chains = [c for r, c in sorted(chains.items()) if len(c) >= 2]
    assert len(chains) >= 1
    kf_block = {k: q for q, k in enumerate(x for c in chains for x in c)}   # block id: chain by chain, keyframe order
    for bw in (9, 6):
        off, got = _layout(levels_exe, str(tmp_path), [len(c) for c in chains], bw)
        per = T // bw
        assert (off >= 0).all() and ((off % T) % bw == 0).all() and ((off % T) + bw <= T).all(), "a block straddles two tiles"
        assert len(np.unique(off)) == len(off)
        for g, c in enumerate(chains):
            tiles = off[[kf_block[k] for k in c]] // T
            assert (got[tiles] == g).all()
            counts = np.bincount(tiles, minlength=len(got))[np.unique(tiles)]
            assert (counts <= per).all() and (counts == per).sum() >= len(counts) - 1, "a tile short of whole keyframes"
            assert len(np.unique(tiles)) == math.ceil(len(c) / per)
        if bw != 9:
            continue
        n_sb = len(got)
        pose_first = [n_sb]
        for c in chains:
            pose_first.append(pose_first[-1] + math.ceil(6 * len(c) / T))
        nt = pose_first[-1]
        m = np.eye(nt, dtype=bool)
        pose_tile = {}
        for g, c in enumerate(chains):
            for q, k in enumerate(c):
                pose_tile[k] = pose_first[g] + (6 * q) // T
        for a, b in zip(ii, jj):
            ta, tb = off[kf_block[a]] // T, off[kf_block[b]] // T
            for x, y in [(ta, tb), (ta, pose_tile[a]), (ta, pose_tile[b]), (tb, pose_tile[a]), (tb, pose_tile[b])]:
                m[max(x, y), min(x, y)] = True
        m[n_sb:, n_sb:] = np.tril(np.ones((nt - n_sb, nt - n_sb), bool))
        group = list(got) + [-1] * (nt - n_sb)
        pl = _levels(levels_exe, str(tmp_path), m, group)
        L = _structure(m)
        n_levels = {}
        lp = pl["lvl_ptr"]
        for l in range(len(lp) - 1):
            c0, c1 = int(lp[l]), int(lp[l + 1])
            if group[c0] < 0:
                continue
            for k in range(c0, c1):
                assert not L[k, c0:k].any()
            for g in {group[k] for k in range(c0, c1)}:
                n_levels[g] = n_levels.get(g, 0) + 1
        for g, c in enumerate(chains):
            nt_g = math.ceil(len(c) / per)
            assert n_levels[g] <= math.ceil(math.log2(nt_g + 1)), (config, g, n_levels[g], nt_g)


GPU_CASES = {"ba": ([7, 4, 2, 1], "ba"), "pgo": ([9, 3, 5], "pgo"), "cap": ([34], "cap")}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(GPU_CASES))
@pytest.mark.parametrize("kind", ["well", "cond1e10"])
def test_levels_factor(h, case, kind):  # noqa: F811
    """factor + solve with the level schedule: bitwise the width-1 and the blocked plan's L, tile inverses and x, and
    |A - L L^T| <= gamma_{n+16} |L||L^T| (+ the residual's own rounding)"""
    sizes, shape = GPU_CASES[case]
    mask, group = {"ba": _ba_mask, "pgo": _pgo_mask, "cap": lambda s: _cap_mask(s[0])}[shape](sizes)
    nt = len(mask)
    n = nt * T - 17
    A, _ = _matrix(mask, n, kind, zlib.crc32(f"levels-{case}-{kind}".encode()))
    b = (A.astype(LD) @ np.random.default_rng(3).standard_normal(n).astype(LD)).astype(np.float64)
    lev = _factor(h, mask, [A], [b], "group", group)[0]
    for name, ref in [("width1", _factor(h, mask, [A], [b], "width1")[0]), ("blocked", _factor(h, mask, [A], [b])[0])]:
        assert ref["flag"] == 0 and lev["flag"] == 0
        _same_bits(f"L (levels vs {name})", lev["L"], ref["L"])
        _same_bits(f"tile inverses (levels vs {name})", lev["linv"], ref["linv"])
        _same_bits(f"x (levels vs {name})", lev["x"], ref["x"])
    L = lev["L"][:n, :n]
    low = np.tril(np.ones((n, n), bool))
    R = np.abs(A - L @ L.T)[low]
    mag = (np.abs(L) @ np.abs(L).T)[low].astype(LD) / (1 - gamma(n))
    _within(f"levels factor L {case}-{kind}", R, _bound(gamma(n + 16) + gamma(n + 1), mag, 0) + _bound(LD(2.0) ** -53, np.abs(A)[low], 0))
