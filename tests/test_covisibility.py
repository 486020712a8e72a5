"""cvb_covisibility: the covisibility graph of a whole map in one call (Keyframe::UpdateCovisibilityConnections for every
keyframe), in the canonical form include/covins_b200.h defines (rules 1-4).
CPU: the oracle (oracle/covis.py, the reference's per-keyframe counter loop) equals an independent restatement — the
scipy.sparse product A @ A.T of the 0/1 keyframe x landmark matrix, then rules 3-4 in vectorised numpy — on hand cases
and random maps; the small hand cases are also pinned to literal lists.
GPU: through the C-ABI, nbr_ptr / nbr_kf / nbr_w equal the oracle exactly: hand cases, the synthetic maps the bundle
adjustment tests use (with and without the outlier mask of a GBA round), a map with one landmark seen by every
keyframe; the sizing protocol; chunked == unchunked (the pair budget is an argument of the library's internal function,
reached through tests/cpp/covis_harness.cu); repeatability; launch counts; refused inputs; the C++ shim on mock containers.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import covis as ora

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


# ------------------------------------------------------------------------------------------------------------------
# maps
# ------------------------------------------------------------------------------------------------------------------
def _csr(tracks):
    """list of observer lists → (lm_obs_ptr, obs_kf)"""
    ptr = np.concatenate([[0], np.cumsum([len(t) for t in tracks])]).astype(np.int32)
    kf = np.array([k for t in tracks for k in t], np.int32)
    return ptr, kf


def _case(K, tracks, min_weight=15, obs_skip=None, lm_valid=None):
    ptr, kf = _csr(tracks)
    return dict(K=K, lm_obs_ptr=ptr, obs_kf=kf, min_weight=min_weight,
                obs_skip=None if obs_skip is None else np.asarray(obs_skip, np.uint8),
                lm_valid=None if lm_valid is None else np.asarray(lm_valid, np.uint8))


def random_map(seed, K, L, window=12, max_track=10):
    """tracks over a window of neighbouring keyframes (so that some weights pass 15), in random observer order"""
    rng = np.random.default_rng(seed)
    tracks = []
    for _ in range(L):
        a = int(rng.integers(0, K))
        near = np.arange(max(0, a - window), min(K, a + window + 1))
        n = int(min(len(near), rng.integers(0, max_track + 1)))
        tracks.append(rng.choice(near, n, replace=False).tolist())
    return tracks


STRONG3 = [[0, 1, 2]] * 20                       # keyframes 0, 1, 2 share 20 landmarks
EQUAL = [[0, 1]] * 3 + [[2, 0]] * 3 + [[2, 3]] * 5 + [[4, 1]] * 5


def hand_cases():
    rnd = random_map(3, 40, 900)
    n_rnd = sum(len(t) for t in rnd)
    rng = np.random.default_rng(4)
    c = {
        # both keyframes fall back to their single best neighbour, each other
        "two_below_threshold": _case(2, [[0, 1]] * 3),
        # keyframe 3's best neighbour (1) has strong neighbours of its own and would not pick 3: the edge still exists on both sides
        "fallback_into_strong": _case(4, STRONG3 + [[3, 1]] * 2),
        # 0 sees 1 and 2 equally (3 each): its fallback is the lower index, 1; 2's own best is 3, so 0-2 is not an edge
        "equal_weights_argmax": _case(5, EQUAL),
        # the same weights all reaching the threshold: rows ordered by weight, equal weights by index
        "equal_weights_order": _case(5, EQUAL, min_weight=3),
        "no_shared_landmark": _case(3, [[0, 1]] * 4 + [[2]]),
        "one_keyframe": _case(1, [[0], [], [0]]),
        "no_landmarks": _case(3, []),
        "short_tracks_only": _case(4, [[], [1], [3], []]),
        "no_keyframes": _case(0, []),
        # one skipped observation takes w(0,1) and w(1,2) from 15 to 14: 1 falls back to its best, 0, and loses 2
        "skip_drops_below": _case(3, [[0, 1, 2]] * 15, obs_skip=[0, 1, 0] + [0] * 42),
        # the two landmarks that tie 3 to 1 are invalid: 3's row is empty
        "invalid_landmark_removes_edge": _case(4, STRONG3 + [[3, 1]] * 2, lm_valid=[1] * 20 + [0, 0]),
        "min_weight_1": _case(40, rnd, min_weight=1),
        "min_weight_unreachable": _case(40, rnd, min_weight=10 ** 6),
        "random_masks": _case(40, rnd, min_weight=6, obs_skip=rng.random(n_rnd) < 0.2, lm_valid=rng.random(len(rnd)) < 0.9),
    }
    return c


CASES = hand_cases()
LITERAL = {   # name → (nbr_ptr, nbr_kf, nbr_w)
    "two_below_threshold": ([0, 1, 2], [1, 0], [3, 3]),
    "fallback_into_strong": ([0, 2, 5, 7, 8], [1, 2, 0, 2, 3, 0, 1, 1], [20, 20, 20, 20, 2, 20, 20, 2]),
    "equal_weights_argmax": ([0, 1, 3, 4, 5, 6], [1, 4, 0, 3, 2, 1], [3, 5, 3, 5, 5, 5]),
    "equal_weights_order": ([0, 2, 4, 6, 7, 8], [1, 2, 4, 0, 3, 0, 2, 1], [3, 3, 5, 3, 5, 3, 5, 5]),
    "no_shared_landmark": ([0, 1, 2, 2], [1, 0], [4, 4]),
    "skip_drops_below": ([0, 2, 3, 4], [2, 1, 0, 0], [15, 14, 14, 15]),
    "invalid_landmark_removes_edge": ([0, 2, 4, 6, 6], [1, 2, 0, 2, 0, 1], [20] * 6),
}


def independent(lm_obs_ptr, obs_kf, K, obs_skip=None, lm_valid=None, min_weight=15):
    """A @ A.T on the 0/1 keyframe x landmark matrix, then rules 3-4 vectorised"""
    L = len(lm_obs_ptr) - 1
    lm = np.repeat(np.arange(L), np.diff(lm_obs_ptr))
    kf = np.asarray(obs_kf)[:len(lm)].astype(np.int64)
    take = np.ones(len(lm), bool)
    if obs_skip is not None:
        take &= np.asarray(obs_skip)[:len(lm)] == 0
    if lm_valid is not None:
        take &= np.asarray(lm_valid)[lm] != 0
    A = sp.csr_matrix((np.ones(take.sum(), np.int64), (kf[take], lm[take])), shape=(K, max(L, 1)))
    assert A.nnz == take.sum() and (A.data == 1).all()
    W = sp.coo_matrix(A @ A.T)
    off = (W.row != W.col) & (W.data > 0)
    i, j, w = W.row[off].astype(np.int64), W.col[off].astype(np.int64), W.data[off]
    strong = w >= min_weight
    has_strong = np.bincount(i[strong], minlength=K) > 0
    order = np.lexsort((j, -w, i))                                   # per row: weight descending, index ascending
    first = order[np.concatenate([[True], i[order][1:] != i[order][:-1]])] if len(i) else order
    best = np.full(K, -1)
    best[i[first]] = j[first]
    conn = strong | (~has_strong[i] & (best[i] == j)) | (~has_strong[j] & (best[j] == i))
    sel = order[conn[order]]
    nbr_ptr = np.concatenate([[0], np.cumsum(np.bincount(i[sel], minlength=K))]).astype(np.int32)
    return nbr_ptr, j[sel].astype(np.int32), w[sel].astype(np.int32)


def _same(got, ref):
    return all(np.array_equal(a, b) and a.dtype == b.dtype for a, b in zip(got, ref))


def _args(c):
    return c["lm_obs_ptr"], c["obs_kf"], c["K"], c["obs_skip"], c["lm_valid"], c["min_weight"]


# ------------------------------------------------------------------------------------------------------------------
# CPU: the oracle
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_equals_independent_restatement_on_hand_cases(name):
    ref = ora.covisibility(*_args(CASES[name]))
    assert _same(ref, independent(*_args(CASES[name])))
    if name in LITERAL:
        assert all(np.array_equal(a, b) for a, b in zip(ref, LITERAL[name]))


@pytest.mark.parametrize("seed", range(6))
def test_oracle_equals_independent_restatement_on_random_maps(seed):
    rng = np.random.default_rng(100 + seed)
    K = int(rng.integers(2, 120))
    tracks = random_map(seed, K, int(rng.integers(1, 3000)), window=int(rng.integers(1, 20)), max_track=int(rng.integers(2, 16)))
    n = sum(len(t) for t in tracks)
    ptr, kf = _csr(tracks)
    skip = (rng.random(n) < 0.1).astype(np.uint8) if seed % 2 else None
    valid = (rng.random(len(tracks)) < 0.9).astype(np.uint8) if seed % 3 else None
    mw = int(rng.integers(1, 20))
    ref = ora.covisibility(ptr, kf, K, skip, valid, mw)
    assert _same(ref, independent(ptr, kf, K, skip, valid, mw))
    assert ref[0][-1] == len(ref[1]) > 0


def test_oracle_refuses_a_duplicate_observer():
    with pytest.raises(AssertionError):
        ora.covisibility(*_csr([[0, 1, 0]]), 2)


# ------------------------------------------------------------------------------------------------------------------
# GPU, through the C-ABI
# ------------------------------------------------------------------------------------------------------------------
def _raw(ctx, K, ptr, kf, skip=None, valid=None, min_weight=15, cap=0, nbr_kf=None, nbr_w=None, L=None, nbr_ptr="own", n_total="own"):
    """one cvb_covisibility call on caller-held arrays → (status, nbr_ptr, n_total)"""
    from covins_b200 import lib
    p = lambda a: None if a is None else a.ctypes.data
    own_ptr = np.full(max(K, 0) + 1, -7, np.int32)
    n = C.c_int64(-7)
    rc = lib().cvb_covisibility(ctx.handle, K, len(ptr) - 1 if L is None else L, p(ptr), p(kf), p(skip), p(valid), min_weight,
                                p(own_ptr) if nbr_ptr == "own" else None, p(nbr_kf), p(nbr_w), cap, C.byref(n) if n_total == "own" else None)
    return rc, own_ptr, n.value


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_hand_cases_equal_the_oracle(ctx, name):
    from covins_b200 import mapgraph
    got = mapgraph.covisibility(ctx, *_args(CASES[name]))
    assert _same(got, ora.covisibility(*_args(CASES[name])))


@pytest.mark.gpu
@pytest.mark.parametrize("config,gba_mask", [("C1", False), ("C1", True), ("C3", False), ("C3", True)])
def test_synthetic_maps_equal_the_oracle(ctx, config, gba_mask):
    """the arrays the bundle-adjustment tests build; the mask is what a GBA's outlier round erased from the map"""
    from covins_b200 import mapgraph, optimization as O, synth_map
    p = synth_map.make_config(config)
    skip = None
    if gba_mask:
        skip = O.global_bundle_adjustment(ctx, p, iterations_limit=2)["obs_removed"].astype(np.uint8)
        assert 0 < skip.sum() < len(skip)
    got = mapgraph.covisibility(ctx, p["lm_obs_ptr"], p["obs_kf"], p["K"], obs_skip=skip)
    ref = ora.covisibility(p["lm_obs_ptr"], p["obs_kf"], p["K"], obs_skip=skip)
    assert _same(got, ref)
    assert len(ref[1]) > 4 * p["K"] and ref[2].max() >= 15


def skewed_map():
    """100 000 short tracks beside one landmark every one of 2 000 keyframes observes (2 M of the pairs)"""
    tracks = random_map(9, 2000, 100_000, window=10, max_track=8)
    tracks.insert(50_000, np.random.default_rng(1).permutation(2000).tolist())
    return _csr(tracks)


@pytest.mark.gpu
def test_one_landmark_seen_by_every_keyframe(ctx):
    from covins_b200 import mapgraph
    ptr, kf = skewed_map()
    got = mapgraph.covisibility(ctx, ptr, kf, 2000)
    assert _same(got, ora.covisibility(ptr, kf, 2000))
    got1 = mapgraph.covisibility(ctx, ptr, kf, 2000, min_weight=1)               # every pair of keyframes is an edge
    assert _same(got1, ora.covisibility(ptr, kf, 2000, min_weight=1)) and len(got1[1]) == 2000 * 1999


@pytest.mark.gpu
def test_sizing_protocol(ctx):
    c = CASES["random_masks"]
    ref = ora.covisibility(*_args(c))
    n = len(ref[1])
    a = (c["K"], c["lm_obs_ptr"], c["obs_kf"], c["obs_skip"], c["lm_valid"], c["min_weight"])
    rc, nbr_ptr, n_total = _raw(ctx, *a, cap=0)                                  # null arrays: the size and nbr_ptr only
    assert rc == 0 and n_total == n and np.array_equal(nbr_ptr, ref[0])
    kf = np.full(n, -5, np.int32); w = np.full(n, -5, np.int32)
    rc, nbr_ptr, n_total = _raw(ctx, *a, cap=n - 1, nbr_kf=kf, nbr_w=w)          # one short: the arrays stay untouched
    assert rc == 0 and n_total == n and np.array_equal(nbr_ptr, ref[0]) and (kf == -5).all() and (w == -5).all()
    rc, nbr_ptr, n_total = _raw(ctx, *a, cap=n, nbr_kf=kf, nbr_w=w)
    assert rc == 0 and n_total == n and _same((nbr_ptr, kf, w), ref)


def _n_pairs(ptr, kf, K):
    n = np.diff(ptr).astype(np.int64)
    return int((n * (n - 1) // 2).sum())


@pytest.mark.gpu
def test_two_runs_are_identical_and_launches_do_not_depend_on_the_map(ctx):
    from covins_b200 import synth_map
    counts = []
    p = synth_map.make_config("C1")
    for K, ptr, kf in [(40, CASES["min_weight_1"]["lm_obs_ptr"], CASES["min_weight_1"]["obs_kf"]), (p["K"], p["lm_obs_ptr"], p["obs_kf"])]:
        rc, _, n = _raw(ctx, K, ptr, kf, cap=0)
        outs = []
        for _ in range(2):
            kf_o = np.empty(n, np.int32); w_o = np.empty(n, np.int32)
            l0 = ctx.launch_count()
            rc, nbr_ptr, n_total = _raw(ctx, K, ptr, kf, cap=n, nbr_kf=kf_o, nbr_w=w_o)
            counts.append(ctx.launch_count() - l0)
            assert rc == 0 and n_total == n > 0
            outs.append(nbr_ptr.tobytes() + kf_o.tobytes() + w_o.tobytes())
        assert outs[0] == outs[1]
    assert len(set(counts)) == 1 and counts[0] == 8       # expand, sort, encode; row stats, connect, scan, sort, decode


def _build(src, exe, compiler):
    import covins_b200
    if not os.path.exists(covins_b200.LIB_PATH):
        covins_b200.build()
    if compiler == "nvcc":
        subprocess.check_call([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr", "-o", exe,
                               os.path.join(ROOT, "tests", "cpp", src)])
    else:
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-o", exe, os.path.join(ROOT, "tests", "cpp", src),
                               "-L" + os.path.join(ROOT, "covins_b200"), "-lcovins_b200", "-Wl,-rpath," + os.path.join(ROOT, "covins_b200")])


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("covis_harness") / "covis_harness")
    _build("covis_harness.cu", exe, "nvcc")
    return exe


def test_harness_builds(harness):
    assert os.access(harness, os.X_OK)


def _run_harness(harness, d, K, ptr, kf, min_weight, budget, skip=None, valid=None):
    for name, a in (("ptr", ptr), ("kf", kf), ("skip", skip), ("valid", valid)):
        if a is not None:
            np.ascontiguousarray(a).tofile(d / f"{name}.bin")
    r = subprocess.run([harness, str(d), str(K), str(min_weight), str(budget)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = tuple(np.fromfile(d / f"out_{n}.bin", np.int32) for n in ("ptr", "kf", "w"))
    return out, int(np.fromfile(d / "out_launches.bin", np.int64)[0])


@pytest.mark.gpu
def test_chunked_equals_one_chunk(ctx, harness, tmp_path):
    """a small pair budget takes the path a map with more pairs than the workspace budget takes: the pair range in chunks
    (cut inside landmarks), partial counts merged by key.  Same bytes; the launches follow the number of chunks only."""
    from covins_b200 import mapgraph
    c = CASES["random_masks"]
    lm = np.repeat(np.arange(len(c["lm_valid"])), np.diff(c["lm_obs_ptr"]))
    n = np.bincount(lm[(c["lm_valid"][lm] != 0) & (c["obs_skip"] == 0)])          # participating observers per landmark
    pairs = int((n * (n - 1) // 2).sum())
    one = mapgraph.covisibility(ctx, *_args(c))
    assert _same(one, ora.covisibility(*_args(c)))
    for budget in (10 ** 9, pairs // 2 + 1, 97, 7):
        got, launches = _run_harness(harness, tmp_path, c["K"], c["lm_obs_ptr"], c["obs_kf"], c["min_weight"], budget, c["obs_skip"], c["lm_valid"])
        chunks = -(-pairs // min(budget, pairs))
        assert _same(got, one), budget
        assert launches == 5 * chunks + 3, (budget, chunks, launches)
    # the skewed map: chunk boundaries fall inside the landmark every keyframe observes
    d = tmp_path / "skewed"; d.mkdir()
    ptr, kf = skewed_map()
    got, launches = _run_harness(harness, d, 2000, ptr, kf, 15, 700_001)
    assert _same(got, mapgraph.covisibility(ctx, ptr, kf, 2000)) and launches == 5 * -(-_n_pairs(ptr, kf, 2000) // 700_001) + 3


@pytest.mark.gpu
def test_invalid_input_is_refused_before_any_launch(ctx):
    from covins_b200 import lib, mapgraph
    ptr, kf = _csr([[0, 1], [1, 2], [2, 0, 1]])
    one = np.zeros(1, np.int32)
    bad = {
        "null nbr_ptr": dict(K=3, ptr=ptr, kf=kf, nbr_ptr=None),
        "null n_total": dict(K=3, ptr=ptr, kf=kf, n_total=None),
        "null lm_obs_ptr": dict(K=3, ptr=None, kf=kf, L=3),
        "null obs_kf": dict(K=3, ptr=ptr, kf=None),
        "null outputs with cap": dict(K=3, ptr=ptr, kf=kf, cap=4),
        "negative K": dict(K=-1, ptr=ptr, kf=kf),
        "negative L": dict(K=3, ptr=ptr, kf=kf, L=-1),
        "negative cap": dict(K=3, ptr=ptr, kf=kf, cap=-1, nbr_kf=one, nbr_w=one),
        "ptr not from 0": dict(K=3, ptr=ptr + 1, kf=kf),
        "ptr decreasing": dict(K=3, ptr=np.array([0, 4, 2, 7], np.int32), kf=kf),
        "kf too large": dict(K=2, ptr=ptr, kf=kf),
        "kf negative": dict(K=3, ptr=ptr, kf=np.array([0, 1, 1, -1, 2, 0, 1], np.int32)),
        "min_weight 0": dict(K=3, ptr=ptr, kf=kf, min_weight=0),
        "duplicate observer": dict(K=3, ptr=ptr, kf=np.array([0, 1, 1, 2, 2, 0, 2], np.int32)),
    }
    for name, kw in bad.items():
        l0 = ctx.launch_count()
        rc, _, _ = _raw(ctx, kw.pop("K"), kw.pop("ptr"), kw.pop("kf"), **kw)
        assert rc == 1, name                                                       # CVB_ERR_INVALID
        assert b"cvb_covisibility" in lib().cvb_last_error(ctx.handle), name
        assert ctx.launch_count() == l0, name
        assert _same(mapgraph.covisibility(ctx, ptr, kf, 3, min_weight=1), ora.covisibility(ptr, kf, 3, min_weight=1)), name


# ------------------------------------------------------------------------------------------------------------------
# the C++ shim on mock containers
# ------------------------------------------------------------------------------------------------------------------
def test_shim_covis_compiles_and_refuses_missing_input(tmp_path):
    exe = str(tmp_path / "shim_covis_test")
    _build("shim_covis_test.cpp", exe, "g++")
    assert subprocess.run([exe, str(tmp_path), "15"]).returncode == 2            # nothing dumped: refused before any GPU work


@pytest.mark.gpu
@pytest.mark.parametrize("with_invalid", [False, True])
def test_shim_on_mock_containers_equals_the_oracle(tmp_path, with_invalid):
    """covins_b200::UpdateCovisibilityConnections: every mock keyframe's lists equal the oracle's for the same map; invalid
    keyframes and landmarks are absent from the flattening (as in GlobalBundleAdjustment) and keep empty lists"""
    from covins_b200 import synth_map
    p = synth_map.make_map(seed=21, n_agents=2, kf_per_agent=40, n_lm=2000)
    K, L = p["K"], p["L"]
    rng = np.random.default_rng(2)
    kf_invalid = (rng.random(K) < 0.1 if with_invalid else np.zeros(K, bool)).astype(np.uint8)
    lm_invalid = (rng.random(L) < 0.1 if with_invalid else np.zeros(L, bool)).astype(np.uint8)
    p["lm_obs_ptr"].astype(np.int32).tofile(tmp_path / "ptr.bin"); p["obs_kf"].astype(np.int32).tofile(tmp_path / "kf.bin")
    kf_invalid.tofile(tmp_path / "kf_invalid.bin"); lm_invalid.tofile(tmp_path / "lm_invalid.bin")
    exe = str(tmp_path / "shim_covis_test")
    _build("shim_covis_test.cpp", exe, "g++")
    subprocess.check_call([exe, str(tmp_path), "15"])
    # an invalid keyframe keeps its number here and loses its observations: the valid keyframes' order is the same
    ref = ora.covisibility(p["lm_obs_ptr"], p["obs_kf"], K, obs_skip=kf_invalid[p["obs_kf"]], lm_valid=1 - lm_invalid)
    assert np.array_equal(np.fromfile(tmp_path / "out_cnt.bin", np.int32), np.diff(ref[0]))
    assert np.array_equal(np.fromfile(tmp_path / "out_kf.bin", np.int32), ref[1])
    assert np.array_equal(np.fromfile(tmp_path / "out_w.bin", np.int32), ref[2])
    assert len(ref[1]) > 2 * K and (not with_invalid or (np.diff(ref[0])[kf_invalid == 1] == 0).all())
