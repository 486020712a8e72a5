"""The bundle adjustment sharded over an in-process rank group (cvb_group_create, cvb_ba_solve_group, cvb_gba_group).

  - a group of one is bitwise equal to O.solve / cvb_gba;
  - groups of 2 and 3, with and without the peer path, take the world = 1 solve's decisions and reach its states up to
    summation order (the tolerances of test_ba_restart_sharded.py's sharded solves); two runs are bitwise identical;
  - the group all-reduce alone equals a numpy sum in rank order, bit for bit, across chunk boundaries;
  - refused and failed calls leave no thread behind;
  - the C++ shim's GlobalBundleAdjustment(ContextGroup&, ...) against its single-context overload.
Contexts share device 0 unless a test says otherwise.  The peer path needs a device per rank (a shared-device group refuses
it), so it runs only in the distinct-device variants, which need as many GPUs as ranks and skip without them.
"""
import os
import subprocess

import numpy as np
import pytest
import torch

import covins_b200
from covins_b200 import optimization as O
from covins_b200 import synth_map
from test_ba_map_shapes import singular_imu
from test_ba_restart_sharded import RESULT_KEYS, _assert_bitwise, _case, _rel

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_TWO_GPUS = pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two GPUs")
LAYOUTS = ["shared", pytest.param("distinct", marks=_TWO_GPUS)]
# (layout, peer path): the all-reduce path on one device and on distinct devices, the peer path on distinct devices
PATHS = [("shared", False), pytest.param("distinct", False, marks=_TWO_GPUS), pytest.param("distinct", True, marks=_TWO_GPUS)]


def _need_devices(layout, world):
    if layout == "distinct" and torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")


def _threads():
    return len(os.listdir("/proc/self/task"))


class _Grp:
    """n contexts (all on device 0, or dealt over the visible devices) and the group over them"""

    def __init__(self, n, layout="shared"):
        ndev = torch.cuda.device_count() if layout == "distinct" else 1
        self.ctxs = [covins_b200.Context(r % ndev) for r in range(n)]
        self.g = O.Group(self.ctxs)

    def __enter__(self):
        return self.g

    def __exit__(self, *a):
        self.g.close()
        for c in self.ctxs:
            c.close()


def _solve_kw(kw):
    return {k: v for k, v in kw.items() if k in ("visual_only", "cauchy_reproj", "cauchy_edge", "edges", "obs_skip")}


# ---------------------------------------------------------------------------------------------- group of one
@pytest.mark.parametrize("case", ["tiny_vo", "tiny_vi", "small_const", "unified_equi", "pgo", "tol_vo"])
def test_group_of_one_is_bitwise_the_single_solve(ctx, case):
    p, kw, n = _case(case)
    ref = O.solve(ctx, p, n, **kw)
    with _Grp(1) as g:
        for peer in (False, True):
            _assert_bitwise(O.solve_group(g, p, n, peer_path=peer, **_solve_kw(kw)), ref, f"group of 1, peer {peer}")


def test_group_of_one_gba_is_bitwise_cvb_gba(ctx):
    p = synth_map.make_map(seed=21, n_agents=2, kf_per_agent=20, n_lm=600, outlier_frac=0.02)
    ref = O.global_bundle_adjustment(ctx, p, iterations_limit=4)
    with _Grp(1) as g:
        got = O.global_bundle_adjustment_group(g, p, iterations_limit=4)
    _assert_bitwise(got, ref, "gba group of 1")
    assert np.array_equal(got["obs_removed"], ref["obs_removed"])


# ---------------------------------------------------------------------------------------------- sharded groups
GROUP_CASES = [(2, c) for c in ("tiny_vo", "tiny_vi", "clean2_const", "tol_vo", "c1_vi")] + \
              [(3, c) for c in ("tiny_vi", "clean2_const")]
_single = {}


def _single_run(ctx, case):
    if case not in _single:
        p, kw, n = _case(case)
        _single[case] = (p, kw, n, O.solve(ctx, p, n, **kw))
    return _single[case]


# The rank-order sum is not gloo's order: on the 24-keyframe tiny maps a few weakly observed landmarks amplify the
# difference to 1.3e-8 and the cost to 1.2e-10 (tiny_vi, world 3; poses and speed-biases stay below 1e-12, measured on an
# H100), so they get 1e-7 / 1e-9.  Every other state keeps the sharded tests' 1e-8 / 1e-10.
TINY_LM_TOL, TINY_COST_TOL = 1e-7, 1e-9


def _check_sharded(p, one, got, world, c1=False, lm_tol=None, cost_tol=None):
    assert got["iterations"] == one["iterations"], (got["iterations"], one["iterations"])
    assert got["steps"] == one["steps"], (got["steps"], one["steps"])
    assert got["termination"] == one["termination"]
    inc = one["lm_owner"] >= 0
    owner = np.full(len(inc), -1); owner[inc] = O.lm_owner_of_rank(int(inc.sum()), world)
    assert np.array_equal(got["lm_owner"], owner)
    well = inc & (np.abs(one["lm"]).max(1) < 100.0) if c1 else inc
    state_tol, cost_tol_default = (1e-6, 1e-6) if c1 else (1e-8, 1e-10)
    e = dict(pose=_rel(got["pose"], one["pose"]), sb=_rel(got["speedbias"], one["speedbias"]),
             lm=_rel(got["lm"][well], one["lm"][well]), cost=np.abs(got["cost"] / one["cost"] - 1).max())
    assert np.array_equal(got["lm"][~inc], np.asarray(p["lm"], np.float64)[~inc])
    return e, state_tol, cost_tol or cost_tol_default, lm_tol or state_tol


@pytest.mark.parametrize("layout,peer", PATHS)
@pytest.mark.parametrize("world,case", GROUP_CASES)
def test_group_solve_matches_world_one(ctx, world, case, layout, peer):
    _need_devices(layout, world)
    p, kw, n, one = _single_run(ctx, case)
    with _Grp(world, layout) as g:
        got = O.solve_group(g, p, n, peer_path=peer, **_solve_kw(kw))
    if case == "clean2_const":
        inc = one["lm_owner"] >= 0
        assert len(p["loop_i"]) > 0                                 # loop edges are dealt across the ranks
        if world == 3:
            assert int(inc.sum()) % 3 != 0                          # the last round of landmark blocks is incomplete
    e, st, ct, lt = _check_sharded(p, one, got, world, c1=case == "c1_vi",
                                   **(dict(lm_tol=TINY_LM_TOL, cost_tol=TINY_COST_TOL) if case.startswith("tiny") else {}))
    print(f"[group] world {world} {case} {layout} peer {peer}: " + ", ".join(f"{k} {v:.3e}" for k, v in e.items()))
    assert e["pose"] < st and e["sb"] < st and e["lm"] < lt and e["cost"] < ct


@pytest.mark.parametrize("layout,peer", PATHS)
def test_group_solve_is_deterministic(ctx, layout, peer):
    p, kw, n, one = _single_run(ctx, "clean2_const")
    world = 3 if layout == "shared" else 2
    with _Grp(world, layout) as g:
        a = O.solve_group(g, p, n, peer_path=peer, **_solve_kw(kw))
        b = O.solve_group(g, p, n, peer_path=peer, **_solve_kw(kw))
    _assert_bitwise(b, a, "second run")
    e, st, ct, lt = _check_sharded(p, one, a, world)
    assert e["pose"] < st and e["sb"] < st and e["lm"] < lt and e["cost"] < ct


# ---------------------------------------------------------------------------------------------- the collective alone
CH = O.GROUP_ALLREDUCE_CHUNK


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("n", [1, 2, 3])
def test_group_allreduce_is_the_rank_order_sum(layout, n):
    rng = np.random.default_rng(n)
    with _Grp(n, layout) as g:
        for count in (0, 1, 7, 1001, CH - 1, CH, CH + 1, 2 * CH + 3):
            # mixed magnitudes and signs: a different summation order changes the last bits
            x = rng.standard_normal((n, count)) * 10.0 ** rng.integers(-8, 9, (n, count))
            ref = x[0].copy()
            for q in range(1, n):
                ref = ref + x[q]
            out = g.allreduce_diag(x)
            for r in range(n):
                assert np.array_equal(out[r].view(np.uint64), ref.view(np.uint64)), (count, r)


# ---------------------------------------------------------------------------------------------- group GBA
TH = 0.92


def _gba_map():
    return synth_map.make_map(seed=21, n_agents=2, kf_per_agent=20, n_lm=600, outlier_frac=0.02)


@pytest.mark.parametrize("layout,peer", PATHS)
@pytest.mark.parametrize("world", [2, 3])
def test_group_gba_matches_cvb_gba(ctx, world, layout, peer):
    _need_devices(layout, world)
    p = _gba_map()
    # round 1 on one context: every norm must stay clear of the threshold, so summation order cannot move an observation
    n = len(p["loop_i"])
    e1 = dict(i=p["loop_i"], j=p["loop_j"], q=p["loop_q"], t=p["loop_t"],
              sqrt_info=np.tile(O.GBA_LOOP_SQRT_INFO[None], (n, 1, 1)), robust=np.zeros(n, np.uint8))
    s = O.BaSolver(ctx, p, visual_only=False, edges=e1)
    try:
        s.iterate(5)
        norms = s.reproj_norms()
    finally:
        s.close()
    used = norms != -1.0
    margin = np.abs(norms[used] - TH).min()
    print(f"[group gba] round-1 norms: {int((norms[used] > TH).sum())} above {TH}, margin {margin:.3e}")
    assert margin >= 1e-6
    ref = O.global_bundle_adjustment(ctx, p, iterations_limit=4, th_outlier=TH)
    assert ref["obs_removed"].any()
    with _Grp(world, layout) as g:
        got = O.global_bundle_adjustment_group(g, p, iterations_limit=4, th_outlier=TH, peer_path=peer)
    assert np.array_equal(got["obs_removed"], ref["obs_removed"])
    e, st, ct, lt = _check_sharded(p, ref, got, world)
    print(f"[group gba] world {world} {layout} peer {peer}: " + ", ".join(f"{k} {v:.3e}" for k, v in e.items()))
    assert e["pose"] < st and e["sb"] < st and e["lm"] < lt and e["cost"] < ct


# ---------------------------------------------------------------------------------------------- refusals, failures
def test_group_create_refusals(ctx):
    lib = covins_b200.lib()
    import ctypes as C
    c2 = covins_b200.Context(0)
    try:
        t0 = _threads()
        h = C.c_void_p()
        for handles, n in (([], 0), ([ctx.handle] * 17, 17), ([ctx.handle, None], 2), ([ctx.handle, c2.handle, ctx.handle], 3)):
            arr = (C.c_void_p * max(len(handles), 1))(*handles)
            assert lib.cvb_group_create(arr, n, C.byref(h)) == 1, n
            assert not h.value
        assert b"same context" in lib.cvb_last_error(ctx.handle)
        assert _threads() == t0
    finally:
        c2.close()


def test_group_refuses_malformed_problem_and_survives_failure(ctx):
    p, kw, n = _case("tiny_vi")
    bad_edges = dict(i=np.array([0], np.int32), j=np.array([p["K"]], np.int32), q=np.array([[0, 0, 0, 1.0]]),
                     t=np.zeros((1, 3)), sqrt_info=np.eye(6)[None], robust=np.zeros(1, np.uint8))
    with pytest.raises(covins_b200.CvbError) as single:
        O.solve(ctx, p, n, edges=bad_edges, **kw)
    with _Grp(2) as g:
        t0 = _threads()
        launches = [c.launch_count() for c in g.contexts]
        with pytest.raises(covins_b200.CvbError) as grp:
            O.solve_group(g, p, n, edges=bad_edges, **kw)
        assert str(grp.value) == str(single.value)                  # same status, same message
        assert [c.launch_count() for c in g.contexts] == launches    # refused before any launch
        assert _threads() == t0
        # the peer path needs a device per rank: refused before any launch
        for call in (lambda: O.solve_group(g, p, n, peer_path=True, **kw),
                     lambda: O.global_bundle_adjustment_group(g, p, iterations_limit=2, peer_path=True)):
            with pytest.raises(covins_b200.CvbError) as shared:
                call()
            assert "status 3" in str(shared.value) and "share device" in str(shared.value), str(shared.value)
        assert [c.launch_count() for c in g.contexts] == launches
        assert _threads() == t0
        # a failure inside the ranks (the engine refuses a singular IMU covariance on every rank)
        with pytest.raises(covins_b200.CvbError) as failed:
            O.solve_group(g, singular_imu(), 3, visual_only=False)
        assert "status 4" in str(failed.value) and "rank" in str(failed.value), str(failed.value)
        assert _threads() == t0
        # the group is usable after a failure
        _, _, _, one = _single_run(ctx, "tiny_vi")
        e, st, ct, lt = _check_sharded(p, one, O.solve_group(g, p, 6, visual_only=False), 2,
                                       lm_tol=TINY_LM_TOL, cost_tol=TINY_COST_TOL)
        assert e["pose"] < st and e["sb"] < st and e["lm"] < lt and e["cost"] < ct
        assert _threads() == t0


# ---------------------------------------------------------------------------------------------- C++ shim
def test_shim_context_group_gba_matches_single_context(tmp_path):
    exe = str(tmp_path / "shim_group_test")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-o", exe,
                           os.path.join(ROOT, "tests", "cpp", "shim_group_test.cpp"), "-L" + os.path.join(ROOT, "covins_b200"),
                           "-lcovins_b200", "-Wl,-rpath," + os.path.join(ROOT, "covins_b200")])
    p = _gba_map()   # its round-1 norms stay >= 1e-6 from the threshold (test_group_gba_matches_cvb_gba asserts it)
    for k, v in p.items():
        if isinstance(v, np.ndarray):
            np.ascontiguousarray(v).tofile(str(tmp_path / (k + ".bin")))
    subprocess.check_call([exe, str(tmp_path), "single", "1", "0"])
    single = {k: np.fromfile(tmp_path / f"single_{k}.bin") for k in ("pose", "sb", "lm")}
    for peer in (0,):   # two ranks on device 0: the all-reduce path (the shim's default)
        subprocess.check_call([exe, str(tmp_path), "group", "2", str(peer)])
        group = {k: np.fromfile(tmp_path / f"group_{k}.bin") for k in ("pose", "sb", "lm")}
        assert np.array_equal(np.fromfile(tmp_path / "group_nobs.bin", np.int32), np.fromfile(tmp_path / "single_nobs.bin", np.int32))
        e = {k: _rel(group[k], single[k]) for k in single}
        print(f"[shim group] peer {peer}: " + ", ".join(f"{k} {v:.3e}" for k, v in e.items()))
        assert max(e.values()) < 1e-8, e
