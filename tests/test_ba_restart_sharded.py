"""The bundle adjustment's restart and landmark-sharded paths against the fresh single-rank solve.

  (a) cvb_ba_restart returns to the state the problem was created with: create → iterate, restart → iterate and two
      restarts in a row → iterate all repeat a fresh O.solve bit for bit, and so does a world = 1 BaSolver with an
      all-reduce installed (it restarts inside __init__, like every multi-GPU solve);
  (b) the Jacobi scale fixed at iteration 0 is 1 / (1 + |column|) of the unscaled Jacobian, after create and after a
      restart: checked against the CPU oracle's Jacobian in extended precision;
  (c) a solve sharded over `world` ranks (landmark blocks c % world, IMU factors and edges dealt round-robin, the reduced
      camera system summed by a host-staged gloo all-reduce) on one GPU equals the world = 1 solve up to summation order.
"""
import datetime
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from covins_b200 import optimization as O
from covins_b200 import synth_map
from oracle import ba_oracle as bo

pytestmark = pytest.mark.gpu
RTOL = 1e-5  # test_gpu_ba.py: final states within 1e-5 relative of the oracle


def _rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-12) if np.size(b) else 0.0


# ---------------------------------------------------------------------------------------------- problems
def _tol_map():
    """noise-free two-agent map: the visual-only solve stops on the function tolerance after 10 of 20 iterations"""
    return synth_map.make_map(seed=3, n_agents=2, kf_per_agent=12, n_lm=300, outlier_frac=0.0, pix_noise=0.0,
                              lm_noise=0.001, drift_trans=0.0005, drift_yaw_deg=0.005)


def _case(name):
    """→ (problem, BaSolver / O.solve keyword arguments, iterations)"""
    if name in ("tiny_vo", "tiny_vi"):
        return synth_map.make_config("tiny"), dict(visual_only=name == "tiny_vo"), 6
    if name == "small_const":    # loaded / GBA-fixed keyframes; some landmarks drop below 2 observations
        p = synth_map.make_config("small")
        p["pose_const"] = p["pose_const"].copy(); p["pose_const"][[3, 7, 20]] = 1
        skip = np.zeros(len(p["obs_kf"]), np.uint8); skip[::7] = 1
        return p, dict(visual_only=False, obs_skip=skip), 4
    if name == "unified_equi":
        p = synth_map.with_camera_model(synth_map.make_config("tiny"), 1, 1, xi=0.9, seed=7)
        return p, dict(visual_only=False), 5
    if name == "pgo":
        p = synth_map.make_map(seed=5, n_agents=3, kf_per_agent=60, n_lm=10, drift_trans=0.01, drift_yaw_deg=0.1)
        pp = dict(K=p["K"], L=0, pose=p["pose"], pose_const=p["pose_const"], extr=p["extr"], cam_of_kf=p.get("cam_of_kf"))
        return pp, dict(visual_only=True, cauchy_reproj=0.0, cauchy_edge=0.5, edges=O.pgo_edges(p, p["pose"])), 10
    if name == "tol_vo":
        return _tol_map(), dict(visual_only=True), 20
    if name == "clean2_const":   # the clean two-agent map of test_single_solve_matches_oracle_small_clean
        p = synth_map.make_map(seed=21, n_agents=2, kf_per_agent=40, n_lm=2000, outlier_frac=0.0)
        p["pose_const"] = p["pose_const"].copy(); p["pose_const"][[3, 7, 20]] = 1
        skip = np.zeros(len(p["obs_kf"]), np.uint8); skip[::7] = 1
        return p, dict(visual_only=False, obs_skip=skip), 8
    if name == "c1_vi":
        return synth_map.make_config("C1"), dict(visual_only=False), 4
    raise KeyError(name)


RESULT_KEYS = ("pose", "speedbias", "lm", "lm_owner", "cost", "steps", "iterations", "termination", "initial_cost",
               "final_cost")


def _assert_bitwise(got, ref, what):
    for k in RESULT_KEYS:
        a, b = got[k], ref[k]
        if isinstance(b, np.ndarray):
            assert a.shape == b.shape and np.array_equal(a, b), f"{what}: {k} differs (max |diff| " \
                f"{np.abs(a - b).max() if a.shape == b.shape and a.size else 'shape'})"
        else:
            assert a == b, f"{what}: {k} {a!r} != {b!r}"


# ---------------------------------------------------------------------------------------------- (a) restart
@pytest.mark.parametrize("case", ["tiny_vo", "tiny_vi", "small_const", "unified_equi", "pgo", "tol_vo"])
def test_restart_repeats_the_solve_bitwise(ctx, case):
    p, kw, n = _case(case)
    fresh = O.solve(ctx, p, n, **kw)
    if case == "tol_vo":
        assert fresh["iterations"] < n and fresh["termination"].startswith("CONVERGENCE"), \
            (fresh["iterations"], fresh["termination"])
    # solvers are closed in `finally`: a failed assertion must not keep an engine alive past the session's context
    s = O.BaSolver(ctx, p, **kw)
    try:
        sc0 = s.debug_vector(0)
        s.iterate(n)
        _assert_bitwise(s.result(), fresh, "create → iterate")
        for restarts in (1, 2):
            for _ in range(restarts):
                s.restart()
            sc = s.debug_vector(0)
            assert np.array_equal(sc[0], sc0[0]) and np.array_equal(sc[1], sc0[1]), \
                f"Jacobi scale after {restarts} restart(s) differs from create: max rel " \
                f"{_rel(np.concatenate(sc), np.concatenate(sc0)):.3e}"
            s.iterate(n)
            _assert_bitwise(s.result(), fresh, f"{restarts} restart(s) → iterate")
    finally:
        s.close()
    # the single-process form of the multi-GPU sequence: create, install the all-reduce, restart (inside __init__)
    s = O.BaSolver(ctx, p, allreduce=lambda user, ptr, count, stream: 0, **kw)
    try:
        s.iterate(n)
        _assert_bitwise(s.result(), fresh, "BaSolver(allreduce=no-op)")
    finally:
        s.close()


# ---------------------------------------------------------------------------------------------- (b) Jacobi scale
# The engine's column norms and the oracle's differ only by the rounding of the analytic vs autograd Jacobian entries
# and of the sums of squares (no cancellation: every term is >= 0), so a few ulp: 1e-9 leaves six orders of margin,
# while a scale computed from an already scaled Jacobian (restart without the mask) is off by O(1).  Measured on an H100:
# at most 5.8e-14.
SCALE_RTOL = 1e-9


@pytest.mark.parametrize("case", ["tiny_vo", "tiny_vi", "small"])
def test_jacobi_scale_matches_extended_precision(ctx, case):
    p = synth_map.make_config("small" if case == "small" else "tiny")
    vo = case == "tiny_vo"
    pr = bo.Problem(p, visual_only=vo, loop_loss=1.0)
    _, _, J, _ = pr.evaluate(pr.pose, pr.sb, pr.lm)
    Jc = J.tocoo()
    colsq = np.zeros(pr.n, np.longdouble)
    np.add.at(colsq, Jc.col, Jc.data.astype(np.longdouble) ** 2)
    ref = np.where(pr.active, 1 / (1 + np.sqrt(colsq)), 0)
    act = pr.active
    s = O.BaSolver(ctx, p, visual_only=vo)
    try:
        for stage in ("create", "restart"):
            if stage == "restart":
                s.iterate(3)
                s.restart()
            c, l = s.debug_vector(0)
            got = np.concatenate([c, l])
            assert got.shape == ref.shape
            assert np.all(got[~act] == 0.0), f"{stage}: inactive columns must have scale 0"
            err = np.abs((got[act] - ref[act]) / ref[act]).max()
            print(f"[jacobi scale] {case} after {stage}: max relative error vs extended precision {float(err):.3e}")
            assert err < SCALE_RTOL, (stage, float(err))
    finally:
        s.close()


# ---------------------------------------------------------------------------------------------- (c) sharded solves
SHARD_CASES = {2: ["tiny_vo", "tiny_vi", "clean2_const", "tol_vo", "c1_vi"], 3: ["tiny_vi", "clean2_const"]}


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _host_allreduce(device):
    """All-reduce callback staged through the host: gloo sums a CPU copy of the engine's buffer.  Works for any number
    of ranks per GPU (NCCL refuses two ranks on one device)."""

    class _Ptr:
        def __init__(self, ptr, n):
            self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f8", "data": (ptr, False), "version": 3}

    def fn(user, ptr, count, stream):
        try:
            ext = torch.cuda.ExternalStream(stream, device=device)
            ext.synchronize()
            with torch.cuda.stream(ext):
                t = torch.as_tensor(_Ptr(ptr, count), device=device)
                h = t.cpu()
                dist.all_reduce(h)
                t.copy_(h)
            ext.synchronize()
            return 0
        except Exception as e:  # never let an exception cross the C boundary
            print("allreduce callback failed:", e, flush=True)
            return 1
    return fn


def _worker(rank, world, port, out_dir, cases):
    import covins_b200
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=300))
    try:
        dev = rank % torch.cuda.device_count()
        ctx = covins_b200.Context(dev)
        out = {}
        for name in cases:
            p, kw, n = _case(name)
            s = O.BaSolver(ctx, p, rank=rank, world=world, allreduce=_host_allreduce(torch.device("cuda", dev)),
                           p2p=False, **kw)
            out[name + ".scale_cam"], out[name + ".scale_lm"] = s.debug_vector(0)
            s.iterate(n)
            r = s.result()
            for k in RESULT_KEYS:
                out[name + "." + k] = np.asarray(r[k])
            out[name + ".norms"] = s.reproj_norms()
            s.close()
        np.savez(os.path.join(out_dir, f"rank{rank}.npz"), **out)
        ctx.close()
    finally:
        dist.destroy_process_group()


def _load_case(npz, name):
    r = {k: npz[name + "." + k] for k in RESULT_KEYS + ("scale_cam", "scale_lm", "norms")}
    for k in ("iterations", "initial_cost", "final_cost"):
        r[k] = r[k].item()
    r["termination"] = str(r["termination"])
    r["steps"] = [str(x) for x in r["steps"]]
    return r


@pytest.fixture(scope="module")
def sharded_runs(tmp_path_factory):
    """world → per-rank results of every case of SHARD_CASES[world]; one spawn per world size"""
    runs = {}

    def get(world):
        if world not in runs:
            d = tmp_path_factory.mktemp(f"world{world}")
            mp.spawn(_worker, args=(world, _free_port(), str(d), SHARD_CASES[world]), nprocs=world, join=True)
            files = [np.load(d / f"rank{r}.npz") for r in range(world)]
            runs[world] = {name: [_load_case(f, name) for f in files] for name in SHARD_CASES[world]}
        return runs[world]
    return get


@pytest.fixture(scope="module")
def single_runs(ctx):
    runs = {}

    def get(name):
        if name not in runs:
            p, kw, n = _case(name)
            s = O.BaSolver(ctx, p, **kw)
            sc = s.debug_vector(0)
            s.iterate(n)
            r = s.result()
            r["scale_cam"], r["scale_lm"] = sc
            r["norms"] = s.reproj_norms()
            s.close()
            runs[name] = (p, kw, r)
        return runs[name]
    return get


@pytest.mark.parametrize("world,case", [(w, c) for w in sorted(SHARD_CASES) for c in SHARD_CASES[w]])
def test_sharded_solve_matches_single_rank(sharded_runs, single_runs, world, case):
    p, kw, one = single_runs(case)
    ranks = sharded_runs(world)[case]
    inc = one["lm_owner"] >= 0
    n_in = int(inc.sum())
    if case == "clean2_const":
        assert len(p["loop_i"]) > 0                            # loop edges are dealt across the ranks
        if world == 3:
            assert n_in % 3 != 0                               # the last round of landmark blocks is incomplete
    # ---- trust-region path: identical decisions
    for r, res in enumerate(ranks):
        assert res["iterations"] == one["iterations"], (r, res["iterations"], one["iterations"])
        assert res["steps"] == one["steps"], (r, res["steps"], one["steps"])
        assert res["termination"] == one["termination"], (r, res["termination"], one["termination"])
        assert np.array_equal(res["pose"], ranks[0]["pose"]) and np.array_equal(res["speedbias"], ranks[0]["speedbias"])
        assert np.array_equal(res["cost"], ranks[0]["cost"])
    # ---- landmark ownership and write-back
    owner = np.full(len(inc), -1); owner[inc] = O.lm_owner_of_rank(n_in, world)
    for r, res in enumerate(ranks):
        assert np.array_equal(res["lm_owner"], owner), r
        assert np.array_equal(res["lm"][owner != r], np.asarray(p["lm"], np.float64)[owner != r]), r
    # ---- Jacobi scale right after the restart
    nc_own = np.arange(n_in) % world
    for r, res in enumerate(ranks):
        assert np.array_equal(res["scale_cam"], ranks[0]["scale_cam"]), r
        own = np.repeat(nc_own == r, 3)
        assert np.array_equal(res["scale_lm"][own], one["scale_lm"][own]), r
        assert np.all(res["scale_lm"][~own] == 0.0), r
    sc, sc1 = ranks[0]["scale_cam"], one["scale_cam"]
    assert np.array_equal(sc == 0, sc1 == 0)
    cam_err = np.max(np.abs(sc - sc1) / np.where(sc1 != 0, sc1, 1.0))
    # ---- merged states vs world = 1 (summation order is the only difference)
    merged = O.merge_sharded_landmarks(ranks)
    c1 = case == "c1_vi"
    well = inc & (np.abs(one["lm"]).max(1) < 100.0) if c1 else inc
    state_tol, cost_tol = (1e-6, 1e-6) if c1 else (1e-8, 1e-10)
    e_pose, e_sb = _rel(merged["pose"], one["pose"]), _rel(merged["speedbias"], one["speedbias"])
    e_lm = _rel(merged["lm"][well], one["lm"][well])
    e_cost = np.abs(merged["cost"] / one["cost"] - 1).max()
    # ---- corrected reprojection norms: -1 on the other ranks' observations; merged = world 1
    obs_lm = np.repeat(np.arange(len(inc)), np.diff(p["lm_obs_ptr"]))
    obs_owner = owner[obs_lm]
    norms = ranks[0]["norms"].copy()
    for r, res in enumerate(ranks):
        assert np.all(res["norms"][obs_owner != r] == -1.0), r
        norms[obs_owner == r] = res["norms"][obs_owner == r]
    def norm_err(m):
        return np.abs(norms[m] - one["norms"][m]).max() / max(np.abs(one["norms"][m]).max(), 1.0)
    e_norms, e_norms_well = norm_err(slice(None)), norm_err(well[obs_lm])
    print(f"[sharded] world {world} {case}: scale cam rel {cam_err:.3e}, pose {e_pose:.3e}, speedbias {e_sb:.3e}, "
          f"lm {e_lm:.3e}, cost {e_cost:.3e}, norms {e_norms:.3e} (well landmarks {e_norms_well:.3e})")
    assert cam_err < 1e-13
    assert e_pose < state_tol and e_sb < state_tol and e_lm < state_tol
    assert e_cost < cost_tol
    # the norms follow the states: on C1 (gross outliers, poorly constrained landmarks) only the well landmarks'
    # observations are held to 1e-9 (measured on an H100: 6.1e-11 there, 4.8e-9 over all observations)
    assert e_norms_well < 1e-9
    if case == "tiny_vi" and world == 2:
        ref = bo.solve(bo.Problem(p, visual_only=False, loop_loss=1.0), 6)
        assert merged["iterations"] == ref["iterations"]
        assert _rel(merged["pose"], ref["pose"].numpy()) < RTOL and _rel(merged["speedbias"], ref["sb"].numpy()) < RTOL
        assert _rel(merged["lm"], ref["lm"].numpy()) < RTOL
