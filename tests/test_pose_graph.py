"""Optimization::PoseGraphOptimization with its write-back in one call (cvb_pgo, covins_b200/csrc/pgo.cu).

CPU: oracle/pgo.py against the edge list of oracle/ba_oracle.py and against an independent einsum restatement of the
write-back; hand cases pin each rule of the edge construction and of the landmark erasure.
GPU: cvb_pgo's solve is bitwise cvb_ba_solve fed the oracle's edges and start poses, and its write-back is bitwise the
oracle's; the C++ shim on mock containers leaves the same container state as the composition it replaced."""
import os
import subprocess

import numpy as np
import pytest

from covins_b200 import optimization as O, synth_map
from oracle import ba_oracle as bo
from oracle import pgo as ora

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def small_map(seed=5, **kw):
    return synth_map.make_map(seed=seed, n_agents=3, kf_per_agent=40, n_lm=300, drift_trans=0.01, drift_yaw_deg=0.1, **kw)


def rot(rng):
    q = rng.normal(size=4)
    return synth_map.quat_to_rot(q / np.linalg.norm(q))


def spd(rng):
    A = rng.normal(size=(6, 6))
    return A @ A.T * 1e-2 + np.eye(6) * 1e-3


def chain(kf_id, agent, seed=0, n_lm=40):
    """a hand-made map: keyframes listed agent by agent, poses on a curve, every landmark seen by two keyframes"""
    rng = np.random.default_rng(seed)
    K = len(kf_id)
    pose = np.zeros((K, 7))
    for k in range(K):
        pose[k, :4] = synth_map.rot_to_quat(synth_map.rot_exp(rng.normal(size=3) * 0.2))
        pose[k, 4:] = [0.5 * kf_id[k], 0.1 * kf_id[k] ** 2, agent[k]]
    obs_kf = np.sort(rng.integers(0, K, (n_lm, 2)), 1)
    obs_kf[:, 1] = np.where(obs_kf[:, 1] == obs_kf[:, 0], (obs_kf[:, 0] + 1) % K, obs_kf[:, 1])
    obs_kf = np.sort(obs_kf, 1)
    return dict(K=K, L=n_lm, pose=pose, pose_const=(np.asarray(kf_id) == 0).astype(np.uint8), agent_of=np.asarray(agent, np.int32),
                kf_id=np.asarray(kf_id, np.int32), extr=np.array([[0, 0, 0, 1.0, 0, 0, 0]]), lm=rng.normal(size=(n_lm, 3)) * 5,
                lm_obs_ptr=np.arange(0, 2 * n_lm + 1, 2, dtype=np.int32), obs_kf=obs_kf.reshape(-1).astype(np.int32),
                speedbias=rng.normal(size=(K, 9)), loop_i=np.zeros(0, np.int32), loop_j=np.zeros(0, np.int32),
                loop_q=np.zeros((0, 4)), loop_t=np.zeros((0, 3)), loop_cov=np.zeros((0, 6, 6)))


def add_loops(p, pairs, seed=1):
    rng = np.random.default_rng(seed)
    n = len(pairs)
    p.update(loop_i=np.array([a for a, _ in pairs], np.int32), loop_j=np.array([b for _, b in pairs], np.int32),
             loop_q=np.stack([synth_map.rot_to_quat(rot(rng)) for _ in range(n)]), loop_t=rng.normal(size=(n, 3)),
             loop_cov=np.stack([spd(rng) for _ in range(n)]))
    return p


def perturb_vio(pr, seed=3):
    rng = np.random.default_rng(seed)
    T = pr["T_ws"].copy()
    for k in range(len(T)):
        T[k, :3, :3] = synth_map.rot_exp(rng.normal(size=3) * 0.01) @ T[k, :3, :3]
        T[k, :3, 3] += rng.normal(size=3) * 0.05
    return T


# ------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("covins_mode", [True, False])
def test_oracle_edges_equal_ba_oracle_pgo_edges(covins_mode):
    p = small_map()
    if not covins_mode:
        p["loop_cov"] = np.stack([spd(np.random.default_rng(l)) for l in range(len(p["loop_i"]))])
    pr = O.pgo_map_problem(p, covins_mode=covins_mode)
    got = ora.pgo_edges(pr)
    ref = bo.pgo_edges(p, p["pose"], covins_mode=covins_mode)
    assert len(p["loop_i"]) > 0
    assert np.array_equal(got["i"], ref["i"]) and np.array_equal(got["j"], ref["j"])
    assert np.array_equal(got["robust"], ref["robust"].astype(bool))
    nl = len(p["loop_i"])
    kind = got["kind"]
    assert (kind[:nl] == ora.EDGE_LOOP).all() and (kind[nl:] != ora.EDGE_LOOP).all()
    if covins_mode:
        assert np.array_equal(got["sqrt_info"], ref["sqrt_info"])
    else:
        assert np.array_equal(got["sqrt_info"][nl:], ref["sqrt_info"][nl:])
        assert np.abs(got["sqrt_info"][:nl] - ref["sqrt_info"][:nl]).max() <= 1e-12 * np.abs(ref["sqrt_info"][:nl]).max()
    # the measured rotations are the same matrices; ba_oracle turns them into quaternions through sqrt(1 +- ...) / 2, which
    # loses relative accuracy on a small component (its error is ~eps / |q_c|), so the quaternions agree to 1e-15 / |q_c|
    Tv = pr["T_ws_vio"]
    Rv = bo._quat_to_rot_np(p["pose"][:, :4])
    R_got = ora.rel_transform(Tv[got["i"][nl:]], Tv[got["j"][nl:]])[:, :3, :3]
    R_ref = np.einsum("nji,njk->nik", Rv[ref["i"][nl:]], Rv[ref["j"][nl:]])
    assert np.abs(R_got - R_ref).max() <= 1e-15
    sign = np.sign((got["q"] * ref["q"]).sum(1))[:, None]
    assert (np.abs(got["q"] - sign * ref["q"]) * np.abs(ref["q"]) <= 1e-15).all()
    assert np.abs(got["t"] - ref["t"]).max() <= 1e-15 * np.abs(ref["t"]).max()


def einsum_writeback(pr, pose7):
    Tu, Tc = pr["T_ws"], ora.pose7_to_transform(pose7)
    v = np.einsum("krx,kcx,kc->kr", Tc[:, :3, :3], Tu[:, :3, :3], pr["velocity"])
    ref = pr["lm_ref"]
    ok = ref >= 0
    A, C = Tu[ref[ok]], Tc[ref[ok]]
    ps = np.einsum("lcr,lc->lr", A[:, :3, :3], pr["lm_pos"][ok] - A[:, :3, 3])
    lm = pr["lm_pos"].copy()
    lm[ok] = np.einsum("lrc,lc->lr", C[:, :3, :3], ps) + C[:, :3, 3]
    # the scale of an entry: the sum of its products' magnitudes (a cancelling sum has no ulp of its own)
    sv = np.einsum("krx,kcx,kc->kr", np.abs(Tc[:, :3, :3]), np.abs(Tu[:, :3, :3]), np.abs(pr["velocity"]))
    sps = np.einsum("lcr,lc->lr", np.abs(A[:, :3, :3]), np.abs(pr["lm_pos"][ok] - A[:, :3, 3]))
    sl = np.einsum("lrc,lc->lr", np.abs(C[:, :3, :3]), sps) + np.abs(C[:, :3, 3])
    return v, lm, sv, sl, ok


def test_writeback_matches_einsum():
    rng = np.random.default_rng(7)
    for s in range(10):
        p = chain(list(range(30)), [0] * 30, seed=s, n_lm=200)
        p["lm"] *= 10.0 ** (s % 4)
        pr = O.pgo_map_problem(p)
        pr["lm_ref"][::7] = -1
        pose7 = np.concatenate([np.stack([synth_map.rot_to_quat(rot(rng)) for _ in range(30)]), rng.normal(size=(30, 3)) * 10], 1)
        wb = ora.writeback(pr, pose7)
        v, lm, sv, sl, ok = einsum_writeback(pr, pose7)
        # a velocity entry nests one 3-term sum of products inside another (R_c R_u^T first, then times v): twice the
        # rounding steps of a landmark entry, so twice the bound
        assert (np.abs(wb["velocity_out"] - v) <= 4 * np.spacing(sv)).all()
        assert (np.abs(wb["lm_out"][ok] - lm[ok]) <= 2 * np.spacing(sl)).all()
        assert np.array_equal(bits(wb["lm_out"][~ok]), bits(pr["lm_pos"][~ok]))
        assert np.array_equal(wb["T_ws_out"].reshape(-1, 4, 4), ora.pose7_to_transform(pose7))


def test_oracle_conversions_round_trip():
    rng = np.random.default_rng(8)
    for _ in range(200):
        q = synth_map.rot_to_quat(rot(rng))
        p7 = np.concatenate([q, rng.normal(size=3)])
        T = ora.pose7_to_transform(p7)[0]
        back = ora.transform_to_pose7(T)
        s = np.sign(back[:4] @ q)
        assert np.abs(back[:4] - s * q).max() < 1e-15 * 4 and np.array_equal(back[4:], p7[4:])
    A = spd(rng)
    S = ora.sqrt_info_from_cov(A)
    assert np.allclose(S, np.linalg.cholesky(np.linalg.inv(A)).T, rtol=1e-10, atol=1e-12)
    assert ora.sqrt_info_from_cov(-np.eye(6)) is None


def hand_cases():
    """name -> (problem dict of pgo_map_problem, options): each pins one rule"""
    cases = {}
    # duplicate pairs: keyframe 4's successor is its predecessor, so the neighbour walk meets a pair already inserted
    p = chain(list(range(6)), [0] * 6)
    pr = O.pgo_map_problem(p)
    pr["kf_succ"][4] = 3
    cases["duplicate_pairs"] = (pr, {})
    # id gaps after culling (the walk counts steps by id, the links skip the culled keyframes)
    ids = [0, 1, 2, 3, 4, 5, 6, 9, 10, 14, 15, 21]
    cases["id_gaps"] = (O.pgo_map_problem(chain(ids, [0] * len(ids))), {})
    # agents with one keyframe
    cases["single_keyframe_agents"] = (O.pgo_map_problem(add_loops(chain([0, 0, 1, 2, 3, 0], [0, 1, 1, 1, 1, 2]), [(0, 3), (5, 4)])), {})
    cases["no_neighbours"] = (O.pgo_map_problem(chain(list(range(10)), [0] * 10)), dict(use_nbr=False))
    loops = add_loops(chain(list(range(12)), [0] * 12), [(0, 11), (1, 10), (2, 9)])
    cases["covins_loops"] = (O.pgo_map_problem(loops, covins_mode=True), {})
    cases["covins_g_loops"] = (O.pgo_map_problem(loops, covins_mode=False), dict(use_robust=False))
    # the three erase cases: no reference with observations, no reference without, a reference outside the keyframes
    p = chain(list(range(8)), [0] * 8, n_lm=12)
    pr = O.pgo_map_problem(p)
    pr["lm_ref"][:3] = -1; pr["lm_has_obs"][1] = 0; pr["lm_ref"][3:5] = -2
    cases["landmark_erase"] = (pr, {})
    p = chain(list(range(10)), [0] * 10)
    pr = O.pgo_map_problem(p)
    pr["T_ws_init"] = perturb_vio(pr, seed=4)
    pr["T_ws_vio"] = perturb_vio(pr, seed=5)
    cases["init_and_vio_differ"] = (pr, {})
    return cases


def test_hand_case_topologies():
    c = hand_cases()
    topo = lambda name, **kw: [(a, b, k) for a, b, k in ora.edge_topology(c[name][0], **kw)]
    S1, S23, S45 = ora.EDGE_S1, ora.EDGE_S23, ora.EDGE_S45
    # keyframe 4 (id 4): successor edge (4, 3), then its walk reaches 3 (skipped), 2 and 1
    t = topo("duplicate_pairs")
    assert [e for e in t if e[0] == 4] == [(4, 3, S1), (4, 2, S23), (4, 1, S23)]
    # id 21 at index 11: five steps back through the links, whatever the ids
    t = topo("id_gaps")
    assert [e for e in t if e[0] == 11 and e[1] != 11 and e[1] < 11][-5:] == [(11, 10, S1), (11, 9, S23), (11, 8, S23), (11, 7, S45), (11, 6, S45)]
    # index 3 has id 3: two steps (3 - j > 0 for j = 1, 2)
    assert [e for e in t if e[0] == 3 and e[1] < 3] == [(3, 2, S1), (3, 1, S23)]
    t = topo("single_keyframe_agents")
    assert t[:2] == [(0, 3, ora.EDGE_LOOP), (5, 4, ora.EDGE_LOOP)] and not any(e[0] in (0, 5) and e[2] != ora.EDGE_LOOP for e in t)
    t = topo("no_neighbours", use_nbr=False)
    assert t == [(k, k + 1, S1) for k in range(9)]
    pr = c["covins_g_loops"][0]
    e = ora.pgo_edges(pr, use_robust=False)
    assert not e["robust"].any() and np.allclose(e["sqrt_info"][0], np.linalg.cholesky(np.linalg.inv(pr["loop_cov"][0])).T)
    e = ora.pgo_edges(c["covins_loops"][0])
    assert e["robust"][:3].all() and not e["robust"][3:].any() and np.array_equal(e["sqrt_info"][0], ora.weights()[0])
    pr = c["landmark_erase"][0]
    wb = ora.writeback(pr, ora.start_poses(pr))
    assert wb["lm_erase"].tolist()[:5] == [1, 0, 1, 1, 1] and not wb["lm_erase"][5:].any()
    assert np.array_equal(bits(wb["lm_out"][:5]), bits(pr["lm_pos"][:5]))
    pr = c["init_and_vio_differ"][0]
    assert not np.array_equal(ora.start_poses(pr), ora.start_poses(dict(pr, T_ws_init=None)))


def refusals():
    """name -> (problem, message fragment): input the parent shim threw on or dereferenced null for, and invalid input"""
    out = {}
    base = O.pgo_map_problem(chain(list(range(8)), [0] * 8))
    pr = dict(base, kf_succ=base["kf_succ"].copy()); pr["kf_succ"][3] = -2
    out["successor_outside"] = (pr, "successor")
    pr = dict(base, kf_pred=base["kf_pred"].copy()); pr["kf_pred"][4] = -1
    out["walk_needs_absent_predecessor"] = (pr, "neighbour")
    pr = dict(base, kf_pred=base["kf_pred"].copy()); pr["kf_pred"][2] = -2
    out["walk_through_culled_keyframe"] = (pr, "neighbour")
    pr = O.pgo_map_problem(chain([0, 1, 4], [0] * 3))           # id 4 wants three predecessors, the chain has two
    out["id_gap_too_early"] = (pr, "neighbour")
    pr = O.pgo_map_problem(add_loops(chain(list(range(8)), [0] * 8), [(2, 2)]))
    out["loop_to_itself"] = (pr, "loop 0")
    pr = O.pgo_map_problem(add_loops(chain(list(range(8)), [0] * 8), [(1, 6), (2, 5)]), covins_mode=False)
    pr["loop_cov"][1] = -np.eye(6)
    out["covariance_not_positive_definite"] = (pr, "loop 1")
    pr = dict(base, T_ws=base["T_ws"].copy()); pr["T_ws"][2, 0, 3] = np.nan
    out["non_finite_pose"] = (pr, "finite")
    pr = dict(base, lm_ref=base["lm_ref"].copy()); pr["lm_ref"][0] = 8
    out["landmark_reference_out_of_range"] = (pr, "lm_ref")
    return out


@pytest.mark.parametrize("name", ["successor_outside", "walk_needs_absent_predecessor", "walk_through_culled_keyframe", "id_gap_too_early",
                                  "loop_to_itself", "covariance_not_positive_definite"])
def test_oracle_refuses(name):
    pr, msg = refusals()[name]
    with pytest.raises(ora.Refused):
        ora.edge_topology(pr)


def test_shim_pgo_compiles_and_refuses_missing_input(tmp_path):
    exe = str(tmp_path / "shim_pgo_test")
    _build_shim(exe)
    assert subprocess.run([exe, str(tmp_path)]).returncode == 2     # nothing dumped: refused before any GPU work


def _build_shim(exe):
    import covins_b200
    if not os.path.exists(covins_b200.LIB_PATH):
        covins_b200.build()
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-o", exe, os.path.join(ROOT, "tests", "cpp", "shim_pgo_test.cpp"),
                           "-L" + os.path.join(ROOT, "covins_b200"), "-lcovins_b200", "-Wl,-rpath," + os.path.join(ROOT, "covins_b200")])


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------
def _reference(ctx, pr, opts):
    """cvb_ba_solve fed the oracle's edges and start poses, then the oracle's write-back of its poses"""
    wt = opts.get("wt", (10.0, 1.0, 10.0, 2.0, 3.0))
    edges = ora.pgo_edges(pr, wt=wt, use_nbr=opts.get("use_nbr", True), use_robust=opts.get("use_robust", True))
    K = len(pr["kf_id"])
    pp = dict(K=K, pose=ora.start_poses(pr), pose_const=pr["pose_const"], extr=np.array([[0, 0, 0, 1.0, 0, 0, 0]]))
    sol = O.pose_graph_optimization(ctx, pp, edges, iterations=opts.get("iterations", 10), robust_th=opts.get("robust_th", 0.5))
    return edges, sol, ora.writeback(pr, sol["pose"])


def _check(ctx, pr, opts=None):
    opts = opts or {}
    edges, sol, wb = _reference(ctx, pr, opts)
    l0 = ctx.launch_count()
    got = O.pose_graph_optimization_map(ctx, pr, **opts)
    n_pgo = ctx.launch_count() - l0
    assert got["n_edge"] == len(edges["i"])
    assert np.array_equal(bits(got["pose"]), bits(sol["pose"]))
    assert np.array_equal(bits(got["cost"]), bits(sol["cost"])) and got["steps"] == sol["steps"]
    assert got["iterations"] == sol["iterations"] and got["termination"] == sol["termination"]
    assert np.array_equal(bits(got["T_ws"].reshape(-1, 16)), bits(wb["T_ws_out"]))
    if pr.get("velocity") is not None:
        assert np.array_equal(bits(got["velocity"]), bits(wb["velocity_out"]))
    assert np.array_equal(bits(got["lm"]), bits(wb["lm_out"]))
    assert np.array_equal(got["lm_erase"], wb["lm_erase"].astype(bool))
    return got, sol, n_pgo


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["C1", "C2", "C3"])
def test_cvb_pgo_is_bitwise_the_solve_and_the_oracle(ctx, config):
    p = synth_map.make_config(config)
    pr = O.pgo_map_problem(p)
    pr["T_ws_vio"] = perturb_vio(pr)       # the chain's measurements differ from the start poses
    got, sol, _ = _check(ctx, pr)
    assert np.abs(got["pose"][:, 4:] - ora.start_poses(pr)[:, 4:]).max() > 1e-4   # it moved


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(hand_cases()))
def test_cvb_pgo_hand_cases(ctx, name):
    pr, opts = hand_cases()[name]
    _check(ctx, pr, opts)


@pytest.mark.gpu
def test_cvb_pgo_repeats_and_launches_two_kernels_besides_the_solve(ctx):
    p = small_map()
    pr = O.pgo_map_problem(p)
    pr["T_ws_vio"] = perturb_vio(pr)
    edges = ora.pgo_edges(pr)
    pp = dict(K=len(pr["kf_id"]), pose=ora.start_poses(pr), pose_const=pr["pose_const"], extr=np.array([[0, 0, 0, 1.0, 0, 0, 0]]))
    l0 = ctx.launch_count()
    O.pose_graph_optimization(ctx, pp, edges)
    n_solve = ctx.launch_count() - l0
    a, _, n_pgo = _check(ctx, pr)
    b = O.pose_graph_optimization_map(ctx, pr)
    assert n_pgo == n_solve + 2
    for k in ("pose", "T_ws", "velocity", "lm", "cost"):
        assert np.array_equal(bits(a[k]), bits(b[k])), k
    # the same map with ten times the landmarks: the same launches
    big = synth_map.make_map(seed=5, n_agents=3, kf_per_agent=40, n_lm=3000, drift_trans=0.01, drift_yaw_deg=0.1)
    prb = O.pgo_map_problem(big)
    prb["T_ws_vio"] = pr["T_ws_vio"]
    l0 = ctx.launch_count()
    O.pose_graph_optimization_map(ctx, prb)
    assert ctx.launch_count() - l0 == n_pgo


@pytest.mark.gpu
def test_cvb_pgo_without_landmarks_or_velocities(ctx):
    p = chain(list(range(10)), [0] * 10, n_lm=0)
    pr = O.pgo_map_problem(p)
    got, _, _ = _check(ctx, pr)
    assert got["lm"].shape == (0, 3) and got["lm_erase"].shape == (0,)
    got, _, _ = _check(ctx, dict(pr, velocity=None))
    assert got["velocity"] is None


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(refusals()))
def test_cvb_pgo_refusals_launch_nothing(ctx, name):
    from covins_b200._lib import CvbError
    pr, msg = refusals()[name]
    l0 = ctx.launch_count()
    with pytest.raises(CvbError, match=msg):
        O.pose_graph_optimization_map(ctx, pr)
    assert ctx.launch_count() == l0


def _dump(d, p, **extra):
    for k, v in dict(p, **extra).items():
        if isinstance(v, np.ndarray):
            np.ascontiguousarray(v).tofile(os.path.join(d, k + ".bin"))


@pytest.mark.gpu
def test_shim_leaves_the_containers_as_the_replaced_composition(tmp_path):
    exe = str(tmp_path / "shim_pgo_test")
    _build_shim(exe)
    rng = np.random.default_rng(11)
    # the PGO map of test_shim.py, with VIO poses, corrected start poses for some keyframes and every landmark-erase case
    p = synth_map.make_map(seed=5, n_agents=3, kf_per_agent=40, n_lm=50, drift_trans=0.01, drift_yaw_deg=0.1)
    pr = O.pgo_map_problem(p)
    vio = np.stack([ora.transform_to_pose7(T) for T in perturb_vio(pr)])
    init = np.stack([ora.transform_to_pose7(T) for T in perturb_vio(pr, seed=9)])
    ref_mode = rng.integers(0, 4, p["L"]).astype(np.int32)
    ref_mode[:10] = 0
    cov = {k: v for k, v in p.items() if k != "loop_cov"}
    d1 = tmp_path / "covins"
    d1.mkdir()
    _dump(str(d1), cov, pose_vio=vio, pose_init=init, init_mask=(np.arange(p["K"]) % 3 == 0).astype(np.uint8), lm_ref_mode=ref_mode)
    out = subprocess.run([exe, str(d1)], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "differing=0" in out.stdout and "erased=0" not in out.stdout
    # the COVINS_G chain of shim_relpose_cov_test: twelve keyframes, loops i <-> 11 - i whitened by their covariances
    c = add_loops(chain(list(range(12)), [0] * 12, n_lm=30), [(i, 11 - i) for i in range(6)], seed=12)
    d2 = tmp_path / "covins_g"
    d2.mkdir()
    _dump(str(d2), c)
    out = subprocess.run([exe, str(d2)], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "covins=0" in out.stdout and "differing=0" in out.stdout
