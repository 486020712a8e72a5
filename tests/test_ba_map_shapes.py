"""The bundle adjustment on map shapes that steer the engine's set-up (covins_b200/csrc/ba_engine.cu, engine_setup) into
branches the BASELINE-shaped maps of test_gpu_ba.py never reach, each against the CPU oracle through the public C-ABI:

  cams_mixed          one calibration per agent (cam_of_kf = agent), three projection / distortion models in one map:
                      the per-keyframe gather of extrinsics, intrinsics, distortion and model, and the per-observation
                      model dispatch; plus the corrected residual norms and the cost at x0, held to rounding;
  cams_radtan_gba     per-agent radtan calibrations through GlobalBundleAdjustment, both rounds, vs the compiled port;
  imu_split           IMU chains broken into pieces of 1, 2, 13-17, 21, 22 and 29 keyframes: chains either side of a
                      tile of 14 speed-bias / 21 pose blocks, and keyframes without any IMU factor (isolated blocks);
  const_agent         a whole agent constant (a loaded map) and constant keyframes inside another agent's IMU chain;
  vo_tile_edges       visual-only single-agent maps of 126, 132, 252 and 258 pose columns (either side of a 128-column tile);
  pgo_threshold       a pose graph whose short-range components have 63, 64 and 65 keyframes (nested dissection starts at
                      64) with between-edges of span 8 (stays in the chain) and 9 (both ends go to the border);
  landmark_extremes   a landmark seen by every keyframe, landmarks left with exactly 2 and 1 usable observations, and an
                      observation of a point behind its camera (zero residual block);
  singular_imu        an IMU noise model whose preintegrated covariance is singular is refused, like the oracle does.

Every builder asserts the structural fact its case exists for (computed in Python), so the CPU part of this file checks
that the maps have the shapes they claim; the GPU part solves them."""
import numpy as np
import pytest

import covins_b200
from covins_b200 import optimization as O
from covins_b200 import synth_map as sm
from oracle import ba_oracle as bo
from test_gpu_ba import RTOL, _compare, _port_compare, _rel

TILE = 128                       # cvb_chol::T: columns per tile of the reduced camera system
SB_PER_TILE, POSE_PER_TILE = TILE // 9, TILE // 6   # 14 speed-bias blocks, 21 pose blocks
ND_MIN = 64                      # pose-graph components of at least this many keyframes get nested dissection
BORDER_SPAN = 8                  # edges spanning more keyframes than this put both endpoints on the border

# The corrected norms and the cost at x0 are pure function evaluations of the same formulas in double precision.  A
# pixel coordinate (~500 px) carries a few ulp (~1e-13 px) of rounding, divided by sigma >= 2, so every norm agrees to
# ~1e-13 absolute; relative to max(norm, 0.01) that is <= 1e-11.  The cost is a sum of such non-negative terms in a
# different order (~n eps).  A wrong camera or model for an observation is off by O(1).  Measured on an H100 (700 W):
# norms 1.1e-12, cost 4.4e-16 relative.
NORM_RTOL = 1e-10
COST_RTOL = 1e-12

# pinhole / radtan, unified (xi 0.9) / equidistant, pinhole / FOV
MODELS3 = [(0, 0, 0.0), (1, 1, 0.9), (0, 2, 0.0)]


# ---------------------------------------------------------------------------------------------- helpers
def per_agent_cameras(p, models, seed, pix_noise=1.0):
    """The map observed through one calibration per agent: intrinsics scaled by 0.9-1.1, the extrinsic rotated by ~1 deg
    and shifted by ~1 cm, a (cam_model, dist_model, xi) per agent, cam_of_kf = agent_of.  Inlier observations are
    re-projected from the ground truth through the observing keyframe's own camera (+ pixel noise); gross outliers keep
    their random pixels (as synth_map.with_camera_model does for one camera)."""
    rng = np.random.default_rng(seed)
    agent = np.asarray(p["agent_of"])
    assert len(models) == int(agent.max()) + 1
    R0, t0 = sm.quat_to_rot(p["extr"][0][:4]), p["extr"][0][4:]
    extr, intr, dist = [], [], []
    for _, dm, _ in models:
        R = R0 @ sm.rot_exp(rng.normal(0, np.deg2rad(1.0) / np.sqrt(3), 3))
        extr.append(np.concatenate([sm.rot_to_quat(R), t0 + rng.normal(0, 0.01 / np.sqrt(3), 3)]))
        intr.append(sm.EUROC_INTR * rng.uniform(0.9, 1.1, 4))
        dist.append(np.array(sm.DEFAULT_DIST[dm], float))
    q = dict(p)
    q.update(cam_of_kf=agent.astype(np.int32), extr=np.array(extr), intr=np.array(intr), dist=np.array(dist),
             cam_model=np.array([m[0] for m in models], np.int32), dist_model=np.array([m[1] for m in models], np.int32),
             cam_xi=np.array([m[2] for m in models], float))
    R_ws, t_ws = sm.quat_to_rot(p["gt_pose"][:, :4]), p["gt_pose"][:, 4:]
    obs_lm = np.repeat(np.arange(p["L"]), np.diff(p["lm_obs_ptr"]))
    k = p["obs_kf"]
    ps = np.einsum("nji,nj->ni", R_ws[k], p["gt_lm"][obs_lm] - t_ws[k])
    uv = np.empty((len(k), 2))
    for c, (cm, dm, xi) in enumerate(models):
        m = agent[k] == c
        Rc, tc = sm.quat_to_rot(q["extr"][c][:4]), q["extr"][c][4:]
        uv[m] = sm.project_model((ps[m] - tc) @ Rc, q["intr"][c], q["dist"][c], cm, dm, xi)
    uv += rng.normal(0, pix_noise, uv.shape)
    out = p["obs_is_outlier"]
    uv[out] = p["obs_uv"][out]
    q["obs_uv"] = uv.astype(np.float32)
    return q


def drop_imu(p, factors):
    """The map without the IMU factors `factors` (indices), their raw sample ranges removed with them."""
    keep = np.ones(len(p["imu_i"]), bool)
    keep[np.asarray(factors, np.int64)] = False
    n = np.diff(p["imu_ptr"])
    samples = np.repeat(keep, n)
    q = dict(p)
    q.update(imu_i=p["imu_i"][keep], imu_j=p["imu_j"][keep], imu_acc0=p["imu_acc0"][keep], imu_gyr0=p["imu_gyr0"][keep],
             imu_dt=p["imu_dt"][samples], imu_acc=p["imu_acc"][samples], imu_gyr=p["imu_gyr"][samples],
             imu_ptr=np.concatenate([[0], np.cumsum(n[keep])]).astype(np.int32))
    return q


def _components(K, pairs):
    """connected components of keyframes linked by `pairs`, as sorted member lists in order of their first keyframe"""
    parent = list(range(K))

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x
    for a, b in pairs:
        a, b = find(int(a)), find(int(b))
        if a != b:
            parent[max(a, b)] = min(a, b)
    comps = {}
    for k in range(K):
        comps.setdefault(find(k), []).append(k)
    return [comps[r] for r in sorted(comps)]


def imu_chains(p):
    """lengths of the IMU chains (components of the IMU factor graph, single keyframes included) in keyframe order"""
    return [len(c) for c in _components(p["K"], zip(p["imu_i"], p["imu_j"]))]


def _between_from_gt(p, i, j, rng):
    """T_s1_s2 between keyframes i and j from the ground truth + 1 cm / 0.2 deg noise (as make_map's loop constraints)"""
    R = sm.quat_to_rot(p["gt_pose"][:, :4]); t = p["gt_pose"][:, 4:]
    R12 = R[i].T @ R[j] @ sm.rot_exp(rng.normal(0, np.deg2rad(0.2), 3))
    return sm.rot_to_quat(R12), R[i].T @ (t[j] - t[i]) + rng.normal(0, 0.01, 3)


def _obs_lm(p):
    return np.repeat(np.arange(p["L"]), np.diff(p["lm_obs_ptr"]))


def _camera_z(p, pose, kf, x):
    """depth of world points x [n,3] in the cameras of keyframes kf [n] at `pose`"""
    R, t = sm.quat_to_rot(pose[kf, :4]), pose[kf, 4:]
    cam = np.asarray(p.get("cam_of_kf", np.zeros(p["K"], np.int32)))[kf]
    Rsc, tsc = sm.quat_to_rot(p["extr"][cam, :4]), p["extr"][cam, 4:]
    ps = np.einsum("nji,nj->ni", R, x - t)
    return np.einsum("nji,nj->ni", Rsc, ps - tsc)[:, 2]


def _with_observations(p, lm_new, obs):
    """append landmarks `lm_new` [m,3] (initial = ground truth) and observations `obs` = [(lm, kf, u, v)] (sigma 2, not
    outliers); the CSR stays sorted by (landmark, keyframe)"""
    q = dict(p)
    m = len(lm_new)
    if m:
        q["lm"] = np.concatenate([p["lm"], lm_new]); q["gt_lm"] = np.concatenate([p["gt_lm"], lm_new]); q["L"] = p["L"] + m
    ol = np.concatenate([_obs_lm(p), [o[0] for o in obs]]).astype(np.int64)
    ok = np.concatenate([p["obs_kf"], [o[1] for o in obs]]).astype(np.int64)
    uv = np.concatenate([p["obs_uv"], np.array([[o[2], o[3]] for o in obs], np.float32).reshape(-1, 2)])
    sig = np.concatenate([p["obs_sigma"], np.full(len(obs), 2.0)])
    outl = np.concatenate([p["obs_is_outlier"], np.zeros(len(obs), bool)])
    order = np.lexsort((ok, ol))
    assert np.all(np.diff(ol[order] * (p["K"] + 1) + ok[order]) > 0), "duplicate observation"
    q.update(obs_kf=ok[order].astype(np.int32), obs_uv=uv[order], obs_sigma=sig[order], obs_is_outlier=outl[order],
             lm_obs_ptr=np.concatenate([[0], np.cumsum(np.bincount(ol, minlength=q["L"]))]).astype(np.int32))
    return q


# ---------------------------------------------------------------------------------------------- cases
def cams_mixed():
    p = per_agent_cameras(sm.make_map(seed=31, n_agents=3, kf_per_agent=15, n_lm=400), MODELS3, seed=32)
    # three different calibrations, the camera of a keyframe is its agent's, and all three models observe landmarks
    assert len(p["extr"]) == 3 and np.array_equal(p["cam_of_kf"], p["agent_of"])
    assert len({tuple(r) for r in p["intr"]}) == 3 and len({tuple(r) for r in p["extr"]}) == 3
    assert sorted(zip(p["cam_model"], p["dist_model"])) == [(0, 0), (0, 2), (1, 1)]
    assert np.all(np.bincount(p["agent_of"][p["obs_kf"]], minlength=3) > 500)
    return p


def cams_radtan_gba():
    p = per_agent_cameras(sm.make_map(seed=33, n_agents=3, kf_per_agent=40, n_lm=3000), [(0, 0, 0.0)] * 3, seed=34)
    assert np.array_equal(p["cam_of_kf"], p["agent_of"]) and len({tuple(r) for r in p["intr"]}) == 3
    assert np.all(p["cam_model"] == 0) and np.all(p["dist_model"] == 0)
    return p


IMU_SPLIT = [[29, 14, 2], [22, 21, 1, 1], [15, 13, 17]]


def imu_split():
    p = sm.make_map(seed=35, n_agents=3, kf_per_agent=45, n_lm=600)
    cut = []
    for a, lens in enumerate(IMU_SPLIT):
        for c in np.cumsum(lens)[:-1]:          # drop the factor into the first keyframe of every piece
            cut.append(int(np.flatnonzero(p["imu_j"] == a * 45 + c)[0]))
    q = drop_imu(p, cut)
    assert imu_chains(q) == [n for lens in IMU_SPLIT for n in lens]
    # chains either side of a speed-bias tile (14 | 15 blocks) and of a pose tile (21 | 22 blocks), and isolated keyframes
    assert SB_PER_TILE == 14 and POSE_PER_TILE == 21
    assert {1, 2, 14, 15, 21, 22} <= set(imu_chains(q))
    return q


def isolated_keyframes(p):
    has = np.zeros(p["K"], bool)
    has[p["imu_i"]] = True; has[p["imu_j"]] = True
    return np.flatnonzero(~has)


def const_agent():
    p = sm.make_map(seed=37, n_agents=3, kf_per_agent=20, n_lm=500)
    p["pose_const"] = p["pose_const"].copy()
    p["pose_const"][p["agent_of"] == 1] = 1                  # a loaded map: every keyframe of agent 1
    p["pose_const"][[45, 46, 52]] = 1                        # inside agent 2's IMU chain (keyframes 40-59)
    assert imu_chains(p) == [20, 20, 20]
    for k in (45, 46, 52):                                   # IMU factors on both sides of each
        assert k in p["imu_i"] and k in p["imu_j"]
    return p


VO_TILE_K = [21, 22, 42, 43]


def vo_tile_edges(K):
    p = sm.make_map(seed=40 + K, n_agents=1, kf_per_agent=K, n_lm=300)
    # visual-only with landmarks: the plain layout, 6 columns per keyframe, within one pose block of a tile boundary
    assert min(abs(6 * K - TILE), abs(6 * K - 2 * TILE)) < 6
    return p


def pgo_threshold():
    rng = np.random.default_rng(41)
    p = sm.make_map(seed=41, n_agents=1, kf_per_agent=192, n_lm=10, drift_trans=0.05, drift_yaw_deg=0.5,
                    loops_intra=0, loops_per_pair=0)
    loops = [(5, 100), (40, 170), (90, 150), (20, 130)]      # every component tied to the gauge component (0-62)
    meas = [_between_from_gt(p, i, j, rng) for i, j in loops]
    p.update(loop_i=np.array([i for i, _ in loops], np.int32), loop_j=np.array([j for _, j in loops], np.int32),
             loop_q=np.array([m[0] for m in meas]), loop_t=np.array([m[1] for m in meas]), loop_cov=np.tile(np.eye(6), (4, 1, 1)))
    e = O.pgo_edges(p, p["pose"])
    lo, hi = np.minimum(e["i"], e["j"]), np.maximum(e["i"], e["j"])
    cross = (hi - lo <= BORDER_SPAN) & (((lo <= 62) & (hi >= 63)) | ((lo <= 126) & (hi >= 127)))
    e = {k: v[~cross] for k, v in e.items()}
    extra = [(70, 78), (140, 149)]                           # spans 8 and 9
    meas = [_between_from_gt(p, i, j, rng) for i, j in extra]
    S1 = np.diag([10.0] * 3 + [1.0] * 3) * 10.0               # the successor edges' weights (pgo_edges)
    e = dict(i=np.concatenate([e["i"], [i for i, _ in extra]]).astype(np.int32),
             j=np.concatenate([e["j"], [j for _, j in extra]]).astype(np.int32),
             q=np.concatenate([e["q"], [m[0] for m in meas]]), t=np.concatenate([e["t"], [m[1] for m in meas]]),
             sqrt_info=np.concatenate([e["sqrt_info"], np.tile(S1, (2, 1, 1))]),
             robust=np.concatenate([e["robust"], [False, False]]))
    span = np.abs(e["i"] - e["j"])
    comps = _components(p["K"], [(i, j) for i, j, s in zip(e["i"], e["j"], span) if s <= BORDER_SPAN])
    assert [len(c) for c in comps] == [ND_MIN - 1, ND_MIN, ND_MIN + 1] and [c[0] for c in comps] == [0, 63, 127]
    assert (span == BORDER_SPAN).sum() == 1 and (span == BORDER_SPAN + 1).sum() == 1
    border = set(e["i"][span > BORDER_SPAN]) | set(e["j"][span > BORDER_SPAN])
    assert {140, 149} <= border and not {70, 78} & border
    assert {int(np.searchsorted([63, 127], k, side="right")) for k in border} == {0, 1, 2}
    return p, e


def landmark_extremes():
    p = sm.make_map(seed=43, n_agents=2, kf_per_agent=16, n_lm=400)
    K = p["K"]
    # a far point in front of every camera: 12 m along the mean optical axis from the mean camera centre
    R, t = sm.quat_to_rot(p["gt_pose"][:, :4]), p["gt_pose"][:, 4:]
    Rsc, tsc = sm.quat_to_rot(p["extr"][0][:4]), p["extr"][0][4:]
    axis = (R @ Rsc)[:, :, 2].mean(0)
    X = (t + R @ tsc).mean(0) + 12.0 * axis / np.linalg.norm(axis)
    kfs = np.arange(K)
    rng = np.random.default_rng(44)
    in_cam = lambda k, x: Rsc.T @ (R[k].T @ (x - t[k]) - tsc)          # noqa: E731  (ground-truth camera frame)
    pc = np.stack([in_cam(k, X) for k in kfs])
    assert np.all(pc[:, 2] > 1.0) and np.all((pc[:, :2] ** 2).sum(1) / pc[:, 2] ** 2 < 0.75)   # monotone radtan
    uv = sm.project_radtan(pc) + rng.normal(0, 1.0, (K, 2))
    obs = [(p["L"], k, uv[k, 0], uv[k, 1]) for k in kfs]
    # The cameras look up (EuRoC body z): a point 0.35 m above the lowest camera is in front of it and of its temporal
    # neighbour, and behind the cameras that fly higher.  It is observed by those two and by the camera it is furthest
    # behind (in the ground truth and at x0, 10 cm or more): that observation's residual block is zero.
    lb = p["L"] + 1
    lo = int(np.argmin((t + R @ tsc)[:, 2]))
    nb = lo + 1 if lo + 1 < K and p["agent_of"][lo + 1] == p["agent_of"][lo] else lo - 1
    Y = (t[lo] + R[lo] @ tsc) + 0.35 * (R[lo] @ Rsc)[:, 2]
    zy = np.stack([_camera_z(p, s, kfs, np.tile(Y, (K, 1))) for s in (p["gt_pose"], p["pose"])])
    kb = int(np.argmin(zy.max(0)))
    assert zy[:, [lo, nb]].min() > 0.2 and zy[:, kb].max() < -0.1
    for k in sorted((lo, nb)):
        u = sm.project_radtan(in_cam(k, Y)[None])[0] + rng.normal(0, 1.0, 2)
        obs.append((lb, k, u[0], u[1]))
    obs.append((lb, kb, 300.0, 200.0))
    q = _with_observations(p, np.stack([X, Y]), obs)
    ol = _obs_lm(q)
    assert np.array_equal(q["obs_kf"][ol == p["L"]], kfs)                 # seen by every keyframe
    assert len(q["obs_kf"][ol == lb]) == 3
    # obs_skip: one landmark left with exactly 2 usable observations, one with exactly 1
    skip = np.zeros(len(q["obs_kf"]), np.uint8)
    n_obs = np.diff(q["lm_obs_ptr"])
    many = [l for l in np.flatnonzero(n_obs >= 4) if l not in (lb, p["L"])]
    l2, l1 = many[0], many[1]
    skip[q["lm_obs_ptr"][l2] + 2:q["lm_obs_ptr"][l2 + 1]] = 1
    skip[q["lm_obs_ptr"][l1] + 1:q["lm_obs_ptr"][l1 + 1]] = 1
    usable = np.bincount(ol[skip == 0], minlength=q["L"])
    assert usable[l2] == 2 and usable[l1] == 1 and usable[lb] >= 3
    return q, skip, dict(l1=l1, l2=l2, lb=lb, kb=kb, usable=usable)


def singular_imu():
    p = sm.make_config("tiny")
    p["imu_noise"] = p["imu_noise"].copy(); p["imu_noise"][3] = 0.0     # zero gyroscope random-walk sigma
    return p


# ---------------------------------------------------------------------------------------------- CPU: helpers and shapes
def test_per_agent_cameras_reproject_exactly_without_noise():
    """noise-free, the inlier observations are the projections of the ground truth through each keyframe's own camera
    (the oracle's residual model), and the outliers are the map's"""
    p0 = sm.make_map(seed=31, n_agents=3, kf_per_agent=15, n_lm=400)
    p = per_agent_cameras(p0, MODELS3, seed=32, pix_noise=0.0)
    pr = bo.Problem(dict(p, pose=p["gt_pose"], lm=p["gt_lm"]), visual_only=True, cauchy_reproj=None)
    _, r, _, info = pr.evaluate(pr.pose, pr.sb, pr.lm, with_jac=False)
    r0, n, m = info["reproj"]
    res = np.abs(r[r0:r0 + n * m].reshape(n, m)).max(1) * pr.o_sigma.numpy()        # pixels
    inl = ~p["obs_is_outlier"][pr.obs_sel]
    assert res[inl].max() < 1e-3                              # float32 storage of the pixels
    assert np.median(res[~inl]) > 10.0
    assert np.array_equal(p["obs_uv"][p0["obs_is_outlier"]], p0["obs_uv"][p0["obs_is_outlier"]])
    # each agent's camera differs from the map's by the stated amounts
    assert np.all(np.abs(p["intr"] / sm.EUROC_INTR - 1) <= 0.1)
    ang = 2 * np.degrees(np.arccos(np.minimum(1.0, np.abs(p["extr"][:, :4] @ p0["extr"][0][:4]))))
    assert np.all((ang > 0.05) & (ang < 4.0)) and np.all(np.linalg.norm(p["extr"][:, 4:] - p0["extr"][0][4:], axis=1) < 0.05)


def test_drop_imu_keeps_the_other_factors_samples():
    p = sm.make_map(seed=35, n_agents=2, kf_per_agent=10, n_lm=50)
    drop = [3, 4, 12]
    q = drop_imu(p, drop)
    keep = np.setdiff1d(np.arange(len(p["imu_i"])), drop)
    assert np.array_equal(q["imu_i"], p["imu_i"][keep]) and len(q["imu_ptr"]) == len(keep) + 1
    for a, f in enumerate(keep):
        s, e = p["imu_ptr"][f], p["imu_ptr"][f + 1]
        s2, e2 = q["imu_ptr"][a], q["imu_ptr"][a + 1]
        assert np.array_equal(q["imu_acc"][s2:e2], p["imu_acc"][s:e]) and np.array_equal(q["imu_dt"][s2:e2], p["imu_dt"][s:e])
        assert np.array_equal(q["imu_gyr"][s2:e2], p["imu_gyr"][s:e]) and np.array_equal(q["imu_acc0"][a], p["imu_acc0"][f])
    # factors 3, 4 link keyframes 3-4 and 4-5 of agent 0: keyframe 4 is isolated; factor 12 splits agent 1 at 13|14
    assert imu_chains(q) == [4, 1, 5, 4, 6]


@pytest.mark.parametrize("case", ["cams_mixed", "cams_radtan_gba", "imu_split", "const_agent", "pgo_threshold",
                                  "landmark_extremes", "vo_tile_edges"])
def test_map_shapes_reach_their_branches(case):
    if case == "vo_tile_edges":
        for K in VO_TILE_K:
            vo_tile_edges(K)
    else:
        globals()[case]()
    if case == "imu_split":
        assert list(isolated_keyframes(imu_split())) == [88, 89]


def test_oracle_refuses_singular_imu_covariance():
    with pytest.raises(np.linalg.LinAlgError):
        bo.Problem(singular_imu(), visual_only=False, loop_loss=1.0)


# ---------------------------------------------------------------------------------------------- GPU vs oracle
@pytest.mark.gpu
@pytest.mark.parametrize("visual_only", [True, False])
def test_cams_mixed_matches_oracle(ctx, visual_only):
    p = cams_mixed()
    pr = bo.Problem(p, visual_only=visual_only, loop_loss=1.0)
    s = O.BaSolver(ctx, p, visual_only=visual_only)
    try:
        norms = s.reproj_norms()
        s.iterate(5)
        got = s.result()
    finally:
        s.close()
    ref_norms = bo.corrected_reproj_norms(pr, pr.pose, pr.sb, pr.lm)
    outside = np.ones(len(norms), bool); outside[pr.obs_sel] = False
    assert np.all(norms[outside] == -1.0)
    n_err = np.abs(norms[pr.obs_sel] - ref_norms) / np.maximum(ref_norms, 0.01)
    ref = bo.solve(pr, 5)
    c_err = abs(got["initial_cost"] / ref["cost"][0] - 1)
    print(f"[cams_mixed vo={visual_only}] norms at x0: max rel err {n_err.max():.3e} ({n_err.max() / NORM_RTOL:.3f} of tol); "
          f"initial cost rel err {c_err:.3e} ({c_err / COST_RTOL:.3f} of tol)")
    assert n_err.max() < NORM_RTOL
    assert c_err < COST_RTOL
    _compare(got, ref, p)
    assert got["final_cost"] < got["initial_cost"]


@pytest.mark.gpu
def test_cams_radtan_gba_matches_cpu_port(ctx):
    from oracle import ba_port as bp
    p = cams_radtan_gba()
    got = O.global_bundle_adjustment(ctx, p, iterations_limit=6)
    ref = bp.global_bundle_adjustment(p, iterations_limit=6)
    assert np.array_equal(got["obs_removed"], ref["obs_removed"]) and got["obs_removed"].sum() > 100
    well = (got["lm_owner"] >= 0) & (np.abs(ref["lm"]).max(1) < 100.0)
    _port_compare(got, ref, p, lm_mask=well)


@pytest.mark.gpu
def test_imu_split_matches_oracle(ctx):
    p = imu_split()
    iso = isolated_keyframes(p)
    s = O.BaSolver(ctx, p, visual_only=False)
    try:
        scale = s.debug_vector(0)[0].reshape(p["K"], 15)
        s.iterate(5)
        got = s.result()
    finally:
        s.close()
    # no factor touches an isolated keyframe's speed-bias: zero column → Jacobi scale exactly 1, gradient and step 0
    assert np.all(scale[iso, 6:] == 1.0)
    assert np.array_equal(got["speedbias"][iso], p["speedbias"][iso])
    ref = bo.solve(bo.Problem(p, visual_only=False, loop_loss=1.0), 5)
    _compare(got, ref, p)
    assert np.abs(got["pose"][iso] - p["pose"][iso]).max() > 0      # their poses are still solved for


@pytest.mark.gpu
def test_const_agent_matches_oracle(ctx):
    p = const_agent()
    got = O.solve(ctx, p, 5, visual_only=False)
    ref = bo.solve(bo.Problem(p, visual_only=False, loop_loss=1.0), 5)
    _compare(got, ref, p)
    c = p["pose_const"].astype(bool)
    assert np.array_equal(got["pose"][c], p["pose"][c])
    assert np.abs(got["speedbias"][p["agent_of"] == 1] - p["speedbias"][p["agent_of"] == 1]).max() > 0


@pytest.mark.gpu
@pytest.mark.parametrize("K", VO_TILE_K)
def test_vo_tile_edges_match_oracle(ctx, K):
    # 5 iterations: at K = 43 the oracle's 6th step meets the function tolerance within rounding, a coin toss
    p = vo_tile_edges(K)
    got = O.solve(ctx, p, 5, visual_only=True)
    ref = bo.solve(bo.Problem(p, visual_only=True, loop_loss=1.0), 5)
    _compare(got, ref, p)


@pytest.mark.gpu
def test_pgo_threshold_matches_oracle(ctx):
    """criteria of test_gpu_ba.py::test_pgo_matches_oracle"""
    p, edges = pgo_threshold()
    ref = bo.pose_graph_optimization(p, edges, iterations=10)
    got = O.pose_graph_optimization(ctx, p, edges, iterations=10)
    assert got["iterations"] == ref["result"]["iterations"]
    assert _rel(got["pose"], ref["pose"]) < RTOL
    assert np.allclose(got["cost"], ref["result"]["cost"], rtol=1e-6)
    assert got["final_cost"] < 0.8 * got["initial_cost"]


@pytest.mark.gpu
def test_landmark_extremes_match_oracle(ctx):
    p, skip, f = landmark_extremes()
    got = O.solve(ctx, p, 5, visual_only=False, obs_skip=skip)
    ref = bo.solve(bo.Problem(p, visual_only=False, loop_loss=1.0, use_obs=~skip.astype(bool)), 5)
    _compare(got, ref, p)
    assert np.array_equal(got["lm_owner"] < 0, f["usable"] < 2)
    assert got["lm_owner"][f["l1"]] == -1 and got["lm_owner"][f["l2"]] >= 0
    assert np.array_equal(got["lm"][f["l1"]], p["lm"][f["l1"]])


@pytest.mark.gpu
def test_singular_imu_covariance_is_refused(ctx):
    p = singular_imu()
    with pytest.raises(covins_b200.CvbError, match="IMU preintegration covariance"):
        O.solve(ctx, p, 3, visual_only=False)
    with pytest.raises(covins_b200.CvbError, match="IMU preintegration covariance"):
        O.global_bundle_adjustment(ctx, p, iterations_limit=3)
    # visual-only does not use the IMU factors and stays valid; a valid problem in the same context still solves
    O.solve(ctx, p, 1, visual_only=True)
    q = sm.make_config("tiny")
    got = O.solve(ctx, q, 6, visual_only=False)
    ref = bo.solve(bo.Problem(q, visual_only=False, loop_loss=1.0), 6)
    _compare(got, ref, q)
