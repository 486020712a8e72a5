"""cvb_verify_landmark_candidates_seeded_batch (placerec.verify_landmark_candidates_seeded): the COVINS verification chain of a query
keyframe's candidates in one call, against the composed oracle (oracle/verify_se3.py:verify_landmark_seeded) and against the chain
of the existing calls with the glue done on the host (tools/verify_se3_timing.py:chain_existing_calls)."""
import ctypes as C
import importlib.util
import os
import subprocess

import numpy as np
import pytest

from covins_b200 import placerec as PR, synth
from oracle import verify_se3 as ov
from ransac_helpers import ROOT, _build_shim

PRM = dict(min_matches=25, threshold=9.0, max_iterations=200, min_ransac_inliers=15, thr=50.0, num_best=4, probability=0.99, th=9.5,
           desc_th_low=50, num_octaves=1, scale_factor=2.0, th_outlier_align=0.9)
CVB_ERR_INVALID, CVB_ERR_UNSUPPORTED = 1, 3


def _rigid(R, t):
    T = np.eye(4); T[:3, :3] = R; T[:3, 3] = t
    return T


def _view(kp, octave, desc, lm_valid, lm_pos, lm_maxdist, lm_desc, K, Tcw, img_bounds):
    return PR.KfView(kp, octave, desc, lm_valid, lm_pos, lm_maxdist, lm_desc, K, Tcw, img_bounds)


def scene(seed, n_cand, n_kp=1000, unrelated=(), wrong_desc=0.2, search_only=0.15, pix_noise=0.0):
    """a query keyframe and n_cand candidates over shared landmarks, built on synth.se3_search_scene: its first keyframe is the query
    (camera at the world origin) with its landmarks moved onto the rays of their keypoints, so that every bearing is exact.  Every
    candidate sees a random share of the query's landmarks from its own pose, at exactly the query's world positions (noise-free),
    with a share wrong_desc of its landmark keypoints carrying the descriptor of another landmark (wrong DenseMatcher matches) and
    pix_noise on its keypoints; the candidates in `unrelated` see none of them.  All keyframes share one extrinsic T_sc.
    A candidate keypoint has the index of the query keypoint of the same landmark, and a share search_only of them is left to
    SearchBySE3: their keypoint descriptor is near the query's landmark descriptor instead of its keypoint descriptor (the
    DenseMatcher compares keypoint descriptors, the search compares a landmark's descriptor with the other keyframe's keypoints),
    and their landmark descriptor near the query's keypoint descriptor, so both search directions agree (the search's agreement
    test reads match2[i] with the query index i, feature_matcher_be.cpp:489, which the shared index satisfies).
    → (query, cands (placerec.LandmarkKf), seeds, true T12 per candidate)"""
    views, _, _, _, _ = synth.se3_search_scene(seed, n_kp=n_kp, n_shared=min(300, n_kp // 2), pix_noise=0.0)
    rng = np.random.default_rng(seed + 1000)
    q = views[0]
    K = q["K"]
    cam = dict(intr=np.array([K[0, 0], K[1, 1], K[0, 2], K[1, 2]]), dist=np.zeros(4), cam_model=0, dist_model=0, xi=0.0)
    slots = np.flatnonzero(q["lm_valid"])
    ray = np.linalg.solve(K, np.concatenate([q["kp"].astype(np.float64), np.ones((n_kp, 1))], 1).T).T
    P = q["lm_pos"].copy()
    P[slots] = ray[slots] * q["lm_pos"][slots, 2:3]                        # on the keypoint's ray, at the scene's depth
    bear = ray / np.linalg.norm(ray, axis=1, keepdims=True)
    bear[q["lm_valid"] == 0] = rng.normal(0, 1, (int((q["lm_valid"] == 0).sum()), 3))
    bear /= np.linalg.norm(bear, axis=1, keepdims=True)
    T_sc = _rigid(synth._rot(rng.normal(0, 0.05, 3)), rng.normal(0, 0.05, 3))
    Tsc_inv = np.linalg.inv(T_sc)
    qv = _view(q["kp"], q["octave"], q["desc"], q["lm_valid"], P, q["lm_maxdist"], q["lm_desc"], K, q["Tcw"], q["img_bounds"])
    query = PR.LandmarkKf(qv, Tsc_inv, T_sc, cam, bear, rng.uniform(1e-6, 1e-5, n_kp))
    img_w, img_h = q["img_bounds"][1], q["img_bounds"][3]
    cands, truth = [], []
    for c in range(n_cand):
        T_wc = _rigid(synth._rot(rng.normal(0, 0.05, 3)), rng.normal(0, 0.15, 3))
        Tcw = np.linalg.inv(T_wc)
        kp = np.stack([rng.uniform(0, img_w, n_kp), rng.uniform(0, img_h, n_kp)], -1).astype(np.float32)
        desc = rng.integers(0, 256, (n_kp, 32), dtype=np.uint8); lm_desc = rng.integers(0, 256, (n_kp, 32), dtype=np.uint8)
        lm_valid = np.zeros(n_kp, np.uint8); lm_pos = np.zeros((n_kp, 3)); lm_maxdist = np.ones(n_kp)
        if c not in unrelated:
            pc = P[slots] @ Tcw[:3, :3].T + Tcw[:3, 3]
            u = pc @ K.T
            u = u[:, :2] / u[:, 2:3]
            vis = np.flatnonzero((pc[:, 2] > 0.5) & (u[:, 0] > 5) & (u[:, 0] < img_w - 5) & (u[:, 1] > 5) & (u[:, 1] < img_h - 5))
            vis = vis[rng.random(len(vis)) < 0.7]
            src = slots[vis]
            dst = src
            kp[dst] = (u[vis] + rng.normal(0, pix_noise, (len(vis), 2))).astype(np.float32)
            roll = rng.random(len(vis))
            wrong, alone = roll < wrong_desc, (roll >= wrong_desc) & (roll < wrong_desc + search_only)
            src_d = src.copy(); src_d[wrong] = rng.choice(slots, int(wrong.sum()))
            desc[dst] = q["desc"][src_d] ^ synth._flip_mask(rng, (len(vis), 32))
            desc[dst[alone]] = q["lm_desc"][src[alone]] ^ synth._flip_mask(rng, (int(alone.sum()), 32))
            lm_desc[dst] = q["desc"][src] ^ synth._flip_mask(rng, (len(vis), 32))
            lm_valid[dst] = 1; lm_valid[dst[rng.random(len(vis)) < 0.05]] = 0
            lm_pos[dst] = P[src]
            lm_maxdist[dst] = np.linalg.norm(pc[vis], axis=1) * rng.uniform(0.9, 2.5, len(vis))
        v = _view(kp, np.zeros(n_kp, np.float32), desc, lm_valid, lm_pos, lm_maxdist, lm_desc, K, Tcw, q["img_bounds"])
        cands.append(PR.LandmarkKf(v, T_wc @ Tsc_inv, T_sc, cam))
        truth.append(T_wc)
    return query, cands, rng.integers(0, 2**63, n_cand, dtype=np.uint64), truth


BITWISE = ("n_matches", "best_sample", "best_model", "best_count", "iterations", "consumed", "T12", "T21", "n_found", "match12", "stage", "n_corr")


def _same(a, b):
    a = np.ascontiguousarray(a); b = np.ascontiguousarray(np.asarray(b, a.dtype)).reshape(a.shape)
    return np.array_equal(a.view(np.uint8), b.view(np.uint8))


def _cmp_refine(g, r):
    assert np.array_equal(g["n_inliers"], r["n_inliers"]) and np.array_equal(g["solve_iterations"], r["solve_iterations"])
    assert np.array_equal(g["removed"], r["removed"])
    assert np.abs(g["T12_out"] - r["T12_out"]).max() < 1e-9


# --------------------------------------------------------------------------------------------------------------- CPU
def test_oracle_recovers_true_pose_noise_free():
    query, cands, seeds, truth = scene(3, 3, unrelated=(2,))
    r = ov.verify_landmark_seeded(query, cands, seeds, **PRM)
    for c in (0, 1):
        assert r["n_matches"][c] >= PRM["min_matches"] and r["best_count"][c] >= PRM["min_ransac_inliers"], c
        assert (r["stage"][c] == 1).any() and (r["stage"][c] == 2).any()            # the wrong descriptors are rejected
        assert np.abs(r["T12"][c] - truth[c]).max() < 1e-6, c
        assert r["n_corr"][c] >= 12 and r["n_inliers"][c] > 0
        T = synth_pose(r["T12_out"][c])
        assert np.abs(T - truth[c]).max() < 1e-6, c
    assert r["n_matches"][2] < PRM["min_matches"] and r["best_sample"][2] == -1 and r["n_corr"][2] == 0
    assert not r["T12"][2].any() and not r["T12_out"][2].any()


def synth_pose(p7):
    x, y, z, w = p7[:4] / np.linalg.norm(p7[:4])
    T = np.eye(4)
    T[:3, :3] = [[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                 [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]]
    T[:3, 3] = p7[4:]
    return T


def test_glue_equals_numpy_restatement():
    query, cands, seeds, _ = scene(4, 2, n_kp=300)
    rng = np.random.default_rng(0)
    nq = query.view.n
    # gather: dense rows, the used candidates' matches in ascending idxA
    seg = np.concatenate([[0], np.cumsum([k.view.n for k in cands])]).astype(np.int32)
    oA, oB, n_out = [], [], []
    for k in cands:
        a = rng.choice(nq, 40, replace=False); b = rng.choice(k.view.n, 40, replace=False)
        o = np.argsort(b)
        oA.append(np.concatenate([a[o], np.full(k.view.n - 40, -1)])); oB.append(np.concatenate([b[o], np.full(k.view.n - 40, -1)])); n_out.append(40)
    n_out[1] = 10                                                                   # below min_matches: no problem
    rows, P = ov.gather_problems(query, cands, np.concatenate(oA), np.concatenate(oB), n_out, seg, 25)
    i0 = np.sort(oA[0][:40])
    assert np.array_equal(P["prob_ptr"], [0, 40, 40]) and np.array_equal(P["src"], i0)
    assert np.array_equal(P["pts"], cands[0].view.a["lm_pos"][rows[0, i0]]) and np.array_equal(P["bearings"], query.bearings[i0])
    assert np.array_equal(P["sigma"], query.sigma_angle[i0]) and (rows[1] >= 0).sum() == 10
    # the gate and T12 / T21 bitwise against an element-wise restatement
    R = synth._rot(rng.normal(0, 0.3, 3)); M = np.concatenate([R, rng.normal(0, 1, (3, 1))], 1)
    Tcw = cands[0].view.Tcw.reshape(4, 4)
    g, T12, T21, p7 = ov.pose_glue(0, 20, M, query.T_sc, Tcw, 15)
    Ts = query.T_sc.reshape(4, 4)
    A = np.zeros((3, 4))
    for r in range(3):
        A[r] =((M[r, 0] * Ts[0] + M[r, 1] * Ts[1]) + M[r, 2] * Ts[2]) + M[r, 3] * Ts[3]
    Bi = np.zeros((3, 4)); Bi[:, :3] = A[:, :3].T; Bi[:, 3] = -((A[0, :3] * A[0, 3] + A[1, :3] * A[1, 3]) + A[2, :3] * A[2, 3])
    Ci = np.eye(4); Ci[:3, :3] = Tcw[:3, :3].T; Ci[:3, 3] = -((Tcw[0, :3] * Tcw[0, 3] + Tcw[1, :3] * Tcw[1, 3]) + Tcw[2, :3] * Tcw[2, 3])
    E = np.eye(4)
    for r in range(3):
        E[r] = ((Bi[r, 0] * Ci[0] + Bi[r, 1] * Ci[1]) + Bi[r, 2] * Ci[2]) + Bi[r, 3] * Ci[3]
    assert g and _same(T12, E)
    F = np.eye(4); F[:3, :3] = E[:3, :3].T; F[:3, 3] = -((E[0, :3] * E[0, 3] + E[1, :3] * E[1, 3]) + E[2, :3] * E[2, 3])
    assert _same(T21, F) and np.abs(T12 @ T21 - np.eye(4)).max() < 1e-12
    assert np.abs(synth_pose(p7) - T12).max() < 1e-12
    for bs, bc in ((-1, 0), (0, 14)):                                               # no model / too few inliers: stop
        g, T12, T21, p7 = ov.pose_glue(bs, bc, M, query.T_sc, Tcw, 15)
        assert not g and not T12.any() and not T21.any() and not p7.any()
    # masks and the LandmarkVector order
    row = np.full(nq, -1); row[[3, 5, 9]] = [7, 8, 2]
    a1, a2, st = ov.already_masks(True, row, np.array([3, 5, 9]), np.array([1, 0, 1]), nq, 20)
    assert np.flatnonzero(a1).tolist() == [3, 9] and np.flatnonzero(a2).tolist() == [2, 7] and st[[3, 5, 9]].tolist() == [2, 1, 2]
    a1, a2, _ = ov.already_masks(False, row, np.array([3, 5, 9]), np.array([1, 0, 1]), nq, 20)
    assert a1.all() and a2.all()
    m12 = np.full(nq, -1); m12[[5, 11]] = [4, 6]
    ent, st2 = ov.landmark_vector(row, st, m12)
    assert np.flatnonzero(ent >= 0).tolist() == [3, 5, 9, 11] and ent[[3, 5, 9, 11]].tolist() == [7, 4, 2, 6] and st2[[5, 11]].tolist() == [3, 3]
    # pA_c / pB_c bitwise against the shim's order
    ent = np.full(nq, -1); lmv = np.flatnonzero(query.view.a["lm_valid"])[:30]
    cv = np.flatnonzero(cands[0].view.a["lm_valid"])[:30]
    ent[lmv] = cv
    rp = ov.residual_pairs(query, cands[0], ent)
    def mul4(A, B):
        O = np.zeros((4, 4))
        for r in range(4):
            for c in range(4):
                s = 0.0
                for k in range(4):
                    s += A[r, k] * B[k, c]
                O[r, c] = s
        return O
    def inv(T):
        I = np.eye(4); I[:3, :3] = T[:3, :3].T
        for r in range(3):
            I[r, 3] = -(I[r, 0] * T[0, 3] + I[r, 1] * T[1, 3] + I[r, 2] * T[2, 3])
        return I
    TA = inv(mul4(query.T_ws.reshape(4, 4), query.T_sc.reshape(4, 4))); TB = inv(mul4(cands[0].T_ws.reshape(4, 4), query.T_sc.reshape(4, 4)))
    pa = [[TA[r, 0] * w[0] + TA[r, 1] * w[1] + TA[r, 2] * w[2] + TA[r, 3] for r in range(3)] for w in query.view.a["lm_pos"][lmv]]
    pb = [[TB[r, 0] * w[0] + TB[r, 1] * w[1] + TB[r, 2] * w[2] + TB[r, 3] for r in range(3)] for w in cands[0].view.a["lm_pos"][cv]]
    assert _same(rp["pA_c"], np.array(pa)) and _same(rp["pB_c"], np.array(pb))
    assert np.array_equal(rp["sigmaA"], (query.view.a["octave"][lmv] + np.float32(1)).astype(np.float64) * 2.0)


# --------------------------------------------------------------------------------------------------------------- GPU
def _chain():
    spec = importlib.util.spec_from_file_location("verify_se3_timing", os.path.join(ROOT, "tools", "verify_se3_timing.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m.chain_existing_calls


@pytest.mark.gpu
@pytest.mark.parametrize("n_cand", [1, 8, 32])
def test_fused_equals_composed_oracle(ctx, n_cand):
    query, cands, seeds, _ = scene(10 + n_cand, n_cand, unrelated=(n_cand - 1,) if n_cand > 1 else (), pix_noise=0.5)
    g = PR.verify_landmark_candidates_seeded(ctx, query, cands, seeds, **PRM)
    r = ov.verify_landmark_seeded(query, cands, seeds, **PRM)
    for k in BITWISE:
        assert _same(g[k], r[k]), k
    _cmp_refine(g, r)
    assert (g["n_inliers"] > 0).sum() >= max(1, n_cand - 1)
    # SearchBySE3 adds entries (stage 3) and they reach the refinement
    live = g["best_sample"] >= 0
    assert (g["n_found"][live] > 0).all() and (g["n_found"] == (g["stage"] == 3).sum(1)).all()
    assert (g["n_corr"][live] > (g["stage"][live] == 2).sum(1)).all()


@pytest.mark.gpu
@pytest.mark.parametrize("n_cand", [1, 8])
def test_fused_equals_chain_of_existing_calls(ctx, n_cand):
    query, cands, seeds, _ = scene(20 + n_cand, n_cand, pix_noise=0.5)
    g = PR.verify_landmark_candidates_seeded(ctx, query, cands, seeds, **PRM)
    r = _chain()(ctx, query, cands, seeds, **PRM)
    for k in BITWISE + ("T12_out", "n_inliers", "solve_iterations", "removed"):
        assert _same(g[k], r[k]), k
    assert (g["n_found"] > 0).all() and (g["stage"] == 3).any()


@pytest.mark.gpu
def test_candidate_alone_equals_in_batch(ctx):
    query, cands, seeds, _ = scene(31, 6, unrelated=(2,), pix_noise=0.5)
    g = PR.verify_landmark_candidates_seeded(ctx, query, cands, seeds, **PRM)
    for c in (0, 2, 5):
        a = PR.verify_landmark_candidates_seeded(ctx, query, [cands[c]], seeds[c:c + 1], **PRM)
        for k in g:
            assert _same(g[k][c:c + 1], a[k]), (c, k)


@pytest.mark.gpu
def test_edge_cases(ctx):
    query, cands, seeds, _ = scene(41, 3, n_kp=400, unrelated=(1,))
    assert PR.verify_landmark_candidates_seeded(ctx, query, [], np.zeros(0, np.uint64), **PRM)["n_matches"].shape == (0,)
    # below min_matches (unrelated), no RANSAC model (min_matches 0 lets a candidate with < 4 matches through), too few pairs
    p = dict(PRM, min_matches=0, min_ransac_inliers=0)
    few = scene(42, 1, n_kp=400)[1][0]
    keep = np.flatnonzero(few.view.a["lm_valid"])[:3]
    lv = np.zeros(few.view.n, np.uint8); lv[keep] = 1
    a = dict(few.view.a); a["lm_valid"] = lv
    few.view = PR.KfView(a["kp"], a["octave"], a["desc"], lv, a["lm_pos"], a["lm_maxdist"], a["lm_desc"], few.view.K, few.view.Tcw, few.view.img)
    g = PR.verify_landmark_candidates_seeded(ctx, query, [cands[0], cands[1], few], seeds, **p)
    r = ov.verify_landmark_seeded(query, [cands[0], cands[1], few], seeds, **p)
    for k in BITWISE:
        assert _same(g[k], r[k]), k
    _cmp_refine(g, r)
    assert g["n_matches"][2] <= 3 and g["best_sample"][2] == -1 and g["n_corr"][2] == 0
    # a candidate that passes the gate with fewer than 12 residual pairs: n_inliers = 0, T12_out = the start pose
    q2, (sc,), s2, _ = scene(43, 1, n_kp=400, wrong_desc=0.0, search_only=0.0)
    keep = np.flatnonzero(sc.view.a["lm_valid"])[:9]
    lv = np.zeros(sc.view.n, np.uint8); lv[keep] = 1
    a = dict(sc.view.a)
    sc.view = PR.KfView(a["kp"], a["octave"], a["desc"], lv, a["lm_pos"], a["lm_maxdist"], a["lm_desc"], sc.view.K, sc.view.Tcw, sc.view.img)
    p = dict(PRM, min_matches=5, min_ransac_inliers=5)
    g = PR.verify_landmark_candidates_seeded(ctx, q2, [sc], s2, **p)
    r = ov.verify_landmark_seeded(q2, [sc], s2, **p)
    for k in BITWISE:
        assert _same(g[k], r[k]), k
    _cmp_refine(g, r)
    assert g["best_count"][0] >= 5 and 0 < g["n_corr"][0] < 12 and g["n_inliers"][0] == 0
    assert _same(g["T12_out"][0], ov.pose7(g["T12"][0])) and not g["removed"].any() and not g["solve_iterations"].any()
    # a candidate with zero keypoints, a query with no valid landmarks, a query with zero keypoints
    v = query.view
    empty = PR.LandmarkKf(PR.KfView(np.zeros((0, 2)), np.zeros(0), np.zeros((0, 32)), np.zeros(0), np.zeros((0, 3)), np.zeros(0), np.zeros((0, 32)),
                                    v.K, cands[0].view.Tcw, v.img), cands[0].T_ws, cands[0].T_sc, cands[0].cam)
    for qq, cc in ((query, [empty]), (PR.LandmarkKf(PR.KfView(v.a["kp"], v.a["octave"], v.a["desc"], np.zeros(v.n), v.a["lm_pos"], v.a["lm_maxdist"],
                                                              v.a["lm_desc"], v.K, v.Tcw, v.img), query.T_ws, query.T_sc, query.cam, query.bearings,
                                                    query.sigma_angle), cands[:2]), (empty, cands[:2])):
        g = PR.verify_landmark_candidates_seeded(ctx, qq, cc, seeds[:len(cc)], **PRM)
        assert not g["n_matches"].any() and (g["best_sample"] == -1).all() and not g["n_corr"].any() and not g["T12_out"].any()


def _rc(ctx, query, cands, seeds, prm=PRM, edit=None):
    """the status of the raw C call (the arguments of placerec.verify_landmark_candidates_seeded); edit(q, arr, P, R, keep) may break
    one of them and returns the seed pointer to pass"""
    n, nq = len(cands), query.view.n
    keep = []
    q = query.cstruct()
    arr = (PR.CLandmarkKf * max(n, 1))(*[c.cstruct() for c in cands])
    P = PR.CLandmarkVerifyParams(float(prm["thr"]), int(prm["num_best"]), int(prm["min_matches"]), float(prm["threshold"]), int(prm["max_iterations"]),
                                 float(prm["probability"]), int(prm["min_ransac_inliers"]),
                                 PR.CSearchParams(float(prm["th"]), int(prm["desc_th_low"]), int(prm["num_octaves"]), float(prm["scale_factor"])),
                                 float(prm["th_outlier_align"]))
    bufs = [np.zeros(max(n, 1) * 16 * max(nq, 1), np.float64) for _ in PR.CLandmarkVerifyResult._fields_]
    R = PR.CLandmarkVerifyResult(*[b.ctypes.data for b in bufs])
    s = np.ascontiguousarray(seeds, np.uint64)
    sp = s.ctypes.data if edit is None else edit(q, arr, P, R, keep)
    return PR.lib().cvb_verify_landmark_candidates_seeded_batch(ctx.handle, C.byref(q), arr, n, C.byref(P), sp, C.byref(R))


@pytest.mark.gpu
def test_bad_arguments_are_refused(ctx):
    query, cands, seeds, _ = scene(51, 2, n_kp=300)
    s = np.ascontiguousarray(seeds, np.uint64)
    assert _rc(ctx, query, cands, seeds) == 0
    n0 = ctx.launch_count()
    for bad in (dict(num_best=0), dict(num_best=5), dict(max_iterations=-1), dict(max_iterations=(2**31 - 1 - 64) // 11 + 1), dict(thr=0.0),
                dict(thr=300.0), dict(scale_factor=1.0), dict(num_octaves=0), dict(th=0.0)):
        assert _rc(ctx, query, cands, seeds, dict(PRM, **bad)) == CVB_ERR_INVALID, bad

    def bad_grid(q, arr, P, R, keep):                   # grid_ptr[0] != 0: a malformed view
        g = np.array(query.view.a["grid_ptr"]); g[0] = 1
        keep.append(g); q.view.grid_ptr = g.ctypes.data
        return s.ctypes.data

    def neg_n(q, arr, P, R, keep):
        arr[1].view.n = -1
        return s.ctypes.data

    def set_null(obj, field):
        def f(q, arr, P, R, keep):
            setattr({"q": q, "R": R}[obj], field, None)
            return s.ctypes.data
        return f
    edits = [lambda q, arr, P, R, keep: None, bad_grid, neg_n, set_null("q", "bearings"), set_null("q", "sigma_angle")]
    edits += [set_null("R", k) for k, _ in PR.CLandmarkVerifyResult._fields_ if k not in ("match12", "stage", "removed")]
    for e in edits:
        assert _rc(ctx, query, cands, seeds, edit=e) == CVB_ERR_INVALID
    for cam in (dict(cands[1].cam, cam_model=2), dict(cands[1].cam, dist_model=3)):
        c1 = PR.LandmarkKf(cands[1].view, cands[1].T_ws, cands[1].T_sc, cam)
        assert _rc(ctx, query, [cands[0], c1], seeds) == CVB_ERR_UNSUPPORTED
        q1 = PR.LandmarkKf(query.view, query.T_ws, query.T_sc, cam, query.bearings, query.sigma_angle)
        assert _rc(ctx, q1, cands, seeds) == CVB_ERR_UNSUPPORTED
        with pytest.raises(Exception, match="Unknown (projection|distortion) type"):
            PR.verify_landmark_candidates_seeded(ctx, query, [cands[0], c1], seeds, **PRM)
    assert ctx.launch_count() == n0                                                # nothing launched
    assert _rc(ctx, query, [], np.zeros(0, np.uint64)) == 0                        # n_cand = 0 succeeds


def _dump_scene(d, query, cands, seeds, prm):
    for k, kf in enumerate([query] + list(cands)):
        a = kf.view.a
        for name in ("kp", "octave", "desc", "lm_valid", "lm_pos", "lm_maxdist", "lm_desc"):
            np.ascontiguousarray(a[name]).tofile(d / f"kf{k}_{name}.bin")
        kf.view.Tcw.astype(np.float64).tofile(d / f"kf{k}_Tcw.bin"); kf.T_ws.tofile(d / f"kf{k}_Tws.bin"); kf.T_sc.tofile(d / f"kf{k}_Tsc.bin")
        kf.view.K.astype(np.float64).tofile(d / f"kf{k}_K.bin")
        np.concatenate([np.asarray(kf.cam["intr"], np.float64), np.asarray(kf.cam["dist"], np.float64)]).tofile(d / f"kf{k}_cam.bin")
    query.bearings.tofile(d / "kf0_bearings.bin"); query.sigma_angle.tofile(d / "kf0_sigma.bin")
    np.ascontiguousarray(seeds, np.uint64).tofile(d / "seeds.bin")
    np.array([prm[k] for k in ("thr", "num_best", "min_matches", "threshold", "max_iterations", "probability", "min_ransac_inliers", "th", "desc_th_low",
                               "num_octaves", "scale_factor", "th_outlier_align")], np.float64).tofile(d / "params.bin")


def test_shim_verify_se3_compiles_and_refuses_incomplete_input(tmp_path):
    exe = str(tmp_path / "shim_verify_se3_test")
    _build_shim("shim_verify_se3_test.cpp", exe)
    assert subprocess.run([exe, str(tmp_path)]).returncode == 2                     # nothing dumped: refused before any GPU work
    query, cands, seeds, _ = scene(61, 1, n_kp=200)
    _dump_scene(tmp_path, query, cands, seeds, PRM)
    (tmp_path / "kf1_lm_pos.bin").unlink()
    assert subprocess.run([exe, str(tmp_path)]).returncode == 2                     # a candidate array missing


@pytest.mark.gpu
def test_shim_on_mock_containers_equals_python(ctx, tmp_path):
    query, cands, seeds, _ = scene(60, 4, unrelated=(2,), pix_noise=0.5)
    prm = dict(PRM, th_outlier_align=0.35)                                         # low enough that the purge removes pairs
    exe = str(tmp_path / "shim_verify_se3_test")
    _build_shim("shim_verify_se3_test.cpp", exe)
    _dump_scene(tmp_path, query, cands, seeds, prm)
    subprocess.check_call([exe, str(tmp_path)])
    g = PR.verify_landmark_candidates_seeded(ctx, query, cands, seeds, **prm)
    n, nq = len(cands), query.view.n
    ints = np.fromfile(tmp_path / "lmv_ints.bin", np.int32).reshape(n, 6)
    assert np.array_equal(ints, np.stack([g["n_matches"], g["best_sample"], g["best_count"], g["n_found"], g["n_corr"], g["n_inliers"]], 1))
    assert _same(np.fromfile(tmp_path / "lmv_pose.bin").reshape(n, 7), g["T12_out"])
    T12 = np.fromfile(tmp_path / "lmv_T12.bin").reshape(n, 4, 4)
    for c in range(n):
        if g["n_inliers"][c] == 0:
            assert _same(T12[c], g["T12"][c])                                       # as handed to the refinement (zero if stopped)
        else:
            assert np.abs(T12[c] - synth_pose(g["T12_out"][c])).max() < 1e-12
    # the written-back LandmarkVectors: match12 with the purge quirk (matches1[r] = nullptr for purged residual index r)
    lv = g["match12"].copy()
    for c in range(n):
        r = np.flatnonzero(g["removed"][c, :g["n_corr"][c]])
        lv[c, r] = -1
    assert g["removed"].any() and np.array_equal(np.fromfile(tmp_path / "lmv_lv.bin", np.int32).reshape(n, nq), lv)
