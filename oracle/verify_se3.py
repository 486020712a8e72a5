"""The verification chain of cvb_verify_landmark_candidates_seeded_batch composed from the existing oracles — TEST
INFRASTRUCTURE ONLY.

compose() runs the five stages of the call on one query and its candidates: DenseMatcher landmark matching, the seeded GP3P
RANSAC, the gate with T12 / T21, SearchBySE3 and the relative-pose refinement.  The three glue steps between them
(gather_problems, pose_glue with already_masks, residual_pairs) are numpy restatements of the call's definition; the stages
themselves are passed in.  verify_landmark_seeded composes the existing oracles (oracle.knn.landmark_match_batch,
oracle.seeded.ransac_absolute_pose_seeded, oracle.geom.search_by_se3, oracle.relpose_oracle.optimize_relative_pose); it adds
no numerical oracle of its own.  Keyframes are duck-typed like covins_b200.placerec.LandmarkKf (.view a KfView, .bearings,
.sigma_angle, .T_ws, .T_sc, .cam)."""
import math

import numpy as np

from . import geom as og
from . import knn as oknn
from . import relpose_oracle as orp
from . import seeded as osd


def gather_problems(query, cands, outA, outB, n_out, seg, min_matches):
    """the RANSAC problems: per candidate its matches as a dense row idxA -> idxB (-1), and, when it has at least min_matches,
    one correspondence per match in ascending idxA (pts = candidate landmark, f / sigma of the query keypoint).
    → (rows [C, nq], dict(prob_ptr, pts, bearings, sigma, src)), src the query keypoint of each correspondence"""
    nq = query.view.n
    rows = np.full((len(cands), nq), -1, np.int64)
    ptr, pts, f, sg, src = [0], [], [], [], []
    for c, k in enumerate(cands):
        s0, m = int(seg[c]), int(n_out[c])
        rows[c, np.asarray(outA[s0:s0 + m], np.int64)] = np.asarray(outB[s0:s0 + m], np.int64)
        i = np.flatnonzero(rows[c] >= 0) if m >= min_matches else np.zeros(0, np.int64)
        pts.append(k.view.a["lm_pos"][rows[c, i]]); f.append(query.bearings[i]); sg.append(query.sigma_angle[i]); src.append(i)
        ptr.append(ptr[-1] + len(i))
    return rows, dict(prob_ptr=np.array(ptr, np.int32), pts=np.concatenate(pts).reshape(-1, 3), bearings=np.concatenate(f).reshape(-1, 3),
                      sigma=np.concatenate(sg), src=np.concatenate(src).astype(np.int64))


def _mul44(A, B):
    """rows 0..2 of A B, each entry four products summed left to right; row 3 = 0 0 0 1"""
    O = np.zeros((4, 4)); O[3, 3] = 1.0
    for r in range(3):
        for c in range(4):
            O[r, c] = ((float(A[r, 0]) * float(B[0, c]) + float(A[r, 1]) * float(B[1, c])) + float(A[r, 2]) * float(B[2, c])) + float(A[r, 3]) * float(B[3, c])
    return O


def rigid_inv(T):
    """[R^T | -R^T t] of rows 0..2 of T in the shim's inv_rigid order; row 3 = 0 0 0 1"""
    T = np.asarray(T, np.float64).reshape(4, 4)
    I = np.zeros((4, 4)); I[3, 3] = 1.0
    I[:3, :3] = T[:3, :3].T
    for r in range(3):
        I[r, 3] = -((float(T[0, r]) * float(T[0, 3]) + float(T[1, r]) * float(T[1, 3])) + float(T[2, r]) * float(T[2, 3]))
    return I


def shim_mul4(A, B):
    """the shim's mul4 (s = 0; s += A(r,k) B(k,c) for k = 0..3), all four rows"""
    A = np.asarray(A, np.float64).reshape(4, 4); B = np.asarray(B, np.float64).reshape(4, 4)
    O = np.zeros((4, 4))
    for r in range(4):
        for c in range(4):
            s = 0.0
            for k in range(4):
                s += float(A[r, k]) * float(B[k, c])
            O[r, c] = s
    return O


def pose7(T):
    """the shim's transform_to_pose7: [qx, qy, qz, qw, x, y, z] by Eigen's matrix-to-quaternion branches"""
    T = np.asarray(T, np.float64).reshape(4, 4)
    q = [0.0] * 4
    tr = (float(T[0, 0]) + float(T[1, 1])) + float(T[2, 2])
    if tr > 0:
        t = math.sqrt(tr + 1.0)
        q[3] = 0.5 * t
        t = 0.5 / t
        q[0] = (float(T[2, 1]) - float(T[1, 2])) * t; q[1] = (float(T[0, 2]) - float(T[2, 0])) * t; q[2] = (float(T[1, 0]) - float(T[0, 1])) * t
    else:
        i = 0
        if T[1, 1] > T[0, 0]:
            i = 1
        if T[2, 2] > T[i, i]:
            i = 2
        j, k = (i + 1) % 3, (i + 2) % 3
        t = math.sqrt(((float(T[i, i]) - float(T[j, j])) - float(T[k, k])) + 1.0)
        q[i] = 0.5 * t
        t = 0.5 / t
        q[3] = (float(T[k, j]) - float(T[j, k])) * t
        q[j] = (float(T[j, i]) + float(T[i, j])) * t
        q[k] = (float(T[k, i]) + float(T[i, k])) * t
    return np.array(q + [float(T[0, 3]), float(T[1, 3]), float(T[2, 3])])


def pose_glue(best_sample, best_count, best_model, T_sc, Tcw, min_ransac_inliers):
    """the gate and the transforms of one candidate → (go, T12 [4,4], T21 [4,4], pose7(T12)); zeros when it stops"""
    if not (best_sample >= 0 and best_count >= min_ransac_inliers):
        return False, np.zeros((4, 4)), np.zeros((4, 4)), np.zeros(7)
    M = np.eye(4); M[:3] = np.asarray(best_model, np.float64).reshape(3, 4)
    T12 = _mul44(rigid_inv(_mul44(M, np.asarray(T_sc, np.float64).reshape(4, 4))), rigid_inv(Tcw))
    return True, T12, rigid_inv(T12), pose7(T12)


def already_masks(go, row, src, inlier, nq, n2):
    """SearchBySE3's already-matched masks of one candidate and stages 1 / 2: row [nq] its idxA -> idxB, src / inlier its RANSAC
    correspondences' query keypoints and inlier flags.  A candidate that stops gets all-ones masks (the search finds nothing)."""
    a1 = np.full(nq, 0 if go else 1, np.uint8); a2 = np.full(n2, 0 if go else 1, np.uint8)
    stage = (row >= 0).astype(np.uint8)
    if go:
        i = np.asarray(src)[np.asarray(inlier, bool)]
        a1[i] = 1; a2[row[i]] = 1; stage[i] = 2
    return a1, a2, stage


def landmark_vector(row, stage, m12):
    """the LandmarkVector after SearchBySE3: the RANSAC inliers (stage 2), then the search's matches (stage 3) → (entries [nq], stage)"""
    stage = stage.copy()
    ent = np.where(stage == 2, row, -1)
    add = (stage != 2) & (np.asarray(m12) >= 0)
    ent[add] = np.asarray(m12)[add]; stage[add] = 3
    return ent, stage


def residual_pairs(query, cand, ent):
    """the refinement's residual pairs of one candidate, in ascending query keypoint, as the shim's OptimizeRelativePose builds them"""
    qa, ca = query.view.a, cand.view.a
    i = np.flatnonzero(ent >= 0)
    i = i[(qa["lm_valid"][i] != 0) & (ca["lm_valid"][ent[i]] != 0)]
    b = ent[i]
    TcwA = rigid_inv(shim_mul4(query.T_ws, query.T_sc)); TcwB = rigid_inv(shim_mul4(cand.T_ws, query.T_sc))

    def apply(T, P):
        return np.stack([((T[r, 0] * P[:, 0] + T[r, 1] * P[:, 1]) + T[r, 2] * P[:, 2]) + T[r, 3] for r in range(3)], 1)

    sig = lambda o: (o.astype(np.float32) + np.float32(1.0)).astype(np.float64) * 2.0
    return dict(pA_c=apply(TcwA, qa["lm_pos"][i]), pB_c=apply(TcwB, ca["lm_pos"][b]), kpA=qa["kp"][i], kpB=ca["kp"][b],
                sigmaA=sig(qa["octave"][i]), sigmaB=sig(ca["octave"][b]))


def compose(query, cands, seeds, prm, match, ransac, search, refine):
    """the five stages with the glue between them.  match(A, skipA, B, skipB, seg, thr, num_best) → (outA, outB, n_out);
    ransac(prob_ptr, pts, bearings, sigma, cam_off, cam_rot, seeds, threshold, max_iterations, probability) → result dict;
    search(view1, views2, T12s, T21s, already1s, already2s, th, desc_th_low, num_octaves, scale_factor) → (match12 [k, nq],
    n_found [k]) over the candidates that continue; refine(T12 pose7, residual dict, camA, camB, th_outlier_align) → (T12_out,
    removed, n_inliers, (it1, it2)), called only with at least 12 pairs.  → the result dict of
    covins_b200.placerec.verify_landmark_candidates_seeded with detail"""
    C, nq = len(cands), query.view.n
    qa = query.view.a
    seg = np.concatenate([[0], np.cumsum([k.view.n for k in cands])]).astype(np.int32)
    B = np.concatenate([k.view.a["desc"] for k in cands]).reshape(-1, 32) if C else np.zeros((0, 32), np.uint8)
    skB = np.concatenate([1 - k.view.a["lm_valid"] for k in cands]).astype(np.uint8) if C else np.zeros(0, np.uint8)
    if nq and len(B):
        oA, oB, n_out = match(qa["desc"], (1 - qa["lm_valid"]).astype(np.uint8), B, skB, seg, prm["thr"], prm["num_best"])
    else:
        oA = oB = np.zeros(0, np.int32); n_out = np.zeros(C, np.int32)
    rows, P = gather_problems(query, cands, oA, oB, n_out, seg, prm["min_matches"])
    Tsc = np.asarray(query.T_sc, np.float64).reshape(4, 4)
    rr = ransac(P["prob_ptr"], P["pts"], P["bearings"], P["sigma"], np.tile(Tsc[:3, 3], (C, 1)), np.tile(Tsc[:3, :3], (C, 1, 1)), seeds,
                prm["threshold"], prm["max_iterations"], prm["probability"])
    out = dict(n_matches=np.asarray(n_out, np.int32), T12=np.zeros((C, 4, 4)), T21=np.zeros((C, 4, 4)), n_found=np.zeros(C, np.int32),
               n_corr=np.zeros(C, np.int32), T12_out=np.zeros((C, 7)), n_inliers=np.zeros(C, np.int32), solve_iterations=np.zeros((C, 2), np.int32),
               match12=np.full((C, nq), -1, np.int32), stage=np.zeros((C, nq), np.uint8), removed=np.zeros((C, nq), np.uint8))
    for k in ("best_sample", "best_model", "best_count", "iterations", "consumed"):
        out[k] = rr[k]
    go, p7, masks = [], [], []
    for c in range(C):
        g, T12, T21, q7 = pose_glue(rr["best_sample"][c], rr["best_count"][c], rr["best_model"][c], Tsc, cands[c].view.Tcw.reshape(4, 4),
                                    prm["min_ransac_inliers"])
        out["T12"][c], out["T21"][c] = T12, T21
        b, e = P["prob_ptr"][c], P["prob_ptr"][c + 1]
        masks.append(already_masks(g, rows[c], P["src"][b:e], rr["inlier_mask"][b:e], nq, cands[c].view.n))
        go.append(g); p7.append(q7)
    live = [c for c in range(C) if go[c]]
    m12 = np.full((C, nq), -1, np.int64)
    if live:
        ms, nf = search(query.view, [cands[c].view for c in live], [out["T12"][c] for c in live], [out["T21"][c] for c in live],
                        [masks[c][0] for c in live], [masks[c][1] for c in live], prm["th"], prm["desc_th_low"], prm["num_octaves"],
                        prm["scale_factor"])
        for j, c in enumerate(live):
            m12[c] = ms[j]; out["n_found"][c] = nf[j]
    for c in range(C):
        ent, st = landmark_vector(rows[c], masks[c][2], m12[c])
        out["stage"][c] = st
        if not go[c]:
            continue
        out["match12"][c] = ent
        rp = residual_pairs(query, cands[c], ent)
        n = len(rp["sigmaA"])
        out["n_corr"][c] = n
        out["T12_out"][c] = p7[c]
        if n >= 12:
            T, removed, ninl, its = refine(p7[c], rp, query.cam, cands[c].cam, prm["th_outlier_align"])
            out["T12_out"][c] = T; out["n_inliers"][c] = ninl; out["solve_iterations"][c] = its; out["removed"][c, :n] = removed
    return out


def _oracle_match(A, skipA, B, skipB, seg, thr, num_best):
    oA, oB, _, n = oknn.landmark_match_batch(A, skipA, B, skipB, seg, thr, num_best)
    return oA, oB, n


def _oracle_search(v1, v2s, T12s, T21s, a1s, a2s, th, desc_th_low, num_octaves, scale_factor):
    r = [og.search_by_se3(v1, v2, T12, T21, a1, a2, th, desc_th_low, num_octaves, scale_factor) for v2, T12, T21, a1, a2 in zip(v2s, T12s, T21s, a1s, a2s)]
    return np.stack([x[0] for x in r]), np.array([x[1] for x in r], np.int32)


def _oracle_refine(p7, rp, camA, camB, th):
    o = orp.optimize_relative_pose(p7, camA=camA, camB=camB, th_outlier_align=th, **rp)
    its = (o["r1"]["iterations"], o["r2"]["iterations"] if o["r2"] is not None else 0)
    return o["T12"], o["removed"].astype(np.uint8), o["n_inliers"], its


def verify_landmark_seeded(query, cands, seeds, **prm):
    """same arguments (the keyword parameters of covins_b200.placerec.verify_landmark_candidates_seeded, every one given) and result
    dict (with detail) as that call, composed from the existing oracles"""
    return compose(query, cands, np.asarray(seeds, np.uint64), prm, _oracle_match, osd.ransac_absolute_pose_seeded, _oracle_search, _oracle_refine)
