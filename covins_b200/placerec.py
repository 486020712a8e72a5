"""Host-side mirror of the place-recognition steps that follow the k-NN / DenseMatcher stage (SURVEY §8a M8 / V1), over
the C-ABI:

  search_by_se3_batch(...)      ↔ FeatureMatcher::SearchBySE3           (feature_matcher_be.cpp:293-498)
  score_absolute_pose(...)      ↔ FrameAbsolutePoseSacProblem scoring   (FrameAbsolutePoseSacProblem.h:95-126; Se3Solver GP3P RANSAC)
  score_relative_pose(...)      ↔ FrameRelativePoseSacProblem scoring   (frame-relative-pose-sac-problem.hpp:69-104)
  ransac_select(...)            ↔ the model-selection rule of opengv::sac::Ransac::computeModel replayed over batched scores
  ransac_absolute_pose(...)     ↔ the whole GP3P RANSAC of Se3Solver::projectiveAlignment from caller-supplied samples
  ransac_noncentral_relative_pose(...) ↔ the 17-point RANSAC of RelNonCentralPosSolver::computeNonCentralRelPose from
                                  caller-supplied samples
  ransac_central_relative_pose(...) ↔ the 5-point RANSAC of RelNonCentralPosSolver::computePose from caller-supplied samples
  relative_pose_covariance(...) ↔ the sampling-based 6x6 covariance of RelNonCentralPosSolver::computeNonCentralRelPose (17-point
                                  re-solves from caller-supplied samples)
  ransac_*_seeded(...), relative_pose_covariance_seeded(...) ↔ the same calls with the samples drawn on the GPU from one seed
                                  per problem, as the reference draws its own (include/covins_b200.h, "Seeded samples")
  verify_noncentral_relative_pose_seeded(...) ↔ the whole verification of RelNonCentralPosSolver::computeNonCentralRelPose
                                  (pairwise matching, 5-point and 17-point RANSAC, covariance) for all candidates in one call
  verify_noncentral_relative_pose_sift_seeded(...) ↔ the same with SIFT descriptors (exact L2 matching)
  verify_landmark_candidates_seeded(...) ↔ the COVINS verification of PlaceRecognition::ComputeSE3 (DenseMatcher landmark
                                  matching, GP3P RANSAC, SearchBySE3, OptimizeRelativePose) for all candidates in one call

`KfView` flattens what the reference reads of a Keyframe (the C++ shim does the same from the containers)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._lib import Context, lib, c_vp

GRID_COLS, GRID_ROWS = 64, 48          # FRAME_GRID_COLS / FRAME_GRID_ROWS (typedefs_base.hpp:59-60)


class CKfView(C.Structure):
    _fields_ = [("n", C.c_int32)] + [(k, c_vp) for k in ("kp", "octave", "desc", "lm_valid", "lm_pos", "lm_maxdist", "lm_desc", "grid_ptr", "grid_idx")] + \
               [("grid_w_inv", C.c_double), ("grid_h_inv", C.c_double), ("K", C.c_double * 9), ("Tcw", C.c_double * 16), ("img", C.c_double * 4)]


class CSearchParams(C.Structure):
    _fields_ = [("th", C.c_double), ("desc_th_low", C.c_int32), ("num_octaves", C.c_int32), ("scale_factor", C.c_double)]


def assign_features_to_grid(kp, img_w, img_h):
    """KeyframeBase::AssignFeaturesToGrid (keyframe_base.cpp:122-143): cell = round(x * 64/w), round(y * 48/h); members in
    ascending keypoint order.  Keypoints whose cell index reaches 64 / 48 are left out (the reference writes out of bounds)."""
    kp = np.asarray(kp, np.float32).reshape(-1, 2)
    w_inv, h_inv = GRID_COLS / float(img_w), GRID_ROWS / float(img_h)
    px = np.floor(kp[:, 0].astype(np.float64) * w_inv + 0.5).astype(np.int64)      # std::round of a non-negative value
    py = np.floor(kp[:, 1].astype(np.float64) * h_inv + 0.5).astype(np.int64)
    ok = (px >= 0) & (px < GRID_COLS) & (py >= 0) & (py < GRID_ROWS)
    cell = px * GRID_ROWS + py
    idx = np.flatnonzero(ok)
    order = idx[np.argsort(cell[idx], kind="stable")]
    ptr = np.zeros(GRID_COLS * GRID_ROWS + 1, np.int32)
    np.add.at(ptr, cell[idx] + 1, 1)
    return np.cumsum(ptr).astype(np.int32), order.astype(np.int32), w_inv, h_inv


class KfView:
    """the arrays FeatureMatcher::SearchBySE3 reads of one keyframe"""

    def __init__(self, kp, octave, desc, lm_valid, lm_pos, lm_maxdist, lm_desc, K, Tcw, img_bounds, img_w=752, img_h=480):
        n = len(kp)
        self.a = dict(kp=np.ascontiguousarray(kp, np.float32).reshape(n, 2), octave=np.ascontiguousarray(octave, np.float32),
                      desc=np.ascontiguousarray(desc, np.uint8).reshape(n, 32), lm_valid=np.ascontiguousarray(lm_valid, np.uint8),
                      lm_pos=np.ascontiguousarray(lm_pos, np.float64).reshape(n, 3), lm_maxdist=np.ascontiguousarray(lm_maxdist, np.float64),
                      lm_desc=np.ascontiguousarray(lm_desc, np.uint8).reshape(n, 32))
        gp, gi, w_inv, h_inv = assign_features_to_grid(self.a["kp"], img_w, img_h)
        self.a["grid_ptr"], self.a["grid_idx"] = gp, gi
        self.n, self.K, self.Tcw, self.img = n, np.asarray(K, np.float64).reshape(9), np.asarray(Tcw, np.float64).reshape(16), np.asarray(img_bounds, np.float64)
        self.grid_w_inv, self.grid_h_inv = w_inv, h_inv

    def cstruct(self, cls=CKfView):
        s = cls()
        s.n = self.n
        for k in ("kp", "octave", "desc", "lm_valid", "lm_pos", "lm_maxdist", "lm_desc", "grid_ptr", "grid_idx"):
            setattr(s, k, self.a[k].ctypes.data)
        s.grid_w_inv, s.grid_h_inv = self.grid_w_inv, self.grid_h_inv
        s.K[:] = self.K.tolist(); s.Tcw[:] = self.Tcw.tolist(); s.img[:] = self.img.tolist()
        return s


def search_by_se3_batch(ctx: Context, kf1: KfView, kf2s, T12, T21, already1, already2, th=9.5, desc_th_low=50, num_octaves=1, scale_factor=2.0,
                        debug=False):
    """→ (match12 [n_pairs, n1] i32: index of the KF2 keypoint whose landmark becomes matches12[i] or -1, n_found [n_pairs])."""
    n_pairs = len(kf2s)
    arr = (CKfView * max(n_pairs, 1))(*[k.cstruct() for k in kf2s])
    k1 = kf1.cstruct()
    T12 = np.ascontiguousarray(T12, np.float64).reshape(n_pairs, 16); T21 = np.ascontiguousarray(T21, np.float64).reshape(n_pairs, 16)
    a1 = np.ascontiguousarray(already1, np.uint8).reshape(n_pairs, kf1.n)
    a2 = np.ascontiguousarray(np.concatenate([np.asarray(a, np.uint8) for a in already2]) if n_pairs else np.zeros(0, np.uint8))
    prm = CSearchParams(float(th), int(desc_th_low), int(num_octaves), float(scale_factor))
    m12 = np.full((n_pairs, kf1.n), -1, np.int32); nf = np.zeros(max(n_pairs, 1), np.int32)
    m1 = np.full((n_pairs, kf1.n), -1, np.int32); m2 = np.full(max(len(a2), 1), -1, np.int32)
    ctx.check(lib().cvb_search_by_se3_batch(ctx.handle, C.byref(k1), arr, n_pairs, T12.ctypes.data, T21.ctypes.data, a1.ctypes.data, a2.ctypes.data,
                                            C.byref(prm), m12.ctypes.data, nf.ctypes.data, m1.ctypes.data, m2.ctypes.data))
    if debug:
        return m12, nf[:n_pairs], m1, m2[:len(a2)]
    return m12, nf[:n_pairs]


class CProjLandmarks(C.Structure):
    _fields_ = [("m", C.c_int32)] + [(k, c_vp) for k in ("valid", "pos", "normal", "min_dist", "max_dist", "max_distance", "desc", "feat_idx")]


def _proj_args(kf: KfView, kf_lm_cand, Tcw, cam: dict, lms: dict, matched, th, desc_th_low, num_octaves, scale_factor, struct_cls, prm_cls):
    """flat arguments shared by the product call and the oracle binding (which passes its own struct classes)"""
    m = len(lms["pos"])
    a = dict(valid=np.ascontiguousarray(lms["valid"], np.uint8), pos=np.ascontiguousarray(lms["pos"], np.float64).reshape(m, 3),
             normal=np.ascontiguousarray(lms["normal"], np.float64).reshape(m, 3), min_dist=np.ascontiguousarray(lms["min_dist"], np.float64),
             max_dist=np.ascontiguousarray(lms["max_dist"], np.float64), max_distance=np.ascontiguousarray(lms["max_distance"], np.float64),
             desc=np.ascontiguousarray(lms["desc"], np.uint8).reshape(m, 32), feat_idx=np.ascontiguousarray(lms["feat_idx"], np.int32))
    L = struct_cls(); L.m = m
    for k, v in a.items():
        setattr(L, k, v.ctypes.data)
    keep = [a, np.ascontiguousarray(kf_lm_cand, np.int32), np.ascontiguousarray(Tcw, np.float64).reshape(16),
            np.ascontiguousarray(cam["intr"], np.float64).reshape(4), np.ascontiguousarray(cam["dist"], np.float64).reshape(4),
            np.ascontiguousarray(matched, np.uint8)]
    prm = prm_cls(float(th), int(desc_th_low), int(num_octaves), float(scale_factor))
    return L, prm, keep, m


def search_by_projection(ctx: Context, kf: KfView, kf_lm_cand, Tcw, cam: dict, lms: dict, matched, th=10.0, desc_th_low=50, num_octaves=1,
                         scale_factor=2.0):
    """FeatureMatcher::SearchByProjection (feature_matcher_be.cpp:168-291) → (action [m], best_idx [m], n_matches); kf.a['lm_valid'][idx]
    = pKF->GetLandmark(idx) != nullptr; lms: dict(valid, pos, normal, min_dist, max_dist, max_distance, desc, feat_idx)."""
    L, prm, keep, m = _proj_args(kf, kf_lm_cand, Tcw, cam, lms, matched, th, desc_th_low, num_octaves, scale_factor, CProjLandmarks, CSearchParams)
    k = kf.cstruct()
    action = np.zeros(max(m, 1), np.int32); best = np.full(max(m, 1), -1, np.int32); nm = C.c_int32(0)
    ctx.check(lib().cvb_search_by_projection(ctx.handle, C.byref(k), keep[1].ctypes.data, keep[2].ctypes.data, keep[3].ctypes.data, keep[4].ctypes.data,
                                             int(cam.get("cam_model", 0)), int(cam.get("dist_model", 0)), float(cam.get("xi", 0.0)), C.byref(L),
                                             keep[5].ctypes.data, C.byref(prm), action.ctypes.data, best.ctypes.data, C.byref(nm)))
    return action[:m], best[:m], int(nm.value)


def _score(ctx, fn, args, n_hyp, n, want_scores, want_inliers):
    sc = np.zeros((n_hyp, n)) if want_scores else None
    inl = np.zeros((n_hyp, n), np.uint8) if want_inliers else None
    cnt = np.zeros(max(n_hyp, 1), np.int32)
    ctx.check(fn(ctx.handle, *args, sc.ctypes.data if sc is not None else None, inl.ctypes.data if inl is not None else None, cnt.ctypes.data))
    return sc, inl, cnt[:n_hyp]


def score_absolute_pose(ctx: Context, models, pts, bearings, sigma, cam_off, cam_rot, threshold, want_scores=True, want_inliers=True):
    """models [H,3,4] = [R|t] (body in world); → (scores [H,n], inlier [H,n], n_inliers [H])"""
    m = np.ascontiguousarray(models, np.float64).reshape(-1, 12); p = np.ascontiguousarray(pts, np.float64).reshape(-1, 3)
    f = np.ascontiguousarray(bearings, np.float64).reshape(-1, 3); s = np.ascontiguousarray(sigma, np.float64)
    co = np.ascontiguousarray(cam_off, np.float64).reshape(3); cr = np.ascontiguousarray(cam_rot, np.float64).reshape(9)
    return _score(ctx, lib().cvb_score_absolute_pose_batch, (m.ctypes.data, len(m), p.ctypes.data, f.ctypes.data, s.ctypes.data, len(p), co.ctypes.data,
                                                             cr.ctypes.data, float(threshold)), len(m), len(p), want_scores, want_inliers)


def score_relative_pose(ctx: Context, models, f1, f2, sigma1, sigma2, threshold, want_scores=True, want_inliers=True):
    m = np.ascontiguousarray(models, np.float64).reshape(-1, 12)
    a = np.ascontiguousarray(f1, np.float64).reshape(-1, 3); b = np.ascontiguousarray(f2, np.float64).reshape(-1, 3)
    s1 = np.ascontiguousarray(sigma1, np.float64); s2 = np.ascontiguousarray(sigma2, np.float64)
    return _score(ctx, lib().cvb_score_relative_pose_batch, (m.ctypes.data, len(m), a.ctypes.data, b.ctypes.data, s1.ctypes.data, s2.ctypes.data, len(a),
                                                             float(threshold)), len(m), len(a), want_scores, want_inliers)


def ransac_select(n_inliers, n_points, sample_size, max_iterations, probability=0.99):
    """opengv::sac::Ransac::computeModel's model selection replayed over the batched inlier counts (hypothesis h is the
    model of iteration h): the best model so far wins on a strictly larger inlier count, and the adaptive iteration bound
    k = log(1 - p) / log(1 - w^s) stops the scan exactly where the sequential loop would stop.  → (best index or -1, iterations used)"""
    best, best_n, k, it = -1, 0, float(max_iterations), 0
    log_p = np.log(1.0 - probability)
    while it < min(k, max_iterations, len(n_inliers)):
        c = int(n_inliers[it])
        if c > best_n:
            best_n, best = c, it
            w = c / float(n_points)
            pno = 1.0 - w ** sample_size
            pno = min(max(pno, np.finfo(float).eps), 1.0 - np.finfo(float).eps)
            k = log_p / np.log(pno)
        it += 1
    return best, it


class CAbsRansacProblems(C.Structure):
    _fields_ = [("n_prob", C.c_int32)] + [(k, c_vp) for k in ("prob_ptr", "pts", "f", "sigma", "cam_off", "cam_rot", "samples")] + \
               [("n_samples", C.c_int32)]


class CRansacResult(C.Structure):
    """cvb_abs_ransac_result and cvb_rel_ransac_result (the same layout)"""
    _fields_ = [(k, c_vp) for k in ("best_sample", "best_model", "best_count", "iterations", "consumed", "inlier_mask", "sample_model",
                                    "sample_valid", "sample_count")]


CAbsRansacResult = CRelRansacResult = CRansacResult   # the names of the per-call result structs, kept for existing callers


def _ransac(ctx, fn, P, n_prob, ns, n, threshold, max_iterations, probability, per_sample, seeds=None, k=0, want_drawn=False):
    """one RANSAC call fn on the problems P (n_prob problems, ns samples each, n correspondences) → its result dict; with seeds
    (a seeded call fn, sample size k) also drawn [n_prob, ns, k] when want_drawn"""
    r = dict(best_sample=np.zeros(n_prob, np.int32), best_model=np.zeros((n_prob, 3, 4)), best_count=np.zeros(n_prob, np.int32),
             iterations=np.zeros(n_prob, np.int32), consumed=np.zeros(n_prob, np.int32), inlier_mask=np.zeros(n, np.uint8))
    if per_sample:
        r.update(sample_model=np.zeros((n_prob, ns, 3, 4)), sample_valid=np.zeros((n_prob, ns), np.uint8),
                 sample_count=np.zeros((n_prob, ns), np.int32))
    R = CRansacResult(*[r[k].ctypes.data if k in r else None for k, _ in CRansacResult._fields_])
    if seeds is None:
        ctx.check(fn(ctx.handle, C.byref(P), float(threshold), int(max_iterations), float(probability), C.byref(R)))
        return r
    if want_drawn:
        r["drawn"] = np.full((n_prob, ns, k), -1, np.int32)
    ctx.check(fn(ctx.handle, C.byref(P), seeds.ctypes.data, float(threshold), int(max_iterations), float(probability), C.byref(R),
                 r["drawn"].ctypes.data if want_drawn else None))
    return r


def _seeds(seeds, n_prob):
    s = np.ascontiguousarray(seeds, np.uint64).reshape(-1)
    if len(s) != n_prob:
        raise ValueError(f"{len(s)} seeds for {n_prob} problems")
    return s


def ransac_absolute_pose(ctx: Context, prob_ptr, pts, bearings, sigma, cam_off, cam_rot, samples, threshold, max_iterations, probability=0.99,
                         per_sample=False):
    """Se3Solver::projectiveAlignment's GP3P RANSAC for a batch of problems (cvb_ransac_absolute_pose_batch): P3P hypothesis per sample,
    scoring and ransac_select-style selection on the GPU.  prob_ptr [n_prob+1] correspondence ranges; pts / bearings [N,3], sigma [N];
    cam_off [n_prob,3], cam_rot [n_prob,3,3] (camera in the body frame); samples [n_prob, n_samples, 4] problem-local indices.
    → dict(best_sample, best_model [n_prob,3,4], best_count, iterations, consumed, inlier_mask [N]) and, with per_sample,
    sample_model [n_prob,n_samples,3,4], sample_valid, sample_count."""
    ptr = np.ascontiguousarray(prob_ptr, np.int32); n_prob = len(ptr) - 1
    p = np.ascontiguousarray(pts, np.float64).reshape(-1, 3); f = np.ascontiguousarray(bearings, np.float64).reshape(-1, 3)
    s = np.ascontiguousarray(sigma, np.float64).reshape(-1)
    co = np.ascontiguousarray(cam_off, np.float64).reshape(n_prob, 3); cr = np.ascontiguousarray(cam_rot, np.float64).reshape(n_prob, 9)
    smp = np.ascontiguousarray(samples, np.int32).reshape(n_prob, -1, 4); ns = smp.shape[1]
    P = CAbsRansacProblems(n_prob, ptr.ctypes.data, p.ctypes.data, f.ctypes.data, s.ctypes.data, co.ctypes.data, cr.ctypes.data, smp.ctypes.data, ns)
    return _ransac(ctx, lib().cvb_ransac_absolute_pose_batch, P, n_prob, ns, len(p), threshold, max_iterations, probability, per_sample)


def ransac_absolute_pose_seeded(ctx: Context, prob_ptr, pts, bearings, sigma, cam_off, cam_rot, seeds, threshold, max_iterations, probability=0.99,
                                per_sample=False, n_samples=0, want_drawn=False):
    """ransac_absolute_pose with the samples drawn on the GPU (cvb_ransac_absolute_pose_seeded_batch): seeds [n_prob] uint64, one per
    problem; the selection draws until opengv's bound ends it.  n_samples sizes the per-sample outputs (per_sample) and drawn
    [n_prob, n_samples, 4] (want_drawn: the drawn indices, -1 where not drawn)."""
    ptr = np.ascontiguousarray(prob_ptr, np.int32); n_prob = len(ptr) - 1
    p = np.ascontiguousarray(pts, np.float64).reshape(-1, 3); f = np.ascontiguousarray(bearings, np.float64).reshape(-1, 3)
    s = np.ascontiguousarray(sigma, np.float64).reshape(-1)
    co = np.ascontiguousarray(cam_off, np.float64).reshape(n_prob, 3); cr = np.ascontiguousarray(cam_rot, np.float64).reshape(n_prob, 9)
    P = CAbsRansacProblems(n_prob, ptr.ctypes.data, p.ctypes.data, f.ctypes.data, s.ctypes.data, co.ctypes.data, cr.ctypes.data, None, int(n_samples))
    return _ransac(ctx, lib().cvb_ransac_absolute_pose_seeded_batch, P, n_prob, int(n_samples), len(p), threshold, max_iterations, probability,
                   per_sample, _seeds(seeds, n_prob), 4, want_drawn)


class CRelRansacProblems(C.Structure):
    _fields_ = [("n_prob", C.c_int32)] + [(k, c_vp) for k in ("prob_ptr", "f1", "f2", "sigma1", "sigma2", "cam1", "cam2", "cam_ptr1", "cam_off1",
                                                               "cam_rot1", "cam_ptr2", "cam_off2", "cam_rot2", "samples")] + [("n_samples", C.c_int32)]


def ransac_noncentral_relative_pose(ctx: Context, prob_ptr, f1, f2, sigma1, sigma2, cam1, cam2, cam_ptr1, cam_off1, cam_rot1, cam_ptr2, cam_off2,
                                    cam_rot2, samples, threshold, max_iterations, probability=0.99, per_sample=False):
    """RelNonCentralPosSolver::computeNonCentralRelPose's 17-point RANSAC for a batch of problems
    (cvb_ransac_noncentral_relative_pose_batch): 17-point hypothesis per sample, scoring per camera pair and ransac_select-style
    selection on the GPU.  prob_ptr [n_prob+1] correspondence ranges; f1 / f2 [N,3] bearings in their cameras' frames, sigma1 /
    sigma2 [N], cam1 / cam2 [N] problem-local camera indices; cam_ptr1 [n_prob+1] rig-1 camera ranges, cam_off1 [C1,3],
    cam_rot1 [C1,3,3] (cameras in the rig frame), rig 2 likewise; samples [n_prob, n_samples, 17] problem-local indices.
    → dict(best_sample, best_model [n_prob,3,4] (X1 = R X2 + t), best_count, iterations, consumed, inlier_mask [N]) and, with
    per_sample, sample_model [n_prob,n_samples,3,4], sample_valid, sample_count."""
    ptr = np.ascontiguousarray(prob_ptr, np.int32); n_prob = len(ptr) - 1
    a = np.ascontiguousarray(f1, np.float64).reshape(-1, 3); b = np.ascontiguousarray(f2, np.float64).reshape(-1, 3)
    s1 = np.ascontiguousarray(sigma1, np.float64).reshape(-1); s2 = np.ascontiguousarray(sigma2, np.float64).reshape(-1)
    c1 = np.ascontiguousarray(cam1, np.int32).reshape(-1); c2 = np.ascontiguousarray(cam2, np.int32).reshape(-1)
    cp1 = np.ascontiguousarray(cam_ptr1, np.int32); cp2 = np.ascontiguousarray(cam_ptr2, np.int32)
    co1 = np.ascontiguousarray(cam_off1, np.float64).reshape(-1, 3); cr1 = np.ascontiguousarray(cam_rot1, np.float64).reshape(-1, 9)
    co2 = np.ascontiguousarray(cam_off2, np.float64).reshape(-1, 3); cr2 = np.ascontiguousarray(cam_rot2, np.float64).reshape(-1, 9)
    smp = np.ascontiguousarray(samples, np.int32).reshape(n_prob, -1, 17); ns = smp.shape[1]
    P = CRelRansacProblems(n_prob, *[x.ctypes.data for x in (ptr, a, b, s1, s2, c1, c2, cp1, co1, cr1, cp2, co2, cr2, smp)], ns)
    return _ransac(ctx, lib().cvb_ransac_noncentral_relative_pose_batch, P, n_prob, ns, len(a), threshold, max_iterations, probability, per_sample)


def ransac_noncentral_relative_pose_seeded(ctx: Context, prob_ptr, f1, f2, sigma1, sigma2, cam1, cam2, cam_ptr1, cam_off1, cam_rot1, cam_ptr2,
                                           cam_off2, cam_rot2, seeds, threshold, max_iterations, probability=0.99, per_sample=False, n_samples=0,
                                           want_drawn=False):
    """ransac_noncentral_relative_pose with the samples drawn on the GPU (cvb_ransac_noncentral_relative_pose_seeded_batch); seeds,
    n_samples and want_drawn as ransac_absolute_pose_seeded (drawn [n_prob, n_samples, 17])."""
    ptr = np.ascontiguousarray(prob_ptr, np.int32); n_prob = len(ptr) - 1
    a = np.ascontiguousarray(f1, np.float64).reshape(-1, 3); b = np.ascontiguousarray(f2, np.float64).reshape(-1, 3)
    s1 = np.ascontiguousarray(sigma1, np.float64).reshape(-1); s2 = np.ascontiguousarray(sigma2, np.float64).reshape(-1)
    c1 = np.ascontiguousarray(cam1, np.int32).reshape(-1); c2 = np.ascontiguousarray(cam2, np.int32).reshape(-1)
    cp1 = np.ascontiguousarray(cam_ptr1, np.int32); cp2 = np.ascontiguousarray(cam_ptr2, np.int32)
    co1 = np.ascontiguousarray(cam_off1, np.float64).reshape(-1, 3); cr1 = np.ascontiguousarray(cam_rot1, np.float64).reshape(-1, 9)
    co2 = np.ascontiguousarray(cam_off2, np.float64).reshape(-1, 3); cr2 = np.ascontiguousarray(cam_rot2, np.float64).reshape(-1, 9)
    P = CRelRansacProblems(n_prob, *[x.ctypes.data for x in (ptr, a, b, s1, s2, c1, c2, cp1, co1, cr1, cp2, co2, cr2)], None, int(n_samples))
    return _ransac(ctx, lib().cvb_ransac_noncentral_relative_pose_seeded_batch, P, n_prob, int(n_samples), len(a), threshold, max_iterations,
                   probability, per_sample, _seeds(seeds, n_prob), 17, want_drawn)


class CCentralRelRansacProblems(C.Structure):
    _fields_ = [("n_prob", C.c_int32)] + [(k, c_vp) for k in ("prob_ptr", "f1", "f2", "sigma1", "sigma2", "samples")] + [("n_samples", C.c_int32)]


def ransac_central_relative_pose(ctx: Context, prob_ptr, f1, f2, sigma1, sigma2, samples, threshold, max_iterations, probability=0.99,
                                 per_sample=False):
    """RelNonCentralPosSolver::computePose's 5-point RANSAC for a batch of problems (cvb_ransac_central_relative_pose_batch):
    5-point hypothesis per sample, scoring and ransac_select-style selection on the GPU.  prob_ptr [n_prob+1] correspondence
    ranges; f1 / f2 [N,3] unit bearings, sigma1 / sigma2 [N]; samples [n_prob, n_samples, 5] problem-local indices.
    → dict(best_sample, best_model [n_prob,3,4] (X1 = R X2 + t, |t| = 1), best_count, iterations, consumed, inlier_mask [N]) and,
    with per_sample, sample_model [n_prob,n_samples,3,4], sample_valid, sample_count."""
    ptr = np.ascontiguousarray(prob_ptr, np.int32); n_prob = len(ptr) - 1
    a = np.ascontiguousarray(f1, np.float64).reshape(-1, 3); b = np.ascontiguousarray(f2, np.float64).reshape(-1, 3)
    s1 = np.ascontiguousarray(sigma1, np.float64).reshape(-1); s2 = np.ascontiguousarray(sigma2, np.float64).reshape(-1)
    smp = np.ascontiguousarray(samples, np.int32).reshape(n_prob, -1, 5); ns = smp.shape[1]
    P = CCentralRelRansacProblems(n_prob, *[x.ctypes.data for x in (ptr, a, b, s1, s2, smp)], ns)
    return _ransac(ctx, lib().cvb_ransac_central_relative_pose_batch, P, n_prob, ns, len(a), threshold, max_iterations, probability, per_sample)


def ransac_central_relative_pose_seeded(ctx: Context, prob_ptr, f1, f2, sigma1, sigma2, seeds, threshold, max_iterations, probability=0.99,
                                        per_sample=False, n_samples=0, want_drawn=False):
    """ransac_central_relative_pose with the samples drawn on the GPU (cvb_ransac_central_relative_pose_seeded_batch); seeds,
    n_samples and want_drawn as ransac_absolute_pose_seeded (drawn [n_prob, n_samples, 5])."""
    ptr = np.ascontiguousarray(prob_ptr, np.int32); n_prob = len(ptr) - 1
    a = np.ascontiguousarray(f1, np.float64).reshape(-1, 3); b = np.ascontiguousarray(f2, np.float64).reshape(-1, 3)
    s1 = np.ascontiguousarray(sigma1, np.float64).reshape(-1); s2 = np.ascontiguousarray(sigma2, np.float64).reshape(-1)
    P = CCentralRelRansacProblems(n_prob, *[x.ctypes.data for x in (ptr, a, b, s1, s2)], None, int(n_samples))
    return _ransac(ctx, lib().cvb_ransac_central_relative_pose_seeded_batch, P, n_prob, int(n_samples), len(a), threshold, max_iterations,
                   probability, per_sample, _seeds(seeds, n_prob), 5, want_drawn)


class CRelCovResult(C.Structure):
    _fields_ = [(k, c_vp) for k in ("cov", "n_valid", "sample_delta", "sample_valid")]


def relative_pose_covariance(ctx: Context, prob_ptr, f1, f2, cam1, cam2, cam_ptr1, cam_off1, cam_rot1, cam_ptr2, cam_off2, cam_rot2, samples,
                             ref_model, per_sample=False, sigma1=None, sigma2=None):
    """The sampling-based 6x6 covariance of RelNonCentralPosSolver::computeNonCentralRelPose for a batch of problems
    (cvb_noncentral_relative_pose_covariance_batch): a 17-point re-solve per sample, its deviation
    delta = [2 vec(q); t_s - t_ref] (q the quaternion of R_ref^T R_s, w >= 0) from the reference model, and
    cov = sum delta delta^T / n_valid over the valid samples, on the GPU.  Arguments as ransac_noncentral_relative_pose (sigma1 /
    sigma2 are accepted and not read); samples [n_prob, n_samples, 17] problem-local indices, normally drawn from the inlier
    mask of the RANSAC; ref_model [n_prob,3,4] (X1 = R X2 + t), normally its best_model (all zeros: the problem is skipped).
    → dict(cov [n_prob,6,6] (rotation then translation), n_valid [n_prob]) and, with per_sample, sample_delta
    [n_prob,n_samples,6], sample_valid [n_prob,n_samples]."""
    ptr = np.ascontiguousarray(prob_ptr, np.int32); n_prob = len(ptr) - 1
    a = np.ascontiguousarray(f1, np.float64).reshape(-1, 3); b = np.ascontiguousarray(f2, np.float64).reshape(-1, 3)
    c1 = np.ascontiguousarray(cam1, np.int32).reshape(-1); c2 = np.ascontiguousarray(cam2, np.int32).reshape(-1)
    cp1 = np.ascontiguousarray(cam_ptr1, np.int32); cp2 = np.ascontiguousarray(cam_ptr2, np.int32)
    co1 = np.ascontiguousarray(cam_off1, np.float64).reshape(-1, 3); cr1 = np.ascontiguousarray(cam_rot1, np.float64).reshape(-1, 9)
    co2 = np.ascontiguousarray(cam_off2, np.float64).reshape(-1, 3); cr2 = np.ascontiguousarray(cam_rot2, np.float64).reshape(-1, 9)
    smp = np.ascontiguousarray(samples, np.int32).reshape(n_prob, -1, 17); ns = smp.shape[1]
    ref = np.ascontiguousarray(ref_model, np.float64).reshape(n_prob, 12)
    r = dict(cov=np.zeros((n_prob, 6, 6)), n_valid=np.zeros(n_prob, np.int32))
    if per_sample:
        r.update(sample_delta=np.zeros((n_prob, ns, 6)), sample_valid=np.zeros((n_prob, ns), np.uint8))
    P = CRelRansacProblems(n_prob, ptr.ctypes.data, a.ctypes.data, b.ctypes.data, None, None,
                           *[x.ctypes.data for x in (c1, c2, cp1, co1, cr1, cp2, co2, cr2, smp)], ns)
    R = CRelCovResult(*[r[k].ctypes.data if k in r else None for k, _ in CRelCovResult._fields_])
    ctx.check(lib().cvb_noncentral_relative_pose_covariance_batch(ctx.handle, C.byref(P), ref.ctypes.data, C.byref(R)))
    return r


def relative_pose_covariance_seeded(ctx: Context, prob_ptr, f1, f2, cam1, cam2, cam_ptr1, cam_off1, cam_rot1, cam_ptr2, cam_off2, cam_rot2,
                                    inlier_mask, seeds, ref_model, n_samples=300, per_sample=False, want_drawn=False, sigma1=None, sigma2=None):
    """relative_pose_covariance with the samples drawn on the GPU (cvb_noncentral_relative_pose_covariance_seeded_batch): n_samples
    17-point subsets per problem of its inliers in inlier_mask [N] (normally the RANSAC's), drawn from seeds [n_prob] uint64.
    A problem with fewer than 17 inliers or a zero ref_model gets n_valid 0.  want_drawn: also drawn [n_prob, n_samples, 17], the
    problem-local correspondence indices (-1 where not drawn)."""
    ptr = np.ascontiguousarray(prob_ptr, np.int32); n_prob = len(ptr) - 1
    a = np.ascontiguousarray(f1, np.float64).reshape(-1, 3); b = np.ascontiguousarray(f2, np.float64).reshape(-1, 3)
    c1 = np.ascontiguousarray(cam1, np.int32).reshape(-1); c2 = np.ascontiguousarray(cam2, np.int32).reshape(-1)
    cp1 = np.ascontiguousarray(cam_ptr1, np.int32); cp2 = np.ascontiguousarray(cam_ptr2, np.int32)
    co1 = np.ascontiguousarray(cam_off1, np.float64).reshape(-1, 3); cr1 = np.ascontiguousarray(cam_rot1, np.float64).reshape(-1, 9)
    co2 = np.ascontiguousarray(cam_off2, np.float64).reshape(-1, 3); cr2 = np.ascontiguousarray(cam_rot2, np.float64).reshape(-1, 9)
    mask = np.ascontiguousarray(inlier_mask, np.uint8).reshape(-1)
    ref = np.ascontiguousarray(ref_model, np.float64).reshape(n_prob, 12)
    seeds = _seeds(seeds, n_prob); ns = int(n_samples)
    r = dict(cov=np.zeros((n_prob, 6, 6)), n_valid=np.zeros(n_prob, np.int32))
    if per_sample:
        r.update(sample_delta=np.zeros((n_prob, ns, 6)), sample_valid=np.zeros((n_prob, ns), np.uint8))
    if want_drawn:
        r["drawn"] = np.full((n_prob, ns, 17), -1, np.int32)
    P = CRelRansacProblems(n_prob, ptr.ctypes.data, a.ctypes.data, b.ctypes.data, None, None,
                           *[x.ctypes.data for x in (c1, c2, cp1, co1, cr1, cp2, co2, cr2)], None, ns)
    R = CRelCovResult(*[r[k].ctypes.data if k in r else None for k, _ in CRelCovResult._fields_])
    ctx.check(lib().cvb_noncentral_relative_pose_covariance_seeded_batch(ctx.handle, C.byref(P), ref.ctypes.data, mask.ctypes.data, seeds.ctypes.data,
                                                                         C.byref(R), r["drawn"].ctypes.data if want_drawn else None))
    return r


class CVerifyKeyframes(C.Structure):
    _fields_ = [("n_kf", C.c_int32)] + [(k, c_vp) for k in ("kf_ptr", "desc", "bearings", "sigma")]


class CVerifyCandidates(C.Structure):
    _fields_ = [("n_cand", C.c_int32)] + [(k, c_vp) for k in ("cam_ptr1", "cam_off1", "cam_rot1", "cam_ptr2", "cam_off2", "cam_rot2", "pair_ptr",
                                                               "pairs")]


class CVerifyParams(C.Structure):
    _fields_ = [("img_match_thres", C.c_float), ("ratio_thres", C.c_float), ("threshold5", C.c_double), ("max_iterations5", C.c_int32),
                ("threshold17", C.c_double), ("max_iterations17", C.c_int32), ("probability", C.c_double), ("n_cov_samples", C.c_int32)]


class CVerifyResult(C.Structure):
    _fields_ = [(k, c_vp) for k in ("n_matches", "best_sample5", "best_model5", "best_count5", "iterations5", "consumed5", "best_sample", "best_model",
                                    "best_count", "iterations", "consumed", "cov", "n_valid", "corr")] + \
               [("corr_cap", C.c_int32), ("n_total", C.c_int32)]


def verify_noncentral_relative_pose_seeded(ctx: Context, kf_ptr, desc, bearings, sigma, cam_ptr1, cam_off1, cam_rot1, cam_ptr2, cam_off2, cam_rot2,
                                           pair_ptr, pairs, seeds5, seeds, img_match_thres, ratio_thres, threshold5, max_iterations5, threshold17,
                                           max_iterations17, probability=0.99, n_cov_samples=300, corr_cap=None):
    """RelNonCentralPosSolver::computeNonCentralRelPose's verification of place-recognition candidates in one call
    (cvb_verify_noncentral_relative_pose_seeded_batch): per pairing (kf1, kf2, cam1, cam2) the fused 2-NN + ratio filter of
    match_candidates_hamming and a seeded 5-point RANSAC on its matches; per candidate a seeded 17-point RANSAC on the pairings'
    5-point inliers and the seeded covariance on its inliers.  Keyframe table: kf_ptr [n_kf+1] row offsets into desc [R,32] u8,
    bearings [R,3], sigma [R].  Candidates: rigs as ransac_noncentral_relative_pose (cam_ptr1 [n_cand+1], ...), pair_ptr
    [n_cand+1], pairs [n_pairings,4] (kf1, kf2, cam1, cam2); seeds5 [n_pairings], seeds [n_cand] uint64.
    corr_cap: capacity of the correspondence list (None: room for every match, 0: no list).
    → dict(n_matches, best_sample5, best_model5 [P,3,4], best_count5, iterations5, consumed5 (per pairing); best_sample,
    best_model [C,3,4], best_count, iterations, consumed, cov [C,6,6], n_valid (per candidate); n_total; and, unless
    corr_cap = 0 or n_total > corr_cap, corr [n_total,5] = (pairing, row1, row2, inlier5, inlier17))."""
    return _verify_noncentral(ctx, "cvb_verify_noncentral_relative_pose_seeded_batch", np.ascontiguousarray(desc, np.uint8).reshape(-1, 32), kf_ptr,
                              bearings, sigma, cam_ptr1, cam_off1, cam_rot1, cam_ptr2, cam_off2, cam_rot2, pair_ptr, pairs, seeds5, seeds,
                              img_match_thres, ratio_thres, threshold5, max_iterations5, threshold17, max_iterations17, probability, n_cov_samples,
                              corr_cap)


def verify_noncentral_relative_pose_sift_seeded(ctx: Context, kf_ptr, desc, bearings, sigma, cam_ptr1, cam_off1, cam_rot1, cam_ptr2, cam_off2,
                                                cam_rot2, pair_ptr, pairs, seeds5, seeds, img_match_thres, ratio_thres, threshold5, max_iterations5,
                                                threshold17, max_iterations17, probability=0.99, n_cov_samples=300, corr_cap=None):
    """verify_noncentral_relative_pose_seeded with SIFT descriptors (cvb_verify_noncentral_relative_pose_sift_seeded_batch): desc
    [R,128] float32, integer-valued in [0,255] as cv::xfeatures2d::SIFT writes them (otherwise CVB_ERR_UNSUPPORTED); each pairing
    is matched by the fused 2-NN + ratio filter of match_candidates_l2 (exact L2).  Other arguments and the result dict as
    verify_noncentral_relative_pose_seeded; the reference's SIFT thresholds are about img_match_thres=500, ratio_thres=0.8."""
    return _verify_noncentral(ctx, "cvb_verify_noncentral_relative_pose_sift_seeded_batch", np.ascontiguousarray(desc, np.float32).reshape(-1, 128),
                              kf_ptr, bearings, sigma, cam_ptr1, cam_off1, cam_rot1, cam_ptr2, cam_off2, cam_rot2, pair_ptr, pairs, seeds5, seeds,
                              img_match_thres, ratio_thres, threshold5, max_iterations5, threshold17, max_iterations17, probability, n_cov_samples,
                              corr_cap)


def _verify_noncentral(ctx: Context, fn, dsc, kf_ptr, bearings, sigma, cam_ptr1, cam_off1, cam_rot1, cam_ptr2, cam_off2, cam_rot2, pair_ptr, pairs,
                       seeds5, seeds, img_match_thres, ratio_thres, threshold5, max_iterations5, threshold17, max_iterations17, probability,
                       n_cov_samples, corr_cap):
    """the body of verify_noncentral_relative_pose{,_sift}_seeded: the C call fn on the contiguous descriptor table dsc"""
    kp = np.ascontiguousarray(kf_ptr, np.int32); n_kf = len(kp) - 1
    f = np.ascontiguousarray(bearings, np.float64).reshape(-1, 3)
    sg = np.ascontiguousarray(sigma, np.float64).reshape(-1)
    cp1 = np.ascontiguousarray(cam_ptr1, np.int32); cp2 = np.ascontiguousarray(cam_ptr2, np.int32); n_cand = len(cp1) - 1
    co1 = np.ascontiguousarray(cam_off1, np.float64).reshape(-1, 3); cr1 = np.ascontiguousarray(cam_rot1, np.float64).reshape(-1, 9)
    co2 = np.ascontiguousarray(cam_off2, np.float64).reshape(-1, 3); cr2 = np.ascontiguousarray(cam_rot2, np.float64).reshape(-1, 9)
    pp = np.ascontiguousarray(pair_ptr, np.int32); pr = np.ascontiguousarray(pairs, np.int32).reshape(-1, 4); P = len(pr)
    s5 = _seeds(seeds5, P); s17 = _seeds(seeds, n_cand)
    if corr_cap is None:
        corr_cap = int(sum(kp[a + 1] - kp[a] for a in pr[:, 0])) if P and n_kf > 0 and pr[:, 0].min() >= 0 and pr[:, 0].max() < n_kf else 0
    r = dict(n_matches=np.zeros(P, np.int32), best_sample5=np.zeros(P, np.int32), best_model5=np.zeros((P, 3, 4)), best_count5=np.zeros(P, np.int32),
             iterations5=np.zeros(P, np.int32), consumed5=np.zeros(P, np.int32), best_sample=np.zeros(n_cand, np.int32),
             best_model=np.zeros((n_cand, 3, 4)), best_count=np.zeros(n_cand, np.int32), iterations=np.zeros(n_cand, np.int32),
             consumed=np.zeros(n_cand, np.int32), cov=np.zeros((n_cand, 6, 6)), n_valid=np.zeros(n_cand, np.int32))
    corr = np.zeros((max(int(corr_cap), 1), 5), np.int32)
    K = CVerifyKeyframes(n_kf, *[x.ctypes.data for x in (kp, dsc, f, sg)])
    D = CVerifyCandidates(n_cand, *[x.ctypes.data for x in (cp1, co1, cr1, cp2, co2, cr2, pp, pr)])
    Pm = CVerifyParams(float(img_match_thres), float(ratio_thres), float(threshold5), int(max_iterations5), float(threshold17), int(max_iterations17),
                       float(probability), int(n_cov_samples))
    R = CVerifyResult(*[r[k].ctypes.data for k, _ in CVerifyResult._fields_[:13]], corr.ctypes.data if corr_cap else None, int(corr_cap), 0)
    ctx.check(getattr(lib(), fn)(ctx.handle, C.byref(K), C.byref(D), C.byref(Pm), s5.ctypes.data, s17.ctypes.data, C.byref(R)))
    r["n_total"] = int(R.n_total)
    if corr_cap and R.n_total <= corr_cap:
        r["corr"] = corr[:R.n_total].copy()
    return r


class CLandmarkKf(C.Structure):
    _fields_ = [("view", CKfView), ("bearings", c_vp), ("sigma_angle", c_vp), ("T_ws", C.c_double * 16), ("T_sc", C.c_double * 16),
                ("intr", C.c_double * 4), ("dist", C.c_double * 4), ("cam_model", C.c_int32), ("dist_model", C.c_int32), ("xi", C.c_double)]


class CLandmarkVerifyParams(C.Structure):
    _fields_ = [("thr", C.c_float), ("num_best", C.c_int32), ("min_matches", C.c_int32), ("threshold", C.c_double), ("max_iterations", C.c_int32),
                ("probability", C.c_double), ("min_ransac_inliers", C.c_int32), ("search", CSearchParams), ("th_outlier_align", C.c_double)]


class CLandmarkVerifyResult(C.Structure):
    _fields_ = [(k, c_vp) for k in ("n_matches", "best_sample", "best_model", "best_count", "iterations", "consumed", "T12", "T21", "n_found", "n_corr",
                                    "T12_out", "n_inliers", "solve_iterations", "match12", "stage", "removed")]


class LandmarkKf:
    """a keyframe of verify_landmark_candidates_seeded: the KfView SearchBySE3 reads, plus bearings [n,3] (unit, camera frame) and
    sigma_angle [n] (read of the query only), T_ws / T_sc (4x4 body in world, camera in body) and the camera model
    cam = dict(intr[4], dist[4], cam_model=0, dist_model=0, xi=0) of optimize_relative_pose"""

    def __init__(self, view: KfView, T_ws, T_sc, cam: dict, bearings=None, sigma_angle=None):
        self.view, self.cam = view, cam
        self.T_ws = np.asarray(T_ws, np.float64).reshape(16); self.T_sc = np.asarray(T_sc, np.float64).reshape(16)
        self.bearings = np.ascontiguousarray(np.zeros((view.n, 3)) if bearings is None else bearings, np.float64).reshape(view.n, 3)
        self.sigma_angle = np.ascontiguousarray(np.ones(view.n) if sigma_angle is None else sigma_angle, np.float64).reshape(view.n)

    def cstruct(self):
        s = CLandmarkKf()
        s.view = self.view.cstruct()
        s.bearings, s.sigma_angle = self.bearings.ctypes.data, self.sigma_angle.ctypes.data
        s.T_ws[:] = self.T_ws.tolist(); s.T_sc[:] = self.T_sc.tolist()
        s.intr[:] = [float(x) for x in np.asarray(self.cam["intr"]).reshape(4)]; s.dist[:] = [float(x) for x in np.asarray(self.cam["dist"]).reshape(4)]
        s.cam_model, s.dist_model, s.xi = int(self.cam.get("cam_model", 0)), int(self.cam.get("dist_model", 0)), float(self.cam.get("xi", 0.0))
        return s


def landmark_verify_prepared(ctx: Context, query: LandmarkKf, cands, seeds, min_matches, threshold, max_iterations, min_ransac_inliers, thr=50.0,
                             num_best=4, probability=0.99, th=9.5, desc_th_low=50, num_octaves=1, scale_factor=2.0, th_outlier_align=1.3, detail=True):
    """PlaceRecognition::ComputeSE3's verification of place-recognition candidates in one call
    (cvb_verify_landmark_candidates_seeded_batch): DenseMatcher landmark matching of the query against every candidate, a seeded
    GP3P RANSAC per candidate with at least min_matches matches, the gate (best_count >= min_ransac_inliers), SearchBySE3 and the
    relative-pose refinement.  cands: LandmarkKf list, seeds [n_cand] uint64.  detail: also the [n_cand, n_query] outputs.
    → dict(n_matches, best_sample, best_model [C,3,4], best_count, iterations, consumed, T12 / T21 [C,4,4], n_found, n_corr,
    T12_out [C,7], n_inliers, solve_iterations [C,2]) and, with detail, match12 [C,nq] i32, stage [C,nq] u8 (0 none, 1 DenseMatcher
    match not kept by the RANSAC, 2 RANSAC inlier, 3 added by SearchBySE3), removed [C,nq] u8 (by residual index, < n_corr).
    Packs the arguments once and returns (call, result dict): call() runs the C call on them and returns the filled dict."""
    C_, nq = len(cands), query.view.n
    s = _seeds(seeds, C_)
    r = dict(n_matches=np.zeros(C_, np.int32), best_sample=np.zeros(C_, np.int32), best_model=np.zeros((C_, 3, 4)), best_count=np.zeros(C_, np.int32),
             iterations=np.zeros(C_, np.int32), consumed=np.zeros(C_, np.int32), T12=np.zeros((C_, 4, 4)), T21=np.zeros((C_, 4, 4)),
             n_found=np.zeros(C_, np.int32), n_corr=np.zeros(C_, np.int32), T12_out=np.zeros((C_, 7)), n_inliers=np.zeros(C_, np.int32),
             solve_iterations=np.zeros((C_, 2), np.int32))
    if detail:
        r.update(match12=np.zeros((C_, nq), np.int32), stage=np.zeros((C_, nq), np.uint8), removed=np.zeros((C_, nq), np.uint8))
    q = query.cstruct()
    arr = (CLandmarkKf * max(C_, 1))(*[c.cstruct() for c in cands])
    prm = CLandmarkVerifyParams(float(thr), int(num_best), int(min_matches), float(threshold), int(max_iterations), float(probability),
                                int(min_ransac_inliers), CSearchParams(float(th), int(desc_th_low), int(num_octaves), float(scale_factor)),
                                float(th_outlier_align))
    R = CLandmarkVerifyResult(*[r[k].ctypes.data if k in r else None for k, _ in CLandmarkVerifyResult._fields_])
    keep = (q, arr, prm, R, s, query, cands)

    def call():
        ctx.check(lib().cvb_verify_landmark_candidates_seeded_batch(ctx.handle, C.byref(keep[0]), keep[1], C_, C.byref(keep[2]), keep[4].ctypes.data,
                                                                    C.byref(keep[3])))
        return r
    return call, r


def verify_landmark_candidates_seeded(ctx: Context, query: LandmarkKf, cands, seeds, min_matches, threshold, max_iterations, min_ransac_inliers,
                                      **kw):
    """PlaceRecognition::ComputeSE3's verification of place-recognition candidates in one call
    (cvb_verify_landmark_candidates_seeded_batch); the arguments and result of landmark_verify_prepared, which see"""
    call, _ = landmark_verify_prepared(ctx, query, cands, seeds, min_matches, threshold, max_iterations, min_ransac_inliers, **kw)
    return call()
