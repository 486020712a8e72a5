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


class CAbsRansacResult(C.Structure):
    _fields_ = [(k, c_vp) for k in ("best_sample", "best_model", "best_count", "iterations", "consumed", "inlier_mask", "sample_model",
                                    "sample_valid", "sample_count")]


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
    r = dict(best_sample=np.zeros(n_prob, np.int32), best_model=np.zeros((n_prob, 3, 4)), best_count=np.zeros(n_prob, np.int32),
             iterations=np.zeros(n_prob, np.int32), consumed=np.zeros(n_prob, np.int32), inlier_mask=np.zeros(len(p), np.uint8))
    if per_sample:
        r.update(sample_model=np.zeros((n_prob, ns, 3, 4)), sample_valid=np.zeros((n_prob, ns), np.uint8),
                 sample_count=np.zeros((n_prob, ns), np.int32))
    P = CAbsRansacProblems(n_prob, ptr.ctypes.data, p.ctypes.data, f.ctypes.data, s.ctypes.data, co.ctypes.data, cr.ctypes.data, smp.ctypes.data, ns)
    R = CAbsRansacResult(*[r[k].ctypes.data if k in r else None for k, _ in CAbsRansacResult._fields_])
    ctx.check(lib().cvb_ransac_absolute_pose_batch(ctx.handle, C.byref(P), float(threshold), int(max_iterations), float(probability), C.byref(R)))
    return r


class CRelRansacProblems(C.Structure):
    _fields_ = [("n_prob", C.c_int32)] + [(k, c_vp) for k in ("prob_ptr", "f1", "f2", "sigma1", "sigma2", "cam1", "cam2", "cam_ptr1", "cam_off1",
                                                               "cam_rot1", "cam_ptr2", "cam_off2", "cam_rot2", "samples")] + [("n_samples", C.c_int32)]


class CRelRansacResult(CAbsRansacResult):
    pass


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
    r = dict(best_sample=np.zeros(n_prob, np.int32), best_model=np.zeros((n_prob, 3, 4)), best_count=np.zeros(n_prob, np.int32),
             iterations=np.zeros(n_prob, np.int32), consumed=np.zeros(n_prob, np.int32), inlier_mask=np.zeros(len(a), np.uint8))
    if per_sample:
        r.update(sample_model=np.zeros((n_prob, ns, 3, 4)), sample_valid=np.zeros((n_prob, ns), np.uint8),
                 sample_count=np.zeros((n_prob, ns), np.int32))
    P = CRelRansacProblems(n_prob, *[x.ctypes.data for x in (ptr, a, b, s1, s2, c1, c2, cp1, co1, cr1, cp2, co2, cr2, smp)], ns)
    R = CRelRansacResult(*[r[k].ctypes.data if k in r else None for k, _ in CRelRansacResult._fields_])
    ctx.check(lib().cvb_ransac_noncentral_relative_pose_batch(ctx.handle, C.byref(P), float(threshold), int(max_iterations), float(probability),
                                                              C.byref(R)))
    return r


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
    r = dict(best_sample=np.zeros(n_prob, np.int32), best_model=np.zeros((n_prob, 3, 4)), best_count=np.zeros(n_prob, np.int32),
             iterations=np.zeros(n_prob, np.int32), consumed=np.zeros(n_prob, np.int32), inlier_mask=np.zeros(len(a), np.uint8))
    if per_sample:
        r.update(sample_model=np.zeros((n_prob, ns, 3, 4)), sample_valid=np.zeros((n_prob, ns), np.uint8),
                 sample_count=np.zeros((n_prob, ns), np.int32))
    P = CCentralRelRansacProblems(n_prob, *[x.ctypes.data for x in (ptr, a, b, s1, s2, smp)], ns)
    R = CRelRansacResult(*[r[k].ctypes.data if k in r else None for k, _ in CRelRansacResult._fields_])
    ctx.check(lib().cvb_ransac_central_relative_pose_batch(ctx.handle, C.byref(P), float(threshold), int(max_iterations), float(probability),
                                                           C.byref(R)))
    return r
