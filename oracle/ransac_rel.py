"""ctypes binding of oracle/ransac_rel_oracle.c (17-point hypotheses + non-central relative-pose RANSAC selection) — TEST
INFRASTRUCTURE ONLY."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libcovins_ransac_rel_oracle.so")
_LIB = None
c_vp = C.c_void_p


def build(out=LIB_PATH):
    """-ffp-contract=off: the CUDA path is compared bit for bit against plain IEEE evaluation"""
    subprocess.check_call(["gcc", "-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-Wall", "-Wextra", "-std=c11", "-fvisibility=hidden",
                           "-ffp-contract=off", "-shared", "-o", out, os.path.join(_HERE, "ransac_rel_oracle.c"), "-lm"])


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            build()
        _LIB = C.CDLL(LIB_PATH)
    return _LIB


def _rig(off, rot):
    return np.ascontiguousarray(off, np.float64).reshape(-1, 3), np.ascontiguousarray(rot, np.float64).reshape(-1, 9)


def rel17(f1, f2, cam1, cam2, cam_off1, cam_rot1, cam_off2, cam_rot2, sample):
    """one problem's correspondences and rigs, one sample of 17 local indices → (model [3,4] (zeros if invalid), valid, rank ratio
    min |r_kk| / max |r_kk| of the QR (0 when the QR is not reached))"""
    a = np.ascontiguousarray(f1, np.float64).reshape(-1, 3); b = np.ascontiguousarray(f2, np.float64).reshape(-1, 3)
    c1 = np.ascontiguousarray(cam1, np.int32); c2 = np.ascontiguousarray(cam2, np.int32)
    co1, cr1 = _rig(cam_off1, cam_rot1); co2, cr2 = _rig(cam_off2, cam_rot2)
    s = np.ascontiguousarray(sample, np.int32).reshape(17)
    model = np.zeros((3, 4)); ratio = C.c_double(0.0)
    v = lib().ora_rel17(len(a), c_vp(a.ctypes.data), c_vp(b.ctypes.data), c_vp(c1.ctypes.data), c_vp(c2.ctypes.data), len(co1), c_vp(co1.ctypes.data),
                        c_vp(cr1.ctypes.data), len(co2), c_vp(co2.ctypes.data), c_vp(cr2.ctypes.data), c_vp(s.ctypes.data),
                        c_vp(model.ctypes.data), C.byref(ratio))
    return model, bool(v), ratio.value


def rel_pair_model(model, cam_off1, cam_rot1, cam_off2, cam_rot2):
    """camera-pair model [R_p|t_p] [3,4] of a rig-frame model (camera 1 of rig 1, camera 2 of rig 2)"""
    M = np.ascontiguousarray(model, np.float64).reshape(12); out = np.zeros((3, 4))
    co1, cr1 = _rig(cam_off1, cam_rot1); co2, cr2 = _rig(cam_off2, cam_rot2)
    lib().ora_rel_pair_model(c_vp(M.ctypes.data), c_vp(co1.ctypes.data), c_vp(cr1.ctypes.data), c_vp(co2.ctypes.data), c_vp(cr2.ctypes.data),
                             c_vp(out.ctypes.data))
    return out


def score_noncentral_relative_pose(models, f1, f2, sigma1, sigma2, cam1, cam2, cam_off1, cam_rot1, cam_off2, cam_rot2, threshold):
    """rig-frame models [H,3,4] over one problem → (scores [H,n], inlier [H,n], n_inliers [H])"""
    m = np.ascontiguousarray(models, np.float64).reshape(-1, 12)
    a = np.ascontiguousarray(f1, np.float64).reshape(-1, 3); b = np.ascontiguousarray(f2, np.float64).reshape(-1, 3)
    s1 = np.ascontiguousarray(sigma1, np.float64); s2 = np.ascontiguousarray(sigma2, np.float64)
    c1 = np.ascontiguousarray(cam1, np.int32); c2 = np.ascontiguousarray(cam2, np.int32)
    co1, cr1 = _rig(cam_off1, cam_rot1); co2, cr2 = _rig(cam_off2, cam_rot2)
    H, n = len(m), len(a)
    sc = np.zeros((H, n)); inl = np.zeros((H, n), np.uint8); cnt = np.zeros(max(H, 1), np.int32)
    lib().ora_score_noncentral_relative_pose(c_vp(m.ctypes.data), H, n, c_vp(a.ctypes.data), c_vp(b.ctypes.data), c_vp(s1.ctypes.data),
                                             c_vp(s2.ctypes.data), c_vp(c1.ctypes.data), c_vp(c2.ctypes.data), len(co1), c_vp(co1.ctypes.data),
                                             c_vp(cr1.ctypes.data), len(co2), c_vp(co2.ctypes.data), c_vp(cr2.ctypes.data), C.c_double(threshold),
                                             c_vp(sc.ctypes.data), c_vp(inl.ctypes.data), c_vp(cnt.ctypes.data))
    return sc, inl, cnt[:H]


def rel_hypotheses(f1, f2, cam1, cam2, cam_off1, cam_rot1, cam_off2, cam_rot2, samples):
    """17-point hypotheses of one problem's samples [S,17] → (models [S,3,4], valid [S])"""
    a = np.ascontiguousarray(f1, np.float64).reshape(-1, 3); b = np.ascontiguousarray(f2, np.float64).reshape(-1, 3)
    c1 = np.ascontiguousarray(cam1, np.int32); c2 = np.ascontiguousarray(cam2, np.int32)
    co1, cr1 = _rig(cam_off1, cam_rot1); co2, cr2 = _rig(cam_off2, cam_rot2)
    smp = np.ascontiguousarray(samples, np.int32).reshape(-1, 17)
    models = np.zeros((len(smp), 3, 4)); valid = np.zeros(len(smp), np.uint8)
    lib().ora_rel_hypotheses(len(a), c_vp(a.ctypes.data), c_vp(b.ctypes.data), c_vp(c1.ctypes.data), c_vp(c2.ctypes.data), len(co1),
                             c_vp(co1.ctypes.data), c_vp(cr1.ctypes.data), len(co2), c_vp(co2.ctypes.data), c_vp(cr2.ctypes.data),
                             c_vp(smp.ctypes.data), len(smp), c_vp(models.ctypes.data), c_vp(valid.ctypes.data))
    return models, valid


def ransac_noncentral_relative_pose(prob_ptr, f1, f2, sigma1, sigma2, cam1, cam2, cam_ptr1, cam_off1, cam_rot1, cam_ptr2, cam_off2, cam_rot2,
                                    samples, threshold, max_iterations, probability=0.99, per_sample=False):
    """same arguments and result dict as covins_b200.placerec.ransac_noncentral_relative_pose"""
    ptr = np.ascontiguousarray(prob_ptr, np.int32); n_prob = len(ptr) - 1
    a = np.ascontiguousarray(f1, np.float64).reshape(-1, 3); b = np.ascontiguousarray(f2, np.float64).reshape(-1, 3)
    s1 = np.ascontiguousarray(sigma1, np.float64).reshape(-1); s2 = np.ascontiguousarray(sigma2, np.float64).reshape(-1)
    c1 = np.ascontiguousarray(cam1, np.int32).reshape(-1); c2 = np.ascontiguousarray(cam2, np.int32).reshape(-1)
    cp1 = np.ascontiguousarray(cam_ptr1, np.int32); cp2 = np.ascontiguousarray(cam_ptr2, np.int32)
    co1, cr1 = _rig(cam_off1, cam_rot1); co2, cr2 = _rig(cam_off2, cam_rot2)
    smp = np.ascontiguousarray(samples, np.int32).reshape(n_prob, -1, 17); ns = smp.shape[1]
    r = dict(best_sample=np.zeros(n_prob, np.int32), best_model=np.zeros((n_prob, 3, 4)), best_count=np.zeros(n_prob, np.int32),
             iterations=np.zeros(n_prob, np.int32), consumed=np.zeros(n_prob, np.int32), inlier_mask=np.zeros(len(a), np.uint8))
    if per_sample:
        r.update(sample_model=np.zeros((n_prob, ns, 3, 4)), sample_valid=np.zeros((n_prob, ns), np.uint8),
                 sample_count=np.zeros((n_prob, ns), np.int32))
    g = lambda k: c_vp(r[k].ctypes.data) if k in r else None
    lib().ora_ransac_noncentral_relative_pose(n_prob, *[c_vp(x.ctypes.data) for x in (ptr, a, b, s1, s2, c1, c2, cp1, co1, cr1, cp2, co2, cr2, smp)],
                                              ns, C.c_double(threshold), int(max_iterations), C.c_double(probability), g("best_sample"),
                                              g("best_model"), g("best_count"), g("iterations"), g("consumed"), g("inlier_mask"), g("sample_model"),
                                              g("sample_valid"), g("sample_count"))
    return r
