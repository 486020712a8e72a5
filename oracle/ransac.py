"""ctypes binding of oracle/ransac_oracle.c (P3P hypotheses + absolute-pose RANSAC selection) — TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libcovins_ransac_oracle.so")
_LIB = None
c_vp = C.c_void_p


def build(out=LIB_PATH):
    """-ffp-contract=off: the CUDA path is compared bit for bit against plain IEEE evaluation"""
    subprocess.check_call(["gcc", "-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-Wall", "-Wextra", "-std=c11", "-fvisibility=hidden",
                           "-ffp-contract=off", "-shared", "-o", out, os.path.join(_HERE, "ransac_oracle.c"), "-lm"])


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            build()
        _LIB = C.CDLL(LIB_PATH)
        _LIB.ora_p3p.restype = C.c_int
        _LIB.ora_p3p.argtypes = [c_vp, c_vp, c_vp]
    return _LIB


def p3p(f, x):
    """bearings f [3,3] (camera frame), world points x [3,3] → list of (R [3,3], t [3]) with lambda_i f_i = R x_i + t"""
    f = np.ascontiguousarray(f, np.float64).reshape(9); x = np.ascontiguousarray(x, np.float64).reshape(9)
    out = np.zeros((4, 12))
    k = lib().ora_p3p(f.ctypes.data, x.ctypes.data, out.ctypes.data)
    return [(out[i].reshape(3, 4)[:, :3].copy(), out[i].reshape(3, 4)[:, 3].copy()) for i in range(k)]


def abs_hypotheses(pts, f, cam_off, cam_rot, samples):
    """hypotheses of one problem's samples [S,4] → (models [S,3,4], valid [S])"""
    p = np.ascontiguousarray(pts, np.float64).reshape(-1, 3); fb = np.ascontiguousarray(f, np.float64).reshape(-1, 3)
    co = np.ascontiguousarray(cam_off, np.float64).reshape(3); cr = np.ascontiguousarray(cam_rot, np.float64).reshape(9)
    smp = np.ascontiguousarray(samples, np.int32).reshape(-1, 4)
    models = np.zeros((len(smp), 3, 4)); valid = np.zeros(len(smp), np.uint8)
    lib().ora_abs_hypotheses(len(p), c_vp(p.ctypes.data), c_vp(fb.ctypes.data), c_vp(co.ctypes.data), c_vp(cr.ctypes.data), c_vp(smp.ctypes.data),
                             len(smp), c_vp(models.ctypes.data), c_vp(valid.ctypes.data))
    return models, valid


def ransac_absolute_pose(prob_ptr, pts, bearings, sigma, cam_off, cam_rot, samples, threshold, max_iterations, probability=0.99, per_sample=False):
    """same arguments and result dict as covins_b200.placerec.ransac_absolute_pose"""
    ptr = np.ascontiguousarray(prob_ptr, np.int32); n_prob = len(ptr) - 1
    p = np.ascontiguousarray(pts, np.float64).reshape(-1, 3); fb = np.ascontiguousarray(bearings, np.float64).reshape(-1, 3)
    s = np.ascontiguousarray(sigma, np.float64).reshape(-1)
    co = np.ascontiguousarray(cam_off, np.float64).reshape(n_prob, 3); cr = np.ascontiguousarray(cam_rot, np.float64).reshape(n_prob, 9)
    smp = np.ascontiguousarray(samples, np.int32).reshape(n_prob, -1, 4); ns = smp.shape[1]
    r = dict(best_sample=np.zeros(n_prob, np.int32), best_model=np.zeros((n_prob, 3, 4)), best_count=np.zeros(n_prob, np.int32),
             iterations=np.zeros(n_prob, np.int32), consumed=np.zeros(n_prob, np.int32), inlier_mask=np.zeros(len(p), np.uint8))
    if per_sample:
        r.update(sample_model=np.zeros((n_prob, ns, 3, 4)), sample_valid=np.zeros((n_prob, ns), np.uint8),
                 sample_count=np.zeros((n_prob, ns), np.int32))
    g = lambda k: c_vp(r[k].ctypes.data) if k in r else None
    lib().ora_ransac_absolute_pose(n_prob, c_vp(ptr.ctypes.data), c_vp(p.ctypes.data), c_vp(fb.ctypes.data), c_vp(s.ctypes.data),
                                   c_vp(co.ctypes.data), c_vp(cr.ctypes.data), c_vp(smp.ctypes.data), ns, C.c_double(threshold),
                                   int(max_iterations), C.c_double(probability), g("best_sample"), g("best_model"), g("best_count"),
                                   g("iterations"), g("consumed"), g("inlier_mask"), g("sample_model"), g("sample_valid"), g("sample_count"))
    return r
