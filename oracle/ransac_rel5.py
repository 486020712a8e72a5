"""ctypes binding of oracle/ransac_rel5_oracle.c (5-point hypotheses + central relative-pose RANSAC selection) — TEST
INFRASTRUCTURE ONLY."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libcovins_ransac_rel5_oracle.so")
_LIB = None
c_vp = C.c_void_p


def build(out=LIB_PATH):
    """-ffp-contract=off: the CUDA path is compared bit for bit against plain IEEE evaluation"""
    subprocess.check_call(["gcc", "-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-Wall", "-Wextra", "-std=c11", "-fvisibility=hidden",
                           "-ffp-contract=off", "-shared", "-o", out, os.path.join(_HERE, "ransac_rel5_oracle.c"), "-lm"])


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            build()
        _LIB = C.CDLL(LIB_PATH)
    return _LIB


def rel5(f1, f2, sample):
    """one central problem's bearings, one sample of 5 local indices → dict(model [3,4] (zeros if invalid), valid, and for the
    real roots of the degree-10 polynomial, ascending: z [R], E [R,3,3] (scaled to tr(E E^T) / 2 = 1), cand [R,4,3,4] (the four
    decompositions in order), quality [R,4])"""
    a = np.ascontiguousarray(f1, np.float64).reshape(-1, 3); b = np.ascontiguousarray(f2, np.float64).reshape(-1, 3)
    s = np.ascontiguousarray(sample, np.int32).reshape(5)
    model = np.zeros((3, 4)); nr = C.c_int32(0)
    z = np.zeros(10); E = np.zeros((10, 3, 3)); cand = np.zeros((10, 4, 3, 4)); q = np.zeros((10, 4))
    v = lib().ora_rel5(len(a), c_vp(a.ctypes.data), c_vp(b.ctypes.data), c_vp(s.ctypes.data), c_vp(model.ctypes.data), C.byref(nr),
                       *[c_vp(x.ctypes.data) for x in (z, E, cand, q)])
    k = nr.value
    return dict(model=model, valid=bool(v), z=z[:k], E=E[:k], cand=cand[:k], quality=q[:k])


def ransac_central_relative_pose(prob_ptr, f1, f2, sigma1, sigma2, samples, threshold, max_iterations, probability=0.99, per_sample=False):
    """same arguments and result dict as covins_b200.placerec.ransac_central_relative_pose"""
    ptr = np.ascontiguousarray(prob_ptr, np.int32); n_prob = len(ptr) - 1
    a = np.ascontiguousarray(f1, np.float64).reshape(-1, 3); b = np.ascontiguousarray(f2, np.float64).reshape(-1, 3)
    s1 = np.ascontiguousarray(sigma1, np.float64).reshape(-1); s2 = np.ascontiguousarray(sigma2, np.float64).reshape(-1)
    smp = np.ascontiguousarray(samples, np.int32).reshape(n_prob, -1, 5); ns = smp.shape[1]
    r = dict(best_sample=np.zeros(n_prob, np.int32), best_model=np.zeros((n_prob, 3, 4)), best_count=np.zeros(n_prob, np.int32),
             iterations=np.zeros(n_prob, np.int32), consumed=np.zeros(n_prob, np.int32), inlier_mask=np.zeros(len(a), np.uint8))
    if per_sample:
        r.update(sample_model=np.zeros((n_prob, ns, 3, 4)), sample_valid=np.zeros((n_prob, ns), np.uint8),
                 sample_count=np.zeros((n_prob, ns), np.int32))
    g = lambda k: c_vp(r[k].ctypes.data) if k in r else None
    lib().ora_ransac_central_relative_pose(n_prob, *[c_vp(x.ctypes.data) for x in (ptr, a, b, s1, s2, smp)], ns, C.c_double(threshold),
                                           int(max_iterations), C.c_double(probability), g("best_sample"), g("best_model"), g("best_count"),
                                           g("iterations"), g("consumed"), g("inlier_mask"), g("sample_model"), g("sample_valid"),
                                           g("sample_count"))
    return r
