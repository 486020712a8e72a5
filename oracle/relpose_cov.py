"""ctypes binding of oracle/relpose_cov_oracle.c (the sampling-based 6x6 covariance of the non-central relative pose from
17-point re-solves) — TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libcovins_relpose_cov_oracle.so")
_LIB = None
c_vp = C.c_void_p


def build(out=LIB_PATH):
    """-ffp-contract=off: the CUDA path is compared bit for bit against plain IEEE evaluation"""
    subprocess.check_call(["gcc", "-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-Wall", "-Wextra", "-std=c11", "-fvisibility=hidden",
                           "-ffp-contract=off", "-shared", "-o", out, os.path.join(_HERE, "relpose_cov_oracle.c"), "-lm"])


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            build()
        _LIB = C.CDLL(LIB_PATH)
    return _LIB


def deviation(ref_model, model):
    """delta [6] = [2 vec(q); t - t_ref] of a 3x4 model against a 3x4 reference, q the quaternion of R_ref^T R (w >= 0)"""
    a = np.ascontiguousarray(ref_model, np.float64).reshape(12); b = np.ascontiguousarray(model, np.float64).reshape(12)
    d = np.zeros(6)
    lib().ora_rel_deviation(c_vp(a.ctypes.data), c_vp(b.ctypes.data), c_vp(d.ctypes.data))
    return d


def noncentral_relative_pose_covariance(prob_ptr, f1, f2, cam1, cam2, cam_ptr1, cam_off1, cam_rot1, cam_ptr2, cam_off2, cam_rot2, samples,
                                        ref_model, per_sample=False, threads=0, sigma1=None, sigma2=None):
    """same arguments and result dict as covins_b200.placerec.relative_pose_covariance (sigma1 / sigma2 are not read);
    threads: OpenMP threads for the per-sample solves (0: all)"""
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
    g = lambda k: c_vp(r[k].ctypes.data) if k in r else None
    lib().ora_noncentral_relative_pose_covariance(n_prob, *[c_vp(x.ctypes.data) for x in (ptr, a, b, c1, c2, cp1, co1, cr1, cp2, co2, cr2, smp)], ns,
                                                  c_vp(ref.ctypes.data), int(threads), g("cov"), g("n_valid"), g("sample_delta"),
                                                  g("sample_valid"))
    return r
