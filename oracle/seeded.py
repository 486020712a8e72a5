"""ctypes binding of oracle/sampler_oracle.c (Philox4x64-10 and the seeded k-subset rule) and the seeded forms of the four RANSAC /
covariance oracles — TEST INFRASTRUCTURE ONLY.

Each seeded driver is a thin layer over its sample-supplied oracle: it draws the samples with the C sampler and feeds them to
that oracle.  A RANSAC problem gets 11 * max_iterations samples (at least n_samples), enough for any selection: opengv's bound
reads at most max_iterations valid and 10 * max_iterations invalid ones.  The rules the sample-supplied form does not have are
applied here: a problem with fewer than k correspondences (covariance: inliers) draws nothing."""
import ctypes as C
import os
import subprocess

import numpy as np

from . import ransac as orr
from . import ransac_rel as orel
from . import ransac_rel5 as orel5
from . import relpose_cov as ocov

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libcovins_sampler_oracle.so")
_LIB = None
c_vp = C.c_void_p
WAVE = 64   # the GPU draws a RANSAC's samples in waves of 64: the rows of `drawn` it fills


def build(out=LIB_PATH):
    subprocess.check_call(["gcc", "-O3", "-march=x86-64-v3", "-fPIC", "-Wall", "-Wextra", "-std=c11", "-fvisibility=hidden", "-ffp-contract=off",
                           "-shared", "-o", out, os.path.join(_HERE, "sampler_oracle.c")])


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            build()
        _LIB = C.CDLL(LIB_PATH)
        _LIB.ora_seeded_samples.argtypes = [C.c_uint64, C.c_uint64, C.c_uint32, C.c_int, C.c_int64, C.c_int, c_vp]
    return _LIB


def philox(key, counter):
    """Philox4x64-10 block of counter [4] under key [2] → [4] uint64"""
    k = np.ascontiguousarray(key, np.uint64).reshape(2); c = np.ascontiguousarray(counter, np.uint64).reshape(4)
    out = np.zeros(4, np.uint64)
    lib().ora_philox4x64_10(c_vp(c.ctypes.data), c_vp(k.ctypes.data), c_vp(out.ctypes.data))
    return out


def samples(seed, stream, m, k, n, s0=0):
    """samples s0 .. s0 + n - 1 of key (seed, stream): [n, k] ordered k-subsets of [0, m)"""
    assert 0 < k <= min(m, 64)
    out = np.zeros((n, k), np.int32)
    lib().ora_seeded_samples(int(seed), int(stream), int(m), int(k), int(s0), int(n), c_vp(out.ctypes.data))
    return out


def _ransac_seeded(oracle, k, b, seeds, threshold, max_iterations, probability, per_sample, n_samples, want_drawn):
    ptr = np.asarray(b["prob_ptr"], np.int64); n_prob = len(ptr) - 1
    S = max(int(n_samples), 11 * int(max_iterations), 1)
    smp = np.zeros((n_prob, S, k), np.int32)
    for i in range(n_prob):
        n = ptr[i + 1] - ptr[i]
        if n >= k:
            smp[i] = samples(seeds[i], 0, n, k, S)
    r = oracle(**b, samples=smp, threshold=threshold, max_iterations=max_iterations, probability=probability, per_sample=per_sample)
    drawn = np.full((n_prob, n_samples, k), -1, np.int32)
    for i in range(n_prob):
        if ptr[i + 1] - ptr[i] < k:       # draws nothing: no selection at all (the supplied form would skip its samples)
            r["best_sample"][i] = -1; r["best_count"][i] = 0; r["iterations"][i] = 0; r["consumed"][i] = 0; r["best_model"][i] = 0.0
            continue
        rows = n_samples if per_sample else min(n_samples, -(-int(r["consumed"][i]) // WAVE) * WAVE)
        drawn[i, :rows] = smp[i, :rows]
    if per_sample:
        for key in ("sample_model", "sample_valid", "sample_count"):
            r[key] = np.ascontiguousarray(r[key][:, :n_samples])
    if want_drawn:
        r["drawn"] = drawn
    return r


def ransac_absolute_pose_seeded(prob_ptr, pts, bearings, sigma, cam_off, cam_rot, seeds, threshold, max_iterations, probability=0.99,
                                per_sample=False, n_samples=0, want_drawn=False):
    """same arguments and result dict as covins_b200.placerec.ransac_absolute_pose_seeded"""
    b = dict(prob_ptr=prob_ptr, pts=pts, bearings=bearings, sigma=sigma, cam_off=cam_off, cam_rot=cam_rot)
    return _ransac_seeded(orr.ransac_absolute_pose, 4, b, np.asarray(seeds, np.uint64), threshold, max_iterations, probability, per_sample,
                          n_samples, want_drawn)


def ransac_noncentral_relative_pose_seeded(prob_ptr, f1, f2, sigma1, sigma2, cam1, cam2, cam_ptr1, cam_off1, cam_rot1, cam_ptr2, cam_off2,
                                           cam_rot2, seeds, threshold, max_iterations, probability=0.99, per_sample=False, n_samples=0,
                                           want_drawn=False):
    """same arguments and result dict as covins_b200.placerec.ransac_noncentral_relative_pose_seeded"""
    b = dict(prob_ptr=prob_ptr, f1=f1, f2=f2, sigma1=sigma1, sigma2=sigma2, cam1=cam1, cam2=cam2, cam_ptr1=cam_ptr1, cam_off1=cam_off1,
             cam_rot1=cam_rot1, cam_ptr2=cam_ptr2, cam_off2=cam_off2, cam_rot2=cam_rot2)
    return _ransac_seeded(orel.ransac_noncentral_relative_pose, 17, b, np.asarray(seeds, np.uint64), threshold, max_iterations, probability,
                          per_sample, n_samples, want_drawn)


def ransac_central_relative_pose_seeded(prob_ptr, f1, f2, sigma1, sigma2, seeds, threshold, max_iterations, probability=0.99, per_sample=False,
                                        n_samples=0, want_drawn=False):
    """same arguments and result dict as covins_b200.placerec.ransac_central_relative_pose_seeded"""
    b = dict(prob_ptr=prob_ptr, f1=f1, f2=f2, sigma1=sigma1, sigma2=sigma2)
    return _ransac_seeded(orel5.ransac_central_relative_pose, 5, b, np.asarray(seeds, np.uint64), threshold, max_iterations, probability,
                          per_sample, n_samples, want_drawn)


def relative_pose_covariance_seeded(prob_ptr, f1, f2, cam1, cam2, cam_ptr1, cam_off1, cam_rot1, cam_ptr2, cam_off2, cam_rot2, inlier_mask, seeds,
                                    ref_model, n_samples=300, per_sample=False, want_drawn=False, sigma1=None, sigma2=None):
    """same arguments and result dict as covins_b200.placerec.relative_pose_covariance_seeded"""
    ptr = np.asarray(prob_ptr, np.int64); n_prob = len(ptr) - 1
    mask = np.asarray(inlier_mask, np.uint8).reshape(-1)
    ref = np.array(ref_model, np.float64).reshape(n_prob, 12)
    seeds = np.asarray(seeds, np.uint64)
    if n_samples == 0:
        r = dict(cov=np.zeros((n_prob, 6, 6)), n_valid=np.zeros(n_prob, np.int32))
        if per_sample:
            r.update(sample_delta=np.zeros((n_prob, 0, 6)), sample_valid=np.zeros((n_prob, 0), np.uint8))
        if want_drawn:
            r["drawn"] = np.zeros((n_prob, 0, 17), np.int32)
        return r
    smp = np.zeros((n_prob, n_samples, 17), np.int32)
    drawn = np.full((n_prob, n_samples, 17), -1, np.int32)
    for i in range(n_prob):
        inl = np.flatnonzero(mask[ptr[i]:ptr[i + 1]])
        if not ref[i].any() or len(inl) < 17:
            ref[i] = 0.0                  # draws nothing: skipped like a problem without a reference model
            continue
        smp[i] = inl[samples(seeds[i], 1, len(inl), 17, n_samples)]
        drawn[i] = smp[i]
    r = ocov.noncentral_relative_pose_covariance(prob_ptr, f1, f2, cam1, cam2, cam_ptr1, cam_off1, cam_rot1, cam_ptr2, cam_off2, cam_rot2, smp, ref,
                                                 per_sample=per_sample)
    if want_drawn:
        r["drawn"] = drawn
    return r
