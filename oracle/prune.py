"""ctypes binding of oracle/prune_oracle.c (the sequential keyframe-culling pass of cvb_redundant_keyframes) — TEST
INFRASTRUCTURE ONLY.  The rule and its assumptions head the C file."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libcovins_prune_oracle.so")
_LIB = None


def build(out=LIB_PATH):
    """one thread, as the reference runs the pass under the map lock; -ffp-contract=off: the th_red product and the time
    difference are compared bit for bit against the CUDA path's rounded operations"""
    subprocess.check_call(["gcc", "-O3", "-march=x86-64-v3", "-fPIC", "-Wall", "-Wextra", "-std=c11", "-fvisibility=hidden",
                           "-ffp-contract=off", "-shared", "-o", out, os.path.join(_HERE, "prune_oracle.c")])


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            build()
        _LIB = C.CDLL(LIB_PATH)
        _LIB.ora_redundant_keyframes.restype = C.c_int
        _LIB.ora_redundant_keyframes.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 8 + [C.c_double, C.c_double, C.c_int, C.c_void_p]
    return _LIB


def redundant_keyframes(lm_obs_ptr, obs_kf, obs_octave, kf_pred, kf_time, kf_protect, th_red, max_time_dist, th_obs=3,
                        obs_skip=None, lm_valid=None):
    """→ culled [K] uint8, the same arguments as covins_b200.mapgraph.redundant_keyframes (num_octaves only bounds the input)"""
    ptr = np.ascontiguousarray(lm_obs_ptr, np.int32); kf = np.ascontiguousarray(obs_kf, np.int32)
    octv = np.ascontiguousarray(obs_octave, np.int32); pred = np.ascontiguousarray(kf_pred, np.int32)
    time = np.ascontiguousarray(kf_time, np.float64); prot = np.ascontiguousarray(kf_protect, np.uint8)
    skip = None if obs_skip is None else np.ascontiguousarray(obs_skip, np.uint8)
    valid = None if lm_valid is None else np.ascontiguousarray(lm_valid, np.uint8)
    K = len(pred)
    culled = np.zeros(K, np.uint8)
    p = lambda a: None if a is None else a.ctypes.data
    rc = lib().ora_redundant_keyframes(K, len(ptr) - 1, p(ptr), p(kf), p(octv), p(skip), p(valid), p(pred), p(time), p(prot), float(th_red),
                                       float(max_time_dist), int(th_obs), p(culled))
    assert rc == 0, "ora_redundant_keyframes: input outside the pass's definition"
    return culled
