"""Host-side mirror of the reference's map maintenance on top of the C-ABI.

`covisibility` is Keyframe::UpdateCovisibilityConnections (keyframe_be.cpp:559-608) for every keyframe of a map in one
call: the canonical, order-independent graph include/covins_b200.h defines for cvb_covisibility, on the landmark /
observation CSR of the flat bundle-adjustment problem (`lm_obs_ptr`, `obs_kf`, `obs_skip`).
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._lib import Context, lib


def _opt(a, n, what):
    if a is None:
        return None
    a = np.ascontiguousarray(a, np.uint8)
    assert a.shape == (n,), f"{what} has shape {a.shape}, expected ({n},)"
    return a


def covisibility(ctx: Context, lm_obs_ptr, obs_kf, K: int, obs_skip=None, lm_valid=None, min_weight: int = 15):
    """→ (nbr_ptr [K+1] i32, nbr_kf [n] i32, nbr_w [n] i32): keyframe i's connected keyframes and their shared-landmark
    counts at [nbr_ptr[i], nbr_ptr[i+1]), weight descending then index ascending (GetConnectedKeyframes order).
    obs_skip [n_obs] (1 = the observation does not take part), lm_valid [L] (0 = the landmark does not take part);
    min_weight 15 is the reference's hard-coded threshold."""
    ptr = np.ascontiguousarray(lm_obs_ptr, np.int32)
    kf = np.ascontiguousarray(obs_kf, np.int32)
    assert ptr.ndim == 1 and len(ptr) >= 1 and kf.ndim == 1, "lm_obs_ptr is [L+1], obs_kf is [n_obs]"
    L = len(ptr) - 1
    assert len(kf) >= int(ptr[-1]), "obs_kf is shorter than lm_obs_ptr[L]"
    skip = _opt(obs_skip, len(kf), "obs_skip")
    valid = _opt(lm_valid, L, "lm_valid")
    p = lambda a: None if a is None else a.ctypes.data
    nbr_ptr = np.zeros(K + 1, np.int32)
    n_total = C.c_int64(0)
    cap = min(K * max(K - 1, 0), 64 * K)          # a first guess; the call reports the size when it does not fit
    while True:
        nbr_kf = np.empty(cap, np.int32); nbr_w = np.empty(cap, np.int32)
        ctx.check(lib().cvb_covisibility(ctx.handle, int(K), L, p(ptr), p(kf), p(skip), p(valid), int(min_weight), p(nbr_ptr),
                                         p(nbr_kf), p(nbr_w), cap, C.byref(n_total)))
        if n_total.value <= cap:
            return nbr_ptr, nbr_kf[:n_total.value].copy(), nbr_w[:n_total.value].copy()
        cap = n_total.value
