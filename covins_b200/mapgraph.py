"""Host-side mirror of the reference's map maintenance on top of the C-ABI.

`covisibility` is Keyframe::UpdateCovisibilityConnections (keyframe_be.cpp:559-608) for every keyframe of a map in one
call: the canonical, order-independent graph include/covins_b200.h defines for cvb_covisibility, on the landmark /
observation CSR of the flat bundle-adjustment problem (`lm_obs_ptr`, `obs_kf`, `obs_skip`).
`redundant_keyframes` is the redundancy pruning of Map::Clean (map_be.cpp:745-811): the reference's sequential culling
pass on the same CSR, reproduced exactly by parallel rounds (cvb_redundant_keyframes).
`landmark_outliers` is the landmark outlier removal of Map::Clean (map_be.cpp:448-454, 698-743): the outlier observations and
the landmarks left with too few good observers, on the flat bundle-adjustment problem (cvb_landmark_outliers).
`rigid_transform` is the transform loop of the merge constructor Map(map_target, map_tofuse, T) (map_be.cpp:365-380): the
fused map's keyframe poses, velocities and landmark positions moved into the target's world frame (cvb_map_rigid_transform).
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


def redundant_keyframes(ctx: Context, lm_obs_ptr, obs_kf, obs_octave, kf_pred, kf_time, kf_protect, th_red: float,
                        max_time_dist: float, th_obs: int = 3, num_octaves: int = 8, obs_skip=None, lm_valid=None):
    """→ (culled [K] u8, rounds): the keyframes the sequential redundancy-culling pass of Map::Clean (map_be.cpp:745-811)
    removes, as include/covins_b200.h defines it for cvb_redundant_keyframes, and the number of parallel rounds the call
    took.  obs_octave [n_obs] (obs_sigma / 2 - 1 of the GBA problem), kf_pred [K] (the chain predecessor, -1 for none),
    kf_time [K], kf_protect [K] (1 = never culled); obs_skip / lm_valid as for covisibility."""
    ptr = np.ascontiguousarray(lm_obs_ptr, np.int32)
    kf = np.ascontiguousarray(obs_kf, np.int32)
    octv = np.ascontiguousarray(obs_octave, np.int32)
    assert ptr.ndim == 1 and len(ptr) >= 1 and kf.ndim == 1, "lm_obs_ptr is [L+1], obs_kf is [n_obs]"
    L = len(ptr) - 1
    assert len(kf) >= int(ptr[-1]) and octv.shape == kf.shape, "obs_kf / obs_octave are shorter than lm_obs_ptr[L]"
    pred = np.ascontiguousarray(kf_pred, np.int32)
    K = len(pred)
    time = np.ascontiguousarray(kf_time, np.float64)
    prot = np.ascontiguousarray(kf_protect, np.uint8)
    assert time.shape == (K,) and prot.shape == (K,), "kf_time and kf_protect are [K]"
    skip = _opt(obs_skip, len(kf), "obs_skip")
    valid = _opt(lm_valid, L, "lm_valid")
    p = lambda a: None if a is None else a.ctypes.data
    culled = np.zeros(K, np.uint8)
    rounds = C.c_int32(0)
    ctx.check(lib().cvb_redundant_keyframes(ctx.handle, K, L, p(ptr), p(kf), p(octv), p(skip), p(valid), p(pred), p(time), p(prot),
                                            float(th_red), float(max_time_dist), int(th_obs), int(num_octaves), p(culled),
                                            C.byref(rounds)))
    return culled, rounds.value


def landmark_outliers(ctx: Context, p: dict, lm_valid=None, th_outlier: float = 0.92, cauchy: float = 1.0, min_obs: int = 2,
                      want_norms: bool = False):
    """→ (obs_outlier [n_obs] u8, lm_erase [L] u8, norms [n_obs] f64 or None): the rule include/covins_b200.h defines for
    cvb_landmark_outliers on the flat problem `p` (the dict optimization.py takes; p["obs_skip"], when present, marks the
    observations that do not take part).  obs_outlier is 1 for norm > th_outlier, 2 for a point the camera cannot project;
    lm_erase marks the participating landmarks left with fewer than min_obs good observations; norms (want_norms) is the
    loss-corrected residual norm cvb_ba_reproj_norms reports, -1 for observations that do not take part."""
    from .optimization import _Flat
    flat = _Flat(p, obs_skip=p.get("obs_skip"), use_imu=False)
    valid = _opt(lm_valid, flat.L, "lm_valid")
    obs_outlier = np.zeros(flat.n_obs, np.uint8)
    lm_erase = np.zeros(flat.L, np.uint8)
    norms = np.zeros(flat.n_obs) if want_norms else None
    n_out, n_erased = C.c_int64(0), C.c_int32(0)
    p_ = lambda a: None if a is None else a.ctypes.data
    ctx.check(lib().cvb_landmark_outliers(ctx.handle, C.byref(flat.s), p_(valid), float(th_outlier), float(cauchy), int(min_obs),
                                          p_(obs_outlier), p_(lm_erase), p_(norms), C.byref(n_out), C.byref(n_erased)))
    assert n_out.value == int(np.count_nonzero(obs_outlier)) and n_erased.value == int(lm_erase.sum())
    return obs_outlier, lm_erase, norms


def is_rigid(T) -> bool:
    """cvb_map_rigid_transform's test of T: finite entries, last row exactly [0 0 0 1], every entry of R^T R within 1e-9 of
    I and det R > 0"""
    T = np.asarray(T, np.float64)
    if T.shape != (4, 4) or not np.isfinite(T).all() or T[3].tolist() != [0.0, 0.0, 0.0, 1.0]:
        return False
    R = T[:3, :3].tolist()
    for a in range(3):
        for b in range(3):
            if not abs((R[0][a] * R[0][b] + R[1][a] * R[1][b]) + R[2][a] * R[2][b] - (1.0 if a == b else 0.0)) <= 1e-9:
                return False
    return (R[0][0] * (R[1][1] * R[2][2] - R[1][2] * R[2][1]) - R[0][1] * (R[1][0] * R[2][2] - R[1][2] * R[2][0])) \
        + R[0][2] * (R[1][0] * R[2][1] - R[1][1] * R[2][0]) > 0.0


def rigid_transform(ctx: Context, T, T_ws, vel=None, lm_pos=None, kf_sel=None, lm_sel=None):
    """→ (T_ws' [K,4,4], vel' [K,3] or None, lm_pos' [L,3]): the fused map's keyframe poses T_ws [K,4,4] (or [K,16],
    row-major), velocities vel [K,3] (optional) and landmark positions lm_pos [L,3] moved by T = T_wtarget_wtofuse
    [4,4]: T_ws <- T T_ws, v <- R v, p <- R p + t, for the entries kf_sel [K] / lm_sel [L] select (all when None), the
    others returned unchanged.  The inputs are not modified.  A T that is not rigid raises ValueError before any device
    work."""
    T = np.ascontiguousarray(T, np.float64)
    if not is_rigid(T):
        raise ValueError("T is not rigid (finite entries, R^T R = I within 1e-9, det R > 0, last row [0 0 0 1])")
    ws = np.array(T_ws, np.float64, order="C").reshape(-1, 16)
    K = len(ws)
    v = None if vel is None else np.array(vel, np.float64, order="C").reshape(K, 3)
    p = np.array(lm_pos if lm_pos is not None else np.zeros((0, 3)), np.float64, order="C").reshape(-1, 3)
    ks, ls = _opt(kf_sel, K, "kf_sel"), _opt(lm_sel, len(p), "lm_sel")
    p_ = lambda a: None if a is None else a.ctypes.data
    ctx.check(lib().cvb_map_rigid_transform(ctx.handle, T.ctypes.data, K, p_(ws), p_(v), len(p), p_(p), p_(ks), p_(ls)))
    return ws.reshape(K, 4, 4), v, p
