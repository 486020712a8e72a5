"""oracle/lm_outliers.py — CPU restatement of cvb_landmark_outliers, the landmark outlier removal of Map::Clean
(map_be.cpp:448-454, 698-743).

TEST INFRASTRUCTURE ONLY (imported from tests/ and tools/; nothing under covins_b200/ imports it).

ASSUMPTION (parity unpinned beyond the source): the reference does not record its rule; include/covins_b200.h defines a
canonical one from behaviour this tree already pins, restated here:
  1. an observation takes part iff obs_skip is None or 0 for it, and its landmark iff lm_valid is None or non-zero for it
     (rule 1 of cvb_covisibility);
  2. norm of a participating observation = the loss-corrected residual norm of the autograd oracle (ba_oracle.reproj_residual
     scaled as ba_oracle.corrected_reproj_norms scales it: sqrt(s) * sqrt(1 / (1 + s / cauchy^2)), s = |r|^2; cauchy <= 0:
     |r|), for EVERY participating observation, landmarks with fewer than two observers included;
  3. obs_outlier = 2 if the point is not projectable (pinhole: z <= 1e-10; unified: z + xi |p| <= 1e-10 or p = 0), else 1
     if norm > th_outlier, else 0; 0 for observations that do not take part (the non-projectable clause follows the
     ORB-SLAM isDepthPositive lineage and is pure assumption);
  4. lm_erase = 1 iff the landmark takes part and fewer than min_obs of its participating observations have obs_outlier 0;
  5. norms: the norm of each participating observation, -1 for the others.
K == 0, L == 0 or n_obs == 0: nothing is flagged.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle import ba_oracle as bo


def participating(p: dict, lm_valid=None):
    """→ (take part [n_obs] bool, landmark of each observation [n_obs], landmark takes part [L] bool)"""
    L = int(p.get("L", 0))
    ptr = np.asarray(p.get("lm_obs_ptr", np.zeros(1)), np.int64)
    obs_lm = np.repeat(np.arange(L), np.diff(ptr))
    lm_in = np.ones(L, bool) if lm_valid is None else np.asarray(lm_valid).astype(bool)
    part = lm_in[obs_lm]
    if p.get("obs_skip") is not None:
        part &= ~np.asarray(p["obs_skip"]).astype(bool)
    return part, obs_lm, lm_in


def _cameras(p: dict, kf):
    K = int(p["K"])
    cam = np.asarray(p["cam_of_kf"] if p.get("cam_of_kf") is not None else np.zeros(K, np.int64), np.int64)[kf]
    ncam = len(np.asarray(p["extr"]).reshape(-1, 7))
    pick = lambda name, default: np.asarray(p[name] if p.get(name) is not None else default)[cam]
    return (np.asarray(p["extr"], float).reshape(-1, 7)[cam], np.asarray(p["intr"], float)[cam], np.asarray(p["dist"], float)[cam],
            pick("cam_model", np.zeros(ncam, np.int64)).astype(np.int64), pick("dist_model", np.zeros(ncam, np.int64)).astype(np.int64),
            pick("cam_xi", np.zeros(ncam)).astype(float))


def projectable(p: dict, sel):
    """the plain restatement of aslam's projection test for observations `sel`: the camera-frame point of the landmark"""
    kf = np.asarray(p["obs_kf"], np.int64)[sel]
    L = int(p["L"])
    lm = np.asarray(p["lm"], float).reshape(-1, 3)[np.repeat(np.arange(L), np.diff(np.asarray(p["lm_obs_ptr"], np.int64)))[sel]]
    extr, _, _, cm, _, xi = _cameras(p, kf)
    pose = np.asarray(p["pose"], float)[kf]
    Rws = bo._quat_to_rot_np(pose[:, :4]); Rsc = bo._quat_to_rot_np(extr[:, :4])
    ps = np.einsum("nji,nj->ni", Rws, lm - pose[:, 4:])
    pc = np.einsum("nji,nj->ni", Rsc, ps - extr[:, 4:])
    d = np.linalg.norm(pc, axis=1)
    den = np.where(cm == 1, pc[:, 2] + xi * d, pc[:, 2])
    return (den > 1e-10) & ((cm == 0) | (d > 0))


def norms(p: dict, sel, cauchy: float = 1.0):
    """loss-corrected residual norms of observations `sel` from the autograd oracle's residual"""
    kf = np.asarray(p["obs_kf"], np.int64)[sel]
    L = int(p["L"])
    lm = np.asarray(p["lm"], float).reshape(-1, 3)[np.repeat(np.arange(L), np.diff(np.asarray(p["lm_obs_ptr"], np.int64)))[sel]]
    extr, intr, dist, cm, dm, xi = _cameras(p, kf)
    t = lambda a: torch.tensor(a)
    r = bo.reproj_residual(t(np.asarray(p["pose"], float)[kf]), t(lm), t(extr), t(intr), t(dist),
                           t(np.asarray(p["obs_uv"], np.float32)[sel].astype(float)), t(np.asarray(p["obs_sigma"], float)[sel]),
                           t(cm), t(dm), t(xi)).numpy()
    s = (r * r).sum(1)
    scale = np.sqrt(1.0 / (1.0 + s / (cauchy * cauchy))) if cauchy > 0 else np.ones_like(s)
    return np.sqrt(s) * scale


def decide(part, obs_lm, lm_in, norm, proj, th_outlier: float = 0.92, min_obs: int = 2):
    """rules 3-4 on given norms and projectability (arrays over all observations; entries outside `part` are not read)
    → (obs_outlier [n_obs] u8, lm_erase [L] u8)"""
    part, proj, norm = np.asarray(part, bool), np.asarray(proj, bool), np.asarray(norm, float)
    out = np.zeros(len(obs_lm), np.uint8)
    out[part & ~proj] = 2
    out[part & proj & (norm > th_outlier)] = 1
    good = np.bincount(obs_lm[part & (out == 0)], minlength=len(lm_in))
    return out, (np.asarray(lm_in, bool) & (good < min_obs)).astype(np.uint8)


def landmark_outliers(p: dict, lm_valid=None, th_outlier: float = 0.92, cauchy: float = 1.0, min_obs: int = 2):
    """→ (obs_outlier [n_obs] u8, lm_erase [L] u8, norms [n_obs]: -1 where the observation does not take part)"""
    n = len(p.get("obs_kf", [])); L = int(p.get("L", 0))
    nrm = np.full(n, -1.0)
    if int(p["K"]) == 0 or L == 0 or n == 0:
        return np.zeros(n, np.uint8), np.zeros(L, np.uint8), nrm
    part, obs_lm, lm_in = participating(p, lm_valid)
    sel = np.flatnonzero(part)
    proj = np.zeros(n, bool)
    if len(sel):
        nrm[sel] = norms(p, sel, cauchy)
        proj[sel] = projectable(p, sel)
    out, erase = decide(part, obs_lm, lm_in, nrm, proj, th_outlier, min_obs)
    return out, erase, nrm
