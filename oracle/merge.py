"""The rigid transform of the merge constructor Map(map_target, map_tofuse, T) (map_be.cpp:334-381, the loop at :365-380),
restated in numpy float64 in the operation order include/covins_b200.h gives cvb_map_rigid_transform.

ASSUMPTIONS (the merge constructor is not in this tree; the rule is restated from SURVEY.md's citations):
  * the fused map's keyframe poses T_ws and velocities are transformed, T_ws <- T T_ws and v <- R v; IMU biases are not;
  * T_ws_vio_ is left unchanged: the pose graph reads it only as relative transforms between keyframes of one agent
    (opt.cpp:947-1021), which a common left factor does not change;
  * landmark positions are transformed, p <- R p + t;
  * loop constraints, ids and the union of the two maps are host container work (covins_b200::MergeMaps).

Every output entry is its products summed left to right, each product and each sum rounded once (numpy's elementwise
float64 multiply and add never fuse), so the device's __dmul_rn / __dadd_rn chain gives the same bits.
"""
from __future__ import annotations

import numpy as np


def is_rigid(T) -> bool:
    """the rigidity test of cvb_map_rigid_transform: finite entries, last row exactly [0 0 0 1], every entry of R^T R within
    1e-9 of I (each entry (R[0,a] R[0,b] + R[1,a] R[1,b]) + R[2,a] R[2,b]), det R > 0 by cofactors along the first row"""
    T = np.asarray(T, np.float64).reshape(4, 4)
    if not np.isfinite(T).all() or not (T[3, 0] == 0.0 and T[3, 1] == 0.0 and T[3, 2] == 0.0 and T[3, 3] == 1.0):
        return False
    R = [[float(T[r, c]) for c in range(3)] for r in range(3)]
    for a in range(3):
        for b in range(3):
            s = (R[0][a] * R[0][b] + R[1][a] * R[1][b]) + R[2][a] * R[2][b]
            if not abs(s - (1.0 if a == b else 0.0)) <= 1e-9:
                return False
    det = (R[0][0] * (R[1][1] * R[2][2] - R[1][2] * R[2][1]) - R[0][1] * (R[1][0] * R[2][2] - R[1][2] * R[2][0])) \
        + R[0][2] * (R[1][0] * R[2][1] - R[1][1] * R[2][0])
    return det > 0.0


def rigid_transform(T, T_ws, vel=None, lm_pos=None, kf_sel=None, lm_sel=None):
    """→ (T_ws' [K,4,4], vel' [K,3] or None, lm_pos' [L,3]); unselected entries are copies of the inputs"""
    T = np.asarray(T, np.float64).reshape(4, 4)
    X = np.asarray(T_ws, np.float64).reshape(-1, 4, 4)
    K = len(X)
    Y = X.copy()
    ks = np.ones(K, bool) if kf_sel is None else np.asarray(kf_sel).astype(bool)
    for r in range(4):
        for c in range(4):
            Y[ks, r, c] = ((T[r, 0] * X[ks, 0, c] + T[r, 1] * X[ks, 1, c]) + T[r, 2] * X[ks, 2, c]) + T[r, 3] * X[ks, 3, c]
    V = None
    if vel is not None:
        v = np.asarray(vel, np.float64).reshape(K, 3)
        V = v.copy()
        for r in range(3):
            V[ks, r] = (T[r, 0] * v[ks, 0] + T[r, 1] * v[ks, 1]) + T[r, 2] * v[ks, 2]
    p = np.asarray(lm_pos if lm_pos is not None else np.zeros((0, 3)), np.float64).reshape(-1, 3)
    P = p.copy()
    ls = np.ones(len(p), bool) if lm_sel is None else np.asarray(lm_sel).astype(bool)
    for r in range(3):
        P[ls, r] = ((T[r, 0] * p[ls, 0] + T[r, 1] * p[ls, 1]) + T[r, 2] * p[ls, 2]) + T[r, 3]
    return Y, V, P
