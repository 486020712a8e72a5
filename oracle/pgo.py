"""Optimization::PoseGraphOptimization (optimization_be.cpp:833-1086) around its solve, restated in float64 in the operation
order include/covins_b200.h gives cvb_pgo: the edge list built from the keyframe chain, the start poses, and the
write-back of poses, velocities and landmarks.

Every product, sum and difference is rounded on its own in the order written (Python floats and numpy's elementwise float64
operations never fuse), sqrt and division are correctly rounded, so the device's __dmul_rn / __dadd_rn / __dsub_rn chain in
include/covins_b200_pose.h gives the same bits.  Poses are row-major 4x4 arrays, pose7 = qx, qy, qz, qw, x, y, z.

The problem is the dict covins_b200.optimization.pgo_map_problem builds: T_ws, T_ws_init (or None), T_ws_vio [K,4,4];
kf_pred, kf_succ, kf_id, pose_const [K]; velocity [K,3] or None; loop_i, loop_j [n], loop_q [n,4], loop_t [n,3], loop_cov
[n,6,6] or None; lm_pos [L,3], lm_ref [L] (-1 none, -2 not among the keyframes), lm_has_obs [L].
"""
from __future__ import annotations

import math

import numpy as np

EDGE_LOOP, EDGE_S1, EDGE_S23, EDGE_S45 = 0, 1, 2, 3


class Refused(ValueError):
    """input cvb_pgo refuses with CVB_ERR_INVALID before any launch"""


def transform_to_pose7(T) -> np.ndarray:
    """Eigen::Quaterniond(R) (w >= 0 branch, keyframe_base.cpp:490-499) and the translation"""
    T = [float(x) for x in np.asarray(T, np.float64).reshape(16)]
    m00, m11, m22 = T[0], T[5], T[10]
    q = [0.0] * 4
    tr = (m00 + m11) + m22
    if tr > 0:
        t = math.sqrt(tr + 1.0)
        q[3] = 0.5 * t
        t = 0.5 / t
        q[0] = (T[9] - T[6]) * t
        q[1] = (T[2] - T[8]) * t
        q[2] = (T[4] - T[1]) * t
    else:
        i = 0
        if m11 > m00:
            i = 1
        if m22 > T[5 * i]:
            i = 2
        j = (i + 1) % 3
        k = (j + 1) % 3
        t = math.sqrt(((T[5 * i] - T[5 * j]) - T[5 * k]) + 1.0)
        q[i] = 0.5 * t
        t = 0.5 / t
        q[3] = (T[4 * k + j] - T[4 * j + k]) * t
        q[j] = (T[4 * j + i] + T[4 * i + j]) * t
        q[k] = (T[4 * k + i] + T[4 * i + k]) * t
    return np.array(q + [T[3], T[7], T[11]])


def pose7_to_transform(p) -> np.ndarray:
    """Utils::Ceres2Transform (utils_base.cpp:28-43), vectorised over a leading axis"""
    p = np.asarray(p, np.float64).reshape(-1, 7)
    x, y, z, w = p[:, 0], p[:, 1], p[:, 2], p[:, 3]
    n = 1.0 / np.sqrt(((x * x + y * y) + z * z) + w * w)
    x, y, z, w = x * n, y * n, z * n, w * n
    T = np.zeros((len(p), 4, 4))
    T[:, 0, 0] = 1.0 - 2.0 * (y * y + z * z); T[:, 0, 1] = 2.0 * (x * y - z * w); T[:, 0, 2] = 2.0 * (x * z + y * w)
    T[:, 1, 0] = 2.0 * (x * y + z * w); T[:, 1, 1] = 1.0 - 2.0 * (x * x + z * z); T[:, 1, 2] = 2.0 * (y * z - x * w)
    T[:, 2, 0] = 2.0 * (x * z - y * w); T[:, 2, 1] = 2.0 * (y * z + x * w); T[:, 2, 2] = 1.0 - 2.0 * (x * x + y * y)
    T[:, :3, 3] = p[:, 4:]
    T[:, 3, 3] = 1.0
    return T


def rel_transform(Ta, Tb) -> np.ndarray:
    """Ta^-1 Tb of rigid transforms: Ra^T Rb and Ra^T (tb - ta), every entry summed from 0 over m = 0, 1, 2"""
    Ta = np.asarray(Ta, np.float64).reshape(-1, 4, 4); Tb = np.asarray(Tb, np.float64).reshape(-1, 4, 4)
    R = np.zeros_like(Ta)
    for r in range(3):
        for c in range(3):
            s = np.zeros(len(Ta))
            for m in range(3):
                s = s + Ta[:, m, r] * Tb[:, m, c]
            R[:, r, c] = s
        s = np.zeros(len(Ta))
        for m in range(3):
            s = s + Ta[:, m, r] * (Tb[:, m, 3] - Ta[:, m, 3])
        R[:, r, 3] = s
    R[:, 3, 3] = 1.0
    return R


def sqrt_info_from_cov(cov):
    """LLT(cov^-1).matrixL().transpose() (optimization_be.cpp:922-923) through two Cholesky factorisations and the inverse
    of the first factor; None when a pivot is not > 0"""
    cov = [float(x) for x in np.asarray(cov, np.float64).reshape(36)]
    L = [0.0] * 36; X = [0.0] * 36; P = [0.0] * 36; M = [0.0] * 36
    for c in range(6):
        for r in range(c, 6):
            s = cov[6 * r + c]
            for m in range(c):
                s = s - L[6 * r + m] * L[6 * c + m]
            if r == c:
                if not s > 0:
                    return None
                L[6 * c + c] = math.sqrt(s)
            else:
                L[6 * r + c] = s / L[6 * c + c]
    for c in range(6):
        for r in range(c, 6):
            s = 1.0 if r == c else 0.0
            for m in range(c, r):
                s = s - L[6 * r + m] * X[6 * m + c]
            X[6 * r + c] = s / L[6 * r + r]
    for r in range(6):
        for c in range(6):
            s = 0.0
            for m in range(max(r, c), 6):
                s = s + X[6 * m + r] * X[6 * m + c]
            P[6 * r + c] = s
    for c in range(6):
        for r in range(c, 6):
            s = P[6 * r + c]
            for m in range(c):
                s = s - M[6 * r + m] * M[6 * c + m]
            if r == c:
                if not s > 0:
                    return None
                M[6 * c + c] = math.sqrt(s)
            else:
                M[6 * r + c] = s / M[6 * c + c]
    return np.array(M).reshape(6, 6).T.copy()


def weights(wt=(10.0, 1.0, 10.0, 2.0, 3.0)):
    """S1, S23, S45 (optimization_be.cpp:896-903)"""
    wt_r, wt_t, n1, n23, n45 = wt
    d1 = np.array([wt_r * n1] * 3 + [wt_t * n1] * 3)
    return np.diag(d1), np.diag(d1 / n23), np.diag(d1 / n45)


def edge_topology(pr: dict, use_nbr=True):
    """(i, j, kind) of every edge in the rule's order; Refused where cvb_pgo refuses"""
    K = len(pr["kf_id"])
    pred, succ, kid = np.asarray(pr["kf_pred"]), np.asarray(pr["kf_succ"]), np.asarray(pr["kf_id"])
    cov = pr.get("loop_cov")
    out = []
    for l in range(len(pr["loop_i"])):
        if cov is not None and sqrt_info_from_cov(cov[l]) is None:
            raise Refused(f"loop {l}: covariance is not positive definite")
        a, b = int(pr["loop_i"][l]), int(pr["loop_j"][l])
        if not (0 <= a < K and 0 <= b < K and a != b):
            raise Refused(f"loop {l}: keyframes ({a}, {b}) invalid")
        out.append((a, b, EDGE_LOOP))
    seen = set()

    def push(a, b, kind):
        if (a, b) not in seen:
            seen.add((a, b))
            out.append((a, b, kind))
    for k in range(K):
        if succ[k] == -2:
            raise Refused(f"keyframe {k}: its successor is not among the keyframes")
        if succ[k] >= 0:
            push(k, int(succ[k]), EDGE_S1)
    if use_nbr:
        step_kind = [None, EDGE_S1, EDGE_S23, EDGE_S23, EDGE_S45, EDGE_S45]
        for k in range(K):
            t, conn = k, []
            for j in range(1, 6):
                if int(kid[k]) - j > 0:
                    t = int(pred[t])
                    if t < 0:
                        raise Refused(f"keyframe {k}: neighbour {j} is absent or not among the keyframes")
                    conn.append(t)
            for c, t in enumerate(conn):
                push(k, t, step_kind[c + 1])
    return out


def pgo_edges(pr: dict, wt=(10.0, 1.0, 10.0, 2.0, 3.0), use_nbr=True, use_robust=True):
    """the edges cvb_pgo hands its solve, as the flat edge dict of covins_b200.optimization (i, j, q, t, sqrt_info,
    robust) plus kind"""
    topo = edge_topology(pr, use_nbr)
    S = weights(wt)
    n = len(topo)
    I = np.array([e[0] for e in topo], np.int32); J = np.array([e[1] for e in topo], np.int32)
    kind = np.array([e[2] for e in topo], np.int32)
    Q = np.zeros((n, 4)); T = np.zeros((n, 3)); SI = np.zeros((n, 6, 6))
    cov = pr.get("loop_cov")
    nl = len(pr["loop_i"])
    for e in range(nl):
        Q[e] = pr["loop_q"][e]; T[e] = pr["loop_t"][e]
        SI[e] = S[0] if cov is None else sqrt_info_from_cov(cov[e])
    if n > nl:
        Tv = np.asarray(pr["T_ws_vio"], np.float64)
        R = rel_transform(Tv[I[nl:]], Tv[J[nl:]])
        for e in range(nl, n):
            p7 = transform_to_pose7(R[e - nl])
            Q[e] = p7[:4]; T[e] = p7[4:]
            SI[e] = S[kind[e] - 1]
    return dict(i=I, j=J, kind=kind, q=Q, t=T, sqrt_info=SI, robust=(kind == EDGE_LOOP) & bool(use_robust))


def start_poses(pr: dict) -> np.ndarray:
    """transform_to_pose7 of T_ws_init (T_ws when None), optimization_be.cpp:854-868"""
    T0 = pr.get("T_ws_init")
    T0 = pr["T_ws"] if T0 is None else T0
    return np.stack([transform_to_pose7(T) for T in np.asarray(T0, np.float64)]).reshape(-1, 7)


def writeback(pr: dict, pose7) -> dict:
    """what the shim writes back after the solve (optimization_be.cpp:1033-1083): T_ws_out, velocity_out, lm_out, lm_erase"""
    Tu = np.asarray(pr["T_ws"], np.float64).reshape(-1, 4, 4)
    Tc = pose7_to_transform(pose7)
    out = dict(T_ws_out=Tc.reshape(-1, 16))
    v = pr.get("velocity")
    if v is not None:
        v = np.asarray(v, np.float64)
        vo = np.zeros_like(v)
        for r in range(3):
            s = np.zeros(len(v))
            for c in range(3):
                m = np.zeros(len(v))
                for x in range(3):
                    m = m + Tc[:, r, x] * Tu[:, c, x]
                s = s + m * v[:, c]
            vo[:, r] = s
        out["velocity_out"] = vo
    pw = np.asarray(pr["lm_pos"], np.float64).reshape(-1, 3)
    ref = np.asarray(pr["lm_ref"], np.int64)
    has = np.asarray(pr["lm_has_obs"]).astype(bool)
    lo = pw.copy()
    ok = ref >= 0
    k = ref[ok]
    A, C, p = Tu[k], Tc[k], pw[ok]
    ps = np.zeros((len(k), 3))
    for r in range(3):
        s = np.zeros(len(k))
        for c in range(3):
            s = s + A[:, c, r] * (p[:, c] - A[:, c, 3])
        ps[:, r] = s
    for r in range(3):
        lo[ok, r] = ((C[:, r, 0] * ps[:, 0] + C[:, r, 1] * ps[:, 1]) + C[:, r, 2] * ps[:, 2]) + C[:, r, 3]
    out["lm_out"] = lo
    out["lm_erase"] = ((ref == -2) | ((ref == -1) & has)).astype(np.uint8)
    return out
