"""Seeded synthetic multi-agent visual-inertial map (SURVEY.md §8d) in the flat interchange format behind the
C-ABI (SURVEY.md Appendix B; struct cvb_ba_problem in include/covins_b200.h).  numpy only, deterministic.

Canonical orders (the reference iterates pointer-ordered containers, SURVEY §8c): keyframes by
(client_id, kf_id); landmarks by id; the observations of a landmark sorted by keyframe index.

Conventions (restated from upstream robopt_open / aslam — assumptions, SURVEY Appendix A):
  pose block  [qx,qy,qz,qw, x,y,z] = T_ws (keyframe_base.cpp:486-499); speed-bias [v_w, b_a, b_g];
  camera: pinhole + radtan, EuRoC cam0 (covins_frontend/config/EuRoC.yaml:9-17,34-41).
"""
from __future__ import annotations

import numpy as np

EUROC_INTR = np.array([458.654, 457.296, 367.215, 248.375])
EUROC_DIST = np.array([-0.28340811, 0.07395907, 0.00019359, 1.76187114e-05])
EUROC_TBC = np.array([[0.0148655429818, -0.999880929698, 0.00414029679422, -0.0216401454975],
                      [0.999557249008, 0.0149672133247, 0.025715529948, -0.064676986768],
                      [-0.0257744366974, 0.00375618835797, 0.999660727178, 0.00981073058949],
                      [0.0, 0.0, 0.0, 1.0]])
IMG_W, IMG_H = 752, 480
G = 9.81
IMU_HZ, KF_HZ = 200, 4
# IMU noise parameters handed to the preintegration (VINS-Mono-style: used as per-sample sigmas in V*Q*V^T),
# EuRoC-like (SURVEY §8d): sigma_a_c, sigma_g_c, sigma_aw_c, sigma_gw_c, g
IMU_NOISE = np.array([2e-3 * np.sqrt(200.0), 1.7e-4 * np.sqrt(200.0), 3e-3, 2e-5, G])


# ------------------------------------------------------------------------------------------------ SO(3)
def rot_to_quat(R):
    """[...,3,3] → [...,4] (x,y,z,w), w >= 0."""
    R = np.asarray(R)
    m00, m11, m22 = R[..., 0, 0], R[..., 1, 1], R[..., 2, 2]
    q = np.empty(R.shape[:-2] + (4,))
    w = np.sqrt(np.maximum(0, 1 + m00 + m11 + m22)) / 2
    x = np.sqrt(np.maximum(0, 1 + m00 - m11 - m22)) / 2
    y = np.sqrt(np.maximum(0, 1 - m00 + m11 - m22)) / 2
    z = np.sqrt(np.maximum(0, 1 - m00 - m11 + m22)) / 2
    x = np.copysign(x, R[..., 2, 1] - R[..., 1, 2])
    y = np.copysign(y, R[..., 0, 2] - R[..., 2, 0])
    z = np.copysign(z, R[..., 1, 0] - R[..., 0, 1])
    q[..., 0], q[..., 1], q[..., 2], q[..., 3] = x, y, z, w
    return q / np.linalg.norm(q, axis=-1, keepdims=True)


def quat_to_rot(q):
    q = np.asarray(q)
    x, y, z, w = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    R = np.empty(q.shape[:-1] + (3, 3))
    R[..., 0, 0] = 1 - 2 * (y * y + z * z); R[..., 0, 1] = 2 * (x * y - z * w); R[..., 0, 2] = 2 * (x * z + y * w)
    R[..., 1, 0] = 2 * (x * y + z * w); R[..., 1, 1] = 1 - 2 * (x * x + z * z); R[..., 1, 2] = 2 * (y * z - x * w)
    R[..., 2, 0] = 2 * (x * z - y * w); R[..., 2, 1] = 2 * (y * z + x * w); R[..., 2, 2] = 1 - 2 * (x * x + y * y)
    return R


def rot_exp(phi):
    phi = np.asarray(phi, float)
    th = np.linalg.norm(phi, axis=-1)[..., None, None]
    K = np.zeros(phi.shape[:-1] + (3, 3))
    K[..., 0, 1], K[..., 0, 2] = -phi[..., 2], phi[..., 1]
    K[..., 1, 0], K[..., 1, 2] = phi[..., 2], -phi[..., 0]
    K[..., 2, 0], K[..., 2, 1] = -phi[..., 1], phi[..., 0]
    small = th < 1e-8
    ths = np.where(small, 1.0, th)
    a = np.where(small, 1.0, np.sin(ths) / ths)
    b = np.where(small, 0.5, (1 - np.cos(ths)) / (ths * ths))
    return np.eye(3) + a * K + b * (K @ K)


def _euler_R(yaw, pitch, roll):
    cy, sy, cp, sp, cr, sr = np.cos(yaw), np.sin(yaw), np.cos(pitch), np.sin(pitch), np.cos(roll), np.sin(roll)
    R = np.empty(yaw.shape + (3, 3))
    R[..., 0, 0] = cy * cp; R[..., 0, 1] = cy * sp * sr - sy * cr; R[..., 0, 2] = cy * sp * cr + sy * sr
    R[..., 1, 0] = sy * cp; R[..., 1, 1] = sy * sp * sr + cy * cr; R[..., 1, 2] = sy * sp * cr - cy * sr
    R[..., 2, 0] = -sp; R[..., 2, 1] = cp * sr; R[..., 2, 2] = cp * cr
    return R


# ------------------------------------------------------------------------------------------------ camera
def project_radtan(pc, intr=EUROC_INTR, dist=EUROC_DIST):
    """pinhole + radtan (SURVEY Appendix A.3). pc [...,3] camera frame → uv [...,2]."""
    x, y = pc[..., 0] / pc[..., 2], pc[..., 1] / pc[..., 2]
    k1, k2, p1, p2 = dist
    r2 = x * x + y * y
    rad = 1 + k1 * r2 + k2 * r2 * r2
    xd = x * rad + 2 * p1 * x * y + p2 * (r2 + 2 * x * x)
    yd = y * rad + p1 * (r2 + 2 * y * y) + 2 * p2 * x * y
    return np.stack([intr[0] * xd + intr[2], intr[1] * yd + intr[3]], -1)


class _Traj:
    """Smooth 6-dof agent trajectory: sum of 3 sinusoids per axis + yaw sweep (SURVEY §8d)."""

    def __init__(self, rng, agent):
        self.A = rng.uniform(0.7, 1.7, (3, 3)) * np.array([1.0, 1.0, 0.35])[None, :]  # amplitude per (sinusoid, axis)
        self.w = rng.uniform(0.05, 0.22, (3, 3)) * np.array([[1.0], [1.9], [3.1]])
        self.ph = rng.uniform(0, 2 * np.pi, (3, 3))
        self.c = np.array([1.5 * np.cos(agent * 1.3), 1.5 * np.sin(agent * 1.3), 0.3 * agent])
        self.yaw_rate = rng.uniform(0.06, 0.12) * (1 if agent % 2 == 0 else -1)
        self.yaw0 = rng.uniform(0, 2 * np.pi)
        self.pr = rng.uniform(0.03, 0.08, 2); self.pw = rng.uniform(0.3, 0.6, 2); self.pp = rng.uniform(0, 6.28, 2)

    def pos(self, t, d=0):
        t = np.asarray(t)[..., None, None]
        arg = self.w * t + self.ph
        if d == 0:
            v = self.A * np.sin(arg)
        elif d == 1:
            v = self.A * self.w * np.cos(arg)
        else:
            v = -self.A * self.w ** 2 * np.sin(arg)
        out = v.sum(-2)
        return out + self.c if d == 0 else out

    def euler(self, t, d=0):
        t = np.asarray(t)
        if d == 0:
            return (self.yaw0 + self.yaw_rate * t + 0.3 * np.sin(0.21 * t), self.pr[0] * np.sin(self.pw[0] * t + self.pp[0]),
                    self.pr[1] * np.sin(self.pw[1] * t + self.pp[1]))
        return (self.yaw_rate + 0.3 * 0.21 * np.cos(0.21 * t), self.pr[0] * self.pw[0] * np.cos(self.pw[0] * t + self.pp[0]),
                self.pr[1] * self.pw[1] * np.cos(self.pw[1] * t + self.pp[1]))

    def R(self, t):
        return _euler_R(*self.euler(t))

    def omega_body(self, t):
        yaw, pitch, roll = self.euler(t)
        dy, dp, dr = self.euler(t, 1)
        return np.stack([dr - dy * np.sin(pitch), dp * np.cos(roll) + dy * np.cos(pitch) * np.sin(roll),
                         -dp * np.sin(roll) + dy * np.cos(pitch) * np.cos(roll)], -1)


def make_map(seed: int, n_agents: int, kf_per_agent: int, n_lm: int, mean_track: float = 8.0, outlier_frac: float = 0.05,
             pix_noise: float = 1.0, drift_trans: float = 0.002, drift_yaw_deg: float = 0.02, lm_noise: float = 0.01,
             with_imu: bool = True, loops_per_pair: int = 3, loops_intra: int = 2, candidate_window: int = 0):
    """→ dict of numpy arrays: the flat problem (initial = drifted state) plus ground truth under 'gt_*'.
    candidate_window > 0 (stress configs: C5 has 10^6 landmarks x 10^4 keyframes): a landmark's observers are searched only
    among its anchor's temporal neighbours (+- window) and the same time window of two other agents, instead of among all
    keyframes."""
    rng = np.random.default_rng(seed)
    K = n_agents * kf_per_agent
    dt_kf, dt_imu = 1.0 / KF_HZ, 1.0 / IMU_HZ
    spk = IMU_HZ // KF_HZ
    R_sc, t_sc = EUROC_TBC[:3, :3], EUROC_TBC[:3, 3]

    trajs = [_Traj(rng, a) for a in range(n_agents)]
    t_kf = np.arange(kf_per_agent) * dt_kf
    R_ws = np.concatenate([tr.R(t_kf) for tr in trajs])             # [K,3,3]
    p_ws = np.concatenate([tr.pos(t_kf) for tr in trajs])           # [K,3]
    v_w = np.concatenate([tr.pos(t_kf, 1) for tr in trajs])
    agent_of = np.repeat(np.arange(n_agents), kf_per_agent)
    kf_id = np.tile(np.arange(kf_per_agent), n_agents)
    R_wc = R_ws @ R_sc
    p_wc = p_ws + (R_ws @ t_sc)

    # ---- landmarks: back-projected from a random anchor KF, then tracked in other KFs that see them ----
    anchor = rng.integers(0, K, n_lm)
    xn = rng.uniform(-0.62, 0.62, n_lm); yn = rng.uniform(-0.42, 0.42, n_lm)
    depth = rng.uniform(1.0, 15.0, n_lm)
    pc = np.stack([xn * depth, yn * depth, depth], -1)
    lm_gt = np.einsum("nij,nj->ni", R_wc[anchor], pc) + p_wc[anchor]

    obs_lm, obs_kf = [], []
    want = np.clip(rng.geometric(1.0 / (mean_track - 1.0), n_lm) + 1, 2, 40)
    chunk = max(1, 8_000_000 // K)
    # camera-frame coordinates of every (landmark, KF) pair as ONE GEMM: pcam[c,k,:] = P[c] @ R_wc[k] - p_wc[k] @ R_wc[k]
    Rcat = np.ascontiguousarray(R_wc.transpose(1, 0, 2).reshape(3, 3 * K)).astype(np.float32)      # [3, K*3]
    off = np.einsum("kj,kji->ki", p_wc, R_wc).reshape(1, 3 * K).astype(np.float32)
    if candidate_window > 0:
        chunk = 20_000
        R32, p32 = R_wc.astype(np.float32), p_wc.astype(np.float32)
    for s in range(0, n_lm, chunk):
        P = lm_gt[s:s + chunk].astype(np.float32)                    # [c,3]; float32 is enough for the visibility test
        c = P.shape[0]
        if candidate_window > 0:
            # candidate keyframes: the anchor's agent and two other agents, each a time window around the anchor's time
            a = anchor[s:s + c]
            w = candidate_window
            t0 = kf_id[a]
            others = (agent_of[a][:, None] + rng.integers(1, max(n_agents, 2), (c, 2))) % n_agents
            ag = np.concatenate([agent_of[a][:, None], others], 1)                                 # [c,3]
            tt = np.clip(t0[:, None] + np.arange(-w, w + 1)[None, :], 0, kf_per_agent - 1)         # [c,2w+1]
            cand = (ag[:, :, None] * kf_per_agent + tt[:, None, :]).reshape(c, -1)                  # [c, 3(2w+1)]
            cand = np.sort(cand, axis=1)
            dup = np.concatenate([np.zeros((c, 1), bool), cand[:, 1:] == cand[:, :-1]], 1)          # clipped windows repeat indices
            d = P[:, None, :] - p32[cand]
            pc_ = np.einsum("cnji,cnj->cni", R32[cand], d)
            z = pc_[..., 2]
            vis = (z > 0.5) & (z < 20.0) & ~dup
            iz = 1.0 / np.where(vis, z, np.float32(1))
            xn_ = pc_[..., 0] * iz; yn_ = pc_[..., 1] * iz
            r2 = xn_ * xn_ + yn_ * yn_
            vis &= r2 < 0.75
            rad = 1 + np.float32(EUROC_DIST[0]) * r2 + np.float32(EUROC_DIST[1]) * r2 * r2
            xn_ *= rad; yn_ *= rad
            vis &= (np.abs(xn_ * np.float32(EUROC_INTR[0]) + np.float32(EUROC_INTR[2] - IMG_W / 2)) < IMG_W / 2 - 8)
            vis &= (np.abs(yn_ * np.float32(EUROC_INTR[1]) + np.float32(EUROC_INTR[3] - IMG_H / 2)) < IMG_H / 2 - 8)
            vis |= (cand == a[:, None]) & ~dup
            rows, cc = np.nonzero(vis)
            cols = cand[rows, cc]
            ar = a[rows]
            key = np.where(agent_of[cols] == agent_of[ar], np.abs(kf_id[cols] - kf_id[ar]).astype(np.float64), 30.0 + rng.uniform(0, 60, len(rows)))
            key = key + rng.uniform(0, 12, len(rows))
            key[cols == ar] = -1.0
            o = np.lexsort((key, rows))
            rows, cols = rows[o], cols[o]
            start_of_row = np.searchsorted(rows, np.arange(c))
            rank_ = np.arange(len(rows)) - start_of_row[rows]
            keep = rank_ < want[s:s + c][rows]
            rows, cols = rows[keep], cols[keep]
            o = np.lexsort((cols, rows))
            obs_lm.append(s + rows[o]); obs_kf.append(cols[o])
            continue
        pcam = (P @ Rcat - off).reshape(c, K, 3)
        z = pcam[..., 2]
        vis = (z > 0.5) & (z < 20.0)
        iz = 1.0 / np.where(vis, z, np.float32(1))
        xn_ = pcam[..., 0] * iz; yn_ = pcam[..., 1] * iz
        r2 = xn_ * xn_ + yn_ * yn_
        vis &= r2 < 0.75                                              # stay inside the monotone region of radtan
        rad = 1 + np.float32(EUROC_DIST[0]) * r2 + np.float32(EUROC_DIST[1]) * r2 * r2
        xn_ *= rad; yn_ *= rad
        vis &= (np.abs(xn_ * np.float32(EUROC_INTR[0]) + np.float32(EUROC_INTR[2] - IMG_W / 2)) < IMG_W / 2 - 8)
        vis &= (np.abs(yn_ * np.float32(EUROC_INTR[1]) + np.float32(EUROC_INTR[3] - IMG_H / 2)) < IMG_H / 2 - 8)
        a = anchor[s:s + c]
        vis[np.arange(c), a] = True                                   # the anchor always observes its landmark
        rows, cols = np.nonzero(vis)
        # prefer temporal neighbours of the anchor, keep a share of far / cross-agent views
        ar = a[rows]
        key = np.where(agent_of[cols] == agent_of[ar], np.abs(kf_id[cols] - kf_id[ar]).astype(np.float64),
                       30.0 + rng.uniform(0, 60, len(rows)))
        key = key + rng.uniform(0, 12, len(rows))
        key[cols == ar] = -1.0
        o = np.lexsort((key, rows))
        rows, cols = rows[o], cols[o]
        start_of_row = np.searchsorted(rows, np.arange(c))
        rank = np.arange(len(rows)) - start_of_row[rows]
        keep = rank < want[s:s + c][rows]
        rows, cols = rows[keep], cols[keep]
        o = np.lexsort((cols, rows))                                  # observations of a LM sorted by KF index
        obs_lm.append(s + rows[o]); obs_kf.append(cols[o])
    obs_lm = np.concatenate(obs_lm); obs_kf = np.concatenate(obs_kf).astype(np.int32)
    cnt = np.bincount(obs_lm, minlength=n_lm)
    lm_obs_ptr = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int32)
    n_obs = len(obs_kf)
    pcam = np.einsum("nji,nj->ni", R_wc[obs_kf], lm_gt[obs_lm] - p_wc[obs_kf])
    uv = project_radtan(pcam) + rng.normal(0, pix_noise, (n_obs, 2))
    out = rng.random(n_obs) < outlier_frac
    uv[out] = np.stack([rng.uniform(8, IMG_W - 8, out.sum()), rng.uniform(8, IMG_H - 8, out.sum())], -1)
    octave = rng.integers(0, 8, n_obs)
    obs_sigma = (octave + 1) * 2.0                                    # opt.cpp:183-184

    # ---- drifted initial state: per-agent smooth drift applied to KFs and to the LMs anchored there ----
    dist_trav = np.concatenate([np.concatenate([[0], np.cumsum(np.linalg.norm(np.diff(tr.pos(t_kf), axis=0), axis=1))]) for tr in trajs])
    dyaw = np.deg2rad(drift_yaw_deg) * dist_trav * np.repeat(rng.choice([-1, 1], n_agents), kf_per_agent)
    dtr = drift_trans * dist_trav[:, None] * np.repeat(rng.normal(0, 1, (n_agents, 3)), kf_per_agent, axis=0)
    dtr[agent_of == 0] *= 0.2; dyaw[agent_of == 0] *= 0.2
    Rd = rot_exp(np.stack([np.zeros(K), np.zeros(K), dyaw], -1))     # drift about the first pose of the agent
    first = (agent_of * kf_per_agent)
    p0 = p_ws[first]
    R_ws_i = Rd @ R_ws
    p_ws_i = np.einsum("kij,kj->ki", Rd, p_ws - p0) + p0 + dtr
    lm_i = np.einsum("nij,nj->ni", Rd[anchor], lm_gt - p0[anchor]) + p0[anchor] + dtr[anchor] + rng.normal(0, lm_noise, (n_lm, 3))
    v_i = np.einsum("kij,kj->ki", Rd, v_w) + rng.normal(0, 0.02, (K, 3))

    pose = np.concatenate([rot_to_quat(R_ws_i), p_ws_i], -1)
    pose_gt = np.concatenate([rot_to_quat(R_ws), p_ws], -1)
    pose_const = np.zeros(K, np.uint8); pose_const[0] = 1            # KF (0, map id): opt.cpp:88-89
    extr = np.concatenate([rot_to_quat(R_sc), t_sc])[None, :]

    prob = dict(K=K, L=n_lm, pose=pose, pose_const=pose_const, cam_of_kf=np.zeros(K, np.int32), extr=extr,
                intr=EUROC_INTR[None, :].copy(), dist=EUROC_DIST[None, :].copy(), lm=lm_i, lm_obs_ptr=lm_obs_ptr,
                obs_kf=obs_kf, obs_uv=uv.astype(np.float32), obs_sigma=obs_sigma.astype(np.float64),
                agent_of=agent_of.astype(np.int32), kf_id=kf_id.astype(np.int32),
                gt_pose=pose_gt, gt_lm=lm_gt, obs_is_outlier=out)

    # ---- IMU: 200 Hz samples between consecutive KFs of an agent (factor of KF j links pred i → j) ----
    ba_gt = np.zeros((K, 3)); bg_gt = np.zeros((K, 3))
    if with_imu:
        imu_i, imu_j, imu_dt, imu_acc, imu_gyr, acc0, gyr0, ptr = [], [], [], [], [], [], [], [0]
        sa, sg, saw, sgw, _ = IMU_NOISE
        for a, tr in enumerate(trajs):
            ba = rng.normal(0, 0.02, 3); bg = rng.normal(0, 0.002, 3)
            for k in range(kf_per_agent):
                gi = a * kf_per_agent + k
                ba_gt[gi], bg_gt[gi] = ba, bg
                if k == kf_per_agent - 1:
                    break
                ts = t_kf[k] + np.arange(spk + 1) * dt_imu
                Rt = tr.R(ts)
                acc = np.einsum("nji,nj->ni", Rt, tr.pos(ts, 2) + np.array([0, 0, G])) + ba + rng.normal(0, sa, (spk + 1, 3))
                gyr = tr.omega_body(ts) + bg + rng.normal(0, sg, (spk + 1, 3))
                imu_i.append(gi); imu_j.append(gi + 1)
                acc0.append(acc[0]); gyr0.append(gyr[0])
                imu_dt.append(np.full(spk, dt_imu)); imu_acc.append(acc[1:]); imu_gyr.append(gyr[1:])
                ptr.append(ptr[-1] + spk)
                ba = ba + rng.normal(0, saw * np.sqrt(dt_kf * dt_imu), 3); bg = bg + rng.normal(0, sgw * np.sqrt(dt_kf * dt_imu), 3)
        prob.update(imu_i=np.array(imu_i, np.int32), imu_j=np.array(imu_j, np.int32), imu_ptr=np.array(ptr, np.int32),
                    imu_dt=np.concatenate(imu_dt), imu_acc=np.concatenate(imu_acc), imu_gyr=np.concatenate(imu_gyr),
                    imu_acc0=np.array(acc0), imu_gyr0=np.array(gyr0), imu_noise=IMU_NOISE.copy())
    else:
        prob.update(imu_i=np.zeros(0, np.int32), imu_j=np.zeros(0, np.int32), imu_ptr=np.zeros(1, np.int32),
                    imu_dt=np.zeros(0), imu_acc=np.zeros((0, 3)), imu_gyr=np.zeros((0, 3)), imu_acc0=np.zeros((0, 3)),
                    imu_gyr0=np.zeros((0, 3)), imu_noise=IMU_NOISE.copy())
    sb = np.concatenate([v_i, ba_gt + rng.normal(0, 0.005, (K, 3)), bg_gt + rng.normal(0, 0.0005, (K, 3))], -1)
    prob["speedbias"] = sb
    prob["gt_speedbias"] = np.concatenate([v_w, ba_gt, bg_gt], -1)

    # ---- loop constraints: T_s1_s2 = truth + noise (1 cm / 0.2 deg) ----
    li, lj = [], []
    for a in range(n_agents):
        for _ in range(loops_intra):
            i = rng.integers(0, kf_per_agent // 3); j = rng.integers(2 * kf_per_agent // 3, kf_per_agent)
            li.append(a * kf_per_agent + i); lj.append(a * kf_per_agent + j)
        for b in range(a + 1, n_agents):
            for _ in range(loops_per_pair):
                li.append(a * kf_per_agent + rng.integers(0, kf_per_agent)); lj.append(b * kf_per_agent + rng.integers(0, kf_per_agent))
    li, lj = np.array(li, np.int32).reshape(-1), np.array(lj, np.int32).reshape(-1)
    nl = len(li)
    R12 = np.einsum("nji,njk->nik", R_ws[li], R_ws[lj]) @ rot_exp(rng.normal(0, np.deg2rad(0.2), (nl, 3))) if nl else np.zeros((0, 3, 3))
    t12 = np.einsum("nji,nj->ni", R_ws[li], p_ws[lj] - p_ws[li]) + rng.normal(0, 0.01, (nl, 3)) if nl else np.zeros((0, 3))
    prob.update(loop_i=li, loop_j=lj, loop_q=rot_to_quat(R12) if nl else np.zeros((0, 4)), loop_t=t12,
                loop_cov=np.tile(np.eye(6)[None], (nl, 1, 1)))
    return prob


# named configs of BASELINE.json (SURVEY §8 sizes)
CONFIGS = {
    "tiny": dict(n_agents=2, kf_per_agent=12, n_lm=300),
    "small": dict(n_agents=2, kf_per_agent=40, n_lm=2000),
    "C1": dict(n_agents=1, kf_per_agent=200, n_lm=10_000),
    "C2": dict(n_agents=2, kf_per_agent=400, n_lm=40_000),
    "C3": dict(n_agents=5, kf_per_agent=400, n_lm=100_000),
    # BASELINE.json config 5: 12-agent 10k-KF / 1M-landmark stress map (observers searched in a +-40-keyframe window of three agents)
    "C5": dict(n_agents=12, kf_per_agent=834, n_lm=1_000_000, candidate_window=40),
    "C5s": dict(n_agents=12, kf_per_agent=100, n_lm=60_000, candidate_window=40),      # small stand-in with the same generator path (tests)
}


# default distortion coefficients per dist_model: EuRoC radtan, a mild equidistant lens, FOV with w = 0.93
DEFAULT_DIST = {0: EUROC_DIST, 1: np.array([-0.013, 0.02, -0.012, 0.002]), 2: np.array([0.93, 0.0, 0.0, 0.0])}


def project_model(pc, intr, d, cam_model: int, dist_model: int, xi: float = 0.0):
    """camera-frame points pc [n,3] → pixels [n,2] through one GlobalEuclideanReprError<Camera, Distortion> model:
    cam_model 0 pinhole / 1 unified(xi), dist_model 0 radtan / 1 equidistant / 2 fisheye (FOV)."""
    den = pc[:, 2] + (xi * np.linalg.norm(pc, axis=1) if cam_model == 1 else 0.0)
    x, y = pc[:, 0] / den, pc[:, 1] / den
    r2 = x * x + y * y
    if dist_model == 0:
        rad = 1 + d[0] * r2 + d[1] * r2 * r2
        xd = x * rad + 2 * d[2] * x * y + d[3] * (r2 + 2 * x * x); yd = y * rad + d[2] * (r2 + 2 * y * y) + 2 * d[3] * x * y
    elif dist_model == 1:
        r = np.sqrt(r2); th = np.arctan(r); t2 = th * th
        s = np.where(r > 1e-8, th * (1 + d[0] * t2 + d[1] * t2 ** 2 + d[2] * t2 ** 3 + d[3] * t2 ** 4) / np.maximum(r, 1e-12), 1.0)
        xd, yd = s * x, s * y
    else:
        w = d[0]; c = 2 * np.tan(0.5 * w); r = np.sqrt(r2)
        s = np.where(r2 < 1e-5, c / w, np.arctan(c * r) / (w * np.maximum(r, 1e-12)))
        xd, yd = s * x, s * y
    return np.stack([intr[0] * xd + intr[2], intr[1] * yd + intr[3]], -1)


def with_camera_model(p: dict, cam_model: int, dist_model: int, dist=None, xi: float = 0.0, seed: int = 0, pix_noise: float = 1.0):
    """The same map observed through another GlobalEuclideanReprError<Camera, Distortion> instantiation
    (optimization_be.cpp:186-231): cam_model 0 pinhole / 1 unified(xi), dist_model 0 radtan / 1 equidistant / 2 fisheye (FOV).
    The inlier observations are re-projected from the ground truth with the new model (+ pixel noise); gross outliers keep
    their random pixels."""
    q = dict(p)
    d = np.asarray(DEFAULT_DIST[dist_model] if dist is None else dist, float)
    rng = np.random.default_rng(seed)
    R_ws = quat_to_rot(p["gt_pose"][:, :4]); t_ws = p["gt_pose"][:, 4:]
    R_sc = quat_to_rot(p["extr"][0][:4]); t_sc = p["extr"][0][4:]
    obs_lm = np.repeat(np.arange(p["L"]), np.diff(p["lm_obs_ptr"]))
    k = p["obs_kf"]
    ps = np.einsum("nji,nj->ni", R_ws[k], p["gt_lm"][obs_lm] - t_ws[k])
    pc = (ps - t_sc) @ R_sc
    uv = project_model(pc, p["intr"][0], d, cam_model, dist_model, xi) + rng.normal(0, pix_noise, (len(k), 2))
    keep = p["obs_is_outlier"]
    uv[keep] = p["obs_uv"][keep]
    q["obs_uv"] = uv.astype(np.float32)
    q["dist"] = d[None, :].copy()
    q["cam_model"] = np.array([cam_model], np.int32); q["dist_model"] = np.array([dist_model], np.int32); q["cam_xi"] = np.array([xi])
    return q


_CACHE_VERSION = "r02b"   # bump when make_map changes


def make_config(name: str, seed: int | None = None, **kw):
    """Named BASELINE config.  The map is a pure function of (name, seed, kw): the big ones (C2 14 s, C3 60 s of numpy)
    are cached as .npz under $COVINS_B200_CACHE (default /tmp/covins_b200_cache) so that the tests, bench.py and its CPU arm
    — separate processes on the same box — generate them once."""
    import os
    cfg = dict(CONFIGS[name]); cfg.update(kw)
    seed = seed if seed is not None else list(CONFIGS).index(name)
    K = cfg["n_agents"] * cfg["kf_per_agent"]
    path = None
    if K >= 400 and os.environ.get("COVINS_B200_CACHE", "") != "off":
        d = os.environ.get("COVINS_B200_CACHE", "/tmp/covins_b200_cache")
        tag = "_".join(f"{k}={v}" for k, v in sorted(cfg.items()))
        path = os.path.join(d, f"{_CACHE_VERSION}_{name}_{seed}_{tag}.npz")
        if os.path.exists(path):
            try:
                with np.load(path) as z:
                    p = {k: z[k] for k in z.files}
                p["K"] = int(p["K"]); p["L"] = int(p["L"])
                return p
            except Exception:
                pass
    p = make_map(seed, **cfg)
    if path is not None:
        try:
            os.makedirs(os.path.dirname(path), exist_ok=True)
            tmp = path + f".{os.getpid()}.tmp.npz"
            np.savez(tmp, **p)
            os.replace(tmp, path)
        except Exception:
            pass
    return p
