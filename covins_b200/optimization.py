"""Host-side mirror of the reference's `Optimization` class on the flat problem format, over the C-ABI.

  global_bundle_adjustment(...)  ↔ Optimization::GlobalBundleAdjustment  (optimization_be.cpp:56-618)
  pose_graph_optimization(...)   ↔ Optimization::PoseGraphOptimization   (optimization_be.cpp:833-1086)
  BaSolver                       ↔ one ceres::Problem + ceres::Solve (create / iterate / result), used by bench.py
                                   and by the multi-GPU path (landmark-block sharding + all-reduce callback)
  Group, solve_group(...), global_bundle_adjustment_group(...)
                                 ↔ the same solves sharded over several contexts of this process (one host thread
                                   per rank, in-process all-reduce in rank order, optional peer path)

`problem` is the dict produced by covins_b200.synth_map (or by the C++ shim's flatten step): numpy arrays in the
canonical orders of SURVEY.md §8c.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._lib import Context, lib, c_vp


class BaProblem(C.Structure):
    _fields_ = [("K", C.c_int32), ("L", C.c_int32), ("n_obs", C.c_int32), ("n_imu", C.c_int32), ("n_edge", C.c_int32),
                ("n_cam", C.c_int32)] + [(n, c_vp) for n in (
                    "pose", "speedbias", "pose_const", "cam_of_kf", "extr", "intr", "dist", "lm", "lm_obs_ptr", "obs_kf",
                    "obs_uv", "obs_sigma", "obs_skip", "imu_i", "imu_j", "imu_ptr", "imu_dt", "imu_acc", "imu_gyr",
                    "imu_acc0", "imu_gyr0", "imu_noise", "edge_i", "edge_j", "edge_q", "edge_t", "edge_sqrt_info",
                    "edge_robust", "cam_model", "dist_model", "cam_xi")]


class BaOptions(C.Structure):
    _fields_ = [("max_iterations", C.c_int32), ("visual_only", C.c_int32), ("cauchy_reproj", C.c_double),
                ("cauchy_edge", C.c_double), ("rank", C.c_int32), ("world", C.c_int32)]


class BaResult(C.Structure):
    _fields_ = [("pose", c_vp), ("speedbias", c_vp), ("lm", c_vp), ("lm_owner", c_vp), ("cost_history", c_vp),
                ("step_status", c_vp), ("cost_history_cap", C.c_int32), ("n_cost_history", C.c_int32),
                ("iterations", C.c_int32), ("termination", C.c_int32), ("initial_cost", C.c_double),
                ("final_cost", C.c_double)]


class GbaOptions(C.Structure):
    _fields_ = [("iterations_limit", C.c_int32), ("visual_only", C.c_int32), ("outlier_removal", C.c_int32),
                ("th_outlier", C.c_double)]


ALLREDUCE_FN = C.CFUNCTYPE(C.c_int, c_vp, c_vp, C.c_size_t, c_vp)

TERMINATION = {0: "NO_CONVERGENCE", 1: "CONVERGENCE(gradient)", 2: "CONVERGENCE(parameter)", 3: "CONVERGENCE(function)",
               4: "FAILURE"}
STEP = {1: "accepted", 2: "rejected", 3: "invalid", 4: "converged"}

GBA_LOOP_SQRT_INFO = np.diag([100.0] * 3 + [1e4] * 3)  # optimization_be.cpp:238-240, 534-536


def _arr(a, dt):
    return None if a is None else np.ascontiguousarray(a, dtype=dt)


class _Flat:
    """Keeps the contiguous arrays alive and exposes the ctypes struct."""

    def __init__(self, p: dict, edges: dict | None = None, obs_skip=None, use_imu: bool = True):
        K = int(p["K"]); L = int(p.get("L", 0))
        self.a = a = {}
        a["pose"] = _arr(p["pose"], np.float64)
        a["speedbias"] = _arr(p.get("speedbias"), np.float64)
        a["pose_const"] = _arr(p["pose_const"], np.uint8)
        a["cam_of_kf"] = _arr(p.get("cam_of_kf"), np.int32)
        a["extr"] = _arr(p["extr"], np.float64).reshape(-1, 7)
        a["intr"] = _arr(p.get("intr", np.zeros((len(a["extr"]), 4))), np.float64)
        a["dist"] = _arr(p.get("dist", np.zeros((len(a["extr"]), 4))), np.float64)
        # GlobalEuclideanReprError<Camera, Distortion> template arguments per calibration (None = pinhole / radtan)
        a["cam_model"] = _arr(p.get("cam_model"), np.int32); a["dist_model"] = _arr(p.get("dist_model"), np.int32)
        a["cam_xi"] = _arr(p.get("cam_xi"), np.float64)
        a["lm"] = _arr(p.get("lm", np.zeros((0, 3))), np.float64)
        a["lm_obs_ptr"] = _arr(p.get("lm_obs_ptr", np.zeros(1)), np.int32)
        a["obs_kf"] = _arr(p.get("obs_kf", np.zeros(0)), np.int32)
        a["obs_uv"] = _arr(p.get("obs_uv", np.zeros((0, 2))), np.float32)
        a["obs_sigma"] = _arr(p.get("obs_sigma", np.zeros(0)), np.float64)
        a["obs_skip"] = _arr(obs_skip, np.uint8)
        n_imu = len(p.get("imu_i", [])) if use_imu else 0
        for k, dt in (("imu_i", np.int32), ("imu_j", np.int32), ("imu_ptr", np.int32), ("imu_dt", np.float64),
                      ("imu_acc", np.float64), ("imu_gyr", np.float64), ("imu_acc0", np.float64), ("imu_gyr0", np.float64),
                      ("imu_noise", np.float64)):
            a[k] = _arr(p.get(k), dt) if n_imu else None
        if edges is None and len(p.get("loop_i", [])) > 0:   # GBA: the map's loop constraints (optimization_be.cpp:539-556)
            n = len(p["loop_i"])
            edges = dict(i=p["loop_i"], j=p["loop_j"], q=p["loop_q"], t=p["loop_t"],
                         sqrt_info=np.tile(GBA_LOOP_SQRT_INFO[None], (n, 1, 1)), robust=np.ones(n, np.uint8))
        n_edge = 0
        if edges is not None and len(edges["i"]) > 0:
            n_edge = len(edges["i"])
            a["edge_i"] = _arr(edges["i"], np.int32); a["edge_j"] = _arr(edges["j"], np.int32)
            a["edge_q"] = _arr(edges["q"], np.float64); a["edge_t"] = _arr(edges["t"], np.float64)
            a["edge_sqrt_info"] = _arr(np.asarray(edges["sqrt_info"]).reshape(n_edge, 36), np.float64)
            a["edge_robust"] = _arr(edges["robust"], np.uint8)
        s = BaProblem()
        s.K, s.L, s.n_obs, s.n_imu, s.n_edge, s.n_cam = K, L, len(a["obs_kf"]), n_imu, n_edge, len(a["extr"])
        for name, _ in BaProblem._fields_[6:]:
            v = a.get(name)
            setattr(s, name, v.ctypes.data if v is not None else None)
        self.s = s
        self.K, self.L, self.n_obs = K, L, s.n_obs


class _Res:
    def __init__(self, K, L, cap=64):
        self.pose = np.zeros((K, 7)); self.sb = np.zeros((K, 9)); self.lm = np.zeros((max(L, 1), 3))
        self.owner = np.zeros(max(L, 1), np.int32); self.hist = np.zeros(cap); self.status = np.zeros(cap, np.uint8)
        r = BaResult()
        r.pose, r.speedbias, r.lm, r.lm_owner = self.pose.ctypes.data, self.sb.ctypes.data, self.lm.ctypes.data, self.owner.ctypes.data
        r.cost_history, r.step_status, r.cost_history_cap = self.hist.ctypes.data, self.status.ctypes.data, cap
        self.r = r
        self.L = L

    def as_dict(self):
        r = self.r
        n = r.n_cost_history
        return dict(pose=self.pose, speedbias=self.sb, lm=self.lm[:self.L], lm_owner=self.owner[:self.L],
                    cost=self.hist[:n].copy(), steps=[STEP.get(int(x), "?") for x in self.status[:max(n - 1, 0)]],
                    iterations=int(r.iterations), termination=TERMINATION.get(int(r.termination), "?"),
                    initial_cost=float(r.initial_cost), final_cost=float(r.final_cost))


class BaSolver:
    """create → iterate(n) → result(); one ceres::Problem/Solve equivalent living on the GPU."""

    def __init__(self, ctx: Context, p: dict, visual_only=False, cauchy_reproj=1.0, cauchy_edge=1.0, edges=None,
                 obs_skip=None, rank=0, world=1, allreduce=None, p2p=None):
        import os
        if p2p is None:
            p2p = os.environ.get("COVINS_B200_P2P", "1") != "0"
        self.ctx = ctx
        self.flat = _Flat(p, edges=edges, obs_skip=obs_skip, use_imu=not visual_only)
        o = BaOptions(0, int(visual_only), float(cauchy_reproj), float(cauchy_edge), rank, world)
        self.h = c_vp()
        self._cb = None
        # the all-reduce must be installed before iteration 0 runs inside create() when world > 1: create() only
        # evaluates rank-local quantities that are summed lazily, so we create first and restart after installing it.
        ctx.check(lib().cvb_ba_create(ctx.handle, C.byref(self.flat.s), C.byref(o), C.byref(self.h)))
        self.p2p = False
        if allreduce is not None:
            self._cb = ALLREDUCE_FN(allreduce)
            ctx.check(lib().cvb_ba_set_allreduce(self.h, self._cb, None))
            if world > 1 and p2p:
                # peer path (CUDA IPC over NVLink): reduce-scatter by pull + column-distributed factorisation; falls back to
                # the all-reduce + replicated factorisation when peer mapping is unavailable (CVB_ERR_UNSUPPORTED = 3)
                rc = lib().cvb_ba_enable_p2p(self.h)
                if rc not in (0, 3):
                    ctx.check(rc)
                self.p2p = rc == 0
            ctx.check(lib().cvb_ba_restart(self.h))

    def restart(self):
        self.ctx.check(lib().cvb_ba_restart(self.h))

    def iterate(self, n: int) -> int:
        done = C.c_int(0)
        self.ctx.check(lib().cvb_ba_iterate(self.h, n, C.byref(done)))
        return done.value

    def reproj_norms(self):
        out = np.zeros(max(self.flat.n_obs, 1))
        self.ctx.check(lib().cvb_ba_reproj_norms(self.h, out.ctypes.data, self.flat.n_obs))
        return out[:self.flat.n_obs]

    def debug_vector(self, which: int):
        """(camera part [K*per], landmark part [3*L_in]) of an internal vector; see cvb_ba_debug_vector."""
        ncp = C.c_int64(); nt = C.c_int64()
        self.ctx.check(lib().cvb_ba_debug_vector(self.h, which, None, 0, C.byref(ncp), C.byref(nt)))
        out = np.zeros(nt.value)
        self.ctx.check(lib().cvb_ba_debug_vector(self.h, which, out.ctypes.data, nt.value, None, None))
        return out[:ncp.value], out[ncp.value:]

    def timing(self, reset=True):
        out = (C.c_double * 6)()
        self.ctx.check(lib().cvb_ba_timing(self.h, out, int(reset)))
        return dict(linearize_ms=out[0], build_schur_ms=out[1], factor_ms=out[2], solve_ms=out[3], step_ms=out[4],
                    factor_flops=out[5])

    def result(self):
        res = _Res(self.flat.K, self.flat.L)
        self.ctx.check(lib().cvb_ba_result_get(self.h, C.byref(self.flat.s), C.byref(res.r)))
        return res.as_dict()

    def close(self):
        if self.h:
            lib().cvb_ba_destroy(self.h)
            self.h = c_vp()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def torch_allreduce():
    """All-reduce callback for BaSolver(world > 1): sums `count` doubles at a device pointer over the default
    torch.distributed group (NCCL over NVLink), ordered on the engine's stream.  This is the only exchange of the
    GBA data path: the reduced normal equations (S, g_c, y_b) and a handful of scalars per iteration."""
    import torch
    import torch.distributed as dist

    class _Ptr:
        def __init__(self, ptr, n):
            self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f8", "data": (ptr, False), "version": 3}

    import os
    debug = os.environ.get("COVINS_B200_AR_DEBUG")
    state = {"n": 0}

    def fn(user, ptr, count, stream):
        try:
            if debug:
                state["n"] += 1
                print(f"[allreduce rank {dist.get_rank()}] #{state['n']} count={count}", flush=True)
            ext = torch.cuda.ExternalStream(stream)
            with torch.cuda.stream(ext):
                t = torch.as_tensor(_Ptr(ptr, count), device="cuda")
                # NCCL caps a single call's element count comfortably above 2^31 bytes, but chunk anyway for safety
                step = 1 << 28
                for a in range(0, count, step):
                    dist.all_reduce(t[a:a + step])
            return 0
        except Exception as e:  # never let an exception cross the C boundary
            print("allreduce callback failed:", e, flush=True)
            return 1
    return fn


def lm_owner_of_rank(n_included: int, world: int):
    """Landmark-block sharding rule of the engine: the i-th landmark that is in the problem belongs to rank i % world."""
    return np.arange(n_included) % max(world, 1)


def merge_sharded_landmarks(results: list):
    """Combine per-rank results of a sharded solve: poses/speed-biases are replicated, each landmark is taken from
    the rank that owns it (result['lm_owner'])."""
    out = dict(results[0])
    lm = results[0]["lm"].copy()
    owner = results[0]["lm_owner"]
    for r, res in enumerate(results):
        m = owner == r
        lm[m] = res["lm"][m]
    out["lm"] = lm
    return out


def global_bundle_adjustment(ctx: Context, p: dict, iterations_limit=10, visual_only=False, outlier_removal=True,
                             th_outlier=0.92):
    """Optimization::GlobalBundleAdjustment(map, interations_limit, time_limit, visual_only, outlier_removal, -):
    two-round VI bundle adjustment; defaults gba_iteration_limit 10, th_gba_outlier_global 0.92
    (config/config_backend.yaml:115,118).  → dict(pose, speedbias, lm, obs_removed, ...)."""
    flat = _Flat(p, use_imu=not visual_only)
    res = _Res(flat.K, flat.L)
    removed = np.zeros(max(flat.n_obs, 1), np.uint8)
    g = GbaOptions(int(iterations_limit), int(visual_only), int(outlier_removal), float(th_outlier))
    ctx.check(lib().cvb_gba(ctx.handle, C.byref(flat.s), C.byref(g), C.byref(res.r), removed.ctypes.data))
    out = res.as_dict()
    out["obs_removed"] = removed[:flat.n_obs].astype(bool)
    return out


GROUP_ALLREDUCE_CHUNK = 1 << 21   # CVB_GROUP_ALLREDUCE_CHUNK: doubles per chunk of the group all-reduce


class Group:
    """cvb_group over Contexts of this process: rank r = contexts[r].  Several contexts may share a device.  The group
    does not own the contexts; close it before them."""

    def __init__(self, contexts):
        self.contexts = list(contexts)
        self.ctx = self.contexts[0] if self.contexts else None
        arr = (c_vp * max(len(self.contexts), 1))(*[c.handle for c in self.contexts])
        self.h = c_vp()
        rc = lib().cvb_group_create(arr, len(self.contexts), C.byref(self.h))
        if rc != 0:
            if self.ctx is None:
                from ._lib import CvbError
                raise CvbError(f"status {rc}: cvb_group_create")
            self.ctx.check(rc)

    @property
    def n(self):
        return len(self.contexts)

    def allreduce_diag(self, bufs):
        """the group all-reduce alone: bufs [n][count] float64 (rank r's buffer) → what every rank holds afterwards"""
        x = np.ascontiguousarray(bufs, np.float64).reshape(self.n, -1)
        out = np.zeros_like(x)
        self.ctx.check(lib().cvb_group_allreduce_diag(self.h, x.ctypes.data, x.shape[1], out.ctypes.data))
        return out

    def close(self):
        if self.h:
            lib().cvb_group_destroy(self.h)
            self.h = c_vp()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def solve_group(group: Group, p: dict, max_iterations: int, visual_only=False, cauchy_reproj=1.0, cauchy_edge=1.0,
                edges=None, obs_skip=None, peer_path=False):
    """solve() sharded over the ranks of `group` (cvb_ba_solve_group): merged result, landmarks from their owners.
    peer_path: reduce-scatter by peer pull + column-distributed factorisation (a device per rank; not yet verified on
    several devices, so off by default) instead of the all-reduce of the packed reduced system."""
    flat = _Flat(p, edges=edges, obs_skip=obs_skip, use_imu=not visual_only)
    res = _Res(flat.K, flat.L)
    o = BaOptions(int(max_iterations), int(visual_only), float(cauchy_reproj), float(cauchy_edge), 0, 1)
    group.ctx.check(lib().cvb_ba_solve_group(group.h, C.byref(flat.s), C.byref(o), int(bool(peer_path)), C.byref(res.r)))
    return res.as_dict()


def global_bundle_adjustment_group(group: Group, p: dict, iterations_limit=10, visual_only=False, outlier_removal=True,
                                   th_outlier=0.92, peer_path=False):
    """global_bundle_adjustment() sharded over the ranks of `group` (cvb_gba_group)."""
    flat = _Flat(p, use_imu=not visual_only)
    res = _Res(flat.K, flat.L)
    removed = np.zeros(max(flat.n_obs, 1), np.uint8)
    g = GbaOptions(int(iterations_limit), int(visual_only), int(outlier_removal), float(th_outlier))
    group.ctx.check(lib().cvb_gba_group(group.h, C.byref(flat.s), C.byref(g), int(bool(peer_path)), C.byref(res.r),
                                        removed.ctypes.data))
    out = res.as_dict()
    out["obs_removed"] = removed[:flat.n_obs].astype(bool)
    return out


def _quat_to_rot(q):
    """[qx,qy,qz,qw] (Hamilton, Eigen coefficient order, keyframe_base.cpp:490-499) → R, vectorised."""
    q = np.asarray(q, np.float64)
    x, y, z, w = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = np.empty((len(q), 3, 3))
    R[:, 0, 0] = 1 - 2 * (y * y + z * z); R[:, 0, 1] = 2 * (x * y - z * w); R[:, 0, 2] = 2 * (x * z + y * w)
    R[:, 1, 0] = 2 * (x * y + z * w); R[:, 1, 1] = 1 - 2 * (x * x + z * z); R[:, 1, 2] = 2 * (y * z - x * w)
    R[:, 2, 0] = 2 * (x * z - y * w); R[:, 2, 1] = 2 * (y * z + x * w); R[:, 2, 2] = 1 - 2 * (x * x + y * y)
    return R


def _rot_to_quat(R):
    t = lambda v: np.sqrt(np.maximum(0.0, v)) / 2
    w = t(1 + R[:, 0, 0] + R[:, 1, 1] + R[:, 2, 2])
    x = np.copysign(t(1 + R[:, 0, 0] - R[:, 1, 1] - R[:, 2, 2]), R[:, 2, 1] - R[:, 1, 2])
    y = np.copysign(t(1 - R[:, 0, 0] + R[:, 1, 1] - R[:, 2, 2]), R[:, 0, 2] - R[:, 2, 0])
    z = np.copysign(t(1 - R[:, 0, 0] - R[:, 1, 1] + R[:, 2, 2]), R[:, 1, 0] - R[:, 0, 1])
    q = np.stack([x, y, z, w], 1)
    return q / np.linalg.norm(q, axis=1, keepdims=True)


def pgo_edges(p: dict, vio_pose, wt=(10.0, 1.0, 10.0, 2.0, 3.0), covins_mode=True, use_robust=True, use_nbr=True):
    """Edge list of Optimization::PoseGraphOptimization (optimization_be.cpp:886-1021), the host-side problem
    construction (the C++ shim does the same on the reference containers): loop edges first (sqrt_info = the keyframe
    weights diag(wt_kf_r, wt_kf_t)*wt_kf_n1 in COVINS mode :896-898, else chol(cov^-1)^T :922-923; Cauchy when
    use_robust), then one successor edge per keyframe with a successor of the same agent (:947-972), then up to five
    predecessor edges per keyframe with weights /1, /n23, /n23, /n45, /n45 (:976-1021), measured on the VIO poses and
    de-duplicated on the ordered (kf, other) pair.  Defaults config_backend.yaml:126-130."""
    wt_r, wt_t, n1, n23, n45 = wt
    S1 = np.diag([wt_r] * 3 + [wt_t] * 3) * n1
    vio_pose = np.asarray(vio_pose, np.float64)
    Rv = _quat_to_rot(vio_pose[:, :4]); tv = vio_pose[:, 4:]
    K = int(p["K"])
    agent, kid = np.asarray(p["agent_of"]), np.asarray(p["kf_id"])
    nl = len(p["loop_i"])
    I = [np.asarray(p["loop_i"], np.int64)]; J = [np.asarray(p["loop_j"], np.int64)]
    kind = [np.full(nl, -1)]                                   # -1 loop, 1..5 = which neighbour
    idx = np.arange(K)
    succ = idx[:-1][agent[1:] == agent[:-1]] if K > 1 else idx[:0]
    I.append(succ); J.append(succ + 1); kind.append(np.full(len(succ), 1))
    if use_nbr:
        ii = np.repeat(idx, 5); kk = np.tile(np.arange(1, 6), K)
        ok = kid[ii] - kk > 0
        ii, kk = ii[ok], kk[ok]
        I.append(ii); J.append(ii - kk); kind.append(kk)
    I = np.concatenate(I); J = np.concatenate(J); kind = np.concatenate(kind)
    # de-duplicate non-loop edges on the ordered pair, first occurrence wins (std::set semantics of the reference)
    key = I * (K + 1) + J
    keep = np.ones(len(I), bool)
    nz = np.flatnonzero(kind > 0)
    _, first = np.unique(key[nz], return_index=True)
    mask = np.zeros(len(nz), bool); mask[first] = True
    keep[nz] = mask
    I, J, kind = I[keep], J[keep], kind[keep]
    Rrel = np.einsum("nji,njk->nik", Rv[I], Rv[J])
    Q = _rot_to_quat(Rrel); T = np.einsum("nji,nj->ni", Rv[I], tv[J] - tv[I])
    SI = np.empty((len(I), 6, 6))
    SI[:] = S1
    SI[(kind == 2) | (kind == 3)] = S1 / n23
    SI[(kind == 4) | (kind == 5)] = S1 / n45
    loops = kind < 0
    if nl:
        Q[:nl] = np.asarray(p["loop_q"], np.float64); T[:nl] = np.asarray(p["loop_t"], np.float64)
        if not covins_mode:
            SI[:nl] = np.stack([np.linalg.cholesky(np.linalg.inv(c)).T for c in np.asarray(p["loop_cov"])])
    return dict(i=I.astype(np.int32), j=J.astype(np.int32), q=Q, t=T, sqrt_info=SI, robust=loops & bool(use_robust))


def pose_graph_optimization(ctx: Context, p: dict, edges: dict, iterations=10, robust_th=0.5):
    """Optimization::PoseGraphOptimization solve: poses only, `edges` = loop + successor + neighbour edges built as in
    optimization_be.cpp:886-1021; pgo_iteration_limit 10, robust_loss_th 0.5 (config_backend.yaml:121,125)."""
    pp = dict(K=p["K"], L=0, pose=p["pose"], pose_const=p["pose_const"], extr=p["extr"], cam_of_kf=p.get("cam_of_kf"))
    flat = _Flat(pp, edges=edges, use_imu=False)
    res = _Res(flat.K, 0)
    o = BaOptions(int(iterations), 1, 0.0, float(robust_th), 0, 1)
    ctx.check(lib().cvb_ba_solve(ctx.handle, C.byref(flat.s), C.byref(o), C.byref(res.r)))
    return res.as_dict()


class PgoProblem(C.Structure):
    _fields_ = [("K", C.c_int32)] + [(n, c_vp) for n in ("T_ws", "T_ws_init", "T_ws_vio", "kf_pred", "kf_succ", "kf_id", "pose_const",
                                                          "velocity")] + \
               [("n_loop", C.c_int32)] + [(n, c_vp) for n in ("loop_i", "loop_j", "loop_q", "loop_t", "loop_cov")] + \
               [("L", C.c_int32)] + [(n, c_vp) for n in ("lm_pos", "lm_ref", "lm_has_obs")]


class PgoOptions(C.Structure):
    _fields_ = [("wt_kf_r", C.c_double), ("wt_kf_t", C.c_double), ("wt_kf_n1", C.c_double), ("wt_kf_n23", C.c_double),
                ("wt_kf_n45", C.c_double), ("use_nbr_kfs", C.c_int32), ("use_robust_loss", C.c_int32), ("robust_loss_th", C.c_double),
                ("iteration_limit", C.c_int32)]


class PgoResult(C.Structure):
    _fields_ = [("T_ws_out", c_vp), ("velocity_out", c_vp), ("lm_out", c_vp), ("lm_erase", c_vp), ("ba", BaResult),
                ("n_edge", C.c_int32), ("bad_loop", C.c_int32)]


def _chain_links(agent_of):
    """predecessor / successor indices of keyframes listed agent by agent in id order (-1 at a chain's ends)"""
    agent = np.asarray(agent_of)
    K = len(agent)
    same = agent[1:] == agent[:-1] if K > 1 else np.zeros(0, bool)
    pred = np.full(K, -1, np.int32); succ = np.full(K, -1, np.int32)
    idx = np.arange(K, dtype=np.int32)
    pred[1:][same] = idx[:-1][same]
    succ[:-1][same] = idx[1:][same]
    return pred, succ


def pgo_map_problem(p: dict, covins_mode=True, T_ws_init=None) -> dict:
    """The map cvb_pgo takes (include/covins_b200.h), from a flat problem (covins_b200.synth_map or mapio.read_map):
    T_ws from p["T_ws"] or else p["pose"]; T_ws_vio from p["T_ws_vio"] or else T_ws; kf_pred / kf_succ from p or else the
    agents' chains; velocity from speedbias; lm_ref / lm_has_obs from p (mapio's id_reference) or else each landmark's first
    observer, as the reference's landmarks are anchored; loop_cov only in COVINS_G mode (covins_mode False)."""
    K = int(p["K"])
    if p.get("T_ws") is not None:
        T_ws = np.ascontiguousarray(p["T_ws"], np.float64).reshape(K, 4, 4)
    else:
        pose = np.asarray(p["pose"], np.float64)
        T_ws = np.tile(np.eye(4), (K, 1, 1))
        T_ws[:, :3, :3] = _quat_to_rot(pose[:, :4]); T_ws[:, :3, 3] = pose[:, 4:]
    T_vio = p.get("T_ws_vio")
    pred, succ = (p["kf_pred"], p["kf_succ"]) if p.get("kf_pred") is not None else _chain_links(p["agent_of"])
    ptr = np.asarray(p.get("lm_obs_ptr", np.zeros(1)), np.int64)
    n_obs = np.diff(ptr)
    if p.get("lm_ref") is not None:
        lm_ref, has = np.asarray(p["lm_ref"]), np.asarray(p["lm_has_obs"])
    else:
        obs_kf = np.asarray(p.get("obs_kf", np.zeros(0)), np.int32)
        has = n_obs > 0
        lm_ref = np.full(len(n_obs), -1, np.int32)
        lm_ref[has] = obs_kf[ptr[:-1][has]]
    sb = p.get("speedbias")
    nl = len(p.get("loop_i", []))
    return dict(T_ws=T_ws, T_ws_init=None if T_ws_init is None else np.asarray(T_ws_init, np.float64).reshape(K, 4, 4),
                T_ws_vio=T_ws if T_vio is None else np.asarray(T_vio, np.float64).reshape(K, 4, 4),
                kf_pred=np.asarray(pred, np.int32), kf_succ=np.asarray(succ, np.int32), kf_id=np.asarray(p["kf_id"], np.int32),
                pose_const=np.asarray(p["pose_const"], np.uint8), velocity=None if sb is None else np.asarray(sb, np.float64)[:, :3],
                loop_i=np.asarray(p.get("loop_i", np.zeros(0)), np.int32), loop_j=np.asarray(p.get("loop_j", np.zeros(0)), np.int32),
                loop_q=np.asarray(p.get("loop_q", np.zeros((0, 4))), np.float64).reshape(nl, 4),
                loop_t=np.asarray(p.get("loop_t", np.zeros((0, 3))), np.float64).reshape(nl, 3),
                loop_cov=None if covins_mode else np.asarray(p["loop_cov"], np.float64).reshape(nl, 6, 6),
                lm_pos=np.asarray(p.get("lm", np.zeros((0, 3))), np.float64).reshape(-1, 3),
                lm_ref=np.asarray(lm_ref, np.int32), lm_has_obs=np.asarray(has, np.uint8))


def pose_graph_optimization_map(ctx: Context, p: dict, wt=(10.0, 1.0, 10.0, 2.0, 3.0), covins_mode=True, use_robust=True,
                                use_nbr=True, iterations=10, robust_th=0.5, T_ws_init=None, cap=64):
    """Optimization::PoseGraphOptimization with its write-back (optimization_be.cpp:833-1086) in one cvb_pgo call: the edges of
    the keyframe chain, the solve and what the server writes into its map afterwards.  `p` is a flat problem or a dict of
    pgo_map_problem (it has T_ws).  Returns T_ws [K,4,4] (what SetPoseTws receives), pose [K,7] (the solved pose7),
    velocity [K,3] (None without velocities), lm [L,3] (re-anchored; others keep their bits), lm_erase [L] bool, the
    solver's cost history / steps / iterations / termination, and n_edge."""
    pr = p if "lm_pos" in p else pgo_map_problem(p, covins_mode, T_ws_init)
    K, L, nl = len(pr["kf_id"]), len(pr["lm_pos"]), len(pr["loop_i"])
    a = {k: (None if v is None else np.ascontiguousarray(v)) for k, v in pr.items()}
    s = PgoProblem()
    s.K, s.n_loop, s.L = K, nl, L
    for name, _ in PgoProblem._fields_:
        if name not in ("K", "n_loop", "L"):
            v = a.get(name)
            setattr(s, name, v.ctypes.data if v is not None and v.size else None)
    o = PgoOptions(*[float(w) for w in wt], int(use_nbr), int(use_robust), float(robust_th), int(iterations))
    T_out = np.zeros((K, 4, 4)); vel = np.zeros((K, 3)); lm = np.zeros((max(L, 1), 3)); erase = np.zeros(max(L, 1), np.uint8)
    res = _Res(K, 0, cap)
    r = PgoResult()
    r.T_ws_out, r.velocity_out, r.lm_out, r.lm_erase = T_out.ctypes.data, vel.ctypes.data, lm.ctypes.data, erase.ctypes.data
    r.ba = res.r
    r.ba.speedbias = r.ba.lm = r.ba.lm_owner = None
    ctx.check(lib().cvb_pgo(ctx.handle, C.byref(s), C.byref(o), C.byref(r)))
    res.r = r.ba
    out = res.as_dict()
    for k in ("speedbias", "lm", "lm_owner"):
        out.pop(k)
    out.update(T_ws=T_out, velocity=vel if pr.get("velocity") is not None else None, lm=lm[:L], lm_erase=erase[:L].astype(bool),
               n_edge=int(r.n_edge))
    return out


def solve(ctx: Context, p: dict, max_iterations: int, visual_only=False, cauchy_reproj=1.0, cauchy_edge=1.0, edges=None,
          obs_skip=None):
    """one ceres::Solve on the flat problem (single GPU)."""
    s = BaSolver(ctx, p, visual_only, cauchy_reproj, cauchy_edge, edges, obs_skip)
    s.iterate(max_iterations)
    out = s.result()
    s.close()
    return out


def dense_cholesky_solve(ctx: Context, A, b):
    A = np.ascontiguousarray(A, np.float64); b = np.ascontiguousarray(b, np.float64)
    x = np.zeros_like(b); ms = C.c_double()
    ctx.check(lib().cvb_dense_cholesky_solve(ctx.handle, A.ctypes.data, len(b), b.ctypes.data, x.ctypes.data, C.byref(ms)))
    return x, ms.value


class RelPoseProblem(C.Structure):
    _fields_ = [("n", C.c_int32)] + [(k, c_vp) for k in ("pA_c", "pB_c", "kpA", "kpB", "sigmaA", "sigmaB")] + \
               [("intrA", C.c_double * 4), ("distA", C.c_double * 4), ("intrB", C.c_double * 4), ("distB", C.c_double * 4),
                ("cam_model_A", C.c_int32), ("dist_model_A", C.c_int32), ("cam_model_B", C.c_int32), ("dist_model_B", C.c_int32),
                ("xiA", C.c_double), ("xiB", C.c_double), ("T12", C.c_double * 7)]


def optimize_relative_pose(ctx: Context, T12, pA_c, pB_c, kpA, kpB, sigmaA, sigmaB, camA: dict, camB: dict, th_outlier_align=1.3):
    """Optimization::OptimizeRelativePose (optimization_be.cpp:620-831) on flattened residual pairs: → dict(T12 [7], removed [n]
    bool (by residual index), n_inliers (the reference's return value), iterations (2), cost (history of both solves)).
    cam*: dict(intr[4], dist[4], cam_model=0, dist_model=0, xi=0)."""
    a = [np.ascontiguousarray(pA_c, np.float64).reshape(-1, 3), np.ascontiguousarray(pB_c, np.float64).reshape(-1, 3),
         np.ascontiguousarray(kpA, np.float32).reshape(-1, 2), np.ascontiguousarray(kpB, np.float32).reshape(-1, 2),
         np.ascontiguousarray(sigmaA, np.float64), np.ascontiguousarray(sigmaB, np.float64)]
    n = len(a[0])
    s = RelPoseProblem()
    s.n = n
    for k, v in zip(("pA_c", "pB_c", "kpA", "kpB", "sigmaA", "sigmaB"), a):
        setattr(s, k, v.ctypes.data)
    for tag, cam in (("A", camA), ("B", camB)):
        getattr(s, "intr" + tag)[:] = [float(x) for x in np.asarray(cam["intr"]).reshape(4)]
        getattr(s, "dist" + tag)[:] = [float(x) for x in np.asarray(cam["dist"]).reshape(4)]
        setattr(s, "cam_model_" + tag, int(cam.get("cam_model", 0))); setattr(s, "dist_model_" + tag, int(cam.get("dist_model", 0)))
        setattr(s, "xi" + tag, float(cam.get("xi", 0.0)))
    s.T12[:] = [float(x) for x in np.asarray(T12).reshape(7)]
    out = np.zeros(7); removed = np.zeros(max(n, 1), np.uint8); ninl = C.c_int32(0); info = np.zeros(19)
    ctx.check(lib().cvb_optimize_relative_pose(ctx.handle, C.byref(s), float(th_outlier_align), out.ctypes.data, removed.ctypes.data,
                                               C.byref(ninl), info.ctypes.data))
    nh = int(info[2])
    return dict(T12=out, removed=removed[:n].astype(bool), n_inliers=int(ninl.value), iterations=(int(info[0]), int(info[1])),
                cost=info[3:3 + min(nh, 16)].copy())
