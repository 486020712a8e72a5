"""Each trust-region iteration of the bundle adjustment (covins_b200/csrc/ba_engine.cu), checked in lockstep against the
oracle's Jacobian in extended precision through the public diagnostic cvb_ba_debug_vector (BaSolver.debug_vector).

The end-to-end suites (test_gpu_ba.py, test_ba_map_shapes.py, test_ba_restart_sharded.py) compare states after several
iterations.  They cannot see a subtly wrong normal matrix: the fixed point depends only on the gradient, and near the
optimum a step error of e changes the next cost at second order.  Here the engine is driven one iteration at a time.
Before each iteration the oracle (oracle/ba_oracle.py) evaluates r and its autograd Jacobian J at the GPU's own state,
J is scaled by the oracle's Jacobi scale at x0 (Js), and every vector the iteration produced is held against longdouble
algebra on Js and r:

  0 scale   1 / (1 + |J(x0)_j|) on active columns, 0 on constant poses          relative, C_SCALE
  1 colsq   column sums of squares of Js (no cancellation)                       relative, C_COLSQ
  2 diag    sqrt(clip(colsq, 1e-6, 1e32)) of the returned colsq, 1 if inactive   bitwise
  3 g       Js^T r                                         |err| <= gamma(C_G) |Js|^T |r|
  4 grad    g / diag of the returned vectors                                     bitwise
  8 gs      g_c - W Hll_mu^-1 g_l, Hll_mu = Hll + mu diag_l^2 (camera part)     |err| <= gamma(C_GS) (|Jc|^T|r| + |W| K |Jl|^T|r|)
  7 x_c     residual of the reduced system S x_c = gs with the reference S and the GPU's gs (Demmel's componentwise
            bound for Cholesky, independent of cond(S)):  |S x_c - gs| <= gamma(C_XC) (d (d^T |x_c|) + |gs| + A |x_c|),
            d = sqrt(diag S), A = |Jc|^T|Jc| + |W| |Hll_mu^-1| |W|^T + |Y| |Hll_mu| |Y|^T, Y = W Hll_mu^-1 (the
            rounding of the assembly, the inverse taken as the exact inverse of a Hll_mu perturbed by O(u) |Hll_mu|)
  7 x_l     Hll_mu^-1 (g_l - W_l^T x_c) from the GPU's x_c (back-substitution alone)
                                                           |err| <= gamma(C_XL) K (|Jl|^T|r| + |W|^T |x_c|)
  5 gn      -x * diag                                                            bitwise
  6 step    step * diag on the dogleg path: = gn when |gn| <= radius; otherwise (ca, cb) recomputed with the engine's
            formula from the radius and alpha = |grad|^2 / |Js (grad / diag)|^2 of the reference, so alpha checks the
            J*v kernels                                    |err| <= gamma(C_STEP) (|ca| |grad| + |cb| |gn|)

K is the block-diagonal matrix of kappa_l |Hll_mu,l^-1| (kappa_l the 1-norm condition number of the damped 3x3 block): the
kernels apply an explicit inverse, so a landmark's terms in gs and x_l carry its own conditioning, and nothing else in a
bound depends on the conditioning of the system.  u = 2^-53 and gamma(c) = c u / (1 - c u).

Per iteration also: the step status against the reference gain ratio rho (model change from Js, candidate cost from the
oracle at Plus(state, step * scale)); an accepted step's new state against the oracle's Plus (C_PLUS ulps of the
magnitudes), constant poses bitwise unchanged; a rejected step leaves the state bitwise unchanged and the next iteration
reuses vectors 0-5, 7 and 8 bitwise; every cost-history entry against the oracle's cost at the same state (1e-12
relative, test_ba_map_shapes.COST_RTOL); mu follows the step statuses from 1e-8 (x10 after an invalid step,
max(1e-8, mu / 5) after an accepted one) and the radius the gain ratios from 1e4, which the step check relies on.

A missing damping term mu diag^2 (mu >= 1e-8) moves the residual of the reduced system by mu diag_i^2 |x_i|.  Every
solve asserts that this exceeds the x_c residual bound by DAMPING_VISIBLE in at least one row, and prints the margin
("damping/bound"), so the residual check provably resolves the damping in each case.  The bounds are calibrated on an H100: each constant is
at least 100x the worst value measured over all cases (listed beside it), and `pytest -s` prints every check's worst
err/bound per case.  The whole file runs in about 45 s on one H100 (the oracle's autograd Jacobians dominate).

Cases: tiny (visual-only and visual-inertial, Cauchy(1) loop edges), a clean 80-keyframe visual-inertial map (1200
camera columns, 10 tiles of S), the map shapes of test_ba_map_shapes.py (per-agent cameras, broken IMU chains with
zero speed-bias columns that take the diag clip, a constant agent, 2-observation landmarks and obs_skip, 126 and 258
pose columns around the 128-column tile boundary), pose graphs with Cauchy(0.5) on the robust edges (no landmark
part), and two maps built to leave the Gauss-Newton branch: a pose graph with scaled information (Cauchy point and
dogleg with alpha from the between-edges alone) and a visual-inertial map far from its optimum without the
reprojection loss (rejected steps and the reuse path).  Each case asserts the branches and column kinds it exists for."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

import test_ba_map_shapes as shapes
from covins_b200 import optimization as O
from covins_b200 import synth_map as sm
from oracle import ba_oracle as bo
from test_ba_map_shapes import COST_RTOL
from test_cholesky_kernels import LD, _bound, _same_bits, _within, gamma

# ------------------------------------------------------------------------------------------------ bounds
# gamma(C) per check.  Measured worst err / (u * magnitude) over all cases on an H100 SXM (700 W), and the headroom of C:
C_SCALE = 1e5              # 525    (190x)  the analytic Jacobian at x0 vs autograd, through 1 / (1 + |J_j|)
C_COLSQ = 5e6              # 4.8e4  (105x)  analytic vs autograd entries that cancel (rotation columns of long arms)
C_G = 5e3                  # 43     (118x)
C_GS = 500                 # 3.1    (163x)
C_XC = 3.2e4               # 317    (101x)  gamma(C_XC) = 3.6e-12; see DAMPING_VISIBLE
C_XL = 200                 # 1.2    (172x)
C_STEP = 5e3               # 34     (146x)  the dogleg branch; Gauss-Newton steps are exact
C_PLUS = 200               # 1.1    (175x)
REL_RADIUS = 1e-13         # 3e-16  (330x)  the radius the test tracks vs the norm of step * diag
# The damping term mu diag_i^2 x_i of the reduced system must stand above the x_c residual bound in some row of every
# solve, or the residual check could not tell a missing or wrong damping from rounding.  Smallest measured on an H100
# (max over active rows of mu diag_i^2 |x_i| / bound_i, over all solves of a case): 9.3 (pgo_threshold), 10 (the
# 126-column map), 12-60 elsewhere; with C_XC's 100x headroom the term is ~1e3 times the largest rounding seen.
DAMPING_VISIBLE = 4.0
RHO_AMBIGUOUS = 1e-6       # a gain ratio this close (relative) to 0.25 or 0.75 may round either way in the engine

MIN_MU, MU_INC = 1e-8, 10.0
MIN_DIAG, MAX_DIAG = 1e-6, 1e32
RADIUS0 = 1e4


# ------------------------------------------------------------------------------------------------ cases
def _pgo(p, edges):
    pp = dict(K=p["K"], L=0, pose=p["pose"], pose_const=p["pose_const"], extr=p["extr"], cam_of_kf=p.get("cam_of_kf"))
    return pp, dict(visual_only=True, cauchy_reproj=0.0, cauchy_edge=0.5, edges=edges), \
        dict(visual_only=True, edges=edges, cauchy_edges=0.5)


def _gba(p, visual_only, obs_skip=None):
    use = None if obs_skip is None else ~obs_skip.astype(bool)
    return p, dict(visual_only=visual_only, obs_skip=obs_skip), dict(visual_only=visual_only, loop_loss=1.0, use_obs=use)


def case_tiny(visual_only):
    p = sm.make_config("tiny")
    assert len(p["loop_i"]) > 0           # loop edges, under Cauchy(1) as in round 2 of GlobalBundleAdjustment
    return _gba(p, visual_only)


def case_small():
    # the C1-like map of test_gpu_ba.py without gross outliers: 80 keyframes x 15 = 1200 camera columns, 10 tiles of S
    p = sm.make_map(seed=21, n_agents=2, kf_per_agent=40, n_lm=2000, outlier_frac=0.0)
    assert p["K"] * 15 == 1200 and len(p["loop_i"]) > 0
    return _gba(p, False)


def case_landmark_extremes():
    p, skip, _ = shapes.landmark_extremes()
    return _gba(p, False, skip)


def case_pgo():
    p = sm.make_map(seed=5, n_agents=3, kf_per_agent=60, n_lm=10, drift_trans=0.01, drift_yaw_deg=0.1)
    return _pgo(p, bo.pgo_edges(p, p["pose"]))


def case_pgo_threshold():
    return _pgo(*shapes.pgo_threshold())


def case_pgo_far():
    """The pose graph of case_pgo drifted 20x further, every information matrix scaled by 1e3 and no robust edge: the
    minimiser is unchanged and the Gauss-Newton step in the scaled space grows 1e3-fold, longer than the trust radius.
    The first steps take the Cauchy point and the interpolated dogleg, whose alpha comes from J*v over the between-edges
    alone."""
    p = sm.make_map(seed=5, n_agents=3, kf_per_agent=60, n_lm=10, drift_trans=0.05, drift_yaw_deg=1.0)
    e = bo.pgo_edges(p, p["pose"])
    e["sqrt_info"] = e["sqrt_info"] * 1e3
    e["robust"] = np.zeros_like(e["robust"])
    return _pgo(p, e)


def case_vi_far():
    """A tiny-sized visual-inertial map with 1 m landmark noise, 25x the drift and no reprojection loss: steps longer than
    the radius (Cauchy point, dogleg), and a linearisation poor enough that some are rejected (the reuse path)."""
    p = sm.make_map(seed=3, n_agents=2, kf_per_agent=12, n_lm=300, lm_noise=1.0, drift_trans=0.05, drift_yaw_deg=0.5)
    assert len(p["loop_i"]) > 0 and len(p["imu_i"]) > 0
    return p, dict(visual_only=False, cauchy_reproj=0.0), dict(visual_only=False, cauchy_reproj=None, loop_loss=1.0)


CASES = {
    "tiny_vo": (lambda: case_tiny(True), 6, {"loops"}),
    "tiny_vi": (lambda: case_tiny(False), 6, {"loops"}),
    "small": (case_small, 5, {"loops"}),
    "cams_mixed": (lambda: _gba(shapes.cams_mixed(), False), 5, set()),
    "imu_split": (lambda: _gba(shapes.imu_split(), False), 5, {"clip"}),
    "const_agent": (lambda: _gba(shapes.const_agent(), False), 5, {"inactive"}),
    "landmark_extremes": (case_landmark_extremes, 5, {"two_obs"}),
    "vo_tile_edges_21": (lambda: _gba(shapes.vo_tile_edges(21), True), 5, set()),
    "vo_tile_edges_43": (lambda: _gba(shapes.vo_tile_edges(43), True), 5, set()),
    "pgo": (case_pgo, 6, {"no_landmarks"}),
    "pgo_threshold": (case_pgo_threshold, 6, {"no_landmarks"}),
    "pgo_far": (case_pgo_far, 4, {"no_landmarks", "cauchy", "dogleg", "accepted"}),
    "vi_far": (case_vi_far, 8, {"cauchy", "dogleg", "accepted", "rejected"}),
}
NCAM = {"small": 1200, "vo_tile_edges_21": 126, "vo_tile_edges_43": 258}


# ------------------------------------------------------------------------------------------------ longdouble algebra
def _ld(a):
    return np.asarray(a, LD)


def _inv3(H):
    """inverse of symmetric 3x3 blocks [n,3,3] by the adjugate, in the blocks' precision"""
    a, b, c, d, e, f = H[:, 0, 0], H[:, 0, 1], H[:, 0, 2], H[:, 1, 1], H[:, 1, 2], H[:, 2, 2]
    A, B, C = d * f - e * e, c * e - b * f, b * e - c * d
    det = a * A + b * B + c * C
    out = np.empty_like(H)
    out[:, 0, 0] = A; out[:, 0, 1] = out[:, 1, 0] = B; out[:, 0, 2] = out[:, 2, 0] = C
    out[:, 1, 1] = a * f - c * c; out[:, 1, 2] = out[:, 2, 1] = b * c - a * e; out[:, 2, 2] = a * d - b * b
    return out / det[:, None, None]


def _blockdiag(B):
    n = len(B)
    i = np.arange(3 * n).reshape(n, 3)
    rows = np.repeat(i, 3, axis=1).reshape(-1)
    cols = np.tile(i, (1, 3)).reshape(-1)
    return sp.csr_matrix((B.reshape(-1), (rows, cols)), shape=(3 * n, 3 * n), dtype=LD)


def _residual_rounding(prob, state, info, m):
    """magnitudes each residual is rounded at, where it cancels: a reprojection residual is a difference of pixels (the
    observed |uv| / sigma), a between-edge one a difference of rotations (2) and translations (|t2 - t1| + |t_m|) under
    sqrt_info, an IMU one differences of positions, velocities and biases under its sqrt_info.  A between-edge measured
    on the initial state has r = 0 up to this rounding, and the IMU residuals of a converging solve approach it."""
    out = np.zeros(m, LD)
    if "reproj" in info:
        r0, n, k = info["reproj"]
        out[r0:r0 + n * k] = (np.abs(prob.o_uv.numpy()) / prob.o_sigma.numpy()[:, None]).reshape(-1)
    if "edges" in info:
        r0, n, k = info["edges"]
        e, t = prob.edges, state[0].numpy()[:, 4:]
        T = np.linalg.norm(t[e["j"]] - t[e["i"]], axis=1) + np.linalg.norm(e["t"].numpy(), axis=1)
        mag = np.concatenate([np.full((n, 3), 2.0), np.repeat(T[:, None], 3, 1)], 1)
        out[r0:r0 + n * k] = np.einsum("nij,nj->ni", np.abs(e["S"].numpy()), mag).reshape(-1)
    if "imu" in info:
        r0, n, k = info["imu"]
        pre, pose, sb = prob.imu, state[0].numpy(), state[1].numpy()
        i, j = prob.imu_i, prob.imu_j
        T, g = pre["dt_sum"].numpy(), abs(prob.imu["g"])
        nrm = lambda a: np.linalg.norm(a, axis=-1)                                   # noqa: E731
        mp = nrm(pre["alpha"].numpy()) + 0.5 * g * T * T + nrm(pose[i, 4:]) + nrm(pose[j, 4:]) + T * nrm(sb[i, :3])
        mv = nrm(pre["beta"].numpy()) + g * T + nrm(sb[i, :3]) + nrm(sb[j, :3])
        mba, mbg = nrm(sb[i, 3:6]) + nrm(sb[j, 3:6]), nrm(sb[i, 6:]) + nrm(sb[j, 6:])
        mag = np.repeat(np.stack([mp, np.full(n, 2.0), mv, mba, mbg], 1), 3, axis=1)
        out[r0:r0 + n * k] = np.einsum("nij,nj->ni", np.abs(pre["sqrt_info"].numpy()), mag).reshape(-1)
    return out


class Linearisation:
    """Js, r and the damped Schur pieces at one state, in longdouble"""

    def __init__(self, prob, state, scale_ld):
        self.cost, r, J, info = prob.evaluate(*state)
        nc = prob.ncam
        self.r = _ld(r)
        absr = np.abs(self.r) + _residual_rounding(prob, state, info, len(r))
        self.Js = (J.astype(LD) @ sp.diags(scale_ld)).tocsr()
        self.absJ = abs(self.Js)
        self.colsq = np.asarray(self.Js.multiply(self.Js).sum(0), LD).reshape(-1)
        self.g = self.Js.T @ self.r
        self.absg = self.absJ.T @ absr                              # |Js|^T |r|
        self.nc, self.nl = nc, (prob.n - nc) // 3
        Jc, Jl = self.Js[:, :nc].tocsc(), self.Js[:, nc:].tocsc()
        aJc, aJl = abs(Jc), abs(Jl)
        self.Hcc = (Jc.T @ Jc).toarray()
        self.absHcc = (aJc.T @ aJc)
        if self.nl:
            Hl = (Jl.T @ Jl).tocsr()
            dg = [Hl.diagonal(k) for k in (-2, -1, 0, 1, 2)]
            B = np.empty((self.nl, 3, 3), LD)
            for a in range(3):
                for b in range(3):
                    B[:, a, b] = dg[b - a + 2][3 * np.arange(self.nl) + min(a, b)]
            self.Hll = B
            self.W, self.absW = (Jc.T @ Jl).tocsr(), (aJc.T @ aJl).tocsr()

    def damped(self, mu, active):
        """Hll_mu^-1, K, gs, S and its assembly magnitude for damping mu"""
        mu = LD(mu)
        dsq = np.clip(self.colsq, MIN_DIAG, MAX_DIAG)               # diag^2
        nc = self.nc
        d = {}
        gc, gl = self.g[:nc], self.g[nc:]
        S = self.Hcc.copy()
        A = self.absHcc.toarray()
        mag_gs = self.absg[:nc].copy()
        if self.nl:
            Hmu = self.Hll.copy()
            for a in range(3):
                Hmu[:, a, a] += mu * dsq[nc:].reshape(-1, 3)[:, a]
            Hinv = _inv3(Hmu)
            kappa = np.abs(Hmu).sum(1).max(1) * np.abs(Hinv).sum(1).max(1)
            Hi, K = _blockdiag(Hinv), _blockdiag(kappa[:, None, None] * np.abs(Hinv))
            S -= (self.W @ Hi @ self.W.T).toarray()
            # rounding of W Hll_mu^-1 W^T: the products (|W| |Hll_mu^-1| |W|^T), and the inverse as the exact inverse of
            # Hll_mu perturbed by O(u) |Hll_mu| (|Y| |Hll_mu| |Y|^T, Y = W Hll_mu^-1).  A landmark's kappa does not enter:
            # its weak direction is the one W barely sees.
            Y = self.W @ Hi
            A += (self.absW @ _blockdiag(np.abs(Hinv)) @ self.absW.T + abs(Y) @ _blockdiag(np.abs(Hmu)) @ abs(Y).T).toarray()
            d.update(gs=gc - self.W @ (Hi @ gl), Hi=Hi, K=K, kappa=kappa)
            mag_gs += self.absW @ (K @ self.absg[nc:])
        else:
            d["gs"] = gc.copy()
        idx = np.arange(nc)
        S[idx, idx] += np.where(active[:nc], mu * dsq[:nc], 0)
        S[idx[~active[:nc]], idx[~active[:nc]]] = 1
        d.update(S=S, A=A, mag_gs=mag_gs)
        return d


class Checks:
    """err/bound pairs per check, over all iterations of a case; finish() prints every check's worst and asserts"""

    def __init__(self, case):
        self.case, self.d, self.bits = case, {}, []

    def within(self, tag, err, bound):
        e, b = self.d.setdefault(tag, ([], []))
        e.append(np.asarray(err, LD).ravel()); b.append(np.asarray(bound, LD).ravel())

    def same_bits(self, tag, a, b):
        try:
            _same_bits(tag, a, b)
        except AssertionError as e:
            self.bits.append(f"[{self.case}] {e}")

    def same_values(self, tag, a, b):
        d = ~(np.asarray(a) == np.asarray(b))
        if d.any():
            self.bits.append(f"[{self.case}] {tag}: {int(d.sum())} of {d.size} values differ, first at {int(np.argmax(d))}")

    def finish(self):
        fails = list(self.bits)
        for tag, (e, b) in sorted(self.d.items()):
            try:
                _within(f"[{self.case}] {tag}", np.concatenate(e), np.concatenate(b))
            except AssertionError as ex:
                fails.append(str(ex))
        assert not fails, "\n".join(fails)


def _state(res):
    return (torch.tensor(res["pose"]), torch.tensor(res["speedbias"]), torch.tensor(res["lm"]))


def _vec(s, which):
    c, l = s.debug_vector(which)
    return np.concatenate([c, l])


def _dogleg(gn_norm, g_norm, g_dot_gn, alpha, radius):
    """(branch, ca, cb) of the engine (ba_engine.cu, engine_iterate) in longdouble"""
    if gn_norm <= radius:
        return "gn", LD(0), LD(1)
    if g_norm * alpha >= radius:
        return "cauchy", -(radius / g_norm), LD(0)
    b_dot_a = -alpha * g_dot_gn
    a2 = (alpha * g_norm) ** 2
    bma2 = a2 - 2 * b_dot_a + gn_norm * gn_norm
    c = b_dot_a - a2
    dd = np.sqrt(c * c + bma2 * (radius * radius - a2))
    beta = (dd - c) / bma2 if c <= 0 else (radius * radius - a2) / (dd + c)
    return "dogleg", -alpha * (1 - beta), beta


def run_case(ctx, name):
    build, n_iter, expect = CASES[name]
    p, gkw, okw = build()
    prob = bo.Problem(p, **okw)
    nc = prob.ncam
    active = prob.active
    chk = Checks(name)
    seen = set()
    s = O.BaSolver(ctx, p, **gkw)
    try:
        res = s.result()
        state = _state(res)
        # the oracle's Jacobi scale at x0 (from the GPU's start state, which is the map's)
        ref_cost0, _, J0, _ = prob.evaluate(*state)
        cost0 = res["cost"][0]
        cs0 = np.asarray(J0.astype(LD).multiply(J0.astype(LD)).sum(0), LD).reshape(-1)
        scale_ref = np.where(active, 1 / (1 + np.sqrt(cs0)), LD(0))
        scale = _vec(s, 0)
        assert len(scale) == prob.n
        chk.within("0 scale", abs(scale - scale_ref), _bound(gamma(C_SCALE), scale_ref, 8))
        chk.same_bits("0 scale inactive", scale[~active], np.zeros((~active).sum()))
        if (~active).any():
            seen.add("inactive")
        if nc == prob.n:
            seen.add("no_landmarks")
        # landmark parts of colsq and g are rewritten when a step is accepted (the next linearisation): read them at
        # the state they belong to
        lm_fresh = (_vec(s, 1)[nc:], _vec(s, 3)[nc:])
        mu, radius = MIN_MU, RADIUS0          # radius None: a gain ratio at a threshold left the engine's unknown
        damp_vis = []
        lin = dmp = prev = None
        for it in range(n_iter):
            s.iterate(1)
            res = s.result()
            done = res["termination"] != "NO_CONVERGENCE"
            status = res["steps"][it] if it < len(res["steps"]) else "converged"
            v = {w: _vec(s, w) for w in range(9)}
            reuse = prev is not None and prev["status"] == "rejected"
            cur = dict(v)                            # vectors 1 and 3 with the landmark part this iteration used
            cur[1], cur[3] = np.concatenate([v[1][:nc], lm_fresh[0]]), np.concatenate([v[3][:nc], lm_fresh[1]])
            if lin is None or prev["status"] == "accepted":
                lin = Linearisation(prob, state, scale_ref)
            if reuse:
                for w in (0, 1, 2, 3, 4, 5, 7, 8):
                    chk.same_bits(f"reuse of vector {w}", cur[w], prev["v"][w])
            else:
                dmp = lin.damped(mu, active)
                colsq, g = cur[1], cur[3]
                # 1 colsq, 2 diag, 3 g, 4 grad
                chk.within("1 colsq", abs(colsq - lin.colsq), _bound(gamma(C_COLSQ), lin.colsq, 64))
                chk.same_bits("1 colsq inactive", colsq[~active], np.zeros((~active).sum()))
                diag = np.where(active, np.sqrt(np.clip(colsq, MIN_DIAG, MAX_DIAG)), 1.0)
                chk.same_bits("2 diag", v[2], diag)
                if np.any(active & (colsq < MIN_DIAG)):
                    seen.add("clip")
                chk.within("3 g", abs(g - lin.g), _bound(gamma(C_G), lin.absg, 64))
                chk.same_bits("4 grad", v[4], np.where(active, g / v[2], 0.0))
                # 8 gs (camera part; the landmark part is unused)
                gs = v[8][:nc]
                chk.within("8 gs", np.where(active[:nc], abs(gs - dmp["gs"]), 0), _bound(gamma(C_GS), dmp["mag_gs"], 64))
                chk.same_bits("8 gs inactive", gs[~active[:nc]], np.zeros((~active[:nc]).sum()))
                # 7 x, camera part: residual of the reduced system with the GPU's right-hand side
                xc = _ld(v[7][:nc])
                S = dmp["S"]
                dS = np.sqrt(np.abs(np.diag(S)))
                axc = np.abs(xc)
                resid = S @ xc - _ld(gs)
                bnd = _bound(gamma(C_XC), dS * (dS @ axc) + np.abs(_ld(gs)) + dmp["A"] @ axc, nc)
                chk.within("7 x_c residual", abs(resid), bnd)
                # how far the damping term of the best-resolved row stands above that bound
                ac = active[:nc] & (bnd > 0)
                damp = LD(mu) * np.clip(lin.colsq[:nc], MIN_DIAG, MAX_DIAG) * axc
                damp_vis.append(float(np.max(damp[ac] / bnd[ac])) if ac.any() else 0.0)
                chk.same_bits("7 x_c inactive", v[7][:nc][~active[:nc]], np.zeros((~active[:nc]).sum()))
                # 7 x, landmark part: back-substitution from the GPU's x_c
                if lin.nl:
                    xl_ref = dmp["Hi"] @ (lin.g[nc:] - lin.W.T @ xc)
                    mag = dmp["K"] @ (lin.absg[nc:] + lin.absW.T @ axc)
                    chk.within("7 x_l", abs(_ld(v[7][nc:]) - xl_ref), _bound(gamma(C_XL), mag, 64))
                    if (np.bincount(prob.o_lm, minlength=prob.L)[prob.lm_in] == 2).any():
                        seen.add("two_obs")
                # 5 gn
                chk.same_bits("5 gn", v[5], np.where(active, -(v[7] * v[2]), 0.0))
            # 6 step on the dogleg path
            grad, gn, diag, step = _ld(v[4]), _ld(v[5]), _ld(v[2]), v[6]
            sd = _ld(step) * diag
            gn_norm, g_norm = np.sqrt(gn @ gn), np.sqrt(grad @ grad)
            jg = lin.Js @ (grad / diag)
            alpha = (grad @ grad) / (jg @ jg)
            gn_step = np.where(active, v[5] / v[2], 0.0)       # gn / diag (0 * grad + 1 * gn is gn up to a zero's sign)
            if radius is None:
                # the engine's radius is not known exactly: the branch from the step, the radius from its length
                r_step = np.sqrt(sd @ sd)
                branch, ca, cb = _dogleg(gn_norm, g_norm, grad @ gn, alpha,
                                         gn_norm if np.all(step == gn_step) else min(r_step, gn_norm * (1 - 1e-12)))
                radius = None if branch == "gn" else float(r_step)
            else:
                branch, ca, cb = _dogleg(gn_norm, g_norm, grad @ gn, alpha, LD(radius))
                if branch != "gn":
                    chk.within("6 |step*diag| = radius", abs(np.sqrt(sd @ sd) - LD(radius)),
                               _bound(LD(REL_RADIUS), LD(radius), 1))
            seen.add(branch)
            if branch == "gn":
                chk.same_values("6 step (Gauss-Newton)", step, gn_step)
            chk.within(f"6 step ({branch})", np.where(active, abs(sd - (ca * grad + cb * gn)), 0),
                       _bound(gamma(C_STEP), abs(ca) * abs(grad) + abs(cb) * abs(gn), 8))
            # status against the reference gain ratio
            jv = lin.Js @ _ld(step)
            mc = -(jv @ (lin.r + jv / 2))
            delta = step * scale
            cand = prob.plus(*state, delta)
            ccost = prob.evaluate(*cand, with_jac=False)[0]
            rho = (LD(lin.cost) - LD(ccost)) / mc if mc > 0 else LD(-np.inf)
            if status == "converged":
                assert done
                break
            # cost history: the oracle's cost at the GPU's state after the iteration
            cost = res["cost"][it + 1]
            ref_cost = prob.evaluate(*_state(res), with_jac=False)[0]
            assert abs(cost - ref_cost) <= COST_RTOL * abs(ref_cost), (name, it, cost, ref_cost)
            if status == "accepted":
                seen.add("accepted")
                assert rho > 1e-3 * (1 - 1e-6), (name, it, float(rho))
                new = _state(res)
                for part, (a, b, o) in enumerate(zip(new, cand, state)):
                    a, b, o = a.numpy(), b.numpy(), o.numpy()
                    mag = np.abs(o) + np.abs(a - o) + (1.0 if part == 0 else 0.0)
                    chk.within("accepted state vs Plus", abs(_ld(a) - _ld(b)), _bound(gamma(C_PLUS), mag, 4))
                c = prob.const
                chk.same_bits("constant poses", new[0].numpy()[c], state[0].numpy()[c])
                if min(abs(rho / LD(0.25) - 1), abs(rho / LD(0.75) - 1)) <= RHO_AMBIGUOUS:
                    radius = None
                elif radius is not None:
                    if rho < 0.25:
                        radius *= 0.5
                    if rho > 0.75:
                        radius = max(radius, 3.0 * float(np.sqrt(sd @ sd)))
                mu = max(MIN_MU, 2.0 * mu / MU_INC)
                state = new
                lm_fresh = (v[1][nc:], v[3][nc:])
            elif status == "rejected":
                seen.add("rejected")
                assert mc > 0 and rho <= 1e-3 * (1 + 1e-6), (name, it, float(mc), float(rho))
                for a, b in zip(_state(res), state):
                    chk.same_bits("rejected: state unchanged", a.numpy(), b.numpy())
                radius = None if radius is None else radius * 0.5
            else:
                assert status == "invalid", status
                seen.add("invalid")
                mu *= MU_INC
            if status != "accepted":
                # no linearisation ran: the landmark parts of colsq and g the engine holds are still the ones used
                chk.same_bits("1 colsq landmark part kept", v[1][nc:], lm_fresh[0])
                chk.same_bits("3 g landmark part kept", v[3][nc:], lm_fresh[1])
            prev = dict(status=status, v=cur)
            if done:
                break
        assert abs(cost0 - ref_cost0) <= COST_RTOL * abs(ref_cost0), (name, cost0, ref_cost0)
        if status == "accepted" and nc < prob.n:
            # the landmark parts of the last linearisation, which no later iteration consumed
            fin = Linearisation(prob, state, scale_ref)
            chk.within("1 colsq", abs(lm_fresh[0] - fin.colsq[nc:]), _bound(gamma(C_COLSQ), fin.colsq[nc:], 64))
            chk.within("3 g", abs(lm_fresh[1] - fin.g[nc:]), _bound(gamma(C_G), fin.absg[nc:], 64))
    finally:
        s.close()
    print(f"[{name}] steps {res['steps']}, reached {sorted(seen)}")
    print(f"[{name}] damping/bound: smallest over {len(damp_vis)} solves of the best row {min(damp_vis):.3g}")
    chk.finish()
    assert min(damp_vis) >= DAMPING_VISIBLE, f"{name}: a damping term mu diag^2 is not resolved by the x_c bound"
    if name in NCAM:
        assert nc == NCAM[name]
    missing = expect - seen - {"loops"}
    assert not missing, f"{name} did not reach {sorted(missing)}"


# ------------------------------------------------------------------------------------------------ tests
def test_dogleg_helper_geometry():
    """_dogleg restates the engine's branch formulas: the interpolated point lies on the sphere of the radius, and the
    branches meet continuously at their boundaries"""
    rng = np.random.default_rng(3)
    for _ in range(100):
        g = _ld(rng.normal(size=20)); gn = _ld(rng.normal(size=20)) * 10
        alpha = LD(rng.uniform(0.01, 0.2))
        gn_norm, g_norm = np.sqrt(gn @ gn), np.sqrt(g @ g)
        radius = LD(rng.uniform(float(alpha * g_norm), float(gn_norm)))
        b, ca, cb = _dogleg(gn_norm, g_norm, g @ gn, alpha, radius)
        assert b == "dogleg"
        d = ca * g + cb * gn
        assert abs(np.sqrt(d @ d) / radius - 1) < 1e-15
        assert 0 <= cb <= 1
    assert _dogleg(LD(1), LD(1), LD(0), LD(1), LD(2))[0] == "gn"
    assert _dogleg(LD(5), LD(4), LD(0), LD(1), LD(2))[0] == "cauchy"


def test_blockdiag_inverse_in_longdouble():
    rng = np.random.default_rng(4)
    M = rng.normal(size=(50, 3, 3))
    H = _ld(M @ M.transpose(0, 2, 1) + 0.1 * np.eye(3))
    Hi = _inv3(H)
    err = np.abs(np.einsum("nij,njk->nik", H, Hi) - np.eye(3)).max()
    assert err < 1e-14
    B = _blockdiag(H)
    assert B.dtype == LD and np.array_equal(B.toarray()[3:6, 3:6], H[1])


@pytest.mark.parametrize("case", sorted(CASES))
def test_case_builders(case):
    """every case map builds and has the structure its checks need (the GPU test asserts what each reaches)"""
    p, gkw, okw = CASES[case][0]()
    prob = bo.Problem(p, **okw)
    if case in NCAM:
        assert prob.ncam == NCAM[case]
    if "no_landmarks" in CASES[case][2]:
        assert prob.n == prob.ncam
    if case == "const_agent":
        assert (~prob.active).sum() == 6 * int(np.sum(p["pose_const"]))


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(CASES))
def test_iteration_algebra(ctx, case):
    run_case(ctx, case)
