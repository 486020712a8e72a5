"""Central relative-pose (5-point) RANSAC from caller-supplied samples (cvb_ransac_central_relative_pose_batch).
CPU: the oracle's 5-point solve against ground truth and against an independent numpy restatement (SVD null space, the ten
cubics from numpy polynomial products, the eigenvectors of an action matrix, SVD decomposition of E), its invalid samples, its
selection against placerec.ransac_select, and its score against the existing relative-pose scoring oracle.  GPU: the C-ABI call
is bit-identical to the oracle, its mask and count equal cvb_score_relative_pose_batch, a noise-free scene gives the true pose and
inlier set, bad arguments are refused, and the C++ wrapper equals the Python path."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
from scipy.signal import convolve

from covins_b200 import placerec as PR
from oracle import geom as og
from oracle import ransac_rel5 as orel

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
S = 5


def _rand_rot(rng):
    q = rng.normal(size=4); q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _problem(rng, n, outlier_frac=0.3, noise=0.0, rotation_only=False, sigma=(1e-6, 1e-5)):
    """one pairing: X1 = R X2 + t, points at 1-30 m in front of camera 1, |t| ~ N(0, 2) per axis (0 for rotation_only), a share of
    the camera-2 bearings replaced by random directions"""
    R, t = _rand_rot(rng), (np.zeros(3) if rotation_only else rng.normal(0, 2, 3))
    d = rng.normal(0, 1, (n, 3)); d[:, 2] = np.abs(d[:, 2]) + 1.0; d /= np.linalg.norm(d, axis=1, keepdims=True)
    X1 = d * rng.uniform(1, 30, n)[:, None]
    X2 = (X1 - t) @ R                                   # R^T (X1 - t)
    f1, f2 = X1.copy(), X2.copy()
    f1 += rng.normal(0, noise, f1.shape) * np.linalg.norm(f1, axis=1, keepdims=True)
    f2 += rng.normal(0, noise, f2.shape) * np.linalg.norm(f2, axis=1, keepdims=True)
    out = rng.random(n) < outlier_frac
    f1 /= np.linalg.norm(f1, axis=1, keepdims=True)
    tn = np.linalg.norm(t)
    for i in np.flatnonzero(out):                       # random directions, at least ~3 degrees off their epipolar plane
        nrm = R.T @ np.cross(t, f1[i]) if tn > 0 else None
        while True:
            f2[i] = rng.normal(0, 1, 3); f2[i] /= np.linalg.norm(f2[i])
            if nrm is None or abs(f2[i] @ nrm) > 0.05 * np.linalg.norm(nrm):
                break
    f2 /= np.linalg.norm(f2, axis=1, keepdims=True)
    return dict(f1=f1, f2=f2, s1=rng.uniform(*sigma, n), s2=rng.uniform(*sigma, n), R=R, t=t / tn if tn > 0 else t, inlier=~out)


def _batch(seed, specs, n_samples, repeat_frac=0.1):
    """specs: (n, outlier share, rotation_only) per problem → (arguments of ransac_central_relative_pose, problems)"""
    rng = np.random.default_rng(seed)
    probs = [_problem(rng, n, of, rotation_only=rot) for n, of, rot in specs]
    samples = np.zeros((len(specs), n_samples, S), np.int32)
    for i, (n, *_) in enumerate(specs):
        if n >= S:
            samples[i] = np.stack([rng.choice(n, S, replace=False) for _ in range(n_samples)])
            rep = rng.random(n_samples) < repeat_frac                          # repeated indices
            samples[i, rep, 4] = samples[i, rep, 1]
        elif n > 0:
            samples[i] = rng.integers(0, n, (n_samples, S))
    cat = lambda k, shape: np.concatenate([p[k] for p in probs]) if probs else np.zeros(shape)
    ptr = np.concatenate([[0], np.cumsum([len(p["f1"]) for p in probs])]).astype(np.int32)
    b = dict(prob_ptr=ptr, f1=cat("f1", (0, 3)), f2=cat("f2", (0, 3)), sigma1=cat("s1", 0), sigma2=cat("s2", 0), samples=samples)
    return b, probs


def _pose_err(M, R, t):
    return max(np.abs(M[:, :3] - R).max(), np.abs(M[:, 3] - t).max())


# ------------------------------------------------------------------------------------------------- 5-point solve (CPU)
def test_rel5_solutions_include_ground_truth():
    rng = np.random.default_rng(0)
    worst = 0.0
    for k in range(2000):
        p = _problem(rng, S, outlier_frac=0.0)
        r = orel.rel5(p["f1"], p["f2"], np.arange(S))
        assert r["valid"] and len(r["z"]) >= 1, k
        errs = np.array([[_pose_err(r["cand"][i, c], p["R"], p["t"]) for c in range(4)] for i in range(len(r["z"]))])
        i, c = np.unravel_index(np.argmin(errs), errs.shape)
        worst = max(worst, errs[i, c])
        assert errs[i, c] < 1e-8, (k, errs[i, c])
        # the true pose is one of the four candidates of its E, and the others are not it
        assert (errs[i] < 1e-8).sum() == 1, k
        assert np.all(np.diff(r["z"]) > 0) and len(r["z"]) % 2 == 0, k   # ascending; complex roots come in pairs
    assert worst < 1e-8


def _poly_mul(a, b):
    """product of polynomials in (x, y, z) as dense coefficient arrays c[i, j, k] of x^i y^j z^k"""
    return convolve(a, b, method="direct")


def _numpy_rel5(f1, f2):
    """independent restatement: null space by SVD, the ten cubics from numpy polynomial products, the eigenvectors of the action
    matrix of x on the basis (x^2, xy, xz, y^2, yz, z^2, x, y, z, 1) refined by Newton steps on the cubics.  → (list of (E, xyz), skip) where skip
    marks a near-double root (0 < |imag| <= 1e-6 relative)"""
    Q = np.stack([np.outer(a, b).ravel() for a, b in zip(f1, f2)])
    basis = np.linalg.svd(Q)[2][5:]                                            # X, Y, Z, W rows
    Ep = []
    for i in range(9):
        c = np.zeros((2, 2, 2)); c[1, 0, 0], c[0, 1, 0], c[0, 0, 1], c[0, 0, 0] = basis[:, i]
        Ep.append(c)
    E = [[Ep[3 * r + c] for c in range(3)] for r in range(3)]
    pad = lambda c: np.pad(c, [(0, 4 - s) for s in c.shape])
    EEt = [[sum(_poly_mul(E[r][m], E[k][m]) for m in range(3)) for k in range(3)] for r in range(3)]
    tr = EEt[0][0] + EEt[1][1] + EEt[2][2]
    eqs = [pad(2 * sum(_poly_mul(EEt[r][k], E[k][c]) for k in range(3)) - _poly_mul(tr, E[r][c])) for r in range(3) for c in range(3)]
    det = sum(pad(_poly_mul(E[0][c], _poly_mul(E[1][(c + 1) % 3], E[2][(c + 2) % 3]) - _poly_mul(E[1][(c + 2) % 3], E[2][(c + 1) % 3])))
              for c in range(3))
    eqs.append(det)
    lead = [(3, 0, 0), (2, 1, 0), (2, 0, 1), (1, 2, 0), (1, 1, 1), (1, 0, 2), (0, 3, 0), (0, 2, 1), (0, 1, 2), (0, 0, 3)]
    rest = [(2, 0, 0), (1, 1, 0), (1, 0, 1), (0, 2, 0), (0, 1, 1), (0, 0, 2), (1, 0, 0), (0, 1, 0), (0, 0, 1), (0, 0, 0)]
    A = np.array([[e[m] for m in lead + rest] for e in eqs])
    C3 = np.array(eqs)
    B = np.linalg.solve(A[:, :10], A[:, 10:])
    M = np.zeros((10, 10))
    M[:6] = -B[:6]                                                             # x * (x^2, xy, xz, y^2, yz, z^2) = leading terms 0..5
    for row, col in ((6, 0), (7, 1), (8, 2), (9, 6)):                          # x * (x, y, z, 1) = (x^2, xy, xz, x)
        M[row, col] = 1.0
    w, V = np.linalg.eig(M)
    sols, skip = [], False
    for k in range(10):
        v = V[:, k] / V[9, k]
        xyz = v[6:9]
        rel = np.abs(xyz.imag).max() / max(np.abs(xyz).max(), 1e-300)
        if rel > 0:
            skip |= rel <= 1e-6
            continue
        xyz = xyz.real
        for _ in range(4):                                                     # Newton (least squares) on the ten cubics
            pw = [np.array([1.0, v, v * v, v ** 3]) for v in xyz]
            dpw = [np.array([0.0, 1.0, 2 * v, 3 * v * v]) for v in xyz]
            F = np.einsum("eijk,i,j,k->e", C3, *pw)
            J = np.stack([np.einsum("eijk,i,j,k->e", C3, *[dpw[a] if a == b else pw[a] for a in range(3)]) for b in range(3)], 1)
            xyz = xyz - np.linalg.lstsq(J, F, rcond=None)[0]
        Em = (xyz[0] * basis[0] + xyz[1] * basis[1] + xyz[2] * basis[2] + basis[3]).reshape(3, 3)
        sols.append(Em * np.sqrt(2.0) / np.linalg.norm(Em))
    return sols, skip


def _numpy_candidates(E):
    U, _, Vt = np.linalg.svd(E)
    if np.linalg.det(U) < 0:
        U = -U
    if np.linalg.det(Vt) < 0:
        Vt = -Vt
    W = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
    t = U[:, 2]
    return [np.c_[R, s * t] for R in (U @ W @ Vt, U @ W.T @ Vt) for s in (1.0, -1.0)]


def _numpy_quality(M, f1, f2):
    R, t = M[:, :3], M[:, 3]
    q = 0.0
    for a, b in zip(f1, f2):
        u = R @ b
        A = np.array([[a @ a, -(a @ u)], [a @ u, -(u @ u)]])
        l0, l1 = np.linalg.solve(A, np.array([t @ a, t @ u]))
        X = (l0 * a + t + l1 * u) / 2
        X2 = R.T @ (X - t)
        q += (1 - a @ X / np.linalg.norm(X)) + (1 - b @ X2 / np.linalg.norm(X2))
    return q


def _same_up_to_sign(A, B, tol):
    return min(np.abs(A - B).max(), np.abs(A + B).max()) < tol


def test_rel5_equals_numpy_restatement():
    rng = np.random.default_rng(1)
    compared = chosen = 0
    for k in range(600):
        p = _problem(rng, 40, outlier_frac=0.0, noise=1e-3 if k % 2 else 0.0)
        s = rng.choice(40, S, replace=False)
        f1, f2 = p["f1"][s], p["f2"][s]
        r = orel.rel5(p["f1"], p["f2"], s)
        sols, skip = _numpy_rel5(f1, f2)
        if skip:
            continue
        # the same real solution set, E up to sign
        assert len(sols) == len(r["E"]), (k, len(sols), len(r["E"]))
        for E in sols:
            assert any(_same_up_to_sign(E, Eo, 1e-7) for Eo in r["E"]), k
        # the same four candidates per E
        for i, Eo in enumerate(r["E"]):
            ref = _numpy_candidates(Eo)
            for M in r["cand"][i]:
                assert any(np.abs(M - Mr).max() < 1e-7 for Mr in ref), k
        compared += 1
        if not r["valid"]:
            continue
        # the same choice where the quality margin is clear
        cands = r["cand"].reshape(-1, 3, 4)
        q = np.array([_numpy_quality(M, f1, f2) for M in cands])
        order = np.argsort(q)
        if len(q) > 1 and q[order[1]] - q[order[0]] > 1e-6:
            assert np.abs(cands[order[0]] - r["model"]).max() < 1e-7, k
            chosen += 1
        assert np.allclose(q, r["quality"].reshape(-1), atol=1e-9), k
    assert compared >= 500 and chosen >= 150, (compared, chosen)


def test_rel5_invalid_samples():
    rng = np.random.default_rng(2)
    for k in range(200):
        p = _problem(rng, 30, outlier_frac=0.0)
        s = np.arange(S); s[3] = s[1]
        r = orel.rel5(p["f1"], p["f2"], s)
        assert not r["valid"] and not r["model"].any()                        # a repeated index
        q = _problem(rng, 4, outlier_frac=0.0)
        assert not orel.rel5(q["f1"], q["f2"], np.r_[np.arange(4), 0])["valid"]   # n < 5
        f2 = p["f2"].copy(); f2[2, 1] = np.inf
        assert not orel.rel5(p["f1"], f2, np.arange(S))["valid"]              # a non-finite bearing
        # pure rotation: t = 0 makes E degenerate; whatever comes out is finite
        p = _problem(rng, 30, outlier_frac=0.0, rotation_only=True)
        r = orel.rel5(p["f1"], p["f2"], np.arange(S))
        assert np.isfinite(r["model"]).all() and (r["valid"] or not r["model"].any())


# ------------------------------------------------------------------------------------------------- selection (CPU)
def _expected_selection(valid, count, n, max_iterations, probability):
    """placerec.ransac_select over the valid samples in order (at most 10 * max_iterations invalid ones are skipped)"""
    idx, skipped, stop = [], 0, len(valid)
    for s in range(len(valid)):
        if skipped >= 10 * max_iterations:
            stop = s
            break
        if valid[s]:
            idx.append(s)
        else:
            skipped += 1
    best, it = PR.ransac_select(np.asarray(count)[idx], n, S, max_iterations, probability)
    consumed = (idx[it - 1] + 1 if it > 0 else 0) if it < len(idx) else stop
    return (idx[best] if best >= 0 else -1), it, consumed


def _check_selection(b, r, max_iterations, probability):
    ptr = b["prob_ptr"]
    for i in range(len(ptr) - 1):
        n = ptr[i + 1] - ptr[i]
        best, it, consumed = _expected_selection(r["sample_valid"][i], r["sample_count"][i], n, max_iterations, probability)
        assert (r["best_sample"][i], r["iterations"][i], r["consumed"][i]) == (best, it, consumed), i
        if best >= 0:
            assert r["best_count"][i] == r["sample_count"][i][best] and np.array_equal(r["best_model"][i], r["sample_model"][i][best])
        else:
            assert r["best_count"][i] == 0 and not r["best_model"][i].any() and not r["inlier_mask"][ptr[i]:ptr[i + 1]].any()


def test_oracle_selection_equals_ransac_select():
    specs = [(0, 0.0, False), (4, 0.0, False), (5, 0.0, False), (120, 0.3, False), (120, 0.1, True), (200, 0.5, False)]
    b, _ = _batch(4, specs, 200)
    for thr, max_it, prob in ((9.0, 150, 0.99), (9.0, 150, 0.999999), (9.0, 5, 0.99), (1e-3, 40, 0.99)):
        r = orel.ransac_central_relative_pose(**b, threshold=thr, max_iterations=max_it, probability=prob, per_sample=True)
        _check_selection(b, r, max_it, prob)
        lazy = orel.ransac_central_relative_pose(**b, threshold=thr, max_iterations=max_it, probability=prob)
        for k in lazy:
            assert np.array_equal(lazy[k], r[k]), k
    r = orel.ransac_central_relative_pose(**b, threshold=9.0, max_iterations=150, per_sample=True)
    assert 0 < r["iterations"][3] < 150 and (r["sample_valid"][3][:r["consumed"][3]] == 0).any()   # adaptive stop, invalid ones interleaved
    assert not r["sample_valid"][:2].any()                                                           # n < 5
    assert np.isfinite(r["sample_model"]).all()
    # skip limit: max_iterations 2 → at most 20 invalid samples are read
    b2 = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in b.items()}
    b2["samples"][:, :60, 4] = b2["samples"][:, :60, 0]
    r = orel.ransac_central_relative_pose(**b2, threshold=9.0, max_iterations=2, per_sample=True)
    _check_selection(b2, r, 2, 0.99)
    assert r["consumed"][3] == 20 and r["iterations"][3] == 0 and r["best_sample"][3] == -1


def test_selected_model_score_equals_scoring_oracle():
    b, _ = _batch(6, [(300, 0.3, False), (500, 0.1, False)], 100)
    r = orel.ransac_central_relative_pose(**b, threshold=9.0, max_iterations=100, per_sample=True)
    ptr = b["prob_ptr"]
    for i in range(2):
        sl = slice(ptr[i], ptr[i + 1])
        _, inl, cnt = og.score_relative_pose(r["best_model"][i][None], b["f1"][sl], b["f2"][sl], b["sigma1"][sl], b["sigma2"][sl], threshold=9.0)
        assert r["best_sample"][i] >= 0 and cnt[0] == r["best_count"][i] and np.array_equal(inl[0], r["inlier_mask"][sl])
        valid = np.flatnonzero(r["sample_valid"][i])[:20]
        _, _, cnt = og.score_relative_pose(r["sample_model"][i][valid], b["f1"][sl], b["f2"][sl], b["sigma1"][sl], b["sigma2"][sl], threshold=9.0)
        assert np.array_equal(cnt, r["sample_count"][i][valid])


# ------------------------------------------------------------------------------------------------- GPU (C-ABI)
GPU_SPECS = [(0, 0.0, False), (1, 0.0, False), (4, 0.0, False), (5, 0.0, False), (6, 0.2, False), (50, 0.4, False), (300, 0.3, False),
             (1000, 0.05, False), (300, 0.6, False), (300, 0.1, True), (1000, 0.0, False)]


def _gpu_vs_oracle(ctx, b, thr, max_it, prob):
    g = PR.ransac_central_relative_pose(ctx, **b, threshold=thr, max_iterations=max_it, probability=prob, per_sample=True)
    r = orel.ransac_central_relative_pose(**b, threshold=thr, max_iterations=max_it, probability=prob, per_sample=True)
    for k in r:
        assert np.array_equal(g[k].view(np.uint8), r[k].view(np.uint8)), k
    return g


@pytest.mark.gpu
def test_gpu_equals_oracle_bitwise(ctx):
    b, _ = _batch(7, GPU_SPECS, 150)
    for thr, max_it, prob in ((9.0, 300, 0.99), (9.0, 300, 0.999999), (0.5, 300, 0.99), (9.0, 1, 0.99), (9.0, 0, 0.99)):
        g = _gpu_vs_oracle(ctx, b, thr, max_it, prob)
        _check_selection(b, g, max_it, prob)
    assert g["sample_valid"].sum() > 800 and (g["sample_valid"][3:] == 0).sum() > 50
    # fewer samples than the bound needs: the 60 % outlier problem runs out of samples at p = 0.999999
    g = _gpu_vs_oracle(ctx, b, 9.0, 300, 0.999999)
    assert g["consumed"][8] == 150 and g["iterations"][8] < 300
    # the selected model through the existing scoring kernel: same count and mask
    g = PR.ransac_central_relative_pose(ctx, **b, threshold=9.0, max_iterations=300)
    ptr, checked = b["prob_ptr"], 0
    for i in range(len(ptr) - 1):
        if g["best_sample"][i] < 0:
            continue
        sl = slice(ptr[i], ptr[i + 1])
        _, inl, c = PR.score_relative_pose(ctx, g["best_model"][i][None], b["f1"][sl], b["f2"][sl], b["sigma1"][sl], b["sigma2"][sl], 9.0,
                                           want_scores=False)
        assert c[0] == g["best_count"][i] and np.array_equal(inl[0], g["inlier_mask"][sl]), i
        checked += 1
    assert checked >= 6
    # without the per-sample outputs the kernel stops at the adaptive bound: same selection
    lean = PR.ransac_central_relative_pose(ctx, **b, threshold=9.0, max_iterations=3)
    full = PR.ransac_central_relative_pose(ctx, **b, threshold=9.0, max_iterations=3, per_sample=True)
    for k in lean:
        assert np.array_equal(lean[k], full[k]), k


@pytest.mark.gpu
def test_gpu_noise_free_scene_gives_ground_truth(ctx):
    b, probs = _batch(11, [(1000, 0.1, False), (300, 0.3, False), (1000, 0.2, False)], 300, repeat_frac=0.0)
    g = _gpu_vs_oracle(ctx, b, 1.0, 300, 0.99)
    ptr = b["prob_ptr"]
    for i, p in enumerate(probs):
        assert g["best_sample"][i] >= 0 and g["iterations"][i] < 100
        assert _pose_err(g["best_model"][i], p["R"], p["t"]) < 1e-8, i
        assert np.array_equal(g["inlier_mask"][ptr[i]:ptr[i + 1]].astype(bool), p["inlier"])
        assert g["best_count"][i] == p["inlier"].sum()


@pytest.mark.gpu
def test_gpu_bad_arguments_are_refused(ctx):
    from covins_b200._lib import lib
    b, _ = _batch(5, [(0, 0.0, False), (57, 0.3, False), (100, 0.3, False)], 20)
    keep = []

    def call(n_prob=3, ns=20, max_it=300, per_sample=(False, False, False), **over):
        a = {k: np.ascontiguousarray(v) for k, v in b.items()}
        a.update(over)
        keep.append(a)
        res = {k: np.zeros(s, dt) for k, s, dt in (("bs", 3, np.int32), ("bm", 36, np.float64), ("bc", 3, np.int32), ("it", 3, np.int32),
                                                    ("us", 3, np.int32), ("sm", 3 * 20 * 12, np.float64), ("sv", 60, np.uint8), ("sc", 60, np.int32))}
        keep.append(res)
        ptr = lambda k: a[k].ctypes.data if a[k] is not None else None
        P = PR.CCentralRelRansacProblems(n_prob, *[ptr(k) for k in ("prob_ptr", "f1", "f2", "sigma1", "sigma2", "samples")], ns)
        opt = [res[k].ctypes.data if on else None for k, on in zip(("sm", "sv", "sc"), per_sample)]
        R = PR.CRelRansacResult(res["bs"].ctypes.data, res["bm"].ctypes.data, res["bc"].ctypes.data, res["it"].ctypes.data, res["us"].ctypes.data,
                                None, *opt)
        return lib().cvb_ransac_central_relative_pose_batch(ctx.handle, C.byref(P), 9.0, max_it, 0.99, C.byref(R))

    assert call() == 0 and call(per_sample=(True, True, True)) == 0
    assert call(n_prob=0) == 0
    assert call(per_sample=(True, False, True)) == 1 and call(per_sample=(False, False, True)) == 1
    bad = b["samples"].copy(); bad[1, 7, 2] = 57
    assert call(samples=bad) == 1
    bad = b["samples"].copy(); bad[2, 0, 0] = -1
    assert call(samples=bad) == 1
    assert call(n_prob=-1) == 1 and call(ns=-1) == 1 and call(max_it=-1) == 1
    assert call(f1=None) == 1 and call(sigma2=None) == 1 and call(samples=None) == 1 and call(prob_ptr=None) == 1
    assert call(prob_ptr=np.array([0, 57, 50, 157], np.int32)) == 1
    assert lib().cvb_ransac_central_relative_pose_batch(ctx.handle, None, 9.0, 300, 0.99, None) == 1


# ------------------------------------------------------------------------------------------------- C++ wrapper
def _build_shim(out):
    import covins_b200
    if not os.path.exists(covins_b200.LIB_PATH):
        covins_b200.build()
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-o", out, os.path.join(ROOT, "tests", "cpp", "shim_ransac_rel5_test.cpp"),
                           "-L" + os.path.join(ROOT, "covins_b200"), "-lcovins_b200", "-Wl,-rpath," + os.path.join(ROOT, "covins_b200")])


def test_shim_ransac_rel5_compiles_and_links(tmp_path):
    exe = str(tmp_path / "shim_ransac_rel5_test")
    _build_shim(exe)
    assert os.path.exists(exe)


@pytest.mark.gpu
def test_shim_ransac_rel5_equals_python_path(ctx, tmp_path):
    exe = str(tmp_path / "shim_ransac_rel5_test")
    _build_shim(exe)
    b, _ = _batch(9, [(300, 0.3, False), (0, 0.0, False), (1000, 0.1, False), (5, 0.0, False)], 120)
    for k, v in b.items():
        np.ascontiguousarray(v).tofile(tmp_path / f"{k}.bin")
    np.array([9.0, 100.0, 0.99]).tofile(tmp_path / "params.bin")
    subprocess.check_call([exe, str(tmp_path)])
    g = PR.ransac_central_relative_pose(ctx, **b, threshold=9.0, max_iterations=100, probability=0.99)
    ints = np.fromfile(tmp_path / "out_ints.bin", np.int32).reshape(-1, 4)
    assert np.array_equal(ints, np.stack([g["best_sample"], g["best_count"], g["iterations"], g["consumed"]], 1))
    assert np.array_equal(np.fromfile(tmp_path / "out_models.bin").reshape(-1, 3, 4), g["best_model"])
    assert np.array_equal(np.fromfile(tmp_path / "out_mask.bin", np.uint8), g["inlier_mask"])
    assert (g["best_sample"][[0, 2]] >= 0).all()
