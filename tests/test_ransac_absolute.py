"""Absolute-pose RANSAC from caller-supplied samples (cvb_ransac_absolute_pose_batch).
CPU: the oracle's P3P against ground truth and against an independent numpy restatement (Grunert's quartic + SVD alignment), and
its selection against placerec.ransac_select.  GPU: the C-ABI call is bit-identical to the oracle, its mask and count equal
cvb_score_absolute_pose_batch on the selected model, a noise-free scene gives the true pose and inlier set, bad arguments are
refused, and the C++ wrapper equals the Python path."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from covins_b200 import placerec as PR, synth
from oracle import ransac as orr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rand_rot(rng):
    q = rng.normal(size=4); q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _rot_err(A, B):
    return 2 * np.arcsin(min(1.0, np.linalg.norm(A - B) / (2 * np.sqrt(2))))


def _p3p_cases(seed, n=2400):
    """(bearings [3,3], world points [3,3], R, t, well_conditioned): depths 1-30 m; every 8th sample has two points 1 cm
    apart, every 8th (offset 4) three world points within 1e-3 of a line"""
    rng = np.random.default_rng(seed)
    for i in range(n):
        R, t = _rand_rot(rng), rng.normal(0, 5, 3)
        d = rng.normal(0, 1, (3, 3)); d[:, 2] = np.abs(d[:, 2]) + 0.5; d /= np.linalg.norm(d, axis=1, keepdims=True)
        pc = d * rng.uniform(1, 30, 3)[:, None]
        kind = "two_close" if i % 8 == 0 else "collinear" if i % 8 == 4 else "generic"
        if kind == "two_close":
            pc[1] = pc[0] + rng.normal(0, 0.01 / np.sqrt(3), 3)
        elif kind == "collinear":
            pc[2] = pc[0] + rng.uniform(0.3, 2.0) * (pc[1] - pc[0]) + rng.normal(0, 1e-3, 3)
        f = pc / np.linalg.norm(pc, axis=1, keepdims=True)
        x = (pc - t) @ R                                  # x_c = R x + t
        yield f, x, R, t, kind == "generic"


def test_p3p_recovers_ground_truth():
    n_good = n_sol = 0
    for f, x, R, t, good in _p3p_cases(0):
        sols = orr.p3p(f, x)
        assert len(sols) <= 4
        for Rs, ts in sols:
            pc = x @ Rs.T + ts
            depth = np.einsum("ij,ij->i", pc, f)
            assert depth.min() > 0
            assert np.abs(pc / np.linalg.norm(pc, axis=1, keepdims=True) - f).max() < 1e-9
        if good:
            n_good += 1
            assert any(_rot_err(Rs, R) < 1e-8 and np.linalg.norm(ts - t) < 1e-8 * max(np.linalg.norm(t), 1.0) for Rs, ts in sols)
        n_sol += len(sols)
    assert n_good >= 1800 and n_sol > 2400


def _grunert(f, x):
    """independent restatement: Grunert's quartic in v = s3/s1 (resultant of the two distance equations in u = s2/s1) via np.roots,
    depths from the law of cosines, pose by SVD alignment of the camera-frame points to the world points"""
    P = np.polynomial.polynomial
    a2, b2, c2 = np.sum((x[1] - x[2]) ** 2), np.sum((x[0] - x[2]) ** 2), np.sum((x[0] - x[1]) ** 2)
    ca, cb, cg = f[1] @ f[2], f[0] @ f[2], f[0] @ f[1]
    # b2 (1 + u^2 - 2u cg) = c2 (1 + v^2 - 2v cb);  a2 (1 + v^2 - 2v cb) = b2 (u^2 + v^2 - 2uv ca): coefficients of u^k as polynomials in v
    w = np.array([1.0, -2 * cb, 1.0])
    p2, p1, p0 = np.array([b2]), np.array([-2 * b2 * cg]), P.polysub([b2], c2 * w)
    q2, q1, q0 = np.array([-b2]), np.array([0.0, 2 * b2 * ca]), P.polysub(a2 * w, [0.0, 0.0, b2])
    m = lambda *ps: P.polymul(ps[0], ps[1]) if len(ps) == 2 else P.polymul(ps[0], m(*ps[1:]))
    r20, r21, r10 = P.polysub(m(p2, q0), m(q2, p0)), P.polysub(m(p2, q1), m(q2, p1)), P.polysub(m(p1, q0), m(q1, p0))
    res = P.polysub(m(r20, r20), m(r21, r10))
    out = []
    for v in np.roots(res[::-1]):
        if abs(v.imag) > 1e-6 * max(1.0, abs(v)):
            continue
        v = v.real
        u = -P.polyval(v, r20) / P.polyval(v, r21)
        s1 = np.sqrt(b2 / (1 + v * v - 2 * v * cb))
        s = np.array([s1, u * s1, v * s1])
        if s.min() <= 0:
            continue
        pc = f * s[:, None]
        xm, pm = x.mean(0), pc.mean(0)
        U, _, Vt = np.linalg.svd((pc - pm).T @ (x - xm))
        R = U @ np.diag([1, 1, np.linalg.det(U @ Vt)]) @ Vt
        out.append((R, pm - R @ xm))
    return out


def test_p3p_equals_grunert_restatement():
    compared = 0
    for f, x, R, t, good in _p3p_cases(1, n=2000):
        if not good:
            continue
        ours, ref = orr.p3p(f, x), _grunert(f, x)
        close = lambda A, B: _rot_err(A[0], B[0]) < 1e-6 and np.linalg.norm(A[1] - B[1]) < 1e-6 * max(np.linalg.norm(B[1]), 1.0)
        # a pair of nearly equal real roots can come back from np.roots as complex: compare only where the sets are well separated
        if any(close(A, B) for i, A in enumerate(ref) for B in ref[i + 1:]):
            continue
        assert all(any(close(A, B) for B in ref) for A in ours), (ours, ref)
        assert all(any(close(A, B) for A in ours) for B in ref), (ours, ref)
        compared += 1
    assert compared >= 1450


# ------------------------------------------------------------------------------------------------- scenes and selection
def _problem(rng, n, outlier_frac=0.3, sigma=(1e-6, 1e-5), noise=0.0):
    """one problem: camera (c, Rc) in the body frame, body-in-world Twb, world points seen at 1-30 m, a share of bearings
    replaced by random directions"""
    Rc, c = _rand_rot(rng), rng.normal(0, 0.05, 3)
    R, t = _rand_rot(rng), rng.normal(0, 3, 3)
    d = rng.normal(0, 1, (n, 3)); d[:, 2] = np.abs(d[:, 2]) + 1.0; d /= np.linalg.norm(d, axis=1, keepdims=True)
    pc = d * rng.uniform(1, 30, n)[:, None]
    pw = (pc @ Rc.T + c) @ R.T + t                    # p_b = Rc p_c + c, p_w = R p_b + t
    f = pc + rng.normal(0, noise, pc.shape) * np.linalg.norm(pc, axis=1, keepdims=True)
    out = rng.random(n) < outlier_frac
    f[out] = rng.normal(0, 1, (out.sum(), 3))
    f /= np.linalg.norm(f, axis=1, keepdims=True)
    return dict(pts=pw, f=f, sigma=rng.uniform(*sigma, n), c=c, Rc=Rc, T=np.concatenate([R, t[:, None]], 1), inlier=~out)


def _batch(seed, sizes, n_samples, outlier_frac=0.3):
    rng = np.random.default_rng(seed)
    probs = [_problem(rng, n, outlier_frac) for n in sizes]
    samples = np.zeros((len(sizes), n_samples, 4), np.int32)
    for i, (n, pr) in enumerate(zip(sizes, probs)):
        if n >= 4:
            samples[i] = np.stack([rng.choice(n, 4, replace=False) for _ in range(n_samples)])
            rep = rng.random(n_samples) < 0.1                                   # repeated indices
            samples[i, rep, 3] = samples[i, rep, 1]
        if n >= 30:                                                             # world points 0..9 exactly collinear
            a, b = pr["pts"][0], pr["pts"][1]
            for j in range(2, 10):
                pr["pts"][j] = a + (j / 2.0) * (b - a)
            samples[i, 5:10, :3] = [[0, 1, 2], [3, 4, 5], [6, 7, 8], [2, 5, 9], [1, 4, 7]]
    ptr = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    cat = lambda k: np.concatenate([p[k] for p in probs]) if sum(sizes) else np.zeros((0, 3) if k != "sigma" else 0)
    return dict(prob_ptr=ptr, pts=cat("pts"), bearings=cat("f"), sigma=cat("sigma"), cam_off=np.stack([p["c"] for p in probs]),
                cam_rot=np.stack([p["Rc"] for p in probs]), samples=samples), probs


def _expected_selection(valid, count, n, max_iterations, probability):
    """placerec.ransac_select over the valid samples in order (opengv's skipped_count: at most 10 * max_iterations invalid ones)"""
    idx, skipped, stop = [], 0, len(valid)
    for s in range(len(valid)):
        if skipped >= 10 * max_iterations:
            stop = s
            break
        if valid[s]:
            idx.append(s)
        else:
            skipped += 1
    best, it = PR.ransac_select(np.asarray(count)[idx], n, 4, max_iterations, probability)
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
    b, _ = _batch(3, [0, 3, 4, 57, 400, 400], 400, outlier_frac=0.6)
    for thr, max_it, prob in ((25.0, 300, 0.99), (25.0, 300, 0.999999), (25.0, 7, 0.99), (1e-3, 40, 0.99)):
        r = orr.ransac_absolute_pose(**b, threshold=thr, max_iterations=max_it, probability=prob, per_sample=True)
        _check_selection(b, r, max_it, prob)
        lazy = orr.ransac_absolute_pose(**b, threshold=thr, max_iterations=max_it, probability=prob)
        for k in ("best_sample", "best_model", "best_count", "iterations", "consumed", "inlier_mask"):
            assert np.array_equal(lazy[k], r[k]), k
    assert (r["sample_valid"][4] == 0).sum() > 40                                  # invalid samples interleaved
    # skip limit: max_iterations 2 → at most 20 invalid samples are read
    b2 = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in b.items()}
    b2["samples"][:, :60, 3] = b2["samples"][:, :60, 0]
    r = orr.ransac_absolute_pose(**b2, threshold=25.0, max_iterations=2, per_sample=True)
    _check_selection(b2, r, 2, 0.99)
    assert r["consumed"][4] == 20 and r["iterations"][4] == 0 and r["best_sample"][4] == -1
    # problems with fewer than 4 correspondences never have a hypothesis
    assert not r["sample_valid"][:2].any() and r["sample_valid"][2].any()


# ------------------------------------------------------------------------------------------------- GPU (C-ABI)
def _gpu_vs_oracle(ctx, b, thr, max_it, prob):
    g = PR.ransac_absolute_pose(ctx, **b, threshold=thr, max_iterations=max_it, probability=prob, per_sample=True)
    r = orr.ransac_absolute_pose(**b, threshold=thr, max_iterations=max_it, probability=prob, per_sample=True)
    for k in r:
        assert np.array_equal(g[k], r[k]), k
    return g


@pytest.mark.gpu
def test_gpu_equals_oracle_bitwise(ctx):
    b, _ = _batch(7, [0, 3, 4, 57, 1000, 2000], 350)
    for thr, max_it, prob in ((25.0, 300, 0.99), (25.0, 300, 0.999999), (0.5, 300, 0.99), (25.0, 3, 0.99)):
        g = _gpu_vs_oracle(ctx, b, thr, max_it, prob)
        _check_selection(b, g, max_it, prob)
    assert g["sample_valid"][3:].sum() > 500 and (g["sample_valid"][3:] == 0).sum() > 60
    # the selected model through the existing scoring kernel: same count and mask (shared per-correspondence score)
    ptr = b["prob_ptr"]
    for i in range(len(ptr) - 1):
        if g["best_sample"][i] < 0:
            continue
        s = slice(ptr[i], ptr[i + 1])
        _, inl, cnt = PR.score_absolute_pose(ctx, g["best_model"][i][None], b["pts"][s], b["bearings"][s], b["sigma"][s], b["cam_off"][i], b["cam_rot"][i], 25.0,
                                             want_scores=False)
        assert cnt[0] == g["best_count"][i] and np.array_equal(inl[0], g["inlier_mask"][s])
    # without the per-sample outputs the kernel stops at the adaptive bound: same selection
    lean = PR.ransac_absolute_pose(ctx, **b, threshold=25.0, max_iterations=3)
    for k in lean:
        assert np.array_equal(lean[k], g[k]), k


@pytest.mark.gpu
def test_gpu_noise_free_scene_gives_ground_truth(ctx):
    rng = np.random.default_rng(11)
    sizes = [1000, 300, 1000]
    probs = [_problem(rng, n, 0.3) for n in sizes]
    samples = np.stack([np.stack([rng.choice(n, 4, replace=False) for _ in range(400)]) for n in sizes]).astype(np.int32)
    b = dict(prob_ptr=np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32), pts=np.concatenate([p["pts"] for p in probs]),
             bearings=np.concatenate([p["f"] for p in probs]), sigma=np.concatenate([p["sigma"] for p in probs]),
             cam_off=np.stack([p["c"] for p in probs]), cam_rot=np.stack([p["Rc"] for p in probs]), samples=samples)
    g = _gpu_vs_oracle(ctx, b, 1.0, 300, 0.99)
    ptr = b["prob_ptr"]
    for i, p in enumerate(probs):
        assert g["best_sample"][i] >= 0 and g["iterations"][i] < 60
        assert np.abs(g["best_model"][i] - p["T"]).max() < 1e-9
        assert np.array_equal(g["inlier_mask"][ptr[i]:ptr[i + 1]].astype(bool), p["inlier"])
        assert g["best_count"][i] == p["inlier"].sum()


@pytest.mark.gpu
def test_gpu_bad_arguments_are_refused(ctx):
    from covins_b200._lib import lib
    b, _ = _batch(5, [0, 57, 100], 20)
    keep = []

    def call(n_prob=3, ns=20, max_it=300, **over):
        a = {k: np.ascontiguousarray(v) for k, v in b.items()}
        a.update(over)
        keep.append(a)
        res = {k: np.zeros(s, dt) for k, s, dt in (("bs", 3, np.int32), ("bm", 36, np.float64), ("bc", 3, np.int32), ("it", 3, np.int32),
                                                    ("us", 3, np.int32))}
        keep.append(res)
        ptr = lambda k: a[k].ctypes.data if a[k] is not None else None
        P = PR.CAbsRansacProblems(n_prob, ptr("prob_ptr"), ptr("pts"), ptr("bearings"), ptr("sigma"), ptr("cam_off"), ptr("cam_rot"), ptr("samples"), ns)
        R = PR.CAbsRansacResult(res["bs"].ctypes.data, res["bm"].ctypes.data, res["bc"].ctypes.data, res["it"].ctypes.data, res["us"].ctypes.data,
                                None, None, None, None)
        return lib().cvb_ransac_absolute_pose_batch(ctx.handle, C.byref(P), 25.0, max_it, 0.99, C.byref(R))

    assert call() == 0
    assert call(n_prob=0) == 0
    bad = b["samples"].copy(); bad[1, 7, 2] = 57
    assert call(samples=bad) == 1
    bad = b["samples"].copy(); bad[2, 0, 0] = -1
    assert call(samples=bad) == 1
    assert call(n_prob=-1) == 1 and call(ns=-1) == 1 and call(max_it=-1) == 1
    assert call(pts=None) == 1 and call(samples=None) == 1 and call(cam_rot=None) == 1 and call(prob_ptr=None) == 1
    assert call(prob_ptr=np.array([0, 57, 50, 157], np.int32)) == 1
    assert lib().cvb_ransac_absolute_pose_batch(ctx.handle, None, 25.0, 300, 0.99, None) == 1


# ------------------------------------------------------------------------------------------------- C++ wrapper
def _build_shim(out):
    import covins_b200
    if not os.path.exists(covins_b200.LIB_PATH):
        covins_b200.build()
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-o", out, os.path.join(ROOT, "tests", "cpp", "shim_ransac_test.cpp"),
                           "-L" + os.path.join(ROOT, "covins_b200"), "-lcovins_b200", "-Wl,-rpath," + os.path.join(ROOT, "covins_b200")])


def test_shim_ransac_compiles_and_links(tmp_path):
    exe = str(tmp_path / "shim_ransac_test")
    _build_shim(exe)
    assert os.path.exists(exe)


@pytest.mark.gpu
def test_shim_ransac_equals_python_path(ctx, tmp_path):
    exe = str(tmp_path / "shim_ransac_test")
    _build_shim(exe)
    b, _ = _batch(9, [57, 0, 1000, 4], 320)
    for k, v in b.items():
        np.ascontiguousarray(v).tofile(tmp_path / f"{k}.bin")
    np.array([25.0, 300.0, 0.99]).tofile(tmp_path / "params.bin")
    subprocess.check_call([exe, str(tmp_path)])
    g = PR.ransac_absolute_pose(ctx, **b, threshold=25.0, max_iterations=300, probability=0.99)
    ints = np.fromfile(tmp_path / "out_ints.bin", np.int32).reshape(-1, 4)
    assert np.array_equal(ints, np.stack([g["best_sample"], g["best_count"], g["iterations"], g["consumed"]], 1))
    assert np.array_equal(np.fromfile(tmp_path / "out_models.bin").reshape(-1, 3, 4), g["best_model"])
    assert np.array_equal(np.fromfile(tmp_path / "out_mask.bin", np.uint8), g["inlier_mask"])
    assert (g["best_sample"][[0, 2]] >= 0).all()
