"""Non-central relative-pose (17-point) RANSAC from caller-supplied samples (cvb_ransac_noncentral_relative_pose_batch).
CPU: the oracle's 17-point solve against ground truth and against an independent numpy restatement (SVD null vector, SVD polar
factor, lstsq translation), its rank test on central rigs and repeated points, its selection against placerec.ransac_select, and
its per-camera-pair score against the existing relative-pose scoring oracle.  GPU: the C-ABI call is bit-identical to the oracle,
its mask and count equal cvb_score_relative_pose_batch over the camera-pair models, a noise-free scene gives the true pose and
inlier set, bad arguments are refused, and the C++ wrapper equals the Python path."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from covins_b200 import placerec as PR
from oracle import geom as og
from oracle import ransac_rel as orel

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
S = 17


def _rand_rot(rng):
    q = rng.normal(size=4); q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _rig(rng, ncam, central=False):
    """ncam cameras like consecutive keyframes on a curved path: centres on an arc (not collinear for ncam >= 3), each with its
    own orientation; central: every camera at the first one's centre"""
    th = np.sort(rng.uniform(0.0, 0.8, ncam)); rad = rng.uniform(3, 8)
    c = np.stack([rad * np.sin(th), rng.normal(0, 0.3, ncam), rad * (1 - np.cos(th))], 1)
    if central:
        c[:] = c[0]
    return c, np.stack([_rand_rot(rng) for _ in range(ncam)])


def _problem(rng, n, nc1=3, nc2=3, outlier_frac=0.3, central=False, noise=0.0, sigma=(1e-6, 1e-5)):
    """one candidate: rig 1, rig 2 and the rig-frame pose X1 = R X2 + t; points at 1-30 m in front of a camera of rig 1,
    correspondences over all camera pairs, a share of the rig-2 bearings replaced by random directions"""
    c1, R1 = _rig(rng, nc1, central); c2, R2 = _rig(rng, nc2, central)
    R, t = _rand_rot(rng), rng.normal(0, 2, 3)
    j1, j2 = rng.integers(0, nc1, n), rng.integers(0, nc2, n)
    d = rng.normal(0, 1, (n, 3)); d[:, 2] = np.abs(d[:, 2]) + 1.0; d /= np.linalg.norm(d, axis=1, keepdims=True)
    X1 = c1[j1] + np.einsum("nij,nj->ni", R1[j1], d * rng.uniform(1, 30, n)[:, None])
    X2 = (X1 - t) @ R                                   # R^T (X1 - t)
    f1 = np.einsum("nji,nj->ni", R1[j1], X1 - c1[j1])
    f2 = np.einsum("nji,nj->ni", R2[j2], X2 - c2[j2])
    f1 += rng.normal(0, noise, f1.shape) * np.linalg.norm(f1, axis=1, keepdims=True)
    f2 += rng.normal(0, noise, f2.shape) * np.linalg.norm(f2, axis=1, keepdims=True)
    out = rng.random(n) < outlier_frac
    f2[out] = rng.normal(0, 1, (out.sum(), 3))
    f1 /= np.linalg.norm(f1, axis=1, keepdims=True); f2 /= np.linalg.norm(f2, axis=1, keepdims=True)
    return dict(f1=f1, f2=f2, s1=rng.uniform(*sigma, n), s2=rng.uniform(*sigma, n), cam1=j1.astype(np.int32), cam2=j2.astype(np.int32),
                c1=c1, R1=R1, c2=c2, R2=R2, T=np.concatenate([R, t[:, None]], 1), inlier=~out)


def _batch(seed, specs, n_samples, outlier_frac=0.3, repeat_frac=0.1):
    """specs: (n, nc1, nc2, central) per problem → (arguments of ransac_noncentral_relative_pose, problems)"""
    rng = np.random.default_rng(seed)
    probs = [_problem(rng, n, a, b, outlier_frac, central) for n, a, b, central in specs]
    samples = np.zeros((len(specs), n_samples, S), np.int32)
    for i, (n, *_) in enumerate(specs):
        if n >= S:
            samples[i] = np.stack([rng.choice(n, S, replace=False) for _ in range(n_samples)])
            rep = rng.random(n_samples) < repeat_frac                          # repeated indices
            samples[i, rep, 16] = samples[i, rep, 3]
    cat = lambda k, shape: np.concatenate([p[k] for p in probs]) if probs else np.zeros(shape)
    ptr = lambda k: np.concatenate([[0], np.cumsum([len(p[k]) for p in probs])]).astype(np.int32)
    b = dict(prob_ptr=ptr("f1"), f1=cat("f1", (0, 3)), f2=cat("f2", (0, 3)), sigma1=cat("s1", 0), sigma2=cat("s2", 0),
             cam1=cat("cam1", 0).astype(np.int32), cam2=cat("cam2", 0).astype(np.int32), cam_ptr1=ptr("c1"), cam_off1=cat("c1", (0, 3)),
             cam_rot1=cat("R1", (0, 3, 3)), cam_ptr2=ptr("c2"), cam_off2=cat("c2", (0, 3)), cam_rot2=cat("R2", (0, 3, 3)), samples=samples)
    return b, probs


def _rig_args(p):
    return p["cam1"], p["cam2"], p["c1"], p["R1"], p["c2"], p["R2"]


def _t_close(a, b, tol):
    return np.linalg.norm(a - b) < tol * max(np.linalg.norm(b), 1.0)


# ------------------------------------------------------------------------------------------------- 17-point solve (CPU)
def test_rel17_recovers_ground_truth():
    rng = np.random.default_rng(0)
    ok = 0
    ratios = []
    for k in range(2000):
        p = _problem(rng, S, 3, 3, outlier_frac=0.0)
        M, valid, ratio = orel.rel17(p["f1"], p["f2"], *_rig_args(p), np.arange(S))
        assert valid, k
        ratios.append(ratio)
        assert np.abs(M[:, :3] - p["T"][:, :3]).max() < 1e-8, k
        assert _t_close(M[:, 3], p["T"][:, 3], 1e-8), k
        ok += 1
    assert ok == 2000 and min(ratios) > 1e-7        # generic noise-free samples stay far above the 1e-10 rank tolerance


def _numpy_rel17(p, s):
    """independent restatement: null vector of A by SVD, polar factor by SVD, t by lstsq"""
    rows, G, H = [], [], []
    dm = []
    for i in s:
        a, b = p["cam1"][i], p["cam2"][i]
        d1 = p["R1"][a] @ p["f1"][i]; m1 = np.cross(p["c1"][a], d1)
        d2 = p["R2"][b] @ p["f2"][i]; m2 = np.cross(p["c2"][b], d2)
        rows.append(np.r_[np.outer(d1, d2).ravel(), (np.outer(d1, m2) + np.outer(m1, d2)).ravel()])
        dm.append((d1, m1, d2, m2))
    _, sv, Vt = np.linalg.svd(np.array(rows))
    if sv[-2] < 1e-12 * sv[0]:
        return None                                     # rank below 17
    x = Vt[-1]
    Rp = x[9:].reshape(3, 3)
    if np.linalg.det(Rp) < 0:
        Rp = -Rp
    U, _, Vt = np.linalg.svd(Rp)
    R = U @ Vt
    for d1, m1, d2, m2 in dm:
        G.append(np.cross(R @ d2, d1)); H.append(-(d1 @ R @ m2 + m1 @ R @ d2))
    t = np.linalg.lstsq(np.array(G), np.array(H), rcond=None)[0]
    return R, t


def test_rel17_equals_numpy_restatement():
    rng = np.random.default_rng(1)
    compared = 0
    for k in range(600):
        p = _problem(rng, 40, 3, 3, outlier_frac=0.0, noise=1e-3 if k % 2 else 0.0)
        s = rng.choice(40, S, replace=False)
        M, valid, ratio = orel.rel17(p["f1"], p["f2"], *_rig_args(p), s)
        ref = _numpy_rel17(p, s)
        # nine or more correspondences of one camera pair span at most eight rows: both restatements see the rank drop
        assert valid == (ref is not None), (k, ratio)
        if not valid:
            continue
        R, t = ref
        assert np.abs(M[:, :3] - R).max() < 1e-9, (k, ratio)
        assert _t_close(M[:, 3], t, 1e-9), (k, ratio)
        compared += 1
    assert compared >= 590


def test_rel17_degenerate_samples_are_invalid():
    rng = np.random.default_rng(2)
    for k in range(200):
        # every camera of each rig at one centre: the generalised epipolar system loses rank
        p = _problem(rng, 30, 3, 3, outlier_frac=0.0, central=True)
        M, valid, ratio = orel.rel17(p["f1"], p["f2"], *_rig_args(p), np.arange(S))
        assert not valid and ratio < 1e-12 and not M.any(), (k, ratio)
        # a repeated point (the same correspondence at two indices)
        p = _problem(rng, 30, 3, 3, outlier_frac=0.0)
        for key in ("f1", "f2", "cam1", "cam2"):
            p[key][16] = p[key][5]
        M, valid, ratio = orel.rel17(p["f1"], p["f2"], *_rig_args(p), np.arange(S))
        assert not valid and ratio < 1e-12, (k, ratio)
        # a repeated index
        s = np.arange(S); s[9] = s[2]
        assert not orel.rel17(p["f1"], p["f2"], *_rig_args(p), s)[1]
        # fewer than 17 correspondences, non-finite input
        q = _problem(rng, 16, 3, 3, outlier_frac=0.0)
        assert not orel.rel17(q["f1"], q["f2"], *_rig_args(q), np.r_[np.arange(16), 0])[1]
        p["f2"][7, 1] = np.nan
        assert not orel.rel17(p["f1"], p["f2"], *_rig_args(p), np.arange(S))[1]


def test_identity_rig_score_equals_central_scoring_oracle():
    rng = np.random.default_rng(3)
    p = _problem(rng, 500, 1, 1, outlier_frac=0.3, noise=1e-3)
    I = np.eye(3)[None]; z = np.zeros((1, 3))
    models = np.stack([np.concatenate([_rand_rot(rng), rng.normal(0, 2, (3, 1))], 1) for _ in range(20)] + [p["T"]])
    zero = np.zeros(500, np.int32)
    sc, inl, cnt = orel.score_noncentral_relative_pose(models, p["f1"], p["f2"], p["s1"], p["s2"], zero, zero, z, I, z, I, 9.0)
    rs, ri, rc = og.score_relative_pose(models, p["f1"], p["f2"], p["s1"], p["s2"], threshold=9.0)
    assert np.array_equal(sc.view(np.uint64), rs.view(np.uint64)) and np.array_equal(inl, ri) and np.array_equal(cnt, rc)
    assert 0 < cnt[-1] < 500
    for k in range(len(models)):
        assert np.array_equal(orel.rel_pair_model(models[k], z, I, z, I), models[k])


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
    specs = [(0, 1, 1, False), (16, 2, 3, False), (17, 3, 3, False), (120, 3, 3, False), (120, 3, 2, True), (200, 4, 3, False)]
    b, _ = _batch(4, specs, 200, outlier_frac=0.05)
    for thr, max_it, prob in ((9.0, 150, 0.99), (9.0, 150, 0.999999), (9.0, 5, 0.99), (1e-3, 40, 0.99)):
        r = orel.ransac_noncentral_relative_pose(**b, threshold=thr, max_iterations=max_it, probability=prob, per_sample=True)
        _check_selection(b, r, max_it, prob)
        lazy = orel.ransac_noncentral_relative_pose(**b, threshold=thr, max_iterations=max_it, probability=prob)
        for k in lazy:
            assert np.array_equal(lazy[k], r[k]), k
    r = orel.ransac_noncentral_relative_pose(**b, threshold=9.0, max_iterations=150, per_sample=True)
    assert 0 < r["iterations"][3] < 150 and (r["sample_valid"][3][:r["consumed"][3]] == 0).any()   # adaptive stop, invalid ones interleaved
    assert not r["sample_valid"][:2].any() and not r["sample_valid"][4].any()                        # n < 17; central rigs
    # skip limit: max_iterations 2 → at most 20 invalid samples are read
    b2 = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in b.items()}
    b2["samples"][:, :60, 16] = b2["samples"][:, :60, 0]
    r = orel.ransac_noncentral_relative_pose(**b2, threshold=9.0, max_iterations=2, per_sample=True)
    _check_selection(b2, r, 2, 0.99)
    assert r["consumed"][3] == 20 and r["iterations"][3] == 0 and r["best_sample"][3] == -1


# ------------------------------------------------------------------------------------------------- GPU (C-ABI)
GPU_SPECS = [(0, 1, 1, False), (16, 2, 2, False), (17, 3, 3, False), (18, 1, 4, False), (300, 3, 3, True), (300, 4, 2, False),
             (2000, 3, 3, False), (300, 2, 4, False)]


def _gpu_vs_oracle(ctx, b, thr, max_it, prob):
    g = PR.ransac_noncentral_relative_pose(ctx, **b, threshold=thr, max_iterations=max_it, probability=prob, per_sample=True)
    r = orel.ransac_noncentral_relative_pose(**b, threshold=thr, max_iterations=max_it, probability=prob, per_sample=True)
    for k in r:
        assert np.array_equal(g[k], r[k]), k
    return g


@pytest.mark.gpu
def test_gpu_equals_oracle_bitwise(ctx):
    b, _ = _batch(7, GPU_SPECS, 150)
    for thr, max_it, prob in ((9.0, 100, 0.99), (9.0, 100, 0.999999), (0.5, 100, 0.99), (9.0, 3, 0.99)):
        g = _gpu_vs_oracle(ctx, b, thr, max_it, prob)
        _check_selection(b, g, max_it, prob)
    assert g["sample_valid"].sum() > 500 and (g["sample_valid"][2:] == 0).sum() > 100
    assert not g["sample_valid"][4].any()                                          # the central-rig problem
    # the selected model through the existing scoring kernel, one camera pair at a time: same count and mask
    ptr, cp1, cp2 = b["prob_ptr"], b["cam_ptr1"], b["cam_ptr2"]
    g = PR.ransac_noncentral_relative_pose(ctx, **b, threshold=9.0, max_iterations=100)
    checked = 0
    for i in range(len(ptr) - 1):
        if g["best_sample"][i] < 0:
            continue
        sl = slice(ptr[i], ptr[i + 1])
        c1, c2 = b["cam1"][sl], b["cam2"][sl]
        mask = np.zeros(ptr[i + 1] - ptr[i], np.uint8); cnt = 0
        for j1 in range(cp1[i + 1] - cp1[i]):
            for j2 in range(cp2[i + 1] - cp2[i]):
                sel = np.flatnonzero((c1 == j1) & (c2 == j2))
                if not len(sel):
                    continue
                P = orel.rel_pair_model(g["best_model"][i], b["cam_off1"][cp1[i] + j1], b["cam_rot1"][cp1[i] + j1], b["cam_off2"][cp2[i] + j2],
                                       b["cam_rot2"][cp2[i] + j2])
                _, inl, c = PR.score_relative_pose(ctx, P[None], b["f1"][sl][sel], b["f2"][sl][sel], b["sigma1"][sl][sel], b["sigma2"][sl][sel], 9.0,
                                                   want_scores=False)
                mask[sel] = inl[0]; cnt += int(c[0])
        assert cnt == g["best_count"][i] and np.array_equal(mask, g["inlier_mask"][sl]), i
        checked += 1
    assert checked >= 3
    # without the per-sample outputs the kernel stops at the adaptive bound: same selection
    lean = PR.ransac_noncentral_relative_pose(ctx, **b, threshold=9.0, max_iterations=3)
    full = PR.ransac_noncentral_relative_pose(ctx, **b, threshold=9.0, max_iterations=3, per_sample=True)
    for k in lean:
        assert np.array_equal(lean[k], full[k]), k


@pytest.mark.gpu
def test_gpu_noise_free_scene_gives_ground_truth(ctx):
    b, probs = _batch(11, [(1000, 3, 3, False), (300, 2, 3, False), (1000, 4, 4, False)], 300, outlier_frac=0.1, repeat_frac=0.0)
    g = _gpu_vs_oracle(ctx, b, 1.0, 300, 0.99)
    ptr = b["prob_ptr"]
    for i, p in enumerate(probs):
        assert g["best_sample"][i] >= 0 and g["iterations"][i] < 100
        assert np.abs(g["best_model"][i][:, :3] - p["T"][:, :3]).max() < 1e-8 and _t_close(g["best_model"][i][:, 3], p["T"][:, 3], 1e-8)
        assert np.array_equal(g["inlier_mask"][ptr[i]:ptr[i + 1]].astype(bool), p["inlier"])
        assert g["best_count"][i] == p["inlier"].sum()


@pytest.mark.gpu
def test_gpu_bad_arguments_are_refused(ctx):
    from covins_b200._lib import lib
    b, _ = _batch(5, [(0, 1, 1, False), (57, 3, 3, False), (100, 2, 3, False)], 20)
    keep = []

    def call(n_prob=3, ns=20, max_it=300, per_sample=(False, False, False), **over):
        a = {k: np.ascontiguousarray(v) for k, v in b.items()}
        a.update(over)
        keep.append(a)
        res = {k: np.zeros(s, dt) for k, s, dt in (("bs", 3, np.int32), ("bm", 36, np.float64), ("bc", 3, np.int32), ("it", 3, np.int32),
                                                    ("us", 3, np.int32), ("sm", 3 * 20 * 12, np.float64), ("sv", 60, np.uint8), ("sc", 60, np.int32))}
        keep.append(res)
        ptr = lambda k: a[k].ctypes.data if a[k] is not None else None
        P = PR.CRelRansacProblems(n_prob, *[ptr(k) for k in ("prob_ptr", "f1", "f2", "sigma1", "sigma2", "cam1", "cam2", "cam_ptr1", "cam_off1",
                                                             "cam_rot1", "cam_ptr2", "cam_off2", "cam_rot2", "samples")], ns)
        opt = [res[k].ctypes.data if on else None for k, on in zip(("sm", "sv", "sc"), per_sample)]
        R = PR.CRelRansacResult(res["bs"].ctypes.data, res["bm"].ctypes.data, res["bc"].ctypes.data, res["it"].ctypes.data, res["us"].ctypes.data,
                                None, *opt)
        return lib().cvb_ransac_noncentral_relative_pose_batch(ctx.handle, C.byref(P), 9.0, max_it, 0.99, C.byref(R))

    assert call() == 0 and call(per_sample=(True, True, True)) == 0
    assert call(n_prob=0) == 0
    assert call(per_sample=(True, False, True)) == 1 and call(per_sample=(False, False, True)) == 1
    bad = b["samples"].copy(); bad[1, 7, 2] = 57
    assert call(samples=bad) == 1
    bad = b["samples"].copy(); bad[2, 0, 0] = -1
    assert call(samples=bad) == 1
    assert call(n_prob=-1) == 1 and call(ns=-1) == 1 and call(max_it=-1) == 1
    assert call(f1=None) == 1 and call(cam2=None) == 1 and call(samples=None) == 1 and call(cam_rot1=None) == 1 and call(prob_ptr=None) == 1
    assert call(cam_ptr2=None) == 1
    assert call(prob_ptr=np.array([0, 57, 50, 157], np.int32)) == 1
    assert call(cam_ptr1=np.array([0, 1, 0, 6], np.int32)) == 1
    bad = b["cam1"].copy(); bad[60] = 2                                             # rig 1 of problem 2 has 2 cameras
    assert call(cam1=bad) == 1
    bad = b["cam2"].copy(); bad[157 - 1] = -1
    assert call(cam2=bad) == 1
    # a rig of 9 cameras (the cap is CVB_REL_MAX_CAMS = 8)
    big = np.array([0, 1, 10, 12], np.int32)
    assert call(cam_ptr1=big, cam_off1=np.zeros((12, 3)), cam_rot1=np.tile(np.eye(3), (12, 1, 1))) == 1
    assert lib().cvb_ransac_noncentral_relative_pose_batch(ctx.handle, None, 9.0, 300, 0.99, None) == 1


# ------------------------------------------------------------------------------------------------- C++ wrapper
def _build_shim(out):
    import covins_b200
    if not os.path.exists(covins_b200.LIB_PATH):
        covins_b200.build()
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-o", out, os.path.join(ROOT, "tests", "cpp", "shim_ransac_rel_test.cpp"),
                           "-L" + os.path.join(ROOT, "covins_b200"), "-lcovins_b200", "-Wl,-rpath," + os.path.join(ROOT, "covins_b200")])


def test_shim_ransac_rel_compiles_and_links(tmp_path):
    exe = str(tmp_path / "shim_ransac_rel_test")
    _build_shim(exe)
    assert os.path.exists(exe)


@pytest.mark.gpu
def test_shim_ransac_rel_equals_python_path(ctx, tmp_path):
    exe = str(tmp_path / "shim_ransac_rel_test")
    _build_shim(exe)
    b, _ = _batch(9, [(300, 3, 3, False), (0, 1, 1, False), (1000, 2, 4, False), (17, 1, 2, False)], 120, outlier_frac=0.1)
    for k, v in b.items():
        np.ascontiguousarray(v).tofile(tmp_path / f"{k}.bin")
    np.array([9.0, 100.0, 0.99]).tofile(tmp_path / "params.bin")
    subprocess.check_call([exe, str(tmp_path)])
    g = PR.ransac_noncentral_relative_pose(ctx, **b, threshold=9.0, max_iterations=100, probability=0.99)
    ints = np.fromfile(tmp_path / "out_ints.bin", np.int32).reshape(-1, 4)
    assert np.array_equal(ints, np.stack([g["best_sample"], g["best_count"], g["iterations"], g["consumed"]], 1))
    assert np.array_equal(np.fromfile(tmp_path / "out_models.bin").reshape(-1, 3, 4), g["best_model"])
    assert np.array_equal(np.fromfile(tmp_path / "out_mask.bin", np.uint8), g["inlier_mask"])
    assert (g["best_sample"][[0, 2]] >= 0).all()
