"""Sampling-based 6x6 covariance of the non-central relative pose from caller-supplied 17-point samples
(cvb_noncentral_relative_pose_covariance_batch).
CPU: the oracle's deviation against scipy's quaternion, noise-free and noisy scenes, the covariance against numpy's second
moment over the oracle's per-sample deviations, exact symmetry and PSD, the noise-squared scaling, and the samples that are
invalid.  GPU: the C-ABI call is bit-identical to the oracle (per-sample outputs included) and repeatable, a batch of more than
65535 problems works, the RANSAC-to-covariance pipeline gives a positive-definite covariance, bad arguments are refused, and
the C++ wrapper equals the Python path and feeds PoseGraphOptimization's COVINS_G loop edges."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from covins_b200 import placerec as PR
from oracle import relpose_cov as ocov
from ransac_helpers import _build_shim, _rand_rot
from test_ransac_relative import _problem

S = 17


def _batch(seed, specs, n_samples, noise=1e-3, outlier_frac=0.0):
    """specs: (n, nc1, nc2, central) per problem → (arguments of relative_pose_covariance without ref_model, problems).  The samples
    of a problem are drawn from its true inliers (any indices when it has fewer than 17)."""
    rng = np.random.default_rng(seed)
    probs = [_problem(rng, n, a, b, outlier_frac, central, noise=noise) for n, a, b, central in specs]
    samples = np.zeros((len(specs), n_samples, S), np.int32)
    for i, p in enumerate(probs):
        idx = np.flatnonzero(p["inlier"])
        if n_samples == 0:
            continue
        if len(idx) >= S:
            samples[i] = np.stack([rng.choice(idx, S, replace=False) for _ in range(n_samples)])
        elif len(p["f1"]) > 0:
            samples[i] = rng.integers(0, len(p["f1"]), (n_samples, S))
    cat = lambda k, shape: np.concatenate([p[k] for p in probs]) if probs else np.zeros(shape)
    ptr = lambda k: np.concatenate([[0], np.cumsum([len(p[k]) for p in probs])]).astype(np.int32)
    b = dict(prob_ptr=ptr("f1"), f1=cat("f1", (0, 3)), f2=cat("f2", (0, 3)), sigma1=cat("s1", 0), sigma2=cat("s2", 0),
             cam1=cat("cam1", 0).astype(np.int32), cam2=cat("cam2", 0).astype(np.int32), cam_ptr1=ptr("c1"), cam_off1=cat("c1", (0, 3)),
             cam_rot1=cat("R1", (0, 3, 3)), cam_ptr2=ptr("c2"), cam_off2=cat("c2", (0, 3)), cam_rot2=cat("R2", (0, 3, 3)), samples=samples)
    return b, probs


def _truth(probs):
    return np.stack([p["T"] for p in probs])


def _scipy_delta(ref, M):
    q = Rotation.from_matrix(ref[:, :3].T @ M[:, :3]).as_quat()   # x y z w
    q = -q if q[3] < 0 else q
    return np.r_[2 * q[:3], M[:, 3] - ref[:, 3]]


# ------------------------------------------------------------------------------------------------- oracle (CPU)
def test_deviation_equals_scipy():
    # Both restatements are exact for an exact rotation; they spread the rounding of R_ref^T R_s (|m^T m - I| of a few 1e-16)
    # over q differently when they take different branches.  Samples near their reference (the covariance's use) agree to
    # 1e-15; arbitrary rotations to 1e-15 plus twice that departure from orthonormality.
    rng = np.random.default_rng(0)
    worst_near, worst_far, branches = 0.0, 0.0, set()
    for k in range(3000):
        ref = np.c_[_rand_rot(rng), rng.normal(0, 2, 3)]
        near = k % 2 == 1
        dR = Rotation.from_rotvec(rng.normal(0, 0.05, 3)).as_matrix() if near else _rand_rot(rng)
        M = np.c_[ref[:, :3] @ dR, ref[:, 3] + rng.normal(0, 0.1, 3)]
        err = np.abs(ocov.deviation(ref, M) - _scipy_delta(ref, M)).max()
        m = ref[:, :3].T @ M[:, :3]
        if near:
            worst_near = max(worst_near, err)
        else:
            worst_far = max(worst_far, err - 2 * np.abs(m.T @ m - np.eye(3)).max())
        branches.add(-1 if np.trace(m) > 0 else int(np.argmax(np.diag(m))))
        assert not ocov.deviation(ref, ref).any()                         # exactly 0 for the reference itself
    assert worst_near < 1e-15 and worst_far < 1e-15 and branches == {-1, 0, 1, 2}, (worst_near, worst_far, branches)


def test_noise_free_scene_gives_zero_covariance():
    b, probs = _batch(1, [(200, 3, 3, False), (300, 3, 3, False), (150, 3, 3, False)], 120, noise=0.0, outlier_frac=0.2)
    r = ocov.noncentral_relative_pose_covariance(**b, ref_model=_truth(probs), per_sample=True)
    assert r["sample_valid"].all() and (r["n_valid"] == 120).all()
    assert np.abs(r["sample_delta"]).max() < 1e-8
    assert np.abs(r["cov"]).max() < 1e-16                                  # about 0: the rounding of the solves only


def test_covariance_equals_numpy_second_moment():
    b, probs = _batch(2, [(400, 3, 3, False), (300, 2, 2, False), (500, 4, 3, False)], 300, noise=1e-3)
    r = ocov.noncentral_relative_pose_covariance(**b, ref_model=_truth(probs), per_sample=True)
    for i in range(len(probs)):
        v = r["sample_valid"][i].astype(bool)
        d = r["sample_delta"][i][v]
        assert r["n_valid"][i] == v.sum() > 250
        assert np.allclose(r["cov"][i], d.T @ d / len(d), rtol=1e-12, atol=0), i
        assert not r["sample_delta"][i][~v].any()
    # the lean call (no per-sample outputs) and the single-thread call give the same bits
    for kw in (dict(), dict(threads=1)):
        lean = ocov.noncentral_relative_pose_covariance(**b, ref_model=_truth(probs), **kw)
        assert np.array_equal(lean["cov"].view(np.uint64), r["cov"].view(np.uint64)) and np.array_equal(lean["n_valid"], r["n_valid"])


def test_covariance_is_exactly_symmetric_and_psd():
    b, probs = _batch(3, [(300, 3, 3, False)] * 6, 300, noise=2e-3, outlier_frac=0.1)
    r = ocov.noncentral_relative_pose_covariance(**b, ref_model=_truth(probs))
    for c in r["cov"]:
        assert np.array_equal(c, c.T)
        w = np.linalg.eigvalsh(c)
        assert w.min() > -1e-12 * w.max() and w.max() > 0


def test_doubling_the_noise_scales_the_diagonal_by_four():
    # The same seed draws the same scene and the same standard-normal perturbations; only their scale doubles.  The minimal
    # 17-point solve amplifies bearing noise strongly (at 1e-6 the median deviation is already ~2e-3 and the largest are O(1)),
    # so the noise is kept at 1e-9 and 2e-9, where every deviation is linear in it: every diagonal ratio lies in [3.9, 4.1].
    ratios = []
    for seed in (4, 5, 7):
        covs = []
        for noise in (1e-9, 2e-9):
            b, probs = _batch(seed, [(400, 3, 3, False), (300, 3, 3, False)], 300, noise=noise)
            covs.append(ocov.noncentral_relative_pose_covariance(**b, ref_model=_truth(probs))["cov"])
        ratios.append(np.diagonal(covs[1], axis1=1, axis2=2) / np.diagonal(covs[0], axis1=1, axis2=2))
    ratios = np.concatenate(ratios)
    assert np.all((ratios > 3.9) & (ratios < 4.1)), ratios


def _invalid_batch(n_samples=40):
    """five problems: repeated indices in every third sample, fewer than 17 correspondences, a non-finite bearing used by some
    samples, central rigs, and a zero reference model → (arguments, reference models, expected valid flags)"""
    b, probs = _batch(6, [(200, 3, 3, False), (16, 2, 2, False), (200, 3, 2, False), (200, 3, 3, True), (200, 2, 3, False)], n_samples)
    ref = _truth(probs)
    expect = np.ones((5, n_samples), bool)
    b["samples"][0, ::3, 16] = b["samples"][0, ::3, 2]
    expect[0, ::3] = False
    expect[1] = False
    bad = 7
    b["f2"][b["prob_ptr"][2] + bad, 1] = np.nan
    expect[2] = ~(b["samples"][2] == bad).any(1)
    expect[3] = False
    ref[4] = 0.0
    expect[4] = False
    return b, ref, expect


def test_invalid_samples_are_skipped():
    b, ref, expect = _invalid_batch()
    r = ocov.noncentral_relative_pose_covariance(**b, ref_model=ref, per_sample=True)
    assert 0 < expect[2].sum() < 40
    assert np.array_equal(r["sample_valid"].astype(bool), expect)
    assert np.array_equal(r["n_valid"], expect.sum(1))
    assert not r["sample_delta"][~expect].any()
    for i in (1, 3, 4):
        assert not r["cov"][i].any()
    for i in (0, 2):
        d = r["sample_delta"][i][expect[i]]
        assert np.allclose(r["cov"][i], d.T @ d / len(d), rtol=1e-12, atol=0)
    # the zero-model problem's samples are not read: out-of-range indices change nothing
    b["samples"][4] = 10 ** 6
    r2 = ocov.noncentral_relative_pose_covariance(**b, ref_model=ref, per_sample=True)
    for k in r:
        assert np.array_equal(r[k], r2[k]), k


# ------------------------------------------------------------------------------------------------- GPU (C-ABI)
def _gpu_vs_oracle(ctx, b, ref):
    g = PR.relative_pose_covariance(ctx, **b, ref_model=ref, per_sample=True)
    r = ocov.noncentral_relative_pose_covariance(**b, ref_model=ref, per_sample=True)
    for k in r:
        assert np.array_equal(g[k].view(np.uint8), r[k].view(np.uint8)), k
    lean = PR.relative_pose_covariance(ctx, **b, ref_model=ref)
    for k in lean:
        assert np.array_equal(lean[k].view(np.uint8), g[k].view(np.uint8)), k
    return g


GPU_SPECS = [(300, 1, 1, False), (300, 2, 3, False), (1000, 3, 3, False), (400, 8, 8, False), (250, 5, 7, False), (16, 2, 2, False),
             (300, 3, 3, True), (300, 4, 4, False), (17, 1, 2, False), (0, 1, 1, False)]


@pytest.mark.gpu
def test_gpu_equals_oracle_bitwise(ctx):
    for ns in (0, 1, 7, 300, 301):
        b, probs = _batch(10 + ns, GPU_SPECS, ns, noise=1e-3)
        ref = _truth(probs)
        ref[7] = 0.0                                                       # a RANSAC without a model: skipped
        g = _gpu_vs_oracle(ctx, b, ref)
        assert g["n_valid"][7] == 0 and not g["cov"][7].any()
        assert (g["n_valid"][[0, 5, 6, 9]] == 0).all()                     # one camera per side, n < 17, central rigs, no correspondences
        if ns >= 7:
            assert (g["n_valid"][[1, 2, 3, 4]] > 0).all()
    # the invalid cases of the CPU test, on the GPU
    b, ref, expect = _invalid_batch(300)
    g = _gpu_vs_oracle(ctx, b, ref)
    assert np.array_equal(g["sample_valid"].astype(bool), expect)
    # two calls give the same bits
    b, probs = _batch(20, GPU_SPECS, 300, noise=2e-3)
    g1 = PR.relative_pose_covariance(ctx, **b, ref_model=_truth(probs), per_sample=True)
    g2 = PR.relative_pose_covariance(ctx, **b, ref_model=_truth(probs), per_sample=True)
    for k in g1:
        assert np.array_equal(g1[k].view(np.uint8), g2[k].view(np.uint8)), k


@pytest.mark.gpu
def test_gpu_more_than_65535_problems(ctx):
    b1, probs = _batch(21, [(40, 2, 3, False), (40, 3, 2, False)], 1, noise=1e-3)
    reps = 32800                                                           # 65600 problems, one sample each
    n1 = np.diff(b1["prob_ptr"]); c1 = np.diff(b1["cam_ptr1"]); c2 = np.diff(b1["cam_ptr2"])
    ptr = lambda counts: np.concatenate([[0], np.cumsum(np.tile(counts, reps))]).astype(np.int32)
    b = dict(prob_ptr=ptr(n1), cam_ptr1=ptr(c1), cam_ptr2=ptr(c2), samples=np.tile(b1["samples"], (reps, 1, 1)))
    for k in ("f1", "f2", "cam1", "cam2", "cam_off1", "cam_rot1", "cam_off2", "cam_rot2"):
        b[k] = np.concatenate([b1[k]] * reps)
    ref = np.tile(_truth(probs), (reps, 1, 1))
    ref[-1] = 0.0
    g = PR.relative_pose_covariance(ctx, **b, ref_model=ref, per_sample=True)
    r = ocov.noncentral_relative_pose_covariance(**b, ref_model=ref, per_sample=True)
    for k in r:
        assert np.array_equal(g[k].view(np.uint8), r[k].view(np.uint8)), k
    assert g["n_valid"][:-1].all() and g["n_valid"][-1] == 0
    assert np.array_equal(g["cov"][-3], g["cov"][1]) and g["cov"][1].any()


@pytest.mark.gpu
def test_gpu_ransac_to_covariance_pipeline(ctx):
    rng = np.random.default_rng(22)
    b, probs = _batch(23, [(1000, 3, 3, False), (500, 2, 3, False), (800, 4, 4, False), (600, 3, 2, False)], 400, noise=1e-3, outlier_frac=0.3)
    # the RANSAC's own samples: any indices
    ptr = b["prob_ptr"]
    b["samples"] = np.stack([np.stack([rng.choice(ptr[i + 1] - ptr[i], S, replace=False) for _ in range(400)]) for i in range(len(probs))])
    g = PR.ransac_noncentral_relative_pose(ctx, **b, threshold=9.0, max_iterations=300)
    assert (g["best_sample"] >= 0).all()
    # 300 covariance samples per problem from its inlier mask
    cov_samples = np.stack([np.stack([rng.choice(np.flatnonzero(g["inlier_mask"][ptr[i]:ptr[i + 1]]), S, replace=False) for _ in range(300)])
                            for i in range(len(probs))]).astype(np.int32)
    bc = dict(b, samples=cov_samples)
    c = _gpu_vs_oracle(ctx, bc, g["best_model"])
    for i in range(len(probs)):
        assert c["n_valid"][i] > 290
        cov = c["cov"][i]
        assert np.array_equal(cov, cov.T)
        L = np.linalg.cholesky(cov)                                        # positive definite
        sqrt_info = np.linalg.cholesky(np.linalg.inv(cov)).T              # LLT(cov^-1).matrixL().transpose()
        assert np.isfinite(L).all() and np.isfinite(sqrt_info).all()


@pytest.mark.gpu
def test_gpu_bad_arguments_are_refused(ctx):
    from covins_b200._lib import lib
    b, probs = _batch(24, [(0, 1, 1, False), (57, 3, 3, False), (100, 2, 3, False)], 20)
    ref0 = _truth(probs)
    keep = []

    def call(n_prob=3, ns=20, per_sample=(False, False), ref=ref0, cov=True, n_valid=True, **over):
        a = {k: np.ascontiguousarray(v) for k, v in b.items()}
        a.update(over)
        keep.append(a)
        res = {k: np.zeros(s, dt) for k, s, dt in (("cov", 3 * 36, np.float64), ("nv", 3, np.int32), ("sd", 3 * 20 * 6, np.float64), ("sv", 60, np.uint8))}
        rf = np.ascontiguousarray(ref, np.float64) if ref is not None else None
        keep.extend([res, rf])
        ptr = lambda k: a[k].ctypes.data if a[k] is not None else None
        P = PR.CRelRansacProblems(n_prob, *[ptr(k) for k in ("prob_ptr", "f1", "f2", "sigma1", "sigma2", "cam1", "cam2", "cam_ptr1", "cam_off1",
                                                             "cam_rot1", "cam_ptr2", "cam_off2", "cam_rot2", "samples")], ns)
        opt = [res[k].ctypes.data if on else None for k, on in zip(("sd", "sv"), per_sample)]
        R = PR.CRelCovResult(res["cov"].ctypes.data if cov else None, res["nv"].ctypes.data if n_valid else None, *opt)
        return lib().cvb_noncentral_relative_pose_covariance_batch(ctx.handle, C.byref(P), rf.ctypes.data if rf is not None else None, C.byref(R))

    assert call() == 0 and call(per_sample=(True, True)) == 0
    assert call(n_prob=0) == 0
    assert call(sigma1=None, sigma2=None) == 0                             # not read
    assert call(per_sample=(True, False)) == 1 and call(per_sample=(False, True)) == 1
    bad = b["samples"].copy(); bad[1, 7, 2] = 57
    assert call(samples=bad) == 1
    bad = b["samples"].copy(); bad[2, 0, 0] = -1
    assert call(samples=bad) == 1
    zero = ref0.copy(); zero[2] = 0.0
    assert call(samples=bad, ref=zero) == 0                                # a skipped problem's samples are not read
    assert call(n_prob=-1) == 1 and call(ns=-1) == 1
    assert call(f1=None) == 1 and call(cam2=None) == 1 and call(samples=None) == 1 and call(cam_rot1=None) == 1 and call(prob_ptr=None) == 1
    assert call(cam_ptr2=None) == 1 and call(ref=None) == 1 and call(cov=False) == 1 and call(n_valid=False) == 1
    assert call(prob_ptr=np.array([0, 57, 50, 157], np.int32)) == 1
    assert call(cam_ptr1=np.array([0, 1, 0, 6], np.int32)) == 1
    bad = b["cam1"].copy(); bad[60] = 2                                    # rig 1 of problem 2 has 2 cameras
    assert call(cam1=bad) == 1
    big = np.array([0, 1, 10, 12], np.int32)                              # a rig of 9 cameras
    assert call(cam_ptr1=big, cam_off1=np.zeros((12, 3)), cam_rot1=np.tile(np.eye(3), (12, 1, 1))) == 1
    for i, v in ((3, np.nan), (11, np.inf)):
        bad = ref0.copy(); bad[1].reshape(-1)[i] = v
        assert call(ref=bad) == 1                                          # not finite
    bad = ref0.copy(); bad[2, :, :3] *= 1.00001
    assert call(ref=bad) == 1                                              # R^T R - I = 2e-5
    ok = ref0.copy(); ok[2, :, :3] *= 1.0000001
    assert call(ref=ok) == 0                                               # 2e-7 is within 1e-6
    assert lib().cvb_noncentral_relative_pose_covariance_batch(ctx.handle, None, None, None) == 1


# ------------------------------------------------------------------------------------------------- C++ wrapper
def test_shim_relpose_cov_compiles_and_links(tmp_path):
    exe = str(tmp_path / "shim_relpose_cov_test")
    _build_shim("shim_relpose_cov_test.cpp", exe)
    assert os.path.exists(exe)


@pytest.mark.gpu
def test_shim_relpose_cov_equals_python_path_and_feeds_pgo(ctx, tmp_path):
    exe = str(tmp_path / "shim_relpose_cov_test")
    _build_shim("shim_relpose_cov_test.cpp", exe)
    rng = np.random.default_rng(25)
    b, probs = _batch(26, [(800, 3, 3, False), (0, 1, 1, False), (600, 2, 4, False), (500, 3, 2, False)], 200, noise=1e-3, outlier_frac=0.2)
    ptr = b["prob_ptr"]
    for i in (0, 2, 3):
        b["samples"][i] = np.stack([rng.choice(ptr[i + 1] - ptr[i], S, replace=False) for _ in range(200)])
    g = PR.ransac_noncentral_relative_pose(ctx, **b, threshold=9.0, max_iterations=200)
    assert g["best_sample"][1] == -1 and (g["best_sample"][[0, 2, 3]] >= 0).all()
    cov_samples = np.zeros((4, 300, S), np.int32)
    for i in (0, 2, 3):
        inl = np.flatnonzero(g["inlier_mask"][ptr[i]:ptr[i + 1]])
        cov_samples[i] = np.stack([rng.choice(inl, S, replace=False) for _ in range(300)])
    for k, v in dict(b, cov_samples=cov_samples).items():
        np.ascontiguousarray(v).tofile(tmp_path / f"{k}.bin")
    np.array([9.0, 200.0, 0.99]).tofile(tmp_path / "params.bin")
    subprocess.check_call([exe, str(tmp_path)])
    c = PR.relative_pose_covariance(ctx, **dict(b, samples=cov_samples), ref_model=g["best_model"])
    assert np.array_equal(np.fromfile(tmp_path / "out_models.bin").reshape(-1, 3, 4), g["best_model"])
    assert np.array_equal(np.fromfile(tmp_path / "out_cov.bin").reshape(-1, 6, 6), c["cov"])
    assert np.array_equal(np.fromfile(tmp_path / "out_n_valid.bin", np.int32), c["n_valid"])
    assert c["n_valid"][1] == 0 and (c["n_valid"][[0, 2, 3]] > 250).all()
    pgo = np.fromfile(tmp_path / "out_pgo.bin")
    assert pgo[-1] == 3 and np.isfinite(pgo).all()                         # three loop edges, no not-PD exit
