"""Seeded samples: the RANSAC and covariance calls with their samples drawn on the GPU from one seed per problem
(cvb_ransac_*_seeded_batch, cvb_noncentral_relative_pose_covariance_seeded_batch).
CPU: the C sampler's Philox4x64-10 against numpy.random.Philox and the known answer, its subset rule against a numpy
restatement with an explicit permutation, distinct in-range indices, uniform index frequencies, and each seeded oracle against
its sample-supplied oracle fed the samples it drew.  GPU: every output of the four calls is bit-identical to the seeded oracle
and to the sample-supplied call given the drawn samples; problems with too few correspondences draw nothing; all-invalid
problems end at opengv's skip limit; invalid samples ahead of a valid one are skipped; a problem gives the same bits alone and in
a batch; bad arguments are refused before any launch; the C++ wrapper's seeded overloads equal the Python path."""
import ctypes as C
import subprocess

import numpy as np
import pytest

from covins_b200 import placerec as PR
from oracle import ransac as orr
from oracle import ransac_rel as orel
from oracle import ransac_rel5 as orel5
from oracle import relpose_cov as ocov
from oracle import seeded as osd
import test_ransac_absolute as TA
import test_ransac_central as TC
import test_ransac_relative as TR
import test_relpose_covariance as TV
from ransac_helpers import _build_shim


# ------------------------------------------------------------------------------------------------- sampler (CPU)
def test_philox_known_answer():
    got = osd.philox([0, 0], [0, 0, 0, 0])
    assert [int(x) for x in got] == [0x16554d9eca36314c, 0xdb20fe9d672d0fdc, 0xd7e772cee186176b, 0x7e68b68aec7ba23b]


def test_philox_equals_numpy():
    rng = np.random.default_rng(0)
    for t in range(20):
        k = rng.integers(0, 2**64 - 1, 2, dtype=np.uint64, endpoint=True)
        c = rng.integers(0, 2**64 - 1, 4, dtype=np.uint64, endpoint=True)
        if t == 0:
            c[0] = np.uint64(2**64 - 1)                                   # the increment carries into the next word
        key = int(k[0]) | (int(k[1]) << 64)
        cnt = sum(int(c[i]) << (64 * i) for i in range(4))
        # numpy's first block is for the given counter plus one
        want = np.random.Philox(key=key, counter=cnt).random_raw(4)
        nxt = (cnt + 1) % 2**256
        assert np.array_equal(osd.philox(k, [(nxt >> (64 * i)) & (2**64 - 1) for i in range(4)]), want), t


def _numpy_subset(seed, stream, m, k, s, perm):
    """the subset rule with an explicit m-length permutation (restored afterwards) and numpy's Philox for the stream"""
    u = []
    for b in range((k + 7) // 8):
        words = np.random.Philox(key=int(seed) | (int(stream) << 64), counter=(s + (b << 64) - 1) % 2**256).random_raw(4)
        for w in words:
            u += [int(w) & 0xffffffff, int(w) >> 32]
    out, swaps = [], []
    for i in range(k):
        j = i + ((u[i] * (m - i)) >> 32)
        perm[i], perm[j] = perm[j], perm[i]
        swaps.append((i, j))
        out.append(int(perm[i]))
    for i, j in reversed(swaps):
        perm[i], perm[j] = perm[j], perm[i]
    return out


def test_subset_rule_equals_numpy_restatement():
    for k in (4, 5, 17):
        for m in (k, k + 1, 1000, 2**20):
            perm = np.arange(m)
            for seed, stream in ((0, 0), (12345, 1), (2**64 - 1, 0)):
                got = osd.samples(seed, stream, m, k, 12, s0=3)
                for t in range(12):
                    assert got[t].tolist() == _numpy_subset(seed, stream, m, k, 3 + t, perm), (k, m, seed, t)


def test_samples_are_distinct_and_in_range():
    for k in (4, 5, 17):
        for m in (k, k + 1, 40, 1000, 2**31 - 1):
            s = osd.samples(99, 0, m, k, 2000)
            assert s.min() >= 0 and s.max() < m
            assert all(len(set(r)) == k for r in s.tolist()), (k, m)
        assert sorted(osd.samples(5, 1, k, k, 1)[0].tolist()) == list(range(k))   # m = k: a permutation


def test_index_frequencies_are_uniform():
    # 10^5 fixed-seed samples: each index's count in every position is within 10 % of N / m (about 4.5 standard deviations), and
    # its count over all positions within 5 % of k N / m
    N, m = 100_000, 50
    for k in (4, 5, 17):
        s = osd.samples(2024, 0, m, k, N)
        per_pos = np.stack([np.bincount(s[:, i], minlength=m) for i in range(k)])
        assert np.abs(per_pos / (N / m) - 1).max() < 0.10, k
        assert np.abs(per_pos.sum(0) / (k * N / m) - 1).max() < 0.05, k


# ------------------------------------------------------------------------------------------------- the four calls
def _drop_samples(b):
    return {k: v for k, v in b.items() if k != "samples"}


def _abs_batch(seed, sizes, outlier):
    b, _ = TA._batch(seed, sizes, 10, outlier_frac=outlier)
    return _drop_samples(b)


def _rel_batch(seed, sizes, outlier):
    b, _ = TR._batch(seed, [(n, 3, 3, False) for n in sizes], 1, outlier_frac=outlier)
    return _drop_samples(b)


def _central_batch(seed, sizes, outlier):
    b, _ = TC._batch(seed, [(n, outlier, False) for n in sizes], 1)
    return _drop_samples(b)


# kind: (sample size, batch builder, bearing key, GPU seeded, GPU supplied, seeded oracle, supplied oracle, threshold)
KINDS = {
    "absolute": (4, _abs_batch, "bearings", PR.ransac_absolute_pose_seeded, PR.ransac_absolute_pose, osd.ransac_absolute_pose_seeded,
                 orr.ransac_absolute_pose, 25.0),
    "noncentral": (17, _rel_batch, "f2", PR.ransac_noncentral_relative_pose_seeded, PR.ransac_noncentral_relative_pose,
                   osd.ransac_noncentral_relative_pose_seeded, orel.ransac_noncentral_relative_pose, 9.0),
    "central": (5, _central_batch, "f2", PR.ransac_central_relative_pose_seeded, PR.ransac_central_relative_pose,
                osd.ransac_central_relative_pose_seeded, orel5.ransac_central_relative_pose, 9.0),
}


def _spoil(b, key, prob, frac, rng):
    """bearings of problem prob set to NaN: all of them (frac 1: every sample invalid) or a share (invalid samples in between)"""
    lo, hi = b["prob_ptr"][prob], b["prob_ptr"][prob + 1]
    f = b[key].copy()
    idx = np.arange(lo, hi) if frac >= 1 else lo + np.flatnonzero(rng.random(hi - lo) < frac)
    f[idx] = np.nan
    b[key] = f


def _scene(kind, seed, n_prob, outlier):
    """n_prob problems of 20-300 correspondences; with n_prob >= 8 also n = k, n < k, n = 0, an all-invalid problem and one with
    invalid bearings (30 %; 5 % for the 17-point solver, whose samples would otherwise almost never be valid)"""
    k, build, key = KINDS[kind][:3]
    rng = np.random.default_rng(seed)
    sizes = [int(x) for x in rng.integers(max(20, k + 3), 300, n_prob)]
    if n_prob >= 8:
        sizes[1], sizes[2], sizes[3] = k, k - 1, 0
    b = build(seed, sizes, outlier)
    if n_prob >= 8:
        _spoil(b, key, 4, 1.0, rng)
        _spoil(b, key, 5, 0.3 if k < 17 else 0.05, rng)
    seeds = rng.integers(0, 2**64 - 1, n_prob, dtype=np.uint64, endpoint=True)
    return b, seeds, sizes


def _bytes_equal(a, b, keys=None):
    for k in keys or b:
        assert np.array_equal(np.ascontiguousarray(a[k]).view(np.uint8), np.ascontiguousarray(b[k]).view(np.uint8)), k


def test_seeded_oracles_equal_supplied_oracles_fed_drawn():
    for kind, (k, _, _, _, _, seeded, supplied, thr) in KINDS.items():
        b, seeds, sizes = _scene(kind, 1, 8, 0.3)
        for max_it in (0, 1, 30):
            ns = max(11 * max_it, 1)
            r = seeded(**b, seeds=seeds, threshold=thr, max_iterations=max_it, per_sample=True, n_samples=ns, want_drawn=True)
            keep = [i for i, n in enumerate(sizes) if n >= k]
            smp = np.where(r["drawn"] >= 0, r["drawn"], 0)
            want = supplied(**b, samples=smp, threshold=thr, max_iterations=max_it, per_sample=True)
            for key in want:
                if key == "inlier_mask":
                    assert np.array_equal(r[key], want[key]), (kind, key)
                else:
                    assert np.array_equal(r[key][keep], want[key][keep]), (kind, max_it, key)
            small = [i for i, n in enumerate(sizes) if n < k]
            assert (r["drawn"][small] == -1).all() and not r["iterations"][small].any() and not r["consumed"][small].any()
            assert (r["best_sample"][small] == -1).all()
            if max_it:
                assert r["consumed"][4] == 10 * max_it and r["iterations"][4] == 0 and r["best_sample"][4] == -1, kind
    # the covariance
    b, probs = TV._batch(3, [(200, 3, 3, False), (150, 2, 3, False), (16, 2, 2, False), (120, 3, 3, False)], 1, outlier_frac=0.2)
    b = _drop_samples(b)
    mask = np.concatenate([p["inlier"] for p in probs]).astype(np.uint8)
    ref = TV._truth(probs); ref[3] = 0.0
    r = osd.relative_pose_covariance_seeded(**b, inlier_mask=mask, seeds=[1, 2, 3, 4], ref_model=ref, n_samples=60, per_sample=True, want_drawn=True)
    want = ocov.noncentral_relative_pose_covariance(**b, samples=np.where(r["drawn"] >= 0, r["drawn"], 0), ref_model=np.r_[ref[:2], 0 * ref[2:]],
                                                    per_sample=True)
    _bytes_equal(r, want)
    assert (r["n_valid"][:2] == 60).all() and not r["n_valid"][2:].any() and (r["drawn"][2:] == -1).all()


# ------------------------------------------------------------------------------------------------- GPU
def _check_seeded(ctx, kind, b, seeds, sizes, max_it, prob=0.99, n_samples=130):
    k, _, _, gpu, gpu_supplied, oracle, _, thr = KINDS[kind]
    kw = dict(threshold=thr, max_iterations=max_it, probability=prob)
    # every output, per-sample ones and the drawn samples included, against the seeded oracle; with and without the per-sample
    # outputs (without them the kernel stops at the bound, and only the waves it reached are drawn)
    for per_sample in (True, False):
        g = gpu(ctx, **b, seeds=seeds, **kw, per_sample=per_sample, n_samples=n_samples, want_drawn=True)
        r = oracle(**b, seeds=seeds, **kw, per_sample=per_sample, n_samples=n_samples, want_drawn=True)
        _bytes_equal(g, r)
    small = [i for i, n in enumerate(sizes) if n < k]
    assert not g["iterations"][small].any() and not g["consumed"][small].any() and (g["best_sample"][small] == -1).all()
    assert (g["drawn"][small] == -1).all()
    # against the sample-supplied call given the drawn samples, with enough of them that it cannot run out
    ns = max(11 * max_it, 1)
    full = gpu(ctx, **b, seeds=seeds, **kw, per_sample=True, n_samples=ns, want_drawn=True)
    keep = [i for i, n in enumerate(sizes) if n >= k]
    sup = gpu_supplied(ctx, **b, samples=np.where(full["drawn"] >= 0, full["drawn"], 0), **kw, per_sample=True)
    for key in sup:
        if key == "inlier_mask":
            assert np.array_equal(full[key], sup[key])
        else:
            _bytes_equal({key: full[key][keep]}, {key: sup[key][keep]})
    for key in ("best_sample", "best_model", "best_count", "iterations", "consumed", "inlier_mask"):
        _bytes_equal({key: full[key]}, {key: g[key]})
    return g


@pytest.mark.gpu
@pytest.mark.parametrize("kind", list(KINDS))
def test_gpu_seeded_equals_oracle_and_supplied_call(ctx, kind):
    k = KINDS[kind][0]
    for n_prob, outlier, max_its in ((1, 0.05, (300,)), (8, 0.3, (0, 1, 300)), (32, 0.5, (300,)), (60, 0.05, (1, 300))):
        b, seeds, sizes = _scene(kind, 10 + n_prob, n_prob, outlier)
        for max_it in max_its:
            g = _check_seeded(ctx, kind, b, seeds, sizes, max_it)
            if n_prob >= 8 and max_it:
                # every hypothesis invalid: opengv's skip limit, which needs more samples than max_iterations plus headroom
                assert g["consumed"][4] == 10 * max_it and g["iterations"][4] == 0 and g["best_sample"][4] == -1
    if kind == "noncentral":                                                    # a rig whose cameras share one centre: rank-deficient
        b, _ = TR._batch(5, [(200, 3, 3, True), (200, 3, 3, False)], 1, outlier_frac=0.05)
        g = _check_seeded(ctx, kind, _drop_samples(b), np.array([7, 8], np.uint64), [200, 200], 20)
        assert g["consumed"][0] == 200 and g["iterations"][0] == 0 and g["best_sample"][0] == -1 and g["best_sample"][1] >= 0
    # n_prob = 0
    b, seeds, sizes = _scene(kind, 3, 1, 0.3)
    b0 = {key: (v[:1] if "ptr" in key else v[:0]) for key, v in b.items()}
    g = KINDS[kind][3](ctx, **b0, seeds=np.zeros(0, np.uint64), threshold=9.0, max_iterations=300, n_samples=10, want_drawn=True)
    assert len(g["best_sample"]) == 0 and g["drawn"].shape == (0, 10, k)


def _invalid_first_problem(kind):
    """one outlier-free problem with 20 % NaN bearings and a seed whose sample 0 holds a NaN index and sample 1 none: the
    selection must skip sample 0 and select sample 1"""
    k, build, key = KINDS[kind][:3]
    b = build(41, [200], 0.0)
    rng = np.random.default_rng(41)
    _spoil(b, key, 0, 0.2, rng)
    bad = ~np.isfinite(b[key]).all(1)
    seed = next(s for s in range(1000) if bad[osd.samples(s, 0, 200, k, 2)[0]].any() and not bad[osd.samples(s, 0, 200, k, 2)[1]].any())
    return b, np.array([seed], np.uint64)


def test_oracle_seeded_skips_invalid_samples_ahead_of_valid_ones():
    for kind, (k, _, _, _, _, oracle, _, thr) in KINDS.items():
        b, seeds = _invalid_first_problem(kind)
        r = oracle(**b, seeds=seeds, threshold=thr, max_iterations=1)
        assert (r["consumed"][0], r["iterations"][0], r["best_sample"][0]) == (2, 1, 1), kind


@pytest.mark.gpu
@pytest.mark.parametrize("kind", list(KINDS))
def test_gpu_seeded_skips_invalid_samples_ahead_of_valid_ones(ctx, kind):
    # the selection reads more samples than max_iterations and still selects a model
    b, seeds = _invalid_first_problem(kind)
    g = _check_seeded(ctx, kind, b, seeds, [200], 1)
    assert (g["consumed"][0], g["iterations"][0], g["best_sample"][0]) == (2, 1, 1)
    assert g["best_count"][0] > 0


@pytest.mark.gpu
@pytest.mark.parametrize("kind", list(KINDS))
def test_gpu_seeded_problem_alone_equals_batch(ctx, kind):
    _, _, _, gpu, _, _, _, thr = KINDS[kind]
    b, seeds, sizes = _scene(kind, 77, 32, 0.3)
    kw = dict(threshold=thr, max_iterations=300, n_samples=64, want_drawn=True)
    g = gpu(ctx, **b, seeds=seeds, **kw)
    ptr = b["prob_ptr"]
    for i in range(32):
        one = {}
        for key, v in b.items():
            if key == "prob_ptr":
                one[key] = np.array([0, ptr[i + 1] - ptr[i]], np.int32)
            elif key in ("cam_off", "cam_rot"):
                one[key] = v[i:i + 1]
            elif key in ("cam_ptr1", "cam_ptr2"):
                one[key] = np.array([0, v[i + 1] - v[i]], np.int32)
            elif key in ("cam_off1", "cam_rot1", "cam_off2", "cam_rot2"):
                cp = b["cam_ptr1" if key.endswith("1") else "cam_ptr2"]
                one[key] = v[cp[i]:cp[i + 1]]
            else:
                one[key] = v[ptr[i]:ptr[i + 1]]
        a = gpu(ctx, **one, seeds=seeds[i:i + 1], **kw)
        for key in a:
            want = g[key][ptr[i]:ptr[i + 1]] if key == "inlier_mask" else g[key][i:i + 1]
            _bytes_equal({key: a[key]}, {key: want})


@pytest.mark.gpu
def test_gpu_seeded_covariance(ctx):
    specs = [(300, 3, 3, False), (16, 2, 2, False), (200, 2, 3, False), (17, 2, 2, False), (400, 3, 3, False)]
    b, probs = TV._batch(21, specs, 1, outlier_frac=0.3)
    b = _drop_samples(b)
    mask = np.concatenate([p["inlier"] for p in probs]).astype(np.uint8)
    mask[300 + 16 + 200:300 + 16 + 200 + 17] = 1                                 # problem 3: exactly 17 inliers
    ref = TV._truth(probs); ref[2] = 0.0
    seeds = np.array([11, 12, 13, 14, 2**64 - 1], np.uint64)
    for ns in (0, 1, 300):
        for per_sample in (True, False):
            g = PR.relative_pose_covariance_seeded(ctx, **b, inlier_mask=mask, seeds=seeds, ref_model=ref, n_samples=ns, per_sample=per_sample,
                                                   want_drawn=True)
            r = osd.relative_pose_covariance_seeded(**b, inlier_mask=mask, seeds=seeds, ref_model=ref, n_samples=ns, per_sample=per_sample,
                                                    want_drawn=True)
            _bytes_equal(g, r)
    assert g["n_valid"][0] > 250 and g["n_valid"][4] > 250 and g["n_valid"][3] > 0 and not g["n_valid"][[1, 2]].any()
    assert (g["drawn"][[1, 2]] == -1).all()
    ptr = b["prob_ptr"]
    for i in (0, 3, 4):                                                         # every drawn index is an inlier
        assert mask[ptr[i] + g["drawn"][i]].all()
    # the sample-supplied call given the drawn samples (the skipped problems have a zero reference there)
    ref_sup = ref.copy(); ref_sup[1] = 0.0
    g = PR.relative_pose_covariance_seeded(ctx, **b, inlier_mask=mask, seeds=seeds, ref_model=ref, n_samples=300, per_sample=True, want_drawn=True)
    sup = PR.relative_pose_covariance(ctx, **b, samples=np.where(g["drawn"] >= 0, g["drawn"], 0), ref_model=ref_sup, per_sample=True)
    _bytes_equal({k: g[k] for k in sup}, sup)
    # one problem alone gives the bits it gets in the batch
    i, lo, hi = 4, ptr[4], ptr[5]
    cp1, cp2 = b["cam_ptr1"], b["cam_ptr2"]
    one = dict(prob_ptr=np.array([0, hi - lo], np.int32), f1=b["f1"][lo:hi], f2=b["f2"][lo:hi], cam1=b["cam1"][lo:hi], cam2=b["cam2"][lo:hi],
               cam_ptr1=np.array([0, cp1[i + 1] - cp1[i]], np.int32), cam_off1=b["cam_off1"][cp1[i]:cp1[i + 1]], cam_rot1=b["cam_rot1"][cp1[i]:cp1[i + 1]],
               cam_ptr2=np.array([0, cp2[i + 1] - cp2[i]], np.int32), cam_off2=b["cam_off2"][cp2[i]:cp2[i + 1]], cam_rot2=b["cam_rot2"][cp2[i]:cp2[i + 1]])
    a = PR.relative_pose_covariance_seeded(ctx, **one, inlier_mask=mask[lo:hi], seeds=seeds[4:], ref_model=ref[4:], n_samples=300, per_sample=True,
                                           want_drawn=True)
    _bytes_equal(a, {k: v[4:] for k, v in g.items()})


@pytest.mark.gpu
def test_gpu_seeded_ransac_feeds_seeded_covariance(ctx):
    b, probs = TR._batch(31, [(400, 3, 3, False), (300, 2, 3, False)], 1, outlier_frac=0.05)
    b = _drop_samples(b)
    seeds = np.array([5, 6], np.uint64)
    g = PR.ransac_noncentral_relative_pose_seeded(ctx, **b, seeds=seeds, threshold=9.0, max_iterations=300)
    assert (g["best_sample"] >= 0).all()
    cov_args = {k: v for k, v in b.items() if k not in ("sigma1", "sigma2")}
    c = PR.relative_pose_covariance_seeded(ctx, **cov_args, inlier_mask=g["inlier_mask"], seeds=seeds, ref_model=g["best_model"], n_samples=300)
    assert (c["n_valid"] > 200).all()
    for m in c["cov"]:
        assert np.array_equal(m, m.T)


@pytest.mark.gpu
def test_gpu_seeded_bad_arguments_are_refused(ctx):
    from covins_b200._lib import lib
    L = lib()
    b, seeds, _ = _scene("absolute", 2, 3, 0.3)
    ptr = b["prob_ptr"]; N = int(ptr[-1])
    keep = []

    def arr(x, dt):
        a = np.ascontiguousarray(x, dt); keep.append(a); return a.ctypes.data

    res = [arr(np.zeros(s, dt), dt) for s, dt in ((3, np.int32), (36, np.float64), (3, np.int32), (3, np.int32), (3, np.int32))]
    R = PR.CRansacResult(*res, None, None, None, None)
    smp = arr(np.zeros((3, 4, 17), np.int32), np.int32)
    sd = arr(seeds, np.uint64)
    launches = ctx.launch_count()

    def abs_call(samples=None, seed=sd, n_prob=3):
        P = PR.CAbsRansacProblems(n_prob, arr(ptr, np.int32), arr(b["pts"], np.float64), arr(b["bearings"], np.float64), arr(b["sigma"], np.float64),
                                  arr(b["cam_off"], np.float64), arr(b["cam_rot"], np.float64), samples, 4)
        return L.cvb_ransac_absolute_pose_seeded_batch(ctx.handle, C.byref(P), seed, 25.0, 300, 0.99, C.byref(R), None)

    assert abs_call(samples=smp) == 1 and abs_call(seed=None) == 1 and abs_call(samples=smp, n_prob=0) == 1
    assert abs_call(seed=None, n_prob=0) == 0
    rb, rseeds, _ = _scene("noncentral", 2, 3, 0.3)
    rel = [arr(rb[k], np.int32 if k in ("prob_ptr", "cam1", "cam2", "cam_ptr1", "cam_ptr2") else np.float64)
           for k in ("prob_ptr", "f1", "f2", "sigma1", "sigma2", "cam1", "cam2", "cam_ptr1", "cam_off1", "cam_rot1", "cam_ptr2", "cam_off2", "cam_rot2")]
    for samples, seed in ((smp, sd), (None, None)):
        P = PR.CRelRansacProblems(3, *rel, samples, 4)
        assert L.cvb_ransac_noncentral_relative_pose_seeded_batch(ctx.handle, C.byref(P), seed, 9.0, 300, 0.99, C.byref(R), None) == 1
        P = PR.CCentralRelRansacProblems(3, *rel[:5], samples, 4)
        assert L.cvb_ransac_central_relative_pose_seeded_batch(ctx.handle, C.byref(P), seed, 9.0, 300, 0.99, C.byref(R), None) == 1
    cov = arr(np.zeros((3, 36)), np.float64); nv = arr(np.zeros(3, np.int32), np.int32)
    CR = PR.CRelCovResult(cov, nv, None, None)
    ref = arr(np.zeros((3, 12)), np.float64)
    mask = arr(np.ones(int(rb["prob_ptr"][-1]), np.uint8), np.uint8)
    for samples, m, seed in ((smp, mask, sd), (None, None, sd), (None, mask, None)):
        P = PR.CRelRansacProblems(3, *rel, samples, 4)
        assert L.cvb_noncentral_relative_pose_covariance_seeded_batch(ctx.handle, C.byref(P), ref, m, seed, C.byref(CR), None) == 1
    assert ctx.launch_count() == launches                                        # refused before any launch
    P = PR.CRelRansacProblems(3, *rel, None, 4)
    assert L.cvb_noncentral_relative_pose_covariance_seeded_batch(ctx.handle, C.byref(P), ref, mask, sd, C.byref(CR), None) == 0
    assert N > 0


# ------------------------------------------------------------------------------------------------- C++ wrapper
def _run_shim(tmp_path, mode, b, seeds, params):
    """tests/cpp/shim_seeded_test <mode> on the batch b (its samples are not passed: the seeded forms take none)"""
    tmp_path.mkdir(exist_ok=True)
    exe = str(tmp_path / "shim_seeded_test")
    _build_shim("shim_seeded_test.cpp", exe)
    for key, v in _drop_samples(b).items():
        np.ascontiguousarray(v).tofile(tmp_path / f"{key}.bin")
    np.ascontiguousarray(seeds, np.uint64).tofile(tmp_path / "seeds.bin")
    np.array(params, np.float64).tofile(tmp_path / "params.bin")
    subprocess.check_call([exe, mode, str(tmp_path)])


def _check_shim_ransac(tmp_path, g):
    ints = np.fromfile(tmp_path / "seeded_ints.bin", np.int32).reshape(-1, 4)
    assert np.array_equal(ints, np.stack([g["best_sample"], g["best_count"], g["iterations"], g["consumed"]], 1))
    assert np.array_equal(np.fromfile(tmp_path / "seeded_models.bin").reshape(-1, 3, 4), g["best_model"])
    assert np.array_equal(np.fromfile(tmp_path / "seeded_mask.bin", np.uint8), g["inlier_mask"])


def test_shim_seeded_compiles_and_links(tmp_path):
    exe = str(tmp_path / "shim_seeded_test")
    _build_shim("shim_seeded_test.cpp", exe)
    assert subprocess.run([exe, "abs", str(tmp_path)]).returncode == 2        # nothing dumped: refused before any GPU work


@pytest.mark.gpu
def test_shim_seeded_ransac_equals_python_path(ctx, tmp_path):
    seeds = np.array([3, 2**64 - 1, 12345, 7], np.uint64)
    b, _ = TA._batch(9, [57, 0, 1000, 4], 20)
    _run_shim(tmp_path / "abs", "abs", b, seeds, [25.0, 300.0, 0.99])
    g = PR.ransac_absolute_pose_seeded(ctx, **_drop_samples(b), seeds=seeds, threshold=25.0, max_iterations=300)
    _check_shim_ransac(tmp_path / "abs", g)
    assert (g["best_sample"][[0, 2]] >= 0).all() and g["best_sample"][1] == -1 and g["consumed"][1] == 0
    b, _ = TR._batch(9, [(300, 3, 3, False), (0, 1, 1, False), (1000, 2, 4, False), (17, 1, 2, False)], 20, outlier_frac=0.05)
    _run_shim(tmp_path / "rel", "rel", b, seeds, [9.0, 100.0, 0.99])
    g = PR.ransac_noncentral_relative_pose_seeded(ctx, **_drop_samples(b), seeds=seeds, threshold=9.0, max_iterations=100)
    _check_shim_ransac(tmp_path / "rel", g)
    assert (g["best_sample"][[0, 2]] >= 0).all()
    b, _ = TC._batch(9, [(300, 0.3, False), (0, 0.0, False), (1000, 0.1, False), (5, 0.0, False)], 20)
    _run_shim(tmp_path / "rel5", "rel5", b, seeds, [9.0, 100.0, 0.99])
    g = PR.ransac_central_relative_pose_seeded(ctx, **_drop_samples(b), seeds=seeds, threshold=9.0, max_iterations=100)
    _check_shim_ransac(tmp_path / "rel5", g)
    assert (g["best_sample"][[0, 2]] >= 0).all()


@pytest.mark.gpu
def test_shim_seeded_covariance_equals_python_path(ctx, tmp_path):
    b, _ = TV._batch(26, [(800, 3, 3, False), (0, 1, 1, False), (600, 2, 4, False), (500, 3, 2, False)], 20, noise=1e-3, outlier_frac=0.05)
    seeds = np.array([11, 12, 13, 14], np.uint64)
    _run_shim(tmp_path, "cov", b, seeds, [9.0, 200.0, 0.99])
    bs = _drop_samples(b)
    g = PR.ransac_noncentral_relative_pose_seeded(ctx, **bs, seeds=seeds, threshold=9.0, max_iterations=200)
    c = PR.relative_pose_covariance_seeded(ctx, **{k: v for k, v in bs.items() if k not in ("sigma1", "sigma2")}, inlier_mask=g["inlier_mask"],
                                           seeds=seeds, ref_model=g["best_model"], n_samples=300)
    assert np.array_equal(np.fromfile(tmp_path / "seeded_models.bin").reshape(-1, 3, 4), g["best_model"])
    assert np.array_equal(np.fromfile(tmp_path / "seeded_cov.bin").reshape(-1, 6, 6), c["cov"])
    assert np.array_equal(np.fromfile(tmp_path / "seeded_n_valid.bin", np.int32), c["n_valid"])
    assert c["n_valid"][1] == 0 and (c["n_valid"][[0, 2, 3]] > 250).all()
