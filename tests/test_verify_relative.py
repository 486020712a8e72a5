"""cvb_verify_noncentral_relative_pose_seeded_batch (placerec.verify_noncentral_relative_pose_seeded): the COVINS_G verification
chain of a query keyframe's candidates in one call, against the composed oracle (oracle/verify.py:verify_noncentral_seeded) and
against the chain of the four existing calls with the glue done on the host."""
import ctypes as C
import importlib.util
import os
import subprocess

import numpy as np
import pytest

from covins_b200 import placerec as PR, synth
from oracle import verify as ov
from ransac_helpers import ROOT, _build_shim

PRM = dict(img_match_thres=50.0, ratio_thres=0.8, threshold5=9.0, max_iterations5=300, threshold17=9.0, max_iterations17=300,
           probability=0.99)
CVB_ERR_INVALID = 1
PAIRINGS = [(0, 0), (1, 1), (2, 2), (0, 1), (1, 2), (2, 0)]   # (query camera, candidate camera)


def _small_rot(rng, deg):
    w = rng.normal(0, 1, 3); w *= np.deg2rad(deg) * rng.uniform(0.2, 1.0) / np.linalg.norm(w)
    K = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]]); a = np.linalg.norm(w)
    return np.eye(3) + np.sin(a) / a * K + (1 - np.cos(a)) / a ** 2 * K @ K


def _rig(rng, n_cam=3):
    return rng.normal(0, 0.5, (n_cam, 3)), np.stack([_small_rot(rng, 10) for _ in range(n_cam)])


def _keyframe(rng, X, codes, off, rot, n_kp, lm_frac, outlier, sigma):
    """n_kp rows: a share lm_frac observes random points of X (rig frame) through camera (off, rot), a share `outlier` of those with a
    random bearing; the rest are keypoints without a landmark (random code and bearing)"""
    n_lm = int(round(n_kp * lm_frac))
    ids = rng.choice(len(X), n_lm, replace=False)
    desc = rng.integers(0, 256, (n_kp, 32), dtype=np.uint8)
    f = rng.normal(0, 1, (n_kp, 3))
    slots = rng.permutation(n_kp)[:n_lm]
    desc[slots] = codes[ids] ^ synth._flip_mask(rng, (n_lm, 32))
    f[slots] = (X[ids] - off) @ rot                      # Rc^T (X - c)
    bad = slots[rng.random(n_lm) < outlier]
    f[bad] = rng.normal(0, 1, (len(bad), 3))
    f /= np.linalg.norm(f, axis=1, keepdims=True)
    return desc, f, rng.uniform(*sigma, n_kp)


def scene(seed, n_cand, n_kp=1000, outlier=0.3, lm_frac=0.6, n_pts=1500, sigma=(1e-6, 1e-5), pairings=PAIRINGS):
    """two 3-camera rigs over shared points per candidate: the query rig (keyframes 0-2) and, per candidate, a rig at a random pose
    [R|t] (X1 = R X2 + t, keyframes 3 + 3c ..); outlier: the share of a candidate keyframe's landmark rows with a random bearing.
    → the keyword arguments of verify_noncentral_relative_pose_seeded without PRM, and the true poses"""
    rng = np.random.default_rng(seed)
    d = rng.normal(0, 1, (n_pts, 3)); d[:, 2] = np.abs(d[:, 2]) + 2.0; d /= np.linalg.norm(d, axis=1, keepdims=True)
    X = d * rng.uniform(4, 30, n_pts)[:, None]
    codes = rng.integers(0, 256, (n_pts, 32), dtype=np.uint8)
    off1, rot1 = _rig(rng)
    kfs = [_keyframe(rng, X, codes, off1[j], rot1[j], n_kp, lm_frac, 0.0, sigma) for j in range(3)]
    co2, cr2, poses, pairs, pair_ptr = [], [], [], [], [0]
    for c in range(n_cand):
        R, t = _small_rot(rng, 20), rng.normal(0, 1, 3)
        off2, rot2 = _rig(rng)
        X2 = (X - t) @ R                                  # R^T (X1 - t)
        base = len(kfs)
        kfs += [_keyframe(rng, X2, codes, off2[j], rot2[j], n_kp, lm_frac, outlier, sigma) for j in range(3)]
        co2.append(off2); cr2.append(rot2); poses.append((R, t))
        pairs += [(a, base + b, a, b) for a, b in pairings]
        pair_ptr.append(len(pairs))
    kf_ptr = np.concatenate([[0], np.cumsum([len(k[0]) for k in kfs])]).astype(np.int32)
    S = dict(kf_ptr=kf_ptr, desc=np.concatenate([k[0] for k in kfs]), bearings=np.concatenate([k[1] for k in kfs]),
             sigma=np.concatenate([k[2] for k in kfs]), cam_ptr1=np.arange(n_cand + 1, dtype=np.int32) * 3,
             cam_off1=np.tile(off1, (n_cand, 1)), cam_rot1=np.tile(rot1, (n_cand, 1, 1)), cam_ptr2=np.arange(n_cand + 1, dtype=np.int32) * 3,
             cam_off2=np.concatenate(co2).reshape(-1, 3) if n_cand else np.zeros((0, 3)),
             cam_rot2=np.concatenate(cr2).reshape(-1, 3, 3) if n_cand else np.zeros((0, 3, 3)),
             pair_ptr=np.array(pair_ptr, np.int32), pairs=np.array(pairs, np.int32).reshape(-1, 4),
             seeds5=rng.integers(0, 2**63, len(pairs), dtype=np.uint64), seeds=rng.integers(0, 2**63, n_cand, dtype=np.uint64))
    return S, poses


def _cmp(g, r):
    for k in r:
        a = np.ascontiguousarray(g[k]); b = np.ascontiguousarray(r[k])
        if k in ("best_model", "best_model5", "cov"):
            assert a.shape == b.shape and np.array_equal(a.view(np.uint8), b.astype(np.float64).view(np.uint8)), k
        else:
            assert np.array_equal(np.asarray(a, np.int64), np.asarray(b, np.int64)), k


# --------------------------------------------------------------------------------------------------------------- CPU
def test_oracle_recovers_true_pose_noise_free():
    S, poses = scene(1, 2)
    r = ov.verify_noncentral_seeded(**S, **PRM, n_cov_samples=20)
    assert (r["n_matches"] > 50).all() and (r["best_sample5"] >= 0).all()
    assert (r["corr"][:, 3] == 0).any() and (r["corr"][:, 3] == 1).any()          # the 5-point RANSACs reject the wrong bearings
    for c, (R, t) in enumerate(poses):
        M = r["best_model"][c].reshape(3, 4)
        assert r["best_sample"][c] >= 0 and r["n_valid"][c] > 0
        assert np.abs(M[:, :3] - R).max() < 1e-6 and np.abs(M[:, 3] - t).max() < 1e-6, c


def test_glue_equals_numpy_restatement():
    S, _ = scene(2, 3, n_kp=300)
    kp, P = S["kf_ptr"], S["pairs"]
    rng = np.random.default_rng(0)
    mts = [np.where(rng.random(kp[a + 1] - kp[a]) < 0.3, rng.integers(0, max(kp[b + 1] - kp[b], 1), kp[a + 1] - kp[a]), -1) for a, b, _, _ in P]
    g = ov.gather_matches(kp, S["bearings"], S["sigma"], P, mts)
    # gather: the accepted rows of each pairing in query order
    rows = [np.flatnonzero(m >= 0) for m in mts]
    qa = np.concatenate([kp[a] + r_ for (a, _, _, _), r_ in zip(P, rows)]); tb = np.concatenate([kp[b] + m[r_] for (_, b, _, _), m, r_ in zip(P, mts, rows)])
    assert np.array_equal(g["prob_ptr"], np.concatenate([[0], np.cumsum([len(r_) for r_ in rows])]))
    assert np.array_equal(g["f1"], S["bearings"][qa]) and np.array_equal(g["f2"], S["bearings"][tb])
    assert np.array_equal(g["sigma1"], S["sigma"][qa]) and np.array_equal(g["sigma2"], S["sigma"][tb])
    assert np.array_equal(g["row1"], np.concatenate(rows)) and np.array_equal(g["row2"], np.concatenate([m[r_] for m, r_ in zip(mts, rows)]))
    # merge: per candidate the 5-point inliers of its pairings in order, with the pairing's cameras
    mask5 = (rng.random(len(g["f1"])) < 0.6).astype(np.uint8)
    m = ov.merge_inliers(S["pair_ptr"], P, g, mask5)
    pairing = np.repeat(np.arange(len(P)), np.diff(g["prob_ptr"]))
    cand = np.searchsorted(S["pair_ptr"], pairing, side="right") - 1
    src = np.flatnonzero(mask5)                                                    # pairings are already in candidate order
    assert np.array_equal(m["src"], src)
    assert np.array_equal(m["prob_ptr"], np.concatenate([[0], np.cumsum(np.bincount(cand[src], minlength=len(S["pair_ptr"]) - 1))]))
    assert np.array_equal(m["cam1"], P[pairing[src], 2]) and np.array_equal(m["cam2"], P[pairing[src], 3])
    assert np.array_equal(m["f1"], g["f1"][src]) and np.array_equal(m["sigma2"], g["sigma2"][src])


def test_shim_verify_compiles_and_links(tmp_path):
    exe = str(tmp_path / "shim_verify_test")
    _build_shim("shim_verify_test.cpp", exe)
    assert subprocess.run([exe, str(tmp_path)]).returncode == 2        # nothing dumped: refused before any GPU work


# --------------------------------------------------------------------------------------------------------------- GPU
def _chain():
    spec = importlib.util.spec_from_file_location("verify_timing", os.path.join(ROOT, "tools", "verify_timing.py"))
    mod = importlib.util.module_from_spec(spec); spec.loader.exec_module(mod)
    return mod.chain_existing_calls


@pytest.mark.gpu
@pytest.mark.parametrize("n_cand", [1, 8, 32])
def test_gpu_equals_composed_oracle_bitwise(ctx, n_cand):
    S, _ = scene(10 + n_cand, n_cand)
    g = PR.verify_noncentral_relative_pose_seeded(ctx, **S, **PRM)
    r = ov.verify_noncentral_seeded(**S, **PRM)
    _cmp(g, r)
    assert (g["best_sample"] >= 0).all() and (g["n_valid"] > 0).all()
    c = g["corr"]
    assert (c[:, 3] == 0).any() and (c[:, 4] == 0).any() and (c[:, 4] == 1).any()


@pytest.mark.gpu
@pytest.mark.parametrize("n_cand", [1, 8])
def test_gpu_equals_chain_of_existing_calls(ctx, n_cand):
    S, _ = scene(20 + n_cand, n_cand, outlier=0.05)
    g = PR.verify_noncentral_relative_pose_seeded(ctx, **S, **PRM)
    _cmp(g, _chain()(ctx, S, PRM, 300))


@pytest.mark.gpu
def test_gpu_candidate_alone_equals_batch(ctx):
    S, _ = scene(30, 8)
    g = PR.verify_noncentral_relative_pose_seeded(ctx, **S, **PRM)
    pp = S["pair_ptr"]
    for c in (0, 5, 7):
        a, b = pp[c], pp[c + 1]
        one = dict(S, cam_ptr1=np.array([0, 3], np.int32), cam_off1=S["cam_off1"][3 * c:3 * c + 3], cam_rot1=S["cam_rot1"][3 * c:3 * c + 3],
                   cam_ptr2=np.array([0, 3], np.int32), cam_off2=S["cam_off2"][3 * c:3 * c + 3], cam_rot2=S["cam_rot2"][3 * c:3 * c + 3],
                   pair_ptr=np.array([0, b - a], np.int32), pairs=S["pairs"][a:b], seeds5=S["seeds5"][a:b], seeds=S["seeds"][c:c + 1])
        s = PR.verify_noncentral_relative_pose_seeded(ctx, **one, **PRM)
        for k in ("n_matches", "best_sample5", "best_model5", "best_count5", "iterations5", "consumed5"):
            assert np.array_equal(s[k], g[k][a:b]), k
        for k in ("best_sample", "best_model", "best_count", "iterations", "consumed", "cov", "n_valid"):
            assert np.array_equal(np.ascontiguousarray(s[k]).view(np.uint8), np.ascontiguousarray(g[k][c:c + 1]).view(np.uint8)), k
        sel = (g["corr"][:, 0] >= a) & (g["corr"][:, 0] < b)
        exp = g["corr"][sel].copy(); exp[:, 0] -= a
        assert np.array_equal(s["corr"], exp)


def _edge_scene():
    """candidate 0: keyframe 3 has 0 rows (as query and as train), keyframe 4 one row, keyframe 5 rows unrelated to the query
    (0 matches), keyframe 9 four rows copied from query keyframe 0 (4 matches), plus one ordinary pairing; candidate 1: 12 rows
    copied from keyframe 0 (keyframe 10) and a pairing without matches, fewer than 17 correspondences in all"""
    S, _ = scene(40, 2, n_kp=400)
    rng = np.random.default_rng(1)
    kp = S["kf_ptr"]
    rows = [np.arange(kp[k], kp[k + 1]) for k in range(len(kp) - 1)]
    rows[3] = rows[3][:0]; rows[4] = rows[4][:1]
    keep = np.concatenate(rows)
    desc, bear, sig = S["desc"][keep].copy(), S["bearings"][keep].copy(), S["sigma"][keep].copy()
    n = [len(r_) for r_ in rows]
    new_kp = np.concatenate([[0], np.cumsum(n)]).astype(np.int32)
    desc[new_kp[5]:new_kp[6]] = rng.integers(0, 256, (n[5], 32), dtype=np.uint8)
    desc = np.concatenate([desc, S["desc"][:4], S["desc"][:12]]); bear = np.concatenate([bear, bear[:4], bear[:12]])
    sig = np.concatenate([sig, sig[:4], sig[:12]])
    new_kp = np.concatenate([new_kp, [new_kp[-1] + 4, new_kp[-1] + 16]]).astype(np.int32)
    pairs = np.array([(0, 3, 0, 0), (3, 0, 0, 0), (1, 4, 1, 1), (2, 5, 2, 2), (0, 9, 0, 0), (0, 6, 0, 0),    # candidate 0
                      (0, 10, 0, 1), (1, 5, 1, 2)], np.int32)                                                 # candidate 1
    S.update(kf_ptr=new_kp, desc=desc, bearings=bear, sigma=sig, pairs=pairs, pair_ptr=np.array([0, 6, 8], np.int32),
             seeds5=np.arange(8, dtype=np.uint64) * 977 + 5)
    return S


@pytest.mark.gpu
def test_gpu_edge_cases(ctx):
    S = _edge_scene()
    g = PR.verify_noncentral_relative_pose_seeded(ctx, **S, **PRM)
    r = ov.verify_noncentral_seeded(**S, **PRM)
    _cmp(g, r)
    assert list(g["n_matches"][:4]) == [0, 0, 0, 0] and g["n_matches"][4] == 4 and (g["best_sample5"][:5] == -1).all()
    assert g["best_sample"][1] == -1 and g["n_valid"][1] == 0
    # a capacity below n_total: only n_total
    small = PR.verify_noncentral_relative_pose_seeded(ctx, **S, **PRM, corr_cap=int(g["n_total"]) - 1)
    assert small["n_total"] == g["n_total"] and "corr" not in small
    _cmp({k: v for k, v in small.items() if k != "corr"}, {k: v for k, v in r.items() if k != "corr"})
    # no candidates
    z = PR.verify_noncentral_relative_pose_seeded(ctx, **dict(S, cam_ptr1=[0], cam_ptr2=[0], cam_off1=np.zeros((0, 3)), cam_rot1=np.zeros((0, 9)),
                                                         cam_off2=np.zeros((0, 3)), cam_rot2=np.zeros((0, 9)), pair_ptr=[0], pairs=np.zeros((0, 4)),
                                                         seeds5=[], seeds=[]), **PRM)
    assert z["n_total"] == 0 and len(z["best_sample"]) == 0


@pytest.mark.gpu
def test_gpu_bad_arguments_are_refused(ctx):
    S, _ = scene(50, 2, n_kp=200)
    L = PR.lib()

    def call(prm=None, seed5=True, seed=True, **over):
        T = {k: np.ascontiguousarray(v).copy() for k, v in S.items()}
        T.update({k: np.ascontiguousarray(v) for k, v in over.items()})
        p = dict(PRM, n_cov_samples=30); p.update(prm or {})
        kp, pr, pp = T["kf_ptr"].astype(np.int32), T["pairs"].astype(np.int32), T["pair_ptr"].astype(np.int32)
        cp1, cp2 = T["cam_ptr1"].astype(np.int32), T["cam_ptr2"].astype(np.int32)
        K = PR.CVerifyKeyframes(len(kp) - 1, kp.ctypes.data, T["desc"].ctypes.data, T["bearings"].ctypes.data, T["sigma"].ctypes.data)
        co1 = np.ascontiguousarray(T["cam_off1"], np.float64); cr1 = np.ascontiguousarray(T["cam_rot1"], np.float64)
        co2 = np.ascontiguousarray(T["cam_off2"], np.float64); cr2 = np.ascontiguousarray(T["cam_rot2"], np.float64)
        D = PR.CVerifyCandidates(len(cp1) - 1, *[x.ctypes.data for x in (cp1, co1, cr1, cp2, co2, cr2, pp, pr)])
        Pm = PR.CVerifyParams(p["img_match_thres"], p["ratio_thres"], p["threshold5"], p["max_iterations5"], p["threshold17"], p["max_iterations17"],
                              p["probability"], p["n_cov_samples"])
        bufs = [np.zeros(4096, np.float64) for _ in range(13)]
        R = PR.CVerifyResult(*[b.ctypes.data for b in bufs], None, 0, 0)
        s5 = np.ascontiguousarray(T["seeds5"], np.uint64); s = np.ascontiguousarray(T["seeds"], np.uint64)
        before = ctx.launch_count()
        rc = L.cvb_verify_noncentral_relative_pose_seeded_batch(ctx.handle, C.byref(K), C.byref(D), C.byref(Pm), s5.ctypes.data if seed5 else None,
                                                                 s.ctypes.data if seed else None, C.byref(R))
        assert ctx.launch_count() == before or rc == 0
        return rc

    assert call() == 0
    kp = S["kf_ptr"].copy(); kp[2] = kp[1] - 1
    cases = [dict(kf_ptr=kp), dict(pair_ptr=np.array([0, 7, 6], np.int32)), dict(cam_ptr2=np.array([0, 4, 3], np.int32)),
             dict(pairs=np.where(np.arange(S["pairs"].size).reshape(-1, 4) == 1, 99, S["pairs"])),
             dict(pairs=np.where(np.arange(S["pairs"].size).reshape(-1, 4) == 3, 3, S["pairs"])),
             dict(cam_ptr1=np.array([0, 9, 12], np.int32), cam_off1=np.zeros((12, 3)), cam_rot1=np.tile(np.eye(3), (12, 1, 1)))]
    for over in cases:
        assert call(**over) == CVB_ERR_INVALID, over
    assert call(seed5=False) == CVB_ERR_INVALID and call(seed=False) == CVB_ERR_INVALID
    assert call(prm=dict(max_iterations5=(2**31 - 1 - 64) // 11 + 1)) == CVB_ERR_INVALID
    assert call(prm=dict(max_iterations17=-1)) == CVB_ERR_INVALID and call(prm=dict(n_cov_samples=-1)) == CVB_ERR_INVALID


@pytest.mark.gpu
def test_shim_verify_equals_python_path(ctx, tmp_path):
    S, _ = scene(60, 3)
    exe = str(tmp_path / "shim_verify_test")
    _build_shim("shim_verify_test.cpp", exe)
    types = dict(kf_ptr=np.int32, desc=np.uint8, bearings=np.float64, sigma=np.float64, cam_ptr1=np.int32, cam_off1=np.float64, cam_rot1=np.float64,
                 cam_ptr2=np.int32, cam_off2=np.float64, cam_rot2=np.float64, pair_ptr=np.int32, pairs=np.int32, seeds5=np.uint64, seeds=np.uint64)
    for k, t in types.items():
        np.ascontiguousarray(S[k], t).tofile(tmp_path / f"{k}.bin")
    np.array([PRM["img_match_thres"], PRM["ratio_thres"], PRM["threshold5"], PRM["max_iterations5"], PRM["threshold17"], PRM["max_iterations17"],
              PRM["probability"], 300], np.float64).tofile(tmp_path / "params.bin")
    subprocess.check_call([exe, str(tmp_path)])
    g = PR.verify_noncentral_relative_pose_seeded(ctx, **S, **PRM)
    P, Cn = len(S["pairs"]), len(S["seeds"])
    ints = np.fromfile(tmp_path / "verify_ints.bin", np.int32)
    assert np.array_equal(ints[:5 * P].reshape(P, 5), np.stack([g["n_matches"], g["best_sample5"], g["best_count5"], g["iterations5"], g["consumed5"]], 1))
    assert np.array_equal(ints[5 * P:].reshape(Cn, 5), np.stack([g["best_sample"], g["best_count"], g["iterations"], g["consumed"], g["n_valid"]], 1))
    models = np.fromfile(tmp_path / "verify_models.bin").reshape(-1, 3, 4)
    assert np.array_equal(models[:P], g["best_model5"]) and np.array_equal(models[P:], g["best_model"])
    assert np.array_equal(np.fromfile(tmp_path / "verify_cov.bin").reshape(-1, 6, 6), g["cov"])
    assert np.array_equal(np.fromfile(tmp_path / "verify_corr.bin", np.int32).reshape(-1, 5), g["corr"])
