"""cvb_verify_noncentral_relative_pose_sift_seeded_batch (placerec.verify_noncentral_relative_pose_sift_seeded): the COVINS_G
verification chain with SIFT descriptors in one call, against the composed oracle
(oracle/verify_sift.py:verify_noncentral_sift_seeded) and against the chain of the existing calls (cvb_match_l2_batch, then the
seeded 5-point, 17-point and covariance calls) with the glue done on the host.  The scene is the geometry of
tests/test_verify_relative.py with SIFT-like codes."""
import ctypes as C
import subprocess

import numpy as np
import pytest

from covins_b200 import placerec as PR, synth
from oracle import verify_sift as ovs
from ransac_helpers import _build_shim
from test_verify_relative import PAIRINGS, _chain, _cmp, _rig, _small_rot

PRM = dict(img_match_thres=500.0, ratio_thres=0.8, threshold5=9.0, max_iterations5=300, threshold17=9.0, max_iterations17=300,
           probability=0.99)
CVB_ERR_INVALID, CVB_ERR_UNSUPPORTED = 1, 3


def _codes(rng, n):
    """SIFT-like codes as synth.sift_keyframes makes them: a clipped Gamma, L2-normalised to 512, rounded and clipped to 0..255"""
    g = rng.gamma(0.7, 1.0, (n, synth.SIFT_DIM))
    return np.clip(np.rint(g / np.linalg.norm(g, axis=1, keepdims=True) * 512.0), 0, 255)


def _keyframe(rng, X, codes, off, rot, n_kp, lm_frac, outlier, sigma, noise=6.0):
    """n_kp rows: a share lm_frac observes random points of X (rig frame) through camera (off, rot) with the point's code plus
    rint(N(0, noise)), clipped, a share `outlier` of those with a random bearing; the rest are keypoints without a landmark
    (random code and bearing)"""
    n_lm = int(round(n_kp * lm_frac))
    ids = rng.choice(len(X), n_lm, replace=False)
    desc = _codes(rng, n_kp)
    f = rng.normal(0, 1, (n_kp, 3))
    slots = rng.permutation(n_kp)[:n_lm]
    desc[slots] = np.clip(codes[ids] + np.rint(rng.normal(0, noise, (n_lm, synth.SIFT_DIM))), 0, 255)
    f[slots] = (X[ids] - off) @ rot                      # Rc^T (X - c)
    bad = slots[rng.random(n_lm) < outlier]
    f[bad] = rng.normal(0, 1, (len(bad), 3))
    f /= np.linalg.norm(f, axis=1, keepdims=True)
    return desc.astype(np.float32), f, rng.uniform(*sigma, n_kp)


def scene(seed, n_cand, n_kp=300, outlier=0.3, lm_frac=0.6, n_pts=600, sigma=(1e-6, 1e-5), pairings=PAIRINGS):
    """test_verify_relative.scene with SIFT rows (desc [R,128] float32): two 3-camera rigs over shared points per candidate, the
    query rig (keyframes 0-2) and per candidate a rig at a random pose [R|t] (X1 = R X2 + t, keyframes 3 + 3c ..).  n_pts is
    smaller than the ORB scene's so that a pairing of 300-keypoint keyframes shares about as large a share of its landmarks.
    → the keyword arguments of verify_noncentral_relative_pose_sift_seeded without PRM, and the true poses"""
    rng = np.random.default_rng(seed)
    d = rng.normal(0, 1, (n_pts, 3)); d[:, 2] = np.abs(d[:, 2]) + 2.0; d /= np.linalg.norm(d, axis=1, keepdims=True)
    X = d * rng.uniform(4, 30, n_pts)[:, None]
    codes = _codes(rng, n_pts)
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


def _oracle(S, **kw):
    return ovs.verify_noncentral_sift_seeded(**S, **PRM, **kw)


# --------------------------------------------------------------------------------------------------------------- CPU
def test_oracle_recovers_true_pose_noise_free():
    S, poses = scene(1, 2)
    r = _oracle(S, n_cov_samples=20)
    assert (r["n_matches"] >= 17).all() and (r["best_sample5"] >= 0).all()
    assert (r["corr"][:, 3] == 0).any() and (r["corr"][:, 3] == 1).any()          # the 5-point RANSACs reject the wrong bearings
    for c, (R, t) in enumerate(poses):
        M = r["best_model"][c].reshape(3, 4)
        assert r["best_sample"][c] >= 0 and r["n_valid"][c] > 0
        assert np.abs(M[:, :3] - R).max() < 1e-6 and np.abs(M[:, 3] - t).max() < 1e-6, c


def test_shim_verify_sift_compiles_and_links(tmp_path):
    exe = str(tmp_path / "shim_verify_sift_test")
    _build_shim("shim_verify_sift_test.cpp", exe)
    assert subprocess.run([exe, str(tmp_path)]).returncode == 2        # nothing dumped: refused before any GPU work


# --------------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("n_cand", [1, 8, 32])
def test_gpu_equals_composed_oracle_bitwise(ctx, n_cand):
    S, _ = scene(10 + n_cand, n_cand)
    g = PR.verify_noncentral_relative_pose_sift_seeded(ctx, **S, **PRM)
    _cmp(g, _oracle(S))
    assert (g["best_sample"] >= 0).all() and (g["n_valid"] > 0).all()
    c = g["corr"]
    assert (c[:, 3] == 0).any() and (c[:, 4] == 0).any() and (c[:, 4] == 1).any()


@pytest.mark.gpu
@pytest.mark.parametrize("n_cand", [1, 8])
def test_gpu_equals_chain_of_existing_calls(ctx, n_cand):
    S, _ = scene(20 + n_cand, n_cand, outlier=0.05)
    g = PR.verify_noncentral_relative_pose_sift_seeded(ctx, **S, **PRM)
    _cmp(g, _chain()(ctx, S, PRM, 300, metric="l2"))


@pytest.mark.gpu
def test_gpu_candidate_alone_equals_batch(ctx):
    S, _ = scene(30, 8)
    g = PR.verify_noncentral_relative_pose_sift_seeded(ctx, **S, **PRM)
    pp = S["pair_ptr"]
    for c in (0, 5, 7):
        a, b = pp[c], pp[c + 1]
        one = dict(S, cam_ptr1=np.array([0, 3], np.int32), cam_off1=S["cam_off1"][3 * c:3 * c + 3], cam_rot1=S["cam_rot1"][3 * c:3 * c + 3],
                   cam_ptr2=np.array([0, 3], np.int32), cam_off2=S["cam_off2"][3 * c:3 * c + 3], cam_rot2=S["cam_rot2"][3 * c:3 * c + 3],
                   pair_ptr=np.array([0, b - a], np.int32), pairs=S["pairs"][a:b], seeds5=S["seeds5"][a:b], seeds=S["seeds"][c:c + 1])
        s = PR.verify_noncentral_relative_pose_sift_seeded(ctx, **one, **PRM)
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
    S, _ = scene(40, 2)
    rng = np.random.default_rng(1)
    kp = S["kf_ptr"]
    rows = [np.arange(kp[k], kp[k + 1]) for k in range(len(kp) - 1)]
    rows[3] = rows[3][:0]; rows[4] = rows[4][:1]
    keep = np.concatenate(rows)
    desc, bear, sig = S["desc"][keep].copy(), S["bearings"][keep].copy(), S["sigma"][keep].copy()
    n = [len(r_) for r_ in rows]
    new_kp = np.concatenate([[0], np.cumsum(n)]).astype(np.int32)
    desc[new_kp[5]:new_kp[6]] = _codes(rng, n[5])
    desc = np.concatenate([desc, S["desc"][:4], S["desc"][:12]]); bear = np.concatenate([bear, bear[:4], bear[:12]])
    sig = np.concatenate([sig, sig[:4], sig[:12]])
    new_kp = np.concatenate([new_kp, [new_kp[-1] + 4, new_kp[-1] + 16]]).astype(np.int32)
    pairs = np.array([(0, 3, 0, 0), (3, 0, 0, 0), (1, 4, 1, 1), (2, 5, 2, 2), (0, 9, 0, 0), (0, 6, 0, 0),    # candidate 0
                      (0, 10, 0, 1), (1, 5, 1, 2)], np.int32)                                                 # candidate 1
    S.update(kf_ptr=new_kp, desc=desc, bearings=bear, sigma=sig, pairs=pairs, pair_ptr=np.array([0, 6, 8], np.int32),
             seeds5=np.arange(8, dtype=np.uint64) * 977 + 5)
    return S


def test_edge_scene_matches():
    """the edge scene has the match counts its cases need (the oracle's matching alone, no GPU)"""
    S = _edge_scene()
    r = _oracle(S, n_cov_samples=0)
    assert list(r["n_matches"][:4]) == [0, 0, 0, 0] and r["n_matches"][4] == 4 and r["n_matches"][6] == 12
    assert r["n_matches"][5] >= 17 and r["n_matches"][7] == 0 and r["best_sample"][1] == -1


@pytest.mark.gpu
def test_gpu_edge_cases(ctx):
    S = _edge_scene()
    g = PR.verify_noncentral_relative_pose_sift_seeded(ctx, **S, **PRM)
    r = _oracle(S)
    _cmp(g, r)
    assert list(g["n_matches"][:4]) == [0, 0, 0, 0] and g["n_matches"][4] == 4 and (g["best_sample5"][:5] == -1).all()
    assert g["best_sample"][1] == -1 and g["n_valid"][1] == 0
    # a capacity below n_total: only n_total
    small = PR.verify_noncentral_relative_pose_sift_seeded(ctx, **S, **PRM, corr_cap=int(g["n_total"]) - 1)
    assert small["n_total"] == g["n_total"] and "corr" not in small
    _cmp({k: v for k, v in small.items() if k != "corr"}, {k: v for k, v in r.items() if k != "corr"})
    # no candidates
    z = PR.verify_noncentral_relative_pose_sift_seeded(ctx, **dict(S, cam_ptr1=[0], cam_ptr2=[0], cam_off1=np.zeros((0, 3)), cam_rot1=np.zeros((0, 9)),
                                                              cam_off2=np.zeros((0, 3)), cam_rot2=np.zeros((0, 9)), pair_ptr=[0], pairs=np.zeros((0, 4)),
                                                              seeds5=[], seeds=[]), **PRM)
    assert z["n_total"] == 0 and len(z["best_sample"]) == 0


@pytest.mark.gpu
def test_gpu_bad_arguments_are_refused_before_any_launch(ctx):
    S, _ = scene(50, 2, n_kp=200)
    L = PR.lib()

    def call(prm=None, seed5=True, seed=True, **over):
        T = {k: np.ascontiguousarray(v).copy() for k, v in S.items()}
        T.update({k: np.ascontiguousarray(v) for k, v in over.items()})
        p = dict(PRM, n_cov_samples=30); p.update(prm or {})
        kp, pr, pp = T["kf_ptr"].astype(np.int32), T["pairs"].astype(np.int32), T["pair_ptr"].astype(np.int32)
        cp1, cp2 = T["cam_ptr1"].astype(np.int32), T["cam_ptr2"].astype(np.int32)
        dsc = np.ascontiguousarray(T["desc"], np.float32)
        K = PR.CVerifyKeyframes(len(kp) - 1, kp.ctypes.data, dsc.ctypes.data, T["bearings"].ctypes.data, T["sigma"].ctypes.data)
        co1 = np.ascontiguousarray(T["cam_off1"], np.float64); cr1 = np.ascontiguousarray(T["cam_rot1"], np.float64)
        co2 = np.ascontiguousarray(T["cam_off2"], np.float64); cr2 = np.ascontiguousarray(T["cam_rot2"], np.float64)
        D = PR.CVerifyCandidates(len(cp1) - 1, *[x.ctypes.data for x in (cp1, co1, cr1, cp2, co2, cr2, pp, pr)])
        Pm = PR.CVerifyParams(p["img_match_thres"], p["ratio_thres"], p["threshold5"], p["max_iterations5"], p["threshold17"], p["max_iterations17"],
                              p["probability"], p["n_cov_samples"])
        bufs = [np.zeros(4096, np.float64) for _ in range(13)]
        R = PR.CVerifyResult(*[b.ctypes.data for b in bufs], None, 0, 0)
        s5 = np.ascontiguousarray(T["seeds5"], np.uint64); s = np.ascontiguousarray(T["seeds"], np.uint64)
        before = ctx.launch_count()
        rc = L.cvb_verify_noncentral_relative_pose_sift_seeded_batch(ctx.handle, C.byref(K), C.byref(D), C.byref(Pm),
                                                                      s5.ctypes.data if seed5 else None, s.ctypes.data if seed else None, C.byref(R))
        return rc, ctx.launch_count() - before

    rc, launched = call()
    assert rc == 0 and launched > 0
    # every CVB_ERR_INVALID case of the ORB call
    kp = S["kf_ptr"].copy(); kp[2] = kp[1] - 1
    invalid = [dict(kf_ptr=kp), dict(pair_ptr=np.array([0, 7, 6], np.int32)), dict(cam_ptr2=np.array([0, 4, 3], np.int32)),
               dict(pairs=np.where(np.arange(S["pairs"].size).reshape(-1, 4) == 1, 99, S["pairs"])),
               dict(pairs=np.where(np.arange(S["pairs"].size).reshape(-1, 4) == 3, 3, S["pairs"])),
               dict(cam_ptr1=np.array([0, 9, 12], np.int32), cam_off1=np.zeros((12, 3)), cam_rot1=np.tile(np.eye(3), (12, 1, 1))),
               dict(seed5=False), dict(seed=False), dict(prm=dict(max_iterations5=(2**31 - 1 - 64) // 11 + 1)),
               dict(prm=dict(max_iterations17=-1)), dict(prm=dict(n_cov_samples=-1))]
    for over in invalid:
        assert call(**over) == (CVB_ERR_INVALID, 0), over
    # a descriptor value that is not an integer in [0, 255], in a row of the last keyframe
    for v in (0.5, -1.0, 256.0, np.nan, np.inf, -np.inf):
        desc = S["desc"].copy(); desc[-1, 77] = v
        assert call(desc=desc) == (CVB_ERR_UNSUPPORTED, 0), v
    desc = S["desc"].copy(); desc[0, 0], desc[1, 1] = 0.0, 255.0      # the range's ends are accepted
    assert call(desc=desc)[0] == 0


@pytest.mark.gpu
def test_shim_verify_sift_equals_python_path(ctx, tmp_path):
    S, _ = scene(60, 3)
    exe = str(tmp_path / "shim_verify_sift_test")
    _build_shim("shim_verify_sift_test.cpp", exe)
    types = dict(kf_ptr=np.int32, desc=np.float32, bearings=np.float64, sigma=np.float64, cam_ptr1=np.int32, cam_off1=np.float64,
                 cam_rot1=np.float64, cam_ptr2=np.int32, cam_off2=np.float64, cam_rot2=np.float64, pair_ptr=np.int32, pairs=np.int32,
                 seeds5=np.uint64, seeds=np.uint64)
    for k, t in types.items():
        np.ascontiguousarray(S[k], t).tofile(tmp_path / f"{k}.bin")
    np.array([PRM["img_match_thres"], PRM["ratio_thres"], PRM["threshold5"], PRM["max_iterations5"], PRM["threshold17"], PRM["max_iterations17"],
              PRM["probability"], 300], np.float64).tofile(tmp_path / "params.bin")
    subprocess.check_call([exe, str(tmp_path)])
    g = PR.verify_noncentral_relative_pose_sift_seeded(ctx, **S, **PRM)
    P, Cn = len(S["pairs"]), len(S["seeds"])
    ints = np.fromfile(tmp_path / "verify_ints.bin", np.int32)
    assert np.array_equal(ints[:5 * P].reshape(P, 5), np.stack([g["n_matches"], g["best_sample5"], g["best_count5"], g["iterations5"], g["consumed5"]], 1))
    assert np.array_equal(ints[5 * P:].reshape(Cn, 5), np.stack([g["best_sample"], g["best_count"], g["iterations"], g["consumed"], g["n_valid"]], 1))
    models = np.fromfile(tmp_path / "verify_models.bin").reshape(-1, 3, 4)
    assert np.array_equal(models[:P], g["best_model5"]) and np.array_equal(models[P:], g["best_model"])
    assert np.array_equal(np.fromfile(tmp_path / "verify_cov.bin").reshape(-1, 6, 6), g["cov"])
    assert np.array_equal(np.fromfile(tmp_path / "verify_corr.bin", np.int32).reshape(-1, 5), g["corr"])
