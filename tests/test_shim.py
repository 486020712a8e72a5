"""The C++ host shim (covins_b200/csrc/host/covins_b200_shim.hpp) on mock containers.
CPU: it compiles and links against libcovins_b200.so with -Wall -Werror (host-logic check, no GPU).
GPU: GlobalBundleAdjustment / PoseGraphOptimization / MatchCandidatesORB called through the reference-shaped C++
surface give the same states as the flat-problem API (they differ only by the container → flat conversion and the
map's idpair keyframe order, i.e. by floating-point reordering)."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "cpp", "shim_test")


def build_shim_test():
    import covins_b200
    if not os.path.exists(covins_b200.LIB_PATH):
        covins_b200.build()
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-o", EXE, os.path.join(ROOT, "tests", "cpp", "shim_test.cpp"),
                           "-L" + os.path.join(ROOT, "covins_b200"), "-lcovins_b200", "-Wl,-rpath,$ORIGIN/../../covins_b200"])


def test_shim_compiles_and_links():
    build_shim_test()
    assert os.path.exists(EXE)


def _dump(p, d):
    for k, v in p.items():
        if isinstance(v, np.ndarray):
            np.ascontiguousarray(v).tofile(os.path.join(d, k + ".bin"))


def _rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-12)


@pytest.mark.gpu
@pytest.mark.parametrize("mode,visual_only", [("gba", False), ("gba_visual", True), ("gba_cams", False)])
def test_shim_gba_equals_flat_api(ctx, tmp_path, mode, visual_only):
    """gba_cams: the visual-inertial GBA on a map with one pinhole / radtan calibration per agent (intrinsics and
    extrinsic differ): the shim gives every mock keyframe its own camera, the flat problem maps keyframes to cameras"""
    from covins_b200 import optimization as O, synth_map
    if not os.path.exists(EXE):
        build_shim_test()
    # few gross outliers: with ill-posed two-view landmarks in the problem the comparison across two different keyframe
    # orders (and therefore summation orders) is dominated by their sensitivity, not by the shim
    p = synth_map.make_map(seed=21, n_agents=2, kf_per_agent=40, n_lm=2000, outlier_frac=0.01)
    if mode == "gba_cams":
        from test_ba_map_shapes import per_agent_cameras
        p = per_agent_cameras(p, [(0, 0, 0.0)] * 2, seed=22)
        assert len({tuple(r) for r in p["intr"]}) == 2 and np.array_equal(p["cam_of_kf"], p["agent_of"])
    _dump(p, str(tmp_path))
    subprocess.check_call([EXE, str(tmp_path), "gba_visual" if visual_only else "gba"])
    ref = O.global_bundle_adjustment(ctx, p, iterations_limit=4, visual_only=visual_only)
    pose = np.fromfile(tmp_path / "out_pose.bin").reshape(-1, 7)
    lm = np.fromfile(tmp_path / "out_lm.bin").reshape(-1, 3)
    sb = np.fromfile(tmp_path / "out_sb.bin").reshape(-1, 9)
    sign = np.sign((pose[:, :4] * ref["pose"][:, :4]).sum(1))[:, None]      # q and -q are the same rotation
    # The shim's keyframe order (idpair) differs from the flat problem's (agent-major): same problem, different
    # summation/elimination order.  The visual-inertial system is ill-conditioned (IMU weights ~1e4 next to pixel
    # residuals), so rounding differences are amplified to ~1e-5..1e-4 relative; visual-only stays at ~1e-6.
    tol = 2e-5 if visual_only else 3e-4
    assert _rel(pose[:, :4] * sign, ref["pose"][:, :4]) < tol and _rel(pose[:, 4:], ref["pose"][:, 4:]) < tol
    if not visual_only:
        assert _rel(sb, ref["speedbias"]) < tol
    well = (ref["lm_owner"] >= 0) & (np.abs(ref["lm"]).max(1) < 100)
    assert _rel(lm[well], ref["lm"][well]) < tol
    # round-1 outliers were erased from the containers (optimization_be.cpp:282-288)
    nobs = np.fromfile(tmp_path / "out_nobs.bin", dtype=np.int32)
    removed_per_lm = np.add.reduceat(ref["obs_removed"].astype(np.int64), p["lm_obs_ptr"][:-1])
    assert np.array_equal(nobs, np.diff(p["lm_obs_ptr"]) - removed_per_lm)


@pytest.mark.gpu
def test_shim_pgo_equals_flat_api(ctx, tmp_path):
    from covins_b200 import optimization as O, synth_map
    from oracle import ba_oracle as bo
    if not os.path.exists(EXE):
        build_shim_test()
    p = synth_map.make_map(seed=5, n_agents=3, kf_per_agent=40, n_lm=50, drift_trans=0.01, drift_yaw_deg=0.1)
    _dump(p, str(tmp_path))
    subprocess.check_call([EXE, str(tmp_path), "pgo"])
    edges = bo.pgo_edges(p, p["pose"], covins_mode=True)       # the edge list the reference builds (:886-1021)
    ref = O.pose_graph_optimization(ctx, p, edges, iterations=10)
    pose = np.fromfile(tmp_path / "out_pose.bin").reshape(-1, 7)
    sign = np.sign((pose[:, :4] * ref["pose"][:, :4]).sum(1))[:, None]
    assert _rel(pose[:, :4] * sign, ref["pose"][:, :4]) < 1e-6 and _rel(pose[:, 4:], ref["pose"][:, 4:]) < 1e-6
    assert np.abs(pose[:, 4:] - p["pose"][:, 4:]).max() > 1e-3      # it did move


@pytest.mark.gpu
def test_shim_match_candidates_equals_oracle(tmp_path):
    from covins_b200 import synth
    from oracle import knn as ora
    if not os.path.exists(EXE):
        build_shim_test()
    desc, _ = synth.orb_keyframes(seed=12, n_kf=7, n_feat=400, n_lm=600, window=600)
    lens = [400, 400, 0, 399, 57, 400]
    t = np.concatenate([desc[i + 1][:l] for i, l in enumerate(lens)])
    seg = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    desc[0].tofile(tmp_path / "q.bin"); t.tofile(tmp_path / "t.bin"); seg.tofile(tmp_path / "seg.bin")
    subprocess.check_call([EXE, str(tmp_path), "match"])
    out = np.fromfile(tmp_path / "match_out.bin", dtype=np.int32)
    i2, d2 = ora.knn_hamming_batch(desc[0], t, seg, 2)
    mt, md, cnt = ora.ratio_filter(i2, d2.astype(np.float32), 40.0, 0.8)
    pos = 0
    for s in range(len(lens)):
        n, disc = out[pos], out[pos + 1]; pos += 2
        assert n == cnt[s]
        assert disc == (1 if n < 25 else 0)                       # matches_thres / matches_thres_merge = 25
        q = np.flatnonzero(mt[s] >= 0)
        got = out[pos:pos + 3 * n].reshape(-1, 3); pos += 3 * n
        assert np.array_equal(got[:, 0], q) and np.array_equal(got[:, 1], mt[s][q]) and np.array_equal(got[:, 2], md[s][q].astype(np.int32))
    # the resident-map database (covins_b200::DescriptorDatabase) gives the same img_matches per candidate
    out_db = np.fromfile(tmp_path / "match_db_out.bin", dtype=np.int32)
    pos = 0
    for s in range(len(lens)):
        n = out_db[pos]; pos += 1
        q = np.flatnonzero(mt[s] >= 0)
        assert n == cnt[s]
        got = out_db[pos:pos + 3 * n].reshape(-1, 3); pos += 3 * n
        assert np.array_equal(got[:, 0], q) and np.array_equal(got[:, 1], mt[s][q]) and np.array_equal(got[:, 2], md[s][q].astype(np.int32))
    assert pos == len(out_db)
    # covins_b200::ComputeLandmarkDescriptors: the first (up to) 9 rows of every candidate as one landmark's observers
    out_lm = np.fromfile(tmp_path / "lmdesc_out.bin", dtype=np.int32)
    sizes = [min(l, 9) for l in lens]
    cand = np.concatenate([t[seg[i]:seg[i] + n] for i, n in enumerate(sizes)])
    rb, rd = ora.landmark_descriptor(cand, np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32))
    assert np.array_equal(out_lm[:len(lens)], rb)
    got_d = out_lm[len(lens):].astype(np.uint8).reshape(len(lens), 32)
    for i in range(len(lens)):
        assert np.array_equal(got_d[i], rd[i] if rb[i] >= 0 else np.full(32, 0xAB, np.uint8))


@pytest.mark.gpu
def test_shim_search_by_se3_and_dense_matcher_adaptor(ctx, tmp_path):
    """FeatureMatcher::SearchBySE3 and estd2::DenseMatcher::match<ALGO> through the reference-shaped C++ wrappers on mock
    containers == the flat-array API == the oracle"""
    from covins_b200 import placerec as PR, synth
    from oracle import geom as og, knn as ora
    if not os.path.exists(EXE):
        build_shim_test()
    views, T12, T21, a1, a2 = synth.se3_search_scene(21, n_kp=600, n_shared=200)
    for pre, v in zip(("k1", "k2"), views):
        for k in ("kp", "octave", "desc", "lm_valid", "lm_pos", "lm_maxdist", "lm_desc", "K", "Tcw"):
            np.ascontiguousarray(v[k]).tofile(os.path.join(tmp_path, f"{pre}_{k}.bin"))
    np.ascontiguousarray(T12).tofile(tmp_path / "T12.bin"); np.ascontiguousarray(T21).tofile(tmp_path / "T21.bin")
    subprocess.check_call([EXE, str(tmp_path), "search"])
    out = np.fromfile(tmp_path / "search_out.bin", np.int32)
    mk = lambda v: PR.KfView(v["kp"], v["octave"], v["desc"], v["lm_valid"], v["lm_pos"], v["lm_maxdist"], v["lm_desc"], v["K"], v["Tcw"], v["img_bounds"])
    k1, k2 = mk(views[0]), mk(views[1])
    zero1, zero2 = np.zeros(k1.n, np.uint8), np.zeros(k2.n, np.uint8)      # the wrapper starts from empty matches12
    r12, rnf, rm1, rm2 = og.search_by_se3(k1, k2, T12, T21, zero1, zero2)
    # (the reference's agreement rule match2[i] == i, :485-496, lets almost nothing through: nf is tiny by construction)
    assert out[0] == rnf and np.array_equal(out[1:], r12) and (rm1 >= 0).sum() > 40 and (rm2 >= 0).sum() > 40
    dense = np.fromfile(tmp_path / "dense_out.bin", np.int32).reshape(-1, 3)
    ra, rb, rd = ora.landmark_match(views[0]["desc"], 1 - views[0]["lm_valid"], views[1]["desc"], 1 - views[1]["lm_valid"], 50.0, 4)
    assert np.array_equal(dense[:, 0], ra) and np.array_equal(dense[:, 1], rb) and np.array_equal(dense[:, 2], rd.astype(np.int32)) and len(ra) > 20


@pytest.mark.gpu
def test_shim_optimize_relative_pose(ctx, tmp_path):
    """Optimization::OptimizeRelativePose through the reference-shaped C++ wrapper == the flat-array API (same T12, same
    return value, matches1 nulled at the purged RESIDUAL indices)"""
    from covins_b200 import optimization as O, synth
    if not os.path.exists(EXE):
        build_shim_test()
    kw, gt, out = synth.relpose_case(5, n=80)
    for k in ("pA_c", "pB_c", "kpA", "kpB", "sigmaA", "sigmaB", "T12"):
        np.ascontiguousarray(kw[k]).tofile(tmp_path / f"{k}.bin")
    np.asarray(kw["camA"]["intr"], np.float64).tofile(tmp_path / "intr.bin"); np.asarray(kw["camA"]["dist"], np.float64).tofile(tmp_path / "dist.bin")
    np.array([0.9]).tofile(tmp_path / "th.bin")
    subprocess.check_call([EXE, str(tmp_path), "relpose"])
    o = np.fromfile(tmp_path / "relpose_out.bin")
    ref = O.optimize_relative_pose(ctx, th_outlier_align=0.9, **kw)
    sign = np.sign(o[:4] @ ref["T12"][:4])
    assert np.abs(o[:4] * sign - ref["T12"][:4]).max() < 1e-9 and np.abs(o[4:7] - ref["T12"][4:]).max() < 1e-9
    assert int(o[7]) == ref["n_inliers"] and ref["removed"].sum() >= 3
    assert np.array_equal(o[8:8 + 80] == 0.0, ref["removed"]) and np.all(o[8 + 80:] == 0.0)
