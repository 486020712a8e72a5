"""cvb_landmark_outliers: the landmark outlier removal of Map::Clean (map_be.cpp:448-454, 698-743); include/covins_b200.h
states the rule and oracle/lm_outliers.py carries the assumption.
CPU: the oracle equals an independent from-scratch restatement (per-landmark loops, the camera-frame point and the pixel
from synth_map's projection) on hand cases that each pin one clause (also pinned to literal flags), on random maps over the
six camera models with points moved behind a camera, and on C1; the C++ shim compiles and refuses missing input.
GPU: the norms are bitwise those of cvb_ba_reproj_norms on C1 and C3 (also after a GBA); flags and erasures equal the
oracle's up to norms within the bundle adjustment tests' tolerance of the threshold; the six camera models; repeatability
and a launch count that does not depend on the map; refused inputs and empty maps; the C++ shim on mock containers.
"""
import math
import os
import subprocess

import numpy as np
import pytest

from covins_b200 import synth_map
from oracle import covis as ora_covis
from oracle import lm_outliers as ora

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RTOL = 1e-5   # tests/test_gpu_ba.py: the bundle adjustment's agreement with the autograd oracle
CAMERA_MODELS = [(0, 0, 0.0), (0, 1, 0.0), (0, 2, 0.0), (1, 0, 0.9), (1, 1, 0.9), (1, 2, 0.9)]


# ------------------------------------------------------------------------------------------------------------------
# maps
# ------------------------------------------------------------------------------------------------------------------
INTR = np.array([[400.0, 400.0, 320.0, 240.0]])


def hand_map(tracks, K, offsets=None, kf_z=None, lm_z=None, skip=None):
    """keyframe k at (0.1 k, 0, kf_z[k]) looking along +z; landmark l at (0.1 l, 0.05 l, lm_z[l]) (default 5); observation
    o = the exact pinhole pixel + offsets[o] pixels in u (default 0); sigma 2"""
    ptr = np.concatenate([[0], np.cumsum([len(t) for t in tracks])]).astype(np.int32)
    kf = np.array([k for t in tracks for k in t], np.int32)
    L = len(tracks)
    pose = np.zeros((K, 7)); pose[:, 3] = 1.0; pose[:, 4] = 0.1 * np.arange(K)
    if kf_z is not None:
        pose[:, 6] = kf_z
    lm = np.stack([0.1 * np.arange(L), 0.05 * np.arange(L), np.full(L, 5.0) if lm_z is None else np.asarray(lm_z, float)], 1)
    obs_lm = np.repeat(np.arange(L), np.diff(ptr))
    pc = lm[obs_lm] - pose[kf, 4:]
    with np.errstate(divide="ignore", invalid="ignore"):
        uv = np.stack([400.0 * pc[:, 0] / pc[:, 2] + 320.0, 400.0 * pc[:, 1] / pc[:, 2] + 240.0], 1)
    uv = np.nan_to_num(uv)
    if offsets is not None:
        uv[:, 0] += np.asarray(offsets, float)
    extr = np.zeros((1, 7)); extr[0, 3] = 1.0
    p = dict(K=K, L=L, pose=pose, pose_const=np.zeros(K, np.uint8), extr=extr, intr=INTR.copy(), dist=np.zeros((1, 4)), lm=lm,
             lm_obs_ptr=ptr, obs_kf=kf, obs_uv=uv.astype(np.float32), obs_sigma=np.full(len(kf), 2.0))
    if skip is not None:
        p["obs_skip"] = np.asarray(skip, np.uint8)
    return p


OUT = 10.0   # a 10-pixel error at sigma 2: norm 5 / sqrt(26) = 0.98 > 0.92


def hand_cases():
    big = 2000
    return {   # name → (map, call arguments, literal obs_outlier, literal lm_erase)
        "all_inliers": (hand_map([[0, 1, 2]], 3), {}, [0, 0, 0], [0]),
        "one_outlier_two_left": (hand_map([[0, 1, 2]], 3, offsets=[0, 0, OUT]), {}, [0, 0, 1], [0]),
        "two_outliers_one_left": (hand_map([[0, 1, 2]], 3, offsets=[OUT, 0, OUT]), {}, [1, 0, 1], [1]),
        "behind_every_camera": (hand_map([[0, 1]], 2, lm_z=[-5.0]), {}, [2, 2], [1]),
        # keyframe 2 stands beyond the point: behind it only
        "behind_one_camera": (hand_map([[0, 1, 2]], 3, kf_z=[0, 0, 8]), {}, [0, 0, 2], [0]),
        "min_obs_1": (hand_map([[0, 1, 2]], 3, offsets=[0, OUT, OUT]), dict(min_obs=1), [0, 1, 1], [0]),
        "min_obs_2": (hand_map([[0, 1, 2]], 3, offsets=[0, OUT, OUT]), dict(min_obs=2), [0, 1, 1], [1]),
        "min_obs_3": (hand_map([[0, 1, 2]], 3, offsets=[0, 0, OUT]), dict(min_obs=3), [0, 0, 1], [1]),
        # a skipped observation neither counts nor is flagged, however bad
        "obs_skip": (hand_map([[0, 1, 2]], 3, offsets=[OUT, 0, OUT], skip=[1, 0, 0]), {}, [0, 0, 1], [1]),
        "lm_valid": (hand_map([[0, 1], [0, 1]], 2, offsets=[0, 0, OUT, OUT]), dict(lm_valid=np.array([1, 0], np.uint8)), [0, 0, 0, 0], [0, 0]),
        "loses_all_observers": (hand_map([[0, 1], [0, 1]], 2, skip=[1, 1, 0, 0]), {}, [0, 0, 0, 0], [1, 0]),
        "no_loss": (hand_map([[0, 1, 2]], 3, offsets=[0, 0, 3.0]), dict(cauchy=0.0), [0, 0, 1], [0]),
        # 2 000 observers: every third one an outlier, then all but one
        "thousands_of_observers": (hand_map([list(range(big)), list(range(big))], big,
                                            offsets=[OUT if o % 3 == 0 else 0 for o in range(big)] + [0] + [OUT] * (big - 1)), {},
                                   [1 if o % 3 == 0 else 0 for o in range(big)] + [0] + [1] * (big - 1), [0, 1]),
    }


CASES = hand_cases()


def random_map(seed):
    """a small synthetic map through one of the six camera models, some landmarks reflected through an observer's camera
    centre (behind it), random masks and parameters"""
    rng = np.random.default_rng(seed)
    p = synth_map.make_map(seed=seed, n_agents=int(rng.integers(1, 3)), kf_per_agent=int(rng.integers(8, 20)), n_lm=int(rng.integers(50, 300)))
    cm, dm, xi = CAMERA_MODELS[seed % 6]
    p = synth_map.with_camera_model(p, cm, dm, xi=xi, seed=seed)
    p = behind_some_cameras(p, rng, 0.05)
    n = len(p["obs_kf"])
    if seed % 2:
        p["obs_skip"] = (rng.random(n) < 0.1).astype(np.uint8)
    kw = dict(th_outlier=float(rng.uniform(0.3, 1.5)), cauchy=float(rng.choice([0.0, 0.5, 1.0, 2.0])), min_obs=int(rng.integers(1, 4)))
    if seed % 3:
        kw["lm_valid"] = (rng.random(p["L"]) < 0.9).astype(np.uint8)
    return p, kw


def behind_some_cameras(p, rng, frac):
    """landmark l → 2 c - X, c the camera centre of its first observer: the point is then behind that camera"""
    p = dict(p)
    lm = np.array(p["lm"], float)
    ptr, kf = p["lm_obs_ptr"], p["obs_kf"]
    R_ws = synth_map.quat_to_rot(p["pose"][:, :4])
    for l in np.flatnonzero(rng.random(p["L"]) < frac):
        if ptr[l + 1] > ptr[l]:
            k = kf[ptr[l]]
            c = p["pose"][k, 4:] + R_ws[k] @ np.asarray(p["extr"]).reshape(-1, 7)[0, 4:]
            lm[l] = 2 * c - lm[l]
    p["lm"] = lm
    return p


# ------------------------------------------------------------------------------------------------------------------
# the independent restatement: per landmark, per observation, from scratch
# ------------------------------------------------------------------------------------------------------------------
def restated(p, lm_valid=None, th_outlier=0.92, cauchy=1.0, min_obs=2, norms_in=None):
    K, L = int(p["K"]), int(p["L"])
    ptr, kfs = p["lm_obs_ptr"], p["obs_kf"]
    n = len(kfs)
    out, erase, norms = np.zeros(n, np.uint8), np.zeros(L, np.uint8), np.full(n, -1.0)
    if K == 0 or L == 0 or n == 0:
        return out, erase, norms
    skip = p.get("obs_skip")
    extr = np.asarray(p["extr"], float).reshape(-1, 7)
    for l in range(L):
        if lm_valid is not None and not lm_valid[l]:
            continue
        good = 0
        for o in range(ptr[l], ptr[l + 1]):
            if skip is not None and skip[o]:
                continue
            k = int(kfs[o])
            c = int(p["cam_of_kf"][k]) if p.get("cam_of_kf") is not None else 0
            cm = int(p["cam_model"][c]) if p.get("cam_model") is not None else 0
            dm = int(p["dist_model"][c]) if p.get("dist_model") is not None else 0
            xi = float(p["cam_xi"][c]) if cm == 1 else 0.0
            R_ws = synth_map.quat_to_rot(p["pose"][k][None, :4])[0]
            R_sc = synth_map.quat_to_rot(extr[c][None, :4])[0]
            pc = R_sc.T @ (R_ws.T @ (p["lm"][l] - p["pose"][k][4:]) - extr[c][4:])
            d = math.sqrt(pc @ pc)
            den = pc[2] + xi * d if cm == 1 else pc[2]
            if not (den > 1e-10):
                out[o], norms[o] = 2, 0.0
                continue
            uv = synth_map.project_model(pc[None], p["intr"][c], p["dist"][c], cm, dm, xi)[0]
            r = (uv - p["obs_uv"][o].astype(float)) / p["obs_sigma"][o]
            s = float(r @ r)
            norms[o] = math.sqrt(s) * (math.sqrt(1.0 / (1.0 + s / (cauchy * cauchy))) if cauchy > 0 else 1.0)
            v = norms[o] if norms_in is None else norms_in[o]
            if v > th_outlier:
                out[o] = 1
            else:
                good += 1
        erase[l] = good < min_obs
    return out, erase, norms


def _agree(p, kw, tol=1e-9):
    """oracle == restatement: norms to tol, flags exactly (on the restatement's own norms, and on the oracle's norms where the
    two are within tol of the threshold)"""
    o_out, o_erase, o_norm = ora.landmark_outliers(p, **kw)
    r_out, r_erase, r_norm = restated(p, **kw)
    part = o_norm >= 0
    assert np.array_equal(part, r_norm >= 0)
    assert np.allclose(o_norm[part], r_norm[part], rtol=tol, atol=tol)
    assert np.array_equal(o_out, r_out) and np.array_equal(o_erase, r_erase)
    s_out, s_erase, _ = restated(p, norms_in=o_norm, **kw)
    assert np.array_equal(o_out, s_out) and np.array_equal(o_erase, s_erase)
    return o_out, o_erase, o_norm


# ------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_equals_restatement_on_hand_cases(name):
    p, kw, lit_out, lit_erase = CASES[name]
    out, erase, _ = _agree(p, kw)
    assert out.tolist() == lit_out and erase.tolist() == lit_erase


def test_threshold_exactly_hit_and_just_exceeded():
    """norm == th_outlier is not an outlier, the next double below th_outlier makes it one"""
    p, _, _, _ = CASES["one_outlier_two_left"]
    _, _, norms = ora.landmark_outliers(p)
    for th, flag in ((norms[2], 0), (np.nextafter(norms[2], 0.0), 1)):
        part, obs_lm, lm_in = ora.participating(p)
        out, _ = ora.decide(part, obs_lm, lm_in, norms, np.ones(3, bool), th_outlier=th)
        r_out, _, _ = restated(p, th_outlier=th, norms_in=norms)
        assert out[2] == r_out[2] == flag


@pytest.mark.parametrize("seed", range(12))
def test_oracle_equals_restatement_on_random_maps(seed):
    p, kw = random_map(seed)
    out, _, _ = _agree(p, kw)
    assert (out == 2).any()


def test_oracle_equals_restatement_on_c1():
    p = synth_map.make_config("C1")
    out, erase, _ = _agree(p, {})
    assert (out == 1).sum() >= 0.9 * p["obs_is_outlier"].sum() and erase.sum() > 0


def test_shim_outlier_compiles_and_refuses_missing_input(tmp_path):
    exe = str(tmp_path / "shim_outlier_test")
    _build_shim(exe)
    assert subprocess.run([exe, str(tmp_path), "0.92", "1.0", "2"]).returncode == 2     # nothing dumped: refused before any GPU work


def _build_shim(exe):
    import covins_b200
    if not os.path.exists(covins_b200.LIB_PATH):
        covins_b200.build()
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-o", exe, os.path.join(ROOT, "tests", "cpp", "shim_outlier_test.cpp"),
                           "-L" + os.path.join(ROOT, "covins_b200"), "-lcovins_b200", "-Wl,-rpath," + os.path.join(ROOT, "covins_b200")])


# ------------------------------------------------------------------------------------------------------------------
# GPU, through the C-ABI
# ------------------------------------------------------------------------------------------------------------------
def _gpu(ctx, p, **kw):
    from covins_b200 import mapgraph
    return mapgraph.landmark_outliers(ctx, p, want_norms=True, **kw)


def _ba_norms(ctx, p):
    from covins_b200 import optimization as O
    s = O.BaSolver(ctx, p, visual_only=False, cauchy_reproj=1.0, obs_skip=p.get("obs_skip"))
    try:
        return s.reproj_norms()
    finally:
        s.close()


def _check_against_oracle(p, kw, got):
    """norms to RTOL; flags and erasures exactly, except observations whose oracle norm lies within RTOL of the threshold"""
    out, erase, norms = got
    o_out, o_erase, o_norm = ora.landmark_outliers(p, **kw)
    part = o_norm >= 0
    assert np.array_equal(norms >= 0, part)
    assert np.allclose(norms[part], o_norm[part], rtol=RTOL, atol=RTOL)
    th = kw.get("th_outlier", 0.92)
    near = part & (np.abs(o_norm - th) <= RTOL * th)
    assert np.array_equal(out[~near], o_out[~near])
    assert near.sum() <= max(2, 1e-4 * part.sum()), int(near.sum())
    if not near.any():
        assert np.array_equal(erase, o_erase)
    # the landmark rule on the GPU's own flags reproduces its erasures exactly
    part_, obs_lm, lm_in = ora.participating(p, kw.get("lm_valid"))
    ref_out, ref_erase = ora.decide(part_, obs_lm, lm_in, norms, out != 2, th_outlier=th, min_obs=kw.get("min_obs", 2))
    assert np.array_equal(ref_out, out) and np.array_equal(ref_erase, erase)
    return int(near.sum())


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_hand_cases_equal_the_oracle(ctx, name):
    p, kw, lit_out, lit_erase = CASES[name]
    out, erase, norms = _gpu(ctx, p, **kw)
    assert out.tolist() == lit_out and erase.tolist() == lit_erase
    _check_against_oracle(p, kw, (out, erase, norms))


@pytest.mark.gpu
def test_threshold_exactly_hit_and_just_exceeded_on_the_gpu(ctx):
    p, _, _, _ = CASES["one_outlier_two_left"]
    norms = _gpu(ctx, p)[2]
    assert _gpu(ctx, p, th_outlier=float(norms[2]))[0][2] == 0
    assert _gpu(ctx, p, th_outlier=float(np.nextafter(norms[2], 0.0)))[0][2] == 1


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["C1", "C3"])
def test_norms_are_bitwise_those_of_the_bundle_adjustment(ctx, config):
    """every observation the BA includes (5 % synthetic gross outliers), at the map's state and after a cvb_gba"""
    from covins_b200 import optimization as O
    p = synth_map.make_config(config)
    states = [p]
    if config == "C1":
        g = O.global_bundle_adjustment(ctx, p, iterations_limit=3)
        states.append(dict(p, pose=g["pose"], lm=g["lm"], obs_skip=g["obs_removed"].astype(np.uint8)))
    for q in states:
        ref = _ba_norms(ctx, q)
        out, erase, norms = _gpu(ctx, q)
        inc = ref != -1.0
        assert inc.sum() > 0.9 * len(ref)
        diff = norms[inc].view(np.uint64) != ref[inc].view(np.uint64)
        assert not diff.any(), (int(diff.sum()), float(np.abs(norms[inc] - ref[inc]).max()))
        assert np.array_equal(out[inc] == 1, ref[inc] > 0.92)
        if config == "C1":
            _check_against_oracle(q, {}, (out, erase, norms))


@pytest.mark.gpu
@pytest.mark.parametrize("model", range(6))
def test_camera_models_equal_the_oracle(ctx, model):
    cm, dm, xi = CAMERA_MODELS[model]
    rng = np.random.default_rng(model)
    p = behind_some_cameras(synth_map.with_camera_model(synth_map.make_config("small"), cm, dm, xi=xi, seed=model), rng, 0.05)
    got = _gpu(ctx, p)
    assert (got[0] == 2).sum() > 10 and (got[0] == 1).sum() > 100
    _check_against_oracle(p, {}, got)
    assert np.array_equal(got[2].view(np.uint64)[_ba_norms(ctx, p) != -1.0], _ba_norms(ctx, p)[_ba_norms(ctx, p) != -1.0].view(np.uint64))


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(12))
def test_random_maps_equal_the_oracle(ctx, seed):
    p, kw = random_map(seed)
    _check_against_oracle(p, kw, _gpu(ctx, p, **kw))


@pytest.mark.gpu
def test_two_runs_are_identical_and_launches_do_not_depend_on_the_map(ctx):
    for p in (CASES["all_inliers"][0], synth_map.make_config("C1"), synth_map.make_config("C3")):
        outs = []
        for _ in range(2):
            l0 = ctx.launch_count()
            out, erase, norms = _gpu(ctx, p)
            assert ctx.launch_count() - l0 == 2          # one pass over the observations, one over the landmarks
            outs.append(out.tobytes() + erase.tobytes() + norms.tobytes())
        assert outs[0] == outs[1]


@pytest.mark.gpu
def test_empty_maps(ctx):
    from covins_b200 import lib
    import ctypes as C
    from covins_b200.optimization import BaProblem
    l0 = ctx.launch_count()
    for p in (hand_map([], 3), hand_map([[], []], 3), dict(hand_map([], 0), K=0)):
        out, erase, norms = _gpu(ctx, p)
        assert not out.any() and not erase.any() and (norms == -1).all()
    n_o, n_l = C.c_int64(5), C.c_int32(5)
    s = BaProblem()
    assert lib().cvb_landmark_outliers(ctx.handle, C.byref(s), None, 0.92, 1.0, 2, None, None, None, C.byref(n_o), C.byref(n_l)) == 0
    assert n_o.value == 0 and n_l.value == 0 and ctx.launch_count() == l0


@pytest.mark.gpu
def test_invalid_input_is_refused_before_any_launch(ctx):
    from covins_b200 import CvbError
    base, _, _, _ = CASES["one_outlier_two_left"]
    bad = {
        "kf out of range": (dict(obs_kf=np.array([0, 1, 3], np.int32)), {}),
        "kf negative": (dict(obs_kf=np.array([0, -1, 2], np.int32)), {}),
        "cam out of range": (dict(cam_of_kf=np.array([0, 1, 0], np.int32)), {}),
        "ptr decreasing": (dict(lm_obs_ptr=np.array([0, 3, 2, 3], np.int32), L=3, lm=np.zeros((3, 3))), {}),
        "ptr not from 0": (dict(lm_obs_ptr=np.array([1, 3], np.int32)), {}),
        "sigma 0": (dict(obs_sigma=np.array([2.0, 0.0, 2.0])), {}),
        "sigma negative": (dict(obs_sigma=np.array([2.0, -2.0, 2.0])), {}),
        "sigma inf": (dict(obs_sigma=np.array([2.0, np.inf, 2.0])), {}),
        "sigma NaN": (dict(obs_sigma=np.array([2.0, np.nan, 2.0])), {}),
        "th NaN": ({}, dict(th_outlier=float("nan"))),
        "th 0": ({}, dict(th_outlier=0.0)),
        "th negative": ({}, dict(th_outlier=-1.0)),
        "cauchy inf": ({}, dict(cauchy=float("inf"))),
        "cauchy NaN": ({}, dict(cauchy=float("nan"))),
        "min_obs 0": ({}, dict(min_obs=0)),
    }
    for name, (pk, kw) in bad.items():
        l0 = ctx.launch_count()
        with pytest.raises(CvbError, match="status 1"):
            _gpu(ctx, dict(base, **pk), **kw)
        assert ctx.launch_count() == l0, name
    for cm, dm, msg in ((2, 0, "Unknown projection type"), (0, 3, "Unknown distortion type")):
        l0 = ctx.launch_count()
        with pytest.raises(CvbError, match=f"status 3.*{msg}"):
            _gpu(ctx, dict(base, cam_model=np.array([cm], np.int32), dist_model=np.array([dm], np.int32), cam_xi=np.zeros(1)))
        assert ctx.launch_count() == l0
    got = _gpu(ctx, base)                                           # the context still works
    assert got[0].tolist() == [0, 0, 1]


# ------------------------------------------------------------------------------------------------------------------
# the C++ shim on mock containers
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_shim_on_mock_containers_equals_the_oracle(tmp_path):
    """covins_b200::RemoveLandmarkOutliers: EraseLandmark / EraseObservation for exactly the oracle's outlier observations in
    canonical order, then map->EraseLandmark for its erased landmarks in order, then the covisibility lists of what is left"""
    p = behind_some_cameras(synth_map.make_map(seed=23, n_agents=2, kf_per_agent=60, n_lm=4000), np.random.default_rng(23), 0.02)
    K, L = p["K"], p["L"]
    cam = np.zeros(18); cam[:7] = np.asarray(p["extr"]).reshape(-1, 7)[0]; cam[7:11] = p["intr"][0]; cam[11:15] = p["dist"][0]
    for name, a, dt in (("pose", p["pose"], np.float64), ("cam", cam, np.float64), ("lm", p["lm"], np.float64), ("ptr", p["lm_obs_ptr"], np.int32),
                        ("kf", p["obs_kf"], np.int32), ("uv", p["obs_uv"], np.float32), ("oct", p["obs_sigma"] / 2 - 1, np.float32)):
        np.ascontiguousarray(a, dt).tofile(tmp_path / f"{name}.bin")
    exe = str(tmp_path / "shim_outlier_test")
    _build_shim(exe)
    subprocess.check_call([exe, str(tmp_path), "0.92", "1.0", "2"])
    q = dict(p, cam_of_kf=np.zeros(K, np.int32))
    out, erase, _ = ora.landmark_outliers(q)
    assert (out == 1).sum() > 100 and (out == 2).sum() > 0 and erase.sum() > 0
    obs_lm = np.repeat(np.arange(L), np.diff(p["lm_obs_ptr"]))
    feat = np.zeros(len(out), np.int64)           # observation o is the n-th feature of its keyframe, n in CSR order
    seen = np.zeros(K, np.int64)
    for o, k in enumerate(p["obs_kf"]):
        feat[o] = seen[k]; seen[k] += 1
    expect = []
    for o in np.flatnonzero(out):
        expect += [[0, p["obs_kf"][o], feat[o]], [1, obs_lm[o], p["obs_kf"][o]]]
    expect += [[2, l, 0] for l in np.flatnonzero(erase)]
    log = np.fromfile(tmp_path / "out_log.bin", np.int32).reshape(-1, 3)
    assert np.array_equal(log, np.array(expect, np.int32).reshape(-1, 3))
    ref = ora_covis.covisibility(p["lm_obs_ptr"], p["obs_kf"], K, obs_skip=(out != 0).astype(np.uint8), lm_valid=(erase == 0).astype(np.uint8))
    cnt = np.fromfile(tmp_path / "out_cnt.bin", np.int32)
    assert np.array_equal(cnt, np.diff(ref[0]))
    assert np.array_equal(np.fromfile(tmp_path / "out_kf.bin", np.int32), ref[1])
    assert np.array_equal(np.fromfile(tmp_path / "out_w.bin", np.int32), ref[2])
