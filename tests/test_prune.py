"""cvb_redundant_keyframes: the keyframes the sequential redundancy-culling pass of Map::Clean (map_be.cpp:745-811)
removes, found by parallel rounds (include/covins_b200.h states the rule; oracle/prune_oracle.c carries the assumption).
CPU: the C oracle (incremental, one thread) equals an independent plain-Python restatement that recomputes red_C(k) and
pred_C(k) from scratch for every k: on hand cases that each pin one clause (also pinned to literal sets), on random small
maps and on C1; a naive "evaluate all, cull all" differs on the two chain cases; the rule is monotone in C and the
oracle's set is its own fixed point; the C++ shim compiles and refuses missing input.
GPU: through the C-ABI the culled set equals the oracle's: hand cases, C1 and C3 with and without the outlier mask a GBA
round erases, at a setting that culls a third of the map over hundreds of rounds and one that culls nothing; repeatability
and launch counts; refused inputs; empty maps; the C++ shim on mock containers.
"""
import os
import subprocess

import numpy as np
import pytest

from oracle import covis as ora_covis
from oracle import prune as ora

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------------------------
# maps
# ------------------------------------------------------------------------------------------------------------------
def _case(tracks, K, octs=None, pred=None, time=None, protect=(), th_red=0.5, max_time_dist=100.0, th_obs=3, skip=None, valid=None):
    """tracks: observer lists per landmark; octs: the octaves, same shape (default 0); one chain 0 .. K-1 at times 0 .. K-1"""
    ptr = np.concatenate([[0], np.cumsum([len(t) for t in tracks])]).astype(np.int32)
    kf = np.array([k for t in tracks for k in t], np.int32)
    octv = np.array([o for t in (octs or [[0] * len(t) for t in tracks]) for o in t], np.int32)
    prot = np.zeros(K, np.uint8)
    prot[list(protect)] = 1
    return dict(lm_obs_ptr=ptr, obs_kf=kf, obs_octave=octv,
                kf_pred=np.array(pred if pred is not None else np.arange(K) - 1, np.int32),
                kf_time=np.array(time if time is not None else np.arange(K), np.float64), kf_protect=prot, th_red=th_red,
                max_time_dist=max_time_dist, th_obs=th_obs,
                obs_skip=None if skip is None else np.asarray(skip, np.uint8), lm_valid=None if valid is None else np.asarray(valid, np.uint8))


ALL_BUT_1 = (0, 2, 3, 4, 5)


def hand_cases():
    return {   # name → (case, literal culled set)
        # others at octave o + 1 count ...
        "octave_plus_one_counts": (_case([[1, 2, 3, 4]], 6, octs=[[1, 2, 2, 2]], protect=ALL_BUT_1), {1}),
        # ... at o + 2 they do not
        "octave_plus_two_does_not": (_case([[1, 2, 3, 4]], 6, octs=[[1, 2, 2, 3]], protect=ALL_BUT_1), set()),
        "exactly_th_obs_others": (_case([[1, 2, 3, 4]], 6, protect=ALL_BUT_1), {1}),
        "one_other_too_few": (_case([[1, 2, 3]], 6, protect=ALL_BUT_1), set()),
        # red = 1 of n = 2 at th_red 0.5: red == th_red * n is not enough
        "red_equal_to_th_red_n": (_case([[1, 2, 3, 4], [1, 2]], 6, protect=ALL_BUT_1), set()),
        "red_above_th_red_n": (_case([[1, 2, 3, 4], [1, 2]], 6, protect=ALL_BUT_1, th_red=0.49), {1}),
        # n(1) = 0, even at th_red 0: 0 > 0 fails
        "no_landmarks": (_case([[0, 2, 3, 4]], 6, protect=(0, 2, 3, 4, 5), th_red=0.0), set()),
        "protected": (_case([[1, 2, 3, 4]], 6, protect=range(6)), set()),
        # 0 has no predecessor, 5 no successor: both redundant, neither culled
        "missing_pred_or_succ": (_case([[0, 1, 2, 3], [5, 2, 3, 4]], 6, protect=(1, 2, 3, 4)), set()),
        # succ(1) - pred(1) = 2.5 - 0.5 = max_time_dist: culled; 3 has a gap of 2.5 > 2: kept
        "gap_equal_to_max_time_dist": (_case([[1, 2, 4, 5], [3, 2, 4, 5]], 6, time=[0.5, 1.5, 2.5, 3.0, 5.5, 6.0], protect=(0, 2, 4, 5),
                                             max_time_dist=2.0), {1}),
        # two agents interleaved in the canonical order: chains 0-2-4-6 and 1-3-5-7; 2 and 3 are redundant
        "two_agents": (_case([[2, 0, 4, 6], [3, 1, 5, 7]], 8, pred=[-1, -1, 0, 1, 2, 3, 4, 5], time=[0, 0, 1, 1, 2, 2, 3, 3],
                             protect=(0, 1, 4, 5, 6, 7), max_time_dist=2.0), {2, 3}),
        # one skipped observation of 4 leaves 1 two others on landmark 0; landmark 1 (redundant for 1) is invalid: n(1) = 1
        "skipped_observation_and_invalid_landmark": (_case([[1, 2, 3, 4], [1, 2, 3, 4]], 6, protect=ALL_BUT_1, th_red=0.0,
                                                           skip=[0, 0, 0, 1, 0, 0, 0, 0], valid=[1, 0]), set()),
        # culling 1 leaves 2 with only two others on the landmark they share: 2 is kept
        "cull_makes_next_non_redundant": (_case([[1, 2, 3, 4]], 6, protect=(0, 3, 4, 5)), {1}),
        # culling 1 moves pred_C(2) to 0: succ(2) - pred_C(2) = 3 - 0 > 2, so 2 is kept
        "cull_widens_next_gap": (_case([[1, 3, 4, 5], [2, 3, 4, 5]], 6, protect=(0, 3, 4, 5), max_time_dist=2.0), {1}),
    }


CASES = hand_cases()


def random_case(seed):
    """A agents' chains interleaved in index order, tracks over a window of neighbouring keyframes, random octaves, masks"""
    rng = np.random.default_rng(seed)
    A = int(rng.integers(1, 4)); per = int(rng.integers(3, 30)); K = A * per
    agent = np.tile(np.arange(A), per); kid = np.repeat(np.arange(per), A)             # canonical (kf id, agent) order
    pred = np.where(kid > 0, np.arange(K) - A, -1)
    time = kid + rng.uniform(0, 0.9, K)
    tracks, octs = [], []
    for _ in range(int(rng.integers(1, 25 * K))):
        c = int(rng.integers(0, K)); near = np.arange(max(0, c - 4 * A), min(K, c + 4 * A + 1))
        t = rng.choice(near, int(min(len(near), rng.integers(1, 9))), replace=False).tolist()
        tracks.append(t); octs.append(rng.integers(0, 8, len(t)).tolist())
    n = sum(len(t) for t in tracks)
    c = _case(tracks, K, octs=octs, pred=pred, time=time, protect=np.nonzero(rng.random(K) < 0.1)[0], th_red=float(rng.uniform(0.2, 0.9)),
              max_time_dist=float(rng.uniform(1.0, 6.0)), th_obs=int(rng.integers(1, 5)),
              skip=(rng.random(n) < 0.1) if seed % 2 else None, valid=(rng.random(len(tracks)) < 0.9) if seed % 3 else None)
    return c


def synthetic(p, skip, setting):
    """the flat problem of a synthetic map: chains by agent, 10 Hz timestamps, each agent's first keyframe and the loop
    constraints' keyframes protected, octave = obs_sigma / 2 - 1"""
    K = p["K"]
    prot = (p["kf_id"] == 0).astype(np.uint8)
    prot[p["loop_i"]] = 1; prot[p["loop_j"]] = 1
    return dict(lm_obs_ptr=p["lm_obs_ptr"], obs_kf=p["obs_kf"], obs_octave=(p["obs_sigma"] / 2 - 1).astype(np.int32),
                kf_pred=np.where(p["kf_id"] > 0, np.arange(K) - 1, -1).astype(np.int32), kf_time=p["kf_id"] / 10.0, kf_protect=prot,
                th_obs=3, obs_skip=p["obs_is_outlier"].astype(np.uint8) if skip else None, lm_valid=None, **SETTINGS[setting])


SETTINGS = {"culls_a_third": dict(th_red=0.75, max_time_dist=1.0), "culls_nothing": dict(th_red=0.9, max_time_dist=1.0)}


# ------------------------------------------------------------------------------------------------------------------
# the independent restatement: no incremental state
# ------------------------------------------------------------------------------------------------------------------
def _participating(c):
    ptr, kf, octv = c["lm_obs_ptr"], c["obs_kf"], c["obs_octave"]
    obs = []   # (keyframe, landmark, octave)
    for l in range(len(ptr) - 1):
        if c["lm_valid"] is not None and not c["lm_valid"][l]:
            continue
        for o in range(ptr[l], ptr[l + 1]):
            if c["obs_skip"] is None or not c["obs_skip"][o]:
                obs.append((int(kf[o]), l, int(octv[o])))
    return obs


def passes(c, obs, k, C):
    """the culling test of keyframe k for the culled set C, from scratch"""
    K = len(c["kf_pred"])
    mine = [(l, o) for (kk, l, o) in obs if kk == k]
    if c["kf_protect"][k] or not mine:
        return False
    red = 0
    for l, o in mine:
        others = sum(1 for (kk, ll, oo) in obs if ll == l and kk != k and kk not in C and oo <= o + 1)
        red += others >= c["th_obs"]
    if not float(red) > c["th_red"] * float(len(mine)):
        return False
    p = int(c["kf_pred"][k])
    while p >= 0 and p in C:
        p = int(c["kf_pred"][p])
    succ = [j for j in range(K) if c["kf_pred"][j] == k]
    return p >= 0 and len(succ) == 1 and c["kf_time"][succ[0]] - c["kf_time"][p] <= c["max_time_dist"]


def restated(c):
    obs = _participating(c)
    C = set()
    for k in range(len(c["kf_pred"])):
        if passes(c, obs, k, C):
            C.add(k)
    return C


def naive(c):
    """every keyframe tested against the empty set and all passing ones culled at once: NOT the pass"""
    obs = _participating(c)
    return {k for k in range(len(c["kf_pred"])) if passes(c, obs, k, set())}


def _oracle(c):
    return ora.redundant_keyframes(**c)


def _set(culled):
    return set(np.nonzero(culled)[0].tolist())


# ------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_equals_restatement_on_hand_cases(name):
    c, literal = CASES[name]
    got = _set(_oracle(c))
    assert got == restated(c) == literal


def test_naive_parallel_culling_differs_on_the_chain_cases():
    for name in ("cull_makes_next_non_redundant", "cull_widens_next_gap"):
        c, literal = CASES[name]
        assert naive(c) == {1, 2} != literal, name


@pytest.mark.parametrize("seed", range(8))
def test_oracle_equals_restatement_on_random_maps(seed):
    c = random_case(seed)
    assert _set(_oracle(c)) == restated(c)


def test_oracle_equals_restatement_on_c1():
    from covins_b200 import synth_map
    p = synth_map.make_config("C1")
    for setting in SETTINGS:
        c = synthetic(p, False, setting)
        obs = _participating(c)
        by_lm = {}
        for kk, l, o in obs:
            by_lm.setdefault(l, []).append((kk, o))
        got = _set(_oracle(c))
        # the restatement with the observers indexed by landmark (same rule, from scratch for every k)
        C = set()
        mine = {}
        for kk, l, o in obs:
            mine.setdefault(kk, []).append((l, o))
        for k in range(p["K"]):
            if c["kf_protect"][k] or k not in mine:
                continue
            red = sum(sum(1 for kk, oo in by_lm[l] if kk != k and kk not in C and oo <= o + 1) >= 3 for l, o in mine[k])
            pr = int(c["kf_pred"][k])
            while pr >= 0 and pr in C:
                pr = int(c["kf_pred"][pr])
            s = k + 1 if k + 1 < p["K"] and c["kf_pred"][k + 1] == k else -1
            if float(red) > c["th_red"] * len(mine[k]) and pr >= 0 and s >= 0 and c["kf_time"][s] - c["kf_time"][pr] <= c["max_time_dist"]:
                C.add(k)
        assert got == C, setting
        assert (len(got) > 0.2 * p["K"]) == (setting == "culls_a_third") and (len(got) == 0) == (setting == "culls_nothing")


@pytest.mark.parametrize("seed", range(4))
def test_rule_is_monotone_and_the_oracle_is_its_fixed_point(seed):
    """passes(k, C2) implies passes(k, C1) for C1 ⊆ C2 ⊆ {0..k-1}; and k is culled iff it passes under the culls below it"""
    c = random_case(100 + seed)
    obs = _participating(c)
    culled = _set(_oracle(c))
    rng = np.random.default_rng(seed)
    K = len(c["kf_pred"])
    for k in range(K):
        assert (k in culled) == passes(c, obs, k, {j for j in culled if j < k})
        below = np.arange(k)
        for _ in range(3):
            C2 = set(below[rng.random(k) < 0.5].tolist())
            C1 = {j for j in C2 if rng.random() < 0.5}
            assert not passes(c, obs, k, C2) or passes(c, obs, k, C1)


def test_shim_prune_compiles_and_refuses_missing_input(tmp_path):
    exe = str(tmp_path / "shim_prune_test")
    _build_shim(exe)
    assert subprocess.run([exe, str(tmp_path), "0.5", "1.0", "3"]).returncode == 2     # nothing dumped: refused before any GPU work


def _build_shim(exe):
    import covins_b200
    if not os.path.exists(covins_b200.LIB_PATH):
        covins_b200.build()
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-o", exe, os.path.join(ROOT, "tests", "cpp", "shim_prune_test.cpp"),
                           "-L" + os.path.join(ROOT, "covins_b200"), "-lcovins_b200", "-Wl,-rpath," + os.path.join(ROOT, "covins_b200")])


# ------------------------------------------------------------------------------------------------------------------
# GPU, through the C-ABI
# ------------------------------------------------------------------------------------------------------------------
def _gpu(ctx, c, num_octaves=8):
    from covins_b200 import mapgraph
    return mapgraph.redundant_keyframes(ctx, num_octaves=num_octaves, **c)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_hand_cases_equal_the_oracle(ctx, name):
    c, literal = CASES[name]
    got, rounds = _gpu(ctx, c)
    assert np.array_equal(got, _oracle(c)) and _set(got) == literal and rounds >= 0


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(8))
def test_random_maps_equal_the_oracle(ctx, seed):
    c = random_case(seed)
    assert np.array_equal(_gpu(ctx, c)[0], _oracle(c))


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["C1", "C3"])
@pytest.mark.parametrize("gba_mask", [False, True])
@pytest.mark.parametrize("setting", sorted(SETTINGS))
def test_synthetic_maps_equal_the_oracle(ctx, config, gba_mask, setting):
    """the mask is the gross outliers a GBA round erases (obs_is_outlier of the synthetic map)"""
    from covins_b200 import synth_map
    p = synth_map.make_config(config)
    c = synthetic(p, gba_mask, setting)
    got, rounds = _gpu(ctx, c)
    ref = _oracle(c)
    assert np.array_equal(got, ref)
    if setting == "culls_a_third":
        assert ref.sum() >= 0.2 * p["K"] and rounds > 10, (int(ref.sum()), rounds)
    else:
        assert ref.sum() == 0 and rounds == 1


@pytest.mark.gpu
def test_two_runs_are_identical_and_launches_follow_the_rounds(ctx):
    from covins_b200 import synth_map
    p = synth_map.make_config("C1")
    for c in (synthetic(p, True, "culls_a_third"), synthetic(p, False, "culls_nothing"), random_case(3)):
        outs = []
        for _ in range(2):
            l0 = ctx.launch_count()
            got, rounds = _gpu(ctx, c)
            assert ctx.launch_count() - l0 == 1 + 3 * rounds       # histogram once; evaluate, commit, re-link per round
            outs.append((got.tobytes(), rounds))
        assert outs[0] == outs[1]


@pytest.mark.gpu
def test_empty_maps(ctx):
    from covins_b200 import lib
    empty = _case([], 0)
    assert _gpu(ctx, empty)[0].shape == (0,)
    rc = lib().cvb_redundant_keyframes(ctx.handle, 0, 0, None, None, None, None, None, None, None, None, 0.5, 1.0, 3, 8, None, None)
    assert rc == 0
    l0 = ctx.launch_count()
    got, rounds = _gpu(ctx, _case([], 5))                              # keyframes without landmarks
    assert not got.any() and rounds == 0 and ctx.launch_count() == l0


@pytest.mark.gpu
def test_invalid_input_is_refused_before_any_launch(ctx):
    from covins_b200 import CvbError, lib
    base, _ = CASES["exactly_th_obs_others"]
    bad = {
        "duplicate observer": dict(obs_kf=np.array([1, 2, 3, 2], np.int32)),
        "octave too large": dict(obs_octave=np.array([0, 0, 8, 0], np.int32)),
        "octave negative": dict(obs_octave=np.array([0, -1, 0, 0], np.int32)),
        "kf_pred not below k": dict(kf_pred=np.array([-1, 1, 1, 2, 3, 4], np.int32)),
        "kf_pred below -1": dict(kf_pred=np.array([-2, 0, 1, 2, 3, 4], np.int32)),
        "two successors": dict(kf_pred=np.array([-1, 0, 0, 2, 3, 4], np.int32)),
        "th_red NaN": dict(th_red=float("nan")),
        "th_red above 1": dict(th_red=1.5),
        "th_red negative": dict(th_red=-0.1),
        "max_time_dist 0": dict(max_time_dist=0.0),
        "max_time_dist NaN": dict(max_time_dist=float("nan")),
        "th_obs 0": dict(th_obs=0),
        "ptr decreasing": dict(lm_obs_ptr=np.array([0, 4, 2], np.int32)),
        "ptr not from 0": dict(lm_obs_ptr=np.array([1, 4], np.int32)),
        "kf out of range": dict(obs_kf=np.array([1, 2, 3, 6], np.int32)),
    }
    for name, kw in bad.items():
        c = dict(base, **kw)
        l0 = ctx.launch_count()
        with pytest.raises(CvbError, match="status 1: cvb_redundant_keyframes"):
            _gpu(ctx, c)
        assert ctx.launch_count() == l0, name
    l0 = ctx.launch_count()
    with pytest.raises(CvbError, match="status 1: cvb_redundant_keyframes"):
        _gpu(ctx, base, num_octaves=0)
    assert ctx.launch_count() == l0
    assert np.array_equal(_gpu(ctx, base)[0], _oracle(base))                  # the context still works


# ------------------------------------------------------------------------------------------------------------------
# the C++ shim on mock containers
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_shim_on_mock_containers_equals_the_oracle(tmp_path):
    """covins_b200::PruneRedundantKeyframes: SetInvalid on exactly the oracle's set in ascending canonical order (the mock
    map orders keyframes by (keyframe id, agent), interleaving the agents), then the covisibility lists of the rest"""
    from covins_b200 import synth_map
    p = synth_map.make_map(seed=23, n_agents=2, kf_per_agent=60, n_lm=4000)
    K = p["K"]
    octv = (p["obs_sigma"] / 2 - 1).astype(np.int32)
    loops = np.stack([p["loop_i"], p["loop_j"]], 1).astype(np.int32)
    for name, a in (("ptr", p["lm_obs_ptr"]), ("kf", p["obs_kf"]), ("oct", octv), ("agent", p["agent_of"]), ("kfid", p["kf_id"]), ("loops", loops)):
        np.ascontiguousarray(a, np.int32).tofile(tmp_path / f"{name}.bin")
    (p["kf_id"] / 10.0).tofile(tmp_path / "time.bin")
    exe = str(tmp_path / "shim_prune_test")
    _build_shim(exe)
    subprocess.check_call([exe, str(tmp_path), "0.75", "1.0", "3"])
    # the expected result in canonical order: keyframe number n has canonical index rank[n]
    order = np.lexsort((p["agent_of"], p["kf_id"]))                                 # canonical index → keyframe number
    rank = np.empty(K, np.int64); rank[order] = np.arange(K)
    ptr, kf = p["lm_obs_ptr"], rank[p["obs_kf"]]
    lm = np.repeat(np.arange(p["L"]), np.diff(ptr))
    o = np.lexsort((kf, lm))                                                        # each landmark's observers by canonical index
    prot = (p["kf_id"][order] == 0).astype(np.uint8)
    prot[rank[loops.reshape(-1)]] = 1
    pred_num = np.where(p["kf_id"] > 0, np.arange(K) - 1, -1)
    c = dict(lm_obs_ptr=ptr, obs_kf=kf[o].astype(np.int32), obs_octave=octv[o], kf_pred=np.where(pred_num[order] >= 0, rank[pred_num[order]], -1).astype(np.int32),
             kf_time=p["kf_id"][order] / 10.0, kf_protect=prot, th_red=0.75, max_time_dist=1.0, th_obs=3, obs_skip=None, lm_valid=None)
    culled = _oracle(c)
    assert culled.sum() > 0.1 * K
    inv = np.fromfile(tmp_path / "out_invalidated.bin", np.int32)
    assert np.array_equal(inv, order[np.nonzero(culled)[0]])
    # covisibility of the remaining keyframes, in canonical order, mapped back to keyframe numbers
    ref = ora_covis.covisibility(c["lm_obs_ptr"], c["obs_kf"], K, obs_skip=culled[c["obs_kf"]])
    cnt = np.fromfile(tmp_path / "out_cnt.bin", np.int32)
    assert np.array_equal(cnt[order], np.diff(ref[0]))
    got_kf = np.fromfile(tmp_path / "out_kf.bin", np.int32); got_w = np.fromfile(tmp_path / "out_w.bin", np.int32)
    start = np.concatenate([[0], np.cumsum(cnt)])
    for i in range(K):
        n = order[i]
        assert np.array_equal(got_kf[start[n]:start[n + 1]], order[ref[1][ref[0][i]:ref[0][i + 1]]])
        assert np.array_equal(got_w[start[n]:start[n + 1]], ref[2][ref[0][i]:ref[0][i + 1]])
