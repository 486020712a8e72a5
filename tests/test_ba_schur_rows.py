"""The Schur complement of the bundle adjustment, built one hi-keyframe row of S blocks at a time (schur_row_kernel,
covins_b200/csrc/ba_engine.cu), on the map shapes its row structure has edges at:

  long_row     keyframes with more observations than the kernel stages in shared memory (ROW_STAGE_MAX = 512), so Y of
               the rest of the row is recomputed where it is used, and blocks of more than 64 pair terms
  pair_counts  S blocks of exactly 1, 32 and 33 pair terms (a lane with no term, one term per lane, one lane with two),
               set by skipping observations of a keyframe
  sparse       a keyframe with no observation (its row only writes yb = 0) and landmarks left with one observation
               (not part of the landmark system)
  sharded      pair_counts over a group of two ranks on one device: each rank's rows see only its landmarks' observations

Each single-rank case asserts that the reduced right-hand side (debug vector 8), the linear-solve x (vector 7) and the
final state are bitwise the same over a repeated solve and a restart, that every iteration is within the extended-
precision bounds of test_ba_step_algebra.py (run_case on the same map), and that they are bitwise the values recorded in
tests/golden/ba_schur_rows.json from the build before the row kernel (obs_Y_kernel, kf_visual_kernel and schur_kernel,
same summation orders).  The sharded case runs through the in-process rank group (cvb_ba_solve_group), which returns
only the merged result: it has no restart and no debug vectors, so it asserts that two group solves give the same bits,
the golden hash of the merged state, and the world = 1 solve up to summation order.

The golden file was recorded on an H100 at commit 6699d84, the last commit with obs_Y_kernel / schur_kernel, with
`PYTHONPATH=. python tests/test_ba_schur_rows.py --record`.  Re-recording at a later commit turns the hashes into a
comparison of the code with itself: record only from a build whose Schur complement is independent of the code tested."""
import hashlib
import json
import os
import sys

import numpy as np
import pytest

import covins_b200
import test_ba_step_algebra as alg
from covins_b200 import optimization as O
from covins_b200 import synth_map as sm

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ba_schur_rows.json")
ROW_STAGE_MAX = 512
N_ITER = 4


def _obs_lm(p):
    return np.repeat(np.arange(p["L"]), np.diff(p["lm_obs_ptr"]))


def _pairs(p, skip):
    """(hi, lo) → number of pair terms, and observations per keyframe, as the engine lists them: landmarks with at least
    two kept observations; pairs (a, b), b <= a in observation order, keyed by (kf[a], kf[b])"""
    kf, lm = np.asarray(p["obs_kf"]), _obs_lm(p)
    keep = skip == 0
    cnt = np.bincount(lm[keep], minlength=p["L"])
    use = keep & (cnt[lm] >= 2)
    counts = {}
    by_lm = {}
    for o in np.flatnonzero(use):
        by_lm.setdefault(int(lm[o]), []).append(o)
    for obs in by_lm.values():
        for i, a in enumerate(obs):
            for b in obs[:i + 1]:
                key = (int(kf[a]), int(kf[b]))
                counts[key] = counts.get(key, 0) + 1
    return counts, np.bincount(kf[use], minlength=p["K"])


def _set_block(p, skip, hi, lo, n):
    """skip observations of keyframe hi on landmarks it shares with lo until the block (hi, lo) has n pair terms"""
    kf, lm = np.asarray(p["obs_kf"]), _obs_lm(p)
    for _ in range(10):
        c = _pairs(p, skip)[0].get((hi, lo), 0)
        if c == n:
            return
        assert c > n, (hi, lo, c, n)
        keep = skip == 0
        in_lo = set(lm[keep & (kf == lo)].tolist())
        cand = [o for o in np.flatnonzero(keep & (kf == hi)) if lm[o] in in_lo]
        skip[cand[:c - n]] = 1
    raise AssertionError("block not reached")


def case_long_row():
    p = sm.make_map(seed=61, n_agents=1, kf_per_agent=8, n_lm=1500, outlier_frac=0.0)
    return p, np.zeros(len(p["obs_kf"]), np.uint8)


def case_pair_counts():
    p = sm.make_map(seed=62, n_agents=1, kf_per_agent=14, n_lm=700, outlier_frac=0.0)
    skip = np.zeros(len(p["obs_kf"]), np.uint8)
    counts = _pairs(p, skip)[0]
    # three blocks of disjoint keyframes, hi > lo, with enough shared landmarks to cut down to the targets
    used, plan = set(), []
    for n in (33, 32, 1):
        hi, lo = next(k for k, c in sorted(counts.items(), key=lambda kv: -kv[1])
                      if k[0] != k[1] and c > n + 8 and not (set(k) & used))
        used |= {hi, lo}
        plan.append((hi, lo, n))
    for hi, lo, n in plan:
        _set_block(p, skip, hi, lo, n)
    return p, skip


def case_sparse():
    p = sm.make_map(seed=63, n_agents=2, kf_per_agent=10, n_lm=600, outlier_frac=0.0)
    kf, lm = np.asarray(p["obs_kf"]), _obs_lm(p)
    skip = (kf == 5).astype(np.uint8)            # keyframe 5 keeps no observation; the IMU chain holds it
    for l in range(0, p["L"], 9):                 # every 9th landmark keeps only its first observation
        obs = np.flatnonzero(lm == l)
        skip[obs[1:]] = 1
    return p, skip


CASES = {"long_row": case_long_row, "pair_counts": case_pair_counts, "sparse": case_sparse}


def _digest(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a, np.float64).tobytes())
    return h.hexdigest()


def _run(s, n):
    """vectors 7 and 8 after each iteration, then the final state"""
    out = []
    for _ in range(n):
        s.iterate(1)
        out.append(np.concatenate(s.debug_vector(8)))
        out.append(np.concatenate(s.debug_vector(7)))
    r = s.result()
    out += [r["pose"], r["speedbias"], r["lm"], np.asarray(r["cost"])]
    return out


def _single(ctx, name):
    p, skip = CASES[name]()
    s = O.BaSolver(ctx, p, visual_only=False, obs_skip=skip)
    try:
        a = _run(s, N_ITER)
        s.restart()
        b = _run(s, N_ITER)
    finally:
        s.close()
    s = O.BaSolver(ctx, p, visual_only=False, obs_skip=skip)
    try:
        c = _run(s, N_ITER)
    finally:
        s.close()
    return a, b, c


def _sharded(ctx):
    p, skip = case_pair_counts()
    ctxs = [covins_b200.Context(0) for _ in range(2)]
    g = O.Group(ctxs)
    try:
        got = [O.solve_group(g, p, N_ITER, obs_skip=skip) for _ in range(2)]
    finally:
        g.close()
        for c in ctxs:
            c.close()
    one = O.solve(ctx, p, N_ITER, obs_skip=skip)
    return got, one


def _state(r):
    return [r["pose"], r["speedbias"], r["lm"], np.asarray(r["cost"])]


def _golden():
    with open(GOLDEN) as f:
        return json.load(f)


# ---------------------------------------------------------------------------------------------------------- structure
def test_case_shapes():
    """each map has the row structure it exists for"""
    p, skip = case_long_row()
    counts, per_kf = _pairs(p, skip)
    assert per_kf.max() > ROW_STAGE_MAX and max(counts.values()) > 64
    p, skip = case_pair_counts()
    counts = _pairs(p, skip)[0]
    off = [c for (h, l), c in counts.items() if h != l]
    for n in (1, 32, 33):
        assert n in off, n
    assert max(counts.values()) > 64
    p, skip = case_sparse()
    counts, per_kf = _pairs(p, skip)
    assert per_kf[5] == 0 and (per_kf > 0).sum() == p["K"] - 1
    lm = _obs_lm(p)
    assert (np.bincount(lm[skip == 0], minlength=p["L"]) == 1).sum() >= 50


# ---------------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_row_schur_is_repeatable_and_golden(ctx, name):
    a, b, c = _single(ctx, name)
    for i, (x, y, z) in enumerate(zip(a, b, c)):
        assert np.array_equal(x, y, equal_nan=True), f"{name}: restart differs in output {i}"
        assert np.array_equal(x, z, equal_nan=True), f"{name}: repeated solve differs in output {i}"
    assert _digest(*a) == _golden()[name], f"{name}: differs from the recorded values"


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_row_schur_within_extended_precision(ctx, name, monkeypatch):
    def build():
        p, skip = CASES[name]()
        return alg._gba(p, False, skip)
    monkeypatch.setitem(alg.CASES, name, (build, N_ITER, set()))
    alg.run_case(ctx, name)


@pytest.mark.gpu
def test_row_schur_sharded_world_two(ctx):
    got, one = _sharded(ctx)
    for x, y in zip(_state(got[0]), _state(got[1])):
        assert np.array_equal(x, y), "sharded solve is not repeatable"
    assert got[0]["steps"] == one["steps"]
    inc = one["lm_owner"] >= 0
    for key in ("pose", "speedbias"):
        assert np.abs(got[0][key] - one[key]).max() <= 1e-8 * max(1.0, np.abs(one[key]).max()), key
    assert np.abs(got[0]["lm"][inc] - one["lm"][inc]).max() <= 1e-8 * max(1.0, np.abs(one["lm"][inc]).max())
    assert _digest(*_state(got[0])) == _golden()["sharded"], "sharded: differs from the recorded values"


def _record():
    ctx = covins_b200.Context(0)
    out = {name: _digest(*_single(ctx, name)[0]) for name in sorted(CASES)}
    out["sharded"] = _digest(*_state(_sharded(ctx)[0][0]))
    ctx.close()
    os.makedirs(os.path.dirname(GOLDEN), exist_ok=True)
    with open(GOLDEN, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    if "--record" in sys.argv:
        _record()
