"""Place-recognition requests against the map descriptor database spread over a rank group (cvb_db_group_*), one rank per
device, at group sizes 1, 2, 4 and 8 (capped by the device count):

  C5 SIFT   300 queries against 10 000 keyframes x 300 rows (cvb_db_group_match_l2)
  C3 ORB    1 000 queries against 2 000 keyframes x 1 000 rows (cvb_db_group_match_hamming)

and, for reference, the same request on the single-context database (cvb_db).  Every database of a workload is built
first; the requests then alternate between them, so that each size sees the same conditions.  Each request is timed
host to host (a host clock around the call, which ends in a synchronise of rank 0's stream); the median, min and max
over --reps requests after --warmup requests of every size are reported.  Every group's outputs are checked bit-identical
to the single database's.  The card's name and power limit are printed next to the numbers; a size above the device count
is reported "not measured".

  python tools/db_group_timing.py [--reps 60] [--warmup 5] [--only c5|c3] [--json PATH]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZES = (1, 2, 4, 8)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out or ["unknown"]
    except (OSError, subprocess.SubprocessError):
        return ["unknown"]


def c5_map():
    """300 SIFT queries, 10 000 keyframes x 300 rows (u8 values): ten seeded blocks of 1 000 keyframes; the query is a
    keyframe of the first block, so it shares landmarks with that block's keyframes"""
    from covins_b200 import synth
    blocks = []
    for b in range(10):
        d, _ = synth.sift_keyframes(seed=50 + b, n_kf=1001 if b == 0 else 1000, n_feat=300)
        blocks.append(d.astype(np.uint8))
    q = blocks[0][0].astype(np.float32)
    blocks[0] = blocks[0][1:]
    return q, blocks, 300


def c3_map():
    from covins_b200 import synth
    d, _ = synth.orb_keyframes(seed=3, n_kf=2001, n_feat=1000)
    return d[0], [d[1:]], 1000


def bits(x):
    x = np.ascontiguousarray(x)
    return x.view(np.int32) if x.dtype == np.float32 else x.astype(np.int64)


def run(name, kind, make, ctxs, a):
    import covins_b200.matching as M
    from covins_b200 import optimization as O
    q, blocks, n_feat = make()
    n_kf = sum(len(b) for b in blocks)
    fdt = np.float32 if kind == "sift" else np.uint8

    def fill(db):
        for b in blocks:
            db.append(b.reshape(-1, b.shape[-1]).astype(fdt), [n_feat] * len(b))

    dbs = {"single": M.DescriptorDatabase(ctxs[0], reserve_rows=n_kf * n_feat, kind=kind)}
    fill(dbs["single"])
    groups = []
    for n in SIZES:
        if n <= len(ctxs):
            groups.append(O.Group(ctxs[:n]))
            dbs[n] = M.DescriptorDatabaseGroup(groups[-1], kind=kind)
            fill(dbs[n])
    match = "match_l2" if kind == "sift" else "match_hamming"
    times = {k: [] for k in dbs}
    last = {}
    for rep in range(a.warmup + a.reps):
        for k, db in dbs.items():
            t0 = time.perf_counter()
            out = getattr(db, match)(q)
            dt = time.perf_counter() - t0
            if rep >= a.warmup:
                times[k].append(dt)
            last[k] = out
    ref = last["single"]
    res = {"workload": name, "kind": kind, "nq": len(q), "n_kf": n_kf, "rows_per_kf": n_feat,
           "accepted_matches": int(ref[0].sum()), "reps": a.reps, "warmup": a.warmup, "sizes": {}}
    for k in list(dbs):
        same = all(np.array_equal(bits(u), bits(v)) for u, v in zip(last[k], ref))
        v = np.array(times[k]) * 1e3
        res["sizes"][str(k)] = {"median_ms": float(np.median(v)), "min_ms": float(v.min()), "max_ms": float(v.max()),
                                "identical_to_single": bool(same)}
        if k != "single":
            res["sizes"][str(k)]["rows_per_rank"] = [int(x) for x in dbs[k].size_per_rank()[2]]
    for n in SIZES:
        if n > len(ctxs):
            res["sizes"][str(n)] = "not measured"
    for db in dbs.values():
        db.close()
    for g in groups:
        g.close()
    print(f"{name}: {len(q)} queries vs {n_kf} keyframes x {n_feat} rows ({kind}); {res['accepted_matches']} accepted matches")
    for k, r in res["sizes"].items():
        label = "cvb_db" if k == "single" else f"group of {k}"
        if isinstance(r, str):
            print(f"  {label:12s} {r}")
        else:
            print(f"  {label:12s} median {r['median_ms']:8.3f} ms  (min {r['min_ms']:.3f}, max {r['max_ms']:.3f})  "
                  f"identical: {r['identical_to_single']}")
    assert all(isinstance(r, str) or r["identical_to_single"] for r in res["sizes"].values()), "outputs differ"
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--only", choices=("c5", "c3"), default=None)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    assert a.reps >= 50, "the medians are taken over at least 50 requests"

    import torch
    import covins_b200
    n_dev = torch.cuda.device_count()
    if n_dev < 1:
        raise SystemExit("no CUDA device: nothing can be measured")
    ctxs = [covins_b200.Context(d) for d in range(min(n_dev, max(SIZES)))]
    cards = card()
    print("cards (name, power limit):", "; ".join(cards))
    out = {"cards": cards, "devices": n_dev, "workloads": []}
    if a.only in (None, "c5"):
        out["workloads"].append(run("C5 SIFT", "sift", c5_map, ctxs, a))
    if a.only in (None, "c3"):
        out["workloads"].append(run("C3 ORB", "orb", c3_map, ctxs, a))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)
    for c in ctxs:
        c.close()


if __name__ == "__main__":
    main()
