#!/usr/bin/env python
"""Times the removal of a culled set of keyframes from the resident map descriptor database: one cvb_db_remove_batch call
against the per-keyframe loop of cvb_db_remove (highest index first) that it replaces.

Databases, at the sizes of BASELINE configs C3 and C5:
  * C3 ORB: 2 000 keyframes x 1 000 rows; the removed set is the one cvb_redundant_keyframes (K14) culls on the C3
    synthetic map (the problem of tools/prune_bench.py);
  * C5 ORB: 10 008 keyframes x 1 000 rows, and C5 SIFT: 10 008 keyframes x 300 rows; a seeded 30 % of the keyframes.
Rows are random bytes: the cost of a removal depends only on the shapes.

One JSON line per database, with the card's name, power limit and SM clocks read in the same run:
  * batch_ms_*: end-to-end host time of one cvb_db_remove_batch call (it returns after its one synchronisation), median,
    min and max over --reps calls, each on a freshly built database (the first build is a warm-up);
  * batch_kernel_ms: the K18 kernel's summed time in that call from a torch.profiler (CUPTI) pass of its own, and
    batch_copy_ms the device-to-device copies back; moved_bytes = 4 x the kept suffix bytes (gathered: read + write,
    copied back: read + write), and their rate over the batch's device time against the H100 SXM data-sheet 3.35 TB/s;
  * loop_ms: the loop of cvb_db_remove from the highest index down, on another fresh database.  The loop stops after
    --loop-budget-s seconds; then loop_extrapolated is true, the remaining removals' time is predicted from a least-squares
    fit t = a + b * moved bytes over the measured ones, and the rest of the set goes in one batch so that the comparison
    below still runs;
  * equal: the batch database and the loop database answer one request (500 rows of a surviving keyframe) identically,
    and their sizes agree.
There is no fallback: without a CUDA device the script fails.
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
sys.path.insert(0, os.path.join(ROOT, "tools"))

HBM_BYTES_PER_S = 3.35e12
TILE_BYTES = {"orb": 36864, "sift": 16896}     # one 128-row operand tile (cvb_tc::tile_bytes)
DIM = {"orb": 32, "sift": 128}


def c3_culled_set(ctx):
    """the keyframes K14 culls on the C3 synthetic map, with tools/prune_bench.py's thresholds"""
    from covins_b200 import mapgraph, synth_map
    from prune_bench import problem
    culled, _ = mapgraph.redundant_keyframes(ctx, **problem(synth_map.make_config("C3"), 0.75, 1.0))
    return np.flatnonzero(culled)


def moved_bytes(kind, lens, removed):
    """4 x the bytes of rows and tiles kept after the first removed keyframe that holds rows (what one batch moves)"""
    gone = np.zeros(len(lens), bool)
    gone[removed] = True
    first = int(np.flatnonzero(gone & (lens > 0))[0])
    kept = ~gone[first:]
    rows = lens[first:][kept].sum() * DIM[kind]
    tiles = ((lens[first:][kept] + 127) // 128).sum() * TILE_BYTES[kind]
    return 4 * int(rows + tiles)


def tail_bytes(kind, lens_now, i):
    """the bytes one cvb_db_remove(i) moves: 4 x the rows and tiles after keyframe i"""
    tail = lens_now[i + 1:]
    return 4 * int(tail.sum() * DIM[kind] + ((tail + 127) // 128).sum() * TILE_BYTES[kind])


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--cases", default="C3-orb,C5-orb,C5-sift")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--loop-budget-s", type=float, default=30.0)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("db_remove_bench: no CUDA device (there is no CPU fallback)")
    import covins_b200
    from covins_b200 import matching as M
    from torch.profiler import ProfilerActivity, profile
    card = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader", "-i", "0"],
                                   text=True).strip()
    ctx = covins_b200.Context(0)
    rng = np.random.default_rng(a.seed)
    for case in a.cases.split(","):
        config, kind = case.split("-")
        K, rows = {"C3": 2000, "C5": 10_008}[config], {"orb": 1000, "sift": 300}[kind]
        if config == "C3":
            removed = c3_culled_set(ctx)
            assert len(removed) and removed.max() < K
        else:
            removed = np.sort(rng.choice(K, size=int(0.3 * K), replace=False))
        order = rng.permutation(removed)                     # the batch takes them unsorted
        lens = np.full(K, rows, np.int64)
        data = rng.integers(0, 256, size=(K * rows, DIM[kind]), dtype=np.uint8)
        if kind == "sift":
            data = data.astype(np.float32)
        rpk = lens.astype(np.int32)

        def fresh():
            db = M.DescriptorDatabase(ctx, kind=kind)
            db.append(data, rpk)
            torch.cuda.synchronize()
            return db

        # ---- the batch
        batch_ms = []
        fresh().close()                                      # warm-up: allocations and the pool
        for _ in range(a.reps):
            db = fresh()
            t0 = time.perf_counter()
            db.remove_batch(order)
            batch_ms.append((time.perf_counter() - t0) * 1e3)
            db.close()
        db = fresh()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            db.remove_batch(order)
            torch.cuda.synchronize()
        ev = prof.key_averages()
        kern_ms = sum(e.device_time_total for e in ev if "db_remove_gather_kernel" in e.key) / 1e3
        copy_ms = sum(e.device_time_total for e in ev if "Memcpy DtoD" in e.key) / 1e3
        batch_db = db
        nbytes = moved_bytes(kind, lens, removed)
        dev_s = (kern_ms + copy_ms) / 1e3
        # ---- the loop, highest index first
        loop_db = fresh()
        lens_now = lens.copy()
        times, moved = [], []
        t_start = time.perf_counter()
        down = np.sort(removed)[::-1]
        done = 0
        for i in down:
            moved.append(tail_bytes(kind, lens_now, int(i)))
            t0 = time.perf_counter()
            loop_db.remove(int(i))
            times.append(time.perf_counter() - t0)
            lens_now = np.delete(lens_now, int(i))
            done += 1
            if time.perf_counter() - t_start > a.loop_budget_s:
                break
        loop_s = float(np.sum(times))
        extrapolated = done < len(down)
        fit = None
        if extrapolated:
            rest = [int(i) for i in down[done:]]
            rest_bytes = []
            for i in rest:
                rest_bytes.append(tail_bytes(kind, lens_now, i))
                lens_now = np.delete(lens_now, i)
            A = np.stack([np.ones(len(moved)), np.asarray(moved, np.float64)], 1)
            coef = np.linalg.lstsq(A, np.asarray(times), rcond=None)[0]
            loop_s += float(coef[0] * len(rest) + coef[1] * np.sum(rest_bytes))
            fit = dict(s_per_call=float(coef[0]), s_per_GB=float(coef[1] * 1e9))
            loop_db.remove_batch(rest)                       # the rest at once, so that the databases can be compared
        # ---- equality on one request
        first_kept = int(np.flatnonzero(~np.isin(np.arange(K), removed))[0])
        q = data[first_kept * rows:first_kept * rows + min(rows, 500)]
        match = "match_hamming" if kind == "orb" else "match_l2"
        r1, r2 = getattr(batch_db, match)(q), getattr(loop_db, match)(q)
        equal = batch_db.size() == loop_db.size() == (K - len(removed), int((K - len(removed)) * rows)) and all(
            np.array_equal(np.ascontiguousarray(x).view(np.int32), np.ascontiguousarray(y).view(np.int32)) for x, y in zip(r1, r2))
        matches = int(r1[0].sum())
        batch_db.close(); loop_db.close()
        print(json.dumps(dict(
            case=case, card=card, n_kf=K, rows_per_kf=rows, removed=int(len(removed)), first_removed=int(removed.min()),
            db_bytes=int(K * rows * DIM[kind] + K * ((rows + 127) // 128) * TILE_BYTES[kind]),
            batch_ms_median=round(float(np.median(batch_ms)), 3), batch_ms_min=round(min(batch_ms), 3), batch_ms_max=round(max(batch_ms), 3),
            reps=a.reps, batch_kernel_ms=round(kern_ms, 3), batch_copy_ms=round(copy_ms, 3), moved_bytes=nbytes,
            moved_GBps=round(nbytes / dev_s / 1e9, 1) if dev_s > 0 else None,
            moved_share_of_3_35TBps=round(nbytes / dev_s / HBM_BYTES_PER_S, 3) if dev_s > 0 else None,
            loop_ms=round(loop_s * 1e3, 1), loop_measured_removals=done, loop_extrapolated=extrapolated, loop_fit=fit,
            loop_over_batch=round(loop_s * 1e3 / float(np.median(batch_ms)), 1), request_matches=matches, equal=bool(equal))), flush=True)
        assert equal, f"{case}: the batch and the loop databases differ"
        assert matches > 0
        del data
    ctx.close()


if __name__ == "__main__":
    main()
