#!/usr/bin/env python
"""Times the merge of two agents' maps (Map(map_target, map_tofuse, T), map_be.cpp:334-381) at the sizes of BASELINE
configs C3 (2 000 keyframes / 100 k landmarks) and C5 (10 k keyframes / 1 M landmarks).

One JSON line per measurement, each with the card's name, power limit and SM clock read in the same run:
  * "k16": cvb_map_rigid_transform on random rigid poses, velocities and positions of the config's size (the transform
    does not depend on the map's structure): end-to-end host time of one call (median, min and max of --calls after
    --warmup; the pageable copies both ways included), the kernel's time from a torch.profiler (CUPTI) pass of its own, the
    bytes it must move (pose, velocity and position read and written once) and their rate against the H100 SXM data-sheet
    3.35 TB/s.  The output is checked bitwise against oracle/merge.py;
  * "db_merge": for ORB (1 000 rows per keyframe) and SIFT (300 rows per keyframe), a target database and a fused one of
    the config's keyframe count each; the time of cvb_db_merge against the path it replaces, appending the fused map's rows
    to the target from the host (pageable numpy rows; for SIFT, float32 rows checked and quantised on the host).  Each
    repetition starts from a freshly built target.  The merged database is checked against the host-appended one on one
    request;
  * "shim_e2e" (C3 only): what covins_b200::MergeMaps does, through Python, on the C3 synthetic map: poses to 4x4
    matrices, cvb_map_rigid_transform, cvb_db_merge of ORB databases as above, and the merged map's covisibility graph.
Not measured: C5 end to end (building the C5 map's observation structure takes minutes of numpy), the C++ shim's own
container walk, and the host containers' union, which the library does not do.
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

HBM_BYTES_PER_S = 3.35e12
SIZES = {"C3": (2000, 100_000), "C5": (10_008, 1_000_000)}
ROWS = {"orb": 1000, "sift": 300}


def rigid(rng, t=10.0):
    q, r = np.linalg.qr(rng.normal(size=(3, 3)))
    q = q * np.sign(np.diag(r))
    T = np.eye(4)
    T[:3, :3] = q if np.linalg.det(q) > 0 else -q
    T[:3, 3] = rng.normal(size=3) * t
    return T


def timed(fn, calls, warmup):
    import torch
    for _ in range(warmup):
        fn()
    ms = []
    for _ in range(calls):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ms.append((time.perf_counter() - t0) * 1e3)
    return dict(ms_median=round(float(np.median(ms)), 3), ms_min=round(min(ms), 3), ms_max=round(max(ms), 3), calls=calls)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--configs", default="C3,C5")
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--db-calls", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile-calls", type=int, default=5)
    ap.add_argument("--no-e2e", action="store_true")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("merge_bench: no CUDA device (there is no CPU fallback)")
    import covins_b200
    from covins_b200 import mapgraph
    from covins_b200 import matching as M
    from oracle import merge as ora
    card = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader", "-i", "0"],
                                   text=True).strip()
    ctx = covins_b200.Context(0)
    rng = np.random.default_rng(0)
    for name in a.configs.split(","):
        K, L = SIZES[name]
        # ---- K16
        T = rigid(rng, 1e3)
        ws = np.stack([rigid(rng) for _ in range(K)])
        vel, lm = rng.normal(size=(K, 3)), rng.normal(size=(L, 3)) * 50
        call = lambda: mapgraph.rigid_transform(ctx, T, ws, vel, lm)
        host = timed(call, a.calls, a.warmup)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.profile_calls):
                call()
        ev = prof.key_averages()
        kern_s = sum(e.device_time_total for e in ev if "rigid_transform_kernel" in e.key) / a.profile_calls / 1e6
        copy_ms = sum(e.device_time_total for e in ev if "Memcpy" in e.key) / a.profile_calls / 1e3
        nbytes = 2 * (128 * K + 24 * K + 24 * L)
        got, ref = call(), ora.rigid_transform(T, ws, vel, lm)
        equal = all(np.array_equal(x.view(np.uint64), y.view(np.uint64)) for x, y in zip(got, ref))
        print(json.dumps(dict(what="k16", config=name, card=card, K=K, L=L, **host, kernel_ms=round(kern_s * 1e3, 4),
                              copies_ms=round(copy_ms, 3), kernel_bytes=nbytes,
                              kernel_GBps=round(nbytes / kern_s / 1e9, 1) if kern_s > 0 else None,
                              kernel_share_of_3_35TBps=round(nbytes / kern_s / HBM_BYTES_PER_S, 3) if kern_s > 0 else None,
                              equal_to_oracle=equal)), flush=True)
        assert equal, f"{name}: K16 differs from the oracle"
        del ws, vel, lm, got, ref
        # ---- cvb_db_merge against the host re-append
        for kind in ("orb", "sift"):
            rows = ROWS[kind]
            dim = 32 if kind == "orb" else 128
            dt = np.uint8 if kind == "orb" else np.float32
            tgt = rng.integers(0, 256, size=(K * rows, dim), dtype=np.uint8).astype(dt)
            fus = rng.integers(0, 256, size=(K * rows, dim), dtype=np.uint8).astype(dt)
            rpk = np.full(K, rows, np.int32)
            src = M.DescriptorDatabase(ctx, kind=kind)
            src.append(fus, rpk)
            merge_ms, append_ms = [], []
            for rep in range(a.db_calls + 1):        # the first repetition is a warm-up
                for path in ("merge", "append"):
                    dst = M.DescriptorDatabase(ctx, kind=kind)
                    dst.append(tgt, rpk)
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    if path == "merge":
                        dst.merge(src)
                    else:
                        dst.append(fus, rpk)
                    torch.cuda.synchronize()
                    if rep:
                        (merge_ms if path == "merge" else append_ms).append((time.perf_counter() - t0) * 1e3)
                    if rep == a.db_calls:
                        res = getattr(dst, "match_hamming" if kind == "orb" else "match_l2")(tgt[:500])
                        if path == "merge":
                            merged = res
                        else:
                            same = all(np.array_equal(np.asarray(x).view(np.int32), np.asarray(y).view(np.int32)) for x, y in zip(merged, res))
                    dst.close()
            src.close()
            print(json.dumps(dict(what="db_merge", config=name, card=card, kind=kind, n_kf_each=K, rows_per_kf=rows,
                                  fused_row_bytes=int(K * rows * dim), merge_ms_median=round(float(np.median(merge_ms)), 3),
                                  merge_ms_min=round(min(merge_ms), 3), reappend_ms_median=round(float(np.median(append_ms)), 3),
                                  reappend_ms_min=round(min(append_ms), 3), calls=a.db_calls, equal_to_reappend=bool(same))), flush=True)
            assert same, f"{name} {kind}: the merged database differs from the re-appended one"
            del tgt, fus
        # ---- the shim's steps through Python
        if name == "C3" and not a.no_e2e:
            from covins_b200 import synth_map
            p = synth_map.make_config("C3")
            Kc = int(p["K"])
            desc = rng.integers(0, 256, size=(Kc * ROWS["orb"], 32), dtype=np.uint8)
            rpk = np.full(Kc // 2, ROWS["orb"], np.int32)
            db_f = M.DescriptorDatabase(ctx)
            db_f.append(desc[len(rpk) * ROWS["orb"]:2 * len(rpk) * ROWS["orb"]], rpk)
            vel = rng.normal(size=(Kc, 3))
            steps, total = {}, []
            for rep in range(a.warmup + a.calls):
                db_t = M.DescriptorDatabase(ctx)          # a fresh target each time, built outside the timed window
                db_t.append(desc[:len(rpk) * ROWS["orb"]], rpk)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                ws = np.zeros((Kc, 4, 4))
                ws[:, :3, :3] = synth_map.quat_to_rot(np.asarray(p["pose"])[:, :4])
                ws[:, :3, 3] = np.asarray(p["pose"])[:, 4:]
                ws[:, 3, 3] = 1.0
                t1 = time.perf_counter()
                mapgraph.rigid_transform(ctx, T, ws, vel, p["lm"])
                t2 = time.perf_counter()
                db_t.merge(db_f)
                torch.cuda.synchronize()
                t3 = time.perf_counter()
                mapgraph.covisibility(ctx, p["lm_obs_ptr"], p["obs_kf"], Kc)
                t4 = time.perf_counter()
                db_t.close()
                if rep >= a.warmup:
                    total.append((t4 - t0) * 1e3)
                    for k, v in (("flatten", t1 - t0), ("k16", t2 - t1), ("db_merge", t3 - t2), ("covisibility", t4 - t3)):
                        steps.setdefault(k, []).append(v * 1e3)
            print(json.dumps(dict(what="shim_e2e", config="C3", card=card, K=Kc, L=int(p["L"]), n_obs=len(p["obs_kf"]),
                                  ms_median=round(float(np.median(total)), 3), ms_min=round(min(total), 3), ms_max=round(max(total), 3),
                                  calls=a.calls, steps_ms_median={k: round(float(np.median(v)), 3) for k, v in steps.items()})), flush=True)
            db_f.close()
    ctx.close()


if __name__ == "__main__":
    main()
