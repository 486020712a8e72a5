#!/usr/bin/env python
"""Times cvb_redundant_keyframes (the redundancy-culling pass of Map::Clean in one call) on the synthetic maps of BASELINE
configs C3 (2 000 keyframes / 100 k landmarks) and C5 (10 k keyframes / 1 M landmarks), beside the CPU arm: the
sequential pass of oracle/prune_oracle.c on one thread, as the reference runs it under the map lock.

The maps' keyframe chains are the agents' trajectories (10 Hz timestamps); each agent's first keyframe and the loop
constraints' keyframes are protected; octave = obs_sigma / 2 - 1.  Per config one JSON line with
  * the card's name and power limit, read in the same run;
  * K, L, n_obs, the number culled and the number of rounds;
  * end-to-end host time of one call (host validation, copies both ways, every round; median and spread over --calls
    calls after --warmup);
  * device time per call: the summed durations of the call's kernels and copies from a torch.profiler (CUPTI) trace of
    --profile-calls further calls, taken in a pass of its own so that tracing does not slow the end-to-end figure;
  * the C oracle's single-thread time (median of --oracle-calls) and whether its set equals the call's.
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


def problem(p, th_red, max_time_dist):
    K = p["K"]
    prot = (p["kf_id"] == 0).astype(np.uint8)
    prot[p["loop_i"]] = 1; prot[p["loop_j"]] = 1
    return dict(lm_obs_ptr=p["lm_obs_ptr"], obs_kf=p["obs_kf"], obs_octave=(p["obs_sigma"] / 2 - 1).astype(np.int32),
                kf_pred=np.where(p["kf_id"] > 0, np.arange(K) - 1, -1).astype(np.int32), kf_time=p["kf_id"] / 10.0, kf_protect=prot,
                th_red=th_red, max_time_dist=max_time_dist, th_obs=3)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--configs", default="C3,C5")
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile-calls", type=int, default=3)
    ap.add_argument("--oracle-calls", type=int, default=3)
    ap.add_argument("--th-red", type=float, default=0.75)
    ap.add_argument("--max-time-dist", type=float, default=1.0)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("prune_bench: no CUDA device (there is no CPU fallback)")
    import covins_b200
    from covins_b200 import mapgraph, synth_map
    from oracle import prune as ora
    card = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], text=True).strip()
    ctx = covins_b200.Context(0)
    for name in a.configs.split(","):
        p = synth_map.make_config(name)
        c = problem(p, a.th_red, a.max_time_dist)
        call = lambda: mapgraph.redundant_keyframes(ctx, **c)
        for _ in range(a.warmup):
            culled, rounds = call()
        host = []
        for _ in range(a.calls):
            t0 = time.perf_counter()
            call()
            host.append((time.perf_counter() - t0) * 1e3)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.profile_calls):
                call()
        dev_us = sum(e.device_time_total for e in prof.key_averages())
        top = {e.key[:60]: round(e.device_time_total / a.profile_calls / 1e3, 4)
               for e in sorted(prof.key_averages(), key=lambda e: -e.device_time_total)[:6]}
        ora_ms = []
        for _ in range(a.oracle_calls):
            t0 = time.perf_counter()
            ref = ora.redundant_keyframes(**c)
            ora_ms.append((time.perf_counter() - t0) * 1e3)
        print(json.dumps(dict(
            config=name, card=card, K=p["K"], L=p["L"], n_obs=int(len(p["obs_kf"])), th_red=a.th_red, max_time_dist=a.max_time_dist, th_obs=3,
            culled=int(culled.sum()), rounds=rounds, calls=a.calls,
            host_ms_median=round(float(np.median(host)), 3), host_ms_min=round(min(host), 3), host_ms_max=round(max(host), 3),
            device_ms_per_call=round(dev_us / a.profile_calls / 1e3, 3), device_ms_top=top,
            host_ms_per_round=round(float(np.median(host)) / max(rounds, 1), 4),
            oracle_1thread_ms=round(float(np.median(ora_ms)), 1), equal_to_oracle=bool(np.array_equal(culled, ref)))), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
