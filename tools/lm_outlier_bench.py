#!/usr/bin/env python
"""Times cvb_landmark_outliers (the landmark outlier removal of Map::Clean in one call) on the synthetic maps of BASELINE
configs C3 (2 000 keyframes / 100 k landmarks) and C5 (10 k keyframes / 1 M landmarks), both with their 5 % gross outliers,
at the default rule (th_outlier 0.92, Cauchy 1, min_obs 2, no norms requested).

Per config one JSON line with
  * the card's name and power limit, read in the same run;
  * K, L, n_obs, the outlier observations (by flag) and the erased landmarks;
  * end-to-end host time of one call (host validation, copies both ways; median and spread over --calls calls after
    --warmup);
  * device time per call: the summed durations of the call's kernels and copies from a torch.profiler (CUPTI) trace of
    --profile-calls further calls, taken in a pass of its own so that tracing does not slow the end-to-end figure, and the
    two kernels' share;
  * the bytes the kernels must move, computed from the shapes (per observation obs_kf, obs_uv, obs_sigma and the flag; per
    landmark lm_obs_ptr, the position, the good-observation count and the flag; per keyframe its pose and camera), and the
    rate that gives over the kernels' time against the H100 SXM data-sheet 3.35 TB/s;
  * the CPU column: oracle/lm_outliers.py (the torch FP64 residual and the numpy rule) on this host's cores, the median of
    --oracle-calls, with the core count;
  * whether the call equals the oracle (flags exactly except where the oracle's norm lies within 1e-5 of th_outlier, and
    erasures exactly; the script fails otherwise).
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


def kernel_bytes(K, L, n_obs):
    per_obs = 4 + 8 + 8 + 1               # obs_kf, obs_uv (2 x f32), obs_sigma, obs_outlier
    per_lm = 4 + 24 + 4 + 4 + 1           # lm_obs_ptr, lm, good (atomic, read by the landmark pass), lm_erase
    per_kf = 7 * 8 + 7 * 8 + 4 * 8 + 4 * 8 + 8 + 4   # pose, extr, intr, dist, xi, model
    return n_obs * per_obs + L * per_lm + K * per_kf


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--configs", default="C3,C5")
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile-calls", type=int, default=3)
    ap.add_argument("--oracle-calls", type=int, default=1)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("lm_outlier_bench: no CUDA device (there is no CPU fallback)")
    import covins_b200
    from covins_b200 import mapgraph, synth_map
    from oracle import lm_outliers as ora
    card = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], text=True).strip()
    ctx = covins_b200.Context(0)
    for name in a.configs.split(","):
        p = synth_map.make_config(name)
        K, L, n_obs = int(p["K"]), int(p["L"]), len(p["obs_kf"])
        call = lambda: mapgraph.landmark_outliers(ctx, p)
        for _ in range(a.warmup):
            out, erase, _ = call()
        host = []
        for _ in range(a.calls):
            t0 = time.perf_counter()
            call()
            host.append((time.perf_counter() - t0) * 1e3)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.profile_calls):
                call()
        ev = prof.key_averages()
        dev_us = sum(e.device_time_total for e in ev)
        kern_us = sum(e.device_time_total for e in ev if "lo_obs_kernel" in e.key or "lo_lm_kernel" in e.key)
        top = {e.key[:60]: round(e.device_time_total / a.profile_calls / 1e3, 4) for e in sorted(ev, key=lambda e: -e.device_time_total)[:6]}
        kern_s = kern_us / a.profile_calls / 1e6
        nbytes = kernel_bytes(K, L, n_obs)
        ora_ms = []
        for _ in range(a.oracle_calls):
            t0 = time.perf_counter()
            r_out, r_erase, r_norm = ora.landmark_outliers(p)
            ora_ms.append((time.perf_counter() - t0) * 1e3)
        _, _, norms = mapgraph.landmark_outliers(ctx, p, want_norms=True)
        near = (r_norm >= 0) & (np.abs(r_norm - 0.92) <= 1e-5 * 0.92)
        equal = bool(np.array_equal(out[~near], r_out[~near]) and (near.any() or np.array_equal(erase, r_erase))
                     and np.allclose(norms[r_norm >= 0], r_norm[r_norm >= 0], rtol=1e-5, atol=1e-5))
        print(json.dumps(dict(
            config=name, card=card, K=K, L=L, n_obs=n_obs, outliers=int((out == 1).sum()), not_projectable=int((out == 2).sum()),
            erased=int(erase.sum()), calls=a.calls,
            host_ms_median=round(float(np.median(host)), 3), host_ms_min=round(min(host), 3), host_ms_max=round(max(host), 3),
            device_ms_per_call=round(dev_us / a.profile_calls / 1e3, 3), kernels_ms_per_call=round(kern_s * 1e3, 4), device_ms_top=top,
            kernel_bytes=nbytes, kernel_GBps=round(nbytes / kern_s / 1e9, 1) if kern_s > 0 else None,
            kernel_share_of_3_35TBps=round(nbytes / kern_s / HBM_BYTES_PER_S, 3) if kern_s > 0 else None,
            oracle_ms=round(float(np.median(ora_ms)), 1), oracle_cores=os.cpu_count(), near_threshold=int(near.sum()),
            equal_to_oracle=equal)), flush=True)
        assert equal, f"{name}: the call differs from the oracle"
    ctx.close()


if __name__ == "__main__":
    main()
