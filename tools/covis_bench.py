#!/usr/bin/env python
"""Times cvb_covisibility (the covisibility graph of a whole map in one call) on the synthetic maps of BASELINE configs
C3 (2 000 keyframes / 100 k landmarks) and C5 (10 k keyframes / 1 M landmarks), beside a CPU arm: the scipy.sparse product
A @ A.T of the keyframe x landmark matrix, row blocks on all host cores (the product only, without rules 3-4).

Per config one JSON line with
  * the card's name and power limit, read in the same run;
  * counted from shapes: observations, shared-landmark pairs, distinct keyframe pairs, directed edges in the result, and
    the bytes the pair list needs to move (8 B per pair written by the expansion, read and written once per 8-bit radix
    pass over the 2*ceil(log2 K) key bits, read once by the run-length encode);
  * end-to-end host time of one call (host validation, copies both ways, every kernel; median and spread over --calls
    calls after --warmup);
  * device time per call: the summed durations of the call's kernels and copies from a torch.profiler (CUPTI) trace of
    --calls further calls, taken in a pass of its own so that tracing does not slow the end-to-end figure.
There is no fallback: without a CUDA device the script fails.
"""
import argparse
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ProcessPoolExecutor

import numpy as np
import scipy.sparse as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

_A = None


def _block_product(rows):
    return (_A[rows[0]:rows[1]] @ _A.T).nnz


def cpu_arm(p, workers):
    """A @ A.T in row blocks over `workers` processes → (seconds, distinct keyframe pairs)"""
    global _A
    lm = np.repeat(np.arange(p["L"]), np.diff(p["lm_obs_ptr"]))
    _A = sp.csr_matrix((np.ones(len(lm), np.int32), (p["obs_kf"], lm)), shape=(p["K"], p["L"]))
    cuts = np.linspace(0, p["K"], 4 * workers + 1).astype(int)
    t0 = time.perf_counter()
    with ProcessPoolExecutor(workers) as ex:     # fork: the workers share _A
        nnz = sum(ex.map(_block_product, zip(cuts[:-1], cuts[1:])))
    dt = time.perf_counter() - t0
    has_obs = int((np.bincount(p["obs_kf"], minlength=p["K"]) > 0).sum())
    return dt, (nnz - has_obs) // 2


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--configs", default="C3,C5")
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--min-weight", type=int, default=15)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("covis_bench: no CUDA device (there is no CPU fallback)")
    import covins_b200
    from covins_b200 import mapgraph, synth_map
    card = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], text=True).strip()
    ctx = covins_b200.Context(0)
    workers = os.cpu_count() or 1
    for name in a.configs.split(","):
        p = synth_map.make_config(name)
        K, L = p["K"], p["L"]
        call = lambda: mapgraph.covisibility(ctx, p["lm_obs_ptr"], p["obs_kf"], K, min_weight=a.min_weight)
        for _ in range(a.warmup):
            nbr_ptr, nbr_kf, nbr_w = call()
        host = []
        for _ in range(a.calls):
            t0 = time.perf_counter()
            call()
            host.append((time.perf_counter() - t0) * 1e3)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.calls):
                call()
        dev_us = sum(e.device_time_total for e in prof.key_averages())
        kernels = {e.key[:60]: round(e.device_time_total / a.calls / 1e3, 4) for e in sorted(prof.key_averages(), key=lambda e: -e.device_time_total)[:8]}
        n = np.diff(p["lm_obs_ptr"]).astype(np.int64)
        pairs = int((n * (n - 1) // 2).sum())
        passes = -(-2 * max(1, int(K - 1).bit_length()) // 8)
        cpu_s, kf_pairs = cpu_arm(p, workers)
        print(json.dumps(dict(
            config=name, card=card, K=K, L=L, n_obs=int(len(p["obs_kf"])), min_weight=a.min_weight, pairs=pairs, keyframe_pairs=kf_pairs,
            directed_edges=int(len(nbr_kf)), pair_list_bytes=pairs * 8 * (2 + 2 * passes), calls=a.calls,
            host_ms_median=round(float(np.median(host)), 3), host_ms_min=round(min(host), 3), host_ms_max=round(max(host), 3),
            device_ms_per_call=round(dev_us / a.calls / 1e3, 3), device_ms_top=kernels,
            cpu_spgemm_ms=round(cpu_s * 1e3, 1), cpu_workers=workers)), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
