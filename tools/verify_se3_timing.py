"""The COVINS verification of a query keyframe's candidates (1000 keypoints per keyframe) at 1, 8 and 32 candidates:
  (a) cvb_verify_landmark_candidates_seeded_batch: the whole chain in one call;
  (b) chain_existing_calls: the same work through the existing calls on the same inputs and seeds: cvb_landmark_match_batch (the
      candidates as segments), the RANSAC problems gathered on the host (numpy), cvb_ransac_absolute_pose_seeded_batch, the gate,
      T12 / T21 and the already-masks on the host, cvb_search_by_se3_batch over the candidates that continue, the residual pairs on
      the host and one cvb_optimize_relative_pose per candidate.  The host glue is oracle/verify_se3.py's.
Both are timed alternately in one session: the whole call (host clock around the synchronous calls, median of --reps) and the
device time of their kernels (torch.profiler, a separate run).  Every result of every timed call is checked identical between
(a) and (b).  The fused call is also split into the packing of its arguments (Python) and the C call alone.  Prints the GPU name and power limit read in the same run; --out writes the table as JSON.
  python tools/verify_se3_timing.py [--reps 30] [--out verify_se3_timing.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from covins_b200 import matching as M, optimization as O, placerec as PR   # noqa: E402
from oracle import verify_se3 as ov                                         # noqa: E402

KEYS = ("n_matches", "best_sample", "best_model", "best_count", "iterations", "consumed", "T12", "T21", "n_found", "n_corr", "T12_out", "n_inliers",
        "solve_iterations", "match12", "stage", "removed")


def chain_existing_calls(ctx, query, cands, seeds, **prm):
    """the result dict of placerec.verify_landmark_candidates_seeded (with detail) from the existing calls and host glue"""
    def match(A, skipA, B, skipB, seg, thr, num_best):
        res = M.landmark_match(ctx, A, skipA, B, skipB, seg, thr, num_best)
        oA = np.full(len(B), -1, np.int32); oB = np.full(len(B), -1, np.int32)
        n = np.zeros(len(seg) - 1, np.int32)
        for s, (a, b, _) in enumerate(res):
            oA[seg[s]:seg[s] + len(a)] = a; oB[seg[s]:seg[s] + len(b)] = b; n[s] = len(a)
        return oA, oB, n

    def ransac(prob_ptr, pts, bearings, sigma, cam_off, cam_rot, seeds_, threshold, max_iterations, probability):
        return PR.ransac_absolute_pose_seeded(ctx, prob_ptr, pts, bearings, sigma, cam_off, cam_rot, seeds_, threshold, max_iterations, probability)

    def search(v1, v2s, T12s, T21s, a1s, a2s, th, desc_th_low, num_octaves, scale_factor):
        return PR.search_by_se3_batch(ctx, v1, v2s, np.stack(T12s), np.stack(T21s), np.stack(a1s), a2s, th, desc_th_low, num_octaves, scale_factor)

    def refine(p7, rp, camA, camB, th):
        o = O.optimize_relative_pose(ctx, p7, camA=camA, camB=camB, th_outlier_align=th, **rp)
        return o["T12"], o["removed"].astype(np.uint8), o["n_inliers"], o["iterations"]

    return ov.compose(query, cands, np.asarray(seeds, np.uint64), prm, match, ransac, search, refine)


def _same(a, b):
    return all(np.array_equal(np.ascontiguousarray(a[k]).view(np.uint8), np.ascontiguousarray(np.asarray(b[k], a[k].dtype)).view(np.uint8)) for k in KEYS)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch
    from torch.profiler import profile, ProfilerActivity
    from test_verify_landmark import PRM, scene
    assert torch.cuda.is_available(), "needs a GPU"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    gpu = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)
    print("GPU:", gpu)
    ctx = PR.Context(0)
    rows = []
    for n_cand in (1, 8, 32):
        query, cands, seeds, _ = scene(100 + n_cand, n_cand, pix_noise=0.5)
        fused = lambda: PR.verify_landmark_candidates_seeded(ctx, query, cands, seeds, **PRM)   # noqa: E731
        chain = lambda: chain_existing_calls(ctx, query, cands, seeds, **PRM)                     # noqa: E731
        ref = fused()
        assert _same(ref, chain()), "the fused call and the chain differ"
        for _ in range(3):
            fused(); chain()
        tf, tc, tp, tk, same = [], [], [], [], True
        for _ in range(a.reps):
            t0 = time.perf_counter(); g = fused(); tf.append(time.perf_counter() - t0)
            t0 = time.perf_counter(); h = chain(); tc.append(time.perf_counter() - t0)
            t0 = time.perf_counter(); call, _ = PR.landmark_verify_prepared(ctx, query, cands, seeds, **PRM); tp.append(time.perf_counter() - t0)
            t0 = time.perf_counter(); k = call(); tk.append(time.perf_counter() - t0)   # the C call alone, arguments packed
            same &= _same(g, ref) and _same(h, ref) and _same(k, ref)
        dev = []
        for fn in (fused, chain):
            with profile(activities=[ProfilerActivity.CUDA]) as pr:
                for _ in range(5):
                    fn()
                torch.cuda.synchronize()
            ev = [e for e in pr.events() if e.device_type.name == "CUDA" and "Memcpy" not in e.name and "Memset" not in e.name]
            dev.append(sum(e.device_time for e in ev) / 5 / 1e3)
        row = dict(n_cand=n_cand, fused_ms=float(np.median(tf)) * 1e3, chain_ms=float(np.median(tc)) * 1e3,
                   fused_pack_ms=float(np.median(tp)) * 1e3, fused_c_call_ms=float(np.median(tk)) * 1e3,
                   fused_ms_range=[float(np.min(tf)) * 1e3, float(np.max(tf)) * 1e3], chain_ms_range=[float(np.min(tc)) * 1e3, float(np.max(tc)) * 1e3],
                   fused_kernels_ms=dev[0],
                   chain_kernels_ms=dev[1], identical=bool(same), n_matches=int(ref["n_matches"].sum()), n_corr=int(ref["n_corr"].sum()))
        rows.append(row)
        print(json.dumps(row), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(dict(gpu=gpu, rows=rows), fh, indent=1)
    assert all(r["identical"] for r in rows)


if __name__ == "__main__":
    main()
