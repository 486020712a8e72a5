"""Absolute-pose RANSAC at a COVINS-mode size: n_prob candidates, 1000 correspondences each, 300 iterations plus headroom for
skipped samples.  Compares
  (a) cvb_ransac_absolute_pose_batch: one call for the batch (host clock around the synchronous call, and the kernel's device
      time from torch.profiler's CUDA activity);
  (b) the two-step path: hypotheses on the host (oracle P3P, the first max_iterations samples of every problem), one
      cvb_score_absolute_pose_batch call per problem, placerec.ransac_select — timed end to end;
  (c) the oracle RANSAC on the host cores (OpenMP over problems).
Every result of (a) is checked against (c).  Prints the GPU name and power limit with the numbers.
  python tools/ransac_timing.py [--reps 100] [--outlier 0.5]"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=100)
    ap.add_argument("--outlier", type=float, default=0.5)
    ap.add_argument("--n", type=int, default=1000)
    ap.add_argument("--samples", type=int, default=400)
    a = ap.parse_args()
    import torch
    import covins_b200
    from covins_b200 import placerec as PR
    from oracle import ransac as orr
    from test_ransac_absolute import _batch
    assert torch.cuda.is_available(), "needs a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print(f"GPU: {torch.cuda.get_device_name(0)} | {q.stdout.strip()} | host cores: {os.cpu_count()}")
    ctx = covins_b200.Context(0)
    thr, max_it, prob = 25.0, 300, 0.99
    for n_prob in (1, 8, 32):
        b, _ = _batch(100 + n_prob, [a.n] * n_prob, a.samples, outlier_frac=a.outlier)
        ref = orr.ransac_absolute_pose(**b, threshold=thr, max_iterations=max_it, probability=prob)
        got = PR.ransac_absolute_pose(ctx, **b, threshold=thr, max_iterations=max_it, probability=prob)
        for k in ref:
            assert np.array_equal(ref[k], got[k]), k
        for _ in range(10):
            PR.ransac_absolute_pose(ctx, **b, threshold=thr, max_iterations=max_it, probability=prob)
        t0 = time.perf_counter()
        for _ in range(a.reps):
            PR.ransac_absolute_pose(ctx, **b, threshold=thr, max_iterations=max_it, probability=prob)
        t_a = (time.perf_counter() - t0) / a.reps * 1e3
        from torch.profiler import profile, ProfilerActivity
        with profile(activities=[ProfilerActivity.CUDA]) as pr:
            for _ in range(20):
                PR.ransac_absolute_pose(ctx, **b, threshold=thr, max_iterations=max_it, probability=prob)
        ev = [e for e in pr.events() if "ransac_abs_kernel" in e.name]
        k_a = np.mean([e.device_time for e in ev]) / 1e3 if ev else float("nan")
        ptr = b["prob_ptr"]

        def two_step():
            out = []
            for i in range(n_prob):
                s = slice(ptr[i], ptr[i + 1])
                models, valid = orr.abs_hypotheses(b["pts"][s], b["bearings"][s], b["cam_off"][i], b["cam_rot"][i], b["samples"][i][:max_it])
                _, _, cnt = PR.score_absolute_pose(ctx, models[valid > 0], b["pts"][s], b["bearings"][s], b["sigma"][s], b["cam_off"][i], b["cam_rot"][i],
                                                   thr, want_scores=False, want_inliers=False)
                out.append(PR.ransac_select(cnt, ptr[i + 1] - ptr[i], 4, max_it, prob))
            return out
        two_step()
        reps_b = max(5, a.reps // 10)
        t0 = time.perf_counter()
        for _ in range(reps_b):
            two_step()
        t_b = (time.perf_counter() - t0) / reps_b * 1e3
        t0 = time.perf_counter()
        for _ in range(reps_b):
            orr.ransac_absolute_pose(**b, threshold=thr, max_iterations=max_it, probability=prob)
        t_c = (time.perf_counter() - t0) / reps_b * 1e3
        print(f"n_prob {n_prob:2d} x {a.n} corr, {a.samples} samples, outliers {a.outlier:.0%}: iterations used {got['iterations'].min()}-"
              f"{got['iterations'].max()} | (a) call {t_a:.3f} ms, kernel {k_a:.3f} ms | (b) host P3P + scoring + select {t_b:.3f} ms | "
              f"(c) oracle RANSAC on {os.cpu_count()} host cores {t_c:.3f} ms")
    ctx.close()


if __name__ == "__main__":
    main()
