"""Absolute-pose RANSAC at a COVINS-mode size: n_prob candidates, 1000 correspondences each, 300 iterations plus headroom for
skipped samples.  Compares
  (a) cvb_ransac_absolute_pose_batch: one call for the batch (host clock around the synchronous call, and the kernel's device
      time from torch.profiler's CUDA activity);
  (b) the two-step path: hypotheses on the host (oracle P3P, the first max_iterations samples of every problem), one
      cvb_score_absolute_pose_batch call per problem, placerec.ransac_select — timed end to end;
  (c) the oracle RANSAC on the host cores (OpenMP over problems).
Every result of (a) is checked against (c).  Prints the GPU name and power limit with the numbers.
With --relative, the non-central relative-pose (17-point) RANSAC instead, at 5 % and 30 % outliers, 3-camera rigs per side:
  (a) cvb_ransac_noncentral_relative_pose_batch (whole call, and kernel time from torch.profiler);
  (b) host 17-point solves with the oracle (the first max_iterations samples of every problem, one thread), plus the oracle's
      selection over them (host scoring per camera pair, placerec.ransac_select);
  (c) the oracle RANSAC on the host cores.
With --central, the central relative-pose (5-point) RANSAC, n_prob 1, 6 and 60 (one and ten candidates x six pairings), 300 and
1000 correspondences, 5 % and 30 % outliers:
  (a) cvb_ransac_central_relative_pose_batch (whole call, and kernel time from torch.profiler);
  (c) the oracle RANSAC on the host cores.
  python tools/ransac_timing.py [--reps 100] [--outlier 0.5] [--relative | --central]"""
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
    ap.add_argument("--relative", action="store_true", help="time the non-central relative-pose (17-point) RANSAC")
    ap.add_argument("--central", action="store_true", help="time the central relative-pose (5-point) RANSAC")
    a = ap.parse_args()
    if a.relative:
        return relative(a)
    if a.central:
        return central(a)
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


def relative(a):
    import torch
    import covins_b200
    from covins_b200 import placerec as PR
    from oracle import ransac_rel as orel
    from test_ransac_relative import _batch
    from torch.profiler import profile, ProfilerActivity
    assert torch.cuda.is_available(), "needs a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print(f"GPU: {torch.cuda.get_device_name(0)} | {q.stdout.strip()} | host cores: {os.cpu_count()}")
    ctx = covins_b200.Context(0)
    thr, max_it, prob = 9.0, 300, 0.99
    kw = dict(threshold=thr, max_iterations=max_it, probability=prob)
    for outlier in (0.05, 0.3):
        for n_prob in (1, 8, 32):
            b, _ = _batch(200 + n_prob, [(a.n, 3, 3, False)] * n_prob, a.samples, outlier_frac=outlier, repeat_frac=0.0)
            ref = orel.ransac_noncentral_relative_pose(**b, **kw)
            got = PR.ransac_noncentral_relative_pose(ctx, **b, **kw)
            for k in ref:
                assert np.array_equal(ref[k], got[k]), k
            for _ in range(3):
                PR.ransac_noncentral_relative_pose(ctx, **b, **kw)
            reps = max(3, a.reps // (10 if outlier > 0.1 else 1))
            t0 = time.perf_counter()
            for _ in range(reps):
                PR.ransac_noncentral_relative_pose(ctx, **b, **kw)
            t_a = (time.perf_counter() - t0) / reps * 1e3
            with profile(activities=[ProfilerActivity.CUDA]) as pr:
                for _ in range(5):
                    PR.ransac_noncentral_relative_pose(ctx, **b, **kw)
            ev = [e for e in pr.events() if "ransac_rel_kernel" in e.name]
            k_a = np.mean([e.device_time for e in ev]) / 1e3 if ev else float("nan")
            ptr, cp1, cp2 = b["prob_ptr"], b["cam_ptr1"], b["cam_ptr2"]

            def host_path():
                out = []
                for i in range(n_prob):
                    s = slice(ptr[i], ptr[i + 1])
                    rig = (b["cam1"][s], b["cam2"][s], b["cam_off1"][cp1[i]:cp1[i + 1]], b["cam_rot1"][cp1[i]:cp1[i + 1]],
                           b["cam_off2"][cp2[i]:cp2[i + 1]], b["cam_rot2"][cp2[i]:cp2[i + 1]])
                    models, valid = orel.rel_hypotheses(b["f1"][s], b["f2"][s], *rig, b["samples"][i][:max_it])
                    _, _, cnt = orel.score_noncentral_relative_pose(models[valid > 0], b["f1"][s], b["f2"][s], b["sigma1"][s], b["sigma2"][s],
                                                                   *rig, thr)
                    out.append(PR.ransac_select(cnt, ptr[i + 1] - ptr[i], 17, max_it, prob))
                return out
            host_path()
            reps_b = 3
            t0 = time.perf_counter()
            for _ in range(reps_b):
                host_path()
            t_b = (time.perf_counter() - t0) / reps_b * 1e3
            t0 = time.perf_counter()
            for _ in range(reps_b):
                orel.ransac_noncentral_relative_pose(**b, **kw)
            t_c = (time.perf_counter() - t0) / reps_b * 1e3
            print(f"relative | outliers {outlier:.0%} | n_prob {n_prob:2d} x {a.n} corr, {a.samples} samples: iterations used "
                  f"{got['iterations'].min()}-{got['iterations'].max()} | (a) call {t_a:.3f} ms, kernel {k_a:.3f} ms | (b) host 17-pt solves + "
                  f"selection {t_b:.3f} ms | (c) oracle RANSAC on {os.cpu_count()} host cores {t_c:.3f} ms")
    ctx.close()


def central(a):
    import torch
    import covins_b200
    from covins_b200 import placerec as PR
    from oracle import ransac_rel5 as orel
    from test_ransac_central import _batch
    from torch.profiler import profile, ProfilerActivity
    assert torch.cuda.is_available(), "needs a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print(f"GPU: {torch.cuda.get_device_name(0)} | {q.stdout.strip()} | host cores: {os.cpu_count()}")
    ctx = covins_b200.Context(0)
    thr, max_it, prob = 9.0, 300, 0.99
    kw = dict(threshold=thr, max_iterations=max_it, probability=prob)
    for n in (300, 1000):
        for outlier in (0.05, 0.3):
            for n_prob in (1, 6, 60):
                b, _ = _batch(300 + n_prob, [(n, outlier, False)] * n_prob, a.samples, repeat_frac=0.0)
                ref = orel.ransac_central_relative_pose(**b, **kw)
                got = PR.ransac_central_relative_pose(ctx, **b, **kw)
                for k in ref:
                    assert np.array_equal(ref[k], got[k]), k
                for _ in range(3):
                    PR.ransac_central_relative_pose(ctx, **b, **kw)
                reps = max(3, a.reps // 10)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(reps):
                    PR.ransac_central_relative_pose(ctx, **b, **kw)
                t_a = (time.perf_counter() - t0) / reps * 1e3
                with profile(activities=[ProfilerActivity.CUDA]) as pr:
                    for _ in range(5):
                        PR.ransac_central_relative_pose(ctx, **b, **kw)
                ev = [e for e in pr.events() if "ransac_rel_kernel" in e.name]
                k_a = np.mean([e.device_time for e in ev]) / 1e3 if ev else float("nan")
                t0 = time.perf_counter()
                for _ in range(3):
                    orel.ransac_central_relative_pose(**b, **kw)
                t_c = (time.perf_counter() - t0) / 3 * 1e3
                print(f"central | {n} corr | outliers {outlier:.0%} | n_prob {n_prob:2d}, {a.samples} samples: iterations used "
                      f"{got['iterations'].min()}-{got['iterations'].max()} | (a) call {t_a:.3f} ms, kernel {k_a:.3f} ms | "
                      f"(c) oracle RANSAC on {os.cpu_count()} host cores {t_c:.3f} ms | bit-identical to the oracle")
    ctx.close()


if __name__ == "__main__":
    main()
