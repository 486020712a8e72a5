"""Helpers shared by the RANSAC and covariance tests: random rotations, the expected sequential selection, the bitwise
GPU-vs-oracle comparison and the build of a C++ wrapper test."""
import os
import subprocess

import numpy as np

from covins_b200 import placerec as PR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rand_rot(rng):
    q = rng.normal(size=4); q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _expected_selection(valid, count, n, sample_size, max_iterations, probability):
    """placerec.ransac_select over the valid samples in order (opengv's skipped_count: at most 10 * max_iterations invalid ones)"""
    idx, skipped, stop = [], 0, len(valid)
    for s in range(len(valid)):
        if skipped >= 10 * max_iterations:
            stop = s
            break
        if valid[s]:
            idx.append(s)
        else:
            skipped += 1
    best, it = PR.ransac_select(np.asarray(count)[idx], n, sample_size, max_iterations, probability)
    consumed = (idx[it - 1] + 1 if it > 0 else 0) if it < len(idx) else stop
    return (idx[best] if best >= 0 else -1), it, consumed


def _check_selection(b, r, sample_size, max_iterations, probability):
    ptr = b["prob_ptr"]
    for i in range(len(ptr) - 1):
        n = ptr[i + 1] - ptr[i]
        best, it, consumed = _expected_selection(r["sample_valid"][i], r["sample_count"][i], n, sample_size, max_iterations, probability)
        assert (r["best_sample"][i], r["iterations"][i], r["consumed"][i]) == (best, it, consumed), i
        if best >= 0:
            assert r["best_count"][i] == r["sample_count"][i][best] and np.array_equal(r["best_model"][i], r["sample_model"][i][best])
        else:
            assert r["best_count"][i] == 0 and not r["best_model"][i].any() and not r["inlier_mask"][ptr[i]:ptr[i + 1]].any()


def _gpu_vs_oracle(ctx, gpu, oracle, b, thr, max_it, prob):
    """the GPU call gpu (a placerec.ransac_* function) against its oracle, every output with the per-sample ones, byte for byte"""
    g = gpu(ctx, **b, threshold=thr, max_iterations=max_it, probability=prob, per_sample=True)
    r = oracle(**b, threshold=thr, max_iterations=max_it, probability=prob, per_sample=True)
    for k in r:
        assert np.array_equal(g[k].view(np.uint8), r[k].view(np.uint8)), k
    return g


def _build_shim(source, out):
    """compiles tests/cpp/<source> against the library with -Wall -Werror"""
    import covins_b200
    if not os.path.exists(covins_b200.LIB_PATH):
        covins_b200.build()
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-o", out, os.path.join(ROOT, "tests", "cpp", source),
                           "-L" + os.path.join(ROOT, "covins_b200"), "-lcovins_b200", "-Wl,-rpath," + os.path.join(ROOT, "covins_b200")])
