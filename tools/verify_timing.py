"""The COVINS_G verification of a query keyframe's candidates (6 pairings each, 1000 keypoints per keyframe, 3-camera rigs, 300
covariance samples) at 1, 8 and 32 candidates and 5 % / 30 % wrong bearings:
  (a) cvb_verify_noncentral_relative_pose_seeded_batch: the whole chain in one call;
  (b) the chain of the existing calls on the same inputs and seeds: one cvb_match_hamming_batch per query keyframe (its pairings
      as segments), the matches gathered on the host (numpy), cvb_ransac_central_relative_pose_seeded_batch, the inliers merged on
      the host, cvb_ransac_noncentral_relative_pose_seeded_batch, cvb_noncentral_relative_pose_covariance_seeded_batch.
Both are timed alternately in one session: the whole call (host clock around the synchronous calls, median of --reps) and the
device time of their kernels (torch.profiler, a separate run).  Every result of every timed call is checked identical between
(a) and (b).  Prints the GPU name and power limit read in the same run; --out writes the table as JSON.
--sift: the same with SIFT descriptors (300 keypoints per keyframe, the scene of tests/test_verify_relative_sift.py): (a) is
cvb_verify_noncentral_relative_pose_sift_seeded_batch, (b) matches with one cvb_match_l2_batch per query keyframe.
  python tools/verify_timing.py [--sift] [--reps 30] [--out verify_timing.json]"""
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

from covins_b200 import matching as M, placerec as PR   # noqa: E402

KEYS = ("n_matches", "best_sample5", "best_model5", "best_count5", "iterations5", "consumed5", "best_sample", "best_model", "best_count",
        "iterations", "consumed", "cov", "n_valid", "corr")


def chain_existing_calls(ctx, S, prm, n_cov_samples, metric="hamming"):
    """(b): the existing calls with the glue in numpy → the result dict of placerec.verify_noncentral_relative_pose_seeded
    (metric="hamming", desc [R,32] u8) or verify_noncentral_relative_pose_sift_seeded (metric="l2", desc [R,128] float32)"""
    kp, desc, f, sg = S["kf_ptr"], S["desc"], S["bearings"], S["sigma"]
    pairs, pair_ptr = np.asarray(S["pairs"]).reshape(-1, 4), np.asarray(S["pair_ptr"])
    P = len(pairs)
    match, dim = (M.match_candidates_hamming, 32) if metric == "hamming" else (M.match_candidates_l2, 128)
    mts, nm = [None] * P, np.zeros(P, np.int32)
    for a in np.unique(pairs[:, 0]):                       # one matcher call per query keyframe, its pairings as segments
        qs = np.flatnonzero(pairs[:, 0] == a)
        seg = np.concatenate([[0], np.cumsum([kp[b + 1] - kp[b] for b in pairs[qs, 1]])]).astype(np.int32)
        t = np.concatenate([desc[kp[b]:kp[b + 1]] for b in pairs[qs, 1]]).reshape(-1, dim)
        mt, _, n = match(ctx, desc[kp[a]:kp[a + 1]], t, seg, prm["img_match_thres"], prm["ratio_thres"])
        for i, q in enumerate(qs):
            mts[q], nm[q] = mt[i], n[i]
    rows = [np.flatnonzero(m >= 0) for m in mts]
    qa = np.concatenate([kp[a] + r for (a, _, _, _), r in zip(pairs, rows)]).astype(np.int64)
    tb = np.concatenate([kp[b] + m[r] for (_, b, _, _), m, r in zip(pairs, mts, rows)]).astype(np.int64)
    ptr5 = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int32)
    r5 = PR.ransac_central_relative_pose_seeded(ctx, ptr5, f[qa], f[tb], sg[qa], sg[tb], S["seeds5"], prm["threshold5"], prm["max_iterations5"],
                                                prm["probability"])
    pairing = np.repeat(np.arange(P), np.diff(ptr5))
    cand = np.searchsorted(pair_ptr, pairing, side="right") - 1
    src = np.flatnonzero(r5["inlier_mask"])                # pairings are in candidate order
    ptr17 = np.concatenate([[0], np.cumsum(np.bincount(cand[src], minlength=len(pair_ptr) - 1))]).astype(np.int32)
    rig = {k: S[k] for k in ("cam_ptr1", "cam_off1", "cam_rot1", "cam_ptr2", "cam_off2", "cam_rot2")}
    c1, c2 = pairs[pairing[src], 2], pairs[pairing[src], 3]
    r17 = PR.ransac_noncentral_relative_pose_seeded(ctx, ptr17, f[qa[src]], f[tb[src]], sg[qa[src]], sg[tb[src]], c1, c2, **rig, seeds=S["seeds"],
                                                    threshold=prm["threshold17"], max_iterations=prm["max_iterations17"],
                                                    probability=prm["probability"])
    rc = PR.relative_pose_covariance_seeded(ctx, ptr17, f[qa[src]], f[tb[src]], c1, c2, **rig, inlier_mask=r17["inlier_mask"], seeds=S["seeds"],
                                            ref_model=r17["best_model"], n_samples=n_cov_samples)
    inl17 = np.zeros(len(qa), np.int32)
    inl17[src] = r17["inlier_mask"]
    corr = np.stack([pairing, np.concatenate(rows), tb - np.repeat(kp[pairs[:, 1]], np.diff(ptr5)), r5["inlier_mask"], inl17], 1)
    out = dict(n_matches=nm, n_total=int(ptr5[-1]), corr=corr.astype(np.int32).reshape(-1, 5), cov=rc["cov"], n_valid=rc["n_valid"])
    for k in ("best_sample", "best_model", "best_count", "iterations", "consumed"):
        out[k + "5"] = r5[k]; out[k] = r17[k]
    return out


def _same(a, b):
    return all(np.array_equal(np.ascontiguousarray(a[k]).view(np.uint8), np.ascontiguousarray(b[k]).view(np.uint8)) for k in KEYS)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--out", default="")
    ap.add_argument("--sift", action="store_true", help="the SIFT scene (300 keypoints per keyframe) and the SIFT call")
    a = ap.parse_args()
    import torch
    from torch.profiler import profile, ProfilerActivity
    if a.sift:
        from test_verify_relative_sift import PRM, scene
        verify, metric, n_kp = PR.verify_noncentral_relative_pose_sift_seeded, "l2", 300
    else:
        from test_verify_relative import PRM, scene
        verify, metric, n_kp = PR.verify_noncentral_relative_pose_seeded, "hamming", 1000
    assert torch.cuda.is_available(), "needs a GPU"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    gpu = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)
    print("GPU:", gpu)
    ctx = PR.Context(0)
    rows = []
    for outlier in (0.05, 0.3):
        for n_cand in (1, 8, 32):
            S, _ = scene(100 + n_cand, n_cand, n_kp=n_kp, outlier=outlier)
            fused = lambda: verify(ctx, **S, **PRM)                                        # noqa: E731
            chain = lambda: chain_existing_calls(ctx, S, PRM, 300, metric=metric)          # noqa: E731
            ref = fused()
            assert _same(ref, chain()), "the fused call and the chain differ"
            for _ in range(3):
                fused(); chain()
            tf, tc, same = [], [], True
            for _ in range(a.reps):
                t0 = time.perf_counter(); g = fused(); tf.append(time.perf_counter() - t0)
                t0 = time.perf_counter(); h = chain(); tc.append(time.perf_counter() - t0)
                same &= _same(g, ref) and _same(h, ref)
            dev = []
            for fn in (fused, chain):
                with profile(activities=[ProfilerActivity.CUDA]) as pr:
                    for _ in range(5):
                        fn()
                    torch.cuda.synchronize()
                ev = [e for e in pr.events() if e.device_type.name == "CUDA" and "Memcpy" not in e.name and "Memset" not in e.name]
                dev.append(sum(e.device_time for e in ev) / 5 / 1e3)
            row = dict(n_cand=n_cand, outlier=outlier, fused_ms=float(np.median(tf)) * 1e3, chain_ms=float(np.median(tc)) * 1e3,
                       fused_kernels_ms=dev[0], chain_kernels_ms=dev[1], identical=bool(same), n_total=int(ref["n_total"]))
            rows.append(row)
            print(json.dumps(row), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(dict(gpu=gpu, rows=rows), fh, indent=1)
    assert all(r["identical"] for r in rows)


if __name__ == "__main__":
    main()
