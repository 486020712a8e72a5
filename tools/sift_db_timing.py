"""SIFT place-recognition request against a C3-sized map, three ways, alternating in one process:

  resident    the map database (cvb_db_match_l2_dev: device query, dense device outputs; cvb_db_match_l2: host query in,
              compacted accepted matches out), keyframes appended once before the timed region;
  batch       cvb_match_l2_batch on the same candidates (CV_32F rows uploaded, checked and quantised on every call);
  raw         the raw-pointer device path, cvb_knn_l2_u8_batch_dev (k = 2) on u8 rows already in HBM (the tensor-core
              kernel builds its operand tiles in the call's memory first).

Device calls are timed with CUDA events, host calls with a host clock around a call that ends in a device synchronise.
Outputs are asserted equal (the raw path's 2-NN lists through the same distance + ratio filter).  Reports the median of
--reps alternating repeats after --warmup, the achieved pairs/s, and the bytes and int8 operations the request needs,
computed from the shapes, next to the data-sheet bounds (3.35 TB/s, 1979 dense int8 TOP/s; not measured).

  python tools/sift_db_timing.py [--n-kf 2000] [--n-feat 300] [--nq 300] [--reps 20] [--warmup 3] [--json PATH]
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

HBM_BPS = 3.35e12        # H100 SXM data sheet
INT8_OPS = 1979e12       # H100 SXM data sheet, dense


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-kf", type=int, default=2000)
    ap.add_argument("--n-feat", type=int, default=300)
    ap.add_argument("--nq", type=int, default=300)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()

    import torch
    import covins_b200
    from covins_b200 import matching as M, synth

    ctx = covins_b200.Context(0)
    dev = torch.device("cuda", 0)
    desc, _ = synth.sift_keyframes(seed=5, n_kf=a.n_kf + 1, n_feat=a.n_feat)
    q = np.ascontiguousarray(desc[0][:a.nq])
    t = np.ascontiguousarray(desc[1:].reshape(-1, 128))
    seg = synth.seg_ptr_uniform(a.n_kf, a.n_feat)
    rows = len(t)
    thr, ratio = 500.0, 0.8

    db = M.DescriptorDatabase(ctx, reserve_rows=rows, kind="sift")
    t0 = time.perf_counter()
    db.append(t, [a.n_feat] * a.n_kf)
    append_s = time.perf_counter() - t0
    dq = torch.from_numpy(q.astype(np.uint8)).to(dev)
    dt = torch.from_numpy(t.astype(np.uint8)).to(dev)
    dseg = torch.from_numpy(seg).to(dev)
    torch.cuda.synchronize()

    def compact(mt, md, nm):
        kf, qq = np.nonzero(mt >= 0)
        return nm, kf, qq, mt[kf, qq], md[kf, qq]

    def ev_time(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        r = fn()
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1) * 1e-3, r

    def host_time(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        return time.perf_counter() - t0, r

    paths = {
        "resident_dev": lambda: ev_time(lambda: db.match_l2_dev(dq, thr, ratio)),
        "resident_host": lambda: host_time(lambda: db.match_l2(q, thr, ratio)),
        "batch": lambda: host_time(lambda: M.match_candidates_l2(ctx, q, t, seg, thr, ratio)),
        "raw_dev": lambda: ev_time(lambda: M.knn_match_l2(ctx, dq, dt, (dseg, seg), 2)),
    }
    times = {k: [] for k in paths}
    last = {}
    for rep in range(a.warmup + a.reps):
        for k, f in paths.items():
            dt_s, r = f()
            if rep >= a.warmup:
                times[k].append(dt_s)
            last[k] = r

    # equal outputs
    ref = compact(*last["batch"])
    mt, md, nm = (x.cpu().numpy() for x in last["resident_dev"])
    bits = lambda u: np.ascontiguousarray(u).view(np.int32) if np.asarray(u).dtype == np.float32 else np.asarray(u, np.int64)
    same = lambda x, y: all(np.array_equal(bits(u), bits(v)) for u, v in zip(x, y))
    assert same(compact(mt, md, nm), ref), "resident device request differs from cvb_match_l2_batch"
    assert same(last["resident_host"], ref), "resident host request differs from cvb_match_l2_batch"
    idx, dist = (x.cpu().numpy() for x in last["raw_dev"])
    d0, d1 = dist[..., 0], dist[..., 1]
    ok = (idx[..., 0] >= 0) & (idx[..., 1] >= 0) & (d0 <= np.float32(thr)) & (d0 < np.float32(ratio) * d1)
    raw_mt = np.where(ok, idx[..., 0], -1)
    assert np.array_equal(raw_mt, last["batch"][0]), "raw-pointer path differs from cvb_match_l2_batch"
    assert np.array_equal(d0[ok].view(np.int32), last["batch"][1][ok].view(np.int32))

    # what the request needs, from the shapes
    tile_row_bytes = (128 * 128 + 128 * 4) / 128          # the L2 operand tiles (tc_match.cu, XtL2): u8 row + |t|^2
    out_bytes = a.n_kf * a.nq * 8 + a.n_kf * 4
    need = {
        "resident_dev": rows * tile_row_bytes + a.nq * 128 + out_bytes,
        "raw_dev": rows * (128 + 2 * tile_row_bytes) + a.nq * 128 + a.n_kf * a.nq * 16,
    }
    ops = 2.0 * 128 * a.nq * rows
    pairs = float(a.nq) * rows
    res = {"card": card(), "n_kf": a.n_kf, "n_feat": a.n_feat, "nq": a.nq, "rows": rows, "reps": a.reps,
           "accepted_matches": int(ref[0].sum()), "append_s": append_s, "int8_ops": ops,
           "bound_compute_s": ops / INT8_OPS, "paths": {}}
    for k, v in times.items():
        med = float(np.median(v))
        r = {"median_s": med, "min_s": float(np.min(v)), "max_s": float(np.max(v)), "gpairs_per_s": pairs / med / 1e9,
             "int8_tops": ops / med / 1e12}
        if k in need:
            r["bytes"] = need[k]
            r["bound_hbm_s"] = need[k] / HBM_BPS
        res["paths"][k] = r
    print(f"{res['card']}; {a.n_kf} keyframes x {a.n_feat} rows, {a.nq} queries; {res['accepted_matches']} accepted matches; "
          f"append {append_s * 1e3:.1f} ms")
    print(f"data-sheet bounds (not measured): compute {ops / INT8_OPS * 1e6:.1f} us, "
          f"HBM {need['resident_dev'] / HBM_BPS * 1e6:.1f} us (resident), {need['raw_dev'] / HBM_BPS * 1e6:.1f} us (raw)")
    for k, r in res["paths"].items():
        print(f"  {k:14s} median {r['median_s'] * 1e3:8.3f} ms  (min {r['min_s'] * 1e3:.3f}, max {r['max_s'] * 1e3:.3f})  "
              f"{r['gpairs_per_s']:7.1f} Gpairs/s  {r['int8_tops']:6.1f} int8 TOP/s")
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)
    db.close()
    ctx.close()


if __name__ == "__main__":
    main()
