"""Time the in-process group GBA (cvb_gba_group) against cvb_gba on one device, on a named synthetic config (default C3).

Layouts, each timed `--repeats` times after one warm-up call:
  single      cvb_gba on device 0
  devices     a group with one rank per visible device (a group of one on a one-GPU machine)
  shared2     a group of 2 ranks sharing device 0
Reports the GBA wall time (both rounds, set-up included) and the trust-region iterations of both rounds per second of it,
and checks every group's merged states against cvb_gba's (states 1e-6 relative, cost 1e-6, the tolerances of the C1 sharded
tests) and its round-1 outlier set.  The card's name and power limit are read in the same command.
  python tools/group_timing.py [--config C3] [--iterations 10] [--repeats 3] [--peer]
--peer asks for the peer path in the `devices` layout (it needs a device per rank; `shared2` always takes the all-reduce
path).
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import covins_b200
from covins_b200 import optimization as O, synth_map


def rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-12))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C3")
    ap.add_argument("--iterations", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--peer", action="store_true")
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(f"GPU: {gpu}", flush=True)
    ndev = torch.cuda.device_count()
    t0 = time.time()
    p = synth_map.make_config(a.config)
    print(f"{a.config}: generated in {time.time() - t0:.1f} s, K={p['K']} L={p['L']} obs={len(p['obs_kf'])}, {ndev} device(s)")
    peer = a.peer
    ctx0 = covins_b200.Context(0)

    def timed(fn):
        fn()   # warm-up: module load, pool growth
        ts, out = [], None
        for _ in range(a.repeats):
            torch.cuda.synchronize()
            t = time.perf_counter()
            out = fn()
            ts.append(time.perf_counter() - t)
        return out, ts

    ref, ts = timed(lambda: O.global_bundle_adjustment(ctx0, p, iterations_limit=a.iterations))
    its = 5 + ref["iterations"]
    rows = [dict(layout="single", ranks=1, e2e_s=min(ts), e2e_all=ts, it_per_s=its / min(ts))]
    print(json.dumps(rows[-1]), flush=True)
    layouts = [("devices", list(range(ndev))), ("shared2", [0, 0])]
    for name, devs in layouts:
        ctxs = [ctx0] + [covins_b200.Context(d) for d in devs[1:]]
        g = O.Group(ctxs)
        use_peer = peer and name == "devices"
        got, ts = timed(lambda: O.global_bundle_adjustment_group(g, p, iterations_limit=a.iterations, peer_path=use_peer))
        g.close()
        for c in ctxs[1:]:
            c.close()
        inc = ref["lm_owner"] >= 0
        well = inc & (np.abs(ref["lm"]).max(1) < 100.0)
        err = dict(pose=rel(got["pose"], ref["pose"]), sb=rel(got["speedbias"], ref["speedbias"]),
                   lm=rel(got["lm"][well], ref["lm"][well]), cost=float(np.abs(got["cost"] / ref["cost"] - 1).max()))
        ok = (got["iterations"] == ref["iterations"] and got["steps"] == ref["steps"] and
              np.array_equal(got["obs_removed"], ref["obs_removed"]) and max(err.values()) < 1e-6)
        rows.append(dict(layout=name, ranks=len(devs), devices=devs, e2e_s=min(ts), e2e_all=ts,
                         it_per_s=(5 + got["iterations"]) / min(ts), matches_world1=bool(ok), err=err,
                         obs_removed_diff=int((got["obs_removed"] != ref["obs_removed"]).sum())))
        print(json.dumps(rows[-1]), flush=True)
    ctx0.close()
    print(f"peer path (devices layout): {peer}; iterations per GBA: 5 (round 1) + {ref['iterations']} (round 2)")
    if not all(r.get("matches_world1", True) for r in rows):
        sys.exit(1)


if __name__ == "__main__":
    main()
