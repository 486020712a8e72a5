#!/usr/bin/env python
"""Times Optimization::PoseGraphOptimization with its write-back (optimization_be.cpp:833-1086) at the sizes of BASELINE
configs C3 (5 agents x 400 keyframes, 100 k landmarks) and C5 (12 x 834 keyframes, 1 M landmarks).

The pose graph reads only poses, chains, loops and each landmark's reference keyframe, so the maps are built directly at
those sizes (no observation structure): agents on smooth trajectories, VIO poses that drift from them, loops between
agents, every landmark anchored to a random keyframe.  One JSON line per config, with the card's name, power limit and
SM clocks read in the same run:
  * "cvb_pgo_ms": covins_b200.optimization.pose_graph_optimization_map, end-to-end host time of one call (median, min
    and max of --calls after --warmup; the pageable copies both ways included);
  * "parent_ms": the composition it replaces on the same map: optimization.pgo_edges (host edge list) +
    optimization.pose_graph_optimization (cvb_ba_solve) + oracle/pgo.py's write-back (numpy, vectorised);
  * "k17a_us" / "k17b_us": device time of pgo_edges_kernel / pgo_writeback_kernel from a torch.profiler (CUPTI) pass of
    its own, and K17b's compulsory bytes over its time (the reference keyframes' poses each landmark gathers are not
    counted);
  * the outputs of cvb_pgo are checked bitwise against cvb_ba_solve fed oracle/pgo.py's edges and its write-back.
Not measured: the C++ shim's container walk around the call, and the reference's host loop itself (not in this tree).
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

SIZES = {"C3": (5, 400, 100_000), "C5": (12, 834, 1_000_000)}


def make_problem(n_agents, kf_per_agent, n_lm, seed=0):
    from covins_b200 import synth_map
    rng = np.random.default_rng(seed)
    K = n_agents * kf_per_agent
    agent = np.repeat(np.arange(n_agents), kf_per_agent).astype(np.int32)
    kid = np.tile(np.arange(kf_per_agent), n_agents).astype(np.int32)
    pose = np.zeros((K, 7))
    vio = np.zeros((K, 7))
    for a in range(n_agents):
        s = slice(a * kf_per_agent, (a + 1) * kf_per_agent)
        t = np.arange(kf_per_agent) * 0.2
        yaw = 0.05 * t + a
        pos = np.stack([10 * np.cos(0.03 * t + a), 10 * np.sin(0.03 * t + a), 0.1 * np.sin(t)], 1)
        drift = np.cumsum(rng.normal(size=(kf_per_agent, 3)) * 0.01, 0)
        for k, (y, p, d) in enumerate(zip(yaw, pos, drift)):
            R = synth_map.rot_exp(np.array([0, 0, y]))
            pose[s][k, :4] = synth_map.rot_to_quat(R)
            pose[s][k, 4:] = p
            vio[s][k, :4] = synth_map.rot_to_quat(synth_map.rot_exp(rng.normal(size=3) * 1e-3) @ R)
            vio[s][k, 4:] = p + d
    nl = 4 * n_agents
    li = rng.integers(0, K, nl).astype(np.int32)
    lj = ((li + kf_per_agent + rng.integers(0, kf_per_agent, nl)) % K).astype(np.int32)
    keep = li != lj
    li, lj = li[keep], lj[keep]
    p = dict(K=K, L=n_lm, pose=pose, pose_const=(kid == 0).astype(np.uint8), agent_of=agent, kf_id=kid,
             extr=np.array([[0, 0, 0, 1.0, 0, 0, 0]]), speedbias=rng.normal(size=(K, 9)), lm=rng.normal(size=(n_lm, 3)) * 20,
             loop_i=li, loop_j=lj, loop_q=np.tile([0, 0, 0, 1.0], (len(li), 1)), loop_t=rng.normal(size=(len(li), 3)))
    return p, vio


def timed(fn, calls, warmup):
    import torch
    for _ in range(warmup):
        fn()
    ms = []
    for _ in range(calls):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ms.append((time.perf_counter() - t0) * 1e3)
    return dict(ms_median=round(float(np.median(ms)), 3), ms_min=round(min(ms), 3), ms_max=round(max(ms), 3), calls=calls)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="C3,C5")
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    args = ap.parse_args()
    import torch
    from covins_b200 import Context, optimization as O
    from oracle import pgo as ora
    if not torch.cuda.is_available():
        raise SystemExit("pgo_bench: no CUDA device (there is no fallback)")
    card = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader", "-i", "0"],
                                   text=True).strip()
    ctx = Context(0)
    for name in args.configs.split(","):
        p, vio = make_problem(*SIZES[name])
        pr = O.pgo_map_problem(p)
        pr["T_ws_vio"] = ora.pose7_to_transform(vio)
        pr["lm_ref"] = np.random.default_rng(1).integers(0, p["K"], p["L"]).astype(np.int32)
        pr["lm_has_obs"] = np.ones(p["L"], np.uint8)
        # correctness at this size: bitwise the solve fed the oracle's edges, and the oracle's write-back
        got = O.pose_graph_optimization_map(ctx, pr)
        edges = ora.pgo_edges(pr)
        pp = dict(K=p["K"], pose=ora.start_poses(pr), pose_const=pr["pose_const"], extr=p["extr"])
        sol = O.pose_graph_optimization(ctx, pp, edges)
        wb = ora.writeback(pr, sol["pose"])
        same = bool(np.array_equal(got["pose"].view(np.uint64), sol["pose"].view(np.uint64)) and
                    np.array_equal(got["T_ws"].reshape(-1, 16).view(np.uint64), wb["T_ws_out"].view(np.uint64)) and
                    np.array_equal(got["velocity"].view(np.uint64), wb["velocity_out"].view(np.uint64)) and
                    np.array_equal(got["lm"].view(np.uint64), wb["lm_out"].view(np.uint64)))

        def parent():
            e = O.pgo_edges(p, vio, covins_mode=True)
            s = O.pose_graph_optimization(ctx, p, e)
            ora.writeback(pr, s["pose"])
        t_new = timed(lambda: O.pose_graph_optimization_map(ctx, pr), args.calls, args.warmup)
        t_old = timed(parent, args.calls, args.warmup)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                O.pose_graph_optimization_map(ctx, pr)
            torch.cuda.synchronize()
        dev = {}
        for ev in prof.events():
            for key, kname in (("k17a", "pgo_edges_kernel"), ("k17b", "pgo_writeback_kernel")):
                if kname in ev.name and ev.device_type.name == "CUDA":
                    dev.setdefault(key, []).append(ev.device_time)
        K, L = p["K"], p["L"]
        # K17b's compulsory traffic: per keyframe the solved pose, T_ws and velocity read, T_ws_out, pose and velocity written;
        # per landmark lm_ref, lm_has_obs and the position read, the position and the erase flag written
        b_bytes = K * (56 + 128 + 24 + 128 + 56 + 24) + L * (4 + 1 + 24 + 24 + 1)
        k17a = float(np.median(dev["k17a"])) if "k17a" in dev else None
        k17b = float(np.median(dev["k17b"])) if "k17b" in dev else None
        rec = dict(bench="pgo", config=name, K=K, L=L, n_loop=int(len(p["loop_i"])), n_edge=got["n_edge"], iterations=got["iterations"],
                   bitwise_equal_to_solve_and_oracle=same, cvb_pgo_ms=t_new, parent_ms=t_old, k17a_us=k17a, k17b_us=k17b,
                   k17b_bytes=b_bytes, k17b_GBps=round(b_bytes / (k17b * 1e-6) / 1e9, 1) if k17b else None, card=card)
        line = json.dumps(rec)
        print(line, flush=True)
        if args.out:
            with open(args.out, "a") as f:
                f.write(line + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
