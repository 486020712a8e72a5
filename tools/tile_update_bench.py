"""Development aid: the Cholesky's bulk trailing update (tile_update_kernel) timed on its own, against a register-only DMMA
probe and cuBLAS DGEMM at the same flop count.

  python tools/tile_update_bench.py [--reps N] [--rounds R] [--cholesky NAME=PATH ...]

Builds tools/tile_update_bench.cu once per cholesky.cu source (default: this tree's, named "tree") into a temporary
directory, and runs the builds R times in alternation.  Each run prints, per pass (the first bulk pass of a dense 94-tile
pose part, 4095 targets x 4 panels, and one half way through, 1128 targets), the kernel time L2-warm and after a 256 MB
flush, TFLOP/s, the bytes counted from shapes (1 MB of operands and 256 KB of C per target) and a hash of the result.
Then cuBLAS DGEMM (torch.mm, FP64) at each pass's flop count, and the card's name, power limit and SM clocks."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def build(src, exe):
    subprocess.check_call([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
                           "-I", os.path.join(ROOT, "covins_b200", "csrc"), f'-DCHOLESKY_CU="{os.path.abspath(src)}"',
                           "-o", exe, os.path.join(ROOT, "tools", "tile_update_bench.cu")])


def dgemm(gflop, reps):
    """torch.mm of (4096 x K) by (K x 4096) in FP64, K chosen for the flop count; median time and TFLOP/s"""
    import torch
    n = 4096
    k = max(16, round(gflop * 1e9 / (2 * n * n) / 16) * 16)
    a = torch.rand(n, k, dtype=torch.float64, device="cuda")
    b = torch.rand(k, n, dtype=torch.float64, device="cuda")
    for _ in range(2):
        torch.mm(a, b)
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        torch.mm(a, b)
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    ms.sort()
    med = ms[len(ms) // 2]
    return {"kernel": "cublas_dgemm", "shape": [n, k, n], "gflop": round(2 * n * n * k * 1e-9, 2), "ms_median": round(med, 4),
            "tflops_median": round(2 * n * n * k / med * 1e-9, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=1)
    ap.add_argument("--cholesky", action="append", default=[], metavar="NAME=PATH")
    args = ap.parse_args()
    srcs = [s.split("=", 1) for s in args.cholesky] or [["tree", os.path.join(ROOT, "covins_b200", "csrc", "cholesky.cu")]]
    with tempfile.TemporaryDirectory() as tmp:
        exes = []
        for name, src in srcs:
            exe = os.path.join(tmp, f"tile_update_bench_{name}")
            build(src, exe)
            exes.append((name, exe))
        gflop = {}
        for rnd in range(args.rounds):
            for name, exe in exes:
                out = subprocess.run([exe, str(args.reps)], capture_output=True, text=True)
                if out.returncode != 0:
                    sys.exit(f"{name}: exit {out.returncode}: {out.stderr}")
                for line in out.stdout.splitlines():
                    rec = json.loads(line)
                    if "gflop" in rec:
                        gflop[rec["pass"]] = rec["gflop"]
                    print(json.dumps({"build": name, "round": rnd, **rec}), flush=True)
    for p, g in gflop.items():
        print(json.dumps({"pass": p, **dgemm(g, args.reps)}), flush=True)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({"card": card}))


if __name__ == "__main__":
    main()
