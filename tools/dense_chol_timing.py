"""Development aid: factor time of the tiled Cholesky on a seeded dense SPD matrix against torch.linalg.cholesky.

  python tools/dense_chol_timing.py [n] [out_dir]

n defaults to 12032 (94 tiles, about the pose part of C3).  Prints one JSON line: the factor time of
cvb_dense_cholesky_solve (CUDA events around the factorisation only; best and median of 5 calls after one warm-up call),
the time of torch.linalg.cholesky on the same matrix (FP64, same card), the relative residual of the solution, and the
card's name and power limit.  With out_dir, the solution of the first call is saved there as dense_x_<n>.npy for
comparing builds bit for bit."""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import covins_b200
from covins_b200 import optimization as O

n = int(sys.argv[1]) if len(sys.argv) > 1 else 12032
out_dir = sys.argv[2] if len(sys.argv) > 2 else None
rng = np.random.default_rng(12032)
# SPD and dense, built element by element (no BLAS reduction order in the input): Kac-Murdock-Szego 0.999^|i-j| + 0.5 I (no zero tile)
idx = np.arange(n, dtype=np.float64)
A = np.power(0.999, np.abs(idx[:, None] - idx[None, :])) + 0.5 * np.eye(n)
b = rng.standard_normal(n)

ctx = covins_b200.Context(0)
x0, _ = O.dense_cholesky_solve(ctx, A, b)   # warm-up (module load, workspaces)
ours, x = [], None
for _ in range(5):
    xi, ms = O.dense_cholesky_solve(ctx, A, b)
    ours.append(ms)
    if x is None:
        x = xi
    assert np.array_equal(xi, x), "repeated solves differ"
res = float(np.linalg.norm(A @ x - b) / np.linalg.norm(b))
if out_dir:
    os.makedirs(out_dir, exist_ok=True)
    np.save(os.path.join(out_dir, f"dense_x_{n}.npy"), x)

At = torch.from_numpy(A).cuda()
torch.linalg.cholesky(At)
torch.cuda.synchronize()
ref = []
for _ in range(5):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    torch.linalg.cholesky(At)
    e1.record()
    torch.cuda.synchronize()
    ref.append(e0.elapsed_time(e1))
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
print(json.dumps({"n": n, "factor_ms_best": min(ours), "factor_ms_median": float(np.median(ours)),
                  "torch_cholesky_ms_best": min(ref), "torch_cholesky_ms_median": float(np.median(ref)),
                  "rel_residual": res, "card": card}))
ctx.close()
