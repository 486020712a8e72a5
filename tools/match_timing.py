"""Development aid (needs a GPU): time the matching kernels (POPC/DP4A scalar vs wgmma) on resident data."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import covins_b200
from covins_b200 import matching as M, synth

ctx = covins_b200.Context(0)
dev = torch.device("cuda", 0)
g = torch.Generator(device=dev).manual_seed(1)

def timeit(fn, n=10, w=3):
    for _ in range(w): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n

for name, n_kf, nf, nq in (("ORB C3", 2000, 1000, 1000), ("ORB C2", 800, 1000, 1000), ("ORB C5", 10000, 1000, 1000)):
    t = torch.randint(0, 256, (n_kf * nf, 32), dtype=torch.uint8, device=dev, generator=g)
    q = t[:nq].clone()
    h_seg = synth.seg_ptr_uniform(n_kf, nf); d_seg = torch.from_numpy(h_seg).to(dev)
    for kern in ("popc", "tc"):
        os.environ["COVINS_B200_MATCH_KERNEL"] = kern
        ms = timeit(lambda: M.match_candidates_hamming(ctx, q, t, (d_seg, h_seg), 40.0, 0.8))
        ms2 = timeit(lambda: M.knn_match_hamming(ctx, q, t, (d_seg, h_seg), 2))
        print(f"{name:8s} {kern:5s}: fused match {ms:8.3f} ms = {nq*n_kf*nf/ms/1e6:9.1f} Gpairs/s | knn k=2 {ms2:8.3f} ms = {nq*n_kf*nf/ms2/1e6:9.1f} Gpairs/s", flush=True)
    if name == "ORB C3":
        skipA = (torch.rand(nq, device=dev, generator=g) < 0.6).to(torch.uint8); skipB = (torch.rand(n_kf * nf, device=dev, generator=g) < 0.6).to(torch.uint8)
        for kern in ("popc", "tc"):
            os.environ["COVINS_B200_MATCH_KERNEL"] = kern
            ms = timeit(lambda: M.landmark_match(ctx, q, skipA, t, skipB, (d_seg, h_seg)), n=5)
            print(f"{name:8s} {kern:5s}: DenseMatcher landmark match {ms:8.3f} ms = {nq*n_kf*nf/ms/1e6:9.1f} Gpairs/s (all pairs counted)", flush=True)
    del t
for name, n_kf, nf, nq in (("SIFT C5/8", 1250, 300, 300), ("SIFT C5", 10000, 300, 300)):
    t = torch.randint(0, 256, (n_kf * nf, 128), dtype=torch.uint8, device=dev, generator=g)
    q = t[:nq].clone()
    h_seg = synth.seg_ptr_uniform(n_kf, nf); d_seg = torch.from_numpy(h_seg).to(dev)
    for kern in ("popc", "tc"):
        os.environ["COVINS_B200_MATCH_KERNEL"] = kern
        ms = timeit(lambda: M.knn_match_l2(ctx, q, t, (d_seg, h_seg), 2))
        print(f"{name:9s} {kern:5s}: knn k=2 {ms:8.3f} ms = {nq*n_kf*nf/ms/1e6:9.1f} Gpairs/s", flush=True)
    del t
