"""Development aid: latency + phase breakdown of the diagonal-tile kernel (run under gpurun)."""
import ctypes as C, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import covins_b200
from covins_b200._lib import lib

ctx = covins_b200.Context(0)
us = C.c_double(); ph = np.zeros(10, np.int64)
ctx.check(lib().cvb_microbench_potrf(ctx.handle, 200, C.byref(us), ph.ctypes.data_as(C.c_void_p)))
names = ["start", "loaded", "4 block cols factored", "6 block cols factored", "factored", "inverted",
         "sum diag-block steps", "sum step 1 + barrier", "sum step 2 + barrier", "last inverse block row"]
print(f"potrf_inv_kernel: {us.value:.1f} us per tile (back-to-back launches)")
for n, v in zip(names, ph):
    print(f"  {n:22s} {int(v):8d} cycles")
lat = np.zeros(8)
ctx.check(lib().cvb_microbench_latency(ctx.handle, lat.ctypes.data_as(C.POINTER(C.c_double))))
for n, v in zip(["dep DFMA", "8-way indep DFMA (per op)", "dep rsqrt(double)+add", "dep SHFL double", "STS+LDS round trip",
                 "dep DMUL", "dep FFMA", "SM clock MHz (est)"], lat):
    print(f"  {n:28s} {v:9.1f}")
mm = np.zeros(2)
ctx.check(lib().cvb_microbench_minmax(ctx.handle, mm.ctypes.data_as(C.POINTER(C.c_double))))
print(f"  integer min/max issue rate (lane-instr/clk/SM): 32-bit {mm[0]:.1f}, packed u16x2 {mm[1]:.1f}")
