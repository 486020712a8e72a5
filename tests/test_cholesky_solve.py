"""The triangular solves of the tiled Cholesky (subst_kernel in covins_b200/csrc/cholesky.cu): one persistent launch per
direction whose CTAs take tile rows from a ticket and wait on per-row flags.

A harness (tests/cpp/solve_harness.cu) factors a host matrix once and runs solve_grid, the launch helper behind solve(),
with 1, 2 and 3 CTAs and with as many as fit on the device, then ten more times with one FactorStreams.  The solution must
meet the forward-error bound of tests/test_cholesky_kernels.py and be bitwise the same for every grid size and every
repetition: the subtractions of a row happen in a fixed order whichever CTA forms it and however the CTAs interleave, and
the flags are cleared for every solve (a stale flag would let a row read a result before it is written)."""
import os
import subprocess
import zlib

import numpy as np
import pytest
from test_cholesky_kernels import LD, T, U, _bound, _matrix, _pattern, _same_bits, _within

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
GRIDS = [1, 2, 3, 0]   # 0 = as many CTAs as fit on the device
REPS = 10

# (pattern, nt, n): dense up to 40 tile columns (a chain of 40 dependent rows, more rows than CTAs in the small grids),
# and the sparse patterns of the factorisation tests; "ba" solves with its own column groups (the level plan)
CASES = [("dense", 1, T - 17), ("dense", 5, 5 * T), ("dense", 40, 40 * T - 17), ("banded", 12, 12 * T - 17),
         ("arrow", 12, 12 * T), ("gaps", 10, 10 * T - 17), ("random0", 12, 12 * T - 17), ("random1", 12, 12 * T),
         ("ba", 10, 10 * T - 17)]
IDS = [f"{p}-nt{nt}-n{n}" for p, nt, n in CASES]


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("solve_harness") / "solve_harness")
    subprocess.check_call([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
                           "-o", exe, os.path.join(ROOT, "tests", "cpp", "solve_harness.cu")])
    return exe


def test_solve_harness_builds(harness):
    assert os.access(harness, os.X_OK)


def _run(harness, tmp, case):
    p, nt, n = case
    mask, group = _pattern(p, nt)
    A, kappa = _matrix(mask, n, "well", zlib.crc32(repr(case).encode()))
    xs = np.random.default_rng(11).standard_normal(n)
    b = (A.astype(LD) @ xs.astype(LD)).astype(np.float64)
    grp = np.asarray(group if group is not None else [-1] * nt, np.int32)
    arrays = [np.array([nt, n, REPS, 0 if group is None else 1], np.int32), np.tril(mask).astype(np.int32), grp, A, b,
              np.array(GRIDS, np.int32)]
    fin, fout = os.path.join(tmp, "in.bin"), os.path.join(tmp, "out.bin")
    with open(fin, "wb") as f:
        for a in arrays:
            a = np.ascontiguousarray(a)
            f.write(np.int64(a.nbytes).tobytes())
            f.write(a.tobytes())
    r = subprocess.run([harness, fin, fout], capture_output=True, text=True)
    assert r.returncode == 0, f"solve_harness exited with {r.returncode}: {r.stderr}"
    with open(fout, "rb") as f:
        raw = f.read()
    out, pos = [], 0
    while pos < len(raw):
        nb = int(np.frombuffer(raw, np.int64, 1, pos)[0])
        out.append(raw[pos + 8:pos + 8 + nb])
        pos += 8 + nb
    assert len(out) == 1 + len(GRIDS) + REPS
    flag = int(np.frombuffer(out[0], np.int32)[0])
    xs_out = [np.frombuffer(o, np.float64) for o in out[1:]]
    return flag, xs_out, xs, kappa, n


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_solve_grids_and_repeats(harness, tmp_path, case):
    """x meets ||x - x*||_inf / ||x*||_inf <= 4 n u kappa_2(A) and is bitwise the same for 1, 2, 3 and all CTAs and over
    ten further solves with the same streams"""
    flag, runs, xs, kappa, n = _run(harness, str(tmp_path), case)
    assert flag == 0
    ref = runs[-1 - REPS]   # as many CTAs as fit
    assert np.isfinite(ref).all()
    err = np.abs(ref[:n].astype(LD) - xs).max() / np.abs(xs).max()
    _within(f"solve x {case}", err, _bound(4 * n * U, LD(kappa), 0))
    for g, x in zip(GRIDS, runs[:len(GRIDS)]):
        _same_bits(f"x ({g} CTAs)", x, ref)
    for r, x in enumerate(runs[len(GRIDS):]):
        _same_bits(f"x (repeat {r})", x, ref)
