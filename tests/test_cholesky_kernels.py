"""The tiled FP64 Cholesky (covins_b200/csrc/cholesky.cu) kernel by kernel and as a whole, against extended precision.

A harness (tests/cpp/chol_harness.cu, built here with the library's flags) compiles cholesky.cu into its own translation
unit and runs one launch of tile_update_kernel, syrk_kernel, trsm_kernel, chain_gemm_kernel<0|1> or potrf_inv_kernel on
host tiles, or the packing, factor() and solve() of cvb_dense_cholesky_solve under a chosen plan.

Every result is checked one of three ways:
  - against a longdouble reference (11 more mantissa bits than the kernels' doubles) under a rigorous rounding-error
    bound, elementwise |err| <= bound with u = 2^-53 and gamma_m = m u / (1 - m u).  The bounds hold for any order of
    summation, so they do not depend on how DMMA accumulates, but one operand read from the wrong place is far over them.
    The reference's own rounding is added to each bound (_bound: gamma_m with the longdouble unit roundoff, for the m
    roundings of a reference sum and the few operations that form err and the bound).  The largest err/bound of each
    check is printed (-s);
  - bitwise, where the design promises identical bits: tile_update_kernel vs syrk_kernel, run to run, the blocked vs the
    column-by-column vs the column-group schedule, and everything a launch must leave alone (NaN guard tiles around the
    packed array, operand tiles, the quadrant above the diagonal of a diagonal tile, the upper triangle of the tile
    potrf_inv_kernel factors);
  - exact values a kernel must write: the +0.0 above the diagonal of every tile inverse, which fwd_kernel and bwd_kernel
    read as part of the whole tile.  The harness fills the inverse (and solution) buffers with NaN before each launch,
    as a reused workspace holds stale values, so an element the kernel skips shows up."""
import os
import subprocess
import zlib

import numpy as np
import pytest
import scipy.linalg as sl
from test_tile_plan import _random_mask, _structure

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
T = 128
LD = np.longdouble
U = LD(2.0) ** -53
UL = LD(np.finfo(LD).eps) / 2   # unit roundoff of the reference arithmetic (2^-64 for x87 extended precision)
gpu = pytest.mark.gpu
UPPER_Q = np.zeros((T, T), bool)   # the quadrant above the diagonal of a diagonal tile: never read nor written
UPPER_Q[:64, 64:] = True
STRICT_UPPER = np.triu(np.ones((T, T), bool), 1)


def gamma(m):
    return m * U / (1 - m * U)


def _bound(coef, mag, m_ref):
    """bound on |got - ref| when |got - exact| <= coef * M: ref and the computed magnitude mag are longdouble sums of at
    most m_ref roundings each, so |ref - exact| <= gL M and mag >= (1 - gL) M, with gL = gamma_{m_ref + 3} in the
    longdouble unit roundoff (+3: forming err, the product coef * mag and the division)"""
    gl = (m_ref + 3) * UL / (1 - (m_ref + 3) * UL)
    return (coef + gl) * np.asarray(mag, LD) / (1 - gl)


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("chol_harness") / "chol_harness")
    subprocess.check_call([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
                           "-o", exe, os.path.join(ROOT, "tests", "cpp", "chol_harness.cu")])
    return exe


class Harness:
    """runs the harness on a list of arrays, returns its output arrays as raw bytes; caches results per key"""

    def __init__(self, exe, tmp):
        self.exe, self.tmp, self.cache = exe, tmp, {}

    def __call__(self, mode, *arrays):
        fin, fout = os.path.join(self.tmp, "in.bin"), os.path.join(self.tmp, "out.bin")
        with open(fin, "wb") as f:
            for a in arrays:
                a = np.ascontiguousarray(a)
                f.write(np.int64(a.nbytes).tobytes())
                f.write(a.tobytes())
        r = subprocess.run([self.exe, mode, fin, fout], capture_output=True, text=True)
        assert r.returncode == 0, f"chol_harness {mode} exited with {r.returncode}: {r.stderr}"
        with open(fout, "rb") as f:
            raw = f.read()
        out, pos = [], 0
        while pos < len(raw):
            nb = int(np.frombuffer(raw, np.int64, 1, pos)[0])
            out.append(raw[pos + 8:pos + 8 + nb])
            pos += 8 + nb
        return out

    def cached(self, key, fn):
        if key not in self.cache:
            self.cache[key] = fn()
        return self.cache[key]


@pytest.fixture(scope="module")
def h(harness, tmp_path_factory):
    return Harness(harness, str(tmp_path_factory.mktemp("chol_io")))


def _f64(b, *shape):
    return np.frombuffer(b, np.float64).reshape(shape) if shape else np.frombuffer(b, np.float64)


def _within(tag, err, bound):
    """|err| <= bound elementwise (NaN fails); prints the largest err/bound"""
    err, bound = np.asarray(err, LD).ravel(), np.asarray(bound, LD).ravel()
    ok = err <= bound
    ratio = np.where(bound > 0, err / np.where(bound > 0, bound, 1), np.where(err > 0, LD(np.inf), LD(0)))
    worst = float(np.max(np.where(np.isnan(ratio), LD(np.inf), ratio))) if ratio.size else 0.0
    print(f"{tag}: max err/bound = {worst:.3g}")
    assert ok.all(), f"{tag}: {int((~ok).sum())} of {ok.size} elements over the bound (max err/bound {worst:.3g}), " \
                     f"first at flat index {int(np.argmin(ok))}"


def _same_bits(tag, a, b):
    d = np.ascontiguousarray(a, np.float64).view(np.uint64) != np.ascontiguousarray(b, np.float64).view(np.uint64)
    assert not d.any(), f"{tag}: {int(d.sum())} of {d.size} values differ bitwise, first at {tuple(np.argwhere(d)[0])}"


def _sym(A):
    """exactly symmetric copy of the lower triangle"""
    return np.tril(A) + np.tril(A, -1).T


def test_harness_builds(harness):
    assert os.access(harness, os.X_OK)


# ---------------------------------------------------------------- trailing update (tile_update_kernel, syrk_kernel)
# name: (k0, [(i, j, mask)]): target tiles (i >= j) and the panels k0 + q of the bits q of mask
UPDATE_CASES = {
    "mask_1": (0, [(1, 1, 0b1), (2, 1, 0b1), (3, 3, 0b1)]),
    "mask_1111": (0, [(4, 4, 0b1111), (5, 4, 0b1111), (6, 5, 0b1111), (6, 6, 0b1111)]),
    "mask_1010": (0, [(4, 4, 0b1010), (6, 4, 0b1010), (7, 7, 0b1010)]),
    "mask_1001": (0, [(5, 4, 0b1001), (4, 4, 0b1001), (7, 5, 0b1001)]),
    "high_bit": (0, [(32, 32, 1 << 31), (33, 32, 1 << 31)]),
    "mask_32": (0, [(32, 32, 0xFFFFFFFF), (33, 32, 0xFFFFFFFF), (33, 33, 0xFFFFFFFF)]),
    "k0_5": (5, [(9, 9, 0b1011), (10, 9, 0b0110), (12, 10, 0b1111), (12, 12, 0b0001)]),
    # 153 pairs (> 132 SMs: several waves), diagonal and off-diagonal targets at every position of a 17-tile band
    "waves": (0, [(i, j, (1, 2, 3)[(i + j) % 3]) for j in range(2, 19) for i in range(j, 19)]),
}


def _update_input(case):
    """packed tiles S (index 0 and the last are NaN guard tiles), tile_of, pair list.  Every panel tile up to the mask's
    highest bit exists, read or not; all values are distinct, each tile scaled by its own power of two"""
    k0, pairs = UPDATE_CASES[case]
    rng = np.random.default_rng(zlib.crc32(case.encode()))
    nt = max(i for i, _, _ in pairs) + 1
    tiles = {(i, j) for i, j, _ in pairs}
    for i, j, m in pairs:
        for q in range(m.bit_length()):
            tiles |= {(i, k0 + q), (j, k0 + q)}
    order = sorted(tiles)
    tile_of = np.full((nt, nt), -1, np.int32)
    for (i, j), p in zip(order, rng.permutation(len(order))):
        tile_of[i, j] = p + 1
    S = rng.standard_normal((len(order) + 2, T, T)) * np.exp2(rng.integers(-8, 9, len(order) + 2))[:, None, None]
    S[0] = S[-1] = np.nan
    return k0, pairs, nt, tile_of, S


def _update_run(h, case, kernel, rep=0):
    def run():
        k0, pairs, nt, tile_of, S = _update_input(case)
        pi, pj, pm = (np.array([p[c] for p in pairs], np.uint32).view(np.int32) for c in range(3))
        out = h("update", np.array([nt, k0, {"tile_update": 0, "syrk": 1}[kernel]], np.int32), tile_of, pi, pj, pm, S)
        return _f64(out[0], *S.shape)
    return h.cached(("update", case, kernel, rep), run)


def _update_ref(h, case):
    def ref():
        k0, pairs, nt, tile_of, S = _update_input(case)
        out = {}
        for i, j, m in pairs:
            C = S[tile_of[i, j]].astype(LD)
            val, mag, ks = C.copy(), np.abs(C), [k0 + q for q in range(32) if m >> q & 1]
            for k in ks:
                A, B = S[tile_of[i, k]].astype(LD), S[tile_of[j, k]].astype(LD)
                val -= A @ B.T
                mag += np.abs(A) @ np.abs(B).T
            out[(i, j)] = (val, _bound(gamma(T + len(ks)), mag, T + len(ks)))
        return out
    return h.cached(("update_ref", case), ref)


@gpu
@pytest.mark.parametrize("kernel", ["tile_update", "syrk"])
@pytest.mark.parametrize("case", list(UPDATE_CASES))
def test_update_accuracy(h, case, kernel):
    """|C_gpu - (C - sum_p A_ip A_jp^T)| <= gamma_{T+np} (|C| + sum_p |A_ip||A_jp|^T), np = panels in the mask"""
    _, pairs, _, tile_of, _ = _update_input(case)
    got, ref = _update_run(h, case, kernel), _update_ref(h, case)
    errs, bnds = [], []
    for i, j, _ in pairs:
        sel = ~UPPER_Q if i == j else np.ones((T, T), bool)
        val, bnd = ref[(i, j)]
        errs.append(np.abs(got[tile_of[i, j]].astype(LD) - val)[sel])
        bnds.append(bnd[sel])
    _within(f"update {kernel} {case}", np.concatenate(errs), np.concatenate(bnds))


@gpu
@pytest.mark.parametrize("kernel", ["tile_update", "syrk"])
@pytest.mark.parametrize("case", list(UPDATE_CASES))
def test_update_writes_only_targets(h, case, kernel):
    """guard tiles, operand and other tiles, and the quadrant above the diagonal of a diagonal target are bitwise
    unchanged"""
    _, pairs, _, tile_of, S = _update_input(case)
    got = _update_run(h, case, kernel)
    target = {int(tile_of[i, j]): i == j for i, j, _ in pairs}
    for t in range(len(S)):
        if t not in target:
            _same_bits(f"non-target tile {t}", got[t], S[t])
        elif target[t]:
            _same_bits(f"upper quadrant of diagonal target tile {t}", got[t][UPPER_Q], S[t][UPPER_Q])


@gpu
@pytest.mark.parametrize("case", list(UPDATE_CASES))
def test_update_kernels_bit_identical(h, case):
    """tile_update_kernel subtracts each panel's product on its own in increasing panel order, as syrk_kernel does"""
    _same_bits(f"tile_update vs syrk {case}", _update_run(h, case, "tile_update"), _update_run(h, case, "syrk"))


@gpu
@pytest.mark.parametrize("case", ["mask_1111", "mask_32", "waves"])
def test_update_run_to_run(h, case):
    _same_bits(f"tile_update run to run {case}", _update_run(h, case, "tile_update"), _update_run(h, case, "tile_update", 1))


# ---------------------------------------------------------------- panel solves (trsm_kernel, chain_gemm_kernel)
def _tile_inverse(rng):
    """a lower-triangular tile inverse with exact zeros above the diagonal, as potrf_inv_kernel stores it"""
    M = rng.standard_normal((T, T))
    L = np.linalg.cholesky(M @ M.T / T + 0.5 * np.eye(T))
    return np.tril(sl.solve_triangular(L, np.eye(T), lower=True))


@gpu
def test_trsm(h):
    """X = A Linv^T for three row tiles: |X - A Linv^T| <= gamma_T |A||Linv|^T"""
    rng = np.random.default_rng(11)
    A = rng.standard_normal((3, T, T)) * np.array([2.0 ** -30, 1.0, 2.0 ** 30])[:, None, None]
    A[1] *= np.exp(rng.uniform(-5, 5, T))[:, None]   # rows of different magnitude
    Linv = _tile_inverse(rng)
    got = _f64(h("trsm", np.array([3], np.int32), A, Linv)[0], 3, T, T)
    Al, Ll = A.astype(LD), Linv.astype(LD)
    _within("trsm", np.abs(got - Al @ Ll.T), _bound(gamma(T), np.abs(Al) @ np.abs(Ll).T, T))


@gpu
def test_chain_solve(h):
    """chain_gemm_kernel<0>: C = C Q^T in place, |X - C Q^T| <= gamma_T |C||Q|^T"""
    rng = np.random.default_rng(12)
    C = rng.standard_normal((T, T)) * np.exp(rng.uniform(-5, 5, T))[:, None]
    Q = _tile_inverse(rng)
    got = _f64(h("chain0", C, Q)[0], T, T)
    Cl, Ql = C.astype(LD), Q.astype(LD)
    _within("chain0", np.abs(got - Cl @ Ql.T), _bound(gamma(T), np.abs(Cl) @ np.abs(Ql).T, T))


@gpu
def test_chain_update(h):
    """chain_gemm_kernel<1>: C -= P P^T on the lower triangle, |err| <= gamma_{T+1} (|C| + |P||P|^T); the strictly upper
    triangle is bitwise unchanged"""
    rng = np.random.default_rng(13)
    C = rng.standard_normal((T, T)) * 4.0
    P = rng.standard_normal((T, T)) * np.exp(rng.uniform(-3, 3, T))[:, None]
    got = _f64(h("chain1", C, P)[0], T, T)
    Cl, Pl = C.astype(LD), P.astype(LD)
    low = ~STRICT_UPPER
    _within("chain1", np.abs(got - (Cl - Pl @ Pl.T))[low], _bound(gamma(T + 1), np.abs(Cl) + np.abs(Pl) @ np.abs(Pl).T, T + 1)[low])
    _same_bits("chain1 upper triangle", got[STRICT_UPPER], C[STRICT_UPPER])


# ---------------------------------------------------------------- diagonal tile (potrf_inv_kernel)
def _spd_tiles():
    rng = np.random.default_rng(21)
    M = rng.standard_normal((T, T))
    A0 = M @ M.T / T + 0.5 * np.eye(T)
    d = np.exp(rng.permutation(np.linspace(np.log(1e-4), np.log(1e4), T)))   # the unit mix of the BA system
    Q, _ = np.linalg.qr(rng.standard_normal((T, T)))
    tiles = {"random": A0, "graded": d[:, None] * A0 * d[None, :], "cond1e10": (Q * np.logspace(0, -10, T)) @ Q.T,
             "scaled_up": A0 * 2.0 ** 400, "scaled_down": A0 * 2.0 ** -400}
    return {k: _sym(v) for k, v in tiles.items()}


def _with_upper_garbage(A, rng):
    """the tile as the kernel gets it: lower triangle of A, distinct values above the diagonal that it must not read"""
    return np.where(STRICT_UPPER, rng.standard_normal((T, T)) * 1e3, A)


def _potrf_failures():
    """tiles whose factorisation must set the flag"""
    rng = np.random.default_rng(22)
    M = rng.standard_normal((T, T))
    A0 = _sym(M @ M.T / T + 0.5 * np.eye(T))
    L0 = np.linalg.cholesky(A0)
    out = {}
    for p in [0, 1, 15, 16, 17, 64, 126, 127]:   # A = L0 L0^T - (L0[p,p]^2 + delta) e_p e_p^T: pivot p is -delta
        A = A0.copy()
        A[p, p] -= 1.5 * L0[p, p] ** 2
        out[f"negative_{p}"] = A
    for p in [0, 17, 127]:                       # diagonal matrix: every operation on the way to pivot p is exact
        A = np.diag(np.exp2(rng.integers(-4, 5, T)).astype(np.float64))
        A[p, p] = 0.0
        out[f"zero_{p}"] = A
    for r, c in [(100, 37), (127, 0)]:
        A = A0.copy()
        A[r, c] = np.nan
        out[f"nan_{r}_{c}"] = A
    return out


def _potrf_run(h, tiles):
    rng = np.random.default_rng(23)
    names = list(tiles)
    inp = np.stack([_with_upper_garbage(tiles[k], rng) for k in names])
    o = h("potrf", inp)
    L, X = _f64(o[0], len(names), T, T), _f64(o[1], len(names), T, T)
    flags = np.frombuffer(o[2], np.int32)
    return {k: (inp[q], L[q], X[q], int(flags[q])) for q, k in enumerate(names)}


@gpu
@pytest.mark.parametrize("kind", ["random", "graded", "cond1e10", "scaled_up", "scaled_down"])
def test_potrf_factor(h, kind):
    """flag 0, diag(L) > 0, |A - L L^T| <= gamma_{T+16} |L||L^T| on the lower triangle (Higham Thm 10.3 with slack for the
    1-ulp rsqrt and the division done as two multiplications); the upper triangle of the tile is bitwise unchanged"""
    A = _spd_tiles()[kind]
    inp, out, _, flag = h.cached("potrf", lambda: _potrf_run(h, _spd_tiles()))[kind]
    assert flag == 0
    L = np.tril(out)
    assert (np.diag(L) > 0).all()
    Ll = L.astype(LD)
    low = ~STRICT_UPPER
    _within(f"potrf L {kind}", np.abs(A.astype(LD) - Ll @ Ll.T)[low], _bound(gamma(T + 16), np.abs(Ll) @ np.abs(Ll).T, T + 1)[low])
    _same_bits(f"potrf upper triangle {kind}", out[STRICT_UPPER], inp[STRICT_UPPER])


@gpu
@pytest.mark.parametrize("kind", ["random", "graded", "cond1e10", "scaled_up", "scaled_down"])
def test_potrf_inverse(h, kind):
    """the stored inverse X has exact +0.0 above the diagonal (fwd_kernel / bwd_kernel read the whole tile; the output
    buffer held NaN before the launch, so the kernel must write these zeros) and
    |X L - I| <= 4 T u |X||L| (the left residual: the recursive doubling forms X21 = -X22 (L21 X11))"""
    _, out, X, _ = h.cached("potrf", lambda: _potrf_run(h, _spd_tiles()))[kind]
    assert (X[STRICT_UPPER].view(np.uint64) == 0).all(), "tile inverse not exactly +0.0 above the diagonal"
    Xl, Ll = X.astype(LD), np.tril(out).astype(LD)
    _within(f"potrf inverse {kind}", np.abs(Xl @ Ll - np.eye(T, dtype=LD)), _bound(4 * T * U, np.abs(Xl) @ np.abs(Ll), T + 1))


@gpu
@pytest.mark.parametrize("case", list(_potrf_failures()))
def test_potrf_flags_failure(h, case):
    _, _, _, flag = h.cached("potrf_fail", lambda: _potrf_run(h, _potrf_failures()))[case]
    assert flag == 1


# ---------------------------------------------------------------- whole factor + solve (factor(), solve())
def _pattern(name, nt):
    """tile mask (lower, bool) and column groups (None = main sequence only)"""
    i, j = np.indices((nt, nt))
    if name == "dense":
        return np.tril(np.ones((nt, nt), bool)), None
    if name == "banded":
        return (i - j >= 0) & (i - j <= 2), None
    if name == "arrow":
        m = np.eye(nt, dtype=bool)
        m[-2:, :] = True
        return np.tril(m), None
    if name == "gaps":   # (k+1, k) missing at block ends (k = 3; L(4,3) = 0), column 1 without rows (test_tile_plan)
        assert nt == 10
        m = np.eye(nt, dtype=bool)
        for a, b in [(2, 0), (3, 0), (5, 3), (6, 3), (6, 5), (8, 5), (9, 8), (9, 6), (7, 4)]:
            m[a, b] = True
        L = _structure(m)
        assert not L[1, 0] and not L[4, 3] and not L[8, 7]
        return m, None
    if name.startswith("random"):
        return _random_mask(np.random.default_rng(int(name[-1])), nt, 0.3), None
    if name == "ba":     # IMU-chain-like groups first: each a band coupled to its own pose tiles only; then the poses
        assert nt == 10
        sizes, links = [2, 2, 1], [[5], [6, 7], [8]]
        m, group, c = np.eye(nt, dtype=bool), [-1] * nt, 0
        for g, s in enumerate(sizes):
            for t in range(c, c + s):
                group[t] = g
                if t > c:
                    m[t, t - 1] = True
                m[links[g], t] = True
            c += s
        m[c:, c:] |= np.tril(np.random.default_rng(4).random((nt - c, nt - c)) < 0.5)
        return m, group
    raise ValueError(name)


def _matrix(mask, n, kind, seed):
    """SPD matrix on the tile pattern: well conditioned (kappa_2 ~ 11), graded (D A D, D over 1e-3..1e3), or kappa_2 = 1e10.
    Returns A and kappa_2 (None for graded: there a normwise forward-error bound says nothing)"""
    rng = np.random.default_rng(seed)
    nt = len(mask)
    A = np.zeros((nt * T, nt * T))
    for a, b in zip(*np.nonzero(np.tril(mask))):
        A[a * T:(a + 1) * T, b * T:(b + 1) * T] = rng.standard_normal((T, T))
    A = _sym(A[:n, :n])
    lam = np.linalg.eigvalsh(A)
    lo = (lam[-1] - lam[0]) * (1e-10 if kind == "cond1e10" else 0.1)
    A[np.diag_indices(n)] += lo - lam[0]
    kappa = (lam[-1] - lam[0] + lo) / lo
    if kind == "graded":
        d = np.exp(rng.permutation(np.linspace(np.log(1e-3), np.log(1e3), n)))
        return _sym(d[:, None] * A * d[None, :]), None
    return A, kappa


PLAN = {"blocked": 0, "group": 1, "width1": 2}


def _factor(h, mask, As, bs, plan="blocked", group=None):
    """factor + solve each (A, b) in one process; per run: dense lower L (nt T x nt T), packed L, tile_of, inverses, x, flag"""
    nt, n = len(mask), len(As[0])
    grp = np.asarray(group if group is not None else [-1] * nt, np.int32)
    o = h("factor", np.array([nt, n, PLAN[plan], len(As)], np.int32), np.tril(mask).astype(np.int32), grp,
          np.stack(As), np.stack(bs))
    runs = []
    for r in range(len(As)):
        Lp, tile_of, linv, x, flag = o[5 * r:5 * r + 5]
        Lp = _f64(Lp, -1, T, T)
        tile_of = np.frombuffer(tile_of, np.int32).reshape(nt, nt)
        L = np.zeros((nt * T, nt * T))
        for a in range(nt):
            for b in range(a + 1):
                if tile_of[a, b] >= 0:
                    L[a * T:(a + 1) * T, b * T:(b + 1) * T] = Lp[tile_of[a, b]]
        runs.append(dict(L=np.tril(L), Lp=Lp, tile_of=tile_of, linv=_f64(linv, nt, T, T), x=_f64(x),
                         flag=int(np.frombuffer(flag, np.int32)[0])))
    return runs


FACTOR_CASES = [("dense", nt, T * nt - pad, "well") for nt in [1, 2, 4, 5, 8, 9] for pad in [0, 17]] + \
    [("dense", 5, 5 * T - 17, kind) for kind in ["graded", "cond1e10"]] + \
    [(p, 10 if p in ("gaps", "ba") else 9, (10 if p in ("gaps", "ba") else 9) * T - 17, kind)
     for p in ["banded", "arrow", "gaps", "random0", "random1", "ba"] for kind in ["well", "graded", "cond1e10"]]
FACTOR_IDS = [f"{p}-nt{nt}-n{n}-{kind}" for p, nt, n, kind in FACTOR_CASES]


def _factor_case(h, case):
    def run():
        p, nt, n, kind = case
        mask, group = _pattern(p, nt)
        A, kappa = _matrix(mask, n, kind, zlib.crc32(repr(case).encode()))
        xs = np.random.default_rng(7).standard_normal(n)
        b = (A.astype(LD) @ xs.astype(LD)).astype(np.float64)
        runs = {"blocked": _factor(h, mask, [A, A], [b, b]),
                "width1": _factor(h, mask, [A], [b], "width1"),
                "one_group": _factor(h, mask, [A], [b], "group", [0] * nt)}
        if group is not None:
            runs["groups"] = _factor(h, mask, [A], [b], "group", group)
        return dict(A=A, kappa=kappa, xs=xs, runs=runs, n=n, nt=nt)
    return h.cached(("factor", case), run)


@gpu
@pytest.mark.parametrize("case", FACTOR_CASES, ids=FACTOR_IDS)
def test_factor_schedules_bit_identical(h, case):
    """L, every tile inverse and x are bitwise the same under the blocked plan, a second factorisation in the same process,
    the width-1 plan (one-rank owner map), every column in one column group (all work on the group streams) and, for the
    BA-like pattern, its own column groups.  The quadrant above the diagonal of every diagonal tile stays zero, and every
    tile inverse is written with exact +0.0 above its diagonal (its buffer held NaN before the factorisation)."""
    c = _factor_case(h, case)
    ref = c["runs"]["blocked"][0]
    others = [("blocked, second run", c["runs"]["blocked"][1])] + \
        [(k, v[0]) for k, v in c["runs"].items() if k != "blocked"]
    for name, r in [("blocked", ref)] + others:
        assert r["flag"] == 0, name
        for k in range(c["nt"]):
            assert (r["Lp"][r["tile_of"][k, k]][UPPER_Q] == 0).all(), f"{name}: upper quadrant of diagonal tile {k} written"
            assert (r["linv"][k][STRICT_UPPER].view(np.uint64) == 0).all(), \
                f"{name}: tile inverse {k} not exactly +0.0 above the diagonal"
    for name, r in others:
        _same_bits(f"L ({name})", r["L"], ref["L"])
        _same_bits(f"tile inverses ({name})", r["linv"], ref["linv"])
        _same_bits(f"x ({name})", r["x"], ref["x"])


@gpu
@pytest.mark.parametrize("case", FACTOR_CASES, ids=FACTOR_IDS)
def test_factor_backward_error(h, case):
    """|A - L L^T| <= gamma_{n+16} |L||L^T| over the whole lower triangle, fill tiles included.  The residual is formed in
    float64, so its own rounding, gamma_{n+1} |L||L^T| + u |A|, is added to the bound (|L||L^T| itself is computed in
    float64 and divided by 1 - gamma_n to bound the exact one from above)"""
    c = _factor_case(h, case)
    A, n = c["A"], c["n"]
    L = c["runs"]["blocked"][0]["L"][:n, :n]
    assert (np.diag(L) > 0).all()
    low = np.tril(np.ones((n, n), bool))
    R = np.abs(A - L @ L.T)[low]
    mag = (np.abs(L) @ np.abs(L).T)[low].astype(LD) / (1 - gamma(n))
    _within(f"factor L {FACTOR_IDS[FACTOR_CASES.index(case)]}", R,
            _bound(gamma(n + 16) + gamma(n + 1), mag, 0) + _bound(U, np.abs(A)[low], 0))


@gpu
@pytest.mark.parametrize("case", [c for c in FACTOR_CASES if c[3] != "graded"],
                         ids=[i for c, i in zip(FACTOR_CASES, FACTOR_IDS) if c[3] != "graded"])
def test_factor_forward_error(h, case):
    """manufactured solution: b = A x* in longdouble, rounded; ||x - x*||_inf / ||x*||_inf <= 4 n u kappa_2(A)"""
    c = _factor_case(h, case)
    n, xs = c["n"], c["xs"]
    x = c["runs"]["blocked"][0]["x"]
    err = np.abs(x[:n].astype(LD) - xs).max() / np.abs(xs).max()
    _within(f"factor x {FACTOR_IDS[FACTOR_CASES.index(case)]}", err, _bound(4 * n * U, LD(c["kappa"]), 0))


# name: (pattern, nt, n, plan, failing row)
FAIL_CASES = {
    "tile_column_0": ("dense", 4, 4 * T, "blocked", 5),
    "block_last_column": ("dense", 9, 9 * T, "blocked", 3 * T + 40),
    "block_middle_column": ("dense", 9, 9 * T, "blocked", 5 * T + 77),
    "column_group": ("ba", 10, 10 * T - 17, "groups", T + 3),
    "padded_last_row": ("dense", 5, 5 * T - 17, "blocked", 5 * T - 18),
}


@gpu
@pytest.mark.parametrize("case", list(FAIL_CASES))
def test_factor_flags_failure(h, case):
    """a negative pivot (A[p,p] lowered by 1.5 L[p,p]^2) sets the flag; the next, SPD, input factored in the same process
    clears it and is solved"""
    p, nt, n, plan, row = FAIL_CASES[case]
    mask, group = _pattern(p, nt)
    A, kappa = _matrix(mask, n, "well", zlib.crc32(case.encode()))
    L0 = np.linalg.cholesky(A)
    bad = A.copy()
    bad[row, row] -= 1.5 * L0[row, row] ** 2
    xs = np.random.default_rng(8).standard_normal(n)
    b = (A.astype(LD) @ xs.astype(LD)).astype(np.float64)
    runs = _factor(h, mask, [bad, A], [b, b], "group" if plan == "groups" else plan, group if plan == "groups" else None)
    assert runs[0]["flag"] == 1, "non-positive pivot not flagged"
    assert runs[1]["flag"] == 0, "flag not reset by the next factorisation"
    err = np.abs(runs[1]["x"][:n].astype(LD) - xs).max() / np.abs(xs).max()
    _within(f"factor x after a failure {case}", err, _bound(4 * n * U, LD(kappa), 0))
