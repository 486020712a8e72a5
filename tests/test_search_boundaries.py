"""SearchByProjection (K10b) and SearchBySE3 (K10) at their rounding boundaries.

Builders place landmarks and keypoints within a few ulps of each decision the searches take, on both sides, by stepping
one input with np.nextafter and keeping the inputs whose value in the oracle's own operation order (plain float64 / float32
scalars, which never fuse) lands where intended.  Each builder checks itself on the CPU: every boundary has cases on both
sides, and each image bound and float-rounding midpoint has a case where a fused (fx * xd + cx as one FMA, computed exactly) or reciprocal
(x = X * (1 / Z)) evaluation lands on the other side from the plain one, so the scenes tell the orders apart.

SearchByProjection's decisions: the image bounds, the pc.z / 1e-10 validity limit, d3 against min_dist / max_dist, the
viewing cone, PredictScale at ratio = 1.2^n, the float rounding of u and v at midpoints and ties, the cell range's floor / ceil
on cell edges and its clamps at column 0 / 63 and row 0 / 47, the keypoint radius test at levels 0, 2 and 3, the octave gate,
Hamming ties at desc_th_low and the first strict minimum.  SearchBySE3's, in both directions: the image bounds, pc.z < 0,
<= th_low from 1 to 2 and < th_low from 2 to 1, PredictScale at 1.2^n, and the agreement rule match2[i] == i.

The GPU must equal the C oracle bit for bit on these scenes.  That is pinned for the pinhole and unified models with radtan
distortion only: the equidistant and FOV models call atan / tan, which CUDA does not round correctly, so they differ from the
host libm in the last bits at a constructed boundary; they are covered by random-scene parity.
"""
import functools
import math
import os
import shutil
import subprocess
from fractions import Fraction

import numpy as np
import pytest

from covins_b200 import placerec as PR, synth
from covins_b200.synth_map import EUROC_DIST, EUROC_INTR
from oracle import geom as og
from test_geom import _py_grid, _py_rt, _py_search_by_projection, _view, py_predict_scale, py_project3

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W, H = 752, 480
PINHOLE = dict(intr=EUROC_INTR, dist=EUROC_DIST, cam_model=0, dist_model=0, xi=0.0)
UNIFIED = dict(intr=EUROC_INTR, dist=np.array([-0.21, 0.04, 0.0011, -0.0007]), cam_model=1, dist_model=0, xi=0.8)
ALL_MODELS = [dict(intr=EUROC_INTR, dist=d, cam_model=c, dist_model=m, xi=xi)
              for c, xi in ((0, 0.0), (1, 0.9)) for m, d in ((0, EUROC_DIST), (1, np.array([-0.013, 0.02, -0.012, 0.002])), (2, np.array([0.9, 0, 0, 0])))]


def _fma(a, b, c):
    return float(Fraction(a) * Fraction(b) + Fraction(c))       # exact, then one rounding


def _project_alt(cam, pc):
    """project3 as a contracting compiler may evaluate it: x = X * (1 / den) and u = fma(fx, xd, cx), v = fma(fy, yd, cy)"""
    intr, d = [float(v) for v in cam["intr"]], [float(v) for v in cam["dist"]]
    den = pc[2] if cam["cam_model"] == 0 else pc[2] + float(cam["xi"]) * math.sqrt(pc[0] * pc[0] + pc[1] * pc[1] + pc[2] * pc[2])
    if not den > 1e-10:
        return None
    iz = 1.0 / den
    x, y = pc[0] * iz, pc[1] * iz
    r2 = x * x + y * y
    rad = 1.0 + d[0] * r2 + d[1] * r2 * r2
    xd = x * rad + 2.0 * d[2] * x * y + d[3] * (r2 + 2.0 * x * x)
    yd = y * rad + d[2] * (r2 + 2.0 * y * y) + 2.0 * d[3] * x * y
    return _fma(intr[0], xd, intr[2]), _fma(intr[1], yd, intr[3])


def _steps(x, k):
    """x moved k ulps (k < 0: down)"""
    for _ in range(abs(k)):
        x = float(np.nextafter(x, math.inf if k > 0 else -math.inf))
    return x


class Scene:
    """one keyframe and a list of candidate landmarks; every landmark has its own keypoint (descriptor 10 bits away, the other
    landmarks ~128 bits away), so its action is 1 iff it passes every gate"""

    def __init__(self, seed, cam, Tcw):
        self.rng = np.random.default_rng(seed)
        self.cam, self.Tcw = cam, np.asarray(Tcw, np.float64)
        T = self.Tcw.reshape(16).tolist()
        self.T = T
        self.Ow = [-(T[r] * T[3] + T[4 + r] * T[7] + T[8 + r] * T[11]) for r in range(3)]
        self.kp, self.oct, self.kdesc, self.lm = [], [], [], []
        self.cases = {}                     # decision -> list of (landmark, side of the boundary, found: action 1 expected)
        self.cells = {}                     # keypoint -> grid cell it is filed in, where that is not its own

    def desc(self):
        return self.rng.integers(0, 256, 32, dtype=np.uint8)

    def add_kp(self, x, y, desc, octave=0, cell=None):
        self.kp.append((x, y)); self.oct.append(octave); self.kdesc.append(desc)
        if cell is not None:
            self.cells[len(self.kp) - 1] = cell
        return len(self.kp) - 1

    def near(self, desc, flips=10):
        d = np.unpackbits(desc.copy())
        d[self.rng.choice(256, flips, replace=False)] ^= 1
        return np.packbits(d)

    def add_lm(self, pw, decision=None, side=None, kp_xy=None, normal=None, min_dist=0.0, max_dist=1e9, max_distance=None, octave=0,
               desc=None, flips=10, cell=None, found=None):
        """a landmark at pw and, at kp_xy (default: its projection), a keypoint 'flips' bits away (filed in grid cell `cell` if
        given); found = whether the landmark takes that keypoint (default: side)"""
        pw = [float(v) for v in pw]
        PO = [pw[r] - self.Ow[r] for r in range(3)]
        d3 = math.sqrt(PO[0] * PO[0] + PO[1] * PO[1] + PO[2] * PO[2])
        if normal is None:
            normal = [PO[r] / d3 for r in range(3)]
        if max_distance is None:
            max_distance = float(np.float32(d3))                  # ratio 1: level 0
        desc = self.desc() if desc is None else desc
        if kp_xy is None:
            u, v = py_project3(self.cam, _py_rt(self.T, pw))
            kp_xy = (min(max(u, 3.0), 744.0), min(max(v, 3.0), 473.0))
        if flips is not None:
            self.add_kp(kp_xy[0], kp_xy[1], self.near(desc, flips), octave, cell)
        self.lm.append(dict(pos=pw, normal=list(normal), min_dist=min_dist, max_dist=max_dist, max_distance=max_distance, desc=desc))
        i = len(self.lm) - 1
        if decision is not None:
            self.cases.setdefault(decision, []).append((i, side, side if found is None else found))
        return i

    def pw_of(self, pc):
        """world point of camera point pc (float64 numpy; callers step the result and recompute)"""
        R = self.Tcw[:3, :3]; t = self.Tcw[:3, 3]
        return R.T @ (np.asarray(pc, np.float64) - t)

    def arrays(self):
        n, m = len(self.kp), len(self.lm)
        view = dict(kp=np.asarray(self.kp, np.float32).reshape(n, 2), octave=np.asarray(self.oct, np.float32), desc=np.stack(self.kdesc),
                    lm_valid=np.zeros(n, np.uint8), lm_pos=np.zeros((n, 3)), lm_maxdist=np.ones(n), lm_desc=np.zeros((n, 32), np.uint8),
                    K=np.eye(3), Tcw=self.Tcw, img_bounds=np.array([0.0, W, 0.0, H]))
        lms = {k: np.array([l[k] for l in self.lm]) for k in ("pos", "normal", "min_dist", "max_dist", "max_distance", "desc")}
        lms["valid"] = np.ones(m, np.uint8); lms["feat_idx"] = np.full(m, -1, np.int32)
        if self.cells:
            grid = {c: [k for k in ks if k not in self.cells] for c, ks in _py_grid(view["kp"]).items()}
            for k, c in self.cells.items():
                grid.setdefault(c, []).append(k)
            view["grid"] = {c: sorted(ks) for c, ks in grid.items()}
        return view, np.full(n, -1, np.int32), self.Tcw, self.cam, lms, np.zeros(n, np.uint8)


def _kfview(view):
    """KfView of a scene's keyframe, with the scene's own grid filing if it has one"""
    kv = _view(view)
    if "grid" in view:
        ptr, idx = [0], []
        for c in range(64 * 48):
            idx += view["grid"].get((c // 48, c % 48), [])
            ptr.append(len(idx))
        kv.a["grid_ptr"] = np.asarray(ptr, np.int32); kv.a["grid_idx"] = np.asarray(idx, np.int32)
    return kv


def _pw_at(S, u, v, z=6.0):
    """a world point whose projection (oracle order) is (u, v) to well below a float ulp: Newton on the camera-frame X, Y"""
    pc = [(u - float(S.cam["intr"][2])) / float(S.cam["intr"][0]) * z, (v - float(S.cam["intr"][3])) / float(S.cam["intr"][1]) * z, z]
    for _ in range(40):
        f = py_project3(S.cam, pc); h = 1e-7
        fx = py_project3(S.cam, [pc[0] + h, pc[1], z]); fy = py_project3(S.cam, [pc[0], pc[1] + h, z])
        J = np.array([[fx[0] - f[0], fy[0] - f[0]], [fx[1] - f[1], fy[1] - f[1]]]) / h
        d = np.linalg.solve(J, [u - f[0], v - f[1]])
        pc = [pc[0] + d[0], pc[1] + d[1], z]
    return S.pw_of(pc).tolist()


def _pose(rng):
    T = np.eye(4); T[:3, :3] = synth._rot(rng.normal(0, 0.1, 3)); T[:3, 3] = rng.normal(0, 0.2, 3)
    return T


def _threshold_cases(S, axis, bound, other, passes, name, kp_xy, k=4, window=400):
    """landmarks whose projection's coordinate `axis` (plain order) takes the k values nearest `bound` on each side, plus up to
    three inputs where the fused / reciprocal evaluation decides passes() the other way (the row `other` of the other
    coordinate is moved until one exists); kp_xy(pw) places each landmark's keypoint → number of such inputs"""
    cam = S.cam
    z = 6.0
    for t in range(16):
        pc = [0.0, 0.0, z]
        pc[1 - axis] = (other + 5.0 * t - float(cam["intr"][3 - axis])) / float(cam["intr"][1 - axis]) * z
        lo, hi = -40.0 * z, 40.0 * z                            # bisection on the camera-frame coordinate for coord == bound
        for _ in range(200):
            mid = 0.5 * (lo + hi); pc[axis] = mid
            (lo, hi) = (mid, hi) if py_project3(cam, pc)[axis] < bound else (lo, mid)
        pc[axis] = lo
        pw0 = S.pw_of(pc)
        seen = {}
        for s in range(-window, window + 1):
            pw = pw0.copy(); pw[axis] = _steps(float(pw0[axis]), s)
            pcs = _py_rt(S.T, pw.tolist())
            val = py_project3(cam, pcs)[axis]
            alt = _project_alt(cam, pcs)[axis]
            seen.setdefault(val, []).append((pw, passes(alt) != passes(val)))
        flips = [(v, pw) for v in seen for pw, f in seen[v] if f]
        if flips:
            break
    vals = sorted(seen)
    below = [v for v in vals if v < bound][-k:]; above = [v for v in vals if v >= bound][:k]
    for v, pw in [(v, seen[v][0][0]) for v in below + above] + flips[:3]:
        S.add_lm(pw, name, passes(v), kp_xy=kp_xy(pw))
    return len(flips)


def _image_bound_cases(S, axis, bound, other):
    """the image bound `bound` of coordinate `axis` (>= on the low side, < on the high side); the keypoint 7 px inside"""
    name = f"image {'uv'[axis]} {'>=' if bound == 0.0 else '<'} {bound}"
    passes = (lambda v: v >= bound) if bound == 0.0 else (lambda v: v < bound)

    def kp_xy(pw):
        xy = [0.0, 0.0]; xy[axis] = bound + (7.0 if bound == 0.0 else -7.0)
        xy[1 - axis] = py_project3(S.cam, _py_rt(S.T, pw.tolist()))[1 - axis]
        return tuple(xy)
    return name, _threshold_cases(S, axis, bound, other, passes, name, kp_xy)


def _midpoint_cases(S, axis, f_lo, other, th=10.0):
    """the float rounding of u (axis 0) or v (axis 1) at the midpoint M of the floats f_lo < f_hi, M itself included (a tie: to
    the even one).  The keypoint sits th below f_lo on that axis, on the float row of the other coordinate: inside the radius
    of t = f_lo, outside that of t = f_hi, so the landmark takes it iff its coordinate rounds down"""
    f_lo = np.float32(f_lo)
    f_hi = np.nextafter(f_lo, np.float32(np.inf))
    M = (float(f_lo) + float(f_hi)) / 2
    even = "even" if (f_lo.view(np.int32) & 1) == 0 else "odd"
    name = f"float rounding of {'uv'[axis]} at a midpoint ({even} below)"

    def kp_xy(pw):
        xy = [0.0, 0.0]; xy[axis] = float(f_lo - np.float32(th))
        xy[1 - axis] = float(np.float32(py_project3(S.cam, _py_rt(S.T, pw.tolist()))[1 - axis]))
        return tuple(xy)
    return name, _threshold_cases(S, axis, M, other, lambda v: np.float32(v) == f_lo, name, kp_xy)


def projection_boundary_scene(cam, seed=0):
    """K10b boundary scene for a pinhole or unified radtan camera → (scene, arrays, search kwargs, {decision: n fused flips})"""
    rng = np.random.default_rng(seed)
    S = Scene(seed, cam, _pose(rng))
    flips = {}
    # the four image bounds (>= on the low side, < on the high side)
    for axis, bound, other in ((0, 0.0, 240.0), (0, float(W), 120.0), (1, 0.0, 200.0), (1, float(H), 560.0)):
        name, nf = _image_bound_cases(S, axis, bound, other)
        flips[name] = nf
    # the float rounding of u and v at midpoints, with an even and an odd float below the midpoint
    for axis, f_lo, other in ((0, 300.25, 330.0), (0, float(np.nextafter(np.float32(420.5), np.float32(1e9))), 150.0), (1, 260.125, 520.0),
                              (1, float(np.nextafter(np.float32(180.75), np.float32(1e9))), 200.0)):
        name, nf = _midpoint_cases(S, axis, f_lo, other)
        flips[name] = nf
    # den > 1e-10 (pc.z < 0 first): a point on the optical axis, in a camera-frame scene of its own below
    # d3 against min_dist / max_dist and the viewing cone, at a point in the middle of the image
    base_pc = [0.4, -0.3, 5.0]
    pw = S.pw_of(base_pc).tolist()
    PO = [pw[r] - S.Ow[r] for r in range(3)]
    d3 = math.sqrt(PO[0] * PO[0] + PO[1] * PO[1] + PO[2] * PO[2])
    for k in (-2, -1, 0, 1, 2):
        md = _steps(d3, k)
        S.add_lm(pw, "d3 < min_dist", not d3 < md, min_dist=md)
        S.add_lm(pw, "d3 > max_dist", not d3 > md, max_dist=md)
    # viewing cone PO.n < 0.5 d3: n tilted until PO.n crosses 0.5 d3 (n need not be unit)
    half = 0.5 * d3
    n0 = [PO[r] / d3 * 0.5 for r in range(3)]
    dot = lambda n: PO[0] * n[0] + PO[1] * n[1] + PO[2] * n[2]
    cone = {}
    for s in range(-400, 401):
        n = list(n0); n[2] = _steps(n0[2], s)
        cone.setdefault(dot(n) - half, n)
    diffs = sorted(cone)
    for dv in [v for v in diffs if v < 0][-3:] + [v for v in diffs if v >= 0][:3]:
        S.add_lm(pw, "PO.n < 0.5 d3", dv >= 0, normal=cone[dv])
    return S, flips


def pz_scene(cam, seed=1):
    """pc.z < 0 and the 1e-10 validity limit: points on the optical axis of an identity pose (pc = pw exactly)"""
    S = Scene(seed, cam, np.eye(4))
    lim = 1e-10 if cam["cam_model"] == 0 else 1e-10 / (1.0 + float(cam["xi"]))
    zs = [-1e-300, -0.0, 0.0] + [_steps(lim, k) for k in range(-3, 4)]
    for z in zs:
        den = z if cam["cam_model"] == 0 else z + float(cam["xi"]) * math.sqrt(z * z)
        ok = not z < 0 and den > 1e-10
        S.add_lm([0.0, 0.0, z], "pc.z < 0 / den > 1e-10", ok, kp_xy=(float(cam["intr"][2]) + 2.0, float(cam["intr"][3])),
                 normal=[0.0, 0.0, 1.0], max_distance=1.0)
    return S


def scale_scene(cam, seed=2, sf=1.2, num_octaves=8):
    """PredictScale at ratio = sf^n (n-fold product and neighbours) and the octave gate: the landmark's keypoint sits at octave
    n + 1, so it is found iff the level is n + 1 or n + 2"""
    rng = np.random.default_rng(seed)
    S = Scene(seed, cam, _pose(rng))
    col = 0
    for n in range(1, 6):
        p = 1.0
        for _ in range(n):
            p = p * sf
        for k in (-1, 0, 1):
            target = _steps(p, k)
            for j in range(200):                                   # a depth at which some max distance gives the ratio exactly
                pw = S.pw_of([-2.0 + 0.45 * col, -1.2 + 0.5 * (col % 5), 6.0 + 1e-4 * j]).tolist()
                PO = [pw[r] - S.Ow[r] for r in range(3)]
                d3 = math.sqrt(PO[0] * PO[0] + PO[1] * PO[1] + PO[2] * PO[2])
                md = _max_distance_for(target, d3)
                if md is not None:
                    break
            col += 1
            lvl = py_predict_scale(md, d3, sf, num_octaves)
            S.add_lm(pw, f"level at {sf}^{n}", lvl in (n + 1, n + 2), max_distance=md, octave=n + 1)
    return S, dict(num_octaves=num_octaves, scale_factor=sf)


def _max_distance_for(target, d3):
    """a max distance whose ratio to float(d3) is exactly target, or None"""
    cur = float(np.float32(d3))
    md = target * cur
    for s in range(-8, 9):
        if _steps(md, s) / cur == target:
            return _steps(md, s)
    return None


def radius_scene(cam, seed=3, th=10.0):
    """sqrtf(dx^2 + dy^2) <= radius at +-1 float ulp, the octave gate, Hamming ties at desc_th_low and first-strict-minimum ties
    in grid order"""
    rng = np.random.default_rng(seed)
    S = Scene(seed, cam, _pose(rng))
    for j, k in enumerate((-2, -1, 0, 1, 2)):
        pw = S.pw_of([-1.5 + 0.7 * j, 0.8, 5.0]).tolist()
        u, v = py_project3(cam, _py_rt(S.T, pw))
        tx, ty = np.float32(u), np.float32(v)
        x = np.float32(tx + np.float32(th))                        # keypoint k float ulps around tx + radius, same row
        x = np.nextafter(x, np.float32(np.inf if k > 0 else -np.inf)) if k else x
        for _ in range(abs(k) - 1):
            x = np.nextafter(x, np.float32(np.inf if k > 0 else -np.inf))
        dx = np.float32(x - tx)
        nrm = float(np.sqrt(np.float32(dx * dx)))
        S.add_lm(pw, "|kp - t| <= radius", nrm <= th, kp_xy=(float(x), float(ty)))
    for j, o in enumerate((-1, 0, 1, 2)):                          # octave gate at level 0: octaves -1 and 0 pass
        pw = S.pw_of([-1.5 + 0.7 * j, -0.9, 5.0]).tolist()
        S.add_lm(pw, "octave in [level - 1, level]", o in (-1, 0), octave=o)
    th_low = 50
    for j, f in enumerate((th_low - 1, th_low, th_low + 1)):       # bestDist <= desc_th_low
        pw = S.pw_of([-1.5 + 0.7 * j, 0.0, 5.0]).tolist()
        S.add_lm(pw, "bestDist <= th_low", f <= th_low, flips=f)
    # first strict minimum: two keypoints at equal distance, one cell apart in x; the lower grid cell wins
    pw = S.pw_of([1.6, 0.0, 5.0]).tolist()
    u, v = py_project3(cam, _py_rt(S.T, pw))
    d = S.desc()
    i = S.add_lm(pw, None, desc=d, kp_xy=(u + 6.0, v), flips=12)
    S.first_min = (i, S.add_kp(u - 6.0, v, S.near(d, 12)))       # 12 px apart: always in different cells; the left one wins
    S.cases["first strict minimum"] = [(i, True, True)]
    return S


def grid_scene(cam, seed=4, th=10.0):
    """the search's cell range: floor((t - r) / cell width) and ceil((t + r) / cell width) with (t -+ r) / width one float step
    below, at and above an integer, in columns and rows, and the clamps at column 0 / 63 and row 0 / 47 (raw index just outside
    and just inside).  A keypoint inside the radius is filed in the cell the range does or does not reach: the reference's own
    filing (round to the nearest cell) keeps every keypoint inside the radius within reach, so only a scene's own filing shows
    these decisions in the output."""
    S = Scene(seed, cam, _pose(np.random.default_rng(seed)))
    w_inv, h_inv = 64 / float(W), 48 / float(H)
    cw, ch = W / 64, H / 48                                        # 11.75 and 10 px: exact
    rows = iter(range(60, 440, 22))
    for axis, k, inv, width in ((0, 21, w_inv, cw), (0, 40, w_inv, cw), (1, 14, h_inv, ch), (1, 30, h_inv, ch)):
        for low in (True, False):                                  # floor of the low end / ceil of the high end
            edge = np.float32(k * width + (th if low else -th))
            for step in (-1, 0, 1):
                t = np.float32(edge)
                for _ in range(abs(step)):
                    t = np.nextafter(t, np.float32(np.inf if step > 0 else -np.inf))
                q = (float(t) - th) * inv if low else (float(t) + th) * inv
                reach = math.floor(q) <= k - 1 if low else math.ceil(q) >= k + 1
                other = float(next(rows)) if axis == 0 else 150.0 + 40.0 * (step + 2) + (0.0 if low else 300.0)
                uv = [0.0, 0.0]; uv[axis] = float(t); uv[1 - axis] = other
                tt = [np.float32(c) for c in uv]
                xy = [float(c) for c in tt]; xy[axis] += -5.0 if low else 5.0
                cell = [int(math.floor(c * i + 0.5)) for c, i in zip(xy, (w_inv, h_inv))]
                cell[axis] = k - 1 if low else k + 1
                dec = f"{'floor' if low else 'ceil'} on a {'column' if axis == 0 else 'row'} edge"
                S.add_lm(_pw_at(S, *uv), dec, reach, kp_xy=tuple(xy), cell=tuple(cell))
    for j, (axis, t, lim) in enumerate(((0, 4.0, 0), (0, 12.0, 0), (0, 748.0, 63), (0, 730.0, 63), (1, 4.0, 0), (1, 12.0, 0), (1, 476.0, 47),
                                        (1, 455.0, 47))):
        uv = [0.0, 0.0]; uv[axis] = t; uv[1 - axis] = 100.0 + 70.0 * (j % 4) if axis == 0 else 60.0 + 90.0 * (j % 4)
        inv = (w_inv, h_inv)[axis]
        raw = math.floor((t - th) * inv) if lim == 0 else math.ceil((t + th) * inv)
        xy = list(uv); xy[axis] += 3.0 if lim == 0 else -3.0
        cell = [int(math.floor(c * i + 0.5)) for c, i in zip(xy, (w_inv, h_inv))]
        cell[axis] = lim
        S.add_lm(_pw_at(S, *uv), f"clamp at {'column' if axis == 0 else 'row'} {lim}", raw < 0 if lim == 0 else raw > lim, kp_xy=tuple(xy),
                 cell=tuple(cell), found=True)
    return S


def radius_level_scene(cam, level, seed=5, sf=1.2):
    """the keypoint test sqrtf(dx^2 + dy^2) <= th * pow(sf, level) at level >= 2, with th chosen so that the radius F is a float
    and the repeated product (th * sf) * sf ... is below it: keypoints at F - 1 ulp, F and F + 1 ulp from t = (1, 240)"""
    p = math.pow(sf, level)
    for m in range(int(14.4 * 2 ** 20), int(14.4 * 2 ** 20) + 4000):
        F = m / 2 ** 20
        for th in (_steps(F / p, s) for s in range(-2, 3)):
            rep = th
            for _ in range(level):
                rep = rep * sf
            if th * p == F and rep < F:
                break
        else:
            continue
        break
    S = Scene(seed, cam, _pose(np.random.default_rng(seed)))
    S.rep_radius = rep
    ratio = (prod_n(sf, level - 1) + prod_n(sf, level)) / 2           # a ratio well inside `level`
    for j, k in enumerate((-1, 0, 1)):
        pw = _pw_at(S, 1.0, 240.0, z=5.0 + j)
        PO = [pw[r] - S.Ow[r] for r in range(3)]
        d3 = math.sqrt(PO[0] * PO[0] + PO[1] * PO[1] + PO[2] * PO[2])
        md = ratio * float(np.float32(d3))
        assert py_predict_scale(md, d3, sf, 8) == level
        x = np.float32(1.0) + np.float32(F)
        for _ in range(abs(k)):
            x = np.nextafter(x, np.float32(np.inf if k > 0 else -np.inf))
        nrm = float(np.sqrt(np.float32(np.float32(x - np.float32(1.0)) ** 2)))
        S.add_lm(pw, f"|kp - t| <= th * {sf}^{level}", nrm <= F, kp_xy=(float(x), 240.0), max_distance=md, octave=level,
                 desc=None, flips=10 + j)
        if k == 0:
            S.tell = (nrm <= F) != (nrm <= rep)                        # the repeated product decides this keypoint the other way
    return S, dict(th=th, num_octaves=8, scale_factor=sf)


def _run_oracle(S, **kw):
    args = S.arrays()
    return args, og.search_by_projection(_kfview(args[0]), *args[1:], **kw)


SCENE_NAMES = [f"{c}-{k}" for c in ("pinhole", "unified") for k in ("gates", "pz", "scale", "radius", "grid", "radius-l2", "radius-l3")]


@functools.lru_cache(maxsize=None)
def _scene(name):
    """(scene, search kwargs[, fused flips per decision]) of a boundary scene, built once on first use"""
    cam = PINHOLE if name.startswith("pinhole") else UNIFIED
    kind = name.split("-", 1)[1]
    if kind == "gates":
        S, flips = projection_boundary_scene(cam)
        return S, {}, flips
    if kind == "pz":
        return pz_scene(cam), {}, None
    if kind == "scale":
        return (*scale_scene(cam), None)
    if kind == "radius":
        return radius_scene(cam), {}, None
    if kind == "grid":
        return grid_scene(cam), {}, None
    return (*radius_level_scene(cam, int(kind[-1])), None)


@pytest.mark.parametrize("name", SCENE_NAMES)
def test_projection_boundary_scene_checks_itself(name):
    """every boundary has cases on both sides; the oracle decides each as the builder intended (action 1 iff the landmark takes
    its keypoint) and equals the plain-Python restatement"""
    S, kw, _ = _scene(name)
    args, (a, b, nm) = _run_oracle(S, **kw)
    for dec, cases in S.cases.items():
        if dec != "first strict minimum":
            assert {side for _, side, _ in cases} == {True, False}, dec
        for i, _, found in cases:
            assert (a[i] == 1) == found, (dec, i)
    ra, rb, rnm = _py_search_by_projection(*args, **{("th_low" if k == "desc_th_low" else k): v for k, v in kw.items()})
    assert np.array_equal(a, ra) and np.array_equal(b, rb) and nm == rnm


@pytest.mark.parametrize("cam", ["pinhole", "unified"])
def test_projection_boundaries_tell_fused_from_plain(cam):
    """each image bound and each float-rounding midpoint has a case where the fused / reciprocal evaluation lands on the other
    side; each midpoint family reaches the midpoint itself (a tie); at levels 2 and 3 the repeated product th * sf * ... decides
    the keypoint at the radius the other way"""
    S, _, flips = _scene(f"{cam}-gates")
    assert len(flips) == 8 and all(n >= 1 for n in flips.values()), flips
    for dec, cases in S.cases.items():
        if dec.startswith("float rounding"):
            assert any(S.lm[i]["pos"] and _tie(S, i, dec) for i, _, _ in cases), dec
    for lv in (2, 3):
        assert _scene(f"{cam}-radius-l{lv}")[0].tell


def _tie(S, i, dec):
    axis = 0 if " u " in dec else 1
    c = py_project3(S.cam, _py_rt(S.T, S.lm[i]["pos"]))[axis]
    f = np.float32(c)
    lo, hi = (f, np.nextafter(f, np.float32(np.inf))) if float(f) <= c else (np.nextafter(f, np.float32(-np.inf)), f)
    return c == (float(lo) + float(hi)) / 2


def test_first_strict_minimum_takes_the_lower_grid_cell():
    S = _scene("pinhole-radius")[0]
    _, (a, b, _) = _run_oracle(S)
    i, left = S.first_min
    assert a[i] == 1 and b[i] == left


@pytest.mark.parametrize("model", range(6), ids=[f"cam{c['cam_model']}-dist{c['dist_model']}" for c in ALL_MODELS])
def test_random_projection_scene_oracle_vs_restatement(model):
    view, kf_lm_cand, Tcw, cam, lms, matched = synth.projection_search_scene(10 + model, n_kp=400, n_lm=300, cam=ALL_MODELS[model])
    for kw in (dict(), dict(num_octaves=8, scale_factor=1.2)):
        a, b, nm = og.search_by_projection(_view(view), kf_lm_cand, Tcw, cam, lms, matched, **kw)
        ra, rb, rnm = _py_search_by_projection(view, kf_lm_cand, Tcw, cam, lms, matched, **kw)
        assert np.array_equal(a, ra) and np.array_equal(b, rb) and nm == rnm


# ---------------------------------------------------------------------------------------------- K10 boundary scene
def se3_scale_scene(seed=20, sf=1.2, num_octaves=8):
    """synth.se3_search_scene with every landmark's max distance set so that its ratio is the n-fold product sf^n (or a
    neighbour) for its own n, and the keypoints of its point at octave n + 1: each match hangs on PredictScale's boundary"""
    views, T12, T21, a1, a2 = synth.se3_search_scene(seed, n_kp=400, n_shared=120)
    rng = np.random.default_rng(seed)
    inv = [{p: s for s, p in v["point_of_slot"].items()} for v in views]
    level_of_point, levels = {}, []
    for c, (Tsrc, Tab, Kd) in enumerate(((views[0]["Tcw"], T21, views[1]["K"]), (views[1]["Tcw"], T12, views[0]["K"]))):
        v = views[c]
        T1 = np.asarray(Tsrc).reshape(16).tolist(); T2 = np.asarray(Tab).reshape(16).tolist()
        for s in np.flatnonzero(v["lm_valid"]):
            p = v["point_of_slot"][int(s)]
            n = level_of_point.setdefault(p, int(rng.integers(1, 6)))
            k = int(rng.integers(-1, 2))
            pc = _py_rt(T2, _py_rt(T1, v["lm_pos"][s].tolist()))
            d3 = math.sqrt(pc[0] * pc[0] + pc[1] * pc[1] + pc[2] * pc[2])
            target = _steps(prod_n(sf, n), k)
            md = _max_distance_for(target, d3)
            for j in range(1, 200):                                # move the landmark by micrometres until the ratio is hit
                if md is not None:
                    break
                v["lm_pos"][s, 2] += 1e-6
                pc = _py_rt(T2, _py_rt(T1, v["lm_pos"][s].tolist()))
                d3 = math.sqrt(pc[0] * pc[0] + pc[1] * pc[1] + pc[2] * pc[2])
                md = _max_distance_for(target, d3)
            cur = float(np.float32(d3))
            v["lm_maxdist"][s] = md
            ratio, pl = md / cur, 0
            while prod_n(sf, pl) < ratio and pl < num_octaves - 1:
                pl += 1
            levels.append((c, int(s), py_predict_scale(md, d3, sf, num_octaves), pl))
    for c in range(2):
        for p, s in inv[c].items():
            views[c]["octave"][s] = level_of_point.get(p, 0) + 1
    return views, T12, T21, a1, a2, dict(num_octaves=num_octaves, scale_factor=sf), levels


def prod_n(sf, n):
    p = 1.0
    for _ in range(n):
        p = p * sf
    return p


def test_se3_scale_scene_checks_itself():
    """both sides of the level boundary occur among the matches the oracle finds and misses"""
    views, T12, T21, a1, a2, kw, levels = se3_scale_scene()
    k1, k2 = _view(views[0]), _view(views[1])
    m12, nf, m1, m2 = og.search_by_se3(k1, k2, T12, T21, a1, a2, **kw)
    assert (m1 >= 0).sum() > 10 and (m2 >= 0).sum() > 10
    # the logarithms and the repeated product disagree on some landmarks in each direction: the scene tells them apart
    for c in range(2):
        assert any(lg != pl for cc, _, lg, pl in levels if cc == c)
        assert any(lg == pl for cc, _, lg, pl in levels if cc == c)


class Se3Scene:
    """two keyframes with identity poses (T12 = T21 = I) whose keypoints are added in pairs, so keypoint i exists in both; a probe
    is a landmark of one keyframe and the keypoint of the other it should (or should not) take"""
    K = np.array([[458.654, 0, 367.215], [0, 457.296, 248.375], [0, 0, 1.0]])

    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)
        self.kf = [dict(kp=[], desc=[], lm_valid=[], lm_pos=[], lm_desc=[]) for _ in range(2)]
        self.cases = {}                     # decision -> list of (direction 0 = 1->2 / 1 = 2->1, landmark, side, expected match)
        self.filler = 0

    def desc(self):
        return self.rng.integers(0, 256, 32, dtype=np.uint8)

    def near(self, d, flips):
        b = np.unpackbits(d.copy()); b[self.rng.choice(256, flips, replace=False)] ^= 1
        return np.packbits(b)

    def spare_xy(self):
        self.filler += 1
        return (20.0 + 9.0 * (self.filler % 80), 466.0 - 0.05 * self.filler)

    def pair(self, kp, desc, lm):
        """keypoint i in both keyframes: kp[c] = (x, y), desc[c], lm[c] = (pos, landmark descriptor) or None → i"""
        for c in range(2):
            K = self.kf[c]
            K["kp"].append(kp[c] if kp[c] is not None else self.spare_xy()); K["desc"].append(desc[c] if desc[c] is not None else self.desc())
            K["lm_valid"].append(lm[c] is not None)
            K["lm_pos"].append(lm[c][0] if lm[c] is not None else [0.0, 0.0, 0.0])
            K["lm_desc"].append(lm[c][1] if lm[c] is not None else self.desc())
        return len(self.kf[0]["kp"]) - 1

    def probe(self, c, pw, kp_xy, decision, side, found=None, flips=10):
        """a landmark of keyframe c at pw and the keypoint of the other keyframe at kp_xy, `flips` bits from it"""
        d = self.desc()
        kp, desc, lm = [None, None], [None, None], [None, None]
        lm[c] = ([float(v) for v in pw], d)
        kp[1 - c] = kp_xy; desc[1 - c] = self.near(d, flips)
        i = self.pair(kp, desc, lm)
        self.cases.setdefault(decision, []).append((c, i, side, side if found is None else found))
        return i

    def uv(self, pw):
        """SearchBySE3's projection with identity poses, in the oracle's order"""
        K = self.K.reshape(9).tolist()
        p = [(K[3 * r] * pw[0] + K[3 * r + 1] * pw[1]) + K[3 * r + 2] * pw[2] for r in range(3)]
        return p[0] / p[2], p[1] / p[2]

    def views(self):
        out = []
        for K in self.kf:
            n = len(K["kp"])
            out.append(dict(kp=np.asarray(K["kp"], np.float32), octave=np.zeros(n, np.float32), desc=np.stack(K["desc"]),
                            lm_valid=np.asarray(K["lm_valid"], np.uint8), lm_pos=np.asarray(K["lm_pos"], np.float64), lm_maxdist=np.ones(n),
                            lm_desc=np.stack(K["lm_desc"]), K=self.K, Tcw=np.eye(4), img_bounds=np.array([0.0, W, 0.0, H])))
        return out, np.eye(4), np.eye(4), np.zeros(len(out[0]["kp"]), np.uint8), np.zeros(len(out[1]["kp"]), np.uint8)


def se3_boundary_scene(seed=21, th_low=50):
    """K10 at its gates, in both directions: the four image bounds (KF2's bounds in both directions), pc.z < 0, bestDist <= th_low
    from 1 to 2 and < th_low from 2 to 1 (best distances th_low - 1, th_low, th_low + 1 in each), and the agreement rule
    match2[i] == i: agreeing pairs, mutual matches at different indices (not reported), and i -> j with match2[i] == i
    (reported, the reference's reading)"""
    S = Se3Scene(seed)
    z = 6.0
    for c in range(2):
        for axis, bound, other in ((0, 0.0, 240.0), (0, float(W), 120.0), (1, 0.0, 200.0), (1, float(H), 560.0)):
            oth = other + 40.0 * c
            pw = [0.0, 0.0, z]
            pw[1 - axis] = (oth - Se3Scene.K[1 - axis, 2]) / Se3Scene.K[1 - axis, 1 - axis] * z
            lo, hi = -40.0 * z, 40.0 * z
            for _ in range(200):
                mid = 0.5 * (lo + hi); pw[axis] = mid
                (lo, hi) = (mid, hi) if S.uv(pw)[axis] < bound else (lo, mid)
            pw[axis] = lo
            seen = {}
            for st in range(-300, 301):
                q = list(pw); q[axis] = _steps(pw[axis], st)
                seen.setdefault(S.uv(q)[axis], q)
            vals = sorted(seen)
            for v in [v for v in vals if v < bound][-4:] + [v for v in vals if v >= bound][:4]:
                q = seen[v]
                xy = [0.0, 0.0]; xy[axis] = bound + (7.0 if bound == 0.0 else -7.0); xy[1 - axis] = float(np.float32(S.uv(q)[1 - axis]))
                ok = v >= bound if bound == 0.0 else v < bound
                S.probe(c, q, tuple(xy), f"image {'uv'[axis]} {'>=' if bound == 0.0 else '<'} {bound}", ok)
        for zz in (-1e-3, -0.0, 1e-3):                             # pc = (0, 0, z): u = cx for z != 0
            S.probe(c, [0.0, 0.0, zz], (367.215 + 2.0, 248.375), "pc.z < 0", not zz < 0, found=zz > 0)
        for j, f in enumerate((th_low - 1, th_low, th_low + 1)):
            pw = [(-0.6 + 0.3 * j) * z, (0.2 - 0.15 * c) * z, z]
            u, v = S.uv(pw)
            S.probe(c, pw, (u + 1.0, v), f"bestDist {'<=' if c == 0 else '<'} th_low", f <= th_low if c == 0 else f < th_low, flips=f)
    # the agreement rule: landmark of KF1 keypoint i at A_i -> KF2 keypoint at B; landmark of KF2 keypoint at B -> KF1 keypoint at A
    agree = []
    for j in range(3):
        A = [(-0.5 + 0.25 * j) * z, -0.3 * z, z]; B = [(-0.5 + 0.25 * j) * z, 0.25 * z, z]
        d1, d2 = S.desc(), S.desc()
        i = S.pair([S.uv(A), S.uv(B)], [S.near(d2, 8), S.near(d1, 8)], [(B, d1), (A, d2)])   # at one index: reported
        agree.append((i, i))
    for j in range(3):
        A = [(0.1 + 0.2 * j) * z, -0.3 * z, z]; B = [(0.1 + 0.2 * j) * z, 0.25 * z, z]
        d1, d2 = S.desc(), S.desc()
        i = S.pair([S.uv(A), None], [S.near(d2, 8), None], [(B, d1), None])                  # KF1 keypoint i -> KF2 keypoint k
        k = S.pair([None, S.uv(B)], [None, S.near(d1, 8)], [None, (A, d2)])                  # and back: mutual, not reported
        agree.append((i, -1))
    A = [0.65 * z, -0.3 * z, z]; B = [0.65 * z, 0.25 * z, z]; C = [0.85 * z, 0.25 * z, z]
    d1, d2, d3 = S.desc(), S.desc(), S.desc()
    i = S.pair([S.uv(A), S.uv(C)], [S.near(d3, 8), None], [(B, d1), (A, d3)])                # KF2 keypoint i's landmark -> KF1 i
    k = S.pair([None, S.uv(B)], [None, S.near(d1, 8)], [None, None])                          # KF1 i -> KF2 k: reported as k
    agree.append((i, k))
    S.agree = agree
    return S


def test_se3_boundary_scene_checks_itself():
    """every gate has cases on both sides in each direction, the oracle decides each as built, and the agreement cases come out
    as built (reported and not reported)"""
    S = se3_boundary_scene()
    views, T12, T21, a1, a2 = S.views()
    m12, nf, m1, m2 = og.search_by_se3(_view(views[0]), _view(views[1]), T12, T21, a1, a2)
    for dec, cases in S.cases.items():
        for c in {cc for cc, _, _, _ in cases}:
            assert {side for cc, _, side, _ in cases if cc == c} == {True, False}, (dec, c)
        for c, i, _, found in cases:
            assert ((m1 if c == 0 else m2)[i] >= 0) == found, (dec, c, i)
    for dec in S.cases:                                            # the gates in both directions, each threshold rule in its own
        assert {c for c, _, _, _ in S.cases[dec]} == ({0} if "<=" in dec else {1} if "th_low" in dec else {0, 1}), dec
    assert [int(m12[i]) for i, _ in S.agree] == [k for _, k in S.agree]
    assert nf == int((m12 >= 0).sum())


@pytest.mark.gpu
def test_cuda_se3_boundary_scene_equals_oracle(ctx):
    S = se3_boundary_scene()
    views, T12, T21, a1, a2 = S.views()
    k1, k2 = _view(views[0]), _view(views[1])
    r = og.search_by_se3(k1, k2, T12, T21, a1, a2)
    g = PR.search_by_se3_batch(ctx, k1, [k2], T12[None], T21[None], a1[None], [a2], debug=True)
    assert np.array_equal(g[2][0], r[2]) and np.array_equal(g[3], r[3])
    assert np.array_equal(g[0][0], r[0]) and g[1][0] == r[1]


# ---------------------------------------------------------------------------------------------- SASS guard
def _find_nvcc():
    for c in (shutil.which("nvcc"), os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")):
        if c and os.path.exists(c) and os.path.exists(os.path.join(os.path.dirname(c), "cuobjdump")):
            return c
    return None


NVCC = _find_nvcc()


def _sass(flags, tmp):
    nvcc = NVCC
    src = os.path.join(ROOT, "covins_b200", "csrc", "geom_kernels.cu")
    obj = os.path.join(tmp, "g%d.o" % len(flags))
    subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC,-fvisibility=hidden",
                           "--expt-relaxed-constexpr", *flags, "-c", src, "-o", obj])
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump")
    out = subprocess.check_output([cuobjdump, "-sass", obj], text=True)
    funcs, cur = {}, None
    for line in out.splitlines():
        if "Function : " in line:
            cur = line.split("Function : ")[1].strip(); funcs[cur] = []
        elif cur and "/*" in line:
            funcs[cur].append(line.strip())
    return funcs


@pytest.mark.skipif(NVCC is None, reason="needs nvcc and cuobjdump")
def test_geom_kernels_do_not_contract(tmp_path):
    """the kernels of geom_kernels.cu whose bit-exactness rests on user code alone compile to the same SASS with and without
    -fmad=false: no multiply-add is contracted.  search_proj_kernel is left out because libdevice's atan / tan are contracted
    inside; ransac_abs.cu / ransac_rel.cu are not checked because each kernel there gets one DFMA inside the inlined libdevice
    log of the adaptive iteration bound, which is only compared with an integer count."""
    a = _sass([], str(tmp_path)); b = _sass(["-fmad=false"], str(tmp_path))
    names = [f for f in a if any(k in f for k in ("search_se3_kernel", "score_abs_kernel", "score_rel_kernel", "lmv_"))]
    assert len(names) >= 6, list(a)
    for f in names:
        assert a[f] == b[f], f


# ---------------------------------------------------------------------------------------------- GPU parity (C-ABI)
@pytest.mark.gpu
@pytest.mark.parametrize("name", SCENE_NAMES)
def test_cuda_projection_boundaries_equal_oracle(ctx, name):
    S, kw, _ = _scene(name)
    args, r = _run_oracle(S, **kw)
    g = PR.search_by_projection(ctx, _kfview(args[0]), *args[1:], **kw)
    wrong = sorted({dec for dec, cases in S.cases.items() for i, _, _ in cases if g[0][i] != r[0][i] or g[1][i] != r[1][i]})
    assert not wrong and g[2] == r[2], wrong


@pytest.mark.gpu
def test_cuda_se3_boundaries_equal_oracle(ctx):
    views, T12, T21, a1, a2, kw, _ = se3_scale_scene()
    k1, k2 = _view(views[0]), _view(views[1])
    r = og.search_by_se3(k1, k2, T12, T21, a1, a2, **kw)
    d1 = sorted(int(np.unpackbits(views[0]["lm_desc"][i] ^ views[1]["desc"][r[2][i]]).sum()) for i in np.flatnonzero(r[2] >= 0))
    for extra in (dict(), dict(desc_th_low=d1[len(d1) // 2])):          # <= (1 -> 2) and < (2 -> 1) on an attained distance
        r = og.search_by_se3(k1, k2, T12, T21, a1, a2, **kw, **extra)
        g = PR.search_by_se3_batch(ctx, k1, [k2], T12[None], T21[None], a1[None], [a2], debug=True, **kw, **extra)
        assert np.array_equal(g[2][0], r[2]) and np.array_equal(g[3], r[3]), extra
        assert np.array_equal(g[0][0], r[0]) and g[1][0] == r[1], extra


@pytest.mark.gpu
@pytest.mark.parametrize("model", range(6), ids=[f"cam{c['cam_model']}-dist{c['dist_model']}" for c in ALL_MODELS])
def test_cuda_projection_random_scenes_every_model(ctx, model):
    for seed, n_kp, n_lm in ((30 + model, 1000, 800), (40 + model, 300, 1500)):
        view, kf_lm_cand, Tcw, cam, lms, matched = synth.projection_search_scene(seed, n_kp=n_kp, n_lm=n_lm, cam=ALL_MODELS[model])
        for kw in (dict(), dict(num_octaves=8, scale_factor=1.2), dict(th=25.0, desc_th_low=60)):
            g = PR.search_by_projection(ctx, _view(view), kf_lm_cand, Tcw, cam, lms, matched, **kw)
            r = og.search_by_projection(_view(view), kf_lm_cand, Tcw, cam, lms, matched, **kw)
            assert np.array_equal(g[0], r[0]) and np.array_equal(g[1], r[1]) and g[2] == r[2], (seed, kw)


def _crowd_scene(n_in):
    """one landmark with n_in keypoints inside its search radius (and one just outside), plus a second, ordinary landmark"""
    S = Scene(50, PINHOLE, np.eye(4))
    pw = [0.2, 0.1, 5.0]
    u, v = py_project3(PINHOLE, pw)
    d = S.desc()
    S.add_lm(pw, None, desc=d, flips=None)
    for j in range(n_in):
        a = 2 * math.pi * j / n_in
        S.add_kp(u + 6.0 * math.cos(a), v + 6.0 * math.sin(a), S.near(d, 20 + j % 7))
    S.add_kp(u + 14.0, v, S.near(d, 1))
    S.add_lm([-0.5, -0.3, 4.0])
    return S


@pytest.mark.gpu
def test_cuda_projection_candidate_cap(ctx):
    """48 keypoints in one radius are searched and equal the oracle; 49 are refused whole, action / best_idx untouched"""
    args, r = _run_oracle(_crowd_scene(48))
    g = PR.search_by_projection(ctx, _view(args[0]), *args[1:])
    assert np.array_equal(g[0], r[0]) and np.array_equal(g[1], r[1]) and g[2] == r[2] == 2
    args, r = _run_oracle(_crowd_scene(49))
    assert r[2] == 2                                                   # the oracle has no cap
    import ctypes as C
    from covins_b200._lib import lib
    L, prm, keep, m = PR._proj_args(_view(args[0]), *args[1:], 10.0, 50, 1, 2.0, PR.CProjLandmarks, PR.CSearchParams)
    kf = _view(args[0]); k = kf.cstruct()
    action = np.full(m, 77, np.int32); best = np.full(m, 77, np.int32); nm = C.c_int32(-5)
    rc = lib().cvb_search_by_projection(ctx.handle, C.byref(k), keep[1].ctypes.data, keep[2].ctypes.data, keep[3].ctypes.data, keep[4].ctypes.data,
                                        0, 0, 0.0, C.byref(L), keep[5].ctypes.data, C.byref(prm), action.ctypes.data, best.ctypes.data, C.byref(nm))
    assert rc == 3                                                     # CVB_ERR_UNSUPPORTED
    assert "more than 48 keypoints in a search radius" in lib().cvb_last_error(ctx.handle).decode()
    assert (action == 77).all() and (best == 77).all()
