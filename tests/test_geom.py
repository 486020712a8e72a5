"""Guided search (SearchBySE3) and RANSAC hypothesis scoring (SURVEY §8a M8 / V1): the C oracle against independent
numpy restatements (CPU), the CUDA path against the oracle bit for bit (GPU, through the C-ABI)."""
import math

import numpy as np
import pytest

from covins_b200 import placerec as PR, synth
from oracle import geom as og


def _view(v):
    return PR.KfView(v["kp"], v["octave"], v["desc"], v["lm_valid"], v["lm_pos"], v["lm_maxdist"], v["lm_desc"], v["K"], v["Tcw"], v["img_bounds"])


# ---------------------------------------------------------------------------------------------- independent restatements
def _py_grid(kp, w=752, h=480):
    grid = {}
    for i, (x, y) in enumerate(np.asarray(kp, np.float32)):
        px = int(np.floor(float(x) * (64 / w) + 0.5)); py = int(np.floor(float(y) * (48 / h) + 0.5))
        if 0 <= px < 64 and 0 <= py < 48:
            grid.setdefault((px, py), []).append(i)
    return grid


def _py_search(src, dst, Tcw_src, Tab, Kdst, img, already, th, th_low, strict):
    """one direction of FeatureMatcher::SearchBySE3 in plain python/numpy (num_octaves = 1 → predicted level 0)"""
    grid = _py_grid(dst["kp"])
    out = np.full(len(src["kp"]), -1, np.int32)
    bits = np.unpackbits(dst["desc"], axis=1)
    for i in range(len(src["kp"])):
        if not src["lm_valid"][i] or already[i]:
            continue
        p1 = Tcw_src[:3, :3] @ src["lm_pos"][i] + Tcw_src[:3, 3]
        p2 = Tab[:3, :3] @ p1 + Tab[:3, 3]
        if p2[2] < 0:
            continue
        pr = Kdst @ p2; u, v = pr[0] / pr[2], pr[1] / pr[2]
        if not (img[0] <= u < img[1] and img[2] <= v < img[3]):
            continue
        radius = th
        tx, ty = np.float32(u), np.float32(v)
        cx0 = max(0, int(np.floor((float(tx) - radius) * 64 / 752))); cx1 = min(63, int(np.ceil((float(tx) + radius) * 64 / 752)))
        cy0 = max(0, int(np.floor((float(ty) - radius) * 48 / 480))); cy1 = min(47, int(np.ceil((float(ty) + radius) * 48 / 480)))
        best, bd = -1, 1 << 30
        lb = np.unpackbits(src["lm_desc"][i])
        for ix in range(cx0, cx1 + 1):
            for iy in range(cy0, cy1 + 1):
                for idx in grid.get((ix, iy), []):
                    dx = np.float32(dst["kp"][idx, 0]) - tx; dy = np.float32(dst["kp"][idx, 1]) - ty
                    if float(np.sqrt(np.float32(dx * dx + dy * dy))) > radius:
                        continue
                    if int(dst["octave"][idx]) < -1 or int(dst["octave"][idx]) > 0:
                        continue
                    d = int((bits[idx] != lb).sum())
                    if d < bd:
                        bd, best = d, idx
        if best >= 0 and (bd < th_low if strict else bd <= th_low):
            out[i] = best
    return out


def test_grid_assignment_matches_plain_loop():
    rng = np.random.default_rng(0)
    kp = np.stack([rng.uniform(0, 752, 3000), rng.uniform(0, 480, 3000)], -1).astype(np.float32)
    kp[:5] = [[751.9, 10], [10, 479.9], [0, 0], [751.0, 479.0], [5.87, 4.99]]       # cells 64 / 48 (dropped) and the corners
    ptr, idx, _, _ = PR.assign_features_to_grid(kp, 752, 480)
    ref = _py_grid(kp)
    for ix in range(64):
        for iy in range(48):
            c = ix * 48 + iy
            assert idx[ptr[c]:ptr[c + 1]].tolist() == ref.get((ix, iy), [])
    assert ptr[-1] == sum(len(v) for v in ref.values()) and ptr[-1] < 3000


@pytest.mark.parametrize("seed", [0, 1])
def test_search_by_se3_oracle_vs_python_restatement(seed):
    views, T12, T21, a1, a2 = synth.se3_search_scene(seed, n_kp=400, n_shared=120)
    k1, k2 = _view(views[0]), _view(views[1])
    m12, nf, m1, m2 = og.search_by_se3(k1, k2, T12, T21, a1, a2)
    r1 = _py_search(views[0], views[1], views[0]["Tcw"], T21, views[1]["K"], views[1]["img_bounds"], a1, 9.5, 50, strict=False)
    r2 = _py_search(views[1], views[0], views[1]["Tcw"], T12, views[0]["K"], views[1]["img_bounds"], a2, 9.5, 50, strict=True)
    assert np.array_equal(m1, r1) and np.array_equal(m2, r2)
    assert (m1 >= 0).sum() > 40 and (m2 >= 0).sum() > 40
    # the agreement rule as written in the reference (:485-496): match2[i] == i, with i a KF1 index
    ref12 = np.where((r1 >= 0) & (r2[:len(r1)] == np.arange(len(r1))), r1, -1)
    assert np.array_equal(m12, ref12) and nf == (ref12 >= 0).sum()


def test_search_by_se3_reference_quirks():
    """(a) the agreement test reads match2[i]: a genuine mutual match (i ↔ j, i != j) is NOT reported, while i ↔ i is;
    (b) direction 2→1 is gated by KF2's image bounds; (c) <= vs < on the descriptor threshold."""
    views, T12, T21, a1, a2 = synth.se3_search_scene(3, n_kp=300, n_shared=100)
    a1[:] = 0; a2[:] = 0
    k1, k2 = _view(views[0]), _view(views[1])
    m12, nf, m1, m2 = og.search_by_se3(k1, k2, T12, T21, a1, a2)
    mutual = [(i, int(m1[i])) for i in range(len(m1)) if m1[i] >= 0 and m2[m1[i]] == i]
    assert len(mutual) > 20                                     # plenty of true mutual matches exist …
    assert nf == sum(1 for i in range(len(m1)) if m1[i] >= 0 and m2[i] == i)   # … but only "match2[i] == i" counts
    assert nf < len(mutual)
    # (b) shrink KF2's image bounds: direction 2→1 loses matches although the projections land in KF1
    v2 = dict(views[1]); v2["img_bounds"] = np.array([0.0, 300.0, 0.0, 480.0])
    _, _, _, m2b = og.search_by_se3(k1, _view(v2), T12, T21, a1, a2)
    assert (m2b >= 0).sum() < (m2 >= 0).sum()
    # (c) a threshold equal to an attained best distance: direction 1 keeps it (<=), direction 2 drops it (<)
    d1 = [int(np.unpackbits(views[0]["lm_desc"][i] ^ views[1]["desc"][m1[i]]).sum()) for i in range(len(m1)) if m1[i] >= 0]
    thr = int(np.median(d1))
    _, _, m1c, m2c = og.search_by_se3(k1, k2, T12, T21, a1, a2, desc_th_low=thr)
    kept1 = [int(np.unpackbits(views[0]["lm_desc"][i] ^ views[1]["desc"][m1c[i]]).sum()) for i in range(len(m1c)) if m1c[i] >= 0]
    kept2 = [int(np.unpackbits(views[1]["lm_desc"][i] ^ views[0]["desc"][m2c[i]]).sum()) for i in range(len(m2c)) if m2c[i] >= 0]
    assert max(kept1) == thr and max(kept2) < thr


def _rand_pose(rng):
    R = synth._rot(rng.normal(0, 0.5, 3)); t = rng.normal(0, 1.0, 3)
    return np.concatenate([R, t[:, None]], 1)


def _scoring_case(seed, n=300, H=40):
    rng = np.random.default_rng(seed)
    Rc = synth._rot(rng.normal(0, 0.3, 3)); c = rng.normal(0, 0.05, 3)           # camera in the body frame
    Twb = _rand_pose(rng)
    pts = rng.uniform(-5, 5, (n, 3)) + np.array([0, 0, 12.0])
    pb = (pts - Twb[:, 3]) @ Twb[:, :3]                                            # R^T (p - t)
    pc = (pb - c) @ Rc
    f = pc / np.linalg.norm(pc, axis=1, keepdims=True)
    out = rng.random(n) < 0.3
    f[out] = rng.normal(0, 1, (out.sum(), 3)); f /= np.linalg.norm(f, axis=1, keepdims=True)
    sigma = rng.uniform(1e-6, 1e-5, n)
    models = np.stack([Twb] + [Twb + np.concatenate([np.zeros((3, 3)), rng.normal(0, 0.05, (3, 1))], 1) for _ in range(H - 1)])
    return models, pts, f, sigma, c, Rc


def test_absolute_pose_scoring_oracle_vs_numpy():
    models, pts, f, sigma, c, Rc = _scoring_case(0)
    sc, inl, cnt = og.score_absolute_pose(models, pts, f, sigma, c, Rc, threshold=25.0)
    for h in (0, 1, 17):
        R, t = models[h][:, :3], models[h][:, 3]
        b = (pts - t) @ R                                  # R^T (p - t)
        q = (b - c) @ Rc
        q /= np.linalg.norm(q, axis=1, keepdims=True)
        ref = ((q - f) ** 2).sum(1) / sigma
        assert np.allclose(sc[h], ref, rtol=1e-9, atol=1e-12)
        assert np.array_equal(inl[h].astype(bool), sc[h] < 25.0) and cnt[h] == (sc[h] < 25.0).sum()
    assert cnt[0] > 150 and cnt[0] == cnt.max()            # the true pose explains the 70 % inlier correspondences


def test_relative_pose_scoring_oracle_vs_numpy():
    rng = np.random.default_rng(1)
    n, H = 250, 30
    T12 = _rand_pose(rng); T12[:, 3] *= 0.3
    X1 = rng.uniform(-3, 3, (n, 3)) + np.array([0, 0, 8.0])
    X2 = (X1 - T12[:, 3]) @ T12[:, :3]
    f1 = X1 / np.linalg.norm(X1, axis=1, keepdims=True); f2 = X2 / np.linalg.norm(X2, axis=1, keepdims=True)
    f2[rng.random(n) < 0.25] = np.array([0.0, 0.0, 1.0])
    s1 = rng.uniform(1e-6, 1e-5, n); s2 = rng.uniform(1e-6, 1e-5, n)
    models = np.stack([T12] + [T12 + np.concatenate([np.zeros((3, 3)), rng.normal(0, 0.03, (3, 1))], 1) for _ in range(H - 1)])
    sc, inl, cnt = og.score_relative_pose(models, f1, f2, s1, s2, threshold=9.0)
    for h in (0, 5):
        R, t = models[h][:, :3], models[h][:, 3]
        u = f2 @ R.T
        lam = np.zeros((n, 2))
        for i in range(n):                                  # triangulate2: 2x2 solve per correspondence
            A = np.array([[f1[i] @ f1[i], -(f1[i] @ u[i])], [f1[i] @ u[i], -(u[i] @ u[i])]])
            lam[i] = np.linalg.solve(A, np.array([t @ f1[i], t @ u[i]]))
        X = (lam[:, :1] * f1 + t + lam[:, 1:] * u) / 2
        r1 = X / np.linalg.norm(X, axis=1, keepdims=True)
        r2 = (X - t) @ R; r2 /= np.linalg.norm(r2, axis=1, keepdims=True)
        ref = ((r1 - f1) ** 2).sum(1) * 0.5 / s1 + ((r2 - f2) ** 2).sum(1) * 0.5 / s2
        assert np.allclose(sc[h], ref, rtol=1e-7, atol=1e-10)
    assert cnt[0] > 150 and cnt[0] == cnt.max()


def test_ransac_select_replays_the_sequential_rule():
    cnt = np.array([3, 10, 10, 50, 49, 120, 5, 119, 300, 2])
    best, used = PR.ransac_select(cnt, n_points=400, sample_size=3, max_iterations=300)
    assert best == 8 and used <= len(cnt)                   # strictly-greater rule: index 5 is replaced by 8, ties keep the first


# ---------------------------------------------------------------------------------------------- GPU parity (C-ABI)
@pytest.mark.gpu
def test_cuda_search_by_se3_equals_oracle(ctx):
    scenes = [synth.se3_search_scene(s, n_kp=1000, n_shared=300) for s in (5, 6, 7)] + [synth.se3_search_scene(8, n_kp=200, n_shared=50)]
    # batch: one query keyframe against three candidates (the candidates come from different scenes: same KF1 arrays)
    v1 = scenes[0][0][0]
    k1 = _view(v1)
    k2s = [_view(sc[0][1]) for sc in scenes[:3]]
    T12 = np.stack([sc[1] for sc in scenes[:3]]); T21 = np.stack([sc[2] for sc in scenes[:3]])
    a1 = np.stack([sc[3] for sc in scenes[:3]]); a2 = [sc[4] for sc in scenes[:3]]
    m12, nf, m1, m2 = PR.search_by_se3_batch(ctx, k1, k2s, T12, T21, a1, a2, debug=True)
    off = 0
    for p in range(3):
        r12, rnf, r1, r2 = og.search_by_se3(k1, k2s[p], T12[p], T21[p], a1[p], a2[p])
        assert np.array_equal(m12[p], r12) and nf[p] == rnf and np.array_equal(m1[p], r1) and np.array_equal(m2[off:off + k2s[p].n], r2), p
        off += k2s[p].n
    assert (m1[0] >= 0).sum() > 100
    # different sizes (n1 != n2), several octaves, larger radius
    views, T12s, T21s, b1, b2 = synth.se3_search_scene(9, n_kp=500, n_shared=150, n_octaves_data=3)
    va, vb = dict(views[0]), dict(views[1])
    for k in ("kp", "octave", "desc", "lm_valid", "lm_pos", "lm_maxdist", "lm_desc"):
        vb[k] = vb[k][:350]
    ka, kb = _view(va), _view(vb)
    for kw in (dict(th=9.5, num_octaves=3), dict(th=25.0, num_octaves=1), dict(th=9.5, num_octaves=3, desc_th_low=30)):
        g = PR.search_by_se3_batch(ctx, ka, [kb], T12s[None], T21s[None], b1[None], [b2[:350]], debug=True, **kw)
        r = og.search_by_se3(ka, kb, T12s, T21s, b1, b2[:350], **kw)
        assert np.array_equal(g[0][0], r[0]) and g[1][0] == r[1] and np.array_equal(g[2][0], r[2]) and np.array_equal(g[3], r[3]), kw
    # empty batch / empty keyframe
    e = PR.search_by_se3_batch(ctx, ka, [], np.zeros((0, 16)), np.zeros((0, 16)), np.zeros((0, ka.n), np.uint8), [])
    assert e[0].shape == (0, ka.n)


@pytest.mark.gpu
def test_cuda_scoring_equals_oracle_bitwise(ctx):
    models, pts, f, sigma, c, Rc = _scoring_case(4, n=1000, H=300)        # Se3Solver: up to 300 RANSAC iterations
    sc, inl, cnt = PR.score_absolute_pose(ctx, models, pts, f, sigma, c, Rc, 25.0)
    rs, ri, rc = og.score_absolute_pose(models, pts, f, sigma, c, Rc, 25.0)
    assert np.array_equal(sc, rs) and np.array_equal(inl, ri) and np.array_equal(cnt, rc)
    _, _, cnt_only = PR.score_absolute_pose(ctx, models, pts, f, sigma, c, Rc, 25.0, want_scores=False, want_inliers=False)
    assert np.array_equal(cnt_only, rc)
    rng = np.random.default_rng(2)
    n, H = 777, 64
    T12 = _rand_pose(rng); T12[:, 3] *= 0.3
    X1 = rng.uniform(-3, 3, (n, 3)) + np.array([0, 0, 8.0]); X2 = (X1 - T12[:, 3]) @ T12[:, :3]
    f1 = X1 / np.linalg.norm(X1, axis=1, keepdims=True); f2 = X2 / np.linalg.norm(X2, axis=1, keepdims=True)
    s1 = rng.uniform(1e-6, 1e-5, n); s2 = rng.uniform(1e-6, 1e-5, n)
    models = np.stack([T12] + [T12 + np.concatenate([np.zeros((3, 3)), rng.normal(0, 0.03, (3, 1))], 1) for _ in range(H - 1)])
    g = PR.score_relative_pose(ctx, models, f1, f2, s1, s2, 9.0)
    r = og.score_relative_pose(models, f1, f2, s1, s2, 9.0)
    assert np.array_equal(g[0], r[0]) and np.array_equal(g[1], r[1]) and np.array_equal(g[2], r[2])
    best, used = PR.ransac_select(g[2], n, 5, 300)
    assert best == 0


# ---------------------------------------------------------------------------------------------- SearchByProjection
def _py_rt(T, p):
    """rows 0..2 of T (4x4, row-major flat) applied to p, each row summed left to right"""
    return [(T[4 * r] * p[0] + T[4 * r + 1] * p[1] + T[4 * r + 2] * p[2]) + T[4 * r + 3] for r in range(3)]


def py_project3(cam, pc):
    """camera_->project3 in plain float64, the oracle's operation order: pinhole (0) / unified (1) x radtan (0) / equidistant
    (1) / FOV (2); None = not projectable"""
    intr, d = [float(v) for v in cam["intr"]], [float(v) for v in cam["dist"]]
    dm = cam.get("dist_model", 0)
    den = pc[2]
    if cam.get("cam_model", 0) == 1:
        den = pc[2] + float(cam["xi"]) * math.sqrt(pc[0] * pc[0] + pc[1] * pc[1] + pc[2] * pc[2])
    if not den > 1e-10:
        return None
    x, y = pc[0] / den, pc[1] / den
    r2 = x * x + y * y
    if dm == 0:
        rad = 1.0 + d[0] * r2 + d[1] * r2 * r2
        xd = x * rad + 2.0 * d[2] * x * y + d[3] * (r2 + 2.0 * x * x)
        yd = y * rad + d[2] * (r2 + 2.0 * y * y) + 2.0 * d[3] * x * y
    else:
        s = 1.0
        if dm == 1:
            r = math.sqrt(r2)
            if r >= 1e-8:
                th = math.atan(r); t2 = th * th
                s = th * (1.0 + d[0] * t2 + d[1] * t2 * t2 + d[2] * t2 * t2 * t2 + d[3] * t2 * t2 * t2 * t2) / r
        elif d[0] * d[0] >= 1e-5:
            w = d[0]; c = 2.0 * math.tan(0.5 * w)
            s = c / w if r2 < 1e-5 else math.atan(c * math.sqrt(r2)) / (w * math.sqrt(r2))
        xd, yd = s * x, s * y
    return intr[0] * xd + intr[2], intr[1] * yd + intr[3]


def py_predict_scale(maxdist, d3, sf, num_octaves):
    """LandmarkBase::PredictScale: ceil(log(maxdist / float(d3)) / log(sf)) clamped to [0, num_octaves - 1]"""
    n = math.ceil(math.log(maxdist / float(np.float32(d3))) / math.log(sf))
    return min(max(n, 0), num_octaves - 1)


def _py_search_by_projection(view, kf_lm_cand, Tcw, cam, lms, matched, th=10.0, th_low=50, num_octaves=1, scale_factor=2.0):
    """plain python restatement (every camera model, octaves), sequential like the reference; float64 / float32 scalars in the
    oracle's operation order, so that it agrees at rounding boundaries too"""
    grid = view["grid"] if "grid" in view else _py_grid(view["kp"])      # a scene may file keypoints in cells of its choice
    matched = matched.copy(); has_lm = view["lm_valid"].copy(); lm_cand = kf_lm_cand.copy(); feat = lms["feat_idx"].copy()
    bits = np.unpackbits(view["desc"], axis=1)
    T = [float(v) for v in np.asarray(Tcw, np.float64).reshape(16)]
    Ow = [-(T[r] * T[3] + T[4 + r] * T[7] + T[8 + r] * T[11]) for r in range(3)]
    img = [float(v) for v in view["img_bounds"]]
    w_inv, h_inv = 64 / 752.0, 48 / 480.0
    kp = np.asarray(view["kp"], np.float32)
    m = len(lms["pos"]); action = np.zeros(m, np.int32); best_idx = np.full(m, -1, np.int32); nm = 0
    for i in range(m):
        if not lms["valid"][i]:
            continue
        pw = [float(v) for v in lms["pos"][i]]
        pc = _py_rt(T, pw)
        if pc[2] < 0:
            continue
        uv = py_project3(cam, pc)
        if uv is None or not (img[0] <= uv[0] < img[1] and img[2] <= uv[1] < img[3]):
            continue
        PO = [pw[r] - Ow[r] for r in range(3)]; n = [float(v) for v in lms["normal"][i]]
        d3 = math.sqrt(PO[0] * PO[0] + PO[1] * PO[1] + PO[2] * PO[2])
        if d3 < lms["min_dist"][i] or d3 > lms["max_dist"][i] or PO[0] * n[0] + PO[1] * n[1] + PO[2] * n[2] < 0.5 * d3:
            continue
        level = py_predict_scale(float(lms["max_distance"][i]), d3, scale_factor, num_octaves)
        radius = th * math.pow(scale_factor, level)
        tx, ty = np.float32(uv[0]), np.float32(uv[1])
        cx0 = max(0, math.floor((float(tx) - radius) * w_inv)); cx1 = min(63, math.ceil((float(tx) + radius) * w_inv))
        cy0 = max(0, math.floor((float(ty) - radius) * h_inv)); cy1 = min(47, math.ceil((float(ty) + radius) * h_inv))
        if cx0 >= 64 or cx1 < 0 or cy0 >= 48 or cy1 < 0:
            continue
        lb = np.unpackbits(lms["desc"][i]); ham = lambda k: int((bits[k] != lb).sum())
        bd, best = 256, -1
        for ix in range(cx0, cx1 + 1):
            for iy in range(cy0, cy1 + 1):
                for idx in grid.get((ix, iy), []):
                    dx = kp[idx, 0] - tx; dy = kp[idx, 1] - ty
                    if not float(np.sqrt(np.float32(dx * dx + dy * dy))) <= radius or matched[idx]:
                        continue
                    if not level - 1 <= int(view["octave"][idx]) <= level:
                        continue
                    dd = ham(idx)
                    if dd < bd:
                        bd, best = dd, idx
        if best < 0 or bd > th_low:
            continue
        best_idx[i] = best
        ex = feat[i]
        if ex != -1:
            keep = ham(ex) < bd or (has_lm[best] and ham(best) < bd)
            if keep:
                action[i] = 3; continue
            had, displaced = has_lm[best], lm_cand[best]
            has_lm[ex] = 0; lm_cand[ex] = -1; has_lm[best] = 1; lm_cand[best] = i; feat[i] = best
            if had and displaced >= 0:
                feat[displaced] = -1
            action[i] = 2
        else:
            matched[best] = 1; action[i] = 1; nm += 1
    return action, best_idx, nm


def test_search_by_projection_oracle_vs_python_restatement():
    view, kf_lm_cand, Tcw, cam, lms, matched = synth.projection_search_scene(0, n_kp=600, n_lm=500)
    a, b, nm = og.search_by_projection(_view(view), kf_lm_cand, Tcw, cam, lms, matched)
    ra, rb, rnm = _py_search_by_projection(view, kf_lm_cand, Tcw, cam, lms, matched)
    assert np.array_equal(a, ra) and np.array_equal(b, rb) and nm == rnm
    assert nm > 40 and (a == 2).sum() >= 3 and (a == 3).sum() >= 3      # new matches, remaps and kept observations all occur
    # order dependence: competitors for one keypoint — the earlier landmark takes it
    taken = b[a == 1]
    assert len(set(taken.tolist())) == len(taken)


@pytest.mark.gpu
@pytest.mark.parametrize("model", ["radtan", "equi_unified"])
def test_cuda_search_by_projection_equals_oracle(ctx, model):
    from covins_b200.synth_map import EUROC_INTR
    cam = None if model == "radtan" else dict(intr=EUROC_INTR, dist=np.array([-0.013, 0.02, -0.012, 0.002]), cam_model=1, dist_model=1, xi=0.9)
    for seed, n_kp, n_lm in ((1, 1000, 800), (2, 300, 2000), (3, 50, 10)):
        view, kf_lm_cand, Tcw, cam_, lms, matched = synth.projection_search_scene(seed, n_kp=n_kp, n_lm=n_lm, cam=cam)
        for kw in (dict(), dict(th=25.0, desc_th_low=60), dict(num_octaves=3, scale_factor=1.2)):
            g = PR.search_by_projection(ctx, _view(view), kf_lm_cand, Tcw, cam_, lms, matched, **kw)
            r = og.search_by_projection(_view(view), kf_lm_cand, Tcw, cam_, lms, matched, **kw)
            assert np.array_equal(g[0], r[0]) and np.array_equal(g[1], r[1]) and g[2] == r[2], (seed, kw)
    assert g[2] >= 0
