"""The SIFT form of the resident map database (cvb_db_create(ctx, 128), cvb_db_append_sift, cvb_db_match_l2[_dev]): every
request must give, keyframe by keyframe, exactly what cvb_match_l2_batch gives on the same candidates — indices, float
distances, order — on the scalar kernel and on the tensor-core kernel reading the resident L2 operand tiles."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import golden_cases
from covins_b200 import matching as M
from covins_b200 import synth
from covins_b200._lib import lib

pytestmark = pytest.mark.gpu

CVB_ERR_INVALID, CVB_ERR_UNSUPPORTED = 1, 3


@pytest.fixture(params=["default", "tc", "popc"])
def kernel(request, monkeypatch):
    if request.param == "default":
        monkeypatch.delenv("COVINS_B200_MATCH_KERNEL", raising=False)
    else:
        monkeypatch.setenv("COVINS_B200_MATCH_KERNEL", request.param)
    return request.param


def _reference(ctx, q, rows, lens, thr, ratio):
    """cvb_match_l2_batch on the keyframes `lens` (rows concatenated) → the database's host outputs"""
    seg = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    mt, md, nm = M.match_candidates_l2(ctx, q, rows, seg, thr, ratio)
    kf, qq = np.nonzero(mt >= 0)
    return nm, kf, qq, mt[kf, qq], md[kf, qq]


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.int32) if a.dtype == np.float32 else a.astype(np.int64)


def _same(got, ref):
    """equal indices and bit-identical float distances"""
    return len(got) == len(ref) and all(np.array_equal(_bits(a), _bits(b)) for a, b in zip(got, ref))


def _dev(db, q, thr, ratio):
    import torch
    mt, md, nm = db.match_l2_dev(torch.from_numpy(q.astype(np.uint8)).cuda(), thr, ratio)
    torch.cuda.synchronize()
    mt, md, nm = mt.cpu().numpy(), md.cpu().numpy(), nm.cpu().numpy()
    kf, qq = np.nonzero(mt >= 0)
    return nm, kf, qq, mt[kf, qq], md[kf, qq]


def test_golden_through_database(ctx, kernel, golden_dir):
    g, names = golden_cases(os.path.join(golden_dir, "knn_l2.npz"))
    for n in names:
        q = g[n + "/q"].astype(np.float32); t = g[n + "/t"].astype(np.float32)
        db = M.DescriptorDatabase(ctx, kind="sift")
        db.append(t, [len(t)])
        nm, kf, qq, tt, dd = db.match_l2(q, 500.0, 0.8)
        ref = g[n + "/match"]
        assert np.array_equal(kf, np.zeros(len(qq))) and np.array_equal(qq, np.flatnonzero(ref >= 0)), n
        assert np.array_equal(tt, ref[ref >= 0]) and nm[0] == (ref >= 0).sum(), n
        acc = np.flatnonzero(ref >= 0)
        assert np.array_equal(dd, g[n + "/dist"][acc, 0]), n          # bit-exact float distances
        db.close()


def test_ragged_appends_removals_and_dev(ctx, kernel):
    """C2/C3-like request: 300 queries against ragged keyframes appended in several calls, then removals of the first, a
    middle and the last keyframe and appends after them; host and device requests, repeated"""
    s, _ = synth.sift_keyframes(seed=31, n_kf=161, n_feat=300, n_lm=500, window=500)
    q = s[0]
    lens = ([0, 1, 127, 128, 129, 300, 0, 255, 256, 257] * 16)[:160]
    rows = [s[i + 1][:n] for i, n in enumerate(lens)]
    db = M.DescriptorDatabase(ctx, kind="sift")
    for a, b in ((0, 1), (1, 7), (7, 90), (90, 160)):
        db.append(np.concatenate(rows[a:b]).reshape(-1, 128), lens[a:b])
    keep = list(range(len(lens)))

    def check():
        ref = _reference(ctx, q, np.concatenate([rows[i] for i in keep]).reshape(-1, 128), [lens[i] for i in keep], 500.0, 0.8)
        assert db.size() == (len(keep), sum(lens[i] for i in keep))
        got = db.match_l2(q, 500.0, 0.8)
        assert len(ref[1]) > 0
        for a, b in zip(got, ref):
            assert np.array_equal(_bits(a), _bits(b)), (a[:20], b[:20], len(a), len(b))
        assert _same(db.match_l2(q, 500.0, 0.8), got)                      # repeat calls: identical bits
        assert _same(_dev(db, q, 500.0, 0.8), ref)

    check()
    for victim in ("first", "middle", "last"):
        i = {"first": 0, "middle": len(keep) // 2, "last": len(keep) - 1}[victim]
        db.remove(i); keep.pop(i)
        check()
    extra = [s[1][:300], s[2][:129], s[3][:0]]
    db.append(np.concatenate(extra).reshape(-1, 128), [300, 129, 0])
    rows += extra; lens += [300, 129, 0]; keep += [len(lens) - 3, len(lens) - 2, len(lens) - 1]
    check()
    db.remove(len(keep) - 1); keep.pop()
    check()
    db.close()


def test_tc_and_popc_agree_at_c3_size(ctx, monkeypatch):
    """C3-sized map (2 000 keyframes x 300 rows) and a 300-row query: the tensor-core kernel on the resident tiles and the
    scalar kernel on the packed rows give identical bits, host and device requests"""
    s, _ = synth.sift_keyframes(seed=5, n_kf=2001, n_feat=300)
    db = M.DescriptorDatabase(ctx, reserve_rows=2000 * 300, kind="sift")
    db.append(s[1:].reshape(-1, 128), [300] * 2000)
    out = {}
    for k in ("tc", "popc"):
        monkeypatch.setenv("COVINS_B200_MATCH_KERNEL", k)
        out[k] = (db.match_l2(s[0]), _dev(db, s[0], 500.0, 0.8))
    monkeypatch.delenv("COVINS_B200_MATCH_KERNEL", raising=False)
    assert _same(out["tc"][0], out["popc"][0]) and _same(out["tc"][1], out["popc"][0])
    assert out["tc"][0][0].sum() > 100
    db.close()


_TWO_SQUARES = {x * x + y * y: (x, y) for x in range(256) for y in range(256)}


def _row_with_d2(d2, rng):
    """a u8 row whose squared norm is exactly d2 (so that its distance to the zero row is sqrtf(d2)): components of 255,
    the rest (a few 255^2) as four squares"""
    for k in (1, 2, 3):
        n255 = max(0, d2 // 65025 - k)
        rem = d2 - n255 * 65025
        four = next(((a, b) + _TWO_SQUARES[rem - a * a - b * b] for a in range(255, -1, -1) for b in range(a, -1, -1)
                     if rem - a * a - b * b in _TWO_SQUARES), None)
        if four is not None:
            break
    assert four is not None and n255 + 4 <= 128
    r = np.zeros(128, np.int64)
    r[rng.permutation(128)[:n255 + 4]] = [255] * n255 + list(four)
    assert (r * r).sum() == d2
    return r


def _sqrt_ties(lo, hi):
    """integers D in [lo, hi) with sqrtf(D) == sqrtf(D + 1): distinct squared distances that tie as floats"""
    d = np.arange(lo, hi, dtype=np.int64)
    f = np.sqrt(d.astype(np.float32))
    return d[:-1][f[:-1] == f[1:]]


def test_float_sqrt_ties(ctx, kernel):
    """rows whose squared distances differ but whose sqrtf is equal: OpenCV compares the float distances, so the lower
    trainIdx stays first although the later row is nearer in d2.  Pairs placed inside a quad, across the 128-row tile
    boundary and far apart; with ratio > 1 the tie decides the accepted trainIdx."""
    rng = np.random.default_rng(3)
    ties = _sqrt_ties(7_800_000, 8_000_000)
    assert len(ties) > 100
    pairs = [(0, 1), (127, 128), (5, 200), (126, 129), (64, 66)]
    kfs, lens = [], []
    for k, (i, j) in enumerate(pairs):
        D = int(ties[7 * k + 3])
        kf = [_row_with_d2(int(rng.integers(D + 5000, 8_100_000)), rng) for _ in range(300)]
        kf[i] = _row_with_d2(D + 1, rng)             # lower index, larger d2
        kf[j] = _row_with_d2(D, rng)                 # same float distance
        kfs.append(np.array(kf, np.float32)); lens.append(300)
    s, _ = synth.sift_keyframes(seed=9, n_kf=1, n_feat=140)
    q = np.concatenate([np.zeros((1, 128), np.float32), s[0]])     # 141 queries: two query blocks
    t = np.concatenate(kfs)
    db = M.DescriptorDatabase(ctx, kind="sift")
    db.append(t, lens)
    for thr, ratio in ((1e9, 1.5), (1e9, 1.0), (500.0, 0.8)):
        ref = _reference(ctx, q, t, lens, thr, ratio)
        got = db.match_l2(q, thr, ratio)
        assert _same(got, ref)
        assert _same(_dev(db, q, thr, ratio), ref)
        if ratio > 1:
            first = got[2] == 0
            assert np.array_equal(got[3][first], [i for i, _ in pairs])   # the tie keeps the lower trainIdx
    db.close()


def test_cap_and_n_total(ctx, kernel):
    s, _ = synth.sift_keyframes(seed=17, n_kf=9, n_feat=300, n_lm=400, window=400)
    db = M.DescriptorDatabase(ctx, kind="sift")
    db.append(s[1:].reshape(-1, 128), [300] * 8)
    nm, kf, qq, tt, dd = db.match_l2(s[0])
    total = len(kf)
    assert total == nm.sum() and total > 10
    q = np.ascontiguousarray(s[0], np.float32)
    for cap in (0, 1, total // 2, total, total + 5):
        o = [np.full(max(cap, 1), -7, np.int32) for _ in range(3)] + [np.full(max(cap, 1), -7, np.float32)]
        n2 = np.zeros(8, np.int32)
        tot = C.c_int32(-1)
        rc = lib().cvb_db_match_l2(ctx.handle, db.handle, q.ctypes.data, len(q), 500.0, 0.8, n2.ctypes.data, o[0].ctypes.data,
                                   o[1].ctypes.data, o[2].ctypes.data, o[3].ctypes.data, cap, C.byref(tot))
        assert rc == 0 and tot.value == total and np.array_equal(n2, nm)
        m = min(cap, total)
        assert _same((o[0][:m], o[1][:m], o[2][:m], o[3][:m]), (kf[:m], qq[:m], tt[:m], dd[:m]))
        assert (o[0][m:cap] == -7).all()                                   # nothing written past the accepted matches
    db.close()


# ------------------------------------------------------------------------------------------------------------ refusals
def _create(ctx, desc_bytes):
    h = C.c_void_p()
    return lib().cvb_db_create(ctx.handle, desc_bytes, C.byref(h)), h


@pytest.mark.parametrize("bad", [0.5, -1.0, 256.0, np.nan, np.inf, -np.inf, 1e30])
def test_refuses_non_integer_rows_without_launch(ctx, bad):
    s, _ = synth.sift_keyframes(seed=2, n_kf=3, n_feat=50)
    db = M.DescriptorDatabase(ctx, kind="sift")
    db.append(s[0], [50])
    before, launches = db.size(), ctx.launch_count()
    rows = s[1:].reshape(-1, 128).copy()
    rows[77, 31] = bad
    rpk = np.array([50, 50], np.int32)
    rc = lib().cvb_db_append_sift(ctx.handle, db.handle, rows.ctypes.data, rpk.ctypes.data, 2)
    assert rc == CVB_ERR_UNSUPPORTED
    q = s[2].copy(); q[3, 100] = bad
    tot = C.c_int32()
    o = np.empty(64, np.int32); d = np.empty(64, np.float32); n2 = np.empty(1, np.int32)
    rc = lib().cvb_db_match_l2(ctx.handle, db.handle, q.ctypes.data, len(q), 500.0, 0.8, n2.ctypes.data, o.ctypes.data,
                               o.ctypes.data, o.ctypes.data, d.ctypes.data, 16, C.byref(tot))
    assert rc == CVB_ERR_UNSUPPORTED
    assert ctx.launch_count() == launches and db.size() == before
    db.append(s[1], [50])                                                 # still usable
    assert db.size() == (2, 100)
    db.close()


def test_refuses_wrong_kind_calls(ctx):
    import torch
    orb = M.DescriptorDatabase(ctx)
    sift = M.DescriptorDatabase(ctx, kind="sift")
    launches = ctx.launch_count()
    f = np.zeros((4, 128), np.float32); u = np.zeros((4, 32), np.uint8); rpk = np.array([4], np.int32)
    dq = torch.zeros((4, 128), dtype=torch.uint8, device="cuda")
    dmt = torch.empty((1, 4), dtype=torch.int32, device="cuda"); dmd = torch.empty((1, 4), dtype=torch.float32, device="cuda")
    dnm = torch.empty((1,), dtype=torch.int32, device="cuda")
    o = np.empty(8, np.int32); d = np.empty(8, np.float32); tot = C.c_int32()
    L = lib()
    assert L.cvb_db_append_sift(ctx.handle, orb.handle, f.ctypes.data, rpk.ctypes.data, 1) == CVB_ERR_INVALID
    assert b"holds ORB" in L.cvb_last_error(ctx.handle)
    assert L.cvb_db_append(ctx.handle, sift.handle, u.ctypes.data, rpk.ctypes.data, 1) == CVB_ERR_INVALID
    assert b"holds SIFT" in L.cvb_last_error(ctx.handle)
    assert L.cvb_db_match_l2(ctx.handle, orb.handle, f.ctypes.data, 4, 500.0, 0.8, None, o.ctypes.data, o.ctypes.data,
                             o.ctypes.data, d.ctypes.data, 8, C.byref(tot)) == CVB_ERR_INVALID
    assert L.cvb_db_match_hamming(ctx.handle, sift.handle, u.ctypes.data, 4, 40.0, 0.8, None, o.ctypes.data, o.ctypes.data,
                                  o.ctypes.data, d.ctypes.data, 8, C.byref(tot)) == CVB_ERR_INVALID
    assert b"holds SIFT" in L.cvb_last_error(ctx.handle)
    assert L.cvb_db_match_l2_dev(ctx.handle, orb.handle, dq.data_ptr(), 4, 500.0, 0.8, dmt.data_ptr(), dmd.data_ptr(),
                                 dnm.data_ptr(), None) == CVB_ERR_INVALID
    assert L.cvb_db_match_hamming_dev(ctx.handle, sift.handle, dq.data_ptr(), 4, 40.0, 0.8, dmt.data_ptr(), dmd.data_ptr(),
                                      dnm.data_ptr(), None) == CVB_ERR_INVALID
    assert ctx.launch_count() == launches and orb.size() == (0, 0) and sift.size() == (0, 0)
    orb.close(); sift.close()


@pytest.mark.parametrize("desc_bytes", [0, 1, 16, 31, 33, 64, 127, 129, 256, -32])
def test_refuses_other_row_sizes(ctx, desc_bytes):
    rc, h = _create(ctx, desc_bytes)
    assert rc == CVB_ERR_UNSUPPORTED and not h.value
    for ok in (32, 128):
        rc, h = _create(ctx, ok)
        assert rc == 0 and h.value
        lib().cvb_db_destroy(ctx.handle, h)
