"""The resident map descriptor database spread over a rank group (cvb_db_group_*): after every append and remove, a request
gives bit-identical outputs to one DescriptorDatabase fed the same sequence — per-keyframe counts, matches compacted by
(global keyframe, queryIdx), cap truncation and n_total — and the keyframes sit where the placement rule puts them.
Refusals leave every rank unchanged.  Contexts share device 0 unless the layout is "distinct" (one device per rank, skipped
with fewer than two GPUs)."""
import ctypes as C

import numpy as np
import pytest
import torch

import covins_b200
from covins_b200 import matching as M
from covins_b200 import optimization as O
from covins_b200 import synth
from covins_b200._lib import lib

pytestmark = pytest.mark.gpu

CVB_ERR_INVALID, CVB_ERR_UNSUPPORTED = 1, 3
_TWO_GPUS = pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two GPUs")
LAYOUTS = [("shared", 1), ("shared", 2), ("shared", 3), pytest.param(("distinct", 0), marks=_TWO_GPUS)]
KINDS = {"orb": (32, 40.0, 0.8), "sift": (128, 500.0, 0.8)}


class _Grp:
    """n contexts on device 0, or one per visible device (n = 0: every device), and the group over them"""

    def __init__(self, layout):
        kind, n = layout
        ndev = torch.cuda.device_count() if kind == "distinct" else 1
        n = n or min(ndev, 16)
        self.ctxs = [covins_b200.Context(r % ndev) for r in range(n)]
        self.g = O.Group(self.ctxs)

    def close(self):
        self.g.close()
        for c in self.ctxs:
            c.close()


@pytest.fixture(params=LAYOUTS, ids=lambda p: f"{p[0]}{p[1] or ''}")
def grp(request):
    g = _Grp(request.param)
    yield g
    g.close()


def _maps(kind, n_kf, n_feat=300, seed=7):
    if kind == "orb":
        d, _ = synth.orb_keyframes(seed=seed, n_kf=n_kf + 1, n_feat=n_feat, n_lm=600, window=600)
    else:
        d, _ = synth.sift_keyframes(seed=seed, n_kf=n_kf + 1, n_feat=n_feat, n_lm=600, window=600)
    return d[0], [d[i + 1] for i in range(n_kf)]


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.int32) if a.dtype == np.float32 else a.astype(np.int64)


def _assert_same(got, ref):
    assert len(got) == len(ref)
    for a, b in zip(got, ref):
        assert np.array_equal(_bits(a), _bits(b)), (a[:20], b[:20], len(a), len(b))


class _Placement:
    """the placement rule replayed: each keyframe to the rank with the fewest rows, the lowest rank on a tie"""

    def __init__(self, n):
        self.rows = np.zeros(n, np.int64)
        self.kf = []          # global order: (rank, rows)

    def append(self, lens):
        for n in lens:
            r = int(np.argmin(self.rows))       # argmin returns the first minimum
            self.rows[r] += n
            self.kf.append((r, n))

    def remove(self, i):
        r, n = self.kf.pop(i)
        self.rows[r] -= n


def _raw(db, kind, q, cap, nq=None):
    """one host request through the C-ABI with an exact cap → (rc, n_matches, 4 outputs [:cap], n_total)"""
    dim, thr, ratio = KINDS[kind]
    n_kf = db.size()[0]
    qa = np.ascontiguousarray(q, np.uint8 if kind == "orb" else np.float32).reshape(-1, dim)
    nq = len(qa) if nq is None else nq
    nm = np.full(max(n_kf, 1), -5, np.int32)
    o = [np.full(max(cap, 1), -7, np.int32) for _ in range(3)] + [np.full(max(cap, 1), -7, np.float32)]
    tot = C.c_int32(-1)
    if isinstance(db, M.DescriptorDatabaseGroup):
        fn = lib().cvb_db_group_match_hamming if kind == "orb" else lib().cvb_db_group_match_l2
        rc = fn(db.handle, qa.ctypes.data, nq, thr, ratio, nm.ctypes.data, *(a.ctypes.data for a in o), cap, C.byref(tot))
    else:
        fn = lib().cvb_db_match_hamming if kind == "orb" else lib().cvb_db_match_l2
        rc = fn(db.ctx.handle, db.handle, qa.ctypes.data, nq, thr, ratio, nm.ctypes.data, *(a.ctypes.data for a in o), cap,
                C.byref(tot))
    return rc, nm[:n_kf], o, tot.value


def _check(one, db, place, kind, q):
    dim, thr, ratio = KINDS[kind]
    n_kf, n_rows, per = db.size_per_rank()
    assert (n_kf, n_rows) == one.size() == (len(place.kf), int(place.rows.sum()))
    assert np.array_equal(per, place.rows)
    match = "match_hamming" if kind == "orb" else "match_l2"
    ref = getattr(one, match)(q, thr, ratio)
    got = getattr(db, match)(q, thr, ratio)
    _assert_same(got, ref)
    _assert_same(getattr(db, match)(q, thr, ratio), got)                 # repeat: identical bits
    total = len(ref[1])
    for cap in sorted({0, 1, total // 2, max(total - 1, 0)}):            # cap below the total (and 0)
        r1 = _raw(one, kind, q, cap)
        r2 = _raw(db, kind, q, cap)
        assert r1[0] == r2[0] == 0 and r1[3] == r2[3] == total
        assert np.array_equal(r1[1], r2[1])
        for a, b in zip(r1[2], r2[2]):
            assert np.array_equal(_bits(a), _bits(b))                   # same writes, same untouched tail
    r1, r2 = _raw(one, kind, q, 16, nq=0), _raw(db, kind, q, 16, nq=0)  # nq == 0
    assert r1[0] == r2[0] == 0 and r1[3] == r2[3] == 0 and np.array_equal(r1[1], r2[1])
    return total


@pytest.mark.parametrize("kind", ["orb", "sift"])
def test_sequence_equals_single_database(grp, kind):
    """appends in uneven batches (zero-row keyframes included), removals of the first, a middle and the last keyframe and
    of every keyframe one rank holds, then more appends: after every step the group equals one database"""
    q, kfs = _maps(kind, 70)
    lens = ([300, 0, 129, 1, 128, 257, 0, 40, 255, 300, 17] * 7)[:70]
    rows = [k[:n] for k, n in zip(kfs, lens)]
    one = M.DescriptorDatabase(grp.ctxs[0], kind=kind)
    db = M.DescriptorDatabaseGroup(grp.g, kind=kind)
    place = _Placement(grp.g.n)
    dim = KINDS[kind][0]
    _check(one, db, place, kind, q)                                      # empty database

    def append(a, b):
        chunk = np.concatenate(rows[a:b]).reshape(-1, dim)
        one.append(chunk, lens[a:b]); db.append(chunk, lens[a:b]); place.append(lens[a:b])

    def remove(i):
        one.remove(i); db.remove(i); place.remove(i)

    totals = []
    for a, b in ((0, 1), (1, 2), (2, 9), (9, 10), (10, 41), (41, 60)):
        append(a, b)
        totals.append(_check(one, db, place, kind, q))
    for which in ("first", "middle", "last"):
        n = len(place.kf)
        remove({"first": 0, "middle": n // 2, "last": n - 1}[which])
        totals.append(_check(one, db, place, kind, q))
    victim = grp.g.n - 1                                                 # every keyframe of the last rank
    while any(r == victim for r, _ in place.kf):
        remove(next(i for i, (r, _) in enumerate(place.kf) if r == victim))
    assert place.rows[victim] == 0
    totals.append(_check(one, db, place, kind, q))
    append(60, 70)
    totals.append(_check(one, db, place, kind, q))
    assert max(totals) > 50
    db.close(); one.close()


@pytest.mark.parametrize("kind", ["orb", "sift"])
def test_c3_size_equals_single_database(kind):
    """a C3-sized map (2 000 keyframes): the single database scans it with the tensor-core kernel, the ranks' smaller shares
    may take the other kernel; the outputs stay bit-identical for groups of 1, 2 and 3 on one device"""
    nq, n_feat = (1000, 1000) if kind == "orb" else (300, 300)
    if kind == "orb":
        d, _ = synth.orb_keyframes(seed=3, n_kf=2001, n_feat=n_feat)
    else:
        d, _ = synth.sift_keyframes(seed=5, n_kf=2001, n_feat=n_feat)
    q, t = d[0][:nq], d[1:].reshape(-1, KINDS[kind][0])
    ctxs = [covins_b200.Context(0) for _ in range(3)]
    one = M.DescriptorDatabase(ctxs[0], kind=kind)
    one.append(t, [n_feat] * 2000)
    match = "match_hamming" if kind == "orb" else "match_l2"
    ref = getattr(one, match)(q)
    assert ref[0].sum() > 100
    for n in (1, 2, 3):
        g = O.Group(ctxs[:n])
        db = M.DescriptorDatabaseGroup(g, kind=kind)
        db.append(t, [n_feat] * 2000)
        _assert_same(getattr(db, match)(q), ref)
        db.close(); g.close()
    one.close()
    for c in ctxs:
        c.close()


# ------------------------------------------------------------------------------------------------------------ refusals
def _launches(grp):
    return [c.launch_count() for c in grp.ctxs]


def _sizes(*dbs):
    return [(n_kf, n_rows, tuple(per)) for n_kf, n_rows, per in (db.size_per_rank() for db in dbs)]


def test_refusals_leave_every_rank_unchanged(grp):
    q, kfs = _maps("sift", 12, n_feat=200, seed=11)
    sift = M.DescriptorDatabaseGroup(grp.g, kind="sift")
    orb = M.DescriptorDatabaseGroup(grp.g, kind="orb")
    sift.append(np.concatenate(kfs[:9]), [200] * 9)
    orb.append(np.zeros((64, 32), np.uint8), [32, 32])
    before = _sizes(sift, orb)
    ref = sift.match_l2(q)
    launches = _launches(grp)
    L = lib()
    f = np.ascontiguousarray(np.concatenate(kfs[9:]), np.float32)
    u = np.zeros((600, 32), np.uint8)
    rpk = np.array([200, 200, 200], np.int32)
    bad_rpk = np.array([200, -1, 401], np.int32)
    o = np.empty(64, np.int32); d = np.empty(64, np.float32); nm = np.empty(16, np.int32); tot = C.c_int32()
    c0 = grp.ctxs[0].handle

    def msg():
        return L.cvb_last_error(c0)

    # wrong row kind
    assert L.cvb_db_group_append(sift.handle, u.ctypes.data, rpk.ctypes.data, 3) == CVB_ERR_INVALID and b"holds SIFT" in msg()
    assert L.cvb_db_group_append_sift(orb.handle, f.ctypes.data, rpk.ctypes.data, 3) == CVB_ERR_INVALID and b"holds ORB" in msg()
    assert L.cvb_db_group_match_hamming(sift.handle, u.ctypes.data, 4, 40.0, 0.8, None, o.ctypes.data, o.ctypes.data,
                                        o.ctypes.data, d.ctypes.data, 64, C.byref(tot)) == CVB_ERR_INVALID
    assert L.cvb_db_group_match_l2(orb.handle, f.ctypes.data, 4, 500.0, 0.8, None, o.ctypes.data, o.ctypes.data,
                                   o.ctypes.data, d.ctypes.data, 64, C.byref(tot)) == CVB_ERR_INVALID
    # SIFT values that are not integers in [0, 255]: rows and query
    for bad in (0.5, -1.0, 256.0, np.nan, np.inf):
        fb = f.copy(); fb[333, 17] = bad
        assert L.cvb_db_group_append_sift(sift.handle, fb.ctypes.data, rpk.ctypes.data, 3) == CVB_ERR_UNSUPPORTED
        qb = np.ascontiguousarray(q, np.float32).copy(); qb[5, 100] = bad
        assert L.cvb_db_group_match_l2(sift.handle, qb.ctypes.data, len(qb), 500.0, 0.8, nm.ctypes.data, o.ctypes.data,
                                       o.ctypes.data, o.ctypes.data, d.ctypes.data, 64, C.byref(tot)) == CVB_ERR_UNSUPPORTED
    # bad counts, rows and arguments
    assert L.cvb_db_group_append_sift(sift.handle, f.ctypes.data, bad_rpk.ctypes.data, 3) == CVB_ERR_INVALID
    assert L.cvb_db_group_append_sift(sift.handle, None, rpk.ctypes.data, 3) == CVB_ERR_INVALID
    assert L.cvb_db_group_append_sift(sift.handle, f.ctypes.data, None, 3) == CVB_ERR_INVALID
    assert L.cvb_db_group_append_sift(sift.handle, f.ctypes.data, rpk.ctypes.data, -1) == CVB_ERR_INVALID
    qf = np.ascontiguousarray(q, np.float32)
    for nq, cap, out in ((-1, 64, o), (len(qf), -1, o), (len(qf), 64, None)):
        optr = out.ctypes.data if out is not None else None
        assert L.cvb_db_group_match_l2(sift.handle, qf.ctypes.data, nq, 500.0, 0.8, nm.ctypes.data, optr, optr, optr,
                                       d.ctypes.data, cap, C.byref(tot)) == CVB_ERR_INVALID
    # bad indices
    for i in (-1, 9, 1 << 30):
        assert L.cvb_db_group_remove(sift.handle, i) == CVB_ERR_INVALID and b"out of range" in msg()
    assert _launches(grp) == launches
    assert _sizes(sift, orb) == before
    _assert_same(sift.match_l2(q), ref)                                   # the next request is unchanged
    sift.close(); orb.close()


def test_refuses_other_row_sizes(grp):
    for desc_bytes in (0, 16, 64, 129):
        h = C.c_void_p()
        assert lib().cvb_db_group_create(grp.g.h, desc_bytes, C.byref(h)) == CVB_ERR_UNSUPPORTED and not h.value
