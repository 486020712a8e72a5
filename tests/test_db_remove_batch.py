"""A batch of keyframes leaves the resident map descriptor database in one call (cvb_db_remove_batch and its group form).

After every removal set three databases must answer alike: the batch, the one-by-one loop of cvb_db_remove from the highest
index down, and a database freshly appended with only the kept keyframes' rows.  Compared bit for bit: cvb_db_size, host
and _dev requests with either matching kernel, host requests truncated by the cap, and a following append, remove and
merge.  Refusals leave the database unchanged and launch nothing; a batch's launches do not depend on how many keyframes
go.  A group of two ranks equals one database after the same sequence, rows_per_rank included."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import covins_b200
from covins_b200 import matching as M
from covins_b200 import optimization as O
from covins_b200 import synth
from covins_b200._lib import lib

CVB_ERR_INVALID = 1
KINDS = {"orb": (32, 40.0, 0.8), "sift": (128, 500.0, 0.8)}
LENS = [1, 127, 128, 129, 300, 1000, 0]          # rows per keyframe in turn, an empty keyframe among them
N_KF = 24


def _keyframes(kind, seed):
    """(query rows, [N_KF] keyframes' rows)"""
    gen = synth.orb_keyframes if kind == "orb" else synth.sift_keyframes
    d, _ = gen(seed=seed, n_kf=N_KF + 3, n_feat=1000, n_lm=1500, window=1500)
    return d[0][:300], [d[i + 1][:LENS[i % len(LENS)]] for i in range(N_KF + 2)]


def _db(ctx, kind, kfs):
    db = M.DescriptorDatabase(ctx, kind=kind)
    if kfs:
        db.append(np.concatenate(kfs), [len(k) for k in kfs])
    return db


def _bits(a):
    return np.ascontiguousarray(a).view(np.int32)


def _raw(db, kind, q, cap):
    """one host request through the C-ABI with an exact cap → (n_matches, 4 outputs incl. the untouched tail, n_total)"""
    dim, thr, ratio = KINDS[kind]
    n_kf = db.size()[0]
    qa = np.ascontiguousarray(q, np.uint8 if kind == "orb" else np.float32).reshape(-1, dim)
    nm = np.full(max(n_kf, 1), -5, np.int32)
    o = [np.full(max(cap, 1), -7, np.int32) for _ in range(3)] + [np.full(max(cap, 1), -7, np.float32)]
    tot = C.c_int32(-1)
    fn = lib().cvb_db_match_hamming if kind == "orb" else lib().cvb_db_match_l2
    assert fn(db.ctx.handle, db.handle, qa.ctypes.data, len(qa), thr, ratio, nm.ctypes.data, *(a.ctypes.data for a in o), cap,
              C.byref(tot)) == 0
    return [nm[:n_kf]] + [_bits(a) for a in o] + [np.array([tot.value])]


def _requests(db, kind, q):
    """the size, and every output of a host and a device request with either matching kernel (the database's own choice,
    then the tensor cores forced), and of host requests whose cap truncates the list"""
    _, thr, ratio = KINDS[kind]
    out = [np.array(db.size(), np.int64)]
    for kernel in (None, "tc"):
        if kernel:
            os.environ["COVINS_B200_MATCH_KERNEL"] = kernel
        try:
            if kind == "orb":
                host = db.match_hamming(q, thr, ratio)
                dev = db.match_hamming_dev(torch.from_numpy(np.ascontiguousarray(q, np.uint8)).cuda(), thr, ratio)
            else:
                host = db.match_l2(q, thr, ratio)
                dev = db.match_l2_dev(torch.from_numpy(np.ascontiguousarray(q, np.float32).astype(np.uint8)).cuda(), thr, ratio)
            torch.cuda.synchronize()
        finally:
            os.environ.pop("COVINS_B200_MATCH_KERNEL", None)
        out += [_bits(a) for a in host] + [t.cpu().numpy().view(np.int32) for t in dev]
    total = len(out[2])
    for cap in sorted({0, 1, total // 2, max(total - 1, 0)}):
        out += _raw(db, kind, q, cap)
    return out


def _same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert x.shape == y.shape and np.array_equal(x, y), (x[:20], y[:20])


def _sets(rng):
    n = N_KF
    return {"none": [], "first": [0], "last": [n - 1], "middle": [n // 2], "all": list(range(n)),
            "every_other": list(range(1, n, 2)), "runs": list(range(3, 7)) + list(range(12, 15)) + [n - 2, n - 1],
            "random30": [int(i) for i in rng.permutation(rng.choice(n, size=int(0.3 * n), replace=False))]}


def test_index_lists_are_checked_before_the_call():
    """the Python wrappers pass int32; a list that is not 1-D integers, or an index that int32 would wrap, is refused"""
    assert M._kf_indices([]).dtype == np.int32 and len(M._kf_indices(())) == 0
    got = M._kf_indices(np.array([7, 0, 3], np.uint64))
    assert got.dtype == np.int32 and got.flags.c_contiguous and got.tolist() == [7, 0, 3]
    assert M._kf_indices(np.arange(10, dtype=np.int64)[::3]).tolist() == [0, 3, 6, 9]
    for bad in ([1.0], [True, False], [[1, 2]], ["1"]):
        with pytest.raises(TypeError):
            M._kf_indices(bad)
    for bad in ([2 ** 31], [-2 ** 31 - 1], np.array([1, 2 ** 40], np.int64)):
        with pytest.raises(ValueError):
            M._kf_indices(bad)
    assert M._kf_indices([-1]).tolist() == [-1]          # in int32: the library refuses it, naming the index


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["orb", "sift"])
@pytest.mark.parametrize("which", ["none", "first", "last", "middle", "all", "every_other", "runs", "random30"])
def test_batch_equals_the_loop_and_a_fresh_database(ctx, kind, which):
    q, kfs = _keyframes(kind, seed=21)
    rm = _sets(np.random.default_rng(5))[which]
    assert which != "random30" or rm != sorted(rm)                     # given unsorted
    base, extra = kfs[:N_KF], kfs[N_KF:]
    batch, loop = _db(ctx, kind, base), _db(ctx, kind, base)
    batch.remove_batch(rm)
    for i in sorted(rm, reverse=True):
        loop.remove(i)
    kept = [k for i, k in enumerate(base) if i not in set(rm)]
    fresh = _db(ctx, kind, kept)
    ref = _requests(fresh, kind, q)
    assert ref[0].tolist() == [len(kept), sum(len(k) for k in kept)]
    assert which == "all" or len(ref[2]) > 20                            # the requests accept matches
    _same(_requests(batch, kind, q), ref)
    _same(_requests(loop, kind, q), ref)
    # then an append, a removal and a merge
    src = _db(ctx, kind, extra[:1] + base[:3])
    for d in (batch, loop, fresh):
        d.append(extra[1], [len(extra[1])])
        if d.size()[0] > 1:
            d.remove(d.size()[0] // 2)
        d.merge(src)
    ref = _requests(fresh, kind, q)
    _same(_requests(batch, kind, q), ref)
    _same(_requests(loop, kind, q), ref)
    for d in (batch, loop, fresh, src):
        d.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["orb", "sift"])
def test_batched_removals_in_turn_and_as_a_merge_source(ctx, kind):
    """two batches in a row equal one loop; a batch-compacted database merged into another equals the host-appended one"""
    q, kfs = _keyframes(kind, seed=22)
    base = kfs[:N_KF]
    batch, loop = _db(ctx, kind, base), _db(ctx, kind, base)
    batch.remove_batch([9, 2, 17])
    batch.remove_batch(np.array([0, 5, 20], np.int64))                   # indices of the database after the first batch
    keep = [i for i in range(N_KF) if i not in (9, 2, 17)]
    keep = [k for j, k in enumerate(keep) if j not in (0, 5, 20)]
    for i in (17, 9, 2):
        loop.remove(i)
    for i in (20, 5, 0):
        loop.remove(i)
    fresh = _db(ctx, kind, [base[i] for i in keep])
    _same(_requests(batch, kind, q), _requests(fresh, kind, q))
    _same(_requests(loop, kind, q), _requests(fresh, kind, q))
    dst, one = _db(ctx, kind, kfs[N_KF:]), _db(ctx, kind, kfs[N_KF:] + [base[i] for i in keep])
    dst.merge(batch)
    _same(_requests(dst, kind, q), _requests(one, kind, q))
    for d in (batch, loop, fresh, dst, one):
        d.close()


@pytest.mark.gpu
def test_refusals_leave_the_database_unchanged_and_launch_nothing(ctx):
    q, kfs = _keyframes("orb", seed=23)
    db = _db(ctx, "orb", kfs[:N_KF])
    before = _requests(db, "orb", q)
    L = lib()

    def call(idx, n):
        a = None if idx is None else np.ascontiguousarray(idx, np.int32)
        return L.cvb_db_remove_batch(ctx.handle, db.handle, None if a is None else a.ctypes.data, n)

    l0 = ctx.launch_count()
    for idx, n, what in (([3, 7, 3], 3, b"index 3 given twice"), ([1, N_KF], 2, b"index 24 out of range"),
                         ([-1], 1, b"index -1 out of range"), ([1, 2], -1, b"negative count n = -1"),
                         (None, 2, b"null index list with n = 2"), ([2, 2 ** 31 - 1], 2, b"out of range")):
        assert call(idx, n) == CVB_ERR_INVALID
        assert what in L.cvb_last_error(ctx.handle), L.cvb_last_error(ctx.handle)
    assert call(None, 0) == 0 and call([5], 0) == 0                     # n == 0: nothing
    assert ctx.launch_count() == l0
    _same(_requests(db, "orb", q), before)
    with pytest.raises(covins_b200.CvbError):
        db.remove_batch([0, 0])
    with pytest.raises(TypeError):
        db.remove_batch([1.5])
    with pytest.raises(ValueError):
        db.remove_batch([1, 2 ** 31])
    _same(_requests(db, "orb", q), before)
    db.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["orb", "sift"])
def test_launches_do_not_depend_on_how_many_go(ctx, kind):
    """one gather launch per array, whether 1, 8 or 20 keyframes go (a kept keyframe follows each set); removing only
    empty keyframes moves nothing"""
    _, kfs = _keyframes(kind, seed=24)
    base = kfs[:N_KF]
    counts = []
    for rm in ([3], [2, 4, 8, 9, 10, 13, 15, 16], list(range(20))):
        db = _db(ctx, kind, base)
        l0 = ctx.launch_count()
        db.remove_batch(rm)
        counts.append(ctx.launch_count() - l0)
        db.close()
    assert counts == [2, 2, 2], counts
    db = _db(ctx, kind, base)
    empty = [i for i, k in enumerate(base) if len(k) == 0]
    assert empty
    l0 = ctx.launch_count()
    db.remove_batch(empty)
    assert ctx.launch_count() == l0 and db.size()[0] == N_KF - len(empty)
    db.close()


# ------------------------------------------------------------------------------------------------------------------ group
def _layouts():
    two = pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two GPUs")
    return [pytest.param(1, id="shared2"), pytest.param(2, id="distinct", marks=two)]


class _Placement:
    """the placement rule replayed: each keyframe to the rank with the fewest rows, the lowest rank on a tie"""

    def __init__(self, n):
        self.rows = np.zeros(n, np.int64)
        self.kf = []

    def append(self, lens):
        for n in lens:
            r = int(np.argmin(self.rows))
            self.rows[r] += n
            self.kf.append((r, n))

    def remove_batch(self, idx):
        for i in sorted(idx, reverse=True):
            r, n = self.kf.pop(i)
            self.rows[r] -= n


@pytest.mark.gpu
@pytest.mark.parametrize("ndev", _layouts())
@pytest.mark.parametrize("kind", ["orb", "sift"])
def test_group_equals_one_database(ctx, kind, ndev):
    _, thr, ratio = KINDS[kind]
    match = "match_hamming" if kind == "orb" else "match_l2"
    q, kfs = _keyframes(kind, seed=25)
    ctxs = [covins_b200.Context(r % ndev) for r in range(2)]
    g = O.Group(ctxs)
    grp = one = None
    try:
        grp, one, place = M.DescriptorDatabaseGroup(g, kind=kind), _db(ctx, kind, []), _Placement(2)

        def append(part):
            rows, lens = np.concatenate(part), [len(k) for k in part]
            grp.append(rows, lens); one.append(rows, lens); place.append(lens)

        def check():
            n_kf, n_rows, per = grp.size_per_rank()
            assert (n_kf, n_rows) == one.size() == (len(place.kf), int(place.rows.sum()))
            assert np.array_equal(per, place.rows)
            got, ref = getattr(grp, match)(q, thr, ratio), getattr(one, match)(q, thr, ratio)
            for a, b in zip(got, ref):
                assert np.array_equal(_bits(a), _bits(b))
            return len(ref[1])

        append(kfs[:N_KF])
        rng = np.random.default_rng(9)
        totals = []
        for rm in ([], [0], [N_KF // 2, 1, N_KF - 2],
                   [int(i) for i in rng.permutation(rng.choice(N_KF - 4, size=6, replace=False))]):
            grp.remove_batch(rm); one.remove_batch(rm); place.remove_batch(rm)
            totals.append(check())
        rank1 = [i for i, (r, _) in enumerate(place.kf) if r == 1]          # every keyframe rank 1 holds
        grp.remove_batch(rank1[::-1]); one.remove_batch(rank1[::-1]); place.remove_batch(rank1)
        assert place.rows[1] == 0
        totals.append(check())
        append(kfs[N_KF:])                                                  # placement follows the new state
        totals.append(check())
        grp.remove(0)
        one.remove(0); place.remove_batch([0])
        totals.append(check())
        assert max(totals) > 20
        launches = [c.launch_count() for c in ctxs]
        for idx, n in (([1, 1], 2), ([0, 10 ** 6], 2), ([0], -1)):
            a = np.ascontiguousarray(idx, np.int32)
            assert lib().cvb_db_group_remove_batch(grp.handle, a.ctypes.data, n) == CVB_ERR_INVALID
        assert lib().cvb_db_group_remove_batch(grp.handle, None, 1) == CVB_ERR_INVALID
        assert [c.launch_count() for c in ctxs] == launches
        check()
    finally:
        for d in (grp, one):                                             # the databases before their group
            if d is not None:
                d.close()
        g.close()
        for c in ctxs:
            c.close()
