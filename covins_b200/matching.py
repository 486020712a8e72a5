"""Host-side mirror of the reference's matching step on top of the C-ABI.

Names follow the reference: `knn_match` is cv::DescriptorMatcher::knnMatch as called in
PlaceRecognitionG::ComputeSE3 (covins_backend/src/covins_backend/placerec_gen_be.cpp:82-100),
`match_candidates` is that call fused with the distance+ratio filter of :102-114 for a list of
candidate keyframes, `landmark_match` is DenseMatcher<LandmarkMatchingAlgorithm> as called in
PlaceRecognition::ComputeSE3 (placerec_be.cpp:85-90).

numpy arrays go through the host-buffer entry points (copies included); torch CUDA tensors go
through the `_dev` entry points on the current torch stream (no copies, no sync).
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._lib import Context, lib


def _np(a, dt):
    return np.ascontiguousarray(a, dtype=dt)


def _ptr(a):
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return a.ctypes.data
    return a.data_ptr()  # torch tensor


def _seg(seg_ptr, n_rows):
    if seg_ptr is None:
        seg_ptr = np.array([0, n_rows], np.int32)
    return _np(seg_ptr, np.int32)


def _kf_indices(indices):
    """a batch of keyframe indices as the contiguous int32 array cvb_db_remove_batch takes; anything that is not a 1-D list
    of integers, or an index outside int32 (which the conversion would wrap onto another keyframe), is refused here"""
    a = np.asarray(indices)
    if a.size == 0:
        return np.zeros(0, np.int32)
    if a.ndim != 1 or not np.issubdtype(a.dtype, np.integer):
        raise TypeError(f"keyframe indices must be a 1-D list of integers, got dtype {a.dtype} and shape {a.shape}")
    lo, hi = np.iinfo(np.int32).min, np.iinfo(np.int32).max
    bad = a[(a < lo) | (a > hi)]
    if bad.size:
        raise ValueError(f"keyframe index {int(bad[0])} is outside int32")
    return np.ascontiguousarray(a, np.int32)


def _is_torch(x):
    return hasattr(x, "data_ptr")


def _torch_stream():
    import torch
    s = torch.cuda.current_stream().cuda_stream
    return s if s else 1  # 0 would select the ctx's own stream; 1 == cudaStreamLegacy (torch's default stream)


# ------------------------------------------------------------------------------------------------
# Hamming k-NN (ORB)
# ------------------------------------------------------------------------------------------------
def knn_match_hamming(ctx: Context, q, t, seg_ptr=None, k: int = 2):
    """→ (idx [n_seg, nq, k] i32 segment-local trainIdx, dist [n_seg, nq, k] i32)."""
    if _is_torch(q):
        import torch
        h_seg = _seg(seg_ptr[1] if isinstance(seg_ptr, tuple) else seg_ptr, t.shape[0])
        d_seg = seg_ptr[0] if isinstance(seg_ptr, tuple) else torch.from_numpy(h_seg).to(q.device)
        ns, nq = len(h_seg) - 1, q.shape[0]
        idx = torch.empty((ns, nq, k), dtype=torch.int32, device=q.device)
        dist = torch.empty((ns, nq, k), dtype=torch.int32, device=q.device)
        ctx.check(lib().cvb_knn_hamming_batch_dev(ctx.handle, _ptr(q), nq, _ptr(t), _ptr(d_seg), _ptr(h_seg), ns, k,
                                                  _ptr(idx), _ptr(dist), _torch_stream()))
        return idx, dist
    q = _np(q, np.uint8); t = _np(t, np.uint8)
    assert q.ndim == 2 and q.shape[1] == 32 and t.shape[1] == 32, "ORB descriptors are 32-byte rows"
    seg = _seg(seg_ptr, len(t))
    ns, nq = len(seg) - 1, len(q)
    idx = np.empty((ns, nq, k), np.int32); dist = np.empty((ns, nq, k), np.int32)
    ctx.check(lib().cvb_knn_hamming_batch(ctx.handle, _ptr(q), nq, _ptr(t), _ptr(seg), ns, k, _ptr(idx), _ptr(dist)))
    return idx, dist


def match_candidates_hamming(ctx: Context, q, t, seg_ptr=None, thr: float = 40.0, ratio: float = 0.8):
    """knnMatch(k=2) + distance/ratio filter (placerec_gen_be.cpp:99-114) per candidate segment.
    → (match_train [n_seg, nq] i32 (-1 = rejected), match_dist [n_seg, nq] f32, n_matches [n_seg] i32).
    Defaults: img_match_thres 40.0, ratio_thres 0.8 (config/config_backend.yaml:38-39)."""
    if _is_torch(q):
        import torch
        h_seg = _seg(seg_ptr[1] if isinstance(seg_ptr, tuple) else seg_ptr, t.shape[0])
        d_seg = seg_ptr[0] if isinstance(seg_ptr, tuple) else torch.from_numpy(h_seg).to(q.device)
        ns, nq = len(h_seg) - 1, q.shape[0]
        mt = torch.empty((ns, nq), dtype=torch.int32, device=q.device)
        md = torch.empty((ns, nq), dtype=torch.float32, device=q.device)
        nm = torch.empty((ns,), dtype=torch.int32, device=q.device)
        ctx.check(lib().cvb_match_hamming_batch_dev(ctx.handle, _ptr(q), nq, _ptr(t), _ptr(d_seg), _ptr(h_seg), ns,
                                                    thr, ratio, _ptr(mt), _ptr(md), _ptr(nm), _torch_stream()))
        return mt, md, nm
    q = _np(q, np.uint8); t = _np(t, np.uint8)
    seg = _seg(seg_ptr, len(t))
    ns, nq = len(seg) - 1, len(q)
    mt = np.empty((ns, nq), np.int32); md = np.empty((ns, nq), np.float32); nm = np.empty(ns, np.int32)
    ctx.check(lib().cvb_match_hamming_batch(ctx.handle, _ptr(q), nq, _ptr(t), _ptr(seg), ns, thr, ratio, _ptr(mt),
                                            _ptr(md), _ptr(nm)))
    return mt, md, nm


class DescriptorDatabase:
    """The merged map's descriptors resident in HBM (cvb_db_*): keyframes are appended once, a place-recognition
    request (placerec_gen_be.cpp:60-135) uploads only the query keyframe and downloads only the accepted matches.
    kind="orb": 32-byte rows, match_hamming[_dev]; kind="sift": CV_32F rows x 128 kept as exact u8, match_l2[_dev]."""

    def __init__(self, ctx: Context, reserve_rows: int = 0, kind: str = "orb"):
        import ctypes as C
        assert kind in ("orb", "sift"), kind
        self.ctx = ctx
        self.kind = kind
        self._dim = 32 if kind == "orb" else 128
        h = C.c_void_p()
        ctx.check(lib().cvb_db_create(ctx.handle, self._dim, C.byref(h)))
        self.handle = h
        self._cap = 1 << 16
        if reserve_rows:
            ctx.check(lib().cvb_db_reserve(ctx.handle, self.handle, int(reserve_rows)))

    def append(self, rows, rows_per_kf):
        """rows = the descriptor matrices of the new keyframes, concatenated: u8 [sum(rows_per_kf), 32] (ORB) or float32
        [sum(rows_per_kf), 128] (SIFT, integer-valued in [0,255])."""
        rpk = np.ascontiguousarray(np.asarray(rows_per_kf, np.int32).reshape(-1))
        if self.kind == "orb":
            rows = _np(rows, np.uint8).reshape(-1, 32)
            fn = lib().cvb_db_append
        else:
            rows = _np(rows, np.float32).reshape(-1, 128)
            fn = lib().cvb_db_append_sift
        assert int(rpk.sum()) == len(rows), "rows_per_kf does not add up to the number of rows"
        self.ctx.check(fn(self.ctx.handle, self.handle, _ptr(rows), _ptr(rpk), len(rpk)))

    def remove(self, kf_index: int):
        """a keyframe leaves the map (culling / erase): later keyframes move down by one index"""
        self.ctx.check(lib().cvb_db_remove(self.ctx.handle, self.handle, int(kf_index)))

    def remove_batch(self, indices):
        """a batch of keyframes leaves the map in one call (cvb_db_remove_batch): indices as before the call, in any order;
        the result equals remove() of each from the highest to the lowest.  A survivor's index drops by the number of
        removed indices below it."""
        idx = _kf_indices(indices)
        self.ctx.check(lib().cvb_db_remove_batch(self.ctx.handle, self.handle, _ptr(idx), len(idx)))

    def merge(self, other: "DescriptorDatabase"):
        """two agents' maps are merged: other's keyframes are appended after this database's, in other's order, copied
        device to device (cvb_db_merge; no descriptor crosses PCIe).  other is left unchanged.  Both must be of one kind and
        on one Context."""
        self.ctx.check(lib().cvb_db_merge(self.ctx.handle, self.handle, other.handle))

    def size(self):
        import ctypes as C
        n_kf, n_rows = C.c_int32(), C.c_int64()
        self.ctx.check(lib().cvb_db_size(self.handle, C.byref(n_kf), C.byref(n_rows)))
        return n_kf.value, n_rows.value

    def _match(self, fn, q, thr, ratio):
        import ctypes as C
        n_kf, _ = self.size()
        nm = np.zeros(n_kf, np.int32)
        while True:
            cap = self._cap
            out = [np.empty(cap, np.int32), np.empty(cap, np.int32), np.empty(cap, np.int32), np.empty(cap, np.float32)]
            tot = C.c_int32()
            self.ctx.check(fn(self.ctx.handle, self.handle, _ptr(q), len(q), thr, ratio, _ptr(nm), _ptr(out[0]), _ptr(out[1]),
                              _ptr(out[2]), _ptr(out[3]), cap, C.byref(tot)))
            if tot.value <= cap:
                return (nm,) + tuple(o[:tot.value] for o in out)
            self._cap = int(tot.value * 1.25) + 16

    def _match_dev(self, fn, q, thr, ratio):
        import torch
        n_kf, _ = self.size()
        nq = q.shape[0]
        mt = torch.empty((n_kf, nq), dtype=torch.int32, device=q.device)
        md = torch.empty((n_kf, nq), dtype=torch.float32, device=q.device)
        nm = torch.empty((n_kf,), dtype=torch.int32, device=q.device)
        self.ctx.check(fn(self.ctx.handle, self.handle, _ptr(q), nq, thr, ratio, _ptr(mt), _ptr(md), _ptr(nm), _torch_stream()))
        return mt, md, nm

    def match_hamming(self, q, thr: float = 40.0, ratio: float = 0.8):
        """→ (n_matches [n_kf] i32, m_kf, m_query, m_train (keyframe-local), m_dist): the accepted matches ordered by
        (keyframe, queryIdx) — per keyframe the reference's img_matches vector."""
        return self._match(lib().cvb_db_match_hamming, _np(q, np.uint8).reshape(-1, 32), thr, ratio)

    def match_hamming_dev(self, q, thr: float = 40.0, ratio: float = 0.8):
        """device request: q = CUDA torch tensor u8 [nq, 32] → (match_train [n_kf, nq] i32, match_dist [n_kf, nq] f32,
        n_matches [n_kf] i32) as CUDA tensors; no copies (cvb_db_match_hamming_dev)."""
        return self._match_dev(lib().cvb_db_match_hamming_dev, q, thr, ratio)

    def match_l2(self, q, thr: float = 500.0, ratio: float = 0.8):
        """SIFT database: q = float32 [nq, 128] (integer-valued in [0,255]) → the outputs of match_hamming, with the
        semantics of match_candidates_l2 per keyframe (img_match_thres 500 for SIFT, config_backend.yaml:38)."""
        return self._match(lib().cvb_db_match_l2, _np(q, np.float32).reshape(-1, 128), thr, ratio)

    def match_l2_dev(self, q, thr: float = 500.0, ratio: float = 0.8):
        """SIFT database, device request: q = CUDA torch tensor u8 [nq, 128] (see quantize_u8) → the outputs of
        match_hamming_dev (cvb_db_match_l2_dev)."""
        return self._match_dev(lib().cvb_db_match_l2_dev, q, thr, ratio)

    def close(self):
        if self.handle:
            lib().cvb_db_destroy(self.ctx.handle, self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class DescriptorDatabaseGroup:
    """DescriptorDatabase with its keyframes spread over the ranks of an optimization.Group (cvb_db_group_*): each appended
    keyframe goes to the rank holding the fewest rows (the lowest rank on a tie), and a request scans every rank's share
    on that rank.  Indices, removals and the host requests' outputs are bit-identical to one DescriptorDatabase fed the same
    appends and removes.  Give it a group of its own: its requests are serialised with every other call on the group.
    The group must outlive the database."""

    def __init__(self, group, kind: str = "orb"):
        assert kind in ("orb", "sift"), kind
        self.group = group
        self.ctx = group.ctx          # rank 0's context carries the messages
        self.kind = kind
        h = C.c_void_p()
        self.ctx.check(lib().cvb_db_group_create(group.h, 32 if kind == "orb" else 128, C.byref(h)))
        self.handle = h
        self._cap = 1 << 16

    def append(self, rows, rows_per_kf):
        """as DescriptorDatabase.append"""
        rpk = np.ascontiguousarray(np.asarray(rows_per_kf, np.int32).reshape(-1))
        if self.kind == "orb":
            rows = _np(rows, np.uint8).reshape(-1, 32)
            fn = lib().cvb_db_group_append
        else:
            rows = _np(rows, np.float32).reshape(-1, 128)
            fn = lib().cvb_db_group_append_sift
        assert int(rpk.sum()) == len(rows), "rows_per_kf does not add up to the number of rows"
        self.ctx.check(fn(self.handle, _ptr(rows), _ptr(rpk), len(rpk)))

    def remove(self, kf_index: int):
        """a keyframe leaves the map: later keyframes move down by one global index"""
        self.ctx.check(lib().cvb_db_group_remove(self.handle, int(kf_index)))

    def remove_batch(self, indices):
        """as DescriptorDatabase.remove_batch; each rank compacts its share on its own device (cvb_db_group_remove_batch)"""
        idx = _kf_indices(indices)
        self.ctx.check(lib().cvb_db_group_remove_batch(self.handle, _ptr(idx), len(idx)))

    def merge(self, other: "DescriptorDatabaseGroup"):
        """as DescriptorDatabase.merge, rank by rank on the group's devices (cvb_db_group_merge): other's keyframes follow
        this database's in global order, each staying on the rank that holds it.  Both must be on one Group."""
        self.ctx.check(lib().cvb_db_group_merge(self.handle, other.handle))

    def size(self):
        """→ (n_kf, n_rows)"""
        return self.size_per_rank()[:2]

    def size_per_rank(self):
        """→ (n_kf, n_rows, rows_per_rank int64 [group size])"""
        n_kf, n_rows = C.c_int32(), C.c_int64()
        per = np.zeros(self.group.n, np.int64)
        self.ctx.check(lib().cvb_db_group_size(self.handle, C.byref(n_kf), C.byref(n_rows), _ptr(per)))
        return n_kf.value, n_rows.value, per

    def _match(self, fn, q, thr, ratio):
        n_kf, _ = self.size()
        nm = np.zeros(n_kf, np.int32)
        while True:
            cap = self._cap
            out = [np.empty(cap, np.int32), np.empty(cap, np.int32), np.empty(cap, np.int32), np.empty(cap, np.float32)]
            tot = C.c_int32()
            self.ctx.check(fn(self.handle, _ptr(q), len(q), thr, ratio, _ptr(nm), _ptr(out[0]), _ptr(out[1]), _ptr(out[2]),
                              _ptr(out[3]), cap, C.byref(tot)))
            if tot.value <= cap:
                return (nm,) + tuple(o[:tot.value] for o in out)
            self._cap = int(tot.value * 1.25) + 16

    def match_hamming(self, q, thr: float = 40.0, ratio: float = 0.8):
        """as DescriptorDatabase.match_hamming, m_kf = global keyframe index"""
        return self._match(lib().cvb_db_group_match_hamming, _np(q, np.uint8).reshape(-1, 32), thr, ratio)

    def match_l2(self, q, thr: float = 500.0, ratio: float = 0.8):
        """as DescriptorDatabase.match_l2, m_kf = global keyframe index"""
        return self._match(lib().cvb_db_group_match_l2, _np(q, np.float32).reshape(-1, 128), thr, ratio)

    def close(self):
        if self.handle:
            lib().cvb_db_group_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# ------------------------------------------------------------------------------------------------
# L2 k-NN (SIFT)
# ------------------------------------------------------------------------------------------------
def knn_match_l2(ctx: Context, q, t, seg_ptr=None, k: int = 2):
    """float32 rows (host) → (idx [n_seg,nq,k] i32, dist [n_seg,nq,k] f32 = sqrt(sum (a-b)^2))."""
    if _is_torch(q):
        import torch
        assert q.dtype == torch.uint8, "device path takes the HBM-resident u8 layout (see quantize_u8)"
        h_seg = _seg(seg_ptr[1] if isinstance(seg_ptr, tuple) else seg_ptr, t.shape[0])
        d_seg = seg_ptr[0] if isinstance(seg_ptr, tuple) else torch.from_numpy(h_seg).to(q.device)
        ns, nq = len(h_seg) - 1, q.shape[0]
        idx = torch.empty((ns, nq, k), dtype=torch.int32, device=q.device)
        dist = torch.empty((ns, nq, k), dtype=torch.float32, device=q.device)
        ctx.check(lib().cvb_knn_l2_u8_batch_dev(ctx.handle, _ptr(q), nq, _ptr(t), _ptr(d_seg), _ptr(h_seg), ns,
                                                q.shape[1], k, _ptr(idx), _ptr(dist), _torch_stream()))
        return idx, dist
    q = _np(q, np.float32); t = _np(t, np.float32)
    seg = _seg(seg_ptr, len(t))
    ns, nq = len(seg) - 1, len(q)
    idx = np.empty((ns, nq, k), np.int32); dist = np.empty((ns, nq, k), np.float32)
    ctx.check(lib().cvb_knn_l2_batch(ctx.handle, _ptr(q), nq, _ptr(t), _ptr(seg), ns, q.shape[1], k, _ptr(idx),
                                     _ptr(dist)))
    return idx, dist


def match_candidates_l2(ctx: Context, q, t, seg_ptr=None, thr: float = 500.0, ratio: float = 0.8):
    """SIFT branch of placerec_gen_be.cpp:86-114 (img_match_thres 500 for SIFT, config_backend.yaml:38)."""
    q = _np(q, np.float32); t = _np(t, np.float32)
    seg = _seg(seg_ptr, len(t))
    ns, nq = len(seg) - 1, len(q)
    mt = np.empty((ns, nq), np.int32); md = np.empty((ns, nq), np.float32); nm = np.empty(ns, np.int32)
    ctx.check(lib().cvb_match_l2_batch(ctx.handle, _ptr(q), nq, _ptr(t), _ptr(seg), ns, q.shape[1], thr, ratio,
                                       _ptr(mt), _ptr(md), _ptr(nm)))
    return mt, md, nm


def shard_rows(n_rows_total: int, world: int, seg_ptr=None):
    """Contiguous row ranges of the map-wide database per rank.  With seg_ptr (keyframe boundaries) the cuts fall on
    keyframe boundaries (SURVEY §8e: sharded by KF block); → int64 [world+1] row offsets."""
    if seg_ptr is None:
        return np.linspace(0, n_rows_total, world + 1).astype(np.int64)
    seg = np.asarray(seg_ptr, np.int64)
    target = np.linspace(0, n_rows_total, world + 1)
    cut = seg[np.searchsorted(seg, target, side="left").clip(0, len(seg) - 1)]
    cut[0], cut[-1] = 0, n_rows_total
    return np.maximum.accumulate(cut)


def knn_merge_shards(ctx: Context, idx_all, dist_all, row_offset, k: int):
    """idx_all/dist_all: torch [G, n, k] (shard-local trainIdx; int32 Hamming or float32 L2 distances), row_offset
    torch int32 [G] → merged (idx [n, k] global trainIdx, dist [n, k]), cvb_knn_merge_shards_dev."""
    import torch
    G, n = idx_all.shape[0], idx_all.shape[1]
    idx_all = idx_all.contiguous(); dist_all = dist_all.contiguous()
    out_i = torch.empty((n, k), dtype=torch.int32, device=idx_all.device)
    out_d = torch.empty((n, k), dtype=dist_all.dtype, device=idx_all.device)
    ctx.check(lib().cvb_knn_merge_shards_dev(ctx.handle, _ptr(idx_all), _ptr(dist_all),
                                             1 if dist_all.dtype == torch.float32 else 0, _ptr(row_offset), G, n, k,
                                             _ptr(out_i), _ptr(out_d), _torch_stream()))
    return out_i, out_d


def knn_match_sharded(ctx: Context, q, t_local, row_offset: int, k: int = 2, metric: str = "hamming", group=None):
    """Map-wide k-NN, database sharded over the ranks of `group` (torch.distributed, NCCL): local top-k on this rank's
    rows, ONE all-gather of the (idx, dist) lists (G*k*nq*8 B) and the shard offsets, local merge (SURVEY §8e).
    q replicated on every rank (torch u8 on the device); t_local = this rank's rows; row_offset = its first global row.
    Every rank returns the same (idx [nq,k] global trainIdx, dist [nq,k])."""
    import torch
    import torch.distributed as dist
    if metric == "hamming":
        li, ld = knn_match_hamming(ctx, q, t_local, None, k)
    else:
        li, ld = knn_match_l2(ctx, q, t_local, None, k)
    li, ld = li[0].contiguous(), ld[0].contiguous()          # one segment = the whole shard
    world = dist.get_world_size(group)
    idx_all = torch.empty((world,) + tuple(li.shape), dtype=li.dtype, device=li.device)
    dist_all = torch.empty((world,) + tuple(ld.shape), dtype=ld.dtype, device=ld.device)
    off = torch.tensor([row_offset], dtype=torch.int32, device=li.device)
    off_all = torch.empty((world,), dtype=torch.int32, device=li.device)
    dist.all_gather_into_tensor(idx_all, li, group=group)
    dist.all_gather_into_tensor(dist_all, ld, group=group)
    dist.all_gather_into_tensor(off_all, off, group=group)
    return knn_merge_shards(ctx, idx_all, dist_all, off_all, k)


def quantize_u8(ctx: Context, x):
    """torch f32 CUDA tensor → (u8 tensor, bad flag tensor): the exact HBM-resident SIFT layout."""
    import torch
    out = torch.empty(x.shape, dtype=torch.uint8, device=x.device)
    bad = torch.zeros(1, dtype=torch.int32, device=x.device)
    ctx.check(lib().cvb_quantize_u8_dev(ctx.handle, _ptr(x), x.numel(), _ptr(out), _ptr(bad), _torch_stream()))
    return out, bad


# ------------------------------------------------------------------------------------------------
# DenseMatcher<LandmarkMatchingAlgorithm> (COVINS mode)
# ------------------------------------------------------------------------------------------------
def landmark_match(ctx: Context, A, skipA, B, skipB, seg_ptr=None, thr: float = 50.0, num_best: int = 4):
    """→ list over candidate segments of (idxA, idxB, dist) arrays ordered by idxB — the `Matches`
    vector of placerec_be.cpp:91 — for numpy inputs; for torch inputs the raw
    (outA, outB, outD, n_out) device tensors (slice [seg_ptr[s], seg_ptr[s]+n_out[s]))."""
    if _is_torch(A):
        import torch
        h_seg = _seg(seg_ptr[1] if isinstance(seg_ptr, tuple) else seg_ptr, B.shape[0])
        d_seg = seg_ptr[0] if isinstance(seg_ptr, tuple) else torch.from_numpy(h_seg).to(A.device)
        ns, rows = len(h_seg) - 1, B.shape[0]
        oA = torch.empty(rows, dtype=torch.int32, device=A.device)
        oB = torch.empty(rows, dtype=torch.int32, device=A.device)
        oD = torch.empty(rows, dtype=torch.float32, device=A.device)
        n = torch.empty(ns, dtype=torch.int32, device=A.device)
        ctx.check(lib().cvb_landmark_match_batch_dev(ctx.handle, _ptr(A), _ptr(skipA), A.shape[0], _ptr(B), _ptr(skipB),
                                                     _ptr(d_seg), _ptr(h_seg), ns, thr, num_best, _ptr(oA), _ptr(oB),
                                                     _ptr(oD), _ptr(n), _torch_stream()))
        return oA, oB, oD, n
    A = _np(A, np.uint8); B = _np(B, np.uint8)
    sA = _np(skipA, np.uint8) if skipA is not None else None
    sB = _np(skipB, np.uint8) if skipB is not None else None
    seg = _seg(seg_ptr, len(B))
    ns, rows = len(seg) - 1, len(B)
    oA = np.empty(max(rows, 1), np.int32); oB = np.empty(max(rows, 1), np.int32); oD = np.empty(max(rows, 1), np.float32)
    n = np.empty(ns, np.int32)
    ctx.check(lib().cvb_landmark_match_batch(ctx.handle, _ptr(A), _ptr(sA), len(A), _ptr(B), _ptr(sB), _ptr(seg), ns,
                                             thr, num_best, _ptr(oA), _ptr(oB), _ptr(oD), _ptr(n)))
    out = []
    for s in range(ns):
        a, b = seg[s], seg[s] + n[s]
        out.append((oA[a:b].copy(), oB[a:b].copy(), oD[a:b].copy()))
    return out


def landmark_descriptors(ctx: Context, cand, lm_ptr, old_desc=None):
    """Landmark::ComputeDescriptor for a batch of landmarks (landmark_be.cpp:49-92): cand u8 [rows, 32] = descriptor rows
    of the valid observers of every landmark, concatenated; lm_ptr i32 [n_lm+1].  → (best_idx [n_lm] i32 (-1 = landmark
    without observers), desc [n_lm, 32] u8; rows of landmarks without observers keep old_desc (zeros if not given))."""
    if _is_torch(cand):
        import torch
        n = lm_ptr.shape[0] - 1
        best = torch.empty((n,), dtype=torch.int32, device=cand.device)
        out = old_desc.clone() if old_desc is not None else torch.zeros((n, 32), dtype=torch.uint8, device=cand.device)
        ctx.check(lib().cvb_landmark_descriptor_batch_dev(ctx.handle, _ptr(cand), _ptr(lm_ptr), n, _ptr(best), _ptr(out),
                                                          _torch_stream()))
        return best, out
    cand = _np(cand, np.uint8).reshape(-1, 32); lm_ptr = np.ascontiguousarray(lm_ptr, np.int32)
    n = len(lm_ptr) - 1
    best = np.empty(n, np.int32)
    out = np.ascontiguousarray(old_desc, np.uint8).copy() if old_desc is not None else np.zeros((n, 32), np.uint8)
    ctx.check(lib().cvb_landmark_descriptor_batch(ctx.handle, _ptr(cand), _ptr(lm_ptr), n, _ptr(best), _ptr(out)))
    return best, out


def microbench_popc(ctx: Context, iters: int = 20000) -> float:
    v = C.c_double()
    ctx.check(lib().cvb_microbench_popc(ctx.handle, iters, C.byref(v)))
    return v.value
