"""GPU parity tests of the matching half, all through the C-ABI (covins_b200.matching → libcovins_b200.so):
bit-exact against (1) the committed cv2.BFMatcher golden vectors, (2) the CPU oracle on seeded inputs,
(3) size-independent properties at BASELINE.json's full sizes."""
import os

import numpy as np
import pytest

from conftest import golden_cases
from covins_b200 import matching as M
from covins_b200 import synth
from oracle import knn as ora

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------- golden
def test_hamming_knn_matches_cv2_golden(ctx, golden_dir):
    g, names = golden_cases(os.path.join(golden_dir, "knn_hamming.npz"))
    for n in names:
        idx, dist = M.knn_match_hamming(ctx, g[n + "/q"], g[n + "/t"], k=2)
        assert np.array_equal(idx[0], g[n + "/idx"]), n
        d = np.where(idx[0] >= 0, dist[0].astype(np.float32), np.inf)
        assert np.array_equal(d, g[n + "/dist"]), n
        mt, md, nm = M.match_candidates_hamming(ctx, g[n + "/q"], g[n + "/t"], thr=40.0, ratio=0.8)
        assert np.array_equal(mt[0], g[n + "/match"]), n
        assert nm[0] == (g[n + "/match"] >= 0).sum()


def test_l2_knn_matches_cv2_golden(ctx, golden_dir):
    g, names = golden_cases(os.path.join(golden_dir, "knn_l2.npz"))
    for n in names:
        q = g[n + "/q"].astype(np.float32); t = g[n + "/t"].astype(np.float32)
        idx, dist = M.knn_match_l2(ctx, q, t, k=2)
        assert np.array_equal(idx[0], g[n + "/idx"]), n
        d = np.where(idx[0] >= 0, dist[0], np.inf)
        assert np.array_equal(d, g[n + "/dist"]), n  # bit-exact float distances
        mt, md, nm = M.match_candidates_l2(ctx, q, t, thr=500.0, ratio=0.8)
        assert np.array_equal(mt[0], g[n + "/match"]), n


# ---------------------------------------------------------------------------------------------- oracle
@pytest.mark.parametrize("k", [1, 2, 3, 4])
def test_hamming_batch_ragged_vs_oracle(ctx, k):
    rng = np.random.default_rng(10 + k)
    desc, _ = synth.orb_keyframes(seed=5, n_kf=9, n_feat=700, n_lm=1500, window=1500)
    q = desc[0][:613]
    lens = [700, 0, 1, 2, 3, 257, 512, 699]
    t = np.concatenate([desc[i + 1][:l] for i, l in enumerate(lens)])
    seg = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    idx, dist = M.knn_match_hamming(ctx, q, t, seg, k=k)
    ri, rd = ora.knn_hamming_batch(q, t, seg, k=k)
    assert np.array_equal(idx, ri) and np.array_equal(dist, rd)


def test_hamming_split_path_vs_oracle(ctx):
    """one long segment, few queries → row-split + merge path; heavy ties to stress the merge rule"""
    rng = np.random.default_rng(42)
    base = rng.integers(0, 256, (40, 32), dtype=np.uint8)
    t = base[rng.integers(0, 40, 50_000)]
    t ^= (rng.integers(0, 256, t.shape, dtype=np.uint8) & rng.integers(0, 256, t.shape, dtype=np.uint8)
          & rng.integers(0, 256, t.shape, dtype=np.uint8) & rng.integers(0, 256, t.shape, dtype=np.uint8) & 3)
    q = base[rng.integers(0, 40, 37)]
    for k in (2, 4):
        idx, dist = M.knn_match_hamming(ctx, q, t, None, k=k)
        ri, rd = ora.knn_hamming(q, t, k=k)
        assert np.array_equal(idx[0], ri) and np.array_equal(dist[0], rd)
    mt, md, nm = M.match_candidates_hamming(ctx, q, t, None, 40.0, 0.8)
    ri, rd = ora.knn_hamming(q, t, k=2)
    rmt, rmd, rc = ora.ratio_filter(ri, rd.astype(np.float32), 40.0, 0.8)
    assert np.array_equal(mt[0], rmt) and nm[0] == rc


def test_fused_filter_vs_oracle(ctx):
    desc, _ = synth.orb_keyframes(seed=7, n_kf=21, n_feat=500, n_lm=900, window=900)
    q = desc[0]
    t = desc[1:].reshape(-1, 32)
    seg = synth.seg_ptr_uniform(20, 500)
    mt, md, nm = M.match_candidates_hamming(ctx, q, t, seg, 40.0, 0.8)
    ri, rd = ora.knn_hamming_batch(q, t, seg, k=2)
    rmt, rmd, rc = ora.ratio_filter(ri, rd.astype(np.float32), 40.0, 0.8)
    assert np.array_equal(mt, rmt) and np.array_equal(nm, rc)
    assert np.array_equal(md[mt >= 0], rmd[rmt >= 0])
    assert nm.max() > 25  # covisible neighbours clear placerec.matches_thres (config_backend.yaml:74)


def test_l2_batch_and_split_vs_oracle(ctx):
    s, _ = synth.sift_keyframes(seed=3, n_kf=7, n_feat=300, n_lm=500, window=500)
    q = s[0][:211]
    lens = [300, 0, 2, 129, 300, 77]
    t = np.concatenate([s[i + 1][:l] for i, l in enumerate(lens)])
    seg = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    for k in (1, 2, 4):
        idx, dist = M.knn_match_l2(ctx, q, t, seg, k=k)
        ri, rd = ora.knn_l2_batch(q, t, seg, k=k)
        rd = np.where(ri >= 0, rd, np.finfo(np.float32).max)
        assert np.array_equal(idx, ri) and np.array_equal(dist, rd)
    # long single segment with duplicated rows (ties in the sqrt domain) → split path
    rng = np.random.default_rng(0)
    tl = s.reshape(-1, 128)[rng.integers(0, 400, 20_000)]
    idx, dist = M.knn_match_l2(ctx, q[:19], tl, None, k=2)
    ri, rd = ora.knn_l2(q[:19], tl, k=2)
    assert np.array_equal(idx[0], ri) and np.array_equal(dist[0], rd)


def test_l2_rejects_non_integer_descriptors(ctx):
    import covins_b200
    q = np.full((4, 128), 0.5, np.float32); t = np.zeros((8, 128), np.float32)
    with pytest.raises(covins_b200.CvbError):
        M.knn_match_l2(ctx, q, t)
    with pytest.raises(covins_b200.CvbError):
        M.knn_match_l2(ctx, np.zeros((4, 64), np.float32), np.zeros((8, 64), np.float32))


@pytest.mark.parametrize("seed", [0, 1])
def test_landmark_match_vs_oracle(ctx, seed):
    desc, lm = synth.orb_keyframes(seed=20 + seed, n_kf=13, n_feat=600, n_lm=800, window=800)
    A, skipA = desc[0], (lm[0] < 0).astype(np.uint8)
    lens = [600, 0, 1, 333, 600, 600, 45, 600, 600, 600, 600, 599]
    B = np.concatenate([desc[i + 1][:l] for i, l in enumerate(lens)])
    skipB = np.concatenate([(lm[i + 1][:l] < 0) for i, l in enumerate(lens)]).astype(np.uint8)
    seg = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    out = M.landmark_match(ctx, A, skipA, B, skipB, seg, thr=50.0, num_best=4)
    tot = 0
    for s in range(len(lens)):
        ra, rb, rd = ora.landmark_match(A, skipA, B[seg[s]:seg[s + 1]], skipB[seg[s]:seg[s + 1]], 50.0, 4)
        a, b, d = out[s]
        assert np.array_equal(a, ra) and np.array_equal(b, rb) and np.array_equal(d, rd), s
        tot += len(ra)
    assert tot > 100


def test_landmark_match_ties_and_displacement_chains(ctx):
    rng = np.random.default_rng(5)
    base = rng.integers(0, 256, (10, 32), dtype=np.uint8)

    def mk(n):
        d = base[rng.integers(0, 10, n)].copy()
        return d ^ (rng.integers(0, 256, (n, 32), dtype=np.uint8) & rng.integers(0, 256, (n, 32), dtype=np.uint8)
                    & rng.integers(0, 256, (n, 32), dtype=np.uint8))
    for nb in (1, 2, 4):
        A, B = mk(200), mk(260)
        skipA = (rng.random(200) < 0.2).astype(np.uint8); skipB = (rng.random(260) < 0.2).astype(np.uint8)
        (a, b, d), = M.landmark_match(ctx, A, skipA, B, skipB, None, 50.0, nb)
        ra, rb, rd = ora.landmark_match(A, skipA, B, skipB, 50.0, nb)
        assert np.array_equal(a, ra) and np.array_equal(b, rb) and np.array_equal(d, rd)
    # no skip masks at all
    (a, b, d), = M.landmark_match(ctx, A, None, B, None, None, 50.0, 4)
    ra, rb, rd = ora.landmark_match(A, None, B, None, 50.0, 4)
    assert np.array_equal(a, ra) and np.array_equal(b, rb)


def test_landmark_match_large_shared_memory_on_two_devices(ctx):
    """The DenseMatcher's assignment kernel needs more than 48 KB of dynamic shared memory here ((2 nA num_best + 2 max_len)
    int32), which each device has to allow separately: the same call on device 0, then on device 1."""
    import torch
    import covins_b200
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    desc, lm = synth.orb_keyframes(seed=31, n_kf=3, n_feat=2000, n_lm=3000, window=3000)
    A, skipA = desc[0], (lm[0] < 0).astype(np.uint8)
    B, skipB = desc[1:].reshape(-1, 32), (lm[1:] < 0).reshape(-1).astype(np.uint8)
    seg = synth.seg_ptr_uniform(2, 2000)
    assert (2 * len(A) * 4 + 2 * 2000) * 4 > 48 * 1024
    ref = [ora.landmark_match(A, skipA, B[seg[s]:seg[s + 1]], skipB[seg[s]:seg[s + 1]], 50.0, 4) for s in range(2)]
    assert sum(len(r[0]) for r in ref) > 100
    ctx1 = covins_b200.Context(1)
    try:
        for c in (ctx, ctx1):
            out = M.landmark_match(c, A, skipA, B, skipB, seg, thr=50.0, num_best=4)
            for s in range(2):
                assert all(np.array_equal(x, r) for x, r in zip(out[s], ref[s])), (c.device, s)
    finally:
        ctx1.close()


# ---------------------------------------------------------------------------------------------- device path
def test_device_path_equals_host_path(ctx):
    import torch
    desc, lm = synth.orb_keyframes(seed=9, n_kf=6, n_feat=400, n_lm=600, window=600)
    q = desc[0]; t = desc[1:].reshape(-1, 32); seg = synth.seg_ptr_uniform(5, 400)
    hi, hd = M.knn_match_hamming(ctx, q, t, seg, 2)
    dq = torch.from_numpy(q).cuda(); dt = torch.from_numpy(t).cuda()
    di, dd = M.knn_match_hamming(ctx, dq, dt, seg, 2)
    torch.cuda.synchronize()
    assert np.array_equal(di.cpu().numpy(), hi) and np.array_equal(dd.cpu().numpy(), hd)
    mt, md, nm = M.match_candidates_hamming(ctx, dq, dt, seg)
    hmt, hmd, hnm = M.match_candidates_hamming(ctx, q, t, seg)
    torch.cuda.synchronize()
    assert np.array_equal(mt.cpu().numpy(), hmt) and np.array_equal(nm.cpu().numpy(), hnm)


# ---------------------------------------------------------------------------------------------- full size
def test_full_size_properties_c3(ctx):
    """BASELINE config 3 size: one 1000-feature query KF against 2000 candidate KFs (2 Gpair).
    Properties: (a) the candidate that IS the query returns idx == own row, distance 0 for every row and
    passes the ratio test wherever the row is unique; (b) permuting candidate order permutes the result;
    (c) a sample of 16 candidates equals the oracle bit-for-bit."""
    import torch
    n_kf, nf = 2000, 1000
    g = torch.Generator(device="cuda").manual_seed(1)
    t = torch.randint(0, 256, (n_kf * nf, 32), dtype=torch.uint8, device="cuda", generator=g)
    q = t[777 * nf:778 * nf].clone()
    seg = synth.seg_ptr_uniform(n_kf, nf)
    idx, dist = M.knn_match_hamming(ctx, q, t, seg, 2)
    mt, md, nm = M.match_candidates_hamming(ctx, q, t, seg)
    torch.cuda.synchronize()
    own = idx[777, :, 0].cpu().numpy()
    assert np.array_equal(own, np.arange(nf)) and int(dist[777, :, 0].max()) == 0
    assert int(nm[777]) == nf and int(nm.sum()) == nf  # random codes: nothing else passes thr 40
    perm = torch.randperm(n_kf, device="cuda", generator=g)
    tp = t.view(n_kf, nf, 32)[perm].reshape(-1, 32).contiguous()
    idx_p, dist_p = M.knn_match_hamming(ctx, q, tp, seg, 2)
    torch.cuda.synchronize()
    assert torch.equal(idx_p, idx[perm]) and torch.equal(dist_p, dist[perm])
    sample = [0, 1, 5, 100, 776, 777, 778, 999, 1000, 1234, 1500, 1776, 1900, 1997, 1998, 1999]
    tn = t.view(n_kf, nf, 32)[sample].reshape(-1, 32).cpu().numpy()
    ri, rd = ora.knn_hamming_batch(q.cpu().numpy(), tn, synth.seg_ptr_uniform(len(sample), nf), 2)
    assert np.array_equal(idx[sample].cpu().numpy(), ri) and np.array_equal(dist[sample].cpu().numpy(), rd)


def test_descriptor_database_matches_batch_call_and_oracle(ctx):
    """cvb_db_*: keyframes appended in several calls (ragged, one empty) stay resident; a query returns exactly the
    accepted matches of cvb_match_hamming_batch, compacted in (keyframe, queryIdx) order (= img_matches per KF)."""
    desc, _ = synth.orb_keyframes(seed=11, n_kf=14, n_feat=600, n_lm=900, window=900)
    lens = [600, 0, 1, 333, 600, 257, 128, 600, 17, 600, 599, 64, 600]
    t = np.concatenate([desc[i + 1][:l] for i, l in enumerate(lens)])
    seg = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    db = M.DescriptorDatabase(ctx)
    assert db.size() == (0, 0)
    cut = [0, 4, 5, 13]
    for a, b in zip(cut[:-1], cut[1:]):
        db.append(t[seg[a]:seg[b]], lens[a:b])
    assert db.size() == (len(lens), int(seg[-1]))
    for q in (desc[0], desc[0][:77], desc[5][:600]):
        for thr, ratio in ((40.0, 0.8), (64.0, 0.95)):
            nm, m_kf, m_q, m_t, m_d = db.match_hamming(q, thr, ratio)
            mt, md, rn = M.match_candidates_hamming(ctx, q, t, seg, thr, ratio)
            ri, rd = ora.knn_hamming_batch(q, t, seg, k=2)
            omt, omd, onm = ora.ratio_filter(ri, rd.astype(np.float32), thr, ratio)
            assert np.array_equal(mt, omt) and np.array_equal(rn, onm)
            assert np.array_equal(nm, rn)
            kf, qq = np.nonzero(mt >= 0)          # row-major = (keyframe, queryIdx) order
            assert len(kf) == len(m_kf) == int(nm.sum())
            assert np.array_equal(m_kf, kf) and np.array_equal(m_q, qq)
            assert np.array_equal(m_t, mt[kf, qq]) and np.array_equal(m_d, md[kf, qq])
    # capacity retry path: a tiny initial capacity must give the same answer
    db._cap = 3
    nm2, *rest = db.match_hamming(desc[0], 64.0, 0.95)
    assert int(nm2.sum()) == len(rest[0]) > 3
    # keyframes leave the map (culling, keyframe_be.cpp:413-440): cvb_db_remove cuts the segment out, later indices drop by one
    keep = list(range(len(lens)))
    for victim in (3, 0, len(lens) - 3, 1):          # middle, first, (then) last-but-one, the empty one
        db.remove(victim)
        keep.pop(victim)
        t2 = np.concatenate([t[seg[i]:seg[i + 1]] for i in keep]); seg2 = np.concatenate([[0], np.cumsum([lens[i] for i in keep])]).astype(np.int32)
        assert db.size() == (len(keep), int(seg2[-1]))
        nm3, k3, q3, t3, d3 = db.match_hamming(desc[0], 40.0, 0.8)
        mt, md, rn = M.match_candidates_hamming(ctx, desc[0], t2, seg2, 40.0, 0.8)
        kf, qq = np.nonzero(mt >= 0)
        assert np.array_equal(nm3, rn) and np.array_equal(k3, kf) and np.array_equal(q3, qq) and np.array_equal(t3, mt[kf, qq])
    import covins_b200
    with pytest.raises(covins_b200.CvbError):
        db.remove(len(keep))
    db.close()


def test_l2_host_path_single_long_segment_chunked(ctx):
    """ADVICE r1 (high): cvb_knn_l2_batch on ONE long segment takes the chunked tensor-core path; its chunk tables must not
    alias the quantised descriptors staged by the host wrapper.  ~200k rows, 700 queries, vs the oracle on the first rows
    and vs the scalar kernel on all of them."""
    import os
    s, _ = synth.sift_keyframes(seed=41, n_kf=700, n_feat=300)
    t = s.reshape(-1, 128)                       # 210k rows, one segment
    q = s[3][:300].copy(); q = np.concatenate([q, s[10][:300], s[500][:100]])
    idx, dist = M.knn_match_l2(ctx, q, t, None, k=2)
    os.environ["COVINS_B200_MATCH_KERNEL"] = "popc"
    try:
        idx_s, dist_s = M.knn_match_l2(ctx, q, t, None, k=2)
    finally:
        os.environ.pop("COVINS_B200_MATCH_KERNEL", None)
    assert np.array_equal(idx, idx_s) and np.array_equal(dist, dist_s)
    ri, rd = ora.knn_l2(q[:8], t, k=2)           # rows 0..2 of q and t were the ones the aliasing bug overwrote
    assert np.array_equal(idx[0][:8], ri) and np.array_equal(dist[0][:8], rd)
    assert idx[0][0, 0] == 3 * 300 and dist[0][0, 0] == 0.0


@pytest.mark.parametrize("metric", ["hamming", "l2"])
def test_mapwide_sharded_knn_merge_equals_single_call(ctx, metric):
    """SURVEY §8e map-wide k-NN: per-shard CUDA top-k (3 shards incl. one with fewer than k rows and an empty one) →
    cvb_knn_merge_shards_dev == the single-call k-NN over the whole database, bit-exact, ties across shards included."""
    import torch
    rng = np.random.default_rng(33)
    dim = 32 if metric == "hamming" else 128
    base = rng.integers(0, 256, (50, dim), dtype=np.uint8)
    t = base[rng.integers(0, 50, 5000)].copy()
    q = base[:64].copy()
    cuts = [0, 2, 2, 2600, 5000]                       # shard sizes 2, 0, 2598, 2400
    k = 3
    dev = torch.device("cuda", 0)
    tq, tt = torch.from_numpy(q).to(dev), torch.from_numpy(t).to(dev)
    knn = M.knn_match_hamming if metric == "hamming" else M.knn_match_l2
    ri, rd = knn(ctx, tq, tt, None, k)
    li_all, ld_all = [], []
    for a, b in zip(cuts[:-1], cuts[1:]):
        if b > a:
            li, ld = knn(ctx, tq, tt[a:b].contiguous(), None, k)
            li_all.append(li[0]); ld_all.append(ld[0])
        else:                                          # an empty shard contributes "no neighbour" lists
            li_all.append(torch.full((len(q), k), -1, dtype=torch.int32, device=dev))
            ld_all.append(torch.zeros((len(q), k), dtype=ri.dtype if False else rd.dtype, device=dev))
    off = torch.tensor(cuts[:-1], dtype=torch.int32, device=dev)
    mi, md = M.knn_merge_shards(ctx, torch.stack(li_all), torch.stack(ld_all), off, k)
    torch.cuda.synchronize()
    assert torch.equal(mi, ri[0]) and torch.equal(md, rd[0])
    oi, od = ora.merge_shards(torch.stack(li_all).cpu().numpy(), torch.stack(ld_all).cpu().numpy(), cuts[:-1], k)
    assert np.array_equal(mi.cpu().numpy(), oi) and np.array_equal(md.cpu().numpy(), od)


def test_landmark_descriptor_batch_vs_oracle(ctx):
    """K-M7 Landmark::ComputeDescriptor batched (landmark_be.cpp:49-92): bit-exact vs the oracle for landmark sizes
    0..300 (register path, > 256-observer recompute path), host and device entry points, old descriptors kept for
    landmarks without observers."""
    import torch
    from test_oracle_knn import _lm_desc_case
    rng = np.random.default_rng(9)
    sizes = [0, 1, 2, 3, 8, 31, 32, 33, 64, 100, 0, 256, 257, 300] + list(rng.integers(2, 20, 400))
    cand, lm_ptr = _lm_desc_case(12, sizes)
    old = rng.integers(0, 256, (len(sizes), 32), dtype=np.uint8)
    rb, rd = ora.landmark_descriptor(cand, lm_ptr)
    rd[rb < 0] = old[rb < 0]
    b, d = M.landmark_descriptors(ctx, cand, lm_ptr, old)
    assert np.array_equal(b, rb) and np.array_equal(d, rd)
    dev = torch.device("cuda", 0)
    tb, td = M.landmark_descriptors(ctx, torch.from_numpy(cand).to(dev), torch.from_numpy(lm_ptr).to(dev), torch.from_numpy(old).to(dev))
    torch.cuda.synchronize()
    assert np.array_equal(tb.cpu().numpy(), rb) and np.array_equal(td.cpu().numpy(), rd)
