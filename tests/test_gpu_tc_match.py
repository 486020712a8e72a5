"""GPU: the wgmma (tensor-core) matching kernel (tc_match.cu) forced on via COVINS_B200_MATCH_KERNEL=tc must be
bit-identical to the oracle / golden vectors / the scalar POPC kernel for every mode it serves."""
import os

import numpy as np
import pytest

from conftest import golden_cases
from covins_b200 import matching as M
from covins_b200 import synth
from oracle import knn as ora

pytestmark = pytest.mark.gpu


@pytest.fixture()
def tc(monkeypatch):
    monkeypatch.setenv("COVINS_B200_MATCH_KERNEL", "tc")
    yield
    monkeypatch.delenv("COVINS_B200_MATCH_KERNEL", raising=False)


def test_tc_hamming_golden(ctx, tc, golden_dir):
    g, names = golden_cases(os.path.join(golden_dir, "knn_hamming.npz"))
    for n in names:
        idx, dist = M.knn_match_hamming(ctx, g[n + "/q"], g[n + "/t"], k=2)
        assert np.array_equal(idx[0], g[n + "/idx"]), n
        d = np.where(idx[0] >= 0, dist[0].astype(np.float32), np.inf)
        assert np.array_equal(d, g[n + "/dist"]), n
        mt, md, nm = M.match_candidates_hamming(ctx, g[n + "/q"], g[n + "/t"], thr=40.0, ratio=0.8)
        assert np.array_equal(mt[0], g[n + "/match"]), n


def test_tc_l2_golden(ctx, tc, golden_dir):
    g, names = golden_cases(os.path.join(golden_dir, "knn_l2.npz"))
    for n in names:
        q = g[n + "/q"].astype(np.float32); t = g[n + "/t"].astype(np.float32)
        idx, dist = M.knn_match_l2(ctx, q, t, k=2)
        assert np.array_equal(idx[0], g[n + "/idx"]), n
        d = np.where(idx[0] >= 0, dist[0], np.inf)
        assert np.array_equal(d, g[n + "/dist"]), n


@pytest.mark.parametrize("k", [1, 2, 4])
def test_tc_hamming_ragged_batch_vs_oracle(ctx, tc, k):
    desc, _ = synth.orb_keyframes(seed=5, n_kf=9, n_feat=700, n_lm=1500, window=1500)
    q = desc[0][:613]
    lens = [700, 0, 1, 2, 3, 257, 512, 699]
    t = np.concatenate([desc[i + 1][:l] for i, l in enumerate(lens)])
    seg = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    idx, dist = M.knn_match_hamming(ctx, q, t, seg, k=k)
    ri, rd = ora.knn_hamming_batch(q, t, seg, k=k)
    assert np.array_equal(idx, ri) and np.array_equal(dist, rd)


def test_tc_ties_and_filter_vs_oracle(ctx, tc):
    rng = np.random.default_rng(42)
    base = rng.integers(0, 256, (40, 32), dtype=np.uint8)
    t = base[rng.integers(0, 40, 30_000)]
    t ^= (rng.integers(0, 256, t.shape, dtype=np.uint8) & rng.integers(0, 256, t.shape, dtype=np.uint8)
          & rng.integers(0, 256, t.shape, dtype=np.uint8) & rng.integers(0, 256, t.shape, dtype=np.uint8) & 3)
    q = base[rng.integers(0, 40, 300)]
    seg = np.array([0, 5000, 5000, 17001, 30000], np.int32)
    idx, dist = M.knn_match_hamming(ctx, q, t, seg, k=2)
    ri, rd = ora.knn_hamming_batch(q, t, seg, k=2)
    assert np.array_equal(idx, ri) and np.array_equal(dist, rd)
    mt, md, nm = M.match_candidates_hamming(ctx, q, t, seg, 40.0, 0.8)
    rmt, rmd, rc = ora.ratio_filter(ri, rd.astype(np.float32), 40.0, 0.8)
    assert np.array_equal(mt, rmt) and np.array_equal(nm, rc)


def test_tc_l2_vs_oracle(ctx, tc):
    s, _ = synth.sift_keyframes(seed=3, n_kf=7, n_feat=300, n_lm=500, window=500)
    q = s[0][:211]
    lens = [300, 0, 2, 129, 300, 77]
    t = np.concatenate([s[i + 1][:l] for i, l in enumerate(lens)])
    seg = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    for k in (1, 2, 4):
        idx, dist = M.knn_match_l2(ctx, q, t, seg, k=k)
        ri, rd = ora.knn_l2_batch(q, t, seg, k=k)
        assert np.array_equal(idx, ri) and np.array_equal(dist, rd)


def test_tc_landmark_match_vs_oracle(ctx, tc):
    desc, lm = synth.orb_keyframes(seed=20, n_kf=13, n_feat=600, n_lm=800, window=800)
    A, skipA = desc[0], (lm[0] < 0).astype(np.uint8)
    lens = [600, 0, 1, 333, 600, 600, 45, 600, 600, 600, 600, 599]
    B = np.concatenate([desc[i + 1][:l] for i, l in enumerate(lens)])
    skipB = np.concatenate([(lm[i + 1][:l] < 0) for i, l in enumerate(lens)]).astype(np.uint8)
    seg = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    out = M.landmark_match(ctx, A, skipA, B, skipB, seg, thr=50.0, num_best=4)
    for s in range(len(lens)):
        ra, rb, rd = ora.landmark_match(A, skipA, B[seg[s]:seg[s + 1]], skipB[seg[s]:seg[s + 1]], 50.0, 4)
        a, b, d = out[s]
        assert np.array_equal(a, ra) and np.array_equal(b, rb) and np.array_equal(d, rd), s


def test_tc_equals_popc_kernel_at_full_size(ctx, monkeypatch):
    import torch
    n_kf, nf = 500, 1000
    g = torch.Generator(device="cuda").manual_seed(7)
    t = torch.randint(0, 256, (n_kf * nf, 32), dtype=torch.uint8, device="cuda", generator=g)
    q = t[77 * nf:78 * nf].clone()
    seg = synth.seg_ptr_uniform(n_kf, nf)
    monkeypatch.setenv("COVINS_B200_MATCH_KERNEL", "popc")
    i0, d0 = M.knn_match_hamming(ctx, q, t, seg, 2)
    m0 = M.match_candidates_hamming(ctx, q, t, seg)
    monkeypatch.setenv("COVINS_B200_MATCH_KERNEL", "tc")
    i1, d1 = M.knn_match_hamming(ctx, q, t, seg, 2)
    m1 = M.match_candidates_hamming(ctx, q, t, seg)
    torch.cuda.synchronize()
    assert torch.equal(i0, i1) and torch.equal(d0, d1)
    assert all(torch.equal(a, b) for a, b in zip(m0, m1))


@pytest.mark.parametrize("metric,k", [("hamming", 2), ("hamming", 4), ("l2", 2), ("l2", 3)])
def test_tc_single_long_segment_chunked_equals_scalar(ctx, monkeypatch, metric, k):
    """Map-wide k-NN (one segment of 200k rows): the segment is cut into chunks for the tensor-core kernel and the chunk
    lists are merged by (distance, index); must be bit-identical to the scalar split/merge path, duplicates included."""
    import torch
    rng = np.random.default_rng(77)
    dim = 32 if metric == "hamming" else 128
    base = rng.integers(0, 256, (3000, dim), dtype=np.uint8)
    t = base[rng.integers(0, 3000, 200_003)].copy()          # many exact duplicates → ties across chunk boundaries
    noise = rng.random(t.shape) < 0.01
    t[noise] ^= rng.integers(1, 256, int(noise.sum()), dtype=np.uint8)
    q = base[:700].copy()
    dev = torch.device("cuda", 0)
    tq, tt = torch.from_numpy(q).to(dev), torch.from_numpy(t).to(dev)
    knn = M.knn_match_hamming if metric == "hamming" else M.knn_match_l2
    monkeypatch.delenv("COVINS_B200_MATCH_KERNEL", raising=False)
    i1, d1 = knn(ctx, tq, tt, None, k)
    monkeypatch.setenv("COVINS_B200_MATCH_KERNEL", "popc")
    i0, d0 = knn(ctx, tq, tt, None, k)
    torch.cuda.synchronize()
    assert torch.equal(i1, i0) and torch.equal(d1, d0)
    if metric == "hamming":
        ri, rd = ora.knn_hamming(q[:64], t, k)
        assert np.array_equal(i1[0, :64].cpu().numpy(), ri) and np.array_equal(d1[0, :64].cpu().numpy(), rd)


def test_tc_database_resident_tiles_vs_oracle(ctx, tc):
    """The map database keeps the tensor-core operand tiles of its keyframes (written at append time): host and device requests,
    appends in several calls, ragged / empty keyframes and removals must all give the oracle's accepted matches."""
    import torch
    desc, _ = synth.orb_keyframes(seed=12, n_kf=16, n_feat=700, n_lm=1200, window=1200)
    lens = [700, 0, 1, 129, 700, 256, 128, 127, 700, 17, 700, 699, 64, 700, 385]
    t = np.concatenate([desc[i + 1][:l] for i, l in enumerate(lens)])
    seg = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    db = M.DescriptorDatabase(ctx)
    for a, b in ((0, 1), (1, 6), (6, 15)):
        db.append(t[seg[a]:seg[b]], lens[a:b])
    keep = list(range(len(lens)))

    def check():
        t2 = np.concatenate([t[seg[i]:seg[i + 1]] for i in keep]); seg2 = np.concatenate([[0], np.cumsum([lens[i] for i in keep])]).astype(np.int32)
        for q in (desc[0], desc[0][:77]):
            ri, rd = ora.knn_hamming_batch(q, t2, seg2, k=2)
            omt, omd, onm = ora.ratio_filter(ri, rd.astype(np.float32), 45.0, 0.85)
            nm, m_kf, m_q, m_t, m_d = db.match_hamming(q, 45.0, 0.85)
            kf, qq = np.nonzero(omt >= 0)
            assert np.array_equal(nm, onm) and np.array_equal(m_kf, kf) and np.array_equal(m_q, qq)
            assert np.array_equal(m_t, omt[kf, qq]) and np.array_equal(m_d, omd[kf, qq])
            mt, md, dn = db.match_hamming_dev(torch.from_numpy(q).cuda(), 45.0, 0.85)
            assert np.array_equal(mt.cpu().numpy(), omt) and np.array_equal(dn.cpu().numpy(), onm)
            assert np.array_equal(md.cpu().numpy()[omt >= 0], omd[omt >= 0])

    check()
    for victim in (4, 0, len(lens) - 3, 0):
        db.remove(victim); keep.pop(victim)
        check()
    db.append(desc[15][:300], [300]); lens.append(300); t = np.concatenate([t, desc[15][:300]]); seg = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    keep.append(len(lens) - 1)
    check()
    db.close()
