"""Merging two agents' maps: cvb_map_rigid_transform (the transform of the merge constructor Map(map_target, map_tofuse, T),
map_be.cpp:334-381), cvb_db_merge / cvb_db_group_merge (the fused map's keyframes joining the target's resident descriptor
database in HBM) and the C++ shim's MergeMaps.
CPU: oracle/merge.py equals np.einsum to 0 ulp on integer-valued inputs and to 2 ulp (of the entry's largest product) on
random ones; T = I returns the inputs' bits; the Python wrapper refuses what the C rule refuses; the shim compiles.
GPU: the transform is bitwise the oracle's on C1 and C3 maps and at a 1e4 m translation, with and without selection masks,
for K = 0, L = 0 and no velocities, in one launch, the same run to run; refusals launch nothing.  A merged database answers
every request (host and _dev, ORB and SIFT, both matching kernels) bit for bit like one fed the same keyframes from the host,
across keyframe sizes at the 128-row tile boundary, empty sides, two merges, a removal across the old boundary and a later
append, with src unchanged, and without a launch or a host-to-device copy.  A group of two ranks on one device merges to
the single merged database's outputs (distinct devices are skipped with fewer than two GPUs).  The shim on mock containers
writes the oracle's states back in the reference's order, leaves the target's objects alone, joins the databases and leaves
the covisibility graph of the merged map.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from covins_b200 import mapgraph, synth, synth_map
from oracle import covis as ora_covis
from oracle import merge as ora

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CVB_ERR_INVALID, CVB_ERR_UNSUPPORTED = 1, 3


# ------------------------------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------------------------------
def rot(rng):
    q, r = np.linalg.qr(rng.normal(size=(3, 3)))
    q = q * np.sign(np.diag(r))
    return q if np.linalg.det(q) > 0 else -q


def rigid(rng, t_scale=10.0):
    T = np.eye(4)
    T[:3, :3] = rot(rng)
    T[:3, 3] = rng.normal(size=3) * t_scale
    return T


def poses_of(p):
    """the synthetic map's T_ws [K,4,4] from its [q, t] poses"""
    K = int(p["K"])
    T = np.zeros((K, 4, 4))
    T[:, :3, :3] = synth_map.quat_to_rot(np.asarray(p["pose"])[:, :4])
    T[:, :3, 3] = np.asarray(p["pose"])[:, 4:]
    T[:, 3, 3] = 1.0
    return T


def random_state(rng, K, L):
    return np.stack([rigid(rng) for _ in range(K)]) if K else np.zeros((0, 4, 4)), rng.normal(size=(K, 3)), rng.normal(size=(L, 3)) * 20


def einsum_ref(T, ws, vel, lm):
    R, t = T[:3, :3], T[:3, 3]
    return np.einsum("ij,kjl->kil", T, ws), np.einsum("ij,kj->ki", R, vel), np.einsum("ij,lj->li", R, lm) + t


def bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


# ------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------
def test_oracle_equals_einsum_exactly_on_integer_inputs():
    rng = np.random.default_rng(0)
    for perm in ([0, 1, 2], [1, 2, 0], [2, 0, 1], [1, 0, 2]):
        T = np.eye(4)
        T[:3, :3] = np.eye(3)[perm] * rng.choice([-1.0, 1.0], size=(3, 1))
        if np.linalg.det(T[:3, :3]) < 0:
            T[0, :3] *= -1
        T[:3, 3] = rng.integers(-1000, 1000, size=3)
        ws = rng.integers(-50, 50, size=(20, 4, 4)).astype(float)
        vel, lm = rng.integers(-9, 9, size=(20, 3)).astype(float), rng.integers(-10**6, 10**6, size=(30, 3)).astype(float)
        got, ref = ora.rigid_transform(T, ws, vel, lm), einsum_ref(T, ws, vel, lm)
        for a, b in zip(got, ref):
            assert np.array_equal(bits(a), bits(b))


def test_oracle_equals_einsum_within_two_ulp_on_random_inputs():
    rng = np.random.default_rng(1)
    for s in range(20):
        T = rigid(rng, t_scale=10.0 ** (s % 5))
        ws, vel, lm = random_state(rng, 50, 200)
        got, ref = ora.rigid_transform(T, ws, vel, lm), einsum_ref(T, ws, vel, lm)
        # the scale of an entry: the sum of its products' magnitudes (a cancelling sum has no ulp of its own)
        scale = (np.einsum("ij,kjl->kil", np.abs(T), np.abs(ws)), np.einsum("ij,kj->ki", np.abs(T[:3, :3]), np.abs(vel)),
                 np.einsum("ij,lj->li", np.abs(T[:3, :3]), np.abs(lm)) + np.abs(T[:3, 3]))
        for a, b, m in zip(got, ref, scale):
            assert (np.abs(a - b) <= 2 * np.spacing(m)).all()


def test_identity_returns_the_input_bits():
    rng = np.random.default_rng(2)
    ws, vel, lm = random_state(rng, 30, 100)
    for a, b in zip(ora.rigid_transform(np.eye(4), ws, vel, lm), (ws, vel, lm)):
        assert np.array_equal(bits(a), bits(b))


def non_rigid():
    rng = np.random.default_rng(3)
    T = rigid(rng)
    out = {"scaled": np.diag([2.0, 2.0, 2.0, 1.0]), "reflection": np.diag([1.0, 1.0, -1.0, 1.0]), "shear": np.eye(4) + np.eye(4, k=1) * 1e-3,
           "zero": np.zeros((4, 4))}
    for name, (r, c, v) in {"last row 0": (3, 0, 1e-12), "last row 3": (3, 3, 1.0 + 1e-15), "nan": (0, 0, np.nan), "inf t": (1, 3, np.inf),
                            "nan t": (2, 3, np.nan)}.items():
        out[name] = T.copy()
        out[name][r, c] = v
    out["R off by 2e-9"] = T.copy()
    out["R off by 2e-9"][0, 0] += 2e-9
    return out


def test_wrapper_refuses_what_the_c_rule_refuses():
    rng = np.random.default_rng(4)
    ws, vel, lm = random_state(rng, 3, 4)
    for name, T in non_rigid().items():
        assert not ora.is_rigid(T) and not mapgraph.is_rigid(T), name
        with pytest.raises(ValueError, match="not rigid"):
            mapgraph.rigid_transform(None, T, ws, vel, lm)       # refused before the context is used
    ok = [np.eye(4), rigid(rng), rigid(rng, 1e4)]
    near = rigid(rng)
    near[0, 0] += 2e-10
    for T in ok + [near]:
        assert ora.is_rigid(T) and mapgraph.is_rigid(T)


def test_shim_merge_compiles_and_refuses_missing_input(tmp_path):
    exe = str(tmp_path / "shim_merge_test")
    _build_shim(exe)
    assert subprocess.run([exe, str(tmp_path)]).returncode == 2     # nothing dumped: refused before any GPU work


def _build_shim(exe):
    import covins_b200
    if not os.path.exists(covins_b200.LIB_PATH):
        covins_b200.build()
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-o", exe, os.path.join(ROOT, "tests", "cpp", "shim_merge_test.cpp"),
                           "-L" + os.path.join(ROOT, "covins_b200"), "-lcovins_b200", "-Wl,-rpath," + os.path.join(ROOT, "covins_b200")])


# ------------------------------------------------------------------------------------------------------------------
# GPU: K16 cvb_map_rigid_transform
# ------------------------------------------------------------------------------------------------------------------
def _check_k16(ctx, T, ws, vel, lm, kf_sel=None, lm_sel=None):
    l0 = ctx.launch_count()
    got = mapgraph.rigid_transform(ctx, T, ws, vel, lm, kf_sel, lm_sel)
    assert ctx.launch_count() - l0 == (1 if len(ws) + len(lm) else 0)
    ref = ora.rigid_transform(T, ws, vel, lm, kf_sel, lm_sel)
    for a, b in zip(got, ref):
        assert (a is None) == (b is None)
        if a is not None:
            assert np.array_equal(bits(a), bits(b)), int((bits(a) != bits(b)).sum())
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["C1", "C3"])
def test_k16_is_bitwise_the_oracle_on_synthetic_maps(ctx, config):
    p = synth_map.make_config(config)
    rng = np.random.default_rng(5)
    ws, lm = poses_of(p), np.asarray(p["lm"], np.float64)
    vel = rng.normal(size=(len(ws), 3))
    for T in (rigid(rng), rigid(rng, 1e4)):
        got = _check_k16(ctx, T, ws, vel, lm)
        again = mapgraph.rigid_transform(ctx, T, ws, vel, lm)            # the same run to run
        for a, b in zip(got, again):
            assert np.array_equal(bits(a), bits(b))


@pytest.mark.gpu
def test_k16_at_a_1e4_m_translation(ctx):
    rng = np.random.default_rng(6)
    T = rigid(rng)
    T[:3, 3] = [1e4, -1e4, 0.5e4]
    ws, vel, lm = random_state(rng, 1000, 20000)
    _check_k16(ctx, T, ws, vel, lm)


@pytest.mark.gpu
def test_k16_identity_returns_the_input_bits(ctx):
    ws, vel, lm = random_state(np.random.default_rng(7), 100, 1000)
    for a, b in zip(mapgraph.rigid_transform(ctx, np.eye(4), ws, vel, lm), (ws, vel, lm)):
        assert np.array_equal(bits(a), bits(b))


@pytest.mark.gpu
def test_k16_selection_masks_leave_the_others_untouched(ctx):
    rng = np.random.default_rng(8)
    T = rigid(rng)
    ws, vel, lm = random_state(rng, 300, 3000)
    ks, ls = (rng.random(300) < 0.5).astype(np.uint8) * rng.integers(1, 255, size=300).astype(np.uint8), (rng.random(3000) < 0.3).astype(np.uint8)
    got = _check_k16(ctx, T, ws, vel, lm, ks, ls)
    assert np.array_equal(bits(got[0][ks == 0]), bits(ws[ks == 0])) and np.array_equal(bits(got[1][ks == 0]), bits(vel[ks == 0]))
    assert np.array_equal(bits(got[2][ls == 0]), bits(lm[ls == 0]))
    assert not np.array_equal(bits(got[0][ks != 0]), bits(ws[ks != 0]))
    for k, l in ((np.zeros(300, np.uint8), np.zeros(3000, np.uint8)), (np.ones(300, np.uint8), np.ones(3000, np.uint8))):
        _check_k16(ctx, T, ws, vel, lm, k, l)


@pytest.mark.gpu
def test_k16_empty_sides_and_no_velocity(ctx):
    rng = np.random.default_rng(9)
    T = rigid(rng)
    ws, vel, lm = random_state(rng, 40, 70)
    _check_k16(ctx, T, ws, None, lm)
    _check_k16(ctx, T, ws[:0], vel[:0], lm)
    _check_k16(ctx, T, ws, vel, lm[:0])
    _check_k16(ctx, T, ws[:0], None, lm[:0])
    from covins_b200._lib import lib
    l0 = ctx.launch_count()
    assert lib().cvb_map_rigid_transform(ctx.handle, T.ctypes.data, 0, None, None, 0, None, None, None) == 0
    assert ctx.launch_count() == l0


@pytest.mark.gpu
def test_k16_refusals_launch_nothing(ctx):
    from covins_b200._lib import lib
    rng = np.random.default_rng(10)
    ws, vel, lm = random_state(rng, 5, 5)
    f = lib().cvb_map_rigid_transform
    good = np.ascontiguousarray(rigid(rng))
    cases = {name: (T, 5, 5, True, True) for name, T in non_rigid().items()}
    cases.update({"K < 0": (good, -1, 5, True, True), "L < 0": (good, 5, -1, True, True), "null T_ws": (good, 5, 5, False, True),
                  "null lm": (good, 5, 5, True, False)})
    before = (bits(ws).copy(), bits(vel).copy(), bits(lm).copy())
    for name, (T, K, L, has_ws, has_lm) in cases.items():
        T = np.ascontiguousarray(T, np.float64)
        l0 = ctx.launch_count()
        rc = f(ctx.handle, T.ctypes.data, K, ws.ctypes.data if has_ws else None, vel.ctypes.data, L, lm.ctypes.data if has_lm else None, None, None)
        assert rc == CVB_ERR_INVALID and ctx.launch_count() == l0, name
    assert f(ctx.handle, None, 5, ws.ctypes.data, vel.ctypes.data, 5, lm.ctypes.data, None, None) == CVB_ERR_INVALID
    for a, b in zip((ws, vel, lm), before):
        assert np.array_equal(bits(a), b)
    _check_k16(ctx, good, ws, vel, lm)                                   # the context still works


# ------------------------------------------------------------------------------------------------------------------
# GPU: cvb_db_merge
# ------------------------------------------------------------------------------------------------------------------
KINDS = {"orb": (40.0, 0.8), "sift": (500.0, 0.8)}
SIZES = [1, 127, 128, 129, 300]


def _keyframes(kind, n_kf, seed):
    """(query rows, [n_kf] keyframes' rows with the row counts of SIZES in turn)"""
    gen = synth.orb_keyframes if kind == "orb" else synth.sift_keyframes
    d, _ = gen(seed=seed, n_kf=n_kf + 1, n_feat=300, n_lm=600, window=600)
    return d[0], [d[i + 1][:SIZES[(i + seed) % len(SIZES)]] for i in range(n_kf)]


def _db(ctx, kind, kfs):
    from covins_b200 import matching as M
    db = M.DescriptorDatabase(ctx, kind=kind)
    if kfs:
        db.append(np.concatenate(kfs), [len(k) for k in kfs])
    return db


def _requests(db, kind, q):
    """every output of a host request and of the device request, with either matching kernel"""
    import torch
    from covins_b200 import matching as M
    thr, ratio = KINDS[kind]
    out = []
    for kernel in (None, "tc"):
        if kernel:
            os.environ["COVINS_B200_MATCH_KERNEL"] = kernel
        try:
            if kind == "orb":
                host = db.match_hamming(q, thr, ratio)
                dq = torch.from_numpy(np.ascontiguousarray(q, np.uint8)).cuda()
                dev = db.match_hamming_dev(dq, thr, ratio)
            else:
                host = db.match_l2(q, thr, ratio)
                dq = torch.from_numpy(np.ascontiguousarray(q, np.float32).astype(np.uint8)).cuda()
                dev = db.match_l2_dev(dq, thr, ratio)
            torch.cuda.synchronize()
        finally:
            os.environ.pop("COVINS_B200_MATCH_KERNEL", None)
        out.append([np.ascontiguousarray(a).view(np.int32) for a in host] + [t.cpu().numpy().view(np.int32) for t in dev])
    out.append(np.array(db.size(), np.int64))
    return out


def _same(a, b):
    assert np.array_equal(a[-1], b[-1]), (a[-1], b[-1])
    for x, y in zip(a[:-1], b[:-1]):
        for u, v in zip(x, y):
            assert u.shape == v.shape and np.array_equal(u, v)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["orb", "sift"])
def test_db_merge_equals_the_host_appended_database(ctx, kind):
    q, kfs = _keyframes(kind, 13, seed=11)
    for split in (0, 5, 13):                             # an empty dst, both sides, an empty src
        dst, src, one = _db(ctx, kind, kfs[:split]), _db(ctx, kind, kfs[split:]), _db(ctx, kind, kfs)
        src_before = _requests(src, kind, q)
        l0 = ctx.launch_count()
        dst.merge(src)
        assert ctx.launch_count() == l0                  # rows and tiles are copied, not expanded
        _same(_requests(dst, kind, q), _requests(one, kind, q))
        _same(_requests(src, kind, q), src_before)       # src unchanged
        for d in (dst, src, one):
            d.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["orb", "sift"])
def test_db_merge_twice_then_remove_across_the_boundary_and_append(ctx, kind):
    q, kfs = _keyframes(kind, 16, seed=12)
    a, b, c = kfs[:5], kfs[5:11], kfs[11:15]
    dst, s1, s2, one = _db(ctx, kind, a), _db(ctx, kind, b), _db(ctx, kind, c), _db(ctx, kind, a + b + c)
    dst.merge(s1)
    dst.merge(s2)
    dst.merge(s1)                                        # the same src again
    one.append(np.concatenate(b), [len(k) for k in b])
    _same(_requests(dst, kind, q), _requests(one, kind, q))
    for i in (5, 4, 3, 12):                              # the old boundaries, then inside
        dst.remove(i)
        one.remove(i)
        _same(_requests(dst, kind, q), _requests(one, kind, q))
    for d in (dst, one):
        d.append(np.concatenate([kfs[15], kfs[0]]), [len(kfs[15]), len(kfs[0])])
    _same(_requests(dst, kind, q), _requests(one, kind, q))
    for d in (dst, s1, s2, one):
        d.close()


@pytest.mark.gpu
def test_db_merge_refusals_leave_dst_unchanged(ctx):
    import covins_b200
    from covins_b200._lib import lib
    q, kfs = _keyframes("orb", 4, seed=13)
    _, sk = _keyframes("sift", 2, seed=13)
    dst, src, sift = _db(ctx, "orb", kfs[:2]), _db(ctx, "orb", kfs[2:]), _db(ctx, "sift", sk)
    before = _requests(dst, "orb", q)
    other = covins_b200.Context(0)
    try:
        foreign = _db(other, "orb", kfs[2:])
        for s, code in ((dst, CVB_ERR_INVALID), (sift, CVB_ERR_INVALID), (foreign, CVB_ERR_UNSUPPORTED)):
            l0 = ctx.launch_count()
            assert lib().cvb_db_merge(ctx.handle, dst.handle, s.handle) == code
            assert ctx.launch_count() == l0
        assert b"another context" in lib().cvb_last_error(ctx.handle)
        assert lib().cvb_db_merge(ctx.handle, dst.handle, None) == CVB_ERR_INVALID
        _same(_requests(dst, "orb", q), before)
        foreign.close()
    finally:
        other.close()
    dst.merge(src)
    _same(_requests(dst, "orb", q), _requests(_db(ctx, "orb", kfs), "orb", q))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["orb", "sift"])
def test_db_merge_copies_no_descriptor_over_pcie(ctx, kind):
    """the profiler's memcpy records during the merge: device-to-device only (the append it replaces is host-to-device)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    _, kfs = _keyframes(kind, 40, seed=14)
    dst, src = _db(ctx, kind, kfs[:20]), _db(ctx, kind, kfs[20:])
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        dst.merge(src)
        torch.cuda.synchronize()
    kinds = [e.name for e in prof.events() if "memcpy" in e.name.lower()]
    assert kinds and all("htod" not in k.lower().replace(" ", "") for k in kinds), kinds
    assert any("dtod" in k.lower().replace(" ", "") for k in kinds), kinds
    dst.close()
    src.close()


# ------------------------------------------------------------------------------------------------------------------
# GPU: cvb_db_group_merge
# ------------------------------------------------------------------------------------------------------------------
def _group_layouts():
    import torch
    two = pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two GPUs")
    return [pytest.param(1, id="shared2"), pytest.param(2, id="distinct", marks=two)]


@pytest.mark.gpu
@pytest.mark.parametrize("ndev", _group_layouts())
@pytest.mark.parametrize("kind", ["orb", "sift"])
def test_group_merge_equals_one_merged_database(ctx, kind, ndev):
    import covins_b200
    from covins_b200 import matching as M
    from covins_b200 import optimization as O
    thr, ratio = KINDS[kind]
    match = "match_hamming" if kind == "orb" else "match_l2"
    q, kfs = _keyframes(kind, 14, seed=15)
    ctxs = [covins_b200.Context(r % ndev) for r in range(2)]
    g = O.Group(ctxs)
    g2 = O.Group([covins_b200.Context(0)])
    try:
        def group_db(part):
            d = M.DescriptorDatabaseGroup(g, kind=kind)
            if part:
                d.append(np.concatenate(part), [len(k) for k in part])
            return d
        dst, src = group_db(kfs[:6]), group_db(kfs[6:12])
        src_before = getattr(src, match)(q, thr, ratio)
        dst.merge(src)
        one = _db(ctx, kind, kfs[:12])
        for d in (dst, one):
            d.remove(6)
            d.append(np.concatenate(kfs[12:]), [len(k) for k in kfs[12:]])
        n_kf, n_rows, per = dst.size_per_rank()
        assert (n_kf, n_rows) == one.size() and per.sum() == n_rows
        for a, b in zip(getattr(dst, match)(q, thr, ratio), getattr(one, match)(q, thr, ratio)):
            assert np.array_equal(np.ascontiguousarray(a).view(np.int32), np.ascontiguousarray(b).view(np.int32))
        for a, b in zip(getattr(src, match)(q, thr, ratio), src_before):
            assert np.array_equal(np.ascontiguousarray(a).view(np.int32), np.ascontiguousarray(b).view(np.int32))
        from covins_b200._lib import lib
        other = M.DescriptorDatabaseGroup(g2, kind=kind)
        assert lib().cvb_db_group_merge(dst.handle, dst.handle) == CVB_ERR_INVALID
        assert lib().cvb_db_group_merge(dst.handle, other.handle) == CVB_ERR_UNSUPPORTED
        assert dst.size() == one.size()
        for d in (dst, src, other, one):
            d.close()
    finally:
        g.close()
        g2.close()
        for c in ctxs + g2.contexts:
            c.close()


# ------------------------------------------------------------------------------------------------------------------
# the C++ shim on mock containers
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_shim_merge_maps_on_mock_containers(tmp_path):
    """covins_b200::MergeMaps: the fused map's valid keyframes and landmarks get the oracle's states, written keyframes first
    (SetPoseTws, SetStateVelocity) then landmarks; the target's objects and the invalid ones keep their bits; the merged map
    holds both maps and both loop constraints; its covisibility is cvb_covisibility's of the merged flat map; the merged
    database matches like one appended from the host (checked inside the program)"""
    rng = np.random.default_rng(16)
    maps = [synth_map.make_map(seed=31 + a, n_agents=1, kf_per_agent=30 + 10 * a, n_lm=1500) for a in range(2)]
    K = [int(m["K"]) for m in maps]
    L = [int(m["L"]) for m in maps]
    pose = np.concatenate([poses_of(m) for m in maps]).reshape(-1, 16)
    vel = rng.normal(size=(sum(K), 3))
    kf_agent = np.repeat([0, 1], K).astype(np.int32)
    lm = np.concatenate([m["lm"] for m in maps])
    lm_agent = np.repeat([0, 1], L).astype(np.int32)
    kf_inv = np.zeros(sum(K), np.uint8)
    kf_inv[[3, K[0] + 7]] = 1
    lm_inv = np.zeros(sum(L), np.uint8)
    lm_inv[[10, L[0] + 20, L[0] + 21]] = 1
    ptr = np.concatenate([maps[0]["lm_obs_ptr"], maps[1]["lm_obs_ptr"][1:] + maps[0]["lm_obs_ptr"][-1]]).astype(np.int32)
    obs_kf = np.concatenate([maps[0]["obs_kf"], maps[1]["obs_kf"] + K[0]]).astype(np.int32)
    q, kfs = _keyframes("orb", sum(K), seed=17)
    T = rigid(rng, 1e3)
    for name, a, dt in (("T", T, np.float64), ("pose", pose, np.float64), ("vel", vel, np.float64), ("kf_agent", kf_agent, np.int32),
                        ("kf_inv", kf_inv, np.uint8), ("lm", lm, np.float64), ("lm_agent", lm_agent, np.int32), ("lm_inv", lm_inv, np.uint8),
                        ("ptr", ptr, np.int32), ("kf", obs_kf, np.int32), ("desc", np.concatenate(kfs), np.uint8),
                        ("rpk", [len(k) for k in kfs], np.int32), ("q", q, np.uint8)):
        np.ascontiguousarray(a, dt).tofile(tmp_path / f"{name}.bin")
    exe = str(tmp_path / "shim_merge_test")
    _build_shim(exe)
    subprocess.check_call([exe, str(tmp_path)])
    ksel = (kf_agent == 1) & (kf_inv == 0)
    lsel = (lm_agent == 1) & (lm_inv == 0)
    ref_ws, ref_vel, ref_lm = ora.rigid_transform(T, pose, vel, lm, ksel, lsel)
    assert np.array_equal(bits(np.fromfile(tmp_path / "out_pose.bin")), bits(ref_ws.reshape(-1)))
    assert np.array_equal(bits(np.fromfile(tmp_path / "out_vel.bin")), bits(ref_vel.reshape(-1)))
    assert np.array_equal(bits(np.fromfile(tmp_path / "out_lm.bin")), bits(ref_lm.reshape(-1)))
    log = np.fromfile(tmp_path / "out_log.bin", np.int32).reshape(-1, 2)
    expect = [[c, k] for k in np.flatnonzero(ksel) for c in (0, 1)] + [[2, l] for l in np.flatnonzero(lsel)]
    assert np.array_equal(log, np.array(expect, np.int32))
    assert np.fromfile(tmp_path / "out_sizes.bin", np.int32).tolist() == [sum(K), sum(L), 2, sum(K), K[1]]
    # the merged map's canonical flat form: valid keyframes by number, valid landmarks, observations by valid keyframes
    index = np.cumsum(kf_inv == 0) - 1
    keep_lm = np.flatnonzero(lm_inv == 0)
    c_ptr, c_kf = [0], []
    for l in keep_lm:
        obs = [index[k] for k in sorted(obs_kf[ptr[l]:ptr[l + 1]]) if not kf_inv[k]]
        c_kf += obs
        c_ptr.append(len(c_kf))
    ref = ora_covis.covisibility(np.array(c_ptr, np.int32), np.array(c_kf, np.int32), int((kf_inv == 0).sum()))
    valid = np.flatnonzero(kf_inv == 0)
    cnt = np.fromfile(tmp_path / "out_cnt.bin", np.int32)
    assert np.array_equal(cnt[valid], np.diff(ref[0])) and not cnt[kf_inv != 0].any()
    assert np.array_equal(np.fromfile(tmp_path / "out_kf.bin", np.int32), valid[ref[1]])
    assert np.array_equal(np.fromfile(tmp_path / "out_w.bin", np.int32), ref[2])
