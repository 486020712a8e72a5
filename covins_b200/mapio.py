"""Reader / writer of the COVINS on-disk map format (SURVEY.md §8f-1) ⇄ the flat problem behind the C-ABI.

A saved map (`Map::SaveToFile`, covins_backend/src/covins_backend/map_be.cpp:835-912) is a directory

    <dir>/keyframes/keyframes<i>.txt      one cereal *binary* archive of a MsgKeyframe  (file-save field order,
                                          covins_comm/include/covins/covins_base/msgs/msg_keyframe.hpp:129-143)
    <dir>/mappoints/mappoints<i>.txt      one MsgLandmark (msgs/msg_landmark.hpp:69-73); landmarks with < 2 observations
                                          or without reference keyframe are not written (map_be.cpp:880-886)
    <dir>/mapdata.txt                     MsgMap: the loop constraints (map_be.hpp:126-136)

and is read back by `Map::LoadFromFile` (map_be.cpp:508-700), which lists the two directories (any file name, any
order) and rebuilds the containers.  The encoding restated here is cereal's BinaryOutputArchive (vendored header-only
at covins_comm/thirdparty/cereal: archives/binary.hpp, types/vector.hpp, types/utility.hpp,
types/concepts/pair_associative_container.hpp): arithmetic values raw little-endian;
`bool` one byte; enums as their `int`; `std::pair` = first, second; `std::vector` / `std::map` / = a uint64 size tag,
then the elements (vectors of arithmetic types as one raw block; map items as key, value in key order);
Eigen matrices by the reference's own `save` (msg_keyframe.hpp:211-234): int32 rows, int32 cols, raw column-major
data; `cv::Mat` by msg_keyframe.hpp:237-285: int rows, cols, type, bool continuous, raw rows.

PARITY PINNED by reference-written bytes: tests/golden/covins_map_ref/ is written by the vendored cereal + the
reference's own message headers and `save` templates (oracle/ref/cereal_fixture_gen.cpp, built by oracle/ref/Makefile);
tests/test_mapio_cereal.py checks that this module decodes those files to the values that went in and re-encodes them
byte for byte.  (The reference ships no saved map; the fixture is a small synthetic one.)

`write_map(dir, problem)` turns a flat problem (covins_b200.synth_map) into such a directory; `read_map(dir)` turns a
directory into the flat problem that `optimization.BaSolver / global_bundle_adjustment / pgo_edges` and the matching
calls consume — "the same serialized map" of BASELINE.json's north_star.
"""
from __future__ import annotations

import os
import struct

import numpy as np

KFRANGE, MAPRANGE = 65535, 255          # typedefs_base.hpp:51-52
DEFPAIR = (KFRANGE, MAPRANGE)           # typedefs_base.hpp:56
CV_8U, CV_32F = 0, 5


# ------------------------------------------------------------------------------------------------ primitives
class _W:
    def __init__(self):
        self.b = bytearray()

    def raw(self, x): self.b += x
    def u8(self, v): self.b += struct.pack("<B", int(v))
    def i32(self, v): self.b += struct.pack("<i", int(v))
    def u64(self, v): self.b += struct.pack("<Q", int(v))
    def f64(self, v): self.b += struct.pack("<d", float(v))
    def idpair(self, p): self.u64(p[0]); self.u64(p[1])

    def eigen(self, a, dtype=np.float64, shape=None):
        """Eigen::Matrix save (msg_keyframe.hpp:211-221): rows, cols (int32), column-major data"""
        a = np.asarray(a, dtype)
        if a.ndim == 1:
            a = a.reshape(-1, 1)
        if shape is not None:
            assert a.shape == shape, (a.shape, shape)
        self.i32(a.shape[0]); self.i32(a.shape[1])
        self.b += np.asfortranarray(a).tobytes(order="F")

    def eigen_vec(self, arr, dtype, shape):
        """std::vector<Eigen fixed-size, aligned_allocator>: size tag + every element"""
        arr = np.asarray(arr, dtype).reshape((-1,) + shape)
        self.u64(len(arr))
        for e in arr:
            self.eigen(e, dtype, shape)

    def f64_vec(self, v):
        v = np.ascontiguousarray(v, np.float64).reshape(-1)
        self.u64(len(v)); self.b += v.tobytes()

    def cvmat(self, m, cvtype):
        """cv::Mat save (msg_keyframe.hpp:237-262), always written continuous"""
        if m is None or np.size(m) == 0:
            rows = cols = 0; data = b""
        else:
            m = np.ascontiguousarray(m, np.uint8 if cvtype == CV_8U else np.float32)
            rows, cols = m.shape; data = m.tobytes()
        self.i32(rows); self.i32(cols); self.i32(cvtype); self.u8(1); self.b += data


class _R:
    def __init__(self, b):
        self.b = memoryview(b); self.o = 0

    def _take(self, n):
        if self.o + n > len(self.b):
            raise ValueError("truncated COVINS archive")
        v = self.b[self.o:self.o + n]; self.o += n
        return v

    def u8(self): return struct.unpack("<B", self._take(1))[0]
    def i32(self): return struct.unpack("<i", self._take(4))[0]
    def u64(self): return struct.unpack("<Q", self._take(8))[0]
    def f64(self): return struct.unpack("<d", self._take(8))[0]
    def idpair(self): return (self.u64(), self.u64())

    def eigen(self, dtype=np.float64):
        r, c = self.i32(), self.i32()
        if r < 0 or c < 0 or r * c > (1 << 28):
            raise ValueError("implausible Eigen dimensions in archive")
        a = np.frombuffer(self._take(r * c * np.dtype(dtype).itemsize), dtype).reshape((r, c), order="F")
        return np.array(a)

    def eigen_vec(self, dtype):
        n = self.u64()
        return [self.eigen(dtype) for _ in range(n)]

    def f64_vec(self):
        n = self.u64()
        return np.frombuffer(self._take(8 * n), np.float64).copy()

    def cvmat(self):
        rows, cols, t, cont = self.i32(), self.i32(), self.i32(), self.u8()
        depth, ch = t & 7, (t >> 3) + 1
        es = {0: 1, 1: 1, 2: 2, 3: 2, 4: 4, 5: 4, 6: 8}[depth] * ch
        dt = {0: np.uint8, 1: np.int8, 2: np.uint16, 3: np.int16, 4: np.int32, 5: np.float32, 6: np.float64}[depth]
        data = self._take(rows * cols * es)      # row by row or in one block: the same bytes either way (:264-285)
        m = np.frombuffer(data, dt).reshape(rows, cols * ch) if rows * cols else np.zeros((0, 0), dt)
        return np.array(m), t

    def done(self): return self.o == len(self.b)


# ------------------------------------------------------------------------------------------------ messages
_CALIB_SCALARS = ("a_max", "g_max", "sigma_a_c", "sigma_g_c", "sigma_ba", "sigma_bg", "sigma_aw_c", "sigma_gw_c", "tau", "g")


def _w_calib(w: _W, c: dict):
    """VICalibration::serialize (typedefs_base.hpp:376-380)"""
    w.eigen(c["T_SC"], np.float64, (4, 4)); w.i32(c["cam_model"]); w.i32(c["dist_model"])
    w.eigen(c["img_dims"], np.float64, (2, 1)); w.eigen(c["dist_coeffs"]); w.eigen(c["intrinsics"])
    w.eigen(c["K"], np.float64, (3, 3))
    for k in _CALIB_SCALARS:
        w.f64(c[k])
    w.eigen(c["a0"], np.float64, (3, 1)); w.i32(c["rate"]); w.f64(c["delay_cam0_to_imu"]); w.f64(c["delay_cam1_to_imu"])


def _r_calib(r: _R) -> dict:
    c = dict(T_SC=r.eigen(), cam_model=r.i32(), dist_model=r.i32(), img_dims=r.eigen().reshape(-1),
             dist_coeffs=r.eigen().reshape(-1), intrinsics=r.eigen().reshape(-1), K=r.eigen())
    for k in _CALIB_SCALARS:
        c[k] = r.f64()
    c["a0"] = r.eigen().reshape(-1); c["rate"] = r.i32(); c["delay_cam0_to_imu"] = r.f64(); c["delay_cam1_to_imu"] = r.f64()
    return c


def encode_keyframe(kf: dict) -> bytes:
    """MsgKeyframe, save_to_file branch (msg_keyframe.hpp:129-143)"""
    w = _W()
    w.f64(kf["timestamp"]); w.idpair(kf["id"])
    _w_calib(w, kf["calibration"])
    for k in ("img_dim_x_min", "img_dim_y_min", "img_dim_x_max", "img_dim_y_max"):
        w.i32(kf[k])
    for sfx in ("", "_add"):
        w.eigen_vec(kf["keypoints_distorted" + sfx], np.float32, (2, 1))
        w.eigen_vec(kf["keypoints_undistorted" + sfx], np.float32, (2, 1))
        w.eigen_vec(kf["keypoints_aors" + sfx], np.float32, (4, 1))
        d = kf["descriptors" + sfx]
        w.cvmat(d, CV_32F if (d is not None and np.asarray(d).dtype == np.float32) else CV_8U)
    for k in ("T_s_c", "T_w_s", "T_w_s_vio"):
        w.eigen(kf[k], np.float64, (4, 4))
    for k in ("velocity", "bias_gyro", "bias_accel", "lin_acc", "ang_vel", "lin_acc_init", "ang_vel_init"):
        w.eigen(kf[k], np.float64, (3, 1))
    pre = kf["preintegration"]           # PreintegrationData::serialize (msg_keyframe.hpp:37-42)
    for k in ("acc", "gyr", "lin_bias_accel", "lin_bias_gyro"):
        w.eigen(pre[k], np.float64, (3, 1))
    for k in ("dt", "lin_acc_x", "lin_acc_y", "lin_acc_z", "ang_vel_x", "ang_vel_y", "ang_vel_z"):
        w.f64_vec(pre[k])
    lms = kf["landmarks"]                # std::map<int, idpair>: feature index → landmark id
    w.u64(len(lms))
    for fi in sorted(lms):
        w.i32(fi); w.idpair(lms[fi])
    w.idpair(kf["id_predecessor"]); w.idpair(kf["id_successor"])
    w.cvmat(kf.get("img"), CV_8U)
    return bytes(w.b)


def decode_keyframe(b: bytes) -> dict:
    r = _R(b)
    kf = dict(timestamp=r.f64(), id=r.idpair(), calibration=_r_calib(r))
    for k in ("img_dim_x_min", "img_dim_y_min", "img_dim_x_max", "img_dim_y_max"):
        kf[k] = r.i32()
    for sfx in ("", "_add"):
        for k, n in (("keypoints_distorted", 2), ("keypoints_undistorted", 2), ("keypoints_aors", 4)):
            v = r.eigen_vec(np.float32)
            kf[k + sfx] = np.array([e.reshape(-1) for e in v], np.float32).reshape(-1, n)
        kf["descriptors" + sfx], _ = r.cvmat()
    for k in ("T_s_c", "T_w_s", "T_w_s_vio"):
        kf[k] = r.eigen()
    for k in ("velocity", "bias_gyro", "bias_accel", "lin_acc", "ang_vel", "lin_acc_init", "ang_vel_init"):
        kf[k] = r.eigen().reshape(-1)
    pre = {k: r.eigen().reshape(-1) for k in ("acc", "gyr", "lin_bias_accel", "lin_bias_gyro")}
    for k in ("dt", "lin_acc_x", "lin_acc_y", "lin_acc_z", "ang_vel_x", "ang_vel_y", "ang_vel_z"):
        pre[k] = r.f64_vec()
    kf["preintegration"] = pre
    kf["landmarks"] = {}
    for _ in range(r.u64()):
        fi = r.i32(); kf["landmarks"][fi] = r.idpair()
    kf["id_predecessor"] = r.idpair(); kf["id_successor"] = r.idpair()
    kf["img"], _ = r.cvmat()
    if not r.done():
        raise ValueError("trailing bytes after MsgKeyframe")
    return kf


def encode_landmark(lm: dict) -> bytes:
    """MsgLandmark, save_to_file branch (msg_landmark.hpp:69-73): id, pos_w, observations (map<idpair,int>), id_reference"""
    w = _W()
    w.idpair(lm["id"]); w.eigen(lm["pos_w"], np.float64, (3, 1))
    obs = lm["observations"]
    w.u64(len(obs))
    for kfid in sorted(obs):
        w.idpair(kfid); w.i32(obs[kfid])
    w.idpair(lm["id_reference"])
    return bytes(w.b)


def decode_landmark(b: bytes) -> dict:
    r = _R(b)
    lm = dict(id=r.idpair(), pos_w=r.eigen().reshape(-1), observations={})
    for _ in range(r.u64()):
        k = r.idpair(); lm["observations"][k] = r.i32()
    lm["id_reference"] = r.idpair()
    if not r.done():
        raise ValueError("trailing bytes after MsgLandmark")
    return lm


def encode_mapdata(m: dict) -> bytes:
    """MsgMap::serialize (map_be.hpp:126-136): id_map, keyframes1, keyframes2, transforms12 (4x4), cov (6x6)"""
    w = _W()
    w.u64(m["id_map"])
    for k in ("keyframes1", "keyframes2"):
        w.u64(len(m[k]))
        for p in m[k]:
            w.idpair(p)
    w.eigen_vec(m["transforms12"], np.float64, (4, 4))
    w.eigen_vec(m["cov"], np.float64, (6, 6))
    return bytes(w.b)


def decode_mapdata(b: bytes) -> dict:
    r = _R(b)
    m = dict(id_map=r.u64())
    for k in ("keyframes1", "keyframes2"):
        m[k] = [r.idpair() for _ in range(r.u64())]
    m["transforms12"] = r.eigen_vec(np.float64); m["cov"] = r.eigen_vec(np.float64)
    if not r.done():
        raise ValueError("trailing bytes after MsgMap")
    return m


# ------------------------------------------------------------------------------------------------ flat problem ⇄ map
def _T(q, t):
    from .optimization import _quat_to_rot
    T = np.eye(4); T[:3, :3] = _quat_to_rot(np.asarray(q, np.float64)[None])[0]; T[:3, 3] = t
    return T


def _qt(T):
    from .optimization import _rot_to_quat
    return np.concatenate([_rot_to_quat(np.asarray(T)[None, :3, :3])[0], np.asarray(T)[:3, 3]])


def write_map(path: str, p: dict, descriptors=None, map_id: int = 0, descriptors_add=None, keypoints_add=None):
    """Flat problem → COVINS map directory.  Every observation of a keyframe becomes one of its keypoints (feature index =
    its position among the keyframe's observations in landmark order); `descriptors` (optional, [n_obs, 32] u8) are the
    ORB rows of those features.  Octave is recovered from sigma = 2 (octave + 1) (optimization_be.cpp:183-184).
    `descriptors_add` (optional, list of K arrays [n_k, 32] u8 or [n_k, 128] f32): the ADDITIONAL feature set of every
    keyframe (descriptors_add_, keyframe_be.hpp:111) — the set the place-recognition k-NN runs on
    (placerec_gen_be.cpp:82-100); `keypoints_add` (optional, list of K arrays [n_k, 2] f32) their distorted keypoints."""
    os.makedirs(os.path.join(path, "keyframes"), exist_ok=True)
    os.makedirs(os.path.join(path, "mappoints"), exist_ok=True)
    K, L = int(p["K"]), int(p["L"])
    agent = np.asarray(p["agent_of"]); kid = np.asarray(p["kf_id"])
    ids = [(int(kid[k]), int(agent[k])) for k in range(K)]
    obs_lm = np.repeat(np.arange(L), np.diff(p["lm_obs_ptr"]))
    order = np.argsort(p["obs_kf"], kind="stable")
    kf_ptr = np.concatenate([[0], np.cumsum(np.bincount(p["obs_kf"], minlength=K))])
    feat_of_obs = np.empty(len(order), np.int64)
    feat_of_obs[order] = np.arange(len(order)) - kf_ptr[np.asarray(p["obs_kf"])[order]]
    noise = p.get("imu_noise", np.array([0.0, 0.0, 0.0, 0.0, 9.81]))
    imu_of_j = {int(j): f for f, j in enumerate(p["imu_j"])}
    for k in range(K):
        c = int(p["cam_of_kf"][k]) if p.get("cam_of_kf") is not None else 0
        T_sc = _T(p["extr"][c][:4], p["extr"][c][4:])
        fx, fy, cx, cy = p["intr"][c]
        sel = order[kf_ptr[k]:kf_ptr[k + 1]]
        uv = np.asarray(p["obs_uv"], np.float32)[sel]
        octv = np.rint(np.asarray(p["obs_sigma"])[sel] / 2.0 - 1.0).astype(np.float32)
        aors = np.zeros((len(sel), 4), np.float32); aors[:, 1] = octv
        calib = dict(T_SC=T_sc, cam_model=0, dist_model=0, img_dims=[752.0, 480.0], dist_coeffs=p["dist"][c], intrinsics=p["intr"][c],
                     K=[[fx, 0, cx], [0, fy, cy], [0, 0, 1]], a_max=0.0, g_max=0.0, sigma_a_c=noise[0], sigma_g_c=noise[1],
                     sigma_ba=0.0, sigma_bg=0.0, sigma_aw_c=noise[2], sigma_gw_c=noise[3], tau=0.0, g=noise[4], a0=[0, 0, 0],
                     rate=200, delay_cam0_to_imu=0.0, delay_cam1_to_imu=0.0)
        pre = dict(acc=np.zeros(3), gyr=np.zeros(3), lin_bias_accel=p["speedbias"][k][3:6], lin_bias_gyro=p["speedbias"][k][6:9],
                   dt=[], lin_acc_x=[], lin_acc_y=[], lin_acc_z=[], ang_vel_x=[], ang_vel_y=[], ang_vel_z=[])
        acc0 = gyr0 = np.zeros(3)
        if k in imu_of_j:
            f = imu_of_j[k]; a, b = int(p["imu_ptr"][f]), int(p["imu_ptr"][f + 1])
            acc, gyr = np.asarray(p["imu_acc"])[a:b], np.asarray(p["imu_gyr"])[a:b]
            pre.update(dt=np.asarray(p["imu_dt"])[a:b], lin_acc_x=acc[:, 0], lin_acc_y=acc[:, 1], lin_acc_z=acc[:, 2],
                       ang_vel_x=gyr[:, 0], ang_vel_y=gyr[:, 1], ang_vel_z=gyr[:, 2], acc=acc[0], gyr=gyr[0])
            acc0, gyr0 = p["imu_acc0"][f], p["imu_gyr0"][f]
        d_add = None if descriptors_add is None else np.asarray(descriptors_add[k])
        n_add = 0 if d_add is None else len(d_add)
        kp_add = np.zeros((n_add, 2), np.float32) if keypoints_add is None else np.asarray(keypoints_add[k], np.float32).reshape(n_add, 2)
        same_prev = k > 0 and agent[k - 1] == agent[k]
        same_next = k + 1 < K and agent[k + 1] == agent[k]
        T_ws = _T(p["pose"][k][:4], p["pose"][k][4:])
        kf = dict(timestamp=float(kid[k]) * 0.25, id=ids[k], calibration=calib, img_dim_x_min=0, img_dim_y_min=0, img_dim_x_max=752,
                  img_dim_y_max=480, keypoints_distorted=uv, keypoints_undistorted=uv, keypoints_aors=aors,
                  descriptors=None if descriptors is None else np.asarray(descriptors, np.uint8)[sel],
                  keypoints_distorted_add=kp_add, keypoints_undistorted_add=kp_add,
                  keypoints_aors_add=np.zeros((len(kp_add), 4), np.float32), descriptors_add=d_add,
                  T_s_c=T_sc, T_w_s=T_ws, T_w_s_vio=T_ws, velocity=p["speedbias"][k][0:3], bias_gyro=p["speedbias"][k][6:9],
                  bias_accel=p["speedbias"][k][3:6], lin_acc=np.zeros(3), ang_vel=np.zeros(3), lin_acc_init=acc0, ang_vel_init=gyr0,
                  preintegration=pre, landmarks={int(feat_of_obs[o]): (int(obs_lm[o]), 0) for o in sel},
                  id_predecessor=ids[k - 1] if same_prev else DEFPAIR, id_successor=ids[k + 1] if same_next else DEFPAIR, img=None)
        with open(os.path.join(path, "keyframes", f"keyframes{k}.txt"), "wb") as f:
            f.write(encode_keyframe(kf))
    for l in range(L):
        a, b = int(p["lm_obs_ptr"][l]), int(p["lm_obs_ptr"][l + 1])
        if b - a < 2:                       # Map::SaveToFile skips them (map_be.cpp:880-882)
            continue
        obs = {ids[int(p["obs_kf"][o])]: int(feat_of_obs[o]) for o in range(a, b)}
        lm = dict(id=(l, 0), pos_w=p["lm"][l], observations=obs, id_reference=ids[int(p["obs_kf"][a])])
        with open(os.path.join(path, "mappoints", f"mappoints{l}.txt"), "wb") as f:
            f.write(encode_landmark(lm))
    nl = len(p.get("loop_i", []))
    m = dict(id_map=map_id, keyframes1=[ids[int(i)] for i in p.get("loop_i", [])], keyframes2=[ids[int(j)] for j in p.get("loop_j", [])],
             transforms12=[_T(p["loop_q"][e], p["loop_t"][e]) for e in range(nl)],
             cov=[np.asarray(p["loop_cov"][e]) if "loop_cov" in p else np.eye(6) for e in range(nl)])
    with open(os.path.join(path, "mapdata.txt"), "wb") as f:
        f.write(encode_mapdata(m))


def read_map(path: str) -> dict:
    """COVINS map directory → flat problem (+ `descriptors` [n_obs, 32] of the observed features, `kf_descriptors` — the
    per-keyframe `descriptors` matrices that DenseMatcher / ComputeDescriptor read (keyframe_base.cpp:258-260,
    landmark_be.cpp:57-64) — and `kf_descriptors_add`, the per-keyframe `descriptors_add` matrices that the
    place-recognition k-NN (cvb_match_hamming_batch / cvb_db_*) must be fed with, as placerec_gen_be.cpp:82-100 does).
    Canonical orders as in synth_map: keyframes by
    (client_id, kf_id), landmarks by (client_id, id), a landmark's observations by keyframe index."""
    def _load(sub, dec):
        d = os.path.join(path, sub)
        out = []
        for fn in sorted(os.listdir(d)):       # LoadFromFile takes whatever readdir returns (map_be.cpp:529-562)
            with open(os.path.join(d, fn), "rb") as f:
                out.append(dec(f.read()))
        return out
    kfs = sorted(_load("keyframes", decode_keyframe), key=lambda k: (k["id"][1], k["id"][0]))
    lms = sorted(_load("mappoints", decode_landmark), key=lambda l: (l["id"][1], l["id"][0]))
    with open(os.path.join(path, "mapdata.txt"), "rb") as f:
        md = decode_mapdata(f.read())
    K, L = len(kfs), len(lms)
    index = {k["id"]: i for i, k in enumerate(kfs)}
    pose = np.array([_qt(k["T_w_s"]) for k in kfs]).reshape(K, 7)
    sb = np.array([np.concatenate([k["velocity"], k["bias_accel"], k["bias_gyro"]]) for k in kfs]).reshape(K, 9)
    # distinct cameras (extrinsics + intrinsics + distortion)
    cams, cam_of_kf, extr, intr, dist = {}, np.zeros(K, np.int32), [], [], []
    for i, k in enumerate(kfs):
        c = k["calibration"]
        key = (k["T_s_c"].tobytes(), c["intrinsics"].tobytes(), c["dist_coeffs"].tobytes())
        if key not in cams:
            cams[key] = len(cams); extr.append(_qt(k["T_s_c"])); intr.append(c["intrinsics"][:4]); dist.append(np.resize(c["dist_coeffs"], 4))
        cam_of_kf[i] = cams[key]
    lm_pos = np.array([l["pos_w"] for l in lms]).reshape(L, 3)
    lm_obs_ptr, obs_kf, obs_uv, obs_sigma, desc = [0], [], [], [], []
    for l in lms:
        for kfid, fi in sorted(l["observations"].items(), key=lambda kv: index.get(kv[0], 1 << 60)):
            if kfid not in index:
                continue
            k = kfs[index[kfid]]
            obs_kf.append(index[kfid]); obs_uv.append(k["keypoints_distorted"][fi])
            obs_sigma.append(2.0 * (float(k["keypoints_aors"][fi][1]) + 1.0))      # optimization_be.cpp:183-184
            if k["descriptors"].size:
                desc.append(k["descriptors"][fi])
        lm_obs_ptr.append(len(obs_kf))
    imu_i, imu_j, ptr, dts, accs, gyrs, acc0, gyr0 = [], [], [0], [], [], [], [], []
    for j, k in enumerate(kfs):
        pre = k["preintegration"]
        if len(pre["dt"]) == 0 or k["id_predecessor"] not in index:
            continue
        imu_i.append(index[k["id_predecessor"]]); imu_j.append(j)
        dts.append(pre["dt"]); accs.append(np.stack([pre["lin_acc_x"], pre["lin_acc_y"], pre["lin_acc_z"]], 1))
        gyrs.append(np.stack([pre["ang_vel_x"], pre["ang_vel_y"], pre["ang_vel_z"]], 1))
        acc0.append(k["lin_acc_init"]); gyr0.append(k["ang_vel_init"]); ptr.append(ptr[-1] + len(pre["dt"]))
    c0 = kfs[0]["calibration"] if K else None
    nl = len(md["keyframes1"])
    p = dict(K=K, L=L, pose=pose, speedbias=sb, pose_const=np.array([1 if (k["id"][0] == 0 and k["id"][1] == md["id_map"]) else 0 for k in kfs], np.uint8),   # optimization_be.cpp:88-89
             cam_of_kf=cam_of_kf, extr=np.array(extr).reshape(-1, 7), intr=np.array(intr).reshape(-1, 4), dist=np.array(dist).reshape(-1, 4),
             lm=lm_pos, lm_obs_ptr=np.array(lm_obs_ptr, np.int32), obs_kf=np.array(obs_kf, np.int32),
             obs_uv=np.array(obs_uv, np.float32).reshape(-1, 2), obs_sigma=np.array(obs_sigma, np.float64),
             agent_of=np.array([k["id"][1] for k in kfs], np.int32), kf_id=np.array([k["id"][0] for k in kfs], np.int32),
             imu_i=np.array(imu_i, np.int32), imu_j=np.array(imu_j, np.int32), imu_ptr=np.array(ptr, np.int32),
             imu_dt=np.concatenate(dts) if dts else np.zeros(0), imu_acc=np.concatenate(accs) if accs else np.zeros((0, 3)),
             imu_gyr=np.concatenate(gyrs) if gyrs else np.zeros((0, 3)), imu_acc0=np.array(acc0).reshape(-1, 3),
             imu_gyr0=np.array(gyr0).reshape(-1, 3),
             imu_noise=np.array([c0["sigma_a_c"], c0["sigma_g_c"], c0["sigma_aw_c"], c0["sigma_gw_c"], c0["g"]]) if K else np.zeros(5),
             loop_i=np.array([index[a] for a in md["keyframes1"]], np.int32), loop_j=np.array([index[b] for b in md["keyframes2"]], np.int32),
             loop_q=np.array([_qt(T)[:4] for T in md["transforms12"]]).reshape(nl, 4),
             loop_t=np.array([_qt(T)[4:] for T in md["transforms12"]]).reshape(nl, 3),
             loop_cov=np.array(md["cov"]).reshape(nl, 6, 6),
             descriptors=np.array(desc, np.uint8).reshape(-1, 32) if desc else np.zeros((0, 32), np.uint8),
             kf_descriptors=[k["descriptors"] for k in kfs], kf_descriptors_add=[k["descriptors_add"] for k in kfs],
             kf_keypoints_add=[k["keypoints_distorted_add"] for k in kfs], lm_ids=[l["id"] for l in lms])
    # what the pose graph's write-back reads (covins_b200.optimization.pgo_map_problem): the stored 4x4 poses, the chain links and
    # each landmark's reference keyframe, as keyframe indices (-1 none, -2 a keyframe that is not in the map)
    link = lambda i: -1 if i == DEFPAIR else index.get(i, -2)
    p.update(T_ws=np.array([k["T_w_s"] for k in kfs], np.float64).reshape(K, 4, 4),
             T_ws_vio=np.array([k["T_w_s_vio"] for k in kfs], np.float64).reshape(K, 4, 4),
             kf_pred=np.array([link(k["id_predecessor"]) for k in kfs], np.int32), kf_succ=np.array([link(k["id_successor"]) for k in kfs], np.int32),
             lm_ref=np.array([link(l["id_reference"]) for l in lms], np.int32),
             lm_has_obs=np.array([len(l["observations"]) > 0 for l in lms], np.uint8))
    return p
