"""ctypes loader for libcovins_b200.so (the C-ABI of include/covins_b200.h).

There is no CPU fallback: if the shared library is missing this raises, and if no CUDA device is
present every compute call fails with CVB_ERR_CUDA — the product path never routes through oracle/.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libcovins_b200.so")
_lib = None

c_i32p = C.POINTER(C.c_int32)
c_u8p = C.POINTER(C.c_uint8)
c_f32p = C.POINTER(C.c_float)
c_f64p = C.POINTER(C.c_double)
c_vp = C.c_void_p


class CvbError(RuntimeError):
    pass


def build(force: bool = False) -> str:
    """Compile every CUDA source for sm_90a with nvcc (in-tree: covins_b200/libcovins_b200.so)."""
    args = ["make", "-C", os.path.join(_HERE, "csrc"), "-j8", "-s"]
    if force:
        args.append("-B")
    subprocess.check_call(args)
    return LIB_PATH


# name: (restype, [argtypes])  — must list every symbol include/covins_b200.h declares
SIGNATURES = {
    "cvb_version": (C.c_int, []),
    "cvb_ctx_create": (C.c_int, [C.c_int, C.POINTER(c_vp)]),
    "cvb_ctx_destroy": (C.c_int, [c_vp]),
    "cvb_last_error": (C.c_char_p, [c_vp]),
    "cvb_ctx_sync": (C.c_int, [c_vp]),
    "cvb_launch_count": (C.c_int64, [c_vp]),
    "cvb_knn_hamming_batch": (C.c_int, [c_vp, c_vp, C.c_int, c_vp, c_vp, C.c_int, C.c_int, c_vp, c_vp]),
    "cvb_knn_hamming_batch_dev": (C.c_int, [c_vp, c_vp, C.c_int, c_vp, c_vp, c_vp, C.c_int, C.c_int, c_vp, c_vp, c_vp]),
    "cvb_match_hamming_batch": (C.c_int, [c_vp, c_vp, C.c_int, c_vp, c_vp, C.c_int, C.c_float, C.c_float, c_vp, c_vp, c_vp]),
    "cvb_match_hamming_batch_dev": (C.c_int, [c_vp, c_vp, C.c_int, c_vp, c_vp, c_vp, C.c_int, C.c_float, C.c_float,
                                              c_vp, c_vp, c_vp, c_vp]),
    "cvb_db_create": (C.c_int, [c_vp, C.c_int, C.POINTER(c_vp)]),
    "cvb_db_destroy": (C.c_int, [c_vp, c_vp]),
    "cvb_db_reserve": (C.c_int, [c_vp, c_vp, C.c_int64]),
    "cvb_db_append": (C.c_int, [c_vp, c_vp, c_vp, c_vp, C.c_int]),
    "cvb_db_size": (C.c_int, [c_vp, C.POINTER(C.c_int32), C.POINTER(C.c_int64)]),
    "cvb_db_match_hamming": (C.c_int, [c_vp, c_vp, c_vp, C.c_int, C.c_float, C.c_float, c_vp, c_vp, c_vp, c_vp, c_vp,
                                       C.c_int, C.POINTER(C.c_int32)]),
    "cvb_db_match_hamming_dev": (C.c_int, [c_vp, c_vp, c_vp, C.c_int, C.c_float, C.c_float, c_vp, c_vp, c_vp, c_vp]),
    "cvb_knn_l2_batch": (C.c_int, [c_vp, c_vp, C.c_int, c_vp, c_vp, C.c_int, C.c_int, C.c_int, c_vp, c_vp]),
    "cvb_knn_l2_u8_batch_dev": (C.c_int, [c_vp, c_vp, C.c_int, c_vp, c_vp, c_vp, C.c_int, C.c_int, C.c_int, c_vp, c_vp, c_vp]),
    "cvb_match_l2_batch": (C.c_int, [c_vp, c_vp, C.c_int, c_vp, c_vp, C.c_int, C.c_int, C.c_float, C.c_float, c_vp, c_vp, c_vp]),
    "cvb_knn_merge_shards_dev": (C.c_int, [c_vp, c_vp, c_vp, C.c_int, c_vp, C.c_int, C.c_int64, C.c_int, c_vp, c_vp, c_vp]),
    "cvb_landmark_descriptor_batch": (C.c_int, [c_vp, c_vp, c_vp, C.c_int, c_vp, c_vp]),
    "cvb_landmark_descriptor_batch_dev": (C.c_int, [c_vp, c_vp, c_vp, C.c_int, c_vp, c_vp, c_vp]),
    "cvb_quantize_u8_dev": (C.c_int, [c_vp, c_vp, C.c_int64, c_vp, c_vp, c_vp]),
    "cvb_landmark_match_batch": (C.c_int, [c_vp, c_vp, c_vp, C.c_int, c_vp, c_vp, c_vp, C.c_int, C.c_float, C.c_int,
                                           c_vp, c_vp, c_vp, c_vp]),
    "cvb_landmark_match_batch_dev": (C.c_int, [c_vp, c_vp, c_vp, C.c_int, c_vp, c_vp, c_vp, c_vp, C.c_int, C.c_float,
                                               C.c_int, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "cvb_microbench_popc": (C.c_int, [c_vp, C.c_int, c_f64p]),
    "cvb_microbench_minmax": (C.c_int, [c_vp, c_f64p]),
    "cvb_microbench_latency": (C.c_int, [c_vp, c_f64p]),
    "cvb_microbench_potrf": (C.c_int, [c_vp, C.c_int, c_f64p, c_vp]),
    "cvb_dense_cholesky_solve": (C.c_int, [c_vp, c_vp, C.c_int, c_vp, c_vp, c_f64p]),
    "cvb_ba_create": (C.c_int, [c_vp, c_vp, c_vp, C.POINTER(c_vp)]),
    "cvb_ba_set_allreduce": (C.c_int, [c_vp, c_vp, c_vp]),
    "cvb_ba_restart": (C.c_int, [c_vp]),
    "cvb_ba_enable_p2p": (C.c_int, [c_vp]),
    "cvb_db_remove": (C.c_int, [c_vp, c_vp, C.c_int]),
    "cvb_optimize_relative_pose": (C.c_int, [c_vp, c_vp, C.c_double, c_vp, c_vp, c_vp, c_vp]),
    "cvb_search_by_se3_batch": (C.c_int, [c_vp, c_vp, c_vp, C.c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "cvb_search_by_projection": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, C.c_int, C.c_int, C.c_double, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "cvb_score_absolute_pose_batch": (C.c_int, [c_vp, c_vp, C.c_int, c_vp, c_vp, c_vp, C.c_int, c_vp, c_vp, C.c_double, c_vp, c_vp, c_vp]),
    "cvb_score_relative_pose_batch": (C.c_int, [c_vp, c_vp, C.c_int, c_vp, c_vp, c_vp, c_vp, C.c_int, C.c_double, c_vp, c_vp, c_vp]),
    "cvb_ransac_absolute_pose_batch": (C.c_int, [c_vp, c_vp, C.c_double, C.c_int, C.c_double, c_vp]),
    "cvb_ransac_noncentral_relative_pose_batch": (C.c_int, [c_vp, c_vp, C.c_double, C.c_int, C.c_double, c_vp]),
    "cvb_ransac_central_relative_pose_batch": (C.c_int, [c_vp, c_vp, C.c_double, C.c_int, C.c_double, c_vp]),
    "cvb_ba_iterate": (C.c_int, [c_vp, C.c_int, C.POINTER(C.c_int)]),
    "cvb_ba_result_get": (C.c_int, [c_vp, c_vp, c_vp]),
    "cvb_ba_reproj_norms": (C.c_int, [c_vp, c_vp, C.c_int]),
    "cvb_ba_debug_vector": (C.c_int, [c_vp, C.c_int, c_vp, C.c_int64, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "cvb_ba_timing": (C.c_int, [c_vp, c_f64p, C.c_int]),
    "cvb_ba_destroy": (C.c_int, [c_vp]),
    "cvb_ba_solve": (C.c_int, [c_vp, c_vp, c_vp, c_vp]),
    "cvb_gba": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp]),
}


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise CvbError(f"{LIB_PATH} is missing — run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(there is no CPU fallback)")
        _lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(_lib, name)
            fn.restype = res
            fn.argtypes = args
    return _lib


class Context:
    """One cvb_ctx: one device, one stream, grow-only device workspaces. Not thread-safe."""

    def __init__(self, device: int = 0):
        self._h = c_vp()
        rc = lib().cvb_ctx_create(device, C.byref(self._h))
        if rc != 0:
            raise CvbError(f"cvb_ctx_create(device={device}) failed with status {rc}: no usable CUDA device "
                           "(libcovins_b200 has no CPU fallback)")
        self.device = device

    @property
    def handle(self):
        return self._h

    def check(self, rc: int):
        if rc != 0:
            msg = lib().cvb_last_error(self._h)
            raise CvbError(f"status {rc}: {msg.decode() if msg else ''}")

    def sync(self):
        self.check(lib().cvb_ctx_sync(self._h))

    def launch_count(self) -> int:
        return int(lib().cvb_launch_count(self._h))

    def close(self):
        if self._h:
            lib().cvb_ctx_destroy(self._h)
            self._h = c_vp()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
