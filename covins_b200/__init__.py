"""covins_b200 — H100-native (sm_90a) implementation of the COVINS server hot path:
place-recognition descriptor matching and PGO / global bundle adjustment, behind the C-ABI of
include/covins_b200.h.  Python here is only the host-side mirror used by tests and bench.py; the
reference-facing host code is C++ (covins_b200/csrc/host)."""
from ._lib import Context, CvbError, build, lib, LIB_PATH  # noqa: F401
