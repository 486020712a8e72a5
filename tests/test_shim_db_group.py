"""The C++ wrapper's DescriptorDatabase over a ContextGroup (covins_b200_shim.hpp): MatchAll equals the single-context
database's, ORB and SIFT, before and after a removal."""
import subprocess

import numpy as np
import pytest

from covins_b200 import synth
from ransac_helpers import _build_shim


def test_shim_db_group_compiles_and_links(tmp_path):
    exe = str(tmp_path / "shim_db_group_test")
    _build_shim("shim_db_group_test.cpp", exe)
    assert subprocess.run([exe, str(tmp_path), "2"]).returncode == 2     # nothing dumped: stops before any GPU work


@pytest.mark.gpu
def test_shim_db_group_equals_single_context(tmp_path):
    exe = str(tmp_path / "shim_db_group_test")
    _build_shim("shim_db_group_test.cpp", exe)
    lens = [300, 0, 129, 1, 300, 128, 257, 40]
    o, _ = synth.orb_keyframes(seed=41, n_kf=len(lens) + 1, n_feat=300, n_lm=600, window=600)
    s, _ = synth.sift_keyframes(seed=43, n_kf=len(lens) + 1, n_feat=300, n_lm=600, window=600)
    np.concatenate([o[i + 1][:n] for i, n in enumerate(lens)]).tofile(tmp_path / "orb_t.bin")
    np.concatenate([s[i + 1][:n] for i, n in enumerate(lens)]).tofile(tmp_path / "sift_t.bin")
    o[0].tofile(tmp_path / "orb_q.bin"); s[0].tofile(tmp_path / "sift_q.bin")
    np.concatenate([[0], np.cumsum(lens)]).astype(np.int32).tofile(tmp_path / "seg.bin")
    np.array([40.0, 0.8, 500.0, 0.8], np.float32).tofile(tmp_path / "thr.bin")
    assert subprocess.run([exe, str(tmp_path), "3"]).returncode == 0
    counts = np.fromfile(tmp_path / "counts.bin", np.int32)
    assert (counts > 0).all(), counts
