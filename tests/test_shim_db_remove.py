"""The C++ wrapper's DescriptorDatabase::RemoveKeyframes (covins_b200_shim.hpp): one batch equals a loop of RemoveKeyframe
from the highest index down, for the single-context and the group database, ORB and SIFT."""
import subprocess

import numpy as np
import pytest

from covins_b200 import synth
from ransac_helpers import _build_shim


def test_shim_db_remove_compiles_and_links(tmp_path):
    exe = str(tmp_path / "shim_db_remove_test")
    _build_shim("shim_db_remove_test.cpp", exe)
    assert subprocess.run([exe, str(tmp_path), "2"]).returncode == 2     # nothing dumped: stops before any GPU work


@pytest.mark.gpu
def test_shim_remove_keyframes_equals_the_loop(tmp_path):
    exe = str(tmp_path / "shim_db_remove_test")
    _build_shim("shim_db_remove_test.cpp", exe)
    lens = [300, 0, 129, 1, 300, 128, 257, 40, 300, 127, 0, 200]
    o, _ = synth.orb_keyframes(seed=51, n_kf=len(lens) + 1, n_feat=300, n_lm=600, window=600)
    s, _ = synth.sift_keyframes(seed=53, n_kf=len(lens) + 1, n_feat=300, n_lm=600, window=600)
    np.concatenate([o[i + 1][:n] for i, n in enumerate(lens)]).tofile(tmp_path / "orb_t.bin")
    np.concatenate([s[i + 1][:n] for i, n in enumerate(lens)]).tofile(tmp_path / "sift_t.bin")
    o[0].tofile(tmp_path / "orb_q.bin"); s[0].tofile(tmp_path / "sift_q.bin")
    np.concatenate([[0], np.cumsum(lens)]).astype(np.int32).tofile(tmp_path / "seg.bin")
    np.array([7, 1, 3, 10, 4], np.int32).tofile(tmp_path / "rm.bin")     # unsorted, an empty keyframe among them
    np.array([40.0, 0.8, 500.0, 0.8], np.float32).tofile(tmp_path / "thr.bin")
    assert subprocess.run([exe, str(tmp_path), "2"]).returncode == 0
    counts = np.fromfile(tmp_path / "counts.bin", np.int32)
    assert (counts > 0).all(), counts
