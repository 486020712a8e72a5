"""The SIFT form of the C++ wrapper's DescriptorDatabase (covins_b200_shim.hpp) against MatchCandidatesSIFT and the Python path."""
import subprocess

import numpy as np
import pytest

from covins_b200 import matching as M, synth
from ransac_helpers import _build_shim


def _read(path):
    v = np.fromfile(path, np.int32)
    out, pos = [], 0
    while pos < len(v):
        n = v[pos]
        out.append(v[pos + 1:pos + 1 + 3 * n].reshape(-1, 3))
        pos += 1 + 3 * n
    return out


def test_shim_sift_db_compiles_and_links(tmp_path):
    exe = str(tmp_path / "shim_sift_db_test")
    _build_shim("shim_sift_db_test.cpp", exe)
    assert subprocess.run([exe, str(tmp_path)]).returncode == 2        # nothing dumped: stops before any GPU work


@pytest.mark.gpu
def test_shim_sift_db_equals_match_candidates(ctx, tmp_path):
    exe = str(tmp_path / "shim_sift_db_test")
    _build_shim("shim_sift_db_test.cpp", exe)
    s, _ = synth.sift_keyframes(seed=23, n_kf=7, n_feat=300, n_lm=500, window=500)
    lens = [300, 0, 129, 1, 300, 128]
    t = np.concatenate([s[i + 1][:n] for i, n in enumerate(lens)])
    seg = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    s[0].tofile(tmp_path / "q.bin"); t.tofile(tmp_path / "t.bin"); seg.tofile(tmp_path / "seg.bin")
    np.array([500.0, 0.8], np.float32).tofile(tmp_path / "thr.bin")
    subprocess.check_call([exe, str(tmp_path)])
    ref = _read(tmp_path / "sift_all.bin")
    got = _read(tmp_path / "sift_db.bin")
    assert len(got) == len(ref) == len(lens)
    assert all(np.array_equal(a, b) for a, b in zip(got, ref))
    assert sum(len(a) for a in ref) > 0
    mt, md, nm = M.match_candidates_l2(ctx, s[0], t, seg, 500.0, 0.8)
    for k in range(len(lens)):
        qq = np.flatnonzero(mt[k] >= 0)
        assert np.array_equal(ref[k][:, 0], qq) and np.array_equal(ref[k][:, 1], mt[k][qq])
        assert np.array_equal(ref[k][:, 2], md[k][qq].view(np.int32))
    rm = _read(tmp_path / "sift_db_rm.bin")
    assert len(rm) == len(lens) - 1
    assert all(np.array_equal(a, b) for a, b in zip(rm, ref[:1] + ref[2:]))
