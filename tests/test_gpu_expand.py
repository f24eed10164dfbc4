"""The record-path dynamics-expansion kernels (rollout.cu): k_expand_lie_rec (default) must write the same [A_e B_e] blocks, bit for bit, as
k_expand_lie (TO_EXPAND_V1=1) -- after to_expand at the benchmark size and at sizes with partial knot blocks, and inside iLQR iterations whose
expansions are the overlapped mode 1 / mode 2 launches over the late list.  The kernel choice is read once per process, so the two runs are
subprocesses of profiles/scripts/expand_ab.py."""
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPT = os.path.join(ROOT, "profiles", "scripts", "expand_ab.py")


def _dump(path, **env):
    e = dict(os.environ); e.update(env)
    subprocess.run([sys.executable, SCRIPT, str(path)], check=True, env=e, timeout=900, stdout=subprocess.DEVNULL)
    return np.load(path)


def test_record_dynamics_expansion_is_bit_identical(tmp_path):
    a = _dump(tmp_path / "v1.npz", TO_EXPAND_V1="1")
    b = _dump(tmp_path / "v2.npz", TO_EXPAND_V1="0")
    assert sorted(a.files) == sorted(b.files) and len(a.files) >= 40
    for k in a.files:
        if k.endswith("_sha256"):
            continue
        assert np.all(np.isfinite(a[k])), k
        assert np.array_equal(a[k], b[k]), f"{k}: max |v1 - v2| = {np.max(np.abs(a[k] - b[k])):.3e}"
    for k in a.files:
        if k.endswith("_sha256"):
            assert np.array_equal(a[k], b[k]), f"{k}: digests differ"
    # the closed-form columns (positions, velocities) are in the blocks of both: 1 on the diagonal
    ab = a["ABe_3_5"]
    assert np.all(ab[..., [0, 1, 2, 6, 7, 8], [0, 1, 2, 6, 7, 8]] == 1.0)
