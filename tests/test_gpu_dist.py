"""GPU test of the sharded (multi-GPU) evaluation: needs >= 2 devices, skipped otherwise (on a single H100 it skips;
tools/dist_check.py is the same check for a multi-GPU session). The sharded layout on one GPU, through a one-rank
communicator, is tested in tests/test_gpu_sharded_single_rank.py."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_two_gpu_sharded_evaluation_matches_oracle():
    from gpy_b200 import _ffi
    if _ffi.lib().gpx_device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", "29533", os.path.join(ROOT, "tools", "dist_check.py"), "700,2048"]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = [l for l in out.stdout.splitlines() if l.startswith("G=2")]
    assert len(lines) == 4, out.stdout
    for l in lines:
        f = l.split()
        lml_abs = float(f[f.index("abs") + 1])
        grad_rel = float(f[f.index("grad") + 2])
        assert lml_abs <= 1e-8 and grad_rel <= 1e-6, l
        assert float(f[f.index("predict") + 1]) <= 1e-7, l
        assert float(f[f.index("L") + 2]) <= 1e-10, l          # the sharded woodbury_chol, gathered collectively


def test_two_gpu_row_sharded_sparse_matches_oracle():
    """gpx_sparse_eval with a communicator: data rows sharded over 2 GPUs, psi statistics / Knm gradients all-reduced
    (the pattern of var_dtc_parallel.py:113-131); every rank must reproduce the oracle on the whole data set."""
    from gpy_b200 import _ffi
    if _ffi.lib().gpx_device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", "29534", os.path.join(ROOT, "tools", "dist_sparse_check.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = [l for l in out.stdout.splitlines() if l.startswith("SPARSE G=2")]
    assert len(lines) == 4, out.stdout
    for l in lines:
        f = l.split()
        assert float(f[f.index("lml") + 4]) <= 1e-8 and float(f[f.index("grad") + 2]) <= 1e-6, l
        assert float(f[f.index("Zgrad") + 2]) <= 1e-6 and float(f[f.index("predict") + 1]) <= 1e-6, l
