"""Launch accounting of the composite sparse evaluation (gpx_sparse_eval_multi), as tests/test_gpu_launch_accounting.py
does for the other calls: around each call the CUDA kernel activities recorded by torch.profiler are counted and compared
with the call's total_launches() delta (the child contexts' factorisations, the elementwise rank-P pass, one Knm and one
Kmm reduction per part, the composite gradients_X and its reduce included); then sparse_get after it."""
import json
import os
import tempfile

import pytest

import sparse_composite_oracle as so
from gpy_b200 import _ffi

pytestmark = pytest.mark.gpu


def _kernels(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)["traceEvents"]
    return [ev["name"] for ev in events if ev.get("cat") == "kernel"]


def test_composite_sparse_calls_count_every_launch():
    X, Y, Z, nv = so.case_data(1500, 600, 3, 2, 71, True)
    parts = [so.descriptor(p) for p in so.KERNELS["m52_x_rbf_plus_exp"]]
    e = _ffi.Engine(0)
    try:
        e.sparse_set_data(X, Y)
        _kernels(lambda: None)
        e.sparse_eval_multi(parts, Z, 0.05)   # warm-up: child contexts and their workspaces
        e.sparse_eval_multi(parts, Z, nv)
        for noise, what in ((0.05, "scalar"), (nv, "per-point")):
            l0 = e.total_launches()
            names = _kernels(lambda: e.sparse_eval_multi(parts, Z, noise))
            assert len(names) == e.total_launches() - l0, (what, len(names), e.total_launches() - l0)
            assert sum("gradx_multi_kernel" in n for n in names) == 2                       # Knm and Kmm
            assert sum("grad_full_multi" in n for n in names) == 2 * len(parts)            # one per part, each
            assert sum("add_rank_p" in n for n in names) == 1
            for w in e.SPARSE_GET:
                l0 = e.total_launches()
                names = _kernels(lambda: e.sparse_get(w))
                assert len(names) == e.total_launches() - l0, (what, w, len(names), e.total_launches() - l0)
    finally:
        e.close()
