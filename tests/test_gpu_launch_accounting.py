"""Launch accounting: gpx_total_launches of a context counts every kernel a call on that context issues, including the
kernels the sparse evaluation runs on its child contexts (the factorisations of Kmm and of B = I + A) and the assembles
it issues on their streams. Around each call, the CUDA kernel activities recorded by torch.profiler are counted (copies
and memsets are not kernels) and compared with the call's total_launches() delta."""
import ctypes
import json
import os
import tempfile

import numpy as np
import pytest

from gpy_b200 import _ffi

pytestmark = pytest.mark.gpu


def _kernels(fn):
    """names of the CUDA kernels that ran while fn() ran"""
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
    return [e["name"] for e in events if e.get("cat") == "kernel"]


def _counted(eng, fn, what):
    l0 = eng.total_launches()
    names = _kernels(fn)
    assert len(names) == eng.total_launches() - l0, (what, len(names), eng.total_launches() - l0, sorted(set(names)))
    return names


def _problem(N, D, P, seed):
    rng = np.random.default_rng(seed)
    X = rng.uniform(-3, 3, (N, D))
    Y = np.stack([np.sin(X).sum(1) / np.sqrt(D) + 0.1 * rng.standard_normal(N) for _ in range(P)], 1)
    return rng, X, Y


def test_profiler_sees_the_library_kernels():
    e = _ffi.Engine(0)
    try:
        _, X, _ = _problem(300, 3, 1, 1)
        _kernels(lambda: None)   # the first profiling session sets the tracer up
        names = _counted(e, lambda: e.kern_K_device_only("rbf", True, 1.0, [1.0, 1.5, 2.0], X), "kern_K")
        assert any("kbuild_kernel" in n for n in names), names
    finally:
        e.close()


def test_sparse_calls_count_every_launch():
    """M = 600: the child factorisations run the blocked sweep with its look-ahead stream (Mpad = 640, three blocks)."""
    rng, X, Y = _problem(1500, 3, 2, 2)
    Z = X[rng.permutation(1500)[:600]] + 0.01 * rng.standard_normal((600, 3))
    ls = [1.2, 1.6, 2.1]
    nv = rng.uniform(0.01, 0.3, 1500)
    e = _ffi.Engine(0)
    try:
        _counted(e, lambda: e.sparse_set_data(X, Y), "sparse_set_data")
        e.sparse_eval("rbf", True, 1.1, ls, Z, 0.05)   # warm-up: child contexts and their workspaces
        e.sparse_eval_het("rbf", True, 1.1, ls, Z, nv)
        _counted(e, lambda: e.sparse_eval("rbf", True, 1.1, ls, Z, 0.05), "sparse_eval")
        for what in e.SPARSE_GET:
            _counted(e, lambda: e.sparse_get(what), "sparse_get " + what)
        _counted(e, lambda: e.sparse_eval_het("matern52", False, 0.9, 1.7, Z, nv), "sparse_eval_het")
        for what in e.SPARSE_GET:
            _counted(e, lambda: e.sparse_get(what), "sparse_get %s after het" % what)
    finally:
        e.close()


def test_kernel_and_part_calls_pdinv_and_exact_evaluation_count_every_launch():
    """the part calls on the single kernel as one part (its columns in order) run the kernels of the single-kernel calls;
    on the same covariance with the columns in reverse order they keep the composite kernels"""
    rng, X, Y = _problem(1100, 3, 1, 3)
    X2 = rng.uniform(-3, 3, (260, 3))
    ls = np.array([1.2, 1.6, 2.1])
    single, part, keep = _ffi.GpxKernPart(), _ffi.GpxKernPart(), []
    _ffi._fill_part(single, ("matern52", True, 0, [0, 1, 2], 1.3, ls), keep)
    _ffi._fill_part(part, ("matern52", True, 0, [2, 1, 0], 1.3, ls[::-1].copy()), keep)
    e = _ffi.Engine(0)
    L, h, p = _ffi.lib(), e._h, _ffi._ptr
    try:
        for x2 in (None, X2):
            M = 1100 if x2 is None else 260
            dL = rng.standard_normal((1100, M))
            out, gx = np.empty((1100, M)), np.empty((1100, 3))
            dv, dl, g = np.zeros(1), np.zeros(3), np.zeros(4)
            calls = {
                "kern_K": lambda: L.gpx_kern_K(h, 3, 1, 1.3, p(ls), p(X), 1100, p(x2), M, 3, p(out)),
                "kern_grad_full": lambda: L.gpx_kern_grad_full(h, 3, 1, 1.3, p(ls), p(X), 1100, p(x2), M, 3, p(dL), p(dv),
                                                               p(dl)),
                "kern_grad_X": lambda: L.gpx_kern_grad_X(h, 3, 1, 1.3, p(ls), p(X), 1100, p(x2), M, 3, p(dL), p(gx)),
                "single_part_K": lambda: L.gpx_kern_part_K(h, ctypes.byref(single), p(X), 1100, p(x2), M, 3, p(out)),
                "single_part_grad_full": lambda: L.gpx_kern_part_grad_full(h, ctypes.byref(single), p(X), 1100, p(x2), M, 3,
                                                                           p(dL), p(g)),
                "kern_part_K": lambda: L.gpx_kern_part_K(h, ctypes.byref(part), p(X), 1100, p(x2), M, 3, p(out)),
                "kern_part_grad_full": lambda: L.gpx_kern_part_grad_full(h, ctypes.byref(part), p(X), 1100, p(x2), M, 3, p(dL),
                                                                         p(g)),
            }
            seen = {}
            for name, call in calls.items():
                assert call() == 0
                rc = []
                seen[name] = _counted(e, lambda: rc.append(call()), "%s X2=%s" % (name, x2 is not None))
                assert rc == [0]
            assert sorted(seen["single_part_K"]) == sorted(seen["kern_K"]), seen
            assert sorted(seen["single_part_grad_full"]) == sorted(seen["kern_grad_full"]), seen
            assert not any("multi" in k for k in seen["kern_K"] + seen["kern_grad_full"]), seen
            for name in ("kern_part_K", "kern_part_grad_full"):
                assert all("multi" in k for k in seen[name]), seen[name]
        e.set_data(X, Y)
        e.exact_eval("matern32", True, 1.3, ls, 0.05)
        _counted(e, lambda: e.exact_eval("rbf", True, 1.3, ls, 0.05), "exact_eval (5 blocks)")
        _counted(e, lambda: e.predict(X2[:20], full_cov=True), "predict full_cov")
        _counted(e, lambda: e.get("K"), "get K")
        A = e.get("K") + 0.1 * np.eye(1100)
        _counted(e, lambda: _ffi.pdinv(A, engine=e), "pdinv")
    finally:
        e.close()
