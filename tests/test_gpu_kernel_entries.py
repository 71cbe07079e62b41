"""The stand-alone kernel entries (gpx_kern_K, gpx_kern_grad_full, gpx_kern_grad_X and the one-part gpx_kern_part_K,
gpx_kern_part_grad_full) on an engine's own context work with the kernel they are given and leave the context's last
evaluation alone. (Their launch accounting is in test_gpu_launch_accounting.py.)"""
import ctypes

import numpy as np
import pytest

from gpy_b200 import _ffi
from oracle import gpy_oracle as o

pytestmark = pytest.mark.gpu

# RatQuad + StdPeriodic x RBF + White on D = 3
COMPOSITE = [("ratquad", True, 0, [0, 1, 2], 0.8, np.array([1.0, 1.4, 1.9]), {"power": 1.3}),
             ("stdperiodic", False, 1, [0], 1.1, 1.2, {"period": 2.0}),
             ("rbf", True, 1, [1, 2], 1.0, np.array([1.0, 1.5])),
             ("white", False, 2, [], 0.1, None)]
PERIODIC = ("stdperiodic", True, 0, [0, 1], 0.9, np.array([0.8, 1.3]), {"period": np.array([1.5, 2.5]), "ARD_period": True})


def _results(e, Xs):
    """everything an engine hands out about its last evaluation"""
    out = {w: e.get(w) for w in _ffi.GET}
    out["mu"], out["var"] = e.predict(Xs)
    out["mu_full"], out["cov"] = e.predict(Xs, full_cov=True)
    return out


def _stand_alone_calls(e, rng):
    """every stand-alone entry on e's own context, on inputs of another size and another D than e's data"""
    L, h, p = _ffi.lib(), e._h, _ffi._ptr
    part, keep = _ffi.GpxKernPart(), []
    n = _ffi._fill_part(part, PERIODIC, keep)
    X, X2 = rng.uniform(-2, 2, (250, 2)), rng.uniform(-2, 2, (180, 2))
    ls = np.array([0.7, 1.6])
    for x2 in (None, X2):
        M = 250 if x2 is None else 180
        out, dL, gx = np.empty((250, M)), rng.standard_normal((250, M)), np.empty((250, 2))
        grad, dv, dl = np.zeros(n), np.zeros(1), np.zeros(2)
        assert L.gpx_kern_part_K(h, ctypes.byref(part), p(X), 250, p(x2), M, 2, p(out)) == 0
        assert L.gpx_kern_part_grad_full(h, ctypes.byref(part), p(X), 250, p(x2), M, 2, p(dL), p(grad)) == 0
        assert L.gpx_kern_K(h, 3, 1, 1.3, p(ls), p(X), 250, p(x2), M, 2, p(out)) == 0
        assert L.gpx_kern_grad_full(h, 2, 1, 1.3, p(ls), p(X), 250, p(x2), M, 2, p(dL), p(dv), p(dl)) == 0
        assert L.gpx_kern_grad_X(h, 0, 1, 1.3, p(ls), p(X), 250, p(x2), M, 2, p(dL), p(gx)) == 0


def test_stand_alone_calls_leave_the_last_evaluation_alone():
    rng = np.random.default_rng(3)
    X, Y = o.synthetic(700, 3, seed=4)
    Xs = rng.uniform(-2, 2, (40, 3))
    e = _ffi.Engine(0)
    try:
        e.set_data(X, Y)
        for evaluate in (lambda: e.exact_eval_multi(COMPOSITE, 0.05),
                         lambda: e.exact_eval("rbf", True, 1.3, np.array([1.1, 1.6, 2.2]), 0.05)):
            evaluate()
            before = _results(e, Xs)
            _stand_alone_calls(e, rng)
            after = _results(e, Xs)
            for w in before:
                assert np.array_equal(after[w], before[w]), w
    finally:
        e.close()

