"""Build-container-only: the reference's own GPLVM (GPy/models/gplvm.py, via oracle/ref_gpy.py) over the plugin pair, with the
C ABI replaced by a test double that answers from the oracle. GPLVM.parameters_changed runs unchanged: its
kern.gradients_X(dL_dK, X, None) receives the plugin's DeviceGradient and takes the device input gradient, once per
evaluation, and the model equals the stock one."""
import os
import types

import numpy as np
import pytest

import gplvm_oracle as go
from oracle import gpy_oracle as o

pytestmark = pytest.mark.skipif(not os.path.isdir(os.environ.get("GPX_REFERENCE", "/root/reference") + "/GPy"),
                                reason="reference tree not present")


class FakeEngine(object):
    """test double of _ffi.Engine for one stationary kernel: the exact evaluation and gpx_exact_grad_X from the oracle"""

    def __init__(self, device=0):
        self.calls = []
        self.eval_serial = 0

    def set_data(self, X, Y):
        self.X, self.Y = np.array(X), np.array(Y)
        self.eval_serial += 1
        self.calls.append("set_data")

    def exact_eval(self, kind, ARD, variance, lengthscale, noise, jitter=1e-8, max_tries=5):
        self.calls.append("exact_eval")
        self.eval_serial += 1
        self.kern = o.StationaryOracle(kind, self.X.shape[1], variance, lengthscale, ARD)
        lml, g, self.res = o.eval_lml_grad(self.X, self.Y, kind, ARD, variance, lengthscale, noise)
        return lml, g, 0.0

    def exact_grad_X(self):
        self.calls.append("exact_grad_X")
        return self.kern.gradients_X(self.res["dL_dK"], self.X)

    def get(self, which):
        self.calls.append(which)
        return {"dL_dK": self.res["dL_dK"], "alpha": self.res["alpha"], "L": self.res["L"]}[which]


def fake_ffi(host_calls):
    def kern_grad_X(kind, ARD, var, ls, X, dL_dK, X2=None):
        host_calls.append("kern_grad_X")
        return o.StationaryOracle(kind, X.shape[1], var, ls, ARD).gradients_X(dL_dK, X, X2)

    def kern_K(kind, ARD, var, ls, X, X2=None):
        return o.StationaryOracle(kind, X.shape[1], var, ls, ARD).K(X, X2)

    def kern_grad_full(kind, ARD, var, ls, X, dL_dK, X2=None):
        dv, dl = o.StationaryOracle(kind, X.shape[1], var, ls, ARD).update_gradients_full(dL_dK, X, X2)
        return dv, np.atleast_1d(dl)
    return types.SimpleNamespace(kern_K=kern_K, kern_Kdiag=lambda kind, var, N: np.full(N, var), kern_grad_X=kern_grad_X,
                                 kern_grad_full=kern_grad_full, Engine=FakeEngine)


def test_reference_gplvm_runs_on_the_plugin_pair():
    from oracle import ref_gpy
    from gpy_b200 import gpy_plugin
    GPLVM, ns = go.reference_gplvm()
    G = ref_gpy.load()
    host_calls = []
    B = gpy_plugin.make(G.RBF, G.Exponential, G.Matern32, G.Matern52, G.ExactGaussianInference, ffi=fake_ffi(host_calls))
    _, Y = go.latent_data(40, 3, 4, seed=3)
    np.random.seed(7)
    stock = GPLVM(Y, 2, kernel=G.Matern52(2, variance=1.2, lengthscale=[0.9, 1.3], ARD=True))
    np.random.seed(7)
    plug = GPLVM(Y, 2, kernel=B.Matern52(2, variance=1.2, lengthscale=[0.9, 1.3], ARD=True))
    host_calls.clear()                        # the constructor evaluated with the stock inference
    plug.inference_method = B.ExactGaussianInference()
    plug.parameters_changed()
    eng = plug.inference_method.engine
    assert eng.calls == ["set_data", "exact_eval", "exact_grad_X"] and host_calls == []
    assert abs(plug.log_likelihood() - stock.log_likelihood()) < 1e-10
    np.testing.assert_allclose(plug.gradient, stock.gradient, rtol=1e-9, atol=1e-12)
    # a new iterate of the latent points: one upload, one evaluation, one input gradient
    plug.X[0, 0] = plug.X[0, 0] + 0.1
    stock.X[0, 0] = stock.X[0, 0] + 0.1
    assert eng.calls[3:] == ["set_data", "exact_eval", "exact_grad_X"]
    np.testing.assert_allclose(plug.gradient, stock.gradient, rtol=1e-9, atol=1e-12)
    # the handle of an earlier evaluation takes the stand-alone route with the matrix it materialises
    old = plug.grad_dict["dL_dK"]
    plug.kern.variance[:] = 1.5
    n = len(eng.calls)
    plug.kern.gradients_X(old, plug.X, None)
    assert "exact_grad_X" not in eng.calls[n:] and host_calls == ["kern_grad_X"]
