"""The reference's OWN SparseGP (GPy/core/sparse_gp.py, executed unmodified through oracle/ref_gpy.py) over a plugin sum
kernel, B.Add([B.RBF(ARD), Bias, White]) with B.VarDTC(), against the stock pair (the reference's VarDTC, Add, RBF, Bias,
White): one engine call per evaluation, and SparseGP._update_gradients (:108-119) lands on the device's numbers through
the handles. On the CPU the engine is a test double answering from tests/sparse_composite_oracle.py; on the GPU it is the
device. A RatQuad inside the sum keeps the stock VarDTC. Skipped where the reference tree does not exist."""
import os
import types

import numpy as np
import pytest

import sparse_composite_oracle as so

pytestmark = pytest.mark.skipif(not os.path.isdir(os.environ.get("GPX_REFERENCE", "/root/reference") + "/GPy"),
                                reason="reference tree not present")


class FakeSparseEngine(object):
    """the sparse entry points of _ffi.Engine a composite needs, answered by the NumPy restatement"""

    def __init__(self, device=0):
        self.calls, self.sparse_serial = [], 0

    def sparse_set_data(self, X, Y):
        self.X, self.Y = np.array(X), np.array(Y)
        self.calls.append("sparse_set_data")

    def sparse_eval_multi(self, parts, Z, noise):
        self.calls.append("sparse_eval_multi")
        self.sparse_serial += 1
        ps = []
        for d in parts:
            p = dict(kind=d[0], ARD=d[1], term=d[2], dims=list(d[3]), variance=d[4])
            if d[0] not in ("white", "bias"):
                p["lengthscale"] = d[5]
            ps.append(p)
        lml, g, Zg, self.res = so.sparse_composite_eval(self.X, self.Y, Z, ps, noise)
        return (lml, g, Zg, self.res["dL_dthetaL"]) if np.ndim(noise) > 0 else (lml, g, Zg)

    def sparse_get(self, what):
        return {"woodbury_vector": self.res["woodbury_vector"], "woodbury_inv": self.res["woodbury_inv"],
                "Kmm": self.res["Kmm"], "Lm": self.res["Lm"]}[what]


def _setup(fake):
    from oracle import ref_gpy
    from gpy_b200 import gpy_plugin
    S = ref_gpy.load_sparse_models()
    C = ref_gpy.load_combination()
    G = S.G
    kw = {}
    if fake:
        from test_periodic_ratquad_plugin_cpu import fake_ffi
        f = fake_ffi()
        kw["ffi"] = types.SimpleNamespace(kern_K=f.kern_K, kern_Kdiag=f.kern_Kdiag, kern_grad_full=f.kern_grad_full,
                                          kern_part_K=f.kern_part_K, kern_part_grad_full=f.kern_part_grad_full,
                                          Engine=FakeSparseEngine)
    B = gpy_plugin.make(G.RBF, G.Exponential, G.Matern32, G.Matern52, G.ExactGaussianInference, Add=C.Add, Prod=C.Prod,
                        VarDTC=G.VarDTC, RatQuad=G.stationary.RatQuad, **kw)
    return S, C, G, B


def _pair(fake, N, M):
    S, C, G, B = _setup(fake)
    X, Y, Z, _ = so.case_data(N, M, 3, 1, 91, False)
    ls = [0.9, 1.4, 2.1]
    stock = S.SparseGP(X, Y, Z.copy(), C.Add([G.RBF(3, variance=1.3, lengthscale=ls, ARD=True), C.Bias(3, variance=0.4),
                                              C.White(3, variance=0.07)]),
                       G.Gaussian(variance=0.08), inference_method=G.VarDTC(limit=3))
    plug = S.SparseGP(X, Y, Z.copy(), B.Add([B.RBF(3, variance=1.3, lengthscale=ls, ARD=True), C.Bias(3, variance=0.4),
                                             C.White(3, variance=0.07)]),
                      G.Gaussian(variance=0.08), inference_method=B.VarDTC())
    return S, C, G, B, X, Y, Z, stock, plug


def _compare(stock, plug):
    l_s, l_p = float(np.squeeze(stock.log_likelihood())), float(np.squeeze(plug.log_likelihood()))
    assert abs(l_p - l_s) <= 1e-9 * max(1.0, abs(l_s))
    gs, gp = np.asarray(stock.gradient), np.asarray(plug.gradient)
    np.testing.assert_allclose(gp, gs, rtol=1e-8, atol=1e-8 * np.abs(gs).max())


def test_stock_sparse_gp_over_a_plugin_sum_kernel_cpu():
    S, C, G, B, X, Y, Z, stock, plug = _pair(True, 120, 14)
    _compare(stock, plug)
    eng = plug.inference_method.engine
    n0 = eng.calls.count("sparse_eval_multi")
    for m in (stock, plug):
        m.kern.parts[0].variance[:] = 0.9
        m.parameters_changed()                                # sparse_gp.py:76-81: one evaluation
    assert eng.calls.count("sparse_eval_multi") == n0 + 1 and eng.calls.count("sparse_set_data") == 1
    _compare(stock, plug)


def test_a_ratquad_inside_the_sum_keeps_the_stock_vardtc_cpu():
    S, C, G, B = _setup(True)
    X, Y, Z, _ = so.case_data(60, 8, 2, 1, 92, False)
    k = B.Add([B.RBF(2, variance=1.1, lengthscale=1.3), B.RatQuad(2, variance=0.5, lengthscale=1.2, power=0.8)])
    inf = B.VarDTC()
    post, lml, gd = inf.inference(k, X, Z, G.Gaussian(variance=0.1), Y)
    assert isinstance(gd["dL_dKnm"], np.ndarray) and inf._engine is None
    k0 = C.Add([G.RBF(2, variance=1.1, lengthscale=1.3), G.stationary.RatQuad(2, variance=0.5, lengthscale=1.2, power=0.8)])
    post0, lml0, gd0 = G.VarDTC().inference(k0, X, Z, G.Gaussian(variance=0.1), Y)
    assert abs(float(np.squeeze(lml)) - float(np.squeeze(lml0))) <= 1e-9 * max(1.0, abs(float(np.squeeze(lml0))))


def test_a_stale_handle_is_refused_cpu():
    S, C, G, B, X, Y, Z, stock, plug = _pair(True, 60, 8)
    post, lml, gd = plug.inference_method.inference(plug.kern, X, np.asarray(plug.Z), plug.likelihood, Y)
    plug.kern.parts[0].variance[:] = 2.0
    with pytest.raises(ValueError, match="stale"):
        plug.kern.update_gradients_full(gd["dL_dKnm"], X, np.asarray(plug.Z))
    with pytest.raises(TypeError):
        np.asarray(gd["dL_dKnm"])


@pytest.mark.gpu
def test_stock_sparse_gp_over_a_plugin_sum_kernel_gpu():
    S, C, G, B, X, Y, Z, stock, plug = _pair(False, 900, 60)
    _compare(stock, plug)
    for m in (stock, plug):
        m.kern.parts[0].lengthscale[:] = [1.2, 0.8, 1.7]
        m.parameters_changed()
    _compare(stock, plug)
