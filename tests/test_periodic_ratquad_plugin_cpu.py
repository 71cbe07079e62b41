"""The GPy plugin with RatQuad and StdPeriodic leaves, driven by the reference's OWN GPRegression / Add / Prod / White
(GPy/core/gp.py, models/gp_regression.py, kern/src/add.py, prod.py, static.py, executed through oracle/ref_gpy.py) on a
test double of the C ABI that answers from the oracle of tests/periodic_oracle.py. Skipped where the reference tree does
not exist."""
import importlib
import os
import types

import numpy as np
import pytest

import periodic_oracle as po
from test_periodic_ratquad_cpu import FakeEngine

pytestmark = pytest.mark.skipif(not os.path.isdir(os.environ.get("GPX_REFERENCE", "/root/reference") + "/GPy"),
                                reason="reference tree not present")


def _desc_dict(d):
    q = dict(kind=d[0], ARD=d[1], term=d[2], dims=list(range(len(d[3]))), variance=d[4], lengthscale=d[5])
    q.update(d[6])
    return q


def fake_ffi():
    from test_gpy_plugin_cpu import fake_ffi as base
    ffi = base()

    def kern_part_K(desc, X, X2=None):
        return po.make_part(_desc_dict(desc))[0].K(X, X2)

    def kern_part_grad_full(desc, X, dL_dK, X2=None):
        return po.make_part(_desc_dict(desc))[0].update_gradients_full(dL_dK, X, X2)

    return types.SimpleNamespace(kern_K=ffi.kern_K, kern_Kdiag=ffi.kern_Kdiag, kern_grad_full=ffi.kern_grad_full,
                                 kern_part_K=kern_part_K, kern_part_grad_full=kern_part_grad_full, Engine=FakeEngine)


def _setup():
    from oracle import ref_gpy
    from gpy_b200 import gpy_plugin
    M = ref_gpy.load_models()
    C = ref_gpy.load_combination()
    G = M.G
    sp = importlib.import_module("GPy.kern.src.standard_periodic")
    B = gpy_plugin.make(G.RBF, G.Exponential, G.Matern32, G.Matern52, G.ExactGaussianInference, ffi=fake_ffi(),
                        Add=C.Add, Prod=C.Prod, RatQuad=G.stationary.RatQuad, StdPeriodic=sp.StdPeriodic)
    K = types.SimpleNamespace(RBF=G.RBF, RatQuad=G.stationary.RatQuad, StdPeriodic=sp.StdPeriodic, Add=C.Add, Prod=C.Prod)
    return M, C, K, B


def _mauna_loa(K, White):
    return K.Add([K.RBF(1, variance=4.0, lengthscale=50.0),
                  K.Prod([K.RBF(1, variance=2.0, lengthscale=90.0),
                          K.StdPeriodic(1, variance=1.0, period=1.0, lengthscale=1.3)]),
                  K.RatQuad(1, variance=0.5, lengthscale=1.2, power=0.8),
                  K.RBF(1, variance=0.1, lengthscale=0.15),
                  White(1, variance=0.05)])


def test_stock_gpregression_with_the_mauna_loa_kernel_through_the_plugin():
    M, C, K, B = _setup()
    X, Y = po.mauna_loa_data(120, seed=5)
    stock = M.GPRegression(X, Y, _mauna_loa(K, C.White), noise_var=0.01)
    plug = M.GPRegression(X, Y, _mauna_loa(B, C.White), noise_var=0.01)
    assert type(plug) is type(stock)
    assert isinstance(plug.kern.parts[1].parts[1], K.StdPeriodic) and isinstance(plug.kern.parts[2], K.RatQuad)
    plug.inference_method = B.ExactGaussianInference()
    plug.parameters_changed()
    eng = plug.inference_method.engine
    assert eng.calls == ["set_data", "exact_eval_multi"]                  # one engine call per evaluation
    assert [d[0] for d in eng.descs[-1]] == ["rbf", "rbf", "stdperiodic", "ratquad", "rbf", "white"]
    assert abs(plug.log_likelihood() - stock.log_likelihood()) <= 1e-9
    np.testing.assert_allclose(plug.gradient, stock.gradient, rtol=1e-8, atol=1e-10)
    n0 = eng.calls.count("exact_eval_multi")
    for m in (plug, stock):
        m.kern.parts[2].power[:] = 1.1
        m.kern.parts[1].parts[1].period[:] = 1.05
        m.parameters_changed()
    assert eng.calls.count("exact_eval_multi") == n0 + 1                 # one evaluation -> one engine call
    assert abs(plug.log_likelihood() - stock.log_likelihood()) <= 1e-9
    np.testing.assert_allclose(plug.gradient, stock.gradient, rtol=1e-8, atol=1e-10)
    plug.optimize(max_iters=15)
    stock.optimize(max_iters=15)
    assert abs(plug.log_likelihood() - stock.log_likelihood()) <= 1e-5 * max(1.0, abs(stock.log_likelihood()))
    np.testing.assert_allclose(plug.param_array, stock.param_array, rtol=1e-3)
    assert eng.calls.count("set_data") == 1 and "exact_eval" not in eng.calls


@pytest.mark.parametrize("which", ["RatQuad", "StdPeriodic"])
def test_a_lone_plugin_leaf_is_one_composite_call(which):
    M, C, K, B = _setup()
    X, Y = po.mauna_loa_data(80, seed=6)
    X = np.hstack([X - 1990.0, np.sin(X)])
    if which == "RatQuad":
        mk = lambda K: K.RatQuad(2, variance=1.3, lengthscale=[3.0, 1.5], power=0.9, ARD=True)   # noqa: E731
    else:
        mk = lambda K: K.StdPeriodic(2, variance=1.3, period=[1.0, 2.5], lengthscale=0.9, ARD1=True)   # noqa: E731
    stock = M.GPRegression(X, Y, mk(K), noise_var=0.05)
    plug = M.GPRegression(X, Y, mk(B), noise_var=0.05)
    plug.inference_method = B.ExactGaussianInference()
    plug.parameters_changed()
    eng = plug.inference_method.engine
    assert eng.calls == ["set_data", "exact_eval_multi"] and len(eng.descs[-1]) == 1
    assert abs(plug.log_likelihood() - stock.log_likelihood()) <= 1e-9
    np.testing.assert_allclose(plug.gradient, stock.gradient, rtol=1e-8, atol=1e-10)
    # the stand-alone entries (a dense dL_dK, as GPy's generic code hands it over) give the stock kernel's numbers
    kp, ks = plug.kern, stock.kern
    np.testing.assert_allclose(kp.K(X, X[:9]), ks.K(X, X[:9]), rtol=1e-13, atol=1e-15)
    dL = np.random.default_rng(1).standard_normal((80, 9))
    kp.update_gradients_full(dL, X, X[:9])
    ks.update_gradients_full(dL, X, X[:9])
    np.testing.assert_allclose(kp.gradient, ks.gradient, rtol=1e-12, atol=1e-12)


def test_sparse_plugin_keeps_the_stock_vardtc_for_the_new_leaves():
    """kernel_types (single-kernel and VarDTC routing) does not include RatQuad / StdPeriodic"""
    M, C, K, B = _setup()
    from gpy_b200 import gpy_plugin
    from oracle import ref_gpy
    G = M.G
    B2 = gpy_plugin.make(G.RBF, G.Exponential, G.Matern32, G.Matern52, G.ExactGaussianInference, ffi=fake_ffi(),
                         VarDTC=G.VarDTC, RatQuad=K.RatQuad, StdPeriodic=K.StdPeriodic)
    ref_gpy.load_sparse_models()
    X, Y = po.mauna_loa_data(60, seed=7)
    X = X - 1990.0
    Z = X[::6].copy()
    lik = G.Gaussian(variance=0.1)
    k = B2.RatQuad(1, variance=1.0, lengthscale=2.0)
    post, lml, gd = B2.VarDTC().inference(k, X, Z, lik, Y)
    post0, lml0, gd0 = G.VarDTC().inference(K.RatQuad(1, variance=1.0, lengthscale=2.0), X, Z, lik, Y)
    assert abs(float(np.squeeze(lml)) - float(np.squeeze(lml0))) <= 1e-9 * max(1.0, abs(float(np.squeeze(lml0))))
