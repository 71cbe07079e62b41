"""The plugin's B.VarGauss without a GPU: GPy's own GPVariationalGaussianApproximation over B.VarGauss (plugin kernels
through a host kernel stand-in, the two gpx_vargauss_* entries through the host engine of tests/test_vargauss_cpu.py)
against the same model with the stock inference and kernels, and every route to the stock method."""
import importlib
import os
import sys
import types

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), HERE, os.path.join(HERE, "golden")]

import vargauss_oracle as vo  # noqa: E402
from test_vargauss_cpu import HostVarGaussEngine  # noqa: E402

BAR = 1e-10


def _reference():
    try:
        from oracle import ref_gpy
        S = ref_gpy.load_sparse_models()
    except ImportError:
        pytest.skip("reference tree not present")
    if not os.path.isdir(os.environ.get("GPX_REFERENCE", "/root/reference")):
        pytest.skip("reference tree not present")
    from ep_reference import load_reference_ep
    load_reference_ep()
    C = ref_gpy.load_combination()
    vg = importlib.import_module("GPy.inference.latent_function_inference.var_gauss")
    sys.modules["GPy.inference.latent_function_inference"].VarGauss = vg.VarGauss
    model = importlib.import_module("GPy.models.gp_var_gauss").GPVariationalGaussianApproximation
    lik = types.SimpleNamespace(Bernoulli=importlib.import_module("GPy.likelihoods.bernoulli").Bernoulli,
                                StudentT=importlib.import_module("GPy.likelihoods.student_t").StudentT,
                                Gaussian=importlib.import_module("GPy.likelihoods.gaussian").Gaussian)
    return S, C, vg, model, lik


def _plugin():
    S, C, vg, model, lik = _reference()
    from gpy_b200 import gpy_plugin
    from test_periodic_ratquad_plugin_cpu import fake_ffi
    f = fake_ffi()
    ffi = types.SimpleNamespace(kern_K=f.kern_K, kern_Kdiag=f.kern_Kdiag, kern_grad_full=f.kern_grad_full,
                                kern_part_K=f.kern_part_K, kern_part_grad_full=f.kern_part_grad_full,
                                Engine=HostVarGaussEngine)
    G = S.G
    B = gpy_plugin.make(G.RBF, G.Exponential, G.Matern32, G.Matern52, G.ExactGaussianInference, Add=C.Add, Prod=C.Prod,
                        VarGauss=vg.VarGauss, ffi=ffi)
    return S, C, G, B, vg, model, lik


def _kern(ns, B, C, composite):
    if not composite:
        return ns.RBF(3, variance=1.4, lengthscale=[0.8, 1.3, 1.9], ARD=True)
    k = ns.RBF(3, variance=1.3, lengthscale=[0.9, 1.4, 2.1], ARD=True)
    m = ns.Matern52(2, variance=1.1, lengthscale=1.2, active_dims=[0, 1])
    prod, add = (B.Prod, B.Add) if ns is B else (C.Prod, C.Add)
    return add([prod([k, m]), C.Bias(3, variance=0.4)])


@pytest.mark.parametrize("case,composite", [("bernoulli_rbf_ard_n127", False), ("gaussian_rbf_ard_n129", False),
                                            ("bernoulli_m52_x_rbf_bias_n128", True)])
def test_reference_model_over_plugin_matches_the_stock_pair(case, composite):
    S, C, G, B, vg, model, lik = _plugin()
    parts, lik_spec = vo.CASES[case][:2]
    X, Y, alpha, beta, _ = vo.case_data(case)

    def make(ns, plugin):
        m = model(X, Y, _kern(ns, B, C, composite), vo.make_likelihood(lik_spec, lik))
        if plugin:
            m.inference_method = B.VarGauss(m.alpha, m.beta)
        m.alpha[:] = alpha[:, None]
        m.beta[:] = beta
        m.parameters_changed()
        return m

    stock, plug = make(G, False), make(B, True)
    assert [c[0] for c in plug.inference_method.engine.calls][-2:] == ["begin", "finish"]
    l_s, l_p = float(np.squeeze(stock.log_likelihood())), float(np.squeeze(plug.log_likelihood()))
    assert abs(l_p - l_s) <= BAR * abs(l_s)
    np.testing.assert_allclose(np.asarray(plug.alpha.gradient), np.asarray(stock.alpha.gradient), rtol=0,
                               atol=BAR * np.abs(stock.alpha.gradient).max())
    np.testing.assert_allclose(np.asarray(plug.beta.gradient), np.asarray(stock.beta.gradient), rtol=0,
                               atol=BAR * np.abs(stock.beta.gradient).max())
    gk_s, gk_p = np.asarray(stock.kern.gradient), np.asarray(plug.kern.gradient)
    o = vo.vargauss_eval(parts, X, Y, alpha, beta, vo.make_likelihood(lik_spec, lik))
    np.testing.assert_allclose(gk_p, o["grad"], rtol=1e-9, atol=0)
    if lik_spec == "gaussian":                      # dF_dv constant: the stock kernel gradient is the derivative too
        np.testing.assert_allclose(gk_p, gk_s, rtol=1e-9, atol=0)
    else:                                           # the stock one scales the rows (var_gauss.py:66)
        assert np.abs(gk_p - gk_s).max() > 1e-6 * np.abs(gk_s).max()


def test_plugin_vargauss_sends_anything_else_to_the_stock_method():
    S, C, G, B, vg, model, lik = _plugin()
    X, Y, alpha, beta, _ = vo.case_data("bernoulli_rbf_iso_n60")
    from paramz import Param
    a, b = Param("alpha", alpha[:, None]), Param("beta", beta.copy())
    method = B.VarGauss(a, b)

    def quiet():
        return method._engine is None or not method.engine.calls

    method.inference(G.RBF(3), X, lik.Bernoulli(), Y)                                     # the reference's own kernel
    assert quiet()
    method.inference(C.Add([B.RBF(3), G.Matern32(3)]), X, lik.Bernoulli(), Y)             # a foreign leaf
    assert quiet()
    with pytest.raises(AssertionError):                                                   # two output columns
        method.inference(B.RBF(3), X, lik.Bernoulli(), np.hstack([Y, Y]))
    assert quiet()
    with pytest.raises(NotImplementedError):                                              # a mean function
        method.inference(B.RBF(3), X, lik.Bernoulli(), Y, mean_function=object())
    assert quiet()
    try:
        method.inference(B.RBF(3), X.tolist(), lik.Bernoulli(), Y)                        # X not an ndarray
    except Exception:   # the stock method raises where it raises
        pass
    assert quiet()
    for bad in (0.0, np.inf):
        b2 = beta.copy()
        b2[4] = bad
        method.beta = Param("beta", b2)
        with np.errstate(all="ignore"):
            try:
                method.inference(B.RBF(3), X, lik.Bernoulli(), Y)
            except Exception:   # the stock method raises where it raises
                pass
        assert quiet()
    method.beta = b
    _, l_dev, gd = method.inference(B.RBF(3), X, lik.Bernoulli(), Y)
    assert not quiet()
    _, l_ref, _ = vg.VarGauss(Param("alpha", alpha[:, None]), Param("beta", beta.copy())).inference(
        G.RBF(3), X, lik.Bernoulli(), Y)
    assert abs(l_dev - l_ref) <= BAR * abs(l_ref)
    assert set(gd) == {"dL_dK", "dL_dthetaL"}
