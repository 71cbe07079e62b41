"""The plugin's B.SVGP without a GPU: GPy's own core SVGP over B.SVGP (plugin kernels through a host kernel stand-in, the
two gpx_svgp_* entries through a host engine that restates them with tests/svgp_oracle.py) against GPy's own SVGP with
the stock inference and kernels, and every route to the stock method."""
import importlib
import os
import sys
import types

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), HERE, os.path.join(HERE, "golden")]

import svgp_oracle as so  # noqa: E402
from gpy_b200.svgp import triang_to_flat  # noqa: E402

BAR = 1e-10


class _GivenDF(object):
    """a likelihood that hands the engine's restatement the dF_dmu / dF_dv it was given"""

    def __init__(self, dmu, dv):
        self.dmu, self.dv = np.asarray(dmu).reshape(-1, 1), np.asarray(dv).reshape(-1, 1)

    def variational_expectations(self, Y, m, v, Y_metadata=None):
        return np.zeros_like(m), self.dmu, self.dv, None


class HostSVGPEngine(object):
    """gpx_svgp_begin / gpx_svgp_finish on the host"""

    def __init__(self, device=0):
        self.calls, self.sparse_serial = [], 0

    def sparse_set_data(self, X, Y):
        self.calls.append(("set_data",))
        self.X, self.Y = np.array(X, dtype=np.float64), np.array(Y, dtype=np.float64)
        self.sN, self.sD, self.sP = X.shape[0], X.shape[1], 1

    def svgp_begin(self, parts, Z, q_m, q_L, row0, nb, max_tries=5):
        from test_laplace_cpu import _parts_of
        self.calls.append(("begin", row0, nb))
        self.args = (_parts_of(parts), self.X[row0:row0 + nb], self.Y[row0:row0 + nb], np.array(Z), np.array(q_m),
                     np.array(q_L))
        o = so.svgp_eval(*self.args, _GivenDF(np.zeros(nb), np.zeros(nb)))
        self.sM = Z.shape[0]
        return o["mu"], o["v"], o["KL"], 0.0

    def svgp_finish(self, dF_dmu, dF_dv):
        self.calls.append(("finish",))
        o = so.svgp_eval(*self.args, _GivenDF(dF_dmu, dF_dv))
        return o["grad"], o["dZ"], o["dL_dm"], o["dL_dchol"]


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
    core = importlib.import_module("GPy.core.svgp")
    inf = importlib.import_module("GPy.inference.latent_function_inference.svgp")
    lik = types.SimpleNamespace(Bernoulli=importlib.import_module("GPy.likelihoods.bernoulli").Bernoulli,
                                StudentT=importlib.import_module("GPy.likelihoods.student_t").StudentT,
                                Gaussian=importlib.import_module("GPy.likelihoods.gaussian").Gaussian)
    return S, C, core, inf, lik


def _plugin():
    S, C, core, inf, lik = _reference()
    from gpy_b200 import gpy_plugin
    from test_periodic_ratquad_plugin_cpu import fake_ffi
    f = fake_ffi()

    def kern_grad_X(kind, ARD, variance, lengthscale, X, dL_dK, X2=None):
        part = dict(kind=kind, ARD=ARD, term=0, dims=list(range(X.shape[1])), variance=variance, lengthscale=lengthscale)
        return so.CompositeOracle([part]).gradients_X(dL_dK, X, X2)

    ffi = types.SimpleNamespace(kern_K=f.kern_K, kern_Kdiag=f.kern_Kdiag, kern_grad_full=f.kern_grad_full,
                                kern_grad_X=kern_grad_X, kern_part_K=f.kern_part_K,
                                kern_part_grad_full=f.kern_part_grad_full, Engine=HostSVGPEngine)
    G = S.G
    B = gpy_plugin.make(G.RBF, G.Exponential, G.Matern32, G.Matern52, G.ExactGaussianInference, Add=C.Add, Prod=C.Prod,
                        SVGP=inf.SVGP, ffi=ffi)
    return S, C, G, B, core, inf, lik


def _kern(ns, B, C, composite):
    if not composite:
        return ns.RBF(3, variance=1.4, lengthscale=[0.8, 1.3, 1.9], ARD=True)
    k = ns.RBF(3, variance=1.3, lengthscale=[0.9, 1.4, 2.1], ARD=True)
    m = ns.Matern52(2, variance=1.1, lengthscale=1.2, active_dims=[0, 1])
    prod, add = (B.Prod, B.Add) if ns is B else (C.Prod, C.Add)
    return add([prod([k, m]), C.Bias(3, variance=0.4)])


@pytest.mark.parametrize("case,composite", [("bernoulli_rbf_ard", False), ("studentt_matern52_ard", False),
                                            ("bernoulli_composite", True)])
def test_reference_svgp_over_plugin_matches_the_stock_pair(case, composite):
    S, C, G, B, core, inf, lik = _plugin()
    parts, lik_spec, N, M, seed, opts = so.CASES[case]
    X, Y, Z, q_m, q_L, Xnew, bs = so.case_data(case)
    if lik_spec != "bernoulli":
        composite = False

    class RefSVGP(core.SVGP):
        # paramz exposes a linked parameter under its name; the test-only paramz stand-in does not, so the two names
        # core/svgp.py:55 reads are given here
        q_u_mean = property(lambda self: self.m)
        q_u_chol = property(lambda self: self.chol)

    def model(ns, method):
        m = RefSVGP(X, Y, Z.copy(), _kern(ns, B, C, composite), so.make_likelihood(lik_spec, lik))
        m.inference_method = method
        m.q_u_mean[:] = q_m[:, None]
        m.q_u_chol[:] = triang_to_flat(q_L)[:, None]
        m.parameters_changed()
        return m

    stock = model(G, inf.SVGP())
    plug = model(B, B.SVGP())
    assert [c[0] for c in plug.inference_method.engine.calls][-2:] == ["begin", "finish"]
    l_s, l_p = float(np.squeeze(stock.log_likelihood())), float(np.squeeze(plug.log_likelihood()))
    assert abs(l_p - l_s) <= BAR * abs(l_s)
    gs, gp = np.asarray(stock.gradient), np.asarray(plug.gradient)
    # dL_dchol differs by the reference's S^-1 rounding (tests/svgp_oracle.py), hence the bar on the largest entry
    np.testing.assert_allclose(gp, gs, rtol=0, atol=1e-9 * np.abs(gs).max())


def test_plugin_svgp_sends_anything_else_to_the_stock_method():
    S, C, G, B, core, inf, lik = _plugin()
    X, Y, Z, q_m, q_L, Xnew, bs = so.case_data("bernoulli_rbf_iso")
    m0, ch = q_m[:, None], triang_to_flat(q_L)[:, None]
    method = B.SVGP()

    def quiet():
        return method._engine is None or not method.engine.calls

    method.inference(m0, ch, G.RBF(3), X, Z, lik.Bernoulli(), Y)                       # the reference's own kernel
    assert quiet()
    method.inference(np.hstack([m0, m0]), np.hstack([ch, ch]), B.RBF(3), X, Z, lik.Bernoulli(), np.hstack([Y, Y]))
    assert quiet()                                                                      # two latent functions
    method.inference(m0, ch, C.Add([B.RBF(3), G.Matern32(3)]), X, Z, lik.Bernoulli(), Y)   # a foreign leaf
    assert quiet()
    with pytest.raises(Exception):                                                      # a mean function
        method.inference(m0, ch, B.RBF(3), X, Z, lik.Bernoulli(), Y, mean_function=object())
    assert quiet()
    _, l_dev, gd = method.inference(m0, ch, B.RBF(3), X, Z, lik.Bernoulli(), Y)
    assert not quiet()
    _, l_ref, _ = inf.SVGP().inference(m0, ch, G.RBF(3), X, Z, lik.Bernoulli(), Y)
    assert abs(l_dev - l_ref) <= BAR * abs(l_ref)
    assert set(gd) == {"dL_dKmm", "dL_dKmn", "dL_dKdiag", "dL_dm", "dL_dchol", "dL_dthetaL"}
