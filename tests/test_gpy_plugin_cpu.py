"""Build-container-only: the reference-side binding (gpy_b200/gpy_plugin.py) wired onto the UNMODIFIED reference classes
(GPy 1.14.2 via oracle/ref_gpy.py). No GPU here, so the C ABI is replaced by a test double that answers from the oracle;
what is tested is the WIRING: GPy's slicing metaclass wraps the plugin methods, the two-call contract of
GP.parameters_changed (GPy/core/gp.py:278-280) works through the DeviceGradient handle, foreign dL_dK / foreign kernels
take the generic / stock paths, and the result equals the stock reference classes."""
import os
import types

import numpy as np
import pytest

from oracle import gpy_oracle as o

pytestmark = pytest.mark.skipif(not os.path.isdir(os.environ.get("GPX_REFERENCE", "/root/reference") + "/GPy"),
                                reason="reference tree not present")


class FakeEngine(object):
    """test double of _ffi.Engine: same methods, numbers from the oracle."""

    def __init__(self, device=0):
        self.calls = []

    def set_data(self, X, Y):
        self.X, self.Y = np.array(X), np.array(Y)
        self.calls.append("set_data")

    def exact_eval(self, kind, ARD, variance, lengthscale, noise, jitter=1e-8, max_tries=5):
        self.calls.append("exact_eval")
        self.eval_serial = getattr(self, "eval_serial", 0) + 1
        self.theta = (kind, ARD, variance, np.array(lengthscale, copy=True))
        lml, g, self.res = o.eval_lml_grad(self.X, self.Y, kind, ARD, variance, lengthscale, noise)
        return lml, g, 0.0

    def predict(self, Xnew, full_cov=False):
        kind, ARD, var, ls = self.theta
        k = o.StationaryOracle(kind, self.X.shape[1], var, ls if ARD else float(np.atleast_1d(ls)[0]), ARD)
        return o.raw_predict(k, self.X, self.res["L"], self.res["alpha"], Xnew, full_cov)

    def exact_eval_het(self, kind, ARD, variance, lengthscale, noise_variances, jitter=1e-8, max_tries=5):
        self.calls.append("exact_eval_het")
        lml, g, self.res = o.eval_lml_grad(self.X, self.Y, kind, ARD, variance, lengthscale, np.asarray(noise_variances))
        nk = g.size - self.X.shape[0]
        dn = g[nk:]
        return lml, np.concatenate([g[:nk], [dn.sum()]]), dn, 0.0

    def get(self, which):
        return {"L": self.res["L"], "alpha": self.res["alpha"], "Kinv": self.res["Wi"], "dL_dK": self.res["dL_dK"],
                "K": self.res["K"]}[which]


def fake_ffi():
    def kern_K(kind, ARD, var, ls, X, X2=None):
        return o.StationaryOracle(kind, X.shape[1], var, ls, ARD).K(X, X2)

    def kern_Kdiag(kind, var, N):
        return np.full(N, var)

    def kern_grad_full(kind, ARD, var, ls, X, dL_dK, X2=None):
        dv, dl = o.StationaryOracle(kind, X.shape[1], var, ls, ARD).update_gradients_full(dL_dK, X, X2)
        return dv, np.atleast_1d(dl)

    return types.SimpleNamespace(kern_K=kern_K, kern_Kdiag=kern_Kdiag, kern_grad_full=kern_grad_full, Engine=FakeEngine)


@pytest.fixture(scope="module")
def setup():
    from oracle import ref_gpy
    from gpy_b200 import gpy_plugin
    G = ref_gpy.load()
    B = gpy_plugin.make(G.RBF, G.Exponential, G.Matern32, G.Matern52, G.ExactGaussianInference, ffi=fake_ffi())
    return G, B


@pytest.mark.parametrize("name,kind", [("RBF", "rbf"), ("Matern32", "matern32"), ("Matern52", "matern52"),
                                       ("Exponential", "exponential")])
@pytest.mark.parametrize("ARD", [False, True])
def test_plugin_equals_stock_reference(setup, name, kind, ARD):
    G, B = setup
    X, Y = o.synthetic(90, 4, 3)
    Xwide = np.hstack([X, np.random.default_rng(0).standard_normal((90, 2))])   # active_dims slicing: use cols 0..3 of 6
    ls = np.array([1.1, 1.4, 1.9, 2.3]) if ARD else 1.7
    stock = getattr(G, name)(4, variance=1.3, lengthscale=ls, ARD=ARD, active_dims=[0, 1, 2, 3])
    plug = getattr(B, name)(4, variance=1.3, lengthscale=ls, ARD=ARD, active_dims=[0, 1, 2, 3])
    assert isinstance(plug, getattr(G, name))                       # a real GPy kernel
    np.testing.assert_allclose(plug.K(Xwide), stock.K(Xwide), rtol=1e-13)          # went through _slice_K
    np.testing.assert_allclose(plug.K(Xwide, Xwide[:7]), stock.K(Xwide, Xwide[:7]), rtol=1e-13)
    np.testing.assert_array_equal(plug.Kdiag(Xwide), stock.Kdiag(Xwide))
    # one GP.parameters_changed() with the plugin pair vs the stock pair (gp.py:278-280)
    from oracle import ref_gpy
    lik_s, lik_p = G.Gaussian(variance=0.07), G.Gaussian(variance=0.07)
    inf_s, inf_p = G.ExactGaussianInference(), B.ExactGaussianInference()
    post_s, lml_s, gd_s = inf_s.inference(stock, Xwide, lik_s, Y)
    post_p, lml_p, gd_p = inf_p.inference(plug, Xwide, lik_p, Y)
    lik_s.update_gradients(gd_s["dL_dthetaL"]); lik_p.update_gradients(gd_p["dL_dthetaL"])
    stock.update_gradients_full(gd_s["dL_dK"], Xwide); plug.update_gradients_full(gd_p["dL_dK"], Xwide)
    assert abs(lml_s - lml_p) < 1e-10
    np.testing.assert_allclose(plug.variance.gradient, stock.variance.gradient, rtol=1e-10)
    np.testing.assert_allclose(plug.lengthscale.gradient, stock.lengthscale.gradient, rtol=1e-10)
    np.testing.assert_allclose(lik_p.variance.gradient, lik_s.variance.gradient, rtol=1e-10)
    np.testing.assert_allclose(post_p.woodbury_vector, post_s.woodbury_vector, rtol=1e-10)
    np.testing.assert_allclose(np.asarray(gd_p["dL_dK"]), gd_s["dL_dK"], rtol=1e-9, atol=1e-12)   # handle -> ndarray
    assert inf_p.engine.calls == ["set_data", "exact_eval"]
    inf_p.inference(plug, Xwide, lik_p, Y)
    assert inf_p.engine.calls == ["set_data", "exact_eval", "exact_eval"]        # data stays resident across iterates
    # a foreign (plain ndarray) dL_dK takes the generic reduction
    dL = np.random.default_rng(1).standard_normal((90, 90))
    stock.update_gradients_full(dL, Xwide); plug.update_gradients_full(dL, Xwide)
    np.testing.assert_allclose(plug.lengthscale.gradient, stock.lengthscale.gradient, rtol=1e-10)
    # a stale handle (kernel parameters changed since) must NOT short-circuit
    plug.variance[:] = 2.0
    plug.update_gradients_full(gd_p["dL_dK"], Xwide)
    stock.variance[:] = 2.0
    stock.update_gradients_full(gd_s["dL_dK"], Xwide)
    np.testing.assert_allclose(plug.variance.gradient, stock.variance.gradient, rtol=1e-9)


def test_unsupported_cases_fall_back_to_stock_method(setup):
    G, B = setup
    X, Y = o.synthetic(40, 2, 1)
    inf = B.ExactGaussianInference()
    stock_kernel = G.RBF(2)                      # not a plugin kernel -> stock inference, no engine call
    post, lml, gd = inf.inference(stock_kernel, X, G.Gaussian(variance=0.1), Y)
    assert isinstance(gd["dL_dK"], np.ndarray) and inf._engine is None
    plug = B.RBF(2)
    Kpre = plug.K(X)
    post, lml2, gd = inf.inference(plug, X, G.Gaussian(variance=0.1), Y, K=Kpre)   # precomputed K -> stock
    assert abs(lml - lml2) < 1e-10 and inf._engine is None


def test_plugin_heteroscedastic_likelihood_equals_stock_reference(setup):
    """The reference's own HeteroscedasticGaussian (likelihoods/gaussian.py:347-362) through the plugin inference: the
    vector `variance` is routed to the per-point entry (gpx_exact_eval_het) and dL_dthetaL comes back through the
    likelihood's own exact_inference_gradients — equal to the stock ExactGaussianInference with the stock kernel."""
    G, B = setup
    N = 60
    X, Y = o.synthetic(N, 3, 7)
    md = {"output_index": np.arange(N)[:, None]}
    nv = np.random.default_rng(2).uniform(0.02, 0.3, N)
    stock, plug = G.Matern32(3, variance=1.2, lengthscale=1.6), B.Matern32(3, variance=1.2, lengthscale=1.6)
    lik_s, lik_p = G.HeteroscedasticGaussian(md), G.HeteroscedasticGaussian(md)
    lik_s.variance[:] = nv.reshape(lik_s.variance.shape)
    lik_p.variance[:] = nv.reshape(lik_p.variance.shape)
    inf_s, inf_p = G.ExactGaussianInference(), B.ExactGaussianInference()
    post_s, lml_s, gd_s = inf_s.inference(stock, X, lik_s, Y, None, md)
    post_p, lml_p, gd_p = inf_p.inference(plug, X, lik_p, Y, None, md)
    assert inf_p.engine.calls == ["set_data", "exact_eval_het"]
    assert abs(lml_s - lml_p) < 1e-10
    np.testing.assert_allclose(np.asarray(gd_p["dL_dthetaL"]).reshape(-1), np.asarray(gd_s["dL_dthetaL"]).reshape(-1), rtol=1e-9,
                               atol=1e-12)
    lik_s.update_gradients(gd_s["dL_dthetaL"]); lik_p.update_gradients(gd_p["dL_dthetaL"])
    np.testing.assert_allclose(np.asarray(lik_p.variance.gradient).reshape(-1), np.asarray(lik_s.variance.gradient).reshape(-1),
                               rtol=1e-9, atol=1e-12)
    stock.update_gradients_full(gd_s["dL_dK"], X); plug.update_gradients_full(gd_p["dL_dK"], X)
    np.testing.assert_allclose(plug.variance.gradient, stock.variance.gradient, rtol=1e-10)
    np.testing.assert_allclose(plug.lengthscale.gradient, stock.lengthscale.gradient, rtol=1e-10)


def test_plugin_inference_serialises_as_the_stock_class(setup):
    """`to_dict()` (exact_gaussian_inference.py:24-35) is inherited: a model saved to JSON names the stock class, so it loads
    on a machine without the library (CPU-equivalent fallback on load, like pickling: GPy/kern/src/rbf.py:313-318)."""
    G, B = setup
    d = B.ExactGaussianInference().to_dict()
    assert d["class"] == "GPy.inference.latent_function_inference.exact_gaussian_inference.ExactGaussianInference"
    import pickle
    inf = B.ExactGaussianInference()
    X, Y = o.synthetic(30, 2, 1)
    inf.inference(B.RBF(2), X, G.Gaussian(variance=0.1), Y)
    st = inf.__getstate__()
    assert st["_engine"] is None                       # the device handle does not travel
