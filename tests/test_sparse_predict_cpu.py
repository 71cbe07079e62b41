"""Sparse prediction without a GPU: the NumPy restatement of tests/sparse_predict_cases.py against the reference's own
VarDTC posterior (tests/golden/sparse_predict), and the host routing of LazySparsePosterior._raw_predict on test doubles
of the engine: the evaluated kernel and Z make one sparse_predict call, anything else takes the formula on the fetched
woodbury arrays, and the reference's own SparseGP over the plugin's VarDTC reaches the same call."""
import glob
import os

import numpy as np
import pytest

import gpy_b200
import sparse_predict_cases as cases
from gpy_b200 import _ffi
from gpy_b200.sparse import LazySparsePosterior
from oracle import gpy_oracle as o
from test_host_model_cpu import FakeSparseEngine

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = sorted(glob.glob(os.path.join(HERE, "golden", "sparse_predict", "*.npz")))


def test_every_case_has_a_fixture():
    assert sorted(os.path.basename(p)[:-4] for p in FIXTURES) == sorted(cases.CASES)


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[:-4])
def test_restatement_matches_the_reference_fixtures(path):
    f = np.load(path)
    c = cases.CASES[os.path.basename(path)[:-4]]
    kern = cases.oracle_kernel(c)
    wv, wi = f["woodbury_vector"], f["woodbury_inv"]
    mu, var = cases.predict(wv, wi, kern, f["Z"], f["Xnew"])
    mu_f, cov = cases.predict(wv, wi, kern, f["Z"], f["Xnew"], full_cov=True)
    assert mu.shape == f["mu"].shape and var.shape == f["var"].shape == (f["Xnew"].shape[0], 1)
    for got, want in ((mu, f["mu"]), (var, f["var"]), (mu_f, f["mu_full"]), (cov, f["cov"])):
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12 * np.abs(want).max())
    if "clip" in path:
        assert np.all(f["var"] == cases.CLIP) and np.all(var == cases.CLIP)   # the reference clips every entry
        assert np.abs(f["cov"]).max() < 1e-17                                 # the full covariance is not clipped


# ---- routing on test doubles ---------------------------------------------------------------------------------------------
class PredictEngine(FakeSparseEngine):
    """the sparse test double with gpx_sparse_predict, answered by the restatement from the evaluation it holds"""

    def sparse_eval(self, kind, ARD, variance, lengthscale, Z, noise_variance):
        self.theta, self.Z = (kind, ARD, variance, lengthscale), np.array(Z)
        return super(PredictEngine, self).sparse_eval(kind, ARD, variance, lengthscale, Z, noise_variance)

    def kern(self):
        kind, ARD, variance, lengthscale = self.theta
        return o.StationaryOracle(kind, self.Z.shape[1], variance, lengthscale, ARD)

    def sparse_predict(self, Xnew, full_cov=False):
        self.calls.append("sparse_predict")
        return cases.predict(self.res["woodbury_vector"], self.res["woodbury_inv"], self.kern(), self.Z, Xnew, full_cov)


@pytest.fixture
def host_kernels(monkeypatch):
    """the stand-alone kernel calls of the host route answered by the restatement"""
    def kern_of(kind, ARD, variance, lengthscale, D):
        return o.StationaryOracle(kind, D, variance, lengthscale, ARD)
    monkeypatch.setattr(_ffi, "kern_K", lambda kind, ARD, v, ls, X, X2=None: kern_of(kind, ARD, v, ls, X.shape[1]).K(X, X2))
    monkeypatch.setattr(_ffi, "kern_Kdiag", lambda kind, v, N: np.full(N, v))


def _model(engine, seed=4, D=3, P=2):
    rng = np.random.default_rng(seed)
    X = rng.uniform(-2, 2, (80, D))
    Y = np.sin(X.sum(1, keepdims=True) + np.arange(P)) + 0.1 * rng.standard_normal((80, P))
    Z = X[:9] + 0.05
    k = gpy_b200.RBF(D, variance=1.2, lengthscale=[0.9, 1.4, 1.7], ARD=True)
    m = gpy_b200.SparseGPRegression(X, Y, kernel=k, Z=Z, engine=engine)
    return m, rng.uniform(-2.5, 2.5, (7, D))


def _host(m, kern, Xnew, full_cov):
    """the reference's formula on the posterior the engine holds"""
    eng = m.inference_method.engine
    return cases.predict(eng.res["woodbury_vector"], eng.res["woodbury_inv"], kern, m.Z.values, Xnew, full_cov)


@pytest.mark.parametrize("full_cov", [False, True])
def test_the_evaluated_kernel_makes_one_sparse_predict_call(full_cov):
    eng = PredictEngine()
    m, Xnew = _model(eng)
    n = len(eng.calls)
    mu, var = m.predict(Xnew, full_cov=full_cov, include_likelihood=False)
    assert eng.calls[n:] == ["sparse_predict"]
    rm, rv = _host(m, eng.kern(), Xnew, full_cov)
    np.testing.assert_array_equal(mu, rm)
    np.testing.assert_array_equal(var, rv)
    # predict adds the Gaussian noise to the same call's result, predict_noiseless does not
    mu2, var2 = m.predict(Xnew, full_cov=full_cov)
    noise = float(m.likelihood.variance[0])
    np.testing.assert_array_equal(var2, rv + (noise * np.eye(7) if full_cov else noise))
    mu3, var3 = m.predict_noiseless(Xnew, full_cov=full_cov)
    np.testing.assert_array_equal(var3, rv)
    assert eng.calls[n:] == ["sparse_predict"] * 3 and "woodbury_inv" not in eng.calls


def test_predict_keeps_its_positional_order_and_takes_another_likelihood():
    eng = PredictEngine()
    m, Xnew = _model(eng)
    _, v0 = m.predict(Xnew, False, False)
    lik = gpy_b200.Gaussian(variance=0.25)
    _, v1 = m.predict(Xnew, False, True, None, None, lik)
    np.testing.assert_array_equal(v1, v0 + 0.25)


def test_another_kernel_takes_the_host_route(host_kernels):
    eng = PredictEngine()
    m, Xnew = _model(eng)
    other = gpy_b200.Matern52(3, variance=0.7, lengthscale=1.3)
    n = len(eng.calls)
    for full_cov in (False, True):
        mu, var = m.predict(Xnew, full_cov=full_cov, include_likelihood=False, kern=other)
        rm, rv = _host(m, o.StationaryOracle("matern52", 3, 0.7, 1.3, False), Xnew, full_cov)
        np.testing.assert_allclose(mu, rm, rtol=1e-13, atol=1e-15)
        if full_cov:
            np.testing.assert_allclose(var, rv, rtol=1e-12, atol=1e-14)
        else:   # the host fallback does not clip (SparsePosterior._raw_predict); these variances are far above 1e-15
            assert var.min() > 1e-6
            np.testing.assert_allclose(var, rv, rtol=1e-12, atol=1e-14)
    assert "sparse_predict" not in eng.calls[n:]
    # a kernel equal in every parameter is the evaluated kernel: the device route
    same = gpy_b200.RBF(3, variance=1.2, lengthscale=[0.9, 1.4, 1.7], ARD=True)
    m.predict(Xnew, kern=same)
    assert eng.calls[-1] == "sparse_predict"


def test_predictive_variable_other_than_z_takes_the_host_route(host_kernels):
    eng = PredictEngine()
    m, Xnew = _model(eng)
    n = len(eng.calls)
    Z2 = m.Z.values + 0.5
    mu, var = m.posterior._raw_predict(m.kern, Xnew, Z2)
    assert "sparse_predict" not in eng.calls[n:]
    rm, rv = cases.predict(eng.res["woodbury_vector"], eng.res["woodbury_inv"], eng.kern(), Z2, Xnew)
    np.testing.assert_allclose(mu, rm, rtol=1e-13, atol=1e-15)
    np.testing.assert_allclose(var, rv, rtol=1e-12, atol=1e-14)
    Z3 = m.Z.values.copy()
    Z3[4, 1] += 1e-12                                          # one coordinate moved by 1e-12: not the evaluated Z
    m.posterior._raw_predict(m.kern, Xnew, Z3)
    assert "sparse_predict" not in eng.calls[n:]
    m.posterior._raw_predict(m.kern, Xnew, m.Z.values.copy())
    assert eng.calls[-1] == "sparse_predict"


def test_an_engine_without_sparse_predict_and_a_keyless_posterior_take_the_host_route(host_kernels):
    eng = FakeSparseEngine()
    m, Xnew = _model(eng)
    mu, var = m.predict(Xnew, include_likelihood=False)
    assert "sparse_predict" not in eng.calls and mu.shape == (7, 2) and var.shape == (7, 1)
    eng2 = PredictEngine()
    m2, _ = _model(eng2)
    post = LazySparsePosterior(eng2)                       # the one-argument constructor stays valid: no key, no Z
    post._raw_predict(m2.kern, Xnew, m2.Z.values)
    assert "sparse_predict" not in eng2.calls


def test_a_stale_posterior_refuses_the_device_route():
    eng = PredictEngine()
    m, Xnew = _model(eng)
    post = m.posterior
    m.likelihood.variance[:] = 0.3
    m.parameters_changed()
    with pytest.raises(RuntimeError, match="stale"):
        post._raw_predict(m.kern, Xnew, m.Z.values)


def test_the_reference_sparse_gp_over_the_plugin_vardtc_reaches_the_engine():
    """the reference's own SparseGP.predict (gp.py:290-365 -> posterior._raw_predict with pred_var = Z, sparse_gp.py:63)
    over B.VarDTC and a plugin kernel: one sparse_predict call with the sliced inputs, the stock model's numbers"""
    if not os.path.isdir(os.environ.get("GPX_REFERENCE", "/root/reference") + "/GPy"):
        pytest.skip("reference tree not present")
    from test_real_gpy_sparse_model import _data, _plugin, fake_sparse_ffi
    ffi = fake_sparse_ffi()
    ffi.Engine = lambda device=0: PredictEngine()
    S, G, B = _plugin(ffi)
    X, Y, Z = _data(120, 11, 3, P=2, seed=6)
    Xnew = np.random.default_rng(2).uniform(-3, 3, (9, 3))
    stock = S.SparseGP(X, Y, Z.copy(), G.RBF(2, variance=1.1, lengthscale=1.6, active_dims=[0, 2]),
                       G.Gaussian(variance=0.1))
    plug = S.SparseGP(X, Y, Z.copy(), B.RBF(2, variance=1.1, lengthscale=1.6, active_dims=[0, 2]),
                      G.Gaussian(variance=0.1), inference_method=B.VarDTC())
    eng = plug.inference_method.engine
    for full_cov in (False, True):
        n = len(eng.calls)
        mp, vp = plug.predict(Xnew, full_cov=full_cov)
        assert eng.calls[n:] == ["sparse_predict"]
        ms, vs = stock.predict(Xnew, full_cov=full_cov)
        np.testing.assert_allclose(mp, ms, rtol=1e-9, atol=1e-12)
        np.testing.assert_allclose(vp, vs, rtol=1e-9, atol=1e-12)
    n = len(eng.calls)
    plug.predict(Xnew, kern=B.RBF(2, variance=0.5, lengthscale=1.0, active_dims=[0, 2]))
    assert "sparse_predict" not in eng.calls[n:]


def test_the_abi_export_is_declared_bound_and_built():
    with open(os.path.join(os.path.dirname(HERE), "include", "gpx.h")) as fh:
        assert "int gpx_sparse_predict(gpx_ctx* ctx, const double* Xnew, int64_t M, int full_cov, double* mu, double* var);" \
            in fh.read()
    assert "gpx_sparse_predict" in _ffi.EXPORTS
    if not os.path.exists(_ffi.LIB_PATH):
        pytest.skip("libgpx.so not built")
    assert hasattr(_ffi.lib(), "gpx_sparse_predict")
