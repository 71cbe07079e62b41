"""The variational Gaussian approximation on the device (gpx_vargauss_*, gpy_b200.VarGauss): the reference's fixtures
replayed with their own dF_dm / dF_dv, the Gaussian-likelihood optimum against the exact evaluation at sizes where no N^3
NumPy is needed, checkgrad through the mirror's model, bit-identical repeats, the rejections, launch counts and the
posterior's consumers."""
import ctypes
import glob
import os

import numpy as np
import pytest

import vargauss_oracle as vo
from test_gpu_laplace import _sweep_launches, mirror_kernel

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = sorted(glob.glob(os.path.join(HERE, "golden", "vargauss", "*.npz")))
EPS = np.finfo(np.float64).eps


def _B():
    import gpy_b200
    return gpy_b200


def _rel(a, b):
    b = np.asarray(b, dtype=np.float64)
    return float(np.abs(np.asarray(a) - b).max() / max(np.abs(b).max(), 1e-300)) if b.size else 0.0


def _replay(eng, name, z):
    parts = vo.CASES[name][0]
    eng.set_data(z["X"], z["Y"])
    m, var, kl, jit = eng.vargauss_begin([vo.descriptor(p) for p in parts], z["alpha"], z["beta"])
    da, db, kg = eng.vargauss_finish(z["dF_dm"], z["dF_dv"])
    return m, var, kl, jit, da, db, kg


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[:-4])
def test_fixture(path):
    """bound, alpha and beta gradients against the reference's own VarGauss, the kernel gradient against the oracle's
    (column-scaled) form. Bars: a few hundred eps times cond(A) <= 1 + max beta^2 lambda_max(K)"""
    B = _B()
    name = os.path.basename(path)[:-4]
    z = np.load(path)
    parts, lik_spec = vo.CASES[name][:2]
    K = vo.CompositeOracle(parts).K(z["X"])
    bar = 300 * EPS * vo.cond_bound(K, z["beta"])
    m, var, kl, jit, da, db, kg = _replay(B.Engine(), name, z)
    lml = float(np.sum(z["F"])) - kl
    o = vo.vargauss_eval(parts, z["X"], z["Y"], z["alpha"], z["beta"], vo.make_likelihood(lik_spec, B))
    margins = dict(lml=abs(lml - float(z["lml"])) / max(1.0, abs(float(z["lml"]))), m=_rel(m, z["m"]),
                   var=_rel(var, z["var"]), dalpha=_rel(da, z["dalpha"]), dbeta=_rel(db, z["dbeta"]),
                   kgrad=_rel(kg, o["grad"]))
    print(name, "bar %.1e" % bar, " ".join("%s %.1e" % kv for kv in margins.items()))
    for k, v in margins.items():
        assert v <= bar, k


def _gaussian_optimum(N, seed=3):
    """alpha = (K + s2 I)^-1 y, beta = 1 / sigma: the bound equals the exact log marginal likelihood there"""
    B = _B()
    rng = np.random.default_rng(seed)
    X = rng.uniform(-3, 3, size=(N, 3))
    Y = np.sin(X[:, :1]) + 0.5 * X[:, 1:2] + 0.3 * rng.standard_normal((N, 1))
    s2 = 0.3
    parts = [("rbf", True, 0, [0, 1, 2], 1.2, [0.9, 1.3, 1.7])]
    eng = B.Engine()
    eng.set_data(X, Y)
    lml_exact, g_exact, _ = eng.exact_eval_multi(parts, s2, jitter=0.0)
    alpha = eng.get("alpha")[:, 0].copy()
    beta = np.full(N, 1.0 / np.sqrt(s2))
    m, var, kl, jit = eng.vargauss_begin(parts, alpha, beta)
    F, dF_dm, dF_dv, _ = B.Gaussian(variance=s2).variational_expectations(Y, m[:, None], var[:, None])
    da, db, kg = eng.vargauss_finish(dF_dm[:, 0], dF_dv[:, 0])
    return dict(lml_exact=lml_exact, g_exact=np.asarray(g_exact), bound=float(F.sum()) - kl, m=m, da=da, db=db, kg=kg,
                jit=jit, beta=beta)


@pytest.mark.parametrize("N", [4097, 16384])
def test_gaussian_optimum_matches_the_exact_evaluation(N):
    """at the optimum of alpha and beta the bound is the exact LML, its alpha and beta gradients vanish and, by the
    envelope theorem, its kernel gradient is the exact one. cond(K + s2 I) <= 1 + N 1.2 / 0.3 sets the bars"""
    r = _gaussian_optimum(N)
    c = 1 + N * 1.2 / 0.3
    assert r["jit"] == 0.0
    assert abs(r["bound"] - r["lml_exact"]) <= 100 * EPS * c * abs(r["lml_exact"])
    assert np.abs(r["da"]).max() <= 100 * EPS * c * np.abs(r["m"]).max()
    assert np.abs(r["db"]).max() <= 1e3 * EPS * c * N
    np.testing.assert_allclose(r["kg"], r["g_exact"][:r["kg"].size], rtol=100 * EPS * c, atol=0)


def _model(lik, seed=5, N=40):
    B = _B()
    rng = np.random.default_rng(seed)
    X = rng.uniform(-2, 2, size=(N, 2))
    f = np.sin(2 * X[:, :1]) + 0.5 * X[:, 1:]
    if lik == "bernoulli":
        Y, L = (f + 0.3 * rng.standard_normal((N, 1)) > 0).astype(float), B.Bernoulli()
    else:
        Y, L = f + 0.2 * rng.standard_t(3.0, size=(N, 1)), B.StudentT(deg_free=4.0, sigma2=0.5)
    k = B.Matern52(2, variance=1.2, lengthscale=[0.9, 1.4], ARD=True)
    m = B.GPVariationalGaussianApproximation(X, Y, k, L)
    m.alpha.values[...] = 0.3 * rng.standard_normal((N, 1))
    m.beta.values[...] = rng.uniform(0.5, 2.0, N)
    m.parameters_changed()
    return m


@pytest.mark.parametrize("lik", ["bernoulli", "studentt"])
def test_checkgrad(lik):
    """every parameter, the 2 N variational ones included. StudentT's expectations are 20-point Gauss-Hermite sums whose
    dF_dv is the quadrature of d2logpdf_df2 / 2, not the derivative of the quadrature of logpdf; the two differ by about
    1e-3 here, hence its tolerance"""
    m = _model(lik)
    assert m.checkgrad(step=1e-5, tolerance=1e-3 if lik == "bernoulli" else 1e-2, verbose=True)


def test_repeated_calls_are_bit_identical():
    B = _B()
    z = np.load(os.path.join(HERE, "golden", "vargauss", "bernoulli_m52_x_rbf_bias_n128.npz"))
    eng = B.Engine()
    a = _replay(eng, "bernoulli_m52_x_rbf_bias_n128", z)
    b = _replay(eng, "bernoulli_m52_x_rbf_bias_n128", z)
    c = _replay(B.Engine(), "bernoulli_m52_x_rbf_bias_n128", z)
    d = eng.vargauss_finish(z["dF_dm"], z["dF_dv"])                      # a finish after a finish factors A again
    for x in (b, c):
        for u, v in zip(a, x):
            np.testing.assert_array_equal(u, v)
    for u, v in zip(a[4:], d):
        np.testing.assert_array_equal(u, v)
    e = eng.vargauss_finish(2 * z["dF_dm"], z["dF_dv"])
    assert not np.array_equal(e[0], a[4])


def test_rejections():
    B = _B()
    from gpy_b200 import _ffi
    z = np.load(os.path.join(HERE, "golden", "vargauss", "bernoulli_rbf_iso_n60.npz"))
    X, Y = z["X"], z["Y"]
    N = X.shape[0]
    parts = (_ffi.GpxKernPart * 1)()
    keep = []
    _ffi._fill_part(parts[0], ("rbf", False, 0, [0, 1, 2], 1.0, 1.0), keep)
    v, w = np.ones(N), np.empty(N)
    p, q = v.ctypes.data_as(_ffi._dp), w.ctypes.data_as(_ffi._dp)
    kg = np.zeros(2)
    g = kg.ctypes.data_as(_ffi._dp)
    d = ctypes.c_double()
    eng = B.Engine()
    L, h = eng._L, eng._h

    def begin(a=p, b=p, prt=parts):
        return L.gpx_vargauss_begin(h, prt, 1, a, b, 5, q, q, ctypes.byref(d), ctypes.byref(d))

    def finish():
        return L.gpx_vargauss_finish(h, p, p, q, q, g)

    assert begin() == -2                                                   # no data
    eng.set_data(X, np.hstack([Y, Y]))
    assert begin() == -2                                                   # P = 2
    eng.set_data(X, Y)
    assert finish() == -2                                                  # no begin
    assert begin(prt=None) == -2
    assert begin(a=None) == -2
    assert L.gpx_vargauss_begin(h, parts, 1, p, p, 5, q, q, None, ctypes.byref(d)) == -2
    for bad in (0.0, np.nan, np.inf):
        b = np.ones(N)
        b[7] = bad
        assert begin(b=b.ctypes.data_as(_ffi._dp)) == -2
    with pytest.raises(ValueError):
        eng.vargauss_begin([("rbf", False, 0, [0, 1, 2], 1.0, 1.0)], v, np.zeros(N))
    assert begin() == 0
    assert L.gpx_vargauss_finish(h, None, p, q, q, g) == -2
    assert L.gpx_vargauss_finish(h, p, p, q, q, None) == -2
    assert finish() == 0
    assert finish() == 0
    eng.laplace_begin([("rbf", False, 0, [0, 1, 2], 1.0, 1.0)])            # another Laplace call: a new begin is needed
    assert finish() == -2
    assert begin() == 0
    eng.exact_eval("rbf", False, 1.0, 1.0, 0.1)                           # an exact evaluation releases K
    assert finish() == -2
    assert begin() == 0
    eng.set_data(X, Y)                                                     # new data
    assert finish() == -2
    uid = ctypes.create_string_buffer(128)                                 # a communicator attached: single-GPU only
    assert L.gpx_comm_unique_id(uid) == 0
    assert L.gpx_comm_init(h, uid.raw, 0, 1) == 0
    eng.set_data(X, Y)
    assert begin() == -2
    assert finish() == -2
    eng.close()
    m = _model("bernoulli")
    m.beta.values[3] = 0.0
    with pytest.raises(ValueError):
        m.parameters_changed()


@pytest.mark.parametrize("N", [300, 1300])
def test_launch_counts_do_not_depend_on_N(N):
    B = _B()
    rng = np.random.default_rng(N)
    X = rng.uniform(-2, 2, size=(N, 3))
    Y = (X[:, :1] > 0).astype(float)
    eng = B.Engine()
    eng.set_data(X, Y)
    parts = [("rbf", True, 0, [0, 1, 2], 1.0, [1.0, 1.2, 0.8]), ("bias", False, 1, [], 0.3, None)]
    F = _sweep_launches(N)
    eng.vargauss_begin(parts, 0.1 * np.ones(N), np.ones(N))
    assert eng.stats()["launches"] - F == 7
    eng.vargauss_finish(np.ones(N), -0.2 * np.ones(N))
    assert eng.stats()["launches"] == 8 + 2
    eng.vargauss_finish(np.ones(N), -0.2 * np.ones(N))
    assert eng.stats()["launches"] - F == 8 + 2 + 1


def test_posterior_consumers():
    """woodbury_vector alpha and woodbury_inv (K + B^-2)^-1: predict, the joint covariance, the samples and the
    predictive gradients against the host formulas"""
    B = _B()
    name = "bernoulli_m52_x_rbf_bias_n128"
    parts, lik_spec = vo.CASES[name][:2]
    X, Y, alpha, beta, Xnew = vo.case_data(name)
    kern = mirror_kernel(parts)
    from gpy_b200.param import Param
    a, b = Param("alpha", alpha[:, None], transform=None), Param("beta", beta.copy(), transform=None)
    inf = B.VarGauss(a, b)
    post, lml, gd = inf.inference(kern, X, vo.make_likelihood(lik_spec, B), Y)
    eng = inf.engine
    ko = vo.CompositeOracle(parts)
    K = ko.K(X)
    Wi = np.linalg.inv(K + np.diag(beta ** -2.0))
    c = np.linalg.cond(K + np.diag(beta ** -2.0))
    np.testing.assert_array_equal(post.woodbury_vector[:, 0], alpha)
    np.testing.assert_allclose(post.woodbury_inv, Wi, rtol=0, atol=100 * EPS * c * np.abs(Wi).max())
    with pytest.raises(ValueError):
        eng.get("dL_dK")
    Kx = ko.K(X, Xnew)
    mu, var = post._raw_predict(kern, Xnew, X)
    np.testing.assert_allclose(mu[:, 0], Kx.T.dot(alpha), rtol=0, atol=1e-12)
    np.testing.assert_allclose(var[:, 0], np.clip(ko.Kdiag(Xnew) - np.sum(Wi.dot(Kx) * Kx, 0), 1e-15, np.inf),
                               rtol=0, atol=1e-11)
    z = np.load(os.path.join(HERE, "golden", "vargauss", name + ".npz"))
    np.testing.assert_allclose(mu[:, 0], z["pmu"], rtol=0, atol=1e-10)
    np.testing.assert_allclose(var[:, 0], z["pvar"], rtol=0, atol=1e-10)
    X2 = Xnew[:11] + 0.1
    cov = eng.posterior_covariance(Xnew, X2)
    np.testing.assert_allclose(cov, ko.K(Xnew, X2) - Kx.T.dot(Wi).dot(ko.K(X, X2)), rtol=0, atol=1e-11)
    zz = np.random.default_rng(0).standard_normal((3, Xnew.shape[0]))
    f, jit = eng.posterior_samples(Xnew, zz)
    Sig = ko.K(Xnew) - Kx.T.dot(Wi).dot(Kx)
    Ls = np.linalg.cholesky(Sig + jit * np.eye(Sig.shape[0]))
    np.testing.assert_allclose(f, (Kx.T.dot(alpha)).reshape(1, -1) + zz.dot(Ls.T), rtol=0, atol=1e-8)
    # the predictive gradients of a single kernel against the host formula with the stand-alone kernel calls
    name = "bernoulli_matern32_ard_n60"
    parts, lik_spec = vo.CASES[name][:2]
    X, Y, alpha, beta, Xnew = vo.case_data(name)
    kern = mirror_kernel(parts)
    a, b = Param("alpha", alpha[:, None], transform=None), Param("beta", beta.copy(), transform=None)
    inf = B.VarGauss(a, b, engine=eng)
    post, _, _ = inf.inference(kern, X, vo.make_likelihood(lik_spec, B), Y)
    dmu, dvar = post._predictive_gradients(kern, Xnew)
    from gpy_b200.model import host_predictive_gradients
    hmu, hvar = host_predictive_gradients(kern, post, Xnew, X)
    np.testing.assert_allclose(dmu, hmu, rtol=0, atol=1e-11)
    np.testing.assert_allclose(dvar, hvar, rtol=0, atol=1e-11)
