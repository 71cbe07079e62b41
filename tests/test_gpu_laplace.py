"""The Laplace approximation on the device (gpx_laplace_*, gpy_b200.Laplace): the reference's fixtures, the posterior's
consumers, gradients and optimisation through the mirror's GP, context reuse, the rejections and the launch counts."""
import ctypes
import glob
import os

import numpy as np
import pytest

import laplace_oracle as lo

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = sorted(glob.glob(os.path.join(HERE, "golden", "laplace", "*.npz")))


def _B():
    import gpy_b200
    return gpy_b200


def mirror_kernel(parts):
    B = _B()
    cls = {"rbf": B.RBF, "exponential": B.Exponential, "matern32": B.Matern32, "matern52": B.Matern52}
    terms = {}
    for p in parts:
        if p["kind"] == "bias":
            k = B.Bias(lo.D, variance=p["variance"])
        else:
            d = p["dims"]
            k = cls[p["kind"]](len(d), variance=p["variance"], lengthscale=p["lengthscale"], ARD=p.get("ARD", False),
                               active_dims=d)
        terms.setdefault(p["term"], []).append(k)
    prods = []
    for t in sorted(terms):
        k = terms[t][0]
        for q in terms[t][1:]:
            k = k * q
        prods.append(k)
    out = prods[0]
    for q in prods[1:]:
        out = out + q
    return out


def likelihood(spec):
    return lo.make_likelihood(spec, _B())


def evaluate(name, engine=None):
    """one Laplace evaluation of a fixture case through the mirror -> (inference, posterior, lml, kernel gradient,
    dL_dthetaL, kernel)"""
    B = _B()
    parts, lik, _, _ = lo.CASES[name]
    X, Y, _ = lo.case_data(name)
    kern = mirror_kernel(parts)
    inf = B.Laplace(engine=engine)
    post, lml, gd = inf.inference(kern, X, likelihood(lik), Y)
    kern.update_gradients_full(gd["dL_dK"], X)
    return inf, post, lml, np.asarray(kern.gradient).copy(), np.asarray(gd["dL_dthetaL"]), kern


def _rel(a, b):
    b = np.asarray(b, dtype=np.float64)
    return float(np.abs(np.asarray(a) - b).max() / max(1.0, np.abs(b).max())) if b.size else 0.0


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[:-4])
def test_fixture(path):
    """LML and gradients against the reference's own Laplace. The bars are those the NumPy restatement meets against the
    same fixtures (tests/test_laplace_cpu.py): Brent's last step on the flat objective moves with rounding."""
    name = os.path.basename(path)[:-4]
    z = np.load(path)
    X, _, Xnew = lo.case_data(name)
    inf, post, lml, kg, dth, kern = evaluate(name)
    margins = dict(lml=abs(lml - float(z["lml"])) / abs(float(z["lml"])), grad=_rel(kg, z["grad"]),
                   dL_dthetaL=_rel(dth, z["dL_dthetaL"]), f_hat=_rel(inf.f_hat, z["f_hat"]))
    mu, var = post._raw_predict(kern, Xnew, X)
    margins["mu"], margins["var"] = _rel(mu, z["mu"]), _rel(var, z["var"])
    print(name, " ".join("%s %.1e" % kv for kv in margins.items()))
    assert inf.iterations == int(z["iterations"])
    assert margins["lml"] <= 1e-8
    for k in ("grad", "dL_dthetaL", "f_hat", "mu", "var"):
        assert margins[k] <= 1e-6, k
    if "woodbury_inv" in z:
        np.testing.assert_allclose(post.woodbury_inv, z["woodbury_inv"], rtol=0,
                                   atol=1e-5 * max(1.0, float(np.abs(z["woodbury_inv"]).max())))


def test_posterior_members_and_consumers():
    """K, alpha, L, LiW12, K_Wi_i from gpx_get, and the predictive gradients, the joint covariance and the samples
    against the host formulas on the device's own posterior (posterior.py:109-130,220-302; gp.py:438-474,601-629)"""
    B = _B()
    name = "bernoulli_rbf_ard_x_m52_bias_n150"
    parts, lik, _, _ = lo.CASES[name]
    X, Y, Xnew = lo.case_data(name)
    eng = B.Engine()
    inf, post, lml, _, _, kern = evaluate(name, eng)
    ko = lo.CompositeOracle(parts)
    K = ko.K(X)
    np.testing.assert_allclose(eng.get("K"), K, rtol=0, atol=1e-13)
    np.testing.assert_array_equal(post.woodbury_vector, eng.get("alpha"))
    ref = lo.b_statistics(K, inf.W, lo.make_likelihood(lik, B).log_concave)
    np.testing.assert_allclose(eng.get("L"), ref[4], rtol=0, atol=1e-12)
    np.testing.assert_allclose(eng.get("Linv"), ref[5], rtol=0, atol=1e-11)
    Wi = post.woodbury_inv
    np.testing.assert_allclose(Wi, ref[0], rtol=0, atol=1e-12)
    # woodbury_chol is the reference's lazy value (posterior.py:152-159): Li of pdinv(woodbury_inv), (N, N, 1)
    from scipy.linalg import lapack
    Li = lapack.dtrtri(np.linalg.cholesky(ref[0]), lower=1)[0]
    wc = post.woodbury_chol
    assert wc.shape == (X.shape[0], X.shape[0], 1)
    np.testing.assert_allclose(wc[:, :, 0], Li, rtol=0, atol=1e-9 * np.abs(Li).max())
    with pytest.raises(ValueError):
        eng.get("dL_dK")
    a = post.woodbury_vector
    Kx = ko.K(X, Xnew)
    mu, var = post._raw_predict(kern, Xnew, X)
    np.testing.assert_allclose(mu, Kx.T.dot(a), rtol=0, atol=1e-12)
    np.testing.assert_allclose(var, np.clip(ko.Kdiag(Xnew) - np.sum(Wi.dot(Kx) * Kx, 0), 1e-15, np.inf)[:, None],
                               rtol=0, atol=1e-12)
    X2 = Xnew[:11] + 0.1
    cov = eng.posterior_covariance(Xnew, X2)
    np.testing.assert_allclose(cov, ko.K(Xnew, X2) - Kx.T.dot(Wi).dot(ko.K(X, X2)), rtol=0, atol=1e-12)
    np.testing.assert_allclose(post.covariance_between_points(kern, X, Xnew, X2), cov, rtol=0, atol=0)
    # another kernel: the same formula on the host with woodbury_inv
    other = [dict(p, variance=0.5 * p["variance"]) for p in parts]
    ko2 = lo.CompositeOracle(other)
    c2 = post.covariance_between_points(mirror_kernel(other), X, Xnew, X2)
    np.testing.assert_allclose(c2, ko2.K(Xnew, X2) - ko2.K(Xnew, X).dot(Wi).dot(ko2.K(X, X2)), rtol=0, atol=1e-12)
    z = np.random.default_rng(0).standard_normal((3, Xnew.shape[0]))
    f, jit = eng.posterior_samples(Xnew, z)
    Sig = ko.K(Xnew) - Kx.T.dot(Wi).dot(Kx)
    Ls = np.linalg.cholesky(Sig + jit * np.eye(Sig.shape[0]))
    np.testing.assert_allclose(f, (Kx.T.dot(a)).reshape(1, -1) + z.dot(Ls.T), rtol=0, atol=1e-9)
    # the predictive gradients of a single kernel against the host formula with the stand-alone kernel calls
    name = "bernoulli_matern32_ard_n150"
    X, Y, Xnew = lo.case_data(name)
    inf, post, _, _, _, kern = evaluate(name, eng)
    dmu, dvar = post._predictive_gradients(kern, Xnew)
    from gpy_b200.model import host_predictive_gradients
    hmu, hvar = host_predictive_gradients(kern, post, Xnew, X)
    np.testing.assert_allclose(dmu, hmu, rtol=0, atol=1e-11)
    np.testing.assert_allclose(dvar, hvar, rtol=0, atol=1e-11)


def _gp(lik, seed=5, N=80):
    B = _B()
    rng = np.random.default_rng(seed)
    X = rng.uniform(-2, 2, size=(N, 2))
    f = np.sin(2 * X[:, :1]) + 0.5 * X[:, 1:]
    if lik == "bernoulli":
        Y, L = (f + 0.3 * rng.standard_normal((N, 1)) > 0).astype(float), B.Bernoulli()
    else:
        # t_scale2 large enough that no W is clipped: with a clipped W the reference's own gradient is not that of its
        # LML (the implicit terms assume the unclipped Hessian), on the host as well as here
        Y, L = f + 0.2 * rng.standard_t(3.0, size=(N, 1)), B.StudentT(deg_free=4.0, sigma2=0.5)
    k = B.Matern52(2, variance=1.2, lengthscale=[0.9, 1.4], ARD=True)
    return B.GP(X, Y, k, L, inference_method=B.Laplace())


@pytest.mark.parametrize("lik", ["bernoulli", "studentt"])
def test_checkgrad(lik):
    m = _gp(lik)
    assert m.checkgrad(step=1e-5, tolerance=1e-3, verbose=True)
    if lik == "studentt":
        names = [p.name for p in m._free()]
        assert "t_scale2" in names and "deg_free" in names


def test_optimize_converges_and_predicts():
    m = _gp("bernoulli", seed=7, N=120)
    l0 = float(m.log_likelihood())
    r = m.optimize(max_iters=60)
    assert np.isfinite(r["f"]) and -r["f"] >= l0
    p, v = m.predict(np.array([[0.3, -0.2], [1.5, 1.0]]))
    assert p.shape == (2, 1) and np.all((p > 0) & (p < 1)) and np.all(np.isnan(v))


def test_exact_laplace_exact_on_one_context_is_bit_identical_to_fresh_contexts():
    B = _B()
    X, Y, _ = lo.case_data("bernoulli_rbf_ard_n150")
    Yr = np.sin(X[:, :1])

    def exact(eng):
        eng.set_data(X, Yr)
        return eng.exact_eval("matern32", True, 1.1, [0.7, 1.2, 1.5], 0.1)

    shared = B.Engine()
    e1 = exact(shared)
    _, _, l1, g1, _, _ = evaluate("bernoulli_rbf_ard_n150", shared)
    e2 = exact(shared)
    with pytest.raises(ValueError):    # the exact evaluation released the Laplace buffers: a new begin is needed
        shared.laplace_matvec(np.ones(X.shape[0]))
    f0 = exact(B.Engine())
    _, _, l0, g0, _, _ = evaluate("bernoulli_rbf_ard_n150", B.Engine())
    for a in (e1, e2):
        assert a[0] == f0[0]
        np.testing.assert_array_equal(a[1], f0[1])
    assert l1 == l0
    np.testing.assert_array_equal(g1, g0)


def _raw(eng):
    return eng._L, eng._h


def test_rejections():
    B = _B()
    from gpy_b200 import _ffi
    X, Y, _ = lo.case_data("bernoulli_rbf_iso_n60")
    N = X.shape[0]
    parts = (_ffi.GpxKernPart * 1)()
    keep = []
    _ffi._fill_part(parts[0], ("rbf", False, 0, [0, 1, 2], 1.0, 1.0), keep)
    v = np.ones(N)
    p = v.ctypes.data_as(_ffi._dp)
    d = ctypes.c_double()
    eng = B.Engine()
    L, h = _raw(eng)
    assert L.gpx_laplace_begin(h, parts, 1) == -2                        # no data
    eng.set_data(X, np.hstack([Y, Y]))
    assert L.gpx_laplace_begin(h, parts, 1) == -2                        # P = 2
    eng.set_data(X, Y)
    assert L.gpx_laplace_newton(h, p, p, p, 5, p, p, ctypes.byref(d)) == -2   # no begin
    assert L.gpx_laplace_finish(h, p, p, p, 0, None, 5, ctypes.byref(d), p, p, None, ctypes.byref(d)) == -2
    assert L.gpx_laplace_matvec(h, p, p) == -2
    assert L.gpx_laplace_begin(h, None, 1) == -2
    assert L.gpx_laplace_begin(h, parts, 1) == 0
    assert L.gpx_laplace_newton(h, None, p, p, 5, p, p, ctypes.byref(d)) == -2
    assert L.gpx_laplace_newton(h, p, p, p, 5, p, p, None) == -2
    kg = np.zeros(2)
    assert L.gpx_laplace_finish(h, p, p, p, 1, None, 5, ctypes.byref(d), p, kg.ctypes.data_as(_ffi._dp), p,
                                ctypes.byref(d)) == -2                   # nlik > 0 without the array
    assert L.gpx_laplace_finish(h, p, p, p, 0, None, 5, None, p, kg.ctypes.data_as(_ffi._dp), None,
                                ctypes.byref(d)) == -2
    # a communicator attached: single-GPU only
    uid = ctypes.create_string_buffer(128)
    assert L.gpx_comm_unique_id(uid) == 0
    assert L.gpx_comm_init(h, uid.raw, 0, 1) == 0
    eng.set_data(X, Y)
    assert L.gpx_laplace_begin(h, parts, 1) == -2
    eng.close()


def _sweep_launches(N):
    """launches of the factor-and-invert sweep of an N x N matrix: a gpx_pdinv that returns no matrices on a fresh
    context, less its data binding and load"""
    B = _B()
    from gpy_b200 import _ffi
    eng = B.Engine()
    t0 = eng.total_launches()
    _ffi.pdinv(np.eye(N) * 2.0, want=(), engine=eng)
    return eng.total_launches() - t0 - 2


@pytest.mark.parametrize("N", [300, 700, 1300])
def test_launch_counts_do_not_depend_on_N(N):
    B = _B()
    rng = np.random.default_rng(N)
    X = rng.uniform(-2, 2, size=(N, 3))
    Y = (X[:, :1] > 0).astype(float)
    eng = B.Engine()
    eng.set_data(X, Y)
    eng.laplace_begin([("rbf", True, 0, [0, 1, 2], 1.0, [1.0, 1.2, 0.8]), ("bias", False, 1, [], 0.3, None)])
    assert eng.stats()["launches"] == 2
    F = _sweep_launches(N)
    W = np.full(N, 0.3)
    eng.laplace_newton(W, np.ones(N), np.zeros(N))
    assert eng.stats()["launches"] - F == 11
    eng.laplace_finish(W, np.zeros(N), np.ones(N))
    assert eng.stats()["launches"] - F == 16 + 2


def test_large_case_matches_host_restatement():
    B = _B()
    N = 4096
    rng = np.random.default_rng(9)
    X = rng.uniform(-3, 3, size=(N, 3))
    Y = (np.sin(X[:, :1]) + 0.5 * X[:, 1:2] + 0.3 * rng.standard_normal((N, 1)) > 0).astype(float)
    parts = lo._single("rbf", True)
    kern = mirror_kernel(parts)
    inf = B.Laplace()
    post, lml, gd = inf.inference(kern, X, B.Bernoulli(), Y)
    kern.update_gradients_full(gd["dL_dK"], X)
    r = lo.laplace_eval(X, Y, parts, B.Bernoulli())
    print("N = 4096: lml %.3e rel, grad %.3e, iterations %d / %d" % (
        abs(lml - r["lml"]) / abs(r["lml"]), _rel(kern.gradient, r["grad"]), inf.iterations, r["iterations"]))
    assert inf.iterations == r["iterations"]
    assert abs(lml - r["lml"]) <= 2e-9 * abs(r["lml"])
    assert _rel(kern.gradient, r["grad"]) <= 1e-6
