"""SVGP on the device (gpx_svgp_begin / gpx_svgp_finish, gpy_b200.SVGP) against the NumPy restatement of
tests/svgp_oracle.py, which tests/test_svgp_cpu.py pins to the reference's own SVGP.inference.

Bars: the device forms Kmm^-1 Kmn by triangular products with Lm^-1 and sums in other orders than LAPACK, so the
deviation grows with the condition number of the matrix jitchol factored, cond(Kmm + jitter I); dL_dchol and the KL term
carry S = q_L q_L^T, so they grow with cond(S) as well. Against the restatement every comparison uses
rel <= 1e-14 max(cond(Kmm + jitter I), cond(S), 1e3): 1e-11 at well-conditioned cases, 1e-10 at cond = 1e4. Against the
reference's fixtures (tests/golden/svgp) the bars of tests/test_svgp_cpu.py hold, and the jitter the device's ladder
added must be the restatement's."""
import ctypes
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), HERE]

import svgp_oracle as so  # noqa: E402
import gpy_b200  # noqa: E402
from gpy_b200 import _ffi  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    return _ffi.Engine(0)


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300)


GOLDEN = os.path.join(HERE, "golden", "svgp")


def _bar(o):
    bar = 1e-14 * max(o["cond_Kmm_jit"], o["cond_S"], 1e3)
    assert bar <= 1e-6, "the case must stay well-conditioned enough to test something"
    return bar


def _gbar(bar, cond):
    """the kernel gradient, dL/dZ, woodbury_inv and the predictive variance read Kmm^-1 S Kmm^-1, a second factor of
    Kmm^-1, so their rounding grows as cond^2 once cond is large: max(100 bar, 1e-18 cond^2) (the second term takes over
    above cond = 1e4; the ladder case, cond(Kmm + jitter I) = 8.8e6, measures 1.5e-5 on the gradient and 6e-5 on the
    variance)"""
    return max(100 * bar, 1e-18 * cond * cond)


def _same_jitter(d, o, Kdiag):
    assert abs(d["jit"] - o["jitter"]) <= 1e-12 * Kdiag


def device_eval(eng, parts, X, Y, Z, q_m, q_L, lik, batch_scale=1.0, row0=0, nb=None):
    nb = X.shape[0] - row0 if nb is None else nb
    mu, v, KL, jit = eng.svgp_begin([so.descriptor(p) for p in parts], Z, q_m, q_L, row0, nb)
    Yb = Y[row0:row0 + nb]
    F, dmu, dv, dth = lik.variational_expectations(Yb, mu[:, None], v[:, None])
    grad, dZ, dm, dchol = eng.svgp_finish(dmu[:, 0] * batch_scale, dv[:, 0] * batch_scale)
    return dict(lml=F.sum() * batch_scale - KL, grad=grad, dZ=dZ, dL_dm=dm, dL_dchol=dchol, mu=mu, v=v, KL=KL, jit=jit)


@pytest.mark.parametrize("name", sorted(so.CASES))
def test_cases_match_restatement(eng, name):
    parts, lik_spec, N, M, seed, opts = so.CASES[name]
    X, Y, Z, q_m, q_L, Xnew, bs = so.case_data(name)
    lik = so.make_likelihood(lik_spec, gpy_b200)
    o = so.svgp_eval(parts, X, Y, Z, q_m, q_L, lik, bs, Xnew)
    eng.sparse_set_data(X, Y)
    d = device_eval(eng, parts, X, Y, Z, q_m, q_L, lik, bs)
    _same_jitter(d, o, parts[0]["variance"])
    bar = _bar(o)
    assert abs(d["lml"] - o["lml"]) <= bar * max(abs(o["lml"]), 1.0)
    for k in ("mu", "v", "dL_dm", "dL_dchol"):
        assert _rel(d[k], o[k]) <= bar, (k, _rel(d[k], o[k]), bar)
    for k in ("grad", "dZ"):
        assert _rel(d[k], o[k]) <= _gbar(bar, o["cond_Kmm_jit"]), (k, _rel(d[k], o[k]), bar)
    # the reference's own numbers (tests/golden/make_svgp.py), with the bars of tests/test_svgp_cpu.py
    f = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
    rbar = 1e-13 * max(float(f["cond_Kmm_jit"]), 1e2)
    assert abs(d["lml"] - float(f["lml"])) <= rbar * max(abs(float(f["lml"])), 1.0)
    for k in ("mu", "v", "dL_dm"):
        assert _rel(d[k], f[k]) <= rbar, (k, _rel(d[k], f[k]), rbar)
    for k in ("grad", "dZ"):
        assert _rel(d[k], f[k]) <= _gbar(10 * rbar, float(f["cond_Kmm_jit"])), (k, _rel(d[k], f[k]), rbar)
    assert np.max(np.abs(d["dL_dchol"][np.tril_indices(M)] - f["dL_dchol"])) <= \
        1e-13 * max(float(f["cond_Kmm_jit"]), float(f["cond_S"]), 1e2) * max(np.max(np.abs(f["dL_dchol"])), 1.0)
    pm, pv = eng.sparse_predict(Xnew)
    # the variance reads woodbury_inv = Kmm^-1 - Kmm^-1 S Kmm^-1, whose terms carry cond^2 and cancel: _gbar
    assert _rel(pm[:, 0], f["pmu"]) <= rbar and _rel(pv[:, 0], f["pvar"]) <= _gbar(rbar, float(f["cond_Kmm_jit"]))
    assert _rel(eng.sparse_get("woodbury_vector")[:, 0], o["wv"]) <= bar
    assert _rel(eng.sparse_get("woodbury_inv"), o["wi"]) <= _gbar(bar, o["cond_Kmm_jit"])
    pm, pv = eng.sparse_predict(Xnew)
    assert _rel(pm[:, 0], o["pmu"]) <= bar
    assert _rel(pv[:, 0], o["pvar"]) <= _gbar(bar, o["cond_Kmm_jit"])


@pytest.mark.parametrize("nb,M,row0", [(1, 7, 5), (127, 1, 0), (129, 33, 3), (300, 300, 11), (700, 129, 0),
                                       (513, 64, 187)])
def test_edge_shapes_on_resident_data(eng, nb, M, row0):
    rng = np.random.default_rng(nb * 1000 + M)
    N = 900
    X = rng.uniform(-2, 2, (N, 3))
    Y = (rng.standard_normal((N, 1)) > 0).astype(float)
    Z = rng.uniform(-2, 2, (M, 3))
    q_m, q_L = so.random_q(M, nb + M)
    parts = [dict(kind="matern52", term=0, dims=[0, 1, 2], variance=1.4, lengthscale=[0.3, 0.35, 0.4], ARD=True)]
    lik = gpy_b200.Bernoulli()
    bs = N / float(nb)
    eng.sparse_set_data(X, Y)
    d = device_eval(eng, parts, X, Y, Z, q_m, q_L, lik, bs, row0, nb)
    o = so.svgp_eval(parts, X[row0:row0 + nb], Y[row0:row0 + nb], Z, q_m, q_L, lik, bs)
    _same_jitter(d, o, 1.4)
    bar = _bar(o)
    assert abs(d["lml"] - o["lml"]) <= bar * max(abs(o["lml"]), 1.0)
    for k in ("mu", "v", "dL_dm", "dL_dchol"):
        assert _rel(d[k], o[k]) <= bar, (k, _rel(d[k], o[k]), bar)
    for k in ("grad", "dZ"):
        assert _rel(d[k], o[k]) <= _gbar(bar, o["cond_Kmm_jit"]), (k, _rel(d[k], o[k]), bar)


def test_large_batch(eng):
    """Nb = 16384 and M = 1024 on resident data of 65536 rows"""
    rng = np.random.default_rng(5)
    N, M, nb, row0 = 65536, 1024, 16384, 20000
    X = rng.uniform(-2, 2, (N, 3))
    Y = (np.sin(2 * X[:, :1]) + 0.3 * rng.standard_normal((N, 1)) > 0).astype(float)
    Z = rng.uniform(-2, 2, (M, 3))
    q_m, q_L = so.random_q(M, 9, scale=0.02)
    # lengthscales short enough for 1024 inducing points in the cube to keep Kmm well-conditioned (checked by _bar)
    parts = [dict(kind="rbf", term=0, dims=[0, 1, 2], variance=1.0, lengthscale=[0.12, 0.14, 0.16], ARD=True)]
    lik = gpy_b200.Bernoulli()
    eng.sparse_set_data(X, Y)
    d = device_eval(eng, parts, X, Y, Z, q_m, q_L, lik, N / nb, row0, nb)
    o = so.svgp_eval(parts, X[row0:row0 + nb], Y[row0:row0 + nb], Z, q_m, q_L, lik, N / nb)
    _same_jitter(d, o, 1.0)
    bar = _bar(o)
    assert abs(d["lml"] - o["lml"]) <= bar * max(abs(o["lml"]), 1.0)
    for k in ("mu", "v", "dL_dm", "dL_dchol"):
        assert _rel(d[k], o[k]) <= bar, (k, _rel(d[k], o[k]), bar)
    for k in ("grad", "dZ"):
        assert _rel(d[k], o[k]) <= _gbar(bar, o["cond_Kmm_jit"]), (k, _rel(d[k], o[k]), bar)


def test_launch_counts_do_not_depend_on_nb(eng):
    rng = np.random.default_rng(3)
    X = rng.uniform(-2, 2, (2000, 3))
    Y = (rng.standard_normal((2000, 1)) > 0).astype(float)
    Z = rng.uniform(-2, 2, (50, 3))
    q_m, q_L = so.random_q(50, 3)
    eng.sparse_set_data(X, Y)
    counts = []
    for parts in (so._single("rbf", True), so.COMPOSITE):
        device_eval(eng, parts, X, Y, Z, q_m, q_L, gpy_b200.Bernoulli(), 1.0, 0, 100)   # first-use set-up of the factor
        per = []
        for nb in (100, 1000, 2000):
            l0 = eng.total_launches()
            device_eval(eng, parts, X, Y, Z, q_m, q_L, gpy_b200.Bernoulli(), 1.0, 0, nb)
            per.append(eng.total_launches() - l0)
        assert len(set(per)) == 1, per
        counts.append(per[0])
    assert counts[0] < counts[1]


def _model(lik, N=120, M=15, seed=0, batchsize=None):
    rng = np.random.default_rng(seed)
    X = rng.uniform(-2, 2, (N, 3))
    f = np.sin(1.3 * X[:, :1]) + 0.5 * X[:, 1:2]
    Y = (f + 0.3 * rng.standard_normal((N, 1)) > 0).astype(float) if isinstance(lik, gpy_b200.Bernoulli) else \
        f + 0.2 * rng.standard_normal((N, 1))
    Z = rng.uniform(-2, 2, (M, 3))
    m = gpy_b200.SVGP(X, Y, Z, gpy_b200.RBF(3, ARD=True), lik, batchsize=batchsize, seed=seed)
    q_m, q_L = so.random_q(M, seed + 1)
    m.m.values[:, 0] = q_m
    m.chol.values[:, 0] = q_L[np.tril_indices(M)]
    m.parameters_changed()
    return m


def test_checkgrad_gaussian():
    """the Gaussian likelihood's expectations are exact: every parameter (theta, Z, the noise variance, q_u_chol,
    q_u_mean) passes finite differences"""
    m = _model(gpy_b200.Gaussian(variance=0.3))
    assert m.checkgrad(step=1e-5, tolerance=1e-4)


def test_checkgrad_studentt_likelihood_and_mean():
    """StudentT's expectations use the 20-point Gauss-Hermite rule (likelihood.py:358-411). dF_dmu and dF_dtheta are the
    exact derivatives of that rule's F (its grid does not move with m's shift or theta), but dF_dv (E[d2logp]/2, Price's
    theorem) is not, so the reference's gradient of everything that moves v differs from finite differences of its own
    bound by the quadrature error (tests/test_svgp_cpu.py shows it). The likelihood's parameters and q_u_mean are checked
    at 1e-4; theta, Z and q_u_chol at 5e-2, the size of that quadrature error on this case."""
    m = _model(gpy_b200.StudentT(deg_free=5.0, sigma2=1.0))
    x = m.optimizer_array.copy()
    m.optimizer_array = x
    g = m._grads_transformed()
    sizes = [p.size for p in m._flat()]
    names = [p.name for p in m._flat()]
    starts = np.cumsum([0] + sizes)
    idx = np.concatenate([np.arange(starts[i], starts[i + 1]) for i, n in enumerate(names)
                          if n in ("t_scale2", "deg_free", "q_u_mean")])
    assert idx.size == 2 + m.num_inducing
    for i in idx:
        xp, xm = x.copy(), x.copy()
        xp[i] += 1e-5
        xm[i] -= 1e-5
        m.optimizer_array = xp
        fp = m.objective_function()
        m.optimizer_array = xm
        fm = m.objective_function()
        num = (fp - fm) / 2e-5
        assert abs(num - g[i]) <= 1e-4 * max(abs(num), 1e-2), (names, i, num, g[i])
    m.optimizer_array = x
    assert m.checkgrad(step=1e-5, tolerance=5e-2)


def test_adam_over_minibatches_raises_the_full_bound():
    rng = np.random.default_rng(11)
    N, M = 4000, 30
    X = rng.uniform(-2, 2, (N, 3))
    Y = (np.sin(1.5 * X[:, :1]) + 0.3 * rng.standard_normal((N, 1)) > 0).astype(float)
    Z = X[rng.choice(N, M, replace=False)].copy()
    m = gpy_b200.SVGP(X, Y, Z, gpy_b200.RBF(3, ARD=True), gpy_b200.Bernoulli(), batchsize=400, seed=1)

    def full_bound():
        r, n = m._row0, m._nb
        m.set_data(0, N)
        m.parameters_changed()
        b = m.log_likelihood()
        m.set_data(r, n)
        return b

    b0 = full_bound()
    x = m.optimizer_array.copy()
    mom, vel = np.zeros_like(x), np.zeros_like(x)
    for t in range(1, 151):   # Adam on the negative bound
        g = m.stochastic_grad(x)
        mom = 0.9 * mom + 0.1 * g
        vel = 0.999 * vel + 0.001 * g * g
        x = x - 0.02 * (mom / (1 - 0.9 ** t)) / (np.sqrt(vel / (1 - 0.999 ** t)) + 1e-8)
    m.optimizer_array = x
    assert full_bound() > b0 + 0.05 * abs(b0)


def test_posterior_consumers_match_restatement():
    m = _model(gpy_b200.Bernoulli(), N=200, M=25, seed=4)
    parts = [dict(kind="rbf", term=0, dims=[0, 1, 2], variance=float(m.kern.variance.values[0]),
                  lengthscale=list(m.kern.lengthscale.values), ARD=True)]
    M = 25
    o = so.svgp_eval(parts, m.X_all, m.Y_all, m.Z.values, m.m.values[:, 0], so.flat_to_triang(m.chol.values[:, 0], M),
                     gpy_b200.Bernoulli(), 1.0, np.random.default_rng(2).uniform(-2.5, 2.5, (31, 3)))
    Xnew = np.random.default_rng(2).uniform(-2.5, 2.5, (31, 3))
    mu, var = m.predict_noiseless(Xnew)
    bar = _bar(o)
    assert _rel(mu[:, 0], o["pmu"]) <= bar and _rel(var[:, 0], o["pvar"]) <= bar
    # predictive gradients by the reference's formula (gp.py:438-474) on the restatement's posterior
    kern = so.CompositeOracle(parts)
    dmu, dvar = m.predictive_gradients(Xnew)
    Z = m.Z.values
    eps = 1e-6
    for d in range(3):
        Xp, Xm = Xnew.copy(), Xnew.copy()
        Xp[:, d] += eps
        Xm[:, d] -= eps
        fd = (kern.K(Z, Xp).T.dot(o["wv"]) - kern.K(Z, Xm).T.dot(o["wv"])) / (2 * eps)
        assert _rel(dmu[:, d, 0], fd) <= 1e-6

        def pvar(A):
            Kx = kern.K(Z, A)
            return kern.Kdiag(A) - np.sum(np.dot(o["wi"].T, Kx) * Kx, 0)
        assert _rel(dvar[:, d], (pvar(Xp) - pvar(Xm)) / (2 * eps)) <= 1e-6
    np.random.seed(3)
    f = m.posterior_samples_f(Xnew, size=4000)
    assert np.max(np.abs(f.mean(axis=2)[:, 0] - o["pmu"])) <= 0.1


def test_rejections_leave_the_posterior(eng):
    rng = np.random.default_rng(8)
    X = rng.uniform(-2, 2, (100, 3))
    Y = (rng.standard_normal((100, 1)) > 0).astype(float)
    Z = rng.uniform(-2, 2, (10, 3))
    q_m, q_L = so.random_q(10, 8)
    parts = [so.descriptor(p) for p in so._single("rbf", True)]
    eng.sparse_set_data(X, Y)
    device_eval(eng, so._single("rbf", True), X, Y, Z, q_m, q_L, gpy_b200.Bernoulli())
    wv = eng.sparse_get("woodbury_vector").copy()
    for row0, nb in ((-1, 10), (95, 10), (0, 0), (0, 101)):
        with pytest.raises(_ffi.GpxArgumentError):
            eng.svgp_begin(parts, Z, q_m, q_L, row0, nb)
    with pytest.raises(_ffi.GpxArgumentError):
        eng.svgp_begin([("ratquad", False, 0, [0, 1, 2], 1.0, 1.0, {"power": 2.0})], Z, q_m, q_L, 0, 10)
    with pytest.raises(_ffi.GpxArgumentError):
        eng.svgp_begin(parts, Z[:0], q_m[:0], q_L[:0, :0], 0, 10)
    L = _ffi.lib()
    dp = ctypes.POINTER(ctypes.c_double)
    assert L.gpx_svgp_begin(eng._h, None, 1, None, 10, None, None, 0, 10, 5, None, None, None, None) == -2
    assert L.gpx_svgp_finish(eng._h, None, None, None, None, None, None) == -2
    assert np.array_equal(eng.sparse_get("woodbury_vector"), wv)
    # P != 1, and a finish without a begin on the current data
    eng.sparse_set_data(X, np.hstack([Y, Y]))
    with pytest.raises(_ffi.GpxArgumentError):
        eng.svgp_begin(parts, Z, q_m, q_L, 0, 10)
    eng.sparse_set_data(X, Y)
    z = np.zeros(10)
    g, dZ, dm, dc = np.zeros(4), np.zeros((10, 3)), np.zeros(10), np.zeros((10, 10))
    assert L.gpx_svgp_finish(eng._h, z.ctypes.data_as(dp), z.ctypes.data_as(dp), g.ctypes.data_as(dp),
                             dZ.ctypes.data_as(dp), dm.ctypes.data_as(dp), dc.ctypes.data_as(dp)) == -2


def test_zero_diagonal_gives_minus_inf(eng):
    """the reference's bound with a zero on q_u_chol's diagonal (tests/golden/svgp/bernoulli_zero_diag.npz): -inf, no
    exception; the mirror and the device return the same"""
    f = dict(np.load(os.path.join(GOLDEN, "bernoulli_zero_diag.npz")))
    X, Y, Z, q_m, q_L, Xnew, bs = so.case_data("bernoulli_rbf_iso")
    q_L[3, 3] = 0.0
    inf = gpy_b200.SVGPInference(engine=eng)
    with np.errstate(divide="ignore", invalid="ignore"):
        _, lml, _ = inf.inference(q_m[:, None], q_L[np.tril_indices(q_L.shape[0])][:, None], gpy_b200.RBF(3, variance=1.4,
                                  lengthscale=1.1), X, Z, gpy_b200.Bernoulli(), Y)
    assert lml == float(f["lml"]) == -np.inf
