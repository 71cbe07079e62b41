"""The joint posterior on the device (gpx_posterior_covariance, gpx_posterior_samples, gpx_sparse_posterior_samples): the
covariance between point sets against the NumPy restatement of tests/posterior_samples_oracle.py over N, test-point counts
at the tile edges, kernels and both tensor paths; samples with a given z against mu + chol(Sigma + jitter I) z; the
jitter ladder and the not-PD return; seeded statistics; the sparse model with its shared woodbury_inv; the invariants of
the three entries (untouched posterior, repeatability, rejections, launch counts); and the mirror's model methods end to
end. The reference's own GP over plugin kernels is covered by tests/test_posterior_samples_cpu.py with a test double of
the engine."""
import ctypes

import numpy as np
import pytest

import gpy_b200
import posterior_samples_oracle as pso
import predictive_gradients_oracle as po
import sparse_composite_oracle as so
import wide_composites_oracle as wo
from gpy_b200 import _ffi
from sparse_composite_oracle import CompositeOracle

pytestmark = pytest.mark.gpu


def engine(oz=0):
    e = _ffi.Engine(0)
    e.set_option("ozaki", oz)
    return e


def evaluate(e, parts, X, Y, noise):
    e.set_data(X, Y)
    p = parts[0]
    if len(parts) == 1 and p["kind"] in ("rbf", "exponential", "matern32", "matern52"):
        if np.ndim(noise) > 0:
            return e.exact_eval_het(p["kind"], p.get("ARD", False), p["variance"], p["lengthscale"], noise)
        return e.exact_eval(p["kind"], p.get("ARD", False), p["variance"], p["lengthscale"], noise)
    return e.exact_eval_multi([wo.descriptor(q) for q in parts], noise)


def cov_close(got, want, atol=1e-10):
    """the full-covariance rule of test_gpu_routes.py: rtol 1e-7, atol 1e-10 (1e-6 for Exponential)"""
    assert got.shape == want.shape
    np.testing.assert_allclose(got, want, rtol=1e-7, atol=atol)


def points(M, seed, D=3):
    return np.random.default_rng(seed).uniform(-2.2, 2.2, size=(M, D))


# ---- covariance over N, test-point counts and tensor paths ---------------------------------------------------------------
PAIRS = [(1, 1), (7, 128), (129, 300), (300, 7), (128, 129)]


@pytest.mark.parametrize("oz", [0, 1])
@pytest.mark.parametrize("N", [150, 700, 1300])
def test_covariance_over_N_and_point_counts(N, oz):
    parts = po.KERNELS["matern52_ard"]
    X, Y, _, noise = po.case_data(N, 2, 3, 2, N, False)
    kern = CompositeOracle(parts)
    e = engine(oz)
    evaluate(e, parts, X, Y, noise)
    for M1, M2 in PAIRS:
        X1, X2 = points(M1, M1 + N), points(M2, M2 + 7 * N)
        cov_close(e.posterior_covariance(X1, X2), pso.covariance_between_points(kern, X, noise, X1, X2))
        c1 = e.posterior_covariance(X1)
        cov_close(c1, pso.covariance_between_points(kern, X, noise, X1))
        assert np.array_equal(c1, c1.T)
        cov_close(c1, e.predict(X1, full_cov=True)[1])


SINGLE = [k + s for k in ("rbf", "exponential", "matern32", "matern52") for s in ("_iso", "_ard")]
MIXED = {
    "ratquad_x_periodic": [wo.ratquad([0, 1], 0, True), wo.stdperiodic([1, 2], 0, True, False, variance=0.8),
                           wo.static("white", 1, 0.05)],
    "mauna_loa": [wo.stationary("rbf", [0, 1, 2], 0, False, variance=1.5, scale=2.0),
                  wo.stationary("rbf", [0], 1, False, variance=0.6), wo.stdperiodic([0], 1, False, False),
                  wo.ratquad([1, 2], 2, False, power=0.7, variance=0.4),
                  wo.stationary("rbf", [2], 3, False, variance=0.1, scale=0.3), wo.static("white", 3, 0.02)],
}


@pytest.mark.parametrize("oz", [0, 1])
@pytest.mark.parametrize("kname", SINGLE + ["rbf_bias_white", "m52_x_rbf", "het"] + sorted(MIXED))
def test_covariance_over_kernels(kname, oz):
    het = kname == "het"
    parts = MIXED.get(kname) or po.KERNELS["rbf_ard" if het else kname]
    kern = wo.WideOracle(parts)
    X, Y, _, noise = po.case_data(700, 2, 3, 1, 11, het)
    e = engine(oz)
    evaluate(e, parts, X, Y, noise)
    X1, X2 = points(129, 1), points(7, 2)
    atol = 1e-6 if "exponential" in kname else 1e-10
    cov_close(e.posterior_covariance(X1, X2), pso.covariance_between_points(kern, X, noise, X1, X2), atol)
    cov_close(e.posterior_covariance(X2), pso.covariance_between_points(kern, X, noise, X2), atol)


def test_exponential_at_coincident_points_on_a_dyadic_grid():
    """on a dyadic grid with power-of-two lengthscales r is exact, so coincident points have r = 0 on both sides, and an
    explicit X2 = X1 agrees with the symmetric form"""
    g = np.arange(-8, 8) / 4.0
    X = np.array(np.meshgrid(g, g[::3])).reshape(2, -1).T.copy()
    Y = np.sin(X.sum(1, keepdims=True))
    parts = [dict(kind="exponential", term=0, dims=[0, 1], variance=1.0, lengthscale=[2.0, 0.5], ARD=True)]
    kern = wo.WideOracle(parts)
    e = engine()
    evaluate(e, parts, X, Y, 0.0625)
    X1 = X[::7].copy()
    want = pso.covariance_between_points(kern, X, 0.0625, X1, X1)
    cov_close(e.posterior_covariance(X1, X1.copy()), want)
    cov_close(e.posterior_covariance(X1), want)


# ---- samples ---------------------------------------------------------------------------------------------------------
def exact_reference(kname, N, P, M, seed, het=False):
    parts = MIXED.get(kname) or po.KERNELS[kname]
    kern = wo.WideOracle(parts)
    X, Y, _, noise = po.case_data(N, 2, 3, P, seed, het)
    Xn = points(M, seed + 1)
    mu, Sig = pso.exact_predict_full(kern, X, Y, noise, Xn)
    return parts, X, Y, noise, Xn, mu, Sig


def sample_close(f, f0, Sig, jit):
    cond = np.linalg.cond(Sig + jit * np.eye(Sig.shape[0]))
    assert cond <= 1e6
    tol = max(1e-9, 1e-13 * cond) * max(1.0, np.abs(f0).max())
    assert np.abs(f - f0).max() <= tol, (np.abs(f - f0).max(), tol)


@pytest.mark.parametrize("oz", [0, 1])
@pytest.mark.parametrize("kname,P,M", [("rbf_ard", 1, 40), ("matern32_iso", 3, 129), ("m52_x_rbf", 1, 7),
                                       ("rbf_bias_white", 2, 16), ("mauna_loa", 1, 40), ("het", 1, 16)])
def test_samples_with_a_given_z(kname, P, M, oz):
    het = kname == "het"
    parts, X, Y, noise, Xn, mu, Sig = exact_reference("rbf_ard" if het else kname, 700, P, M, 21, het)
    z = np.random.default_rng(3).standard_normal((P * 5, M))
    e = engine(oz)
    evaluate(e, parts, X, Y, noise)
    f, jit = e.posterior_samples(Xn, z)
    f0, jit0 = pso.samples(mu, Sig, z)
    assert jit == jit0 == 0.0
    sample_close(f, f0, Sig, jit)


def test_square_root_recovered_from_samples():
    """S >= M: L from (f - mu) and z by least squares, L L^T = Sigma"""
    parts, X, Y, noise, Xn, mu, Sig = exact_reference("matern52_ard", 700, 1, 16, 5)
    z = np.random.default_rng(4).standard_normal((64, 16))
    e = engine()
    evaluate(e, parts, X, Y, noise)
    f, jit = e.posterior_samples(Xn, z)
    Lt = np.linalg.lstsq(z, f - mu[:, 0][None, :], rcond=None)[0]
    np.testing.assert_allclose(Lt.T @ Lt, Sig + jit * np.eye(16), rtol=1e-7, atol=1e-10)
    assert np.allclose(np.triu(Lt.T, 1), 0.0, atol=1e-9)


def test_repeated_points_engage_the_jitter_ladder_and_max_tries_zero_is_not_pd():
    parts, X, Y, noise, Xn, mu, Sig = exact_reference("rbf_ard", 700, 1, 9, 8)
    Xr = np.concatenate([Xn, Xn[:4]])
    _, Sr = pso.exact_predict_full(wo.WideOracle(parts), X, Y, noise, Xr)
    e = engine()
    evaluate(e, parts, X, Y, noise)
    z = np.random.default_rng(1).standard_normal((6, Xr.shape[0]))
    f, jit = e.posterior_samples(Xr, z)
    assert jit > 0 and np.isclose(pso.jitter_ladder(Sr), jit, rtol=1e-12, atol=0).any(), jit
    f0 = z.dot(np.linalg.cholesky(Sr + jit * np.eye(13)).T) + mu[[*range(9), 0, 1, 2, 3], 0][None, :]
    assert np.abs(f - f0).max() <= 1e-6
    with pytest.raises(np.linalg.LinAlgError):
        e.posterior_samples(Xr, z, max_tries=0)


def test_seeded_statistics():
    parts, X, Y, noise, Xn, mu, Sig = exact_reference("matern32_iso", 700, 1, 16, 9)
    e = engine()
    evaluate(e, parts, X, Y, noise)
    np.random.seed(12)
    z = pso.standard_normals(16, 1, 20000)
    f, jit = e.posterior_samples(Xn, z)
    assert jit == 0.0
    d = f - f.mean(0)
    C = d.T @ d / (f.shape[0] - 1)
    sd = np.sqrt((np.outer(np.diag(Sig), np.diag(Sig)) + Sig ** 2) / f.shape[0])
    assert np.all(np.abs(C - Sig) <= 5 * sd)
    assert np.all(np.abs(f.mean(0) - mu[:, 0]) <= 5 * np.sqrt(np.diag(Sig) / f.shape[0]))


# ---- sparse ----------------------------------------------------------------------------------------------------------
def spread_points(X, M):
    idx = [0]
    d = np.linalg.norm(X - X[0], axis=1)
    for _ in range(M - 1):
        i = int(np.argmax(d))
        idx.append(i)
        d = np.minimum(d, np.linalg.norm(X - X[i], axis=1))
    return X[idx].copy()


@pytest.mark.parametrize("M", [50, 129, 300])
def test_sparse_samples(M):
    parts = po.KERNELS["m52_x_rbf"]
    kern = CompositeOracle(parts)
    X, Y, _, noise = po.case_data(2000, M, 3, 2, M, False)
    Z = spread_points(X, M)
    wv, wi = po.sparse_posterior(kern, X, Y, Z, noise)
    Xn = points(40, M)
    mu, Sig = pso.sparse_predict_full(wv, wi, kern, Z, Xn)
    z = np.random.default_rng(M).standard_normal((2 * 3, 40))
    e = engine()
    e.sparse_set_data(X, Y)
    e.sparse_eval_multi([so.descriptor(q) for q in parts], Z, noise)
    f, jit = e.sparse_posterior_samples(Xn, z)
    f0, jit0 = pso.samples(mu, Sig, z)
    assert jit == jit0 == 0.0
    sample_close(f, f0, Sig, jit)
    e.sparse_predictive_gradients(Xn)   # reuses the W the samples formed
    assert np.array_equal(e.sparse_posterior_samples(Xn, z)[0], f)
    e2 = engine()
    e2.sparse_set_data(X, Y)
    e2.sparse_eval_multi([so.descriptor(q) for q in parts], Z, noise)
    g = e2.sparse_predictive_gradients(Xn)   # forms W first this time
    assert np.array_equal(e2.sparse_posterior_samples(Xn, z)[0], f)
    assert all(np.array_equal(a, b) for a, b in zip(g, e.sparse_predictive_gradients(Xn)))


# ---- invariants ------------------------------------------------------------------------------------------------------
def snapshot(e, Xn, sparse=False, sharded=False):
    s = {"stats": e.stats(), "predict": e.predict(Xn), "predict_full": e.predict(Xn, full_cov=True)}
    for w in ("L", "alpha") if sharded else ("L", "alpha", "Kinv", "dL_dK", "K", "Linv"):
        s[w] = e.get(w)
    if not sharded:
        s["pg"] = e.predictive_gradients(Xn)
    if sparse:
        for w in ("woodbury_vector", "woodbury_inv", "Kmm", "Lm"):
            s[w] = e.sparse_get(w)
        s["spg"] = e.sparse_predictive_gradients(Xn)
    return s


def same(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(same(a[k], b[k]) for k in a)
    if isinstance(a, (tuple, list)):
        return len(a) == len(b) and all(same(x, y) for x, y in zip(a, b))
    return np.array_equal(np.asarray(a), np.asarray(b))


def raw_call(e, name, *args):
    return getattr(e._L, name)(e._h, *args)


@pytest.mark.parametrize("oz", [0, 1])
def test_nothing_the_posterior_returns_changes(oz):
    parts = po.KERNELS["rbf_ard"]
    X, Y, _, noise = po.case_data(700, 2, 3, 1, 2, False)
    Z = spread_points(X, 60)
    e = engine(oz)
    e.sparse_set_data(X, Y)
    e.sparse_eval_multi([so.descriptor(q) for q in parts], Z, noise)
    evaluate(e, parts, X, Y, noise)
    Xn = points(20, 3)
    z = np.random.default_rng(0).standard_normal((4, 20))
    before = snapshot(e, Xn, sparse=True)
    f1, c1 = e.posterior_samples(Xn, z), e.posterior_covariance(Xn, Xn[:5])
    s1 = e.sparse_posterior_samples(Xn, z)
    assert same(snapshot(e, Xn, sparse=True), before)
    assert same(e.posterior_samples(Xn, z), f1) and same(e.posterior_covariance(Xn, Xn[:5]), c1)
    assert same(e.sparse_posterior_samples(Xn, z), s1)
    Xr = np.concatenate([Xn, Xn])
    with pytest.raises(np.linalg.LinAlgError):   # not PD
        e.posterior_samples(Xr, np.zeros((1, 40)), max_tries=0)
    with pytest.raises(np.linalg.LinAlgError):
        e.sparse_posterior_samples(Xr, np.zeros((1, 40)), max_tries=0)
    assert same(snapshot(e, Xn, sparse=True), before)
    dp = ctypes.POINTER(ctypes.c_double)
    x, zz, out, jit = _ffi._ptr(Xn), _ffi._ptr(z), _ffi._ptr(np.empty(400)), ctypes.byref(ctypes.c_double())
    for name in ("gpx_posterior_samples", "gpx_sparse_posterior_samples"):
        for args in ((x, 0, zz, 4, 5, out, jit), (x, 20, zz, 0, 5, out, jit), (None, 20, zz, 4, 5, out, jit),
                     (x, 20, None, 4, 5, out, jit), (x, 20, zz, 4, 5, dp(), jit), (x, 20, zz, 4, 5, out, None)):
            assert raw_call(e, name, *args) == -2
    assert raw_call(e, "gpx_posterior_covariance", x, 0, None, 0, out) == -2
    assert raw_call(e, "gpx_posterior_covariance", None, 5, None, 0, out) == -2
    assert same(snapshot(e, Xn, sparse=True), before)
    fresh = engine()
    with pytest.raises(_ffi.GpxArgumentError):
        fresh.posterior_covariance(Xn)
    with pytest.raises(_ffi.GpxArgumentError):
        fresh.posterior_samples(Xn, z)
    with pytest.raises(_ffi.GpxArgumentError):
        fresh.sparse_posterior_samples(Xn, z)


def test_a_communicator_is_rejected():
    from test_gpu_sharded_single_rank import attach
    parts = po.KERNELS["rbf_iso"]
    X, Y, _, noise = po.case_data(300, 2, 3, 1, 4, False)
    e = attach(_ffi.Engine(0))
    evaluate(e, parts, X, Y, noise)
    Xn = points(9, 1)
    before = snapshot(e, Xn, sharded=True)
    for call in (lambda: e.posterior_covariance(Xn), lambda: e.posterior_samples(Xn, np.ones((2, 9)))):
        with pytest.raises(_ffi.GpxArgumentError):
            call()
    assert same(snapshot(e, Xn, sharded=True), before)
    e.sparse_set_data(X, Y)
    e.sparse_eval("rbf", False, 1.0, 1.2, spread_points(X, 20), noise)
    with pytest.raises(_ffi.GpxArgumentError):
        e.sparse_posterior_samples(Xn, np.ones((2, 9)))


# ---- launches --------------------------------------------------------------------------------------------------------
def factor_launches(M):
    """what gpx_pdinv of an M x M matrix launches on a context of its own that returns no matrices"""
    e = engine()
    n0 = e.total_launches()
    _ffi.pdinv(np.eye(M) * 2.0, want=(), engine=e)
    return e.total_launches() - n0


@pytest.mark.parametrize("M", [7, 129])
def test_launch_counts(M):
    parts = po.KERNELS["m52_x_rbf"]
    X, Y, _, noise = po.case_data(700, 2, 3, 1, 3, False)
    Xn, z = points(M, 2), np.random.default_rng(2).standard_normal((3, M))
    F = factor_launches(M)
    e = engine()
    evaluate(e, parts, X, Y, noise)
    n0 = e.total_launches()
    e.posterior_covariance(Xn, Xn[:3])
    e.posterior_covariance(Xn)
    assert e.total_launches() - n0 == 14
    n0 = e.total_launches()
    e.posterior_samples(Xn, z)
    assert e.total_launches() - n0 == 13 + F
    e.sparse_set_data(X, Y)
    e.sparse_eval_multi([so.descriptor(q) for q in parts], spread_points(X, 50), noise)
    n0 = e.total_launches()
    e.sparse_posterior_samples(Xn, z)
    assert e.total_launches() - n0 == 12 + 5 + (F - 1)   # the child has bound order M already
    n0 = e.total_launches()
    e.sparse_posterior_samples(Xn, z)
    assert e.total_launches() - n0 == 12 + F - 1


# ---- end to end ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P", [1, 3])
def test_mirror_model_samples(P):
    X, Y, _, _ = po.case_data(500, 2, 3, P, 6, False)
    Y = 3.0 * Y + 1.5
    m = gpy_b200.GPRegression(X, Y, gpy_b200.Matern52(3, ARD=True, lengthscale=[1.0, 1.3, 1.6]), normalizer=True,
                              noise_var=0.05)
    Xn = points(12, 4)
    np.random.seed(5)
    fs = m.posterior_samples_f(Xn, size=7)
    state = np.random.get_state()
    assert fs.shape == (12, P, 7)
    np.random.seed(5)
    z = pso.standard_normals(12, P, 7)
    assert same(np.random.get_state(), state)
    mu, Sig = pso.exact_predict_full(CompositeOracle([dict(kind="matern52", term=0, dims=[0, 1, 2], variance=1.0,
                                                           lengthscale=[1.0, 1.3, 1.6], ARD=True)]),
                                     X, (Y - Y.mean(0)) / Y.std(0), 0.05, Xn)
    f0, _ = pso.samples(mu, Sig, z)
    want = pso.as_fsim(f0, P) * Y.std(0)[None, :, None] + Y.mean(0)[None, :, None]
    np.testing.assert_allclose(fs, want, rtol=1e-8, atol=1e-8)
    np.random.seed(5)
    assert same(m.posterior_samples_f(Xn, size=7), fs)
    np.random.seed(5)
    ys = m.posterior_samples(Xn, size=7)
    assert ys.shape == (12, P, 7) and not np.array_equal(ys, fs)
    np.random.seed(5)
    fs2 = m.posterior_samples_f(Xn, size=7)
    noise = np.random.normal(0.0, np.sqrt(0.05), size=fs2[:, 0].size)
    np.testing.assert_allclose(ys[:, 0], fs2[:, 0] + noise.reshape(12, 7), rtol=1e-12, atol=1e-12)
    cov = m.posterior_covariance_between_points(Xn, Xn)
    assert cov.shape == ((12, 12) if P == 1 else (12, 12, P))

