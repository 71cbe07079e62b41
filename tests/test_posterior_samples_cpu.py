"""The joint posterior without a GPU: the NumPy restatement of tests/posterior_samples_oracle.py against the reference's
own GP / VarDTC posterior (the committed fixtures of tests/golden/posterior_samples), the random stream the mirror's
posterior_samples_f consumes against the reference's, and the mirror's host logic (shapes, normalizer, likelihood noise,
the fallbacks to the reference's host route) on test doubles of the engine that answer from that restatement."""
import glob
import os

import numpy as np
import pytest
from scipy.linalg import solve_triangular

import gpy_b200
import posterior_samples_cases as cases
import posterior_samples_oracle as pso
import predictive_gradients_oracle as po
import wide_composites_oracle as wo
from gpy_b200.inference import HostPosterior, PosteriorExact
from gpy_b200.model import Standardize, draw_standard_normals

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = sorted(glob.glob(os.path.join(HERE, "golden", "posterior_samples", "*.npz")))


def _name(p):
    return os.path.basename(p)[:-4]


def _noise(f):
    n = f["noise"]
    return float(n) if n.ndim == 0 else n


def _normalised(Y):
    Yn, mean, std = po.standardize(Y)
    return Yn, mean, std


def test_fixture_set_covers_the_cases():
    names = {_name(p) for p in FIXTURES}
    assert names == set(cases.CASES)


@pytest.mark.parametrize("path", FIXTURES, ids=_name)
def test_restatement_matches_the_reference_fixtures(path):
    f = np.load(path)
    c = cases.CASES[_name(path)]
    kern = wo.WideOracle(c["parts"])
    X, Y, noise = f["X"], f["Y"], _noise(f)
    norm = bool(c.get("normalizer"))
    Yn, mean, std = _normalised(Y) if norm else (Y, None, None)

    def close(got, want):
        np.testing.assert_allclose(got, want, rtol=0, atol=1e-12 * max(1.0, np.abs(want).max()))

    if c.get("sparse"):
        wv, wi = po.sparse_posterior(kern, X, Y, f["Z"], noise)
        mu, Sig = pso.sparse_predict_full(wv, wi, kern, f["Z"], f["Xnew"])
    else:
        mu, Sig = pso.exact_predict_full(kern, X, Yn, noise, f["Xnew"])
        cov = pso.covariance_between_points(kern, X, noise, f["X1"], f["X2"])
        lik = cov + np.eye(cov.shape[0]) * noise if np.ndim(noise) == 0 else None
        if norm:   # gp.py:779-784
            scale = (lambda v: v[..., None] * std ** 2) if Y.shape[1] > 1 else (lambda v: v * std ** 2)
            cov, lik = scale(cov), scale(lik)
        close(cov, f["cov"])
        if lik is not None:
            close(lik, f["cov_lik"])
    close(mu, f["mu"])
    close(Sig, f["Sigma"])
    if "fsim" not in f.files:   # P > 1 with a normalizer: the reference's inverse_variance does not broadcast (gp.py:614)
        assert norm and Y.shape[1] > 1
        return
    # the reference's draw: per output one standard_normal((size, M)), then numpy's SVD square root (legacy
    # RandomState.multivariate_normal)
    np.random.seed(int(f["seed"]))
    P, S, M = Y.shape[1], int(f["size"]), f["Xnew"].shape[0]
    z = pso.standard_normals(M, P, S)
    st = np.random.get_state()
    assert np.array_equal(st[1], f["rng_key"]) and st[2] == int(f["rng_pos"])
    m, v = (mu * std + mean, f["Sigma"] * std ** 2) if norm else (mu, f["Sigma"])
    _, s, vh = np.linalg.svd(v)
    root = np.sqrt(s)[:, None] * vh
    for d in range(P):
        close((z[d * S:(d + 1) * S] @ root + m[:, d]).T, f["fsim"][:, d, :])


# ---- test doubles ----------------------------------------------------------------------------------------------------
@pytest.fixture
def host_kernels(monkeypatch):
    """the mirror kernels' stand-alone calls answered by the oracle"""
    from gpy_b200 import _ffi
    from oracle import gpy_oracle as o
    monkeypatch.setattr(_ffi, "kern_K", lambda kind, ARD, v, ls, X, X2=None:
                        o.StationaryOracle(kind, X.shape[1], v, ls, ARD).K(X, X2))
    monkeypatch.setattr(_ffi, "kern_Kdiag", lambda kind, v, N: np.full(N, v))


class JointEngine(object):
    """test double of gpy_b200._ffi.Engine for one exact posterior of a WideOracle kernel over the engine's columns"""

    def __init__(self, parts, X, Y, noise):
        self.kern, self.X, self.noise = wo.WideOracle(parts), X, noise
        self.L = pso.exact_factor(self.kern, X, noise)
        self.alpha = pso.cho_solve_sym(self.L @ self.L.T, Y)
        self.Y, self.eval_serial, self.calls = Y, 1, []

    def get(self, which):
        self.calls.append(which)
        return {"L": self.L, "alpha": self.alpha}[which]

    def predict(self, Xnew, full_cov=False):
        self.calls.append("predict")
        mu, Sig = pso.exact_predict_full(self.kern, self.X, self.Y, self.noise, Xnew)
        return mu, (Sig if full_cov else np.diag(Sig)[:, None])

    def posterior_covariance(self, X1, X2=None):
        self.calls.append("posterior_covariance")
        return pso.covariance_between_points(self.kern, self.X, self.noise, X1, X2)

    def posterior_samples(self, Xnew, z, max_tries=5):
        self.calls.append("posterior_samples")
        mu, Sig = pso.exact_predict_full(self.kern, self.X, self.Y, self.noise, Xnew)
        return pso.samples(mu, Sig, z, max_tries)


PARTS = [dict(kind="matern52", term=0, dims=[0, 1, 2], variance=1.0, lengthscale=[1.0, 1.3, 1.6], ARD=True)]


def _kern():
    return gpy_b200.Matern52(3, variance=1.0, lengthscale=[1.0, 1.3, 1.6], ARD=True)


def _model(P=1, normalizer=False, noise=0.05, N=60, seed=3):
    """a GPRegression whose posterior is a device posterior over JointEngine (no evaluation runs)"""
    X, Y, _, _ = po.case_data(N, 2, 3, P, seed, False)
    Y = 2.0 * Y + 0.5
    m = gpy_b200.GPRegression.__new__(gpy_b200.GPRegression)
    m.kern, m.X, m.Y, m.output_dim, m.mean_function = _kern(), X, Y, P, None
    m.likelihood = gpy_b200.Gaussian(variance=noise)
    m.normalizer = Standardize() if normalizer else None
    Yn = Y
    if normalizer:
        m.normalizer.scale_by(Y)
        Yn = m.normalizer.normalize(Y)
    eng = JointEngine(PARTS, X, Yn, noise)
    m.posterior = PosteriorExact(eng, N, P, m.kern._state_key())
    return m, eng


def _xnew(M=6, seed=4):
    return np.random.default_rng(seed).uniform(-2, 2, size=(M, 3))


@pytest.mark.parametrize("P", [1, 3])
@pytest.mark.parametrize("normalizer", [False, True])
def test_device_route_shapes_stream_and_normalizer(P, normalizer):
    m, eng = _model(P, normalizer)
    Xn = _xnew()
    np.random.seed(7)
    fs = m.posterior_samples_f(Xn, size=4)
    after = np.random.get_state()
    assert fs.shape == (6, P, 4) and eng.calls == ["posterior_samples"]
    np.random.seed(7)
    for _ in range(P):   # what np.random.multivariate_normal(m, v, 4) consumes per output
        np.random.standard_normal((4, 6))
    st = np.random.get_state()
    assert np.array_equal(st[1], after[1]) and st[2] == after[2]
    np.random.seed(7)
    z = draw_standard_normals(6, P, 4)
    f, _ = eng.posterior_samples(Xn, z)
    want = pso.as_fsim(f, P)
    if normalizer:
        want = want * m.normalizer.std[None, :, None] + m.normalizer.mean[None, :, None]
    np.testing.assert_array_equal(fs, want)


def test_mirror_draw_leaves_the_rng_where_the_reference_does():
    """the reference's posterior_samples_f consumed the stream recorded in the fixture; the mirror's draw ends there too"""
    f = np.load(os.path.join(HERE, "golden", "posterior_samples", "exact_rbf_ard.npz"))
    c = cases.CASES["exact_rbf_ard"]
    m, _ = _model()
    m.X, m.Y = f["X"], f["Y"]
    m.kern = gpy_b200.RBF(3, variance=0.9, lengthscale=c["parts"][0]["lengthscale"], ARD=True)
    eng = JointEngine(c["parts"], f["X"], f["Y"], float(f["noise"]))
    m.posterior = PosteriorExact(eng, f["X"].shape[0], 1, m.kern._state_key())
    np.random.seed(int(f["seed"]))
    fs = m.posterior_samples_f(f["Xnew"], size=int(f["size"]))
    st = np.random.get_state()
    assert np.array_equal(st[1], f["rng_key"]) and st[2] == int(f["rng_pos"])
    # same distribution, other square root: the sample means over the draws agree only loosely; the stream is the point
    assert fs.shape == f["fsim"].shape


def test_posterior_samples_adds_the_gaussian_noise_per_entry():
    m, _ = _model(P=2)
    Xn = _xnew()
    np.random.seed(3)
    ys = m.posterior_samples(Xn, size=5)
    np.random.seed(3)
    fs = m.posterior_samples_f(Xn, size=5)
    want = fs.copy()
    for d in range(2):   # gaussian.py:316-327, one np.random.normal(f_j, sqrt(variance), size=1) per entry
        want[:, d] = np.array([np.random.normal(v, scale=np.sqrt(0.05), size=1) for v in fs[:, d].flatten()]).reshape(6, 5)
    np.testing.assert_array_equal(ys, want)


def test_heteroscedastic_samples_fail_like_the_reference():
    lik = gpy_b200.HeteroscedasticGaussian({"output_index": np.arange(4)[:, None]}, variance=0.1)
    with pytest.raises(ValueError):
        lik.samples(np.zeros((3, 2)))


def test_mixed_noise_samples_restate_the_reference_loop():
    liks = [gpy_b200.Gaussian(variance=0.1), gpy_b200.Gaussian(variance=0.4)]
    mix = gpy_b200.inference.MixedNoise(liks)
    gp = np.arange(12.0).reshape(6, 2)
    meta = {"output_index": np.array([1, 0, 1, 1, 0, 0])[:, None]}
    np.random.seed(9)
    got = mix.samples(gp, meta)
    np.random.seed(9)
    want = np.zeros((6, 2))
    ind = meta["output_index"].flatten()
    for j in np.unique(ind):   # mixed_noise.py:72-82
        flt = ind == j
        g = gp[flt, :]
        want[flt, :] = np.array([np.random.normal(v, scale=np.sqrt(liks[j].variance[0]), size=1)
                                 for v in g.flatten()]).reshape(g.shape[0], 2)
    np.testing.assert_array_equal(got, want)


def test_covariance_between_points_on_the_device_with_likelihood_and_normalizer():
    m, eng = _model(P=1, normalizer=True)
    X1, X2 = _xnew(5, 1), _xnew(5, 2)
    cov = m.posterior_covariance_between_points(X1, X2)
    assert eng.calls.count("posterior_covariance") == 1 and "L" not in eng.calls
    raw = pso.covariance_between_points(eng.kern, m.X, 0.05, X1, X2)
    np.testing.assert_allclose(cov, (raw + 0.05 * np.eye(5)) * m.normalizer.std ** 2, rtol=1e-14, atol=0)
    m3, _ = _model(P=3, normalizer=True)
    c3 = m3.posterior_covariance_between_points(X1, X2, include_likelihood=False)
    assert c3.shape == (5, 5, 3)


def test_foreign_kernel_takes_the_host_route(host_kernels):
    m, eng = _model()
    other = gpy_b200.RBF(3, variance=0.7, lengthscale=1.1)
    Xn = _xnew()
    np.random.seed(2)
    fs = m.posterior_samples_f(Xn, size=3, kern=other)
    assert "posterior_samples" not in eng.calls and "L" in eng.calls
    np.random.seed(2)
    ko = wo.WideOracle([dict(kind="rbf", term=0, dims=[0, 1, 2], variance=0.7, lengthscale=1.1, ARD=False)])
    tmp = solve_triangular(eng.L, ko.K(m.X, Xn), lower=True)
    mu, v = ko.K(m.X, Xn).T @ eng.alpha, ko.K(Xn) - tmp.T @ tmp
    want = np.random.multivariate_normal(mu[:, 0], v, 3).T[:, None, :]
    np.testing.assert_allclose(fs, want, rtol=1e-10, atol=1e-12)
    c = m.posterior.covariance_between_points(other, m.X, Xn, Xn[:2])
    assert "posterior_covariance" not in eng.calls
    np.testing.assert_allclose(c, HostPosterior(eng.L, eng.alpha, None).covariance_between_points(other, m.X, Xn, Xn[:2]))


def test_sharded_engine_takes_the_host_route(host_kernels):
    m, eng = _model()
    eng.sharded = True
    Xn = _xnew()
    m.posterior_samples_f(Xn, size=2)
    m.posterior_covariance_between_points(Xn, Xn, include_likelihood=False)
    assert "posterior_samples" not in eng.calls and "posterior_covariance" not in eng.calls


def test_generic_inference_path_covariance_is_the_reference_formula():
    X, Y, _, _ = po.case_data(40, 2, 3, 1, 5, False)
    ko = wo.WideOracle(PARTS)
    L = pso.exact_factor(ko, X, 0.1)
    X1, X2 = _xnew(4, 1), _xnew(3, 2)
    got = HostPosterior(L, None, None).covariance_between_points(ko, X, X1, X2)
    np.testing.assert_allclose(got, pso.covariance_between_points(ko, X, 0.1, X1, X2), rtol=1e-13, atol=1e-15)


def test_reference_gp_over_plugin_kernels_lands_on_the_device():
    """the reference's own GP.posterior_covariance_between_points (gp.py:735-786) over plugin B.RBF and B.Add: one
    posterior_covariance engine call, the stock model's numbers"""
    if not os.path.isdir(os.environ.get("GPX_REFERENCE", "/root/reference") + "/GPy"):
        pytest.skip("reference tree not present")
    from test_host_model_cpu import FakeEngine as MultiFakeEngine
    from test_gpy_plugin_cpu import fake_ffi
    from oracle import gpy_oracle as o
    from oracle import ref_gpy
    from gpy_b200 import gpy_plugin

    class Engine(MultiFakeEngine):
        def posterior_covariance(self, X1, X2=None):
            self.calls.append("posterior_covariance")
            K = (lambda A, B=None: o.composite_K(self.res["kparts"], A, B)) if self.theta is None else \
                o.StationaryOracle(self.theta[0], self.X.shape[1], self.theta[2], self.theta[3], self.theta[1]).K
            t1 = solve_triangular(self.res["L"], K(self.X, X1), lower=True)
            t2 = solve_triangular(self.res["L"], K(self.X, X2), lower=True)
            return K(X1, X2) - t1.T @ t2

    M = ref_gpy.load_models()
    C = ref_gpy.load_combination()
    G = M.G
    ffi = fake_ffi()
    ffi.Engine = Engine
    B = gpy_plugin.make(G.RBF, G.Exponential, G.Matern32, G.Matern52, G.ExactGaussianInference, ffi=ffi, Add=C.Add,
                        Prod=C.Prod)
    X, Y = o.synthetic(80, 3, seed=2)
    X1, X2 = _xnew(5, 1), _xnew(4, 2)
    for build in (lambda K: K.RBF(3, variance=1.2, lengthscale=1.1),
                  lambda K: (B.Add if K is B else C.Add)([K.RBF(3, variance=1.2, lengthscale=1.1),
                                                          K.Matern32(3, variance=0.5, lengthscale=2.0)])):
        stock = M.GPRegression(X, Y, build(G), noise_var=0.1)
        plug = M.GPRegression(X, Y, build(B), noise_var=0.1)
        plug.inference_method = B.ExactGaussianInference()
        plug.parameters_changed()
        eng = plug.inference_method.engine
        n = len(eng.calls)
        got = plug.posterior_covariance_between_points(X1, X2, include_likelihood=False)
        assert eng.calls[n:] == ["posterior_covariance"]
        np.testing.assert_allclose(got, stock.posterior_covariance_between_points(X1, X2, include_likelihood=False),
                                   rtol=1e-9, atol=1e-12)
