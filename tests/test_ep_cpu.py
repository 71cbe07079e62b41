"""Expectation propagation without a GPU: the NumPy restatement against the reference's fixtures, the blocked sweep
against the rank-1 chain, the Cody moments against the reference's Bernoulli, and the mirror's rejections."""
import glob
import importlib
import os

import numpy as np
import pytest

import ep_oracle as eo

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = sorted(glob.glob(os.path.join(HERE, "golden", "ep", "*.npz")))
KEYS = ("grad", "tau_tilde", "v_tilde", "cav_tau", "cav_v", "mu", "var")


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[:-4])
def test_oracle_matches_reference_fixture(path):
    """the restatement calls LAPACK as GPy's util/linalg.py does and meets the reference to rounding, with the same
    sweeps and the same draws from numpy's global generator"""
    name = os.path.basename(path)[:-4]
    z = np.load(path)
    r = eo.case_eval(name)
    np.testing.assert_array_equal(r["sweeps"], z["sweeps"])
    assert r["next_random"] == z["next_random"]
    assert abs(r["lml"] - z["lml"]) <= 1e-12 * max(1.0, abs(z["lml"]))
    assert abs(r["log_Z_tilde"] - z["log_Z_tilde"]) <= 1e-12 * max(1.0, abs(z["log_Z_tilde"]))
    for k in KEYS:
        np.testing.assert_allclose(r[k], z[k], rtol=0, atol=1e-12 * max(1.0, float(np.abs(z[k]).max())), err_msg=k)
    if "woodbury_inv" in z:
        np.testing.assert_allclose(r["woodbury_inv"], z["woodbury_inv"], rtol=0,
                                   atol=1e-12 * max(1.0, float(np.abs(z["woodbury_inv"]).max())))


@pytest.mark.parametrize("name", ["rbf_ard_n150", "matern32_iso_n333", "matern52_iso_damped_n150"])
def test_blocked_sweep_matches_the_rank1_chain(name):
    a, b = eo.case_eval(name), eo.case_eval(name, blocked=True)
    np.testing.assert_array_equal(a["sweeps"], b["sweeps"])
    assert abs(a["lml"] - b["lml"]) <= 1e-11 * max(1.0, abs(a["lml"]))
    for k in KEYS:
        np.testing.assert_allclose(b[k], a[k], rtol=0, atol=1e-10 * max(1.0, float(np.abs(a[k]).max())), err_msg=k)


def _ref_bernoulli():
    try:
        from oracle import ref_gpy
        ref_gpy.load()
    except ImportError:
        pytest.skip("reference tree not present")
    return importlib.import_module("GPy.likelihoods.bernoulli").Bernoulli()


def test_cody_moments_match_the_reference_bernoulli():
    """a grid of z = sign v / sqrt(tau^2 + tau) across both cut-offs of util/univariate_Gaussian.py (|z| = 0.6629 and
    |z| / sqrt(2) >= 4, both signs) and several cavity precisions"""
    lik = _ref_bernoulli()
    zs = np.concatenate([np.linspace(-12, 12, 241), [-5.6569, -5.6568, -0.6629, -0.6628, 0.0, 0.6628, 0.6629, 5.6568,
                                                     5.6569, 30.0, -30.0]])
    for tau in (0.05, 1.0, 7.5):
        q = np.sqrt(tau ** 2 + tau)
        for z in zs:
            for y in (1.0, 0.0, -1.0):
                sign = 1.0 if y == 1 else -1.0
                v = sign * z * q
                assert eo.moments(y, tau, v) == lik.moments_match_ep(y, tau, v)


def test_rng_stream_after_a_run_matches_in_both_modes():
    for name in ("rbf_iso_n60", "rbf_ard_parallel_n150"):
        z = np.load(os.path.join(HERE, "golden", "ep", name + ".npz"))
        assert eo.case_eval(name)["next_random"] == z["next_random"]


def test_mirror_rejections():
    import gpy_b200 as B
    X = np.zeros((4, 3))
    with pytest.raises(ValueError, match="bad value for Bernoulli observation"):
        B.EP().inference(B.RBF(3), X, B.Bernoulli(), np.array([[0.], [1.], [2.], [1.]]))
    with pytest.raises(NotImplementedError):
        B.EP().inference(B.RBF(3), X, B.Bernoulli(), np.ones((4, 1)), mean_function=object())
    with pytest.raises(NotImplementedError):
        B.EP().inference(B.RBF(3), X, B.StudentT(), np.ones((4, 1)))
    with pytest.raises(ValueError, match="ep_mode"):
        class Eng(object):
            N = 4

            def set_data(self, X, Y):
                pass

            def ep_begin(self, parts):
                return 2
        B.EP(ep_mode="other", engine=Eng()).inference(B.RBF(3), X, B.Bernoulli(), np.ones((4, 1)))


def test_posterior_ep_has_no_variance_clip():
    import gpy_b200 as B
    assert B.PosteriorEP._var_floor is None and B.PosteriorLaplace._var_floor == 1e-15
    assert issubclass(B.PosteriorEP, B.PosteriorLaplace)
    assert np.array_equal(B.Bernoulli().ep_gradients(np.ones((3, 1)), np.ones(3), np.ones(3), np.ones(3)), np.zeros(0))


class HostEPEngine(object):
    """every EP entry on the host: the blocked restatement of ep_oracle on the K of the described kernel"""

    def __init__(self, device=0):
        self.calls = []

    def set_data(self, X, Y):
        self.calls.append(("set_data",))
        self.X, self.N = np.array(X), X.shape[0]

    def ep_begin(self, parts):
        from test_laplace_cpu import _parts_of
        self.calls.append(("begin", parts))
        self.parts = _parts_of(parts)
        self.kern = eo.CompositeOracle(self.parts)
        self.K = self.kern.K(self.X)
        self.y = None
        return int(sum(b.size for b in self.kern.grads_full(np.zeros_like(self.K), self.X)))

    def ep_start(self, tau_tilde=None, v_tilde=None, parallel=False, max_tries=5):
        self.calls.append(("start", tau_tilde is not None))
        if tau_tilde is None:
            self.Sigma, self.mu = self.K + 1e-7 * np.eye(self.N), np.zeros(self.N)
        else:
            self.mu, self.Sigma, _ = eo.recompute(self.K, tau_tilde, v_tilde)
            self.Sigma[np.diag_indices(self.N)] += 1e-7
        return 0.0

    def ep_sweep(self, order, tau_tilde, v_tilde, eta=1., delta=1., parallel=False, max_tries=5):
        self.calls.append(("sweep",))
        st = {k: np.empty(self.N) for k in ("ct", "cv", "Z", "mh", "s2")}
        st["tt"], st["vt"] = np.array(tau_tilde, dtype=float), np.array(v_tilde, dtype=float)
        y = self.y if self.y is not None else self._labels
        self.Sigma, self.mu = eo.sweep(self.Sigma, self.mu, st, y, np.asarray(order), eta, delta, parallel, True)
        self.mu, self.Sigma, _ = eo.recompute(self.K, st["tt"], st["vt"])
        return st["tt"], st["vt"], st["ct"], st["cv"], st["Z"], st["mh"], st["s2"], 0.0

    def ep_finish(self, tau_tilde, v_tilde, max_tries=5):
        self.calls.append(("finish",))
        mu, Sigma, L = eo.recompute(self.K, tau_tilde, v_tilde)
        r = np.sqrt(tau_tilde)
        aux = np.linalg.solve(np.dot(L, L.T), r * np.dot(self.K, v_tilde))
        alpha = (v_tilde - r * aux)[:, None]
        Li = np.linalg.inv(L)
        Wi = np.dot((Li * r[None, :]).T, Li * r[None, :])
        dL_dK = 0.5 * (np.dot(alpha, alpha.T) - Wi)
        kgrad = np.concatenate(self.kern.grads_full(dL_dK, self.X))
        return (np.sum(2.0 * np.log(np.diag(L))), float(np.dot(v_tilde, np.dot(Sigma, v_tilde))), np.diag(dL_dK).copy(),
                kgrad, 0.0)


def _plugin():
    from ep_reference import load_reference_ep
    from oracle import ref_gpy
    from gpy_b200 import gpy_plugin
    try:
        M = ref_gpy.load_models()
    except ImportError:
        pytest.skip("reference tree not present")
    C = ref_gpy.load_combination()
    G = M.G
    EP, Bern, ObsAr = load_reference_ep()
    from test_periodic_ratquad_plugin_cpu import fake_ffi
    import types
    f = fake_ffi()

    class Eng(HostEPEngine):
        def set_data(self, X, Y):
            super(Eng, self).set_data(X, Y)
            self._labels = np.array(Y)[:, 0]

    ffi = types.SimpleNamespace(kern_K=f.kern_K, kern_Kdiag=f.kern_Kdiag, kern_grad_full=f.kern_grad_full,
                                kern_part_K=f.kern_part_K, kern_part_grad_full=f.kern_part_grad_full, Engine=Eng)
    B = gpy_plugin.make(G.RBF, G.Exponential, G.Matern32, G.Matern52, G.ExactGaussianInference, Add=C.Add, Prod=C.Prod,
                        EP=EP, ffi=ffi)
    return M, C, G, B, EP, Bern, ObsAr


@pytest.mark.parametrize("case", ["rbf_ard_n150", "rbf_ard_x_m52_bias_n150"])
def test_reference_gp_over_plugin_ep_matches_the_stock_pair(case):
    M, C, G, B, EP, Bern, ObsAr = _plugin()
    parts, _, seed, _ = eo.CASES[case]
    X, Y, _ = eo.case_data(case)

    def kern(ns):
        if len(parts) == 1:
            return ns.RBF(3, variance=parts[0]["variance"], lengthscale=parts[0]["lengthscale"], ARD=True)
        k = ns.RBF(3, variance=1.3, lengthscale=[0.9, 1.4, 2.1], ARD=True)
        m = ns.Matern52(2, variance=1.1, lengthscale=1.2, active_dims=[0, 1])
        prod, add = (B.Prod, B.Add) if ns is B else (C.Prod, C.Add)
        return add([prod([k, m]), C.Bias(3, variance=0.4)])

    np.random.seed(seed)
    stock = M.GP(X, Y, kern(G), Bern(), inference_method=EP())
    r_stock = np.random.random()
    np.random.seed(seed)
    plug = M.GP(X, Y, kern(B), Bern(), inference_method=B.EP())
    assert np.random.random() == r_stock
    names = [c[0] for c in plug.inference_method.engine.calls]
    assert names[:3] == ["set_data", "begin", "start"] and names[-1] == "finish"
    l_s, l_p = float(np.squeeze(stock.log_likelihood())), float(np.squeeze(plug.log_likelihood()))
    assert abs(l_p - l_s) <= 1e-11 * abs(l_s)
    gs, gp = np.asarray(stock.gradient), np.asarray(plug.gradient)
    np.testing.assert_allclose(gp, gs, rtol=0, atol=1e-10 * np.abs(gs).max())
    ga_s, ga_p = stock.inference_method.ga_approx_old, plug.inference_method.ga_approx_old
    assert type(ga_p) is type(ga_s)
    np.testing.assert_allclose(ga_p.tau, ga_s.tau, rtol=0, atol=1e-10)
    assert len(plug.inference_method._ep_approximation) == 4


def test_plugin_ep_sends_anything_else_to_the_stock_method_and_continues_its_sites():
    M, C, G, B, EP, Bern, ObsAr = _plugin()
    X, Y, _ = eo.case_data("rbf_iso_n60")
    Yo = ObsAr(Y)
    inf = B.EP(ep_mode="nested")
    np.random.seed(1)
    inf.inference(G.RBF(3), X, Bern(), Yo)                                       # the reference's own kernel
    assert inf._engine is None or not inf.engine.calls
    with pytest.raises(Exception):
        inf.inference(B.RBF(3), X, Bern(), Yo, mean_function=object())           # a mean function: the stock method
    assert inf._engine is None or not inf.engine.calls
    inf.inference(B.RBF(3), X, Bern(), Yo, K=G.RBF(3).K(X))                     # a precomputed K: the stock method
    assert inf._engine is None or not inf.engine.calls
    # the device continues from the stock method's sites (warm start), as two stock calls do
    ref = EP(ep_mode="nested")
    np.random.seed(1)
    ref.inference(G.RBF(3), X, Bern(), Yo)
    ref.inference(G.RBF(3), X, Bern(), Yo, K=G.RBF(3).K(X))
    _, l_ref, _ = ref.inference(G.RBF(3), X, Bern(), Yo)
    _, l_dev, _ = inf.inference(B.RBF(3), X, Bern(), Yo)
    assert ("start", True) in inf.engine.calls
    assert abs(l_dev - l_ref) <= 1e-11 * abs(l_ref)
