"""The Laplace approximation without a GPU: the NumPy restatement against the reference's fixtures, the mirror's
likelihoods against the reference's classes, and the host loop of gpy_b200.Laplace on a test double of the engine."""
import glob
import importlib
import os
import types

import numpy as np
import pytest

import laplace_oracle as lo

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = sorted(glob.glob(os.path.join(HERE, "golden", "laplace", "*.npz")))


def _mirror():
    import gpy_b200
    return types.SimpleNamespace(Bernoulli=gpy_b200.Bernoulli, StudentT=gpy_b200.StudentT)


def test_every_case_has_a_fixture():
    assert sorted(os.path.basename(p)[:-4] for p in FIXTURES) == sorted(lo.CASES)


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[:-4])
def test_oracle_matches_reference_fixture(path):
    name = os.path.basename(path)[:-4]
    parts, lik, N, _ = lo.CASES[name]
    z = np.load(path)
    X, Y, Xnew = lo.case_data(name)
    np.testing.assert_array_equal(X, z["X"])
    np.testing.assert_array_equal(Y, z["Y"])
    r = lo.laplace_eval(X, Y, parts, lo.make_likelihood(lik, _mirror()), Xnew)
    assert r["iterations"] == int(z["iterations"])
    # every Brent step too: the restatement calls LAPACK as GPy's util/linalg.py does and meets the reference to rounding
    np.testing.assert_allclose(r["brent"], z["brent"], rtol=1e-12, atol=0)
    assert abs(r["lml"] - float(z["lml"])) <= 1e-12 * max(1.0, abs(float(z["lml"])))
    for k in ("grad", "dL_dthetaL", "f_hat", "Ki_f", "W", "diag_Ki_W_i", "mu", "var"):
        scale = max(1.0, float(np.abs(z[k]).max())) if z[k].size else 1.0
        np.testing.assert_allclose(r[k], z[k], rtol=0, atol=1e-12 * scale, err_msg=k)
    if "woodbury_inv" in z:
        np.testing.assert_allclose(r["woodbury_inv"], z["woodbury_inv"], rtol=0,
                                   atol=1e-12 * max(1.0, float(np.abs(z["woodbury_inv"]).max())))


def _ref_likelihoods():
    try:
        from oracle import ref_gpy
        ref_gpy.load()
    except ImportError:
        pytest.skip("reference tree not present")
    return (importlib.import_module("GPy.likelihoods.bernoulli").Bernoulli,
            importlib.import_module("GPy.likelihoods.student_t").StudentT)


def test_mirror_likelihoods_match_reference_classes():
    RB, RS = _ref_likelihoods()
    import gpy_b200 as B
    rng = np.random.RandomState(3)
    f = rng.randn(200, 1) * 4
    yb = (rng.rand(200, 1) > 0.5).astype(float)
    ys = rng.randn(200, 1) * 2
    for ref, mine, y in ((RB(), B.Bernoulli(), yb), (RS(deg_free=3.7, sigma2=0.4), B.StudentT(deg_free=3.7, sigma2=0.4), ys)):
        for fn in ("logpdf", "dlogpdf_df", "d2logpdf_df2", "d3logpdf_df3"):
            a, b = getattr(ref, fn)(f, y), getattr(mine, fn)(f, y)
            np.testing.assert_allclose(b, a, rtol=1e-14, atol=0, err_msg=fn)
        for a, b in zip(ref._laplace_gradients(f, y), mine._laplace_gradients(f, y)):
            assert a.shape == b.shape
            np.testing.assert_allclose(b, a, rtol=1e-14, atol=0)
        assert ref.log_concave == mine.log_concave and ref.size == mine.size
    mu, var = rng.randn(20, 1), rng.rand(20, 1) + 0.1
    np.testing.assert_allclose(B.Bernoulli().predictive_values(mu, var)[0], RB().predictive_values(mu, var)[0],
                               rtol=1e-14)
    for df in (3.7, 1.5):   # the reference's quadrature, and NaN for deg_free <= 2
        ref = RS(deg_free=df, sigma2=0.4)
        ref.deg_free = ref.v   # student_t.py reads the parameter by its name, an attribute paramz adds when it is linked
        a, b = ref.predictive_values(mu, var), B.StudentT(deg_free=df, sigma2=0.4).predictive_values(mu, var)
        for x, y in zip(b, a):
            assert np.shape(x) == np.shape(y)
            np.testing.assert_allclose(x, y, rtol=1e-14, atol=0)


class FakeEngine(object):
    """the engine's Laplace entries on the host (laplace_oracle's algebra), recording every call"""

    def __init__(self, K):
        self.K, self.calls, self.N, self.eval_serial = K, [], K.shape[0], 0

    def set_data(self, X, Y):
        self.calls.append(("set_data", X.shape, Y.shape))

    def laplace_begin(self, parts):
        self.calls.append(("begin", parts))
        return 2

    def laplace_matvec(self, v):
        self.calls.append(("matvec",))
        return np.dot(self.K, np.asarray(v).reshape(-1, 1))

    def laplace_newton(self, W, b, Ki_f, max_tries=5):
        self.calls.append(("newton", np.array(W), np.array(b)))
        K_Wi_i = lo.b_statistics(self.K, np.asarray(W).reshape(-1, 1), True)[0]
        a = b.reshape(-1, 1) - np.dot(K_Wi_i, np.dot(self.K, b.reshape(-1, 1)))
        d = a - Ki_f.reshape(-1, 1)
        return d, np.dot(self.K, d), 0.0

    def laplace_finish(self, W, Ki_f, dW_df, g=None, max_tries=5):
        self.calls.append(("finish", np.array(W), None if g is None else np.array(g)))
        _, logdet, _, Ki_W_i, _, _ = lo.b_statistics(self.K, np.asarray(W).reshape(-1, 1), True)
        return logdet, np.diag(Ki_W_i).copy(), np.zeros(2), np.zeros(0 if g is None else g.shape[0]), 0.0


def _model_inputs(lik="bernoulli"):
    import gpy_b200 as B
    X, Y, _ = lo.case_data("bernoulli_rbf_iso_n60" if lik == "bernoulli" else "studentt_matern52_ard_n150")
    k = B.RBF(3, variance=1.4, lengthscale=1.1)
    return B, X, Y, k


def test_host_loop_calls_the_entries_in_order():
    B, X, Y, k = _model_inputs()
    K = lo.CompositeOracle(lo._single("rbf", False)).K(X)
    eng = FakeEngine(K)
    inf = B.Laplace(engine=eng)
    post, lml, gd = inf.inference(k, X, B.Bernoulli(), Y)
    names = [c[0] for c in eng.calls]
    z = np.load(os.path.join(HERE, "golden", "laplace", "bernoulli_rbf_iso_n60.npz"))
    n = int(z["iterations"])
    assert names == ["set_data", "begin", "matvec"] + ["newton", "matvec"] * n + ["finish"]
    assert eng.calls[1][1] == [("rbf", False, 0, [0, 1, 2], 1.4, 1.1)]
    assert inf.iterations == n
    # the line search takes f_trial = f + s K dKi_f, not K (Ki_f + s dKi_f): Brent's last step on the flat objective
    # moves with that rounding, and f_hat with it
    assert abs(lml - float(z["lml"])) < 1e-9 * abs(float(z["lml"]))
    np.testing.assert_allclose(inf.f_hat, z["f_hat"], rtol=0, atol=1e-6)
    assert gd["dL_dthetaL"].shape == (0,)
    # the same data is not uploaded again
    inf.inference(k, X, B.Bernoulli(), Y)
    assert [c[0] for c in eng.calls].count("set_data") == 1


def test_clipped_W_goes_to_the_device_and_unclipped_into_b():
    B, X, Y, _ = _model_inputs("studentt")
    k = B.Matern52(3, variance=0.6, lengthscale=[0.8, 1.3, 1.9], ARD=True)
    K = lo.CompositeOracle(lo._single("matern52", True, 0.6)).K(X)
    eng = FakeEngine(K)
    lik = B.StudentT(deg_free=3.0, sigma2=0.05)
    B.Laplace(engine=eng).inference(k, X, lik, Y)
    for c in eng.calls:
        if c[0] in ("newton", "finish"):
            assert c[1].min() >= 1e-6
    fin = [c for c in eng.calls if c[0] == "finish"][0]
    assert fin[2].shape == (2, X.shape[0])


def test_reference_exceptions():
    B, X, Y, k = _model_inputs()
    eng = FakeEngine(np.eye(X.shape[0]))
    with pytest.raises(AssertionError):
        B.Laplace(engine=eng).inference(k, X, B.Bernoulli(), Y, mean_function=object())

    class NaNLik(B.Bernoulli):
        def d2logpdf_df2(self, f, y, Y_metadata=None):
            return np.full_like(f, np.nan)

    with pytest.raises(ValueError, match="W is NaN"):
        B.Laplace(engine=FakeEngine(np.eye(X.shape[0]))).inference(k, X, NaNLik(), Y)
    with pytest.raises(ValueError, match="one output column"):
        B.Laplace(engine=eng).inference(k, X, B.Bernoulli(), np.hstack([Y, Y]))


def _parts_of(desc):
    """Engine.laplace_begin descriptors -> laplace_oracle part dicts"""
    return [dict(kind=k, ARD=a, term=t, dims=list(d), variance=v, lengthscale=l) for (k, a, t, d, v, l) in
            [tuple(x[:6]) for x in desc]]


class HostLaplaceEngine(FakeEngine):
    """every Laplace entry on the host: the algebra of laplace_oracle on the K of the described kernel"""

    def __init__(self, device=0):
        super(HostLaplaceEngine, self).__init__(np.zeros((0, 0)))

    def set_data(self, X, Y):
        super(HostLaplaceEngine, self).set_data(X, Y)
        self.X, self.N = np.array(X), X.shape[0]

    def laplace_begin(self, parts):
        self.calls.append(("begin", parts))
        self.kern = lo.CompositeOracle(_parts_of(parts))
        self.K = self.kern.K(self.X)
        return int(sum(b.size for b in self.kern.grads_full(np.zeros_like(self.K), self.X)))

    def laplace_finish(self, W, Ki_f, dW_df, g=None, max_tries=5):
        self.calls.append(("finish", np.array(W), None if g is None else np.array(g)))
        K, Ki_f = self.K, Ki_f.reshape(-1, 1)
        K_Wi_i, logdet, I_KW_i, Ki_W_i, _, _ = lo.b_statistics(K, np.asarray(W).reshape(-1, 1), True)
        dL_dfhat = -0.5 * np.diag(Ki_W_i)[:, None] * dW_df.reshape(-1, 1)
        dL_dK = 0.5 * (np.dot(Ki_f, Ki_f.T) - K_Wi_i) + np.dot(Ki_f, dL_dfhat.T).dot(I_KW_i)
        kgrad = np.concatenate(self.kern.grads_full(dL_dK, self.X))
        imp = np.zeros(0) if g is None else np.array([float(dL_dfhat.T.dot(I_KW_i).dot(K).dot(gt)) for gt in g])
        return logdet, np.diag(Ki_W_i).copy(), kgrad, imp, 0.0


def _plugin():
    from oracle import ref_gpy
    from gpy_b200 import gpy_plugin
    M = ref_gpy.load_models()
    C = ref_gpy.load_combination()
    G = M.G
    lap = importlib.import_module("GPy.inference.latent_function_inference.laplace")
    from test_periodic_ratquad_plugin_cpu import fake_ffi
    f = fake_ffi()
    ffi = types.SimpleNamespace(kern_K=f.kern_K, kern_Kdiag=f.kern_Kdiag, kern_grad_full=f.kern_grad_full,
                                kern_part_K=f.kern_part_K, kern_part_grad_full=f.kern_part_grad_full,
                                Engine=HostLaplaceEngine)
    B = gpy_plugin.make(G.RBF, G.Exponential, G.Matern32, G.Matern52, G.ExactGaussianInference, Add=C.Add, Prod=C.Prod,
                        Laplace=lap.Laplace, ffi=ffi)
    return M, C, G, B, lap


@pytest.mark.parametrize("case", ["bernoulli_rbf_ard_n150", "studentt_composite_n150"])
def test_reference_gp_over_plugin_laplace_matches_the_stock_pair(case):
    _ref_likelihoods()
    M, C, G, B, lap = _plugin()
    RB, RS = _ref_likelihoods()
    parts, lik, _, _ = lo.CASES[case]
    X, Y, _ = lo.case_data(case)

    def kern(ns):
        if len(parts) == 1:
            return ns.RBF(3, variance=parts[0]["variance"], lengthscale=parts[0]["lengthscale"], ARD=True)
        k = ns.RBF(3, variance=1.3, lengthscale=[0.9, 1.4, 2.1], ARD=True)
        m = ns.Matern52(2, variance=1.1, lengthscale=1.2, active_dims=[0, 1])
        prod, add = (B.Prod, B.Add) if ns is B else (C.Prod, C.Add)
        return add([prod([k, m]), C.Bias(3, variance=0.4)])

    def L():
        return lo.make_likelihood(lik, types.SimpleNamespace(Bernoulli=RB, StudentT=RS))

    stock = M.GP(X, Y, kern(G), L(), inference_method=lap.Laplace())
    plug = M.GP(X, Y, kern(B), L(), inference_method=B.Laplace())
    names = [c[0] for c in plug.inference_method.engine.calls]
    assert names[:3] == ["set_data", "begin", "matvec"] and names[-1] == "finish"
    l_s, l_p = float(np.squeeze(stock.log_likelihood())), float(np.squeeze(plug.log_likelihood()))
    assert abs(l_p - l_s) <= 1e-8 * abs(l_s)
    gs, gp = np.asarray(stock.gradient), np.asarray(plug.gradient)
    np.testing.assert_allclose(gp, gs, rtol=0, atol=1e-6 * np.abs(gs).max())
    np.testing.assert_allclose(plug.inference_method.f_hat, stock.inference_method.f_hat, rtol=0, atol=1e-6)


def test_plugin_laplace_sends_anything_else_to_the_stock_method():
    M, C, G, B, lap = _plugin()
    RB, _ = _ref_likelihoods()
    X, Y, _ = lo.case_data("bernoulli_rbf_iso_n60")
    inf = B.Laplace()
    inf.inference(G.RBF(3), X, RB(), Y)                                          # the reference's own kernel
    with pytest.raises(AssertionError):
        inf.inference(B.RBF(3), X, RB(), Y, mean_function=object())
    assert inf._engine is None or not inf.engine.calls
    inf.inference(B.RBF(3), X, RB(), Y)
    assert inf.engine.calls[-1][0] == "finish"
