"""GPU parity tests (run on the H100 with -m gpu): the CUDA path through the C ABI against the CPU oracle on the same
seeded inputs. Tolerances are those of BASELINE.json's north star: 1e-8 absolute on the log marginal likelihood,
1e-6 relative on gradients (fp64 throughout)."""
import os

import numpy as np
import pytest

import gpy_b200
from gpy_b200 import _ffi
from oracle import gpy_oracle as o

pytestmark = pytest.mark.gpu

LML_ATOL = 1e-8
GRAD_RTOL = 1e-6


@pytest.fixture(scope="module")
def eng():
    e = _ffi.Engine(0)
    yield e
    e.close()


def rel(a, b):
    return float(np.max(np.abs(np.asarray(a) - np.asarray(b))) / max(float(np.max(np.abs(b))), 1e-300))


def theta(D, ARD, seed):
    rng = np.random.default_rng(seed)
    ls = np.sqrt(D) * rng.uniform(0.7, 1.4, D) if ARD else float(np.sqrt(D) * rng.uniform(0.7, 1.4))
    return float(rng.uniform(0.5, 2.0)), ls, float(rng.uniform(0.01, 0.1))


CASES = [(k, a, n, d) for (k, a, d) in [("rbf", True, 8), ("rbf", False, 2), ("matern52", True, 5), ("matern32", False, 3),
                                       ("exponential", True, 4), ("exponential", False, 1), ("matern32", True, 7),
                                       ("matern52", False, 6)]
         for n in (1, 2, 127, 128, 129, 500, 1300)]


@pytest.mark.parametrize("kind,ARD,N,D", CASES)
def test_lml_and_gradient_match_oracle(eng, kind, ARD, N, D):
    X, Y = o.synthetic(N, D, seed=N + D)
    var, ls, noise = theta(D, ARD, N)
    lml0, g0, res = o.eval_lml_grad(X, Y, kind, ARD, var, ls, noise)
    eng.set_data(X, Y)
    lml, g, jit = eng.exact_eval(kind, ARD, var, ls, noise)
    assert jit == 0.0
    assert abs(lml - lml0) <= LML_ATOL, (lml, lml0)
    np.testing.assert_allclose(g, g0, rtol=GRAD_RTOL, atol=1e-9)
    if N <= 500:
        assert rel(eng.get("L"), res["L"]) < 1e-10
        assert rel(eng.get("alpha"), res["alpha"]) < 1e-9
        assert rel(eng.get("Kinv"), res["Wi"]) < 1e-9
        assert rel(eng.get("dL_dK"), res["dL_dK"]) < 1e-9
        assert rel(eng.get("K"), res["K"]) < 1e-12
        assert rel(eng.get("Linv"), np.linalg.inv(res["L"])) < 1e-9


@pytest.mark.parametrize("nb", [128, 256, 384, 1024])
def test_block_size_does_not_change_the_answer(nb):
    e = _ffi.Engine(0)
    e.set_option("nb", nb)
    X, Y = o.synthetic(1700, 4, seed=11)
    var, ls, noise = theta(4, True, 5)
    lml0, g0, _ = o.eval_lml_grad(X, Y, "rbf", True, var, ls, noise)
    e.set_data(X, Y)
    lml, g, _ = e.exact_eval("rbf", True, var, ls, noise)
    assert abs(lml - lml0) <= LML_ATOL
    np.testing.assert_allclose(g, g0, rtol=GRAD_RTOL)
    e.close()


def test_metric_size_n4096_against_oracle():
    """N=4096, D=8 (the smallest size of the BASELINE.json metric): LML, gradient and alpha against the oracle, on both
    tensor paths (option ozaki = 0 and 1). N = 4096 is the smallest size at which the int8 path also runs the panel GEMM
    on the tensor cores."""
    X, Y = o.synthetic(4096, 8, seed=3)
    var, ls, noise = o.theta_bench(8, True)
    lml0, g0, res = o.eval_lml_grad(X, Y, "matern32", True, var, ls, noise)
    for oz in (0, 1):
        e = _ffi.Engine(0)
        e.set_option("ozaki", oz)
        e.set_data(X, Y)
        lml, g, _ = e.exact_eval("matern32", True, var, ls, noise)
        assert abs(lml - lml0) <= LML_ATOL, (oz, lml, lml0)
        np.testing.assert_allclose(g, g0, rtol=GRAD_RTOL, err_msg="ozaki = %d" % oz)
        assert rel(e.get("alpha"), res["alpha"]) < 1e-9, oz
        e.close()


def test_config3_kernel_matern52_d32_n4096_against_oracle():
    """BASELINE.json configs[2] uses Matern52, D=32, isotropic lengthscale (GPy default ARD=False): one evaluation at
    N=4096 against the oracle at the initial theta of that optimisation and at a second, less smooth theta."""
    X, Y = o.synthetic(4096, 32, seed=0)
    e = _ffi.Engine(0)
    e.set_data(X, Y)
    for (var, ls, noise) in ((1.0, float(np.sqrt(32)), 0.1), (0.6, 3.1, 0.02)):
        lml0, g0, res = o.eval_lml_grad(X, Y, "matern52", False, var, ls, noise)
        lml, g, _ = e.exact_eval("matern52", False, var, ls, noise)
        assert abs(lml - lml0) <= LML_ATOL, (lml, lml0)
        np.testing.assert_allclose(g, g0, rtol=GRAD_RTOL)
        assert rel(e.get("alpha"), res["alpha"]) < 1e-9
    e.close()


def test_config3_optimize_loop_final_lml_matches_cpu_run():
    """BASELINE.json configs[2] in small: GPRegression Matern52 D=32, full optimize() (L-BFGS-B on the Logexp-transformed
    parameters, GPy/core/gp.py:663-684) on the device against the SAME loop run on the CPU oracle from the same theta_0
    (SURVEY.md §8d config 3: "final LML vs CPU"). The trajectory is parity-unpinned in the reference (paramz's optimizer,
    its only test asserts nothing); what must agree is where the loop ends."""
    N, D = 1500, 32
    X, Y = o.synthetic(N, D, seed=0)
    k = gpy_b200.Matern52(D, variance=1.0, lengthscale=float(np.sqrt(D)))
    m = gpy_b200.GPRegression(X, Y, k, noise_var=0.1)
    lml_start = m.log_likelihood()
    res = m.optimize(max_iters=60)
    lml_c, th_c, n_c, lml_c0 = o.optimize_lbfgsb(X, Y, "matern52", False, 1.0, float(np.sqrt(D)), 0.1, max_iters=60)
    assert abs(lml_start - lml_c0) <= LML_ATOL
    th_g = np.concatenate([k.variance.values, k.lengthscale.values, m.likelihood.variance.values])
    # the device and the CPU loop see objectives that agree to ~1e-11, so they take the same path until round-off decides a
    # line-search branch; both must end at the same optimum
    assert abs(m.log_likelihood() - lml_c) <= 1e-5 * max(1.0, abs(lml_c)), (m.log_likelihood(), lml_c, res["n_evals"], n_c)
    np.testing.assert_allclose(th_g, th_c, rtol=2e-3)
    assert m.log_likelihood() > lml_start
    # and the evaluation AT the device's final theta agrees with the oracle to the per-evaluation tolerances
    lml0, g0, _ = o.eval_lml_grad(X, Y, "matern52", False, float(th_g[0]), float(th_g[1]), float(th_g[2]))
    assert abs(m.log_likelihood() - lml0) <= LML_ATOL
    np.testing.assert_allclose(m.gradient, g0, rtol=GRAD_RTOL, atol=1e-7)


def test_multiple_outputs_and_large_D(eng):
    rng = np.random.default_rng(0)
    X = rng.uniform(-3, 3, (400, 64))
    Y = rng.standard_normal((400, 3))
    ls = 8.0 * rng.uniform(0.8, 1.2, 64)
    lml0, g0, res = o.eval_lml_grad(X, Y, "matern52", True, 1.2, ls, 0.3)
    eng.set_data(X, Y)
    lml, g, _ = eng.exact_eval("matern52", True, 1.2, ls, 0.3)
    assert abs(lml - lml0) <= LML_ATOL
    np.testing.assert_allclose(g, g0, rtol=GRAD_RTOL, atol=1e-9)
    assert rel(eng.get("alpha"), res["alpha"]) < 1e-9


def test_golden_fixtures(eng):
    """tests/golden/*.npz (tests/golden/make_golden.py): LML, gradient, alpha and predictions."""
    gdir = os.path.join(os.path.dirname(__file__), "golden")
    files = sorted(f for f in os.listdir(gdir) if f.endswith(".npz"))
    assert files
    for fn in files:
        z = np.load(os.path.join(gdir, fn))
        kind, ARD = str(z["kind"]), bool(z["ARD"])
        ls = z["lengthscale"] if ARD else float(z["lengthscale"])
        eng.set_data(z["X"], z["Y"])
        lml, g, _ = eng.exact_eval(kind, ARD, float(z["variance"]), ls, float(z["noise"]))
        assert abs(lml - float(z["lml"])) <= LML_ATOL, fn
        np.testing.assert_allclose(g, z["grad"], rtol=GRAD_RTOL, atol=1e-9, err_msg=fn)
        assert rel(eng.get("alpha"), z["alpha"]) < 1e-8, fn
        mu, var = eng.predict(z["Xnew"])
        np.testing.assert_allclose(mu, z["mu"], rtol=1e-8, atol=1e-10, err_msg=fn)
        np.testing.assert_allclose(var + float(z["noise"]), z["var"], rtol=1e-7, atol=1e-10, err_msg=fn)


@pytest.mark.parametrize("kind", o.KINDS)
@pytest.mark.parametrize("ARD", [False, True])
def test_kernel_plugin_calls(kind, ARD):
    """Kern.K / Kdiag / update_gradients_full as stand-alone plugin calls (test_kernel.py fixtures: 10x6 and 20x6
    standard normal; test_cython.py: 300x10 / 20x10)."""
    rng = np.random.default_rng(7)
    for (n, m, d) in ((10, 20, 6), (300, 20, 10), (257, 131, 3)):
        X, X2 = rng.standard_normal((n, d)), rng.standard_normal((m, d))
        ls = rng.uniform(0.8, 2.0, d) if ARD else float(rng.uniform(0.8, 2.0))
        cls = {"rbf": gpy_b200.RBF, "exponential": gpy_b200.Exponential, "matern32": gpy_b200.Matern32,
               "matern52": gpy_b200.Matern52}[kind]
        k = cls(d, variance=0.7, lengthscale=ls, ARD=ARD)
        ko = o.StationaryOracle(kind, d, 0.7, ls, ARD)
        assert rel(k.K(X), ko.K(X)) < 1e-13
        assert rel(k.K(X, X2), ko.K(X, X2)) < 1e-13
        np.testing.assert_array_equal(k.Kdiag(X), ko.Kdiag(X))
        for XX2, shape in ((None, (n, n)), (X2, (n, m))):
            dL = rng.standard_normal(shape)
            k.update_gradients_full(dL, X, XX2)
            v0, l0 = ko.update_gradients_full(dL, X, XX2)
            np.testing.assert_allclose(k.variance.gradient, v0, rtol=1e-10)
            np.testing.assert_allclose(k.lengthscale.gradient, l0, rtol=1e-9, atol=1e-12)


def test_jitter_ladder_and_failure(eng):
    """jitchol semantics (GPy/util/linalg.py:56-75; test_linalg.py:20-37): duplicated inputs with zero noise are
    singular -> the ladder adds mean(diag)*1e-6*10^k; the result equals the oracle run with the same ladder."""
    Xd = np.repeat(o.synthetic(100, 2, 9)[0], 2, axis=0)
    Yd = np.sin(Xd[:, :1])
    eng.set_data(Xd, Yd)
    lml, g, jit = eng.exact_eval("rbf", False, 1.0, 2.0, 0.0, jitter=0.0)
    assert jit > 0
    k = o.StationaryOracle("rbf", 2, 1.0, 2.0, False)
    Ky = k.K(Xd)
    L, jit0 = o.jitchol(Ky)
    assert np.isclose(jit, jit0, rtol=1e-12)
    alpha = o.dpotrs(L, Yd)[0]
    lml0 = 0.5 * (-Yd.size * o.LOG_2_PI - 2 * np.sum(np.log(np.diag(L))) - np.sum(alpha * Yd))
    assert abs(lml - lml0) <= 1e-6 * abs(lml0)   # ill-conditioned by construction (cond ~ 1e6 / jitter)
    with pytest.raises(np.linalg.LinAlgError):
        eng.exact_eval("rbf", False, 1.0, 2.0, 0.0, jitter=0.0, max_tries=0)


def test_gpregression_model_api():
    """GPRegression through the plugin mirror: log_likelihood/gradient, checkgrad (test_model.py:790-833), predict vs the
    pinv formula (test_model.py:83-105), optimize improves the objective (test_model.py:510-517)."""
    rng = np.random.default_rng(3)
    X = rng.uniform(-3, 3, (40, 2))
    Y = np.sin(X[:, :1]) + 0.05 * rng.standard_normal((40, 1))
    for kern in (gpy_b200.RBF(2, ARD=True), gpy_b200.Matern52(2), gpy_b200.Matern32(2, ARD=True), gpy_b200.Exponential(2)):
        m = gpy_b200.GPRegression(X, Y, kern)
        kind, ard, var, ls = kern._theta()
        lml0, g0, _ = o.eval_lml_grad(X, Y, kind, ard, var, ls, 1.0)
        assert abs(m.log_likelihood() - lml0) <= LML_ATOL
        np.testing.assert_allclose(m.gradient, g0, rtol=GRAD_RTOL)
        assert m.checkgrad()
    m = gpy_b200.GPRegression(X, Y, gpy_b200.RBF(2, ARD=True))
    f0 = m.objective_function()
    m.optimize(max_iters=60)
    assert m.objective_function() < f0 - 1.0
    # predict_noiseless vs explicit pinv
    Xn = rng.uniform(-3, 3, (9, 2))
    k = m.kern
    Kinv = np.linalg.pinv(k.K(X) + np.eye(40) * (float(m.likelihood.variance[0]) + 1e-8))
    mu_hat = k.K(Xn, X).dot(Kinv).dot(Y)
    K_hat = k.K(Xn) - k.K(Xn, X).dot(Kinv).dot(k.K(X, Xn))
    mu, cov = m.predict_noiseless(Xn, full_cov=True)
    np.testing.assert_allclose(mu, mu_hat, rtol=1e-6, atol=1e-7)
    np.testing.assert_allclose(cov, K_hat, rtol=1e-5, atol=1e-7)
    mu, var = m.predict(Xn)
    np.testing.assert_allclose(var, np.diag(K_hat)[:, None] + float(m.likelihood.variance[0]), rtol=1e-5, atol=1e-7)


def test_full_size_properties():
    """BASELINE.json configs[1] size (N=16384, D=8, RBF ARD): size-independent checks.
    (1) analytic gradient == central finite difference of the device LML; (2) LML is invariant under a permutation of
    the data; (3) alpha solves Ky alpha = y (residual through an independent device K build of a row block)."""
    N, D = 16384, 8
    X, Y = o.synthetic(N, D)
    var, ls, noise = o.theta_bench(D, True)
    e = _ffi.Engine(0)
    e.set_data(X, Y)
    lml, g, _ = e.exact_eval("rbf", True, var, ls, noise)
    th = np.concatenate([[var], ls, [noise]])
    for i in (0, 3, D + 1):
        h = 1e-5 * th[i]
        tp, tm = th.copy(), th.copy()
        tp[i] += h
        tm[i] -= h
        fp = e.exact_eval("rbf", True, tp[0], tp[1:-1], tp[-1])[0]
        fm = e.exact_eval("rbf", True, tm[0], tm[1:-1], tm[-1])[0]
        fd = (fp - fm) / (2 * h)
        assert abs(fd - g[i]) <= 2e-5 * abs(g[i]), (i, fd, g[i])
    lml_again, g_again, _ = e.exact_eval("rbf", True, var, ls, noise)
    assert lml_again == lml and np.array_equal(g_again, g)     # deterministic: fixed-order reductions
    alpha = e.get("alpha")
    rows = np.arange(0, N, 257)
    Krows = _ffi.kern_K("rbf", True, var, ls, X[rows], X)
    resid = Krows.dot(alpha) + (noise + 1e-8) * alpha[rows] - Y[rows]
    assert np.max(np.abs(resid)) < 1e-8
    perm = np.random.default_rng(0).permutation(N)
    e.set_data(X[perm], Y[perm])
    lml_p, g_p, _ = e.exact_eval("rbf", True, var, ls, noise)
    assert abs(lml_p - lml) <= 1e-7
    np.testing.assert_allclose(g_p, g, rtol=1e-8)
    e.close()


def test_pdinv_and_jitchol_on_device():
    """GPy/util/linalg.py:56-75,193-214 as stand-alone device calls (gpx_pdinv); same fixture as
    GPy/testing/test_linalg.py:8-37: the corrupted matrix needs exactly five rounds of jitter."""
    from test_oracle import _corrupt
    A = _corrupt(0)
    L = _ffi.jitchol(A, maxtries=5)
    diff = L.dot(L.T) - A
    np.testing.assert_allclose(diff, np.eye(20) * np.diag(diff).mean(), atol=1e-12)
    L0, jit0 = o.jitchol(A, maxtries=5)
    np.testing.assert_allclose(np.diag(diff).mean(), jit0, rtol=1e-6)
    with pytest.raises(np.linalg.LinAlgError):
        _ffi.jitchol(A, maxtries=4)
    Aneg = A.copy()
    Aneg[3, 3] = -1.0
    with pytest.raises(np.linalg.LinAlgError):
        _ffi.jitchol(Aneg)
    rng = np.random.default_rng(1)
    for n in (5, 128, 300, 1111):
        B = rng.standard_normal((n, n + 10))
        S = B.dot(B.T) + n * np.eye(n)
        Ai, L, Li, logdet, jit = _ffi.pdinv(S)
        Ai0, L0, Li0, logdet0 = o.pdinv(S)
        assert jit == 0.0 and abs(logdet - logdet0) < 1e-9 * abs(logdet0)
        assert rel(L, L0) < 1e-12 and rel(Li, Li0) < 1e-11 and rel(Ai, Ai0) < 1e-11


def test_inference_generic_path_mean_function_and_precomputed_K():
    """exact_gaussian_inference.py:42-53: mean_function and K= arguments (off the fused path, still on the device for
    the N^3 part)."""
    rng = np.random.default_rng(5)
    X = rng.uniform(-3, 3, (150, 2))
    Y = np.sin(X[:, :1]) + 0.3 * X[:, 1:] + 0.05 * rng.standard_normal((150, 1))

    class LinMean(object):
        def f(self, X):
            return 0.3 * X[:, 1:2]

    k = gpy_b200.RBF(2, variance=1.2, lengthscale=[1.0, 2.0], ARD=True)
    lik = gpy_b200.Gaussian(variance=0.05)
    inf = gpy_b200.ExactGaussianInference()
    post, lml, gd = inf.inference(k, X, lik, Y, mean_function=LinMean())
    ko = o.StationaryOracle("rbf", 2, 1.2, [1.0, 2.0], True)
    res = o.exact_inference(ko, X, Y - 0.3 * X[:, 1:2], 0.05)
    assert abs(lml - res["log_marginal"]) < 1e-8
    assert rel(gd["dL_dK"], res["dL_dK"]) < 1e-9 and rel(gd["dL_dm"], res["alpha"]) < 1e-9
    post2, lml2, gd2 = inf.inference(k, X, lik, Y, K=ko.K(X))
    res2 = o.exact_inference(ko, X, Y, 0.05)
    assert abs(lml2 - res2["log_marginal"]) < 1e-8 and rel(post2.woodbury_chol, res2["L"]) < 1e-11
    m = gpy_b200.GPRegression(X, Y, k, noise_var=0.05, mean_function=LinMean())
    assert abs(m.log_likelihood() - res["log_marginal"]) < 1e-8
    mu, var = m.predict(X[:4])
    mu0, var0 = o.predict(ko, X, res["L"], res["alpha"], X[:4], 0.05)
    np.testing.assert_allclose(mu, mu0 + 0.3 * X[:4, 1:2], rtol=1e-8, atol=1e-9)
    np.testing.assert_allclose(var, var0, rtol=1e-7, atol=1e-9)


@pytest.mark.parametrize("kind", o.KINDS)
@pytest.mark.parametrize("ARD", [False, True])
def test_gradients_X(kind, ARD):
    """Stationary.gradients_X (stationary.py:245-252; native helper stationary_utils.c:1-14), fixtures of
    GPy/testing/test_cython.py:57-81: square (300 x 300) and rectangular (300 x 20) dL_dK."""
    rng = np.random.default_rng(11)
    for (n, m, d) in ((300, 20, 10), (257, 131, 3), (40, 700, 5)):
        X, Z = rng.standard_normal((n, d)), rng.standard_normal((m, d))
        ls = rng.uniform(0.8, 2.0, d) if ARD else float(rng.uniform(0.8, 2.0))
        cls = {"rbf": gpy_b200.RBF, "exponential": gpy_b200.Exponential, "matern32": gpy_b200.Matern32,
               "matern52": gpy_b200.Matern52}[kind]
        k = cls(d, variance=0.7, lengthscale=ls, ARD=ARD)
        ko = o.StationaryOracle(kind, d, 0.7, ls, ARD)
        dKxx, dKxz = rng.standard_normal((n, n)), rng.standard_normal((n, m))
        np.testing.assert_allclose(k.gradients_X(dKxx, X), ko.gradients_X(dKxx, X), rtol=1e-9, atol=1e-11)
        np.testing.assert_allclose(k.gradients_X(dKxz, X, Z), ko.gradients_X(dKxz, X, Z), rtol=1e-9, atol=1e-11)


def test_combination_and_static_kernels():
    """GPy/kern/src/add.py:60-86, prod.py:59-110, static.py:63-185 through the mirror: K, gradients and a full
    GPRegression evaluation (generic inference path: device-built parts + gpx_pdinv) against oracle-built references."""
    rng = np.random.default_rng(8)
    X = rng.uniform(-3, 3, (120, 3))
    Y = np.sin(X[:, :1]) + 0.1 * rng.standard_normal((120, 1))
    k1 = gpy_b200.RBF(3, variance=1.1, lengthscale=[1.0, 1.5, 2.0], ARD=True)
    k2 = gpy_b200.Matern32(2, variance=0.6, lengthscale=1.3, active_dims=[0, 2])
    o1 = o.StationaryOracle("rbf", 3, 1.1, [1.0, 1.5, 2.0], True)
    o2 = o.StationaryOracle("matern32", 2, 0.6, 1.3, False)
    Xs2 = X[:, [0, 2]]
    ksum = k1 + k2 + gpy_b200.White(3, variance=0.2) + gpy_b200.Bias(3, variance=0.3)
    Ksum0 = o1.K(X) + o2.K(Xs2) + 0.2 * np.eye(120) + 0.3
    assert isinstance(ksum, gpy_b200.Add) and len(ksum.parts) == 4
    assert rel(ksum.K(X), Ksum0) < 1e-13
    kprod = k1 * k2
    assert rel(kprod.K(X), o1.K(X) * o2.K(Xs2)) < 1e-13
    dL = rng.standard_normal((120, 120))
    kprod.update_gradients_full(dL, X)
    v1, l1 = o1.update_gradients_full(dL * o2.K(Xs2), X)
    v2, l2 = o2.update_gradients_full(dL * o1.K(X), Xs2)
    np.testing.assert_allclose(k1.variance.gradient, v1, rtol=1e-9)
    np.testing.assert_allclose(k1.lengthscale.gradient, l1, rtol=1e-9)
    np.testing.assert_allclose(k2.variance.gradient, v2, rtol=1e-9)
    np.testing.assert_allclose(k2.lengthscale.gradient, l2, rtol=1e-9)
    # GPRegression with the sum kernel: LML against a direct dense computation, gradient against finite differences
    m = gpy_b200.GPRegression(X, Y, ksum, noise_var=0.05)
    Ky = Ksum0 + (0.05 + 1e-8) * np.eye(120)
    L = np.linalg.cholesky(Ky)
    alpha = np.linalg.solve(Ky, Y)
    lml0 = 0.5 * (-120 * o.LOG_2_PI - 2 * np.log(np.diag(L)).sum() - float(np.squeeze(Y.T.dot(alpha))))
    assert abs(m.log_likelihood() - lml0) < 1e-8
    assert len(m.gradient) == 1 + 3 + 1 + 1 + 1 + 1 + 1 and m.checkgrad()


@pytest.mark.parametrize("kind,ARD,N,M,D,P", [("rbf", True, 700, 40, 3, 1), ("matern52", False, 1500, 300, 4, 2),
                                               ("exponential", True, 2100, 129, 2, 1), ("matern32", True, 600, 600, 5, 1)])
def test_sparse_gp_vardtc(kind, ARD, N, M, D, P):
    """Sparse GP regression (VarDTC, GPy/inference/latent_function_inference/var_dtc.py:66-215 + core/sparse_gp.py:108-119)
    through the mirror: bound, kernel / noise gradients, inducing-point gradients and predictions against the oracle
    (which is pinned to the unmodified reference VarDTC, tests/test_reference_crosscheck.py)."""
    rng = np.random.default_rng(N + M)
    X = rng.uniform(-3, 3, (N, D))
    Y = np.stack([np.sin(X).sum(1) / np.sqrt(D) + 0.1 * rng.standard_normal(N) for _ in range(P)], 1)
    Z = X[rng.permutation(N)[:M]].copy() + 0.01 * rng.standard_normal((M, D))
    ls = np.sqrt(D) * rng.uniform(0.7, 1.3, D) if ARD else float(np.sqrt(D) * 0.9)
    cls = {"rbf": gpy_b200.RBF, "exponential": gpy_b200.Exponential, "matern32": gpy_b200.Matern32,
           "matern52": gpy_b200.Matern52}[kind]
    k = cls(D, variance=1.3, lengthscale=ls, ARD=ARD)
    m = gpy_b200.SparseGPRegression(X, Y, kernel=k, Z=Z)
    m.likelihood.variance.values[...] = 0.05
    m.parameters_changed()
    lml0, g0, Zg0, res = o.sparse_eval(X, Y, Z, kind, ARD, 1.3, ls, 0.05)
    np.testing.assert_allclose(m.posterior.woodbury_vector, res["woodbury_vector"], rtol=1e-6, atol=1e-7)
    np.testing.assert_allclose(m.posterior.woodbury_inv, res["woodbury_inv"], rtol=1e-4,
                               atol=1e-6 * np.abs(res["woodbury_inv"]).max())
    Kmm0 = o.StationaryOracle(kind, D, 1.3, ls, ARD).K(Z) + 1e-8 * np.eye(M)
    np.testing.assert_allclose(m.posterior.K, Kmm0, rtol=1e-12, atol=1e-12)
    Lm = np.tril(m.posterior.K_chol)
    np.testing.assert_allclose(Lm.dot(Lm.T), Kmm0, rtol=1e-9, atol=1e-10)
    assert abs(m.log_likelihood() - lml0) <= 1e-8 * max(1.0, abs(lml0))
    g = np.concatenate([k.variance.gradient, k.lengthscale.gradient, m.likelihood.variance.gradient])
    np.testing.assert_allclose(g, g0, rtol=1e-6, atol=1e-8)
    np.testing.assert_allclose(m.Z.gradient, Zg0, rtol=1e-6, atol=1e-8)
    Xn = rng.uniform(-3, 3, (11, D))
    mu, var = m.predict(Xn, include_likelihood=False)
    ko = o.StationaryOracle(kind, D, 1.3, ls, ARD)
    mu0, var0 = o.sparse_raw_predict(ko, Z, res["woodbury_vector"], res["woodbury_inv"], Xn)
    np.testing.assert_allclose(mu, mu0, rtol=1e-6, atol=1e-8)
    np.testing.assert_allclose(var, var0, rtol=1e-5, atol=1e-8)
    if N <= 700:
        assert m.checkgrad(step=1e-5)   # 1e-6 drowns the O(1e-2) inducing-point gradients in fp64 round-off of the bound


@pytest.mark.parametrize("kind,ARD,N,D,P", [("rbf", True, 300, 3, 1), ("matern52", False, 700, 2, 2), ("exponential", True, 129, 4, 1)])
def test_heteroscedastic_noise(kind, ARD, N, D, P):
    """One noise variance per data point (HeteroscedasticGaussian, likelihoods/gaussian.py:347-362): gpx_exact_eval_het
    against the oracle (pinned to the reference's own objects in tests/test_reference_crosscheck.py): LML, kernel
    gradients, the N per-point noise gradients diag(dL_dK), alpha."""
    rng = np.random.default_rng(N)
    X = rng.uniform(-3, 3, (N, D))
    Y = np.stack([np.sin(X).sum(1) + 0.2 * rng.standard_normal(N) for _ in range(P)], 1)
    ls = rng.uniform(0.8, 2.0, D) if ARD else 1.3
    nv = rng.uniform(0.01, 0.3, N)
    lml0, g0, res = o.eval_lml_grad(X, Y, kind, ARD, 1.4, ls, nv)
    e = _ffi.Engine(0)
    e.set_data(X, Y)
    lml, g, dn, _ = e.exact_eval_het(kind, ARD, 1.4, ls, nv)
    nl = D if ARD else 1
    assert abs(lml - lml0) <= LML_ATOL
    np.testing.assert_allclose(g[:1 + nl], g0[:1 + nl], rtol=GRAD_RTOL, atol=1e-9)
    np.testing.assert_allclose(dn, g0[1 + nl:], rtol=GRAD_RTOL, atol=1e-9)
    assert abs(g[-1] - dn.sum()) <= 1e-9 * max(1.0, np.abs(dn).sum())
    assert rel(e.get("alpha"), res["alpha"]) < 1e-9
    # the homoscedastic call on the same context afterwards is unaffected
    lml1, g1, _ = e.exact_eval(kind, ARD, 1.4, ls, 0.1)
    lml2, g2, _ = o.eval_lml_grad(X, Y, kind, ARD, 1.4, ls, 0.1)
    assert abs(lml1 - lml2) <= LML_ATOL
    np.testing.assert_allclose(g1, g2, rtol=GRAD_RTOL, atol=1e-9)
    e.close()


def test_mixed_noise_model():
    """MixedNoise (likelihoods/mixed_noise.py:14-53) through the heteroscedastic device path: one Gaussian per output index;
    parameter vector [variance, lengthscale, noise_0, noise_1], LML / gradients against the oracle (pinned to the reference's
    MixedNoise objects in tests/test_reference_crosscheck.py), gradient check, prediction with Y_metadata."""
    rng = np.random.default_rng(11)
    N, D = 300, 2
    X, Y = o.synthetic(N, D, 21)
    idx = rng.integers(0, 2, N)
    md = {"output_index": idx[:, None]}
    lik = gpy_b200.MixedNoise([gpy_b200.Gaussian(0.04), gpy_b200.Gaussian(0.25)])
    m = gpy_b200.GP(X, Y, gpy_b200.RBF(D, variance=1.2, lengthscale=[1.1, 1.9], ARD=True), lik, Y_metadata=md)
    nv = np.array([0.04, 0.25])[idx]
    lml0, g0, res = o.eval_lml_grad(X, Y, "rbf", True, 1.2, np.array([1.1, 1.9]), nv)
    assert abs(m.log_likelihood() - lml0) <= LML_ATOL
    dn = g0[1 + D:]
    want = np.concatenate([g0[:1 + D], [dn[idx == 0].sum(), dn[idx == 1].sum()]])
    assert len(m.gradient) == 1 + D + 2
    np.testing.assert_allclose(m.gradient, want, rtol=GRAD_RTOL, atol=1e-9)
    assert m.checkgrad()
    Xn = rng.uniform(-2, 2, (6, D))
    mdn = {"output_index": np.array([0, 1, 1, 0, 0, 1])[:, None]}
    mu, var = m.predict(Xn, Y_metadata=mdn)
    ko = o.StationaryOracle("rbf", D, 1.2, np.array([1.1, 1.9]), True)
    mu0, var0 = o.raw_predict(ko, X, res["L"], res["alpha"], Xn)
    np.testing.assert_allclose(mu, mu0, rtol=1e-7, atol=1e-9)
    np.testing.assert_allclose(var, var0 + np.array([0.04, 0.25])[mdn["output_index"]], rtol=1e-7, atol=1e-9)


def test_sparse_golden_fixtures():
    """tests/golden/sparse/*.npz: bound, gradients and inducing-input gradients produced by the reference's own VarDTC."""
    gdir = os.path.join(os.path.dirname(__file__), "golden", "sparse")
    files = sorted(f for f in os.listdir(gdir) if f.endswith(".npz"))
    assert files
    for fn in files:
        z = np.load(os.path.join(gdir, fn))
        kind, ARD, D = str(z["kind"]), bool(z["ARD"]), z["X"].shape[1]
        ls = z["lengthscale"] if ARD else float(z["lengthscale"])
        cls = {"rbf": gpy_b200.RBF, "exponential": gpy_b200.Exponential, "matern32": gpy_b200.Matern32,
               "matern52": gpy_b200.Matern52}[kind]
        k = cls(D, variance=float(z["variance"]), lengthscale=ls, ARD=ARD)
        m = gpy_b200.SparseGPRegression(z["X"], z["Y"], kernel=k, Z=z["Z"])
        m.likelihood.variance.values[...] = float(z["noise"])
        m.parameters_changed()
        lml0 = float(z["lml"])
        assert abs(m.log_likelihood() - lml0) <= 1e-8 * max(1.0, abs(lml0)), fn
        g = np.concatenate([k.variance.gradient, k.lengthscale.gradient, m.likelihood.variance.gradient])
        np.testing.assert_allclose(g, z["grad"], rtol=1e-6, atol=1e-8, err_msg=fn)
        # dL/dZ is the worst-conditioned output: for the Matern-5/2 fixture cond(Kmm) = 2e8 and the reference's own fp64
        # result differs from an extended-precision evaluation of the same formulas by 7.7e-8 (2e-8 of max|dL/dZ|);
        # (reproduce: python tools/sparse_dz_extended_precision.py);
        # hence the absolute floor relative to the largest entry
        np.testing.assert_allclose(m.Z.gradient, z["Zgrad"], rtol=1e-6, atol=1e-7 * np.abs(z["Zgrad"]).max(), err_msg=fn)
        np.testing.assert_allclose(m.posterior.woodbury_vector, z["woodbury_vector"], rtol=1e-6, atol=1e-7, err_msg=fn)


def test_heteroscedastic_golden_fixtures(eng):
    """tests/golden/het/*.npz: numbers produced by the reference's own HeteroscedasticGaussian + ExactGaussianInference."""
    gdir = os.path.join(os.path.dirname(__file__), "golden", "het")
    files = sorted(f for f in os.listdir(gdir) if f.endswith(".npz"))
    assert files
    for fn in files:
        z = np.load(os.path.join(gdir, fn))
        kind, ARD = str(z["kind"]), bool(z["ARD"])
        ls = z["lengthscale"] if ARD else float(z["lengthscale"])
        eng.set_data(z["X"], z["Y"])
        lml, g, dn, _ = eng.exact_eval_het(kind, ARD, float(z["variance"]), ls, z["noise_variances"])
        nk = z["grad"].size - z["noise_variances"].size
        assert abs(lml - float(z["lml"])) <= LML_ATOL, fn
        np.testing.assert_allclose(np.concatenate([g[:nk], dn]), z["grad"], rtol=GRAD_RTOL, atol=1e-9, err_msg=fn)
        assert rel(eng.get("alpha"), z["alpha"]) < 1e-8, fn


def test_heteroscedastic_model():
    """gpy_b200.GPHeteroscedasticRegression (models/gp_heteroscedastic_regression.py:10-37): parameter vector
    [variance, lengthscale, N noise variances], gradient check, prediction with Y_metadata."""
    rng = np.random.default_rng(5)
    N = 40
    X = rng.uniform(-3, 3, (N, 1))
    Y = np.sin(X) + rng.standard_normal((N, 1)) * (0.05 + 0.2 * (X > 0))
    m = gpy_b200.GPHeteroscedasticRegression(X, Y, gpy_b200.Matern32(1, lengthscale=1.2))
    m.likelihood.variance.values[...] = rng.uniform(0.02, 0.2, N)
    m.parameters_changed()
    assert len(m.gradient) == 1 + 1 + N
    lml0, g0, res = o.eval_lml_grad(X, Y, "matern32", False, 1.0, 1.2, m.likelihood.variance.values.copy())
    assert abs(m.log_likelihood() - lml0) <= LML_ATOL
    np.testing.assert_allclose(m.gradient, g0, rtol=GRAD_RTOL, atol=1e-9)
    assert m.checkgrad(step=1e-5)
    Xn = rng.uniform(-3, 3, (5, 1))
    mu, var = m.predict(Xn, Y_metadata={"output_index": np.arange(5)[:, None]})
    mu0, var0 = o.raw_predict(o.StationaryOracle("matern32", 1, 1.0, 1.2, False), X, res["L"], res["alpha"], Xn)
    np.testing.assert_allclose(mu, mu0, rtol=1e-8, atol=1e-10)
    np.testing.assert_allclose(var, var0 + m.likelihood.variance.values[:5].reshape(-1, 1), rtol=1e-7, atol=1e-10)
    d = m.optimize(max_iters=15)
    assert np.isfinite(m.log_likelihood()) and m.log_likelihood() >= lml0 - 1e-6


def test_sparse_engine_reuse_with_fewer_points():
    """The same context evaluated first with (N, M) = (700, 130) and then with (690, 129): same padded extents, so the
    psi1 buffers must be re-zeroed beyond the new N and M (stale entries would enter the k-ranges of the GEMMs)."""
    rng = np.random.default_rng(9)
    e = _ffi.Engine(0)
    for (N, M) in ((700, 130), (690, 129), (700, 130)):
        X = rng.uniform(-3, 3, (N, 3))
        Y = np.sin(X).sum(1, keepdims=True) + 0.1 * rng.standard_normal((N, 1))
        Z = X[rng.permutation(N)[:M]].copy() + 0.01 * rng.standard_normal((M, 3))
        ls = np.array([1.4, 1.9, 2.2])
        e.sparse_set_data(X, Y)
        lml, g, dZ = e.sparse_eval("matern32", True, 1.1, ls, Z, 0.06)
        lml0, g0, Zg0, _ = o.sparse_eval(X, Y, Z, "matern32", True, 1.1, ls, 0.06)
        assert abs(lml - lml0) <= 1e-8 * max(1.0, abs(lml0)), (N, M)
        np.testing.assert_allclose(g, g0, rtol=1e-6, atol=1e-8)
        np.testing.assert_allclose(dZ, Zg0, rtol=1e-6, atol=1e-7 * np.abs(Zg0).max())
    e.close()


@pytest.mark.parametrize("d", [20, 40, 64])
def test_kernel_gradient_reductions_large_input_dimension(d):
    """update_gradients_full / gradients_X with 16 < D <= 64 (the register-resident ARD sums are instantiated for 8, 16, 32
    and 64 dimensions; the fused evaluation is covered at D=64 by test_multiple_outputs_and_large_D)."""
    rng = np.random.default_rng(d)
    n, m = 150, 70
    X, X2 = rng.standard_normal((n, d)), rng.standard_normal((m, d))
    ls = np.sqrt(d) * rng.uniform(0.8, 1.6, d)
    k = gpy_b200.Matern52(d, variance=0.9, lengthscale=ls, ARD=True)
    ko = o.StationaryOracle("matern52", d, 0.9, ls, True)
    for XX2, shape in ((None, (n, n)), (X2, (n, m))):
        dL = rng.standard_normal(shape)
        k.update_gradients_full(dL, X, XX2)
        v0, l0 = ko.update_gradients_full(dL, X, XX2)
        np.testing.assert_allclose(k.variance.gradient, v0, rtol=1e-10)
        np.testing.assert_allclose(k.lengthscale.gradient, l0, rtol=1e-9, atol=1e-12)
        gx = k.gradients_X(dL, X, XX2)
        np.testing.assert_allclose(gx, ko.gradients_X(dL, X, XX2), rtol=1e-9, atol=1e-12)


def _composite_case(D=5):
    k = gpy_b200.Add([gpy_b200.Prod([gpy_b200.RBF(2, variance=1.2, lengthscale=[1.0, 2.0], ARD=True, active_dims=[0, 1]),
                                     gpy_b200.Matern32(2, variance=0.8, lengthscale=1.5, active_dims=[2, 3])]),
                      gpy_b200.Matern52(D, variance=0.5, lengthscale=np.linspace(1.5, 2.5, D), ARD=True),
                      gpy_b200.Exponential(1, variance=0.3, lengthscale=2.0, active_dims=[4]),
                      gpy_b200.White(D, variance=0.05), gpy_b200.Bias(D, variance=0.3)])
    parts = [dict(kind="rbf", term=0, dims=[0, 1], variance=1.2, lengthscale=np.array([1.0, 2.0]), ARD=True),
             dict(kind="matern32", term=0, dims=[2, 3], variance=0.8, lengthscale=1.5, ARD=False),
             dict(kind="matern52", term=1, dims=list(range(D)), variance=0.5, lengthscale=np.linspace(1.5, 2.5, D), ARD=True),
             dict(kind="exponential", term=2, dims=[4], variance=0.3, lengthscale=2.0, ARD=False),
             dict(kind="white", term=3, dims=None, variance=0.05), dict(kind="bias", term=4, dims=None, variance=0.3)]
    return k, parts


@pytest.mark.parametrize("N", [150, 700, 1300])
def test_composite_kernels_on_the_fused_device_path(N):
    """Sum / product / White / Bias kernels (add.py:60-99, prod.py:59-68,377-396, static.py:63-185) through
    gpx_exact_eval_multi: LML, every part's gradient, alpha, K and predictions against the oracle. N = 700 / 1300 force
    option ozaki = 1 and take the int8 (Ozaki) sweep with the stored K^-1; N = 150 is a single block and takes the DMMA
    sweep + plain LAUUM. The default (DMMA) path on several blocks is tests/test_gpu_routes.py::test_route_matrix_composite."""
    D = 5
    X, Y = o.synthetic(N, D, seed=N)
    k, parts = _composite_case(D)
    eng = _ffi.Engine(0)
    eng.set_option("ozaki", 1 if N >= 700 else 0)     # N = 150: one panel only, DMMA path with the plain K^-1 store
    m = gpy_b200.GPRegression(X, Y, k, noise_var=0.04, engine=eng)
    lml0, g0, res = o.composite_eval_lml_grad(X, Y, parts, 0.04)
    assert abs(m.log_likelihood() - lml0) <= LML_ATOL
    np.testing.assert_allclose(m.gradient, g0, rtol=GRAD_RTOL, atol=1e-9)
    assert rel(m.posterior.woodbury_vector, res["alpha"]) < 1e-9
    if N <= 700:
        assert rel(m.posterior.K, res["K"]) < 1e-12
        assert rel(m.posterior.woodbury_chol, res["L"]) < 1e-10
    Xn = np.random.default_rng(N).uniform(-3, 3, (9, D))
    Kx = o.composite_K(res["kparts"], X, Xn)
    tmp = o.dtrtrs(res["L"], Kx, lower=1)[0]
    mu, var = m.predict(Xn, include_likelihood=False)
    np.testing.assert_allclose(mu, Kx.T @ res["alpha"], rtol=1e-8, atol=1e-10)
    np.testing.assert_allclose(var[:, 0], o.composite_Kdiag(res["kparts"], Xn) - np.square(tmp).sum(0), rtol=1e-7, atol=1e-9)
    mu2, cov = m.predict(Xn, full_cov=True, include_likelihood=False)
    np.testing.assert_allclose(cov, o.composite_K(res["kparts"], Xn) - tmp.T @ tmp, rtol=1e-7, atol=1e-9)
    if N == 150:
        assert m.checkgrad()
        f0 = m.objective_function()
        m.optimize(max_iters=10)
        assert m.objective_function() < f0
    # a single-kernel evaluation on the same context afterwards is unaffected
    eng = m.inference_method.engine
    lml1, g1, _ = eng.exact_eval("rbf", False, 1.1, 1.7, 0.05)
    lml2, g2, _ = o.eval_lml_grad(X, Y, "rbf", False, 1.1, 1.7, 0.05)
    assert abs(lml1 - lml2) <= LML_ATOL
    np.testing.assert_allclose(g1, g2, rtol=GRAD_RTOL, atol=1e-9)


@pytest.mark.parametrize("oz", [0, 1])
def test_tensor_path_selection_gives_the_same_answer(oz):
    """option ozaki = 0 (fp64 DMMA GEMMs) and 1 (wgmma int8 digit-split GEMMs) both meet the tolerances against the
    oracle, on a size with several panels, a non-multiple-of-block tail and P = 2 outputs."""
    rng = np.random.default_rng(3)
    N, D = 1700, 6
    X = rng.uniform(-3, 3, (N, D))
    Y = np.stack([np.sin(X).sum(1) / np.sqrt(D) + 0.1 * rng.standard_normal(N) for _ in range(2)], 1)
    var, ls, noise = 1.3, np.sqrt(D) * np.linspace(0.8, 1.4, D), 0.02
    lml0, g0, res = o.eval_lml_grad(X, Y, "matern52", True, var, ls, noise)
    e = _ffi.Engine(0)
    e.set_option("ozaki", oz)
    e.set_data(X, Y)
    lml, g, _ = e.exact_eval("matern52", True, var, ls, noise)
    assert abs(lml - lml0) <= LML_ATOL
    np.testing.assert_allclose(g, g0, rtol=GRAD_RTOL, atol=1e-9)
    assert rel(e.get("alpha"), res["alpha"]) < 1e-9
    assert rel(e.get("Kinv"), res["Wi"]) < 1e-8
    assert rel(e.get("L"), res["L"]) < 1e-10
    e.close()
