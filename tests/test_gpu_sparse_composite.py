"""Sparse GP regression (VarDTC) with composite kernels on the device (gpx_sparse_eval_multi): against the reference
fixtures of tests/golden/sparse_composite and the NumPy restatement of tests/sparse_composite_oracle.py, the mirror model
end to end, metamorphic identities at the benchmark's shape, the single-kernel evaluations around a composite one, launch
accounting and the rejections. Tolerances are those of tests/test_gpu_sparse_routes.py."""
import glob
import os

import numpy as np
import pytest

import gpy_b200
import sparse_composite_oracle as so
from gpy_b200 import _ffi

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = sorted(glob.glob(os.path.join(HERE, "golden", "sparse_composite", "*.npz")))
LML_RTOL = 1e-8
GRAD_RTOL = 1e-6
MAXNORM_FLOOR = 1e-7


def _close_maxnorm(a, b, what):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    err = np.abs(a - b).max()
    assert err <= MAXNORM_FLOOR * max(np.abs(b).max(), 1e-300), (what, err, np.abs(b).max())


def _check(out, lml, grad, Zg, dR=None):
    assert abs(out[0] - lml) <= LML_RTOL * abs(lml), (out[0], lml)
    np.testing.assert_allclose(out[1], grad, rtol=GRAD_RTOL, atol=1e-9 * np.abs(grad).max())
    _close_maxnorm(out[2], Zg, "dZ")
    if dR is not None:
        _close_maxnorm(out[3], dR, "dL_dR")


def _descs(parts):
    return [so.descriptor(p) for p in parts]


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[:-4])
def test_device_matches_the_reference_fixtures(path):
    f = np.load(path)
    noise = f["noise"]
    noise = float(noise) if noise.ndim == 0 else noise
    e = _ffi.Engine(0)
    try:
        e.sparse_set_data(f["X"], f["Y"])
        out = e.sparse_eval_multi(_descs(so.KERNELS[str(f["kernel"])]), f["Z"], noise)
        _check(out, float(f["lml"]), f["grad"], f["Zgrad"], f["dL_dR"] if "dL_dR" in f.files else None)
        _close_maxnorm(e.sparse_get("woodbury_vector"), f["woodbury_vector"], "woodbury_vector")
        _close_maxnorm(e.sparse_get("woodbury_inv"), f["woodbury_inv"], "woodbury_inv")
    finally:
        e.close()


@pytest.mark.parametrize("M", [50, 129, 300])
def test_device_matches_the_oracle_on_one_to_three_kmm_blocks(M):
    """nb = 128: Kmm on 1, 2 and 3 blocks; every kernel, both noise forms, P = 2 for one kernel"""
    e = _ffi.Engine(0)
    e.set_option("nb", 128)
    try:
        for i, kname in enumerate(sorted(so.KERNELS)):
            P = 2 if i == 1 else 1
            for het in (False, True):
                X, Y, Z, noise = so.case_data(1000, M, 3, P, 40 + i + M, het)
                e.sparse_set_data(X, Y)
                out = e.sparse_eval_multi(_descs(so.KERNELS[kname]), Z, noise)
                lml, grad, Zg, res = so.sparse_composite_eval(X, Y, Z, so.KERNELS[kname], noise)
                _check(out, lml, grad, Zg, res["dL_dthetaL"] if het else None)
                _close_maxnorm(e.sparse_get("Kmm"), res["Kmm"], "Kmm")
                _close_maxnorm(e.sparse_get("Lm"), res["Lm"], "Lm")
    finally:
        e.close()


def _mirror_kernel():
    K = gpy_b200.kern
    return K.Add([K.Prod([K.Matern52(2, variance=1.1, lengthscale=1.2, active_dims=[0, 1]),
                          K.RBF(2, variance=0.8, lengthscale=[1.5, 0.7], ARD=True, active_dims=[1, 2])]),
                  K.Exponential(1, variance=0.3, lengthscale=2.5, active_dims=[0]),
                  K.White(3, variance=0.05)])


def test_mirror_model_posterior_predictions_checkgrad_and_optimize():
    X, Y, Z, _ = so.case_data(1100, 129, 3, 1, 51, False)
    m = gpy_b200.SparseGPRegression(X, Y, kernel=_mirror_kernel(), Z=Z)
    m.inference_method.engine.set_option("nb", 128)
    m.likelihood.variance[:] = 0.08
    parts = so.KERNELS["m52_x_rbf_plus_exp"] + [dict(kind="white", term=2, variance=0.05)]
    lml, grad, Zg, res = so.sparse_composite_eval(X, Y, Z, parts, 0.08)
    assert abs(m.log_likelihood() - lml) <= LML_RTOL * abs(lml)
    g = np.concatenate([np.asarray(p.gradient, dtype=np.float64).reshape(-1) for p in m.flattened_parameters()])
    np.testing.assert_allclose(g[Z.size:], grad, rtol=GRAD_RTOL, atol=1e-9 * np.abs(grad).max())
    _close_maxnorm(g[:Z.size].reshape(Z.shape), Zg, "Z.gradient")
    post = m.posterior
    _close_maxnorm(post.woodbury_vector, res["woodbury_vector"], "woodbury_vector")
    _close_maxnorm(post.woodbury_inv, res["woodbury_inv"], "woodbury_inv")
    _close_maxnorm(post.K, res["Kmm"], "Kmm")
    _close_maxnorm(post.K_chol, res["Lm"], "Lm")
    Xn = np.random.default_rng(3).uniform(-2, 2, (40, 3))
    kern = so.CompositeOracle(parts)
    Kx = kern.K(Z, Xn)
    mu0 = Kx.T @ res["woodbury_vector"]
    for full_cov in (False, True):
        mu, var = m.predict(Xn, full_cov=full_cov, include_likelihood=False)
        if full_cov:
            var0 = kern.K(Xn) - Kx.T @ res["woodbury_inv"] @ Kx
        else:
            var0 = (kern.Kdiag(Xn) - np.sum((res["woodbury_inv"].T @ Kx) * Kx, 0))[:, None]
        _close_maxnorm(mu, mu0, "mu")
        _close_maxnorm(var, var0, "var full_cov=%s" % full_cov)
    assert m.checkgrad(step=1e-5, tolerance=1e-3, sample=8)
    l0 = m.log_likelihood()
    m.optimize(max_iters=10)
    assert m.log_likelihood() > l0


def test_benchmark_shape_metamorphic():
    """N = 262144, M = 4096, D = 16: RBF(ARD) x Bias(1) is RBF(ARD), and RBF(a, l) + RBF(b, l) is RBF(a + b, l). With
    a = b the two covariances agree to the bit (a k + a k = 2 (a k) = (2 a) k in binary floating point), so that only the
    order of the reductions differs; unequal a, b would perturb Kmm in its last bits, and cond(Kmm) carries that into the
    gradients at about 1e-10."""
    rng = np.random.default_rng(11)
    N, M, D = 262144, 4096, 16
    X = rng.standard_normal((N, D))
    Y = (np.sin(X[:, :3]).sum(1) + 0.1 * rng.standard_normal(N))[:, None]
    Z = X[rng.permutation(N)[:M]] + 0.01 * rng.standard_normal((M, D))
    ls = np.linspace(2.0, 5.0, D)
    dims = list(range(D))
    e = _ffi.Engine(0)

    def rel(a, b):   # entry by entry
        return float(np.max(np.abs(np.asarray(a) - np.asarray(b)) / np.abs(np.asarray(b))))

    def maxrel(a, b):   # dL/dZ: of its largest entry
        return np.abs(a - b).max() / np.abs(b).max()

    try:
        e.sparse_set_data(X, Y)
        l1, g1, z1 = e.sparse_eval("rbf", True, 1.3, ls, Z, 0.05)
        lp, gp, zp = e.sparse_eval_multi([("rbf", True, 0, dims, 1.3, ls), ("bias", False, 0, [], 1.0, None)], Z, 0.05)
        print("\nRBF(ARD) x Bias(1): bound %.1e grad %.1e dZ %.1e" % (
            rel(lp, l1), rel(np.r_[gp[:1 + D], gp[-1]], np.r_[g1[:1 + D], g1[-1]]), maxrel(zp, z1)))
        assert rel(lp, l1) <= 1e-10
        assert rel(gp[:1 + D], g1[:1 + D]) <= 1e-10 and rel(gp[-1], g1[-1]) <= 1e-10
        assert maxrel(zp, z1) <= 1e-10
        a, b, l = 0.65, 0.65, 3.0
        l2, g2, z2 = e.sparse_eval("rbf", False, a + b, l, Z, 0.05)
        ls_, gs, zs = e.sparse_eval_multi([("rbf", False, 0, dims, a, l), ("rbf", False, 1, dims, b, l)], Z, 0.05)
        print("RBF(a, l) + RBF(a, l): bound %.1e grad %.1e dZ %.1e" % (
            rel(ls_, l2), rel([gs[0], gs[2], gs[1] + gs[3], gs[4]], [g2[0], g2[0], g2[1], g2[2]]), maxrel(zs, z2)))
        assert rel(ls_, l2) <= 1e-10
        # d/da = d/db = d/dvariance; the lengthscale gradients split as a : b; the noise gradient is the same
        assert rel(gs[0], g2[0]) <= 1e-10 and rel(gs[2], g2[0]) <= 1e-10
        assert rel(gs[1] + gs[3], g2[1]) <= 1e-10 and rel(gs[1], g2[1] * a / (a + b)) <= 1e-10
        assert rel(gs[4], g2[2]) <= 1e-10
        assert maxrel(zs, z2) <= 1e-10
    finally:
        e.close()


def test_single_kernel_evaluations_around_a_composite_one_are_bit_identical():
    X, Y, Z, nv = so.case_data(1500, 300, 3, 2, 61, True)
    e = _ffi.Engine(0)
    e.set_option("nb", 128)
    try:
        e.set_data(X[:700], Y[:700, :1])
        e.exact_eval("matern52", True, 1.2, [1.1, 1.5, 0.9], 0.05)
        K0, L0 = e.get("K"), e.get("L")
        e.sparse_set_data(X, Y)
        s0 = e.sparse_eval("rbf", True, 1.1, [0.9, 1.4, 2.1], Z, 0.05)
        h0 = e.sparse_eval_het("matern32", False, 0.9, 1.3, Z, nv)
        gets0 = {w: e.sparse_get(w) for w in e.SPARSE_GET}
        e.sparse_eval_multi(_descs(so.KERNELS["m52_x_rbf_plus_exp"]), Z, 0.05)
        e.sparse_eval_multi(_descs(so.KERNELS["rbf_bias_white"]), Z[:129], nv)
        s1 = e.sparse_eval("rbf", True, 1.1, [0.9, 1.4, 2.1], Z, 0.05)
        h1 = e.sparse_eval_het("matern32", False, 0.9, 1.3, Z, nv)
        gets1 = {w: e.sparse_get(w) for w in e.SPARSE_GET}
        assert s0[0] == s1[0] and np.array_equal(s0[1], s1[1]) and np.array_equal(s0[2], s1[2])
        assert h0[0] == h1[0] and all(np.array_equal(a, b) for a, b in zip(h0[1:], h1[1:]))
        assert all(np.array_equal(gets0[w], gets1[w]) for w in gets0)
        assert np.array_equal(e.get("K"), K0) and np.array_equal(e.get("L"), L0)
    finally:
        e.close()


def test_rejections():
    X, Y, Z, _ = so.case_data(300, 20, 3, 1, 81, False)
    e = _ffi.Engine(0)
    try:
        e.sparse_set_data(X, Y)
        rq = ("ratquad", False, 1, [0], 0.5, 1.2, {"power": 0.8})
        sp = ("stdperiodic", False, 1, [0], 0.5, 1.2, {"period": 1.0})
        rbf = ("rbf", False, 0, [0, 1], 1.0, 1.0)
        for bad, what in (([rbf, rq], "RatQuad"), ([rbf, sp], "StdPeriodic")):
            with pytest.raises(_ffi.GpxArgumentError, match="not on the sparse evaluation"):
                e.sparse_eval_multi(bad, Z, 0.05)
        with pytest.raises(_ffi.GpxArgumentError, match="active dim outside the data"):
            e.sparse_eval_multi([("rbf", False, 0, [0, 3], 1.0, 1.0)], Z, 0.05)
        with pytest.raises(_ffi.GpxArgumentError):
            e.sparse_set_data(np.zeros((10, 65)), np.zeros((10, 1)))
        with pytest.raises(_ffi.GpxArgumentError):
            e.sparse_set_data(np.zeros((10, 3)), np.zeros((10, 9)))
        # a rejected kernel leaves the last evaluation's posterior in place
        e.sparse_set_data(X, Y)
        out = e.sparse_eval_multi([rbf, ("white", False, 1, [], 0.1, None)], Z, 0.05)
        wv = e.sparse_get("woodbury_vector")
        with pytest.raises(_ffi.GpxArgumentError):
            e.sparse_eval_multi([rbf, rq], Z, 0.05)
        assert np.isfinite(out[0]) and np.array_equal(e.sparse_get("woodbury_vector"), wv)
    finally:
        e.close()
