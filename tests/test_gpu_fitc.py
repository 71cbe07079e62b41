"""FITC sparse GP regression on the device (gpx_sparse_eval_fitc) against the reference's own FITC (tests/golden/fitc) and
the NumPy restatement (tests/fitc_oracle.py): the bound, kernel / noise / inducing-point gradients, dL_dKdiag and the
posterior; predict, predictive gradients and samples served from a FITC posterior; every register width of the composite
reductions; checkgrad of the mirror model as GPy/testing/fitc.py does it; a large case against the restatement streamed
over row chunks on the host; VarDTC and FITC alternating on one context; the rejections; and a launch count that does not
depend on N. Tolerances: |dLML| <= 1e-8 (relative to max(1, |LML|)), gradients 1e-6 of their largest entry."""
import glob
import os

import numpy as np
import pytest

import fitc_oracle as fo
from sparse_composite_oracle import CompositeOracle

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = sorted(glob.glob(os.path.join(HERE, "golden", "fitc", "*.npz")))


def _name(path):
    return os.path.basename(path)[:-4]


def _engine(X, Y):
    from gpy_b200 import _ffi
    e = _ffi.Engine(0)
    e.sparse_set_data(X, Y)
    return e


def _parts(parts):
    return [fo.descriptor(p) for p in parts]


def _close(got, want, tol=1e-6):
    want = np.asarray(want, dtype=np.float64)
    np.testing.assert_allclose(got, want, rtol=tol, atol=tol * max(np.abs(want).max(), 1e-300))


def _lml_close(got, want):
    assert abs(got - want) <= 1e-8 * max(1.0, abs(want)), (got, want)


@pytest.mark.parametrize("path", FIXTURES, ids=_name)
def test_fixture(path):
    f = np.load(path)
    parts = fo.CASES[_name(path)][0]
    e = _engine(f["X"], f["Y"])
    lml, grad, dZ, dR = e.sparse_eval_fitc(_parts(parts), f["Z"], float(f["noise"]))
    _lml_close(lml, float(f["lml"]))
    _close(grad, f["grad"])
    _close(dZ, f["Zgrad"])
    _close(dR, f["dL_dKdiag"])
    _close(e.sparse_get("woodbury_vector"), f["woodbury_vector"])
    if "woodbury_inv" in f:
        _close(e.sparse_get("woodbury_inv"), f["woodbury_inv"])
        _close(e.sparse_get("Kmm"), f["K"], 1e-12)
        _close(e.sparse_get("Lm"), f["K_chol"], 1e-10)
    else:   # the M x M arrays against the restatement
        res = fo.fitc_eval(f["X"], f["Y"], f["Z"], parts, float(f["noise"]))[3]
        _close(e.sparse_get("woodbury_inv"), res["woodbury_inv"])
        _close(e.sparse_get("Kmm"), res["K"], 1e-12)
        _close(e.sparse_get("Lm"), res["K_chol"], 1e-10)
    mu, var = e.sparse_predict(f["Xnew"])
    _close(mu, f["mu"])
    _close(var, f["var"])


@pytest.mark.parametrize("name", ["rbf_iso_m50", "m52_x_rbf_bias_m50", "rbf_ard_m129"])
def test_predictive_gradients_and_samples_from_a_fitc_posterior(name):
    X, Y, Z, noise, Xnew = fo.case_data(name)
    parts = fo.CASES[name][0]
    e = _engine(X, Y)
    e.sparse_eval_fitc(_parts(parts), Z, noise)
    res = fo.fitc_eval(X, Y, Z, parts, noise)[3]
    # the full covariance against the oracle's FITC posterior (posterior.py:238-270)
    k = CompositeOracle(parts)
    Kx = k.K(Xnew, Z)
    Sigma = k.K(Xnew) - Kx @ res["woodbury_inv"] @ Kx.T
    mu_f, cov = e.sparse_predict(Xnew, full_cov=True)
    _close(mu_f, Kx @ res["woodbury_vector"])
    np.testing.assert_allclose(cov, Sigma, rtol=0, atol=1e-8 * np.abs(Sigma).max())
    # predictive gradients against central differences of the device's own prediction
    dmu, dvar = e.sparse_predictive_gradients(Xnew)
    h = 1e-5
    for d in range(X.shape[1]):
        Xp, Xm = Xnew.copy(), Xnew.copy()
        Xp[:, d] += h
        Xm[:, d] -= h
        (mp, vp), (mm, vm) = e.sparse_predict(Xp), e.sparse_predict(Xm)
        _close(dmu[:, d, :], (mp - mm) / (2 * h), 1e-6)
        _close(dvar[:, d], ((vp - vm) / (2 * h))[:, 0], 1e-6)
    # samples: mu + chol(Sigma + jitter I) z with the device's Sigma and jitter
    z = np.random.default_rng(5).standard_normal((3, Xnew.shape[0]))
    fs, jit = e.sparse_posterior_samples(Xnew, z)
    L = np.linalg.cholesky(cov + jit * np.eye(cov.shape[0]))
    want = mu_f[:, 0][None, :] + (L @ z.T).T
    np.testing.assert_allclose(fs, want, rtol=0, atol=1e-8 * np.abs(want).max())


@pytest.mark.parametrize("D", [4, 8, 16, 32], ids=lambda d: "stacked%d" % (2 * d))
def test_every_register_width_of_the_composite_reductions(D):
    """RBF(ARD) x Matern52(ARD) + Bias on all D columns: 2 D stacked dims (8 / 16 / 32 / 64)"""
    rng = np.random.default_rng(D)
    N, M = 300, 60
    X = rng.uniform(-1.0, 1.0, (N, D))
    Y = np.sin(X.sum(1, keepdims=True)) + 0.1 * rng.standard_normal((N, 1))
    Z = X[rng.choice(N, M, replace=False)] + 0.02 * rng.standard_normal((M, D))
    dims = list(range(D))
    parts = [dict(kind="rbf", term=0, dims=dims, variance=1.1, lengthscale=list(D ** 0.5 * (1.0 + 0.05 * np.arange(D))),
                  ARD=True),
             dict(kind="matern52", term=0, dims=dims, variance=0.9, lengthscale=list(1.5 * D ** 0.5 + 0.05 * np.arange(D)),
                  ARD=True),
             dict(kind="bias", term=1, variance=0.2)]
    e = _engine(X, Y)
    lml, grad, dZ, dR = e.sparse_eval_fitc(_parts(parts), Z, 0.05)
    wl, wg, wZ, res = fo.fitc_eval(X, Y, Z, parts, 0.05)
    _lml_close(lml, wl)
    _close(grad, wg)
    _close(dZ, wZ)
    _close(dR, res["dL_dKdiag"])


@pytest.mark.parametrize("D", [1, 2])
def test_checkgrad_of_the_mirror_model(D):
    """GPy/testing/fitc.py:27-37: SparseGPRegression on 20 points, inference_method = FITC(), checkgrad"""
    import gpy_b200 as gb
    rng = np.random.default_rng(D)
    X = rng.uniform(-3.0, 3.0, (20, D))
    Y = np.prod(np.sin(X), axis=1, keepdims=True) + 0.05 * rng.standard_normal((20, 1))
    m = gb.SparseGPRegression(X, Y)
    m.inference_method = gb.FITC()
    m.parameters_changed()
    assert m.checkgrad()


def test_large_case_against_the_restatement_streamed_over_rows():
    """N = 65536, M = 4096, D = 16, RBF(ARD): the host oracle streams the N x M products over row chunks"""
    rng = np.random.default_rng(7)
    N, M, D, chunk = 65536, 4096, 16, 8192
    X = rng.uniform(-1.0, 1.0, (N, D))
    Y = np.sin(X @ rng.standard_normal(D))[:, None] + 0.1 * rng.standard_normal((N, 1))
    Z = X[rng.choice(N, M, replace=False)] + 0.01 * rng.standard_normal((M, D))
    var, ls, noise = 1.3, 1.2 + 0.1 * np.arange(D), 0.05
    e = _engine(X, Y)
    lml, grad, dZ, dR = e.sparse_eval_fitc([("rbf", True, 0, list(range(D)), var, ls)], Z, noise)

    def K(A, B):
        As, Bs = A / ls, B / ls
        r2 = (As ** 2).sum(1)[:, None] + (Bs ** 2).sum(1)[None, :] - 2 * As @ Bs.T
        return var * np.exp(-0.5 * np.maximum(r2, 0.0))

    Kmm = K(Z, Z) + 1e-6 * np.eye(M)
    L = np.linalg.cholesky(Kmm)
    Li = np.linalg.inv(L)
    Kmmi = Li.T @ Li
    A = np.eye(M)
    URiy = np.zeros((M, 1))
    sig = np.empty(N)
    for i in range(0, N, chunk):
        U = K(X[i:i + chunk], Z)
        LiUT = Li @ U.T
        sig[i:i + chunk] = var + noise - (LiUT ** 2).sum(0)
        bs = 1.0 / sig[i:i + chunk]
        A += (LiUT * np.sqrt(bs)) @ (LiUT * np.sqrt(bs)).T
        URiy += (U.T * bs) @ Y[i:i + chunk]
    beta = 1.0 / sig
    LA = np.linalg.cholesky(A)
    b = np.linalg.solve(LA, Li @ URiy)
    v = Li.T @ np.linalg.solve(LA.T, b)
    LAi_Li = np.linalg.solve(LA, Li)
    P = LAi_Li.T @ LAi_Li
    want_lml = (-0.5 * N * np.log(2 * np.pi) - np.log(np.diag(LA)).sum() + 0.5 * np.log(beta).sum()
                - 0.5 * (beta * Y[:, 0] ** 2).sum() + 0.5 * (b ** 2).sum())
    _lml_close(lml, want_lml)
    dLdR = np.empty(N)
    for i in range(0, N, chunk):
        U = K(X[i:i + chunk], Z)
        Uv = U @ v
        y, bs = Y[i:i + chunk], beta[i:i + chunk]
        dLdR[i:i + chunk] = 0.5 * ((U * (U @ P)).sum(1) - 1.0 / bs + (y ** 2).sum(1) - 2 * (Uv * y).sum(1)
                                   + (Uv ** 2).sum(1)) * bs ** 2
    _close(dR, dLdR)
    _close(grad[-1], dLdR.sum())
    _close(e.sparse_get("woodbury_vector"), v)
    _close(e.sparse_get("woodbury_inv"), Kmmi - P)


def test_vardtc_and_fitc_alternating_on_one_context_match_fresh_contexts():
    X, Y, Z, noise, _ = fo.case_data("rbf_ard_bias_white_m129")
    parts = _parts(fo.CASES["rbf_ard_bias_white_m129"][0])

    def fitc(e):
        out = e.sparse_eval_fitc(parts, Z, noise)
        return out + (e.sparse_get("woodbury_inv"), e.sparse_get("Kmm"))

    def vardtc(e):
        out = e.sparse_eval_multi(parts, Z, noise)
        return out + (e.sparse_get("woodbury_inv"), e.sparse_get("Kmm"))

    fresh_f, fresh_v = fitc(_engine(X, Y)), vardtc(_engine(X, Y))
    e = _engine(X, Y)
    seq = [vardtc(e), fitc(e), vardtc(e), fitc(e)]
    for got, want in zip(seq, [fresh_v, fresh_f, fresh_v, fresh_f]):
        for a, b in zip(got, want):
            assert np.array_equal(np.asarray(a), np.asarray(b))


def test_rejections():
    from gpy_b200 import _ffi
    X, Y, Z, noise, _ = fo.case_data("rbf_iso_m50")
    rbf = [("rbf", False, 0, [0, 1, 2], 1.0, 1.0)]
    with pytest.raises(_ffi.GpxArgumentError, match="set_data"):
        _ffi.Engine(0).sparse_eval_fitc(rbf, Z, noise)
    e = _engine(X, np.hstack([Y, Y]))
    with pytest.raises(_ffi.GpxArgumentError, match="one output column"):
        e.sparse_eval_fitc(rbf, Z, noise)
    e = _engine(X, Y)
    with pytest.raises(_ffi.GpxArgumentError, match="RatQuad"):
        e.sparse_eval_fitc([("ratquad", False, 0, [0, 1, 2], 1.0, 1.0, {"power": 2.0})], Z, noise)
    with pytest.raises(_ffi.GpxArgumentError, match="M must be positive"):
        e.sparse_eval_fitc(rbf, Z[:0], noise)
    rc = _ffi.lib().gpx_sparse_eval_fitc(e._h, None, 1, None, 5, noise, None, None, None, None)
    assert rc == -2
    # a negative noise variance makes sigma* negative: LinAlgError naming the first such point (point 0 here)
    with pytest.raises(np.linalg.LinAlgError, match="data point 0 "):
        e.sparse_eval_fitc(rbf, Z, -10.0)
    # the context is still usable
    lml = e.sparse_eval_fitc(rbf, Z, noise)[0]
    assert np.isfinite(lml)


def test_a_communicator_is_rejected():
    from test_gpu_sharded_single_rank import nccl_library, sharded_engine
    if not (os.environ.get("GPX_NCCL_LIB") or nccl_library()):
        pytest.skip("NCCL not available")
    from gpy_b200 import _ffi
    X, Y, Z, noise, _ = fo.case_data("rbf_iso_m50")
    e = sharded_engine()
    e.sparse_set_data(X, Y)
    with pytest.raises(_ffi.GpxArgumentError, match="single-GPU"):
        e.sparse_eval_fitc([("rbf", False, 0, [0, 1, 2], 1.0, 1.0)], Z, noise)


@pytest.mark.parametrize("composite", [False, True], ids=["single", "composite"])
def test_launch_count_does_not_depend_on_n(composite):
    rng = np.random.default_rng(3)
    parts = ([("rbf", True, 0, [0, 1, 2], 1.0, [1.0, 1.2, 1.4])] if not composite else
             [("rbf", True, 0, [0, 1, 2], 1.0, [1.0, 1.2, 1.4]), ("bias", False, 1, [], 0.3, None)])
    Z = rng.uniform(-1, 1, (70, 3))
    counts = []
    for N in (500, 3000):
        X = rng.uniform(-1, 1, (N, 3))
        e = _engine(X, np.sin(X[:, :1]))
        e.sparse_eval_fitc(parts, Z, 0.1)   # first call allocates
        t0 = e.total_launches()
        e.sparse_eval_fitc(parts, Z, 0.1)
        counts.append(e.total_launches() - t0)
    assert counts[0] == counts[1]
