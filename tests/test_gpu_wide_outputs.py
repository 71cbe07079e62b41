"""The exact evaluation with more than 8 output columns (the wide route of include/gpx.h: solves on the DMMA GEMM, K^-1
always stored, every reduction through the composite pass) against the NumPy restatement, the entries that serve it
(gpx_get, gpx_predict, gpx_exact_grad_X), the ones that reject it, and the narrow route left as it was."""
import numpy as np
import pytest

import gpy_b200
import gplvm_oracle as go
from gpy_b200 import _ffi
from oracle import gpy_oracle as o
from sparse_composite_oracle import CompositeOracle, descriptor

pytestmark = pytest.mark.gpu

KERNELS = {
    "rbf_ard": [dict(kind="rbf", term=0, dims=[0, 1, 2], variance=1.2, lengthscale=[0.8, 1.3, 1.9], ARD=True)],
    "rbf_bias_white": [dict(kind="rbf", term=0, dims=[0, 1, 2], variance=1.3, lengthscale=[0.9, 1.4, 2.1], ARD=True),
                       dict(kind="bias", term=1, variance=0.4), dict(kind="white", term=2, variance=0.07)],
}
NOISE = 0.3


def _close(a, b, rtol):
    np.testing.assert_allclose(np.asarray(a), np.asarray(b), rtol=rtol, atol=rtol * 1e-3 * np.abs(b).max())


def _eval(eng, kname, X, Y):
    eng.set_data(X, Y)
    parts = KERNELS[kname]
    if kname == "rbf_ard":   # the single-kernel entry: its result layout, the composite pass behind it
        p = parts[0]
        return eng.exact_eval(p["kind"], True, p["variance"], p["lengthscale"], NOISE)
    return eng.exact_eval_multi([descriptor(p) for p in parts], NOISE)


@pytest.mark.parametrize("N,P", [(1025, 9), (1025, 64), (1025, 1000), (4097, 9), (4097, 64), (4097, 1000)])
@pytest.mark.parametrize("kname", sorted(KERNELS))
def test_wide_evaluation_matches_the_restatement(kname, N, P):
    X, Y = go.latent_data(N, 3, P, seed=N + P)
    eng = _ffi.Engine()
    lml, grad, jit = _eval(eng, kname, X, Y)
    assert jit == 0.0
    lml0, grad0, dX0, res = go.gplvm_eval(X, Y, KERNELS[kname], NOISE)
    assert abs(lml - lml0) <= 1e-8 * max(1.0, abs(lml0))
    _close(grad, grad0, 1e-6)
    _close(eng.get("alpha"), res["alpha"], 1e-8)
    _close(eng.exact_grad_X(), dX0, 1e-6)
    Xnew = np.random.default_rng(N).uniform(-1.5, 1.5, size=(37, 3))
    mu, var = eng.predict(Xnew)
    kern = CompositeOracle(KERNELS[kname])
    mu0, var0 = o.raw_predict(kern, X, res["L"], res["alpha"], Xnew)
    assert mu.shape == (37, P)
    _close(mu, mu0, 1e-8)
    _close(var, var0, 1e-8)
    if N == 1025:   # the N x N selectors
        _close(eng.get("Kinv"), res["Wi"], 1e-8)
        _close(eng.get("dL_dK"), res["dL_dK"], 1e-8)
        _close(eng.get("L"), res["L"], 1e-10)
        _close(eng.get("K"), res["K"], 1e-12)
        mu2, cov = eng.predict(Xnew[:5], full_cov=True)
        mu20, cov0 = o.raw_predict(kern, X, res["L"], res["alpha"], Xnew[:5], full_cov=True)
        _close(mu2, mu20, 1e-8)
        _close(cov, cov0, 1e-8)


def test_mirror_gp_regression_with_many_outputs():
    X, Y = go.latent_data(600, 3, 40, seed=5)
    p = KERNELS["rbf_ard"][0]
    m = gpy_b200.GPRegression(X, Y, gpy_b200.RBF(3, variance=p["variance"], lengthscale=p["lengthscale"], ARD=True),
                              noise_var=NOISE)
    lml0, grad0, _, res = go.gplvm_eval(X, Y, KERNELS["rbf_ard"], NOISE)
    assert abs(m.log_likelihood() - lml0) <= 1e-8 * abs(lml0)
    _close(m.gradient, grad0, 1e-6)
    mu, var = m.predict(X[:7])
    assert mu.shape == (7, 40) and var.shape == (7, 1)


def test_p8_is_bit_identical_after_a_wide_evaluation():
    X, Y = go.latent_data(1300, 3, 9, seed=8)
    fresh = _ffi.Engine()
    r0 = _eval(fresh, "rbf_ard", X, Y[:, :8])
    a0, s0 = fresh.get("alpha"), fresh.stats()["launches"]
    reused = _ffi.Engine()
    _eval(reused, "rbf_ard", X, Y)
    r1 = _eval(reused, "rbf_ard", X, Y[:, :8])
    assert r1[0] == r0[0]
    np.testing.assert_array_equal(r1[1], r0[1])
    np.testing.assert_array_equal(reused.get("alpha"), a0)
    assert reused.stats()["launches"] == s0


def test_entries_without_a_wide_route_reject_it():
    X, Y = go.latent_data(300, 3, 12, seed=6)
    eng = _ffi.Engine()
    _eval(eng, "rbf_ard", X, Y)
    a0 = eng.get("alpha")
    p = KERNELS["rbf_ard"][0]
    with pytest.raises(_ffi.GpxArgumentError, match="8 output columns"):
        eng.predictive_gradients(X[:3])
    with pytest.raises(_ffi.GpxArgumentError, match="8 output columns"):
        eng.posterior_covariance(X[:3])
    with pytest.raises(_ffi.GpxArgumentError, match="8 output columns"):
        eng.posterior_samples(X[:3], np.zeros((12, 3)))
    with pytest.raises(_ffi.GpxArgumentError):                       # the Laplace / EP entries take one column
        eng.laplace_begin([descriptor(p)])
    with pytest.raises(_ffi.GpxArgumentError, match="1024"):
        eng.set_data(X, np.zeros((300, 1025)))
    np.testing.assert_array_equal(eng.get("alpha"), a0)             # the rejections left the evaluation as it was
    with pytest.raises(_ffi.GpxArgumentError, match="8 output columns"):
        eng.exact_eval_het(p["kind"], True, p["variance"], p["lengthscale"], np.full(300, NOISE))
