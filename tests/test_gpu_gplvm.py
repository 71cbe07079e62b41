"""GPLVM on the device: gpx_exact_grad_X against the NumPy restatement (tests/gplvm_oracle.py) on every K^-1 route, the
mirror's GPLVM against the reference's own GPLVM (tests/golden/gplvm), checkgrad, a short optimisation, the rejections
and the launch accounting."""
import ctypes
import glob
import os

import numpy as np
import pytest

import gpy_b200
import gplvm_oracle as go
from gpy_b200 import _ffi
from sparse_composite_oracle import CompositeOracle, descriptor

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = sorted(glob.glob(os.path.join(HERE, "golden", "gplvm", "*.npz")))
NS = dict(RBF=gpy_b200.RBF, Exponential=gpy_b200.Exponential, Matern32=gpy_b200.Matern32, Matern52=gpy_b200.Matern52,
          Bias=gpy_b200.Bias, White=gpy_b200.White, Add=gpy_b200.Add, Prod=gpy_b200.Prod)

RBF_ARD = [dict(kind="rbf", term=0, dims=[0, 1, 2], variance=1.2, lengthscale=[0.8, 1.3, 1.9], ARD=True)]
M52_ISO = [dict(kind="matern52", term=0, dims=[0, 1, 2], variance=0.9, lengthscale=1.1)]
COMPOSITES = {
    "rbf_bias_white": [dict(kind="rbf", term=0, dims=[0, 1, 2], variance=1.3, lengthscale=[0.9, 1.4, 2.1], ARD=True),
                       dict(kind="bias", term=1, variance=0.4), dict(kind="white", term=2, variance=0.07)],
    "m32_x_rbf_plus_exp": [dict(kind="matern32", term=0, dims=[0, 1], variance=1.1, lengthscale=1.2),
                           dict(kind="rbf", term=0, dims=[1, 2], variance=0.8, lengthscale=[1.5, 0.7], ARD=True),
                           dict(kind="exponential", term=1, dims=[0], variance=0.3, lengthscale=2.5)],
}


def _close_rel(a, b, rtol):
    a, b = np.asarray(a), np.asarray(b)
    np.testing.assert_allclose(a, b, rtol=rtol, atol=1e-9 * np.abs(b).max())


def _engine_eval(eng, parts, X, Y, noise, single=False):
    eng.set_data(X, Y)
    if single:
        p = parts[0]
        return eng.exact_eval(p["kind"], p.get("ARD", False), p["variance"], p["lengthscale"], noise)
    return eng.exact_eval_multi([descriptor(p) for p in parts], noise)


# ---- the entry against the restatement, on every route that stores or forms K^-1 ----------------------------------------
@pytest.mark.parametrize("case", [
    ("rbf_ard_fine", RBF_ARD, 300, 3, True, 0),              # single kernel, nt <= 8: fine LAUUM stores K^-1
    ("rbf_ard_fused", RBF_ARD, 1300, 3, True, 0),            # single kernel, nt > 8: K^-1 formed on demand
    ("m52_iso_fused", M52_ISO, 1100, 2, True, 0),
    ("rbf_ard_int8", RBF_ARD, 2100, 2, True, 1),             # the int8 sweep accumulates K^-1
    ("rbf_bias_white", COMPOSITES["rbf_bias_white"], 1025, 8, False, 0),
    ("m32_x_rbf_plus_exp", COMPOSITES["m32_x_rbf_plus_exp"], 700, 1, False, 0),
], ids=lambda c: c[0])
def test_exact_grad_X_matches_the_restatement(case):
    _, parts, N, P, single, ozaki = case
    X, Y = go.latent_data(N, 3, P, seed=N + P)
    eng = _ffi.Engine()
    eng.set_option("ozaki", ozaki)
    lml, grad, _ = _engine_eval(eng, parts, X, Y, 0.3, single)
    lml0, grad0, dX0, _ = go.gplvm_eval(X, Y, parts, 0.3)
    assert abs(lml - lml0) <= 1e-8 * max(1.0, abs(lml0))
    dX = eng.exact_grad_X()
    assert dX.shape == (N, 3)
    _close_rel(dX, dX0, 1e-6)


def test_grad_X_changes_nothing_the_evaluation_returns():
    X, Y = go.latent_data(1300, 3, 2, seed=4)
    eng = _ffi.Engine()
    p = RBF_ARD[0]
    eng.set_data(X, Y)
    eng.exact_eval(p["kind"], True, p["variance"], p["lengthscale"], 0.2)
    st0 = eng.stats()
    a0 = eng.get("alpha")
    mu0, var0 = eng.predict(X[:9])
    g1 = eng.exact_grad_X()
    g2 = eng.exact_grad_X()
    np.testing.assert_array_equal(g1, g2)
    assert eng.stats() == st0
    np.testing.assert_array_equal(eng.get("alpha"), a0)
    mu1, var1 = eng.predict(X[:9])
    np.testing.assert_array_equal(mu0, mu1)
    np.testing.assert_array_equal(var0, var1)
    # K^-1 formed for the input gradient is the one gpx_get(KINV) forms
    eng2 = _ffi.Engine()
    eng2.set_data(X, Y)
    eng2.exact_eval(p["kind"], True, p["variance"], p["lengthscale"], 0.2)
    np.testing.assert_array_equal(eng.get("Kinv"), eng2.get("Kinv"))


def test_launch_counts_do_not_depend_on_N():
    counts = []
    for N in (300, 1300):
        X, Y = go.latent_data(N, 3, 2, seed=N)
        eng = _ffi.Engine()
        _engine_eval(eng, COMPOSITES["rbf_bias_white"], X, Y, 0.2)
        t0 = eng.total_launches()
        eng.exact_grad_X()
        counts.append(eng.total_launches() - t0)
    assert counts == [2, 2]
    X, Y = go.latent_data(1300, 3, 2, seed=3)
    eng = _ffi.Engine()
    _engine_eval(eng, RBF_ARD, X, Y, 0.2, single=True)
    t0 = eng.total_launches()
    eng.exact_grad_X()
    t1 = eng.total_launches()
    eng.exact_grad_X()
    assert (t1 - t0, eng.total_launches() - t1) == (3, 2)    # the plain LAUUM once, then the two launches


def test_rejections_leave_nothing_touched():
    L = _ffi.lib()
    X, Y = go.latent_data(200, 3, 1, seed=9)
    eng = _ffi.Engine()
    eng.set_data(X, Y)
    with pytest.raises(_ffi.GpxArgumentError):                # no evaluation
        eng.exact_grad_X()
    p = RBF_ARD[0]
    eng.exact_eval(p["kind"], True, p["variance"], p["lengthscale"], 0.2)
    assert L.gpx_exact_grad_X(eng._h, None) == -2             # null pointer
    eng.exact_eval_het(p["kind"], True, p["variance"], p["lengthscale"], np.full(200, 0.2))
    with pytest.raises(_ffi.GpxArgumentError):                # heteroscedastic
        eng.exact_grad_X()
    eng.exact_eval_multi([("ratquad", False, 0, [0, 1, 2], 1.0, 1.2, {"power": 2.0})], 0.2)
    with pytest.raises(_ffi.GpxArgumentError):                # no device input gradient
        eng.exact_grad_X()
    eng.laplace_begin([descriptor(p)])
    with pytest.raises(_ffi.GpxArgumentError):                # no exact evaluation after the Laplace begin
        eng.exact_grad_X()
    t0 = eng.total_launches()
    with pytest.raises(_ffi.GpxArgumentError):
        eng.exact_grad_X()
    assert eng.total_launches() == t0


def test_finished_laplace_and_ep_posteriors_and_a_communicator_are_rejected():
    """their evaluations leave have_eval (and, for EP, a stored K^-1) set: the rejection is what keeps the call from
    returning a gradient for a dL_dK those posteriors do not have"""
    from test_gpu_sharded_single_rank import attach
    X, Y = go.latent_data(300, 3, 1, seed=10)
    part = descriptor(RBF_ARD[0])
    eng = _ffi.Engine()
    eng.set_data(X, np.sign(Y))
    eng.laplace_begin([part])
    W = np.full(300, 0.2)
    eng.laplace_newton(W, np.ones(300), np.zeros(300))
    eng.laplace_finish(W, np.zeros(300), np.ones(300))
    with pytest.raises(_ffi.GpxArgumentError, match="Laplace / EP"):
        eng.exact_grad_X()
    eng.ep_begin([part])
    eng.ep_start()
    eng.ep_finish(np.full(300, 0.5), 0.3 * np.sign(Y[:, 0]))
    with pytest.raises(_ffi.GpxArgumentError, match="Laplace / EP"):
        eng.exact_grad_X()
    t1 = eng.total_launches()
    with pytest.raises(_ffi.GpxArgumentError):
        eng.exact_grad_X()
    assert eng.total_launches() == t1
    e = attach(_ffi.Engine())
    e.set_data(X, Y)
    e.exact_eval("rbf", True, 1.2, [0.8, 1.3, 1.9], 0.2)
    with pytest.raises(_ffi.GpxArgumentError, match="single-GPU"):
        e.exact_grad_X()


# ---- the mirror's GPLVM against the reference's own -------------------------------------------------------------------
@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[:-4])
def test_mirror_gplvm_matches_the_reference(path):
    f = np.load(path)
    name = os.path.basename(path)[:-4]
    case = go.CASES[name]
    Y = f["Y"]
    kern = case["kernel"](NS) if case["kernel"] is not None else None
    np.random.seed(int(f["seed"]))
    m = gpy_b200.GPLVM(Y, int(f["Q"]), kernel=kern, normalizer=case.get("normalizer", False))
    np.testing.assert_array_equal(m.latent_mean.values, f["X0"])
    m.likelihood.variance[:] = float(f["noise"])
    assert abs(m.log_likelihood() - float(f["lml"])) <= 1e-8 * max(1.0, abs(float(f["lml"])))
    _close_rel(m.gradient, f["grad"], 1e-6)
    mu, var = m.predict(f["Xnew"])
    _close_rel(mu, f["mu"], 1e-8)
    _close_rel(var, f["var"], 1e-8)


def test_checkgrad_on_the_latent_points_and_the_hyper_parameters():
    _, Y = go.latent_data(30, 3, 4, seed=21)
    np.random.seed(3)
    m = gpy_b200.GPLVM(Y, 2)
    assert m.checkgrad()


def test_short_optimize_raises_the_likelihood():
    _, Y = go.latent_data(150, 3, 6, seed=22)
    np.random.seed(4)
    m = gpy_b200.GPLVM(Y, 2)
    l0 = m.log_likelihood()
    m.optimize(max_iters=25)
    assert m.log_likelihood() > l0 + 1.0
    assert np.all(np.isfinite(m.latent_mean.values))
