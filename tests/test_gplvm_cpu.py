"""GPLVM without a GPU: the NumPy restatement (tests/gplvm_oracle.py) against the reference's own GPLVM (the fixtures of
tests/golden/gplvm), the mirror's latent initialisation against the reference's, and the mirror's host logic (parameter
order and transforms, one device input gradient per evaluation, the fallback of a stale handle) on a test double of the
engine that answers from the restatement."""
import glob
import os

import numpy as np
import pytest

import gpy_b200
import gplvm_oracle as go
from gpy_b200 import _ffi
from gpy_b200.gplvm import initialize_latent
from gpy_b200.kern import flatten_parts, part_descriptor
from oracle import gpy_oracle as o

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = sorted(glob.glob(os.path.join(HERE, "golden", "gplvm", "*.npz")))
NS = dict(RBF=gpy_b200.RBF, Exponential=gpy_b200.Exponential, Matern32=gpy_b200.Matern32, Matern52=gpy_b200.Matern52,
          Bias=gpy_b200.Bias, White=gpy_b200.White, Add=gpy_b200.Add, Prod=gpy_b200.Prod)


def parts_of(kern):
    """the mirror kernel as the restatement's part dicts"""
    out = []
    for leaf, term in flatten_parts(kern):
        kind, ard, t, dims, var, ls = part_descriptor(leaf, term)[:6]
        d = dict(kind=kind, term=t, variance=var)
        if kind not in ("white", "bias"):
            d.update(dims=list(dims), lengthscale=ls, ARD=bool(ard))
        out.append(d)
    return out


def test_fixture_set_covers_the_cases():
    assert {os.path.basename(p)[:-4] for p in FIXTURES} == set(go.CASES)


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[:-4])
def test_initialisation_and_restatement_match_the_reference(path):
    f = np.load(path)
    case = go.CASES[os.path.basename(path)[:-4]]
    Y, Q = f["Y"], int(f["Q"])
    np.random.seed(int(f["seed"]))
    X0, fracs = initialize_latent("PCA", Q, Y)
    np.testing.assert_array_equal(X0, f["X0"])
    kern = case["kernel"](NS) if case["kernel"] is not None else \
        gpy_b200.RBF(Q, lengthscale=fracs, ARD=Q > 1) + gpy_b200.Bias(Q, np.exp(-2))
    Yn = Y
    if case.get("normalizer"):
        Yn = (Y - Y.mean(0)) / np.where(Y.std(0) == 0, 1.0, Y.std(0))
    lml, grad, dX, _ = go.gplvm_eval(X0, Yn, parts_of(kern), float(f["noise"]))
    assert abs(lml - float(f["lml"])) <= 1e-9 * abs(float(f["lml"]))
    full = np.concatenate([dX.reshape(-1), grad])
    np.testing.assert_allclose(full, f["grad"], rtol=1e-8, atol=1e-11 * np.abs(f["grad"]).max())


def test_random_init_draws_like_the_reference():
    Y = np.random.default_rng(0).standard_normal((20, 4))
    np.random.seed(5)
    X, fracs = initialize_latent("random", 3, Y)
    np.random.seed(5)
    Xr = np.random.normal(0, 1, (20, 3))
    np.testing.assert_allclose(X, (Xr - Xr.mean(0)) / (Xr - Xr.mean(0)).std(0), rtol=1e-14)
    assert fracs.max() == 1.0


# ---- host logic on a test double of the engine ----------------------------------------------------------------------
class FakeEngine(object):
    """answers the exact evaluation and gpx_exact_grad_X from the restatement"""

    def __init__(self):
        self.eval_serial, self.grad_X_calls, self.N, self.D, self.P = 0, 0, 0, 0, 0

    def set_data(self, X, Y):
        self.X, self.Y = np.array(X), np.array(Y)
        self.N, self.D = X.shape
        self.P = Y.shape[1]
        self.eval_serial += 1

    def exact_eval_multi(self, parts, noise, jitter=1e-8, max_tries=5):
        self.parts = [dict(kind=k, ARD=a, term=t, dims=d, variance=v, lengthscale=ls) for (k, a, t, d, v, ls) in parts]
        self.lml, grad, self.dX, _ = go.gplvm_eval(self.X, self.Y, self.parts, noise)
        self.eval_serial += 1
        return self.lml, grad, 0.0

    def exact_eval(self, kind, ARD, variance, lengthscale, noise, jitter=1e-8, max_tries=5):
        lml, grad, _ = self.exact_eval_multi([(kind, ARD, 0, list(range(self.D)), variance, lengthscale)], noise)
        return lml, grad, 0.0

    def exact_grad_X(self):
        self.grad_X_calls += 1
        return self.dX.copy()


@pytest.fixture
def host_grad_X(monkeypatch):
    """the stand-alone gradients_X answered by the restatement, counted"""
    calls = []

    def grad_X(kind, ARD, v, ls, X, dL, X2=None):
        calls.append(X.shape)
        return o.StationaryOracle(kind, X.shape[1], v, ls, ARD).gradients_X(np.asarray(dL), X, X2)
    monkeypatch.setattr(_ffi, "kern_grad_X", grad_X)
    return calls


def _model(kernel=None, N=25, P=3, Q=2, seed=2):
    _, Y = go.latent_data(N, 3, P, seed)
    eng = FakeEngine()
    np.random.seed(seed)
    return gpy_b200.GPLVM(Y, Q, kernel=kernel, engine=eng), eng, Y


def test_parameter_order_and_transforms():
    m, eng, _ = _model()
    names = [p.name for p in m.flattened_parameters()]
    assert names == ["latent_mean", "variance", "lengthscale", "variance", "variance"]
    assert m.latent_mean.transform is None and m.latent_mean.values.shape == (25, 2)
    assert all(p.transform is not None for p in m.flattened_parameters()[1:])
    x = m.optimizer_array
    np.testing.assert_array_equal(x[:50], m.latent_mean.values.reshape(-1))   # unconstrained: the values themselves
    g = m._grads_transformed()
    np.testing.assert_array_equal(g[:50], -m.latent_mean.gradient.reshape(-1))
    np.testing.assert_array_equal(m.gradient[:50], eng.dX.reshape(-1))


def test_one_device_input_gradient_per_evaluation_for_a_combination(host_grad_X):
    m, eng, _ = _model()
    assert eng.grad_X_calls == 1
    x = m.optimizer_array
    m.optimizer_array = x + 0.01
    m.likelihood.variance[:] = 0.5
    assert eng.grad_X_calls == 3 and host_grad_X == []
    m2, eng2, _ = _model(kernel=gpy_b200.Matern32(2, variance=0.9, lengthscale=[0.8, 1.2], ARD=True))
    assert eng2.grad_X_calls == 1 and host_grad_X == []


def test_a_stale_handle_takes_the_stand_alone_route(host_grad_X, monkeypatch):
    m, eng, _ = _model()
    old = m.grad_dict["dL_dK"]
    monkeypatch.setattr(old, "__array__", lambda dtype=None, copy=None: np.zeros(old.shape))
    m.likelihood.variance[:] = 0.7            # a new evaluation: the old handle no longer describes the device
    n = eng.grad_X_calls
    g = m.kern.gradients_X(old, m.X, None)
    assert eng.grad_X_calls == n and len(host_grad_X) == 1 and np.all(g == 0)
    # the current handle on other inputs is not the evaluation's either
    X2 = m.X + 1.0
    monkeypatch.setattr(m.grad_dict["dL_dK"], "__array__", lambda dtype=None, copy=None: np.zeros((25, 25)))
    m.kern.gradients_X(m.grad_dict["dL_dK"], X2, None)
    assert eng.grad_X_calls == n and len(host_grad_X) == 2


def test_mirror_gradients_match_the_restatement():
    m, eng, Y = _model(P=4)
    lml, grad, dX, _ = go.gplvm_eval(m.X, Y, parts_of(m.kern), float(m.likelihood.variance[0]))
    np.testing.assert_allclose(m.gradient, np.concatenate([dX.reshape(-1), grad]), rtol=1e-12, atol=1e-14)
    assert m.log_likelihood() == lml
