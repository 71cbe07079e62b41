"""The variational Gaussian approximation on the host: the NumPy restatement (tests/vargauss_oracle.py) against the
fixtures the reference's own VarGauss.inference wrote (tests/golden/vargauss), the one term where the device departs from
the reference (the scaling side of dF_dK), the identities the device relies on, and the mirror's host logic through a host
engine. The central differences of the reference's bound run where its tree exists."""
import glob
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), HERE, os.path.join(HERE, "golden")]

import vargauss_oracle as vo  # noqa: E402
import gpy_b200  # noqa: E402
from gpy_b200.vargauss import GPVariationalGaussianApproximation, VarGauss  # noqa: E402

FIXTURES = sorted(glob.glob(os.path.join(HERE, "golden", "vargauss", "*.npz")))
HAVE_REF = os.path.isdir(os.environ.get("GPX_REFERENCE", "/root/reference"))
needs_ref = pytest.mark.skipif(not HAVE_REF, reason="the reference tree is not present")


def _name(path):
    return os.path.basename(path)[:-4]


def _oracle(name, row_scaling=False, Xnew=None):
    parts, lik_spec, N, seed, _ = vo.CASES[name]
    X, Y, alpha, beta, _ = vo.case_data(name)
    return vo.vargauss_eval(parts, X, Y, alpha, beta, vo.make_likelihood(lik_spec, gpy_b200), row_scaling, Xnew)


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300)) if b.size else 0.0


def test_every_case_has_a_fixture():
    assert sorted(_name(p) for p in FIXTURES) == sorted(vo.CASES)


@pytest.mark.parametrize("path", FIXTURES, ids=_name)
def test_oracle_matches_the_reference(path):
    f = np.load(path)
    name = _name(path)
    X, Y, alpha, beta, Xnew = vo.case_data(name)
    np.testing.assert_array_equal(f["X"], X)
    np.testing.assert_array_equal(f["beta"], beta)
    o = _oracle(name, Xnew=Xnew)
    bar = 1e-12 * vo.cond_bound(vo.CompositeOracle(vo.CASES[name][0]).K(X), beta)
    assert abs(o["lml"] - f["lml"]) <= bar * max(1.0, abs(float(f["lml"])))
    for k in ("m", "var", "dalpha", "dbeta", "dF_dm", "dF_dv"):
        assert _rel(o[k], f[k]) <= bar, k
    np.testing.assert_allclose(o["dL_dthetaL"], f["dL_dthetaL"], rtol=bar, atol=bar)
    if "pmu" in f.files:
        assert _rel(o["pmu"], f["pmu"]) <= 1e-16 * f["cond_K"] * 100 + 1e-12
        assert _rel(o["pvar"], f["pvar"]) <= 1e-16 * f["cond_K"] * 1000 + 1e-12


@pytest.mark.parametrize("path", FIXTURES, ids=_name)
def test_row_scaling_reproduces_the_reference_kernel_gradient(path):
    """the reference's dF_dK with its rows scaled: the only difference from the oracle is that one term"""
    f = np.load(path)
    o = _oracle(_name(path), row_scaling=True)
    assert _rel(o["grad"], f["grad_ref"]) <= 1e-9


@pytest.mark.parametrize("path", [p for p in FIXTURES if _name(p).startswith("gaussian")], ids=_name)
def test_column_scaling_equals_the_reference_where_dF_dv_is_constant(path):
    f = np.load(path)
    o = _oracle(_name(path))
    assert np.ptp(o["dF_dv"]) == 0.0
    assert _rel(o["grad"], f["grad_ref"]) <= 1e-9


def test_column_scaling_differs_from_the_reference_for_bernoulli():
    """the size of the deviation on one Bernoulli case: the reference's kernel gradient is off by up to one per cent"""
    name = "bernoulli_matern32_ard_n60"
    col, row = _oracle(name)["grad"], _oracle(name, row_scaling=True)["grad"]
    d = np.abs(col - row) / np.maximum(np.abs(col), 1e-12)
    assert 5e-3 < d.max() < 2e-2


def test_dkl_dbeta_identity_with_jitter():
    """diag(KB^T (Ai - Ai^2)) = (|e_j - Ai_:j|^2 + j (|Ai_:j|^2 - Ai_jj)) / beta_j when Ai = (I + BKB + j I)^-1"""
    rng = np.random.default_rng(3)
    N, j = 40, 1e-3
    X = rng.normal(size=(N, 2))
    K = np.exp(-0.5 * ((X[:, None] - X[None]) ** 2).sum(-1))
    be = rng.uniform(0.3, 3, N) * np.where(rng.uniform(size=N) < 0.3, -1, 1)
    Ai = np.linalg.inv(np.eye(N) * (1 + j) + K * be[:, None] * be[None])
    ref = np.diag((K * be[:, None]).T.dot(Ai - Ai.dot(Ai)))
    dev = (((np.eye(N) - Ai) ** 2).sum(0) + j * ((Ai ** 2).sum(0) - np.diag(Ai))) / be
    assert _rel(dev, ref) <= 1e-12


def _bound(name, theta_shift=None, alpha=None, beta=None):
    from make_vargauss import reference_inference
    parts, lik_spec, N, seed, _ = vo.CASES[name]
    X, Y, a0, b0, _ = vo.case_data(name)
    parts = [dict(p) for p in parts]
    if theta_shift is not None:
        q, key, h = theta_shift
        v = np.array(parts[q][key], dtype=np.float64)
        if v.ndim:
            v[h[1]] += h[0]
        else:
            v = v + h[0]
        parts[q][key] = v if v.ndim else float(v)
    _, lml, _, _, _, _, _ = reference_inference(parts, lik_spec, X, Y, a0 if alpha is None else alpha,
                                                b0 if beta is None else beta)
    return float(lml)


@needs_ref
@pytest.mark.parametrize("name", ["bernoulli_matern32_ard_n60", "bernoulli_m52_x_rbf_bias_n128"])
def test_oracle_kernel_gradient_is_the_derivative_of_the_reference_bound(name):
    o = _oracle(name)
    h = 1e-5
    parts = vo.CASES[name][0]
    got = []
    for q, p in enumerate(parts):
        for key in ("variance", "lengthscale"):
            if key not in p:
                continue
            for i in range(np.size(p[key])):
                num = (_bound(name, (q, key, (h, i))) - _bound(name, (q, key, (-h, i)))) / (2 * h)
                got.append(num)
    row = _oracle(name, row_scaling=True)["grad"]
    np.testing.assert_allclose(o["grad"], got, rtol=1e-6, atol=1e-6 * np.abs(got).max())
    assert np.abs(row - got).max() > 1e3 * np.abs(o["grad"] - got).max()


class HostVarGaussEngine(object):
    """gpx_vargauss_begin / gpx_vargauss_finish on the host through the oracle"""

    def __init__(self, device=0):
        self.calls, self.eval_serial = [], 0

    def set_data(self, X, Y):
        self.calls.append(("set_data",))
        self.X, self.Y = np.array(X, dtype=np.float64), np.array(Y, dtype=np.float64)
        self.N = X.shape[0]

    def vargauss_begin(self, parts, alpha, beta, max_tries=5):
        from test_laplace_cpu import _parts_of
        self.calls.append(("begin",))
        if not np.all(np.isfinite(beta)) or np.any(np.asarray(beta) == 0):
            raise gpy_b200._ffi.GpxArgumentError("beta must be finite and non-zero")
        self.args = (_parts_of(parts), self.X, self.Y, np.array(alpha), np.array(beta))
        o = vo.vargauss_eval(*self.args, _GivenDF(np.zeros(self.N), np.zeros(self.N)))
        return o["m"], o["var"], o["KL"], o["jitter"]

    def vargauss_finish(self, dF_dm, dF_dv):
        self.calls.append(("finish",))
        self.eval_serial += 1
        o = vo.vargauss_eval(*self.args, _GivenDF(dF_dm, dF_dv))
        return o["dalpha"], o["dbeta"], o["grad"]


class _GivenDF(object):
    def __init__(self, dm, dv):
        self.dm, self.dv = np.asarray(dm).reshape(-1, 1), np.asarray(dv).reshape(-1, 1)

    def variational_expectations(self, Y, m, v, Y_metadata=None):
        return np.zeros_like(m), self.dm, self.dv, None


_KINDS = {"rbf": gpy_b200.RBF, "exponential": gpy_b200.Exponential, "matern32": gpy_b200.Matern32,
          "matern52": gpy_b200.Matern52}


def _mirror_kernel(parts):
    """the mirror's kernel for a single stationary part or tests/laplace_oracle.COMPOSITE"""
    if len(parts) == 1:
        p = parts[0]
        return _KINDS[p["kind"]](3, variance=p["variance"], lengthscale=p["lengthscale"], ARD=p["ARD"])
    k = gpy_b200.RBF(3, variance=1.3, lengthscale=[0.9, 1.4, 2.1], ARD=True)
    m = gpy_b200.Matern52(2, variance=1.1, lengthscale=1.2, active_dims=[0, 1])
    return gpy_b200.Add([gpy_b200.Prod([k, m]), gpy_b200.Bias(3, variance=0.4)])


@pytest.mark.parametrize("name", ["bernoulli_rbf_ard_n127", "studentt_matern52_ard_n128", "bernoulli_m52_x_rbf_bias_n128"])
def test_mirror_model_over_a_host_engine_matches_the_oracle(name):
    parts, lik_spec, N, seed, _ = vo.CASES[name]
    X, Y, alpha, beta, _ = vo.case_data(name)
    lik = vo.make_likelihood(lik_spec, gpy_b200)
    eng = HostVarGaussEngine()
    m = GPVariationalGaussianApproximation(X, Y, _mirror_kernel(parts), lik, engine=eng)
    assert m.name == "VarGP"
    assert [p.name for p in m.flattened_parameters()][-2:] == ["alpha", "beta"]
    np.testing.assert_array_equal(m.alpha.values, np.zeros((N, 1)))
    np.testing.assert_array_equal(m.beta.values, np.ones(N))
    assert m.alpha.transform is None and m.beta.transform is None
    m.alpha.values[...] = alpha[:, None]
    m.beta.values[...] = beta
    m.parameters_changed()
    o = vo.vargauss_eval(parts, X, Y, alpha, beta, lik)
    assert abs(m.log_likelihood() - o["lml"]) <= 1e-12 * abs(o["lml"])
    np.testing.assert_allclose(m.alpha.gradient[:, 0], o["dalpha"], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(m.beta.gradient, o["dbeta"], rtol=1e-12, atol=1e-12)
    n = len(o["dL_dthetaL"])
    g = np.asarray(m.gradient)
    np.testing.assert_allclose(g[:o["grad"].size], o["grad"], rtol=1e-12, atol=1e-12)
    if n:
        np.testing.assert_allclose(g[o["grad"].size:o["grad"].size + n], o["dL_dthetaL"], rtol=1e-12, atol=1e-12)
    assert [c[0] for c in eng.calls][-2:] == ["begin", "finish"]


def test_mirror_rejects_what_the_reference_rejects():
    X, Y, alpha, beta, _ = vo.case_data("bernoulli_rbf_iso_n60")
    eng = HostVarGaussEngine()
    m = GPVariationalGaussianApproximation(X, Y, gpy_b200.RBF(3), gpy_b200.Bernoulli(), engine=eng)
    for bad in (0.0, np.nan, np.inf):
        b = np.ones(X.shape[0])
        b[5] = bad
        with pytest.raises(ValueError):
            VarGauss(m.alpha, b, engine=eng).inference(m.kern, X, m.likelihood, Y)
    with pytest.raises(NotImplementedError):
        VarGauss(m.alpha, m.beta, engine=eng).inference(m.kern, X, m.likelihood, Y, mean_function=object())
    with pytest.raises(AssertionError):
        VarGauss(m.alpha, m.beta, engine=eng).inference(m.kern, X, m.likelihood, np.hstack([Y, Y]))
