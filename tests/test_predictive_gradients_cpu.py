"""GP.predictive_gradients without a GPU: the NumPy restatement of tests/predictive_gradients_oracle.py against the
reference's own GP / SparseGP (the committed fixtures of tests/golden/predictive_gradients) and against central
differences of the prediction, and the mirror's host logic (device route, active-dims scatter, normalizer, the `kern=`
and generic-path fallbacks, the rejections) on test doubles of the engine and of the stand-alone kernel calls that answer
from that restatement."""
import glob
import os
import types

import numpy as np
import pytest
from scipy.linalg import cho_factor, cho_solve

import gpy_b200
import predictive_gradients_oracle as po
from gpy_b200 import _ffi
from gpy_b200.inference import HostPosterior, PosteriorExact
from gpy_b200.sparse import SparsePosterior
from oracle import gpy_oracle as o
from sparse_composite_oracle import CompositeOracle

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = sorted(glob.glob(os.path.join(HERE, "golden", "predictive_gradients", "*.npz")))


def _noise(f):
    n = f["noise"]
    return float(n) if n.ndim == 0 else n


def _oracle(f):
    """the restatement's Jacobians for a fixture's inputs"""
    kern = CompositeOracle(po.KERNELS[str(f["kernel"])])
    X, Y, Xnew = f["X"], f["Y"], f["Xnew"]
    if bool(f["sparse"]):
        wv, wi = po.sparse_posterior(kern, X, Y, f["Z"], _noise(f))
        return po.jacobians(kern, wv, wi, Xnew, f["Z"])
    Yn, _, std = po.standardize(Y) if bool(f["normalizer"]) else (Y, None, None)
    wv, wi = po.exact_posterior(kern, X, Yn, _noise(f))
    mj, vj = po.jacobians(kern, wv, wi, Xnew, X)
    return po.denormalize(mj, vj, std) if bool(f["normalizer"]) else (mj, vj)


def test_fixture_set_covers_the_kinds_composites_outputs_normalizer_het_sparse_and_an_ill_conditioned_case():
    names = {os.path.basename(p)[:-4] for p in FIXTURES}
    assert {"exact_%s" % k for k in po.KERNELS} <= names
    assert {"exact_rbf_bias_white_p3", "exact_rbf_ard_p1_norm", "exact_m52_x_rbf_p3_norm", "exact_rbf_ard_het",
            "exact_rbf_ard_illcond", "sparse_rbf_ard_scalar", "sparse_rbf_bias_white_het",
            "sparse_m52_x_rbf_p3_scalar"} <= names
    f = np.load(os.path.join(HERE, "golden", "predictive_gradients", "exact_rbf_ard_illcond.npz"))
    assert 3e7 <= float(f["cond"]) <= 3e8


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[:-4])
def test_oracle_matches_the_reference_fixtures(path):
    f = np.load(path)
    mj, vj = _oracle(f)
    assert mj.shape == f["mean_jac"].shape and vj.shape == f["var_jac"].shape
    # cond(Ky) ~ 6e7: the two fp64 inverses differ by ~cond * eps, and the variance Jacobian, a difference of nearly equal
    # terms (K(X*, X) Ky^-1 is close to a row of the identity's neighbourhood), loses two more digits
    tm, tv = (1e-12, 1e-12) if "illcond" not in path else (1e-8, 1e-6)
    np.testing.assert_allclose(mj, f["mean_jac"], rtol=0, atol=tm * np.abs(f["mean_jac"]).max())
    np.testing.assert_allclose(vj, f["var_jac"], rtol=0, atol=tv * np.abs(f["var_jac"]).max())


def _predict(kern, wv, wi, Xpred, Xnew):
    """posterior.py:238-302 (diagonal variance) with the restatement's kernel"""
    Kx = kern.K(Xpred, Xnew)
    return np.dot(Kx.T, wv), kern.Kdiag(Xnew) - np.sum(np.dot(wi, Kx) * Kx, 0)


@pytest.mark.parametrize("kname", ["rbf_ard", "matern52_iso", "exponential_ard", "rbf_bias_white", "m52_x_rbf"])
@pytest.mark.parametrize("sparse", [False, True])
def test_oracle_matches_central_differences_of_predict(kname, sparse):
    """as the reference's test_model.py:1547-1574: each Jacobian against central differences of the prediction"""
    kern = CompositeOracle(po.KERNELS[kname])
    X, Y, Z, noise = po.case_data(120, 20, 3, 2, 5, False)
    wv, wi = po.sparse_posterior(kern, X, Y, Z, noise) if sparse else po.exact_posterior(kern, X, Y, noise)
    Xp = Z if sparse else X
    Xnew = np.random.default_rng(9).uniform(-1.5, 1.5, size=(5, 3))
    mj, vj = po.jacobians(kern, wv, wi, Xnew, Xp)
    h = 1e-6
    for q in range(3):
        E = np.zeros_like(Xnew)
        E[:, q] = h
        mp, vp = _predict(kern, wv, wi, Xp, Xnew + E)
        mm, vm = _predict(kern, wv, wi, Xp, Xnew - E)
        np.testing.assert_allclose(mj[:, q, :], (mp - mm) / (2 * h), rtol=1e-5, atol=1e-7)
        np.testing.assert_allclose(vj[:, q], (vp - vm) / (2 * h), rtol=1e-5, atol=1e-7)


# ---- host logic on test doubles -------------------------------------------------------------------------------------
class FakeEngine(object):
    """answers gpx_predictive_gradients / gpx_get from the restatement for the engine's own columns Xe"""

    def __init__(self, parts, Xe, Y, noise):
        self.kern, self.Xe = CompositeOracle(parts), Xe
        self.wv, self.wi = po.exact_posterior(self.kern, Xe, Y, noise)
        self.eval_serial, self.calls = 1, []

    def predictive_gradients(self, Xn):
        self.calls.append(Xn.shape)
        return po.jacobians(self.kern, self.wv, self.wi, Xn, self.Xe)

    def get(self, which):
        self.calls.append(which)
        return {"alpha": self.wv, "Kinv": self.wi}[which]


@pytest.fixture
def host_kernels(monkeypatch):
    """the stand-alone kernel calls answered by the restatement"""
    def kern_of(kind, ARD, variance, lengthscale, D):
        return o.StationaryOracle(kind, D, variance, lengthscale, ARD)
    monkeypatch.setattr(_ffi, "kern_K", lambda kind, ARD, v, ls, X, X2=None: kern_of(kind, ARD, v, ls, X.shape[1]).K(X, X2))
    monkeypatch.setattr(_ffi, "kern_Kdiag", lambda kind, v, N: np.full(N, v))
    monkeypatch.setattr(_ffi, "kern_grad_X", lambda kind, ARD, v, ls, X, dL, X2=None:
                        kern_of(kind, ARD, v, ls, X.shape[1]).gradients_X(np.asarray(dL), X, X2))


def _model(kern, parts, X, Y, noise=0.1, normalizer=None, engine_cols=None):
    """a GPRegression whose posterior is a device posterior over FakeEngine (no evaluation runs)"""
    m = gpy_b200.GPRegression.__new__(gpy_b200.GPRegression)
    m.kern, m.X, m.Y, m.output_dim = kern, X, Y, Y.shape[1]
    m.normalizer = normalizer
    Yn = Y
    if normalizer is not None:
        normalizer.scale_by(Y)
        Yn = normalizer.normalize(Y)
    eng = FakeEngine(parts, X if engine_cols is None else X[:, engine_cols], Yn, noise)
    key = kern._state_key() if hasattr(kern, "_state_key") else gpy_b200.kern.composite_state_key(kern)
    m.posterior = PosteriorExact(eng, X.shape[0], Y.shape[1], key)
    return m, eng


def _data(P=1, D=3, N=60, seed=3):
    X, Y, _, _ = po.case_data(N, 2, D, P, seed, False)
    return X, Y, np.random.default_rng(seed + 1).uniform(-2, 2, size=(4, D))


def test_device_route_shapes_and_one_engine_call():
    X, Y, Xnew = _data(P=3)
    k = gpy_b200.RBF(3, variance=0.9, lengthscale=[0.8, 1.5, 2.2], ARD=True)
    m, eng = _model(k, po.KERNELS["rbf_ard"], X, Y)
    mj, vj = m.predictive_gradients(Xnew)
    assert mj.shape == (4, 3, 3) and vj.shape == (4, 3)
    assert eng.calls == [(4, 3)]
    wv, wi = po.exact_posterior(CompositeOracle(po.KERNELS["rbf_ard"]), X, Y, 0.1)
    rm, rv = po.jacobians(CompositeOracle(po.KERNELS["rbf_ard"]), wv, wi, Xnew, X)
    np.testing.assert_array_equal(mj, rm)
    np.testing.assert_array_equal(vj, rv)


def test_single_kernel_on_a_subset_of_columns_scatters_into_them():
    X, Y, Xnew = _data(D=4)
    k = gpy_b200.Matern32(2, variance=1.1, lengthscale=0.7, active_dims=[1, 3])
    part = [dict(kind="matern32", term=0, dims=[0, 1], variance=1.1, lengthscale=0.7)]
    m, eng = _model(k, part, X, Y, engine_cols=[1, 3])
    mj, vj = m.predictive_gradients(Xnew)
    assert eng.calls == [(4, 2)] and mj.shape == (4, 4, 1) and vj.shape == (4, 4)
    assert not mj[:, [0, 2]].any() and not vj[:, [0, 2]].any()
    ref = po.jacobians(eng.kern, eng.wv, eng.wi, Xnew[:, [1, 3]], X[:, [1, 3]])
    np.testing.assert_array_equal(mj[:, [1, 3]], ref[0])
    np.testing.assert_array_equal(vj[:, [1, 3]], ref[1])


@pytest.mark.parametrize("P", [1, 3])
def test_normalizer_scales_as_the_reference(P):
    X, Y, Xnew = _data(P=P)
    Y = 5.0 * Y + 2.0
    k = gpy_b200.RBF(3, variance=0.9, lengthscale=[0.8, 1.5, 2.2], ARD=True)
    m, eng = _model(k, po.KERNELS["rbf_ard"], X, Y, normalizer=gpy_b200.model.Standardize())
    mj, vj = m.predictive_gradients(Xnew)
    rm, rv = po.jacobians(eng.kern, eng.wv, eng.wi, Xnew, X)
    std = Y.std(0)
    np.testing.assert_allclose(mj, rm * std, rtol=1e-14)
    if P > 1:
        assert vj.shape == (4, 3, P)                      # inverse_covariance adds the output axis (gp.py:469-470)
        np.testing.assert_allclose(vj, rv[..., None] * std ** 2, rtol=1e-14)
    else:
        np.testing.assert_allclose(vj, rv * std ** 2, rtol=1e-14)


def test_another_kernel_takes_the_reference_formula_on_the_fetched_posterior(host_kernels):
    X, Y, Xnew = _data()
    k = gpy_b200.RBF(3, variance=0.9, lengthscale=[0.8, 1.5, 2.2], ARD=True)
    m, eng = _model(k, po.KERNELS["rbf_ard"], X, Y)
    other = gpy_b200.Matern52(3, variance=1.2, lengthscale=1.3)
    mj, vj = m.predictive_gradients(Xnew, kern=other)
    assert set(eng.calls) == {"alpha", "Kinv"}            # no device Jacobian call: the posterior is fetched instead
    rm, rv = po.jacobians(CompositeOracle(po.KERNELS["matern52_iso"]), eng.wv, eng.wi, Xnew, X)
    np.testing.assert_allclose(mj, rm, rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(vj, rv, rtol=1e-12, atol=1e-14)


def test_generic_path_posterior_takes_the_reference_formula(host_kernels):
    X, Y, Xnew = _data()
    k = gpy_b200.RBF(3, variance=1.2, lengthscale=1.3)
    kern = CompositeOracle(po.KERNELS["rbf_iso"])
    Ky = kern.K(X) + (0.1 + 1e-8) * np.eye(X.shape[0])
    L = np.linalg.cholesky(Ky)
    alpha = cho_solve((L, True), Y)
    m = gpy_b200.GPRegression.__new__(gpy_b200.GPRegression)
    m.kern, m.X, m.Y, m.output_dim, m.normalizer = k, X, Y, 1, None
    m.posterior = HostPosterior(L, alpha, None)
    mj, vj = m.predictive_gradients(Xnew)
    rm, rv = po.jacobians(kern, alpha, cho_solve(cho_factor(Ky, lower=True), np.eye(X.shape[0])), Xnew, X)
    np.testing.assert_allclose(mj, rm, rtol=1e-10, atol=1e-13)
    np.testing.assert_allclose(vj, rv, rtol=1e-10, atol=1e-13)


@pytest.mark.parametrize("leaf", ["ratquad", "stdperiodic"])
def test_ratquad_and_stdperiodic_raise_not_implemented_and_never_reach_the_device(leaf):
    X, Y, Xnew = _data()
    k = (gpy_b200.RatQuad(3, variance=1.0, lengthscale=1.0, power=2.0) if leaf == "ratquad"
         else gpy_b200.StdPeriodic(3, variance=1.0, period=1.0, lengthscale=1.0))
    m, eng = _model(k, po.KERNELS["rbf_iso"], X, Y)
    with pytest.raises(NotImplementedError):
        m.predictive_gradients(Xnew)
    assert "Kinv" not in eng.calls and all(not isinstance(c, tuple) for c in eng.calls)


def test_stale_posterior_raises():
    X, Y, Xnew = _data()
    k = gpy_b200.RBF(3, variance=0.9, lengthscale=[0.8, 1.5, 2.2], ARD=True)
    m, eng = _model(k, po.KERNELS["rbf_ard"], X, Y)
    eng.eval_serial += 1                                  # a later evaluation on the same engine
    with pytest.raises(RuntimeError):
        m.predictive_gradients(Xnew)
    assert eng.calls == []


# ---- the host formula with composite and static kernels ---------------------------------------------------------------
def _generic_model(kern, parts, X, Y, noise=0.1):
    """a GPRegression on the generic inference path: a HostPosterior over the restatement's factor"""
    kern_o = CompositeOracle(parts)
    Ky = kern_o.K(X) + (noise + 1e-8) * np.eye(X.shape[0])
    L = np.linalg.cholesky(Ky)
    m = gpy_b200.GPRegression.__new__(gpy_b200.GPRegression)
    m.kern, m.X, m.Y, m.output_dim, m.normalizer, m.mean_function = kern, X, Y, Y.shape[1], None, None
    m.posterior = HostPosterior(L, cho_solve((L, True), Y), None)
    return m, kern_o, m.posterior.woodbury_vector, cho_solve((L, True), np.eye(X.shape[0]))


def _sparse_model(kern, parts, X, Y, Z, noise=0.08):
    """a SparseGPRegression whose posterior holds the restatement's VarDTC woodbury vector and woodbury_inv"""
    kern_o = CompositeOracle(parts)
    wv, wi = po.sparse_posterior(kern_o, X, Y, Z, noise)
    m = gpy_b200.SparseGPRegression.__new__(gpy_b200.SparseGPRegression)
    m.kern, m.X, m.Y, m.likelihood = kern, X, Y, None
    m.Z = types.SimpleNamespace(values=Z)
    m.posterior = SparsePosterior(wi, wv, None, None)
    return m, kern_o, wv, wi


@pytest.mark.parametrize("other", ["rbf_bias_white", "m52_x_rbf"])
def test_composite_kern_on_the_exact_model_takes_the_reference_formula(host_kernels, other):
    X, Y, Xnew = _data(P=2)
    k = gpy_b200.RBF(3, variance=0.9, lengthscale=[0.8, 1.5, 2.2], ARD=True)
    m, eng = _model(k, po.KERNELS["rbf_ard"], X, Y)
    mj, vj = m.predictive_gradients(Xnew, kern=po.mirror_kernel(po.KERNELS[other]))
    assert set(eng.calls) == {"alpha", "Kinv"}
    rm, rv = po.jacobians(CompositeOracle(po.KERNELS[other]), eng.wv, eng.wi, Xnew, X)
    np.testing.assert_allclose(mj, rm, rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(vj, rv, rtol=1e-12, atol=1e-14)


@pytest.mark.parametrize("kname", ["rbf_bias_white", "m52_x_rbf"])
def test_composite_on_the_generic_path_takes_the_reference_formula(host_kernels, kname):
    X, Y, Xnew = _data()
    m, kern_o, wv, wi = _generic_model(po.mirror_kernel(po.KERNELS[kname]), po.KERNELS[kname], X, Y)
    mj, vj = m.predictive_gradients(Xnew)
    rm, rv = po.jacobians(kern_o, wv, wi, Xnew, X)
    np.testing.assert_allclose(mj, rm, rtol=1e-10, atol=1e-13)
    np.testing.assert_allclose(vj, rv, rtol=1e-10, atol=1e-13)


@pytest.mark.parametrize("static", ["white", "bias"])
def test_a_lone_static_kernel_has_zero_jacobians(host_kernels, static):
    """static.py:27-31, 41-42: neither K(X*, X) nor Kdiag depends on the inputs"""
    X, Y, Xnew = _data(P=2)
    k = (gpy_b200.White if static == "white" else gpy_b200.Bias)(3, variance=0.6)
    m, _, _, _ = _generic_model(k, [dict(kind=static, term=0, variance=0.6)], X, Y)
    mj, vj = m.predictive_gradients(Xnew)
    assert mj.shape == (4, 3, 2) and vj.shape == (4, 3)
    assert not mj.any() and not vj.any()


def test_composite_kern_on_the_sparse_model_takes_the_reference_formula(host_kernels):
    X, Y, Z, _ = po.case_data(120, 20, 3, 2, 11, False)
    Xnew = np.random.default_rng(12).uniform(-2, 2, (5, 3))
    m, _, wv, wi = _sparse_model(po.mirror_kernel(po.KERNELS["rbf_ard"]), po.KERNELS["rbf_ard"], X, Y, Z)
    mj, vj = m.predictive_gradients(Xnew, kern=po.mirror_kernel(po.KERNELS["rbf_bias_white"]))
    rm, rv = po.jacobians(CompositeOracle(po.KERNELS["rbf_bias_white"]), wv, wi, Xnew, Z)
    np.testing.assert_allclose(mj, rm, rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(vj, rv, rtol=1e-12, atol=1e-14)


def _central_differences(predict, Xnew, h=1e-6):
    """(mean, variance) Jacobians of predict by central differences, as the reference's test_model.py:1547-1574"""
    dm, dv = [], []
    for q in range(Xnew.shape[1]):
        E = np.zeros_like(Xnew)
        E[:, q] = h
        (mp, vp), (mm, vm) = predict(Xnew + E), predict(Xnew - E)
        dm.append((mp - mm) / (2 * h))
        dv.append(((vp - vm) / (2 * h))[:, 0])
    return np.stack(dm, axis=1), np.stack(dv, axis=1)


@pytest.mark.parametrize("kname", ["rbf_ard", "matern32_iso", "rbf_bias_white", "m52_x_rbf"])
def test_mirror_host_route_matches_central_differences_of_its_predict(host_kernels, kname):
    """the mirror's own predictive_gradients (host formula) against central differences of the mirror's own predict, on the
    generic exact path and, through another kernel object of the same kernel, on the sparse model"""
    X, Y, Z, _ = po.case_data(120, 20, 3, 2, 13, False)
    Xnew = np.random.default_rng(14).uniform(-1.5, 1.5, (5, 3))
    m, _, _, _ = _generic_model(po.mirror_kernel(po.KERNELS[kname]), po.KERNELS[kname], X, Y)
    mj, vj = m.predictive_gradients(Xnew)
    fm, fv = _central_differences(lambda x: m.predict(x, include_likelihood=False), Xnew)
    np.testing.assert_allclose(mj, fm, rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(vj, fv, rtol=1e-5, atol=1e-7)
    s, _, _, _ = _sparse_model(po.mirror_kernel(po.KERNELS[kname]), po.KERNELS[kname], X, Y, Z)
    mj, vj = s.predictive_gradients(Xnew, kern=po.mirror_kernel(po.KERNELS[kname]))
    fm, fv = _central_differences(lambda x: s.predict(x, include_likelihood=False), Xnew)
    np.testing.assert_allclose(mj, fm, rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(vj, fv, rtol=1e-5, atol=1e-7)
