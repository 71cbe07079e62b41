"""GP.predictive_gradients on the device (gpx_predictive_gradients, gpx_sparse_predictive_gradients): parity with the
reference's fixtures and with the NumPy restatement of tests/predictive_gradients_oracle.py over shapes at the MAX_P and
tile edges on both tensor paths, consistency with central differences of the device prediction, and the invariants of
the two entries (determinism, an untouched posterior, the documented launch counts, the rejections)."""
import glob
import os

import numpy as np
import pytest
from scipy.linalg import cho_factor, cho_solve

import gpy_b200
import predictive_gradients_oracle as po
from predictive_gradients_oracle import mirror_kernel
import sparse_composite_oracle as so
from gpy_b200 import _ffi
from sparse_composite_oracle import CompositeOracle

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = sorted(glob.glob(os.path.join(HERE, "golden", "predictive_gradients", "*.npz")))
SINGLE = ("rbf", "exponential", "matern32", "matern52")
TOL = 1e-8   # of each Jacobian's largest entry, cond(Ky) <= 1e6


def evaluate(e, parts, X, Y, noise):
    """one exact evaluation of the parts on engine e"""
    e.set_data(X, Y)
    p = parts[0]
    if len(parts) == 1 and p["kind"] in SINGLE:
        ls = p["lengthscale"]
        if np.ndim(noise) > 0:
            return e.exact_eval_het(p["kind"], p.get("ARD", False), p["variance"], ls, noise)
        return e.exact_eval(p["kind"], p.get("ARD", False), p["variance"], ls, noise)
    return e.exact_eval_multi([so.descriptor(q) for q in parts], noise)


def sparse_evaluate(e, parts, X, Y, Z, noise):
    e.sparse_set_data(X, Y)
    return e.sparse_eval_multi([so.descriptor(q) for q in parts], Z, noise)


def kmm_cond(kern, Z):
    """cond(Kmm + 1e-8 I): the sparse Jacobians rest on woodbury_inv = Lm^-T (I - B^-1) Lm^-1, which an fp64 evaluation
    on either side carries with ~cond * eps relative error. The 1e-8 bar holds for cond <= 1e6, as for Ky."""
    return np.linalg.cond(kern.K(Z) + po.JITTER * np.eye(Z.shape[0]))


def spread_points(X, M):
    """M rows of X by farthest-point selection: inducing points that keep cond(Kmm) low"""
    idx = [0]
    d = np.linalg.norm(X - X[0], axis=1)
    for _ in range(M - 1):
        i = int(np.argmax(d))
        idx.append(i)
        d = np.minimum(d, np.linalg.norm(X - X[i], axis=1))
    return X[idx].copy()


def assert_close(got, want, tol=TOL):
    assert got.shape == want.shape
    err = np.abs(got - want).max()
    assert err <= tol * np.abs(want).max(), (err, np.abs(want).max())


def refined_solve(A, B, iters=3):
    """A^-1 B with iterative refinement, residuals in extended precision (x87 long double): the extended-precision
    reference of the ill-conditioned case"""
    c = cho_factor(A, lower=True)
    x = cho_solve(c, B)
    Al, Bl = A.astype(np.longdouble), B.astype(np.longdouble)
    for _ in range(iters):
        r = Bl - Al @ x.astype(np.longdouble)
        x = x + cho_solve(c, r.astype(np.float64))
    return x


# ---- parity with the reference's fixtures ---------------------------------------------------------------------------
def _fixture_model(f, e):
    kname, X, Y, noise = str(f["kernel"]), f["X"], f["Y"], f["noise"]
    kern = mirror_kernel(po.KERNELS[kname])
    if bool(f["sparse"]):
        lik, meta = None, None
        if noise.ndim > 0:
            meta = {"output_index": np.arange(X.shape[0])[:, None]}
            lik = gpy_b200.HeteroscedasticGaussian(meta)
            lik.variance.values[...] = noise.reshape(lik.variance.values.shape)
        m = gpy_b200.SparseGPRegression(X, Y, kern, Z=f["Z"], engine=e, likelihood=lik, Y_metadata=meta)
        if noise.ndim == 0:
            m.likelihood.variance.values[...] = float(noise)
            m.parameters_changed()
        return m
    if noise.ndim > 0:
        m = gpy_b200.GPHeteroscedasticRegression(X, Y, kern, engine=e)
        m.likelihood.variance.values[...] = noise.reshape(m.likelihood.variance.values.shape)
        m.parameters_changed()
        return m
    return gpy_b200.GPRegression(X, Y, kern, noise_var=float(noise), normalizer=True if bool(f["normalizer"]) else None,
                                 engine=e)


@pytest.mark.parametrize("oz", [0, 1])
@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[:-4])
def test_matches_the_reference_fixtures(path, oz):
    f = np.load(path)
    e = _ffi.Engine(0)
    e.set_option("ozaki", oz)
    m = _fixture_model(f, e)
    mj, vj = m.predictive_gradients(f["Xnew"])
    if "illcond" not in path:
        if bool(f["sparse"]):
            assert kmm_cond(CompositeOracle(po.KERNELS[str(f["kernel"])]), f["Z"]) <= 1e6
        assert_close(mj, f["mean_jac"])
        assert_close(vj, f["var_jac"])
        return
    # cond(Ky) ~ 6e7: within 16x the fp64 reference's own error against an extended-precision evaluation
    kern = CompositeOracle(po.KERNELS[str(f["kernel"])])
    X, Xnew = f["X"], f["Xnew"]
    Ky = kern.K(X) + (float(f["noise"]) + po.JITTER) * np.eye(X.shape[0])
    wv = refined_solve(Ky, f["Y"])
    V = refined_solve(Ky, kern.K(X, Xnew))
    mx = kern.gradients_X(np.broadcast_to(wv[:, 0][None, :], (Xnew.shape[0], X.shape[0])), Xnew, X)[:, :, None]
    vx = -2.0 * kern.gradients_X(np.ascontiguousarray(V.T), Xnew, X)
    for got, ref, ext in ((mj, f["mean_jac"], mx), (vj, f["var_jac"], vx)):
        e_ref, e_dev = np.abs(ref - ext).max(), np.abs(got - ext).max()
        assert e_dev <= 16 * e_ref + 1e-15 * np.abs(ext).max(), (e_dev, e_ref)


# ---- shapes: N, tensor path, M* at the MAX_P and tile edges ---------------------------------------------------------
MSTARS = (1, 7, 8, 9, 129)


@pytest.mark.parametrize("oz", [0, 1])
@pytest.mark.parametrize("N", [150, 700, 1300])
def test_single_kernel_over_N_tensor_paths_and_test_point_counts(N, oz):
    parts = po.KERNELS["matern52_ard"]
    X, Y, _, noise = po.case_data(N, 2, 3, 2, N, False)
    kern = CompositeOracle(parts)
    wv, wi = po.exact_posterior(kern, X, Y, noise)
    e = _ffi.Engine(0)
    e.set_option("ozaki", oz)
    evaluate(e, parts, X, Y, noise)
    rng = np.random.default_rng(N + oz)
    for Ms in MSTARS:
        Xnew = rng.uniform(-2.2, 2.2, size=(Ms, 3))
        mj, vj = e.predictive_gradients(Xnew)
        rm, rv = po.jacobians(kern, wv, wi, Xnew, X)
        assert_close(mj, rm)
        assert_close(vj, rv)


@pytest.mark.parametrize("oz", [0, 1])
@pytest.mark.parametrize("case", ["rbf_bias_white", "m52_x_rbf", "het"])
def test_composites_and_heteroscedastic(case, oz):
    kname = "rbf_ard" if case == "het" else case
    parts = po.KERNELS[kname]
    X, Y, _, noise = po.case_data(700, 2, 3, 3 if case == "rbf_bias_white" else 1, 17, case == "het")
    kern = CompositeOracle(parts)
    wv, wi = po.exact_posterior(kern, X, Y, noise)
    e = _ffi.Engine(0)
    e.set_option("ozaki", oz)
    evaluate(e, parts, X, Y, noise)
    Xnew = np.random.default_rng(5).uniform(-2.2, 2.2, size=(129, 3))
    mj, vj = e.predictive_gradients(Xnew)
    rm, rv = po.jacobians(kern, wv, wi, Xnew, X)
    assert_close(mj, rm)
    assert_close(vj, rv)


@pytest.mark.parametrize("M", [50, 129, 300])
@pytest.mark.parametrize("case", ["matern52_ard", "m52_x_rbf", "rbf_bias_white_het"])
def test_sparse_over_inducing_counts(M, case):
    """inducing points spread by farthest-point selection: cond(Kmm + 1e-8 I) stays <= 1e6 (2.4e4 at most here), so the
    1e-8 bar of the exact model applies"""
    het = case.endswith("_het")
    parts = po.KERNELS[case[:-4] if het else case]
    X, Y, _, noise = po.case_data(2000, M, 3, 2, M, het)
    Z = spread_points(X, M)
    kern = CompositeOracle(parts)
    assert kmm_cond(kern, Z) <= 1e6
    wv, wi = po.sparse_posterior(kern, X, Y, Z, noise)
    e = _ffi.Engine(0)
    sparse_evaluate(e, parts, X, Y, Z, noise)
    rng = np.random.default_rng(M)
    for Ms in (1, 9, 129):
        Xnew = rng.uniform(-2.2, 2.2, size=(Ms, 3))
        mj, vj = e.sparse_predictive_gradients(Xnew)
        rm, rv = po.jacobians(kern, wv, wi, Xnew, Z)
        assert_close(mj, rm)
        assert_close(vj, rv)


def test_sparse_with_an_ill_conditioned_kmm():
    """RBF(ARD) on 300 random inducing points: cond(Kmm + 1e-8 I) = 6.2e9. Both fp64 woodbury_inv carry ~cond * eps
    (1.4e-6) relative error, and so does the woodbury vector: that is the bar here"""
    parts = po.KERNELS["rbf_ard"]
    X, Y, Z, noise = po.case_data(2000, 300, 3, 2, 300, False)
    kern = CompositeOracle(parts)
    c = kmm_cond(kern, Z)
    assert 1e9 <= c <= 1e10
    wv, wi = po.sparse_posterior(kern, X, Y, Z, noise)
    e = _ffi.Engine(0)
    sparse_evaluate(e, parts, X, Y, Z, noise)
    Xnew = np.random.default_rng(300).uniform(-2.2, 2.2, size=(129, 3))
    mj, vj = e.sparse_predictive_gradients(Xnew)
    rm, rv = po.jacobians(kern, wv, wi, Xnew, Z)
    assert_close(mj, rm, max(TOL, c * np.finfo(float).eps))
    assert_close(vj, rv, c * np.finfo(float).eps)


# ---- consistency with the device prediction ---------------------------------------------------------------------------
def test_jacobians_match_central_differences_of_the_device_predict_at_N_4096():
    """central differences with step 1e-5 of gpx_predict's mean and variance; the difference quotient is good to
    ~1e-9 of the largest entry here (truncation h^2, rounding eps / h), the tolerance is 1e-6 of it"""
    parts = po.KERNELS["rbf_ard"]
    X, Y, _, noise = po.case_data(4096, 2, 3, 1, 41, False)
    e = _ffi.Engine(0)
    evaluate(e, parts, X, Y, noise)
    Xnew = np.random.default_rng(4).uniform(-2.0, 2.0, size=(16, 3))
    mj, vj = e.predictive_gradients(Xnew)
    h = 1e-5
    for q in range(3):
        E = np.zeros_like(Xnew)
        E[:, q] = h
        mp, vp = e.predict(Xnew + E)
        mm, vm = e.predict(Xnew - E)
        assert np.abs(mj[:, q, :] - (mp - mm) / (2 * h)).max() <= 1e-6 * np.abs(mj).max()
        assert np.abs(vj[:, q] - ((vp - vm) / (2 * h))[:, 0]).max() <= 1e-6 * np.abs(vj).max()


# ---- invariants -------------------------------------------------------------------------------------------------------
def _exact_state(e, Xs):
    out = {w: e.get(w) for w in _ffi.GET}
    out["mu"], out["var"] = e.predict(Xs)
    out["mu_full"], out["cov"] = e.predict(Xs, full_cov=True)
    out["stats"] = e.stats()
    return out


def _sparse_state(e):
    out = {w: e.sparse_get(w) for w in e.SPARSE_GET}
    out["stats"] = e.stats()
    return out


def _same(a, b):
    for k in a:
        if isinstance(a[k], dict):
            assert a[k] == b[k], k
        else:
            np.testing.assert_array_equal(a[k], b[k], err_msg=k)


def _reduction_launches(sumD, P):
    g = 4 if sumD <= 8 else 2 if sumD <= 16 else 1
    return -(-(P + 1) // g) + 1


@pytest.mark.parametrize("which", ["single", "composite"])
def test_exact_calls_are_deterministic_leave_the_posterior_alone_and_count_their_launches(which):
    parts = po.KERNELS["rbf_ard" if which == "single" else "m52_x_rbf"]
    X, Y, _, noise = po.case_data(1300, 2, 3, 2, 23, False)
    e = _ffi.Engine(0)
    evaluate(e, parts, X, Y, noise)
    rng = np.random.default_rng(1)
    Xs, Xnew = rng.uniform(-2, 2, (20, 3)), rng.uniform(-2, 2, (129, 3))
    e.get("Kinv")                     # a K^-1 made by gpx_get stays valid too
    before = _exact_state(e, Xs)
    l0 = e.total_launches()
    a = e.predictive_gradients(Xnew)
    sumD = 3 if which == "single" else 4
    assert e.total_launches() - l0 == 2 + 3 * -(-129 // 8) + _reduction_launches(sumD, 2)
    b = e.predictive_gradients(Xnew)
    np.testing.assert_array_equal(a[0], b[0])
    np.testing.assert_array_equal(a[1], b[1])
    _same(before, _exact_state(e, Xs))


def test_sparse_calls_are_deterministic_leave_the_posterior_alone_and_count_their_launches():
    parts = po.KERNELS["rbf_bias_white"]
    X, Y, Z, noise = po.case_data(3000, 129, 3, 3, 29, False)
    e = _ffi.Engine(0)
    sparse_evaluate(e, parts, X, Y, Z, noise)
    Xnew = np.random.default_rng(2).uniform(-2, 2, (77, 3))
    before = _sparse_state(e)
    l0 = e.total_launches()
    a = e.sparse_predictive_gradients(Xnew)
    assert e.total_launches() - l0 == 8 + _reduction_launches(3, 3)      # woodbury_inv formed by the first call
    l0 = e.total_launches()
    b = e.sparse_predictive_gradients(Xnew)
    assert e.total_launches() - l0 == 3 + _reduction_launches(3, 3)      # and kept for the later calls
    np.testing.assert_array_equal(a[0], b[0])
    np.testing.assert_array_equal(a[1], b[1])
    _same(before, _sparse_state(e))
    # a new evaluation drops the kept woodbury_inv: the next call forms the new one
    e.sparse_eval_multi([so.descriptor(q) for q in parts], Z, 2.5 * noise)
    l0 = e.total_launches()
    c = e.sparse_predictive_gradients(Xnew)
    assert e.total_launches() - l0 == 8 + _reduction_launches(3, 3)
    kern = CompositeOracle(parts)
    wv, wi = po.sparse_posterior(kern, X, Y, Z, 2.5 * noise)
    rm, rv = po.jacobians(kern, wv, wi, Xnew, Z)
    assert_close(c[0], rm)
    assert_close(c[1], rv)


def test_rejections_leave_the_posterior_intact():
    L, p = _ffi.lib(), _ffi._ptr
    X, Y, Z, noise = po.case_data(300, 40, 3, 1, 31, False)
    Xnew = np.random.default_rng(3).uniform(-2, 2, (5, 3))
    dmu, dvar = np.empty((5, 3, 1)), np.empty((5, 3))
    e = _ffi.Engine(0)
    # no data and no evaluation yet
    with pytest.raises(_ffi.GpxArgumentError):
        e.predictive_gradients(Xnew)
    with pytest.raises(_ffi.GpxArgumentError):
        e.sparse_predictive_gradients(Xnew)
    assert L.gpx_predictive_gradients(e._h, p(Xnew), 5, p(dmu), p(dvar)) == -2
    assert L.gpx_sparse_predictive_gradients(e._h, p(Xnew), 5, p(dmu), p(dvar)) == -2
    evaluate(e, po.KERNELS["rbf_ard"], X, Y, noise)
    Xs = Xnew
    before = _exact_state(e, Xs)
    assert L.gpx_predictive_gradients(e._h, p(Xnew), 0, p(dmu), p(dvar)) == -2
    assert L.gpx_predictive_gradients(e._h, None, 5, p(dmu), p(dvar)) == -2
    assert L.gpx_predictive_gradients(e._h, p(Xnew), 5, None, p(dvar)) == -2
    assert L.gpx_predictive_gradients(e._h, p(Xnew), 5, p(dmu), None) == -2
    _same(before, _exact_state(e, Xs))
    # a RatQuad part: no device input gradient
    e.exact_eval_multi([("ratquad", False, 0, [0, 1, 2], 1.0, 1.2, {"power": 1.5})], noise)
    before = _exact_state(e, Xs)
    with pytest.raises(_ffi.GpxArgumentError, match="RatQuad / StdPeriodic"):
        e.predictive_gradients(Xnew)
    _same(before, _exact_state(e, Xs))
    # sparse: M < 1 and null pointers
    sparse_evaluate(e, po.KERNELS["rbf_ard"], X, Y, Z, noise)
    sb = _sparse_state(e)
    assert L.gpx_sparse_predictive_gradients(e._h, p(Xnew), 0, p(dmu), p(dvar)) == -2
    assert L.gpx_sparse_predictive_gradients(e._h, p(Xnew), 5, p(dmu), None) == -2
    _same(sb, _sparse_state(e))


def test_mirror_models_take_the_device_route_for_their_kernel():
    """GPRegression / SparseGPRegression.predictive_gradients: one device call for the evaluated kernel, the reference's
    formula on the stand-alone calls for another kernel; both agree with the restatement"""
    X, Y, Z, noise = po.case_data(500, 60, 3, 1, 37, False)
    Xnew = np.random.default_rng(6).uniform(-2, 2, (9, 3))
    e = _ffi.Engine(0)
    k = gpy_b200.RBF(2, variance=0.9, lengthscale=[0.8, 2.2], ARD=True, active_dims=[0, 2])
    m = gpy_b200.GPRegression(X, Y, k, noise_var=noise, engine=e)
    l0 = e.total_launches()
    mj, vj = m.predictive_gradients(Xnew)
    assert e.total_launches() - l0 == 2 + 3 * 2 + _reduction_launches(2, 1)
    kern = CompositeOracle([dict(kind="rbf", term=0, dims=[0, 2], variance=0.9, lengthscale=[0.8, 2.2], ARD=True)])
    wv, wi = po.exact_posterior(kern, X, Y, noise)
    rm, rv = po.jacobians(kern, wv, wi, Xnew, X)
    assert_close(mj, rm)
    assert_close(vj, rv)
    other = gpy_b200.Matern32(3, variance=1.1, lengthscale=1.4)
    om, ov = m.predictive_gradients(Xnew, kern=other)
    rm, rv = po.jacobians(CompositeOracle([dict(kind="matern32", term=0, dims=[0, 1, 2], variance=1.1, lengthscale=1.4)]),
                          wv, wi, Xnew, X)
    assert_close(om, rm)
    assert_close(ov, rv)
    s = gpy_b200.SparseGPRegression(X, Y, mirror_kernel(po.KERNELS["m52_x_rbf"]), Z=Z, engine=e)
    s.likelihood.variance.values[...] = noise
    s.parameters_changed()
    sm, sv = s.predictive_gradients(Xnew)
    kern = CompositeOracle(po.KERNELS["m52_x_rbf"])
    wv, wi = po.sparse_posterior(kern, X, Y, Z, noise)
    rm, rv = po.jacobians(kern, wv, wi, Xnew, Z)
    assert kmm_cond(kern, Z) <= 1e6
    assert_close(sm, rm)
    assert_close(sv, rv)
