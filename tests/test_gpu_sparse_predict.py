"""Sparse prediction on the device (gpx_sparse_predict): the reference's own VarDTC predictions (tests/golden/sparse_predict)
including the exact 1e-15 clip; shapes over 1 to 3 Kmm blocks, test-point counts at the tile edges, P, single and
composite kernels with both noise forms against the NumPy restatement of tests/sparse_predict_cases.py on the device's own
woodbury arrays; the invariants (rows independent of the chunking, one mean for both variance forms, an exactly symmetric
covariance); the benchmark's shape against an extended-precision reference, with the chunk count of the rule in gpx.h; a
bounded footprint at 3e6 test points; a one-rank communicator; rejections; launch accounting; the mirror's model."""
import ctypes
import glob
import os

import numpy as np
import pytest

import gpy_b200
import sparse_composite_oracle as so
import sparse_predict_cases as cases
from gpy_b200 import _ffi
from sparse_composite_oracle import CompositeOracle

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = sorted(glob.glob(os.path.join(HERE, "golden", "sparse_predict", "*.npz")))
MAXNORM = 1e-7          # max-norm error relative to the largest entry (the rule of test_gpu_sparse_composite.py)
MAXNORM_EXP = 1e-6      # Exponential at points on Z: k is first order in r ~ 1e-8 there (test_gpu_routes.py)
STATIONARY = ("rbf", "exponential", "matern32", "matern52")
TILE, RSPLIT, CACHED = 128, 64, 1 << 30


def chunk_rows(M, P, Mn):
    """the chunk rule of include/gpx.h"""
    Mz = -(-M // TILE) * TILE
    Lc = max(TILE, (CACHED // (16 * Mz + 520 * P + 1096)) // TILE * TILE)
    return min(Lc, -(-Mn // TILE) * TILE)


def close(got, want, what, tol=MAXNORM):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    err = np.abs(got - want).max()
    assert err <= tol * max(np.abs(want).max(), 1e-300), (what, err, np.abs(want).max())


def evaluate(e, parts, X, Y, Z, noise):
    e.sparse_set_data(X, Y)
    p = parts[0]
    if len(parts) == 1 and p["kind"] in STATIONARY:
        if np.ndim(noise) > 0:
            return e.sparse_eval_het(p["kind"], p.get("ARD", False), p["variance"], p["lengthscale"], Z, noise)
        return e.sparse_eval(p["kind"], p.get("ARD", False), p["variance"], p["lengthscale"], Z, noise)
    return e.sparse_eval_multi([so.descriptor(q) for q in parts], Z, noise)


def restated(e, parts, Z, Xnew, full_cov=False):
    """the reference's formula on the device's own woodbury_vector and woodbury_inv"""
    return cases.predict(e.sparse_get("woodbury_vector"), e.sparse_get("woodbury_inv"), CompositeOracle(parts), Z, Xnew,
                         full_cov)


# ---- the reference's own predictions ------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[:-4])
def test_device_matches_the_reference_fixtures(path):
    f = np.load(path)
    c = cases.CASES[os.path.basename(path)[:-4]]
    noise = f["noise"]
    noise = float(noise) if noise.ndim == 0 else noise
    tol = MAXNORM_EXP if any(p["kind"] == "exponential" for p in c["parts"]) else MAXNORM
    e = _ffi.Engine(0)
    try:
        evaluate(e, c["parts"], f["X"], f["Y"], f["Z"], noise)
        mu, var = e.sparse_predict(f["Xnew"])
        mu_f, cov = e.sparse_predict(f["Xnew"], full_cov=True)
        if "clip" in path:
            assert np.all(var == cases.CLIP)                      # exactly the reference's clip value
            assert np.abs(cov).max() < 1e-17                      # the full covariance is not clipped
        else:
            close(var, f["var"], "var", tol)
            close(cov, f["cov"], "cov", tol)
        close(mu, f["mu"], "mu", tol)
        close(mu_f, f["mu_full"], "mu (full_cov)", tol)
    finally:
        e.close()


# ---- shapes ------------------------------------------------------------------------------------------------------------
KERNELS = {"single": [dict(kind="matern52", term=0, dims=[0, 1, 2], variance=1.1, lengthscale=[1.2, 0.8, 1.6], ARD=True)],
           "composite": so.KERNELS["m52_x_rbf_plus_exp"]}


@pytest.mark.parametrize("P", [1, 3])
@pytest.mark.parametrize("M", [50, 129, 300])
def test_shapes_against_the_restatement(M, P):
    """nb = 128: Kmm on 1, 2 and 3 blocks; M* at the tile edges; single and composite kernels with scalar and per-point
    noise. Also: the mean is the same bits for both variance forms, the covariance is exactly symmetric and its diagonal
    is the diagonal call's (which is clipped; these variances are far above the clip)."""
    e = _ffi.Engine(0)
    e.set_option("nb", 128)
    try:
        for kname, parts in KERNELS.items():
            tol = MAXNORM_EXP if kname == "composite" else MAXNORM
            for het in (False, True):
                X, Y, Z, noise = so.case_data(400, M, 3, P, 17 * M + P + het, het)
                evaluate(e, parts, X, Y, Z, noise)
                for Mn in (1, 127, 128, 129):
                    Xnew = np.random.default_rng(Mn).uniform(-2.2, 2.2, (Mn, 3))
                    mu, var = e.sparse_predict(Xnew)
                    mu_f, cov = e.sparse_predict(Xnew, full_cov=True)
                    rm, rv = restated(e, parts, Z, Xnew)
                    _, rc = restated(e, parts, Z, Xnew, full_cov=True)
                    what = "%s het=%s M*=%d" % (kname, het, Mn)
                    assert mu.shape == (Mn, P) and var.shape == (Mn, 1) and cov.shape == (Mn, Mn)
                    close(mu, rm, "mu " + what, tol)
                    close(var, rv, "var " + what, tol)
                    close(cov, rc, "cov " + what, tol)
                    np.testing.assert_array_equal(mu_f, mu)
                    np.testing.assert_array_equal(cov, cov.T)
                    assert var.min() > 1e-6
                    close(np.diag(cov)[:, None], var, "diag(cov) " + what, 1e-9)
    finally:
        e.close()


# ---- the benchmark's shape -----------------------------------------------------------------------------------------------
N_B, M_B, D_B = 262144, 4096, 16


@pytest.fixture(scope="module")
def bench_model():
    rng = np.random.default_rng(0)
    X = rng.uniform(-3, 3, (N_B, D_B))
    Y = np.sin(X).sum(1, keepdims=True) / np.sqrt(D_B) + 0.1 * rng.standard_normal((N_B, 1))
    Z = X[rng.permutation(N_B)[:M_B]].copy()
    ls = np.sqrt(D_B) * np.linspace(0.8, 1.25, D_B)
    e = _ffi.Engine(0)
    e.sparse_set_data(X, Y)
    e.sparse_eval("rbf", True, 1.0, ls, Z, 0.05)
    yield e, Z, ls
    e.close()


def _rbf_K(A, B, ls, dtype):
    """the reference's RBF K(A, B) (stationary.py _unscaled_dist on inputs scaled by the lengthscale) in `dtype`"""
    A, B = (np.asarray(A, dtype=dtype) / np.asarray(ls, dtype=dtype)), (np.asarray(B, dtype=dtype) / np.asarray(ls, dtype=dtype))
    r2 = (A * A).sum(1)[:, None] + (B * B).sum(1)[None, :] - 2 * A.dot(B.T)
    return np.exp(-0.5 * np.maximum(r2, 0))


def test_benchmark_shape_chunks_rows_and_accuracy(bench_model):
    """M* = 40000 at M = 4096 is three chunks of the rule (asserted through the launch count); rows are the same bits alone,
    in a block of 129 and inside the multi-chunk call; a sample of rows is within 4x the fp64 host route's error of the
    formula in extended precision on the device's own W and woodbury_vector"""
    e, Z, ls = bench_model
    Mn = 40000
    Lc = chunk_rows(M_B, 1, Mn)
    nchunks = -(-Mn // Lc)
    assert Lc == 15872 and nchunks == 3
    Xnew = np.random.default_rng(5).uniform(-3, 3, (Mn, D_B))
    l0 = e.total_launches()
    mu, var = e.sparse_predict(Xnew)
    assert e.total_launches() - l0 == 6 * nchunks + 5            # the first call after the evaluation forms W
    l0 = e.total_launches()
    mu2, var2 = e.sparse_predict(Xnew)
    assert e.total_launches() - l0 == 6 * nchunks
    np.testing.assert_array_equal(mu2, mu)
    np.testing.assert_array_equal(var2, var)
    for rows in ([0], [Lc - 1], [Lc], [2 * Lc + 7], [Mn - 1]):
        ma, va = e.sparse_predict(Xnew[rows])
        np.testing.assert_array_equal(ma, mu[rows])
        np.testing.assert_array_equal(va, var[rows])
    blk = np.arange(Lc - 64, Lc + 65)                            # 129 rows across the first chunk boundary
    mb, vb = e.sparse_predict(Xnew[blk])
    np.testing.assert_array_equal(mb, mu[blk])
    np.testing.assert_array_equal(vb, var[blk])
    # accuracy on a sample of rows
    wv, W = e.sparse_get("woodbury_vector"), e.sparse_get("woodbury_inv")
    idx = np.random.default_rng(6).choice(Mn, 8, replace=False)
    ld = np.longdouble
    Kl = _rbf_K(Xnew[idx], Z, ls, ld)
    mu_l = Kl.dot(wv.astype(ld))
    var_l = 1.0 - (Kl.dot(W.astype(ld)) * Kl).sum(1)
    Kh = _rbf_K(Xnew[idx], Z, ls, np.float64)
    mu_h = np.dot(Kh, wv)
    var_h = 1.0 - np.sum(np.dot(Kh, W) * Kh, 1)
    for dev, host, ref, what in ((mu[idx, 0], mu_h[:, 0], mu_l[:, 0], "mu"), (var[idx, 0], var_h, var_l, "var")):
        e_dev = float(np.abs(dev - ref).max())
        e_host = float(np.abs(host - ref).max())
        assert e_dev <= 4 * e_host + 1e-15 * float(np.abs(ref).max()), (what, e_dev, e_host)


def test_three_million_points_stay_within_the_pool(bench_model):
    """M* = 3e6 at M = 4096 (unchunked: 2 x 3e6 x 4096 x 8 B = 197 GB of K(X*, Z) and V^T) completes, and afterwards the
    device holds no more than the pool's cached 1 GiB above what it held before the call"""
    import torch
    e, Z, ls = bench_model
    e.sparse_predict(Z[:10])                                     # W formed, pool warmed

    def used():
        torch.cuda.synchronize()
        free, total = torch.cuda.mem_get_info(0)
        return total - free

    u0 = used()
    Mn = 3_000_000
    Xnew = np.random.default_rng(7).uniform(-3, 3, (Mn, D_B))
    mu, var = e.sparse_predict(Xnew)
    assert np.isfinite(mu).all() and np.isfinite(var).all() and var.min() >= cases.CLIP
    assert used() - u0 <= CACHED, (used() - u0)
    ma, va = e.sparse_predict(Xnew[-129:])                        # the last, partial chunk: the same bits in a block
    np.testing.assert_array_equal(ma, mu[-129:])
    np.testing.assert_array_equal(va, var[-129:])


# ---- communicator, rejections, launches ----------------------------------------------------------------------------------
def test_one_rank_communicator_is_bit_identical_to_a_plain_context():
    from test_gpu_sharded_single_rank import attach
    X, Y, Z, noise = so.case_data(500, 140, 3, 2, 31, False)
    parts = KERNELS["single"]
    Xnew = np.random.default_rng(3).uniform(-2.2, 2.2, (300, 3))
    out = []
    for e in (_ffi.Engine(0), attach(_ffi.Engine(0))):
        try:
            evaluate(e, parts, X, Y, Z, noise)
            out.append(e.sparse_predict(Xnew) + e.sparse_predict(Xnew, full_cov=True))
        finally:
            e.close()
    for a, b in zip(*out):
        np.testing.assert_array_equal(a, b)


def _posterior_state(e, Xt, z):
    return [e.sparse_get("woodbury_vector"), e.sparse_get("woodbury_inv"), e.sparse_get("Kmm"), e.sparse_get("Lm"),
            *e.sparse_predictive_gradients(Xt), *e.sparse_posterior_samples(Xt, z), e.stats()]


def test_rejections_leave_the_posterior_untouched():
    X, Y, Z, noise = so.case_data(300, 60, 3, 1, 41, False)
    Xt = np.random.default_rng(4).uniform(-2, 2, (9, 3))
    z = np.random.default_rng(5).standard_normal((2, 9))
    L = _ffi.lib()
    mu, var = np.empty((9, 1)), np.empty(9)
    p = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))   # noqa: E731
    e = _ffi.Engine(0)
    try:
        assert L.gpx_sparse_predict(e._h, p(Xt), 9, 0, p(mu), p(var)) == -2          # no sparse evaluation
        evaluate(e, KERNELS["single"], X, Y, Z, noise)
        before = _posterior_state(e, Xt, z)
        for args in ((None, 9, 0, p(mu), p(var)), (p(Xt), 9, 0, None, p(var)), (p(Xt), 9, 1, p(mu), None),
                     (p(Xt), 0, 0, p(mu), p(var)), (p(Xt), -3, 1, p(mu), p(var))):
            assert L.gpx_sparse_predict(e._h, *args) == -2
        assert L.gpx_sparse_predict(None, p(Xt), 9, 0, p(mu), p(var)) == -2
        e.sparse_predict(Xt)
        e.sparse_predict(Xt, full_cov=True)
        after = _posterior_state(e, Xt, z)
        for a, b in zip(before[:-1], after[:-1]):
            np.testing.assert_array_equal(a, b)
        assert before[-1] == after[-1]
    finally:
        e.close()


def test_launch_accounting_and_one_w_per_evaluation():
    """gpx.h: 6 launches per chunk of the diagonal, 8 for the full covariance, plus the 5 that form W on the first of
    predict / predictive gradients / samples after an evaluation"""
    X, Y, Z, noise = so.case_data(300, 60, 3, 1, 43, False)
    Xt = np.random.default_rng(8).uniform(-2, 2, (20, 3))
    e = _ffi.Engine(0)
    try:
        def launches(fn):
            l0 = e.total_launches()
            fn()
            return e.total_launches() - l0
        evaluate(e, KERNELS["single"], X, Y, Z, noise)
        assert launches(lambda: e.sparse_predict(Xt)) == 6 + 5
        assert launches(lambda: e.sparse_predict(Xt)) == 6
        assert launches(lambda: e.sparse_predict(Xt, full_cov=True)) == 8
        R = 2                                                    # P = 1, 3 stacked dims: one channel group, one final
        assert launches(lambda: e.sparse_predictive_gradients(Xt)) == 3 + R
        evaluate(e, KERNELS["single"], X, Y, Z, noise)
        assert launches(lambda: e.sparse_predictive_gradients(Xt)) == 8 + R
        assert launches(lambda: e.sparse_predict(Xt, full_cov=True)) == 8
    finally:
        e.close()


# ---- the mirror's model --------------------------------------------------------------------------------------------------
def test_mirror_predict_predict_noiseless_and_another_kernel():
    X, Y, Z, _ = so.case_data(400, 40, 3, 2, 51, False)
    k = gpy_b200.Matern52(3, variance=1.1, lengthscale=[1.2, 0.8, 1.6], ARD=True)
    m = gpy_b200.SparseGPRegression(X, Y, kernel=k, Z=Z)
    m.likelihood.variance[:] = 0.08
    m.parameters_changed()
    e = m.inference_method.engine
    Xnew = np.random.default_rng(9).uniform(-2.2, 2.2, (200, 3))
    for full_cov in (False, True):
        l0 = e.total_launches()
        mu, var = m.predict_noiseless(Xnew, full_cov=full_cov)
        assert e.total_launches() - l0 in ((6, 11) if not full_cov else (8, 13))   # one device call
        rm, rv = restated(e, KERNELS["single"], Z, Xnew, full_cov)
        close(mu, rm, "mu")
        close(var, rv, "var")
        mu2, var2 = m.predict(Xnew, full_cov=full_cov)
        np.testing.assert_array_equal(mu2, mu)
        np.testing.assert_array_equal(var2, var + (0.08 * np.eye(200) if full_cov else 0.08))
    other = gpy_b200.RBF(3, variance=0.7, lengthscale=1.3)
    mo, vo = m.predict_noiseless(Xnew, kern=other)               # the host route with the stand-alone kernel calls
    rm, rv = cases.predict(e.sparse_get("woodbury_vector"), e.sparse_get("woodbury_inv"),
                           CompositeOracle([dict(kind="rbf", term=0, dims=[0, 1, 2], variance=0.7, lengthscale=1.3)]),
                           Z, Xnew)
    close(mo, rm, "mu (kern=)")
    close(vo, rv, "var (kern=)")
