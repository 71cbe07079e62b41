"""Every route of the sparse (VarDTC) evaluation against the CPU oracle and, for ill-conditioned Kmm, against an
extended-precision reference; the stand-alone kernel calls at the edges of their instantiations.

`gpx_sparse_eval` / `gpx_sparse_eval_het` factor Kmm + 1e-8 I (jitchol's ladder, at most 5 rungs) and B = I + A on two
child contexts with the blocked sweep of the exact path. The outer block of an M x M factorisation is the option `nb` of
the engine (the children follow the parent), else by size: one block up to Mpad = 512, 256 below 2048, 512 up to 8192.
After a sparse evaluation `Engine.stats()` reports both factorisations, and each case checks them:

    tries            attempts on Kmm (1 = no jitter ladder)
    update_launches  (tries + 1) u   (u = 2 nblk - 3 trailing updates per sweep of nblk >= 2 blocks, 0 for one:
                                      every attempt on Kmm and the one on B)

A change of a block threshold therefore fails here instead of quietly moving a case to another route. The counts come
from the sweeps themselves (`gemm_update_kernel` launches, as for the exact path); the kernel-level accounting of the
sparse evaluation, children included, is checked against torch.profiler by tests/test_gpu_launch_accounting.py.

| route / edge                                            | case                                                      |
|---------------------------------------------------------|-----------------------------------------------------------|
| one Kmm block: M = 1                                    | rbf ARD N 1000 M 1 D 2                                    |
| one block, N below one tile, D = 1, M = one tile, M > N | matern32 iso N 127 M 128 D 1                              |
| one block, M > N, P = 2                                 | matern52 ARD N 200 M 300 D 3                              |
| one block, D = 8 (register width), N tail tile, P = 3   | exponential ARD N 2049 M 129 D 8                          |
| NB 256 by size, 3 blocks, D = 16                        | matern52 ARD N 3000 M 700 D 16 (scalar + per-point noise) |
| nb 128, 5 blocks                                        | rbf ARD N 4000 M 600 D 4 (both noise models)              |
| nb 128, 3 blocks, D = MAX_D, P = MAX_P                  | matern32 ARD N 1500 M 300 D 64 P 8 (both)                 |
| NB 512 by size with a 128 tail, Z = exact rows of X     | rbf ARD N 12001 M 2049 D 16: the benchmark's route (both) |
| nb 128, Z = exact rows of X, not smooth at r = 0        | exponential iso N 1500 M 300 D 3 (both)                   |
| jitter ladder on Kmm (tries_Kmm = 2), nb 128, 3 blocks  | test_kmm_jitter_ladder                                    |
| context reuse                                           | M 129 -> 300 -> 129, P 1 -> 3, D 3 -> 5, sparse -> exact  |
|                                                         | -> sparse                                                 |
| the benchmark's shape (N 262107, M 4096: 8 x 512)       | test_benchmark_shape_metamorphic (device against itself)  |
| ill-conditioned Kmm (cond 1e4 .. 1e10), nb 128, 3 blocks | test_ill_conditioned_kmm_against_extended_precision       |

The NB 512 case keeps N at 12001 so that the oracle stays short: 10 s per evaluation on one CPU core (measured with
numpy's OpenBLAS on the build machine).

The extended-precision VarDTC reference (np.longdouble, 64-bit significand, hand-written Cholesky and triangular solves)
and its CPU self-tests run without a GPU; tools/sparse_dz_extended_precision.py evaluates the golden fixtures with it.
"""
import functools
import os

import numpy as np
import pytest

import gpy_b200
from oracle import gpy_oracle as o

LD = np.longdouble
LML_RTOL = 1e-8
GRAD_RTOL = 1e-6
MAXNORM_FLOOR = 1e-7     # dZ and dL_dR: absolute floor relative to the largest entry


def _ffi():
    from gpy_b200 import _ffi as f
    return f


def assert_sparse_route(st, nblk, tries_kmm=1):
    """the stats of the last sparse evaluation: Kmm factored in tries_kmm attempts, each sweep over nblk outer blocks"""
    u = 0 if nblk == 1 else 2 * nblk - 3
    assert st["tries"] == tries_kmm, ("tries", st["tries"], tries_kmm)
    assert st["update_launches"] == (tries_kmm + 1) * u, ("update_launches", st["update_launches"], nblk, tries_kmm)


# --------------------------------------------------------------------------------------------------------------------
# problems and comparisons
# --------------------------------------------------------------------------------------------------------------------
def problem(N, M, D, P, seed, exact_z=False):
    """X uniform in [-3, 3]^D; Z rows of X (exactly, or moved by 0.01 noise), or for M > N all of X plus uniform points"""
    rng = np.random.default_rng(seed)
    X = rng.uniform(-3, 3, (N, D))
    Y = np.stack([np.sin(X).sum(1) / np.sqrt(D) + 0.1 * (q + 1) * np.cos((q + 1) * X[:, 0]) + 0.1 * rng.standard_normal(N)
                  for q in range(P)], 1)
    if M <= N:
        Z = X[rng.permutation(N)[:M]].copy()
    else:
        Z = np.concatenate([X, rng.uniform(-3, 3, (M - N, D))])[rng.permutation(M)]
    if not exact_z:
        Z = Z + 0.01 * rng.standard_normal((M, D))
    return rng, X, Y, Z


def theta(kind, D, ARD, rng, scale=1.0):
    ls = scale * (np.sqrt(D) * rng.uniform(0.7, 1.3, D) if ARD else float(np.sqrt(D) * 0.9))
    return 1.3, ls


def maxrel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.max(np.abs(a - b)) / max(float(np.max(np.abs(b))), 1e-300))


def check_scalar(out, ref, tag):
    lml, g, dZ = out
    lml0, g0, Zg0, _ = ref
    assert abs(lml - lml0) <= LML_RTOL * max(1.0, abs(lml0)), (tag, lml, lml0)
    np.testing.assert_allclose(g, g0, rtol=GRAD_RTOL, atol=1e-8, err_msg=tag)
    np.testing.assert_allclose(dZ, Zg0, rtol=GRAD_RTOL, atol=MAXNORM_FLOOR * np.abs(Zg0).max(), err_msg=tag)


def check_het(out, ref, tag):
    lml, g, dZ, dR = out
    lml0, g0, Zg0, _ = ref
    nk = g.size
    assert abs(lml - lml0) <= LML_RTOL * max(1.0, abs(lml0)), (tag, lml, lml0)
    np.testing.assert_allclose(g, g0[:nk], rtol=GRAD_RTOL, atol=1e-8, err_msg=tag)
    np.testing.assert_allclose(dZ, Zg0, rtol=GRAD_RTOL, atol=MAXNORM_FLOOR * np.abs(Zg0).max(), err_msg=tag)
    dR0 = g0[nk:].reshape(dR.shape)
    np.testing.assert_allclose(dR, dR0, rtol=GRAD_RTOL, atol=MAXNORM_FLOOR * np.abs(dR0).max(), err_msg=tag)


def check_posterior(e, res, var, tag):
    """woodbury_vector, woodbury_inv, Kmm and Lm through gpx_sparse_get"""
    np.testing.assert_allclose(e.sparse_get("woodbury_vector"), res["woodbury_vector"], rtol=1e-6, atol=1e-7, err_msg=tag)
    np.testing.assert_allclose(e.sparse_get("woodbury_inv"), res["woodbury_inv"], rtol=1e-4,
                               atol=1e-6 * np.abs(res["woodbury_inv"]).max(), err_msg=tag)
    Kmm0 = res["Kmm"]
    np.testing.assert_allclose(e.sparse_get("Kmm"), Kmm0, rtol=1e-12, atol=1e-12 * var, err_msg=tag)
    Lm = np.tril(e.sparse_get("Lm"))
    np.testing.assert_allclose(Lm @ Lm.T, Kmm0, rtol=1e-9, atol=1e-10 * var, err_msg=tag)


# (what, kind, ARD, N, M, D, P, option nb, Kmm blocks, Z exact rows of X, lengthscale scale). The oracle is the yardstick
# here, so every case keeps cond(Kmm + 1e-8 I) <= 1.1e5 (the lengthscale scale does that where M is dense in the inputs):
# at cond 5e9 the oracle's own dL/dZ is 3e-6 off the true value, see test_ill_conditioned_kmm_against_extended_precision.
ROUTE_CASES = [
    ("M1", "rbf", True, 1000, 1, 2, 1, 0, 1, False, 1.0),
    ("N-below-tile-D1", "matern32", False, 127, 128, 1, 1, 0, 1, False, 0.02),
    ("M-above-N", "matern52", True, 200, 300, 3, 2, 0, 1, False, 1.0),
    ("D8-tail", "exponential", True, 2049, 129, 8, 3, 0, 1, False, 1.0),
    ("NB256-3blk", "matern52", True, 3000, 700, 16, 1, 0, 3, False, 1.0),
    ("nb128-5blk", "rbf", True, 4000, 600, 4, 1, 128, 5, False, 0.5),
    ("maxD-maxP", "matern32", True, 1500, 300, 64, 8, 128, 3, False, 1.0),
    ("NB512-bench-route", "rbf", True, 12001, 2049, 16, 1, 0, 5, True, 1.0),
    ("exact-Z-exponential", "exponential", False, 1500, 300, 3, 1, 128, 3, True, 1.0),
]
PREDICT_CASES = ("M-above-N", "exact-Z-exponential")


@pytest.mark.gpu
@pytest.mark.parametrize("what,kind,ARD,N,M,D,P,nb,nblk,exact_z,ls_scale", ROUTE_CASES, ids=[c[0] for c in ROUTE_CASES])
def test_sparse_route_matrix(what, kind, ARD, N, M, D, P, nb, nblk, exact_z, ls_scale):
    rng, X, Y, Z = problem(N, M, D, P, seed=N + M + D, exact_z=exact_z)
    var, ls = theta(kind, D, ARD, rng, ls_scale)
    e = _ffi().Engine(0)
    try:
        if nb:
            e.set_option("nb", nb)
        e.sparse_set_data(X, Y)
        out = e.sparse_eval(kind, ARD, var, ls, Z, 0.05)
        assert_sparse_route(e.stats(), nblk)
        ref = o.sparse_eval(X, Y, Z, kind, ARD, var, ls, 0.05)
        check_scalar(out, ref, what)
        check_posterior(e, ref[3], var, what)
        if nblk > 1:   # the per-point noise entry point on the same multi-block route
            nv = rng.uniform(0.01, 0.3, N)
            out_h = e.sparse_eval_het(kind, ARD, var, ls, Z, nv)
            assert_sparse_route(e.stats(), nblk)
            ref_h = o.sparse_eval(X, Y, Z, kind, ARD, var, ls, nv)
            check_het(out_h, ref_h, what + " het")
            check_posterior(e, ref_h[3], var, what + " het")
    finally:
        e.close()
    if what in PREDICT_CASES:
        cls = {"rbf": gpy_b200.RBF, "exponential": gpy_b200.Exponential, "matern32": gpy_b200.Matern32,
               "matern52": gpy_b200.Matern52}[kind]
        k = cls(D, variance=var, lengthscale=ls, ARD=ARD)
        m = gpy_b200.SparseGPRegression(X, Y, kernel=k, Z=Z)
        m.likelihood.variance.values[...] = 0.05
        m.parameters_changed()
        res = ref[3]
        Xn = np.concatenate([X[:7], Z[:7], rng.uniform(-3, 3, (7, D))])
        mu, v = m.predict(Xn, include_likelihood=False)
        ko = o.StationaryOracle(kind, D, var, ls, ARD)
        mu0, v0 = o.sparse_raw_predict(ko, Z, res["woodbury_vector"], res["woodbury_inv"], Xn)
        np.testing.assert_allclose(mu, mu0, rtol=1e-6, atol=1e-8)
        np.testing.assert_allclose(v, v0, rtol=1e-5, atol=1e-8)


# --------------------------------------------------------------------------------------------------------------------
# jitter ladder on Kmm, context reuse
# --------------------------------------------------------------------------------------------------------------------
def ladder_problem(N=900, M=300, D=2, seed=31):
    """Kmm = 1e10 K(Z, Z) with 50 rows of Z repeated: the 1e-8 jitter is below the rounding of the 1e10 diagonal, so the
    first factorisation meets a zero or negative pivot (on LAPACK and on the device alike), and mean(diag) 1e-6 I (the
    first rung) makes it well-posed (cond 6.7e6 after the rung).
    Y and the noise are scaled with the variance, so that B = I + A is as well conditioned as in the unscaled problem."""
    rng = np.random.default_rng(seed)
    X = rng.uniform(-3, 3, (N, D))
    Y = 1e5 * (np.sin(X).sum(1, keepdims=True) + 0.1 * rng.standard_normal((N, 1)))
    Z = rng.uniform(-3, 3, (M, D))
    Z[rng.choice(M, 50, replace=False)] = Z[rng.choice(M, 50, replace=False)]
    return X, Y, Z, 1e10, np.array([0.2, 0.25]), 0.05e10


@pytest.mark.gpu
def test_kmm_jitter_ladder():
    X, Y, Z, var, ls, noise = ladder_problem()
    Kmm = o.StationaryOracle("rbf", 2, var, ls, True).K(Z) + 1e-8 * np.eye(Z.shape[0])
    _, jit0 = o.jitchol(Kmm)
    assert jit0 > 0                                            # LAPACK needed the ladder as well
    e = _ffi().Engine(0)
    try:
        e.set_option("nb", 128)
        e.sparse_set_data(X, Y)
        out = e.sparse_eval("rbf", True, var, ls, Z, noise)
        assert_sparse_route(e.stats(), 3, tries_kmm=2)
        ref = o.sparse_eval(X, Y, Z, "rbf", True, var, ls, noise)
        # the gradients scale with 1 / variance here: relative tolerances only
        assert abs(out[0] - ref[0]) <= LML_RTOL * abs(ref[0]), (out[0], ref[0])
        np.testing.assert_allclose(out[1], ref[1], rtol=GRAD_RTOL, atol=0)
        np.testing.assert_allclose(out[2], ref[2], rtol=GRAD_RTOL, atol=MAXNORM_FLOOR * np.abs(ref[2]).max())
        Lm = np.tril(e.sparse_get("Lm"))                        # the factor of Kmm + the first rung
        np.testing.assert_allclose(Lm @ Lm.T, Kmm + jit0 * np.eye(Z.shape[0]), rtol=1e-9, atol=1e-10 * var)
        # a well-posed evaluation on the same engine: one attempt, nothing of the ladder left
        rng, X2, Y2, Z2 = problem(1100, 300, 2, 1, seed=5)
        e.sparse_set_data(X2, Y2)
        out = e.sparse_eval("matern52", True, 1.1, np.array([1.3, 1.7]), Z2, 0.04)
        assert_sparse_route(e.stats(), 3)
        ref = o.sparse_eval(X2, Y2, Z2, "matern52", True, 1.1, np.array([1.3, 1.7]), 0.04)
        check_scalar(out, ref, "after ladder")
        check_posterior(e, ref[3], 1.1, "after ladder")
    finally:
        e.close()


def fresh_sparse(X, Y, Z, kind, ARD, var, ls, noise, nb=0):
    e = _ffi().Engine(0)
    try:
        if nb:
            e.set_option("nb", nb)
        e.sparse_set_data(X, Y)
        return e.sparse_eval(kind, ARD, var, ls, Z, noise)
    finally:
        e.close()


def same_bits(a, b):
    return a[0] == b[0] and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


@pytest.mark.gpu
def test_sparse_reuse_across_shapes():
    """One engine through M 129 -> 300 -> 129 (Mpad 256 -> 384 -> 256: the M x M buffers are freed and re-allocated while
    the child contexts survive), P 1 -> 3 and D 3 -> 5 (the whole sparse state is re-allocated). Every step equals a fresh
    engine bit for bit and the oracle at the usual tolerances."""
    rng = np.random.default_rng(12)
    X5 = rng.uniform(-3, 3, (1000, 5))
    Y3 = np.stack([np.sin(X5).sum(1) + 0.1 * q * X5[:, 1] + 0.1 * rng.standard_normal(1000) for q in range(3)], 1)
    Zall = X5[rng.permutation(1000)[:300]] + 0.01 * rng.standard_normal((300, 5))
    steps = [(3, 1, 129), (3, 1, 300), (3, 1, 129), (3, 3, 129), (5, 3, 129), (5, 3, 300)]
    e = _ffi().Engine(0)
    try:
        for i, (D, P, M) in enumerate(steps):
            X, Y, Z = X5[:, :D].copy(), Y3[:, :P].copy(), Zall[:M, :D].copy()
            ls = 0.5 * np.sqrt(D) * np.linspace(0.8, 1.2, D)    # cond(Kmm) <= 2.6e4
            kind = ("matern32", "rbf")[i % 2]
            e.sparse_set_data(X, Y)
            out = e.sparse_eval(kind, True, 1.2, ls, Z, 0.05)
            assert same_bits(out, fresh_sparse(X, Y, Z, kind, True, 1.2, ls, 0.05)), (D, P, M)
            ref = o.sparse_eval(X, Y, Z, kind, True, 1.2, ls, 0.05)
            check_scalar(out, ref, "D%d P%d M%d" % (D, P, M))
            check_posterior(e, ref[3], 1.2, "D%d P%d M%d" % (D, P, M))
    finally:
        e.close()


@pytest.mark.gpu
def test_sparse_exact_sparse_interleaved():
    """A sparse evaluation, an exact one on the same engine (other data), and the first sparse evaluation again: bit for
    bit the same as the first time."""
    rng, X, Y, Z = problem(1500, 300, 3, 2, seed=44)
    ls = np.array([1.2, 1.5, 1.9])
    e = _ffi().Engine(0)
    try:
        e.set_option("nb", 128)
        e.sparse_set_data(X, Y)
        first = e.sparse_eval("matern52", True, 1.1, ls, Z, 0.05)
        ref = o.sparse_eval(X, Y, Z, "matern52", True, 1.1, ls, 0.05)
        check_scalar(first, ref, "first")
        Xe, Ye = o.synthetic(700, 3, seed=3)
        e.set_data(Xe, Ye)
        lml, g, _ = e.exact_eval("rbf", True, 1.3, ls, 0.05)
        lml0, g0, _ = o.eval_lml_grad(Xe, Ye, "rbf", True, 1.3, ls, 0.05)
        assert abs(lml - lml0) <= 1e-8
        np.testing.assert_allclose(g, g0, rtol=GRAD_RTOL, atol=1e-9)
        again = e.sparse_eval("matern52", True, 1.1, ls, Z, 0.05)
        assert_sparse_route(e.stats(), 3)
        assert same_bits(again, first)
        check_posterior(e, ref[3], 1.1, "again")
    finally:
        e.close()


# --------------------------------------------------------------------------------------------------------------------
# the benchmark's shape: the device against itself
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_benchmark_shape_metamorphic():
    """RBF ARD, N = 262144 - 37 (a row tail), M = 4096 (8 Kmm blocks of 512), D = 16, Z rows of X as SparseGPRegression
    picks them; about 27 GB of device memory. Permuting the data rows moves other points into the tail tile and across
    the reduction chunks: the bound and the gradients stay; permuting Z permutes dL/dZ and keeps the bound."""
    N, M, D = 262144 - 37, 4096, 16
    rng = np.random.default_rng(0)
    X = rng.uniform(-3, 3, (N, D))
    Y = np.sin(X).sum(1, keepdims=True) / np.sqrt(D) + 0.1 * rng.standard_normal((N, 1))
    Z = X[rng.permutation(N)[:M]].copy()
    ls = np.sqrt(D) * rng.uniform(0.95, 1.05, D)
    e = _ffi().Engine(0)
    try:
        e.sparse_set_data(X, Y)
        base = e.sparse_eval("rbf", True, 1.0, ls, Z, 0.05)
        assert_sparse_route(e.stats(), 8)
        assert np.all(np.isfinite(base[1])) and np.all(np.isfinite(base[2]))
        pr = rng.permutation(N)
        e.sparse_set_data(X[pr], Y[pr])
        rows = e.sparse_eval("rbf", True, 1.0, ls, Z, 0.05)
        assert_sparse_route(e.stats(), 8)
        pz = rng.permutation(M)
        zp = e.sparse_eval("rbf", True, 1.0, ls, Z[pz], 0.05)
    finally:
        e.close()
    print("\nbenchmark shape: bound %.10e; rows permuted: bound %.1e grad %.1e dZ %.1e; Z permuted: bound %.1e dZ %.1e" % (
        base[0], abs(rows[0] - base[0]) / abs(base[0]), float(np.max(np.abs(rows[1] - base[1]) / np.abs(base[1]))),
        maxrel(rows[2], base[2]), abs(zp[0] - base[0]) / abs(base[0]), maxrel(zp[2], base[2][pz])))
    assert abs(rows[0] - base[0]) <= 1e-10 * abs(base[0])
    np.testing.assert_allclose(rows[1], base[1], rtol=1e-10, atol=0)
    # dL/dZ goes through B^-1 (cond(B) ~ N / noise) formed from the reordered sums of A: 4.9e-10 (rows permuted) and
    # 5.4e-10 (Z permuted) of max|dL/dZ| measured on an H100 at 400 W
    assert maxrel(rows[2], base[2]) <= 2e-9
    assert abs(zp[0] - base[0]) <= 1e-10 * abs(base[0])
    np.testing.assert_allclose(zp[1], base[1], rtol=1e-10, atol=0)
    assert maxrel(zp[2], base[2][pz]) <= 2e-9


# --------------------------------------------------------------------------------------------------------------------
# extended-precision VarDTC reference
# --------------------------------------------------------------------------------------------------------------------
def ld_chol(A):
    """lower Cholesky factor, column by column, in the dtype of A (no fp64 LAPACK involved)"""
    n = A.shape[0]
    L = np.zeros_like(A)
    for j in range(n):
        s = A[j, j] - np.dot(L[j, :j], L[j, :j])
        if not s > 0:
            raise np.linalg.LinAlgError("extended-precision Cholesky: pivot %d is %r" % (j, s))
        L[j, j] = np.sqrt(s)
        if j + 1 < n:
            L[j + 1:, j] = (A[j + 1:, j] - np.dot(L[j + 1:, :j], L[j, :j])) / L[j, j]
    return L


def ld_solve_lower(L, B, trans=False):
    """L X = B (trans=False) or L^T X = B (trans=True), forward / backward substitution"""
    n = L.shape[0]
    X = np.array(B, dtype=L.dtype, copy=True)
    if not trans:
        for i in range(n):
            X[i] = (X[i] - np.dot(L[i, :i], X[:i])) / L[i, i]
    else:
        for i in range(n - 1, -1, -1):
            X[i] = (X[i] - np.dot(L[i + 1:, i], X[i + 1:])) / L[i, i]
    return X


def ld_backsub_both_sides(L, X, transpose="left"):
    """GPy/util/linalg.py:381-390: L^-T X L^-1 (transpose='left') or L^-1 X L^-T"""
    if transpose == "left":
        tmp = ld_solve_lower(L, X, trans=True)
        return ld_solve_lower(L, tmp.T, trans=True).T
    tmp = ld_solve_lower(L, X)
    return ld_solve_lower(L, tmp.T).T


def ld_dist(X, X2, ls, ARD):
    """scaled distance by direct differences (no cancellation-prone expansion): the reference VALUE, not its path"""
    if ARD:
        X, X2 = X / ls, X2 / ls
    d = X[:, None, :] - X2[None, :, :]
    r = np.sqrt((d * d).sum(-1))
    return r if ARD else r / ls


def ld_K_of_r(kind, var, r):
    s3, s5 = np.sqrt(LD(3)), np.sqrt(LD(5))
    return {"rbf": lambda: var * np.exp(-r * r / 2), "exponential": lambda: var * np.exp(-r),
            "matern32": lambda: var * (1 + s3 * r) * np.exp(-s3 * r),
            "matern52": lambda: var * (1 + s5 * r + LD(5) / 3 * r * r) * np.exp(-s5 * r)}[kind]()


def ld_dK_dr(kind, var, r):
    s3, s5 = np.sqrt(LD(3)), np.sqrt(LD(5))
    return {"rbf": lambda: -r * var * np.exp(-r * r / 2), "exponential": lambda: -var * np.exp(-r),
            "matern32": lambda: -3 * var * r * np.exp(-s3 * r),
            "matern52": lambda: var * (LD(10) / 3 * r - 5 * r - 5 * s5 / 3 * r * r) * np.exp(-s5 * r)}[kind]()


def _inv(r):
    return np.where(r != 0, 1 / np.where(r != 0, r, 1), 0)


def ld_gradients_X(kind, var, ls, ARD, dL_dK, X, X2=None):
    """stationary.py:245-252"""
    same = X2 is None
    X2 = X if same else X2
    r = ld_dist(X, X2, ls, ARD)
    tmp = _inv(r) * ld_dK_dr(kind, var, r) * dL_dK
    if same:
        tmp = tmp + tmp.T
    g = np.stack([(tmp * (X[:, q][:, None] - X2[:, q][None, :])).sum(1) for q in range(X.shape[1])], 1)
    return g / ls ** 2


def ld_kernel_grads(kind, var, ls, ARD, dL_dK, X, X2):
    """update_gradients_full (stationary.py:193-213): d/d variance, d/d lengthscale (1 or D entries)"""
    r = ld_dist(X, X2, ls, ARD)
    dv = (ld_K_of_r(kind, var, r) * dL_dK).sum() / var
    dL_dr = ld_dK_dr(kind, var, r) * dL_dK
    if not ARD:
        return dv, np.array([-(dL_dr * r).sum() / ls])
    tmp = dL_dr * _inv(r)
    return dv, np.array([-(tmp * (X[:, q][:, None] - X2[:, q][None, :]) ** 2).sum() / ls[q] ** 3
                         for q in range(X.shape[1])])


def vardtc_extended(X, Y, Z, kind, ARD, variance, lengthscale, noise):
    """var_dtc.py:66-276 + sparse_gp.py:108-119 (scalar noise, Kmm + 1e-8 I without a ladder) in extended precision:
    bound, grad [variance, lengthscale.., noise variance], dL/dZ, woodbury_vector and cond(Kmm + 1e-8 I)"""
    X, Y, Z = X.astype(LD), Y.astype(LD), Z.astype(LD)
    var, noise = LD(variance), LD(noise)
    ls = np.asarray(lengthscale).astype(LD) if ARD else LD(float(lengthscale))
    N, P = Y.shape
    M = Z.shape[0]
    beta = 1 / max(noise, LD(1e-8))
    eye = np.eye(M, dtype=LD)
    Kmm = ld_K_of_r(kind, var, ld_dist(Z, Z, ls, ARD)) + LD(1e-8) * eye
    Lm = ld_chol(Kmm)
    psi1 = ld_K_of_r(kind, var, ld_dist(X, Z, ls, ARD))
    Lmi_psi1 = ld_solve_lower(Lm, psi1.T)
    A = beta * (Lmi_psi1 @ Lmi_psi1.T)
    B = eye + A
    LB = ld_chol(B)
    LBi_Lmi_psi1 = ld_solve_lower(LB, Lmi_psi1)
    v = LBi_Lmi_psi1 @ (beta * Y)
    wv = ld_solve_lower(Lm, ld_solve_lower(LB, v, trans=True), trans=True)
    data_fit = (v * v).sum()
    DBi = ld_backsub_both_sides(LB, P * eye + v @ v.T)
    dL_dKmm = ld_backsub_both_sides(Lm, -DBi / 2 - B * P / 2 + P * eye)
    dL_dpsi2 = beta * ld_backsub_both_sides(Lm, P * eye - DBi) / 2
    dL_dpsi1 = (beta * Y) @ wv.T + 2 * psi1 @ dL_dpsi2
    trYYT, psi0 = (Y * Y).sum(), N * var
    log2pi = np.log(2 * np.arccos(LD(-1)))
    trA = np.trace(A)
    lml = (-N * P / LD(2) * (log2pi - np.log(beta)) - beta * trYYT / 2 - P / LD(2) * (beta * psi0 - trA)
           - P * np.log(np.diag(LB)).sum() + data_fit / 2)
    dL_dR = -N * P * beta / 2 + trYYT * beta ** 2 / 2 + P / LD(2) * (psi0 * beta ** 2 - trA * beta) \
        + beta * ((A * DBi).sum() / 2 - data_fit)
    dv1, dl1 = ld_kernel_grads(kind, var, ls, ARD, dL_dpsi1, X, Z)
    dv2, dl2 = ld_kernel_grads(kind, var, ls, ARD, dL_dKmm, Z, Z)
    grad = np.concatenate([[-P * beta * N / 2 + dv1 + dv2], dl1 + dl2, [dL_dR]])
    Zg = ld_gradients_X(kind, var, ls, ARD, dL_dKmm, Z) + ld_gradients_X(kind, var, ls, ARD, dL_dpsi1.T, Z, X)
    cond = float(np.linalg.cond(Kmm.astype(np.float64)))
    return dict(lml=lml, grad=grad, dZ=Zg, wv=wv, cond=cond)


def ext_errors(ref, lml, g, dZ, wv):
    """distance of one result from the extended-precision reference: the bound relative, the gradient relative per entry,
    dL/dZ and the woodbury vector relative to their largest entry"""
    def diff(a, b):
        return np.abs((np.asarray(a, dtype=LD).reshape(b.shape) - b).astype(np.float64))

    def big(b):
        return float(np.max(np.abs(b.astype(np.float64))))
    return dict(lml=float(diff(lml, ref["lml"])) / max(1.0, abs(float(ref["lml"]))),
                grad=float(np.max(diff(g, ref["grad"]) / np.abs(ref["grad"].astype(np.float64)))),
                dZ=float(np.max(diff(dZ, ref["dZ"]))) / big(ref["dZ"]),
                wv=float(np.max(diff(wv, ref["wv"]))) / big(ref["wv"]))


# the tolerances of the oracle comparisons above, as distances from the true value
NORTH_STAR = dict(lml=LML_RTOL, grad=GRAD_RTOL, dZ=MAXNORM_FLOOR, wv=1e-6)
EXT_LS = 0.7 * np.array([1.0, 1.1, 1.2])


def clustered_problem(spread, N=1000, M=300, seed=6):
    """RBF ARD in three dimensions, Z drawn in [-3 spread, 3 spread]^3: spread 1 -> cond(Kmm + 1e-8 I) ~ 1e4, 0.6 -> 1e7,
    0.02 -> the jitter floor (M variance / 1e-8 ~ 3e10). spread 0: Z are rows of X moved by 0.01 (as the other tests pick
    them) with lengthscales 1.4 .. 2.1: cond 5.4e9, the oracle's dL/dZ 2.8e-6 of its largest entry off the true value."""
    rng = np.random.default_rng(seed)
    X = rng.uniform(-3, 3, (N, 3))
    Y = np.sin(X).sum(1, keepdims=True) / np.sqrt(3) + 0.1 * rng.standard_normal((N, 1))
    if spread == 0:
        Z = X[rng.permutation(N)[:M]] + 0.01 * rng.standard_normal((M, 3))
        return X, Y, Z, 1.2, np.sqrt(3) * np.linspace(0.8, 1.2, 3), 0.05
    Z = spread * rng.uniform(-3, 3, (M, 3))
    return X, Y, Z, 1.0, EXT_LS, 0.05


@functools.lru_cache(maxsize=None)
def ext_case(spread, N=1000, M=300):
    X, Y, Z, var, ls, noise = clustered_problem(spread, N, M)
    return vardtc_extended(X, Y, Z, "rbf", True, var, ls, noise)


def oracle_ext_errors(spread, N=1000, M=300):
    X, Y, Z, var, ls, noise = clustered_problem(spread, N, M)
    lml, g, dZ, res = o.sparse_eval(X, Y, Z, "rbf", True, var, ls, noise)
    return ext_errors(ext_case(spread, N, M), lml, g, dZ, res["woodbury_vector"])


def test_extended_vardtc_agrees_with_the_oracle_when_well_conditioned():
    X, Y, Z, _, ls, _ = clustered_problem(1.0, N=300, M=40)
    ref = vardtc_extended(X, Y, Z, "rbf", True, 1.2, ls, 0.1)
    assert ref["cond"] < 1e4
    lml, g, dZ, res = o.sparse_eval(X, Y, Z, "rbf", True, 1.2, ls, 0.1)
    err = ext_errors(ref, lml, g, dZ, res["woodbury_vector"])
    assert max(err.values()) <= 1e-11, err
    # every kind through the generic kernel formulas (dL/dZ and the kernel gradients), iso as well
    for kind, ARD, lsk in (("matern52", False, 1.4), ("exponential", True, ls), ("matern32", False, 1.2)):
        ref = vardtc_extended(X, Y, Z, kind, ARD, 0.9, lsk, 0.1)
        lml, g, dZ, res = o.sparse_eval(X, Y, Z, kind, ARD, 0.9, lsk, 0.1)
        err = ext_errors(ref, lml, g, dZ, res["woodbury_vector"])
        assert max(err.values()) <= 1e-10, (kind, err)


def test_extended_vardtc_shows_the_oracle_error_growth():
    """fp64 loses digits with cond(Kmm): from cond 1e4 to the jitter floor the oracle's distance from the
    extended-precision result grows by orders of magnitude in the gradient, dL/dZ and the woodbury vector."""
    lo, hi = ext_case(1.0, 500, 200), ext_case(0.02, 500, 200)
    assert lo["cond"] < 1e5 and hi["cond"] > 1e10, (lo["cond"], hi["cond"])
    elo, ehi = oracle_ext_errors(1.0, 500, 200), oracle_ext_errors(0.02, 500, 200)
    for k in ("grad", "dZ", "wv"):
        assert ehi[k] > 100 * elo[k], (k, elo, ehi)


@pytest.mark.gpu
@pytest.mark.parametrize("spread", [1.0, 0.6, 0.02, 0.0])
def test_ill_conditioned_kmm_against_extended_precision(spread):
    """device error <= max(north-star tolerance, 4 x the fp64 oracle's own error), output by output, Kmm on 3 blocks"""
    X, Y, Z, var, ls, noise = clustered_problem(spread)
    ref = ext_case(spread)
    ora = oracle_ext_errors(spread)
    e = _ffi().Engine(0)
    try:
        e.set_option("nb", 128)
        e.sparse_set_data(X, Y)
        lml, g, dZ = e.sparse_eval("rbf", True, var, ls, Z, noise)
        assert_sparse_route(e.stats(), 3)
        dev = ext_errors(ref, lml, g, dZ, e.sparse_get("woodbury_vector"))
    finally:
        e.close()
    print("\nsparse extended-precision check spread=%g cond(Kmm)=%.2e\n  device %s\n  oracle %s" % (
        spread, ref["cond"], dev, ora))
    for k in NORTH_STAR:
        assert dev[k] <= max(NORTH_STAR[k], 4 * ora[k]), (k, dev, ora, ref["cond"])


# --------------------------------------------------------------------------------------------------------------------
# stand-alone kernel calls at the edges of their instantiations
# --------------------------------------------------------------------------------------------------------------------
KERNEL_SHAPES = [(1, 1), (127, 5), (128, 128), (129, 31), (300, 257)]


@pytest.mark.gpu
@pytest.mark.parametrize("D", [1, 8, 9, 16, 17, 32, 33])
@pytest.mark.parametrize("ARD", [False, True])
@pytest.mark.parametrize("kind", o.KINDS)
def test_kernel_calls_at_instantiation_edges(kind, ARD, D):
    """gpx_kern_K, gpx_kern_grad_full and gpx_kern_grad_X (register widths 8, 16, 32, 64; gradients_X chunks of 32
    columns) with X2 absent and given, at the tolerances of tests/test_gpu_parity.py::test_kernel_plugin_calls and
    ::test_gradients_X."""
    f = _ffi()
    rng = np.random.default_rng(100 * D + 2 * o.KINDS.index(kind) + ARD)
    for n, m in KERNEL_SHAPES:
        X, X2 = rng.standard_normal((n, D)), rng.standard_normal((m, D))
        ls = np.sqrt(D) * rng.uniform(0.8, 1.6, D) if ARD else float(np.sqrt(D) * rng.uniform(0.8, 1.6))
        ko = o.StationaryOracle(kind, D, 0.7, ls, ARD)
        for x2 in (None, X2):
            tag = "%s ARD=%s D=%d n=%d m=%s" % (kind, ARD, D, n, None if x2 is None else m)
            cols = n if x2 is None else m
            K = f.kern_K(kind, ARD, 0.7, ls, X, x2)
            K0 = ko.K(X, x2)
            assert maxrel(K, K0) < 1e-13, tag
            dL = rng.standard_normal((n, cols))
            dv, dl = f.kern_grad_full(kind, ARD, 0.7, ls, X, dL, x2)
            v0, l0 = ko.update_gradients_full(dL, X, x2)
            np.testing.assert_allclose(dv, v0, rtol=1e-10, atol=1e-13, err_msg=tag)
            np.testing.assert_allclose(dl, l0, rtol=1e-9, atol=1e-12, err_msg=tag)
            gx = f.kern_grad_X(kind, ARD, 0.7, ls, X, dL, x2)
            np.testing.assert_allclose(gx, ko.gradients_X(dL, X, x2), rtol=1e-9, atol=1e-11, err_msg=tag)


@pytest.mark.gpu
@pytest.mark.parametrize("ARD", [False, True])
def test_kernel_calls_with_exact_copies_off_the_diagonal(ARD):
    """X2 holds exact copies of rows of X: r = 0 off the diagonal of a non-symmetric call, where the Exponential kernel is
    not smooth. Both sides form r from |x|^2 + |x'|^2 - 2 x.x' (stationary.py:130-148) and get ~1e-8 instead of 0 there,
    which the Exponential kernel passes on to K at first order: those entries are held to 1e-7 variance (the other
    entries as above). The gradients at those pairs are multiplied by the exact difference 0."""
    f = _ffi()
    rng = np.random.default_rng(3 + ARD)
    n, m, D = 129, 31, 3
    X = rng.standard_normal((n, D))
    X2 = rng.standard_normal((m, D))
    src = rng.choice(n, 10, replace=False)
    X2[:10] = X[src]
    copy = np.zeros((n, m), dtype=bool)
    copy[src, np.arange(10)] = True
    ls = rng.uniform(0.8, 1.6, D) if ARD else 1.2
    ko = o.StationaryOracle("exponential", D, 0.7, ls, ARD)
    K, K0 = f.kern_K("exponential", ARD, 0.7, ls, X, X2), ko.K(X, X2)
    assert np.all(np.isfinite(K))
    assert maxrel(np.where(copy, 0, K), np.where(copy, 0, K0)) < 1e-13
    assert np.all(np.abs(K - 0.7)[copy] <= 1e-7 * 0.7), K[copy]
    dL = rng.standard_normal((n, m))
    dv, dl = f.kern_grad_full("exponential", ARD, 0.7, ls, X, dL, X2)
    v0, l0 = ko.update_gradients_full(dL, X, X2)
    slack = 1e-7 * np.abs(dL[copy]).sum()           # K at the copies, and r dK/dr there (iso lengthscale)
    np.testing.assert_allclose(dv, v0, rtol=1e-10, atol=slack)
    np.testing.assert_allclose(dl, l0, rtol=1e-9, atol=slack)
    gx = f.kern_grad_X("exponential", ARD, 0.7, ls, X, dL, X2)
    assert np.all(np.isfinite(gx))
    np.testing.assert_allclose(gx, ko.gradients_X(dL, X, X2), rtol=1e-9, atol=1e-11)


# --------------------------------------------------------------------------------------------------------------------
# the outer block is read once per workspace
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_gpx_nb_narrowed_after_allocation_keeps_the_allocated_block(monkeypatch):
    """GPX_NB set to a narrower block after gpx_set_data: the workspace was sized for NB 256 (Npad 1152: 4 x 256 + 128,
    7 trailing updates) and the evaluation keeps that block rather than switching to 128 (9 blocks, 15 updates). A new
    allocation picks the variable up."""
    X, Y = o.synthetic(1025, 2, seed=4)
    e = _ffi().Engine(0)
    try:
        monkeypatch.delenv("GPX_NB", raising=False)
        e.set_option("ozaki", 0)
        e.set_data(X, Y)
        monkeypatch.setenv("GPX_NB", "128")
        lml, g, _ = e.exact_eval("matern32", False, 1.1, 1.4, 0.05)
        assert e.stats()["update_launches"] == 7
        lml0, g0, _ = o.eval_lml_grad(X, Y, "matern32", False, 1.1, 1.4, 0.05)
        assert abs(lml - lml0) <= 1e-8
        np.testing.assert_allclose(g, g0, rtol=GRAD_RTOL, atol=1e-9)
        e.set_data(X[:800], Y[:800])                        # Npad 896: a new workspace, now with NB 128
        e.exact_eval("matern32", False, 1.1, 1.4, 0.05)
        assert e.stats()["update_launches"] == 2 * 7 - 3
    finally:
        e.close()
