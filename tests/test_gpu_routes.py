"""Every route of the exact evaluation, on both tensor paths, against the CPU oracle (and, for ill-conditioned problems, an
extended-precision reference).

`gpx_exact_eval` picks its kernels from the padded size, the outer block NB (option `nb`, else by size: one block up to
512, 256 below 2048, 512 up to 8192, 1024 above), option `ozaki`, the noise model and the kernel type. Each case of the
route matrix states the route and the number of outer blocks it expects and checks both through `Engine.stats()`, so a
change of a threshold fails here instead of quietly moving a case to another route:

    update_int8_ops > 0      iff the sweep ran on the int8 tensor cores (`run_sweep_chain`)
    lauum_flops > 0          iff K^-1 came from `gemm_lauum_kernel` (fused, or plain for composite kernels)
    update_launches          2 nblk - 3 on the DMMA sweep (U1 for every block but the last, U2 where a block follows
                             block k+1), 2 nblk - 1 on the int8 sweep (its U2 also carries the K^-1 tiles)

| route                                                        | cases                                                  |
|--------------------------------------------------------------|--------------------------------------------------------|
| dmma-fine: DMMA sweep, nt <= 8, fine LAUUM + `grad_kinv`       | 1024 rbf; het see below; ladder/reuse none             |
| dmma-fused: DMMA sweep, nt > 8, `gemm_lauum_kernel` epilogue   | 1025, 2049 (NB 512, 128 tail), 8192 (NB 512),          |
|                                                              | 8193 (NB 1024, 128 tail), 1300 P=8 D=64, het 1025,     |
|                                                              | ladder 1200, reuse 1700/1650, repeat, extended 1100    |
| int8-dmmapanel: `run_sweep_chain`, panel GEMM on DMMA (<4096) | 700 (3 x 256), 1700 nb=128, 1700 nb=384, 1300 P=8      |
|                                                              | D=64, het 1700, ladder 1200, reuse, repeat, extended   |
| int8-ozpanel: `run_sweep_chain`, panel GEMM on int8 (>=4096)  | 4097 (NB 512, tail), 4097 nb=1024, het 4097            |
| multi-dmma: composite kernel, plain LAUUM + `grad_kinv_multi`  | 700, 2049                                              |
| multi-int8: composite kernel, int8 sweep + `grad_kinv_multi`   | 2049                                                   |
| jitter ladder, first failing minor in block k > 0           | test_ladder_fails_in_a_later_block (both paths)         |
| context reuse                                                | N 1700 -> 1650 (same Npad), ozaki 1 -> 0 -> 1, P 1 -> 3, |
|                                                              | int8 single kernel -> int8 composite kernel            |
| `gpx_pdinv` multi-block                                      | 2049, 4097: noisy kernel, graded D A D, non-PD tail    |

The fine-LAUUM route with one block (N <= 512) is covered by tests/test_gpu_parity.py.

The extended-precision reference (np.longdouble, 64-bit significand) has CPU self-tests that run without a GPU.
"""
import functools

import numpy as np
import pytest
from scipy import linalg as sla

from oracle import gpy_oracle as o

LML_ATOL = 1e-8
GRAD_RTOL = 1e-6
LD = np.longdouble
EPS = np.finfo(np.float64).eps


def _ffi():
    from gpy_b200 import _ffi as f
    return f


def rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.max(np.abs(a - b)) / max(float(np.max(np.abs(b))), 1e-300))


def theta(D, ARD, seed):
    rng = np.random.default_rng(seed)
    ls = np.sqrt(D) * rng.uniform(0.7, 1.4, D) if ARD else float(np.sqrt(D) * rng.uniform(0.7, 1.4))
    return float(rng.uniform(0.5, 2.0)), ls, float(rng.uniform(0.01, 0.1))


def data(N, D, P, seed):
    rng = np.random.default_rng(seed)
    X = rng.uniform(-3, 3, (N, D))
    Y = np.stack([np.sin(X).sum(1) / np.sqrt(D) + 0.1 * (q + 1) * np.cos(X[:, 0] * (q + 1)) + 0.1 * rng.standard_normal(N)
                  for q in range(P)], 1)
    return X, Y


def probe_points(X, seed, m=200):
    """m points: half of them training points, the rest new points in the same box."""
    rng = np.random.default_rng(seed)
    D = X.shape[1]
    return np.concatenate([X[rng.choice(X.shape[0], m // 2, replace=False)], rng.uniform(-3, 3, (m - m // 2, D))])


def engine(oz, nb):
    e = _ffi().Engine(0)
    e.set_option("ozaki", oz)
    if nb:
        e.set_option("nb", nb)
    return e


INT8_ROUTES = ("int8-dmmapanel", "int8-ozpanel", "multi-int8")
FUSED_ROUTES = ("dmma-fused", "multi-dmma")


def assert_route(st, route, nblk, tries=1):
    int8 = route in INT8_ROUTES
    assert (st["update_int8_ops"] > 0) == int8, (route, st)
    assert (st["lauum_flops"] > 0) == (route in FUSED_ROUTES), (route, st)
    per_try = 2 * nblk - (1 if int8 else 3)
    assert st["update_launches"] == tries * per_try, (route, nblk, st)
    assert st["tries"] == tries, st


# --------------------------------------------------------------------------------------------------------------------
# A. the route matrix
# --------------------------------------------------------------------------------------------------------------------
# (route, kind, ARD, N, D, P, option ozaki, option nb, outer blocks)
ROUTE_CASES = [
    ("dmma-fine", "rbf", True, 1024, 3, 1, 0, 0, 4),                 # 4 x 256, nt = 8
    ("dmma-fused", "matern32", False, 1025, 2, 1, 0, 0, 5),          # nt = 9: 4 x 256 + 128
    ("dmma-fused", "matern52", True, 2049, 5, 2, 0, 0, 5),           # NB 512: 4 x 512 + 128
    ("dmma-fused", "exponential", False, 8192, 4, 1, 0, 0, 16),      # NB 512 up to Npad 8192
    ("dmma-fused", "rbf", True, 8193, 8, 1, 0, 0, 9),                # Npad 8320: NB 1024, 8 x 1024 + 128
    ("int8-dmmapanel", "matern52", False, 700, 3, 1, 1, 0, 3),       # 3 x 256, panel GEMM on DMMA
    ("int8-ozpanel", "rbf", False, 4097, 6, 1, 1, 0, 9),             # panel GEMM on int8, 8 x 512 + 128
    ("int8-ozpanel", "matern32", True, 4097, 4, 1, 1, 1024, 5),      # 4 x 1024 + 128
    ("int8-dmmapanel", "exponential", True, 1700, 3, 1, 1, 128, 14),
    ("int8-dmmapanel", "rbf", False, 1700, 2, 3, 1, 384, 5),         # 4 x 384 + 256
    ("dmma-fused", "matern32", True, 1300, 64, 8, 0, 0, 6),          # widest: P = MAX_P, D = 64
    ("int8-dmmapanel", "matern52", True, 1300, 64, 8, 1, 0, 6),
]


def _ids(c):
    return "%s-%s%s-N%d-D%d-P%d-oz%d-nb%d" % (c[0], c[1], "ard" if c[2] else "iso", c[3], c[4], c[5], c[6], c[7])


def mean_atol(kind, alpha):
    """The predictive mean at a training point: r(x, x) comes from |x|^2 + |x'|^2 - 2 x.x' (stationary.py:130-148) and is
    ~1e-8 instead of 0 after the cancellation; the Exponential kernel, not smooth at r = 0, passes that on to k(x, x) at
    first order, so each side's mean there is off by up to ~1e-8 |alpha_i| variance / lengthscale (measured: 5e-8)."""
    return 1e-10 if kind != "exponential" else 1e-7 * float(np.abs(alpha).max())


def var_atol(kind):
    """the same cancellation in k(x, x) and k(X, x) of the predictive variance (measured: up to 2e-7 at N = 8192)"""
    return 1e-10 if kind != "exponential" else 1e-6


def check_gets(e, res, int8, N):
    """L, L^-1, K^-1 and dL_dK element by element (the int8 path keeps 7 digits in U and K^-1)."""
    if N > 2200:
        return
    tol = 1e-8 if int8 else 1e-9
    assert rel(e.get("L"), res["L"]) < 1e-10
    assert rel(e.get("Linv"), o.dtrtri(res["L"])) < tol
    assert rel(e.get("Kinv"), res["Wi"]) < tol
    assert rel(e.get("dL_dK"), res["dL_dK"]) < tol


@pytest.mark.gpu
@pytest.mark.parametrize("route,kind,ARD,N,D,P,oz,nb,nblk", ROUTE_CASES, ids=[_ids(c) for c in ROUTE_CASES])
def test_route_matrix(route, kind, ARD, N, D, P, oz, nb, nblk):
    X, Y = data(N, D, P, seed=N + D)
    var, ls, noise = theta(D, ARD, N + P)
    lml0, g0, res = o.eval_lml_grad(X, Y, kind, ARD, var, ls, noise)
    e = engine(oz, nb)
    e.set_data(X, Y)
    lml, g, jit = e.exact_eval(kind, ARD, var, ls, noise)
    assert_route(e.stats(), route, nblk)
    assert jit == 0.0
    assert abs(lml - lml0) <= LML_ATOL, (lml, lml0)
    np.testing.assert_allclose(g, g0, rtol=GRAD_RTOL, atol=1e-9)
    assert rel(e.get("alpha"), res["alpha"]) < 1e-9
    check_gets(e, res, oz == 1, N)
    ko = o.StationaryOracle(kind, D, var, ls, ARD)
    Xn = probe_points(X, N)
    mu, v = e.predict(Xn)
    mu0, v0 = o.raw_predict(ko, X, res["L"], res["alpha"], Xn)
    np.testing.assert_allclose(mu, mu0, rtol=1e-8, atol=mean_atol(kind, res["alpha"]))
    np.testing.assert_allclose(v, v0, rtol=1e-7, atol=var_atol(kind))
    mu, cov = e.predict(Xn[95:107], full_cov=True)
    _, cov0 = o.raw_predict(ko, X, res["L"], res["alpha"], Xn[95:107], full_cov=True)
    np.testing.assert_allclose(cov, cov0, rtol=1e-7, atol=var_atol(kind))
    e.close()


# (route, kind, ARD, N, D, option ozaki, outer blocks): P = 2 outputs, one noise variance per point
HET_CASES = [
    ("dmma-fused", "rbf", True, 1025, 3, 0, 5),              # diag(dL_dK) from the gemm_lauum_kernel epilogue
    ("int8-dmmapanel", "matern52", False, 1700, 2, 1, 7),    # from grad_kinv_kernel after run_sweep_chain
    ("int8-ozpanel", "exponential", True, 4097, 2, 1, 9),
]


@pytest.mark.gpu
@pytest.mark.parametrize("route,kind,ARD,N,D,oz,nblk", HET_CASES, ids=[_ids(c[:5] + (2, c[5], 0)) for c in HET_CASES])
def test_route_matrix_per_point_noise(route, kind, ARD, N, D, oz, nblk):
    X, Y = data(N, D, 2, seed=N)
    var, ls, _ = theta(D, ARD, N)
    nv = np.random.default_rng(N).uniform(0.01, 0.3, N)
    lml0, g0, res = o.eval_lml_grad(X, Y, kind, ARD, var, ls, nv)
    e = engine(oz, 0)
    e.set_data(X, Y)
    lml, g, dn, _ = e.exact_eval_het(kind, ARD, var, ls, nv)
    assert_route(e.stats(), route, nblk)
    nl = D if ARD else 1
    assert abs(lml - lml0) <= LML_ATOL
    np.testing.assert_allclose(g[:1 + nl], g0[:1 + nl], rtol=GRAD_RTOL, atol=1e-9)
    np.testing.assert_allclose(dn, g0[1 + nl:], rtol=GRAD_RTOL, atol=1e-9)
    assert abs(g[-1] - dn.sum()) <= 1e-9 * max(1.0, np.abs(dn).sum())
    assert rel(e.get("alpha"), res["alpha"]) < 1e-9
    check_gets(e, res, oz == 1, N)
    Xn = probe_points(X, N)
    mu, v = e.predict(Xn)
    mu0, v0 = o.raw_predict(o.StationaryOracle(kind, D, var, ls, ARD), X, res["L"], res["alpha"], Xn)
    np.testing.assert_allclose(mu, mu0, rtol=1e-8, atol=mean_atol(kind, res["alpha"]))
    np.testing.assert_allclose(v, v0, rtol=1e-7, atol=var_atol(kind))
    e.close()


# (route, N, option ozaki, outer blocks)
COMPOSITE_CASES = [("multi-dmma", 700, 0, 3), ("multi-dmma", 2049, 0, 5), ("multi-int8", 2049, 1, 5)]


@pytest.mark.gpu
@pytest.mark.parametrize("route,N,oz,nblk", COMPOSITE_CASES, ids=["%s-N%d" % (c[0], c[1]) for c in COMPOSITE_CASES])
def test_route_matrix_composite(route, N, oz, nblk):
    from test_gpu_parity import _composite_case
    D = 5
    X, Y = o.synthetic(N, D, seed=N)
    _, parts = _composite_case(D)
    tup = [(p["kind"], p.get("ARD", False), p["term"], p["dims"], p["variance"], p.get("lengthscale")) for p in parts]
    e = engine(oz, 0)
    e.set_data(X, Y)
    lml, g, _ = e.exact_eval_multi(tup, 0.04)
    assert_route(e.stats(), route, nblk)
    lml0, g0, res = o.composite_eval_lml_grad(X, Y, parts, 0.04)
    assert abs(lml - lml0) <= LML_ATOL
    np.testing.assert_allclose(g, g0, rtol=GRAD_RTOL, atol=1e-9)
    assert rel(e.get("alpha"), res["alpha"]) < 1e-9
    check_gets(e, res, oz == 1, N)
    Xn = probe_points(X, N)
    Kx = o.composite_K(res["kparts"], X, Xn)
    tmp = o.dtrtrs(res["L"], Kx, lower=1)[0]
    mu, v = e.predict(Xn)
    np.testing.assert_allclose(mu, Kx.T @ res["alpha"], rtol=1e-8, atol=1e-10)
    np.testing.assert_allclose(v[:, 0], o.composite_Kdiag(res["kparts"], Xn) - np.square(tmp).sum(0), rtol=1e-7, atol=1e-10)
    mu, cov = e.predict(Xn[95:107], full_cov=True)
    t = tmp[:, 95:107]
    np.testing.assert_allclose(cov, o.composite_K(res["kparts"], Xn[95:107]) - t.T @ t, rtol=1e-7, atol=1e-10)
    e.close()


# --------------------------------------------------------------------------------------------------------------------
# B. jitter ladder and context state
# --------------------------------------------------------------------------------------------------------------------
def later_block_singular(N=1200, D=2, seed=4):
    """Distinct inputs except the last 50 rows, which repeat the first 50: with zero noise the first non-positive pivot
    is row 1151, inside the last outer block (rows 1024..1199 of 5 blocks of 256)."""
    X, _ = o.synthetic(N, D, seed)
    X[-50:] = X[:50]
    Y = np.sin(X[:, :1]) + 0.3 * X[:, 1:]
    return X, Y


@pytest.mark.gpu
@pytest.mark.parametrize("oz,route", [(0, "dmma-fused"), (1, "int8-dmmapanel")])
def test_ladder_fails_in_a_later_block(oz, route):
    X, Y = later_block_singular()
    N = X.shape[0]
    e = engine(oz, 0)
    e.set_data(X, Y)
    lml, g, jit = e.exact_eval("exponential", False, 1.0, 1.3, 0.0, jitter=0.0)
    assert_route(e.stats(), route, 5, tries=2)      # one failed factorisation, then the first rung of the ladder
    Ky = o.StationaryOracle("exponential", 2, 1.0, 1.3, False).K(X)
    with pytest.raises(np.linalg.LinAlgError):
        np.linalg.cholesky(Ky)
    L, jit0 = o.jitchol(Ky)
    assert jit0 > 0 and np.isclose(jit, jit0, rtol=1e-12), (jit, jit0)
    alpha = o.dpotrs(L, Y)[0]
    lml0 = 0.5 * (-Y.size * o.LOG_2_PI - 2 * np.sum(np.log(np.diag(L))) - np.sum(alpha * Y))
    # cond(Ky + jitter) ~ 1e9 here: the device's LML is less accurate than LAPACK's at that conditioning (see
    # test_ill_conditioned_against_extended_precision; measured 6.2e-5 relative on both paths, the ladder test of
    # tests/test_gpu_parity.py with N = 200 holds 1e-6)
    assert abs(lml - lml0) <= 2e-4 * abs(lml0)
    with pytest.raises(np.linalg.LinAlgError):
        e.exact_eval("exponential", False, 1.0, 1.3, 0.0, jitter=0.0, max_tries=0)
    assert e.stats()["tries"] == 1
    # the same context, a well-posed theta: nothing of the failed factorisations may leak into the result
    var, ls, noise = 1.2, np.array([1.1, 1.6]), 0.05
    lml0, g0, res = o.eval_lml_grad(X, Y, "matern32", True, var, ls, noise)
    lml, g, jit = e.exact_eval("matern32", True, var, ls, noise)
    assert_route(e.stats(), route, 5)
    assert jit == 0.0 and abs(lml - lml0) <= LML_ATOL
    np.testing.assert_allclose(g, g0, rtol=GRAD_RTOL, atol=1e-9)
    check_gets(e, res, oz == 1, N)
    assert rel(e.get("alpha"), res["alpha"]) < 1e-9
    e.close()


def check_eval(e, X, Y, kind, ARD, var, ls, noise, int8):
    lml0, g0, res = o.eval_lml_grad(X, Y, kind, ARD, var, ls, noise)
    lml, g, _ = e.exact_eval(kind, ARD, var, ls, noise)
    assert abs(lml - lml0) <= LML_ATOL, (X.shape, Y.shape, lml, lml0)
    np.testing.assert_allclose(g, g0, rtol=GRAD_RTOL, atol=1e-9)
    assert rel(e.get("alpha"), res["alpha"]) < 1e-9
    check_gets(e, res, int8, X.shape[0])
    return e.stats()


@pytest.mark.gpu
@pytest.mark.parametrize("oz", [0, 1])
def test_reuse_with_fewer_points_same_padding(oz):
    """N = 1700 then 1650 (both Npad = 1792) then 1700 again on one context: the rows beyond the new N must not reach
    any result, and K^-1 of the earlier size must never be returned."""
    e = engine(oz, 0)
    X, Y = data(1700, 3, 1, seed=17)
    for n, th in ((1700, 0), (1650, 1), (1700, 2)):
        e.set_data(X[:n], Y[:n])
        var, ls, noise = theta(3, True, th)
        st = check_eval(e, X[:n], Y[:n], "rbf", True, var, ls, noise, oz == 1)
        assert_route(st, "int8-dmmapanel" if oz else "dmma-fused", 7)
    e.close()


@pytest.mark.gpu
def test_reuse_across_tensor_paths():
    """ozaki 1 -> 0 -> 1 on the same data and context, a different theta each time."""
    e = _ffi().Engine(0)
    X, Y = data(1700, 4, 2, seed=23)
    e.set_data(X, Y)
    for i, oz in enumerate((1, 0, 1)):
        e.set_option("ozaki", oz)
        var, ls, noise = theta(4, False, 30 + i)
        st = check_eval(e, X, Y, "matern52", False, var, ls, noise, oz == 1)
        assert_route(st, "int8-dmmapanel" if oz else "dmma-fused", 7)
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("oz", [0, 1])
def test_reuse_with_more_outputs(oz):
    """P = 1 then P = 3 on one context (the output count changes the buffers and the forward substitution widths)."""
    e = engine(oz, 0)
    X, Y = data(1300, 2, 3, seed=5)
    for P, th in ((1, 3), (3, 4), (1, 5)):
        e.set_data(X, Y[:, :P])
        var, ls, noise = theta(2, True, th)
        st = check_eval(e, X, Y[:, :P], "exponential", True, var, ls, noise, oz == 1)
        assert_route(st, "int8-dmmapanel" if oz else "dmma-fused", 6)
    e.close()


@pytest.mark.gpu
def test_composite_after_single_kernel_on_the_int8_path():
    """A single-kernel evaluation on the int8 path, then a composite one on the same engine and data: the composite result
    must be bit for bit that of a fresh engine. The single-kernel build of Ky announces its first block row by an event, and
    the first diagonal block of the int8 sweep starts after it; the composite build is one launch, and the sweep after it
    must wait for all of it. An engine that kept the earlier evaluation's event would start D(0) while block row 0 is still
    being written; this test may still pass there by timing luck. What rules the race out is that the event is handed from
    the build to the sweep of the same evaluation."""
    from test_gpu_parity import _composite_case
    N, D = 2049, 5
    X, Y = o.synthetic(N, D, seed=N)
    _, parts = _composite_case(D)
    tup = [(p["kind"], p.get("ARD", False), p["term"], p["dims"], p["variance"], p.get("lengthscale")) for p in parts]
    fresh = engine(1, 0)
    fresh.set_data(X, Y)
    lml_f, g_f, _ = fresh.exact_eval_multi(tup, 0.04)
    assert_route(fresh.stats(), "multi-int8", 5)
    kinv_f = fresh.get("Kinv")
    fresh.close()
    e = engine(1, 0)
    e.set_data(X, Y)
    var, ls, noise = theta(D, True, 3)
    e.exact_eval("rbf", True, var, ls, noise)
    assert_route(e.stats(), "int8-dmmapanel", 5)
    lml, g, _ = e.exact_eval_multi(tup, 0.04)
    assert_route(e.stats(), "multi-int8", 5)
    assert lml == lml_f and np.array_equal(g, g_f)
    assert np.array_equal(e.get("Kinv"), kinv_f)
    e.close()
    lml0, g0, res = o.composite_eval_lml_grad(X, Y, parts, 0.04)
    assert abs(lml - lml0) <= LML_ATOL
    np.testing.assert_allclose(g, g0, rtol=GRAD_RTOL, atol=1e-9)
    assert rel(kinv_f, res["Wi"]) < 1e-8


@pytest.mark.gpu
@pytest.mark.parametrize("oz", [0, 1])
def test_same_theta_twice_is_bit_identical(oz):
    """Fixed-order reductions: the same evaluation twice gives the same bits (LML, gradient, per-point noise gradient)."""
    X, Y = data(1700, 3, 2, seed=8)
    nv = np.random.default_rng(8).uniform(0.01, 0.2, 1700)
    e = engine(oz, 0)
    e.set_data(X, Y)
    out = [e.exact_eval_het("matern32", True, 1.1, np.array([1.2, 1.9, 2.4]), nv) for _ in range(2)]
    assert out[0][0] == out[1][0]
    assert np.array_equal(out[0][1], out[1][1]) and np.array_equal(out[0][2], out[1][2])
    out = [e.exact_eval("rbf", False, 0.9, 1.7, 0.03) for _ in range(2)]
    assert out[0][0] == out[1][0] and np.array_equal(out[0][1], out[1][1])
    e.close()


# --------------------------------------------------------------------------------------------------------------------
# C. ill-conditioned problems against an extended-precision reference
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


def ld_tri_inv(L):
    """L^-1 of a lower triangular L, row by row"""
    n = L.shape[0]
    X = np.zeros_like(L)
    for i in range(n):
        X[i, :i] = -np.dot(L[i, :i], X[:i, :i]) / L[i, i]
        X[i, i] = 1 / L[i, i]
    return X


def ld_rbf(X, X2, var, ls):
    d = (X[:, None, :] - X2[None, :, :]) / ls
    return var * np.exp(-(d * d).sum(-1) / 2)


def ld_reference(X, Y, var, ls, noise, Xn):
    """RBF ARD exact GP in extended precision: Ky = K + (noise + 1e-8) I (exact_gaussian_inference.py:55-56), LML, gradient
    [variance, lengthscale.., noise], alpha and the noise-free predictive variance at Xn."""
    X, Y, Xn, ls = X.astype(LD), Y.astype(LD), Xn.astype(LD), np.asarray(ls).astype(LD)
    var = LD(var)
    N, P = Y.shape
    K = ld_rbf(X, X, var, ls)
    Ky = K + (LD(noise) + LD(1e-8)) * np.eye(N, dtype=LD)
    L = ld_chol(Ky)
    Li = ld_tri_inv(L)
    Kinv = Li.T @ Li
    alpha = Li.T @ (Li @ Y)
    lml = -LD(0.5) * N * P * np.log(2 * np.arccos(LD(-1))) - P * np.log(np.diag(L)).sum() - (alpha * Y).sum() / 2
    dL = (alpha @ alpha.T - P * Kinv) / 2
    KdL = K * dL
    g = [KdL.sum() / var]
    for q in range(X.shape[1]):
        dq = X[:, q:q + 1] - X[:, q:q + 1].T
        g.append((KdL * dq * dq).sum() / ls[q] ** 3)
    g.append(np.trace(dL))
    v = Li @ ld_rbf(X, Xn, var, ls)
    pvar = var - (v * v).sum(0)
    return dict(lml=lml, grad=np.array(g, dtype=LD), alpha=alpha, pvar=pvar)


def ill_problem(N=1100, seed=2):
    """smooth RBF in two dimensions, lengthscale about 1.5 sqrt(D): cond(Ky) ~ N variance / noise"""
    X, Y = o.synthetic(N, 2, seed)
    Xn = probe_points(X, seed, 60)
    return X, Y, 1.0, np.array([2.0, 2.3]), Xn


@functools.lru_cache(maxsize=None)
def ld_case(noise, N=1100):
    X, Y, var, ls, Xn = ill_problem(N)
    return ld_reference(X, Y, var, ls, noise, Xn)


def errors(ref, lml, g, alpha, pvar):
    """distance of one result from the extended-precision reference: LML absolute, gradient relative per entry, alpha
    relative in the max norm, predictive variance absolute"""
    def diff(a, b):
        return np.abs((np.asarray(a, dtype=LD).reshape(b.shape) - b).astype(np.float64))
    return dict(lml=float(diff(lml, ref["lml"])),
                grad=float(np.max(diff(g, ref["grad"]) / np.abs(ref["grad"].astype(np.float64)))),
                alpha=float(np.max(diff(alpha, ref["alpha"])) / np.max(np.abs(ref["alpha"].astype(np.float64)))),
                pvar=float(np.max(diff(pvar, ref["pvar"]))))


def oracle_errors(noise, N=1100):
    X, Y, var, ls, Xn = ill_problem(N)
    lml, g, res = o.eval_lml_grad(X, Y, "rbf", True, var, ls, noise)
    _, pv = o.raw_predict(o.StationaryOracle("rbf", 2, var, ls, True), X, res["L"], res["alpha"], Xn)
    return errors(ld_case(noise, N), lml, g, res["alpha"], pv)


# the tolerances of the oracle comparisons above, as distances from the true value
NORTH_STAR = dict(lml=LML_ATOL, grad=GRAD_RTOL, alpha=1e-9, pvar=1e-10)


def test_extended_reference_agrees_with_the_oracle_when_well_conditioned():
    X, Y = o.synthetic(300, 2, 1)
    Xn = probe_points(X, 1, 40)
    ls = np.array([0.9, 1.3])
    ref = ld_reference(X, Y, 1.1, ls, 0.1, Xn)
    lml, g, res = o.eval_lml_grad(X, Y, "rbf", True, 1.1, ls, 0.1)
    _, pv = o.raw_predict(o.StationaryOracle("rbf", 2, 1.1, ls, True), X, res["L"], res["alpha"], Xn)
    err = errors(ref, lml, g, res["alpha"], pv)
    assert err["lml"] <= 1e-12 * abs(lml), err
    assert err["grad"] <= 1e-11 and err["alpha"] <= 1e-12 and err["pvar"] <= 1e-13, err


def test_extended_reference_shows_the_oracle_error_growth():
    """fp64 loses about log10 cond(Ky) digits: from noise 1e-2 to 1e-6 the oracle's distance from the extended-precision
    result grows by orders of magnitude in the LML, the gradient and alpha (alpha's stays within eps cond(Ky)). The
    predictive variance, a sum of squares of L^-1 k(X, x*), does not grow."""
    lo, hi = oracle_errors(1e-2), oracle_errors(1e-6)
    X, Y, var, ls, _ = ill_problem()
    cond = np.linalg.cond(o.StationaryOracle("rbf", 2, var, ls, True).K(X) + (1e-6 + 1e-8) * np.eye(X.shape[0]))
    assert cond > 1e8
    for k in ("lml", "grad", "alpha"):
        assert hi[k] > 100 * lo[k], (k, lo, hi)
    assert hi["alpha"] < EPS * cond, (hi, cond)
    assert max(lo["pvar"], hi["pvar"]) < 1e-14, (lo, hi)


ILL_CONFIGS = [(0, 0, "dmma-fused", 5), (1, 0, "int8-dmmapanel", 5), (1, 128, "int8-dmmapanel", 9)]


@pytest.mark.gpu
@pytest.mark.parametrize("noise", [1e-2, 1e-4, 1e-6])
@pytest.mark.parametrize("oz,nb,route,nblk", ILL_CONFIGS, ids=["oz%d-nb%d" % c[:2] for c in ILL_CONFIGS])
def test_ill_conditioned_against_extended_precision(oz, nb, route, nblk, noise):
    """device error <= max(north-star tolerance, 4 x the fp64 oracle's own error), output by output; on the int8 path
    also the claim of DESIGN.md section 5.1: gradient within 1e-6 wherever cond(Ky) <= 3e7."""
    X, Y, var, ls, Xn = ill_problem()
    ref = ld_case(noise)
    ora = oracle_errors(noise)
    e = engine(oz, nb)
    e.set_data(X, Y)
    lml, g, jit = e.exact_eval("rbf", True, var, ls, noise)
    assert jit == 0.0
    assert_route(e.stats(), route, nblk)
    _, pv = e.predict(Xn)
    dev = errors(ref, lml, g, e.get("alpha"), pv)
    e.close()
    Ky = o.StationaryOracle("rbf", 2, var, ls, True).K(X) + (noise + 1e-8) * np.eye(X.shape[0])
    cond = float(np.linalg.cond(Ky))
    print("\nextended-precision check oz=%d nb=%d noise=%g cond(Ky)=%.2e\n  device %s\n  oracle %s" % (
        oz, nb, noise, cond, dev, ora))
    for k in NORTH_STAR:
        # LML and alpha above cond(Ky) ~ 1e8 are the exception: the device forms alpha = U (U^T y) and the quadratic form
        # from the inverted factor, less accurate than LAPACK's triangular solves (measured at cond 4.6e8 on an H100 at
        # 400 W: LML off by 0.028 on the DMMA path and 0.022 / 0.0055 on the int8 path with NB 256 / 128, against
        # LAPACK's 7.9e-4; alpha 1.1e-7 / 9.7e-8 / 9.2e-8 against 1.2e-8)
        factor = {"lml": 64, "alpha": 16}.get(k, 4) if cond > 1e8 else 4
        # the int8 path computes the predictive variance from U with 7 digits: 1.0e-10 measured at noise 1e-6 (about 1e-4
        # of the variance at a training point), 9e-13 at noise 1e-2
        floor = 4e-10 if (k == "pvar" and oz) else NORTH_STAR[k]
        assert dev[k] <= max(floor, factor * ora[k]), (k, dev, ora, cond)
    if oz and cond <= 3e7:
        assert dev["grad"] <= GRAD_RTOL, (dev, cond)


# --------------------------------------------------------------------------------------------------------------------
# D. gpx_pdinv on several outer blocks
# --------------------------------------------------------------------------------------------------------------------
def lapack_pdinv(A, lower=True):
    L = sla.cholesky(A, lower=lower)
    L = L if lower else L.T
    Li = sla.solve_triangular(L, np.eye(A.shape[0]), lower=True)
    return Li.T @ Li, L, Li, 2 * np.log(np.diag(L)).sum()


def lapack_spread(A):
    """LAPACK's result and how far two LAPACK evaluations of it lie apart: L, L^-1 and the log-determinant from the
    lower (L L^T) against the upper (U^T U) factorisation, which round differently; A^-1 from A against A in reversed
    order (every elimination step differs), mapped back. The device's distance from LAPACK is held to 4 times this."""
    r = np.arange(A.shape[0])[::-1]
    Ai1, L1, Li1, ld1 = lapack_pdinv(A)
    _, L2, Li2, ld2 = lapack_pdinv(A, lower=False)
    Ai2 = lapack_pdinv(A[np.ix_(r, r)])[0][np.ix_(r, r)]
    # the two triangular factorisations share the order of their last pivot's cancellation, so for a matrix whose
    # ill-conditioning sits in its last row they agree on L^-1 far better than either is accurate: L^-1 gets A^-1's spread
    sAi = rel(Ai2, Ai1)
    return (Ai1, L1, Li1, ld1), dict(Ai=sAi, L=rel(L2, L1), Li=max(rel(Li2, Li1), sAi), logdet=abs(ld2 - ld1) / abs(ld1))


def pdinv_matrix(n, which):
    X, _ = o.synthetic(n, 3, seed=n)
    if which == "singular_tail":      # the last row repeats the first: the only non-positive pivot is in the last block
        X[-1] = X[0]
        return o.StationaryOracle("exponential", 3, 1.0, 1.5, False).K(X), None
    A = o.StationaryOracle("matern52", 3, 1.0, 2.0, False).K(X) + 1e-6 * np.eye(n)
    if which == "graded":
        d = np.logspace(-4, 4, n)[np.random.default_rng(n).permutation(n)]
        return d[:, None] * A * d[None, :], d
    return A, None


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["noisy", "graded", "singular_tail"])
@pytest.mark.parametrize("n", [2049, 4097])
def test_pdinv_multi_block(n, which):
    f = _ffi()
    A, d = pdinv_matrix(n, which)
    if which == "singular_tail":
        L0, jit0 = o.jitchol(A)
        assert jit0 > 0
        Aj = A + jit0 * np.eye(n)
    else:
        Aj, jit0 = A, 0.0
    Ai, L, Li, logdet, jit = f.pdinv(A)
    assert np.isclose(jit, jit0, rtol=1e-12, atol=0), (jit, jit0)
    # compare on the scale-free matrix: D A D has L = D L_A, L^-1 = L_A^-1 D^-1, A^-1 = D^-1 A^-1 D^-1
    s = np.ones(n) if d is None else d
    As = Aj / s[:, None] / s[None, :]
    (Ai0, L0, Li0, logdet0), spread = lapack_spread(As)
    Ai, L, Li = Ai * s[:, None] * s[None, :], L / s[:, None], Li * s[None, :]
    logdet = logdet - 2 * np.log(s).sum()
    dev = dict(Ai=rel(Ai, Ai0), L=rel(L, L0), Li=rel(Li, Li0), logdet=abs(logdet - logdet0) / abs(logdet0))
    print("\npdinv n=%d %s: LAPACK spread %s\n  device %s" % (n, which, spread, dev))
    assert rel(L @ L.T, As) <= 1e-14                      # backward error, independent of the conditioning
    for k, floor in (("L", 1e-12), ("Li", 1e-11), ("Ai", 1e-11), ("logdet", 1e-12)):
        assert dev[k] <= max(floor, 4 * spread[k]), (k, dev, spread)
