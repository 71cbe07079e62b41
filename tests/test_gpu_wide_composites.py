"""The composite kernels and the predictive gradients at every register width and channel group: stacked active dims up to
64 and up to 8 outputs, against tests/wide_composites_oracle.py (itself checked against the reference by
tests/test_wide_composites_cpu.py) and the reference fixtures of tests/golden/wide_composites.

Each case asserts, through the oracle module's restatement of the device's choice, the instantiation it runs, so that a
device with another SM count cannot quietly move a case off its target:

| kernel (gpx_multi.cu)                     | picked by                | cases                                                 |
|-------------------------------------------|--------------------------|-------------------------------------------------------|
| grad_kinv_multi<DREG, EXT>                | per part max(D, nacc)    | A: 8 / 16 / 32 / 64 with and without RatQuad / StdPeriodic |
| grad_full_multi<DREG, EXT>                | per part                 | B (stand-alone part entries) and C (sparse, EXT off)  |
| gradx_multi<DREG>                         | sumD                     | C: sumD 9, 17, 33, 64 -> 16, 32, 64, 64               |
| pred_grad<DREG, NCH>                      | sumD                     | D: <8,4> <16,2> <32,1> <64,1>, channel groups >= 2    |
| pred_grad column chunks                   | gradx_chunks             | D: chunks of 96 / 160 with a partial last chunk       |
"""
import functools
import os
import glob

import numpy as np
import pytest
from scipy.linalg import cho_factor, cho_solve

import gpy_b200
import predictive_gradients_oracle as po
import sparse_composite_oracle as so
import wide_composites_oracle as wo
from oracle import gpy_oracle as o
from gpy_b200 import _ffi

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = sorted(glob.glob(os.path.join(HERE, "golden", "wide_composites", "*.npz")))
LML_ATOL = 1e-8
GRAD_RTOL = 1e-6
PG_TOL = 1e-8        # of each Jacobian's largest entry, cond <= 1e6
COND_MAX = 1e6
D64 = 64


@functools.lru_cache(maxsize=1)
def num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def rel(a, b):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape, (a.shape, b.shape)
    return float(np.abs(a - b).max() / np.abs(b).max())


def assert_close(got, want, tol=PG_TOL):
    assert got.shape == want.shape
    err = np.abs(got - want).max()
    assert err <= tol * np.abs(want).max(), (err, np.abs(want).max())


def engine(oz=0):
    e = _ffi.Engine(0)
    e.set_option("ozaki", oz)
    return e


def descs(parts):
    return [wo.descriptor(p) for p in parts]


# ======================================================================================================================
# A. exact composite evaluation: every grad_kinv_multi instantiation, on both tensor paths
# ======================================================================================================================
def _exact_cases():
    c = wo.perm(D64, 11)
    S, Q, R, B = wo.stationary, wo.stdperiodic, wo.ratquad, wo.static
    cases = {
        # name: parts (the expected (DREG, EXT) of every part's gradient pass follows)
        "sumD8": ([S("rbf", c[:5], 0, True), S("matern32", c[5:8], 0, False)], [(8, False)] * 2),
        "sumD9_bias_white": ([S("matern52", c[:9], 0, True), B("bias", 0, 0.8), B("white", 1, 0.05)],
                             [(16, False), (8, False), (8, False)]),
        "sumD16_shared": ([S("rbf", c[:12], 0, True), S("exponential", c[8:12], 1, False)], [(16, False), (8, False)]),
        "sumD17_static_prods": ([S("matern32", c[:17], 0, True), B("bias", 0, 0.9), B("white", 1, 0.7), B("bias", 1, 0.1)],
                                [(32, False), (8, False), (8, False), (8, False)]),
        "sumD32": ([S("rbf", c[:32], 0, True)], [(32, False)]),
        "sumD33": ([S("matern52", c[:33], 0, True), B("bias", 1, 0.3)], [(64, False), (8, False)]),
        "sumD64_wide_beside_narrow": ([S("matern52", c[:33], 0, True), S("rbf", c[33:41], 1, True),
                                       S("exponential", c[41:], 1, False), B("white", 1, 0.2), B("bias", 2, 0.1)],
                                      [(64, False), (8, False), (32, False), (8, False), (8, False)]),
        "eight_parts_x8": (wo.eight_parts(c), [(8, False)] * 8),
        "ratquad_ard64": ([R(c, 0, True, power=0.8)], [(64, True)]),
        "stdperiodic8_iso": ([Q(c[:8], 0, False, False), S("matern52", c[8:12], 0, True)], [(16, True), (8, True)]),
        "stdperiodic9_ard": ([Q(c[:9], 0, True, True), S("rbf", c[9:20], 0, False)], [(32, True), (16, True)]),
        "ratquad17_x_rbf": ([R(c[:17], 0, False), S("rbf", c[10:27], 0, True), Q(c[30:33], 1, True, False)],
                            [(32, True), (32, True), (8, True)]),
    }
    for a1 in (False, True):
        for a2 in (False, True):
            cases["stdperiodic32_%d%d" % (a1, a2)] = ([Q(c[:32], 0, a1, a2)], [(64, True)])
    return cases


EXACT = _exact_cases()
# every StdPeriodic-on-32-dims variant once per tensor path at N = 700, the rest at N = 700 and 2049 (several outer blocks,
# a row tail)
EXACT_RUNS = [(k, N, oz) for k in EXACT for N in (700, 2049) for oz in (0, 1)
              if not (k.startswith("stdperiodic32") and N == 2049 and k != "stdperiodic32_11")]


@functools.lru_cache(maxsize=4)
def exact_reference(name, N):
    parts = EXACT[name][0]
    X, Y = wo.data(N, D64, 2, N + sum(map(ord, name)))
    lml, g, res = wo.exact_eval(X, Y, parts, 0.1)
    w = np.linalg.eigvalsh(res["Ky"])
    return X, Y, lml, g, res, w[-1] / w[0]


@pytest.mark.parametrize("name,N,oz", EXACT_RUNS, ids=["%s-N%d-oz%d" % r for r in EXACT_RUNS])
def test_exact_composite(name, N, oz):
    parts, routes = EXACT[name]
    assert [wo.grad_route(parts, i) for i in range(len(parts))] == routes
    assert wo.sum_dims(parts) <= 64
    X, Y, lml0, g0, res, cond = exact_reference(name, N)
    assert cond <= COND_MAX, cond
    e = engine(oz)
    e.set_data(X, Y)
    lml, g, jit = e.exact_eval_multi(descs(parts), 0.1)
    assert jit == 0.0
    assert abs(lml - lml0) <= LML_ATOL, (lml, lml0)
    np.testing.assert_allclose(g, g0, rtol=GRAD_RTOL, atol=1e-9)
    assert rel(e.get("alpha"), res["alpha"]) < 1e-9
    kern = res["kern"]
    Xn = np.random.default_rng(N).uniform(-2.0, 2.0, (40, D64))
    mu, v = e.predict(Xn)
    mu0, v0 = o.raw_predict(kern, X, res["L"], res["alpha"], Xn)
    assert rel(mu, mu0) < 1e-9        # mu = K(X, Xn)^T alpha carries alpha's max-norm error (7 digits of U on the int8 path)
    np.testing.assert_allclose(v, v0, rtol=1e-7, atol=1e-10)
    mu, cov = e.predict(Xn[:12], full_cov=True)
    _, cov0 = o.raw_predict(kern, X, res["L"], res["alpha"], Xn[:12], full_cov=True)
    np.testing.assert_allclose(cov, cov0, rtol=1e-7, atol=1e-10)
    e.close()


# ---- the reference fixtures ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("oz", [0, 1])
@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[:-4])
def test_matches_the_reference_fixtures(path, oz):
    f = np.load(path)
    parts = wo.fixture_kernels()[str(f["kernel"])]
    e = engine(oz)
    e.set_data(f["X"], f["Y"])
    if "lml" in f.files:
        lml, g, _ = e.exact_eval_multi(descs(parts), float(f["noise"]))
        assert abs(lml - float(f["lml"])) <= LML_ATOL
        np.testing.assert_allclose(g, f["grad"], rtol=GRAD_RTOL, atol=1e-9)
        assert rel(e.get("alpha"), f["alpha"]) < 1e-9
    else:
        e.exact_eval_multi(descs(parts), float(f["noise"]))
        mj, vj = e.predictive_gradients(f["Xnew"])
        assert_close(mj, f["mean_jac"])
        assert_close(vj, f["var_jac"])
    e.close()


# ======================================================================================================================
# B. stand-alone part entries: gpx_kern_part_K / gpx_kern_part_grad_full (grad_full_multi with and without EXT)
# ======================================================================================================================
LD = np.longdouble


def _ld_block(p, X, X2, dL):
    """K and the gradient block of one part with every per-pair term and every sum in extended precision (x87 long
    double): the reference's own rounding sits far below the bars. Differences are formed directly, not by the
    |x|^2 + |x'|^2 - 2 x.x' expansion; the diagonal of K(X, X) has exactly zero distance on both sides."""
    kind, var = p["kind"], LD(p["variance"])
    A = X.astype(LD)
    Bm = A if X2 is None else X2.astype(LD)
    diff = A[:, None, :] - Bm[None, :, :]
    dL = dL.astype(LD)
    if kind == "stdperiodic":
        T = np.asarray(p["period"], dtype=LD) * np.ones(A.shape[1], dtype=LD)
        l = np.asarray(p["lengthscale"], dtype=LD) * np.ones(A.shape[1], dtype=LD)
        u = diff / T
        s, cs = np.sin(np.pi * u), np.cos(np.pi * u)   # standard_periodic.py:130-131, 511-513
        k = np.exp(-0.5 * np.sum(np.square(s / l), -1))
        W = var * k * dL
        dper = np.einsum("ij,ijq->q", W, s * cs * (np.pi * u / T) / l ** 2)
        dlen = np.einsum("ij,ijq->q", W, s * s / l ** 3)
        g = [[np.sum(k * dL)], dper if p["ARD_period"] else [dper.sum()], dlen if p["ARD"] else [dlen.sum()]]
        return var * k, np.concatenate([np.asarray(x, dtype=LD) for x in g])
    ard = p.get("ARD", False)
    l = np.asarray(p["lengthscale"], dtype=LD)
    sc = diff / l if ard else diff
    r = np.sqrt(np.sum(sc * sc, -1)) / (1 if ard else l)
    if kind == "ratquad":
        lg = np.log1p(r * r / 2)
        k = np.exp(-LD(p["power"]) * lg)
        dk = -LD(p["power"]) * r * np.exp(-(LD(p["power"]) + 1) * lg)
    else:
        k = o.K_of_r(kind, LD(1), r)
        dk = o.dK_dr(kind, LD(1), r)
    dLr = var * dk * dL
    if ard:                                         # stationary.py:205-213,225-235: 1/r with 1/0 := 0
        inv = np.where(r != 0, 1 / np.where(r != 0, r, 1), 0)
        dl = -np.einsum("ij,ijq->q", dLr * inv, sc * sc) / l
    else:
        dl = [-np.sum(dLr * r) / l]
    g = [[np.sum(k * dL)], dl]
    if kind == "ratquad":
        g.append([np.sum(dL * -var * k * lg)])      # stationary.py:795-798
    return var * k, np.concatenate([np.asarray(x, dtype=LD).reshape(-1) for x in g])


PART_KINDS = ("rbf", "exponential", "matern32", "matern52", "ratquad", "stdperiodic")
PART_RUNS = [(k, d, ard) for k in PART_KINDS for d in (8, 9, 16, 17, 32, 33, 64) for ard in (False, True)
             if not (k == "stdperiodic" and d > 32)]


def _part(kind, d, ard, cols):
    if kind == "stdperiodic":
        return wo.stdperiodic(cols[:d], 0, ard, not ard if d % 2 else ard)   # every ARD1 / ARD2 pairing over the dims
    if kind == "ratquad":
        return wo.ratquad(cols[:d], 0, ard)
    return wo.stationary(kind, cols[:d], 0, ard)


@pytest.mark.parametrize("kind,d,ard", PART_RUNS, ids=["%s-d%d-%s" % (k, d, "ard" if a else "iso") for k, d, a in PART_RUNS])
def test_stand_alone_part_entries(kind, d, ard):
    rng = np.random.default_rng(d + 100 * PART_KINDS.index(kind) + ard)
    cols = wo.perm(D64, d)
    p = _part(kind, d, ard, cols)
    dreg, ext = wo.grad_route([p], 0)
    assert ext == (kind in ("ratquad", "stdperiodic"))
    assert dreg == wo.width(max(d, wo.part_nacc(p)))
    X, X2 = rng.uniform(-2, 2, (300, D64)), rng.uniform(-2, 2, (170, D64))
    desc = wo.descriptor(p)
    for B in (None, X2):
        Xs, Bs = X[:, cols[:d]], None if B is None else B[:, cols[:d]]
        M = X.shape[0] if B is None else B.shape[0]
        pos = rng.uniform(0.1, 1.0, (300, M))
        sgn = rng.standard_normal((300, M))
        if B is None:
            pos, sgn = pos + pos.T, sgn + sgn.T
        K0, gpos = _ld_block(p, Xs, Bs, pos)
        got = _ffi.kern_part_K(desc, X, B)
        assert np.abs(got - K0).max() <= 1e-12 * np.abs(K0).max()
        assert np.all(np.abs(got - K0) <= 1e-12 * np.abs(K0) + 1e-15)
        gp = _ffi.kern_part_grad_full(desc, X, pos, B)
        assert gp.size == gpos.size
        assert np.abs(gp - gpos).max() <= 1e-10 * np.abs(gpos).max(), (np.abs(gp - gpos).max(), np.abs(gpos).max())
        _, gsgn = _ld_block(p, Xs, Bs, sgn)
        gs = _ffi.kern_part_grad_full(desc, X, sgn, B)
        assert np.abs(gs - gsgn).max() <= 1e-9 * np.abs(gsgn).max(), (np.abs(gs - gsgn).max(), np.abs(gsgn).max())


# ======================================================================================================================
# C. sparse composite evaluation: gradx_multi<16 / 32 / 64> for dL/dZ, grad_full_multi per part
# ======================================================================================================================
def _sparse_kernels():
    c = wo.perm(D64, 23)
    S, B = wo.stationary, wo.static
    return {
        9: [S("matern52", c[:6], 0, True), S("rbf", c[6:9], 0, False), B("bias", 1, 0.3)],
        17: [S("rbf", c[:17], 0, True), B("white", 1, 0.05)],
        33: [S("matern32", c[:20], 0, True), S("exponential", c[20:33], 1, True), B("bias", 1, 0.6)],
        64: [S("matern52", c[:33], 0, True), S("rbf", c[33:56], 0, False), S("exponential", c[:8], 1, False),
             B("white", 2, 0.02)],
    }


SPARSE = _sparse_kernels()
SPARSE_RUNS = [(s, P, het) for s in (9, 17, 33, 64) for P in (1, 3) for het in (False, True)]


def sparse_data(N, M, P, het, seed, parts, D=D64):
    X, Y = wo.data(N, D, P, seed)
    Z = wo.spread_points(X, M)
    noise = 0.05 + 0.1 * np.random.default_rng(seed).uniform(size=N) if het else 0.08
    kern = so.CompositeOracle(parts)
    cond = np.linalg.cond(kern.K(Z) + 1e-8 * np.eye(M))
    assert cond <= COND_MAX, cond
    return X, Y, Z, noise


def _maxnorm(a, b, what, tol=1e-7):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape, what
    assert np.abs(a - b).max() <= tol * np.abs(b).max(), (what, np.abs(a - b).max(), np.abs(b).max())


@pytest.mark.parametrize("sumD,P,het", SPARSE_RUNS, ids=["sumD%d-P%d-%s" % (s, P, "het" if h else "scalar")
                                                         for s, P, h in SPARSE_RUNS])
def test_sparse_composite(sumD, P, het):
    parts = SPARSE[sumD]
    assert wo.sum_dims(parts) == sumD
    assert wo.width(sumD) == {9: 16, 17: 32, 33: 64, 64: 64}[sumD]        # gradx_multi's instantiation
    X, Y, Z, noise = sparse_data(1500, 160, P, het, 7 * sumD + P, parts)
    lml, grad, Zg, res = so.sparse_composite_eval(X, Y, Z, parts, noise)
    e = engine()
    e.sparse_set_data(X, Y)
    out = e.sparse_eval_multi(descs(parts), Z, noise)
    assert abs(out[0] - lml) <= 1e-8 * abs(lml), (out[0], lml)
    np.testing.assert_allclose(out[1], grad, rtol=GRAD_RTOL, atol=1e-9 * np.abs(grad).max())
    _maxnorm(out[2], Zg, "dZ")
    if het:
        _maxnorm(out[3], res["dL_dthetaL"], "dL_dR")
    _maxnorm(e.sparse_get("woodbury_vector"), res["woodbury_vector"], "woodbury_vector")
    _maxnorm(e.sparse_get("woodbury_inv"), res["woodbury_inv"], "woodbury_inv")
    e.close()


# ======================================================================================================================
# D. predictive gradients: every pred_grad instantiation, channel groups, column chunks, coincident points
# ======================================================================================================================
def _reduction_launches(sumD, P):
    return wo.pred_grad_launches(sumD, P)


def exact_posterior(kern, X, Y, noise):
    Ky = kern.K(X) + (noise + po.JITTER) * np.eye(X.shape[0])
    w = np.linalg.eigvalsh(Ky)
    assert w[-1] / w[0] <= COND_MAX, w[-1] / w[0]
    c = cho_factor(Ky, lower=True)
    return cho_solve(c, Y), cho_solve(c, np.eye(X.shape[0]))


def check_pg(e, kern, wv, wi, Xnew, Xpred, sparse, first=False):
    """one device call against the oracle, with its launch count"""
    sumD = wo.sum_dims(kern.parts)
    P = wv.shape[1]
    l0 = e.total_launches()
    mj, vj = (e.sparse_predictive_gradients if sparse else e.predictive_gradients)(Xnew)
    R = _reduction_launches(sumD, P)
    want = (8 if first else 3) + R if sparse else 2 + 3 * -(-Xnew.shape[0] // 8) + R
    assert e.total_launches() - l0 == want
    rm, rv = po.jacobians(kern, wv, wi, Xnew, Xpred)
    assert_close(mj, rm)
    assert_close(vj, rv)


def _single_runs():
    return [(k, D, ard) for k in wo.STATIONARY for D in (9, 17, 33, 64) for ard in (False, True)]


SINGLE_RUNS = _single_runs()


@pytest.mark.parametrize("kind,D,ard", SINGLE_RUNS, ids=["%s-D%d-%s" % (k, D, "ard" if a else "iso") for k, D, a in SINGLE_RUNS])
def test_pred_grad_single_kernels(kind, D, ard):
    """the single-kernel evaluations (gpx_exact_eval, gpx_sparse_eval_multi with one part) at D 9 .. 64"""
    p = wo.stationary(kind, list(range(D)), 0, ard)
    dreg, nch = wo.pred_grad_route(D)
    assert (dreg, nch) == {9: (16, 2), 17: (32, 1), 33: (64, 1), 64: (64, 1)}[D]
    X, Y = wo.data(700, D, 2, D + 3 * ard)
    kern = wo.WideOracle([p])
    wv, wi = exact_posterior(kern, X, Y, 0.1)
    Xnew = np.random.default_rng(1000 + D).uniform(-2.0, 2.0, (129, D))
    # test points on training / inducing rows: their own pair drops out (x - x' = 0). Not for the Exponential kernel on
    # these inputs: its k(x, x) takes the ~1e-8 left by the cancellation in r at first order (test_pred_grad_coincident_points
    # has it on inputs where r = 0 exactly)
    ncoin = 0 if kind == "exponential" else 3
    Xnew[:ncoin] = X[:ncoin]
    e = engine()
    e.set_data(X, Y)
    e.exact_eval(kind, ard, p["variance"], p["lengthscale"], 0.1)
    check_pg(e, kern, wv, wi, Xnew, X, False)
    Z = wo.spread_points(X, 90)
    assert np.linalg.cond(kern.K(Z) + 1e-8 * np.eye(90)) <= COND_MAX
    swv, swi = po.sparse_posterior(kern, X, Y, Z, 0.1)
    Xnew[:ncoin] = Z[:ncoin]
    e.sparse_set_data(X, Y)
    e.sparse_eval_multi(descs([p]), Z, 0.1)
    check_pg(e, kern, swv, swi, Xnew, Z, True, first=True)
    e.close()


def _group_kernels():
    c = wo.perm(D64, 31)
    S, B = wo.stationary, wo.static
    return {
        8: [S("rbf", c[:5], 0, True), S("matern32", c[5:8], 0, False), B("bias", 1, 0.4)],
        12: [S("matern52", c[:9], 0, True), S("exponential", c[6:9], 0, False), B("white", 1, 0.05)],
        24: [S("rbf", c[:17], 0, True), S("matern32", c[17:24], 1, True)],
        64: [S("rbf", c[:33], 0, True), S("matern32", c[33:41], 0, False), S("exponential", c[41:], 1, True, variance=0.5),
             B("bias", 2, 0.2)],
    }


GROUPS = _group_kernels()
GROUP_RUNS = [(8, (4, 7, 8), 1025), (12, (1, 2, 8), 2049), (24, (1, 3), 1025), (64, (1, 3), 2049)]
N_GROUPS = 4097


@functools.lru_cache(maxsize=1)
def _group_data(sumD, Pmax):
    X, Y = wo.data(N_GROUPS, D64, Pmax, sumD)
    return X, Y


@pytest.mark.parametrize("sumD,Ps,Mbig", GROUP_RUNS, ids=["sumD%d" % r[0] for r in GROUP_RUNS])
def test_pred_grad_channel_groups_and_chunks_exact(sumD, Ps, Mbig):
    """N = 4097 training points; M* = Mbig (several chunks of more than 32 columns, the last one partial), 1 and 129"""
    parts = GROUPS[sumD]
    assert wo.sum_dims(parts) == sumD
    dreg, nch = wo.pred_grad_route(sumD)
    assert (dreg, nch) == {8: (8, 4), 12: (16, 2), 24: (32, 1), 64: (64, 1)}[sumD]
    groups = [wo.channel_groups(sumD, P) for P in Ps]
    assert any(len(g) >= 2 for g in groups)
    if sumD == 8:    # P = 4: the variance channel alone in launch 2; P = 7: in a full second group; P = 8: three launches
        assert groups[0][1] == (4, 1, True) and groups[1][1] == (4, 4, True) and len(groups[2]) == 3
    nchunk, mchunk, last = wo.gradx_chunks(Mbig, N_GROUPS, num_sms())
    assert mchunk > 32 and last < mchunk and nchunk >= 2, (nchunk, mchunk, last)
    X, Yall = _group_data(sumD, max(Ps))
    kern = wo.WideOracle(parts)
    Ky = kern.K(X) + (0.1 + po.JITTER) * np.eye(N_GROUPS)
    w = np.linalg.eigvalsh(Ky)
    assert w[-1] / w[0] <= COND_MAX
    c = cho_factor(Ky, lower=True)
    wi = cho_solve(c, np.eye(N_GROUPS))
    Xnew = np.random.default_rng(1000 + sumD).uniform(-2.0, 2.0, (Mbig, D64))
    e = engine()
    for P in Ps:
        Y = np.ascontiguousarray(Yall[:, :P])
        wv = cho_solve(c, Y)
        e.set_data(X, Y)
        e.exact_eval_multi(descs(parts), 0.1)
        for Ms in (Mbig, 1, 129):
            check_pg(e, kern, wv, wi, Xnew[:Ms], X, False)
    e.close()


@pytest.mark.parametrize("sumD,Ps,Mbig", GROUP_RUNS, ids=["sumD%d" % r[0] for r in GROUP_RUNS])
def test_pred_grad_channel_groups_sparse(sumD, Ps, Mbig):
    parts = GROUPS[sumD]
    X, Yall = _group_data(sumD, max(Ps))
    kern = so.CompositeOracle(parts)
    Z = wo.spread_points(X, 300)
    assert np.linalg.cond(kern.K(Z) + 1e-8 * np.eye(300)) <= COND_MAX
    Xnew = np.random.default_rng(sumD + 1).uniform(-2.0, 2.0, (Mbig, D64))
    e = engine()
    for P in Ps:
        Y = np.ascontiguousarray(Yall[:, :P])
        wv, wi = po.sparse_posterior(kern, X, Y, Z, 0.08)
        e.sparse_set_data(X, Y)
        e.sparse_eval_multi(descs(parts), Z, 0.08)
        check_pg(e, kern, wv, wi, Xnew, Z, True, first=True)
        check_pg(e, kern, wv, wi, Xnew[:129], Z, True)
    e.close()


def _coincident_case():
    """inputs on a grid of 1/4 and lengthscales that are powers of two: |x|^2 + |x'|^2 - 2 x.x' is exact on both sides,
    so coincident points have r = 0 exactly (the Exponential kernel, dk/dr != 0 at r = 0, then takes GPy's 1/0 := 0)"""
    rng = np.random.default_rng(41)
    D = 20
    X = rng.integers(-8, 9, (900, D)) / 4.0
    Y = np.sin(X[:, :4].sum(1, keepdims=True)) + 0.1 * rng.standard_normal((900, 1))
    Y = np.concatenate([Y, np.cos(X[:, 4:6].sum(1, keepdims=True))], 1)
    parts = [dict(kind="exponential", term=0, dims=list(range(9)), variance=1.1, lengthscale=4.0),
             dict(kind="rbf", term=0, dims=list(range(9, 17)), variance=0.9, lengthscale=np.array([2.0, 4.0] * 4),
                  ARD=True),
             dict(kind="matern32", term=1, dims=[17, 18, 19], variance=0.5, lengthscale=np.array([2.0, 1.0, 2.0]),
                  ARD=True),
             dict(kind="exponential", term=2, dims=[0, 5, 17], variance=0.3, lengthscale=np.array([2.0, 4.0, 2.0]),
                  ARD=True)]
    return X, Y, parts


def _coincident_points(rng, P, D=20):
    """rows equal to P's rows (all dims), equal only on the Exponential factor's dims 0-8, only on the RBF factor's 9-16"""
    Xn = rng.integers(-8, 9, (48, D)) / 4.0
    Xn[:16] = P[:16]
    Xn[16:32, :9] = P[16:32, :9]
    Xn[32:48, 9:17] = P[32:48, 9:17]
    return Xn


def test_pred_grad_coincident_points():
    X, Y, parts = _coincident_case()
    kern = wo.WideOracle(parts)
    wv, wi = exact_posterior(kern, X, Y, 0.1)
    rng = np.random.default_rng(5)
    Xnew = _coincident_points(rng, X)
    e = engine()
    e.set_data(X, Y)
    e.exact_eval_multi(descs(parts), 0.1)
    check_pg(e, kern, wv, wi, Xnew, X, False)
    Z = wo.spread_points(X, 120, offset=0.0)    # on the grid: r = 0 exactly where Z meets the data
    assert np.linalg.cond(kern.K(Z) + 1e-8 * np.eye(120)) <= COND_MAX
    swv, swi = po.sparse_posterior(kern, X, Y, Z, 0.1)
    e.sparse_set_data(X, Y)
    e.sparse_eval_multi(descs(parts), Z, 0.1)
    check_pg(e, kern, swv, swi, _coincident_points(rng, Z), Z, True, first=True)
    e.close()


def test_mirror_models():
    """GPRegression.predictive_gradients for a single ARD kernel on 40 of 64 columns (the scatter into the data's
    columns), with the normalizer at P = 8; SparseGPRegression.predictive_gradients for a sumD-33 composite"""
    cols = wo.perm(D64, 3)[:40]
    X, Y = wo.data(800, D64, 8, 77)
    Y = Y * np.linspace(0.5, 3.0, 8) + np.arange(8)
    p = wo.stationary("matern52", cols, 0, True)
    k = gpy_b200.Matern52(40, variance=p["variance"], lengthscale=p["lengthscale"], ARD=True, active_dims=cols)
    e = engine()
    m = gpy_b200.GPRegression(X, Y, k, noise_var=0.1, normalizer=True, engine=e)
    Xnew = np.random.default_rng(8).uniform(-2, 2, (33, D64))
    l0 = e.total_launches()
    mj, vj = m.predictive_gradients(Xnew)
    assert e.total_launches() - l0 == 2 + 3 * 5 + _reduction_launches(40, 8)
    kern = wo.WideOracle([p])
    Yn, _, std = po.standardize(Y)
    wv, wi = exact_posterior(kern, X, Yn, 0.1)
    rm, rv = po.denormalize(*po.jacobians(kern, wv, wi, Xnew, X), std)
    assert_close(mj, rm)
    assert_close(vj, rv)
    assert np.all(mj[:, [q for q in range(D64) if q not in cols], :] == 0)
    parts = SPARSE[33]
    X, Y = wo.data(1200, D64, 2, 78)
    Z = wo.spread_points(X, 150)
    ck = so.CompositeOracle(parts)
    assert np.linalg.cond(ck.K(Z) + 1e-8 * np.eye(150)) <= COND_MAX
    s = gpy_b200.SparseGPRegression(X, Y, wo.mirror_kernel(parts, D64), Z=Z, engine=e)
    s.likelihood.variance.values[...] = 0.08
    s.parameters_changed()
    sm, sv = s.predictive_gradients(Xnew)
    wv, wi = po.sparse_posterior(ck, X, Y, Z, 0.08)
    rm, rv = po.jacobians(ck, wv, wi, Xnew, Z)
    assert_close(sm, rm)
    assert_close(sv, rv)
    e.close()


# ======================================================================================================================
# E. an ill-conditioned case at sumD 64 against an extended-precision reference
# ======================================================================================================================
def refined_solve(A, B, iters=3):
    """A^-1 B with iterative refinement, residuals in extended precision (x87 long double)"""
    c = cho_factor(A, lower=True)
    x = cho_solve(c, B)
    Al, Bl = A.astype(np.longdouble), B.astype(np.longdouble)
    for _ in range(iters):
        r = Bl - Al @ x.astype(np.longdouble)
        x = x + cho_solve(c, r.astype(np.float64))
    return x


@pytest.mark.parametrize("oz", [0, 1])
def test_ill_conditioned_sumD64(oz):
    """cond(Ky) ~ 1e8: alpha and the predictive gradients against iterative refinement in extended precision. On the DMMA
    path within 16x the fp64 oracle's own error. The int8 path keeps 7 digits in U, and above cond(Ky) ~ 1e8 its alpha is
    documented as less accurate than LAPACK's (include/gpx.h). There the bar is 100x the fp64 oracle's error (measured on
    an H100: 51x on the mean Jacobian, 18x on the variance Jacobian)"""
    c = wo.perm(D64, 11)   # long lengthscales: K's spectrum decays far enough on 700 points in 64 dims
    parts = [wo.stationary("rbf", c[:33], 0, True, scale=25.0), wo.stationary("rbf", c[33:], 0, False, scale=25.0)]
    X, Y = wo.data(700, D64, 1, 64)
    kern = wo.WideOracle(parts)
    K = kern.K(X)
    lam = np.linalg.eigvalsh(K)
    noise = lam[-1] / 1e8 - po.JITTER
    Ky = K + (noise + po.JITTER) * np.eye(700)
    w = np.linalg.eigvalsh(Ky)
    assert 3e7 <= w[-1] / w[0] <= 3e8, w[-1] / w[0]
    Xnew = np.random.default_rng(9).uniform(-2, 2, (40, D64))
    wv64, wi64 = po.exact_posterior(kern, X, Y, noise)
    rm64, rv64 = po.jacobians(kern, wv64, wi64, Xnew, X)
    wv = refined_solve(Ky, Y)
    V = refined_solve(Ky, kern.K(X, Xnew))
    mx = kern.gradients_X(np.broadcast_to(wv[:, 0][None, :], (40, 700)), Xnew, X)[:, :, None]
    vx = -2.0 * kern.gradients_X(np.ascontiguousarray(V.T), Xnew, X)
    e = engine(oz)
    e.set_data(X, Y)
    e.exact_eval_multi(descs(parts), noise)
    mj, vj = e.predictive_gradients(Xnew)
    for got, ref, ext in ((e.get("alpha"), wv64, wv), (mj, rm64, mx), (vj, rv64, vx)):
        e_ref, e_dev = np.abs(ref - ext).max(), np.abs(got - ext).max()
        assert e_dev <= (16 if oz == 0 else 100) * e_ref + 1e-15 * np.abs(ext).max(), (e_dev, e_ref)
    e.close()
