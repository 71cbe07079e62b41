"""A one-part composite description that is exactly a single stationary kernel (one part of kind RBF .. Matern52 on the
columns 0 .. D-1 in order) runs the single-kernel kernels: the composite and part entries give the same bits as the
single-kernel entries and launch as many kernels. Any other one-part description (its columns permuted or a subset of
them, a RatQuad part) keeps the composite kernels, which shows in the launch count of an evaluation."""
import ctypes

import numpy as np
import pytest

from gpy_b200 import _ffi

pytestmark = pytest.mark.gpu

D = 3
RUNS = [(k, ard) for k in ("rbf", "exponential", "matern32", "matern52") for ard in (False, True)]
IDS = ["%s-%s" % (k, "ard" if a else "iso") for k, a in RUNS]
LS = np.array([0.9, 1.4, 2.1])


def _theta(ard):
    return 1.3, (LS if ard else 1.2)


def _desc(kind, ard, dims=(0, 1, 2)):
    """the part on the given columns; with ARD each column keeps its lengthscale"""
    var, ls = _theta(ard)
    return (kind, ard, 0, list(dims), var, LS[list(dims)] if ard else ls)


def _problem(N, seed):
    rng = np.random.default_rng(seed)
    X = rng.uniform(-3, 3, (N, D))
    Y = np.sin(X).sum(1, keepdims=True) / np.sqrt(D) + 0.1 * rng.standard_normal((N, 1))
    return rng, X, Y


def _launches(e, fn):
    l0 = e.total_launches()
    out = fn()
    return out, e.total_launches() - l0


def _same_bits(a, b):
    a, b = (np.ascontiguousarray(np.asarray(v, dtype=np.float64)) for v in (a, b))
    return a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64))


def _assert_same(single, part):
    (out_s, n_s), (out_p, n_p) = single, part
    assert len(out_s) == len(out_p)
    for a, b in zip(out_s, out_p):
        assert _same_bits(a, b), (a, b)
    assert n_s == n_p


EXACT = [(300, 0), (1100, 0), (1100, 1)]   # fine LAUUM route; fused LAUUM route; int8 sweep (first block row split off)


@pytest.mark.parametrize("N,ozaki", EXACT, ids=["n%d-oz%d" % r for r in EXACT])
@pytest.mark.parametrize("kind,ard", RUNS, ids=IDS)
def test_exact_evaluation(kind, ard, N, ozaki):
    _, X, Y = _problem(N, 11)
    var, ls = _theta(ard)
    e = _ffi.Engine(0)
    try:
        e.set_option("ozaki", ozaki)
        e.set_data(X, Y)
        e.exact_eval(kind, ard, var, ls, 0.05)
        single = _launches(e, lambda: e.exact_eval(kind, ard, var, ls, 0.05))
        part = _launches(e, lambda: e.exact_eval_multi([_desc(kind, ard)], 0.05))
        _assert_same(single, part)
    finally:
        e.close()


@pytest.mark.parametrize("het", [False, True], ids=["scalar", "per-point"])
@pytest.mark.parametrize("kind,ard", RUNS, ids=IDS)
def test_sparse_evaluation(kind, ard, het):
    rng, X, Y = _problem(700, 12)
    Z = X[rng.permutation(700)[:130]] + 0.01 * rng.standard_normal((130, D))
    noise = rng.uniform(0.01, 0.3, 700) if het else 0.05
    var, ls = _theta(ard)
    e = _ffi.Engine(0)
    try:
        e.sparse_set_data(X, Y)
        call = (lambda: e.sparse_eval_het(kind, ard, var, ls, Z, noise)) if het else \
               (lambda: e.sparse_eval(kind, ard, var, ls, Z, noise))
        call()   # child contexts and their workspaces
        single = _launches(e, call)
        part = _launches(e, lambda: e.sparse_eval_multi([_desc(kind, ard)], Z, noise))
        _assert_same(single, part)
    finally:
        e.close()


@pytest.mark.parametrize("kind,ard", RUNS, ids=IDS)
def test_kern_K_and_grad_full(kind, ard):
    rng, X, _ = _problem(300, 13)
    X2 = rng.uniform(-3, 3, (170, D))
    var, ls = _theta(ard)
    k, a, lsv = _ffi._theta(kind, ard, ls, D)
    part, keep = _ffi.GpxKernPart(), []
    _ffi._fill_part(part, _desc(kind, ard), keep)
    e = _ffi.Engine(0)
    L, h, p = _ffi.lib(), e._h, _ffi._ptr
    try:
        for x2 in (None, X2):
            M = 300 if x2 is None else 170
            dL = rng.standard_normal((300, M))

            def kern_K():
                out = np.empty((300, M))
                assert L.gpx_kern_K(h, k, a, var, p(lsv), p(X), 300, p(x2), M, D, p(out)) == 0
                return [out]

            def part_K():
                out = np.empty((300, M))
                assert L.gpx_kern_part_K(h, ctypes.byref(part), p(X), 300, p(x2), M, D, p(out)) == 0
                return [out]

            def grad_full():
                dv, dl = np.zeros(1), np.zeros(lsv.size)
                assert L.gpx_kern_grad_full(h, k, a, var, p(lsv), p(X), 300, p(x2), M, D, p(dL), p(dv), p(dl)) == 0
                return [np.concatenate([dv, dl])]

            def part_grad_full():
                g = np.zeros(1 + lsv.size)
                assert L.gpx_kern_part_grad_full(h, ctypes.byref(part), p(X), 300, p(x2), M, D, p(dL), p(g)) == 0
                return [g]

            _assert_same(_launches(e, kern_K), _launches(e, part_K))
            _assert_same(_launches(e, grad_full), _launches(e, part_grad_full))
    finally:
        e.close()


OTHER = {
    "permuted": ("matern52", True, 0, [2, 1, 0], 1.3, LS[::-1].copy()),   # the single kernel's covariance, columns reversed
    "subset": ("rbf", True, 0, [0, 1], 1.3, LS[:2].copy()),
    "ratquad": ("ratquad", False, 0, [0, 1, 2], 1.3, 1.2, {"power": 1.5}),
}


@pytest.mark.parametrize("name", list(OTHER))
def test_other_one_part_descriptions_keep_the_composite_route(name):
    """N = 1100: the single kernel reduces K^-1 in the fused LAUUM epilogue; a composite stores K^-1 and reduces it in one
    more launch per part. The sparse evaluation adds the rank-P term of dL_dKnm in one more launch for a composite."""
    desc = OTHER[name]
    rng, X, Y = _problem(1100, 14)
    var, ls = _theta(True)
    e = _ffi.Engine(0)
    try:
        e.set_data(X, Y)
        e.exact_eval("matern52", True, var, ls, 0.05)
        (lml_s, _, _), n_s = _launches(e, lambda: e.exact_eval("matern52", True, var, ls, 0.05))
        (lml_p, _, _), n_p = _launches(e, lambda: e.exact_eval_multi([desc], 0.05))
        assert n_p == n_s + 1
        if name == "permuted":
            assert abs(lml_p - lml_s) <= 1e-9 * abs(lml_s)
        if name == "ratquad":   # no gradients_X on the device: not on the sparse evaluation
            return
        Z = X[rng.permutation(1100)[:130]] + 0.01 * rng.standard_normal((130, D))
        e.sparse_set_data(X, Y)
        e.sparse_eval("matern52", True, var, ls, Z, 0.05)
        (lml_s, _, _), n_s = _launches(e, lambda: e.sparse_eval("matern52", True, var, ls, Z, 0.05))
        (lml_p, _, _), n_p = _launches(e, lambda: e.sparse_eval_multi([desc], Z, 0.05))
        assert n_p == n_s + 1
        if name == "permuted":
            assert abs(lml_p - lml_s) <= 1e-9 * abs(lml_s)
    finally:
        e.close()
