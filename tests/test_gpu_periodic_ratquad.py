"""RatQuad and StdPeriodic on the fused composite evaluation (gpx_exact_eval_multi) and the stand-alone part entries
(gpx_kern_part_K / gpx_kern_part_grad_full), against the CPU oracle of tests/periodic_oracle.py and the stored reference
numbers of tests/golden/reference/periodic_mauna_loa_n300.npz.

| what                                                         | where                                                   |
|--------------------------------------------------------------|---------------------------------------------------------|
| each new kind alone, every ARD variant, one block            | N = 150                                                 |
| the same on multi-dmma / multi-int8                          | N = 700, 2049 (DMMA); 2049 with ozaki = 1 (int8)        |
| Mauna Loa composite on years 1958-2025, both paths           | N = 2049: LML, gradient, alpha, predict, checkgrad, optimize |
| the composite at the fixture's size                          | N = 300, against the reference's own numbers            |
| stand-alone part entries                                     | new kinds vs the oracle; kinds 0-3 vs gpx_kern_K / _grad_full |
"""
import os

import numpy as np
import pytest

from oracle import gpy_oracle as o
import periodic_oracle as po

LML_ATOL = 1e-8
GRAD_RTOL = 1e-6
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference")

INT8_ROUTES = ("multi-int8",)


def assert_route(st, route, nblk, tries=1):
    """the route of the last evaluation from its stats (as tests/test_gpu_routes.py checks it)"""
    int8 = route in INT8_ROUTES
    assert (st["update_int8_ops"] > 0) == int8, (route, st)
    assert (st["lauum_flops"] > 0) == (not int8), (route, st)
    per_try = 2 * nblk - (1 if int8 else 3)
    assert st["update_launches"] == tries * per_try, (route, nblk, st)
    assert st["tries"] == tries, st


def engine(oz):
    import gpy_b200
    e = gpy_b200.Engine()
    e.set_option("ozaki", oz)
    return e


# (name, mirror kernel factory on D dims, oracle part dict)
def _ratquad(ARD, D):
    import gpy_b200
    ls = np.linspace(0.9, 1.9, D) if ARD else 1.3
    return (gpy_b200.RatQuad(D, variance=1.4, lengthscale=ls, power=0.7, ARD=ARD),
            dict(kind="ratquad", term=0, dims=list(range(D)), variance=1.4, lengthscale=ls, power=0.7, ARD=ARD))


def _periodic(ARD1, ARD2, D):
    import gpy_b200
    T = np.linspace(1.1, 2.3, D) if ARD1 else 1.7
    ls = np.linspace(0.8, 1.4, D) if ARD2 else 1.1
    return (gpy_b200.StdPeriodic(D, variance=1.2, period=T, lengthscale=ls, ARD1=ARD1, ARD2=ARD2),
            dict(kind="stdperiodic", term=0, dims=list(range(D)), variance=1.2, period=T, lengthscale=ls, ARD=ARD2,
                 ARD_period=ARD1))


VARIANTS = {"ratquad-iso": lambda D: _ratquad(False, D), "ratquad-ard": lambda D: _ratquad(True, D),
            "periodic-iso-iso": lambda D: _periodic(False, False, D), "periodic-ard-iso": lambda D: _periodic(True, False, D),
            "periodic-iso-ard": lambda D: _periodic(False, True, D), "periodic-ard-ard": lambda D: _periodic(True, True, D)}
CASES = [(v, 150, 0, None, 0) for v in VARIANTS] + \
        [(v, N, 0, "multi-dmma", nb) for v in ("ratquad-ard", "periodic-ard-ard", "periodic-iso-iso")
         for (N, nb) in ((700, 3), (2049, 5))] + \
        [(v, 2049, 1, "multi-int8", 5) for v in ("ratquad-ard", "periodic-ard-iso")]


@pytest.mark.gpu
@pytest.mark.parametrize("variant,N,oz,route,nblk", CASES, ids=["%s-N%d-oz%d" % (c[0], c[1], c[2]) for c in CASES])
def test_new_kind_alone(variant, N, oz, route, nblk):
    import gpy_b200
    D = 3
    X, Y = o.synthetic(N, D, seed=N + 7)
    k, part = VARIANTS[variant](D)
    e = engine(oz)
    m = gpy_b200.GPRegression(X, Y, k, noise_var=0.05, engine=e)
    lml0, g0, _ = po.composite_eval(X, Y, [part], 0.05)
    assert abs(m.log_likelihood() - lml0) <= LML_ATOL
    np.testing.assert_allclose(m.gradient, g0, rtol=GRAD_RTOL, atol=1e-9)
    if route is not None:
        assert_route(e.stats(), route, nblk)


class _CompositeOracleKern(object):
    def __init__(self, kparts):
        self.kparts = kparts

    def K(self, X, X2=None):
        return o.composite_K(self.kparts, X, X2)

    def Kdiag(self, X):
        return o.composite_Kdiag(self.kparts, X)


def _mauna_loa_mirror():
    import gpy_b200
    return gpy_b200.Add([gpy_b200.RBF(1, variance=4.0, lengthscale=50.0),
                         gpy_b200.Prod([gpy_b200.RBF(1, variance=2.0, lengthscale=90.0),
                                        gpy_b200.StdPeriodic(1, variance=1.0, period=1.0, lengthscale=1.3)]),
                         gpy_b200.RatQuad(1, variance=0.5, lengthscale=1.2, power=0.8),
                         gpy_b200.RBF(1, variance=0.1, lengthscale=0.15),
                         gpy_b200.White(1, variance=0.05)])


@pytest.mark.gpu
@pytest.mark.parametrize("oz,route", [(0, "multi-dmma"), (1, "multi-int8")])
def test_mauna_loa_composite(oz, route):
    import gpy_b200
    N = 2049
    X, Y = po.mauna_loa_data(N, seed=3)
    e = engine(oz)
    m = gpy_b200.GPRegression(X, Y, _mauna_loa_mirror(), noise_var=0.01, engine=e)
    assert_route(e.stats(), route, 5)
    lml0, g0, res = po.composite_eval(X, Y, po.mauna_loa_parts(), 0.01)
    assert abs(m.log_likelihood() - lml0) <= LML_ATOL
    np.testing.assert_allclose(m.gradient, g0, rtol=GRAD_RTOL, atol=1e-9)
    alpha = np.asarray(m.posterior.woodbury_vector)
    assert np.max(np.abs(alpha - res["alpha"])) <= 1e-6 * np.max(np.abs(res["alpha"]))
    Xn = np.linspace(1950.0, 2030.0, 37)[:, None]
    kern0 = _CompositeOracleKern(res["kparts"])
    for full in (False, True):
        mu, var = m.predict(Xn, full_cov=full)
        mu0, var0 = o.predict(kern0, X, res["L"], res["alpha"], Xn, 0.01, full_cov=full)
        np.testing.assert_allclose(mu, mu0, rtol=1e-7, atol=1e-8)
        np.testing.assert_allclose(var, var0, rtol=1e-6, atol=1e-8)
    assert m.checkgrad()
    f0 = m.objective_function()
    m.optimize(max_iters=10)
    assert m.objective_function() < f0


@pytest.mark.gpu
def test_mauna_loa_against_the_reference():
    """the composite at the stored fixture's size against the reference's own numbers (Add / Prod / RBF / StdPeriodic /
    RatQuad / White / ExactGaussianInference of GPy)"""
    import gpy_b200
    with np.load(os.path.join(GOLD, "periodic_mauna_loa_n300.npz")) as z:
        r = {k: z[k] for k in z.files}
    for oz in (0, 1):
        m = gpy_b200.GPRegression(r["X"], r["Y"], _mauna_loa_mirror(), noise_var=float(r["noise"]), engine=engine(oz))
        assert abs(m.log_likelihood() - float(r["lml"])) <= LML_ATOL
        np.testing.assert_allclose(m.gradient, r["grad"], rtol=GRAD_RTOL, atol=1e-9)


PART_CASES = [("ratquad", False, False), ("ratquad", True, False), ("stdperiodic", False, False),
              ("stdperiodic", True, False), ("stdperiodic", False, True), ("stdperiodic", True, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,ard,ardp", PART_CASES)
def test_stand_alone_part_entries(kind, ard, ardp):
    from gpy_b200 import _ffi
    D = 3
    rng = np.random.default_rng(11)
    X, X2 = rng.uniform(-2, 2, (230, D)), rng.uniform(-2, 2, (170, D))
    if kind == "ratquad":
        _, p = _ratquad(ard, D)
    else:                      # the periodic argument is formed from raw differences: time-like inputs keep their digits
        _, p = _periodic(ardp, ard, D)
        X, X2 = X + 1990.0, X2 + 1990.0
    k = po.make_part(p)[0]
    desc = po.descriptor(p)
    for A, B in ((X, None), (X, X2)):
        K0 = k.K(A, B)
        np.testing.assert_allclose(_ffi.kern_part_K(desc, A, B), K0, rtol=1e-12, atol=1e-14)
        dL = rng.standard_normal(K0.shape)
        if B is None:
            dL = dL + dL.T
        np.testing.assert_allclose(_ffi.kern_part_grad_full(desc, A, dL, B), k.update_gradients_full(dL, A, B),
                                   rtol=1e-9, atol=1e-9)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["rbf", "exponential", "matern32", "matern52"])
@pytest.mark.parametrize("ARD", [False, True])
def test_part_entries_agree_with_the_single_kernel_entries(kind, ARD):
    from gpy_b200 import _ffi
    D = 3
    rng = np.random.default_rng(5)
    X, X2 = rng.uniform(-3, 3, (200, D)), rng.uniform(-3, 3, (150, D))
    ls = np.array([0.9, 1.4, 2.1]) if ARD else 1.3
    desc = (kind, ARD, 0, list(range(D)), 1.2, ls)
    for B in (None, X2):
        np.testing.assert_allclose(_ffi.kern_part_K(desc, X, B), _ffi.kern_K(kind, ARD, 1.2, ls, X, B), rtol=1e-14, atol=0)
        dL = rng.uniform(0.0, 1.0, (200, 200 if B is None else 150))    # positive: no cancellation in the sums
        if B is None:
            dL = dL + dL.T
        dv, dl = _ffi.kern_grad_full(kind, ARD, 1.2, ls, X, dL, B)
        np.testing.assert_allclose(_ffi.kern_part_grad_full(desc, X, dL, B), np.concatenate([[dv], dl]), rtol=1e-14, atol=0)


@pytest.mark.gpu
def test_rejections():
    import gpy_b200
    from gpy_b200 import _ffi
    X, Y = o.synthetic(300, 33, seed=2)
    e = gpy_b200.Engine()
    e.set_data(X, Y)
    for kind in ("ratquad", "stdperiodic"):
        with pytest.raises(_ffi.GpxArgumentError, match="unknown kernel kind"):
            e.exact_eval(kind, False, 1.0, 1.0, 0.1)
    wide = ("stdperiodic", True, 0, list(range(33)), 1.0, np.ones(33), {"period": np.ones(33), "ARD_period": True})
    with pytest.raises(_ffi.GpxArgumentError, match="does not fit"):
        e.exact_eval_multi([wide], 0.1)
    with pytest.raises(_ffi.GpxArgumentError, match="power"):
        e.exact_eval_multi([("ratquad", False, 0, [0], 1.0, 1.0, {"power": 0.0})], 0.1)
    with pytest.raises(_ffi.GpxArgumentError, match="period"):
        e.exact_eval_multi([("stdperiodic", False, 0, [0], 1.0, 1.0, {"period": -1.0})], 0.1)
    with pytest.raises(_ffi.GpxArgumentError, match="period"):
        _ffi.kern_part_K(("stdperiodic", False, 0, [0], 1.0, 1.0, {"period": 0.0}), X[:, :1])


@pytest.mark.gpu
def test_old_kinds_after_a_periodic_evaluation():
    """a composite of the old kinds on an engine that evaluated a periodic one gives what a fresh engine gives, bit for bit"""
    import gpy_b200
    X, Y = o.synthetic(700, 3, seed=9)
    old = [("rbf", True, 0, [0, 1], 1.2, np.array([1.0, 2.0])), ("matern32", False, 0, [2], 0.8, 1.5),
           ("bias", False, 1, [], 0.3, None)]
    wide = [("rbf", False, 0, [0], 1.0, 1.0), ("stdperiodic", True, 0, [0, 1, 2], 1.1, np.ones(3),
                                               {"period": np.array([1.0, 2.0, 3.0]), "ARD_period": True}),
            ("ratquad", True, 1, [0, 1, 2], 0.7, np.array([1.0, 1.5, 2.0]), {"power": 1.3})]
    fresh = gpy_b200.Engine()
    fresh.set_data(X, Y)
    lml0, g0, _ = fresh.exact_eval_multi(old, 0.05)
    used = gpy_b200.Engine()
    used.set_data(X, Y)
    used.exact_eval_multi(wide, 0.05)
    lml1, g1, _ = used.exact_eval_multi(old, 0.05)
    assert lml1 == lml0
    assert np.array_equal(g1, g0)
    assert np.array_equal(used.get("alpha"), fresh.get("alpha"))
