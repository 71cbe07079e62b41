"""RatQuad and StdPeriodic without a GPU: the oracle of tests/periodic_oracle.py against the reference's own kernels
(stored results under tests/golden/reference/, rewritten from the reference tree with GPX_WRITE_REFERENCE_GOLDEN=1),
the oracle's gradients against finite differences, the mirror's host logic on a fake engine, and the C ABI."""
import importlib
import os

import numpy as np
import pytest

from oracle import gpy_oracle as o
import periodic_oracle as po

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference")
WRITE = os.environ.get("GPX_WRITE_REFERENCE_GOLDEN") == "1"


def _reference(name, compute):
    path = os.path.join(GOLD, name + ".npz")
    if WRITE:
        os.makedirs(GOLD, exist_ok=True)
        np.savez_compressed(path, **{k: np.asarray(v) for k, v in compute().items()})
    with np.load(path) as z:
        return {k: z[k] for k in z.files}


def _ref_modules():
    from oracle import ref_gpy
    G = ref_gpy.load()
    C = ref_gpy.load_combination()
    sp = importlib.import_module("GPy.kern.src.standard_periodic")
    return G, C, sp


def _grad_of(kern):
    return np.concatenate([np.atleast_1d(np.asarray(p.gradient, dtype=np.float64)).reshape(-1) * np.ones(p.size)
                           for p in kern.flattened_parameters()])


KERNEL_CASES = [("ratquad", False, False), ("ratquad", True, False), ("stdperiodic", False, False),
                ("stdperiodic", True, False), ("stdperiodic", False, True), ("stdperiodic", True, True)]


def _case(kind, ard, ardp, D=3):
    if kind == "ratquad":
        ls = np.array([0.9, 1.4, 2.1]) if ard else 1.3
        return dict(kind=kind, term=0, dims=list(range(D)), variance=1.4, lengthscale=ls, power=0.7, ARD=ard)
    T = np.array([1.1, 1.7, 2.3]) if ardp else 1.7
    ls = np.array([0.8, 1.1, 1.4]) if ard else 1.1
    return dict(kind=kind, term=0, dims=list(range(D)), variance=1.2, period=T, lengthscale=ls, ARD=ard, ARD_period=ardp)


def _inputs():
    rng = np.random.default_rng(21)
    X, X2 = rng.uniform(-2, 2, (40, 3)) + 1990.0, rng.uniform(-2, 2, (25, 3)) + 1990.0
    dL = rng.standard_normal((40, 40))
    return X, X2, dL + dL.T, rng.standard_normal((40, 25))


@pytest.mark.parametrize("kind,ard,ardp", KERNEL_CASES)
def test_oracle_kernels_against_the_reference(kind, ard, ardp):
    p = _case(kind, ard, ardp)
    X, X2, dLs, dLr = _inputs()

    def compute():
        G, C, sp = _ref_modules()
        if kind == "ratquad":
            k = G.stationary.RatQuad(3, variance=p["variance"], lengthscale=p["lengthscale"], power=p["power"], ARD=ard)
        else:
            k = sp.StdPeriodic(3, variance=p["variance"], period=p["period"], lengthscale=p["lengthscale"], ARD1=ardp,
                               ARD2=ard)
        out = dict(K=k.K(X), K2=k.K(X, X2), Kdiag=k.Kdiag(X))
        k.update_gradients_full(dLs, X)
        out["grad_sym"] = _grad_of(k)
        k.update_gradients_full(dLr, X, X2)
        out["grad_rect"] = _grad_of(k)
        return out

    r = _reference("periodic_kernel_%s_%d%d" % (kind, ard, ardp), compute)
    k = po.make_part(p)[0]
    np.testing.assert_allclose(k.K(X), r["K"], rtol=1e-14, atol=0)
    np.testing.assert_allclose(k.K(X, X2), r["K2"], rtol=1e-14, atol=0)
    np.testing.assert_allclose(k.Kdiag(X), r["Kdiag"], rtol=1e-14, atol=0)
    np.testing.assert_allclose(k.update_gradients_full(dLs, X), r["grad_sym"], rtol=1e-14, atol=1e-14)
    np.testing.assert_allclose(k.update_gradients_full(dLr, X, X2), r["grad_rect"], rtol=1e-14, atol=1e-14)


def test_mauna_loa_oracle_against_the_reference():
    """LML and the full gradient of RBF + RBF x StdPeriodic + RatQuad + RBF + White through the reference's own Add, Prod,
    kernels, Gaussian likelihood and ExactGaussianInference (the three calls of GP.parameters_changed, gp.py:278-280)"""
    X, Y = po.mauna_loa_data(300, seed=1)
    parts = po.mauna_loa_parts()

    def compute():
        G, C, sp = _ref_modules()
        k = C.Add([G.RBF(1, variance=4.0, lengthscale=50.0),
                   C.Prod([G.RBF(1, variance=2.0, lengthscale=90.0),
                           sp.StdPeriodic(1, variance=1.0, period=1.0, lengthscale=1.3)]),
                   G.stationary.RatQuad(1, variance=0.5, lengthscale=1.2, power=0.8),
                   G.RBF(1, variance=0.1, lengthscale=0.15),
                   C.White(1, variance=0.05)])
        lik = G.Gaussian(variance=0.01)
        post, lml, gd = G.ExactGaussianInference().inference(k, X, lik, Y, None, None)
        lik.update_gradients(gd["dL_dthetaL"])
        k.update_gradients_full(gd["dL_dK"], X)
        grad = np.concatenate([_grad_of(k), np.atleast_1d(lik.variance.gradient).reshape(-1)])
        return dict(X=X, Y=Y, noise=0.01, lml=float(lml), grad=grad, alpha=np.asarray(post.woodbury_vector))

    r = _reference("periodic_mauna_loa_n300", compute)
    lml, g, res = po.composite_eval(r["X"], r["Y"], parts, float(r["noise"]))
    assert g.size == 2 + 2 + 3 + 3 + 2 + 1 + 1
    assert abs(lml - float(r["lml"])) <= 1e-10 * abs(lml)
    np.testing.assert_allclose(g, r["grad"], rtol=1e-10, atol=1e-10)
    np.testing.assert_allclose(res["alpha"], r["alpha"], rtol=1e-10, atol=1e-12)


def _set_theta(p, theta):
    """the oracle part dict p with its gradient-block parameters replaced by theta (block order)"""
    q = dict(p)
    D = len(p["dims"])
    q["variance"] = theta[0]
    if p["kind"] == "ratquad":
        nl = D if p["ARD"] else 1
        q["lengthscale"] = theta[1:1 + nl] if p["ARD"] else theta[1]
        q["power"] = theta[1 + nl]
    else:
        npd = D if p["ARD_period"] else 1
        q["period"] = theta[1:1 + npd] if p["ARD_period"] else theta[1]
        q["lengthscale"] = theta[1 + npd:] if p["ARD"] else theta[1 + npd]
    return q


def _theta(p):
    v = [p["variance"]]
    if p["kind"] == "ratquad":
        return np.concatenate([v, np.atleast_1d(p["lengthscale"]), [p["power"]]])
    return np.concatenate([v, np.atleast_1d(p["period"]), np.atleast_1d(p["lengthscale"])])


@pytest.mark.parametrize("kind,ard,ardp", KERNEL_CASES)
def test_oracle_gradients_against_finite_differences(kind, ard, ardp):
    p = _case(kind, ard, ardp)
    X, X2, dLs, dLr = _inputs()
    if kind == "ratquad":      # Stationary's r^2 = |x|^2 + |x'|^2 - 2 x.x' (stationary.py:130-148) loses ~1e-9 near 1990
        X, X2 = X - 1990.0, X2 - 1990.0
    for B, dL in ((None, dLs), (X2, dLr)):
        g = po.make_part(p)[0].update_gradients_full(dL, X, B)
        th = _theta(p)
        for i in range(th.size):
            h = 1e-6 * th[i]
            tp, tm = th.copy(), th.copy()
            tp[i] += h
            tm[i] -= h
            fp = np.sum(dL * po.make_part(_set_theta(p, tp))[0].K(X, B))
            fm = np.sum(dL * po.make_part(_set_theta(p, tm))[0].K(X, B))
            assert abs((fp - fm) / (2 * h) - g[i]) <= 1e-6 * max(1.0, abs(g[i])), (i, g[i], (fp - fm) / (2 * h))


# ---------------------------------------------------------------------------------------------------------------------
# the mirror's host logic on a fake engine
# ---------------------------------------------------------------------------------------------------------------------
class FakeEngine(object):
    """test double of gpy_b200._ffi.Engine for the composite evaluation: numbers from the oracle."""

    def __init__(self, device=0):
        self.calls, self.descs = [], []

    def set_data(self, X, Y):
        self.calls.append("set_data")
        self.X, self.Y = np.array(X), np.array(Y)
        self.N, self.P = self.Y.shape

    def exact_eval_multi(self, parts, noise, jitter=1e-8, max_tries=5):
        self.calls.append("exact_eval_multi")
        self.descs.append(parts)
        dicts = []
        for d in parts:
            q = dict(kind=d[0], ARD=d[1], term=d[2], dims=d[3], variance=d[4], lengthscale=d[5])
            if len(d) > 6:
                q.update(d[6])
            dicts.append(q)
        lml, g, self.res = po.composite_eval(self.X, self.Y, dicts, noise)
        return lml, g, 0.0

    def exact_eval(self, *a, **k):
        self.calls.append("exact_eval")
        raise AssertionError("a new kind must not take the single-kernel evaluation")

    exact_eval_het = exact_eval


def _mirror_composite():
    import gpy_b200
    return gpy_b200.Add([gpy_b200.Prod([gpy_b200.RBF(1, variance=2.0, lengthscale=9.0),
                                        gpy_b200.StdPeriodic(2, variance=1.1, period=[1.0, 2.0], lengthscale=1.3, ARD1=True,
                                                             active_dims=[0, 1])]),
                         gpy_b200.RatQuad(2, variance=0.5, lengthscale=[1.2, 0.7], power=0.8, ARD=True, active_dims=[1, 2]),
                         gpy_b200.White(1, variance=0.05)])


def test_parameter_order_and_gradient_scatter():
    import gpy_b200
    rng = np.random.default_rng(2)
    X = rng.uniform(0, 5, (60, 3))
    Y = np.sin(X[:, :1]) + 0.1 * rng.standard_normal((60, 1))
    eng = FakeEngine()
    m = gpy_b200.GPRegression(X, Y, _mirror_composite(), noise_var=0.02, engine=eng)
    assert eng.calls == ["set_data", "exact_eval_multi"]
    names = [p.name for p in m.flattened_parameters()]
    assert names == ["variance", "lengthscale", "variance", "period", "lengthscale", "variance", "lengthscale", "power",
                     "variance", "variance"]
    desc = eng.descs[-1]
    assert [d[0] for d in desc] == ["rbf", "stdperiodic", "ratquad", "white"]
    assert desc[1][6]["ARD_period"] is True and desc[1][3] == [0, 1] and desc[2][6] == {"power": 0.8}
    lml, g, _ = po.composite_eval(X, Y, [dict(kind="rbf", term=0, dims=[0], variance=2.0, lengthscale=9.0),
                                         dict(kind="stdperiodic", term=0, dims=[0, 1], variance=1.1, period=[1.0, 2.0],
                                              lengthscale=1.3, ARD_period=True),
                                         dict(kind="ratquad", term=1, dims=[1, 2], variance=0.5, lengthscale=[1.2, 0.7],
                                              power=0.8, ARD=True),
                                         dict(kind="white", term=2, variance=0.05)], 0.02)
    assert m.log_likelihood() == lml
    np.testing.assert_array_equal(m.gradient, g)
    per = m.kern.parts[0].parts[1]
    np.testing.assert_array_equal(per.period.gradient, g[3:5])
    np.testing.assert_array_equal(m.kern.parts[1].power.gradient, g[9:10])


@pytest.mark.parametrize("which", ["ratquad", "stdperiodic"])
def test_a_lone_new_leaf_is_one_composite_call(which):
    import gpy_b200
    rng = np.random.default_rng(3)
    X = rng.uniform(0, 5, (50, 2))
    Y = np.sin(X[:, :1])
    k = gpy_b200.RatQuad(2, power=1.5) if which == "ratquad" else gpy_b200.StdPeriodic(2, period=2.0, ARD2=True)
    eng = FakeEngine()
    m = gpy_b200.GPRegression(X, Y, k, noise_var=0.1, engine=eng)
    assert eng.calls == ["set_data", "exact_eval_multi"]
    assert len(eng.descs[-1]) == 1 and eng.descs[-1][0][0] == which
    assert m.gradient.size == (4 if which == "ratquad" else 5)
    with pytest.raises(NotImplementedError):
        k.gradients_X(np.ones((50, 50)), X)


@pytest.mark.parametrize("which", ["ratquad", "stdperiodic"])
def test_sparse_model_with_a_new_leaf_raises(which):
    import gpy_b200
    rng = np.random.default_rng(4)
    X = rng.uniform(0, 5, (40, 1))
    k = gpy_b200.RatQuad(1) if which == "ratquad" else gpy_b200.StdPeriodic(1)
    with pytest.raises(NotImplementedError, match="sparse"):
        gpy_b200.SparseGPRegression(X, np.sin(X), kernel=k, Z=X[:5].copy(), engine=FakeEngine())


def test_abi_exports():
    from gpy_b200 import _ffi
    for name in ("gpx_kern_part_K", "gpx_kern_part_grad_full"):
        assert name in _ffi.EXPORTS
    assert _ffi.KIND["ratquad"] == 6 and _ffi.KIND["stdperiodic"] == 7
    assert [f[0] for f in _ffi.GpxKernPart._fields_][-3:] == ["power", "ard_period", "period"]
    if os.path.exists(_ffi.LIB_PATH):
        L = _ffi.lib()
        assert hasattr(L, "gpx_kern_part_K") and hasattr(L, "gpx_kern_part_grad_full")
