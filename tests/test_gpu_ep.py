"""Expectation propagation on the device (gpx_ep_*, gpy_b200.EP): the reference's fixtures, the block edges against the
blocked restatement, the posterior's consumers, gradients and optimisation through GPClassification, repeatability,
context reuse and the rejections."""
import ctypes
import glob
import os

import numpy as np
import pytest

import ep_oracle as eo
from test_gpu_laplace import mirror_kernel

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = sorted(glob.glob(os.path.join(HERE, "golden", "ep", "*.npz")))
# measured on an H100 80GB HBM3 against the reference's fixtures (N <= 333): LML <= 5.3e-15 relative, sites, cavities,
# kernel gradients, predictions and Wi <= 2.0e-14 (the cavity precisions, largest); N = 4096 against the blocked
# restatement: LML 9.2e-14, sites 2.8e-14. The bars leave a factor of about 5 over the largest of these
LML_BAR = 5e-13
BAR = 2e-13


def _B():
    import gpy_b200
    return gpy_b200


def _rel(a, b):
    b = np.asarray(b, dtype=np.float64)
    return float(np.abs(np.asarray(a) - b).max() / max(1.0, np.abs(b).max())) if b.size else 0.0


def run_case(name, engine=None):
    """the case through the mirror, as tests/golden/make_ep.py runs the reference -> dict of its results"""
    B = _B()
    parts, N, seed, opts = eo.CASES[name]
    X, Y, Xnew = eo.case_data(name)
    kw = {k: opts[k] for k in ("eta", "delta", "max_iters", "parallel_updates", "ep_mode") if k in opts}
    inf = B.EP(engine=engine, **kw)
    kern = mirror_kernel(parts)
    lik = B.Bernoulli()
    np.random.seed(seed)
    sweeps = []
    post, lml, gd = inf.inference(kern, X, lik, Y)
    sweeps.append(inf.iterations)
    if opts.get("calls") == 2:
        post, lml, gd = inf.inference(kern, X, lik, Y)
        sweeps.append(inf.iterations)
    if "theta2" in opts:
        kern = mirror_kernel(eo.scaled_parts(parts, opts["theta2"]))
        post, lml, gd = inf.inference(kern, X, lik, Y)
    nxt = np.random.random()
    kern.update_gradients_full(gd["dL_dK"], X)
    mu, var = post._raw_predict(kern, Xnew, X)
    _, ga, cav, logZ = inf._ep_approximation
    return dict(lml=float(lml), grad=np.asarray(kern.gradient).copy(), tau_tilde=ga.tau, v_tilde=ga.v, cav_tau=cav.tau,
                cav_v=cav.v, log_Z_tilde=logZ, sweeps=np.array(sweeps), mu=mu, var=var, next_random=nxt, post=post,
                inf=inf, kern=kern)


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[:-4])
def test_fixture(path):
    """every fixture of the reference's own EP: equal sweep counts and RNG draw, and the values within the bars set from
    the measured deviations above (the blocked rank-128 updates and the DMMA products round differently from the
    reference's DSYR chain and LAPACK calls)"""
    name = os.path.basename(path)[:-4]
    z = np.load(path)
    r = run_case(name)
    np.testing.assert_array_equal(r["sweeps"], z["sweeps"])
    assert r["next_random"] == z["next_random"]
    print(name, "lml %.3e" % (abs(r["lml"] - z["lml"]) / max(1.0, abs(z["lml"]))),
          " ".join("%s %.3e" % (k, _rel(r[k], z[k])) for k in ("grad", "tau_tilde", "v_tilde", "cav_tau", "cav_v", "mu",
                                                                   "var")),
          "Wi %.3e" % _rel(r["post"].woodbury_inv, z["woodbury_inv"]) if "woodbury_inv" in z else "")
    assert abs(r["lml"] - z["lml"]) <= LML_BAR * max(1.0, abs(z["lml"]))
    for k, bar in (("grad", BAR), ("tau_tilde", BAR), ("v_tilde", BAR), ("cav_tau", BAR), ("cav_v", BAR),
                   ("mu", BAR), ("var", BAR)):
        assert _rel(r[k], z[k]) <= bar, (k, _rel(r[k], z[k]))
    if "woodbury_inv" in z:
        assert _rel(r["post"].woodbury_inv, z["woodbury_inv"]) <= BAR


def test_device_moments_at_the_final_cavity_match_the_host_restatement():
    B = _B()
    X, Y, _ = eo.case_data("rbf_ard_n150")
    eng = B.Engine()
    eng.set_data(np.ascontiguousarray(X), np.ascontiguousarray(Y))
    eng.ep_begin([("rbf", True, 0, [0, 1, 2], 1.4, [0.8, 1.3, 1.9])])
    eng.ep_start(parallel=True)
    N = X.shape[0]
    t, v, ct, cv, Z, mh, s2, _ = eng.ep_sweep(np.arange(N), np.zeros(N), np.zeros(N), parallel=True)
    t, v, ct, cv, Z, mh, s2, _ = eng.ep_sweep(np.arange(N), t, v, parallel=True)
    for i in range(N):
        zh, m, s = eo.moments(Y[i, 0], ct[i], cv[i])
        assert abs(Z[i] - zh) <= 1e-14 * max(1.0, abs(zh))
        assert abs(mh[i] - m) <= 1e-13 * max(1.0, abs(m))
        assert abs(s2[i] - s) <= 1e-13 * max(1.0, abs(s))


@pytest.mark.parametrize("N", [127, 128, 129, 255, 257, 700])
def test_block_edges_against_the_blocked_restatement(N):
    B = _B()
    rng = np.random.default_rng(N)
    X = rng.uniform(-2.0, 2.0, size=(N, 3))
    Y = (np.sin(1.3 * X[:, :1]) + 0.4 * rng.standard_normal((N, 1)) > 0).astype(np.float64)
    parts = eo._single("matern52", True)
    K = eo.CompositeOracle(parts).K(X)
    np.random.seed(N)
    st, it = eo.run_ep(K, Y[:, 0], blocked=True)
    ref = eo.marginal(K, st, parts, X)
    np.random.seed(N)
    inf = B.EP()
    kern = mirror_kernel(parts)
    _, lml, gd = inf.inference(kern, X, B.Bernoulli(), Y)
    assert inf.iterations == it
    assert abs(lml - ref["lml"]) <= LML_BAR * max(1.0, abs(ref["lml"]))
    ga = inf._ep_approximation[1]
    assert _rel(ga.tau, st["tt"]) <= BAR and _rel(ga.v, st["vt"]) <= BAR


def test_posterior_consumers_and_repeatability():
    B = _B()
    r1 = run_case("rbf_ard_n150")
    r2 = run_case("rbf_ard_n150")
    assert r1["lml"] == r2["lml"] and np.array_equal(r1["tau_tilde"], r2["tau_tilde"])   # bit-identical repeat
    X, Y, Xnew = eo.case_data("rbf_ard_n150")
    m = B.GPClassification(X, Y, kernel=mirror_kernel(eo.CASES["rbf_ard_n150"][0]))
    mu, var = m._raw_predict(Xnew)
    Wi = m.posterior.woodbury_inv
    Kx = m.kern.K(X, Xnew)
    assert _rel(var[:, 0], m.kern.Kdiag(Xnew) - (Wi.dot(Kx) * Kx).sum(0)) <= 1e-10
    p, _ = m.predict(Xnew)
    assert np.all((p > 0) & (p < 1))
    dmu, dvar = m.predictive_gradients(Xnew)
    assert np.all(np.isfinite(dmu)) and np.all(np.isfinite(dvar))
    C = m.posterior_covariance_between_points(Xnew[:5], Xnew[:5], include_likelihood=False)
    assert _rel(np.diag(C), var[:5, 0]) <= 1e-9
    f = m.posterior_samples_f(Xnew[:4], size=3)
    assert np.all(np.isfinite(f))


def test_checkgrad_and_optimize_alternated():
    B = _B()
    X, Y, _ = eo.case_data("rbf_iso_n60")
    np.random.seed(3)
    m = B.GPClassification(X, Y, kernel=B.RBF(3, variance=1.2, lengthscale=0.9))
    assert m.checkgrad()
    start = float(m.log_likelihood())
    m.optimize(max_iters=30)
    assert float(m.log_likelihood()) >= start
    p, _ = m.predict(X[:10])
    assert np.all((p > 0) & (p < 1))


def test_exact_ep_laplace_exact_on_one_context_is_bit_identical_to_fresh_contexts():
    B = _B()
    X, Y, _ = eo.case_data("rbf_ard_n150")
    Yr = np.sin(X[:, :1])
    shared = B.Engine()

    def ep(eng):
        np.random.seed(5)
        inf = B.EP(engine=eng)
        _, lml, _ = inf.inference(B.RBF(3, variance=1.1, lengthscale=0.9), X, B.Bernoulli(), Y)
        return lml

    def lap(eng):
        _, lml, _ = B.Laplace(engine=eng).inference(B.RBF(3, variance=1.1, lengthscale=0.9), X, B.Bernoulli(), Y)
        return lml

    def exact(eng):
        m = B.GPRegression(X, Yr, kernel=B.RBF(3), engine=eng)
        return float(m.log_likelihood())

    got = [exact(shared), ep(shared), lap(shared), exact(shared)]
    want = [exact(B.Engine()), ep(B.Engine()), lap(B.Engine()), exact(B.Engine())]
    assert got == want


def test_rejections():
    B = _B()
    from gpy_b200 import _ffi
    L = _ffi.lib()
    h = ctypes.c_void_p()
    assert L.gpx_create(0, ctypes.byref(h)) == 0
    try:
        parts = (_ffi.GpxKernPart * 1)()
        keep = []
        _ffi._fill_part(parts[0], ("rbf", False, 0, [0, 1], 1.0, 1.0), keep)
        N = 40
        X = np.random.default_rng(0).uniform(size=(N, 2))
        d = ctypes.c_double()
        p = np.zeros(N).ctypes.data_as(_ffi._dp)
        order = np.arange(N, dtype=np.int64)
        op = order.ctypes.data_as(ctypes.POINTER(ctypes.c_int64))
        assert L.gpx_ep_begin(h, parts, 1) == -2                                    # no data
        Y2 = np.zeros((N, 2))
        assert L.gpx_set_data(h, X.ctypes.data_as(_ffi._dp), N, 2, Y2.ctypes.data_as(_ffi._dp), 2) == 0
        assert L.gpx_ep_begin(h, parts, 1) == -2                                    # P = 2
        Ybad = np.full((N, 1), 0.5)
        assert L.gpx_set_data(h, X.ctypes.data_as(_ffi._dp), N, 2, Ybad.ctypes.data_as(_ffi._dp), 1) == 0
        assert L.gpx_ep_begin(h, parts, 1) == -2                                    # labels
        Y = (X[:, :1] > 0.5).astype(np.float64)
        assert L.gpx_set_data(h, X.ctypes.data_as(_ffi._dp), N, 2, Y.ctypes.data_as(_ffi._dp), 1) == 0
        assert L.gpx_ep_start(h, None, None, 0, 0, 5, ctypes.byref(d)) == -2        # no begin
        assert L.gpx_ep_finish(h, p, p, 5, ctypes.byref(d), ctypes.byref(d), p, p, ctypes.byref(d)) == -2
        assert L.gpx_ep_begin(h, None, 1) == -2
        assert L.gpx_ep_begin(h, parts, 1) == 0
        assert L.gpx_ep_sweep(h, op, 1.0, 1.0, 0, 5, p, p, p, p, p, p, p, ctypes.byref(d)) == -2   # no start
        assert L.gpx_ep_start(h, None, None, 1, 0, 5, ctypes.byref(d)) == -2        # warm without sites
        assert L.gpx_ep_start(h, None, None, 0, 0, 5, ctypes.byref(d)) == 0
        assert L.gpx_ep_sweep(h, op, 1.0, 1.0, 1, 5, p, p, p, p, p, p, p, ctypes.byref(d)) == -2   # parallel differs
        bad = order.copy()
        bad[3] = 4
        assert L.gpx_ep_sweep(h, bad.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)), 1.0, 1.0, 0, 5, p, p, p, p, p, p,
                              p, ctypes.byref(d)) == -2                             # not a permutation
        assert L.gpx_ep_sweep(h, op, 1.0, 1.0, 0, 5, None, p, p, p, p, p, p, ctypes.byref(d)) == -2
        assert L.gpx_ep_finish(h, p, p, 5, None, ctypes.byref(d), p, p, ctypes.byref(d)) == -2
    finally:
        L.gpx_destroy(h)


def _sweep_launches(N):
    from test_gpu_laplace import _sweep_launches as f
    return f(N)


@pytest.mark.parametrize("N", [300, 700, 1300])
def test_launch_counts(N):
    """beyond F, the factor sweep of B (once per attempt of the ladder): begin 3, cold start 1, a sequential sweep 3 per
    block of 128 sites + 13, a parallel sweep 15, a warm start 14 and the finish 11 + nparts"""
    B = _B()
    rng = np.random.default_rng(N)
    X = rng.uniform(-2, 2, size=(N, 3))
    Y = (X[:, :1] > 0).astype(float)
    eng = B.Engine()
    eng.set_data(X, Y)
    eng.ep_begin([("rbf", True, 0, [0, 1, 2], 1.0, [1.0, 1.2, 0.8]), ("bias", False, 1, [], 0.3, None)])
    assert eng.stats()["launches"] == 3
    F = _sweep_launches(N)
    nblk = (N + 127) // 128
    for parallel, per_sweep in ((False, 3 * nblk + 13), (True, 15)):
        eng.ep_start(parallel=parallel)
        assert eng.stats()["launches"] == 1
        t, v = np.zeros(N), np.zeros(N)
        for k in range(2):
            t, v = eng.ep_sweep(np.random.RandomState(k).permutation(N), t, v, parallel=parallel)[:2]
            assert eng.stats()["launches"] - F * eng.stats()["tries"] == per_sweep
        eng.ep_start(t, v, parallel=parallel)
        assert eng.stats()["launches"] - F * eng.stats()["tries"] == 14
    eng.ep_finish(t, v)
    assert eng.stats()["launches"] - F * eng.stats()["tries"] == 11 + 2
    eng.close()


def test_n4096_matches_the_blocked_restatement():
    """32 blocks per sweep: equal sweeps, the LML and the sites within the fixtures' bars"""
    B = _B()
    N = 4096
    rng = np.random.default_rng(7)
    X = rng.uniform(-2.0, 2.0, size=(N, 3))
    Y = (np.sin(1.3 * X[:, :1]) + 0.6 * X[:, 1:2] + 0.4 * rng.standard_normal((N, 1)) > 0).astype(np.float64)
    parts = eo._single("rbf", True)
    K = eo.CompositeOracle(parts).K(X)
    np.random.seed(11)
    st, it = eo.run_ep(K, Y[:, 0], blocked=True)
    ref = eo.marginal(K, st, parts, X)
    np.random.seed(11)
    inf = B.EP()
    _, lml, _ = inf.inference(mirror_kernel(parts), X, B.Bernoulli(), Y)
    assert inf.iterations == it
    print("N=4096 lml rel %.3e tau %.3e v %.3e" % (abs(lml - ref["lml"]) / abs(ref["lml"]),
                                                    _rel(inf._ep_approximation[1].tau, st["tt"]),
                                                    _rel(inf._ep_approximation[1].v, st["vt"])))
    assert abs(lml - ref["lml"]) <= LML_BAR * max(1.0, abs(ref["lml"]))
