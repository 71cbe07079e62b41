"""Sparse EP on the device (gpx_epdtc_*, gpy_b200.EPDTC, gpy_b200.SparseGPClassification): the reference's fixtures, block
and tile edges against the blocked M-space restatement, N = 8192 / M = 512, the posterior's consumers, gradients and
optimisation, repeatability, context reuse, launch counts and the rejections."""
import ctypes
import glob
import os

import numpy as np
import pytest

import epdtc_oracle as eo
from sparse_composite_oracle import CompositeOracle
from test_gpu_laplace import mirror_kernel

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = sorted(glob.glob(os.path.join(HERE, "golden", "epdtc", "*.npz")))
# measured on an H100 80GB HBM3 against the reference's fixtures with cond(Kmm) < 1e6: sites and posterior mu / Sigma_diag
# <= 4.3e-13, the bound <= 5.0e-15, kernel gradients, dL/dZ and predictions <= 1.1e-12 (relative to the largest entry).
# With cond(Kmm) = 2.0e7 (N = 1300, M = 129) the largest deviation is 7.6e-10, at 2.3e10 (M = 300) 4.5e-8, and with the
# ladder (repeated inducing points) 3.6e-9: the M-space form carries A = LLT^-1, whose rounding grows with cond(Kmm),
# where the reference refactors LLT. The bars leave a factor of about 5 over the measured values; the ill-conditioned
# ones are min(1e-6, cond(Kmm) eps)
SITE_BAR = 2e-12
LML_BAR = 1e-13
GRAD_BAR = 5e-12


def ill_bar(cond):
    return min(1e-6, cond * np.finfo(float).eps)


def _B():
    import gpy_b200
    return gpy_b200


def _rel(a, b):
    b = np.asarray(b, dtype=np.float64)
    return float(np.abs(np.asarray(a) - b).max() / max(1.0, np.abs(b).max())) if b.size else 0.0


def _kgrad(gd):
    if "part_grads" in gd:
        return np.concatenate([np.atleast_1d(g) for g in gd["part_grads"]])
    return np.concatenate([np.atleast_1d(gd["dvariance"]), np.atleast_1d(gd["dlengthscale"])])


def _mirror(parts):
    """mirror_kernel with a White part added as its own term"""
    B = _B()
    white = [p for p in parts if p["kind"] == "white"]
    k = mirror_kernel([p for p in parts if p["kind"] != "white"])
    return B.Add([k] + [B.White(3, variance=p["variance"]) for p in white]) if white else k


def run_case(name, engine=None):
    """the case through the mirror, as tests/golden/make_epdtc.py runs the reference"""
    B = _B()
    parts, N, M, seed, opts = eo.CASES[name]
    X, Y, Z, Xnew = eo.case_data(name)
    kw = {k: opts[k] for k in ("eta", "delta", "max_iters", "parallel_updates", "ep_mode") if k in opts}
    inf = B.EPDTC(engine=engine, **kw)
    kern = _mirror(parts)
    lik = B.Bernoulli()
    np.random.seed(seed)
    sweeps = []
    post, lml, gd = inf.inference(kern, X, Z, lik, Y)
    sweeps.append(inf.iterations)
    if opts.get("calls") == 2:
        post, lml, gd = inf.inference(kern, X, Z, lik, Y)
        sweeps.append(inf.iterations)
    if "theta2" in opts:
        kern = _mirror(eo.scaled_parts(parts, opts["theta2"]))
        post, lml, gd = inf.inference(kern, X, Z, lik, Y)
    if "z2" in opts:
        Z = Z + opts["z2"]
        post, lml, gd = inf.inference(kern, X, Z, lik, Y)
    nxt = np.random.random()
    mu, var = post._raw_predict(kern, Xnew, Z)
    pp, ga, logZ = inf._ep_approximation
    return dict(lml=float(lml), grad=_kgrad(gd), dZ=gd["dZ"], tau_tilde=ga.tau, v_tilde=ga.v, post_mu=pp.mu,
                post_sd=pp.Sigma_diag, log_Z_tilde=logZ, sweeps=np.array(sweeps), mu=mu, var=var, next_random=nxt,
                post=post, inf=inf, kern=kern)


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[:-4])
def test_fixture(path):
    name = os.path.basename(path)[:-4]
    z = np.load(path)
    r = run_case(name)
    np.testing.assert_array_equal(r["sweeps"], z["sweeps"])
    assert r["next_random"] == z["next_random"]
    devs = {k: _rel(r[k], z[k]) for k in ("tau_tilde", "v_tilde", "post_mu", "post_sd", "grad", "dZ", "mu", "var")}
    devs["lml"] = abs(r["lml"] - z["lml"]) / max(1.0, abs(z["lml"]))
    print(name, "cond %.1e" % z["cond_Kmm"], " ".join("%s %.2e" % kv for kv in devs.items()))
    ill = "ladder" in name or float(z["cond_Kmm"]) >= 1e6
    for k, v in devs.items():
        bar = ill_bar(float(z["cond_Kmm"])) if ill else (SITE_BAR if k in ("tau_tilde", "v_tilde", "post_mu", "post_sd")
                                   else LML_BAR if k == "lml" else GRAD_BAR)
        assert v <= bar, (k, v)


def _problem(N, M, seed=3, D=3):
    rng = np.random.default_rng(seed)
    X = rng.uniform(-2.0, 2.0, size=(N, D))
    Y = (np.sin(1.3 * X[:, :1]) + 0.6 * X[:, 1:2] + 0.4 * rng.standard_normal((N, 1)) > 0).astype(np.float64)
    Z = rng.uniform(-2.0, 2.0, size=(M, D)) * (1.0 + M / 64.0) ** (1.0 / D)   # spread: Kmm stays well conditioned
    return X, Y, Z


def _device_vs_blocked(N, M, max_iters, bar):
    B = _B()
    # short lengthscales keep Kmm well conditioned; one inducing point needs a long one, or nearly every site sits at the
    # eps clip where the held diagonal is rounding
    ls = [0.4, 0.5, 0.6] if M > 1 else [2.0, 2.5, 3.0]
    parts = [dict(kind="rbf", term=0, dims=[0, 1, 2], variance=1.4, lengthscale=ls, ARD=True)]
    X, Y, Z = _problem(N, M)
    inf = B.EPDTC(max_iters=max_iters, epsilon=0.0)   # exactly max_iters sweeps on both sides
    np.random.seed(11)
    inf.inference(mirror_kernel(parts), X, Z, B.Bernoulli(), Y)
    pp, ga, logZ = inf._ep_approximation
    kern = CompositeOracle(parts)
    np.random.seed(11)
    st, it = eo.run_epdtc(kern.K(Z), kern.K(Z, X), Y[:, 0], max_iters=max_iters, epsilon=0.0,
                           blocked=True)
    assert it == inf.iterations
    for a, b in ((ga.tau, st["tt"]), (ga.v, st["vt"]), (pp.mu, st["mu"]), (pp.Sigma_diag, st["sd"])):
        assert _rel(a, b) <= bar, _rel(a, b)
    return _rel(ga.tau, st["tt"])


@pytest.mark.parametrize("N,M", [(127, 1), (128, 127), (129, 128), (300, 129), (700, 300), (257, 129)])
def test_block_and_tile_edges(N, M):
    d = _device_vs_blocked(N, M, 3, 1e-9)
    print("N %d M %d sites %.2e" % (N, M, d))


def test_n8192_m512_against_blocked():
    d = _device_vs_blocked(8192, 512, 2, 1e-8)
    print("N 8192 M 512 sites %.2e" % d)


def test_device_drift_n8192_m512():
    """diag(Knm A Kmn) of the device's downdated A after the last of 64 blocks against the recompute's diagonal at the
    same sites (option "epdtc_drift"), on the second sweep of a run. The NumPy form of the same measurement gives 5.7e-12
    of the diagonal's scale at this cond(Kmm) (test_epdtc_cpu)"""
    B = _B()
    rng = np.random.default_rng(7)
    N, M = 8192, 512
    X = rng.uniform(-2.0, 2.0, size=(N, 3))
    Z = rng.uniform(-2.0, 2.0, size=(M, 3))
    Y = (np.sin(1.3 * X[:, :1]) + 0.6 * X[:, 1:2] > 0).astype(np.float64)
    parts = [("rbf", 1, 0, [0, 1, 2], 1.0, np.array([0.4, 0.4, 0.4]))]
    eng = B.Engine()
    eng.sparse_set_data(X, Y)
    outs = []
    for opt in (0, 1):
        eng.set_option("epdtc_drift", opt)
        eng.epdtc_begin(parts, Z)
        eng.epdtc_start()
        r = eng.epdtc_sweep(np.random.default_rng(1).permutation(N), np.zeros(N), np.zeros(N))
        r = eng.epdtc_sweep(np.random.default_rng(2).permutation(N), r[0], r[1])
        outs.append(r)
    eng.set_option("epdtc_drift", 0)
    np.testing.assert_array_equal(outs[0][0], outs[1][0])      # the option changes only what sigma_diag reports
    d = np.max(np.abs(outs[1][9] - outs[0][9])) / np.max(outs[0][9])
    print("device drift N 8192 M 512: %.2e" % d)
    assert d <= 1e-10


def test_repeat_is_bit_identical_and_launches_follow_blocks():
    B = _B()
    X, Y, Z = _problem(700, 129)
    eng = B.Engine()
    eng.sparse_set_data(X, Y)
    parts = [("rbf", 1, 0, [0, 1, 2], 1.3, np.array([0.8, 1.1, 1.6]))]
    outs, counts = [], []
    for N in (700, 700):
        eng.epdtc_begin(parts, Z)
        eng.epdtc_start()
        l0 = eng.total_launches()
        r = eng.epdtc_sweep(np.arange(N), np.zeros(N), np.zeros(N))
        counts.append(eng.total_launches() - l0)
        outs.append(np.concatenate([r[0], r[1], r[8], r[9]]))
    np.testing.assert_array_equal(outs[0], outs[1])
    X2, Y2, _ = _problem(300, 129)
    eng.sparse_set_data(X2, Y2)
    eng.epdtc_begin(parts, Z)
    eng.epdtc_start()
    l0 = eng.total_launches()
    eng.epdtc_sweep(np.arange(300), np.zeros(300), np.zeros(300))
    c300 = eng.total_launches() - l0
    per_block = (counts[0] - c300) // (6 - 3)
    assert counts[0] - c300 == per_block * 3 and per_block == 9, (counts[0], c300)


def test_posterior_consumers_and_sparse_get():
    B = _B()
    X, Y, Z = _problem(300, 40)
    m = B.SparseGPClassification(X, Y, kernel=B.RBF(3, lengthscale=np.array([0.9, 1.2, 1.5]), ARD=True), Z=Z)
    post = m.posterior
    Kmm, Lm, W, wv = post.K, post.K_chol, post.woodbury_inv, post.woodbury_vector
    np.testing.assert_allclose(Kmm, Lm @ Lm.T, rtol=0, atol=1e-12)
    Xn = np.random.default_rng(4).uniform(-2, 2, size=(17, 3))
    Kx = m.kern.K(Z, Xn)
    mu, var = m.predict(Xn, include_likelihood=False)
    np.testing.assert_allclose(mu, Kx.T @ wv, rtol=0, atol=1e-10)
    np.testing.assert_allclose(var[:, 0], np.maximum(m.kern.Kdiag(Xn) - np.sum((W @ Kx) * Kx, 0), 1e-15), atol=1e-10)
    p, _ = m.predict(Xn)
    assert np.all((p > 0) & (p < 1))
    dmu, dvar = m.predictive_gradients(Xn)
    assert dmu.shape[0] == 17 and np.all(np.isfinite(dmu)) and np.all(np.isfinite(dvar))
    f = m.posterior_samples_f(Xn, size=4)
    assert f.shape == (17, 1, 4) and np.all(np.isfinite(f))


def test_checkgrad_and_optimize():
    B = _B()
    X, Y, Z = _problem(200, 12)
    np.random.seed(0)
    m = B.SparseGPClassification(X, Y, Z=Z)   # alternated: the sites stay fixed, the bound is smooth in theta and Z
    assert m.checkgrad(step=1e-5, tolerance=1e-3)
    m2 = B.SparseGPClassification(X, Y, Z=Z)
    f0 = m2.objective_function()
    m2.optimize(max_iters=30)
    assert m2.objective_function() <= f0


def test_one_context_matches_fresh_contexts():
    B = _B()
    X, Y, Z = _problem(300, 50)
    eng = B.Engine()
    kern = lambda: B.RBF(3, variance=1.2, lengthscale=np.array([0.9, 1.2, 1.5]), ARD=True)  # noqa: E731
    Yr = np.sin(X[:, :1])
    m_exact = B.GPRegression(X, Yr, kern(), engine=eng)
    np.random.seed(5)
    r1 = B.EPDTC(engine=eng).inference(kern(), X, Z, B.Bernoulli(), Y)[1]
    m_sp = B.SparseGPRegression(X, Yr, kern(), Z=Z, engine=eng)
    r2 = B.EP(engine=eng).inference(kern(), X, B.Bernoulli(), Y)[1]
    np.random.seed(5)
    f1 = B.EPDTC().inference(kern(), X, Z, B.Bernoulli(), Y)[1]
    f_sp = B.SparseGPRegression(X, Yr, kern(), Z=Z).log_likelihood()
    f2 = B.EP().inference(kern(), X, B.Bernoulli(), Y)[1]
    f_exact = B.GPRegression(X, Yr, kern()).log_likelihood()
    assert r1 == f1 and m_sp.log_likelihood() == f_sp
    assert abs(r2 - f2) <= 1e-12 * abs(f2)
    assert m_exact.log_likelihood() == f_exact


def test_rejections():
    B = _B()
    L = B._ffi.lib()
    X, Y, Z = _problem(130, 5)
    eng = B.Engine()
    h = eng._h
    from gpy_b200._ffi import GpxKernPart, _fill_part, _ptr
    arr = (GpxKernPart * 1)()
    keep = []
    _fill_part(arr[0], ("rbf", 0, 0, [0, 1, 2], 1.0, 1.0), keep, 0)
    Zc = np.ascontiguousarray(Z)
    jit = ctypes.c_double()
    assert L.gpx_epdtc_begin(h, arr, 1, _ptr(Zc), 5) == -2                # no data
    eng.sparse_set_data(X, Y)
    assert L.gpx_epdtc_start(h, None, None, 0, 0, 5, ctypes.byref(jit), None, None) == -2   # before begin
    assert L.gpx_epdtc_begin(h, arr, 1, None, 5) == -2                    # null Z
    assert L.gpx_epdtc_begin(h, arr, 1, _ptr(Zc), 0) == -2                # M < 1
    eng2 = B.Engine()
    eng2.sparse_set_data(X, np.hstack([Y, Y]))
    assert L.gpx_epdtc_begin(eng2._h, arr, 1, _ptr(Zc), 5) == -2          # P = 2
    eng3 = B.Engine()
    eng3.sparse_set_data(X, Y + 2.0)
    assert L.gpx_epdtc_begin(eng3._h, arr, 1, _ptr(Zc), 5) == -2          # labels
    assert L.gpx_epdtc_begin(h, arr, 1, _ptr(Zc), 5) == 0
    t = np.zeros(130)
    o = [np.zeros(130) for _ in range(7)]
    order = np.arange(130, dtype=np.int64)
    op = order.ctypes.data_as(ctypes.POINTER(ctypes.c_int64))
    assert L.gpx_epdtc_sweep(h, op, 1.0, 1.0, 0, 5, *[_ptr(a) for a in o], ctypes.byref(jit), None, None) == -2
    with pytest.raises(NotImplementedError):
        B.EPDTC().inference(B.RatQuad(3), X, Z, B.Bernoulli(), Y)
    with pytest.raises(ValueError):
        B.EPDTC().inference(B.RBF(3), X, Z, B.Bernoulli(), Y, mean_function=object())
