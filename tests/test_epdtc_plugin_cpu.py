"""Sparse EP without a GPU: the mirror's host logic (gpy_b200.EPDTC) and the plugin's B.EPDTC over a host engine that
restates every gpx_epdtc_* entry (the blocked M-space sweep of tests/epdtc_oracle.py, the marginal by the reference's own
VarDTC), against the reference's fixtures and the reference's own EPDTC + SparseGP."""
import os
import types

import numpy as np
import pytest

import epdtc_oracle as eo

HERE = os.path.dirname(os.path.abspath(__file__))
# the host engine runs the blocked restatement, whose rounding differs from the reference's chain (test_epdtc_cpu)
BAR = 1e-9


def _reference():
    try:
        from oracle import ref_gpy
        S = ref_gpy.load_sparse_models()
    except ImportError:
        pytest.skip("reference tree not present")
    from epdtc_reference import load_reference_epdtc
    EPDTC, Bern, ObsAr = load_reference_epdtc()
    return ref_gpy, S, EPDTC, Bern, ObsAr


class HostEPDTCEngine(object):
    """every sparse EP entry on the host"""

    def __init__(self, device=0):
        self.calls, self.sparse_serial = [], 0

    def sparse_set_data(self, X, Y):
        self.calls.append(("set_data",))
        self.X, self.y = np.array(X, dtype=np.float64), np.array(Y, dtype=np.float64)[:, 0]
        self.sN, self.sD, self.sP = X.shape[0], X.shape[1], 1

    def epdtc_begin(self, parts, Z):
        from test_laplace_cpu import _parts_of
        self.calls.append(("begin",))
        self.parts = _parts_of(parts)
        kern = eo.CompositeOracle(self.parts)
        self.Z = np.array(Z, dtype=np.float64)
        self.Kmm, self.Kmn = kern.K(self.Z), kern.K(self.Z, self.X)
        self.sM = self.Z.shape[0]
        return 0

    def epdtc_start(self, tau_tilde=None, v_tilde=None, parallel=False, max_tries=5):
        self.calls.append(("start", tau_tilde is not None))
        if tau_tilde is None:
            Lm = eo.jitchol(self.Kmm)
            Vm = np.linalg.solve(Lm, self.Kmn)
            self.LLT, self.mu, self.sd = self.Kmm.copy(), np.zeros(self.sN), np.sum(Vm * Vm, 0) + 1e-8
        else:
            self.mu, sd, self.LLT = eo.recompute(self.Kmm, self.Kmn, np.asarray(tau_tilde), np.asarray(v_tilde))
            self.sd = sd + 1e-8
        return 0.0, self.mu.copy(), self.sd.copy()

    def epdtc_sweep(self, order, tau_tilde, v_tilde, eta=1., delta=1., parallel=False, max_tries=5):
        self.calls.append(("sweep", np.array(order)))
        st = {k: np.empty(self.sN) for k in ("ct", "cv", "Z", "mh", "s2")}
        st["tt"], st["vt"] = np.array(tau_tilde, dtype=float), np.array(v_tilde, dtype=float)
        eo.sweep(self.Kmn, self.LLT, self.mu, self.sd, st, self.y, np.asarray(order), eta, delta, parallel, True)
        self.mu, sd, self.LLT = eo.recompute(self.Kmm, self.Kmn, st["tt"], st["vt"])
        self.sd = np.maximum(sd, eo.EPS)
        return (st["tt"], st["vt"], st["ct"], st["cv"], st["Z"], st["mh"], st["s2"], 0.0, self.mu.copy(),
                self.sd.copy())

    def epdtc_finish(self, tau_tilde, v_tilde, max_tries=5):
        """VarDTC at Y = v~ / tau~, precision tau~ and Lm = jitchol(Kmm) by the reference's own VarDTC and kernels"""
        import sys
        sys.path.insert(0, os.path.join(HERE, "golden"))
        import make_laplace as ml
        ref_gpy, _, _, Bern, _ = _reference()
        self.calls.append(("finish",))
        kern = ml.reference_kernel(self.parts, self.sD)
        t, v = np.asarray(tau_tilde), np.asarray(v_tilde)
        _, lml, gd = ref_gpy.load().VarDTC().inference(kern, self.X, self.Z, Bern(), (v / t)[:, None], precision=t,
                                                        Lm=eo.jitchol(self.Kmm))
        kern.update_gradients_diag(gd["dL_dKdiag"], self.X)
        g = kern.gradient.copy()
        kern.update_gradients_full(gd["dL_dKnm"], self.X, self.Z)
        g += kern.gradient
        kern.update_gradients_full(gd["dL_dKmm"], self.Z, None)
        g += kern.gradient
        dZ = kern.gradients_X(gd["dL_dKmm"], self.Z) + kern.gradients_X(gd["dL_dKnm"].T, self.Z, self.X)
        self.sparse_serial += 1
        return float(np.squeeze(lml)), np.asarray(g, dtype=np.float64), np.asarray(dZ), 0.0


def _mirror_case(name, eng):
    import gpy_b200 as B
    from test_gpu_laplace import mirror_kernel
    parts, N, M, seed, opts = eo.CASES[name]
    X, Y, Z, Xnew = eo.case_data(name)
    kw = {k: opts[k] for k in ("eta", "delta", "max_iters", "parallel_updates", "ep_mode") if k in opts}
    inf = B.EPDTC(engine=eng, **kw)
    kern = mirror_kernel(parts)
    np.random.seed(seed)
    sweeps = []
    post, lml, gd = inf.inference(kern, X, Z, B.Bernoulli(), Y)
    sweeps.append(inf.iterations)
    if opts.get("calls") == 2:
        post, lml, gd = inf.inference(kern, X, Z, B.Bernoulli(), Y)
        sweeps.append(inf.iterations)
    if "theta2" in opts:
        post, lml, gd = inf.inference(mirror_kernel(eo.scaled_parts(parts, opts["theta2"])), X, Z, B.Bernoulli(), Y)
    if "z2" in opts:
        post, lml, gd = inf.inference(kern, X, Z + opts["z2"], B.Bernoulli(), Y)
    return inf, float(lml), gd, np.array(sweeps), np.random.random()


@pytest.mark.parametrize("name", ["rbf_iso_n60_m10", "rbf_ard_parallel_n150_m50", "matern52_iso_damped_n150_m50",
                                  "rbf_iso_maxiters2_n150_m50", "rbf_ard_nested_warm_n150_m50",
                                  "rbf_ard_alternated_theta_n150_m50", "rbf_ard_alternated_z_n150_m50",
                                  "rbf_ard_x_m52_bias_n150_m50", "rbf_iso_far_n150_m10"])
def test_mirror_host_logic_matches_the_reference(name):
    """one permutation per sweep in both update modes (numpy's generator ends in the reference's state), the stopping
    rule (equal sweep counts), the warm start of nested mode, the reuse of alternated mode and the 3-tuple"""
    _reference()
    z = np.load(os.path.join(HERE, "golden", "epdtc", name + ".npz"))
    eng = HostEPDTCEngine()
    inf, lml, gd, sweeps, nxt = _mirror_case(name, eng)
    np.testing.assert_array_equal(sweeps, z["sweeps"])
    assert nxt == z["next_random"]
    assert len(inf._ep_approximation) == 3
    pp, ga, logZ = inf._ep_approximation
    for a, b in ((ga.tau, z["tau_tilde"]), (ga.v, z["v_tilde"]), (pp.mu, z["post_mu"]), (pp.Sigma_diag, z["post_sd"])):
        assert np.max(np.abs(a - b)) <= BAR * max(1.0, np.max(np.abs(b)))
    assert abs(logZ - float(z["log_Z_tilde"])) <= BAR * abs(float(z["log_Z_tilde"]))
    assert abs(lml - float(z["lml"])) <= BAR * abs(float(z["lml"]))
    np.testing.assert_allclose(gd["dZ"], z["dZ"], rtol=0, atol=1e-7 * np.abs(z["dZ"]).max())
    names = [c[0] for c in eng.calls]
    starts = [c for c in eng.calls if c[0] == "start"]
    opts = eo.CASES[name][4]
    if opts.get("calls") == 2:                               # nested: the second run starts warm from ga_approx_old
        assert starts == [("start", False), ("start", True)]
    if "theta2" in opts or "z2" in opts:                     # alternated: the second call reuses the sites
        assert names[-2:] == ["begin", "finish"] and len(starts) == 1
    orders = [c[1] for c in eng.calls if c[0] == "sweep"]
    assert all(sorted(o) == list(range(eo.CASES[name][1])) for o in orders)


def test_mirror_always_reset_and_rejections():
    import gpy_b200 as B
    _reference()
    X, Y, Z, _ = eo.case_data("rbf_iso_n60_m10")
    eng = HostEPDTCEngine()
    inf = B.EPDTC(engine=eng, always_reset=True, ep_mode="nested")
    inf.inference(B.RBF(3), X, Z, B.Bernoulli(), Y)
    inf.inference(B.RBF(3), X, Z, B.Bernoulli(), Y)
    assert [c for c in eng.calls if c[0] == "start"] == [("start", False), ("start", False)]
    with pytest.raises(NotImplementedError):
        B.EPDTC(engine=eng).inference(B.RBF(3), X, Z, B.StudentT(), Y)
    with pytest.raises(ValueError, match="Mean function"):
        B.EPDTC(engine=eng).inference(B.RBF(3), X, Z, B.Bernoulli(), Y, mean_function=object())
    with pytest.raises(NotImplementedError):
        B.EPDTC(engine=eng).inference(B.RatQuad(3), X, Z, B.Bernoulli(), Y)
    with pytest.raises(NotImplementedError):
        B.EPDTC(engine=eng).inference(B.Add([B.RBF(3), B.StdPeriodic(3)]), X, Z, B.Bernoulli(), Y)
    with pytest.raises(ValueError, match="bad value for Bernoulli observation"):
        B.EPDTC(engine=eng).inference(B.RBF(3), X, Z, B.Bernoulli(), Y + 2.0)
    with pytest.raises(ValueError, match="ep_mode"):
        B.EPDTC(engine=eng, ep_mode="other").inference(B.RBF(3), X, Z, B.Bernoulli(), Y)
    n = len(eng.calls)
    assert all(c[0] != "begin" for c in eng.calls[n:])


def _plugin():
    ref_gpy, S, EPDTC, Bern, ObsAr = _reference()
    from gpy_b200 import gpy_plugin
    from test_periodic_ratquad_plugin_cpu import fake_ffi
    C = ref_gpy.load_combination()
    G = S.G
    f = fake_ffi()
    ffi = types.SimpleNamespace(kern_K=f.kern_K, kern_Kdiag=f.kern_Kdiag, kern_grad_full=f.kern_grad_full,
                                kern_part_K=f.kern_part_K, kern_part_grad_full=f.kern_part_grad_full,
                                Engine=HostEPDTCEngine)
    B = gpy_plugin.make(G.RBF, G.Exponential, G.Matern32, G.Matern52, G.ExactGaussianInference, Add=C.Add, Prod=C.Prod,
                        EPDTC=EPDTC, ffi=ffi)
    return S, C, G, B, EPDTC, Bern, ObsAr


@pytest.mark.parametrize("case", ["rbf_ard_n150_m50", "rbf_ard_x_m52_bias_n150_m50"])
def test_reference_sparse_gp_over_plugin_epdtc_matches_the_stock_pair(case):
    S, C, G, B, EPDTC, Bern, ObsAr = _plugin()
    import sys
    ref = sys.modules[EPDTC.__module__]
    parts, _, _, seed, _ = eo.CASES[case]
    X, Y, Z, _ = eo.case_data(case)

    def kern(ns):
        if len(parts) == 1:
            return ns.RBF(3, variance=parts[0]["variance"], lengthscale=parts[0]["lengthscale"], ARD=True)
        k = ns.RBF(3, variance=1.3, lengthscale=[0.9, 1.4, 2.1], ARD=True)
        m = ns.Matern52(2, variance=1.1, lengthscale=1.2, active_dims=[0, 1])
        prod, add = (B.Prod, B.Add) if ns is B else (C.Prod, C.Add)
        return add([prod([k, m]), C.Bias(3, variance=0.4)])

    np.random.seed(seed)
    stock = S.SparseGP(X, Y, Z.copy(), kern(G), Bern(), inference_method=EPDTC())
    r_stock = np.random.random()
    np.random.seed(seed)
    plug = S.SparseGP(X, Y, Z.copy(), kern(B), Bern(), inference_method=B.EPDTC())
    assert np.random.random() == r_stock
    names = [c[0] for c in plug.inference_method.engine.calls]
    assert names[:3] == ["set_data", "begin", "start"] and names[-1] == "finish"
    l_s, l_p = float(np.squeeze(stock.log_likelihood())), float(np.squeeze(plug.log_likelihood()))
    assert abs(l_p - l_s) <= BAR * abs(l_s)
    gs, gp = np.asarray(stock.gradient), np.asarray(plug.gradient)
    np.testing.assert_allclose(gp, gs, rtol=0, atol=1e-7 * np.abs(gs).max())
    im = plug.inference_method
    assert type(im.ga_approx_old) is ref.gaussianApproximation
    assert len(im._ep_approximation) == 3 and type(im._ep_approximation[0]) is ref.posteriorParamsDTC
    np.testing.assert_allclose(im.ga_approx_old.tau, stock.inference_method.ga_approx_old.tau, rtol=0, atol=BAR)


def test_plugin_epdtc_sends_anything_else_to_the_stock_method_and_continues_its_sites():
    S, C, G, B, EPDTC, Bern, ObsAr = _plugin()
    X, Y, Z, _ = eo.case_data("rbf_iso_n60_m10")
    Yo = ObsAr(Y)
    inf = B.EPDTC(ep_mode="nested")

    def quiet():
        return inf._engine is None or not inf.engine.calls

    np.random.seed(1)
    inf.inference(G.RBF(3), X, Z, Bern(), Yo)                                    # the reference's own kernel
    assert quiet()
    with pytest.raises(Exception):
        inf.inference(B.RBF(3), X, Z, Bern(), Yo, mean_function=object())        # a mean function: the stock method
    assert quiet()
    Lm = eo.jitchol(G.RBF(3).K(Z))
    with pytest.raises(UnboundLocalError):   # a precomputed Lm: the stock method, which reads Kmm it did not form (:445-459)
        inf.inference(B.RBF(3), X, Z, Bern(), Yo, Lm=Lm)
    assert quiet()
    from test_periodic_ratquad_plugin_cpu import fake_ffi  # noqa: F401
    inf.inference(C.Add([B.RBF(3), G.Matern32(3)]), X, Z, Bern(), Yo)            # a foreign leaf: the stock method
    assert quiet()
    # the device continues from the stock method's sites (a warm start), as the stock calls do
    refm = EPDTC(ep_mode="nested")
    np.random.seed(1)
    refm.inference(G.RBF(3), X, Z, Bern(), Yo)
    with pytest.raises(Exception):   # the stock method runs EP before VarDTC rejects the mean function
        refm.inference(G.RBF(3), X, Z, Bern(), Yo, mean_function=object())
    refm.inference(C.Add([G.RBF(3), G.Matern32(3)]), X, Z, Bern(), Yo)
    np.random.seed(2)
    _, l_ref, _ = refm.inference(G.RBF(3), X, Z, Bern(), Yo)
    np.random.seed(2)
    _, l_dev, _ = inf.inference(B.RBF(3), X, Z, Bern(), Yo)
    assert ("start", True) in inf.engine.calls
    assert abs(l_dev - l_ref) <= BAR * abs(l_ref)
