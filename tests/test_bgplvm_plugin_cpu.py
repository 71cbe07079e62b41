"""The reference's own BayesianGPLVM (GPy/models/bayesian_gplvm.py, run with the real psi_comp package through
bgplvm_oracle.reference_bayesian_gplvm) over the plugin's B.VarDTC and B.RBF on a host double of the engine: the same bound
and gradients as the stock model and as gpy_b200.BayesianGPLVM from the same seed; the stand-alone psi calls; every
fallback to the reference's methods; a stale handle. No GPU needed."""
import os
import types

import numpy as np
import pytest

import bgplvm_oracle as bo

REF = os.path.isdir(os.environ.get("GPX_REFERENCE", "/root/reference") + "/GPy")
pytestmark = pytest.mark.skipif(not REF, reason="reference tree not present")


class FakeEngine(object):
    """the sparse entries the plugin calls, restated on the host by tests/bgplvm_oracle.py"""

    def __init__(self, device=0):
        self.sparse_serial, self.calls = 0, []

    def set_option(self, name, value):
        pass

    def sparse_set_data(self, X, Y):
        self.X, self.Y = np.array(X, dtype=np.float64), np.array(Y, dtype=np.float64)

    def sparse_eval_psi(self, rbf, S, Z, noise):
        kind, ard, term, dims, variance, ls = rbf
        assert kind == "rbf" and list(dims) == list(range(self.X.shape[1]))
        r = bo.vardtc_psi(variance, np.atleast_1d(ls), ard, np.asarray(Z), self.X, np.asarray(S), self.Y, noise)
        self.sparse_serial += 1
        self.calls.append("sparse_eval_psi")
        return r["lml"], r["grad"], r["dZ"], r["dmu"], r["dS"]


def _plugin():
    from gpy_b200 import gpy_plugin
    BG, S, V = bo.reference_bayesian_gplvm()
    G = S.G
    calls = []

    def psi_stats(rbf, mu, Sv, Z):
        calls.append("psi_stats")
        return bo.psi_stats(rbf[4], np.atleast_1d(rbf[5]), Z, mu, Sv)

    def psi_grads(rbf, mu, Sv, Z, d0, d1, d2):
        calls.append("psi_grads")
        return bo.psi_derivs(d0, d1, d2, rbf[4], np.atleast_1d(rbf[5]), Z, mu, Sv, rbf[1])

    from test_periodic_ratquad_plugin_cpu import fake_ffi
    f = fake_ffi()
    ffi = types.SimpleNamespace(kern_K=f.kern_K, kern_Kdiag=f.kern_Kdiag, kern_grad_full=f.kern_grad_full,
                                kern_part_K=f.kern_part_K, kern_part_grad_full=f.kern_part_grad_full, Engine=FakeEngine,
                                psi_stats=psi_stats, psi_grads=psi_grads)
    Bf = gpy_plugin.make(G.RBF, G.Exponential, G.Matern32, G.Matern52, G.ExactGaussianInference, VarDTC=G.VarDTC, ffi=ffi)
    return BG, G, V, Bf, calls


def _models(Y, Q, M, seed, ard=True):
    """the stock reference model and the same model over the plugin pair, from the same seed"""
    BG, G, V, Bf, calls = _plugin()
    np.random.seed(seed)
    m0 = BG(Y, Q, num_inducing=M)
    ls = np.asarray(m0.kern.lengthscale, dtype=np.float64)
    np.random.seed(seed)
    m1 = BG(Y, Q, num_inducing=M, kernel=Bf.RBF(Q, lengthscale=ls, ARD=True), inference_method=Bf.VarDTC())
    return m0, m1, Bf, calls


@pytest.mark.parametrize("name", ["default_p1", "default_p12"])
def test_reference_model_over_the_plugin_matches_the_stock_model_and_the_mirror(name):
    import gpy_b200
    c = bo.CASES[name]
    _, _, _, Y, _ = bo.case_inputs(c)
    m0, m1, Bf, calls = _models(Y, c["Q"], c["M"], c["seed"])
    b0, g0 = float(np.squeeze(m0.log_likelihood())), np.asarray(m0.gradient)
    b1, g1 = float(np.squeeze(m1.log_likelihood())), np.asarray(m1.gradient)
    assert m1.inference_method.engine.calls == ["sparse_eval_psi"]      # one device evaluation, no host psi call
    assert calls == []
    assert abs(b1 - b0) <= 1e-8 * max(1.0, abs(b0))
    assert np.max(np.abs(g1 - g0)) <= 1e-6 * np.max(np.abs(g0))
    from test_bgplvm_mirror_cpu import HostEngine
    np.random.seed(c["seed"])
    m2 = gpy_b200.BayesianGPLVM(Y, c["Q"], num_inducing=c["M"], engine=HostEngine())
    np.testing.assert_array_equal(m2.latent_mean.values, np.asarray(m0.X.mean))
    np.testing.assert_array_equal(m2.latent_variance.values, np.asarray(m0.X.variance))
    np.testing.assert_array_equal(m2.Z.values, np.asarray(m0.Z))
    np.testing.assert_allclose(m2.kern.lengthscale.values, np.asarray(m0.kern.lengthscale), rtol=1e-15)
    assert abs(m2.log_likelihood() - b0) <= 1e-8 * max(1.0, abs(b0))
    assert np.max(np.abs(m2.gradient - g0)) <= 1e-6 * np.max(np.abs(g0))


def test_stand_alone_psi_calls_go_to_the_device_entries():
    BG, G, V, Bf, calls = _plugin()
    f = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bgplvm", "psi.npz"))
    k = Bf.RBF(3, variance=float(f["variance"]), lengthscale=f["ls"], ARD=True)
    qX = V.NormalPosterior(f["mu"], f["S"])
    np.testing.assert_allclose(k.psi1(f["Z"], qX), f["psi1_ard"], rtol=1e-12)
    np.testing.assert_allclose(k.psi2(f["Z"], qX), f["psi2_ard"], rtol=1e-12)
    np.testing.assert_allclose(k.psi0(f["Z"], qX), f["psi0_ard"], rtol=1e-15)
    dZ = k.gradients_Z_expectations(f["dL0"], f["dL1"], f["dL2"], f["Z"], qX)
    dmu, dS = k.gradients_qX_expectations(f["dL0"], f["dL1"], f["dL2"], f["Z"], qX)
    k.update_gradients_expectations(f["dL0"], f["dL1"], f["dL2"], f["Z"], qX)
    np.testing.assert_allclose(dZ, f["dZ_ard"], rtol=1e-9, atol=1e-9 * np.abs(f["dZ_ard"]).max())
    np.testing.assert_allclose(dmu, f["dmu_ard"], rtol=1e-9, atol=1e-9 * np.abs(f["dmu_ard"]).max())
    np.testing.assert_allclose(dS, f["dS_ard"], rtol=1e-9, atol=1e-9 * np.abs(f["dS_ard"]).max())
    np.testing.assert_allclose(np.r_[np.atleast_1d(k.variance.gradient), k.lengthscale.gradient], f["grad_ard"], rtol=1e-9)
    assert calls == ["psi_stats", "psi_stats", "psi_grads", "psi_grads", "psi_grads"]
    n = len(calls)
    k.psi2n(f["Z"], qX)                                                    # per-point psi2: the reference's own
    assert len(calls) == n


def test_every_fallback_takes_the_stock_method():
    BG, G, V, Bf, calls = _plugin()
    c = bo.CASES["default_p1"]
    mu, S, Z, Y, _ = bo.case_inputs(c)
    vd = Bf.VarDTC()
    qX = V.NormalPosterior(mu, S)
    lik = G.Gaussian(variance=0.1)
    rbf = Bf.RBF(3, ARD=True)
    assert vd._psi_route(rbf, qX, lik, None, None, None, None, None, None, None, None)
    for args in ((rbf, mu, lik),                                          # certain inputs
                 (G.RBF(3, ARD=True), qX, lik),                           # not a plugin kernel
                 (Bf.Matern32(3), qX, lik),                               # not an RBF
                 (Bf.RBF(2, active_dims=[0, 1]), qX, lik),                # not on every latent column
                 (Bf.RBF(2, active_dims=[1, 0]), V.NormalPosterior(mu[:, :2], S[:, :2]), lik)):   # not in order
        assert not vd._psi_route(args[0], args[1], args[2], None, None, None, None, None, None, None, None)
    assert not vd._psi_route(rbf, qX, lik, None, object(), None, None, None, None, None, None)      # mean function
    assert not vd._psi_route(rbf, qX, lik, None, None, np.ones(len(mu)), None, None, None, None, None)   # precision
    assert not vd._psi_route(rbf, qX, lik, None, None, None, None, None, None, np.ones((len(mu), len(Z))), None)
    wide = V.NormalPosterior(np.zeros((4, 17)), np.ones((4, 17)))
    assert not vd._psi_route(Bf.RBF(17, ARD=True), wide, lik, None, None, None, None, None, None, None, None)
    het = G.HeteroscedasticGaussian({"output_index": np.arange(len(mu))[:, None]})
    assert not vd._psi_route(rbf, qX, het, {"output_index": np.arange(len(mu))[:, None]}, None, None, None, None, None,
                             None, None)

    class SpikeAndSlab(object):
        mean, variance = mu, S
    assert not vd._psi_route(rbf, SpikeAndSlab(), lik, None, None, None, None, None, None, None, None)
    # a fallback evaluation is the stock VarDTC: it asks the kernel for host psi-statistics
    post, lml, gd = vd.inference(rbf, qX, Z, lik, Y, mean_function=None, psi0=rbf.psi0(Z, qX))
    assert not isinstance(gd["dL_dpsi1"], type(None)) and isinstance(gd["dL_dpsi1"], np.ndarray)


def test_a_stale_or_foreign_handle_is_refused():
    c = bo.CASES["default_p1"]
    _, _, _, Y, _ = bo.case_inputs(c)
    m0, m1, Bf, calls = _models(Y, c["Q"], c["M"], c["seed"])
    gd = m1.grad_dict
    h = gd["dL_dpsi1"]
    with pytest.raises(TypeError):
        np.asarray(h)
    with pytest.raises(ValueError, match="inducing inputs"):
        m1.kern.gradients_Z_expectations(gd["dL_dpsi0"], h, gd["dL_dpsi2"], np.asarray(m1.Z) + 1.0, m1.X)
    m1.kern.variance[:] = 1.7                                              # a new evaluation: the old handle is stale
    with pytest.raises(ValueError, match="stale"):
        m1.kern.gradients_qX_expectations(gd["dL_dpsi0"], h, gd["dL_dpsi2"], m1.Z, m1.X)
