"""The sparse GPLVM on the CPU: the NumPy restatement (tests/sparse_gplvm_oracle.py) against every reference fixture
(tests/golden/make_sparse_gplvm.py), and the host logic of the mirror gpy_b200.SparseGPLVM and of the plugin's VarDTC
handles over a test double of the engine that answers from the restatement. The reference's own SparseGPLVM runs
unchanged over B.VarDTC(): its kern.gradients_X(dL_dKnm, X, Z) (sparse_gplvm.py:34) takes one device input gradient,
whatever the shape of dL_dKnm (N = M included), and dL_dKnm.T (sparse_gp.py:118) still gives dL/dZ."""
import glob
import os
import types

import numpy as np
import pytest

import sparse_gplvm_oracle as sg

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sparse_gplvm")
CASES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLD, "*.npz")) if not p.endswith("het.npz"))
REF = os.path.isdir(os.environ.get("GPX_REFERENCE", "/root/reference") + "/GPy")


def _load(name):
    return np.load(os.path.join(GOLD, name + ".npz"))


def _parts_of(d):
    """CompositeOracle parts of the kernel a fixture's model holds after its construction"""
    case = sg.CASES[d]
    return sg.case_parts(case, case["Q"])


@pytest.mark.parametrize("name", CASES)
def test_the_restatement_matches_the_reference_fixture(name):
    d = _load(name)
    lml, grad, dX, res = sg.sparse_gplvm_eval(d["X0"], d["Y"], d["Z0"], _parts_of(name), float(d["noise"]))
    assert abs(lml - float(d["lml"])) <= 1e-9 * max(1.0, abs(float(d["lml"])))
    np.testing.assert_allclose(grad, d["grad"], rtol=1e-8, atol=1e-9 * np.abs(d["grad"]).max())


def test_the_restatement_matches_the_heteroscedastic_fixture():
    d = _load("het")
    parts = [dict(kind="rbf", term=0, dims=[0, 1], variance=1.1, lengthscale=[0.9, 1.3], ARD=True)]
    lml, grad, dX, res = sg.sparse_gplvm_eval(d["X"], d["Y"], d["Z"], parts, d["noise"])
    assert abs(lml - float(d["lml"])) <= 1e-9 * max(1.0, abs(float(d["lml"])))
    np.testing.assert_allclose(dX, d["dX"], rtol=1e-8, atol=1e-10 * np.abs(d["dX"]).max())


def test_the_fixtures_cover_the_wide_route_and_the_orientation_case():
    shapes = {n: (_load(n)["Y"].shape, _load(n)["Z0"].shape) for n in CASES}
    assert {y[1] for y, _ in shapes.values()} >= {1, 8, 9, 12, 64, 257}
    assert any(y[0] == z[0] for y, z in shapes.values())                 # N = M
    assert any(z[0] % 128 and z[0] > 128 for _, z in shapes.values())    # M past one tile, not a multiple of it


class FakeEngine(object):
    """the sparse entries of _ffi.Engine the sparse GPLVM uses, answered by the restatement"""

    def __init__(self, device=0):
        self.calls, self.sparse_serial = [], 0

    def set_option(self, name, value):
        self.calls.append("set_option %s=%d" % (name, value))

    def sparse_set_data(self, X, Y):
        if Y.shape[1] > 8:
            assert "set_option sparse_wide=1" in self.calls, "more than 8 output columns need the option sparse_wide"
        self.X, self.Y = np.array(X), np.array(Y)
        self.calls.append("sparse_set_data")

    def _eval(self, parts, Z, noise):
        self.sparse_serial += 1
        self.parts, self.Z = parts, np.array(Z)
        lml, grad, dX, self.res = sg.sparse_gplvm_eval(self.X, self.Y, Z, parts, noise)
        self.dX = dX
        n = self.X.size + self.Z.size
        return lml, grad[n:], grad[self.X.size:n].reshape(self.Z.shape)

    def sparse_eval(self, kind, ARD, variance, lengthscale, Z, noise):
        self.calls.append("sparse_eval")
        parts = [dict(kind=kind, term=0, dims=list(range(self.X.shape[1])), variance=variance, lengthscale=lengthscale,
                      ARD=ARD)]
        return self._eval(parts, Z, noise)

    def sparse_eval_multi(self, parts, Z, noise):
        self.calls.append("sparse_eval_multi")
        ps = []
        for d in parts:
            p = dict(kind=d[0], ARD=d[1], term=d[2], dims=list(d[3]), variance=d[4])
            if d[0] not in ("white", "bias"):
                p["lengthscale"] = d[5]
            ps.append(p)
        return self._eval(ps, Z, noise)

    def sparse_grad_X(self):
        self.calls.append("sparse_grad_X")
        return self.dX.copy()

    def sparse_get(self, what):
        return {"woodbury_vector": self.res["woodbury_vector"], "woodbury_inv": self.res["woodbury_inv"],
                "Kmm": self.res["Kmm"], "Lm": self.res["Lm"]}[what]


@pytest.mark.parametrize("name", ["default_p1", "default_p9", "rbf_ard_bias_white", "m32_x_rbf_bias", "default_n_eq_m"])
def test_the_mirror_on_a_host_double_matches_the_fixture(name):
    import gpy_b200
    d = _load(name)
    case = sg.CASES[name]
    kern = case["kernel"](vars(gpy_b200)) if case["kernel"] is not None else None
    eng = FakeEngine()
    np.random.seed(int(d["seed"]))
    m = gpy_b200.SparseGPLVM(d["Y"], case["Q"], kernel=kern, num_inducing=case["M"], engine=eng)
    np.testing.assert_array_equal(m.latent_space.values, d["X0"])      # initialize_latent, then the permutation for Z
    np.testing.assert_array_equal(m.Z.values, d["Z0"])
    m.likelihood.variance[:] = float(d["noise"])
    assert abs(m.log_likelihood() - float(d["lml"])) <= 1e-9 * max(1.0, abs(float(d["lml"])))
    np.testing.assert_allclose(m.gradient, d["grad"], rtol=1e-8, atol=1e-9 * np.abs(d["grad"]).max())
    assert eng.calls[-1] == "sparse_grad_X"
    names = m.parameter_names()
    assert names[0].endswith("latent space") and names[1].endswith("inducing inputs")
    # the optimizer space: latent and inducing inputs as they are, the rest through Logexp
    x = m.optimizer_array
    nfree = m.latent_space.values.size + m.Z.values.size
    np.testing.assert_array_equal(x[:m.latent_space.values.size], d["X0"].reshape(-1))
    assert x.size == d["grad"].size and nfree < x.size


def test_the_mirror_takes_a_lone_kernel_on_some_columns():
    import gpy_b200
    d = _load("default_p9")
    eng = FakeEngine()
    X = np.column_stack([d["X0"], np.linspace(-1, 1, d["X0"].shape[0])])
    kern = gpy_b200.RBF(2, variance=1.0, lengthscale=1.0, active_dims=[0, 1])
    m = gpy_b200.SparseGPLVM(d["Y"], 3, X=X, kernel=kern, num_inducing=10, engine=eng)
    g = m.latent_space.gradient
    assert g.shape == X.shape and np.all(g[:, 2] == 0.0) and np.abs(g[:, :2]).max() > 0


def _plugin(ffi_engine):
    from oracle import ref_gpy
    from gpy_b200 import gpy_plugin
    SGPLVM, ns, S = sg.reference_sparse_gplvm()
    C = ref_gpy.load_combination()
    G = S.G
    from test_periodic_ratquad_plugin_cpu import fake_ffi
    f = fake_ffi()
    from oracle import gpy_oracle as o

    def kern_grad_X(kind, ARD, var, ls, X, dL_dK, X2=None):      # the model's constructor runs the stock VarDTC
        return o.StationaryOracle(kind, X.shape[1], var, ls, ARD).gradients_X(dL_dK, X, X2)
    ffi = types.SimpleNamespace(kern_K=f.kern_K, kern_Kdiag=f.kern_Kdiag, kern_grad_full=f.kern_grad_full,
                                kern_grad_X=kern_grad_X, kern_part_K=f.kern_part_K,
                                kern_part_grad_full=f.kern_part_grad_full, Engine=ffi_engine)
    B = gpy_plugin.make(G.RBF, G.Exponential, G.Matern32, G.Matern52, G.ExactGaussianInference, Add=C.Add, Prod=C.Prod,
                        VarDTC=G.VarDTC)
    Bf = gpy_plugin.make(G.RBF, G.Exponential, G.Matern32, G.Matern52, G.ExactGaussianInference, Add=C.Add, Prod=C.Prod,
                         VarDTC=G.VarDTC, ffi=ffi)
    return SGPLVM, ns, G, C, B, Bf


def _reference_over_plugin(name, Bf, ns, SGPLVM, C):
    d = _load(name)
    case = sg.CASES[name]
    # the fixtures' kernels with the plugin's leaves and combinations (`+` / `*` would build the stock Add / Prod)
    kern = {"rbf_ard_bias_white": lambda: Bf.Add([Bf.RBF(2, 1.2, [0.8, 1.3], ARD=True), C.Bias(2, 0.1), C.White(2, 0.05)]),
            "m32_x_rbf_bias": lambda: Bf.Add([Bf.Prod([Bf.Matern32(2, variance=0.9, lengthscale=1.2),
                                                       Bf.RBF(2, variance=1.1, lengthscale=[0.7, 1.5], ARD=True)]),
                                              C.Bias(2, 0.2)])}.get(name, lambda: Bf.RBF(case["Q"]))()
    np.random.seed(int(d["seed"]))
    m = SGPLVM(d["Y"], case["Q"], kernel=kern, num_inducing=case["M"])
    m.inference_method = Bf.VarDTC()
    m.likelihood.variance[:] = float(d["noise"])
    return m, d


@pytest.mark.skipif(not REF, reason="reference tree not present")
@pytest.mark.parametrize("name", ["default_p1", "default_p12", "rbf_ard_bias_white",
                                  "m32_x_rbf_bias", "default_n_eq_m"])
def test_the_reference_sparse_gplvm_runs_on_the_plugin_pair(name):
    SGPLVM, ns, G, C, B, Bf = _plugin(FakeEngine)
    m, d = _reference_over_plugin(name, Bf, ns, SGPLVM, C)
    m.parameters_changed()
    eng = m.inference_method.engine
    evals = sum(c.startswith("sparse_eval") for c in eng.calls)
    assert eng.calls[-1] == "sparse_grad_X" and eng.calls.count("sparse_grad_X") == evals   # one per evaluation
    assert abs(float(np.squeeze(m.log_likelihood())) - float(d["lml"])) <= 1e-9 * max(1.0, abs(float(d["lml"])))
    np.testing.assert_allclose(np.asarray(m.gradient), d["grad"], rtol=1e-8, atol=1e-9 * np.abs(d["grad"]).max())


@pytest.mark.skipif(not REF, reason="reference tree not present")
def test_the_handle_orientation_decides_when_n_equals_m():
    SGPLVM, ns, G, C, B, Bf = _plugin(FakeEngine)
    m, d = _reference_over_plugin("default_n_eq_m", Bf, ns, SGPLVM, C)
    m.parameters_changed()
    h = m.grad_dict["dL_dKnm"]
    assert h.shape[0] == h.shape[1] and not h.transposed and h.T.transposed and not h.T.T.transposed
    eng = m.inference_method.engine
    dX = m.kern.gradients_X(h, m.X, m.Z)
    dZ = m.kern.gradients_X(h.T, m.Z, m.X)
    np.testing.assert_array_equal(dZ, h.dZ)
    np.testing.assert_allclose(dX, eng.dX, rtol=0, atol=0)
    assert not np.allclose(dX, dZ)
    n = eng.calls.count("sparse_grad_X")
    m.kern.gradients_X(h, m.X, m.Z)
    assert eng.calls.count("sparse_grad_X") == n                         # fetched once per evaluation


@pytest.mark.skipif(not REF, reason="reference tree not present")
def test_a_stale_or_foreign_handle_is_refused():
    SGPLVM, ns, G, C, B, Bf = _plugin(FakeEngine)
    m, d = _reference_over_plugin("default_p1", Bf, ns, SGPLVM, C)
    m.parameters_changed()
    h = m.grad_dict["dL_dKnm"]
    X, Z = np.array(m.X), np.array(m.Z)
    with pytest.raises(ValueError, match="inputs"):
        m.kern.gradients_X(h, X + 1.0, Z)
    m.kern.variance[:] = 1.7                                              # a new evaluation: the old handle is stale
    with pytest.raises(ValueError, match="stale"):
        m.kern.gradients_X(h, X, Z)
    with pytest.raises(TypeError):
        np.asarray(h)
