"""The sparse GPLVM on the device: every reference fixture (tests/golden/make_sparse_gplvm.py) through the C ABI, the
mirror gpy_b200.SparseGPLVM and the reference's own SparseGPLVM over the plugin pair; checkgrad of the latent inputs;
the wide route (P > 8) against the sum of its 8-column slices through the narrow route; gpx_sparse_grad_X after the
posterior consumers; every -2 rejection; launch counts. Held to 1e-8 on the LML and 1e-6 relative on gradients."""
import glob
import json
import os

import numpy as np
import pytest

import sparse_gplvm_oracle as sg
from sparse_composite_oracle import descriptor

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sparse_gplvm")
CASES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLD, "*.npz")) if not p.endswith("het.npz"))
REF = os.path.isdir(os.environ.get("GPX_REFERENCE", "/root/reference") + "/GPy")
MARGINS = {}


def _margins_out():
    d = os.environ.get("GPX_MARGINS_DIR")
    if d:
        os.makedirs(d, exist_ok=True)
        with open(os.path.join(d, "sparse_gplvm_margins.json"), "w") as f:
            json.dump(MARGINS, f, indent=1, sort_keys=True)


def _ffi():
    from gpy_b200 import _ffi
    return _ffi


def _load(name):
    return np.load(os.path.join(GOLD, name + ".npz"))


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.max(np.abs(a - b)) / max(np.abs(b).max(), 1e-300))


def _device_eval(e, X, Y, Z, parts, noise):
    """-> (lml, grad [X, Z, kernel.., noise], dX) on the device"""
    if Y.shape[1] > 8:
        e.set_option("sparse_wide", 1)
    e.sparse_set_data(X, Y)
    lml, g, dZ = e.sparse_eval_multi([descriptor(p) for p in parts], Z, noise)[:3]
    dX = e.sparse_grad_X()
    return lml, np.concatenate([dX.reshape(-1), dZ.reshape(-1), g]), dX


@pytest.mark.parametrize("name", CASES)
def test_every_fixture_through_the_c_abi(name):
    d = _load(name)
    case = sg.CASES[name]
    e = _ffi().Engine(0)
    lml, g, dX = _device_eval(e, d["X0"], d["Y"], d["Z0"], sg.case_parts(case, case["Q"]), float(d["noise"]))
    MARGINS["abi_" + name] = dict(lml=abs(lml - float(d["lml"])), grad=_rel(g, d["grad"]))
    assert abs(lml - float(d["lml"])) <= 1e-8 * max(1.0, abs(float(d["lml"])))
    assert _rel(g, d["grad"]) <= 1e-6
    mu, var = e.sparse_predict(d["Xnew"])
    np.testing.assert_allclose(mu, d["mu"], rtol=1e-6, atol=1e-9 * np.abs(d["mu"]).max())
    np.testing.assert_allclose(var + float(d["noise"]), d["var"], rtol=1e-6)
    _margins_out()


def test_the_heteroscedastic_fixture_through_the_c_abi():
    d = _load("het")
    e = _ffi().Engine(0)
    e.sparse_set_data(d["X"], d["Y"])
    lml = e.sparse_eval_het("rbf", True, 1.1, np.array([0.9, 1.3]), d["Z"], d["noise"])[0]
    dX = e.sparse_grad_X()
    MARGINS["abi_het"] = dict(lml=abs(lml - float(d["lml"])), dX=_rel(dX, d["dX"]))
    assert abs(lml - float(d["lml"])) <= 1e-8 * max(1.0, abs(float(d["lml"])))
    assert _rel(dX, d["dX"]) <= 1e-6


@pytest.mark.parametrize("name", ["default_p1", "default_p9", "default_p257", "rbf_ard_bias_white", "m32_x_rbf_bias",
                                  "default_n1300_m129", "default_n_eq_m"])
def test_the_mirror_matches_the_fixture(name):
    import gpy_b200
    d = _load(name)
    case = sg.CASES[name]
    kern = case["kernel"](vars(gpy_b200)) if case["kernel"] is not None else None
    np.random.seed(int(d["seed"]))
    m = gpy_b200.SparseGPLVM(d["Y"], case["Q"], kernel=kern, num_inducing=case["M"])
    np.testing.assert_array_equal(m.latent_space.values, d["X0"])
    np.testing.assert_array_equal(m.Z.values, d["Z0"])
    m.likelihood.variance[:] = float(d["noise"])
    assert abs(m.log_likelihood() - float(d["lml"])) <= 1e-8 * max(1.0, abs(float(d["lml"])))
    assert _rel(m.gradient, d["grad"]) <= 1e-6
    mu, var = m.predict(d["Xnew"])
    np.testing.assert_allclose(mu, d["mu"], rtol=1e-6, atol=1e-9 * np.abs(d["mu"]).max())
    np.testing.assert_allclose(var, d["var"], rtol=1e-6)


@pytest.mark.skipif(not REF, reason="reference tree not present")
@pytest.mark.parametrize("name", ["default_p12", "rbf_ard_bias_white", "default_n_eq_m"])
def test_the_reference_sparse_gplvm_over_the_plugin_pair(name):
    from oracle import ref_gpy
    from gpy_b200 import gpy_plugin
    SGPLVM, ns, S = sg.reference_sparse_gplvm()
    C = ref_gpy.load_combination()
    G = S.G
    B = gpy_plugin.make(G.RBF, G.Exponential, G.Matern32, G.Matern52, G.ExactGaussianInference, Add=C.Add, Prod=C.Prod,
                        VarDTC=G.VarDTC)
    d = _load(name)
    case = sg.CASES[name]
    kern = B.Add([B.RBF(2, 1.2, [0.8, 1.3], ARD=True), C.Bias(2, 0.1), C.White(2, 0.05)]) \
        if name == "rbf_ard_bias_white" else B.RBF(case["Q"])
    np.random.seed(int(d["seed"]))
    m = SGPLVM(d["Y"], case["Q"], kernel=kern, num_inducing=case["M"])
    m.inference_method = B.VarDTC()
    m.likelihood.variance[:] = float(d["noise"])
    lml = float(np.squeeze(m.log_likelihood()))
    MARGINS["plugin_" + name] = dict(lml=abs(lml - float(d["lml"])), grad=_rel(m.gradient, d["grad"]))
    assert abs(lml - float(d["lml"])) <= 1e-8 * max(1.0, abs(float(d["lml"])))
    assert _rel(m.gradient, d["grad"]) <= 1e-6


def test_checkgrad_of_the_latent_inputs():
    import gpy_b200
    d = _load("default_p12")
    np.random.seed(int(d["seed"]))
    m = gpy_b200.SparseGPLVM(d["Y"][:60], 2, num_inducing=8)
    assert m.checkgrad(step=1e-6, tolerance=1e-4, sample=40)


def _wide_problem(N, M, P, seed):
    rng = np.random.default_rng(seed)
    X = rng.uniform(-2, 2, size=(N, 3))
    Y = np.sin(X.dot(rng.standard_normal((3, P)))) + 0.1 * rng.standard_normal((N, P))
    Z = rng.uniform(-2, 2, size=(M, 3))
    return X, Y, Z


WIDE = [(1025, 129), (1025, 512), (4097, 129), (4097, 512), (65536, 129), (65536, 512)]


@pytest.mark.parametrize("N,M", WIDE)
@pytest.mark.parametrize("kernel", ["rbf_ard", "composite"])
def test_the_wide_route_is_the_sum_of_narrow_slices(N, M, kernel):
    """with shared noise the bound and all its gradients are sums over output columns: P = 64 at once against 8 slices of
    8 columns through the unchanged narrow route, on the device itself"""
    P = 64
    X, Y, Z = _wide_problem(N, M, P, N + M)
    # short lengthscales keep Kmm well conditioned: dL/dZ is a difference of its Kmm and Knm shares and loses ~cond(Kmm)
    # digits to any change of summation order (a Z of 512 points at lengthscale ~1 put 1.4e-5 between the two routes)
    if kernel == "rbf_ard":
        parts = [dict(kind="rbf", term=0, dims=[0, 1, 2], variance=1.3, lengthscale=[0.35, 0.5, 0.6], ARD=True)]
    else:
        parts = [dict(kind="matern32", term=0, dims=[0, 1, 2], variance=0.9, lengthscale=0.4),
                 dict(kind="rbf", term=0, dims=[0, 1], variance=1.1, lengthscale=[0.3, 0.5], ARD=True),
                 dict(kind="bias", term=1, variance=0.2)]
    noise = 0.05
    Xnew = np.random.default_rng(7).uniform(-2, 2, size=(300, 3))
    e = _ffi().Engine(0)
    lml, g, dX = _device_eval(e, X, Y, Z, parts, noise)
    wv = e.sparse_get("woodbury_vector")
    mu, var = e.sparse_predict(Xnew)
    lml_s, g_s, dX_s = 0.0, np.zeros_like(g), np.zeros_like(dX)
    for q0 in range(0, P, 8):
        ls, gs, dxs = _device_eval(e, X, Y[:, q0:q0 + 8], Z, parts, noise)
        lml_s += ls
        g_s += gs
        dX_s += dxs
        np.testing.assert_allclose(e.sparse_get("woodbury_vector"), wv[:, q0:q0 + 8], rtol=1e-8,
                                   atol=1e-10 * np.abs(wv).max())
        ms, vs = e.sparse_predict(Xnew)
        np.testing.assert_allclose(ms, mu[:, q0:q0 + 8], rtol=1e-8, atol=1e-10 * np.abs(mu).max())
        np.testing.assert_allclose(vs, var, rtol=1e-9)
    nX, nZ = X.size, Z.size
    m = dict(lml=abs(lml - lml_s) / abs(lml_s), dX=_rel(g[:nX], g_s[:nX]), dZ=_rel(g[nX:nX + nZ], g_s[nX:nX + nZ]),
             kern=_rel(g[nX + nZ:], g_s[nX + nZ:]))
    MARGINS["wide_%s_n%d_m%d" % (kernel, N, M)] = m
    _margins_out()
    assert m["lml"] <= 1e-10 and m["dX"] <= 1e-6 and m["dZ"] <= 1e-6 and m["kern"] <= 1e-6


def test_grad_x_is_untouched_by_the_posterior_consumers():
    X, Y, Z = _wide_problem(1500, 140, 3, 5)
    parts = [dict(kind="matern52", term=0, dims=[0, 1, 2], variance=1.1, lengthscale=[0.8, 1.2, 1.6], ARD=True)]
    e = _ffi().Engine(0)
    _, _, dX0 = _device_eval(e, X, Y, Z, parts, 0.1)
    Xnew = X[:50] + 0.05
    e.sparse_get("woodbury_vector")
    e.sparse_get("woodbury_inv")
    e.sparse_predict(Xnew)
    e.sparse_predict(Xnew, full_cov=True)
    e.sparse_predictive_gradients(Xnew)
    e.sparse_posterior_samples(Xnew, np.random.default_rng(0).standard_normal((3 * 2, 50)))
    np.testing.assert_array_equal(e.sparse_grad_X(), dX0)
    np.testing.assert_array_equal(e.sparse_grad_X(), dX0)


def _rejects(fn, *a):
    with pytest.raises(_ffi().GpxArgumentError):
        fn(*a)


def test_every_rejection():
    f = _ffi()
    X, Y, Z = _wide_problem(400, 30, 1, 6)
    parts = [("rbf", False, 0, [0, 1, 2], 1.0, 1.0)]
    e = f.Engine(0)
    _rejects(e.sparse_grad_X)                                            # no data, no evaluation
    e.sparse_set_data(X, Y)
    _rejects(e.sparse_grad_X)                                            # no evaluation
    e.sparse_eval_multi(parts, Z, 0.1)
    e.sparse_grad_X()
    e.sparse_eval_fitc(parts, Z, 0.1)                                    # FITC wrote dL_dKnm^T
    _rejects(e.sparse_grad_X)
    e.sparse_eval_multi(parts, Z, 0.1)
    e.sparse_set_data(X, Y)                                              # new data
    _rejects(e.sparse_grad_X)
    e.sparse_eval_multi(parts, Z, 0.1)
    M = Z.shape[0]
    e.svgp_begin(parts, Z, np.zeros(M), np.eye(M), 0, 100)              # SVGP
    _rejects(e.sparse_grad_X)
    e.sparse_set_data(X, np.sign(Y))
    e.sparse_eval_multi(parts, Z, 0.1)
    e.epdtc_begin(parts, Z)                                              # sparse EP
    _rejects(e.sparse_grad_X)
    assert f.lib().gpx_sparse_grad_X(e._h, None) == -2                   # null pointers
    assert f.lib().gpx_sparse_grad_X(None, None) == -2
    # more than 8 outputs: the entries that keep the narrow limit
    Xw, Yw, Zw = _wide_problem(300, 20, 12, 8)
    w = f.Engine(0)
    _rejects(w.sparse_set_data, Xw, Yw)                                   # a context keeps the limit of 8 unless told
    w.set_option("sparse_wide", 1)
    w.sparse_set_data(Xw, Yw)
    _rejects(w.sparse_eval_het, "rbf", False, 1.0, 1.0, Zw, np.full(300, 0.1))
    _rejects(w.sparse_eval_multi, parts, Zw, np.full(300, 0.1))
    w.sparse_eval_multi(parts, Zw, 0.1)
    dX = w.sparse_grad_X()
    _rejects(w.sparse_predictive_gradients, Xw[:5])
    _rejects(w.sparse_posterior_samples, Xw[:5], np.zeros((12, 5)))
    _rejects(w.sparse_eval_fitc, parts, Zw, 0.1)
    np.testing.assert_array_equal(w.sparse_grad_X(), dX)                 # the rejections touched nothing
    _rejects(w.sparse_set_data, Xw, np.zeros((300, 1025)))


def test_launch_counts():
    f = _ffi()
    parts = [("rbf", True, 0, [0, 1, 2], 1.0, [1.0, 1.2, 0.8])]
    counts = {}
    for N, P in [(1025, 12), (4097, 12), (4097, 300)]:
        X, Y, Z = _wide_problem(N, 200, P, 9)
        e = f.Engine(0)
        e.set_option("sparse_wide", 1)
        e.sparse_set_data(X, Y)
        n0 = e.total_launches()
        e.sparse_eval_multi(parts, Z, 0.1)
        n1 = e.total_launches()
        e.sparse_grad_X()
        counts[(N, P)] = (n1 - n0, e.total_launches() - n1)
    assert {c[1] for c in counts.values()} == {2}
    assert len({c[0] for c in counts.values()}) == 1, counts

