"""CPU tests of FITC: the NumPy restatement (tests/fitc_oracle.py) against the reference's own FITC (the committed
fixtures everywhere, the live reference where its tree exists), and the routing of the mirror's gpy_b200.FITC and the
plugin's B.FITC on test doubles of the engine: the entry called, its arguments, the reference's exceptions, and the
reference's own SparseGP over B.FITC against the stock pair."""
import glob
import os
import types

import numpy as np
import pytest

import fitc_oracle as fo

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = sorted(glob.glob(os.path.join(HERE, "golden", "fitc", "*.npz")))
HAVE_REF = os.path.isdir(os.environ.get("GPX_REFERENCE", "/root/reference") + "/GPy")


def _name(path):
    return os.path.basename(path)[:-4]


def test_every_case_has_a_fixture():
    assert sorted(_name(p) for p in FIXTURES) == sorted(fo.CASES)


@pytest.mark.parametrize("path", FIXTURES, ids=_name)
def test_oracle_matches_the_reference_fixture(path):
    f = np.load(path)
    parts = fo.CASES[_name(path)][0]
    lml, grad, Zgrad, res = fo.fitc_eval(f["X"], f["Y"], f["Z"], parts, float(f["noise"]))
    assert abs(lml - float(f["lml"])) <= 1e-12 * max(1.0, abs(float(f["lml"])))
    # the per-point and Z gradients sum terms of Kmm^-1's size in another operation order than the reference's: at
    # M = 300 (cond(Kmm) ~ 1e8) the two agree to 1e-9 of the largest entry, at M <= 129 to 1e-12
    tol = 1e-9 if f["Z"].shape[0] > 129 else 1e-12
    for got, want in ((grad, f["grad"]), (res["dL_dKdiag"], f["dL_dKdiag"]), (Zgrad, f["Zgrad"]),
                      (res["woodbury_vector"], f["woodbury_vector"])):
        np.testing.assert_allclose(got, want, rtol=tol, atol=tol * np.abs(want).max())
    mu, var = fo.predict(res, parts, f["Z"], f["Xnew"])
    np.testing.assert_allclose(mu, f["mu"], rtol=1e-12, atol=1e-12 * np.abs(f["mu"]).max())
    np.testing.assert_allclose(var, f["var"], rtol=1e-11, atol=1e-13)
    if "woodbury_inv" in f:
        for k in ("woodbury_inv", "K", "K_chol"):
            np.testing.assert_allclose(res[k], f[k], rtol=tol, atol=tol * np.abs(f[k]).max())


@pytest.mark.skipif(not HAVE_REF, reason="reference tree not present")
@pytest.mark.parametrize("name", ["rbf_ard_m129", "matern52_iso_m300", "rbf_ard_bias_white_m129"])
def test_oracle_matches_the_live_reference(name):
    from oracle import ref_gpy
    X, Y, Z, noise, Xnew = fo.case_data(name)
    parts = fo.CASES[name][0]
    r = fo.reference_fitc(ref_gpy, X, Y, Z, parts, noise, Xnew)
    lml, grad, Zgrad, res = fo.fitc_eval(X, Y, Z, parts, noise)
    assert abs(lml - r["lml"]) <= 1e-12 * abs(r["lml"])
    tol = 1e-9 if Z.shape[0] > 129 else 1e-12
    np.testing.assert_allclose(grad, r["grad"], rtol=tol, atol=tol * np.abs(r["grad"]).max())
    np.testing.assert_allclose(Zgrad, r["Zgrad"], rtol=tol, atol=tol * np.abs(r["Zgrad"]).max())
    for k in ("woodbury_inv", "K", "K_chol"):
        np.testing.assert_allclose(res[k], r[k], rtol=1e-12, atol=1e-12 * np.abs(r[k]).max())


# ---- routing on test doubles -------------------------------------------------------------------------------------------
class FakeFITCEngine(object):
    """the sparse entry points FITC needs, answered by the NumPy restatement; records every call"""

    def __init__(self, device=0):
        self.calls, self.sparse_serial = [], 0

    def sparse_set_data(self, X, Y):
        self.X, self.Y = np.array(X), np.array(Y)
        self.calls.append(("sparse_set_data", self.X.shape, self.Y.shape))

    def sparse_eval_fitc(self, parts, Z, noise):
        self.calls.append(("sparse_eval_fitc", [tuple(p) for p in parts], np.array(Z), noise))
        self.sparse_serial += 1
        ps = []
        for d in parts:
            p = dict(kind=d[0], ARD=d[1], term=d[2], dims=list(d[3]), variance=d[4])
            if d[0] not in ("white", "bias"):
                p["lengthscale"] = d[5]
            ps.append(p)
        lml, g, Zg, self.res = fo.fitc_eval(self.X, self.Y, Z, ps, noise)
        return lml, g, Zg, self.res["dL_dKdiag"]

    def sparse_eval(self, kind, ARD, variance, lengthscale, Z, noise):   # the VarDTC a new model starts with
        self.calls.append(("sparse_eval",))
        self.sparse_serial += 1
        return 0.0, np.zeros(np.size(lengthscale) + 2), np.zeros(np.shape(Z))

    def sparse_get(self, what):
        return {"woodbury_vector": self.res["woodbury_vector"], "woodbury_inv": self.res["woodbury_inv"],
                "Kmm": self.res["K"], "Lm": self.res["K_chol"]}[what]


def _data(P=1, N=40, M=9, D=2, seed=3):
    rng = np.random.default_rng(seed)
    X = rng.uniform(-2, 2, (N, D))
    Y = np.sin(X.sum(1, keepdims=True) + np.arange(P)) + 0.05 * rng.standard_normal((N, P))
    return X, Y, X[:M] + 0.01


def test_mirror_single_kernel_calls_the_fitc_entry_with_one_part():
    import gpy_b200 as gb
    X, Y, Z = _data()
    eng = FakeFITCEngine()
    kern = gb.RBF(2, variance=1.3, lengthscale=[0.7, 1.2], ARD=True)
    post, lml, gd = gb.FITC(engine=eng).inference(kern, X, Z, gb.Gaussian(variance=0.1), Y)
    name, parts, Zs, noise = eng.calls[-1]
    assert name == "sparse_eval_fitc" and noise == 0.1
    assert parts == [("rbf", True, 0, [0, 1], 1.3, parts[0][5])]
    np.testing.assert_array_equal(parts[0][5], [0.7, 1.2])
    np.testing.assert_array_equal(Zs, Z)
    want = fo.fitc_eval(X, Y, Z, [dict(kind="rbf", term=0, dims=[0, 1], variance=1.3, lengthscale=[0.7, 1.2],
                                       ARD=True)], 0.1)
    assert lml == want[0]
    assert gd["dvariance"] == want[1][0] and list(gd["dlengthscale"]) == list(want[1][1:3])
    assert gd["dL_dthetaL"] == want[1][-1]
    np.testing.assert_array_equal(gd["dZ"], want[2])
    np.testing.assert_array_equal(gd["dL_dKdiag"], want[3]["dL_dKdiag"])
    np.testing.assert_array_equal(post.woodbury_vector, want[3]["woodbury_vector"])


def test_mirror_composite_returns_part_blocks():
    import gpy_b200 as gb
    X, Y, Z = _data(D=3)
    eng = FakeFITCEngine()
    kern = gb.Add([gb.RBF(3, variance=1.1, lengthscale=1.3), gb.Bias(3, variance=0.3)])
    _, _, gd = gb.FITC(engine=eng).inference(kern, X, Z, gb.Gaussian(variance=0.1), Y)
    assert [p[0] for p in eng.calls[-1][1]] == ["rbf", "bias"]
    assert [len(b) for b in gd["part_grads"]] == [2, 1]


def test_mirror_raises_what_the_reference_raises():
    import gpy_b200 as gb
    X, Y, Z = _data()
    kern = gb.RBF(2)
    inf = gb.FITC(engine=FakeFITCEngine())
    with pytest.raises(AssertionError):
        inf.inference(kern, X, Z, gb.Gaussian(variance=0.1), Y, mean_function=object())
    het = gb.HeteroscedasticGaussian({"output_index": np.arange(X.shape[0])[:, None]})
    with pytest.raises(NotImplementedError, match="no hetero noise"):
        inf.inference(kern, X, Z, het, Y, Y_metadata={"output_index": np.arange(X.shape[0])[:, None]})
    with pytest.raises(ValueError):
        inf.inference(kern, X, Z, gb.Gaussian(variance=0.1), np.hstack([Y, Y]))
    assert not any(c[0] == "sparse_eval_fitc" for c in inf.engine.calls)


def test_mirror_model_passes_y_metadata_by_keyword():
    """SparseGPRegression.parameters_changed must not land Y_metadata in FITC's mean_function slot"""
    import gpy_b200 as gb
    X, Y, Z = _data()
    m = gb.SparseGPRegression(X, Y, Z=Z, engine=FakeFITCEngine())
    m.inference_method = gb.FITC(engine=FakeFITCEngine())
    m.parameters_changed()
    assert m.inference_method.engine.calls[-1][0] == "sparse_eval_fitc"


def _plugin():
    from oracle import ref_gpy
    from gpy_b200 import gpy_plugin
    import importlib
    S = ref_gpy.load_sparse_models()
    C = ref_gpy.load_combination()
    G = S.G
    FITC = importlib.import_module("GPy.inference.latent_function_inference.fitc").FITC
    from test_periodic_ratquad_plugin_cpu import fake_ffi
    f = fake_ffi()
    ffi = types.SimpleNamespace(kern_K=f.kern_K, kern_Kdiag=f.kern_Kdiag, kern_grad_full=f.kern_grad_full,
                                kern_part_K=f.kern_part_K, kern_part_grad_full=f.kern_part_grad_full,
                                Engine=FakeFITCEngine)
    B = gpy_plugin.make(G.RBF, G.Exponential, G.Matern32, G.Matern52, G.ExactGaussianInference, Add=C.Add, Prod=C.Prod,
                        VarDTC=G.VarDTC, FITC=FITC, ffi=ffi)
    return S, C, G, B, FITC


@pytest.mark.skipif(not HAVE_REF, reason="reference tree not present")
@pytest.mark.parametrize("composite", [False, True], ids=["rbf_ard", "rbf_ard_bias_white"])
def test_reference_sparse_gp_over_plugin_fitc_matches_the_stock_pair(composite):
    S, C, G, B, FITC = _plugin()
    X, Y, Z = _data(N=60, M=11, D=3)
    ls = [0.9, 1.4, 2.1]

    def kern(ns):
        k = ns.RBF(3, variance=1.3, lengthscale=ls, ARD=True)
        add = B.Add if ns is B else C.Add
        return add([k, C.Bias(3, variance=0.4), C.White(3, variance=0.07)]) if composite else k

    stock = S.SparseGP(X, Y, Z.copy(), kern(G), G.Gaussian(variance=0.08), inference_method=FITC())
    plug = S.SparseGP(X, Y, Z.copy(), kern(B), G.Gaussian(variance=0.08), inference_method=B.FITC())
    assert [c[0] for c in plug.inference_method.engine.calls] == ["sparse_set_data", "sparse_eval_fitc"]
    l_s, l_p = float(np.squeeze(stock.log_likelihood())), float(np.squeeze(plug.log_likelihood()))
    assert abs(l_p - l_s) <= 1e-10 * abs(l_s)
    gs, gp = np.asarray(stock.gradient), np.asarray(plug.gradient)
    np.testing.assert_allclose(gp, gs, rtol=1e-9, atol=1e-9 * np.abs(gs).max())
    np.testing.assert_allclose(plug.grad_dict["dL_dKdiag"], stock.grad_dict["dL_dKdiag"], rtol=1e-9, atol=1e-12)


@pytest.mark.skipif(not HAVE_REF, reason="reference tree not present")
def test_plugin_fitc_sends_anything_else_to_the_stock_method():
    S, C, G, B, FITC = _plugin()
    X, Y, Z = _data(D=3)
    inf = B.FITC()
    inf.inference(G.RBF(3), X, Z, G.Gaussian(variance=0.1), Y)                   # the reference's own kernel
    with pytest.raises(AssertionError):
        inf.inference(B.RBF(3), X, Z, G.Gaussian(variance=0.1), Y, mean_function=object())
    assert inf._engine is None or not inf.engine.calls
    inf.inference(B.RBF(3), X, Z, G.Gaussian(variance=0.1), Y)
    assert inf.engine.calls[-1][0] == "sparse_eval_fitc"
