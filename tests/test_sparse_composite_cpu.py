"""Sparse GP regression (VarDTC) with composite kernels, without a GPU: the NumPy restatement of
tests/sparse_composite_oracle.py against the reference's own objects (the committed fixtures of
tests/golden/sparse_composite, and a live run where the reference tree exists) and against finite differences; the
mirror's VarDTC / SparseGPRegression host logic on a test double of the engine that answers from that restatement."""
import glob
import os

import numpy as np
import pytest

import gpy_b200
import sparse_composite_oracle as so

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = sorted(glob.glob(os.path.join(HERE, "golden", "sparse_composite", "*.npz")))
HAVE_REF = os.path.isdir(os.environ.get("GPX_REFERENCE", "/root/reference") + "/GPy")


def _noise(f):
    n = f["noise"]
    return float(n) if n.ndim == 0 else n


def test_fixture_set_covers_the_three_kernels_both_noise_forms_and_two_outputs():
    names = {os.path.basename(p)[:-4] for p in FIXTURES}
    assert names == {"%s_p%d_%s" % (k, P, n) for k in so.KERNELS for P in (1, 2) for n in ("scalar", "het")}


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[:-4])
def test_oracle_matches_the_reference_fixtures(path):
    f = np.load(path)
    lml, grad, Zg, res = so.sparse_composite_eval(f["X"], f["Y"], f["Z"], so.KERNELS[str(f["kernel"])], _noise(f))
    assert abs(lml - float(f["lml"])) <= 1e-12 * abs(float(f["lml"]))
    np.testing.assert_allclose(grad, f["grad"], rtol=1e-11, atol=1e-12 * np.abs(f["grad"]).max())
    np.testing.assert_allclose(Zg, f["Zgrad"], rtol=1e-11, atol=1e-12 * np.abs(f["Zgrad"]).max())
    np.testing.assert_allclose(res["woodbury_vector"], f["woodbury_vector"], rtol=1e-11, atol=1e-13)
    if "dL_dR" in f.files:
        np.testing.assert_allclose(res["dL_dthetaL"], f["dL_dR"], rtol=1e-11, atol=1e-12 * np.abs(f["dL_dR"]).max())


@pytest.mark.skipif(not HAVE_REF, reason="reference tree not present")
def test_oracle_matches_the_reference_objects_live():
    """a case the fixtures do not hold: four terms, shared columns, White inside a product"""
    import importlib.util
    spec = importlib.util.spec_from_file_location("mk_sc", os.path.join(HERE, "golden", "make_sparse_composite.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    from oracle import ref_gpy
    S, C = ref_gpy.load_sparse_models(), ref_gpy.load_combination()
    parts = [dict(kind="rbf", term=0, dims=[0, 2], variance=0.7, lengthscale=[1.1, 0.8], ARD=True),
             dict(kind="white", term=0, variance=0.5),
             dict(kind="matern32", term=1, dims=[1], variance=0.6, lengthscale=0.9),
             dict(kind="rbf", term=1, dims=[0, 1, 2], variance=1.2, lengthscale=1.6),
             dict(kind="bias", term=2, variance=0.3),
             dict(kind="exponential", term=3, dims=[2, 0], variance=0.4, lengthscale=[0.7, 1.9], ARD=True)]
    for het in (False, True):
        X, Y, Z, noise = so.case_data(150, 25, 3, 2, 7, het)
        r = mk.evaluate(C, S.G, X, Y, Z, parts, noise)
        lml, grad, Zg, res = so.sparse_composite_eval(X, Y, Z, parts, noise)
        assert abs(lml - r["lml"]) <= 1e-12 * abs(r["lml"])
        np.testing.assert_allclose(grad, r["grad"], rtol=1e-11, atol=1e-12 * np.abs(r["grad"]).max())
        np.testing.assert_allclose(Zg, r["Zgrad"], rtol=1e-11, atol=1e-12 * np.abs(r["Zgrad"]).max())


def _flat_theta(parts):
    th = []
    for p in parts:
        th.append(p["variance"])
        if p["kind"] not in ("white", "bias"):
            th.extend(np.atleast_1d(p["lengthscale"]).tolist())
    return np.array(th)


def _with_theta(parts, th):
    out, i = [], 0
    for p in parts:
        q = dict(p)
        q["variance"] = th[i]
        i += 1
        if p["kind"] not in ("white", "bias"):
            n = np.atleast_1d(p["lengthscale"]).size
            q["lengthscale"] = th[i:i + n].copy() if p.get("ARD") else float(th[i])
            i += n
        out.append(q)
    return out


@pytest.mark.parametrize("kname", sorted(so.KERNELS))
def test_oracle_against_finite_differences(kname):
    parts = so.KERNELS[kname]
    X, Y, Z, noise = so.case_data(60, 9, 3, 2, 3, False)
    lml, grad, Zg, _ = so.sparse_composite_eval(X, Y, Z, parts, noise)
    th = np.concatenate([_flat_theta(parts), [noise]])
    h = 1e-6
    num = []
    for i in range(th.size):
        tp, tm = th.copy(), th.copy()
        tp[i] += h * th[i]
        tm[i] -= h * th[i]
        fp = so.sparse_composite_eval(X, Y, Z, _with_theta(parts, tp[:-1]), tp[-1])[0]
        fm = so.sparse_composite_eval(X, Y, Z, _with_theta(parts, tm[:-1]), tm[-1])[0]
        num.append((fp - fm) / (2 * h * th[i]))
    np.testing.assert_allclose(grad, num, rtol=2e-5, atol=1e-5)
    for (a, d) in ((0, 0), (3, 1), (8, 2)):
        Zp, Zm = Z.copy(), Z.copy()
        Zp[a, d] += h
        Zm[a, d] -= h
        num = (so.sparse_composite_eval(X, Y, Zp, parts, noise)[0] - so.sparse_composite_eval(X, Y, Zm, parts, noise)[0]) / (2 * h)
        assert abs(num - Zg[a, d]) <= 2e-5 * max(1.0, abs(num))


# ---- the mirror on a test double of the engine ------------------------------------------------------------------
def _desc_to_part(d):
    p = dict(kind=d[0], ARD=d[1], term=d[2], dims=list(d[3]), variance=d[4])
    if d[0] not in ("white", "bias"):
        p["lengthscale"] = d[5]
    return p


class FakeEngine(object):
    def __init__(self):
        self.calls, self.sparse_serial = [], 0

    def sparse_set_data(self, X, Y):
        self.X, self.Y = np.array(X), np.array(Y)
        self.sN, self.sD = self.X.shape
        self.sP = self.Y.shape[1]
        self.calls.append("sparse_set_data")

    def sparse_eval_multi(self, parts, Z, noise):
        self.calls.append("sparse_eval_multi")
        self.sparse_serial += 1
        self.parts = [_desc_to_part(d) for d in parts]
        lml, g, Zg, self.res = so.sparse_composite_eval(self.X, self.Y, Z, self.parts, noise)
        if np.ndim(noise) > 0:
            return lml, g, Zg, self.res["dL_dthetaL"]
        return lml, g, Zg

    def sparse_get(self, what):
        return {"woodbury_vector": self.res["woodbury_vector"], "woodbury_inv": self.res["woodbury_inv"],
                "Kmm": self.res["Kmm"], "Lm": self.res["Lm"]}[what]


def _mirror_kernel():
    K = gpy_b200.kern
    return K.Add([K.Prod([K.Matern52(2, variance=1.1, lengthscale=1.2, active_dims=[0, 1]),
                          K.RBF(2, variance=0.8, lengthscale=[1.5, 0.7], ARD=True, active_dims=[1, 2])]),
                  K.Exponential(1, variance=0.3, lengthscale=2.5, active_dims=[0]),
                  K.White(3, variance=0.05)])


def test_mirror_model_parameter_order_gradient_and_one_call_per_evaluation():
    X, Y, Z, _ = so.case_data(80, 10, 3, 1, 4, False)
    eng = FakeEngine()
    m = gpy_b200.SparseGPRegression(X, Y, kernel=_mirror_kernel(), Z=Z, engine=eng)
    m.likelihood.variance[:] = 0.08
    assert eng.calls.count("sparse_set_data") == 1 and eng.calls[-1] == "sparse_eval_multi"
    parts = so.KERNELS["m52_x_rbf_plus_exp"] + [dict(kind="white", term=2, variance=0.05)]
    lml, grad, Zg, _ = so.sparse_composite_eval(X, Y, Z, parts, 0.08)
    assert abs(m.log_likelihood() - lml) <= 1e-12 * abs(lml)
    # reference link order: Z, then the kernel's leaves' parameters, then the likelihood's
    names = [p.name for p in m.flattened_parameters()]
    assert names[0] == "inducing inputs" and len(names) == 1 + 2 + 2 + 2 + 1 + 1
    g = np.concatenate([np.asarray(p.gradient, dtype=np.float64).reshape(-1) for p in m.flattened_parameters()])
    np.testing.assert_allclose(g, np.concatenate([Zg.reshape(-1), grad]), rtol=1e-12, atol=1e-12)
    assert m.checkgrad(step=1e-6, tolerance=1e-4)
    n0 = eng.calls.count("sparse_eval_multi")
    x = m.optimizer_array
    m.optimizer_array = x
    assert eng.calls.count("sparse_eval_multi") == n0 + 1
    l0 = m.log_likelihood()
    m.optimize(max_iters=8)
    assert m.log_likelihood() > l0


def test_mirror_per_point_noise_routes_dL_dR_to_the_likelihood():
    from gpy_b200.inference import HeteroscedasticGaussian
    X, Y, Z, nv = so.case_data(70, 8, 3, 1, 5, True)
    meta = {"output_index": np.arange(70)[:, None]}
    lik = HeteroscedasticGaussian(meta)
    lik.variance.values[...] = nv.reshape(lik.variance.values.shape)
    K = gpy_b200.kern
    kern = K.Add([K.RBF(3, variance=1.3, lengthscale=[0.9, 1.4, 2.1], ARD=True), K.Bias(3, variance=0.4),
                  K.White(3, variance=0.07)])
    eng = FakeEngine()
    m = gpy_b200.SparseGPRegression(X, Y, kernel=kern, Z=Z, engine=eng, likelihood=lik, Y_metadata=meta)
    lml, grad, Zg, res = so.sparse_composite_eval(X, Y, Z, so.KERNELS["rbf_bias_white"], nv)
    assert abs(m.log_likelihood() - lml) <= 1e-12 * abs(lml)
    np.testing.assert_allclose(np.asarray(m.likelihood.variance.gradient).reshape(-1), res["dL_dthetaL"].reshape(-1),
                               rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(np.asarray(m.kern.parts[0].lengthscale.gradient), grad[1:4], rtol=1e-12)


@pytest.mark.parametrize("leaf", ["ratquad", "stdperiodic"])
def test_a_composite_with_a_ratquad_or_stdperiodic_leaf_is_not_sparse(leaf):
    K = gpy_b200.kern
    new = K.RatQuad(1, active_dims=[0]) if leaf == "ratquad" else K.StdPeriodic(1, active_dims=[0])
    X, Y, Z, _ = so.case_data(30, 5, 2, 1, 6, False)
    eng = FakeEngine()
    for kern in (K.Add([K.RBF(2), new]), K.Prod([K.RBF(2), new]) + K.Bias(2)):
        with pytest.raises(NotImplementedError, match="sparse"):
            gpy_b200.sparse.VarDTC(engine=eng).inference(kern, X, Z, gpy_b200.inference.Gaussian(), Y)
    assert "sparse_eval_multi" not in eng.calls
