"""The oracle restatement against the UNMODIFIED reference (GPy 1.14.2). What the reference returned for every case is
stored under tests/golden/reference (large matrices as a fixed, seeded sample of their entries), so the comparison runs
anywhere. With GPX_WRITE_REFERENCE_GOLDEN=1 and the reference tree present (GPX_REFERENCE, imported through
oracle/ref_gpy.py + the test-only paramz stand-in) the reference is run again and the stored files are rewritten."""
import json
import os

import numpy as np
import pytest

from oracle import gpy_oracle as o

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference")
WRITE = os.environ.get("GPX_WRITE_REFERENCE_GOLDEN") == "1"
_G = []


def G():
    """the reference's modules (only needed to rewrite the stored results)"""
    if not _G:
        from oracle import ref_gpy
        _G.append(ref_gpy.load())
    return _G[0]


def _reference(name, compute):
    """-> dict of arrays: the reference's result for this case (stored; recomputed by compute() when rewriting)"""
    path = os.path.join(GOLD, name + ".npz")
    if WRITE:
        os.makedirs(GOLD, exist_ok=True)
        np.savez_compressed(path, **{k: np.asarray(v) for k, v in compute().items()})
    with np.load(path) as z:
        return {k: z[k] for k in z.files}


def _sample(A, n=256):
    """a fixed, seeded sample of the entries of A (the same entries for every array of that size)"""
    A = np.asarray(A).reshape(-1)
    idx = np.random.default_rng(A.size).choice(A.size, min(n, A.size), replace=False)
    return A[idx]


@pytest.mark.parametrize("kind", o.KINDS)
@pytest.mark.parametrize("ARD", [False, True])
def test_oracle_equals_reference(kind, ARD):
    from oracle import ref_gpy
    for (N, D, seed) in ((60, 1, 0), (150, 4, 1), (333, 8, 2)):
        X, Y = o.synthetic(N, D, seed)
        rng = np.random.default_rng(seed)
        ls = rng.uniform(0.8, 2.5, D) if ARD else float(rng.uniform(0.8, 2.5))
        var, noise = float(rng.uniform(0.5, 2)), float(rng.uniform(0.01, 0.2))
        Xn = rng.uniform(-3, 3, (6, D))

        def compute():
            r = ref_gpy.evaluate(G(), X, Y, kind, ARD, var, ls, noise, Xn)
            return dict(lml=r["lml"], grad=r["grad"], K=_sample(r["K"]), L=_sample(r["L"]), alpha=r["alpha"],
                        dL_dK=_sample(r["dL_dK"]), mu=r["mu"], var=r["var"])
        r = _reference("exact_%s_%s_n%d" % (kind, "ard" if ARD else "iso", N), compute)
        lml, g, res = o.eval_lml_grad(X, Y, kind, ARD, var, ls, noise)
        assert abs(r["lml"] - lml) <= 1e-10 * max(1.0, abs(lml))
        np.testing.assert_allclose(g, r["grad"], rtol=1e-10, atol=1e-12)
        np.testing.assert_allclose(_sample(res["K"]), r["K"], rtol=0, atol=1e-14)
        np.testing.assert_allclose(_sample(res["L"]), r["L"], rtol=1e-12, atol=1e-14)
        np.testing.assert_allclose(res["alpha"], r["alpha"], rtol=1e-10, atol=1e-12)
        np.testing.assert_allclose(_sample(res["dL_dK"]), r["dL_dK"], rtol=1e-10, atol=1e-12)
        kern = o.StationaryOracle(kind, D, var, ls, ARD)
        mu, pv = o.predict(kern, X, res["L"], res["alpha"], Xn, noise)
        np.testing.assert_allclose(mu, r["mu"], rtol=1e-10, atol=1e-12)
        np.testing.assert_allclose(pv, r["var"], rtol=1e-9, atol=1e-12)


def test_oracle_linalg_equals_reference_linalg():
    """jitchol ladder / pdinv / tdot / symmetrify of GPy/util/linalg.py, same inputs as GPy/testing/test_linalg.py:8-18."""
    from test_oracle import _corrupt
    A = _corrupt(3)
    rng = np.random.default_rng(0)
    B = rng.standard_normal((50, 7))
    S = B.dot(B.T) + 50 * np.eye(50)

    def compute():
        g = G()
        try:
            g.linalg.jitchol(A, maxtries=4)
            raised4 = False
        except np.linalg.LinAlgError:
            raised4 = True
        Ai, Lr, Li, ld = g.linalg.pdinv(S)
        return dict(L=g.linalg.jitchol(A, maxtries=5), raised4=raised4, tdot=g.linalg.tdot(B), Ai=Ai, Lr=Lr, ld=ld)
    r = _reference("linalg", compute)
    L, jit = o.jitchol(A, maxtries=5)
    np.testing.assert_array_equal(L, r["L"])
    assert bool(r["raised4"])
    with pytest.raises(np.linalg.LinAlgError):
        o.jitchol(A, maxtries=4)
    np.testing.assert_array_equal(o.tdot(B), r["tdot"])
    Ai2, L2, Li2, ld2 = o.pdinv(S)
    np.testing.assert_array_equal(r["Ai"], Ai2)
    np.testing.assert_array_equal(r["Lr"], L2)
    assert r["ld"] == ld2


def test_reference_native_helper_matches():
    """The reference's own stationary_utils.c (compiled by oracle/Makefile into oracle/_ref) against the reference's
    NumPy reduction Stationary._lengthscale_grads_pure (stationary.py:234-235): mirrors GPy/testing/test_cython.py:83-98."""
    libs = o._load_native()
    if libs["ref"] is None:
        pytest.skip("oracle/_ref not built")
    rng = np.random.default_rng(1)
    X, Z = rng.standard_normal((300, 10)), rng.standard_normal((20, 10))
    for i, (tmp, A, B) in enumerate(((rng.standard_normal((300, 300)), X, X), (rng.standard_normal((300, 20)), X, Z))):
        g_ref = _reference("lengthscale_grads_pure_%d" % i, lambda: dict(g=G().RBF(10)._lengthscale_grads_pure(tmp, A, B)))["g"]
        g_c = o.lengthscale_grads_native(tmp, A, B, np.ones(10), "ref")
        assert np.allclose(g_ref, g_c)


def test_oracle_gradients_X_equals_reference():
    rng = np.random.default_rng(2)
    X, Z = rng.standard_normal((60, 4)), rng.standard_normal((25, 4))
    for name, kind in (("RBF", "rbf"), ("Matern32", "matern32"), ("Matern52", "matern52"), ("Exponential", "exponential")):
        for ARD in (False, True):
            ls = np.array([1.0, 1.5, 2.0, 0.8]) if ARD else 1.3
            ko = o.StationaryOracle(kind, 4, 0.9, ls, ARD)
            d1, d2 = rng.standard_normal((60, 60)), rng.standard_normal((60, 25))

            def compute():
                kr = getattr(G(), name)(4, variance=0.9, lengthscale=ls, ARD=ARD)
                return dict(gX=kr.gradients_X(d1, X), gXZ=kr.gradients_X(d2, X, Z))
            r = _reference("gradients_X_%s_%s" % (kind, "ard" if ARD else "iso"), compute)
            np.testing.assert_allclose(ko.gradients_X(d1, X), r["gX"], rtol=1e-12, atol=1e-14)
            np.testing.assert_allclose(ko.gradients_X(d2, X, Z), r["gXZ"], rtol=1e-12, atol=1e-14)


@pytest.mark.parametrize("kind", ["rbf", "matern32", "exponential"])
@pytest.mark.parametrize("ARD", [False, True])
def test_oracle_vardtc_equals_reference(kind, ARD):
    """Sparse GP regression: oracle.vardtc_inference / sparse_eval against the unmodified
    GPy/inference/latent_function_inference/var_dtc.py (+ gradient wiring of core/sparse_gp.py:108-119)."""
    from oracle import ref_gpy
    X, Y = o.synthetic(300, 3, 4)
    rng = np.random.default_rng(4)
    Z = X[rng.permutation(300)[:20]].copy()
    ls = np.array([1.2, 1.7, 2.1]) if ARD else 1.6
    def compute():
        r = ref_gpy.evaluate_sparse(G(), X, Y, Z, kind, ARD, 1.3, ls, 0.07)
        return dict(lml=r["lml"], grad=r["grad"], Zgrad=r["Zgrad"], woodbury_vector=r["woodbury_vector"],
                    woodbury_inv=r["woodbury_inv"], dL_dKnm=_sample(r["dL_dKnm"]))
    r = _reference("vardtc_%s_%s" % (kind, "ard" if ARD else "iso"), compute)
    lml, g, Zg, res = o.sparse_eval(X, Y, Z, kind, ARD, 1.3, ls, 0.07)
    assert abs(lml - r["lml"]) <= 1e-9 * abs(r["lml"])
    np.testing.assert_allclose(g, r["grad"], rtol=1e-8, atol=1e-10)
    np.testing.assert_allclose(Zg, r["Zgrad"], rtol=1e-8, atol=1e-10)
    np.testing.assert_allclose(res["woodbury_vector"], r["woodbury_vector"], rtol=1e-8, atol=1e-12)
    np.testing.assert_allclose(res["woodbury_inv"], r["woodbury_inv"], rtol=1e-7, atol=1e-10)
    np.testing.assert_allclose(_sample(res["dL_dKnm"]), r["dL_dKnm"], rtol=1e-8, atol=1e-12)


@pytest.mark.parametrize("kind,ARD,P", [("rbf", True, 1), ("matern52", False, 1), ("exponential", True, 2)])
def test_oracle_vardtc_heteroscedastic_equals_reference(kind, ARD, P):
    """Sparse GP regression with one noise variance per data point: the het_noise branches of the unmodified
    var_dtc.py (:127-128, :221-227, :241-257, :267-269) with the reference's HeteroscedasticGaussian, against
    oracle.vardtc_inference with a noise vector."""
    from oracle import ref_gpy
    rng = np.random.default_rng(14)
    N, M = 260, 24
    X = rng.uniform(-3, 3, (N, 3))
    Y = np.stack([np.sin(X).sum(1) + 0.2 * rng.standard_normal(N) for _ in range(P)], 1)
    Z = X[rng.permutation(N)[:M]].copy()
    ls = np.array([1.2, 1.7, 2.1]) if ARD else 1.6
    nv = rng.uniform(0.01, 0.4, N)
    def compute():
        r = ref_gpy.evaluate_sparse_het(G(), X, Y, Z, kind, ARD, 1.3, ls, nv)
        return {k: r[k] for k in ("lml", "grad", "Zgrad", "woodbury_vector", "woodbury_inv")}
    r = _reference("vardtc_het_%s_%s_p%d" % (kind, "ard" if ARD else "iso", P), compute)
    lml, g, Zg, res = o.sparse_eval(X, Y, Z, kind, ARD, 1.3, ls, nv)
    assert abs(lml - r["lml"]) <= 1e-9 * abs(r["lml"])
    assert g.shape == r["grad"].shape
    np.testing.assert_allclose(g, r["grad"], rtol=1e-8, atol=1e-9)
    np.testing.assert_allclose(Zg, r["Zgrad"], rtol=1e-8, atol=1e-10)
    np.testing.assert_allclose(res["woodbury_vector"], r["woodbury_vector"], rtol=1e-8, atol=1e-12)
    np.testing.assert_allclose(res["woodbury_inv"], r["woodbury_inv"], rtol=1e-7, atol=1e-10)


@pytest.mark.parametrize("kind,ARD", [("rbf", True), ("matern32", False)])
def test_oracle_heteroscedastic_equals_reference(kind, ARD):
    """One noise variance per data point: oracle restatement against the reference's HeteroscedasticGaussian +
    ExactGaussianInference objects (likelihoods/gaussian.py:347-362, models/gp_heteroscedastic_regression.py:22-37)."""
    from oracle import ref_gpy
    for (N, D, seed) in ((70, 2, 3), (211, 5, 4)):
        X, Y = o.synthetic(N, D, seed)
        rng = np.random.default_rng(seed)
        ls = rng.uniform(0.8, 2.5, D) if ARD else float(rng.uniform(0.8, 2.5))
        var = float(rng.uniform(0.5, 2))
        nv = rng.uniform(0.01, 0.3, N)
        r = _reference("exact_het_%s_%s_n%d" % (kind, "ard" if ARD else "iso", N), lambda: {
            k: v for k, v in ref_gpy.evaluate_het(G(), X, Y, kind, ARD, var, ls, nv).items() if k in ("lml", "grad", "alpha")})
        lml, g, res = o.eval_lml_grad(X, Y, kind, ARD, var, ls, nv)
        assert g.size == r["grad"].size == 1 + (D if ARD else 1) + N
        assert abs(r["lml"] - lml) <= 1e-10 * max(1.0, abs(lml))
        np.testing.assert_allclose(g, r["grad"], rtol=1e-10, atol=1e-12)
        np.testing.assert_allclose(res["alpha"], r["alpha"], rtol=1e-10, atol=1e-12)


def test_mirror_heteroscedastic_likelihood_matches_reference_class():
    """gpy_b200.inference.HeteroscedasticGaussian (host mirror) against the reference class: variance lookup, gradient
    routing and predictive values for the same Y_metadata (likelihoods/gaussian.py:347-373)."""
    from gpy_b200.inference import HeteroscedasticGaussian
    rng = np.random.default_rng(0)
    N = 17
    md = {"output_index": np.arange(N)[:, None]}
    mir = HeteroscedasticGaussian(md)
    nv = rng.uniform(0.1, 1.0, N)
    mir.variance.values[...] = nv
    sub = {"output_index": np.array([3, 0, 11])[:, None]}
    dd = rng.standard_normal(N)
    mu, var = rng.standard_normal((3, 1)), rng.uniform(0.1, 1, (3, 1))

    def compute():
        ref = G().HeteroscedasticGaussian(md)
        ref.variance[:] = nv.reshape(ref.variance.shape)
        m0, v0 = ref.predictive_values(mu.copy(), var.copy(), False, sub)
        return dict(gv=ref.gaussian_variance(sub), eig=ref.exact_inference_gradients(dd, md), m0=m0, v0=v0)
    r = _reference("heteroscedastic_likelihood", compute)
    np.testing.assert_array_equal(r["gv"].reshape(-1), mir.gaussian_variance(sub).reshape(-1))
    np.testing.assert_array_equal(r["eig"].reshape(-1), np.asarray(mir.exact_inference_gradients(dd, md)).reshape(-1))
    m0, v0 = r["m0"], r["v0"]
    m1, v1 = mir.predictive_values(mu.copy(), var.copy(), False, sub)
    np.testing.assert_allclose(np.asarray(v0).reshape(-1), np.asarray(v1).reshape(-1), rtol=0, atol=0)
    np.testing.assert_array_equal(m0, m1)


def test_mixed_noise_mirror_and_oracle_equal_reference():
    """MixedNoise (likelihoods/mixed_noise.py:14-53): the reference's own MixedNoise + ExactGaussianInference objects against
    (a) the oracle fed the per-point variance vector, with the noise gradients summed per output index, and (b) the host
    mirror class (variance lookup, gradient routing, predictive values)."""
    from oracle import ref_gpy
    from gpy_b200.inference import Gaussian, MixedNoise
    rng = np.random.default_rng(7)
    N, D = 157, 3
    X, Y = o.synthetic(N, D, 5)
    idx = rng.integers(0, 3, N)
    nl = [0.02, 0.3, 0.11]
    ls = rng.uniform(0.8, 2.5, D)
    nv = np.asarray(nl)[idx]
    lml, g, res = o.eval_lml_grad(X, Y, "matern52", True, 1.3, ls, nv)
    gk, dn = g[:1 + D], g[1 + D:]
    gsum = np.array([dn[idx == j].sum() for j in range(3)])
    sub = {"output_index": np.array([2, 0, 1, 1])[:, None]}
    mu, var = rng.standard_normal((4, 1)), rng.uniform(0.1, 1, (4, 1))

    def compute():
        r = ref_gpy.evaluate_mixed(G(), X, Y, "matern52", True, 1.3, ls, nl, idx)
        m0, v0 = r["likelihood"].predictive_values(mu.copy(), var.copy(), False, sub)
        return dict(variance=r["variance"], lml=r["lml"], grad=r["grad"], alpha=r["alpha"],
                    output_index=r["Y_metadata"]["output_index"],
                    eig=r["likelihood"].exact_inference_gradients(dn, r["Y_metadata"]), m0=m0, v0=v0)
    r = _reference("mixed_noise", compute)
    np.testing.assert_array_equal(r["variance"], nv)
    assert abs(r["lml"] - lml) <= 1e-10 * max(1.0, abs(lml))
    np.testing.assert_allclose(np.concatenate([gk, gsum]), r["grad"], rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(res["alpha"], r["alpha"], rtol=1e-10, atol=1e-12)
    mir = MixedNoise([Gaussian(v) for v in nl])
    md = {"output_index": r["output_index"]}
    np.testing.assert_array_equal(mir.gaussian_variance(md), nv)
    np.testing.assert_array_equal(mir.exact_inference_gradients(dn, md), r["eig"])
    m0, v0 = r["m0"], r["v0"]
    m1, v1 = mir.predictive_values(mu.copy(), var.copy(), False, sub)
    np.testing.assert_allclose(np.asarray(v0).reshape(-1), np.asarray(v1).reshape(-1), rtol=0, atol=0)
    np.testing.assert_array_equal(m0, m1)
    mir.update_gradients(gsum)
    np.testing.assert_allclose([float(l.variance.gradient[0]) for l in mir.likelihoods_list], gsum)


def test_cited_reference_locations_exist():
    """Every `GPy/...:line` location cited in include/gpx.h and INTEGRATION.md must exist in the reference tree (file
    present, at least that many lines) — the citations are how parity is audited. The line counts of the reference's
    files are stored in tests/golden/reference/line_counts.json."""
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    counts_path = os.path.join(GOLD, "line_counts.json")
    if WRITE:
        from oracle import ref_gpy
        counts = {}
        for dp, _, files in os.walk(os.path.join(ref_gpy.REF, "GPy")):
            for f in files:
                if f.endswith((".py", ".pyx", ".c")):
                    full = os.path.join(dp, f)
                    counts[os.path.relpath(full, ref_gpy.REF)] = sum(1 for _ in open(full, errors="replace"))
        with open(counts_path, "w") as fh:
            json.dump(counts, fh, indent=0, sort_keys=True)
    with open(counts_path) as fh:
        counts = json.load(fh)
    texts = [open(os.path.join(root, "include", "gpx.h")).read(), open(os.path.join(root, "INTEGRATION.md")).read()]
    pat = re.compile(r"(GPy/[A-Za-z0-9_/]+\.(?:py|pyx|c)):(\d+)(?:-(\d+))?")
    seen = 0
    for t in texts:
        for m in pat.finditer(t):
            assert m.group(1) in counts, m.group(0)
            last = int(m.group(3) or m.group(2))
            assert last <= counts[m.group(1)], (m.group(0), counts[m.group(1)])
            seen += 1
    assert seen >= 20


def test_composite_oracle_equals_reference_add_prod_static():
    """oracle.composite_* (restating add.py:60-99, prod.py:59-68,377-396, static.py:63-185) against the reference's own
    Add / Prod / White / Bias objects: K, Kdiag and every parameter gradient for a foreign dL_dK."""
    from oracle import ref_gpy
    rng = np.random.default_rng(5)
    N, D = 40, 5
    X = rng.uniform(-2, 2, (N, D))
    X2 = rng.uniform(-2, 2, (17, D))
    parts = [dict(kind="rbf", term=0, dims=[0, 1], variance=1.2, lengthscale=np.array([1.0, 2.0]), ARD=True),
             dict(kind="matern32", term=0, dims=[2, 3], variance=0.8, lengthscale=1.5, ARD=False),
             dict(kind="matern52", term=1, dims=list(range(D)), variance=0.5, lengthscale=np.linspace(1.5, 2.5, D), ARD=True),
             dict(kind="white", term=2, dims=None, variance=0.05), dict(kind="bias", term=3, dims=None, variance=0.3)]
    kp = o.composite_parts(parts)
    Y = np.sin(X).sum(1, keepdims=True) + 0.1 * rng.standard_normal((N, 1))

    def compute():
        C = ref_gpy.load_combination()
        G, add, prod, static = C.G, C, C, C
        k_rbf = G.RBF(2, variance=1.2, lengthscale=[1.0, 2.0], ARD=True, active_dims=[0, 1])
        k_m32 = G.Matern32(2, variance=0.8, lengthscale=1.5, active_dims=[2, 3])
        k_m52 = G.Matern52(D, variance=0.5, lengthscale=np.linspace(1.5, 2.5, D), ARD=True)
        k_w, k_b = static.White(D, variance=0.05), static.Bias(D, variance=0.3)
        kern = add.Add([prod.Prod([k_rbf, k_m32]), k_m52, k_w, k_b])
        K, KX2, Kdiag = kern.K(X), kern.K(X, X2), kern.Kdiag(X)
        # gradients: one evaluation through the reference's own inference + Add/Prod.update_gradients_full
        lik = G.Gaussian(variance=0.1)
        post, lml, gd = G.ExactGaussianInference().inference(kern, X, lik, Y)
        kern.update_gradients_full(gd["dL_dK"], X)
        k_rbf, k_m32 = kern.parts[0].parts            # Prod copies its factors (prod.py:36-41): read the linked copies
        k_m52, k_w, k_b = kern.parts[1:]
        ref_grad = np.concatenate([np.atleast_1d(k_rbf.variance.gradient), np.atleast_1d(k_rbf.lengthscale.gradient).reshape(-1),
                                   np.atleast_1d(k_m32.variance.gradient), np.atleast_1d(k_m32.lengthscale.gradient).reshape(-1),
                                   np.atleast_1d(k_m52.variance.gradient), np.atleast_1d(k_m52.lengthscale.gradient).reshape(-1),
                                   np.atleast_1d(k_w.variance.gradient), np.atleast_1d(k_b.variance.gradient),
                                   np.atleast_1d(gd["dL_dthetaL"])])
        return dict(K=K, KX2=KX2, Kdiag=Kdiag, lml=float(lml), grad=ref_grad)
    r = _reference("composite_add_prod_static", compute)
    np.testing.assert_allclose(o.composite_K(kp, X), r["K"], rtol=1e-14, atol=1e-15)
    np.testing.assert_allclose(o.composite_K(kp, X, X2), r["KX2"], rtol=1e-14, atol=1e-15)
    np.testing.assert_allclose(o.composite_Kdiag(kp, X), r["Kdiag"], rtol=1e-14)
    lml0, g0, _ = o.composite_eval_lml_grad(X, Y, parts, 0.1)
    assert abs(lml0 - float(r["lml"])) < 1e-10
    np.testing.assert_allclose(g0, r["grad"], rtol=1e-10, atol=1e-12)
