"""SVGP on the host: the NumPy restatement (tests/svgp_oracle.py) against the reference's own SVGP.inference with the
gradient wiring of core/svgp.py, the mirror likelihoods' variational_expectations against the reference's, and the
mirror's rejections. The reference runs through oracle/ref_gpy.py where its tree exists; those tests skip elsewhere."""
import importlib
import os
import sys
import types

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), HERE, os.path.join(HERE, "golden")]

import svgp_oracle as so  # noqa: E402
import gpy_b200  # noqa: E402
from gpy_b200.svgp import SVGPInference, flat_to_triang, triang_to_flat  # noqa: E402

HAVE_REF = os.path.isdir(os.environ.get("GPX_REFERENCE", "/root/reference"))
needs_ref = pytest.mark.skipif(not HAVE_REF, reason="the reference tree is not present")


def _ref():
    from ep_reference import load_reference_ep
    load_reference_ep()
    import make_laplace as ml
    lik = types.SimpleNamespace(Bernoulli=importlib.import_module("GPy.likelihoods.bernoulli").Bernoulli,
                                StudentT=importlib.import_module("GPy.likelihoods.student_t").StudentT,
                                Gaussian=importlib.import_module("GPy.likelihoods.gaussian").Gaussian)
    return importlib.import_module("GPy.inference.latent_function_inference.svgp"), ml, lik


def reference_eval(name):
    """the reference's SVGP.inference and core/svgp.py:53-62 for one case -> (lml, grad, dZ, gd, post)"""
    svgp, ml, mods = _ref()
    parts, lik_spec, N, M, seed, opts = so.CASES[name]
    X, Y, Z, q_m, q_L, Xnew, bs = so.case_data(name)
    kern = ml.reference_kernel(parts, X.shape[1])
    if lik_spec == "poisson":
        lik = importlib.import_module("GPy.likelihoods.poisson").Poisson()
    else:
        lik = so.make_likelihood(lik_spec, mods)
    post, lml, gd = svgp.SVGP().inference(q_m[:, None], triang_to_flat(q_L)[:, None], kern, X, Z, lik, Y,
                                          batch_scale=bs)
    kern.update_gradients_full(gd["dL_dKmm"], Z)
    g = kern.gradient.copy()
    kern.update_gradients_full(gd["dL_dKmn"], Z, X)
    g += kern.gradient.copy()
    kern.update_gradients_diag(gd["dL_dKdiag"], X)
    g += kern.gradient.copy()
    dZ = kern.gradients_X(gd["dL_dKmm"], Z) + kern.gradients_X(gd["dL_dKmn"], Z, X)
    mu, var = post._raw_predict(kern, Xnew, Z)
    return lml, g, dZ, gd, (mu, var)


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300)


GOLDEN = os.path.join(HERE, "golden", "svgp")


def fixture(name):
    return dict(np.load(os.path.join(GOLDEN, name + ".npz")))


def ref_bar(f):
    """restatement against the reference: rounding grows with the condition number of the matrix jitchol factored"""
    return 1e-13 * max(float(f["cond_Kmm_jit"]), 1e2)


@pytest.mark.parametrize("name", sorted(so.CASES))
def test_restatement_matches_fixtures(name):
    """the fixtures were written by the reference's own SVGP.inference (tests/golden/make_svgp.py)"""
    parts, lik_spec, N, M, seed, opts = so.CASES[name]
    X, Y, Z, q_m, q_L, Xnew, bs = so.case_data(name)
    f = fixture(name)
    o = so.svgp_eval(parts, X, Y, Z, q_m, q_L, so.make_likelihood(lik_spec, gpy_b200), bs, Xnew)
    assert abs(o["jitter"] - float(f["jitter"])) <= 1e-12 * np.mean(np.abs(o["mu"]) + 1.0)
    bar = ref_bar(f)
    assert bar <= 1e-5, "the case must stay well-conditioned enough to test something"
    assert abs(o["lml"] - float(f["lml"])) <= bar * max(abs(float(f["lml"])), 1.0)
    for k in ("mu", "v", "pmu", "pvar", "dL_dm"):
        assert _rel(o[k], f[k]) <= bar, (k, _rel(o[k], f[k]), bar)
    for k in ("grad", "dZ"):   # dL_dKmm carries Kmm^-1 S Kmm^-1: ten times the bar
        assert _rel(o[k], f[k]) <= 10 * bar, (k, _rel(o[k], f[k]), bar)
    if f["dL_dthetaL"].size:
        assert _rel(o["dL_dthetaL"], f["dL_dthetaL"]) <= bar
    # dL_dchol: the no-S^-1 form against the reference's dpotri form; the reference leaves cond(S) eps noise in the
    # entries that are exactly zero in the other form
    ref = f["dL_dchol"]
    assert np.max(np.abs(triang_to_flat(o["dL_dchol"]) - ref)) <= \
        1e-13 * max(float(f["cond_Kmm_jit"]), float(f["cond_S"]), 1e2) * max(np.max(np.abs(ref)), 1.0)


def test_zero_diagonal_fixture_and_restatement():
    """the reference's bound with a zero on q_u_chol's diagonal is -inf, without an exception; so is the restatement's"""
    f = fixture("bernoulli_zero_diag")
    assert float(f["lml"]) == -np.inf
    parts, lik_spec, N, M, seed, opts = so.CASES["bernoulli_rbf_iso"]
    X, Y, Z, q_m, q_L, Xnew, bs = so.case_data("bernoulli_rbf_iso")
    q_L[3, 3] = 0.0
    with np.errstate(divide="ignore", invalid="ignore"):
        o = so.svgp_eval(parts, X, Y, Z, q_m, q_L, gpy_b200.Bernoulli())
    assert o["lml"] == -np.inf


def test_studentt_dF_dv_is_not_the_derivative_of_the_quadrature():
    """why checkgrad on everything that moves v cannot be tight with StudentT: the reference's dF_dv = E[d2 log p] / 2
    on the 20-point rule differs from d/dv of the same rule's F, while the Gaussian's closed form agrees"""
    rng = np.random.default_rng(0)
    Y, m = rng.standard_normal((40, 1)), rng.standard_normal((40, 1))
    v = rng.uniform(0.2, 1.0, (40, 1))
    for lik, lo, hi in ((gpy_b200.Gaussian(variance=0.3), 0.0, 1e-7), (gpy_b200.StudentT(deg_free=4.0, sigma2=0.1), 1e-2,
                                                                      np.inf)):
        _, _, dv, _ = lik.variational_expectations(Y, m, v)
        fd = (lik.variational_expectations(Y, m, v + 1e-6)[0] - lik.variational_expectations(Y, m, v - 1e-6)[0]) / 2e-6
        err = np.max(np.abs(fd - dv)) / np.max(np.abs(fd))
        assert lo <= err <= hi, (type(lik).__name__, err)


@needs_ref
@pytest.mark.parametrize("spec", ["bernoulli", "gaussian", ("studentt", 3.0, 0.05)])
def test_variational_expectations_bit_identical(spec):
    _, _, mods = _ref()
    rng = np.random.default_rng(7)
    m = rng.standard_normal((57, 1))
    v = rng.uniform(0.01, 2.0, (57, 1))
    Y = (rng.standard_normal((57, 1)) > 0).astype(float) if spec == "bernoulli" else rng.standard_normal((57, 1))
    ours = so.make_likelihood(spec, gpy_b200).variational_expectations(Y, m, v)
    theirs = so.make_likelihood(spec, mods).variational_expectations(Y, m, v)
    for a, b in zip(ours, theirs):
        if b is None:
            assert a is None
        else:
            assert np.array_equal(np.asarray(a), np.asarray(b))


@needs_ref
def test_reference_zero_diagonal_bound():
    """what the reference does with a zero on q_u_chol's diagonal: no exception, the bound is -inf"""
    svgp, ml, mods = _ref()
    X, Y, Z, q_m, q_L, Xnew, bs = so.case_data("bernoulli_rbf_iso")
    q_L = q_L.copy()
    q_L[3, 3] = 0.0
    kern = ml.reference_kernel(so.CASES["bernoulli_rbf_iso"][0], X.shape[1])
    with np.errstate(divide="ignore"):
        _, lml, _ = svgp.SVGP().inference(q_m[:, None], triang_to_flat(q_L)[:, None], kern, X, Z, mods.Bernoulli(), Y)
    assert lml == -np.inf


def test_no_si_dchol_is_the_dpotri_form():
    """lower(S^-1 L) = diag(1 / L_ii): the restatement's two forms of dL_dchol agree on a well-conditioned case"""
    parts, lik_spec, N, M, seed, opts = so.CASES["bernoulli_rbf_ard"]
    X, Y, Z, q_m, q_L, Xnew, bs = so.case_data("bernoulli_rbf_ard")
    o = so.svgp_eval(parts, X, Y, Z, q_m, q_L, gpy_b200.Bernoulli(), bs)
    assert _rel(o["dL_dchol"], o["dL_dchol_ref"]) <= 1e-13 * max(o["cond_Kmm"], o["cond_S"])


def test_flat_triangle_round_trip():
    L = np.tril(np.arange(1.0, 17.0).reshape(4, 4))
    assert np.array_equal(flat_to_triang(triang_to_flat(L), 4), L)
    assert np.array_equal(triang_to_flat(L), L[np.tril_indices(4)])


class _NoDevice(object):
    """an engine that must not be reached: the rejections happen before any device call"""

    def __getattr__(self, name):
        raise AssertionError("the engine was used")


def _inputs(M=5, N=20, D=3):
    rng = np.random.default_rng(1)
    return (np.zeros((M, 1)), triang_to_flat(np.eye(M))[:, None], rng.uniform(size=(N, D)), rng.uniform(size=(M, D)),
            (rng.uniform(size=(N, 1)) > 0.5).astype(float))


def test_rejections():
    inf = SVGPInference(engine=_NoDevice())
    m, ch, X, Z, Y = _inputs()
    k = gpy_b200.RBF(3)
    lik = gpy_b200.Bernoulli()
    with pytest.raises(NotImplementedError):
        inf.inference(m, ch, k, X, Z, lik, Y, mean_function=object())
    with pytest.raises(NotImplementedError):
        inf.inference(np.zeros((5, 2)), np.hstack([ch, ch]), k, X, Z, lik, np.hstack([Y, Y]))
    with pytest.raises(NotImplementedError):
        inf.inference(m, ch, gpy_b200.RatQuad(3), X, Z, lik, Y)
    with pytest.raises(ValueError):
        inf.inference(m[:4], ch, k, X, Z, lik, Y)
    tiny = flat_to_triang(ch[:, 0], 5)
    tiny[2, 2] = 1e-200
    with pytest.raises(ValueError, match="Cholesky representation unstable"):
        inf.inference(m, triang_to_flat(tiny)[:, None], k, X, Z, lik, Y)
    with pytest.raises(NotImplementedError):
        gpy_b200.SVGP(X, np.hstack([Y, Y]), Z, k, lik, engine=_NoDevice())
    with pytest.raises(NotImplementedError):
        gpy_b200.SVGP(X, Y, Z, k, lik, mean_function=object(), engine=_NoDevice())
