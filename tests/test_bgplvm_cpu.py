"""The NumPy restatement of the Bayesian GPLVM (tests/bgplvm_oracle.py) against the reference's own fixtures and against
central differences of its own bound. No GPU needed."""
import glob
import os

import numpy as np
import pytest

import bgplvm_oracle as bo

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bgplvm")
CASES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLD, "*.npz")) if not p.endswith("psi.npz"))


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.max(np.abs(a - b) / np.maximum(np.abs(b), 1e-300 + np.max(np.abs(b)) * 1e-6)))


def test_every_case_has_a_fixture():
    assert sorted(bo.CASES) == CASES


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference(name):
    f = np.load(os.path.join(GOLD, name + ".npz"))
    mu, S, Z, Y, Xnew = bo.case_inputs(bo.CASES[name])
    for k, v in (("mu", mu), ("S", S), ("Z", Z), ("Y", Y), ("Xnew", Xnew)):
        np.testing.assert_array_equal(f[k], v)
    r = bo.vardtc_psi(float(f["variance"]), f["ls"], bool(f["ard"]), Z, mu, S, Y, float(f["noise"]))
    assert abs(r["lml"] - float(f["lml"])) <= 1e-8 * max(1.0, abs(float(f["lml"])))
    for k in ("grad", "dZ", "dmu", "dS"):
        assert _rel(r[k], f[k]) <= 1e-6, k
    k, gmu, gS = bo.kl(mu, S)
    assert abs((r["lml"] - k) - float(f["bound"])) <= 1e-8 * max(1.0, abs(float(f["bound"])))
    np.testing.assert_allclose(gmu, f["kl_mu"], rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(gS, f["kl_S"], rtol=1e-12, atol=1e-14)


@pytest.mark.parametrize("tag", ["ard", "iso"])
def test_psi_oracle_matches_reference(tag):
    f = np.load(os.path.join(GOLD, "psi.npz"))
    ls = f["ls"] if tag == "ard" else f["ls"][:1]
    p0, p1, p2 = bo.psi_stats(float(f["variance"]), ls, f["Z"], f["mu"], f["S"])
    np.testing.assert_allclose(p0, f["psi0_" + tag], rtol=1e-14)
    np.testing.assert_allclose(p1, f["psi1_" + tag], rtol=1e-12)
    np.testing.assert_allclose(p2, f["psi2_" + tag], rtol=1e-12)
    g, dZ, dmu, dS = bo.psi_derivs(f["dL0"], f["dL1"], f["dL2"], float(f["variance"]), ls, f["Z"], f["mu"], f["S"],
                                   tag == "ard")
    for k, v in (("grad", g), ("dZ", dZ), ("dmu", dmu), ("dS", dS)):
        assert _rel(v, f[k + "_" + tag]) <= 1e-9, k


@pytest.mark.parametrize("ard", [True, False])
def test_restated_bound_central_differences(ard):
    c = dict(bo.CASES["default_p1"], N=15, M=5, P=2, ard=ard, ls=[0.9, 1.3, 1.7] if ard else [1.2])
    mu, S, Z, Y, _ = bo.case_inputs(c)
    theta = dict(variance=1.1, ls=np.array(c["ls"]), noise=0.07)

    def f(mu, S, Z, variance, ls, noise):
        return bo.bgplvm_eval(variance, ls, ard, Z, mu, S, Y, noise)

    b, g = f(mu, S, Z, **theta)
    flat = [mu, S, Z, np.array([theta["variance"]]), theta["ls"], np.array([theta["noise"]])]
    sizes = [a.size for a in flat]
    x0 = np.concatenate([a.ravel() for a in flat])

    def unpack(x):
        out, o = [], 0
        for a, n in zip(flat, sizes):
            out.append(x[o:o + n].reshape(a.shape))
            o += n
        return out

    def fx(x):
        m, s, z, v, l, nz = unpack(x)
        return f(m, s, z, float(v[0]), l, float(nz[0]))[0]

    rng = np.random.default_rng(3)
    for i in rng.choice(x0.size, 25, replace=False):
        h = 1e-6 * max(1.0, abs(x0[i]))
        if i >= mu.size and i < mu.size + S.size:
            h = 1e-3 * x0[i]
        e = np.zeros_like(x0)
        e[i] = h
        fd = (fx(x0 + e) - fx(x0 - e)) / (2 * h)
        assert abs(fd - g[i]) <= 1e-5 * max(1.0, abs(g[i])), (i, fd, g[i])
