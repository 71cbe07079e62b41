"""Sparse EP (EPDTC) on the host: the NumPy restatement (tests/epdtc_oracle.py), per site and in the device's blocked
M-space form, against the fixtures the reference's own EPDTC wrote (tests/golden/epdtc), the drift of the blocked form,
and the mirror's host logic on a fake engine."""
import glob
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), HERE]

import epdtc_oracle as eo  # noqa: E402
from sparse_composite_oracle import CompositeOracle  # noqa: E402

FIX = os.path.join(HERE, "golden", "epdtc")
NAMES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(FIX, "*.npz")))
SITE_KEYS = ("tau_tilde", "v_tilde", "post_mu", "post_sd")


def bar(cond, blocked):
    """relative bar on the sites, the posterior mu / Sigma_diag and log Z~: 1e-12 where cond(Kmm) < 1e6 (largest measured:
    5.7e-13 per site, 4.8e-13 blocked). Past that the rounding of the reference's factorisations grows with cond(Kmm) and
    the blocked form's A = LLT^-1 with it: 0.1 cond eps per site (measured 8.4e-11 at cond 2.0e7, 3.3e-11 at 2.3e10),
    cond eps blocked (1.7e-10 and 3.7e-8)"""
    if cond < 1e6:
        return 1e-12
    return max(1e-12, (1.0 if blocked else 0.1) * cond * np.finfo(float).eps)


def rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300))


def test_fixtures_cover_the_cases():
    assert set(NAMES) == set(eo.CASES)


@pytest.mark.parametrize("blocked", [False, True])
@pytest.mark.parametrize("name", [n for n in NAMES if "ladder" not in n])
def test_oracle_matches_reference(name, blocked):
    """both forms against every fixture (the alternated ones: the sites of the run, which the second call reuses)"""
    f = np.load(os.path.join(FIX, name + ".npz"))
    r = eo.case_eval(name, blocked=blocked)
    assert list(r["sweeps"]) == list(f["sweeps"])
    assert r["next_random"] == f["next_random"]
    b = bar(float(f["cond_Kmm"]), blocked)
    for k in SITE_KEYS:
        assert rel(r[k], f[k]) <= b, (k, rel(r[k], f[k]))
    assert abs(r["log_Z_tilde"] - float(f["log_Z_tilde"])) <= b * max(1.0, abs(float(f["log_Z_tilde"])))


def test_oracle_on_the_ladder():
    """repeated inducing points make Kmm singular (cond 1.9e20) and every factorisation takes jitchol's ladder: the
    per-site form follows the reference's factorisations to 2.7e-13 (bar 1e-12); the blocked form cannot invert LLT
    there, so only the device's own bar (test_gpu_epdtc) covers it"""
    name = "rbf_iso_ladder_n150_m50"
    f = np.load(os.path.join(FIX, name + ".npz"))
    r = eo.case_eval(name, blocked=False)
    assert list(r["sweeps"]) == list(f["sweeps"])
    assert r["next_random"] == f["next_random"]
    for k in SITE_KEYS:
        assert rel(r[k], f[k]) <= 1e-12, (k, rel(r[k], f[k]))


def test_far_points_reach_the_clip():
    f = np.load(os.path.join(FIX, "rbf_iso_far_n150_m10.npz"))
    assert np.sum(f["post_sd"] <= eo.EPS) > 0


def test_blocked_drift_n8192_m512():
    """the downdates of A over one sweep of 64 blocks against the recompute's diagonal at the same sites. Measured: 5.7e-12
    of the diagonal's scale at cond(Kmm) = 1.2e4 and 1.2e-9 at cond(Kmm) = 3.9e6: the drift follows cond(Kmm) eps, as the
    recompute's own rounding does, and does not grow with the number of blocks enough to need a periodic rebuild of A"""
    rng = np.random.default_rng(7)
    N, M = 8192, 512
    X = rng.uniform(-2.0, 2.0, size=(N, eo.D))
    Z = rng.uniform(-2.0, 2.0, size=(M, eo.D))
    y = (np.sin(1.3 * X[:, 0]) + 0.6 * X[:, 1] > 0).astype(np.float64)
    kern = CompositeOracle([dict(kind="rbf", term=0, dims=[0, 1, 2], variance=1.0, lengthscale=[0.4] * 3, ARD=True)])
    Kmm, Kmn = kern.K(Z), kern.K(Z, X)
    assert np.linalg.cond(Kmm) < 1e5
    tt = rng.uniform(0.05, 2.0, N)
    vt = rng.standard_normal(N) * tt
    dA, dR = eo.blocked_drift(Kmm, Kmn, tt, vt, y, rng.permutation(N))
    assert np.max(np.abs(dA - dR)) <= 1e-10 * np.max(dR)
