"""The Bayesian GPLVM on the device: every reference fixture (tests/golden/make_bgplvm.py) through the C ABI
(gpx_sparse_eval_psi) and the mirror gpy_b200.BayesianGPLVM; the stand-alone psi entries; checkgrad of the mirror;
repeated calls bit for bit; every -2 rejection; launch counts that do not depend on N; a certain-input evaluation before
and after a psi evaluation; gpx_sparse_grad_X after it. Held to 1e-8 on the bound (relative to max(1, |bound|)) and 1e-6
relative on every gradient block."""
import glob
import json
import os

import numpy as np
import pytest

import bgplvm_oracle as bo

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bgplvm")
CASES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLD, "*.npz")) if not p.endswith("psi.npz"))
MARGINS = {}


def _margins_out():
    d = os.environ.get("GPX_MARGINS_DIR")
    if d:
        os.makedirs(d, exist_ok=True)
        with open(os.path.join(d, "bgplvm_margins.json"), "w") as f:
            json.dump(MARGINS, f, indent=1, sort_keys=True)


def _ffi():
    from gpy_b200 import _ffi
    return _ffi


def _load(name):
    return np.load(os.path.join(GOLD, name + ".npz"))


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.max(np.abs(a - b)) / max(np.abs(b).max(), 1e-300))


def _rbf(f):
    Q = f["mu"].shape[1]
    ard = bool(f["ard"])
    return ("rbf", ard, 0, list(range(Q)), float(f["variance"]), f["ls"] if ard else float(f["ls"][0]))


def _eval(e, f, S=None, Z=None):
    if f["Y"].shape[1] > 8:
        e.set_option("sparse_wide", 1)
    e.sparse_set_data(f["mu"], f["Y"])
    return e.sparse_eval_psi(_rbf(f), f["S"] if S is None else S, f["Z"] if Z is None else Z, float(f["noise"]))


@pytest.mark.parametrize("name", CASES)
def test_c_abi_matches_reference(name):
    f = _load(name)
    e = _ffi().Engine()
    lml, g, dZ, dmu, dS = _eval(e, f)
    m = {"lml": abs(lml - float(f["lml"])) / max(1.0, abs(float(f["lml"]))), "grad": _rel(g, f["grad"]),
         "dZ": _rel(dZ, f["dZ"]), "dmu": _rel(dmu, f["dmu"]), "dS": _rel(dS, f["dS"])}
    mu, var = e.sparse_predict(f["Xnew"])
    m["pred_mu"] = _rel(mu, f["pred_mu"])
    m["pred_var"] = _rel(var.reshape(-1, 1), f["pred_var"])
    m["woodbury_vector"] = _rel(e.sparse_get("woodbury_vector"), f["woodbury_vector"])
    MARGINS["abi_" + name] = m
    _margins_out()
    assert m["lml"] <= 1e-8, m
    for k, v in m.items():
        assert v <= 1e-6, (k, m)


@pytest.mark.parametrize("name", CASES)
def test_mirror_matches_reference(name):
    import gpy_b200
    f = _load(name)
    Q = f["mu"].shape[1]
    ard = bool(f["ard"])
    kern = gpy_b200.RBF(Q, variance=float(f["variance"]), lengthscale=f["ls"] if ard else float(f["ls"][0]), ARD=ard)
    m = gpy_b200.BayesianGPLVM(f["Y"], Q, X=f["mu"], X_variance=f["S"], Z=f["Z"], kernel=kern, num_inducing=len(f["Z"]))
    m.likelihood.variance[:] = float(f["noise"])
    bound = m.log_likelihood()
    g = m.gradient
    N = f["mu"].size
    ref = np.concatenate([(f["dmu"] + f["kl_mu"]).ravel(), (f["dS"] + f["kl_S"]).ravel(), f["dZ"].ravel(), f["grad"]])
    mm = {"bound": abs(bound - float(f["bound"])) / max(1.0, abs(float(f["bound"]))),
          "mu": _rel(g[:N], ref[:N]), "S": _rel(g[N:2 * N], ref[N:2 * N]), "rest": _rel(g[2 * N:], ref[2 * N:])}
    MARGINS["mirror_" + name] = mm
    _margins_out()
    assert mm["bound"] <= 1e-8, mm
    for k, v in mm.items():
        assert v <= 1e-6, (k, mm)
    mu, var = m.predict(f["Xnew"], include_likelihood=False)
    assert _rel(mu, f["pred_mu"]) <= 1e-6 and _rel(var, f["pred_var"]) <= 1e-6


@pytest.mark.parametrize("tag", ["ard", "iso"])
def test_standalone_psi_entries(tag):
    f = _load("psi")
    e = _ffi().Engine()
    Q = f["mu"].shape[1]
    rbf = ("rbf", tag == "ard", 0, list(range(Q)), float(f["variance"]), f["ls"] if tag == "ard" else float(f["ls"][0]))
    p0, p1, p2 = e.psi_stats(rbf, f["mu"], f["S"], f["Z"])
    g, dZ, dmu, dS = e.psi_grads(rbf, f["mu"], f["S"], f["Z"], f["dL0"], f["dL1"], f["dL2"])
    m = {"psi0": _rel(p0, f["psi0_" + tag]), "psi1": _rel(p1, f["psi1_" + tag]), "psi2": _rel(p2, f["psi2_" + tag]),
         "grad": _rel(g, f["grad_" + tag]), "dZ": _rel(dZ, f["dZ_" + tag]), "dmu": _rel(dmu, f["dmu_" + tag]),
         "dS": _rel(dS, f["dS_" + tag])}
    MARGINS["psi_" + tag] = m
    _margins_out()
    for k, v in m.items():
        assert v <= 1e-9, (k, m)
    assert np.array_equal(p2, p2.T)


def test_repeated_calls_bit_for_bit():
    f = _load("n1300_m129")
    e = _ffi().Engine()
    a = _eval(e, f)
    b = _eval(e, f)
    assert a[0] == b[0]
    for x, y in zip(a[1:], b[1:]):
        assert np.array_equal(x, y)
    rbf = _rbf(f)
    s1 = e.psi_stats(rbf, f["mu"], f["S"], f["Z"])
    s2 = e.psi_stats(rbf, f["mu"], f["S"], f["Z"])
    assert np.array_equal(s1[1], s2[1]) and np.array_equal(s1[2], s2[2])


def test_certain_eval_unchanged_around_psi_eval():
    f = _load("default_p8")
    e = _ffi().Engine()
    e.sparse_set_data(f["mu"], f["Y"])
    ls = f["ls"]
    a = e.sparse_eval("rbf", True, float(f["variance"]), ls, f["Z"], float(f["noise"]))
    e.sparse_eval_psi(_rbf(f), f["S"], f["Z"], float(f["noise"]))
    b = e.sparse_eval("rbf", True, float(f["variance"]), ls, f["Z"], float(f["noise"]))
    assert a[0] == b[0] and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


def test_grad_X_rejected_after_psi_eval():
    f = _load("default_p1")
    L = _ffi().lib()
    e = _ffi().Engine()
    e.sparse_set_data(f["mu"], f["Y"])
    e.sparse_eval("rbf", True, float(f["variance"]), f["ls"], f["Z"], float(f["noise"]))
    e.sparse_grad_X()
    e.sparse_eval_psi(_rbf(f), f["S"], f["Z"], float(f["noise"]))
    dX = np.empty(f["mu"].shape)
    assert L.gpx_sparse_grad_X(e._h, dX.ctypes.data_as(_ffi()._dp)) == -2


def test_rejections():
    ffi = _ffi()
    f = _load("default_p1")
    e = ffi.Engine()
    e.sparse_set_data(f["mu"], f["Y"])
    Q = f["mu"].shape[1]
    with pytest.raises(ffi.GpxError):   # another kernel
        e.sparse_eval_psi(("matern32", True, 0, list(range(Q)), 1.0, f["ls"]), f["S"], f["Z"], 0.1)
    with pytest.raises(ffi.GpxError):   # not on the columns 0 .. Q-1 in order
        e.sparse_eval_psi(("rbf", True, 0, [1, 0, 2], 1.0, f["ls"]), f["S"], f["Z"], 0.1)
    for bad in (0.0, -1.0, np.nan, np.inf):
        S = f["S"].copy()
        S[3, 1] = bad
        with pytest.raises(ffi.GpxError):
            e.sparse_eval_psi(_rbf(f), S, f["Z"], 0.1)
        with pytest.raises(ffi.GpxError):
            e.psi_stats(_rbf(f), f["mu"], S, f["Z"])
    L = ffi.lib()
    lml = np.zeros(1)
    g, dZ = np.zeros(5), np.zeros(f["Z"].shape)
    dmu = np.zeros(f["mu"].shape)
    arr = (ffi.GpxKernPart * 1)()
    keep = []
    ffi._fill_part(arr[0], _rbf(f), keep)
    p = ffi._ptr
    S, Z = np.ascontiguousarray(f["S"]), np.ascontiguousarray(f["Z"])
    assert L.gpx_sparse_eval_psi(e._h, arr, 1, None, p(Z), len(Z), 0.1, p(lml), p(g), p(dZ), p(dmu), p(dmu)) == -2
    assert L.gpx_sparse_eval_psi(e._h, arr, 1, p(S), p(Z), len(Z), 0.1, p(lml), p(g), p(dZ), None, p(dmu)) == -2
    assert L.gpx_sparse_eval_psi(e._h, arr, 2, p(S), p(Z), len(Z), 0.1, p(lml), p(g), p(dZ), p(dmu), p(dmu)) == -2
    e2 = ffi.Engine()   # no data set
    assert L.gpx_sparse_eval_psi(e2._h, arr, 1, p(S), p(Z), len(Z), 0.1, p(lml), p(g), p(dZ), p(dmu), p(dmu)) == -2


def test_launch_counts_do_not_depend_on_N():
    f = _load("default_p1")
    counts = []
    for N in (60, 600, 6000):
        rng = np.random.default_rng(N)
        mu = rng.uniform(-1.5, 1.5, size=(N, 3))
        S = rng.uniform(0.05, 0.3, size=(N, 3))
        Y = np.sin(mu[:, :1])
        e = _ffi().Engine()
        e.sparse_set_data(mu, Y)
        e.sparse_eval_psi(_rbf(f), S, f["Z"], 0.1)   # warm: allocations
        t0 = e.total_launches()
        e.sparse_eval_psi(_rbf(f), S, f["Z"], 0.1)
        counts.append(e.total_launches() - t0)
    assert counts[0] == counts[1] == counts[2], counts
    MARGINS["launches"] = counts[0]
    _margins_out()


def test_mirror_checkgrad_and_optimise():
    import gpy_b200
    f = _load("default_p1")
    Y = f["Y"][:30]
    np.random.seed(3)
    m = gpy_b200.BayesianGPLVM(Y, 2, num_inducing=6)
    assert m.checkgrad(tolerance=1e-4)
    b0 = -m.log_likelihood()
    m.optimize(max_iters=5)
    assert -m.log_likelihood() < b0


def test_more_rejections():
    ffi = _ffi()
    L = ffi.lib()
    p = ffi._ptr
    f = _load("psi")
    mu, S, Z = (np.ascontiguousarray(f[k]) for k in ("mu", "S", "Z"))
    N, Q = mu.shape
    M = len(Z)
    arr = (ffi.GpxKernPart * 1)()
    keep = []
    ffi._fill_part(arr[0], ("rbf", True, 0, list(range(Q)), 1.0, f["ls"]), keep)
    p1, p2 = np.zeros((N, M)), np.zeros((M, M))
    d0, d1, d2 = (np.ascontiguousarray(f[k]) for k in ("dL0", "dL1", "dL2"))
    g, dZ, dmu, dS = np.zeros(Q + 1), np.zeros((M, Q)), np.zeros((N, Q)), np.zeros((N, Q))
    e = ffi.Engine()
    assert L.gpx_psi_stats(None, arr, p(mu), p(S), N, p(Z), M, Q, p(p1), p(p2)) == -2                  # no context
    assert L.gpx_psi_stats(e._h, arr, p(mu), p(S), N, p(Z), M, Q, None, p(p2)) == -2
    assert L.gpx_psi_grads(None, arr, p(mu), p(S), N, p(Z), M, Q, p(d0), p(d1), p(d2), p(g), p(dZ), p(dmu),
                           p(dS)) == -2
    for i in range(3):                                                    # a null dL_dpsi
        ds = [p(d0), p(d1), p(d2)]
        ds[i] = None
        assert L.gpx_psi_grads(e._h, arr, p(mu), p(S), N, p(Z), M, Q, *ds, p(g), p(dZ), p(dmu), p(dS)) == -2
    assert L.gpx_psi_grads(e._h, arr, p(mu), p(S), N, p(Z), M, Q, p(d0), p(d1), p(d2), p(g), p(dZ), None, p(dS)) == -2
    m32 = (ffi.GpxKernPart * 1)()
    ffi._fill_part(m32[0], ("matern32", True, 0, list(range(Q)), 1.0, f["ls"]), keep)
    assert L.gpx_psi_grads(e._h, m32, p(mu), p(S), N, p(Z), M, Q, p(d0), p(d1), p(d2), p(g), p(dZ), p(dmu),
                           p(dS)) == -2
    assert L.gpx_psi_stats(e._h, m32, p(mu), p(S), N, p(Z), M, Q, p(p1), p(p2)) == -2
    # more than 16 latent columns
    Q2 = 17
    mu2, S2, Z2 = np.zeros((N, Q2)), np.ones((N, Q2)), np.zeros((M, Q2))
    wide = (ffi.GpxKernPart * 1)()
    ffi._fill_part(wide[0], ("rbf", False, 0, list(range(Q2)), 1.0, 1.0), keep)
    assert L.gpx_psi_stats(e._h, wide, p(mu2), p(S2), N, p(Z2), M, Q2, p(p1), p(p2)) == -2
    e.sparse_set_data(mu2, np.ones((N, 1)))
    with pytest.raises(ffi.GpxError):
        e.sparse_eval_psi(("rbf", False, 0, list(range(Q2)), 1.0, 1.0), S2, Z2, 0.1)
    assert L.gpx_sparse_eval_psi(None, arr, 1, p(S), p(Z), M, 0.1, p(g), p(g), p(dZ), p(dmu), p(dS)) == -2
