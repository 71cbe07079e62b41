"""Test-only NumPy restatement of the sparse EP (EPDTC, GPy/inference/latent_function_inference/expectation_propagation.py:
436-611) for the probit Bernoulli likelihood: the site sweeps, the recompute, log Z~ and the update orders.

`run_epdtc` follows expectation_propagation, _init_approximations, _local_updates, posteriorParamsDTC._update_rank1 and
_recompute line by line. Its sweep is either the reference's chain (`blocked=False`: LLT += dtau k_i k_i^T, jitchol, V =
L^-1 Kmn at every site) or the device's M-space form (`blocked=True`): blocks of TILE sites of the order, P = A Kmn[:, I]
with A = LLT^-1, G = Kmn[:, I]^T P, mu_I = mu0[I] + Kmn[:, I]^T u, dense EP's chain on G with the cavity on the clipped
diagonal, Y = P (I + U)^-1, u -= Y g, A -= Y diag(c) Y^T. The marginal (VarDTC at precision tau~) is not restated here;
the committed fixtures of tests/golden/epdtc were written by the reference's own EPDTC + VarDTC (tests/golden/make_epdtc.py)
and pin both the restatement and the device.
"""
import numpy as np
from scipy.linalg import lapack

from ep_oracle import EPS, TILE, moments
from laplace_oracle import COMPOSITE, D, _single, jitchol  # noqa: F401
from sparse_composite_oracle import CompositeOracle


def site(i, Sd, mui, st, y, eta, delta):
    """cavityParams._update_i, moments_match_ep and gaussianApproximation._update_i at the held Sigma_diag Sd -> (dtau, dv)"""
    st["ct"][i] = 1. / Sd - eta * st["tt"][i]
    st["cv"][i] = mui / Sd - eta * st["vt"][i]
    st["Z"][i], st["mh"][i], st["s2"][i] = moments(y[i], st["ct"][i], st["cv"][i])
    dtau = delta / eta * (1. / st["s2"][i] - 1. / Sd)
    dv = delta / eta * (st["mh"][i] / st["s2"][i] - mui / Sd)
    prev = st["tt"][i]
    st["tt"][i] += dtau
    if st["tt"][i] < EPS:
        st["tt"][i] = EPS
        dtau = st["tt"][i] - prev
    st["vt"][i] += dv
    return dtau, dv


def recompute(Kmm, Kmn, tt, vt):
    """posteriorParamsDTC._recompute (:175-185) -> (mu, Sigma_diag (unclipped), LLT)"""
    LLT = Kmm + np.dot(Kmn * tt[None, :], Kmn.T)
    L = jitchol(LLT)
    V, _ = lapack.dtrtrs(L, Kmn, lower=1)
    Sigma = np.dot(V.T, V)
    return np.dot(Sigma, vt), np.diag(Sigma).copy(), LLT


def sweep(Kmn, LLT, mu, sd, st, y, order, eta, delta, parallel, blocked):
    """_local_updates (:553-572) -> (mu, sd) as the reference holds them after the sweep"""
    if parallel:
        for i in order:
            site(i, sd[i], mu[i], st, y, eta, delta)
        return mu, sd
    if not blocked:
        LLT = LLT.copy()
        for i in order:
            dtau, dv = site(i, sd[i], mu[i], st, y, eta, delta)
            k = Kmn[:, i]
            LLT += dtau * np.outer(k, k)                                             # DSYR (lower) + jitchol's read
            L = jitchol(np.tril(LLT) + np.tril(LLT, -1).T)
            V, _ = lapack.dtrtrs(L, Kmn, lower=1)
            sd = np.maximum(np.sum(V * V, -2), EPS)
            si = np.sum(V.T * V[:, i], -1)
            mu = mu + (dv - dtau * mu[i]) * si
        return mu, sd
    A = np.linalg.inv(LLT)
    A = 0.5 * (A + A.T)
    mu0, u = mu.copy(), np.zeros(Kmn.shape[0])
    first = True
    for k0 in range(0, len(order), TILE):
        I = order[k0:k0 + TILE]
        m = len(I)
        Kb = Kmn[:, I]
        P = np.dot(A, Kb)
        G = np.dot(Kb.T, P)
        muI = mu0[I] + np.dot(Kb.T, u)
        c, g = np.zeros(m), np.zeros(m)
        R = np.zeros((m, m))
        for j in range(m):
            Sd = sd[I[0]] if (j == 0 and first) else max(G[j, j], EPS)
            dtau, dv = site(I[j], Sd, muI[j], st, y, eta, delta)
            s = G[:, j].copy()
            c[j] = dtau / (1. + dtau * s[j])
            g[j] = c[j] * (muI[j] + s[j] * dv) - dv
            muI -= g[j] * s
            G -= c[j] * np.outer(s, s)
            R[j, j + 1:] = s[j + 1:]
        first = False
        Y = np.empty_like(P)
        for j in range(m):
            Y[:, j] = P[:, j] - np.dot(Y[:, :j] * c[:j], R[:j, j])
        A = A - np.dot(Y * c, Y.T)
        u = u - np.dot(Y, g)
    mu = mu0 + np.dot(Kmn.T, u)
    return mu, np.maximum(np.einsum("an,ab,bn->n", Kmn, A, Kmn), EPS)


def blocked_drift(Kmm, Kmn, tt, vt, y, order, eta=1., delta=1.):
    """one blocked sweep from the sites (tt, vt) -> (diag(Knm A Kmn) after the last block, the recompute's diagonal) at
    the same sites: the drift the downdates of A accumulate over the sweep"""
    st = {k: np.empty(len(tt)) for k in ("ct", "cv", "Z", "mh", "s2")}
    st["tt"], st["vt"] = tt.copy(), vt.copy()
    mu, sd0, LLT = recompute(Kmm, Kmn, st["tt"], st["vt"])
    _, dA = sweep(Kmn, LLT, mu, np.maximum(sd0, EPS), st, y, order, eta, delta, False, True)
    _, dR, _ = recompute(Kmm, Kmn, st["tt"], st["vt"])
    return dA, np.maximum(dR, EPS)


def log_Z_tilde(st):
    """:514-520"""
    mu_tilde = st["vt"] / st["tt"]
    mu_cav = st["cv"] / st["ct"]
    s2 = 1. / st["ct"] + 1. / st["tt"]
    return np.sum(np.log(st["Z"]) + 0.5 * np.log(2 * np.pi) + 0.5 * np.log(s2) + 0.5 * ((mu_cav - mu_tilde) ** 2) / s2)


def run_epdtc(Kmm, Kmn, y, tt0=None, vt0=None, eta=1., delta=1., epsilon=1e-6, max_iters=np.inf, parallel=False,
              blocked=False):
    """expectation_propagation (:484-512) with np.random's global generator for the orders -> (state, sweeps)"""
    N = Kmn.shape[1]
    st = {k: np.empty(N) for k in ("ct", "cv", "Z", "mh", "s2")}
    if tt0 is None:
        Lm = jitchol(Kmm)
        Vm, _ = lapack.dtrtrs(Lm, Kmn, lower=1)
        st["tt"], st["vt"] = np.zeros(N), np.zeros(N)
        LLT, mu, sd = Kmm.copy(), np.zeros(N), np.sum(Vm * Vm, -2) + 1e-8
    else:
        st["tt"], st["vt"] = tt0.copy(), vt0.copy()
        mu, sd, LLT = recompute(Kmm, Kmn, st["tt"], st["vt"])
        sd = sd + 1e-8
    old = None
    stop, it = False, 0
    while not stop and it < max_iters:
        order = np.random.permutation(N)
        sweep(Kmn, LLT, mu, sd, st, y, order, eta, delta, parallel, blocked)
        mu, sd, LLT = recompute(Kmm, Kmn, st["tt"], st["vt"])
        sd = np.maximum(sd, EPS)
        if it > 0:
            stop = (np.mean(np.square(st["tt"] - old[0])) < epsilon) and (np.mean(np.square(st["vt"] - old[1])) < epsilon)
        old = (st["tt"].copy(), st["vt"].copy())
        it += 1
    st["logZ"] = log_Z_tilde(st)
    st["mu"], st["sd"] = mu, sd
    return st, it


# the committed fixtures (tests/golden/epdtc): kernel parts, N, M, seed and the options
CASES = {}
for _i, (_k, _ard, _n, _m) in enumerate([("rbf", False, 60, 10), ("rbf", True, 150, 50), ("exponential", False, 150, 10),
                                          ("exponential", True, 60, 10), ("matern32", False, 333, 129),
                                          ("matern32", True, 150, 50), ("matern52", False, 60, 50),
                                          ("matern52", True, 333, 50)]):
    CASES["%s_%s_n%d_m%d" % (_k, "ard" if _ard else "iso", _n, _m)] = (_single(_k, _ard), _n, _m, 80 + _i, {})
CASES["rbf_ard_n1300_m129"] = (_single("rbf", True), 1300, 129, 89, {})
CASES["rbf_ard_n150_m300"] = (_single("rbf", True), 150, 300, 90, {"ladder": True})
CASES["rbf_ard_x_m52_bias_n150_m50"] = (COMPOSITE, 150, 50, 91, {})
CASES["rbf_iso_white_n150_m50"] = (_single("rbf", False) + [dict(kind="white", term=1, variance=0.05)], 150, 50, 92, {})
CASES["rbf_iso_pm1_n150_m50"] = (_single("rbf", False), 150, 50, 93, {"pm1": True})
CASES["rbf_ard_parallel_n150_m50"] = (_single("rbf", True), 150, 50, 94, {"parallel_updates": True})
CASES["matern52_iso_damped_n150_m50"] = (_single("matern52", False), 150, 50, 95, {"eta": 0.7, "delta": 0.5})
CASES["rbf_iso_maxiters2_n150_m50"] = (_single("rbf", False), 150, 50, 96, {"max_iters": 2})
CASES["rbf_ard_nested_warm_n150_m50"] = (_single("rbf", True), 150, 50, 97, {"ep_mode": "nested", "calls": 2})
CASES["rbf_ard_alternated_theta_n150_m50"] = (_single("rbf", True), 150, 50, 98, {"theta2": 1.7})
CASES["rbf_ard_alternated_z_n150_m50"] = (_single("rbf", True), 150, 50, 99, {"z2": 0.3})
CASES["rbf_iso_far_n150_m10"] = (_single("rbf", False), 150, 10, 100, {"far": True})
CASES["rbf_iso_ladder_n150_m50"] = (_single("rbf", False), 150, 50, 101, {"dupz": True})


def case_data(name):
    """inputs of one case: X (N x D), Y (N x 1), Z (M x D), Xnew (29 x D)"""
    parts, N, M, seed, opts = CASES[name]
    rng = np.random.default_rng(seed)
    X = rng.uniform(-2.0, 2.0, size=(N, D))
    f = np.sin(1.3 * X[:, :1]) + 0.6 * X[:, 1:2] - 0.3 * X[:, 2:3]
    Y = (f + 0.4 * rng.standard_normal((N, 1)) > 0).astype(np.float64)
    if opts.get("pm1"):
        Y = 2.0 * Y - 1.0
    Z = rng.uniform(-2.0, 2.0, size=(M, D))
    if opts.get("far"):          # a third of the points far from every inducing point: their Sigma_diag sits at the clip
        X[: N // 3] += 40.0
    if opts.get("dupz"):         # repeated inducing points: Kmm is singular and jitchol's ladder adds jitter
        Z[M // 2:] = Z[: M - M // 2]
    Xnew = rng.uniform(-2.5, 2.5, size=(29, D))
    return X, Y, Z, Xnew


def scaled_parts(parts, s):
    """the parts with every variance multiplied by s (the changed theta of the alternated case)"""
    return [dict(p, variance=p["variance"] * s) for p in parts]


def case_eval(name, blocked=False):
    """the sweeps of a case through the restatement, as tests/golden/make_epdtc.py runs the reference"""
    parts, N, M, seed, opts = CASES[name]
    X, Y, Z, Xnew = case_data(name)
    y = Y[:, 0]
    kw = dict(eta=opts.get("eta", 1.), delta=opts.get("delta", 1.), max_iters=opts.get("max_iters", np.inf),
              parallel=opts.get("parallel_updates", False), blocked=blocked)
    np.random.seed(seed)
    kern = CompositeOracle(parts)
    Kmm, Kmn = kern.K(Z), kern.K(Z, X)
    st, it = run_epdtc(Kmm, Kmn, y, **kw)
    sweeps = [it]
    if opts.get("calls") == 2:
        st, it = run_epdtc(Kmm, Kmn, y, st["tt"], st["vt"], **kw)
        sweeps.append(it)
    return dict(tau_tilde=st["tt"], v_tilde=st["vt"], cav_tau=st["ct"], cav_v=st["cv"], log_Z_tilde=st["logZ"],
                post_mu=st["mu"], post_sd=st["sd"], sweeps=np.array(sweeps), next_random=np.random.random(),
                cond_Kmm=np.linalg.cond(Kmm))
