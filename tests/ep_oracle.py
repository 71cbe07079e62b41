"""Test-only NumPy restatement of expectation propagation (GPy/inference/latent_function_inference/expectation_propagation.py:
187-434) for the probit Bernoulli likelihood, with the gradient wiring of GPy/core/gp.py:278-280.

`ep_eval` follows EP.inference, expectation_propagation, _init_approximations, _local_updates, posteriorParams._recompute,
_ep_marginal and _inference line by line on NumPy / SciPy (LAPACK called as GPy's util/linalg.py calls it). Its sweep is
either the reference's chain of rank-1 updates (`blocked=False`) or the device's formulation (`blocked=True`): blocks of
TILE sites of the order, the chain on Sigma[I, I], S = Sigma[:, I] (I + U)^-1, Sigma -= S diag(c) S^T, mu -= S g. The
probit moments restate util/univariate_Gaussian.py's Cody functions branch for branch. The committed fixtures of
tests/golden/ep were written by the reference's own EP (tests/golden/make_ep.py) and pin this restatement.
"""
import numpy as np
from scipy.linalg import lapack

from laplace_oracle import COMPOSITE, D, _single, jitchol  # noqa: F401
from sparse_composite_oracle import CompositeOracle

TILE = 128
EPS = np.finfo(float).eps

# W. J. Cody's rational approximations (Math. Comp. 23, 1969), as util/univariate_Gaussian.py:160-185 tabulates them
P1 = [3.05326634961232344e-1, 3.60344899949804439e-1, 1.25781726111229246e-1, 1.60837851487422766e-2,
      6.58749161529837803e-4, 1.63153871373020978e-2]
Q1 = [2.56852019228982242e+0, 1.87295284992346047e+0, 5.27905102951428412e-1, 6.05183413124413191e-2,
      2.33520497626869185e-3]
P2 = [5.64188496988670089e-1, 8.88314979438837594e+0, 6.61191906371416295e+1, 2.98635138197400131e+2,
      8.81952221241769090e+2, 1.71204761263407058e+3, 2.05107837782607147e+3, 1.23033935479799725e+3,
      2.15311535474403846e-8]
Q2 = [1.57449261107098347e+1, 1.17693950891312499e+2, 5.37181101862009858e+2, 1.62138957456669019e+3,
      3.29079923573345963e+3, 4.36261909014324716e+3, 3.43936767414372164e+3, 1.23033935480374942e+3]
P3 = [3.16112374387056560e+0, 1.13864154151050156e+2, 3.77485237685302021e+2, 3.20937758913846947e+3,
      1.85777706184603153e-1]
Q3 = [2.36012909523441209e+1, 2.44024637934444173e+2, 1.28261652607737228e+3, 2.84423683343917062e+3]
LIMIT1, LIMIT2 = 0.6629, 5.6569
LN2PI, LN2 = 1.83787706640934533908193770913, 0.69314718055994530941723212146
SQRTPI, SQRT2 = 1.77245385090551602729816748334, 1.41421356237309504880168872421


def _log_pdf(z):
    return -0.5 * (LN2PI + z * z)


def _r3(y):
    nom, den = y * P3[4], y
    for i in range(3):
        nom = (nom + P3[i]) * y
        den = (den + Q3[i]) * y
    return (nom + P3[3]) / (den + Q3[3])


def _helper(x):
    if x >= LIMIT2:
        y = 2.0 / (x * x)
        res, den = y * P1[5], y
        for i in range(4):
            res = (res + P1[i]) * y
            den = (den + Q1[i]) * y
        return 1.0 - SQRTPI * y * (res + P1[4]) / (den + Q1[4])
    y = x / SQRT2
    res, den = y * P2[8], y
    for i in range(7):
        res = (res + P2[i]) * y
        den = (den + Q2[i]) * y
    return SQRTPI * y * (res + P2[7]) / (den + Q2[7])


def log_cdf(z):
    if abs(z) < LIMIT1:
        return np.log1p((z / SQRT2) * _r3(0.5 * z * z)) - LN2
    if z < 0.0:
        return _log_pdf(z) - np.log(-z) + np.log(_helper(-z))
    return np.log1p(-(np.exp(_log_pdf(z))) * _helper(z) / z)


def dlog_cdf(z):
    if abs(z) < LIMIT1:
        return 2.0 * np.exp(_log_pdf(z)) / (1.0 + (z / SQRT2) * _r3(0.5 * z * z))
    if z < 0.0:
        return -z / _helper(-z)
    t = np.exp(_log_pdf(z))
    return t / (1.0 - t * _helper(z) / z)


def moments(y, tau, v):
    """Bernoulli.moments_match_ep with the probit link (bernoulli.py:59-92) -> (Z_hat, mu_hat, sigma2_hat)"""
    sign = 1. if y == 1 else -1.
    z = sign * v / np.sqrt(tau ** 2 + tau)
    r = dlog_cdf(z)
    lz = log_cdf(z)
    mu_hat = v / tau + sign * r / np.sqrt(tau ** 2 + tau)
    sigma2_hat = 1. / tau - (r / (tau ** 2 + tau)) * (z + r)
    return np.exp(lz), mu_hat, sigma2_hat


def site(i, Sii, mui, st, y, eta, delta):
    """the cavity, the moments and the site update of site i (:27-29, :52-68) on the state dict st -> (dtau, dv)"""
    st["ct"][i] = 1. / Sii - eta * st["tt"][i]
    st["cv"][i] = mui / Sii - eta * st["vt"][i]
    st["Z"][i], st["mh"][i], st["s2"][i] = moments(y[i], st["ct"][i], st["cv"][i])
    dtau = delta / eta * (1. / st["s2"][i] - 1. / Sii)
    dv = delta / eta * (st["mh"][i] / st["s2"][i] - mui / Sii)
    prev = st["tt"][i]
    st["tt"][i] += dtau
    if st["tt"][i] < EPS:
        st["tt"][i] = EPS
        dtau = st["tt"][i] - prev
    st["vt"][i] += dv
    return dtau, dv


def recompute(K, tt, vt):
    """posteriorParams._recompute (:129-143) with mean_prior = 0 -> (mu, Sigma, L)"""
    N = len(tt)
    r = np.sqrt(tt)
    SK = r[:, None] * K
    B = np.eye(N) + SK * r[None, :]
    L = jitchol(B)
    V, _ = lapack.dtrtrs(L, SK, lower=1)
    Sigma = K - np.dot(V.T, V)
    aux, _ = lapack.dpotrs(L, r * np.dot(K, vt), lower=1)
    alpha = vt - r * aux
    return np.dot(K, alpha), Sigma, L


def sweep(Sigma, mu, st, y, order, eta, delta, parallel, blocked):
    """_local_updates (:330-351) -> (Sigma, mu)"""
    if parallel:
        d = np.diag(Sigma).copy()
        for i in order:
            site(i, d[i], mu[i], st, y, eta, delta)
        return Sigma, mu
    if not blocked:
        for i in order:
            dtau, dv = site(i, Sigma[i, i], mu[i], st, y, eta, delta)
            si = Sigma[i, :].copy()
            ci = dtau / (1. + dtau * si[i])
            mu = mu - (ci * (mu[i] + si[i] * dv) - dv) * si
            Sigma = Sigma - ci * np.outer(si, si)
        return Sigma, mu
    Sigma, mu = Sigma.copy(), mu.copy()
    for k0 in range(0, len(order), TILE):
        I = order[k0:k0 + TILE]
        m = len(I)
        P = Sigma[:, I].copy()
        G = P[I].copy()
        muI = mu[I].copy()
        c, g = np.zeros(m), np.zeros(m)
        R = np.zeros((m, m))
        for j in range(m):
            dtau, dv = site(I[j], G[j, j], muI[j], st, y, eta, delta)
            s = G[:, j].copy()
            c[j] = dtau / (1. + dtau * s[j])
            g[j] = c[j] * (muI[j] + s[j] * dv) - dv
            muI -= g[j] * s
            G -= c[j] * np.outer(s, s)
            R[j, j + 1:] = s[j + 1:]
        # S (I + U) = P with U[l, j] = c_l s_l[j] (l < j): forward substitution over the columns
        S = np.empty_like(P)
        for j in range(m):
            S[:, j] = P[:, j] - np.dot(S[:, :j] * c[:j], R[:j, j])
        Sigma = Sigma - np.dot(S * c, S.T)
        mu = mu - np.dot(S, g)
    return Sigma, mu


def log_Z_tilde(st):
    """:353-361"""
    tt, vt, ct, cv = st["tt"], st["vt"], st["ct"], st["cv"]
    return np.sum((np.log(st["Z"]) + 0.5 * np.log(2 * np.pi) + 0.5 * np.log(1 + tt / ct)
                   - 0.5 * ((vt) ** 2 * 1. / (ct + tt))
                   + 0.5 * (cv * (((tt / ct) * cv - 2.0 * vt) * 1. / (ct + tt)))))


def run_ep(K, y, tt0=None, vt0=None, eta=1., delta=1., epsilon=1e-6, max_iters=np.inf, parallel=False, blocked=False):
    """expectation_propagation (:279-310) with np.random's global generator for the orders -> (state, sweeps)"""
    N = K.shape[0]
    st = {k: np.empty(N) for k in ("ct", "cv", "Z", "mh", "s2")}
    if tt0 is None:
        st["tt"], st["vt"] = np.zeros(N), np.zeros(N)
        Sigma = K.copy()
        Sigma[np.diag_indices(N)] += 1e-7
        mu = np.zeros(N)
    else:
        st["tt"], st["vt"] = tt0.copy(), vt0.copy()
        mu, Sigma, _ = recompute(K, st["tt"], st["vt"])
        Sigma[np.diag_indices(N)] += 1e-7
    old = None
    stop, it = False, 0
    while not stop and it < max_iters:
        order = np.random.permutation(N)
        Sigma, mu = sweep(Sigma, mu, st, y, order, eta, delta, parallel, blocked)
        mu, Sigma, _ = recompute(K, st["tt"], st["vt"])
        if it > 0:
            stop = (np.mean(np.square(st["tt"] - old[0])) < epsilon) and (np.mean(np.square(st["vt"] - old[1])) < epsilon)
        old = (st["tt"].copy(), st["vt"].copy())
        it += 1
    st["logZ"] = log_Z_tilde(st)
    return st, it


def marginal(K, st, parts, X, Xnew=None):
    """_ep_marginal + _inference (:363-395) and the kernel gradient of gp.py:280 -> dict"""
    tt, vt = st["tt"], st["vt"]
    mu, Sigma, L = recompute(K, tt, vt)
    B_logdet = np.sum(2.0 * np.log(np.diag(L)))
    lml = 0.5 * (-len(tt) * np.log(2 * np.pi) - B_logdet + np.sum(vt * np.dot(Sigma, vt))) + st["logZ"]
    r = np.sqrt(tt)
    aux, _ = lapack.dpotrs(L, r * np.dot(K, vt), lower=1)
    alpha = (vt - r * aux)[:, None]
    LWi, _ = lapack.dtrtrs(L, np.diag(r), lower=1)
    Wi = np.dot(LWi.T, LWi)
    dL_dK = 0.5 * (np.dot(alpha, alpha.T) - Wi)
    kern = CompositeOracle(parts)
    out = dict(lml=float(lml), grad=np.concatenate(kern.grads_full(dL_dK, X)), alpha=alpha, woodbury_inv=Wi)
    if Xnew is not None:
        Kx = kern.K(X, Xnew)
        out["mu"] = np.dot(Kx.T, alpha)
        out["var"] = (kern.Kdiag(Xnew) - (np.dot(Wi, Kx) * Kx).sum(0))[:, None]
    return out


# the committed fixtures (tests/golden/ep): kernel parts, N, seed and the EP options
CASES = {}
for _i, (_k, _ard, _n) in enumerate([("rbf", False, 60), ("rbf", True, 150), ("exponential", False, 150),
                                      ("exponential", True, 60), ("matern32", False, 333), ("matern32", True, 150),
                                      ("matern52", False, 60), ("matern52", True, 333)]):
    CASES["%s_%s_n%d" % (_k, "ard" if _ard else "iso", _n)] = (_single(_k, _ard), _n, 60 + _i, {})
CASES["rbf_ard_n1300"] = (_single("rbf", True), 1300, 69, {})
CASES["rbf_ard_x_m52_bias_n150"] = (COMPOSITE, 150, 70, {})
CASES["rbf_iso_pm1_n150"] = (_single("rbf", False), 150, 71, {"pm1": True})
CASES["rbf_ard_parallel_n150"] = (_single("rbf", True), 150, 72, {"parallel_updates": True})
CASES["matern52_iso_damped_n150"] = (_single("matern52", False), 150, 73, {"eta": 0.7, "delta": 0.5})
CASES["rbf_iso_maxiters2_n150"] = (_single("rbf", False), 150, 74, {"max_iters": 2})
CASES["rbf_ard_nested_warm_n150"] = (_single("rbf", True), 150, 75, {"ep_mode": "nested", "calls": 2})
CASES["rbf_ard_alternated_theta_n150"] = (_single("rbf", True), 150, 76, {"theta2": 1.7})
SMALL_N = 150   # fixtures up to this size also hold woodbury_inv


def case_data(name):
    """inputs of one case: X (N x D), Y (N x 1), Xnew (29 x D)"""
    parts, N, seed, opts = CASES[name]
    rng = np.random.default_rng(seed)
    X = rng.uniform(-2.0, 2.0, size=(N, D))
    f = np.sin(1.3 * X[:, :1]) + 0.6 * X[:, 1:2] - 0.3 * X[:, 2:3]
    Y = (f + 0.4 * rng.standard_normal((N, 1)) > 0).astype(np.float64)
    if opts.get("pm1"):
        Y = 2.0 * Y - 1.0
    Xnew = rng.uniform(-2.5, 2.5, size=(29, D))
    return X, Y, Xnew


def scaled_parts(parts, s):
    """the parts with every variance multiplied by s (the changed theta of the alternated case)"""
    return [dict(p, variance=p["variance"] * s) for p in parts]


def case_eval(name, blocked=False):
    """the case through the restatement, as tests/golden/make_ep.py runs the reference (np.random.seed(seed) first)"""
    parts, N, seed, opts = CASES[name]
    X, Y, Xnew = case_data(name)
    y = Y[:, 0]
    kw = dict(eta=opts.get("eta", 1.), delta=opts.get("delta", 1.), max_iters=opts.get("max_iters", np.inf),
              parallel=opts.get("parallel_updates", False), blocked=blocked)
    np.random.seed(seed)
    K = CompositeOracle(parts).K(X)
    st, it = run_ep(K, y, **kw)
    sweeps = [it]
    if opts.get("calls") == 2:
        st, it = run_ep(K, y, st["tt"], st["vt"], **kw)
        sweeps.append(it)
    if "theta2" in opts:
        parts = scaled_parts(parts, opts["theta2"])
        K = CompositeOracle(parts).K(X)
    out = marginal(K, st, parts, X, Xnew)
    out.update(tau_tilde=st["tt"], v_tilde=st["vt"], cav_tau=st["ct"], cav_v=st["cv"], log_Z_tilde=st["logZ"],
               sweeps=np.array(sweeps), next_random=np.random.random())
    return out
