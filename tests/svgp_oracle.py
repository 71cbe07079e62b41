"""Test-only NumPy restatement of the SVGP bound and its gradients (GPy/inference/latent_function_inference/svgp.py:10-118)
with the gradient wiring of GPy/core/svgp.py:49-66, one latent function, no mean function, for any kernel the composite
oracle knows and any likelihood with `variational_expectations`.

`svgp_eval` follows SVGP.inference line by line (jitchol, dpotri, dpotrs as GPy's util/linalg.py calls them), except that
dL_dchol is formed without S^-1: lower(S^-1 L) = lower(L^-T) = diag(1 / L_ii), so
    dL_dchol = 2 tril((dF_dS - Kmm^-1 / 2) L) + diag(1 / L_ii),
which is what the device computes. The reference's dpotri leaves rounding noise of order cond(S) eps where this lower
triangle is exactly zero; tests/test_svgp_cpu.py compares the two forms with a bar that says so.
"""
import numpy as np
from scipy.linalg import lapack

from laplace_oracle import COMPOSITE, D, Poisson, _single, jitchol  # noqa: F401
from sparse_composite_oracle import CompositeOracle
from gpy_b200.laplace import quadrature_expectations


class PoissonVE(Poisson):
    """laplace_oracle's Poisson with the generic quadrature of likelihood.py:358-411 (no parameters)"""

    def variational_expectations(self, Y, m, v, gh_points=None, Y_metadata=None):
        return quadrature_expectations(self, Y, m, v, None, gh_points)


def flat_to_triang(flat, M):
    L = np.zeros((M, M))
    L[np.tril_indices(M)] = np.asarray(flat, dtype=np.float64).reshape(-1)
    return L


def svgp_eval(parts, X, Y, Z, q_m, q_L, lik, batch_scale=1.0, Xnew=None):
    """one SVGP.parameters_changed on the batch X, Y -> dict: lml, grad (every leaf's block in order), dZ, dL_dm (M,),
    dL_dchol (M x M lower), dL_dchol_ref (the reference's dpotri form), dL_dthetaL, mu, v, KL, wv, wi, cond_Kmm, cond_S
    and, with Xnew, the latent mean and variance there (posterior.py:220-248 with pred_var = Z)"""
    kern = CompositeOracle(parts)
    M = Z.shape[0]
    q_m = np.asarray(q_m, dtype=np.float64).reshape(M, 1)
    L = np.asarray(q_L, dtype=np.float64)
    S = L.dot(L.T)
    logdetS = 2. * np.sum(np.log(np.abs(np.diag(L))))
    Kmm, Kmn, Knn_diag = kern.K(Z), kern.K(Z, X), kern.Kdiag(X)
    Lm = jitchol(Kmm)
    logdetKmm = 2. * np.sum(np.log(np.diag(Lm)))
    Kmmi, _ = lapack.dpotri(np.asfortranarray(Lm), lower=1)
    Kmmi = np.tril(Kmmi) + np.tril(Kmmi, -1).T
    A, _ = lapack.dpotrs(Lm, Kmn, lower=1)
    mu = np.dot(A.T, q_m)
    tmp = np.dot(L.T, A)
    v = (np.sum(np.square(tmp), 0) + (Knn_diag - np.sum(A * Kmn, 0)))[:, None]
    Kmmim = np.dot(Kmmi, q_m)
    KL = -0.5 * logdetS - 0.5 * M + 0.5 * logdetKmm + 0.5 * np.sum(Kmmi * S) + 0.5 * np.sum(q_m * Kmmim)
    F, dF_dmu, dF_dv, dF_dthetaL = lik.variational_expectations(Y, mu, v)
    F, dF_dmu, dF_dv = F * batch_scale, dF_dmu * batch_scale, dF_dv * batch_scale
    if dF_dthetaL is not None:
        dF_dthetaL = dF_dthetaL.sum(1).sum(1) * batch_scale
    Adv = A * dF_dv.T
    Admu = A.dot(dF_dmu)
    AdvA = np.dot(Adv, A.T)
    T = S.dot(Kmmi)
    R = AdvA.dot(T)
    dF_dKmm = -Admu.dot(Kmmim.T) + AdvA - R - R.T
    dF_dKmm = 0.5 * (dF_dKmm + dF_dKmm.T)
    dKL_dKmm = 0.5 * Kmmi - 0.5 * Kmmi.dot(S).dot(Kmmi) - 0.5 * Kmmim.dot(Kmmim.T)
    dL_dKmm = dF_dKmm - dKL_dKmm
    dL_dKmn = Kmmim.dot(dF_dmu.T) + np.dot(2. * (T - np.eye(M)).T, Adv)
    dL_dm = (Admu - Kmmim)[:, 0]
    dL_dchol = 2. * np.tril((AdvA - 0.5 * Kmmi).dot(L)) + np.diag(1.0 / np.diag(L))
    Si, _ = lapack.dpotri(np.asfortranarray(L), lower=1)
    Si = np.tril(Si) + np.tril(Si, -1).T
    dL_dchol_ref = np.tril(2. * (AdvA - 0.5 * (Kmmi - Si)).dot(L))
    # the kernel's gradient (core/svgp.py:53-60) and dL/dZ (:61-62)
    g = [a + b + c for a, b, c in zip(kern.grads_full(dL_dKmm, Z), kern.grads_full(dL_dKmn, Z, X),
                                      kern.grads_diag(dF_dv.sum(1), X))]
    dZ = kern.gradients_X(dL_dKmm, Z) + kern.gradients_X(dL_dKmn, Z, X)
    wv = Kmmim[:, 0]
    tmp2, _ = lapack.dpotrs(Lm, Kmm - S, lower=1)
    wi, _ = lapack.dpotrs(Lm, tmp2.T, lower=1)
    jitter = float(np.mean(np.diag(Lm.dot(Lm.T)) - np.diag(Kmm)))   # what jitchol's ladder added (0 up to rounding)
    out = dict(jitter=jitter, cond_Kmm_jit=np.linalg.cond(Kmm + (jitter if jitter > 1e-12 * np.mean(np.diag(Kmm)) else 0.)
                                                          * np.eye(M)),
               lml=F.sum() - KL, grad=np.concatenate(g), dZ=dZ, dL_dm=dL_dm, dL_dchol=dL_dchol, dL_dchol_ref=dL_dchol_ref,
               dL_dthetaL=dF_dthetaL, mu=mu[:, 0], v=v[:, 0], KL=KL, wv=wv, wi=wi, cond_Kmm=np.linalg.cond(Kmm),
               cond_S=np.linalg.cond(S))
    if Xnew is not None:
        Kx = kern.K(Z, Xnew)
        out["pmu"] = np.dot(Kx.T, wv)
        out["pvar"] = np.clip(kern.Kdiag(Xnew) - np.sum(np.dot(wi.T, Kx) * Kx, 0), 1e-15, np.inf)
    return out


def random_q(M, seed, scale=0.3):
    """a q(u) away from the identity: m ~ N(0, 1), q_L lower triangular with a positive diagonal and off-diagonal entries
    of size scale / sqrt(M), so that cond(q_L q_L^T) stays moderate at any M"""
    rng = np.random.default_rng(seed)
    m = rng.standard_normal(M)
    L = np.tril(scale / np.sqrt(M) * rng.standard_normal((M, M)), -1) + np.diag(rng.uniform(0.5, 1.2, M))
    return m, L


# cases shared by the CPU and GPU tests: kernel parts, likelihood, N, M, seed, options
CASES = {}
for _i, (_k, _ard) in enumerate([("rbf", False), ("rbf", True), ("exponential", False), ("exponential", True),
                                  ("matern32", False), ("matern32", True), ("matern52", False), ("matern52", True)]):
    CASES["bernoulli_%s_%s" % (_k, "ard" if _ard else "iso")] = (_single(_k, _ard), "bernoulli", 150, 40, 300 + _i, {})
CASES["gaussian_rbf_ard"] = (_single("rbf", True), "gaussian", 150, 40, 310, {})
CASES["studentt_matern52_ard"] = (_single("matern52", True, 0.6), ("studentt", 3.0, 0.05), 150, 40, 311, {})
CASES["poisson_rbf_iso"] = (_single("rbf", False, 0.8), "poisson", 150, 40, 312, {})
CASES["bernoulli_rbf_white"] = (_single("rbf", False) + [dict(kind="white", term=1, variance=1e-6)], "bernoulli", 150, 30,
                                313, {})
CASES["bernoulli_composite"] = (COMPOSITE, "bernoulli", 150, 40, 314, {})
CASES["bernoulli_batch_scale"] = (_single("rbf", True), "bernoulli", 150, 40, 315, {"batch_scale": 7.5})
# M > Nb with lengthscales short enough for 200 inducing points in the cube to keep Kmm well-conditioned
CASES["bernoulli_m_gt_nb"] = ([dict(kind="rbf", term=0, dims=[0, 1, 2], variance=1.4, lengthscale=[0.3, 0.35, 0.4],
                                    ARD=True)], "bernoulli", 60, 200, 316, {})
CASES["bernoulli_dupz"] = (_single("rbf", False), "bernoulli", 150, 40, 317, {"dupz": True})
CASES["bernoulli_negdiag"] = (_single("matern32", True), "bernoulli", 150, 40, 318, {"negdiag": True})
CASES["bernoulli_identity"] = (_single("rbf", True), "bernoulli", 150, 40, 319, {"identity": True})


def case_data(name):
    """inputs of one case: X (N x D), Y (N x 1), Z (M x D), q_m (M,), q_L (M x M), Xnew (29 x D), batch_scale"""
    parts, lik, N, M, seed, opts = CASES[name]
    rng = np.random.default_rng(seed)
    X = rng.uniform(-2.0, 2.0, size=(N, D))
    f = np.sin(1.3 * X[:, :1]) + 0.6 * X[:, 1:2] - 0.3 * X[:, 2:3]
    if lik == "bernoulli":
        Y = (f + 0.4 * rng.standard_normal((N, 1)) > 0).astype(np.float64)
    elif lik == "poisson":
        Y = rng.poisson(np.exp(0.7 * f)).astype(np.float64)
    else:
        Y = f + 0.2 * rng.standard_t(2.0, size=(N, 1))
    Z = rng.uniform(-2.0, 2.0, size=(M, D))
    if opts.get("dupz"):
        Z[M // 2:] = Z[: M - M // 2]
    q_m, q_L = random_q(M, seed + 1000)
    if opts.get("negdiag"):
        q_L[::3] *= -1.0            # rows with a negative diagonal entry (GPy does not constrain it)
    if opts.get("identity"):
        q_m, q_L = np.zeros(M), np.eye(M)
    Xnew = rng.uniform(-2.5, 2.5, size=(29, D))
    return X, Y, Z, q_m, q_L, Xnew, opts.get("batch_scale", 1.0)


def make_likelihood(spec, module):
    """the case's likelihood from `module` (gpy_b200, or a namespace of the reference's Bernoulli, StudentT, Gaussian)"""
    if spec == "bernoulli":
        return module.Bernoulli()
    if spec == "gaussian":
        return module.Gaussian(variance=0.3)
    if spec == "poisson":
        return PoissonVE()
    return module.StudentT(deg_free=spec[1], sigma2=spec[2])


def descriptor(p):
    return (p["kind"], p.get("ARD", False), p["term"], list(p.get("dims") or []), p["variance"], p.get("lengthscale"))
