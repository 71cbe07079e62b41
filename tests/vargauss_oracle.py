"""Test-only NumPy restatement of the variational Gaussian approximation (GPy/inference/latent_function_inference/
var_gauss.py:34-69), one output column, no mean function, for any kernel the composite oracle knows and any likelihood with
`variational_expectations`.

`vargauss_eval` follows VarGauss.inference line by line (pdinv as GPy's util/linalg.py:193-214 runs it: jitchol, then
dpotri), except for one term. The reference's dF_dK (:66) is np.dot(tmp * dF_dv, tmp.T) with dF_dv of shape (N, 1), which
scales the rows of tmp; the derivative of sum_i dF_dv_i Sigma_ii in K scales its columns, tmp diag(dF_dv) tmp^T. Both
forms are here (`row_scaling`), so the tests can show that this term is the only difference and that the column form is
the derivative of the bound. The two agree when dF_dv is constant (the Gaussian likelihood).
"""
import numpy as np
from scipy.linalg import lapack

from laplace_oracle import COMPOSITE, D, _single, jitchol  # noqa: F401
from sparse_composite_oracle import CompositeOracle
from svgp_oracle import PoissonVE


def pdinv(A, maxtries=5):
    """util/linalg.py:193-214 -> (Ai, L, logdet, jitter the ladder added)"""
    L = jitchol(A, maxtries)
    logdet = 2. * np.sum(np.log(np.diag(L)))
    Ai, _ = lapack.dpotri(np.asfortranarray(L), lower=1)
    Ai = np.tril(Ai) + np.tril(Ai, -1).T
    jitter = float(np.mean(np.diag(L.dot(L.T)) - np.diag(A)))
    return Ai, L, logdet, jitter


def vargauss_eval(parts, X, Y, alpha, beta, lik, row_scaling=False, Xnew=None, K=None):
    """one VarGauss.inference plus the kernel gradient of gp.py:280 -> dict: lml, F, KL, m, var, dF_dm, dF_dv,
    dalpha, dbeta, dL_dthetaL, grad (every leaf's block in order), dL_dK, jitter, cond_A, cond_K and, with Xnew, the latent
    mean and variance there (posterior.py:220-248 with woodbury_vector = alpha, woodbury_inv = (K + B^-2)^-1)"""
    kern = CompositeOracle(parts)
    N = X.shape[0]
    alpha = np.asarray(alpha, dtype=np.float64).reshape(N, 1)
    beta = np.asarray(beta, dtype=np.float64).reshape(N)
    K = kern.K(X) if K is None else K
    m = K.dot(alpha)
    KB = K * beta[:, None]
    BKB = KB * beta[None, :]
    A = np.eye(N) + BKB
    Ai, LA, Alogdet, jitter = pdinv(A)
    Sigma = np.diag(beta ** -2) - Ai / beta[:, None] / beta[None, :]
    var = np.diag(Sigma).reshape(-1, 1)
    F, dF_dm, dF_dv, dF_dthetaL = lik.variational_expectations(Y, m, var)
    dL_dthetaL = np.array([]) if dF_dthetaL is None else dF_dthetaL.sum(1).sum(1)
    dF_da = np.dot(K, dF_dm)
    dF_db = -2 * np.sum(Sigma ** 2 * (dF_dv * beta), 0)
    KL = 0.5 * (Alogdet + np.trace(Ai) - N + np.sum(m * alpha))
    A_A2 = Ai - Ai.dot(Ai)
    dKL_db = np.diag(np.dot(KB.T, A_A2))
    dKL_dK = 0.5 * (alpha * alpha.T + beta[:, None] * beta[None, :] * A_A2)
    tmp = Ai * beta[:, None] / beta[None, :]
    scaled = tmp * dF_dv if row_scaling else tmp * dF_dv.T
    dF_dK = alpha * dF_dm.T + np.dot(scaled, tmp.T)
    dL_dK = dF_dK - dKL_dK
    out = dict(lml=float(F.sum() - KL), F=float(F.sum()), KL=float(KL), m=m[:, 0], var=var[:, 0], dF_dm=dF_dm[:, 0],
               dF_dv=dF_dv[:, 0], dalpha=(dF_da - m)[:, 0], dbeta=dF_db - dKL_db, dL_dthetaL=dL_dthetaL,
               grad=np.concatenate(kern.grads_full(dL_dK, X)), dL_dK=dL_dK, jitter=jitter, cond_A=np.linalg.cond(A),
               cond_K=np.linalg.cond(K), woodbury_inv=np.linalg.inv(K + np.diag(beta ** -2.0)) if N <= 400 else None)
    if Xnew is not None:
        wi = (beta[:, None] * Ai) * beta[None, :]
        Kx = kern.K(X, Xnew)
        out["pmu"] = np.dot(Kx.T, alpha)[:, 0]
        out["pvar"] = np.clip(kern.Kdiag(Xnew) - np.sum(np.dot(wi, Kx) * Kx, 0), 1e-15, np.inf)
    return out


def cond_bound(K, beta):
    """the bound on cond(A) the tests derive their bars from: 1 + max beta_i^2 lambda_max(K)"""
    return 1.0 + float(np.max(np.square(beta))) * float(np.linalg.eigvalsh(K)[-1])


# cases shared by the fixtures, the CPU and the GPU tests: kernel parts, likelihood, N, seed, beta ("rand", "init": the
# model's initial alpha = 0 and beta = 1, "neg": some entries negative, "wide": |beta| from 1e-3 to 1e3)
CASES = {}
for _i, (_k, _ard, _n) in enumerate([("rbf", False, 60), ("rbf", True, 127), ("exponential", False, 128),
                                      ("exponential", True, 129), ("matern32", False, 333), ("matern32", True, 60),
                                      ("matern52", False, 128), ("matern52", True, 1300)]):
    CASES["bernoulli_%s_%s_n%d" % (_k, "ard" if _ard else "iso", _n)] = (_single(_k, _ard), "bernoulli", _n, 60 + _i,
                                                                         "rand")
CASES["gaussian_rbf_ard_n129"] = (_single("rbf", True), "gaussian", 129, 70, "rand")
CASES["gaussian_matern32_iso_n60"] = (_single("matern32", False), "gaussian", 60, 71, "neg")
CASES["studentt_matern52_ard_n128"] = (_single("matern52", True, 0.6), ("studentt", 3.0, 0.05), 128, 72, "rand")
CASES["poisson_rbf_iso_n127"] = (_single("rbf", False, 0.8), "poisson", 127, 73, "rand")
CASES["bernoulli_rbf_white_n60"] = (_single("rbf", False) + [dict(kind="white", term=1, variance=0.05)], "bernoulli", 60,
                                    74, "rand")
CASES["bernoulli_m52_x_rbf_bias_n128"] = (COMPOSITE, "bernoulli", 128, 75, "rand")
CASES["bernoulli_rbf_iso_n1"] = (_single("rbf", False), "bernoulli", 1, 76, "rand")
CASES["bernoulli_rbf_ard_init_n129"] = (_single("rbf", True), "bernoulli", 129, 77, "init")
CASES["bernoulli_matern32_ard_negbeta_n128"] = (_single("matern32", True), "bernoulli", 128, 78, "neg")
CASES["studentt_rbf_iso_widebeta_n128"] = (_single("rbf", False), ("studentt", 3.0, 0.05), 128, 79, "wide")


def case_data(name):
    """inputs of one case: X (N x D), Y (N x 1), alpha (N,), beta (N,), Xnew (29 x D)"""
    parts, lik, N, seed, bmode = CASES[name]
    rng = np.random.default_rng(seed)
    X = rng.uniform(-2.0, 2.0, size=(N, D))
    f = np.sin(1.3 * X[:, :1]) + 0.6 * X[:, 1:2] - 0.3 * X[:, 2:3]
    if lik == "bernoulli":
        Y = (f + 0.4 * rng.standard_normal((N, 1)) > 0).astype(np.float64)
    elif lik == "poisson":
        Y = rng.poisson(np.exp(0.7 * f)).astype(np.float64)
    else:
        Y = f + 0.2 * rng.standard_t(2.0, size=(N, 1))
    alpha = 0.3 * rng.standard_normal(N)
    beta = rng.uniform(0.5, 2.0, N)
    if bmode == "init":
        alpha, beta = np.zeros(N), np.ones(N)
    elif bmode == "neg":
        beta[::3] *= -1.0
    elif bmode == "wide":
        beta = rng.permutation(np.logspace(-3, 3, N)) * np.where(rng.uniform(size=N) < 0.3, -1.0, 1.0)
    Xnew = rng.uniform(-2.5, 2.5, size=(29, D))
    return X, Y, alpha, beta, Xnew


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
    """the part as Engine.vargauss_begin takes it"""
    return (p["kind"], p.get("ARD", False), p["term"], list(p.get("dims") or []), p["variance"], p.get("lengthscale"))
