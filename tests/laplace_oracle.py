"""Test-only NumPy restatement of the Laplace approximation (GPy/inference/latent_function_inference/laplace.py:122-353)
with the gradient wiring of GPy/core/gp.py:278-280, for any kernel the composite oracle knows and any likelihood object
with GPy's interface.

`laplace_eval` follows Laplace.inference, rasm_mode, mode_computations and _compute_B_statistics line by line on NumPy /
SciPy (LAPACK dpotrf / dtrtrs called as GPy's util/linalg.py calls them), counting Newton iterations and recording
Brent's steps; the kernel gradient is update_gradients_full with the dense dL_dK through
tests/sparse_composite_oracle.CompositeOracle. The committed fixtures of tests/golden/laplace were written by the
reference's own Laplace (tests/golden/make_laplace.py) and pin this restatement; the GPU tests compare the device
against both.
"""
import numpy as np
from scipy import linalg, optimize
from scipy.linalg import lapack
from scipy.special import gammaln

from sparse_composite_oracle import CompositeOracle

D = 3   # input columns of every fixture case


def _safe_exp(f):
    return np.exp(np.clip(f, -np.inf, np.log(np.finfo(np.float64).max)))


class Poisson(object):
    """GPy.likelihoods.Poisson with its log link (poisson.py, link_functions.py:205-222) through the chain rules of
    likelihood.py:544-656 (the link's derivatives are all exp(f)); test-only, no parameters"""
    log_concave = False
    size = 0

    def logpdf(self, f, y, Y_metadata=None):
        lf = _safe_exp(f)
        return -lf + y * np.log(lf) - gammaln(y + 1)

    def dlogpdf_df(self, f, y, Y_metadata=None):
        lf = _safe_exp(f)
        return (y / lf - 1) * lf

    def d2logpdf_df2(self, f, y, Y_metadata=None):
        lf = _safe_exp(f)
        d1 = np.clip(lf, -np.inf, np.sqrt(np.finfo(np.float64).max)) ** 2
        return -y / (lf ** 2) * d1 + (y / lf - 1) * lf

    def d3logpdf_df3(self, f, y, Y_metadata=None):
        lf = _safe_exp(f)
        d1 = np.clip(lf, -np.inf, np.nextafter(np.finfo(np.float64).max ** (1 / 3.0), -np.inf)) ** 3
        return 2 * y / lf ** 3 * d1 + 3 * (-y / (lf ** 2)) * lf * lf + (y / lf - 1) * lf

    def _laplace_gradients(self, f, y, Y_metadata=None):
        z = np.zeros((0, f.shape[0], f.shape[1]))
        return z, z.copy(), z.copy()

    def predictive_values(self, mu, var, full_cov=False, Y_metadata=None):
        raise NotImplementedError


def jitchol(A, maxtries=5):
    """util/linalg.py:56-75: LAPACK dpotrf on the C-contiguous A (its upper triangle keeps A's entries, as there)"""
    A = np.ascontiguousarray(A)
    L, info = lapack.dpotrf(A, lower=1)
    if info == 0:
        return L
    else:
        diagA = np.diag(A)
        if np.any(diagA <= 0.):
            raise np.linalg.LinAlgError("not pd: non-positive diagonal elements")
        jitter = diagA.mean() * 1e-6
        num_tries = 1
        while num_tries <= maxtries and np.isfinite(jitter):
            try:
                return linalg.cholesky(A + np.eye(A.shape[0]) * jitter, lower=True)
            except linalg.LinAlgError:
                jitter *= 10
            finally:
                num_tries += 1
        raise np.linalg.LinAlgError("not positive definite, even with jitter.")


def b_statistics(K, W, log_concave):
    """_compute_B_statistics (laplace.py:308-353) -> K_Wi_i, logdet_I_KW, I_KW_i, Ki_W_i, L, LiW12"""
    if not log_concave:
        W = np.clip(W, 1e-6, 1e+30)
    if np.any(np.isnan(W)):
        raise ValueError('One or more element(s) of W is NaN')
    W_12 = np.sqrt(W)
    B = np.eye(K.shape[0]) + W_12 * K * W_12.T
    L = jitchol(B)
    LiW12 = lapack.dtrtrs(np.asfortranarray(L), np.diagflat(W_12), lower=1, trans=0, unitdiag=0)[0]   # linalg.py:95-113
    K_Wi_i = np.dot(LiW12.T, LiW12)
    C = np.dot(LiW12, K)
    Ki_W_i = K - C.T.dot(C)
    I_KW_i = np.eye(K.shape[0]) - np.dot(K, K_Wi_i)
    logdet_I_KW = 2 * np.sum(np.log(np.diag(L)))
    return K_Wi_i, logdet_I_KW, I_KW_i, Ki_W_i, L, LiW12


def laplace_eval(X, Y, parts, likelihood, Xnew=None, tol=1e-4, max_iter=30, K=None):
    """One Laplace evaluation -> dict(lml, grad (kernel, paramz order), dL_dthetaL, f_hat, Ki_f, W, diag_Ki_W_i,
    iterations, brent, woodbury_inv, L, LiW12[, mu, var]). K: kern.K(X) as given (default: the composite oracle's)"""
    kern = CompositeOracle(parts)
    K = kern.K(X) if K is None else K
    Ki_f = np.zeros_like(Y)
    f = np.dot(K, Ki_f)

    def obj(Ki_f, f):
        ll = -0.5 * np.sum(np.dot(Ki_f.T, f)) + np.sum(likelihood.logpdf(f, Y))
        return -np.inf if np.isnan(ll) else ll

    difference, iteration, steps = np.inf, 0, []
    while difference > tol and iteration < max_iter:                                   # :179-226
        W = -likelihood.d2logpdf_df2(f, Y)
        grad = likelihood.dlogpdf_df(f, Y)
        b = W * f + grad
        W12BiW12 = b_statistics(K, W, likelihood.log_concave)[0]
        full_step_Ki_f = b - np.dot(W12BiW12, np.dot(K, b))
        dKi_f = full_step_Ki_f - Ki_f

        def inner_obj(step_size):
            Ki_f_trial = Ki_f + step_size * dKi_f
            return -obj(Ki_f_trial, np.dot(K, Ki_f_trial))

        step = optimize.brent(inner_obj, tol=1e-4, maxiter=12)
        steps.append(step)
        Ki_f_new = Ki_f + step * dKi_f
        f_new = np.dot(K, Ki_f_new)
        difference = np.abs(obj(Ki_f_new, f_new) - obj(Ki_f, f))
        Ki_f, f = Ki_f_new, f_new
        iteration += 1
    f_hat = f
    W = -likelihood.d2logpdf_df2(f_hat, Y)                                              # :243-306
    K_Wi_i, logdet_I_KW, I_KW_i, Ki_W_i, L, LiW12 = b_statistics(K, W, likelihood.log_concave)
    lml = -0.5 * np.sum(np.dot(Ki_f.T, f_hat)) + np.sum(likelihood.logpdf(f_hat, Y)) - 0.5 * logdet_I_KW
    dW_df = -likelihood.d3logpdf_df3(f_hat, Y)
    dL_dfhat = -0.5 * (np.diag(Ki_W_i)[:, None] * dW_df)
    dL_dK = 0.5 * (np.dot(Ki_f, Ki_f.T) - K_Wi_i) + np.dot(Ki_f, dL_dfhat.T).dot(I_KW_i)
    dL_dthetaL = np.zeros(likelihood.size)
    if likelihood.size > 0:
        dlik_dthetaL, dlik_grad_dthetaL, dlik_hess_dthetaL = likelihood._laplace_gradients(f_hat, Y)
        for t in range(likelihood.size):
            exp_t = (np.sum(dlik_dthetaL[t, :, :])
                     + 0.5 * np.sum(np.diag(Ki_W_i) * np.squeeze(dlik_hess_dthetaL[t, :, :])))
            dfhat_dthetaL = np.dot(I_KW_i, np.dot(K, dlik_grad_dthetaL[t, :, :]))
            dL_dthetaL[t] = np.sum(exp_t + np.dot(dL_dfhat.T, dfhat_dthetaL))
    grad = np.concatenate(kern.grads_full(dL_dK, X))
    out = dict(lml=float(lml), grad=grad, dL_dthetaL=dL_dthetaL, f_hat=f_hat, Ki_f=Ki_f, W=W,
               diag_Ki_W_i=np.diag(Ki_W_i).copy(), iterations=iteration, brent=np.array(steps), woodbury_inv=K_Wi_i,
               L=L, LiW12=LiW12, logdet=logdet_I_KW)
    if Xnew is not None:                                                                 # posterior.py:220-248
        Kx = kern.K(X, Xnew)
        out["mu"] = np.dot(Kx.T, Ki_f)
        var = kern.Kdiag(Xnew) - np.sum(np.dot(K_Wi_i, Kx) * Kx, 0)
        out["var"] = np.clip(var, 1e-15, np.inf)[:, None]
    return out


def _single(kind, ard, variance=1.4):
    ls = [0.8, 1.3, 1.9] if ard else 1.1
    return [dict(kind=kind, term=0, dims=[0, 1, 2], variance=variance, lengthscale=ls, ARD=ard)]


COMPOSITE = [dict(kind="rbf", term=0, dims=[0, 1, 2], variance=1.3, lengthscale=[0.9, 1.4, 2.1], ARD=True),
             dict(kind="matern52", term=0, dims=[0, 1], variance=1.1, lengthscale=1.2),
             dict(kind="bias", term=1, variance=0.4)]
STUDENT_T = ("studentt", 3.0, 0.05)   # deg_free, t_scale2: heavy tails on noisy data, W < 1e-6 at the outliers

# the committed fixtures (tests/golden/laplace): kernel parts, likelihood, N, seed
CASES = {}
for _i, (_k, _ard, _n) in enumerate([("rbf", False, 60), ("rbf", True, 150), ("exponential", False, 150),
                                      ("exponential", True, 60), ("matern32", False, 333), ("matern32", True, 150),
                                      ("matern52", False, 60), ("matern52", True, 333)]):
    CASES["bernoulli_%s_%s_n%d" % (_k, "ard" if _ard else "iso", _n)] = (_single(_k, _ard), "bernoulli", _n, 40 + _i)
CASES["bernoulli_rbf_ard_n1300"] = (_single("rbf", True), "bernoulli", 1300, 50)
CASES["bernoulli_rbf_ard_x_m52_bias_n150"] = (COMPOSITE, "bernoulli", 150, 51)
CASES["studentt_matern52_ard_n150"] = (_single("matern52", True, 0.6), STUDENT_T, 150, 52)
CASES["studentt_composite_n150"] = (COMPOSITE, STUDENT_T, 150, 53)
CASES["poisson_rbf_iso_n150"] = (_single("rbf", False, 0.8), "poisson", 150, 54)
SMALL_N = 150   # fixtures up to this size also hold woodbury_inv


def case_data(name):
    """inputs of one case: X (N x D), Y (N x 1), Xnew (29 x D)"""
    parts, lik, N, seed = CASES[name]
    rng = np.random.default_rng(seed)
    X = rng.uniform(-2.0, 2.0, size=(N, D))
    f = np.sin(1.3 * X[:, :1]) + 0.6 * X[:, 1:2] - 0.3 * X[:, 2:3]
    if lik == "bernoulli":
        Y = (f + 0.4 * rng.standard_normal((N, 1)) > 0).astype(np.float64)
    elif lik == "poisson":
        Y = rng.poisson(np.exp(0.7 * f)).astype(np.float64)
    else:
        Y = f + 0.2 * rng.standard_t(2.0, size=(N, 1))
        Y[::17] += 4.0   # outliers
    Xnew = rng.uniform(-2.5, 2.5, size=(29, D))
    return X, Y, Xnew


def make_likelihood(spec, module):
    """the case's likelihood from `module` (gpy_b200 or the reference's likelihood modules: an object with attributes
    Bernoulli, StudentT); Poisson is this file's restatement"""
    if spec == "bernoulli":
        return module.Bernoulli()
    if spec == "poisson":
        return Poisson()
    return module.StudentT(deg_free=spec[1], sigma2=spec[2])


def descriptor(p):
    """the part as Engine.laplace_begin takes it"""
    return (p["kind"], p.get("ARD", False), p["term"], list(p.get("dims") or []), p["variance"], p.get("lengthscale"))
