"""Test-only NumPy restatement of GP.predictive_gradients (GPy/core/gp.py:438-474) for the exact and the sparse model:

    mean_jac[m, q, p] = sum_n alpha[n, p] dk(x*_m, x_n)/dx*_mq     kern.gradients_X(woodbury_vector[:, p:p+1].T, Xnew, X)
    var_jac[m, q]     = gradients_X_diag(1, Xnew) - 2 sum_n (K(Xnew, X) W)[m, n] dk(x*_m, x_n)/dx*_mq

with X the training inputs (exact) or Z (sparse, sparse_gp.py:52-54), alpha the woodbury vector and W the woodbury_inv.
gradients_X_diag is zero for the stationary and static kernels (stationary.py:360-361, static.py:27-31). The kernel is a
sparse_composite_oracle.CompositeOracle; the normalizer step is gp.py:466-472 with GPy's Standardize.
"""
import numpy as np
from scipy.linalg import cho_factor, cho_solve

from oracle import gpy_oracle as o
from sparse_composite_oracle import CompositeOracle, case_data  # noqa: F401  (case_data: shared inputs)

JITTER = 1e-8   # exact_gaussian_inference.py:56

# the kernels of the tests and fixtures, on D = 3 columns: the four stationary kinds alone (iso / ARD), and two composites
KERNELS = {}
for _kind in ("rbf", "exponential", "matern32", "matern52"):
    KERNELS[_kind + "_iso"] = [dict(kind=_kind, term=0, dims=[0, 1, 2], variance=1.2, lengthscale=1.3)]
    KERNELS[_kind + "_ard"] = [dict(kind=_kind, term=0, dims=[0, 1, 2], variance=0.9, lengthscale=[0.8, 1.5, 2.2],
                                    ARD=True)]
KERNELS["rbf_bias_white"] = [dict(kind="rbf", term=0, dims=[0, 1, 2], variance=1.3, lengthscale=[0.9, 1.4, 2.1], ARD=True),
                             dict(kind="bias", term=1, variance=0.4),
                             dict(kind="white", term=2, variance=0.07)]
KERNELS["m52_x_rbf"] = [dict(kind="matern52", term=0, dims=[0, 1], variance=1.1, lengthscale=1.2),
                        dict(kind="rbf", term=0, dims=[1, 2], variance=0.8, lengthscale=[1.5, 0.7], ARD=True)]


def mirror_kernel(parts, D=3):
    """the mirror's kernel object (gpy_b200) for a list of part dicts: Add over terms of Prod over factors"""
    import gpy_b200
    terms = {}
    for p in parts:
        if p["kind"] in ("white", "bias"):
            k = (gpy_b200.White if p["kind"] == "white" else gpy_b200.Bias)(D, variance=p["variance"])
        else:
            cls = {"rbf": gpy_b200.RBF, "exponential": gpy_b200.Exponential, "matern32": gpy_b200.Matern32,
                   "matern52": gpy_b200.Matern52}[p["kind"]]
            k = cls(len(p["dims"]), variance=p["variance"], lengthscale=p["lengthscale"], ARD=p.get("ARD", False),
                    active_dims=p["dims"])
        terms.setdefault(p["term"], []).append(k)
    ts = [ks[0] if len(ks) == 1 else gpy_b200.Prod(ks) for _, ks in sorted(terms.items())]
    return ts[0] if len(ts) == 1 else gpy_b200.Add(ts)


def jacobians(kern, woodbury_vector, woodbury_inv, Xnew, Xpred):
    """gp.py:438-462 -> (mean_jac (N*, Q, P), var_jac (N*, Q)); the 1 x N row the reference passes as dL_dK is broadcast"""
    wv = np.asarray(woodbury_vector, dtype=np.float64)
    Ms, N = Xnew.shape[0], wv.shape[0]
    mean_jac = np.empty((Ms, Xnew.shape[1], wv.shape[1]))
    for p in range(wv.shape[1]):
        mean_jac[:, :, p] = kern.gradients_X(np.broadcast_to(wv[:, p][None, :], (Ms, N)), Xnew, Xpred)
    alpha = -2.0 * np.dot(kern.K(Xnew, Xpred), woodbury_inv)
    return mean_jac, kern.gradients_X(alpha, Xnew, Xpred)


def exact_posterior(kern, X, Y, noise):
    """alpha = Ky^-1 Y and Ky^-1, Ky = K + diag(noise + 1e-8) (exact_gaussian_inference.py:53-60); noise scalar or (N,)"""
    Ky = kern.K(X) + np.diag(np.broadcast_to(np.asarray(noise, dtype=np.float64) + JITTER, (X.shape[0],)))
    c = cho_factor(Ky, lower=True)
    return cho_solve(c, Y), cho_solve(c, np.eye(X.shape[0]))


def sparse_posterior(kern, X, Y, Z, noise):
    """the woodbury vector and woodbury_inv of VarDTC (var_dtc.py:201-214)"""
    r = o.vardtc_inference(kern, X, Z, noise, Y)
    return r["woodbury_vector"], r["woodbury_inv"]


def standardize(Y):
    """GPy's Standardize (normalizer.py:85-113): -> (normalised Y, mean, std)"""
    mean, std = Y.mean(0), Y.std(0)
    std[std == 0] = 1.0
    return (Y - mean) / std, mean, std


def denormalize(mean_jac, var_jac, std):
    """gp.py:466-472: inverse_mean(J) - inverse_mean(0) = J std; var: inverse_covariance (adds the P axis) when P > 1"""
    mean_jac = mean_jac * std
    var_jac = var_jac[..., None] * std ** 2 if std.size > 1 else var_jac * std ** 2
    return mean_jac, var_jac


def exact_case(kname, N, D, P, seed, het=False, normalizer=False, Ms=7):
    """-> dict of inputs and the oracle's Jacobians for one exact-model case"""
    X, Y, _, noise = case_data(N, 2, D, P, seed, het)
    Xnew = np.random.default_rng(seed + 1).uniform(-2.0, 2.0, size=(Ms, D))
    kern = CompositeOracle(KERNELS[kname])
    Yn, _, std = standardize(Y) if normalizer else (Y, None, None)
    wv, wi = exact_posterior(kern, X, Yn, noise)
    mj, vj = jacobians(kern, wv, wi, Xnew, X)
    if normalizer:
        mj, vj = denormalize(mj, vj, std)
    return dict(X=X, Y=Y, Xnew=Xnew, noise=np.asarray(noise, dtype=np.float64), mean_jac=mj, var_jac=vj)


def sparse_case(kname, N, M, D, P, seed, het=False, Ms=7):
    X, Y, Z, noise = case_data(N, M, D, P, seed, het)
    Xnew = np.random.default_rng(seed + 1).uniform(-2.0, 2.0, size=(Ms, D))
    kern = CompositeOracle(KERNELS[kname])
    wv, wi = sparse_posterior(kern, X, Y, Z, noise)
    mj, vj = jacobians(kern, wv, wi, Xnew, Z)
    return dict(X=X, Y=Y, Z=Z, Xnew=Xnew, noise=np.asarray(noise, dtype=np.float64), mean_jac=mj, var_jac=vj)
