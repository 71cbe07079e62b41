"""Test-only NumPy restatement of FITC sparse GP regression (GPy/inference/latent_function_inference/fitc.py:19-88,
Snelson & Ghahramani's SPGP) with the gradient wiring of GPy/core/sparse_gp.py:108-118, for any kernel the composite
oracle knows (a single stationary kernel is one part).

`fitc_inference` follows fitc.py line by line on the oracle's own pdinv / jitchol / dtrtrs / tdot (oracle/gpy_oracle.py);
`fitc_eval` adds SparseGP._update_gradients (update_gradients_diag with dL_dKdiag = dL_dR, update_gradients_full with
dL_dKnm and dL_dKmm, gradients_X for Z.gradient) through tests/sparse_composite_oracle.CompositeOracle. `reference_fitc`
runs the reference's own FITC + kernels (through oracle/ref_gpy.py) where the reference tree exists; it writes the
fixtures of tests/golden/fitc and backs the CPU cross-check.
"""
import importlib

import numpy as np

from oracle import gpy_oracle as o
from sparse_composite_oracle import CompositeOracle

CONST_JITTER = 1e-6   # fitc.py:18
D = 3                 # input columns of every fixture case


def fitc_inference(kern, X, Z, noise_variance, Y):
    """fitc.py:19-88 -> dict(log_marginal, dL_dKmm, dL_dKdiag (N), dL_dKnm (N x M), dL_dthetaL, woodbury_vector,
    woodbury_inv, K (Kmm + jitter), K_chol)"""
    num_inducing = Z.shape[0]
    num_data, output_dim = Y.shape
    sigma_n = float(noise_variance)
    Kmm = kern.K(Z).copy()                                                        # :33
    Knn = kern.Kdiag(X)                                                           # :34
    U = kern.K(X, Z)                                                              # :35-36
    o.diag_add(Kmm, CONST_JITTER)                                                 # :39
    Kmmi, L, Li, _ = o.pdinv(Kmm)                                                 # :40
    LiUT = np.dot(Li, U.T)                                                        # :42
    sigma_star = Knn + sigma_n - np.sum(np.square(LiUT), 0)                       # :43
    beta_star = 1.0 / sigma_star                                                  # :44
    A = o.tdot(LiUT * np.sqrt(beta_star)) + np.eye(num_inducing)                  # :47
    LA, _ = o.jitchol(A)                                                          # :48
    URiy = np.dot(U.T * beta_star, Y)                                             # :51
    tmp, _ = o.dtrtrs(L, URiy, lower=1)                                           # :52
    b, _ = o.dtrtrs(LA, tmp, lower=1)                                             # :53
    tmp, _ = o.dtrtrs(LA, b, lower=1, trans=1)                                    # :54
    v, _ = o.dtrtrs(L, tmp, lower=1, trans=1)                                     # :55
    tmp, _ = o.dtrtrs(LA, Li, lower=1, trans=0)                                   # :56
    P = o.tdot(tmp.T)                                                             # :57
    log_marginal = (-0.5 * num_data * output_dim * np.log(2 * np.pi)              # :60-64
                    - np.sum(np.log(np.diag(LA))) * output_dim
                    + 0.5 * output_dim * np.sum(np.log(beta_star))
                    - 0.5 * np.sum(np.square(Y.T * np.sqrt(beta_star)))
                    + 0.5 * np.sum(np.square(b)))
    Uv = np.dot(U, v)                                                             # :66
    dL_dR = 0.5 * (np.sum(U * np.dot(U, P), 1) - 1.0 / beta_star + np.sum(np.square(Y), 1)
                   - 2.0 * np.sum(Uv * Y, 1) + np.sum(np.square(Uv), 1)) * beta_star ** 2            # :67
    vvT_P = o.tdot(v.reshape(-1, 1)) + P                                          # :71
    dL_dK = 0.5 * (Kmmi - vvT_P)                                                  # :72
    KiU = np.dot(Kmmi, U.T)                                                       # :73
    dL_dK += np.dot(KiU * dL_dR, KiU.T)                                           # :74
    vY = np.dot(v.reshape(-1, 1), Y.T)                                            # :77
    dL_dU = vY - np.dot(vvT_P, U.T)                                               # :78
    dL_dU *= beta_star                                                            # :79
    dL_dU -= 2.0 * KiU * dL_dR                                                    # :80
    return dict(log_marginal=float(log_marginal), dL_dKmm=dL_dK, dL_dKdiag=dL_dR, dL_dKnm=dL_dU.T,
                dL_dthetaL=float(np.sum(dL_dR)),                                  # gaussian.py:78-79
                woodbury_vector=v, woodbury_inv=Kmmi - P, K=Kmm, K_chol=L)       # :86


def fitc_eval(X, Y, Z, parts, noise_variance):
    """One SparseGP.parameters_changed() with FITC -> (lml, grad [every part's block, noise], Zgrad, res)"""
    X = np.ascontiguousarray(X, dtype=np.float64)
    Z = np.ascontiguousarray(Z, dtype=np.float64)
    Y = np.ascontiguousarray(Y, dtype=np.float64)
    kern = CompositeOracle(parts)
    res = fitc_inference(kern, X, Z, noise_variance, Y)
    g0 = kern.grads_diag(res["dL_dKdiag"], X)                                   # sparse_gp.py:110
    g1 = kern.grads_full(res["dL_dKnm"], X, Z)                                  # :112
    g2 = kern.grads_full(res["dL_dKmm"], Z, None)                               # :114
    grad = np.concatenate([a + b + c for a, b, c in zip(g0, g1, g2)] + [[res["dL_dthetaL"]]])
    Zgrad = kern.gradients_X(res["dL_dKmm"], Z)                                 # :117
    Zgrad = Zgrad + kern.gradients_X(res["dL_dKnm"].T, Z, X)                    # :118
    return res["log_marginal"], grad, Zgrad, res


def predict(res, parts, Z, Xnew):
    """posterior.py:238-270 with pred_var = Z on the FITC posterior -> (mu, var), var clipped at 1e-15 (:248)"""
    mu, var = o.sparse_raw_predict(CompositeOracle(parts), Z, res["woodbury_vector"], res["woodbury_inv"], Xnew)
    return mu, np.clip(var, 1e-15, np.inf)


def descriptor(p):
    """the part as Engine.sparse_eval_fitc takes it"""
    return (p["kind"], p.get("ARD", False), p["term"], list(p.get("dims") or []), p["variance"], p.get("lengthscale"))


def _single(kind, ard, variance=1.2):
    ls = [0.8, 1.3, 1.9] if ard else 1.1
    return [dict(kind=kind, term=0, dims=[0, 1, 2], variance=variance, lengthscale=ls, ARD=ard)]


# the committed fixtures (tests/golden/fitc): kernel parts, N, M, seed, Z a subset of X
CASES = {
    "rbf_iso_m50": (_single("rbf", False), 200, 50, 11, False),
    "rbf_ard_m129": (_single("rbf", True), 300, 129, 12, False),
    "exponential_iso_m50": (_single("exponential", False), 200, 50, 13, False),
    "exponential_ard_m50": (_single("exponential", True), 200, 50, 14, False),
    "matern32_iso_m50": (_single("matern32", False), 200, 50, 15, False),
    "matern32_ard_m129": (_single("matern32", True), 300, 129, 16, False),
    "matern52_iso_m300": (_single("matern52", False), 500, 300, 17, False),
    "matern52_ard_m50": (_single("matern52", True), 200, 50, 18, False),
    "rbf_ard_bias_white_m129": ([dict(kind="rbf", term=0, dims=[0, 1, 2], variance=1.3, lengthscale=[0.9, 1.4, 2.1],
                                      ARD=True),
                                 dict(kind="bias", term=1, variance=0.4),
                                 dict(kind="white", term=2, variance=0.07)], 300, 129, 19, False),
    "m52_x_rbf_bias_m50": ([dict(kind="matern52", term=0, dims=[0, 1], variance=1.1, lengthscale=1.2),
                            dict(kind="rbf", term=0, dims=[1, 2], variance=0.8, lengthscale=[1.5, 0.7], ARD=True),
                            dict(kind="bias", term=1, variance=0.3)], 200, 50, 20, False),
    "rbf_iso_z_subset_m50": (_single("rbf", False), 200, 50, 21, True),
}
SMALL_M = 50   # the fixtures of this many inducing points also hold the M x M posterior arrays


def case_data(name):
    """inputs of one case: X (N x D), Y (N x 1), Z (M x D), noise, Xnew (37 x D)"""
    parts, N, M, seed, subset = CASES[name]
    rng = np.random.default_rng(seed)
    X = rng.uniform(-2.0, 2.0, size=(N, D))
    Y = np.sin(X.sum(1, keepdims=True)) + 0.1 * rng.standard_normal((N, 1))
    idx = rng.choice(N, M, replace=False)
    Z = X[idx].copy() if subset else X[idx] + 0.05 * rng.standard_normal((M, D))
    Xnew = rng.uniform(-2.5, 2.5, size=(37, D))
    return X, Y, Z, 0.08, Xnew


def reference_fitc(ref_gpy, X, Y, Z, parts, noise, Xnew=None):
    """the reference's own FITC (fitc.py, unmodified) over its own kernels and Gaussian likelihood, with the gradient
    wiring of sparse_gp.py:108-118 -> dict(lml, grad, Zgrad, dL_dKdiag, woodbury_vector, woodbury_inv, K, K_chol[, mu,
    var])"""
    import os
    import sys
    golden = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    if golden not in sys.path:
        sys.path.append(golden)
    import make_sparse_composite as msc   # ref_kernel: the reference's composite for a list of parts
    S = ref_gpy.load_sparse_models()
    C = ref_gpy.load_combination()
    G = S.G
    FITC = importlib.import_module("GPy.inference.latent_function_inference.fitc").FITC
    msc.D = X.shape[1]
    kern = msc.ref_kernel(C, G, parts)
    lik = G.Gaussian(variance=noise)
    post, lml, gd = FITC().inference(kern, X, Z, lik, Y)                       # sparse_gp.py:77-80
    lik.update_gradients(gd["dL_dthetaL"])                                     # :84
    kern.update_gradients_diag(gd["dL_dKdiag"], X)                             # :110
    kg = kern.gradient.copy()
    kern.update_gradients_full(gd["dL_dKnm"], X, Z)                            # :112
    kg += kern.gradient
    kern.update_gradients_full(gd["dL_dKmm"], Z, None)                         # :114
    kg += kern.gradient
    Zg = kern.gradients_X(gd["dL_dKmm"], Z)                                    # :117
    Zg = Zg + kern.gradients_X(gd["dL_dKnm"].T, Z, X)                          # :118
    out = dict(lml=float(np.squeeze(lml)),
               grad=np.concatenate([np.asarray(kg, dtype=np.float64), np.asarray(lik.variance.gradient).reshape(-1)]),
               Zgrad=np.asarray(Zg), dL_dKdiag=np.asarray(gd["dL_dKdiag"], dtype=np.float64).reshape(-1),
               woodbury_vector=np.asarray(post.woodbury_vector), woodbury_inv=np.asarray(post.woodbury_inv),
               K=np.asarray(post._K), K_chol=np.asarray(post._K_chol))
    if Xnew is not None:
        mu, var = post._raw_predict(kern, Xnew, Z, full_cov=False)
        out["mu"], out["var"] = np.asarray(mu), np.asarray(var)
    return out
