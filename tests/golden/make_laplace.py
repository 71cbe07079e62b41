"""Writes tests/golden/laplace/*.npz: the Laplace approximation produced by the reference's own Laplace
(GPy/inference/latent_function_inference/laplace.py), likelihoods (bernoulli.py, student_t.py, poisson.py) and kernels
(stationary.py, rbf.py, add.py, prod.py, static.py), executed through oracle/ref_gpy.py, with the gradient wiring of
GPy/core/gp.py:278-280:

    lml, grad, dL_dthetaL              the log marginal, the kernel gradient (paramz order), the likelihood's gradient
    f_hat, Ki_f, W, diag_Ki_W_i        the mode, Ki_f_hat, W at the mode (unclipped) and diag(Ki_W_i) (laplace.py:302-305)
    iterations, brent                  Newton iterations and each one's Brent step
    mu, var                            the posterior's latent predictions at Xnew (posterior.py:220-248)
    woodbury_inv                       only for N <= 150 (K_Wi_i)

Run from the repository root where the reference tree exists:  python tests/golden/make_laplace.py
The kernels, likelihoods and inputs are those of tests/laplace_oracle.py (CASES, case_data)."""
import importlib
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), HERE]

from oracle import ref_gpy  # noqa: E402
import laplace_oracle as lo  # noqa: E402
import make_sparse_composite as msc  # noqa: E402


def reference_kernel(parts, D):
    """the reference's own kernel object for a list of parts (stationary.py, rbf.py, add.py, prod.py, static.py)"""
    S = ref_gpy.load_sparse_models()
    C = ref_gpy.load_combination()
    msc.D = D
    return msc.ref_kernel(C, S.G, parts)


def reference_likelihood(lik_spec):
    mods = types.SimpleNamespace(Bernoulli=importlib.import_module("GPy.likelihoods.bernoulli").Bernoulli,
                                 StudentT=importlib.import_module("GPy.likelihoods.student_t").StudentT)
    return importlib.import_module("GPy.likelihoods.poisson").Poisson() if lik_spec == "poisson" else \
        lo.make_likelihood(lik_spec, mods)


def reference_laplace(parts, lik_spec, X, Y, Xnew):
    lap = importlib.import_module("GPy.inference.latent_function_inference.laplace")
    kern = reference_kernel(parts, X.shape[1])
    lik = reference_likelihood(lik_spec)
    steps = []
    brent = lap.optimize.brent

    def counting(*a, **k):
        s = brent(*a, **k)
        steps.append(s)
        return s

    lap.optimize = types.SimpleNamespace(brent=counting)
    try:
        inf = lap.Laplace()
        post, lml, gd = inf.inference(kern, X, lik, Y)
    finally:
        lap.optimize = sys.modules["scipy.optimize"]
    kern.update_gradients_full(gd["dL_dK"], X)                                   # gp.py:280
    mu, var = post._raw_predict(kern, Xnew, X, full_cov=False)
    return dict(lml=float(np.squeeze(lml)), grad=np.asarray(kern.gradient, dtype=np.float64).copy(),
                dL_dthetaL=np.asarray(gd["dL_dthetaL"], dtype=np.float64).reshape(-1), f_hat=inf.f_hat,
                Ki_f=np.asarray(post.woodbury_vector), W=np.asarray(inf.W), diag_Ki_W_i=np.diag(inf.Ki_W_i).copy(),
                iterations=len(steps), brent=np.array(steps), mu=np.asarray(mu), var=np.asarray(var),
                woodbury_inv=np.asarray(post.woodbury_inv))


def main():
    import scipy.optimize  # noqa: F401
    os.makedirs(os.path.join(HERE, "laplace"), exist_ok=True)
    for name in lo.CASES:
        parts, lik, N, _ = lo.CASES[name]
        X, Y, Xnew = lo.case_data(name)
        r = reference_laplace(parts, lik, X, Y, Xnew)
        if N > lo.SMALL_N:
            del r["woodbury_inv"]
        np.savez_compressed(os.path.join(HERE, "laplace", name + ".npz"), X=X, Y=Y, Xnew=Xnew, **r)
        print(name, r["lml"], "iterations", r["iterations"], "clipped W", int(np.sum(r["W"] < 1e-6)))


if __name__ == "__main__":
    main()
