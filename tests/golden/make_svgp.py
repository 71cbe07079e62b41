"""Writes tests/golden/svgp/*.npz: the SVGP bound and gradients as the reference's own SVGP.inference
(GPy/inference/latent_function_inference/svgp.py:12-118) computes them with its likelihoods and kernels, executed through
oracle/ref_gpy.py, with the gradient wiring of GPy/core/svgp.py:53-62:

    lml, grad, dZ                   the bound, the kernel gradient (paramz order) and dL/dZ
    dL_dm, dL_dchol, dL_dthetaL     the variational and likelihood gradients (dL_dchol flat, np.tril_indices order)
    mu, v                           the marginals of q(f) the reference handed its likelihood
    pmu, pvar                       Posterior(mean, cov, K)._raw_predict at Xnew with pred_var = Z
    cond_Kmm, cond_Kmm_jit, jitter  cond(K(Z, Z)), cond(K(Z, Z) + jitter I) and the jitter jitchol's ladder added
    cond_S                          cond(q_L q_L^T); host_seconds the reference's time for the inference call
The case "bernoulli_zero_diag" records what the reference does with a zero on q_u_chol's diagonal: no exception, the
bound is -inf (its dpotri fails quietly; np.isinf(Si) stays false).

Run from the repository root where the reference tree exists:  python tests/golden/make_svgp.py
The kernels and inputs are those of tests/svgp_oracle.py (CASES, case_data)."""
import importlib
import os
import sys
import time
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), HERE]

import svgp_oracle as so  # noqa: E402
import make_laplace as ml  # noqa: E402
from ep_reference import load_reference_ep  # noqa: E402

OUT = os.path.join(HERE, "svgp")
ZERO_DIAG = "bernoulli_zero_diag"   # bernoulli_rbf_iso with q_L[3, 3] = 0


class _Capture(object):
    """the reference's likelihood, recording the (mu, v) its variational_expectations receives"""

    def __init__(self, lik):
        self.lik = lik

    def variational_expectations(self, Y, m, v, Y_metadata=None):
        self.mu, self.v = m[:, 0].copy(), v[:, 0].copy()
        return self.lik.variational_expectations(Y, m, v, Y_metadata=Y_metadata)


def reference_case(name):
    load_reference_ep()
    svgp = importlib.import_module("GPy.inference.latent_function_inference.svgp")
    mods = types.SimpleNamespace(Bernoulli=importlib.import_module("GPy.likelihoods.bernoulli").Bernoulli,
                                 StudentT=importlib.import_module("GPy.likelihoods.student_t").StudentT,
                                 Gaussian=importlib.import_module("GPy.likelihoods.gaussian").Gaussian)
    base = "bernoulli_rbf_iso" if name == ZERO_DIAG else name
    parts, lik_spec, N, M, seed, opts = so.CASES[base]
    X, Y, Z, q_m, q_L, Xnew, bs = so.case_data(base)
    if name == ZERO_DIAG:
        q_L = q_L.copy()
        q_L[3, 3] = 0.0
    kern = ml.reference_kernel(parts, X.shape[1])
    lik = _Capture(importlib.import_module("GPy.likelihoods.poisson").Poisson() if lik_spec == "poisson"
                   else so.make_likelihood(lik_spec, mods))
    t0 = time.perf_counter()
    with np.errstate(divide="ignore", invalid="ignore"):
        post, lml, gd = svgp.SVGP().inference(q_m[:, None], q_L[np.tril_indices(M)][:, None], kern, X, Z, lik, Y,
                                              batch_scale=bs)
    host = time.perf_counter() - t0
    out = dict(lml=lml, mu=lik.mu, v=lik.v, dL_dm=gd["dL_dm"][:, 0], dL_dchol=gd["dL_dchol"][:, 0], host_seconds=host)
    if name != ZERO_DIAG:
        kern.update_gradients_full(gd["dL_dKmm"], Z)
        g = kern.gradient.copy()
        kern.update_gradients_full(gd["dL_dKmn"], Z, X)
        g += kern.gradient.copy()
        kern.update_gradients_diag(gd["dL_dKdiag"], X)
        g += kern.gradient.copy()
        mu, var = post._raw_predict(kern, Xnew, Z)
        o = so.svgp_eval(parts, X, Y, Z, q_m, q_L, so.make_likelihood(lik_spec, mods) if lik_spec != "poisson"
                         else so.PoissonVE(), bs)
        out.update(grad=g, dZ=kern.gradients_X(gd["dL_dKmm"], Z) + kern.gradients_X(gd["dL_dKmn"], Z, X),
                   dL_dthetaL=np.zeros(0) if gd["dL_dthetaL"] is None else np.asarray(gd["dL_dthetaL"]).reshape(-1),
                   pmu=mu[:, 0], pvar=var[:, 0], cond_Kmm=o["cond_Kmm"], cond_Kmm_jit=o["cond_Kmm_jit"],
                   jitter=o["jitter"], cond_S=o["cond_S"])
    return out


def main():
    os.makedirs(OUT, exist_ok=True)
    for name in sorted(so.CASES) + [ZERO_DIAG]:
        out = reference_case(name)
        np.savez_compressed(os.path.join(OUT, name + ".npz"), **out)
        print(name, out["lml"], out.get("cond_Kmm_jit"))


if __name__ == "__main__":
    main()
