"""Writes tests/golden/vargauss/*.npz: the variational Gaussian approximation as the reference's own VarGauss.inference
(GPy/inference/latent_function_inference/var_gauss.py:34-69) computes it with its likelihoods and kernels, executed
through oracle/ref_gpy.py, with the kernel gradient of GPy/core/gp.py:280:

    X, Y, alpha, beta                    the inputs (theta is the case's kernel in tests/vargauss_oracle.py)
    m, var, F, dF_dm, dF_dv, KL, lml     what the reference computed and handed its likelihood
    dalpha, dbeta, dL_dthetaL            alpha.gradient, beta.gradient and dL_dthetaL
    grad_ref                             the reference's kernel gradient (its row-scaled dF_dK)
    pmu, pvar                            Posterior(mean, cov, K)._raw_predict at Xnew (only where cond(K) < 1e8: the
                                         reference forms them through jitchol(K))
    cond_K, cond_A                       cond(K) and cond(I + B K B)

Run from the repository root where the reference tree exists:  python tests/golden/make_vargauss.py"""
import importlib
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), HERE]

import vargauss_oracle as vo  # noqa: E402
import make_laplace as ml  # noqa: E402
from ep_reference import load_reference_ep  # noqa: E402

OUT = os.path.join(HERE, "vargauss")


class _Capture(object):
    """the reference's likelihood, recording what its variational_expectations receives and returns"""

    def __init__(self, lik):
        self.lik = lik

    def variational_expectations(self, Y, m, v, Y_metadata=None):
        out = self.lik.variational_expectations(Y, m, v, Y_metadata=Y_metadata)
        self.m, self.v, self.F, self.dF_dm, self.dF_dv = m[:, 0].copy(), v[:, 0].copy(), out[0], out[1], out[2]
        return out


def reference_modules():
    load_reference_ep()
    return (importlib.import_module("GPy.inference.latent_function_inference.var_gauss"),
            types.SimpleNamespace(Bernoulli=importlib.import_module("GPy.likelihoods.bernoulli").Bernoulli,
                                  StudentT=importlib.import_module("GPy.likelihoods.student_t").StudentT,
                                  Gaussian=importlib.import_module("GPy.likelihoods.gaussian").Gaussian,
                                  Poisson=importlib.import_module("GPy.likelihoods.poisson").Poisson))


def reference_likelihood(spec, mods):
    return mods.Poisson() if spec == "poisson" else vo.make_likelihood(spec, mods)


def reference_inference(parts, lik_spec, X, Y, alpha, beta):
    """the reference's VarGauss.inference -> (posterior, lml, grad dict, kernel, captured likelihood, alpha, beta)"""
    vg, mods = reference_modules()
    from paramz import Param
    kern = ml.reference_kernel(parts, X.shape[1])
    lik = _Capture(reference_likelihood(lik_spec, mods))
    a, b = Param("alpha", alpha.reshape(-1, 1).copy()), Param("beta", beta.copy())
    post, lml, gd = vg.VarGauss(a, b).inference(kern, X, lik, Y)
    kern.update_gradients_full(gd["dL_dK"], X)
    return post, lml, gd, kern, lik, a, b


def reference_case(name):
    parts, lik_spec, N, seed, _ = vo.CASES[name]
    X, Y, alpha, beta, Xnew = vo.case_data(name)
    post, lml, gd, kern, lik, a, b = reference_inference(parts, lik_spec, X, Y, alpha, beta)
    K = np.asarray(kern.K(X))
    A = np.eye(N) + K * beta[:, None] * beta[None, :]
    out = dict(X=X, Y=Y, alpha=alpha, beta=beta, Xnew=Xnew, m=lik.m, var=lik.v, F=np.asarray(lik.F)[:, 0],
               dF_dm=np.asarray(lik.dF_dm)[:, 0], dF_dv=np.asarray(lik.dF_dv)[:, 0], lml=float(lml),
               KL=float(np.sum(lik.F) - lml), dalpha=np.asarray(a.gradient)[:, 0], dbeta=np.asarray(b.gradient).copy(),
               dL_dthetaL=np.asarray(gd["dL_dthetaL"], dtype=np.float64).reshape(-1),
               grad_ref=np.asarray(kern.gradient, dtype=np.float64).copy(), cond_K=np.linalg.cond(K),
               cond_A=np.linalg.cond(A))
    if out["cond_K"] < 1e8:
        mu, var = post._raw_predict(kern, Xnew, X)
        out.update(pmu=np.asarray(mu)[:, 0], pvar=np.asarray(var)[:, 0])
    return out


def main():
    os.makedirs(OUT, exist_ok=True)
    for name in sorted(vo.CASES):
        out = reference_case(name)
        np.savez_compressed(os.path.join(OUT, name + ".npz"), **out)
        print(name, out["lml"], "cond_K %.3g cond_A %.3g" % (out["cond_K"], out["cond_A"]), "pmu" in out)


if __name__ == "__main__":
    main()
