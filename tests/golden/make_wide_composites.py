"""Writes tests/golden/wide_composites/*.npz: exact GP regression and GP.predictive_gradients with composite kernels on 64
input columns, produced by the reference's own Add, Prod, RBF, Exponential, Matern32 / 52, RatQuad, StdPeriodic, White,
Bias, Gaussian likelihood and ExactGaussianInference (GPy/kern/src/add.py, prod.py, stationary.py, rbf.py,
standard_periodic.py, static.py; GPy/inference/latent_function_inference/exact_gaussian_inference.py; GPy/core/gp.py),
executed through oracle/ref_gpy.py.

Run from the repository root where the reference tree exists:  python tests/golden/make_wide_composites.py
The kernels and inputs are those of tests/wide_composites_oracle.py (fixture_kernels, data)."""
import importlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

from oracle import ref_gpy  # noqa: E402
import wide_composites_oracle as wo  # noqa: E402

N, D, MS = 300, wo.FIXTURE_D, 9
# (kernel, P, noise, seed, predictive gradients)
CASES = [("ratquad_ard64", 1, 0.08, 501, False), ("periodic32_x_rbf", 1, 0.08, 502, False),
         ("eight_parts64", 1, 0.08, 503, False), ("pg_sumd17", 8, 0.08, 504, True), ("pg_sumd64", 8, 0.08, 505, True)]


def ref_kernel(G, C, sp, parts):
    """the reference's own composite for a list of part dicts: Add over terms of Prod over factors"""
    leaves = {}
    for p in parts:
        kind = p["kind"]
        if kind in ("white", "bias"):
            k = (C.White if kind == "white" else C.Bias)(D, variance=p["variance"])
        elif kind == "ratquad":
            k = G.stationary.RatQuad(len(p["dims"]), variance=p["variance"], lengthscale=p["lengthscale"], power=p["power"],
                                     ARD=p["ARD"], active_dims=p["dims"])
        elif kind == "stdperiodic":
            k = sp.StdPeriodic(len(p["dims"]), variance=p["variance"], period=p["period"], lengthscale=p["lengthscale"],
                               ARD1=p["ARD_period"], ARD2=p["ARD"], active_dims=p["dims"])
        else:
            cls = {"rbf": G.RBF, "exponential": G.Exponential, "matern32": G.Matern32, "matern52": G.Matern52}[kind]
            k = cls(len(p["dims"]), variance=p["variance"], lengthscale=p["lengthscale"], ARD=p["ARD"], active_dims=p["dims"])
        leaves.setdefault(p["term"], []).append(k)
    terms = [ks[0] if len(ks) == 1 else C.Prod(ks) for _, ks in sorted(leaves.items())]
    return terms[0] if len(terms) == 1 else C.Add(terms)


def _grad_of(kern):
    return np.concatenate([np.atleast_1d(np.asarray(p.gradient, dtype=np.float64)).reshape(-1) * np.ones(p.size)
                           for p in kern.flattened_parameters()])


def main():
    S = ref_gpy.load_sparse_models()
    C = ref_gpy.load_combination()
    G = S.G
    sp = importlib.import_module("GPy.kern.src.standard_periodic")
    kernels = wo.fixture_kernels()
    os.makedirs(os.path.join(HERE, "wide_composites"), exist_ok=True)
    for name, P, noise, seed, pg in CASES:
        X, Y = wo.data(N, D, P, seed)
        kern = ref_kernel(G, C, sp, kernels[name])
        out = dict(X=X, Y=Y, noise=np.float64(noise), kernel=name, seed=seed)
        if pg:   # GP.predictive_gradients (gp.py:418-474) on the reference's own exact posterior
            m = S.GP(X, Y, kern, G.Gaussian(variance=noise))
            Xnew = np.random.default_rng(seed + 1).uniform(-2.0, 2.0, (MS, D))
            mean_jac, var_jac = m.predictive_gradients(Xnew)
            out.update(Xnew=Xnew, mean_jac=np.asarray(mean_jac), var_jac=np.asarray(var_jac))
        else:    # the three calls of GP.parameters_changed (gp.py:278-280)
            lik = G.Gaussian(variance=noise)
            post, lml, gd = G.ExactGaussianInference().inference(kern, X, lik, Y, None, None)
            lik.update_gradients(gd["dL_dthetaL"])
            kern.update_gradients_full(gd["dL_dK"], X)
            out.update(lml=np.float64(lml), alpha=np.asarray(post.woodbury_vector),
                       grad=np.concatenate([_grad_of(kern), np.atleast_1d(lik.variance.gradient).reshape(-1)]))
        np.savez_compressed(os.path.join(HERE, "wide_composites", name + ".npz"), **out)
        print(name, {k: float(np.abs(v).max()) for k, v in out.items() if k in ("lml", "mean_jac", "var_jac")})


if __name__ == "__main__":
    main()
