"""Writes tests/golden/posterior_samples/*.npz: the joint posterior of the reference's own GP and VarDTC posterior
(GPy/core/gp.py:601-629,735-786; GPy/inference/latent_function_inference/posterior.py:109-130,238-302) over its own
kernels (stationary.py, rbf.py, standard_periodic.py, add.py, prod.py, static.py), likelihoods and normalizer, executed
through oracle/ref_gpy.py:

    cov, cov_lik        GP.posterior_covariance_between_points(X1, X2) with include_likelihood off / on (X1, X2 of one
                        size, as the Gaussian likelihood's full-covariance noise term needs); the normalizer applied
    mu, Sigma           GP._raw_predict(Xnew, full_cov=True) (normalised space)
    fsim, rng_after     GP.posterior_samples_f(Xnew, S) after np.random.seed(SEED) (an SVD square root of Sigma), and
                        the legacy global RNG state after the call (its key array and position)

Run from the repository root where the reference tree exists:  python tests/golden/make_posterior_samples.py
The kernels and inputs are those of tests/wide_composites_oracle.py (parts) and sparse_composite_oracle.case_data."""
import importlib
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), HERE]

from oracle import ref_gpy  # noqa: E402
import make_wide_composites as mwc  # noqa: E402  (ref_kernel: the reference's composite for a list of parts)
import posterior_samples_cases as cases  # noqa: E402

SEED, S = 1234, 5
mwc.D = cases.D   # the input columns the static parts are built for


def main():
    Sm = ref_gpy.load_sparse_models()
    C = ref_gpy.load_combination()
    G = Sm.G
    sp = importlib.import_module("GPy.kern.src.standard_periodic")
    os.makedirs(os.path.join(HERE, "posterior_samples"), exist_ok=True)
    for name, c in cases.CASES.items():
        X, Y, Z, noise, X1, X2, Xnew = cases.inputs(c)
        kern = mwc.ref_kernel(G, C, sp, c["parts"])
        out = dict(X=X, Y=Y, X1=X1, X2=X2, Xnew=Xnew, noise=np.asarray(noise, dtype=np.float64), seed=SEED, size=S)
        if c.get("sparse"):
            post = G.VarDTC(limit=3).inference(kern, X, Z, G.Gaussian(variance=noise), Y, None)[0]
            m = types.SimpleNamespace(kern=kern, posterior=post, _predictive_variable=Z, mean_function=None,
                                      normalizer=None, output_dim=Y.shape[1])
            m._raw_predict = types.MethodType(Sm.GP._raw_predict, m)
            m.posterior_samples_f = types.MethodType(Sm.GP.posterior_samples_f, m)
            out["Z"] = Z
        else:
            if np.ndim(noise) > 0:
                meta = {"output_index": np.arange(X.shape[0])[:, None]}
                lik = G.HeteroscedasticGaussian(meta)
                lik.variance[:] = np.asarray(noise).reshape(lik.variance.shape)
            else:
                lik = G.Gaussian(variance=noise)
            m = Sm.GP(X, Y, kern, lik, Y_metadata=None if np.ndim(noise) == 0 else meta,
                      normalizer=True if c.get("normalizer") else None)
            out["cov"] = np.asarray(m.posterior_covariance_between_points(X1, X2, include_likelihood=False))
            if np.ndim(noise) == 0:
                out["cov_lik"] = np.asarray(m.posterior_covariance_between_points(X1, X2, include_likelihood=True))
        mu, Sigma = m._raw_predict(Xnew, full_cov=True)
        out.update(mu=np.asarray(mu), Sigma=np.asarray(Sigma))
        if not (c.get("normalizer") and Y.shape[1] > 1):   # gp.py:614-615 broadcasts std^2 over Sigma's last axis: fails
            np.random.seed(SEED)
            out["fsim"] = np.asarray(m.posterior_samples_f(Xnew, size=S))
            st = np.random.get_state()
            out.update(rng_key=st[1], rng_pos=np.int64(st[2]))
        np.savez_compressed(os.path.join(HERE, "posterior_samples", name + ".npz"), **out)
        print(name, {k: float(np.abs(v).max()) for k, v in out.items() if k in ("cov", "Sigma", "fsim")})


if __name__ == "__main__":
    main()
