"""Writes tests/golden/predictive_gradients/*.npz: GP.predictive_gradients (GPy/core/gp.py:418-474) of the reference's own
GP and SparseGP (GPy/core/gp.py, GPy/core/sparse_gp.py) over its own kernels (stationary.py, rbf.py, add.py, prod.py,
static.py), likelihoods and inference, executed through oracle/ref_gpy.py.

Run from the repository root where the reference tree exists:  python tests/golden/make_predictive_gradients.py
The kernels and inputs are those of tests/predictive_gradients_oracle.py (KERNELS, case_data)."""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), HERE]

from oracle import ref_gpy  # noqa: E402
import make_sparse_composite as msc  # noqa: E402  (ref_kernel: the reference's composite for a list of parts)
import predictive_gradients_oracle as po  # noqa: E402

N, M, D, MS = 150, 30, 3, 9
# (name, kernel, P, het, normalizer, sparse, seed); "illcond": the noise is set so that cond(Ky) is about 1e8
CASES = ([("exact_%s" % k, k, 1, False, False, False, 300 + i) for i, k in enumerate(sorted(po.KERNELS))]
         + [("exact_rbf_bias_white_p3", "rbf_bias_white", 3, False, False, False, 331),
            ("exact_rbf_ard_p1_norm", "rbf_ard", 1, False, True, False, 332),
            ("exact_m52_x_rbf_p3_norm", "m52_x_rbf", 3, False, True, False, 333),
            ("exact_rbf_ard_het", "rbf_ard", 1, True, False, False, 334),
            ("exact_rbf_ard_illcond", "rbf_ard", 1, False, False, False, 335),
            ("sparse_rbf_ard_scalar", "rbf_ard", 1, False, False, True, 336),
            ("sparse_rbf_bias_white_het", "rbf_bias_white", 1, True, False, True, 337),
            ("sparse_m52_x_rbf_p3_scalar", "m52_x_rbf", 3, False, False, True, 338)])


def likelihood(G, noise, n):
    if np.ndim(noise) > 0:
        meta = {"output_index": np.arange(n)[:, None]}
        lik = G.HeteroscedasticGaussian(meta)
        lik.variance[:] = np.asarray(noise).reshape(lik.variance.shape)
        return lik, meta
    return G.Gaussian(variance=noise), None


def main():
    S = ref_gpy.load_sparse_models()
    C = ref_gpy.load_combination()
    G = S.G
    os.makedirs(os.path.join(HERE, "predictive_gradients"), exist_ok=True)
    for name, kname, P, het, norm, sparse, seed in CASES:
        X, Y, Z, noise = po.case_data(N, M, D, P, seed, het)
        Xnew = np.random.default_rng(seed + 1).uniform(-2.0, 2.0, size=(MS, D))
        kern = msc.ref_kernel(C, G, po.KERNELS[kname])
        extra = {}
        if name.endswith("illcond"):
            lam = np.linalg.eigvalsh(kern.K(X))
            noise = lam[-1] / 2e8 - po.JITTER
            extra["cond"] = np.float64(np.linalg.cond(kern.K(X) + (noise + po.JITTER) * np.eye(N)))
        lik, meta = likelihood(G, noise, N)
        if sparse:   # the reference's GP.predictive_gradients on its VarDTC posterior, predictive variable Z (sparse_gp.py:52-54)
            post = G.VarDTC(limit=3).inference(kern, X, Z, lik, Y, meta)[0]
            m = types.SimpleNamespace(kern=kern, posterior=post, _predictive_variable=Z, output_dim=P, normalizer=None)
            m.predictive_gradients = types.MethodType(S.GP.predictive_gradients, m)
        else:
            m = S.GP(X, Y, kern, lik, Y_metadata=meta, normalizer=True if norm else None)
        mean_jac, var_jac = m.predictive_gradients(Xnew)
        np.savez_compressed(os.path.join(HERE, "predictive_gradients", name + ".npz"), X=X, Y=Y, Z=Z, Xnew=Xnew,
                            noise=np.asarray(noise, dtype=np.float64), kernel=kname, normalizer=norm, sparse=sparse,
                            seed=seed, mean_jac=np.asarray(mean_jac), var_jac=np.asarray(var_jac), **extra)
        print(name, np.abs(mean_jac).max(), np.abs(var_jac).max(), extra)


if __name__ == "__main__":
    main()
