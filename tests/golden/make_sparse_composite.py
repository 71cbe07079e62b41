"""Writes tests/golden/sparse_composite/*.npz: sparse GP regression (VarDTC) with composite kernels, produced by the
reference's own VarDTC, Add, Prod, White, Bias and stationary kernels (GPy/inference/latent_function_inference/var_dtc.py,
GPy/kern/src/add.py, prod.py, static.py, stationary.py, rbf.py, executed through oracle/ref_gpy.py), with the gradient
wiring of GPy/core/sparse_gp.py:108-119 and, for per-point noise, the reference's HeteroscedasticGaussian.

Run from the repository root where the reference tree exists:  python tests/golden/make_sparse_composite.py
The kernels and inputs are those of tests/sparse_composite_oracle.py (KERNELS, case_data)."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

from oracle import ref_gpy  # noqa: E402
import sparse_composite_oracle as so  # noqa: E402

N, M, D = 300, 40, 3
CASES = [(kname, P, het, 100 + 10 * i + 2 * (P - 1) + int(het))
         for i, kname in enumerate(sorted(so.KERNELS)) for P in (1, 2) for het in (False, True)]


def ref_kernel(C, G, parts):
    """the reference's own composite for a list of part dicts: Add over terms of Prod over factors"""
    leaves = {}
    for p in parts:
        if p["kind"] == "white":
            k = C.White(D, variance=p["variance"])
        elif p["kind"] == "bias":
            k = C.Bias(D, variance=p["variance"])
        else:
            cls = {"rbf": G.RBF, "exponential": G.Exponential, "matern32": G.Matern32, "matern52": G.Matern52}[p["kind"]]
            k = cls(len(p["dims"]), variance=p["variance"], lengthscale=p["lengthscale"], ARD=p.get("ARD", False),
                    active_dims=p["dims"])
        leaves.setdefault(p["term"], []).append(k)
    terms = [ks[0] if len(ks) == 1 else C.Prod(ks) for _, ks in sorted(leaves.items())]
    return terms[0] if len(terms) == 1 else C.Add(terms)


def evaluate(C, G, X, Y, Z, parts, noise):
    kern = ref_kernel(C, G, parts)
    het = np.ndim(noise) > 0
    meta = {"output_index": np.arange(X.shape[0])[:, None]} if het else None
    if het:
        lik = G.HeteroscedasticGaussian(meta)
        lik.variance[:] = np.asarray(noise).reshape(lik.variance.shape)
    else:
        lik = G.Gaussian(variance=noise)
    post, lml, gd = G.VarDTC(limit=3).inference(kern, X, Z, lik, Y, meta)      # sparse_gp.py:77-80
    kern.update_gradients_diag(gd["dL_dKdiag"], X)                             # :110
    kg = kern.gradient.copy()
    kern.update_gradients_full(gd["dL_dKnm"], X, Z)                            # :112
    kg += kern.gradient
    kern.update_gradients_full(gd["dL_dKmm"], Z, None)                         # :114
    kg += kern.gradient
    Zg = kern.gradients_X(gd["dL_dKmm"], Z)                                    # :117
    Zg = Zg + kern.gradients_X(gd["dL_dKnm"].T, Z, X)                          # :118
    out = dict(lml=float(np.squeeze(lml)), Zgrad=np.asarray(Zg), woodbury_vector=np.asarray(post.woodbury_vector),
               woodbury_inv=np.asarray(post.woodbury_inv), Kmm=np.asarray(kern.K(Z)))
    if het:
        out["grad"] = np.asarray(kg, dtype=np.float64)
        out["dL_dR"] = np.asarray(gd["dL_dthetaL"], dtype=np.float64).reshape(X.shape[0], Y.shape[1])
    else:
        out["grad"] = np.concatenate([np.asarray(kg, dtype=np.float64), [float(np.sum(gd["dL_dthetaL"]))]])
    return out


def main():
    S = ref_gpy.load_sparse_models()
    C = ref_gpy.load_combination()
    G = S.G
    os.makedirs(os.path.join(HERE, "sparse_composite"), exist_ok=True)
    for kname, P, het, seed in CASES:
        X, Y, Z, noise = so.case_data(N, M, D, P, seed, het)
        r = evaluate(C, G, X, Y, Z, so.KERNELS[kname], noise)
        name = "%s_p%d_%s" % (kname, P, "het" if het else "scalar")
        np.savez_compressed(os.path.join(HERE, "sparse_composite", name + ".npz"), X=X, Y=Y, Z=Z,
                            noise=np.asarray(noise, dtype=np.float64), kernel=kname, seed=seed, **r)
        print(name, r["lml"])


if __name__ == "__main__":
    main()
