"""Writes tests/golden/fitc/*.npz: FITC sparse GP regression produced by the reference's own FITC
(GPy/inference/latent_function_inference/fitc.py), Gaussian likelihood and kernels (stationary.py, rbf.py, add.py,
prod.py, static.py), executed through oracle/ref_gpy.py, with the gradient wiring of GPy/core/sparse_gp.py:108-118:

    lml, grad, Zgrad, dL_dKdiag        the bound, [kernel gradient (paramz order), noise], Z.gradient, dL_dR (fitc.py:67)
    woodbury_vector, mu, var           the posterior's v and its predictions at Xnew (posterior.py:220-248)
    woodbury_inv, K, K_chol            only for M = 50 (Kmm^-1 - P, Kmm + 1e-6 I, L of fitc.py:86)

Run from the repository root where the reference tree exists:  python tests/golden/make_fitc.py
The kernels and inputs are those of tests/fitc_oracle.py (CASES, case_data)."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), HERE]

from oracle import ref_gpy  # noqa: E402
import fitc_oracle as fo  # noqa: E402


def main():
    os.makedirs(os.path.join(HERE, "fitc"), exist_ok=True)
    for name in fo.CASES:
        X, Y, Z, noise, Xnew = fo.case_data(name)
        r = fo.reference_fitc(ref_gpy, X, Y, Z, fo.CASES[name][0], noise, Xnew)
        if Z.shape[0] != fo.SMALL_M:
            for k in ("woodbury_inv", "K", "K_chol"):
                del r[k]
        np.savez_compressed(os.path.join(HERE, "fitc", name + ".npz"), X=X, Y=Y, Z=Z, Xnew=Xnew, noise=noise, **r)
        sig = 1.0 / np.abs(r["dL_dKdiag"]).max()
        print(name, r["lml"], "max |grad|", float(np.abs(r["grad"]).max()), sig)


if __name__ == "__main__":
    main()
