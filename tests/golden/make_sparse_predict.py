"""Writes tests/golden/sparse_predict/*.npz: predictions of the reference's own VarDTC posterior
(GPy/inference/latent_function_inference/var_dtc.py:213 -> posterior.py:220-248, Posterior._raw_predict with pred_var = Z)
over its own kernels (stationary.py, rbf.py, add.py, prod.py, static.py) and likelihoods, executed through
oracle/ref_gpy.py:

    woodbury_vector, woodbury_inv   the posterior VarDTC.inference returns
    mu, var                         _raw_predict(kern, Xnew, Z, full_cov=False): var clipped at 1e-15 (posterior.py:248)
    mu_full, cov                    _raw_predict(kern, Xnew, Z, full_cov=True)

Run from the repository root where the reference tree exists:  python tests/golden/make_sparse_predict.py
The kernels and inputs are those of tests/sparse_predict_cases.py."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), HERE]

from oracle import ref_gpy  # noqa: E402
import make_sparse_composite as msc  # noqa: E402  (ref_kernel: the reference's composite for a list of parts)
import sparse_predict_cases as cases  # noqa: E402

msc.D = cases.D   # the input columns the static parts are built for


def main():
    Sm = ref_gpy.load_sparse_models()
    C = ref_gpy.load_combination()
    G = Sm.G
    os.makedirs(os.path.join(HERE, "sparse_predict"), exist_ok=True)
    for name, c in cases.CASES.items():
        X, Y, Z, noise, Xnew = cases.inputs(c)
        kern = msc.ref_kernel(C, G, c["parts"])
        het = np.ndim(noise) > 0
        meta = {"output_index": np.arange(X.shape[0])[:, None]} if het else None
        if het:
            lik = G.HeteroscedasticGaussian(meta)
            lik.variance[:] = np.asarray(noise).reshape(lik.variance.shape)
        else:
            lik = G.Gaussian(variance=noise)
        post = G.VarDTC(limit=3).inference(kern, X, Z, lik, Y, meta)[0]
        mu, var = post._raw_predict(kern, Xnew, Z, full_cov=False)
        mu_full, cov = post._raw_predict(kern, Xnew, Z, full_cov=True)
        out = dict(X=X, Y=Y, Z=Z, Xnew=Xnew, noise=np.asarray(noise, dtype=np.float64),
                   woodbury_vector=np.asarray(post.woodbury_vector), woodbury_inv=np.asarray(post.woodbury_inv),
                   mu=np.asarray(mu), var=np.asarray(var), mu_full=np.asarray(mu_full), cov=np.asarray(cov))
        np.savez_compressed(os.path.join(HERE, "sparse_predict", name + ".npz"), **out)
        print(name, {k: float(np.abs(out[k]).max()) for k in ("mu", "var", "cov")}, "min var", float(out["var"].min()))


if __name__ == "__main__":
    main()
