"""Writes tests/golden/sparse_gplvm/*.npz from the reference's own SparseGPLVM (GPy/models/sparse_gplvm.py,
SparseGPRegression, SparseGP, VarDTC, Add / Prod / static kernels and util/initialization.py executed verbatim through
oracle/ref_gpy.py). Each fixture records the numpy global seed set right before the model is built, the latent
initialisation X0, the inducing inputs Z0 the model drew, the log marginal likelihood, the full gradient in paramz order
[latent space (row-major), inducing inputs (row-major), kernel.., noise] and predict at new latent points.
The case `het` is the evaluation SparseGP.parameters_changed makes with a HeteroscedasticGaussian likelihood (the
reference's own VarDTC.inference, sparse_gp.py:77-80); it records the bound and kern.gradients_X(grad_dict['dL_dKnm'], X, Z)
from that grad dict as `dX`.
Run from the repository root:
    python tests/golden/make_sparse_gplvm.py [case ...]      (no case: all of them)
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
OUT = os.path.join(ROOT, "tests", "golden", "sparse_gplvm")

from gplvm_oracle import latent_data  # noqa: E402
from sparse_gplvm_oracle import CASES, case_inputs, reference_sparse_gplvm  # noqa: E402

HET = dict(N=90, P=1, Q=2, M=12, data_seed=41, seed=42)


def het_inputs():
    """latent X (N x Q), Y (N x P), Z (M x Q) and per-point noise variances of the `het` case"""
    X, Y = latent_data(HET["N"], HET["Q"], HET["P"], HET["data_seed"])
    rng = np.random.default_rng(HET["seed"])
    Z = X[rng.permutation(HET["N"])[:HET["M"]]].copy()
    noise = rng.uniform(0.1, 0.6, size=HET["N"])
    return X, Y, Z, noise


def main():
    SparseGPLVM, ns, M = reference_sparse_gplvm()
    os.makedirs(OUT, exist_ok=True)
    for name, case in CASES.items():
        if len(sys.argv) > 1 and name not in sys.argv[1:]:
            continue
        Y, Xnew = case_inputs(case)
        kern = case["kernel"](ns) if case["kernel"] is not None else None
        np.random.seed(case["seed"])
        m = SparseGPLVM(Y, case["Q"], kernel=kern, num_inducing=case["M"])
        X0 = np.array(m.X.values if hasattr(m.X, "values") else m.X, dtype=np.float64)
        Z0 = np.array(m.Z.values if hasattr(m.Z, "values") else m.Z, dtype=np.float64)
        m.likelihood.variance[:] = case["noise"]
        mu, var = m.predict(Xnew)
        np.savez(os.path.join(OUT, name + ".npz"), Y=Y, X0=X0, Z0=Z0, Xnew=Xnew, lml=float(m.log_likelihood()),
                 grad=np.asarray(m.gradient, dtype=np.float64).copy(), mu=np.asarray(mu), var=np.asarray(var),
                 seed=case["seed"], Q=case["Q"], noise=case["noise"])
        print(name, Y.shape, Z0.shape, float(m.log_likelihood()))
    if len(sys.argv) == 1 or "het" in sys.argv[1:]:
        X, Y, Z, noise = het_inputs()
        G = M.G
        kern = G.RBF(HET["Q"], 1.1, [0.9, 1.3], ARD=True)
        meta = {"output_index": np.arange(HET["N"])[:, None]}
        lik = G.HeteroscedasticGaussian(meta)
        lik.variance[:] = noise.reshape(lik.variance.shape)
        post, lml, gd = G.VarDTC().inference(kern, X, Z, lik, Y, meta)            # sparse_gp.py:77-80
        dX = np.asarray(kern.gradients_X(gd["dL_dKnm"], X, Z), dtype=np.float64)     # sparse_gplvm.py:34
        np.savez(os.path.join(OUT, "het.npz"), X=X, Y=Y, Z=Z, noise=noise, lml=float(lml), dX=dX)
        print("het", Y.shape, float(lml))


if __name__ == "__main__":
    main()
