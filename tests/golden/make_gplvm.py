"""Writes tests/golden/gplvm/*.npz from the reference's own GPLVM (GPy/models/gplvm.py, GP, Add / Prod / static kernels and
util/initialization.py executed verbatim through oracle/ref_gpy.py). Each fixture records the latent initialisation (numpy
global seed `seed` right before the model is built), the log marginal likelihood, the full gradient in paramz order
[latent_mean (row-major), kernel.., noise] and predict at new latent points. Run from the repository root:
    python tests/golden/make_gplvm.py [case ...]      (no case: all of them)
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
OUT = os.path.join(ROOT, "tests", "golden", "gplvm")

from gplvm_oracle import CASES, case_inputs, reference_gplvm  # noqa: E402


def main():
    GPLVM, ns = reference_gplvm()
    os.makedirs(OUT, exist_ok=True)
    for name, case in CASES.items():
        if len(sys.argv) > 1 and name not in sys.argv[1:]:
            continue
        Y, Xnew = case_inputs(case)
        kern = case["kernel"](ns) if case["kernel"] is not None else None
        np.random.seed(case["seed"])
        m = GPLVM(Y, case["Q"], kernel=kern, normalizer=case.get("normalizer", False))
        X0 = np.array(m.X.values if hasattr(m.X, "values") else m.X, dtype=np.float64)
        m.likelihood.variance[:] = case["noise"]
        mu, var = m.predict(Xnew)
        np.savez(os.path.join(OUT, name + ".npz"), Y=Y, X0=X0, Xnew=Xnew, lml=float(m.log_likelihood()),
                 grad=np.asarray(m.gradient, dtype=np.float64).copy(), mu=np.asarray(mu), var=np.asarray(var),
                 seed=case["seed"], Q=case["Q"], noise=case["noise"])
        print(name, Y.shape, float(m.log_likelihood()))


if __name__ == "__main__":
    main()
