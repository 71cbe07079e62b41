"""The cases of the joint-posterior fixtures (tests/golden/make_posterior_samples.py): kernels as part dicts of
tests/wide_composites_oracle.py and the inputs of each case."""
import numpy as np

import wide_composites_oracle as wo
from sparse_composite_oracle import case_data

N, M, D, MS = 150, 30, 3, 9

MAUNA_LOA = [wo.stationary("rbf", [0, 1, 2], 0, False, variance=1.5, scale=2.0),
             wo.stationary("rbf", [0], 1, False, variance=0.6), wo.stdperiodic([0], 1, False, False),
             wo.ratquad([1, 2], 2, False, power=0.7, variance=0.4),
             wo.stationary("rbf", [2], 3, False, variance=0.1, scale=0.3), wo.static("white", 3, 0.02)]

CASES = {
    "exact_rbf_ard": dict(parts=[wo.stationary("rbf", [0, 1, 2], 0, True, variance=0.9)], P=1, seed=601),
    "exact_matern32_iso": dict(parts=[wo.stationary("matern32", [0, 1, 2], 0, False, variance=1.2)], P=1, seed=602),
    "exact_m52_x_rbf_bias_white": dict(parts=[wo.stationary("matern52", [0, 1], 0, False, variance=1.1),
                                              wo.stationary("rbf", [1, 2], 0, True, variance=0.8),
                                              wo.static("bias", 1, 0.4), wo.static("white", 2, 0.07)], P=1, seed=603),
    "exact_mauna_loa": dict(parts=MAUNA_LOA, P=1, seed=604),
    "exact_rbf_ard_het": dict(parts=[wo.stationary("rbf", [0, 1, 2], 0, True, variance=0.9)], P=1, seed=605, het=True),
    "exact_m52_p3_norm": dict(parts=[wo.stationary("matern52", [0, 1, 2], 0, True, variance=1.0)], P=3, seed=606,
                              normalizer=True),
    "exact_rbf_p1_norm": dict(parts=[wo.stationary("rbf", [0, 1, 2], 0, False, variance=1.0)], P=1, seed=607,
                              normalizer=True),
    "sparse_rbf_ard": dict(parts=[wo.stationary("rbf", [0, 1, 2], 0, True, variance=0.9)], P=1, seed=608, sparse=True),
}


def inputs(c):
    """-> X, Y, Z, noise, X1, X2, Xnew of a case (Y scaled and shifted where a normalizer is used)"""
    X, Y, Z, noise = case_data(N, M, D, c["P"], c["seed"], c.get("het", False))
    if c.get("normalizer"):
        Y = 2.5 * Y + np.arange(1, c["P"] + 1)
    rng = np.random.default_rng(c["seed"] + 1)
    X1, X2, Xnew = (rng.uniform(-2.0, 2.0, size=(MS, D)) for _ in range(3))
    return X, Y, Z, noise, X1, X2, Xnew
