"""Test-only NumPy restatement of one GPLVM evaluation (GPy/models/gplvm.py:46-49 on GP.parameters_changed, gp.py:269-282):
the exact evaluation of a composite kernel, then X.gradient = kern.gradients_X(dL_dK, X, None) with
dL_dK = 1/2 (alpha alpha^T - P Ky^-1) (exact_gaussian_inference.py:70). The kernel is a sparse_composite_oracle
.CompositeOracle; the reference fixtures' cases (tests/golden/make_gplvm.py) are listed here so that the generator and the
tests build the same inputs.
"""
import numpy as np

from oracle import gpy_oracle as o
from sparse_composite_oracle import CompositeOracle


def gplvm_eval(X, Y, parts, noise):
    """-> (lml, grad [every leaf's block in order, noise], dX (N x Q), res of gpy_oracle.exact_inference)"""
    kern = CompositeOracle(parts)
    res = o.exact_inference(kern, X, Y, noise)
    grad = np.concatenate(kern.grads_full(res["dL_dK"], X) + [[res["dL_dthetaL"]]])
    return res["log_marginal"], grad, kern.gradients_X(res["dL_dK"], X), res


def latent_data(N, Q, P, seed):
    """latent points X (N x Q) and observations Y (N x P): smooth functions of X plus noise"""
    rng = np.random.default_rng(seed)
    X = rng.uniform(-1.5, 1.5, size=(N, Q))
    W = rng.standard_normal((Q, P))
    Y = np.sin(X.dot(W) + np.arange(P)) + 0.3 * np.cos(2.0 * X[:, :1]) + 0.05 * rng.standard_normal((N, P))
    return X, Y


def case_inputs(case):
    """Y (N x P) of a fixture case and its new latent points Xnew (7 x Q)"""
    _, Y = latent_data(case["N"], 3, case["P"], case["data_seed"])
    Xnew = np.random.default_rng(case["data_seed"] + 1).uniform(-1.5, 1.5, size=(7, case["Q"]))
    return Y, Xnew


# kernels by namespace (the reference's classes or gpy_b200's): None is GPLVM's default RBF(ARD) + Bias(exp(-2))
def _rbf_bias_white(ns):     # the kernel of the reference's test_GPLVM_rbf_bias_white_kern_2D
    return ns["RBF"](2, 0.5, 0.9 * np.ones(1), ARD=False) + ns["Bias"](2, 0.1) + ns["White"](2, 0.05)


def _matern52_ard(ns):
    return ns["Matern52"](2, variance=1.3, lengthscale=[0.8, 1.4], ARD=True)


def _m32_x_rbf_bias(ns):
    return ns["Matern32"](2, variance=0.9, lengthscale=1.2) * ns["RBF"](2, variance=1.1, lengthscale=[0.7, 1.5], ARD=True) \
        + ns["Bias"](2, 0.2)


CASES = {
    "default_p3": dict(N=80, P=3, Q=2, seed=11, data_seed=1, noise=0.3, kernel=None),
    "default_p1": dict(N=70, P=1, Q=1, seed=12, data_seed=2, noise=0.2, kernel=None),
    "default_p8_q3": dict(N=90, P=8, Q=3, seed=13, data_seed=3, noise=0.25, kernel=None),
    "rbf_bias_white": dict(N=60, P=5, Q=2, seed=14, data_seed=4, noise=0.4, kernel=_rbf_bias_white),
    "matern52_ard_n1300": dict(N=1300, P=3, Q=2, seed=15, data_seed=5, noise=0.2, kernel=_matern52_ard),
    "m32_x_rbf_bias": dict(N=75, P=4, Q=2, seed=16, data_seed=6, noise=0.3, kernel=_m32_x_rbf_bias),
    "default_normalizer": dict(N=65, P=4, Q=2, seed=17, data_seed=7, noise=0.3, kernel=None, normalizer=True),
    # more output columns than the narrow route's 8: the wide route
    "default_p9": dict(N=70, P=9, Q=2, seed=18, data_seed=8, noise=0.3, kernel=None),
    "default_p64": dict(N=100, P=64, Q=3, seed=19, data_seed=9, noise=0.3, kernel=None),
    "matern52_ard_p257": dict(N=150, P=257, Q=2, seed=20, data_seed=10, noise=0.3, kernel=_matern52_ard),
}


def reference_gplvm():
    """the reference's own GPLVM class (GPy/models/gplvm.py verbatim over oracle/ref_gpy.py's GP, Add / Prod and static
    kernels; build container only) and its kernel classes by name"""
    import importlib
    import sys
    from oracle import ref_gpy
    M = ref_gpy.load_models()
    C = ref_gpy.load_combination()
    kern_pkg = sys.modules["GPy.kern"]
    kern_pkg.Bias, kern_pkg.White = C.Bias, C.White                     # names gplvm.py:8 reads from GPy.kern
    sys.modules["GPy.core"].Param = importlib.import_module("paramz").Param
    sys.modules["GPy.likelihoods"].Gaussian = M.G.Gaussian
    gplvm = importlib.import_module("GPy.models.gplvm")
    ns = dict(RBF=M.G.RBF, Exponential=M.G.Exponential, Matern32=M.G.Matern32, Matern52=M.G.Matern52, Bias=C.Bias,
              White=C.White, Add=C.Add, Prod=C.Prod)
    return gplvm.GPLVM, ns
