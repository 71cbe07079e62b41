"""Test-only NumPy restatement of one sparse GPLVM evaluation (GPy/models/sparse_gplvm.py:29-34 on
SparseGP.parameters_changed, sparse_gp.py:76-119): the VarDTC evaluation of a composite kernel (oracle/gpy_oracle
.vardtc_inference), then X.gradient = kern.gradients_X_diag(dL_dKdiag, X) + kern.gradients_X(dL_dKnm, X, Z). The diagonal
term is zero for every stationary and static kernel (stationary.py:360-361, static.py:30-31). The kernel is a
sparse_composite_oracle.CompositeOracle. The reference fixtures' cases (tests/golden/make_sparse_gplvm.py) are listed here
so that the generator and the tests build the same inputs.
"""
import numpy as np

from oracle import gpy_oracle as o
from sparse_composite_oracle import CompositeOracle
from gplvm_oracle import latent_data


def sparse_gplvm_eval(X, Y, Z, parts, noise):
    """-> (lml, grad [X row-major, Z row-major, every leaf's block in order, noise], dX (N x Q), res of vardtc_inference).
    noise: a scalar, or one variance per data point (then grad has no noise entry)."""
    X = np.ascontiguousarray(X, dtype=np.float64)
    Z = np.ascontiguousarray(Z, dtype=np.float64)
    kern = CompositeOracle(parts)
    res = o.vardtc_inference(kern, X, Z, noise, np.ascontiguousarray(Y, dtype=np.float64))
    g0 = kern.grads_diag(res["dL_dKdiag"], X)                                   # sparse_gp.py:110
    g1 = kern.grads_full(res["dL_dKnm"], X, Z)                                  # :112
    g2 = kern.grads_full(res["dL_dKmm"], Z, None)                               # :114
    kgrad = np.concatenate([a + b + c for a, b, c in zip(g0, g1, g2)])
    dZ = kern.gradients_X(res["dL_dKmm"], Z) + kern.gradients_X(res["dL_dKnm"].T, Z, X)   # :117-118
    dX = kern.gradients_X(res["dL_dKnm"], X, Z)                                 # sparse_gplvm.py:34
    tail = [[res["dL_dthetaL"]]] if np.ndim(noise) == 0 else []
    grad = np.concatenate([dX.reshape(-1), dZ.reshape(-1), kgrad] + tail)
    return res["log_marginal"], grad, dX, res


def case_inputs(case):
    """Y (N x P) of a fixture case and its new latent points Xnew (7 x Q)"""
    _, Y = latent_data(case["N"], 3, case["P"], case["data_seed"])
    Xnew = np.random.default_rng(case["data_seed"] + 1).uniform(-1.5, 1.5, size=(7, case["Q"]))
    return Y, Xnew


def default_parts(Q, variance=1.0, lengthscale=1.0):
    """SparseGPRegression's default kernel RBF(input_dim), isotropic (sparse_gp_regression.py:36-37)"""
    return [dict(kind="rbf", term=0, dims=list(range(Q)), variance=variance, lengthscale=lengthscale)]


# kernels by namespace (the reference's classes or gpy_b200's), and the same kernel as CompositeOracle parts
def _rbf_ard_bias_white(ns):
    return ns["RBF"](2, 1.2, [0.8, 1.3], ARD=True) + ns["Bias"](2, 0.1) + ns["White"](2, 0.05)


def _rbf_ard_bias_white_parts(Q):
    return [dict(kind="rbf", term=0, dims=[0, 1], variance=1.2, lengthscale=[0.8, 1.3], ARD=True),
            dict(kind="bias", term=1, variance=0.1), dict(kind="white", term=2, variance=0.05)]


def _m32_x_rbf_bias(ns):
    return ns["Matern32"](2, variance=0.9, lengthscale=1.2) * ns["RBF"](2, variance=1.1, lengthscale=[0.7, 1.5], ARD=True) \
        + ns["Bias"](2, 0.2)


def _m32_x_rbf_bias_parts(Q):
    return [dict(kind="matern32", term=0, dims=[0, 1], variance=0.9, lengthscale=1.2),
            dict(kind="rbf", term=0, dims=[0, 1], variance=1.1, lengthscale=[0.7, 1.5], ARD=True),
            dict(kind="bias", term=1, variance=0.2)]


CASES = {
    "default_p1": dict(N=70, P=1, Q=2, M=10, seed=31, data_seed=21, noise=0.2, kernel=None),
    "default_p8": dict(N=90, P=8, Q=3, M=12, seed=32, data_seed=22, noise=0.25, kernel=None),
    "default_p9": dict(N=80, P=9, Q=2, M=10, seed=33, data_seed=23, noise=0.3, kernel=None),
    "default_p12": dict(N=100, P=12, Q=2, M=15, seed=34, data_seed=24, noise=0.3, kernel=None),
    "default_p64": dict(N=120, P=64, Q=3, M=20, seed=35, data_seed=25, noise=0.3, kernel=None),
    "default_p257": dict(N=150, P=257, Q=2, M=16, seed=36, data_seed=26, noise=0.3, kernel=None),
    "rbf_ard_bias_white": dict(N=60, P=5, Q=2, M=9, seed=37, data_seed=27, noise=0.4, kernel=_rbf_ard_bias_white,
                               parts=_rbf_ard_bias_white_parts),
    "m32_x_rbf_bias": dict(N=75, P=4, Q=2, M=11, seed=38, data_seed=28, noise=0.3, kernel=_m32_x_rbf_bias,
                           parts=_m32_x_rbf_bias_parts),
    # M not a multiple of the 128-row tile, N past one tile row
    "default_n1300_m129": dict(N=1300, P=3, Q=2, M=129, seed=39, data_seed=29, noise=0.2, kernel=None),
    # as many inducing points as data points: dL_dKnm is square, its orientation decides the answer
    "default_n_eq_m": dict(N=40, P=3, Q=2, M=40, seed=40, data_seed=30, noise=0.3, kernel=None),
}


def case_parts(case, Q):
    return case["parts"](Q) if case.get("parts") else default_parts(Q)


def reference_sparse_gplvm():
    """the reference's own SparseGPLVM class (GPy/models/sparse_gplvm.py verbatim over oracle/ref_gpy.py's SparseGP, Add /
    Prod and static kernels; build container only) and its kernel classes by name.

    The paramz stand-in's Param is not an ObsAr, so GP.__init__ (gp.py:42-45) would wrap the latent Param into a plain
    ObsAr and link_parameter would then fail. The real Param IS an ObsAr (paramz/param.py), and GP.__init__ takes its
    copy; gp.py's name ObsAr is given that meaning here (an isinstance test that accepts a Param, and the stand-in ObsAr
    as constructor), without touching the stand-in itself."""
    import importlib
    import sys
    from oracle import ref_gpy
    M = ref_gpy.load_sparse_models()
    C = ref_gpy.load_combination()
    kern_pkg = sys.modules["GPy.kern"]
    kern_pkg.Bias, kern_pkg.White = C.Bias, C.White
    Param = importlib.import_module("paramz").Param
    sys.modules["GPy.core"].Param = Param
    gp_mod = sys.modules["GPy.core.gp"]
    if not getattr(gp_mod, "_param_is_obsar", False):
        real = gp_mod.ObsAr

        class _Meta(type):
            def __instancecheck__(cls, x):
                return isinstance(x, (real, Param))

            def __call__(cls, *a, **kw):
                return real(*a, **kw)

        gp_mod.ObsAr = _Meta("ObsAr", (object,), {})
        gp_mod._param_is_obsar = True
    sgplvm = importlib.import_module("GPy.models.sparse_gplvm")
    ns = dict(RBF=M.G.RBF, Exponential=M.G.Exponential, Matern32=M.G.Matern32, Matern52=M.G.Matern52, Bias=C.Bias,
              White=C.White, Add=C.Add, Prod=C.Prod)
    return sgplvm.SparseGPLVM, ns, M
