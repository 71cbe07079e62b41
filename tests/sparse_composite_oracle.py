"""Test-only NumPy restatement of sparse GP regression (VarDTC) with a composite kernel: a sum of products of RBF ..
Matern52, White and Bias leaves, each stationary leaf on its own active dims.

The inference itself is oracle/gpy_oracle.vardtc_inference (var_dtc.py:66-276) run with the composite as its kernel. The
gradient wiring restates GPy/core/sparse_gp.py:108-119 leaf by leaf, the way the reference's Add and Prod hand it down:
    update_gradients_diag  Add passes dL_dKdiag to every term (add.py:79-80), Prod hands each factor dL_dKdiag times the
                           other factors' Kdiag (prod.py:386-394)
    update_gradients_full  the same with dL_dK and K (add.py:76-77, prod.py:377-385)
    gradients_X            Add sums its parts' (add.py:88-100); Prod hands each factor dL_dK times the other factors' K
                           (prod.py:397-407); White / Bias have none (static.py:41-42); a leaf on a subset of the columns
                           scatters its gradient into them (kernel_slice_operations.py:138-150)
`parts` are dicts(kind, term, dims, variance, [lengthscale, ARD]) as gpy_oracle.composite_parts takes them.
"""
import numpy as np

from oracle import gpy_oracle as o


class CompositeOracle(object):
    """K / Kdiag of the composite and its per-leaf gradient blocks (paramz order: variance, lengthscale..)."""

    def __init__(self, parts):
        self.parts = parts
        self.kparts = o.composite_parts(parts)

    def K(self, X, X2=None):
        return o.composite_K(self.kparts, X, X2)

    def Kdiag(self, X):
        return o.composite_Kdiag(self.kparts, X)

    def _others(self, i, fn):
        """product over the other factors of leaf i's term of fn(leaf kernel, dims), or None"""
        out = None
        t = self.kparts[i][2]
        for j, (k, dims, tj) in enumerate(self.kparts):
            if j != i and tj == t:
                v = fn(k, dims)
                out = v if out is None else out * v
        return out

    def grads_diag(self, dL_dKdiag, X):
        blocks = []
        for i, (k, dims, _) in enumerate(self.kparts):
            other = self._others(i, lambda k2, d2: k2.Kdiag(o._slice(X, d2)))
            g = dL_dKdiag if other is None else dL_dKdiag * other
            n = 0 if isinstance(k, o.StaticOracle) else k.lengthscale.size
            blocks.append(np.concatenate([[np.sum(g)], np.zeros(n)]))   # stationary.py:175-183, static.py:94-95
        return blocks

    def grads_full(self, dL_dK, X, X2=None):
        blocks = []
        for i, (k, dims, _) in enumerate(self.kparts):
            other = self._others(i, lambda k2, d2: k2.K(o._slice(X, d2), None if X2 is None else o._slice(X2, d2)))
            g = dL_dK if other is None else dL_dK * other
            dv, dl = k.update_gradients_full(g, o._slice(X, dims), None if X2 is None else o._slice(X2, dims))
            blocks.append(np.concatenate([[dv], np.atleast_1d(dl).reshape(-1)]))
        return blocks

    def gradients_X(self, dL_dK, X, X2=None):
        out = np.zeros(X.shape)
        for i, (k, dims, _) in enumerate(self.kparts):
            if isinstance(k, o.StaticOracle):
                continue
            other = self._others(i, lambda k2, d2: k2.K(o._slice(X, d2), None if X2 is None else o._slice(X2, d2)))
            g = dL_dK if other is None else dL_dK * other
            out[:, dims] += k.gradients_X(g, o._slice(X, dims), None if X2 is None else o._slice(X2, dims))
        return out


def sparse_composite_eval(X, Y, Z, parts, noise_variance):
    """One SparseGP.parameters_changed() with a composite kernel -> (lml, grad, Zgrad, res). grad = every leaf's block in
    order, then d/d noise variance for a scalar noise; with one noise variance per data point, the blocks only and
    res["dL_dthetaL"] is dL_dR (N x P)."""
    X = np.ascontiguousarray(X, dtype=np.float64)
    Z = np.ascontiguousarray(Z, dtype=np.float64)
    Y = np.ascontiguousarray(Y, dtype=np.float64)
    kern = CompositeOracle(parts)
    res = o.vardtc_inference(kern, X, Z, noise_variance, Y)
    g0 = kern.grads_diag(res["dL_dKdiag"], X)                                   # sparse_gp.py:110
    g1 = kern.grads_full(res["dL_dKnm"], X, Z)                                  # :112
    g2 = kern.grads_full(res["dL_dKmm"], Z, None)                               # :114
    grad = np.concatenate([a + b + c for a, b, c in zip(g0, g1, g2)])
    Zgrad = kern.gradients_X(res["dL_dKmm"], Z)                                 # :117
    Zgrad = Zgrad + kern.gradients_X(res["dL_dKnm"].T, Z, X)                    # :118
    if np.ndim(noise_variance) == 0:
        grad = np.concatenate([grad, [res["dL_dthetaL"]]])
    return res["log_marginal"], grad, Zgrad, res


def descriptor(p):
    """the part as Engine.sparse_eval_multi / exact_eval_multi take it"""
    return (p["kind"], p.get("ARD", False), p["term"], list(p.get("dims") or []), p["variance"], p.get("lengthscale"))


# the kernels of the committed reference fixtures (tests/golden/sparse_composite), on D = 3 columns
KERNELS = {
    # RBF(ARD, all dims) + Bias + White
    "rbf_bias_white": [dict(kind="rbf", term=0, dims=[0, 1, 2], variance=1.3, lengthscale=[0.9, 1.4, 2.1], ARD=True),
                       dict(kind="bias", term=1, variance=0.4),
                       dict(kind="white", term=2, variance=0.07)],
    # Matern52(iso, dims [0, 1]) x RBF(ARD, dims [1, 2]) + Exponential(dim 0): dim 1 is shared by two parts
    "m52_x_rbf_plus_exp": [dict(kind="matern52", term=0, dims=[0, 1], variance=1.1, lengthscale=1.2),
                           dict(kind="rbf", term=0, dims=[1, 2], variance=0.8, lengthscale=[1.5, 0.7], ARD=True),
                           dict(kind="exponential", term=1, dims=[0], variance=0.3, lengthscale=2.5)],
    # Matern32 x Bias
    "m32_x_bias": [dict(kind="matern32", term=0, dims=[0, 1, 2], variance=0.9, lengthscale=1.1),
                   dict(kind="bias", term=0, variance=1.7)],
}


def case_data(N, M, D, P, seed, het):
    """inputs of one fixture case: X (N x D), Y (N x P), Z = M rows of X jittered, noise (scalar or N per-point)"""
    rng = np.random.default_rng(seed)
    X = rng.uniform(-2.0, 2.0, size=(N, D))
    Y = np.sin(X.sum(1, keepdims=True) + np.arange(P)) + 0.1 * rng.standard_normal((N, P))
    Z = X[rng.choice(N, M, replace=False)] + 0.05 * rng.standard_normal((M, D))
    noise = 0.05 + 0.1 * rng.uniform(size=N) if het else 0.08
    return X, Y, Z, noise
