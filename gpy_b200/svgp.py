"""Stochastic variational sparse GPs (SVGP) for any likelihood, with the M x Nb and M x M work on the H100.

Mirrors:
    GPy.inference.latent_function_inference.SVGP.inference   GPy/inference/latent_function_inference/svgp.py:10-118
    GPy.core.SVGP                                           GPy/core/svgp.py:10-97
(one output column, one latent function, no mean function; Hensman, Fusi and Lawrence 2013, Hensman, Matthews and
Ghahramani 2015.)

One step is gpx_svgp_begin (Kmm, jitchol, Kmn of the batch, A = Kmm^-1 Kmn, the marginals mu, v of q(f) and the KL term)
-> likelihood.variational_expectations(Y, mu, v) on the host -> gpx_svgp_finish (every gradient, reduced on the device to
the kernel's parameters and dL/dZ). Any likelihood object with `variational_expectations` works. The whole data set stays
on the device; a minibatch is a contiguous row range of it, so a step uploads only Z, theta, q_u_mean and q_u_chol.
"""
import numpy as np

from . import _ffi
from .inference import _DataKey
from .kern import (RatQuad, StdPeriodic, Stationary, composite_state_key, flatten_parts, part_descriptor, part_ngrad,
                   scatter_leaf_gradients, single_kernel)
from .param import Logexp, Param
from .sparse import LazySparsePosterior, SparseGPRegression


def triang_to_flat(L):
    """choleskies.triang_to_flat for one M x M lower triangle: its entries in np.tril_indices(M) order"""
    return L[np.tril_indices(L.shape[0])]


def q_triangle(q_u_mean, q_u_chol, M):
    """q_u_chol (M (M + 1) / 2 x 1, GPy's flat form) -> its M x M lower triangle L, after the reference's check"""
    if q_u_mean.shape[0] != M or q_u_chol.shape[0] != M * (M + 1) // 2:
        raise ValueError("q_u_mean must be M x 1 and q_u_chol M (M + 1) / 2 x 1 for M = %d inducing inputs" % M)
    L = flat_to_triang(q_u_chol[:, 0], M)
    # svgp.py:19-26 raises when Si = dpotri(L) holds an infinite entry. Si_ii >= 1 / L_ii^2, so a tiny nonzero diagonal
    # entry overflows it; this is the test made here. (An ill-conditioned L can overflow an entry of Si while every
    # 1 / L_ii^2 stays finite: the reference raises there and this does not.) An exact zero does not raise in the
    # reference (dpotri fails quietly): the bound is then -inf (logdetS = -inf), as the device computes it.
    d = np.abs(np.diag(L))
    with np.errstate(divide="ignore", over="ignore"):
        if np.any((d > 0) & np.isinf(1.0 / np.square(d))):
            raise ValueError("Cholesky representation unstable")
    return L


def flat_to_triang(flat, M):
    """choleskies.flat_to_triang for one latent function: the M x M lower triangle of the flat q_u_chol"""
    L = np.zeros((M, M))
    L[np.tril_indices(M)] = np.asarray(flat, dtype=np.float64).reshape(-1)
    return L


class SVGPInference(object):
    """Drop-in for GPy's SVGP inference: inference(q_u_mean, q_u_chol, kern, X, Z, likelihood, Y, ...) ->
    (posterior, log_marginal, grad_dict). The bound is F.sum() batch_scale - KL. The dense dL_dKmm / dL_dKmn are not
    formed on the host: grad_dict carries the kernel's gradients already summed over core/svgp.py:53-60 (`dvariance` /
    `dlengthscale` for a single kernel, `part_grads`, one block per flattened leaf, for a composite) and `dZ` (:61-62),
    with `dL_dKdiag`, `dL_dm`, `dL_dchol` (flat) and `dL_dthetaL` as the reference returns them."""

    def __init__(self, device=0, engine=None, max_tries=5):
        self.device, self._engine, self._data_key, self.max_tries = device, engine, _DataKey(), max_tries

    @property
    def engine(self):
        if self._engine is None:
            self._engine = _ffi.Engine(self.device)
        return self._engine

    def on_optimization_start(self):
        pass

    def on_optimization_end(self):
        pass

    def invalidate_data(self):
        self._data_key.invalidate()

    def inference(self, q_u_mean, q_u_chol, kern, X, Z, likelihood, Y, mean_function=None, Y_metadata=None,
                  KL_scale=1.0, batch_scale=1.0):
        X = np.asarray(X, dtype=np.float64)
        return self.batch_inference(q_u_mean, q_u_chol, kern, X, Z, likelihood, Y, 0, X.shape[0], mean_function,
                                    Y_metadata, batch_scale)

    @staticmethod
    def _parts(kern):
        """-> (leaves or None, part descriptors, state key, slice) for a kernel the device evaluates; slice(A) gives the
        columns of A the device sees"""
        leaves = None if single_kernel(kern) else flatten_parts(kern)
        for k in ([kern] if leaves is None else [q for q, _ in leaves]):
            if isinstance(k, (RatQuad, StdPeriodic)):
                raise NotImplementedError("gpy_b200.SVGP: %s is not on the device's sparse evaluation (RBF, Exponential, "
                                          "Matern32, Matern52, White, Bias and their sums and products are)"
                                          % type(k).__name__)
        if leaves is None and not isinstance(kern, Stationary):
            raise TypeError("gpy_b200.SVGP accelerates gpy_b200.kern stationary kernels and sums / products of them "
                            "with White and Bias")
        if leaves is None:
            kind, ard, var, ls = kern._theta()
            return leaves, [(kind, ard, 0, list(range(kern.input_dim)), var, ls)], kern._state_key(), kern._slice_X
        return leaves, [part_descriptor(k, t) for k, t in leaves], composite_state_key(kern), lambda A: A

    def batch_inference(self, q_u_mean, q_u_chol, kern, X, Z, likelihood, Y, row0, nb, mean_function=None,
                        Y_metadata=None, batch_scale=1.0, data_token=None):
        """the inference on the rows [row0, row0 + nb) of the data X, Y, which stay on the device. Without data_token the
        data are compared with what the device holds (one pass over X and Y) and uploaded when they differ; with a
        data_token (an object that stands for the content of X and Y, which the caller must not change under it) they are
        uploaded only when the token changes, so a step costs nothing on the host that grows with the number of rows."""
        if mean_function is not None:
            raise NotImplementedError("gpy_b200.SVGP: a mean function is not on the device path")
        q_u_mean = np.asarray(q_u_mean, dtype=np.float64)
        q_u_chol = np.asarray(q_u_chol, dtype=np.float64)
        if np.ndim(Y) != 2 or np.shape(Y)[1] != 1 or q_u_mean.ndim != 2 or q_u_mean.shape[1] != 1 \
                or q_u_chol.ndim != 2 or q_u_chol.shape[1] != 1:
            raise NotImplementedError("gpy_b200.SVGP takes one output column and one latent function")
        leaves, parts, key, slice_ = self._parts(kern)
        L = q_triangle(q_u_mean, q_u_chol, np.shape(Z)[0])
        eng = self.engine
        if data_token is None or data_token is not getattr(self, "_data_token", None):
            Xs = np.ascontiguousarray(slice_(np.asarray(X, dtype=np.float64)), dtype=np.float64)
            Yc = np.ascontiguousarray(Y, dtype=np.float64)
            if data_token is not None or not self._data_key.matches(Xs, Yc):
                eng.sparse_set_data(Xs, Yc)
                if data_token is None:
                    self._data_key.remember(Xs, Yc)
                else:
                    self._data_key.invalidate()
            self._data_token = data_token
        Zs = np.ascontiguousarray(slice_(np.asarray(Z, dtype=np.float64)), dtype=np.float64)
        post, lml, grad, gd = self.device_inference(q_u_mean, L, parts, key, Zs, likelihood,
                                                    np.asarray(Y)[row0:row0 + nb], row0, nb, Y_metadata, batch_scale)
        if leaves is None:
            gd["dvariance"], gd["dlengthscale"] = grad[0], grad[1:]
        else:
            blocks, i = [], 0
            for k, _ in leaves:
                blocks.append(grad[i:i + part_ngrad(k)])
                i += part_ngrad(k)
            gd["part_grads"] = blocks
        return post, lml, gd

    def device_inference(self, q_u_mean, L, parts, key, Zs, likelihood, Yb, row0, nb, Y_metadata=None,
                         batch_scale=1.0):
        """one step on the data the engine holds, for q_u_mean (M x 1) and L = q_triangle(..): begin, the likelihood's variational_expectations on the batch's Yb,
        finish -> (posterior, bound, the kernel's gradient block, grad dict without the kernel's entries)"""
        eng = self.engine
        mu, v, KL, _ = eng.svgp_begin(parts, Zs, q_u_mean[:, 0], L, row0, nb, self.max_tries)
        F, dF_dmu, dF_dv, dF_dthetaL = likelihood.variational_expectations(Yb, mu[:, None], v[:, None],
                                                                          Y_metadata=Y_metadata)
        F, dF_dmu, dF_dv = F * batch_scale, dF_dmu * batch_scale, dF_dv * batch_scale               # svgp.py:66-67
        if dF_dthetaL is not None:
            dF_dthetaL = dF_dthetaL.sum(1).sum(1) * batch_scale
        grad, dZ, dL_dm, dL_dchol = eng.svgp_finish(dF_dmu[:, 0], dF_dv[:, 0])
        with np.errstate(invalid="ignore"):
            log_marginal = F.sum() - KL
        gd = {"dZ": dZ, "dL_dKdiag": dF_dv.sum(1), "dL_dm": dL_dm[:, None], "dL_dchol": triang_to_flat(dL_dchol)[:, None],
              "dL_dthetaL": dF_dthetaL, "mu": mu, "v": v, "KL": KL}
        return LazySparsePosterior(eng, key, Zs), float(log_marginal), grad, gd


class SVGP(SparseGPRegression):
    """GPy.core.SVGP (core/svgp.py:10-97) without a mean function, with one latent function. Parameters (and gradients)
    in the reference's order: [inducing inputs, the kernel's, the likelihood's, q_u_chol, q_u_mean]; q_u_mean starts at 0
    and q_u_chol at the flat identity (:44-47).

    With a `batchsize` the whole X, Y go to the device once and `new_batch` draws contiguous slices of batchsize rows:
    the start row is drawn uniformly from [0, N - batchsize] by numpy's Generator seeded with `seed` (the reference draws
    its slices with climin's draw_mini_slices, which this project does not depend on). batch_scale = N / batchsize
    (:51)."""

    def __init__(self, X, Y, Z, kernel, likelihood, mean_function=None, name="SVGP", Y_metadata=None, batchsize=None,
                 num_latent_functions=None, device=0, engine=None, seed=0):
        if mean_function is not None:
            raise NotImplementedError("gpy_b200.SVGP: a mean function is not on the device path")
        X = np.asarray(X, dtype=np.float64)
        Y = np.asarray(Y, dtype=np.float64)
        if num_latent_functions is None:
            num_latent_functions = Y.shape[1]                                  # :39-41
        if num_latent_functions != 1 or Y.shape[1] != 1:
            raise NotImplementedError("gpy_b200.SVGP takes one output column and one latent function")
        # private copies: the device holds them for the model's life and is keyed on _data_token, not on their content
        self.X_all, self.Y_all = np.array(X, copy=True), np.array(Y, copy=True)
        self._data_token = object()
        self.batchsize = batchsize
        self._rng = np.random.default_rng(seed)
        self._row0, self._nb = 0, X.shape[0]
        if batchsize is not None:
            if not 1 <= batchsize <= X.shape[0]:
                raise ValueError("batchsize must be in [1, N]")
            self._row0, self._nb = self._draw()
        M = np.asarray(Z).shape[0]
        self.m = Param("q_u_mean", np.zeros((M, 1)), transform=None)
        self.m.values = np.zeros((M, 1))
        self.chol = Param("q_u_chol", triang_to_flat(np.eye(M))[:, None], transform=None)
        self.chol.values = triang_to_flat(np.eye(M))[:, None].copy()
        self._svgp_ready = False
        inf = SVGPInference(device=device, engine=engine)
        super(SVGP, self).__init__(X, Y, kernel=kernel, Z=Z, device=device, engine=engine, name=name, likelihood=likelihood,
                                   Y_metadata=Y_metadata, inference_method=inf)
        self.link_parameter(self.chol)                                         # :44-47 (chol, then m)
        self.link_parameter(self.m)
        self._svgp_ready = True
        self.parameters_changed()

    q_u_mean = property(lambda self: self.m.values)
    q_u_chol = property(lambda self: self.chol.values)

    def _draw(self):
        nb = int(self.batchsize)
        return int(self._rng.integers(0, self.X_all.shape[0] - nb + 1)), nb

    def parameters_changed(self):
        """core/svgp.py:49-73"""
        if not getattr(self, "_svgp_ready", False):
            return
        batch_scale = float(self.X_all.shape[0]) / float(self._nb)
        self.posterior, self._log_marginal_likelihood, gd = self.inference_method.batch_inference(
            self.m.values, self.chol.values, self.kern, self.X_all, self.Z.values, self.likelihood, self.Y_all,
            self._row0, self._nb, Y_metadata=self.Y_metadata, batch_scale=batch_scale, data_token=self._data_token)
        self.grad_dict = gd
        if "part_grads" in gd:
            scatter_leaf_gradients(flatten_parts(self.kern), gd["part_grads"])
        else:
            self.kern.variance.gradient = np.atleast_1d(gd["dvariance"])
            self.kern.lengthscale.gradient = np.atleast_1d(gd["dlengthscale"])
        self.Z.gradient = gd["dZ"]
        if gd["dL_dthetaL"] is not None:
            self.likelihood.update_gradients(gd["dL_dthetaL"])
        self.m.gradient = gd["dL_dm"]
        self.chol.gradient = gd["dL_dchol"]

    # ---- batches (:75-97) ----------------------------------------------------------------------------------------
    @property
    def X(self):
        return self.X_all[self._row0:self._row0 + self._nb]

    @X.setter
    def X(self, v):
        pass   # SparseGPRegression.__init__ assigns the data; the batch is a row range of X_all

    @property
    def Y(self):
        return self.Y_all[self._row0:self._row0 + self._nb]

    @Y.setter
    def Y(self, v):
        pass

    def set_data(self, row0, nb):
        """the batch as a row range [row0, row0 + nb) of the whole data, without an evaluation"""
        if not (0 <= row0 and 1 <= nb and row0 + nb <= self.X_all.shape[0]):
            raise ValueError("the batch rows must lie inside the data")
        self._row0, self._nb = int(row0), int(nb)

    def new_batch(self):
        """the next slice: (row0, nb) of batchsize rows, the start drawn as the class documents"""
        if self.batchsize is None:
            return 0, self.X_all.shape[0]
        return self._draw()

    def stochastic_grad(self, parameters):
        """set_data(new_batch()), then the objective's gradient at `parameters` (optimizer space)"""
        self.set_data(*self.new_batch())
        self.optimizer_array = parameters
        return self._grads_transformed()

    # ---- optimizer space: Z, q_u_chol and q_u_mean unconstrained, the kernel's and likelihood's through Logexp --------
    def _free(self):
        return (self.Z, self.chol, self.m)

    @property
    def optimizer_array(self):
        return np.concatenate([p.values.reshape(-1) if any(p is q for q in self._free()) else
                               Logexp.finv(p.values).reshape(-1) for p in self._flat()])

    @optimizer_array.setter
    def optimizer_array(self, x):
        i = 0
        for p in self._flat():
            v = x[i:i + p.size]
            p.values[...] = (v if any(p is q for q in self._free()) else Logexp.f(v)).reshape(p.values.shape)
            i += p.size
        self.parameters_changed()

    def _grads_transformed(self):
        g = []
        for p in self._flat():
            gp = np.asarray(p.gradient, dtype=np.float64).reshape(-1)
            g.append(gp if any(p is q for q in self._free()) else gp * Logexp.gradfactor(p.values).reshape(-1))
        return -np.concatenate(g)

    def checkgrad(self, step=1e-6, tolerance=1e-3, sample=12, seed=0):
        """finite differences on a random sample of every parameter's entries (at most `sample` per parameter)"""
        x = self.optimizer_array.copy()
        self.optimizer_array = x
        g = self._grads_transformed()
        rng = np.random.default_rng(seed)
        idx, i = [], 0
        for p in self._flat():
            idx.append(i + rng.choice(p.size, size=min(sample, p.size), replace=False))
            i += p.size
        ok = True
        for i in np.concatenate(idx):
            xp, xm = x.copy(), x.copy()
            xp[i] += step
            xm[i] -= step
            self.optimizer_array = xp
            fp = self.objective_function()
            self.optimizer_array = xm
            fm = self.objective_function()
            num = (fp - fm) / (2 * step)
            if not (abs(num - g[i]) <= tolerance * max(abs(num), 1e-2)):
                ok = False
        self.optimizer_array = x
        return ok
