"""Host-side mirror of GPy's sparse GP regression (VarDTC and FITC), computing the N-dependent work on the H100.

Mirrors:
    GPy.inference.latent_function_inference.VarDTC.inference   GPy/inference/latent_function_inference/var_dtc.py:66-215
    GPy.inference.latent_function_inference.FITC.inference     GPy/inference/latent_function_inference/fitc.py:19-88
    GPy.core.SparseGP.parameters_changed / _update_gradients   GPy/core/sparse_gp.py:76-119
    GPy.models.SparseGPRegression                              GPy/models/sparse_gp_regression.py:33-59
(Gaussian likelihood, certain inputs, no mean function — BASELINE.json configs[4]; scalar noise through gpx_sparse_eval,
one noise variance per data point — the `het_noise` branches var_dtc.py:127-128,221-227,241-257,267-269 with a
HeteroscedasticGaussian likelihood — through gpx_sparse_eval_het. A sum of products of RBF .. Matern52, White and Bias
leaves (kern.flatten_parts) goes through gpx_sparse_eval_multi, with either noise form.)

ONE call, gpx_sparse_eval, does the whole evaluation on the device — psi1 = K(X, Z), tmp = Lm^-1 psi1^T, A = beta tmp
tmp^T, the two M x M factor-and-invert sweeps (Kmm, B = I + A), every M x M product, dL_dKnm = (beta Y) C^T + 2 psi1
dL_dpsi2 and all reductions to kernel / inducing-point / noise gradients. Only X, Y (once), Z and theta go in; the
bound, 2 + nl gradient entries and dZ (M x D) come back; the posterior is fetched lazily (gpx_sparse_get). With an engine
attached to a NCCL communicator, X and Y are this rank's rows (gpy_b200.dist.shard_rows).
"""
import numpy as np

from . import _ffi
from .inference import Gaussian, HeteroscedasticGaussian, PosteriorExact, _DataKey, evaluated_kernel
from .model import (draw_standard_normals, host_predictive_gradients, likelihood_samples, sample_normal,
                    scatter_active_dims)
from .kern import (RBF, RatQuad, StdPeriodic, Stationary, composite_state_key, flatten_parts, part_descriptor,
                   part_ngrad, scatter_leaf_gradients, single_kernel)
from .param import Logexp, Param, Parameterized

CONST_JITTER = 1e-8  # var_dtc.py:24


class SparsePosterior(object):
    """Posterior(woodbury_inv, woodbury_vector, K=Kmm, K_chol=Lm) (var_dtc.py:213; posterior.py:238-270)."""

    def __init__(self, woodbury_inv, woodbury_vector, K, K_chol):
        self.woodbury_inv, self.woodbury_vector, self.K, self.K_chol = woodbury_inv, woodbury_vector, K, K_chol

    def _raw_predict(self, kern, Xnew, pred_var, full_cov=False):
        """posterior.py:238-270 with pred_var = Z (sparse_gp.py:52-54)."""
        Kx = kern.K(pred_var, Xnew)
        mu = np.dot(Kx.T, self.woodbury_vector)
        if full_cov:
            return mu, kern.K(Xnew) - np.dot(Kx.T, np.dot(self.woodbury_inv, Kx))
        return mu, (kern.Kdiag(Xnew) - np.sum(np.dot(self.woodbury_inv.T, Kx) * Kx, 0))[:, None]


class LazySparsePosterior(object):
    """Posterior of the last gpx_sparse_eval; its arrays are produced on the device on first touch (var_dtc.py:201-214).
    kern_key and Z (as the evaluation sliced it) describe the evaluation, so that _raw_predict can tell when the device
    holds what a prediction needs; without them every prediction takes the host route."""

    def __init__(self, engine, kern_key=None, Z=None):
        self._eng, self._serial, self._c = engine, engine.sparse_serial, {}
        self._kern_key = kern_key
        self._Z = None if Z is None else np.array(Z, dtype=np.float64, copy=True)

    def _check_fresh(self):
        if self._eng.sparse_serial != self._serial:
            raise RuntimeError("stale sparse posterior: the engine has evaluated other parameters since")

    def _get(self, what):
        if what not in self._c:
            self._check_fresh()
            self._c[what] = self._eng.sparse_get(what)
        return self._c[what]

    woodbury_vector = property(lambda self: self._get("woodbury_vector"))
    woodbury_inv = property(lambda self: self._get("woodbury_inv"))
    K = property(lambda self: self._get("Kmm"))
    K_chol = property(lambda self: self._get("Lm"))

    def _predictive_gradients(self, Xnew):
        """gp.py:438-462 with the predictive variable Z on the device (gpx_sparse_predictive_gradients)"""
        self._check_fresh()
        return self._eng.sparse_predictive_gradients(Xnew)

    def _posterior_samples(self, Xnew, z):
        """gp.py:601-629 with the predictive variable Z on the device (gpx_sparse_posterior_samples) -> f in z's layout"""
        self._check_fresh()
        return self._eng.sparse_posterior_samples(Xnew, z)[0]

    def materialise(self):
        for w in ("woodbury_vector", "woodbury_inv"):
            self._get(w)
        return self

    def _on_device(self, kern, pred_var):
        """the prediction can come from the device: kern is the evaluated kernel (inference.evaluated_kernel), pred_var
        is the evaluated Z once sliced the same way, and the engine has gpx_sparse_predict"""
        return (self._kern_key is not None and getattr(self._eng, "sparse_predict", None) is not None
                and evaluated_kernel(kern, self._kern_key)
                and np.array_equal(PosteriorExact._engine_X(kern, pred_var), self._Z))

    def _raw_predict(self, kern, Xnew, pred_var, full_cov=False):
        """posterior.py:220-248 with pred_var = Z (sparse_gp.py:52-54). With the evaluated kernel and Z one
        gpx_sparse_predict call (the diagonal clipped at 1e-15 as the reference clips it); otherwise the formula on the
        fetched woodbury arrays (SparsePosterior._raw_predict)."""
        if not self._on_device(kern, pred_var):
            return SparsePosterior._raw_predict(self, kern, Xnew, pred_var, full_cov)
        self._check_fresh()
        return self._eng.sparse_predict(PosteriorExact._engine_X(kern, Xnew), full_cov=full_cov)


class VarDTC(object):
    """Drop-in for GPy's VarDTC: inference(kern, X, Z, likelihood, Y) -> (posterior, log_marginal, grad_dict).
    `grad_dict['dL_dKnm']` is never materialised (N x M); instead the dict carries the kernel's gradients already summed
    over sparse_gp.py:110-115 (`dvariance` / `dlengthscale` for a single kernel, `part_grads`, one block per flattened
    leaf, for a composite), `dZ` (:117-118) and `dL_dthetaL`."""

    const_jitter = CONST_JITTER

    def __init__(self, device=0, engine=None, limit=1):
        self.device, self._engine, self._data_key = device, engine, _DataKey()

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

    def inference(self, kern, X, Z, likelihood, Y, Y_metadata=None, mean_function=None, precision=None):
        if mean_function is not None:
            raise NotImplementedError("sparse GP with a mean function is not on the accelerated path")
        leaves = None if single_kernel(kern) else flatten_parts(kern)
        for k in ([kern] if leaves is None else [q for q, _ in leaves]):
            if isinstance(k, (RatQuad, StdPeriodic)):
                raise NotImplementedError("gpy_b200.VarDTC: %s is not on the device's sparse evaluation (RBF, Exponential, "
                                          "Matern32, Matern52, White, Bias and their sums and products are)"
                                          % type(k).__name__)
        if leaves is None and not isinstance(kern, Stationary):
            raise TypeError("gpy_b200.VarDTC accelerates gpy_b200.kern stationary kernels and sums / products of them "
                            "with White and Bias")
        eng = self.engine
        if leaves is not None:
            return self._inference_multi(eng, kern, leaves, X, Z, likelihood, Y, Y_metadata, precision)
        Xs = kern._slice_X(X)
        Zs = kern._slice_X(Z)
        Y = np.ascontiguousarray(Y, dtype=np.float64)
        if not self._data_key.matches(Xs, Y):
            if Y.shape[1] > 8:
                eng.set_option("sparse_wide", 1)                   # the sparse state's wide route (P <= 1024)
            eng.sparse_set_data(Xs, Y)
            self._data_key.remember(Xs, Y)
        num_data, output_dim = Y.shape
        num_inducing = Zs.shape[0]
        kind, ard, var, ls = kern._theta()
        if precision is None:
            gv = np.asarray(likelihood.gaussian_variance(Y_metadata), dtype=np.float64)
            if gv.size > 1:                                                                # het_noise (var_dtc.py:82-84)
                if gv.size != num_data:
                    raise ValueError("one noise variance per data point expected")
                lml, grad, dZ, dR = eng.sparse_eval_het(kind, ard, var, ls, Zs, gv.reshape(-1))
                dL_dthetaL = likelihood.exact_inference_gradients(dR, Y_metadata)         # var_dtc.py:176
                return LazySparsePosterior(eng, kern._state_key(), Zs), float(lml), {
                    "dvariance": grad[0], "dlengthscale": grad[1:], "dZ": dZ, "dL_dthetaL": dL_dthetaL, "num_data": num_data}
        elif np.size(precision) > 1:
            pv = np.asarray(precision, dtype=np.float64).reshape(-1)
            lml, grad, dZ, dR = eng.sparse_eval_het(kind, ard, var, ls, Zs, 1.0 / pv)
            return LazySparsePosterior(eng, kern._state_key(), Zs), float(lml), {
                "dvariance": grad[0], "dlengthscale": grad[1:], "dZ": dZ, "dL_dthetaL": dR, "num_data": num_data}
        noise_var = None
        if precision is None:
            noise_var = float(np.squeeze(np.asarray(likelihood.gaussian_variance(Y_metadata))))
            precision = 1.0 / np.fmax(float(np.squeeze(np.asarray(likelihood.gaussian_variance(Y_metadata)))),
                                      self.const_jitter)                                   # var_dtc.py:79-80
        beta = float(precision)
        lml, grad, dZ = eng.sparse_eval(kind, ard, var, ls, Zs, noise_var if noise_var is not None else 1.0 / beta)
        post = LazySparsePosterior(eng, kern._state_key(), Zs)
        return post, float(lml), {"dvariance": grad[0], "dlengthscale": grad[1:-1], "dZ": dZ,
                                  "dL_dthetaL": float(grad[-1]), "num_data": num_data}


    def _inference_multi(self, eng, kern, leaves, X, Z, likelihood, Y, Y_metadata, precision):
        """a composite kernel: one gpx_sparse_eval_multi; gradients returned per leaf (`part_grads`)"""
        Xs = np.ascontiguousarray(X, dtype=np.float64)
        Zs = np.ascontiguousarray(Z, dtype=np.float64)
        Y = np.ascontiguousarray(Y, dtype=np.float64)
        if not self._data_key.matches(Xs, Y):
            if Y.shape[1] > 8:
                eng.set_option("sparse_wide", 1)                   # the sparse state's wide route (P <= 1024)
            eng.sparse_set_data(Xs, Y)
            self._data_key.remember(Xs, Y)
        num_data = Y.shape[0]
        parts = [part_descriptor(k, t) for k, t in leaves]
        if precision is None:
            gv = np.asarray(likelihood.gaussian_variance(Y_metadata), dtype=np.float64)
            noise = gv.reshape(-1) if gv.size > 1 else float(np.squeeze(gv))                 # het_noise: var_dtc.py:82-84
        elif np.size(precision) > 1:
            noise = 1.0 / np.asarray(precision, dtype=np.float64).reshape(-1)
        else:
            noise = 1.0 / float(precision)
        het = np.ndim(noise) > 0
        if het and noise.size != num_data:
            raise ValueError("one noise variance per data point expected")
        out = eng.sparse_eval_multi(parts, Zs, noise)
        lml, grad, dZ = out[:3]
        blocks, i = [], 0
        for k, _ in leaves:
            blocks.append(grad[i:i + part_ngrad(k)])
            i += part_ngrad(k)
        if het:
            dL_dthetaL = likelihood.exact_inference_gradients(out[3], Y_metadata) if precision is None else out[3]
        else:
            dL_dthetaL = float(grad[-1])
        return LazySparsePosterior(eng, composite_state_key(kern), Zs), float(lml), {
            "part_grads": blocks, "dZ": dZ, "dL_dthetaL": dL_dthetaL, "num_data": num_data}


class FITC(object):
    """Drop-in for GPy's FITC (fitc.py:11-88, Snelson & Ghahramani's SPGP): inference(kern, X, Z, likelihood, Y,
    mean_function=None, Y_metadata=None) -> (posterior, log_marginal, grad_dict), with the reference's argument order and
    exceptions. ONE gpx_sparse_eval_fitc call does the whole evaluation and the gradient reductions of sparse_gp.py:108-118;
    the grad dict has VarDTC's shape (`dvariance` / `dlengthscale` or `part_grads`, `dZ`, `dL_dthetaL`) plus the N-vector
    `dL_dKdiag`. The posterior (woodbury_inv = Kmm^-1 - P, woodbury_vector = v, fitc.py:86) serves predict, predictive
    gradients and samples on the device like VarDTC's. Select it as the reference's tests do (GPy/testing/fitc.py:31):
    `m.inference_method = gpy_b200.FITC()`."""

    const_jitter = 1e-6  # fitc.py:18

    def __init__(self, device=0, engine=None):
        self.device, self._engine, self._data_key = device, engine, _DataKey()

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

    def inference(self, kern, X, Z, likelihood, Y, mean_function=None, Y_metadata=None):
        assert mean_function is None, "inference with a mean function not implemented"                 # fitc.py:21
        sigma_n = np.asarray(likelihood.gaussian_variance(Y_metadata), dtype=np.float64)
        if sigma_n.size > 1:                                                                               # :27-29
            raise NotImplementedError("no hetero noise with this implementation of FITC")
        Y = np.ascontiguousarray(Y, dtype=np.float64)
        num_data, output_dim = Y.shape
        if output_dim != 1:   # the reference fails on tdot(v.reshape(-1, 1)) + P (:71) with a broadcasting ValueError
            raise ValueError("FITC takes one output column (fitc.py:71 reshapes v to a column); Y has %d" % output_dim)
        leaves = None if single_kernel(kern) else flatten_parts(kern)
        for k in ([kern] if leaves is None else [q for q, _ in leaves]):
            if isinstance(k, (RatQuad, StdPeriodic)):
                raise NotImplementedError("gpy_b200.FITC: %s is not on the device's sparse evaluation (RBF, Exponential, "
                                          "Matern32, Matern52, White, Bias and their sums and products are)"
                                          % type(k).__name__)
        if leaves is None and not isinstance(kern, Stationary):
            raise TypeError("gpy_b200.FITC accelerates gpy_b200.kern stationary kernels and sums / products of them "
                            "with White and Bias")
        if leaves is None:
            Xs, Zs = kern._slice_X(X), kern._slice_X(Z)
            kind, ard, var, ls = kern._theta()
            parts, key = [(kind, ard, 0, list(range(Xs.shape[1])), var, ls)], kern._state_key()
        else:
            Xs, Zs = X, Z
            parts, key = [part_descriptor(k, t) for k, t in leaves], composite_state_key(kern)
        Xs = np.ascontiguousarray(Xs, dtype=np.float64)
        Zs = np.ascontiguousarray(Zs, dtype=np.float64)
        eng = self.engine
        if not self._data_key.matches(Xs, Y):
            eng.sparse_set_data(Xs, Y)
            self._data_key.remember(Xs, Y)
        lml, grad, dZ, dR = eng.sparse_eval_fitc(parts, Zs, float(np.squeeze(sigma_n)))
        gd = {"dZ": dZ, "dL_dKdiag": dR, "dL_dthetaL": float(grad[-1]), "num_data": num_data}
        if leaves is None:
            gd["dvariance"], gd["dlengthscale"] = grad[0], grad[1:-1]
        else:
            blocks, i = [], 0
            for k, _ in leaves:
                blocks.append(grad[i:i + part_ngrad(k)])
                i += part_ngrad(k)
            gd["part_grads"] = blocks
        return LazySparsePosterior(eng, key, Zs), float(lml), gd


class SparseGPRegression(Parameterized):
    """GPy.models.SparseGPRegression (sparse_gp_regression.py:33-59) / GPy.core.SparseGP (sparse_gp.py:38-119).
    Parameter (and gradient) order as in the reference: [inducing inputs, the kernel's parameters in link order (a single
    kernel: variance, lengthscale), the likelihood's]."""

    def __init__(self, X, Y, kernel=None, Z=None, num_inducing=10, device=0, engine=None, name="sparse_gp", likelihood=None,
                 Y_metadata=None, inference_method=None):
        super(SparseGPRegression, self).__init__(name)
        X = np.asarray(X, dtype=np.float64)
        Y = np.asarray(Y, dtype=np.float64)
        num_data, input_dim = X.shape
        if kernel is None:
            kernel = RBF(input_dim)                                            # sparse_gp_regression.py:36-37
        if Z is None:
            i = np.random.permutation(num_data)[:min(num_inducing, num_data)]  # :41-43
            Z = X[i].copy()
        else:
            assert Z.shape[1] == input_dim
        self.X, self.Y = X, Y
        self.kern = kernel
        # :47; core/sparse_gp.py:41 accepts any likelihood: a HeteroscedasticGaussian (with its Y_metadata) selects VarDTC's
        # het_noise branches
        self.likelihood = Gaussian() if likelihood is None else likelihood
        self.Y_metadata = Y_metadata
        self.Z = Param("inducing inputs", np.array(Z, dtype=np.float64), transform=None)
        self.Z.values = np.array(Z, dtype=np.float64)                          # keep the M x D shape
        self.Z.gradient = np.zeros_like(self.Z.values)
        self.num_inducing = self.Z.values.shape[0]
        self.inference_method = VarDTC(device=device, engine=engine) if inference_method is None else inference_method
        self.link_parameter(self.Z)                                            # sparse_gp.py:61 (index 0)
        self.link_parameter(self.kern)
        self.link_parameter(self.likelihood)
        self.parameters_changed()

    # ---- one evaluation: sparse_gp.py:76-119 ------------------------------------------------------------------------
    def parameters_changed(self):
        Z = self.Z.values
        self.posterior, self._log_marginal_likelihood, gd = self.inference_method.inference(
            self.kern, self.X, Z, self.likelihood, self.Y, Y_metadata=self.Y_metadata)
        self.grad_dict = gd
        self.likelihood.update_gradients(gd["dL_dthetaL"])                                     # :84
        if "part_grads" in gd:                                                 # :110-115 summed on the device, per leaf
            scatter_leaf_gradients(flatten_parts(self.kern), gd["part_grads"])
        else:
            self.kern.variance.gradient = np.atleast_1d(gd["dvariance"])
            self.kern.lengthscale.gradient = np.atleast_1d(gd["dlengthscale"])
        self.Z.gradient = gd["dZ"]                                             # :117-118

    def log_likelihood(self):
        return self._log_marginal_likelihood

    def objective_function(self):
        return -float(self._log_marginal_likelihood)

    # ---- optimizer space: Z unconstrained, the positive parameters through Logexp ---------------------------------------
    def _flat(self):
        return self.flattened_parameters()      # Z, then the kernel's and the likelihood's parameters in link order

    def _free(self):
        """the leading parameters without a transform"""
        return [self.Z]

    @property
    def optimizer_array(self):
        free = self._free()
        out = [p.values.reshape(-1) for p in free]
        for p in self._flat()[len(free):]:
            out.append(Logexp.finv(p.values).reshape(-1))
        return np.concatenate(out)

    @optimizer_array.setter
    def optimizer_array(self, x):
        free = self._free()
        i = 0
        for p in free:
            p.values[...] = x[i:i + p.values.size].reshape(p.values.shape)
            i += p.values.size
        for p in self._flat()[len(free):]:
            p.values[...] = Logexp.f(x[i:i + p.size]).reshape(p.values.shape)
            i += p.size
        self.parameters_changed()

    def _grads_transformed(self):
        free = self._free()
        g = [np.asarray(p.gradient).reshape(-1) for p in free]
        for p in self._flat()[len(free):]:
            g.append(np.asarray(p.gradient, dtype=np.float64).reshape(-1) * Logexp.gradfactor(p.values).reshape(-1))
        return -np.concatenate(g)

    def optimize(self, max_iters=1000, messages=False):
        from scipy.optimize import fmin_l_bfgs_b
        self.n_evals = 0
        self.inference_method.on_optimization_start()                          # gp.py:677

        def fg(x):
            self.n_evals += 1
            self.optimizer_array = x
            return self.objective_function(), self._grads_transformed()

        x, f, d = fmin_l_bfgs_b(fg, self.optimizer_array, maxfun=max_iters, maxiter=max_iters)
        self.optimizer_array = x
        d["n_evals"] = self.n_evals
        return d

    def checkgrad(self, step=1e-6, tolerance=1e-3, sample=12, seed=0):
        """finite differences on the kernel / noise parameters and on a random sample of the unconstrained coordinates
        (inducing inputs, and latent inputs in the sparse GPLVM)."""
        x = self.optimizer_array.copy()
        self.optimizer_array = x
        g = self._grads_transformed()
        nz = sum(p.values.size for p in self._free())
        rng = np.random.default_rng(seed)
        idx = np.concatenate([rng.choice(nz, size=min(sample, nz), replace=False), np.arange(nz, x.size)])
        ok = True
        for i in idx:
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

    def predict(self, Xnew, full_cov=False, include_likelihood=True, Y_metadata=None, kern=None, likelihood=None):
        """gp.py:290-365 with the sparse posterior (predictive variable = Z). With the evaluated kernel the latent part is
        one gpx_sparse_predict call; another kern= takes the reference's formula on the fetched woodbury arrays."""
        kern = self.kern if kern is None else kern
        mu, var = self.posterior._raw_predict(kern, np.asarray(Xnew, dtype=np.float64), self.Z.values, full_cov)
        if include_likelihood:
            likelihood = self.likelihood if likelihood is None else likelihood
            if isinstance(likelihood, HeteroscedasticGaussian) and Y_metadata is None:
                raise ValueError("a heteroscedastic likelihood needs Y_metadata (output_index) for the new points, or "
                                 "include_likelihood=False (gp_heteroscedastic_regression.py:13-15)")
            mu, var = likelihood.predictive_values(mu, var, full_cov, Y_metadata=Y_metadata)
        return mu, var

    def predict_noiseless(self, Xnew, full_cov=False, Y_metadata=None, kern=None):
        """gp.py:367-393: predict without the likelihood's variance"""
        return self.predict(Xnew, full_cov, include_likelihood=False, Y_metadata=Y_metadata, kern=kern)

    def posterior_samples_f(self, X, size=10, kern=None):
        """gp.py:601-629 with the predictive variable Z (sparse_gp.py:52-54) -> (Nnew, output_dim, size). The standard
        normals are drawn as GP.posterior_samples_f draws them; with the evaluated kernel the rest is one
        gpx_sparse_posterior_samples call (Sigma = K(X) - K(X, Z) W K(Z, X) through its Cholesky factor and jitchol's
        ladder), another kern= takes the reference's host route. posterior_covariance_between_points is not offered: the
        reference raises for a sparse posterior (posterior.py:119-120)."""
        X = np.asarray(X, dtype=np.float64)
        if kern is None or kern is self.kern:
            M, P = X.shape[0], self.Y.shape[1]
            Xs = self.kern._slice_X(X) if single_kernel(self.kern) else np.ascontiguousarray(X)
            z = draw_standard_normals(M, P, size)
            f = self.posterior._posterior_samples(Xs, z)
            return np.ascontiguousarray(f.reshape(P, size, M).transpose(2, 0, 1))
        m, v = self.posterior._raw_predict(kern, X, self.Z.values, full_cov=True)
        return sample_normal(m, v, size)

    def posterior_samples(self, X, size=10, Y_metadata=None, likelihood=None, kern=None):
        """gp.py:631-652: posterior_samples_f, then likelihood.samples per output"""
        fsim = self.posterior_samples_f(X, size, kern=kern)
        return likelihood_samples(self.likelihood if likelihood is None else likelihood, fsim, Y_metadata)

    def predictive_gradients(self, Xnew, kern=None):
        """gp.py:418-474 with the predictive variable Z (sparse_gp.py:52-54): with the evaluated kernel one
        gpx_sparse_predictive_gradients call, with any other kernel the reference's formula on the stand-alone calls"""
        Xnew = np.asarray(Xnew, dtype=np.float64)
        if kern is None or kern is self.kern:
            Xs = self.kern._slice_X(Xnew) if single_kernel(self.kern) else np.ascontiguousarray(Xnew)
            return tuple(scatter_active_dims(self.kern, g, Xnew.shape[1])
                         for g in self.posterior._predictive_gradients(Xs))
        return host_predictive_gradients(kern, self.posterior, Xnew, self.Z.values)
