"""Host-side mirror of GPy's sparse GP regression (VarDTC), computing the N-dependent work on the H100.

Mirrors:
    GPy.inference.latent_function_inference.VarDTC.inference   GPy/inference/latent_function_inference/var_dtc.py:66-215
    GPy.core.SparseGP.parameters_changed / _update_gradients   GPy/core/sparse_gp.py:76-119
    GPy.models.SparseGPRegression                              GPy/models/sparse_gp_regression.py:33-59
(Gaussian likelihood, certain inputs, no mean function — BASELINE.json configs[4]; scalar noise through gpx_sparse_eval,
one noise variance per data point — the `het_noise` branches var_dtc.py:127-128,221-227,241-257,267-269 with a
HeteroscedasticGaussian likelihood — through gpx_sparse_eval_het.)

ONE call, gpx_sparse_eval, does the whole evaluation on the device — psi1 = K(X, Z), tmp = Lm^-1 psi1^T, A = beta tmp
tmp^T, the two M x M factor-and-invert sweeps (Kmm, B = I + A), every M x M product, dL_dKnm = (beta Y) C^T + 2 psi1
dL_dpsi2 and all reductions to kernel / inducing-point / noise gradients. Only X, Y (once), Z and theta go in; the
bound, 2 + nl gradient entries and dZ (M x D) come back; the posterior is fetched lazily (gpx_sparse_get). With an engine
attached to a NCCL communicator, X and Y are this rank's rows (gpy_b200.dist.shard_rows).
"""
import numpy as np

from . import _ffi
from .inference import Gaussian, HeteroscedasticGaussian, _DataKey
from .kern import RBF, Stationary
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
    """Posterior of the last gpx_sparse_eval; its arrays are produced on the device on first touch (var_dtc.py:201-214)."""

    def __init__(self, engine):
        self._eng, self._serial, self._c = engine, engine.sparse_serial, {}

    def _get(self, what):
        if what not in self._c:
            if self._eng.sparse_serial != self._serial:
                raise RuntimeError("stale sparse posterior: the engine has evaluated other parameters since")
            self._c[what] = self._eng.sparse_get(what)
        return self._c[what]

    woodbury_vector = property(lambda self: self._get("woodbury_vector"))
    woodbury_inv = property(lambda self: self._get("woodbury_inv"))
    K = property(lambda self: self._get("Kmm"))
    K_chol = property(lambda self: self._get("Lm"))

    def materialise(self):
        for w in ("woodbury_vector", "woodbury_inv"):
            self._get(w)
        return self

    _raw_predict = SparsePosterior._raw_predict


class VarDTC(object):
    """Drop-in for GPy's VarDTC: inference(kern, X, Z, likelihood, Y) -> (posterior, log_marginal, grad_dict).
    `grad_dict['dL_dKnm']` is never materialised (N x M); instead the dict carries the already-reduced contributions
    `Knm_dvariance`, `Knm_dlengthscale`, `Knm_dZ`, which SparseGP._update_gradients adds (sparse_gp.py:112,118)."""

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
        if not isinstance(kern, Stationary):
            raise TypeError("gpy_b200.VarDTC accelerates gpy_b200.kern stationary kernels")
        eng = self.engine
        Xs = kern._slice_X(X)
        Zs = kern._slice_X(Z)
        Y = np.ascontiguousarray(Y, dtype=np.float64)
        if not self._data_key.matches(Xs, Y):
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
                return LazySparsePosterior(eng), float(lml), {"dvariance": grad[0], "dlengthscale": grad[1:], "dZ": dZ,
                                                              "dL_dthetaL": dL_dthetaL, "num_data": num_data}
        elif np.size(precision) > 1:
            pv = np.asarray(precision, dtype=np.float64).reshape(-1)
            lml, grad, dZ, dR = eng.sparse_eval_het(kind, ard, var, ls, Zs, 1.0 / pv)
            return LazySparsePosterior(eng), float(lml), {"dvariance": grad[0], "dlengthscale": grad[1:], "dZ": dZ,
                                                          "dL_dthetaL": dR, "num_data": num_data}
        noise_var = None
        if precision is None:
            noise_var = float(np.squeeze(np.asarray(likelihood.gaussian_variance(Y_metadata))))
            precision = 1.0 / np.fmax(float(np.squeeze(np.asarray(likelihood.gaussian_variance(Y_metadata)))),
                                      self.const_jitter)                                   # var_dtc.py:79-80
        beta = float(precision)
        lml, grad, dZ = eng.sparse_eval(kind, ard, var, ls, Zs, noise_var if noise_var is not None else 1.0 / beta)
        post = LazySparsePosterior(eng)
        return post, float(lml), {"dvariance": grad[0], "dlengthscale": grad[1:-1], "dZ": dZ,
                                  "dL_dthetaL": float(grad[-1]), "num_data": num_data}


class SparseGPRegression(Parameterized):
    """GPy.models.SparseGPRegression (sparse_gp_regression.py:33-59) / GPy.core.SparseGP (sparse_gp.py:38-119).
    Parameter (and gradient) order as in the reference: [inducing inputs, kern.variance, kern.lengthscale, noise]."""

    def __init__(self, X, Y, kernel=None, Z=None, num_inducing=10, device=0, engine=None, name="sparse_gp", likelihood=None,
                 Y_metadata=None):
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
        self.inference_method = VarDTC(device=device, engine=engine)
        self.link_parameter(self.Z)                                            # sparse_gp.py:61 (index 0)
        self.link_parameter(self.kern)
        self.link_parameter(self.likelihood)
        self.parameters_changed()

    # ---- one evaluation: sparse_gp.py:76-119 ------------------------------------------------------------------------
    def parameters_changed(self):
        Z = self.Z.values
        self.posterior, self._log_marginal_likelihood, gd = self.inference_method.inference(
            self.kern, self.X, Z, self.likelihood, self.Y, self.Y_metadata)
        self.grad_dict = gd
        self.likelihood.update_gradients(gd["dL_dthetaL"])                                     # :84
        self.kern.variance.gradient = np.atleast_1d(gd["dvariance"])          # :110-114 summed on the device
        self.kern.lengthscale.gradient = np.atleast_1d(gd["dlengthscale"])
        self.Z.gradient = gd["dZ"]                                             # :117-118

    def log_likelihood(self):
        return self._log_marginal_likelihood

    def objective_function(self):
        return -float(self._log_marginal_likelihood)

    # ---- optimizer space: Z unconstrained, the positive parameters through Logexp ---------------------------------------
    def _flat(self):
        return [self.Z, self.kern.variance, self.kern.lengthscale, self.likelihood.variance]

    @property
    def optimizer_array(self):
        out = [self.Z.values.reshape(-1)]
        for p in self._flat()[1:]:
            out.append(Logexp.finv(p.values).reshape(-1))
        return np.concatenate(out)

    @optimizer_array.setter
    def optimizer_array(self, x):
        nz = self.Z.values.size
        self.Z.values[...] = x[:nz].reshape(self.Z.values.shape)
        i = nz
        for p in self._flat()[1:]:
            p.values[...] = Logexp.f(x[i:i + p.size]).reshape(p.values.shape)
            i += p.size
        self.parameters_changed()

    def _grads_transformed(self):
        g = [np.asarray(self.Z.gradient).reshape(-1)]
        for p in self._flat()[1:]:
            g.append(np.asarray(p.gradient, dtype=np.float64).reshape(-1) * Logexp.gradfactor(p.values).reshape(-1))
        return -np.concatenate(g)

    def optimize(self, max_iters=1000, messages=False):
        from scipy.optimize import fmin_l_bfgs_b
        self.n_evals = 0

        def fg(x):
            self.n_evals += 1
            self.optimizer_array = x
            return self.objective_function(), self._grads_transformed()

        x, f, d = fmin_l_bfgs_b(fg, self.optimizer_array, maxfun=max_iters, maxiter=max_iters)
        self.optimizer_array = x
        d["n_evals"] = self.n_evals
        return d

    def checkgrad(self, step=1e-6, tolerance=1e-3, sample=12, seed=0):
        """finite differences on the kernel / noise parameters and on a random sample of inducing-point coordinates."""
        x = self.optimizer_array.copy()
        self.optimizer_array = x
        g = self._grads_transformed()
        nz = self.Z.values.size
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

    def predict(self, Xnew, full_cov=False, include_likelihood=True, Y_metadata=None):
        """gp.py:290-365 with the sparse posterior (predictive variable = Z)."""
        mu, var = self.posterior._raw_predict(self.kern, np.asarray(Xnew, dtype=np.float64), self.Z.values, full_cov)
        if include_likelihood:
            if isinstance(self.likelihood, HeteroscedasticGaussian) and Y_metadata is None:
                raise ValueError("a heteroscedastic likelihood needs Y_metadata (output_index) for the new points, or "
                                 "include_likelihood=False (gp_heteroscedastic_regression.py:13-15)")
            mu, var = self.likelihood.predictive_values(mu, var, full_cov, Y_metadata=Y_metadata)
        return mu, var
