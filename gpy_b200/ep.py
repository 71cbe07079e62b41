"""Expectation propagation for GP classification on the H100 (probit Bernoulli likelihood).

Mirrors:
    GPy.inference.latent_function_inference.EP   GPy/inference/latent_function_inference/expectation_propagation.py:187-434
        (inference, expectation_propagation, _init_approximations, _stop_criteria, _log_Z_tilde, _ep_marginal, _inference;
        EPDTC and the to_dict / loading serialisation stay out)
    GPy.inference.latent_function_inference.posterior.PosteriorEP   posterior.py:305-336
    GPy.models.GPClassification                                     GPy/models/gp_classification.py:10-39
    GPy.inference.latent_function_inference.EPDTC    expectation_propagation.py:436-611 (no to_dict serialisation)
    GPy.models.SparseGPClassification                GPy/models/sparse_gp_classification.py:14-60
The sites, the stopping rule, log Z~ and the update order (np.random.permutation on numpy's global generator, one draw per
sweep in both update modes, as the reference draws it) stay on the host; the sweeps (site updates and the recompute of
Sigma and mu) and the marginal with its kernel gradient are the gpx_ep_* calls.
"""
import numpy as np

from .kern import DeviceGradient, RBF, single_kernel
from .inference import _LazyAlpha
from .laplace import Bernoulli, PosteriorLaplace, _kernel_parts
from .model import GP
from .sparse import LazySparsePosterior, SparseGPRegression

log_2_pi = np.log(2 * np.pi)


class marginalMoments(object):
    """expectation_propagation.py:16-20"""

    def __init__(self, num_data):
        self.Z_hat = np.empty(num_data, dtype=np.float64)
        self.mu_hat = np.empty(num_data, dtype=np.float64)
        self.sigma2_hat = np.empty(num_data, dtype=np.float64)


class cavityParams(object):
    """expectation_propagation.py:23-29"""

    def __init__(self, num_data):
        self.tau = np.empty(num_data, dtype=np.float64)
        self.v = np.empty(num_data, dtype=np.float64)


class gaussianApproximation(object):
    """expectation_propagation.py:48-51: the site parameters"""

    def __init__(self, v, tau):
        self.tau = tau
        self.v = v


class PosteriorEP(PosteriorLaplace):
    """The posterior EP returns (:395: woodbury_inv = Wi, woodbury_vector = alpha, K), with PosteriorLaplace's members on
    the device (U~ U~^T of the last gpx_ep_finish is Wi) and the reference PosteriorEP's _raw_predict (posterior.py:305-336):
    no clip of the variance."""

    _var_floor = None


def _is_probit_bernoulli(likelihood):
    if isinstance(likelihood, Bernoulli):
        return True
    link = getattr(likelihood, "gp_link", None)
    return type(likelihood).__name__ == "Bernoulli" and type(link).__name__ == "Probit"


class posteriorParamsDTC(object):
    """expectation_propagation.py:144-185: mu and Sigma_diag of the sparse EP's last recompute (from the device)"""

    def __init__(self, mu, Sigma_diag):
        self.mu = mu
        self.Sigma_diag = Sigma_diag


class _EPBase(object):
    """EPBase (expectation_propagation.py:187-244): the options, reset, the stopping rule and the run loop EP and EPDTC
    share"""

    def __init__(self, epsilon=1e-6, eta=1., delta=1., always_reset=False, max_iters=np.inf, ep_mode="alternated",
                 parallel_updates=False, device=0, engine=None):
        self.always_reset = always_reset
        self.epsilon, self.eta, self.delta, self.max_iters = epsilon, eta, delta, max_iters
        self.ep_mode = ep_mode
        self.parallel_updates = parallel_updates
        self.loading = False
        self.device = device
        self._engine = engine
        from .inference import _DataKey
        self._data_key = _DataKey()
        self.reset()

    def reset(self):
        self.ga_approx_old = None
        self._ep_approximation = None

    def on_optimization_start(self):
        self._ep_approximation = None

    def on_optimization_end(self):
        pass

    def __getstate__(self):
        from .inference import _DataKey
        d = dict(self.__dict__)
        d["_engine"], d["_data_key"] = None, _DataKey()
        return d

    @property
    def engine(self):
        if self._engine is None:
            from . import _ffi
            self._engine = _ffi.Engine(self.device)
        return self._engine

    def invalidate_data(self):
        self._data_key.invalidate()

    def _stop_criteria(self, ga_approx):
        tau_diff = np.mean(np.square(ga_approx.tau - self.ga_approx_old.tau))
        v_diff = np.mean(np.square(ga_approx.v - self.ga_approx_old.v))
        return ((tau_diff < self.epsilon) and (v_diff < self.epsilon))

    def _run_sweeps(self, num_data, sweep):
        """the loop of expectation_propagation (:300-309, :495-509): one update order drawn per sweep in both update
        modes, sweep(update_order) runs it with the recompute, ga_approx_old saved after every sweep"""
        stop = False
        iterations = 0
        while not stop and (iterations < self.max_iters):
            update_order = np.random.permutation(num_data)                        # :332, :555
            ga_approx = sweep(update_order)
            if iterations > 0:
                stop = self._stop_criteria(ga_approx)
            self.ga_approx_old = gaussianApproximation(ga_approx.v.copy(), ga_approx.tau.copy())
            iterations += 1
        self.iterations = iterations


class EP(_EPBase):
    """Drop-in for GPy's EP (expectation_propagation.py:187-434) with the probit Bernoulli likelihood, one output column and
    no mean function: `inference(kern, X, likelihood, Y, ...)` returns (posterior, log_marginal, {'dL_dK', 'dL_dthetaL',
    'dL_dm'}) with the sweeps and the marginal on the device. dL_dK is a DeviceGradient handle carrying the reduced kernel
    gradient."""

    def inference(self, kern, X, likelihood, Y, mean_function=None, Y_metadata=None, precision=None, K=None):
        if mean_function is not None:
            raise NotImplementedError("gpy_b200.EP: a mean function is not supported on the device")
        if not _is_probit_bernoulli(likelihood):
            raise NotImplementedError("gpy_b200.EP: only the Bernoulli likelihood with the probit link is supported")
        if K is not None:
            raise NotImplementedError("gpy_b200.EP: a precomputed K is not supported; the device builds K")
        desc = _kernel_parts(kern)
        if desc is None:
            raise ValueError("gpy_b200.EP: the kernel is not one the device evaluates (a sum of products of "
                             "stationary, StdPeriodic, White and Bias kernels)")
        parts, key, leaves = desc
        single = single_kernel(kern)
        Xs = kern._slice_X(X) if single else np.asarray(X)
        from .kern import part_ngrad
        return self.device_inference(Xs, Y, likelihood, Y_metadata, parts, key, [part_ngrad(l) for l, _ in leaves],
                                     single)

    def device_inference(self, Xs, Y, likelihood, Y_metadata, parts, key, ngrads, single):
        """:246-277 for the kernel described by parts (Engine.ep_begin's descriptors on the columns of Xs), keyed `key`,
        whose leaves have ngrads gradient entries each; single: one stationary kernel"""
        if self.always_reset and not self.loading:
            self.reset()
        num_data, output_dim = Y.shape
        assert output_dim == 1, "ep in 1D only (for now!)"
        Yv = np.asarray(Y, dtype=np.float64)
        if np.any(~((Yv == 1) | (Yv == 0) | (Yv == -1))):
            raise ValueError("bad value for Bernoulli observation (0, 1)")                   # bernoulli.py:67-72
        Xs = np.ascontiguousarray(Xs, dtype=np.float64)
        Yc = np.ascontiguousarray(Yv)
        eng = self.engine
        if not self._data_key.matches(Xs, Yc):
            eng.set_data(Xs, Yc)
            self._data_key.remember(Xs, Yc)
        eng.ep_begin(parts)
        # _ep_approximation keeps the reference's shape (post_params, ga_approx, cav_params, log_Z_tilde); Sigma stays
        # on the device, so post_params is None
        if self.ep_mode == "nested" and not self.loading:
            self._ep_approximation = None
            _, ga_approx, cav_params, log_Z_tilde = self._ep_approximation = self.expectation_propagation(eng, num_data)
        elif self.ep_mode == "alternated" or self.loading:
            if getattr(self, "_ep_approximation", None) is None:
                _, ga_approx, cav_params, log_Z_tilde = self._ep_approximation = self.expectation_propagation(eng,
                                                                                                          num_data)
            else:
                _, ga_approx, cav_params, log_Z_tilde = self._ep_approximation
        else:
            raise ValueError("ep_mode value not valid")
        self.loading = False
        return self._inference(eng, Y, ga_approx, cav_params, likelihood, log_Z_tilde, ngrads, single, key, parts,
                               Y_metadata=Y_metadata)

    def expectation_propagation(self, eng, num_data):
        """:279-310 with the sweeps on the device -> (None, ga_approx, cav_params, log_Z_tilde)"""
        marg_moments = marginalMoments(num_data)
        cav_params = cavityParams(num_data)
        ga_approx = self._init_approximations(eng, num_data)

        def sweep(update_order):
            (ga_approx.tau, ga_approx.v, cav_params.tau, cav_params.v, marg_moments.Z_hat, marg_moments.mu_hat,
             marg_moments.sigma2_hat, _) = eng.ep_sweep(update_order, ga_approx.tau, ga_approx.v, eta=self.eta,
                                                        delta=self.delta, parallel=self.parallel_updates)
            return ga_approx

        self._run_sweeps(num_data, sweep)
        log_Z_tilde = self._log_Z_tilde(marg_moments, ga_approx, cav_params)
        return (None, ga_approx, cav_params, log_Z_tilde)

    def _init_approximations(self, eng, num_data):
        """:312-328: zero sites and Sigma = K + 1e-7 I, or the recompute from the sites of the last run"""
        if self.ga_approx_old is None:
            v_tilde, tau_tilde = np.zeros((2, num_data))
            eng.ep_start(parallel=self.parallel_updates)
            return gaussianApproximation(v_tilde, tau_tilde)
        assert self.ga_approx_old.v.size == num_data, "data size mis-match: did you change the data? try resetting!"
        ga_approx = gaussianApproximation(self.ga_approx_old.v, self.ga_approx_old.tau)
        eng.ep_start(ga_approx.tau, ga_approx.v, parallel=self.parallel_updates)
        return ga_approx

    def _log_Z_tilde(self, marg_moments, ga_approx, cav_params):
        return np.sum((
            np.log(marg_moments.Z_hat)
            + 0.5 * np.log(2 * np.pi) + 0.5 * np.log(1 + ga_approx.tau / cav_params.tau)
            - 0.5 * ((ga_approx.v) ** 2 * 1. / (cav_params.tau + ga_approx.tau))
            + 0.5 * (cav_params.v * (((ga_approx.tau / cav_params.tau) * cav_params.v - 2.0 * ga_approx.v)
                                     * 1. / (cav_params.tau + ga_approx.tau)))
        ))

    def _ep_marginal(self, eng, ga_approx, Z_tilde):
        """:363-377 with mean_prior = 0: B_logdet and v~^T Sigma v~ from gpx_ep_finish"""
        B_logdet, vSv, diag_dL_dK, kgrad, _ = eng.ep_finish(ga_approx.tau, ga_approx.v)
        log_marginal = 0.5 * (-len(ga_approx.tau) * log_2_pi - B_logdet + vSv - 0.0)
        log_marginal += Z_tilde
        return log_marginal, diag_dL_dK, kgrad

    def _inference(self, eng, Y, ga_approx, cav_params, likelihood, Z_tilde, ngrads, single, key, parts, Y_metadata=None):
        """:379-395"""
        log_marginal, diag_dL_dK, kgrad = self._ep_marginal(eng, ga_approx, Z_tilde)
        N = Y.shape[0]
        if single:
            dL_dK = DeviceGradient(eng, key, kgrad[0], kgrad[1:] if parts[0][1] else kgrad[1], N)
        else:
            part_grads, i = [], 0
            for n in ngrads:
                part_grads.append(kgrad[i:i + n])
                i += n
            dL_dK = DeviceGradient(eng, key, None, None, N, part_grads=part_grads)
        dL_dthetaL = likelihood.ep_gradients(Y, cav_params.tau, cav_params.v, diag_dL_dK, Y_metadata=Y_metadata,
                                             quad_mode='gh')
        post = PosteriorEP(eng, N, 1, key)
        return post, log_marginal, {"dL_dK": dL_dK, "dL_dthetaL": dL_dthetaL, "dL_dm": _LazyAlpha(post)}


class GPClassification(GP):
    """GPy.models.GPClassification (gp_classification.py:10-39): RBF kernel, Bernoulli likelihood and EP by default."""

    def __init__(self, X, Y, kernel=None, Y_metadata=None, mean_function=None, inference_method=None, likelihood=None,
                 normalizer=False, device=0, engine=None):
        if kernel is None:
            kernel = RBF(X.shape[1])
        if likelihood is None:
            likelihood = Bernoulli()
        if inference_method is None:
            inference_method = EP(device=device, engine=engine)
        super(GPClassification, self).__init__(X, Y, kernel, likelihood, mean_function=mean_function,
                                               inference_method=inference_method, name="gp_classification",
                                               device=device, engine=engine, Y_metadata=Y_metadata,
                                               normalizer=normalizer)


class EPDTC(_EPBase):
    """Drop-in for GPy's EPDTC (expectation_propagation.py:436-611) with the probit Bernoulli likelihood, one output column
    and no mean function: `inference(kern, X, Z, likelihood, Y, ...)` returns (posterior, log_marginal, grad_dict) in
    VarDTC's shape (`dvariance` / `dlengthscale` or `part_grads`, `dZ`, `dL_dthetaL`). The sweeps run on the device in
    M-space (gpx_epdtc_sweep); the marginal is VarDTC at Y = v~ / tau~ and precision tau~ plus log Z~ (:474-482, the DTC
    form of :514-520). _ep_approximation is the reference's 3-tuple (post_params, ga_approx, log_Z_tilde)."""

    def inference(self, kern, X, Z, likelihood, Y, mean_function=None, Y_metadata=None, Lm=None, dL_dKmm=None, psi0=None,
                  psi1=None, psi2=None):
        from .kern import RatQuad, StdPeriodic, flatten_parts, single_kernel, Stationary
        if mean_function is not None:                                              # var_dtc.py:85-86 (het_noise)
            raise ValueError('Mean function not implemented with uncertain inputs or heteroscedasticity')
        if not _is_probit_bernoulli(likelihood):
            raise NotImplementedError("gpy_b200.EPDTC: only the Bernoulli likelihood with the probit link is supported")
        if any(a is not None for a in (Lm, dL_dKmm, psi0, psi1, psi2)):
            raise NotImplementedError("gpy_b200.EPDTC: precomputed Lm, dL_dKmm or psi statistics are not supported")
        leaves = None if single_kernel(kern) else flatten_parts(kern)
        for k in ([kern] if leaves is None else [q for q, _ in (leaves or [])]):
            if isinstance(k, (RatQuad, StdPeriodic)):
                raise NotImplementedError("gpy_b200.EPDTC: %s is not on the device's sparse evaluation (RBF, "
                                          "Exponential, Matern32, Matern52, White, Bias and their sums and products are)"
                                          % type(k).__name__)
        if leaves is None and not isinstance(kern, Stationary):
            raise TypeError("gpy_b200.EPDTC accelerates gpy_b200.kern stationary kernels and sums / products of them "
                            "with White and Bias")
        desc = _kernel_parts(kern)
        parts, key, fl = desc
        single = leaves is None
        Xs = kern._slice_X(X) if single else np.asarray(X)
        Zs = kern._slice_X(Z) if single else np.asarray(Z)
        from .kern import part_ngrad
        return self.device_inference(Xs, Zs, Y, parts, key, [part_ngrad(q) for q, _ in fl], single)

    def device_inference(self, Xs, Zs, Y, parts, key, ngrads, single):
        """:437-482 for the kernel described by parts at the columns of Xs and Zs"""
        if self.always_reset and not self.loading:
            self.reset()
        num_data, output_dim = Y.shape
        assert output_dim == 1, "ep in 1D only (for now!)"
        Yv = np.asarray(Y, dtype=np.float64)
        if np.any(~((Yv == 1) | (Yv == 0) | (Yv == -1))):
            raise ValueError("bad value for Bernoulli observation (0, 1)")                   # bernoulli.py:67-72
        Xs = np.ascontiguousarray(Xs, dtype=np.float64)
        Zs = np.ascontiguousarray(Zs, dtype=np.float64)
        Yc = np.ascontiguousarray(Yv)
        eng = self.engine
        if not self._data_key.matches(Xs, Yc):
            eng.sparse_set_data(Xs, Yc)
            self._data_key.remember(Xs, Yc)
        # begin builds Kmn and factors Kmm for the sweeps; in alternated mode with kept sites only finish reads them, and
        # finish (VarDTC) builds both again (DESIGN §7d counts the cost)
        eng.epdtc_begin(parts, Zs)
        if self.ep_mode == "nested" and not self.loading:
            self._ep_approximation = None
            post_params, ga_approx, log_Z_tilde = self._ep_approximation = self.expectation_propagation(eng, num_data)
        elif self.ep_mode == "alternated" or self.loading:
            if getattr(self, "_ep_approximation", None) is None:
                post_params, ga_approx, log_Z_tilde = self._ep_approximation = self.expectation_propagation(eng,
                                                                                                        num_data)
            else:
                post_params, ga_approx, log_Z_tilde = self._ep_approximation
        else:
            raise ValueError("ep_mode value not valid")
        self.loading = False
        lml, grad, dZ, _ = eng.epdtc_finish(ga_approx.tau, ga_approx.v)
        lml += log_Z_tilde                                                                  # var_dtc.py:166-170
        gd = {"dZ": dZ, "dL_dthetaL": np.zeros(0), "num_data": num_data}
        if single:
            gd["dvariance"], gd["dlengthscale"] = grad[0], grad[1:]
        else:
            blocks, i = [], 0
            for n in ngrads:
                blocks.append(grad[i:i + n])
                i += n
            gd["part_grads"] = blocks
        return LazySparsePosterior(eng, key, Zs), float(lml), gd

    def expectation_propagation(self, eng, num_data):
        """:484-512 with the sweeps on the device -> (post_params, ga_approx, log_Z_tilde)"""
        marg_moments = marginalMoments(num_data)
        cav_params = cavityParams(num_data)
        ga_approx, post_params = self._init_approximations(eng, num_data)

        def sweep(update_order):
            (ga_approx.tau, ga_approx.v, cav_params.tau, cav_params.v, marg_moments.Z_hat, marg_moments.mu_hat,
             marg_moments.sigma2_hat, _, post_params.mu, post_params.Sigma_diag) = eng.epdtc_sweep(
                update_order, ga_approx.tau, ga_approx.v, eta=self.eta, delta=self.delta, parallel=self.parallel_updates)
            return ga_approx

        self._run_sweeps(num_data, sweep)
        log_Z_tilde = self._log_Z_tilde(marg_moments, ga_approx, cav_params)
        return post_params, ga_approx, log_Z_tilde

    def _init_approximations(self, eng, num_data):
        """:522-551: zero sites, LLT = Kmm and Sigma_diag = diag(Qnn) + 1e-8, or the recompute from the sites of the
        last run plus 1e-8"""
        if self.ga_approx_old is None:
            v_tilde, tau_tilde = np.zeros((2, num_data))
            _, mu, sd = eng.epdtc_start(parallel=self.parallel_updates)
            return gaussianApproximation(v_tilde, tau_tilde), posteriorParamsDTC(mu, sd)
        assert self.ga_approx_old.v.size == num_data, "data size mis-match: did you change the data? try resetting!"
        ga_approx = gaussianApproximation(self.ga_approx_old.v, self.ga_approx_old.tau)
        _, mu, sd = eng.epdtc_start(ga_approx.tau, ga_approx.v, parallel=self.parallel_updates)
        return ga_approx, posteriorParamsDTC(mu, sd)

    def _log_Z_tilde(self, marg_moments, ga_approx, cav_params):
        """:514-520"""
        mu_tilde = ga_approx.v / ga_approx.tau
        mu_cav = cav_params.v / cav_params.tau
        sigma2_sigma2tilde = 1. / cav_params.tau + 1. / ga_approx.tau
        return np.sum((np.log(marg_moments.Z_hat) + 0.5 * np.log(2 * np.pi) + 0.5 * np.log(sigma2_sigma2tilde)
                       + 0.5 * ((mu_cav - mu_tilde) ** 2) / (sigma2_sigma2tilde)))


class SparseGPClassification(SparseGPRegression):
    """GPy.models.SparseGPClassification (sparse_gp_classification.py:14-60): RBF kernel, Bernoulli likelihood and EPDTC
    by default, Z drawn from X with np.random.permutation. predict goes through Bernoulli.predictive_values over the
    device posterior."""

    def __init__(self, X, Y=None, likelihood=None, kernel=None, Z=None, num_inducing=10, Y_metadata=None,
                 mean_function=None, inference_method=None, normalizer=False, device=0, engine=None):
        if mean_function is not None:
            raise ValueError('Mean function not implemented with uncertain inputs or heteroscedasticity')
        if normalizer:
            raise NotImplementedError("gpy_b200.SparseGPClassification: a normalizer is not supported")
        X = np.asarray(X, dtype=np.float64)
        if kernel is None:
            kernel = RBF(X.shape[1])
        if likelihood is None:
            likelihood = Bernoulli()
        if Z is None:
            i = np.random.permutation(X.shape[0])[:num_inducing]                # sparse_gp_classification.py:42-44
            Z = X[i].copy()
        else:
            assert Z.shape[1] == X.shape[1]
        if inference_method is None:
            inference_method = EPDTC(device=device, engine=engine)
        super(SparseGPClassification, self).__init__(X, Y, kernel=kernel, Z=Z, device=device, engine=engine,
                                                     name="SparseGPClassification", likelihood=likelihood,
                                                     Y_metadata=Y_metadata, inference_method=inference_method)
