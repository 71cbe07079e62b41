"""Expectation propagation for GP classification on the H100 (probit Bernoulli likelihood).

Mirrors:
    GPy.inference.latent_function_inference.EP   GPy/inference/latent_function_inference/expectation_propagation.py:187-434
        (inference, expectation_propagation, _init_approximations, _stop_criteria, _log_Z_tilde, _ep_marginal, _inference;
        EPDTC and the to_dict / loading serialisation stay out)
    GPy.inference.latent_function_inference.posterior.PosteriorEP   posterior.py:305-336
    GPy.models.GPClassification                                     GPy/models/gp_classification.py:10-39
The sites, the stopping rule, log Z~ and the update order (np.random.permutation on numpy's global generator, one draw per
sweep in both update modes, as the reference draws it) stay on the host; the sweeps (site updates and the recompute of
Sigma and mu) and the marginal with its kernel gradient are the gpx_ep_* calls.
"""
import numpy as np

from .kern import DeviceGradient, RBF, single_kernel
from .inference import _LazyAlpha
from .laplace import Bernoulli, PosteriorLaplace, _kernel_parts
from .model import GP

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


class EP(object):
    """Drop-in for GPy's EP (expectation_propagation.py:187-434) with the probit Bernoulli likelihood, one output column and
    no mean function: `inference(kern, X, likelihood, Y, ...)` returns (posterior, log_marginal, {'dL_dK', 'dL_dthetaL',
    'dL_dm'}) with the sweeps and the marginal on the device. dL_dK is a DeviceGradient handle carrying the reduced kernel
    gradient."""

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
        stop = False
        iterations = 0
        while not stop and (iterations < self.max_iters):
            update_order = np.random.permutation(num_data)                        # :332
            (ga_approx.tau, ga_approx.v, cav_params.tau, cav_params.v, marg_moments.Z_hat, marg_moments.mu_hat,
             marg_moments.sigma2_hat, _) = eng.ep_sweep(update_order, ga_approx.tau, ga_approx.v, eta=self.eta,
                                                        delta=self.delta, parallel=self.parallel_updates)
            if iterations > 0:
                stop = self._stop_criteria(ga_approx)
            self.ga_approx_old = gaussianApproximation(ga_approx.v.copy(), ga_approx.tau.copy())
            iterations += 1
        self.iterations = iterations
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
