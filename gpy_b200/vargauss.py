"""The variational Gaussian approximation (Opper & Archambeau 2009) for any likelihood, with the N^2 / N^3 work on the H100.

Mirrors:
    GPy.inference.latent_function_inference.VarGauss      GPy/inference/latent_function_inference/var_gauss.py:10-69
    GPy.models.GPVariationalGaussianApproximation          GPy/models/gp_var_gauss.py:11-29
(one output column, no mean function.)

One evaluation is gpx_vargauss_begin (K, m = K alpha, the factor of A = I + B K B, var = diag(Sigma) and the KL term) ->
likelihood.variational_expectations(Y, m, var) on the host -> gpx_vargauss_finish (the alpha, beta and kernel gradients,
the posterior). Any likelihood object with `variational_expectations` works.

The kernel gradient is the derivative of the bound. The reference's dF_dK (var_gauss.py:66) scales the rows of tmp by
dF_dv where the columns belong, so for a likelihood whose dF_dv is not constant its kernel gradient is not the derivative
of its own log marginal (for the Gaussian likelihood the two agree); the log marginal and the alpha and beta gradients
are the reference's.
"""
import numpy as np

from .kern import DeviceGradient, part_ngrad, single_kernel
from .laplace import PosteriorLaplace, _kernel_parts
from .model import GP
from .param import Param


def check_beta(beta):
    """beta as a flat float array; a zero or non-finite entry raises ValueError (B^-2 and Sigma are not defined there)"""
    b = np.asarray(beta, dtype=np.float64).reshape(-1)
    if not np.all(np.isfinite(b)) or np.any(b == 0):
        raise ValueError("VarGauss: beta must be finite and non-zero")
    return b


class VarGauss(object):
    """Drop-in for GPy's VarGauss (var_gauss.py:10-69): `inference(kern, X, likelihood, Y, ...)` returns
    (posterior, log_marginal, {'dL_dK', 'dL_dthetaL'}) and sets `alpha.gradient` and `beta.gradient` (:58-59). dL_dK is a
    DeviceGradient handle carrying the reduced kernel gradient; the posterior is a PosteriorLaplace on the device with
    woodbury_vector = alpha and woodbury_inv = B A^-1 B = (K + B^-2)^-1."""

    def __init__(self, alpha, beta, device=0, engine=None, max_tries=5):
        self.alpha, self.beta = alpha, beta
        self.device, self._engine, self.max_tries = device, engine, max_tries
        from .inference import _DataKey
        self._data_key = _DataKey()

    def on_optimization_start(self):
        pass

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

    def inference(self, kern, X, likelihood, Y, mean_function=None, Y_metadata=None, Z=None):
        if mean_function is not None:                                                       # :34-35
            raise NotImplementedError
        num_data, output_dim = np.shape(Y)
        assert output_dim == 1, "Only one output supported"                                 # :37
        desc = _kernel_parts(kern)
        if desc is None:
            raise ValueError("gpy_b200.VarGauss: the kernel is not one the device evaluates (a sum of products of "
                             "stationary, StdPeriodic, White and Bias kernels)")
        parts, key, leaves = desc
        single = single_kernel(kern)
        Xs = kern._slice_X(X) if single else np.asarray(X)
        return self.device_inference(Xs, Y, likelihood, Y_metadata, parts, key, [part_ngrad(l) for l, _ in leaves],
                                     single)

    def device_inference(self, Xs, Y, likelihood, Y_metadata, parts, key, ngrads, single):
        """one evaluation for the kernel described by parts (Engine.vargauss_begin's descriptors on the columns of Xs),
        keyed `key`, whose leaves have ngrads gradient entries each; single: one stationary kernel"""
        alpha = np.asarray(self.alpha, dtype=np.float64).reshape(-1)
        beta = check_beta(self.beta)
        Xs = np.ascontiguousarray(Xs, dtype=np.float64)
        Y = np.ascontiguousarray(Y, dtype=np.float64)
        N = Y.shape[0]
        eng = self.engine
        if not self._data_key.matches(Xs, Y):
            eng.set_data(Xs, Y)
            self._data_key.remember(Xs, Y)
        m, var, KL, _ = eng.vargauss_begin(parts, alpha, beta, self.max_tries)
        F, dF_dm, dF_dv, dF_dthetaL = likelihood.variational_expectations(Y, m[:, None], var[:, None],
                                                                          Y_metadata=Y_metadata)
        if dF_dthetaL is not None:                                                          # :46-50
            dL_dthetaL = dF_dthetaL.sum(1).sum(1)
        else:
            dL_dthetaL = np.array([])
        dalpha, dbeta, kgrad = eng.vargauss_finish(np.reshape(dF_dm, -1), np.reshape(dF_dv, -1))
        log_marginal = F.sum() - KL
        self.alpha.gradient = dalpha[:, None]
        self.beta.gradient = dbeta
        if single:
            dL_dK = DeviceGradient(eng, key, kgrad[0], kgrad[1:] if parts[0][1] else kgrad[1], N)
        else:
            part_grads, i = [], 0
            for n in ngrads:
                part_grads.append(kgrad[i:i + n])
                i += n
            dL_dK = DeviceGradient(eng, key, None, None, N, part_grads=part_grads)
        self.m, self.var, self.KL = m[:, None], var[:, None], KL
        return PosteriorLaplace(eng, N, 1, key), log_marginal, {"dL_dK": dL_dK, "dL_dthetaL": dL_dthetaL}


class GPVariationalGaussianApproximation(GP):
    """GPy.models.GPVariationalGaussianApproximation (gp_var_gauss.py:11-29): the name 'VarGP', parameters (and gradients)
    in the order kern, likelihood, alpha, beta; alpha starts at 0 (N x 1) and beta at 1 (N), both unconstrained."""

    def __init__(self, X, Y, kernel, likelihood, Y_metadata=None, device=0, engine=None):
        num_data = np.shape(Y)[0]
        self.alpha = Param("alpha", np.zeros((num_data, 1)), transform=None)
        self.beta = Param("beta", np.ones(num_data), transform=None)
        inf = VarGauss(self.alpha, self.beta, device=device, engine=engine)
        super(GPVariationalGaussianApproximation, self).__init__(X, Y, kernel, likelihood, name="VarGP",
                                                                 inference_method=inf, Y_metadata=Y_metadata,
                                                                 device=device, engine=engine)
        self.link_parameter(self.alpha)
        self.link_parameter(self.beta)
