"""The Laplace approximation for non-Gaussian likelihoods on the H100 (GP classification, robust and count regression).

Mirrors:
    GPy.inference.latent_function_inference.Laplace   GPy/inference/latent_function_inference/laplace.py:24-353
        (inference, rasm_mode, mode_computations; LaplaceBlock, EP and the quadrature LOO stay out)
    GPy.likelihoods.Bernoulli with the probit link     GPy/likelihoods/bernoulli.py, link_functions.py:109-126 and the
                                                       chain rules of likelihood.py:544-733
    GPy.likelihoods.StudentT (identity link)           GPy/likelihoods/student_t.py
The N^2 / N^3 work (K, the factorisation of B = I + W^1/2 K W^1/2 per Newton step, the mode computations and the kernel
gradient) is the gpx_laplace_* calls; the O(N) likelihood terms, Brent's line search and the loop stay on the host, as in
the reference. Any likelihood object with GPy's interface (logpdf, dlogpdf_df, d2logpdf_df2, d3logpdf_df3,
_laplace_gradients, log_concave, size) works, GPy's own included.
"""
import warnings

import numpy as np
from scipy import optimize
from scipy.integrate import quad
from scipy.special import gammaln, ndtr
from scipy.special import psi as digamma

from .inference import PosteriorExact
from .kern import DeviceGradient, composite_state_key, flatten_parts, part_descriptor, part_ngrad, single_kernel
from .param import Param, Parameterized

_sqrt_2pi = np.sqrt(2 * np.pi)
_lim_val_square = np.sqrt(np.finfo(np.float64).max)
_lim_val_exp = np.log(np.finfo(np.float64).max)
_lim_val_cube = np.nextafter(np.finfo(np.float64).max ** (1 / 3.0), -np.inf)


def std_norm_pdf(x):
    """util/univariate_Gaussian.py:10-12"""
    x = np.clip(x, -1e150, 1e150)
    return np.exp(-np.square(x) / 2) / _sqrt_2pi


def _chain_1(df_dg, dg_dx):
    """util/misc.py:36-45"""
    if np.all(dg_dx == 1.):
        return df_dg
    return df_dg * dg_dx


def _chain_2(d2f_dg2, dg_dx, df_dg, d2g_dx2):
    """util/misc.py:47-58"""
    if np.all(dg_dx == 1.) and np.all(d2g_dx2 == 0):
        return d2f_dg2
    dg_dx_2 = np.clip(dg_dx, -np.inf, _lim_val_square) ** 2
    return d2f_dg2 * dg_dx_2 + df_dg * d2g_dx2


def _chain_3(d3f_dg3, dg_dx, d2f_dg2, d2g_dx2, df_dg, d3g_dx3):
    """util/misc.py:60-70"""
    if np.all(dg_dx == 1.) and np.all(d2g_dx2 == 0) and np.all(d3g_dx3 == 0):
        return d3f_dg3
    dg_dx_3 = np.clip(dg_dx, -np.inf, _lim_val_cube) ** 3
    return d3f_dg3 * dg_dx_3 + 3 * d2f_dg2 * dg_dx * d2g_dx2 + df_dg * d3g_dx3


def _gh_points(T=20):
    """likelihood.py:268-271: the T-point Gauss-Hermite rule"""
    return np.polynomial.hermite.hermgauss(T)


def quadrature_expectations(lik, Y, m, v, dlogpdf_dtheta=None, gh=None):
    """Likelihood.variational_expectations (likelihood.py:358-411): E_q[log p(y | f)] and its derivatives in m and v for
    q(f) = N(m, v) by Gauss-Hermite quadrature on lik's logpdf, dlogpdf_df and d2logpdf_df2; dlogpdf_dtheta(f, y) -> the
    (size, N, T) parameter derivatives on the grid, or None for a likelihood without parameters. -> (F, dF_dm, dF_dv,
    dF_dtheta (size, N, P) or None)"""
    gh_x, gh_w = _gh_points() if gh is None else gh
    shape = m.shape
    m, v, Y = m.flatten(), v.flatten(), Y.flatten()
    X = gh_x[None, :] * np.sqrt(2. * v[:, None]) + m[:, None]
    logp = lik.logpdf(X, Y[:, None])
    dlogp_dx = lik.dlogpdf_df(X, Y[:, None])
    d2logp_dx2 = lik.d2logpdf_df2(X, Y[:, None])
    F = np.dot(logp, gh_w) / np.sqrt(np.pi)
    dF_dm = np.dot(dlogp_dx, gh_w) / np.sqrt(np.pi)
    dF_dv = np.dot(d2logp_dx2, gh_w) / np.sqrt(np.pi)
    dF_dv /= 2.
    if not (np.all(np.isfinite(dF_dv)) and np.all(np.isfinite(dF_dm))):
        # the reference stops on an undefined name here (likelihood.py:400-403)
        raise NameError("name 'stop' is not defined")
    dF_dtheta = None
    if dlogpdf_dtheta is not None:
        dt = np.dot(dlogpdf_dtheta(X, Y[:, None]), gh_w) / np.sqrt(np.pi)
        dF_dtheta = dt.reshape(dt.shape[0], shape[0], shape[1])
    return F.reshape(*shape), dF_dm.reshape(*shape), dF_dv.reshape(*shape), dF_dtheta


class Bernoulli(Parameterized):
    """GPy.likelihoods.Bernoulli with its default probit link (bernoulli.py; link_functions.py:109-126): y in {0, 1},
    p(y = 1 | f) = Phi(f). Log-concave, no parameters."""

    log_concave = True
    size = 0

    def __init__(self, name="Bernoulli"):
        super(Bernoulli, self).__init__(name)

    # the probit link (link_functions.py:116-126)
    @staticmethod
    def _transf(f):
        return ndtr(f)

    @staticmethod
    def _d3transf(f):
        return (np.clip(f, -np.inf, _lim_val_square) ** 2 - 1.) * std_norm_pdf(f)

    # the link-level terms (bernoulli.py)
    @staticmethod
    def logpdf_link(inv_link_f, y, Y_metadata=None):
        p = np.where(y == 1, inv_link_f, 1. - inv_link_f)
        return np.log(np.clip(p, 1e-9, np.inf))

    @staticmethod
    def dlogpdf_dlink(inv_link_f, y, Y_metadata=None):
        ff = np.clip(inv_link_f, 1e-9, 1 - 1e-9)
        denom = np.where(y == 1, ff, -(1 - ff))
        return 1. / denom

    @staticmethod
    def d2logpdf_dlink2(inv_link_f, y, Y_metadata=None):
        arg = np.where(y == 1, inv_link_f, 1. - inv_link_f)
        return -1. / np.square(np.clip(arg, 1e-9, 1e9))

    @staticmethod
    def d3logpdf_dlink3(inv_link_f, y, Y_metadata=None):
        state = np.seterr(divide="ignore")
        try:
            return np.where(y == 1, 2. / (inv_link_f ** 3), -2. / ((1. - inv_link_f) ** 3))
        finally:
            np.seterr(**state)

    # the f-level terms through the chain rules (likelihood.py:544-656)
    def logpdf(self, f, y, Y_metadata=None):
        return self.logpdf_link(self._transf(f), y)

    def dlogpdf_df(self, f, y, Y_metadata=None):
        return _chain_1(self.dlogpdf_dlink(self._transf(f), y), std_norm_pdf(f))

    def d2logpdf_df2(self, f, y, Y_metadata=None):
        g = self._transf(f)
        return _chain_2(self.d2logpdf_dlink2(g, y), std_norm_pdf(f), self.dlogpdf_dlink(g, y), -f * std_norm_pdf(f))

    def d3logpdf_df3(self, f, y, Y_metadata=None):
        g = self._transf(f)
        return _chain_3(self.d3logpdf_dlink3(g, y), std_norm_pdf(f), self.d2logpdf_dlink2(g, y), -f * std_norm_pdf(f),
                        self.dlogpdf_dlink(g, y), self._d3transf(f))

    def variational_expectations(self, Y, m, v, gh_points=None, Y_metadata=None):
        """bernoulli.py:94-115 (probit): the 20-point Gauss-Hermite rule on log Phi(y_sign f), p clipped to [1e-9, 1 - 1e-9]
        -> (F, dF_dmu, dF_dv, None)"""
        gh_x, gh_w = _gh_points() if gh_points is None else gh_points
        gh_w = gh_w / np.sqrt(np.pi)
        shape = m.shape
        m, v, Y = m.flatten(), v.flatten(), Y.flatten()
        Ysign = np.where(Y == 1, 1, -1)
        X = gh_x[None, :] * np.sqrt(2. * v[:, None]) + (m * Ysign)[:, None]
        p = ndtr(X)
        p = np.clip(p, 1e-9, 1. - 1e-9)
        N = std_norm_pdf(X)
        F = np.log(p).dot(gh_w)
        NoverP = N / p
        dF_dm = (NoverP * Ysign[:, None]).dot(gh_w)
        dF_dv = -0.5 * (NoverP ** 2 + NoverP * X).dot(gh_w)
        return F.reshape(*shape), dF_dm.reshape(*shape), dF_dv.reshape(*shape), None

    def _laplace_gradients(self, f, y, Y_metadata=None):
        """likelihood.py:722-733 for a likelihood without parameters: three (0, N, 1) arrays"""
        z = np.zeros((0, f.shape[0], f.shape[1]))
        return z, z.copy(), z.copy()

    def update_gradients(self, grad):
        pass

    def predictive_mean(self, mu, variance, Y_metadata=None):
        return ndtr(mu / np.sqrt(1 + variance))                                   # bernoulli.py predictive_mean (probit)

    def predictive_variance(self, mu, variance, pred_mean, Y_metadata=None):
        return np.nan

    def ep_gradients(self, Y, cav_tau, cav_v, dL_dKdiag, Y_metadata=None, quad_mode='gk', boost_grad=1.):
        """likelihood.py:273-309 for a likelihood without parameters"""
        return np.zeros(0)

    def predictive_values(self, mu, var, full_cov=False, Y_metadata=None):
        """likelihood.py:734-755"""
        pred_mean = self.predictive_mean(mu, var, Y_metadata=Y_metadata)
        return pred_mean, self.predictive_variance(mu, var, pred_mean, Y_metadata=Y_metadata)


class StudentT(Parameterized):
    """GPy.likelihoods.StudentT with its identity link (student_t.py): parameters t_scale2 (sigma2) and deg_free (v), in
    that order. Not log-concave: Laplace clips its W to [1e-6, 1e30] for B (laplace.py:319-321)."""

    log_concave = False

    def __init__(self, deg_free=5, sigma2=2, name="Student_T"):
        super(StudentT, self).__init__(name)
        self.sigma2 = Param("t_scale2", float(sigma2))
        self.v = Param("deg_free", float(deg_free))
        self.link_parameter(self.sigma2)
        self.link_parameter(self.v)

    size = property(lambda self: 2)

    def _sv(self):
        return float(self.sigma2.values.reshape(-1)[0]), float(self.v.values.reshape(-1)[0])

    def update_gradients(self, grads):
        self.sigma2.gradient = np.atleast_1d(grads[0])
        self.v.gradient = np.atleast_1d(grads[1])

    def logpdf(self, f, y, Y_metadata=None):
        s2, v = self._sv()
        e = y - f
        return (+gammaln((v + 1) * 0.5) - gammaln(v * 0.5) - 0.5 * np.log(s2 * v * np.pi)
                - 0.5 * (v + 1) * np.log(1 + (1 / v) * ((e ** 2) / s2)))

    def dlogpdf_df(self, f, y, Y_metadata=None):
        s2, v = self._sv()
        e = y - f
        return ((v + 1) * e) / (v * s2 + (e ** 2))

    def d2logpdf_df2(self, f, y, Y_metadata=None):
        s2, v = self._sv()
        e = y - f
        return ((v + 1) * (e ** 2 - v * s2)) / ((s2 * v + e ** 2) ** 2)

    def d3logpdf_df3(self, f, y, Y_metadata=None):
        s2, v = self._sv()
        e = y - f
        return -(2 * (v + 1) * (-e) * (e ** 2 - 3 * v * s2)) / ((e ** 2 + s2 * v) ** 3)

    def _laplace_gradients(self, f, y, Y_metadata=None):
        """likelihood.py:722-733 with the identity link: d/d(t_scale2, deg_free) of logpdf, its f-derivative and its
        second f-derivative, each (2, N, 1)"""
        s2, df = self._sv()
        e = y - f
        e2 = np.square(e)
        dvar = df * (e2 - s2) / (2 * s2 * (s2 * df + e2))
        dv = 0.5 * digamma(0.5 * (df + 1)) - 0.5 * digamma(0.5 * df) - 1.0 / (2 * df)
        dv = dv + 0.5 * (df + 1) * e2 / (df * (e2 + s2 * df))
        dv = dv - 0.5 * np.log1p(e2 / (s2 * df))
        d1var = (df * (df + 1) * (-e)) / ((s2 * df + e ** 2) ** 2)
        d1v = e * (e2 - s2) / (e2 + s2 * df) ** 2
        d2var = (df * (df + 1) * (s2 * df - 3 * (e ** 2))) / ((s2 * df + (e ** 2)) ** 3)
        e2_s2v = e ** 2 + s2 * df
        d2v = (-s2 * (df + 1) + e2 - s2 * df) / e2_s2v ** 2 - 2 * s2 * (df + 1) * (e2 - s2 * df) / e2_s2v ** 3
        return np.array((dvar, dv)), np.array((d1var, d1v)), np.array((d2var, d2v))

    def variational_expectations(self, Y, m, v, gh_points=None, Y_metadata=None):
        """likelihood.py:358-411 (the generic quadrature; student_t.py has no closed form) -> (F, dF_dmu, dF_dv,
        dF_dtheta (2, N, P): t_scale2, deg_free)"""
        return quadrature_expectations(self, Y, m, v, lambda f, y: self._laplace_gradients(f, y)[0], gh_points)

    def predictive_mean(self, mu, sigma, Y_metadata=None):
        return mu                                                                  # the identity link (student_t.py)

    def conditional_variance(self, gp):
        _, df = self._sv()
        return df / (df - 2.0)

    def predictive_variance(self, mu, variance, predictive_mean=None, Y_metadata=None):
        """student_t.py predictive_variance: NaN for deg_free <= 2, else Likelihood.predictive_variance
        (likelihood.py:440-498) restated: the same quad integrands, the p < 1e-10 cutoffs and the same limits (the second
        integral runs from +inf to +inf as there, so its value is 0 and the variance is E(V(y|f)) - mu^2)"""
        _, df = self._sv()
        if df <= 2.0:
            return np.empty(mu.shape) * np.nan
        normalizer = np.sqrt(2 * np.pi * variance)
        fmin_v, fmin_m, fmax = -np.inf, np.inf, np.inf

        def int_var(f, m, v):
            p = np.exp(np.clip(-(0.5 / v) * np.square(f - m), -np.inf, _lim_val_exp))
            return 0. if p < 1e-10 else self.conditional_variance(f) * p

        def sc(a):   # one row's value as a scalar, so that the integrand returns a float (the same arithmetic)
            return float(np.asarray(a).reshape(-1)[0])

        exp_var = np.array([quad(int_var, fmin_v, fmax, args=(sc(mj), sc(s2j)))[0]
                            for mj, s2j in zip(mu, variance)])[:, None] / normalizer
        if predictive_mean is None:
            predictive_mean = self.predictive_mean(mu, variance)
        predictive_mean_sq = predictive_mean ** 2

        def int_pred_mean_sq(f, m, v, predictive_mean_sq):
            p = np.exp(-(0.5 / v) * np.square(f - m))
            return 0. if p < 1e-10 else f ** 2 * p

        exp_exp2 = np.array([quad(int_pred_mean_sq, fmin_m, fmax, args=(sc(mj), sc(s2j), sc(pm2j)))[0]
                             for mj, s2j, pm2j in zip(mu, variance, predictive_mean_sq)])[:, None] / normalizer
        return exp_var + (exp_exp2 - predictive_mean_sq)

    def predictive_values(self, mu, var, full_cov=False, Y_metadata=None):
        """likelihood.py:734-755"""
        pred_mean = self.predictive_mean(mu, var, Y_metadata=Y_metadata)
        return pred_mean, self.predictive_variance(mu, var, pred_mean, Y_metadata=Y_metadata)


class PosteriorLaplace(PosteriorExact):
    """The posterior Laplace returns (laplace.py:146: woodbury_vector = Ki_f_hat, woodbury_inv = K_Wi_i, K), its members
    on the device: woodbury_inv is U~ U~^T of the last gpx_laplace_finish, woodbury_chol the reference's lazy value
    (posterior.py:143-173), and _raw_predict the reference Posterior's formula (posterior.py:220-248) on the device with its
    1e-15 clip of the diagonal variance. The joint posterior and the predictive gradients take the exact model's device
    routes, which read the same U~; for another kernel they use woodbury_inv on the host."""

    @property
    def woodbury_chol(self):
        """posterior.py:152-159: Li of pdinv(woodbury_inv) (util/linalg.py:193-214: the inverse of jitchol's factor), in
        the (N, N, 1) array np.atleast_3d gives it"""
        if "woodbury_chol" not in self._cache:
            from . import _ffi
            Li = _ffi.pdinv(self.woodbury_inv, want=("Li",))[2]
            self._cache["woodbury_chol"] = np.atleast_3d(np.ascontiguousarray(Li))
        return self._cache["woodbury_chol"]

    def covariance_between_points(self, kern, X, X1, X2):
        """K(X1, X2) - K(X1, X) K_Wi_i K(X, X2): gpx_posterior_covariance for the evaluated kernel, else with woodbury_inv
        on the host (the factor form of posterior.py:109-130 needs a woodbury_chol L with L L^T = woodbury_inv^-1, which
        this posterior does not have)"""
        if self._on_device(kern):
            return super(PosteriorLaplace, self).covariance_between_points(kern, X, X1, X2)
        X2 = X1 if X2 is None else X2
        return kern.K(X1, X2) - kern.K(X1, X).dot(self.woodbury_inv).dot(kern.K(X, X2))

    _var_floor = 1e-15   # the clip of the diagonal variance (posterior.py:245); PosteriorEP has none

    def _floor(self, var):
        return var if self._var_floor is None else np.clip(var, self._var_floor, np.inf)

    def _raw_predict(self, kern, Xnew, pred_var=None, full_cov=False):
        if not self._is_evaluated(kern):
            Kx = kern.K(pred_var, Xnew)
            mu = np.dot(Kx.T, self.woodbury_vector)
            if full_cov:
                return mu, kern.K(Xnew) - np.dot(Kx.T, np.dot(self.woodbury_inv, Kx))
            var = kern.Kdiag(Xnew) - np.sum(np.dot(self.woodbury_inv, Kx) * Kx, 0)
            return mu, self._floor(var)[:, None]
        self._check_fresh()
        mu, var = self._engine.predict(self._engine_X(kern, Xnew), full_cov=full_cov)
        return mu, (var if full_cov else self._floor(var))


def _kernel_parts(kern):
    """the part descriptors of a kernel the device evaluates, its state key and its leaves; None for anything else"""
    fl = flatten_parts(kern)
    if fl is None:
        return None
    if single_kernel(kern):
        kind, ard, var, ls = kern._theta()
        return [(kind, ard, 0, list(range(kern.input_dim)), var, ls)], kern._state_key(), fl
    return [part_descriptor(leaf, term) for (leaf, term) in fl], composite_state_key(kern), fl


class Laplace(object):
    """Drop-in for GPy's Laplace (laplace.py:24-353): `inference(kern, X, likelihood, Y, ...)` returns
    (posterior, log_marginal, {'dL_dK', 'dL_dthetaL'}) with the N^2 / N^3 work on the device. Every evaluation starts the
    mode search from Ki_f = 0 (:138). dL_dK is a DeviceGradient handle carrying the reduced kernel gradient."""

    def __init__(self, device=0, engine=None):
        self._mode_finding_tolerance = 1e-4
        self._mode_finding_max_iter = 30
        self.bad_fhat = False
        self.first_run = True
        self._previous_Ki_fhat = None
        self.device = device
        self._engine = engine
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

    def inference(self, kern, X, likelihood, Y, mean_function=None, Y_metadata=None):
        assert mean_function is None, "inference with a mean function not implemented"   # :126
        desc = _kernel_parts(kern)
        if desc is None:
            raise ValueError("gpy_b200.Laplace: the kernel is not one the device evaluates (a sum of products of "
                             "stationary, StdPeriodic, White and Bias kernels)")
        parts, key, leaves = desc
        # a single kernel's part runs on its sliced columns 0 .. input_dim - 1, a composite's parts index X's columns
        single = single_kernel(kern)
        Xs = kern._slice_X(X) if single else np.asarray(X)
        return self.device_inference(Xs, Y, likelihood, Y_metadata, parts, key, [part_ngrad(l) for l, _ in leaves],
                                     single)

    def device_inference(self, Xs, Y, likelihood, Y_metadata, parts, key, ngrads, single):
        """one evaluation for the kernel described by parts (Engine.laplace_begin's descriptors on the columns of Xs),
        keyed `key`, whose leaves have ngrads gradient entries each; single: one stationary kernel (its DeviceGradient
        carries variance and lengthscale, else one block per leaf)"""
        Xs = np.ascontiguousarray(Xs, dtype=np.float64)
        Y = np.ascontiguousarray(Y, dtype=np.float64)
        if Y.ndim != 2 or Y.shape[1] != 1:
            raise ValueError("gpy_b200.Laplace takes one output column")
        eng = self.engine
        if not self._data_key.matches(Xs, Y):
            eng.set_data(Xs, Y)
            self._data_key.remember(Xs, Y)
        eng.laplace_begin(parts)
        self.first_run = False
        Ki_f_init = np.zeros_like(Y)                                                          # :138
        f_hat, Ki_fhat = self.rasm_mode(eng, Y, likelihood, Ki_f_init, Y_metadata=Y_metadata)
        log_marginal, dL_dK, dL_dthetaL = self.mode_computations(eng, f_hat, Ki_fhat, Y, likelihood, ngrads, single,
                                                                 key, parts, Y_metadata)
        self._previous_Ki_fhat = Ki_fhat.copy()
        post = PosteriorLaplace(eng, Y.shape[0], 1, key)
        return post, log_marginal, {"dL_dK": dL_dK, "dL_dthetaL": dL_dthetaL}

    @staticmethod
    def _clip_W(W, log_concave):
        """_compute_B_statistics' clip for a likelihood that is not log-concave (:319-321), and its NaN check (:327)"""
        if not log_concave:
            W = np.clip(W, 1e-6, 1e+30)
        if np.any(np.isnan(W)):
            raise ValueError('One or more element(s) of W is NaN')
        return W

    def rasm_mode(self, eng, Y, likelihood, Ki_f_init, Y_metadata=None):
        """laplace.py:148-231 with K products on the device: f = K Ki_f by gpx_laplace_matvec, one gpx_laplace_newton per
        iteration for the direction dKi_f and K dKi_f, so that the line search's f_trial = f + s K dKi_f needs no product"""
        Ki_f = Ki_f_init.copy()
        f = eng.laplace_matvec(Ki_f)

        def obj(Ki_f, f):
            ll = -0.5 * np.sum(np.dot(Ki_f.T, f)) + np.sum(likelihood.logpdf(f, Y, Y_metadata=Y_metadata))
            if np.isnan(ll):
                return -np.inf
            return ll

        difference = np.inf
        iteration = 0
        self.brent_steps = []
        while difference > self._mode_finding_tolerance and iteration < self._mode_finding_max_iter:
            W = -likelihood.d2logpdf_df2(f, Y, Y_metadata=Y_metadata)
            if np.any(np.isnan(W)):
                raise ValueError('One or more element(s) of W is NaN')
            grad = likelihood.dlogpdf_df(f, Y, Y_metadata=Y_metadata)
            if np.any(np.isnan(grad)):
                raise ValueError('One or more element(s) of grad is NaN')
            b = W * f + grad
            dKi_f, Kd, _ = eng.laplace_newton(self._clip_W(W, likelihood.log_concave), b, Ki_f)

            def inner_obj(step_size):
                return -obj(Ki_f + step_size * dKi_f, f + step_size * Kd)

            step = optimize.brent(inner_obj, tol=1e-4, maxiter=12)
            self.brent_steps.append(step)
            Ki_f_new = Ki_f + step * dKi_f
            f_new = eng.laplace_matvec(Ki_f_new)                                              # :210
            old_obj = obj(Ki_f, f)
            new_obj = obj(Ki_f_new, f_new)
            if new_obj < old_obj:
                raise ValueError("Shouldn't happen, brent optimization failing")
            difference = np.abs(new_obj - old_obj)
            Ki_f = Ki_f_new
            f = f_new
            iteration += 1
        self.iterations = iteration
        if difference > self._mode_finding_tolerance:
            if not self.bad_fhat:
                warnings.warn("Not perfect mode found (f_hat). difference: {}, iteration: {} out of max {}".format(
                    difference, iteration, self._mode_finding_max_iter))
            self.bad_fhat = True
        elif self.bad_fhat:
            self.bad_fhat = False
            warnings.warn("f_hat now fine again. difference: {}, iteration: {} out of max {}".format(
                difference, iteration, self._mode_finding_max_iter))
        return f, Ki_f

    def mode_computations(self, eng, f_hat, Ki_f, Y, likelihood, ngrads, single, key, parts, Y_metadata):
        """laplace.py:233-306 around gpx_laplace_finish"""
        W = -likelihood.d2logpdf_df2(f_hat, Y, Y_metadata=Y_metadata)
        if np.any(np.isnan(W)):
            raise ValueError('One or more element(s) of W is NaN')
        Wc = self._clip_W(W, likelihood.log_concave)
        dW_df = -likelihood.d3logpdf_df3(f_hat, Y, Y_metadata=Y_metadata)
        if np.any(np.isnan(dW_df)):
            raise ValueError('One or more element(s) of dW_df is NaN')
        lik_grads = likelihood.size > 0 and not getattr(likelihood, "is_fixed", False)
        if lik_grads:
            dlik_dthetaL, dlik_grad_dthetaL, dlik_hess_dthetaL = likelihood._laplace_gradients(f_hat, Y,
                                                                                               Y_metadata=Y_metadata)
        logdet, diag_Ki_W_i, kgrad, imp, _ = eng.laplace_finish(
            Wc, Ki_f, dW_df, dlik_grad_dthetaL.reshape(likelihood.size, -1) if lik_grads else None)
        log_marginal = (-0.5 * np.sum(np.dot(Ki_f.T, f_hat)) + np.sum(likelihood.logpdf(f_hat, Y, Y_metadata=Y_metadata))
                        - 0.5 * logdet)
        N = Y.shape[0]
        part_grads, i = [], 0
        for n in ngrads:
            part_grads.append(kgrad[i:i + n])
            i += n
        if single:
            dL_dK = DeviceGradient(eng, key, kgrad[0], kgrad[1:] if parts[0][1] else kgrad[1], N)
        else:
            dL_dK = DeviceGradient(eng, key, None, None, N, part_grads=part_grads)
        if lik_grads:
            dL_dthetaL = np.zeros(likelihood.size)
            for t in range(likelihood.size):
                exp_t = (np.sum(dlik_dthetaL[t, :, :])
                         + 0.5 * np.sum(diag_Ki_W_i * np.squeeze(dlik_hess_dthetaL[t, :, :])))
                dL_dthetaL[t] = np.sum(exp_t + imp[t])
        else:
            dL_dthetaL = np.zeros(likelihood.size)
        self.W = W                                                                              # :302-305
        self.f_hat = f_hat
        self.Ki_W_i_diag = diag_Ki_W_i
        return log_marginal, dL_dK, dL_dthetaL
