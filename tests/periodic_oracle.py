"""CPU restatement of GPy's RatQuad and StdPeriodic kernels and of exact inference with composite kernels that contain
them (test infrastructure only). Each line cites the reference file:line it restates; the stationary / static kinds and
the linear algebra are oracle/gpy_oracle.py's."""
import numpy as np

from oracle import gpy_oracle as o


class RatQuadOracle(object):
    """GPy.kern.RatQuad (stationary.py:747-802) on Stationary's scaled distance (stationary.py:151-168)."""

    def __init__(self, input_dim, variance=1.0, lengthscale=1.0, power=2.0, ARD=False):
        self.input_dim, self.ARD = input_dim, ARD
        self.variance, self.power = float(variance), float(power)
        self.lengthscale = np.asarray(lengthscale, dtype=np.float64).reshape(-1)
        assert self.lengthscale.size == (input_dim if ARD else 1)

    def _r(self, X, X2=None):
        return o.scaled_dist(X, X2, self.lengthscale, self.ARD)

    def K(self, X, X2=None):
        r2 = np.square(self._r(X, X2))
        return self.variance * np.exp(-self.power * np.log1p(r2 / 2.))                           # :785-788

    def dK_dr(self, r):
        return -self.variance * self.power * r * np.exp(-(self.power + 1) * np.log1p(np.square(r) / 2.))   # :790-793

    def Kdiag(self, X):
        return np.full(X.shape[0], self.variance)                                                # stationary.py:170-173

    def update_gradients_full(self, dL_dK, X, X2=None):
        """-> [variance, lengthscale.., power]: Stationary.update_gradients_full (stationary.py:193-213) then :795-798"""
        r = self._r(X, X2)
        dvar = np.sum(self.K(X, X2) * dL_dK) / self.variance
        dL_dr = self.dK_dr(r) * dL_dK
        if self.ARD:
            tmp = dL_dr * (1.0 / np.where(r != 0.0, r, np.inf))
            dl = o.lengthscale_grads_pure(tmp, X, X if X2 is None else X2, self.lengthscale)
        else:
            dl = np.atleast_1d(-np.sum(dL_dr * r) / self.lengthscale)
        r2 = np.square(r)
        dK_dpow = -self.variance * np.exp(self.power * (np.log(2.) - np.log1p(r2 + 1))) * np.log1p(r2 / 2.)
        return np.concatenate([[dvar], dl, [np.sum(dL_dK * dK_dpow)]])


class StdPeriodicOracle(object):
    """GPy.kern.StdPeriodic (standard_periodic.py:56-94,125-139,501-548)."""

    def __init__(self, input_dim, variance=1.0, period=1.0, lengthscale=1.0, ARD1=False, ARD2=False):
        self.input_dim, self.ARD1, self.ARD2 = input_dim, ARD1, ARD2
        self.variance = float(variance)
        self.period = np.asarray(period, dtype=np.float64).reshape(-1)
        self.lengthscale = np.asarray(lengthscale, dtype=np.float64).reshape(-1)
        assert self.period.size == (input_dim if ARD1 else 1)
        assert self.lengthscale.size == (input_dim if ARD2 else 1)

    def K(self, X, X2=None):
        if X2 is None:
            X2 = X
        base = np.pi * (X[:, None, :] - X2[None, :, :]) / self.period                             # :130
        exp_dist = np.exp(-0.5 * np.sum(np.square(np.sin(base) / self.lengthscale), axis=-1))     # :131
        return self.variance * exp_dist

    def Kdiag(self, X):
        return np.full(X.shape[0], self.variance)                                                 # :134-138

    def update_gradients_full(self, dL_dK, X, X2=None):
        """-> [variance, period.., lengthscale..] (:501-526)"""
        if X2 is None:
            X2 = X
        base = np.pi * (X[:, None, :] - X2[None, :, :]) / self.period
        sin_base = np.sin(base)
        exp_dist = np.exp(-0.5 * np.sum(np.square(sin_base / self.lengthscale), axis=-1))
        dwl = self.variance * (1.0 / np.square(self.lengthscale)) * sin_base * np.cos(base) * (base / self.period)
        dl = self.variance * np.square(sin_base) / np.power(self.lengthscale, 3)
        dvar = np.sum(exp_dist * dL_dK)
        if self.ARD1:
            dper = (dwl * exp_dist[:, :, None] * dL_dK[:, :, None]).sum(0).sum(0)
        else:
            dper = np.atleast_1d(np.sum(dwl.sum(-1) * exp_dist * dL_dK))
        if self.ARD2:
            dlen = (dl * exp_dist[:, :, None] * dL_dK[:, :, None]).sum(0).sum(0)
        else:
            dlen = np.atleast_1d(np.sum(dl.sum(-1) * exp_dist * dL_dK))
        return np.concatenate([[dvar], dper, dlen])


class _Block(object):
    """an oracle kernel of gpy_oracle with update_gradients_full returning its whole gradient block"""

    def __init__(self, k):
        self.k = k

    def K(self, X, X2=None):
        return self.k.K(X, X2)

    def Kdiag(self, X):
        return self.k.Kdiag(X)

    def update_gradients_full(self, dL_dK, X, X2=None):
        dv, dl = self.k.update_gradients_full(dL_dK, X, X2)
        return np.concatenate([[dv], np.atleast_1d(dl).reshape(-1)])


def make_part(p):
    """dict(kind, term, dims, variance, [lengthscale, ARD, power, period, ARD_period]) -> (oracle kernel, dims, term)"""
    kind, dims = p["kind"], p.get("dims")
    if kind in ("white", "bias"):
        return _Block(o.StaticOracle(kind, p["variance"])), None, p["term"]
    dims = np.asarray(dims)
    if kind == "ratquad":
        k = RatQuadOracle(len(dims), p["variance"], p["lengthscale"], p["power"], p.get("ARD", False))
    elif kind == "stdperiodic":
        k = StdPeriodicOracle(len(dims), p["variance"], p["period"], p["lengthscale"], p.get("ARD_period", False),
                              p.get("ARD", False))
    else:
        k = _Block(o.StationaryOracle(kind, len(dims), p["variance"], p["lengthscale"], p.get("ARD", False)))
    return k, dims, p["term"]


def descriptor(p):
    """the same part as Engine.exact_eval_multi takes it"""
    d = (p["kind"], p.get("ARD", False), p["term"], list(p.get("dims") or []), p["variance"], p.get("lengthscale"))
    if p["kind"] == "ratquad":
        d += ({"power": p["power"]},)
    elif p["kind"] == "stdperiodic":
        d += ({"period": p["period"], "ARD_period": p.get("ARD_period", False)},)
    return d


def composite_eval(X, Y, parts, noise_variance):
    """one GP.parameters_changed() with a composite kernel (as gpy_oracle.composite_eval_lml_grad, with these kinds too)
    -> (lml, grad [per part: its block; noise], res)"""
    X = np.ascontiguousarray(X, dtype=np.float64)
    Y = np.ascontiguousarray(Y, dtype=np.float64)
    kparts = [make_part(p) for p in parts]
    K = o.composite_K(kparts, X)
    Ky = K.copy()
    o.diag_add(Ky, noise_variance + 1e-8)                                                         # exact_gaussian_inference.py:56
    Wi, LW, _, W_logdet = o.pdinv(Ky)
    alpha, _ = o.dpotrs(LW, Y, lower=1)
    lml = 0.5 * (-Y.size * np.log(2 * np.pi) - Y.shape[1] * W_logdet - np.sum(alpha * Y))
    dL_dK = 0.5 * (o.tdot(alpha) - Y.shape[1] * Wi)
    grad = []
    for i, (k, dims, t) in enumerate(kparts):
        other = None
        for j, (k2, dims2, t2) in enumerate(kparts):
            if j != i and t2 == t:
                Kj = k2.K(o._slice(X, dims2))
                other = Kj if other is None else other * Kj
        grad.append(k.update_gradients_full(dL_dK if other is None else dL_dK * other, o._slice(X, dims), None))
    grad.append([np.trace(dL_dK)])
    return float(lml), np.concatenate(grad), dict(L=LW, alpha=alpha, K=K, Wi=Wi, dL_dK=dL_dK, kparts=kparts)


def mauna_loa_parts():
    """RBF + RBF x StdPeriodic + RatQuad + RBF + White on one time axis (Rasmussen & Williams section 5.4.3), in years"""
    return [dict(kind="rbf", term=0, dims=[0], variance=4.0, lengthscale=50.0),
            dict(kind="rbf", term=1, dims=[0], variance=2.0, lengthscale=90.0),
            dict(kind="stdperiodic", term=1, dims=[0], variance=1.0, period=1.0, lengthscale=1.3),
            dict(kind="ratquad", term=2, dims=[0], variance=0.5, lengthscale=1.2, power=0.8),
            dict(kind="rbf", term=3, dims=[0], variance=0.1, lengthscale=0.15),
            dict(kind="white", term=4, variance=0.05)]


def mauna_loa_data(N, seed=0):
    """time-like inputs X = 1958 + 67 u (years), a trend plus a yearly cycle plus noise"""
    rng = np.random.default_rng(seed)
    X = np.sort(1958.0 + 67.0 * rng.uniform(size=N))[:, None]
    t = X[:, 0]
    Y = 0.03 * (t - 1990.0) + 0.6 * np.sin(2 * np.pi * t) + 0.2 * np.cos(4 * np.pi * t) + 0.1 * rng.standard_normal(N)
    return X, Y[:, None]
