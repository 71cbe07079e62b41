"""ctypes binding of libgpx.so (C ABI: include/gpx.h). The CUDA library is the product: if it is missing or
cannot be loaded this module raises — there is NO CPU fallback anywhere in gpy_b200."""
import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libgpx.so")

KIND = {"rbf": 0, "exponential": 1, "matern32": 2, "matern52": 3, "white": 4, "bias": 5, "ratquad": 6, "stdperiodic": 7}
GET = {"L": 0, "alpha": 1, "Kinv": 2, "dL_dK": 3, "K": 4, "Linv": 5}

_dp = ctypes.POINTER(ctypes.c_double)
_vp = ctypes.c_void_p


class GpxStats(ctypes.Structure):
    _fields_ = [("total_ms", ctypes.c_float), ("kbuild_ms", ctypes.c_float), ("sweep_ms", ctypes.c_float),
                ("update_ms", ctypes.c_float), ("lauum_ms", ctypes.c_float), ("solve_ms", ctypes.c_float),
                ("update_flops", ctypes.c_double), ("lauum_flops", ctypes.c_double), ("kbuild_bytes", ctypes.c_double),
                ("launches", ctypes.c_int64), ("update_launches", ctypes.c_int32), ("tries", ctypes.c_int32),
                ("update_int8_ops", ctypes.c_double)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class GpxKernPart(ctypes.Structure):
    """gpx_kern_part of include/gpx.h: one factor of a composite kernel."""
    _fields_ = [("kind", ctypes.c_int), ("ard", ctypes.c_int), ("term", ctypes.c_int), ("ndims", ctypes.c_int),
                ("dims", ctypes.POINTER(ctypes.c_int)), ("variance", ctypes.c_double), ("lengthscale", _dp),
                ("power", ctypes.c_double), ("ard_period", ctypes.c_int), ("period", _dp)]


def _fill_part(slot, desc, keep, i=0):
    """one part descriptor (kind, ARD, term, dims, variance, lengthscale[, extra]) -> the gpx_kern_part `slot`; the arrays it
    points at are appended to `keep`. extra: {"power": a} (RatQuad) or {"period": T, "ARD_period": bool} (StdPeriodic).
    -> number of gradient entries of the part."""
    kind, ard, term, dims, variance, lengthscale = desc[:6]
    extra = desc[6] if len(desc) > 6 else {}
    static = kind in ("white", "bias")
    d = np.ascontiguousarray([] if static else dims, dtype=np.int32)
    ls = np.ascontiguousarray([1.0] if static else np.atleast_1d(lengthscale), dtype=np.float64).reshape(-1)
    if not static and ls.size != (d.size if ard else 1):
        raise ValueError("part %d: lengthscale does not match its active dims" % i)
    keep += [d, ls]
    slot.kind, slot.ard, slot.term, slot.ndims = KIND[kind], int(bool(ard)), int(term), int(d.size)
    slot.dims = d.ctypes.data_as(ctypes.POINTER(ctypes.c_int))
    slot.variance, slot.lengthscale = float(variance), _ptr(ls)
    n = 1 + (0 if static else ls.size)
    if kind == "ratquad":
        slot.power = float(extra["power"])
        n += 1
    elif kind == "stdperiodic":
        ard_p = bool(extra.get("ARD_period", False))
        T = np.ascontiguousarray(np.atleast_1d(extra["period"]), dtype=np.float64).reshape(-1)
        if T.size != (d.size if ard_p else 1):
            raise ValueError("part %d: period does not match its active dims" % i)
        keep.append(T)
        slot.ard_period, slot.period = int(ard_p), _ptr(T)
        n += T.size
    return n


EXPORTS = {
    # name: (restype, argtypes)
    "gpx_last_error": (ctypes.c_char_p, []),
    "gpx_version": (ctypes.c_char_p, []),
    "gpx_device_count": (ctypes.c_int, []),
    "gpx_create": (ctypes.c_int, [ctypes.c_int, ctypes.POINTER(_vp)]),
    "gpx_destroy": (ctypes.c_int, [_vp]),
    "gpx_set_data": (ctypes.c_int, [_vp, _dp, ctypes.c_int64, ctypes.c_int, _dp, ctypes.c_int]),
    "gpx_exact_eval": (ctypes.c_int, [_vp, ctypes.c_int, ctypes.c_int, ctypes.c_double, _dp, ctypes.c_double,
                                      ctypes.c_double, ctypes.c_int, _dp, _dp, _dp]),
    "gpx_exact_eval_het": (ctypes.c_int, [_vp, ctypes.c_int, ctypes.c_int, ctypes.c_double, _dp, _dp, ctypes.c_double,
                                          ctypes.c_int, _dp, _dp, _dp, _dp]),
    "gpx_exact_eval_multi": (ctypes.c_int, [_vp, ctypes.POINTER(GpxKernPart), ctypes.c_int, ctypes.c_double, ctypes.c_double,
                                            ctypes.c_int, _dp, _dp, _dp]),
    "gpx_get": (ctypes.c_int, [_vp, ctypes.c_int, _dp]),
    "gpx_predict": (ctypes.c_int, [_vp, _dp, ctypes.c_int64, ctypes.c_int, _dp, _dp]),
    "gpx_predictive_gradients": (ctypes.c_int, [_vp, _dp, ctypes.c_int64, _dp, _dp]),
    "gpx_exact_grad_X": (ctypes.c_int, [_vp, _dp]),
    "gpx_sparse_grad_X": (ctypes.c_int, [_vp, _dp]),
    "gpx_sparse_predictive_gradients": (ctypes.c_int, [_vp, _dp, ctypes.c_int64, _dp, _dp]),
    "gpx_posterior_covariance": (ctypes.c_int, [_vp, _dp, ctypes.c_int64, _dp, ctypes.c_int64, _dp]),
    "gpx_posterior_samples": (ctypes.c_int, [_vp, _dp, ctypes.c_int64, _dp, ctypes.c_int64, ctypes.c_int, _dp, _dp]),
    "gpx_sparse_posterior_samples": (ctypes.c_int, [_vp, _dp, ctypes.c_int64, _dp, ctypes.c_int64, ctypes.c_int, _dp,
                                                    _dp]),
    "gpx_kern_K": (ctypes.c_int, [_vp, ctypes.c_int, ctypes.c_int, ctypes.c_double, _dp, _dp, ctypes.c_int64, _dp,
                                  ctypes.c_int64, ctypes.c_int, _dp]),
    "gpx_kern_Kdiag": (ctypes.c_int, [ctypes.c_int, ctypes.c_double, ctypes.c_int64, _dp]),
    "gpx_kern_part_K": (ctypes.c_int, [_vp, ctypes.POINTER(GpxKernPart), _dp, ctypes.c_int64, _dp, ctypes.c_int64,
                                       ctypes.c_int, _dp]),
    "gpx_kern_part_grad_full": (ctypes.c_int, [_vp, ctypes.POINTER(GpxKernPart), _dp, ctypes.c_int64, _dp, ctypes.c_int64,
                                               ctypes.c_int, _dp, _dp]),
    "gpx_kern_grad_full": (ctypes.c_int, [_vp, ctypes.c_int, ctypes.c_int, ctypes.c_double, _dp, _dp, ctypes.c_int64,
                                          _dp, ctypes.c_int64, ctypes.c_int, _dp, _dp, _dp]),
    "gpx_kern_grad_X": (ctypes.c_int, [_vp, ctypes.c_int, ctypes.c_int, ctypes.c_double, _dp, _dp, ctypes.c_int64, _dp,
                                       ctypes.c_int64, ctypes.c_int, _dp, _dp]),
    "gpx_sparse_set_data": (ctypes.c_int, [_vp, _dp, ctypes.c_int64, ctypes.c_int, _dp, ctypes.c_int]),
    "gpx_sparse_eval": (ctypes.c_int, [_vp, ctypes.c_int, ctypes.c_int, ctypes.c_double, _dp, _dp, ctypes.c_int64,
                                       ctypes.c_double, _dp, _dp, _dp]),
    "gpx_sparse_get": (ctypes.c_int, [_vp, ctypes.c_int, _dp]),
    "gpx_sparse_predict": (ctypes.c_int, [_vp, _dp, ctypes.c_int64, ctypes.c_int, _dp, _dp]),
    "gpx_sparse_eval_multi": (ctypes.c_int, [_vp, ctypes.POINTER(GpxKernPart), ctypes.c_int, _dp, ctypes.c_int64,
                                             ctypes.c_double, _dp, _dp, _dp, _dp, _dp]),
    "gpx_sparse_eval_het": (ctypes.c_int, [_vp, ctypes.c_int, ctypes.c_int, ctypes.c_double, _dp, _dp, ctypes.c_int64,
                                           _dp, _dp, _dp, _dp, _dp]),
    "gpx_sparse_eval_fitc": (ctypes.c_int, [_vp, ctypes.POINTER(GpxKernPart), ctypes.c_int, _dp, ctypes.c_int64,
                                            ctypes.c_double, _dp, _dp, _dp, _dp]),
    "gpx_psi_stats": (ctypes.c_int, [_vp, ctypes.POINTER(GpxKernPart), _dp, _dp, ctypes.c_int64, _dp, ctypes.c_int64,
                                     ctypes.c_int, _dp, _dp]),
    "gpx_psi_grads": (ctypes.c_int, [_vp, ctypes.POINTER(GpxKernPart), _dp, _dp, ctypes.c_int64, _dp, ctypes.c_int64,
                                     ctypes.c_int, _dp, _dp, _dp, _dp, _dp, _dp, _dp]),
    "gpx_sparse_eval_psi": (ctypes.c_int, [_vp, ctypes.POINTER(GpxKernPart), ctypes.c_int, _dp, _dp, ctypes.c_int64,
                                           ctypes.c_double, _dp, _dp, _dp, _dp, _dp]),
    "gpx_laplace_begin": (ctypes.c_int, [_vp, ctypes.POINTER(GpxKernPart), ctypes.c_int]),
    "gpx_laplace_matvec": (ctypes.c_int, [_vp, _dp, _dp]),
    "gpx_laplace_newton": (ctypes.c_int, [_vp, _dp, _dp, _dp, ctypes.c_int, _dp, _dp, _dp]),
    "gpx_laplace_finish": (ctypes.c_int, [_vp, _dp, _dp, _dp, ctypes.c_int, _dp, ctypes.c_int, _dp, _dp, _dp, _dp, _dp]),
    "gpx_ep_begin": (ctypes.c_int, [_vp, ctypes.POINTER(GpxKernPart), ctypes.c_int]),
    "gpx_ep_start": (ctypes.c_int, [_vp, _dp, _dp, ctypes.c_int, ctypes.c_int, ctypes.c_int, _dp]),
    "gpx_ep_sweep": (ctypes.c_int, [_vp, ctypes.POINTER(ctypes.c_int64), ctypes.c_double, ctypes.c_double, ctypes.c_int,
                                    ctypes.c_int, _dp, _dp, _dp, _dp, _dp, _dp, _dp, _dp]),
    "gpx_ep_finish": (ctypes.c_int, [_vp, _dp, _dp, ctypes.c_int, _dp, _dp, _dp, _dp, _dp]),
    "gpx_vargauss_begin": (ctypes.c_int, [_vp, ctypes.POINTER(GpxKernPart), ctypes.c_int, _dp, _dp, ctypes.c_int, _dp,
                                          _dp, _dp, _dp]),
    "gpx_vargauss_finish": (ctypes.c_int, [_vp, _dp, _dp, _dp, _dp, _dp]),
    "gpx_epdtc_begin": (ctypes.c_int, [_vp, ctypes.POINTER(GpxKernPart), ctypes.c_int, _dp, ctypes.c_int64]),
    "gpx_epdtc_start": (ctypes.c_int, [_vp, _dp, _dp, ctypes.c_int, ctypes.c_int, ctypes.c_int, _dp, _dp, _dp]),
    "gpx_epdtc_sweep": (ctypes.c_int, [_vp, ctypes.POINTER(ctypes.c_int64), ctypes.c_double, ctypes.c_double,
                                       ctypes.c_int, ctypes.c_int, _dp, _dp, _dp, _dp, _dp, _dp, _dp, _dp, _dp, _dp]),
    "gpx_epdtc_finish": (ctypes.c_int, [_vp, _dp, _dp, ctypes.c_int, _dp, _dp, _dp, _dp]),
    "gpx_svgp_begin": (ctypes.c_int, [_vp, ctypes.POINTER(GpxKernPart), ctypes.c_int, _dp, ctypes.c_int64, _dp, _dp,
                                      ctypes.c_int64, ctypes.c_int64, ctypes.c_int, _dp, _dp, _dp, _dp]),
    "gpx_svgp_finish": (ctypes.c_int, [_vp, _dp, _dp, _dp, _dp, _dp, _dp]),
    "gpx_pdinv": (ctypes.c_int, [_vp, _dp, ctypes.c_int64, ctypes.c_int, _dp, _dp, _dp, _dp, _dp]),
    "gpx_get_stats": (ctypes.c_int, [_vp, ctypes.POINTER(GpxStats)]),
    "gpx_total_launches": (ctypes.c_int64, [_vp]),
    "gpx_measure_fp64_peak": (ctypes.c_int, [_vp, _dp]),
    "gpx_set_option": (ctypes.c_int, [_vp, ctypes.c_char_p, ctypes.c_int64]),
    "gpx_comm_unique_id": (ctypes.c_int, [ctypes.c_char_p]),
    "gpx_comm_init": (ctypes.c_int, [_vp, ctypes.c_char_p, ctypes.c_int, ctypes.c_int]),
}

_lib = None


def lib():
    """Load libgpx.so (once). Raises RuntimeError if the CUDA extension has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError("gpy_b200: CUDA library %s not built (run `python -c 'import __graft_entry__ as g; "
                               "g.build()'` or `make -C gpy_b200/csrc`); there is no CPU fallback" % LIB_PATH)
        L = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in EXPORTS.items():
            fn = getattr(L, name)
            fn.restype, fn.argtypes = res, args
        _lib = L
    return _lib


class GpxError(RuntimeError):
    pass


class GpxArgumentError(GpxError, ValueError):
    """rc == -2: an argument outside its domain (variance / lengthscale <= 0 or NaN, bad shapes). It is a ValueError so
    that an optimizer loop counts it as a failed evaluation the way paramz does (a Logexp underflow to exactly 0 or a
    NaN iterate must not abort `optimize()`), and still a GpxError for callers that catch the library's own class."""


def _ptr(a):
    return a.ctypes.data_as(_dp) if a is not None else None


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def check(rc, what):
    """rc < 0: CUDA/argument error -> GpxError; rc > 0: not positive definite -> numpy.linalg.LinAlgError, the class
    GPy raises from jitchol (GPy/util/linalg.py:64,75)."""
    if rc == 0:
        return
    msg = lib().gpx_last_error().decode()
    if rc > 0:
        raise np.linalg.LinAlgError("not positive definite, even with jitter. (leading minor %d)" % rc)
    if rc == -2:
        raise GpxArgumentError("%s: %s" % (what, msg))
    raise GpxError("%s failed (%d): %s" % (what, rc, msg))


def _inputs(X, X2=None, dL_dK=None):
    """inputs of a stand-alone kernel call: X (N x D), X2 (M x D, or None: X itself) and, if given, dL_dK (N x M) as
    contiguous float64 arrays -> (X, N, D, X2, M, dL_dK)"""
    X = _f64(X)
    N, D = X.shape
    X2 = None if X2 is None else _f64(X2)
    M = N if X2 is None else X2.shape[0]
    if dL_dK is not None:
        dL_dK = _f64(dL_dK)
        if dL_dK.shape != (N, M):
            raise ValueError("dL_dK must be %d x %d" % (N, M))
    return X, N, D, X2, M, dL_dK


def _theta(kind, ARD, lengthscale, D):
    ls = _f64(np.atleast_1d(lengthscale)).reshape(-1)
    if ARD:
        if ls.size != D:
            raise ValueError("ARD lengthscale must have %d entries" % D)
    elif ls.size != 1:
        raise ValueError("isotropic lengthscale must be a scalar")
    return KIND[kind], int(bool(ARD)), ls


class Engine(object):
    """One device context (gpx_ctx): owns the HBM-resident X, Y and the N x N factor workspace of one model."""

    def __init__(self, device=0):
        self._h = _vp()
        self._L = lib()
        check(self._L.gpx_create(int(device), ctypes.byref(self._h)), "gpx_create")
        self.N = self.D = self.P = 0
        self.sN = self.sD = self.sP = self.sM = 0   # shape of the sparse data set and of Z (sparse_set_data, sparse_eval*)
        self.device = device
        self.eval_serial = 0      # bumped by every evaluation: lazy posterior views check it before fetching

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            self._L.gpx_destroy(self._h)
            self._h = _vp()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_option(self, name, value):
        check(self._L.gpx_set_option(self._h, name.encode(), int(value)), "gpx_set_option")

    def set_data(self, X, Y):
        X, Y = _f64(X), _f64(Y)
        if X.ndim != 2 or Y.ndim != 2 or X.shape[0] != Y.shape[0]:
            raise ValueError("X must be N x D and Y N x P")
        (N, D), P = X.shape, Y.shape[1]
        self.eval_serial += 1
        check(self._L.gpx_set_data(self._h, _ptr(X), N, D, _ptr(Y), P), "gpx_set_data")
        self.N, self.D, self.P = N, D, P      # a rejected data set leaves the engine's shapes as they were

    def exact_eval(self, kind, ARD, variance, lengthscale, noise, jitter=1e-8, max_tries=5):
        """-> (log_marginal, gradient[variance, lengthscale.., noise], extra_jitter_used)"""
        k, a, ls = _theta(kind, ARD, lengthscale, self.D)
        lml = ctypes.c_double()
        jit = ctypes.c_double()
        grad = np.zeros(ls.size + 2)
        rc = self._L.gpx_exact_eval(self._h, k, a, float(variance), _ptr(ls), float(noise), float(jitter), int(max_tries),
                                    ctypes.byref(lml), _ptr(grad), ctypes.byref(jit))
        self.eval_serial += 1
        check(rc, "gpx_exact_eval")
        return lml.value, grad, jit.value

    def exact_eval_het(self, kind, ARD, variance, lengthscale, noise_variances, jitter=1e-8, max_tries=5):
        """one noise variance per data point -> (log_marginal, gradient[variance, lengthscale.., sum], dnoise (N,), jitter)"""
        k, a, ls = _theta(kind, ARD, lengthscale, self.D)
        nv = _f64(np.asarray(noise_variances).reshape(-1))
        if nv.size != self.N:
            raise ValueError("need one noise variance per data point")
        lml = ctypes.c_double()
        jit = ctypes.c_double()
        grad = np.zeros(ls.size + 2)
        dnoise = np.zeros(self.N)
        rc = self._L.gpx_exact_eval_het(self._h, k, a, float(variance), _ptr(ls), _ptr(nv), float(jitter), int(max_tries),
                                        ctypes.byref(lml), _ptr(grad), _ptr(dnoise), ctypes.byref(jit))
        self.eval_serial += 1
        check(rc, "gpx_exact_eval_het")
        return lml.value, grad, dnoise, jit.value

    def exact_eval_multi(self, parts, noise, jitter=1e-8, max_tries=5):
        """composite kernel: parts = [(kind, ARD, term, dims, variance, lengthscale)], ordered by term; a "ratquad" part
        appends {"power": a}, a "stdperiodic" part {"period": T, "ARD_period": bool} (ARD then refers to its lengthscale) ->
        (log_marginal, gradient [per part: variance, lengthscale.. (none for white / bias), power (ratquad); stdperiodic:
        variance, period.., lengthscale..; then noise], extra_jitter)"""
        arr = (GpxKernPart * len(parts))()
        keep, ngrad = [], 1
        for i, desc in enumerate(parts):
            ngrad += _fill_part(arr[i], desc, keep, i)
        lml, jit = ctypes.c_double(), ctypes.c_double()
        grad = np.zeros(ngrad)
        rc = self._L.gpx_exact_eval_multi(self._h, arr, len(parts), float(noise), float(jitter), int(max_tries),
                                          ctypes.byref(lml), _ptr(grad), ctypes.byref(jit))
        self.eval_serial += 1
        check(rc, "gpx_exact_eval_multi")
        return lml.value, grad, jit.value

    def get(self, which):
        if which == "alpha":
            out = np.empty((self.N, self.P))
        else:
            out = np.empty((self.N, self.N), order="F")
        check(self._L.gpx_get(self._h, GET[which], _ptr(out)), "gpx_get")
        return out

    def predict(self, Xnew, full_cov=False):
        Xnew = _f64(Xnew)
        M = Xnew.shape[0]
        mu = np.empty((M, self.P))
        var = np.empty((M, M), order="F") if full_cov else np.empty(M)
        check(self._L.gpx_predict(self._h, _ptr(Xnew), M, int(full_cov), _ptr(mu), _ptr(var)), "gpx_predict")
        return mu, (var if full_cov else var[:, None])

    def _pred_grads(self, fn, name, Xnew, D, P):
        Xnew = _f64(Xnew)
        if Xnew.ndim != 2 or (D and Xnew.shape[1] != D):   # D == 0: no data yet, the entry rejects the call (-2)
            raise ValueError("Xnew must be M x %d" % D)
        M = Xnew.shape[0]
        dmu, dvar = np.empty((M, D, P)), np.empty((M, D))
        check(fn(self._h, _ptr(Xnew), M, _ptr(dmu), _ptr(dvar)), name)
        return dmu, dvar

    def predictive_gradients(self, Xnew):
        """GP.predictive_gradients (gp.py:418-474) with the last exact evaluation -> (dmu (M, D, P), dvar (M, D))"""
        return self._pred_grads(self._L.gpx_predictive_gradients, "gpx_predictive_gradients", Xnew, self.D, self.P)

    def exact_grad_X(self):
        """kern.gradients_X(dL_dK, X, None) of the last exact evaluation (gplvm.py:47-49) at the data it holds -> (N, D)"""
        dX = np.empty((self.N, self.D))
        check(self._L.gpx_exact_grad_X(self._h, _ptr(dX)), "gpx_exact_grad_X")
        return dX

    def sparse_predictive_gradients(self, Xnew):
        """the same with the last sparse evaluation (predictive variable Z) -> (dmu (M, D, P), dvar (M, D))"""
        return self._pred_grads(self._L.gpx_sparse_predictive_gradients, "gpx_sparse_predictive_gradients", Xnew,
                                self.sD, self.sP)

    def posterior_covariance(self, X1, X2=None):
        """Posterior.covariance_between_points (posterior.py:109-130) with the last exact evaluation -> (M1, M2)
        K(X1, X2) - K(X1, X) Ky^-1 K(X, X2); X2 None: X2 = X1, exactly symmetric with zero distance on the diagonal"""
        X1 = _f64(X1)
        X2 = None if X2 is None else _f64(X2)
        for A in (X1,) if X2 is None else (X1, X2):
            if A.ndim != 2 or (self.D and A.shape[1] != self.D):
                raise ValueError("test points must be M x %d" % self.D)
        M1 = X1.shape[0]
        M2 = M1 if X2 is None else X2.shape[0]
        cov = np.empty((M1, M2))
        check(self._L.gpx_posterior_covariance(self._h, _ptr(X1), M1, _ptr(X2), M2 if X2 is not None else 0, _ptr(cov)),
              "gpx_posterior_covariance")
        return cov

    def _samples(self, fn, name, Xnew, z, max_tries, D, P):
        Xnew, z = _f64(Xnew), _f64(z)
        if Xnew.ndim != 2 or (D and Xnew.shape[1] != D):
            raise ValueError("Xnew must be M x %d" % D)
        M = Xnew.shape[0]
        if z.ndim != 2 or z.shape[1] != M:
            raise ValueError("z must be nz x %d (P S standard-normal vectors, output-major)" % M)
        nz = z.shape[0]
        f = np.empty((nz, M))
        jit = ctypes.c_double()
        check(fn(self._h, _ptr(Xnew), M, _ptr(z), nz, int(max_tries), _ptr(f), ctypes.byref(jit)), name)
        return f, jit.value

    def posterior_samples(self, Xnew, z, max_tries=5):
        """joint samples of the latent function at Xnew from the last exact evaluation: z (P S, M) standard normals,
        output-major -> (f (P S, M) in z's layout, f_j = mu[:, j // S] + chol(Sigma + jitter I) z_j, jitter used)"""
        return self._samples(self._L.gpx_posterior_samples, "gpx_posterior_samples", Xnew, z, max_tries, self.D, self.P)

    def sparse_posterior_samples(self, Xnew, z, max_tries=5):
        """the same with the last sparse evaluation (predictive variable Z)"""
        return self._samples(self._L.gpx_sparse_posterior_samples, "gpx_sparse_posterior_samples", Xnew, z, max_tries,
                             self.sD, self.sP)

    def kern_K_device_only(self, kind, ARD, variance, lengthscale, X, X2=None):
        """build K(X, X2) on the device without bringing it back; -> (kernel ms, algorithmic GB/s)."""
        X, N, D, X2, M, _ = _inputs(X, X2)
        k, a, ls = _theta(kind, ARD, lengthscale, D)
        check(self._L.gpx_kern_K(self._h, k, a, float(variance), _ptr(ls), _ptr(X), N, _ptr(X2), M, D, None), "gpx_kern_K")
        st = self.stats()
        return st["kbuild_ms"], st["kbuild_bytes"] / st["kbuild_ms"] * 1e-6

    # ---- sparse GP regression (VarDTC) building blocks ---------------------------------------------------------
    def sparse_set_data(self, X, Y):
        X, Y = _f64(X), _f64(Y)
        (N, D), P = X.shape, Y.shape[1]
        check(self._L.gpx_sparse_set_data(self._h, _ptr(X), N, D, _ptr(Y), P), "gpx_sparse_set_data")
        self.sN, self.sD, self.sP = N, D, P   # a rejected data set leaves the engine's shapes as they were

    def sparse_grad_X(self):
        """kern.gradients_X(dL_dKnm, X, Z) of the last VarDTC evaluation (sparse_gplvm.py:34) at the data it holds -> (N, D)"""
        dX = np.empty((self.sN, self.sD))
        check(self._L.gpx_sparse_grad_X(self._h, _ptr(dX)), "gpx_sparse_grad_X")
        return dX

    def sparse_eval(self, kind, ARD, variance, lengthscale, Z, noise_variance):
        """one whole VarDTC evaluation on the device -> (lml, grad [variance, lengthscale.., noise], dZ (M x D))"""
        Z = _f64(Z)
        M = Z.shape[0]
        k, a, ls = _theta(kind, ARD, lengthscale, self.sD)
        lml = ctypes.c_double()
        grad = np.zeros(ls.size + 2)
        dZ = np.empty((M, self.sD))
        check(self._L.gpx_sparse_eval(self._h, k, a, float(variance), _ptr(ls), _ptr(Z), M, float(noise_variance),
                                      ctypes.byref(lml), _ptr(grad), _ptr(dZ)), "gpx_sparse_eval")
        self.sM, self._snl = M, ls.size
        self.sparse_serial = getattr(self, "sparse_serial", 0) + 1
        return lml.value, grad, dZ

    def sparse_eval_het(self, kind, ARD, variance, lengthscale, Z, noise_variances):
        """VarDTC with one noise variance per data point (var_dtc.py het_noise branches) ->
        (lml, grad [variance, lengthscale..], dZ (M x D), dL_dR (N x P))"""
        Z = _f64(Z)
        M = Z.shape[0]
        k, a, ls = _theta(kind, ARD, lengthscale, self.sD)
        nv = _f64(np.asarray(noise_variances, dtype=np.float64).reshape(-1))
        if nv.size != self.sN:
            raise ValueError("one noise variance per data point expected (%d given, N = %d)" % (nv.size, self.sN))
        lml = ctypes.c_double()
        grad = np.zeros(ls.size + 1)
        dZ = np.empty((M, self.sD))
        dR = np.empty((self.sN, self.sP))
        check(self._L.gpx_sparse_eval_het(self._h, k, a, float(variance), _ptr(ls), _ptr(Z), M, _ptr(nv),
                                          ctypes.byref(lml), _ptr(grad), _ptr(dZ), _ptr(dR)), "gpx_sparse_eval_het")
        self.sM, self._snl = M, ls.size
        self.sparse_serial = getattr(self, "sparse_serial", 0) + 1
        return lml.value, grad, dZ, dR

    def sparse_eval_multi(self, parts, Z, noise):
        """VarDTC with a composite kernel (parts as exact_eval_multi takes them; RBF .. Matern52, White, Bias). noise: a
        scalar variance -> (lml, grad [every part's block, noise], dZ (M x D)); one variance per data point ->
        (lml, grad [every part's block], dZ, dL_dR (N x P))"""
        Z = _f64(Z)
        M = Z.shape[0]
        arr = (GpxKernPart * len(parts))()
        keep, ngrad = [], 0
        for i, desc in enumerate(parts):
            ngrad += _fill_part(arr[i], desc, keep, i)
        nv = np.asarray(noise, dtype=np.float64).reshape(-1)
        het = nv.size > 1 or np.ndim(noise) > 0
        if het and nv.size != self.sN:
            raise ValueError("one noise variance per data point expected (%d given, N = %d)" % (nv.size, self.sN))
        nv = _f64(nv)
        lml = ctypes.c_double()
        grad = np.zeros(ngrad + (0 if het else 1))
        dZ = np.empty((M, self.sD))
        dR = np.empty((self.sN, self.sP)) if het else None
        check(self._L.gpx_sparse_eval_multi(self._h, arr, len(parts), _ptr(Z), M, 0.0 if het else float(nv[0]),
                                            _ptr(nv) if het else None, ctypes.byref(lml), _ptr(grad), _ptr(dZ), _ptr(dR)),
              "gpx_sparse_eval_multi")
        self.sM = M
        self.sparse_serial = getattr(self, "sparse_serial", 0) + 1
        return (lml.value, grad, dZ, dR) if het else (lml.value, grad, dZ)

    def sparse_eval_psi(self, rbf, S, Z, noise):
        """VarDTC with uncertain inputs q(X) = N(X, diag(S)) (var_dtc.py:107-123, sparse_gp.py:88-107) for the X of
        sparse_set_data, the RBF part `rbf` (a part description on the columns 0 .. D-1) and a scalar noise variance ->
        (lml without the KL term, grad [variance, lengthscale.., noise], dZ (M x D), dmu (N x D), dS (N x D))"""
        Z, S = _f64(Z), _f64(S)
        M = Z.shape[0]
        if S.shape != (self.sN, self.sD):
            raise ValueError("S must be N x D (%d x %d)" % (self.sN, self.sD))
        arr = (GpxKernPart * 1)()
        keep = []
        ngrad = _fill_part(arr[0], rbf, keep)
        lml = ctypes.c_double()
        grad = np.zeros(ngrad + 1)
        dZ = np.empty((M, self.sD))
        dmu, dS = np.empty((self.sN, self.sD)), np.empty((self.sN, self.sD))
        check(self._L.gpx_sparse_eval_psi(self._h, arr, 1, _ptr(S), _ptr(Z), M, float(noise), ctypes.byref(lml),
                                          _ptr(grad), _ptr(dZ), _ptr(dmu), _ptr(dS)), "gpx_sparse_eval_psi")
        self.sM = M
        self.sparse_serial = getattr(self, "sparse_serial", 0) + 1
        return lml.value, grad, dZ, dmu, dS

    def psi_stats(self, rbf, mu, S, Z):
        """the RBF psi-statistics (rbf_psi_comp.py:8-51) -> (psi0 (N,), psi1 (N x M), psi2 = sum_n psi2_n (M x M))"""
        mu, S, Z = _f64(mu), _f64(S), _f64(Z)
        (N, Q), M = mu.shape, Z.shape[0]
        arr = (GpxKernPart * 1)()
        keep = []
        _fill_part(arr[0], rbf, keep)
        psi1, psi2 = np.empty((N, M)), np.empty((M, M))
        check(self._L.gpx_psi_stats(self._h, arr, _ptr(mu), _ptr(S), N, _ptr(Z), M, Q, _ptr(psi1), _ptr(psi2)),
              "gpx_psi_stats")
        return np.full(N, float(rbf[4])), psi1, psi2

    def psi_grads(self, rbf, mu, S, Z, dL_dpsi0, dL_dpsi1, dL_dpsi2):
        """psiDerivativecomputations (rbf_psi_comp.py:53-73) for an (M x M) dL_dpsi2 -> (grad [variance, lengthscale..],
        dZ (M x Q), dmu (N x Q), dS (N x Q))"""
        mu, S, Z = _f64(mu), _f64(S), _f64(Z)
        (N, Q), M = mu.shape, Z.shape[0]
        d0 = _f64(np.broadcast_to(np.asarray(dL_dpsi0, dtype=np.float64).reshape(-1), (N,)))
        d1, d2 = _f64(dL_dpsi1), _f64(dL_dpsi2)
        if d1.shape != (N, M) or d2.shape != (M, M):
            raise ValueError("dL_dpsi1 must be N x M and dL_dpsi2 M x M")
        arr = (GpxKernPart * 1)()
        keep = []
        ngrad = _fill_part(arr[0], rbf, keep)
        grad, dZ, dmu, dS = np.zeros(ngrad), np.empty((M, Q)), np.empty((N, Q)), np.empty((N, Q))
        check(self._L.gpx_psi_grads(self._h, arr, _ptr(mu), _ptr(S), N, _ptr(Z), M, Q, _ptr(d0), _ptr(d1), _ptr(d2),
                                    _ptr(grad), _ptr(dZ), _ptr(dmu), _ptr(dS)), "gpx_psi_grads")
        return grad, dZ, dmu, dS

    def sparse_eval_fitc(self, parts, Z, noise):
        """one FITC evaluation (fitc.py:19-88 with the gradient wiring of sparse_gp.py:108-118) with the kernel described
        by parts (as sparse_eval_multi takes them; a single kernel is one part on all columns) and a scalar noise variance
        -> (lml, grad [every part's block, noise], dZ (M x D), dL_dKdiag (N)). A non-positive effective noise raises
        numpy.linalg.LinAlgError naming the data point."""
        Z = _f64(Z)
        M = Z.shape[0]
        arr = (GpxKernPart * len(parts))()
        keep, ngrad = [], 0
        for i, desc in enumerate(parts):
            ngrad += _fill_part(arr[i], desc, keep, i)
        lml = ctypes.c_double()
        grad = np.zeros(ngrad + 1)
        dZ = np.empty((M, self.sD))
        dR = np.empty(self.sN)
        rc = self._L.gpx_sparse_eval_fitc(self._h, arr, len(parts), _ptr(Z), M, float(noise), ctypes.byref(lml),
                                          _ptr(grad), _ptr(dZ), _ptr(dR))
        if rc > 0:
            raise np.linalg.LinAlgError(self._L.gpx_last_error().decode())
        check(rc, "gpx_sparse_eval_fitc")
        self.sM = M
        self.sparse_serial = getattr(self, "sparse_serial", 0) + 1
        return lml.value, grad, dZ, dR

    # ---- Laplace approximation (laplace.py:122-353) -----------------------------------------------------------------
    def _vec(self, v, what):
        v = _f64(np.asarray(v, dtype=np.float64).reshape(-1))
        if v.size != self.N:
            raise ValueError("%s must have one value per data point (%d given, N = %d)" % (what, v.size, self.N))
        return v

    def laplace_begin(self, parts):
        """K(X, X) of the kernel described by parts (as exact_eval_multi takes them) into the buffer kept for the Laplace
        evaluation; -> the number of kernel gradient entries"""
        arr = (GpxKernPart * len(parts))()
        keep, ngrad = [], 0
        for i, desc in enumerate(parts):
            ngrad += _fill_part(arr[i], desc, keep, i)
        self.eval_serial += 1
        check(self._L.gpx_laplace_begin(self._h, arr, len(parts)), "gpx_laplace_begin")
        self._lap_ngrad = ngrad
        return ngrad

    def laplace_matvec(self, v):
        """K v with the kept K -> (N, 1)"""
        v = self._vec(v, "v")
        out = np.empty(self.N)
        check(self._L.gpx_laplace_matvec(self._h, _ptr(v), _ptr(out)), "gpx_laplace_matvec")
        return out[:, None]

    def laplace_newton(self, W, b, Ki_f, max_tries=5):
        """one Newton direction (laplace.py:184-199) -> (dKi_f (N, 1), K dKi_f (N, 1), jitter); a B that stays not positive
        definite raises numpy.linalg.LinAlgError as jitchol does"""
        W, b, Ki_f = self._vec(W, "W"), self._vec(b, "b"), self._vec(Ki_f, "Ki_f")
        d, Kd, jit = np.empty(self.N), np.empty(self.N), ctypes.c_double()
        rc = self._L.gpx_laplace_newton(self._h, _ptr(W), _ptr(b), _ptr(Ki_f), int(max_tries), _ptr(d), _ptr(Kd),
                                        ctypes.byref(jit))
        self.eval_serial += 1
        check(rc, "gpx_laplace_newton")
        return d[:, None], Kd[:, None], jit.value

    def laplace_finish(self, W, Ki_f, dW_df, dlik_grad_dthetaL=None, max_tries=5):
        """the mode computations (laplace.py:243-306) -> (logdet_I_KW, diag(Ki_W_i) (N,), kernel gradient block,
        dL_dthetaL_imp (nlik,), jitter). dlik_grad_dthetaL: nlik x N (or None)"""
        W, Ki_f, dW_df = self._vec(W, "W"), self._vec(Ki_f, "Ki_f"), self._vec(dW_df, "dW_df")
        g = None if dlik_grad_dthetaL is None else _f64(np.asarray(dlik_grad_dthetaL, dtype=np.float64).reshape(-1, self.N))
        nlik = 0 if g is None else g.shape[0]
        logdet, jit = ctypes.c_double(), ctypes.c_double()
        diag, kgrad, imp = np.empty(self.N), np.zeros(getattr(self, "_lap_ngrad", 0)), np.zeros(nlik)
        rc = self._L.gpx_laplace_finish(self._h, _ptr(W), _ptr(Ki_f), _ptr(dW_df), nlik, _ptr(g) if nlik else None,
                                        int(max_tries), ctypes.byref(logdet), _ptr(diag), _ptr(kgrad),
                                        _ptr(imp) if nlik else None, ctypes.byref(jit))
        self.eval_serial += 1
        check(rc, "gpx_laplace_finish")
        return logdet.value, diag, kgrad, imp, jit.value

    # ---- expectation propagation (expectation_propagation.py:187-434) ----------------------------------------------
    def ep_begin(self, parts):
        """K(X, X) of the kernel described by parts (as laplace_begin) for EP with the probit Bernoulli likelihood; the
        labels of set_data must be in {-1, 0, 1}. -> the number of kernel gradient entries"""
        arr = (GpxKernPart * len(parts))()
        keep, ngrad = [], 0
        for i, desc in enumerate(parts):
            ngrad += _fill_part(arr[i], desc, keep, i)
        self.eval_serial += 1
        check(self._L.gpx_ep_begin(self._h, arr, len(parts)), "gpx_ep_begin")
        self._lap_ngrad = ngrad
        return ngrad

    def ep_start(self, tau_tilde=None, v_tilde=None, parallel=False, max_tries=5):
        """_init_approximations (:312-328): cold without sites, warm (the recompute from them) with -> jitter"""
        warm = tau_tilde is not None
        t = self._vec(tau_tilde, "tau_tilde") if warm else None
        v = self._vec(v_tilde, "v_tilde") if warm else None
        jit = ctypes.c_double()
        rc = self._L.gpx_ep_start(self._h, _ptr(t) if warm else None, _ptr(v) if warm else None, int(warm),
                                  int(bool(parallel)), int(max_tries), ctypes.byref(jit))
        self.eval_serial += 1
        check(rc, "gpx_ep_start")
        return jit.value

    def ep_sweep(self, order, tau_tilde, v_tilde, eta=1., delta=1., parallel=False, max_tries=5):
        """one sweep of the sites in the given order, then the recompute -> (tau_tilde, v_tilde, cav_tau, cav_v, Z_hat,
        mu_hat, sigma2_hat, jitter), N values each but the jitter"""
        order = np.ascontiguousarray(np.asarray(order).reshape(-1), dtype=np.int64)
        if order.size != self.N:
            raise ValueError("order must hold N = %d entries (%d given)" % (self.N, order.size))
        t, v = self._vec(tau_tilde, "tau_tilde").copy(), self._vec(v_tilde, "v_tilde").copy()
        outs = [np.empty(self.N) for _ in range(5)]
        jit = ctypes.c_double()
        rc = self._L.gpx_ep_sweep(self._h, order.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)), float(eta), float(delta),
                                  int(bool(parallel)), int(max_tries), _ptr(t), _ptr(v), *[_ptr(o) for o in outs],
                                  ctypes.byref(jit))
        self.eval_serial += 1
        check(rc, "gpx_ep_sweep")
        return (t, v, *outs, jit.value)

    def ep_finish(self, tau_tilde, v_tilde, max_tries=5):
        """_ep_marginal + _inference (:363-395) -> (logdet_B, v~^T Sigma v~, diag(dL_dK) (N,), kernel gradient block,
        jitter); the posterior stays for get / predict"""
        t, v = self._vec(tau_tilde, "tau_tilde"), self._vec(v_tilde, "v_tilde")
        logdet, vsv, jit = ctypes.c_double(), ctypes.c_double(), ctypes.c_double()
        diag, kgrad = np.empty(self.N), np.zeros(getattr(self, "_lap_ngrad", 0))
        rc = self._L.gpx_ep_finish(self._h, _ptr(t), _ptr(v), int(max_tries), ctypes.byref(logdet), ctypes.byref(vsv),
                                   _ptr(diag), _ptr(kgrad), ctypes.byref(jit))
        self.eval_serial += 1
        check(rc, "gpx_ep_finish")
        return logdet.value, vsv.value, diag, kgrad, jit.value

    # ---- variational Gaussian approximation (var_gauss.py:34-69) -----------------------------------------------------
    def vargauss_begin(self, parts, alpha, beta, max_tries=5):
        """K of the kernel described by parts (as laplace_begin takes them) kept on the device, m = K alpha and the
        factor of A = I + B K B, B = diag(beta) -> (m (N,), var = diag(Sigma) (N,), KL, jitter). A beta entry that is zero
        or not finite raises GpxArgumentError; an A that stays not positive definite numpy.linalg.LinAlgError"""
        a, b = self._vec(alpha, "alpha"), self._vec(beta, "beta")
        arr = (GpxKernPart * len(parts))()
        keep, ngrad = [], 0
        for i, desc in enumerate(parts):
            ngrad += _fill_part(arr[i], desc, keep, i)
        m, var = np.empty(self.N), np.empty(self.N)
        kl, jit = ctypes.c_double(), ctypes.c_double()
        rc = self._L.gpx_vargauss_begin(self._h, arr, len(parts), _ptr(a), _ptr(b), int(max_tries), _ptr(m), _ptr(var),
                                        ctypes.byref(kl), ctypes.byref(jit))
        self.eval_serial += 1
        check(rc, "gpx_vargauss_begin")
        self._lap_ngrad = ngrad
        return m, var, kl.value, jit.value

    def vargauss_finish(self, dF_dm, dF_dv):
        """the gradients of F.sum() - KL for the likelihood's dF_dm and dF_dv at the last vargauss_begin's (m, var) ->
        (dalpha (N,), dbeta (N,), kernel gradient block); the posterior stays for get / predict"""
        g, dv = self._vec(dF_dm, "dF_dm"), self._vec(dF_dv, "dF_dv")
        da, db, kgrad = np.empty(self.N), np.empty(self.N), np.zeros(getattr(self, "_lap_ngrad", 0))
        rc = self._L.gpx_vargauss_finish(self._h, _ptr(g), _ptr(dv), _ptr(da), _ptr(db), _ptr(kgrad))
        self.eval_serial += 1
        check(rc, "gpx_vargauss_finish")
        return da, db, kgrad

    # ---- sparse expectation propagation (EPDTC, expectation_propagation.py:436-611) -----------------------------------
    def _svec(self, v, what):
        v = _f64(np.asarray(v, dtype=np.float64).reshape(-1))
        if v.size != self.sN:
            raise ValueError("%s must have one value per data point (%d given, N = %d)" % (what, v.size, self.sN))
        return v

    def epdtc_begin(self, parts, Z):
        """Kmm, Kmn and jitchol(Kmm) of the kernel described by parts (as sparse_eval_multi takes them) at the inducing
        inputs Z, for sparse EP with the probit Bernoulli likelihood on the data of sparse_set_data (labels in {-1, 0, 1})
        -> the number of kernel gradient entries"""
        Z = _f64(Z)
        M = Z.shape[0]
        arr = (GpxKernPart * len(parts))()
        keep, ngrad = [], 0
        for i, desc in enumerate(parts):
            ngrad += _fill_part(arr[i], desc, keep, i)
        rc = self._L.gpx_epdtc_begin(self._h, arr, len(parts), _ptr(Z), M)
        if rc > 0:
            raise np.linalg.LinAlgError(self._L.gpx_last_error().decode())
        check(rc, "gpx_epdtc_begin")
        self.sM = M
        self._epdtc_ngrad = ngrad
        return ngrad

    def epdtc_start(self, tau_tilde=None, v_tilde=None, parallel=False, max_tries=5):
        """_init_approximations (:522-551): cold without sites, warm (the recompute from them) with ->
        (jitter, mu, Sigma_diag)"""
        warm = tau_tilde is not None
        t = self._svec(tau_tilde, "tau_tilde") if warm else None
        v = self._svec(v_tilde, "v_tilde") if warm else None
        jit, mu, sd = ctypes.c_double(), np.empty(self.sN), np.empty(self.sN)
        rc = self._L.gpx_epdtc_start(self._h, _ptr(t) if warm else None, _ptr(v) if warm else None, int(warm),
                                     int(bool(parallel)), int(max_tries), ctypes.byref(jit), _ptr(mu), _ptr(sd))
        if rc > 0:
            raise np.linalg.LinAlgError(self._L.gpx_last_error().decode())
        check(rc, "gpx_epdtc_start")
        return jit.value, mu, sd

    def epdtc_sweep(self, order, tau_tilde, v_tilde, eta=1., delta=1., parallel=False, max_tries=5):
        """one sweep of the sites in the given order, then the recompute -> (tau_tilde, v_tilde, cav_tau, cav_v, Z_hat,
        mu_hat, sigma2_hat, jitter, mu, Sigma_diag)"""
        order = np.ascontiguousarray(np.asarray(order).reshape(-1), dtype=np.int64)
        if order.size != self.sN:
            raise ValueError("order must hold N = %d entries (%d given)" % (self.sN, order.size))
        t, v = self._svec(tau_tilde, "tau_tilde").copy(), self._svec(v_tilde, "v_tilde").copy()
        outs = [np.empty(self.sN) for _ in range(5)]
        mu, sd = np.empty(self.sN), np.empty(self.sN)
        jit = ctypes.c_double()
        rc = self._L.gpx_epdtc_sweep(self._h, order.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)), float(eta),
                                     float(delta), int(bool(parallel)), int(max_tries), _ptr(t), _ptr(v),
                                     *[_ptr(o) for o in outs], ctypes.byref(jit), _ptr(mu), _ptr(sd))
        if rc > 0:
            raise np.linalg.LinAlgError(self._L.gpx_last_error().decode())
        check(rc, "gpx_epdtc_sweep")
        return (t, v, *outs, jit.value, mu, sd)

    def epdtc_finish(self, tau_tilde, v_tilde, max_tries=5):
        """VarDTC at Y = v~ / tau~ and precision tau~ (:474-482) without log Z~ -> (lml, kernel gradient block,
        dZ (M x D), jitter); the posterior stays for sparse_get / sparse_predict"""
        t, v = self._svec(tau_tilde, "tau_tilde"), self._svec(v_tilde, "v_tilde")
        lml, jit = ctypes.c_double(), ctypes.c_double()
        grad, dZ = np.zeros(getattr(self, "_epdtc_ngrad", 0)), np.empty((self.sM, self.sD))
        rc = self._L.gpx_epdtc_finish(self._h, _ptr(t), _ptr(v), int(max_tries), ctypes.byref(lml), _ptr(grad), _ptr(dZ),
                                      ctypes.byref(jit))
        if rc > 0:
            raise np.linalg.LinAlgError(self._L.gpx_last_error().decode())
        check(rc, "gpx_epdtc_finish")
        self.sparse_serial = getattr(self, "sparse_serial", 0) + 1
        return lml.value, grad, dZ, jit.value

    # ---- stochastic variational sparse GP (SVGP, svgp.py:10-118) -------------------------------------------------------
    def svgp_begin(self, parts, Z, q_m, q_L, row0, nb, max_tries=5):
        """the marginals of q(f) on the rows [row0, row0 + nb) of the data of sparse_set_data (P = 1) for the kernel
        described by parts (as sparse_eval_multi takes them), inducing inputs Z, q(u) = N(q_m, q_L q_L^T) (q_L: M x M lower
        triangular) -> (mu (nb,), v (nb,), KL, jitter)"""
        Z = _f64(Z)
        M = Z.shape[0]
        m = _f64(np.asarray(q_m, dtype=np.float64).reshape(-1))
        L = _f64(q_L)
        if m.size != M or L.shape != (M, M):
            raise ValueError("q_m must hold M = %d values and q_L be M x M" % M)
        arr = (GpxKernPart * len(parts))()
        keep, ngrad = [], 0
        for i, desc in enumerate(parts):
            ngrad += _fill_part(arr[i], desc, keep, i)
        nb = int(nb)
        mu, v = np.empty(max(nb, 0)), np.empty(max(nb, 0))
        kl, jit = ctypes.c_double(), ctypes.c_double()
        rc = self._L.gpx_svgp_begin(self._h, arr, len(parts), _ptr(Z), M, _ptr(m), _ptr(L), int(row0), nb, int(max_tries),
                                    _ptr(mu), _ptr(v), ctypes.byref(kl), ctypes.byref(jit))
        if rc > 0:
            raise np.linalg.LinAlgError(self._L.gpx_last_error().decode())
        check(rc, "gpx_svgp_begin")
        self.sM = M
        self._svgp_ngrad, self._svgp_nb = ngrad, nb
        return mu, v, kl.value, jit.value

    def svgp_finish(self, dF_dmu, dF_dv):
        """the gradients of the bound for the batch-scaled dF_dmu, dF_dv of the last svgp_begin's batch -> (kernel gradient
        block, dZ (M x D), dL_dm (M,), dL_dchol (M x M, lower triangular)); the posterior stays for sparse_get / predict"""
        nb = getattr(self, "_svgp_nb", 0)
        a = _f64(np.asarray(dF_dmu, dtype=np.float64).reshape(-1))
        b = _f64(np.asarray(dF_dv, dtype=np.float64).reshape(-1))
        if a.size != nb or b.size != nb:
            raise ValueError("dF_dmu and dF_dv must hold one value per row of the last batch (%d)" % nb)
        M = self.sM
        grad, dZ = np.zeros(getattr(self, "_svgp_ngrad", 0)), np.empty((M, self.sD))
        dm, dchol = np.empty(M), np.empty((M, M))
        check(self._L.gpx_svgp_finish(self._h, _ptr(a), _ptr(b), _ptr(grad), _ptr(dZ), _ptr(dm), _ptr(dchol)),
              "gpx_svgp_finish")
        self.sparse_serial = getattr(self, "sparse_serial", 0) + 1
        return grad, dZ, dm, dchol

    SPARSE_GET = {"woodbury_vector": 0, "woodbury_inv": 1, "Kmm": 2, "Lm": 3}

    def sparse_get(self, what):
        which = self.SPARSE_GET[what]
        out = np.empty((self.sM, self.sP)) if which == 0 else np.empty((self.sM, self.sM), order="F")
        check(self._L.gpx_sparse_get(self._h, which, _ptr(out)), "gpx_sparse_get")
        return out

    def sparse_predict(self, Xnew, full_cov=False):
        """Posterior._raw_predict (posterior.py:220-248) of the last sparse evaluation with the predictive variable Z ->
        (mu (M, P), var (M, 1), clipped at 1e-15, or the full covariance (M, M)); the diagonal streams over chunks of
        test points (gpx_sparse_predict)"""
        Xnew = _f64(Xnew)
        if Xnew.ndim != 2 or (self.sD and Xnew.shape[1] != self.sD):   # sD == 0: no data yet, the entry rejects the call
            raise ValueError("Xnew must be M x %d" % self.sD)
        M = Xnew.shape[0]
        mu = np.empty((M, self.sP))
        var = np.empty((M, M), order="F") if full_cov else np.empty(M)
        check(self._L.gpx_sparse_predict(self._h, _ptr(Xnew), M, int(bool(full_cov)), _ptr(mu), _ptr(var)),
              "gpx_sparse_predict")
        return mu, (var if full_cov else var[:, None])

    def stats(self):
        s = GpxStats()
        check(self._L.gpx_get_stats(self._h, ctypes.byref(s)), "gpx_get_stats")
        return s.as_dict()

    def measure_fp64_peak(self):
        """fp64 DMMA issue peak of this device in TFLOP/s (roofline denominator, measured live)."""
        v = ctypes.c_double()
        check(self._L.gpx_measure_fp64_peak(self._h, ctypes.byref(v)), "gpx_measure_fp64_peak")
        return v.value

    def total_launches(self):
        return int(self._L.gpx_total_launches(self._h))


def kern_K(kind, ARD, variance, lengthscale, X, X2=None):
    X, N, D, X2, M, _ = _inputs(X, X2)
    k, a, ls = _theta(kind, ARD, lengthscale, D)
    out = np.empty((N, M))
    check(lib().gpx_kern_K(None, k, a, float(variance), _ptr(ls), _ptr(X), N, _ptr(X2), M, D, _ptr(out)), "gpx_kern_K")
    return out


def kern_part_K(desc, X, X2=None):
    """K(X, X2) (N x M) of one composite part descriptor (as Engine.exact_eval_multi takes it; dims index X's columns)."""
    part, keep = GpxKernPart(), []
    _fill_part(part, desc, keep)
    X, N, D, X2, M, _ = _inputs(X, X2)
    out = np.empty((N, M))
    check(lib().gpx_kern_part_K(None, ctypes.byref(part), _ptr(X), N, _ptr(X2), M, D, _ptr(out)), "gpx_kern_part_K")
    return out


def kern_part_grad_full(desc, X, dL_dK, X2=None):
    """update_gradients_full of one composite part for a dense dL_dK (N x M) -> its gradient block."""
    part, keep = GpxKernPart(), []
    n = _fill_part(part, desc, keep)
    X, N, D, X2, M, dL_dK = _inputs(X, X2, dL_dK)
    grad = np.zeros(n)
    check(lib().gpx_kern_part_grad_full(None, ctypes.byref(part), _ptr(X), N, _ptr(X2), M, D, _ptr(dL_dK), _ptr(grad)),
          "gpx_kern_part_grad_full")
    return grad


def kern_Kdiag(kind, variance, N):
    out = np.empty(N)
    check(lib().gpx_kern_Kdiag(KIND[kind], float(variance), N, _ptr(out)), "gpx_kern_Kdiag")
    return out


def kern_grad_X(kind, ARD, variance, lengthscale, X, dL_dK, X2=None):
    """Stationary.gradients_X (stationary.py:245-252) on the device -> N x D."""
    X, N, D, X2, M, dL_dK = _inputs(X, X2, dL_dK)
    k, a, ls = _theta(kind, ARD, lengthscale, D)
    out = np.empty((N, D))
    check(lib().gpx_kern_grad_X(None, k, a, float(variance), _ptr(ls), _ptr(X), N, _ptr(X2), M, D, _ptr(dL_dK), _ptr(out)),
          "gpx_kern_grad_X")
    return out


def pdinv(A, maxtries=5, want=("Ai", "L", "Li"), engine=None):
    """GPy.util.linalg.pdinv (linalg.py:193-214) on the device: -> (Ai, L, Li, logdet) (entries not in `want` are None)
    plus the jitter the jitchol ladder (linalg.py:56-75) had to add. Raises numpy.linalg.LinAlgError like the reference."""
    A = _f64(A)
    N = A.shape[0]
    if A.ndim != 2 or A.shape[1] != N:
        raise ValueError("A must be square")
    outs = {k: (np.empty((N, N), order="F") if k in want else None) for k in ("Ai", "L", "Li")}
    logdet, jit = ctypes.c_double(), ctypes.c_double()
    h = engine._h if engine is not None else None
    rc = lib().gpx_pdinv(h, _ptr(np.ascontiguousarray(A)), N, int(maxtries), _ptr(outs["Ai"]), _ptr(outs["L"]), _ptr(outs["Li"]),
                         ctypes.byref(logdet), ctypes.byref(jit))
    if rc > 0:
        raise np.linalg.LinAlgError(lib().gpx_last_error().decode())
    check(rc, "gpx_pdinv")
    return outs["Ai"], outs["L"], outs["Li"], logdet.value, jit.value


def jitchol(A, maxtries=5, engine=None):
    """GPy.util.linalg.jitchol (linalg.py:56-75) on the device: lower Cholesky factor, jitter ladder included."""
    return pdinv(A, maxtries, want=("L",), engine=engine)[1]


def kern_grad_full(kind, ARD, variance, lengthscale, X, dL_dK, X2=None):
    X, N, D, X2, M, dL_dK = _inputs(X, X2, dL_dK)
    k, a, ls = _theta(kind, ARD, lengthscale, D)
    dv = ctypes.c_double()
    dl = np.zeros(ls.size)
    check(lib().gpx_kern_grad_full(None, k, a, float(variance), _ptr(ls), _ptr(X), N, _ptr(X2), M, D, _ptr(dL_dK),
                                   ctypes.byref(dv), _ptr(dl)), "gpx_kern_grad_full")
    return dv.value, dl


_psi_engine = None


def _scratch():
    """the context of the stand-alone psi entries outside an evaluation (created on first use, device 0)"""
    global _psi_engine
    if _psi_engine is None:
        _psi_engine = Engine()
    return _psi_engine


def psi_stats(rbf, mu, S, Z):
    """the RBF psi-statistics of an RBF part description (Engine.psi_stats) on a context of their own"""
    return _scratch().psi_stats(rbf, mu, S, Z)


def psi_grads(rbf, mu, S, Z, dL_dpsi0, dL_dpsi1, dL_dpsi2):
    """psiDerivativecomputations (Engine.psi_grads) on a context of their own"""
    return _scratch().psi_grads(rbf, mu, S, Z, dL_dpsi0, dL_dpsi1, dL_dpsi2)
