"""The reference-side binding: plugin classes that subclass GPy's OWN kernel / inference classes and route the hot
path through libgpx (see INTEGRATION.md). Use where GPy (+ paramz) is importable:

    import GPy
    from gpy_b200 import gpy_plugin
    B = gpy_plugin.load()                       # subclasses of GPy.kern.RBF/Matern32/Matern52/Exponential/RatQuad/StdPeriodic,
                                                # Add, Prod + inference
    m = GPy.models.GPRegression(X, Y, kernel=B.RBF(D, ARD=True))
    m.inference_method = B.ExactGaussianInference()      # same hook the reference's tests use (GPy/testing/fitc.py:31)
    m.optimize()                                # paramz loop unchanged; one gpx_exact_eval per iterate

`make(...)` takes the base classes explicitly so that the wiring can be exercised against the unmodified reference
modules in the build container (tests/test_gpy_plugin_cpu.py) where the full `import GPy` is impossible (no paramz).

The sparse model is a drop-in the same way — the reference's own `GPy.core.SparseGP` / `SparseGPRegression`, UNCHANGED:

    m = GPy.core.SparseGP(X, Y, Z, B.RBF(D, ARD=True), GPy.likelihoods.Gaussian(), inference_method=B.VarDTC())

`B.VarDTC.inference` makes ONE `gpx_sparse_eval` (or `gpx_sparse_eval_het`; `gpx_sparse_eval_multi` for a `B.Add` /
`B.Prod` over plugin stationary leaves and GPy's own White / Bias) and returns a grad_dict whose `dL_dKnm` / `dL_dKmm` are
handles carrying the gradients the device already reduced; `SparseGP._update_gradients` (core/sparse_gp.py:108-119) then
calls the kernel's `update_gradients_diag / update_gradients_full / gradients_X` exactly as written there and gets those
numbers back (the N x M matrix dL_dKnm never exists).
`B.FITC` (over GPy's own `FITC`) does the same with ONE `gpx_sparse_eval_fitc`, and hands back the real N-vector
`dL_dKdiag` beside the handles.

The methods `K`, `Kdiag`, `update_gradients_full`, `update_gradients_diag`, `gradients_X` are defined in the class bodies on purpose:
`KernCallsViaSlicerMeta` only wraps names it finds in the class dict (GPy/kern/src/kernel_slice_operations.py:14-57), and
the wrapper hands them X already sliced to `active_dims` (GPy/kern/src/kern.py:112-117).
"""
import types

import numpy as np

from . import _ffi
from .inference import PosteriorExact, _DataKey, _LazyAlpha
from .kern import DeviceGradient

_KINDS = {"RBF": "rbf", "Exponential": "exponential", "Matern32": "matern32", "Matern52": "matern52"}
_PART_KINDS = {"RatQuad": "ratquad", "StdPeriodic": "stdperiodic"}


class SparseDeviceGradient(object):
    """Stand-in for `grad_dict['dL_dKnm']` (N x M) / `grad_dict['dL_dKmm']` (M x M) of VarDTC.inference
    (var_dtc.py:178-188). The device evaluation has already reduced both to d/d(variance, lengthscale) and dL/dZ
    (core/sparse_gp.py:110-118); the handle carries its share, keyed by the kernel state and the inducing inputs they were
    computed for. `.T` flips `transposed` (the shape cannot tell the orientation when N = M): SparseGP passes
    `dL_dKnm.T` to `gradients_X` for dL/dZ (:118), SparseGPLVM the untransposed `dL_dKnm` for dL/dX (sparse_gplvm.py:34),
    which a VarDTC handle (`engine`, `X`, `Z` given) reduces on the device from what the evaluation left there
    (gpx_sparse_grad_X, once per handle). It cannot turn into an ndarray: the N x M matrix is never formed. A composite
    kernel's handle carries one gradient block per flattened leaf (`part_grads`) instead of dvariance / dlengthscale."""

    def __init__(self, key, role, shape, dvariance, dlengthscale, dZ, part_grads=None, engine=None, X=None, Z=None,
                 transposed=False):
        self._key, self.role, self.shape = key, role, shape
        self.dvariance, self.dlengthscale, self.dZ = dvariance, dlengthscale, dZ
        self.part_grads = part_grads
        self.ndim, self.dtype = 2, np.dtype(np.float64)
        self.transposed = transposed
        self._engine, self._X, self._Z = engine, X, Z
        self._serial = getattr(engine, "sparse_serial", None)
        self._dX = [None]                     # shared with the .T views

    def matches(self, key):
        return self._key == key

    @property
    def T(self):
        h = SparseDeviceGradient(self._key, self.role, self.shape[::-1], self.dvariance, self.dlengthscale, self.dZ,
                                 self.part_grads, transposed=not self.transposed)
        h._engine, h._X, h._Z, h._serial, h._dX = self._engine, self._X, self._Z, self._serial, self._dX
        return h

    def wants_dX(self):
        """True for dL_dKnm as VarDTC returned it (rows = data points): gradients_X then asks for dL/dX"""
        return self.role == "knm" and not self.transposed

    def grad_X(self, X, X2):
        """kern.gradients_X(dL_dKnm, X, Z) from the device, for the X and Z the evaluation ran on"""
        if self._engine is None:
            raise ValueError("gradients_X of dL_dKnm: this evaluation keeps no input gradient on the device (VarDTC does)")
        if getattr(self._engine, "sparse_serial", None) != self._serial:
            raise ValueError("stale gradient handle: the device has evaluated again since")
        X = np.asarray(X)
        if X.shape != self._X.shape or not np.array_equal(X, self._X) or \
                (X2 is not None and not np.array_equal(np.asarray(X2), self._Z)):
            raise ValueError("gradients_X of dL_dKnm takes the inputs and inducing inputs of the evaluation")
        if self._dX[0] is None:
            self._dX[0] = self._engine.sparse_grad_X()
        return self._dX[0]

    def __array__(self, dtype=None, copy=None):
        raise TypeError("%s of the device VarDTC evaluation is a handle to already-reduced gradients; the matrix itself is "
                        "never materialised (use a gpy_plugin kernel, or the stock VarDTC)" % (
                            "dL_dKnm" if self.role == "knm" else "dL_dKmm"))


class PsiDeviceGradient(object):
    """Stand-in for `grad_dict['dL_dpsi1']` (N x M) / `grad_dict['dL_dpsi2']` (M x M) of VarDTC.inference with uncertain
    inputs (var_dtc.py:178-183). The device evaluation (gpx_sparse_eval_psi) has already reduced them, with dL_dpsi0 and
    dL_dKmm, to the kernel's gradient, dZ and the gradients of q(X)'s mean and variance; the plugin RBF's
    update_gradients_expectations, gradients_Z_expectations and gradients_qX_expectations (sparse_gp.py:95-107,
    bayesian_gplvm.py:92-97) hand those back when given this handle for the kernel state, Z and q(X) it was computed for,
    while the engine holds that evaluation."""

    def __init__(self, key, role, shape, grad, dZ, dmu, dS, engine, mu, S, Z):
        self._key, self.role, self.shape = key, role, shape
        self.grad, self.dZ, self.dmu, self.dS = grad, dZ, dmu, dS
        self.ndim, self.dtype = 2, np.dtype(np.float64)
        self._engine, self._mu, self._S, self._Z = engine, mu, S, Z
        self._serial = getattr(engine, "sparse_serial", None)

    def sibling(self, role, shape):
        h = PsiDeviceGradient(self._key, role, shape, self.grad, self.dZ, self.dmu, self.dS, self._engine, self._mu,
                              self._S, self._Z)
        h._serial = self._serial
        return h

    def check(self, key, Z, qX):
        """ValueError unless the handle belongs to this kernel state, Z, q(X) and the engine's last evaluation"""
        if key != self._key or getattr(self._engine, "sparse_serial", None) != self._serial:
            raise ValueError("stale gradient handle: the device has evaluated other parameters since")
        if not (np.array_equal(np.asarray(Z), self._Z) and np.array_equal(np.asarray(qX.mean), self._mu)
                and np.array_equal(np.asarray(qX.variance), self._S)):
            raise ValueError("the psi gradient handle takes the inducing inputs and q(X) of its evaluation")

    def __array__(self, dtype=None, copy=None):
        raise TypeError("dL_d%s of the device evaluation is a handle to already-reduced gradients; the matrix itself is "
                        "never materialised (use the gpy_plugin RBF, or the stock VarDTC)" % self.role)


def _normal_posterior(qX):
    """q(X) is a NormalPosterior (not a spike-and-slab one): the device's psi-statistics apply"""
    return type(qX).__name__ == "NormalPosterior" and hasattr(qX, "mean") and hasattr(qX, "variance")


def _make_kernel(base, kind, ffi):
    class B200Kernel(base):
        _gpx_kind = kind

        def _gpx_theta(self):
            ls = np.asarray(self.lengthscale.values if hasattr(self.lengthscale, "values") else self.lengthscale,
                            dtype=np.float64).reshape(-1)
            return kind, bool(self.ARD), float(np.asarray(self.variance).reshape(-1)[0]), (ls if self.ARD else float(ls[0]))

        def _gpx_state_key(self):
            k, ard, var, ls = self._gpx_theta()
            return (k, ard, var, tuple(np.atleast_1d(ls).tolist()), tuple(np.atleast_1d(self.active_dims).tolist()))

        def K(self, X, X2=None):
            k, ard, var, ls = self._gpx_theta()
            return ffi.kern_K(k, ard, var, ls, np.asarray(X, dtype=np.float64),
                              None if X2 is None else np.asarray(X2, dtype=np.float64))

        def Kdiag(self, X):
            return ffi.kern_Kdiag(kind, float(np.asarray(self.variance).reshape(-1)[0]), int(np.asarray(X).shape[0]))

        def update_gradients_full(self, dL_dK, X, X2=None, reset=True):
            if isinstance(dL_dK, DeviceGradient) and X2 is None and dL_dK.matches(self._gpx_state_key()):
                self.variance.gradient = dL_dK.dvariance
                self.lengthscale.gradient = dL_dK.dlengthscale
                return
            if isinstance(dL_dK, SparseDeviceGradient):          # core/sparse_gp.py:112,114 on the device's reductions
                if not dL_dK.matches(self._gpx_state_key()):
                    raise ValueError("stale gradient handle: the kernel parameters changed since the sparse evaluation")
                self.variance.gradient = dL_dK.dvariance
                self.lengthscale.gradient = dL_dK.dlengthscale if self.ARD else np.sum(dL_dK.dlengthscale)
                return
            k, ard, var, ls = self._gpx_theta()
            dv, dl = ffi.kern_grad_full(k, ard, var, ls, np.asarray(X, dtype=np.float64),
                                        np.asarray(dL_dK, dtype=np.float64),
                                        None if X2 is None else np.asarray(X2, dtype=np.float64))
            self.variance.gradient = dv
            self.lengthscale.gradient = dl if self.ARD else dl[0]

        def update_gradients_diag(self, dL_dKdiag, X):
            self.variance.gradient = np.sum(dL_dKdiag)
            self.lengthscale.gradient = 0.

        def gradients_X(self, dL_dK, X, X2=None):
            """stationary.py:245-252,348-366 (gpx_kern_grad_X); with a handle of the device VarDTC evaluation: the dL/dZ
            it already holds (core/sparse_gp.py:117-118), or for the untransposed dL_dKnm dL/dX from the device
            (sparse_gplvm.py:34)."""
            if isinstance(dL_dK, SparseDeviceGradient):
                if not dL_dK.matches(self._gpx_state_key()):
                    raise ValueError("stale gradient handle: the kernel parameters changed since the sparse evaluation")
                return dL_dK.grad_X(X, X2) if dL_dK.wants_dX() else dL_dK.dZ
            if isinstance(dL_dK, DeviceGradient) and X2 is None:   # gplvm.py:49 on the exact evaluation of this kernel on X
                g = dL_dK.grad_X(self._gpx_state_key(), X)
                if g is not None:
                    return g
            k, ard, var, ls = self._gpx_theta()
            return ffi.kern_grad_X(k, ard, var, ls, np.asarray(X, dtype=np.float64), np.asarray(dL_dK, dtype=np.float64),
                                   None if X2 is None else np.asarray(X2, dtype=np.float64))

        if kind == "rbf":
            # the expectations under q(X) = N(mu, diag(S)) (rbf.py:344-367): the device's psi-statistics for a
            # NormalPosterior on up to 16 latent columns; a spike-and-slab posterior and psi2n stay the reference's
            def _gpx_psi_ok(self, qX):
                return _normal_posterior(qX) and 1 <= np.asarray(qX.mean).shape[1] <= 16

            def _gpx_psi_desc(self, Q):
                k, ard, var, ls = self._gpx_theta()
                return ("rbf", ard, 0, list(range(Q)), var, ls)

            def _gpx_psi_args(self, Z, qX):
                mu = np.ascontiguousarray(qX.mean, dtype=np.float64)
                S = np.ascontiguousarray(qX.variance, dtype=np.float64)
                return self._gpx_psi_desc(mu.shape[1]), mu, S, np.ascontiguousarray(Z, dtype=np.float64)

            def psi0(self, Z, variational_posterior):
                if not self._gpx_psi_ok(variational_posterior):
                    return super(B200Kernel, self).psi0(Z, variational_posterior)
                return np.full(np.asarray(variational_posterior.mean).shape[0], self._gpx_theta()[2])

            def psi1(self, Z, variational_posterior):
                if not self._gpx_psi_ok(variational_posterior):
                    return super(B200Kernel, self).psi1(Z, variational_posterior)
                return ffi.psi_stats(*self._gpx_psi_args(Z, variational_posterior))[1]

            def psi2(self, Z, variational_posterior):
                if not self._gpx_psi_ok(variational_posterior):
                    return super(B200Kernel, self).psi2(Z, variational_posterior)
                return ffi.psi_stats(*self._gpx_psi_args(Z, variational_posterior))[2]

            def _gpx_psi_derivs(self, dL_dpsi0, dL_dpsi1, dL_dpsi2, Z, qX):
                """(grad [variance, lengthscale..], dZ, dmu, dS): from the handle of the device evaluation, or from
                gpx_psi_grads for host arrays; None when the reference's method applies"""
                if isinstance(dL_dpsi1, PsiDeviceGradient):
                    dL_dpsi1.check(self._gpx_state_key(), Z, qX)
                    return dL_dpsi1.grad, dL_dpsi1.dZ, dL_dpsi1.dmu, dL_dpsi1.dS
                if not self._gpx_psi_ok(qX) or np.ndim(dL_dpsi2) != 2:
                    return None
                return ffi.psi_grads(*self._gpx_psi_args(Z, qX), dL_dpsi0, dL_dpsi1, dL_dpsi2)

            def update_gradients_expectations(self, dL_dpsi0, dL_dpsi1, dL_dpsi2, Z, variational_posterior):
                r = self._gpx_psi_derivs(dL_dpsi0, dL_dpsi1, dL_dpsi2, Z, variational_posterior)
                if r is None:
                    return super(B200Kernel, self).update_gradients_expectations(dL_dpsi0, dL_dpsi1, dL_dpsi2, Z,
                                                                                 variational_posterior)
                self.variance.gradient = r[0][0]
                self.lengthscale.gradient = r[0][1:] if self.ARD else r[0][1]

            def gradients_Z_expectations(self, dL_dpsi0, dL_dpsi1, dL_dpsi2, Z, variational_posterior):
                r = self._gpx_psi_derivs(dL_dpsi0, dL_dpsi1, dL_dpsi2, Z, variational_posterior)
                if r is None:
                    return super(B200Kernel, self).gradients_Z_expectations(dL_dpsi0, dL_dpsi1, dL_dpsi2, Z,
                                                                            variational_posterior)
                return r[1]

            def gradients_qX_expectations(self, dL_dpsi0, dL_dpsi1, dL_dpsi2, Z, variational_posterior):
                r = self._gpx_psi_derivs(dL_dpsi0, dL_dpsi1, dL_dpsi2, Z, variational_posterior)
                if r is None:
                    return super(B200Kernel, self).gradients_qX_expectations(dL_dpsi0, dL_dpsi1, dL_dpsi2, Z,
                                                                             variational_posterior)
                return r[2], r[3]

    B200Kernel.__name__ = B200Kernel.__qualname__ = base.__name__
    return B200Kernel


def _make_part_kernel(base, kind, ffi):
    """GPy.kern.RatQuad (stationary.py:747-802) / GPy.kern.StdPeriodic (standard_periodic.py:21-548) with K, Kdiag and
    update_gradients_full on the device (gpx_kern_part_K / gpx_kern_part_grad_full, or the block a fused composite evaluation
    already reduced); gradients_X and update_gradients_diag stay GPy's."""

    class B200PartKernel(base):
        _gpx_part_kind = kind

        def _gpx_desc(self, dims, term):
            """(kind, ARD, term, dims, variance, lengthscale, extra) for ffi.Engine.exact_eval_multi / kern_part_*"""
            var = float(np.asarray(self.variance).reshape(-1)[0])
            ls = np.array(self.lengthscale, dtype=np.float64).reshape(-1)
            if kind == "ratquad":
                ard, extra = bool(self.ARD), {"power": float(np.asarray(self.power).reshape(-1)[0])}
            else:
                T = np.array(self.period, dtype=np.float64).reshape(-1)
                ard, extra = bool(self.ARD2), {"period": T if self.ARD1 else float(T[0]), "ARD_period": bool(self.ARD1)}
            return (kind, ard, term, [int(d) for d in dims], var, ls if ard else float(ls[0]), extra)

        def _gpx_state_key(self):
            return _composite_key(self)

        def K(self, X, X2=None):
            X = np.asarray(X, dtype=np.float64)
            return ffi.kern_part_K(self._gpx_desc(range(X.shape[1]), 0), X,
                                   None if X2 is None else np.asarray(X2, dtype=np.float64))

        def Kdiag(self, X):
            return ffi.kern_Kdiag(kind, float(np.asarray(self.variance).reshape(-1)[0]), int(np.asarray(X).shape[0]))

        def update_gradients_full(self, dL_dK, X, X2=None, reset=True):
            if isinstance(dL_dK, DeviceGradient) and X2 is None and dL_dK.part_grads is not None \
                    and dL_dK.matches(_composite_key(self)):
                _set_part_gradients(self, dL_dK.part_grads[0])
                return
            X = np.asarray(X, dtype=np.float64)
            _set_part_gradients(self, ffi.kern_part_grad_full(self._gpx_desc(range(X.shape[1]), 0), X,
                                                              np.asarray(dL_dK, dtype=np.float64),
                                                              None if X2 is None else np.asarray(X2, dtype=np.float64)))

    B200PartKernel.__name__ = B200PartKernel.__qualname__ = base.__name__
    return B200PartKernel


def _set_part_gradients(leaf, g):
    """a RatQuad [variance, lengthscale.., power] / StdPeriodic [variance, period.., lengthscale..] gradient block -> the
    leaf's parameters (scalars for the isotropic ones, as GPy's own update_gradients_full assigns them)"""
    g = np.asarray(g, dtype=np.float64)
    nl = np.asarray(leaf.lengthscale).size
    leaf.variance.gradient = g[0]
    if leaf._gpx_part_kind == "ratquad":
        leaf.lengthscale.gradient = g[1:1 + nl] if leaf.ARD else g[1]
        leaf.power.gradient = g[1 + nl]
    else:
        npd = np.asarray(leaf.period).size
        leaf.period.gradient = g[1:1 + npd] if leaf.ARD1 else g[1]
        leaf.lengthscale.gradient = g[1 + npd:] if leaf.ARD2 else g[1 + npd]


def _leaf_ngrad(leaf):
    """entries of one leaf's block in the gradient of exact_eval_multi"""
    if hasattr(leaf, "_gpx_part_kind"):
        return 1 + np.asarray(leaf.lengthscale).size + (1 if leaf._gpx_part_kind == "ratquad" else np.asarray(leaf.period).size)
    return 1 + (np.asarray(leaf.lengthscale).size if hasattr(leaf, "lengthscale") else 0)


def _set_leaf_gradients(kern, part_grads):
    """every flattened leaf of kern gets its block of a composite device evaluation"""
    for (leaf, _), g in zip(_flatten(kern), part_grads):
        if hasattr(leaf, "_gpx_part_kind"):
            _set_part_gradients(leaf, g)
            continue
        leaf.variance.gradient = g[0]
        if hasattr(leaf, "lengthscale"):
            leaf.lengthscale.gradient = g[1:] if leaf.ARD else g[1]


def _check_sparse_handle(kern, h):
    if h.part_grads is None or not h.matches(_composite_key(kern)):
        raise ValueError("stale gradient handle: the kernel parameters changed since the sparse evaluation")


def _make_combination(base, is_prod):
    """Add / Prod over GPy's own class: K, Kdiag ... stay the reference's; update_gradients_full recognises the handle of
    a fused composite evaluation and hands every leaf the gradient the device already reduced for it (the stock methods
    would build every factor's N x N matrix on the host: add.py:76-77, prod.py:377-385). The handles of the device VarDTC
    are recognised by update_gradients_full and gradients_X (core/sparse_gp.py:112-118): the stock Prod.gradients_X would
    multiply a handle by an ndarray (prod.py:397-407), the stock Add.gradients_X would count dZ once per leaf
    (add.py:88-100)."""

    class B200Combination(base):
        def update_gradients_full(self, dL_dK, X, X2=None):
            if isinstance(dL_dK, SparseDeviceGradient):
                _check_sparse_handle(self, dL_dK)
                _set_leaf_gradients(self, dL_dK.part_grads)
                return
            if isinstance(dL_dK, DeviceGradient) and X2 is None and dL_dK.part_grads is not None \
                    and dL_dK.matches(_composite_key(self)):
                _set_leaf_gradients(self, dL_dK.part_grads)
                return
            return super(B200Combination, self).update_gradients_full(np.asarray(dL_dK, dtype=np.float64), X, X2)

        def gradients_X(self, dL_dK, X, X2=None):
            if isinstance(dL_dK, SparseDeviceGradient):   # one gpx_sparse_grad_X for the whole combination
                _check_sparse_handle(self, dL_dK)
                return dL_dK.grad_X(X, X2) if dL_dK.wants_dX() else dL_dK.dZ
            if isinstance(dL_dK, DeviceGradient) and X2 is None:   # one gpx_exact_grad_X for the whole combination
                leaves = _flatten(self)
                if leaves is not None and not any(hasattr(l, "_gpx_part_kind") for l, _ in leaves):
                    g = dL_dK.grad_X(_composite_key(self), X)
                    if g is not None:
                        return g
            return super(B200Combination, self).gradients_X(dL_dK, X, X2)

    B200Combination.__name__ = B200Combination.__qualname__ = base.__name__
    B200Combination._gpx_is_prod = is_prod
    return B200Combination


def _is_leaf(k):
    return hasattr(k, "_gpx_kind") or hasattr(k, "_gpx_part_kind") or type(k).__name__ in ("White", "Bias")


def _flatten(kern):
    """GPy kernel object -> [(leaf, term)] when it is a leaf, a product of leaves or a sum of those; else None"""
    def product(k, term):
        if _is_leaf(k):
            return [(k, term)]
        if getattr(k, "_gpx_is_prod", None) is True and all(_is_leaf(q) for q in k.parts):
            return [(q, term) for q in k.parts]
        return None

    if getattr(kern, "_gpx_is_prod", None) is False:
        out = []
        for t, part in enumerate(kern.parts):
            fl = product(part, t)
            if fl is None:
                return None
            out.extend(fl)
        return out
    return product(kern, 0)


def _leaf_descriptor(leaf, term):
    if hasattr(leaf, "_gpx_part_kind"):
        return leaf._gpx_desc(np.atleast_1d(leaf.active_dims).astype(int).tolist(), term)
    var = float(np.asarray(leaf.variance).reshape(-1)[0])
    if not hasattr(leaf, "_gpx_kind"):
        return (type(leaf).__name__.lower(), False, term, [], var, None)
    kind, ard, var, ls = leaf._gpx_theta()
    return (kind, ard, term, np.atleast_1d(leaf.active_dims).astype(int).tolist(), var, ls)


def _composite_key(kern):
    fl = _flatten(kern)
    if fl is None:
        return None
    return tuple((t,) + tuple(repr(x) for x in _leaf_descriptor(leaf, t)) for (leaf, t) in fl)


def _make_vardtc(base, kernel_types, ffi):
    from .sparse import LazySparsePosterior

    class B200VarDTC(base):
        """GPy.inference.latent_function_inference.VarDTC with the whole evaluation on the device (gpx_sparse_eval /
        gpx_sparse_eval_het; gpx_sparse_eval_multi for a B.Add / B.Prod over plugin stationary leaves and GPy's own White /
        Bias). Certain inputs, Gaussian / HeteroscedasticGaussian noise, no mean function; anything else goes to the stock
        method (var_dtc.py:66-215)."""

        def __init__(self, limit=1, device=0, engine=None):
            super(B200VarDTC, self).__init__(limit)
            self.device, self._engine, self._data_key = device, engine, _DataKey()

        @property
        def engine(self):
            if self._engine is None:
                self._engine = ffi.Engine(self.device)
            return self._engine

        def invalidate_data(self):
            self._data_key.invalidate()

        def __getstate__(self):
            """the stock class pickles as its cache limit (var_dtc.py:39-41: Cacher objects cannot be pickled); the device
            handle is dropped the same way (precedent: GPy/kern/src/rbf.py:313-318)"""
            return {"limit": self.limit, "device": self.device}

        def __setstate__(self, state):
            super(B200VarDTC, self).__setstate__(state["limit"])   # var_dtc.py:43-48 rebuilds the caches
            self.device, self._engine, self._data_key = state.get("device", 0), None, _DataKey()

        def inference(self, kern, X, Z, likelihood, Y, Y_metadata=None, mean_function=None, precision=None, Lm=None,
                      dL_dKmm=None, psi0=None, psi1=None, psi2=None, Z_tilde=None):
            if self._psi_route(kern, X, likelihood, Y_metadata, mean_function, precision, Lm, dL_dKmm, psi0, psi1,
                               psi2):
                return self._inference_psi(kern, X, Z, likelihood, Y, Y_metadata, Z_tilde)
            plain_X = isinstance(X, np.ndarray)                    # a VariationalPosterior is not an ndarray subclass
            leaves = _flatten(kern) if hasattr(kern, "_gpx_is_prod") else None
            if leaves is not None and any(not (hasattr(l, "_gpx_kind") or type(l).__name__ in ("White", "Bias"))
                                          for l, _ in leaves):
                leaves = None                                      # RatQuad / StdPeriodic: no device gradients_X
            if ((leaves is None and not isinstance(kern, kernel_types)) or not plain_X or mean_function is not None
                    or Lm is not None or dL_dKmm is not None or psi0 is not None or psi1 is not None or psi2 is not None):
                return super(B200VarDTC, self).inference(kern, X, Z, likelihood, Y, Y_metadata, mean_function, precision,
                                                         Lm, dL_dKmm, psi0, psi1, psi2, Z_tilde)
            if precision is None:                                  # var_dtc.py:78-80
                variance = np.asarray(likelihood.gaussian_variance(Y_metadata), dtype=np.float64).reshape(-1)
            else:
                variance = 1.0 / np.asarray(precision, dtype=np.float64).reshape(-1)
            Xs = np.ascontiguousarray(kern._slice_X(np.asarray(X)), dtype=np.float64)
            Zs = np.ascontiguousarray(kern._slice_X(np.asarray(Z)), dtype=np.float64)
            Yc = np.ascontiguousarray(Y, dtype=np.float64)
            N, P = Yc.shape
            M = Zs.shape[0]
            eng = self.engine
            if not self._data_key.matches(Xs, Yc):
                if P > 8:
                    eng.set_option("sparse_wide", 1)               # the sparse state's wide route (P <= 1024)
                eng.sparse_set_data(Xs, Yc)
                self._data_key.remember(Xs, Yc)
            if leaves is not None:
                return self._inference_multi(eng, kern, leaves, Xs, Zs, likelihood, variance, N, P, M, Y_metadata,
                                             Z_tilde)
            k, ard, var, ls = kern._gpx_theta()
            if variance.size > 1:                                  # het_noise (var_dtc.py:82-84)
                lml, grad, dZ, dR = eng.sparse_eval_het(k, ard, var, ls, Zs, variance)
                beta = 1.0 / np.fmax(variance, self.const_jitter)
                dL_dthetaL = likelihood.exact_inference_gradients(dR, Y_metadata)         # :176
                gk = grad
            else:
                lml, grad, dZ = eng.sparse_eval(k, ard, var, ls, Zs, float(variance[0]))
                beta = np.full(N, 1.0 / max(float(variance[0]), self.const_jitter))
                dL_dthetaL = likelihood.exact_inference_gradients(np.atleast_1d(grad[-1]), Y_metadata)
                gk = grad[:-1]
            if Z_tilde is not None:
                lml += Z_tilde                                     # var_dtc.py:166-170
            dL_dKdiag = -0.5 * P * beta                            # _compute_dL_dpsi: dL_dpsi0 (:218)
            key = kern._gpx_state_key()
            dlen = np.atleast_1d(gk[1:])
            knm = SparseDeviceGradient(key, "knm", (N, M), gk[0] - dL_dKdiag.sum(), dlen, dZ, engine=eng, X=Xs, Z=Zs)
            kmm = SparseDeviceGradient(key, "kmm", (M, M), 0.0, np.zeros_like(dlen), np.zeros_like(dZ))
            post = LazySparsePosterior(eng, key, Zs)
            return post, lml, {"dL_dKmm": kmm, "dL_dKdiag": dL_dKdiag, "dL_dKnm": knm, "dL_dthetaL": dL_dthetaL,
                               "dL_dm": None}

        def _psi_route(self, kern, X, likelihood, Y_metadata, mean_function, precision, Lm, dL_dKmm, psi0, psi1, psi2):
            """uncertain inputs on the device: a NormalPosterior X on up to 16 columns, a lone plugin RBF on all of them in
            order, a scalar Gaussian noise, no mean function and nothing precomputed"""
            if not _normal_posterior(X) or getattr(kern, "_gpx_kind", None) != "rbf":
                return False
            if mean_function is not None or precision is not None or any(
                    a is not None for a in (Lm, dL_dKmm, psi0, psi1, psi2)):
                return False
            Q = np.asarray(X.mean).shape[1]
            if not (1 <= Q <= 16) or not np.array_equal(np.atleast_1d(kern.active_dims), np.arange(Q)):
                return False
            return np.asarray(likelihood.gaussian_variance(Y_metadata)).size == 1

        def _inference_psi(self, kern, X, Z, likelihood, Y, Y_metadata, Z_tilde):
            """ONE gpx_sparse_eval_psi (var_dtc.py:66-215 with uncertain inputs, sparse_gp.py:88-107); dL_dpsi0 is the
            real N-vector (:218), dL_dpsi1 / dL_dpsi2 are handles carrying the reduced gradients, dL_dKmm a handle of
            zeros (its share is inside the expectations' gradients)"""
            mu = np.ascontiguousarray(X.mean, dtype=np.float64)
            S = np.ascontiguousarray(X.variance, dtype=np.float64)
            Zs = np.ascontiguousarray(Z, dtype=np.float64)
            Yc = np.ascontiguousarray(Y, dtype=np.float64)
            N, P = Yc.shape
            M = Zs.shape[0]
            eng = self.engine
            if not self._data_key.matches(mu, Yc):
                if P > 8:
                    eng.set_option("sparse_wide", 1)
                eng.sparse_set_data(mu, Yc)
                self._data_key.remember(mu, Yc)
            noise = float(np.asarray(likelihood.gaussian_variance(Y_metadata)).reshape(-1)[0])
            k, ard, var, ls = kern._gpx_theta()
            lml, grad, dZ, dmu, dS = eng.sparse_eval_psi(("rbf", ard, 0, list(range(mu.shape[1])), var, ls), S, Zs, noise)
            if Z_tilde is not None:
                lml += Z_tilde                                     # var_dtc.py:166-170
            beta = 1.0 / max(noise, self.const_jitter)
            key = kern._gpx_state_key()
            h1 = PsiDeviceGradient(key, "psi1", (N, M), grad[:-1], dZ, dmu, dS, eng, mu, S, Zs)
            kmm = SparseDeviceGradient(key, "kmm", (M, M), 0.0, np.zeros(grad.size - 2), np.zeros_like(dZ))
            dL_dthetaL = likelihood.exact_inference_gradients(np.atleast_1d(grad[-1]), Y_metadata)
            return LazySparsePosterior(eng, key, Zs), lml, {
                "dL_dKmm": kmm, "dL_dpsi0": np.full(N, -0.5 * P * beta), "dL_dpsi1": h1,
                "dL_dpsi2": h1.sibling("psi2", (M, M)), "dL_dthetaL": dL_dthetaL}

        def _inference_multi(self, eng, kern, leaves, Xs, Zs, likelihood, variance, N, P, M, Y_metadata, Z_tilde):
            """a sum / product kernel: ONE gpx_sparse_eval_multi. GPy's stock update_gradients_diag runs first
            (sparse_gp.py:110) and gives each leaf sum(dL_dKdiag) times the other variances of its term (add.py:79-80,
            prod.py:386-394); the dL_dKnm handle carries each leaf's total minus that share, the dL_dKmm handle zeros."""
            het = variance.size > 1
            out = eng.sparse_eval_multi([_leaf_descriptor(l, t) for (l, t) in leaves], Zs,
                                        variance if het else float(variance[0]))
            lml, grad, dZ = out[:3]
            if het:
                beta = 1.0 / np.fmax(variance, self.const_jitter)
                dL_dthetaL = likelihood.exact_inference_gradients(out[3], Y_metadata)     # var_dtc.py:176
            else:
                beta = np.full(N, 1.0 / max(float(variance[0]), self.const_jitter))
                dL_dthetaL = likelihood.exact_inference_gradients(np.atleast_1d(grad[-1]), Y_metadata)
            if Z_tilde is not None:
                lml += Z_tilde                                     # var_dtc.py:166-170
            dL_dKdiag = -0.5 * P * beta                            # _compute_dL_dpsi: dL_dpsi0 (:218)
            h_knm, h_kmm = _composite_handles(kern, leaves, grad, dL_dKdiag.sum(), dZ, N, M, engine=eng, X=Xs, Z=Zs)
            return LazySparsePosterior(eng, h_knm._key, Zs), lml, {"dL_dKmm": h_kmm, "dL_dKdiag": dL_dKdiag,
                                                                  "dL_dKnm": h_knm, "dL_dthetaL": dL_dthetaL,
                                                                  "dL_dm": None}

    B200VarDTC.__name__ = B200VarDTC.__qualname__ = "VarDTC"
    return B200VarDTC


def _composite_handles(kern, leaves, grad, diag, dZ, N, M, engine=None, X=None, Z=None):
    """the dL_dKnm / dL_dKmm handles of a fused composite sparse evaluation. GPy's stock update_gradients_diag runs first
    (sparse_gp.py:110) and gives each leaf sum(dL_dKdiag) = diag times the other variances of its term (add.py:79-80,
    prod.py:386-394); the dL_dKnm handle carries each leaf's total minus that share, the dL_dKmm handle zeros."""
    knm, zeros, i = [], [], 0
    for j, (leaf, t) in enumerate(leaves):
        n = _leaf_ngrad(leaf)
        g = np.array(grad[i:i + n], dtype=np.float64)
        other = 1.0
        for q, (l2, t2) in enumerate(leaves):
            if q != j and t2 == t:
                other *= float(np.asarray(l2.variance).reshape(-1)[0])
        g[0] -= diag * other
        knm.append(g)
        zeros.append(np.zeros(n))
        i += n
    key = _composite_key(kern)
    return (SparseDeviceGradient(key, "knm", (N, M), None, None, dZ, part_grads=knm, engine=engine, X=X, Z=Z),
            SparseDeviceGradient(key, "kmm", (M, M), None, None, np.zeros_like(dZ), part_grads=zeros))


def _make_fitc(base, kernel_types, ffi):
    from .sparse import LazySparsePosterior

    class B200FITC(base):
        """GPy.inference.latent_function_inference.FITC with the whole evaluation on the device (gpx_sparse_eval_fitc) for
        a plugin stationary kernel or a B.Add / B.Prod over plugin stationary leaves and GPy's own White / Bias, Gaussian
        noise, one output column and no mean function; anything else goes to the stock method (fitc.py:19-88), which
        raises what the reference raises. The grad dict has the stock keys: dL_dKnm / dL_dKmm are handles of the
        gradients the device already reduced (as B.VarDTC returns them), dL_dKdiag is the real N-vector dL_dR (:67)."""

        def __init__(self, device=0, engine=None):
            super(B200FITC, self).__init__()
            self.device, self._engine, self._data_key = device, engine, _DataKey()

        @property
        def engine(self):
            if self._engine is None:
                self._engine = ffi.Engine(self.device)
            return self._engine

        def invalidate_data(self):
            self._data_key.invalidate()

        def __getstate__(self):
            d = dict(self.__dict__)
            d["_engine"], d["_data_key"] = None, _DataKey()
            return d

        def inference(self, kern, X, Z, likelihood, Y, mean_function=None, Y_metadata=None):
            leaves = _flatten(kern) if hasattr(kern, "_gpx_is_prod") else None
            if leaves is not None and any(not (hasattr(l, "_gpx_kind") or type(l).__name__ in ("White", "Bias"))
                                          for l, _ in leaves):
                leaves = None                                      # RatQuad / StdPeriodic: no device gradients_X
            variance = np.asarray(likelihood.gaussian_variance(Y_metadata), dtype=np.float64).reshape(-1)
            if ((leaves is None and not isinstance(kern, kernel_types)) or not isinstance(X, np.ndarray)
                    or mean_function is not None or variance.size > 1 or np.shape(Y)[1] != 1):
                return super(B200FITC, self).inference(kern, X, Z, likelihood, Y, mean_function, Y_metadata)
            Xs = np.ascontiguousarray(kern._slice_X(np.asarray(X)), dtype=np.float64)
            Zs = np.ascontiguousarray(kern._slice_X(np.asarray(Z)), dtype=np.float64)
            Yc = np.ascontiguousarray(Y, dtype=np.float64)
            N, M = Yc.shape[0], Zs.shape[0]
            eng = self.engine
            if not self._data_key.matches(Xs, Yc):
                eng.sparse_set_data(Xs, Yc)
                self._data_key.remember(Xs, Yc)
            if leaves is not None:
                parts = [_leaf_descriptor(l, t) for (l, t) in leaves]
            else:
                k, ard, var, ls = kern._gpx_theta()
                parts = [(k, ard, 0, list(range(Xs.shape[1])), var, ls)]
            lml, grad, dZ, dL_dR = eng.sparse_eval_fitc(parts, Zs, float(variance[0]))
            dL_dthetaL = likelihood.exact_inference_gradients(dL_dR, Y_metadata)          # fitc.py:82
            if leaves is not None:
                knm, kmm = _composite_handles(kern, leaves, grad, dL_dR.sum(), dZ, N, M)
                key = knm._key
            else:
                key = kern._gpx_state_key()
                dlen = np.atleast_1d(grad[1:-1])
                knm = SparseDeviceGradient(key, "knm", (N, M), grad[0] - dL_dR.sum(), dlen, dZ)
                kmm = SparseDeviceGradient(key, "kmm", (M, M), 0.0, np.zeros_like(dlen), np.zeros_like(dZ))
            return LazySparsePosterior(eng, key, Zs), lml, {"dL_dKmm": kmm, "dL_dKdiag": dL_dR, "dL_dKnm": knm,
                                                           "dL_dthetaL": dL_dthetaL}

    B200FITC.__name__ = B200FITC.__qualname__ = "FITC"
    return B200FITC


def _make_laplace(base, kernel_types, ffi):
    from .laplace import Laplace as _DeviceLaplace

    class B200Laplace(base):
        """GPy.inference.latent_function_inference.Laplace with the N^2 / N^3 work on the device (gpx_laplace_*), for a
        plugin stationary kernel or a B.Add / B.Prod over plugin leaves and GPy's own White / Bias, any GPy likelihood (its
        own per-point terms are used), one output column and no mean function; anything else goes to the stock method
        (laplace.py:122-146), which raises what the reference raises. dL_dK is a handle of the gradient the device already
        reduced, as B.ExactGaussianInference returns it."""

        def __init__(self, device=0, engine=None):
            super(B200Laplace, self).__init__()
            self.device, self._engine = device, engine
            self._dev = None

        @property
        def engine(self):
            if self._engine is None:
                self._engine = ffi.Engine(self.device)
            return self._engine

        def invalidate_data(self):
            if self._dev is not None:
                self._dev.invalidate_data()

        def __getstate__(self):
            d = dict(self.__dict__)
            d["_engine"], d["_dev"] = None, None
            return d

        def inference(self, kern, X, likelihood, Y, mean_function=None, Y_metadata=None):
            leaves = None
            if not isinstance(kern, kernel_types):
                leaves = _flatten(kern) if hasattr(kern, "_gpx_is_prod") or hasattr(kern, "_gpx_part_kind") else None
            if ((leaves is None and not isinstance(kern, kernel_types)) or not isinstance(X, np.ndarray)
                    or mean_function is not None or np.ndim(Y) != 2 or np.shape(Y)[1] != 1):
                return super(B200Laplace, self).inference(kern, X, likelihood, Y, mean_function, Y_metadata)
            if self._dev is None:
                self._dev = _DeviceLaplace(engine=self.engine)
            dev = self._dev
            dev.bad_fhat = self.bad_fhat
            if leaves is not None:
                parts = [_leaf_descriptor(l, t) for (l, t) in leaves]
                Xs, key, ngrads, single = X, _composite_key(kern), [_leaf_ngrad(l) for l, _ in leaves], False
            else:
                Xs = kern._slice_X(X)[0] if _returns_tuple(kern, X) else kern._slice_X(X)
                k, ard, var, ls = kern._gpx_theta()
                parts = [(k, ard, 0, list(range(np.shape(Xs)[1])), var, ls)]
                key, ngrads, single = kern._gpx_state_key(), [1 + np.size(ls)], True
            out = dev.device_inference(Xs, Y, likelihood, Y_metadata, parts, key, ngrads, single)
            self.bad_fhat, self.first_run = dev.bad_fhat, False
            self.f_hat, self.W, self._previous_Ki_fhat = dev.f_hat, dev.W, dev._previous_Ki_fhat   # laplace.py:302-305
            return out

    B200Laplace.__name__ = B200Laplace.__qualname__ = "Laplace"
    return B200Laplace


def _make_ep(base, kernel_types, ffi):
    import sys
    from .ep import EP as _DeviceEP
    ref = sys.modules[base.__module__]   # the reference's gaussianApproximation, so that the stock method continues

    class B200EP(base):
        """GPy.inference.latent_function_inference.EP with the sweeps and the marginal on the device (gpx_ep_*), for a
        plugin stationary kernel or a B.Add / B.Prod over plugin leaves and GPy's own White / Bias, GPy's Bernoulli with
        the probit link, ndarray X, one output column and no mean function; anything else goes to the stock method
        (expectation_propagation.py:246-277). Both keep the sites in ga_approx_old as the reference's
        gaussianApproximation and the approximation in _ep_approximation, so either continues from the other's sites.
        dL_dK is a handle of the gradient the device already reduced, as B.ExactGaussianInference returns it."""

        def __init__(self, epsilon=1e-6, eta=1., delta=1., always_reset=False, max_iters=np.inf, ep_mode="alternated",
                     parallel_updates=False, loading=False, device=0, engine=None):
            super(B200EP, self).__init__(epsilon=epsilon, eta=eta, delta=delta, always_reset=always_reset,
                                         max_iters=max_iters, ep_mode=ep_mode, parallel_updates=parallel_updates,
                                         loading=loading)
            self.device, self._engine = device, engine
            self._dev = None

        @property
        def engine(self):
            if self._engine is None:
                self._engine = ffi.Engine(self.device)
            return self._engine

        def invalidate_data(self):
            if self._dev is not None:
                self._dev.invalidate_data()

        def __getstate__(self):
            d = dict(self.__dict__)
            d["_engine"], d["_dev"] = None, None
            return d

        def _on_device(self, kern, X, likelihood, Y, mean_function, K):
            link = getattr(likelihood, "gp_link", None)
            return (isinstance(X, np.ndarray) and mean_function is None and K is None and np.ndim(Y) == 2
                    and np.shape(Y)[1] == 1 and type(likelihood).__name__ == "Bernoulli"
                    and type(link).__name__ == "Probit"
                    and (isinstance(kern, kernel_types) or hasattr(kern, "_gpx_is_prod")
                         or hasattr(kern, "_gpx_part_kind")))

        def inference(self, kern, X, likelihood, Y, mean_function=None, Y_metadata=None, precision=None, K=None):
            leaves = None
            if self._on_device(kern, X, likelihood, Y, mean_function, K) and not isinstance(kern, kernel_types):
                leaves = _flatten(kern)
            if not self._on_device(kern, X, likelihood, Y, mean_function, K) or (
                    leaves is None and not isinstance(kern, kernel_types)):
                return super(B200EP, self).inference(kern, X, likelihood, Y, mean_function=mean_function,
                                                     Y_metadata=Y_metadata, precision=precision, K=K)
            if self._dev is None:
                self._dev = _DeviceEP(engine=self.engine)
            dev = self._dev
            for name in ("epsilon", "eta", "delta", "always_reset", "max_iters", "ep_mode", "parallel_updates",
                         "loading", "ga_approx_old", "_ep_approximation"):
                setattr(dev, name, getattr(self, name, None))
            if leaves is not None:
                parts = [_leaf_descriptor(l, t) for (l, t) in leaves]
                Xs, key, ngrads, single = X, _composite_key(kern), [_leaf_ngrad(l) for l, _ in leaves], False
            else:
                Xs = kern._slice_X(X)[0] if _returns_tuple(kern, X) else kern._slice_X(X)
                k, ard, var, ls = kern._gpx_theta()
                parts = [(k, ard, 0, list(range(np.shape(Xs)[1])), var, ls)]
                key, ngrads, single = kern._gpx_state_key(), [1 + np.size(ls)], True
            try:
                return dev.device_inference(Xs, np.asarray(Y), likelihood, Y_metadata, parts, key, ngrads, single)
            finally:
                old = dev.ga_approx_old
                self.ga_approx_old = None if old is None else ref.gaussianApproximation(old.v, old.tau)
                self._ep_approximation, self.loading = dev._ep_approximation, dev.loading

    B200EP.__name__ = B200EP.__qualname__ = "EP"
    return B200EP


def _make_epdtc(base, kernel_types, ffi):
    import sys
    from .ep import EPDTC as _DeviceEPDTC
    ref = sys.modules[base.__module__]   # the reference's gaussianApproximation / posteriorParamsDTC

    class B200EPDTC(base):
        """GPy.inference.latent_function_inference.EPDTC with the sweeps (in M-space) and the marginal on the device
        (gpx_epdtc_*), for a plugin stationary kernel or a B.Add / B.Prod over plugin stationary leaves and GPy's own White /
        Bias, GPy's Bernoulli with the probit link, ndarray X, one output column, no mean function and no precomputed Lm,
        dL_dKmm or psi statistics; anything else goes to the stock method (expectation_propagation.py:437-482). Both keep
        the sites in ga_approx_old as the reference's gaussianApproximation and _ep_approximation as the reference's
        3-tuple (posteriorParamsDTC, gaussianApproximation, log_Z_tilde), so either continues from the other's sites. The
        grad dict is B.VarDTC's: dL_dKnm / dL_dKmm are handles of the gradients the device already reduced."""

        def __init__(self, epsilon=1e-6, eta=1., delta=1., always_reset=False, max_iters=np.inf, ep_mode="alternated",
                     parallel_updates=False, loading=False, device=0, engine=None):
            super(B200EPDTC, self).__init__(epsilon=epsilon, eta=eta, delta=delta, always_reset=always_reset,
                                            max_iters=max_iters, ep_mode=ep_mode, parallel_updates=parallel_updates,
                                            loading=loading)
            self.device, self._engine = device, engine
            self._dev = None

        @property
        def engine(self):
            if self._engine is None:
                self._engine = ffi.Engine(self.device)
            return self._engine

        def invalidate_data(self):
            if self._dev is not None:
                self._dev.invalidate_data()

        def __getstate__(self):
            d = dict(self.__dict__)
            d["_engine"], d["_dev"] = None, None
            return d

        def __setstate__(self, state):
            self.__dict__.update(state)

        def _leaves(self, kern, X, likelihood, Y, mean_function, extra):
            """-> None (the stock method), False (a single plugin kernel) or the leaves of a plugin sum / product"""
            link = getattr(likelihood, "gp_link", None)
            if not (isinstance(X, np.ndarray) and mean_function is None and all(a is None for a in extra)
                    and np.ndim(Y) == 2 and np.shape(Y)[1] == 1 and type(likelihood).__name__ == "Bernoulli"
                    and type(link).__name__ == "Probit"):
                return None
            if isinstance(kern, kernel_types):
                return False
            if not hasattr(kern, "_gpx_is_prod"):
                return None
            leaves = _flatten(kern)
            if leaves is None or any(not (hasattr(l, "_gpx_kind") or type(l).__name__ in ("White", "Bias"))
                                     for l, _ in leaves):
                return None                                        # RatQuad / StdPeriodic: no device gradients_X
            return leaves

        def inference(self, kern, X, Z, likelihood, Y, mean_function=None, Y_metadata=None, Lm=None, dL_dKmm=None,
                      psi0=None, psi1=None, psi2=None):
            leaves = self._leaves(kern, X, likelihood, Y, mean_function, (Lm, dL_dKmm, psi0, psi1, psi2))
            if leaves is None:
                return super(B200EPDTC, self).inference(kern, X, Z, likelihood, Y, mean_function=mean_function,
                                                        Y_metadata=Y_metadata, Lm=Lm, dL_dKmm=dL_dKmm, psi0=psi0,
                                                        psi1=psi1, psi2=psi2)
            if self._dev is None:
                self._dev = _DeviceEPDTC(engine=self.engine)
            dev = self._dev
            for name in ("epsilon", "eta", "delta", "always_reset", "max_iters", "ep_mode", "parallel_updates",
                         "loading", "ga_approx_old", "_ep_approximation"):
                setattr(dev, name, getattr(self, name, None))
            if leaves:
                parts = [_leaf_descriptor(l, t) for (l, t) in leaves]
                Xs, Zs, key, ngrads = np.asarray(X), np.asarray(Z), _composite_key(kern), [_leaf_ngrad(l) for l, _ in leaves]
            else:
                Xs = kern._slice_X(X)[0] if _returns_tuple(kern, X) else kern._slice_X(X)
                Zs = kern._slice_X(Z)[0] if _returns_tuple(kern, Z) else kern._slice_X(Z)
                k, ard, var, ls = kern._gpx_theta()
                parts = [(k, ard, 0, list(range(np.shape(Xs)[1])), var, ls)]
                key, ngrads = kern._gpx_state_key(), [1 + np.size(ls)]
            try:
                post, lml, gd = dev.device_inference(Xs, Zs, np.asarray(Y), parts, key, ngrads, not leaves)
            finally:
                old = dev.ga_approx_old
                self.ga_approx_old = None if old is None else ref.gaussianApproximation(old.v, old.tau)
                app = dev._ep_approximation
                if app is not None:
                    pp, ga, logZ = app
                    app = (ref.posteriorParamsDTC(pp.mu, pp.Sigma_diag), ref.gaussianApproximation(ga.v, ga.tau), logZ)
                self._ep_approximation, self.loading = app, dev.loading
            N, M = np.shape(Y)[0], np.shape(Zs)[0]
            tau = np.asarray(self._ep_approximation[1].tau, dtype=np.float64)
            dL_dKdiag = -0.5 * tau                                 # _compute_dL_dpsi: dL_dpsi0 at precision tau~ (:218)
            dL_dthetaL = likelihood.exact_inference_gradients(np.zeros((N, 1)), Y_metadata)   # var_dtc.py:176
            dZ = gd["dZ"]
            if leaves:
                h_knm, h_kmm = _composite_handles(kern, leaves, np.concatenate(gd["part_grads"]), dL_dKdiag.sum(), dZ,
                                                  N, M)
            else:
                dlen = np.atleast_1d(gd["dlengthscale"])
                h_knm = SparseDeviceGradient(key, "knm", (N, M), gd["dvariance"] - dL_dKdiag.sum(), dlen, dZ)
                h_kmm = SparseDeviceGradient(key, "kmm", (M, M), 0.0, np.zeros_like(dlen), np.zeros_like(dZ))
            return post, lml, {"dL_dKmm": h_kmm, "dL_dKdiag": dL_dKdiag, "dL_dKnm": h_knm, "dL_dthetaL": dL_dthetaL,
                               "dL_dm": None}

    B200EPDTC.__name__ = B200EPDTC.__qualname__ = "EPDTC"
    return B200EPDTC


def _make_svgp(base, kernel_types, ffi):
    from .svgp import SVGPInference, q_triangle

    class B200SVGP(base):
        """GPy.inference.latent_function_inference.SVGP with Kmm, Kmn, A = Kmm^-1 Kmn, the marginals, the KL term and every
        gradient on the device (gpx_svgp_begin / _finish) around the likelihood's own variational_expectations on the
        host, for a plugin stationary kernel or a B.Add / B.Prod over plugin stationary leaves and GPy's own White / Bias,
        any likelihood, ndarray X, one output column and one latent function, no mean function; anything else goes to the
        stock method (svgp.py:12-118). The grad dict has the stock keys: dL_dKmn / dL_dKmm are handles of the gradients the
        device already reduced (GPy's unchanged SVGP.parameters_changed passes them to update_gradients_full and
        gradients_X, core/svgp.py:53-62), dL_dKdiag, dL_dm, dL_dchol (flat) and dL_dthetaL are the real arrays."""

        def __init__(self, device=0, engine=None):
            super(B200SVGP, self).__init__()
            self.device, self._engine = device, engine
            self._dev = None

        @property
        def engine(self):
            if self._engine is None:
                self._engine = ffi.Engine(self.device)
            return self._engine

        def invalidate_data(self):
            if self._dev is not None:
                self._dev.invalidate_data()

        def __getstate__(self):
            d = dict(self.__dict__)
            d["_engine"], d["_dev"] = None, None
            return d

        def _leaves(self, kern, X, Y, q_u_mean, mean_function):
            """-> None (the stock method), False (a single plugin kernel) or the leaves of a plugin sum / product"""
            if not (isinstance(X, np.ndarray) and mean_function is None and np.ndim(Y) == 2 and np.shape(Y)[1] == 1
                    and np.ndim(q_u_mean) == 2 and np.shape(q_u_mean)[1] == 1):
                return None
            if isinstance(kern, kernel_types):
                return False
            if not hasattr(kern, "_gpx_is_prod"):
                return None
            leaves = _flatten(kern)
            if leaves is None or any(not (hasattr(l, "_gpx_kind") or type(l).__name__ in ("White", "Bias"))
                                     for l, _ in leaves):
                return None                                        # RatQuad / StdPeriodic: no device gradients_X
            return leaves

        def inference(self, q_u_mean, q_u_chol, kern, X, Z, likelihood, Y, mean_function=None, Y_metadata=None,
                      KL_scale=1.0, batch_scale=1.0):
            leaves = self._leaves(kern, X, Y, q_u_mean, mean_function)
            if leaves is None:
                return super(B200SVGP, self).inference(q_u_mean, q_u_chol, kern, X, Z, likelihood, Y, mean_function,
                                                       Y_metadata, KL_scale, batch_scale)
            if self._dev is None:
                self._dev = SVGPInference(engine=self.engine)
            dev = self._dev
            if leaves:
                parts = [_leaf_descriptor(l, t) for (l, t) in leaves]
                Xs, Zs, key = np.asarray(X), np.asarray(Z), _composite_key(kern)
            else:
                Xs = kern._slice_X(X)[0] if _returns_tuple(kern, X) else kern._slice_X(X)
                Zs = kern._slice_X(Z)[0] if _returns_tuple(kern, Z) else kern._slice_X(Z)
                k, ard, var, ls = kern._gpx_theta()
                parts = [(k, ard, 0, list(range(np.shape(Xs)[1])), var, ls)]
                key = kern._gpx_state_key()
            Xs = np.ascontiguousarray(Xs, dtype=np.float64)
            Zs = np.ascontiguousarray(Zs, dtype=np.float64)
            Yc = np.ascontiguousarray(Y, dtype=np.float64)
            q_m = np.asarray(q_u_mean, dtype=np.float64)
            L = q_triangle(q_m, np.asarray(q_u_chol, dtype=np.float64), Zs.shape[0])
            eng = self.engine
            if not dev._data_key.matches(Xs, Yc):
                eng.sparse_set_data(Xs, Yc)
                dev._data_key.remember(Xs, Yc)
            N, M = Yc.shape[0], Zs.shape[0]
            post, lml, grad, gd = dev.device_inference(q_m, L, parts, key, Zs, likelihood, Yc, 0, N, Y_metadata,
                                                       batch_scale)
            dL_dKdiag, dZ = gd["dL_dKdiag"], gd["dZ"]
            if leaves:
                h_knm, h_kmm = _composite_handles(kern, leaves, grad, dL_dKdiag.sum(), dZ, N, M)
            else:
                dlen = np.atleast_1d(grad[1:])
                h_knm = SparseDeviceGradient(key, "knm", (N, M), grad[0] - dL_dKdiag.sum(), dlen, dZ)
                h_kmm = SparseDeviceGradient(key, "kmm", (M, M), 0.0, np.zeros_like(dlen), np.zeros_like(dZ))
            return post, lml, {"dL_dKmm": h_kmm, "dL_dKmn": h_knm.T, "dL_dKdiag": dL_dKdiag, "dL_dm": gd["dL_dm"],
                               "dL_dchol": gd["dL_dchol"], "dL_dthetaL": gd["dL_dthetaL"]}

    B200SVGP.__name__ = B200SVGP.__qualname__ = "SVGP"
    return B200SVGP


def _make_vargauss(base, kernel_types, ffi):
    from .vargauss import VarGauss as _DeviceVarGauss

    class B200VarGauss(base):
        """GPy.inference.latent_function_inference.VarGauss with the N^2 / N^3 work on the device (gpx_vargauss_*), for a
        plugin stationary kernel or a B.Add / B.Prod over plugin leaves and GPy's own White / Bias, any GPy likelihood
        with variational_expectations, ndarray X, one output column, no mean function and a finite, non-zero beta;
        anything else goes to the stock method (var_gauss.py:34-69), which raises what the reference raises. Under GPy's
        own model: m.inference_method = B.VarGauss(m.alpha, m.beta). dL_dK is a handle of the gradient the device
        already reduced; it is the derivative of the bound, where the stock method's dF_dK scales the wrong side
        (var_gauss.py:66) unless dF_dv is constant."""

        def __init__(self, alpha, beta, device=0, engine=None):
            super(B200VarGauss, self).__init__(alpha, beta)
            self.device, self._engine = device, engine
            self._dev = None

        @property
        def engine(self):
            if self._engine is None:
                self._engine = ffi.Engine(self.device)
            return self._engine

        def invalidate_data(self):
            if self._dev is not None:
                self._dev.invalidate_data()

        def __getstate__(self):
            d = dict(self.__dict__)
            d["_engine"], d["_dev"] = None, None
            return d

        def inference(self, kern, X, likelihood, Y, mean_function=None, Y_metadata=None, Z=None):
            leaves = None
            if not isinstance(kern, kernel_types):
                leaves = _flatten(kern) if hasattr(kern, "_gpx_is_prod") or hasattr(kern, "_gpx_part_kind") else None
            b = np.asarray(self.beta, dtype=np.float64)
            if ((leaves is None and not isinstance(kern, kernel_types)) or not isinstance(X, np.ndarray)
                    or mean_function is not None or np.ndim(Y) != 2 or np.shape(Y)[1] != 1
                    or not np.all(np.isfinite(b)) or np.any(b == 0)):
                return super(B200VarGauss, self).inference(kern, X, likelihood, Y, mean_function, Y_metadata, Z)
            if self._dev is None:
                self._dev = _DeviceVarGauss(self.alpha, self.beta, engine=self.engine)
            dev = self._dev
            dev.alpha, dev.beta = self.alpha, self.beta
            if leaves is not None:
                parts = [_leaf_descriptor(l, t) for (l, t) in leaves]
                Xs, key, ngrads, single = X, _composite_key(kern), [_leaf_ngrad(l) for l, _ in leaves], False
            else:
                Xs = kern._slice_X(X)[0] if _returns_tuple(kern, X) else kern._slice_X(X)
                k, ard, var, ls = kern._gpx_theta()
                parts = [(k, ard, 0, list(range(np.shape(Xs)[1])), var, ls)]
                key, ngrads, single = kern._gpx_state_key(), [1 + np.size(ls)], True
            return dev.device_inference(Xs, Y, likelihood, Y_metadata, parts, key, ngrads, single)

    B200VarGauss.__name__ = B200VarGauss.__qualname__ = "VarGauss"
    return B200VarGauss


def make(RBF, Exponential, Matern32, Matern52, ExactGaussianInference, ffi=_ffi, Add=None, Prod=None, VarDTC=None,
         RatQuad=None, StdPeriodic=None, FITC=None, Laplace=None, EP=None, EPDTC=None, SVGP=None,
         VarGauss=None):
    """Build the plugin classes on top of the given GPy base classes (Add / Prod optional: composite kernels; VarDTC /
    FITC optional: the sparse model; Laplace / EP / EPDTC optional: non-Gaussian likelihoods; SVGP optional: the
    stochastic variational sparse GP; VarGauss optional: the variational Gaussian approximation; RatQuad / StdPeriodic optional: leaves
    the composite evaluation knows, alone or inside Add / Prod)."""
    kernels = {n: _make_kernel(b, _KINDS[n], ffi) for n, b in
               (("RBF", RBF), ("Exponential", Exponential), ("Matern32", Matern32), ("Matern52", Matern52))}
    kernel_types = tuple(kernels.values())      # the single-kernel evaluations (exact and VarDTC) take these only
    for n, b in (("RatQuad", RatQuad), ("StdPeriodic", StdPeriodic)):
        if b is not None:
            kernels[n] = _make_part_kernel(b, _PART_KINDS[n], ffi)
    if Add is not None and Prod is not None:
        kernels["Add"], kernels["Prod"] = _make_combination(Add, False), _make_combination(Prod, True)

    class B200ExactGaussianInference(ExactGaussianInference):
        """GPy.inference.latent_function_inference.ExactGaussianInference with the fused device evaluation; anything the
        accelerated path does not cover (mean function, precomputed K, foreign kernels) goes to the stock method."""

        def __init__(self, device=0, engine=None):
            super(B200ExactGaussianInference, self).__init__()
            self.device, self._engine, self._data_key = device, engine, _DataKey()

        @property
        def engine(self):
            if self._engine is None:
                self._engine = ffi.Engine(self.device)
            return self._engine

        def invalidate_data(self):
            """force an upload at the next inference whatever the content"""
            self._data_key.invalidate()

        def __getstate__(self):
            """pickling goes back to a device-less object (precedent: GPy/kern/src/rbf.py:313-318 drops its GPU state);
            the engine is re-created lazily and the data re-uploaded at the next inference"""
            d = dict(self.__dict__)
            d["_engine"], d["_data_key"] = None, _DataKey()
            return d

        def inference(self, kern, X, likelihood, Y, mean_function=None, Y_metadata=None, K=None, variance=None,
                      Z_tilde=None):
            parts = None
            if mean_function is None and K is None and not isinstance(kern, kernel_types):
                # sums / products, and a lone RatQuad / StdPeriodic (a one-part composite)
                parts = _flatten(kern) if hasattr(kern, "_gpx_is_prod") or hasattr(kern, "_gpx_part_kind") else None
            if parts is None and (mean_function is not None or K is not None or not isinstance(kern, kernel_types)):
                return super(B200ExactGaussianInference, self).inference(kern, X, likelihood, Y, mean_function,
                                                                         Y_metadata, K, variance, Z_tilde)
            if variance is None:
                variance = likelihood.gaussian_variance(Y_metadata)
            nvec = np.asarray(variance, dtype=np.float64).reshape(-1)
            het = nvec.size > 1                      # HeteroscedasticGaussian (likelihoods/gaussian.py:347-362)
            if parts is not None:
                if het:
                    return super(B200ExactGaussianInference, self).inference(kern, X, likelihood, Y, mean_function,
                                                                             Y_metadata, K, variance, Z_tilde)
                # sum / product kernel (add.py, prod.py, static.py): ONE gpx_exact_eval_multi, data resident
                Xc = np.ascontiguousarray(X, dtype=np.float64)
                Yc = np.ascontiguousarray(Y, dtype=np.float64)
                if not self._data_key.matches(Xc, Yc):
                    self.engine.set_data(Xc, Yc)
                    self._data_key.remember(Xc, Yc)
                lml, grad, _ = self.engine.exact_eval_multi([_leaf_descriptor(l, t) for (l, t) in parts], float(nvec[0]),
                                                            jitter=1e-8, max_tries=5)
                if Z_tilde is not None:
                    lml += Z_tilde
                pg, i = [], 0
                for (leaf, _) in parts:
                    n = _leaf_ngrad(leaf)
                    pg.append(grad[i:i + n])
                    i += n
                key = _composite_key(kern)
                post = PosteriorExact(self.engine, Yc.shape[0], Yc.shape[1], key)
                dL_dK = DeviceGradient(self.engine, key, None, None, Yc.shape[0], part_grads=pg, X=self._data_key._X)
                return post, lml, {"dL_dK": dL_dK, "dL_dthetaL": grad[-1], "dL_dm": _LazyAlpha(post)}
            noise = None if het else float(nvec[0])
            Xs = np.ascontiguousarray(kern._slice_X(X)[0] if _returns_tuple(kern, X) else kern._slice_X(X),
                                      dtype=np.float64)
            Yc = np.ascontiguousarray(Y, dtype=np.float64)
            if not self._data_key.matches(Xs, Yc):   # exact content comparison (GP.set_XY has no hook into inference)
                self.engine.set_data(Xs, Yc)
                self._data_key.remember(Xs, Yc)
            k, ard, var, ls = kern._gpx_theta()
            if het:
                lml, grad, dnoise, _ = self.engine.exact_eval_het(k, ard, var, ls, nvec, jitter=1e-8, max_tries=5)
                dL_dthetaL = likelihood.exact_inference_gradients(dnoise, Y_metadata)   # gaussian.py:358-359
            else:
                lml, grad, _ = self.engine.exact_eval(k, ard, var, ls, noise, jitter=1e-8, max_tries=5)
                dL_dthetaL = grad[-1]
            if Z_tilde is not None:
                lml += Z_tilde
            post = PosteriorExact(self.engine, Yc.shape[0], Yc.shape[1], kern._gpx_state_key())
            dlen = grad[1:-1] if ard else grad[1]
            dL_dK = DeviceGradient(self.engine, kern._gpx_state_key(), grad[0], dlen, Yc.shape[0],
                                   X=None if het else self._data_key._X)
            return post, lml, {"dL_dK": dL_dK, "dL_dthetaL": dL_dthetaL, "dL_dm": _LazyAlpha(post)}

    B200ExactGaussianInference.__name__ = B200ExactGaussianInference.__qualname__ = "ExactGaussianInference"
    extra = {}
    if VarDTC is not None:
        extra["VarDTC"] = _make_vardtc(VarDTC, kernel_types, ffi)
    if FITC is not None:
        extra["FITC"] = _make_fitc(FITC, kernel_types, ffi)
    if Laplace is not None:
        extra["Laplace"] = _make_laplace(Laplace, kernel_types, ffi)
    if EP is not None:
        extra["EP"] = _make_ep(EP, kernel_types, ffi)
    if EPDTC is not None:
        extra["EPDTC"] = _make_epdtc(EPDTC, kernel_types, ffi)
    if SVGP is not None:
        extra["SVGP"] = _make_svgp(SVGP, kernel_types, ffi)
    if VarGauss is not None:
        extra["VarGauss"] = _make_vargauss(VarGauss, kernel_types, ffi)
    return types.SimpleNamespace(ExactGaussianInference=B200ExactGaussianInference, **kernels, **extra)


def _returns_tuple(kern, X):
    """Kern._slice_X returns the sliced array; some paramz versions wrap cached results — accept both."""
    r = kern._slice_X(X)
    return isinstance(r, tuple)


def load():
    """Plugin classes over an installed GPy."""
    import GPy
    from GPy.inference.latent_function_inference import EP, FITC, ExactGaussianInference, Laplace, VarDTC, VarGauss
    from GPy.inference.latent_function_inference.expectation_propagation import EPDTC
    from GPy.inference.latent_function_inference.svgp import SVGP
    return make(GPy.kern.RBF, GPy.kern.Exponential, GPy.kern.Matern32, GPy.kern.Matern52, ExactGaussianInference,
                Add=GPy.kern.Add, Prod=GPy.kern.Prod, VarDTC=VarDTC, RatQuad=GPy.kern.RatQuad, StdPeriodic=GPy.kern.StdPeriodic,
                FITC=FITC, Laplace=Laplace, EP=EP, EPDTC=EPDTC, SVGP=SVGP, VarGauss=VarGauss)
