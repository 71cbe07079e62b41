"""Host-side mirror of GPy's stationary-kernel plugin interface, computing on the H100 through libgpx.

Same names, argument meaning and error behaviour as the reference classes:
    GPy.kern.RBF           GPy/kern/src/rbf.py:13-52,177-178
    GPy.kern.Exponential   GPy/kern/src/stationary.py:378-386
    GPy.kern.Matern32      GPy/kern/src/stationary.py:457-492
    GPy.kern.Matern52      GPy/kern/src/stationary.py:556-589
    GPy.kern.RatQuad       GPy/kern/src/stationary.py:747-802
    GPy.kern.StdPeriodic   GPy/kern/src/standard_periodic.py:21-94,125-139,501-548
base: GPy.kern.src.stationary.Stationary (stationary.py:23-243) and GPy.kern.Kern (kern.py:12-145).
`K`, `Kdiag`, `update_gradients_full`, `update_gradients_diag` take/return NumPy arrays exactly like the reference;
there is no NumPy implementation behind them — every call goes through the C ABI (include/gpx.h).
"""
import numpy as np

from . import _ffi
from .param import Param, Parameterized


class DeviceGradient(object):
    """Lazy, device-backed stand-in for the N x N `dL_dK` that ExactGaussianInference hands to
    `kern.update_gradients_full` (GPy/core/gp.py:278-280). The fused device evaluation has already reduced it to
    the kernel's parameter gradients; this handle carries them (keyed by the kernel state they were computed for)
    and only materialises the matrix (2 GiB at N=16384) if somebody treats it as an ndarray."""

    def __init__(self, engine, key, dvariance, dlengthscale, N, part_grads=None, X=None):
        self._engine, self._key = engine, key
        self.dvariance, self.dlengthscale = dvariance, dlengthscale
        self.part_grads = part_grads          # composite kernels: one [variance, lengthscale..] array per flattened part
        self.shape = (N, N)
        self.ndim = 2
        self.dtype = np.dtype(np.float64)
        self._host = None
        self._X = X                           # a private copy of the inputs the engine evaluated on (None: unknown)
        self._serial = getattr(engine, "eval_serial", None)
        self._dX = None

    def matches(self, key):
        return self._key == key

    def grad_X(self, key, X):
        """kern.gradients_X(dL_dK, X, None) from the device (gpx_exact_grad_X, fetched once per handle) when this is the
        dL_dK of the engine's current evaluation of the kernel keyed `key` on exactly these inputs X (the kernel's columns
        as the engine holds them); None otherwise"""
        if self._X is None or not self.matches(key) or getattr(self._engine, "eval_serial", None) != self._serial:
            return None
        X = np.asarray(X)
        if X.shape != self._X.shape or not np.array_equal(X, self._X):
            return None
        if self._dX is None:
            self._dX = self._engine.exact_grad_X()
        return self._dX

    def __array__(self, dtype=None, copy=None):
        if self._host is None:
            self._host = np.ascontiguousarray(self._engine.get("dL_dK"))  # symmetric: C == F order
        return self._host if dtype is None else self._host.astype(dtype)

    def __getitem__(self, idx):
        return self.__array__()[idx]


class Kern(Parameterized):
    """Subset of GPy.kern.Kern (kern.py:12-145) the exact-GP path uses: active_dims slicing + the abstract plugin
    methods."""

    def __init__(self, input_dim, active_dims, name):
        super(Kern, self).__init__(name)
        self.input_dim = int(input_dim)
        if active_dims is None:
            active_dims = np.arange(self.input_dim)
        self.active_dims = np.atleast_1d(np.asarray(active_dims, dtype=np.int64))
        assert self.active_dims.size == self.input_dim, "input_dim=%d does not match len(active_dim)=%d" % (
            self.input_dim, self.active_dims.size)

    def _slice_X(self, X):
        """kern.py:112-117: column-select the active dims and cast to float."""
        X = np.asarray(X)
        if X.shape[1] == self.input_dim and np.array_equal(self.active_dims, np.arange(self.input_dim)):
            return np.ascontiguousarray(X, dtype=np.float64)
        return np.ascontiguousarray(X[:, self.active_dims], dtype=np.float64)

    def K(self, X, X2=None):
        raise NotImplementedError

    def Kdiag(self, X):
        raise NotImplementedError

    def update_gradients_full(self, dL_dK, X, X2=None):
        raise NotImplementedError

    # kern.py:311-360: operator overloading builds combination kernels
    def __add__(self, other):
        return self.add(other)

    def add(self, other, name="sum"):
        assert isinstance(other, Kern), "only kernels can be added to kernels..."
        return Add([self, other], name=name)

    def __mul__(self, other):
        return self.prod(other)

    def prod(self, other, name="mul"):
        assert isinstance(other, Kern), "only kernels can be multiplied to kernels..."
        return Prod([self, other], name)

    @property
    def is_fixed(self):
        ps = self.flattened_parameters()
        return bool(ps) and all(p.is_fixed for p in ps)


class Stationary(Kern):
    """GPy.kern.src.stationary.Stationary (stationary.py:23-243): variance + (ARD) lengthscale, K = K_of_r(r)."""

    _kind = None

    def __init__(self, input_dim, variance=1., lengthscale=None, ARD=False, active_dims=None, name="stationary"):
        super(Stationary, self).__init__(input_dim, active_dims, name)
        self.ARD = bool(ARD)
        # stationary.py:61-77: default / shape checking of the lengthscale
        if not ARD:
            if lengthscale is None:
                lengthscale = np.ones(1)
            else:
                lengthscale = np.asarray(lengthscale, dtype=np.float64)
                assert lengthscale.size == 1, "Only 1 lengthscale needed for non-ARD kernel"
        else:
            if lengthscale is not None:
                lengthscale = np.asarray(lengthscale, dtype=np.float64)
                assert lengthscale.size in [1, input_dim], "Bad number of lengthscales"
                if lengthscale.size != input_dim:
                    lengthscale = np.ones(input_dim) * lengthscale
            else:
                lengthscale = np.ones(self.input_dim)
        self.lengthscale = Param("lengthscale", lengthscale)
        self.variance = Param("variance", variance)
        assert self.variance.size == 1
        self.link_parameters(self.variance, self.lengthscale)  # stationary.py:81

    # -- state key used to recognise gradients precomputed by the fused evaluation ------------------------------
    def _state_key(self):
        return (self._kind, self.ARD, float(self.variance[0]), tuple(self.lengthscale.values.tolist()),
                tuple(self.active_dims.tolist()))

    def _theta(self):
        ls = self.lengthscale.values if self.ARD else self.lengthscale.values[0]
        return self._kind, self.ARD, float(self.variance[0]), ls

    # -- plugin interface -------------------------------------------------------------------------------------
    def K(self, X, X2=None):
        """stationary.py:105-115 -> gpx_kern_K."""
        X = self._slice_X(X)
        X2 = None if X2 is None else self._slice_X(X2)
        kind, ard, var, ls = self._theta()
        return _ffi.kern_K(kind, ard, var, ls, X, X2)

    def Kdiag(self, X):
        """stationary.py:170-173 -> gpx_kern_Kdiag."""
        return _ffi.kern_Kdiag(self._kind, float(self.variance[0]), int(np.asarray(X).shape[0]))

    def update_gradients_full(self, dL_dK, X, X2=None, reset=True):
        """stationary.py:193-213. A DeviceGradient handle from our ExactGaussianInference short-circuits to the
        gradients the fused epilogue already reduced on the device; any other dL_dK goes through gpx_kern_grad_full."""
        if isinstance(dL_dK, DeviceGradient) and X2 is None and dL_dK.matches(self._state_key()):
            self.variance.gradient = np.atleast_1d(dL_dK.dvariance)
            self.lengthscale.gradient = np.atleast_1d(dL_dK.dlengthscale).copy()
            return
        Xs = self._slice_X(X)
        X2s = None if X2 is None else self._slice_X(X2)
        kind, ard, var, ls = self._theta()
        dv, dl = _ffi.kern_grad_full(kind, ard, var, ls, Xs, np.asarray(dL_dK, dtype=np.float64), X2s)
        self.variance.gradient = np.atleast_1d(dv)
        self.lengthscale.gradient = np.atleast_1d(dl)

    def gradients_X(self, dL_dK, X, X2=None):
        """stationary.py:245-252 -> gpx_kern_grad_X (needed by inducing-point / latent-variable models). The DeviceGradient of
        this kernel's exact evaluation on X is reduced on the device from what the evaluation stored (gpx_exact_grad_X):
        dL_dK is never formed on the host."""
        Xs = self._slice_X(X)
        X2s = None if X2 is None else self._slice_X(X2)
        g = device_grad_X(self, dL_dK, Xs, X2, self._state_key())
        if g is None:
            kind, ard, var, ls = self._theta()
            g = _ffi.kern_grad_X(kind, ard, var, ls, Xs, np.asarray(dL_dK, dtype=np.float64), X2s)
        if Xs.shape[1] == np.asarray(X).shape[1]:
            return g
        full = np.zeros(np.asarray(X).shape)       # kernel_slice_operations.py:138-150: scatter into the full X
        full[:, self.active_dims] = g
        return full

    def gradients_X_diag(self, dL_dKdiag, X):
        """stationary.py:368-369."""
        return np.zeros(np.asarray(X).shape)

    def update_gradients_diag(self, dL_dKdiag, X):
        """stationary.py:182-192."""
        self.variance.gradient = np.atleast_1d(np.sum(dL_dKdiag))
        self.lengthscale.gradient = np.zeros_like(self.lengthscale.values)

    def reset_gradients(self):
        """stationary.py:175-180."""
        self.variance.gradient = np.zeros(1)
        self.lengthscale.gradient = np.zeros_like(self.lengthscale.values)


class RBF(Stationary):
    """GPy.kern.RBF (rbf.py:13-52): k(r) = variance * exp(-0.5 r^2)."""
    _kind = "rbf"

    def __init__(self, input_dim, variance=1., lengthscale=None, ARD=False, active_dims=None, name="rbf"):
        super(RBF, self).__init__(input_dim, variance, lengthscale, ARD, active_dims, name)


class Exponential(Stationary):
    """GPy.kern.Exponential (stationary.py:378-386): k(r) = variance * exp(-r)."""
    _kind = "exponential"

    def __init__(self, input_dim, variance=1., lengthscale=None, ARD=False, active_dims=None, name="Exponential"):
        super(Exponential, self).__init__(input_dim, variance, lengthscale, ARD, active_dims, name)


class Matern32(Stationary):
    """GPy.kern.Matern32 (stationary.py:457-492)."""
    _kind = "matern32"

    def __init__(self, input_dim, variance=1., lengthscale=None, ARD=False, active_dims=None, name="Mat32"):
        super(Matern32, self).__init__(input_dim, variance, lengthscale, ARD, active_dims, name)


class Matern52(Stationary):
    """GPy.kern.Matern52 (stationary.py:556-589)."""
    _kind = "matern52"

    def __init__(self, input_dim, variance=1., lengthscale=None, ARD=False, active_dims=None, name="Mat52"):
        super(Matern52, self).__init__(input_dim, variance, lengthscale, ARD, active_dims, name)


class _PartKern(object):
    """RatQuad and StdPeriodic: evaluated on the device as composite parts (gpx_exact_eval_multi inside a model,
    gpx_kern_part_K / gpx_kern_part_grad_full stand-alone). Subclasses give their descriptor extra and gradient block."""

    def part_desc(self, dims, term):
        """(kind, ARD, term, dims, variance, lengthscale, extra) for Engine.exact_eval_multi"""
        ls = self.lengthscale.values if self._ard_ls() else self.lengthscale.values[0]
        return (self._kind, self._ard_ls(), term, list(dims), float(self.variance[0]), ls, self._extra())

    def K(self, X, X2=None):
        X = self._slice_X(X)
        X2 = None if X2 is None else self._slice_X(X2)
        return _ffi.kern_part_K(self.part_desc(range(self.input_dim), 0), X, X2)

    def Kdiag(self, X):
        return _ffi.kern_Kdiag(self._kind, float(self.variance[0]), int(np.asarray(X).shape[0]))

    def update_gradients_full(self, dL_dK, X, X2=None, reset=True):
        """A DeviceGradient handle of a fused evaluation of this kernel hands over the block the device reduced; any other
        dL_dK goes through gpx_kern_part_grad_full."""
        if X2 is None and scatter_part_gradients(self, dL_dK):
            return
        Xs = self._slice_X(X)
        X2s = None if X2 is None else self._slice_X(X2)
        self._set_gradients(_ffi.kern_part_grad_full(self.part_desc(range(self.input_dim), 0), Xs,
                                                     np.asarray(dL_dK, dtype=np.float64), X2s))

    def gradients_X(self, dL_dK, X, X2=None):
        raise NotImplementedError("%s.gradients_X: the device has no input-gradient kernel for this kind yet" % type(self).__name__)

    def gradients_X_diag(self, dL_dKdiag, X):
        return np.zeros(np.asarray(X).shape)


class RatQuad(_PartKern, Stationary):
    """GPy.kern.RatQuad (stationary.py:747-802): k(r) = variance (1 + r^2/2)^-power."""
    _kind = "ratquad"

    def __init__(self, input_dim, variance=1., lengthscale=None, power=2., ARD=False, active_dims=None, name="RatQuad"):
        super(RatQuad, self).__init__(input_dim, variance, lengthscale, ARD, active_dims, name)
        self.power = Param("power", power)
        self.link_parameter(self.power)                   # stationary.py:760: after variance, lengthscale

    def _ard_ls(self):
        return self.ARD

    def _extra(self):
        return {"power": float(self.power[0])}

    def _state_key(self):
        return Stationary._state_key(self) + (float(self.power[0]),)

    def _set_gradients(self, g):
        self.variance.gradient = np.atleast_1d(g[0])
        self.lengthscale.gradient = np.atleast_1d(g[1:-1]).copy()
        self.power.gradient = np.atleast_1d(g[-1])

    def update_gradients_diag(self, dL_dKdiag, X):
        """stationary.py:800-802."""
        Stationary.update_gradients_diag(self, dL_dKdiag, X)
        self.power.gradient = np.zeros(1)

    def reset_gradients(self):
        Stationary.reset_gradients(self)
        self.power.gradient = np.zeros(1)


class StdPeriodic(_PartKern, Kern):
    """GPy.kern.StdPeriodic (standard_periodic.py:21-94): k = variance exp(-1/2 sum_q (sin(pi (x_q - x'_q) / T_q) / l_q)^2).
    ARD1: one period per dim; ARD2: one lengthscale per dim."""
    _kind = "stdperiodic"

    def __init__(self, input_dim, variance=1., period=None, lengthscale=None, ARD1=False, ARD2=False, active_dims=None,
                 name="std_periodic"):
        super(StdPeriodic, self).__init__(input_dim, active_dims, name)
        self.ARD1, self.ARD2 = bool(ARD1), bool(ARD2)
        # standard_periodic.py:62-84
        if not self.ARD1:
            if period is not None:
                period = np.asarray(period, dtype=np.float64)
                assert period.size == 1, "Only one period needed for non-ARD kernel"
            else:
                period = np.ones(1)
        else:
            if period is not None:
                period = np.asarray(period, dtype=np.float64)
                assert period.size == input_dim, "bad number of periods"
            else:
                period = np.ones(input_dim)
        if not self.ARD2:
            if lengthscale is not None:
                lengthscale = np.asarray(lengthscale, dtype=np.float64)
                assert lengthscale.size == 1, "Only one lengthscale needed for non-ARD kernel"
            else:
                lengthscale = np.ones(1)
        else:
            if lengthscale is not None:
                lengthscale = np.asarray(lengthscale, dtype=np.float64)
                assert lengthscale.size == input_dim, "bad number of lengthscales"
            else:
                lengthscale = np.ones(input_dim)
        self.variance = Param("variance", variance)
        assert self.variance.size == 1, "Variance size must be one"
        self.period = Param("period", period)
        self.lengthscale = Param("lengthscale", lengthscale)
        self.link_parameters(self.variance, self.period, self.lengthscale)   # standard_periodic.py:94

    def _ard_ls(self):
        return self.ARD2

    def _extra(self):
        return {"period": self.period.values.copy() if self.ARD1 else float(self.period[0]), "ARD_period": self.ARD1}

    def _state_key(self):
        return (self._kind, self.ARD1, self.ARD2, float(self.variance[0]), tuple(self.period.values.tolist()),
                tuple(self.lengthscale.values.tolist()), tuple(self.active_dims.tolist()))

    def _set_gradients(self, g):
        npd = self.period.size
        self.variance.gradient = np.atleast_1d(g[0])
        self.period.gradient = np.atleast_1d(g[1:1 + npd]).copy()
        self.lengthscale.gradient = np.atleast_1d(g[1 + npd:]).copy()

    def update_gradients_diag(self, dL_dKdiag, X):
        """standard_periodic.py:544-548."""
        self.variance.gradient = np.atleast_1d(np.sum(dL_dKdiag))
        self.period.gradient = np.zeros_like(self.period.values)
        self.lengthscale.gradient = np.zeros_like(self.lengthscale.values)

    def reset_gradients(self):
        self.variance.gradient = np.zeros(1)
        self.period.gradient = np.zeros_like(self.period.values)
        self.lengthscale.gradient = np.zeros_like(self.lengthscale.values)


SINGLE_KINDS = ("rbf", "exponential", "matern32", "matern52")


def single_kernel(kern):
    """True for a kernel the single-kernel device evaluation takes (gpx_exact_eval and friends): RBF .. Matern52. RatQuad is
    a Stationary too, but only the composite evaluation knows it."""
    return isinstance(kern, Stationary) and kern._kind in SINGLE_KINDS


def part_ngrad(leaf):
    """gradient entries of one flattened leaf in the result of Engine.exact_eval_multi"""
    if isinstance(leaf, _PartKern):
        return sum(p.size for p in leaf.flattened_parameters())
    return 1 + (leaf.lengthscale.size if isinstance(leaf, Stationary) else 0)


# ----------------------------------------------------------------------------------------------------------------------
# combination / static kernels (SURVEY.md §8f item 4). Mirrors GPy/kern/src/add.py:60-99, prod.py:59-68,377-396,
# static.py:63-185. A GP whose kernel is a sum of products of stationary / White / Bias leaves is evaluated by ONE device
# call (gpx_exact_eval_multi: the K-build multiplies / adds the parts in registers, every part's gradient is reduced from
# the stored K^-1 with the other factors of its term recomputed on the fly); `flatten_parts` is the translation.
# The stand-alone K / update_gradients_full methods below (foreign dL_dK, nested structures the flattening does not cover)
# build the parts' matrices on the device and do the O(N^2) glue in NumPy on the host.
# ----------------------------------------------------------------------------------------------------------------------
def flatten_parts(kern):
    """-> list of (leaf kernel, term index) for a kernel that is a leaf, a product of leaves, or a sum of those; None for
    anything else (e.g. a product containing a sum), which then takes the generic inference path."""
    def leaf(k):
        return isinstance(k, (Stationary, StdPeriodic, White, Bias))

    def product(k, term):
        if leaf(k):
            return [(k, term)]
        if isinstance(k, Prod) and all(leaf(q) for q in k.parts):
            return [(q, term) for q in k.parts]
        return None

    if isinstance(kern, Add):
        out = []
        for t, part in enumerate(kern.parts):
            fl = product(part, t)
            if fl is None:
                return None
            out.extend(fl)
        return out
    return product(kern, 0)


def part_descriptor(leaf, term):
    """(kind, ARD, term, dims, variance, lengthscale[, extra]) of one leaf for Engine.exact_eval_multi"""
    if isinstance(leaf, _PartKern):
        return leaf.part_desc(leaf.active_dims.tolist(), term)
    if isinstance(leaf, White):
        return ("white", False, term, [], float(leaf.variance[0]), None)
    if isinstance(leaf, Bias):
        return ("bias", False, term, [], float(leaf.variance[0]), None)
    kind, ard, var, ls = leaf._theta()
    return (kind, ard, term, leaf.active_dims.tolist(), var, ls)


def composite_state_key(kern):
    fl = flatten_parts(kern)
    if fl is None:
        return None
    return tuple((t, type(k).__name__, float(k.variance[0]),
                  tuple(k.lengthscale.values.tolist()) if isinstance(k, Stationary) else (),
                  tuple(k.active_dims.tolist())) + ((k._state_key(),) if isinstance(k, _PartKern) else ()) for (k, t) in fl)


def device_grad_X(kern, dL_dK, X, X2, key):
    """kern.gradients_X(dL_dK, X, X2) from the device, or None: only X2 = None with the DeviceGradient of the engine's
    current exact evaluation of kern (state key `key`) on exactly X, and only for leaves with a device input gradient
    (RatQuad / StdPeriodic have none)"""
    if X2 is not None or not isinstance(dL_dK, DeviceGradient):
        return None
    leaves = flatten_parts(kern)
    if leaves is None or any(isinstance(k, _PartKern) for k, _ in leaves):
        return None
    return dL_dK.grad_X(key, X)


def scatter_part_gradients(kern, dL_dK):
    """hand the per-part gradients of a fused composite evaluation to the leaves (what Add / Prod.update_gradients_full do
    with a dense dL_dK); -> False if the handle does not belong to this kernel state"""
    if not (isinstance(dL_dK, DeviceGradient) and dL_dK.part_grads is not None and dL_dK.matches(composite_state_key(kern))):
        return False
    scatter_leaf_gradients(flatten_parts(kern), dL_dK.part_grads)
    return True


def scatter_leaf_gradients(leaves, part_grads):
    """set each flattened leaf's gradient from its block of a composite device evaluation (paramz order)"""
    for (leaf, _), g in zip(leaves, part_grads):
        if isinstance(leaf, _PartKern):
            leaf._set_gradients(g)
            continue
        leaf.variance.gradient = np.atleast_1d(g[0])
        if isinstance(leaf, Stationary):
            leaf.lengthscale.gradient = np.atleast_1d(g[1:]).copy()



class CombinationKernel(Kern):
    """GPy.kern.src.kern.CombinationKernel (kern.py:363-451): a kernel made of parts; active dims = union."""

    def __init__(self, kernels, name):
        assert all(isinstance(p, Kern) for p in kernels)
        input_dim = int(max(int(np.max(p.active_dims)) for p in kernels) + 1)
        super(CombinationKernel, self).__init__(input_dim, np.arange(input_dim), name)
        self.parts = list(kernels)
        for p in self.parts:
            self.link_parameter(p)

    def _slice_X(self, X):
        return np.ascontiguousarray(X, dtype=np.float64)


class Add(CombinationKernel):
    """GPy.kern.Add (add.py:11-86)."""

    def __init__(self, subkerns, name="sum"):
        flat = []
        for s in subkerns:                       # add.py:20-27: nested sums are flattened
            flat.extend(s.parts if isinstance(s, Add) else [s])
        super(Add, self).__init__(flat, name)

    def K(self, X, X2=None):
        out = None
        for p in self.parts:
            Kp = p.K(X, X2)
            out = Kp if out is None else out + Kp
        return out

    def Kdiag(self, X):
        return sum(p.Kdiag(X) for p in self.parts)

    def update_gradients_full(self, dL_dK, X, X2=None):
        if X2 is None and scatter_part_gradients(self, dL_dK):
            return
        dL_dK = np.asarray(dL_dK, dtype=np.float64)
        for p in self.parts:
            if not p.is_fixed:
                p.update_gradients_full(dL_dK, X, X2)

    def update_gradients_diag(self, dL_dKdiag, X):
        for p in self.parts:
            p.update_gradients_diag(dL_dKdiag, X)

    def gradients_X(self, dL_dK, X, X2=None):
        """add.py:88-100; the DeviceGradient of this kernel's exact evaluation on X: one gpx_exact_grad_X for the sum"""
        g = device_grad_X(self, dL_dK, X, X2, composite_state_key(self))
        if g is not None:
            return g
        return sum(p.gradients_X(dL_dK, X, X2) for p in self.parts)

    def gradients_X_diag(self, dL_dKdiag, X):
        """add.py:102-105"""
        target = np.zeros(np.asarray(X).shape)
        for p in self.parts:
            target += p.gradients_X_diag(dL_dKdiag, X)
        return target


class Prod(CombinationKernel):
    """GPy.kern.Prod (prod.py:23-110)."""

    def __init__(self, kernels, name="mul"):
        flat = []
        for s in kernels:
            flat.extend(s.parts if isinstance(s, Prod) else [s])
        super(Prod, self).__init__(flat, name)

    def K(self, X, X2=None):
        out = None
        for p in self.parts:
            Kp = p.K(X, X2)
            out = Kp if out is None else out * Kp
        return out

    def Kdiag(self, X):
        out = None
        for p in self.parts:
            Kp = p.Kdiag(X)
            out = Kp if out is None else out * Kp
        return out

    def update_gradients_full(self, dL_dK, X, X2=None):
        """prod.py:377-385: each part sees dL_dK times the product of the other parts."""
        if X2 is None and scatter_part_gradients(self, dL_dK):
            return
        dL_dK = np.asarray(dL_dK, dtype=np.float64)
        Ks = [p.K(X, X2) for p in self.parts]
        for i, p in enumerate(self.parts):
            other = None
            for j, Kj in enumerate(Ks):
                if j != i:
                    other = Kj if other is None else other * Kj
            p.update_gradients_full(dL_dK * other if other is not None else dL_dK, X, X2)

    def gradients_X(self, dL_dK, X, X2=None):
        """prod.py:397-407; the DeviceGradient of this kernel's exact evaluation on X: one gpx_exact_grad_X"""
        g = device_grad_X(self, dL_dK, X, X2, composite_state_key(self))
        if g is not None:
            return g
        dL_dK = np.asarray(dL_dK, dtype=np.float64)
        Ks = [p.K(X, X2) for p in self.parts]
        out = 0.0
        for i, p in enumerate(self.parts):
            other = None
            for j, Kj in enumerate(Ks):
                if j != i:
                    other = Kj if other is None else other * Kj
            out = out + p.gradients_X(dL_dK * other if other is not None else dL_dK, X, X2)
        return out

    def gradients_X_diag(self, dL_dKdiag, X):
        """prod.py:409-418"""
        target = np.zeros(np.asarray(X).shape)
        if len(self.parts) == 2:
            target += self.parts[0].gradients_X_diag(dL_dKdiag * self.parts[1].Kdiag(X), X)
            target += self.parts[1].gradients_X_diag(dL_dKdiag * self.parts[0].Kdiag(X), X)
        else:
            k = self.Kdiag(X) * dL_dKdiag
            for p in self.parts:
                target += p.gradients_X_diag(k / p.Kdiag(X), X)
        return target


class Static(Kern):
    """GPy.kern.src.static.Static (static.py:11-61): a variance parameter, no dependence on X."""

    def __init__(self, input_dim, variance, active_dims, name):
        super(Static, self).__init__(input_dim, active_dims, name)
        self.variance = Param("variance", variance)
        self.link_parameter(self.variance)

    def Kdiag(self, X):
        ret = np.empty((np.asarray(X).shape[0],), dtype=np.float64)
        ret[:] = self.variance[0]
        return ret

    def gradients_X(self, dL_dK, X, X2=None):
        return np.zeros(np.asarray(X).shape)

    def gradients_X_diag(self, dL_dKdiag, X):
        """static.py:30-31"""
        return np.zeros(np.asarray(X).shape)

    def update_gradients_diag(self, dL_dKdiag, X):
        self.variance.gradient = np.atleast_1d(np.sum(dL_dKdiag))


class White(Static):
    """GPy.kern.White (static.py:63-99)."""

    def __init__(self, input_dim, variance=1., active_dims=None, name="white"):
        super(White, self).__init__(input_dim, variance, active_dims, name)

    def K(self, X, X2=None):
        n = np.asarray(X).shape[0]
        if X2 is None:
            return np.eye(n) * self.variance[0]
        return np.zeros((n, np.asarray(X2).shape[0]))

    def update_gradients_full(self, dL_dK, X, X2=None):
        self.variance.gradient = np.atleast_1d(np.trace(np.asarray(dL_dK)) if X2 is None else 0.)


class Bias(Static):
    """GPy.kern.Bias (static.py:142-185)."""

    def __init__(self, input_dim, variance=1., active_dims=None, name="bias"):
        super(Bias, self).__init__(input_dim, variance, active_dims, name)

    def K(self, X, X2=None):
        shape = (np.asarray(X).shape[0], np.asarray(X).shape[0] if X2 is None else np.asarray(X2).shape[0])
        return np.full(shape, self.variance[0], dtype=np.float64)

    def update_gradients_full(self, dL_dK, X, X2=None):
        self.variance.gradient = np.atleast_1d(np.asarray(dL_dK).sum())
