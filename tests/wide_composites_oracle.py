"""Test-only helpers for the wide composite kernels: a Python restatement of how the device picks its kernel
instantiations (register width DREG, channels per launch NCH, column chunks), an oracle for composites that mixes every
kind (tests/periodic_oracle.py's RatQuad / StdPeriodic beside oracle/gpy_oracle.py's stationary and static kinds), and
the kernels and inputs of tests/test_gpu_wide_composites.py and tests/golden/make_wide_composites.py.

The route restatement mirrors gpx_multi.cu (dreg_for, launch_grad_kinv_multi / launch_grad_full_multi, launch_gradx_multi,
pred_grad_nch, launch_pg_t, pred_grad_launches) and gpx_points.cu (gradx_chunks); tests/test_wide_composites_cpu.py checks
it against the formulas include/gpx.h documents.
"""
import numpy as np

from oracle import gpy_oracle as o
import periodic_oracle as pro

TILE = 128
MAX_D = 64
MAX_PARTS = 8
STATIONARY = ("rbf", "exponential", "matern32", "matern52")


# ---- the device's choice of instantiation -----------------------------------------------------------------------------
def width(d):
    """the register width of the instantiation that holds d accumulators: 8, 16, 32 or 64"""
    assert 0 <= d <= MAX_D, d
    return 8 if d <= 8 else 16 if d <= 16 else 32 if d <= 32 else 64


def ndims(p):
    return 0 if p["kind"] in ("white", "bias") else len(p["dims"])


def part_nacc(p):
    """per-dim register accumulators of a part's gradient pass: ARD lengthscales of a stationary or RatQuad part, period and
    lengthscale of every dim of a StdPeriodic part"""
    if p["kind"] == "stdperiodic":
        return 2 * ndims(p)
    return ndims(p) if (p["kind"] in STATIONARY + ("ratquad",) and p.get("ARD", False)) else 0


def part_nred(p):
    """per-tile partial sums of a part: its gradient entries and tr(dL_dK); three for a static part"""
    if p["kind"] in ("white", "bias"):
        return 3
    d = ndims(p)
    nl = d if p.get("ARD", False) else 1
    if p["kind"] == "ratquad":
        return 2 + nl + 1
    if p["kind"] == "stdperiodic":
        return 1 + (d if p.get("ARD_period", False) else 1) + nl + 1
    return 1 + nl + 1


def has_ext(parts):
    return any(p["kind"] in ("ratquad", "stdperiodic") for p in parts)


def grad_route(parts, i):
    """(DREG, EXT) of grad_kinv_multi_kernel / grad_full_multi_kernel for part i: DREG from max(ndims, nacc)"""
    p = parts[i]
    return width(max(ndims(p), part_nacc(p))), has_ext(parts)


def sum_dims(parts):
    return sum(ndims(p) for p in parts)


def pred_grad_nch(sumD):
    """channels per pred_grad launch: (P + 1) x DREG accumulators where up to 32 fit"""
    return 4 if sumD <= 8 else 2 if sumD <= 16 else 1


def pred_grad_route(sumD):
    """(DREG, NCH) of pred_grad_kernel: <8,4> <16,2> <32,1> <64,1>"""
    return width(max(sumD, 1)), pred_grad_nch(sumD)


def channel_groups(sumD, P):
    """the channel-group launches of launch_pg_t: [(c0, channels, holds the variance channel)]; channel P is the variance"""
    g = pred_grad_nch(sumD)
    out = []
    for c0 in range(0, P + 1, g):
        n = min(g, P + 1 - c0)
        out.append((c0, n, c0 + n == P + 1))
    return out


def pred_grad_launches(sumD, P):
    """R = ceil((P + 1) / g) + 1: the channel-group launches and the reduction"""
    return len(channel_groups(sumD, P)) + 1


def gradx_chunks(nrows, ncols, num_sms):
    """gradx_chunks of gpx_points.cu: the ncols column points split into chunks so that ~4 waves of CTAs (128 row points
    each) are in flight -> (chunks, chunk length, length of the last chunk)"""
    ntile = -(-nrows // TILE)
    n = max(1, min(-(-ncols // 32), -(-(4 * num_sms) // ntile)))
    mchunk = -(-(-(-ncols // n)) // 32) * 32
    nchunk = -(-ncols // mchunk)
    return nchunk, mchunk, ncols - (nchunk - 1) * mchunk


# ---- an oracle for composites of every kind ---------------------------------------------------------------------------
class _RowBlocks(object):
    """a RatQuad / StdPeriodic oracle evaluated over blocks of rows: the StdPeriodic restatement forms N x M x D arrays, and
    its sums are linear in the rows of dL_dK, so the blocks add up to the same reduction"""

    def __init__(self, k, rows=256):
        self.k, self.rows = k, rows

    def K(self, X, X2=None):
        X2f = X if X2 is None else X2
        if X2 is None and not isinstance(self.k, pro.StdPeriodicOracle):
            return self.k.K(X)
        return np.concatenate([self.k.K(X[i:i + self.rows], X2f) for i in range(0, X.shape[0], self.rows)], 0)

    def Kdiag(self, X):
        return self.k.Kdiag(X)

    def update_gradients_full(self, dL_dK, X, X2=None):
        if X2 is None and not isinstance(self.k, pro.StdPeriodicOracle):
            return self.k.update_gradients_full(dL_dK, X)
        X2f = X if X2 is None else X2
        return sum(self.k.update_gradients_full(dL_dK[i:i + self.rows], X[i:i + self.rows], X2f)
                   for i in range(0, X.shape[0], self.rows))


def make_part(p):
    """part dict -> (oracle kernel, dims, term) with update_gradients_full returning the part's whole gradient block"""
    k, dims, term = pro.make_part(p)
    if p["kind"] in ("ratquad", "stdperiodic"):
        k = _RowBlocks(k)
    elif p["kind"] in STATIONARY:   # no identity-keyed memo: every call here slices fresh inputs, and N x N results add up
        k.k._memo = lambda tag, X, X2, fn: fn()
    return k, dims, term


class WideOracle(object):
    """K, Kdiag, the gradient blocks (update_gradients_full through Add / Prod, add.py:76-77, prod.py:377-385) and
    gradients_X (add.py:88-100, prod.py:397-407, stationary.py:245-252; the stationary kinds RBF .. Matern52 only) of a
    composite of any parts, as sparse_composite_oracle.CompositeOracle states them for the stationary and static kinds."""

    def __init__(self, parts):
        self.parts = parts
        self.kparts = [make_part(p) for p in parts]

    def K(self, X, X2=None):
        return o.composite_K(self.kparts, X, X2)

    def Kdiag(self, X):
        return o.composite_Kdiag(self.kparts, X)

    def _others(self, i, X, X2):
        out = None
        t = self.kparts[i][2]
        for j, (k, dims, tj) in enumerate(self.kparts):
            if j != i and tj == t:
                v = k.K(o._slice(X, dims), None if X2 is None else o._slice(X2, dims))
                out = v if out is None else out * v
        return out

    def grads_full(self, dL_dK, X, X2=None):
        """-> the concatenated gradient blocks of every part, in order"""
        blocks = []
        for i, (k, dims, _) in enumerate(self.kparts):
            other = self._others(i, X, X2)
            g = dL_dK if other is None else dL_dK * other
            blocks.append(k.update_gradients_full(g, o._slice(X, dims), None if X2 is None else o._slice(X2, dims)))
        return np.concatenate(blocks)

    def gradients_X(self, dL_dK, X, X2=None):
        out = np.zeros(X.shape)
        for i, (k, dims, _) in enumerate(self.kparts):
            if self.parts[i]["kind"] not in STATIONARY:
                assert self.parts[i]["kind"] in ("white", "bias"), "no input gradient for " + self.parts[i]["kind"]
                continue
            other = self._others(i, X, X2)
            g = dL_dK if other is None else dL_dK * other
            out[:, dims] += k.k.gradients_X(g, o._slice(X, dims), None if X2 is None else o._slice(X2, dims))
        return out


def exact_eval(X, Y, parts, noise):
    """one GP.parameters_changed() with the composite (exact_gaussian_inference.py:37-74) -> (lml, grad [blocks, noise],
    res dict(L, alpha, Wi, dL_dK, Ky))"""
    kern = WideOracle(parts)
    K = kern.K(X)
    Ky = K.copy()
    o.diag_add(Ky, noise + 1e-8)
    Wi, L, _, logdet = o.pdinv(Ky)
    alpha, _ = o.dpotrs(L, Y, lower=1)
    lml = 0.5 * (-Y.size * np.log(2 * np.pi) - Y.shape[1] * logdet - np.sum(alpha * Y))
    dL_dK = 0.5 * (o.tdot(alpha) - Y.shape[1] * Wi)
    grad = np.concatenate([kern.grads_full(dL_dK, X), [np.trace(dL_dK)]])
    return float(lml), grad, dict(L=L, alpha=alpha, Wi=Wi, dL_dK=dL_dK, Ky=Ky, kern=kern)


# ---- kernels and inputs -----------------------------------------------------------------------------------------------
def ls_for(d, scale=1.3):
    """a lengthscale ~ sqrt(part dims): on U(-2, 2) inputs the scaled distances stay O(1), so K is not nearly diagonal"""
    return scale * np.sqrt(d)


def stationary(kind, dims, term, ARD, variance=1.0, scale=1.3):
    d = len(dims)
    ls = ls_for(d, scale) * np.linspace(0.8, 1.25, d) if ARD else ls_for(d, scale)
    return dict(kind=kind, term=term, dims=list(dims), variance=variance, lengthscale=ls, ARD=ARD)


def ratquad(dims, term, ARD, power=0.9, variance=1.0):
    p = stationary("rbf", dims, term, ARD, variance)
    p.update(kind="ratquad", power=power)
    return p


def stdperiodic(dims, term, ARD1, ARD2, variance=1.0):
    """on U(-2, 2) inputs, periods between 2 and 4 keep the arguments pi d / T spread over a whole period; lengthscales
    ~ sqrt(dims) keep the exponent O(1)"""
    d = len(dims)
    T = np.linspace(2.0, 4.0, d) if ARD1 else 3.1
    ls = 0.75 * np.sqrt(d) * np.linspace(0.8, 1.25, d) if ARD2 else 0.75 * np.sqrt(d)
    return dict(kind="stdperiodic", term=term, dims=list(dims), variance=variance, period=T, lengthscale=ls, ARD=ARD2,
                ARD_period=ARD1)


def static(kind, term, variance):
    return dict(kind=kind, term=term, variance=variance)


def perm(D, seed):
    """the columns 0..D-1 in a fixed random order: stacked rows that are not the data's columns in order"""
    return [int(i) for i in np.random.default_rng(seed).permutation(D)]


def data(N, D, P, seed):
    """X ~ U(-2, 2)^D, Y = sin of a few columns' sum (one phase per output) + 0.1 eps"""
    rng = np.random.default_rng(seed)
    X = rng.uniform(-2.0, 2.0, (N, D))
    Y = np.sin(X[:, :min(D, 5)].sum(1, keepdims=True) / np.sqrt(min(D, 5)) + np.arange(P)) \
        + 0.1 * rng.standard_normal((N, P))
    return X, Y


def spread_points(X, M, offset=0.01):
    """M rows of X by farthest-point selection (inducing points that keep cond(Kmm) low), moved off the data by `offset`
    times a fixed normal draw: at a data point r comes from the cancellation in |x|^2 + |z|^2 - 2 x.z and is ~1e-8 instead
    of 0 on either side, which the Exponential kernel (not smooth at r = 0) passes on to Knm at first order"""
    idx = [0]
    d = np.linalg.norm(X - X[0], axis=1)
    for _ in range(M - 1):
        i = int(np.argmax(d))
        idx.append(i)
        d = np.minimum(d, np.linalg.norm(X - X[i], axis=1))
    return X[idx] + offset * np.random.default_rng(M).standard_normal((M, X.shape[1]))


def descriptor(p):
    """the part as Engine.exact_eval_multi / sparse_eval_multi / kern_part_* take it"""
    return pro.descriptor(p)


def mirror_kernel(parts, D):
    """the mirror's kernel object (gpy_b200) for part dicts of the stationary and static kinds: Add over terms of Prod"""
    import gpy_b200
    terms = {}
    for p in parts:
        if p["kind"] in ("white", "bias"):
            k = (gpy_b200.White if p["kind"] == "white" else gpy_b200.Bias)(D, variance=p["variance"])
        else:
            cls = {"rbf": gpy_b200.RBF, "exponential": gpy_b200.Exponential, "matern32": gpy_b200.Matern32,
                   "matern52": gpy_b200.Matern52}[p["kind"]]
            k = cls(len(p["dims"]), variance=p["variance"], lengthscale=p["lengthscale"], ARD=p.get("ARD", False),
                    active_dims=p["dims"])
        terms.setdefault(p["term"], []).append(k)
    ts = [ks[0] if len(ks) == 1 else gpy_b200.Prod(ks) for _, ks in sorted(terms.items())]
    return ts[0] if len(ts) == 1 else gpy_b200.Add(ts)


# the kernels of the reference fixtures (tests/golden/wide_composites), on D = 64 columns
FIXTURE_D = 64


def fixture_kernels():
    P64 = perm(64, 7)
    return {
        "ratquad_ard64": [ratquad(P64, 0, True, power=0.8)],
        "periodic32_x_rbf": [stdperiodic(P64[:32], 0, True, True), stationary("rbf", P64[16:48], 0, True)],
        "eight_parts64": eight_parts(P64),
        "pg_sumd17": [stationary("matern52", P64[:17], 0, True), static("bias", 0, 0.7), static("white", 1, 0.05)],
        "pg_sumd64": [stationary("rbf", P64[:33], 0, True), stationary("matern32", P64[33:41], 0, False),
                      stationary("exponential", P64[41:], 1, True, variance=0.5)],
    }


def eight_parts(cols):
    """eight parts on 8 dims each (sumD 64): every part's gradient pass at DREG 8 while the K-build stacks 64 rows; sums of
    products, iso and ARD, every stationary kind"""
    kinds = ("rbf", "matern52", "matern32", "exponential", "rbf", "matern52", "matern32", "rbf")
    terms = (0, 0, 1, 2, 2, 2, 3, 3)
    return [stationary(k, cols[8 * i:8 * i + 8], terms[i], i % 2 == 0, variance=0.6 + 0.1 * i)
            for i, k in enumerate(kinds)]
