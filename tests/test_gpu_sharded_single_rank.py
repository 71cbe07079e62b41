"""The sharded exact evaluation on one GPU, through a one-rank NCCL communicator.

`gpx_comm_init(ctx, uid, 0, 1)` puts a context on the sharded path of gpx_dist.cu: whole-block padding, the row-owned
workspace, the column-owned U storage (`SU`), the copy-back, `launch_uv_blk`, `launch_finalize_raw`, the collective
`get("L")` and the sharded `predict`, all through a real communicator in this process. tests/test_gpu_dist.py runs the same
path on two GPUs and skips on one; this file is what checks it on a single device.

The sharded layout picks its outer block NB itself (gpx_dist.cu `dist_set_data`): option `nb`, else 256, 512 from
N = 8192, 1024 from N = 32768, capped at N rounded up to 128, and pads the matrix to whole blocks. Each case states its
block count and checks it through `Engine.stats()`:

    update_launches  tries (2 nblk - 3) for nblk >= 2, 0 for one block (U1 for every block but the last, U2 where a block
                     follows block k+1); update_int8_ops 0: the sharded sweep is DMMA only, option `ozaki` has no effect

| case                                        | N, nb -> blocks                                                   |
|---------------------------------------------|-------------------------------------------------------------------|
| one block                                   | 1, 127, 128, 200, 256 (default NB); 100 at nb 128                 |
| second block almost all padding             | 257 (NB 256); 1025 at nb 1024                                     |
| several blocks with a tail                  | 700 (3 x 256), 1025 at nb 128 / 384, 8193 (NB 512: 17 blocks)     |
| ill-conditioned, extended precision         | 1100 (5 blocks), noise 1e-2 / 1e-4 / 1e-6                         |
| jitter ladder                               | 200 (one block), 1200 (failing minor in block 4 of 5)             |
| context reuse                               | N 200 <-> 1025 <-> 1100, D 3 -> 5, P 1 -> 3, nb 256 -> 128        |

Every result is compared with the CPU oracle and with a plain (no communicator) engine on the same data; N = 8193 with the
plain engine only (the oracle takes half a minute there).

NCCL is loaded from the installed `nvidia.nccl` package (GPX_NCCL_LIB, unless set). If it cannot be loaded on a machine
with a device, the tests fail: they never skip for it.
"""
import ctypes
import os

import numpy as np
import pytest

from oracle import gpy_oracle as o
from test_gpu_routes import (GRAD_RTOL, LML_ATOL, NORTH_STAR, data, errors, ill_problem, later_block_singular, ld_case,
                             mean_atol, oracle_errors, rel, theta, var_atol)

ORACLE_MAX_N = 4096


def _ffi():
    from gpy_b200 import _ffi as f
    return f


def sharded_blocks(N, nb=0):
    """outer blocks of the sharded layout for N points (gpx_dist.cu dist_pick_nb / dist_set_data, GPX_NB unset)"""
    from gpy_b200 import dist as gdist
    NB = nb or (1024 if N >= 32768 else 512 if N >= 8192 else 256)
    return gdist.block_layout(N, min(NB, -(-N // 128) * 128), 1)[1]


def assert_blocks(st, nblk, tries=1):
    assert st["update_launches"] == tries * (2 * nblk - 3 if nblk >= 2 else 0), (nblk, st)
    assert st["tries"] == tries, st
    assert st["update_int8_ops"] == 0, st


def nccl_library():
    """libnccl.so.2 of the installed nvidia.nccl package, or None"""
    try:
        import nvidia.nccl
    except ImportError:
        return None
    for d in nvidia.nccl.__path__:
        p = os.path.join(d, "lib", "libnccl.so.2")
        if os.path.isfile(p):
            return p
    return None


def attach(e):
    """a one-rank communicator on engine e (raises when NCCL cannot be loaded or initialised)"""
    f = _ffi()
    if not os.environ.get("GPX_NCCL_LIB") and nccl_library():
        os.environ["GPX_NCCL_LIB"] = nccl_library()
    uid = ctypes.create_string_buffer(128)
    rc = f.lib().gpx_comm_unique_id(uid)
    if rc != 0 and "NCCL_SOCKET_IFNAME" not in os.environ:
        # the bootstrap found no usable network interface; one rank in one process needs only the loopback
        os.environ["NCCL_SOCKET_IFNAME"] = "lo"
        rc = f.lib().gpx_comm_unique_id(uid)
    f.check(rc, "gpx_comm_unique_id")
    f.check(f.lib().gpx_comm_init(e._h, uid.raw, 0, 1), "gpx_comm_init")
    return e


def sharded_engine(nb=0):
    e = attach(_ffi().Engine(0))
    if nb:
        e.set_option("nb", nb)
    return e


def plain_engine():
    e = _ffi().Engine(0)
    e.set_option("ozaki", 0)
    return e


def probes(X, seed, m=64):
    """m points: up to m / 2 training points, the rest new points in the same box"""
    rng = np.random.default_rng(seed)
    k = min(X.shape[0], m // 2)
    return np.concatenate([X[rng.choice(X.shape[0], k, replace=False)], rng.uniform(-3, 3, (m - k, X.shape[1]))])


def evaluate(e, X, Y, kind, ARD, var, ls, noise, Xn, get_L=True):
    lml, g, jit = e.exact_eval(kind, ARD, var, ls, noise)
    r = dict(lml=lml, g=g, jit=jit, stats=e.stats(), alpha=e.get("alpha"), pred=e.predict(Xn),
             cov=e.predict(Xn[:12], full_cov=True))
    if get_L:
        r["L"] = e.get("L")
    return r


def assert_matches(r, lml0, g0, alpha0, L0, mu0, v0, cov0, kind):
    """the tolerances of tests/test_gpu_routes.py (DMMA path)"""
    assert abs(r["lml"] - lml0) <= LML_ATOL, (r["lml"], lml0)
    np.testing.assert_allclose(r["g"], g0, rtol=GRAD_RTOL, atol=1e-9)
    assert rel(r["alpha"], alpha0) < 1e-9
    if L0 is not None:
        assert rel(r["L"], L0) < 1e-10
    np.testing.assert_allclose(r["pred"][0], mu0, rtol=1e-8, atol=mean_atol(kind, alpha0))
    np.testing.assert_allclose(r["pred"][1], v0, rtol=1e-7, atol=var_atol(kind))
    np.testing.assert_allclose(r["cov"][1], cov0, rtol=1e-7, atol=var_atol(kind))


def check_against_oracle(r, X, Y, kind, ARD, var, ls, noise, Xn):
    lml0, g0, res = o.eval_lml_grad(X, Y, kind, ARD, var, ls, noise)
    ko = o.StationaryOracle(kind, X.shape[1], var, ls, ARD)
    mu0, v0 = o.raw_predict(ko, X, res["L"], res["alpha"], Xn)
    _, cov0 = o.raw_predict(ko, X, res["L"], res["alpha"], Xn[:12], full_cov=True)
    assert_matches(r, lml0, g0, res["alpha"], res["L"] if "L" in r else None, mu0, v0, cov0, kind)


# --------------------------------------------------------------------------------------------------------------------
# A. the route matrix of the sharded layout
# --------------------------------------------------------------------------------------------------------------------
# (kind, ARD, N, D, P, option nb, outer blocks)
CASES = [
    ("rbf", True, 1, 1, 1, 0, 1),
    ("matern32", False, 127, 8, 3, 0, 1),
    ("matern52", True, 128, 9, 1, 0, 1),
    ("exponential", True, 200, 64, 8, 0, 1),
    ("rbf", False, 256, 8, 1, 0, 1),
    ("matern52", False, 100, 1, 3, 128, 1),
    ("exponential", False, 257, 9, 1, 0, 2),       # the second block holds one row
    ("rbf", True, 700, 8, 3, 0, 3),                # 3 x 256, tail of 188
    ("matern32", True, 1025, 9, 1, 128, 9),
    ("matern52", True, 1025, 64, 8, 384, 3),
    ("exponential", True, 1025, 1, 3, 1024, 2),    # the second block holds one row
    ("rbf", True, 8193, 8, 1, 0, 17),              # NB 512 by size, 16 x 512 + 1
]


def _ids(c):
    return "%s-%s-N%d-D%d-P%d-nb%d-blk%d" % (c[0], "ard" if c[1] else "iso", c[2], c[3], c[4], c[5], c[6])


def test_case_block_counts():
    """each case's stated block count is what the layout gives"""
    for c in CASES:
        assert sharded_blocks(c[2], c[5]) == c[6], c
    assert [sharded_blocks(n) for n in (200, 1100, 1200, 1700, 2049)] == [1, 5, 5, 7, 9]
    assert [sharded_blocks(n, nb) for n, nb in ((100, 128), (1100, 128), (1025, 128))] == [1, 9, 9]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,ARD,N,D,P,nb,nblk", CASES, ids=[_ids(c) for c in CASES])
def test_sharded_route_matrix(kind, ARD, N, D, P, nb, nblk):
    X, Y = data(N, D, P, seed=N + D)
    var, ls, noise = theta(D, ARD, N + P)
    Xn = probes(X, N)
    e = sharded_engine(nb)
    e.set_data(X, Y)
    r = evaluate(e, X, Y, kind, ARD, var, ls, noise, Xn)
    e.close()
    assert_blocks(r["stats"], nblk)
    assert r["jit"] == 0.0
    p = plain_engine()
    p.set_data(X, Y)
    q = evaluate(p, X, Y, kind, ARD, var, ls, noise, Xn)
    p.close()
    assert_matches(r, q["lml"], q["g"], q["alpha"], q["L"], q["pred"][0], q["pred"][1], q["cov"][1], kind)
    if N <= ORACLE_MAX_N:
        check_against_oracle(r, X, Y, kind, ARD, var, ls, noise, Xn)


# --------------------------------------------------------------------------------------------------------------------
# B. ill-conditioned problems against the extended-precision reference of tests/test_gpu_routes.py
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("noise", [1e-2, 1e-4, 1e-6])
def test_sharded_ill_conditioned_against_extended_precision(noise):
    """device error <= max(north-star tolerance, factor x the fp64 oracle's own error), with the factors of
    test_ill_conditioned_against_extended_precision"""
    X, Y, var, ls, Xn = ill_problem()
    ref = ld_case(noise)
    ora = oracle_errors(noise)
    e = sharded_engine()
    e.set_data(X, Y)
    lml, g, jit = e.exact_eval("rbf", True, var, ls, noise)
    assert jit == 0.0
    assert_blocks(e.stats(), 5)
    _, pv = e.predict(Xn)
    dev = errors(ref, lml, g, e.get("alpha"), pv)
    e.close()
    Ky = o.StationaryOracle("rbf", 2, var, ls, True).K(X) + (noise + 1e-8) * np.eye(X.shape[0])
    cond = float(np.linalg.cond(Ky))
    print("\nsharded extended-precision check noise=%g cond(Ky)=%.2e\n  device %s\n  oracle %s" % (noise, cond, dev, ora))
    for k in NORTH_STAR:
        factor = {"lml": 64, "alpha": 16}.get(k, 4) if cond > 1e8 else 4
        assert dev[k] <= max(NORTH_STAR[k], factor * ora[k]), (k, dev, ora, cond)


# --------------------------------------------------------------------------------------------------------------------
# C. jitter ladder under the communicator
# --------------------------------------------------------------------------------------------------------------------
def _minor(excinfo):
    return int(str(excinfo.value).rsplit("leading minor", 1)[1].strip(" )"))


@pytest.mark.gpu
@pytest.mark.parametrize("N,nblk", [(200, 1), (1200, 5)])
def test_sharded_jitter_ladder(N, nblk):
    """The last 50 inputs repeat the first 50 and the noise is zero: the first non-positive pivot is row 151 (one block) or
    1151 (block 4 of 5). The jitter is GPy's jitchol's, max_tries = 0 raises with the failing minor in the last block, as
    the plain engine does (the sharded `info` is all-reduced with max), and a well-posed theta afterwards matches the
    oracle."""
    X, Y = later_block_singular(N)
    e = sharded_engine()
    e.set_data(X, Y)
    lml, g, jit = e.exact_eval("exponential", False, 1.0, 1.3, 0.0, jitter=0.0)
    assert_blocks(e.stats(), nblk, tries=2)
    Ky = o.StationaryOracle("exponential", 2, 1.0, 1.3, False).K(X)
    L, jit0 = o.jitchol(Ky)
    assert jit0 > 0 and np.isclose(jit, jit0, rtol=1e-12), (jit, jit0)
    alpha = o.dpotrs(L, Y)[0]
    lml0 = 0.5 * (-Y.size * o.LOG_2_PI - 2 * np.sum(np.log(np.diag(L))) - np.sum(alpha * Y))
    assert abs(lml - lml0) <= 2e-4 * abs(lml0)     # cond ~ 1e9: see test_ladder_fails_in_a_later_block
    with pytest.raises(np.linalg.LinAlgError) as sharded_err:
        e.exact_eval("exponential", False, 1.0, 1.3, 0.0, jitter=0.0, max_tries=0)
    assert e.stats()["tries"] == 1
    p = plain_engine()
    p.set_data(X, Y)
    with pytest.raises(np.linalg.LinAlgError) as plain_err:
        p.exact_eval("exponential", False, 1.0, 1.3, 0.0, jitter=0.0, max_tries=0)
    p.close()
    # rows N-50.. repeat rows 0..49: the first failing minor is row N-49 unless rounding leaves that pivot just positive
    for err in (sharded_err, plain_err):
        assert N - 49 <= _minor(err) <= N, str(err.value)
    var, ls, noise = 1.2, np.array([1.1, 1.6]), 0.05
    Xn = probes(X, N)
    r = evaluate(e, X, Y, "matern32", True, var, ls, noise, Xn)
    e.close()
    assert_blocks(r["stats"], nblk)
    assert r["jit"] == 0.0
    check_against_oracle(r, X, Y, "matern32", True, var, ls, noise, Xn)


# --------------------------------------------------------------------------------------------------------------------
# D. determinism, options, context reuse, rejections
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_sharded_same_theta_twice_and_ozaki_option():
    """The same theta twice gives the same bits; option ozaki = 1 leaves the sharded (DMMA-only) evaluation unchanged."""
    X, Y = data(1700, 3, 2, seed=8)
    Xn = probes(X, 8)
    e = sharded_engine()
    e.set_data(X, Y)
    e.set_option("ozaki", 0)
    runs = [evaluate(e, X, Y, "matern32", True, 1.1, np.array([1.2, 1.9, 2.4]), 0.03, Xn) for _ in range(2)]
    e.set_option("ozaki", 1)
    runs.append(evaluate(e, X, Y, "matern32", True, 1.1, np.array([1.2, 1.9, 2.4]), 0.03, Xn))
    e.close()
    for r in runs:
        assert_blocks(r["stats"], 7)
    for r in runs[1:]:
        assert r["lml"] == runs[0]["lml"]
        for k in ("g", "alpha", "L"):
            assert np.array_equal(r[k], runs[0][k]), k
        for k in ("pred", "cov"):
            assert all(np.array_equal(a, b) for a, b in zip(r[k], runs[0][k])), k


@pytest.mark.gpu
def test_sharded_context_reuse():
    """One context: N from one block to several and back, to another N of the same padding, D 3 -> 5, P 1 -> 3 and option
    nb 256 -> 128 between evaluations; every result matches the oracle."""
    X, Y = data(1100, 5, 3, seed=11)
    e = sharded_engine(256)
    steps = [(200, 3, 1, None, 1), (1025, 3, 1, None, 5), (200, 3, 1, None, 1), (1025, 5, 1, None, 5),
             (1025, 5, 3, None, 5), (1100, 5, 3, None, 5), (1100, 5, 3, 128, 9), (100, 5, 3, None, 1),
             (1025, 5, 1, None, 9)]
    for i, (N, D, P, nb, nblk) in enumerate(steps):
        if nb:
            e.set_option("nb", nb)
        Xs, Ys = X[:N, :D], Y[:N, :P]
        e.set_data(Xs, Ys)
        var, ls, noise = theta(D, True, i)
        Xn = probes(Xs, i)
        r = evaluate(e, Xs, Ys, "rbf", True, var, ls, noise, Xn)
        assert_blocks(r["stats"], nblk)
        check_against_oracle(r, Xs, Ys, "rbf", True, var, ls, noise, Xn)
    e.close()


@pytest.mark.gpu
def test_sharded_rejections_leave_the_evaluation_intact():
    """What the sharded context does not support returns -2 and changes nothing that get / predict return."""
    f = _ffi()
    X, Y = data(700, 3, 2, seed=7)
    Xn = probes(X, 7)
    Z = X[::35] + 0.01
    parts = [("rbf", True, 0, [0, 1, 2], 1.1, np.array([1.3, 1.7, 2.1])), ("white", False, 0, [], 0.1, None)]
    e = sharded_engine()
    e.sparse_set_data(X, Y)      # so that the composite sparse evaluation gets as far as its communicator check
    e.set_data(X, Y)
    var, ls, noise = theta(3, True, 7)
    e.exact_eval("matern52", True, var, ls, noise)
    before = dict(alpha=e.get("alpha"), L=e.get("L"), pred=e.predict(Xn), cov=e.predict(Xn[:12], full_cov=True))
    calls = [
        lambda: e.exact_eval_het("matern52", True, var, ls, np.full(700, noise)),
        lambda: e.exact_eval_multi(parts, noise),
        lambda: f.pdinv(o.StationaryOracle("rbf", 3, 1.0, 1.5, False).K(X[:300]) + 0.1 * np.eye(300), engine=e),
        lambda: e.predictive_gradients(Xn),
        lambda: e.sparse_eval_multi(parts, Z, noise),
    ] + [(lambda w=w: e.get(w)) for w in ("Kinv", "dL_dK", "K", "Linv")]
    for i, call in enumerate(calls):
        with pytest.raises(f.GpxArgumentError):
            call()
        assert np.array_equal(e.get("alpha"), before["alpha"]), i
        assert np.array_equal(e.get("L"), before["L"]), i
        for k, full in (("pred", False), ("cov", True)):
            got = e.predict(Xn[:12] if full else Xn, full_cov=full)
            assert all(np.array_equal(a, b) for a, b in zip(got, before[k])), (i, k)
    e.close()


# --------------------------------------------------------------------------------------------------------------------
# E. the sparse evaluation with a one-rank communicator
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_sparse_with_a_one_rank_communicator_is_bit_identical():
    """With one rank the all-reduces of the row-sharded sparse evaluation are skipped: the results are those of a plain
    context bit for bit."""
    X, Y = data(3000, 4, 2, seed=13)
    Z = X[::60] + 0.01
    nv = np.random.default_rng(13).uniform(0.01, 0.2, 3000)
    ls = np.array([1.2, 1.6, 2.0, 2.4])
    out = []
    for e in (plain_engine(), sharded_engine()):
        e.sparse_set_data(X, Y)
        r = list(e.sparse_eval("matern52", True, 1.3, ls, Z, 0.05)) + [e.sparse_get("woodbury_vector")]
        r += list(e.sparse_eval_het("rbf", False, 0.9, 1.7, Z, nv)) + [e.sparse_get("woodbury_inv")]
        out.append(r)
        e.close()
    for i, (a, b) in enumerate(zip(*out)):
        assert np.array_equal(a, b), i


# --------------------------------------------------------------------------------------------------------------------
# F. teardown
# --------------------------------------------------------------------------------------------------------------------
def _threads():
    return len(os.listdir("/proc/self/task"))


@pytest.mark.gpu
def test_destroy_and_reattach_release_the_communicator():
    """attach, evaluate (N = 2049), destroy, several times; then one context attached again and again. After the first
    cycle neither the device's free memory nor the process's thread count may keep falling / growing: a communicator that
    is not destroyed keeps its device buffers and its proxy threads."""
    import torch
    X, Y = data(2049, 3, 1, seed=3)

    def free():
        torch.cuda.synchronize()
        return torch.cuda.mem_get_info(0)[0]

    def evaluate_on(e):
        e.set_data(X, Y)
        e.exact_eval("rbf", True, 1.0, np.array([1.5, 2.0, 2.5]), 0.05)
        assert_blocks(e.stats(), 9)

    free0 = free()
    e = sharded_engine()
    evaluate_on(e)
    footprint = free0 - free()
    e.close()
    base, threads = free(), _threads()
    trace = []
    for _ in range(4):
        e = sharded_engine()
        evaluate_on(e)
        e.close()
        trace.append((base - free(), _threads() - threads))
    e = sharded_engine()
    evaluate_on(e)
    held, held_threads = free(), _threads()     # one live context: its cycle's footprint is held from here on
    for _ in range(4):
        attach(e)
        evaluate_on(e)
        trace.append((held - free(), _threads() - held_threads))
    e.close()
    trace.append((base - free(), _threads() - threads))
    print("\none cycle holds %.1f MiB; growth after the first cycle (MiB, threads): %s" % (
        footprint / 2**20, [("%.1f" % (m / 2**20), t) for m, t in trace]))
    assert footprint > 0
    # the cycle's own buffers come and go; what may stay is allocator granularity, far below one communicator (measured on
    # an H100 80GB HBM3: one cycle holds 494 MiB; a communicator that was never destroyed kept 388 MiB and 2 threads)
    assert max(m for m, _ in trace) <= footprint / 16, trace
    assert max(t for _, t in trace) <= 1, trace
