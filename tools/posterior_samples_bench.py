"""Time the joint posterior on the device (gpx_posterior_samples, gpx_sparse_posterior_samples) against the route the
reference takes through the plugin.

Exact case: one RBF(ARD) evaluation at N = 16384, D = 8 (BASELINE.json configs[1]), then for M* in {128, 1024, 4096} and
S = 1000 samples:
    device  one gpx_posterior_samples call (z drawn on the host beforehand; it returns after f is on the host)
    host    today's route: gpx_predict(full_cov=1) (two N x M* matrices to the host, the M* x M* covariance in a host loop),
            then numpy's np.random.multivariate_normal (SVD); at M* = 4096 it is not run
The device time of one call is split by torch.profiler (CUDA activities, a run of its own) into the K-builds, the L^-1
extraction, the triangular GEMM T^T = K(X*, X) L^-T (achieved TFLOP/s over the executed tiles, against the DMMA rate
gpx_measure_fp64_peak measures), the Sigma GEMM, the factorisation of Sigma (every kernel between the combine and the
extraction of L_Sigma), the sample GEMM and the rest (mean, combine, z layout, mean add).
The host time of the CUDA runtime calls of one call is listed beside (torch.profiler, CPU and CUDA activities).
Sparse case: one VarDTC RBF(ARD) evaluation at N = 262144, M = 4096, D = 16, then gpx_sparse_posterior_samples at
M* = 1024, S = 1000 (woodbury_inv kept from a first call).
Largest case: N = 32768, M* = 4096, one covariance between two halves of the points and 100 samples, to show they fit.
Medians of --steps calls after --warmup; the card's name, power limit and SM clock are read in the same run. Needs a GPU.

    python tools/posterior_samples_bench.py [--steps 5] [--warmup 2] [--out profiles/h100_posterior_samples.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
TILE = 128


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, watts, sm, smax = [s.strip() for s in q.split(",")]
    return dict(name=name, power_limit=watts, sm_clock=sm, sm_clock_max=smax)


def median_ms(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(steps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts)), ts


def kernels(fn):
    """(name, start us, device us) of every kernel one call launches, in launch order (torch.profiler, a run of its own)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = []
    for ev in prof.events():
        if ev.device_type is None or "cuda" not in str(ev.device_type).lower():
            continue
        us = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        out.append((ev.name, ev.time_range.start, us))
    return sorted(out, key=lambda e: e[1])


def runtime_calls(fn, top=6):
    """host time of the CUDA runtime calls of one call (torch.profiler's CUDA runtime events), the largest first"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    tot = {}
    for ev in prof.events():
        if ev.name.startswith("cuda") and (ev.device_type is None or "cuda" not in str(ev.device_type).lower()):
            tot[ev.name] = tot.get(ev.name, 0.0) + ev.cpu_time_total * 1e-3
    return dict(sorted(tot.items(), key=lambda kv: -kv[1])[:top])


def split_exact(ks):
    """phases of one gpx_posterior_samples call from its kernels in launch order"""
    ph = dict(kbuild=0.0, linv_extract=0.0, tri_gemm=0.0, sigma_gemm=0.0, factor=0.0, sample_gemm=0.0, other=0.0)
    names = [k[0] for k in ks]
    ext = [i for i, n in enumerate(names) if "joint_extract" in n]
    gem = [i for i, n in enumerate(names) if "gemm_panel" in n]
    comb = [i for i, n in enumerate(names) if "joint_combine" in n]
    for i, (n, _, us) in enumerate(ks):
        ms = us * 1e-3
        if "kbuild" in n or "prep" in n:
            ph["kbuild"] += ms
        elif i == ext[0]:
            ph["linv_extract"] += ms
        elif i == gem[0]:
            ph["tri_gemm"] += ms
        elif i == gem[1]:
            ph["sigma_gemm"] += ms
        elif i == gem[-1]:
            ph["sample_gemm"] += ms
        elif comb[0] < i < ext[-1]:
            ph["factor"] += ms
        else:
            ph["other"] += ms
    return ph


def exact_case(steps, warmup, M, S, peak, host):
    from gpy_b200 import _ffi
    from oracle import gpy_oracle as o
    N, D = 16384, 8
    X, Y = o.synthetic(N, D, seed=1)
    ls = np.sqrt(D) * np.linspace(0.8, 1.3, D)
    e = _ffi.Engine(0)
    e.set_data(X, Y)
    e.exact_eval("rbf", True, 1.2, ls, 0.1)
    Xn = np.random.default_rng(M).uniform(X.min(0), X.max(0), size=(M, D))
    z = np.random.default_rng(1).standard_normal((S, M))
    f, jit = e.posterior_samples(Xn, z)
    dev, dev_all = median_ms(lambda: e.posterior_samples(Xn, z), steps, warmup)
    ph = split_exact(kernels(lambda: e.posterior_samples(Xn, z)))
    api = runtime_calls(lambda: e.posterior_samples(Xn, z))
    Ls, Np = (M + TILE - 1) // TILE * TILE, N
    nt = Np // TILE
    tri_flops = 2.0 * Ls * TILE * TILE * nt * (nt + 1) / 2
    rec = dict(N=N, D=D, M_star=M, S=S, jitter_used=jit, device_ms=dev, device_ms_all=dev_all, phases_ms=ph,
               runtime_api_ms=api,
               tri_gemm_tflops=tri_flops / (ph["tri_gemm"] * 1e-3) / 1e12 if ph["tri_gemm"] else None,
               tri_gemm_flops=tri_flops, fp64_dmma_peak_tflops=peak)
    rec["tri_gemm_share_of_peak"] = rec["tri_gemm_tflops"] / peak if rec["tri_gemm_tflops"] else None
    if host:
        def today():
            mu, v = e.predict(Xn, full_cov=True)
            np.random.multivariate_normal(mu[:, 0], v, S)
        t0 = time.perf_counter()
        today()
        rec["host_route_ms"] = (time.perf_counter() - t0) * 1e3
        rec["host_route_runs"] = 1
    else:
        rec["host_route_ms"] = "not run"
    e.close()
    print(json.dumps({k: v for k, v in rec.items() if k != "device_ms_all"}), flush=True)
    return rec


def sparse_case(steps, warmup, Ms, S):
    from gpy_b200 import _ffi
    N, M, D = 262144, 4096, 16
    rng = np.random.default_rng(2)
    X = rng.uniform(-2, 2, size=(N, D))
    Y = np.sin(X[:, :3].sum(1, keepdims=True)) + 0.1 * rng.standard_normal((N, 1))
    Z = X[rng.choice(N, M, replace=False)]
    e = _ffi.Engine(0)
    e.sparse_set_data(X, Y)
    e.sparse_eval("rbf", True, 1.0, np.full(D, 2.0), Z, 0.05)
    Xn = rng.uniform(-2, 2, size=(Ms, D))
    z = np.random.default_rng(3).standard_normal((S, Ms))
    t0 = time.perf_counter()
    _, jit = e.sparse_posterior_samples(Xn, z)
    first = (time.perf_counter() - t0) * 1e3
    dev, dev_all = median_ms(lambda: e.sparse_posterior_samples(Xn, z), steps, warmup)
    rec = dict(N=N, M=M, D=D, M_star=Ms, S=S, jitter_used=jit, first_call_ms=first, device_ms=dev, device_ms_all=dev_all)
    e.close()
    print(json.dumps({k: v for k, v in rec.items() if k != "device_ms_all"}), flush=True)
    return rec


def largest_case():
    """N = 32768, M* = 4096: the covariance and S = 100 samples fit on one card (times of single calls)"""
    from gpy_b200 import _ffi
    from oracle import gpy_oracle as o
    N, D, M = 32768, 8, 4096
    X, Y = o.synthetic(N, D, seed=3)
    e = _ffi.Engine(0)
    e.set_data(X, Y)
    e.exact_eval("rbf", True, 1.2, np.sqrt(D) * np.linspace(0.8, 1.3, D), 0.1)
    Xn = np.random.default_rng(5).uniform(X.min(0), X.max(0), size=(M, D))
    t0 = time.perf_counter()
    cov = e.posterior_covariance(Xn[:M // 2], Xn[M // 2:])
    t1 = time.perf_counter()
    f, jit = e.posterior_samples(Xn, np.random.default_rng(6).standard_normal((100, M)))
    t2 = time.perf_counter()
    rec = dict(N=N, D=D, M_star=M, cov_shape=list(cov.shape), cov_ms=(t1 - t0) * 1e3, samples=100, samples_ms=(t2 - t1) * 1e3,
               jitter_used=jit, finite=bool(np.isfinite(cov).all() and np.isfinite(f).all()))
    e.close()
    print(json.dumps(rec), flush=True)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from gpy_b200 import _ffi
    peak = _ffi.Engine(0).measure_fp64_peak()
    res = dict(card=card(), fp64_dmma_peak_tflops=peak, exact=[], sparse=[])
    for M in (128, 1024, 4096):
        res["exact"].append(exact_case(a.steps, a.warmup, M, 1000, peak, host=M <= 1024))
    res["sparse"].append(sparse_case(a.steps, a.warmup, 1024, 1000))
    res["largest"] = largest_case()
    res["card_after"] = card()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
