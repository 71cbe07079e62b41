"""Time sparse prediction on the device (gpx_sparse_predict) against the host route SparseGP.predict took before it.

Model: one VarDTC RBF(ARD) evaluation at N = 262144, M = 4096, D = 16 (BASELINE.json configs[4]). Then
    device   gpx_sparse_predict, diagonal variance, at M* = 1e3, 1e4, 1e5, 1e6; full covariance at M* = 4096
    host     the route a posterior without the evaluation's key takes (SparsePosterior._raw_predict): K(Z, Xnew) from the
             stand-alone kernel call, copied to the host, woodbury_vector and woodbury_inv fetched on first touch, the
             products in NumPy; at M* <= 1e5. Its first call (which fetches W) is reported on its own.
Each call returns with its results on the host; the host clock around it is the call time: the median of --steps calls
after --warmup. GEMM TFLOP/s = 2 M^2 M* (M and M* padded to 128) / GEMM time; for the full covariance the flops add the
lower tiles of V^T K(Z, X*). The GEMM time comes from torch.profiler (CUDA activities, a run of its own, which also splits
the call into K-build, GEMM, mean, variance, memsets, copies and the rest); the share of peak is against the DMMA rate
gpx_measure_fp64_peak measures. The card's name, power limit and SM clock are read in the same run. Needs a GPU.

    python tools/sparse_predict_bench.py [--steps 5] [--warmup 2] [--out profiles/h100_sparse_predict.json]
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
N, M, D = 262144, 4096, 16


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


def phases(fn):
    """device ms of one call by kernel family (torch.profiler, CUDA activities)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    ph = dict(kbuild=0.0, gemm=0.0, mean=0.0, variance=0.0, memset=0.0, copy=0.0, other=0.0)
    for ev in prof.events():
        if ev.device_type is None or "cuda" not in str(ev.device_type).lower():
            continue
        ms = (ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total) * 1e-3
        n = ev.name
        key = ("kbuild" if ("kbuild" in n or "prep" in n) else "gemm" if "gemm_panel" in n else
               "mean" if ("row_dot" in n or "uv_reduce" in n) else "variance" if "sparse_var" in n else
               "memset" if "Memset" in n else "copy" if "Memcpy" in n else "other")
        ph[key] += ms
    return ph


def model():
    from gpy_b200 import _ffi
    rng = np.random.default_rng(0)
    X = rng.uniform(-3, 3, (N, D))
    Y = np.sin(X).sum(1, keepdims=True) / np.sqrt(D) + 0.1 * rng.standard_normal((N, 1))
    Z = X[rng.permutation(N)[:M]].copy()
    ls = np.full(D, np.sqrt(D))
    e = _ffi.Engine(0)
    e.sparse_set_data(X, Y)
    e.sparse_eval("rbf", True, 1.0, ls, Z, 0.05)
    return e, Z, ls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import gpy_b200
    from gpy_b200.sparse import LazySparsePosterior
    e, Z, ls = model()
    peak = e.measure_fp64_peak()
    res = dict(card=card(), N=N, M=M, D=D, kernel="RBF ARD", fp64_dmma_peak_tflops=peak, steps=a.steps, warmup=a.warmup,
               device=[], host=[])
    rng = np.random.default_rng(1)
    for Ms, full_cov in ((1000, False), (10000, False), (100000, False), (1000000, False), (4096, True)):
        Xn = rng.uniform(-3, 3, (Ms, D))
        t, ts = median_ms(lambda: e.sparse_predict(Xn, full_cov=full_cov), a.steps, a.warmup)
        ph = phases(lambda: e.sparse_predict(Xn, full_cov=full_cov))
        # executed GEMM tiles: V^T = K(X*, Z) W (2 Mz^2 L), and for the full covariance the lower tiles of V^T K(Z, X*)
        Mz, L = -(-M // 128) * 128, -(-Ms // 128) * 128
        nt = L // 128
        flops = 2.0 * Mz * Mz * L + (nt * (nt + 1) / 2 * 2.0 * 128 * 128 * Mz if full_cov else 0.0)
        rec = dict(M_star=Ms, full_cov=full_cov, call_ms=t, call_ms_all=ts, phases_ms=ph, gemm_flops=flops,
                   gemm_tflops=flops / (ph["gemm"] * 1e-3) / 1e12 if ph["gemm"] else None)
        rec["gemm_share_of_peak"] = rec["gemm_tflops"] / peak if rec["gemm_tflops"] else None
        rec["call_tflops"] = flops / (t * 1e-3) / 1e12
        res["device"].append(rec)
        print(json.dumps({k: v for k, v in rec.items() if k != "call_ms_all"}), flush=True)
    k = gpy_b200.RBF(D, variance=1.0, lengthscale=ls, ARD=True)
    for Ms in (1000, 10000, 100000):
        Xn = rng.uniform(-3, 3, (Ms, D))
        post = LazySparsePosterior(e)            # no key: the host route, woodbury arrays fetched on first touch
        t0 = time.perf_counter()
        post._raw_predict(k, Xn, Z)
        first = (time.perf_counter() - t0) * 1e3
        t, ts = median_ms(lambda: post._raw_predict(k, Xn, Z), a.steps, a.warmup)
        mu_d, var_d = e.sparse_predict(Xn)
        mu_h, var_h = post._raw_predict(k, Xn, Z)
        rec = dict(M_star=Ms, first_call_ms=first, call_ms=t, call_ms_all=ts,
                   max_abs_diff_mu=float(np.abs(mu_d - mu_h).max()), max_abs_diff_var=float(np.abs(var_d - var_h).max()))
        res["host"].append(rec)
        print(json.dumps({k_: v for k_, v in rec.items() if k_ != "call_ms_all"}), flush=True)
    res["card_after"] = card()
    e.close()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
