"""Time FITC (gpx_sparse_eval_fitc) against VarDTC (gpx_sparse_eval) at the benchmark's sparse shape.

Model: RBF(ARD), N = 262144, M = 4096, D = 16 (BASELINE.json configs[4]) on one context, as a user switching methods
would run it (two contexts would hold both methods' M x N buffers, about 70 GB); the two evaluations alternate, --warmup
rounds first. Each call returns with its results on the host, so the
host clock around it is the evaluation's time: the median of --steps calls per method. Reported per method:
    eval_ms              median time per evaluation (all values in eval_ms_all)
    launches             kernels per evaluation (gpx_total_launches)
    device_used_gb       device memory in use after the run (cudaMemGetInfo: CUDA context, data, FITC's five M x N buffers)
    phases_ms            device time by kernel family from torch.profiler (CUDA activities) in a run of its own
    gemm_tflops          the N M^2 GEMM flops (below) over the profiler's GEMM time, and its share of the DMMA rate
                         gpx_measure_fp64_peak measures
GEMM flops, with nt = M / 128 tiles and k-depth N padded to 128, 2 128^2 N per executed tile:
    VarDTC  tmp (triangular, nt (nt + 1) / 2 tiles) + A (lower tiles) + dL_dKnm^T (nt^2)
    FITC    tmp + A + F1 = P psi1^T (nt^2) + F2 = Kmm^-1 psi1^T (nt^2) + F2 diag(dL_dR) F2^T (lower tiles)
The card's name and power limit are read before and after. Needs a GPU.

    python tools/fitc_bench.py [--steps 5] [--warmup 1] [--out profiles/h100_fitc.json]
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


def phases(fn):
    """device ms of one call by kernel family (torch.profiler, CUDA activities)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    ph = dict(kbuild=0.0, gemm=0.0, factor=0.0, fitc_per_point=0.0, grad_reductions=0.0, memset=0.0, copy=0.0, other=0.0)
    for ev in prof.events():
        if ev.device_type is None or "cuda" not in str(ev.device_type).lower():
            continue
        ms = (ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total) * 1e-3
        n = ev.name
        key = ("kbuild" if ("kbuild" in n or "prep" in n) else "gemm" if "gemm_panel" in n else
               "fitc_per_point" if ("fitc_" in n or "col_sqnorm" in n or "scale_cols" in n) else
               "grad_reductions" if "grad" in n else
               "factor" if ("sweep" in n or "update" in n or "trsm" in n or "potrf" in n or "assemble" in n
                            or "diag" in n) else
               "memset" if "Memset" in n else "copy" if "Memcpy" in n else "other")
        ph[key] += ms
    return ph


def gemm_flops(method):
    nt, Np = -(-M // 128), -(-N // 128) * 128
    tri, full = nt * (nt + 1) / 2, nt * nt
    tiles = 2 * tri + full if method == "vardtc" else 3 * tri + 2 * full
    return tiles * 2.0 * 128 * 128 * Np


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from gpy_b200 import _ffi
    rng = np.random.default_rng(0)
    X = rng.uniform(-3, 3, (N, D))
    Y = np.sin(X).sum(1, keepdims=True) / np.sqrt(D) + 0.1 * rng.standard_normal((N, 1))
    Z = X[rng.permutation(N)[:M]].copy()
    ls = np.full(D, np.sqrt(D))
    res = dict(card=card(), N=N, M=M, D=D, kernel="RBF ARD", noise=0.05, steps=a.steps, warmup=a.warmup,
               timing="host clock around the synchronous call, median", methods={})
    e = _ffi.Engine(0)
    e.sparse_set_data(X, Y)
    engines = {"vardtc": e, "fitc": e}
    calls = {"vardtc": lambda e: e.sparse_eval("rbf", True, 1.0, ls, Z, 0.05),
             "fitc": lambda e: e.sparse_eval_fitc([("rbf", True, 0, list(range(D)), 1.0, ls)], Z, 0.05)}
    peak = engines["vardtc"].measure_fp64_peak()
    res["fp64_dmma_peak_tflops"] = peak
    times = {k: [] for k in calls}
    launches, outs = {}, {}
    for r in range(a.warmup + a.steps):
        for name, fn in calls.items():
            e = engines[name]
            l0 = e.total_launches()
            t0 = time.perf_counter()
            outs[name] = fn(e)
            t = (time.perf_counter() - t0) * 1e3
            launches[name] = e.total_launches() - l0
            if r >= a.warmup:
                times[name].append(t)
    free, total = torch.cuda.mem_get_info()
    for name, fn in calls.items():
        ph = phases(lambda: fn(engines[name]))
        fl = gemm_flops(name)
        rec = dict(eval_ms=float(np.median(times[name])), eval_ms_all=times[name], launches=int(launches[name]),
                   lml=float(outs[name][0]), phases_ms=ph, gemm_flops=fl,
                   gemm_tflops=fl / (ph["gemm"] * 1e-3) / 1e12 if ph["gemm"] else None)
        rec["gemm_share_of_peak"] = rec["gemm_tflops"] / peak if rec["gemm_tflops"] else None
        res["methods"][name] = rec
        print(name, json.dumps({k: v for k, v in rec.items() if k != "eval_ms_all"}), flush=True)
    res["device_used_gb"] = (total - free) / 1e9
    res["fitc_over_vardtc"] = res["methods"]["fitc"]["eval_ms"] / res["methods"]["vardtc"]["eval_ms"]
    res["card_after"] = card()
    e.close()
    print(json.dumps({k: res[k] for k in ("card", "fitc_over_vardtc", "device_used_gb")}), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
