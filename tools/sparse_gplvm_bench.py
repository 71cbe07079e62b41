"""Time one sparse GPLVM step on the device, split into the VarDTC evaluation (gpx_sparse_eval, RBF(ARD)) and the input
gradient (gpx_sparse_grad_X), at N = 65536, M = 1024, Q = 8 with P in {12, 256} and at N = 262144, M = 1024, P = 12 (P > 8:
the wide route). Each entry ends in a device synchronisation, so the host clock around it is the call's time; the median
of --reps calls after one warm-up is reported. A separate profiled evaluation (torch.profiler, CUDA activities) gives the
device time of the fp64 DMMA GEMM launches (gemm_panel_kernel), and their rate from the flops the route's GEMMs need,
counted from the shapes below. The card's name and power limit are read in the same run.
    python tools/sparse_gplvm_bench.py --out profiles/h100_sparse_gplvm.json
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gpy_b200 import _ffi  # noqa: E402

T = 128


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                       text=True).strip()
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def timed(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return 1e3 * float(np.median(ts))


def gemm_flops(N, M, P):
    """flops of the gemm_panel_kernel launches of one evaluation (gpx_sparse.cu): tiles times 2 * 128^2 * k-depth"""
    pad = lambda n: (n + T - 1) // T * T  # noqa: E731
    Np, Mp, mt = pad(N), pad(M), pad(M) // T
    tri = mt * (mt + 1) // 2
    f = 2 * T * T * Np * tri                 # tmp = Lm^-1 psi1^T, triangular operand: k-range (r + 1) tiles
    f += 2 * T * T * Np * tri                # A = tmp tmp^T, lower tiles
    f += 2 * T * T * Mp * tri                # B^-1 = UB UB^T, lower tiles
    f += 4 * 2 * Mp ** 3                     # the two sandwiches (dL_dKmm, W2)
    if P > 8:
        Pp = pad(P)
        f += 2 * Pp * Mp * Np                # t^T = Y^T tmp^T
        f += 2 * T * T * Pp * tri            # v^T, triangular operand: k-range (c + 1) tiles
        f += 2 * 2 * Pp * Mp * Mp            # w^T, C^T
        f += 2 * T * T * Pp * tri            # w w^T, lower tiles
        f += 2 * Mp * Np * (Mp + Pp)         # dL_dKnm^T = [W2 | C] [psi1 | beta Y]^T
    else:
        f += 2 * Mp * Np * Mp                # dL_dKnm^T = W2 psi1^T
    return float(f)


def profile_gemm(fn):
    """device time (ms) of the gemm_panel_kernel launches of one call of fn, and of all its kernels"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    gemm = tot = 0.0
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if ev.key.startswith("cuda") or ev.key.startswith("Memcpy") or ev.key.startswith("Memset"):
            continue
        tot += t
        if "gemm_panel_kernel" in ev.key:
            gemm += t
    return gemm * 1e-3, tot * 1e-3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--small", action="store_true", help="a tiny shape, for a dry run of the script")
    args = ap.parse_args()
    shapes = [(65536, 1024, 12), (65536, 1024, 256), (262144, 1024, 12)]
    if args.small:
        shapes = [(4096, 256, 12)]
    Q = 8
    rows = []
    for N, M, P in shapes:
        rng = np.random.default_rng(N + M + P)
        X = rng.standard_normal((N, Q))
        Y = np.sin(X.dot(rng.standard_normal((Q, P)))) + 0.1 * rng.standard_normal((N, P))
        Z = X[rng.permutation(N)[:M]].copy()
        ls = np.linspace(1.5, 3.0, Q)
        eng = _ffi.Engine()
        eng.set_option("sparse_wide", 1)
        eng.sparse_set_data(X, Y)
        ev = lambda: eng.sparse_eval("rbf", True, 1.0, ls, Z, 0.1)  # noqa: E731
        t_eval = timed(ev, args.reps)
        t_gx = timed(lambda: eng.sparse_grad_X(), args.reps)
        n0 = eng.total_launches()
        ev()
        n1 = eng.total_launches()
        eng.sparse_grad_X()
        n2 = eng.total_launches()
        gemm_ms, kern_ms = profile_gemm(ev)
        fl = gemm_flops(N, M, P)
        row = dict(N=N, M=M, Q=Q, P=P, eval_ms=t_eval, grad_X_ms=t_gx, total_ms=t_eval + t_gx,
                   eval_launches=int(n1 - n0), grad_X_launches=int(n2 - n1),
                   eval_kernels_device_ms=kern_ms, gemm_device_ms=gemm_ms, gemm_gflop=fl * 1e-9,
                   gemm_tflops=fl / (gemm_ms * 1e-3) * 1e-12 if gemm_ms > 0 else None)
        print(json.dumps(row), flush=True)
        rows.append(row)
        eng.close()
    rec = dict(what="sparse GPLVM step on the device: gpx_sparse_eval (RBF(ARD), Q = 8) and gpx_sparse_grad_X, median host "
                    "time of synchronised calls; GEMM device time from torch.profiler over one evaluation", card=card(),
               rows=rows)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
