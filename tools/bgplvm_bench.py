"""Time one Bayesian GPLVM evaluation on the device (gpx_sparse_eval_psi, RBF(ARD)) at N in {4096, 65536}, M in {128, 512},
Q in {5, 10} and P in {1, 12}, and split it by kernel: the psi2 pass (psi2_pair_kernel without gradients +
psi2_finish_kernel) and the psi2 gradient pass (psi2_pair_kernel with gradients + psi_n_kernel + psi_nfin_kernel +
psi_m_kernel), from one evaluation profiled with torch.profiler (CUDA activities) after the timed ones. The evaluation
ends in a device synchronisation, so the host clock around it is its time; the median of --reps calls after one warm-up
is reported.
Rates: the psi2 pass visits N M (M + 1) / 2 (n, m, m') triples, the gradient pass twice that (its pair pass and its
per-point pass). Each triple needs at least 3 Q fp64 operations for its exponent (a subtraction, a multiplication and a
fused multiply-add per latent dimension) besides the exp; `fp64_share` is that count over the pass's device time, against
the H100 SXM data sheet's 34 TFLOP/s fp64 on the CUDA cores (the psi kernels use no tensor cores; the card's own clock and
power limit are recorded beside it).
    python tools/bgplvm_bench.py --out profiles/h100_bgplvm.json
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

FP64_PEAK = 34e12   # H100 SXM data sheet, fp64 on the CUDA cores (dense)


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                                        "--format=csv,noheader"], text=True).strip()
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def problem(N, M, Q, P, seed=0):
    rng = np.random.default_rng(seed)
    mu = rng.uniform(-2.0, 2.0, size=(N, Q))
    S = rng.uniform(0.01, 0.2, size=(N, Q))
    Z = mu[rng.permutation(N)[:M]].copy()
    Y = np.sin(mu.dot(rng.standard_normal((Q, P)))) + 0.05 * rng.standard_normal((N, P))
    rbf = ("rbf", True, 0, list(range(Q)), 1.0, np.linspace(0.8, 1.6, Q))
    return mu, S, Z, Y, rbf


def kernel_ms(fn):
    """device ms of the psi2 pass and of the psi2 gradient pass in one profiled call"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    fwd = grad = 0.0
    for ev in prof.events():
        name = ev.name
        dt = getattr(ev, "device_time", None)
        if dt is None:
            dt = ev.cuda_time
        if ("psi2_pair_kernel" in name and ("false" in name or "Lb0E" in name)) or "psi2_finish_kernel" in name:
            fwd += dt
        elif "psi2_pair_kernel" in name or "psi_n_kernel" in name or "psi_nfin_kernel" in name or "psi_m_kernel" in name:
            grad += dt
    return fwd * 1e-3, grad * 1e-3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    rec = {"card_before": card(), "rows": []}
    for N in (4096, 65536):
        for M in (128, 512):
            for Q in (5, 10):
                for P in (1, 12):
                    mu, S, Z, Y, rbf = problem(N, M, Q, P)
                    e = _ffi.Engine()
                    if P > 8:
                        e.set_option("sparse_wide", 1)
                    e.sparse_set_data(mu, Y)
                    fn = lambda: e.sparse_eval_psi(rbf, S, Z, 0.05)  # noqa: E731
                    fn()
                    ts = []
                    for _ in range(a.reps):
                        t0 = time.perf_counter()
                        fn()
                        ts.append(time.perf_counter() - t0)
                    l0 = e.total_launches()
                    fn()
                    launches = e.total_launches() - l0
                    fwd, grad = kernel_ms(fn)
                    tri = N * M * (M + 1) / 2.0
                    row = dict(N=N, M=M, Q=Q, P=P, eval_ms=1e3 * float(np.median(ts)), launches=launches,
                               psi2_ms=fwd, psi2_grad_ms=grad,
                               psi2_triples_per_s=tri / (fwd * 1e-3), psi2_grad_triples_per_s=2 * tri / (grad * 1e-3),
                               psi2_fp64_share=3 * Q * tri / (fwd * 1e-3) / FP64_PEAK,
                               psi2_grad_fp64_share=3 * Q * 2 * tri / (grad * 1e-3) / FP64_PEAK)
                    rec["rows"].append(row)
                    print(json.dumps(row), flush=True)
                    del e
    rec["card_after"] = card()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
