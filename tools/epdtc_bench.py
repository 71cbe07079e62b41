"""Measure the sparse EP on the device (gpy_b200.EPDTC over gpx_epdtc_*): GP classification with the probit Bernoulli
likelihood and RBF(ARD), D = 8, sequential updates, 5 sweeps, at N = 65536 / 262144 with M = 1024. Writes
profiles/h100_epdtc.json (or --out) with, per size:
  ms of the full run (begin, cold start, 5 sweeps, finish), per sweep, and of the finish (VarDTC at precision tau~);
  ms of the recompute alone (a warm start: LLT, its factor, A = U U^T, V = L^-1 Kmn, Sigma_diag and mu);
  from torch.profiler over one sweep, the block loop by kernel: site chains, solves, M-space GEMMs (P^T = KbT A, G and
  the rank-128 update of A), the rest (gather, mirror, row dots), and the GEMMs' TFLOP/s against gpx_measure_fp64_peak.
For context, dense EP (gpy_b200.EP) at N = 16384 next to EPDTC at N = 16384, M = 1024. The card name, power limit and SM
clock are read in the same run (nvidia-smi queries only). Medians of --repeats runs after one warm-up run.

    python tools/epdtc_bench.py [--sizes 65536 262144] [--out profiles/h100_epdtc.json]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from laplace_bench import D, LS, card, data  # noqa: E402

TILE = 128
SWEEPS = 5


def parts():
    return [("rbf", 1, 0, list(range(D)), 1.3, np.array(LS))]


def one_run(eng, X, Y, Z):
    """begin, cold start, SWEEPS sweeps, finish -> (ms total, ms per sweep list, ms finish)"""
    N = X.shape[0]
    t0 = time.perf_counter()
    eng.epdtc_begin(parts(), Z)
    eng.epdtc_start()
    tt, vt = np.zeros(N), np.zeros(N)
    per = []
    rng = np.random.default_rng(1)
    for _ in range(SWEEPS):
        s0 = time.perf_counter()
        out = eng.epdtc_sweep(rng.permutation(N), tt, vt)
        tt, vt = out[0], out[1]
        per.append(1e3 * (time.perf_counter() - s0))
    f0 = time.perf_counter()
    eng.epdtc_finish(tt, vt)
    t1 = time.perf_counter()
    return 1e3 * (t1 - t0), per, 1e3 * (t1 - f0), tt, vt


def profile_sweep(eng, N, tt, vt):
    import torch
    from torch.profiler import ProfilerActivity, profile
    eng.epdtc_start(tt, vt)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.epdtc_sweep(np.random.default_rng(2).permutation(N), tt, vt)
        torch.cuda.synchronize()
    cat = {"chain": 0.0, "solve": 0.0, "gemm": 0.0, "other": 0.0}
    for ev in prof.key_averages():
        us = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
        n = ev.key
        k = "chain" if "ep_chain" in n else "solve" if "ep_solve" in n else "gemm" if "gemm" in n else "other"
        cat[k] += us / 1e3
    return cat


def block_gemm_flops(N, M):
    Mp = -(-M // TILE) * TILE
    mt = Mp // TILE
    per_block = 2.0 * TILE * Mp * Mp + 2.0 * TILE * TILE * Mp + 2.0 * TILE * TILE * TILE * (mt * (mt + 1) // 2)
    return per_block * (-(-N // TILE))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[65536, 262144])
    ap.add_argument("--M", type=int, default=1024)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_epdtc.json"))
    ap.add_argument("--no-dense", action="store_true")
    a = ap.parse_args()
    import gpy_b200
    eng = gpy_b200.Engine()
    res = {"card": card(), "kernel": "RBF ARD, D = %d" % D, "sweeps": SWEEPS, "updates": "sequential",
           "fp64_peak_tflops": eng.measure_fp64_peak(), "sizes": {}}
    for N in a.sizes + ([] if a.no_dense else [16384]):
        X, Y = data(N)
        Z = X[np.random.default_rng(5).permutation(N)[:a.M]].copy()
        eng.sparse_set_data(X, Y)
        one_run(eng, X, Y, Z)                                       # warm-up
        runs = [one_run(eng, X, Y, Z) for _ in range(a.repeats)]
        tt, vt = runs[-1][3], runs[-1][4]
        rec = []
        for _ in range(a.repeats):
            eng.epdtc_begin(parts(), Z)
            t0 = time.perf_counter()
            eng.epdtc_start(tt, vt)
            rec.append(1e3 * (time.perf_counter() - t0))
        cat = profile_sweep(eng, N, tt, vt)
        fl = block_gemm_flops(N, a.M)
        r = {"N": N, "M": a.M, "run_ms": float(np.median([x[0] for x in runs])),
             "sweep_ms": float(np.median([np.median(x[1]) for x in runs])),
             "finish_ms": float(np.median([x[2] for x in runs])), "recompute_ms": float(np.median(rec)),
             "block_loop_by_kernel_ms (one sweep, profiled)": cat,
             "block_gemm_tflops": fl / (cat["gemm"] * 1e-3) / 1e12 if cat["gemm"] > 0 else None}
        res["sizes"]["epdtc_N%d_M%d" % (N, a.M)] = r
        print(json.dumps(r), flush=True)
    if not a.no_dense:
        N = 16384
        X, Y = data(N)
        m = gpy_b200.EP(max_iters=SWEEPS, epsilon=0.0)
        k = gpy_b200.RBF(D, variance=1.3, lengthscale=np.array(LS), ARD=True)
        m.inference(k, X, gpy_b200.Bernoulli(), Y)
        ts = []
        for _ in range(a.repeats):
            m.reset()
            t0 = time.perf_counter()
            m.inference(k, X, gpy_b200.Bernoulli(), Y)
            ts.append(1e3 * (time.perf_counter() - t0))
        res["sizes"]["dense_ep_N16384"] = {"N": N, "run_ms": float(np.median(ts)), "sweeps": m.iterations}
        print(json.dumps(res["sizes"]["dense_ep_N16384"]), flush=True)
    res["reference_host"] = ("the reference's EPDTC at the fixture sizes (N <= 1300, M <= 300) takes the host_seconds "
                             "recorded in tests/golden/epdtc/*.npz, on the CPU build machine; at these sizes: not measured")
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print("wrote", a.out)


if __name__ == "__main__":
    main()
