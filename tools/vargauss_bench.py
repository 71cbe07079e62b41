"""Time one evaluation of the variational Gaussian approximation on the device: gpx_vargauss_begin, the probit
Bernoulli's variational expectations on the host (20-point Gauss-Hermite), gpx_vargauss_finish, with RBF(ARD) on D = 8
inputs at N in {4096, 16384, 32768}. Records the median host time of whole evaluations (each entry ends in a device
synchronisation) after one warm-up, the device time of each phase (gpx_get_stats of both entries), launches, the device
memory in use after the evaluation (K, the factor and Ai / S; the finish's two temporaries, which bring the peak to the
predicted 40 Npad^2 bytes, are back in the pool by then and are not measured), the sweep, LAUUM and GEMM rates
against gpx_measure_fp64_peak, the card's name and power limit read in the same run, and parity with
tests/vargauss_oracle.py at N = 4096.
    python tools/vargauss_bench.py --out profiles/h100_vargauss.json
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import gpy_b200  # noqa: E402
from gpy_b200 import _ffi  # noqa: E402

PHASES = ("kbuild_ms", "sweep_ms", "update_ms", "lauum_ms", "solve_ms", "total_ms")


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                       text=True).strip()
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def problem(N, D=8, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.uniform(-2, 2, size=(N, D))
    Y = (np.sin(X[:, :1]) + 0.3 * X[:, 1:2] + 0.3 * rng.standard_normal((N, 1)) > 0).astype(np.float64)
    parts = [("rbf", True, 0, list(range(D)), 1.3, np.linspace(1.5, 3.0, D))]
    alpha = 0.1 * rng.standard_normal(N)
    beta = rng.uniform(0.5, 2.0, N)
    return X, Y, parts, alpha, beta


def evaluate(eng, parts, Y, alpha, beta, lik):
    m, var, kl, _ = eng.vargauss_begin(parts, alpha, beta)
    sb = eng.stats()
    F, dF_dm, dF_dv, _ = lik.variational_expectations(Y, m[:, None], var[:, None])
    da, db, kg = eng.vargauss_finish(dF_dm[:, 0], dF_dv[:, 0])
    sf = eng.stats()
    return dict(lml=float(F.sum()) - kl, dalpha=da, dbeta=db, kgrad=kg), sb, sf


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sizes", default="4096,16384,32768")
    args = ap.parse_args()
    import torch
    torch.cuda.init()
    free0 = torch.cuda.mem_get_info()[0]
    lik = gpy_b200.Bernoulli()
    eng = _ffi.Engine()
    peak = eng.measure_fp64_peak()
    rows = []
    for N in [int(s) for s in args.sizes.split(",")]:
        X, Y, parts, alpha, beta = problem(N)
        eng.set_data(X, Y)
        ts, out, sb, sf = [], None, None, None
        for r in range(args.reps + 1):
            t0 = time.perf_counter()
            out, sb, sf = evaluate(eng, parts, Y, alpha, beta, lik)
            if r:
                ts.append(time.perf_counter() - t0)
        used = free0 - torch.cuda.mem_get_info()[0]
        Np = float(-(-N // 128) * 128)
        ph = {k: float(sb[k] + sf[k]) for k in PHASES}
        row = dict(N=N, eval_ms=1e3 * float(np.median(ts)), phases_ms=ph, launches_begin=int(sb["launches"]),
                   launches_finish=int(sf["launches"]), device_bytes_in_use=int(used),
                   predicted_peak_bytes=int(40 * Np * Np),
                   sweep_tflops=2 * Np ** 3 / 3 / (ph["sweep_ms"] * 1e9) if ph["sweep_ms"] else None,
                   lauum_tflops=Np ** 3 / 3 / (ph["lauum_ms"] * 1e9) if ph["lauum_ms"] else None,
                   gemm_tflops=Np ** 3 / (ph["update_ms"] * 1e9) if ph["update_ms"] else None)
        if N == 4096:
            import vargauss_oracle as vo
            o = vo.vargauss_eval([dict(kind="rbf", term=0, dims=list(range(8)), variance=1.3,
                                       lengthscale=np.linspace(1.5, 3.0, 8), ARD=True)], X, Y, alpha, beta, lik)

            def rel(a, b):
                return float(np.abs(np.asarray(a) - b).max() / np.abs(b).max())
            row["parity"] = dict(lml=abs(out["lml"] - o["lml"]) / abs(o["lml"]), dalpha=rel(out["dalpha"], o["dalpha"]),
                                 dbeta=rel(out["dbeta"], o["dbeta"]), kgrad=rel(out["kgrad"], o["grad"]),
                                 cond_A=float(o["cond_A"]))
        print(json.dumps(row), flush=True)
        rows.append(row)
    rec = dict(what="one VarGauss evaluation on the device: gpx_vargauss_begin, the probit Bernoulli's variational "
                    "expectations on the host, gpx_vargauss_finish; RBF(ARD), D = 8; median host time of %d evaluations "
                    "after one warm-up; phases are device times summed over both entries; TFLOP/s count 2 N^3 / 3 for "
                    "the sweep, N^3 / 3 for the LAUUM and N^3 for the GEMM (N padded to 128)" % args.reps,
               card=card(), fp64_peak_tflops=peak, rows=rows)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
