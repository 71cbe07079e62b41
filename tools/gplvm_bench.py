"""Time one GPLVM evaluation on the device, split into the exact evaluation (gpx_exact_eval_multi with GPLVM's default
kernel RBF(ARD) + Bias) and the input gradient (gpx_exact_grad_X), at N in {4096, 16384}, Q in {2, 10} and
P in {12, 256, 1024} (the exact evaluation's wide route, more than 8 output columns). Each entry ends in a device
synchronisation, so the host clock around it is the call's time; the median of --reps calls after one warm-up is reported, with the card's name and power limit read
in the same run.
    python tools/gplvm_bench.py --out profiles/h100_gplvm.json
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    rows = []
    for N in (4096, 16384):
        for Q in (2, 10):
            for P in (12, 256, 1024):
                rng = np.random.default_rng(N + Q + P)
                X = rng.standard_normal((N, Q))
                Y = np.sin(X.dot(rng.standard_normal((Q, P)))) + 0.1 * rng.standard_normal((N, P))
                parts = [("rbf", True, 0, list(range(Q)), 1.0, np.linspace(0.8, 1.6, Q)), ("bias", False, 1, [], np.exp(-2), None)]
                eng = _ffi.Engine()
                eng.set_data(X, Y)
                t_eval = timed(lambda: eng.exact_eval_multi(parts, 0.1), args.reps)
                t_gx = timed(lambda: eng.exact_grad_X(), args.reps)
                t0 = eng.total_launches()
                eng.exact_grad_X()
                row = dict(N=N, Q=Q, P=P, eval_ms=t_eval, grad_X_ms=t_gx, total_ms=t_eval + t_gx,
                           grad_X_launches=int(eng.total_launches() - t0))
                print(json.dumps(row), flush=True)
                rows.append(row)
                eng.close()
    rec = dict(what="GPLVM evaluation on the device: gpx_exact_eval_multi (RBF(ARD) + Bias) and gpx_exact_grad_X, median "
                    "host time of synchronised calls", card=card(), rows=rows)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
