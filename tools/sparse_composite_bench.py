"""Time one sparse GP regression (VarDTC) evaluation with a composite kernel beside the single RBF(ARD) evaluation at the
benchmark's shape (BASELINE.json configs[4]: N = 262144, M = 4096, D = 16).

Cases:
    rbf               RBF(ARD) through gpx_sparse_eval (the benchmark's kernel)
    rbf_bias_white    RBF(ARD) + Bias + White through gpx_sparse_eval_multi
    m52_x_rbf_bias    Matern52(ARD, dims 0-7) x RBF(ARD, dims 8-15) + Bias through gpx_sparse_eval_multi

Each case runs in a fresh worker process (one library load each), so that `--parent-lib` can time the single RBF(ARD)
evaluation with another build of libgpx.so, alternating with this one `--rounds` times in the same run. A worker warms
up, then records CUDA events on the current stream around each evaluation (an evaluation returns after its results are
on the host) and the library's launch count per evaluation. The median over `--steps` is reported, with the card's name
and power limit read in the same run. Needs a GPU.

    python tools/sparse_composite_bench.py [--steps 5] [--warmup 2] [--rounds 3] [--parent-lib PATH] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N, M, D = 262144, 4096, 16
CASES = ("rbf", "rbf_bias_white", "m52_x_rbf_bias")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, watts = [s.strip() for s in q.split(",")]
    return name, watts


def worker(case, lib, steps, warmup):
    sys.path.insert(0, ROOT)
    from gpy_b200 import _ffi
    if lib:   # another build: bind the entries it has (an older one lacks gpx_sparse_eval_multi)
        import ctypes
        have = ctypes.CDLL(lib)
        _ffi.EXPORTS = {k: v for k, v in _ffi.EXPORTS.items() if hasattr(have, k)}
        _ffi.LIB_PATH = lib
    import torch
    rng = np.random.default_rng(0)
    X = rng.uniform(-3, 3, (N, D))
    Y = np.sin(X).sum(1, keepdims=True) / np.sqrt(D) + 0.1 * rng.standard_normal((N, 1))
    Z = X[rng.permutation(N)[:M]].copy()
    ls = np.full(D, np.sqrt(D))
    lo, hi = list(range(8)), list(range(8, 16))
    eng = _ffi.Engine(0)
    eng.sparse_set_data(X, Y)
    if case == "rbf":
        call = lambda: eng.sparse_eval("rbf", True, 1.0, ls, Z, 0.05)   # noqa: E731
    elif case == "rbf_bias_white":
        parts = [("rbf", True, 0, list(range(D)), 1.0, ls), ("bias", False, 1, [], 0.3, None),
                 ("white", False, 2, [], 0.01, None)]
        call = lambda: eng.sparse_eval_multi(parts, Z, 0.05)   # noqa: E731
    else:
        parts = [("matern52", True, 0, lo, 1.0, ls[:8]), ("rbf", True, 0, hi, 1.0, ls[8:]),
                 ("bias", False, 1, [], 0.3, None)]
        call = lambda: eng.sparse_eval_multi(parts, Z, 0.05)   # noqa: E731
    for _ in range(warmup):
        call()
    ms, launches = [], []
    for _ in range(steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        l0 = eng.total_launches()
        e0.record()
        out = call()
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
        launches.append(eng.total_launches() - l0)
    eng.close()
    return dict(case=case, lib="parent" if lib else "this", ms_median=float(np.median(ms)), ms=ms,
                launches=int(np.median(launches)), lml=float(out[0]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3, help="alternations of the RBF(ARD) case (with --parent-lib)")
    ap.add_argument("--parent-lib", default=None, help="another libgpx.so to time the RBF(ARD) case with")
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker", default=None, help=argparse.SUPPRESS)
    ap.add_argument("--lib", default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        print(json.dumps(worker(a.worker, a.lib, a.steps, a.warmup)), flush=True)
        return
    name, watts = card()

    def run(case, lib=None):
        cmd = [sys.executable, os.path.abspath(__file__), "--worker", case, "--steps", str(a.steps), "--warmup",
               str(a.warmup)] + (["--lib", os.path.abspath(lib)] if lib else [])
        line = json.loads(subprocess.run(cmd, capture_output=True, text=True, check=True).stdout.strip().splitlines()[-1])
        line.update(card=name, power_limit=watts, N=N, M=M, D=D)
        print(json.dumps(line), flush=True)
        return line

    lines = [run(c) for c in CASES]
    if a.parent_lib:
        for _ in range(a.rounds):
            lines.append(run("rbf", a.parent_lib))
            lines.append(run("rbf"))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
