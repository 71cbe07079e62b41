"""Time the Mauna Loa-shaped composite kernel (RBF + RBF x StdPeriodic + RatQuad + RBF + White, Rasmussen & Williams
section 5.4.3) on the fused composite evaluation, beside the single-kernel RBF evaluation at the same N.

D = 1 time-like inputs (years 1958-2025), N = 4096 and 16384, both tensor paths (fp64 DMMA, int8 digit split). For each
case: CUDA-event ms per evaluation from Engine.stats() after warm-up, its kbuild / sweep / lauum split, and the RBF
evaluation's ms. At N = 4096 the LML and gradient are checked against the CPU oracle (tests/periodic_oracle.py). The card's
name and power limit are read in the same run. Needs a GPU; prints one JSON line per case.

    python tools/periodic_composite_bench.py [--sizes 4096 16384] [--steps 5] [--warmup 2] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, watts = [s.strip() for s in q.split(",")]
    return name, watts


def timed(fn, eng, steps, warmup):
    for _ in range(warmup):
        fn()
    rows = []
    for _ in range(steps):
        fn()
        rows.append(eng.stats())
    med = lambda k: float(np.median([r[k] for r in rows]))   # noqa: E731
    return {k: med(k) for k in ("total_ms", "kbuild_ms", "sweep_ms", "lauum_ms")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[4096, 16384])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import gpy_b200
    import periodic_oracle as po
    name, watts = card()
    parts = po.mauna_loa_parts()
    desc = [po.descriptor(p) for p in parts]
    lines = []
    for N in a.sizes:
        X, Y = po.mauna_loa_data(N, seed=0)
        ref = po.composite_eval(X, Y, parts, 0.01) if N <= 4096 else None
        for oz in (0, 1):
            eng = gpy_b200.Engine()
            eng.set_option("ozaki", oz)
            eng.set_data(X, Y)
            out = {}
            comp = timed(lambda: out.update(r=eng.exact_eval_multi(desc, 0.01)), eng, a.steps, a.warmup)
            rbf = timed(lambda: eng.exact_eval("rbf", False, 4.0, 50.0, 0.01), eng, a.steps, a.warmup)
            line = dict(N=N, path="int8" if oz else "dmma", composite=comp, rbf_total_ms=rbf["total_ms"], card=name,
                        power_limit=watts)
            if ref is not None:
                lml, g, _ = out["r"]
                line["parity"] = dict(dlml=abs(lml - ref[0]),
                                      grad_rel=float(np.max(np.abs(g - ref[1]) / np.maximum(np.abs(ref[1]), 1e-300))))
            print(json.dumps(line), flush=True)
            lines.append(line)
            eng.close()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
