"""Measure the Laplace approximation on the device (gpy_b200.Laplace over gpx_laplace_*): GP classification with a Bernoulli
(probit) likelihood and RBF(ARD), D = 8, at N = 4096 / 16384 / 32768, beside the exact evaluation of the same kernel at the
same N. Writes profiles/h100_laplace.json (or --out) with, per N:
  ms per evaluation, Newton steps, the per-phase split summed over the evaluation's device calls (K-build, factor =
  B-build + sweep, mat-vecs, finish GEMM, LAUUM, reductions and glue), the wall time outside them (the host's likelihood
  terms and line search, K v products, transfers), achieved TFLOP/s of the sweep and of the GEMM against
  gpx_measure_fp64_peak, and the exact evaluation's ms; then, in a profiled evaluation of its own, the device ms by kernel
  family (torch.profiler), which splits the "reductions and glue" phase (gradient reduction, rank-1 update, scaling) and
  leaves the rest of that phase to the stream-ordered allocation of the finish's two temporaries.
The card name, power limit and SM clock are read in the same run (nvidia-smi queries only).

    python tools/laplace_bench.py [--sizes 4096 16384 32768] [--out profiles/h100_laplace.json]
    python tools/laplace_bench.py --reference-host --out profiles/h100_laplace.json
        adds the reference's own Laplace on the host at N = 4096 (needs the reference tree; no GPU) to an existing file
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
D = 8


def data(N, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.uniform(-3, 3, size=(N, D))
    f = np.sin(X[:, :1]) + 0.5 * X[:, 1:2] - 0.3 * X[:, 2:3]
    Y = (f + 0.3 * rng.standard_normal((N, 1)) > 0).astype(np.float64)
    return X, Y


LS = [1.5, 2.0, 2.5, 3.0, 3.5, 4.0, 4.5, 5.0]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, sm, smmax = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": pl, "sm_clock": sm, "sm_clock_max": smmax}
    except Exception as e:   # noqa: BLE001
        return {"error": str(e)}


class Timed(object):
    """wraps an Engine: sums the per-phase stats of every Laplace call"""

    def __init__(self, eng):
        self.eng, self.acc, self.calls = eng, {}, {}

    def __getattr__(self, name):
        fn = getattr(self.eng, name)
        if not name.startswith("laplace_"):
            return fn

        def call(*a, **k):
            out = fn(*a, **k)
            if name != "laplace_matvec":
                s = self.eng.stats()
                for f in ("total_ms", "kbuild_ms", "sweep_ms", "update_ms", "lauum_ms", "solve_ms"):
                    self.acc[f] = self.acc.get(f, 0.0) + s[f]
                # device time of the call outside the named phases: scaling, diag(Ki_W_i) glue, rank-1 update and the
                # kernel-gradient reductions
                self.acc["other_ms"] = self.acc.get("other_ms", 0.0) + s["total_ms"] - sum(
                    s[f] for f in ("kbuild_ms", "sweep_ms", "update_ms", "lauum_ms", "solve_ms"))
                self.acc["sweep_flops"] = self.acc.get("sweep_flops", 0.0) + (
                    self.eng.N ** 3 * (2.0 / 3.0) if name in ("laplace_newton", "laplace_finish") else 0.0)
            self.calls[name] = self.calls.get(name, 0) + 1
            return out
        return call


def kernel_split(fn):
    """device ms of one call by kernel family (torch.profiler, CUDA activities): what the event phases lump together"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    fam = [("grad_reduction", ("grad_kinv_multi",)), ("rank1_update", ("laplace_rank1",)),
           ("u_scaling", ("laplace_scale_u",)), ("vector_glue", ("laplace_vec",)), ("col_sqnorm", ("col_sqnorm",)),
           ("b_build", ("laplace_bbuild",)), ("kbuild", ("kbuild", "prep")),
           ("matvecs", ("row_dot", "uv_", "utv")), ("gemm_and_lauum", ("gemm_panel", "gemm_lauum")),
           ("memset", ("Memset",)), ("copy", ("Memcpy",))]
    out = {k: 0.0 for k, _ in fam}
    out["factor_sweep"] = 0.0
    for ev in prof.events():
        if ev.device_type is None or "cuda" not in str(ev.device_type).lower():
            continue
        ms = (ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total) * 1e-3
        key = next((k for k, pats in fam if any(q in ev.name for q in pats)), "factor_sweep")
        out[key] += ms
    return out


def measure(N, peak):
    import gpy_b200 as B
    X, Y = data(N)
    kern = B.RBF(D, variance=1.3, lengthscale=LS, ARD=True)
    eng = B.Engine()
    out = {"N": N}
    for rep in range(2):    # the first evaluation warms up (allocations, module load)
        t = Timed(eng)
        inf = B.Laplace(engine=t)
        t0 = time.perf_counter()
        post, lml, gd = inf.inference(kern, X, B.Bernoulli(), Y)
        ms = (time.perf_counter() - t0) * 1e3
    a = t.acc
    Np = (N + 127) // 128 * 128
    gemm_flops = float(Np) ** 3     # C = LiW12 K with A lower triangular: half of 2 Np^3
    out.update(lml=float(lml), ms_per_eval=ms, newton_steps=inf.iterations, calls=t.calls,
               phases_ms={"kbuild": a["kbuild_ms"], "factor": a["sweep_ms"], "matvecs": a["solve_ms"],
                          "finish_gemm": a["update_ms"], "lauum": a["lauum_ms"], "reductions_and_glue": a["other_ms"],
                          "host_and_transfers": ms - a["total_ms"]},
               factor_tflops=a["sweep_flops"] / (a["sweep_ms"] * 1e9) if a["sweep_ms"] else None,
               gemm_tflops=gemm_flops / (a["update_ms"] * 1e9) if a["update_ms"] else None,
               fp64_peak_tflops=peak)
    out["kernel_split_ms"] = kernel_split(lambda: B.Laplace(engine=eng).inference(kern, X, B.Bernoulli(), Y))
    eng.set_data(X, Y)
    ex = []
    for _ in range(3):
        eng.exact_eval("rbf", True, 1.3, LS, 0.1)
        ex.append(eng.stats()["total_ms"])
    out["exact_ms"] = min(ex[1:])
    eng.close()
    return out


def reference_host(N=4096):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import importlib
    from oracle import ref_gpy
    G = ref_gpy.load()
    lap = importlib.import_module("GPy.inference.latent_function_inference.laplace")
    bern = importlib.import_module("GPy.likelihoods.bernoulli")
    X, Y = data(N)
    k = G.RBF(D, variance=1.3, lengthscale=LS, ARD=True)
    t0 = time.perf_counter()
    _, lml, _ = lap.Laplace().inference(k, X, bern.Bernoulli(), Y)
    ms = (time.perf_counter() - t0) * 1e3
    import platform
    import scipy
    return {"N": N, "ms_per_eval": ms, "lml": float(lml), "cpus": os.cpu_count(),
            "host": "%d-core %s host, NumPy %s, SciPy %s" % (os.cpu_count(), platform.machine(), np.__version__,
                                                             scipy.__version__),
            "note": "the reference's own Laplace with NumPy / SciPy on the host, one evaluation"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="*", default=[4096, 16384, 32768])
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_laplace.json"))
    ap.add_argument("--reference-host", action="store_true")
    args = ap.parse_args()
    if args.reference_host:
        res = json.load(open(args.out)) if os.path.exists(args.out) else {}
        res["reference_host"] = reference_host()
        print(json.dumps(res["reference_host"]))
    else:
        import gpy_b200 as B
        e = B.Engine()
        peak = e.measure_fp64_peak()
        e.close()
        res = {"card": card(), "kernel": "RBF(ARD), D = 8", "likelihood": "Bernoulli (probit)", "runs": []}
        for N in args.sizes:
            r = measure(N, peak)
            print(json.dumps(r), flush=True)
            res["runs"].append(r)
        res["card_after"] = card()
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
