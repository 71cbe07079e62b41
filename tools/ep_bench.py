"""Measure expectation propagation on the device (gpy_b200.EP over gpx_ep_*): GP classification with the probit Bernoulli
likelihood and RBF(ARD), D = 8, sequential updates, at N = 4096 / 16384. Writes profiles/h100_ep.json (or --out) with, per N:
  sweeps to convergence, ms of one full EP run (the cold start, every sweep and the marginal) and of one "alternated"-mode
  evaluation at a changed theta (gpx_ep_begin + gpx_ep_finish: K, the factor of B, Wi and the kernel gradient);
  ms per sweep split by the call's event phases (site updates = the block loop, factor of B, the recompute's two GEMMs,
  its mat-vecs) and, from torch.profiler over one sweep, the block loop by kernel (site chains, solves, rank-128 updates);
  the rank-128 updates' TFLOP/s (lower tiles only) and the recompute GEMMs' against gpx_measure_fp64_peak.
The card name, power limit and SM clock are read in the same run (nvidia-smi queries only).

    python tools/ep_bench.py [--sizes 4096 16384] [--out profiles/h100_ep.json]
    python tools/ep_bench.py --reference-host --out profiles/h100_ep.json
        adds the reference's own EP on the host at N = 1300 (needs the reference tree; no GPU) to an existing file
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


class Timed(object):
    """wraps an Engine: keeps the stats of every gpx_ep_sweep and the wall time of each EP call"""

    def __init__(self, eng):
        self.eng, self.sweeps, self.wall = eng, [], {}

    def __getattr__(self, name):
        fn = getattr(self.eng, name)
        if not name.startswith("ep_"):
            return fn

        def call(*a, **k):
            t0 = time.perf_counter()
            out = fn(*a, **k)
            self.wall[name] = self.wall.get(name, 0.0) + (time.perf_counter() - t0) * 1e3
            if name == "ep_sweep":
                self.sweeps.append(self.eng.stats())
            return out
        return call


def sweep_kernels(eng, N):
    """device ms of one sequential sweep by kernel (torch.profiler, CUDA activities)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    t, v = np.full(N, 0.5), np.zeros(N)
    eng.ep_start(t, v)
    order = np.random.RandomState(1).permutation(N)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.ep_sweep(order, t, v)
        torch.cuda.synchronize()
    evs = [ev for ev in prof.events() if ev.device_type is not None and "cuda" in str(ev.device_type).lower()]
    evs.sort(key=lambda ev: ev.time_range.start)
    # the blocks' rank-128 updates are the GEMM_UPDATE launches before the recompute's first B-build; those after it are
    # the factor sweep's trailing updates and the recompute's Sigma = K - D D^T
    first_b = next((i for i, ev in enumerate(evs) if "laplace_bbuild" in ev.name), len(evs))
    out = {"site_chain": 0.0, "solve": 0.0, "rank128_updates": 0.0, "rank128_launches": 0, "recompute": 0.0}
    for i, ev in enumerate(evs):
        ms = (ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total) * 1e-3
        if "ep_chain" in ev.name:
            out["site_chain"] += ms
        elif "ep_solve" in ev.name:
            out["solve"] += ms
        elif "gemm_update" in ev.name and i < first_b:
            out["rank128_updates"] += ms
            out["rank128_launches"] += 1
        elif i >= first_b:
            out["recompute"] += ms
    return out


def measure(N, peak):
    import gpy_b200 as B
    X, Y = data(N)
    eng = B.Engine()
    out = {"N": N}
    for rep in range(2):    # the first run warms up (allocations, module load)
        t = Timed(eng)
        inf = B.EP(engine=t)
        np.random.seed(0)
        t0 = time.perf_counter()
        inf.inference(B.RBF(D, variance=1.3, lengthscale=LS, ARD=True), X, B.Bernoulli(), Y)
        ms = (time.perf_counter() - t0) * 1e3
    k2 = B.RBF(D, variance=1.4, lengthscale=LS, ARD=True)
    t1 = time.perf_counter()
    inf.inference(k2, X, B.Bernoulli(), Y)                  # alternated: the sites are kept, begin + finish only
    alt_ms = (time.perf_counter() - t1) * 1e3
    s = t.sweeps
    n = len(s)
    avg = {f: sum(x[f] for x in s) / n for f in ("total_ms", "sweep_ms", "update_ms", "solve_ms")}
    site_ms = avg["total_ms"] - avg["sweep_ms"] - avg["update_ms"] - avg["solve_ms"]
    Np = (N + TILE - 1) // TILE * TILE
    nt = Np // TILE
    nblk = (N + TILE - 1) // TILE
    rank128_flops = nblk * nt * (nt + 1) / 2 * 2.0 * TILE ** 3          # lower tiles, k-depth 128, per sweep
    recompute_flops = float(Np) ** 3 + nt * (nt + 1) / 2 * 2.0 * TILE ** 2 * Np   # D = K U~ (B triangular), K - D D^T
    ks = sweep_kernels(eng, N)
    out.update(sweeps=inf.iterations, ms_full_ep=ms, ms_alternated_eval=alt_ms, ms_per_sweep=avg["total_ms"],
               sweep_phases_ms={"site_updates_block_loop": site_ms, "factor_of_B": avg["sweep_ms"],
                                "recompute_gemms": avg["update_ms"], "recompute_matvecs": avg["solve_ms"]},
               sweep_kernels_ms=ks,
               rank128_tflops=rank128_flops / (ks["rank128_updates"] * 1e9) if ks["rank128_updates"] else None,
               recompute_gemm_tflops=recompute_flops / (avg["update_ms"] * 1e9) if avg["update_ms"] else None,
               fp64_peak_tflops=peak, wall_ms_by_call=t.wall)
    eng.close()
    return out


def reference_host(N=1300):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import platform
    import scipy
    from ep_reference import load_reference_ep
    import make_laplace as ml
    EP, Bern, ObsAr = load_reference_ep()
    X, Y = data(N)
    parts = [dict(kind="rbf", term=0, dims=list(range(D)), variance=1.3, lengthscale=LS, ARD=True)]
    k = ml.reference_kernel(parts, D)
    np.random.seed(0)
    inf = EP()
    t0 = time.perf_counter()
    _, lml, _ = inf.inference(k, X, Bern(), ObsAr(Y))
    ms = (time.perf_counter() - t0) * 1e3
    return {"N": N, "ms_full_ep": ms, "lml": float(lml),
            "host": "%d-core %s host, NumPy %s, SciPy %s" % (os.cpu_count(), platform.machine(), np.__version__,
                                                             scipy.__version__),
            "note": "the reference's own EP (sequential updates) with NumPy / SciPy on the host, one inference call"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="*", default=[4096, 16384])
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_ep.json"))
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
        res = {"card": card(), "kernel": "RBF(ARD), D = 8", "likelihood": "Bernoulli (probit)",
               "updates": "sequential", "runs": []}
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
