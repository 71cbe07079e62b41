"""BASELINE.json metric in one run (SURVEY.md §8d): exact-GP log-marginal + gradient evaluations per second, fp64, RBF ARD
D=8, on one GPU at N in {512, 4096, 16384, 65536} (median of 3 after one warm-up, CUDA-event time) as absolute numbers and
as a fraction of the fp64 DMMA roofline (N^3 flops), beside the CPU oracle (GPy's operation sequence) on this host at
N in {512, 4096} (median of 3 after one warm-up; N=16384 is the cpu_baseline leg of bench.py;
N=65536 needs ~400 GiB of host memory with GPy's temporaries and is not run)."""
import json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from gpy_b200 import _ffi
from oracle import gpy_oracle as o
from bench import synthetic, theta_for_step, ensure_oracle_native

D = 8
sizes = [int(s) for s in sys.argv[1].split(",")] if len(sys.argv) > 1 else [512, 4096, 16384, 65536]
cpu_sizes = [int(s) for s in sys.argv[2].split(",")] if len(sys.argv) > 2 else [512, 4096]
native = ensure_oracle_native()
eng = _ffi.Engine(0)
peak = eng.measure_fp64_peak()
rows = []
for N in sizes:
    X, Y = synthetic(N, D)
    eng.set_data(X, Y)
    ms = []
    for s in range(4):
        lml, g, _ = eng.exact_eval("rbf", True, *theta_for_step(D, s))
        ms.append(eng.stats()["total_ms"])
    t = float(np.median(ms[1:]))
    row = {"N": N, "gpu_ms_per_eval": t, "gpu_evals_per_s": 1e3 / t, "tflops_N3": N ** 3 / t * 1e-9,
           "frac_of_fp64_dmma_peak": N ** 3 / t * 1e-9 / peak, "lml": lml}
    if N in cpu_sizes:
        cs = []
        for s in range(4):
            th = theta_for_step(D, s)
            t0 = time.perf_counter()
            l0, g0, _ = o.eval_lml_grad(X, Y, "rbf", True, *th, native=native)
            cs.append(time.perf_counter() - t0)
        row.update({"cpu_s_per_eval": float(np.median(cs[1:])), "cpu_evals_per_s": 1.0 / float(np.median(cs[1:])),
                    "parity_lml_abs": abs(l0 - lml), "parity_grad_rel_max": float(np.max(np.abs(g - g0) / np.abs(g0)))})
    rows.append(row)
    print(json.dumps(row), flush=True)
try:
    from threadpoolctl import threadpool_info
    blas = [{k: i.get(k) for k in ("internal_api", "version", "num_threads", "threading_layer")} for i in threadpool_info()]
except Exception:  # noqa: BLE001
    blas = None
print(json.dumps({"metric": "exact-GP log-marginal+grad evals/sec (fp64), RBF ARD D=8", "fp64_dmma_peak_tflops": peak,
                  "host_cpus": os.cpu_count(), "blas": blas, "rows": rows}))
