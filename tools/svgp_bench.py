"""Measure one SVGP step on the device (gpx_svgp_begin -> the likelihood's quadrature on the host -> gpx_svgp_finish):
probit Bernoulli, RBF(ARD), D = 8, 2^20 rows resident on the device, a contiguous minibatch of Nb rows, M inducing
inputs. Writes profiles/h100_svgp.json (or --out) with, per (Nb, M):
  the median ms per step and its split into begin / host quadrature / finish (host clock; both entries end in a device
  synchronise, as they return their results), the launches per step;
  the M^2 Nb products' flops (8 M^2 NBp, NBp = Nb padded to 128, counted from the shapes as include/gpx.h states them)
  over the begin + finish time: an end-to-end rate of the two entries, which also contain the M^3 work, the K builds and
  the reductions, against gpx_measure_fp64_peak measured in the same run.
The card name, power limit and SM clock are read in the same run (nvidia-smi queries only). Medians of --repeats steps
after one warm-up step per shape, each step at a new batch (row0 drawn from a seeded generator).

    python tools/svgp_bench.py [--nb 4096 16384 65536] [--m 512 1024 2048] [--out profiles/h100_svgp.json]
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

import gpy_b200  # noqa: E402
from gpy_b200 import _ffi  # noqa: E402

TILE = 128
N = 1 << 20


def parts():
    return [("rbf", 1, 0, list(range(D)), 1.3, np.array(LS))]


def step(eng, lik, Y, Z, q_m, q_L, row0, nb):
    t0 = time.perf_counter()
    mu, v, kl, _ = eng.svgp_begin(parts(), Z, q_m, q_L, row0, nb)
    t1 = time.perf_counter()
    F, dmu, dv, _ = lik.variational_expectations(Y[row0:row0 + nb], mu[:, None], v[:, None])
    s = N / float(nb)
    t2 = time.perf_counter()
    eng.svgp_finish(dmu[:, 0] * s, dv[:, 0] * s)
    t3 = time.perf_counter()
    return (t1 - t0) * 1e3, (t2 - t1) * 1e3, (t3 - t2) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nb", type=int, nargs="+", default=[4096, 16384, 65536])
    ap.add_argument("--m", type=int, nargs="+", default=[512, 1024, 2048])
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_svgp.json"))
    a = ap.parse_args()
    eng = _ffi.Engine(0)
    X, Y = data(N)
    eng.sparse_set_data(X, Y)
    lik = gpy_b200.Bernoulli()
    peak = eng.measure_fp64_peak()
    rng = np.random.default_rng(0)
    rows = []
    for M in a.m:
        Z = X[rng.choice(N, M, replace=False)].copy()
        q_m = 0.1 * rng.standard_normal(M)
        q_L = np.tril(0.01 * rng.standard_normal((M, M)), -1) + np.eye(M)
        for nb in a.nb:
            step(eng, lik, Y, Z, q_m, q_L, 0, nb)                                         # warm-up of the shape
            times, launches = [], []
            for _ in range(a.repeats):
                row0 = int(rng.integers(0, N - nb + 1))
                l0 = eng.total_launches()
                times.append(step(eng, lik, Y, Z, q_m, q_L, row0, nb))
                launches.append(eng.total_launches() - l0)
            t = np.median(np.array(times), axis=0)
            nbp = (nb + TILE - 1) // TILE * TILE
            flops = 8.0 * M * M * nbp
            dev_ms = float(t[0] + t[2])
            rows.append({"Nb": nb, "M": M, "ms_step": float(t.sum()), "ms_begin": float(t[0]),
                         "ms_host_quadrature": float(t[1]), "ms_finish": float(t[2]),
                         "launches_per_step": sorted(set(launches)),
                         "mnb_products_gflop": flops * 1e-9,
                         "mnb_products_tflops_over_begin_finish": flops / (dev_ms * 1e-3) * 1e-12,
                         "share_of_fp64_peak": flops / (dev_ms * 1e-3) * 1e-12 / peak})
            print(json.dumps(rows[-1]), flush=True)
    # the mirror's model: a stochastic_grad step (new batch, begin, quadrature, finish, gradients in optimizer space) with
    # the data resident; its host work does not grow with N
    M0, nb0 = a.m[0], a.nb[0]
    Z = X[rng.choice(N, M0, replace=False)].copy()
    m = gpy_b200.SVGP(X, Y, Z, gpy_b200.RBF(D, variance=1.3, lengthscale=np.array(LS), ARD=True), lik, batchsize=nb0,
                      engine=eng)
    x = m.optimizer_array.copy()
    m.stochastic_grad(x)
    mt = []
    for _ in range(a.repeats):
        t0 = time.perf_counter()
        m.stochastic_grad(x)
        mt.append((time.perf_counter() - t0) * 1e3)
    model = {"Nb": nb0, "M": M0, "ms_stochastic_grad": float(np.median(mt))}
    print(json.dumps(model), flush=True)
    out = {"model_step": model, "workload": "SVGP step, probit Bernoulli, RBF ARD D = %d, N = %d resident rows" % (D, N),
           "timing": "host clock around each entry (each ends in a device synchronise); medians of %d steps" % a.repeats,
           "fp64_peak_tflops_measured": peak, "card": card(), "rows": rows}
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
