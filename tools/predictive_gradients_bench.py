"""Time GP.predictive_gradients on the device against the host route the reference takes through the plugin.

Exact case: one RBF(ARD) evaluation at N = 16384, D = 8 (BASELINE.json configs[1]), then for M* in {1, 8, 64, 1024}:
    device  one gpx_predictive_gradients call (it returns after the Jacobians are on the host)
    host    the reference's GP.predictive_gradients over the plugin pair: K(X*, X) and gradients_X through the stand-alone
            device calls, -2 K(X*, X) K^-1 as a host np.dot, with K^-1 fetched once per posterior (gpx_get, timed apart)
The device time is split by torch.profiler (CUDA activities, a run of its own) into the K-build (point prep and K(X, X*)),
the U passes (utv / uv kernels: 2 ceil(M*/8) passes over U = L^-T, Npad^2/2 doubles each, reported as achieved bytes/s
against the data sheet's 3.35 TB/s) and the Jacobian reduction (pred_grad kernels).
Sparse case: one VarDTC RBF(ARD) evaluation at N = 262144, M = 4096, D = 16, M* in {1, 1024}, device and host routes;
the device call is timed on repeated calls (woodbury_inv kept from the first) and as the first call after an evaluation.
Medians of --steps calls after --warmup; the card's name, power limit and SM clock are read in the same run. Needs a GPU.

    python tools/predictive_gradients_bench.py [--steps 5] [--warmup 2] [--out profiles/h100_predictive_gradients.json]
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
HBM_BPS = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, watts, sm, smax = [s.strip() for s in q.split(",")]
    return dict(name=name, power_limit=watts, sm_clock=sm, sm_clock_max=smax)


def median_ms(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(steps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts)), ts


def split_ms(fn):
    """device time per phase of one call, from a torch.profiler run of its own"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = dict(kbuild=0.0, u_passes=0.0, reduction=0.0, other=0.0)
    for ev in prof.events():
        if ev.device_type is None or "cuda" not in str(ev.device_type).lower():
            continue
        name, us = ev.name, ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        if "prep" in name or "kbuild" in name:
            out["kbuild"] += us / 1e3
        elif "utv" in name or "uv_" in name:
            out["u_passes"] += us / 1e3
        elif "pred_grad" in name:
            out["reduction"] += us / 1e3
        else:
            out["other"] += us / 1e3
    return out


def exact_case(steps, warmup):
    from gpy_b200 import _ffi
    N, D = 16384, 8
    rng = np.random.default_rng(0)
    X = rng.uniform(-3, 3, (N, D))
    Y = np.sin(X).sum(1, keepdims=True) / np.sqrt(D) + 0.1 * rng.standard_normal((N, 1))
    ls = np.full(D, np.sqrt(D))
    e = _ffi.Engine(0)
    e.set_data(X, Y)
    e.exact_eval("rbf", True, 1.0, ls, 0.05)
    npad = (N + 127) // 128 * 128
    t0 = time.perf_counter()
    Kinv = e.get("Kinv")
    fetch_ms = (time.perf_counter() - t0) * 1e3
    alpha = e.get("alpha")
    rows = []
    for Ms in (1, 8, 64, 1024):
        Xn = rng.uniform(-3, 3, (Ms, D))
        dev_ms, dev_all = median_ms(lambda: e.predictive_gradients(Xn), steps, warmup)
        ph = split_ms(lambda: e.predictive_gradients(Xn))

        def host():
            mj = _ffi.kern_grad_X("rbf", True, 1.0, ls, Xn, np.broadcast_to(alpha[:, 0][None, :], (Ms, N)), X)
            a = -2.0 * np.dot(_ffi.kern_K("rbf", True, 1.0, ls, Xn, X), Kinv)
            return mj, _ffi.kern_grad_X("rbf", True, 1.0, ls, Xn, a, X)
        host_ms, host_all = median_ms(host, steps, warmup)
        passes = 2 * -(-Ms // 8)
        ubytes = passes * npad * npad / 2 * 8
        rows.append(dict(M_star=Ms, device_ms=dev_ms, device_all_ms=dev_all, host_ms=host_ms, host_all_ms=host_all,
                         split_ms=ph, u_passes=passes, u_bytes=ubytes,
                         u_bytes_per_s=ubytes / (ph["u_passes"] * 1e-3) if ph["u_passes"] > 0 else None,
                         u_share_of_hbm_peak=(ubytes / (ph["u_passes"] * 1e-3)) / HBM_BPS if ph["u_passes"] > 0 else None))
        print(json.dumps(rows[-1]), flush=True)
    return dict(N=N, D=D, kernel="RBF(ARD)", kinv_fetch_ms=fetch_ms, rows=rows)


def sparse_case(steps, warmup):
    from gpy_b200 import _ffi
    N, M, D = 262144, 4096, 16
    rng = np.random.default_rng(0)
    X = rng.uniform(-3, 3, (N, D))
    Y = np.sin(X).sum(1, keepdims=True) / np.sqrt(D) + 0.1 * rng.standard_normal((N, 1))
    Z = X[rng.permutation(N)[:M]].copy()
    ls = np.full(D, np.sqrt(D))
    e = _ffi.Engine(0)
    e.sparse_set_data(X, Y)
    e.sparse_eval("rbf", True, 1.0, ls, Z, 0.05)
    t0 = time.perf_counter()
    Wi = e.sparse_get("woodbury_inv")
    fetch_ms = (time.perf_counter() - t0) * 1e3
    wv = e.sparse_get("woodbury_vector")
    rows = []
    for Ms in (1, 1024):
        Xn = rng.uniform(-3, 3, (Ms, D))
        dev_ms, dev_all = median_ms(lambda: e.sparse_predictive_gradients(Xn), steps, warmup)
        first = []   # the first call after an evaluation also forms woodbury_inv (kept for the later calls)
        for _ in range(steps):
            e.sparse_eval("rbf", True, 1.0, ls, Z, 0.05)
            t0 = time.perf_counter()
            e.sparse_predictive_gradients(Xn)
            first.append((time.perf_counter() - t0) * 1e3)

        def host():
            mj = _ffi.kern_grad_X("rbf", True, 1.0, ls, Xn, np.broadcast_to(wv[:, 0][None, :], (Ms, M)), Z)
            a = -2.0 * np.dot(_ffi.kern_K("rbf", True, 1.0, ls, Xn, Z), Wi)
            return mj, _ffi.kern_grad_X("rbf", True, 1.0, ls, Xn, a, Z)
        host_ms, host_all = median_ms(host, steps, warmup)
        rows.append(dict(M_star=Ms, device_ms=dev_ms, device_all_ms=dev_all, device_first_call_ms=float(np.median(first)),
                         device_first_call_all_ms=first, host_ms=host_ms, host_all_ms=host_all))
        print(json.dumps(rows[-1]), flush=True)
    return dict(N=N, M=M, D=D, kernel="RBF(ARD)", woodbury_inv_fetch_ms=fetch_ms, rows=rows)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_predictive_gradients.json"))
    a = ap.parse_args()
    res = dict(card=card(), steps=a.steps, warmup=a.warmup, exact=exact_case(a.steps, a.warmup),
               sparse=sparse_case(a.steps, a.warmup))
    res["card_after"] = card()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print("wrote", a.out)


if __name__ == "__main__":
    main()
