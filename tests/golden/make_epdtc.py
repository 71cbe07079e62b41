"""Writes tests/golden/epdtc/*.npz: the sparse EP as the reference's own EPDTC
(GPy/inference/latent_function_inference/expectation_propagation.py:436-611) and VarDTC (var_dtc.py) compute it with its
Bernoulli likelihood (probit) and kernels, executed through oracle/ref_gpy.py, after np.random.seed(seed), with the
gradient wiring of GPy/core/sparse_gp.py:100-119:

    lml, grad, dZ                   the bound, the kernel gradient (paramz order) and dL/dZ
    tau_tilde, v_tilde              the sites; cav_tau, cav_v the cavity parameters; log_Z_tilde
    post_mu, post_sd                mu and Sigma_diag of the last run's posteriorParamsDTC
    sweeps                          the sweeps of each EP run
    mu, var                         Posterior._raw_predict at Xnew with pred_var = Z
    next_random                     np.random.random() after the run: the orders drew from numpy's global generator
    cond_Kmm                        the condition number of K(Z, Z); host_seconds the reference's time for the case

Run from the repository root where the reference tree exists:  python tests/golden/make_epdtc.py
The kernels and inputs are those of tests/epdtc_oracle.py (CASES, case_data)."""
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), HERE]

import epdtc_oracle as eo  # noqa: E402
import make_laplace as ml  # noqa: E402
from epdtc_reference import load_reference_epdtc  # noqa: E402


def reference_case(name):
    EPDTC, Bern, ObsAr = load_reference_epdtc()
    parts, N, M, seed, opts = eo.CASES[name]
    X, Y, Z, Xnew = eo.case_data(name)
    kern = ml.reference_kernel(parts, X.shape[1])
    lik = Bern()
    kw = {k: opts[k] for k in ("eta", "delta", "max_iters", "parallel_updates", "ep_mode") if k in opts}
    inf = EPDTC(**kw)
    sweeps = []
    run, loc = inf.expectation_propagation, inf._local_updates

    def counted_run(*a, **k):
        sweeps.append(0)
        return run(*a, **k)

    def counted_local(*a, **k):
        sweeps[-1] += 1
        return loc(*a, **k)

    inf.expectation_propagation, inf._local_updates = counted_run, counted_local
    t0 = time.perf_counter()
    np.random.seed(seed)
    Yo = ObsAr(Y)
    post, lml, gd = inf.inference(kern, X, Z, lik, Yo)
    if opts.get("calls") == 2:
        post, lml, gd = inf.inference(kern, X, Z, lik, Yo)
    if "theta2" in opts:
        kern = ml.reference_kernel(eo.scaled_parts(parts, opts["theta2"]), X.shape[1])
        post, lml, gd = inf.inference(kern, X, Z, lik, Yo)
    if "z2" in opts:
        Z = Z + opts["z2"]
        post, lml, gd = inf.inference(kern, X, Z, lik, Yo)
    secs = time.perf_counter() - t0
    # sparse_gp.py:100-119
    kern.update_gradients_diag(gd["dL_dKdiag"], X)
    g = kern.gradient.copy()
    kern.update_gradients_full(gd["dL_dKnm"], X, Z)
    g += kern.gradient
    kern.update_gradients_full(gd["dL_dKmm"], Z, None)
    g += kern.gradient
    dZ = kern.gradients_X(gd["dL_dKmm"], Z) + kern.gradients_X(gd["dL_dKnm"].T, Z, X)
    mu, var = post._raw_predict(kern, Xnew, Z, full_cov=False)
    pp, ga, logZ = inf._ep_approximation
    return dict(lml=float(np.squeeze(lml)), grad=np.asarray(g, dtype=np.float64), dZ=np.asarray(dZ),
                tau_tilde=np.asarray(ga.tau).copy(), v_tilde=np.asarray(ga.v).copy(),
                log_Z_tilde=float(logZ), post_mu=np.asarray(pp.mu).copy(), post_sd=np.asarray(pp.Sigma_diag).copy(),
                sweeps=np.array(sweeps), mu=np.asarray(mu), var=np.asarray(var), next_random=np.random.random(),
                cond_Kmm=np.linalg.cond(kern.K(Z)), host_seconds=secs, Z_final=Z)


def main():
    os.makedirs(os.path.join(HERE, "epdtc"), exist_ok=True)
    for name in (sys.argv[1:] or eo.CASES):
        X, Y, Z, Xnew = eo.case_data(name)
        r = reference_case(name)
        np.savez_compressed(os.path.join(HERE, "epdtc", name + ".npz"), X=X, Y=Y, Z=Z, Xnew=Xnew, **r)
        print(name, r["lml"], "sweeps", r["sweeps"], "at the clip", int(np.sum(r["post_sd"] <= eo.EPS)),
              "cond %.2e" % r["cond_Kmm"], "%.1f s" % r["host_seconds"])


if __name__ == "__main__":
    main()
