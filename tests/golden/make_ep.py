"""Writes tests/golden/ep/*.npz: expectation propagation as the reference's own EP
(GPy/inference/latent_function_inference/expectation_propagation.py) computes it with its Bernoulli likelihood (probit)
and kernels (stationary.py, rbf.py, add.py, prod.py, static.py), executed through oracle/ref_gpy.py, after
np.random.seed(seed), with the gradient wiring of GPy/core/gp.py:278-280:

    lml, grad                       the log marginal and the kernel gradient (paramz order)
    tau_tilde, v_tilde              the sites; cav_tau, cav_v the cavity parameters; log_Z_tilde
    sweeps                          the sweeps of each EP run
    mu, var                         PosteriorEP._raw_predict at Xnew (posterior.py:305-336)
    woodbury_inv                    only for N <= 150 (Wi)
    next_random                     np.random.random() after the run: the orders drew from numpy's global generator

The reference's own expectation_propagation.py is loaded by tests/ep_reference.py.
Run from the repository root where the reference tree exists:  python tests/golden/make_ep.py
The kernels and inputs are those of tests/ep_oracle.py (CASES, case_data)."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), HERE]

from oracle import ref_gpy  # noqa: E402
import ep_oracle as eo  # noqa: E402
import make_laplace as ml  # noqa: E402
from ep_reference import load_reference_ep  # noqa: E402


def reference_case(name):
    EP, Bern, ObsAr = load_reference_ep()
    parts, N, seed, opts = eo.CASES[name]
    X, Y, Xnew = eo.case_data(name)
    kern = ml.reference_kernel(parts, X.shape[1])
    lik = Bern()
    kw = {k: opts[k] for k in ("eta", "delta", "max_iters", "parallel_updates", "ep_mode") if k in opts}
    inf = EP(**kw)
    sweeps = []                                     # the sweeps of each EP run: _local_updates calls per run
    run, loc = inf.expectation_propagation, inf._local_updates

    def counted_run(*a, **k):
        sweeps.append(0)
        return run(*a, **k)

    def counted_local(*a, **k):
        sweeps[-1] += 1
        return loc(*a, **k)

    inf.expectation_propagation, inf._local_updates = counted_run, counted_local
    np.random.seed(seed)
    Yo = ObsAr(Y)
    post, lml, gd = inf.inference(kern, X, lik, Yo)
    if opts.get("calls") == 2:
        post, lml, gd = inf.inference(kern, X, lik, Yo)
    if "theta2" in opts:
        kern = ml.reference_kernel(eo.scaled_parts(parts, opts["theta2"]), X.shape[1])
        post, lml, gd = inf.inference(kern, X, lik, Yo)
    kern.update_gradients_full(gd["dL_dK"], X)                                   # gp.py:280
    mu, var = post._raw_predict(kern, Xnew, X, full_cov=False)
    ga, cav, logZ = inf._ep_approximation[1], inf._ep_approximation[2], inf._ep_approximation[3]
    return dict(lml=float(np.squeeze(lml)), grad=np.asarray(kern.gradient, dtype=np.float64).copy(),
                tau_tilde=np.asarray(ga.tau).copy(), v_tilde=np.asarray(ga.v).copy(), cav_tau=np.asarray(cav.tau).copy(),
                cav_v=np.asarray(cav.v).copy(), log_Z_tilde=float(logZ), sweeps=np.array(sweeps), mu=np.asarray(mu),
                var=np.asarray(var), woodbury_inv=np.asarray(post.woodbury_inv), next_random=np.random.random())


def main():
    os.makedirs(os.path.join(HERE, "ep"), exist_ok=True)
    for name in (sys.argv[1:] or eo.CASES):
        N = eo.CASES[name][1]
        X, Y, Xnew = eo.case_data(name)
        r = reference_case(name)
        if N > eo.SMALL_N:
            del r["woodbury_inv"]
        np.savez_compressed(os.path.join(HERE, "ep", name + ".npz"), X=X, Y=Y, Xnew=Xnew, **r)
        print(name, r["lml"], "sweeps", r["sweeps"], "tau~ at the clip", int(np.sum(r["tau_tilde"] <= eo.EPS)))


if __name__ == "__main__":
    main()
