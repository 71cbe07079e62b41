"""The cases of the sparse-prediction fixtures (tests/golden/make_sparse_predict.py) and a test-only NumPy restatement of
the prediction the reference's VarDTC posterior makes, Posterior._raw_predict (posterior.py:220-248) with pred_var = Z:

    mu   = K(Xnew, Z) woodbury_vector
    var  = clip(Kdiag(Xnew) - rowsum((K(Xnew, Z) W) o K(Xnew, Z)), 1e-15)     (full_cov = False; posterior.py:248)
    cov  = K(Xnew) - K(Xnew, Z) W K(Z, Xnew)                                  (full_cov = True; not clipped)

Kernels are part dicts of tests/sparse_composite_oracle.py (CompositeOracle); the test points of every case lie on Z, on X
and far from both."""
import numpy as np

from sparse_composite_oracle import CompositeOracle, case_data

N, M, D = 200, 30, 3
CLIP = 1e-15   # posterior.py:248

CASES = {
    "rbf_ard_p1": dict(parts=[dict(kind="rbf", term=0, dims=[0, 1, 2], variance=1.3, lengthscale=[0.9, 1.4, 2.1],
                                   ARD=True)], P=1, seed=701),
    "matern32_iso_p3": dict(parts=[dict(kind="matern32", term=0, dims=[0, 1, 2], variance=0.9, lengthscale=1.1)], P=3,
                            seed=702),
    "exponential_ard_het": dict(parts=[dict(kind="exponential", term=0, dims=[0, 1, 2], variance=1.1,
                                            lengthscale=[1.6, 2.4, 1.9], ARD=True)], P=1, seed=703, het=True),
    "rbf_bias_white": dict(parts=[dict(kind="rbf", term=0, dims=[0, 1, 2], variance=1.3, lengthscale=[0.9, 1.4, 2.1],
                                       ARD=True),
                                  dict(kind="bias", term=1, variance=0.4),
                                  dict(kind="white", term=2, variance=0.07)], P=1, seed=704),
    "m52_x_rbf_bias_p2": dict(parts=[dict(kind="matern52", term=0, dims=[0, 1], variance=1.1, lengthscale=1.2),
                                     dict(kind="rbf", term=0, dims=[1, 2], variance=0.8, lengthscale=[1.5, 0.7],
                                          ARD=True),
                                     dict(kind="bias", term=1, variance=0.3)], P=2, seed=705),
    # kernel variance 1e-18: every diagonal variance falls below the clip, the reference returns exactly 1e-15
    "clip_rbf_tiny_variance": dict(parts=[dict(kind="rbf", term=0, dims=[0, 1, 2], variance=1e-18, lengthscale=1.0)],
                                   P=1, seed=706),
}


def inputs(c):
    """-> X, Y, Z, noise, Xnew of a case; Xnew: 6 rows of Z, 6 rows of X, 6 points far from both"""
    X, Y, Z, noise = case_data(N, M, D, c["P"], c["seed"], c.get("het", False))
    rng = np.random.default_rng(c["seed"] + 1)
    far = 8.0 + rng.uniform(0.0, 1.0, size=(6, D))
    Xnew = np.concatenate([Z[:6], X[10:16], far])
    return X, Y, Z, noise, Xnew


def predict(woodbury_vector, woodbury_inv, kern, Z, Xnew, full_cov=False):
    """posterior.py:220-248 -> (mu (M*, P), var (M*, 1) clipped, or cov (M*, M*))"""
    Kx = kern.K(Z, Xnew)
    mu = Kx.T.dot(woodbury_vector)
    if full_cov:
        return mu, kern.K(Xnew) - Kx.T.dot(woodbury_inv.dot(Kx))
    var = (kern.Kdiag(Xnew) - np.sum(woodbury_inv.T.dot(Kx) * Kx, 0))[:, None]
    return mu, np.clip(var, CLIP, np.inf)


def oracle_kernel(c):
    return CompositeOracle(c["parts"])
