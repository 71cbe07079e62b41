"""Test-only NumPy restatement of the joint posterior of GPy's exact and sparse models:

    covariance_between_points  K(X1, X2) - (L^-1 K(X, X1))^T (L^-1 K(X, X2))          posterior.py:109-130
    _raw_predict(full_cov)     mu = K(X*, X) alpha, Sigma = K(X*) - tmp^T tmp         posterior.py:273-302 (exact)
                               mu = K(X*, Z) wv,    Sigma = K(X*) - K(X*, Z) W K(Z, X*) posterior.py:238-270 (sparse)
    jitchol                    plain Cholesky, then mean(diag) 1e-6 10^k, k < maxtries util/linalg.py:56-75
    samples                    f_j = mu[:, j // S] + chol(Sigma + jitter I) z_j, z as np.random.multivariate_normal
                               draws it (one standard_normal((S, M)) per output)

The kernel is any object with K(X, X2=None) (sparse_composite_oracle.CompositeOracle, wide_composites_oracle.WideOracle).
"""
import numpy as np
from scipy.linalg import cho_factor, cho_solve, solve_triangular

JITTER = 1e-8   # exact_gaussian_inference.py:56


def exact_factor(kern, X, noise):
    """L of Ky = K + diag(noise + 1e-8) and alpha's solver"""
    Ky = kern.K(X) + np.diag(np.broadcast_to(np.asarray(noise, dtype=np.float64) + JITTER, (X.shape[0],)))
    return np.linalg.cholesky(Ky)


def covariance_between_points(kern, X, noise, X1, X2=None):
    """posterior.py:109-130; X2 None: K(X1) (exact zero distance on the diagonal) on the left"""
    L = exact_factor(kern, X, noise)
    tmp1 = solve_triangular(L, kern.K(X, X1), lower=True)
    tmp2 = tmp1 if X2 is None else solve_triangular(L, kern.K(X, X2), lower=True)
    return kern.K(X1, X2) - tmp1.T.dot(tmp2)


def exact_predict_full(kern, X, Y, noise, Xnew):
    """posterior.py:273-302 with full_cov -> (mu (M, P), Sigma (M, M))"""
    L = exact_factor(kern, X, noise)
    alpha = cho_solve((L, True), Y)
    Kx = kern.K(X, Xnew)
    tmp = solve_triangular(L, Kx, lower=True)
    return Kx.T.dot(alpha), kern.K(Xnew) - tmp.T.dot(tmp)


def sparse_predict_full(woodbury_vector, woodbury_inv, kern, Z, Xnew):
    """posterior.py:238-270 with pred_var = Z and full_cov -> (mu, Sigma)"""
    Kx = kern.K(Z, Xnew)
    return Kx.T.dot(woodbury_vector), kern.K(Xnew) - Kx.T.dot(woodbury_inv.dot(Kx))


def jitchol(A, maxtries=5):
    """util/linalg.py:56-75 -> (L, jitter added); raises LinAlgError like the reference"""
    A = np.ascontiguousarray(A)
    try:
        return np.linalg.cholesky(A), 0.0
    except np.linalg.LinAlgError:
        pass
    diagA = np.diag(A)
    if np.any(diagA <= 0.0):
        raise np.linalg.LinAlgError("not pd: non-positive diagonal elements")
    jitter = diagA.mean() * 1e-6
    num_tries = 1
    while num_tries <= maxtries and np.isfinite(jitter):
        try:
            return np.linalg.cholesky(A + np.eye(A.shape[0]) * jitter), jitter
        except np.linalg.LinAlgError:
            jitter *= 10
        num_tries += 1
    raise np.linalg.LinAlgError("not positive definite, even with jitter.")


def jitter_ladder(Sigma, maxtries=5):
    """the jitters jitchol may add: mean(diag) 1e-6 10^k, k < maxtries"""
    return [np.diag(Sigma).mean() * 1e-6 * 10.0 ** k for k in range(maxtries)]


def standard_normals(M, P, S):
    """what np.random.multivariate_normal(m, v, S) draws for P outputs in turn -> (P S, M)"""
    return np.concatenate([np.random.standard_normal((S, M)) for _ in range(P)], axis=0)


def samples(mu, Sigma, z, maxtries=5):
    """f (P S, M) in z's layout from mu (M, P) and Sigma through jitchol -> (f, jitter)"""
    L, jit = jitchol(Sigma, maxtries)
    P = mu.shape[1]
    S = z.shape[0] // P
    f = z.dot(L.T) + np.repeat(mu.T, S, axis=0)
    return f, jit


def as_fsim(f, P):
    """f (P S, M) -> GPy's (M, P, S)"""
    M = f.shape[1]
    return f.reshape(P, -1, M).transpose(2, 0, 1)


def cho_solve_sym(A, B):
    return cho_solve(cho_factor(A, lower=True), B)
