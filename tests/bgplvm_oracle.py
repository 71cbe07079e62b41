"""Test-only NumPy restatement of one Bayesian GPLVM evaluation (GPy/models/bayesian_gplvm.py:20-101 on
SparseGP.parameters_changed, sparse_gp.py:76-107): the RBF psi-statistics and their derivatives (rbf_psi_comp.py:8-136), the
uncertain-input VarDTC evaluation (var_dtc.py:66-262) and the NormalPrior KL term (variational.py:29-37). The fixture cases
(tests/golden/make_bgplvm.py) are listed here so that the generator and the tests build the same inputs.
"""
import numpy as np
import scipy.linalg as sla

from gplvm_oracle import latent_data
from sparse_composite_oracle import CompositeOracle


def psi_stats(variance, ls, Z, mu, S):
    """-> psi0 (N,), psi1 (N x M), psi2 = sum_n psi2_n (M x M)"""
    l2 = np.square(np.broadcast_to(ls, (mu.shape[1],)))
    d1 = 1.0 / (S + l2)
    psi1 = variance * np.exp(-0.5 * np.log1p(S / l2).sum(1)[:, None]
                             - 0.5 * np.einsum("nmq,nq->nm", np.square(mu[:, None, :] - Z[None, :, :]), d1))
    d2 = 1.0 / (2.0 * S + l2)
    zh = 0.5 * (Z[:, None, :] + Z[None, :, :])
    e1 = -0.25 * (np.square(Z[:, None, :] - Z[None, :, :]) / l2).sum(-1)
    psi2 = np.zeros((Z.shape[0], Z.shape[0]))
    for n in range(mu.shape[0]):
        e = -0.5 * np.log1p(2.0 * S[n] / l2).sum() + e1 - (np.square(mu[n] - zh) * d2[n]).sum(-1)
        psi2 += np.exp(e)
    return np.full(mu.shape[0], float(variance)), psi1, variance * variance * psi2


def psi_derivs(dL_dpsi0, dL_dpsi1, dL_dpsi2, variance, ls, Z, mu, S, ard):
    """psiDerivativecomputations -> (grad [variance, lengthscale (1 or Q)], dZ, dmu, dS)"""
    Q = mu.shape[1]
    l = np.broadcast_to(ls, (Q,)).astype(np.float64)
    l2 = l * l
    _, psi1, _ = psi_stats(variance, ls, Z, mu, S)
    L1 = dL_dpsi1 * psi1
    Zmu = Z[None, :, :] - mu[:, None, :]
    d1 = 1.0 / (S + l2)
    Zmu2d = np.square(Zmu) * d1[:, None, :]
    dvar = L1.sum() / variance
    dmu = np.einsum("nm,nmq,nq->nq", L1, Zmu, d1)
    dS = np.einsum("nm,nmq,nq->nq", L1, Zmu2d - 1.0, d1) / 2.0
    dZ = -np.einsum("nm,nmq,nq->mq", L1, Zmu, d1)
    dl = np.einsum("nm,nmq,nq->q", L1, Zmu2d + (S / l2)[:, None, :], d1 * l)
    dLs = 0.5 * (dL_dpsi2 + dL_dpsi2.T)
    d2 = 1.0 / (2.0 * S + l2)
    zh = 0.5 * (Z[:, None, :] + Z[None, :, :])
    dz = Z[:, None, :] - Z[None, :, :]
    e1 = -0.25 * (np.square(dz) / l2).sum(-1)
    for n in range(mu.shape[0]):
        diff = mu[n] - zh                                                            # M x M x Q
        L2 = dLs * variance ** 2 * np.exp(-0.5 * np.log1p(2.0 * S[n] / l2).sum() + e1 - (np.square(diff) * d2[n]).sum(-1))
        Ls, sa, sb = L2.sum(), np.einsum("ab,abq->q", L2, diff), np.einsum("ab,abq->q", L2, np.square(diff))
        dvar += 2.0 * Ls / variance
        dmu[n] += -2.0 * d2[n] * sa
        dS[n] += 2.0 * d2[n] ** 2 * sb - d2[n] * Ls
        dl += 2.0 * l * (S[n] * d2[n] / l2 * Ls + d2[n] ** 2 * sb) + np.einsum("ab,abq->q", L2, np.square(dz)) / (2.0 * l ** 3)
        dZ += 2.0 * (np.einsum("ab,abq->aq", L2, -dz) / (2.0 * l2) + np.einsum("ab,abq->aq", L2, diff) * d2[n])
    dvar += np.sum(dL_dpsi0)
    return np.concatenate([[dvar], dl if ard else [dl.sum()]]), dZ, dmu, dS


def _parts(variance, ls, ard, Q):
    return [dict(kind="rbf", term=0, dims=list(range(Q)), variance=variance,
                 lengthscale=list(np.atleast_1d(ls)) if ard else float(np.atleast_1d(ls)[0]), ARD=bool(ard))]


def vardtc_psi(variance, ls, ard, Z, mu, S, Y, noise):
    """the uncertain-input VarDTC evaluation with the gradient wiring of sparse_gp.py:88-107 ->
    dict(lml (no KL), grad [variance, lengthscale.., noise], dZ, dmu, dS, woodbury_vector, woodbury_inv, dL_dpsi*)"""
    N, P = Y.shape
    M, Q = Z.shape
    kern = CompositeOracle(_parts(variance, ls, ard, Q))
    beta = 1.0 / max(noise, 1e-8)
    psi0, psi1, psi2 = psi_stats(variance, ls, Z, mu, S)
    Kmm = kern.K(Z) + 1e-8 * np.eye(M)
    Lm = np.linalg.cholesky(Kmm)
    Lmi = sla.solve_triangular(Lm, np.eye(M), lower=True)
    A = Lmi.dot(psi2 * beta).dot(Lmi.T)
    B = np.eye(M) + A
    LB = np.linalg.cholesky(B)
    tmp = sla.solve_triangular(Lm, psi1.T, lower=True)
    LBi_Lmi_psi1 = sla.solve_triangular(LB, tmp, lower=True)
    VVT = beta * Y
    LBi_Lmi_psi1Vf = LBi_Lmi_psi1.dot(VVT)
    tmp = sla.solve_triangular(LB, LBi_Lmi_psi1Vf, lower=True, trans=1)
    Cpsi1Vf = sla.solve_triangular(Lm, tmp, lower=True, trans=1)
    delit = LBi_Lmi_psi1Vf.dot(LBi_Lmi_psi1Vf.T)
    data_fit = np.trace(delit)
    LBi = sla.solve_triangular(LB, np.eye(M), lower=True)
    DBi = LBi.T.dot(P * np.eye(M) + delit).dot(LBi)
    Lmit = Lmi.T
    dL_dKmm = Lmit.dot(-0.5 * DBi - 0.5 * B * P + P * np.eye(M)).dot(Lmi)
    dL_dpsi0 = -0.5 * P * beta * np.ones(N)
    dL_dpsi1 = VVT.dot(Cpsi1Vf.T)
    dL_dpsi2 = beta * 0.5 * Lmit.dot(P * np.eye(M) - DBi).dot(Lmi)
    trYYT = np.sum(Y * Y)
    lml = (-0.5 * N * P * (np.log(2 * np.pi) - np.log(beta)) - 0.5 * beta * trYYT
           - 0.5 * P * (beta * psi0.sum() - np.trace(A)) - P * np.sum(np.log(np.diag(LB))) + 0.5 * data_fit)
    dL_dR = -0.5 * N * P * beta + 0.5 * trYYT * beta ** 2
    dL_dR += 0.5 * P * (psi0.sum() * beta ** 2 - np.trace(A) * beta)
    dL_dR += beta * (0.5 * np.sum(A * DBi) - data_fit)
    g_psi, dZ_psi, dmu, dS = psi_derivs(dL_dpsi0, dL_dpsi1, dL_dpsi2, variance, ls, Z, mu, S, ard)
    g_kmm = kern.grads_full(dL_dKmm, Z, None)[0]
    dZ = kern.gradients_X(dL_dKmm, Z) + dZ_psi
    Bi = -LBi.T.dot(LBi) + np.eye(M)
    return dict(lml=lml, grad=np.concatenate([g_psi + g_kmm, [dL_dR]]), dZ=dZ, dmu=dmu, dS=dS,
                woodbury_vector=Cpsi1Vf, woodbury_inv=Lmit.dot(Bi).dot(Lmi), dL_dpsi0=dL_dpsi0, dL_dpsi1=dL_dpsi1,
                dL_dpsi2=dL_dpsi2, dL_dKmm=dL_dKmm)


def kl(mu, S):
    """NormalPrior.KL_divergence (variational.py:29-32) and its gradients w.r.t. mu and S (:34-37, sign of the bound)"""
    v = 0.5 * (np.square(mu).sum() + (S - np.log(S)).sum()) - 0.5 * mu.size
    return v, -mu, -0.5 * (1.0 - 1.0 / S)


def bgplvm_eval(variance, ls, ard, Z, mu, S, Y, noise):
    """-> (bound, grad [mu row-major, S row-major, Z row-major, variance, lengthscale.., noise])"""
    r = vardtc_psi(variance, ls, ard, Z, mu, S, Y, noise)
    k, gmu, gS = kl(mu, S)
    return r["lml"] - k, np.concatenate([(r["dmu"] + gmu).ravel(), (r["dS"] + gS).ravel(), r["dZ"].ravel(), r["grad"]])


# fixture cases: N, P, Q, M, seeds, the kernel (variance, lengthscale, ARD), noise and the scale of S
CASES = {
    "default_p1": dict(N=60, P=1, Q=3, M=10, seed=11, variance=1.1, ls=[0.9, 1.3, 1.7], ard=True, noise=0.05, s=(0.05, 0.3)),
    "default_p8": dict(N=70, P=8, Q=3, M=12, seed=12, variance=0.8, ls=[1.2, 0.7, 1.4], ard=True, noise=0.1, s=(0.05, 0.3)),
    "default_p9": dict(N=70, P=9, Q=4, M=12, seed=13, variance=1.0, ls=[1.1, 0.9, 1.6, 2.0], ard=True, noise=0.1,
                       s=(0.05, 0.3)),
    "default_p12": dict(N=80, P=12, Q=5, M=16, seed=14, variance=1.3, ls=[1.0, 1.2, 1.5, 0.8, 2.2], ard=True, noise=0.08,
                        s=(0.02, 0.2)),
    "default_p64": dict(N=90, P=64, Q=3, M=14, seed=15, variance=0.9, ls=[0.8, 1.1, 1.9], ard=True, noise=0.2,
                        s=(0.05, 0.3)),
    "iso": dict(N=60, P=2, Q=3, M=10, seed=16, variance=1.2, ls=[1.1], ard=False, noise=0.07, s=(0.05, 0.3)),
    "n1300_m129": dict(N=1300, P=3, Q=3, M=129, seed=17, variance=1.0, ls=[0.4, 0.5, 0.6], ard=True, noise=0.1,
                       s=(0.01, 0.1)),
    "n_eq_m": dict(N=24, P=2, Q=2, M=24, seed=18, variance=1.0, ls=[0.3, 0.4], ard=True, noise=0.1, s=(0.05, 0.3)),
    "s_tiny": dict(N=50, P=2, Q=3, M=9, seed=19, variance=1.0, ls=[1.0, 1.2, 0.9], ard=True, noise=0.1, s=(5e-7, 2e-6)),
    "s_large": dict(N=50, P=2, Q=3, M=9, seed=20, variance=1.0, ls=[1.0, 1.2, 0.9], ard=True, noise=0.1, s=(8.0, 12.0)),
    "dup_z": dict(N=50, P=2, Q=2, M=10, seed=21, variance=1.0, ls=[1.1, 0.8], ard=True, noise=0.1, s=(0.05, 0.3),
                  dup=True),
    "q12": dict(N=64, P=3, Q=12, M=20, seed=22, variance=1.0, ls=list(np.linspace(1.0, 3.0, 12)), ard=True, noise=0.1,
                s=(0.05, 0.3)),
}


def case_inputs(case):
    """mu (N x Q), S (N x Q), Z (M x Q), Y (N x P) and new latent points Xnew (7 x Q) of a fixture case"""
    mu, Y = latent_data(case["N"], case["Q"], case["P"], case["seed"])
    rng = np.random.default_rng(case["seed"] + 100)
    S = rng.uniform(case["s"][0], case["s"][1], size=mu.shape)
    Z = mu[rng.permutation(case["N"])[:case["M"]]].copy()
    if case.get("dup"):
        Z[1] = Z[0]
    Xnew = rng.uniform(-1.5, 1.5, size=(7, case["Q"]))
    return mu, S, Z, Y, Xnew


def psi_case():
    """the stand-alone psi case: mu, S, Z, kernel and random dL_dpsi0 (N), dL_dpsi1 (N x M), dL_dpsi2 (M x M)"""
    rng = np.random.default_rng(7)
    N, M, Q = 40, 11, 3
    mu = rng.uniform(-1.5, 1.5, size=(N, Q))
    S = rng.uniform(0.05, 0.5, size=(N, Q))
    Z = rng.uniform(-1.5, 1.5, size=(M, Q))
    return dict(mu=mu, S=S, Z=Z, variance=1.3, ls=np.array([0.8, 1.1, 1.6]), dL0=rng.standard_normal(N),
                dL1=rng.standard_normal((N, M)), dL2=rng.standard_normal((M, M)))


_ref_bgplvm = None


def reference_bayesian_gplvm():
    """-> (the reference's own BayesianGPLVM class, the namespace of oracle/ref_gpy.load_sparse_models(), its variational
    module). oracle/ref_gpy.py stubs the psi_comp package for the other tests; this loader installs the reference's real
    GPy/kern/src/psi_comp package (PyCUDA is imported only inside its GPU module's functions) and points rbf.py's
    PSICOMP_RBF at it, so every RBF built afterwards computes its psi-statistics with the unmodified rbf_psi_comp.py.
    Not the reference's code: the paramz stand-in has no parameter indexing, so slicing a NormalPosterior by its kernel's
    active dims (kern.py:112-117 through kernel_slice_operations.py) returns the posterior itself when the dims are every
    column in order, as the real indexing returns an equal view (variational.py:125-141), and a fresh NormalPosterior of
    the sliced arrays otherwise."""
    global _ref_bgplvm
    if _ref_bgplvm is not None:
        return _ref_bgplvm
    import importlib
    import importlib.util
    import sys
    from oracle import ref_gpy
    S = ref_gpy.load_sparse_models()
    path = ref_gpy.REF + "/GPy/kern/src/psi_comp"
    spec = importlib.util.spec_from_file_location("GPy.kern.src.psi_comp", path + "/__init__.py",
                                                  submodule_search_locations=[path])
    real = importlib.util.module_from_spec(spec)
    sys.modules["GPy.kern.src.psi_comp"] = real
    spec.loader.exec_module(real)
    sys.modules["GPy.kern.src"].psi_comp = real
    rbf_mod = sys.modules["GPy.kern.src.rbf"]
    rbf_mod.PSICOMP_RBF, rbf_mod.PSICOMP_RBF_GPU = real.PSICOMP_RBF, real.PSICOMP_RBF_GPU
    V = sys.modules["GPy.core.parameterization.variational"]

    def getitem(self, s):
        cols = s[1] if isinstance(s, tuple) and len(s) == 2 and s[0] == slice(None) else None
        if cols is not None and np.array_equal(np.atleast_1d(cols), np.arange(self.mean.shape[1])):
            return self
        return V.NormalPosterior(np.asarray(self.mean)[s], np.asarray(self.variance)[s])
    V.VariationalPosterior.__getitem__ = getitem
    BG = importlib.import_module("GPy.models.bayesian_gplvm").BayesianGPLVM
    _ref_bgplvm = (BG, S, V)
    return _ref_bgplvm
