"""Writes tests/golden/bgplvm/*.npz from the reference's own code: VarDTC.inference with a NormalPosterior X
(GPy/inference/latent_function_inference/var_dtc.py:66-215, uncertain_inputs), the unmodified RBF psi-statistics module
GPy/kern/src/psi_comp/rbf_psi_comp.py, the RBF kernel's K / update_gradients_full / gradients_X for the Kmm part, and
NormalPrior.KL_divergence / update_gradients_KL (variational.py:29-37), wired as SparseGP._update_gradients
(sparse_gp.py:88-107) and BayesianGPLVM.parameters_changed (bayesian_gplvm.py:86-101) wire them. oracle/ref_gpy.py stubs
the psi_comp package for the other tests; this generator loads the real rbf_psi_comp.py by path (PyCUDA is imported
only inside the GPU module, which is not loaded).
Each fixture records mu, S, Z, Y, the kernel, the noise, the bound without the KL term (`lml`), the bound (`bound`), the
gradient [variance, lengthscale.., noise] (`grad`), dZ, dmu and dS (without the KL gradient), the KL gradients
(`kl_mu`, `kl_S`) and predict at new latent points. `psi.npz` records psi0/psi1/psi2 and psiDerivativecomputations for
random dL_dpsi.
Run from the repository root:
    python tests/golden/make_bgplvm.py [case ...]      (no case: all of them)
"""
import importlib.util
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
OUT = os.path.join(ROOT, "tests", "golden", "bgplvm")

from bgplvm_oracle import CASES, case_inputs, psi_case  # noqa: E402


def reference():
    """-> (G namespace of oracle/ref_gpy.py, the real rbf_psi_comp module, variational module)"""
    from oracle import ref_gpy
    S = ref_gpy.load_sparse_models()
    spec = importlib.util.spec_from_file_location(
        "gpx_ref_rbf_psi_comp", os.path.join(ref_gpy.REF, "GPy", "kern", "src", "psi_comp", "rbf_psi_comp.py"))
    psi = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(psi)
    return S.G, psi, sys.modules["GPy.core.parameterization.variational"]


class PsiKern(object):
    """the reference RBF with its psi-statistics from rbf_psi_comp.py (what RBF.psi0/1/2 call, rbf.py:80-101)"""

    def __init__(self, G, psi, Q, variance, ls, ard):
        self.rbf = G.RBF(Q, variance, np.array(ls, dtype=np.float64), ARD=ard)
        self.psi, self.variance, self.ls = psi, variance, np.array(ls, dtype=np.float64)

    def K(self, X, X2=None):
        return self.rbf.K(X, X2)

    def Kdiag(self, X):
        return self.rbf.Kdiag(X)

    def _stats(self, Z, qX):
        return self.psi.psicomputations(self.variance, self.ls, Z, qX)

    def psi0(self, Z, qX):
        return self._stats(Z, qX)[0]

    def psi1(self, Z, qX):
        return self._stats(Z, qX)[1]

    def psi2(self, Z, qX):
        return self._stats(Z, qX)[2]


def evaluate(G, psi, V, case):
    mu, S, Z, Y, Xnew = case_inputs(case)
    Q = case["Q"]
    kern = PsiKern(G, psi, Q, case["variance"], case["ls"], case["ard"])
    qX = V.NormalPosterior(mu, S)
    lik = G.Gaussian(variance=case["noise"])
    post, lml, gd = G.VarDTC().inference(kern, qX, Z, lik, Y)
    # SparseGP._update_gradients, uncertain branch (sparse_gp.py:88-107)
    kern.rbf.update_gradients_full(gd["dL_dKmm"], Z, None)
    g_kmm = np.asarray(kern.rbf.gradient, dtype=np.float64).copy()
    dvar, dl, dZp, dmu, dS = psi.psiDerivativecomputations(gd["dL_dpsi0"], gd["dL_dpsi1"], gd["dL_dpsi2"],
                                                           case["variance"], kern.ls, Z, qX)
    grad = np.concatenate([[dvar], np.atleast_1d(dl), [0.0]]) + np.concatenate([g_kmm, [0.0]])
    grad[-1] = float(np.sum(gd["dL_dthetaL"]))
    dZ = np.asarray(kern.rbf.gradients_X(gd["dL_dKmm"], Z), dtype=np.float64) + dZp
    # BayesianGPLVM.parameters_changed: minus KL, update_gradients_KL (bayesian_gplvm.py:86-101)
    prior = V.NormalPrior()
    klv = float(prior.KL_divergence(qX))
    qX.mean.gradient[:] = 0.0
    qX.variance.gradient[:] = 0.0
    prior.update_gradients_KL(qX)
    kl_mu, kl_S = np.array(qX.mean.gradient, dtype=np.float64), np.array(qX.variance.gradient, dtype=np.float64)
    Kx = kern.K(Z, Xnew)
    pmu = Kx.T.dot(post.woodbury_vector)
    pvar = kern.Kdiag(Xnew) - np.sum(Kx * np.asarray(post.woodbury_inv).dot(Kx), 0)
    return dict(mu=mu, S=S, Z=Z, Y=Y, Xnew=Xnew, variance=case["variance"], ls=np.array(case["ls"], dtype=np.float64),
                ard=int(case["ard"]), noise=case["noise"], lml=float(np.squeeze(lml)),
                bound=float(np.squeeze(lml)) - klv, grad=grad, dZ=dZ,
                dmu=np.asarray(dmu), dS=np.asarray(dS), kl_mu=kl_mu, kl_S=kl_S, pred_mu=pmu, pred_var=pvar[:, None],
                woodbury_vector=np.asarray(post.woodbury_vector), woodbury_inv=np.asarray(post.woodbury_inv))


def main():
    G, psi, V = reference()
    os.makedirs(OUT, exist_ok=True)
    for name, case in CASES.items():
        if len(sys.argv) > 1 and name not in sys.argv[1:]:
            continue
        r = evaluate(G, psi, V, case)
        np.savez(os.path.join(OUT, name + ".npz"), **r)
        print(name, r["Y"].shape, r["Z"].shape, r["lml"])
    if len(sys.argv) == 1 or "psi" in sys.argv[1:]:
        c = psi_case()
        qX = V.NormalPosterior(c["mu"], c["S"])
        out = {}
        for ard in (True, False):
            ls = c["ls"] if ard else c["ls"][:1]
            p0, p1, p2 = psi.psicomputations(c["variance"], ls, c["Z"], qX)
            dvar, dl, dZ, dmu, dS = psi.psiDerivativecomputations(c["dL0"], c["dL1"], c["dL2"], c["variance"], ls,
                                                                  c["Z"], qX)
            tag = "ard" if ard else "iso"
            out.update({"psi0_" + tag: p0, "psi1_" + tag: p1, "psi2_" + tag: p2,
                        "grad_" + tag: np.concatenate([[dvar], np.atleast_1d(dl)]), "dZ_" + tag: dZ,
                        "dmu_" + tag: dmu, "dS_" + tag: dS})
        np.savez(os.path.join(OUT, "psi.npz"), **{k: v for k, v in c.items()}, **out)
        print("psi")


if __name__ == "__main__":
    main()
