// gpx_psi.cuh — RBF psi-statistics on the device (internal; the public entries are gpx_psi_stats, gpx_psi_grads and
// gpx_sparse_eval_psi in include/gpx.h). Reference: GPy/kern/src/psi_comp/rbf_psi_comp.py:8-136.
#pragma once
#include "gpx_common.cuh"
#include "gpx_ctx.cuh"

namespace gpx {

constexpr int PSI_MAX_Q = 16;   // latent dimensions held in registers by the psi kernels

// one RBF part (isotropic or ARD) on the latent columns 0 .. Q-1 and the shapes of q(X) = N(mu, diag(S)) and Z
struct PsiParams {
  long N = 0, M = 0;
  int Q = 0, ard = 0;
  double variance = 0.0;
  double l[PSI_MAX_Q];    // lengthscale per latent dimension (isotropic: repeated)
};

// the lone RBF part on columns 0 .. Q-1 in order -> pp (-2 with a message otherwise)
int psi_params(const gpx_kern_part* parts, int nparts, int Q, PsiParams* pp);
// S (n x Q host) positive and finite (-2 otherwise)
int psi_check_S(const double* S, long n, int Q);

// Device inputs of one psi computation: mu, S (N x Q row-major), Z (M x Q row-major); pre: [N][2Q+2] per-point factors
// 1/(S + l^2), 1/(2S + l^2) and the two log-denominators, formed by psi_prep. Strided N x M matrices are addressed as
// (n, m) at n * sn + m * sm.
struct PsiDev {
  const double *mu = nullptr, *S = nullptr, *Z = nullptr;
  double* pre = nullptr;
};
int psi_prep(gpx_ctx* c, const PsiParams& pp, const PsiDev& d);                                      // 1 launch
int psi1_build(gpx_ctx* c, const PsiParams& pp, const PsiDev& d, double* psi1, long sn, long sm);    // 1 launch
// psi2 = sum_n psi2_n into out (Mpad x Mpad column-major, leading dimension ld, exactly symmetric, zero outside M x M)
int psi2_build(gpx_ctx* c, const PsiParams& pp, const PsiDev& d, double* out, long ld, long Mpad);   // 2 launches
// psiDerivativecomputations (rbf_psi_comp.py:53-136) for dL_dpsi1 (strided, beside psi1 with the same strides) and
// dL_dpsi2 (M x M column-major, leading dimension ld2, symmetrised here). Host outputs: grad = [variance, lengthscale
// (1 or Q)] WITHOUT the sum of dL_dpsi0, dZ (M x Q), dmu and dS (N x Q), row-major. 5 launches.
int psi_grads(gpx_ctx* c, const PsiParams& pp, const PsiDev& d, const double* psi1, const double* dL1, long sn, long sm,
              const double* dL2, long ld2, double* grad, double* dZ, double* dmu, double* dS);

}  // namespace gpx
