// gpx_ep.cuh — the expectation propagation kernels of gpx_laplace.cu that the sparse EP (gpx_epdtc_*, gpx_sparse.cu)
// shares with the dense one (internal).
#pragma once
#include "gpx_common.cuh"

namespace gpx {

// the site outputs of a sweep (N-vectors)
struct EpSites {
  double *tt, *vt;                      // tau~, v~ (in / out)
  double *ct, *cv, *zh, *mh, *s2;       // cavity tau and v, Z_hat, mu_hat, sigma2_hat
  const double* sgn;                    // +1 for y = 1, -1 for y in {0, -1}
  double eta, delta;
};

constexpr int EP_CHAIN_THREADS = 1024;
constexpr int EP_SOLVE_ROWS = 64;
constexpr int EP_CHAIN_SMEM = (TILE * TILE + 2 * TILE + 2) * 8;
constexpr int EP_SOLVE_SMEM = (TILE * TILE + 2 * TILE + TILE * EP_SOLVE_ROWS) * 8;

// dtc = 0: dense EP, G = Sigma[I, I] read from the stored lower tiles of Sig, mu_I = mu[I].
// dtc = 1: sparse EP, G dense in Sig (TILE x TILE, ld TILE), mu_I = mu[I] + muadd, and the cavity reads the diagonal the
// reference holds: max(G_jj, eps), or sd0[I[0]] for the first site when sd0 is given.
__global__ void ep_chain_kernel(const double* __restrict__ Sig, long ld, const int* __restrict__ I, int m,
                                const double* __restrict__ mu, EpSites e, double* __restrict__ Gout, double* __restrict__ cg,
                                const double* __restrict__ muadd, const double* __restrict__ sd0, int dtc);
// dtc = 0: S = Sigma[:, I] (I + U)^-1 over Npad rows; dtc = 1: Y = P (I + U)^-1 over Mpad rows with P^T in Sig
// (TILE x ld, ld TILE). Rows r < ld; out Sx, Sc (ld x TILE) and mu[r] -= sum_j x_j g_j.
__global__ void ep_solve_kernel(const double* __restrict__ Sig, long ld, const int* __restrict__ I, int m,
                                const double* __restrict__ Gin, const double* __restrict__ cg, double* __restrict__ Sx,
                                double* __restrict__ Sc, double* __restrict__ mu, int dtc);
// parallel_updates=True: every site from the same diag(Sigma) and mu
__global__ void ep_parallel_kernel(long N, const double* __restrict__ sd, const double* __restrict__ mu, EpSites e);

enum { EV_SUB = 0, EV_DIAG = 1, EV_DLDK = 2, EV_ADDDIAG = 3, EV_SIGN = 4 };
__global__ void ep_vec_kernel(int mode, long N, long n, const double* __restrict__ x, const double* __restrict__ y,
                              double* __restrict__ A, long ld, double add, double* __restrict__ o);

}  // namespace gpx
