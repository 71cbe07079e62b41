// gpx_fine.cuh — fine-grained fp64 DMMA kernels of the SERIAL CHAIN of the sweep (internal).
//
// The diagonal-block chain D(k) -> panel rows of the next block -> update of the next diagonal block -> D(k+1) is latency,
// not throughput: with 128 x 128 CTA tiles a 128-deep product keeps 3..35 SMs busy for ~22 us each (one SM's DMMA rate on a
// 128^3 tile). The kernels here cut the same products into 64 x 32 output tiles (16-row strips for the in-place inner
// panel), so that a chain link spreads over up to 132 SMs and lasts a few microseconds. Same arithmetic, same operand
// layout (column-major, m-contiguous), same results up to the summation order inside DMMA.
#pragma once
#include "gpx_common.cuh"

struct gpx_ctx;

namespace gpx {

enum FineMode { FINE_UPDATE = 0, FINE_PANEL = 1, FINE_LAUUM = 2 };

struct FineParams {
  int mode;
  const double* A; long lda;   // element (m, k) of row tile r:    A[r*TILE + m + k*lda]
  const double* B; long ldb;   // element (n, k) of column tile c: B[c*TILE + n + k*ldb]
  double* C; long ldc;         // tile (r, c) at C[r*TILE + c*TILE*ldc]
  int K;                       // k-depth (multiple of 128)
  // FINE_UPDATE: C(r,c) -= A_r B_c^T for columns c in [c0, c0+ncols), rows r in [0, rlow) U [c, nt); the upper-right 64 x 64
  // quarter of a diagonal tile (r == c) is skipped (nothing reads it before the base kernel overwrites it with U)
  int nt, c0, ncols, rlow;
  // FINE_PANEL: C(r,c) = A_r B_c^T for row tiles r in [r0, r0+nr), column tiles c in [0, nc); tri: B is lower triangular
  // (k range of output columns [32h, 32h+32) of tile c ends at c*TILE + 32(h+1))
  int r0, nr, nc, tri;
  int pdl;                     // 1: launch as a programmatic dependent of the kernel before it in the stream (inner update of a
                               // diagonal block behind the in-place inner panel); 0: ordinary launch
  // FINE_LAUUM: C(r,c) = sum_{k >= r*TILE} A_r(:,k) B_c(:,k)^T for the lower tiles c <= r < nt (K^-1 = U U^T of a small matrix:
  // U is upper triangular, row tile r starts at column r*TILE); K = padded order
};

int fine_init();
int launch_fine(const FineParams& p, cudaStream_t st);
// in-place inner panel of a diagonal block at inner step d: S(r, tile column d) <- S(r, tile column d) * Dinv^T for every
// 128-row tile r != d of the nbt-tile block (Dinv = L_dd^-1, 128 x 128 lower triangular, column-major, ld = TILE)
int launch_fine_panel_inplace(double* Sblk, long ld, const double* Dinv, int nbt, int d, cudaStream_t st);
// the whole inner sweep of an (nbt*TILE)^2 diagonal block whose first tile is global tile g0: base block, in-place inner
// panel, inner update per 128 columns (what run_sweep / dist_exact_eval call D(k)); returns the number of launches
int diag_block_sweep(gpx_ctx* c, double* Sblk, long ld, int nbt, int g0, cudaStream_t st);

}  // namespace gpx
