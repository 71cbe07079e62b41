// gpx_multi.cuh — composite kernels on the device (internal): K = sum over terms of products of parts, each part a
// stationary kernel (RBF .. Matern52, RatQuad) or a StdPeriodic kernel on its own active dims, a White or a Bias kernel.
// Mirrors GPy/kern/src/add.py:60-99 (Add.K / update_gradients_full), prod.py:59-68,377-396 (Prod.K; each factor's gradient
// sees dL_dK times the other factors), static.py:63-185 (White, Bias), stationary.py:747-802 (RatQuad) and
// standard_periodic.py:56-94,125-139,501-548 (StdPeriodic).
#pragma once
#include "gpx_common.cuh"

namespace gpx {

constexpr int MAX_PARTS = 8;
// largest result vector of an evaluation: 4 scalars, then every part's gradient block (at most 2 + 2 D entries per part)
constexpr int RES_DOUBLES = 4 + 2 * MAX_D + 2 * MAX_PARTS;

struct PartDev {
  int kind;          // GPX_RBF .. GPX_MATERN52, GPX_WHITE, GPX_BIAS, GPX_RATQUAD, GPX_STDPERIODIC
  int ard;           // lengthscale per dim (StdPeriodic: GPy's ARD2)
  int ard_period;    // StdPeriodic: period per dim (GPy's ARD1)
  int term;          // parts with equal `term` are multiplied, terms are summed (parts sorted by term)
  int D;             // active dims (0 for the static kinds)
  int xoff;          // first row of this part inside the stacked input SoA [sumD][ld]
  double variance;
  double inv_ls_iso;
  double power;      // RatQuad
};

struct MultiKern {
  int nparts;
  int sumD;
  PartDev part[MAX_PARTS];
  int dims[MAX_D];       // column of X behind stacked row (xoff + q)
  double ls[MAX_D];      // its lengthscale (ARD: per dim; iso: the part's single lengthscale repeated)
  double period[MAX_D];  // StdPeriodic: its period (ARD1: per dim; iso: repeated)
};

__host__ __device__ __forceinline__ bool is_static(int kind) { return kind == GPX_WHITE || kind == GPX_BIAS; }
__host__ __device__ __forceinline__ bool is_known(int kind) { return kind >= GPX_RBF && kind <= GPX_STDPERIODIC; }
// a function of the scaled distance r (stationary.py:23-243): RBF .. Matern52 and RatQuad
__host__ __device__ __forceinline__ bool is_stationary(int kind) { return (kind >= GPX_RBF && kind <= GPX_MATERN52) || kind == GPX_RATQUAD; }

// gradient entries of a part (its block of the result vector)
__host__ __device__ inline int part_ngrad(const PartDev& pd) {
  const int nl = pd.ard ? pd.D : 1;
  switch (pd.kind) {
    case GPX_WHITE: case GPX_BIAS: return 1;
    case GPX_RATQUAD: return 2 + nl;                                   // variance, lengthscale(s), power
    case GPX_STDPERIODIC: return 1 + (pd.ard_period ? pd.D : 1) + nl;  // variance, period(s), lengthscale(s)
    default: return 1 + nl;
  }
}
// per-tile partial sums of a part's reduction pass: its gradient entries and tr(dL_dK) (static kinds keep one unused slot)
__host__ __device__ inline int part_nred(const PartDev& pd) { return is_static(pd.kind) ? 3 : part_ngrad(pd) + 1; }
// per-dimension register accumulators of the reduction pass: ARD lengthscales of a stationary part, period and lengthscale
// of every dim of a StdPeriodic part. Must not exceed MAX_D.
__host__ __device__ inline int part_nacc(const PartDev& pd) {
  if (pd.kind == GPX_STDPERIODIC) return 2 * pd.D;
  return (is_stationary(pd.kind) && pd.ard) ? pd.D : 0;
}

struct KBuildMultiParams {
  const double* rowsT; long ld_rows; const double* sq_rows;    // stacked SoA [sumD][ld] and [nparts][ld] of the ROW points
  const double* colsT; long ld_cols; const double* sq_cols;
  double* out; long ld;                                        // out[rowidx + colidx * ld]
  long nrows, ncols;
  int sym, same;                                               // as KBuildParams
  double diag_add;
  MultiKern mk;
};

struct GradKinvMultiParams {
  const double* Kinv; long ld;
  const double* XsT; const double* sq; long ldx;               // stacked SoA of the training points
  const double* alpha;
  long N; int P; int nt;
  int part;                                                    // the part whose parameter sums are reduced by this launch
  int want_noise;                                              // also reduce tr(dL_dK) (done by the first launch only)
  double* partials;                                            // [nt*nt][part_nred] of THIS part, zeroed by the caller
  MultiKern mk;
};

// update_gradients_full of one part of mk for a dense dL_dK: rows = thread-mapped points (X2 of the call), cols = the X
// points; dL_dK element (col point i, row point j) at dL[i * ldd + j]
struct GradFullMultiParams {
  const double* rowsT; long ld_rows; const double* sq_rows;
  const double* colsT; long ld_cols; const double* sq_cols;
  long nrows, ncols;
  int same;
  int part;                                                    // the part whose parameter sums this launch reduces
  const double* dL; long ldd;
  double* partials;                                            // [col tiles][row tiles][part_nred]
  MultiKern mk;
};

// gradients_X of the composite (add.py:88-100, prod.py:397-407) w.r.t. the row points, over its stationary parts (kinds
// RBF .. Matern52; White / Bias enter as factors only): element (row n, col m) of dL_dK at dL[n * ldd + m], or at
// dL[m * ldd + n] when `transposed`. same: the columns are the rows (dL + dL^T, stationary.py:334-336). Output: nrows x Dfull row-major, the parts' sums added per data column in
// part order.
struct GradXMultiParams {
  const double* rowsT; long ld_rows; const double* sq_rows; long nrows;
  const double* colsT; long ld_cols; const double* sq_cols; long ncols;
  const double* dL; long ldd; int transposed; int same;
  int Dfull;
  MultiKern mk;
};

// gradients_X of the exact evaluation's kernel at its N training points with dL_dK = 1/2 (alpha alpha^T - P K^-1) from the
// stored K^-1 (GPy/models/gplvm.py:47-49): the rules of GradXMultiParams with X2 = None
struct ExactGradXParams {
  const double* Kinv; long ld;                                 // lower tiles of K^-1 (diagonal tiles whole), column-major
  const double* alpha; int P;                                  // [P][ldx]
  const double* XsT; const double* sq; long ldx; long N;       // the training points as the evaluation prepared them
  int Dfull;
  MultiKern mk;
};

// predictive gradients (GPy/core/gp.py:438-474) at the row points (the test points) against the column points (training
// or inducing points), with gradx_multi_kernel's rules: channel c < P weights a pair by alpha[c * lda + n] (the mean
// Jacobian of output c), channel P by V[m * ldv + n] with V = W K(X, X*) (the variance Jacobian's Schur term).
struct PredGradParams {
  const double* rowsT; long ld_rows; const double* sq_rows; long nrows;
  const double* colsT; long ld_cols; const double* sq_cols; long ncols;
  const double* alpha; long lda; int P;
  const double* V; long ldv;
  int Dfull;
  MultiKern mk;
};

struct FinalizeMultiParams {
  const double* partials[MAX_PARTS]; long ntiles;
  const double* logdet_part; long nt;
  const double* T; long ld; long N; int P;
  MultiKern mk;
  double* res;   // [0] lml, [1] logdet, [2] quad, [3] d/d noise, then every part's gradient block (part_ngrad entries)
};

int launch_prep_multi(const double* X, long N, int Dfull, long ld, const MultiKern& mk, double* XsT, double* sq, cudaStream_t st);
int launch_kbuild_multi(const KBuildMultiParams& p, int row_tiles, int col_tiles, cudaStream_t st);
int launch_grad_kinv_multi(const GradKinvMultiParams& p, cudaStream_t st);
int launch_grad_full_multi(const GradFullMultiParams& p, int row_tiles, int col_tiles, cudaStream_t st);
// two launches: chunk partials [nchunk][nrows][sumD] into part, then their fixed-order sum into out (device, nrows x Dfull)
int launch_gradx_multi(const GradXMultiParams& p, int nchunk, long mchunk, double* part, double* out, cudaStream_t st);
// the same two launches for ExactGradXParams: partials [nchunk][N][sumD], then out (device, N x Dfull)
int launch_exact_gradx(const ExactGradXParams& p, int nchunk, long mchunk, double* part, double* out, cudaStream_t st);
int launch_finalize_multi(const FinalizeMultiParams& f, cudaStream_t st);
// one reduction launch per group of channels (as many channels per group as the accumulators allow), partials
// [P + 1][nchunk][nrows][sumD] into part, then their fixed-order sum into out (device): dmu (nrows x Dfull x P row-major),
// followed by dvar (nrows x Dfull). RatQuad / StdPeriodic parts: -2.
int launch_pred_grad(const PredGradParams& p, int nchunk, long mchunk, double* part, double* out, cudaStream_t st);
int pred_grad_launches(const MultiKern& mk, int P);   // kernels launch_pred_grad issues
// entry t of part p's reduced sums -> entry t of its gradient block: the stationary lengthscale rule -tot/l
// (stationary.py:210,213) for RBF .. Matern52 and RatQuad; RatQuad's power and StdPeriodic's sums are the gradient as they
// are (stationary.py:797-798, standard_periodic.py:518-526). false: the trace slot (last) or a static part's unused slot.
__host__ __device__ inline bool part_grad_entry(const MultiKern& mk, int p, int t, double tot, double* val) {
  const PartDev& pd = mk.part[p];
  if (t >= part_ngrad(pd)) return false;
  const int nl = pd.ard ? pd.D : 1;
  *val = (t >= 1 && t <= nl && is_stationary(pd.kind)) ? -tot / mk.ls[pd.xoff + (pd.ard ? t - 1 : 0)] : tot;
  return true;
}

}  // namespace gpx
