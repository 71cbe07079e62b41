// gpx_kernels.cuh — launch wrappers of the non-GEMM kernels (internal).
#pragma once
#include "gpx_common.cuh"

namespace gpx {

struct KBuildParams {
  const double* rowsT; long ld_rows;   // thread-mapped operand, SoA [D][ld_rows]
  const double* colsT; long ld_cols;   // walked operand
  const double* sq_rows; const double* sq_cols;
  double* out; long ld;                // out[rowidx + colidx*ld]
  long nrows, ncols;                   // logical extents (beyond: padding)
  int sym;                             // 1: factor workspace mode (lower tiles, zero upper tiles, identity padding, +diag_add)
  int same;                            // 1: both operands are the same point set -> exact zero distance on the diagonal
  double diag_add;                     // noise + jitter (sym mode)
  const double* diag_vec;              // optional per-point noise variances added on the diagonal as well (sym mode)
  int own_G, own_g, own_blk;           // multi-GPU: only row tiles with ((rt / own_blk) % own_G) == own_g (0 = all)
  int loc_rows;                        // multi-GPU: `out` holds only the owned block rows (row tile rt at loc_tile(rt, ..))
  int rt0;                             // first row tile of this launch (the grid's y index counts from here)
  KernParams kp;
};

struct FinalizeParams {
  const double* partials; long ntiles; int nl;
  const double* logdet_part; long nt;
  const double* T; long ld; long N; int P;
  KernParams kp;
  double* res;
};

struct GradFullParams {
  const double* x1T; long ld1; const double* sq1; long N;   // X  (index i, rows of dL_dK)
  const double* x2T; long ld2; const double* sq2; long M;   // X2 (index j, contiguous in dL_dK)
  const double* dL_dK;                                       // N x M row-major (row stride ldd, 0 -> M)
  long ldd;
  int transposed;                                            // gradx only: element (n, m) is read at dL_dK[m*ldd + n]
  // optional rank-P correction added on the fly: dL(i, j) += sum_p ci[p*ldci + i] * cj[p*ldcj + j]
  const double* ci; long ldci; const double* cj; long ldcj; int cP;
  int same;
  double* partials;
  KernParams kp;
};

int launch_prep_x(const double* X, long N, long ldx, const KernParams& kp, double* XsT, double* sq, cudaStream_t st);
int launch_kbuild(const KBuildParams& p, int row_tiles, int col_tiles, cudaStream_t st);
int launch_base(double* S, long ld, double* Ldiag, double* Dinv, double* logdet_part, int* info, int gcol0,
                cudaStream_t st);
int launch_assemble(const double* Sblk, long ld, int nb, double* Prows, long ldp, double* Tm, cudaStream_t st);
int launch_fw_block(const double* Tm, int nb, const double* yres, long ld, int P, double* t, cudaStream_t st);
int launch_fw_panel(const double* Pb, long ldp, long rows, int nb, const double* t, long ld, int P, double* yres,
                    cudaStream_t st);
int launch_utv(const double* U, long ld, long n, int P, const double* Y, double* T, cudaStream_t st, int own_G = 0,
               int own_g = 0, long own_cols = 1, int local_cols = 0);
int launch_uv(const double* U, long ld, long n, int P, const double* T, int ksplit, double* part, double* out,
              cudaStream_t st);
int launch_finalize(const FinalizeParams& f, cudaStream_t st);
int launch_finalize_raw(const FinalizeParams& f, cudaStream_t st);
int launch_uv_blk(const double* U, long ld, long n, int P, const double* T, long blk, int G, int g, double* part,
                  double* out, cudaStream_t st, int local_cols = 0);
int launch_copyback(double* SL, long ldl, double* SU, long ldu, const double* Pbuf, long NB, int G, int g, long npr, int k,
                    int nt, cudaStream_t st);
int launch_extract_L_rows(const double* SL, long ldl, long lrow0, const double* Ldiag, long grow0, long NB, long ncols,
                          double* out, cudaStream_t st);
int launch_extract(int which, const double* S, long ld, const double* Ldiag, const double* Kinv, const double* alpha,
                   int P, long N, double* out, cudaStream_t st);
int launch_transpose_pad(const double* in, long n, int p, long ld, double* out, cudaStream_t st);
int launch_untranspose(const double* in, long n, int p, long ld, double* out, cudaStream_t st);
int launch_gradx(const GradFullParams& p, int nchunk, long mchunk, double* part, double* out, cudaStream_t st);
int launch_col_dot(const double* A, long ld, long rows, long cols, int P, const double* Y, long ldy, double* out, long ldo,
                   cudaStream_t st);
int launch_col_sqnorm(const double* A, long ld, long rows, long cols, double* out, cudaStream_t st);
int launch_row_dot(const double* A, long lda, long rows_pad, long ncols, int P, const double* Y, long ldy, int nsplit,
                   double* part, double* out, cudaStream_t st);
int launch_load_sym(const double* A, long lda, long N, double* S, long ld, double jitter, cudaStream_t st);
int measure_dmma_peak(cudaStream_t st, double* tflops);
int launch_grad_full(const GradFullParams& p, int tiles_j, int tiles_i, cudaStream_t st);

// gradient reductions from a stored K^-1 (lower 128 x 128 tiles, column-major, leading dimension ld): same partial sums as
// the fused epilogue of gemm_lauum_kernel, consumed by finalize_kernel
struct GradKinvParams {
  const double* Kinv; long ld;
  const double* XsT; const double* sq; const double* alpha; long ldx;
  long N; int P; int nt;
  double* partials;        // [nt*nt*csplit][nl+2], zeroed by the caller
  int csplit;              // CTAs per tile (each takes 64/csplit columns of both column halves): 1, 2, 4 or 8 -- small matrices
                           // have too few tiles to fill the machine, and a thread's 64 columns are a serial chain
  double* dnoise_out;      // optional diag(dL_dK)
  KernParams kp;
};
int launch_grad_kinv(const GradKinvParams& p, cudaStream_t st);
int grad_kinv_csplit(int nt, int nred);   // the split launch_grad_kinv expects for this matrix (partials: nt*nt*(MAX_D+2) doubles)

}  // namespace gpx
