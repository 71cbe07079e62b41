// gpx_sparse.cu — sparse GP regression (VarDTC) as one device evaluation.
//
// Reference: GPy/inference/latent_function_inference/var_dtc.py:66-215 with the gradient wiring of
// GPy/core/sparse_gp.py:108-119 (Gaussian likelihood, homoscedastic noise, certain inputs). Everything stays in HBM:
//   psi1 = K(X, Z) in both layouts (8 N M bytes each)                                         var_dtc.py:126
//   Kmm + jitter -> Lm, Lm^-1 (factor-and-invert sweep)                                        :93-95
//   tmp = Lm^-1 psi1^T (M x N, triangular product), A = beta tmp tmp^T, t = tmp Y              :130-132,139
//   B = I + A -> LB, LB^-1; v, C, DBi, dL_dKmm, dL_dpsi2 as M x M DMMA GEMMs                   :135-156,217-233
//   dL_dKnm^T = W2 psi1^T + C (beta Y)^T (M x N, never materialised on the host) reduced straight to
//   d/d(variance, lengthscale) and dL/dZ                                                       sparse_gp.py:112,118
// With a communicator the data rows are sharded: A, t and the Knm gradient pieces are all-reduced (var_dtc_parallel.py).
// Heteroscedastic noise (one variance per data point, the `het_noise` branches var_dtc.py:127-128,221-227,241-257,267-269):
// the same evaluation with the columns of tmp scaled by sqrt(beta_n), dL_dKnm^T's columns by beta_n, and the N per-point
// noise gradients dL_dR from three column reductions over M x N matrices (gpx_sparse_eval_het).
#include <algorithm>
#include <cstring>
#include <vector>

#include "gpx_common.cuh"
#include "gpx_ctx.cuh"
#include "gpx_kernels.cuh"

using namespace gpx;

static int knm_grads_device(gpx_ctx* c, double beta, const double* bvec, double* dvariance, double* dlengthscale,
                            double* dZ);

#define GPX_CHECK(x)            \
  do {                          \
    int rc__ = (x);             \
    if (rc__ != 0) return rc__; \
  } while (0)
#define GPX_FAIL(msg)       \
  do {                      \
    gpx::set_error(msg);    \
    return -2;              \
  } while (0)

struct SparseState {
  long N = 0, Npad = 0, M = 0, Mpad = 0;   // N: rows held by THIS rank (all of them on one GPU)
  long Ntot = 0;                           // rows over all ranks (var_dtc.py num_data)
  long Nw = 0, Mw = 0;                     // extents of psi1 written last time (a smaller N or M must re-zero the padding)
  int D = 0, P = 0;
  double *X = nullptr, *XsT = nullptr, *sqX = nullptr, *Y = nullptr, *Yb = nullptr;   // Y: [P][Npad]
  double *Z = nullptr, *ZsT = nullptr, *sqZ = nullptr;
  double *Kuf = nullptr;   // Mpad x Npad column-major: (a, n) at a + n*Mpad
  double *Kfu = nullptr;   // Npad x Mpad column-major: (n, a) at n + a*Npad
  double *dLt = nullptr;   // Mpad x Npad: dL_dKnm^T
  double *Gm = nullptr, *W2 = nullptr, *Cm = nullptr;   // Mpad x Mpad, Mpad x Mpad, [P][Mpad]
  double *part = nullptr; size_t part_cap = 0;
  KernParams kp{};
  // full-device evaluation (gpx_sparse_eval)
  gpx_ctx *cK = nullptr, *cB = nullptr;             // child contexts holding the factors of Kmm and of B = I + A
  double *mm[10] = {nullptr};                        // Mpad x Mpad work matrices
  double *vec = nullptr;                             // [8][P][Mpad] small vectors
  double *red = nullptr; double *h_red = nullptr;    // scalar reductions
  double *gsum = nullptr;                            // [1 + nl + M*D] gradient pieces summed over ranks
  double *hb = nullptr;                              // het noise: [2][Npad] sqrt(beta_n), beta_n
  double *hs = nullptr;                              // het noise: [2 + P][Npad] column reductions s1, s2, r (see eval)
  double trYYT = 0.0;
  bool have_eval = false;
  double noise = 0.0;
};

namespace {
void free_m(SparseState* s) {
  double** ptrs[] = {&s->Z, &s->ZsT, &s->sqZ, &s->Kuf, &s->Kfu, &s->dLt, &s->Gm, &s->W2, &s->Cm, &s->vec, &s->gsum};
  for (auto p : ptrs) { if (*p) cudaFree(*p); *p = nullptr; }
  for (auto& p : s->mm) { if (p) cudaFree(p); p = nullptr; }
  s->have_eval = false;
  s->M = s->Mpad = 0;
  s->Nw = s->Mw = 0;
}
void free_all(SparseState* s) {
  free_m(s);
  double** ptrs[] = {&s->X, &s->XsT, &s->sqX, &s->Y, &s->Yb, &s->part, &s->red, &s->hb, &s->hs};
  for (auto p : ptrs) { if (*p) cudaFree(*p); *p = nullptr; }
  if (s->h_red) { cudaFreeHost(s->h_red); s->h_red = nullptr; }
  if (s->cK) { gpx_destroy(s->cK); s->cK = nullptr; }
  if (s->cB) { gpx_destroy(s->cB); s->cB = nullptr; }
  s->part_cap = 0;
  s->N = s->Npad = 0;
}
int ensure_part(SparseState* s, size_t bytes) {
  if (s->part_cap >= bytes) return 0;
  if (s->part) cudaFree(s->part);
  s->part = nullptr;
  GPX_CUDA(cudaMalloc(&s->part, bytes));
  s->part_cap = bytes;
  return 0;
}
__global__ void scale_kernel(const double* __restrict__ in, double a, long n, double* __restrict__ out) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = a * in[i];
}
// het noise: column n of a column-major matrix (leading dimension ld, `cols` columns) times f[n]
// (var_dtc.py:127 psi1 * sqrt(precision) carried through Lm^-1; :226 (psi1 * beta))
__global__ void scale_cols_kernel(double* __restrict__ A, long ld, long cols, const double* __restrict__ f) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ld * cols) return;
  A[i] *= f[i / ld];
}
// het noise: out[q][n] = f[n] * Y[q][n]  ([P][ld] layouts)
__global__ void ymul_kernel(const double* __restrict__ Y, const double* __restrict__ f, long ld, int P,
                            double* __restrict__ out) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ld * P) return;
  out[i] = f[i % ld] * Y[i];
}
// out = a X + b Y + cdiag I + d sum_p u_p u_p^T   (n x n, leading dimension ld; X, Y, U may be null)
__global__ void combine_kernel(double* __restrict__ out, long ld, long n, double a, const double* __restrict__ X, double b,
                               const double* __restrict__ Y, double cdiag, double d, const double* __restrict__ U, long ldu,
                               int P) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y;
  if (i >= n) return;
  double v = 0.0;
  if (X) v += a * X[i + j * ld];
  if (Y) v += b * Y[i + j * ld];
  if (i == j) v += cdiag;
  if (U)
    for (int q = 0; q < P; q++) v = fma(d * U[(long)q * ldu + i], U[(long)q * ldu + j], v);
  out[i + j * ld] = v;
}
// lower tiles of a symmetric matrix were computed: mirror them into the upper tiles
__global__ void mirror_tiles_kernel(double* __restrict__ A, long ld, long n) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y;
  if (i >= n || i / TILE >= j / TILE) return;
  A[i + j * ld] = A[j + i * ld];
}
// r[0] = trace(A), r[1] = sum(A .* B) over n x n; single CTA partial sums reduced in fixed order
__global__ void __launch_bounds__(256) trace_dot_kernel(const double* __restrict__ A, const double* __restrict__ B, long ld,
                                                         long n, double* __restrict__ r) {
  __shared__ double sh[2][256];
  double tr = 0.0, dt = 0.0;
  for (long j = blockIdx.x; j < n; j += gridDim.x)
    for (long i = threadIdx.x; i < n; i += 256) {
      const double a = A[i + j * ld];
      dt = fma(a, B[i + j * ld], dt);
      if (i == j) tr += a;
    }
  sh[0][threadIdx.x] = tr; sh[1][threadIdx.x] = dt;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) { sh[0][threadIdx.x] += sh[0][threadIdx.x + o]; sh[1][threadIdx.x] += sh[1][threadIdx.x + o]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) { r[2 * blockIdx.x] = sh[0][0]; r[2 * blockIdx.x + 1] = sh[1][0]; }
}
}  // namespace

namespace gpx {
void sparse_free(gpx_ctx* c) {
  if (!c->sparse) return;
  free_all(c->sparse);
  delete c->sparse;
  c->sparse = nullptr;
}
}  // namespace gpx

extern "C" {

int gpx_sparse_set_data(gpx_ctx* c, const double* X, int64_t N, int D, const double* Y, int P) {
  if (!c || !X || !Y) GPX_FAIL("null argument");
  if (N < 1 || D < 1 || D > MAX_D || P < 1 || P > MAX_P) GPX_FAIL("bad shape (D <= 64, P <= 8)");
  GPX_CUDA(cudaSetDevice(c->device));
  if (!c->sparse) c->sparse = new SparseState();
  SparseState* s = c->sparse;
  const long Npad = (N + TILE - 1) / TILE * TILE;
  if (Npad != s->Npad || D != s->D || P != s->P) {
    GPX_CUDA(cudaStreamSynchronize(c->st));
    free_all(s);
    s->Npad = Npad; s->D = D; s->P = P;
    GPX_CUDA(cudaMalloc(&s->X, (size_t)Npad * D * 8));
    GPX_CUDA(cudaMalloc(&s->XsT, (size_t)Npad * D * 8));
    GPX_CUDA(cudaMalloc(&s->sqX, (size_t)Npad * 8));
    GPX_CUDA(cudaMalloc(&s->Y, (size_t)Npad * P * 8));
    GPX_CUDA(cudaMalloc(&s->Yb, (size_t)Npad * P * 8));
  }
  s->N = N;
  s->have_eval = false;
  {   // trYYT = sum(Y .* Y) (var_dtc.py:37,90); with row shards: summed over the ranks, like num_data
    double t = 0.0;
    for (int64_t i = 0; i < N * (int64_t)P; i++) t += Y[i] * Y[i];
    s->trYYT = t;
    s->Ntot = N;
    int rank = 0, G = 1;
    dist_world(c, &rank, &G);
    if (G > 1) {
      if (!s->red) {
        GPX_CUDA(cudaMalloc(&s->red, 4096 * 8));
        GPX_CUDA(cudaMallocHost(&s->h_red, 4096 * 8));
      }
      s->h_red[0] = (double)N; s->h_red[1] = t;
      GPX_CUDA(cudaMemcpyAsync(s->red, s->h_red, 16, cudaMemcpyHostToDevice, c->st));
      GPX_CHECK(dist_allreduce_sum(c, s->red, 2, c->st));
      GPX_CUDA(cudaMemcpyAsync(s->h_red, s->red, 16, cudaMemcpyDeviceToHost, c->st));
      GPX_CUDA(cudaStreamSynchronize(c->st));
      s->Ntot = (long)llround(s->h_red[0]);
      s->trYYT = s->h_red[1];
    }
  }
  GPX_CUDA(cudaMemcpyAsync(s->X, X, (size_t)N * D * 8, cudaMemcpyHostToDevice, c->st));
  GPX_CUDA(cudaMemcpyAsync(s->Yb, Y, (size_t)N * P * 8, cudaMemcpyHostToDevice, c->st));
  GPX_CHECK(launch_transpose_pad(s->Yb, N, P, Npad, s->Y, c->st));
  c->total_launches++;
  GPX_CUDA(cudaStreamSynchronize(c->st));
  return 0;
}

}  // extern "C"

// psi1 = K(X, Z) in both layouts (Kuf: M x N, Kfu: N x M), left on the device
static int psi_device(gpx_ctx* c, int kind, int ard, double variance, const double* lengthscale, const double* Z,
                      int64_t M) {
  SparseState* s = c->sparse;
  cudaStream_t st = c->st;
  GPX_CHECK(fill_kp(s->kp, kind, ard, s->D, variance, lengthscale));
  const long Mpad = (M + TILE - 1) / TILE * TILE, Npad = s->Npad, N = s->N;
  if (Mpad != s->Mpad) {
    GPX_CUDA(cudaStreamSynchronize(st));
    free_m(s);
    s->Mpad = Mpad;
    GPX_CUDA(cudaMalloc(&s->Z, (size_t)Mpad * s->D * 8));
    GPX_CUDA(cudaMalloc(&s->ZsT, (size_t)Mpad * s->D * 8));
    GPX_CUDA(cudaMalloc(&s->sqZ, (size_t)Mpad * 8));
    GPX_CUDA(cudaMalloc(&s->Kuf, (size_t)Mpad * Npad * 8));
    GPX_CUDA(cudaMalloc(&s->Kfu, (size_t)Mpad * Npad * 8));
    GPX_CUDA(cudaMalloc(&s->dLt, (size_t)Mpad * Npad * 8));
    GPX_CUDA(cudaMalloc(&s->Gm, (size_t)Mpad * Mpad * 8));
    GPX_CUDA(cudaMalloc(&s->W2, (size_t)Mpad * Mpad * 8));
    GPX_CUDA(cudaMalloc(&s->Cm, (size_t)Mpad * s->P * 8));
    GPX_CUDA(cudaMalloc(&s->gsum, (size_t)(MAX_D + 2 + Mpad * s->D) * 8));
    GPX_CUDA(cudaMemsetAsync(s->Gm, 0, (size_t)Mpad * Mpad * 8, st));
    GPX_CUDA(cudaMemsetAsync(s->Kuf, 0, (size_t)Mpad * Npad * 8, st));   // padding stays zero: only valid entries
    GPX_CUDA(cudaMemsetAsync(s->Kfu, 0, (size_t)Mpad * Npad * 8, st));   // are ever written
  }
  s->M = M;
  if (N < s->Nw || M < s->Mw) {   // fewer points than last time inside the same padded extents: stale entries must go
    GPX_CUDA(cudaMemsetAsync(s->Kuf, 0, (size_t)Mpad * Npad * 8, st));
    GPX_CUDA(cudaMemsetAsync(s->Kfu, 0, (size_t)Mpad * Npad * 8, st));
  }
  s->Nw = N; s->Mw = M;
  GPX_CUDA(cudaMemcpyAsync(s->Z, Z, (size_t)M * s->D * 8, cudaMemcpyHostToDevice, st));
  GPX_CHECK(launch_prep_x(s->X, N, Npad, s->kp, s->XsT, s->sqX, st));
  GPX_CHECK(launch_prep_x(s->Z, M, Mpad, s->kp, s->ZsT, s->sqZ, st));
  const int mt = (int)(Mpad / TILE), ntl = (int)(Npad / TILE);
  KBuildParams kb;
  memset(&kb, 0, sizeof(kb));
  kb.kp = s->kp; kb.sym = 0; kb.same = 0;
  // psi1^T: thread-mapped operand = inducing points
  kb.rowsT = s->ZsT; kb.ld_rows = Mpad; kb.sq_rows = s->sqZ; kb.colsT = s->XsT; kb.ld_cols = Npad; kb.sq_cols = s->sqX;
  kb.out = s->Kuf; kb.ld = Mpad; kb.nrows = M; kb.ncols = N;
  GPX_CHECK(launch_kbuild(kb, mt, ntl, st));
  // psi1: thread-mapped operand = data points
  kb.rowsT = s->XsT; kb.ld_rows = Npad; kb.sq_rows = s->sqX; kb.colsT = s->ZsT; kb.ld_cols = Mpad; kb.sq_cols = s->sqZ;
  kb.out = s->Kfu; kb.ld = Npad; kb.nrows = N; kb.ncols = M;
  GPX_CHECK(launch_kbuild(kb, ntl, mt, st));
  c->total_launches += 4;
  return 0;
}

// dL_dKnm^T = W2 psi1^T (+ rank-P term on the fly) reduced to kernel-parameter gradients and dL/dZ; W2 (device, s->W2)
// and C (device, s->Cm as [P][Mpad]) must be in place. Results on the host.
// bvec (device, [Npad], per-point precisions) selects the heteroscedastic form: VVT_factor = beta_n Y_n and the columns of
// W2 psi1^T scaled by beta_n (var_dtc.py:226); W2 is then 2 dL_dpsi2_beta without the scalar beta.
static int knm_grads_device(gpx_ctx* c, double beta, const double* bvec, double* dvariance, double* dlengthscale,
                            double* dZ) {
  SparseState* s = c->sparse;
  cudaStream_t st = c->st;
  const long M = s->M, Mpad = s->Mpad, N = s->N, Npad = s->Npad;
  const int D = s->D, P = s->P;
  const int mt = (int)(Mpad / TILE), ntl = (int)(Npad / TILE);
  if (bvec)
    ymul_kernel<<<(unsigned)((Npad * P + 255) / 256), 256, 0, st>>>(s->Y, bvec, Npad, P, s->Yb);
  else
    scale_kernel<<<(unsigned)((Npad * P + 255) / 256), 256, 0, st>>>(s->Y, beta, Npad * P, s->Yb);
  GPX_CUDA(cudaGetLastError());
  // dLt = W2 * psi1^T  (M x N), W2 symmetric
  {
    GemmParams pg = gemm_defaults();
    pg.mode = GEMM_PANEL; pg.plain = 1;
    pg.A = s->W2; pg.lda = Mpad; pg.B = s->Kfu; pg.ldb = Npad; pg.C = s->dLt; pg.ldc = Mpad;
    pg.K = (int)Mpad; pg.nt = mt; pg.ncols = ntl;
    GPX_CHECK(launch_gemm(pg, dim3(1, 1), st));
  }
  if (bvec) {
    scale_cols_kernel<<<(unsigned)((Mpad * N + 255) / 256), 256, 0, st>>>(s->dLt, Mpad, N, bvec);
    GPX_CUDA(cudaGetLastError());
    c->total_launches++;
  }
  // kernel-parameter gradients of sum(dL_dKnm * K(X, Z)): rows i = data points, columns j = inducing points
  const int nl = s->kp.ard ? D : 1, nred = nl + 1;
  const int nchunk = (int)std::max<long>(1, std::min<long>((N + 31) / 32, (4 * c->num_sms + mt - 1) / mt));
  const long mchunk = ((N + nchunk - 1) / nchunk + 31) / 32 * 32;
  const int nch = (int)((N + mchunk - 1) / mchunk);
  const size_t part_full = (size_t)mt * ntl * nred * 8, part_x = (size_t)nch * M * D * 8 + (size_t)M * D * 8;
  GPX_CHECK(ensure_part(s, std::max(part_full, part_x)));
  GradFullParams gp;
  memset(&gp, 0, sizeof(gp));
  gp.x1T = s->XsT; gp.ld1 = Npad; gp.sq1 = s->sqX; gp.N = N;
  gp.x2T = s->ZsT; gp.ld2 = Mpad; gp.sq2 = s->sqZ; gp.M = M;
  gp.dL_dK = s->dLt; gp.ldd = Mpad; gp.same = 0; gp.partials = s->part; gp.kp = s->kp;
  gp.ci = s->Yb; gp.ldci = Npad; gp.cj = s->Cm; gp.ldcj = Mpad; gp.cP = P;
  GPX_CHECK(launch_grad_full(gp, mt, ntl, st));
  std::vector<double> hp((size_t)mt * ntl * nred);
  GPX_CUDA(cudaMemcpyAsync(hp.data(), s->part, hp.size() * 8, cudaMemcpyDeviceToHost, st));
  GPX_CUDA(cudaStreamSynchronize(st));
  {
    std::vector<double> tot(nred, 0.0);
    for (size_t t = 0; t < (size_t)mt * ntl; t++)
      for (int q = 0; q < nred; q++) tot[q] += hp[t * nred + q];
    *dvariance = tot[0];
    for (int q = 0; q < nl; q++) dlengthscale[q] = -tot[1 + q] / s->kp.ls[q];
  }
  // dL/dZ: gradients_X(dL_dKnm^T, Z, X): rows = inducing points, columns = data points, dL read transposed
  GradFullParams gx;
  memset(&gx, 0, sizeof(gx));
  gx.x1T = s->ZsT; gx.ld1 = Mpad; gx.sq1 = s->sqZ; gx.N = M;
  gx.x2T = s->XsT; gx.ld2 = Npad; gx.sq2 = s->sqX; gx.M = N;
  gx.dL_dK = s->dLt; gx.ldd = Mpad; gx.transposed = 1; gx.same = 0; gx.kp = s->kp;
  gx.ci = s->Cm; gx.ldci = Mpad; gx.cj = s->Yb; gx.ldcj = Npad; gx.cP = P;
  double* dout = s->part + (size_t)nch * M * D;
  GPX_CHECK(launch_gradx(gx, nch, mchunk, s->part, dout, st));
  GPX_CUDA(cudaMemcpyAsync(dZ, dout, (size_t)M * D * 8, cudaMemcpyDeviceToHost, st));
  GPX_CUDA(cudaStreamSynchronize(st));
  c->total_launches += 5;
  return 0;
}

// =================================================================================================================
// Full-device VarDTC evaluation: var_dtc.py:66-215 + sparse_gp.py:108-119 with every M x M product on the DMMA GEMM.
// All products are written as X Y^T (the kernel's native NT form) over column-major operands:
//   Lm, Um = Lm^-T from the factor-and-invert sweep of Kmm + 1e-8 I;  Lmi = Um^T
//   A = beta (Lmi G) Lmi^T;  B = I + A -> LB, UB;  Q = LBi Um^T (= LBi Lmi);  v = Q psi1Vf;  C = Q^T v;  w = UB v
//   B^-1 = UB UB^T;  DBi = P B^-1 + w w^T;  dL_dKmm = Um (..) Um^T;  dL_dpsi2 = beta/2 Um (P I - DBi) Um^T
// =================================================================================================================
static int mm_nt(gpx_ctx* c, const double* A, const double* B, double* C, long Mpad, int plain = 1) {
  GemmParams pg = gemm_defaults();
  pg.mode = GEMM_PANEL; pg.plain = plain;
  pg.A = A; pg.lda = Mpad; pg.B = B; pg.ldb = Mpad; pg.C = C; pg.ldc = Mpad;
  pg.K = (int)Mpad; pg.nt = (int)(Mpad / TILE); pg.ncols = (int)(Mpad / TILE);
  c->total_launches++;
  return launch_gemm(pg, dim3(1, 1), c->st);
}
static int combine(gpx_ctx* c, double* out, long Mpad, long n, double a, const double* X, double b, const double* Y,
                   double cdiag, double d = 0.0, const double* U = nullptr, int P = 0) {
  dim3 grid((unsigned)((n + 255) / 256), (unsigned)n);
  combine_kernel<<<grid, 256, 0, c->st>>>(out, Mpad, n, a, X, b, Y, cdiag, d, U, Mpad, P);
  GPX_CUDA(cudaGetLastError());
  c->total_launches++;
  return 0;
}

// noise_vec == nullptr: scalar noise variance `noise` (grad = [variance, lengthscale.., noise variance]);
// noise_vec (host, one variance per row held by this rank): grad = [variance, lengthscale..], dL_dR (host, N x P row-major)
static int sparse_eval_impl(gpx_ctx* c, int kind, int ard, double variance, const double* lengthscale, const double* Z,
                            int64_t M, double noise, const double* noise_vec, double* lml, double* grad, double* dZ,
                            double* dL_dR_out) {
  if (!c || !c->sparse || !c->sparse->X) GPX_FAIL("gpx_sparse_set_data has not been called");
  if (!Z || !lml || !grad || !dZ || !lengthscale) GPX_FAIL("null argument");
  if (M < 1) GPX_FAIL("M must be positive");
  const bool het = noise_vec != nullptr;
  if (het && !dL_dR_out) GPX_FAIL("null argument");
  GPX_CUDA(cudaSetDevice(c->device));
  SparseState* s = c->sparse;
  cudaStream_t st = c->st;
  s->have_eval = false;
  // per-point precisions beta_n = 1 / max(variance_n, const_jitter) (var_dtc.py:79-84) and the sums over n the bound needs
  std::vector<double> hbeta, hsb;
  double sum_log_beta = 0.0, sum_beta = 0.0;
  if (het) {
    const long Nl = s->N, Npd = s->Npad;
    hbeta.assign((size_t)Npd, 0.0); hsb.assign((size_t)Npd, 0.0);
    for (long n = 0; n < Nl; n++) {
      if (!(noise_vec[n] == noise_vec[n])) GPX_FAIL("noise variance is NaN");
      const double b = 1.0 / std::max(noise_vec[n], 1e-8);
      hbeta[n] = b; hsb[n] = sqrt(b);
      sum_log_beta += log(b); sum_beta += b;
    }
    if (!s->hb) {
      GPX_CUDA(cudaMalloc(&s->hb, (size_t)2 * Npd * 8));
      GPX_CUDA(cudaMalloc(&s->hs, (size_t)(2 + s->P) * Npd * 8));
    }
    GPX_CUDA(cudaMemcpyAsync(s->hb, hsb.data(), (size_t)Npd * 8, cudaMemcpyHostToDevice, st));
    GPX_CUDA(cudaMemcpyAsync(s->hb + Npd, hbeta.data(), (size_t)Npd * 8, cudaMemcpyHostToDevice, st));
    GPX_CUDA(cudaStreamSynchronize(st));   // the host vectors are pageable
  }
  GPX_CHECK(psi_device(c, kind, ard, variance, lengthscale, Z, M));
  const long Mpad = s->Mpad, N = s->Ntot, Npad = s->Npad;
  const int D = s->D, P = s->P, mt = (int)(Mpad / TILE), ntl = (int)(Npad / TILE);
  const int nl = s->kp.ard ? D : 1;
  constexpr int RSPLIT = 64;
  if (!s->mm[0]) {
    for (auto& p : s->mm) GPX_CUDA(cudaMalloc(&p, (size_t)Mpad * Mpad * 8));
    GPX_CUDA(cudaMalloc(&s->vec, (size_t)(8 + RSPLIT) * P * Mpad * 8));
  }
  if (!s->red) {
    GPX_CUDA(cudaMalloc(&s->red, 4096 * 8));
    GPX_CUDA(cudaMallocHost(&s->h_red, 4096 * 8));
  }
  if (!s->cK) { GPX_CHECK(gpx_create(c->device, &s->cK)); GPX_CHECK(gpx_create(c->device, &s->cB)); }
  double *Kd = s->mm[0], *Um = s->mm[1], *Lmi = s->mm[2], *T = s->mm[3], *Ar = s->mm[4], *Bd = s->mm[5], *UB = s->mm[6],
         *LBi = s->mm[7], *DB = s->mm[8], *E = s->mm[9];
  double *tv = s->vec, *vv = tv + (size_t)P * Mpad, *Cv = vv + (size_t)P * Mpad, *wv = Cv + (size_t)P * Mpad,
         *xv = wv + (size_t)P * Mpad, *rpart = s->vec + (size_t)8 * P * Mpad;
  // scalar noise: beta multiplies A, psi1Vf and dL_dpsi2 as a number; per-point noise: it is inside tmp, Y and the columns
  // of dL_dKnm^T already, and the same formulas run with beta = 1
  const double beta = het ? 1.0 : 1.0 / std::max(noise, 1e-8);                           // var_dtc.py:79-80
  s->noise = het ? 0.0 : noise;
  const double *sbv = het ? s->hb : nullptr, *bvec = het ? s->hb + Npad : nullptr;
  // Kmm (dense, zero padded), factor-and-invert with const_jitter (var_dtc.py:93-95)
  GPX_CUDA(cudaMemsetAsync(Kd, 0, (size_t)Mpad * Mpad * 8, st));
  {
    KBuildParams kb;
    memset(&kb, 0, sizeof(kb));
    kb.kp = s->kp; kb.sym = 0; kb.same = 1;
    kb.rowsT = s->ZsT; kb.ld_rows = Mpad; kb.sq_rows = s->sqZ; kb.colsT = s->ZsT; kb.ld_cols = Mpad; kb.sq_cols = s->sqZ;
    kb.out = Kd; kb.ld = Mpad; kb.nrows = M; kb.ncols = M;
    GPX_CHECK(launch_kbuild(kb, mt, mt, st));
  }
  GPX_CUDA(cudaStreamSynchronize(st));
  {
    const int rc = factor_device(s->cK, Kd, Mpad, M, 1e-8, 5, nullptr, nullptr);
    if (rc) return rc;
  }
  if (s->cK->Npad != Mpad) GPX_FAIL("internal: child workspace size");
  GPX_CHECK(launch_assemble(s->cK->S, Mpad, (int)Mpad, Um, Mpad, Lmi, s->cK->st));      // Um (clean upper), Lmi = Um^T
  GPX_CUDA(cudaStreamSynchronize(s->cK->st));
  // tmp = Lm^-1 psi1^T (M x N; var_dtc.py:131,139 dtrtrs) as a product with the triangular inverse, k-range <= row tile.
  // A = tmp tmp^T is then formed from O(1) entries. (Forming G = psi1^T psi1 first and sandwiching it, Lm^-1 G Lm^-T,
  // saves 2 M^2 N flops but cancels ~cond(Kmm) digits: measured 1e-4 instead of 1e-8 on dL/dZ at cond(Kmm) = 2e8.)
  double* Tuf = s->dLt;   // the dL_dKnm^T buffer is free until knm_grads_device
  {
    GemmParams pg = gemm_defaults();
    pg.mode = GEMM_PANEL; pg.plain = 1; pg.tri = 2;
    pg.A = Lmi; pg.lda = Mpad; pg.B = s->Kfu; pg.ldb = Npad; pg.C = Tuf; pg.ldc = Mpad;
    pg.K = (int)Mpad; pg.nt = mt; pg.ncols = ntl;
    GPX_CHECK(launch_gemm(pg, dim3(1, 1), st));
  }
  const double* Yrow = s->Y;   // right-hand side of t = tmp Y
  if (het) {
    // s1_n = sum_a tmp[a, n]^2 (var_dtc.py:249, before the scaling); then tmp[:, n] *= sqrt(beta_n) (:127,131), Y_n likewise
    GPX_CHECK(launch_col_sqnorm(Tuf, Mpad, M, s->N, s->hs, st));
    scale_cols_kernel<<<(unsigned)((Mpad * s->N + 255) / 256), 256, 0, st>>>(Tuf, Mpad, s->N, sbv);
    GPX_CUDA(cudaGetLastError());
    ymul_kernel<<<(unsigned)((Npad * P + 255) / 256), 256, 0, st>>>(s->Y, sbv, Npad, P, s->Yb);
    GPX_CUDA(cudaGetLastError());
    Yrow = s->Yb;
    c->total_launches += 3;
  }
  {
    GemmParams pg = gemm_defaults();   // A_raw = tmp tmp^T (lower tiles), k-depth = Npad
    pg.mode = GEMM_PANEL; pg.plain = 2;
    pg.A = Tuf; pg.lda = Mpad; pg.B = Tuf; pg.ldb = Mpad; pg.C = Ar; pg.ldc = Mpad;
    pg.K = (int)Npad; pg.nt = mt; pg.ncols = mt;
    GPX_CHECK(launch_gemm(pg, dim3(1, 1), st));
  }
  GPX_CHECK(launch_row_dot(Tuf, Mpad, Mpad, s->N, P, Yrow, Npad, RSPLIT, rpart, tv, st));   // t = tmp Y  ([P][Mpad])
  // row shards: A_raw and t are sums over data points -> one M x M and one M x P all-reduce
  // (the pattern of var_dtc_parallel.py:113-131 with NCCL instead of mpi4py)
  GPX_CHECK(dist_allreduce_sum(c, Ar, (size_t)Mpad * Mpad, st));
  GPX_CHECK(dist_allreduce_sum(c, tv, (size_t)Mpad * P, st));
  {
    dim3 grid((unsigned)((Mpad + 255) / 256), (unsigned)Mpad);
    mirror_tiles_kernel<<<grid, 256, 0, st>>>(Ar, Mpad, Mpad);
    GPX_CUDA(cudaGetLastError());
  }
  c->total_launches += 6;
  // B = I + beta A_raw  (var_dtc.py:135-136)
  GPX_CHECK(combine(c, Bd, Mpad, Mpad, beta, Ar, 0.0, nullptr, 1.0));
  GPX_CUDA(cudaStreamSynchronize(st));
  double logdetB = 0.0;
  {
    const int rc = factor_device(s->cB, Bd, Mpad, M, 0.0, 5, &logdetB, nullptr);
    if (rc) return rc;
  }
  GPX_CHECK(launch_assemble(s->cB->S, Mpad, (int)Mpad, UB, Mpad, LBi, s->cB->st));
  GPX_CUDA(cudaStreamSynchronize(s->cB->st));
  // v = LB^-1 (beta t) (:139-141) ; w = LB^-T v ; C = Lm^-T w (:142-143)   [col_dot(A, y) = A^T y]
  scale_kernel<<<(unsigned)((Mpad * P + 255) / 256), 256, 0, st>>>(tv, beta, Mpad * P, xv);
  GPX_CUDA(cudaGetLastError());
  GPX_CHECK(launch_col_dot(UB, Mpad, Mpad, Mpad, P, xv, Mpad, vv, Mpad, st));           // v = UB^T x = LBi x
  GPX_CHECK(launch_col_dot(LBi, Mpad, Mpad, Mpad, P, vv, Mpad, wv, Mpad, st));          // w = LBi^T v
  GPX_CHECK(launch_col_dot(Lmi, Mpad, Mpad, Mpad, P, wv, Mpad, Cv, Mpad, st));          // C = Lmi^T w
  std::vector<double> hstat, hY;
  if (het) {
    // _compute_dL_dR, het_noise (var_dtc.py:241-257): per data point
    //   r_np = (v_p^T LB^-1 Lm^-1 psi1^T)_n = w_p . tmp[:, n]     (here from the scaled tmp: r_np sqrt(beta_n))
    //   s2_n = |LB^-1 Lm^-1 psi1^T[:, n]|^2 = |(Q psi1^T)[:, n]|^2,  Q = LB^-1 Lm^-1 (lower triangular)
    double *s2v = s->hs + Npad, *rv = s->hs + 2 * Npad;
    GPX_CHECK(launch_col_dot(Tuf, Mpad, M, s->N, P, wv, Mpad, rv, Npad, st));
    GPX_CHECK(mm_nt(c, LBi, Um, T, Mpad));                                                // Q = LBi Um^T = LBi Lmi
    {
      GemmParams pg = gemm_defaults();
      pg.mode = GEMM_PANEL; pg.plain = 1; pg.tri = 2;
      pg.A = T; pg.lda = Mpad; pg.B = s->Kfu; pg.ldb = Npad; pg.C = s->dLt; pg.ldc = Mpad;
      pg.K = (int)Mpad; pg.nt = mt; pg.ncols = ntl;
      GPX_CHECK(launch_gemm(pg, dim3(1, 1), st));
    }
    GPX_CHECK(launch_col_sqnorm(s->dLt, Mpad, M, s->N, s2v, st));
    hstat.resize((size_t)(2 + P) * Npad);
    hY.resize((size_t)P * Npad);
    GPX_CUDA(cudaMemcpyAsync(hstat.data(), s->hs, hstat.size() * 8, cudaMemcpyDeviceToHost, st));
    GPX_CUDA(cudaMemcpyAsync(hY.data(), s->Y, hY.size() * 8, cudaMemcpyDeviceToHost, st));
    c->total_launches += 3;
  }
  // Binv = UB UB^T (lower tiles, mirrored) ; DBi = P Binv + w w^T
  GPX_CHECK(mm_nt(c, UB, UB, DB, Mpad, 2));
  {
    dim3 grid((unsigned)((Mpad + 255) / 256), (unsigned)Mpad);
    mirror_tiles_kernel<<<grid, 256, 0, st>>>(DB, Mpad, Mpad);
    GPX_CUDA(cudaGetLastError());
  }
  GPX_CHECK(combine(c, DB, Mpad, Mpad, (double)P, DB, 0.0, nullptr, 0.0, 1.0, wv, P));
  // scalars: trace(A_raw), sum(A_raw .* DBi), |v|^2
  const int RB = 64;
  trace_dot_kernel<<<RB, 256, 0, st>>>(Ar, DB, Mpad, M, s->red);
  GPX_CUDA(cudaGetLastError());
  GPX_CUDA(cudaMemcpyAsync(s->h_red, s->red, 2 * RB * 8, cudaMemcpyDeviceToHost, st));
  std::vector<double> hv((size_t)P * Mpad);
  GPX_CUDA(cudaMemcpyAsync(hv.data(), vv, hv.size() * 8, cudaMemcpyDeviceToHost, st));
  // dL_dKmm = Um (-0.5 DBi - 0.5 P B + P I) Um^T   (var_dtc.py:152-156)
  GPX_CHECK(combine(c, E, Mpad, Mpad, -0.5, DB, -0.5 * P, Bd, (double)P));
  GPX_CHECK(mm_nt(c, Um, E, T, Mpad));
  GPX_CHECK(mm_nt(c, T, Um, Kd, Mpad));                                                  // Kd now holds dL_dKmm
  // W2 = 2 dL_dpsi2 = beta Um (P I - DBi) Um^T     (var_dtc.py:221,231-233)
  GPX_CHECK(combine(c, E, Mpad, Mpad, -1.0, DB, 0.0, nullptr, (double)P));
  GPX_CHECK(mm_nt(c, Um, E, T, Mpad));
  GPX_CHECK(mm_nt(c, T, Um, E, Mpad));
  GPX_CHECK(combine(c, s->W2, Mpad, Mpad, beta, E, 0.0, nullptr, 0.0));
  // Knm part: needs C in s->Cm
  GPX_CUDA(cudaMemcpyAsync(s->Cm, Cv, (size_t)P * Mpad * 8, cudaMemcpyDeviceToDevice, st));
  double dv_knm = 0.0;
  std::vector<double> dl_knm(nl, 0.0);
  GPX_CHECK(knm_grads_device(c, beta, bvec, &dv_knm, dl_knm.data(), dZ));               // dZ <- Knm part
  {
    int rank = 0, G = 1;
    dist_world(c, &rank, &G);
    if (G > 1) {   // sums over this rank's data points -> totals
      std::vector<double> h((size_t)1 + nl + (size_t)M * D);
      h[0] = dv_knm;
      for (int q = 0; q < nl; q++) h[1 + q] = dl_knm[q];
      memcpy(h.data() + 1 + nl, dZ, (size_t)M * D * 8);
      GPX_CUDA(cudaMemcpyAsync(s->gsum, h.data(), h.size() * 8, cudaMemcpyHostToDevice, st));
      GPX_CHECK(dist_allreduce_sum(c, s->gsum, h.size(), st));
      GPX_CUDA(cudaMemcpyAsync(h.data(), s->gsum, h.size() * 8, cudaMemcpyDeviceToHost, st));
      GPX_CUDA(cudaStreamSynchronize(st));
      dv_knm = h[0];
      for (int q = 0; q < nl; q++) dl_knm[q] = h[1 + q];
      memcpy(dZ, h.data() + 1 + nl, (size_t)M * D * 8);
    }
  }
  // Kmm part: kern.update_gradients_full(dL_dKmm, Z) and kern.gradients_X(dL_dKmm, Z)  (sparse_gp.py:114,117)
  const int nred = nl + 1;
  GradFullParams gp;
  memset(&gp, 0, sizeof(gp));
  gp.x1T = s->ZsT; gp.ld1 = Mpad; gp.sq1 = s->sqZ; gp.N = M;
  gp.x2T = s->ZsT; gp.ld2 = Mpad; gp.sq2 = s->sqZ; gp.M = M;
  gp.dL_dK = Kd; gp.ldd = Mpad; gp.same = 1; gp.partials = s->part; gp.kp = s->kp;
  GPX_CHECK(launch_grad_full(gp, mt, mt, st));
  std::vector<double> hp((size_t)mt * mt * nred);
  GPX_CUDA(cudaMemcpyAsync(hp.data(), s->part, hp.size() * 8, cudaMemcpyDeviceToHost, st));
  GPX_CUDA(cudaStreamSynchronize(st));
  double dv_kmm = 0.0;
  std::vector<double> dl_kmm(nl, 0.0);
  {
    std::vector<double> tot(nred, 0.0);
    for (size_t t = 0; t < (size_t)mt * mt; t++)
      for (int q = 0; q < nred; q++) tot[q] += hp[t * nred + q];
    dv_kmm = tot[0];
    for (int q = 0; q < nl; q++) dl_kmm[q] = -tot[1 + q] / s->kp.ls[q];
  }
  {
    const int nchunk = (int)std::max<long>(1, std::min<long>((M + 31) / 32, (4 * c->num_sms + mt - 1) / mt));
    const long mchunk = ((M + nchunk - 1) / nchunk + 31) / 32 * 32;
    const int nch = (int)((M + mchunk - 1) / mchunk);
    GPX_CHECK(ensure_part(s, (size_t)(nch + 1) * M * D * 8));
    GradFullParams gx = gp;
    gx.partials = nullptr;
    double* dout = s->part + (size_t)nch * M * D;
    GPX_CHECK(launch_gradx(gx, nch, mchunk, s->part, dout, st));
    std::vector<double> hz((size_t)M * D);
    GPX_CUDA(cudaMemcpyAsync(hz.data(), dout, hz.size() * 8, cudaMemcpyDeviceToHost, st));
    GPX_CUDA(cudaStreamSynchronize(st));
    for (size_t i = 0; i < hz.size(); i++) dZ[i] += hz[i];
  }
  c->total_launches += 8;
  // ---- scalars on the host (var_dtc.py:237-276, homoscedastic) -----------------------------------------------------
  double trAr = 0.0, sumAD = 0.0, data_fit = 0.0;
  for (int b = 0; b < RB; b++) { trAr += s->h_red[2 * b]; sumAD += s->h_red[2 * b + 1]; }
  for (int q = 0; q < P; q++)
    for (long i = 0; i < M; i++) data_fit += hv[(size_t)q * Mpad + i] * hv[(size_t)q * Mpad + i];
  const double trA = beta * trAr, sumADB = beta * sumAD;
  const double psi0_sum = variance * (double)N;
  const double nd = (double)N, od = (double)P;
  const double log2pi = 1.8378770664093453;
  const double lik_3 = -od * 0.5 * logdetB;
  const double lik_4 = 0.5 * data_fit;
  if (het) {
    // bound (var_dtc.py:267-269) and the N x P per-point noise gradients (:245-257), rows of this rank
    const long Nl = s->N;
    const double *s1 = hstat.data(), *s2 = s1 + Npad, *rs = s2 + Npad;
    double sum_bY2 = 0.0;
    for (long n = 0; n < Nl; n++) {
      const double b = hbeta[n], b2 = b * b;
      const double common = -0.5 * b + 0.5 * od * (variance - s1[n]) * b2 + 0.5 * s2[n] * b2;
      for (int q = 0; q < P; q++) {
        // r was formed from the scaled tmp: undo sqrt(beta_n); an infinite noise variance (beta_n = 0) switches the point off
        const double y = hY[(size_t)q * Npad + n], r = hsb[n] > 0.0 ? rs[(size_t)q * Npad + n] / hsb[n] : 0.0;
        sum_bY2 += b * y * y;
        dL_dR_out[n * P + q] = common + 0.5 * (b * y) * (b * y) - r * y * b2 + 0.5 * r * r * b2;
      }
    }
    double sums[3] = {sum_log_beta, sum_beta, sum_bY2};
    {
      int rank = 0, G = 1;
      dist_world(c, &rank, &G);
      if (G > 1) {   // sums over this rank's rows -> totals
        memcpy(s->h_red, sums, sizeof(sums));
        GPX_CUDA(cudaMemcpyAsync(s->red, s->h_red, sizeof(sums), cudaMemcpyHostToDevice, st));
        GPX_CHECK(dist_allreduce_sum(c, s->red, 3, st));
        GPX_CUDA(cudaMemcpyAsync(s->h_red, s->red, sizeof(sums), cudaMemcpyDeviceToHost, st));
        GPX_CUDA(cudaStreamSynchronize(st));
        memcpy(sums, s->h_red, sizeof(sums));
      }
    }
    const double lik_1h = -0.5 * nd * od * log2pi + 0.5 * od * sums[0] - 0.5 * sums[2];
    const double lik_2h = -0.5 * od * (variance * sums[1] - trA);
    *lml = lik_1h + lik_2h + lik_3 + lik_4;
    grad[0] = -0.5 * od * sums[1] + dv_knm + dv_kmm;                                       // update_gradients_diag (:110)
    for (int q = 0; q < nl; q++) grad[1 + q] = dl_knm[q] + dl_kmm[q];
    s->have_eval = true;
    return 0;
  }
  const double lik_1 = -0.5 * nd * od * (log2pi - log(beta)) - 0.5 * beta * s->trYYT;
  const double lik_2 = -0.5 * od * (beta * psi0_sum - trA);
  *lml = lik_1 + lik_2 + lik_3 + lik_4;
  double dL_dR = -0.5 * nd * od * beta + 0.5 * s->trYYT * beta * beta;
  dL_dR += 0.5 * od * (psi0_sum * beta * beta - trA * beta);
  dL_dR += beta * (0.5 * sumADB - data_fit);
  // d beta / d noise is folded by the reference into dL_dR (gradient wrt the noise VARIANCE): exact_inference_gradients
  // sums dL_dR as is (var_dtc.py:176, gaussian.py:78-79)
  const double dvar_diag = -0.5 * od * beta * nd;                                          // update_gradients_diag (:110)
  grad[0] = dvar_diag + dv_knm + dv_kmm;
  for (int q = 0; q < nl; q++) grad[1 + q] = dl_knm[q] + dl_kmm[q];
  grad[1 + nl] = dL_dR;
  s->have_eval = true;
  return 0;
}

extern "C" {

int gpx_sparse_eval(gpx_ctx* c, int kind, int ard, double variance, const double* lengthscale, const double* Z, int64_t M,
                    double noise, double* lml, double* grad, double* dZ) {
  return sparse_eval_impl(c, kind, ard, variance, lengthscale, Z, M, noise, nullptr, lml, grad, dZ, nullptr);
}

int gpx_sparse_eval_het(gpx_ctx* c, int kind, int ard, double variance, const double* lengthscale, const double* Z,
                        int64_t M, const double* noise_variances, double* lml, double* grad, double* dZ, double* dL_dR) {
  if (!noise_variances) GPX_FAIL("null argument");
  return sparse_eval_impl(c, kind, ard, variance, lengthscale, Z, M, 0.0, noise_variances, lml, grad, dZ, dL_dR);
}

/* which: 0 woodbury_vector (M x P row-major), 1 woodbury_inv (M x M), 2 Kmm (+1e-8 I), 3 Lm (lower, col-major) */
int gpx_sparse_get(gpx_ctx* c, int which, double* out) {
  if (!c || !c->sparse || !c->sparse->have_eval || !out) GPX_FAIL("no sparse evaluation to fetch from");
  GPX_CUDA(cudaSetDevice(c->device));
  SparseState* s = c->sparse;
  cudaStream_t st = c->st;
  const long M = s->M, Mpad = s->Mpad;
  const int P = s->P;
  if (which == 0) {
    std::vector<double> h((size_t)P * Mpad);
    GPX_CUDA(cudaMemcpyAsync(h.data(), s->Cm, h.size() * 8, cudaMemcpyDeviceToHost, st));
    GPX_CUDA(cudaStreamSynchronize(st));
    for (long i = 0; i < M; i++)
      for (int q = 0; q < P; q++) out[i * P + q] = h[(size_t)q * Mpad + i];
    return 0;
  }
  double* src = nullptr;
  if (which == 1) {   // woodbury_inv = Um (I - B^-1) Um^T   (var_dtc.py:207-210); B^-1 = (DBi - w w^T) / P is rebuilt
    double *Um = s->mm[1], *UB = s->mm[6], *T = s->mm[3], *E = s->mm[9], *DB = s->mm[8];
    GPX_CHECK(mm_nt(c, UB, UB, DB, Mpad, 2));
    dim3 grid((unsigned)((Mpad + 255) / 256), (unsigned)Mpad);
    mirror_tiles_kernel<<<grid, 256, 0, st>>>(DB, Mpad, Mpad);
    GPX_CUDA(cudaGetLastError());
    GPX_CHECK(combine(c, E, Mpad, Mpad, -1.0, DB, 0.0, nullptr, 1.0));
    GPX_CHECK(mm_nt(c, Um, E, T, Mpad));
    GPX_CHECK(mm_nt(c, T, Um, E, Mpad));
    src = E;
  } else if (which == 2 || which == 3) {
    // Kmm / Lm from the child context's factor: rebuild Kmm by the kernel build, Lm by extraction
    if (which == 2) {
      double* Kd = s->mm[3];
      GPX_CUDA(cudaMemsetAsync(Kd, 0, (size_t)Mpad * Mpad * 8, st));
      KBuildParams kb;
      memset(&kb, 0, sizeof(kb));
      kb.kp = s->kp; kb.sym = 0; kb.same = 1;
      kb.rowsT = s->ZsT; kb.ld_rows = Mpad; kb.sq_rows = s->sqZ; kb.colsT = s->ZsT; kb.ld_cols = Mpad; kb.sq_cols = s->sqZ;
      kb.out = Kd; kb.ld = Mpad; kb.nrows = M; kb.ncols = M;
      GPX_CHECK(launch_kbuild(kb, (int)(Mpad / TILE), (int)(Mpad / TILE), st));
      GPX_CHECK(combine(c, Kd, Mpad, M, 1.0, Kd, 0.0, nullptr, 1e-8));
      src = Kd;
    } else {
      double* Ld = s->mm[3];
      GPX_CUDA(cudaStreamSynchronize(st));
      GPX_CHECK(launch_extract(GPX_GET_L, s->cK->S, Mpad, s->cK->Ldiag, nullptr, nullptr, 0, Mpad, Ld, s->cK->st));
      GPX_CUDA(cudaStreamSynchronize(s->cK->st));
      src = Ld;
    }
  } else {
    GPX_FAIL("unknown gpx_sparse_get selector");
  }
  GPX_CUDA(cudaMemcpy2DAsync(out, M * 8, src, Mpad * 8, (size_t)M * 8, M, cudaMemcpyDeviceToHost, st));
  GPX_CUDA(cudaStreamSynchronize(st));
  return 0;
}

}  // extern "C"
