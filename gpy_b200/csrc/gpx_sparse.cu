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
#include "gpx_ep.cuh"
#include "gpx_psi.cuh"

using namespace gpx;

struct SparseState {
  long N = 0, Npad = 0, M = 0, Mpad = 0;   // N: rows held by THIS rank (all of them on one GPU)
  long Ntot = 0;                           // rows over all ranks (var_dtc.py num_data)
  long Nw = 0, Mw = 0;                     // extents of psi1 written last time (a smaller N or M must re-zero the padding)
  int D = 0, P = 0;
  long Ppad = 0;                           // P > MAX_P (the wide route): P padded to whole tiles of outputs
  double *X = nullptr, *XsT = nullptr, *sqX = nullptr, *Y = nullptr, *Yb = nullptr;   // Y: [P][Npad] ([Ppad][Npad] wide)
  double* YT = nullptr;                    // wide route: Y as [Npad][Ppad] (row-major, zero padded), the GEMM operand of t
  double *Z = nullptr, *ZsT = nullptr, *sqZ = nullptr;
  double *Kuf = nullptr;   // Mpad x Npad column-major: (a, n) at a + n*Mpad
  double *Kfu = nullptr;   // Npad x Mpad column-major: (n, a) at n + a*Npad; wide route: Ppad more columns, beta Y
  double *dLt = nullptr;   // Mpad x Npad: dL_dKnm^T
  double *Gm = nullptr, *W2 = nullptr, *Cm = nullptr;   // Mpad x Mpad (wide: Ppad more columns, C), Mpad x Mpad, [P][Mpad]
  double *part = nullptr; size_t part_cap = 0;
  int rows_cap = 0, norm_cap = 0;          // stacked coordinate rows of XsT / ZsT, squared-norm rows of sqX / sqZ
  MultiKern mk{};          // the kernel of the last evaluation
  double kdiag = 0.0;      // its Kdiag (psi0 per point)
  // full-device evaluation (gpx_sparse_eval)
  gpx_ctx *cK = nullptr, *cB = nullptr;             // child contexts holding the factors of Kmm and of B = I + A
  double *mm[10] = {nullptr};                        // Mpad x Mpad work matrices
  double *vec = nullptr;                             // [8][P][Mpad] small vectors
  double *red = nullptr; double *h_red = nullptr;    // scalar reductions
  double *gsum = nullptr;                            // [kernel gradient entries + M*D] gradient pieces summed over ranks
  double *hb = nullptr;                              // het noise: [2][Npad] sqrt(beta_n), beta_n
  double *hs = nullptr;                              // het noise: [2 + P][Npad] column reductions s1, s2, r (see eval)
  double trYYT = 0.0;
  bool have_eval = false;
  bool dl_ready = false;                             // dLt, Yb and Cm hold the dL_dKnm^T of the last VarDTC evaluation
                                                     // (gpx_sparse_grad_X reads them; every other writer clears it)
  bool w_ready = false;                              // mm[9] holds woodbury_inv of the current evaluation (formed by
                                                     // gpx_sparse_predictive_gradients, kept for its later calls)
  double noise = 0.0;
  double jitter = 1e-8;                              // const_jitter of the last evaluation (VarDTC 1e-8, FITC 1e-6)
  double *F2 = nullptr, *G = nullptr;                // FITC: Mpad x Npad, Kmm^-1 psi1^T and its columns scaled by dL_dR
  // sparse EP (gpx_epdtc_*): Kmm, A = LLT^-1 (whole, symmetric) and A at the sites zero (Mpad x Mpad each); one block of
  // sites (epb); the site vectors ([EDV_N][Npad]); the update order; the inducing inputs of gpx_epdtc_begin on the host
  double *eK = nullptr, *eA = nullptr, *eA0 = nullptr, *epb = nullptr;
  double *ev = nullptr;
  int* eord = nullptr;
  std::vector<double> eZ;
  bool ep_begun = false;    // gpx_epdtc_begin built Kmm, Kmn and A0 for the current data and Z (psi_device clears it)
  bool ep_ready = false;    // mu0, u and the held diagonal of gpx_epdtc_start / _sweep are on the device
  bool ep_labels = false;   // the labels of the current data were checked
  bool ep_seq = false;      // the sites run sequentially (A is updated)
  bool ep_first = false;    // the next site is the first of a run: its cavity reads the held diagonal of the start
  // SVGP (gpx_svgp_*): M x M work matrices beyond mm (Mpad x Mpad each); small vectors ([SV_MV][Mpad]); one allocation per
  // batch capacity sv_cap (padded rows) holding the four Mpad x sv_cap batch buffers, four sv_cap vectors and the batch's
  // prepared points (svgp_batch)
  double *svm[8] = {nullptr};
  double *svv = nullptr, *svb = nullptr;
  long sv_cap = 0, sv_row0 = 0, sv_nb = 0;
  double sv_jit = 0.0;      // what jitchol's ladder added to Kmm in the last gpx_svgp_begin
  bool sv_begun = false;    // gpx_svgp_begin ran on the current data, kernel and Z (psi_device and set_data clear it)
  bool w_own = false;       // mm[9] is the posterior's own woodbury_inv (SVGP), not formed from B's factor
  Points xpts() const { return Points{XsT, sqX, N, Npad}; }   // this rank's data points, prepared
  Points zpts() const { return Points{ZsT, sqZ, M, Mpad}; }   // the inducing points, prepared
};

namespace {
void free_m(SparseState* s) {
  double** ptrs[] = {&s->Z, &s->ZsT, &s->sqZ, &s->Kuf, &s->Kfu, &s->dLt, &s->Gm, &s->W2, &s->Cm, &s->vec, &s->gsum,
                     &s->F2, &s->G, &s->eK, &s->eA, &s->eA0, &s->epb};
  for (auto p : ptrs) { if (*p) cudaFree(*p); *p = nullptr; }
  for (auto& p : s->mm) { if (p) cudaFree(p); p = nullptr; }
  for (auto& p : s->svm) { if (p) cudaFree(p); p = nullptr; }
  for (double** p : {&s->svv, &s->svb}) { if (*p) cudaFree(*p); *p = nullptr; }
  s->sv_cap = 0;
  s->sv_begun = s->w_own = false;
  s->have_eval = false;
  s->dl_ready = false;
  s->w_ready = false;
  s->ep_begun = s->ep_ready = false;
  s->M = s->Mpad = 0;
  s->Nw = s->Mw = 0;
}
void free_all(SparseState* s) {
  free_m(s);
  double** ptrs[] = {&s->X, &s->XsT, &s->sqX, &s->Y, &s->Yb, &s->YT, &s->part, &s->red, &s->hb, &s->hs, &s->ev};
  for (auto p : ptrs) { if (*p) cudaFree(*p); *p = nullptr; }
  if (s->eord) { cudaFree(s->eord); s->eord = nullptr; }
  if (s->h_red) { cudaFreeHost(s->h_red); s->h_red = nullptr; }
  if (s->cK) { gpx_destroy(s->cK); s->cK = nullptr; }
  if (s->cB) { gpx_destroy(s->cB); s->cB = nullptr; }
  s->part_cap = 0;
  s->rows_cap = s->norm_cap = 0;
  s->N = s->Npad = s->Ppad = 0;
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
// composite route: dL_dKnm^T (a, n) += sum_q C[q][a] (beta Y)[q][n] over the valid entries, so that the composite
// reductions read a complete dL_dKnm (the single-kernel ones add this rank-P term on the fly)
__global__ void add_rank_p_kernel(double* __restrict__ dLt, long ld, long M, long N, const double* __restrict__ C,
                                  const double* __restrict__ Yb, long ldy, int P) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ld * N) return;
  const long a = i % ld, n = i / ld;
  if (a >= M) return;
  double v = dLt[i];
  for (int q = 0; q < P; q++) v = fma(C[(long)q * ld + a], Yb[(long)q * ldy + n], v);
  dLt[i] = v;
}
// uncertain inputs: dL_dpsi1 (n, a) = beta sum_q Y[q][n] C[q][a] (var_dtc.py:218), written at n + a ld (psi1's layout)
__global__ void dl_dpsi1_kernel(const double* __restrict__ Y, long ldy, const double* __restrict__ C, long ldc, int P,
                                double beta, long N, double* __restrict__ out, long ld) {
  const long n = (long)blockIdx.x * blockDim.x + threadIdx.x, a = blockIdx.y;
  if (n >= N) return;
  double v = 0.0;
  for (int q = 0; q < P; q++) v = fma(Y[(long)q * ldy + n], C[(long)q * ldc + a], v);
  out[n + a * ld] = beta * v;
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
// r[b] = partial sum of a[i]^2 over the i = b, b + 256 gridDim.x, ... < n of CTA b, in a fixed order
__global__ void __launch_bounds__(256) sumsq_kernel(const double* __restrict__ a, long n, double* __restrict__ r) {
  __shared__ double sh[256];
  double acc = 0.0;
  for (long i = (long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long)gridDim.x * 256) acc = fma(a[i], a[i], acc);
  sh[threadIdx.x] = acc;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) r[blockIdx.x] = sh[0];
}
// n kernels just issued for context c (on its stream or on a child context's): counted on c, a launch error surfaced
int launched(gpx_ctx* c, int n = 1) {
  c->total_launches += n;
  GPX_CUDA(cudaGetLastError());
  return 0;
}
// XsT / ZsT hold rows_cap stacked coordinate rows and sqX / sqZ norm_cap rows: grown when kernel k needs more (a composite
// stacks every part's active dims, which can exceed D when parts share columns, and keeps one norm row per part)
int ensure_rows(gpx_ctx* c, SparseState* s, const MultiKern& k) {
  const int rows = std::max(s->rows_cap, std::max(1, k.sumD)), norms = std::max(s->norm_cap, k.nparts);
  if (rows == s->rows_cap && norms == s->norm_cap) return 0;
  GPX_CUDA(cudaStreamSynchronize(c->st));
  double** ptrs[] = {&s->XsT, &s->sqX, &s->ZsT, &s->sqZ};
  for (auto p : ptrs) { if (*p) cudaFree(*p); *p = nullptr; }
  s->rows_cap = rows; s->norm_cap = norms;
  GPX_CUDA(cudaMalloc(&s->XsT, (size_t)s->Npad * rows * 8));
  GPX_CUDA(cudaMalloc(&s->sqX, (size_t)s->Npad * norms * 8));
  if (s->Mpad) {
    GPX_CUDA(cudaMalloc(&s->ZsT, (size_t)s->Mpad * rows * 8));
    GPX_CUDA(cudaMalloc(&s->sqZ, (size_t)s->Mpad * norms * 8));
  }
  return 0;
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
  if (N < 1 || D < 1 || D > MAX_D || P < 1 || P > (c->sparse_wide ? GPX_MAX_OUTPUTS : MAX_P))
    GPX_FAIL(c->sparse_wide ? "bad shape (D <= 64, P <= 1024)" : "bad shape (D <= 64, P <= 8; option \"sparse_wide\" takes 1024)");
  if (P > MAX_P && c->dist) GPX_FAIL("more than 8 output columns are single-GPU");
  GPX_CUDA(cudaSetDevice(c->device));
  laplace_release(c);
  if (!c->sparse) c->sparse = new SparseState();
  SparseState* s = c->sparse;
  const long Npad = (N + TILE - 1) / TILE * TILE;
  const bool wide = P > MAX_P;
  const long Ppad = wide ? (P + TILE - 1) / TILE * TILE : 0;
  if (Npad != s->Npad || D != s->D || P != s->P) {
    GPX_CUDA(cudaStreamSynchronize(c->st));
    free_all(s);
    s->Npad = Npad; s->D = D; s->P = P; s->Ppad = Ppad;
    GPX_CUDA(cudaMalloc(&s->X, (size_t)Npad * D * 8));
    GPX_CUDA(cudaMalloc(&s->XsT, (size_t)Npad * D * 8));
    GPX_CUDA(cudaMalloc(&s->sqX, (size_t)Npad * 8));
    s->rows_cap = D; s->norm_cap = 1;
    if (wide) {   // no Yb: the wide route adds the rank-P term of dL_dKnm^T inside its GEMM (knm_grads_device)
      GPX_CUDA(cudaMalloc(&s->Y, (size_t)Npad * Ppad * 8));
      GPX_CUDA(cudaMalloc(&s->YT, (size_t)Npad * Ppad * 8));
    } else {
      GPX_CUDA(cudaMalloc(&s->Y, (size_t)Npad * P * 8));
      GPX_CUDA(cudaMalloc(&s->Yb, (size_t)Npad * P * 8));
    }
  }
  s->N = N;
  s->have_eval = false;
  s->dl_ready = false;
  s->w_ready = false;
  s->ep_begun = s->ep_ready = s->ep_labels = false;
  s->sv_begun = s->w_own = false;
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
  if (wide) {   // YT: rows of Ppad, zero padded; Y = its transpose, [Ppad][Npad]
    GPX_CUDA(cudaMemsetAsync(s->YT, 0, (size_t)Npad * Ppad * 8, c->st));
    GPX_CUDA(cudaMemcpy2DAsync(s->YT, Ppad * 8, Y, (size_t)P * 8, (size_t)P * 8, N, cudaMemcpyHostToDevice, c->st));
    GPX_CHECK(launch_transpose_pad(s->YT, N, (int)Ppad, Npad, s->Y, c->st));
  } else {
    GPX_CUDA(cudaMemcpyAsync(s->Yb, Y, (size_t)N * P * 8, cudaMemcpyHostToDevice, c->st));
    GPX_CHECK(launch_transpose_pad(s->Yb, N, P, Npad, s->Y, c->st));
  }
  c->total_launches++;
  GPX_CUDA(cudaStreamSynchronize(c->st));
  return 0;
}

}  // extern "C"

// psi1 = K(X, Z) of the state's kernel in both layouts (Kuf: M x N, Kfu: N x M), left on the device. build = false (the
// uncertain-input evaluation, which writes its own psi1 into Kfu): Z and the points are set up, no K(X, Z) is built and
// Kuf is not written; FITC and EPDTC, its only readers, build it again before they read it.
static int psi_device(gpx_ctx* c, const double* Z, int64_t M, bool build = true) {
  SparseState* s = c->sparse;
  cudaStream_t st = c->st;
  const MultiKern& k = s->mk;
  GPX_CHECK(ensure_rows(c, s, k));
  const long Mpad = (M + TILE - 1) / TILE * TILE, Npad = s->Npad, N = s->N;
  s->dl_ready = false;
  if (Mpad != s->Mpad || !s->Kuf) {   // (gpx_svgp_begin sets up Z without psi1)
    GPX_CUDA(cudaStreamSynchronize(st));
    free_m(s);
    s->Mpad = Mpad;
    const long Mk = Mpad + s->Ppad;   // k-depth of dL_dKnm^T = [W2 | C] [psi1 | beta Y]^T on the wide route
    GPX_CUDA(cudaMalloc(&s->Z, (size_t)Mpad * s->D * 8));
    GPX_CUDA(cudaMalloc(&s->ZsT, (size_t)Mpad * s->rows_cap * 8));
    GPX_CUDA(cudaMalloc(&s->sqZ, (size_t)Mpad * s->norm_cap * 8));
    GPX_CUDA(cudaMalloc(&s->Kuf, (size_t)Mpad * Npad * 8));
    GPX_CUDA(cudaMalloc(&s->Kfu, (size_t)Mk * Npad * 8));
    GPX_CUDA(cudaMalloc(&s->dLt, (size_t)Mpad * Npad * 8));
    GPX_CUDA(cudaMalloc(&s->Gm, (size_t)Mpad * Mpad * 8));
    GPX_CUDA(cudaMalloc(&s->W2, (size_t)Mpad * Mk * 8));
    GPX_CUDA(cudaMalloc(&s->Cm, (size_t)Mpad * s->P * 8));
    GPX_CUDA(cudaMalloc(&s->gsum, (size_t)(MAX_D + 2 + Mpad * s->D) * 8));
    GPX_CUDA(cudaMemsetAsync(s->Gm, 0, (size_t)Mpad * Mpad * 8, st));
    GPX_CUDA(cudaMemsetAsync(s->Kuf, 0, (size_t)Mpad * Npad * 8, st));   // padding stays zero: only valid entries
    GPX_CUDA(cudaMemsetAsync(s->Kfu, 0, (size_t)Mpad * Npad * 8, st));   // are ever written
  }
  s->M = M;
  s->ep_begun = s->ep_ready = false;   // Kmn changes: a sparse EP run has to begin again
  s->sv_begun = s->w_own = false;
  if (N < s->Nw || M < s->Mw) {   // fewer points than last time inside the same padded extents: stale entries must go
    GPX_CUDA(cudaMemsetAsync(s->Kuf, 0, (size_t)Mpad * Npad * 8, st));
    GPX_CUDA(cudaMemsetAsync(s->Kfu, 0, (size_t)Mpad * Npad * 8, st));
  }
  s->Nw = N; s->Mw = M;
  GPX_CUDA(cudaMemcpyAsync(s->Z, Z, (size_t)M * s->D * 8, cudaMemcpyHostToDevice, st));
  GPX_CHECK(prep_points(c, k, s->X, N, s->D, Npad, s->XsT, s->sqX));
  GPX_CHECK(prep_points(c, k, s->Z, M, s->D, Mpad, s->ZsT, s->sqZ));
  GPX_CHECK(launched(c, 2));
  if (!build) return 0;
  GPX_CHECK(build_K(c, k, s->D, s->zpts(), s->xpts(), s->Kuf, Mpad));   // psi1^T: thread-mapped operand = inducing points
  GPX_CHECK(build_K(c, k, s->D, s->xpts(), s->zpts(), s->Kfu, Npad));   // psi1: thread-mapped operand = data points
  return launched(c, 2);
}

// C = A psi1^T (M x N) on the DMMA GEMM; tri = 2: A is lower triangular (k-range <= row tile)
static int mul_psi1T(gpx_ctx* c, const double* A, double* C, int tri) {
  SparseState* s = c->sparse;
  GemmParams pg = gemm_defaults();
  pg.mode = GEMM_PANEL; pg.plain = 1; pg.tri = tri;
  pg.A = A; pg.lda = s->Mpad; pg.B = s->Kfu; pg.ldb = s->Npad; pg.C = C; pg.ldc = s->Mpad;
  pg.K = (int)s->Mpad; pg.nt = (int)(s->Mpad / TILE); pg.ncols = (int)(s->Npad / TILE);
  GPX_CHECK(launch_gemm(pg, dim3(1, 1), c->st));
  return launched(c);
}

static int knm_reduce(gpx_ctx* c, double* grad, double* dZ);

// output columns of the rank-P term C (beta Y)^T that the Knm reductions add on the fly: a single kernel's up to MAX_P
// columns; a composite's term is added to dL_dKnm^T in one pass first, and the wide route's by its GEMM
static int rank_p_cols(const SparseState* s) {
  return as_single(s->mk, s->D, nullptr) && s->P <= MAX_P ? s->P : 0;
}

// dL_dKnm^T = W2 psi1^T (+ rank-P term: on the fly for a single kernel, added in one pass for a composite, and for P > MAX_P
// by the GEMM itself as [W2 | C] [psi1 | beta Y]^T) reduced to kernel-parameter gradients and dL/dZ; W2 (device, s->W2) and
// C (device, s->Cm as [P][Mpad]; wide route: also as [Ppad][Mpad] in the columns of s->W2 after W2) must be in place.
// Results on the host.
// bvec (device, [Npad], per-point precisions) selects the heteroscedastic form: VVT_factor = beta_n Y_n and the columns of
// W2 psi1^T scaled by beta_n (var_dtc.py:226); W2 is then 2 dL_dpsi2_beta without the scalar beta.
static int knm_grads_device(gpx_ctx* c, double beta, const double* bvec, double* grad, double* dZ) {
  SparseState* s = c->sparse;
  cudaStream_t st = c->st;
  const long Mpad = s->Mpad, N = s->N, Npad = s->Npad;
  const int P = s->P;
  if (P > MAX_P) {   // scalar noise only: beta Y into the columns of Kfu after psi1, k-depth Mpad + Ppad
    const long Ppad = s->Ppad;
    scale_kernel<<<(unsigned)((Npad * Ppad + 255) / 256), 256, 0, st>>>(s->Y, beta, Npad * Ppad, s->Kfu + (size_t)Npad * Mpad);
    GPX_CHECK(launched(c));
    GPX_CHECK(gemm_nt(c, s->W2, Mpad, s->Kfu, Npad, s->dLt, Mpad, Mpad, Npad, Mpad + Ppad, 1, 0));
    GPX_CUDA(cudaGetLastError());
    return knm_reduce(c, grad, dZ);
  }
  if (bvec)
    ymul_kernel<<<(unsigned)((Npad * P + 255) / 256), 256, 0, st>>>(s->Y, bvec, Npad, P, s->Yb);
  else
    scale_kernel<<<(unsigned)((Npad * P + 255) / 256), 256, 0, st>>>(s->Y, beta, Npad * P, s->Yb);
  GPX_CHECK(launched(c));
  GPX_CHECK(mul_psi1T(c, s->W2, s->dLt, 0));   // dLt = W2 * psi1^T  (M x N), W2 symmetric
  if (bvec) {
    scale_cols_kernel<<<(unsigned)((Mpad * N + 255) / 256), 256, 0, st>>>(s->dLt, Mpad, N, bvec);
    GPX_CHECK(launched(c));
  }
  return knm_reduce(c, grad, dZ);
}

// dL_dKnm^T = dLt + sum_q C[q] (Yb[q])^T reduced to kernel-parameter gradients and dL/dZ (results on the host) for the
// data points xp: dLt (Mpad x xp.ld, column-major), C (s->Cm, [P][Mpad]) and Yb ([P][ldy]) must be in place
static int knm_reduce_at(gpx_ctx* c, const Points& xp, double* dLt, const double* Yb, long ldy, double* grad, double* dZ) {
  SparseState* s = c->sparse;
  cudaStream_t st = c->st;
  const long Mpad = s->Mpad, N = xp.n;
  const int P = s->P;
  // kernel-parameter gradients of sum(dL_dKnm * K(X, Z)): rows i = data points, columns j = inducing points
  const MultiKern& k = s->mk;
  const bool single = as_single(k, s->D, nullptr);
  if (!single && P <= MAX_P) {
    add_rank_p_kernel<<<(unsigned)((Mpad * N + 255) / 256), 256, 0, st>>>(dLt, Mpad, s->M, N, s->Cm, Yb, ldy, P);
    GPX_CHECK(launched(c));
  }
  const int cP = rank_p_cols(s);
  GradFullParams gp = grad_params(k, s->D, xp, s->zpts(), dLt, Mpad);
  gp.ci = Yb; gp.ldci = ldy; gp.cj = s->Cm; gp.ldcj = Mpad; gp.cP = cP;
  GPX_CHECK(ensure_part(s, grad_full_doubles(k, s->D, gp) * 8));
  GPX_CHECK(grad_full_sum(c, k, s->D, gp, s->part, grad));
  // dL/dZ: gradients_X(dL_dKnm^T, Z, X): rows = inducing points, columns = data points, dL read transposed
  GradFullParams gx = grad_params(k, s->D, s->zpts(), xp, dLt, Mpad);
  gx.transposed = 1; gx.ci = s->Cm; gx.ldci = Mpad; gx.cj = Yb; gx.ldcj = ldy; gx.cP = cP;
  GPX_CHECK(ensure_part(s, grad_X_doubles(c, k, gx, s->D) * 8));
  return grad_X(c, k, gx, s->D, s->part, dZ);
}
// the same for the data of gpx_sparse_set_data with dL_dKnm^T in s->dLt and the rank-P factor in s->Yb
static int knm_reduce(gpx_ctx* c, double* grad, double* dZ) {
  SparseState* s = c->sparse;
  return knm_reduce_at(c, s->xpts(), s->dLt, s->Yb, s->Npad, grad, dZ);
}

// =================================================================================================================
// Full-device VarDTC evaluation: var_dtc.py:66-215 + sparse_gp.py:108-119 with every M x M product on the DMMA GEMM.
// All products are written as X Y^T (the kernel's native NT form) over column-major operands:
//   Lm, Um = Lm^-T from the factor-and-invert sweep of Kmm + 1e-8 I;  Lmi = Um^T
//   A = beta (Lmi G) Lmi^T;  B = I + A -> LB, UB;  Q = LBi Um^T (= LBi Lmi);  v = Q psi1Vf;  C = Q^T v;  w = UB v
//   B^-1 = UB UB^T;  DBi = P B^-1 + w w^T;  dL_dKmm = Um (..) Um^T;  dL_dpsi2 = beta/2 Um (P I - DBi) Um^T
// =================================================================================================================
static int mm_nt(gpx_ctx* c, const double* A, const double* B, double* C, int plain = 1) {
  const long Mpad = c->sparse->Mpad;
  GemmParams pg = gemm_defaults();
  pg.mode = GEMM_PANEL; pg.plain = plain;
  pg.A = A; pg.lda = Mpad; pg.B = B; pg.ldb = Mpad; pg.C = C; pg.ldc = Mpad;
  pg.K = (int)Mpad; pg.nt = (int)(Mpad / TILE); pg.ncols = (int)(Mpad / TILE);
  GPX_CHECK(launch_gemm(pg, dim3(1, 1), c->st));
  return launched(c);
}
static int combine(gpx_ctx* c, double* out, long n, double a, const double* X, double b, const double* Y, double cdiag,
                   double d = 0.0, const double* U = nullptr, int P = 0) {
  const long Mpad = c->sparse->Mpad;
  dim3 grid((unsigned)((n + 255) / 256), (unsigned)n);
  combine_kernel<<<grid, 256, 0, c->st>>>(out, Mpad, n, a, X, b, Y, cdiag, d, U, Mpad, P);
  return launched(c);
}
// out = Um E Um^T (T: scratch; out may be E)
static int sandwich(gpx_ctx* c, const double* Um, const double* E, double* T, double* out) {
  GPX_CHECK(mm_nt(c, Um, E, T));
  return mm_nt(c, T, Um, out);
}
// B^-1 = UB UB^T: lower tiles, mirrored
static int binv(gpx_ctx* c, const double* UB, double* out) {
  const long Mpad = c->sparse->Mpad;
  GPX_CHECK(mm_nt(c, UB, UB, out, 2));
  mirror_tiles_kernel<<<dim3((unsigned)((Mpad + 255) / 256), (unsigned)Mpad), 256, 0, c->st>>>(out, Mpad, Mpad);
  return launched(c);
}
// Kmm = K(Z, Z), dense and zero padded
static int build_Kmm(gpx_ctx* c, double* Kd) {
  SparseState* s = c->sparse;
  GPX_CUDA(cudaMemsetAsync(Kd, 0, (size_t)s->Mpad * s->Mpad * 8, c->st));
  GPX_CHECK(build_K(c, s->mk, s->D, s->zpts(), s->zpts(), Kd, s->Mpad));
  return launched(c);
}
// factor-and-invert the M x M matrix A (written on c's stream) on the child context ch, then U (clean upper) and
// Linv = U^T out of its factor; the child's launches count on c as well, its trailing updates in c's stats. jitchol's ladder
// with max_tries; *jitter_used (if given): what the ladder added beyond `jitter`
static int factor_child(gpx_ctx* c, gpx_ctx* ch, const double* A, double jitter, double* logdet, double* U, double* Linv,
                        double* jitter_used = nullptr, int max_tries = 5) {
  const long Mpad = c->sparse->Mpad;
  GPX_CUDA(cudaStreamSynchronize(c->st));
  const int64_t l0 = ch->total_launches;
  const int32_t u0 = ch->stats.update_launches;
  const int rc = factor_device(ch, A, Mpad, c->sparse->M, jitter, max_tries, logdet, jitter_used);
  c->total_launches += ch->total_launches - l0;
  c->stats.update_launches += ch->stats.update_launches - u0;
  if (rc) return rc;
  if (ch->Npad != Mpad) GPX_FAIL("internal: child workspace size");
  GPX_CHECK(launch_assemble(ch->S, Mpad, (int)Mpad, U, Mpad, Linv, ch->st));
  GPX_CHECK(launched(c));
  GPX_CUDA(cudaStreamSynchronize(ch->st));
  return 0;
}

// the checks every sparse entry makes before it reads its kernel (`kern`: the lengthscale or the parts, read against the
// data's D; het: per-point noise, dL_dR required)
static int sparse_args(const gpx_ctx* c, const void* kern, const double* Z, int64_t M, const double* lml, const double* grad,
                       const double* dZ, bool het, const double* dL_dR) {
  if (!c || !c->sparse || !c->sparse->X) GPX_FAIL("gpx_sparse_set_data has not been called");
  if (!Z || !lml || !grad || !dZ || !kern) GPX_FAIL("null argument");
  if (M < 1) GPX_FAIL("M must be positive");
  if (het && !dL_dR) GPX_FAIL("null argument");
  return 0;
}

// the kernel's gradient block: sum(dL_dKdiag) = ddiag through update_gradients_diag (sparse_gp.py:110), plus the Knm and
// Kmm reductions (:112-115). A composite's parts see ddiag times the product of the other variances of their term
// (prod.py:386-394, Kdiag = variance for every leaf kind); only the variance entry of a block depends on Kdiag.
static void kern_grads(const SparseState* s, double ddiag, const std::vector<double>& g_knm, const std::vector<double>& g_kmm,
                       double* grad) {
  const MultiKern& mk = s->mk;
  int g = 0;
  for (int p = 0; p < mk.nparts; p++) {
    double other = 1.0;
    for (int q = 0; q < mk.nparts; q++)
      if (q != p && mk.part[q].term == mk.part[p].term) other *= mk.part[q].variance;
    const int n = part_ngrad(mk.part[p]);
    for (int t = 0; t < n; t++) grad[g + t] = (t == 0 ? ddiag * other + g_knm[g] : g_knm[g + t]) + g_kmm[g + t];
    g += n;
  }
}

// uncertain inputs q(X) = N(X, diag(S)) of gpx_sparse_eval_psi: the lone RBF part, S on the host, dmu / dS out (host)
struct PsiCall {
  PsiParams pp;
  const double* S;
  double *dmu, *dS;
};

// One evaluation of the validated kernel k (Kdiag = kdiag, psi0 of every data point), which becomes the state's kernel.
// noise_vec == nullptr: scalar noise variance `noise` (grad = [k's gradient block, noise variance]);
// noise_vec (host, one variance per row held by this rank): grad = [k's gradient block], dL_dR (host, N x P row-major).
// k's block: a single kernel's [variance, lengthscale..]; a composite's part blocks in order (part_ngrad entries each).
// precision (host, one per row; sparse EP's marginal): the per-point form with beta_n = precision_n as given (no floor) and
// Kmm factored with jitchol's ladder (max_tries) and no const_jitter; *jitter_used: what the ladder added.
// psi (scalar noise only): the uncertain-input branches (var_dtc.py:107-123, sparse_gp.py:88-107): psi1 replaces Knm in
// Kfu, A_raw = Lm^-1 psi2 Lm^-T, and the psi gradient passes replace the Knm reductions.
static int sparse_eval_impl(gpx_ctx* c, const MultiKern& k, double kdiag, const double* Z, int64_t M, double noise,
                            const double* noise_vec, double* lml, double* grad, double* dZ, double* dL_dR_out,
                            const double* precision = nullptr, int max_tries = 5, double* jitter_used = nullptr,
                            const PsiCall* psi = nullptr) {
  const bool het = noise_vec != nullptr || precision != nullptr;
  GPX_CUDA(cudaSetDevice(c->device));
  SparseState* s = c->sparse;
  cudaStream_t st = c->st;
  s->have_eval = false;
  s->dl_ready = false;
  s->w_ready = false;
  s->mk = k;
  s->kdiag = kdiag;
  s->jitter = precision ? 0.0 : 1e-8;
  memset(&c->stats, 0, sizeof(c->stats));   // filled below: Kmm's attempts, the trailing updates of both factorisations
  // per-point precisions beta_n = 1 / max(variance_n, const_jitter) (var_dtc.py:79-84) and the sums over n the bound needs
  std::vector<double> hbeta, hsb;
  double sum_log_beta = 0.0, sum_beta = 0.0;
  if (het) {
    const long Nl = s->N, Npd = s->Npad;
    hbeta.assign((size_t)Npd, 0.0); hsb.assign((size_t)Npd, 0.0);
    for (long n = 0; n < Nl; n++) {
      if (precision ? !(precision[n] == precision[n]) : !(noise_vec[n] == noise_vec[n])) GPX_FAIL("noise variance is NaN");
      const double b = precision ? precision[n] : 1.0 / std::max(noise_vec[n], 1e-8);
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
  GPX_CHECK(psi_device(c, Z, M, psi == nullptr));
  const long Mpad = s->Mpad, N = s->Ntot, Npad = s->Npad;
  const int D = s->D, P = s->P, mt = (int)(Mpad / TILE);
  TmpBuf psiS(st), psiPre(st);
  PsiDev pd;
  if (psi) {   // psi1 (rbf_psi_comp.py:22-34) in Kfu, the layout every consumer of psi1 reads
    GPX_CHECK(psiS.alloc((size_t)s->N * D));
    GPX_CHECK(psiPre.alloc((size_t)s->N * (2 * D + 2)));
    GPX_CUDA(cudaMemcpyAsync(psiS.p, psi->S, (size_t)s->N * D * 8, cudaMemcpyHostToDevice, st));
    pd.mu = s->X; pd.S = psiS.p; pd.Z = s->Z; pd.pre = psiPre.p;
    GPX_CHECK(psi_prep(c, psi->pp, pd));
    GPX_CHECK(psi1_build(c, psi->pp, pd, s->Kfu, 1, Npad));
  }
  const int ngk = kern_ngrad(s->mk);   // entries of the kernel's gradient block
  constexpr int RSPLIT = 64;
  // P > MAX_P (scalar noise): every P-column product on the DMMA GEMM, the vectors held transposed as [Mpad][Ppad]
  const bool wide = P > MAX_P;
  const long Ppad = s->Ppad;
  if (!s->mm[0]) {
    for (auto& p : s->mm) GPX_CUDA(cudaMalloc(&p, (size_t)Mpad * Mpad * 8));
    if (wide) GPX_CUDA(cudaMalloc(&s->vec, (size_t)6 * Ppad * Mpad * 8));
    else GPX_CUDA(cudaMalloc(&s->vec, (size_t)(8 + RSPLIT) * P * Mpad * 8));
  }
  if (!s->red) {
    GPX_CUDA(cudaMalloc(&s->red, 4096 * 8));
    GPX_CUDA(cudaMallocHost(&s->h_red, 4096 * 8));
  }
  if (!s->cK) { GPX_CHECK(gpx_create(c->device, &s->cK)); GPX_CHECK(gpx_create(c->device, &s->cB)); }
  // the factorisations of Kmm and B run with the parent's option "nb" (a change re-sizes the child's workspace)
  for (gpx_ctx* ch : {s->cK, s->cB})
    if (ch->NB != c->NB) GPX_CHECK(gpx_set_option(ch, "nb", c->NB));
  double *Kd = s->mm[0], *Um = s->mm[1], *Lmi = s->mm[2], *T = s->mm[3], *Ar = s->mm[4], *Bd = s->mm[5], *UB = s->mm[6],
         *LBi = s->mm[7], *DB = s->mm[8], *E = s->mm[9];
  double *tv = s->vec, *vv = tv + (size_t)P * Mpad, *Cv = vv + (size_t)P * Mpad, *wv = Cv + (size_t)P * Mpad,
         *xv = wv + (size_t)P * Mpad, *rpart = s->vec + (size_t)8 * P * Mpad;
  // wide route: t^T, (beta t)^T, v^T, w^T, C^T ([Mpad][Ppad] each) and w ([Ppad][Mpad])
  double *tT = s->vec, *xT = tT + (size_t)Ppad * Mpad, *vT = xT + (size_t)Ppad * Mpad, *wT = vT + (size_t)Ppad * Mpad,
         *CT = wT + (size_t)Ppad * Mpad, *wq = CT + (size_t)Ppad * Mpad;
  // scalar noise: beta multiplies A, psi1Vf and dL_dpsi2 as a number; per-point noise: it is inside tmp, Y and the columns
  // of dL_dKnm^T already, and the same formulas run with beta = 1
  const double beta = het ? 1.0 : 1.0 / std::max(noise, 1e-8);                           // var_dtc.py:79-80
  s->noise = het ? 0.0 : noise;
  const double *sbv = het ? s->hb : nullptr, *bvec = het ? s->hb + Npad : nullptr;
  // Kmm (dense, zero padded), factor-and-invert with const_jitter (var_dtc.py:93-95)
  GPX_CHECK(build_Kmm(c, Kd));
  if (precision) {   // var_dtc.py:96-98 with Lm = jitchol(Kmm) of the caller: Kmm = Lm Lm^T
    double jit = 0.0;
    const int rc = factor_child(c, s->cK, Kd, 0.0, nullptr, Um, Lmi, &jit, max_tries);
    if (rc) return rc;
    s->jitter = jit;
    if (jitter_used) *jitter_used = jit;
  } else {
    GPX_CHECK(factor_child(c, s->cK, Kd, 1e-8, nullptr, Um, Lmi));                    // Um (clean upper), Lmi = Um^T
  }
  c->stats.tries = s->cK->stats.tries;
  // tmp = Lm^-1 psi1^T (M x N; var_dtc.py:131,139 dtrtrs) as a product with the triangular inverse, k-range <= row tile.
  // A = tmp tmp^T is then formed from O(1) entries. (Forming G = psi1^T psi1 first and sandwiching it, Lm^-1 G Lm^-T,
  // saves 2 M^2 N flops but cancels ~cond(Kmm) digits: measured 1e-4 instead of 1e-8 on dL/dZ at cond(Kmm) = 2e8.)
  double* Tuf = s->dLt;   // the dL_dKnm^T buffer is free until knm_grads_device
  GPX_CHECK(mul_psi1T(c, Lmi, Tuf, 2));
  const double* Yrow = s->Y;   // right-hand side of t = tmp Y
  if (het) {
    // s1_n = sum_a tmp[a, n]^2 (var_dtc.py:249, before the scaling); then tmp[:, n] *= sqrt(beta_n) (:127,131), Y_n likewise
    GPX_CHECK(launch_col_sqnorm(Tuf, Mpad, M, s->N, s->hs, st));
    GPX_CHECK(launched(c));
    scale_cols_kernel<<<(unsigned)((Mpad * s->N + 255) / 256), 256, 0, st>>>(Tuf, Mpad, s->N, sbv);
    GPX_CHECK(launched(c));
    ymul_kernel<<<(unsigned)((Npad * P + 255) / 256), 256, 0, st>>>(s->Y, sbv, Npad, P, s->Yb);
    GPX_CHECK(launched(c));
    Yrow = s->Yb;
  }
  if (psi) {   // A_raw = Lm^-1 psi2 Lm^-T (var_dtc.py:119-121), psi2 summed over the points into Bd (free until B)
    GPX_CHECK(psi2_build(c, psi->pp, pd, Bd, Mpad, Mpad));
    GPX_CHECK(sandwich(c, Lmi, Bd, T, Ar));
  } else {
    GemmParams pg = gemm_defaults();   // A_raw = tmp tmp^T (lower tiles), k-depth = Npad
    pg.mode = GEMM_PANEL; pg.plain = 2;
    pg.A = Tuf; pg.lda = Mpad; pg.B = Tuf; pg.ldb = Mpad; pg.C = Ar; pg.ldc = Mpad;
    pg.K = (int)Npad; pg.nt = mt; pg.ncols = mt;
    GPX_CHECK(launch_gemm(pg, dim3(1, 1), st));
    GPX_CHECK(launched(c));
  }
  if (wide) {
    GPX_CHECK(gemm_nt(c, s->YT, Ppad, Tuf, Mpad, tT, Ppad, Ppad, Mpad, Npad, 1, 0));     // t^T = Y^T tmp^T
    GPX_CUDA(cudaGetLastError());
  } else {
    GPX_CHECK(launch_row_dot(Tuf, Mpad, Mpad, s->N, P, Yrow, Npad, RSPLIT, rpart, tv, st));   // t = tmp Y  ([P][Mpad])
    GPX_CHECK(launched(c, 2));
  }
  // row shards: A_raw and t are sums over data points -> one M x M and one M x P all-reduce
  // (the pattern of var_dtc_parallel.py:113-131 with NCCL instead of mpi4py)
  GPX_CHECK(dist_allreduce_sum(c, Ar, (size_t)Mpad * Mpad, st));
  GPX_CHECK(dist_allreduce_sum(c, tv, (size_t)Mpad * P, st));
  {
    dim3 grid((unsigned)((Mpad + 255) / 256), (unsigned)Mpad);
    mirror_tiles_kernel<<<grid, 256, 0, st>>>(Ar, Mpad, Mpad);
    GPX_CHECK(launched(c));
  }
  // B = I + beta A_raw  (var_dtc.py:135-136)
  GPX_CHECK(combine(c, Bd, Mpad, beta, Ar, 0.0, nullptr, 1.0));
  double logdetB = 0.0;
  GPX_CHECK(factor_child(c, s->cB, Bd, 0.0, &logdetB, UB, LBi));
  // v = LB^-1 (beta t) (:139-141) ; w = LB^-T v ; C = Lm^-T w (:142-143)   [col_dot(A, y) = A^T y]
  if (wide) {   // transposed: v^T = x^T LBi^T, w^T = v^T LBi, C^T = w^T Lmi; GEMM operand B(j, k) = LBi(j, k), UB(j, k), Um(j, k)
    scale_kernel<<<(unsigned)((Mpad * Ppad + 255) / 256), 256, 0, st>>>(tT, beta, Mpad * Ppad, xT);
    GPX_CHECK(launched(c));
    GPX_CHECK(gemm_nt(c, xT, Ppad, LBi, Mpad, vT, Ppad, Ppad, Mpad, Mpad, 1, 1));
    GPX_CHECK(gemm_nt(c, vT, Ppad, UB, Mpad, wT, Ppad, Ppad, Mpad, Mpad, 1, 0));
    GPX_CHECK(gemm_nt(c, wT, Ppad, Um, Mpad, CT, Ppad, Ppad, Mpad, Mpad, 1, 0));
    GPX_CUDA(cudaGetLastError());
  } else {
    scale_kernel<<<(unsigned)((Mpad * P + 255) / 256), 256, 0, st>>>(tv, beta, Mpad * P, xv);
    GPX_CHECK(launched(c));
    GPX_CHECK(launch_col_dot(UB, Mpad, Mpad, Mpad, P, xv, Mpad, vv, Mpad, st));           // v = UB^T x = LBi x
    GPX_CHECK(launch_col_dot(LBi, Mpad, Mpad, Mpad, P, vv, Mpad, wv, Mpad, st));          // w = LBi^T v
    GPX_CHECK(launch_col_dot(Lmi, Mpad, Mpad, Mpad, P, wv, Mpad, Cv, Mpad, st));          // C = Lmi^T w
    GPX_CHECK(launched(c, 3));
  }
  std::vector<double> hstat, hY;
  if (het) {
    // _compute_dL_dR, het_noise (var_dtc.py:241-257): per data point
    //   r_np = (v_p^T LB^-1 Lm^-1 psi1^T)_n = w_p . tmp[:, n]     (here from the scaled tmp: r_np sqrt(beta_n))
    //   s2_n = |LB^-1 Lm^-1 psi1^T[:, n]|^2 = |(Q psi1^T)[:, n]|^2,  Q = LB^-1 Lm^-1 (lower triangular)
    double *s2v = s->hs + Npad, *rv = s->hs + 2 * Npad;
    GPX_CHECK(launch_col_dot(Tuf, Mpad, M, s->N, P, wv, Mpad, rv, Npad, st));
    GPX_CHECK(launched(c));
    GPX_CHECK(mm_nt(c, LBi, Um, T));                                                      // Q = LBi Um^T = LBi Lmi
    GPX_CHECK(mul_psi1T(c, T, s->dLt, 2));
    GPX_CHECK(launch_col_sqnorm(s->dLt, Mpad, M, s->N, s2v, st));
    GPX_CHECK(launched(c));
    hstat.resize((size_t)(2 + P) * Npad);
    hY.resize((size_t)P * Npad);
    GPX_CUDA(cudaMemcpyAsync(hstat.data(), s->hs, hstat.size() * 8, cudaMemcpyDeviceToHost, st));
    GPX_CUDA(cudaMemcpyAsync(hY.data(), s->Y, hY.size() * 8, cudaMemcpyDeviceToHost, st));
  }
  // DBi = P B^-1 + w w^T
  GPX_CHECK(binv(c, UB, DB));
  if (wide) {   // w w^T with k-depth Ppad: lower tiles, mirrored (T is free), then added
    GPX_CHECK(launch_transpose_pad(wT, Mpad, (int)Ppad, Mpad, wq, st));
    GPX_CHECK(launched(c));
    GPX_CHECK(gemm_nt(c, wq, Mpad, wq, Mpad, T, Mpad, Mpad, Mpad, Ppad, 2, 0));
    mirror_tiles_kernel<<<dim3((unsigned)((Mpad + 255) / 256), (unsigned)Mpad), 256, 0, st>>>(T, Mpad, Mpad);
    GPX_CHECK(launched(c));
    GPX_CHECK(combine(c, DB, Mpad, (double)P, DB, 1.0, T, 0.0));
  } else {
    GPX_CHECK(combine(c, DB, Mpad, (double)P, DB, 0.0, nullptr, 0.0, 1.0, wv, P));
  }
  // scalars: trace(A_raw), sum(A_raw .* DBi), |v|^2
  const int RB = 64;
  trace_dot_kernel<<<RB, 256, 0, st>>>(Ar, DB, Mpad, M, s->red);
  GPX_CHECK(launched(c));
  GPX_CUDA(cudaMemcpyAsync(s->h_red, s->red, 2 * RB * 8, cudaMemcpyDeviceToHost, st));
  std::vector<double> hv(wide ? (size_t)RB : (size_t)P * Mpad);
  if (wide) {   // |v|^2 over v^T, whose padding is zero: RB partial sums
    sumsq_kernel<<<RB, 256, 0, st>>>(vT, Mpad * Ppad, s->red + 2 * RB);
    GPX_CHECK(launched(c));
    GPX_CUDA(cudaMemcpyAsync(hv.data(), s->red + 2 * RB, RB * 8, cudaMemcpyDeviceToHost, st));
  } else {
    GPX_CUDA(cudaMemcpyAsync(hv.data(), vv, hv.size() * 8, cudaMemcpyDeviceToHost, st));
  }
  // dL_dKmm = Um (-0.5 DBi - 0.5 P B + P I) Um^T   (var_dtc.py:152-156)
  GPX_CHECK(combine(c, E, Mpad, -0.5, DB, -0.5 * P, Bd, (double)P));
  GPX_CHECK(sandwich(c, Um, E, T, Kd));                                                   // Kd now holds dL_dKmm
  // W2 = 2 dL_dpsi2 = beta Um (P I - DBi) Um^T     (var_dtc.py:221,231-233)
  GPX_CHECK(combine(c, E, Mpad, -1.0, DB, 0.0, nullptr, (double)P));
  GPX_CHECK(sandwich(c, Um, E, T, E));
  GPX_CHECK(combine(c, s->W2, Mpad, beta, E, 0.0, nullptr, 0.0));
  // Knm part: needs C in s->Cm (wide route: and as [Ppad][Mpad] in the columns of W2 after W2)
  if (wide) {
    double* Cext = s->W2 + (size_t)Mpad * Mpad;
    GPX_CHECK(launch_transpose_pad(CT, Mpad, (int)Ppad, Mpad, Cext, st));
    GPX_CHECK(launched(c));
    GPX_CUDA(cudaMemcpyAsync(s->Cm, Cext, (size_t)P * Mpad * 8, cudaMemcpyDeviceToDevice, st));
  } else {
    GPX_CUDA(cudaMemcpyAsync(s->Cm, Cv, (size_t)P * Mpad * 8, cudaMemcpyDeviceToDevice, st));
  }
  std::vector<double> g_knm(ngk, 0.0);
  if (psi) {   // dL_dpsi1 = beta Y C^T, dL_dpsi2 = beta dL_dpsi2_beta (var_dtc.py:218-229) -> the psi gradient passes
    dl_dpsi1_kernel<<<dim3((unsigned)((s->N + 255) / 256), (unsigned)M), 256, 0, st>>>(s->Y, Npad, s->Cm, Mpad, P, beta,
                                                                                       s->N, s->dLt, Npad);
    GPX_CHECK(launched(c));
    GPX_CHECK(combine(c, E, Mpad, 0.5 * beta, E, 0.0, nullptr, 0.0));
    GPX_CHECK(psi_grads(c, psi->pp, pd, s->Kfu, s->dLt, 1, Npad, E, Mpad, g_knm.data(), dZ, psi->dmu, psi->dS));
  } else {
    GPX_CHECK(knm_grads_device(c, beta, bvec, g_knm.data(), dZ));                       // dZ <- Knm part
  }
  {
    int rank = 0, G = 1;
    dist_world(c, &rank, &G);
    if (G > 1) {   // sums over this rank's data points -> totals
      std::vector<double> h((size_t)ngk + (size_t)M * D);
      memcpy(h.data(), g_knm.data(), (size_t)ngk * 8);
      memcpy(h.data() + ngk, dZ, (size_t)M * D * 8);
      GPX_CUDA(cudaMemcpyAsync(s->gsum, h.data(), h.size() * 8, cudaMemcpyHostToDevice, st));
      GPX_CHECK(dist_allreduce_sum(c, s->gsum, h.size(), st));
      GPX_CUDA(cudaMemcpyAsync(h.data(), s->gsum, h.size() * 8, cudaMemcpyDeviceToHost, st));
      GPX_CUDA(cudaStreamSynchronize(st));
      memcpy(g_knm.data(), h.data(), (size_t)ngk * 8);
      memcpy(dZ, h.data() + ngk, (size_t)M * D * 8);
    }
  }
  // Kmm part: kern.update_gradients_full(dL_dKmm, Z) and kern.gradients_X(dL_dKmm, Z)  (sparse_gp.py:114,117)
  const GradFullParams gk = grad_params(s->mk, D, s->zpts(), s->zpts(), Kd, Mpad);
  std::vector<double> g_kmm(ngk, 0.0), hz((size_t)M * D);
  GPX_CHECK(ensure_part(s, grad_full_doubles(s->mk, D, gk) * 8));
  GPX_CHECK(grad_full_sum(c, s->mk, D, gk, s->part, g_kmm.data()));
  GPX_CHECK(ensure_part(s, grad_X_doubles(c, s->mk, gk, D) * 8));
  GPX_CHECK(grad_X(c, s->mk, gk, D, s->part, hz.data()));
  for (size_t i = 0; i < hz.size(); i++) dZ[i] += hz[i];
  // ---- scalars on the host (var_dtc.py:237-276, homoscedastic) -----------------------------------------------------
  double trAr = 0.0, sumAD = 0.0, data_fit = 0.0;
  for (int b = 0; b < RB; b++) { trAr += s->h_red[2 * b]; sumAD += s->h_red[2 * b + 1]; }
  if (wide)
    for (int b = 0; b < RB; b++) data_fit += hv[b];
  else
    for (int q = 0; q < P; q++)
      for (long i = 0; i < M; i++) data_fit += hv[(size_t)q * Mpad + i] * hv[(size_t)q * Mpad + i];
  const double trA = beta * trAr, sumADB = beta * sumAD;
  const double variance = s->kdiag;                                                           // psi0 per point
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
    kern_grads(s, -0.5 * od * sums[1], g_knm, g_kmm, grad);                                 // update_gradients_diag (:110)
    s->have_eval = true;
    s->dl_ready = !precision;
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
  kern_grads(s, dvar_diag, g_knm, g_kmm, grad);
  grad[ngk] = dL_dR;
  s->have_eval = true;
  s->dl_ready = !precision && !psi;
  return 0;
}

extern "C" {

int gpx_sparse_eval(gpx_ctx* c, int kind, int ard, double variance, const double* lengthscale, const double* Z, int64_t M,
                    double noise, double* lml, double* grad, double* dZ) {
  GPX_CHECK(sparse_args(c, lengthscale, Z, M, lml, grad, dZ, false, nullptr));
  MultiKern mk;
  GPX_CHECK(fill_single(mk, kind, ard, c->sparse->D, variance, lengthscale));
  return sparse_eval_impl(c, mk, variance, Z, M, noise, nullptr, lml, grad, dZ, nullptr);
}

int gpx_sparse_eval_het(gpx_ctx* c, int kind, int ard, double variance, const double* lengthscale, const double* Z,
                        int64_t M, const double* noise_variances, double* lml, double* grad, double* dZ, double* dL_dR) {
  if (!noise_variances) GPX_FAIL("null argument");
  GPX_CHECK(sparse_args(c, lengthscale, Z, M, lml, grad, dZ, true, dL_dR));
  if (c->sparse->P > MAX_P) GPX_FAIL("the heteroscedastic sparse evaluation serves at most 8 output columns");
  MultiKern mk;
  GPX_CHECK(fill_single(mk, kind, ard, c->sparse->D, variance, lengthscale));
  return sparse_eval_impl(c, mk, variance, Z, M, 0.0, noise_variances, lml, grad, dZ, dL_dR);
}

int gpx_sparse_eval_multi(gpx_ctx* c, const gpx_kern_part* parts, int nparts, const double* Z, int64_t M,
                          double noise_variance, const double* noise_variances, double* lml, double* grad, double* dZ,
                          double* dL_dR) {
  const bool het = noise_variances != nullptr;
  GPX_CHECK(sparse_args(c, parts, Z, M, lml, grad, dZ, het, dL_dR));
  if (c->dist) GPX_FAIL("composite kernels are single-GPU");
  if (het && c->sparse->P > MAX_P) GPX_FAIL("the heteroscedastic sparse evaluation serves at most 8 output columns");
  MultiKern mk;
  double kdiag;
  GPX_CHECK(fill_mk(mk, parts, nparts, c->sparse->D, &kdiag));
  for (int p = 0; p < mk.nparts; p++)   // dL/dZ needs every part's gradients_X
    if (mk.part[p].kind == GPX_RATQUAD || mk.part[p].kind == GPX_STDPERIODIC)
      GPX_FAIL("RatQuad and StdPeriodic parts are not on the sparse evaluation (no device gradients_X)");
  return sparse_eval_impl(c, mk, kdiag, Z, M, het ? 0.0 : noise_variance, noise_variances, lml, grad, dZ, dL_dR);
}

int gpx_sparse_eval_psi(gpx_ctx* c, const gpx_kern_part* parts, int nparts, const double* S, const double* Z, int64_t M,
                        double noise_variance, double* lml, double* grad, double* dZ, double* dmu, double* dS) {
  GPX_CHECK(sparse_args(c, parts, Z, M, lml, grad, dZ, false, nullptr));
  if (!S || !dmu || !dS) GPX_FAIL("null argument");
  if (c->dist) GPX_FAIL("the uncertain-input evaluation is single-GPU");
  SparseState* s = c->sparse;
  PsiCall pc{};
  GPX_CHECK(psi_params(parts, nparts, s->D, &pc.pp));
  GPX_CHECK(psi_check_S(S, s->N, s->D));
  pc.pp.N = s->N; pc.pp.M = M;
  pc.S = S; pc.dmu = dmu; pc.dS = dS;
  MultiKern mk;
  double kdiag;
  GPX_CHECK(fill_mk(mk, parts, nparts, s->D, &kdiag));
  return sparse_eval_impl(c, mk, kdiag, Z, M, noise_variance, nullptr, lml, grad, dZ, nullptr, nullptr, 5, nullptr, &pc);
}

/* which: 0 woodbury_vector (M x P row-major), 1 woodbury_inv (M x M), 2 Kmm (+ the evaluation's const_jitter I: 1e-8
 * VarDTC, 1e-6 FITC), 3 Lm (lower, col-major) */
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
  if (which == 1 && s->w_own) {   // SVGP: Kmm^-1 - Kmm^-1 S Kmm^-1, formed by gpx_svgp_finish
    src = s->mm[9];
  } else if (which == 1) {   // woodbury_inv = Um (I - B^-1) Um^T   (var_dtc.py:207-210); B^-1 is rebuilt from UB
    double *Um = s->mm[1], *UB = s->mm[6], *T = s->mm[3], *E = s->mm[9], *DB = s->mm[8];
    GPX_CHECK(binv(c, UB, DB));
    GPX_CHECK(combine(c, E, Mpad, -1.0, DB, 0.0, nullptr, 1.0));
    GPX_CHECK(sandwich(c, Um, E, T, E));
    src = E;
  } else if (which == 2) {   // Kmm, rebuilt by the kernel build, + const_jitter
    src = s->mm[3];
    GPX_CHECK(build_Kmm(c, src));
    GPX_CHECK(combine(c, src, M, 1.0, src, 0.0, nullptr, s->jitter));
  } else if (which == 3) {   // Lm, extracted from the child context's factor
    src = s->mm[3];
    GPX_CUDA(cudaStreamSynchronize(st));
    GPX_CHECK(launch_extract(GPX_GET_L, s->cK->S, Mpad, s->cK->Ldiag, nullptr, nullptr, 0, Mpad, src, s->cK->st));
    GPX_CHECK(launched(c));
    GPX_CUDA(cudaStreamSynchronize(s->cK->st));
  } else {
    GPX_FAIL("unknown gpx_sparse_get selector");
  }
  GPX_CUDA(cudaMemcpy2DAsync(out, M * 8, src, Mpad * 8, (size_t)M * 8, M, cudaMemcpyDeviceToHost, st));
  GPX_CUDA(cudaStreamSynchronize(st));
  return 0;
}

}  // extern "C"

// woodbury_inv W of the current evaluation in mm[9], formed as gpx_sparse_get(1) forms it by the first caller after an
// evaluation (predictive gradients, samples or predict) and kept for the later ones: gpx_sparse_get(1) writes the same W
// into mm[9], nothing else writes it
static int woodbury_inv(gpx_ctx* c, double** W) {
  SparseState* s = c->sparse;
  double *Um = s->mm[1], *UB = s->mm[6], *T = s->mm[3], *DB = s->mm[8];
  *W = s->mm[9];
  if (!s->w_ready) {
    GPX_CHECK(binv(c, UB, DB));
    GPX_CHECK(combine(c, *W, s->Mpad, -1.0, DB, 0.0, nullptr, 1.0));
    GPX_CHECK(sandwich(c, Um, *W, T, *W));
    s->w_ready = true;
  }
  return 0;
}

extern "C" {

/* predictive gradients of the last sparse evaluation (gp.py:438-474 with the predictive variable Z, sparse_gp.py:52-54):
 * woodbury_inv W as gpx_sparse_get(1) forms it, into the same scratch and once per evaluation (an optimiser asks for one
 * batch after another on the same posterior), then V = W K(Z, Xnew) on the DMMA GEMM and one fused Jacobian reduction */
int gpx_sparse_predictive_gradients(gpx_ctx* c, const double* Xnew, int64_t Mn, double* dmu, double* dvar) {
  if (!c || !Xnew || !dmu || !dvar) GPX_FAIL("null argument");
  if (!c->sparse || !c->sparse->have_eval) GPX_FAIL("no sparse evaluation to differentiate the prediction of");
  if (Mn < 1) GPX_FAIL("empty Xnew");
  if (c->dist) GPX_FAIL("predictive gradients are single-GPU");
  if (c->sparse->P > MAX_P) GPX_FAIL("predictive gradients serve at most 8 output columns");
  SparseState* s = c->sparse;
  const MultiKern& k = s->mk;
  GPX_CHECK(pred_grad_check(k));
  GPX_CUDA(cudaSetDevice(c->device));
  cudaStream_t st = c->st;
  const long Mpad = s->Mpad;
  PointSet pn;
  GPX_CHECK(upload_points(c, k, Xnew, Mn, s->D, pn));
  double* W = nullptr;
  GPX_CHECK(woodbury_inv(c, &W));
  // K(Xnew, Z) with element (m, a) at m + a * pn.ld (the GEMM's B operand, zero padded), V (Mpad x pn.ld) = W K(Xnew, Z)^T
  double *Kxz = nullptr, *V = nullptr;
  GPX_TMP_ALLOC(&Kxz, (size_t)pn.ld * Mpad * 8, st);
  GPX_TMP_ALLOC(&V, (size_t)Mpad * pn.ld * 8, st);
  int rc = 0;
  if (cudaMemsetAsync(Kxz, 0, (size_t)pn.ld * Mpad * 8, st) != cudaSuccess) { gpx::set_error("gpx_sparse_predictive_gradients: device failure"); rc = -1; }
  if (rc == 0) rc = build_K(c, k, s->D, pn, s->zpts(), Kxz, pn.ld);
  if (rc == 0) rc = launched(c);
  if (rc == 0) {
    GemmParams pg = gemm_defaults();
    pg.mode = GEMM_PANEL; pg.plain = 1;
    pg.A = W; pg.lda = Mpad; pg.B = Kxz; pg.ldb = pn.ld; pg.C = V; pg.ldc = Mpad;
    pg.K = (int)Mpad; pg.nt = (int)(Mpad / TILE); pg.ncols = (int)(pn.ld / TILE);
    rc = launch_gemm(pg, dim3(1, 1), st);
    if (rc == 0) rc = launched(c);
  }
  if (rc == 0) rc = pred_grad(c, k, pn, s->zpts(), s->Cm, Mpad, s->P, V, Mpad, s->D, dmu, dvar);
  GPX_TMP_FREE(Kxz, st); GPX_TMP_FREE(V, st);
  return rc;
}

}  // extern "C"

// mu ([P][L]) = K(Xnew, Z) woodbury_vector for the L padded rows of Kxz (column-major, leading dimension L): MAX_P outputs
// per launch_row_dot; part holds RSPLIT min(P, MAX_P) L doubles
constexpr int MEAN_RSPLIT = 64;
static int sparse_mean(gpx_ctx* c, const double* Kxz, long L, double* part, double* mu) {
  SparseState* s = c->sparse;
  for (int q0 = 0; q0 < s->P; q0 += MAX_P) {
    const int pc = std::min(MAX_P, s->P - q0);
    GPX_CHECK(launch_row_dot(Kxz, L, L, s->M, pc, s->Cm + (size_t)q0 * s->Mpad, s->Mpad, MEAN_RSPLIT, part,
                             mu + (size_t)q0 * L, c->st));
    GPX_CHECK(launched(c, 2));
  }
  return 0;
}

// The latent predictive covariance and mean of the last sparse evaluation at the prepared test points pn (posterior.py:
// 220-238 with pred_var = Z): Sigma = K(Xnew) - K(Xnew, Z) W K(Z, Xnew) into Kss (pn.ld^2, column-major, exactly
// symmetric: the lower tiles of the product term mirrored), mu = K(Xnew, Z) woodbury_vector into mu ([P][pn.ld]).
// V^T = K(Xnew, Z) W and V^T K(Z, Xnew) run on the DMMA GEMM. Launches: 7, plus 5 when it forms W.
static int sparse_joint(gpx_ctx* c, const PointSet& pn, TmpBuf& Kss, TmpBuf& mu) {
  SparseState* s = c->sparse;
  cudaStream_t st = c->st;
  const long Mpad = s->Mpad, L = pn.ld;
  double* W = nullptr;
  GPX_CHECK(woodbury_inv(c, &W));
  TmpBuf Kxz(st), Vt(st), prod(st), part(st);
  GPX_CHECK(Kxz.alloc((size_t)L * Mpad));
  GPX_CHECK(Vt.alloc((size_t)L * Mpad));
  GPX_CHECK(prod.alloc((size_t)L * L));
  GPX_CHECK(Kss.alloc((size_t)L * L));
  GPX_CHECK(mu.alloc((size_t)s->P * L));
  GPX_CHECK(part.alloc((size_t)MEAN_RSPLIT * std::min(s->P, MAX_P) * L));
  // K(Xnew, Z) with element (m, a) at m + a * L: test points thread-mapped, zero padded
  GPX_CUDA(cudaMemsetAsync(Kxz.p, 0, (size_t)L * Mpad * 8, st));
  GPX_CHECK(build_K(c, s->mk, s->D, pn, s->zpts(), Kxz.p, L));
  GPX_CHECK(launched(c));
  GPX_CHECK(gemm_nt(c, Kxz.p, L, W, Mpad, Vt.p, L, L, Mpad, Mpad, 1, 0));          // V^T = K(Xnew, Z) W (W symmetric)
  GPX_CHECK(gemm_nt(c, Vt.p, L, Kxz.p, L, prod.p, L, L, L, Mpad, 2, 0));           // V^T K(Z, Xnew), lower tiles
  GPX_CHECK(sparse_mean(c, Kxz.p, L, part.p, mu.p));                                // mu = K(Xnew, Z) wv
  GPX_CHECK(build_K(c, s->mk, s->D, pn, pn, Kss.p, L));
  GPX_CHECK(launched(c));
  return joint_combine(c, Kss.p, L, 0, prod.p, L, 1, pn.n, pn.n, Kss.p, L, 1);    // Sigma in place of K(Xnew)
}

// var[m] = max(kdiag - sum_{a < M} Vt(m, a) Kxz(m, a), 1e-15) for the n rows of one chunk (posterior.py:244-248: the
// reference's rowsum((K(Xnew, Z) W) o K(Xnew, Z)) and its clip; a NaN stays NaN as under np.clip). Both operands are
// column-major with leading dimension ld. A row's sum depends on M alone: 8 column slices of ceil(M / 8), each summed in
// column order by one thread, then added in slice order, so a row gets the same bits in any chunk at any position.
constexpr int VAR_ROWS = 32, VAR_SLICES = 8;
__global__ void __launch_bounds__(VAR_ROWS * VAR_SLICES) sparse_var_kernel(const double* __restrict__ Kxz,
                                                                           const double* __restrict__ Vt, long ld, long n,
                                                                           long M, double kdiag, double* __restrict__ var) {
  __shared__ double sh[VAR_SLICES][VAR_ROWS];
  const long row = (long)blockIdx.x * VAR_ROWS + threadIdx.x;
  const long chunk = (M + VAR_SLICES - 1) / VAR_SLICES, a0 = threadIdx.y * chunk;
  const long a1 = a0 + chunk < M ? a0 + chunk : M;
  double acc = 0.0;
  if (row < n)
    for (long a = a0; a < a1; a++) acc = fma(Vt[row + a * ld], Kxz[row + a * ld], acc);
  sh[threadIdx.y][threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.y != 0 || row >= n) return;
  double sum = sh[0][threadIdx.x];
#pragma unroll
  for (int q = 1; q < VAR_SLICES; q++) sum += sh[q][threadIdx.x];
  const double v = kdiag - sum;
  var[row] = v < 1e-15 ? 1e-15 : v;
}

namespace {
// rows of one chunk of the diagonal prediction: the largest multiple of 128 whose temporaries, bounded by
// 16 Mpad + 512 min(P, 8) + 8 P + 1096 bytes per row (K(Xc, Z) and V^T, the mean's 64 partial sums of one slab of at most
// 8 outputs, mean and variance, the uploaded and prepared points at D, stacked dims and norms <= 64), fit in the 1 GiB the
// stream-ordered pool keeps cached (gpx_create); never fewer than 128, never more than the test points padded to 128
// (include/gpx.h states the same rule)
long predict_chunk_rows(long Mpad, int P, long Mn) {
  const long per_row = 16 * Mpad + 512 * (long)std::min(P, MAX_P) + 8 * (long)P + 1096;
  const long Lc = std::max<long>(TILE, (1l << 30) / per_row / TILE * TILE);
  return std::min<long>(Lc, (Mn + TILE - 1) / TILE * TILE);
}
}  // namespace

extern "C" {

/* joint samples of the latent function from the last sparse evaluation (posterior.py:238-270 with pred_var = Z, then
 * gp.py:601-629): Sigma and mu from sparse_joint (W = woodbury_inv shared with the predictive gradients and predict) */
int gpx_sparse_posterior_samples(gpx_ctx* c, const double* Xnew, int64_t Mn, const double* z, int64_t nz, int max_tries,
                                 double* f, double* jitter_used) {
  if (!c) GPX_FAIL("null argument");
  if (!c->sparse || !c->sparse->have_eval) GPX_FAIL("no sparse evaluation to take the posterior from");
  if (c->sparse->P > MAX_P) GPX_FAIL("the joint posterior serves at most 8 output columns");
  SparseState* s = c->sparse;
  GPX_CHECK(joint_check(c, Xnew, Mn, z, nz, f, jitter_used, s->P));
  GPX_CUDA(cudaSetDevice(c->device));
  PointSet pn;
  GPX_CHECK(upload_points(c, s->mk, Xnew, Mn, s->D, pn));
  TmpBuf Kss(c->st), mu(c->st);
  GPX_CHECK(sparse_joint(c, pn, Kss, mu));
  return joint_sample(c, Kss.p, pn.ld, Mn, mu.p, pn.ld, z, nz, nz / s->P, max_tries, f, jitter_used);
}

/* SparseGP.predict's latent part (GPy/core/gp.py:303 -> posterior.py:220-248 with pred_var = Z): mu = K(Xnew, Z)
 * woodbury_vector, and the diagonal variance (clipped at 1e-15), streamed over chunks of test points, or the full covariance
 * in one pass. Every rank of a communicator holds the same posterior and predicts the points it is given, alone. */
int gpx_sparse_predict(gpx_ctx* c, const double* Xnew, int64_t Mn, int full_cov, double* mu, double* var) {
  if (!c || !Xnew || !mu || !var) GPX_FAIL("null argument");
  if (!c->sparse || !c->sparse->have_eval) GPX_FAIL("no sparse evaluation to predict from");
  if (Mn < 1) GPX_FAIL("empty Xnew");
  SparseState* s = c->sparse;
  const MultiKern& k = s->mk;
  const int P = s->P;
  GPX_CUDA(cudaSetDevice(c->device));
  cudaStream_t st = c->st;
  if (full_cov) {
    PointSet pn;
    GPX_CHECK(upload_points(c, k, Xnew, Mn, s->D, pn));
    TmpBuf Kss(st), mud(st);
    GPX_CHECK(sparse_joint(c, pn, Kss, mud));
    const long L = pn.ld;
    std::vector<double> h((size_t)P * L);
    GPX_CUDA(cudaMemcpyAsync(h.data(), mud.p, h.size() * 8, cudaMemcpyDeviceToHost, st));
    GPX_CUDA(cudaMemcpy2DAsync(var, Mn * 8, Kss.p, L * 8, (size_t)Mn * 8, Mn, cudaMemcpyDeviceToHost, st));
    if (cudaStreamSynchronize(st) != cudaSuccess) GPX_FAIL_DEVICE("gpx_sparse_predict");
    for (long m = 0; m < Mn; m++)
      for (int q = 0; q < P; q++) mu[m * P + q] = h[(size_t)q * L + m];
    return 0;
  }
  const long Mpad = s->Mpad, Lc = predict_chunk_rows(Mpad, P, Mn);
  double* W = nullptr;
  GPX_CHECK(woodbury_inv(c, &W));
  TmpBuf Kxz(st), Vt(st), part(st), red(st);   // red: [P][Lc] means, then [Lc] variances
  GPX_CHECK(Kxz.alloc((size_t)Lc * Mpad));
  GPX_CHECK(Vt.alloc((size_t)Lc * Mpad));
  GPX_CHECK(part.alloc((size_t)MEAN_RSPLIT * std::min(P, MAX_P) * Lc));
  GPX_CHECK(red.alloc((size_t)(P + 1) * Lc));
  std::vector<double> h((size_t)P * Lc);
  for (long m0 = 0; m0 < Mn; m0 += Lc) {
    const long n = std::min<long>(Lc, Mn - m0);
    PointSet pn;
    GPX_CHECK(upload_points(c, k, Xnew + (size_t)m0 * s->D, n, s->D, pn));
    const long L = pn.ld;   // this chunk's rows padded to 128 (<= Lc)
    // K(Xc, Z) with element (m, a) at m + a * L, zero padded; V^T = K(Xc, Z) W
    GPX_CUDA(cudaMemsetAsync(Kxz.p, 0, (size_t)L * Mpad * 8, st));
    GPX_CHECK(build_K(c, k, s->D, pn, s->zpts(), Kxz.p, L));
    GPX_CHECK(launched(c));
    GPX_CHECK(gemm_nt(c, Kxz.p, L, W, Mpad, Vt.p, L, L, Mpad, Mpad, 1, 0));
    GPX_CHECK(sparse_mean(c, Kxz.p, L, part.p, red.p));                                   // mu ([P][L])
    double* vd = red.p + (size_t)P * L;
    sparse_var_kernel<<<(unsigned)(L / VAR_ROWS), dim3(VAR_ROWS, VAR_SLICES), 0, st>>>(Kxz.p, Vt.p, L, n, s->M, s->kdiag,
                                                                                       vd);
    GPX_CHECK(launched(c));
    GPX_CUDA(cudaMemcpyAsync(h.data(), red.p, (size_t)P * L * 8, cudaMemcpyDeviceToHost, st));
    GPX_CUDA(cudaMemcpyAsync(var + m0, vd, (size_t)n * 8, cudaMemcpyDeviceToHost, st));
    if (cudaStreamSynchronize(st) != cudaSuccess) GPX_FAIL_DEVICE("gpx_sparse_predict");
    for (long m = 0; m < n; m++)
      for (int q = 0; q < P; q++) mu[(m0 + m) * P + q] = h[(size_t)q * L + m];
  }
  return 0;
}

}  // extern "C"

// =================================================================================================================
// FITC (fitc.py:19-88, Snelson & Ghahramani's SPGP) with the gradient wiring of sparse_gp.py:108-118: the per-point-noise
// VarDTC pipeline with the effective noise sigma*_n = Kdiag + sigma^2 - s1_n (s1_n = |Lm^-1 psi1_n^T|^2) formed on the
// device, no trace term, and the chain rule through sigma* in the gradients. The posterior has VarDTC's form
// (woodbury_inv = Um (I - B^-1) Um^T, woodbury_vector = v = Lm^-T LB^-T b), so the sparse predict, predictive gradients and
// samples serve it unchanged. Every N M^2 product runs on the DMMA GEMM; the per-point work is three kernels below, each
// with a fixed reduction order.
// =================================================================================================================
namespace {
constexpr int FITC_RED_BLOCKS = 256;   // partial sums of the bound: one pair per CTA, added on the host in CTA order
// n < N: sigma*_n = kdiag + noise - s1_n (fitc.py:43), beta*_n = 1 / sigma*_n (no floor, :44), sqrt(beta*_n), Yb_n =
// sqrt(beta*_n) y_n and the CTA's partial sums of log(beta*_n) and beta*_n y_n^2 (:60-64); the padding columns get
// beta* = 0. bad: the first n with sigma*_n <= 0 or NaN (atomicMin: the same index whatever the schedule)
__global__ void __launch_bounds__(256) fitc_beta_kernel(const double* __restrict__ s1, long N, long Npad, double kdiag,
                                                        double noise, const double* __restrict__ Y, double* __restrict__ sb,
                                                        double* __restrict__ b, double* __restrict__ Yb,
                                                        double* __restrict__ part, int* __restrict__ bad) {
  __shared__ double sh[2][256];
  double slog = 0.0, sby2 = 0.0;
  for (long n = (long)blockIdx.x * 256 + threadIdx.x; n < Npad; n += (long)gridDim.x * 256) {
    if (n >= N) { sb[n] = 0.0; b[n] = 0.0; Yb[n] = 0.0; continue; }
    const double sig = kdiag + noise - s1[n];
    if (!(sig > 0.0)) atomicMin(bad, (int)n);
    const double be = 1.0 / sig, y = Y[n];
    sb[n] = sqrt(be); b[n] = be; Yb[n] = sqrt(be) * y;
    slog += log(be);
    sby2 += be * y * y;
  }
  sh[0][threadIdx.x] = slog; sh[1][threadIdx.x] = sby2;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) { sh[0][threadIdx.x] += sh[0][threadIdx.x + o]; sh[1][threadIdx.x] += sh[1][threadIdx.x + o]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) { part[2 * blockIdx.x] = sh[0][0]; part[2 * blockIdx.x + 1] = sh[1][0]; }
}
__device__ __forceinline__ double fitc_warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// one warp per column n (8 per CTA), lanes over the M rows in a fixed order: s2_n = psi1_n P psi1_n^T = sum_a Kuf(a, n)
// F1(a, n) with F1 = P psi1^T, (Uv)_n = sum_a Kuf(a, n) v_a, then dL_dR_n (fitc.py:67) and the rank-1 factor of dL_dKnm^T,
// Yb_n = beta*_n (y_n - (Uv)_n) (:77-79); the padding columns get 0
__global__ void __launch_bounds__(256) fitc_dldr_kernel(const double* __restrict__ Kuf, const double* __restrict__ F1,
                                                        long ld, long M, long N, long Npad, const double* __restrict__ v,
                                                        const double* __restrict__ Y, const double* __restrict__ b,
                                                        double* __restrict__ dLdR, double* __restrict__ Yb) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long n = (long)blockIdx.x * 8 + warp;
  if (n >= Npad) return;
  if (n >= N) {
    if (lane == 0) { dLdR[n] = 0.0; Yb[n] = 0.0; }
    return;
  }
  const double *k = Kuf + n * ld, *f = F1 + n * ld;
  double s2 = 0.0, uv = 0.0;
  for (long a = lane; a < M; a += 32) {
    const double ka = k[a];
    s2 = fma(ka, f[a], s2);
    uv = fma(ka, v[a], uv);
  }
  s2 = fitc_warp_sum(s2);
  uv = fitc_warp_sum(uv);
  if (lane != 0) return;
  const double be = b[n], y = Y[n];
  dLdR[n] = 0.5 * (s2 - 1.0 / be + y * y - 2.0 * uv * y + uv * uv) * (be * be);
  Yb[n] = (y - uv) * be;
}
// dL_dKnm^T without its rank-1 term, in place of F1: -F1 diag(beta*) - 2 F2 diag(dL_dR) (fitc.py:78-80), and G = F2
// diag(dL_dR) for the Kmm term F2 diag(dL_dR) F2^T (:73-74), over all Npad columns (the GEMM reads G to k-depth Npad);
// rows a >= M and columns n >= N are zeroed in both
__global__ void fitc_assemble_kernel(double* __restrict__ dLt, const double* __restrict__ F2, double* __restrict__ G,
                                     long ld, long M, long N, long Npad, const double* __restrict__ b,
                                     const double* __restrict__ dLdR) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ld * Npad) return;
  const long a = i % ld, n = i / ld;
  if (a >= M || n >= N) { dLt[i] = 0.0; G[i] = 0.0; return; }
  const double r = dLdR[n], f2 = F2[i];
  dLt[i] = -b[n] * dLt[i] - 2.0 * r * f2;
  G[i] = r * f2;
}
}  // namespace

// One FITC evaluation of the validated kernel k (Kdiag = kdiag): grad = [k's gradient block, d/d noise variance],
// dZ (M x D), dL_dKdiag (N, or null) = dL_dR. Route (NT GEMMs over column-major operands; k-depth M reads psi1 as Kfu,
// k-depth N reads M x N operands M-contiguous):
//   Kmm + 1e-6 I -> Um, Lmi;  tmp = Lmi psi1^T;  s1;  sigma*, beta*;  tmp diag(sqrt beta*);  A = tmp tmp^T;  B = I + A
//   -> UB, LBi;  t = tmp (sqrt(beta*) y);  b = LBi t, v = Lmi^T LBi^T b;  P = Um B^-1 Um^T;  Kmm^-1 = Um Um^T;
//   F1 = P psi1^T, F2 = Kmm^-1 psi1^T;  s2, Uv, dL_dR;  dL_dKmm = 1/2 (Kmm^-1 - v v^T - P) + F2 diag(dL_dR) F2^T;
//   dL_dKnm^T = -F1 diag(beta*) - 2 F2 diag(dL_dR) + v (beta* (y - Uv))^T;  the reductions of VarDTC
static int fitc_eval_impl(gpx_ctx* c, const MultiKern& k, double kdiag, const double* Z, int64_t M, double noise,
                          double* lml, double* grad, double* dZ, double* dL_dKdiag) {
  GPX_CUDA(cudaSetDevice(c->device));
  SparseState* s = c->sparse;
  cudaStream_t st = c->st;
  s->have_eval = false;
  s->w_ready = false;
  s->mk = k;
  s->kdiag = kdiag;
  s->jitter = 1e-6;                                                                     // fitc.py:18
  s->noise = noise;
  memset(&c->stats, 0, sizeof(c->stats));
  GPX_CHECK(psi_device(c, Z, M));
  const long Mpad = s->Mpad, N = s->N, Npad = s->Npad;
  const int D = s->D;
  const int ngk = kern_ngrad(s->mk);
  constexpr int RSPLIT = 64;
  if (!s->mm[0]) {
    for (auto& p : s->mm) GPX_CUDA(cudaMalloc(&p, (size_t)Mpad * Mpad * 8));
    GPX_CUDA(cudaMalloc(&s->vec, (size_t)(8 + RSPLIT) * Mpad * 8));
  }
  if (!s->red) {
    GPX_CUDA(cudaMalloc(&s->red, 4096 * 8));
    GPX_CUDA(cudaMallocHost(&s->h_red, 4096 * 8));
  }
  if (!s->hb) {
    GPX_CUDA(cudaMalloc(&s->hb, (size_t)2 * Npad * 8));
    GPX_CUDA(cudaMalloc(&s->hs, (size_t)(2 + s->P) * Npad * 8));
  }
  if (!s->F2) {
    GPX_CUDA(cudaMalloc(&s->F2, (size_t)Mpad * Npad * 8));
    GPX_CUDA(cudaMalloc(&s->G, (size_t)Mpad * Npad * 8));
  }
  if (!s->cK) { GPX_CHECK(gpx_create(c->device, &s->cK)); GPX_CHECK(gpx_create(c->device, &s->cB)); }
  for (gpx_ctx* ch : {s->cK, s->cB})
    if (ch->NB != c->NB) GPX_CHECK(gpx_set_option(ch, "nb", c->NB));
  double *Kd = s->mm[0], *Um = s->mm[1], *Lmi = s->mm[2], *T = s->mm[3], *Ki = s->mm[4], *Bd = s->mm[5], *UB = s->mm[6],
         *LBi = s->mm[7], *Pm = s->mm[8], *E = s->mm[9];
  double *tv = s->vec, *vv = tv + Mpad, *Cv = vv + Mpad, *wv = Cv + Mpad, *rpart = s->vec + (size_t)8 * Mpad;
  double *sbv = s->hb, *bv = s->hb + Npad, *s1 = s->hs, *dLdR = s->hs + Npad;
  double* Tuf = s->dLt;   // tmp, then F1, then dL_dKnm^T
  // Kmm + const_jitter, factored with jitchol's ladder as pdinv does (fitc.py:38-39, linalg.py:193-214)
  GPX_CHECK(build_Kmm(c, Kd));
  GPX_CHECK(factor_child(c, s->cK, Kd, 1e-6, nullptr, Um, Lmi));
  c->stats.tries = s->cK->stats.tries;
  // tmp = Li U^T (:42), s1 = its column norms, sigma*, beta* and the bound's sums over n (:43-44)
  GPX_CHECK(mul_psi1T(c, Lmi, Tuf, 2));
  GPX_CHECK(launch_col_sqnorm(Tuf, Mpad, M, N, s1, st));
  GPX_CHECK(launched(c));
  int* bad = reinterpret_cast<int*>(s->red + 2 * FITC_RED_BLOCKS);
  GPX_CUDA(cudaMemsetAsync(bad, 0x7f, sizeof(int), st));
  fitc_beta_kernel<<<FITC_RED_BLOCKS, 256, 0, st>>>(s1, N, Npad, kdiag, noise, s->Y, sbv, bv, s->Yb, s->red, bad);
  GPX_CHECK(launched(c));
  GPX_CUDA(cudaMemcpyAsync(s->h_red, s->red, (2 * FITC_RED_BLOCKS + 1) * 8, cudaMemcpyDeviceToHost, st));
  GPX_CUDA(cudaStreamSynchronize(st));
  {
    int first;
    memcpy(&first, s->h_red + 2 * FITC_RED_BLOCKS, sizeof(int));
    if (first < N) {
      gpx::set_error("FITC: the effective noise Kdiag + noise variance - Qdiag of data point " + std::to_string(first) +
                     " is not positive (or is NaN)");
      return 1 + first;
    }
  }
  double sum_log_beta = 0.0, sum_bY2 = 0.0;
  for (int i = 0; i < FITC_RED_BLOCKS; i++) { sum_log_beta += s->h_red[2 * i]; sum_bY2 += s->h_red[2 * i + 1]; }
  // A = tdot(tmp diag(sqrt beta*)) + I, factored with jitchol's ladder (:47-48)
  scale_cols_kernel<<<(unsigned)((Mpad * N + 255) / 256), 256, 0, st>>>(Tuf, Mpad, N, sbv);
  GPX_CHECK(launched(c));
  GPX_CHECK(gemm_nt(c, Tuf, Mpad, Tuf, Mpad, Kd, Mpad, Mpad, Mpad, Npad, 2, 0));   // A_raw, lower tiles (Kd is free)
  GPX_CHECK(launch_row_dot(Tuf, Mpad, Mpad, N, 1, s->Yb, Npad, RSPLIT, rpart, tv, st));   // t = Li U^T diag(beta*) y
  GPX_CHECK(launched(c, 2));
  {
    dim3 grid((unsigned)((Mpad + 255) / 256), (unsigned)Mpad);
    mirror_tiles_kernel<<<grid, 256, 0, st>>>(Kd, Mpad, Mpad);
    GPX_CHECK(launched(c));
  }
  GPX_CHECK(combine(c, Bd, Mpad, 1.0, Kd, 0.0, nullptr, 1.0));
  double logdetB = 0.0;
  GPX_CHECK(factor_child(c, s->cB, Bd, 0.0, &logdetB, UB, LBi));
  // b = LA^-1 Li U^T beta* y, v = Li^T LA^-T b (:51-55)
  GPX_CHECK(launch_col_dot(UB, Mpad, Mpad, Mpad, 1, tv, Mpad, vv, Mpad, st));             // b = UB^T t = LBi t
  GPX_CHECK(launch_col_dot(LBi, Mpad, Mpad, Mpad, 1, vv, Mpad, wv, Mpad, st));            // LBi^T b
  GPX_CHECK(launch_col_dot(Lmi, Mpad, Mpad, Mpad, 1, wv, Mpad, Cv, Mpad, st));            // v = Lmi^T LBi^T b
  GPX_CHECK(launched(c, 3));
  std::vector<double> hb((size_t)M);
  GPX_CUDA(cudaMemcpyAsync(hb.data(), vv, (size_t)M * 8, cudaMemcpyDeviceToHost, st));
  // P = Li^T LA^-T LA^-1 Li = Um B^-1 Um^T (:56-57), Kmm^-1 = Um Um^T (pdinv), both exactly symmetric
  GPX_CHECK(binv(c, UB, Pm));
  GPX_CHECK(sandwich(c, Um, Pm, T, Pm));
  GPX_CHECK(binv(c, Um, Ki));
  // F1 = P U^T, F2 = Kmm^-1 U^T; s2, Uv, dL_dR (:66-67) and Yb = beta* (y - Uv)
  GPX_CHECK(mul_psi1T(c, Pm, Tuf, 0));
  GPX_CHECK(mul_psi1T(c, Ki, s->F2, 0));
  fitc_dldr_kernel<<<(unsigned)((Npad + 7) / 8), 256, 0, st>>>(s->Kuf, Tuf, Mpad, M, N, Npad, Cv, s->Y, bv, dLdR, s->Yb);
  GPX_CHECK(launched(c));
  fitc_assemble_kernel<<<(unsigned)((Mpad * Npad + 255) / 256), 256, 0, st>>>(Tuf, s->F2, s->G, Mpad, M, N, Npad, bv,
                                                                              dLdR);
  GPX_CHECK(launched(c));
  std::vector<double> hr((size_t)N);
  GPX_CUDA(cudaMemcpyAsync(hr.data(), dLdR, (size_t)N * 8, cudaMemcpyDeviceToHost, st));
  // dL_dKmm = 1/2 (Kmm^-1 - v v^T - P) + F2 diag(dL_dR) F2^T (:71-74), the last term lower tiles mirrored
  GPX_CHECK(gemm_nt(c, s->F2, Mpad, s->G, Mpad, Bd, Mpad, Mpad, Mpad, Npad, 2, 0));
  {
    dim3 grid((unsigned)((Mpad + 255) / 256), (unsigned)Mpad);
    mirror_tiles_kernel<<<grid, 256, 0, st>>>(Bd, Mpad, Mpad);
    GPX_CHECK(launched(c));
  }
  GPX_CHECK(combine(c, E, Mpad, 0.5, Ki, -0.5, Pm, 0.0, -0.5, Cv, 1));
  GPX_CHECK(combine(c, Kd, Mpad, 1.0, E, 1.0, Bd, 0.0));
  // the Knm reductions with the rank-1 term v (beta* (y - Uv))^T (:76-78), then the Kmm ones (sparse_gp.py:114,117)
  GPX_CUDA(cudaMemcpyAsync(s->Cm, Cv, (size_t)Mpad * 8, cudaMemcpyDeviceToDevice, st));
  std::vector<double> g_knm(ngk, 0.0), g_kmm(ngk, 0.0), hz((size_t)M * D);
  GPX_CHECK(knm_reduce(c, g_knm.data(), dZ));
  const GradFullParams gk = grad_params(s->mk, D, s->zpts(), s->zpts(), Kd, Mpad);
  GPX_CHECK(ensure_part(s, grad_full_doubles(s->mk, D, gk) * 8));
  GPX_CHECK(grad_full_sum(c, s->mk, D, gk, s->part, g_kmm.data()));
  GPX_CHECK(ensure_part(s, grad_X_doubles(c, s->mk, gk, D) * 8));
  GPX_CHECK(grad_X(c, s->mk, gk, D, s->part, hz.data()));
  for (size_t i = 0; i < hz.size(); i++) dZ[i] += hz[i];
  GPX_CUDA(cudaStreamSynchronize(st));
  // the bound (:60-64); the Kdiag share and the noise gradient are sum(dL_dR) (sparse_gp.py:110, gaussian.py:78-79)
  double data_fit = 0.0, sum_dR = 0.0;
  for (long i = 0; i < M; i++) data_fit += hb[i] * hb[i];
  for (long n = 0; n < N; n++) sum_dR += hr[n];
  const double log2pi = 1.8378770664093453;
  *lml = -0.5 * (double)N * log2pi - 0.5 * logdetB + 0.5 * sum_log_beta - 0.5 * sum_bY2 + 0.5 * data_fit;
  kern_grads(s, sum_dR, g_knm, g_kmm, grad);
  grad[ngk] = sum_dR;
  if (dL_dKdiag) memcpy(dL_dKdiag, hr.data(), (size_t)N * 8);
  s->have_eval = true;
  return 0;
}

extern "C" {

int gpx_sparse_eval_fitc(gpx_ctx* c, const gpx_kern_part* parts, int nparts, const double* Z, int64_t M,
                         double noise_variance, double* lml, double* grad, double* dZ, double* dL_dKdiag) {
  GPX_CHECK(sparse_args(c, parts, Z, M, lml, grad, dZ, false, nullptr));
  if (c->dist) GPX_FAIL("FITC is single-GPU");
  if (c->sparse->P != 1) GPX_FAIL("FITC takes one output column (fitc.py reshapes v to a column)");
  MultiKern mk;
  double kdiag;
  GPX_CHECK(fill_mk(mk, parts, nparts, c->sparse->D, &kdiag));
  for (int p = 0; p < mk.nparts; p++)   // dL/dZ needs every part's gradients_X
    if (mk.part[p].kind == GPX_RATQUAD || mk.part[p].kind == GPX_STDPERIODIC)
      GPX_FAIL("RatQuad and StdPeriodic parts are not on the sparse evaluation (no device gradients_X)");
  return fitc_eval_impl(c, mk, kdiag, Z, M, noise_variance, lml, grad, dZ, dL_dKdiag);
}

}  // extern "C"

// =================================================================================================================
// Sparse EP (EPDTC, expectation_propagation.py:436-611) for the probit Bernoulli likelihood, in M-space.
// The posterior of the sites is Sigma = Knm A Kmn with A = LLT^-1, LLT = Kmm + Kmn diag(tau~) Knm (M x M), and
// mu = mu0 + Knm u, mu0 that of the last recompute. A sequential sweep runs in blocks of TILE sites I of the order:
//   KbT = Kmn[:, I]^T (gather), P^T = KbT A, G = KbT P = Sigma[I, I] (DMMA GEMMs), mu_I = mu0[I] + KbT u;
//   the site chain of dense EP on G (ep_chain_kernel, dtc form: the cavity reads the clipped diagonal the reference holds);
//   Y = P (I + U)^-1 over the M rows (ep_solve_kernel, dtc form), u -= Y g; A -= Y diag(c) Y^T (GEMM_UPDATE), mirrored.
// Sigma -= S diag(c) S^T with S = Knm Y is dense EP's update, which regroups the reference's chain of rank-1 updates; here
// it is carried by A, so nothing of size N x N or N x TILE is formed. _recompute (:175-185): LLT from the GEMM with k-depth
// N, jitchol's ladder on the factor-and-invert sweep, A = U U^T, V = L^-1 Kmn, Sigma_diag = |V[:, n]|^2 and mu = V^T (V v~).
// =================================================================================================================
namespace {
// the site vectors of the sparse EP, s->ev + k * Npad
enum { ED_TT = 0, ED_VT, ED_SGN, ED_CT, ED_CV, ED_ZH, ED_MH, ED_S2, ED_MU0, ED_SD, ED_SDT, ED_QNN, ED_Y, ED_DRIFT, EDV_N };
constexpr int EP_RSPLIT = 64;
double* edv(SparseState* s, int k) { return s->ev + (size_t)k * s->Npad; }
// one block of sites, inside s->epb
struct EpBlock { double *KbT, *PT, *Sx, *Sc, *G, *Gb, *cg, *ku, *u, *t, *part; };
EpBlock ep_block(SparseState* s) {
  const size_t Mp = (size_t)s->Mpad;
  EpBlock b;
  b.KbT = s->epb; b.PT = b.KbT + TILE * Mp; b.Sx = b.PT + TILE * Mp; b.Sc = b.Sx + TILE * Mp; b.G = b.Sc + TILE * Mp;
  b.Gb = b.G + TILE * TILE; b.cg = b.Gb + TILE * TILE; b.ku = b.cg + 2 * TILE; b.u = b.ku + TILE; b.t = b.u + Mp;
  b.part = b.t + Mp;
  return b;
}
size_t ep_block_doubles(long Mpad) { return (size_t)4 * TILE * Mpad + 2 * TILE * TILE + 3 * TILE + (2 + EP_RSPLIT) * Mpad; }

// KbT (TILE x Mpad, ld TILE) = rows I of Kfu, zero beyond m
__global__ void epdtc_gather_kernel(const double* __restrict__ Kfu, long ldk, const int* __restrict__ I, int m, long Mpad,
                                    double* __restrict__ KbT) {
  const long k = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= (long)TILE * Mpad) return;
  const int j = (int)(k % TILE);
  const long a = k / TILE;
  KbT[k] = j < m ? Kfu[I[j] + a * ldk] : 0.0;
}
// o_i = max(x_i, eps) (clip = 1) or x_i + add, for i < N; zero for N <= i < n
__global__ void epdtc_vec_kernel(int clip, long N, long n, const double* __restrict__ x, double add, double* __restrict__ o) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  o[i] = i < N ? (clip ? fmax(x[i], 2.220446049250313e-16) : x[i] + add) : 0.0;
}

// o_n = sum_a K[a, n] W[a, n] over the M rows (diag(Knm A Kmn) with W = A Kmn), one thread per column, fixed order
__global__ void epdtc_coldot_kernel(const double* __restrict__ K, const double* __restrict__ W, long ld, long M, long N,
                                    double* __restrict__ o) {
  const long n = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  double d = 0.0;
  for (long a = 0; a < M; a++) d = fma(K[a + n * ld], W[a + n * ld], d);
  o[n] = d;
}

int ep_vecop(gpx_ctx* c, int clip, const double* x, double add, double* o) {
  SparseState* s = c->sparse;
  epdtc_vec_kernel<<<(unsigned)((s->Npad + 255) / 256), 256, 0, c->st>>>(clip, s->N, s->Npad, x, add, o);
  return launched(c);
}

int epdtc_args(gpx_ctx* c) {
  if (!c) GPX_FAIL("null argument");
  if (c->dist) GPX_FAIL("sparse expectation propagation is single-GPU");
  if (!c->sparse || !c->sparse->X) GPX_FAIL("gpx_sparse_set_data has not been called");
  if (!c->sparse->ep_begun) GPX_FAIL("gpx_epdtc_begin has not been called on this data, kernel and Z");
  return 0;
}

int epdtc_upload(gpx_ctx* c, int slot, const double* h) {
  GPX_CUDA(cudaMemcpyAsync(edv(c->sparse, slot), h, (size_t)c->sparse->N * 8, cudaMemcpyHostToDevice, c->st));
  return 0;
}
int epdtc_download(gpx_ctx* c, int slot, double* h) {
  if (h) GPX_CUDA(cudaMemcpyAsync(h, edv(c->sparse, slot), (size_t)c->sparse->N * 8, cudaMemcpyDeviceToHost, c->st));
  return 0;
}

// posteriorParamsDTC._recompute (:175-185) from the sites in ED_TT / ED_VT: A = LLT^-1, the true diagonal in ED_SDT,
// mu0 in ED_MU0, u = 0. -> 0 or the failing minor of LLT after the ladder
int epdtc_recompute(gpx_ctx* c, int max_tries, double* jitter_used) {
  SparseState* s = c->sparse;
  cudaStream_t st = c->st;
  const long Mpad = s->Mpad, Npad = s->Npad, N = s->N, M = s->M;
  double *R = s->mm[3], *LLT = s->mm[4], *U = s->mm[1], *Linv = s->mm[2];
  const EpBlock b = ep_block(s);
  // LLT = Kmm + (Kmn diag(tau~)) Knm: the scaled copy in the dL_dKnm^T buffer, the product's lower tiles, mirrored
  GPX_CUDA(cudaMemcpyAsync(s->dLt, s->Kuf, (size_t)Mpad * Npad * 8, cudaMemcpyDeviceToDevice, st));
  scale_cols_kernel<<<(unsigned)((Mpad * N + 255) / 256), 256, 0, st>>>(s->dLt, Mpad, N, edv(s, ED_TT));
  GPX_CHECK(launched(c));
  {
    GemmParams pg = gemm_defaults();
    pg.mode = GEMM_PANEL; pg.plain = 2;
    pg.A = s->dLt; pg.lda = Mpad; pg.B = s->Kuf; pg.ldb = Mpad; pg.C = R; pg.ldc = Mpad;
    pg.K = (int)Npad; pg.nt = (int)(Mpad / TILE); pg.ncols = (int)(Mpad / TILE);
    GPX_CHECK(launch_gemm(pg, dim3(1, 1), st));
    GPX_CHECK(launched(c));
  }
  mirror_tiles_kernel<<<dim3((unsigned)((Mpad + 255) / 256), (unsigned)Mpad), 256, 0, st>>>(R, Mpad, Mpad);
  GPX_CHECK(launched(c));
  GPX_CHECK(combine(c, LLT, M, 1.0, s->eK, 1.0, R, 0.0));
  const int rc = factor_child(c, s->cK, LLT, 0.0, nullptr, U, Linv, jitter_used, max_tries);
  if (rc) return rc;
  GPX_CHECK(binv(c, U, s->eA));                                                          // A = U U^T = LLT^-1
  GPX_CHECK(mul_psi1T(c, Linv, s->dLt, 2));                                              // V = L^-1 Kmn
  GPX_CHECK(launch_col_sqnorm(s->dLt, Mpad, M, N, edv(s, ED_SDT), st));
  GPX_CHECK(launch_row_dot(s->dLt, Mpad, Mpad, N, 1, edv(s, ED_VT), Npad, EP_RSPLIT, b.part, b.t, st));   // t = V v~
  GPX_CHECK(launch_col_dot(s->dLt, Mpad, M, N, 1, b.t, Mpad, edv(s, ED_MU0), Npad, st));                   // mu0 = V^T t
  GPX_CHECK(launched(c, 4));
  GPX_CUDA(cudaMemsetAsync(b.u, 0, (size_t)Mpad * 8, st));
  return 0;
}

int epdtc_end(gpx_ctx* c, const char* what) {
  if (cudaStreamSynchronize(c->st) != cudaSuccess) GPX_FAIL_DEVICE(what);
  return 0;
}
}  // namespace

extern "C" {

int gpx_epdtc_begin(gpx_ctx* c, const gpx_kern_part* parts, int nparts, const double* Z, int64_t M) {
  if (!c || !parts || !Z) GPX_FAIL("null argument");
  if (c->dist) GPX_FAIL("sparse expectation propagation is single-GPU");
  if (!c->sparse || !c->sparse->X) GPX_FAIL("gpx_sparse_set_data has not been called");
  SparseState* s = c->sparse;
  if (s->P != 1) GPX_FAIL("sparse expectation propagation takes one output column (P = 1)");
  if (M < 1) GPX_FAIL("M must be positive");
  MultiKern mk;
  double kdiag;
  GPX_CHECK(fill_mk(mk, parts, nparts, s->D, &kdiag));
  for (int p = 0; p < mk.nparts; p++)
    if (mk.part[p].kind == GPX_RATQUAD || mk.part[p].kind == GPX_STDPERIODIC)
      GPX_FAIL("RatQuad and StdPeriodic parts are not on the sparse evaluation (no device gradients_X)");
  GPX_CUDA(cudaSetDevice(c->device));
  cudaStream_t st = c->st;
  const long N = s->N, Npad = s->Npad;
  if (!s->ep_labels) {   // once per data set: gpx_sparse_set_data clears the flag
    std::vector<double> y((size_t)N);
    GPX_CUDA(cudaMemcpy(y.data(), s->Y, (size_t)N * 8, cudaMemcpyDeviceToHost));
    for (double v : y)
      if (!(v == 1.0 || v == 0.0 || v == -1.0)) GPX_FAIL("bad value for Bernoulli observation (0, 1)");
  }
  s->have_eval = s->w_ready = false;
  s->mk = mk;
  s->kdiag = kdiag;
  memset(&c->stats, 0, sizeof(c->stats));
  GPX_CHECK(psi_device(c, Z, M));
  const long Mpad = s->Mpad;
  if (!s->mm[0]) {
    for (auto& p : s->mm) GPX_CUDA(cudaMalloc(&p, (size_t)Mpad * Mpad * 8));
    GPX_CUDA(cudaMalloc(&s->vec, (size_t)(8 + 64) * s->P * Mpad * 8));
  }
  if (!s->red) {
    GPX_CUDA(cudaMalloc(&s->red, 4096 * 8));
    GPX_CUDA(cudaMallocHost(&s->h_red, 4096 * 8));
  }
  if (!s->cK) { GPX_CHECK(gpx_create(c->device, &s->cK)); GPX_CHECK(gpx_create(c->device, &s->cB)); }
  for (gpx_ctx* ch : {s->cK, s->cB})
    if (ch->NB != c->NB) GPX_CHECK(gpx_set_option(ch, "nb", c->NB));
  if (!s->eK) {
    for (double** p : {&s->eK, &s->eA, &s->eA0}) GPX_CUDA(cudaMalloc(p, (size_t)Mpad * Mpad * 8));
    GPX_CUDA(cudaMalloc(&s->epb, ep_block_doubles(Mpad) * 8));
    GPX_CUDA(cudaMemsetAsync(s->epb, 0, ep_block_doubles(Mpad) * 8, st));
  }
  if (!s->ev) {
    GPX_CUDA(cudaMalloc(&s->ev, (size_t)EDV_N * Npad * 8));
    GPX_CUDA(cudaMemsetAsync(s->ev, 0, (size_t)EDV_N * Npad * 8, st));
    GPX_CUDA(cudaMalloc(&s->eord, (size_t)Npad * sizeof(int)));
  }
  s->eZ.assign(Z, Z + (size_t)M * s->D);
  // Kmm (LLT0, no jitter), Lm = jitchol(Kmm); A0 = Kmm^-1 and diag(Knm Kmm^-1 Kmn) for the cold start (:522-535)
  GPX_CHECK(build_Kmm(c, s->eK));
  double jit = 0.0;
  const int rc = factor_child(c, s->cK, s->eK, 0.0, nullptr, s->mm[1], s->mm[2], &jit, 5);
  if (rc) return rc;
  GPX_CHECK(binv(c, s->mm[1], s->eA0));
  GPX_CHECK(mul_psi1T(c, s->mm[2], s->dLt, 2));
  GPX_CHECK(launch_col_sqnorm(s->dLt, Mpad, M, N, edv(s, ED_QNN), st));
  GPX_CHECK(launched(c));
  ep_vec_kernel<<<(unsigned)((Npad + 255) / 256), 256, 0, st>>>(EV_SIGN, N, Npad, s->Y, nullptr, nullptr, 0, 0.0,
                                                                edv(s, ED_SGN));
  GPX_CHECK(launched(c));
  GPX_CHECK(epdtc_end(c, "gpx_epdtc_begin"));
  s->ep_labels = true;
  s->ep_begun = true;
  s->ep_ready = false;
  return 0;
}

int gpx_epdtc_start(gpx_ctx* c, const double* tau_tilde, const double* v_tilde, int warm, int parallel, int max_tries,
                    double* jitter_used, double* mu, double* sigma_diag) {
  if (!c || !jitter_used || (warm && (!tau_tilde || !v_tilde))) GPX_FAIL("null argument");
  GPX_CHECK(epdtc_args(c));
  GPX_CUDA(cudaSetDevice(c->device));
  SparseState* s = c->sparse;
  cudaStream_t st = c->st;
  const long Mpad = s->Mpad, Npad = s->Npad;
  s->ep_ready = false;
  s->ep_seq = !parallel;
  memset(&c->stats, 0, sizeof(c->stats));
  *jitter_used = 0.0;
  const EpBlock b = ep_block(s);
  if (!warm) {   // cold (:536-544): sites 0, LLT = Kmm, mu = 0, Sigma_diag = diag(Knm Kmm^-1 Kmn) + 1e-8
    for (int k : {ED_TT, ED_VT, ED_MU0}) GPX_CUDA(cudaMemsetAsync(edv(s, k), 0, (size_t)Npad * 8, st));
    GPX_CUDA(cudaMemsetAsync(b.u, 0, (size_t)Mpad * 8, st));
    GPX_CUDA(cudaMemcpyAsync(s->eA, s->eA0, (size_t)Mpad * Mpad * 8, cudaMemcpyDeviceToDevice, st));
    GPX_CHECK(ep_vecop(c, 0, edv(s, ED_QNN), 1e-8, edv(s, ED_SD)));
  } else {       // warm (:545-549): the recompute from the kept sites, then 1e-8 on Sigma_diag (no clip)
    GPX_CHECK(epdtc_upload(c, ED_TT, tau_tilde));
    GPX_CHECK(epdtc_upload(c, ED_VT, v_tilde));
    const int rc = epdtc_recompute(c, max_tries, jitter_used);
    if (rc) { epdtc_end(c, "gpx_epdtc_start"); return rc; }
    GPX_CHECK(ep_vecop(c, 0, edv(s, ED_SDT), 1e-8, edv(s, ED_SD)));
  }
  GPX_CHECK(epdtc_download(c, ED_MU0, mu));
  GPX_CHECK(epdtc_download(c, ED_SD, sigma_diag));
  GPX_CHECK(epdtc_end(c, "gpx_epdtc_start"));
  s->ep_first = true;
  s->ep_ready = true;
  return 0;
}

int gpx_epdtc_sweep(gpx_ctx* c, const int64_t* order, double eta, double delta, int parallel, int max_tries,
                    double* tau_tilde, double* v_tilde, double* cav_tau, double* cav_v, double* Z_hat, double* mu_hat,
                    double* sigma2_hat, double* jitter_used, double* mu, double* sigma_diag) {
  if (!c || !order || !tau_tilde || !v_tilde || !cav_tau || !cav_v || !Z_hat || !mu_hat || !sigma2_hat || !jitter_used)
    GPX_FAIL("null argument");
  GPX_CHECK(epdtc_args(c));
  SparseState* s = c->sparse;
  if (!s->ep_ready) GPX_FAIL("gpx_epdtc_start has not been called since gpx_epdtc_begin");
  if (!parallel != s->ep_seq) GPX_FAIL("parallel must be the value gpx_epdtc_start was given");
  const long N = s->N, Npad = s->Npad, Mpad = s->Mpad;
  std::vector<int> ord((size_t)N);
  {
    std::vector<char> seen((size_t)N, 0);
    for (long k = 0; k < N; k++) {
      const int64_t i = order[k];
      if (i < 0 || i >= N || seen[(size_t)i]) GPX_FAIL("order is not a permutation of 0 .. N-1");
      seen[(size_t)i] = 1;
      ord[(size_t)k] = (int)i;
    }
  }
  GPX_CUDA(cudaSetDevice(c->device));
  cudaStream_t st = c->st;
  memset(&c->stats, 0, sizeof(c->stats));
  GPX_CHECK(epdtc_upload(c, ED_TT, tau_tilde));
  GPX_CHECK(epdtc_upload(c, ED_VT, v_tilde));
  EpSites e;
  e.tt = edv(s, ED_TT); e.vt = edv(s, ED_VT); e.ct = edv(s, ED_CT); e.cv = edv(s, ED_CV); e.zh = edv(s, ED_ZH);
  e.mh = edv(s, ED_MH); e.s2 = edv(s, ED_S2); e.sgn = edv(s, ED_SGN); e.eta = eta; e.delta = delta;
  if (!parallel) {   // _local_updates with posteriorParamsDTC._update_rank1 (:553-572), one block of TILE sites at a time
    GPX_CUDA(cudaMemcpyAsync(s->eord, ord.data(), (size_t)N * sizeof(int), cudaMemcpyHostToDevice, st));
    GPX_CUDA(cudaFuncSetAttribute(ep_chain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, EP_CHAIN_SMEM));
    GPX_CUDA(cudaFuncSetAttribute(ep_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, EP_SOLVE_SMEM));
    const EpBlock b = ep_block(s);
    const unsigned solve_grid = (unsigned)std::min<long>(Mpad / EP_SOLVE_ROWS, c->num_sms);
    const unsigned gather_grid = (unsigned)((TILE * Mpad + 255) / 256);
    for (long k0 = 0; k0 < N; k0 += TILE) {
      const int m = (int)std::min<long>(TILE, N - k0);
      const int* I = s->eord + k0;
      epdtc_gather_kernel<<<gather_grid, 256, 0, st>>>(s->Kfu, Npad, I, m, Mpad, b.KbT);
      GPX_CHECK(launched(c));
      GPX_CHECK(gemm_nt(c, b.KbT, TILE, s->eA, Mpad, b.PT, TILE, TILE, Mpad, Mpad, 1, 0));   // P^T = KbT A
      GPX_CHECK(gemm_nt(c, b.KbT, TILE, b.PT, TILE, b.G, TILE, TILE, TILE, Mpad, 1, 0));    // G = KbT P
      GPX_CHECK(launch_row_dot(b.KbT, TILE, TILE, Mpad, 1, b.u, Mpad, EP_RSPLIT, b.part, b.ku, st));   // KbT u
      GPX_CHECK(launched(c, 2));
      ep_chain_kernel<<<1, EP_CHAIN_THREADS, EP_CHAIN_SMEM, st>>>(b.G, TILE, I, m, edv(s, ED_MU0), e, b.Gb, b.cg, b.ku,
                                                                  s->ep_first ? edv(s, ED_SD) : nullptr, 1);
      ep_solve_kernel<<<solve_grid, EP_SOLVE_ROWS, EP_SOLVE_SMEM, st>>>(b.PT, Mpad, I, m, b.Gb, b.cg, b.Sx, b.Sc, b.u, 1);
      GPX_CHECK(launched(c, 2));
      s->ep_first = false;
      GemmParams pu = gemm_defaults();   // A -= Y diag(c) Y^T over the lower tiles, k-depth TILE, then mirrored
      pu.mode = GEMM_UPDATE;
      pu.A = b.Sc; pu.lda = Mpad; pu.B = b.Sx; pu.ldb = Mpad; pu.C = s->eA; pu.ldc = Mpad;
      pu.K = TILE; pu.nt = (int)(Mpad / TILE); pu.c0 = 0; pu.ncols = 0; pu.rlow = 0;
      GPX_CHECK(launch_gemm(pu, dim3(1, 1), st));
      GPX_CHECK(launched(c));
      mirror_tiles_kernel<<<dim3((unsigned)((Mpad + 255) / 256), (unsigned)Mpad), 256, 0, st>>>(s->eA, Mpad, Mpad);
      GPX_CHECK(launched(c));
    }
  } else {           // parallel_updates: every site from the same Sigma_diag and mu
    ep_parallel_kernel<<<(unsigned)((N + 255) / 256), 256, 0, st>>>(N, edv(s, ED_SD), edv(s, ED_MU0), e);
    GPX_CHECK(launched(c));
  }
  const bool drift = c->epdtc_drift && !parallel;
  if (drift) {   // the measurement option: diag(Knm A Kmn) of the downdated A, before the recompute replaces it
    GPX_CHECK(mul_psi1T(c, s->eA, s->dLt, 0));
    epdtc_coldot_kernel<<<(unsigned)((N + 255) / 256), 256, 0, st>>>(s->Kuf, s->dLt, Mpad, s->M, N, edv(s, ED_DRIFT));
    GPX_CHECK(launched(c));
  }
  GPX_CHECK(epdtc_download(c, ED_TT, tau_tilde));
  GPX_CHECK(epdtc_download(c, ED_VT, v_tilde));
  GPX_CHECK(epdtc_download(c, ED_CT, cav_tau));
  GPX_CHECK(epdtc_download(c, ED_CV, cav_v));
  GPX_CHECK(epdtc_download(c, ED_ZH, Z_hat));
  GPX_CHECK(epdtc_download(c, ED_MH, mu_hat));
  GPX_CHECK(epdtc_download(c, ED_S2, sigma2_hat));
  GPX_CHECK(epdtc_end(c, "gpx_epdtc_sweep"));
  s->ep_ready = false;   // A, mu0 and u are those of the updates until the recompute has run
  s->ep_first = false;
  const int rc = epdtc_recompute(c, max_tries, jitter_used);
  if (rc) { epdtc_end(c, "gpx_epdtc_sweep"); return rc; }
  GPX_CHECK(ep_vecop(c, 1, edv(s, ED_SDT), 0.0, edv(s, ED_SD)));                      // np.maximum(Sigma_diag, eps)
  GPX_CHECK(epdtc_download(c, ED_MU0, mu));
  GPX_CHECK(epdtc_download(c, drift ? ED_DRIFT : ED_SD, sigma_diag));
  GPX_CHECK(epdtc_end(c, "gpx_epdtc_sweep"));
  s->ep_ready = true;
  return 0;
}

int gpx_epdtc_finish(gpx_ctx* c, const double* tau_tilde, const double* v_tilde, int max_tries, double* lml, double* grad,
                     double* dZ, double* jitter_used) {
  if (!c || !tau_tilde || !v_tilde || !lml || !grad || !dZ || !jitter_used) GPX_FAIL("null argument");
  GPX_CHECK(epdtc_args(c));
  GPX_CUDA(cudaSetDevice(c->device));
  SparseState* s = c->sparse;
  const long N = s->N;
  // VarDTC.inference at Y = v~ / tau~ and precision = tau~ as they are (:474-482), Lm = jitchol(Kmm)
  std::vector<double> y((size_t)N), dR((size_t)N);
  for (long n = 0; n < N; n++) y[(size_t)n] = v_tilde[n] / tau_tilde[n];
  double* yd = edv(s, ED_Y);
  GPX_CUDA(cudaMemcpyAsync(yd, y.data(), (size_t)N * 8, cudaMemcpyHostToDevice, c->st));
  GPX_CUDA(cudaStreamSynchronize(c->st));
  const std::vector<double> Z = s->eZ;
  double* labels = s->Y;
  s->Y = yd;
  *jitter_used = 0.0;
  const int rc = sparse_eval_impl(c, s->mk, s->kdiag, Z.data(), s->M, 0.0, nullptr, lml, grad, dZ, dR.data(), tau_tilde,
                                  max_tries, jitter_used);
  s->Y = labels;
  return rc;
}

}  // extern "C"

// =================================================================================================================
// SVGP (svgp.py:10-118, Hensman et al. 2013 / 2015) with one output column, one latent function and no mean function, on
// the rows [row0, row0 + nb) of the data of gpx_sparse_set_data. The likelihood's quadrature stays on the host between the
// two entries. Layouts: "M-major" is Mpad x NBp column-major ((a, n) at a + n Mpad), "N-major" NBp x Mpad ((n, a) at
// n + a NBp); every product is the NT DMMA GEMM (C = X Y^T), which reads its Y operand N-major when the contraction runs
// over M and both operands M-major when it runs over the batch. Lmi = Lm^-1, Um = Lm^-T from the factor-and-invert sweep.
//   begin:  Knm (N-major), Kmn (M-major);  Vt = Knm Lmi^T (= (Lm^-1 Kmn)^T, B lower triangular);  A = Um Vt^T
//           (= Kmm^-1 Kmn: dpotrs's two triangular solves, svgp.py:45);  Wt = q_L^T Um;  Bq = Wt Vt^T (= q_L^T A);
//           mu = A^T m, v = colsum(Bq^2) + (Kdiag - colsum(A o Kmn)) (:46-52);  KL (:55) with tr(Kmm^-1 S) = |Wt|_F^2
//   finish: Ki = Um Um^T, S = q_L q_L^T, Tt = Ki S (= T^T, T = S Ki);  Adv = A diag(dF_dv), Vd = diag(dF_dv) Vt;
//           AdvA = Adv A^T (lower tiles, mirrored);  R = AdvA T;  KSK = Ki S Ki;  dL_dKmm (:81-83,60 symmetrised);
//           dL_dKmn^T = (2 (Tt - I) Um) Vd^T + Kmm^-1 m dF_dmu^T (:85-90; the rank-1 term added by the reductions);
//           dL_dchol = 2 tril((AdvA - Ki / 2) q_L) + diag(1 / q_L,ii) (:113-114: S^-1 q_L = q_L^-T is upper triangular,
//           so the reference's dpotri (Si, :22) is not formed); posterior: woodbury_vector = Kmm^-1 m, woodbury_inv =
//           Ki - KSK (posterior.py:166-196 with K = Kmm, cov = S).
// Products of M^2 NBp: Vt (1 M^2 NBp multiply-adds, triangular), A, Bq, dL_dKmn^T (2 each), AdvA (1, lower tiles): 8 M^2 NBp
// flops; of M^3 (Mpad^3 multiply-adds): Wt, Tt, R, KSK, GU, H (2 each) and Ki, S (1 each, lower tiles), 28 M^3 flops, plus
// the factor-and-invert sweep of Kmm.
// =================================================================================================================
namespace {
enum { SV_M = 0, SV_LMM, SV_ADMU, SV_RPART, SV_MV = SV_RPART + 64 };   // [SV_MV][Mpad] vectors of s->svv
enum { SB_MU = 0, SB_V, SB_DMU, SB_DV };                              // [4][sv_cap] vectors of s->svb
constexpr int SV_RB = 64;                                             // CTAs of trace_dot_kernel
// one batch's device buffers inside s->svb: b[0..3] Mpad x ld each, vec[4][ld], prepared points
struct SvBatch { double* b[4]; double* vec[4]; Points x; };
SvBatch sv_batch(SparseState* s) {
  const size_t cap = (size_t)s->sv_cap, Mp = (size_t)s->Mpad;
  const long ld = (s->sv_nb + TILE - 1) / TILE * TILE;
  SvBatch b;
  for (int k = 0; k < 4; k++) b.b[k] = s->svb + k * Mp * cap;
  for (int k = 0; k < 4; k++) b.vec[k] = s->svb + 4 * Mp * cap + k * cap;
  b.x = Points{s->svb + (4 * Mp + 4) * cap, s->svb + (4 * Mp + 4 + MAX_D) * cap, s->sv_nb, ld};
  return b;
}
size_t sv_batch_doubles(long Mpad, long cap) { return (size_t)(4 * Mpad + 4 + MAX_D + MAX_PARTS) * cap; }

// mu_n = sum_a A(a, n) m_a and v_n = sum_a Bq(a, n)^2 + (kdiag - sum_a A(a, n) Kmn(a, n)) over the M rows of M-major
// operands (svgp.py:46-52): one warp per column, lanes over the rows in a fixed order, then the warp's fixed tree
__global__ void __launch_bounds__(256) svgp_marg_kernel(const double* __restrict__ A, const double* __restrict__ K,
                                                        const double* __restrict__ Bq, long ld, long M, long nb,
                                                        const double* __restrict__ m, double kdiag, double* __restrict__ mu,
                                                        double* __restrict__ v) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long n = (long)blockIdx.x * 8 + warp;
  if (n >= nb) return;
  const double *a = A + n * ld, *k = K + n * ld, *b = Bq + n * ld;
  double am = 0.0, ak = 0.0, bb = 0.0;
  for (long i = lane; i < M; i += 32) {
    const double ai = a[i], bi = b[i];
    am = fma(ai, m[i], am);
    ak = fma(ai, k[i], ak);
    bb = fma(bi, bi, bb);
  }
  am = fitc_warp_sum(am);
  ak = fitc_warp_sum(ak);
  bb = fitc_warp_sum(bb);
  if (lane == 0) { mu[n] = am; v[n] = bb + (kdiag - ak); }
}
// out = in diag(d) (M-major in: the column index scales) or diag(d) in (N-major in: the row index scales), `total` entries,
// leading dimension ld (svgp.py:72 Adv = A dF_dv)
__global__ void svgp_scale_kernel(const double* __restrict__ in, long ld, long total, int rows, const double* __restrict__ d,
                                  double* __restrict__ out) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  out[i] = in[i] * d[rows ? i % ld : i / ld];
}
// dL_dKmm = dF_dKmm - dKL_dKmm (svgp.py:60,81-83,116) with dF_dKmm = sym(-Admu Kmmim^T + AdvA - R - R^T), sym(X) =
// (X + X^T) / 2, and dKL_dKmm = Ki / 2 - KSK / 2 - Kmmim Kmmim^T / 2; zero outside the M x M block
__global__ void svgp_dkmm_kernel(const double* __restrict__ AdvA, const double* __restrict__ R, const double* __restrict__ Ki,
                                 const double* __restrict__ KSK, const double* __restrict__ admu,
                                 const double* __restrict__ kim, long ld, long M, double* __restrict__ out) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y;
  if (i >= ld) return;
  if (i >= M || j >= M) { out[i + j * ld] = 0.0; return; }
  const long ij = i + j * ld, ji = j + i * ld;
  const double r = R[ij] + R[ji];
  const double x = -admu[i] * kim[j] + AdvA[ij] - r, xt = -admu[j] * kim[i] + AdvA[ji] - r;
  const double dF = 0.5 * (x + xt);
  const double dKL = 0.5 * Ki[ij] - 0.5 * KSK[ij] - 0.5 * kim[i] * kim[j];
  out[ij] = dF - dKL;
}
// dL_dchol (M x M row-major, the lower triangle; svgp.py:113): 2 H(i, j) + [i == j] / L_ii for j <= i with
// H = (AdvA - Ki / 2) q_L, zero above the diagonal; L_ii read from Lt = q_L^T (column-major, ld)
__global__ void svgp_dchol_kernel(const double* __restrict__ H, const double* __restrict__ Lt, long ld, long M,
                                  double* __restrict__ out) {
  const long j = (long)blockIdx.x * blockDim.x + threadIdx.x, i = blockIdx.y;
  if (j >= M) return;
  double v = 0.0;
  if (j <= i) v = 2.0 * H[i + j * ld] + (i == j ? 1.0 / Lt[i + i * ld] : 0.0);
  out[i * M + j] = v;
}

int svgp_end(gpx_ctx* c, const char* what) {
  if (cudaStreamSynchronize(c->st) != cudaSuccess) GPX_FAIL_DEVICE(what);
  return 0;
}
}  // namespace

extern "C" {

int gpx_svgp_begin(gpx_ctx* c, const gpx_kern_part* parts, int nparts, const double* Z, int64_t M, const double* q_m,
                   const double* q_L, int64_t row0, int64_t nb, int max_tries, double* mu, double* var, double* kl,
                   double* jitter_used) {
  if (!c || !parts || !Z || !q_m || !q_L || !mu || !var || !kl || !jitter_used) GPX_FAIL("null argument");
  if (c->dist) GPX_FAIL("SVGP is single-GPU");
  if (!c->sparse || !c->sparse->X) GPX_FAIL("gpx_sparse_set_data has not been called");
  SparseState* s = c->sparse;
  if (s->P != 1) GPX_FAIL("SVGP takes one output column and one latent function (P = 1)");
  if (M < 1) GPX_FAIL("M must be positive");
  if (row0 < 0 || nb < 1 || row0 > s->N - nb) GPX_FAIL("the batch rows [row0, row0 + nb) are not inside the data");
  MultiKern mk;
  double kdiag;
  GPX_CHECK(fill_mk(mk, parts, nparts, s->D, &kdiag));
  for (int p = 0; p < mk.nparts; p++)
    if (mk.part[p].kind == GPX_RATQUAD || mk.part[p].kind == GPX_STDPERIODIC)
      GPX_FAIL("RatQuad and StdPeriodic parts are not on the sparse evaluation (no device gradients_X)");
  GPX_CUDA(cudaSetDevice(c->device));
  cudaStream_t st = c->st;
  const int D = s->D;
  s->have_eval = s->dl_ready = s->w_ready = s->w_own = s->sv_begun = false;
  s->mk = mk;
  s->kdiag = kdiag;
  memset(&c->stats, 0, sizeof(c->stats));
  // Z and its prepared points without psi1 (psi_device's set-up; psi_device allocates psi1 when it next runs)
  GPX_CHECK(ensure_rows(c, s, mk));
  const long Mpad = (M + TILE - 1) / TILE * TILE;
  if (Mpad != s->Mpad) {
    GPX_CUDA(cudaStreamSynchronize(st));
    free_m(s);
    s->Mpad = Mpad;
    GPX_CUDA(cudaMalloc(&s->Z, (size_t)Mpad * D * 8));
    GPX_CUDA(cudaMalloc(&s->ZsT, (size_t)Mpad * s->rows_cap * 8));
    GPX_CUDA(cudaMalloc(&s->sqZ, (size_t)Mpad * s->norm_cap * 8));
    GPX_CUDA(cudaMalloc(&s->Cm, (size_t)Mpad * s->P * 8));
  }
  s->M = M;
  if (!s->mm[0]) {   // as the other sparse entries allocate them (they expect vec with mm)
    for (auto& p : s->mm) GPX_CUDA(cudaMalloc(&p, (size_t)Mpad * Mpad * 8));
    GPX_CUDA(cudaMalloc(&s->vec, (size_t)(8 + 64) * s->P * Mpad * 8));
  }
  if (!s->svm[0]) {
    for (auto& p : s->svm) GPX_CUDA(cudaMalloc(&p, (size_t)Mpad * Mpad * 8));
    GPX_CUDA(cudaMalloc(&s->svv, (size_t)SV_MV * Mpad * 8));
  }
  if (!s->red) {
    GPX_CUDA(cudaMalloc(&s->red, 4096 * 8));
    GPX_CUDA(cudaMallocHost(&s->h_red, 4096 * 8));
  }
  if (!s->cK) { GPX_CHECK(gpx_create(c->device, &s->cK)); GPX_CHECK(gpx_create(c->device, &s->cB)); }
  for (gpx_ctx* ch : {s->cK, s->cB})
    if (ch->NB != c->NB) GPX_CHECK(gpx_set_option(ch, "nb", c->NB));
  const long L = (nb + TILE - 1) / TILE * TILE;   // the batch's padded rows
  if (L > s->sv_cap) {
    GPX_CUDA(cudaStreamSynchronize(st));
    if (s->svb) cudaFree(s->svb);
    s->svb = nullptr;
    s->sv_cap = 0;
    if (cudaMalloc(&s->svb, sv_batch_doubles(Mpad, L) * 8) != cudaSuccess) {
      cudaGetLastError();
      gpx::set_error("gpx_svgp_begin: out of device memory for the batch buffers (" +
                     std::to_string(sv_batch_doubles(Mpad, L) * 8) + " bytes)");
      return -1;
    }
    s->sv_cap = L;
  }
  s->sv_row0 = row0;
  s->sv_nb = nb;
  const SvBatch b = sv_batch(s);
  // q_L^T and q_L live in svm[6..7], which no other entry writes (gpx_sparse_get uses mm[3] as scratch)
  double *Kd = s->mm[0], *Um = s->mm[1], *Lmi = s->mm[2], *QLt = s->svm[6], *QL = s->svm[7], *Wt = s->mm[5];
  double *vm = s->svv + (size_t)SV_M * Mpad, *lmm = s->svv + (size_t)SV_LMM * Mpad;
  // inputs: Z, m, q_L^T (q_L row-major read as column-major) and q_L (its transpose on the device)
  GPX_CUDA(cudaMemcpyAsync(s->Z, Z, (size_t)M * D * 8, cudaMemcpyHostToDevice, st));
  GPX_CUDA(cudaMemsetAsync(vm, 0, (size_t)Mpad * 8, st));
  GPX_CUDA(cudaMemcpyAsync(vm, q_m, (size_t)M * 8, cudaMemcpyHostToDevice, st));
  GPX_CUDA(cudaMemsetAsync(QLt, 0, (size_t)Mpad * Mpad * 8, st));
  GPX_CUDA(cudaMemcpy2DAsync(QLt, Mpad * 8, q_L, M * 8, M * 8, M, cudaMemcpyHostToDevice, st));
  GPX_CHECK(launch_transpose_pad(QLt, Mpad, (int)Mpad, Mpad, QL, st));
  GPX_CHECK(launched(c));
  // prepared points: Z and the batch rows of X
  GPX_CHECK(prep_points(c, mk, s->Z, M, D, Mpad, s->ZsT, s->sqZ));
  GPX_CHECK(prep_points(c, mk, s->X + (size_t)row0 * D, nb, D, L, b.x.xT, b.x.sq));
  GPX_CHECK(launched(c, 2));
  // Kmm and Lm = jitchol(Kmm) with logdet Kmm (svgp.py:38-42)
  GPX_CHECK(build_Kmm(c, Kd));
  double logdetK = 0.0, jit = 0.0;
  *jitter_used = 0.0;
  const int rc = factor_child(c, s->cK, Kd, 0.0, &logdetK, Um, Lmi, &jit, max_tries);
  if (rc) return rc;
  c->stats.tries = s->cK->stats.tries;
  s->jitter = 0.0;   // the posterior's K is Kmm itself (svgp.py:118); Lm (gpx_sparse_get(3)) carries the ladder's jitter
  s->sv_jit = jit;
  *jitter_used = jit;
  // Knm (N-major) and Kmn (M-major) of the batch, zero padded
  GPX_CUDA(cudaMemsetAsync(b.b[0], 0, (size_t)L * Mpad * 8, st));
  GPX_CUDA(cudaMemsetAsync(b.b[1], 0, (size_t)Mpad * L * 8, st));
  GPX_CHECK(build_K(c, mk, D, b.x, s->zpts(), b.b[0], L));
  GPX_CHECK(build_K(c, mk, D, s->zpts(), b.x, b.b[1], Mpad));
  GPX_CHECK(launched(c, 2));
  GPX_CHECK(gemm_nt(c, b.b[0], L, Lmi, Mpad, b.b[2], L, L, Mpad, Mpad, 1, 1));      // Vt = Knm Lmi^T
  GPX_CHECK(gemm_nt(c, Um, Mpad, b.b[2], L, b.b[3], Mpad, Mpad, L, Mpad, 1, 0));    // A = Um Vt^T
  GPX_CHECK(mm_nt(c, QLt, Lmi, Wt));                                                // Wt = q_L^T Um
  GPX_CHECK(gemm_nt(c, Wt, Mpad, b.b[2], L, b.b[0], Mpad, Mpad, L, Mpad, 1, 0));    // Bq = q_L^T A (Knm is done)
  svgp_marg_kernel<<<(unsigned)((nb + 7) / 8), 256, 0, st>>>(b.b[3], b.b[1], b.b[0], Mpad, M, nb, vm, kdiag,
                                                             b.vec[SB_MU], b.vec[SB_V]);
  GPX_CHECK(launched(c));
  // KL (svgp.py:55): Kmm^-1 m = Lmi^T (Lmi m) (the woodbury vector, into Cm), tr(Kmm^-1 S) = |Wt|_F^2
  GPX_CHECK(launch_col_dot(Um, Mpad, M, M, 1, vm, Mpad, lmm, Mpad, st));            // Lmi m = Um^T m
  GPX_CHECK(launch_col_dot(Lmi, Mpad, M, M, 1, lmm, Mpad, s->Cm, Mpad, st));        // Kmm^-1 m = Lmi^T (Lmi m)
  trace_dot_kernel<<<SV_RB, 256, 0, st>>>(Wt, Wt, Mpad, M, s->red);
  GPX_CHECK(launched(c, 3));
  std::vector<double> kim((size_t)M);
  GPX_CUDA(cudaMemcpyAsync(kim.data(), s->Cm, (size_t)M * 8, cudaMemcpyDeviceToHost, st));
  GPX_CUDA(cudaMemcpyAsync(s->h_red, s->red, 2 * SV_RB * 8, cudaMemcpyDeviceToHost, st));
  GPX_CUDA(cudaMemcpyAsync(mu, b.vec[SB_MU], (size_t)nb * 8, cudaMemcpyDeviceToHost, st));
  GPX_CUDA(cudaMemcpyAsync(var, b.vec[SB_V], (size_t)nb * 8, cudaMemcpyDeviceToHost, st));
  GPX_CHECK(svgp_end(c, "gpx_svgp_begin"));
  double logdetS = 0.0, trKS = 0.0, mKm = 0.0;
  for (long i = 0; i < M; i++) logdetS += log(fabs(q_L[i * M + i]));
  logdetS *= 2.0;
  for (int r = 0; r < SV_RB; r++) trKS += s->h_red[2 * r + 1];
  for (long i = 0; i < M; i++) mKm += q_m[i] * kim[(size_t)i];
  *kl = -0.5 * logdetS - 0.5 * (double)M + 0.5 * logdetK + 0.5 * trKS + 0.5 * mKm;
  s->sv_begun = true;
  return 0;
}

int gpx_svgp_finish(gpx_ctx* c, const double* dF_dmu, const double* dF_dv, double* grad, double* dZ, double* dL_dm,
                    double* dL_dchol) {
  if (!c || !dF_dmu || !dF_dv || !grad || !dZ || !dL_dm || !dL_dchol) GPX_FAIL("null argument");
  if (!c->sparse || !c->sparse->sv_begun) GPX_FAIL("gpx_svgp_begin has not been called on this data, kernel and Z");
  GPX_CUDA(cudaSetDevice(c->device));
  SparseState* s = c->sparse;
  cudaStream_t st = c->st;
  const long Mpad = s->Mpad, M = s->M, nb = s->sv_nb;
  const int D = s->D;
  const SvBatch b = sv_batch(s);
  const long L = b.x.ld;
  double *Kd = s->mm[0], *Um = s->mm[1], *Lmi = s->mm[2], *QLt = s->svm[6], *QL = s->svm[7], *Ki = s->mm[5], *S = s->mm[6],
         *Tt = s->mm[7], *AdvA = s->mm[8], *W = s->mm[9];
  double *R = s->svm[0], *KSK = s->svm[1], *G = s->svm[2], *GU = s->svm[3], *Eh = s->svm[4], *H = s->svm[5];
  double *admu = s->svv + (size_t)SV_ADMU * Mpad, *rpart = s->svv + (size_t)SV_RPART * Mpad;
  s->have_eval = s->dl_ready = s->w_ready = s->w_own = false;
  GPX_CUDA(cudaMemsetAsync(b.vec[SB_DMU], 0, (size_t)2 * s->sv_cap * 8, st));
  GPX_CUDA(cudaMemcpyAsync(b.vec[SB_DMU], dF_dmu, (size_t)nb * 8, cudaMemcpyHostToDevice, st));
  GPX_CUDA(cudaMemcpyAsync(b.vec[SB_DV], dF_dv, (size_t)nb * 8, cudaMemcpyHostToDevice, st));
  GPX_CHECK(binv(c, Um, Ki));                                                        // Kmm^-1 = Um Um^T
  GPX_CHECK(binv(c, QL, S));                                                         // S = q_L q_L^T
  GPX_CHECK(mm_nt(c, Ki, S, Tt));                                                    // Tt = Kmm^-1 S = T^T
  svgp_scale_kernel<<<(unsigned)((Mpad * L + 255) / 256), 256, 0, st>>>(b.b[3], Mpad, Mpad * L, 0, b.vec[SB_DV], b.b[0]);
  svgp_scale_kernel<<<(unsigned)((Mpad * L + 255) / 256), 256, 0, st>>>(b.b[2], L, Mpad * L, 1, b.vec[SB_DV], b.b[1]);
  GPX_CHECK(launched(c, 2));
  GPX_CHECK(gemm_nt(c, b.b[0], Mpad, b.b[3], Mpad, AdvA, Mpad, Mpad, Mpad, L, 2, 0));   // AdvA = Adv A^T, lower tiles
  mirror_tiles_kernel<<<dim3((unsigned)((Mpad + 255) / 256), (unsigned)Mpad), 256, 0, st>>>(AdvA, Mpad, Mpad);
  GPX_CHECK(launched(c));
  GPX_CHECK(launch_row_dot(b.b[3], Mpad, Mpad, nb, 1, b.vec[SB_DMU], L, 64, rpart, admu, st));   // Admu = A dF_dmu
  GPX_CHECK(launched(c, 2));
  GPX_CHECK(mm_nt(c, AdvA, Tt, R));                                                  // R = AdvA S Kmm^-1
  GPX_CHECK(mm_nt(c, Tt, Ki, KSK));                                                  // KSK = Kmm^-1 S Kmm^-1
  svgp_dkmm_kernel<<<dim3((unsigned)((Mpad + 255) / 256), (unsigned)Mpad), 256, 0, st>>>(AdvA, R, Ki, KSK, admu, s->Cm,
                                                                                         Mpad, M, Kd);
  GPX_CHECK(launched(c));
  // dL_dKmn^T = 2 (Tt - I) Adv = (2 (Tt - I) Um) Vd^T, into the Adv buffer (AdvA is formed)
  GPX_CHECK(combine(c, G, Mpad, 2.0, Tt, 0.0, nullptr, -2.0));
  GPX_CHECK(mm_nt(c, G, Lmi, GU));                                                   // GU = G Um
  GPX_CHECK(gemm_nt(c, GU, Mpad, b.b[1], L, b.b[0], Mpad, Mpad, L, Mpad, 1, 0));
  // dL_dchol and the posterior's woodbury_inv
  GPX_CHECK(combine(c, Eh, Mpad, 1.0, AdvA, -0.5, Ki, 0.0));
  GPX_CHECK(mm_nt(c, Eh, QLt, H));                                                   // H = (AdvA - Ki / 2) q_L
  svgp_dchol_kernel<<<dim3((unsigned)((M + 255) / 256), (unsigned)M), 256, 0, st>>>(H, QLt, Mpad, M, Eh);
  GPX_CHECK(launched(c));
  // woodbury_inv = Lm^-T Lm^-1 (Kmm - S) Lm^-T Lm^-1 (posterior.py:187-191 with K = Kmm and K_chol = Lm): Ki - KSK, less
  // j Ki^2 when the ladder factored Kmm + j I (Ki Kmm Ki = Ki - j Ki Ki)
  GPX_CUDA(cudaMemsetAsync(W, 0, (size_t)Mpad * Mpad * 8, st));
  if (s->sv_jit > 0.0) {
    GPX_CHECK(mm_nt(c, Ki, Ki, R));                                                  // R is free: Ki Ki
    GPX_CHECK(combine(c, W, M, 1.0, Ki, -s->sv_jit, R, 0.0));
    GPX_CHECK(combine(c, W, M, 1.0, W, -1.0, KSK, 0.0));
  } else {
    GPX_CHECK(combine(c, W, M, 1.0, Ki, -1.0, KSK, 0.0));
  }
  std::vector<double> hadmu((size_t)M), hkim((size_t)M);
  GPX_CUDA(cudaMemcpyAsync(dL_dchol, Eh, (size_t)M * M * 8, cudaMemcpyDeviceToHost, st));
  GPX_CUDA(cudaMemcpyAsync(hadmu.data(), admu, (size_t)M * 8, cudaMemcpyDeviceToHost, st));
  GPX_CUDA(cudaMemcpyAsync(hkim.data(), s->Cm, (size_t)M * 8, cudaMemcpyDeviceToHost, st));
  // the kernel's gradient block: the Kmn reductions with the rank-1 term Kmm^-1 m dF_dmu^T, then the Kmm ones
  const int ngk = kern_ngrad(s->mk);
  std::vector<double> g_knm(ngk, 0.0), g_kmm(ngk, 0.0), hz((size_t)M * D);
  GPX_CHECK(knm_reduce_at(c, b.x, b.b[0], b.vec[SB_DMU], L, g_knm.data(), dZ));
  const GradFullParams gk = grad_params(s->mk, D, s->zpts(), s->zpts(), Kd, Mpad);
  GPX_CHECK(ensure_part(s, grad_full_doubles(s->mk, D, gk) * 8));
  GPX_CHECK(grad_full_sum(c, s->mk, D, gk, s->part, g_kmm.data()));
  GPX_CHECK(ensure_part(s, grad_X_doubles(c, s->mk, gk, D) * 8));
  GPX_CHECK(grad_X(c, s->mk, gk, D, s->part, hz.data()));
  GPX_CHECK(svgp_end(c, "gpx_svgp_finish"));
  for (size_t i = 0; i < hz.size(); i++) dZ[i] += hz[i];
  double ddiag = 0.0;   // dL_dKdiag = dF_dv through update_gradients_diag (core/svgp.py:60)
  for (long n = 0; n < nb; n++) ddiag += dF_dv[n];
  kern_grads(s, ddiag, g_knm, g_kmm, grad);
  for (long i = 0; i < M; i++) dL_dm[i] = hadmu[(size_t)i] - hkim[(size_t)i];   // dF_dm - dKL_dm (:97,116)
  s->w_ready = s->w_own = true;
  s->have_eval = true;
  return 0;
}

}  // extern "C"

extern "C" {

/* gradients_X(dL_dKnm, X, Z) of the last VarDTC evaluation's kernel at its data points (sparse_gplvm.py:34), reduced from
 * the dL_dKnm^T the evaluation left on the device: rows = data points, columns = inducing points, read untransposed with
 * its rank-P term added as the evaluation's dL/dZ reduction added it. Launches: 2. */
int gpx_sparse_grad_X(gpx_ctx* c, double* dX) {
  if (!c || !dX) GPX_FAIL("null argument");
  if (c->dist) GPX_FAIL("the sparse input gradient is single-GPU");
  if (!c->sparse || !c->sparse->dl_ready)
    GPX_FAIL("no VarDTC evaluation whose dL_dKnm is still on the device (gpx_sparse_eval, _het or _multi first)");
  GPX_CUDA(cudaSetDevice(c->device));
  SparseState* s = c->sparse;
  GradFullParams gp = grad_params(s->mk, s->D, s->xpts(), s->zpts(), s->dLt, s->Mpad);
  gp.ci = s->Yb; gp.ldci = s->Npad; gp.cj = s->Cm; gp.ldcj = s->Mpad; gp.cP = rank_p_cols(s);
  GPX_CHECK(ensure_part(s, grad_X_doubles(c, s->mk, gp, s->D) * 8));
  return grad_X(c, s->mk, gp, s->D, s->part, dX);
}

}  // extern "C"
