// gpx_laplace.cu — the Laplace approximation for non-Gaussian likelihoods on the device (GPy's Laplace,
// GPy/inference/latent_function_inference/laplace.py:122-353), for one output column and no mean function.
//
// The likelihood's per-point quantities (W, its derivatives, the gradient terms of its parameters) are O(N) and come from the
// caller; everything N^2 and N^3 runs here:
//   gpx_laplace_begin  : K(X, X) of the kernel into a buffer kept for the whole evaluation (lapK, zero padded)
//   gpx_laplace_matvec : f = K v
//   gpx_laplace_newton : B = I + W^1/2 K W^1/2 from lapK, factored with jitchol's ladder by the DMMA sweep (S: lower L_B,
//                        upper U_B = L_B^-T), a = b - W^1/2 U_B U_B^T W^1/2 K b, dKi_f = a - Ki_f, Kd = K dKi_f
//   gpx_laplace_finish : the same factor at the mode, U~ = diag(W^1/2) U_B in place (so that U~ U~^T = K_Wi_i and the exact
//                        posterior's consumers read it where they read U), C = U~^T K on the DMMA GEMM for diag(Ki_W_i),
//                        K_Wi_i by the plain LAUUM, v = (I - K_Wi_i K) dL_dfhat, and the kernel gradient from
//                        K_Wi_i + v v^T with alpha' = Ki_f + v through grad_kinv_multi_kernel, one launch per part.
// Every reduction has a fixed order: a result does not depend on the launch configuration.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "gpx_common.cuh"
#include "gpx_ctx.cuh"
#include "gpx_kernels.cuh"

namespace gpx {

// vectors of lapV ([LAP_NV][Npad], zero padded)
enum { LV_W = 0, LV_SW, LV_B, LV_KIF, LV_DWDF, LV_T1, LV_Y, LV_U, LV_A, LV_D, LV_KD, LV_CSQ, LV_DIAG, LV_DLDF, LV_V,
       LV_AP, LV_KV, LAP_NV };
// the small vector glue, one thread per entry i < n (entries N <= i < n are zero on output)
enum { LG_SQRTW = 0, LG_MULW = 1, LG_NEWTON = 2, LG_DIAG = 3, LG_V = 4 };

__global__ void __launch_bounds__(256) laplace_vec_kernel(int mode, long N, long n, const double* __restrict__ w,
                                                          const double* __restrict__ x, const double* __restrict__ y,
                                                          const double* __restrict__ z, const double* __restrict__ K,
                                                          long ldk, double* __restrict__ o1, double* __restrict__ o2) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const bool in = i < N;
  switch (mode) {
    case LG_SQRTW: o1[i] = in ? sqrt(x[i]) : 0.0; break;                        // W_12 = sqrt(W) (laplace.py:328)
    case LG_MULW: o1[i] = in ? w[i] * x[i] : 0.0; break;
    case LG_NEWTON: {                                                            // :196-199
      const double a = in ? x[i] - w[i] * y[i] : 0.0;
      o1[i] = a;
      o2[i] = in ? a - z[i] : 0.0;
      break;
    }
    case LG_DIAG: {                                                              // :347-348, :258
      const double d = in ? K[i + i * ldk] - x[i] : 0.0;
      o1[i] = d;
      o2[i] = in ? -0.5 * (d * y[i]) : 0.0;
      break;
    }
    default: {                                                                   // v = (I - K_Wi_i K) dL_dfhat, a + v
      const double v = in ? x[i] - y[i] : 0.0;
      o1[i] = v;
      o2[i] = in ? z[i] + v : 0.0;
    }
  }
}

// B = I + (w_i K_ij) w_j (+ jitter on the diagonal) into the factor workspace form (lower tiles, zero upper tiles, identity
// padding), laplace.py:329
__global__ void __launch_bounds__(256) laplace_bbuild_kernel(const double* __restrict__ K, long ld, const double* __restrict__ w,
                                                             long N, double* __restrict__ S, double jitter) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ld) return;
  for (long j = blockIdx.y; j < ld; j += gridDim.y) {
    double v;
    if (i >= N || j >= N) v = (i == j) ? 1.0 : 0.0;
    else if (i / TILE < j / TILE) v = 0.0;
    else {
      v = (w[i] * K[i + j * ld]) * w[j];
      if (i == j) v = (1.0 + v) + jitter;
    }
    S[i + j * ld] = v;
  }
}

// U~ = diag(w) U_B in place (every row of the upper and diagonal tiles of S; the diagonal tiles hold zeros below their
// diagonal) and Li = U~^T = L_B^-1 diag(w) (laplace.py:331, LiW12), column-major with leading dimension ld, zero above the
// diagonal and outside N x N. 32 x 32 tiles through shared memory, so that both sides are coalesced.
__global__ void __launch_bounds__(256) laplace_scale_u_kernel(double* __restrict__ S, long ld, const double* __restrict__ w,
                                                              long N, double* __restrict__ Li) {
  __shared__ double t[32][33];
  const long r0 = (long)blockIdx.x * 32, c0 = (long)blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int k = ty; k < 32; k += 8) {
    const long r = r0 + tx, c = c0 + k;
    double v = 0.0;
    if (r / TILE <= c / TILE) {
      v = S[r + c * ld] * w[r];
      S[r + c * ld] = v;
    }
    t[k][tx] = (r <= c && c < N) ? v : 0.0;
  }
  __syncthreads();
  for (int k = ty; k < 32; k += 8) Li[(c0 + tx) + (r0 + k) * ld] = t[tx][k];
}

// A += v v^T over the lower tiles (whole diagonal tiles) of a stored symmetric matrix, inside N x N
__global__ void __launch_bounds__(256) laplace_rank1_kernel(double* __restrict__ A, long ld, const double* __restrict__ v,
                                                            long N) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const double vi = v[i];
  for (long j = blockIdx.y; j < N && j / TILE <= i / TILE; j += gridDim.y) A[i + j * ld] = fma(vi, v[j], A[i + j * ld]);
}

static unsigned lap_grid_y(long n) { return (unsigned)std::max<long>(1, std::min<long>(n, 65535)); }

void laplace_release(gpx_ctx* c) {
  for (double** p : {&c->lapK, &c->lapV}) { if (*p) cudaFree(*p); *p = nullptr; }
  c->lap_cap = 0;
  c->lap_begun = c->lap_post = false;
}

void laplace_free(gpx_ctx* c) {
  laplace_release(c);
  for (auto e : c->lap_ev) cudaEventDestroy(e);
  c->lap_ev.clear();
}

}  // namespace gpx

using namespace gpx;

namespace {

double* lv(gpx_ctx* c, int k) { return c->lapV + (size_t)k * c->Npad; }

int vec(gpx_ctx* c, int mode, const double* w, const double* x, const double* y, const double* z, double* o1,
        double* o2 = nullptr, const double* K = nullptr) {
  laplace_vec_kernel<<<(unsigned)((c->Npad + 255) / 256), 256, 0, c->st>>>(mode, c->N, c->Npad, w, x, y, z, K, c->Npad, o1,
                                                                          o2);
  c->eval_launches++;
  GPX_CUDA(cudaGetLastError());
  return 0;
}

// out = K x over the kept K (zero padded: rows >= N give 0): one partial per row tile and column chunk, fixed-order sum
int kmv(gpx_ctx* c, const double* x, double* out) {
  GPX_CHECK(launch_row_dot(c->lapK, c->Npad, c->Npad, c->N, 1, x, c->Npad, KSPLIT, c->dUvPart, out, c->st));
  c->eval_launches += 2;
  return 0;
}

// out = U (U^T x) with the factor in S. Before the scaling of gpx_laplace_finish U = U_B and x = w o K b gives
// W^1/2 B^-1 W^1/2 K b without its last w (laplace.py:194); after it U = U~ and out = K_Wi_i x (:262)
int uut_mv(gpx_ctx* c, const double* x, double* out) {
  GPX_CHECK(launch_utv(c->S, c->Npad, c->Npad, 1, x, c->dT, c->st));
  GPX_CHECK(launch_uv(c->S, c->Npad, c->Npad, 1, c->dT, KSPLIT, c->dUvPart, out, c->st));
  c->eval_launches += 3;
  return 0;
}

int upload(gpx_ctx* c, int slot, const double* h) {
  GPX_CUDA(cudaMemcpyAsync(lv(c, slot), h, (size_t)c->N * 8, cudaMemcpyHostToDevice, c->st));
  return 0;
}

// per-phase events of one call (timed when the "profile" option is on)
struct LapTimer {
  gpx_ctx* c;
  size_t n = 0;
  std::vector<int> phase;   // phase of the span that ends at mark k (k >= 1)
  int mark(int ph) {
    if (!c->profile && ph >= 0) return 0;
    while (c->lap_ev.size() <= n) {
      cudaEvent_t e;
      GPX_CUDA(cudaEventCreate(&e));
      c->lap_ev.push_back(e);
    }
    GPX_CUDA(cudaEventRecord(c->lap_ev[n], c->st));
    phase.push_back(ph);
    n++;
    return 0;
  }
  // after the stream is synchronised: span k-1 -> k is added to the field of phase[k]
  void finish(gpx_stats& s) {
    for (size_t k = 1; k < n; k++) {
      float ms = 0;
      cudaEventElapsedTime(&ms, c->lap_ev[k - 1], c->lap_ev[k]);
      switch (phase[k]) {
        case 0: s.kbuild_ms += ms; break;
        case 1: s.sweep_ms += ms; break;
        case 2: s.update_ms += ms; break;
        case 3: s.lauum_ms += ms; break;
        case 4: s.solve_ms += ms; break;
        default: break;
      }
    }
    if (n >= 2) cudaEventElapsedTime(&s.total_ms, c->lap_ev[0], c->lap_ev[n - 1]);
  }
};
enum { PH_K = 0, PH_FACTOR = 1, PH_GEMM = 2, PH_LAUUM = 3, PH_MV = 4, PH_OTHER = 5 };

// the checks of gpx_laplace_newton / _finish
int lap_args(const gpx_ctx* c) {
  if (c->dist) GPX_FAIL("the Laplace approximation is single-GPU");
  if (!c->lap_begun) GPX_FAIL("gpx_laplace_begin has not been called on this data");
  return 0;
}

// the start of a call: counters, stats, the posterior of an earlier evaluation is gone (S is overwritten)
void lap_start(gpx_ctx* c) {
  c->have_eval = false;
  c->have_kinv = false;
  c->lap_post = false;
  memset(&c->stats, 0, sizeof(c->stats));
  c->eval_launches = 0;
}

// B = I + W^1/2 K W^1/2 factored with jitchol's ladder (GPy/util/linalg.py:56-75): first as it is, then with mean(diag B)
// 1e-6 10^k added, k < max_tries. w = sqrt(W) is in LV_SW, W (host) gives the mean of B's diagonal. -> 0 or the failing minor
int lap_factor(gpx_ctx* c, const double* W, int max_tries, double* jitter_used) {
  const long ld = c->Npad, N = c->N;
  double extra = 0.0;
  int tries = 0, info = 0;
  for (;;) {
    tries++;
    GPX_CUDA(cudaMemsetAsync(c->info, 0, sizeof(int), c->st));
    laplace_bbuild_kernel<<<dim3((unsigned)((ld + 255) / 256), lap_grid_y(ld)), 256, 0, c->st>>>(c->lapK, ld, lv(c, LV_SW), N,
                                                                                                c->S, extra);
    c->eval_launches++;
    GPX_CUDA(cudaGetLastError());
    GPX_CHECK(sweep_workspace(c));
    GPX_CUDA(cudaMemcpyAsync(c->h_info, c->info, sizeof(int), cudaMemcpyDeviceToHost, c->st));
    GPX_CUDA(cudaStreamSynchronize(c->st));
    info = *c->h_info;
    if (info == 0) break;
    if (tries > max_tries) break;
    double dsum = 0.0;   // diag(B) = 1 + w_i K_ii w_i, K_ii = Kdiag
    for (long i = 0; i < N; i++) {
      const double s = std::sqrt(W[i]);
      dsum += 1.0 + (s * c->kdiag) * s;
    }
    extra = dsum / (double)N * 1e-6 * pow(10.0, tries - 1);
    if (!std::isfinite(extra)) break;
  }
  c->stats.tries = tries;
  c->jitter_extra = extra;
  *jitter_used = extra;
  if (info != 0) gpx::set_error("Laplace: B = I + W^1/2 K W^1/2 is not positive definite, even with jitter.");
  return info;
}

int lap_end(gpx_ctx* c, LapTimer& tm, int64_t l0) {
  GPX_CUDA(cudaStreamSynchronize(c->st));
  tm.finish(c->stats);
  c->total_launches += c->eval_launches;
  c->stats.launches = c->total_launches - l0;
  return 0;
}

}  // namespace

extern "C" {

int gpx_laplace_begin(gpx_ctx* c, const gpx_kern_part* parts, int nparts) {
  if (!c || !parts) GPX_FAIL("null argument");
  if (!c->S) GPX_FAIL("gpx_set_data has not been called");
  if (c->dist) GPX_FAIL("the Laplace approximation is single-GPU");
  if (c->P != 1) GPX_FAIL("the Laplace approximation takes one output column (P = 1)");
  MultiKern mk;
  double kdiag;
  GPX_CHECK(fill_mk(mk, parts, nparts, c->D, &kdiag));
  GPX_CUDA(cudaSetDevice(c->device));
  lap_start(c);
  c->lap_begun = false;
  c->het = false;
  const long ld = c->Npad;
  if (c->lap_cap != ld) {
    for (double** p : {&c->lapK, &c->lapV}) { if (*p) cudaFree(*p); *p = nullptr; }
    c->lap_cap = 0;
    GPX_CUDA(cudaMalloc(&c->lapK, (size_t)ld * ld * 8));
    GPX_CUDA(cudaMalloc(&c->lapV, (size_t)LAP_NV * ld * 8));
    c->lap_cap = ld;
  }
  if (mk.sumD > c->rows_cap || mk.nparts > c->norm_cap) {   // a composite that stacks more rows than D and 1
    for (double** p : {&c->dXsT, &c->dsq}) { if (*p) cudaFree(*p); *p = nullptr; }
    c->rows_cap = std::max(c->rows_cap, mk.sumD); c->norm_cap = std::max(c->norm_cap, mk.nparts);
    GPX_CUDA(cudaMalloc(&c->dXsT, (size_t)c->rows_cap * ld * 8));
    GPX_CUDA(cudaMalloc(&c->dsq, (size_t)c->norm_cap * ld * 8));
  }
  c->mk = mk;
  c->kdiag = kdiag;
  c->noise = c->jitter = c->jitter_extra = 0.0;
  const int64_t l0 = c->total_launches;
  LapTimer tm{c};
  GPX_CHECK(tm.mark(-1));
  GPX_CUDA(cudaMemsetAsync(c->lapK, 0, (size_t)ld * ld * 8, c->st));
  GPX_CUDA(cudaMemsetAsync(c->lapV, 0, (size_t)LAP_NV * ld * 8, c->st));
  const Points tr = train_points(c);
  GPX_CHECK(prep_points(c, mk, c->dX, c->N, c->D, ld, tr.xT, tr.sq));
  GPX_CHECK(build_K(c, mk, c->D, tr, tr, c->lapK, ld));
  c->eval_launches += 2;
  GPX_CHECK(tm.mark(PH_K));
  GPX_CHECK(lap_end(c, tm, l0));
  c->stats.kbuild_bytes = 8.0 * (double)c->N * c->N + 8.0 * (double)c->N * c->D;
  c->lap_begun = true;
  return 0;
}

int gpx_laplace_matvec(gpx_ctx* c, const double* v, double* Kv) {
  if (!c || !v || !Kv) GPX_FAIL("null argument");
  GPX_CHECK(lap_args(c));
  GPX_CUDA(cudaSetDevice(c->device));
  c->eval_launches = 0;
  GPX_CHECK(upload(c, LV_T1, v));
  GPX_CHECK(kmv(c, lv(c, LV_T1), lv(c, LV_KV)));
  GPX_CUDA(cudaMemcpyAsync(Kv, lv(c, LV_KV), (size_t)c->N * 8, cudaMemcpyDeviceToHost, c->st));
  if (cudaStreamSynchronize(c->st) != cudaSuccess) GPX_FAIL_DEVICE("gpx_laplace_matvec");
  c->total_launches += c->eval_launches;
  return 0;
}

int gpx_laplace_newton(gpx_ctx* c, const double* W, const double* b, const double* Ki_f, int max_tries, double* dKi_f,
                       double* Kd, double* jitter_used) {
  if (!c || !W || !b || !Ki_f || !dKi_f || !Kd || !jitter_used) GPX_FAIL("null argument");
  GPX_CHECK(lap_args(c));
  GPX_CUDA(cudaSetDevice(c->device));
  lap_start(c);
  const int64_t l0 = c->total_launches;
  LapTimer tm{c};
  GPX_CHECK(tm.mark(-1));
  GPX_CHECK(upload(c, LV_W, W));
  GPX_CHECK(upload(c, LV_B, b));
  GPX_CHECK(upload(c, LV_KIF, Ki_f));
  GPX_CHECK(vec(c, LG_SQRTW, nullptr, lv(c, LV_W), nullptr, nullptr, lv(c, LV_SW)));
  const int info = lap_factor(c, W, max_tries, jitter_used);
  if (info) { lap_end(c, tm, l0); return info; }
  GPX_CHECK(tm.mark(PH_FACTOR));
  GPX_CHECK(kmv(c, lv(c, LV_B), lv(c, LV_T1)));                                  // K b
  GPX_CHECK(vec(c, LG_MULW, lv(c, LV_SW), lv(c, LV_T1), nullptr, nullptr, lv(c, LV_Y)));
  GPX_CHECK(uut_mv(c, lv(c, LV_Y), lv(c, LV_U)));                                // W^1/2 B^-1 W^1/2 K b, without the w
  GPX_CHECK(vec(c, LG_NEWTON, lv(c, LV_SW), lv(c, LV_B), lv(c, LV_U), lv(c, LV_KIF), lv(c, LV_A), lv(c, LV_D)));
  GPX_CHECK(kmv(c, lv(c, LV_D), lv(c, LV_KD)));                                  // K dKi_f
  GPX_CHECK(tm.mark(PH_MV));
  GPX_CUDA(cudaMemcpyAsync(dKi_f, lv(c, LV_D), (size_t)c->N * 8, cudaMemcpyDeviceToHost, c->st));
  GPX_CUDA(cudaMemcpyAsync(Kd, lv(c, LV_KD), (size_t)c->N * 8, cudaMemcpyDeviceToHost, c->st));
  return lap_end(c, tm, l0);
}

int gpx_laplace_finish(gpx_ctx* c, const double* W, const double* Ki_f, const double* dW_df, int nlik,
                       const double* dlik_grad_dthetaL, int max_tries, double* logdet_I_KW, double* diag_Ki_W_i,
                       double* kgrad, double* dL_dthetaL_imp, double* jitter_used) {
  if (!c || !W || !Ki_f || !dW_df || !logdet_I_KW || !diag_Ki_W_i || !kgrad || !jitter_used) GPX_FAIL("null argument");
  if (nlik < 0) GPX_FAIL("nlik must be non-negative");
  if (nlik > 0 && (!dlik_grad_dthetaL || !dL_dthetaL_imp)) GPX_FAIL("null argument (nlik > 0)");
  GPX_CHECK(lap_args(c));
  GPX_CUDA(cudaSetDevice(c->device));
  lap_start(c);
  cudaStream_t st = c->st;
  const long ld = c->Npad, N = c->N;
  const int nt = (int)(ld / TILE);
  const MultiKern& mk = c->mk;
  size_t need = 0;   // the parts' reduction partials
  for (int q = 0; q < mk.nparts; q++) need += (size_t)nt * nt * part_nred(mk.part[q]);
  if (need > c->mpart_cap) {
    if (c->mpartials) cudaFree(c->mpartials);
    c->mpartials = nullptr;
    c->mpart_cap = 0;
    GPX_CUDA(cudaMalloc(&c->mpartials, need * 8));
    c->mpart_cap = need;
  }
  const int64_t l0 = c->total_launches;
  LapTimer tm{c};
  GPX_CHECK(tm.mark(-1));
  GPX_CHECK(upload(c, LV_W, W));
  GPX_CHECK(upload(c, LV_KIF, Ki_f));
  GPX_CHECK(upload(c, LV_DWDF, dW_df));
  GPX_CHECK(vec(c, LG_SQRTW, nullptr, lv(c, LV_W), nullptr, nullptr, lv(c, LV_SW)));
  // 1. B at the mode -> logdet_I_KW = 2 sum log diag(L_B) (laplace.py:352), per-tile partials summed in tile order
  const int info = lap_factor(c, W, max_tries, jitter_used);
  if (info) { lap_end(c, tm, l0); return info; }
  std::vector<double> ldp(nt);
  GPX_CUDA(cudaMemcpyAsync(ldp.data(), c->logdet_part, (size_t)nt * 8, cudaMemcpyDeviceToHost, st));
  GPX_CHECK(tm.mark(PH_FACTOR));
  // 2.-4. U~ = diag(w) U_B in place, Li = U~^T; alpha = Ki_f; C = Li K (A lower triangular): diag(Ki_W_i) = diag(K) - |C_:i|^2
  {
    TmpBuf Li(st), Cm(st);
    GPX_CHECK(Li.alloc((size_t)ld * ld));
    GPX_CHECK(Cm.alloc((size_t)ld * ld));
    GPX_CHECK(tm.mark(PH_OTHER));
    laplace_scale_u_kernel<<<dim3((unsigned)(ld / 32), (unsigned)(ld / 32)), 256, 0, st>>>(c->S, ld, lv(c, LV_SW), N, Li.p);
    c->eval_launches++;
    GPX_CUDA(cudaGetLastError());
    GPX_CUDA(cudaMemcpyAsync(c->dAlpha, lv(c, LV_KIF), (size_t)ld * 8, cudaMemcpyDeviceToDevice, st));
    GPX_CHECK(tm.mark(PH_OTHER));
    GPX_CHECK(gemm_nt(c, Li.p, ld, c->lapK, ld, Cm.p, ld, ld, ld, ld, 1, 2));
    GPX_CHECK(tm.mark(PH_GEMM));
    Li.release();
    GPX_CHECK(launch_col_sqnorm(Cm.p, ld, ld, N, lv(c, LV_CSQ), st));
    c->eval_launches++;
  }
  // 5. dL_dfhat = -1/2 diag(Ki_W_i) o dW_df (:258)
  GPX_CHECK(vec(c, LG_DIAG, nullptr, lv(c, LV_CSQ), lv(c, LV_DWDF), nullptr, lv(c, LV_DIAG), lv(c, LV_DLDF), c->lapK));
  GPX_CHECK(tm.mark(PH_OTHER));
  // 6. K_Wi_i = U~ U~^T into the lower tiles of c->Kinv (:332)
  GPX_CHECK(lauum_store(c));
  GPX_CHECK(tm.mark(PH_LAUUM));
  // 7. v = dL_dfhat - K_Wi_i K dL_dfhat (= I_KW_i^T dL_dfhat, :262,:271), alpha' = Ki_f + v; 8. K v
  GPX_CHECK(kmv(c, lv(c, LV_DLDF), lv(c, LV_T1)));
  GPX_CHECK(uut_mv(c, lv(c, LV_T1), lv(c, LV_U)));                               // U~ U~^T K dL_dfhat
  GPX_CHECK(vec(c, LG_V, nullptr, lv(c, LV_DLDF), lv(c, LV_U), lv(c, LV_KIF), lv(c, LV_V), lv(c, LV_AP)));
  GPX_CHECK(kmv(c, lv(c, LV_V), lv(c, LV_KV)));
  GPX_CHECK(tm.mark(PH_MV));
  // the kernel gradient: dL_dK's symmetric part 1/2 [(a + v)(a + v)^T - (K_Wi_i + v v^T)] (:267-272), one reduction per part
  laplace_rank1_kernel<<<dim3((unsigned)((N + 255) / 256), lap_grid_y(N)), 256, 0, st>>>(c->Kinv, ld, lv(c, LV_V), N);
  c->eval_launches++;
  GPX_CUDA(cudaGetLastError());
  size_t off = 0;
  for (int q = 0; q < mk.nparts; q++) {
    GPX_CUDA(cudaMemsetAsync(c->mpartials + off, 0, (size_t)nt * nt * part_nred(mk.part[q]) * 8, st));
    GradKinvMultiParams gm;
    memset(&gm, 0, sizeof(gm));
    gm.Kinv = c->Kinv; gm.ld = ld; gm.XsT = c->dXsT; gm.sq = c->dsq; gm.ldx = ld; gm.alpha = lv(c, LV_AP);
    gm.N = N; gm.P = 1; gm.nt = nt; gm.part = q; gm.want_noise = 0; gm.partials = c->mpartials + off; gm.mk = mk;
    GPX_CHECK(launch_grad_kinv_multi(gm, st));
    c->eval_launches++;
    off += (size_t)nt * nt * part_nred(mk.part[q]);
  }
  GPX_CHECK(tm.mark(PH_OTHER));
  std::vector<double> hp(off), kv((size_t)N);
  GPX_CUDA(cudaMemcpyAsync(hp.data(), c->mpartials, off * 8, cudaMemcpyDeviceToHost, st));
  GPX_CUDA(cudaMemcpyAsync(kv.data(), lv(c, LV_KV), (size_t)N * 8, cudaMemcpyDeviceToHost, st));
  GPX_CUDA(cudaMemcpyAsync(diag_Ki_W_i, lv(c, LV_DIAG), (size_t)N * 8, cudaMemcpyDeviceToHost, st));
  GPX_CHECK(lap_end(c, tm, l0));
  double s = 0.0;
  for (int i = 0; i < nt; i++) s += ldp[i];
  *logdet_I_KW = s;
  off = 0;
  int g = 0;
  for (int p = 0; p < mk.nparts; p++) {   // tile order, as grad_full_sum
    const int nred = part_nred(mk.part[p]);
    std::vector<double> tot(nred, 0.0);
    for (size_t t = 0; t < (size_t)nt * nt; t++)
      for (int q = 0; q < nred; q++) tot[q] += hp[off + t * nred + q];
    double v;
    for (int q = 0; q < nred; q++)
      if (part_grad_entry(mk, p, q, tot[q], &v)) kgrad[g + q] = v;
    g += part_ngrad(mk.part[p]);
    off += (size_t)nt * nt * nred;
  }
  // dL_dfhat^T I_KW_i K g_theta = (K v)^T g_theta (:293-295): one mat-vec for every likelihood parameter
  for (int t = 0; t < nlik; t++) {
    double d = 0.0;
    for (long i = 0; i < N; i++) d += kv[i] * dlik_grad_dthetaL[(size_t)t * N + i];
    dL_dthetaL_imp[t] = d;
  }
  c->have_eval = true;
  c->have_kinv = false;   // the stored matrix is K_Wi_i + v v^T: gpx_get(KINV) forms U~ U~^T again
  c->lap_post = true;
  return 0;
}

}  // extern "C"
