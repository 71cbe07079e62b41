// gpx_laplace.cu — the Laplace approximation for non-Gaussian likelihoods on the device (GPy's Laplace,
// GPy/inference/latent_function_inference/laplace.py:122-353), for one output column and no mean function, and expectation
// propagation for the probit Bernoulli likelihood on the same kept K (the second half of this file), and the variational
// Gaussian approximation for any likelihood on it (the last part).
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
#include "gpx_ep.cuh"
#include "gpx_kernels.cuh"

namespace gpx {

// vectors of lapV ([LAP_NV][Npad], zero padded)
enum { LV_W = 0, LV_SW, LV_B, LV_KIF, LV_DWDF, LV_T1, LV_Y, LV_U, LV_A, LV_D, LV_KD, LV_CSQ, LV_DIAG, LV_DLDF, LV_V,
       LV_AP, LV_KV,
       // expectation propagation: sites, their sign, cavities and moments, mu, diag(Sigma), diag(dL_dK)
       LV_TT, LV_VT, LV_SGN, LV_CT, LV_CV, LV_ZH, LV_MH, LV_S2, LV_MU, LV_SD, LV_DL, LAP_NV };
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
  for (double** p : {&c->lapK, &c->lapV, &c->epSig, &c->epBlk}) { if (*p) cudaFree(*p); *p = nullptr; }
  if (c->epOrd) cudaFree(c->epOrd);
  c->epOrd = nullptr;
  c->lap_cap = 0;
  c->lap_begun = c->lap_post = false;
  c->ep_begun = c->ep_ready = c->ep_full = c->ep_labels = false;
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
  c->vg_begun = c->vg_factored = false;
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
  c->ep_begun = c->ep_ready = false;
  c->het = false;
  const long ld = c->Npad;
  if (c->lap_cap != ld) {
    laplace_release(c);
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

// ==== expectation propagation (GPy/inference/latent_function_inference/expectation_propagation.py:187-434) ===============
// EP for the probit Bernoulli likelihood on the kept K of gpx_laplace_begin. A sequential sweep is a chain of N rank-1
// updates of Sigma (:101-105); it runs here in blocks of TILE sites of the update order: the block's chain on its TILE x TILE
// part G = Sigma[I, I] in one CTA (ep_chain_kernel), S = Sigma[:, I] (I + U)^-1 row by row (ep_solve_kernel, U[l, j] =
// c_l s_l[j] for l < j), then Sigma -= S diag(c) S^T as one rank-TILE update on the DMMA GEMM's GEMM_UPDATE mode and
// mu -= S g. That is the chain of rank-1 updates regrouped, not an approximation of it. _recompute (:129-143) is the Laplace
// factor with tau~ in place of W.
namespace gpx {

// W. J. Cody's rational approximations (Math. Comp. 23, 1969) in the form util/univariate_Gaussian.py:26-158 evaluates
// them, with its branch points: erfc for x / sqrt(2) >= 4 (P1, Q1), 0.469 <= x / sqrt(2) < 4 (P2, Q2), erf below (P3, Q3)
__constant__ double EP_P1[6] = {3.05326634961232344e-1, 3.60344899949804439e-1, 1.25781726111229246e-1,
                                1.60837851487422766e-2, 6.58749161529837803e-4, 1.63153871373020978e-2};
__constant__ double EP_Q1[5] = {2.56852019228982242e+0, 1.87295284992346047e+0, 5.27905102951428412e-1,
                                6.05183413124413191e-2, 2.33520497626869185e-3};
__constant__ double EP_P2[9] = {5.64188496988670089e-1, 8.88314979438837594e+0, 6.61191906371416295e+1,
                                2.98635138197400131e+2, 8.81952221241769090e+2, 1.71204761263407058e+3,
                                2.05107837782607147e+3, 1.23033935479799725e+3, 2.15311535474403846e-8};
__constant__ double EP_Q2[8] = {1.57449261107098347e+1, 1.17693950891312499e+2, 5.37181101862009858e+2,
                                1.62138957456669019e+3, 3.29079923573345963e+3, 4.36261909014324716e+3,
                                3.43936767414372164e+3, 1.23033935480374942e+3};
__constant__ double EP_P3[5] = {3.16112374387056560e+0, 1.13864154151050156e+2, 3.77485237685302021e+2,
                                3.20937758913846947e+3, 1.85777706184603153e-1};
__constant__ double EP_Q3[4] = {2.36012909523441209e+1, 2.44024637934444173e+2, 1.28261652607737228e+3,
                                2.84423683343917062e+3};
constexpr double EP_LIMIT1 = 0.6629, EP_LIMIT2 = 5.6569;
constexpr double EP_LN2PI = 1.83787706640934533908193770913, EP_LN2 = 0.69314718055994530941723212146;
constexpr double EP_SQRTPI = 1.77245385090551602729816748334, EP_SQRT2 = 1.41421356237309504880168872421;

__device__ __forceinline__ double ep_log_pdf(double z) { return -0.5 * (EP_LN2PI + z * z); }

__device__ double ep_erf_r3(double y) {   // _erfRationalHelperR3
  double nom = y * EP_P3[4], den = y;
  for (int i = 0; i <= 2; i++) {
    nom = (nom + EP_P3[i]) * y;
    den = (den + EP_Q3[i]) * y;
  }
  return (nom + EP_P3[3]) / (den + EP_Q3[3]);
}

__device__ double ep_erf_helper(double x) {   // _erfRationalHelper: Q(x), x > 0
  if (x >= EP_LIMIT2) {
    const double y = 2.0 / (x * x);
    double res = y * EP_P1[5], den = y;
    for (int i = 0; i <= 3; i++) {
      res = (res + EP_P1[i]) * y;
      den = (den + EP_Q1[i]) * y;
    }
    return 1.0 - EP_SQRTPI * y * (res + EP_P1[4]) / (den + EP_Q1[4]);
  }
  const double y = x / EP_SQRT2;
  double res = y * EP_P2[8], den = y;
  for (int i = 0; i <= 6; i++) {
    res = (res + EP_P2[i]) * y;
    den = (den + EP_Q2[i]) * y;
  }
  return EP_SQRTPI * y * (res + EP_P2[7]) / (den + EP_Q2[7]);
}

__device__ double ep_log_cdf(double z) {   // logCdfNormal
  if (fabs(z) < EP_LIMIT1) return log1p((z / EP_SQRT2) * ep_erf_r3(0.5 * z * z)) - EP_LN2;
  if (z < 0.0) return ep_log_pdf(z) - log(-z) + log(ep_erf_helper(-z));
  return log1p(-(exp(ep_log_pdf(z))) * ep_erf_helper(z) / z);
}

__device__ double ep_dlog_cdf(double z) {   // derivLogCdfNormal
  if (fabs(z) < EP_LIMIT1) return 2.0 * exp(ep_log_pdf(z)) / (1.0 + (z / EP_SQRT2) * ep_erf_r3(0.5 * z * z));
  if (z < 0.0) return -z / ep_erf_helper(-z);
  const double t = exp(ep_log_pdf(z));
  return t / (1.0 - t * ep_erf_helper(z) / z);
}

// site i of _local_updates (:333-351) at mu_i = mui: the cavity (:27-29) and the site update with tau~ clipped at machine
// epsilon (:52-68) read the diagonal the caller holds, Sd; the probit moments (bernoulli.py:59-92). -> the rank-1 update's
// c = dtau / (1 + dtau Sii) and g = c (mu_i + Sii dv) - dv (:101-105: mu -= g s, Sigma -= c s s^T) with Sii the diagonal of
// the Sigma being updated. Dense EP holds Sd = Sii; the DTC form holds a clipped copy (:149-156).
__device__ void ep_site(const EpSites& e, long i, double Sd, double Sii, double mui, double* c_out, double* g_out) {
  const double tau = 1.0 / Sd - e.eta * e.tt[i];
  const double v = mui / Sd - e.eta * e.vt[i];
  const double sgn = e.sgn[i];
  const double q = sqrt(tau * tau + tau);
  const double z = sgn * v / q;
  const double r = ep_dlog_cdf(z);
  const double lz = ep_log_cdf(z);
  const double mh = v / tau + sgn * r / q;
  const double s2 = 1.0 / tau - (r / (tau * tau + tau)) * (z + r);
  const double de = e.delta / e.eta;
  double dtau = de * (1.0 / s2 - 1.0 / Sd);
  const double dv = de * (mh / s2 - mui / Sd);
  const double prev = e.tt[i];
  double t = prev + dtau;
  if (t < 2.220446049250313e-16) {
    t = 2.220446049250313e-16;
    dtau = t - prev;
  }
  e.tt[i] = t;
  e.vt[i] += dv;
  e.ct[i] = tau; e.cv[i] = v; e.zh[i] = exp(lz); e.mh[i] = mh; e.s2[i] = s2;
  const double c = dtau / (1.0 + dtau * Sii);
  *c_out = c;
  *g_out = c * (mui + Sii * dv) - dv;
}

// Sigma(p, q) of the stored lower tiles (diagonal tiles whole)
__device__ __forceinline__ double ep_sym(const double* __restrict__ S, long ld, long p, long q) {
  return (p / TILE >= q / TILE) ? S[p + q * ld] : S[q + p * ld];
}

// the site chain of one block of m <= TILE sites I (one CTA): G = Sigma[I, I] (lower part, row-major in shared memory),
// mu_I; for j = 0 .. m-1 the site update at (G_jj, mu_I[j]), then mu_I -= g s and G -= c s s^T on the trailing part
// (s = G[:, j]). Column l of G keeps s_l below the diagonal (the later steps touch columns > l only): Gout = G, cg = (c, g),
// zero beyond m. dtc: G and mu_I as gpx_ep.cuh describes, and the cavity of site j reads max(G_jj, eps) (sd0[I[0]] for
// the first site of a run), the reference's Sigma_diag, while c and g use G_jj itself.
__global__ void __launch_bounds__(EP_CHAIN_THREADS, 1) ep_chain_kernel(const double* __restrict__ Sig, long ld,
                                                                       const int* __restrict__ I, int m,
                                                                       const double* __restrict__ mu, EpSites e,
                                                                       double* __restrict__ Gout, double* __restrict__ cg,
                                                                       const double* __restrict__ muadd,
                                                                       const double* __restrict__ sd0, int dtc) {
  extern __shared__ double ep_sm[];
  double* G = ep_sm;
  double* s = G + TILE * TILE;
  double* muI = s + TILE;
  double* cgs = muI + TILE;
  const int tid = threadIdx.x, tx = tid & 31, ty = tid >> 5;
  for (int a = ty; a < TILE; a += 32)
    for (int b = tx; b < TILE; b += 32)
      G[a * TILE + b] = (a < m && b <= a) ? (dtc ? Sig[a + b * ld] : ep_sym(Sig, ld, I[a], I[b])) : 0.0;
  if (tid < TILE) muI[tid] = tid < m ? (dtc ? mu[I[tid]] + muadd[tid] : mu[I[tid]]) : 0.0;
  __syncthreads();
  for (int j = 0; j < m; j++) {
    if (tid == 0) {
      double c, g;
      const double Gjj = G[j * TILE + j];
      const double Sd = !dtc ? Gjj : (j == 0 && sd0) ? sd0[I[0]] : fmax(Gjj, 2.220446049250313e-16);
      ep_site(e, I[j], Sd, Gjj, muI[j], &c, &g);
      cgs[0] = c; cgs[1] = g;
      cg[j] = c; cg[TILE + j] = g;
    }
    if (tid > j && tid < m) s[tid] = G[tid * TILE + j];
    __syncthreads();
    const double c = cgs[0], g = cgs[1];
    for (int a = j + 1 + ty; a < m; a += 32) {
      const double ca = c * s[a];
      for (int b = j + 1 + tx; b <= a; b += 32) G[a * TILE + b] -= ca * s[b];
    }
    if (tid > j && tid < m) muI[tid] -= g * s[tid];
    __syncthreads();
  }
  for (int k = tid; k < TILE * TILE; k += EP_CHAIN_THREADS) Gout[k] = G[k];
  if (tid >= m && tid < TILE) { cg[tid] = 0.0; cg[TILE + tid] = 0.0; }
}

// S = Sigma[:, I] (I + U)^-1, one thread per row r (forward substitution in the fixed order l = 0 .. j-1):
// x_j = Sigma(r, I_j) - sum_l (x_l c_l) s_l[j]; out Sx = S, Sc = S diag(c) (Npad x TILE each, zero beyond m) and
// mu_r -= sum_j x_j g_j. G, c and g are those of ep_chain_kernel. dtc: Sigma(r, I_j) is P(r, j), read from P^T in Sig.
__global__ void __launch_bounds__(EP_SOLVE_ROWS) ep_solve_kernel(const double* __restrict__ Sig, long ld,
                                                                 const int* __restrict__ I, int m,
                                                                 const double* __restrict__ Gin,
                                                                 const double* __restrict__ cg, double* __restrict__ Sx,
                                                                 double* __restrict__ Sc, double* __restrict__ mu, int dtc) {
  extern __shared__ double ep_sm[];
  double* G = ep_sm;
  double* cc = G + TILE * TILE;
  double* gg = cc + TILE;
  double* xs = gg + TILE;   // [TILE][EP_SOLVE_ROWS]: x_l c_l of this CTA's rows
  const int t = threadIdx.x;
  for (int k = t; k < TILE * TILE; k += EP_SOLVE_ROWS) G[k] = Gin[k];
  for (int k = t; k < 2 * TILE; k += EP_SOLVE_ROWS) cc[k] = cg[k];
  __syncthreads();
  for (long r = (long)blockIdx.x * EP_SOLVE_ROWS + t; r < ld; r += (long)gridDim.x * EP_SOLVE_ROWS) {
    double dot = 0.0;
    for (int j = 0; j < m; j++) {
      double acc = dtc ? Sig[j + r * TILE] : ep_sym(Sig, ld, r, I[j]);
      const double* Gj = G + j * TILE;
      for (int l = 0; l < j; l++) acc = fma(-xs[l * EP_SOLVE_ROWS + t], Gj[l], acc);
      const double xc = acc * cc[j];
      xs[j * EP_SOLVE_ROWS + t] = xc;
      Sx[r + j * ld] = acc;
      Sc[r + j * ld] = xc;
      dot = fma(acc, gg[j], dot);
    }
    for (int j = m; j < TILE; j++) { Sx[r + j * ld] = 0.0; Sc[r + j * ld] = 0.0; }
    mu[r] -= dot;
  }
}

// parallel_updates=True: every site from the same diag(Sigma) and mu, no rank-1 updates
__global__ void __launch_bounds__(256) ep_parallel_kernel(long N, const double* __restrict__ sd,
                                                          const double* __restrict__ mu, EpSites e) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  double c, g;
  ep_site(e, i, sd[i], sd[i], mu[i], &c, &g);
}

// the EP vector glue, one thread per entry i < n (entries N <= i < n of o are zero)
__global__ void __launch_bounds__(256) ep_vec_kernel(int mode, long N, long n, const double* __restrict__ x,
                                                     const double* __restrict__ y, double* __restrict__ A, long ld,
                                                     double add, double* __restrict__ o) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const bool in = i < N;
  switch (mode) {
    case EV_SUB: o[i] = in ? x[i] - y[i] : 0.0; break;                              // alpha = v~ - U~ U~^T K v~ (:139-140)
    case EV_DIAG: o[i] = in ? (A[i + i * ld] - (x ? x[i] : 0.0)) + add : 0.0; break; // diag(K - V^T V) (+ 1e-7, :319,:326)
    case EV_DLDK: o[i] = in ? 0.5 * (x[i] * x[i] - A[i + i * ld]) : 0.0; break;      // diag(dL_dK) (:393)
    case EV_ADDDIAG: if (in) A[i + i * ld] += add; break;                            // diag.add(Sigma, 1e-7)
    default: o[i] = in ? (x[i] == 1.0 ? 1.0 : -1.0) : 0.0;                          // bernoulli.py:67-70
  }
}

}  // namespace gpx

namespace {

int ep_vec(gpx_ctx* c, int mode, const double* x, const double* y, double* A, double add, double* o) {
  ep_vec_kernel<<<(unsigned)((c->Npad + 255) / 256), 256, 0, c->st>>>(mode, c->N, c->Npad, x, y, A, c->Npad, add, o);
  c->eval_launches++;
  GPX_CUDA(cudaGetLastError());
  return 0;
}

EpSites ep_sites(gpx_ctx* c, double eta, double delta) {
  EpSites e;
  e.tt = lv(c, LV_TT); e.vt = lv(c, LV_VT); e.ct = lv(c, LV_CT); e.cv = lv(c, LV_CV); e.zh = lv(c, LV_ZH);
  e.mh = lv(c, LV_MH); e.s2 = lv(c, LV_S2); e.sgn = lv(c, LV_SGN); e.eta = eta; e.delta = delta;
  return e;
}

// the sweep buffers (and Sigma for sequential updates), kept until laplace_release
int ep_alloc(gpx_ctx* c, bool full) {
  const long ld = c->Npad;
  if (!c->epBlk) GPX_CUDA(cudaMalloc(&c->epBlk, ((size_t)2 * ld * TILE + TILE * TILE + 2 * TILE) * 8));
  if (!c->epOrd) GPX_CUDA(cudaMalloc(&c->epOrd, (size_t)ld * sizeof(int)));
  if (full && !c->epSig) GPX_CUDA(cudaMalloc(&c->epSig, (size_t)ld * ld * 8));
  return 0;
}

int ep_args(const gpx_ctx* c) {
  if (c->dist) GPX_FAIL("expectation propagation is single-GPU");
  if (!c->ep_begun || !c->lap_begun) GPX_FAIL("gpx_ep_begin has not been called on this data");
  return 0;
}

// posteriorParams._recompute (:129-143) from the sites in LV_TT / LV_VT (tt: tau~ on the host, for the jitter ladder's mean):
// B = I + S~^1/2 K S~^1/2 factored, U~ = diag(sqrt tau~) U_B, then Sigma = K - D D^T with D = K U~ (the Laplace factor with
// tau~ for W; ep_full) or only diag(Sigma) = diag(K) - |columns of U~^T K|^2 (parallel updates); `add` on its diagonal;
// alpha = v~ - U~ U~^T K v~ and mu = K alpha
int ep_recompute(gpx_ctx* c, LapTimer& tm, const double* tt, int max_tries, double* jitter_used, double add) {
  cudaStream_t st = c->st;
  const long ld = c->Npad, N = c->N;
  GPX_CHECK(vec(c, LG_SQRTW, nullptr, lv(c, LV_TT), nullptr, nullptr, lv(c, LV_SW)));
  const int info = lap_factor(c, tt, max_tries, jitter_used);
  if (info) return info;
  GPX_CHECK(tm.mark(PH_FACTOR));
  {
    TmpBuf Li(st), Dm(st);
    GPX_CHECK(Li.alloc((size_t)ld * ld));
    GPX_CHECK(Dm.alloc((size_t)ld * ld));
    laplace_scale_u_kernel<<<dim3((unsigned)(ld / 32), (unsigned)(ld / 32)), 256, 0, st>>>(c->S, ld, lv(c, LV_SW), N, Li.p);
    c->eval_launches++;
    GPX_CUDA(cudaGetLastError());
    if (c->ep_full) {
      GPX_CHECK(gemm_nt(c, c->lapK, ld, Li.p, ld, Dm.p, ld, ld, ld, ld, 1, 1));    // D = K Li^T, Li lower triangular
      Li.release();
      GPX_CUDA(cudaMemcpyAsync(c->epSig, c->lapK, (size_t)ld * ld * 8, cudaMemcpyDeviceToDevice, st));
      GemmParams pu = gemm_defaults();
      pu.mode = GEMM_UPDATE;
      pu.A = Dm.p; pu.lda = ld; pu.B = Dm.p; pu.ldb = ld; pu.C = c->epSig; pu.ldc = ld;
      pu.K = (int)ld; pu.nt = (int)(ld / TILE); pu.c0 = 0; pu.ncols = 0; pu.rlow = 0;
      GPX_CHECK(launch_gemm(pu, dim3(1, 1), st));
      c->eval_launches++;
      if (add != 0.0) GPX_CHECK(ep_vec(c, EV_ADDDIAG, nullptr, nullptr, c->epSig, add, nullptr));
    } else {
      GPX_CHECK(gemm_nt(c, Li.p, ld, c->lapK, ld, Dm.p, ld, ld, ld, ld, 1, 2));    // C = Li K, Li lower triangular
      GPX_CHECK(launch_col_sqnorm(Dm.p, ld, ld, N, lv(c, LV_CSQ), st));
      c->eval_launches++;
      GPX_CHECK(ep_vec(c, EV_DIAG, lv(c, LV_CSQ), nullptr, c->lapK, add, lv(c, LV_SD)));
    }
  }
  GPX_CHECK(tm.mark(PH_GEMM));
  GPX_CHECK(kmv(c, lv(c, LV_VT), lv(c, LV_KV)));
  GPX_CHECK(uut_mv(c, lv(c, LV_KV), lv(c, LV_U)));
  GPX_CHECK(ep_vec(c, EV_SUB, lv(c, LV_VT), lv(c, LV_U), nullptr, 0.0, lv(c, LV_A)));
  GPX_CHECK(kmv(c, lv(c, LV_A), lv(c, LV_MU)));
  GPX_CHECK(tm.mark(PH_MV));
  return 0;
}

int ep_download(gpx_ctx* c, int slot, double* h) {
  GPX_CUDA(cudaMemcpyAsync(h, lv(c, slot), (size_t)c->N * 8, cudaMemcpyDeviceToHost, c->st));
  return 0;
}

}  // namespace

extern "C" {

int gpx_ep_begin(gpx_ctx* c, const gpx_kern_part* parts, int nparts) {
  if (!c || !parts) GPX_FAIL("null argument");
  if (!c->S) GPX_FAIL("gpx_set_data has not been called");
  if (c->dist) GPX_FAIL("expectation propagation is single-GPU");
  if (c->P != 1) GPX_FAIL("expectation propagation takes one output column (P = 1)");
  GPX_CUDA(cudaSetDevice(c->device));
  if (!c->ep_labels) {   // once per data set: gpx_set_data releases the Laplace / EP state and with it this flag
    std::vector<double> y((size_t)c->N);
    GPX_CUDA(cudaMemcpy(y.data(), c->dY, (size_t)c->N * 8, cudaMemcpyDeviceToHost));
    for (double v : y)
      if (!(v == 1.0 || v == 0.0 || v == -1.0)) GPX_FAIL("bad value for Bernoulli observation (0, 1)");
  }
  GPX_CHECK(gpx_laplace_begin(c, parts, nparts));
  c->ep_labels = true;
  c->eval_launches = 0;
  GPX_CHECK(ep_vec(c, EV_SIGN, c->dY, nullptr, nullptr, 0.0, lv(c, LV_SGN)));
  if (cudaStreamSynchronize(c->st) != cudaSuccess) GPX_FAIL_DEVICE("gpx_ep_begin");
  c->total_launches += c->eval_launches;
  c->stats.launches += c->eval_launches;
  c->ep_begun = true;
  return 0;
}

int gpx_ep_start(gpx_ctx* c, const double* tau_tilde, const double* v_tilde, int warm, int parallel, int max_tries,
                 double* jitter_used) {
  if (!c || !jitter_used || (warm && (!tau_tilde || !v_tilde))) GPX_FAIL("null argument");
  GPX_CHECK(ep_args(c));
  GPX_CUDA(cudaSetDevice(c->device));
  lap_start(c);
  c->ep_ready = false;
  c->ep_full = !parallel;
  GPX_CHECK(ep_alloc(c, c->ep_full));
  const long ld = c->Npad;
  const int64_t l0 = c->total_launches;
  LapTimer tm{c};
  GPX_CHECK(tm.mark(-1));
  *jitter_used = 0.0;
  if (!warm) {   // _init_approximations, cold (:315-321): sites 0, Sigma = K + 1e-7 I, mu = 0
    GPX_CUDA(cudaMemsetAsync(lv(c, LV_TT), 0, (size_t)ld * 8, c->st));
    GPX_CUDA(cudaMemsetAsync(lv(c, LV_VT), 0, (size_t)ld * 8, c->st));
    GPX_CUDA(cudaMemsetAsync(lv(c, LV_MU), 0, (size_t)ld * 8, c->st));
    if (c->ep_full) {
      GPX_CUDA(cudaMemcpyAsync(c->epSig, c->lapK, (size_t)ld * ld * 8, cudaMemcpyDeviceToDevice, c->st));
      GPX_CHECK(ep_vec(c, EV_ADDDIAG, nullptr, nullptr, c->epSig, 1e-7, nullptr));
    } else {
      GPX_CHECK(ep_vec(c, EV_DIAG, nullptr, nullptr, c->lapK, 1e-7, lv(c, LV_SD)));
    }
  } else {       // warm (:322-326): _recompute from the kept sites, then 1e-7 on Sigma's diagonal
    GPX_CHECK(upload(c, LV_TT, tau_tilde));
    GPX_CHECK(upload(c, LV_VT, v_tilde));
    const int info = ep_recompute(c, tm, tau_tilde, max_tries, jitter_used, 1e-7);
    if (info) { lap_end(c, tm, l0); return info; }
  }
  GPX_CHECK(lap_end(c, tm, l0));
  c->ep_ready = true;
  return 0;
}

int gpx_ep_sweep(gpx_ctx* c, const int64_t* order, double eta, double delta, int parallel, int max_tries,
                 double* tau_tilde, double* v_tilde, double* cav_tau, double* cav_v, double* Z_hat, double* mu_hat,
                 double* sigma2_hat, double* jitter_used) {
  if (!c || !order || !tau_tilde || !v_tilde || !cav_tau || !cav_v || !Z_hat || !mu_hat || !sigma2_hat || !jitter_used)
    GPX_FAIL("null argument");
  GPX_CHECK(ep_args(c));
  if (!c->ep_ready) GPX_FAIL("gpx_ep_start has not been called since gpx_ep_begin");
  if (!parallel != c->ep_full) GPX_FAIL("parallel must be the value gpx_ep_start was given");
  const long N = c->N, ld = c->Npad;
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
  lap_start(c);
  cudaStream_t st = c->st;
  const int64_t l0 = c->total_launches;
  LapTimer tm{c};
  GPX_CHECK(tm.mark(-1));
  GPX_CHECK(upload(c, LV_TT, tau_tilde));
  GPX_CHECK(upload(c, LV_VT, v_tilde));
  const EpSites e = ep_sites(c, eta, delta);
  if (!parallel) {   // _local_updates with the rank-1 updates (:333-351), one block of TILE sites at a time
    GPX_CUDA(cudaMemcpyAsync(c->epOrd, ord.data(), (size_t)N * sizeof(int), cudaMemcpyHostToDevice, st));
    GPX_CUDA(cudaFuncSetAttribute(ep_chain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, EP_CHAIN_SMEM));
    GPX_CUDA(cudaFuncSetAttribute(ep_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, EP_SOLVE_SMEM));
    double* Sx = c->epBlk;
    double* Sc = Sx + (size_t)ld * TILE;
    double* Gb = Sc + (size_t)ld * TILE;
    double* cg = Gb + TILE * TILE;
    const unsigned solve_grid = (unsigned)std::min<long>(ld / EP_SOLVE_ROWS, c->num_sms);
    for (long k0 = 0; k0 < N; k0 += TILE) {
      const int m = (int)std::min<long>(TILE, N - k0);
      const int* I = c->epOrd + k0;
      ep_chain_kernel<<<1, EP_CHAIN_THREADS, EP_CHAIN_SMEM, st>>>(c->epSig, ld, I, m, lv(c, LV_MU), e, Gb, cg, nullptr,
                                                                  nullptr, 0);
      ep_solve_kernel<<<solve_grid, EP_SOLVE_ROWS, EP_SOLVE_SMEM, st>>>(c->epSig, ld, I, m, Gb, cg, Sx, Sc, lv(c, LV_MU),
                                                                        0);
      GPX_CUDA(cudaGetLastError());
      GemmParams pu = gemm_defaults();   // Sigma -= S diag(c) S^T over the lower tiles, k-depth TILE
      pu.mode = GEMM_UPDATE;
      pu.A = Sc; pu.lda = ld; pu.B = Sx; pu.ldb = ld; pu.C = c->epSig; pu.ldc = ld;
      pu.K = TILE; pu.nt = (int)(ld / TILE); pu.c0 = 0; pu.ncols = 0; pu.rlow = 0;
      GPX_CHECK(launch_gemm(pu, dim3(1, 1), st));
      c->eval_launches += 3;
    }
  } else {           // parallel_updates: every site from the same diag(Sigma) and mu
    ep_parallel_kernel<<<(unsigned)((N + 255) / 256), 256, 0, st>>>(N, lv(c, LV_SD), lv(c, LV_MU), e);
    c->eval_launches++;
    GPX_CUDA(cudaGetLastError());
  }
  GPX_CHECK(tm.mark(PH_OTHER));
  GPX_CHECK(ep_download(c, LV_TT, tau_tilde));
  GPX_CHECK(ep_download(c, LV_VT, v_tilde));
  GPX_CHECK(ep_download(c, LV_CT, cav_tau));
  GPX_CHECK(ep_download(c, LV_CV, cav_v));
  GPX_CHECK(ep_download(c, LV_ZH, Z_hat));
  GPX_CHECK(ep_download(c, LV_MH, mu_hat));
  GPX_CHECK(ep_download(c, LV_S2, sigma2_hat));
  if (cudaStreamSynchronize(st) != cudaSuccess) GPX_FAIL_DEVICE("gpx_ep_sweep");
  c->ep_ready = false;   // Sigma and mu are those of the updates until the recompute below has run
  const int info = ep_recompute(c, tm, tau_tilde, max_tries, jitter_used, 0.0);
  if (info) { lap_end(c, tm, l0); return info; }
  GPX_CHECK(lap_end(c, tm, l0));
  c->ep_ready = true;
  return 0;
}

int gpx_ep_finish(gpx_ctx* c, const double* tau_tilde, const double* v_tilde, int max_tries, double* logdet_B,
                  double* vSv, double* diag_dL_dK, double* kgrad, double* jitter_used) {
  if (!c || !tau_tilde || !v_tilde || !logdet_B || !vSv || !diag_dL_dK || !kgrad || !jitter_used)
    GPX_FAIL("null argument");
  GPX_CHECK(ep_args(c));
  GPX_CUDA(cudaSetDevice(c->device));
  lap_start(c);
  cudaStream_t st = c->st;
  const long ld = c->Npad, N = c->N;
  const int nt = (int)(ld / TILE);
  const MultiKern& mk = c->mk;
  size_t need = 0;
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
  GPX_CHECK(upload(c, LV_TT, tau_tilde));
  GPX_CHECK(upload(c, LV_VT, v_tilde));
  GPX_CHECK(vec(c, LG_SQRTW, nullptr, lv(c, LV_TT), nullptr, nullptr, lv(c, LV_SW)));
  // _ep_marginal (:363-377): B at the sites, B_logdet = 2 sum log diag(L) from the per-tile partials
  const int info = lap_factor(c, tau_tilde, max_tries, jitter_used);
  if (info) { lap_end(c, tm, l0); return info; }
  std::vector<double> ldp(nt);
  GPX_CUDA(cudaMemcpyAsync(ldp.data(), c->logdet_part, (size_t)nt * 8, cudaMemcpyDeviceToHost, st));
  GPX_CHECK(tm.mark(PH_FACTOR));
  {
    TmpBuf Li(st);
    GPX_CHECK(Li.alloc((size_t)ld * ld));
    laplace_scale_u_kernel<<<dim3((unsigned)(ld / 32), (unsigned)(ld / 32)), 256, 0, st>>>(c->S, ld, lv(c, LV_SW), N, Li.p);
    c->eval_launches++;
    GPX_CUDA(cudaGetLastError());
  }
  // alpha = v~ - U~ U~^T K v~ (:386-387); c->dT keeps U~^T K v~ for v~^T Sigma v~ = v~^T K v~ - |U~^T K v~|^2
  GPX_CHECK(kmv(c, lv(c, LV_VT), lv(c, LV_KV)));
  GPX_CHECK(uut_mv(c, lv(c, LV_KV), lv(c, LV_U)));
  GPX_CHECK(ep_vec(c, EV_SUB, lv(c, LV_VT), lv(c, LV_U), nullptr, 0.0, c->dAlpha));
  std::vector<double> kv((size_t)N), t((size_t)N);
  GPX_CUDA(cudaMemcpyAsync(kv.data(), lv(c, LV_KV), (size_t)N * 8, cudaMemcpyDeviceToHost, st));
  GPX_CUDA(cudaMemcpyAsync(t.data(), c->dT, (size_t)N * 8, cudaMemcpyDeviceToHost, st));
  GPX_CHECK(tm.mark(PH_MV));
  // Wi = U~ U~^T (:389-391) into the lower tiles of c->Kinv
  GPX_CHECK(lauum_store(c));
  GPX_CHECK(tm.mark(PH_LAUUM));
  // the kernel gradient of dL_dK = 1/2 (alpha alpha^T - Wi) (:393), one reduction per part, and diag(dL_dK)
  size_t off = 0;
  for (int q = 0; q < mk.nparts; q++) {
    GPX_CUDA(cudaMemsetAsync(c->mpartials + off, 0, (size_t)nt * nt * part_nred(mk.part[q]) * 8, st));
    GradKinvMultiParams gm;
    memset(&gm, 0, sizeof(gm));
    gm.Kinv = c->Kinv; gm.ld = ld; gm.XsT = c->dXsT; gm.sq = c->dsq; gm.ldx = ld; gm.alpha = c->dAlpha;
    gm.N = N; gm.P = 1; gm.nt = nt; gm.part = q; gm.want_noise = 0; gm.partials = c->mpartials + off; gm.mk = mk;
    GPX_CHECK(launch_grad_kinv_multi(gm, st));
    c->eval_launches++;
    off += (size_t)nt * nt * part_nred(mk.part[q]);
  }
  GPX_CHECK(ep_vec(c, EV_DLDK, c->dAlpha, nullptr, c->Kinv, 0.0, lv(c, LV_DL)));
  GPX_CHECK(tm.mark(PH_OTHER));
  std::vector<double> hp(off);
  GPX_CUDA(cudaMemcpyAsync(hp.data(), c->mpartials, off * 8, cudaMemcpyDeviceToHost, st));
  GPX_CHECK(ep_download(c, LV_DL, diag_dL_dK));
  GPX_CHECK(lap_end(c, tm, l0));
  double s = 0.0;
  for (int i = 0; i < nt; i++) s += ldp[i];
  *logdet_B = s;
  double a = 0.0, b = 0.0;
  for (long i = 0; i < N; i++) {
    a += v_tilde[i] * kv[i];
    b += t[i] * t[i];
  }
  *vSv = a - b;
  off = 0;
  int g = 0;
  for (int p = 0; p < mk.nparts; p++) {   // tile order, as grad_full_sum
    const int nred = part_nred(mk.part[p]);
    std::vector<double> tot(nred, 0.0);
    for (size_t k = 0; k < (size_t)nt * nt; k++)
      for (int q = 0; q < nred; q++) tot[q] += hp[off + k * nred + q];
    double v;
    for (int q = 0; q < nred; q++)
      if (part_grad_entry(mk, p, q, tot[q], &v)) kgrad[g + q] = v;
    g += part_ngrad(mk.part[p]);
    off += (size_t)nt * nt * nred;
  }
  c->have_eval = true;
  c->have_kinv = true;   // c->Kinv holds Wi = U~ U~^T as it is
  c->lap_post = true;
  return 0;
}

}  // extern "C"

// ==== the variational Gaussian approximation (GPy/inference/latent_function_inference/var_gauss.py:34-69) =================
// Opper & Archambeau's q(f) = N(m, Sigma) with m = K alpha and Sigma = (K^-1 + B^2)^-1, B = diag(beta), on the kept K of
// gpx_laplace_begin. A = I + B K B is factored by the Laplace ladder with w = beta itself (BKB depends on the signs), so
// that Ai = A^-1 = U U^T with U = L_A^-T and Sigma = B^-2 - B^-1 Ai B^-1 (:40). begin needs only the row norms of U for
// diag(Sigma) and tr Ai; finish forms Ai (LAUUM), H = Ai diag(c) Ai (one DMMA GEMM, lower tiles) and one fused pass over
// the lower tiles of Ai and H for the beta gradient and S = B (Ai - H) B + r r^T, the matrix whose -1/2 S + 1/2 g g^T is the
// symmetric part of dL_dK.
namespace gpx {

// partial squared row norms of U (the upper and diagonal tiles of S, zeros below the diagonal inside a diagonal tile):
// part[k * ld + i] = sum of U(i, c)^2 over the columns c < N of chunk k (KSPLIT chunks), zero for rows i >= N
__global__ void __launch_bounds__(256) vargauss_rownorm_kernel(const double* __restrict__ S, long ld, long N,
                                                               double* __restrict__ part) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ld) return;
  const long chunk = (ld + gridDim.y - 1) / gridDim.y;
  const long ce = (long)(blockIdx.y + 1) * chunk, c1 = ce < N ? ce : N;
  const long cs = (long)blockIdx.y * chunk, ct = (i / TILE) * TILE;
  double s = 0.0;
  if (i < N)
    for (long c = cs > ct ? cs : ct; c < c1; c++) s = fma(S[i + c * ld], S[i + c * ld], s);
  part[(long)blockIdx.y * ld + i] = s;
}

// Ai_ii = the row norms summed over the chunks in order, var_i = Sigma_ii = beta_i^-2 - (Ai_ii / beta_i) / beta_i
__global__ void __launch_bounds__(256) vargauss_var_kernel(const double* __restrict__ part, int nsplit, long ld, long N,
                                                           const double* __restrict__ beta, double* __restrict__ aii,
                                                           double* __restrict__ var) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ld) return;
  double s = 0.0;
  for (int k = 0; k < nsplit; k++) s += part[(long)k * ld + i];
  const double b = i < N ? beta[i] : 1.0;
  aii[i] = i < N ? s : 0.0;
  var[i] = i < N ? 1.0 / (b * b) - (s / b) / b : 0.0;
}

// Sc = Ai diag(cv) (whole, cv_j = 0 for j >= N) and the upper tiles of Ai mirrored from its lower tiles, so that H = Sc Ai^T
// runs on the plain DMMA GEMM. 32 x 32 blocks; an upper block reads its transpose through shared memory.
__global__ void __launch_bounds__(256) vargauss_colscale_kernel(double* __restrict__ Ai, long ld, long N,
                                                                const double* __restrict__ cv, double* __restrict__ Sc) {
  __shared__ double t[32][33];
  const long r0 = (long)blockIdx.x * 32, c0 = (long)blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  if (r0 / TILE >= c0 / TILE) {
    for (int k = ty; k < 32; k += 8) {
      const long col = c0 + k;
      Sc[r0 + tx + col * ld] = Ai[r0 + tx + col * ld] * (col < N ? cv[col] : 0.0);
    }
    return;
  }
  for (int k = ty; k < 32; k += 8) t[k][tx] = Ai[(c0 + tx) + (r0 + k) * ld];   // Ai(c0 + tx, r0 + k), a lower tile
  __syncthreads();
  for (int k = ty; k < 32; k += 8) {
    const long col = c0 + k;
    const double v = t[tx][k];                                                  // Ai(c0 + k, r0 + tx) = Ai(r0 + tx, col)
    Ai[r0 + tx + col * ld] = v;
    Sc[r0 + tx + col * ld] = v * (col < N ? cv[col] : 0.0);
  }
}

// The fused pass of gpx_vargauss_finish, one CTA of TILE threads per lower tile (ti >= tj), thread t on row i = ti TILE + t.
// Per element (i, j), with Sigma_ij = delta_ij beta_i^-2 - (Ai_ij / beta_i) / beta_j:
//   F  : Sigma_ij^2 dF_dv_i for column j (and Sigma_ij^2 dF_dv_j for column i off the diagonal tiles), var_gauss.py:52;
//   KL : (delta_ij - Ai_ij)^2 + jit Ai_ij^2 - delta_ij jit Ai_ij, whose column sums times 1 / beta_j are
//        diag(KB^T (Ai - Ai^2)) (:57) because B K B = A - (1 + jit) I;
//   Ai_ij is replaced by S_ij = beta_i beta_j (Ai_ij - H_ij) + r_i r_j (zero outside N x N).
// part[(q nt + t) ld + col], q = 0 (F) / 1 (KL): the sum over the rows of tile t of column col, written by exactly one CTA
// (t >= col's tile: its own column; t < col's tile: the mirror). Column sums are fixed-order shuffle trees.
__global__ void __launch_bounds__(TILE) vargauss_pass_kernel(double* __restrict__ Ai, const double* __restrict__ H, long ld,
                                                             long N, int nt, const double* __restrict__ beta,
                                                             const double* __restrict__ dv, const double* __restrict__ r,
                                                             double jit, double* __restrict__ part) {
  const int ti = blockIdx.x, tj = blockIdx.y;
  if (ti < tj) return;
  __shared__ double sF[TILE / 32][TILE], sK[TILE / 32][TILE];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const long i = (long)ti * TILE + t;
  const bool irow = i < N;
  const double bi = irow ? beta[i] : 1.0, dvi = irow ? dv[i] : 0.0, ri = irow ? r[i] : 0.0;
  double rowF = 0.0, rowK = 0.0;
  for (int jj = 0; jj < TILE; jj++) {
    const long j = (long)tj * TILE + jj;
    const bool in = irow && j < N;
    double f = 0.0, k = 0.0;
    if (in) {
      const double bj = beta[j];
      const double a = Ai[i + j * ld], h = H[i + j * ld];
      const bool d = i == j;
      const double sig = (d ? 1.0 / (bi * bi) : 0.0) - (a / bi) / bj;
      const double s2 = sig * sig;
      f = s2 * dvi;
      const double e = (d ? 1.0 : 0.0) - a;
      k = e * e + jit * (a * a) - (d ? jit * a : 0.0);
      Ai[i + j * ld] = (bi * bj) * (a - h) + ri * r[j];
      rowF = fma(s2, dv[j], rowF);
      rowK += k;
    } else {
      Ai[i + j * ld] = 0.0;
    }
    for (int o = 16; o > 0; o >>= 1) {
      f += __shfl_down_sync(0xffffffffu, f, o);
      k += __shfl_down_sync(0xffffffffu, k, o);
    }
    if (lane == 0) { sF[warp][jj] = f; sK[warp][jj] = k; }
  }
  __syncthreads();
  double cf = 0.0, ck = 0.0;
  for (int w = 0; w < TILE / 32; w++) { cf += sF[w][t]; ck += sK[w][t]; }
  const long col = (long)tj * TILE + t;
  part[((long)ti) * ld + col] = cf;
  part[((long)nt + ti) * ld + col] = ck;
  if (ti > tj) {
    part[((long)tj) * ld + i] = rowF;
    part[((long)nt + tj) * ld + i] = rowK;
  }
}

// dbeta_j = dF_dbeta_j - dKL_dbeta_j = -2 beta_j sum_t F(t, j) - sum_t KL(t, j) / beta_j (tile order), zero for j >= N
__global__ void __launch_bounds__(256) vargauss_dbeta_kernel(const double* __restrict__ part, int nt, long ld, long N,
                                                             const double* __restrict__ beta, double* __restrict__ dbeta) {
  const long j = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= ld) return;
  double f = 0.0, k = 0.0;
  for (int t = 0; t < nt; t++) {
    f += part[(long)t * ld + j];
    k += part[((long)nt + t) * ld + j];
  }
  dbeta[j] = j < N ? -2.0 * f * beta[j] - k / beta[j] : 0.0;
}

}  // namespace gpx

namespace {

// beta from the caller: every entry finite and non-zero (B and B^-2 are formed from it)
int vg_beta_ok(const double* beta, long N) {
  for (long i = 0; i < N; i++)
    if (!std::isfinite(beta[i]) || beta[i] == 0.0) GPX_FAIL("beta must be finite and non-zero");
  return 0;
}

// A = I + B K B with the ladder (the diagonal's mean is 1 + beta_i^2 Kdiag), beta in LV_SW -> 0 or the failing minor
int vg_factor(gpx_ctx* c, int max_tries, double* jitter_used) {
  std::vector<double> b2(c->vg_beta.size());
  for (size_t i = 0; i < b2.size(); i++) b2[i] = c->vg_beta[i] * c->vg_beta[i];
  const int info = lap_factor(c, b2.data(), max_tries, jitter_used);
  if (info) gpx::set_error("VarGauss: A = I + B K B is not positive definite, even with jitter.");
  return info;
}

}  // namespace

extern "C" {

int gpx_vargauss_begin(gpx_ctx* c, const gpx_kern_part* parts, int nparts, const double* alpha, const double* beta,
                       int max_tries, double* m, double* var, double* kl, double* jitter_used) {
  if (!c || !parts || !alpha || !beta || !m || !var || !kl || !jitter_used) GPX_FAIL("null argument");
  if (!c->S) GPX_FAIL("gpx_set_data has not been called");
  if (c->dist) GPX_FAIL("the variational Gaussian approximation is single-GPU");
  if (c->P != 1) GPX_FAIL("the variational Gaussian approximation takes one output column (P = 1)");
  GPX_CHECK(vg_beta_ok(beta, c->N));
  GPX_CHECK(gpx_laplace_begin(c, parts, nparts));   // K into lapK (kbuild_ms, 2 launches)
  const gpx_stats kst = c->stats;
  cudaStream_t st = c->st;
  const long ld = c->Npad, N = c->N;
  c->vg_alpha.assign(alpha, alpha + N);
  c->vg_beta.assign(beta, beta + N);
  c->eval_launches = 0;
  const int64_t l0 = c->total_launches;
  LapTimer tm{c};
  GPX_CHECK(tm.mark(-1));
  GPX_CHECK(upload(c, LV_T1, alpha));
  GPX_CHECK(upload(c, LV_SW, beta));
  GPX_CHECK(kmv(c, lv(c, LV_T1), lv(c, LV_KV)));                                 // m = K alpha (:37)
  GPX_CHECK(tm.mark(PH_MV));
  double jit = 0.0;
  const int info = vg_factor(c, max_tries, &jit);
  *jitter_used = jit;
  if (info) {
    lap_end(c, tm, l0);
    return info;
  }
  std::vector<double> ldp(ld / TILE);
  GPX_CUDA(cudaMemcpyAsync(ldp.data(), c->logdet_part, ldp.size() * 8, cudaMemcpyDeviceToHost, st));
  GPX_CHECK(tm.mark(PH_FACTOR));
  // diag(Ai) from the row norms of U, var = diag(Sigma) (:40-41)
  vargauss_rownorm_kernel<<<dim3((unsigned)((ld + 255) / 256), KSPLIT), 256, 0, st>>>(c->S, ld, N, c->dUvPart);
  vargauss_var_kernel<<<(unsigned)((ld + 255) / 256), 256, 0, st>>>(c->dUvPart, KSPLIT, ld, N, lv(c, LV_SW), lv(c, LV_DIAG),
                                                                    lv(c, LV_U));
  c->eval_launches += 2;
  GPX_CUDA(cudaGetLastError());
  GPX_CHECK(tm.mark(PH_OTHER));
  std::vector<double> aii((size_t)N);
  c->vg_m.resize((size_t)N);
  GPX_CUDA(cudaMemcpyAsync(c->vg_m.data(), lv(c, LV_KV), (size_t)N * 8, cudaMemcpyDeviceToHost, st));
  GPX_CUDA(cudaMemcpyAsync(var, lv(c, LV_U), (size_t)N * 8, cudaMemcpyDeviceToHost, st));
  GPX_CUDA(cudaMemcpyAsync(aii.data(), lv(c, LV_DIAG), (size_t)N * 8, cudaMemcpyDeviceToHost, st));
  GPX_CHECK(lap_end(c, tm, l0));
  c->stats.total_ms += kst.total_ms;
  c->stats.launches += kst.launches;
  // KL = 1/2 (log|A| + tr Ai - N + alpha^T m) (:55), each sum in index order
  double logdet = 0.0, tr = 0.0, am = 0.0;
  for (double v : ldp) logdet += v;
  for (long i = 0; i < N; i++) { tr += aii[i]; am += c->vg_m[i] * alpha[i]; }
  *kl = 0.5 * (logdet + tr - (double)N + am);
  std::memcpy(m, c->vg_m.data(), (size_t)N * 8);
  c->vg_max_tries = max_tries;
  c->vg_begun = c->vg_factored = true;
  return 0;
}

int gpx_vargauss_finish(gpx_ctx* c, const double* dF_dm, const double* dF_dv, double* dalpha, double* dbeta, double* kgrad) {
  if (!c || !dF_dm || !dF_dv || !dalpha || !dbeta || !kgrad) GPX_FAIL("null argument");
  if (c->dist) GPX_FAIL("the variational Gaussian approximation is single-GPU");
  if (!c->vg_begun || !c->lap_begun) GPX_FAIL("gpx_vargauss_begin has not been called on this data and kernel");
  GPX_CUDA(cudaSetDevice(c->device));
  const bool factored = c->vg_factored;
  lap_start(c);
  cudaStream_t st = c->st;
  const long ld = c->Npad, N = c->N;
  const int nt = (int)(ld / TILE);
  const MultiKern& mk = c->mk;
  size_t need = 0;
  for (int q = 0; q < mk.nparts; q++) need += (size_t)nt * nt * part_nred(mk.part[q]);
  if (need > c->mpart_cap) {
    if (c->mpartials) cudaFree(c->mpartials);
    c->mpartials = nullptr;
    c->mpart_cap = 0;
    GPX_CUDA(cudaMalloc(&c->mpartials, need * 8));
    c->mpart_cap = need;
  }
  // the O(N) terms: c = 1 + 2 dF_dv / beta^2, r = alpha - dF_dm
  std::vector<double> cv((size_t)N), rv((size_t)N);
  for (long i = 0; i < N; i++) {
    const double b = c->vg_beta[i];
    cv[i] = 1.0 + 2.0 * dF_dv[i] / (b * b);
    rv[i] = c->vg_alpha[i] - dF_dm[i];
  }
  const int64_t l0 = c->total_launches;
  LapTimer tm{c};
  GPX_CHECK(tm.mark(-1));
  GPX_CHECK(upload(c, LV_SW, c->vg_beta.data()));
  GPX_CHECK(upload(c, LV_B, dF_dm));
  GPX_CHECK(upload(c, LV_W, dF_dv));
  GPX_CHECK(upload(c, LV_T1, cv.data()));
  GPX_CHECK(upload(c, LV_Y, rv.data()));
  GPX_CUDA(cudaMemcpyAsync(c->dAlpha, c->vg_alpha.data(), (size_t)N * 8, cudaMemcpyHostToDevice, st));
  double jit = c->jitter_extra;
  if (!factored) {   // a finish after a finish: the last one scaled the factor in place
    const int info = vg_factor(c, c->vg_max_tries, &jit);
    if (info) {
      lap_end(c, tm, l0);
      return info;
    }
    GPX_CHECK(tm.mark(PH_FACTOR));
  }
  // 1. Ai = U U^T into the lower tiles of c->Kinv
  GPX_CHECK(lauum_store(c));
  GPX_CHECK(tm.mark(PH_LAUUM));
  {
    TmpBuf Sc(st), H(st);
    GPX_CHECK(Sc.alloc((size_t)ld * ld));
    GPX_CHECK(H.alloc((size_t)ld * ld));
    // 2. H = Ai diag(c) Ai: the scaled copy and the mirrored Ai, then one GEMM over the lower tiles
    vargauss_colscale_kernel<<<dim3((unsigned)(ld / 32), (unsigned)(ld / 32)), 256, 0, st>>>(c->Kinv, ld, N, lv(c, LV_T1),
                                                                                            Sc.p);
    c->eval_launches++;
    GPX_CUDA(cudaGetLastError());
    GPX_CHECK(tm.mark(PH_OTHER));
    GPX_CHECK(gemm_nt(c, Sc.p, ld, c->Kinv, ld, H.p, ld, ld, ld, ld, 2, 0));
    GPX_CHECK(tm.mark(PH_GEMM));
    // 3. the fused pass: beta-gradient partials (into Sc, free after the GEMM) and S over Ai
    vargauss_pass_kernel<<<dim3((unsigned)nt, (unsigned)nt), TILE, 0, st>>>(c->Kinv, H.p, ld, N, nt, lv(c, LV_SW),
                                                                            lv(c, LV_W), lv(c, LV_Y), jit, Sc.p);
    vargauss_dbeta_kernel<<<(unsigned)((ld + 255) / 256), 256, 0, st>>>(Sc.p, nt, ld, N, lv(c, LV_SW), lv(c, LV_U));
    c->eval_launches += 2;
    GPX_CUDA(cudaGetLastError());
    // 4. the kernel gradient of dL_dK's symmetric part 1/2 (g g^T - S), g = dF_dm, one reduction per part
    size_t off = 0;
    for (int q = 0; q < mk.nparts; q++) {
      GPX_CUDA(cudaMemsetAsync(c->mpartials + off, 0, (size_t)nt * nt * part_nred(mk.part[q]) * 8, st));
      GradKinvMultiParams gm;
      memset(&gm, 0, sizeof(gm));
      gm.Kinv = c->Kinv; gm.ld = ld; gm.XsT = c->dXsT; gm.sq = c->dsq; gm.ldx = ld; gm.alpha = lv(c, LV_B);
      gm.N = N; gm.P = 1; gm.nt = nt; gm.part = q; gm.want_noise = 0; gm.partials = c->mpartials + off; gm.mk = mk;
      GPX_CHECK(launch_grad_kinv_multi(gm, st));
      c->eval_launches++;
      off += (size_t)nt * nt * part_nred(mk.part[q]);
    }
    GPX_CHECK(tm.mark(PH_OTHER));
    // 5. K dF_dm; 6. the posterior: U~ = diag(beta) U_A in place (Li = U~^T into H, free now), woodbury_vector = alpha
    GPX_CHECK(kmv(c, lv(c, LV_B), lv(c, LV_KV)));
    laplace_scale_u_kernel<<<dim3((unsigned)(ld / 32), (unsigned)(ld / 32)), 256, 0, st>>>(c->S, ld, lv(c, LV_SW), N, H.p);
    c->eval_launches++;
    GPX_CUDA(cudaGetLastError());
    GPX_CHECK(tm.mark(PH_MV));
  }
  std::vector<double> hp(need), kg((size_t)N);
  GPX_CUDA(cudaMemcpyAsync(hp.data(), c->mpartials, need * 8, cudaMemcpyDeviceToHost, st));
  GPX_CUDA(cudaMemcpyAsync(kg.data(), lv(c, LV_KV), (size_t)N * 8, cudaMemcpyDeviceToHost, st));
  GPX_CUDA(cudaMemcpyAsync(dbeta, lv(c, LV_U), (size_t)N * 8, cudaMemcpyDeviceToHost, st));
  GPX_CHECK(lap_end(c, tm, l0));
  for (long i = 0; i < N; i++) dalpha[i] = kg[i] - c->vg_m[i];                  // dF_da - dKL_da (:43,:56)
  size_t off = 0;
  int g = 0;
  for (int p = 0; p < mk.nparts; p++) {   // tile order, as grad_full_sum
    const int nred = part_nred(mk.part[p]);
    std::vector<double> tot(nred, 0.0);
    for (size_t k = 0; k < (size_t)nt * nt; k++)
      for (int q = 0; q < nred; q++) tot[q] += hp[off + k * nred + q];
    double v;
    for (int q = 0; q < nred; q++)
      if (part_grad_entry(mk, p, q, tot[q], &v)) kgrad[g + q] = v;
    g += part_ngrad(mk.part[p]);
    off += (size_t)nt * nt * nred;
  }
  c->have_eval = true;
  c->have_kinv = false;   // the stored matrix is S: gpx_get(KINV) forms U~ U~^T = B Ai B again
  c->lap_post = true;
  c->vg_begun = true;     // K, alpha and beta stay; the factor is scaled, so the next finish factors A again
  return 0;
}

}  // extern "C"
