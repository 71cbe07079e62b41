// gpx_joint.cu — the joint posterior on the device: the covariance between two sets of test points and joint samples of the
// latent function (GPy's Posterior.covariance_between_points, posterior.py:109-130, and GP.posterior_samples_f, gp.py:601-629).
//
// Exact model, with U = L^-T of the evaluation's factor in the upper tiles of S:
//   K(X*, X)        one K-build, test points m-contiguous (the GEMM's A operand), zero padded to whole tiles; the two point
//                   sets of a cross-covariance are stacked [X1; X2] at a tile boundary, so one build serves both
//   L^-1            extracted from U into a temporary, column-major with leading dimension Npad, zero outside N x N
//   T^T = K(X*, X) (L^-1)^T              the plain DMMA GEMM with B lower triangular (tri = 1): N^2 M* flops
//   T1^T T2                              the plain DMMA GEMM (lower tiles only when X2 = X1), then one combine with K(X1, X2)
// Sampling (both models): Sigma is factored with jitchol's ladder in a child context of the caller, so that the caller's
// factor, alpha and stats stay as they are; f = mu + L_Sigma z is the plain DMMA GEMM with A lower triangular (tri = 2).
#include <algorithm>
#include <cstring>
#include <vector>

#include "gpx_common.cuh"
#include "gpx_ctx.cuh"
#include "gpx_kernels.cuh"

namespace gpx {

// ---------------------------------------------------------------------------------------------------------------
// small kernels: factor extraction with a leading dimension, the covariance combine, z's operand layout, the mean add
// ---------------------------------------------------------------------------------------------------------------

// out (ldo x ldo, column-major) = L (lower = 1: the lower factor, diagonal tiles from Ldiag) or L^-1 (lower = 0: U^T) of
// the factor workspace S (leading dimension ld) over the leading N x N block, zero everywhere else
__global__ void __launch_bounds__(256) joint_extract_kernel(int lower, const double* __restrict__ S, long ld,
                                                            const double* __restrict__ Ldiag, long N,
                                                            double* __restrict__ out, long ldo) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ldo) return;
  for (long j = blockIdx.y; j < ldo; j += gridDim.y) {
    double v = 0.0;
    if (i < N && j < N && i >= j) {
      const long ti = i / TILE, tj = j / TILE;
      if (!lower) v = S[j + i * ld];   // L^-1(i, j) = U(j, i)
      else if (ti > tj) v = S[i + j * ld];
      else v = Ldiag[ti * TILE * TILE + (i % TILE) + (j % TILE) * TILE];
    }
    out[i + j * ldo] = v;
  }
}

// out(a, b) = K(a, off2 + b) - prod(a, b) for a < M1, b < M2; K column-major (ldk), prod column-major (ldp), read from its
// lower tiles only when sym (the mirror image stands for the upper ones, so the result is exactly symmetric). out is
// column-major (ldo) when colmajor, else row-major M1 x M2 (ldo = M2). out may be K itself (the in-place symmetric case).
__global__ void __launch_bounds__(256) joint_combine_kernel(const double* K, long ldk, long off2,
                                                            const double* __restrict__ prod, long ldp, int sym, long M1,
                                                            long M2, double* out, long ldo, int colmajor) {
  const long a = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= M1) return;
  for (long b = blockIdx.y; b < M2; b += gridDim.y) {
    const double p = sym ? (a >= b ? prod[a + b * ldp] : prod[b + a * ldp]) : prod[a + b * ldp];
    const double v = K[a + (off2 + b) * ldk] - p;
    out[colmajor ? a + b * ldo : a * ldo + b] = v;
  }
}

// z (nz x M row-major: nz standard-normal vectors of length M) -> the GEMM's B operand: element (j, k) at Zt[j + k * ldz],
// zero for j >= nz or k >= M (ldz and rows_pad whole tiles)
__global__ void __launch_bounds__(256) z_layout_kernel(const double* __restrict__ z, long M, long nz,
                                                       double* __restrict__ Zt, long ldz, long rows_pad) {
  const long j = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= ldz) return;
  for (long k = blockIdx.y; k < rows_pad; k += gridDim.y) Zt[j + k * ldz] = (j < nz && k < M) ? z[j * M + k] : 0.0;
}

// f[j * M + m] = F[m + j * ldf] + mu[(j / S) * ldmu + m]: sample j of output j / S, in the caller's layout
__global__ void __launch_bounds__(256) mean_add_kernel(const double* __restrict__ F, long ldf, const double* __restrict__ mu,
                                                       long ldmu, long M, long nz, long S, double* __restrict__ f) {
  const long m = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  for (long j = blockIdx.y; j < nz; j += gridDim.y) f[j * M + m] = F[m + j * ldf] + mu[(j / S) * ldmu + m];
}

static unsigned grid_y(long n) { return (unsigned)std::max<long>(1, std::min<long>(n, 65535)); }

// ---------------------------------------------------------------------------------------------------------------
// host helpers (gpx_ctx.cuh)
// ---------------------------------------------------------------------------------------------------------------
int TmpBuf::alloc(size_t doubles) {
  if (cudaMallocAsync((void**)&p, doubles * 8, st) != cudaSuccess) {
    cudaGetLastError();
    p = nullptr;
    set_error("joint posterior: out of device memory for a temporary of " + std::to_string(doubles * 8) + " bytes");
    return -1;
  }
  return 0;
}

// U = L^-T of the factor in S (its upper triangle, U(i, j) = S[i + j ld] for i <= j) column-major with zeros below the
// diagonal and in the padding
__global__ void __launch_bounds__(256) extract_u_kernel(const double* __restrict__ S, long ld, long N, double* __restrict__ out) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ld) return;
  for (long j = blockIdx.y; j < ld; j += gridDim.y) out[i + j * ld] = (i <= j && j < N) ? S[i + j * ld] : 0.0;
}

int extract_inverse_factor(gpx_ctx* c, int upper, double* out) {
  const long Npad = c->Npad;
  if (upper)
    extract_u_kernel<<<dim3((unsigned)(Npad / 256 + 1), grid_y(Npad)), 256, 0, c->st>>>(c->S, Npad, c->N, out);
  else
    joint_extract_kernel<<<dim3((unsigned)(Npad / 256 + 1), grid_y(Npad)), 256, 0, c->st>>>(0, c->S, Npad, c->Ldiag, c->N,
                                                                                             out, Npad);
  GPX_CUDA(cudaGetLastError());
  return 0;
}

int gemm_nt(gpx_ctx* c, const double* A, long lda, const double* B, long ldb, double* C, long ldc, long rows, long cols,
            long kdepth, int plain, int tri) {
  GemmParams pg = gemm_defaults();
  pg.mode = GEMM_PANEL; pg.plain = plain; pg.tri = tri;
  pg.A = A; pg.lda = lda; pg.B = B; pg.ldb = ldb; pg.C = C; pg.ldc = ldc;
  pg.K = (int)kdepth; pg.nt = (int)(rows / TILE); pg.ncols = (int)(cols / TILE);
  GPX_CHECK(launch_gemm(pg, dim3(1, 1), c->st));
  c->total_launches++;
  return 0;
}

int joint_combine(gpx_ctx* c, const double* K, long ldk, long off2, const double* prod, long ldp, int sym, long M1, long M2,
                  double* out, long ldo, int colmajor) {
  joint_combine_kernel<<<dim3((unsigned)((M1 + 255) / 256), grid_y(M2)), 256, 0, c->st>>>(K, ldk, off2, prod, ldp, sym, M1,
                                                                                          M2, out, ldo, colmajor);
  c->total_launches++;
  GPX_CUDA(cudaGetLastError());
  return 0;
}

int joint_check(const gpx_ctx* c, const double* X, int64_t M, const double* z, int64_t nz, const double* f,
                const double* jitter_used, int P) {
  if (!X || !z || !f || !jitter_used) GPX_FAIL("null argument");
  if (M < 1) GPX_FAIL("empty Xnew");
  if (nz < 1) GPX_FAIL("no standard-normal vectors (nz < 1)");
  if (nz % P) GPX_FAIL("nz must be a multiple of the number of outputs P (S vectors per output)");
  if (c->dist) GPX_FAIL("the joint posterior is single-GPU");
  return 0;
}

int joint_sample(gpx_ctx* c, const double* Sig, long lds, long M, const double* mu, long ldmu, const double* z, long nz,
                 long S, int max_tries, double* f, double* jitter_used) {
  cudaStream_t st = c->st;
  if (!c->cJ) GPX_CHECK(gpx_create(c->device, &c->cJ));
  gpx_ctx* ch = c->cJ;
  if (ch->NB != c->NB) GPX_CHECK(gpx_set_option(ch, "nb", c->NB));
  ch->ozaki = c->ozaki;
  GPX_CUDA(cudaStreamSynchronize(st));   // Sigma complete before the child's stream reads it
  const int64_t l0 = ch->total_launches;
  double jit = 0.0;
  const int rc = factor_device(ch, Sig, lds, M, 0.0, max_tries, nullptr, &jit);
  c->total_launches += ch->total_launches - l0;
  *jitter_used = jit;
  if (rc) return rc;
  const long Mpad = ch->Npad, nzpad = (nz + TILE - 1) / TILE * TILE;
  TmpBuf L(st), zd(st), Zt(st), F(st), fd(st);
  GPX_CHECK(L.alloc((size_t)Mpad * Mpad));
  GPX_CHECK(zd.alloc((size_t)nz * M));
  GPX_CHECK(Zt.alloc((size_t)nzpad * Mpad));
  GPX_CHECK(F.alloc((size_t)Mpad * nzpad));
  GPX_CHECK(fd.alloc((size_t)nz * M));
  GPX_CUDA(cudaMemcpyAsync(zd.p, z, (size_t)nz * M * 8, cudaMemcpyHostToDevice, st));
  joint_extract_kernel<<<dim3((unsigned)(Mpad / 256 + 1), grid_y(Mpad)), 256, 0, st>>>(1, ch->S, ch->Npad, ch->Ldiag, M,
                                                                                        L.p, Mpad);
  z_layout_kernel<<<dim3((unsigned)(nzpad / 256 + 1), grid_y(Mpad)), 256, 0, st>>>(zd.p, M, nz, Zt.p, nzpad, Mpad);
  c->total_launches += 2;
  GPX_CUDA(cudaGetLastError());
  GPX_CHECK(gemm_nt(c, L.p, Mpad, Zt.p, nzpad, F.p, Mpad, Mpad, nzpad, Mpad, 1, 2));   // L_Sigma z, k-range <= row tile
  mean_add_kernel<<<dim3((unsigned)((M + 255) / 256), grid_y(nz)), 256, 0, st>>>(F.p, Mpad, mu, ldmu, M, nz, S, fd.p);
  c->total_launches++;
  GPX_CUDA(cudaGetLastError());
  GPX_CUDA(cudaMemcpyAsync(f, fd.p, (size_t)nz * M * 8, cudaMemcpyDeviceToHost, st));
  if (cudaStreamSynchronize(st) != cudaSuccess) GPX_FAIL_DEVICE("joint posterior samples");
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// exact model: the product term of K(X1, X) Ky^-1 K(X, X2) and K(X1, X2) for the stacked test points ps (X1 in rows
// [0, M1), X2 in rows [off2, off2 + M2), off2 a whole number of tiles; off2 = 0 and M2 = M1 for X2 = X1). Kss (ps.ld^2)
// receives K(ps, ps) and, for X2 = X1, Sigma in place; prod (ld M1pad) the product term. With mu != nullptr the means
// K(X1, X) alpha go there ([P][ps.ld]).
// ---------------------------------------------------------------------------------------------------------------
static int exact_joint(gpx_ctx* c, const Points& ps, long M1, long off2, long M2, int sym, TmpBuf& Kss, TmpBuf& prod,
                       TmpBuf* mu) {
  cudaStream_t st = c->st;
  const long Ls = ps.ld, Npad = c->Npad, M1pad = (M1 + TILE - 1) / TILE * TILE, M2pad = (M2 + TILE - 1) / TILE * TILE;
  {
    TmpBuf Ks(st), Li(st), Tt(st);
    GPX_CHECK(Ks.alloc((size_t)Ls * Npad));
    GPX_CHECK(Li.alloc((size_t)Npad * Npad));
    GPX_CHECK(Tt.alloc((size_t)Ls * Npad));
    GPX_CUDA(cudaMemsetAsync(Ks.p, 0, (size_t)Ls * Npad * 8, st));
    GPX_CHECK(build_K(c, c->mk, c->D, ps, train_points(c), Ks.p, Ls));   // K(X*, X): test points thread-mapped, m-contiguous
    c->total_launches++;
    joint_extract_kernel<<<dim3((unsigned)(Npad / 256 + 1), grid_y(Npad)), 256, 0, st>>>(0, c->S, Npad, c->Ldiag, c->N,
                                                                                          Li.p, Npad);
    c->total_launches++;
    GPX_CUDA(cudaGetLastError());
    GPX_CHECK(gemm_nt(c, Ks.p, Ls, Li.p, Npad, Tt.p, Ls, Ls, Npad, Npad, 1, 1));        // T^T = K(X*, X) L^-T
    Li.release();
    if (mu) {   // K(X*, X) alpha: one partial sum per row and column chunk, reduced in fixed order
      constexpr int RSPLIT = 64;
      TmpBuf part(st);
      GPX_CHECK(mu->alloc((size_t)c->P * Ls));
      GPX_CHECK(part.alloc((size_t)RSPLIT * c->P * Ls));
      GPX_CHECK(launch_row_dot(Ks.p, Ls, Ls, c->N, c->P, c->dAlpha, Npad, RSPLIT, part.p, mu->p, st));
      c->total_launches += 2;
    }
    Ks.release();
    GPX_CHECK(prod.alloc((size_t)M1pad * (sym ? M1pad : M2pad)));
    GPX_CHECK(gemm_nt(c, Tt.p, Ls, Tt.p + off2, Ls, prod.p, M1pad, M1pad, sym ? M1pad : M2pad, Npad, sym ? 2 : 1, 0));
  }
  GPX_CHECK(Kss.alloc((size_t)Ls * Ls));
  GPX_CHECK(build_K(c, c->mk, c->D, ps, ps, Kss.p, Ls));   // one point set on both sides: exact zero distance on its diagonal only
  c->total_launches++;
  return 0;
}

static int exact_args(const gpx_ctx* c) {
  if (!c->have_eval) GPX_FAIL("no successful gpx_exact_eval to take the posterior from");
  if (c->dist) GPX_FAIL("the joint posterior is single-GPU");
  return 0;
}

}  // namespace gpx

using namespace gpx;

extern "C" {

int gpx_posterior_covariance(gpx_ctx* c, const double* X1, int64_t M1, const double* X2, int64_t M2, double* cov) {
  if (!c || !X1 || !cov) GPX_FAIL("null argument");
  GPX_CHECK(exact_args(c));
  if (c->P > MAX_P) GPX_FAIL("the joint posterior serves at most 8 output columns");
  if (M1 < 1 || (X2 && M2 < 1)) GPX_FAIL("empty point set");
  GPX_CUDA(cudaSetDevice(c->device));
  const int sym = X2 == nullptr;
  if (sym) M2 = M1;
  const long D = c->D, M1pad = (M1 + TILE - 1) / TILE * TILE, off2 = sym ? 0 : M1pad;
  // [X1; zero rows up to the tile boundary; X2]: one point set, one K-build against the training points
  std::vector<double> hx;
  const double* Xs = X1;
  long ns = M1;
  if (!sym) {
    ns = M1pad + M2;
    hx.assign((size_t)ns * D, 0.0);
    memcpy(hx.data(), X1, (size_t)M1 * D * 8);
    memcpy(hx.data() + (size_t)M1pad * D, X2, (size_t)M2 * D * 8);
    Xs = hx.data();
  }
  PointSet ps;
  GPX_CHECK(upload_points(c, c->mk, Xs, ns, (int)D, ps));
  TmpBuf Kss(c->st), prod(c->st), out(c->st);
  GPX_CHECK(exact_joint(c, ps, M1, off2, M2, sym, Kss, prod, nullptr));
  GPX_CHECK(out.alloc((size_t)M1 * M2));
  GPX_CHECK(joint_combine(c, Kss.p, ps.ld, off2, prod.p, M1pad, sym, M1, M2, out.p, M2, 0));
  GPX_CUDA(cudaMemcpyAsync(cov, out.p, (size_t)M1 * M2 * 8, cudaMemcpyDeviceToHost, c->st));
  if (cudaStreamSynchronize(c->st) != cudaSuccess) GPX_FAIL_DEVICE("gpx_posterior_covariance");
  return 0;
}

int gpx_posterior_samples(gpx_ctx* c, const double* Xnew, int64_t M, const double* z, int64_t nz, int max_tries, double* f,
                          double* jitter_used) {
  if (!c) GPX_FAIL("null argument");
  GPX_CHECK(exact_args(c));
  if (c->P > MAX_P) GPX_FAIL("the joint posterior serves at most 8 output columns");
  GPX_CHECK(joint_check(c, Xnew, M, z, nz, f, jitter_used, c->P));
  GPX_CUDA(cudaSetDevice(c->device));
  PointSet ps;
  GPX_CHECK(upload_points(c, c->mk, Xnew, M, c->D, ps));
  TmpBuf Kss(c->st), prod(c->st), mu(c->st);
  GPX_CHECK(exact_joint(c, ps, M, 0, M, 1, Kss, prod, &mu));
  GPX_CHECK(joint_combine(c, Kss.p, ps.ld, 0, prod.p, ps.ld, 1, M, M, Kss.p, ps.ld, 1));   // Sigma in place of K(X*, X*)
  return joint_sample(c, Kss.p, ps.ld, M, mu.p, ps.ld, z, nz, nz / c->P, max_tries, f, jitter_used);
}

}  // extern "C"
