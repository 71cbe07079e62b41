// gpx_psi.cu — the RBF psi-statistics of an uncertain input q(x_n) = N(mu_n, diag(S_n)) and their gradients.
//
// Reference: GPy/kern/src/psi_comp/rbf_psi_comp.py:8-136. Every kernel works in fp64 on the CUDA cores; nothing of size
// N x M x M is formed and every sum runs in a fixed order, so a repeated call gives the same bits.
//   psi_prep      per point: 1/(S + l^2), 1/(2S + l^2) and the two log-denominators, formed once per n        :23-47
//   psi1          psi1[n, m] = variance exp(ld1_n - 1/2 sum_q (mu_nq - z_mq)^2 / (S_nq + l_q^2))         :22-34
//   psi2 pairs    one CTA per 16 x 16 tile of pairs (m >= m') and per slice of the points: the pair factor
//                 exp(-|z_m - z_m'|^2 / 4l^2) once per pair, then sum_n exp(ld2_n - sum_q d_nq (mu_nq - zhat_q)^2)
//                 over the slice in order; a second launch sums the slices in order and mirrors the pair     :36-51
//   gradients     the same pair pass weighted by the symmetrised dL_dpsi2 keeps per pair sum_n L and
//                 sum_n L d_nq (mu_nq - zhat_q) (for dZ); a per-point pass (one thread per n, row ranges of pairs
//                 split over CTAs) keeps per n the sums of L, L (mu - zhat), L (mu - zhat)^2 and the psi1 ones
//                 (for dmu, dS, the lengthscale); a per-inducing-point pass reduces dZ                          :53-136
#include <algorithm>
#include <cmath>
#include <vector>

#include "gpx_psi.cuh"

namespace gpx {

namespace {

constexpr int PT = 16;         // pair tile edge: 256 pairs per CTA, one per thread
constexpr int NC = 32;         // points staged in shared memory per step of the pair kernel
constexpr int PSI_TARGET_CTAS = 1056;   // 8 CTAs per SM of an H100 SXM: the splits are sized to give about this many
constexpr int MAX_NSPLIT = 16;   // CTA columns of the per-point pass

int counted(gpx_ctx* c, int n) {
  c->total_launches += n;
  GPX_CUDA(cudaGetLastError());
  return 0;
}

__global__ void psi_prep_kernel(PsiParams pp, const double* __restrict__ S, double* __restrict__ pre) {
  const long n = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= pp.N) return;
  const int Q = pp.Q;
  double* o = pre + n * (2 * Q + 2);
  double l1 = 0.0, l2 = 0.0;
  for (int q = 0; q < Q; q++) {
    const double s = S[n * Q + q], L2 = pp.l[q] * pp.l[q];
    o[q] = 1.0 / (s + L2);
    o[Q + q] = 1.0 / (2.0 * s + L2);
    l1 += log1p(s / L2);
    l2 += log1p(2.0 * s / L2);
  }
  o[2 * Q] = -0.5 * l1;
  o[2 * Q + 1] = -0.5 * l2;
}

// psi1 in the direct (mu - z)^2 form, one thread per (n, m)
__global__ void psi1_kernel(PsiParams pp, const double* __restrict__ mu, const double* __restrict__ pre,
                            const double* __restrict__ Z, double* __restrict__ out, long sn, long sm) {
  const long n = (long)blockIdx.x * blockDim.x + threadIdx.x, m = blockIdx.y;
  if (n >= pp.N) return;
  const int Q = pp.Q;
  const double* p = pre + n * (2 * Q + 2);
  double e = p[2 * Q];
  for (int q = 0; q < Q; q++) {
    const double d = mu[n * Q + q] - Z[m * Q + q];
    e = fma(-0.5 * d * p[q], d, e);
  }
  out[n * sn + m * sm] = pp.variance * exp(e);
}

__device__ __forceinline__ void tile_of(int t, int& ti, int& tj) {
  int i = (int)((sqrt(8.0 * t + 1.0) - 1.0) * 0.5);
  while ((i + 1) * (i + 2) / 2 <= t) i++;
  while (i * (i + 1) / 2 > t) i--;
  ti = i; tj = t - i * (i + 1) / 2;
}
// slot of the pair (a, b), a >= b, in the pair kernel's output: tile index * 256 + thread
__device__ __forceinline__ long pair_slot(long a, long b) {
  const long ti = a / PT, tj = b / PT;
  return (ti * (ti + 1) / 2 + tj) * (PT * PT) + (a % PT) * PT + (b % PT);
}

// GRAD = false: part[s][pair] = variance^2 sum_{n in slice s} psi2_n[m, m'] (m >= m').
// GRAD = true : with L = dLs psi2_n (dLs: the symmetrised dL_dpsi2), part[s][pair][0] = sum_n L and
//               part[s][pair][1 + q] = sum_n L d_nq (mu_nq - zhat_q); the first slice also writes the per-pair factor
//               cf[m + m' ldc] = w variance^2 dLs exp(-|z_m - z_m'|^2 / 4l^2), w = 1 on the diagonal, else 2
template <int QR, bool GRAD>
__global__ void __launch_bounds__(256) psi2_pair_kernel(PsiParams pp, const double* __restrict__ mu,
                                                        const double* __restrict__ pre, const double* __restrict__ Z,
                                                        const double* __restrict__ dL2, long ld2, long nchunk,
                                                        double* __restrict__ part, double* __restrict__ cf, long ldc) {
  __shared__ double smu[NC][QR], sd[NC][QR], sld[NC];
  int ti, tj;
  tile_of(blockIdx.x, ti, tj);
  const int tid = threadIdx.x, Q = pp.Q;
  const long M = pp.M, N = pp.N, m = (long)ti * PT + tid / PT, mp = (long)tj * PT + tid % PT;
  const bool ok = m < M && mp <= m;
  double zh[QR], g[QR];
  double e1 = 0.0;
#pragma unroll
  for (int q = 0; q < QR; q++) {
    zh[q] = 0.0; g[q] = 0.0;
    if (ok && q < Q) {
      const double a = Z[m * Q + q], b = Z[mp * Q + q], r = (a - b) / pp.l[q];
      zh[q] = 0.5 * (a + b);
      e1 = fma(-0.25 * r, r, e1);
    }
  }
  double pf = pp.variance * pp.variance;
  if (GRAD && ok) pf *= 0.5 * (dL2[m + mp * ld2] + dL2[mp + m * ld2]);
  double acc = 0.0;
  const long n0 = (long)blockIdx.y * nchunk, n1 = min(N, n0 + nchunk);
  const int W = 2 * Q + 2;
  for (long nb = n0; nb < n1; nb += NC) {
    const int nn = (int)min((long)NC, n1 - nb);
    __syncthreads();
    for (int i = tid; i < nn * QR; i += 256) {
      const int r = i / QR, q = i % QR;
      smu[r][q] = q < Q ? mu[(nb + r) * Q + q] : 0.0;
      sd[r][q] = q < Q ? pre[(nb + r) * W + Q + q] : 0.0;
    }
    for (int i = tid; i < nn; i += 256) sld[i] = pre[(nb + i) * W + 2 * Q + 1];
    __syncthreads();
    if (!ok) continue;
    for (int r = 0; r < nn; r++) {
      double e = e1 + sld[r], df[QR];
#pragma unroll
      for (int q = 0; q < QR; q++) {
        df[q] = smu[r][q] - zh[q];
        e = fma(-sd[r][q] * df[q], df[q], e);
      }
      const double v = exp(e);
      acc += v;
      if (GRAD) {
#pragma unroll
        for (int q = 0; q < QR; q++) g[q] = fma(v * sd[r][q], df[q], g[q]);
      }
    }
  }
  const int K = GRAD ? Q + 1 : 1;
  double* o = part + (((long)blockIdx.y * gridDim.x + blockIdx.x) * (PT * PT) + tid) * K;
  o[0] = ok ? pf * acc : 0.0;
  if (GRAD) {
#pragma unroll
    for (int q = 0; q < QR; q++)
      if (q < Q) o[1 + q] = ok ? pf * g[q] : 0.0;
    if (blockIdx.y == 0 && ok) cf[m + mp * ldc] = (m == mp ? 1.0 : 2.0) * pf * exp(e1);
  }
}

// psi2 (n x n, leading dimension ld): the pair sums over the slices in order, the same value on both sides of the
// diagonal; zero outside M x M
__global__ void psi2_finish_kernel(const double* __restrict__ part, int ns, long ntiles, long M, long n,
                                   double* __restrict__ out, long ld) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y;
  if (i >= n) return;
  double v = 0.0;
  if (i < M && j < M) {
    const long slot = pair_slot(max(i, j), min(i, j));
    for (int s = 0; s < ns; s++) v += part[(long)s * ntiles * PT * PT + slot];
  }
  out[i + j * ld] = v;
}

// first row of CTA column s of ms in the per-point pass: rows [row_bound(s), row_bound(s + 1)) hold about 1 / ms of the
// M (M + 1) / 2 pairs
__device__ __forceinline__ long row_bound(int s, int ms, long M) {
  if (s >= ms) return M;
  const double t = 0.5 * (double)M * (double)(M + 1) * s / ms;
  long r = (long)ceil((sqrt(8.0 * t + 1.0) - 1.0) * 0.5);
  while (r > 0 && 0.5 * (double)(r - 1) * (double)r >= t) r--;
  while (r < M && 0.5 * (double)r * (double)(r + 1) < t) r++;
  return r;
}

// one thread per point n, CTA column s: the psi1 sums over m in [s M / ms, (s + 1) M / ms) and the psi2 sums over the
// pairs of the rows [row_bound(s), row_bound(s + 1)), in order, into pn[s][n][4Q + 2]:
//   [sum L1, sum L1 (z - mu)_q, sum L1 (z - mu)_q^2, sum L2, sum L2 (mu - zhat)_q, sum L2 (mu - zhat)_q^2]
// with L1 = dL_dpsi1 psi1 and L2 = cf exp(ld2_n - sum_q d_nq (mu_nq - zhat_q)^2) over ordered pairs (cf carries w)
template <int QR>
__global__ void __launch_bounds__(128) psi_n_kernel(PsiParams pp, const double* __restrict__ mu,
                                                    const double* __restrict__ pre, const double* __restrict__ Z,
                                                    const double* __restrict__ psi1, const double* __restrict__ dL1,
                                                    long sn, long sm, const double* __restrict__ cf, long ldc,
                                                    double* __restrict__ pn) {
  const long n = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= pp.N) return;
  const int Q = pp.Q, s = blockIdx.y, ms = gridDim.y;
  const long M = pp.M, N = pp.N;
  const double* p = pre + n * (2 * Q + 2);
  double* o = pn + ((long)s * N + n) * (4 * Q + 2);
  double mu_[QR];
#pragma unroll
  for (int q = 0; q < QR; q++) mu_[q] = q < Q ? mu[n * Q + q] : 0.0;
  {
    double a[QR], b[QR], L = 0.0;
#pragma unroll
    for (int q = 0; q < QR; q++) { a[q] = 0.0; b[q] = 0.0; }
    const long m0 = s * M / ms, m1 = (s + 1) * M / ms;
    for (long m = m0; m < m1; m++) {
      const double L1 = dL1[n * sn + m * sm] * psi1[n * sn + m * sm];
      L += L1;
#pragma unroll
      for (int q = 0; q < QR; q++)
        if (q < Q) {
          const double df = Z[m * Q + q] - mu_[q], t = L1 * df;
          a[q] += t;
          b[q] = fma(t, df, b[q]);
        }
    }
    o[0] = L;
#pragma unroll
    for (int q = 0; q < QR; q++)
      if (q < Q) { o[1 + q] = a[q]; o[1 + Q + q] = b[q]; }
  }
  double d2[QR], sa[QR], sb[QR], L = 0.0;
#pragma unroll
  for (int q = 0; q < QR; q++) { d2[q] = q < Q ? p[Q + q] : 0.0; sa[q] = 0.0; sb[q] = 0.0; }
  const double ld2n = p[2 * Q + 1];
  const long r1 = row_bound(s + 1, ms, M);
  for (long m = row_bound(s, ms, M); m < r1; m++) {
    double hm[QR];
#pragma unroll
    for (int q = 0; q < QR; q++) hm[q] = q < Q ? fma(-0.5, Z[m * Q + q], mu_[q]) : 0.0;
    for (long mp = 0; mp <= m; mp++) {
      const double c = cf[m + mp * ldc];
      double e = ld2n, df[QR];
#pragma unroll
      for (int q = 0; q < QR; q++) {
        df[q] = q < Q ? fma(-0.5, Z[mp * Q + q], hm[q]) : 0.0;
        e = fma(-d2[q] * df[q], df[q], e);
      }
      const double v = c * exp(e);
      L += v;
#pragma unroll
      for (int q = 0; q < QR; q++) {
        const double t = v * df[q];
        sa[q] += t;
        sb[q] = fma(t, df[q], sb[q]);
      }
    }
  }
  o[1 + 2 * Q] = L;
#pragma unroll
  for (int q = 0; q < QR; q++)
    if (q < Q) { o[2 + 2 * Q + q] = sa[q]; o[2 + 3 * Q + q] = sb[q]; }
}

// per point: the slices summed in order and turned into out[n][3Q + 1] = [dmu (Q), dS (Q), the point's lengthscale terms
// (Q), sum L1 + 2 sum L2] (_psi1compDer :69-79, _psi2compDer :103-134 with the expanded sums written around mu)
__global__ void psi_nfin_kernel(PsiParams pp, const double* __restrict__ S, const double* __restrict__ pre,
                                const double* __restrict__ pn, int ms, double* __restrict__ out) {
  const long n = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= pp.N) return;
  const int Q = pp.Q, K = 4 * Q + 2;
  const long N = pp.N;
  const double* p = pre + n * (2 * Q + 2);
  double L1 = 0.0, L2 = 0.0;
  for (int s = 0; s < ms; s++) { L1 += pn[((long)s * N + n) * K]; L2 += pn[((long)s * N + n) * K + 1 + 2 * Q]; }
  double* o = out + n * (3 * Q + 1);
  for (int q = 0; q < Q; q++) {
    double a = 0.0, b = 0.0, sa = 0.0, sb = 0.0;
    for (int s = 0; s < ms; s++) {
      const double* r = pn + ((long)s * N + n) * K;
      a += r[1 + q]; b += r[1 + Q + q]; sa += r[2 + 2 * Q + q]; sb += r[2 + 3 * Q + q];
    }
    const double d1 = p[q], d2 = p[Q + q], Sq = S[n * Q + q], l = pp.l[q], l2 = l * l;
    o[q] = d1 * a - 2.0 * d2 * sa;
    o[Q + q] = 0.5 * d1 * (d1 * b - L1) + 2.0 * d2 * d2 * sb - d2 * L2;
    o[2 * Q + q] = d1 * l * (d1 * b + Sq / l2 * L1) + 2.0 * l * (Sq * d2 / l2 * L2 + d2 * d2 * sb);
  }
  o[3 * Q] = L1 + 2.0 * L2;
}

// one CTA per inducing point m: dZ[m] = -sum_n L1 (z_m - mu_n) d1_n + sum_m' (-Lp (z_m - z_m') / l^2 + 2 g(m, m')) over
// the pair sums of the gradient pair pass, and the pair part of the lengthscale gradient sum_m' Lp (z_m - z_m')^2 / 2l^3;
// fixed-order block reductions into out[m][2Q]
template <int QR>
__global__ void __launch_bounds__(256, 1) psi_m_kernel(PsiParams pp, const double* __restrict__ mu,
                                                    const double* __restrict__ pre, const double* __restrict__ Z,
                                                    const double* __restrict__ psi1, const double* __restrict__ dL1,
                                                    long sn, long sm, const double* __restrict__ part, int ns,
                                                    long ntiles, double* __restrict__ out) {
  __shared__ double red[8][2 * QR];
  const long m = blockIdx.x, N = pp.N, M = pp.M;
  const int tid = threadIdx.x, Q = pp.Q, W = 2 * Q + 2, K = Q + 1;
  double zm[QR], acc[QR], dl[QR];
#pragma unroll
  for (int q = 0; q < QR; q++) { zm[q] = q < Q ? Z[m * Q + q] : 0.0; acc[q] = 0.0; dl[q] = 0.0; }
  for (long n = tid; n < N; n += 256) {
    const double L1 = dL1[n * sn + m * sm] * psi1[n * sn + m * sm];
#pragma unroll
    for (int q = 0; q < QR; q++)
      if (q < Q) acc[q] -= L1 * (zm[q] - mu[n * Q + q]) * pre[n * W + q];
  }
  for (long mp = tid; mp < M; mp += 256) {
    const long slot = pair_slot(max(m, mp), min(m, mp));
    double Lp = 0.0;
    for (int s = 0; s < ns; s++) Lp += part[((long)s * ntiles * PT * PT + slot) * K];
#pragma unroll
    for (int q = 0; q < QR; q++)
      if (q < Q) {
        double gq = 0.0;
        for (int s = 0; s < ns; s++) gq += part[((long)s * ntiles * PT * PT + slot) * K + 1 + q];
        const double dz = zm[q] - Z[mp * Q + q], l = pp.l[q];
        acc[q] += -Lp * dz / (l * l) + 2.0 * gq;
        dl[q] += Lp * dz * dz / (2.0 * l * l * l);
      }
  }
#pragma unroll
  for (int q = 0; q < QR; q++) {   // butterfly within each warp, then the 8 warps in order
    double a = acc[q], b = dl[q];
    for (int o = 16; o > 0; o >>= 1) {
      a += __shfl_xor_sync(0xffffffffu, a, o);
      b += __shfl_xor_sync(0xffffffffu, b, o);
    }
    if ((tid & 31) == 0) { red[tid >> 5][q] = a; red[tid >> 5][QR + q] = b; }
  }
  __syncthreads();
  if (tid < 2 * Q) {
    const int idx = tid < Q ? tid : QR + tid - Q;
    double v = 0.0;
    for (int w = 0; w < 8; w++) v += red[w][idx];
    out[m * 2 * Q + tid] = v;
  }
}

// the slices of the points for the pair passes: enough CTAs to fill the device, at least NC points per slice
int pair_splits(long N, long ntiles) {
  long ns = (PSI_TARGET_CTAS + ntiles - 1) / ntiles;
  ns = std::min<long>(ns, std::max<long>(1, N / NC));
  return (int)std::max<long>(1, std::min<long>(ns, 64));
}

template <int QR>
int launch_pairs(gpx_ctx* c, bool grad, const PsiParams& pp, const PsiDev& d, const double* dL2, long ld2, long ntiles,
                 int ns, double* part, double* cf, long ldc) {
  const long nchunk = (pp.N + ns - 1) / ns;
  dim3 grid((unsigned)ntiles, (unsigned)ns);
  if (grad)
    psi2_pair_kernel<QR, true><<<grid, PT * PT, 0, c->st>>>(pp, d.mu, d.pre, d.Z, dL2, ld2, nchunk, part, cf, ldc);
  else
    psi2_pair_kernel<QR, false><<<grid, PT * PT, 0, c->st>>>(pp, d.mu, d.pre, d.Z, nullptr, 0, nchunk, part, nullptr, 0);
  return counted(c, 1);
}

template <int QR>
int launch_grad_rest(gpx_ctx* c, const PsiParams& pp, const PsiDev& d, const double* psi1, const double* dL1, long sn,
                     long sm, const double* cf, long ldc, int ms, double* pn, double* outn,
                     const double* part, int ns, long ntiles, double* outm) {
  const unsigned nb = (unsigned)((pp.N + 127) / 128);
  psi_n_kernel<QR><<<dim3(nb, (unsigned)ms), 128, 0, c->st>>>(pp, d.mu, d.pre, d.Z, psi1, dL1, sn, sm, cf, ldc, pn);
  psi_nfin_kernel<<<(unsigned)((pp.N + 255) / 256), 256, 0, c->st>>>(pp, d.S, d.pre, pn, ms, outn);
  psi_m_kernel<QR><<<(unsigned)pp.M, 256, 0, c->st>>>(pp, d.mu, d.pre, d.Z, psi1, dL1, sn, sm, part, ns, ntiles, outm);
  return counted(c, 3);
}

#define PSI_DISPATCH(Q, f, ...) ((Q) <= 8 ? f<8>(__VA_ARGS__) : (Q) <= 12 ? f<12>(__VA_ARGS__) : f<16>(__VA_ARGS__))

}  // namespace

int psi_params(const gpx_kern_part* parts, int nparts, int Q, PsiParams* pp) {
  if (!parts) GPX_FAIL("null argument");
  if (nparts != 1) GPX_FAIL("the psi-statistics take one RBF part");
  const gpx_kern_part& p = parts[0];
  if (p.kind != GPX_RBF) GPX_FAIL("the psi-statistics take an RBF part only");
  if (Q < 1 || Q > PSI_MAX_Q) GPX_FAIL("the psi-statistics take 1 .. 16 latent dimensions");
  if (p.ndims != Q || !p.dims || !p.lengthscale) GPX_FAIL("the RBF part must cover the latent columns 0 .. Q-1 in order");
  for (int q = 0; q < Q; q++)
    if (p.dims[q] != q) GPX_FAIL("the RBF part must cover the latent columns 0 .. Q-1 in order");
  if (!(p.variance > 0.0) || !std::isfinite(p.variance)) GPX_FAIL("the RBF variance must be positive and finite");
  pp->Q = Q;
  pp->ard = p.ard ? 1 : 0;
  pp->variance = p.variance;
  for (int q = 0; q < Q; q++) {
    const double l = p.lengthscale[p.ard ? q : 0];
    if (!(l > 0.0) || !std::isfinite(l)) GPX_FAIL("the RBF lengthscale must be positive and finite");
    pp->l[q] = l;
  }
  return 0;
}

int psi_check_S(const double* S, long n, int Q) {
  if (!S) GPX_FAIL("null argument");
  for (long i = 0; i < n * Q; i++)
    if (!(S[i] > 0.0) || !std::isfinite(S[i])) GPX_FAIL("the latent variances S must be positive and finite");
  return 0;
}

int psi_prep(gpx_ctx* c, const PsiParams& pp, const PsiDev& d) {
  psi_prep_kernel<<<(unsigned)((pp.N + 255) / 256), 256, 0, c->st>>>(pp, d.S, d.pre);
  return counted(c, 1);
}

int psi1_build(gpx_ctx* c, const PsiParams& pp, const PsiDev& d, double* psi1, long sn, long sm) {
  psi1_kernel<<<dim3((unsigned)((pp.N + 255) / 256), (unsigned)pp.M), 256, 0, c->st>>>(pp, d.mu, d.pre, d.Z, psi1, sn, sm);
  return counted(c, 1);
}

int psi2_build(gpx_ctx* c, const PsiParams& pp, const PsiDev& d, double* out, long ld, long Mpad) {
  const long T = (pp.M + PT - 1) / PT, ntiles = T * (T + 1) / 2;
  const int ns = pair_splits(pp.N, ntiles);
  TmpBuf part(c->st);
  GPX_CHECK(part.alloc((size_t)ns * ntiles * PT * PT));
  GPX_CHECK(PSI_DISPATCH(pp.Q, launch_pairs, c, false, pp, d, nullptr, 0, ntiles, ns, part.p, nullptr, 0));
  psi2_finish_kernel<<<dim3((unsigned)((Mpad + 255) / 256), (unsigned)Mpad), 256, 0, c->st>>>(part.p, ns, ntiles, pp.M,
                                                                                            Mpad, out, ld);
  return counted(c, 1);
}

int psi_grads(gpx_ctx* c, const PsiParams& pp, const PsiDev& d, const double* psi1, const double* dL1, long sn, long sm,
              const double* dL2, long ld2, double* grad, double* dZ, double* dmu, double* dS) {
  const long N = pp.N, M = pp.M;
  const int Q = pp.Q;
  const long T = (M + PT - 1) / PT, ntiles = T * (T + 1) / 2;
  const int ns = pair_splits(N, ntiles);
  // the per-point pass: row ranges of about equal pair counts over ms CTA columns
  const long nblk = (N + 127) / 128;
  const int ms = (int)std::max<long>(1, std::min<long>({(PSI_TARGET_CTAS + nblk - 1) / nblk, (long)MAX_NSPLIT, M}));
  TmpBuf part(c->st), cf(c->st), pn(c->st), outn(c->st), outm(c->st);
  GPX_CHECK(part.alloc((size_t)ns * ntiles * PT * PT * (Q + 1)));
  GPX_CHECK(cf.alloc((size_t)M * M));
  GPX_CHECK(pn.alloc((size_t)ms * N * (4 * Q + 2)));
  GPX_CHECK(outn.alloc((size_t)N * (3 * Q + 1)));
  GPX_CHECK(outm.alloc((size_t)M * 2 * Q));
  GPX_CHECK(PSI_DISPATCH(Q, launch_pairs, c, true, pp, d, dL2, ld2, ntiles, ns, part.p, cf.p, M));
  GPX_CHECK(PSI_DISPATCH(Q, launch_grad_rest, c, pp, d, psi1, dL1, sn, sm, cf.p, M, ms, pn.p, outn.p, part.p, ns,
                         ntiles, outm.p));
  std::vector<double> hn((size_t)N * (3 * Q + 1)), hm((size_t)M * 2 * Q);
  GPX_CUDA(cudaMemcpyAsync(hn.data(), outn.p, hn.size() * 8, cudaMemcpyDeviceToHost, c->st));
  GPX_CUDA(cudaMemcpyAsync(hm.data(), outm.p, hm.size() * 8, cudaMemcpyDeviceToHost, c->st));
  GPX_CUDA(cudaStreamSynchronize(c->st));
  std::vector<double> dl((size_t)Q, 0.0);
  double lsum = 0.0;
  for (long n = 0; n < N; n++) {
    const double* o = hn.data() + (size_t)n * (3 * Q + 1);
    for (int q = 0; q < Q; q++) {
      dmu[n * Q + q] = o[q];
      dS[n * Q + q] = o[Q + q];
      dl[q] += o[2 * Q + q];
    }
    lsum += o[3 * Q];
  }
  for (long m = 0; m < M; m++)
    for (int q = 0; q < Q; q++) {
      dZ[m * Q + q] = hm[(size_t)m * 2 * Q + q];
      dl[q] += hm[(size_t)m * 2 * Q + Q + q];
    }
  grad[0] = lsum / pp.variance;
  if (pp.ard) {
    for (int q = 0; q < Q; q++) grad[1 + q] = dl[q];
  } else {
    double t = 0.0;
    for (int q = 0; q < Q; q++) t += dl[q];
    grad[1] = t;
  }
  return 0;
}

}  // namespace gpx

using namespace gpx;

namespace {
// the stand-alone entries' common checks and uploads: mu, S (N x Q), Z (M x Q) and the per-point factors
struct PsiInputs {
  TmpBuf mu, S, Z, pre;
  PsiDev d;
  explicit PsiInputs(cudaStream_t st) : mu(st), S(st), Z(st), pre(st) {}
};
int psi_inputs(gpx_ctx* c, const gpx_kern_part* part, const double* mu, const double* S, int64_t N, const double* Z,
               int64_t M, int Q, PsiParams* pp, PsiInputs& in) {
  if (!c || !part || !mu || !S || !Z) GPX_FAIL("null argument");
  if (N < 1 || M < 1) GPX_FAIL("N and M must be positive");
  GPX_CHECK(psi_params(part, 1, Q, pp));
  GPX_CHECK(psi_check_S(S, N, Q));
  pp->N = N; pp->M = M;
  GPX_CUDA(cudaSetDevice(c->device));
  GPX_CHECK(in.mu.alloc((size_t)N * Q));
  GPX_CHECK(in.S.alloc((size_t)N * Q));
  GPX_CHECK(in.Z.alloc((size_t)M * Q));
  GPX_CHECK(in.pre.alloc((size_t)N * (2 * Q + 2)));
  GPX_CUDA(cudaMemcpyAsync(in.mu.p, mu, (size_t)N * Q * 8, cudaMemcpyHostToDevice, c->st));
  GPX_CUDA(cudaMemcpyAsync(in.S.p, S, (size_t)N * Q * 8, cudaMemcpyHostToDevice, c->st));
  GPX_CUDA(cudaMemcpyAsync(in.Z.p, Z, (size_t)M * Q * 8, cudaMemcpyHostToDevice, c->st));
  in.d.mu = in.mu.p; in.d.S = in.S.p; in.d.Z = in.Z.p; in.d.pre = in.pre.p;
  return psi_prep(c, *pp, in.d);
}
}  // namespace

extern "C" {

int gpx_psi_stats(gpx_ctx* c, const gpx_kern_part* part, const double* mu, const double* S, int64_t N, const double* Z,
                  int64_t M, int Q, double* psi1, double* psi2) {
  if (!psi1 || !psi2) GPX_FAIL("null argument");
  PsiParams pp;
  PsiInputs in(c ? c->st : nullptr);
  GPX_CHECK(psi_inputs(c, part, mu, S, N, Z, M, Q, &pp, in));
  TmpBuf p1(c->st), p2(c->st);
  GPX_CHECK(p1.alloc((size_t)N * M));
  GPX_CHECK(p2.alloc((size_t)M * M));
  GPX_CHECK(psi1_build(c, pp, in.d, p1.p, M, 1));   // row-major N x M, as the host wants it
  GPX_CHECK(psi2_build(c, pp, in.d, p2.p, M, M));
  GPX_CUDA(cudaMemcpyAsync(psi1, p1.p, (size_t)N * M * 8, cudaMemcpyDeviceToHost, c->st));
  GPX_CUDA(cudaMemcpyAsync(psi2, p2.p, (size_t)M * M * 8, cudaMemcpyDeviceToHost, c->st));
  GPX_CUDA(cudaStreamSynchronize(c->st));
  return 0;
}

int gpx_psi_grads(gpx_ctx* c, const gpx_kern_part* part, const double* mu, const double* S, int64_t N, const double* Z,
                  int64_t M, int Q, const double* dL_dpsi0, const double* dL_dpsi1, const double* dL_dpsi2, double* grad,
                  double* dZ, double* dmu, double* dS) {
  if (!dL_dpsi0 || !dL_dpsi1 || !dL_dpsi2 || !grad || !dZ || !dmu || !dS) GPX_FAIL("null argument");
  PsiParams pp;
  PsiInputs in(c ? c->st : nullptr);
  GPX_CHECK(psi_inputs(c, part, mu, S, N, Z, M, Q, &pp, in));
  TmpBuf p1(c->st), d1(c->st), d2(c->st);
  GPX_CHECK(p1.alloc((size_t)N * M));
  GPX_CHECK(d1.alloc((size_t)N * M));
  GPX_CHECK(d2.alloc((size_t)M * M));
  GPX_CUDA(cudaMemcpyAsync(d1.p, dL_dpsi1, (size_t)N * M * 8, cudaMemcpyHostToDevice, c->st));
  GPX_CUDA(cudaMemcpyAsync(d2.p, dL_dpsi2, (size_t)M * M * 8, cudaMemcpyHostToDevice, c->st));
  GPX_CHECK(psi1_build(c, pp, in.d, p1.p, M, 1));
  // dL_dpsi2 row-major is its transpose column-major: the passes read the symmetrised matrix, the same either way
  GPX_CHECK(psi_grads(c, pp, in.d, p1.p, d1.p, M, 1, d2.p, M, grad, dZ, dmu, dS));
  double s0 = 0.0;
  for (int64_t n = 0; n < N; n++) s0 += dL_dpsi0[n];
  grad[0] += s0;   // psi0 = variance (rbf_psi_comp.py:60)
  return 0;
}

}  // extern "C"
