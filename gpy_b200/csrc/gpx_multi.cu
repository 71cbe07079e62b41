// gpx_multi.cu — composite kernels (sums of products of stationary / StdPeriodic / White / Bias parts) evaluated on the device:
// covariance build, gradient reductions from the stored K^-1 and the final assembly. See gpx_multi.cuh for the references.
#include <algorithm>
#include <cstring>

#include "gpx_common.cuh"
#include "gpx_multi.cuh"

namespace gpx {

// ---------------------------------------------------------------------------------------------------------------
// prep: every part's active dims stacked as SoA rows, plus per-part squared norms. A stationary part's dims are scaled the
// way its own Stationary._scaled_dist does (stationary.py:151-168: ARD divides by the lengthscale before the expansion, iso
// afterwards). A StdPeriodic part's dims stay unscaled: its argument pi (x - x') / T is formed from raw differences like
// standard_periodic.py:130 does, so that time-like inputs (years near 2000, period 1) keep the digits the reference keeps.
// ---------------------------------------------------------------------------------------------------------------
__global__ void prep_multi_kernel(const double* __restrict__ X, long N, int Dfull, long ld, MultiKern mk,
                                  double* __restrict__ XsT, double* __restrict__ sq) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ld) return;
  for (int p = 0; p < mk.nparts; p++) {
    const PartDev& pd = mk.part[p];
    const bool scale = pd.ard && is_stationary(pd.kind);
    double s = 0.0;
    for (int q = 0; q < pd.D; q++) {
      double v = 0.0;
      if (i < N) {
        v = X[i * Dfull + mk.dims[pd.xoff + q]];
        if (scale) v = v / mk.ls[pd.xoff + q];
      }
      XsT[(long)(pd.xoff + q) * ld + i] = v;
      s += v * v;
    }
    sq[(long)p * ld + i] = s;
  }
}

int launch_prep_multi(const double* X, long N, int Dfull, long ld, const MultiKern& mk, double* XsT, double* sq,
                      cudaStream_t st) {
  prep_multi_kernel<<<(unsigned)((ld + 255) / 256), 256, 0, st>>>(X, N, Dfull, ld, mk, XsT, sq);
  GPX_CUDA(cudaGetLastError());
  return 0;
}

// scaled distance r of a stationary part at a pair of points held in shared-memory tiles (row point il, column point jl)
__device__ __forceinline__ double part_r(const MultiKern& mk, int p, const double* sR, const double* sC, const double* sSr,
                                         const double* sSc, int il, int jl, bool samept) {
  const PartDev& pd = mk.part[p];
  double dot = 0.0;
  for (int q = 0; q < pd.D; q++) dot = fma(sR[(pd.xoff + q) * TILE + il], sC[(pd.xoff + q) * TILE + jl], dot);
  double r2 = sSr[p * TILE + il] + sSc[p * TILE + jl] - 2.0 * dot;
  if (samept) r2 = 0.0;
  r2 = fmax(r2, 0.0);
  return sqrt(r2) * pd.inv_ls_iso;
}

// RatQuad at unit variance: k = (1 + r^2/2)^-power, dk/dr = -power r (1 + r^2/2)^(-power-1) (stationary.py:785-793);
// lg = log1p(r^2/2) is what the power gradient needs (:797)
__device__ __forceinline__ void ratquad_k_dk(double power, double r, double& k, double& dk, double& lg) {
  lg = log1p(0.5 * r * r);
  k = exp(-power * lg);
  dk = -power * r * exp(-(power + 1.0) * lg);
}

// StdPeriodic at unit variance (standard_periodic.py:125-132): exp(-1/2 sum_q (sin(pi d_q / T_q) / l_q)^2)
__device__ __forceinline__ double periodic_k(const MultiKern& mk, const PartDev& pd, const double* sR, const double* sC, int il,
                                             int jl) {
  double arg = 0.0;
  for (int q = 0; q < pd.D; q++) {
    const double d = sR[(pd.xoff + q) * TILE + il] - sC[(pd.xoff + q) * TILE + jl];
    const double t = sinpi(d / mk.period[pd.xoff + q]) / mk.ls[pd.xoff + q];
    arg = fma(t, t, arg);
  }
  return exp(-0.5 * arg);
}

// value of one part at unit variance, static kinds: White = variance on coincident points of the SAME set
// (static.py:75-79), Bias = variance (static.py:155-157). EXT: the kernel may contain RatQuad / StdPeriodic parts; the
// instantiations without them keep the code (and the register budget) of the kinds RBF .. Matern52, White, Bias.
template <bool EXT>
__device__ __forceinline__ double part_value(const MultiKern& mk, int p, const double* sR, const double* sC, const double* sSr,
                                             const double* sSc, int il, int jl, bool samept) {
  const PartDev& pd = mk.part[p];
  if (pd.kind == GPX_BIAS) return 1.0;
  if (pd.kind == GPX_WHITE) return samept ? 1.0 : 0.0;
  if (EXT && pd.kind == GPX_STDPERIODIC) return periodic_k(mk, pd, sR, sC, il, jl);
  const double rr = part_r(mk, p, sR, sC, sSr, sSc, il, jl, samept);
  if (EXT && pd.kind == GPX_RATQUAD) return exp(-pd.power * log1p(0.5 * rr * rr));
  return k_of_r_unit(pd.kind, rr);
}

__device__ __forceinline__ void load_tiles(const MultiKern& mk, const double* rowsT, long ld_rows, const double* sq_rows, int rt,
                                           const double* colsT, long ld_cols, const double* sq_cols, int ct, double* sR,
                                           double* sC, double* sSr, double* sSc) {
  for (int idx = threadIdx.x; idx < mk.sumD * TILE; idx += blockDim.x) {
    const int q = idx / TILE, m = idx % TILE;
    sR[idx] = rowsT[(long)q * ld_rows + (long)rt * TILE + m];
    sC[idx] = colsT[(long)q * ld_cols + (long)ct * TILE + m];
  }
  for (int idx = threadIdx.x; idx < mk.nparts * TILE; idx += blockDim.x) {
    const int q = idx / TILE, m = idx % TILE;
    sSr[idx] = sq_rows[(long)q * ld_rows + (long)rt * TILE + m];
    sSc[idx] = sq_cols[(long)q * ld_cols + (long)ct * TILE + m];
  }
}

// ---------------------------------------------------------------------------------------------------------------
// covariance build: K = sum_t prod_{p in t} k_p (add.py:60-74, prod.py:59-68), `sym` mode = factor workspace image
// (lower tiles, zero upper tiles, identity padding, + (noise + jitter) on the diagonal: exact_gaussian_inference.py:55-56)
// ---------------------------------------------------------------------------------------------------------------
template <bool EXT>
__global__ void __launch_bounds__(256) kbuild_multi_kernel(KBuildMultiParams p) {
  extern __shared__ __align__(128) unsigned char km_smem[];
  const MultiKern& mk = p.mk;
  double* sR = reinterpret_cast<double*>(km_smem);
  double* sC = sR + (size_t)mk.sumD * TILE;
  double* sSr = sC + (size_t)mk.sumD * TILE;
  double* sSc = sSr + (size_t)mk.nparts * TILE;
  const int ct = blockIdx.x, rt = blockIdx.y;
  const int tid = threadIdx.x, il = tid & (TILE - 1), half = tid >> 7;
  const long gi = (long)rt * TILE + il;
  double* outp = p.out + gi + ((long)ct * TILE + half * 64) * p.ld;
  if (p.sym && rt < ct) {
#pragma unroll 8
    for (int j = 0; j < 64; j++) outp[(long)j * p.ld] = 0.0;
    return;
  }
  load_tiles(mk, p.rowsT, p.ld_rows, p.sq_rows, rt, p.colsT, p.ld_cols, p.sq_cols, ct, sR, sC, sSr, sSc);
  __syncthreads();
  const bool row_valid = gi < p.nrows;
  for (int j = 0; j < 64; j++) {
    const int jl = half * 64 + j;
    const long gj = (long)ct * TILE + jl;
    const bool samept = p.same && gi == gj;
    double val = 0.0, prod = 1.0;
    int cur = mk.part[0].term;
    for (int q = 0; q < mk.nparts; q++) {
      if (mk.part[q].term != cur) { val += prod; prod = 1.0; cur = mk.part[q].term; }
      prod *= mk.part[q].variance * part_value<EXT>(mk, q, sR, sC, sSr, sSc, il, jl, samept);
    }
    val += prod;
    if (p.sym) {
      if (gi == gj) val += p.diag_add;
      if (!row_valid || gj >= p.ncols) val = (gi == gj) ? 1.0 : 0.0;
      outp[(long)j * p.ld] = val;
    } else if (row_valid && gj < p.ncols) {
      outp[(long)j * p.ld] = val;
    }
  }
}

constexpr int MAX_NRED = MAX_D + 3;   // largest part_nred: an ARD RatQuad part on 64 dims

// any RatQuad / StdPeriodic part: the kernels' EXT instantiation
static bool has_ext(const MultiKern& mk) {
  for (int q = 0; q < mk.nparts; q++)
    if (mk.part[q].kind == GPX_RATQUAD || mk.part[q].kind == GPX_STDPERIODIC) return true;
  return false;
}

static int max_nred(const MultiKern& mk) {
  int m = 0;
  for (int q = 0; q < mk.nparts; q++) m = std::max(m, part_nred(mk.part[q]));
  return m;
}
static size_t multi_tile_smem(const MultiKern& mk) {
  return (size_t)(2 * mk.sumD + 2 * mk.nparts) * TILE * 8 + 8 * (size_t)max_nred(mk) * 8;
}
static constexpr int MAX_MULTI_SMEM = (2 * MAX_D + 2 * MAX_PARTS) * TILE * 8 + 8 * MAX_NRED * 8;

template <bool EXT>
static int launch_kbm_t(const KBuildMultiParams& p, int row_tiles, int col_tiles, cudaStream_t st) {
  static bool attr_set = false;
  if (!attr_set) {
    GPX_CUDA(cudaFuncSetAttribute(kbuild_multi_kernel<EXT>, cudaFuncAttributeMaxDynamicSharedMemorySize, MAX_MULTI_SMEM));
    attr_set = true;
  }
  kbuild_multi_kernel<EXT><<<dim3(col_tiles, row_tiles), 256, multi_tile_smem(p.mk), st>>>(p);
  GPX_CUDA(cudaGetLastError());
  return 0;
}

int launch_kbuild_multi(const KBuildMultiParams& p, int row_tiles, int col_tiles, cudaStream_t st) {
  return has_ext(p.mk) ? launch_kbm_t<true>(p, row_tiles, col_tiles, st) : launch_kbm_t<false>(p, row_tiles, col_tiles, st);
}

// ---------------------------------------------------------------------------------------------------------------
// gradient reductions of ONE part: the part sees dL_dK o prod(other factors of its term) (prod.py:377-396; add.py:76-99
// passes dL_dK through unchanged) and reduces it exactly like Stationary.update_gradients_full (stationary.py:193-243),
// RatQuad's (stationary.py:795-798: power sum of dL * -k log1p(r^2/2)), StdPeriodic's (standard_periodic.py:501-526),
// White (static.py:88-92: trace) or Bias (static.py:172-173: sum). Two sources of dL_dK share the per-pair work below:
// 1/2 (alpha alpha^T - P K^-1) from the stored K^-1 (grad_kinv_multi) and a caller's dense matrix (grad_full_multi).
// ---------------------------------------------------------------------------------------------------------------
struct PairSums {   // per-thread sums of one part, besides the per-dim accumulators
  double var = 0.0, iso = 0.0, power = 0.0, noise = 0.0;
};

// one pair (row point il, column point jl) with dL_dK entry dl and weight w (2 for an off-diagonal tile of a symmetric
// sweep). xi: the row point's stacked inputs of the part. gq: ARD lengthscale sums of a stationary part; a StdPeriodic part
// keeps its period sums in gq[0, DREG/2) and its lengthscale sums in gq[DREG/2, DREG) (the launch picks DREG >= 2 D).
template <int DREG, bool EXT>
__device__ __forceinline__ void pair_accumulate(const MultiKern& mk, int pidx, const PartDev& me, const double* sR,
                                                const double* sC, const double* sSr, const double* sSc, int il, int jl,
                                                bool samept, double w, double dl, const double (&xi)[DREG],
                                                double (&gq)[DREG], PairSums& s) {
  for (int q = 0; q < mk.nparts; q++)       // the other factors of this part's term
    if (q != pidx && mk.part[q].term == me.term)
      dl *= mk.part[q].variance * part_value<EXT>(mk, q, sR, sC, sSr, sSc, il, jl, samept);
  if (EXT && me.kind == GPX_STDPERIODIC) {
    constexpr int H = DREG / 2;
    const double k = periodic_k(mk, me, sR, sC, il, jl);
    s.var = fma(w * k, dl, s.var);
    const double W = w * me.variance * k * dl;
#pragma unroll
    for (int q = 0; q < H; q++)
      if (q < me.D) {
        const double T = mk.period[me.xoff + q], l = mk.ls[me.xoff + q];
        const double u = (xi[q] - sC[(me.xoff + q) * TILE + jl]) / T;
        double sn, cs;
        sincospi(u, &sn, &cs);
        const double base = 3.141592653589793 * u;
        gq[q] = fma(W, sn * cs * (base / T) / (l * l), gq[q]);          // standard_periodic.py:511,518-521
        gq[H + q] = fma(W, sn * sn / (l * l * l), gq[H + q]);            // :513,523-526
      }
    return;
  }
  double rr = 0.0, k, dk = 0.0;
  if (is_static(me.kind)) {
    k = part_value<EXT>(mk, pidx, sR, sC, sSr, sSc, il, jl, samept);
  } else {
    rr = part_r(mk, pidx, sR, sC, sSr, sSc, il, jl, samept);
    if (EXT && me.kind == GPX_RATQUAD) {
      double lg;
      ratquad_k_dk(me.power, rr, k, dk, lg);
      s.power = fma(w * dl, -me.variance * k * lg, s.power);
    } else {
      k_dk_of_r_unit(me.kind, rr, k, dk);
    }
  }
  s.var = fma(w * k, dl, s.var);
  const double G = me.variance * dk * dl;
  if (me.ard && is_stationary(me.kind)) {
    const double tmpv = (rr != 0.0) ? w * G / rr : 0.0;     // stationary.py:205,225-232: 1/r with 1/0 := 0
#pragma unroll
    for (int q = 0; q < DREG; q++)
      if (q < me.D) {
        const double df = xi[q] - sC[(me.xoff + q) * TILE + jl];
        gq[q] = fma(tmpv, df * df, gq[q]);
      }
  } else {
    s.iso = fma(w * G, rr, s.iso);
  }
}

// the CTA's sums of one part into out[part_nred], in the order of its gradient block, tr(dL_dK) last. All threads call it.
template <int DREG, bool EXT>
__device__ __forceinline__ void store_part_sums(const PartDev& me, PairSums s, double (&gq)[DREG], double* sRed, double* out) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int nred = part_nred(me);
  const int nl = me.ard ? me.D : 1;
  double* red = sRed + warp * nred;
  s.var = warp_sum(s.var);
  s.noise = warp_sum(s.noise);
  if (lane == 0) { red[0] = s.var; red[nred - 1] = s.noise; }
  if (EXT && me.kind == GPX_STDPERIODIC) {
    constexpr int H = DREG / 2;
    const int np = me.ard_period ? me.D : 1;
    double tp = 0.0, tl = 0.0;
#pragma unroll
    for (int q = 0; q < H; q++)
      if (q < me.D) {
        const double a = warp_sum(gq[q]), b = warp_sum(gq[H + q]);
        tp += a; tl += b;
        if (lane == 0 && me.ard_period) red[1 + q] = a;
        if (lane == 0 && me.ard) red[1 + np + q] = b;
      }
    if (lane == 0 && !me.ard_period) red[1] = tp;                 // isotropic: summed over the dims (:520-521,:525-526)
    if (lane == 0 && !me.ard) red[1 + np] = tl;
  } else if (me.ard && is_stationary(me.kind)) {
#pragma unroll
    for (int q = 0; q < DREG; q++)
      if (q < me.D) {
        const double v = warp_sum(gq[q]);
        if (lane == 0) red[1 + q] = v;
      }
  } else {
    s.iso = warp_sum(s.iso);
    if (lane == 0) red[1] = s.iso;
  }
  if (EXT && me.kind == GPX_RATQUAD) {
    s.power = warp_sum(s.power);
    if (lane == 0) red[1 + nl] = s.power;
  }
  __syncthreads();
  if (tid < nred) {
    double v = 0.0;
#pragma unroll
    for (int wdx = 0; wdx < 8; wdx++) v += sRed[wdx * nred + tid];
    out[tid] = v;
  }
}

// One CTA per lower 128 x 128 tile of the stored K^-1, thread-mapped index = row (contiguous in K^-1). The narrowest
// instantiation without RatQuad / StdPeriodic parts keeps three CTAs per SM, as before those kinds existed.
template <int DREG, bool EXT>
__global__ void __launch_bounds__(256, DREG == 8 ? (EXT ? 2 : 3) : 1) grad_kinv_multi_kernel(GradKinvMultiParams p) {
  extern __shared__ __align__(128) unsigned char gm_smem[];
  const MultiKern& mk = p.mk;
  const int P = p.P;
  double* sR = reinterpret_cast<double*>(gm_smem);
  double* sC = sR + (size_t)mk.sumD * TILE;
  double* sSr = sC + (size_t)mk.sumD * TILE;
  double* sSc = sSr + (size_t)mk.nparts * TILE;
  double* sRed = sSc + (size_t)mk.nparts * TILE;      // [8 warps][nred]
  int r = (int)((sqrtf(8.f * (float)blockIdx.x + 1.f) - 1.f) * 0.5f);
  while (r * (r + 1) / 2 > (int)blockIdx.x) --r;
  while ((r + 1) * (r + 2) / 2 <= (int)blockIdx.x) ++r;
  const int c = blockIdx.x - r * (r + 1) / 2;
  const int tid = threadIdx.x;
  load_tiles(mk, p.XsT, p.ldx, p.sq, r, p.XsT, p.ldx, p.sq, c, sR, sC, sSr, sSc);
  __syncthreads();
  const PartDev me = mk.part[p.part];
  const int il = tid & (TILE - 1), half = tid >> 7;
  const long gi = (long)r * TILE + il;
  double xi[DREG], gq[DREG];
#pragma unroll
  for (int q = 0; q < DREG; q++) { gq[q] = 0.0; xi[q] = q < me.D ? sR[(me.xoff + q) * TILE + il] : 0.0; }
  const double w = (r > c) ? 2.0 : 1.0;
  PairSums s;
  const double* kcol = p.Kinv + gi + ((long)c * TILE + half * 64) * p.ld;
  if (gi < p.N) {
    for (int jj = 0; jj < 64; jj++) {
      const int jl = half * 64 + jj;
      const long gj = (long)c * TILE + jl;
      if (gj >= p.N) break;
      const bool samept = gi == gj;
      const double kinv = kcol[(long)jj * p.ld];
      double aa = 0.0;
      for (int q = 0; q < P; q++) aa = fma(p.alpha[(long)q * p.ldx + gi], p.alpha[(long)q * p.ldx + gj], aa);
      const double dl = 0.5 * (aa - (double)P * kinv);
      if (samept) s.noise += dl;
      pair_accumulate<DREG, EXT>(mk, p.part, me, sR, sC, sSr, sSc, il, jl, samept, w, dl, xi, gq, s);
    }
  }
  if (!p.want_noise) s.noise = 0.0;
  store_part_sums<DREG, EXT>(me, s, gq, sRed, p.partials + ((long)r * p.nt + c) * part_nred(me));
}

// One CTA per 128 x 128 tile of a caller's dense dL_dK: thread-mapped index = row point (contiguous in dL_dK).
template <int DREG, bool EXT>
__global__ void __launch_bounds__(256) grad_full_multi_kernel(GradFullMultiParams p) {
  extern __shared__ __align__(128) unsigned char gf_smem[];
  const MultiKern& mk = p.mk;
  double* sR = reinterpret_cast<double*>(gf_smem);
  double* sC = sR + (size_t)mk.sumD * TILE;
  double* sSr = sC + (size_t)mk.sumD * TILE;
  double* sSc = sSr + (size_t)mk.nparts * TILE;
  double* sRed = sSc + (size_t)mk.nparts * TILE;
  const int ct = blockIdx.x, rt = blockIdx.y;
  const int tid = threadIdx.x;
  load_tiles(mk, p.rowsT, p.ld_rows, p.sq_rows, rt, p.colsT, p.ld_cols, p.sq_cols, ct, sR, sC, sSr, sSc);
  __syncthreads();
  const PartDev me = mk.part[p.part];
  const int il = tid & (TILE - 1), half = tid >> 7;
  const long gi = (long)rt * TILE + il;
  double xi[DREG], gq[DREG];
#pragma unroll
  for (int q = 0; q < DREG; q++) { gq[q] = 0.0; xi[q] = q < me.D ? sR[(me.xoff + q) * TILE + il] : 0.0; }
  PairSums s;
  if (gi < p.nrows) {
    for (int jj = 0; jj < 64; jj++) {
      const int jl = half * 64 + jj;
      const long gj = (long)ct * TILE + jl;
      if (gj >= p.ncols) break;
      pair_accumulate<DREG, EXT>(mk, p.part, me, sR, sC, sSr, sSc, il, jl, p.same && gi == gj, 1.0, p.dL[gj * p.ldd + gi], xi,
                                 gq, s);
    }
  }
  store_part_sums<DREG, EXT>(me, s, gq, sRed, p.partials + ((long)ct * gridDim.y + rt) * part_nred(me));
}

// register accumulators for a part: its active dims and its per-dim sums (part_nacc <= MAX_D, checked by the caller)
static int dreg_for(const PartDev& pd) { return std::max(pd.D, part_nacc(pd)); }

template <int DREG, bool EXT>
static int launch_gkm_t(const GradKinvMultiParams& p, unsigned grid, size_t smem, cudaStream_t st) {
  static bool attr_set = false;
  if (!attr_set) {
    GPX_CUDA(cudaFuncSetAttribute(grad_kinv_multi_kernel<DREG, EXT>, cudaFuncAttributeMaxDynamicSharedMemorySize, MAX_MULTI_SMEM));
    attr_set = true;
  }
  grad_kinv_multi_kernel<DREG, EXT><<<grid, 256, smem, st>>>(p);
  GPX_CUDA(cudaGetLastError());
  return 0;
}

int launch_grad_kinv_multi(const GradKinvMultiParams& p, cudaStream_t st) {
  const int D = dreg_for(p.mk.part[p.part]);
  const unsigned grid = (unsigned)(p.nt * (p.nt + 1) / 2);
  const size_t smem = multi_tile_smem(p.mk);
  if (has_ext(p.mk)) {
    if (D <= 8) return launch_gkm_t<8, true>(p, grid, smem, st);
    if (D <= 16) return launch_gkm_t<16, true>(p, grid, smem, st);
    if (D <= 32) return launch_gkm_t<32, true>(p, grid, smem, st);
    return launch_gkm_t<64, true>(p, grid, smem, st);
  }
  if (D <= 8) return launch_gkm_t<8, false>(p, grid, smem, st);
  if (D <= 16) return launch_gkm_t<16, false>(p, grid, smem, st);
  if (D <= 32) return launch_gkm_t<32, false>(p, grid, smem, st);
  return launch_gkm_t<64, false>(p, grid, smem, st);
}

template <int DREG, bool EXT>
static int launch_gfm_t(const GradFullMultiParams& p, dim3 grid, size_t smem, cudaStream_t st) {
  static bool attr_set = false;
  if (!attr_set) {
    GPX_CUDA(cudaFuncSetAttribute(grad_full_multi_kernel<DREG, EXT>, cudaFuncAttributeMaxDynamicSharedMemorySize, MAX_MULTI_SMEM));
    attr_set = true;
  }
  grad_full_multi_kernel<DREG, EXT><<<grid, 256, smem, st>>>(p);
  GPX_CUDA(cudaGetLastError());
  return 0;
}

int launch_grad_full_multi(const GradFullMultiParams& p, int row_tiles, int col_tiles, cudaStream_t st) {
  const int D = dreg_for(p.mk.part[p.part]);
  const dim3 grid(col_tiles, row_tiles);
  const size_t smem = multi_tile_smem(p.mk);
  if (has_ext(p.mk)) {
    if (D <= 8) return launch_gfm_t<8, true>(p, grid, smem, st);
    if (D <= 16) return launch_gfm_t<16, true>(p, grid, smem, st);
    if (D <= 32) return launch_gfm_t<32, true>(p, grid, smem, st);
    return launch_gfm_t<64, true>(p, grid, smem, st);
  }
  if (D <= 8) return launch_gfm_t<8, false>(p, grid, smem, st);
  if (D <= 16) return launch_gfm_t<16, false>(p, grid, smem, st);
  if (D <= 32) return launch_gfm_t<32, false>(p, grid, smem, st);
  return launch_gfm_t<64, false>(p, grid, smem, st);
}

// ---------------------------------------------------------------------------------------------------------------
// gradients_X of a composite kernel: Add.gradients_X sums the parts' (add.py:88-100), Prod.gradients_X hands each factor
// dL_dK times the other factors (prod.py:397-407), and a stationary factor reduces it like Stationary.gradients_X
// (stationary.py:325-345): tmp = variance (1/r) dk/dr dL (1/0 := 0), grad[n, d] = sum_m tmp (x_n,d - x_m,d) / l^2. White
// and Bias have no input gradient and enter as factors only. The layout is gradx_kernel's: one CTA = 128 row points x one
// column chunk, dL_dK tiles of 128 x 32 through shared memory, per-chunk partials per stacked row reduced in fixed order.
// The row points' stacked inputs sit in shared memory (each thread reads its own column), the chunk's 32 column points
// beside them. Kinds RBF .. Matern52, White and Bias only: the caller rejects RatQuad / StdPeriodic parts.
// ---------------------------------------------------------------------------------------------------------------
// scaled distance of stationary part p between row point il (stride TILE) and chunk column point mm (stride 32)
__device__ __forceinline__ double gx_part_r(const PartDev& pd, int p, const double* sR, const double* sC, const double* sSr,
                                            const double* sSc, int il, int mm, bool samept) {
  double dot = 0.0;
  for (int q = 0; q < pd.D; q++) dot = fma(sR[(pd.xoff + q) * TILE + il], sC[(pd.xoff + q) * 32 + mm], dot);
  double r2 = sSr[p * TILE + il] + sSc[p * 32 + mm] - 2.0 * dot;
  if (samept) r2 = 0.0;
  return sqrt(fmax(r2, 0.0)) * pd.inv_ls_iso;
}

// one pair (row point il, chunk column point mm) with weight dl into the row point's stacked-row sums acc
template <int DREG>
__device__ __forceinline__ void gx_pair(const MultiKern& mk, const double* sR, const double* sC, const double* sSr,
                                        const double* sSc, int il, int mm, bool samept, double dl, double (&acc)[DREG]) {
  for (int pi = 0; pi < mk.nparts; pi++) {
    const PartDev& pd = mk.part[pi];
    if (!is_stationary(pd.kind)) continue;
    const double rr = gx_part_r(pd, pi, sR, sC, sSr, sSc, il, mm, samept);
    if (rr == 0.0) continue;
    double kk, dk;
    k_dk_of_r_unit(pd.kind, rr, kk, dk);
    double t = pd.variance * dk * dl / rr;
    for (int q = 0; q < mk.nparts; q++) {          // the other factors of this part's term
      const PartDev& o = mk.part[q];
      if (q == pi || o.term != pd.term) continue;
      const double v = o.kind == GPX_BIAS ? 1.0
                       : o.kind == GPX_WHITE ? (samept ? 1.0 : 0.0)
                       : k_of_r_unit(o.kind, gx_part_r(o, q, sR, sC, sSr, sSc, il, mm, samept));
      t *= o.variance * v;
    }
#pragma unroll
    for (int q = 0; q < DREG; q++)
      if (q >= pd.xoff && q < pd.xoff + pd.D) acc[q] = fma(t, sR[q * TILE + il] - sC[q * 32 + mm], acc[q]);
  }
}

template <int DREG>
__global__ void __launch_bounds__(TILE) gradx_multi_kernel(GradXMultiParams p, long mchunk, double* __restrict__ part) {
  extern __shared__ __align__(128) unsigned char gxm_smem[];
  const MultiKern& mk = p.mk;
  double (*sdl)[33] = reinterpret_cast<double (*)[33]>(gxm_smem);   // [128][33] dL_dK tile
  double* sR = reinterpret_cast<double*>(gxm_smem) + TILE * 33;     // [sumD][128] row points
  double* sSr = sR + (size_t)mk.sumD * TILE;                        // [nparts][128]
  double* sC = sSr + (size_t)mk.nparts * TILE;                      // [sumD][32] column chunk
  double* sSc = sC + (size_t)mk.sumD * 32;                          // [nparts][32]
  const int tid = threadIdx.x;
  const long r0 = (long)blockIdx.x * TILE, n = r0 + tid;
  const long m_beg = (long)blockIdx.y * mchunk;
  const long m_end = m_beg + mchunk < p.ncols ? m_beg + mchunk : p.ncols;
  for (int q = 0; q < mk.sumD; q++) sR[q * TILE + tid] = p.rowsT[(long)q * p.ld_rows + n];
  for (int q = 0; q < mk.nparts; q++) sSr[q * TILE + tid] = p.sq_rows[(long)q * p.ld_rows + n];
  double acc[DREG];
#pragma unroll
  for (int q = 0; q < DREG; q++) acc[q] = 0.0;
  for (long m0 = m_beg; m0 < m_end; m0 += 32) {
    __syncthreads();
    if (!p.transposed) {
      for (int rr = tid >> 5; rr < TILE; rr += TILE / 32) {
        const long gn = r0 + rr, gm = m0 + (tid & 31);
        double dv = 0.0;
        if (gn < p.nrows && gm < m_end) dv = p.dL[gn * p.ldd + gm];
        sdl[rr][tid & 31] = dv;
      }
    } else {
      for (int mm = 0; mm < 32; mm++) {
        const long gm = m0 + mm;
        double dv = 0.0;
        if (n < p.nrows && gm < m_end) dv = p.dL[gm * p.ldd + n];
        sdl[tid][mm] = dv;
      }
    }
    for (int idx = tid; idx < mk.sumD * 32; idx += TILE) {
      const int q = idx >> 5, mm = idx & 31;
      sC[idx] = (m0 + mm < p.ncols) ? p.colsT[(long)q * p.ld_cols + m0 + mm] : 0.0;
    }
    for (int idx = tid; idx < mk.nparts * 32; idx += TILE) {
      const int q = idx >> 5, mm = idx & 31;
      sSc[idx] = (m0 + mm < p.ncols) ? p.sq_cols[(long)q * p.ld_cols + m0 + mm] : 0.0;
    }
    __syncthreads();
    if (n < p.nrows) {
      const int mlim = (int)((m_end - m0) < 32 ? (m_end - m0) : 32);
      for (int mm = 0; mm < mlim; mm++) {
        const long gm = m0 + mm;
        const bool samept = p.same && n == gm;
        double dl = sdl[tid][mm];
        if (p.same) dl += p.dL[gm * p.ldd + n];                  // tmp + tmp^T (stationary.py:334-336)
        gx_pair<DREG>(mk, sR, sC, sSr, sSc, tid, mm, samept, dl, acc);
      }
    }
  }
  if (n < p.nrows) {
#pragma unroll
    for (int q = 0; q < DREG; q++)
      if (q < mk.sumD) part[((long)blockIdx.y * p.nrows + n) * mk.sumD + q] = acc[q];
  }
}

// gradients_X of the exact evaluation's kernel at its own training points (gpx_exact_grad_X): gradx_multi_kernel's layout
// and rules with the symmetric weight W = dL_dK + dL_dK^T = alpha alpha^T - P K^-1 formed per 128 x 32 tile in shared
// memory. The K^-1 tile comes from the stored lower tiles (a column tile right of the row tile is read transposed, 32
// contiguous doubles per warp); alpha of the chunk's 32 points is staged in slabs of 32 outputs, so any P fits, and each
// thread adds alpha[c][n] alpha[c][m] to its own row of the tile in output order.
template <int DREG>
__global__ void __launch_bounds__(TILE, 1) exact_gradx_kernel(ExactGradXParams p, long mchunk, double* __restrict__ part) {
  extern __shared__ __align__(128) unsigned char egx_smem[];
  const MultiKern& mk = p.mk;
  double (*sw)[33] = reinterpret_cast<double (*)[33]>(egx_smem);    // [128][33] W tile
  double* sA = reinterpret_cast<double*>(egx_smem) + TILE * 33;     // [32][32] alpha slab: [output][chunk point]
  double* sR = sA + 32 * 32;                                        // [sumD][128] row points
  double* sSr = sR + (size_t)mk.sumD * TILE;                        // [nparts][128]
  double* sC = sSr + (size_t)mk.nparts * TILE;                      // [sumD][32] column chunk
  double* sSc = sC + (size_t)mk.sumD * 32;                          // [nparts][32]
  const int tid = threadIdx.x;
  const long r0 = (long)blockIdx.x * TILE, n = r0 + tid;
  const long m_beg = (long)blockIdx.y * mchunk;
  const long m_end = m_beg + mchunk < p.N ? m_beg + mchunk : p.N;
  const double negP = -(double)p.P;
  for (int q = 0; q < mk.sumD; q++) sR[q * TILE + tid] = p.XsT[(long)q * p.ldx + n];
  for (int q = 0; q < mk.nparts; q++) sSr[q * TILE + tid] = p.sq[(long)q * p.ldx + n];
  double acc[DREG];
#pragma unroll
  for (int q = 0; q < DREG; q++) acc[q] = 0.0;
  for (long m0 = m_beg; m0 < m_end; m0 += 32) {
    __syncthreads();
    if (m0 / TILE <= (long)blockIdx.x) {   // stored tile: element (n, m) at Kinv[n + m ld], row n thread-contiguous
      for (int mm = 0; mm < 32; mm++) {
        const long gm = m0 + mm;
        sw[tid][mm] = (n < p.N && gm < m_end) ? negP * p.Kinv[n + gm * p.ld] : 0.0;
      }
    } else {                               // above the diagonal tiles: element (m, n) of the stored tile
      for (int rr = tid >> 5; rr < TILE; rr += TILE / 32) {
        const long gn = r0 + rr, gm = m0 + (tid & 31);
        sw[rr][tid & 31] = (gn < p.N && gm < m_end) ? negP * p.Kinv[gm + gn * p.ld] : 0.0;
      }
    }
    for (int idx = tid; idx < mk.sumD * 32; idx += TILE) {
      const int q = idx >> 5, mm = idx & 31;
      sC[idx] = (m0 + mm < p.N) ? p.XsT[(long)q * p.ldx + m0 + mm] : 0.0;
    }
    for (int idx = tid; idx < mk.nparts * 32; idx += TILE) {
      const int q = idx >> 5, mm = idx & 31;
      sSc[idx] = (m0 + mm < p.N) ? p.sq[(long)q * p.ldx + m0 + mm] : 0.0;
    }
    for (int c0 = 0; c0 < p.P; c0 += 32) {
      __syncthreads();                     // the tile is written and the previous slab consumed
      for (int idx = tid; idx < 32 * 32; idx += TILE) {
        const int c = c0 + (idx >> 5), mm = idx & 31;
        sA[idx] = (c < p.P && m0 + mm < m_end) ? p.alpha[(long)c * p.ldx + m0 + mm] : 0.0;
      }
      __syncthreads();
      if (n < p.N) {
        const int cl = p.P - c0 < 32 ? p.P - c0 : 32;
        for (int c = 0; c < cl; c++) {
          const double an = p.alpha[(long)(c0 + c) * p.ldx + n];
          for (int mm = 0; mm < 32; mm++) sw[tid][mm] = fma(an, sA[c * 32 + mm], sw[tid][mm]);
        }
      }
    }
    if (n < p.N) {
      const int mlim = (int)((m_end - m0) < 32 ? (m_end - m0) : 32);
      for (int mm = 0; mm < mlim; mm++) {
        const long gm = m0 + mm;
        gx_pair<DREG>(mk, sR, sC, sSr, sSc, tid, mm, n == gm, sw[tid][mm], acc);
      }
    }
  }
  if (n < p.N) {
#pragma unroll
    for (int q = 0; q < DREG; q++)
      if (q < mk.sumD) part[((long)blockIdx.y * p.N + n) * mk.sumD + q] = acc[q];
  }
}

// out[n, d] = sum over the stationary parts' stacked rows q on data column d, in part order, of the chunk sums (fixed order)
// divided by l_q (ARD: the points were scaled) or l^2 (iso)
__global__ void gradx_multi_reduce_kernel(const double* __restrict__ part, long N, int nchunk, int Dfull, MultiKern mk,
                                          double* __restrict__ out) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * Dfull) return;
  const long n = i / Dfull;
  const int d = (int)(i % Dfull);
  double s = 0.0;
  for (int pi = 0; pi < mk.nparts; pi++) {
    const PartDev& pd = mk.part[pi];
    if (!is_stationary(pd.kind)) continue;
    for (int q = pd.xoff; q < pd.xoff + pd.D; q++) {
      if (mk.dims[q] != d) continue;
      double t = 0.0;
      for (int c = 0; c < nchunk; c++) t += part[((long)c * N + n) * mk.sumD + q];
      const double l = mk.ls[q];
      s += pd.ard ? t / l : t / (l * l);
    }
  }
  out[i] = s;
}

template <int DREG>
static int launch_gxm_t(const GradXMultiParams& p, dim3 grid, size_t smem, long mchunk, double* part, cudaStream_t st) {
  static bool attr_set = false;
  if (!attr_set) {
    const int mx = (TILE * 33 + (MAX_D + MAX_PARTS) * (TILE + 32)) * 8;
    GPX_CUDA(cudaFuncSetAttribute(gradx_multi_kernel<DREG>, cudaFuncAttributeMaxDynamicSharedMemorySize, mx));
    attr_set = true;
  }
  gradx_multi_kernel<DREG><<<grid, TILE, smem, st>>>(p, mchunk, part);
  GPX_CUDA(cudaGetLastError());
  return 0;
}

int launch_gradx_multi(const GradXMultiParams& p, int nchunk, long mchunk, double* part, double* out, cudaStream_t st) {
  const MultiKern& mk = p.mk;
  if (has_ext(mk)) { set_error("gradients_X: RatQuad / StdPeriodic parts have no input gradient on the device"); return -2; }
  const size_t smem = (size_t)(TILE * 33 + (mk.sumD + mk.nparts) * (TILE + 32)) * 8;
  const dim3 grid((unsigned)((p.nrows + TILE - 1) / TILE), nchunk);
  const int D = mk.sumD;
  int rc;
  if (D <= 8) rc = launch_gxm_t<8>(p, grid, smem, mchunk, part, st);
  else if (D <= 16) rc = launch_gxm_t<16>(p, grid, smem, mchunk, part, st);
  else if (D <= 32) rc = launch_gxm_t<32>(p, grid, smem, mchunk, part, st);
  else rc = launch_gxm_t<64>(p, grid, smem, mchunk, part, st);
  if (rc) return rc;
  gradx_multi_reduce_kernel<<<(unsigned)((p.nrows * p.Dfull + 255) / 256), 256, 0, st>>>(part, p.nrows, nchunk, p.Dfull, mk,
                                                                                         out);
  GPX_CUDA(cudaGetLastError());
  return 0;
}

template <int DREG>
static int launch_egx_t(const ExactGradXParams& p, dim3 grid, size_t smem, long mchunk, double* part, cudaStream_t st) {
  static bool attr_set = false;
  if (!attr_set) {
    const int mx = (TILE * 33 + 32 * 32 + (MAX_D + MAX_PARTS) * (TILE + 32)) * 8;
    GPX_CUDA(cudaFuncSetAttribute(exact_gradx_kernel<DREG>, cudaFuncAttributeMaxDynamicSharedMemorySize, mx));
    attr_set = true;
  }
  exact_gradx_kernel<DREG><<<grid, TILE, smem, st>>>(p, mchunk, part);
  GPX_CUDA(cudaGetLastError());
  return 0;
}

int launch_exact_gradx(const ExactGradXParams& p, int nchunk, long mchunk, double* part, double* out, cudaStream_t st) {
  const MultiKern& mk = p.mk;
  if (has_ext(mk)) { set_error("gradients_X: RatQuad / StdPeriodic parts have no input gradient on the device"); return -2; }
  const size_t smem = (size_t)(TILE * 33 + 32 * 32 + (mk.sumD + mk.nparts) * (TILE + 32)) * 8;
  const dim3 grid((unsigned)((p.N + TILE - 1) / TILE), nchunk);
  const int D = mk.sumD;
  int rc;
  if (D <= 8) rc = launch_egx_t<8>(p, grid, smem, mchunk, part, st);
  else if (D <= 16) rc = launch_egx_t<16>(p, grid, smem, mchunk, part, st);
  else if (D <= 32) rc = launch_egx_t<32>(p, grid, smem, mchunk, part, st);
  else rc = launch_egx_t<64>(p, grid, smem, mchunk, part, st);
  if (rc) return rc;
  gradx_multi_reduce_kernel<<<(unsigned)((p.N * p.Dfull + 255) / 256), 256, 0, st>>>(part, p.N, nchunk, p.Dfull, mk, out);
  GPX_CUDA(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// predictive gradients (GPy/core/gp.py:438-474): the Jacobians of the predictive mean and variance at the test points,
// in gradx_multi_kernel's layout and with its per-pair rules. Row points (one per thread, 128 per CTA) are the test
// points, column points the training / inducing points in chunks of 32. Each pair forms r and dk/dr of every stationary
// part once and feeds up to NCH channels: channel c < P is the mean of output c (the pair weighted by alpha[c][n], a
// broadcast column), channel P the Schur term of the variance (weighted by V[n, m], a 128 x 32 tile through shared
// memory). White is zero between the test and the training set (static.py:75-79), so a term holding it contributes
// nothing; Bias enters as its variance. A launch covers channels [c0, c0 + NCH); its per-chunk partials are reduced in
// fixed order by pred_grad_reduce_kernel.
// ---------------------------------------------------------------------------------------------------------------
template <int DREG, int NCH>
__global__ void __launch_bounds__(TILE) pred_grad_kernel(PredGradParams p, int c0, long mchunk, double* __restrict__ part) {
  extern __shared__ __align__(128) unsigned char pg_smem[];
  const MultiKern& mk = p.mk;
  double (*sv)[33] = reinterpret_cast<double (*)[33]>(pg_smem);     // [128][33] V tile
  double* sR = reinterpret_cast<double*>(pg_smem) + TILE * 33;      // [sumD][128] test points
  double* sSr = sR + (size_t)mk.sumD * TILE;                        // [nparts][128]
  double* sC = sSr + (size_t)mk.nparts * TILE;                      // [sumD][32] column chunk
  double* sSc = sC + (size_t)mk.sumD * 32;                          // [nparts][32]
  double* sA = sSc + (size_t)mk.nparts * 32;                        // [NCH][32] alpha of the chunk's points
  const int tid = threadIdx.x;
  const long r0 = (long)blockIdx.x * TILE, m = r0 + tid;
  const long n_beg = (long)blockIdx.y * mchunk;
  const long n_end = n_beg + mchunk < p.ncols ? n_beg + mchunk : p.ncols;
  const int nch = NCH < p.P + 1 - c0 ? NCH : p.P + 1 - c0;
  const bool has_var = c0 + nch == p.P + 1;                         // the variance channel is the last one
  for (int q = 0; q < mk.sumD; q++) sR[q * TILE + tid] = p.rowsT[(long)q * p.ld_rows + m];
  for (int q = 0; q < mk.nparts; q++) sSr[q * TILE + tid] = p.sq_rows[(long)q * p.ld_rows + m];
  double acc[NCH][DREG];
#pragma unroll
  for (int c = 0; c < NCH; c++)
#pragma unroll
    for (int q = 0; q < DREG; q++) acc[c][q] = 0.0;
  for (long n0 = n_beg; n0 < n_end; n0 += 32) {
    __syncthreads();
    if (has_var) {
      for (int rr = tid >> 5; rr < TILE; rr += TILE / 32) {
        const long gm = r0 + rr, gn = n0 + (tid & 31);
        sv[rr][tid & 31] = (gm < p.nrows && gn < n_end) ? p.V[gm * p.ldv + gn] : 0.0;
      }
    }
    for (int idx = tid; idx < mk.sumD * 32; idx += TILE) {
      const int q = idx >> 5, mm = idx & 31;
      sC[idx] = (n0 + mm < p.ncols) ? p.colsT[(long)q * p.ld_cols + n0 + mm] : 0.0;
    }
    for (int idx = tid; idx < mk.nparts * 32; idx += TILE) {
      const int q = idx >> 5, mm = idx & 31;
      sSc[idx] = (n0 + mm < p.ncols) ? p.sq_cols[(long)q * p.ld_cols + n0 + mm] : 0.0;
    }
    for (int idx = tid; idx < NCH * 32; idx += TILE) {
      const int c = c0 + (idx >> 5), mm = idx & 31;
      sA[idx] = (c < p.P && n0 + mm < n_end) ? p.alpha[(long)c * p.lda + n0 + mm] : 0.0;
    }
    __syncthreads();
    if (m < p.nrows) {
      const int mlim = (int)((n_end - n0) < 32 ? (n_end - n0) : 32);
      for (int mm = 0; mm < mlim; mm++) {
        for (int pi = 0; pi < mk.nparts; pi++) {
          const PartDev& pd = mk.part[pi];
          if (!is_stationary(pd.kind)) continue;
          const double rr = gx_part_r(pd, pi, sR, sC, sSr, sSc, tid, mm, false);
          if (rr == 0.0) continue;
          double kk, dk;
          k_dk_of_r_unit(pd.kind, rr, kk, dk);
          double t = pd.variance * dk / rr;
          for (int q = 0; q < mk.nparts; q++) {          // the other factors of this part's term
            const PartDev& o = mk.part[q];
            if (q == pi || o.term != pd.term) continue;
            const double v = o.kind == GPX_BIAS ? 1.0
                             : o.kind == GPX_WHITE ? 0.0
                             : k_of_r_unit(o.kind, gx_part_r(o, q, sR, sC, sSr, sSc, tid, mm, false));
            t *= o.variance * v;
          }
#pragma unroll
          for (int c = 0; c < NCH; c++) {
            if (c >= nch) break;
            const double w = t * (c0 + c < p.P ? sA[c * 32 + mm] : sv[tid][mm]);
#pragma unroll
            for (int q = 0; q < DREG; q++)
              if (q >= pd.xoff && q < pd.xoff + pd.D) acc[c][q] = fma(w, sR[q * TILE + tid] - sC[q * 32 + mm], acc[c][q]);
          }
        }
      }
    }
  }
  if (m < p.nrows) {
#pragma unroll
    for (int c = 0; c < NCH; c++) {
      if (c >= nch) break;
#pragma unroll
      for (int q = 0; q < DREG; q++)
        if (q < mk.sumD) part[(((long)(c0 + c) * gridDim.y + blockIdx.y) * p.nrows + m) * mk.sumD + q] = acc[c][q];
    }
  }
}

// out: dmu[m, d, c] (nrows x Dfull x P row-major), then dvar[m, d] (nrows x Dfull): per channel and data column the
// chunk sums of the stacked rows on that column, in part order, divided by l_q or l^2 as gradx_multi_reduce_kernel does;
// the variance channel times -2 (gp.py:460-462; gradients_X_diag is zero for these kinds, stationary.py:360-361)
__global__ void pred_grad_reduce_kernel(const double* __restrict__ part, long M, int nchunk, int P, int Dfull, MultiKern mk,
                                        double* __restrict__ out) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * Dfull * (P + 1)) return;
  const long m = i / ((long)Dfull * (P + 1));
  const int d = (int)((i / (P + 1)) % Dfull), c = (int)(i % (P + 1));
  double s = 0.0;
  for (int pi = 0; pi < mk.nparts; pi++) {
    const PartDev& pd = mk.part[pi];
    if (!is_stationary(pd.kind)) continue;
    for (int q = pd.xoff; q < pd.xoff + pd.D; q++) {
      if (mk.dims[q] != d) continue;
      double t = 0.0;
      for (int ch = 0; ch < nchunk; ch++) t += part[(((long)c * nchunk + ch) * M + m) * mk.sumD + q];
      const double l = mk.ls[q];
      s += pd.ard ? t / l : t / (l * l);
    }
  }
  if (c < P) out[(m * Dfull + d) * P + c] = s;
  else out[M * Dfull * P + m * Dfull + d] = -2.0 * s;
}

// channels per launch: (P + 1) x DREG accumulators where up to 32 fit, else channel groups (one launch each)
static int pred_grad_nch(int sumD) { return sumD <= 8 ? 4 : sumD <= 16 ? 2 : 1; }

int pred_grad_launches(const MultiKern& mk, int P) {
  const int g = pred_grad_nch(mk.sumD);
  return (P + 1 + g - 1) / g + 1;
}

template <int DREG, int NCH>
static int launch_pg_t(const PredGradParams& p, dim3 grid, size_t smem, long mchunk, double* part, cudaStream_t st) {
  static bool attr_set = false;
  if (!attr_set) {
    const int mx = (TILE * 33 + (MAX_D + MAX_PARTS) * (TILE + 32) + NCH * 32) * 8;
    GPX_CUDA(cudaFuncSetAttribute(pred_grad_kernel<DREG, NCH>, cudaFuncAttributeMaxDynamicSharedMemorySize, mx));
    attr_set = true;
  }
  for (int c0 = 0; c0 < p.P + 1; c0 += NCH) {
    pred_grad_kernel<DREG, NCH><<<grid, TILE, smem, st>>>(p, c0, mchunk, part);
    GPX_CUDA(cudaGetLastError());
  }
  return 0;
}

int launch_pred_grad(const PredGradParams& p, int nchunk, long mchunk, double* part, double* out, cudaStream_t st) {
  const MultiKern& mk = p.mk;
  if (has_ext(mk)) { set_error("gradients_X: RatQuad / StdPeriodic parts have no input gradient on the device"); return -2; }
  const int nch = pred_grad_nch(mk.sumD);
  const size_t smem = (size_t)(TILE * 33 + (mk.sumD + mk.nparts) * (TILE + 32) + nch * 32) * 8;
  const dim3 grid((unsigned)((p.nrows + TILE - 1) / TILE), nchunk);
  const int D = mk.sumD;
  int rc;
  if (D <= 8) rc = launch_pg_t<8, 4>(p, grid, smem, mchunk, part, st);
  else if (D <= 16) rc = launch_pg_t<16, 2>(p, grid, smem, mchunk, part, st);
  else if (D <= 32) rc = launch_pg_t<32, 1>(p, grid, smem, mchunk, part, st);
  else rc = launch_pg_t<64, 1>(p, grid, smem, mchunk, part, st);
  if (rc) return rc;
  const long tot = p.nrows * p.Dfull * (p.P + 1);
  pred_grad_reduce_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(part, p.nrows, nchunk, p.P, p.Dfull, mk, out);
  GPX_CUDA(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// final assembly: fixed-order sums of the per-tile partials of every part, log-determinant, quadratic form
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) finalize_multi_kernel(FinalizeMultiParams f) {
  __shared__ double sh[256];
  const int tid = threadIdx.x;
  auto block_sum = [&](double s) {
    sh[tid] = s;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) { if (tid < o) sh[tid] += sh[tid + o]; __syncthreads(); }
    const double tot = sh[0];
    __syncthreads();
    return tot;
  };
  double s = 0.0;
  for (long i = tid; i < f.nt; i += 256) s += f.logdet_part[i];
  const double logdet = block_sum(s);
  s = 0.0;
  for (int q = 0; q < f.P; q++)
    for (long i = tid; i < f.N; i += 256) { const double x = f.T[(long)q * f.ld + i]; s = fma(x, x, s); }
  const double quad = block_sum(s);
  if (tid == 0) {
    const double log2pi = 1.8378770664093453;
    f.res[0] = 0.5 * (-(double)f.N * f.P * log2pi - (double)f.P * logdet - quad);
    f.res[1] = logdet;
    f.res[2] = quad;
  }
  int off = 4;
  for (int p = 0; p < f.mk.nparts; p++) {
    const int nred = part_nred(f.mk.part[p]);
    for (int t = 0; t < nred; t++) {
      s = 0.0;
      for (long i = tid; i < f.ntiles; i += 256) s += f.partials[p][i * nred + t];
      const double tot = block_sum(s);
      double v;
      if (tid == 0) {
        if (t == nred - 1) { if (p == 0) f.res[3] = tot; }                             // tr(dL_dK) -> noise (gaussian.py:78-79)
        else if (part_grad_entry(f.mk, p, t, tot, &v)) f.res[off + t] = v;
      }
    }
    off += part_ngrad(f.mk.part[p]);
  }
}

int launch_finalize_multi(const FinalizeMultiParams& f, cudaStream_t st) {
  finalize_multi_kernel<<<1, 256, 0, st>>>(f);
  GPX_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace gpx
