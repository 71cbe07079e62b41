// gpx_gemm.cu — the one fp64 tensor-core GEMM of the engine:  C(tile r,c) (op)= A_r * B_c^T  (NT form).
//
// Every O(N^3) step of the exact-GP evaluation is expressed through this kernel (see DESIGN.md §4):
//   GEMM_UPDATE : S(r,c) -= P_r P_c^T      trailing update of the unified factor-and-invert sweep
//                                          (replaces LAPACK dpotrf's dsyrk/dgemm and dtrtri's trmm, GPy/util/linalg.py:58,209)
//   GEMM_PANEL  : P(r,c') = S(r,panel) Linv_kk^T   panel "solve" as a product with the inverted diagonal block
//   GEMM_LAUUM  : Kinv(r,c) = sum_{k>=r} U_rk U_ck^T   (replaces dpotri, linalg.py:142,210) with the FUSED epilogue that
//                 reduces dL_dK -> (variance, lengthscale, noise) gradients (replaces exact_gaussian_inference.py:70-72,
//                 stationary.py:193-243, stationary_cython.pyx:53-62, likelihoods/gaussian.py:78-79) without writing K^-1.
//
// Machine mapping (sm_90a): wgmma has no f64 kind, so the fp64 tensor path is DMMA.16x8x4 (mma.sync m16n8k4,
// the sm_90 shape: twice the issue rate of the older m8n8k4 on the H100).
// A 128x128 CTA tile is computed by 8 consumer warps (64x32 each, 64 fp64 accumulators per lane); a 9th producer
// warp streams 16-deep k-slabs of both operands into a 4-stage shared-memory ring with 1-D bulk async copies
// (cp.async.bulk -> SASS UBLKCP, the TMA engine) signalled through mbarriers. Operands are m-contiguous
// (column-major), a slab column is one 1 KiB bulk copy; the smem pitch of 132 doubles makes the DMMA fragment
// loads bank-conflict free.
#include <algorithm>
#include <cstdlib>

#include "gpx_common.cuh"

namespace gpx {

constexpr int SLAB_DOUBLES = KSLAB * PITCH;                       // one operand, one stage
constexpr int PIPE_BYTES = 2 * STAGES * SLAB_DOUBLES * 8;         // 135168
constexpr int BAR_BYTES = 128;                                    // 2*STAGES mbarriers at the front of the dynamic smem
// epilogue footprint of the LAUUM kernel: staged accumulators + input tiles + alpha tiles + reduction scratch
static int epi_bytes(int D, int P) {
  const int nphase = D > 32 ? 2 : 1;
  return (64 * (CONSUMER_WARPS * 32 / nphase) + (2 * D + 2 + 2 * P) * TILE + CONSUMER_WARPS * (D + 3)) * 8;
}
constexpr int SMEM_PIPE = BAR_BYTES + PIPE_BYTES;
constexpr int SMEM_MAX = 227 * 1024;
constexpr int SB = 11;   // super-block edge of the tile schedule (SB*SB = 121 <= 132 SMs)

size_t gemm_smem_bytes() { return SMEM_PIPE; }

__device__ __forceinline__ void consumer_bar() { asm volatile("bar.sync 1, %0;" ::"n"(CONSUMER_WARPS * 32) : "memory"); }

// Tile schedule. UPDATE / LAUUM run on a 1-D grid decoded through SB x SB super-blocks so that the ~132 CTAs in flight
// share <= 2*SB row panels and SB column panels (operand streams stay L2-resident). LAUUM enumerates the super-blocks of
// the lower triangle row by row: small r first = longest k-ranges first, so the tail of the launch is made of short tiles.
// block-mapped operand base of row tile r (see GemmParams)
__device__ __forceinline__ long mapped_offset(const GemmParams& p, int r) {
  const int R = r / p.map_blk, t = r % p.map_blk;
  const long pos = (long)(R % p.map_G) * p.map_npr + R / p.map_G;
  return pos * p.map_stride + (long)t * TILE;
}

// LAUUM k-tile sequence of tile row r: all k-tiles >= r, or (multi-GPU) those inside the owned column blocks.
struct KSeq { int first, n0, kb0; };
__device__ __forceinline__ int kseq_init(const GemmParams& p, int r, KSeq& q) {
  if (p.k_G <= 1) { q.first = r; q.n0 = p.nt - r; q.kb0 = 0; return p.nt - r; }
  const int nblk = p.nt / p.k_blk;
  const int kbmin = r / p.k_blk;
  q.kb0 = kbmin + ((p.k_g - kbmin) % p.k_G + p.k_G) % p.k_G;
  if (q.kb0 >= nblk) { q.first = 0; q.n0 = 0; return 0; }
  const int t0 = q.kb0 == kbmin ? r - kbmin * p.k_blk : 0;
  q.first = q.kb0 * p.k_blk + t0;
  q.n0 = p.k_blk - t0;
  return q.n0 + ((nblk - 1 - q.kb0) / p.k_G) * p.k_blk;
}
__device__ __forceinline__ int kseq_tile(const GemmParams& p, const KSeq& q, int j) {
  if (p.k_G <= 1 || j < q.n0) return q.first + j;
  const int jj = j - q.n0;
  return (q.kb0 + p.k_G * (1 + jj / p.k_blk)) * p.k_blk + jj % p.k_blk;
}

template <int MODE>
__device__ __forceinline__ bool decode_tile(const GemmParams& p, int& r, int& c) {
  if (MODE == GEMM_UPDATE) {
    const int ncols = p.ncols > 0 ? p.ncols : p.nt - p.c0;
    const int sbcols = (ncols + SB - 1) / SB;
    const int sb = blockIdx.x / (SB * SB), t = blockIdx.x % (SB * SB);
    const int slot = (sb / sbcols) * SB + t / SB;
    const int col = (sb % sbcols) * SB + t % SB;
    if (col >= ncols) return false;
    c = p.c0 + col;
    r = slot < p.rlow ? slot : c + (slot - p.rlow);
    if (r >= p.nt) return false;
    return p.own_G <= 1 || ((r / p.own_blk) % p.own_G) == p.own_g;
  } else if (MODE == GEMM_LAUUM) {
    const int sb = blockIdx.x / (SB * SB), t = blockIdx.x % (SB * SB);
    int R = (int)((sqrtf(8.f * (float)sb + 1.f) - 1.f) * 0.5f);
    while (R * (R + 1) / 2 > sb) --R;
    while ((R + 1) * (R + 2) / 2 <= sb) ++R;
    const int C = sb - R * (R + 1) / 2;
    r = R * SB + t / SB;
    c = C * SB + t % SB;
    return r < p.nt && c <= r;
  } else if (p.plain) {  // general product: 1-D grid, SB x SB super-blocks over (row tiles nt) x (column tiles ncols)
    const int sbcols = (p.ncols + SB - 1) / SB;
    const int sb = blockIdx.x / (SB * SB), t = blockIdx.x % (SB * SB);
    r = (sb / sbcols) * SB + t / SB;
    c = (sb % sbcols) * SB + t % SB;
    return r < p.nt && c < p.ncols && !(p.plain == 2 && r < c);
  } else {  // GEMM_PANEL: 2-D grid (output column tile, row slot); triangular B: longest k-range first
    c = p.tri ? (int)gridDim.x - 1 - (int)blockIdx.x : (int)blockIdx.x;
    const int slot = blockIdx.y;
    r = slot < p.skip0 ? slot : slot + (p.skip1 - p.skip0);
    if (r >= p.nt) return false;
    return p.own_G <= 1 || ((r / p.own_blk) % p.own_G) == p.own_g;
  }
}

template <int MODE>
__device__ __forceinline__ void gemm_nt_body(const GemmParams& p) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw);
  uint64_t* empty = full + STAGES;
  double* sA = reinterpret_cast<double*>(smem_raw + BAR_BYTES);
  double* sB = sA + STAGES * SLAB_DOUBLES;

  // ---- tile mapping (decode_tile) ---------------------------------------------------------------------------------
  int r, c;
  if (!decode_tile<MODE>(p, r, c)) return;
  int nkt;
  KSeq kq;
  kq.first = 0; kq.n0 = 1 << 30; kq.kb0 = 0;
  if (MODE == GEMM_UPDATE) {
    nkt = p.K / TILE;
  } else if (MODE == GEMM_LAUUM) {
    nkt = kseq_init(p, r, kq);
  } else {
    nkt = p.tri == 1 ? (c + 1) : (p.tri == 2 ? (r + 1) : p.K / TILE);   // tri 1: B lower triangular, 2: A lower triangular
  }
  const double* Aptr = p.A + (p.map_A ? mapped_offset(p, r) : (p.loc_A ? loc_tile(r, p.own_G, p.own_blk) : (long)r) * TILE);
  const double* Bptr = p.B + (p.map_B ? mapped_offset(p, c) : (long)c * TILE);
  const long lda = p.lda, ldb = p.ldb;
  const int nslab = nkt * (TILE / KSLAB);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
#pragma unroll
    for (int s = 0; s < STAGES; s++) { mbar_init(&full[s], 1); mbar_init(&empty[s], CONSUMER_WARPS); }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp >= CONSUMER_WARPS) {
    // ================= producer warpgroup: hands its registers to the consumers, then warp 8 streams the slabs ====
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp != CONSUMER_WARPS) return;
    // one bulk copy per lane per stage (16 A columns + 16 B columns)
    const bool isA = lane < KSLAB;
    const int kc = lane & (KSLAB - 1);
    const double* src_base = isA ? Aptr : Bptr;
    const long ld = isA ? lda : ldb;
    double* dst_base = (isA ? sA : sB) + kc * PITCH;
    for (int it = 0; it < nslab; ++it) {
      const int s = it % STAGES;
      const uint32_t n = it / STAGES;
      if (it >= STAGES) mbar_wait(&empty[s], (n & 1) ^ 1);
      if (lane == 0) mbar_arrive_expect_tx(&full[s], 2 * KSLAB * TILE * 8);
      __syncwarp();
      long kt = MODE == GEMM_LAUUM ? kseq_tile(p, kq, it >> 3) : (it >> 3);
      if (MODE == GEMM_LAUUM && p.k_local) kt = loc_tile((int)kt, p.k_G, p.k_blk);
      const long k = kt * TILE + (it & 7) * KSLAB + kc;
      bulk_g2s(dst_base + s * SLAB_DOUBLES, src_base + k * ld, TILE * 8, &full[s]);
    }
    return;
  }

  // ================= consumer warps (two warpgroups, 232 registers each after the hand-over) =====================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int wm = warp & 1, wn = warp >> 1;   // 2 x 4 warps -> 64 x 32 sub-tiles
  const int g = lane >> 2, tg = lane & 3;
  double acc[8][4][2];
  if (MODE == GEMM_UPDATE) {
    // C -= A B^T  ==  C + (-A) B^T : the accumulators start from the old C tile (loads overlap the pipeline fill),
    // the A fragments are negated on the way in, and the epilogue is store-only.
    const double* Ct = p.C + (p.map_C ? mapped_offset(p, r) : (p.loc_C ? loc_tile(r, p.own_G, p.own_blk) : (long)r) * TILE) +
                       (long)c * TILE * p.ldc;
#pragma unroll
    for (int mb = 0; mb < 8; mb++)
#pragma unroll
      for (int nb = 0; nb < 4; nb++)
#pragma unroll
        for (int e = 0; e < 2; e++)
          acc[mb][nb][e] = Ct[wm * 64 + mb * 8 + g + (long)(wn * 32 + nb * 8 + 2 * tg + e) * p.ldc];
  } else {
#pragma unroll
    for (int mb = 0; mb < 8; mb++)
#pragma unroll
      for (int nb = 0; nb < 4; nb++) { acc[mb][nb][0] = 0.0; acc[mb][nb][1] = 0.0; }
  }

  for (int it = 0; it < nslab; ++it) {
    const int s = it % STAGES;
    const uint32_t n = it / STAGES;
    mbar_wait(&full[s], n & 1);
    const double* a = sA + s * SLAB_DOUBLES + wm * 64 + g;
    const double* b = sB + s * SLAB_DOUBLES + wn * 32 + g;
#pragma unroll
    for (int k4 = 0; k4 < KSLAB / 4; k4++) {
      const int kk = (k4 * 4 + tg) * PITCH;
      double af[8], bf[4];
#pragma unroll
      for (int mb = 0; mb < 8; mb++) af[mb] = (MODE == GEMM_UPDATE) ? -a[kk + mb * 8] : a[kk + mb * 8];
#pragma unroll
      for (int nb = 0; nb < 4; nb++) bf[nb] = b[kk + nb * 8];
#pragma unroll
      for (int mb = 0; mb < 8; mb += 2)
#pragma unroll
        for (int nb = 0; nb < 4; nb++) dmma1684(acc[mb][nb][0], acc[mb][nb][1], acc[mb + 1][nb][0], acc[mb + 1][nb][1],
                                                          af[mb], af[mb + 1], bf[nb]);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[s]);
  }

  // ================= epilogues ===============================================================================
  if (MODE != GEMM_LAUUM) {
    decode_tile<MODE>(p, r, c);
    double* Ct = p.C + (p.map_C ? mapped_offset(p, r) : (p.loc_C ? loc_tile(r, p.own_G, p.own_blk) : (long)r) * TILE) +
                 (long)c * TILE * p.ldc;
#pragma unroll
    for (int mb = 0; mb < 8; mb++) {
      const int i = wm * 64 + mb * 8 + g;
#pragma unroll
      for (int nb = 0; nb < 4; nb++)
#pragma unroll
        for (int e = 0; e < 2; e++) Ct[i + (long)(wn * 32 + nb * 8 + 2 * tg + e) * p.ldc] = acc[mb][nb][e];
    }
    return;
  }

  // ---- LAUUM: fused dL_dK -> gradient reductions ---------------------------------------------------------------
  // The accumulators are staged through shared memory (thread-private columns, conflict-free) and the per-element
  // work runs as a ROLLED loop: unrolled over the 64 accumulators it was ~160 KB of straight-line code per tile and
  // the kernel stalled on instruction fetch (ncu: stalled_no_instruction ~1.1 per issue, DMMA pipe 83 % vs 93 %).
  decode_tile<MODE>(p, r, c);   // recomputed here so that r, c are not live across the main loop
  if (p.partials == nullptr) {   // plain K^-1 = U U^T (gpx_pdinv): store the lower tile, no reductions
    double* ko = p.kinv_out + (long)r * TILE + (long)c * TILE * p.ldc;
#pragma unroll
    for (int mb = 0; mb < 8; mb++)
#pragma unroll
      for (int nb = 0; nb < 4; nb++)
#pragma unroll
        for (int e = 0; e < 2; e++)
          ko[wm * 64 + mb * 8 + g + (long)(wn * 32 + nb * 8 + 2 * tg + e) * p.ldc] = acc[mb][nb][e];
    return;
  }
  const int D = p.kp.D, P = p.P;
  const int nl = p.kp.ard ? D : 1;
  const int nred = nl + 2;
  const int nphase = D > 32 ? 2 : 1;            // large D: the two 64-row halves take turns in the staging area
  const int sthr = CONSUMER_WARPS * 32 / nphase;  // threads per phase
  consumer_bar();  // every consumer is done reading the pipeline buffers; reuse them
  double* sSt = reinterpret_cast<double*>(smem_raw + BAR_BYTES);          // [64][sthr] staged accumulators
  double* sXr = sSt + 64 * sthr;
  double* sXc = sXr + D * TILE;
  double* sSr = sXc + D * TILE;
  double* sSc = sSr + TILE;
  double* sAr = sSc + TILE;
  double* sAc = sAr + P * TILE;
  double* sRed = sAc + P * TILE;
  const int tid = threadIdx.x;
  for (int idx = tid; idx < D * TILE; idx += CONSUMER_WARPS * 32) {
    const int q = idx / TILE, m = idx % TILE;
    sXr[idx] = p.XsT[(long)q * p.ldx + (long)r * TILE + m];
    sXc[idx] = p.XsT[(long)q * p.ldx + (long)c * TILE + m];
  }
  for (int idx = tid; idx < P * TILE; idx += CONSUMER_WARPS * 32) {
    const int q = idx / TILE, m = idx % TILE;
    sAr[idx] = p.alpha[(long)q * p.ldx + (long)r * TILE + m];
    sAc[idx] = p.alpha[(long)q * p.ldx + (long)c * TILE + m];
  }
  if (tid < TILE) { sSr[tid] = p.sq[(long)r * TILE + tid]; sSc[tid] = p.sq[(long)c * TILE + tid]; }

  const double w = (r > c) ? 2.0 : 1.0;   // strictly-lower tiles stand for their mirror image as well
  const bool alpha_here = p.k_G <= 1 || p.k_g == 0;
  const int kind = p.kp.kind;
  const double variance = p.kp.variance, inv_ls = p.kp.inv_ls_iso;
  const bool ard = p.kp.ard != 0;
  double gvar = 0.0, giso = 0.0, gnoise = 0.0;
  double* kout = p.kinv_out ? p.kinv_out + (long)r * TILE + (long)c * TILE * p.ldc : nullptr;
  double* red = sRed + warp * nred;
  const int lt = nphase == 1 ? tid : (warp >> 1) * 32 + lane;   // thread slot inside the staging area
  double* st = sSt + lt;
  const int i0 = wm * 64 + g, j0 = wn * 32 + 2 * tg;

  for (int ph = 0; ph < nphase; ph++) {
    const bool mine = (nphase == 1) || (wm == ph);
    if (mine) {
#pragma unroll
      for (int mb = 0; mb < 8; mb++)
#pragma unroll
        for (int nb = 0; nb < 4; nb++)
#pragma unroll
          for (int e = 0; e < 2; e++) st[((mb * 4 + nb) * 2 + e) * sthr] = acc[mb][nb][e];
    }
    consumer_bar();   // staging (and, first time round, the input tiles) visible
    if (mine) {
#pragma unroll 1
      for (int e = 0; e < 64; e++) {
        const int il = i0 + (e >> 3) * 8, jl = j0 + ((e >> 1) & 3) * 8 + (e & 1);
        const long gi = (long)r * TILE + il, gj = (long)c * TILE + jl;
        const double kinv = st[e * sthr];
        if (kout) kout[il + (long)jl * p.ldc] = kinv;
        double dot = 0.0;
        for (int q = 0; q < D; q++) dot = fma(sXr[q * TILE + il], sXc[q * TILE + jl], dot);
        double r2 = sSr[il] + sSc[jl] - 2.0 * dot;
        if (gi == gj) r2 = 0.0;
        r2 = fmax(r2, 0.0);
        const double rr = sqrt(r2) * inv_ls;
        double k, dk;
        k_dk_of_r_unit(kind, rr, k, dk);
        double aa = 0.0;
        if (alpha_here)   // multi-GPU: K^-1 is summed over the ranks' k-ranges, the alpha alpha^T term counts once
          for (int q = 0; q < P; q++) aa = fma(sAr[q * TILE + il], sAc[q * TILE + jl], aa);
        double dl = 0.5 * (aa - (double)P * kinv);
        if (gi >= p.N || gj >= p.N) dl = 0.0;
        gvar = fma(w * k, dl, gvar);
        if (gi == gj) {
          gnoise += dl;
          if (p.dnoise_out && gi < p.N) p.dnoise_out[gi] = dl;
        }
        const double G = variance * dk * dl;
        if (ard) {
          st[e * sthr] = (rr != 0.0) ? w * G / rr : 0.0;   // stationary.py:205,225-232: 1/r with 1/0 := 0
        } else {
          giso = fma(w * G, rr, giso);
        }
      }
      if (ard) {
        for (int q = 0; q < D; q++) {
          const double* xr = sXr + q * TILE;
          const double* xc = sXc + q * TILE;
          double s = 0.0;
#pragma unroll 4
          for (int e = 0; e < 64; e++) {
            const int il = i0 + (e >> 3) * 8, jl = j0 + ((e >> 1) & 3) * 8 + (e & 1);
            const double df = xr[il] - xc[jl];
            s = fma(st[e * sthr], df * df, s);
          }
          s = warp_sum(s);
          if (lane == 0) red[1 + q] = s;
        }
      }
    }
    if (nphase > 1) consumer_bar();   // the other half may now overwrite the staging area
  }
  gvar = warp_sum(gvar);
  gnoise = warp_sum(gnoise);
  if (lane == 0) { red[0] = gvar; red[nred - 1] = gnoise; }
  if (!ard) {
    giso = warp_sum(giso);
    if (lane == 0) red[1] = giso;
  }
  consumer_bar();
  if (tid < nred) {
    double s = 0.0;
#pragma unroll
    for (int wdx = 0; wdx < CONSUMER_WARPS; wdx++) s += sRed[wdx * nred + tid];
    p.partials[((long)r * p.nt + c) * nred + tid] = s;
  }
}

// one __global__ entry per mode so that profiles name them apart
__global__ void __launch_bounds__(GEMM_THREADS, 1) gemm_update_kernel(const GemmParams p) { gemm_nt_body<GEMM_UPDATE>(p); }
__global__ void __launch_bounds__(GEMM_THREADS, 1) gemm_panel_kernel(const GemmParams p) { gemm_nt_body<GEMM_PANEL>(p); }
__global__ void __launch_bounds__(GEMM_THREADS, 1) gemm_lauum_kernel(const GemmParams p) { gemm_nt_body<GEMM_LAUUM>(p); }

int gemm_init() {
  GPX_CUDA(cudaFuncSetAttribute(gemm_update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_PIPE));
  GPX_CUDA(cudaFuncSetAttribute(gemm_panel_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_PIPE));
  GPX_CUDA(cudaFuncSetAttribute(gemm_lauum_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_MAX));
  return 0;
}

int launch_gemm(const GemmParams& p, dim3 grid, cudaStream_t st) {
  if (p.mode == GEMM_UPDATE) {
    // (slots, columns) domain: rows [0, rlow) U [c, nt) for columns [c0, c0 + ncols)
    const int ncols = p.ncols > 0 ? p.ncols : p.nt - p.c0, nslots = p.rlow + (p.nt - p.c0);
    if (ncols <= 0) return 0;
    grid = dim3((unsigned)(((nslots + SB - 1) / SB) * ((ncols + SB - 1) / SB) * SB * SB), 1, 1);
  } else if (p.mode == GEMM_PANEL && p.plain) {
    grid = dim3((unsigned)(((p.nt + SB - 1) / SB) * ((p.ncols + SB - 1) / SB) * SB * SB), 1, 1);
  } else if (p.mode == GEMM_LAUUM) {
    const int nsr = (p.nt + SB - 1) / SB;
    grid = dim3((unsigned)(nsr * (nsr + 1) / 2 * SB * SB), 1, 1);
  }
  if (grid.x == 0 || grid.y == 0) return 0;
  if (p.mode == GEMM_UPDATE) gemm_update_kernel<<<grid, GEMM_THREADS, SMEM_PIPE, st>>>(p);
  else if (p.mode == GEMM_PANEL) gemm_panel_kernel<<<grid, GEMM_THREADS, SMEM_PIPE, st>>>(p);
  else {
    const int smem = BAR_BYTES + std::max(PIPE_BYTES, epi_bytes(p.kp.D, p.P));
    if (smem > SMEM_MAX) { set_error("LAUUM epilogue does not fit in shared memory"); return -2; }
    gemm_lauum_kernel<<<grid, GEMM_THREADS, smem, st>>>(p);
  }
  GPX_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace gpx
