// gpx_fine.cu — fine-grained fp64 DMMA kernels of the serial chain (see gpx_fine.cuh) and the inner sweep of a diagonal block.
//
//   gemm_fine_kernel<FINE_UPDATE / FINE_PANEL> : 64 x 32 output tile per CTA, 8 warps (4 x 2, 16 x 16 each, DMMA.16x8x4); 32-deep
//       k-chunks of both operands in a 4-stage cp.async ring (16-byte LDGSTS by every thread); smem pitches 68 / 36 doubles
//       (== 4 mod 16: conflict-free fragment loads); two CTAs per SM. A 128-deep product is 4 chunks, i.e. the whole operand
//       strip is in flight at once.
//   fine_panel_inplace_kernel : the in-place inner panel  S(r, d) <- S(r, d) L_dd^-T  in 16-row strips (a CTA owns a full row
//       strip, reads it completely into shared memory before it writes), 8 warps x 16 output columns, triangular k-range.
// Replaces (for the diagonal-block chain only) the 128 x 128-tile launches of gemm_panel_kernel / gemm_update_kernel, i.e. the
// same share of lapack.dpotrf / dtrtri (GPy/util/linalg.py:58,227) as before.
#include <algorithm>
#include <cstdlib>
#include <cstring>

#include "gpx_ctx.cuh"
#include "gpx_fine.cuh"
#include "gpx_kernels.cuh"

namespace gpx {

constexpr int FTM = 64;       // CTA output tile: 64 rows x 32 columns
constexpr int FTN = 32;
constexpr int FKC = 32;       // k-depth of one stage
constexpr int FPA = 68;       // smem pitch (doubles) of a k-column of the A strip (64 values; == 4 mod 16)
constexpr int FPB = 36;       // ... of the B strip (32 values; == 4 mod 16)
constexpr int FSTAGES = 4;
constexpr int F_CONS = 8;     // warps: 4 (m) x 2 (n), 16 x 16 each; two CTAs fit an SM
constexpr int F_THREADS = F_CONS * 32;
constexpr int F_STAGE_A = FKC * FPA;
constexpr int F_STAGE_B = FKC * FPB;
constexpr int F_SMEM = FSTAGES * (F_STAGE_A + F_STAGE_B) * 8;   // 106496 B
constexpr int F_SUB = (TILE / FTM) * (TILE / FTN);                             // 8 CTA tiles per 128 x 128 tile

template <int MODE>
__device__ __forceinline__ bool fine_decode(const FineParams& p, int& r, int& c, int& sm, int& sn) {
  const int t = blockIdx.x / F_SUB, sub = blockIdx.x % F_SUB;
  sm = sub & 1; sn = sub >> 1;
  if (MODE == FINE_UPDATE) {
    const int col = t % p.ncols, slot = t / p.ncols;
    c = p.c0 + col;
    r = slot < p.rlow ? slot : c + (slot - p.rlow);
    if (r >= p.nt) return false;
    return !(r == c && sm == 0 && sn >= 2);      // diagonal tile: rows 0..63 x columns 64..127 lie above the diagonal
  } else if (MODE == FINE_LAUUM) {
    r = (int)((sqrtf(8.f * (float)t + 1.f) - 1.f) * 0.5f);
    while (r * (r + 1) / 2 > t) --r;
    while ((r + 1) * (r + 2) / 2 <= t) ++r;
    c = t - r * (r + 1) / 2;
    return r < p.nt;
  } else {
    const int cc = t % p.nc;
    c = p.tri ? p.nc - 1 - cc : cc;      // longest k-range first
    r = p.r0 + t / p.nc;
    return true;
  }
}

__device__ __forceinline__ void cp_async16(void* dst_smem, const void* src_gmem) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst_smem)), "l"(src_gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// Operand staging: every thread copies six 16-byte pieces per stage with cp.async (LDGSTS). The first version used one bulk
// copy (cp.async.bulk) per k-column from a producer warp: 64 copies of 256..512 B per stage cost ~30 ns EACH on the issuing
// warp -- 2 us per 32-deep chunk, i.e. the kernel ran at the bulk-copy issue rate (10 us for a 128-deep product, 32 us for
// K = 512, whatever the tile shape); bulk copies pay off from ~1 KB up (gemm_nt_body), not for these strips.
template <int MODE>
__global__ void __launch_bounds__(F_THREADS, 2) gemm_fine_kernel(const FineParams p) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  double* sA = reinterpret_cast<double*>(smem_raw);
  double* sB = sA + FSTAGES * F_STAGE_A;

  // the base-block kernel that follows in the diagonal-block chain is launched as a programmatic dependent: let it become
  // resident now (it warms its instruction cache and then waits for this grid to complete)
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  int r, c, sm, sn;
  if (!fine_decode<MODE>(p, r, c, sm, sn)) return;
  int kmax = p.K;
  if (MODE == FINE_PANEL && p.tri) kmax = min(p.K, c * TILE + FTN * (sn + 1));
  const int it0 = MODE == FINE_LAUUM ? r * (TILE / FKC) : 0;     // first k-chunk
  const int nchunk = kmax / FKC - it0;
  const double* Aptr = p.A + (long)r * TILE + sm * FTM;
  const double* Bptr = p.B + (long)c * TILE + sn * FTN;
  const long lda = p.lda, ldb = p.ldb;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  // this grid may itself have been launched as a programmatic dependent (of the in-place inner panel): everything above ran
  // beside that kernel, the operands are read only after it has completed and flushed
  asm volatile("griddepcontrol.wait;" ::: "memory");

  auto load_stage = [&](int it) {
    if (it < nchunk) {
      const int s = it % FSTAGES;
      const long k0 = (long)(it0 + it) * FKC;
      double* dA = sA + s * F_STAGE_A;
      double* dB = sB + s * F_STAGE_B;
#pragma unroll
      for (int i = 0; i < (FKC * FTM / 2) / F_THREADS; i++) {      // A: 32 k-columns x 32 pieces of 2 doubles
        const int q = tid + i * F_THREADS, kc = q >> 5, part = q & 31;
        cp_async16(dA + kc * FPA + part * 2, Aptr + (k0 + kc) * lda + part * 2);
      }
#pragma unroll
      for (int i = 0; i < (FKC * FTN / 2) / F_THREADS; i++) {      // B: 32 k-columns x 16 pieces
        const int q = tid + i * F_THREADS, kc = q >> 4, part = q & 15;
        cp_async16(dB + kc * FPB + part * 2, Bptr + (k0 + kc) * ldb + part * 2);
      }
    }
    cp_async_commit();
  };
#pragma unroll
  for (int s = 0; s < FSTAGES - 1; s++) load_stage(s);

  // warp (wm, wn) owns rows [16 wm, +16) x columns [16 wn, +16) of the CTA tile
  const int wm = warp & 3, wn = warp >> 2;
  const int g = lane >> 2, tg = lane & 3;
  double* Ct = p.C + (long)r * TILE + sm * FTM + ((long)c * TILE + sn * FTN) * p.ldc;
  // FOUR independent accumulator sets (k4 steps i, i+4, ... go to set i & 3, summed at the end): with one set every DMMA of a
  // warp waits for its predecessor on the same 8 x 8 accumulator (~64 clk), and 2 x 2 accumulators per warp kept the tensor
  // pipe at a third of its rate (26 us for the 64 x 32 x 512 tiles of a 512^2 diagonal-block update)
  constexpr int NS = 4;
  double acc[NS][2][2][2];
#pragma unroll
  for (int q = 0; q < NS; q++)
#pragma unroll
    for (int mb = 0; mb < 2; mb++)
#pragma unroll
      for (int nb = 0; nb < 2; nb++) { acc[q][mb][nb][0] = 0.0; acc[q][mb][nb][1] = 0.0; }
  if (MODE == FINE_UPDATE) {   // C - A B^T = C + (-A) B^T: set 0 starts from the old tile, store-only epilogue
#pragma unroll
    for (int mb = 0; mb < 2; mb++)
#pragma unroll
      for (int nb = 0; nb < 2; nb++)
#pragma unroll
        for (int e = 0; e < 2; e++) acc[0][mb][nb][e] = Ct[wm * 16 + mb * 8 + g + (long)(wn * 16 + nb * 8 + 2 * tg + e) * p.ldc];
  }
  for (int it = 0; it < nchunk; ++it) {
    cp_async_wait<FSTAGES - 2>();      // this thread's pieces of stage `it` have landed ...
    __syncthreads();                   // ... and everybody's; everybody is also done with stage it-1 (refilled next)
    load_stage(it + FSTAGES - 1);
    const int s = it % FSTAGES;
    const double* a = sA + s * F_STAGE_A + wm * 16 + g;
    const double* b = sB + s * F_STAGE_B + wn * 16 + g;
#pragma unroll
    for (int k4 = 0; k4 < FKC / 4; k4++) {
      const int k = k4 * 4 + tg;
      double af[2], bf[2];
#pragma unroll
      for (int mb = 0; mb < 2; mb++) af[mb] = (MODE == FINE_UPDATE) ? -a[k * FPA + mb * 8] : a[k * FPA + mb * 8];
#pragma unroll
      for (int nb = 0; nb < 2; nb++) bf[nb] = b[k * FPB + nb * 8];
#pragma unroll
      for (int mb = 0; mb < 2; mb += 2)
#pragma unroll
        for (int nb = 0; nb < 2; nb++) {
          double (&c)[2][2][2] = acc[k4 & (NS - 1)];
          dmma1684(c[mb][nb][0], c[mb][nb][1], c[mb + 1][nb][0], c[mb + 1][nb][1], af[mb], af[mb + 1], bf[nb]);
        }
    }
  }
#pragma unroll
  for (int mb = 0; mb < 2; mb++)
#pragma unroll
    for (int nb = 0; nb < 2; nb++)
#pragma unroll
      for (int e = 0; e < 2; e++)
        Ct[wm * 16 + mb * 8 + g + (long)(wn * 16 + nb * 8 + 2 * tg + e) * p.ldc] =
            (acc[0][mb][nb][e] + acc[1][mb][nb][e]) + (acc[2][mb][nb][e] + acc[3][mb][nb][e]);
}

// ---- in-place inner panel ------------------------------------------------------------------------------------------------
constexpr int IP_ROWS = 16;       // rows per CTA strip
constexpr int IP_PA = 20;         // smem pitch of a 16-value k-column of the strip (== 4 mod 16)
constexpr int IP_THREADS = 256;   // 8 warps x 16 output columns
constexpr int IP_SMEM = 128 + (TILE * IP_PA + TILE * PITCH) * 8;   // 128 + 20480 + 135168

__global__ void __launch_bounds__(IP_THREADS, 1)
fine_panel_inplace_kernel(double* __restrict__ Sblk, long ld, const double* __restrict__ Dinv, int d) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem_raw);
  double* sA = reinterpret_cast<double*>(smem_raw + 128);   // strip: (m, k) at k*IP_PA + m
  double* sB = sA + TILE * IP_PA;                            // Dinv:  (n, k) at k*PITCH + n   (only n >= 16*(k/16) is loaded)
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");   // the inner update behind it may become resident (it waits)
  const int slot = blockIdx.x / (TILE / IP_ROWS), part = blockIdx.x % (TILE / IP_ROWS);
  const int r = slot < d ? slot : slot + 1;
  double* strip = Sblk + (long)r * TILE + part * IP_ROWS + (long)d * TILE * ld;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) { mbar_init(bar, 1); fence_mbar_init(); }
  __syncthreads();
  if (tid == 0) {
    uint32_t bytes = TILE * IP_ROWS * 8;
    for (int j = 0; j < TILE / 16; j++) bytes += 16 * (TILE - 16 * j) * 8;
    mbar_arrive_expect_tx(bar, bytes);
  }
  __syncthreads();
  if (tid < TILE) {
    bulk_g2s(sA + tid * IP_PA, strip + (long)tid * ld, IP_ROWS * 8, bar);
  } else {
    const int k = tid - TILE, n0 = k & ~15;
    bulk_g2s(sB + k * PITCH + n0, Dinv + (long)k * TILE + n0, (TILE - n0) * 8, bar);
  }
  mbar_wait(bar, 0);
  // warp w: output columns [16w, 16w+16), k < 16(w+1)  (L_dd^-1 is lower triangular: B(n, k) = 0 for k > n)
  const int g = lane >> 2, tg = lane & 3;
  double acc[2][2][2];
#pragma unroll
  for (int mi = 0; mi < 2; mi++)
#pragma unroll
    for (int ni = 0; ni < 2; ni++) { acc[mi][ni][0] = 0.0; acc[mi][ni][1] = 0.0; }
  const int nk4 = 4 * (warp + 1);
  const double* b = sB + 16 * warp + g;
  for (int k4 = 0; k4 < nk4; k4++) {
    const int k = k4 * 4 + tg;
    double af[2], bf[2];
#pragma unroll
    for (int mi = 0; mi < 2; mi++) af[mi] = sA[k * IP_PA + mi * 8 + g];
#pragma unroll
    for (int ni = 0; ni < 2; ni++) bf[ni] = b[k * PITCH + ni * 8];
#pragma unroll
    for (int mi = 0; mi < 2; mi += 2)
#pragma unroll
      for (int ni = 0; ni < 2; ni++) dmma1684(acc[mi][ni][0], acc[mi][ni][1], acc[mi + 1][ni][0], acc[mi + 1][ni][1],
                                                          af[mi], af[mi + 1], bf[ni]);
  }
  // every byte of the strip is in shared memory (the mbarrier completed for the whole CTA): overwrite in place
#pragma unroll
  for (int mi = 0; mi < 2; mi++)
#pragma unroll
    for (int ni = 0; ni < 2; ni++)
#pragma unroll
      for (int e = 0; e < 2; e++) strip[mi * 8 + g + (long)(16 * warp + ni * 8 + 2 * tg + e) * ld] = acc[mi][ni][e];
}

int fine_init() {
  GPX_CUDA(cudaFuncSetAttribute(gemm_fine_kernel<FINE_UPDATE>, cudaFuncAttributeMaxDynamicSharedMemorySize, F_SMEM));
  GPX_CUDA(cudaFuncSetAttribute(gemm_fine_kernel<FINE_PANEL>, cudaFuncAttributeMaxDynamicSharedMemorySize, F_SMEM));
  GPX_CUDA(cudaFuncSetAttribute(gemm_fine_kernel<FINE_LAUUM>, cudaFuncAttributeMaxDynamicSharedMemorySize, F_SMEM));
  GPX_CUDA(cudaFuncSetAttribute(fine_panel_inplace_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, IP_SMEM));
  return 0;
}

// launched with the programmatic-stream-serialization attribute (option "base_pdl"): behind a kernel that issues
// griddepcontrol.launch_dependents (the in-place inner panel, another fine GEMM) the CTAs become resident early and block in
// griddepcontrol.wait; behind any other kernel or an event wait this is an ordinary launch
template <int MODE>
static int launch_fine_pdl(const FineParams& p, unsigned grid, cudaStream_t st) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(grid); cfg.blockDim = dim3(F_THREADS); cfg.dynamicSmemBytes = F_SMEM; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = (p.pdl && get_base_pdl()) ? 1 : 0;
  GPX_CUDA(cudaLaunchKernelEx(&cfg, gemm_fine_kernel<MODE>, p));
  return 0;
}

int launch_fine(const FineParams& p0, cudaStream_t st) {
  FineParams p = p0;
  if (p.K <= 0 || p.K % TILE != 0) { set_error("fine GEMM: k-depth must be a positive multiple of 128"); return -2; }
  unsigned grid;
  if (p.mode == FINE_UPDATE) {
    if (p.ncols <= 0) p.ncols = p.nt - p.c0;
    if (p.ncols <= 0) return 0;
    const int nslots = p.rlow + (p.nt - p.c0);
    grid = (unsigned)(nslots * p.ncols * F_SUB);
    if (launch_fine_pdl<FINE_UPDATE>(p, grid, st)) return -1;
  } else if (p.mode == FINE_LAUUM) {
    if (p.nt <= 0) return 0;
    grid = (unsigned)(p.nt * (p.nt + 1) / 2 * F_SUB);
    if (launch_fine_pdl<FINE_LAUUM>(p, grid, st)) return -1;
  } else {
    if (p.nr <= 0 || p.nc <= 0) return 0;
    grid = (unsigned)(p.nr * p.nc * F_SUB);
    if (launch_fine_pdl<FINE_PANEL>(p, grid, st)) return -1;
  }
  GPX_CUDA(cudaGetLastError());
  return 0;
}

int launch_fine_panel_inplace(double* Sblk, long ld, const double* Dinv, int nbt, int d, cudaStream_t st) {
  if (nbt <= 1) return 0;
  fine_panel_inplace_kernel<<<(nbt - 1) * (TILE / IP_ROWS), IP_THREADS, IP_SMEM, st>>>(Sblk, ld, Dinv, d);
  GPX_CUDA(cudaGetLastError());
  return 0;
}

#define GPX_CHECK_F(x) do { int rc__ = (x); if (rc__) return rc__; } while (0)

int diag_block_sweep(gpx_ctx* c, double* Sblk, long ld, int nbt, int g0, cudaStream_t st) {
  for (int d = 0; d < nbt; d++) {
    const int g = g0 + d;
    double* tile = Sblk + (long)d * TILE + (long)d * TILE * ld;
    GPX_CHECK_F(launch_base(tile, ld, c->Ldiag + (long)g * TILE * TILE, c->Dinv + (long)g * TILE * TILE, c->logdet_part + g,
                            c->info, g * TILE, st));
    c->eval_launches++;
    if (nbt == 1) break;
    if (c->fine) {
      GPX_CHECK_F(launch_fine_panel_inplace(Sblk, ld, c->Dinv + (long)g * TILE * TILE, nbt, d, st));
      c->eval_launches++;
      if (d + 1 < nbt) {
        FineParams pu{};
        pu.mode = FINE_UPDATE;
        pu.A = Sblk + (long)d * TILE * ld; pu.lda = ld;
        pu.B = pu.A; pu.ldb = ld;
        pu.C = Sblk; pu.ldc = ld;
        pu.K = TILE; pu.nt = nbt; pu.c0 = d + 1; pu.ncols = nbt - d - 1; pu.rlow = d + 1;
        pu.pdl = 1;
        GPX_CHECK_F(launch_fine(pu, st));
        c->eval_launches++;
      }
    } else {   // option "fine" = 0: the 128 x 128-tile kernels (round-1 form)
      GemmParams pp = gemm_defaults();
      pp.mode = GEMM_PANEL;
      pp.A = Sblk + (long)d * TILE * ld; pp.lda = ld;
      pp.B = c->Dinv + (long)g * TILE * TILE; pp.ldb = TILE;
      pp.C = Sblk + (long)d * TILE * ld; pp.ldc = ld;      // in place: one k-tile deep, tile-local dependence only
      pp.K = TILE; pp.nt = nbt; pp.skip0 = d; pp.skip1 = d + 1; pp.tri = 0;
      GPX_CHECK_F(launch_gemm(pp, dim3(1, nbt - 1), st));
      c->eval_launches++;
      if (d + 1 < nbt) {
        GemmParams pu = gemm_defaults();
        pu.mode = GEMM_UPDATE;
        pu.A = Sblk + (long)d * TILE * ld; pu.lda = ld;
        pu.B = pu.A; pu.ldb = ld;
        pu.C = Sblk; pu.ldc = ld;
        pu.K = TILE; pu.nt = nbt; pu.c0 = d + 1; pu.rlow = d + 1;
        GPX_CHECK_F(launch_gemm(pu, dim3(1, 1), st));
        c->eval_launches++;
      }
    }
  }
  return 0;
}

}  // namespace gpx
