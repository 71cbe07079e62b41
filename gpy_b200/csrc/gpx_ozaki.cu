// gpx_ozaki.cu — the trailing update and K^-1 = U U^T of the factor-and-invert sweep on the Hopper INT8 tensor cores.
//
// wgmma has no f64 kind, so fp64-grade products are formed by an Ozaki split on s8 x s8 -> s32 (exact integer accumulation):
//   every row of a panel P (rows x K) is scaled by a power of two to (-1/2, 1/2) and cut into 8 signed digits of 7 bits, rounded
//   to nearest (|digit| <= 64; int8 planes),
//   P_r P_c^T = sum_{s+t <= 7} 2^(e_r + e_c - 7 (s+t+2)) D_s(r) D_t(c)^T; the 36 digit-pair products of a 32-deep k-chunk are
//   36 wgmma.m64n64k32 accumulated per exponent group g = s + t in its own s32 register accumulator,
//   |digit product sum| <= 64^2 * K * 8 < 2^31 for K <= 65536; the epilogue converts the groups to fp64, sums them smallest
//   first, rescales by the row/column exponents and applies the result to the fp64 target tile.
// Replaces the same reference work as the DMMA GEMM of gpx_gemm.cu: LAPACK dpotrf / dtrtri / dpotri behind
// GPy/util/linalg.py:58,142,209-212 (see DESIGN.md §5 for the digit budget against the 1e-8 / 1e-6 tolerances).
//
// Kernel anatomy (one CTA per SM over a run of consecutive tiles of the list): warpgroup 2 = TMA producer (one warp,
// cp.async.bulk.tensor over the pre-tiled digit planes, mbarrier ring of 32-deep k-chunks), warpgroups 0 and 1 = consumers.
// Eight exponent groups of a 64 x 64 accumulator are 256 s32 registers per thread, more than a thread has, so the two
// consumer warpgroups compute the SAME 64 x 64 sub-tile and split the groups between them (four each, 128 registers):
// warpgroup 0 takes the groups g with g % 4 in {0, 3}, warpgroup 1 those with g % 4 in {1, 2} (18 of the 36 digit pairs each).
// A 128 x 128 output tile of the list is walked as 4 such sub-tiles.
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>

#include "gpx_common.cuh"
#include "gpx_ozaki.cuh"

#include <algorithm>
#include <vector>

namespace gpx {

constexpr int OZ_SUB = 64;                                        // sub-tile edge (wgmma M = N = 64)
constexpr int OZ_NSUB = (OZ_TM / OZ_SUB) * (OZ_TN / OZ_SUB);      // sub-tiles per output tile (bit 0: row half, bit 1: column half)
constexpr int OZ_STAGES = 5;
constexpr int OZ_PLANE = OZ_SUB * OZ_KC;                          // 2048: one digit plane of a 64-row sub-tile, one k-chunk
constexpr int OZ_STAGE_BYTES = 2 * OZ_S * OZ_PLANE;               // 32768: up to 8 A planes + 8 B planes
constexpr int OZ_XCH_BYTES = OZ_SUB * OZ_SUB * 8;                 // 32768: fp64 partial sums handed between the consumers
constexpr int OZ_THREADS = 384;                                   // three warpgroups (setmaxnreg works per warpgroup)
constexpr int OZ_SMEM = OZ_STAGES * OZ_STAGE_BYTES + OZ_XCH_BYTES + 1024 + 256;   // ring + exchange + alignment + barriers

// ---------------------------------------------------------------------------------------------------------------
// PTX helpers (wgmma / TMA tensor copies); mbarrier helpers come from gpx_common.cuh
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* map, int c0, int c1, int c2, int c3, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];" ::"r"(
          smem_u32(dst)),
      "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(smem_u32(bar))
      : "memory");
}
// mbarrier wait with back-off, for the producer waiting for a free stage: its polling must not take issue slots from the
// consumers on the same SM sub-partitions
__device__ __forceinline__ void mbar_wait_backoff(uint64_t* bar, uint32_t parity, unsigned ns) {
  for (;;) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    if (ok) return;
    __nanosleep(ns);
  }
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}
// shared-memory matrix descriptor: no swizzle, K-major, core matrices 8 rows x 16 B; LBO = 128 B between the two core matrices
// along K, SBO = 256 B between 8-row groups (the image of gpx_ozaki.cuh)
__device__ __forceinline__ uint64_t oz_desc(uint32_t saddr) {
  return (uint64_t)((saddr & 0x3FFFF) >> 4) | ((uint64_t)(128 >> 4) << 16) | ((uint64_t)(256 >> 4) << 32);
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// D(64 x 64, s32) += A(64 x 32, s8) B(64 x 32, s8)^T, both operands K-major in shared memory
__device__ __forceinline__ void wgmma_i8(uint32_t (&d)[32], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p;\n\t}"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]),
        "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]),
        "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]),
        "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
      : "l"(da), "l"(db), "r"(1)
      : "memory");
}
__device__ __forceinline__ void named_bar(int id, int nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }

// ---------------------------------------------------------------------------------------------------------------
// 1. digit split: row exponents + 8 signed 7-bit digit planes of a panel, written in the tiled image of gpx_ozaki.cuh
// ---------------------------------------------------------------------------------------------------------------
constexpr int SPLIT_ROWS = 64;
constexpr int SPLIT_KS = 8;      // row maxima: k-slices per row (partial maxima, reduced by the digit kernel)
constexpr int SPLIT_KCB = 4;     // digit kernel: k-chunks (of 32) per CTA
// The split is two kernels so that both have thousands of CTAs: (1) partial row maxima over k-slices, (2) digits of a
// 64-row x 128-column piece per CTA. As ONE kernel (a CTA walked the whole K range of its 64 rows: 256 CTAs at N = 16384, each
// thread 2 x 256 dependent strided loads) it ran at 1.3 TB/s of HBM traffic, 211 us per 16384 x 1024 panel.
__global__ void __launch_bounds__(256) oz_rowmax_kernel(const double* __restrict__ P, long ld, long rows, int nkc_used,
                                                       double* __restrict__ amax_part) {
  __shared__ double smax[2][128];
  const int tid = threadIdx.x, rl = tid & 127, half = tid >> 7;
  const long row = (long)blockIdx.x * 128 + rl;
  const long K = (long)nkc_used * OZ_KC;
  const long kper = (K + SPLIT_KS - 1) / SPLIT_KS;
  const long k0 = (long)blockIdx.y * kper, k1 = min(K, k0 + kper);
  const double* prow = P + row;
  double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;
  long k = k0 + half;
  for (; k + 6 < k1; k += 8) {
    a0 = fmax(a0, fabs(prow[k * ld]));
    a1 = fmax(a1, fabs(prow[(k + 2) * ld]));
    a2 = fmax(a2, fabs(prow[(k + 4) * ld]));
    a3 = fmax(a3, fabs(prow[(k + 6) * ld]));
  }
  for (; k < k1; k += 2) a0 = fmax(a0, fabs(prow[k * ld]));
  smax[half][rl] = fmax(fmax(a0, a1), fmax(a2, a3));
  __syncthreads();
  if (half == 0) amax_part[(long)blockIdx.y * rows + row] = fmax(smax[0][rl], smax[1][rl]);
}

// nkc = k-chunks of the plane LAYOUT (strides), nkc_used <= nkc = k-chunks actually present in this panel (a short last block)
__global__ void __launch_bounds__(256) oz_split_kernel(const double* __restrict__ P, long ld, long rows, int nkc, int nkc_used,
                                                      const double* __restrict__ amax_part, int8_t* __restrict__ planes,
                                                      double* __restrict__ scale) {
  __shared__ double sinv[SPLIT_ROWS];
  const int tid = threadIdx.x, rl = tid & (SPLIT_ROWS - 1), part = tid >> 6;
  const long row = (long)blockIdx.x * SPLIT_ROWS + rl;
  const double* prow = P + row;
  if (part == 0) {
    double amax = 0.0;
#pragma unroll
    for (int q = 0; q < SPLIT_KS; q++) amax = fmax(amax, amax_part[(long)q * rows + row]);
    double inv = 0.0, sc = 0.0;
    if (amax >= 1e-290 && amax <= 1e290) {   // rows of zeros (padding) and rows with infinities get all-zero digits
      int e = 0;
      frexp(amax, &e);                        // amax = m 2^e, m in [0.5, 1): |x| 2^-(e+1) < 1/2 for the whole row
      inv = ldexp(1.0, -(e + 1));
      sc = ldexp(1.0, e + 1 - 7);             // value = 2^(e+1) sum_s d_s 2^(-7 (s+1)); the 2^-7 of both operands folded in here
    }
    sinv[rl] = inv;
    if (blockIdx.y == 0) scale[row] = sc;
  }
  __syncthreads();
  const double inv = sinv[rl];
  const long ngrp = rows / 8;
  const int u_beg = blockIdx.y * SPLIT_KCB * 2, u_end = min(nkc_used * 2, u_beg + SPLIT_KCB * 2);
  for (int u = u_beg + part; u < u_end; u += 4) {   // unit = 16 consecutive k of one row = one 16-byte line of a core matrix
    const int kc = u >> 1, half = u & 1;
    double xs[16];
#pragma unroll
    for (int kk = 0; kk < 16; kk++) xs[kk] = prow[((long)kc * OZ_KC + half * 16 + kk) * ld];   // 16 loads in flight
    uint32_t w[OZ_S][4];
#pragma unroll
    for (int s = 0; s < OZ_S; s++) { w[s][0] = 0; w[s][1] = 0; w[s][2] = 0; w[s][3] = 0; }
#pragma unroll
    for (int kk = 0; kk < 16; kk++) {
      double x = xs[kk] * inv;                                 // exact (power of two), |x| < 1/2
#pragma unroll
      for (int s = 0; s < OZ_S; s++) {
        // round-to-nearest digits WITHOUT the conversion unit (F2I / I2F on fp64 run at a few lanes per SM):
        // x + 1.5 * 2^52 rounds x to an integer whose two's complement sits in the low word
        x *= 128.0;                                            // exact; |x| < 64 (first digit), <= 64 afterwards
        const double t = x + 6755399441055744.0;               // 1.5 * 2^52
        const int d = __double2loint(t);                       // rint(x), |d| <= 64
        x -= (t - 6755399441055744.0);                         // exact remainder, |x| <= 1/2
        w[s][kk >> 2] |= ((uint32_t)d & 0xffu) << (8 * (kk & 3));
      }
    }
    int8_t* base = planes + ((long)kc * ngrp + row / 8) * 256 + half * 128 + (row % 8) * 16;
#pragma unroll
    for (int s = 0; s < OZ_S; s++)
      *reinterpret_cast<uint4*>(base + (long)s * nkc * ngrp * 256) = make_uint4(w[s][0], w[s][1], w[s][2], w[s][3]);
  }
}

int launch_oz_split(const double* P, long ld, long K, OzPlanes& pl, cudaStream_t st) {
  if (K % OZ_KC || K / OZ_KC > pl.nkc) { set_error("launch_oz_split: bad panel width"); return -2; }
  const int nkc_used = (int)(K / OZ_KC);
  oz_rowmax_kernel<<<dim3((unsigned)(pl.rows / 128), SPLIT_KS), 256, 0, st>>>(P, ld, pl.rows, nkc_used, pl.amax_part);
  oz_split_kernel<<<dim3((unsigned)(pl.rows / SPLIT_ROWS), (unsigned)((nkc_used + SPLIT_KCB - 1) / SPLIT_KCB)), 256, 0, st>>>(
      P, ld, pl.rows, pl.nkc, nkc_used, pl.amax_part, pl.planes, pl.scale);
  GPX_CUDA(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// 2. the GEMM
// ---------------------------------------------------------------------------------------------------------------
// exponent group of accumulator slot j of consumer warpgroup w (slots in ascending group order)
__host__ __device__ constexpr int oz_group(int w, int j) {
  return w == 0 ? (j == 0 ? 0 : j == 1 ? 3 : j == 2 ? 4 : 7) : (j == 0 ? 1 : j == 1 ? 2 : j == 2 ? 5 : 6);
}
// k-chunks of a tile: the whole panel width, except OZ_PANEL tiles (triangular B: columns of tile c' see k < (c' + 1) * 128)
__device__ __forceinline__ int oz_tile_nkc(uint32_t t, int nkc) {
  return ((t >> 25) & 3) == OZ_PANEL ? min(nkc, (int)(((t >> 12) & 0x1fff) + 1) * (OZ_TN / OZ_KC)) : nkc;
}
// one 32-deep k-chunk of warpgroup W: the digit pairs (s, g - s) of its groups g < ND. a_base = shared address of digit
// plane 0 of the A sub-tile in this stage; the B planes follow the 8 A planes.
template <int W, int ND>
__device__ __forceinline__ void oz_issue(uint32_t (&acc)[4][32], uint32_t a_base) {
  const uint64_t da0 = oz_desc(a_base), db0 = oz_desc(a_base + OZ_S * OZ_PLANE);
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const int g = oz_group(W, j);
    if (g < ND) {
#pragma unroll
      for (int s = 0; s <= g; s++) wgmma_i8(acc[j], da0 + (uint64_t)((s * OZ_PLANE) >> 4), db0 + (uint64_t)(((g - s) * OZ_PLANE) >> 4));
    }
  }
}
// the k-loop of one sub-tile, then its exponent groups summed in fp64 into f (wgmma needs the digit count at compile time:
// a run-time branch around the instructions makes the compiler serialise them)
template <int W, int ND>
__device__ __forceinline__ void oz_subtile(double (&f)[32], uint32_t ring_s, uint64_t* full, uint64_t* empty, uint32_t& it,
                                           int nkc_t, int tid) {
  uint32_t acc[4][32];
#pragma unroll
  for (int j = 0; j < 4; j++)
#pragma unroll
    for (int e = 0; e < 32; e++) acc[j][e] = 0u;
  for (int kc = 0; kc < nkc_t; kc++, it++) {
    const int st = it % OZ_STAGES;
    mbar_wait(&full[st], (it / OZ_STAGES) & 1);
    wg_fence();
    oz_issue<W, ND>(acc, ring_s + (uint32_t)st * OZ_STAGE_BYTES);
    wg_commit();
    wg_wait<1>();   // the chunk before this one has been read: its stage may be refilled
    if (kc > 0 && tid == 0) mbar_arrive(&empty[(it - 1) % OZ_STAGES]);
  }
  wg_wait<0>();
  if (tid == 0) mbar_arrive(&empty[(it - 1) % OZ_STAGES]);
  // s32 -> fp64 without the conversion unit (I2F.F64 runs at a few lanes per SM): the bit pattern
  // {0x43300000, v ^ 0x80000000} is the double 2^52 + 2^31 + v, one exact DADD takes the offset off
#pragma unroll
  for (int e = 0; e < 32; e++) f[e] = 0.0;
#pragma unroll
  for (int j = 3; j >= 0; j--) {   // smallest magnitude first
    const int g = oz_group(W, j);
    if (g < ND) {
      const double sc = __longlong_as_double((long long)(1023 - 7 * g) << 52);   // 2^(-7 g)
#pragma unroll
      for (int e = 0; e < 32; e++)
        f[e] = fma(__hiloint2double(0x43300000, (int)(acc[j][e] ^ 0x80000000u)) - 4503601774854144.0, sc, f[e]);
    }
  }
}

template <int W>
__device__ __forceinline__ void oz_consume(const OzParams& p, const unsigned char* ring, double* xch, uint64_t* full,
                                           uint64_t* empty, int ti_beg, int ti_end) {
  const int tid = threadIdx.x & 127, warp = tid >> 5, lane = tid & 31;
  const uint32_t ring_s = smem_u32(ring);
  uint32_t it = 0;
  for (int ti = ti_beg; ti < ti_end; ti++) {
    const uint32_t t = p.tiles[ti];
    const int r = t & 0xfff, c = (t >> 12) & 0x1fff, kind = (t >> 25) & 3;
    const bool up = (t >> 27) & 1;
    const int nkc_t = oz_tile_nkc(t, p.nkc);
    for (int sub = 0; sub < OZ_NSUB; sub++) {
      double f[32];
      if (up) oz_subtile<W, OZ_S_UP>(f, ring_s, full, empty, it, nkc_t, tid);
      else oz_subtile<W, OZ_S>(f, ring_s, full, empty, it, nkc_t, tid);
      // warpgroup 0 finishes columns 0..31 of the sub-tile (accumulator elements 0..15), warpgroup 1 columns 32..63: each
      // hands the other half of its partial sums over (the two hold the same elements at the same thread index)
      constexpr int KEEP = W == 0 ? 0 : 16, GIVE = 16 - KEEP;
      named_bar(1, 256);   // the partner has read the previous sub-tile's exchange
#pragma unroll
      for (int e = 0; e < 16; e++) xch[(W * 16 + e) * 128 + tid] = f[GIVE + e];
      named_bar(1, 256);
#pragma unroll
      for (int e = 0; e < 16; e++) f[KEEP + e] += xch[((1 - W) * 16 + e) * 128 + tid];
      // element e of the accumulator: row warp * 16 + lane / 4 + 8 * ((e / 2) % 2), column (e / 4) * 8 + (lane % 4) * 2 + e % 2
      const long gi0 = (long)r * OZ_TM + (sub & 1) * OZ_SUB + warp * 16 + (lane >> 2);
      const long gj0 = (long)c * OZ_TN + (sub >> 1) * OZ_SUB + (lane & 3) * 2;
      const double si[2] = {p.scale[gi0], p.scale[gi0 + 8]};
      const double* scol = kind == OZ_PANEL ? p.scaleB : p.scale;
      double v[16];
#pragma unroll
      for (int e = 0; e < 16; e++) {
        const int ee = KEEP + e;
        v[e] = f[ee] * (si[(ee >> 1) & 1] * __ldg(scol + gj0 + (ee >> 2) * 8 + (ee & 1)));
      }
      // all loads of the target before the first store: with a run-time leading dimension the compiler must otherwise assume
      // that a store may alias the next load and serialise the global round trips
      auto apply = [&](double* C, long ld, int how) {
        double old[16];
        if (how != OZ_LAUUM_SET) {
#pragma unroll
          for (int e = 0; e < 16; e++) {
            const int ee = KEEP + e;
            old[e] = C[gi0 + 8 * ((ee >> 1) & 1) + (gj0 + (ee >> 2) * 8 + (ee & 1)) * ld];
          }
        }
#pragma unroll
        for (int e = 0; e < 16; e++) {
          const int ee = KEEP + e;
          C[gi0 + 8 * ((ee >> 1) & 1) + (gj0 + (ee >> 2) * 8 + (ee & 1)) * ld] =
              how == OZ_UPDATE ? old[e] - v[e] : (how == OZ_LAUUM_ACC ? old[e] + v[e] : v[e]);
        }
      };
      if (kind == OZ_UPDATE) apply(p.S, p.lds, OZ_UPDATE);
      else if (kind == OZ_PANEL) {
        apply(p.P, p.ldp, OZ_LAUUM_SET);
        // the panel rows also take their final place in the workspace (U block column above, L panel below the diagonal
        // block): its digit planes were taken before this launch, nothing reads the fp64 block column any more
        if (p.Pfinal) apply(p.Pfinal, p.lds, OZ_LAUUM_SET);
      } else apply(p.Kinv, p.ldk, kind);
    }
  }
}

// Warp roles: warpgroups 0 and 1 = consumers (setmaxnreg 232: 128 s32 accumulators + 32 fp64 sums per thread), warp 8 =
// TMA producer, warps 9..11 idle (the third warpgroup hands its registers over: 40 each).
__global__ void __launch_bounds__(OZ_THREADS, 1)
oz_gemm_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB, const OzParams p) {
  extern __shared__ unsigned char oz_smem_raw[];
  unsigned char* ring = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(oz_smem_raw) + 1023) & ~(uintptr_t)1023);
  double* xch = reinterpret_cast<double*>(ring + OZ_STAGES * OZ_STAGE_BYTES);
  uint64_t* full = reinterpret_cast<uint64_t*>(ring + OZ_STAGES * OZ_STAGE_BYTES + OZ_XCH_BYTES);
  uint64_t* empty = full + OZ_STAGES;
  const int wg = threadIdx.x >> 7;
  if (threadIdx.x == 0) {
#pragma unroll
    for (int s = 0; s < OZ_STAGES; s++) { mbar_init(&full[s], 1); mbar_init(&empty[s], 2); }
    fence_mbar_init();
    tma_prefetch_desc(&mapA);
    tma_prefetch_desc(&mapB);
  }
  __syncthreads();
  // a CTA owns p.tpc CONSECUTIVE tiles of the list (neighbours in the banded order share operand panels in L2) and then
  // retires: SM slots come free every few tiles, so the high-priority side stream of the sweep (diagonal block, panel of the
  // next step) gets onto the machine while this launch is still running — a fully persistent grid would shut it out
  const int ti_beg = blockIdx.x * p.tpc, ti_end = min(p.ntiles, ti_beg + p.tpc);
  if (wg == 2) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x >= 288) return;
    // ================= TMA producer: lane s < nd loads digit plane s of both operands ================================
    const int lane = threadIdx.x & 31;
    uint32_t it = 0;
    for (int ti = ti_beg; ti < ti_end; ti++) {
      const uint32_t t = p.tiles[ti];
      const int r = t & 0xfff, c = (t >> 12) & 0x1fff;
      const int nd = ((t >> 27) & 1) ? OZ_S_UP : OZ_S;
      const int nkc_t = oz_tile_nkc(t, p.nkc);
      for (int sub = 0; sub < OZ_NSUB; sub++) {
        const int arow = (r * OZ_TM + (sub & 1) * OZ_SUB) / 8, brow = (c * OZ_TN + (sub >> 1) * OZ_SUB) / 8;
        for (int kc = 0; kc < nkc_t; kc++, it++) {
          const int st = it % OZ_STAGES;
          mbar_wait_backoff(&empty[st], ((it / OZ_STAGES) & 1) ^ 1, 64);
          if (lane == 0) mbar_arrive_expect_tx(&full[st], (uint32_t)nd * 2 * OZ_PLANE);
          __syncwarp();
          unsigned char* dst = ring + st * OZ_STAGE_BYTES;
          if (lane < nd) {
            tma_load_4d(dst + lane * OZ_PLANE, &mapA, 0, arow, kc, lane, &full[st]);
            tma_load_4d(dst + (OZ_S + lane) * OZ_PLANE, &mapB, 0, brow, kc, lane, &full[st]);
          }
        }
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    if (wg == 0) oz_consume<0>(p, ring, xch, full, empty, ti_beg, ti_end);
    else oz_consume<1>(p, ring, xch, full, empty, ti_beg, ti_end);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// tile lists of the sweep (host): per panel step the launches U1 | U2 (+ the K^-1 tiles of the step) and the panel GEMM
// ---------------------------------------------------------------------------------------------------------------
// tiles in bands of 8 row tiles x 8 column tiles: the CTAs in flight share a few operand panels in L2
template <class Valid, class Emit>
static void oz_banded(const std::vector<int>& rows, int ct_beg, int ct_end, Valid valid, Emit emit) {
  for (size_t b = 0; b < rows.size(); b += 8)
    for (int cc = ct_beg; cc < ct_end; cc += 8)
      for (size_t i = b; i < std::min(rows.size(), b + 8); i++)
        for (int ct = cc; ct < std::min(ct_end, cc + 8); ct++)
          if (valid(rows[i], ct)) emit(rows[i], ct);
}

void oz_build_lists(long Npad, long NB, std::vector<uint32_t>& tiles, std::vector<OzStep>& steps) {
  const int nt = (int)(Npad / TILE);
  tiles.clear();
  steps.clear();
  for (long o = 0; o < Npad; o += NB) {
    const long nb = std::min(NB, Npad - o);
    const int kt0 = (int)(o / TILE), kt1 = kt0 + (int)(nb / TILE);
    const int next_nbt = kt1 < nt ? (int)(std::min(NB, Npad - (o + nb)) / TILE) : 0;
    OzStep st;
    // S(r, c) -= P_r P_c^T, c in [cbeg, cend), r in [0, kt1) U [c, nt) outside block k+1: the next diagonal block is updated
    // in fp64 by the serial chain of the sweep
    std::vector<int> urows;
    for (int r = 0; r < kt1; r++) urows.push_back(r);
    for (int r = kt1 + next_nbt; r < nt; r++) urows.push_back(r);
    auto emit_update = [&](int cbeg, int cend) {
      oz_banded(urows, cbeg, cend, [&](int r, int c) { return r < kt1 || c <= r; },
                [&](int r, int c) { tiles.push_back(oz_tile(r, c, OZ_UPDATE, r < kt1 ? 1 : 0)); });
    };
    auto count_up = [&](int off, int n) { int u = 0; for (int i = off; i < off + n; i++) u += (tiles[i] >> 27) & 1; return u; };
    // U1: the rest of block column k+1 (rows above the block and below it)
    st.u1_off = (int)tiles.size();
    emit_update(kt1, kt1 + next_nbt);
    st.u1_n = (int)tiles.size() - st.u1_off;
    st.u1_up = count_up(st.u1_off, st.u1_n);
    // U2: the columns after block k+1, then the K^-1 tiles
    st.u2_off = (int)tiles.size();
    emit_update(kt1 + next_nbt, nt);
    {   // K^-1(r, c) (+)= P_r P_c^T for c <= r < kt1: rows of block k see their first contribution at this step
      std::vector<int> rows;
      for (int r = 0; r < kt1; r++) rows.push_back(r);
      oz_banded(rows, 0, kt1, [&](int r, int c) { return c <= r; },
                [&](int r, int c) { tiles.push_back(oz_tile(r, c, r >= kt0 ? OZ_LAUUM_SET : OZ_LAUUM_ACC, 1)); });
    }
    st.u2_n = (int)tiles.size() - st.u2_off;
    st.u2_up = count_up(st.u2_off, st.u2_n);
    {   // panel GEMM on the tensor cores: P(r, c') for the rows outside the diagonal block and block k+1, c' < nb / 128
      st.pan_off = (int)tiles.size();
      const int nbt = kt1 - kt0;
      std::vector<int> rows;
      for (int r = 0; r < kt0; r++) rows.push_back(r);
      for (int r = kt1 + next_nbt; r < nt; r++) rows.push_back(r);
      for (size_t b = 0; b < rows.size(); b += 8)              // bands of 8 row tiles; longest k-range (last column tile) first
        for (int cc = nbt - 1; cc >= 0; cc--)
          for (size_t i = b; i < std::min(rows.size(), b + 8); i++) tiles.push_back(oz_tile(rows[i], cc, OZ_PANEL, rows[i] < kt0 ? 1 : 0));
      st.pan_n = (int)tiles.size() - st.pan_off;
    }
    steps.push_back(st);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn g_encode = nullptr;

int oz_init() {
  if (!g_encode) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    GPX_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
    if (qres != cudaDriverEntryPointSuccess || !fn) { set_error("cuTensorMapEncodeTiled is not available in this driver"); return -1; }
    g_encode = reinterpret_cast<EncodeTiledFn>(fn);
  }
  GPX_CUDA(cudaFuncSetAttribute(oz_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, OZ_SMEM));
  return 0;
}

static int oz_make_map(CUtensorMap* map, const OzPlanes& pl) {
  const cuuint64_t ngrp = (cuuint64_t)(pl.rows / 8);
  cuuint64_t dims[4] = {256, ngrp, (cuuint64_t)pl.nkc, (cuuint64_t)OZ_S};
  cuuint64_t strides[3] = {256, ngrp * 256, (cuuint64_t)pl.nkc * ngrp * 256};
  cuuint32_t box[4] = {256, (cuuint32_t)(OZ_SUB / 8), 1, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  const CUresult r = g_encode(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 4, pl.planes, dims, strides, box, estr,
                              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (" + std::to_string((int)r) + ")"); return -1; }
  return 0;
}

int oz_planes_alloc(OzPlanes& pl, long rows, long K) {
  if (rows % OZ_TM || K % OZ_KC) { set_error("oz_planes_alloc: rows % 128 or K % 32"); return -2; }
  pl.rows = rows;
  pl.nkc = (int)(K / OZ_KC);
  GPX_CUDA(cudaMalloc(&pl.planes, (size_t)OZ_S * rows * K));
  GPX_CUDA(cudaMalloc(&pl.scale, (size_t)rows * 8));
  GPX_CUDA(cudaMalloc(&pl.amax_part, (size_t)rows * 8 * 8));   // SPLIT_KS partial row maxima
  if (oz_make_map(&pl.map, pl)) return -1;
  return 0;
}

void oz_planes_free(OzPlanes& pl) {
  if (pl.planes) cudaFree(pl.planes);
  if (pl.scale) cudaFree(pl.scale);
  if (pl.amax_part) cudaFree(pl.amax_part);
  pl.planes = nullptr; pl.scale = nullptr; pl.amax_part = nullptr; pl.rows = 0; pl.nkc = 0;
}

int launch_oz_gemm(const OzPlanes& pl, const OzParams& p_in, int num_sms, cudaStream_t st, const OzPlanes* plB) {
  if (p_in.ntiles <= 0) return 0;
  OzParams p = p_in;
  // default: 4 tiles per CTA when there is enough work
  if (p.tpc <= 0) p.tpc = std::max(1, std::min(4, p.ntiles / std::max(1, num_sms)));
  const int grid = (p.ntiles + p.tpc - 1) / p.tpc;
  oz_gemm_kernel<<<grid, OZ_THREADS, OZ_SMEM, st>>>(pl.map, plB ? plB->map : pl.map, p);
  GPX_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace gpx
