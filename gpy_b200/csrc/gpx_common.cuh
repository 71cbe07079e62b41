// gpx_common.cuh — shared definitions for the sm_90a exact-GP kernels (internal; the public ABI is include/gpx.h).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>

#include <string>
#include <vector>

#include "../../include/gpx.h"

namespace gpx {

constexpr int TILE = 128;        // base tile edge: GEMM CTA tile, base factor block, padding quantum
constexpr int KSLAB = 16;        // k-depth of one smem pipeline stage
constexpr int PITCH = 132;       // smem row pitch in doubles (== 4 mod 16 -> conflict-free DMMA fragment loads)
constexpr int STAGES = 4;
constexpr int CONSUMER_WARPS = 8;
constexpr int PRODUCER_WARPS = 4;   // one full warpgroup (setmaxnreg is warpgroup-wide); only its first warp works
constexpr int GEMM_THREADS = (CONSUMER_WARPS + PRODUCER_WARPS) * 32;
constexpr int MAX_D = 64;        // fused gradient epilogue limit on the input dimension
constexpr int MAX_P = 8;         // fused path limit on the number of output columns

struct KernParams {
  int kind;         // GPX_RBF ...
  int ard;
  int D;
  double variance;
  double inv_ls_iso;        // 1/l for the isotropic case (r = sqrt(r2) * inv_ls_iso); 1.0 when ard
  double ls[MAX_D];         // lengthscales (ard: D entries; iso: ls[0])
};

// ---------------------------------------------------------------------------------------------------------------
// kernel functions of r (reference: rbf.py:51-52,177-178; stationary.py:382-386,488-492,585-589), unit variance
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ double k_of_r_unit(int kind, double r) {
  switch (kind) {
    case GPX_RBF: return exp(-0.5 * r * r);
    case GPX_EXPONENTIAL: return exp(-r);
    case GPX_MATERN32: { const double s3 = 1.7320508075688772; return (1.0 + s3 * r) * exp(-s3 * r); }
    default: { const double s5 = 2.23606797749979; return (1.0 + s5 * r + (5.0 / 3.0) * r * r) * exp(-s5 * r); }
  }
}
// returns k(r) and dk/dr for unit variance
__device__ __forceinline__ void k_dk_of_r_unit(int kind, double r, double& k, double& dk) {
  switch (kind) {
    case GPX_RBF: k = exp(-0.5 * r * r); dk = -r * k; break;
    case GPX_EXPONENTIAL: k = exp(-r); dk = -k; break;
    case GPX_MATERN32: {
      const double s3 = 1.7320508075688772; const double e = exp(-s3 * r);
      k = (1.0 + s3 * r) * e; dk = -3.0 * r * e; break;
    }
    default: {
      const double s5 = 2.23606797749979; const double e = exp(-s5 * r);
      k = (1.0 + s5 * r + (5.0 / 3.0) * r * r) * e;
      dk = ((10.0 / 3.0) * r - 5.0 * r - (5.0 * s5 / 3.0) * r * r) * e; break;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// PTX helpers: mbarrier + 1-D bulk async copy (TMA engine, SASS UBLKCP) + fp64 tensor MMA (SASS DMMA.16x8x4)
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// global -> shared bulk copy (bytes multiple of 16, both addresses 16-B aligned), completion on an mbarrier
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// D(16x8) += A(16x4, row) * B(4x8, col), the sm_90 fp64 shape (SASS DMMA.16x8x4): lane holds A[g][t], A[g+8][t], B[t][g],
// C[g][2t..2t+1], C[g+8][2t..2t+1] with g = lane>>2, t = lane&3. On the H100 it issues at twice the rate of m8n8k4.
__device__ __forceinline__ void dmma1684(double& c0, double& c1, double& c2, double& c3, double a0, double a1, double b) {
  asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
               : "+d"(c0), "+d"(c1), "+d"(c2), "+d"(c3)
               : "d"(a0), "d"(a1), "d"(b));
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------
void set_error(const std::string& msg);
#define GPX_CUDA(call)                                                                                  \
  do {                                                                                                  \
    cudaError_t e__ = (call);                                                                           \
    if (e__ != cudaSuccess) {                                                                           \
      gpx::set_error(std::string(#call) + " failed: " + cudaGetErrorString(e__) + " at " + __FILE__ + ":" + \
                     std::to_string(__LINE__));                                                         \
      return -1;                                                                                        \
    }                                                                                                   \
  } while (0)

// GEMM launch descriptor (see gpx_gemm.cu)
enum GemmMode { GEMM_UPDATE = 0, GEMM_PANEL = 1, GEMM_LAUUM = 2 };

struct GemmParams {
  int mode;
  // operands: element (m, k) of row-tile r lives at A[r*TILE + m + k*lda]; B likewise with column-tile index
  const double* A; long lda;
  const double* B; long ldb;
  double* C; long ldc;
  int K;        // k-depth (UPDATE / PANEL); LAUUM: padded order of the matrix
  int nt;       // number of row tiles of the (sub)matrix
  int c0;       // first column tile handled (UPDATE: kt1; PANEL: 0)
  int ncols;    // UPDATE/LAUUM: number of column tiles handled (0 = up to nt)
  int rlow;     // UPDATE: rows [0, rlow) above the trailing part take part (upper, inverse region)
  int skip0, skip1;  // PANEL: row tiles [skip0, skip1) (the diagonal block) are skipped
  int tri;      // PANEL: B is lower triangular -> k range of output column tile c' is [0, (c'+1)*TILE)
  int plain;    // PANEL entry used as a general C = A B^T over nt x ncols tiles (super-block schedule); 2 = lower tiles only
  // LAUUM epilogue (fused gradient reductions)
  const double* XsT;    // scaled inputs, SoA [D][ldx]
  const double* sq;     // squared norms of scaled inputs [ldx]
  const double* alpha;  // [P][ldx]
  long ldx;
  int N;                // logical order (rows/cols >= N are padding)
  int P;
  double* partials;     // [tiles][nred]
  double* kinv_out;     // optional: store K^-1 lower tiles (ld = ldc), may be null
  // ---- multi-GPU (all zero / one on a single GPU) ---------------------------------------------------------------
  // block-mapped operands: row tile r of a mapped matrix lives in chunk pos(R) = (R % map_G) * map_npr + R / map_G,
  // R = r / map_blk, at  base + pos * map_stride + (r % map_blk) * TILE  (chunks are map_blk*TILE rows, column-major)
  int map_A, map_B, map_C;     // which of A / B / C use the block mapping
  int map_blk, map_G, map_npr; long map_stride;
  int own_G, own_g, own_blk;   // UPDATE / PANEL: a tile is processed iff ((r / own_blk) % own_G) == own_g
  int k_G, k_g, k_blk;         // LAUUM: only k-tiles inside column blocks kb == k_g (mod k_G), k_blk tiles per block
  // memory-distributed layout: a rank stores only the block rows it owns (row tile r at local tile loc_tile(r, own_G,
  // own_blk)) and, for U = L^-T, only the column blocks it owns (k-tile kt at local tile loc_tile(kt, k_G, k_blk))
  int loc_A, loc_C;            // PANEL: A rows / UPDATE: C rows are local
  int k_local;                 // LAUUM: the k index of A and B is local
  KernParams kp;
  double* dnoise_out;   // LAUUM epilogue, optional: diag(dL_dK)_i per data point (heteroscedastic noise gradients)
};

// local tile index of an OWNED global tile t under a block-cyclic deal of blocks of `blk` tiles over G ranks
__host__ __device__ __forceinline__ long loc_tile(int t, int G, int blk) {
  return G <= 1 ? (long)t : (long)((t / blk) / G) * blk + t % blk;
}

int launch_gemm(const GemmParams& p, dim3 grid, cudaStream_t st);
size_t gemm_smem_bytes();
int gemm_init();  // set max dynamic smem attribute

}  // namespace gpx
