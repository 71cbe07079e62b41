// gpx_ozaki.cuh — fp64-grade GEMM on the INT8 tensor path (wgmma s8 x s8 -> s32, register accumulators, TMA-fed): internal API.
#pragma once
#include <cuda.h>
#include <stdint.h>

#include <vector>

#include "gpx_common.cuh"

struct gpx_ctx;

namespace gpx {

constexpr int OZ_S = 8;         // signed 7-bit digit planes per fp64 operand (56 bits >= the 53-bit significand)
constexpr int OZ_TM = 128;      // output tile rows   (two 64-row wgmma sub-tiles)
constexpr int OZ_TN = 64;       // output tile columns (= wgmma N; 128 with option oz_wide)
constexpr int OZ_KC = 32;       // k-depth of one wgmma .s8 (32 bytes of K)

// Digit planes of one panel (rows x K, K = nkc * 32), stored so that every (plane, k-chunk, 8-row group) is one 256-byte
// block in exactly the shared-memory image wgmma reads (no-swizzle K-major core matrices: two 8 x 16 B core matrices per
// block). A tile of R rows of one (plane, k-chunk) is therefore R*32 contiguous bytes = one TMA box {256, R/8, 1, 1}.
//   byte offset of digit s of element (row i, column k):
//     (((s * nkc + k/32) * (rows/8) + i/8) * 256) + ((k%32)/16)*128 + (i%8)*16 + k%16
struct OzPlanes {
  int8_t* planes = nullptr;     // [S][nkc][rows/8][256]
  double* scale = nullptr;      // [rows]: 2^(e_i + 1 - 7), e_i = exponent of the row maximum over the K columns of the panel
  double* amax_part = nullptr;  // [8][rows]: partial row maxima (scratch of the split)
  long rows = 0;
  int nkc = 0;
  CUtensorMap map;              // the tensor with a 64-row box (one wgmma operand of one plane and k-chunk)
};

// one output tile: bits 0-11 row tile (128 rows), 12-24 column tile (64 columns), 25-26 kind, 27 inverse-part tile
enum OzKind { OZ_UPDATE = 0, OZ_LAUUM_ACC = 1, OZ_LAUUM_SET = 2, OZ_PANEL = 3 };
inline uint32_t oz_tile(int r, int c64, int kind, int upper) {
  return (uint32_t)r | ((uint32_t)c64 << 12) | ((uint32_t)kind << 25) | ((uint32_t)upper << 27);
}

struct OzParams {
  const uint32_t* tiles;   // device tile list of this launch
  int ntiles;
  int nkc;                 // K / 32
  const double* scale;     // row scales of the panel (shared by both operands: C (op)= P_r P_c^T)
  double* S; long lds;     // OZ_UPDATE target:      S(r, c)    -= P_r P_c^T
  double* Kinv; long ldk;  // OZ_LAUUM_* target:     Kinv(r, c) (+)= P_r P_c^T   (lower tiles)
  int dig_lo, dig_up;      // digits per operand for Cholesky-part tiles / inverse-part tiles (<= OZ_S)
  int tpc;                 // consecutive tiles per CTA (0 = default)
  int wide;                // 1: 128 x 128 tiles (column tile index in 128-column units), 0: 128 x 64 tiles
  // OZ_PANEL tiles (wide only): P(r, c') = A_r B_c'^T with A = digit planes of a block column of the workspace
  // (pl of launch_oz_gemm), B = digit planes of L_kk^-1 (plB of launch_oz_gemm), lower triangular: the k-range of output
  // column tile c' ends at (c' + 1) * 128. Result stored (not accumulated) into P.
  double* P; long ldp;
  double* Pfinal;          // optional second target of OZ_PANEL tiles: the block column of the workspace itself (ld = lds)
  const double* scaleB;    // row scales of the B operand's planes (= column scales of the product)
};

// one panel step of the sweep: offsets into the tile list. U0: the next diagonal block only; U1: the rest of block column k+1;
// U2 list: u2_upd update tiles, then the K^-1 tiles; *_up = inverse-part tiles among them
struct OzStep { int u0_off, u0_n, u1_off, u1_n, u2_off, u2_n, u2_upd, u0_up, u1_up, u2_up, u2_upd_up;
                // panel GEMM of the step on the tensor cores: rows outside the diagonal block and the next block
                int pan_off, pan_n, pan_up; };
void oz_build_lists(long Npad, long NB, int cw, int own_G, int own_g, std::vector<uint32_t>& tiles, std::vector<OzStep>& steps);

int oz_init();                                                          // driver entry point + kernel attributes
int oz_planes_alloc(OzPlanes& pl, long rows, long K);                    // buffers + tensor maps
void oz_planes_free(OzPlanes& pl);
int launch_oz_split(const double* P, long ld, long K, OzPlanes& pl, cudaStream_t st);   // P: rows x K column-major, K <= layout
int launch_oz_gemm(const OzPlanes& pl, const OzParams& p, int num_sms, cudaStream_t st, const OzPlanes* plB = nullptr);

// gradient reductions from a stored K^-1 (lower 128 x 128 tiles, column-major, leading dimension ld): same partial sums as
// the fused epilogue of gemm_lauum_kernel, consumed by finalize_kernel
struct GradKinvParams {
  const double* Kinv; long ld;
  const double* XsT; const double* sq; const double* alpha; long ldx;
  long N; int P; int nt;
  double* partials;        // [nt*nt*csplit][nl+2], zeroed by the caller
  int csplit;              // CTAs per tile (each takes 64/csplit columns of both column halves): 1, 2, 4 or 8 -- small matrices
                           // have too few tiles to fill the machine, and a thread's 64 columns are a serial chain
  double* dnoise_out;      // optional diag(dL_dK)
  KernParams kp;
};
int launch_grad_kinv(const GradKinvParams& p, cudaStream_t st);
int grad_kinv_csplit(int nt, int nred);   // the split launch_grad_kinv expects for this matrix (partials: nt*nt*(MAX_D+2) doubles)

}  // namespace gpx
