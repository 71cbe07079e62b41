// gpx_ozaki.cuh — fp64-grade GEMM on the INT8 tensor path (wgmma s8 x s8 -> s32, register accumulators, TMA-fed): internal API.
#pragma once
#include <cuda.h>
#include <stdint.h>

#include <vector>

#include "gpx_common.cuh"

struct gpx_ctx;

namespace gpx {

constexpr int OZ_S = 8;         // signed 7-bit digit planes per fp64 operand (56 bits >= the 53-bit significand); digits used
                                // for Cholesky-part tiles
constexpr int OZ_S_UP = 7;      // digits used for inverse-part / K^-1 tiles, which feed only the gradients (28 digit pairs
                                // instead of 36, gradient error ~6e-10 at N = 16384; DESIGN.md §5.1)
constexpr int OZ_TM = 128;      // output tile rows    (two 64-row wgmma sub-tiles)
constexpr int OZ_TN = 128;      // output tile columns (two 64-column wgmma sub-tiles)
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

// one output tile: bits 0-11 row tile, 12-24 column tile, 25-26 kind, 27 inverse-part tile
enum OzKind { OZ_UPDATE = 0, OZ_LAUUM_ACC = 1, OZ_LAUUM_SET = 2, OZ_PANEL = 3 };
inline uint32_t oz_tile(int r, int c, int kind, int upper) {
  return (uint32_t)r | ((uint32_t)c << 12) | ((uint32_t)kind << 25) | ((uint32_t)upper << 27);
}

struct OzParams {
  const uint32_t* tiles;   // device tile list of this launch
  int ntiles;
  int nkc;                 // K / 32
  const double* scale;     // row scales of the panel (shared by both operands: C (op)= P_r P_c^T)
  double* S; long lds;     // OZ_UPDATE target:      S(r, c)    -= P_r P_c^T
  double* Kinv; long ldk;  // OZ_LAUUM_* target:     Kinv(r, c) (+)= P_r P_c^T   (lower tiles)
  int tpc;                 // consecutive tiles per CTA (0 = default)
  // OZ_PANEL tiles: P(r, c') = A_r B_c'^T with A = digit planes of a block column of the workspace (pl of launch_oz_gemm),
  // B = digit planes of L_kk^-1 (plB of launch_oz_gemm), lower triangular: the k-range of output column tile c' ends at
  // (c' + 1) * 128. Result stored (not accumulated) into P.
  double* P; long ldp;
  double* Pfinal;          // optional second target of OZ_PANEL tiles: the block column of the workspace itself (ld = lds)
  const double* scaleB;    // row scales of the B operand's planes (= column scales of the product)
};

// one panel step of the sweep: offsets into the tile list. U1: block column k+1 outside its diagonal block; U2: the other
// update tiles, then the K^-1 tiles; pan: the panel GEMM rows outside the diagonal block and block k+1; *_up = inverse-part
// tiles among them
struct OzStep { int u1_off, u1_n, u1_up, u2_off, u2_n, u2_up, pan_off, pan_n; };
void oz_build_lists(long Npad, long NB, std::vector<uint32_t>& tiles, std::vector<OzStep>& steps);

int oz_init();                                                          // driver entry point + kernel attributes
int oz_planes_alloc(OzPlanes& pl, long rows, long K);                    // buffers + tensor maps
void oz_planes_free(OzPlanes& pl);
int launch_oz_split(const double* P, long ld, long K, OzPlanes& pl, cudaStream_t st);   // P: rows x K column-major, K <= layout
int launch_oz_gemm(const OzPlanes& pl, const OzParams& p, int num_sms, cudaStream_t st, const OzPlanes* plB = nullptr);

}  // namespace gpx
