// gpx_kernels.cu — the non-GEMM kernels of the exact-GP path: input scaling, covariance build, the 128x128 base
// factor-and-invert block, triangular matrix-vector products, block assembly, result extraction, final reduction.
#include "gpx_common.cuh"

#include <cstring>

#include "gpx_kernels.cuh"

namespace gpx {

// =================================================================================================================
// prep: scaled inputs in SoA layout + squared norms.
// Reference: Stationary._scaled_dist (stationary.py:151-168: ARD divides X by the lengthscale BEFORE the distance
// expansion; iso leaves X alone and divides r afterwards) and the Xsq row sums of _unscaled_dist (:136).
// =================================================================================================================
__global__ void prep_x_kernel(const double* __restrict__ X, long N, long ldx, KernParams kp, double* __restrict__ XsT,
                              double* __restrict__ sq) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ldx) return;
  double s = 0.0;
  for (int q = 0; q < kp.D; q++) {
    double v = 0.0;
    if (i < N) {
      v = X[i * kp.D + q];
      if (kp.ard) v = v / kp.ls[q];
    }
    XsT[(long)q * ldx + i] = v;
    s += v * v;
  }
  sq[i] = s;
}

int launch_prep_x(const double* X, long N, long ldx, const KernParams& kp, double* XsT, double* sq, cudaStream_t st) {
  prep_x_kernel<<<(unsigned)((ldx + 255) / 256), 256, 0, st>>>(X, N, ldx, kp, XsT, sq);
  GPX_CUDA(cudaGetLastError());
  return 0;
}

// =================================================================================================================
// covariance build.  out(rowidx, colidx) at out[rowidx + colidx*ld]; the thread-mapped (contiguous) index is the
// ROW operand. One CTA = one 128x128 tile; the two D x 128 input tiles (SoA) and their squared norms are staged in
// shared memory by 1-D bulk async copies (TMA engine) on an mbarrier; each thread keeps its row point in registers
// and walks 64 columns, writing 256-byte-per-warp coalesced column segments.
// Reference: stationary.py:130-148 (_unscaled_dist: |x|^2+|x'|^2-2x.x', diagonal forced to 0, clip at 0, sqrt),
// :151-168 (scaling), K_of_r (rbf.py:51-52; stationary.py:382-383,488-489,585-586), and, in `sym` mode,
// Ky = K + (noise + jitter) I (exact_gaussian_inference.py:55-56) written straight into the factor workspace
// (lower tiles; upper tiles zero = the initial state of the inverse-factor region; padding = identity).
// =================================================================================================================
template <int KIND>
__device__ __forceinline__ double k_unit(double r) {
  if (KIND == GPX_RBF) return exp(-0.5 * r * r);
  if (KIND == GPX_EXPONENTIAL) return exp(-r);
  if (KIND == GPX_MATERN32) { const double s3 = 1.7320508075688772; return (1.0 + s3 * r) * exp(-s3 * r); }
  const double s5 = 2.23606797749979;
  return (1.0 + s5 * r + (5.0 / 3.0) * r * r) * exp(-s5 * r);
}

template <int DREG, int KIND>
__global__ void __launch_bounds__(256) kbuild_kernel(KBuildParams p) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int D = p.kp.D;
  double* sR = reinterpret_cast<double*>(smem_raw);          // [D][128] row-operand points
  double* sC = sR + (size_t)D * TILE;                        // [D][128] col-operand points
  double* sSr = sC + (size_t)D * TILE;
  double* sSc = sSr + TILE;
  uint64_t* bar = reinterpret_cast<uint64_t*>(sSc + TILE);

  const int ct = blockIdx.x, rt = p.rt0 + blockIdx.y;
  if (p.own_G > 1 && ((rt / p.own_blk) % p.own_G) != p.own_g) return;   // block row owned by another rank
  const int tid = threadIdx.x;
  const int il = tid & (TILE - 1), half = tid >> 7;
  const long gi = (long)rt * TILE + il;
  double* outp = p.out + (p.loc_rows ? loc_tile(rt, p.own_G, p.own_blk) * TILE + il : gi) + ((long)ct * TILE + half * 64) * p.ld;

  if (p.sym && rt < ct) {  // strictly-upper tile of the factor workspace: the inverse-factor region starts at zero
#pragma unroll 8
    for (int j = 0; j < 64; j++) outp[(long)j * p.ld] = 0.0;
    return;
  }
  if (tid == 0) { mbar_init(bar, 1); fence_mbar_init(); }
  __syncthreads();
  if (tid == 0) {
    mbar_arrive_expect_tx(bar, (uint32_t)((2 * D + 2) * TILE * 8));
    for (int q = 0; q < D; q++) {
      bulk_g2s(sR + q * TILE, p.rowsT + (long)q * p.ld_rows + (long)rt * TILE, TILE * 8, bar);
      bulk_g2s(sC + q * TILE, p.colsT + (long)q * p.ld_cols + (long)ct * TILE, TILE * 8, bar);
    }
    bulk_g2s(sSr, p.sq_rows + (long)rt * TILE, TILE * 8, bar);
    bulk_g2s(sSc, p.sq_cols + (long)ct * TILE, TILE * 8, bar);
  }
  mbar_wait(bar, 0);

  double xi[DREG];
#pragma unroll
  for (int q = 0; q < DREG; q++) xi[q] = q < D ? sR[q * TILE + il] : 0.0;
  const double si = sSr[il];
  const double variance = p.kp.variance, inv_ls = p.kp.inv_ls_iso;
  const double* sCj = sC + half * 64;
  const double* sScj = sSc + half * 64;
  // interior tiles (no diagonal, no padding) take the branch-free loop; the tile test is block-uniform
  const bool edge = (rt == ct && p.same) || ((long)rt * TILE + TILE > p.nrows) || ((long)ct * TILE + TILE > p.ncols);
  if (!edge) {
#pragma unroll 4
    for (int j = 0; j < 64; j++) {
      double dot = 0.0;
#pragma unroll
      for (int q = 0; q < DREG; q++)
        if (q < D) dot = fma(xi[q], sCj[q * TILE + j], dot);
      const double r2 = fmax(si + sScj[j] - 2.0 * dot, 0.0);
      outp[0] = variance * k_unit<KIND>(sqrt(r2) * inv_ls);
      outp += p.ld;
    }
    return;
  }
  const bool row_valid = gi < p.nrows;
  for (int j = 0; j < 64; j++) {
    const long gj = (long)ct * TILE + half * 64 + j;
    double dot = 0.0;
#pragma unroll
    for (int q = 0; q < DREG; q++)
      if (q < D) dot = fma(xi[q], sCj[q * TILE + j], dot);
    double r2 = si + sScj[j] - 2.0 * dot;
    if (p.same && gi == gj) r2 = 0.0;
    r2 = fmax(r2, 0.0);
    double v = variance * k_unit<KIND>(sqrt(r2) * inv_ls);
    if (p.sym) {
      if (gi == gj) v = v + p.diag_add + ((p.diag_vec && row_valid) ? p.diag_vec[gi] : 0.0);
      if (!row_valid || gj >= p.ncols) v = (gi == gj) ? 1.0 : 0.0;
      outp[(long)j * p.ld] = v;
    } else if (row_valid && gj < p.ncols) {
      outp[(long)j * p.ld] = v;
    }
  }
}

template <int DREG>
static int launch_kbuild_kind(const KBuildParams& p, dim3 grid, size_t smem, cudaStream_t st) {
#define GPX_KB(KD)                                                                                              \
  do {                                                                                                          \
    static bool attr_set = false;                                                                               \
    if (!attr_set) {                                                                                            \
      GPX_CUDA(cudaFuncSetAttribute(kbuild_kernel<DREG, KD>, cudaFuncAttributeMaxDynamicSharedMemorySize,       \
                                    (int)((2 * MAX_D + 2) * TILE * 8 + 16)));                                   \
      attr_set = true;                                                                                          \
    }                                                                                                           \
    kbuild_kernel<DREG, KD><<<grid, 256, smem, st>>>(p);                                                        \
  } while (0)
  switch (p.kp.kind) {
    case GPX_RBF: GPX_KB(GPX_RBF); break;
    case GPX_EXPONENTIAL: GPX_KB(GPX_EXPONENTIAL); break;
    case GPX_MATERN32: GPX_KB(GPX_MATERN32); break;
    default: GPX_KB(GPX_MATERN52); break;
  }
#undef GPX_KB
  return 0;
}

int launch_kbuild(const KBuildParams& p, int row_tiles, int col_tiles, cudaStream_t st) {
  const int D = p.kp.D;
  const size_t smem = (size_t)(2 * D + 2) * TILE * 8 + 16;
  dim3 grid(col_tiles, row_tiles);
  int rc;
  if (D <= 8) rc = launch_kbuild_kind<8>(p, grid, smem, st);
  else if (D <= 16) rc = launch_kbuild_kind<16>(p, grid, smem, st);
  else if (D <= 32) rc = launch_kbuild_kind<32>(p, grid, smem, st);
  else rc = launch_kbuild_kind<64>(p, grid, smem, st);
  if (rc) return rc;
  GPX_CUDA(cudaGetLastError());
  return 0;
}

// =================================================================================================================
// base block: unified factor-and-invert sweep of one 128x128 diagonal tile by one CTA of 512 threads, the tile resident
// in shared memory.
// On exit: lower = L_dd (to the Ldiag strip), strict upper + reciprocal diagonal = U_dd = L_dd^-T (written back to
// the tile itself: the diagonal tiles of the workspace hold U), Dinv strip = L_dd^-1 (lower, column-major).
// Replaces, for one block: lapack.dpotrf (GPy/util/linalg.py:58) and lapack.dtrtri (:227) incl. the
// "not positive definite" detection that drives jitchol (:59-75).
// The tile is processed in eight 16-column micro-panels jp:
//   (1) one warp factor-and-inverts the 16x16 diagonal micro-block in registers (micro_diag_row),
//   (2) the micro-panel  P = T(:, panel) W^T  (W = inverse of the micro-block) is formed in place with DMMA.16x8x4,
//   (3) T(r,c) -= P_r P_c^T  for the 16x16 micro-tiles c > jp, r in [0..jp] U [c..7] with DMMA.16x8x4 (fragments straight
//       from shared memory, pitch 132 -> conflict-free).
// =================================================================================================================
constexpr int BP = 132;   // pitch (doubles) of the shared tile, column-major: (row, col) at col*BP + row
constexpr int MP = 20;    // pitch of the 16x16 micro operand buffers

// (3) one 16 x (8*NI) piece of a micro-tile update  T(rt, ct) -= P_rt P_ct^T  (k-depth 16) with DMMA.16x8x4
template <int NI>
__device__ __forceinline__ void micro_update(double* T, int c0, int jp, int rt, int ct, int n0, const double* Pd,
                                             int lane) {
  const int g = lane >> 2, tg = lane & 3;
  const double* Ap = (rt == jp) ? Pd : (T + c0 * BP + rt * 16);
  const int apitch = (rt == jp) ? MP : BP;
  const double* Bp = T + c0 * BP + ct * 16 + n0;
  double* Cp = T + (ct * 16 + n0) * BP + rt * 16;
  double c[2][NI][2];
#pragma unroll
  for (int mi = 0; mi < 2; mi++)
#pragma unroll
    for (int ni = 0; ni < NI; ni++)
#pragma unroll
      for (int e = 0; e < 2; e++) c[mi][ni][e] = Cp[(ni * 8 + 2 * tg + e) * BP + mi * 8 + g];
#pragma unroll
  for (int k4 = 0; k4 < 4; k4++) {
    double af[2], bf[NI];
#pragma unroll
    for (int mi = 0; mi < 2; mi++) af[mi] = -Ap[(k4 * 4 + tg) * apitch + mi * 8 + g];
#pragma unroll
    for (int ni = 0; ni < NI; ni++) bf[ni] = Bp[(k4 * 4 + tg) * BP + ni * 8 + g];
#pragma unroll
    for (int mi = 0; mi < 2; mi += 2)
#pragma unroll
      for (int ni = 0; ni < NI; ni++) dmma1684(c[mi][ni][0], c[mi][ni][1], c[mi + 1][ni][0], c[mi + 1][ni][1],
                                                          af[mi], af[mi + 1], bf[ni]);
  }
#pragma unroll
  for (int mi = 0; mi < 2; mi++)
#pragma unroll
    for (int ni = 0; ni < NI; ni++)
#pragma unroll
      for (int e = 0; e < 2; e++) Cp[(ni * 8 + 2 * tg + e) * BP + mi * 8 + g] = c[mi][ni][e];
}

// reciprocal square root on the pivot chain: MUFU.RSQ64H + one third-order correction (branch-free, ~1 ulp; the library
// rsqrt has a special-case branch that splits the basic block the scheduler can interleave)
__device__ __forceinline__ double rsqrt_fast(double x) {
  double y;
  asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(x));   // relative error ~2^-22
  const double t = x * y;
  const double e = fma(-t, y, 1.0);                          // 1 - x y^2
  const double c = fma(0.375, e, 0.5);
  const double ye = y * e;
  return fma(ye, c, y);                                      // y (1 + e/2 + 3 e^2/8): error O(e^3)
}

// stream out the finished column block cb (16 columns): Ldiag and U columns, and rows [16cb, 16cb+16) of Dinv = L^-1 = U^T
__device__ __forceinline__ void base_out_block(const double* T, const double* dinv, const double* ldg, int cb, int t, int nthr,
                                               double* __restrict__ S, long ld, double* __restrict__ Ldiag,
                                               double* __restrict__ Dinv) {
  const int c0 = cb * 16;
  for (int idx = t; idx < 16 * TILE; idx += nthr) {
    const int row = idx & (TILE - 1), col = c0 + (idx >> 7);
    const double x = T[col * BP + row];
    Ldiag[row + col * TILE] = row > col ? x : (row == col ? ldg[row] : 0.0);
    S[row + (long)col * ld] = row > col ? 0.0 : (row == col ? dinv[row] : x);
  }
  for (int idx = t; idx < 16 * TILE; idx += nthr) {
    const int row = c0 + (idx & 15), col = idx >> 4;                     // W(row, col) = U(col, row): column `row` of T
    Dinv[row + col * TILE] = row > col ? T[row * BP + col] : (row == col ? dinv[row] : 0.0);
  }
}

__device__ __forceinline__ void named_sync(int id, int count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }
__device__ __forceinline__ void named_arrive(int id, int count) {
  __threadfence_block();
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// (1) the chain warp: factor-and-invert the 16x16 diagonal micro-block at (c0, c0). Lane r holds ROW r (both half-warps
// mirror each other), so a lane scales its own pivot-column entry without any exchange, and the next pivot
// d_{j+1} = v(j+1,j+1) - p_{j+1}^2 is formed locally in lane j+1: the pivot chain per column is multiply -> fused
// multiply-add -> shuffle -> MUFU.RSQ64H + 4 dependent fp64 operations. p_j(j+1), which the next column needs from lane j+1,
// travels by shuffle, the rest of the column through shared memory (vector loads issued together, off the chain). Writes
// the micro-block back (lower = L, strict upper = U), the operand copies Pd = U micro-block ((r,k) at k*MP+r) and
// Wm = U^T ((c,k) at k*MP+c), and the pivots.
__device__ __noinline__ void micro_diag_row(double* T, int c0, double* Pd, double* Wm, double* psh, double* dinv,
                                            double* ldg, int* info, int gcol0, int lane) {
  const int rr = lane & 15;
  double v[16];
#pragma unroll
  for (int q = 0; q < 16; q++) v[q] = (rr >= q) ? T[(c0 + q) * BP + c0 + rr] : 0.0;
  double my_inv = 0.0, my_l = 0.0;
  int badcol = -1;
  double d = __shfl_sync(0xffffffffu, v[0], 0);
#pragma unroll
  for (int j = 0; j < 16; j++) {
    if (!(d > 0.0) && badcol < 0) badcol = j;
    const double inv = rsqrt_fast(d);
    const double l = d * inv;
    const double p = (rr == j) ? inv : v[j] * inv;
    if (rr == j) { my_inv = inv; my_l = l; }
    v[j] = (rr == j) ? l : p;
    if (j < 15) {
      const double dn = fma(-p, p, v[j + 1]);            // lane j+1: the next pivot, from its own data only
      d = __shfl_sync(0xffffffffu, dn, j + 1);
      const double pn = __shfl_sync(0xffffffffu, p, j + 1);
      v[j + 1] = fma(-p, pn, v[j + 1]);                  // column j+1: every row takes part (rr <= j or rr >= j+1)
    }
    if (j < 14) {
      double* pj = psh + (j & 1) * 16;
      pj[rr] = p;
      __syncwarp();
      double pc[16];
#pragma unroll
      for (int c2 = (j + 2) >> 1; c2 < 8; c2++) {
        const double2 t2 = reinterpret_cast<const double2*>(pj)[c2];
        pc[2 * c2] = t2.x; pc[2 * c2 + 1] = t2.y;
      }
      const bool up = rr <= j;
#pragma unroll
      for (int col = j + 2; col < 16; col++)
        if (up || rr >= col) v[col] = fma(-p, pc[col], v[col]);
    }
  }
  if (badcol >= 0 && lane == 0) atomicCAS(info, 0, gcol0 + c0 + badcol + 1);
  if (lane < 16) {
#pragma unroll
    for (int col = 0; col < 16; col++) {
      T[(c0 + col) * BP + c0 + rr] = v[col];
      const double u = rr < col ? v[col] : (rr == col ? my_inv : 0.0);   // U(rr, col), reciprocal pivot on the diagonal
      Pd[col * MP + rr] = u;
      Wm[rr * MP + col] = u;                                               // W(col, rr) = U(rr, col)
    }
    dinv[c0 + rr] = my_inv; ldg[c0 + rr] = my_l;
  }
  __syncwarp();
}

// one row block of the micro-panel: T(rt, panel jp) <- T(rt, panel jp) W^T (in place), one warp
__device__ __forceinline__ void micro_panel_rows(double* T, int c0, int rt, const double* Wm, int lane) {
  const int g = lane >> 2, tg = lane & 3;
  double* Ap = T + c0 * BP + rt * 16;
  double af[2][4], c[2][2][2];
#pragma unroll
  for (int mi = 0; mi < 2; mi++)
#pragma unroll
    for (int k4 = 0; k4 < 4; k4++) af[mi][k4] = Ap[(k4 * 4 + tg) * BP + mi * 8 + g];
#pragma unroll
  for (int mi = 0; mi < 2; mi++)
#pragma unroll
    for (int ni = 0; ni < 2; ni++) { c[mi][ni][0] = 0.0; c[mi][ni][1] = 0.0; }
#pragma unroll
  for (int k4 = 0; k4 < 4; k4++) {
    double bf[2];
#pragma unroll
    for (int ni = 0; ni < 2; ni++) bf[ni] = Wm[(k4 * 4 + tg) * MP + ni * 8 + g];
#pragma unroll
    for (int mi = 0; mi < 2; mi += 2)
#pragma unroll
      for (int ni = 0; ni < 2; ni++) dmma1684(c[mi][ni][0], c[mi][ni][1], c[mi + 1][ni][0], c[mi + 1][ni][1],
                                                          af[mi][k4], af[mi + 1][k4], bf[ni]);
  }
  __syncwarp();                                       // every lane has read its A fragments: overwrite in place
#pragma unroll
  for (int mi = 0; mi < 2; mi++)
#pragma unroll
    for (int ni = 0; ni < 2; ni++)
#pragma unroll
      for (int e = 0; e < 2; e++) Ap[(ni * 8 + 2 * tg + e) * BP + mi * 8 + g] = c[mi][ni][e];
  __syncwarp();
}

// The serial part of the tile is the chain of its eight diagonal micro-blocks, so the chain warp (warp 0) RUNS AHEAD of the
// other fifteen: it does by itself the only pieces of (2) and (3) the next micro-block needs -- P(jp+1, jp) = T(jp+1, jp) W^T
// and T(jp+1, jp+1) -= P P^T, 32 DMMAs -- and goes straight on to micro-block jp+1, while warps 1..15 do the rest of the
// micro-panel and of the rank-16 update of step jp and stream the finished column block out (Ldiag, U into the workspace
// tile, the rows of L^-1). Producer / consumer hand-overs through named barriers (bar.arrive / bar.sync, two of each kind
// alternating by step parity):
//   A[jp&1]: warp 0 -> bulk : W(jp), U micro-block and P(jp+1, jp) are in shared memory
//   D[jp&1]: bulk -> warp 0 : the rank-16 update of step jp is done (warp 0 needs it before it touches row block jp+2)
//   barrier 7: bulk only, between its micro-panel and its update.
__global__ void __launch_bounds__(512, 1)
base_sweep4_kernel(double* __restrict__ S, long ld, double* __restrict__ Ldiag, double* __restrict__ Dinv,
                   double* __restrict__ logdet_part, int* __restrict__ info, int gcol0) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  double* T = reinterpret_cast<double*>(smem_raw);   // [128][BP]
  double* PdB = T + TILE * BP;
  double* WmB = PdB + 2 * 16 * MP;
  double* psh = WmB + 2 * 16 * MP;
  double* dinv = psh + 64;                           // psh: 2 x (16 values + 16 zeros)
  double* ldg = dinv + TILE;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  constexpr int BAR_A = 1, BAR_D = 3, BAR_BULK = 7;
  if (tid < 64) psh[tid] = 0.0;
  // Launched as a programmatic dependent of the kernel before it: this CTA is resident while that kernel still runs. The
  // time is used to pull the chain warp's code into the instruction cache: one column sweep on an identity block in the
  // (still unused) tile buffer -- measured in situ, the first micro-block of a launch costs 25 000-30 000 cycles against
  // 6 500 for the later ones (cold instruction cache: a one-CTA kernel lands on a fresh SM). griddepcontrol.wait then blocks
  // until the preceding kernel has completed and flushed.
  if (warp == 0) {
    for (int q = lane; q < 16 * 16; q += 32) T[(q >> 4) * BP + (q & 15)] = (q >> 4) == (q & 15) ? 1.0 : 0.0;
    __syncwarp();
    micro_diag_row(T, 0, PdB, WmB, psh, dinv, ldg, info, gcol0, lane);
  }
  __syncthreads();
  if (tid < 64) psh[tid] = 0.0;
  asm volatile("griddepcontrol.wait;" ::: "memory");
  // lower part of the tile -> shared memory, zeros above the diagonal (the inverse region starts from zero); 16-byte pieces
#pragma unroll 8
  for (int idx = tid; idx < TILE * TILE / 2; idx += 512) {
    const int row = (idx & 63) * 2, col = idx >> 6;
    double2 v = make_double2(0.0, 0.0);
    if (row + 1 >= col) v = *reinterpret_cast<const double2*>(S + row + (long)col * ld);
    if (row < col) v.x = 0.0;
    *reinterpret_cast<double2*>(T + col * BP + row) = v;
  }
  __syncthreads();
  if (warp == 0) {
    // ================= chain warp ======================================================================================
    for (int jp = 0; jp < 8; jp++) {
      const int c0 = jp * 16;
      if (jp > 0) {
        micro_update<2>(T, c0 - 16, jp - 1, jp, jp, 0, PdB + ((jp - 1) & 1) * 16 * MP, lane);   // T(jp, jp) -= P(jp, jp-1) P(jp, jp-1)^T
        __syncwarp();
      }
      micro_diag_row(T, c0, PdB + (jp & 1) * 16 * MP, WmB + (jp & 1) * 16 * MP, psh, dinv, ldg, info, gcol0, lane);
      if (jp > 0) named_sync(BAR_D + ((jp - 1) & 1), 512);               // update of step jp-1 done: row block jp+1 is current
      if (jp < 7) micro_panel_rows(T, c0, jp + 1, WmB + (jp & 1) * 16 * MP, lane);
      named_arrive(BAR_A + (jp & 1), 512);
    }
  } else {
    // ================= bulk warps 1..15 =================================================================================
    // the three warps that share the chain warp's SM sub-partition (warps 4, 8, 12) take no DMMA work: DMMA and DFMA share one
    // pipe per sub-partition, and the chain warp's dependent fp64 operations queued behind the bulk DMMAs (its micro-blocks
    // took 10 400 cycles beside the 34 update tiles of step 0 and 7 600 beside the 3 of step 6)
    const int bw = (warp & 3) ? (warp >> 2) * 3 + (warp & 3) - 1 : -1;     // 0..11, or -1 = idle
    for (int jp = 0; jp < 8; jp++) {
      const int c0 = jp * 16;
      const double* Pd = PdB + (jp & 1) * 16 * MP;
      const double* Wm = WmB + (jp & 1) * 16 * MP;
      named_sync(BAR_A + (jp & 1), 512);
      {   // micro-panel: the row blocks other than jp (diagonal) and jp+1 (done by the chain warp)
        const int nrows = jp < 7 ? 6 : 7;
        if (bw >= 0 && bw < nrows) {
          int rt = bw;
          if (rt >= jp) rt += (jp < 7 ? 2 : 1);
          micro_panel_rows(T, c0, rt, Wm, lane);
        }
      }
      named_sync(BAR_BULK, 480);
      if (jp == 7) break;
      int lin = 0;
      for (int ct = jp + 1; ct < 8; ct++) {
        const int nslot = jp + 1 + 8 - ct;                 // rows [0..jp] and [ct..7]
        for (int slot = 0; slot < nslot; slot++) {
          const int rt = slot <= jp ? slot : ct + slot - (jp + 1);
          if (rt == jp + 1 && ct == jp + 1) continue;      // the next diagonal micro-block belongs to the chain warp
          if (lin++ % 12 != bw) continue;
          micro_update<2>(T, c0, jp, rt, ct, 0, Pd, lane);
        }
      }
      named_arrive(BAR_D + (jp & 1), 512);
      base_out_block(T, dinv, ldg, jp, tid - 32, 480, S, ld, Ldiag, Dinv);
    }
  }
  __syncthreads();
  base_out_block(T, dinv, ldg, 7, tid, 512, S, ld, Ldiag, Dinv);
  if (tid < 32) {
    double s = 0.0;
    for (int j = tid; j < TILE; j += 32) s += log(ldg[j]);
    s = warp_sum(s);
    if (tid == 0) *logdet_part = 2.0 * s;
  }
}

int launch_base(double* S, long ld, double* Ldiag, double* Dinv, double* logdet_part, int* info, int gcol0,
                cudaStream_t st) {
  static bool ready = false;
  constexpr int smem = (TILE * BP + 4 * 16 * MP + 64 + 2 * TILE) * 8 + 16;
  if (!ready) {
    ready = true;
    GPX_CUDA(cudaFuncSetAttribute(base_sweep4_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  }
  // programmatic dependent launch: the CTA becomes resident as soon as every CTA of the kernel before it in the stream has
  // started (the fine GEMM issues griddepcontrol.launch_dependents first thing) and warms its instruction cache until that
  // kernel is done; after any other kernel the launch behaves like a plain one
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(1); cfg.blockDim = dim3(512); cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  GPX_CUDA(cudaLaunchKernelEx(&cfg, base_sweep4_kernel, S, ld, Ldiag, Dinv, logdet_part, info, gcol0));
  GPX_CUDA(cudaGetLastError());
  return 0;
}

// =================================================================================================================
// assemble: after the inner sweep of an nb x nb diagonal block (lower tiles = L, upper tiles incl. diagonal = U_kk),
// write  P[o.., :] = U_kk (block-upper part, zeros below) and Tm = U_kk^T = Linv_kk (nb x nb, column-major, ld = nb).
// =================================================================================================================
__global__ void assemble_kernel(const double* __restrict__ Sblk, long ld, int nb, double* __restrict__ Prows, long ldp,
                                double* __restrict__ Tm) {
  __shared__ double tile[32][33];
  const int bx = blockIdx.x * 32, by = blockIdx.y * 32;  // bx: column block, by: row block
  const int tx = threadIdx.x, ty = threadIdx.y;          // 32 x 8
  for (int k = ty; k < 32; k += 8) {
    const int row = by + tx, col = bx + k;
    const double x = (row / TILE <= col / TILE) ? Sblk[row + (long)col * ld] : 0.0;
    Prows[row + (long)col * ldp] = x;
    tile[k][tx] = x;   // tile[col_local][row_local]
  }
  __syncthreads();
  for (int k = ty; k < 32; k += 8) {
    // Tm(row' = col, col' = row): write contiguous in row' -> threads along col
    Tm[(bx + tx) + (long)(by + k) * nb] = tile[tx][k];
  }
}

int launch_assemble(const double* Sblk, long ld, int nb, double* Prows, long ldp, double* Tm, cudaStream_t st) {
  dim3 grid(nb / 32, nb / 32), block(32, 8);
  assemble_kernel<<<grid, block, 0, st>>>(Sblk, ld, nb, Prows, ldp, Tm);
  GPX_CUDA(cudaGetLastError());
  return 0;
}

// =================================================================================================================
// forward substitution t = L^-1 y carried along the sweep, block by block (the quadratic form y^T Ky^-1 y = |t|^2 of the
// log marginal likelihood, exact_gaussian_inference.py:60-62, then rests on the CHOLESKY part of the factorisation only):
//   fw_block : t_k = Linv_kk yres_k                    (Linv_kk = Tm, nb x nb lower triangular, column-major)
//   fw_panel : yres(rows below) -= L(rows below, k) t_k   (the panel rows below the diagonal block)
// =================================================================================================================
// Both are matrix-vector products with a column-major matrix (coalesced along the rows): 128 rows per CTA, the column range
// split over 8 thread groups (blockDim = 128 x 8) and reduced through shared memory in a fixed order. (The first version
// walked all 1024 columns in one dependent loop per thread: 0.37 ms per launch, latency-bound, on the critical side stream.)
constexpr int FW_KSPLIT = 8;
__global__ void __launch_bounds__(TILE * FW_KSPLIT) fw_block_kernel(const double* __restrict__ Tm, int nb,
                                                                     const double* __restrict__ yres, long ld, int P,
                                                                     double* __restrict__ t) {
  __shared__ double red[FW_KSPLIT][TILE];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int i = blockIdx.x * TILE + tx;   // row inside the block
  double acc[MAX_P];
#pragma unroll
  for (int q = 0; q < MAX_P; q++) acc[q] = 0.0;
  const int jend = (blockIdx.x + 1) * TILE < nb ? (blockIdx.x + 1) * TILE : nb;   // zeros right of the diagonal tile
  if (i < nb) {
#pragma unroll 4
    for (int j = ty; j < jend; j += FW_KSPLIT) {
      const double a = Tm[i + (long)j * nb];
#pragma unroll
      for (int q = 0; q < MAX_P; q++)
        if (q < P) acc[q] = fma(a, yres[(long)q * ld + j], acc[q]);
    }
  }
#pragma unroll
  for (int q = 0; q < MAX_P; q++) {
    if (q >= P) break;
    red[ty][tx] = acc[q];
    __syncthreads();
    if (ty == 0 && i < nb) {
      double s = 0.0;
#pragma unroll
      for (int g = 0; g < FW_KSPLIT; g++) s += red[g][tx];
      t[(long)q * ld + i] = s;
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(TILE * FW_KSPLIT) fw_panel_kernel(const double* __restrict__ Pb, long ldp, long rows, int nb,
                                                                     const double* __restrict__ t, long ld, int P,
                                                                     double* __restrict__ yres) {
  __shared__ double red[FW_KSPLIT][TILE];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const long r = (long)blockIdx.x * TILE + tx;
  double acc[MAX_P];
#pragma unroll
  for (int q = 0; q < MAX_P; q++) acc[q] = 0.0;
  if (r < rows) {
#pragma unroll 4
    for (int c = ty; c < nb; c += FW_KSPLIT) {
      const double a = Pb[r + (long)c * ldp];
#pragma unroll
      for (int q = 0; q < MAX_P; q++)
        if (q < P) acc[q] = fma(a, t[(long)q * ld + c], acc[q]);
    }
  }
#pragma unroll
  for (int q = 0; q < MAX_P; q++) {
    if (q >= P) break;
    red[ty][tx] = acc[q];
    __syncthreads();
    if (ty == 0 && r < rows) {
      double s = 0.0;
#pragma unroll
      for (int g = 0; g < FW_KSPLIT; g++) s += red[g][tx];
      yres[(long)q * ld + r] -= s;
    }
    __syncthreads();
  }
}

int launch_fw_block(const double* Tm, int nb, const double* yres, long ld, int P, double* t, cudaStream_t st) {
  fw_block_kernel<<<(unsigned)((nb + TILE - 1) / TILE), dim3(TILE, FW_KSPLIT), 0, st>>>(Tm, nb, yres, ld, P, t);
  GPX_CUDA(cudaGetLastError());
  return 0;
}

int launch_fw_panel(const double* Pb, long ldp, long rows, int nb, const double* t, long ld, int P, double* yres,
                    cudaStream_t st) {
  if (rows <= 0) return 0;
  fw_panel_kernel<<<(unsigned)((rows + TILE - 1) / TILE), dim3(TILE, FW_KSPLIT), 0, st>>>(Pb, ldp, rows, nb, t, ld, P, yres);
  GPX_CUDA(cudaGetLastError());
  return 0;
}

// =================================================================================================================
// triangular matrix-vector products with U = L^-T (upper, column-major, diagonal tiles included):
//   t = U^T y  (= L^-1 y)      one warp per column, coalesced column walk
//   a = U t    (= Ky^-1 y)     thread per row, k-range split over blockIdx.y, partials reduced in fixed order
// Replaces lapack.dpotrs (GPy/util/linalg.py:116-125; exact_gaussian_inference.py:60).
// =================================================================================================================
__global__ void __launch_bounds__(256) utv_kernel(const double* __restrict__ U, long ld, long n, int P,
                                                  const double* __restrict__ Y /*[P][ld]*/, double* __restrict__ T,
                                                  int own_G, int own_g, long own_cols, int local_cols) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long col = (long)blockIdx.x * 8 + warp;
  if (col >= n) return;
  if (own_G > 1 && ((col / own_cols) % own_G) != own_g) return;   // column block owned by another rank
  const long kend = (col / TILE + 1) * TILE;  // zeros below the diagonal inside the diagonal tile
  // memory-distributed layout: U holds only the owned column blocks, block kb at local slot kb / G
  const long lcol = (local_cols && own_G > 1) ? ((col / own_cols) / own_G) * own_cols + col % own_cols : col;
  const double* u = U + lcol * ld;
  double acc[MAX_P];
#pragma unroll
  for (int q = 0; q < MAX_P; q++) acc[q] = 0.0;
#pragma unroll 4
  for (long k = lane; k < kend; k += 32) {
    const double x = u[k];
#pragma unroll
    for (int q = 0; q < MAX_P; q++)
      if (q < P) acc[q] = fma(x, Y[(long)q * ld + k], acc[q]);
  }
#pragma unroll
  for (int q = 0; q < MAX_P; q++)
    if (q < P) {
      const double s = warp_sum(acc[q]);
      if (lane == 0) T[(long)q * ld + col] = s;
    }
}

__global__ void __launch_bounds__(TILE) uv_partial_kernel(const double* __restrict__ U, long ld, long n, int P,
                                                          const double* __restrict__ T, int ksplit,
                                                          double* __restrict__ part /*[ksplit][P][ld]*/) {
  const long row = (long)blockIdx.x * TILE + threadIdx.x;
  const long k0 = (long)blockIdx.x * TILE;   // U(row, k) = 0 for k < row's tile start (upper triangular)
  const long span = n - k0;
  const long chunk = ((span + ksplit - 1) / ksplit + 7) / 8 * 8;
  const long kb = k0 + (long)blockIdx.y * chunk;
  const long ke = kb + chunk < n ? kb + chunk : n;
  double acc[MAX_P];
#pragma unroll
  for (int q = 0; q < MAX_P; q++) acc[q] = 0.0;
#pragma unroll 8
  for (long k = kb; k < ke; k++) {
    const double x = U[row + k * ld];
#pragma unroll
    for (int q = 0; q < MAX_P; q++)
      if (q < P) acc[q] = fma(x, T[(long)q * ld + k], acc[q]);
  }
#pragma unroll
  for (int q = 0; q < MAX_P; q++)
    if (q < P) part[((long)blockIdx.y * P + q) * ld + row] = acc[q];
}

__global__ void uv_reduce_kernel(const double* __restrict__ part, long ld, int P, int ksplit, double* __restrict__ out) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ld * P) return;
  const long q = i / ld, row = i % ld;
  double s = 0.0;
  for (int k = 0; k < ksplit; k++) s += part[((long)k * P + q) * ld + row];
  out[q * ld + row] = s;
}

// general tall-skinny product out[q][row] = sum_c A[row + c*lda] * Y[q*ldy + c] (A: rows x ncols column-major, rows a multiple
// of 128): thread per row (coalesced along rows), the column range split over blockIdx.y, partials reduced in fixed order
__global__ void __launch_bounds__(TILE) row_dot_partial_kernel(const double* __restrict__ A, long lda, long ncols, int P,
                                                               const double* __restrict__ Y, long ldy, int nsplit, long ldo,
                                                               double* __restrict__ part /*[nsplit][P][ldo]*/) {
  const long row = (long)blockIdx.x * TILE + threadIdx.x;
  const long chunk = ((ncols + nsplit - 1) / nsplit + 7) / 8 * 8;
  const long cb = (long)blockIdx.y * chunk;
  const long ce = cb + chunk < ncols ? cb + chunk : ncols;
  double acc[MAX_P];
#pragma unroll
  for (int q = 0; q < MAX_P; q++) acc[q] = 0.0;
#pragma unroll 8
  for (long c = cb; c < ce; c++) {
    const double x = A[row + c * lda];
#pragma unroll
    for (int q = 0; q < MAX_P; q++)
      if (q < P) acc[q] = fma(x, Y[(long)q * ldy + c], acc[q]);
  }
#pragma unroll
  for (int q = 0; q < MAX_P; q++)
    if (q < P) part[((long)blockIdx.y * P + q) * ldo + row] = acc[q];
}
int launch_row_dot(const double* A, long lda, long rows_pad, long ncols, int P, const double* Y, long ldy, int nsplit,
                   double* part, double* out, cudaStream_t st) {
  dim3 grid((unsigned)(rows_pad / TILE), nsplit);
  row_dot_partial_kernel<<<grid, TILE, 0, st>>>(A, lda, ncols, P, Y, ldy, nsplit, rows_pad, part);
  GPX_CUDA(cudaGetLastError());
  uv_reduce_kernel<<<(unsigned)((rows_pad * P + 255) / 256), 256, 0, st>>>(part, rows_pad, P, nsplit, out);
  GPX_CUDA(cudaGetLastError());
  return 0;
}

// multi-GPU: a = U t restricted to the column blocks this rank owns; one partial per (row tile, column block)
__global__ void __launch_bounds__(TILE) uv_partial_blk_kernel(const double* __restrict__ U, long ld, long n, int P,
                                                              const double* __restrict__ T, long blk, int G, int g,
                                                              double* __restrict__ part /*[nblk][P][ld]*/, int local_cols,
                                                              long ldp) {
  const long row = (long)blockIdx.x * TILE + threadIdx.x;
  const long kb = blockIdx.y;
  double acc[MAX_P];
#pragma unroll
  for (int q = 0; q < MAX_P; q++) acc[q] = 0.0;
  const long k0 = kb * blk, k1 = k0 + blk;
  if ((kb % G) == g && k1 > (long)blockIdx.x * TILE) {   // U(row, k) = 0 for k before the row's tile start
    const long kbeg = k0 > (long)blockIdx.x * TILE ? k0 : (long)blockIdx.x * TILE;
    const long koff = local_cols ? (kb / G) * blk - k0 : 0;   // owned column block kb sits at local slot kb / G
#pragma unroll 8
    for (long k = kbeg; k < k1; k++) {
      const double x = U[row + (k + koff) * ld];
#pragma unroll
      for (int q = 0; q < MAX_P; q++)
        if (q < P) acc[q] = fma(x, T[(long)q * ldp + k], acc[q]);
    }
  }
#pragma unroll
  for (int q = 0; q < MAX_P; q++)
    if (q < P) part[((long)kb * P + q) * ldp + row] = acc[q];
}

int launch_uv_blk(const double* U, long ld, long n, int P, const double* T, long blk, int G, int g, double* part,
                  double* out, cudaStream_t st, int local_cols) {
  const int nblk = (int)(n / blk);
  dim3 grid((unsigned)(n / TILE), nblk);
  uv_partial_blk_kernel<<<grid, TILE, 0, st>>>(U, ld, n, P, T, blk, G, g, part, local_cols, ld);
  GPX_CUDA(cudaGetLastError());
  uv_reduce_kernel<<<(unsigned)((ld * P + 255) / 256), 256, 0, st>>>(part, ld, P, nblk, out);
  GPX_CUDA(cudaGetLastError());
  return 0;
}

// multi-GPU (memory-distributed layout): after the all-gather of the panel chunks every rank files its share of block
// column k: the rows BELOW the diagonal block that it owns go into its row-owned workspace SL (the L panel), and the rank
// that owns COLUMN block k stores all rows up to and including the diagonal block (= U(:, k), with U_kk from the owner's
// chunk) in its column-owned U storage SU, at local column slot k / G.
__global__ void copyback_kernel(double* __restrict__ SL, long ldl, double* __restrict__ SU, long ldu,
                                const double* __restrict__ Pbuf, long NB, int nbt, int G, int g, long npr, int k, int nt) {
  const int r = blockIdx.y;                 // row tile
  const int R = r / nbt;
  const bool below = R > k;
  const bool want = below ? ((R % G) == g) : ((k % G) == g);
  if (!want) return;
  const long pos = (long)(R % G) * npr + R / G;
  const double* src = Pbuf + pos * NB * NB + (long)(r % nbt) * TILE;
  double* dst = below ? SL + loc_tile(r, G, nbt) * TILE + (long)k * NB * ldl
                      : SU + (long)r * TILE + (long)(k / G) * NB * ldu;
  const long ldd = below ? ldl : ldu;
  const int m = threadIdx.x & (TILE - 1);
  for (long cc = (long)blockIdx.x * 2 + (threadIdx.x >> 7); cc < NB; cc += (long)gridDim.x * 2)
    dst[m + cc * ldd] = src[m + cc * NB];
}

int launch_copyback(double* SL, long ldl, double* SU, long ldu, const double* Pbuf, long NB, int G, int g, long npr, int k,
                    int nt, cudaStream_t st) {
  dim3 grid(8, nt);
  copyback_kernel<<<grid, 256, 0, st>>>(SL, ldl, SU, ldu, Pbuf, NB, (int)(NB / TILE), G, g, npr, k, nt);
  GPX_CUDA(cudaGetLastError());
  return 0;
}

// multi-GPU finalize: raw local sums only (reduced across ranks by the caller): raw[0..nred) gradient partial sums,
// raw[nred] = log-determinant of the diagonal tiles this rank factored, raw[nred+1] = |T|^2 (T is already global).
__global__ void __launch_bounds__(256) finalize_raw_kernel(FinalizeParams f) {
  __shared__ double sh[256];
  const int tid = threadIdx.x;
  const int nred = f.nl + 2;
  for (int t = 0; t < nred + 2; t++) {
    double s = 0.0;
    if (t < nred) {
      for (long i = tid; i < f.ntiles; i += 256) s += f.partials[i * nred + t];
    } else if (t == nred) {
      for (long i = tid; i < f.nt; i += 256) s += f.logdet_part[i];
    } else {
      for (int q = 0; q < f.P; q++)
        for (long i = tid; i < f.N; i += 256) { const double x = f.T[(long)q * f.ld + i]; s = fma(x, x, s); }
    }
    sh[tid] = s;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) { if (tid < o) sh[tid] += sh[tid + o]; __syncthreads(); }
    if (tid == 0) f.res[t] = sh[0];
    __syncthreads();
  }
}
int launch_finalize_raw(const FinalizeParams& f, cudaStream_t st) {
  finalize_raw_kernel<<<1, 256, 0, st>>>(f);
  GPX_CUDA(cudaGetLastError());
  return 0;
}

int launch_utv(const double* U, long ld, long n, int P, const double* Y, double* T, cudaStream_t st, int own_G,
               int own_g, long own_cols, int local_cols) {
  utv_kernel<<<(unsigned)((n + 7) / 8), 256, 0, st>>>(U, ld, n, P, Y, T, own_G, own_g, own_cols, local_cols);
  GPX_CUDA(cudaGetLastError());
  return 0;
}
int launch_uv(const double* U, long ld, long n, int P, const double* T, int ksplit, double* part, double* out,
              cudaStream_t st) {
  dim3 grid((unsigned)(n / TILE), ksplit);
  uv_partial_kernel<<<grid, TILE, 0, st>>>(U, ld, n, P, T, ksplit, part);
  GPX_CUDA(cudaGetLastError());
  uv_reduce_kernel<<<(unsigned)((ld * P + 255) / 256), 256, 0, st>>>(part, ld, P, ksplit, out);
  GPX_CUDA(cudaGetLastError());
  return 0;
}

// =================================================================================================================
// finalize: fixed-order reduction of the per-tile gradient partials, log-determinant and quadratic form;
// assembles the log marginal likelihood (exact_gaussian_inference.py:62) and the gradient vector
// [d/d variance, d/d lengthscale(s), d/d noise] (stationary.py:199,210,213; gaussian.py:78-79).
// res: [0]=lml, [1..nl+2]=gradient, [nl+3]=logdet, [nl+4]=y^T Ky^-1 y
// =================================================================================================================
__global__ void __launch_bounds__(256) finalize_kernel(FinalizeParams f) {
  __shared__ double sh[256];
  __shared__ double tot[MAX_D + 8];
  const int tid = threadIdx.x;
  const int nred = f.nl + 2;
  for (int t = 0; t < nred; t++) {
    double s = 0.0;
    for (long i = tid; i < f.ntiles; i += 256) s += f.partials[i * nred + t];
    sh[tid] = s;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) { if (tid < o) sh[tid] += sh[tid + o]; __syncthreads(); }
    if (tid == 0) tot[t] = sh[0];
    __syncthreads();
  }
  {  // logdet
    double s = 0.0;
    for (long i = tid; i < f.nt; i += 256) s += f.logdet_part[i];
    sh[tid] = s;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) { if (tid < o) sh[tid] += sh[tid + o]; __syncthreads(); }
    if (tid == 0) tot[nred] = sh[0];
    __syncthreads();
  }
  {  // y^T Ky^-1 y = |L^-1 y|^2
    double s = 0.0;
    for (int q = 0; q < f.P; q++)
      for (long i = tid; i < f.N; i += 256) { const double x = f.T[(long)q * f.ld + i]; s = fma(x, x, s); }
    sh[tid] = s;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) { if (tid < o) sh[tid] += sh[tid + o]; __syncthreads(); }
    if (tid == 0) tot[nred + 1] = sh[0];
    __syncthreads();
  }
  if (tid == 0) {
    const double logdet = tot[nred], quad = tot[nred + 1];
    const double log2pi = 1.8378770664093453;
    f.res[0] = 0.5 * (-(double)f.N * f.P * log2pi - (double)f.P * logdet - quad);
    f.res[1] = tot[0];
    if (f.kp.ard) {
      for (int q = 0; q < f.nl; q++) f.res[2 + q] = -tot[1 + q] / f.kp.ls[q];   // -(sum T (x-x')^2)/l^3, x unscaled
    } else {
      f.res[2] = -tot[1] / f.kp.ls[0];
    }
    f.res[2 + f.nl] = tot[nred - 1];
    f.res[3 + f.nl] = logdet;
    f.res[4 + f.nl] = quad;
  }
}

int launch_finalize(const FinalizeParams& f, cudaStream_t st) {
  finalize_kernel<<<1, 256, 0, st>>>(f);
  GPX_CUDA(cudaGetLastError());
  return 0;
}

// =================================================================================================================
// extraction of N x N results into a dense column-major N x N staging buffer (ld = N) for the device->host copy
// =================================================================================================================
__global__ void extract_kernel(int which, const double* __restrict__ S, long ld, const double* __restrict__ Ldiag,
                               const double* __restrict__ Kinv, const double* __restrict__ alpha, int P, long N,
                               double* __restrict__ out) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;  // row (contiguous in out)
  const long j = blockIdx.y;
  if (i >= N) return;
  const long ti = i / TILE, tj = j / TILE;
  double v = 0.0;
  if (which == GPX_GET_L) {
    if (ti > tj) v = S[i + j * ld];
    else if (ti == tj) v = Ldiag[ti * TILE * TILE + (i % TILE) + (j % TILE) * TILE];
  } else if (which == GPX_GET_LINV) {
    if (i >= j) v = S[j + i * ld];   // Linv(i,j) = U(j,i)
  } else {  // KINV / DLDK from the lower-tile K^-1 store
    const double kinv = (ti > tj || (ti == tj)) ? Kinv[i + j * ld] : Kinv[j + i * ld];
    if (which == GPX_GET_KINV) v = kinv;
    else {
      double aa = 0.0;
      for (int q = 0; q < P; q++) aa += alpha[(long)q * ld + i] * alpha[(long)q * ld + j];
      v = 0.5 * (aa - (double)P * kinv);
    }
  }
  out[i + j * N] = v;
}

// sharded factor: rows [R NB, (R+1) NB) of L out of the OWNER's row-owned workspace (local row offset lrow0) into a dense
// NB x ncols staging block (leading dimension NB): strict block-lower straight from the workspace, diagonal tiles from Ldiag
__global__ void extract_L_rows_kernel(const double* __restrict__ SL, long ldl, long lrow0, const double* __restrict__ Ldiag,
                                      long grow0, long NB, long ncols, double* __restrict__ out) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;   // row inside the block row
  const long j = blockIdx.y;                                     // global column
  if (i >= NB || j >= ncols) return;
  const long gi = grow0 + i, ti = gi / TILE, tj = j / TILE;
  double v = 0.0;
  if (ti > tj) v = SL[lrow0 + i + j * ldl];
  else if (ti == tj) v = Ldiag[ti * TILE * TILE + (gi % TILE) + (j % TILE) * TILE];
  out[i + j * NB] = v;
}

int launch_extract_L_rows(const double* SL, long ldl, long lrow0, const double* Ldiag, long grow0, long NB, long ncols,
                          double* out, cudaStream_t st) {
  dim3 grid((unsigned)((NB + 127) / 128), (unsigned)ncols);
  extract_L_rows_kernel<<<grid, 128, 0, st>>>(SL, ldl, lrow0, Ldiag, grow0, NB, ncols, out);
  GPX_CUDA(cudaGetLastError());
  return 0;
}

int launch_extract(int which, const double* S, long ld, const double* Ldiag, const double* Kinv, const double* alpha,
                   int P, long N, double* out, cudaStream_t st) {
  dim3 grid((unsigned)((N + 255) / 256), (unsigned)N);
  extract_kernel<<<grid, 256, 0, st>>>(which, S, ld, Ldiag, Kinv, alpha, P, N, out);
  GPX_CUDA(cudaGetLastError());
  return 0;
}

// out[p][c] = sum_r A[r + c*ld] * Y[p*ldy + r]  for a tall column-major A (rows x cols): one warp per column
__global__ void __launch_bounds__(256) col_dot_kernel(const double* __restrict__ A, long ld, long rows, long cols, int P,
                                                      const double* __restrict__ Y, long ldy, double* __restrict__ out,
                                                      long ldo) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long col = (long)blockIdx.x * 8 + warp;
  if (col >= cols) return;
  const double* a = A + col * ld;
  double acc[MAX_P];
#pragma unroll
  for (int q = 0; q < MAX_P; q++) acc[q] = 0.0;
#pragma unroll 4
  for (long r = lane; r < rows; r += 32) {
    const double x = a[r];
#pragma unroll
    for (int q = 0; q < MAX_P; q++)
      if (q < P) acc[q] = fma(x, Y[(long)q * ldy + r], acc[q]);
  }
#pragma unroll
  for (int q = 0; q < MAX_P; q++)
    if (q < P) {
      const double s = warp_sum(acc[q]);
      if (lane == 0) out[(long)q * ldo + col] = s;
    }
}
// out[c] = sum_r A[r + c*ld]^2 : squared column norms of a tall column-major matrix, one warp per column
__global__ void __launch_bounds__(256) col_sqnorm_kernel(const double* __restrict__ A, long ld, long rows, long cols,
                                                         double* __restrict__ out) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long col = (long)blockIdx.x * 8 + warp;
  if (col >= cols) return;
  const double* a = A + col * ld;
  double acc = 0.0;
#pragma unroll 4
  for (long r = lane; r < rows; r += 32) acc = fma(a[r], a[r], acc);
  acc = warp_sum(acc);
  if (lane == 0) out[col] = acc;
}
int launch_col_sqnorm(const double* A, long ld, long rows, long cols, double* out, cudaStream_t st) {
  col_sqnorm_kernel<<<(unsigned)((cols + 7) / 8), 256, 0, st>>>(A, ld, rows, cols, out);
  GPX_CUDA(cudaGetLastError());
  return 0;
}
int launch_col_dot(const double* A, long ld, long rows, long cols, int P, const double* Y, long ldy, double* out, long ldo,
                   cudaStream_t st) {
  col_dot_kernel<<<(unsigned)((cols + 7) / 8), 256, 0, st>>>(A, ld, rows, cols, P, Y, ldy, out, ldo);
  GPX_CUDA(cudaGetLastError());
  return 0;
}

// gpx_pdinv: dense symmetric A (N x N, ld = N) -> factor workspace (lower tiles + jitter on the diagonal, zero upper
// tiles, identity padding), and the mean of its diagonal / any non-positive diagonal entry for the jitchol rules.
__global__ void load_sym_kernel(const double* __restrict__ A, long lda, long N, double* __restrict__ S, long ld,
                                double jitter) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const long j = blockIdx.y;
  if (i >= ld) return;
  double v;
  if (i >= N || j >= N) v = (i == j) ? 1.0 : 0.0;
  else if (i / TILE < j / TILE) v = 0.0;
  else v = A[i + j * lda] + ((i == j) ? jitter : 0.0);
  S[i + j * ld] = v;
}
int launch_load_sym(const double* A, long lda, long N, double* S, long ld, double jitter, cudaStream_t st) {
  dim3 grid((unsigned)((ld + 255) / 256), (unsigned)ld);
  load_sym_kernel<<<grid, 256, 0, st>>>(A, lda, N, S, ld, jitter);
  GPX_CUDA(cudaGetLastError());
  return 0;
}

// transpose helpers for host layouts: in [rows][ld_in] (row index slow) -> out[cols... ] generic small kernels
__global__ void transpose_pad_kernel(const double* __restrict__ in, long n, int p, long ld, double* __restrict__ out) {
  // in: n x p row-major (host Y layout) -> out: [p][ld] (SoA), zero padded
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ld) return;
  for (int q = 0; q < p; q++) out[(long)q * ld + i] = i < n ? in[i * p + q] : 0.0;
}
int launch_transpose_pad(const double* in, long n, int p, long ld, double* out, cudaStream_t st) {
  transpose_pad_kernel<<<(unsigned)((ld + 255) / 256), 256, 0, st>>>(in, n, p, ld, out);
  GPX_CUDA(cudaGetLastError());
  return 0;
}
__global__ void untranspose_kernel(const double* __restrict__ in, long n, int p, long ld, double* __restrict__ out) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  for (int q = 0; q < p; q++) out[i * p + q] = in[(long)q * ld + i];
}
int launch_untranspose(const double* in, long n, int p, long ld, double* out, cudaStream_t st) {
  untranspose_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(in, n, p, ld, out);
  GPX_CUDA(cudaGetLastError());
  return 0;
}

// =================================================================================================================
// generic (unfused) gradient reduction for a caller-supplied dL_dK: Stationary.update_gradients_full
// (stationary.py:193-243) for K(X, X2), dL_dK row-major N x M. One CTA per (128 x 128) tile, thread-mapped index is
// the X2 point (contiguous in the row-major dL_dK), per-tile partials reduced by finalize-style fixed order on host.
// =================================================================================================================
// ONE pass over the tile: every element's K, dK/dr and dL_dK are formed once; the ARD lengthscale sums live in DREG
// registers per thread (the first version re-derived the element D+1 times, once per lengthscale).
template <int DREG>
__global__ void __launch_bounds__(256) grad_full_kernel(GradFullParams p) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int D = p.kp.D;
  double* sR = reinterpret_cast<double*>(smem_raw);   // [D][128] thread-mapped operand (X2 points, index j)
  double* sC = sR + (size_t)D * TILE;                 // [D][128] walked operand (X points, index i)
  double* sSr = sC + (size_t)D * TILE;
  double* sSc = sSr + TILE;
  double* sRed = sSc + TILE;                          // [8 warps][nred]
  const int jt = blockIdx.x, it = blockIdx.y;
  const int tid = threadIdx.x;
  for (int idx = tid; idx < D * TILE; idx += 256) {
    const int q = idx / TILE, m = idx % TILE;
    sR[idx] = p.x2T[(long)q * p.ld2 + (long)jt * TILE + m];
    sC[idx] = p.x1T[(long)q * p.ld1 + (long)it * TILE + m];
  }
  if (tid < TILE) { sSr[tid] = p.sq2[(long)jt * TILE + tid]; sSc[tid] = p.sq1[(long)it * TILE + tid]; }
  __syncthreads();
  const int jl = tid & (TILE - 1), half = tid >> 7;
  const long gj = (long)jt * TILE + jl;
  const bool ard = p.kp.ard != 0;
  const int nl = ard ? D : 1;
  const int nred = nl + 1;
  const int warp = tid >> 5, lane = tid & 31;
  double gvar = 0.0, giso = 0.0;
  double gq[DREG], xj[DREG];
#pragma unroll
  for (int q = 0; q < DREG; q++) { gq[q] = 0.0; xj[q] = q < D ? sR[q * TILE + jl] : 0.0; }
  const double sj = sSr[jl];
  const double variance = p.kp.variance, inv_ls = p.kp.inv_ls_iso;
  const long ldd = p.ldd > 0 ? p.ldd : p.M;
  const int kind = p.kp.kind;
  if (gj < p.M) {
    for (int ii = 0; ii < 64; ii++) {
      const int il = half * 64 + ii;
      const long gi = (long)it * TILE + il;
      if (gi >= p.N) break;
      double dot = 0.0;
#pragma unroll
      for (int q = 0; q < DREG; q++)
        if (q < D) dot = fma(xj[q], sC[q * TILE + il], dot);
      double r2 = sj + sSc[il] - 2.0 * dot;
      if (p.same && gi == gj) r2 = 0.0;
      r2 = fmax(r2, 0.0);
      const double rr = sqrt(r2) * inv_ls;
      double k, dk;
      k_dk_of_r_unit(kind, rr, k, dk);
      double dl = p.dL_dK[gi * ldd + gj];
      for (int cp = 0; cp < p.cP; cp++) dl = fma(p.ci[(long)cp * p.ldci + gi], p.cj[(long)cp * p.ldcj + gj], dl);
      const double G = variance * dk * dl;
      gvar = fma(k, dl, gvar);
      if (ard) {
        const double tmpv = (rr != 0.0) ? G / rr : 0.0;       // stationary.py:205,225-232: 1/r with 1/0 := 0
#pragma unroll
        for (int q = 0; q < DREG; q++)
          if (q < D) {
            const double df = xj[q] - sC[q * TILE + il];
            gq[q] = fma(tmpv, df * df, gq[q]);
          }
      } else {
        giso = fma(G, rr, giso);
      }
    }
  }
  gvar = warp_sum(gvar);
  if (lane == 0) sRed[warp * nred + 0] = gvar;
  if (ard) {
#pragma unroll
    for (int q = 0; q < DREG; q++)
      if (q < D) {
        const double sq_ = warp_sum(gq[q]);
        if (lane == 0) sRed[warp * nred + 1 + q] = sq_;
      }
  } else {
    giso = warp_sum(giso);
    if (lane == 0) sRed[warp * nred + 1] = giso;
  }
  __syncthreads();
  if (tid < nred) {
    double s = 0.0;
    for (int w = 0; w < 8; w++) s += sRed[w * nred + tid];
    p.partials[((long)blockIdx.y * gridDim.x + blockIdx.x) * nred + tid] = s;
  }
}

template <int DREG>
static int launch_grad_full_t(const GradFullParams& p, dim3 grid, size_t smem, cudaStream_t st) {
  static bool attr_set = false;
  if (!attr_set) {
    GPX_CUDA(cudaFuncSetAttribute(grad_full_kernel<DREG>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)((2 * MAX_D + 2) * TILE * 8 + 8 * (MAX_D + 2) * 8)));
    attr_set = true;
  }
  grad_full_kernel<DREG><<<grid, 256, smem, st>>>(p);
  GPX_CUDA(cudaGetLastError());
  return 0;
}

int launch_grad_full(const GradFullParams& p, int tiles_j, int tiles_i, cudaStream_t st) {
  const int D = p.kp.D;
  const size_t smem = (size_t)(2 * D + 2) * TILE * 8 + 8 * (MAX_D + 2) * 8;
  dim3 grid(tiles_j, tiles_i);
  if (D <= 8) return launch_grad_full_t<8>(p, grid, smem, st);
  if (D <= 16) return launch_grad_full_t<16>(p, grid, smem, st);
  if (D <= 32) return launch_grad_full_t<32>(p, grid, smem, st);
  return launch_grad_full_t<64>(p, grid, smem, st);
}

// =================================================================================================================
// gradient reductions from the stored K^-1 (same sums as the fused LAUUM epilogue of gpx_gemm.cu):
//    dL_dK = 1/2 (alpha alpha^T - P K^-1)  (exact_gaussian_inference.py:70), tr -> noise (:72, gaussian.py:78-79),
//    sum K o dL_dK / variance (stationary.py:199), ARD / iso lengthscale sums (:202-213, 225-243). One CTA per lower
//    128 x 128 tile; the thread-mapped index is the ROW (contiguous in the column-major K^-1), 64 columns per thread.
// =================================================================================================================
template <int DREG>
__global__ void __launch_bounds__(256) grad_kinv_kernel(GradKinvParams p) {
  extern __shared__ __align__(128) unsigned char gk_smem[];
  const int D = p.kp.D, P = p.P;
  double* sXc = reinterpret_cast<double*>(gk_smem);   // [D][128] column points
  double* sSc = sXc + (size_t)D * TILE;               // [128]
  double* sAc = sSc + TILE;                           // [P][128]
  double* sRed = sAc + (size_t)P * TILE;              // [8 warps][nred]
  // lower tiles only: blockIdx.x enumerates (r, c), c <= r
  const int csplit = p.csplit, tileidx = (int)blockIdx.x / csplit, sidx = (int)blockIdx.x % csplit;
  int r = (int)((sqrtf(8.f * (float)tileidx + 1.f) - 1.f) * 0.5f);
  while (r * (r + 1) / 2 > tileidx) --r;
  while ((r + 1) * (r + 2) / 2 <= tileidx) ++r;
  const int c = tileidx - r * (r + 1) / 2;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  for (int idx = tid; idx < D * TILE; idx += 256) sXc[idx] = p.XsT[(long)(idx / TILE) * p.ldx + (long)c * TILE + idx % TILE];
  for (int idx = tid; idx < P * TILE; idx += 256) sAc[idx] = p.alpha[(long)(idx / TILE) * p.ldx + (long)c * TILE + idx % TILE];
  if (tid < TILE) sSc[tid] = p.sq[(long)c * TILE + tid];
  __syncthreads();
  const int il = tid & (TILE - 1), half = tid >> 7;
  const long gi = (long)r * TILE + il;
  const bool ard = p.kp.ard != 0;
  const int nl = ard ? D : 1, nred = nl + 2;
  double xi[DREG], gq[DREG], ai[MAX_P];
#pragma unroll
  for (int q = 0; q < DREG; q++) { gq[q] = 0.0; xi[q] = q < D ? p.XsT[(long)q * p.ldx + gi] : 0.0; }
#pragma unroll
  for (int q = 0; q < MAX_P; q++) ai[q] = q < P ? p.alpha[(long)q * p.ldx + gi] : 0.0;
  const double si = p.sq[gi];
  const double w = (r > c) ? 2.0 : 1.0;               // strictly-lower tiles stand for their mirror image as well
  const double variance = p.kp.variance, inv_ls = p.kp.inv_ls_iso;
  const int kind = p.kp.kind;
  double gvar = 0.0, giso = 0.0, gnoise = 0.0;
  const double* kcol = p.Kinv + gi + ((long)c * TILE + half * 64) * p.ld;
  if (gi < p.N) {
    const int jj_beg = sidx * (64 / csplit);
    const int jj_end = (int)min((long)(jj_beg + 64 / csplit), p.N - (long)c * TILE - half * 64);   // columns beyond N are padding
    // two columns in flight per thread: one column is a single dependent chain (dot product -> exp -> reductions) and the
    // 16 warps an SM holds at 92 registers leave the fp64 pipe mostly idle (1.8 ms for the 134 M elements of N = 16384)
#pragma unroll 2
    for (int jj = jj_beg; jj < jj_end; jj++) {
      const int jl = half * 64 + jj;
      const long gj = (long)c * TILE + jl;
      const double kinv = kcol[(long)jj * p.ld];
      double dot = 0.0;
#pragma unroll
      for (int q = 0; q < DREG; q++)
        if (q < D) dot = fma(xi[q], sXc[q * TILE + jl], dot);
      double r2 = si + sSc[jl] - 2.0 * dot;
      if (gi == gj) r2 = 0.0;
      r2 = fmax(r2, 0.0);
      double aa = 0.0;
#pragma unroll
      for (int q = 0; q < MAX_P; q++)
        if (q < P) aa = fma(ai[q], sAc[q * TILE + jl], aa);
      const double dl = 0.5 * (aa - (double)P * kinv);
      if (gi == gj) {
        gnoise += dl;
        if (p.dnoise_out) p.dnoise_out[gi] = dl;
      }
      if (kind == GPX_RBF) {
        // dK/dr / r = -K for the RBF kernel (rbf.py:177-178 over stationary.py:205): neither the square root nor the division
        // of the general form is needed; at r = 0 the reference's 1/0 := 0 multiplies (x_i - x_j)^2 = 0 either way
        const double r2s = r2 * (inv_ls * inv_ls);
        const double k = exp(-0.5 * r2s);
        const double kd = w * k * dl;
        gvar += kd;
        const double tmpv = -variance * kd;
        if (ard) {
#pragma unroll
          for (int q = 0; q < DREG; q++)
            if (q < D) {
              const double df = xi[q] - sXc[q * TILE + jl];
              gq[q] = fma(tmpv, df * df, gq[q]);
            }
        } else {
          giso = fma(tmpv, r2s, giso);
        }
        continue;
      }
      const double rr = sqrt(r2) * inv_ls;
      double k, dk;
      k_dk_of_r_unit(kind, rr, k, dk);
      gvar = fma(w * k, dl, gvar);
      const double G = variance * dk * dl;
      if (ard) {
        const double tmpv = (rr != 0.0) ? w * G / rr : 0.0;     // stationary.py:205,225-232: 1/r with 1/0 := 0
#pragma unroll
        for (int q = 0; q < DREG; q++)
          if (q < D) {
            const double df = xi[q] - sXc[q * TILE + jl];
            gq[q] = fma(tmpv, df * df, gq[q]);
          }
      } else {
        giso = fma(w * G, rr, giso);
      }
    }
  }
  gvar = warp_sum(gvar);
  gnoise = warp_sum(gnoise);
  if (lane == 0) { sRed[warp * nred] = gvar; sRed[warp * nred + nred - 1] = gnoise; }
  if (ard) {
#pragma unroll
    for (int q = 0; q < DREG; q++)
      if (q < D) {
        const double s = warp_sum(gq[q]);
        if (lane == 0) sRed[warp * nred + 1 + q] = s;
      }
  } else {
    giso = warp_sum(giso);
    if (lane == 0) sRed[warp * nred + 1] = giso;
  }
  __syncthreads();
  if (tid < nred) {
    double s = 0.0;
#pragma unroll
    for (int wdx = 0; wdx < 8; wdx++) s += sRed[wdx * nred + tid];
    p.partials[(((long)r * p.nt + c) * csplit + sidx) * nred + tid] = s;
  }
}

int grad_kinv_csplit(int nt, int nred) {
  const int tiles = nt * (nt + 1) / 2;
  int cs = 1;
  while (cs < 8 && tiles * cs < 528 && (cs * 2) * nred <= MAX_D + 2) cs *= 2;   // ~4 waves of CTAs on 132 SMs; partials sized for MAX_D + 2 per tile
  return cs;
}

template <int DREG>
static int launch_grad_kinv_t(const GradKinvParams& p, unsigned grid, size_t smem, cudaStream_t st) {
  static bool attr_set = false;
  if (!attr_set) {
    GPX_CUDA(cudaFuncSetAttribute(grad_kinv_kernel<DREG>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)((MAX_D + 1 + MAX_P) * TILE * 8 + 8 * (MAX_D + 2) * 8)));
    attr_set = true;
  }
  grad_kinv_kernel<DREG><<<grid, 256, smem, st>>>(p);
  GPX_CUDA(cudaGetLastError());
  return 0;
}

int launch_grad_kinv(const GradKinvParams& p, cudaStream_t st) {
  const int D = p.kp.D;
  const size_t smem = (size_t)(D + 1 + p.P) * TILE * 8 + 8 * (MAX_D + 2) * 8;
  if (p.csplit != 1 && p.csplit != 2 && p.csplit != 4 && p.csplit != 8) { set_error("grad_kinv: csplit must be 1, 2, 4 or 8"); return -2; }
  const unsigned grid = (unsigned)(p.nt * (p.nt + 1) / 2 * p.csplit);
  if (D <= 8) return launch_grad_kinv_t<8>(p, grid, smem, st);
  if (D <= 16) return launch_grad_kinv_t<16>(p, grid, smem, st);
  if (D <= 32) return launch_grad_kinv_t<32>(p, grid, smem, st);
  return launch_grad_kinv_t<64>(p, grid, smem, st);
}


// =================================================================================================================
// gradients_X: Stationary.gradients_X (stationary.py:245-252, 348-366 -> stationary_utils.c:1-14 _grad_X):
//   grad[n,d] = sum_m tmp[n,m] (X[n,d] - X2[m,d]) / l_d^2,  tmp = (1/r) dK_dr dL_dK  (+ its transpose when X2 is None).
// One CTA = 128 rows n x one m-chunk; dL_dK (N x M row-major) tiles of 128 x 32 go through shared memory so that the
// global reads are coalesced along m; the points are used in scaled form (x/l), hence the final division by l_d only.
// Per-chunk partials are reduced in fixed order by gradx_reduce_kernel.
// =================================================================================================================
template <int DREG>
__global__ void __launch_bounds__(TILE) gradx_kernel(GradFullParams p, long mchunk, double* __restrict__ part) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  double (*sdl)[33] = reinterpret_cast<double (*)[33]>(smem_raw);                 // [128][33] dL_dK tile
  double* sx2 = reinterpret_cast<double*>(smem_raw) + TILE * 33;                    // [D][32] chunk of X2 points (scaled)
  double* ss2 = sx2 + (size_t)p.kp.D * 32;                // [32]
  const int D = p.kp.D;
  const int tid = threadIdx.x;
  const long n = (long)blockIdx.x * TILE + tid;
  const long m_beg = (long)blockIdx.y * mchunk;
  const long m_end = m_beg + mchunk < p.M ? m_beg + mchunk : p.M;
  double xn[DREG], acc[DREG];
#pragma unroll
  for (int q = 0; q < DREG; q++) { xn[q] = (q < D && n < p.N) ? p.x1T[(long)q * p.ld1 + n] : 0.0; acc[q] = 0.0; }
  const double sn = n < p.N ? p.sq1[n] : 0.0;
  const double variance = p.kp.variance, inv_ls = p.kp.inv_ls_iso;
  const long ldd = p.ldd > 0 ? p.ldd : p.M;
  for (long m0 = m_beg; m0 < m_end; m0 += 32) {
    __syncthreads();
    if (!p.transposed) {
      // dL_dK tile rows [n-tile], cols [m0, m0+32): warp w loads rows w, w+4, ... (32 doubles = 256 B per row)
      for (int rr = tid >> 5; rr < TILE; rr += TILE / 32) {
        const long gn = (long)blockIdx.x * TILE + rr, gm = m0 + (tid & 31);
        double dv = 0.0;
        if (gn < p.N && gm < m_end) {
          dv = p.dL_dK[gn * ldd + gm];
          for (int cp = 0; cp < p.cP; cp++) dv = fma(p.ci[(long)cp * p.ldci + gn], p.cj[(long)cp * p.ldcj + gm], dv);
        }
        sdl[rr][tid & 31] = dv;
      }
    } else {
      // transposed storage: element (n, m) at dL_dK[m*ldd + n] -> each thread fills its own row, coalesced along n
      for (int mm = 0; mm < 32; mm++) {
        const long gm = m0 + mm;
        double dv = 0.0;
        if (n < p.N && gm < m_end) {
          dv = p.dL_dK[gm * ldd + n];
          for (int cp = 0; cp < p.cP; cp++) dv = fma(p.ci[(long)cp * p.ldci + n], p.cj[(long)cp * p.ldcj + gm], dv);
        }
        sdl[tid][mm] = dv;
      }
    }
    for (int idx = tid; idx < D * 32; idx += TILE) {
      const int q = idx >> 5, mm = idx & 31;
      sx2[idx] = (m0 + mm < p.M) ? p.x2T[(long)q * p.ld2 + m0 + mm] : 0.0;
    }
    if (tid < 32) ss2[tid] = (m0 + tid < p.M) ? p.sq2[m0 + tid] : 0.0;
    __syncthreads();
    if (n < p.N) {
      const int mlim = (int)((m_end - m0) < 32 ? (m_end - m0) : 32);
      for (int mm = 0; mm < mlim; mm++) {
        const long gm = m0 + mm;
        double dot = 0.0;
#pragma unroll
        for (int q = 0; q < DREG; q++)
          if (q < D) dot = fma(xn[q], sx2[q * 32 + mm], dot);
        double r2 = sn + ss2[mm] - 2.0 * dot;
        if (p.same && n == gm) r2 = 0.0;
        r2 = fmax(r2, 0.0);
        const double rr = sqrt(r2) * inv_ls;
        double kk, dk;
        k_dk_of_r_unit(p.kp.kind, rr, kk, dk);
        double dl = sdl[tid][mm];
        if (p.same) dl += p.dL_dK[gm * ldd + n];            // tmp + tmp^T (stationary.py:343-345); coalesced along n
        const double t = (rr != 0.0) ? variance * dk * dl / rr : 0.0;
#pragma unroll
        for (int q = 0; q < DREG; q++)
          if (q < D) acc[q] = fma(t, xn[q] - sx2[q * 32 + mm], acc[q]);
      }
    }
  }
  if (n < p.N) {
#pragma unroll
    for (int q = 0; q < DREG; q++)
      if (q < D) part[((long)blockIdx.y * p.N + n) * D + q] = acc[q];
  }
}

__global__ void gradx_reduce_kernel(const double* __restrict__ part, long N, int D, int nchunk, KernParams kp,
                                    double* __restrict__ out) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * D) return;
  double s = 0.0;
  for (int c = 0; c < nchunk; c++) s += part[(long)c * N * D + i];
  const int q = (int)(i % D);
  // scaled differences: (x - x')/l summed -> divide once more by l (ARD: l_q; iso: the points are unscaled, r carries 1/l)
  out[i] = kp.ard ? s / kp.ls[q] : s / (kp.ls[0] * kp.ls[0]);
}

int launch_gradx(const GradFullParams& p, int nchunk, long mchunk, double* part, double* out, cudaStream_t st) {
  const int D = p.kp.D;
  const size_t smem = (size_t)(TILE * 33 + D * 32 + 32) * 8;
  dim3 grid((unsigned)((p.N + TILE - 1) / TILE), nchunk);
  static bool attr_set = false;
  if (!attr_set) {
    const int mx = (TILE * 33 + MAX_D * 32 + 32) * 8;
    GPX_CUDA(cudaFuncSetAttribute(gradx_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, mx));
    GPX_CUDA(cudaFuncSetAttribute(gradx_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, mx));
    GPX_CUDA(cudaFuncSetAttribute(gradx_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, mx));
    GPX_CUDA(cudaFuncSetAttribute(gradx_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, mx));
    attr_set = true;
  }
  if (D <= 8) gradx_kernel<8><<<grid, TILE, smem, st>>>(p, mchunk, part);
  else if (D <= 16) gradx_kernel<16><<<grid, TILE, smem, st>>>(p, mchunk, part);
  else if (D <= 32) gradx_kernel<32><<<grid, TILE, smem, st>>>(p, mchunk, part);
  else gradx_kernel<64><<<grid, TILE, smem, st>>>(p, mchunk, part);
  GPX_CUDA(cudaGetLastError());
  gradx_reduce_kernel<<<(unsigned)((p.N * D + 255) / 256), 256, 0, st>>>(part, p.N, D, nchunk, p.kp, out);
  GPX_CUDA(cudaGetLastError());
  return 0;
}

// =================================================================================================================
// roofline denominator: DMMA.16x8x4 issue rate of this device (8 independent accumulator chains per warp,
// 8 warps per CTA, 2 CTAs per SM), timed with CUDA events.
// =================================================================================================================
__global__ void dmma_rate_kernel(double* out, int iters) {
  double c[8][4];
#pragma unroll
  for (int i = 0; i < 8; i++) { c[i][0] = 0.0; c[i][1] = 0.0; c[i][2] = 0.0; c[i][3] = 0.0; }
  const double a = 1.0 + threadIdx.x * 1e-9, b = 1.0 - threadIdx.x * 1e-9;
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int i = 0; i < 8; i++) dmma1684(c[i][0], c[i][1], c[i][2], c[i][3], a, b, b);
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) s += (c[i][0] + c[i][1]) + (c[i][2] + c[i][3]);
  out[(long)blockIdx.x * blockDim.x + threadIdx.x] = s;
}

int measure_dmma_peak(cudaStream_t st, double* tflops) {
  int dev = 0, sms = 0;
  GPX_CUDA(cudaGetDevice(&dev));
  GPX_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int grid = sms * 2, threads = 256, iters = 20000;
  double* out = nullptr;
  GPX_CUDA(cudaMalloc(&out, (size_t)grid * threads * 8));
  cudaEvent_t e0, e1;
  GPX_CUDA(cudaEventCreate(&e0));
  GPX_CUDA(cudaEventCreate(&e1));
  double best = 0;
  for (int rep = 0; rep < 4; rep++) {
    GPX_CUDA(cudaEventRecord(e0, st));
    dmma_rate_kernel<<<grid, threads, 0, st>>>(out, iters);
    GPX_CUDA(cudaEventRecord(e1, st));
    GPX_CUDA(cudaEventSynchronize(e1));
    float ms = 0;
    GPX_CUDA(cudaEventElapsedTime(&ms, e0, e1));
    const double tf = (double)grid * (threads / 32) * iters * 8 * 1024.0 / ms * 1e-9;   // 2 x 16 x 8 x 4 flop per MMA
    if (rep > 0 && tf > best) best = tf;
  }
  cudaEventDestroy(e0); cudaEventDestroy(e1); cudaFree(out);
  *tflops = best;
  return 0;
}

}  // namespace gpx
