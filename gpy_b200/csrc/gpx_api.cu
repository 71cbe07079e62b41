// gpx_api.cu — C ABI (include/gpx.h) and host orchestration of the exact-GP evaluation on one H100.
//
// One evaluation (= one GP.parameters_changed(), GPy/core/gp.py:269-282):
//   prep_x -> kbuild (Ky into the workspace S) -> unified blocked factor-and-invert sweep (S: lower = L, upper = U = L^-T)
//   -> t = U^T y, alpha = U t -> LAUUM K^-1 = U U^T with the fused gradient epilogue -> finalize (LML + gradient).
// Nothing of size N^2 crosses PCIe unless gpx_get asks for it.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>

#include "gpx_common.cuh"
#include "gpx_kernels.cuh"
#include "gpx_ctx.cuh"
#include "gpx_fine.cuh"

namespace gpx {
static thread_local std::string g_err;
void set_error(const std::string& msg) { g_err = msg; }
}  // namespace gpx

using namespace gpx;

void gpx::free_data(gpx_ctx* c) {
  double** ptrs[] = {&c->dX, &c->dXsT, &c->dsq, &c->dY, &c->dT, &c->dAlpha, &c->dUvPart, &c->S, &c->Pbuf, &c->Tm,
                     &c->Ldiag, &c->Dinv, &c->logdet_part, &c->partials, &c->Kinv, &c->staging, &c->dTt};
  for (auto p : ptrs) {
    if (*p) cudaFree(*p);
    *p = nullptr;
  }
  c->staging_cap = 0;
  c->NBw = 0;
  c->have_eval = false;
  c->have_kinv = false;
  if (c->mpartials) cudaFree(c->mpartials);
  c->mpartials = nullptr;
  c->mpart_cap = 0;
  c->rows_cap = c->norm_cap = 0;
  oz_planes_free(c->ozp[0]);
  oz_planes_free(c->ozp[1]);
  oz_planes_free(c->ozpA);
  oz_planes_free(c->ozpB);
  if (c->oz_tiles) cudaFree(c->oz_tiles);
  c->oz_tiles = nullptr;
  for (double** mp : {&c->dYres, &c->dTfw}) { if (*mp) cudaFree(*mp); *mp = nullptr; }
  c->oz_steps.clear();
  c->oz_ready = false;
  c->oz_lists_ready = false;
}

int gpx::alloc_data(gpx_ctx* c, long NB) {
  const long Npad = c->Npad, nt = Npad / TILE;
  GPX_CUDA(cudaMalloc(&c->dX, (size_t)Npad * c->D * 8));
  GPX_CUDA(cudaMalloc(&c->dXsT, (size_t)Npad * c->D * 8));
  GPX_CUDA(cudaMalloc(&c->dsq, (size_t)Npad * 8));
  c->rows_cap = c->D; c->norm_cap = 1;
  const long Pc = c->P > MAX_P ? c->Ppad : c->P;   // the wide route keeps whole tiles of outputs
  GPX_CUDA(cudaMalloc(&c->dY, (size_t)Npad * Pc * 8));
  GPX_CUDA(cudaMalloc(&c->dT, (size_t)Npad * Pc * 8));
  GPX_CUDA(cudaMalloc(&c->dAlpha, (size_t)Npad * Pc * 8));
  if (c->P > MAX_P) GPX_CUDA(cudaMalloc(&c->dTt, (size_t)Npad * Pc * 8));
  GPX_CUDA(cudaMalloc(&c->Tm, (size_t)NB * NB * 8));
  GPX_CUDA(cudaMalloc(&c->Ldiag, (size_t)Npad * TILE * 8));
  GPX_CUDA(cudaMalloc(&c->Dinv, (size_t)Npad * TILE * 8));
  GPX_CUDA(cudaMalloc(&c->logdet_part, (size_t)nt * 8));
  GPX_CUDA(cudaMalloc(&c->partials, (size_t)nt * nt * (MAX_D + 2) * 8));
  return 0;
}

static int ensure_kinv(gpx_ctx* c) {
  if (!c->Kinv) GPX_CUDA(cudaMalloc(&c->Kinv, (size_t)c->Npad * c->Npad * 8));
  return 0;
}

// the outer block for a new workspace of Npad rows: option "nb", else env GPX_NB, else by size
static long choose_nb(const gpx_ctx* c) {
  if (c->NB > 0) return std::min<long>(c->NB, c->Npad);
  const char* e = getenv("GPX_NB");
  if (e && atol(e) >= TILE && atol(e) % TILE == 0) return std::min<long>(atol(e), c->Npad);
  // outer block by size (chosen with the chain schedule): 1024 above N = 8192, 512 from 2048, one block up to 512
  if (c->Npad > 8192) return 1024;
  if (c->Npad >= 2048) return 512;
  if (c->Npad <= 512) return c->Npad;
  return 256;
}
// the outer block of the allocated workspace, fixed until the next allocation
static long pick_nb(const gpx_ctx* c) { return c->NBw > 0 ? c->NBw : choose_nb(c); }

extern "C" {

const char* gpx_last_error(void) { return gpx::g_err.c_str(); }
const char* gpx_version(void) { return "gpx 0.2 (sm_90a: wgmma int8 digit-split GEMM + fp64 DMMA)"; }

int gpx_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return -1; }
  return n;
}

int gpx_create(int device, gpx_ctx** out) {
  if (!out) GPX_FAIL("null out pointer");
  int n = 0;
  GPX_CUDA(cudaGetDeviceCount(&n));
  if (device < 0 || device >= n) GPX_FAIL("no such CUDA device");
  GPX_CUDA(cudaSetDevice(device));
  gpx_ctx* c = new gpx_ctx();
  c->device = device;
  int prio_lo = 0, prio_hi = 0;
  GPX_CUDA(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));
  GPX_CUDA(cudaStreamCreateWithPriority(&c->st, cudaStreamNonBlocking, prio_lo));
  GPX_CUDA(cudaStreamCreateWithPriority(&c->st2, cudaStreamNonBlocking, prio_hi));
  // between the two: the big panel GEMM on st3 must not hold back the small launches of the diagonal-block chain on st2
  GPX_CUDA(cudaStreamCreateWithPriority(&c->st3, cudaStreamNonBlocking, prio_hi < prio_lo - 1 ? prio_hi + 1 : prio_hi));
  GPX_CUDA(cudaMalloc(&c->res, RES_DOUBLES * sizeof(double)));
  GPX_CUDA(cudaMalloc(&c->info, sizeof(int)));
  GPX_CUDA(cudaMallocHost(&c->h_res, RES_DOUBLES * sizeof(double)));
  GPX_CUDA(cudaMallocHost(&c->h_info, sizeof(int)));
  {   // keep freed temporaries of the stand-alone calls cached in the device's default pool
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
      uint64_t keep = 1ull << 30;   // up to 1 GiB stays cached; anything above goes back at the next synchronisation
      cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
    }
    cudaGetLastError();
  }
  GPX_CHECK(gemm_init());
  GPX_CHECK(oz_init());
  GPX_CHECK(fine_init());
  GPX_CUDA(cudaDeviceGetAttribute(&c->num_sms, cudaDevAttrMultiProcessorCount, device));
  *out = c;
  return 0;
}

int gpx_destroy(gpx_ctx* c) {
  if (!c) return 0;
  cudaSetDevice(c->device);
  cudaStreamSynchronize(c->st);
  dist_destroy(c);
  sparse_free(c);
  laplace_free(c);
  if (c->cJ) gpx_destroy(c->cJ);
  free_data(c);
  for (auto e : c->ev) cudaEventDestroy(e);
  for (auto e : c->sync_ev) cudaEventDestroy(e);
  if (c->st2) cudaStreamDestroy(c->st2);
  if (c->st3) cudaStreamDestroy(c->st3);
  if (c->ev_kfirst) cudaEventDestroy(c->ev_kfirst);
  if (c->res) cudaFree(c->res);
  if (c->dNoiseVec) cudaFree(c->dNoiseVec);
  if (c->dDnoise) cudaFree(c->dDnoise);
  if (c->info) cudaFree(c->info);
  if (c->h_res) cudaFreeHost(c->h_res);
  if (c->h_info) cudaFreeHost(c->h_info);
  cudaStreamDestroy(c->st);
  delete c;
  return 0;
}

int gpx_set_option(gpx_ctx* c, const char* name, int64_t value) {
  if (!c || !name) GPX_FAIL("null argument");
  if (!strcmp(name, "nb")) {
    if (value != 0 && (value < TILE || value % TILE)) GPX_FAIL("nb must be a multiple of 128");
    if (value != c->NB) {  // the panel buffers are sized by the block: force a re-allocation at the next gpx_set_data
      GPX_CUDA(cudaSetDevice(c->device));
      GPX_CUDA(cudaStreamSynchronize(c->st));
      free_data(c);
      c->Npad = 0;
    }
    c->NB = value;
    return 0;
  }
  if (!strcmp(name, "profile")) { c->profile = (int)value; return 0; }
  if (!strcmp(name, "epdtc_drift")) { c->epdtc_drift = value ? 1 : 0; return 0; }
  if (!strcmp(name, "sparse_wide")) { c->sparse_wide = value ? 1 : 0; return 0; }
  if (!strcmp(name, "ozaki")) { c->ozaki = value < 0 ? -1 : (value ? 1 : 0); return 0; }
  GPX_FAIL("unknown option");
}

int gpx_set_data(gpx_ctx* c, const double* X, int64_t N, int D, const double* Y, int P) {
  if (!c || !X || !Y) GPX_FAIL("null argument");
  if (N < 1) GPX_FAIL("N must be positive");
  if (D < 1 || D > MAX_D) GPX_FAIL("input dimension must be in [1, 64]");
  if (P < 1 || P > GPX_MAX_OUTPUTS) GPX_FAIL("number of output columns must be in [1, 1024]");
  if (P > MAX_P && c->dist) GPX_FAIL("more than 8 output columns are single-GPU");
  GPX_CUDA(cudaSetDevice(c->device));
  const long Npad = (N + TILE - 1) / TILE * TILE;
  if (c->dist) {
    GPX_CHECK(dist_set_data(c, N, D, P));
  } else if (Npad != c->Npad || D != c->D || P != c->P) {
    GPX_CUDA(cudaStreamSynchronize(c->st));
    free_data(c);
    c->Npad = Npad; c->D = D; c->P = P; c->Ppad = (P + TILE - 1) / TILE * TILE;
    const long NB = choose_nb(c);
    c->NBw = NB;
    GPX_CHECK(alloc_data(c, NB));
    if (P <= MAX_P) GPX_CUDA(cudaMalloc(&c->dUvPart, (size_t)KSPLIT * Npad * P * 8));
    GPX_CUDA(cudaMalloc(&c->S, (size_t)Npad * Npad * 8));
    GPX_CUDA(cudaMalloc(&c->Pbuf, (size_t)2 * Npad * NB * 8));   // double-buffered for the look-ahead
  }
  c->N = N;
  c->have_eval = false;
  c->have_kinv = false;
  laplace_release(c);
  // X: keep the caller's row-major layout on device; Y: SoA [P][Npad] zero padded (staged through dT)
  GPX_CUDA(cudaMemcpyAsync(c->dX, X, (size_t)N * D * 8, cudaMemcpyHostToDevice, c->st));
  if (P > MAX_P) {   // the wide route's GEMM operand: Y row-major with rows of Ppad, zero padded
    GPX_CUDA(cudaMemsetAsync(c->dY, 0, (size_t)c->Npad * c->Ppad * 8, c->st));
    GPX_CUDA(cudaMemcpy2DAsync(c->dY, (size_t)c->Ppad * 8, Y, (size_t)P * 8, (size_t)P * 8, N, cudaMemcpyHostToDevice, c->st));
  } else {
    GPX_CUDA(cudaMemcpyAsync(c->dT, Y, (size_t)N * P * 8, cudaMemcpyHostToDevice, c->st));
    GPX_CHECK(launch_transpose_pad(c->dT, N, P, c->Npad, c->dY, c->st));
    c->total_launches += 1;
  }
  GPX_CUDA(cudaStreamSynchronize(c->st));
  return 0;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------------------------
// event helpers for per-phase accounting on the launching stream
// ---------------------------------------------------------------------------------------------------------------
struct EvSpan { int a, b; int phase; double flops; };
enum { PH_KBUILD = 0, PH_SWEEP = 1, PH_UPDATE = 2, PH_LAUUM = 3, PH_SOLVE = 4, PH_TOTAL = 5 };

static int ev_get(gpx_ctx* c, size_t idx, cudaEvent_t* out) {
  while (c->ev.size() <= idx) {
    cudaEvent_t e;
    GPX_CUDA(cudaEventCreate(&e));
    c->ev.push_back(e);
  }
  *out = c->ev[idx];
  return 0;
}

struct Recorder {
  gpx_ctx* c;
  std::vector<EvSpan> spans;
  size_t next = 0;
  int begin(int phase, double flops = 0) {
    if (!c->profile && phase != PH_TOTAL) return -1;
    cudaEvent_t e;
    if (ev_get(c, next, &e)) return -1;
    cudaEventRecord(e, c->st);
    spans.push_back({(int)next, -1, phase, flops});
    next++;
    return (int)spans.size() - 1;
  }
  void end(int h) {
    if (h < 0) return;
    cudaEvent_t e;
    if (ev_get(c, next, &e)) return;
    cudaEventRecord(e, c->st);
    spans[h].b = (int)next;
    next++;
  }
};

// ---------------------------------------------------------------------------------------------------------------
// the unified blocked factor-and-invert sweep
// ---------------------------------------------------------------------------------------------------------------
GemmParams gpx::gemm_defaults() {
  GemmParams p;
  memset(&p, 0, sizeof(p));
  return p;
}

static int sync_event(gpx_ctx* c, size_t idx, cudaEvent_t* out) {
  while (c->sync_ev.size() <= idx) {
    cudaEvent_t e;
    GPX_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    c->sync_ev.push_back(e);
  }
  *out = c->sync_ev[idx];
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// Ozaki path: tile lists and buffers for (Npad, NB)
// ---------------------------------------------------------------------------------------------------------------
static bool oz_wanted(const gpx_ctx* c) {
  int on = c->ozaki;
  // off by default: on the H100 the fp64 DMMA.16x8x4 GEMMs are faster than the int8 digit split (140 vs 183 ms at
  // N = 16384, H100 80GB HBM3 at a 400 W power limit, profiles/h100_bench_*); option "ozaki" = 1 or GPX_OZAKI=1 selects it
  if (on < 0) { const char* e = getenv("GPX_OZAKI"); on = e ? atoi(e) : 0; }
  if (!on || c->P > MAX_P) return false;   // the int8 sweep's forward substitution carries at most 8 columns
  const long NB = pick_nb(c);
  // wherever there are at least two panels; a single-block matrix has no panel and stays on the DMMA path
  return c->Npad >= 2 * NB && NB % OZ_KC == 0;
}

static int oz_prepare(gpx_ctx* c) {
  const long Npad = c->Npad, NB = pick_nb(c);
  const int nt = (int)(Npad / TILE);
  if (nt >= 4096) GPX_FAIL("matrix too large for the tile encoding");
  if (!c->oz_ready) {
    GPX_CHECK(oz_planes_alloc(c->ozp[0], Npad, NB));
    GPX_CHECK(oz_planes_alloc(c->ozp[1], Npad, NB));
    GPX_CHECK(oz_planes_alloc(c->ozpA, Npad, NB));
    GPX_CHECK(oz_planes_alloc(c->ozpB, NB, NB));
    GPX_CUDA(cudaMalloc(&c->dYres, (size_t)MAX_P * Npad * 8));
    GPX_CUDA(cudaMalloc(&c->dTfw, (size_t)MAX_P * Npad * 8));
    c->oz_ready = true;
    c->oz_lists_ready = false;
  }
  if (c->oz_lists_ready) return 0;
  std::vector<uint32_t> tiles;
  oz_build_lists(Npad, NB, tiles, c->oz_steps);
  GPX_CUDA(cudaMalloc(&c->oz_tiles, tiles.size() * sizeof(uint32_t)));
  GPX_CUDA(cudaMemcpy(c->oz_tiles, tiles.data(), tiles.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
  c->oz_lists_ready = true;
  return 0;
}

// The DMMA sweep. Step k (block column k of width nb):
//   D(k)  inner sweep of the diagonal block (128 columns at a time) + assemble of U_kk / Linv_kk      [side stream]
//   Pn(k) panel GEMM  P = S(:,block k) Linv_kk^T -> Pbuf[k&1], copied back into S                     [side stream]
//   U1(k) trailing update restricted to the columns of block k+1                                        [main stream]
//   U2(k) trailing update of the remaining columns                                                      [main stream]
// Look-ahead: D(k+1), Pn(k+1) only need U1(k), so they run on the high-priority side stream while U2(k) keeps the
// machine busy; U1(k+1) waits for Pn(k+1). A single block is issued on the main stream.
static int run_sweep(gpx_ctx* c, Recorder& rec) {
  const long ld = c->Npad, Npad = c->Npad;
  const int nt = (int)(Npad / TILE);
  const long NB = pick_nb(c);
  const bool la = NB < Npad;
  cudaStream_t sm = c->st;
  cudaStream_t ss = la ? c->st2 : c->st;
  size_t evi = 0;
  cudaEvent_t ev;
  if (la) {  // side stream starts after everything queued so far on the main stream (K build)
    GPX_CHECK(sync_event(c, evi++, &ev));
    GPX_CUDA(cudaEventRecord(ev, sm));
    GPX_CUDA(cudaStreamWaitEvent(ss, ev, 0));
  }
  int kblk = 0;
  for (long o = 0; o < Npad; o += NB, kblk++) {
    const long nb = std::min(NB, Npad - o);
    const int nbt = (int)(nb / TILE), kt0 = (int)(o / TILE), kt1 = kt0 + nbt;
    double* Sblk = c->S + o + o * ld;
    double* Pb = c->Pbuf + (size_t)(kblk & 1) * Npad * NB;
    // ---- D(k): inner sweep of the nb x nb diagonal block ------------------------------------------------------
    GPX_CHECK(diag_block_sweep(c, Sblk, ld, nbt, kt0, ss));
    if (nbt == nt) break;  // single block: done
    // ---- Pn(k): P = S(:, block) * Linv_kk^T; rows of the diagonal block get U_kk ------------------------------
    GPX_CHECK(launch_assemble(Sblk, ld, (int)nb, Pb + o, Npad, c->Tm, ss));
    c->eval_launches++;
    {
      GemmParams pp = gemm_defaults();
      pp.mode = GEMM_PANEL;
      pp.A = c->S + o * ld; pp.lda = ld;
      pp.B = c->Tm; pp.ldb = nb;
      pp.C = Pb; pp.ldc = Npad;
      pp.K = (int)nb; pp.nt = nt; pp.skip0 = kt0; pp.skip1 = kt1; pp.tri = 1;
      GPX_CHECK(launch_gemm(pp, dim3(nbt, nt - nbt), ss));
      c->eval_launches++;
    }
    // the panel rows take their final place in S (U block column above, L panel below)
    if (o > 0)
      GPX_CUDA(cudaMemcpy2DAsync(c->S + o * ld, ld * 8, Pb, Npad * 8, (size_t)o * 8, nb, cudaMemcpyDeviceToDevice, ss));
    if (kt1 < nt)
      GPX_CUDA(cudaMemcpy2DAsync(c->S + o * ld + (o + nb), ld * 8, Pb + (o + nb), Npad * 8,
                                 (size_t)(Npad - o - nb) * 8, nb, cudaMemcpyDeviceToDevice, ss));
    if (la) {
      GPX_CHECK(sync_event(c, evi++, &ev));
      GPX_CUDA(cudaEventRecord(ev, ss));
      GPX_CUDA(cudaStreamWaitEvent(sm, ev, 0));
    }
    // ---- trailing update: S(r,c) -= P_r P_c^T for c >= kt1, r in [0,kt1) U [c,nt), split U1 | U2 ---------------
    if (kt1 < nt) {
      const int next_nbt = (int)(std::min(NB, Npad - (o + nb)) / TILE);
      for (int part = 0; part < 2; part++) {
        const int cbeg = part == 0 ? kt1 : kt1 + next_nbt;
        const int cend = part == 0 ? kt1 + next_nbt : nt;
        if (cbeg < cend) {
          GemmParams pu = gemm_defaults();
          pu.mode = GEMM_UPDATE;
          pu.A = Pb; pu.lda = Npad;
          pu.B = Pb; pu.ldb = Npad;
          pu.C = c->S; pu.ldc = ld;
          pu.K = (int)nb; pu.nt = nt; pu.c0 = cbeg; pu.ncols = cend - cbeg; pu.rlow = kt1;
          double tiles = 0;
          for (int cc = cbeg; cc < cend; cc++) tiles += kt1 + (nt - cc);
          const double flops = tiles * 2.0 * TILE * TILE * (double)nb;
          const int h = rec.begin(PH_UPDATE, flops);
          GPX_CHECK(launch_gemm(pu, dim3(1, 1), sm));
          rec.end(h);
          c->eval_launches++;
          c->stats.update_launches++;
        }
        if (part == 0 && la) {  // block column k+1 is final: the side stream may start D(k+1)
          GPX_CHECK(sync_event(c, evi++, &ev));
          GPX_CUDA(cudaEventRecord(ev, sm));
          GPX_CUDA(cudaStreamWaitEvent(ss, ev, 0));
        }
      }
    }
  }
  if (la) {  // join: the main stream continues after the last side-stream work
    GPX_CHECK(sync_event(c, evi++, &ev));
    GPX_CUDA(cudaEventRecord(ev, ss));
    GPX_CUDA(cudaStreamWaitEvent(sm, ev, 0));
  }
  return 0;
}

// The Ozaki sweep: trailing update and K^-1 = U U^T (accumulated into c->Kinv panel by panel, the panel's digit planes serve
// both) on the int8 tensor cores, the serial chain on its own stream. Per step k:
//   side stream  ss : D(k) -> assemble -> Pc(k): panel rows of block k+1 (fine DMMA tiles) -> U0d(k): diagonal block k+1 -= Pc Pc^T
//                     (fine DMMA tiles, fp64 operands straight from the panel buffer) -> D(k+1) ...
//   third stream s3 : Pr(k): the other panel rows -> digit split of the whole panel -> copy-back -> forward substitution
//   main stream  sm : U1(k): rest of block column k+1 -> U2(k): everything else + the K^-1 tiles          (Ozaki)
// Dependences across streams (events):  Pc(k), Pr(k) read block column k: after U1(k-1);  U0d(k) touches tiles that U2(k-1)
// updates: after U2(k-1);  split(k) after Pc(k);  U1(k) after split(k);  assemble(k+1) overwrites Tm and, with Pc/Pr(k+1), the
// panel buffer of step k-1: after the forward-substitution block of step k on s3 (s3 runs in order, so everything of step
// k-1 there is done as well);  the digit planes of step k are those of step k-2: split(k) is behind Pr(k), which waits for
// U1(k-1), which is behind U2(k-2) on the main stream.
// What the next diagonal block waits for is therefore D(k) + two small launches, and the main stream never waits for a
// diagonal block unless the trailing update is shorter than D. D(0) waits for `first_rows` (the first block row of Ky,
// recorded by this evaluation's build_Ky) if given, else for the whole build.
static int run_sweep_chain(gpx_ctx* c, Recorder& rec, cudaEvent_t first_rows) {
  const long ld = c->Npad, Npad = c->Npad;
  const int nt = (int)(Npad / TILE);
  const long NB = pick_nb(c);
  cudaStream_t sm = c->st, ss = c->st2, s3 = c->st3;
  size_t evi = 0;
  cudaEvent_t ev, ev_u1 = nullptr, ev_u2 = nullptr, ev_fw = nullptr;
  auto link = [&](cudaStream_t from, cudaStream_t to, cudaEvent_t* keep) -> int {   // `to` continues after what `from` holds now
    cudaEvent_t e;
    GPX_CHECK(sync_event(c, evi++, &e));
    GPX_CUDA(cudaEventRecord(e, from));
    if (to) GPX_CUDA(cudaStreamWaitEvent(to, e, 0));
    if (keep) *keep = e;
    return 0;
  };
  GPX_CHECK(link(sm, s3, &ev));                      // K build (all of it); it also stands in for "U1(-1)": block column 0 is final
  GPX_CUDA(cudaStreamWaitEvent(ss, first_rows ? first_rows : ev, 0));
  ev_u1 = ev;
  GPX_CUDA(cudaMemcpyAsync(c->dYres, c->dY, (size_t)c->P * Npad * 8, cudaMemcpyDeviceToDevice, s3));
  int kblk = 0;
  for (long o = 0; o < Npad; o += NB, kblk++) {
    const long nb = std::min(NB, Npad - o);
    const int nbt = (int)(nb / TILE), kt0 = (int)(o / TILE), kt1 = kt0 + nbt;
    const int next_nbt = kt1 < nt ? (int)(std::min(NB, Npad - (o + nb)) / TILE) : 0;
    double* Sblk = c->S + o + o * ld;
    double* Pb = c->Pbuf + (size_t)(kblk & 1) * Npad * NB;
    const gpx_ctx::OzStep& os = c->oz_steps[kblk];
    const OzPlanes& pl = c->ozp[kblk & 1];
    // ---- ss: D(k), assemble ------------------------------------------------------------------------------------------
    GPX_CHECK(diag_block_sweep(c, Sblk, ld, nbt, kt0, ss));
    if (ev_fw) GPX_CUDA(cudaStreamWaitEvent(ss, ev_fw, 0));
    GPX_CHECK(launch_assemble(Sblk, ld, (int)nb, Pb + o, Npad, c->Tm, ss));
    c->eval_launches++;
    cudaEvent_t ev_asm, ev_pc = nullptr;
    GPX_CHECK(link(ss, s3, &ev_asm));
    if (ev_u1) { GPX_CUDA(cudaStreamWaitEvent(ss, ev_u1, 0)); GPX_CUDA(cudaStreamWaitEvent(s3, ev_u1, 0)); }
    // ---- ss: Pc(k), U0d(k) -------------------------------------------------------------------------------------------
    if (next_nbt > 0) {
      FineParams pc{};
      pc.mode = FINE_PANEL;
      pc.A = c->S + o * ld; pc.lda = ld;
      pc.B = c->Tm; pc.ldb = nb;
      pc.C = Pb; pc.ldc = Npad;
      pc.K = (int)nb; pc.r0 = kt1; pc.nr = next_nbt; pc.nc = nbt; pc.tri = 1;
      GPX_CHECK(launch_fine(pc, ss));
      c->eval_launches++;
      GPX_CHECK(link(ss, nullptr, &ev_pc));
      if (ev_u2) GPX_CUDA(cudaStreamWaitEvent(ss, ev_u2, 0));
      FineParams pu{};
      pu.mode = FINE_UPDATE;
      pu.A = Pb; pu.lda = Npad;
      pu.B = Pb; pu.ldb = Npad;
      pu.C = c->S; pu.ldc = ld;
      pu.K = (int)nb; pu.nt = kt1 + next_nbt; pu.c0 = kt1; pu.ncols = next_nbt; pu.rlow = 0;
      GPX_CHECK(launch_fine(pu, ss));
      c->eval_launches++;
    }
    // ---- s3: Pr(k), split, copy-back, forward substitution --------------------------------------------------------------
    // (from N = 4096 on: five launches instead of one only pay once the panel GEMM is a visible share of the step)
    const bool oz_pan = os.pan_n > 0 && Npad >= 4096;
    if (oz_pan) {
      // the panel GEMM itself on the tensor cores: digit planes of block column k of the workspace (A) and of L_kk^-1 (B,
      // lower triangular: per-tile k-range), P = A B^T stored into the panel buffer. 8 digits for the Cholesky rows (they feed
      // the log-determinant), 7 for the rows above (finished block column of U: gradients only)
      GPX_CHECK(launch_oz_split(c->S + o * ld, ld, nb, c->ozpA, s3));
      GPX_CHECK(launch_oz_split(c->Tm, nb, nb, c->ozpB, s3));
      OzParams op;
      memset(&op, 0, sizeof(op));
      op.tiles = c->oz_tiles + os.pan_off; op.ntiles = os.pan_n; op.nkc = (int)(nb / OZ_KC);
      op.scale = c->ozpA.scale; op.scaleB = c->ozpB.scale; op.P = Pb; op.ldp = Npad; op.Pfinal = c->S + o * ld;
      op.S = c->S; op.lds = ld; op.Kinv = c->Kinv; op.ldk = ld;
      GPX_CHECK(launch_oz_gemm(c->ozpA, op, c->num_sms, s3, &c->ozpB));
      c->eval_launches += 5;
    } else if (nt - nbt - next_nbt > 0) {
      GemmParams pp = gemm_defaults();
      pp.mode = GEMM_PANEL;
      pp.A = c->S + o * ld; pp.lda = ld;
      pp.B = c->Tm; pp.ldb = nb;
      pp.C = Pb; pp.ldc = Npad;
      pp.K = (int)nb; pp.nt = nt; pp.skip0 = kt0; pp.skip1 = kt1 + next_nbt; pp.tri = 1;
      GPX_CHECK(launch_gemm(pp, dim3(nbt, nt - nbt - next_nbt), s3));
      c->eval_launches++;
    }
    if (ev_pc) GPX_CUDA(cudaStreamWaitEvent(s3, ev_pc, 0));
    GPX_CHECK(launch_oz_split(Pb, Npad, nb, c->ozp[kblk & 1], s3));
    c->eval_launches++;
    GPX_CHECK(link(s3, sm, nullptr));
    if (oz_pan) {   // the tensor-core panel GEMM stored its rows into the workspace itself: only the rows of block k+1 (Pc) are left
      if (next_nbt > 0)
        GPX_CUDA(cudaMemcpy2DAsync(c->S + o * ld + (o + nb), ld * 8, Pb + (o + nb), Npad * 8, (size_t)next_nbt * TILE * 8, nb,
                                   cudaMemcpyDeviceToDevice, s3));
    } else {
      if (o > 0)
        GPX_CUDA(cudaMemcpy2DAsync(c->S + o * ld, ld * 8, Pb, Npad * 8, (size_t)o * 8, nb, cudaMemcpyDeviceToDevice, s3));
      if (kt1 < nt)
        GPX_CUDA(cudaMemcpy2DAsync(c->S + o * ld + (o + nb), ld * 8, Pb + (o + nb), Npad * 8, (size_t)(Npad - o - nb) * 8, nb,
                                   cudaMemcpyDeviceToDevice, s3));
    }
    GPX_CHECK(launch_fw_block(c->Tm, (int)nb, c->dYres + o, Npad, c->P, c->dTfw + o, s3));
    c->eval_launches++;
    GPX_CHECK(link(s3, nullptr, &ev_fw));
    GPX_CHECK(launch_fw_panel(Pb + (o + nb), Npad, Npad - o - nb, (int)nb, c->dTfw + o, Npad, c->P, c->dYres + (o + nb), s3));
    c->eval_launches++;
    // ---- sm: U1(k), U2(k) on the int8 tensor cores ---------------------------------------------------------------------
    for (int part = 0; part < 2; part++) {
      const int off = part == 0 ? os.u1_off : os.u2_off;
      const int ntl = part == 0 ? os.u1_n : os.u2_n;
      if (ntl > 0) {
        OzParams op;
        memset(&op, 0, sizeof(op));
        op.tiles = c->oz_tiles + off; op.ntiles = ntl; op.nkc = (int)(nb / OZ_KC);
        op.scale = pl.scale; op.S = c->S; op.lds = ld; op.Kinv = c->Kinv; op.ldk = ld;
        const double flops = (double)ntl * 2.0 * OZ_TM * OZ_TN * (double)nb;
        const int nup = part == 0 ? os.u1_up : os.u2_up;
        c->stats.update_int8_ops += ((double)nup * (OZ_S_UP * (OZ_S_UP + 1) / 2) + (double)(ntl - nup) * (OZ_S * (OZ_S + 1) / 2)) *
                                    2.0 * OZ_TM * OZ_TN * (double)nb;
        const int h = rec.begin(PH_UPDATE, flops);
        GPX_CHECK(launch_oz_gemm(pl, op, c->num_sms, sm));
        rec.end(h);
        c->eval_launches++;
        c->stats.update_launches++;
      }
      GPX_CHECK(link(sm, nullptr, part == 0 ? &ev_u1 : &ev_u2));
    }
  }
  GPX_CHECK(link(ss, sm, nullptr));
  GPX_CHECK(link(s3, sm, nullptr));
  return 0;
}

// K^-1 = U U^T on gemm_lauum_kernel, in one of two modes:
//   fused (kinv_out == nullptr): the epilogue reduces dL_dK straight into the gradient partials of the single kernel kp
//     (and diag(dL_dK) for per-point noise); K^-1 is not stored
//   plain store: the lower tiles of K^-1 go to kinv_out (leading dimension Npad); no reductions
static int run_lauum(gpx_ctx* c, double* kinv_out, Recorder* rec, const KernParams* kp = nullptr) {
  const long ld = c->Npad;
  const int nt = (int)(c->Npad / TILE);
  GemmParams pl = gemm_defaults();
  pl.mode = GEMM_LAUUM;
  pl.A = c->S; pl.lda = ld;
  pl.B = c->S; pl.ldb = ld;
  pl.ldc = ld;
  pl.K = (int)c->Npad; pl.nt = nt;
  if (kinv_out) {
    pl.kinv_out = kinv_out;
    pl.kp.D = 1; pl.P = 1;   // the smallest epilogue staging: the plain store does not use it
  } else {
    const int nl = kp->ard ? c->D : 1;
    GPX_CUDA(cudaMemsetAsync(c->partials, 0, (size_t)nt * nt * (nl + 2) * 8, c->st));
    pl.XsT = c->dXsT; pl.sq = c->dsq; pl.alpha = c->dAlpha; pl.ldx = c->Npad;
    pl.N = (int)c->N; pl.P = c->P;
    pl.partials = c->partials;
    pl.dnoise_out = c->het ? c->dDnoise : nullptr;
    pl.kp = *kp;
  }
  double flops = 0;
  for (int r = 0; r < nt; r++) flops += (double)(r + 1) * 2.0 * TILE * TILE * (double)(c->Npad - (long)r * TILE);
  int h = rec ? rec->begin(PH_LAUUM, flops) : -1;
  GPX_CHECK(launch_gemm(pl, dim3(nt, nt), c->st));
  if (rec) rec->end(h);
  c->eval_launches++;
  return 0;
}

int gpx::sweep_workspace(gpx_ctx* c) {
  Recorder rec{c};
  return run_sweep(c, rec);
}

int gpx::lauum_store(gpx_ctx* c) {
  GPX_CHECK(ensure_kinv(c));
  return run_lauum(c, c->Kinv, nullptr);
}

// Ky = K(X, X) + noise + jitter (+ the per-point noise) of the context's kernel into the workspace, training points
// prepared first. On the int8 sweep a single kernel's first block row goes first and *first_rows is the event after it, so
// that the factorisation of the first diagonal block runs beside the rest of the build; otherwise *first_rows = nullptr.
static int build_Ky(gpx_ctx* c, double extra_jitter, bool single, bool int8, Recorder& rec, cudaEvent_t* first_rows) {
  const int nt = (int)(c->Npad / TILE);
  *first_rows = nullptr;
  if (c->mk.sumD > c->rows_cap || c->mk.nparts > c->norm_cap) {   // a composite that stacks more rows than D and 1
    for (double** mp : {&c->dXsT, &c->dsq}) { if (*mp) cudaFree(*mp); *mp = nullptr; }
    c->rows_cap = std::max(c->rows_cap, c->mk.sumD); c->norm_cap = std::max(c->norm_cap, c->mk.nparts);
    GPX_CUDA(cudaMalloc(&c->dXsT, (size_t)c->rows_cap * c->Npad * 8));
    GPX_CUDA(cudaMalloc(&c->dsq, (size_t)c->norm_cap * c->Npad * 8));
  }
  if (!single) {   // the parts' reduction partials, sized by the parts of this evaluation
    size_t need = 0;
    for (int q = 0; q < c->mk.nparts; q++) need += (size_t)nt * nt * part_nred(c->mk.part[q]);
    if (need > c->mpart_cap) {
      if (c->mpartials) cudaFree(c->mpartials);
      c->mpartials = nullptr;
      c->mpart_cap = 0;
      GPX_CUDA(cudaMalloc(&c->mpartials, need * 8));
      c->mpart_cap = need;
    }
  }
  const Points tr = train_points(c);
  GPX_CHECK(prep_points(c, c->mk, c->dX, c->N, c->D, c->Npad, tr.xT, tr.sq));
  c->eval_launches++;
  const KyDiag ky{((c->het ? 0.0 : c->noise) + c->jitter) + extra_jitter, c->het ? c->dNoiseVec : nullptr};
  const int h = rec.begin(PH_KBUILD);
  if (int8 && single) {
    const int nbt0 = (int)(pick_nb(c) / TILE);
    GPX_CHECK(build_K(c, c->mk, c->D, tr, tr, c->S, c->Npad, &ky, 0, nbt0));
    if (!c->ev_kfirst) GPX_CUDA(cudaEventCreateWithFlags(&c->ev_kfirst, cudaEventDisableTiming));
    GPX_CUDA(cudaEventRecord(c->ev_kfirst, c->st));
    *first_rows = c->ev_kfirst;
    GPX_CHECK(build_K(c, c->mk, c->D, tr, tr, c->S, c->Npad, &ky, nbt0, nt - nbt0));
    c->eval_launches++;
  } else {
    GPX_CHECK(build_K(c, c->mk, c->D, tr, tr, c->S, c->Npad, &ky));
  }
  rec.end(h);
  c->eval_launches++;
  return 0;
}

// the single-kernel kernels serve the evaluation (its reductions and result layout): a single stationary kernel and at most
// MAX_P output columns; above that a single kernel runs as its one-part description through the composite pass
static bool single_route(const gpx_ctx* c, KernParams* kp) { return as_single(c->mk, c->D, kp) && c->P <= MAX_P; }

// The wide route's solves on the DMMA GEMM (C = A B^T, column-major operands): T^T = Y^T (L^-1)^T with L^-1 lower (T into
// dTt, [Npad][Ppad]), then alpha = U T with U = L^-T extracted with zeros below the diagonal (full k range), and T once more
// as [Ppad][Npad] for the LML's quadratic term. L^-1 and U pass through c->Kinv, which the LAUUM overwrites afterwards.
static int solve_wide(gpx_ctx* c) {
  const long Npad = c->Npad, Ppad = c->Ppad;
  GPX_CHECK(extract_inverse_factor(c, 0, c->Kinv));
  GemmParams g = gemm_defaults();
  g.mode = GEMM_PANEL; g.plain = 1; g.tri = 1;
  g.A = c->dY; g.lda = Ppad; g.B = c->Kinv; g.ldb = Npad; g.C = c->dTt; g.ldc = Ppad;
  g.K = (int)Npad; g.nt = (int)(Ppad / TILE); g.ncols = (int)(Npad / TILE);
  GPX_CHECK(launch_gemm(g, dim3(1, 1), c->st));
  GPX_CHECK(extract_inverse_factor(c, 1, c->Kinv));
  g = gemm_defaults();
  g.mode = GEMM_PANEL; g.plain = 1; g.tri = 0;
  g.A = c->Kinv; g.lda = Npad; g.B = c->dTt; g.ldb = Ppad; g.C = c->dAlpha; g.ldc = Npad;
  g.K = (int)Npad; g.nt = (int)(Npad / TILE); g.ncols = (int)(Ppad / TILE);
  GPX_CHECK(launch_gemm(g, dim3(1, 1), c->st));
  GPX_CHECK(launch_transpose_pad(c->dTt, Npad, (int)Ppad, Npad, c->dT, c->st));
  c->eval_launches += 5;
  return 0;
}

// Where K^-1 of one evaluation comes from; the gradient reductions follow from it
enum KinvRoute {
  KINV_FUSED,   // DMMA sweep, single kernel, nt > 8: the fused LAUUM epilogue reduces it, nothing is stored
  KINV_FINE,    // DMMA sweep, single kernel, nt <= 8: fine LAUUM into c->Kinv
  KINV_PLAIN,   // DMMA sweep, composite kernel (any nt): plain LAUUM into c->Kinv
  KINV_SWEEP,   // int8 sweep: accumulated into c->Kinv panel by panel
};

// One evaluation on a single GPU (the sharded path is dist_exact_eval): build Ky -> sweep -> solve -> K^-1 per the route ->
// gradient reductions (fused, or from the stored K^-1: grad_kinv, grad_kinv_multi per part) -> finalize. The results land
// in c->h_res, the info flag in *c->h_info; *kinv_stored tells whether c->Kinv now holds K^-1.
static int eval_once(gpx_ctx* c, double extra_jitter, Recorder& rec, bool* kinv_stored) {
  cudaStream_t st = c->st;
  const long ld = c->Npad;
  const int nt = (int)(c->Npad / TILE);
  KernParams kp;
  const bool single = single_route(c, &kp), wide = c->P > MAX_P;
  const int ngrad = kern_ngrad(c->mk), nl = ngrad - 1;   // nl: the single kernel's lengthscales
  const bool int8 = oz_wanted(c);
  const KinvRoute route = int8 ? KINV_SWEEP : !single ? KINV_PLAIN : nt <= 8 ? KINV_FINE : KINV_FUSED;
  *kinv_stored = route != KINV_FUSED;
  GPX_CUDA(cudaMemsetAsync(c->info, 0, sizeof(int), st));
  cudaEvent_t first_rows;
  GPX_CHECK(build_Ky(c, extra_jitter, single, int8, rec, &first_rows));
  if (*kinv_stored) GPX_CHECK(ensure_kinv(c));
  if (int8) GPX_CHECK(oz_prepare(c));
  {
    const int h = rec.begin(PH_SWEEP);
    GPX_CHECK(int8 ? run_sweep_chain(c, rec, first_rows) : run_sweep(c, rec));
    rec.end(h);
  }
  // alpha = U (U^T y). On the int8 sweep t = L^-1 y = U^T y came along with the sweep (forward substitution): one mat-vec
  const double* T = int8 ? c->dTfw : c->dT;
  {
    const int h = rec.begin(PH_SOLVE);
    if (wide) {
      GPX_CHECK(solve_wide(c));
    } else {
      if (!int8) GPX_CHECK(launch_utv(c->S, ld, c->Npad, c->P, c->dY, c->dT, st));
      GPX_CHECK(launch_uv(c->S, ld, c->Npad, c->P, T, KSPLIT, c->dUvPart, c->dAlpha, st));
      c->eval_launches += int8 ? 2 : 3;
    }
    rec.end(h);
  }
  auto mpart = [&](int q) {
    size_t off = 0;
    for (int p = 0; p < q; p++) off += (size_t)nt * nt * part_nred(c->mk.part[p]);
    return c->mpartials + off;
  };
  long grad_tiles = (long)nt * nt;
  if (route == KINV_FUSED) {
    GPX_CHECK(run_lauum(c, nullptr, &rec, &kp));
  } else {
    if (route == KINV_PLAIN) GPX_CHECK(run_lauum(c, c->Kinv, &rec));
    const int h = rec.begin(PH_LAUUM, 0.0);
    if (route == KINV_FINE) {
      // the fused LAUUM kernel has one CTA per 128 x 128 tile -- 10 CTAs for N = 512, each walking up to 512 k alone (136 us
      // of a 0.48 ms evaluation); the fine LAUUM computes K^-1 = U U^T in 64 x 32 tiles (80 CTAs)
      FineParams fl{};
      fl.mode = FINE_LAUUM;
      fl.A = c->S; fl.lda = ld; fl.B = c->S; fl.ldb = ld; fl.C = c->Kinv; fl.ldc = ld; fl.K = (int)c->Npad; fl.nt = nt;
      GPX_CHECK(launch_fine(fl, st));
      c->eval_launches++;
    }
    if (!single) {   // one reduction pass per part
      for (int q = 0; q < c->mk.nparts; q++) {
        GPX_CUDA(cudaMemsetAsync(mpart(q), 0, (size_t)nt * nt * part_nred(c->mk.part[q]) * 8, st));
        GradKinvMultiParams gm;
        memset(&gm, 0, sizeof(gm));
        gm.Kinv = c->Kinv; gm.ld = ld; gm.XsT = c->dXsT; gm.sq = c->dsq; gm.ldx = c->Npad; gm.alpha = c->dAlpha;
        gm.N = c->N; gm.P = c->P; gm.nt = nt; gm.part = q; gm.want_noise = q == 0; gm.partials = mpart(q); gm.mk = c->mk;
        GPX_CHECK(launch_grad_kinv_multi(gm, st));
        c->eval_launches++;
      }
    } else {
      const int csplit = grad_kinv_csplit(nt, nl + 2);
      grad_tiles = (long)nt * nt * csplit;
      GPX_CUDA(cudaMemsetAsync(c->partials, 0, (size_t)grad_tiles * (nl + 2) * 8, st));
      GradKinvParams gk;
      memset(&gk, 0, sizeof(gk));
      gk.csplit = csplit;
      gk.Kinv = c->Kinv; gk.ld = ld;
      gk.XsT = c->dXsT; gk.sq = c->dsq; gk.alpha = c->dAlpha; gk.ldx = c->Npad;
      gk.N = c->N; gk.P = c->P; gk.nt = nt;
      gk.partials = c->partials;
      gk.dnoise_out = c->het ? c->dDnoise : nullptr;
      gk.kp = kp;
      GPX_CHECK(launch_grad_kinv(gk, st));
      c->eval_launches++;
    }
    rec.end(h);
  }
  if (!single) {
    FinalizeMultiParams fm;
    memset(&fm, 0, sizeof(fm));
    for (int q = 0; q < c->mk.nparts; q++) fm.partials[q] = mpart(q);
    fm.ntiles = (long)nt * nt; fm.logdet_part = c->logdet_part; fm.nt = nt;
    fm.T = T; fm.ld = ld; fm.N = c->N; fm.P = c->P; fm.mk = c->mk; fm.res = c->res;
    GPX_CHECK(launch_finalize_multi(fm, st));
  } else {
    FinalizeParams f;
    memset(&f, 0, sizeof(f));
    f.partials = c->partials; f.ntiles = grad_tiles; f.nl = nl;
    f.logdet_part = c->logdet_part; f.nt = nt;
    f.T = T; f.ld = ld; f.N = c->N; f.P = c->P;
    f.kp = kp;
    f.res = c->res;
    GPX_CHECK(launch_finalize(f, st));
  }
  c->eval_launches++;
  GPX_CUDA(cudaMemcpyAsync(c->h_res, c->res, (4 + ngrad) * sizeof(double), cudaMemcpyDeviceToHost, st));
  GPX_CUDA(cudaMemcpyAsync(c->h_info, c->info, sizeof(int), cudaMemcpyDeviceToHost, st));
  return 0;
}

// the parts of a composite kernel -> mk (validated), *kdiag_total = Kdiag of the composite kernel. Dfull: columns of X.
int gpx::fill_mk(MultiKern& mk, const gpx_kern_part* parts, int nparts, int Dfull, double* kdiag_total) {
  if (!parts || nparts < 1 || nparts > MAX_PARTS) GPX_FAIL("number of kernel parts must be in [1, 8]");
  memset(&mk, 0, sizeof(mk));
  mk.nparts = nparts;
  int off = 0;
  double total = 0.0, prod = 1.0;
  for (int p = 0; p < nparts; p++) {
    const gpx_kern_part& in = parts[p];
    PartDev& pd = mk.part[p];
    if (!is_known(in.kind)) GPX_FAIL("unknown kernel kind");
    if (!(in.variance > 0)) GPX_FAIL("variance must be positive");
    if (p > 0 && in.term < parts[p - 1].term) GPX_FAIL("kernel parts must be ordered by term");
    const bool stat = is_static(in.kind), periodic = in.kind == GPX_STDPERIODIC;
    if (!stat && (in.ndims < 1 || !in.dims || !in.lengthscale)) GPX_FAIL("a stationary part needs active dims and a lengthscale");
    if (periodic && !in.period) GPX_FAIL("a StdPeriodic part needs a period");
    if (in.kind == GPX_RATQUAD && !(in.power > 0)) GPX_FAIL("power must be positive");
    pd.kind = in.kind; pd.ard = (!stat && in.ard) ? 1 : 0; pd.ard_period = (periodic && in.ard_period) ? 1 : 0;
    pd.term = in.term; pd.D = stat ? 0 : in.ndims; pd.xoff = off;
    pd.variance = in.variance; pd.inv_ls_iso = 1.0; pd.power = in.kind == GPX_RATQUAD ? in.power : 0.0;
    if (off + pd.D > MAX_D) GPX_FAIL("the parts' active dims add up to more than 64");
    if (part_nacc(pd) > MAX_D) GPX_FAIL("a StdPeriodic part on more than 32 active dims: its gradient reduction does not fit");
    for (int q = 0; q < pd.D; q++) {
      if (in.dims[q] < 0 || in.dims[q] >= Dfull) GPX_FAIL("active dim outside the data");
      const double l = in.lengthscale[pd.ard ? q : 0];
      if (!(l > 0)) GPX_FAIL("lengthscale must be positive");
      mk.dims[off + q] = in.dims[q];
      mk.ls[off + q] = l;
      if (periodic) {
        const double T = in.period[pd.ard_period ? q : 0];
        if (!(T > 0)) GPX_FAIL("period must be positive");
        mk.period[off + q] = T;
      }
    }
    if (is_stationary(pd.kind) && !pd.ard) pd.inv_ls_iso = 1.0 / in.lengthscale[0];
    off += pd.D;
    if (p > 0 && in.term != parts[p - 1].term) { total += prod; prod = 1.0; }
    prod *= in.variance;      // every kind has Kdiag = variance (stationary.py:170-173, static.py:30-33,
                              // standard_periodic.py:134-138)
  }
  total += prod;
  mk.sumD = off;
  *kdiag_total = total;
  return 0;
}

// the checks every exact-evaluation entry makes before it reads its kernel (`kern`: the lengthscale or the parts, read
// against the data's D)
static int eval_args(const gpx_ctx* c, const void* kern, const double* lml, const double* grad, double noise) {
  if (!c || !kern || !lml || !grad) GPX_FAIL("null argument");
  if (!c->S) GPX_FAIL("gpx_set_data has not been called");
  if (!(noise >= 0)) GPX_FAIL("noise variance must be non-negative");
  return 0;
}

// One evaluation of the validated kernel k (Kdiag = kdiag), which becomes the context's kernel. noise_vec == nullptr:
// homoscedastic (`noise`); else N per-point variances (`noise` = their mean, used by the ladder)
static int exact_eval_impl(gpx_ctx* c, const MultiKern& k, double kdiag, double noise, const double* noise_vec, double jitter,
                           int max_tries, double* lml, double* grad, double* dnoise, double* jitter_used) {
  GPX_CUDA(cudaSetDevice(c->device));
  c->het = noise_vec != nullptr;
  if (c->het) {
    if (c->dist) GPX_FAIL("heteroscedastic evaluation is single-GPU");
    if (!dnoise) GPX_FAIL("null argument");
    if (c->het_cap < c->Npad) {
      if (c->dNoiseVec) cudaFree(c->dNoiseVec);
      if (c->dDnoise) cudaFree(c->dDnoise);
      c->dNoiseVec = c->dDnoise = nullptr;
      GPX_CUDA(cudaMalloc(&c->dNoiseVec, (size_t)c->Npad * 8));
      GPX_CUDA(cudaMalloc(&c->dDnoise, (size_t)c->Npad * 8));
      c->het_cap = c->Npad;
    }
    GPX_CUDA(cudaMemcpyAsync(c->dNoiseVec, noise_vec, (size_t)c->N * 8, cudaMemcpyHostToDevice, c->st));
  }
  c->mk = k;
  c->kdiag = kdiag;
  laplace_release(c);
  c->noise = noise;
  c->jitter = jitter;
  c->have_eval = false;
  c->have_kinv = false;
  memset(&c->stats, 0, sizeof(c->stats));
  c->eval_launches = 0;
  Recorder rec{c};
  const int htot = rec.begin(PH_TOTAL);
  double extra = 0.0;
  int tries = 0;
  int info = 0;
  bool kinv_stored = false;
  for (;;) {
    tries++;
    if (c->dist) {
      GPX_CHECK(dist_exact_eval(c, extra));
    } else {
      GPX_CHECK(eval_once(c, extra, rec, &kinv_stored));
      GPX_CUDA(cudaStreamSynchronize(c->st));
    }
    info = *c->h_info;
    if (info == 0) break;
    // jitchol ladder (GPy/util/linalg.py:61-75): the diagonal of Ky is variance + noise + jitter (> 0 here),
    // extra jitter = mean(diag) * 1e-6 * 10^k for k = 0 .. max_tries-1
    if (tries > max_tries) break;
    const double mean_diag = kdiag + (noise + jitter);
    extra = mean_diag * 1e-6 * pow(10.0, tries - 1);
    if (!std::isfinite(extra)) break;
  }
  rec.end(htot);
  GPX_CUDA(cudaStreamSynchronize(c->st));
  c->jitter_extra = extra;
  c->stats.tries = tries;
  // accounting
  for (auto& s : rec.spans) {
    if (s.b < 0) continue;
    float ms = 0;
    cudaEventElapsedTime(&ms, c->ev[s.a], c->ev[s.b]);
    switch (s.phase) {
      case PH_KBUILD: c->stats.kbuild_ms += ms; break;
      case PH_SWEEP: c->stats.sweep_ms += ms; break;
      case PH_UPDATE: c->stats.update_ms += ms; c->stats.update_flops += s.flops; break;
      case PH_LAUUM: c->stats.lauum_ms += ms; c->stats.lauum_flops += s.flops; break;
      case PH_SOLVE: c->stats.solve_ms += ms; break;
      case PH_TOTAL: c->stats.total_ms += ms; break;
    }
  }
  c->stats.kbuild_bytes = 8.0 * (double)c->N * c->N + 8.0 * (double)c->N * c->D;
  c->stats.launches = c->eval_launches;
  c->total_launches += c->eval_launches;
  if (jitter_used) *jitter_used = extra;
  if (info != 0) {
    gpx::set_error("not positive definite, even with jitter.");
    return info;
  }
  *lml = c->h_res[0];
  // the kernel's gradient block and d/d noise: [lml, block, noise, ..] from finalize_kernel, [lml, .., noise, block] from
  // finalize_multi_kernel
  const bool single = single_route(c, nullptr);
  const int n = kern_ngrad(c->mk);
  for (int q = 0; q < n; q++) grad[q] = c->h_res[(single ? 1 : 4) + q];
  grad[n] = c->h_res[single ? 1 + n : 3];
  if (c->het) {
    GPX_CUDA(cudaMemcpyAsync(dnoise, c->dDnoise, (size_t)c->N * 8, cudaMemcpyDeviceToHost, c->st));
    GPX_CUDA(cudaStreamSynchronize(c->st));
  }
  c->have_eval = true;
  c->have_kinv = kinv_stored;
  return 0;
}

extern "C" {

int gpx_exact_eval(gpx_ctx* c, int kind, int ard, double variance, const double* lengthscale, double noise,
                   double jitter, int max_tries, double* lml, double* grad, double* jitter_used) {
  GPX_CHECK(eval_args(c, lengthscale, lml, grad, noise));
  MultiKern mk;
  GPX_CHECK(fill_single(mk, kind, ard, c->D, variance, lengthscale));
  return exact_eval_impl(c, mk, variance, noise, nullptr, jitter, max_tries, lml, grad, nullptr, jitter_used);
}

int gpx_exact_eval_multi(gpx_ctx* c, const gpx_kern_part* parts, int nparts, double noise, double jitter, int max_tries,
                         double* lml, double* grad, double* jitter_used) {
  GPX_CHECK(eval_args(c, parts, lml, grad, noise));
  if (c->dist) GPX_FAIL("composite kernels are single-GPU");
  MultiKern mk;
  double kdiag;
  GPX_CHECK(fill_mk(mk, parts, nparts, c->D, &kdiag));
  return exact_eval_impl(c, mk, kdiag, noise, nullptr, jitter, max_tries, lml, grad, nullptr, jitter_used);
}

int gpx_exact_eval_het(gpx_ctx* c, int kind, int ard, double variance, const double* lengthscale,
                       const double* noise_variances, double jitter, int max_tries, double* lml, double* grad,
                       double* dnoise, double* jitter_used) {
  if (!c || !noise_variances) GPX_FAIL("null argument");
  if (c->P > MAX_P) GPX_FAIL("the heteroscedastic evaluation serves at most 8 output columns");
  double mean = 0.0;
  for (int64_t i = 0; i < c->N; i++) {
    if (!(noise_variances[i] >= 0)) GPX_FAIL("noise variances must be non-negative");
    mean += noise_variances[i];
  }
  mean /= (double)std::max<int64_t>(c->N, 1);
  GPX_CHECK(eval_args(c, lengthscale, lml, grad, mean));
  MultiKern mk;
  GPX_CHECK(fill_single(mk, kind, ard, c->D, variance, lengthscale));
  return exact_eval_impl(c, mk, variance, mean, noise_variances, jitter, max_tries, lml, grad, dnoise, jitter_used);
}

int gpx_measure_fp64_peak(gpx_ctx* c, double* tflops) {
  if (!c || !tflops) GPX_FAIL("null argument");
  GPX_CUDA(cudaSetDevice(c->device));
  return measure_dmma_peak(c->st, tflops);
}

int gpx_get_stats(gpx_ctx* c, gpx_stats* out) {
  if (!c || !out) GPX_FAIL("null argument");
  *out = c->stats;
  return 0;
}
int64_t gpx_total_launches(gpx_ctx* c) { return c ? c->total_launches : -1; }

static int ensure_staging(gpx_ctx* c) {
  const size_t need = (size_t)c->N * c->N * 8;
  if (c->staging && c->staging_cap < need) { cudaFree(c->staging); c->staging = nullptr; }
  if (!c->staging) { GPX_CUDA(cudaMalloc(&c->staging, need)); c->staging_cap = need; }
  return 0;
}

int gpx_get(gpx_ctx* c, int which, double* out) {
  if (!c || !out) GPX_FAIL("null argument");
  if (!c->have_eval) GPX_FAIL("no successful gpx_exact_eval to fetch results from");
  GPX_CUDA(cudaSetDevice(c->device));
  if (c->dist && which == GPX_GET_L) {   // collective: every rank calls it and receives the whole factor
    memset(out, 0, (size_t)c->N * c->N * 8);
    return dist_get_L(c, out);
  }
  if (c->lap_post && which == GPX_GET_DLDK)
    GPX_FAIL("the Laplace posterior keeps no dL_dK: its kernel gradient was reduced by gpx_laplace_finish");
  if (c->dist && which != GPX_GET_ALPHA)
    GPX_FAIL("sharded mode: alpha and L (collective) can be fetched; K^-1 / dL_dK / K stay distributed or are rebuilt by the caller");
  cudaStream_t st = c->st;
  const long N = c->N, ld = c->Npad;
  if (which == GPX_GET_ALPHA) {
    double* tmp = c->dUvPart;   // the wide route has no dUvPart: a temporary of N P doubles
    if (c->P > MAX_P) GPX_TMP_ALLOC(&tmp, (size_t)N * c->P * 8, st);
    GPX_CHECK(launch_untranspose(c->dAlpha, N, c->P, ld, tmp, st));
    c->total_launches++;
    GPX_CUDA(cudaMemcpyAsync(out, tmp, (size_t)N * c->P * 8, cudaMemcpyDeviceToHost, st));
    GPX_CUDA(cudaStreamSynchronize(st));
    if (tmp != c->dUvPart) GPX_TMP_FREE(tmp, st);
    return 0;
  }
  GPX_CHECK(ensure_staging(c));
  if (which == GPX_GET_K) {
    const Points tr = train_points(c);
    GPX_CHECK(build_K(c, c->mk, c->D, tr, tr, c->staging, N));
    c->total_launches++;
  } else if (which == GPX_GET_L || which == GPX_GET_LINV) {
    GPX_CHECK(launch_extract(which, c->S, ld, c->Ldiag, nullptr, nullptr, 0, N, c->staging, st));
    c->total_launches++;
  } else if (which == GPX_GET_KINV || which == GPX_GET_DLDK) {
    if (!c->have_kinv) {   // the fused route reduced K^-1 without storing it: the plain LAUUM stores the same tiles
      GPX_CHECK(ensure_kinv(c));
      const int64_t keep = c->eval_launches;
      GPX_CHECK(run_lauum(c, c->Kinv, nullptr));
      c->total_launches += c->eval_launches - keep;
      c->eval_launches = keep;
      c->have_kinv = true;
    }
    GPX_CHECK(launch_extract(which, c->S, ld, c->Ldiag, c->Kinv, c->dAlpha, c->P, N, c->staging, st));
    c->total_launches++;
  } else {
    GPX_FAIL("unknown gpx_get selector");
  }
  GPX_CUDA(cudaMemcpyAsync(out, c->staging, (size_t)N * N * 8, cudaMemcpyDeviceToHost, st));
  GPX_CUDA(cudaStreamSynchronize(st));
  return 0;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------------------------
// stand-alone kernel calls: K and update_gradients_full of a single kernel (kinds 0-3) or of one composite part (kinds 0-3,
// 6, 7), gradients_X of a single kernel. Each works with the kernel it is given; the context's own (that of its last
// evaluation) is left alone.
// ---------------------------------------------------------------------------------------------------------------
static std::mutex g_scratch_mu;
static gpx_ctx* g_scratch = nullptr;
static int scratch_ctx(gpx_ctx** out) {
  std::lock_guard<std::mutex> lk(g_scratch_mu);
  if (!g_scratch) {
    int dev = 0;
    cudaGetDevice(&dev);
    GPX_CHECK(gpx_create(dev, &g_scratch));
  }
  *out = g_scratch;
  return 0;
}

static int fill_one_part(const gpx_kern_part* part, int D, MultiKern& mk) {
  if (!part) GPX_FAIL("null argument");
  if (is_known(part->kind) && is_static(part->kind)) GPX_FAIL("White / Bias parts have no stand-alone entry");
  if (D < 1 || D > MAX_D) GPX_FAIL("input dimension must be in [1, 64]");
  gpx_kern_part one = *part;
  one.term = 0;
  double kdiag;
  return fill_mk(mk, &one, 1, D, &kdiag);
}

int gpx::fill_single(MultiKern& mk, int kind, int ard, int D, double variance, const double* ls) {
  if (kind < GPX_RBF || kind > GPX_MATERN52) GPX_FAIL("unknown kernel kind");
  if (D < 1 || D > MAX_D) GPX_FAIL("input dimension must be in [1, 64]");
  int dims[MAX_D];
  for (int q = 0; q < D; q++) dims[q] = q;
  gpx_kern_part part{};
  part.kind = kind; part.ard = ard; part.ndims = D; part.dims = dims; part.variance = variance; part.lengthscale = ls;
  double kdiag;
  return fill_mk(mk, &part, 1, D, &kdiag);
}

// K(X, X2) of k into out (N x M row-major; X2 == NULL: K(X, X)) on c (NULL: the scratch context), timed into c's kbuild_ms /
// kbuild_bytes. out == NULL: built on the device only (the result is dropped) -- used to measure the rectangular K(X, Z)
// build of the sparse model at full size.
static int kern_K(gpx_ctx* c, const MultiKern& k, const double* X, int64_t N, const double* X2, int64_t M, int D, double* out,
                  const char* what) {
  if (!c) GPX_CHECK(scratch_ctx(&c));
  GPX_CUDA(cudaSetDevice(c->device));
  PointSet p1, p2;
  GPX_CHECK(upload_points(c, k, X, N, D, p1));
  if (X2) GPX_CHECK(upload_points(c, k, X2, M, D, p2));
  PointSet& pj = X2 ? p2 : p1;   // thread-mapped operand = X2 points (contiguous index of the row-major output)
  double* dout = nullptr;
  GPX_TMP_ALLOC(&dout, (size_t)N * M * 8, c->st);
  cudaEvent_t e0, e1;
  int rc = ev_get(c, 0, &e0) || ev_get(c, 1, &e1);
  if (rc == 0) {
    cudaEventRecord(e0, c->st);
    rc = build_K(c, k, D, pj, p1, dout, M);
    cudaEventRecord(e1, c->st);
  }
  c->total_launches++;
  if (rc == 0 && out && cudaMemcpyAsync(out, dout, (size_t)N * M * 8, cudaMemcpyDeviceToHost, c->st) != cudaSuccess) rc = -1;
  if (cudaStreamSynchronize(c->st) != cudaSuccess) { gpx::set_error(std::string(what) + ": device failure"); rc = -1; }
  if (rc == 0) {
    cudaEventElapsedTime(&c->stats.kbuild_ms, e0, e1);
    c->stats.kbuild_bytes = 8.0 * (double)N * M + 8.0 * (double)(N + M) * D;
  }
  GPX_TMP_FREE(dout, c->st);
  return rc;
}

// update_gradients_full of k for a caller's dL_dK (N x M row-major) on c (NULL: the scratch context) -> k's gradient block
static int kern_grad_full(gpx_ctx* c, const MultiKern& k, const double* X, int64_t N, const double* X2, int64_t M, int D,
                          const double* dL_dK, double* grad) {
  if (!c) GPX_CHECK(scratch_ctx(&c));
  GPX_CUDA(cudaSetDevice(c->device));
  PointSet p1, p2;
  GPX_CHECK(upload_points(c, k, X, N, D, p1));
  if (X2) GPX_CHECK(upload_points(c, k, X2, M, D, p2));
  double *dd = nullptr, *dpart = nullptr;
  GPX_TMP_ALLOC(&dd, (size_t)N * M * 8, c->st);
  const GradFullParams gp = grad_params(k, D, p1, X2 ? p2 : p1, dd, 0);
  GPX_TMP_ALLOC(&dpart, grad_full_doubles(k, D, gp) * 8, c->st);
  GPX_CUDA(cudaMemcpyAsync(dd, dL_dK, (size_t)N * M * 8, cudaMemcpyHostToDevice, c->st));
  const int rc = grad_full_sum(c, k, D, gp, dpart, grad);
  GPX_TMP_FREE(dd, c->st); GPX_TMP_FREE(dpart, c->st);
  return rc;
}

extern "C" {

int gpx_kern_K(gpx_ctx* c, int kind, int ard, double variance, const double* lengthscale, const double* X, int64_t N,
               const double* X2, int64_t M, int D, double* out) {
  if (!X || !lengthscale) GPX_FAIL("null argument");
  MultiKern mk;
  GPX_CHECK(fill_single(mk, kind, ard, D, variance, lengthscale));
  if (!X2) M = N;
  if (N < 1 || M < 1) GPX_FAIL("empty input");
  return kern_K(c, mk, X, N, X2, M, D, out, "gpx_kern_K");
}

int gpx_kern_part_K(gpx_ctx* c, const gpx_kern_part* part, const double* X, int64_t N, const double* X2, int64_t M, int D,
                    double* out) {
  if (!X || !out) GPX_FAIL("null argument");
  MultiKern mk;
  GPX_CHECK(fill_one_part(part, D, mk));
  if (!X2) M = N;
  if (N < 1 || M < 1) GPX_FAIL("empty input");
  return kern_K(c, mk, X, N, X2, M, D, out, "gpx_kern_part_K");
}

int gpx_kern_Kdiag(int kind, double variance, int64_t N, double* out) {
  (void)kind;
  if (!out) GPX_FAIL("null argument");
  for (int64_t i = 0; i < N; i++) out[i] = variance;   // stationary.py:170-173
  return 0;
}

int gpx_kern_grad_full(gpx_ctx* c, int kind, int ard, double variance, const double* lengthscale, const double* X,
                       int64_t N, const double* X2, int64_t M, int D, const double* dL_dK, double* dvariance,
                       double* dlengthscale) {
  if (!X || !dL_dK || !lengthscale || !dvariance || !dlengthscale) GPX_FAIL("null argument");
  MultiKern mk;
  GPX_CHECK(fill_single(mk, kind, ard, D, variance, lengthscale));
  if (!X2) M = N;
  double g[MAX_D + 1];
  GPX_CHECK(kern_grad_full(c, mk, X, N, X2, M, D, dL_dK, g));
  *dvariance = g[0];
  for (int q = 0; q < (ard ? D : 1); q++) dlengthscale[q] = g[1 + q];
  return 0;
}

int gpx_kern_part_grad_full(gpx_ctx* c, const gpx_kern_part* part, const double* X, int64_t N, const double* X2, int64_t M,
                            int D, const double* dL_dK, double* grad) {
  if (!X || !dL_dK || !grad) GPX_FAIL("null argument");
  MultiKern mk;
  GPX_CHECK(fill_one_part(part, D, mk));
  if (!X2) M = N;
  if (N < 1 || M < 1) GPX_FAIL("empty input");
  return kern_grad_full(c, mk, X, N, X2, M, D, dL_dK, grad);
}

int gpx_kern_grad_X(gpx_ctx* c, int kind, int ard, double variance, const double* lengthscale, const double* X, int64_t N,
                    const double* X2, int64_t M, int D, const double* dL_dK, double* grad) {
  if (!X || !dL_dK || !lengthscale || !grad) GPX_FAIL("null argument");
  if (!c) GPX_CHECK(scratch_ctx(&c));
  GPX_CUDA(cudaSetDevice(c->device));
  MultiKern mk;
  GPX_CHECK(fill_single(mk, kind, ard, D, variance, lengthscale));
  if (!X2) M = N;
  PointSet p1, p2;
  GPX_CHECK(upload_points(c, mk, X, N, D, p1));
  if (X2) GPX_CHECK(upload_points(c, mk, X2, M, D, p2));
  double *dd = nullptr, *dpart = nullptr;
  GPX_TMP_ALLOC(&dd, (size_t)N * M * 8, c->st);
  const GradFullParams gp = grad_params(mk, D, p1, X2 ? p2 : p1, dd, 0);
  GPX_TMP_ALLOC(&dpart, grad_X_doubles(c, mk, gp, D) * 8, c->st);
  GPX_CUDA(cudaMemcpyAsync(dd, dL_dK, (size_t)N * M * 8, cudaMemcpyHostToDevice, c->st));
  const int rc = grad_X(c, mk, gp, D, dpart, grad);
  GPX_TMP_FREE(dd, c->st); GPX_TMP_FREE(dpart, c->st);
  return rc;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------------------------
// stand-alone pdinv / jitchol for a caller-supplied symmetric matrix (GPy/util/linalg.py:56-75,193-214)
// ---------------------------------------------------------------------------------------------------------------

// size the workspace of c for an N x N matrix: bind N dummy points (D = 1, P = 1) unless such a data set is bound already
static int bind_dummy_data(gpx_ctx* c, long N) {
  if (c->N == N && c->D == 1 && c->P == 1 && c->S) return 0;
  std::vector<double> zx((size_t)N, 0.0);
  return gpx_set_data(c, zx.data(), N, 1, zx.data(), 1);
}

// Factor-and-invert a dense symmetric matrix that already lives on the device (dA, leading dimension lda, order N) into
// the workspace of context c (lower = L, upper = U = L^-T), with jitchol's ladder (GPy/util/linalg.py:56-75):
// jitter0 is always added; on failure mean(diag)*1e-6*10^k. Returns 0, or the failing minor (>0) / an error (<0).
int gpx::factor_device(gpx_ctx* c, const double* dA, long lda, long N, double jitter0, int max_tries, double* logdet,
                       double* jitter_used) {
  GPX_CHECK(bind_dummy_data(c, N));
  c->have_eval = false;
  c->have_kinv = false;
  c->lap_begun = c->lap_post = false;
  cudaStream_t st = c->st;
  const long ld = c->Npad;
  Recorder rec{c};
  double extra = 0.0;
  int tries = 0, info = 0;
  const int64_t l0 = c->eval_launches;
  for (;;) {
    tries++;
    GPX_CUDA(cudaMemsetAsync(c->info, 0, sizeof(int), st));
    GPX_CHECK(launch_load_sym(dA, lda, N, c->S, ld, jitter0 + extra, st));
    c->eval_launches++;
    GPX_CHECK(run_sweep(c, rec));
    GPX_CUDA(cudaMemcpyAsync(c->h_info, c->info, sizeof(int), cudaMemcpyDeviceToHost, st));
    GPX_CUDA(cudaStreamSynchronize(st));
    info = *c->h_info;
    if (info == 0) break;
    // jitchol's rules need the diagonal: fetch it only on this (rare) path
    std::vector<double> dg((size_t)N);
    GPX_CUDA(cudaMemcpy2DAsync(dg.data(), 8, dA, (size_t)(lda + 1) * 8, 8, (size_t)N, cudaMemcpyDeviceToHost, st));
    GPX_CUDA(cudaStreamSynchronize(st));
    double dsum = 0.0;
    bool nonpos = false;
    for (long i = 0; i < N; i++) { dsum += dg[i] + jitter0; if (!(dg[i] + jitter0 > 0.0)) nonpos = true; }
    if (nonpos) { gpx::set_error("not pd: non-positive diagonal elements"); c->total_launches += c->eval_launches - l0; return info; }
    if (tries > max_tries) break;
    extra = dsum / (double)N * 1e-6 * pow(10.0, tries - 1);     // linalg.py:66-72
    if (!std::isfinite(extra)) break;
  }
  c->total_launches += c->eval_launches - l0;
  c->stats.tries = tries;
  if (jitter_used) *jitter_used = extra;
  if (info != 0) { gpx::set_error("not positive definite, even with jitter."); return info; }
  if (logdet) {   // 2 sum log diag(L) (linalg.py:208): per-tile partials summed in fixed order
    const int nt = (int)(ld / TILE);
    std::vector<double> parts(nt);
    GPX_CUDA(cudaMemcpyAsync(parts.data(), c->logdet_part, (size_t)nt * 8, cudaMemcpyDeviceToHost, st));
    GPX_CUDA(cudaStreamSynchronize(st));
    double s = 0.0;
    for (int i = 0; i < nt; i++) s += parts[i];
    *logdet = s;
  }
  return 0;
}

extern "C" {

int gpx_pdinv(gpx_ctx* c, const double* A, int64_t N, int max_tries, double* Ai, double* L, double* Li, double* logdet,
              double* jitter_used) {
  if (!A || !logdet) GPX_FAIL("null argument");
  if (!c) GPX_CHECK(scratch_ctx(&c));
  if (c->dist) GPX_FAIL("gpx_pdinv is single-GPU");
  if (N < 1) GPX_FAIL("N must be positive");
  GPX_CUDA(cudaSetDevice(c->device));
  GPX_CHECK(bind_dummy_data(c, N));
  cudaStream_t st = c->st;
  const long ld = c->Npad;
  GPX_CHECK(ensure_staging(c));
  GPX_CUDA(cudaMemcpyAsync(c->staging, A, (size_t)N * N * 8, cudaMemcpyHostToDevice, st));
  GPX_CHECK(ensure_kinv(c));
  // the factorisation reads the staged copy; the staging buffer is reused for the results afterwards
  double* dA = c->Kinv;   // park A in the K^-1 buffer (same size class) so that staging stays free for extraction
  GPX_CUDA(cudaMemcpyAsync(dA, c->staging, (size_t)N * N * 8, cudaMemcpyDeviceToDevice, st));
  {
    const int rc = factor_device(c, dA, N, N, 0.0, max_tries, logdet, jitter_used);
    if (rc != 0) return rc;
  }
  const int64_t l0 = c->eval_launches;
  if (Ai) {
    GPX_CHECK(run_lauum(c, c->Kinv, nullptr));
    GPX_CHECK(launch_extract(GPX_GET_KINV, c->S, ld, c->Ldiag, c->Kinv, nullptr, 0, N, c->staging, st));
    c->eval_launches++;
    GPX_CUDA(cudaMemcpyAsync(Ai, c->staging, (size_t)N * N * 8, cudaMemcpyDeviceToHost, st));
    GPX_CUDA(cudaStreamSynchronize(st));
  }
  if (L) {
    GPX_CHECK(launch_extract(GPX_GET_L, c->S, ld, c->Ldiag, nullptr, nullptr, 0, N, c->staging, st));
    c->eval_launches++;
    GPX_CUDA(cudaMemcpyAsync(L, c->staging, (size_t)N * N * 8, cudaMemcpyDeviceToHost, st));
    GPX_CUDA(cudaStreamSynchronize(st));
  }
  if (Li) {
    GPX_CHECK(launch_extract(GPX_GET_LINV, c->S, ld, c->Ldiag, nullptr, nullptr, 0, N, c->staging, st));
    c->eval_launches++;
    GPX_CUDA(cudaMemcpyAsync(Li, c->staging, (size_t)N * N * 8, cudaMemcpyDeviceToHost, st));
    GPX_CUDA(cudaStreamSynchronize(st));
  }
  c->total_launches += c->eval_launches - l0;
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// prediction with the factor of the last evaluation (posterior.py:273-302)
// ---------------------------------------------------------------------------------------------------------------
int gpx_predict(gpx_ctx* c, const double* Xnew, int64_t M, int full_cov, double* mu, double* var) {
  if (!c || !Xnew || !mu || !var) GPX_FAIL("null argument");
  if (!c->have_eval) GPX_FAIL("no successful gpx_exact_eval to predict from");
  if (M < 1) GPX_FAIL("empty Xnew");
  // sharded factor: U = L^-T is column-distributed (block columns dealt round-robin), X / Y / alpha are replicated.
  // Every rank forms K(X, Xnew) and the mean; the variance term sum_i (U^T Kx)_i^2 splits over the owned columns and is
  // all-reduced. All ranks must call gpx_predict together (it contains a collective).
  int drank = 0, dG = 1;
  dist_world(c, &drank, &dG);
  const long dNB = dist_block(c);
  GPX_CUDA(cudaSetDevice(c->device));
  cudaStream_t st = c->st;
  const long ld = c->Npad, N = c->N;
  PointSet pn;
  GPX_CHECK(upload_points(c, c->mk, Xnew, M, c->D, pn));
  // Kx as [M][ld] (each new point one zero-padded column of length ld): thread-mapped operand = training points
  double* Kx = nullptr; double* Tx = nullptr;
  GPX_TMP_ALLOC(&Kx, (size_t)pn.ld * ld * 8, c->st);
  GPX_TMP_ALLOC(&Tx, (size_t)pn.ld * ld * 8, c->st);
  GPX_CUDA(cudaMemsetAsync(Kx, 0, (size_t)pn.ld * ld * 8, st));
  if (dG > 1) GPX_CUDA(cudaMemsetAsync(Tx, 0, (size_t)pn.ld * ld * 8, st));   // columns of other ranks stay zero
  int rc = build_K(c, c->mk, c->D, train_points(c), pn, Kx, ld);
  c->total_launches++;
  // tmp = L^-1 Kx = U^T Kx, MAX_P columns per pass
  for (long m0 = 0; rc == 0 && m0 < M; m0 += MAX_P) {
    const int pc = (int)std::min<long>(MAX_P, M - m0);
    long ldu = ld;
    const double* Ud = c->dist ? dist_U(c, &ldu) : nullptr;   // sharded: the column-owned U storage (local column slots)
    rc = Ud ? launch_utv(Ud, ldu, c->Npad, pc, Kx + m0 * ld, Tx + m0 * ld, st, dG, drank, dNB, 1)
            : launch_utv(c->S, ld, c->Npad, pc, Kx + m0 * ld, Tx + m0 * ld, st);
    c->total_launches++;
  }
  if (!full_cov) {
    // diagonal variance: everything reduces on the device; only M (P + 1) doubles come back
    double* red = nullptr;   // [P][M] means, then [M] sums of squares
    if (rc == 0 && cudaMallocAsync((void**)&red, (size_t)(c->P + 1) * M * 8, c->st) != cudaSuccess) { gpx::set_error("gpx_predict: out of memory"); rc = -1; }
    for (int q0 = 0; rc == 0 && q0 < c->P; q0 += MAX_P) {   // mu = Kx^T alpha, MAX_P outputs per launch
      rc = launch_col_dot(Kx, ld, N, M, std::min(MAX_P, c->P - q0), c->dAlpha + (size_t)q0 * ld, ld, red + (size_t)q0 * M, M, st);
      c->total_launches++;
    }
    if (rc == 0) rc = launch_col_sqnorm(Tx, ld, c->Npad, M, red + (size_t)c->P * M, st);          // sum_i tmp_i^2
    if (rc == 0 && dG > 1) rc = dist_allreduce_sum(c, red + (size_t)c->P * M, (size_t)M, st);
    c->total_launches++;
    std::vector<double> h((size_t)(c->P + 1) * M);
    if (rc == 0 && cudaMemcpyAsync(h.data(), red, h.size() * 8, cudaMemcpyDeviceToHost, st) != cudaSuccess) rc = -1;
    if (cudaStreamSynchronize(st) != cudaSuccess) { gpx::set_error("gpx_predict: device failure"); rc = -1; }
    GPX_TMP_FREE(Kx, c->st); GPX_TMP_FREE(Tx, c->st);
    GPX_TMP_FREE(red, c->st);
    if (rc) return rc;
    for (long m = 0; m < M; m++) {
      for (int q = 0; q < c->P; q++) mu[m * c->P + q] = h[(size_t)q * M + m];
      var[m] = c->kdiag - h[(size_t)c->P * M + m];
    }
    return 0;
  }
  std::vector<double> hK, hT;
  if (rc == 0) {
    hK.resize((size_t)M * ld); hT.resize((size_t)M * ld);
    if (cudaMemcpyAsync(hK.data(), Kx, hK.size() * 8, cudaMemcpyDeviceToHost, st) != cudaSuccess) rc = -1;
    if (cudaMemcpyAsync(hT.data(), Tx, hT.size() * 8, cudaMemcpyDeviceToHost, st) != cudaSuccess) rc = -1;
  }
  std::vector<double> hA((size_t)c->P * ld);
  if (rc == 0 && cudaMemcpyAsync(hA.data(), c->dAlpha, hA.size() * 8, cudaMemcpyDeviceToHost, st) != cudaSuccess) rc = -1;
  if (cudaStreamSynchronize(st) != cudaSuccess) { gpx::set_error("gpx_predict: device failure"); rc = -1; }
  // sums over the training index of this rank's part, completed over the ranks below
  std::vector<double> ssq((size_t)M * M, 0.0);
  if (rc == 0) {
    for (long a = 0; a < M; a++)
      for (long b = 0; b < M; b++) {
        double s = 0.0;
        for (long i = 0; i < N; i++) s += hT[a * ld + i] * hT[b * ld + i];
        ssq[a + b * M] = s;
      }
    if (dG > 1) {
      if ((size_t)pn.ld * ld < ssq.size()) { gpx::set_error("gpx_predict: internal buffer size"); rc = -2; }
      if (rc == 0 && cudaMemcpyAsync(Kx, ssq.data(), ssq.size() * 8, cudaMemcpyHostToDevice, st) != cudaSuccess) rc = -1;
      if (rc == 0) rc = dist_allreduce_sum(c, Kx, ssq.size(), st);
      if (rc == 0 && cudaMemcpyAsync(ssq.data(), Kx, ssq.size() * 8, cudaMemcpyDeviceToHost, st) != cudaSuccess) rc = -1;
      if (cudaStreamSynchronize(st) != cudaSuccess) { gpx::set_error("gpx_predict: device failure"); rc = -1; }
    }
  }
  GPX_TMP_FREE(Kx, c->st); GPX_TMP_FREE(Tx, c->st);
  if (rc) return rc;
  // full covariance (small M): host epilogue mu = Kx^T alpha, var = Kxx - tmp^T tmp
  for (long m = 0; m < M; m++)
    for (int q = 0; q < c->P; q++) {
      double s = 0.0;
      for (long i = 0; i < N; i++) s += hK[m * ld + i] * hA[(size_t)q * ld + i];
      mu[m * c->P + q] = s;
    }
  // K(Xnew, Xnew), built on the device from the prepared new points
  std::vector<double> kxx((size_t)M * M);
  double* dk = nullptr;
  GPX_TMP_ALLOC(&dk, (size_t)M * M * 8, c->st);
  rc = build_K(c, c->mk, c->D, pn, pn, dk, M);
  c->total_launches++;
  if (rc == 0 && cudaMemcpyAsync(kxx.data(), dk, (size_t)M * M * 8, cudaMemcpyDeviceToHost, st) != cudaSuccess) rc = -1;
  if (cudaStreamSynchronize(st) != cudaSuccess) { gpx::set_error("gpx_predict: device failure"); rc = -1; }
  GPX_TMP_FREE(dk, c->st);
  if (rc) return rc;
  for (long a = 0; a < M; a++)
    for (long b = 0; b < M; b++) var[a + b * M] = kxx[a * M + b] - ssq[a + b * M];
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// predictive gradients with the factor of the last evaluation (gp.py:438-474): V = Ky^-1 K(X, Xnew) = U (U^T Kx), MAX_P
// test points per pass over U, then one fused Jacobian reduction; K^-1 is never formed
// ---------------------------------------------------------------------------------------------------------------
int gpx_predictive_gradients(gpx_ctx* c, const double* Xnew, int64_t M, double* dmu, double* dvar) {
  if (!c || !Xnew || !dmu || !dvar) GPX_FAIL("null argument");
  if (!c->have_eval) GPX_FAIL("no successful gpx_exact_eval to differentiate the prediction of");
  if (M < 1) GPX_FAIL("empty Xnew");
  if (c->dist) GPX_FAIL("predictive gradients are single-GPU");
  if (c->P > MAX_P) GPX_FAIL("predictive gradients serve at most 8 output columns");
  const MultiKern& k = c->mk;
  GPX_CHECK(pred_grad_check(k));
  GPX_CUDA(cudaSetDevice(c->device));
  cudaStream_t st = c->st;
  const long ld = c->Npad;
  PointSet pn;
  GPX_CHECK(upload_points(c, k, Xnew, M, c->D, pn));
  // Kx as [M][ld] (as in gpx_predict); T = U^T Kx, then V = U T over Kx in place (a pass reads only its own columns)
  double *Kx = nullptr, *Tx = nullptr, *uvp = nullptr;
  GPX_TMP_ALLOC(&Kx, (size_t)pn.ld * ld * 8, st);
  GPX_TMP_ALLOC(&Tx, (size_t)pn.ld * ld * 8, st);
  GPX_TMP_ALLOC(&uvp, (size_t)KSPLIT * MAX_P * ld * 8, st);
  int rc = 0;
  if (cudaMemsetAsync(Kx, 0, (size_t)pn.ld * ld * 8, st) != cudaSuccess) { gpx::set_error("gpx_predictive_gradients: device failure"); rc = -1; }
  if (rc == 0) rc = build_K(c, k, c->D, train_points(c), pn, Kx, ld);
  c->total_launches++;
  for (long m0 = 0; rc == 0 && m0 < M; m0 += MAX_P) {
    const int pc = (int)std::min<long>(MAX_P, M - m0);
    rc = launch_utv(c->S, ld, c->Npad, pc, Kx + m0 * ld, Tx + m0 * ld, st);
    if (rc == 0) rc = launch_uv(c->S, ld, c->Npad, pc, Tx + m0 * ld, KSPLIT, uvp, Kx + m0 * ld, st);
    c->total_launches += 3;
  }
  if (rc == 0) rc = pred_grad(c, k, pn, train_points(c), c->dAlpha, ld, c->P, Kx, ld, c->D, dmu, dvar);
  GPX_TMP_FREE(Kx, st); GPX_TMP_FREE(Tx, st); GPX_TMP_FREE(uvp, st);
  return rc;
}

// ---------------------------------------------------------------------------------------------------------------
// the input gradient of the last exact evaluation (GPy/models/gplvm.py:47-49): kern.gradients_X(dL_dK, X, None) from the
// stored K^-1 and alpha. The fused route did not store K^-1: the plain LAUUM stores it first, as gpx_get(KINV) does.
// ---------------------------------------------------------------------------------------------------------------
int gpx_exact_grad_X(gpx_ctx* c, double* dX) {
  if (!c || !dX) GPX_FAIL("null argument");
  if (!c->have_eval) GPX_FAIL("no successful exact evaluation to differentiate");
  if (c->lap_post) GPX_FAIL("a Laplace / EP posterior: its dL_dK is not 1/2 (alpha alpha^T - P K^-1)");
  if (c->het) GPX_FAIL("the input gradient of a heteroscedastic evaluation is not served");
  if (c->dist) GPX_FAIL("the input gradient of the exact evaluation is single-GPU");
  GPX_CHECK(pred_grad_check(c->mk));
  GPX_CUDA(cudaSetDevice(c->device));
  if (!c->have_kinv) {
    GPX_CHECK(ensure_kinv(c));
    const int64_t keep = c->eval_launches;
    GPX_CHECK(run_lauum(c, c->Kinv, nullptr));
    c->total_launches += c->eval_launches - keep;
    c->eval_launches = keep;
    c->have_kinv = true;
  }
  return exact_grad_X(c, dX);
}

}  // extern "C"
