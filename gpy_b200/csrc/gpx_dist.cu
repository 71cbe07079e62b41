// gpx_dist.cu — multi-GPU exact-GP evaluation: one process per GPU, NCCL over NVLink/NVSwitch.
//
// The reference has NO multi-device strategy for the exact path (SURVEY.md §2c: its only collectives are mpi4py sums for
// the sparse model, GPy/inference/latent_function_inference/var_dtc_parallel.py:127-130), so this is new design:
//
//   * block rows of width NB are dealt block-cyclically: rank (R mod G) owns block row R of the unified workspace S
//     (its Cholesky rows AND its rows of the inverse region). X, Y are replicated (<= a few MiB).
//   * step k of the sweep: the owner factors-and-inverts the diagonal block and BROADCASTS L_kk^-1 (NB x NB);
//     every rank forms the panel rows it owns, P_R = S(R,k) L_kk^-T, into a chunked panel buffer whose chunks are
//     ordered by owner, so ONE in-place ncclAllGather hands every rank the whole panel; every rank then updates the
//     tiles of its own block rows,  S(r,c) -= P_r P_c^T.
//   * the panel rows above the diagonal block are exactly block column k of U = L^-T, and every rank sees them in the
//     all-gather: the rank that owns COLUMN block k keeps them. U thereby ends up column-distributed at no extra cost,
//     which is what K^-1 = U U^T needs: each rank runs the LAUUM over the k-range of its own column blocks and reduces its
//     gradient partials locally — K^-1 is never communicated; nl+2 scalars (+ logdet) are all-reduced.
//   * alpha = U (U^T y): each rank contributes the entries / partial sums of its column blocks, two N-vector all-reduces.
//
// NCCL is loaded with dlopen at gpx_comm_init time (the library shipped with PyTorch), so libgpx.so itself has no link
// dependency on it.
#include <dlfcn.h>

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "gpx_common.cuh"
#include "gpx_ctx.cuh"
#include "gpx_fine.cuh"
#include "gpx_kernels.cuh"

// ---- minimal NCCL surface (types as in nccl.h 2.x) ---------------------------------------------------------------
extern "C" {
typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
typedef enum { ncclSuccess = 0 } ncclResult_t;
typedef enum { ncclInt8 = 0, ncclChar = 0, ncclUint8 = 1, ncclInt32 = 2, ncclInt = 2, ncclUint32 = 3, ncclInt64 = 4,
               ncclUint64 = 5, ncclFloat16 = 6, ncclHalf = 6, ncclFloat32 = 7, ncclFloat = 7, ncclFloat64 = 8,
               ncclDouble = 8 } ncclDataType_t;
typedef enum { ncclSum = 0, ncclProd = 1, ncclMax = 2, ncclMin = 3 } ncclRedOp_t;
}

namespace {
struct NcclApi {
  void* handle = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*Broadcast)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  ncclResult_t (*CommSplit)(ncclComm_t, int, int, ncclComm_t*, void*) = nullptr;   // optional (NCCL >= 2.18)
};
NcclApi g_nccl;

int load_nccl() {
  if (g_nccl.handle) return 0;
  const char* cands[] = {getenv("GPX_NCCL_LIB"),
                         "/opt/prime-rl/.venv/lib/python3.12/site-packages/nvidia/nccl/lib/libnccl.so.2",
                         "libnccl.so.2", "libnccl.so"};
  for (const char* cnd : cands) {
    if (!cnd) continue;
    g_nccl.handle = dlopen(cnd, RTLD_NOW | RTLD_GLOBAL);
    if (g_nccl.handle) break;
  }
  if (!g_nccl.handle) { gpx::set_error("cannot dlopen libnccl.so.2 (set GPX_NCCL_LIB)"); return -3; }
#define GPX_SYM(field, name)                                                                  \
  *(void**)(&g_nccl.field) = dlsym(g_nccl.handle, name);                                      \
  if (!g_nccl.field) { gpx::set_error(std::string("libnccl lacks ") + name); return -3; }
  GPX_SYM(GetUniqueId, "ncclGetUniqueId")
  GPX_SYM(CommInitRank, "ncclCommInitRank")
  GPX_SYM(CommDestroy, "ncclCommDestroy")
  GPX_SYM(Broadcast, "ncclBroadcast")
  GPX_SYM(AllGather, "ncclAllGather")
  GPX_SYM(AllReduce, "ncclAllReduce")
  GPX_SYM(GetErrorString, "ncclGetErrorString")
#undef GPX_SYM
  *(void**)(&g_nccl.CommSplit) = dlsym(g_nccl.handle, "ncclCommSplit");
  return 0;
}
}  // namespace

#define GPX_NCCL(call)                                                                                       \
  do {                                                                                                       \
    ncclResult_t r__ = (call);                                                                               \
    if (r__ != ncclSuccess) {                                                                                \
      gpx::set_error(std::string(#call) + " failed: " + g_nccl.GetErrorString(r__) + " at " + __FILE__ + ":" + \
                     std::to_string(__LINE__));                                                              \
      return -4;                                                                                             \
    }                                                                                                        \
  } while (0)

struct DistState {
  ncclComm_t comm = nullptr;
  ncclComm_t comm2 = nullptr;  // duplicate communicator for the look-ahead side stream (null: no look-ahead)
  double* Bc2 = nullptr;       // second broadcast buffer
  std::vector<cudaEvent_t> ev;
  int rank = 0, G = 1;
  long NB = 0, npr = 0, nblk = 0;
  double* Bc = nullptr;        // NB x NB broadcast buffer (L_kk^-1)
  double* raw = nullptr;       // device: raw sums for the scalar all-reduce
  double* h_raw = nullptr;     // pinned
  double* blkpart = nullptr;   // [nblk][P][Npad] partials of alpha
  // memory-distributed layout: c->S is the ROW-owned workspace SL (ldl = npr * NB rows x Npad columns: the block rows of
  // the trailing matrix / L / inverse region this rank updates), SU the COLUMN-owned final U = L^-T (Npad rows x npr * NB
  // columns: column block k at local slot k / G). Together 2 Npad^2 / G doubles per rank instead of Npad^2.
  double* SU = nullptr;
  long ldl = 0;
};

using namespace gpx;

namespace gpx {

void dist_free(gpx_ctx* c) {
  if (!c->dist) return;
  DistState* d = c->dist;
  if (d->Bc) cudaFree(d->Bc);
  if (d->Bc2) cudaFree(d->Bc2);
  if (d->blkpart) cudaFree(d->blkpart);
  if (d->SU) cudaFree(d->SU);
  d->Bc = d->Bc2 = d->blkpart = d->SU = nullptr;
}

// everything the communicator brought to the context: the sharded buffers, the NCCL communicators (and their device
// memory and proxy threads), the reduction buffers and events; the context is single-GPU afterwards
void dist_destroy(gpx_ctx* c) {
  if (!c->dist) return;
  DistState* d = c->dist;
  dist_free(c);
  if (d->comm2) g_nccl.CommDestroy(d->comm2);
  if (d->comm) g_nccl.CommDestroy(d->comm);
  if (d->raw) cudaFree(d->raw);
  if (d->h_raw) cudaFreeHost(d->h_raw);
  for (auto e : d->ev) cudaEventDestroy(e);
  delete d;
  c->dist = nullptr;
}

// Collective gpx_get(GPX_GET_L) on a sharded factor (Posterior.woodbury_chol, posterior.py:21-77): block row by block row the
// owner extracts its rows of L into a staging block, broadcasts it, and every rank copies it into its own host matrix
// (N x N column-major). N x NB doubles of device staging; nothing of size N^2 on any device.
int dist_get_L(gpx_ctx* c, double* out) {
  DistState* d = c->dist;
  const long N = c->N, Npad = c->Npad, NB = d->NB;
  cudaStream_t st = c->st;
  double* stage = nullptr;
  GPX_CUDA(cudaMalloc(&stage, (size_t)NB * Npad * 8));
  int rc = 0;
  for (long R = 0; R < d->nblk && rc == 0; R++) {
    const long grow0 = R * NB;
    if (grow0 >= N) break;
    const long ncols = std::min(N, grow0 + NB);            // L is lower triangular: columns beyond the block row are zero
    if (R % d->G == d->rank)
      rc = launch_extract_L_rows(c->S, d->ldl, (R / d->G) * NB, c->Ldiag, grow0, NB, ncols, stage, st);
    if (rc == 0 && g_nccl.Broadcast(stage, stage, (size_t)NB * ncols, ncclDouble, (int)(R % d->G), d->comm, st) != ncclSuccess) {
      gpx::set_error("ncclBroadcast failed in the sharded gpx_get");
      rc = -1;
    }
    const long nrows = std::min(NB, N - grow0);
    if (rc == 0 && cudaMemcpy2DAsync(out + grow0, (size_t)N * 8, stage, (size_t)NB * 8, (size_t)nrows * 8, (size_t)ncols,
                                     cudaMemcpyDeviceToHost, st) != cudaSuccess) rc = -1;
    if (cudaStreamSynchronize(st) != cudaSuccess) rc = -1;   // the staging block is reused by the next block row
  }
  cudaFree(stage);
  c->total_launches += (d->nblk + d->G - 1) / d->G;
  return rc;
}

long dist_block(const gpx_ctx* c) { return c->dist ? c->dist->NB : 0; }

// the column-owned U = L^-T storage of a sharded context (predict): Npad x (npr NB), leading dimension Npad
const double* dist_U(const gpx_ctx* c, long* ld) {
  if (!c->dist || !c->dist->SU) return nullptr;
  *ld = c->Npad;
  return c->dist->SU;
}

int dist_world(const gpx_ctx* c, int* rank, int* nranks) {
  if (c->dist && c->dist->comm) { *rank = c->dist->rank; *nranks = c->dist->G; }
  else { *rank = 0; *nranks = 1; }
  return 0;
}

int dist_allreduce_sum(gpx_ctx* c, double* buf, size_t count, cudaStream_t st) {
  if (!c->dist || !c->dist->comm || c->dist->G <= 1) return 0;
  GPX_NCCL(g_nccl.AllReduce(buf, buf, count, ncclDouble, ncclSum, c->dist->comm, st));
  return 0;
}

static long dist_pick_nb(const gpx_ctx* c, long N) {
  if (c->NB > 0) return c->NB;
  const char* e = getenv("GPX_NB");
  if (e && atol(e) >= TILE && atol(e) % TILE == 0) return atol(e);
  if (N >= 32768) return 1024;
  if (N >= 8192) return 512;
  return 256;
}

int dist_set_data(gpx_ctx* c, int64_t N, int D, int P) {
  DistState* d = c->dist;
  const long NB = std::min<long>(dist_pick_nb(c, N), (N + TILE - 1) / TILE * TILE);
  const long Npad = (N + NB - 1) / NB * NB;      // whole blocks: every rank sees the same block structure
  const long nblk = Npad / NB, npr = (nblk + d->G - 1) / d->G;
  if (Npad != c->Npad || D != c->D || P != c->P || NB != d->NB) {
    GPX_CUDA(cudaStreamSynchronize(c->st));
    free_data(c);   // also whatever single-GPU work allocated on this context before the communicator came
    dist_free(c);
    c->Npad = Npad; c->D = D; c->P = P;
    d->NB = NB; d->nblk = nblk; d->npr = npr;
    GPX_CHECK(alloc_data(c, NB));
    GPX_CUDA(cudaMalloc(&c->dUvPart, (size_t)Npad * P * 8));
    d->ldl = npr * NB;
    GPX_CUDA(cudaMalloc(&c->S, (size_t)d->ldl * Npad * 8));       // owned block rows only
    GPX_CUDA(cudaMalloc(&d->SU, (size_t)Npad * d->ldl * 8));      // owned column blocks of U only
    GPX_CUDA(cudaMemsetAsync(d->SU, 0, (size_t)Npad * d->ldl * 8, c->st));
    GPX_CUDA(cudaMalloc(&c->Pbuf, (size_t)2 * d->G * npr * NB * NB * 8));   // double-buffered (look-ahead)
    GPX_CUDA(cudaMalloc(&d->Bc, (size_t)NB * NB * 8));
    GPX_CUDA(cudaMalloc(&d->Bc2, (size_t)NB * NB * 8));
    GPX_CUDA(cudaMalloc(&d->blkpart, (size_t)nblk * P * Npad * 8));
    GPX_CUDA(cudaMemsetAsync(c->Pbuf, 0, (size_t)2 * d->G * npr * NB * NB * 8, c->st));
  }
  return 0;
}

// One distributed evaluation; results (raw sums) land in d->h_raw, the info flag in *c->h_info. Collective.
int dist_exact_eval(gpx_ctx* c, double extra_jitter) {
  DistState* d = c->dist;
  cudaStream_t st = c->st;
  const long ld = d->ldl, Npad = c->Npad, NB = d->NB;   // ld: leading dimension of the row-owned workspace
  const int nt = (int)(Npad / TILE), nbt = (int)(NB / TILE);
  const int G = d->G, g = d->rank;
  KernParams kp;   // the single-kernel entries alone reach a sharded context
  if (!as_single(c->mk, c->D, &kp)) GPX_FAIL("internal: the sharded evaluation takes a single kernel");
  const int nl = kp.ard ? c->D : 1, nred = nl + 2;
  GPX_CUDA(cudaMemsetAsync(c->info, 0, sizeof(int), st));
  GPX_CUDA(cudaMemsetAsync(c->logdet_part, 0, (size_t)nt * 8, st));
  GPX_CHECK(launch_prep_x(c->dX, c->N, Npad, kp, c->dXsT, c->dsq, st));
  c->eval_launches++;
  {
    KBuildParams kb;
    memset(&kb, 0, sizeof(kb));
    kb.rowsT = c->dXsT; kb.ld_rows = Npad; kb.colsT = c->dXsT; kb.ld_cols = Npad;
    kb.sq_rows = c->dsq; kb.sq_cols = c->dsq;
    kb.out = c->S; kb.ld = ld; kb.nrows = c->N; kb.ncols = c->N; kb.sym = 1; kb.same = 1;
    kb.diag_add = (c->noise + c->jitter) + extra_jitter;
    kb.own_G = G; kb.own_g = g; kb.own_blk = nbt; kb.loc_rows = 1;
    kb.kp = kp;
    GPX_CHECK(launch_kbuild(kb, nt, nt, st));
    c->eval_launches++;
  }
  // ---- sweep -----------------------------------------------------------------------------------------------------
  // Look-ahead (when a second communicator is available): D(k), the broadcast of L_kk^-1, the panel product, the
  // all-gather and the copy-back of step k run on the high-priority side stream (own NCCL communicator) as soon as
  // the columns of block k have received update k-1 (U1); the main stream meanwhile finishes U2(k-1).
  const bool la = d->comm2 != nullptr && d->nblk > 1;
  cudaStream_t sm = st, ss = la ? c->st2 : st;
  ncclComm_t cs = la ? d->comm2 : d->comm;
  size_t evi = 0;
  auto next_event = [&](cudaEvent_t* e) -> int {
    if (d->ev.size() <= evi) {
      cudaEvent_t x;
      GPX_CUDA(cudaEventCreateWithFlags(&x, cudaEventDisableTiming));
      d->ev.push_back(x);
    }
    *e = d->ev[evi++];
    return 0;
  };
  cudaEvent_t ev;
  if (la) {
    GPX_CHECK(next_event(&ev));
    GPX_CUDA(cudaEventRecord(ev, sm));
    GPX_CUDA(cudaStreamWaitEvent(ss, ev, 0));
  }
  const size_t pstride = (size_t)G * d->npr * NB * NB;
  for (int k = 0; k < (int)d->nblk; k++) {
    const long o = (long)k * NB;
    const int kt0 = k * nbt, kt1 = kt0 + nbt;
    const int root = k % G;
    const long pos_k = (long)(k % G) * d->npr + k / G;
    double* Pb = c->Pbuf + (size_t)(k & 1) * pstride;
    double* Bc = (k & 1) ? d->Bc2 : d->Bc;
    if (g == root) {
      double* Sblk = c->S + (long)(k / G) * NB + o * ld;   // the diagonal block inside the owner's local rows
      GPX_CHECK(diag_block_sweep(c, Sblk, ld, nbt, kt0, ss));
      // U_kk into this rank's chunk of the panel buffer, L_kk^-1 into the broadcast buffer
      GPX_CHECK(launch_assemble(Sblk, ld, (int)NB, Pb + pos_k * NB * NB, NB, Bc, ss));
      c->eval_launches++;
    }
    // one block: there is no panel, and the owner's chunk already holds U_kk, which the copy-back files into SU
    if (d->nblk > 1) {
      GPX_NCCL(g_nccl.Broadcast(Bc, Bc, (size_t)NB * NB, ncclDouble, root, cs, ss));
      GemmParams pp = gemm_defaults();
      pp.mode = GEMM_PANEL;
      pp.A = c->S + o * ld; pp.lda = ld; pp.loc_A = 1;
      pp.B = Bc; pp.ldb = NB;
      pp.C = Pb; pp.ldc = NB; pp.map_C = 1;
      pp.map_blk = nbt; pp.map_G = G; pp.map_npr = (int)d->npr; pp.map_stride = NB * NB;
      pp.own_G = G; pp.own_g = g; pp.own_blk = nbt;
      pp.K = (int)NB; pp.nt = nt; pp.skip0 = kt0; pp.skip1 = kt1; pp.tri = 1;
      GPX_CHECK(launch_gemm(pp, dim3(nbt, nt - nbt), ss));
      c->eval_launches++;
      GPX_NCCL(g_nccl.AllGather(Pb + (size_t)g * d->npr * NB * NB, Pb, (size_t)d->npr * NB * NB, ncclDouble, cs, ss));
    }
    GPX_CHECK(launch_copyback(c->S, ld, d->SU, Npad, Pb, NB, G, g, d->npr, k, nt, ss));
    c->eval_launches++;
    if (la) {
      GPX_CHECK(next_event(&ev));
      GPX_CUDA(cudaEventRecord(ev, ss));
      GPX_CUDA(cudaStreamWaitEvent(sm, ev, 0));
    }
    if (kt1 < nt) {
      const int next_nbt = std::min(nbt, nt - kt1);
      for (int part = 0; part < 2; part++) {
        const int cbeg = part == 0 ? kt1 : kt1 + next_nbt;
        const int cend = part == 0 ? kt1 + next_nbt : nt;
        if (cbeg < cend) {
          GemmParams pu = gemm_defaults();
          pu.mode = GEMM_UPDATE;
          pu.A = Pb; pu.lda = NB; pu.map_A = 1;
          pu.B = Pb; pu.ldb = NB; pu.map_B = 1;
          pu.map_blk = nbt; pu.map_G = G; pu.map_npr = (int)d->npr; pu.map_stride = NB * NB;
          pu.own_G = G; pu.own_g = g; pu.own_blk = nbt;
          pu.C = c->S; pu.ldc = ld; pu.loc_C = 1;
          pu.K = (int)NB; pu.nt = nt; pu.c0 = cbeg; pu.ncols = cend - cbeg; pu.rlow = kt1;
          GPX_CHECK(launch_gemm(pu, dim3(1, 1), sm));
          c->eval_launches++;
          c->stats.update_launches++;
        }
        if (part == 0 && la) {
          GPX_CHECK(next_event(&ev));
          GPX_CUDA(cudaEventRecord(ev, sm));
          GPX_CUDA(cudaStreamWaitEvent(ss, ev, 0));
        }
      }
    }
  }
  if (la) {
    GPX_CHECK(next_event(&ev));
    GPX_CUDA(cudaEventRecord(ev, ss));
    GPX_CUDA(cudaStreamWaitEvent(sm, ev, 0));
  }
  // ---- alpha = U (U^T y): owned column blocks, two vector all-reduces ------------------------------------------------
  GPX_CUDA(cudaMemsetAsync(c->dT, 0, (size_t)Npad * c->P * 8, st));
  GPX_CHECK(launch_utv(d->SU, Npad, Npad, c->P, c->dY, c->dT, st, G, g, NB, 1));
  GPX_NCCL(g_nccl.AllReduce(c->dT, c->dT, (size_t)Npad * c->P, ncclDouble, ncclSum, d->comm, st));
  GPX_CHECK(launch_uv_blk(d->SU, Npad, Npad, c->P, c->dT, NB, G, g, d->blkpart, c->dAlpha, st, 1));
  GPX_NCCL(g_nccl.AllReduce(c->dAlpha, c->dAlpha, (size_t)Npad * c->P, ncclDouble, ncclSum, d->comm, st));
  c->eval_launches += 3;
  // ---- K^-1 = U U^T over the owned k-range with the fused gradient epilogue ------------------------------------------
  GPX_CUDA(cudaMemsetAsync(c->partials, 0, (size_t)nt * nt * nred * 8, st));
  {
    GemmParams pl = gemm_defaults();
    pl.mode = GEMM_LAUUM;
    pl.A = d->SU; pl.lda = Npad; pl.B = d->SU; pl.ldb = Npad; pl.C = nullptr; pl.ldc = Npad; pl.k_local = 1;
    pl.K = (int)Npad; pl.nt = nt;
    pl.XsT = c->dXsT; pl.sq = c->dsq; pl.alpha = c->dAlpha; pl.ldx = Npad;
    pl.N = (int)c->N; pl.P = c->P; pl.partials = c->partials; pl.kinv_out = nullptr;
    pl.k_G = G; pl.k_g = g; pl.k_blk = nbt;
    pl.kp = kp;
    GPX_CHECK(launch_gemm(pl, dim3(1, 1), st));
    c->eval_launches++;
  }
  {
    FinalizeParams f;
    memset(&f, 0, sizeof(f));
    f.partials = c->partials; f.ntiles = (long)nt * nt; f.nl = nl;
    f.logdet_part = c->logdet_part; f.nt = nt;
    f.T = c->dT; f.ld = Npad; f.N = c->N; f.P = c->P; f.kp = kp; f.res = d->raw;
    GPX_CHECK(launch_finalize_raw(f, st));
    c->eval_launches++;
  }
  GPX_NCCL(g_nccl.AllReduce(d->raw, d->raw, (size_t)nred + 1, ncclDouble, ncclSum, d->comm, st));   // not |T|^2
  GPX_NCCL(g_nccl.AllReduce(c->info, c->info, 1, ncclInt32, ncclMax, d->comm, st));
  GPX_CUDA(cudaMemcpyAsync(d->h_raw, d->raw, (nred + 2) * sizeof(double), cudaMemcpyDeviceToHost, st));
  GPX_CUDA(cudaMemcpyAsync(c->h_info, c->info, sizeof(int), cudaMemcpyDeviceToHost, st));
  GPX_CUDA(cudaStreamSynchronize(st));
  // assemble (lml, gradient) exactly as finalize_kernel does on a single GPU
  const double* tot = d->h_raw;
  const double logdet = tot[nred], quad = tot[nred + 1];
  const double log2pi = 1.8378770664093453;
  c->h_res[0] = 0.5 * (-(double)c->N * c->P * log2pi - (double)c->P * logdet - quad);
  c->h_res[1] = tot[0];
  for (int q = 0; q < nl; q++) c->h_res[2 + q] = -tot[1 + q] / kp.ls[q];
  c->h_res[2 + nl] = tot[nred - 1];
  c->h_res[3 + nl] = logdet;
  c->h_res[4 + nl] = quad;
  return 0;
}

}  // namespace gpx

extern "C" {

int gpx_comm_unique_id(char id_out[128]) {
  if (!id_out) { gpx::set_error("null argument"); return -2; }
  GPX_CHECK(load_nccl());
  ncclUniqueId id;
  GPX_NCCL(g_nccl.GetUniqueId(&id));
  memcpy(id_out, id.internal, 128);
  return 0;
}

int gpx_comm_init(gpx_ctx* c, const char id[128], int rank, int nranks) {
  if (!c || !id) { gpx::set_error("null argument"); return -2; }
  if (nranks < 1 || rank < 0 || rank >= nranks) { gpx::set_error("bad rank / nranks"); return -2; }
  GPX_CHECK(load_nccl());
  GPX_CUDA(cudaSetDevice(c->device));
  GPX_CUDA(cudaStreamSynchronize(c->st));
  // a second call replaces the communicator: the earlier one is released, and the workspace (with any evaluation in it)
  // goes with it, since its layout was that of the earlier attachment
  dist_destroy(c);
  free_data(c);
  c->Npad = 0;   // the next gpx_set_data allocates the distributed layout
  DistState* d = new DistState();
  ncclUniqueId uid;
  memcpy(uid.internal, id, 128);
  const ncclResult_t r = g_nccl.CommInitRank(&d->comm, nranks, uid, rank);
  if (r != ncclSuccess) {   // the context stays single-GPU
    delete d;
    gpx::set_error(std::string("ncclCommInitRank failed: ") + g_nccl.GetErrorString(r));
    return -4;
  }
  c->dist = d;
  d->rank = rank; d->G = nranks;
  if (g_nccl.CommSplit && nranks > 1 && !getenv("GPX_NO_DIST_LOOKAHEAD")) {
    if (g_nccl.CommSplit(d->comm, 0, rank, &d->comm2, nullptr) != ncclSuccess) d->comm2 = nullptr;
  }
  GPX_CUDA(cudaMalloc(&d->raw, (MAX_D + 8) * sizeof(double)));
  GPX_CUDA(cudaMallocHost(&d->h_raw, (MAX_D + 8) * sizeof(double)));
  return 0;
}

}  // extern "C"
