// gpx_ctx.cuh — the device context behind the opaque gpx_ctx of include/gpx.h (internal).
#pragma once
#include <vector>

#include "gpx_common.cuh"
#include "gpx_kernels.cuh"
#include "gpx_ozaki.cuh"
#include "gpx_multi.cuh"

struct DistState;
struct SparseState;

struct gpx_ctx {
  int device = 0;
  cudaStream_t st = nullptr;
  cudaStream_t st2 = nullptr;   // high-priority side stream: diagonal-block work + panel of the NEXT step (look-ahead)
  cudaStream_t st3 = nullptr;   // high-priority third stream of the Ozaki sweep: rest of the panel, digit split, copy-back, forward
                                // substitution -- everything of step k that the NEXT diagonal block does not wait for
  cudaEvent_t ev_kfirst = nullptr;   // int8 sweep, single kernel: recorded by the Ky build after its first block row, which
                                     // is all D(0) needs; passed on to the sweep by the evaluation that recorded it
  std::vector<cudaEvent_t> sync_ev;
  // data
  long N = 0, Npad = 0;
  int D = 0, P = 0;
  double* dX = nullptr;      // N x D row-major (as given)
  double* dXsT = nullptr;    // [rows_cap][Npad] scaled SoA of the training points, stacked as the kernel needs them
  double* dsq = nullptr;     // [norm_cap][Npad] their squared norms
  int rows_cap = 0, norm_cap = 0;   // rows dXsT and dsq hold: D and 1 from alloc_data, grown by a kernel that needs more
  double* dY = nullptr;      // [P][Npad]
  double* dT = nullptr;      // [P][Npad]  L^-1 y
  double* dAlpha = nullptr;  // [P][Npad]
  double* dUvPart = nullptr; // [KSPLIT][P][Npad]; not allocated for P > MAX_P
  // P > MAX_P (the wide route): dY holds Y as [Npad][Ppad] (row-major, zero padded), dT and dAlpha are [Ppad][Npad], and
  // dTt holds T = L^-1 Y as [Npad][Ppad]; Ppad = P padded to 128
  long Ppad = 0;
  double* dTt = nullptr;
  // workspace
  double* S = nullptr;       // Npad x Npad column-major: lower L, upper U
  double* Pbuf = nullptr;    // Npad x NB
  double* Tm = nullptr;      // NB x NB
  double* Ldiag = nullptr;   // nt tiles of 128x128
  double* Dinv = nullptr;    // nt tiles of 128x128
  double* logdet_part = nullptr;
  double* partials = nullptr;
  int* info = nullptr;
  double* res = nullptr;     // device result vector
  double* h_res = nullptr;   // pinned
  int* h_info = nullptr;     // pinned
  double* Kinv = nullptr;    // lazy (ensure_kinv), Npad x Npad (lower tiles)
  double* staging = nullptr; // lazy, N x N dense
  size_t staging_cap = 0;
  long NB = 0;               // outer block (0 = auto)
  long NBw = 0;              // outer block the workspace was allocated for (Pbuf, Tm, the int8 planes): chosen once per
                             // allocation, so that a later change of GPX_NB cannot run a sweep on buffers sized for another
  // last evaluation
  bool have_eval = false;
  bool have_kinv = false;    // c->Kinv holds K^-1 of the last evaluation (its route stored it, or gpx_get made it)
  gpx::MultiKern mk{};       // the kernel of the last evaluation
  double kdiag = 0;          // its Kdiag (jitter ladder, gpx_predict)
  double noise = 0, jitter = 0, jitter_extra = 0;
  // heteroscedastic evaluation (gpx_exact_eval_het): per-point noise variances in, diag(dL_dK) out
  bool het = false;
  double* dNoiseVec = nullptr; double* dDnoise = nullptr; long het_cap = 0;
  // accounting
  gpx_stats stats{};
  int64_t total_launches = 0;
  int64_t eval_launches = 0;
  std::vector<cudaEvent_t> ev;
  int profile = 1;
  // ---- Ozaki path (gpx_ozaki.cu): trailing update and K^-1 on the INT8 tensor cores ------------------------
  int ozaki = -1;              // option "ozaki": -1 = default (env GPX_OZAKI, else off), 0 = DMMA only, 1 = on where applicable
  int num_sms = 132;
  bool oz_ready = false;       // planes and right-hand-side buffers allocated for (Npad, NB)
  bool oz_lists_ready = false; // tile lists built for (Npad, NB)
  gpx::OzPlanes ozp[2];        // digit planes of the current / next panel (look-ahead double buffer)
  gpx::OzPlanes ozpA, ozpB;    // operands of the panel GEMM P = S(:, block) L_kk^-T on the tensor cores (from N = 4096): block
                               // column of the workspace (Npad x NB), L_kk^-1 (NB x NB)
  uint32_t* oz_tiles = nullptr;
  double* dYres = nullptr;     // [P][Npad] running right-hand side of the forward substitution carried along the sweep
  double* dTfw = nullptr;      // [P][Npad] t = L^-1 y from that substitution (quadratic form of the LML)
  using OzStep = gpx::OzStep;
  std::vector<OzStep> oz_steps;
  // ---- composite kernels (gpx_multi.cu) ---------------------------------------------------------------------------------
  double* mpartials = nullptr; // per part p in turn: [nt*nt][part_nred(p)]
  size_t mpart_cap = 0;        // doubles mpartials holds
  struct DistState* dist = nullptr;   // multi-GPU state (gpx_dist.cu), null on a single GPU
  struct SparseState* sparse = nullptr;   // sparse-GP (VarDTC) state (gpx_sparse.cu)
  gpx_ctx* cJ = nullptr;       // child context holding the factor of the last sampled covariance (gpx_joint.cu), created on
                               // first use: the caller's own factor, alpha and stats stay those of its evaluation
  // ---- Laplace approximation (gpx_laplace.cu) ---------------------------------------------------------------------------
  double* lapK = nullptr;      // K(X, X) of gpx_laplace_begin, Npad x Npad column-major, zero padded, kept for the evaluation
  double* lapV = nullptr;      // the vectors of the Newton steps and of the finish, [LAP_NV][Npad]
  long lap_cap = 0;            // Npad the two are sized for
  bool lap_begun = false;      // lapK holds K of c->mk on the current data (released by laplace_release)
  bool lap_post = false;       // the last evaluation is a Laplace or EP one (gpx_laplace_finish, gpx_ep_finish): no dL_dK
  std::vector<cudaEvent_t> lap_ev;
  // ---- expectation propagation (gpx_laplace.cu, on the kept K above) ----------------------------------------------------
  double* epSig = nullptr;     // Sigma of the sequential updates, Npad x Npad, lower tiles (diagonal tiles whole), zero padded
  double* epBlk = nullptr;     // one block of sites: S, S diag(c) (Npad x TILE each), the chain's G (TILE x TILE), c, g
  int* epOrd = nullptr;        // the update order of a sweep (N entries)
  bool ep_begun = false;       // gpx_ep_begin checked the labels and built K (released with the Laplace buffers)
  bool ep_ready = false;       // mu (and Sigma or its diagonal) of gpx_ep_start / gpx_ep_sweep are on the device
  bool ep_labels = false;      // the labels of the current data were checked by gpx_ep_begin (cleared with the buffers)
  bool ep_full = false;        // epSig holds the whole Sigma (else only its diagonal, in the vector slot, is kept)
  int sparse_wide = 0;         // option "sparse_wide": gpx_sparse_set_data takes up to GPX_MAX_OUTPUTS columns, not 8
  int epdtc_drift = 0;         // option "epdtc_drift": gpx_epdtc_sweep returns diag(Knm A Kmn) after its last block (the
                               // downdated A) in sigma_diag instead of the recompute's diagonal
  // ---- variational Gaussian approximation (gpx_laplace.cu, on the kept K above) ----------------------------------------
  std::vector<double> vg_alpha, vg_beta, vg_m;   // alpha, beta and m = K alpha of the last gpx_vargauss_begin (N each)
  bool vg_begun = false;       // lapK, alpha and beta of gpx_vargauss_begin are current (every other Laplace / EP call clears it)
  bool vg_factored = false;    // S holds the factor of A = I + B K B of that begin (gpx_vargauss_finish scales it in place)
  int vg_max_tries = 0;        // the ladder's max_tries of that begin, for a finish that factors A again
};


namespace gpx {
constexpr int KSPLIT = 32;
GemmParams gemm_defaults();
void free_data(gpx_ctx* c);                                  // every buffer sized by the data set
int alloc_data(gpx_ctx* c, long NB);                         // those of them whose size does not depend on the layout
// multi-GPU hooks implemented in gpx_dist.cu
int dist_set_data(gpx_ctx* c, int64_t N, int D, int P);      // (re)allocates the sharded layout for N points
int dist_exact_eval(gpx_ctx* c, double extra_jitter);
void dist_free(gpx_ctx* c);                                  // the sharded buffers; the communicator stays
void dist_destroy(gpx_ctx* c);                               // the buffers, the communicator and its state
int dist_get_L(gpx_ctx* c, double* out);                                       // collective: sharded woodbury_chol
long dist_block(const gpx_ctx* c);
const double* dist_U(const gpx_ctx* c, long* ld);                               // sharded: column-owned U storage                                             // NB of the sharded layout (0: none)
int dist_world(const gpx_ctx* c, int* rank, int* nranks);                       // (0, 1) without a communicator
int dist_allreduce_sum(gpx_ctx* c, double* buf, size_t count, cudaStream_t st);   // in place, on stream st
void sparse_free(gpx_ctx* c);
int factor_device(gpx_ctx* c, const double* dA, long lda, long N, double jitter0, int max_tries, double* logdet,
                  double* jitter_used);
// the DMMA factor-and-invert sweep over the matrix a caller wrote into S (factor workspace form); the caller zeroes c->info
// first and reads it afterwards. Launches are counted into c->eval_launches (gpx_api.cu)
int sweep_workspace(gpx_ctx* c);
// the plain LAUUM: U U^T of the factor in S into the lower tiles of c->Kinv (allocated on first use), one launch counted
// into c->eval_launches (gpx_api.cu)
int lauum_store(gpx_ctx* c);
void laplace_free(gpx_ctx* c);     // the Laplace buffers and events (gpx_laplace.cu)
void laplace_release(gpx_ctx* c);  // the Laplace / EP buffers (K and the vectors, 8 Npad (Npad + 28) bytes, EP's Sigma and
                                   // block) and flags: called by
                                   // gpx_set_data, gpx_sparse_set_data and every exact evaluation, so that the device memory
                                   // of a finished Laplace evaluation does not stay with the context

// ---- point sets, K-builds and kernel-gradient reductions (gpx_points.cu) ----------------------------------------------
// Temporaries of the stand-alone kernel calls and of gpx_predict: stream-ordered allocations from the device's default memory
// pool (cudaMallocAsync / cudaFreeAsync on the context's stream; gpx_create raises the pool's release threshold so that freed
// blocks stay cached). A plain cudaMalloc / cudaFree pair per call is a device-wide synchronisation point inside any
// optimiser loop that uses foreign inference.
#define GPX_TMP_ALLOC(ptr, bytes, st) GPX_CUDA(cudaMallocAsync((void**)(ptr), (bytes), (st)))
#define GPX_TMP_FREE(p, st) do { if (p) cudaFreeAsync((p), (st)); } while (0)

// Every helper below works with the kernel description k it is given, for host points with D columns (k's dims index them),
// and never falls back on the context's own. as_single is the one place that picks the specialised kernels: true iff k is a
// single stationary kernel, one part of kind RBF .. Matern52 on the dims 0 .. D-1 in order; then *kp (if given) is its
// KernParams, the launch parameter of those kernels. Every other description takes the composite kernels.
bool as_single(const MultiKern& k, int D, KernParams* kp);
int kern_ngrad(const MultiKern& k);   // entries of k's gradient block: every part's block in turn
// n points prepared for a kernel: scaled coordinates xT, SoA [k.sumD][ld], and their squared norms sq, [k.nparts][ld]
struct Points { double* xT = nullptr; double* sq = nullptr; long n = 0, ld = 0; };
struct PointSet : Points {   // host points uploaded and prepared in temporaries it owns
  double* raw = nullptr;
  cudaStream_t st = nullptr;
  ~PointSet() { GPX_TMP_FREE(raw, st); GPX_TMP_FREE(xT, st); GPX_TMP_FREE(sq, st); }
};
struct KyDiag { double add; const double* vec; };   // added to the diagonal of Ky: a constant, and per-point values (or null)

// The K-build and prep launches are counted by the caller (into eval_launches inside an exact evaluation); the other
// helpers count theirs into c->total_launches.
// X: n points, row-major with D columns
int prep_points(gpx_ctx* c, const MultiKern& k, const double* X, long n, int D, long ld, double* xT, double* sq);
int upload_points(gpx_ctx* c, const MultiKern& k, const double* X, long n, int D, PointSet& ps);
// K(rows, cols) into out[i + j * ld] (i: row point, j: column point), row tiles [rt0, rt0 + nrt) (nrt = 0: all of them;
// a part of the rows: single kernel only). ky != nullptr: the factor workspace form of Ky (lower tiles, zero upper tiles,
// identity padding, ky's diagonal terms).
int build_K(gpx_ctx* c, const MultiKern& k, int D, const Points& rows, const Points& cols, double* out, long ld,
            const KyDiag* ky = nullptr, int rt0 = 0, int nrt = 0);
// dL_dK (device; element (i, j) of rows x cols at dL_dK[i * ldd + j], ldd = 0: cols.n) for the reductions below. The caller
// may add the rank-P term (ci, cj, cP) and, for gradients_X, the transposed read.
GradFullParams grad_params(const MultiKern& k, int D, const Points& rows, const Points& cols, const double* dL_dK, long ldd);
// update_gradients_full: one reduction launch per part writes a row of partial sums per tile into `part`
// (grad_full_doubles); they are summed on the host in tile order and mapped to k's gradient block in paramz order into grad
// (every part's block in turn, as part_grad_entry maps it)
size_t grad_full_doubles(const MultiKern& k, int D, const GradFullParams& gp);
int grad_full_sum(gpx_ctx* c, const MultiKern& k, int D, GradFullParams gp, double* part, double* grad);
// gradients_X w.r.t. the row points: chunk partials and the N x D result in `part` (grad_X_doubles); the result is copied
// to `out` on the host. RatQuad / StdPeriodic parts have no device gradients_X (rc -2).
size_t grad_X_doubles(const gpx_ctx* c, const MultiKern& k, const GradFullParams& gp, int D);
int grad_X(gpx_ctx* c, const MultiKern& k, const GradFullParams& gp, int D, double* part, double* out);
// gradients_X of the last exact evaluation's kernel at its training points for its dL_dK, from the stored K^-1 (c->Kinv must
// hold it) and alpha: out (host) N x D row-major. Two launches, counted; temporaries from the stream-ordered pool.
int exact_grad_X(gpx_ctx* c, double* out);
// predictive gradients (gp.py:438-474) of k at the prepared test points against `train`, for the woodbury vector alpha
// ([P][lda], device) and V = woodbury_inv K(train, test) (V[n + m * ldv], device): dmu (n x D x P) and dvar (n x D), host,
// row-major. pred_grad_check: -2 for a kernel without a device input gradient (RatQuad / StdPeriodic parts), before
// anything is launched.
int pred_grad_check(const MultiKern& k);
int pred_grad(gpx_ctx* c, const MultiKern& k, const Points& test, const Points& train, const double* alpha, long lda, int P,
              const double* V, long ldv, int D, double* dmu, double* dvar);
// the training points of the context's last exact evaluation, as it prepared them for c->mk
inline Points train_points(const gpx_ctx* c) { return Points{c->dXsT, c->dsq, c->N, c->Npad}; }

// ---- joint posterior (gpx_joint.cu) ------------------------------------------------------------------------------------
#define GPX_FAIL_DEVICE(what)                             \
  do {                                                    \
    gpx::set_error(std::string(what) + ": device failure"); \
    return -1;                                            \
  } while (0)
// a stream-ordered temporary of doubles, released when it goes out of scope (or earlier, by release()); alloc reports an
// exhausted pool as -1 with a message
struct TmpBuf {
  double* p = nullptr;
  cudaStream_t st;
  explicit TmpBuf(cudaStream_t s) : st(s) {}
  ~TmpBuf() { release(); }
  int alloc(size_t doubles);
  void release() { GPX_TMP_FREE(p, st); p = nullptr; }
};
// L^-1 (upper = 0: lower, as gpx_get(LINV) reads it) or U = L^-T (upper = 1) of the factor in S into out (Npad x Npad
// column-major, zero elsewhere and in the padding). One launch, not counted.
int extract_inverse_factor(gpx_ctx* c, int upper, double* out);
// C = A B^T on the plain DMMA GEMM (GEMM_PANEL entry): rows x cols (whole tiles), k-depth kdepth; plain 2: lower tiles only;
// tri 1: B lower triangular, 2: A lower triangular. One launch, counted.
int gemm_nt(gpx_ctx* c, const double* A, long lda, const double* B, long ldb, double* C, long ldc, long rows, long cols,
            long kdepth, int plain, int tri);
// out(a, b) = K(a, off2 + b) - prod(a, b) (prod's lower tiles mirrored when sym); out column-major (ldo) or row-major
int joint_combine(gpx_ctx* c, const double* K, long ldk, long off2, const double* prod, long ldp, int sym, long M1, long M2,
                  double* out, long ldo, int colmajor);
// the argument checks of a sampling entry (-2 before anything is launched)
int joint_check(const gpx_ctx* c, const double* X, int64_t M, const double* z, int64_t nz, const double* f,
                const double* jitter_used, int P);
// f = mu + L_Sigma z for the device matrix Sigma (M x M, leading dimension lds), factored with jitchol's ladder in the child
// context c->cJ; mu [P][ldmu] (device), S vectors per output; z and f host, nz x M row-major
int joint_sample(gpx_ctx* c, const double* Sig, long lds, long M, const double* mu, long ldmu, const double* z, long nz,
                 long S, int max_tries, double* f, double* jitter_used);

// the parts of a composite kernel -> mk (validated against Dfull columns of X), *kdiag_total = its Kdiag (gpx_api.cu)
int fill_mk(MultiKern& mk, const gpx_kern_part* parts, int nparts, int Dfull, double* kdiag_total);
// the single stationary kernel of the single-kernel entries (kind, ard, variance, lengthscale on all D columns) -> its
// one-part description mk, checked with those entries' messages; its Kdiag is the variance (gpx_api.cu)
int fill_single(MultiKern& mk, int kind, int ard, int D, double variance, const double* ls);
}  // namespace gpx
