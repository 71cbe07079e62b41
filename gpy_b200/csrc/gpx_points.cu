// gpx_points.cu — point sets, K-builds and the kernel-gradient reductions shared by the exact evaluation, the sparse
// evaluation and the stand-alone kernel calls. Each helper is told which kernel description it works with and never falls
// back on the context's own; as_single decides whether it launches the single-kernel or the composite kernels.
#include <algorithm>
#include <cstring>
#include <vector>

#include "gpx_common.cuh"
#include "gpx_ctx.cuh"
#include "gpx_kernels.cuh"

namespace gpx {

bool as_single(const MultiKern& k, int D, KernParams* kp) {
  const PartDev& pd = k.part[0];
  if (k.nparts != 1 || pd.kind < GPX_RBF || pd.kind > GPX_MATERN52 || pd.D != D) return false;
  for (int q = 0; q < D; q++)
    if (k.dims[q] != q) return false;
  if (kp) {
    memset(kp, 0, sizeof(*kp));
    kp->kind = pd.kind; kp->ard = pd.ard; kp->D = D; kp->variance = pd.variance; kp->inv_ls_iso = pd.inv_ls_iso;
    const int nl = pd.ard ? D : 1;
    for (int q = 0; q < MAX_D; q++) kp->ls[q] = q < nl ? k.ls[q] : 1.0;
  }
  return true;
}

int kern_ngrad(const MultiKern& k) {
  int n = 0;
  for (int p = 0; p < k.nparts; p++) n += part_ngrad(k.part[p]);
  return n;
}

int prep_points(gpx_ctx* c, const MultiKern& k, const double* X, long n, int D, long ld, double* xT, double* sq) {
  KernParams kp;
  return as_single(k, D, &kp) ? launch_prep_x(X, n, ld, kp, xT, sq, c->st) : launch_prep_multi(X, n, D, ld, k, xT, sq, c->st);
}

int upload_points(gpx_ctx* c, const MultiKern& k, const double* X, long n, int D, PointSet& ps) {
  ps.n = n; ps.ld = (n + TILE - 1) / TILE * TILE; ps.st = c->st;
  GPX_TMP_ALLOC(&ps.raw, (size_t)n * D * 8, c->st);
  GPX_TMP_ALLOC(&ps.xT, (size_t)ps.ld * std::max(1, k.sumD) * 8, c->st);   // static parts alone stack no rows
  GPX_TMP_ALLOC(&ps.sq, (size_t)ps.ld * k.nparts * 8, c->st);
  GPX_CUDA(cudaMemcpyAsync(ps.raw, X, (size_t)n * D * 8, cudaMemcpyHostToDevice, c->st));
  GPX_CHECK(prep_points(c, k, ps.raw, n, D, ps.ld, ps.xT, ps.sq));
  c->total_launches++;
  return 0;
}

int build_K(gpx_ctx* c, const MultiKern& k, int D, const Points& rows, const Points& cols, double* out, long ld,
            const KyDiag* ky, int rt0, int nrt) {
  const int row_tiles = nrt ? nrt : (int)(rows.ld / TILE), col_tiles = (int)(cols.ld / TILE);
  const int same = rows.xT == cols.xT;   // one point set on both sides: exact zero distance on the diagonal
  KernParams kp;
  if (!as_single(k, D, &kp)) {
    KBuildMultiParams kb;
    memset(&kb, 0, sizeof(kb));
    kb.rowsT = rows.xT; kb.ld_rows = rows.ld; kb.sq_rows = rows.sq;
    kb.colsT = cols.xT; kb.ld_cols = cols.ld; kb.sq_cols = cols.sq;
    kb.out = out; kb.ld = ld; kb.nrows = rows.n; kb.ncols = cols.n; kb.same = same; kb.mk = k;
    if (ky) { kb.sym = 1; kb.diag_add = ky->add; }
    return launch_kbuild_multi(kb, row_tiles, col_tiles, c->st);
  }
  KBuildParams kb;
  memset(&kb, 0, sizeof(kb));
  kb.rowsT = rows.xT; kb.ld_rows = rows.ld; kb.sq_rows = rows.sq;
  kb.colsT = cols.xT; kb.ld_cols = cols.ld; kb.sq_cols = cols.sq;
  kb.out = out; kb.ld = ld; kb.nrows = rows.n; kb.ncols = cols.n; kb.same = same; kb.rt0 = rt0; kb.kp = kp;
  if (ky) { kb.sym = 1; kb.diag_add = ky->add; kb.diag_vec = ky->vec; }
  return launch_kbuild(kb, row_tiles, col_tiles, c->st);
}

GradFullParams grad_params(const MultiKern& k, int D, const Points& rows, const Points& cols, const double* dL_dK, long ldd) {
  GradFullParams gp;
  memset(&gp, 0, sizeof(gp));
  gp.x1T = rows.xT; gp.ld1 = rows.ld; gp.sq1 = rows.sq; gp.N = rows.n;
  gp.x2T = cols.xT; gp.ld2 = cols.ld; gp.sq2 = cols.sq; gp.M = cols.n;
  gp.dL_dK = dL_dK; gp.ldd = ldd; gp.same = rows.xT == cols.xT;
  as_single(k, D, &gp.kp);
  return gp;
}

// partial sums per tile of part p's update_gradients_full reduction: its gradient entries and tr(dL_dK); the single
// kernel's reduction keeps no trace slot
static int grad_full_nred(const MultiKern& k, bool single, int p) {
  return single ? part_ngrad(k.part[0]) : part_nred(k.part[p]);
}

size_t grad_full_doubles(const MultiKern& k, int D, const GradFullParams& gp) {
  const bool single = as_single(k, D, nullptr);
  int nred = 0;
  for (int p = 0; p < k.nparts; p++) nred += grad_full_nred(k, single, p);
  return (size_t)(gp.ld1 / TILE) * (gp.ld2 / TILE) * nred;
}

int grad_full_sum(gpx_ctx* c, const MultiKern& k, int D, GradFullParams gp, double* part, double* grad) {
  const int tiles_j = (int)(gp.ld2 / TILE), tiles_i = (int)(gp.ld1 / TILE);
  const size_t ntile = (size_t)tiles_j * tiles_i;
  const bool single = as_single(k, D, nullptr);
  if (single) {
    gp.partials = part;
    GPX_CHECK(launch_grad_full(gp, tiles_j, tiles_i, c->st));
    c->total_launches++;
  } else {   // the composite reduction maps the column points to threads: rows and columns trade places
    GradFullMultiParams gf;
    memset(&gf, 0, sizeof(gf));
    gf.rowsT = gp.x2T; gf.ld_rows = gp.ld2; gf.sq_rows = gp.sq2;
    gf.colsT = gp.x1T; gf.ld_cols = gp.ld1; gf.sq_cols = gp.sq1;
    if (gp.cP) GPX_FAIL("internal: a composite's reduction takes a complete dL_dK (no rank-P term)");
    gf.nrows = gp.M; gf.ncols = gp.N; gf.same = gp.same; gf.dL = gp.dL_dK; gf.ldd = gp.ldd > 0 ? gp.ldd : gp.M;
    gf.mk = k;
    size_t off = 0;
    for (int p = 0; p < k.nparts; p++) {   // one launch per part, each into its own block of partials
      gf.part = p; gf.partials = part + off;
      GPX_CHECK(launch_grad_full_multi(gf, tiles_j, tiles_i, c->st));
      c->total_launches++;
      off += ntile * grad_full_nred(k, single, p);
    }
  }
  std::vector<double> hp(grad_full_doubles(k, D, gp));
  GPX_CUDA(cudaMemcpyAsync(hp.data(), part, hp.size() * 8, cudaMemcpyDeviceToHost, c->st));
  GPX_CUDA(cudaStreamSynchronize(c->st));
  size_t off = 0;
  int g = 0;
  for (int p = 0; p < k.nparts; p++) {
    const int nred = grad_full_nred(k, single, p);
    std::vector<double> tot(nred, 0.0);
    for (size_t t = 0; t < ntile; t++)
      for (int q = 0; q < nred; q++) tot[q] += hp[off + t * nred + q];
    double v;
    for (int q = 0; q < nred; q++)
      if (part_grad_entry(k, p, q, tot[q], &v)) grad[g + q] = v;
    g += part_ngrad(k.part[p]);
    off += ntile * nred;
  }
  return 0;
}

// the columns are split into chunks so that ~4 waves of CTAs are in flight; the chunks' partials are reduced in fixed order
static void gradx_chunks(const gpx_ctx* c, const GradFullParams& gp, int* nchunk, long* mchunk) {
  const long ntile = (gp.N + TILE - 1) / TILE;
  const int n = (int)std::max<long>(1, std::min<long>((gp.M + 31) / 32, (4 * c->num_sms + ntile - 1) / ntile));
  *mchunk = ((gp.M + n - 1) / n + 31) / 32 * 32;
  *nchunk = (int)((gp.M + *mchunk - 1) / *mchunk);
}

// doubles of one chunk's partials: the kernel's stacked rows (the single kernel's D columns)
size_t grad_X_doubles(const gpx_ctx* c, const MultiKern& k, const GradFullParams& gp, int D) {
  int nchunk;
  long mchunk;
  gradx_chunks(c, gp, &nchunk, &mchunk);
  return (size_t)nchunk * gp.N * std::max(1, k.sumD) + (size_t)gp.N * D;
}

int grad_X(gpx_ctx* c, const MultiKern& k, const GradFullParams& gp, int D, double* part, double* out) {
  int nchunk;
  long mchunk;
  gradx_chunks(c, gp, &nchunk, &mchunk);
  double* dout = part + (size_t)nchunk * gp.N * std::max(1, k.sumD);
  if (as_single(k, D, nullptr)) {
    GPX_CHECK(launch_gradx(gp, nchunk, mchunk, part, dout, c->st));
  } else {
    GradXMultiParams gx;
    memset(&gx, 0, sizeof(gx));
    gx.rowsT = gp.x1T; gx.ld_rows = gp.ld1; gx.sq_rows = gp.sq1; gx.nrows = gp.N;
    gx.colsT = gp.x2T; gx.ld_cols = gp.ld2; gx.sq_cols = gp.sq2; gx.ncols = gp.M;
    if (gp.cP) GPX_FAIL("internal: a composite's reduction takes a complete dL_dK (no rank-P term)");
    gx.dL = gp.dL_dK; gx.ldd = gp.ldd > 0 ? gp.ldd : gp.M; gx.transposed = gp.transposed; gx.same = gp.same;
    gx.Dfull = D; gx.mk = k;
    GPX_CHECK(launch_gradx_multi(gx, nchunk, mchunk, part, dout, c->st));
  }
  c->total_launches += 2;
  GPX_CUDA(cudaMemcpyAsync(out, dout, (size_t)gp.N * D * 8, cudaMemcpyDeviceToHost, c->st));
  GPX_CUDA(cudaStreamSynchronize(c->st));
  return 0;
}

int exact_grad_X(gpx_ctx* c, double* out) {
  GradFullParams gp;   // only its extents: training points x training points
  memset(&gp, 0, sizeof(gp));
  gp.N = gp.M = c->N;
  int nchunk;
  long mchunk;
  gradx_chunks(c, gp, &nchunk, &mchunk);
  ExactGradXParams ep;
  memset(&ep, 0, sizeof(ep));
  ep.Kinv = c->Kinv; ep.ld = c->Npad;
  ep.alpha = c->dAlpha; ep.P = c->P;
  ep.XsT = c->dXsT; ep.sq = c->dsq; ep.ldx = c->Npad; ep.N = c->N;
  ep.Dfull = c->D; ep.mk = c->mk;
  const size_t npart = (size_t)nchunk * c->N * std::max(1, c->mk.sumD), nout = (size_t)c->N * c->D;
  double* buf = nullptr;
  GPX_TMP_ALLOC(&buf, (npart + nout) * 8, c->st);
  int rc = launch_exact_gradx(ep, nchunk, mchunk, buf, buf + npart, c->st);
  if (rc == 0) c->total_launches += 2;   // counted only when both launches were issued
  if (rc == 0 && cudaMemcpyAsync(out, buf + npart, nout * 8, cudaMemcpyDeviceToHost, c->st) != cudaSuccess) rc = -1;
  if (cudaStreamSynchronize(c->st) != cudaSuccess && rc == 0) rc = -1;
  GPX_TMP_FREE(buf, c->st);
  if (rc == -1) set_error("gpx_exact_grad_X: device failure");
  return rc;
}

int pred_grad_check(const MultiKern& k) {
  for (int p = 0; p < k.nparts; p++)
    if (k.part[p].kind == GPX_RATQUAD || k.part[p].kind == GPX_STDPERIODIC)
      GPX_FAIL("gradients_X: RatQuad / StdPeriodic parts have no input gradient on the device");
  return 0;
}

// the Jacobian reduction is the composite one for every kernel: the single kernel's prepared points are those of its
// one-part description (prep_x_kernel = prep_multi_kernel)
int pred_grad(gpx_ctx* c, const MultiKern& k, const Points& test, const Points& train, const double* alpha, long lda, int P,
              const double* V, long ldv, int D, double* dmu, double* dvar) {
  GPX_CHECK(pred_grad_check(k));
  PredGradParams pp;
  memset(&pp, 0, sizeof(pp));
  pp.mk = k;
  pp.rowsT = test.xT; pp.ld_rows = test.ld; pp.sq_rows = test.sq; pp.nrows = test.n;
  pp.colsT = train.xT; pp.ld_cols = train.ld; pp.sq_cols = train.sq; pp.ncols = train.n;
  pp.alpha = alpha; pp.lda = lda; pp.P = P; pp.V = V; pp.ldv = ldv; pp.Dfull = D;
  GradFullParams gp;   // only its extents: test points x training points
  memset(&gp, 0, sizeof(gp));
  gp.N = test.n; gp.M = train.n;
  int nchunk;
  long mchunk;
  gradx_chunks(c, gp, &nchunk, &mchunk);
  const size_t npart = (size_t)(P + 1) * nchunk * test.n * std::max(1, pp.mk.sumD), nout = (size_t)test.n * D * (P + 1);
  double* buf = nullptr;
  GPX_TMP_ALLOC(&buf, (npart + nout) * 8, c->st);
  int rc = launch_pred_grad(pp, nchunk, mchunk, buf, buf + npart, c->st);
  c->total_launches += pred_grad_launches(pp.mk, P);
  const size_t nmu = (size_t)test.n * D * P;
  if (rc == 0 && cudaMemcpyAsync(dmu, buf + npart, nmu * 8, cudaMemcpyDeviceToHost, c->st) != cudaSuccess) rc = -1;
  if (rc == 0 && cudaMemcpyAsync(dvar, buf + npart + nmu, (size_t)test.n * D * 8, cudaMemcpyDeviceToHost, c->st) != cudaSuccess)
    rc = -1;
  if (cudaStreamSynchronize(c->st) != cudaSuccess && rc == 0) rc = -1;
  GPX_TMP_FREE(buf, c->st);
  if (rc == -1) set_error("predictive gradients: device failure");
  return rc;
}

}  // namespace gpx
