// gpx_points.cu — point sets, K-builds and the kernel-gradient reductions shared by the exact evaluation, the sparse
// evaluation and the stand-alone kernel calls, for either kind of covariance function: each helper is told which one it
// works with (Kern: a single stationary kernel or a composite) and never falls back on the context's own.
#include <algorithm>
#include <cstring>
#include <vector>

#include "gpx_common.cuh"
#include "gpx_ctx.cuh"
#include "gpx_kernels.cuh"

namespace gpx {

int prep_points(gpx_ctx* c, Kern k, const double* X, long n, int D, long ld, double* xT, double* sq) {
  return k.kp ? launch_prep_x(X, n, ld, *k.kp, xT, sq, c->st) : launch_prep_multi(X, n, D, ld, *k.mk, xT, sq, c->st);
}

int upload_points(gpx_ctx* c, Kern k, const double* X, long n, int D, PointSet& ps) {
  ps.n = n; ps.ld = (n + TILE - 1) / TILE * TILE; ps.st = c->st;
  GPX_TMP_ALLOC(&ps.raw, (size_t)n * D * 8, c->st);
  GPX_TMP_ALLOC(&ps.xT, (size_t)ps.ld * std::max(1, k.coord_rows()) * 8, c->st);   // static parts alone stack no rows
  GPX_TMP_ALLOC(&ps.sq, (size_t)ps.ld * k.norm_rows() * 8, c->st);
  GPX_CUDA(cudaMemcpyAsync(ps.raw, X, (size_t)n * D * 8, cudaMemcpyHostToDevice, c->st));
  GPX_CHECK(prep_points(c, k, ps.raw, n, D, ps.ld, ps.xT, ps.sq));
  c->total_launches++;
  return 0;
}

int build_K(gpx_ctx* c, Kern k, const Points& rows, const Points& cols, double* out, long ld, const KyDiag* ky, int rt0,
            int nrt) {
  const int row_tiles = nrt ? nrt : (int)(rows.ld / TILE), col_tiles = (int)(cols.ld / TILE);
  const int same = rows.xT == cols.xT;   // one point set on both sides: exact zero distance on the diagonal
  if (k.mk) {
    KBuildMultiParams kb;
    memset(&kb, 0, sizeof(kb));
    kb.rowsT = rows.xT; kb.ld_rows = rows.ld; kb.sq_rows = rows.sq;
    kb.colsT = cols.xT; kb.ld_cols = cols.ld; kb.sq_cols = cols.sq;
    kb.out = out; kb.ld = ld; kb.nrows = rows.n; kb.ncols = cols.n; kb.same = same; kb.mk = *k.mk;
    if (ky) { kb.sym = 1; kb.diag_add = ky->add; }
    return launch_kbuild_multi(kb, row_tiles, col_tiles, c->st);
  }
  KBuildParams kb;
  memset(&kb, 0, sizeof(kb));
  kb.rowsT = rows.xT; kb.ld_rows = rows.ld; kb.sq_rows = rows.sq;
  kb.colsT = cols.xT; kb.ld_cols = cols.ld; kb.sq_cols = cols.sq;
  kb.out = out; kb.ld = ld; kb.nrows = rows.n; kb.ncols = cols.n; kb.same = same; kb.rt0 = rt0; kb.kp = *k.kp;
  if (ky) { kb.sym = 1; kb.diag_add = ky->add; kb.diag_vec = ky->vec; }
  return launch_kbuild(kb, row_tiles, col_tiles, c->st);
}

GradFullParams grad_params(Kern k, const Points& rows, const Points& cols, const double* dL_dK, long ldd) {
  GradFullParams gp;
  memset(&gp, 0, sizeof(gp));
  gp.x1T = rows.xT; gp.ld1 = rows.ld; gp.sq1 = rows.sq; gp.N = rows.n;
  gp.x2T = cols.xT; gp.ld2 = cols.ld; gp.sq2 = cols.sq; gp.M = cols.n;
  gp.dL_dK = dL_dK; gp.ldd = ldd; gp.same = rows.xT == cols.xT;
  if (k.kp) gp.kp = *k.kp;
  return gp;
}

// partial sums per tile of the update_gradients_full reduction: a single kernel's variance and lengthscale(s); part p's
// gradient entries and tr(dL_dK)
static int grad_full_nred(Kern k, int p = 0) { return k.kp ? (k.kp->ard ? k.kp->D : 1) + 1 : part_nred(k.mk->part[p]); }

size_t grad_full_doubles(Kern k, const GradFullParams& gp) {
  int nred = 0;
  for (int p = 0; p < (k.kp ? 1 : k.mk->nparts); p++) nred += grad_full_nred(k, p);
  return (size_t)(gp.ld1 / TILE) * (gp.ld2 / TILE) * nred;
}

int grad_full_sum(gpx_ctx* c, Kern k, GradFullParams gp, double* part, double* grad) {
  const int tiles_j = (int)(gp.ld2 / TILE), tiles_i = (int)(gp.ld1 / TILE), nparts = k.kp ? 1 : k.mk->nparts;
  const size_t ntile = (size_t)tiles_j * tiles_i;
  if (k.kp) {
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
    gf.mk = *k.mk;
    size_t off = 0;
    for (int p = 0; p < nparts; p++) {   // one launch per part, each into its own block of partials
      gf.part = p; gf.partials = part + off;
      GPX_CHECK(launch_grad_full_multi(gf, tiles_j, tiles_i, c->st));
      c->total_launches++;
      off += ntile * grad_full_nred(k, p);
    }
  }
  std::vector<double> hp(grad_full_doubles(k, gp));
  GPX_CUDA(cudaMemcpyAsync(hp.data(), part, hp.size() * 8, cudaMemcpyDeviceToHost, c->st));
  GPX_CUDA(cudaStreamSynchronize(c->st));
  size_t off = 0;
  int g = 0;
  for (int p = 0; p < nparts; p++) {
    const int nred = grad_full_nred(k, p);
    std::vector<double> tot(nred, 0.0);
    for (size_t t = 0; t < ntile; t++)
      for (int q = 0; q < nred; q++) tot[q] += hp[off + t * nred + q];
    double v;
    for (int q = 0; q < nred; q++) {
      if (k.kp) grad[q] = q ? -tot[q] / k.kp->ls[q - 1] : tot[0];   // stationary.py:210,213
      else if (part_grad_entry(*k.mk, p, q, tot[q], &v)) grad[g + q] = v;
    }
    if (!k.kp) g += part_ngrad(k.mk->part[p]);
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

// doubles of one chunk's partials: a single kernel's D columns, a composite's stacked rows
static int gradx_width(Kern k) { return k.kp ? k.kp->D : std::max(1, k.mk->sumD); }

size_t grad_X_doubles(const gpx_ctx* c, Kern k, const GradFullParams& gp, int D) {
  int nchunk;
  long mchunk;
  gradx_chunks(c, gp, &nchunk, &mchunk);
  return (size_t)nchunk * gp.N * gradx_width(k) + (size_t)gp.N * (k.kp ? k.kp->D : D);
}

int grad_X(gpx_ctx* c, Kern k, const GradFullParams& gp, int D, double* part, double* out) {
  int nchunk;
  long mchunk;
  gradx_chunks(c, gp, &nchunk, &mchunk);
  double* dout = part + (size_t)nchunk * gp.N * gradx_width(k);
  if (k.kp) {
    D = k.kp->D;
    GPX_CHECK(launch_gradx(gp, nchunk, mchunk, part, dout, c->st));
  } else {
    GradXMultiParams gx;
    memset(&gx, 0, sizeof(gx));
    gx.rowsT = gp.x1T; gx.ld_rows = gp.ld1; gx.sq_rows = gp.sq1; gx.nrows = gp.N;
    gx.colsT = gp.x2T; gx.ld_cols = gp.ld2; gx.sq_cols = gp.sq2; gx.ncols = gp.M;
    if (gp.cP) GPX_FAIL("internal: a composite's reduction takes a complete dL_dK (no rank-P term)");
    gx.dL = gp.dL_dK; gx.ldd = gp.ldd > 0 ? gp.ldd : gp.M; gx.transposed = gp.transposed; gx.same = gp.same;
    gx.Dfull = D; gx.mk = *k.mk;
    GPX_CHECK(launch_gradx_multi(gx, nchunk, mchunk, part, dout, c->st));
  }
  c->total_launches += 2;
  GPX_CUDA(cudaMemcpyAsync(out, dout, (size_t)gp.N * D * 8, cudaMemcpyDeviceToHost, c->st));
  GPX_CUDA(cudaStreamSynchronize(c->st));
  return 0;
}

int pred_grad_check(Kern k) {
  for (int p = 0; k.mk && p < k.mk->nparts; p++)
    if (k.mk->part[p].kind == GPX_RATQUAD || k.mk->part[p].kind == GPX_STDPERIODIC)
      GPX_FAIL("gradients_X: RatQuad / StdPeriodic parts have no input gradient on the device");
  return 0;
}

int pred_grad(gpx_ctx* c, Kern k, const Points& test, const Points& train, const double* alpha, long lda, int P,
              const double* V, long ldv, int D, double* dmu, double* dvar) {
  GPX_CHECK(pred_grad_check(k));
  PredGradParams pp;
  memset(&pp, 0, sizeof(pp));
  if (k.mk) {
    pp.mk = *k.mk;
  } else {   // a single kernel is the one-part composite on the same prepared points (prep_x_kernel = prep_multi_kernel)
    const KernParams& kp = *k.kp;
    pp.mk.nparts = 1; pp.mk.sumD = kp.D;
    pp.mk.part[0] = PartDev{kp.kind, kp.ard, 0, 0, kp.D, 0, kp.variance, kp.inv_ls_iso, 0.0};
    for (int q = 0; q < kp.D; q++) { pp.mk.dims[q] = q; pp.mk.ls[q] = kp.ls[kp.ard ? q : 0]; }
  }
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
