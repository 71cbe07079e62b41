/* gpx.h — C ABI of the H100 exact-GP engine (libgpx.so).
 *
 * This is the drop-in boundary for ONE hot path of SheffieldML/GPy:
 *     GPRegression -> GP.parameters_changed -> ExactGaussianInference.inference -> Kern.K/Kdiag/update_gradients_full
 * Each entry point names the reference interface it replaces (paths relative to the GPy repository root).
 * Plain C: pointers and sizes only, no torch / numpy types. All inputs, outputs and stored matrices are IEEE fp64; the N^3
 * products run on fp64 tensor instructions (DMMA, the default) or, with option "ozaki" on one GPU wherever the matrix has two
 * or more outer blocks, as int8
 * digit-split products on the wgmma tensor cores whose exact s32 sums are recombined in fp64 (8 digits for the Cholesky
 * part, 7 for the inverse part:
 * |dLML| <= 1e-8 and 1e-6 relative on gradients against the reference, DESIGN.md section 5.1; option "ozaki" selects).
 * The gradient bound is checked on the GPU up to cond(Ky) = 4.6e8. Above cond(Ky) ~ 1e8 the LML and alpha of both paths
 * are less accurate than LAPACK's (DESIGN.md section 5.1). The sparse evaluation stays within 4x the fp64 reference's
 * error up to cond(Kmm + 1e-8 I) = 3e10, the jitter floor (same section).
 *
 * Conventions
 *   - Return value: 0 ok; >0 "matrix not positive definite, leading minor <ret>" (the caller raises
 *     numpy.linalg.LinAlgError as GPy/util/linalg.py:64,75 does); <0 CUDA / argument error, text via gpx_last_error().
 *   - Host buffers are caller-owned and only read/written during the call. Device state lives behind gpx_ctx.
 *   - Matrices returned to the host are column-major (Fortran order) N x N unless stated, which is the layout
 *     LAPACK hands GPy (GPy/util/linalg.py:31-38 force_F_ordered); symmetric results are fully populated.
 *   - kind: 0 RBF (GPy/kern/src/rbf.py:51-52,177-178), 1 Exponential (stationary.py:382-386),
 *           2 Matern32 (stationary.py:488-492), 3 Matern52 (stationary.py:585-589).
 *   - ard:  0 -> `lengthscale` points at 1 double; 1 -> at D doubles (stationary.py:64-79).
 *   - Gradient vector order is paramz's: [kern.variance, kern.lengthscale (1 or D), Gaussian_noise.variance]
 *     (link order stationary.py:81, GPy/core/gp.py:106-107).
 */
#ifndef GPX_H_
#define GPX_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct gpx_ctx gpx_ctx;

enum { GPX_RBF = 0, GPX_EXPONENTIAL = 1, GPX_MATERN32 = 2, GPX_MATERN52 = 3,
       GPX_WHITE = 4, GPX_BIAS = 5, /* static parts of a composite kernel only (GPy/kern/src/static.py:63-99,142-185) */
       GPX_RATQUAD = 6,              /* RatQuad (stationary.py:747-802), composite parts and gpx_kern_part_* only */
       GPX_STDPERIODIC = 7 };        /* StdPeriodic (standard_periodic.py:56-94,125-139,501-548), likewise */

/* Output columns P of gpx_set_data: 1 .. GPX_MAX_OUTPUTS. Up to 8 every route below is open. Above 8 (the wide route) the
 * exact evaluation always stores K^-1 and runs on the fp64 DMMA path whatever option "ozaki" says; its solves are two
 * GEMMs, T = L^-1 Y (lower-triangular operand, N^2 Ppad flops) and alpha = U T (U = L^-T extracted with zeros below the
 * diagonal, 2 N^2 Ppad flops, Ppad = P padded to 128), the quadratic term of the LML is ||T||_F^2, and every part's gradient
 * (a single kernel's too) is reduced by the composite pass; gradients and LML come back in the layout of the entry called.
 * It keeps 32 Npad Ppad bytes of Y, T (twice) and alpha beside the N x N workspace; an allocation that does not fit returns
 * -1 with a message. For P > 8:
 *   served : gpx_exact_eval, gpx_exact_eval_multi, gpx_get (every selector), gpx_predict, gpx_exact_grad_X;
 *   -2     : gpx_exact_eval_het, gpx_predictive_gradients, gpx_posterior_covariance, gpx_posterior_samples, the Laplace and
 *            EP entries (P = 1 only), a context with a communicator attached (gpx_set_data).
 * Output columns P of gpx_sparse_set_data: 1 .. 8, or 1 .. GPX_MAX_OUTPUTS once the context's option "sparse_wide" is 1
 * (gpx_set_option; a context that never sets it keeps the limit of 8 it always had), more than 8 single-GPU only. Up to 8
 * every sparse route is as it was. Above 8 the VarDTC evaluation with scalar noise runs every P-column product on the fp64 DMMA GEMM
 * with Y held padded to whole tiles of outputs (Ppad): t^T = Y^T tmp^T (k-depth N), v, w and C against the triangular
 * factors, w w^T (k-depth Ppad), and dL_dKnm^T = [W2 | C] [psi1 | beta Y]^T in one GEMM of k-depth Mpad + Ppad; data_fit
 * = ||v||_F^2 is reduced on the device. Its launches depend on neither N nor P. It keeps 16 Npad Ppad bytes of Y (both
 * layouts) and 8 Npad Ppad more beside psi1. For P > 8:
 *   served : gpx_sparse_eval, gpx_sparse_eval_multi (scalar noise), gpx_sparse_get (every selector), gpx_sparse_predict
 *            (8 outputs per mean launch), gpx_sparse_grad_X;
 *   -2     : gpx_sparse_eval_het, gpx_sparse_eval_multi with per-point noise, gpx_sparse_predictive_gradients,
 *            gpx_sparse_posterior_samples, FITC, EPDTC and SVGP (P = 1 only), a context with a communicator attached. */
enum { GPX_MAX_OUTPUTS = 1024 };

/* gpx_get selectors */
enum {
  GPX_GET_L = 0,     /* woodbury_chol: lower Cholesky factor of K + (noise+jitter) I, N x N col-major, zeros above diag
                        (GPy/inference/latent_function_inference/exact_gaussian_inference.py:58,74) */
  GPX_GET_ALPHA = 1, /* woodbury_vector alpha = Ky^-1 Y, N x P row-major (exact_gaussian_inference.py:60) */
  GPX_GET_KINV = 2,  /* Wi = Ky^-1, symmetric N x N (GPy/util/linalg.py:210-212) */
  GPX_GET_DLDK = 3,  /* dL_dK = 0.5 (alpha alpha^T - P Ky^-1), symmetric N x N (exact_gaussian_inference.py:70) */
  GPX_GET_K = 4,     /* noise-free K(X,X), symmetric N x N (exact_gaussian_inference.py:53) */
  GPX_GET_LINV = 5   /* L^-1 lower, N x N col-major (GPy/util/linalg.py:209 dtrtri; unused by the exact-GP caller) */
};

/* Library / device ----------------------------------------------------------------------------------------------- */
const char* gpx_last_error(void);      /* thread-local text of the last <0 return */
const char* gpx_version(void);
int gpx_device_count(void);            /* number of visible CUDA devices, <0 on error */

/* One context per model: owns the stream(s), the N x N workspace and (multi-GPU) the NCCL communicator. */
int gpx_create(int device, gpx_ctx** out);
int gpx_destroy(gpx_ctx* ctx);

/* Replaces Kern._slice_X + ObsAr wiring (GPy/kern/src/kern.py:112-117, GPy/core/gp.py:42-62): host X (N x D, row-major,
 * already sliced to active dims) and Y (N x P row-major) are copied to HBM once per (X, Y) identity. */
int gpx_set_data(gpx_ctx* ctx, const double* X, int64_t N, int D, const double* Y, int P);

/* The hot call. Replaces, fused: Stationary.K (stationary.py:105-168) -> diag.add (exact_gaussian_inference.py:55-56)
 * -> pdinv/jitchol/dpotri (GPy/util/linalg.py:56-75,193-214) -> dpotrs (:116-125) -> log marginal + dL_dK
 * (exact_gaussian_inference.py:62-72) -> Stationary.update_gradients_full (stationary.py:193-243, incl.
 * stationary_cython.pyx:53-62) -> Gaussian.exact_inference_gradients (GPy/likelihoods/gaussian.py:78-79).
 *   jitter     : added unconditionally to the diagonal (the reference uses 1e-8, exact_gaussian_inference.py:56)
 *   max_tries  : jitchol ladder length (reference: 5). On a non-PD factorisation the diagonal gets
 *                mean(diag)*1e-6*10^k, k = 0..max_tries-1 (linalg.py:66-74); *jitter_used reports the extra jitter.
 *   lml        : out, log marginal likelihood;  grad: out, (1 + (ard?D:1) + 1) doubles. */
int gpx_exact_eval(gpx_ctx* ctx, int kind, int ard, double variance, const double* lengthscale, double noise,
                   double jitter, int max_tries, double* lml, double* grad, double* jitter_used);

/* The same evaluation with one noise variance PER DATA POINT (HeteroscedasticGaussian, GPy/likelihoods/gaussian.py:347-362;
 * GPy/models/gp_heteroscedastic_regression.py:10-37): Ky = K + diag(noise_variances + jitter)
 * (exact_gaussian_inference.py:55-56 with a vector `variance`), and dL_dthetaL = diag(dL_dK) per point
 * (gaussian.py:358-359 applied to exact_gaussian_inference.py:72) written to dnoise (N doubles) by the fused K^-1
 * epilogue. grad keeps the layout of gpx_exact_eval; its last entry is the sum of dnoise. Single-GPU. */
int gpx_exact_eval_het(gpx_ctx* ctx, int kind, int ard, double variance, const double* lengthscale,
                       const double* noise_variances, double jitter, int max_tries, double* lml, double* grad,
                       double* dnoise, double* jitter_used);

/* Composite kernels on the fused path: K = sum over terms of products of parts (GPy/kern/src/add.py:60-99 Add.K /
 * update_gradients_full; prod.py:59-68,377-396 Prod.K, where every factor's gradient sees dL_dK times the other factors;
 * static.py:63-99 White, :142-185 Bias). Each part is a stationary kernel on its own active dims (column indices into
 * the X of gpx_set_data; kernel_slice_operations.py:59-79), a White or a Bias kernel. Parts with the same `term` are
 * multiplied, terms are summed; parts must be ordered by term. The whole evaluation runs on the device like
 * gpx_exact_eval (K-build, factor-and-invert sweep, K^-1, one gradient-reduction pass per part over the stored K^-1).
 *   grad: out, concatenation over the parts in the given order of each part's gradient block, then d/d noise — the order
 *         paramz gives Add/Prod parameters (kern.py:363-451 link order). Blocks:
 *           RBF .. Matern52   [variance, lengthscale (1 or ndims)]                     (stationary.py:81)
 *           White, Bias       [variance]
 *           RatQuad           [variance, lengthscale (1 or ndims), power]              (stationary.py:81, then :760)
 *           StdPeriodic       [variance, period (1 or ndims), lengthscale (1 or ndims)] (standard_periodic.py:94)
 *         A StdPeriodic part keeps one sum per active dim for its period and one for its lengthscale: 2 ndims <= 64, else
 *         the call fails with -2 (the reduction does not fit).
 * gpx_get / gpx_predict afterwards use the composite kernel. Single-GPU. A one-part description equal to a single
 * stationary kernel (RBF .. Matern52 on the columns 0 .. D-1 in order) takes the single-kernel route, here and in every
 * other entry that takes parts: the same bits and launches as the single-kernel entry. */
typedef struct {
  int kind;                  /* GPX_RBF .. GPX_MATERN52, GPX_WHITE, GPX_BIAS, GPX_RATQUAD, GPX_STDPERIODIC */
  int ard;                   /* lengthscale: 0 -> points at 1 double, 1 -> at ndims doubles (StdPeriodic: GPy's ARD2) */
  int term;                  /* additive term this factor belongs to */
  int ndims;                 /* number of active dims (0 for White / Bias) */
  const int* dims;           /* column indices into X, ndims entries */
  double variance;
  const double* lengthscale;
  double power;              /* RatQuad: k = variance (1 + r^2/2)^-power, power > 0 (stationary.py:785-788) */
  int ard_period;            /* StdPeriodic (GPy's ARD1): 0 -> period points at 1 double, 1 -> at ndims doubles */
  const double* period;      /* StdPeriodic: k = variance exp(-1/2 sum_q (sin(pi (x_q - x'_q) / T_q) / l_q)^2), T_q > 0
                                (standard_periodic.py:125-132) */
} gpx_kern_part;
int gpx_exact_eval_multi(gpx_ctx* ctx, const gpx_kern_part* parts, int nparts, double noise, double jitter, int max_tries,
                         double* lml, double* grad, double* jitter_used);

/* Stand-alone K and update_gradients_full of ONE part (kinds 0-3, 6, 7; White / Bias are rejected) on the given inputs,
 * for callers that hold a kernel object outside an evaluation (PosteriorExact._raw_predict, the generic inference path).
 * X (N x D) and X2 (M x D) are row-major with the D columns `part->dims` index into; X2 == NULL -> X2 = X with exact zero
 * distance on the diagonal. The K-build and the per-pair gradient terms are those of gpx_exact_eval_multi.
 *   gpx_kern_part_K         : out, N x M row-major (like gpx_kern_K; it reports kbuild_ms and kbuild_bytes through
 *                             gpx_get_stats as well, but out must not be NULL).
 *   gpx_kern_part_grad_full : dL_dK N x M row-major in; grad out, the part's gradient block (as above). */
int gpx_kern_part_K(gpx_ctx* ctx, const gpx_kern_part* part, const double* X, int64_t N, const double* X2, int64_t M, int D,
                    double* out);
int gpx_kern_part_grad_full(gpx_ctx* ctx, const gpx_kern_part* part, const double* X, int64_t N, const double* X2,
                            int64_t M, int D, const double* dL_dK, double* grad);

/* Lazy device->host fetch of N^2 / N*P results of the last gpx_exact_eval (Posterior / grad_dict consumers:
 * GPy/inference/latent_function_inference/posterior.py:21-77; exact_gaussian_inference.py:74). */
int gpx_get(gpx_ctx* ctx, int which, double* out_host);

/* PosteriorExact._raw_predict (posterior.py:273-302) on device with the factor of the last eval:
 * mu (M x P row-major) = K(X,Xnew)^T alpha; var (M) = Kdiag(Xnew) - colsum((L^-1 K(X,Xnew))^2)   [full_cov = 0]
 * or var (M x M col-major) = K(Xnew) - tmp^T tmp                                                 [full_cov = 1]. */
int gpx_predict(gpx_ctx* ctx, const double* Xnew, int64_t M, int full_cov, double* mu, double* var);

/* GP.predictive_gradients (GPy/core/gp.py:418-474) on the device with the posterior of the last evaluation:
 *   dmu  (M x D x P row-major): dmu[m, q, p] = sum_n alpha[n, p] dk(x*_m, x_n)/dx*_mq
 *        (kern.gradients_X(woodbury_vector[:, p:p+1].T, Xnew, X), gp.py:442-446)
 *   dvar (M x D row-major):     dvar[m, q] = -2 sum_n V[n, m] dk(x*_m, x_n)/dx*_mq, V = woodbury_inv K(X, Xnew)
 *        (gp.py:448-462; gradients_X_diag is zero for these kernels, stationary.py:360-361, static.py:27-31)
 * D is that of the data set. The kernel is the evaluation's: a single kernel, or a composite of RBF .. Matern52, White
 * (zero between test and training points) and Bias parts; the input-gradient rules are those of gpx_kern_grad_X.
 *   gpx_predictive_gradients        : after gpx_exact_eval / _het / _multi. V = U (U^T K(X, Xnew)) with U = L^-T of the
 *                                     stored factor, MAX_P = 8 test points per pair of triangular passes; K^-1 is never
 *                                     formed. Launches: 2 + 3 ceil(M / 8) + R.
 *   gpx_sparse_predictive_gradients : after gpx_sparse_eval / _het / _multi; X = Z, alpha = woodbury_vector and W =
 *                                     woodbury_inv (var_dtc.py:207-210), formed as gpx_sparse_get(1) forms it, by the
 *                                     first call after an evaluation only (kept for the later calls); V on the DMMA
 *                                     GEMM. Launches: 8 + R for the first call after an evaluation, 3 + R after it.
 * R = ceil((P + 1) / g) + 1 reduction launches, g = 4 channels per launch when the kernel's stacked active dims are
 * <= 8, 2 when <= 16, else 1. Returns -2 without touching the posterior when there is no evaluation, M < 1, a pointer is
 * null, the kernel has a RatQuad or StdPeriodic part (no device input gradient) or a communicator is attached
 * (single-GPU). Nothing that gpx_get, gpx_sparse_get, gpx_predict or gpx_get_stats return changes. */
int gpx_predictive_gradients(gpx_ctx* ctx, const double* Xnew, int64_t M, double* dmu, double* dvar);
int gpx_sparse_predictive_gradients(gpx_ctx* ctx, const double* Xnew, int64_t M, double* dmu, double* dvar);

/* The input gradient of the last exact evaluation, what GPy's GPLVM adds to an evaluation (GPy/models/gplvm.py:47-49:
 * X.gradient = kern.gradients_X(dL_dK, X, None)). After gpx_exact_eval or gpx_exact_eval_multi, dX (N x D row-major, the D
 * of gpx_set_data) receives
 *   dX[n, d] = sum_m W[n, m] dk(x_n, x_m)/dx_n,d,   W = dL_dK + dL_dK^T = alpha alpha^T - P Ky^-1,
 * Stationary.gradients_X with X2 = None (stationary.py:245-252,325-345) summed over the parts as Add.gradients_X does
 * (add.py:88-100); a product's factor sees the other factors (prod.py:397-407); White and Bias enter only as factors; each
 * part's sums land on the data columns of its active dims. The kernel is that of the evaluation (a single kernel runs as
 * its one-part description through the same kernel). W is formed per 128 x 32 tile from the stored K^-1 and alpha, so
 * nothing of size N^2 is written: N^2 pairs x (P + per-part work) FMAs plus 8 N^2 bytes of K^-1 read.
 * Launches: 2, plus 1 when the evaluation took the fused single-kernel route (a single kernel with more than 8 tiles of
 * 128 points on the DMMA path), which does not store K^-1: the plain LAUUM stores it first, exactly as gpx_get(KINV) does,
 * and later calls reuse it. Returns -2 with nothing touched when there is no evaluation, the last one is a Laplace or EP
 * posterior (gpx_laplace_finish, gpx_ep_finish: their dL_dK is another), it is heteroscedastic (gpx_exact_eval_het), a
 * communicator is attached (single-GPU), the kernel has a RatQuad or StdPeriodic part (no device input gradient) or dX is
 * null. Nothing that gpx_get, gpx_predict or gpx_get_stats return changes. Temporaries: 8 N (nchunk sumD + D) bytes from
 * the stream-ordered pool (nchunk: the column chunks of gpx_kern_grad_X, sumD: the parts' stacked active dims). */
int gpx_exact_grad_X(gpx_ctx* ctx, double* dX);

/* The joint posterior of the last evaluation on the device (single-GPU; a context with a communicator attached gets -2).
 *
 * gpx_posterior_covariance : after gpx_exact_eval / _het / _multi. Posterior.covariance_between_points (posterior.py:109-130):
 *   cov (M1 x M2 row-major) = K(X1, X2) - K(X1, X) Ky^-1 K(X, X2) with the evaluation's kernel and factor; X1 (M1 x D) and
 *   X2 (M2 x D) row-major with the D of gpx_set_data. X2 == NULL means X2 = X1: cov is then exactly symmetric and K(X1, X1)
 *   has the exact zero distance on its diagonal, as gpx_kern_K with X2 = NULL. An explicit X2, even one equal to X1, is
 *   built the reference's way: kern.K(X1, X2) does not force coincident points to zero distance (this matters for
 *   Exponential, whose k is first order in r, where |x|^2 + |x'|^2 - 2 x.x' leaves r ~ 1e-8 at coincident points).
 *   Route: one K-build of K([X1; X2], X) (X2 stacked at a tile boundary), L^-1 = U^T extracted into a temporary,
 *   T^T = K(X*, X) L^-T on the DMMA GEMM (B lower triangular, N^2 (M1 + M2) flops), T1^T T2 on the DMMA GEMM, one K-build
 *   of K(X*, X*) and one combine. Launches: 7.
 * gpx_posterior_samples / gpx_sparse_posterior_samples : after an exact (gpx_exact_eval / _het / _multi) or a sparse
 *   (gpx_sparse_eval / _het / _multi) evaluation, every kernel either accepts. GP.posterior_samples_f (gp.py:601-629) with
 *   the latent predictive covariance at Xnew (M x D row-major)
 *     exact : Sigma = K(Xnew) - K(Xnew, X) Ky^-1 K(X, Xnew),  mu = K(Xnew, X) alpha          (posterior.py:273-302)
 *     sparse: Sigma = K(Xnew) - K(Xnew, Z) W K(Z, Xnew),      mu = K(Xnew, Z) woodbury_vector (posterior.py:238-270)
 *   with W = woodbury_inv, formed by the first of gpx_sparse_predictive_gradients / gpx_sparse_posterior_samples /
 *   gpx_sparse_predict after an evaluation and kept for all three. Sigma is factored with jitchol's rules (util/linalg.py:56-75): first plain, then with
 *   mean(diag) 1e-6 10^k added, k < max_tries; *jitter_used reports what was added. z holds nz = P S standard-normal
 *   vectors of length M, row-major nz x M and ordered output-major (S vectors for output 0, then S for output 1, ...), as
 *   numpy's legacy RNG draws them for np.random.multivariate_normal(m, v, S) once per output; f has the same layout:
 *   f_j = mu[:, j / S] + L_Sigma z_j. The samples are drawn from N(mu, Sigma + jitter I) through the Cholesky factor; the
 *   reference samples Sigma itself through numpy's SVD, with no jitter. Sigma is factored in a child context that the
 *   calling context creates on first use and owns. Returns > 0 (the leading minor) when Sigma is not positive definite
 *   after the ladder, as gpx_pdinv; -2 when there is no evaluation of the right kind, M < 1, nz < 1, nz is not a multiple
 *   of P, a pointer is null or a communicator is attached.
 *   Launches: exact 13 + F, sparse 12 + F, plus 5 on the first sparse call after an evaluation, which forms W. F is what
 *   gpx_pdinv of an M x M matrix that returns no matrices launches on a fresh context, binding included; one fewer when
 *   the child context holds an M x M workspace already.
 * None of the three entries changes anything that gpx_get, gpx_sparse_get, gpx_predict, gpx_predictive_gradients,
 * gpx_sparse_predictive_gradients or gpx_get_stats return, on success or failure; the evaluation's factor is only read.
 * Temporaries are stream-ordered (the pool of gpx_predict); an exhausted device returns -1 with a message. Peak bytes of
 * the temporaries, with Ls the test points padded to 128 (M1p + M2p for a cross-covariance, M1p = M1 padded), Np = N
 * padded, Mz = the inducing points padded:
 *   exact  : 8 (Np^2 + 2 Ls Np + 65 P Ls) while T^T is formed, then at most 8 (Ls Np + M1p M2p) and
 *            8 (Ls^2 + M1p M2p + M1 M2); N = 32768 and M = 4096: 10.7 GB beside the evaluation's own workspace
 *   sparse : 8 (2 Ls Mz + 2 Ls^2 + 65 P Ls)
 *   sampling adds 8 (Ls^2 + 2 nzp Ls + 2 nz M) (nzp = nz padded) and, in the child context, the workspace gpx_set_data
 *   allocates for M points. */
int gpx_posterior_covariance(gpx_ctx* ctx, const double* X1, int64_t M1, const double* X2, int64_t M2, double* cov);
int gpx_posterior_samples(gpx_ctx* ctx, const double* Xnew, int64_t M, const double* z, int64_t nz, int max_tries,
                          double* f, double* jitter_used);
int gpx_sparse_posterior_samples(gpx_ctx* ctx, const double* Xnew, int64_t M, const double* z, int64_t nz,
                                 int max_tries, double* f, double* jitter_used);

/* Standalone kernel plugin calls (no context needed beyond a device; ctx may be NULL -> device 0 scratch context).
 * Replaces Stationary.K (stationary.py:105-168): out is N x M ROW-major (what Kern.K returns to NumPy callers).
 * out == NULL: build on the device only and report the kernel time via gpx_get_stats (kbuild_ms, kbuild_bytes). */
int gpx_kern_K(gpx_ctx* ctx, int kind, int ard, double variance, const double* lengthscale, const double* X, int64_t N,
               const double* X2 /* NULL -> K(X,X) with exact zero-distance diagonal */, int64_t M, int D, double* out);
/* Replaces Stationary.Kdiag (stationary.py:170-173); kinds 0-3, 6 and 7 (StdPeriodic.Kdiag, standard_periodic.py:134-138,
 * is the variance as well). */
int gpx_kern_Kdiag(int kind, double variance, int64_t N, double* out);
/* Replaces Stationary.update_gradients_full (stationary.py:193-243) for a caller-supplied dL_dK (N x M row-major). */
int gpx_kern_grad_full(gpx_ctx* ctx, int kind, int ard, double variance, const double* lengthscale, const double* X,
                       int64_t N, const double* X2, int64_t M, int D, const double* dL_dK, double* dvariance,
                       double* dlengthscale);

/* Replaces Stationary.gradients_X (stationary.py:245-252,348-366 and the OpenMP helper GPy/kern/src/stationary_utils.c:1-14
 * _grad_X): grad (N x D row-major) = d/dX of sum(dL_dK * K(X, X2)); X2 == NULL is the symmetric case (tmp + tmp^T). */
int gpx_kern_grad_X(gpx_ctx* ctx, int kind, int ard, double variance, const double* lengthscale, const double* X,
                    int64_t N, const double* X2, int64_t M, int D, const double* dL_dK, double* grad);

/* Replaces pdinv / jitchol for a caller-supplied symmetric positive (semi-)definite matrix A (N x N, dense, symmetric so
 * row- and column-major coincide): GPy/util/linalg.py:193-214 (pdinv -> Ai, L, Li, logdet) and :56-75 (jitchol: first a
 * plain factorisation; on failure LinAlgError if any diagonal entry is <= 0, else jitter mean(diag)*1e-6*10^k, k <
 * max_tries). Ai / L / Li may be NULL (not wanted); L, Li are lower, column-major; returns >0 when not PD. */
int gpx_pdinv(gpx_ctx* ctx, const double* A, int64_t N, int max_tries, double* Ai, double* L, double* Li, double* logdet,
              double* jitter_used);

/* Sparse GP regression (VarDTC): the N-dependent work of GPy/inference/latent_function_inference/var_dtc.py:66-215 and of
 * the gradient wiring GPy/core/sparse_gp.py:108-119 (Gaussian likelihood, homoscedastic, certain inputs). psi1 = K(X, Z)
 * (8 N M bytes) is built and kept in HBM; only M x M / M x P / M x D results cross PCIe.
 *   gpx_sparse_set_data : X (N x D row-major), Y (N x P row-major) -> HBM (no N x N workspace is allocated).
 */
int gpx_sparse_set_data(gpx_ctx* ctx, const double* X, int64_t N, int D, const double* Y, int P);
/* One whole VarDTC evaluation on the device: VarDTC.inference (var_dtc.py:66-215, Gaussian homoscedastic noise, certain
 * inputs, no mean function) + SparseGP._update_gradients (core/sparse_gp.py:108-119) + Gaussian.update_gradients
 * (likelihoods/gaussian.py:78-79). Kmm + 1e-8 I and B = I + A are factored-and-inverted by the same sweep as the exact
 * path (jitchol ladder, util/linalg.py:56-75); every M x M product of :130-156,:201-233 is a DMMA GEMM; only the
 * scalars, dZ (M x D row-major) and the (1 + nl + 1) gradient entries [variance, lengthscale.., noise variance] return.
 * A = beta (Lm^-1 psi1^T)(Lm^-1 psi1^T)^T is formed from tmp = Lm^-1 psi1^T like the reference does (:130-132), not by
 * sandwiching psi1^T psi1, which loses ~cond(Kmm) digits. With a communicator attached (gpx_comm_init) X, Y are THIS
 * rank's rows and A, tmp Y and the Knm gradient pieces are all-reduced (var_dtc_parallel.py:113-131).
 *   gpx_sparse_get: posterior pieces of the last evaluation (var_dtc.py:201-214): 0 woodbury_vector (M x P row-major),
 *                   1 woodbury_inv (M x M), 2 Kmm (+ const_jitter on the diagonal), 3 Lm (lower, column-major). */
int gpx_sparse_eval(gpx_ctx* ctx, int kind, int ard, double variance, const double* lengthscale, const double* Z,
                    int64_t M, double noise_variance, double* lml, double* grad, double* dZ);
int gpx_sparse_get(gpx_ctx* ctx, int which, double* out);
/* SparseGP.predict's latent part on the device: Posterior._raw_predict (posterior.py:220-248) with pred_var = Z, the
 * posterior VarDTC returns (var_dtc.py:213), after gpx_sparse_eval / _het / _multi, with that evaluation's kernel, Z,
 * woodbury_vector and W = woodbury_inv. Xnew is M x D row-major with the D of gpx_sparse_set_data; mu is M x P row-major.
 *   full_cov = 0: var (M) = Kdiag(Xnew) - rowsum((K(Xnew, Z) W) o K(Xnew, Z)), then clipped at 1e-15 as the reference
 *                 clips it (posterior.py:248; a NaN stays NaN).
 *   full_cov = 1: var (M x M column-major) = K(Xnew) - K(Xnew, Z) W K(Z, Xnew), exactly symmetric (the lower tiles of the
 *                 product term mirrored), K(Xnew) with the exact zero distance on its diagonal; not clipped, as in the
 *                 reference.
 * W is formed by the first of gpx_sparse_predictive_gradients, gpx_sparse_posterior_samples and gpx_sparse_predict after an
 * evaluation (5 launches) and kept for all three. V^T = K(Xnew, Z) W runs on the DMMA GEMM; W is used as the reference
 * uses it, not in a factored form.
 * The diagonal streams over chunks of Lc test points, so M is not bounded by device memory:
 *   Lc = min(max(128, floor(2^30 / (16 Mz + 512 min(P, 8) + 8 P + 1096) / 128) 128), M padded to 128), Mz = the inducing
 *   points padded to 128 — the largest multiple of 128 whose temporaries stay within the 1 GiB the stream-ordered pool keeps
 *   cached (Lc = 15872 at Mz = 4096, P = 1). Launches: 6 per chunk (upload, K-build, GEMM, 2 for the mean, 1 variance
 *   reduction), with 2 more for the mean per further slab of 8 outputs when P > 8.
 *   Peak temporaries: 8 Lc (2 Mz + 64 min(P, 8) + P + 1) plus the chunk's points.
 *   A row's mu and var do not depend on the chunking: every GEMM element has a fixed k-order and every reduction runs per
 *   row in a fixed order, so a point predicted alone, in a block or inside a multi-chunk call gets the same bits.
 * The full covariance is one pass: Launches: 8. Peak temporaries: those of gpx_sparse_posterior_samples before sampling,
 *   8 (2 Ls Mz + 2 Ls^2 + 65 P Ls) with Ls = M padded to 128 (M = 4096, Mz = 4096: 539 MB).
 * With a communicator attached every rank holds the same posterior and predicts the points it is given; there is no
 * collective. Returns -2 without touching any state when there is no sparse evaluation, M < 1 or a pointer is null; -1 with
 * a message when the device is out of memory. Nothing that gpx_sparse_get, gpx_sparse_predictive_gradients,
 * gpx_sparse_posterior_samples or gpx_get_stats return changes, on success or failure. */
int gpx_sparse_predict(gpx_ctx* ctx, const double* Xnew, int64_t M, int full_cov, double* mu, double* var);
/* The same evaluation with ONE NOISE VARIANCE PER DATA POINT (HeteroscedasticGaussian, likelihoods/gaussian.py:347-362):
 * the `het_noise` branches of VarDTC.inference — tmp = Lm^-1 (psi1 sqrt(beta))^T (var_dtc.py:127-131), dL_dpsi1 += 2
 * (dL_dpsi2_beta (psi1 beta)^T)^T (:221-227), the bound with sum(log beta_n) and sum(beta_n |Y_n|^2) (:267-269) and the
 * per-point noise gradients dL_dR (:241-257). noise_variances: N values (this rank's rows); grad: (1 + nl) entries
 * [variance, lengthscale..]; dL_dR: N x P row-major, what HeteroscedasticGaussian.exact_inference_gradients indexes by
 * output_index (gaussian.py:358-359). dL_dR needs three column reductions over M x N matrices (|Lm^-1 psi1^T[:, n]|^2,
 * |LB^-1 Lm^-1 psi1^T[:, n]|^2, v^T LB^-1 Lm^-1 psi1^T[:, n]); nothing of size N x M crosses PCIe. gpx_sparse_get serves
 * the posterior of this evaluation as well. */
int gpx_sparse_eval_het(gpx_ctx* ctx, int kind, int ard, double variance, const double* lengthscale, const double* Z,
                        int64_t M, const double* noise_variances, double* lml, double* grad, double* dZ, double* dL_dR);
/* The same evaluation with a COMPOSITE KERNEL: a sum of products of RBF, Exponential, Matern32, Matern52 (each on its own
 * active dims), White and Bias parts, described as for gpx_exact_eval_multi and validated against the D of
 * gpx_sparse_set_data. psi0 is the composite's Kdiag (the sum over terms of the product of the part variances); White is
 * zero in psi1 and the trace of dL_dKmm in the Kmm gradient (static.py:77-93); dL/dZ is Add / Prod.gradients_X
 * (add.py:88-100, prod.py:397-407). noise_variances == NULL: scalar noise, grad = every part's block in order (part_ngrad
 * entries each) then d/d noise variance. noise_variances != NULL: N per-point variances as gpx_sparse_eval_het, grad = the
 * part blocks only, dL_dR (N x P row-major) required. RatQuad / StdPeriodic parts are rejected (-2: they have no device
 * gradients_X), and so is a context with a communicator attached (single-GPU). gpx_sparse_get serves this evaluation's
 * posterior; its Kmm is rebuilt with the composite. */
int gpx_sparse_eval_multi(gpx_ctx* ctx, const gpx_kern_part* parts, int nparts, const double* Z, int64_t M,
                          double noise_variance, const double* noise_variances, double* lml, double* grad, double* dZ,
                          double* dL_dR);
/* The latent-input gradient of the sparse bound (SparseGPLVM, GPy/models/sparse_gplvm.py:33-34): after gpx_sparse_eval,
 * _het or _multi, at any P that evaluation took, dX (N x D row-major, host) = sum_a dL_dKnm[n, a] dk(x_n, z_a)/dx_n, i.e.
 * kern.gradients_X(dL_dKnm, X, Z) of the evaluation's kernel. The gradients_X_diag term is zero for every kernel the sparse
 * evaluation takes (stationary.py:360-361, static.py:30-31) and is not added. It reads the dL_dKnm^T (M x N) the
 * evaluation left on the device, with its rank-P term added as the evaluation's own dL/dZ reduction added it; nothing of
 * size N x M crosses PCIe. Launches: 2. gpx_sparse_get, gpx_sparse_predict, gpx_sparse_predictive_gradients and
 * gpx_sparse_posterior_samples leave it intact. Returns -2 with nothing touched when there is no such evaluation, when a
 * FITC evaluation, EPDTC, SVGP or a new gpx_sparse_set_data has run since, with a communicator attached, or for a null
 * pointer. */
int gpx_sparse_grad_X(gpx_ctx* ctx, double* dX);
/* FITC sparse GP regression (Snelson & Ghahramani's SPGP): FITC.inference
 * (GPy/inference/latent_function_inference/fitc.py:19-88) + SparseGP._update_gradients (core/sparse_gp.py:108-118) +
 * Gaussian.update_gradients, for the data of gpx_sparse_set_data (P = 1) and any kernel gpx_sparse_eval_multi takes (a
 * single RBF .. Matern52 on all columns in order runs the single-kernel kernels). Kmm + 1e-6 I is factored with jitchol's
 * ladder as pdinv does; the effective noise sigma*_n = Kdiag + noise_variance - |Lm^-1 psi1_n^T|^2 is formed on the
 * device, beta*_n = 1 / sigma*_n without a floor, B = I + tmp diag(beta*) tmp^T factored with the ladder. Every N M^2
 * product runs on the DMMA GEMM (about 7 N M^2 flops, VarDTC about 4 N M^2); five M x N buffers (40 N Mz bytes, Mz = M
 * padded to 128) are kept on the context; launches do not depend on N.
 *   grad: the kernel's block (part blocks in order, part_ngrad entries each), then d/d noise variance = sum(dL_dR);
 *   dZ: M x D row-major; dL_dKdiag: N values of dL_dR (fitc.py:67), or NULL.
 * gpx_sparse_get(0..3) then return v, Kmm^-1 - P, Kmm + 1e-6 I and Lm (fitc.py:86), and gpx_sparse_predict /
 * _predictive_gradients / _posterior_samples serve this posterior. Returns 1 + n (numpy.linalg.LinAlgError in the Python
 * layer) with a message naming data point n when sigma*_n <= 0 or NaN, the first such n; >0 as well when a factorisation
 * fails after the ladder. Rejected with -2: P != 1, RatQuad / StdPeriodic parts, a context with a communicator attached
 * (single-GPU), null pointers, M < 1, no data. */
int gpx_sparse_eval_fitc(gpx_ctx* ctx, const gpx_kern_part* parts, int nparts, const double* Z, int64_t M,
                         double noise_variance, double* lml, double* grad, double* dZ, double* dL_dKdiag);

/* The Laplace approximation for a non-Gaussian likelihood (GPy/inference/latent_function_inference/laplace.py:122-353), one
 * output column (gpx_set_data with P = 1) and no mean function. The likelihood's per-point terms stay with the caller (they
 * are O(N)); the N^2 / N^3 work of Rasmussen's mode finding (rasm_mode, :148-231) and of the mode computations (:233-306)
 * runs here. Every entry returns -2 with nothing touched for a null pointer, a communicator (single-GPU), P != 1, and (all
 * but begin) no gpx_laplace_begin on the current data; > 0 (the leading minor) when B stays not positive definite after
 * jitchol's ladder (util/linalg.py:56-75: first as it is, then mean(diag B) 1e-6 10^k added, k < max_tries; *jitter_used
 * reports it). Launch counts below exclude F, the factor-and-invert sweep of an N x N matrix (that of gpx_pdinv), once per
 * attempt of the ladder; none of them depends on N. gpx_get_stats afterwards: launches, tries, and per-phase times
 * (profile option): kbuild_ms (the K-build), sweep_ms (B-build + sweep), update_ms (finish's GEMM), lauum_ms (finish's
 * LAUUM), solve_ms (mat-vecs and their glue), total_ms.
 *
 * gpx_laplace_begin : kern.K(X) (:128) with the kernel of the parts (every kernel gpx_exact_eval_multi takes) into an
 *   N x N buffer kept for the whole evaluation (8 Npad^2 bytes beside the factor workspace; it and the Newton vectors
 *   are released by the next gpx_set_data, gpx_sparse_set_data or exact evaluation on the context). The kernel becomes
 *   the context's kernel and the posterior of any earlier evaluation is gone. Launches: 2.
 * gpx_laplace_matvec : Kv = K v (N values each), np.dot(K, Ki_f) of :170,:210. Launches: 2.
 * gpx_laplace_newton : one Newton direction of rasm_mode (:184-199). W: N values clipped as the caller's likelihood clips them
 *   for B (:319-321); b = W f + dlogpdf_df with the unclipped W (:191-193); Ki_f the current iterate. B = I + (w_i K_ij) w_j,
 *   w = sqrt(W), is formed from the kept K in one pass and factored; a = b - w o (U U^T (w o K b)) with U = L_B^-T (the
 *   reference forms K_Wi_i, C, Ki_W_i and I_KW_i, four N x N products, on every step; only the factor is formed here);
 *   out: dKi_f = a - Ki_f and Kd = K dKi_f (N values each). Launches: 11 + F (+ 1 + F per extra attempt).
 * gpx_laplace_finish : the mode computations at f_hat (:243-306) with the clipped W, Ki_f = Ki_f_hat and
 *   dW_df = -d3logpdf_df3 (N values each):
 *     logdet_I_KW = 2 sum log diag(L_B) (:352);
 *     U~ = diag(w) U_B in place, so that gpx_get(LINV) returns LiW12 = L_B^-1 diag(w) (:331) and gpx_get(L) L_B;
 *     alpha = Ki_f_hat (gpx_get(ALPHA), woodbury_vector);
 *     diag_Ki_W_i (N) = diag(K) - the squared column norms of C = LiW12 K, C on the DMMA GEMM with A lower triangular (:347-348);
 *     dL_dfhat = -1/2 diag_Ki_W_i o dW_df (:258);
 *     K_Wi_i = U~ U~^T (woodbury_inv, :332) by the plain LAUUM; gpx_get(KINV) returns it;
 *     v = dL_dfhat - K_Wi_i K dL_dfhat (= I_KW_i^T dL_dfhat);
 *     kgrad: the kernel's gradient block (as gpx_exact_eval_multi's, without the noise entry) for dL_dK = 1/2 a a^T + a v^T
 *       - 1/2 K_Wi_i (:267-272, a = Ki_f_hat), whose symmetric part 1/2 [(a + v)(a + v)^T - (K_Wi_i + v v^T)] is reduced from
 *       the stored K_Wi_i + v v^T and alpha' = a + v by the exact evaluation's per-part reduction;
 *     dL_dthetaL_imp (nlik) = dL_dfhat^T I_KW_i K g_t = (K v)^T g_t for each row g_t of dlik_grad_dthetaL (nlik x N
 *       row-major; :293-295): one mat-vec whatever nlik.
 *   Afterwards gpx_get(K / ALPHA / KINV / L / LINV) return K, Ki_f_hat, K_Wi_i, L_B and LiW12, gpx_get(DLDK) returns -2, and
 *   gpx_predict, gpx_predictive_gradients, gpx_posterior_covariance and gpx_posterior_samples serve the Laplace posterior
 *   (woodbury_vector Ki_f_hat, woodbury_inv K_Wi_i; gpx_predict does not clip the variance). Launches: 16 + nparts + F.
 *   Peak temporaries: 16 Npad^2 bytes (LiW12 and C; 17.2 GB at N = 32768) beside the factor workspace, K^-1 and K. */
int gpx_laplace_begin(gpx_ctx* ctx, const gpx_kern_part* parts, int nparts);
int gpx_laplace_matvec(gpx_ctx* ctx, const double* v, double* Kv);
int gpx_laplace_newton(gpx_ctx* ctx, const double* W, const double* b, const double* Ki_f, int max_tries, double* dKi_f,
                       double* Kd, double* jitter_used);
int gpx_laplace_finish(gpx_ctx* ctx, const double* W, const double* Ki_f, const double* dW_df, int nlik,
                       const double* dlik_grad_dthetaL, int max_tries, double* logdet_I_KW, double* diag_Ki_W_i, double* kgrad,
                       double* dL_dthetaL_imp, double* jitter_used);

/* Expectation propagation for GP classification (GPy/inference/latent_function_inference/expectation_propagation.py:187-434,
 * the EP class) with the probit Bernoulli likelihood (likelihoods/bernoulli.py:59-92), one output column and no mean
 * function. The sites, the stopping rule, log Z~ and the update order (np.random.permutation, one per sweep) stay with the
 * caller; the N^2 / N^3 work runs here on the K kept as gpx_laplace_begin keeps it (the same buffer and release rules).
 * Every entry returns -2 with nothing touched for a null pointer, a communicator, P != 1 and (all but begin) no gpx_ep_begin
 * on the current data; > 0 (the leading minor) when B = I + S~^1/2 K S~^1/2 stays not positive definite after jitchol's
 * ladder (as gpx_laplace_newton). Launch counts exclude F, the factor sweep of B, once per attempt of the ladder.
 *
 * gpx_ep_begin : K(X, X) of the parts as gpx_laplace_begin builds it (:258-259). -2 also for labels outside {-1, 0, 1}
 *   ("bad value for Bernoulli observation (0, 1)", bernoulli.py:67-72), checked once per data set. Launches: 3.
 * gpx_ep_start : _init_approximations (:312-328). warm = 0: Sigma = K + 1e-7 I, mu = 0, the sites zero (tau_tilde and v_tilde
 *   are not read); warm = 1: _recompute (:129-143) from the given sites (N values each), then 1e-7 on Sigma's diagonal.
 *   parallel: the sweeps that follow update in parallel (parallel_updates=True): only diag(Sigma) is kept; otherwise the
 *   whole Sigma (8 Npad^2 bytes beside K). Launches: 1 cold; 14 + F warm.
 * gpx_ep_sweep : one pass of EP's loop (:296-306): _local_updates in the given order (a permutation of 0 .. N-1, else -2),
 *   then _recompute. parallel must be the value gpx_ep_start was given. tau_tilde, v_tilde: the sites, in and out; out:
 *   the cavity parameters cav_tau, cav_v and the moments Z_hat (= exp log Z_hat), mu_hat, sigma2_hat (N values each).
 *   Sequential updates run in blocks of 128 sites of the order: the block's chain of rank-1 updates on Sigma[I, I] in one
 *   CTA, S = Sigma[:, I] (I + U)^-1 with U[l, j] = c_l s_l[j] (l < j), then Sigma -= S diag(c) S^T on the DMMA GEMM
 *   (GEMM_UPDATE, k-depth 128) and mu -= S g: the reference's chain of DSYR calls, regrouped. _recompute is the Laplace
 *   factor with tau~ in place of W; Sigma = K - D D^T with D = K U~ (sequential) or diag(Sigma) = diag(K) - the squared
 *   column norms of U~^T K (parallel). Launches: 3 per block + 13 + F (sequential), 15 + F (parallel).
 *   gpx_get_stats: solve_ms holds the site updates (chains, solves, rank-128 updates), sweep_ms the factor, update_ms the
 *   recompute's two GEMMs.
 * gpx_ep_finish : _ep_marginal and _inference (:363-395) at the given sites: logdet_B = 2 sum log diag(L_B),
 *   vSv = v~^T Sigma v~ = v~^T K v~ - |U~^T K v~|^2 (Sigma itself is not formed), alpha = v~ - U~ U~^T K v~ (gpx_get(ALPHA),
 *   woodbury_vector), Wi = U~ U~^T (woodbury_inv, gpx_get(KINV)) by the plain LAUUM, diag_dL_dK (N) and kgrad, the
 *   kernel's gradient block (as gpx_laplace_finish's) for dL_dK = 1/2 (alpha alpha^T - Wi). Afterwards gpx_get(DLDK)
 *   returns -2 and gpx_predict, gpx_predictive_gradients, gpx_posterior_covariance and gpx_posterior_samples serve the EP
 *   posterior (gpx_predict does not clip the variance). Launches: 11 + nparts + F. */
int gpx_ep_begin(gpx_ctx* ctx, const gpx_kern_part* parts, int nparts);
int gpx_ep_start(gpx_ctx* ctx, const double* tau_tilde, const double* v_tilde, int warm, int parallel, int max_tries,
                 double* jitter_used);
int gpx_ep_sweep(gpx_ctx* ctx, const int64_t* order, double eta, double delta, int parallel, int max_tries,
                 double* tau_tilde, double* v_tilde, double* cav_tau, double* cav_v, double* Z_hat, double* mu_hat,
                 double* sigma2_hat, double* jitter_used);
int gpx_ep_finish(gpx_ctx* ctx, const double* tau_tilde, const double* v_tilde, int max_tries, double* logdet_B,
                  double* vSv, double* diag_dL_dK, double* kgrad, double* jitter_used);

/* The variational Gaussian approximation (GPy's VarGauss, Opper & Archambeau 2009,
 * GPy/inference/latent_function_inference/var_gauss.py:34-69) for any likelihood, one output column and no mean function:
 * q(f) = N(m, Sigma) with m = K alpha and Sigma = (K^-1 + B^2)^-1, B = diag(beta), alpha and beta (N values each) the
 * variational parameters; beta may be negative. The host evaluates the likelihood's variational expectations (F, dF_dm,
 * dF_dv) at (m, var) between the two entries. The K is kept as gpx_laplace_begin keeps it (the same buffer and release
 * rules). With A = I + B K B factored by jitchol's ladder (the mean of its diagonal is 1 + beta_i^2 Kdiag; jitter_used
 * reports the j it added) and Ai = (A + j I)^-1 = U U^T, U = L_A^-T:
 *
 * gpx_vargauss_begin : K of the parts (every kernel gpx_laplace_begin takes), m = K alpha, A formed from K in one pass with
 *   w = beta and factored; var_i = Sigma_ii = (1 - Ai_ii) / beta_i^2 with Ai_ii the squared norm of row i of U, and
 *   kl = 1/2 (log|A| + tr Ai - N + alpha^T m) (:55). Launches: 7 + F.
 * gpx_vargauss_finish : for dF_dm and dF_dv (N values each) of the last begin: Ai = U U^T by the plain LAUUM;
 *   H = Ai diag(c) Ai, c_i = 1 + 2 dF_dv_i / beta_i^2, on the DMMA GEMM (lower tiles) from a column-scaled copy of Ai; one
 *   fused pass over the lower tiles of Ai and H that sums, per column j, dF_dbeta_j = -2 beta_j sum_i Sigma_ij^2 dF_dv_i and
 *   dKL_dbeta_j = (|e_j - Ai_:j|^2 + j (|Ai_:j|^2 - Ai_jj)) / beta_j (= diag(KB^T (Ai - Ai^2))_j, :57, since
 *   B K B = A - (1 + j) I), and writes S = B (Ai - H) B + r r^T over Ai, r = alpha - dF_dm. Out:
 *     dalpha = K dF_dm - m (:43,:56);
 *     dbeta = dF_dbeta - dKL_dbeta;
 *     kgrad, the kernel's gradient block (as gpx_laplace_finish's) for the symmetric part 1/2 (g g^T - S) of dL_dK,
 *       g = dF_dm, reduced by the exact evaluation's per-part reduction with alpha = g and K^-1 = S. That is the derivative
 *       of the bound. The reference's dF_dK (:66) scales the rows of tmp by dF_dv where the columns belong
 *       (B Ai diag(dF_dv / beta^2) Ai B); the two agree when dF_dv is constant, as for the Gaussian likelihood.
 *   It publishes the posterior: U~ = diag(beta) U in place, woodbury_vector = alpha and woodbury_inv = B Ai B =
 *   (K + B^-2)^-1, which equal the reference's Posterior(mean = m, cov = Sigma, K) in exact arithmetic. Afterwards
 *   gpx_get(K / ALPHA / KINV / L / LINV) return K, alpha, B Ai B, L_A and L_A^-1 B, gpx_get(DLDK) returns -2, and
 *   gpx_predict (it does not clip the variance), gpx_predictive_gradients, gpx_posterior_covariance and
 *   gpx_posterior_samples serve it. finish may be repeated with other dF_dm / dF_dv; as the last one scaled the factor, a
 *   repeated finish factors A again (1 + F more launches). Launches: 8 + nparts.
 * Launch counts exclude F, the factor-and-invert sweep of A, once per attempt of the ladder; none depends on N. Flops: the
 * sweep, N^3 / 3 for the LAUUM and N^3 for the GEMM (N: padded to 128). Peak device memory: five Npad^2 buffers (K, the
 * factor workspace, Ai / S, the scaled copy of Ai and H; 40 Npad^2 bytes, 43 GB at N = 32768); nothing of size N^2 crosses
 * PCIe. gpx_get_stats afterwards: launches, tries, and per-phase times (profile option): kbuild_ms (begin's K-build),
 * sweep_ms (A-build + sweep), update_ms (finish's GEMM), lauum_ms (finish's LAUUM), solve_ms (mat-vecs and the scaling of
 * U), total_ms (the whole call).
 * -2, with nothing touched: a null pointer, a communicator attached, P != 1, a beta entry that is zero or not finite
 * (begin), a finish without a begin on the current data and kernel (any other Laplace or EP call in between counts as
 * another kernel). A value > 0 is A's failing minor after the ladder. */
int gpx_vargauss_begin(gpx_ctx* ctx, const gpx_kern_part* parts, int nparts, const double* alpha, const double* beta,
                       int max_tries, double* m, double* var, double* kl, double* jitter_used);
int gpx_vargauss_finish(gpx_ctx* ctx, const double* dF_dm, const double* dF_dv, double* dalpha, double* dbeta,
                        double* kgrad);

/* Sparse expectation propagation (GPy's EPDTC, expectation_propagation.py:436-611) for the probit Bernoulli likelihood, after
 * gpx_sparse_set_data(X, labels) with P = 1. The sweeps run in M-space: Sigma = Knm A Kmn with A = LLT^-1 (M x M) and
 * mu = mu0 + Knm u, so nothing of size N x N is formed. The kernels are those gpx_sparse_eval_multi takes.
 *   gpx_epdtc_begin  : Kmm (no const jitter), Kmn, Lm = jitchol(Kmm), A0 = Kmm^-1 and diag(Knm Kmm^-1 Kmn); checks the
 *                      labels once per data set ("bad value for Bernoulli observation (0, 1)").
 *   gpx_epdtc_start  : _init_approximations: cold (sites 0, A = A0, Sigma_diag = diag(Qnn) + 1e-8) or warm (the recompute
 *                      from tau_tilde / v_tilde, then + 1e-8). mu / sigma_diag (N each, NULL allowed) receive the
 *                      posteriorParamsDTC the reference holds.
 *   gpx_epdtc_sweep  : one _local_updates pass in the given order, then _recompute (LLT, jitchol's ladder, A, V = L^-1 Kmn,
 *                      Sigma_diag clipped at eps, mu = V^T V v~); arguments as gpx_ep_sweep, plus mu / sigma_diag as above.
 *                      The cavity of a site reads the clipped diagonal the reference holds; the rank-1 algebra the true one.
 *                      Launches: 9 per block of 128 sites (gather, two GEMMs for A Kb and G, a row dot (2), the site chain,
 *                      the solve, GEMM_UPDATE of A, its mirror); 1 per parallel sweep; then 12 for the recompute beyond
 *                      the factor sweep of LLT, and 1 for the clip.
 *   gpx_epdtc_finish : VarDTC at Y = v~ / tau~ and precision tau~ as given (no floor), Kmm = Lm Lm^T from the ladder
 *                      (jitter_used), without log Z~ (the caller adds it): lml, grad (the part blocks in order), dZ (M x D,
 *                      row-major). Afterwards gpx_sparse_get(0..3) and gpx_sparse_predict / _predictive_gradients /
 *                      _posterior_samples serve this posterior.
 * The posterior a sweep updates (A, mu0, u) is that of the sites of the last gpx_epdtc_start or sweep on the context:
 * tau_tilde / v_tilde passed to a sweep must be those sites (the outputs of the previous call, or the warm start's input);
 * the entries do not compare them. finish reads only the sites it is given.
 * Option "epdtc_drift" (gpx_set_option, default 0): a sequential sweep returns diag(Knm A Kmn) of the downdated A after its
 * last block in sigma_diag instead of the recompute's diagonal (2 more launches and M^2 N flops; a measurement of the drift).
 * -2: a communicator attached, P != 1, a null pointer, M < 1, RatQuad / StdPeriodic parts, a call before begin (or a sweep
 * before start). A value > 0 is the leading minor that failed after jitchol's ladder. */
int gpx_epdtc_begin(gpx_ctx* ctx, const gpx_kern_part* parts, int nparts, const double* Z, int64_t M);
int gpx_epdtc_start(gpx_ctx* ctx, const double* tau_tilde, const double* v_tilde, int warm, int parallel, int max_tries,
                    double* jitter_used, double* mu, double* sigma_diag);
int gpx_epdtc_sweep(gpx_ctx* ctx, const int64_t* order, double eta, double delta, int parallel, int max_tries,
                    double* tau_tilde, double* v_tilde, double* cav_tau, double* cav_v, double* Z_hat, double* mu_hat,
                    double* sigma2_hat, double* jitter_used, double* mu, double* sigma_diag);
int gpx_epdtc_finish(gpx_ctx* ctx, const double* tau_tilde, const double* v_tilde, int max_tries, double* lml,
                     double* grad, double* dZ, double* jitter_used);

/* Stochastic variational sparse GP (GPy's SVGP, svgp.py:10-118 with the gradient wiring of core/svgp.py:53-66) with one
 * output column, one latent function and no mean function, for any likelihood: the host evaluates the likelihood's
 * variational expectations (F, dF_dmu, dF_dv) between the two entries. The batch is the rows [row0, row0 + nb) of the data
 * of gpx_sparse_set_data (P = 1), so a step uploads only Z, theta, m and q_L. The kernels are those gpx_sparse_eval_multi
 * takes.
 *   gpx_svgp_begin  : Kmm (no const jitter), Lm = jitchol(Kmm) with max_tries (jitter_used: what the ladder added) and
 *                     logdet Kmm (:38-42); Kmn of the batch; A = Kmm^-1 Kmn as the two triangular products of dpotrs (:45);
 *                     mu = A^T m and var = colsum((q_L^T A)^2) + Kdiag - colsum(A o Kmn) (:46-52), nb each; kl, the KL term
 *                     (:55). q_m: M values; q_L: M x M row-major, read on and below the diagonal (the host expands GPy's
 *                     flat q_u_chol with np.tril_indices(M)); a zero on its diagonal gives kl = +inf and infinite dL_dchol
 *                     entries (the reference's Si). Launches: 14 + F (F: the factor-and-invert sweep of Kmm).
 *   gpx_svgp_finish : the gradients of F.sum() - KL for the batch-scaled dF_dmu and dF_dv (nb each) of the last begin
 *                     (:60-116): grad, the kernel's gradient block (the Kmm, Kmn and Kdiag shares, as gpx_sparse_eval_multi
 *                     orders it); dZ (M x D, row-major); dL_dm (M); dL_dchol (M x M row-major, zero above the diagonal) =
 *                     2 tril((AdvA - Kmm^-1 / 2) q_L) + diag(1 / q_L,ii), which is 2 tril(dL_dS q_L) without forming S^-1.
 *                     It publishes the posterior (woodbury_vector = Kmm^-1 m, woodbury_inv = Kmm^-1 - Kmm^-1 S Kmm^-1
 *                     with Kmm^-1 from the ladder's factor, less j Kmm^-2 when the ladder added j (two more launches),
 *                     posterior.py:166-196 with K = Kmm): afterwards gpx_sparse_get(0..3), gpx_sparse_predict,
 *                     _predictive_gradients and _posterior_samples serve it (gpx_sparse_get(2) is Kmm without the
 *                     ladder's jitter, as the reference's Posterior holds it). It may be repeated with other dF_dmu / dF_dv.
 *                     Launches: 27 for a single kernel, 26 + 2 nparts for a composite.
 * Flops: 8 M^2 NBp on the DMMA GEMM (NBp = nb padded to 128) and 28 M^3 plus the factor sweep (M: padded to 128).
 * Device memory held between the calls: 8 NBp (4 Mpad + 76) bytes for the batch (Kmn in both layouts, A in both layouts
 * and the temporaries that reuse them, four vectors, the prepared points), grown to the largest batch seen, plus
 * 18 Mpad^2 doubles (144 Mpad^2 bytes) of M x M work matrices. Launch counts do not depend on nb. -1 with a message when
 * the batch buffers do not fit.
 * -2, with nothing touched: a null pointer, M < 1, P != 1, a communicator attached, RatQuad / StdPeriodic parts, a row range
 * outside the data, a finish without a begin on the current data, kernel and Z. A value > 0 is the leading minor of Kmm
 * that failed after jitchol's ladder. */
int gpx_svgp_begin(gpx_ctx* ctx, const gpx_kern_part* parts, int nparts, const double* Z, int64_t M, const double* q_m,
                   const double* q_L, int64_t row0, int64_t nb, int max_tries, double* mu, double* var, double* kl,
                   double* jitter_used);
int gpx_svgp_finish(gpx_ctx* ctx, const double* dF_dmu, const double* dF_dv, double* grad, double* dZ, double* dL_dm,
                    double* dL_dchol);

/* Uncertain inputs (Bayesian GPLVM, GPy/models/bayesian_gplvm.py:20-101): the RBF psi-statistics of q(x_n) =
 * N(mu_n, diag(S_n)) (GPy/kern/src/psi_comp/rbf_psi_comp.py:8-136) on the device. The kernel is one RBF part (`parts`,
 * isotropic or ARD) on the latent columns 0 .. Q-1 in order, 1 <= Q <= 16; mu and S are N x Q row-major, S > 0 and
 * finite; Z is M x Q row-major. psi2 is summed over the points; nothing of size N x M x M is formed. Every sum runs in a
 * fixed order, so repeated calls give the same bits. Each entry returns -2 for another kernel, Q out of range, S <= 0 or
 * non-finite, or a null pointer.
 *   gpx_psi_stats : psi1 (N x M row-major, rbf_psi_comp.py:22-34) and psi2 = sum_n psi2_n (M x M, exactly symmetric,
 *                   :36-51); psi0 is the variance. Launches: 4.
 *   gpx_psi_grads : psiDerivativecomputations (:53-136) for dL_dpsi0 (N), dL_dpsi1 (N x M row-major) and dL_dpsi2 (M x M,
 *                   symmetrised as the reference does): grad = [variance, lengthscale (1 or Q)], dZ (M x Q), dmu and dS
 *                   (N x Q), row-major. Launches: 6.
 *   gpx_sparse_eval_psi : VarDTC.inference with uncertain inputs (var_dtc.py:66-215: A = Lm^-1 psi2 Lm^-T beta,
 *                   dL_dpsi0 = -P beta / 2, dL_dpsi1 = beta Y C^T, dL_dpsi2 = beta dL_dpsi2_beta, the homoscedastic
 *                   dL_dR of :258-262) with SparseGP._update_gradients' uncertain branch (core/sparse_gp.py:88-107) and
 *                   gradients_qX_expectations, for the data of gpx_sparse_set_data: its X is mu (D = Q), S is N x Q.
 *                   lml: the bound without the KL term; grad: [variance, lengthscale.., noise variance] with the Kmm part;
 *                   dZ: gradients_X(dL_dKmm, Z) + gradients_Z_expectations (M x Q); dmu, dS: N x Q, without the KL
 *                   gradient. Any P of gpx_sparse_set_data (the wide route above 8). Only O(N Q + M Q) values cross PCIe.
 *                   Afterwards gpx_sparse_get, gpx_sparse_predict, gpx_sparse_predictive_gradients and
 *                   gpx_sparse_posterior_samples serve its posterior at certain test inputs; gpx_sparse_grad_X returns -2.
 *                   Also -2 with a communicator attached or before gpx_sparse_set_data. Launches do not depend on N. */
int gpx_psi_stats(gpx_ctx* ctx, const gpx_kern_part* part, const double* mu, const double* S, int64_t N, const double* Z,
                  int64_t M, int Q, double* psi1, double* psi2);
int gpx_psi_grads(gpx_ctx* ctx, const gpx_kern_part* part, const double* mu, const double* S, int64_t N, const double* Z,
                  int64_t M, int Q, const double* dL_dpsi0, const double* dL_dpsi1, const double* dL_dpsi2, double* grad,
                  double* dZ, double* dmu, double* dS);
int gpx_sparse_eval_psi(gpx_ctx* ctx, const gpx_kern_part* parts, int nparts, const double* S, const double* Z, int64_t M,
                        double noise_variance, double* lml, double* grad, double* dZ, double* dmu, double* dS);

/* Measurement hooks (bench.py): device time of the last eval between CUDA events on the launching stream, the number
 * of kernels this library launched since creation, and per-phase accounting of the last eval. */
typedef struct {
  float total_ms;       /* whole eval, H2D of theta .. D2H of (lml, grad) */
  float kbuild_ms;      /* covariance build kernel */
  float sweep_ms;       /* blocked factor-and-invert sweep (all launches) */
  float update_ms;      /* sum over the outer trailing-update GEMM launches (dominant kernel); on the Ozaki path these launches
                           also accumulate K^-1 = U U^T */
  float lauum_ms;       /* DMMA path: K^-1 = U U^T + fused gradient epilogue; Ozaki path: gradient reductions from the stored K^-1 */
  float solve_ms;       /* alpha / quadratic form */
  double update_flops;  /* algorithmic flops executed by the outer trailing-update launches */
  double lauum_flops;
  double kbuild_bytes;  /* algorithmic bytes of the covariance build (8 N^2 + 8 N D) */
  int64_t launches;     /* kernels launched by the last eval */
  int32_t update_launches;
  int32_t tries;        /* factorisation attempts (1 = no jitter ladder) */
                        /* after a sparse evaluation only update_launches (both M x M factorisations, Kmm's failed attempts
                           included) and tries (of Kmm) are set, the other fields are 0 */
  double update_int8_ops; /* Ozaki path: int8 multiply-add operations (2 per MAC) issued by the update / K^-1 launches, summed
                             over the digit pairs actually computed; 0 on the DMMA path */
} gpx_stats;
int gpx_get_stats(gpx_ctx* ctx, gpx_stats* out);
int64_t gpx_total_launches(gpx_ctx* ctx);
/* Roofline denominator measured on this device: fp64 tensor (DMMA.16x8x4) issue rate in TFLOP/s, CUDA-event timed. */
int gpx_measure_fp64_peak(gpx_ctx* ctx, double* tflops);

/* Tunables, mainly for tests. name is one of
 *   "nb"      outer block size: a multiple of 128, 0 = default: env GPX_NB, else by matrix size. The block is fixed
 *             when the workspace is allocated (gpx_set_data); a later change of GPX_NB takes effect at the next
 *             allocation. The sparse evaluation factors Kmm and B = I + A with the same option,
 *   "profile" 1 (default) = per-phase times in gpx_stats, 0 = total_ms only,
 *   "ozaki"   0 = fp64 DMMA only, 1 = trailing update and K^-1 on the wgmma int8 path where applicable,
 *             -1 = default: env GPX_OZAKI, else 0,
 *   "sparse_wide" 1 = gpx_sparse_set_data takes up to GPX_MAX_OUTPUTS output columns (the sparse wide route), 0 (default)
 *             = at most 8; read by gpx_sparse_set_data only.
 * Any other name fails with "unknown option". */
int gpx_set_option(gpx_ctx* ctx, const char* name, int64_t value);

/* Multi-GPU (one process per GPU). The caller obtains a 128-byte NCCL unique id on rank 0 (gpx_comm_unique_id),
 * ships it to the other ranks with its own plumbing (torch.distributed broadcast), and every rank calls
 * gpx_comm_init. Afterwards gpx_set_data / gpx_exact_eval are collective: block rows are dealt block-cyclically
 * to the ranks, the inverted diagonal block is broadcast and the panel all-gathered (NCCL over NVLink), scalars all-reduced.
 * nranks = 1 is supported: one process on one GPU then runs the same sharded layout and collectives. gpx_comm_init drops
 * the context's data and evaluation (call gpx_set_data again); on a context that already has a communicator it releases
 * that one first. gpx_destroy releases the communicator. */
int gpx_comm_unique_id(char id_out[128]);
int gpx_comm_init(gpx_ctx* ctx, const char id[128], int rank, int nranks);

#ifdef __cplusplus
}
#endif
#endif /* GPX_H_ */
