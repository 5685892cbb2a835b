/*
 * b200gp.h -- C-ABI of libb200gp.so: the H100-native exact-GP posterior path.
 *
 * The reference (ziatdinovmax/gpax v0.1.9) is pure Python on JAX and has no FFI; its two seams on
 * this path are Python callables (SURVEY.md section 8b):
 *   kernel seam     gpax/kernels/kernels.py:17      kernel(X, Z, params, noise, jitter) -> K
 *   posterior seam  gpax/models/gp.py:253-255       get_mvn_posterior(X_new, params, noiseless, **kw)
 * The entry points below are what a ctypes binding placed behind those two callables calls
 * (INTEGRATION.md shows the stub).  Every entry point names the reference lines it replaces.
 *
 * Conventions
 *   - plain C symbols, plain pointers and sizes; no torch / numpy types
 *   - all matrices are fp64, ROW-MAJOR with an explicit leading dimension (elements)
 *   - pointers are HOST pointers unless B2GP_FLAG_DEVICE_PTRS is set in `flags`, in which case every
 *     array argument (not `info`, not `timing`) is a device pointer obtained from b2gp_dev_alloc
 *   - the caller owns every buffer it passes; the library owns only the ctx and its workspaces
 *   - return value: 0 ok, <0 argument / CUDA failure (text via b2gp_last_error).  A numerical failure
 *     is NOT an error status: `info[s] > 0` is the 1-based index of the first non-positive pivot of
 *     draw s and that draw's outputs are NaN (the reference yields NaNs, never an exception, and
 *     post-filters them: gpax/models/gp.py:396-398)
 *   - a ctx is not thread-safe; calls are synchronous from the caller's point of view
 */
#ifndef B200GP_H
#define B200GP_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2GP_VERSION 100

typedef struct b2gp_ctx b2gp_ctx;

/* kernel families: gpax/kernels/kernels.py:44-65 (RBF), 68-91 (Matern-5/2), 94-117 (Periodic);
 * name table gpax/kernels/kernels.py:227-241 */
enum { B2GP_KERNEL_RBF = 0, B2GP_KERNEL_MATERN52 = 1, B2GP_KERNEL_PERIODIC = 2,
       /* NNGP kernels, gpax/kernels/kernels.py:120-224 (erf / ReLU activation): `scale` carries var_w, `period` carries
        * var_b, lengthscale[0] carries the depth.  Taken by b2gp_gram, b2gp_gram_multitask, b2gp_posterior,
        * b2gp_posterior_batch, b2gp_mll and b2gp_mll_v; theta[d+3] = (depth, unused [1, d), var_w, noise, var_b) and the
        * likelihood's grad[d+3] = (0 [0, d), d/dlog var_w, d/dlog noise, d/dlog var_b).  On the posterior and likelihood
        * entry points the depth is an integer in [0, 16] and 1 <= d <= 64.  Every other entry point refuses them. */
       B2GP_KERNEL_NNGP_ERF = 3, B2GP_KERNEL_NNGP_RELU = 4 };

enum {
    B2GP_OK = 0,
    B2GP_ERR_ARG = -1,
    B2GP_ERR_CUDA = -2,
    B2GP_ERR_NOMEM = -3,
    B2GP_ERR_UNSUPPORTED = -4
};

enum {
    B2GP_FLAG_DEVICE_PTRS = 1u << 0, /* array arguments are device pointers                                  */
    B2GP_FLAG_LOWER_ONLY  = 1u << 1, /* b2gp_gram with same_xz: write only the lower triangle (j <= i)       */
    B2GP_FLAG_F32         = 1u << 2, /* b2gp_gram / b2gp_posterior(_batch) / b2gp_sparse_posterior: the DATA arrays (X, Z, y, X_new, Xu,
                                        noise_vec, eps in; K, mean, var, cov, y_sampled out) are float, the reference's default
                                        precision (gpax/utils/utils.py:19-21); theta stays double.  Widened / narrowed on the
                                        device, everything in between is fp64                                  */
    B2GP_FLAG_KPP_DIAG    = 1u << 3, /* b2gp_posterior_gram: Kpp holds only the diagonal of each k_pp, [S, P]; OUT_MEAN / OUT_VAR only */
    B2GP_OUT_MEAN         = 1u << 4, /* b2gp_posterior: produce mean[S,P]                                    */
    B2GP_OUT_VAR          = 1u << 5, /* ... var[S,P] = diag(cov)     (viGP.predict, vigp.py:184-185)         */
    B2GP_OUT_COV          = 1u << 6, /* ... cov[S,P,P]               (get_mvn_posterior, gp.py:272)          */
    B2GP_OUT_SAMPLE       = 1u << 7, /* ... y_sampled[S,n,P] = mean + chol(cov) eps   (gp.py:292)            */
    B2GP_OUT_DMEAN        = 1u << 8, /* the *_grad posteriors: dmean[S,P,d] = d mean[s,p] / d Xnew[p,:]      */
    B2GP_OUT_DVAR         = 1u << 9  /* ... dvar[S,P,d] = d var[s,p] / d Xnew[p,:]                            */
};

/* per-call device timing (CUDA events on the library's own streams), filled when non-NULL.
 * The *_ms stage fields are sums of stream time over the draws (they can exceed total_ms when
 * several draws are in flight); total_ms is first-launch to last-completion on the device,
 * h2d/d2h are the host<->device copies of the host-pointer entry points. */
typedef struct b2gp_timing {
    double total_ms;
    double gram_ms;
    double potrf_ms;
    double trsm_ms;
    double epilogue_ms;
    double h2d_ms;
    double d2h_ms;
    double flops;        /* algorithmic flops of the call: S * (N^3/3 + N^2 (P+1) + ...)  (SURVEY.md 8d) */
    double gram_bytes;   /* algorithmic bytes written by the Gram builds                                 */
    int64_t launches;    /* kernels launched by the call                                                 */
    double host_enqueue_ms; /* host wall time spent issuing the call's work (before waiting for the device)  */
} b2gp_timing;

int  b2gp_version(void);

/* lifecycle --------------------------------------------------------------------------------------
 * One context = one CUDA device = one process per GPU.  (SURVEY.md 8b sketched `b2gp_ctx_create(n_dev, dev_ids, out)` with
 * ncclCommInitAll inside one process; the multi-GPU forms of the path run one process per GPU instead and join their
 * contexts with b2gp_dist_init below.) */
int  b2gp_ctx_create(int device, b2gp_ctx** out);
int  b2gp_ctx_destroy(b2gp_ctx* ctx);
const char* b2gp_last_error(const b2gp_ctx* ctx);
/* options: "streams" (draws in flight, 1..16, default 2); "ozaki" (0: fp64 DMMA only, 6 / 7: int8 wgmma base-256 digit
 * planes, -1: 6 or 7 chosen per call from a bound on cond(K); default 0); the full table is in INTEGRATION.md */
int  b2gp_set_option(b2gp_ctx* ctx, const char* key, int64_t value);
/* the current value of any option that holds one (every key of the table except the action "drop_factor_cache") */
int  b2gp_get_option(b2gp_ctx* ctx, const char* key, int64_t* value);
int  b2gp_device_info(b2gp_ctx* ctx, int* sm_count, int* cc_major, int* cc_minor, size_t* mem_bytes);
/* device timing of the most recent entry-point call on this ctx (every call records total_ms) */
int  b2gp_last_timing(b2gp_ctx* ctx, b2gp_timing* out);

/* device memory, for callers that keep inputs resident in HBM (replaces jax.device_put,
 * gpax/models/gp.py:388-391,416-428) ----------------------------------------------------------------*/
int  b2gp_dev_alloc(b2gp_ctx* ctx, size_t bytes, void** dptr);
int  b2gp_dev_free(b2gp_ctx* ctx, void* dptr);
int  b2gp_host_alloc(b2gp_ctx* ctx, size_t bytes, void** hptr);   /* pinned host memory */
int  b2gp_host_free(b2gp_ctx* ctx, void* hptr);
int  b2gp_h2d(b2gp_ctx* ctx, void* dst_dev, const void* src_host, size_t bytes);
int  b2gp_d2h(b2gp_ctx* ctx, void* dst_host, const void* src_dev, size_t bytes);
int  b2gp_sync(b2gp_ctx* ctx);

/* Gram build -- replaces square_scaled_distance + RBFKernel / MaternKernel / PeriodicKernel
 * (gpax/kernels/kernels.py:28-41, 44-65, 68-91, 94-117).
 *   X[n,d], Z[m,d] row-major; lengthscale[d] (a scalar lengthscale is broadcast by the caller);
 *   K[n,m] with leading dimension ldk.  `diag_add` = noise + jitter is added on i == j iff
 *   same_xz != 0; the caller sets same_xz from the reference's rule `X.shape == Z.shape`
 *   (kernels.py:63, 89, 115).  `period` is read for B2GP_KERNEL_PERIODIC only.                     */
int  b2gp_gram(b2gp_ctx* ctx, int kind,
               const double* X, int64_t n, const double* Z, int64_t m, int d,
               const double* lengthscale, double scale, double period,
               double diag_add, int same_xz,
               double* K, int64_t ldk, unsigned flags);

/* Multi-task Gram matrix -- gpax/kernels/mtkernels.py:19-58 (index_kernel) and 61-125 (MultitaskKernel):
 * K[i,j] = (k_data(x_i, z_j) + jitter if same point) * B[taskX[i], taskZ[j]], plus noise_task[taskX[i]] + jitter on i == j,
 * both iff same_xz (the reference's shape rule).  B[T,T] = W W^T + diag(v) is formed by the caller.  Host fp64 / int32
 * arrays.  The Kronecker form of MultivariateKernel (mtkernels.py:128-192) is this call on inputs repeated once per
 * task with group = T (`group` consecutive rows are one data point; 1 otherwise).                                     */
int  b2gp_gram_multitask(b2gp_ctx* ctx, int kind, const double* X, const int* taskX, int64_t n,
                         const double* Z, const int* taskZ, int64_t m, int d,
                         const double* lengthscale, double scale, double period,
                         const double* B, int T, const double* noise_task, double jitter, int same_xz, int group,
                         double* K, int64_t ldk, unsigned flags);

/* Cholesky factorisation A = L L^T of the lower triangle, in place (row-major, lower); the strict
 * upper triangle is not referenced and not modified.  Stands where the reference inverts k_XX
 * (jnp.linalg.inv, gpax/models/gp.py:271) and where viSparseGP calls jax.scipy.linalg.cholesky
 * (gpax/models/sparse_gp.py:194,201).  *info = 0, or the 1-based index of the first bad pivot.      */
int  b2gp_potrf(b2gp_ctx* ctx, int64_t n, double* A, int64_t lda, int* info, unsigned flags);

/* Triangular solve with the factor: overwrites the nrhs right-hand sides with L^{-1} b.
 * B holds one right-hand side per ROW: B[r, 0..n) is b_r, leading dimension ldb (i.e. the n x nrhs
 * matrix of right-hand sides in column-major order).  Replaces solve_triangular(L, ., lower=True)
 * (gpax/models/sparse_gp.py:197,207,209) and the K^{-1} products of gp.py:272-273.
 * L must be the output of b2gp_potrf made through the same ctx immediately before (the solve
 * reuses the inverted diagonal blocks that factorisation left in the ctx).                          */
int  b2gp_trsm_lower(b2gp_ctx* ctx, int64_t n, int64_t nrhs,
                     const double* L, int64_t ldl, double* B, int64_t ldb, unsigned flags);

/* C[m,n] = beta C + alpha A[m,k] B[n,k]^T (fp64, DMMA tensor pipe); lower_only != 0 updates only
 * j <= i (SYRK when A == B) and needs m >= n: with m > n that is the lower triangle of the leading
 * n x n block plus all n columns of the rows below it (the trapezoid the factorisation updates when
 * right-hand-side rows ride under the matrix).  The trailing-update kernel of the factorisation, exported for the
 * roofline measurement and the parity tests; replaces the jnp.matmul calls of gp.py:272-273.       */
int  b2gp_gemm_nt(b2gp_ctx* ctx, int64_t m, int64_t n, int64_t k, double alpha,
                  const double* A, int64_t lda, const double* B, int64_t ldb,
                  double beta, double* C, int64_t ldc, int lower_only, unsigned flags);

/* The posterior, batched over S hyper-parameter draws -- replaces ExactGP.get_mvn_posterior
 * (gpax/models/gp.py:253-277), _predict's sampling (gp.py:279-293), the vmap over draws in predict
 * (gp.py:393-395) and viGP.predict (gpax/models/vigp.py:178-185).
 *   Xtr[N,d], Xnew[P,d]                    row-major
 *   yres[N] (yres_stride == 0) or yres[S, yres_stride]   y_train minus the mean function (gp.py:262-265)
 *   theta[S, d+3]                          per draw: lengthscale[0..d), k_scale, noise, period
 *   noiseless                              gp.py:260-261: noise_p = noise * (1 - noiseless)
 *   jitter                                 the **kwargs jitter of gp.py:267,269 (default 1e-6)
 *   flags                                  B2GP_OUT_* (+ B2GP_FLAG_DEVICE_PTRS)
 *   mean[S,P], var[S,P], cov[S,P,P]        outputs selected by flags (others may be NULL)
 *   eps[S,n_samp,P], y_sampled[S,n_samp,P] standard-normal draws in, posterior samples out
 *   info[S]                                0 or first bad pivot of k_XX (>0) / of cov (<0, sampling)  */
int  b2gp_posterior(b2gp_ctx* ctx, int kind,
                    const double* Xtr, int64_t N, const double* yres, int64_t yres_stride,
                    const double* Xnew, int64_t P, int d, int64_t S,
                    const double* theta, int noiseless, double jitter, unsigned flags,
                    double* mean, double* var, double* cov,
                    const double* eps, int64_t n_samp, double* y_sampled,
                    int* info, b2gp_timing* timing);

/* The same posterior with everything that may differ between the S members of the batch (SURVEY.md section 8f-3):
 *   Xtr[S, xtr_stride] / Xnew[S, xnew_stride]   per-member training / test inputs (stride in doubles; 0 = shared [N,d] / [P,d]):
 *       the outer task axis of vExactGP (gpax/models/vgp.py:125-172) and the per-draw perturbed inputs X_prime of
 *       UIGP (gpax/models/uigp.py:131-150)
 *   noise_vec[N] or [S, noise_vec_stride]       per-point noise variances added to the diagonal of k_XX on top of
 *       theta's scalar noise: MeasuredNoiseGP (k + diag(measured_noise), gpax/models/mngp.py:92-97) and VarNoiseGP
 *       (k + diag(exp(log_var)), gpax/models/hskgp.py:143-148); NULL = none.
 * All other arguments as b2gp_posterior.                                                                          */
int  b2gp_posterior_batch(b2gp_ctx* ctx, int kind,
                          const double* Xtr, int64_t xtr_stride, int64_t N, const double* yres, int64_t yres_stride,
                          const double* Xnew, int64_t xnew_stride, int64_t P, int d, int64_t S,
                          const double* theta, const double* noise_vec, int64_t noise_vec_stride,
                          int noiseless, double jitter, unsigned flags,
                          double* mean, double* var, double* cov,
                          const double* eps, int64_t n_samp, double* y_sampled,
                          int* info, b2gp_timing* timing);

/* The posterior and its gradient w.r.t. the test inputs -- what jax.grad of the acquisition w.r.t. x needs in
 * gpax/acquisition/optimize.py:70-88 (optimize_acq).  Arguments as b2gp_posterior; flags: any of B2GP_OUT_MEAN,
 * B2GP_OUT_VAR, B2GP_OUT_DMEAN, B2GP_OUT_DVAR, plus B2GP_FLAG_DEVICE_PTRS.  B2GP_FLAG_F32, B2GP_OUT_COV and B2GP_OUT_SAMPLE
 * give B2GP_ERR_UNSUPPORTED.  Kinds RBF, Matern-5/2, Periodic.
 *   dmean[S,P,d]  d mean[s,p] / d Xnew[p,k]
 *   dvar[S,P,d]   d var[s,p]  / d Xnew[p,k]   (k(x, x) is constant, so the same with and without noiseless)
 * The P*d rows d k(Xnew[p], X) / d Xnew[p,k] are solved with the factor of k_XX like k_pX.  mean and var are those of
 * b2gp_posterior for the same inputs, bit for bit under the default "ozaki" = 0.  Under the int8 options (ozaki != 0) the
 * extra rows can move a GEMM of the factorisation or solve to the other side of a dispatch threshold (trsm_rec's
 * 1024-row panel route, the "oz_min_tiles" tile count); mean and var then agree within the digit-plane error.  NaN
 * outputs where info[s] != 0.  Single-draw host-pointer calls share the factor cache of b2gp_posterior.              */
int  b2gp_posterior_grad(b2gp_ctx* ctx, int kind, const double* Xtr, int64_t N, const double* yres, int64_t yres_stride,
                         const double* Xnew, int64_t P, int d, int64_t S, const double* theta, int noiseless, double jitter,
                         unsigned flags, double* mean, double* var, double* dmean, double* dvar,
                         int* info, b2gp_timing* timing);

/* The posterior of MultiTaskGP / CoregGP -- gp.py:253-293 (get_mvn_posterior / _predict) with the linear model of
 * coregionalisation of gpax/kernels/mtkernels.py:197-233 in place of the single-task kernel (gpax/models/mtgp.py,
 * corgp.py).  For latent q = 0..L-1, with B_q = W_q W_q^T + diag(v_q) (mtkernels.py:60-63):
 *     K[i,j] = sum_q (k_q(x_i, x_j) + jitter [same point]) B_q[t_i, t_j]  +  [i == j] L (noise[t_i] + jitter)
 * -- the noise and jitter are added once per latent, as the reference's vmap over the latents does (:228-231); k_pX
 * carries no diagonal term (gp.py:268); noiseless scales only the noise of k_pp (gp.py:260-267).
 *   Xtr[N,d], task_tr[N]    training inputs and their task ids (int32 in [0, T), checked before any launch)
 *   Xnew[P,d], task_new[P]  test inputs and their task ids.  N and P count rows: the Kronecker form of
 *                           MultivariateKernel (mtkernels.py:163-192) repeats every input T times, task index cycling
 *                           fastest, with group = T (`group` consecutive rows are one data point); group = 1 otherwise
 *   theta[S,L,d+2]          per draw and latent: lengthscale[d], k_scale, period (read for Periodic only)
 *   B[S,L,T,T], noise[S,T]  task covariances and per-task noise variances
 * Other arguments and outputs as b2gp_posterior.  Limits: T <= 8, L <= 4, d <= 16.  Kinds RBF, Matern-5/2, Periodic.
 * Host fp64 arrays only: B2GP_FLAG_DEVICE_PTRS and B2GP_FLAG_F32 give B2GP_ERR_UNSUPPORTED.  The call does not use or
 * fill the factor cache of b2gp_posterior; under "ozaki" = -1 it takes 7 digit planes.                                */
int  b2gp_posterior_multitask(b2gp_ctx* ctx, int kind, const double* Xtr, const int* task_tr, int64_t N, const double* yres,
                              int64_t yres_stride, const double* Xnew, const int* task_new, int64_t P, int d, int group, int T,
                              int L, int64_t S, const double* theta, const double* B, const double* noise, int noiseless,
                              double jitter, unsigned flags, double* mean, double* var, double* cov, const double* eps,
                              int64_t n_samp, double* y_sampled, int* info, b2gp_timing* timing);

/* The posterior of b2gp_posterior_multitask and its gradient w.r.t. the test inputs -- what jax.grad of the acquisition
 * w.r.t. x needs in gpax/acquisition/optimize.py:70-88 (optimize_acq) on a MultiTaskGP / CoregGP.  Arguments as
 * b2gp_posterior_multitask without cov / eps / n_samp / y_sampled; flags: any of B2GP_OUT_MEAN, B2GP_OUT_VAR,
 * B2GP_OUT_DMEAN, B2GP_OUT_DVAR.  B2GP_FLAG_F32, B2GP_FLAG_DEVICE_PTRS, B2GP_OUT_COV and B2GP_OUT_SAMPLE give
 * B2GP_ERR_UNSUPPORTED; kinds, limits (T <= 8, L <= 4, d <= 16) and task ids are checked as there, before any launch.
 *   dmean[S,P,d]  d mean[s,p] / d Xnew[p,k]
 *   dvar[S,P,d]   d var[s,p]  / d Xnew[p,k]   (the prior diagonal sum_q (k_q(x,x) + jitter) B_q[t,t] + L (noise[t] +
 *                 jitter) does not depend on x for the three kinds, so the same with and without noiseless)
 * with P and d counting GP rows and data features: each row is differentiated w.r.t. its own inputs, the Kronecker form's
 * repeated rows included; the task ids are constants.  The P*d rows sum_q B_q[t_p, t_i] d k_q(Xnew[p], X[i]) / d Xnew[p,k]
 * are solved with the factor of k_XX like k_pX.  mean and var are those of b2gp_posterior_multitask for the same inputs,
 * bit for bit under the default "ozaki" = 0.  Under the int8 options (ozaki != 0) the extra rows can move a GEMM of the
 * factorisation or solve to the other side of a dispatch threshold (trsm_rec's 1024-row panel route, the "oz_min_tiles"
 * tile count); mean and var then agree within the digit-plane error.  NaN outputs where info[s] != 0; the other draws
 * are unaffected.  Identical calls give identical bits.  No factor cache, as b2gp_posterior_multitask.                 */
int  b2gp_posterior_multitask_grad(b2gp_ctx* ctx, int kind, const double* Xtr, const int* task_tr, int64_t N,
                                   const double* yres, int64_t yres_stride, const double* Xnew, const int* task_new, int64_t P,
                                   int d, int group, int T, int L, int64_t S, const double* theta, const double* B,
                                   const double* noise, int noiseless, double jitter, unsigned flags, double* mean, double* var,
                                   double* dmean, double* dvar, int* info, b2gp_timing* timing);

/* The posterior of b2gp_posterior_batch with the Gram blocks supplied by the caller: the route of a user kernel callable
 * k(X, Z, params, noise, jitter) (gpax/kernels/kernels.py:227-241; gp.py:267-269).  Per draw s:
 *   Kxx[s * kxx_stride]  [N, N]  k_XX = kernel(X, X, params_s, noise_s, jitter); the library factors its symmetric part
 *                                (K + K^T) / 2, as the reference's Cholesky does
 *   Kpx[s * kpx_stride]  [P, N]  k_pX = kernel(X_new, X, params_s, jitter=0.0)
 *   Kpp[s * kpp_stride]  [P, P]  k_pp = kernel(X_new, X_new, params_s, noise_p, jitter) -- its lower triangle is read, and
 *                                var is taken as diag(k_pp) - |v_p|^2.  With B2GP_FLAG_KPP_DIAG: only diag(k_pp), [P]
 *                                per draw, and the outputs are limited to mean / var.  May be NULL for mean-only calls.
 * Strides are in doubles between draws, 0 = shared.  yres, flags (B2GP_OUT_* and B2GP_FLAG_DEVICE_PTRS, which covers the
 * Gram blocks too), outputs, eps and info as b2gp_posterior_batch.  B2GP_FLAG_F32 gives B2GP_ERR_UNSUPPORTED.  The call
 * neither uses nor fills the factor cache; under "ozaki" = -1 it takes 7 digit planes (the cond(K) bound needs k_scale). */
int  b2gp_posterior_gram(b2gp_ctx* ctx, const double* Kxx, int64_t kxx_stride, int64_t N,
                         const double* Kpx, int64_t kpx_stride, const double* Kpp, int64_t kpp_stride, int64_t P, int64_t S,
                         const double* yres, int64_t yres_stride, unsigned flags,
                         double* mean, double* var, double* cov, const double* eps, int64_t n_samp, double* y_sampled,
                         int* info, b2gp_timing* timing);

/* Nystrom / VFE sparse posterior for one theta -- replaces viSparseGP.get_mvn_posterior
 * (gpax/models/sparse_gp.py:173-223).  Xu[M,d] inducing points; theta[d+3] as above;
 * outputs mean[P] and var[P] (B2GP_OUT_VAR) and/or cov[P,P] (B2GP_OUT_COV).                        */
int  b2gp_sparse_posterior(b2gp_ctx* ctx, int kind,
                           const double* Xu, int64_t M, const double* Xtr, int64_t N, const double* yres,
                           const double* Xnew, int64_t P, int d,
                           const double* theta, int noiseless, double jitter, unsigned flags,
                           double* mean, double* var, double* cov,
                           int* info, b2gp_timing* timing);

/* The posterior of b2gp_sparse_posterior with the Gram blocks supplied by the caller: the route of a user kernel callable
 * k(X, Z, params, noise, jitter) in viSparseGP.get_mvn_posterior (gpax/models/sparse_gp.py:173-223):
 *   Kuu [M, M]  kernel(Xu, Xu, params, **kwargs); the library factors (Kuu + Kuu^T) / 2 and adds no jitter (it is in Kuu)
 *   Kuf [M, N]  kernel(Xu, X_train, params, jitter=0)
 *   Kus [M, P]  kernel(Xu, X_new, params, jitter=0)
 *   Kss [P, P]  kernel(X_new, X_new, params, noise_p, **kwargs) (noise_p already inside); its lower triangle is read.
 *               With B2GP_FLAG_KPP_DIAG only its diagonal [P], and the outputs are limited to mean / var.  May be NULL for
 *               mean-only calls.
 * yres [N] and `noise` (the D = noise 1 of sparse_gp.py:191-192) as b2gp_sparse_posterior; every block follows `flags`
 * (B2GP_FLAG_DEVICE_PTRS; B2GP_FLAG_F32 gives B2GP_ERR_UNSUPPORTED).  Outputs, info and timing as b2gp_sparse_posterior. */
int  b2gp_sparse_posterior_gram(b2gp_ctx* ctx, const double* Kuu, int64_t M, const double* Kuf, int64_t N, const double* yres,
                                double noise, const double* Kus, const double* Kss, int64_t P, unsigned flags,
                                double* mean, double* var, double* cov, int* info, b2gp_timing* timing);

/* Fit side (SURVEY.md section 8f-1): value and gradient of the exact-GP log marginal likelihood
 *   log N(yres; 0, K_theta),  K_theta = kernel(X, X, theta, noise, jitter)
 * i.e. the numpyro.sample("y", MultivariateNormal(f_loc, covariance_matrix=k), obs=y) term of
 * gpax/models/gp.py:158-164 and its reverse-mode derivative.  grad[d+3] is w.r.t. (log lengthscale[0..d),
 * log k_scale, log noise, log period); theta (d+3) is a HOST pointer; value, grad, alpha_out[N] = K^{-1} yres
 * (optional) are HOST outputs; X, yres follow `flags`.  d <= 16.                                          */
int  b2gp_mll(b2gp_ctx* ctx, int kind, const double* X, int64_t N, const double* yres, int d,
              const double* theta, double jitter, unsigned flags,
              double* value, double* grad, double* alpha_out, int* info);

/* b2gp_mll with a vector of per-point noise variances on the diagonal, K = kernel(X, X, theta, noise, jitter) + diag(noise_vec)
 * (the likelihoods of gpax/models/mngp.py:92-97 and gpax/models/hskgp.py:143-148), and grad_noise_vec[N] (HOST, optional,
 * needs grad) = d value / d noise_vec[i] = 1/2 (alpha_i^2 - K^{-1}_ii).                                              */
int  b2gp_mll_v(b2gp_ctx* ctx, int kind, const double* X, int64_t N, const double* yres, int d,
                const double* theta, const double* noise_vec, double jitter, unsigned flags,
                double* value, double* grad, double* alpha_out, double* grad_noise_vec, int* info);

/* The likelihood and its gradient from caller-supplied matrices (a user kernel callable's fit):
 *   value   = log N(yres; 0, K)  with K[N, N] (leading dimension ldk) factored as its symmetric part (K + K^T) / 2
 *   grad[j] = 1/2 sum_{a,b} (alpha alpha^T - K^{-1})_{ab} dK_j[a, b],  j < p,  alpha = K^{-1} yres
 * dK is a HOST array of p pointers to N x N matrices (leading dimension lddk); no symmetry is assumed of them.  K, yres and
 * every dK_j are host arrays, or device arrays under B2GP_FLAG_DEVICE_PTRS; host dK_j are streamed through two device
 * buffers, so p is limited by host memory only.  grad[p] and alpha_out[N] are optional HOST outputs (p = 0 or grad = NULL:
 * no gradient).  The factorisation and solves are those of b2gp_mll (every "ozaki" / tall-panel route); the trace runs in
 * a fixed order, so identical calls give identical bits.  NaN value and gradient where info != 0.  B2GP_FLAG_F32 gives
 * B2GP_ERR_UNSUPPORTED.                                                                                                  */
int  b2gp_mll_gram(b2gp_ctx* ctx, const double* K, int64_t N, int64_t ldk, const double* yres,
                   const double* const* dK, int64_t lddk, int64_t p, unsigned flags,
                   double* value, double* grad, double* alpha_out, int* info);

/* The likelihood of MultiTaskGP.model / CoregGP.model (gpax/models/mtgp.py:147-167, corgp.py:66-98): log N(yres; 0, K)
 * with K the LCM covariance of b2gp_posterior_multitask (X[N,d], task[N], group, T, L, theta[L,d+2], B[L,T,T], noise[T]
 * as there, one draw), and its gradient (HOST outputs, all three or none):
 *   grad_theta[L,d+2]  d value / d log(lengthscale_q[k], k_scale_q, period_q)
 *   grad_B[L,T,T]      d value / d B_q[a,b] with the entries of B_q taken as independent (symmetric); the chain rule to
 *                      W_q and v_q is (grad_B_q + grad_B_q^T) W_q and diag(grad_B_q)
 *   grad_noise[T]      d value / d log noise[t]
 * and alpha_out[N] = K^{-1} yres.  The reduction runs in a fixed order: identical calls give identical bits.  Limits,
 * kinds and refused flags as b2gp_posterior_multitask; NaN value and gradient where info != 0.                         */
int  b2gp_mll_multitask(b2gp_ctx* ctx, int kind, const double* X, const int* task, int64_t N, const double* yres, int d,
                        int group, int T, int L, const double* theta, const double* B, const double* noise, double jitter,
                        unsigned flags, double* value, double* grad_theta, double* grad_B, double* grad_noise,
                        double* alpha_out, int* info);

/* Fit side of the sparse GP: the VFE bound of viSparseGP.model (gpax/models/sparse_gp.py:62-114)
 *   log LowRankMVN(yres; 0, W^T W + noise I) - 1/2 clip(sum_n (Kff_nn - Qff_nn) / noise, 0),  W = Luu^{-1} K(Xu, X)
 * and its gradient w.r.t. (log lengthscale[d], log k_scale, log noise, log period) in grad_theta[d+3] and w.r.t. the
 * inducing inputs in grad_Xu[M,d] (the reference differentiates the same expression with JAX; Xu is a numpyro.param,
 * sparse_gp.py:69-70).  theta is a HOST pointer; value / grads are HOST outputs; Xu, X, yres follow `flags`. d <= 16.
 * info = the first bad pivot of Kuu + jitter I, or minus that of I + W W^T / noise; NaN value, grad_theta and grad_Xu
 * where info != 0.                                                                                                    */
int  b2gp_sparse_elbo(b2gp_ctx* ctx, int kind, const double* Xu, int64_t M, const double* X, int64_t N,
                      const double* yres, int d, const double* theta, double jitter, unsigned flags,
                      double* value, double* grad_theta, double* grad_Xu, int* info);

/* b2gp_sparse_elbo plus alpha_out[N] (HOST, optional) = (W^T W + noise I)^{-1} yres, the derivative of the bound w.r.t.
 * the mean vector subtracted from y (sparse_gp.py:71-88's f_loc).  b2gp_sparse_elbo is this call with alpha_out = NULL;
 * the other outputs are the same bits either way.  NaN alpha_out where info != 0.                                    */
int  b2gp_sparse_elbo_ex(b2gp_ctx* ctx, int kind, const double* Xu, int64_t M, const double* X, int64_t N,
                         const double* yres, int d, const double* theta, double jitter, unsigned flags,
                         double* value, double* grad_theta, double* grad_Xu, double* alpha_out, int* info);

/* The bound of b2gp_sparse_elbo from caller-supplied blocks (a user kernel callable's fit, sparse_gp.py:88-103):
 *   Kuu [M, M]     kernel(Xu, Xu, params, jitter=jitter), factored as (Kuu + Kuu^T) / 2; the library adds no jitter
 *   Kuf [M, N]     kernel(Xu, X, params)
 *   kff_diag [N]   diag(kernel(X, X, params, jitter=0)); the trace term is sum kff_diag - |W|_F^2, clipped at 0
 * and yres [N], noise.  Outputs (HOST):
 *   value            the bound
 *   grad[j]          sum Gs * dKuu[j] + sum Guf * dKuf[j] + g_d sum dkff[j],  j < p, where Gs (M x M, symmetric) and
 *                    Guf (M x N) are the adjoints of the bound w.r.t. the symmetrised Kuu and Kuf, g_d = -coef / (2 noise)
 *                    and coef = 1 when the trace term is positive, else 0
 *   grad_log_noise   d value / d log noise (optional)
 *   grad_rows[k, m]  sum_i Gs[m, i] rKuu[k][m, i] + sum_n Guf[m, n] rKuf[k][m, n],  k < q: with rKuu_k, rKuf_k the
 *                    derivatives of Kuu and Kuf w.r.t. Xu[:, k] (row m moving with Xu[m, k]), d value / d Xu[m, k]
 *   alpha_out[N]     (W^T W + noise I)^{-1} yres (optional)
 * dKuu, dKuf, dkff (p each), rKuu, rKuf (q each) are HOST arrays of pointers; any of them, and any entry, may be NULL (a
 * zero block).  No symmetry is assumed of the direction blocks.  Every block is a host array, or a device array under
 * B2GP_FLAG_DEVICE_PTRS; host direction blocks are streamed through two device buffers.  The contraction runs in a fixed
 * order, so identical calls give identical bits.  info as b2gp_sparse_elbo; NaN outputs where info != 0.  B2GP_FLAG_F32
 * gives B2GP_ERR_UNSUPPORTED.                                                                                          */
int  b2gp_sparse_elbo_gram(b2gp_ctx* ctx, const double* Kuu, int64_t M, const double* Kuf, int64_t N, const double* kff_diag,
                           const double* yres, double noise, const double* const* dKuu, const double* const* dKuf,
                           const double* const* dkff, int64_t p, const double* const* rKuu, const double* const* rKuf,
                           int64_t q, unsigned flags, double* value, double* grad, double* grad_log_noise, double* grad_rows,
                           double* alpha_out, int* info);

/* ---- deep kernel learning (gpax/models/vidkl.py, gpax/models/dkl.py) ---------------------------------------------
 * The feature extractor is a dense MLP, H_{l+1} = act(H_l W_l + b_l) with no activation after the last layer.
 * params, per layer l: W_l[in_l, out_l] row-major (haiku's and dkl.py's orientation), then b_l[out_l];
 * widths[n_layers] are the output widths, the last one is z_dim = d <= 16; in_0 = D.                                  */
enum { B2GP_ACT_RELU = 0, B2GP_ACT_TANH = 1 };

/* Z[s] = MLP(X; params + s * params_stride) for S weight sets: Z [S, N, d] (HOST).  X follows `flags`; params and
 * widths are HOST pointers.  n_layers = 0 copies X (D = d).                                                          */
int  b2gp_mlp_forward(b2gp_ctx* ctx, const double* X, int64_t N, int64_t D, int n_layers, const int64_t* widths, int act,
                      const double* params, int64_t S, int64_t params_stride, double* Z, unsigned flags);

/* log N(yres; 0, K(z)) on the embedding z = MLP(X) (the likelihood of viDKL.model / DKL.model) with its gradient:
 *   value, grad_theta[d+3]  as b2gp_mll on the same z (same kernels, same bits), d / dlog theta
 *   grad_z[N, d]            d value / d z (optional); with n_layers = 0 this is d value / d X
 *   grad_params             d value / d params in the params layout (optional)
 * X and yres follow `flags` (a fit uploads X once); theta, params and every output are HOST pointers.  NaN outputs where
 * info != 0.  The reductions run in a fixed order: identical calls give identical bits.                              */
int  b2gp_dkl_mll(b2gp_ctx* ctx, int kind, const double* X, int64_t N, int64_t D, const double* yres,
                  int n_layers, const int64_t* widths, int act, const double* params,
                  const double* theta, double jitter, unsigned flags,
                  double* value, double* grad_theta, double* grad_params, double* grad_z, int* info);

/* The posterior of viDKL / DKL and its gradient w.r.t. the RAW test inputs -- what jax.grad of the acquisition w.r.t. x
 * takes through the network in gpax/acquisition/optimize.py:70-88 (vidkl.py:206-236, dkl.py:113-132 under the grad).
 * For S weight sets (params + s * params_stride) and theta[S, d+3]:
 *   1. X[N,D] and Xnew[P,D] are embedded per weight set as b2gp_mlp_forward does (same kernels, same bits);
 *   2. b2gp_posterior_grad runs on the embeddings (per-draw embeddings when S > 1), dmean_z / dvar_z [S,P,d];
 *   3. one launch pulls them back through the network: dX = J_MLP(x)^T d/dz (mlp_input_vjp_kernel, dkl.cuh).
 * Outputs (HOST): mean / var [S,P] and dmean / dvar [S,P,D], any subset by B2GP_OUT_MEAN / VAR / DMEAN / DVAR; info[S].
 * yres / yres_stride, noiseless and jitter as b2gp_posterior.  mean and var are those of b2gp_posterior on the
 * b2gp_mlp_forward embeddings, on the same route.  n_layers = 0 is b2gp_posterior_grad on X (D = d).  Kinds RBF,
 * Matern-5/2, Periodic; host fp64 arrays only: B2GP_FLAG_F32, B2GP_FLAG_DEVICE_PTRS, B2GP_OUT_COV and B2GP_OUT_SAMPLE
 * give B2GP_ERR_UNSUPPORTED.  S = 1 calls share the factor cache of b2gp_posterior (the key includes the training
 * embedding's bits): nothing this call runs besides the posterior touches the cached factor, so a repeated call with
 * the same weights, theta and training set solves against the cached factor.  NaN outputs where info[s] != 0; the other
 * draws are unaffected.  The pull-back runs in a fixed order: identical calls give identical bits.  b2gp_last_timing
 * reports the whole call (total_ms its wall time).                                                                     */
int  b2gp_dkl_posterior_grad(b2gp_ctx* ctx, int kind, const double* X, int64_t N, int64_t D, const double* yres,
                             int64_t yres_stride, const double* Xnew, int64_t P, int n_layers, const int64_t* widths, int act,
                             const double* params, int64_t S, int64_t params_stride, const double* theta, int noiseless,
                             double jitter, unsigned flags, double* mean, double* var, double* dmean, double* dvar, int* info);

/* B independent exact-GP likelihoods (the per-task likelihoods of vExactGP.model, gpax/models/vgp.py:55-89, and the one
 * of UIGP.model with its input gradient, uigp.py:78-107).  X[B,N,d], yres[B,N], theta[B,d+3]: member b's arrays, layouts
 * as b2gp_mll.  HOST outputs: value[B]; grad[B,d+3] (optional) d value / dlog theta; alpha_out[B,N] (optional) K^{-1} yres;
 * grad_x[B,N,d] (optional, needs grad) d value / dX; info[B].  Member b returns what b2gp_mll and
 * b2gp_dkl_mll(n_layers = 0) return on member b.  A member with info[b] != 0 has NaN outputs; the others are unaffected.
 *   N <= B2GP_MLL_BATCH_SMALL_MAX_N: one launch for the whole batch, one CTA per member that factors, inverts and reduces
 *            in shared memory (gpax_b200/csrc/mll_batch.cuh); counted by the route counter mll_batch_small.
 *   larger N: b2gp_mll / b2gp_dkl_mll(n_layers = 0) per member, so each member's outputs are those calls' bits.
 * Kinds RBF, Matern-5/2, Periodic; d <= 16 (else B2GP_ERR_ARG, as is grad_x without grad).  NNGP kinds, B2GP_FLAG_F32
 * and B2GP_FLAG_DEVICE_PTRS give B2GP_ERR_UNSUPPORTED.  Identical calls give identical bits.                          */
/* The largest N that b2gp_mll_batch's one-launch route takes (at most 128, one potrf leaf): the largest N at which it was
 * measured to win at B = 1 against one b2gp_mll and one b2gp_dkl_mll(n_layers = 0) call for every kind and d in {1, 3}
 * (1.09-1.67x at N = 96 on an H100 80GB HBM3 at 700 W; at N = 112 RBF d = 1 loses, 0.93x; DESIGN.md 4.13).          */
#define B2GP_MLL_BATCH_SMALL_MAX_N 96

int  b2gp_mll_batch(b2gp_ctx* ctx, int kind, const double* X, int64_t N, const double* yres, int d, int64_t B,
                    const double* theta, double jitter, unsigned flags, double* value, double* grad, double* alpha_out,
                    double* grad_x, int* info);

/* S exact-GP likelihoods on one X in lock-step (the chains of a vectorized NUTS round): draw s is b2gp_mll(kind, X,
 * yres + s * yres_stride, theta + s * (d+3)) and returns that call's value, grad, alpha and info bit for bit on the same
 * context options, whatever S and however the draws are grouped.  X[N,d] and yres (yres_stride = 0: one [N] vector for
 * every draw; else >= N doubles between draws) as b2gp_mll; theta[S,d+3] (NNGP kinds: b2gp_mll's layout and depth check
 * per draw).  HOST outputs: value[S]; grad[S,d+3] (optional) d value / dlog theta; alpha_out[S,N] (optional) K^{-1} yres;
 * info[S].  A draw with info[s] != 0 has NaN value, grad and alpha; the others are unaffected.  Routes:
 *   fp64, N < tall_min_fp64:   mll_impl's sequence in groups of draws, every launch (Gram build, recursive factorisation,
 *                              solves, K^{-1}, gradient reduction) covering the whole group: the launches per call do not
 *                              grow with S;
 *   fp64, N >= tall_min_fp64:  the same with the batched tall-panel factorisation, y riding below K;
 *   int8 (ozaki != 0):         one draw at a time (those GEMMs take one draw), one host sync for the call.
 * Groups hold as many draws as an eighth of the device memory takes (option draw_batch: 1 = one draw per group, B >= 2 =
 * groups of B); each group counts once in the route counter mll_draws_batch.  Host fp64 arrays only: B2GP_FLAG_F32 and
 * B2GP_FLAG_DEVICE_PTRS give B2GP_ERR_UNSUPPORTED before any launch; there is no multi-task form (the noise-vector
 * form is b2gp_mll_draws_v).                                                                                           */
int  b2gp_mll_draws(b2gp_ctx* ctx, int kind, const double* X, int64_t N, const double* yres, int64_t yres_stride, int d,
                    int64_t S, const double* theta, double jitter, unsigned flags, double* value, double* grad,
                    double* alpha_out, int* info);

/* b2gp_mll_draws with a per-point noise vector per draw (the chains of MeasuredNoiseGP / VarNoiseGP): draw s is
 * b2gp_mll_v(kind, X, yres + s * yres_stride, theta + s * (d+3), noise_vec + s * nv_stride) and returns that call's
 * value, grad, alpha, grad_noise_vec and info bit for bit, whatever S and the grouping, on every route of
 * b2gp_mll_draws.  noise_vec is required; nv_stride = 0 shares one [N] vector between the draws, else >= N doubles
 * between draws.  grad_noise_vec[S,N] (optional, needs grad) is d value / d noise_vec.  A draw with info[s] != 0 has NaN
 * in all of its outputs.  Routes, groups, the mll_draws_batch counter and the refusals are b2gp_mll_draws'.            */
int  b2gp_mll_draws_v(b2gp_ctx* ctx, int kind, const double* X, int64_t N, const double* yres, int64_t yres_stride, int d,
                      int64_t S, const double* theta, const double* noise_vec, int64_t nv_stride, double jitter,
                      unsigned flags, double* value, double* grad, double* alpha_out, double* grad_noise_vec, int* info);

/* The multi-task counterpart (the likelihood of viMTDKL.model, gpax/models/vi_mtdkl.py): log N(yres; 0, K) with K the
 * LCM covariance of b2gp_mll_multitask on the embedding z = MLP(X), expanded to the GP rows:
 *   X[N, D]                 the network's inputs, N points, without the task column
 *   task[N*group], yres[N*group]  the GP rows, point-major: point p is rows p*group .. p*group+group-1 (group = 1: the
 *                           multitask form, one row per point; group = T: the Kronecker form, task index fastest)
 *   theta[L,d+2], B[L,T,T], noise[T], group, T, L   as b2gp_mll_multitask (RBF and Matern; d = z_dim)
 * HOST outputs: value, grad_theta, grad_B, grad_noise as b2gp_mll_multitask on the expanded z (same kernels, same
 * bits); grad_z[N, d] (optional) d value / dz, each point's rows summed in task order (with n_layers = 0 this is
 * d value / dX); grad_params (optional) in the params layout.  X and yres follow `flags` (B2GP_FLAG_DEVICE_PTRS allowed,
 * B2GP_FLAG_F32 refused); task, theta, B, noise, widths and params are HOST pointers.  Task ids are checked before any
 * launch.  NaN outputs where info != 0.  The reductions run in a fixed order: identical calls give identical bits.   */
int  b2gp_mtdkl_mll(b2gp_ctx* ctx, int kind, const double* X, const int* task, int64_t N, int64_t D, const double* yres,
                    int group, int T, int L, int n_layers, const int64_t* widths, int act, const double* params,
                    const double* theta, const double* B, const double* noise, double jitter,
                    unsigned flags, double* value, double* grad_theta, double* grad_B, double* grad_noise,
                    double* grad_params, double* grad_z, int* info);

/* ---- fully Bayesian MLP (gpax/models/bnn.py over spm.py; gpax_b200/csrc/bnn.cuh) --------------------------------------
 * The network of b2gp_mlp_forward: n_layers >= 1 dense layers with widths[l] outputs (widths[n_layers-1] = O), act on
 * every layer but the last, params in the flat layout (per layer W_l [in, out] row-major, then b_l).
 * b2gp_bnn_loglik: value = sum_{i,o} log N(y[i,o]; MLP(X)[i,o], sigma) -- the likelihood of sPM.model, spm.py:63-77 --
 *   with d value / d sigma and, when grad_params is given, d value / d params in the flat layout.  sigma > 0, finite.  X[N,D], y[N,O] follow
 *   `flags` (B2GP_FLAG_DEVICE_PTRS; B2GP_FLAG_F32 is refused); widths, params and the outputs are HOST pointers.
 *   Deterministic: identical calls give identical bits.
 * Route: fused (two launches: a tile kernel that keeps the weight set, a gradient accumulator and one 32-row tile's
 *   activations in shared memory, and a fixed-order reduction) when 8 * (2 * nparams + 32 * sum_l (width_l | 1)) bytes,
 *   with width_0 = D, plus 2 KB fit in the device's opt-in shared memory per block and n_layers <= 16; otherwise
 *   layered (the b2gp_mlp_forward pass, a residual kernel, b2gp_dkl_mll's backward pass).  Option "bnn_fused" = 0 forces
 *   the layered route.
 * b2gp_bnn_predict: loc[s] = MLP(X; params + s * params_stride) for S weight sets, [S,P,O]; when eps [S,n,P,O]
 *   is given, y_sampled[s] = loc[s] + sigma[s] * mean_k eps[s,k] (k in order; spm.py:150-154).  X follows `flags`,
 *   everything else is a HOST pointer.  Fused (grid (row tiles, draws): one launch per 65535 draws) when
 *   8 * (nparams + 32 * sum_l (width_l | 1)) bytes fit, as above; otherwise the forward pass and a sampling epilogue per
 *   draw.                                                                                                                */
int  b2gp_bnn_loglik(b2gp_ctx* ctx, const double* X, int64_t N, int64_t D, const double* y, int64_t O, int n_layers,
                     const int64_t* widths, int act, const double* params, double sigma, unsigned flags, double* value,
                     double* grad_sigma, double* grad_params);
int  b2gp_bnn_predict(b2gp_ctx* ctx, const double* X, int64_t P, int64_t D, int n_layers, const int64_t* widths, int act,
                      const double* params, int64_t S, int64_t params_stride, int64_t O, const double* sigma,
                      const double* eps, int64_t n, double* loc, double* y_sampled, unsigned flags);

/* b2gp_bnn_predict_grad: loc[s] = MLP(X; params + s * params_stride) for S weight sets of a one-output network
 *   (widths[n_layers-1] = 1, else B2GP_ERR_ARG), [S,P], and its gradient w.r.t. the inputs, dloc[s,p,k] = d loc[s,p] /
 *   d X[p,k], [S,P,D] -- what optimize_acq needs of a BNN at each evaluation.  X and params follow `flags`: under
 *   B2GP_FLAG_DEVICE_PTRS both are device pointers, so the weight sets can stay resident across calls; B2GP_FLAG_F32 gives
 *   B2GP_ERR_UNSUPPORTED.  widths and both outputs are HOST pointers.  Every argument is checked before any launch.
 *   loc is bit-identical to b2gp_bnn_predict's on the same route.  Fused exactly where b2gp_bnn_predict is (one launch
 *   per 65535 draws: the forward pass, then the backward recursion over the tile's activations); otherwise the
 *   b2gp_mlp_forward pass per draw and one input vector-Jacobian product launch per chunk of draws whose hidden
 *   activations fit in 1 GiB.  Deterministic: identical calls give identical bits.                                     */
int  b2gp_bnn_predict_grad(b2gp_ctx* ctx, const double* X, int64_t P, int64_t D, int n_layers, const int64_t* widths, int act,
                           const double* params, int64_t S, int64_t params_stride, double* loc, double* dloc, unsigned flags);

/* Samples of S multivariate normals: y[s,i,:] = mean[s,:] + chol(cov[s]) eps[s,i,:], i < n -- replaces
 * numpyro.distributions.MultivariateNormal(mean, cov).sample (gpax/models/gp.py:292, gpax/acquisition/base_acq.py:221)
 * where the caller changed cov after the posterior call (gpax/models/hskgp.py:201-204 adds the predicted noise variance).
 * info[s] = 0 or the first bad pivot of cov[s] (that member's samples are NaN).                                    */
int  b2gp_mvn_sample(b2gp_ctx* ctx, const double* mean, const double* cov, int64_t S, int64_t P,
                     const double* eps, int64_t n, double* y, int* info, unsigned flags);

/* ---- acquisition epilogues (SURVEY.md section 8f-4) on the posterior's outputs, host or device pointers ----------
 * kind: 0 EI, 1 UCB, 2 UE, 3 POI -- gpax/acquisition/base_acq.py:20-71 (ei), 74-104 (ucb), 107-130 (ue), 133-155 (poi).
 *   mean[R,P], var[R,P] -> out[R,P]; row r is one posterior (R = 1 for viGP / the pooled moments of an MCMC model,
 *   R = number of sub-sampled draws for the q-batch functions, gpax/acquisition/batch_acquisition.py:110-116).
 *   have_best = 0: best_f is derived from each row's mean (max when maximize, else min: base_acq.py:59-60);
 *   param = beta (UCB) or xi (POI).                                                                             */
int  b2gp_acq_moments(b2gp_ctx* ctx, int kind, const double* mean, const double* var, int64_t R, int64_t P,
                      int have_best, double best_f, double param, int maximize, double* out, unsigned flags);
/* Same, from posterior samples y[R,P] (R = S*n rows of y_sampled): column mean and population variance
 * (gpax/acquisition/acquisition.py:31-34), then the acquisition function.  mean_out / var_out [P] optional.      */
int  b2gp_acq_samples(b2gp_ctx* ctx, int kind, const double* y, int64_t R, int64_t P,
                      int have_best, double best_f, double param, int maximize,
                      double* out, double* mean_out, double* var_out, unsigned flags);
/* Knowledge gradient (gpax/acquisition/base_acq.py:158-232) from one posterior: mean[P], cov[P,P] of the candidates,
 * ysim[n,P] simulated observations (base_acq.py:223).  The reference re-inverts the (N+1)x(N+1) training covariance
 * for every candidate and simulation; here the rank-1 (block-inverse) update of the posterior mean is evaluated in
 * closed form.  diag_sub = noise_p + jitter (what `cov` carries on its diagonal beyond the latent covariance),
 * noise_plus_jitter = the diagonal term of the appended training point.  out[P].                                 */
int  b2gp_kg(b2gp_ctx* ctx, const double* mean, const double* cov, int64_t P, const double* ysim, int64_t n,
             double diag_sub, double noise_plus_jitter, int maximize, double* out, unsigned flags);
/* Same with a value per candidate: diag_sub[P], noise_plus_jitter[P] (follow `flags` as the other arrays).  The LCM
 * models (viMTDKL) carry a noise per task, so both terms depend on the candidate's task.                         */
int  b2gp_kg_v(b2gp_ctx* ctx, const double* mean, const double* cov, int64_t P, const double* ysim, int64_t n,
               const double* diag_sub, const double* noise_plus_jitter, int maximize, double* out, unsigned flags);

/* ---- multi-GPU building blocks (SURVEY.md section 8e).  One process per GPU; the exchange steps
 * (panel broadcast, M x M all-reduce) are issued by the host side over NCCL on these same device
 * buffers (gpax_b200/distributed.py).  All array pointers below are DEVICE pointers. ----------------*/

/* ---- in-library multi-GPU (one process per GPU, NCCL loaded at run time; gpax_b200/csrc/dist.cuh) ------------------
 * b2gp_dist_unique_id: rank 0 obtains the 128-byte NCCL id and hands it to the other ranks by any host channel
 *   (gpax_b200/dist.py uses a TCP socket at MASTER_ADDR).  b2gp_dist_init: every rank, same id; builds the world
 *   communicator and the row / column communicators of a grid_rows x grid_cols process grid (rank = row * grid_cols + col).
 * b2gp_dist_posterior (COLLECTIVE, host pointers, inputs replicated on every rank): exact-GP posterior mean and diagonal
 *   variance -- gpax/models/gp.py:253-277 / gpax/models/vigp.py:178-185 -- with k_XX 2-D block-cyclic over the grid in
 *   nb x nb tiles (N a multiple of nb, nb a multiple of 128), generated in place; right-looking Cholesky with the panel
 *   solve spread over the process column, the panel broadcast along process rows and all-gathered down process columns,
 *   look-ahead of one panel, trailing updates on the int8 wgmma kernel; the right-hand sides ride below the matrix.
 *   There is no fp64 trailing update on this path: option "ozaki" = 0 (the default) picks the digit-plane count from
 *   the bound on cond(K) exactly like -1; 6 / 7 force it.
 *   Every rank receives mean[P], var[P] (B2GP_OUT_VAR) and info.
 * b2gp_dist_layout: the block-cyclic index algebra as a pure function (no GPU), see dist.cuh.                         */
int  b2gp_dist_unique_id(void* id128);
int  b2gp_dist_init(b2gp_ctx* ctx, const void* id128, int rank, int nranks, int grid_rows, int grid_cols);
int  b2gp_dist_info(b2gp_ctx* ctx, int* rank, int* nranks, int* grid_rows, int* grid_cols);
int  b2gp_dist_finalize(b2gp_ctx* ctx);
int  b2gp_dist_posterior(b2gp_ctx* ctx, int kind, const double* Xtr, int64_t N, const double* yres,
                         const double* Xnew, int64_t P, int d, const double* theta, int noiseless, double jitter,
                         int64_t nb, unsigned flags, double* mean, double* var, int* info, b2gp_timing* timing);
/* b2gp_dist_sparse_posterior (COLLECTIVE, host pointers): N-sharded Nystrom / VFE posterior --
 *   gpax/models/sparse_gp.py:173-223 -- every rank passes ITS shard of the training set and the same Xu, X_new, theta;
 *   per-rank statistics, one NCCL all-reduce of the M x M matrix + M-vector inside the library, replicated finish.    */
int  b2gp_dist_sparse_posterior(b2gp_ctx* ctx, int kind, const double* Xu, int64_t M, const double* Xtr_shard, int64_t N_shard,
                                const double* y_shard, const double* Xnew, int64_t P, int d, const double* theta,
                                int noiseless, double jitter, unsigned flags, double* mean, double* var, int* info,
                                b2gp_timing* timing);
int  b2gp_dist_layout(int64_t T, int64_t R, int64_t nb, int pr, int pc, int row, int col, int64_t k, int64_t* out6);

/* N-sharded sparse posterior: per-shard statistics, then the posterior from their sum.
 *   Kpart[M,M] (lower) = W W^T / noise,  cpart[M] = W y / noise  with W = Luu^{-1} K(Xu, Xtr_shard)
 *   (gpax/models/sparse_gp.py:193-199, 203-204 restricted to a shard; sums over shards give the full terms).
 *   theta is a HOST pointer (d+3 values).                                                           */
int  b2gp_sparse_partial(b2gp_ctx* ctx, int kind, const double* Xu, int64_t M, const double* Xtr, int64_t N,
                         const double* yres, int d, const double* theta, double jitter,
                         double* Kpart, int64_t ldk, double* cpart, int* info);
/* Ksum is overwritten (+I, then its Cholesky factor): sparse_gp.py:200-217.                          */
int  b2gp_sparse_finish(b2gp_ctx* ctx, int kind, const double* Xu, int64_t M, double* Ksum, int64_t ldk,
                        const double* csum, const double* Xnew, int64_t P, int d, const double* theta,
                        int noiseless, double jitter, unsigned flags,
                        double* mean, double* var, double* cov, int* info);

/* Block-cyclic Cholesky: factor one diagonal block and export the inverted 128x128 sub-blocks
 * (ceil(n/128)*128*128 doubles) so that panel solves can run later / on other blocks.              */
int  b2gp_potrf_inv(b2gp_ctx* ctx, int64_t n, double* A, int64_t lda, double* Linv_out, int* info);
/* B (nrhs rows of length n, leading dimension ldb) <- B L^{-T} using Linv from b2gp_potrf_inv.      */
int  b2gp_trsm_inv(b2gp_ctx* ctx, int64_t n, int64_t nrhs, const double* L, int64_t ldl,
                   const double* Linv, double* B, int64_t ldb);
/* dot[r] (+)= scale * <R[r,0:len), w>,  nrm[r] (+)= |R[r,0:len)|^2 ; either output may be NULL.      */
int  b2gp_rowdot(b2gp_ctx* ctx, int64_t rows, int64_t len, const double* R, int64_t ldr, const double* w,
                 double scale, double* dot, double* nrm, int accumulate);
int  b2gp_copy2d(b2gp_ctx* ctx, double* dst, int64_t ldd, const double* src, int64_t lds, int64_t rows, int64_t cols);

#ifdef __cplusplus
}
#endif
#endif /* B200GP_H */
