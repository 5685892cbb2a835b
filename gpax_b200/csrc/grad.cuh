// grad.cuh -- derivative rows of the cross-covariance w.r.t. the test inputs.
//
// D[p*d + k, i] = d k(x_p, x_i) / d x_p[k] for the P test points x_p and the N training points x_i.  These rows are right-hand
// sides like k_pX: the posterior writes them under [k_pX; y^T] in the slot's matrix and solves them with the same factor, so
// that (with V_p = L^{-1} k(X, x_p), w = L^{-1} y_res)
//   d mean_p / d x_p[k] =      <L^{-1} D_{p,k}, w>
//   d var_p  / d x_p[k] = -2 * <L^{-1} D_{p,k}, V_p>      (k(x, x) is constant for the three stationary kernels)
// (rowdot_grad_kernel, posterior.cuh).  The derivatives are those of the reference's formulas as written
// (gpax/kernels/kernels.py:28-117), i.e. what jax.grad of them gives:
//   RBF       k = s exp(-r2/2)                              dk/dr2 = -k/2
//   Matern    k = s (1 + sqrt5 r + 5/3 r2) exp(-sqrt5 r),  r = sqrt(r2 + 1e-12) and the 5/3 r2 term without the epsilon:
//             dk/dr2 = -(5/6) s exp(-sqrt5 r) (1 + sqrt5 r2 / r)
//   with r2 = |x_p/l - x_i/l|^2 clipped at 0 (kernels.py:41; jax's gradient of the clip is 0 where it clips) and
//   dr2/dx_p[k] = 2 (x_p[k]/l_k - x_i[k]/l_k) / l_k;
//   Periodic  k = s exp(-2 sum_k sin(a_k)^2 / l_k^2), a_k = pi (x_p[k] - x_i[k]) / period:
//             dk/dx_p[k] = -k 2 pi sin(2 a_k) / (period l_k^2)
// HBM-bound: 8 P d N bytes written, the inputs are read once per tile.
#pragma once
#include "common.cuh"
#include "gram.cuh"

// dk/dr2 of RBF / Matern at the unclipped r2 = (x2 - 2 xz) + z2 of lengthscale-scaled inputs (see above); also used by
// mll_dz_kernel (dkl.cuh), so that the likelihood's input gradient differentiates the same formulas
__device__ __forceinline__ double stationary_dk_dr2(int kind, double r2raw, double scale) {
    if (r2raw < 0.0) return 0.0;                         // clipped (kernels.py:41): no gradient flows
    if (kind == B2GP_KERNEL_RBF) return -0.5 * scale * exp(-0.5 * r2raw);
    const double r = sqrt(r2raw + 1e-12);
    const double s5r = 2.23606797749979 * r;
    return -(5.0 / 6.0) * scale * exp(-s5r) * (1.0 + 2.23606797749979 * r2raw / r);
}

constexpr int GDX_BN = 128;     // training points (columns) per CTA
constexpr int GDX_BP = 16;      // test points per CTA
constexpr int GDX_THREADS = 256;

// grid (ceil(N / GDX_BN), ceil(P / GDX_BP)); dynamic shared memory: Zs[d][GDX_BN] | Xs[GDX_BP][d] | ell[d]
__global__ void __launch_bounds__(GDX_THREADS)
gram_dx_kernel(int kind, const double* __restrict__ Xnew, int64_t P, const double* __restrict__ Xtr, int64_t N, int d,
               const double* __restrict__ theta, double* __restrict__ D, int64_t ldd) {
    extern __shared__ __align__(16) double sm[];
    double* Zs = sm;
    double* Xs = Zs + d * GDX_BN;
    double* ell = Xs + GDX_BP * d;
    const int tid = threadIdx.x;
    const int64_t col0 = (int64_t)blockIdx.x * GDX_BN, p0 = (int64_t)blockIdx.y * GDX_BP;
    const bool periodic = (kind == B2GP_KERNEL_PERIODIC);
    for (int k = tid; k < d; k += GDX_THREADS) ell[k] = theta[k];
    __syncthreads();
    const double scale = theta[d], period = theta[d + 2];
    // staged as the Gram kernel stages them: divided by the lengthscale for RBF / Matern (kernels.py:35-36), raw for periodic.
    // Consecutive threads take consecutive columns of one dimension, so the shared-memory stores hit distinct banks.
    for (int idx = tid; idx < GDX_BN * d; idx += GDX_THREADS) {
        const int k = idx / GDX_BN, c = idx % GDX_BN;
        const int64_t gc = col0 + c;
        const double v = gc < N ? Xtr[gc * d + k] : 0.0;
        Zs[k * GDX_BN + c] = periodic ? v : v / ell[k];
    }
    for (int idx = tid; idx < GDX_BP * d; idx += GDX_THREADS) {
        const int r = idx / d, k = idx % d;
        const int64_t gp = p0 + r;
        const double v = gp < P ? Xnew[gp * d + k] : 0.0;
        Xs[r * d + k] = periodic ? v : v / ell[k];
    }
    __syncthreads();
    const int c = tid % GDX_BN;
    const int64_t gc = col0 + c;
    if (gc >= N) return;
    double z2 = 0.0;
    if (!periodic)
        for (int k = 0; k < d; ++k) z2 = fma(Zs[k * GDX_BN + c], Zs[k * GDX_BN + c], z2);
    for (int r = tid / GDX_BN; r < GDX_BP; r += GDX_THREADS / GDX_BN) {
        const int64_t gp = p0 + r;
        if (gp >= P) break;
        const double* x = Xs + r * d;
        double* out = D + gp * d * ldd + gc;
        if (periodic) {
            // one sincos per dimension: the first pass writes -2 pi sin(2 a_k) / (period l_k^2) = -4 pi sin a_k cos a_k / ...
            // and accumulates the exponent; the second multiplies by k, once known (the thread's own entries, still in L2)
            double s = 0.0;
            for (int k = 0; k < d; ++k) {
                double sa, ca;
                sincos(3.141592653589793 * (x[k] - Zs[k * GDX_BN + c]) / period, &sa, &ca);
                const double a = sa / ell[k];                                   // kernels.py:111-113
                s += a * a;
                out[k * ldd] = -(4.0 * 3.141592653589793) * sa * ca / (period * ell[k] * ell[k]);
            }
            const double kv = scale * exp(-2.0 * s);
            for (int k = 0; k < d; ++k) out[k * ldd] *= kv;
            continue;
        }
        double x2 = 0.0, xz = 0.0;
        for (int k = 0; k < d; ++k) {
            x2 = fma(x[k], x[k], x2);
            xz = fma(x[k], Zs[k * GDX_BN + c], xz);
        }
        const double r2raw = (x2 - 2.0 * xz) + z2;      // kernels.py:40
        const double g = stationary_dk_dr2(kind, r2raw, scale);
        for (int k = 0; k < d; ++k) out[k * ldd] = g * 2.0 * (x[k] - Zs[k * GDX_BN + c]) / ell[k];
    }
}

// D[P*d, N] (leading dimension ldd) for test points Xnew[P, d] against Xtr[N, d]
static int launch_gram_dx(b2gp_ctx* ctx, cudaStream_t st, int kind, const double* Xnew, int64_t P, const double* Xtr, int64_t N, int d,
                          const double* theta_dev, double* D, int64_t ldd) {
    if (P <= 0 || N <= 0) return B2GP_OK;
    if (kind < 0 || kind > B2GP_KERNEL_PERIODIC || d < 1 || d > GRAM_MAX_D)
        return set_err(ctx, B2GP_ERR_UNSUPPORTED, "gram_dx", "RBF / Matern / Periodic, 1 <= d <= 64", __FILE__, __LINE__);
    const size_t smem = (size_t)(d * GDX_BN + GDX_BP * d + d) * sizeof(double);
    static PerDeviceOnce attr;
    if (attr.need(ctx->device)) {
        CUDA_TRY(ctx, cudaFuncSetAttribute(gram_dx_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 80 * 1024));
        attr.done(ctx->device);
    }
    dim3 grid((unsigned)ceil_div(N, (int64_t)GDX_BN), (unsigned)ceil_div(P, (int64_t)GDX_BP));
    return launch(ctx, st, grid, GDX_THREADS, smem, gram_dx_kernel, kind, Xnew, P, Xtr, N, d, theta_dev, D, ldd);
}
