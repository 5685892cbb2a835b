// posterior.cuh -- epilogue kernels of the posterior: mean / diagonal variance by row reductions over
// V^T, symmetric fill of the covariance, NaN fill for failed draws, posterior-sample helpers.
//
// With K = L L^T, V^T = k_pX L^{-T} (one row per test point) and w = L^{-1} y_res:
//   mean[p] = <V^T[p,:], w>                          (gpax/models/gp.py:273: k_pX K^{-1} y)
//   var[p]  = k(x_p,x_p) + noise_p + jitter - |V^T[p,:]|^2    (diag of gp.py:272; vigp.py:185)
//   cov     = k_pp - V^T V                            (gp.py:272)
// HBM-bound: each row of V^T (N doubles) is read once.
#pragma once
#include "common.cuh"
#include "gram.cuh"

constexpr int RD_THREADS = 256;

// one CTA per test point: warp-shuffle + shared-memory tree reduction in a fixed order (deterministic)
__global__ void __launch_bounds__(RD_THREADS)
rowdot_kernel(const double* __restrict__ Vt, int64_t ldv, int64_t N, int64_t P, int kind, int d,
              const double* __restrict__ theta, double noise_mult, double jitter, const int* __restrict__ info,
              double* __restrict__ mean, double* __restrict__ var) {
    __shared__ double red1[RD_THREADS / 32], red2[RD_THREADS / 32];
    const int64_t p = blockIdx.x;
    const double* row = Vt + p * ldv;
    const double* w = Vt + P * ldv;
    double s1 = 0.0, s2 = 0.0;
    for (int64_t k = threadIdx.x; k < N; k += RD_THREADS) {
        const double v = row[k];
        s1 = fma(v, w[k], s1);
        s2 = fma(v, v, s2);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        s1 += __shfl_xor_sync(0xffffffffu, s1, o);
        s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    }
    if ((threadIdx.x & 31) == 0) {
        red1[threadIdx.x >> 5] = s1;
        red2[threadIdx.x >> 5] = s2;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double a = 0.0, b = 0.0;
        for (int i = 0; i < RD_THREADS / 32; ++i) {
            a += red1[i];
            b += red2[i];
        }
        const bool bad = (*info != 0);
        const double nan = __longlong_as_double(0x7ff8000000000000LL);
        if (mean) mean[p] = bad ? nan : a;
        if (var) {
            const double kd = cov_self(kind, theta[d]) + (theta[d + 1] * noise_mult + jitter);
            var[p] = bad ? nan : kd - b;
        }
    }
}

// Gradients w.r.t. the test inputs (grad.cuh): the solved derivative rows G = Vt + (P + 1) * ldv, row p*d + k being
// L^{-1} dk(X, x_p)/dx_p[k]; dmean[p, k] = <G[p*d+k], w>, dvar[p, k] = -2 <G[p*d+k], V_p>.  One CTA per test point, the
// same fixed-order reduction as rowdot_kernel (deterministic), GRD_KC derivative rows per pass over V_p and w.
constexpr int GRD_KC = 4;
__global__ void __launch_bounds__(RD_THREADS)
rowdot_grad_kernel(const double* __restrict__ Vt, int64_t ldv, int64_t N, int64_t P, int d, const int* __restrict__ info,
                   double* __restrict__ dmean, double* __restrict__ dvar) {
    __shared__ double red1[GRD_KC][RD_THREADS / 32], red2[GRD_KC][RD_THREADS / 32];
    const int64_t p = blockIdx.x;
    const double* v = Vt + p * ldv;
    const double* w = Vt + P * ldv;
    const double* G = Vt + (P + 1 + p * d) * ldv;
    const bool bad = (*info != 0);
    const double nan = __longlong_as_double(0x7ff8000000000000LL);
    for (int k0 = 0; k0 < d; k0 += GRD_KC) {
        double s1[GRD_KC], s2[GRD_KC];
#pragma unroll
        for (int j = 0; j < GRD_KC; ++j) s1[j] = s2[j] = 0.0;
        for (int64_t i = threadIdx.x; i < N; i += RD_THREADS) {
            const double wi = w[i], vi = v[i];
#pragma unroll
            for (int j = 0; j < GRD_KC; ++j) {
                if (k0 + j < d) {
                    const double g = G[(int64_t)(k0 + j) * ldv + i];
                    s1[j] = fma(g, wi, s1[j]);
                    s2[j] = fma(g, vi, s2[j]);
                }
            }
        }
#pragma unroll
        for (int j = 0; j < GRD_KC; ++j) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                s1[j] += __shfl_xor_sync(0xffffffffu, s1[j], o);
                s2[j] += __shfl_xor_sync(0xffffffffu, s2[j], o);
            }
            if ((threadIdx.x & 31) == 0) {
                red1[j][threadIdx.x >> 5] = s1[j];
                red2[j][threadIdx.x >> 5] = s2[j];
            }
        }
        __syncthreads();
        if (threadIdx.x < GRD_KC && k0 + (int)threadIdx.x < d) {
            const int j = threadIdx.x;
            double a = 0.0, b = 0.0;
            for (int i = 0; i < RD_THREADS / 32; ++i) {
                a += red1[j][i];
                b += red2[j][i];
            }
            if (dmean) dmean[p * d + k0 + j] = bad ? nan : a;
            if (dvar) dvar[p * d + k0 + j] = bad ? nan : -2.0 * b;
        }
        __syncthreads();
    }
}

// C[j][i] = C[i][j] for j < i
__global__ void mirror_lower_kernel(double* C, int64_t ld, int64_t n) {
    const int64_t i = (int64_t)blockIdx.y * 32 + threadIdx.y;
    const int64_t j = (int64_t)blockIdx.x * 32 + threadIdx.x;
    if (i < n && j < i) C[j * ld + i] = C[i * ld + j];
}

// zero the strict upper triangle (the factor of cov is used as a dense GEMM operand)
__global__ void zero_upper_kernel(double* C, int64_t ld, int64_t n) {
    const int64_t i = (int64_t)blockIdx.y * 32 + threadIdx.y;
    const int64_t j = (int64_t)blockIdx.x * 32 + threadIdx.x;
    if (i < n && j < n && j > i) C[i * ld + j] = 0.0;
}

// rows x cols region (leading dimension ld) <- NaN when *info (or *info2) is non-zero
__global__ void nan_if_bad_kernel(double* C, int64_t ld, int64_t rows, int64_t cols, const int* info, const int* info2) {
    const bool bad = (*info != 0) || (info2 && *info2 != 0);
    if (!bad) return;
    const double nan = __longlong_as_double(0x7ff8000000000000LL);
    const int64_t total = rows * cols;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x)
        C[(idx / cols) * ld + idx % cols] = nan;
}

// Y[i, :] = mean[:] for i < rows  (gp.py:292: the loc of the MultivariateNormal)
__global__ void bcast_rows_kernel(double* Y, int64_t ld, int64_t rows, int64_t cols, const double* mean) {
    const int64_t total = rows * cols;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x)
        Y[(idx / cols) * ld + idx % cols] = mean[idx % cols];
}

// strided 2-D copy dst[r, c] = src[r, c]
__global__ void copy2d_kernel(double* dst, int64_t ldd, const double* src, int64_t lds, int64_t rows, int64_t cols) {
    const int64_t total = rows * cols;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x)
        dst[(idx / cols) * ldd + idx % cols] = src[(idx / cols) * lds + idx % cols];
}

// dst[r, c] = src[r, c] * scale[c]^-1 ... used by the sparse path: W_Dinv = W / D with constant D
__global__ void scale_kernel(double* dst, int64_t ldd, const double* src, int64_t lds, int64_t rows, int64_t cols,
                             const double* theta, int d) {
    const double noise = theta[d + 1];
    const int64_t total = rows * cols;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x)
        dst[(idx / cols) * ldd + idx % cols] = src[(idx / cols) * lds + idx % cols] / noise;
}

__global__ void add_diag_kernel(double* C, int64_t ld, int64_t n, double v) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) C[i * ld + i] += v;
}

// grid of a grid-stride kernel: one thread per element, at most 8 CTAs per SM of the largest device a context was
// created on (g_grid_sms)
static inline unsigned grid_for(int64_t total, int threads = 256) {
    const int64_t cap = 8 * (int64_t)g_grid_sms.load(std::memory_order_relaxed);
    int64_t g = ceil_div(total, threads);
    if (g > cap) g = cap;
    if (g < 1) g = 1;
    return (unsigned)g;
}
