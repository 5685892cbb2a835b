// sparse_elbo.cuh -- kernels for the VFE bound of the sparse GP and its gradient (fit side of viSparseGP).
//
// The reference's model (gpax/models/sparse_gp.py:62-114) scores
//     ELBO = log LowRankMVN(y; 0, W^T W + noise I) - 1/2 clip(sum_n (Kff_nn - Qff_nn) / noise, 0)
// with W = Luu^{-1} Kuf, and lets NumPyro's SVI differentiate it w.r.t. the kernel hyper-parameters, the noise
// and the inducing inputs Xu (a numpyro.param, sparse_gp.py:69-70).  Here the reverse pass is written out by hand on
// M x M and M x N matrices (b200gp.cu: b2gp_sparse_elbo) and the last step -- contracting dELBO/dKuf and
// dELBO/dKuu with the kernel's derivatives w.r.t. log-parameters and Xu -- is two fused reductions that recompute
// the kernel and its derivatives on the fly (no derivative matrices are materialised).
#pragma once
#include "common.cuh"
#include "gram.cuh"
#include "mll.cuh"

// K(xa, xb) and derivatives: dlog[k] = dK/dlog(lengthscale_k) (k < d), dlog[d] = dK/dlog(scale), dlog[d+2] = dK/dlog(period),
// dxa[k] = dK/dxa_k
__device__ __forceinline__ double kern_derivs(int kind, int d, const double* xa, const double* xb, const double* theta, double* dlog,
                                              double* dxa) {
    const double scale = theta[d], period = theta[d + 2];
    double K;
    if (kind == B2GP_KERNEL_PERIODIC) {
        double ssum = 0.0, dper = 0.0;
        double q[MLL_MAX_D], sc[MLL_MAX_D];
        for (int k = 0; k < d; ++k) {
            const double a = 3.141592653589793 * (xa[k] - xb[k]) / period;
            const double sn = sin(a), cs = cos(a), l2 = theta[k] * theta[k];
            q[k] = sn * sn / l2;
            sc[k] = sn * cs / l2;
            ssum += q[k];
            dper += sc[k] * a;
        }
        K = scale * exp(-2.0 * ssum);
        for (int k = 0; k < d; ++k) {
            dlog[k] = K * 4.0 * q[k];
            dxa[k] = -K * 4.0 * sc[k] * (3.141592653589793 / period);
        }
        dlog[d + 2] = K * 4.0 * dper;
    } else {
        double r2 = 0.0;
        double q[MLL_MAX_D];
        for (int k = 0; k < d; ++k) {
            const double dl = (xa[k] - xb[k]) / theta[k];
            q[k] = dl * dl;
            r2 += q[k];
        }
        double dK;
        if (kind == B2GP_KERNEL_RBF) {
            K = scale * exp(-0.5 * r2);
            dK = K;
        } else {
            const double r = sqrt(r2 + 1e-12), s5r = 2.23606797749979 * r, ex = exp(-s5r);
            K = scale * (1.0 + s5r + (5.0 / 3.0) * r2) * ex;
            dK = (5.0 / 3.0) * scale * (1.0 + s5r) * ex;
        }
        for (int k = 0; k < d; ++k) {
            dlog[k] = dK * q[k];
            dxa[k] = -dK * (xa[k] - xb[k]) / (theta[k] * theta[k]);
        }
        dlog[d + 2] = 0.0;
    }
    dlog[d] = K;
    dlog[d + 1] = 0.0;
    return K;
}

// One CTA per row a of the left input set A (inducing point a): partial[a][0..d+3) = sum_b G[a,b] dK(A_a, B_b)/dlog(theta),
// gx[a][k] (+)= sum_b Gx[a,b] dK(A_a, B_b)/dA_ak, skipping b == a when skip_diag (the Kuu case, where both arguments move).
// G and Gx are row-major [rowsA x rowsB] with leading dimensions ldg, ldgx.
__global__ void __launch_bounds__(256)
elbo_chain_kernel(int kind, int d, const double* __restrict__ theta, const double* __restrict__ XA, int rowsA, const double* __restrict__ XB,
                  int64_t rowsB, const double* __restrict__ G, int64_t ldg, const double* __restrict__ Gx, int64_t ldgx, int skip_diag,
                  int accumulate, double* __restrict__ partial, double* __restrict__ gx) {
    __shared__ double red[8][2 * MLL_MAX_D + 3];
    const int a = blockIdx.x;
    const int nout = d + 3;
    double xa[MLL_MAX_D];
    for (int k = 0; k < d; ++k) xa[k] = XA[(int64_t)a * d + k];
    double acc[2 * MLL_MAX_D + 3];
#pragma unroll
    for (int k = 0; k < 2 * MLL_MAX_D + 3; ++k) acc[k] = 0.0;
    for (int64_t b = threadIdx.x; b < rowsB; b += 256) {
        double xb[MLL_MAX_D], dlog[MLL_MAX_D + 3], dxa[MLL_MAX_D];
        for (int k = 0; k < d; ++k) xb[k] = XB[b * d + k];
        kern_derivs(kind, d, xa, xb, theta, dlog, dxa);
        const double g = G[(int64_t)a * ldg + b];
        for (int k = 0; k < nout; ++k) acc[k] += g * dlog[k];
        if (!(skip_diag && b == a)) {
            const double g2 = Gx[(int64_t)a * ldgx + b];
            for (int k = 0; k < d; ++k) acc[nout + k] += g2 * dxa[k];
        }
    }
    const int total = nout + d;
    for (int k = 0; k < total; ++k) {
        double v = acc[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5][k] = v;
    }
    __syncthreads();
    if ((int)threadIdx.x < total) {
        double v = 0.0;
        for (int w = 0; w < 8; ++w) v += red[w][threadIdx.x];
        const int k = threadIdx.x;
        if (k < nout) {
            double* dst = partial + (int64_t)a * nout + k;
            *dst = accumulate ? *dst + v : v;
        } else {
            double* dst = gx + (int64_t)a * d + (k - nout);
            *dst = accumulate ? *dst + v : v;
        }
    }
}

// out[k] = sum_a partial[a][k]   (fixed order)
__global__ void colsum_kernel(const double* partial, int64_t rows, int ncols, double* out) {
    const int k = threadIdx.x;
    if (k >= ncols) return;
    double s = 0.0;
    for (int64_t a = 0; a < rows; ++a) s += partial[a * ncols + k];
    out[k] = s;
}

// out[0] = sum_i v[i]  (single block, fixed order)
__global__ void vecsum_kernel(const double* v, int64_t n, double* out) {
    __shared__ double red[256];
    double s = 0.0;
    for (int64_t i = threadIdx.x; i < n; i += 256) s += v[i];
    red[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) out[0] = red[0];
}

// mode 0: dst = tril(src);  1: dst = -triu(src);  2: dst = tril(src) with the diagonal halved (the Phi of the Cholesky
// backward pass);  3: dst = src + src^T;  4: dst = (src + src^T) / 2.  Square n x n, separate leading dimensions; dst may
// not alias src.
__global__ void tri_kernel(double* dst, int64_t ldd, const double* src, int64_t lds, int64_t n, int mode) {
    const int64_t i = (int64_t)blockIdx.y * 32 + threadIdx.y, j = (int64_t)blockIdx.x * 32 + threadIdx.x;
    if (i >= n || j >= n) return;
    const double v = src[i * lds + j];
    double o;
    if (mode == 0)
        o = (j <= i) ? v : 0.0;
    else if (mode == 1)
        o = (j >= i) ? -v : 0.0;
    else if (mode == 2)
        o = (j < i) ? v : (j == i ? 0.5 * v : 0.0);
    else if (mode == 3)
        o = v + src[j * lds + i];
    else
        o = 0.5 * (v + src[j * lds + i]);
    dst[i * ldd + j] = o;
}

// alpha[n] = (y[n] - t[n]) / noise
__global__ void elbo_alpha_kernel(double* alpha, const double* y, const double* t, int64_t n, double noise) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) alpha[i] = (y[i] - t[i]) / noise;
}

// E[n,m] <- alpha[n] beta[m] + (coef * Wt[n,m] - E[n,m]) / noise      (dELBO/dW^T, in place over E = Wt C^{-1})
__global__ void elbo_gw_kernel(double* E, int64_t lde, const double* Wt, int64_t ldw, const double* alpha, const double* beta, int64_t N,
                               int64_t M, double coef, double noise) {
    const int64_t total = N * M;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int64_t n = idx / M, m = idx % M;
        E[n * lde + m] = alpha[n] * beta[m] + (coef * Wt[n * ldw + m] - E[n * lde + m]) / noise;
    }
}

// ---- caller-supplied blocks (b2gp_sparse_elbo_gram: a user kernel callable's fit)
// One CTA (m, y) per row m of the M x M adjoint Gs and of the M x N adjoint Guf, and direction j = j0 + y:
//   rows[j * M + m] = sum_i Gs[m, i] dKuu_j[m, i] + sum_n Guf[m, n] dKuf_j[m, n]
// and CTA (M, y): ksum[j] = sum_n dkff_j[n].  `ptrs` + 3 y holds the direction's (Kuu block [M, ldu], Kuf block [M, ldf],
// kff vector [N]); a NULL pointer is a zero block.  Every sum runs in a fixed order (strided per thread, then the warp
// shuffles, then the 8 warps in turn), so identical calls give identical bits.
constexpr int SGT_THREADS = 256;
__global__ void __launch_bounds__(SGT_THREADS)
sparse_gram_trace_kernel(const double* __restrict__ Gs, int64_t ldgs, const double* __restrict__ Guf, int64_t ldguf, int64_t M,
                         int64_t N, const double* const* __restrict__ ptrs, int64_t ldu, int64_t ldf, int64_t j0,
                         double* __restrict__ rows, double* __restrict__ ksum) {
    __shared__ double red[SGT_THREADS / 32];
    const int64_t m = blockIdx.x, j = j0 + blockIdx.y;
    const double* const* pj = ptrs + 3 * (int64_t)blockIdx.y;
    double s = 0.0;
    if (m < M) {
        const double* du = pj[0];
        const double* df = pj[1];
        if (du)
            for (int64_t i = threadIdx.x; i < M; i += SGT_THREADS) s = fma(Gs[m * ldgs + i], du[m * ldu + i], s);
        if (df)
            for (int64_t n = threadIdx.x; n < N; n += SGT_THREADS) s = fma(Guf[m * ldguf + n], df[m * ldf + n], s);
    } else if (pj[2]) {
        const double* dk = pj[2];
        for (int64_t n = threadIdx.x; n < N; n += SGT_THREADS) s += dk[n];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < SGT_THREADS / 32; ++w) t += red[w];
        if (m < M)
            rows[j * M + m] = t;
        else
            ksum[j] = t;
    }
}

// grad[j] = sum_m rows[j * M + m] + gd * ksum[j], j < p  (fixed order)
__global__ void sparse_gram_finish_kernel(const double* __restrict__ rows, int64_t M, const double* __restrict__ ksum, double gd,
                                          int64_t p, double* __restrict__ grad) {
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= p) return;
    double s = 0.0;
    for (int64_t m = 0; m < M; ++m) s += rows[j * M + m];
    grad[j] = s + gd * ksum[j];
}
