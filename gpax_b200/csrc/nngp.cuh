// nngp.cuh -- the NNGP kernels (gpax/kernels/kernels.py:120-224) on the posterior and likelihood routes.
//
// The Gram matrices themselves come from gram_kernel (gram.cuh).  Here:
//   nngp_diag_kernel       k(x_p, x_p) + noise * noise_mult + jitter per test point: the prior variance of the posterior's
//                          variance epilogue (an NNGP kernel is not stationary, so cov_self does not cover it)
//   nngp_self_kernel       per training point the self-chain k11^(l), l = 0..depth-1, with its forward-mode derivatives
//                          w.r.t. var_b and var_w
//   mll_nngp_grad_kernel   sum over the lower triangle of W_ij dK_ij / dlog(var_w, noise, var_b), W = alpha alpha^T - K^{-1},
//                          running only the cross chain k12 per pair (the self-chains come from nngp_self_kernel)
// The derivatives are those JAX takes of the reference's expressions: zero through jnp.clip where the clip is active, the
// unclipped fraction entering the ReLU step through (pi - theta) * fraction, and the square roots differentiated through
// both of their arguments.  On a ReLU self-term the fraction is a / sqrt(a * a) = 1, the clip is active and theta is
// constant.
//
// theta layout (b2gp_gram's): [0] depth (a double), [d] var_w, [d+1] noise, [d+2] var_b.
#pragma once
#include "common.cuh"
#include "gram.cuh"
#include "mll.cuh"

constexpr int NNGP_MAX_DEPTH = 16;
constexpr int NNGP_THREADS = 256;

// x . x with gram_kernel's fma order, so that a diagonal computed here equals the Gram build's bit for bit
__device__ __forceinline__ double nngp_dot_self(const double* __restrict__ x, int d) {
    double s = 0.0;
    for (int k = 0; k < d; ++k) s = fma(x[k], x[k], s);
    return s;
}

__global__ void nngp_diag_kernel(const double* __restrict__ X, int64_t n, int d, int kind, const double* __restrict__ theta,
                                 double noise_mult, double jitter, double* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double xx = nngp_dot_self(X + i * d, d);
    const double k = nngp_pair(kind == B2GP_KERNEL_NNGP_RELU, xx, xx, xx, d, theta[d + 2], theta[d], (int)theta[0]);
    out[i] = k + (theta[d + 1] * noise_mult + jitter);
}

// One NNGP layer with forward-mode derivatives.  (a, b, c) = (k12, k11, k22) of the layer below and their derivatives
// w.r.t. var_b (*b suffix) and var_w (*w suffix); returns k12 of this layer in v, its derivatives in gb / gw.
__device__ __forceinline__ void nngp_step_fwd(bool relu, double a, double ab, double aw, double b, double bb, double bw, double c,
                                              double cb, double cw, double var_b, double var_w, double& v, double& gb, double& gw) {
    constexpr double pi = 3.141592653589793;
    if (!relu) {
        // var_b + 2 var_w / pi * asin(clip(2 a / sqrt((1 + 2b)(1 + 2c))))       kernels.py:145-151
        const double u = (1.0 + 2.0 * b) * (1.0 + 2.0 * c);
        const double s = sqrt(u);
        const double fr = 2.0 * a / s;
        const double frc = fmin(fmax(fr, -1.0 + 1e-7), 1.0 - 1e-7);
        const double as = asin(frc);
        v = var_b + 2.0 * var_w / pi * as;
        const bool live = (fr == frc);                  // the clip passes the derivative only where it is inactive
        const double k = live ? 2.0 * var_w / pi / sqrt(1.0 - frc * frc) : 0.0;
        // d fr = 2 da / s - fr / (2 u) du,  du = 2 db (1 + 2c) + 2 dc (1 + 2b)
        const double h = fr / (2.0 * u);
        const double dfb = 2.0 * ab / s - h * (2.0 * bb * (1.0 + 2.0 * c) + 2.0 * cb * (1.0 + 2.0 * b));
        const double dfw = 2.0 * aw / s - h * (2.0 * bw * (1.0 + 2.0 * c) + 2.0 * cw * (1.0 + 2.0 * b));
        gb = 1.0 + k * dfb;
        gw = 2.0 / pi * as + k * dfw;
        return;
    }
    // var_b + var_w / (2 pi) * s * (sin th + (pi - th) fr),  s = sqrt(b c),  fr = a / s,  th = acos(clip(fr))   kernels.py:176-183
    const double s = sqrt(b * c);
    const double fr = a / s;
    const double frc = fmin(fmax(fr, -1.0 + 1e-7), 1.0 - 1e-7);
    const double th = acos(frc);
    const double t = sin(th) + (pi - th) * fr;
    v = var_b + var_w / (2.0 * pi) * s * t;
    // ds = (db c + b dc) / (2 s);  dfr = da / s - fr ds / s;  dth = -dfrc / sqrt(1 - frc^2) (0 where clipped);
    // dt = cos th dth - fr dth + (pi - th) dfr, and cos th = frc, so the first two terms cancel wherever dth != 0
    const double dsb = (bb * c + b * cb) / (2.0 * s), dsw = (bw * c + b * cw) / (2.0 * s);
    const double dfb = ab / s - fr * dsb / s, dfw = aw / s - fr * dsw / s;
    const double dtb = (pi - th) * dfb, dtw = (pi - th) * dfw;
    const double cst = var_w / (2.0 * pi);
    gb = 1.0 + cst * (dsb * t + s * dtb);
    gw = s * t / (2.0 * pi) + cst * (dsw * t + s * dtw);
}

// chain[(i * depth + l) * 3 + {0, 1, 2}] = k11^(l), dk11^(l)/dvar_b, dk11^(l)/dvar_w of point i, l = 0..depth-1.
// The draw of a batch is blockIdx.z (theta and chain `bstride` doubles apart).
__global__ void nngp_self_kernel(const double* __restrict__ X, int64_t n, int d, int kind, const double* __restrict__ theta,
                                 double* __restrict__ chain, int64_t bstride) {
    theta += (int64_t)blockIdx.z * bstride;
    chain += (int64_t)blockIdx.z * bstride;
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const bool relu = kind == B2GP_KERNEL_NNGP_RELU;
    const int depth = (int)theta[0];
    const double var_w = theta[d], var_b = theta[d + 2];
    const double xx = nngp_dot_self(X + i * d, d);
    double k = var_b + var_w * xx / d, kb = 1.0, kw = xx / d;     // depth 0, kernels.py:139-140
    double* out = chain + i * depth * 3;
    for (int l = 0; l < depth; ++l) {
        out[3 * l] = k;
        out[3 * l + 1] = kb;
        out[3 * l + 2] = kw;
        double v, gb, gw;
        nngp_step_fwd(relu, k, kb, kw, k, kb, kw, k, kb, kw, var_b, var_w, v, gb, gw);
        k = v;
        kb = gb;
        kw = gw;
    }
}

// Shared memory of mll_nngp_grad_kernel: rows and columns of X, then their self-chains.  The lanes of a warp read 32
// consecutive columns, so each row is padded to an odd number of doubles (no bank conflicts at d = 64 or 16 layers).
__host__ __device__ __forceinline__ int nngp_odd(int n) { return n | 1; }
static inline size_t nngp_grad_smem(int d, int depth) {
    return (size_t)(2 * MLL_TILE * nngp_odd(d) + 2 * MLL_TILE * nngp_odd(3 * depth)) * sizeof(double);
}

// partial[block * 3 + {0, 1, 2}]: sums over the block's lower-triangle entries (off-diagonal entries weighted 2) of
// W_ij dK_ij/dlog var_w, W_ii noise (the diagonal's noise term), W_ij dK_ij/dlog var_b.  Blocks above the diagonal write
// zeros.  Fixed order: each thread's entries in sequence, warp shuffles, then the 8 warps in order.  The draw of a batch
// is blockIdx.z: theta, chain, alpha, Kinv and partial `bstride` doubles apart, X shared.
__global__ void __launch_bounds__(NNGP_THREADS)
mll_nngp_grad_kernel(const double* __restrict__ X, int64_t N, int d, int kind, const double* __restrict__ theta,
                     const double* __restrict__ chain, const double* __restrict__ alpha, const double* __restrict__ Kinv, int64_t ldk,
                     double* __restrict__ partial, int64_t bstride) {
    extern __shared__ __align__(16) double sm[];
    __shared__ double red[NNGP_THREADS / 32][3];
    {
        const int64_t boff = (int64_t)blockIdx.z * bstride;
        theta += boff;
        chain += boff;
        alpha += boff;
        Kinv += boff;
        partial += boff;
    }
    const int64_t ti = blockIdx.y, tj = blockIdx.x;
    const int depth = (int)theta[0];
    double accW = 0.0, accN = 0.0, accB = 0.0;
    if (tj <= ti) {
        const int ldx = nngp_odd(d), nc = 3 * depth, ldc = nngp_odd(nc);
        double* Xr = sm;                        // [MLL_TILE][ldx]
        double* Xc = Xr + MLL_TILE * ldx;       // [MLL_TILE][ldx]
        double* Cr = Xc + MLL_TILE * ldx;       // [MLL_TILE][ldc]: depth x (k11, dk11/dvar_b, dk11/dvar_w)
        double* Cc = Cr + MLL_TILE * ldc;
        const int64_t r0 = ti * MLL_TILE, c0 = tj * MLL_TILE;
        for (int idx = threadIdx.x; idx < MLL_TILE * d; idx += NNGP_THREADS) {
            const int r = idx / d, k = idx % d;
            Xr[r * ldx + k] = (r0 + r < N) ? X[r0 * d + idx] : 0.0;
            Xc[r * ldx + k] = (c0 + r < N) ? X[c0 * d + idx] : 0.0;
        }
        for (int idx = threadIdx.x; idx < MLL_TILE * nc; idx += NNGP_THREADS) {
            const int r = idx / nc, k = idx % nc;
            Cr[r * ldc + k] = (r0 + r < N) ? chain[r0 * nc + idx] : 0.0;
            Cc[r * ldc + k] = (c0 + r < N) ? chain[c0 * nc + idx] : 0.0;
        }
        __syncthreads();
        const bool relu = kind == B2GP_KERNEL_NNGP_RELU;
        const double var_w = theta[d], noise = theta[d + 1], var_b = theta[d + 2];
        for (int e = threadIdx.x; e < MLL_TILE * MLL_TILE; e += NNGP_THREADS) {
            const int li = e / MLL_TILE, lj = e % MLL_TILE;
            const int64_t i = r0 + li, j = c0 + lj;
            if (i >= N || j > i) continue;
            const double W = (alpha[i] * alpha[j] - Kinv[i * ldk + j]) * ((i == j) ? 1.0 : 2.0);
            const double* xi = Xr + li * ldx;
            const double* xj = Xc + lj * ldx;
            double xz = 0.0;
            for (int k = 0; k < d; ++k) xz = fma(xi[k], xj[k], xz);
            double k12 = var_b + var_w * xz / d, gb = 1.0, gw = xz / d;      // depth 0
            const double* ci = Cr + li * ldc;
            const double* cj = Cc + lj * ldc;
            for (int l = 0; l < depth; ++l) {
                double v, nb, nw;
                nngp_step_fwd(relu, k12, gb, gw, ci[3 * l], ci[3 * l + 1], ci[3 * l + 2], cj[3 * l], cj[3 * l + 1], cj[3 * l + 2],
                              var_b, var_w, v, nb, nw);
                k12 = v;
                gb = nb;
                gw = nw;
            }
            accW += W * gw * var_w;
            accB += W * gb * var_b;
            if (i == j) accN += W * noise;
        }
    }
    double v[3] = {accW, accN, accB};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5][k] = v[k];
    }
    __syncthreads();
    if (threadIdx.x < 3) {
        double s = 0.0;
        for (int w = 0; w < NNGP_THREADS / 32; ++w) s += red[w][threadIdx.x];
        partial[((int64_t)blockIdx.y * gridDim.x + blockIdx.x) * 3 + threadIdx.x] = s;
    }
}

// the depth of an NNGP theta: an integer in [0, NNGP_MAX_DEPTH], else an error with a message
static inline int nngp_check_depth(b2gp_ctx* ctx, const char* who, double depth) {
    if (!(depth >= 0.0) || depth != (double)(int64_t)depth)
        return set_err(ctx, B2GP_ERR_ARG, who, "NNGP depth (theta[0]) must be a non-negative integer", __FILE__, __LINE__);
    if (depth > NNGP_MAX_DEPTH)
        return set_err(ctx, B2GP_ERR_UNSUPPORTED, who, "NNGP depth (theta[0]) is at most 16", __FILE__, __LINE__);
    return B2GP_OK;
}

static inline bool is_nngp(int kind) { return kind == B2GP_KERNEL_NNGP_ERF || kind == B2GP_KERNEL_NNGP_RELU; }
