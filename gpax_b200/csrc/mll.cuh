// mll.cuh -- log marginal likelihood of the exact GP and its gradient w.r.t. the log hyper-parameters.
//
// The fit-side hot loop of the reference is the likelihood inside ExactGP.model (gpax/models/gp.py:158-164):
// MultivariateNormal(f_loc, covariance_matrix=k).log_prob(y) -- Cholesky, triangular solve, log-det -- and
// its reverse-mode derivative, evaluated once per SVI step (vigp.py:108-120) or per NUTS leapfrog
// (gp.py:207-218).  Here:
//     value = -1/2 y^T K^{-1} y - sum_i log L_ii - N/2 log(2 pi)
//     d value / d log(theta) = 1/2 sum_ij (alpha_i alpha_j - [K^{-1}]_ij) dK_ij/dlog(theta),  alpha = K^{-1} y
// K^{-1} = L^{-T} L^{-1} is formed with the same DMMA kernels (triangular solve of the identity, then SYRK);
// the reduction against dK/dtheta recomputes K_ij and its derivatives on the fly from X (no N x N derivative
// matrices), one fixed-order two-pass reduction (deterministic).
#pragma once
#include "common.cuh"
#include "gram.cuh"

constexpr int MLL_MAX_D = 16;
constexpr int MLL_TILE = 64;
constexpr int MLL_THREADS = 256;

__global__ void set_identity_kernel(double* B, int64_t ld, int64_t n) {
    const int64_t total = n * n;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = idx / n, j = idx % n;
        B[i * ld + j] = (i == j) ? 1.0 : 0.0;
    }
}

// out[0] = sum_i log L_ii   (single block, fixed order)
__global__ void logdiag_kernel(const double* L, int64_t ld, int64_t n, double* out) {
    __shared__ double red[256];
    double s = 0.0;
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) s += log(L[i * ld + i]);
    red[threadIdx.x] = s;
    __syncthreads();
    for (int o = blockDim.x / 2; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) out[0] = red[0];
}

// partial[block][k], k in [0, d+3): sums over the lower triangle (off-diagonal entries weighted 2) of
//   W_ij * dK_ij/dlog(lengthscale_k) (k < d), dlog(scale) (k = d), dlog(noise) (k = d+1), dlog(period) (k = d+2)
// with W_ij = alpha_i alpha_j - Kinv_ij.
__global__ void __launch_bounds__(MLL_THREADS)
mll_grad_kernel(const double* __restrict__ X, int64_t N, int d, int kind, const double* __restrict__ theta,
                const double* __restrict__ alpha, const double* __restrict__ Kinv, int64_t ldk, double* __restrict__ partial) {
    __shared__ double red[MLL_THREADS / 32][MLL_MAX_D + 3];
    const int64_t ti = blockIdx.y, tj = blockIdx.x;
    const int nout = d + 3;
    double acc[MLL_MAX_D + 3];
#pragma unroll
    for (int k = 0; k < MLL_MAX_D + 3; ++k) acc[k] = 0.0;
    if (tj <= ti) {
        const double scale = theta[d], noise = theta[d + 1], period = theta[d + 2];
        const int64_t r0 = ti * MLL_TILE, c0 = tj * MLL_TILE;
        for (int e = threadIdx.x; e < MLL_TILE * MLL_TILE; e += MLL_THREADS) {
            const int64_t i = r0 + e / MLL_TILE, j = c0 + e % MLL_TILE;
            if (i >= N || j > i) continue;
            const double wgt = (i == j) ? 1.0 : 2.0;
            const double W = (alpha[i] * alpha[j] - Kinv[i * ldk + j]) * wgt;
            if (kind == B2GP_KERNEL_PERIODIC) {
                double ssum = 0.0, dper = 0.0;
                double q[MLL_MAX_D];
                for (int k = 0; k < d; ++k) {
                    const double a = 3.141592653589793 * (X[i * d + k] - X[j * d + k]) / period;
                    const double sn = sin(a), l2 = theta[k] * theta[k];
                    q[k] = sn * sn / l2;
                    ssum += q[k];
                    dper += 2.0 * sn * cos(a) * a / l2;      // d/dlog(period) of -2 sum sin^2(a)/l^2  is  +4 sin cos a / l^2 ... halved below
                }
                const double Kij = scale * exp(-2.0 * ssum);
                for (int k = 0; k < d; ++k) acc[k] += W * Kij * 4.0 * q[k];
                acc[d] += W * Kij;
                acc[d + 2] += W * Kij * 2.0 * dper;
            } else {
                double r2 = 0.0;
                double q[MLL_MAX_D];
                for (int k = 0; k < d; ++k) {
                    const double dl = (X[i * d + k] - X[j * d + k]) / theta[k];
                    q[k] = dl * dl;
                    r2 += q[k];
                }
                double Kij, dK;  // dK = -2 * dK/d(r2): dK/dlog(l_k) = dK * q_k
                if (kind == B2GP_KERNEL_RBF) {
                    Kij = scale * exp(-0.5 * r2);
                    dK = Kij;
                } else {
                    const double r = sqrt(r2 + 1e-12), s5r = 2.23606797749979 * r, ex = exp(-s5r);
                    Kij = scale * (1.0 + s5r + (5.0 / 3.0) * r2) * ex;
                    dK = (5.0 / 3.0) * scale * (1.0 + s5r) * ex;
                }
                for (int k = 0; k < d; ++k) acc[k] += W * dK * q[k];
                acc[d] += W * Kij;
            }
            if (i == j) acc[d + 1] += W * noise;
        }
    }
    for (int k = 0; k < nout; ++k) {
        double v = acc[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5][k] = v;
    }
    __syncthreads();
    if ((int)threadIdx.x < nout) {
        double v = 0.0;
        for (int w = 0; w < MLL_THREADS / 32; ++w) v += red[w][threadIdx.x];
        partial[((int64_t)blockIdx.y * gridDim.x + blockIdx.x) * nout + threadIdx.x] = v;
    }
}

// grad[k] = 1/2 sum_blocks partial[b][k]   (fixed order)
__global__ void mll_finish_kernel(const double* partial, int64_t nblocks, int nout, double* grad) {
    const int k = threadIdx.x;
    if (k >= nout) return;
    double s = 0.0;
    for (int64_t b = 0; b < nblocks; ++b) s += partial[b * nout + k];
    grad[k] = 0.5 * s;
}

// ---- caller-supplied Gram matrices (b2gp_mll_gram, b2gp_posterior_gram)
// A[i, j] = (K[i, j] + K[j, i]) / 2 for j <= i: the symmetric part the reference's Cholesky factors
// (MultivariateNormal(covariance_matrix=k)), written as the lower triangle the factorisation reads.  32 x 32 tiles, the
// transposed tile staged through shared memory so that both reads are coalesced.  An exactly symmetric K is copied
// bit for bit.
constexpr int GCOPY_TILE = 32;
__global__ void gram_copyin_kernel(const double* __restrict__ K, int64_t ldk, int64_t n, double* __restrict__ A, int64_t lda) {
    __shared__ double t[GCOPY_TILE][GCOPY_TILE + 1];
    if (blockIdx.x > blockIdx.y) return;
    const int64_t r0 = (int64_t)blockIdx.y * GCOPY_TILE, c0 = (int64_t)blockIdx.x * GCOPY_TILE;
    for (int y = threadIdx.y; y < GCOPY_TILE; y += blockDim.y) {
        const int64_t i = c0 + y, j = r0 + threadIdx.x;
        if (i < n && j < n) t[y][threadIdx.x] = K[i * ldk + j];   // K[c0 + y, r0 + x]
    }
    __syncthreads();
    for (int y = threadIdx.y; y < GCOPY_TILE; y += blockDim.y) {
        const int64_t i = r0 + y, j = c0 + threadIdx.x;
        if (i < n && j <= i) A[i * lda + j] = 0.5 * (K[i * ldk + j] + t[threadIdx.x][y]);
    }
}

// partial[block * pstride + k0 + k], k < p: sum over the block's 64 x 64 tile of the FULL matrix of W_ij dK_k[i, j], with
// W = alpha alpha^T - K^{-1} formed on the fly from alpha and the lower triangle of K^{-1} (no symmetry assumed of dK_k).
// The block's K^{-1} entries are staged through shared memory (an upper tile reads the transposed lower one), each
// thread keeps its 16 W values in registers, and every dK_k is read once against them: W is formed once per tile
// however many derivative matrices there are.  dK is a device array of p device pointers, leading dimension lddk.
// Fixed-order warp and block sums: identical calls give identical bits.
constexpr int TRACE_CHUNK = 32;   // derivative matrices per block-level reduction round
__global__ void __launch_bounds__(MLL_THREADS)
mll_gram_trace_kernel(const double* __restrict__ alpha, const double* __restrict__ Kinv, int64_t ldk, int64_t N,
                      const double* const* __restrict__ dK, int64_t lddk, int p, int k0, int pstride, double* __restrict__ partial) {
    constexpr int PER = MLL_TILE * MLL_TILE / MLL_THREADS;
    __shared__ double kin[MLL_TILE][MLL_TILE + 1];
    __shared__ double red[MLL_THREADS / 32][TRACE_CHUNK];
    const int64_t r0 = (int64_t)blockIdx.y * MLL_TILE, c0 = (int64_t)blockIdx.x * MLL_TILE;
    const int64_t R0 = r0 > c0 ? r0 : c0, C0 = r0 > c0 ? c0 : r0;   // the lower-triangle block holding this tile's K^{-1}
    for (int e = threadIdx.x; e < MLL_TILE * MLL_TILE; e += MLL_THREADS) {
        const int64_t x = e / MLL_TILE, y = e % MLL_TILE, i = R0 + x, j = C0 + y;
        kin[x][y] = (i < N && j <= i) ? Kinv[i * ldk + j] : 0.0;
    }
    __syncthreads();
    double W[PER];
    int64_t off[PER];
    const int b = threadIdx.x % MLL_TILE;
#pragma unroll
    for (int r = 0; r < PER; ++r) {
        const int a = threadIdx.x / MLL_TILE + r * (MLL_THREADS / MLL_TILE);
        const int64_t i = r0 + a, j = c0 + b;
        off[r] = -1;
        W[r] = 0.0;
        if (i < N && j < N) {
            const double kv = i >= j ? kin[i - R0][j - C0] : kin[j - R0][i - C0];
            W[r] = alpha[i] * alpha[j] - kv;
            off[r] = i * lddk + j;
        }
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int kc = 0; kc < p; kc += TRACE_CHUNK) {
        const int nk = p - kc < TRACE_CHUNK ? p - kc : TRACE_CHUNK;
        for (int kk = 0; kk < nk; ++kk) {
            const double* __restrict__ D = dK[kc + kk];
            double v = 0.0;
#pragma unroll
            for (int r = 0; r < PER; ++r)
                if (off[r] >= 0) v += W[r] * D[off[r]];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
            if (lane == 0) red[warp][kk] = v;
        }
        __syncthreads();
        if ((int)threadIdx.x < nk) {
            double v = 0.0;
            for (int w = 0; w < MLL_THREADS / 32; ++w) v += red[w][threadIdx.x];
            partial[((int64_t)blockIdx.y * gridDim.x + blockIdx.x) * pstride + k0 + kc + threadIdx.x] = v;
        }
        __syncthreads();
    }
}
