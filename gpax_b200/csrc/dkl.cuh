// dkl.cuh -- deep kernel learning: the MLP feature extractor z = MLP(X) and the gradient of the exact-GP log marginal
// likelihood w.r.t. the GP inputs z, which the MLP's backward pass turns into gradients w.r.t. its weights.
//
// The reference's models are viDKL (gpax/models/vidkl.py: 3-layer ReLU MLP, haiku) and DKL (gpax/models/dkl.py:167-177: tanh
// MLP).  Dense layers H_{l+1} = act(H_l W_l + b_l), no activation after the last one.  The products run on gemm_nt (DMMA);
// here are the pieces around them: the bias + activation epilogue, its backward mask, the bias gradient (a fixed-order
// column sum) and a transpose for operands in the wrong orientation.
//
// mll_dz_kernel:  d/dz_i log N(y; 0, K(z)) = 1/2 sum_jl W_jl dK_jl/dz_i with W = alpha alpha^T - K^{-1}.  z_i enters row i
// and column i of K, so the 1/2 cancels:
//     g_i[k] = sum_{j != i} W_ij dk(z_i, z_j)/dz_i[k]
// (k(z, z) is constant for the three stationary kernels, and the noise and jitter on the diagonal do not depend on z).
// The derivatives are gram_dx_kernel's (grad.cuh): the reference's formulas as written.  K^{-1} exists as its lower
// triangle only (mll_impl's SYRK), so W_ij is read at [max(i,j), min(i,j)].  One CTA owns DZ_ROWS rows and walks all
// columns in tiles: for tiles left of the diagonal the rows of K^{-1} are read, right of it the columns (as rows j,
// consecutive i) -- both coalesced; every entry of the lower triangle is read twice, N^2 doubles in all.  Each row's sum
// is accumulated in a fixed order and reduced across the row's threads by a fixed shuffle tree: deterministic, no atomics.
//
// mlp_input_vjp_kernel (bottom of the file): the network's vector-Jacobian product w.r.t. its inputs, which turns the
// posterior's gradient w.r.t. z into the gradient w.r.t. the raw test inputs (b2gp_dkl_posterior_grad, optimize_acq).
#pragma once
#include "common.cuh"
#include "grad.cuh"
#include "mll.cuh"
#include "mtgp.cuh"

constexpr int DZ_ROWS = 32;      // rows i per CTA
constexpr int DZ_COLS = 32;      // columns j per tile
constexpr int DZ_THREADS = 256;  // 8 threads per row, 4 columns each per tile
constexpr int DZ_TPR = DZ_THREADS / DZ_ROWS;

__global__ void __launch_bounds__(DZ_THREADS)
mll_dz_kernel(int kind, const double* __restrict__ Z, int64_t N, int d, const double* __restrict__ theta,
              const double* __restrict__ alpha, const double* __restrict__ Kinv, int64_t ldk, double* __restrict__ G) {
    __shared__ double Ws[DZ_ROWS][DZ_COLS + 1];
    __shared__ double Zi[DZ_ROWS][MLL_MAX_D];
    __shared__ double Zj[DZ_COLS][MLL_MAX_D];
    __shared__ double ell[MLL_MAX_D];
    const int tid = threadIdx.x;
    const int64_t i0 = (int64_t)blockIdx.x * DZ_ROWS;
    const bool periodic = (kind == B2GP_KERNEL_PERIODIC);
    const double scale = theta[d], period = theta[d + 2];
    if (tid < d) ell[tid] = theta[tid];
    __syncthreads();
    // staged as gram_dx_kernel stages them: divided by the lengthscale for RBF / Matern, raw for periodic
    for (int idx = tid; idx < DZ_ROWS * d; idx += DZ_THREADS) {
        const int r = idx / d, k = idx % d;
        const int64_t gi = i0 + r;
        const double v = gi < N ? Z[gi * d + k] : 0.0;
        Zi[r][k] = periodic ? v : v / ell[k];
    }
    const int r = tid / DZ_TPR, q = tid % DZ_TPR;
    const int64_t i = i0 + r;
    double acc[MLL_MAX_D];
#pragma unroll
    for (int k = 0; k < MLL_MAX_D; ++k) acc[k] = 0.0;
    for (int64_t j0 = 0; j0 < N; j0 += DZ_COLS) {
        __syncthreads();
        for (int idx = tid; idx < DZ_ROWS * DZ_COLS; idx += DZ_THREADS) {
            // left of the diagonal block: consecutive threads along a row of K^{-1}; right of it: along a column
            const bool left = j0 < i0;
            const int rr = left ? idx / DZ_COLS : idx % DZ_ROWS, cc = left ? idx % DZ_COLS : idx / DZ_ROWS;
            const int64_t gi = i0 + rr, gj = j0 + cc;
            double w = 0.0;
            if (gi < N && gj < N && gi != gj) {
                const int64_t hi = gi > gj ? gi : gj, lo = gi > gj ? gj : gi;
                w = alpha[gi] * alpha[gj] - Kinv[hi * ldk + lo];
            }
            Ws[rr][cc] = w;
        }
        for (int idx = tid; idx < DZ_COLS * d; idx += DZ_THREADS) {
            const int c = idx / d, k = idx % d;
            const int64_t gj = j0 + c;
            const double v = gj < N ? Z[gj * d + k] : 0.0;
            Zj[c][k] = periodic ? v : v / ell[k];
        }
        __syncthreads();
        if (i >= N) continue;
        for (int c = q; c < DZ_COLS; c += DZ_TPR) {
            const double w = Ws[r][c];
            if (w == 0.0) continue;     // outside the matrix, the diagonal, or an exact zero: contributes nothing
            if (periodic) {
                // gram_dx_kernel's derivative -2 pi sin(2 a_k) / (period l_k^2) k: one sincos per dimension, the terms kept
                // in registers (fully unrolled) until the exponent is known
                double s = 0.0, t[MLL_MAX_D];
#pragma unroll
                for (int k = 0; k < MLL_MAX_D; ++k) {
                    t[k] = 0.0;
                    if (k < d) {
                        double sa, ca;
                        sincos(3.141592653589793 * (Zi[r][k] - Zj[c][k]) / period, &sa, &ca);
                        const double a = sa / ell[k];
                        s += a * a;
                        t[k] = -(4.0 * 3.141592653589793) * sa * ca / (period * ell[k] * ell[k]);
                    }
                }
                const double wk = w * (scale * exp(-2.0 * s));
#pragma unroll
                for (int k = 0; k < MLL_MAX_D; ++k)
                    if (k < d) acc[k] = fma(wk, t[k], acc[k]);
                continue;
            }
            double x2 = 0.0, xz = 0.0, z2 = 0.0;
#pragma unroll
            for (int k = 0; k < MLL_MAX_D; ++k) {
                if (k < d) {
                    x2 = fma(Zi[r][k], Zi[r][k], x2);
                    xz = fma(Zi[r][k], Zj[c][k], xz);
                    z2 = fma(Zj[c][k], Zj[c][k], z2);
                }
            }
            const double wg = w * stationary_dk_dr2(kind, (x2 - 2.0 * xz) + z2, scale);
#pragma unroll
            for (int k = 0; k < MLL_MAX_D; ++k)
                if (k < d) acc[k] = fma(wg, 2.0 * (Zi[r][k] - Zj[c][k]) / ell[k], acc[k]);
        }
    }
    // the DZ_TPR threads of a row are consecutive lanes: a fixed xor tree
#pragma unroll
    for (int k = 0; k < MLL_MAX_D; ++k) {
        if (k < d) {
            double v = acc[k];
#pragma unroll
            for (int o = DZ_TPR / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
            acc[k] = v;
        }
    }
    if (q == 0 && i < N) {
#pragma unroll
        for (int k = 0; k < MLL_MAX_D; ++k)
            if (k < d) G[i * d + k] = acc[k];
    }
}

// mll_lcm_dz_kernel: the same gradient for the LCM covariance of gram_lcm_kernel (mtgp.cuh, viMTDKL):
//     g_i[k] = sum_{j != i} W_ij sum_q B_q[t_i, t_j] dk_q(z_i, z_j)/dz_i[k]
// with latent q's lengthscales ell_q and scale.  The jitter, the noise (L times on the diagonal) and the same-point jitter
// block of the Kronecker form do not depend on z; pairs at one point have z_i = z_j and contribute exactly zero.  RBF and
// Matern only (the reference's viMTDKL samples no period).  mll_dz_kernel's tiling, K^{-1} access and fixed reduction
// order; theta_q and B_q of every latent staged in shared memory as gram_lcm_kernel does, the row and column tiles once
// per latent (scaled by 1 / ell_q), the task ids once.
__global__ void __launch_bounds__(DZ_THREADS)
mll_lcm_dz_kernel(int kind, const double* __restrict__ Z, const int* __restrict__ task, int64_t N, int d, int T, int L,
                  const double* __restrict__ theta, const double* __restrict__ B, const double* __restrict__ alpha,
                  const double* __restrict__ Kinv, int64_t ldk, double* __restrict__ G) {
    __shared__ double Ws[DZ_ROWS][DZ_COLS + 1];
    __shared__ double Zi[MT_MAX_L][DZ_ROWS][MLL_MAX_D];
    __shared__ double Zj[MT_MAX_L][DZ_COLS][MLL_MAX_D];
    __shared__ double th[MT_MAX_L * (MLL_MAX_D + 2)];
    __shared__ double Bs[MT_MAX_L * MT_MAX_T * MT_MAX_T];
    __shared__ int ti[DZ_ROWS], tj[DZ_COLS];
    const int tid = threadIdx.x, nth = d + 2;
    const int64_t i0 = (int64_t)blockIdx.x * DZ_ROWS;
    for (int idx = tid; idx < L * nth; idx += DZ_THREADS) th[idx] = theta[idx];
    for (int idx = tid; idx < L * T * T; idx += DZ_THREADS) Bs[idx] = B[idx];
    if (tid < DZ_ROWS) ti[tid] = i0 + tid < N ? task[i0 + tid] : 0;
    __syncthreads();
    for (int idx = tid; idx < L * DZ_ROWS * d; idx += DZ_THREADS) {
        const int q = idx / (DZ_ROWS * d), r = (idx / d) % DZ_ROWS, k = idx % d;
        const int64_t gi = i0 + r;
        Zi[q][r][k] = (gi < N ? Z[gi * d + k] : 0.0) / th[q * nth + k];
    }
    const int r = tid / DZ_TPR, c0 = tid % DZ_TPR;
    const int64_t i = i0 + r;
    double acc[MLL_MAX_D];
#pragma unroll
    for (int k = 0; k < MLL_MAX_D; ++k) acc[k] = 0.0;
    for (int64_t j0 = 0; j0 < N; j0 += DZ_COLS) {
        __syncthreads();
        for (int idx = tid; idx < DZ_ROWS * DZ_COLS; idx += DZ_THREADS) {
            // left of the diagonal block: consecutive threads along a row of K^{-1}; right of it: along a column
            const bool left = j0 < i0;
            const int rr = left ? idx / DZ_COLS : idx % DZ_ROWS, cc = left ? idx % DZ_COLS : idx / DZ_ROWS;
            const int64_t gi = i0 + rr, gj = j0 + cc;
            double w = 0.0;
            if (gi < N && gj < N && gi != gj) {
                const int64_t hi = gi > gj ? gi : gj, lo = gi > gj ? gj : gi;
                w = alpha[gi] * alpha[gj] - Kinv[hi * ldk + lo];
            }
            Ws[rr][cc] = w;
        }
        for (int idx = tid; idx < L * DZ_COLS * d; idx += DZ_THREADS) {
            const int q = idx / (DZ_COLS * d), c = (idx / d) % DZ_COLS, k = idx % d;
            const int64_t gj = j0 + c;
            Zj[q][c][k] = (gj < N ? Z[gj * d + k] : 0.0) / th[q * nth + k];
        }
        if (tid < DZ_COLS) tj[tid] = j0 + tid < N ? task[j0 + tid] : 0;
        __syncthreads();
        if (i >= N) continue;
        for (int c = c0; c < DZ_COLS; c += DZ_TPR) {
            const double w = Ws[r][c];
            if (w == 0.0) continue;     // outside the matrix, the diagonal, or an exact zero: contributes nothing
            const double* Bp = Bs + ti[r] * T + tj[c];
            for (int q = 0; q < L; ++q) {
                const double* zi = Zi[q][r];
                const double* zj = Zj[q][c];
                const double* ell = th + q * nth;
                double x2 = 0.0, xz = 0.0, z2 = 0.0;
#pragma unroll
                for (int k = 0; k < MLL_MAX_D; ++k) {
                    if (k < d) {
                        x2 = fma(zi[k], zi[k], x2);
                        xz = fma(zi[k], zj[k], xz);
                        z2 = fma(zj[k], zj[k], z2);
                    }
                }
                const double wg = w * Bp[q * T * T] * stationary_dk_dr2(kind, (x2 - 2.0 * xz) + z2, ell[d]);
#pragma unroll
                for (int k = 0; k < MLL_MAX_D; ++k)
                    if (k < d) acc[k] = fma(wg, 2.0 * (zi[k] - zj[k]) / ell[k], acc[k]);
            }
        }
    }
    // the DZ_TPR threads of a row are consecutive lanes: a fixed xor tree
#pragma unroll
    for (int k = 0; k < MLL_MAX_D; ++k) {
        if (k < d) {
            double v = acc[k];
#pragma unroll
            for (int o = DZ_TPR / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
            acc[k] = v;
        }
    }
    if (c0 == 0 && i < N) {
#pragma unroll
        for (int k = 0; k < MLL_MAX_D; ++k)
            if (k < d) G[i * d + k] = acc[k];
    }
}

// G[p, k] = sum_{t < group} Gr[p * group + t, k]: a point's gradient from its `group` rows (the Kronecker form), in task order
__global__ void group_sum_kernel(const double* __restrict__ Gr, int64_t n, int d, int group, double* __restrict__ G) {
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < n * d; idx += (int64_t)gridDim.x * blockDim.x) {
        const int64_t p = idx / d;
        const int k = (int)(idx % d);
        double s = 0.0;
        for (int t = 0; t < group; ++t) s += Gr[(p * group + t) * d + k];
        G[idx] = s;
    }
}

// ---- MLP pieces.  Row-major [rows, cols] with leading dimension ld.
enum { DKL_ACT_NONE = -1 };   // the last layer; B2GP_ACT_RELU / B2GP_ACT_TANH otherwise

// H = act(H + b)
__global__ void mlp_bias_act_kernel(double* __restrict__ H, int64_t ld, int64_t rows, int cols, const double* __restrict__ b, int act) {
    const int64_t total = rows * cols;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = idx / cols;
        const int j = (int)(idx % cols);
        double v = H[i * ld + j] + b[j];
        if (act == B2GP_ACT_RELU) v = v > 0.0 ? v : 0.0;
        else if (act == B2GP_ACT_TANH) v = tanh(v);
        H[i * ld + j] = v;
    }
}

// G *= act'(pre-activation), from the stored activation H: ReLU (h > 0), tanh (1 - h^2)
__global__ void mlp_act_grad_kernel(double* __restrict__ G, int64_t ldg, const double* __restrict__ H, int64_t ldh, int64_t rows,
                                    int cols, int act) {
    const int64_t total = rows * cols;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = idx / cols;
        const int j = (int)(idx % cols);
        const double h = H[i * ldh + j];
        const double m = act == B2GP_ACT_RELU ? (h > 0.0 ? 1.0 : 0.0) : 1.0 - h * h;
        G[i * ldg + j] *= m;
    }
}

// out[j] = sum_i G[i, j]: one CTA per column, strided partial sums then a fixed tree (deterministic)
constexpr int MLP_SUM_THREADS = 256;
__global__ void __launch_bounds__(MLP_SUM_THREADS)
mlp_colsum_kernel(const double* __restrict__ G, int64_t ld, int64_t rows, double* __restrict__ out) {
    __shared__ double red[MLP_SUM_THREADS];
    const int j = blockIdx.x;
    double s = 0.0;
    for (int64_t i = threadIdx.x; i < rows; i += MLP_SUM_THREADS) s += G[i * ld + j];
    red[threadIdx.x] = s;
    __syncthreads();
    for (int o = MLP_SUM_THREADS / 2; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) out[j] = red[0];
}

// B[c, r] = A[r, c]  (A [rows, cols] with lda, B [cols, rows] with ldb), 32 x 32 tiles through shared memory
__global__ void mlp_transpose_kernel(const double* __restrict__ A, int64_t lda, int64_t rows, int64_t cols, double* __restrict__ B,
                                     int64_t ldb) {
    __shared__ double t[32][33];
    const int64_t r0 = (int64_t)blockIdx.y * 32, c0 = (int64_t)blockIdx.x * 32;
    for (int y = threadIdx.y; y < 32; y += blockDim.y) {
        const int64_t r = r0 + y, c = c0 + threadIdx.x;
        if (r < rows && c < cols) t[y][threadIdx.x] = A[r * lda + c];
    }
    __syncthreads();
    for (int y = threadIdx.y; y < 32; y += blockDim.y) {
        const int64_t c = c0 + y, r = r0 + threadIdx.x;
        if (r < rows && c < cols) B[c * ldb + r] = t[threadIdx.x][y];
    }
}

static int launch_transpose(b2gp_ctx* ctx, cudaStream_t st, const double* A, int64_t lda, int64_t rows, int64_t cols, double* B,
                            int64_t ldb) {
    if (rows <= 0 || cols <= 0) return B2GP_OK;
    dim3 grid((unsigned)ceil_div(cols, 32), (unsigned)ceil_div(rows, 32));
    return launch(ctx, st, grid, dim3(32, 8), 0, mlp_transpose_kernel, A, lda, rows, cols, B, ldb);
}

// ---- mlp_input_vjp_kernel: the network's input vector-Jacobian product for the posterior's gradient w.r.t. raw inputs
// (b2gp_dkl_posterior_grad).  Per weight set s, test point p and cotangent row r (d mean / dz, d var / dz):
//     G = cot[r][s, p, :]                                   (the last layer has no activation)
//     G <- (G W_l^T) * act'(H_l[p])   for l = L-1 .. 1       act' from the stored post-activation: ReLU h > 0, tanh 1 - h^2
//     dX[s, r, p, :] = G W_0^T
// mlp_backward_dev's recursion continued one layer further down, for one row instead of N.  One launch covers every
// (s, p, r): a CTA owns one (s, p) and all R rows, so each weight it reads serves R products.  Entry i of G W_l^T is
// row i of W_l [in, out] (row-major, coalesced) dotted with G: one warp per row, lanes striding the row in a fixed
// order, a fixed xor tree across the warp -- identical calls give identical bits.  The G vectors ping-pong between two
// [R][wmax] buffers: shared memory, or (hidden widths too wide for it) a per-CTA slice of global scratch through the same
// code.  The bottom layer is tiled over the input dimension D: grid.y CTAs per (s, p) take VJP_TILE input rows each and
// each recomputes the (small) layers above it, so wide inputs spread over the machine and no buffer grows with D.
constexpr int VJP_THREADS = 256;
constexpr int VJP_WARPS = VJP_THREADS / 32;
constexpr int VJP_TILE = 64;           // input rows of the bottom layer per CTA
constexpr int VJP_MAX_R = 2;
constexpr int VJP_MAX_LAYERS = 64;     // mlp_shape's bound
constexpr size_t VJP_SMEM_MAX = 48 * 1024;   // the G buffers go to global scratch above this (no opt-in needed below it)

struct VjpNet {
    int L, R;
    int64_t width[VJP_MAX_LAYERS + 1];   // width[0] = D, width[l + 1] = out_l
    int64_t woff[VJP_MAX_LAYERS];        // W_l's offset in a weight set's flat parameters
};

__global__ void __launch_bounds__(VJP_THREADS)
mlp_input_vjp_kernel(VjpNet net, const double* __restrict__ params, int64_t pstride, const double* __restrict__ Hk, int64_t hstride,
                     int64_t P, int act, const double* __restrict__ cot0, const double* __restrict__ cot1, double* __restrict__ dX,
                     double* gscratch, int64_t wmax) {
    extern __shared__ __align__(16) double vjp_sm[];
    const int64_t sp = blockIdx.x;                       // s * P + p
    const int64_t s = sp / P, p = sp % P;
    const int L = net.L, R = net.R;
    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
    double* buf = gscratch ? gscratch + ((int64_t)blockIdx.y * gridDim.x + blockIdx.x) * 2 * VJP_MAX_R * wmax : vjp_sm;
    double* G = buf;                                     // G[r * wmax + j]
    double* Gn = buf + VJP_MAX_R * wmax;
    const double* Ps = params + s * pstride;
    const int64_t dz = net.width[L];
    for (int64_t j = threadIdx.x; j < dz; j += VJP_THREADS) {
        G[j] = cot0[sp * dz + j];
        if (R > 1) G[wmax + j] = cot1[sp * dz + j];
    }
    // H_l (l >= 1) of this weight set: [P, width[l]] blocks one after the other, each padded to 8 doubles
    int64_t hoff = 0;
    for (int l = 1; l + 1 < L; ++l) hoff += (P * net.width[l] + 7) / 8 * 8;
    for (int l = L - 1; l >= 1; --l) {
        __syncthreads();
        const int64_t in = net.width[l], out = net.width[l + 1];
        const double* W = Ps + net.woff[l];
        const double* H = Hk + s * hstride + hoff + p * in;
        for (int64_t i = warp; i < in; i += VJP_WARPS) {
            double a0 = 0.0, a1 = 0.0;
            for (int64_t j = lane; j < out; j += 32) {
                const double w = W[i * out + j];
                a0 = fma(w, G[j], a0);
                if (R > 1) a1 = fma(w, G[wmax + j], a1);
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                a0 += __shfl_xor_sync(0xffffffffu, a0, o);
                a1 += __shfl_xor_sync(0xffffffffu, a1, o);
            }
            if (lane == 0) {
                const double h = H[i];
                const double m = act == B2GP_ACT_RELU ? (h > 0.0 ? 1.0 : 0.0) : 1.0 - h * h;
                Gn[i] = a0 * m;
                if (R > 1) Gn[wmax + i] = a1 * m;
            }
        }
        double* t = G;
        G = Gn;
        Gn = t;
        if (l > 1) hoff -= (P * net.width[l - 1] + 7) / 8 * 8;
    }
    __syncthreads();
    // bottom layer: this CTA's VJP_TILE rows of W_0 [D, width[1]]
    const int64_t D = net.width[0], out = net.width[1];
    const double* W = Ps + net.woff[0];
    const int64_t i1 = D < ((int64_t)blockIdx.y + 1) * VJP_TILE ? D : ((int64_t)blockIdx.y + 1) * VJP_TILE;
    for (int64_t i = (int64_t)blockIdx.y * VJP_TILE + warp; i < i1; i += VJP_WARPS) {
        double a0 = 0.0, a1 = 0.0;
        for (int64_t j = lane; j < out; j += 32) {
            const double w = W[i * out + j];
            a0 = fma(w, G[j], a0);
            if (R > 1) a1 = fma(w, G[wmax + j], a1);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            a0 += __shfl_xor_sync(0xffffffffu, a0, o);
            a1 += __shfl_xor_sync(0xffffffffu, a1, o);
        }
        if (lane == 0) {
            double* o = dX + ((s * R) * P + p) * D + i;   // dX [S, R, P, D]
            o[0] = a0;
            if (R > 1) o[P * D] = a1;
        }
    }
}
