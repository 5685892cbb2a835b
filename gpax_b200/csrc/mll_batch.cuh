// mll_batch.cuh -- B independent exact-GP log marginal likelihoods in one launch (b2gp_mll_batch's small route).
//
// vExactGP (gpax/models/vgp.py:55-121) fits one GP per task with its own hyper-parameters, and UIGP (uigp.py:78-129) needs
// the likelihood's gradient w.r.t. all N x d inputs; both run at N of tens to a few hundred points, where one b2gp_mll
// call is ~15 launches and a synchronising copy.  Here member b of the batch is one CTA that keeps everything in shared
// memory:
//   1. K = k(X_b, X_b) + (noise + jitter) I, lower triangle, into the 128 x PD_LD tile S;
//   2. K = L L^T and inv(L) in place: potrf_diag_cta (potrf.cuh), DMMA panels and the 2 x 2 block inverse;
//   3. w = inv(L) y, alpha = inv(L)^T w, log det from the diagonal of inv(L), and K^{-1} = inv(L)^T inv(L) written into
//      S's upper triangle (i < j) and its padding column 128 (the diagonal), so the lower triangle stays intact;
//   4. the d+3 gradient sums over the lower triangle with mllb_grad_pair, the per-pair kernel derivatives recomputed from
//      X as mll_grad_kernel does, reduced in a fixed order (warp xor tree, then the warps in order);
//   5. on request the input gradient g_i[k] = sum_{j != i} W_ij dk(x_i, x_j)/dx_i[k] of mll_dz_kernel (dkl.cuh).
// Steps 3 and 4 walk the lower triangle by a linear index (mllb_tri), so every thread has work and a warp's trip counts
// are uniform; lengthscales and the period are used as reciprocals, and the feature loops are unrolled over MLL_MAX_D
// with a guard, so that the per-thread accumulators stay in registers.  Identical calls give identical bits; a member
// with a non-positive pivot sets only its own info word.
#pragma once
#include "common.cuh"
#include "dkl.cuh"
#include "gram.cuh"
#include "mll.cuh"
#include "potrf.cuh"

constexpr int MLLB_MAX_N = B2GP_LEAF;   // the tile: one potrf_diag leaf (128); the route's bound is B2GP_MLL_BATCH_SMALL_MAX_N
static_assert(B2GP_MLL_BATCH_SMALL_MAX_N <= MLLB_MAX_N, "the small route's bound must fit the shared tile");
constexpr int MLLB_KD = PD_LD - 4;      // the padding column of S that holds diag(K^{-1})
// shared memory: S [128 x PD_LD] + 32 reciprocal pivots | X [128 x MLL_MAX_D] | y, w, alpha, log L_ii [128 each]
//                | theta [MLL_MAX_D + 3] | 1 / lengthscale [MLL_MAX_D] | warp partials [8 x (MLL_MAX_D + 3)]
constexpr int MLLB_SMEM =
    PD_SMEM + (MLLB_MAX_N * MLL_MAX_D + 4 * MLLB_MAX_N + MLL_MAX_D + (MLL_MAX_D + 3) * (1 + PD_THREADS / 32)) * 8;

__device__ __forceinline__ double mllb_kinv(const double* S, int i, int j) {   // K^{-1}_ij from step 3's layout
    return i == j ? S[i * PD_LD + MLLB_KD] : i < j ? S[i * PD_LD + j] : S[j * PD_LD + i];
}

// e -> (r, c), c <= r: the row-major order of a lower triangle (e = r (r + 1) / 2 + c)
__device__ __forceinline__ void mllb_tri(int e, int& r, int& c) {
    int t = (int)((sqrtf(8.0f * (float)e + 1.0f) - 1.0f) * 0.5f);
    if ((t + 1) * (t + 2) / 2 <= e) ++t;
    if (t * (t + 1) / 2 > e) --t;
    r = t;
    c = e - t * (t + 1) / 2;
}

// One pair's terms of mll_grad_kernel's sums: accl[k] += W dK_ij/dlog(ell_k), as += W dK_ij/dlog(scale),
// ap += W dK_ij/dlog(period) (W carrying the pair's weight; the noise term is the caller's).  mll_grad_kernel's expressions
// with ri = 1 / ell and rper = 1 / period.
__device__ __forceinline__ void mllb_grad_pair(int kind, const double* xi, const double* xj, int d, const double* ri, double rper,
                                               double scale, double W, double (&accl)[MLL_MAX_D], double& as, double& ap) {
    if (kind == B2GP_KERNEL_PERIODIC) {
        double ssum = 0.0, dper = 0.0, q[MLL_MAX_D];
#pragma unroll
        for (int k = 0; k < MLL_MAX_D; ++k) {
            q[k] = 0.0;
            if (k < d) {
                double sn, cs;
                const double a = 3.141592653589793 * (xi[k] - xj[k]) * rper;
                sincos(a, &sn, &cs);
                const double rl2 = ri[k] * ri[k];
                q[k] = sn * sn * rl2;
                ssum += q[k];
                dper += 2.0 * sn * cs * a * rl2;
            }
        }
        const double wk = W * scale * exp(-2.0 * ssum);
#pragma unroll
        for (int k = 0; k < MLL_MAX_D; ++k)
            if (k < d) accl[k] += wk * 4.0 * q[k];
        as += wk;
        ap += wk * 2.0 * dper;
    } else {
        double r2 = 0.0, q[MLL_MAX_D];
#pragma unroll
        for (int k = 0; k < MLL_MAX_D; ++k) {
            q[k] = 0.0;
            if (k < d) {
                const double dl = (xi[k] - xj[k]) * ri[k];
                q[k] = dl * dl;
                r2 += q[k];
            }
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
#pragma unroll
        for (int k = 0; k < MLL_MAX_D; ++k)
            if (k < d) accl[k] += W * dK * q[k];
        as += W * Kij;
    }
}

__global__ void __launch_bounds__(PD_THREADS, 1)
mll_batch_small_kernel(int kind, const double* __restrict__ X, int n, const double* __restrict__ y, int d,
                       const double* __restrict__ theta, double jitter, double* __restrict__ value, double* __restrict__ grad,
                       double* __restrict__ alpha_out, double* __restrict__ gx, int* __restrict__ info) {
    extern __shared__ __align__(16) double sm[];
    double* S = sm;
    double* Xs = sm + PD_SMEM / 8;
    double* ys = Xs + MLLB_MAX_N * MLL_MAX_D;
    double* ws = ys + MLLB_MAX_N;
    double* al = ws + MLLB_MAX_N;
    double* lg = al + MLLB_MAX_N;
    double* th = lg + MLLB_MAX_N;
    double* ri = th + MLL_MAX_D + 3;
    double* red = ri + MLL_MAX_D;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int64_t b = blockIdx.x;
    const int nout = d + 3;
    const bool periodic = kind == B2GP_KERNEL_PERIODIC;
    if (tid == 0) info[b] = 0;
    for (int e = tid; e < n * d; e += PD_THREADS) Xs[e] = X[b * n * d + e];
    for (int e = tid; e < n; e += PD_THREADS) ys[e] = y[b * n + e];
    if (tid < nout) th[tid] = theta[b * nout + tid];
    if (tid < d) ri[tid] = 1.0 / theta[b * nout + tid];
    __syncthreads();
    const double scale = th[d], noise = th[d + 1], rper = 1.0 / th[d + 2];

    // 1. K: gram_kernel's covariance functions (cov_from_r2 on the squared scaled distance; the periodic sum), rows >= n zero
    for (int e = tid; e < MLLB_MAX_N * MLLB_MAX_N; e += PD_THREADS) {
        const int i = e >> 7, j = e & 127;
        double v = 0.0;
        if (i < n && j <= i) {
            double s = 0.0;
            for (int k = 0; k < d; ++k) {
                const double t = periodic ? sin(3.141592653589793 * (Xs[i * d + k] - Xs[j * d + k]) * rper) * ri[k]
                                          : (Xs[i * d + k] - Xs[j * d + k]) * ri[k];
                s += t * t;
            }
            v = periodic ? scale * exp(-2.0 * s) : cov_from_r2(kind, s, scale);
            if (i == j) v += noise + jitter;
        }
        S[i * PD_LD + j] = v;
    }
    __syncthreads();

    // 2. S's lower triangle <- inv(L)
    potrf_diag_cta<false>(sm, nullptr, 0, n, nullptr, info + b, 0, nullptr);

    // 3. w = inv(L) y (row i), alpha = inv(L)^T w (column i), log L_ii = -log inv(L)_ii; sums in index order
    if (tid < n) {
        double s = 0.0;
#pragma unroll 4
        for (int k = 0; k <= tid; ++k) s = fma(S[tid * PD_LD + k], ys[k], s);
        ws[tid] = s;
        lg[tid] = -log(S[tid * PD_LD + tid]);
    }
    __syncthreads();
    if (tid < n) {
        double s = 0.0;
#pragma unroll 4
        for (int k = tid; k < n; ++k) s = fma(S[k * PD_LD + tid], ws[k], s);
        al[tid] = s;
    }
    // K^{-1}_cr = sum_{k >= r} inv(L)_kc inv(L)_kr for c <= r: reads the lower triangle, writes above it (a warp shares r, so
    // its trip counts are equal and inv(L)_kr is a broadcast)
    const int ntri = n * (n + 1) / 2;
    for (int e = tid; e < ntri; e += PD_THREADS) {
        int r, c;
        mllb_tri(e, r, c);
        double s = 0.0;
#pragma unroll 4
        for (int k = r; k < n; ++k) s = fma(S[k * PD_LD + c], S[k * PD_LD + r], s);
        S[c * PD_LD + (c == r ? MLLB_KD : r)] = s;
    }
    __syncthreads();
    if (tid == 0) {
        double w2 = 0.0, ld = 0.0;
        for (int i = 0; i < n; ++i) {
            w2 = fma(ws[i], ws[i], w2);
            ld += lg[i];
        }
        value[b] = -0.5 * w2 - ld - 0.5 * (double)n * 1.8378770664093453;   // log(2 pi)
    }
    if (alpha_out)
        for (int i = tid; i < n; i += PD_THREADS) alpha_out[b * n + i] = al[i];

    // 4. gradient w.r.t. log theta: mll_grad_kernel's sums over the lower triangle, off-diagonal pairs weighted 2
    if (grad) {
        double accl[MLL_MAX_D], as = 0.0, an = 0.0, ap = 0.0;
#pragma unroll
        for (int k = 0; k < MLL_MAX_D; ++k) accl[k] = 0.0;
        for (int e = tid; e < ntri; e += PD_THREADS) {
            int i, j;
            mllb_tri(e, i, j);
            const double W = (al[i] * al[j] - mllb_kinv(S, i, j)) * (i == j ? 1.0 : 2.0);
            mllb_grad_pair(kind, Xs + i * d, Xs + j * d, d, ri, rper, scale, W, accl, as, ap);
            if (i == j) an += W * noise;
        }
        // slots: lengthscales [0, d), then scale, noise, period
        double* rw = red + warp * (MLL_MAX_D + 3);
#pragma unroll
        for (int k = 0; k < MLL_MAX_D + 3; ++k) {
            if (k >= d && k < MLL_MAX_D) continue;
            double v = k < MLL_MAX_D ? accl[k] : k == MLL_MAX_D ? as : k == MLL_MAX_D + 1 ? an : ap;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
            if (lane == 0) rw[k < MLL_MAX_D ? k : d + (k - MLL_MAX_D)] = v;
        }
        __syncthreads();
        if (tid < nout) {
            double v = 0.0;
            for (int w = 0; w < PD_THREADS / 32; ++w) v += red[w * (MLL_MAX_D + 3) + tid];
            grad[b * nout + tid] = 0.5 * v;
        }
    }

    // 5. d value / dX: two threads per row (even / odd columns), combined by one xor step
    if (gx) {
        const int i = tid >> 1, h = tid & 1;
        double acc[MLL_MAX_D];
#pragma unroll
        for (int k = 0; k < MLL_MAX_D; ++k) acc[k] = 0.0;
        if (i < n) {
            for (int j = h; j < n; j += 2) {
                if (j == i) continue;
                const double w = al[i] * al[j] - mllb_kinv(S, i, j);
                if (periodic) {   // mll_dz_kernel's -2 pi sin(2 a_k) / (period l_k^2) k
                    double s = 0.0, t[MLL_MAX_D];
#pragma unroll
                    for (int k = 0; k < MLL_MAX_D; ++k) {
                        t[k] = 0.0;
                        if (k < d) {
                            double sa, ca;
                            sincos(3.141592653589793 * (Xs[i * d + k] - Xs[j * d + k]) * rper, &sa, &ca);
                            const double a = sa * ri[k];
                            s += a * a;
                            t[k] = -(4.0 * 3.141592653589793) * sa * ca * rper * ri[k] * ri[k];
                        }
                    }
                    const double wk = w * (scale * exp(-2.0 * s));
#pragma unroll
                    for (int k = 0; k < MLL_MAX_D; ++k)
                        if (k < d) acc[k] = fma(wk, t[k], acc[k]);
                } else {
                    double r2 = 0.0;
#pragma unroll
                    for (int k = 0; k < MLL_MAX_D; ++k)
                        if (k < d) {
                            const double dl = (Xs[i * d + k] - Xs[j * d + k]) * ri[k];
                            r2 = fma(dl, dl, r2);
                        }
                    const double wg = w * stationary_dk_dr2(kind, r2, scale);
#pragma unroll
                    for (int k = 0; k < MLL_MAX_D; ++k)
                        if (k < d) acc[k] = fma(wg, 2.0 * (Xs[i * d + k] - Xs[j * d + k]) * ri[k] * ri[k], acc[k]);
                }
            }
        }
#pragma unroll
        for (int k = 0; k < MLL_MAX_D; ++k) acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], 1);
        if (h == 0 && i < n)
#pragma unroll
            for (int k = 0; k < MLL_MAX_D; ++k)
                if (k < d) gx[(b * n + i) * d + k] = acc[k];
    }
}
