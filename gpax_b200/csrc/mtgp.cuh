// mtgp.cuh -- the linear model of coregionalisation (LCM) of MultiTaskGP / CoregGP: its Gram matrix and the gradient of
// the multi-task log marginal likelihood.
//
// gpax/kernels/mtkernels.py:197-233 sums, over latents q = 0..L-1, the multi-task kernel of latent q (every parameter but
// the noise carries the latent axis, :21):
//     K_q[i,j] = (k_q(x_i, x_j) + jitter [i, j same data point]) * B_q[t_i, t_j]  +  [i == j] (noise[t_i] + jitter)
// with B_q = W_q W_q^T + diag(v_q) (:60-63).  The multitask form (MultitaskKernel, :95-125) has one row per observation
// and its task id in the last input column; the Kronecker form (MultivariateKernel, :163-192) is the same thing on
// inputs repeated once per task, task index cycling fastest, so that a data point is `group` = T consecutive rows and the
// data kernel's jitter covers its whole T x T block.  The noise term is added once per latent: the diagonal carries
// L (noise[t] + jitter).
//
// gram_lcm_kernel builds the sum in one pass and writes each entry once (no N x N scratch per latent): a CTA stages
// theta_q and B_q for every latent in shared memory, then for q = 0..L-1 stages its rows and columns scaled by 1 / ell_q
// and accumulates latent q into the 8 x 2 entries each thread holds in registers.  The data kernel is gram.cuh's
// cov_from_r2 on r2 = (X^2 - 2 X Z) + Z^2 clipped at 0, or the periodic sum.  HBM-bound: 8 bytes written per entry.
//
// mll_lcm_grad_kernel is mll_grad_kernel (mll.cuh) for this covariance: blockIdx.z = latent, the same 64 x 64 tiles of
// the lower triangle and the same thread -> entry map (a thread's column j, and so t_j, is fixed), k_q recomputed on the
// fly, a fixed-order two-pass reduction (no atomics: deterministic).
//
// gram_dx_lcm_kernel writes the derivative rows of k_pX w.r.t. the test inputs (b2gp_posterior_multitask_grad), which
// the posterior solves under [k_pX; y^T] as it solves grad.cuh's rows for the single-task kernel.
//
// Limits: T <= MT_MAX_T tasks, L <= MT_MAX_L latents, d <= MLL_MAX_D input features (checked by the host entries).
#pragma once
#include "common.cuh"
#include "gram.cuh"
#include "grad.cuh"
#include "mll.cuh"

constexpr int MT_MAX_T = 8;
constexpr int MT_MAX_L = 4;

// 32 rows x 128 columns per 256-thread CTA, each thread 8 rows x 2 adjacent columns (16 accumulators), 16-byte stores
constexpr int LCM_BM = 32;

enum { LCM_RECT = 0, LCM_LOWER = 1, LCM_DIAG = 2 };

struct LcmArgs {
    const double* X;       // [n, d]
    const int* tX;         // [n] task ids in [0, T)
    const double* Z;       // [m, d]
    const int* tZ;         // [m]
    int64_t n, m;
    int d, kind, T, L, group;
    const double* theta;   // [L, d+2]: lengthscale[d], k_scale, period
    const double* B;       // [L, T, T]
    const double* noise;   // [T]
    double noise_mult;     // LOWER / DIAG: the diagonal term is noise * noise_mult + jitter, once per latent
    double jitter;
    int mode;              // LCM_RECT: K[n,m], no diagonal terms (k_pX, gp.py:268); LCM_LOWER: X == Z, lower triangle with
                           // the diagonal terms (k_XX, k_pp); LCM_DIAG: K[i] = the diagonal of LCM_LOWER, length n
    double* K;
    int64_t ldk;
};

__global__ void __launch_bounds__(GRAM_THREADS, 2) gram_lcm_kernel(const LcmArgs p) {
    extern __shared__ __align__(16) double sm[];
    const int d = p.d, T = p.T, L = p.L, nth = d + 2;
    const int tid = threadIdx.x;
    const bool periodic = (p.kind == B2GP_KERNEL_PERIODIC);
    if (p.mode == LCM_DIAG) {
        // k_q(x, x) is cov_self: the value the tiled path computes for r2 = 0 (or sin 0 = 0)
        for (int64_t i = (int64_t)blockIdx.x * blockDim.x + tid; i < p.n; i += (int64_t)gridDim.x * blockDim.x) {
            const int t = p.tX[i];
            const double dg = p.noise[t] * p.noise_mult + p.jitter;
            double acc = 0.0;
            for (int q = 0; q < L; ++q)
                acc += (cov_self(p.kind, p.theta[q * nth + d]) + p.jitter) * p.B[(q * T + t) * T + t] + dg;
            p.K[i * p.ldk] = acc;
        }
        return;
    }
    const int64_t row0 = (int64_t)blockIdx.y * LCM_BM;
    const int64_t col0 = (int64_t)blockIdx.x * GRAM_BN;
    const bool lower = (p.mode == LCM_LOWER);
    if (lower && col0 > row0 + LCM_BM - 1) return;
    // layout: Xs[LCM_BM][d] | x2[LCM_BM] | Zt[d][GRAM_BN] | z2[GRAM_BN] | th[L][d+2] | Bs[L][T][T] | tXs[LCM_BM] | tZs[GRAM_BN]
    double* Xs = sm;
    double* x2 = Xs + LCM_BM * d;
    double* Zt = x2 + LCM_BM;
    double* z2 = Zt + d * GRAM_BN;
    double* th = z2 + GRAM_BN;
    double* Bs = th + L * nth;
    int* tXs = reinterpret_cast<int*>(Bs + L * T * T);
    int* tZs = tXs + LCM_BM;
    for (int i = tid; i < L * nth; i += GRAM_THREADS) th[i] = p.theta[i];
    for (int i = tid; i < L * T * T; i += GRAM_THREADS) Bs[i] = p.B[i];
    if (tid < LCM_BM) tXs[tid] = (row0 + tid < p.n) ? p.tX[row0 + tid] : 0;
    else if (tid < LCM_BM + GRAM_BN) tZs[tid - LCM_BM] = (col0 + tid - LCM_BM < p.m) ? p.tZ[col0 + tid - LCM_BM] : 0;

    const int cl = (tid & 63) * 2;
    const int rg = tid >> 6;
    const int64_t gc = col0 + cl;
    const bool col_ok = gc < p.m;
    double acc0[LCM_BM / 4], acc1[LCM_BM / 4];
#pragma unroll
    for (int i = 0; i < LCM_BM / 4; ++i) acc0[i] = acc1[i] = 0.0;
    // LOWER: bit i of sp0 / sp1 = row i of this thread and column gc / gc + 1 are one data point (`group` consecutive rows)
    unsigned sp0 = 0, sp1 = 0;
    if (lower && col_ok) {
        const int64_t pc0 = gc / p.group, pc1 = (gc + 1) / p.group;
#pragma unroll
        for (int i = 0; i < LCM_BM / 4; ++i) {
            const int64_t pr = (row0 + rg + 4 * i) / p.group;
            sp0 |= (unsigned)(pr == pc0) << i;
            sp1 |= (unsigned)(pr == pc1) << i;
        }
    }

    for (int q = 0; q < L; ++q) {
        __syncthreads();   // th / Bs / task ids staged; the previous latent's reads of Xs / Zt are done
        const double* ell = th + q * nth;
        const double scale = ell[d], period = ell[d + 1];
        // rows scaled by 1 / lengthscale (a division, kernels.py:35-36) for RBF / Matern, raw for periodic
        for (int idx = tid; idx < LCM_BM * d; idx += GRAM_THREADS) {
            const int r = idx / d, k = idx % d;
            const int64_t gr = row0 + r;
            const double v = (gr < p.n) ? p.X[gr * d + k] : 0.0;
            Xs[r * d + k] = periodic ? v : v / ell[k];
        }
        for (int idx = tid; idx < GRAM_BN * d; idx += GRAM_THREADS) {
            const int c = idx / d, k = idx % d;
            const int64_t g = col0 + c;
            const double v = (g < p.m) ? p.Z[g * d + k] : 0.0;
            Zt[k * GRAM_BN + c] = periodic ? v : v / ell[k];
        }
        __syncthreads();
        if (!periodic) {
            if (tid < LCM_BM) {
                double s = 0.0;
                for (int k = 0; k < d; ++k) s = fma(Xs[tid * d + k], Xs[tid * d + k], s);
                x2[tid] = s;
            } else if (tid < LCM_BM + GRAM_BN) {
                const int c = tid - LCM_BM;
                double s = 0.0;
                for (int k = 0; k < d; ++k) s = fma(Zt[k * GRAM_BN + c], Zt[k * GRAM_BN + c], s);
                z2[c] = s;
            }
        }
        __syncthreads();
        if (!col_ok) continue;
        const double* Bq = Bs + q * T * T;
        const int tc0 = tZs[cl], tc1 = tZs[cl + 1];
#pragma unroll
        for (int i = 0; i < LCM_BM / 4; ++i) {
            const int rl = rg + 4 * i;
            const int64_t gr = row0 + rl;
            if (gr >= p.n) continue;
            double v0, v1;
            if (!periodic) {
                double xz0 = 0.0, xz1 = 0.0;
                for (int k = 0; k < d; ++k) {
                    const double x = Xs[rl * d + k];
                    xz0 = fma(x, Zt[k * GRAM_BN + cl], xz0);
                    xz1 = fma(x, Zt[k * GRAM_BN + cl + 1], xz1);
                }
                double r20 = (x2[rl] - 2.0 * xz0) + z2[cl];       // kernels.py:40
                double r21 = (x2[rl] - 2.0 * xz1) + z2[cl + 1];
                r20 = r20 < 0.0 ? 0.0 : r20;                      // kernels.py:41
                r21 = r21 < 0.0 ? 0.0 : r21;
                v0 = cov_from_r2(p.kind, r20, scale);
                v1 = cov_from_r2(p.kind, r21, scale);
            } else {
                double s0 = 0.0, s1 = 0.0;
                for (int k = 0; k < d; ++k) {
                    const double x = Xs[rl * d + k];
                    const double a0 = periodic_arg(x, Zt[k * GRAM_BN + cl], period, ell[k]);
                    const double a1 = periodic_arg(x, Zt[k * GRAM_BN + cl + 1], period, ell[k]);
                    s0 += a0 * a0;
                    s1 += a1 * a1;
                }
                v0 = scale * exp(-2.0 * s0);
                v1 = scale * exp(-2.0 * s1);
            }
            const int tr = tXs[rl];
            // the data kernel's own diagonal rule (mtkernels.py:103, 167): jitter where the points coincide
            if ((sp0 >> i) & 1u) v0 += p.jitter;
            if ((sp1 >> i) & 1u) v1 += p.jitter;
            v0 *= Bq[tr * T + tc0];
            v1 *= Bq[tr * T + tc1];
            if (lower) {   // noise[t] + jitter on i == j, once per latent (mtkernels.py:117-121, 183-188)
                const double dg = p.noise[tr] * p.noise_mult + p.jitter;
                if (gr == gc) v0 += dg;
                if (gr == gc + 1) v1 += dg;
            }
            acc0[i] += v0;
            acc1[i] += v1;
        }
    }
    if (!col_ok) return;
    const bool has2 = (gc + 1 < p.m);
    const bool vec_ok = ((p.ldk & 1) == 0) && ((reinterpret_cast<uintptr_t>(p.K) & 15) == 0);
#pragma unroll
    for (int i = 0; i < LCM_BM / 4; ++i) {
        const int64_t gr = row0 + rg + 4 * i;
        if (gr >= p.n) continue;
        const bool w0 = !(lower && gc > gr);
        const bool w1 = has2 && !(lower && gc + 1 > gr);
        double* dst = p.K + gr * p.ldk + gc;
        if (w0 && w1 && vec_ok) {
            *reinterpret_cast<double2*>(dst) = make_double2(acc0[i], acc1[i]);
        } else {
            if (w0) dst[0] = acc0[i];
            if (w1) dst[1] = acc1[i];
        }
    }
}

static inline size_t gram_lcm_smem(int d, int T, int L) {
    return (size_t)(LCM_BM * d + LCM_BM + d * GRAM_BN + GRAM_BN + L * (d + 2) + L * T * T) * sizeof(double) +
           (size_t)(LCM_BM + GRAM_BN) * sizeof(int);
}

// One LCM Gram build (every pointer a device pointer).  LCM_DIAG writes K[i * ldk], i < n.
static int launch_gram_lcm(b2gp_ctx* ctx, cudaStream_t st, int mode, int kind, const double* X, const int* tX, int64_t n,
                           const double* Z, const int* tZ, int64_t m, int d, int T, int L, int group, const double* theta,
                           const double* B, const double* noise, double noise_mult, double jitter, double* K, int64_t ldk) {
    if (n <= 0 || (mode != LCM_DIAG && m <= 0)) return B2GP_OK;
    LcmArgs a;
    a.X = X;
    a.tX = tX;
    a.Z = Z;
    a.tZ = tZ;
    a.n = n;
    a.m = m;
    a.d = d;
    a.kind = kind;
    a.T = T;
    a.L = L;
    a.group = group;
    a.theta = theta;
    a.B = B;
    a.noise = noise;
    a.noise_mult = noise_mult;
    a.jitter = jitter;
    a.mode = mode;
    a.K = K;
    a.ldk = ldk;
    if (mode == LCM_DIAG) return launch(ctx, st, (unsigned)ceil_div(n, (int64_t)GRAM_THREADS), GRAM_THREADS, 0, gram_lcm_kernel, a);
    dim3 grid((unsigned)ceil_div(m, GRAM_BN), (unsigned)ceil_div(n, (int64_t)LCM_BM));
    return launch(ctx, st, grid, GRAM_THREADS, gram_lcm_smem(d, T, L), gram_lcm_kernel, a);
}

// Derivative rows of the LCM cross-covariance k_pX w.r.t. the test inputs (the multi-task counterpart of grad.cuh's
// gram_dx_kernel, solved and reduced by the posterior exactly as those rows are):
//     D[p*d + k, i] = sum_{q=0..L-1} B_q[t_p, t_i] * d k_q(x_p, x_i) / d x_p[k]
// for every GP row p of the test block (the Kronecker form's repeated rows each w.r.t. their own point: same code).  k_pX
// carries no jitter or noise term, so nothing else depends on x_p.  d k_q / d x_p is gram_dx_kernel's formula with
// latent q's lengthscales, scale and period: stationary_dk_dr2 on r2 = (x2 - 2 xz) + z2 of the inputs divided by ell_q
// (clipped as the Gram clips), or the periodic form with one sincos per dimension.  Each thread owns one column i and
// GDX_BP / 4 rows; an element's latents are summed in registers in the order q = 0..L-1 and stored once: identical calls
// give identical bits.  HBM-bound: 8 P d N bytes written.
constexpr int GDXL_BN = 64;     // training points (columns) per CTA
constexpr int GDXL_THREADS = 256;

static inline size_t gram_dx_lcm_smem(int d, int T, int L) {
    return (size_t)(L * d * GDXL_BN + L * GDX_BP * d + L * GDXL_BN + L * GDX_BP + L * (d + 2) + L * T * T) * sizeof(double) +
           (size_t)(GDX_BP + GDXL_BN) * sizeof(int);
}

// grid (ceil(N / GDXL_BN), ceil(P / GDX_BP)); dynamic shared memory gram_dx_lcm_smem(d, T, L) (under 48 KB for d <= 16,
// L <= 4, T <= 8): per latent the scaled columns and rows and their squared norms, theta_q, B_q, the task ids
__global__ void __launch_bounds__(GDXL_THREADS)
gram_dx_lcm_kernel(int kind, const double* __restrict__ Xnew, const int* __restrict__ tNew, int64_t P, const double* __restrict__ Xtr,
                   const int* __restrict__ tTr, int64_t N, int d, int T, int L, const double* __restrict__ theta,
                   const double* __restrict__ B, double* __restrict__ D, int64_t ldd) {
    extern __shared__ __align__(16) double sm[];
    // layout: Zs[L][d][GDXL_BN] | Xs[L][GDX_BP][d] | z2[L][GDXL_BN] | x2[L][GDX_BP] | th[L][d+2] | Bs[L][T][T] | tXs | tZs
    double* Zs = sm;
    double* Xs = Zs + L * d * GDXL_BN;
    double* z2 = Xs + L * GDX_BP * d;
    double* x2 = z2 + L * GDXL_BN;
    double* th = x2 + L * GDX_BP;
    double* Bs = th + L * (d + 2);
    int* tXs = reinterpret_cast<int*>(Bs + L * T * T);
    int* tZs = tXs + GDX_BP;
    const int tid = threadIdx.x, nth = d + 2;
    const int64_t col0 = (int64_t)blockIdx.x * GDXL_BN, p0 = (int64_t)blockIdx.y * GDX_BP;
    const bool periodic = (kind == B2GP_KERNEL_PERIODIC);
    for (int i = tid; i < L * nth; i += GDXL_THREADS) th[i] = theta[i];
    for (int i = tid; i < L * T * T; i += GDXL_THREADS) Bs[i] = B[i];
    if (tid < GDX_BP) tXs[tid] = (p0 + tid < P) ? tNew[p0 + tid] : 0;
    else if (tid < GDX_BP + GDXL_BN) tZs[tid - GDX_BP] = (col0 + tid - GDX_BP < N) ? tTr[col0 + tid - GDX_BP] : 0;
    __syncthreads();
    // staged as gram_lcm_kernel stages them: divided by latent q's lengthscale for RBF / Matern, raw for periodic
    for (int idx = tid; idx < L * GDXL_BN * d; idx += GDXL_THREADS) {
        const int q = idx / (GDXL_BN * d), k = idx / GDXL_BN % d, c = idx % GDXL_BN;
        const int64_t gc = col0 + c;
        const double v = gc < N ? Xtr[gc * d + k] : 0.0;
        Zs[idx] = periodic ? v : v / th[q * nth + k];
    }
    for (int idx = tid; idx < L * GDX_BP * d; idx += GDXL_THREADS) {
        const int q = idx / (GDX_BP * d), r = idx / d % GDX_BP, k = idx % d;
        const int64_t gp = p0 + r;
        const double v = gp < P ? Xnew[gp * d + k] : 0.0;
        Xs[idx] = periodic ? v : v / th[q * nth + k];
    }
    __syncthreads();
    if (!periodic) {
        for (int idx = tid; idx < L * (GDXL_BN + GDX_BP); idx += GDXL_THREADS) {
            const bool col = idx < L * GDXL_BN;
            const int j = col ? idx : idx - L * GDXL_BN;
            const int q = col ? j / GDXL_BN : j / GDX_BP, e = col ? j % GDXL_BN : j % GDX_BP;
            double s = 0.0;
            for (int k = 0; k < d; ++k) {
                const double v = col ? Zs[(q * d + k) * GDXL_BN + e] : Xs[(q * GDX_BP + e) * d + k];
                s = fma(v, v, s);
            }
            (col ? z2 : x2)[j] = s;
        }
        __syncthreads();
    }
    const int c = tid % GDXL_BN;
    const int64_t gc = col0 + c;
    if (gc >= N) return;
    const int tc = tZs[c];
    for (int r = tid / GDXL_BN; r < GDX_BP; r += GDXL_THREADS / GDXL_BN) {
        const int64_t gp = p0 + r;
        if (gp >= P) break;
        const int tr = tXs[r];
        double acc[MLL_MAX_D];
#pragma unroll
        for (int k = 0; k < MLL_MAX_D; ++k) acc[k] = 0.0;
        for (int q = 0; q < L; ++q) {
            const double* ell = th + q * nth;
            const double scale = ell[d], period = ell[d + 1];
            const double b = Bs[(q * T + tr) * T + tc];
            const double* x = Xs + (q * GDX_BP + r) * d;
            const double* z = Zs + q * d * GDXL_BN + c;      // z[k * GDXL_BN]
            if (periodic) {
                // -2 pi sin(2 a_k) / (period l_k^2) = -4 pi sin a_k cos a_k / ..., times k_q once the exponent is known
                double g[MLL_MAX_D], s = 0.0;
#pragma unroll
                for (int k = 0; k < MLL_MAX_D; ++k) {
                    if (k < d) {
                        double sa, ca;
                        sincos(3.141592653589793 * (x[k] - z[k * GDXL_BN]) / period, &sa, &ca);
                        const double a = sa / ell[k];                               // kernels.py:111-113
                        s += a * a;
                        g[k] = -(4.0 * 3.141592653589793) * sa * ca / (period * ell[k] * ell[k]);
                    }
                }
                const double bk = b * (scale * exp(-2.0 * s));
#pragma unroll
                for (int k = 0; k < MLL_MAX_D; ++k)
                    if (k < d) acc[k] += bk * g[k];
                continue;
            }
            double xz = 0.0;
            for (int k = 0; k < d; ++k) xz = fma(x[k], z[k * GDXL_BN], xz);
            const double r2raw = (x2[q * GDX_BP + r] - 2.0 * xz) + z2[q * GDXL_BN + c];   // kernels.py:40
            const double bg = b * stationary_dk_dr2(kind, r2raw, scale);
#pragma unroll
            for (int k = 0; k < MLL_MAX_D; ++k)
                if (k < d) acc[k] += bg * (2.0 * (x[k] - z[k * GDXL_BN]) / ell[k]);
        }
        double* out = D + gp * d * ldd + gc;
#pragma unroll
        for (int k = 0; k < MLL_MAX_D; ++k)
            if (k < d) out[k * ldd] = acc[k];
    }
}

// D[P*d, N] (leading dimension ldd) of the LCM cross-covariance for test rows Xnew[P, d] / tNew[P] against Xtr[N, d] /
// tTr[N], one draw's theta[L, d+2] and B[L, T, T] (device pointers; task ids validated by the caller)
static int launch_gram_dx_lcm(b2gp_ctx* ctx, cudaStream_t st, int kind, const double* Xnew, const int* tNew, int64_t P,
                              const double* Xtr, const int* tTr, int64_t N, int d, int T, int L, const double* theta,
                              const double* B, double* D, int64_t ldd) {
    if (P <= 0 || N <= 0) return B2GP_OK;
    if (kind < 0 || kind > B2GP_KERNEL_PERIODIC || d < 1 || d > MLL_MAX_D || T < 1 || T > MT_MAX_T || L < 1 || L > MT_MAX_L)
        return set_err(ctx, B2GP_ERR_UNSUPPORTED, "gram_dx_lcm", "RBF / Matern / Periodic, d <= 16, T <= 8, L <= 4", __FILE__, __LINE__);
    dim3 grid((unsigned)ceil_div(N, (int64_t)GDXL_BN), (unsigned)ceil_div(P, (int64_t)GDX_BP));
    return launch(ctx, st, grid, GDXL_THREADS, gram_dx_lcm_smem(d, T, L), gram_dx_lcm_kernel, kind, Xnew, tNew, P, Xtr, tTr, N, d, T,
                  L, theta, B, D, ldd);
}

// var[i] += prior[i]: the posterior variance from rowdot_kernel's -|V^T[i,:]|^2 (run with a zero prior) and the LCM
// prior diagonal; a NaN (failed factorisation) stays NaN
__global__ void add_vec_kernel(double* __restrict__ var, const double* __restrict__ prior, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) var[i] = prior[i] + var[i];
}

// Gradient of the multi-task log marginal likelihood.  With W_ij = alpha_i alpha_j - Kinv_ij, latent q = blockIdx.z sums
// over the lower triangle (off-diagonal entries weighted 2):
//   [k < d]  W B_q[t_i,t_j] dk_q/dlog ell_q[k]      [d] W B_q[t_i,t_j] k_q      [d+1] W B_q[t_i,t_j] dk_q/dlog period_q
//   [d+2 + a*T + b]  W (k_q + jitter [same point])  over the entries with t_i = a, t_j = b
//   [d+2 + T*T + t]  W L noise[t] on i == j with t_i = t   (latent 0 only; zero in the other latents' blocks)
// into partial[(q * nblocks + block) * nout + k], nout = d + 2 + T*T + T.
__global__ void __launch_bounds__(MLL_THREADS)
mll_lcm_grad_kernel(const double* __restrict__ X, const int* __restrict__ task, int64_t N, int d, int kind, int T, int L, int group,
                    const double* __restrict__ theta, const double* __restrict__ B, const double* __restrict__ noise, double jitter,
                    const double* __restrict__ alpha, const double* __restrict__ Kinv, int64_t ldk, double* __restrict__ partial) {
    __shared__ double red[MLL_THREADS / 32][MLL_MAX_D + 2];
    __shared__ double redB[MLL_THREADS][MT_MAX_T];
    __shared__ double redN[MLL_THREADS];
    __shared__ int tcol[MLL_THREADS];
    const int64_t ti = blockIdx.y, tj = blockIdx.x;
    const int q = blockIdx.z;
    const int nth = d + 2, nout = d + 2 + T * T + T;
    const int64_t nblocks = (int64_t)gridDim.x * gridDim.y;
    const int64_t blk = (int64_t)blockIdx.y * gridDim.x + blockIdx.x;
    double acc[MLL_MAX_D], accS = 0.0, accP = 0.0, accB[MT_MAX_T], accN = 0.0;   // ell | k_scale | period | B | noise
#pragma unroll
    for (int k = 0; k < MLL_MAX_D; ++k) acc[k] = 0.0;
#pragma unroll
    for (int t = 0; t < MT_MAX_T; ++t) accB[t] = 0.0;
    const int64_t r0 = ti * MLL_TILE, c0 = tj * MLL_TILE;
    const int64_t j = c0 + threadIdx.x % MLL_TILE;     // fixed per thread
    const int tjk = (j < N) ? task[j] : -1;
    const int64_t jp = j / group;
    if (tj <= ti && j < N) {
        const double* th = theta + q * nth;
        const double scale = th[d], period = th[d + 1];
        const double* Bq = B + (int64_t)q * T * T;
        for (int e = threadIdx.x; e < MLL_TILE * MLL_TILE; e += MLL_THREADS) {
            const int64_t i = r0 + e / MLL_TILE;
            if (i >= N || j > i) continue;
            const int tik = task[i];
            const double W = (alpha[i] * alpha[j] - Kinv[i * ldk + j]) * ((i == j) ? 1.0 : 2.0);
            const double b = Bq[tik * T + tjk];
            double Kq, qk[MLL_MAX_D];
            if (kind == B2GP_KERNEL_PERIODIC) {
                double ssum = 0.0, dper = 0.0;
#pragma unroll
                for (int k = 0; k < MLL_MAX_D; ++k) {
                    if (k < d) {
                        const double a = 3.141592653589793 * (X[i * d + k] - X[j * d + k]) / period;
                        const double sn = sin(a), l2 = th[k] * th[k];
                        qk[k] = sn * sn / l2;
                        ssum += qk[k];
                        dper += 2.0 * sn * cos(a) * a / l2;
                    }
                }
                Kq = scale * exp(-2.0 * ssum);
#pragma unroll
                for (int k = 0; k < MLL_MAX_D; ++k)
                    if (k < d) acc[k] += W * b * Kq * 4.0 * qk[k];
                accP += W * b * Kq * 2.0 * dper;
            } else {
                double r2 = 0.0;
#pragma unroll
                for (int k = 0; k < MLL_MAX_D; ++k) {
                    if (k < d) {
                        const double dl = (X[i * d + k] - X[j * d + k]) / th[k];
                        qk[k] = dl * dl;
                        r2 += qk[k];
                    }
                }
                double dK;   // -2 dk/d(r2): dk/dlog(ell_k) = dK * q_k
                Kq = cov_from_r2(kind, r2, scale);
                if (kind == B2GP_KERNEL_RBF) {
                    dK = Kq;
                } else {
                    const double r = sqrt(r2 + 1e-12), s5r = 2.23606797749979 * r;
                    dK = (5.0 / 3.0) * scale * (1.0 + s5r) * exp(-s5r);
                }
#pragma unroll
                for (int k = 0; k < MLL_MAX_D; ++k)
                    if (k < d) acc[k] += W * b * dK * qk[k];
            }
            accS += W * b * Kq;
            const double kb = Kq + ((i / group == jp) ? jitter : 0.0);
#pragma unroll
            for (int t = 0; t < MT_MAX_T; ++t)
                if (t == tik) accB[t] += W * kb;
            if (q == 0 && i == j) accN += W * (double)L * noise[tik];
        }
    }
    // theta block: warp shuffles, then the 8 warps in order
#pragma unroll
    for (int k = 0; k < MLL_MAX_D + 2; ++k) {
        if (k < nth) {
            double v = (k < d) ? acc[k < MLL_MAX_D ? k : 0] : (k == d ? accS : accP);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
            if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5][k] = v;
        }
    }
#pragma unroll
    for (int t = 0; t < MT_MAX_T; ++t) redB[threadIdx.x][t] = accB[t];
    redN[threadIdx.x] = accN;
    tcol[threadIdx.x] = tjk;
    __syncthreads();
    double* out = partial + ((int64_t)q * nblocks + blk) * nout;
    const int o = threadIdx.x, lane = threadIdx.x & 31;
    if (o < nth) {
        double v = 0.0;
        for (int w = 0; w < MLL_THREADS / 32; ++w) v += red[w][o];
        out[o] = v;
    }
    // B entries (a, b) and noise entries t: one warp per output; lane l sums threads l, l + 32, ... whose column task is b
    // (or t), then a shuffle tree -- a fixed order
    for (int r = threadIdx.x >> 5; r < T * T + T; r += MLL_THREADS / 32) {
        const bool isB = r < T * T;
        const int a = isB ? r / T : 0, bb = isB ? r % T : r - T * T;
        double v = 0.0;
        for (int s = lane; s < MLL_THREADS; s += 32)
            if (tcol[s] == bb) v += isB ? redB[s][a] : redN[s];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
        if (lane == 0) out[nth + r] = v;
    }
}

// colsum[q * nout + k] = 1/2 sum over the blocks of latent q of partial[.][k]: one CTA per (q, k), thread t adding blocks
// t, t + 256, ... in order, then a fixed tree -- deterministic.  The host assembles the gradient from these sums (dvalue/dB_q
// with independent entries is the mean of the (a, b) and (b, a) sums; the noise sums sit in latent 0).  The draw of a
// batch is blockIdx.z (partial and colsum `bstride` doubles apart).
constexpr int MLL_FIN_THREADS = 256;
__global__ void __launch_bounds__(MLL_FIN_THREADS)
mll_lcm_finish_kernel(const double* __restrict__ partial, int64_t nblocks, int nout, double* __restrict__ colsum, int64_t bstride) {
    __shared__ double red[MLL_FIN_THREADS];
    partial += (int64_t)blockIdx.z * bstride;
    colsum += (int64_t)blockIdx.z * bstride;
    const int q = blockIdx.x / nout, k = blockIdx.x % nout;
    double s = 0.0;
    for (int64_t b = threadIdx.x; b < nblocks; b += MLL_FIN_THREADS) s += partial[((int64_t)q * nblocks + b) * nout + k];
    red[threadIdx.x] = s;
    __syncthreads();
    for (int o = MLL_FIN_THREADS / 2; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) colsum[blockIdx.x] = 0.5 * red[0];
}
