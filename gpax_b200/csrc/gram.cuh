// gram.cuh -- fused pairwise-distance + covariance-function Gram build.
//
// Replaces square_scaled_distance + RBFKernel / MaternKernel / PeriodicKernel
// (gpax/kernels/kernels.py:28-41, 44-65, 68-91, 94-117): one kernel reads X[n,d], Z[m,d] and the
// hyper-parameters of one draw and writes K[n,m]; no [n,m] intermediate (XZ, r2, the [n,m,d]
// difference tensor of the periodic kernel) ever reaches HBM.
//
// The arithmetic follows the reference operation for operation so that rounding is of the same
// structure: scaled = X / lengthscale (a division), X2 = sum scaled^2, r2 = (X2 - 2*XZ) + Z2 clipped
// at 0, Matern r = sqrt(r2 + 1e-12), periodic arg = (pi * (x - z)) / period.  X2 and XZ use the
// same fma chain, so r2 of a point with itself is exactly 0.
//
// Roofline: HBM writes.  Algorithmic bytes = 8*n*m written + 8*(n+m)*d read (SURVEY.md 8d); with
// B2GP_FLAG_LOWER_ONLY only tiles touching j <= i are produced (the factorisation reads nothing else).
// Tile: 64 rows x 128 columns per 256-thread CTA, each thread 16 rows x 2 adjacent columns, 16-byte
// stores (a warp writes 512 contiguous bytes per row).
#pragma once
#include "common.cuh"

constexpr int GRAM_BM = 64;
constexpr int GRAM_BN = 128;
constexpr int GRAM_THREADS = 256;
constexpr int GRAM_MAX_D = 64;

// theta layout of one draw (device memory): lengthscale[0..d), k_scale, noise, period
struct GramArgs {
    const double* X;
    const double* Z;
    int64_t n, m;
    int d;
    int kind;
    const double* theta;  // device pointer
    double noise_mult;    // diagonal term = noise * noise_mult + jitter, added iff same_xz
    double jitter;
    int same_xz;
    int lower_only;
    double* K;
    int64_t ldk;
    int64_t bstride = 0;  // doubles between the draws' theta and K (Batch, draw = blockIdx.z); X and Z are shared
};

__device__ __forceinline__ double cov_from_r2(int kind, double r2, double scale) {
    // kernels.py:61-62 (RBF) and kernels.py:85-88 (Matern-5/2 with the 1e-12 epsilon of :20-21)
    if (kind == B2GP_KERNEL_RBF) return scale * exp(-0.5 * r2);
    const double r = sqrt(r2 + 1e-12);
    const double s5r = 2.23606797749979 * r;  // 5**0.5 rounded to nearest double, as Python computes it
    return scale * (1.0 + s5r + (5.0 / 3.0) * r2) * exp(-s5r);
}

// NNGP kernels (gpax/kernels/kernels.py:120-183): the infinite-width-network recursion on the three inner products of a
// pair, `depth` times; erf activation (kernels.py:145-151) or ReLU (kernels.py:176-183).
__device__ __forceinline__ double nngp_step(bool relu, double a, double b, double c, double var_b, double var_w) {
    if (!relu) {
        double fr = 2.0 * a / sqrt((1.0 + 2.0 * b) * (1.0 + 2.0 * c));
        fr = fmin(fmax(fr, -1.0 + 1e-7), 1.0 - 1e-7);
        return var_b + 2.0 * var_w / 3.141592653589793 * asin(fr);
    }
    const double s = sqrt(b * c);
    const double fr = a / s;
    const double th = acos(fmin(fmax(fr, -1.0 + 1e-7), 1.0 - 1e-7));
    return var_b + var_w / (2.0 * 3.141592653589793) * s * (sin(th) + (3.141592653589793 - th) * fr);
}
__device__ __forceinline__ double nngp_pair(bool relu, double xz, double xx, double zz, int d, double var_b, double var_w, int depth) {
    double k12 = var_b + var_w * xz / d, k11 = var_b + var_w * xx / d, k22 = var_b + var_w * zz / d;   // depth 0, kernels.py:139-140
    for (int l = 0; l < depth; ++l) {
        const double n12 = nngp_step(relu, k12, k11, k22, var_b, var_w);
        const double n11 = nngp_step(relu, k11, k11, k11, var_b, var_w);
        const double n22 = nngp_step(relu, k22, k22, k22, var_b, var_w);
        k12 = n12;
        k11 = n11;
        k22 = n22;
    }
    return k12;
}

// sin(pi (x - z) / period) / ell: one feature of the periodic kernel's sum (kernels.py:111-113), the expression gram_kernel
// writes inline (routing gram_kernel through this helper changes its register allocation and SASS, which stay as they are)
__device__ __forceinline__ double periodic_arg(double x, double z, double period, double ell) {
    return sin(3.141592653589793 * (x - z) / period) / ell;
}

__global__ void __launch_bounds__(GRAM_THREADS) gram_kernel(const GramArgs p) {
    extern __shared__ __align__(16) double sm[];
    // layout: Xs[GRAM_BM][d] | x2[GRAM_BM] | Zt[d][GRAM_BN] | z2[GRAM_BN] | ell[d]
    const int d = p.d;
    double* Xs = sm;
    double* x2 = Xs + GRAM_BM * d;
    double* Zt = x2 + GRAM_BM;
    double* z2 = Zt + d * GRAM_BN;
    double* ell = z2 + GRAM_BN;

    const int64_t row0 = (int64_t)blockIdx.y * GRAM_BM;
    const int64_t col0 = (int64_t)blockIdx.x * GRAM_BN;
    if (p.lower_only && col0 > row0 + GRAM_BM - 1) return;
    const double* __restrict__ theta = p.theta + (int64_t)blockIdx.z * p.bstride;
    const int tid = threadIdx.x;
    const bool nngp = (p.kind == B2GP_KERNEL_NNGP_ERF || p.kind == B2GP_KERNEL_NNGP_RELU);
    const bool periodic = (p.kind == B2GP_KERNEL_PERIODIC);

    if (tid < d) ell[tid] = theta[tid];
    __syncthreads();
    const double scale = theta[d];
    const double noise = theta[d + 1];
    const double period = theta[d + 2];

    // stage the rows: scaled by 1/lengthscale (division, kernels.py:35-36) for RBF/Matern, raw for periodic
    for (int idx = tid; idx < GRAM_BM * d; idx += GRAM_THREADS) {
        const int r = idx / d, k = idx % d;
        const int64_t gr = row0 + r;
        double v = (gr < p.n) ? p.X[gr * d + k] : 0.0;
        Xs[r * d + k] = (periodic || nngp) ? v : v / ell[k];
    }
    for (int idx = tid; idx < GRAM_BN * d; idx += GRAM_THREADS) {
        const int c = idx / d, k = idx % d;
        const int64_t gc = col0 + c;
        double v = (gc < p.m) ? p.Z[gc * d + k] : 0.0;
        Zt[k * GRAM_BN + c] = (periodic || nngp) ? v : v / ell[k];
    }
    __syncthreads();
    if (!periodic) {
        if (tid < GRAM_BM) {
            double s = 0.0;
            for (int k = 0; k < d; ++k) s = fma(Xs[tid * d + k], Xs[tid * d + k], s);
            x2[tid] = s;
        } else if (tid < GRAM_BM + GRAM_BN) {
            const int c = tid - GRAM_BM;
            double s = 0.0;
            for (int k = 0; k < d; ++k) s = fma(Zt[k * GRAM_BN + c], Zt[k * GRAM_BN + c], s);
            z2[c] = s;
        }
    }
    __syncthreads();

    const int cl = (tid & 63) * 2;  // local column pair
    const int rg = tid >> 6;        // 0..3
    const int64_t gc = col0 + cl;
    if (gc >= p.m) return;
    const bool has2 = (gc + 1 < p.m);
    double* const K = p.K + (int64_t)blockIdx.z * p.bstride;
    const bool vec_ok = ((p.ldk & 1) == 0) && ((reinterpret_cast<uintptr_t>(K) & 15) == 0);
    const double diag_add = noise * p.noise_mult + p.jitter;

#pragma unroll 4
    for (int i = 0; i < GRAM_BM / 4; ++i) {
        const int rl = rg + 4 * i;
        const int64_t gr = row0 + rl;
        if (gr >= p.n) break;
        if (p.lower_only && gc > gr) continue;
        double v0, v1;
        if (!periodic) {
            double xz0 = 0.0, xz1 = 0.0;
            for (int k = 0; k < d; ++k) {
                const double x = Xs[rl * d + k];
                xz0 = fma(x, Zt[k * GRAM_BN + cl], xz0);
                xz1 = fma(x, Zt[k * GRAM_BN + cl + 1], xz1);
            }
            if (nngp) {   // theta: [0] = depth, [d] = var_w, [d+2] = var_b
                const bool relu = p.kind == B2GP_KERNEL_NNGP_RELU;
                const int depth = (int)ell[0];
                v0 = nngp_pair(relu, xz0, x2[rl], z2[cl], d, period, scale, depth);
                v1 = nngp_pair(relu, xz1, x2[rl], z2[cl + 1], d, period, scale, depth);
            } else {
                double r20 = (x2[rl] - 2.0 * xz0) + z2[cl];       // kernels.py:40
                double r21 = (x2[rl] - 2.0 * xz1) + z2[cl + 1];
                r20 = r20 < 0.0 ? 0.0 : r20;                      // kernels.py:41 (clip(0); NaN stays NaN)
                r21 = r21 < 0.0 ? 0.0 : r21;
                v0 = cov_from_r2(p.kind, r20, scale);
                v1 = cov_from_r2(p.kind, r21, scale);
            }
        } else {
            double s0 = 0.0, s1 = 0.0;
            for (int k = 0; k < d; ++k) {
                const double x = Xs[rl * d + k];
                // kernels.py:111-113
                const double a0 = sin(3.141592653589793 * (x - Zt[k * GRAM_BN + cl]) / period) / ell[k];
                const double a1 = sin(3.141592653589793 * (x - Zt[k * GRAM_BN + cl + 1]) / period) / ell[k];
                s0 += a0 * a0;
                s1 += a1 * a1;
            }
            v0 = scale * exp(-2.0 * s0);
            v1 = scale * exp(-2.0 * s1);
        }
        if (p.same_xz) {  // kernels.py:63-64
            if (gr == gc) v0 += diag_add;
            if (gr == gc + 1) v1 += diag_add;
        }
        double* dst = K + gr * p.ldk + gc;
        const bool w1 = has2 && !(p.lower_only && gc + 1 > gr);
        if (w1 && vec_ok) {
            *reinterpret_cast<double2*>(dst) = make_double2(v0, v1);
        } else {
            dst[0] = v0;
            if (w1) dst[1] = v1;
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// Specialised path (RBF / Matern-5/2, d <= 4): the generic kernel above is instruction-issue bound
// (ncu: 80 % issue-active, ~105 instructions per entry of which 26 are fp64).  Here the kernel family and
// d are template parameters, the two columns a thread owns live in registers, the row loop is unrolled,
// the diagonal / lower-triangle predicates are evaluated only in tiles that touch the diagonal, and exp()
// of a non-positive argument is a branch-free 17-operation sequence.

// exp() of a non-positive argument on a short fp64 budget.  n = rint(x log2 e) by the 1.5*2^52 trick,
// r = x - n ln2 (two-term ln2), exp(r) = (P9(r/4))^4 with P9 the degree-9 Taylor polynomial (|r/4| <= 0.087:
// remainder < 7e-18; the two squarings bring the result to ~4 ulp), 2^n applied to the exponent field.
// Range / NaN tests run on the integer pipe (high word of the argument), which is idle while the fp64 pipe is
// the binding resource: |x| > 708 or NaN takes a rare slow path that returns 0 (exact value < 4e-308) or NaN.
__device__ __forceinline__ double exp_quarter_poly(double u) {  // exp(4u), |u| <= 0.087
    double p = 2.7557319223985893e-06;             // 1/9!
    p = fma(p, u, 2.48015873015873e-05);           // 1/8!
    p = fma(p, u, 1.984126984126984e-04);          // 1/7!
    p = fma(p, u, 1.388888888888889e-03);          // 1/6!
    p = fma(p, u, 8.333333333333333e-03);          // 1/5!
    p = fma(p, u, 4.1666666666666664e-02);         // 1/4!
    p = fma(p, u, 1.6666666666666666e-01);         // 1/3!
    p = fma(p, u, 0.5);
    p = fma(p, u, 1.0);
    p = fma(p, u, 1.0);
    p = p * p;
    return p * p;
}
__device__ __forceinline__ double exp_finish(double p, int n, double x) {
    double res = __hiloint2double(__double2hiint(p) + (n << 20), __double2loint(p));
    if ((__double2hiint(x) & 0x7fffffff) > 0x40862000) res = (x != x) ? x : 0.0;   // |x| > 708 or NaN
    return res;
}
__device__ __forceinline__ double exp_nonpos(double x) {
    const double t = fma(x, 1.4426950408889634, 6755399441055744.0);
    const int n = __double2loint(t);
    const double nf = t - 6755399441055744.0;
    double r = fma(nf, -6.93147180369123816490e-01, x);
    r = fma(nf, -1.90821492927058770002e-10, r);
    return exp_finish(exp_quarter_poly(0.25 * r), n, x);
}
// exp(-r2/2) for r2 >= 0 with the -1/2 folded into the reduction: q = r2 + 2 n ln2 = -2r, u = r/4 = -q/8
__device__ __forceinline__ double exp_neg_half(double r2) {
    const double t = fma(r2, -0.7213475204444817, 6755399441055744.0);            // -0.5 * log2(e)
    const int n = __double2loint(t);
    const double nf = t - 6755399441055744.0;
    double q = fma(nf, 2.0 * 6.93147180369123816490e-01, r2);
    q = fma(nf, 2.0 * 1.90821492927058770002e-10, q);
    double p = -2.053180279134653e-14;                             // coefficients of P9(-q/8): (-1/8)^k / k!, k = 9
    p = fma(p, q, 1.47828980097695e-12);                           // k = 8
    p = fma(p, q, -9.46105472625248e-11);                          // k = 7
    p = fma(p, q, 5.298190646701389e-09);                          // k = 6
    p = fma(p, q, -2.5431315104166666e-07);                        // k = 5
    p = fma(p, q, 1.0172526041666666e-05);                         // k = 4
    p = fma(p, q, -3.255208333333333e-04);                         // k = 3
    p = fma(p, q, 7.8125e-03);                                     // k = 2
    p = fma(p, q, -0.125);
    p = fma(p, q, 1.0);
    p = p * p;
    p = p * p;
    double res = __hiloint2double(__double2hiint(p) + (n << 20), __double2loint(p));
    if ((__double2hiint(r2) & 0x7fffffff) > 0x40962000) res = (r2 != r2) ? r2 : 0.0;   // r2 > 1416 or NaN
    return res;
}
// clip at zero on the integer pipe: negative (sign bit set) -> +0; NaN with a clear sign bit stays NaN
__device__ __forceinline__ double clip0(double v) { return (__double2hiint(v) < 0) ? 0.0 : v; }

template <int KIND, int D>
__global__ void __launch_bounds__(GRAM_THREADS) gram_fast_kernel(const GramArgs p) {
    __shared__ double Xs[GRAM_BM][D];
    __shared__ double x2s[GRAM_BM];
    __shared__ double Zt[D][GRAM_BN];
    __shared__ double z2s[GRAM_BN];
    const int64_t row0 = (int64_t)blockIdx.y * GRAM_BM;
    const int64_t col0 = (int64_t)blockIdx.x * GRAM_BN;
    if (p.lower_only && col0 > row0 + GRAM_BM - 1) return;
    const int tid = threadIdx.x;
    const double* __restrict__ theta = p.theta + (int64_t)blockIdx.z * p.bstride;
    double ell[D];
#pragma unroll
    for (int k = 0; k < D; ++k) ell[k] = theta[k];
    const double scale = theta[D];
    const double diag_add = theta[D + 1] * p.noise_mult + p.jitter;

    if (tid < GRAM_BM) {
        const int64_t gr = row0 + tid;
        double s = 0.0;
#pragma unroll
        for (int k = 0; k < D; ++k) {
            const double v = (gr < p.n) ? p.X[gr * D + k] / ell[k] : 0.0;     // kernels.py:35 (a division)
            Xs[tid][k] = v;
            s = fma(v, v, s);
        }
        x2s[tid] = s;
    } else if (tid < GRAM_BM + GRAM_BN) {
        const int c = tid - GRAM_BM;
        const int64_t gc = col0 + c;
        double s = 0.0;
#pragma unroll
        for (int k = 0; k < D; ++k) {
            const double v = (gc < p.m) ? p.Z[gc * D + k] / ell[k] : 0.0;     // kernels.py:36
            Zt[k][c] = v;
            s = fma(v, v, s);
        }
        z2s[c] = s;
    }
    __syncthreads();

    const int cl = (tid & 63) * 2;
    const int rg = tid >> 6;
    const int64_t gc = col0 + cl;
    if (gc >= p.m) return;
    const bool has2 = (gc + 1 < p.m);
    double* const K = p.K + (int64_t)blockIdx.z * p.bstride;
    const bool vec_ok = ((p.ldk & 1) == 0) && ((reinterpret_cast<uintptr_t>(K) & 15) == 0);
    double z0[D], z1[D];
#pragma unroll
    for (int k = 0; k < D; ++k) {
        z0[k] = Zt[k][cl];
        z1[k] = Zt[k][cl + 1];
    }
    const double z20 = z2s[cl], z21 = z2s[cl + 1];
    // does this tile touch the diagonal (i == j somewhere)?  only then are per-entry predicates needed
    const bool on_diag = (row0 < col0 + GRAM_BN) && (col0 < row0 + GRAM_BM);
    const bool full_rows = (row0 + GRAM_BM <= p.n);

#pragma unroll 4
    for (int i = 0; i < GRAM_BM / 4; ++i) {
        const int rl = rg + 4 * i;
        const int64_t gr = row0 + rl;
        if (!full_rows && gr >= p.n) break;
        double xz0 = 0.0, xz1 = 0.0;
#pragma unroll
        for (int k = 0; k < D; ++k) {
            const double x = Xs[rl][k];
            xz0 = fma(x, z0[k], xz0);
            xz1 = fma(x, z1[k], xz1);
        }
        const double x2 = x2s[rl];
        double r20 = (x2 - 2.0 * xz0) + z20;        // kernels.py:40
        double r21 = (x2 - 2.0 * xz1) + z21;
        r20 = clip0(r20);                           // kernels.py:41
        r21 = clip0(r21);
        double v0, v1;
        if (KIND == B2GP_KERNEL_RBF) {              // kernels.py:62
            v0 = scale * exp_neg_half(r20);
            v1 = scale * exp_neg_half(r21);
        } else {                                    // kernels.py:85-88
            const double ra = sqrt(r20 + 1e-12), rb = sqrt(r21 + 1e-12);
            const double sa = 2.23606797749979 * ra, sb = 2.23606797749979 * rb;
            v0 = scale * (1.0 + sa + (5.0 / 3.0) * r20) * exp_nonpos(-sa);
            v1 = scale * (1.0 + sb + (5.0 / 3.0) * r21) * exp_nonpos(-sb);
        }
        double* dst = K + gr * p.ldk + gc;
        bool w0 = true, w1 = has2;
        if (on_diag) {
            if (p.same_xz) {                        // kernels.py:63-64
                if (gr == gc) v0 += diag_add;
                if (gr == gc + 1) v1 += diag_add;
            }
            if (p.lower_only) {
                w0 = (gc <= gr);
                w1 = w1 && (gc + 1 <= gr);
            }
        }
        if (w0 && w1 && vec_ok) {
            *reinterpret_cast<double2*>(dst) = make_double2(v0, v1);
        } else {
            if (w0) dst[0] = v0;
            if (w1) dst[1] = v1;
        }
    }
}

using GramKernel = void (*)(const GramArgs);

// the fixed-d kernel of KIND for d <= 4, else nullptr
template <int KIND>
static GramKernel gram_fast_for(int d) {
    switch (d) {
        case 1: return gram_fast_kernel<KIND, 1>;
        case 2: return gram_fast_kernel<KIND, 2>;
        case 3: return gram_fast_kernel<KIND, 3>;
        case 4: return gram_fast_kernel<KIND, 4>;
        default: return nullptr;
    }
}

// k(x,x) + diagonal term, computed exactly as the Gram kernel computes a diagonal entry
__device__ __forceinline__ double cov_self(int kind, double scale) {
    if (kind == B2GP_KERNEL_PERIODIC) return scale;  // sin(0) = 0, exp(-0) = 1
    return cov_from_r2(kind, 0.0, scale);
}

// `bt`: bt.n Gram matrices of the same X and Z, theta_dev and K bt.stride doubles apart per draw
static int launch_gram(b2gp_ctx* ctx, cudaStream_t st, int kind, const double* X, int64_t n, const double* Z, int64_t m,
                       int d, const double* theta_dev, double noise_mult, double jitter, int same_xz, int lower_only,
                       double* K, int64_t ldk, const Batch& bt = {}) {
    if (n <= 0 || m <= 0) return B2GP_OK;
    if (d < 1 || d > GRAM_MAX_D) return set_err(ctx, B2GP_ERR_UNSUPPORTED, "gram", "1 <= d <= 64", __FILE__, __LINE__);
    GramArgs a;
    a.X = X;
    a.Z = Z;
    a.n = n;
    a.m = m;
    a.d = d;
    a.kind = kind;
    a.theta = theta_dev;
    a.noise_mult = noise_mult;
    a.jitter = jitter;
    a.same_xz = same_xz;
    a.lower_only = lower_only;
    a.K = K;
    a.ldk = ldk;
    a.bstride = bt.stride;
    const size_t smem = (size_t)(GRAM_BM * d + GRAM_BM + d * GRAM_BN + GRAM_BN + d) * sizeof(double);
    static PerDeviceOnce attr;
    if (attr.need(ctx->device)) {
        CUDA_TRY(ctx, cudaFuncSetAttribute(gram_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 110 * 1024));
        attr.done(ctx->device);
    }
    dim3 grid((unsigned)ceil_div(m, GRAM_BN), (unsigned)ceil_div(n, GRAM_BM), (unsigned)bt.n);
    GramKernel fast = nullptr;
    if (kind == B2GP_KERNEL_RBF) fast = gram_fast_for<B2GP_KERNEL_RBF>(d);
    if (kind == B2GP_KERNEL_MATERN52) fast = gram_fast_for<B2GP_KERNEL_MATERN52>(d);
    if (fast) return launch(ctx, st, grid, GRAM_THREADS, 0, fast, a);
    return launch(ctx, st, grid, GRAM_THREADS, smem, gram_kernel, a);
}
