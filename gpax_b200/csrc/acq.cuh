// acq.cuh -- acquisition-function epilogues on the posterior's outputs (SURVEY.md section 8f-4).
//
// Replaces gpax/acquisition/base_acq.py:20-155 (ei, ucb, ue, poi on (mean, var)), the moment reduction of
// gpax/acquisition/acquisition.py:23-36 (_compute_mean_and_var over the [S*n, P] posterior samples) and the
// knowledge gradient of base_acq.py:158-232.  Everything here is elementwise / small reductions on arrays that the
// posterior kernels left in HBM; bound by those few bytes, never by arithmetic.
#pragma once
#include "common.cuh"

enum { ACQ_EI = 0, ACQ_UCB = 1, ACQ_UE = 2, ACQ_POI = 3 };

// standard normal cdf / pdf as numpyro's Normal(0, 1).cdf / exp(log_prob): cdf = ndtr(u) (erfc form: accurate in the tails)
__device__ __forceinline__ double norm_cdf(double u) { return 0.5 * erfc(-u * 0.7071067811865476); }
__device__ __forceinline__ double norm_pdf(double u) { return exp(-0.5 * u * u - 0.9189385332046727); }   // log sqrt(2 pi)

// best[r] = max (maximize) or min of mean[r, 0..P)   -- base_acq.py:59-60, 149-150 (`best_f is None`)
__global__ void __launch_bounds__(256) acq_best_kernel(const double* __restrict__ mean, int64_t ld, int64_t P, int maximize,
                                                       double* __restrict__ best) {
    __shared__ double red[8];
    const double* row = mean + (int64_t)blockIdx.x * ld;
    const double worst = maximize ? -INFINITY : INFINITY;
    double b = worst;
    bool nan = false;
    for (int64_t p = threadIdx.x; p < P; p += 256) {
        const double v = row[p];
        nan |= (v != v);
        b = maximize ? fmax(b, v) : fmin(b, v);
    }
    if (nan) b = __longlong_as_double(0x7ff8000000000000LL);     // jnp.max / min propagate NaN
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double t = __shfl_xor_sync(0xffffffffu, b, o);
        b = (b != b || t != t) ? __longlong_as_double(0x7ff8000000000000LL) : (maximize ? fmax(b, t) : fmin(b, t));
    }
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = b;
    __syncthreads();
    if (threadIdx.x == 0) {
        double r = red[0];
        for (int w = 1; w < 8; ++w) {
            const double t = red[w];
            r = (r != r || t != t) ? __longlong_as_double(0x7ff8000000000000LL) : (maximize ? fmax(r, t) : fmin(r, t));
        }
        best[blockIdx.x] = r;
    }
}

// out[r, p] = acq(mean[r, p], var[r, p]);  best[r] per row (EI / POI), param = beta (UCB) or xi (POI)
__global__ void acq_moments_kernel(int kind, const double* __restrict__ mean, const double* __restrict__ var, int64_t ld, int64_t R,
                                   int64_t P, const double* __restrict__ best, double param, int maximize, double* __restrict__ out,
                                   int64_t ldo) {
    const int64_t total = R * P;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = idx / P, p = idx % P;
        const double mu = mean ? mean[r * ld + p] : 0.0, v = var[r * ld + p];
        double a;
        if (kind == ACQ_EI) {                       // base_acq.py:61-69
            const double sigma = sqrt(v);
            double u = (mu - best[r]) / sigma;
            if (!maximize) u = -u;
            a = sigma * (norm_pdf(u) + u * norm_cdf(u));
        } else if (kind == ACQ_UCB) {               // base_acq.py:97-103
            const double delta = sqrt(param * v);
            a = maximize ? mu + delta : -(mu - delta);
        } else if (kind == ACQ_UE) {                // base_acq.py:129-130
            a = sqrt(v);
        } else {                                    // POI, base_acq.py:148-155
            const double sigma = sqrt(v);
            double u = (mu - best[r] - param) / sigma;
            if (!maximize) u = -u;
            a = norm_cdf(u);
        }
        out[r * ldo + p] = a;
    }
}

// column moments of the posterior samples: mean[p] = mean_r y[r, p], var[p] = mean_r (y[r, p] - mean[p])^2  (numpy's
// var, ddof = 0: acquisition.py:33-34).  Rows containing a NaN are NOT filtered here (the reference filters in predict).
__global__ void sample_moments_kernel(const double* __restrict__ y, int64_t R, int64_t P, double* __restrict__ mean,
                                      double* __restrict__ var) {
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P) return;
    double s = 0.0;
    for (int64_t r = 0; r < R; ++r) s += y[r * P + p];
    const double m = s / (double)R;
    double q = 0.0;
    for (int64_t r = 0; r < R; ++r) {
        const double dlt = y[r * P + p] - m;
        q = fma(dlt, dlt, q);
    }
    mean[p] = m;
    var[p] = q / (double)R;
}

// Knowledge gradient (base_acq.py:158-232) in closed form.  The reference appends (x_c, y_sim) to the training set
// and recomputes the posterior mean over all candidates for every candidate c and simulated value -- P * n
// re-inversions of an (N+1) x (N+1) matrix.  The block-inverse identity gives the same mean without touching K:
//     mean_aug[p] = mean[p] + C0[p, c] (y_sim - mean[c]) / (C0[c, c] + noise + jitter),
// C0 = k(X_new, X_new) - k_pX K^{-1} k_Xp the posterior covariance of the latent function (the `cov` output with its
// diagonal term noise_p + jitter removed).  One CTA per candidate c: for each of the n simulations the extremum over p.
//   cov[P, P] (symmetric; row c is read), ysim[n, P], diag_sub = noise_p + jitter, nj = noise + jitter; or, when
//   diag_sub_v / nj_v are given, per-candidate values diag_sub_v[c], nj_v[c] (a noise per task: the LCM models)
template <bool PER_CANDIDATE>
__global__ void __launch_bounds__(256) kg_kernel(const double* __restrict__ mean, const double* __restrict__ cov, int64_t ldc,
                                                 const double* __restrict__ ysim, int n, int64_t P, double diag_sub, double nj,
                                                 const double* __restrict__ diag_sub_v, const double* __restrict__ nj_v,
                                                 int maximize, const double* __restrict__ best_mean, double* __restrict__ out) {
    __shared__ double red[8];
    const int64_t c = blockIdx.x;
    if (PER_CANDIDATE) {
        diag_sub = diag_sub_v[c];
        nj = nj_v[c];
    }
    const double c0cc = cov[c * ldc + c] - diag_sub;
    const double inv_s = 1.0 / (c0cc + nj);
    const double mc = mean[c];
    double acc = 0.0;
    for (int i = 0; i < n; ++i) {
        const double g = (ysim[(int64_t)i * P + c] - mc) * inv_s;
        double b = maximize ? -INFINITY : INFINITY;
        for (int64_t p = threadIdx.x; p < P; p += 256) {
            const double c0 = (p == c) ? c0cc : cov[c * ldc + p];
            const double v = fma(c0, g, mean[p]);
            b = maximize ? fmax(b, v) : fmin(b, v);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const double t = __shfl_xor_sync(0xffffffffu, b, o);
            b = maximize ? fmax(b, t) : fmin(b, t);
        }
        __syncthreads();
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = b;
        __syncthreads();
        if (threadIdx.x == 0) {
            double r = red[0];
            for (int w = 1; w < 8; ++w) r = maximize ? fmax(r, red[w]) : fmin(r, red[w]);
            double u = r - best_mean[0];              // base_acq.py:213-217
            if (!maximize) u = -u;
            acc += u;
        }
    }
    if (threadIdx.x == 0) out[c] = acc / (double)n;   // kg_values.mean(0), base_acq.py:232
}
