// bnn.cuh -- the fully Bayesian MLP (gpax/models/bnn.py over spm.py): the Gaussian log-likelihood of y under z = MLP(X)
// with its gradient w.r.t. sigma and every weight, and the per-draw predictive forward pass, each fused into one kernel.
//
// The network is bnn.py:55-65: H_{l+1} = act(H_l W_l + b_l) with tanh hidden layers and a linear last layer, weights in
// the flat layout of b2gp_mlp_forward (per layer W_l [in, out] row-major, then b_l).  NUTS evaluates the likelihood up to
// 1,023 times per draw at small N, so the layered route (3 launches per layer forward, 4-6 backward) is launch-bound
// there; these kernels do a whole evaluation in two launches and a whole predict in one.
//
// bnn_loglik_tile_kernel: each CTA stages the weight set and a gradient accumulator of the same size in shared memory
// and walks row tiles of BNN_ROWS rows (tile t, t + gridDim.x, ...).  Per tile: the forward pass with every layer's
// activations kept in shared memory, the residual G = (y - z) / sigma^2 written over z, then the backward pass: bias
// gradient = column sum of G, dW_l = H_l^T G, and G <- (G W_l^T) * act'(H_l) written over H_l (each element is read and
// written by one thread, so in place is safe).  Each gradient element is owned by one thread and accumulated in tile
// order; sum r^2 per thread, then a fixed tree.  The CTA writes one partial row [grad params | sum r^2].
// bnn_reduce_kernel sums the rows in CTA order: no atomics, identical calls give identical bits.  Both kernels have a draw
// axis (grid.y, b2gp_bnn_loglik_draws): CTA (c, j) runs weight set s0 + j with its own 1 / sigma^2 over the same tiles a
// one-draw launch gives CTA c, so every draw gets the bits of its own b2gp_bnn_loglik call.
//
// bnn_predict_kernel: grid (row tiles, draws s0 .. s0 + gridDim.y - 1; more than 65535 draws take several launches).
// CTA (t, s) stages weight set s, runs the forward pass on its tile and writes
// loc[s, p, :] and, given eps, y[s, p, :] = loc + sigma_s * (sum_k eps[s, k, p, :]) / n (k in order): spm.py:150-154,
// Normal(loc, sigma).sample(key, (n,)).mean(0).
//
// bnn_predict_grad_kernel: the same grid and forward pass for a one-output network, then d loc / dX per row: the unit
// cotangent at the output, G <- (G W_l^T) * act'(H_l) in place over the activations for l = L-1 .. 1 (the likelihood
// kernel's step, bnn_tile_pullback) and dX = G W_0^T into the input buffer.  Every element has one owning thread and a
// fixed order: identical calls give identical bits.  Its shared memory is predict's, so it runs wherever predict runs
// fused; otherwise b2gp_bnn_predict_grad keeps the layered forward pass's hidden activations and runs dkl.cuh's
// mlp_input_vjp_kernel with unit cotangents.
//
// Route rule (bnn_fused_smem): the fused kernels run when 8 * (W + T) bytes fit in the device's opt-in shared memory
// per block (227 KB on the H100), with W = 2 * nparams for the likelihood (weights + gradient accumulator) and nparams
// for predict, T = BNN_ROWS * sum_l ld_l one tile's activations (ld_l = width_l rounded up to odd, for conflict-free
// strided reads), and at most BNN_MAX_LAYERS layers.  The default [64, 32] network fits for D <= 64 and O <= 8
// (148 KB at the largest); [512, 512] does not (2.1 MB of weights).  Otherwise the layered route runs: the b2gp_mlp_forward
// pass, bnn_resid_kernel (G and sum r^2) and the DKL backward pass; predict runs the forward pass per draw and
// bnn_sample_kernel.
#pragma once
#include "common.cuh"

constexpr int BNN_ROWS = 32;          // rows per tile
constexpr int BNN_THREADS = 256;
constexpr int BNN_MAX_LAYERS = 16;

// the network's shape as the fused kernels see it: dims[0] = D, dims[l + 1] = width of layer l (dims[L] = O); ld[l] the
// row stride of activation buffer l in shared memory, hoff[l] its offset (doubles) after the weights (and accumulators)
struct BnnNet {
    int L, nparams, htot;
    int dims[BNN_MAX_LAYERS + 1], ld[BNN_MAX_LAYERS + 1], hoff[BNN_MAX_LAYERS + 1];
    int woff[BNN_MAX_LAYERS], boff[BNN_MAX_LAYERS];
};

static inline BnnNet bnn_net(int64_t D, int L, const int64_t* widths) {
    BnnNet n{};
    n.L = L;
    n.dims[0] = (int)D;
    int o = 0;
    for (int l = 0; l < L; ++l) {
        n.dims[l + 1] = (int)widths[l];
        n.woff[l] = o;
        o += n.dims[l] * n.dims[l + 1];
        n.boff[l] = o;
        o += n.dims[l + 1];
    }
    n.nparams = o;
    int h = 0;
    for (int l = 0; l <= L; ++l) {
        n.ld[l] = n.dims[l] | 1;
        n.hoff[l] = h;
        h += BNN_ROWS * n.ld[l];
    }
    n.htot = h;
    return n;
}

// dynamic shared memory of the fused kernels; 0 when the network does not fit (the layered route runs)
static inline size_t bnn_fused_smem(int64_t D, int L, const int64_t* widths, bool grad, size_t optin) {
    if (L < 1 || L > BNN_MAX_LAYERS) return 0;
    double np = 0.0, h = (double)(D | 1);
    int64_t in = D;
    for (int l = 0; l < L; ++l) {
        np += (double)in * widths[l] + widths[l];
        h += (double)(widths[l] | 1);
        in = widths[l];
    }
    const double bytes = 8.0 * ((grad ? 2.0 : 1.0) * np + BNN_ROWS * h);
    const double fixed = grad ? 8.0 * BNN_THREADS : 0.0;   // the likelihood kernel's static reduction buffer
    return bytes + fixed <= (double)optin ? (size_t)bytes : 0;
}

static __device__ __forceinline__ double bnn_act(double v, int act) {
    return act == B2GP_ACT_RELU ? (v > 0.0 ? v : 0.0) : tanh(v);
}

// forward pass of one tile: H[0] staged by the caller, H[l+1] = act(H[l] W_l + b_l) (no activation on the last layer)
static __device__ void bnn_tile_forward(const BnnNet& net, int act, const double* Ws, double* H) {
    for (int l = 0; l < net.L; ++l) {
        const int in = net.dims[l], out = net.dims[l + 1], li = net.ld[l], lo = net.ld[l + 1];
        const double* Hin = H + net.hoff[l];
        double* Hout = H + net.hoff[l + 1];
        const double* W = Ws + net.woff[l];
        const double* b = Ws + net.boff[l];
        const bool last = l + 1 == net.L;
        for (int idx = threadIdx.x; idx < BNN_ROWS * out; idx += BNN_THREADS) {
            const int r = idx / out, j = idx % out;
            double acc = 0.0;
            for (int k = 0; k < in; ++k) acc = fma(Hin[r * li + k], W[k * out + j], acc);
            acc += b[j];
            Hout[r * lo + j] = last ? acc : bnn_act(acc, act);
        }
        __syncthreads();
    }
}

// one step of the tile's backward pass below layer l: G W_l^T with G = H[l+1], written in place over H[l] and masked by
// act'(H[l]) when MASK (the lanes of a warp take the 32 rows of one k: W[k, j] is a broadcast and G, H_l are read at the
// odd row stride, so the loop is free of bank conflicts; lanes along k would read W at a stride of `out` doubles).  Each
// element is read and written by one thread, in a fixed order over j.
template <bool MASK>
static __device__ __forceinline__ void bnn_tile_pullback(const BnnNet& net, int act, const double* Ws, double* H, int l) {
    const int in = net.dims[l], out = net.dims[l + 1], li = net.ld[l], lo = net.ld[l + 1];
    double* Hin = H + net.hoff[l];
    const double* G = H + net.hoff[l + 1];
    const double* W = Ws + net.woff[l];
    for (int idx = threadIdx.x; idx < BNN_ROWS * in; idx += BNN_THREADS) {
        const int k = idx / BNN_ROWS, r = idx % BNN_ROWS;
        double s = 0.0;
        for (int j = 0; j < out; ++j) s = fma(G[r * lo + j], W[k * out + j], s);
        if (MASK) {
            const double h = Hin[r * li + k];
            Hin[r * li + k] = act == B2GP_ACT_RELU ? (h > 0.0 ? s : 0.0) : s * (1.0 - h * h);
        } else {
            Hin[r * li + k] = s;
        }
    }
}

// stage the tile's input rows (zero beyond `rows`)
static __device__ void bnn_stage_x(const BnnNet& net, const double* __restrict__ X, int64_t row0, int64_t rows, double* H) {
    const int D = net.dims[0];
    for (int idx = threadIdx.x; idx < BNN_ROWS * D; idx += BNN_THREADS) {
        const int r = idx / D, k = idx % D;
        H[r * net.ld[0] + k] = row0 + r < rows ? X[(row0 + r) * D + k] : 0.0;
    }
}

// grid (row-tile CTAs, draws s0 .. s0 + gridDim.y - 1): CTA (c, j) stages weight set s = s0 + j (P + s * stride) with
// 1 / sigma_s^2 = inv_s2[s] and writes partial row j * gridDim.x + c.  Every draw sees the grid width and tile order of a
// one-draw launch, so its partial rows do not depend on how many draws share the launch.
__global__ void __launch_bounds__(BNN_THREADS)
bnn_loglik_tile_kernel(const BnnNet net, int act, const double* __restrict__ X, const double* __restrict__ y, int64_t N,
                       const double* __restrict__ P, int64_t stride, const double* __restrict__ inv_s2v, int64_t s0,
                       double* __restrict__ partial) {
    extern __shared__ double sm[];
    __shared__ double red[BNN_THREADS];
    double* Ws = sm;
    double* gs = sm + net.nparams;
    double* H = gs + net.nparams;
    const int np = net.nparams, O = net.dims[net.L];
    const int64_t s = s0 + blockIdx.y;
    const double inv_s2 = inv_s2v[s];
    P += s * stride;
    for (int i = threadIdx.x; i < np; i += BNN_THREADS) {
        Ws[i] = P[i];
        gs[i] = 0.0;
    }
    double r2 = 0.0;
    const int64_t ntiles = (N + BNN_ROWS - 1) / BNN_ROWS;
    for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const int64_t row0 = t * BNN_ROWS;
        __syncthreads();   // the previous tile is done with H (and, on the first, the weights are staged)
        bnn_stage_x(net, X, row0, N, H);
        __syncthreads();
        bnn_tile_forward(net, act, Ws, H);
        double* Z = H + net.hoff[net.L];
        const int lz = net.ld[net.L];
        for (int idx = threadIdx.x; idx < BNN_ROWS * O; idx += BNN_THREADS) {
            const int r = idx / O, o = idx % O;
            double g = 0.0;
            if (row0 + r < N) {
                const double res = y[row0 * O + idx] - Z[r * lz + o];
                r2 = fma(res, res, r2);
                g = res * inv_s2;
            }
            Z[r * lz + o] = g;   // rows beyond N carry G = 0 and add nothing below
        }
        __syncthreads();
        for (int l = net.L - 1; l >= 0; --l) {
            const int in = net.dims[l], out = net.dims[l + 1], li = net.ld[l], lo = net.ld[l + 1];
            double* Hin = H + net.hoff[l];
            const double* G = H + net.hoff[l + 1];
            for (int idx = threadIdx.x; idx < (in + 1) * out; idx += BNN_THREADS) {
                double s = 0.0;
                if (idx < in * out) {
                    const int k = idx / out, j = idx % out;
                    for (int r = 0; r < BNN_ROWS; ++r) s = fma(Hin[r * li + k], G[r * lo + j], s);
                    gs[net.woff[l] + idx] += s;
                } else {
                    const int j = idx - in * out;
                    for (int r = 0; r < BNN_ROWS; ++r) s += G[r * lo + j];
                    gs[net.boff[l] + j] += s;
                }
            }
            __syncthreads();
            if (l == 0) break;
            bnn_tile_pullback<true>(net, act, Ws, H, l);
            __syncthreads();
        }
    }
    red[threadIdx.x] = r2;
    __syncthreads();
    for (int o = BNN_THREADS / 2; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
        __syncthreads();
    }
    double* row = partial + ((int64_t)blockIdx.y * gridDim.x + blockIdx.x) * (np + 1);
    for (int i = threadIdx.x; i < np; i += BNN_THREADS) row[i] = gs[i];
    if (threadIdx.x == 0) row[np] = red[0];
}

// out[j, p] = sum_c partial[j, c, p] over the nrows rows of draw j (blockIdx.y) in order
__global__ void bnn_reduce_kernel(const double* __restrict__ partial, int nrows, int ld, double* __restrict__ out) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= ld) return;
    partial += (int64_t)blockIdx.y * nrows * ld;
    double s = 0.0;
    for (int c = 0; c < nrows; ++c) s += partial[(int64_t)c * ld + p];
    out[(int64_t)blockIdx.y * ld + p] = s;
}

// loc and y_sampled of one (row, output) element of draw s: the epilogue both predict routes share
static __device__ __forceinline__ void bnn_sample_out(double v, int64_t s, int64_t e, int64_t PO, const double* __restrict__ sigma,
                                                      const double* __restrict__ eps, int n, double* __restrict__ loc,
                                                      double* __restrict__ ys) {
    loc[s * PO + e] = v;
    if (eps) {
        double acc = 0.0;
        for (int k = 0; k < n; ++k) acc += eps[(s * n + k) * PO + e];
        ys[s * PO + e] = v + sigma[s] * (acc / n);
    }
}

__global__ void __launch_bounds__(BNN_THREADS)
bnn_predict_kernel(const BnnNet net, int act, const double* __restrict__ X, int64_t Pn, const double* __restrict__ P,
                   int64_t stride, const double* __restrict__ sigma, const double* __restrict__ eps, int n,
                   double* __restrict__ loc, double* __restrict__ ys, int64_t s0) {
    extern __shared__ double sm[];
    double* Ws = sm;
    double* H = sm + net.nparams;
    const int64_t s = s0 + blockIdx.y, row0 = (int64_t)blockIdx.x * BNN_ROWS;
    for (int i = threadIdx.x; i < net.nparams; i += BNN_THREADS) Ws[i] = P[s * stride + i];
    bnn_stage_x(net, X, row0, Pn, H);
    __syncthreads();
    bnn_tile_forward(net, act, Ws, H);
    const int O = net.dims[net.L], lz = net.ld[net.L];
    const double* Z = H + net.hoff[net.L];
    for (int idx = threadIdx.x; idx < BNN_ROWS * O; idx += BNN_THREADS) {
        const int r = idx / O, o = idx % O;
        if (row0 + r < Pn) bnn_sample_out(Z[r * lz + o], s, row0 * O + idx, Pn * O, sigma, eps, n, loc, ys);
    }
}

// bnn_predict_kernel's grid and forward pass for a one-output network, then the gradient of loc w.r.t. the inputs:
// the unit cotangent seeds the (linear) output layer, bnn_tile_pullback runs down the layers over the activations and
// dX = G W_0^T lands in the input buffer, free by then.  Writes loc[s, p] (bit-identical to bnn_predict_kernel's) and
// dloc[s, p, :].  Same shared memory as predict: the weights and one tile.
__global__ void __launch_bounds__(BNN_THREADS)
bnn_predict_grad_kernel(const BnnNet net, int act, const double* __restrict__ X, int64_t Pn, const double* __restrict__ P,
                        int64_t stride, double* __restrict__ loc, double* __restrict__ dloc, int64_t s0) {
    extern __shared__ double sm[];
    double* Ws = sm;
    double* H = sm + net.nparams;
    const int64_t s = s0 + blockIdx.y, row0 = (int64_t)blockIdx.x * BNN_ROWS;
    for (int i = threadIdx.x; i < net.nparams; i += BNN_THREADS) Ws[i] = P[s * stride + i];
    bnn_stage_x(net, X, row0, Pn, H);
    __syncthreads();
    bnn_tile_forward(net, act, Ws, H);
    if (threadIdx.x < BNN_ROWS) {
        double* z = H + net.hoff[net.L] + threadIdx.x * net.ld[net.L];
        if (row0 + threadIdx.x < Pn) loc[s * Pn + row0 + threadIdx.x] = *z;
        *z = 1.0;
    }
    __syncthreads();
    for (int l = net.L - 1; l >= 1; --l) {
        bnn_tile_pullback<true>(net, act, Ws, H, l);
        __syncthreads();
    }
    bnn_tile_pullback<false>(net, act, Ws, H, 0);
    __syncthreads();
    const int D = net.dims[0];
    const int64_t rows = Pn - row0 < BNN_ROWS ? Pn - row0 : BNN_ROWS;
    for (int idx = threadIdx.x; idx < rows * D; idx += BNN_THREADS) {
        const int r = idx / D, k = idx % D;
        dloc[(s * Pn + row0) * D + idx] = H[r * net.ld[0] + k];
    }
}

// layered route: G = (y - z) / sigma^2 over the N*O entries, r2[0] = sum (y - z)^2.  One CTA, a fixed per-thread
// order and a fixed tree: deterministic.
__global__ void __launch_bounds__(BNN_THREADS)
bnn_resid_kernel(const double* __restrict__ z, const double* __restrict__ y, int64_t n, double inv_s2, double* __restrict__ G,
                 double* __restrict__ r2) {
    __shared__ double red[BNN_THREADS];
    double acc = 0.0;
    for (int64_t i = threadIdx.x; i < n; i += BNN_THREADS) {
        const double res = y[i] - z[i];
        acc = fma(res, res, acc);
        G[i] = res * inv_s2;
    }
    red[threadIdx.x] = acc;
    __syncthreads();
    for (int o = BNN_THREADS / 2; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) r2[0] = red[0];
}

// layered route's predict epilogue for draw s: loc[s] = Z, y_sampled[s] as bnn_predict_kernel
__global__ void bnn_sample_kernel(const double* __restrict__ Z, int64_t PO, int64_t s, const double* __restrict__ sigma,
                                  const double* __restrict__ eps, int n, double* __restrict__ loc, double* __restrict__ ys) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < PO; e += (int64_t)gridDim.x * blockDim.x)
        bnn_sample_out(Z[e], s, e, PO, sigma, eps, n, loc, ys);
}
