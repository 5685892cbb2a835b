// gemm_dmma.cuh -- C[m,n] = beta*C + alpha * A[m,k] * B[n,k]^T in fp64 on the DMMA tensor pipe.
//
// This is the trailing-update kernel of the blocked Cholesky (SYRK when A == B and lower_only),
// the B <- B * Linv^T "triangular solve by inverted diagonal block" kernel, and the covariance
// epilogue cov = k_pp - V^T V.  It stands where the reference calls jnp.matmul on the outputs of
// jnp.linalg.inv (gpax/models/gp.py:271-273).
//
// The fp64 tensor instruction used here is `mma.sync.m16n8k4.f64` (DMMA.16x8x4; sm_90 has no fp64 wgmma).  On the
// H100 it issues at twice the rate of the Ampere shape m8n8k4 (DESIGN.md 4.3, tools/dmma_peak.py), with the same
// operand registers: an m16 A fragment is rows g and g + 8, i.e. two m8 fragments (dmma_slice16).  Both operands are
// K-major (rows contiguous in k), so one shared-memory layout and one fragment pattern serve A and B:
//     a = As[(row0 + g) * LDS + 4*kk + t]      b = Bs[(col0 + g) * LDS + 4*kk + t]
// with g = lane/4, t = lane%4.  LDS = 20 doubles (160 B) makes the 8 rows x 32 B a half-warp reads
// land in 8 distinct 32-B bank groups -> conflict-free LDS.64.
//
// Pipeline: STAGES-deep cp.async (LDGSTS) ring of [BM+BN] x 16-double k-slices, one
// __syncthreads per k-slice.  Roofline: DMMA-bound; algorithmic flops per launch 2*m*n*k
// (m*n*k for the lower-only SYRK half).
#pragma once
#include "common.cuh"

// the draw offset of a kernel whose draw is blockIdx.y (Batch), re-read at every use rather than held in registers:
// several configurations run at their register cap
__device__ __forceinline__ int64_t ctaid_y_offset(int64_t bstride) {
    unsigned y;
    asm volatile("mov.u32 %0, %%ctaid.y;" : "=r"(y));
    return (int64_t)y * bstride;
}

struct GemmArgs {
    int m, n, k;
    const double* A;
    int64_t lda;
    const double* B;
    int64_t ldb;
    double* C;
    int64_t ldc;
    double alpha, beta;
    int lower_only;
    int tiles_m, tiles_n;
    int tile_base = 0;  // first 128x128 tile index covered by this launch (tail launches, see gemm_tma.cuh)
    int sub = 0;        // 1: blockIdx.x enumerates the four 64x64 quarters of 128x128 tiles tile_base, tile_base+1, ...
    int64_t bstride = 0;  // doubles between the draws' A, B and C (Batch); a draw is blockIdx.y, or tile / tpd for persistent and sub launches
    int tpd = 0;          // tiles per draw of the persistent kernel and of the sub launches (tiles numbered over the whole batch)
};

constexpr int GEMM_BK = 16;
constexpr int GEMM_LDS = 20;

__device__ __forceinline__ void cp_async_16(void* smem, const void* gmem, int src_bytes) {
    unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gmem), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_8(void* smem, const void* gmem, int src_bytes) {
    unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;\n" ::"r"(s), "l"(gmem), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory");
}

// Fragments (PTX ISA, "Matrix Fragments for mma.m8n8k4 / m16n8k4 / m16n8k8 / m16n8k16", .f64), g = lane/4, t = lane%4:
//   m8n8k4    a: (row g, k t)                     b: (k t, col g)                 c0,c1: (row g, cols 2t, 2t+1)
//   m16n8k4   a0: (g, t)   a1: (g+8, t)           b: (k t, col g)                 c0,c1: row g;  c2,c3: row g+8
//   m16n8k8   a[2j]: (g, t+4j)  a[2j+1]: (g+8, t+4j)   b[j]: (k t+4j, col g)     c as m16n8k4
//   m16n8k16  as m16n8k8 with j = 0..3
__device__ __forceinline__ void dmma884(double& c0, double& c1, double a, double b) {
    asm("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
        : "+d"(c0), "+d"(c1)
        : "d"(a), "d"(b));
}
// c0, c1 = rows g of the 16x8 block, c2, c3 = rows g + 8
__device__ __forceinline__ void dmma1684(double& c0, double& c1, double& c2, double& c3, double a0, double a1, double b0) {
    asm("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};\n"
        : "+d"(c0), "+d"(c1), "+d"(c2), "+d"(c3)
        : "d"(a0), "d"(a1), "d"(b0));
}
__device__ __forceinline__ void dmma1688(double& c0, double& c1, double& c2, double& c3, const double (&a)[4], const double (&b)[2]) {
    asm("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
        : "+d"(c0), "+d"(c1), "+d"(c2), "+d"(c3)
        : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
}
__device__ __forceinline__ void dmma16816(double& c0, double& c1, double& c2, double& c3, const double (&a)[8], const double (&b)[4]) {
    asm("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, "
        "{%0,%1,%2,%3};\n"
        : "+d"(c0), "+d"(c1), "+d"(c2), "+d"(c3)
        : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]), "d"(b[2]),
          "d"(b[3]));
}

// One 16-deep k-slice of a warp tile of MI x NI blocks of 8 x 8 on m16n8k4, the shape every fp64 GEMM kernel here issues
// (gemm_nt_kernel, gemm_tma_kernel, trsm_strip_kernel): the same instructions in the same k order, so the kernels agree
// bit for bit.  `lda(i, q)` returns A at row i*8 + g, k 4q + t (q = 0..3); `ldb(j, q)` B at column j*8 + g, k 4q + t.
// acc[i][j] keeps the m8n8 fragment (row i*8 + g, columns 2t, 2t+1): 8-row blocks 2i' and 2i'+1 are the c0,c1 and
// c2,c3 halves of m16 tile i', and their A values are its a0 and a1.  So the operand registers are those of m8n8k4, at
// twice its rate on Hopper (DESIGN.md 4.3).  Each instruction spans k 4q .. 4q+3 of the zero-filled slice.
template <int MI, int NI, class LA, class LB>
__device__ __forceinline__ void dmma_slice16(double (&acc)[MI][NI][2], LA lda, LB ldb) {
    static_assert(MI % 2 == 0, "m16 tiles");
#pragma unroll
    for (int q = 0; q < GEMM_BK / 4; ++q) {
        double a[MI], b[NI];
#pragma unroll
        for (int i = 0; i < MI; ++i) a[i] = lda(i, q);
#pragma unroll
        for (int j = 0; j < NI; ++j) b[j] = ldb(j, q);
#pragma unroll
        for (int i = 0; i < MI / 2; ++i)
#pragma unroll
            for (int j = 0; j < NI; ++j)
                dmma1684(acc[2 * i][j][0], acc[2 * i][j][1], acc[2 * i + 1][j][0], acc[2 * i + 1][j][1], a[2 * i], a[2 * i + 1], b[j]);
    }
}

// ---------------------------------------------------------------------------------------------- peak probe
// The fp64 tensor-pipe ceiling of each instruction shape, measured instead of assumed: every CTA (one per SM, eight
// warps, two per SM sub-partition) issues `iters` rounds of DMMA_PEAK_ACC independent MMAs of one shape on
// register-resident operands (no shared memory, no epilogue).  SHAPE 0: m8n8k4, 1: m16n8k4, 2: m16n8k8, 3: m16n8k16.
constexpr int DMMA_PEAK_THREADS = 256;
constexpr int DMMA_PEAK_ACC = 8;
__host__ __device__ constexpr int dmma_peak_fma(int shape) { return shape == 0 ? 8 * 8 * 4 : 16 * 8 * (4 << (shape - 1)); }

template <int SHAPE>
__global__ void __launch_bounds__(DMMA_PEAK_THREADS, 1) dmma_peak_kernel(int iters, double* sink) {
    const double x = 1.0 + 1e-3 * (double)(threadIdx.x & 31);
    double a[8], b[4], acc[DMMA_PEAK_ACC][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) a[i] = x * 1e-3 * (double)(i + 1);
#pragma unroll
    for (int j = 0; j < 4; ++j) b[j] = x - 1e-2 * (double)j;
#pragma unroll
    for (int u = 0; u < DMMA_PEAK_ACC; ++u) acc[u][0] = acc[u][1] = acc[u][2] = acc[u][3] = 0.0;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int u = 0; u < DMMA_PEAK_ACC; ++u) {
            double* c = acc[u];
            if (SHAPE == 0) dmma884(c[0], c[1], a[0], b[0]);
            if (SHAPE == 1) dmma1684(c[0], c[1], c[2], c[3], a[0], a[1], b[0]);
            if (SHAPE == 2) dmma1688(c[0], c[1], c[2], c[3], reinterpret_cast<const double(&)[4]>(a), reinterpret_cast<const double(&)[2]>(b));
            if (SHAPE == 3) dmma16816(c[0], c[1], c[2], c[3], a, b);
        }
    }
    double s = 0.0;
#pragma unroll
    for (int u = 0; u < DMMA_PEAK_ACC; ++u) s += acc[u][0] + acc[u][1] + acc[u][2] + acc[u][3];
    if (sink) sink[blockIdx.x * blockDim.x + threadIdx.x] = s;   // keeps the accumulators observable
}

// Load ROWS x 16 doubles (rows [row0, row0+ROWS) of a row-major matrix, columns [k0, k0+16)) into
// shared memory with stride GEMM_LDS; out-of-range rows / columns are zero-filled (cp.async zfill).
template <int ROWS, int NT, bool ALIGNED>
__device__ __forceinline__ void load_slice(double* sm, const double* __restrict__ base, int64_t ld, int rows_total,
                                           int k_total, int row0, int k0, int tid) {
    constexpr int VEC = ALIGNED ? 2 : 1;
    constexpr int CPR = GEMM_BK / VEC;  // chunks per row
#pragma unroll
    for (int c = tid; c < ROWS * CPR; c += NT) {
        const int r = c / CPR;
        const int ch = c % CPR;
        const int gr = row0 + r;
        const int gk = k0 + ch * VEC;
        int bytes = (k_total - gk) * 8;
        bytes = bytes < 0 ? 0 : (bytes > VEC * 8 ? VEC * 8 : bytes);
        if (gr >= rows_total) bytes = 0;
        const double* src = bytes > 0 ? base + (int64_t)gr * ld + gk : base;
        double* dst = sm + r * GEMM_LDS + ch * VEC;
        if (ALIGNED)
            cp_async_16(dst, src, bytes);
        else
            cp_async_8(dst, src, bytes);
    }
}

// KTRI: the in-place k-triangular panel solve of gemm_panel_solve -- one CTA per BM-row strip, column tiles from right to
// left, tile j with k < BN (j + 1) (as gemm_tma_kernel<.., true>, which explains why that order is race-free).
template <int BM, int BN, int WARPS_M, int WARPS_N, int STAGES, bool ALIGNED, int MINB, bool KTRI = false>
__global__ void __launch_bounds__(WARPS_M* WARPS_N * 32, MINB) gemm_nt_kernel(const GemmArgs p) {
    constexpr int NT = WARPS_M * WARPS_N * 32;
    constexpr int WTM = BM / WARPS_M, WTN = BN / WARPS_N;
    constexpr int MI = WTM / 8, NI = WTN / 8;
    constexpr int STAGE_ELEMS = (BM + BN) * GEMM_LDS;
    extern __shared__ __align__(16) double smem[];

    int ti, tj;
    int64_t soff = 0;   // the draw offset of a sub launch (tiles numbered over the batch); others take it from blockIdx.y
    {
        int x = p.sub ? p.tile_base + (int)(blockIdx.x >> 2) : p.tile_base + (int)blockIdx.x;
        if (!KTRI && p.sub) {
            const int draw = x / p.tpd;
            x -= draw * p.tpd;
            soff = (int64_t)draw * p.bstride;
        }
        const int tn = p.sub ? (p.tiles_n + 1) / 2 : p.tiles_n;   // tile columns in units of the indexed (128-wide) tiles
        if (p.lower_only) {
            int t = (int)((sqrt(8.0 * (double)x + 1.0) - 1.0) * 0.5);
            while ((int64_t)(t + 1) * (t + 2) / 2 <= x) ++t;
            while ((int64_t)t * (t + 1) / 2 > x) --t;
            ti = t;
            tj = x - t * (t + 1) / 2;
        } else {
            ti = x / tn;
            tj = x % tn;
        }
        if (p.sub) {
            ti = 2 * ti + (int)((blockIdx.x >> 1) & 1);
            tj = 2 * tj + (int)(blockIdx.x & 1);
            if (p.lower_only && tj > ti) return;
        }
    }
    const int tid = threadIdx.x;
    const int warp = tid >> 5, lane = tid & 31;
    const int wm = warp / WARPS_N, wn = warp % WARPS_N;
    const int g = lane >> 2, t4 = lane & 3;
    const bool vec_ok = ((p.ldc & 1) == 0) && ((reinterpret_cast<uintptr_t>(p.C) & 15) == 0) && ((p.bstride & 1) == 0);

    for (int jj = 0; jj < (KTRI ? p.tiles_n : 1); ++jj) {
    if (KTRI) {
        ti = (int)blockIdx.x;
        tj = p.tiles_n - 1 - jj;
        if (jj > 0) __syncthreads();   // every warp is done with the stages of the previous tile before the prologue refills them
    }
    const int row0 = ti * BM, col0 = tj * BN;
    double acc[MI][NI][2];
#pragma unroll
    for (int i = 0; i < MI; ++i)
#pragma unroll
        for (int j = 0; j < NI; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;

    const int KT = KTRI ? min((p.k + GEMM_BK - 1) / GEMM_BK, ((tj + 1) * BN + GEMM_BK - 1) / GEMM_BK) : (p.k + GEMM_BK - 1) / GEMM_BK;

    // prologue
#pragma unroll
    for (int s = 0; s < STAGES - 1; ++s) {
        if (s < KT) {
            double* As = smem + s * STAGE_ELEMS;
            double* Bs = As + BM * GEMM_LDS;
            load_slice<BM, NT, ALIGNED>(As, p.A + soff + ctaid_y_offset(p.bstride), p.lda, p.m, p.k, row0, s * GEMM_BK, tid);
            load_slice<BN, NT, ALIGNED>(Bs, p.B + soff + ctaid_y_offset(p.bstride), p.ldb, p.n, p.k, col0, s * GEMM_BK, tid);
        }
        cp_async_commit();
    }

    for (int kt = 0; kt < KT; ++kt) {
        cp_async_wait<STAGES - 2>();
        __syncthreads();
        {
            const int nk = kt + STAGES - 1;
            if (nk < KT) {
                double* As = smem + (nk % STAGES) * STAGE_ELEMS;
                double* Bs = As + BM * GEMM_LDS;
                load_slice<BM, NT, ALIGNED>(As, p.A + soff + ctaid_y_offset(p.bstride), p.lda, p.m, p.k, row0, nk * GEMM_BK, tid);
                load_slice<BN, NT, ALIGNED>(Bs, p.B + soff + ctaid_y_offset(p.bstride), p.ldb, p.n, p.k, col0, nk * GEMM_BK, tid);
            }
            cp_async_commit();
        }
        const double* As = smem + (kt % STAGES) * STAGE_ELEMS + (wm * WTM + g) * GEMM_LDS + t4;
        const double* Bs = smem + (kt % STAGES) * STAGE_ELEMS + BM * GEMM_LDS + (wn * WTN + g) * GEMM_LDS + t4;
        dmma_slice16(acc, [&](int i, int q) { return As[i * 8 * GEMM_LDS + q * 4]; },
                     [&](int j, int q) { return Bs[j * 8 * GEMM_LDS + q * 4]; });
    }
    cp_async_wait<0>();

    // epilogue: C = beta*C + alpha*acc.  Fragment (i,j): row g, columns 2*t4, 2*t4+1.
#pragma unroll
    for (int i = 0; i < MI; ++i) {
        const int r = row0 + wm * WTM + i * 8 + g;
        if (r >= p.m) continue;
#pragma unroll
        for (int j = 0; j < NI; ++j) {
            const int c = col0 + wn * WTN + j * 8 + t4 * 2;
            if (c >= p.n) continue;
            if (p.lower_only && c > r) continue;
            double* dst = p.C + soff + ctaid_y_offset(p.bstride) + (int64_t)r * p.ldc + c;
            const bool two = (c + 1 < p.n) && !(p.lower_only && c + 1 > r);
            double v0 = p.alpha * acc[i][j][0], v1 = p.alpha * acc[i][j][1];
            if (two && vec_ok) {
                if (p.beta != 0.0) {
                    const double2 old = *reinterpret_cast<const double2*>(dst);
                    v0 += p.beta * old.x;
                    v1 += p.beta * old.y;
                }
                *reinterpret_cast<double2*>(dst) = make_double2(v0, v1);
            } else {
                if (p.beta != 0.0) v0 += p.beta * dst[0];
                dst[0] = v0;
                if (two) {
                    if (p.beta != 0.0) v1 += p.beta * dst[1];
                    dst[1] = v1;
                }
            }
        }
    }
    }
}

template <int BM, int BN, int WARPS_M, int WARPS_N, int STAGES, int MINB, bool KTRI = false>
static int launch_gemm_cfg(b2gp_ctx* ctx, cudaStream_t st, GemmArgs& a, int nb = 1) {
    constexpr int smem_bytes = STAGES * (BM + BN) * GEMM_LDS * (int)sizeof(double);
    const bool aligned = ((a.lda & 1) == 0) && ((a.ldb & 1) == 0) && ((reinterpret_cast<uintptr_t>(a.A) & 15) == 0) &&
                         ((reinterpret_cast<uintptr_t>(a.B) & 15) == 0) && ((a.bstride & 1) == 0);
    a.tiles_m = (a.m + BM - 1) / BM;
    a.tiles_n = (a.n + BN - 1) / BN;
    int64_t grid = KTRI ? (int64_t)a.tiles_m : a.lower_only ? (int64_t)a.tiles_m * (a.tiles_m + 1) / 2 : (int64_t)a.tiles_m * a.tiles_n;
    if (grid <= 0) return B2GP_OK;
    auto kern = aligned ? gemm_nt_kernel<BM, BN, WARPS_M, WARPS_N, STAGES, true, MINB, KTRI>
                        : gemm_nt_kernel<BM, BN, WARPS_M, WARPS_N, STAGES, false, MINB, KTRI>;
    static PerDeviceOnce attr_set[2];
    if (attr_set[aligned ? 1 : 0].need(ctx->device)) {
        CUDA_TRY(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
        attr_set[aligned ? 1 : 0].done(ctx->device);
    }
    return launch(ctx, PATH_GEMM_NT, st, dim3((unsigned)grid, (unsigned)nb), WARPS_M * WARPS_N * 32, smem_bytes, kern, a);
}

static int gemm_tma_dispatch(b2gp_ctx* ctx, cudaStream_t st, GemmArgs& a, int nb);        // gemm_tma.cuh
static int gemm_tma_panel_dispatch(b2gp_ctx* ctx, cudaStream_t st, GemmArgs& a, int nb);  // gemm_tma.cuh
static int ozaki_dispatch(b2gp_ctx* ctx, cudaStream_t st, int64_t m, int64_t n, int64_t k, double alpha, const double* A, int64_t lda,
                          const double* B, int64_t ldb, double* C, int64_t ldc, bool lower_only, bool overwrite, bool transB,
                          bool ktri);  // ozaki.cuh

// C = beta*C + alpha*A*B^T.  lower_only requires a square C (m == n) whose diagonal is the matrix
// diagonal.  `inplace_rows` marks the B <- B*Linv^T use where C aliases A: that is only safe with a
// single column tile (n <= 128), which the 128-wide configuration guarantees.  `bt`: the same product on bt.n draws, the
// tile counts of the choices below taken over the whole batch (every configuration gives the same bits).
static int gemm_nt(b2gp_ctx* ctx, cudaStream_t st, int64_t m, int64_t n, int64_t k, double alpha, const double* A,
                   int64_t lda, const double* B, int64_t ldb, double beta, double* C, int64_t ldc, bool lower_only,
                   const Batch& bt = {}) {
    if (m <= 0 || n <= 0) return B2GP_OK;
    const int nb = bt.n;
    GemmArgs a;
    a.m = (int)m;
    a.n = (int)n;
    a.k = (int)k;
    a.A = A;
    a.lda = lda;
    a.B = B;
    a.ldb = ldb;
    a.C = C;
    a.ldc = ldc;
    a.alpha = alpha;
    a.beta = beta;
    a.lower_only = lower_only ? 1 : 0;
    a.bstride = bt.stride;
    if (lower_only && m < n) return set_err(ctx, B2GP_ERR_ARG, "gemm_nt", "lower_only needs m >= n", __FILE__, __LINE__);
    // Large rank-k updates C += alpha A B^T (the trailing updates of the factorisation and of the blocked solves) go
    // to the int8 wgmma path when it is enabled (ozaki.cuh).  It needs beta == 1, k within the int32 accumulation bound, enough 128x64 tiles to
    // fill the machine twice, and operands distinct from C (the in-place solve keeps the DMMA kernel).
    if (ctx->ozaki && beta == 1.0 && k >= 512 && C != A && C != B) {
        if (nb != 1) return set_err(ctx, B2GP_ERR_UNSUPPORTED, "gemm_nt", "the int8 route takes one draw", __FILE__, __LINE__);
        const int64_t tm = ceil_div(m, 128), tn = ceil_div(n, 64), sq = ceil_div(n, 128);
        const int64_t toz = lower_only ? sq * (sq + 1) + (tm - sq) * tn : tm * tn;   // lower triangle (+ the rows below it)
        if (toz >= ctx->oz_min_tiles) {
            const int rc = ozaki_dispatch(ctx, st, m, n, k, alpha, A, lda, B, ldb, C, ldc, lower_only, false, false, false);
            if (rc != B2GP_ERR_UNSUPPORTED) return rc;
        }
    }
    if (lower_only && m > n) {
        // trapezoid on the fp64 kernels (their lower-only tile maps are square): the square part, then the rows below it
        RET_IF(gemm_nt(ctx, st, n, n, k, alpha, A, lda, B, ldb, beta, C, ldc, true, bt));
        return gemm_nt(ctx, st, m - n, n, k, alpha, A + n * lda, lda, B, ldb, beta, C + n * ldc, ldc, false, bt);
    }
    // Tile choice.  A 128x128 tile keeps one SM busy for at least 128*128*k/128 cycles (DMMA.16x8x4: 128 fp64
    // FMA/clk/SM measured on the H100), i.e. ~8 us per k = 128, however few tiles there are; when the 128x128 grid would leave most of
    // the SMs idle, spend the same flops on more, smaller tiles.  The in-place triangular-solve
    // use (C aliases A, n <= 128) needs a single column tile, which all three configurations give.
    const int64_t tm128 = ceil_div(m, 128), tn128 = ceil_div(n, 128);
    const int64_t t128 = (lower_only ? tm128 * (tm128 + 1) / 2 : tm128 * tn128) * nb;
    if (t128 >= 112) {
        if (ctx->use_tma) {
            const int rc = gemm_tma_dispatch(ctx, st, a, nb);
            if (rc != B2GP_ERR_UNSUPPORTED) return rc;
        }
        // measured (tools/gemm_cfg.py): 3 stages beat 4 at large k; 16 warps (4 per SM sub-partition) beat 8 at small k
        if (k <= 1024) return launch_gemm_cfg<128, 128, 4, 4, 3, 1>(ctx, st, a, nb);
        return launch_gemm_cfg<128, 128, 2, 4, 3, 1>(ctx, st, a, nb);
    }
    if (lower_only) {
        // square tiles only for the triangular tile map
        return launch_gemm_cfg<64, 64, 2, 4, 4, 2>(ctx, st, a, nb);
    }
    // latency-bound regime: minimise (waves) x (time of one tile), in units of a 32x128 tile; the 128x128 kernel holds
    // one CTA per SM, the two smaller ones two
    const int64_t t64 = ceil_div(m, 64) * tn128 * nb, t32 = ceil_div(m, 32) * tn128 * nb;
    const int64_t c128 = ceil_div(t128, ctx->sm_count) * 4, c64 = ceil_div(t64, 2 * ctx->sm_count) * 2, c32 = ceil_div(t32, 2 * ctx->sm_count) * 1;
    if (c32 <= c64 && c32 <= c128) return launch_gemm_cfg<32, 128, 1, 8, 3, 2>(ctx, st, a, nb);
    if (c64 <= c128) return launch_gemm_cfg<64, 128, 2, 4, 3, 2>(ctx, st, a, nb);
    return launch_gemm_cfg<128, 128, 4, 4, 3, 1>(ctx, st, a, nb);
}

// The fp64 panel solve of the tall-panel factorisation (potrf.cuh, panel_solve_all_rows):  rows (m x n) <- rows Li^T,
// in place, with Li = L_bb^{-1} (n x n, lower, row-major, zero above the diagonal).  The k-triangular extent (column tile
// j needs k < 128 (j + 1)) makes it cost m n^2 flops, the triangular solve's count.  C overwrites A's columns, so a CTA
// owns a whole row strip and walks its column tiles from right to left (gemm_tma_kernel, KTRI) instead of solving into
// scratch and copying back.  128-row strips on the persistent TMA kernel from 16 strips up: with draws in flight on other
// streams the SMs a thin solve leaves idle run their work (DESIGN.md 4.3); below that gemm_nt's latency rule in row strips.
static int gemm_panel_solve(b2gp_ctx* ctx, cudaStream_t st, int64_t m, int64_t n, double* rows, int64_t ldr, const double* Li,
                            int64_t ldli, const Batch& bt = {}) {
    if (m <= 0 || n <= 0) return B2GP_OK;
    const int nb = bt.n;
    GemmArgs a;
    a.m = (int)m;
    a.n = (int)n;
    a.k = (int)n;
    a.A = rows;
    a.lda = ldr;
    a.B = Li;
    a.ldb = ldli;
    a.C = rows;
    a.ldc = ldr;
    a.alpha = 1.0;
    a.beta = 0.0;
    a.lower_only = 0;
    a.bstride = bt.stride;
    const int64_t tm128 = ceil_div(m, 128) * nb;   // strips over the batch
    if (tm128 >= 16) {
        if (ctx->use_tma) {
            const int rc = gemm_tma_panel_dispatch(ctx, st, a, nb);
            if (rc != B2GP_ERR_UNSUPPORTED) return rc;
        }
        return launch_gemm_cfg<128, 128, 4, 4, 3, 1, true>(ctx, st, a, nb);
    }
    const int64_t c128 = ceil_div(tm128, ctx->sm_count) * 4, c64 = ceil_div(ceil_div(m, 64) * nb, 2 * ctx->sm_count) * 2,
                  c32 = ceil_div(ceil_div(m, 32) * nb, 2 * ctx->sm_count);
    if (c32 <= c64 && c32 <= c128) return launch_gemm_cfg<32, 128, 1, 8, 3, 2, true>(ctx, st, a, nb);
    if (c64 <= c128) return launch_gemm_cfg<64, 128, 2, 4, 3, 2, true>(ctx, st, a, nb);
    return launch_gemm_cfg<128, 128, 4, 4, 3, 1, true>(ctx, st, a, nb);
}
