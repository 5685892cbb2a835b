// gemm_tma.cuh -- the large-problem form of the fp64 GEMM/SYRK: persistent CTAs, a TMA producer warp and an
// mbarrier ring feeding eight DMMA consumer warps.
//
// Same contract as gemm_dmma.cuh (C[m,n] = beta C + alpha A[m,k] B[n,k]^T, K-major operands, optional lower-only
// tile map); used when the 128x128 grid fills the machine.  What changes is how the tensor pipe is fed:
//   * operands arrive by TMA (cp.async.bulk.tensor.2d, 128-byte swizzle): one elected lane of warp 0 issues
//     [128 rows x 16 doubles] boxes for A and B and arms the stage's `full` mbarrier with the byte count;
//     out-of-range rows / k are zero-filled by the TMA unit, so ragged m, n, k need no predicates;
//   * consumers never meet at a CTA-wide barrier: each warp waits on `full[stage]`, issues its DMMAs, and
//     releases the slot with one arrive on `empty[stage]` (count 8) -- warps drift apart and keep the pipe busy;
//   * CTAs are persistent (grid = SM count): while the consumers run a tile's epilogue (read-modify-write of C)
//     the producer is already filling the ring with the next tile's first k-slices.
// The consumers issue the same m16n8k4 DMMA in the same k order as gemm_nt_kernel (dmma_slice16), so both give the same bits.
// Shared-memory tile = 128 rows x 128 B, 16-byte chunks XOR-swizzled with (row & 7) by the TMA unit; a fragment
// element (row r, column c) lives at  r*128 + (((c>>1) ^ (r&7)) << 4) + (c&1)*8.
#pragma once
#include <cuda.h>

#include "common.cuh"
#include "gemm_dmma.cuh"

constexpr int TG_BM = 128, TG_BN = 128;
constexpr int TG_CONSUMER_WARPS = 8;
constexpr int TG_THREADS = 32 * (TG_CONSUMER_WARPS + 1);
constexpr int TG_SUB_BYTES = 128 * 128;  // one [128 x 16 doubles] box

typedef CUresult (*PFN_tmapEncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                        const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                        CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_tmapEncodeTiled tmap_encoder() {
    static const PFN_tmapEncodeTiled fn = [] {  // initialised once, thread-safe
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            return (PFN_tmapEncodeTiled)p;
        return (PFN_tmapEncodeTiled) nullptr;
    }();
    return fn;
}

// 3-D fp64 map of `draws` row-major [rows x cols] matrices with leading dimension ld, `dstride` doubles apart (Batch):
// dimensions {cols, rows, draws}, box = 16 columns x 128 rows x 1 draw
static bool make_tmap(CUtensorMap* map, const double* base, int64_t rows, int64_t cols, int64_t ld, int draws, int64_t dstride) {
    PFN_tmapEncodeTiled enc = tmap_encoder();
    if (!enc) return false;
    if (draws == 1) dstride = rows * ld;   // unused, but the encoder wants a legal stride
    if ((dstride & 1) != 0) return false;
    cuuint64_t gdim[3] = {(cuuint64_t)cols, (cuuint64_t)rows, (cuuint64_t)draws};
    cuuint64_t gstride[2] = {(cuuint64_t)ld * 8, (cuuint64_t)dstride * 8};
    cuuint32_t box[3] = {16, 128, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    return enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 3, (void*)base, gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred P1;\n"
        "LAB_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
        "@P1 bra DONE;\n"
        "bra LAB_WAIT;\n"
        "DONE:\n"
        "}\n" ::"r"(bar),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t smem_dst, const CUtensorMap* map, int c0, int c1, uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
                     smem_dst),
                 "l"(map), "r"(bar), "r"(c0), "r"(c1)
                 : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t smem_dst, const CUtensorMap* map, int c0, int c1, int c2, uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(
                     smem_dst),
                 "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
                 : "memory");
}

__device__ __forceinline__ void tile_of(int x, int lower_only, int tiles_n, int& ti, int& tj) {
    if (lower_only) {
        int t = (int)((sqrt(8.0 * (double)x + 1.0) - 1.0) * 0.5);
        while ((int64_t)(t + 1) * (t + 2) / 2 <= x) ++t;
        while ((int64_t)t * (t + 1) / 2 > x) --t;
        ti = t;
        tj = x - t * (t + 1) / 2;
    } else {
        ti = x / tiles_n;
        tj = x % tiles_n;
    }
}

// KTRI: the in-place panel solve  C = A <- A B^T  with B lower triangular (B = L_bb^{-1}, see gemm_panel_solve in
// gemm_dmma.cuh).  A work unit is then a whole 128-row strip: its CTA walks the column tiles from right to left, and
// column tile j stops at k = 128 (j + 1) (B is zero beyond its diagonal block).  Tile j reads columns < 128 (j + 1) and
// writes columns 128 j .. 128 j + 127, so nothing a later tile of the strip reads has been overwritten, and no other CTA
// touches the strip's rows.  Right to left is also heaviest first.
// Batched (Batch): the persistent loop runs over (draw, tile) pairs, tile x of the batch being tile x % tpd of draw x / tpd.
template <int STAGES, int KSUB, bool KTRI = false>
__global__ void __launch_bounds__(TG_THREADS, 1)
gemm_tma_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB, const GemmArgs p, int num_tiles) {
    constexpr int BK = 16 * KSUB;
    constexpr int STAGE_BYTES = 2 * KSUB * TG_SUB_BYTES;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = (uint32_t)__cvta_generic_to_shared(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;             // 128B-swizzled tiles need 1024-byte alignment
    const uint32_t bars = base + STAGES * STAGE_BYTES;        // full[STAGES] then empty[STAGES]
    const uint8_t* sgen = smem_raw + (base - raw);            // generic pointer to the aligned tile area
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int KT = (p.k + BK - 1) / BK;

    if (tid == 0) {
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(bars + 8 * s, 1);
            mbar_init(bars + 8 * (STAGES + s), TG_CONSUMER_WARPS);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == 0) {
        // ------------------------------------------------------------ producer
        if (lane == 0) {
            uint32_t it = 0;
            for (int x = blockIdx.x; x < num_tiles; x += gridDim.x)
            for (int jj = 0; jj < (KTRI ? p.tiles_n : 1); ++jj) {
                const int draw = x / p.tpd, tile = x - draw * p.tpd;
                int ti, tj;
                if (KTRI) {
                    ti = tile;
                    tj = p.tiles_n - 1 - jj;
                } else {
                    tile_of(tile, p.lower_only, p.tiles_n, ti, tj);
                }
                const int row0 = ti * TG_BM, col0 = tj * TG_BN;
                const int KTt = KTRI ? min(KT, ((tj + 1) * TG_BN + BK - 1) / BK) : KT;
                for (int kt = 0; kt < KTt; ++kt, ++it) {
                    const uint32_t s = it % STAGES, ph = (it / STAGES) & 1u;
                    mbar_wait(bars + 8 * (STAGES + s), ph ^ 1u);
                    const uint32_t full = bars + 8 * s;
                    mbar_expect_tx(full, STAGE_BYTES);
                    const uint32_t st = base + s * STAGE_BYTES;
#pragma unroll
                    for (int sub = 0; sub < KSUB; ++sub) {
                        tma_load_3d(st + sub * TG_SUB_BYTES, &mapA, kt * BK + 16 * sub, row0, draw, full);
                        tma_load_3d(st + (KSUB + sub) * TG_SUB_BYTES, &mapB, kt * BK + 16 * sub, col0, draw, full);
                    }
                }
            }
        }
        return;
    }

    // ---------------------------------------------------------------- consumers: 8 warps, 2 x 4, 64 x 32 each
    const int cw = warp - 1;
    const int wm = cw >> 2, wn = cw & 3;
    const int g = lane >> 2, t4 = lane & 3;
    constexpr int MI = 8, NI = 4;
    // byte offsets inside a [128 x 128 B] swizzled box for this lane: row part, and the swizzled position of k = t4.
    // k = 4q + t4 is 16-byte chunk 2q + (t4 >> 1) XOR g, i.e. at x0 ^ (q << 5); the row bases are 128-byte aligned, so
    // the XOR can be applied to the whole row-base + x0 offset (one register instead of four).
    const uint32_t x0 = ((uint32_t)((t4 >> 1) ^ g) << 4) + ((uint32_t)(t4 & 1) << 3);
    const uint32_t a_row = (uint32_t)(wm * 64 + g) * 128u + x0;
    const uint32_t b_row = (uint32_t)(wn * 32 + g) * 128u + x0;
    const bool vec_ok = ((p.ldc & 1) == 0) && ((reinterpret_cast<uintptr_t>(p.C) & 15) == 0);   // bstride is even (make_tmap)

    uint32_t it = 0;
    for (int x = blockIdx.x; x < num_tiles; x += gridDim.x)
    for (int jj = 0; jj < (KTRI ? p.tiles_n : 1); ++jj) {
        int ti = 0, tj;
        if (KTRI)
            tj = p.tiles_n - 1 - jj;   // the strip (ti) is found after the k loop, see the epilogue
        else
            tile_of(x % p.tpd, p.lower_only, p.tiles_n, ti, tj);
        const int KTt = KTRI ? min(KT, ((tj + 1) * TG_BN + BK - 1) / BK) : KT;   // the producer's count
        double acc[MI][NI][2];
#pragma unroll
        for (int i = 0; i < MI; ++i)
#pragma unroll
            for (int j = 0; j < NI; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;

        for (int kt = 0; kt < KTt; ++kt, ++it) {
            const uint32_t s = it % STAGES, ph = (it / STAGES) & 1u;
            mbar_wait(bars + 8 * s, ph);
#pragma unroll
            for (int sub = 0; sub < KSUB; ++sub) {
                const uint8_t* box = sgen + s * STAGE_BYTES + sub * TG_SUB_BYTES;
                dmma_slice16(acc, [&](int i, int q) { return *reinterpret_cast<const double*>(box + (a_row ^ (q << 5)) + i * 1024); },
                             [&](int j, int q) {
                                 return *reinterpret_cast<const double*>(box + KSUB * TG_SUB_BYTES + (b_row ^ (q << 5)) + j * 1024);
                             });
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(bars + 8 * (STAGES + s));
        }

        // epilogue (identical to gemm_nt_kernel); the panel solve (KTRI) has alpha = 1, beta = 0 and no lower-only map.
        // The draw (and the KTRI strip) is derived here from the shuffled tile index rather than kept live across the
        // k loop: the accumulators leave no register to spare.
        const int xs = __shfl_sync(0xffffffffu, x, 0), draw = xs / p.tpd;
        if (KTRI) ti = xs - draw * p.tpd;
        const int row0 = ti * TG_BM, col0 = tj * TG_BN;
        double* const Cd = p.C + (int64_t)draw * p.bstride;
#pragma unroll
        for (int i = 0; i < MI; ++i) {
            const int r = row0 + wm * 64 + i * 8 + g;
            if (r >= p.m) continue;
#pragma unroll
            for (int j = 0; j < NI; ++j) {
                const int c = col0 + wn * 32 + j * 8 + t4 * 2;
                if (c >= p.n) continue;
                if (!KTRI && p.lower_only && c > r) continue;
                double* dst = Cd + (int64_t)r * p.ldc + c;
                const bool two = (c + 1 < p.n) && !(!KTRI && p.lower_only && c + 1 > r);
                double v0 = p.alpha * acc[i][j][0], v1 = p.alpha * acc[i][j][1];
                if (two && vec_ok) {
                    if (!KTRI && p.beta != 0.0) {
                        const double2 old = *reinterpret_cast<const double2*>(dst);
                        v0 += p.beta * old.x;
                        v1 += p.beta * old.y;
                    }
                    *reinterpret_cast<double2*>(dst) = make_double2(v0, v1);
                } else {
                    if (!KTRI && p.beta != 0.0) v0 += p.beta * dst[0];
                    dst[0] = v0;
                    if (two) {
                        if (!KTRI && p.beta != 0.0) v1 += p.beta * dst[1];
                        dst[1] = v1;
                    }
                }
            }
        }
    }
}

// returns B2GP_ERR_UNSUPPORTED when the operands do not meet TMA's alignment rules (caller falls back)
template <int STAGES, int KSUB, bool KTRI = false>
static int launch_gemm_tma(b2gp_ctx* ctx, cudaStream_t st, GemmArgs& a, int nb = 1) {
    constexpr int smem_bytes = STAGES * 2 * KSUB * TG_SUB_BYTES + 2 * STAGES * 8 + 1024;
    const bool ok = ((a.lda & 1) == 0) && ((a.ldb & 1) == 0) && ((reinterpret_cast<uintptr_t>(a.A) & 15) == 0) &&
                    ((reinterpret_cast<uintptr_t>(a.B) & 15) == 0);
    if (!ok) return B2GP_ERR_UNSUPPORTED;
    CUtensorMap mapA, mapB;
    if (!make_tmap(&mapA, a.A, a.m, a.k, a.lda, nb, a.bstride) || !make_tmap(&mapB, a.B, a.n, a.k, a.ldb, nb, a.bstride))
        return B2GP_ERR_UNSUPPORTED;
    a.tiles_m = (a.m + TG_BM - 1) / TG_BM;
    a.tiles_n = (a.n + TG_BN - 1) / TG_BN;
    const int64_t tpd = KTRI ? (int64_t)a.tiles_m : a.lower_only ? (int64_t)a.tiles_m * (a.tiles_m + 1) / 2 : (int64_t)a.tiles_m * a.tiles_n;
    if (tpd <= 0) return B2GP_OK;
    a.tpd = (int)tpd;
    const int64_t tiles = tpd * nb;
    static PerDeviceOnce attr;
    if (attr.need(ctx->device)) {
        CUDA_TRY(ctx, cudaFuncSetAttribute(gemm_tma_kernel<STAGES, KSUB, KTRI>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
        attr.done(ctx->device);
    }
    // Wave quantisation: with T tiles on S SMs the persistent kernel takes ceil(T/S) tile-times.  The T mod S tiles
    // of the last, partial wave are handed to a follow-up launch as 64x64 quarters (2 CTAs/SM): a quarter of the
    // work per CTA on four times the CTAs, so the tail costs ~0.3-0.6 tile-times instead of 1.
    const int S = persist_sms(ctx);
    // Not when C aliases an operand (the in-place leaf solve B <- B Linv^T): there each row block must be read and written
    // by ONE CTA, and the quarters of a tile are four CTAs, two of which would read the columns the other two overwrite.
    const bool inplace = (a.C == a.A || a.C == a.B);
    int64_t main_tiles = tiles;
    if (!inplace && tiles > S && tiles % S != 0) main_tiles = tiles - tiles % S;
    const int grid = (int)(main_tiles < S ? main_tiles : S);
    RET_IF(launch(ctx, PATH_GEMM_TMA, st, grid, TG_THREADS, smem_bytes, gemm_tma_kernel<STAGES, KSUB, KTRI>, mapA, mapB, a, (int)main_tiles));
    if (main_tiles < tiles) {
        GemmArgs t = a;
        t.tile_base = (int)main_tiles;
        t.sub = 1;
        t.tiles_m = (a.m + 63) / 64;
        t.tiles_n = (a.n + 63) / 64;
        constexpr int tail_smem = 4 * (64 + 64) * GEMM_LDS * (int)sizeof(double);
        auto kern = gemm_nt_kernel<64, 64, 2, 4, 4, true, 2>;
        static PerDeviceOnce tattr;
        if (tattr.need(ctx->device)) {
            CUDA_TRY(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, tail_smem));
            tattr.done(ctx->device);
        }
        RET_IF(launch(ctx, PATH_GEMM_NT, st, (unsigned)(4 * (tiles - main_tiles)), 256, tail_smem, kern, t));
    }
    return B2GP_OK;
}

static int gemm_tma_dispatch(b2gp_ctx* ctx, cudaStream_t st, GemmArgs& a, int nb) { return launch_gemm_tma<3, 2>(ctx, st, a, nb); }
static int gemm_tma_panel_dispatch(b2gp_ctx* ctx, cudaStream_t st, GemmArgs& a, int nb) {
    return launch_gemm_tma<3, 2, true>(ctx, st, a, nb);
}
