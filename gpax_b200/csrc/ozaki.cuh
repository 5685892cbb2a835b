// ozaki.cuh -- fp64 GEMM/SYRK on the int8 tensor cores (wgmma) by integer splitting (Ozaki scheme).
//
// sm_90a's fp64 tensor-core rate (DMMA) is a small fraction of its int8 wgmma rate, and int8 products accumulate
// exactly in int32.  C[m,n] += alpha * A[m,k] B[n,k]^T is evaluated as follows.
//   1. slice (oz_slice_kernel): every row of A (and B) is scaled by a power of two 2^-e_i so that |a| < 1, rounded ONCE
//      to the integer I = rint(a 2^(8S-2-e_i)) (|I| <= 2^(8S-2)) and cut into S base-256 digits in two's-complement
//      style, lowest first: d = signed low byte of I in [-128, 127], I <- (I - d) >> 8; the leading digit is what is left
//      (6 bits + a carry).  Full-range int8 digits: 8 bits per plane instead of the 7 of a round-to-nearest base-128 split,
//      so S = 7 planes carry 54 bits and 28 products; S = 6 carry 46 bits and 21 products.
//         a = 2^e_i * sum_q d_q 2^-w(q),   w(q) = 6 + 8 q,  q = 0 .. S-1   (exact to half a unit of the last digit)
//      The digits are stored as S int8 planes [S][rows][k], K-major.
//   2. products (oz_mma_kernel): A_p B_q^T is an int8 GEMM; its int32 result is EXACT (|d d'| <= 2^14, at most S pairs
//      per accumulator, k <= OZ_K_MAX = 16384 per launch: 7 * 2^14 * 2^14 < 2^31; longer k is split by the dispatcher).
//      Its weight 2^-(12 + 8 (p+q)) depends on t = p+q only, so all pairs of one weight class accumulate into the
//      same register accumulator.  Classes t >= S are below the target precision and are dropped: S(S+1)/2 products.
//   3. recombine (epilogue of the same kernel): acc = sum_t 2^-(12+8t) D_t in fp64, smallest class first, and
//      C[i,j] += alpha * 2^(e_i + f_j) * acc.
// Kernel organisation: see oz_mma_kernel.  Operands arrive by TMA (32-byte swizzle, one 32-byte k-block = one wgmma K
// step per stage, every plane fetched once per k-block and pass and used by every pair it takes part in).
#pragma once
#include <cuda.h>

#include "common.cuh"
#include "gemm_tma.cuh"

constexpr int OZ_BM = 128, OZ_BN = 64, OZ_KB = 32;   // 32-byte k-blocks (one MMA K step)
// stages in flight: as many as fit in 227 KB of shared memory -- 6 x 36 KB with 6 planes, 5 x 42 KB with 7
__host__ __device__ constexpr int oz_stages_for(int S) { return S <= 6 ? 6 : 5; }
constexpr int OZ_THREADS = 384;           // two consumer warpgroups + one producer warpgroup (one thread of it issues TMA)
// A tile makes several passes over k, each for a window of weight classes, from the smallest weights down: the first
// takes S-4 .. S-1 (4 x 32 accumulator registers per thread, no partial sum live yet), every later one at most two
// classes (2 x 32 accumulators beside the 64 registers of the fp64 partial sum).  More live accumulators than that
// exceed the 168 registers a consumer thread may hold, and ptxas then serialises the wgmma chain.
__host__ __device__ constexpr int oz_pass_hi(int S, int pass) { return pass == 0 ? S - 1 : S - 5 - 2 * (pass - 1); }
__host__ __device__ constexpr int oz_pass_lo(int S, int pass) {
    return pass == 0 ? S - 4 : (oz_pass_hi(S, pass) - 1 > 0 ? oz_pass_hi(S, pass) - 1 : 0);
}
__host__ __device__ constexpr int oz_passes(int S) { return S <= 4 ? 1 : 1 + (S - 4 + 1) / 2; }
constexpr int OZ_K_MAX = 16384;           // int32 accumulation bound of one launch (see above)
constexpr int OZ_A_TILE = OZ_BM * OZ_KB;  // 4096 B
constexpr int OZ_B_TILE = OZ_BN * OZ_KB;  // 2048 B

struct OzArgs {
    int m, n, kb_count;        // kb_count = padded k / OZ_KB
    int rowsA_pad, rowsB_pad;  // rows of one digit plane (multiple of 128)
    const double* sa;          // 2^e_i per row of A
    const double* sb;          // 2^f_j per row of B
    double* C;
    int64_t ldc;
    double alpha;
    int lower_only;
    int tiles_m, tiles_n;
    int num_tiles;
    const int2* tile_list;  // [num_tiles] (ti, tj) in execution order (host-built, L2-friendly)
    int overwrite;  // 1: C = alpha A B^T (C is not read: beta = 0; C may alias the fp64 source of A, which was copied to planes)
    int ktri;       // 1: B is lower triangular (B[c][k] = 0 for k > c): a column tile needs only the k-blocks up to its last row
    int debug;  // 0 normal; != 0 skip the global read-modify-write (timing experiments only)
    long long* prof;  // optional [gridDim.x][8]: consumer cycles (wait TMA, epilogue), -, tiles, -, producer (wait free stage, total)
};

// ---------------------------------------------------------------------------------------------- slicing
// one CTA per row: row maximum -> exponent, then S digits per element; planes[p][row][kk]
// trans != 0: the operand is the TRANSPOSE of the stored matrix, element (row, kk) = A[kk * lda + row] (small operands only:
// the reads are strided)
template <int S>
__global__ void __launch_bounds__(256) oz_slice_kernel(const double* __restrict__ A, int64_t lda, int rows, int k, int8_t* __restrict__ planes,
                                                       int rows_pad, int kpad, double* __restrict__ scale, int trans,
                                                       const int64_t* __restrict__ rowmap128) {
    __shared__ double red[8];
    const int row = blockIdx.x;
    const int tid = threadIdx.x;
    const int64_t sr = trans ? 1 : lda, sk = trans ? lda : 1;   // strides of (row, kk)
    if (rowmap128) A += (rowmap128[row >> 7] - (int64_t)(row & ~127)) * lda;   // source row = rowmap128[row / 128] + row % 128
    int e = 0;
    if (row < rows) {
        double mx = 0.0;
        for (int kk = tid; kk < k; kk += 256) mx = fmax(mx, fabs(A[(int64_t)row * sr + (int64_t)kk * sk]));
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        if ((tid & 31) == 0) red[tid >> 5] = mx;
        __syncthreads();
        mx = red[0];
        for (int w = 1; w < 8; ++w) mx = fmax(mx, red[w]);
        if (mx > 0.0 && mx < 1e300) frexp(mx, &e);  // mx = f * 2^e, f in [0.5, 1)
        if (e < -900) e = -900;                      // 2^(8S-2-e) below must stay finite
        if (tid == 0) scale[row] = ldexp(1.0, e);
    }
    const double up = ldexp(1.0, 8 * S - 2 - e);     // exact power of two: a * up is the exact scaling
    // 4 consecutive k per thread -> one 32-bit store per plane
    for (int k4 = tid * 4; k4 < kpad; k4 += 1024) {
        int packed[S];
#pragma unroll
        for (int p = 0; p < S; ++p) packed[p] = 0;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int kk = k4 + j;
            long long I = (row < rows && kk < k) ? __double2ll_rn(A[(int64_t)row * sr + (int64_t)kk * sk] * up) : 0ll;
#pragma unroll
            for (int p = S - 1; p > 0; --p) {
                const int d = (int)(signed char)(I & 0xff);          // signed low byte
                packed[p] |= (d & 0xff) << (8 * j);
                I = (I - d) >> 8;
            }
            packed[0] |= ((int)I & 0xff) << (8 * j);
        }
#pragma unroll
        for (int p = 0; p < S; ++p)
            *reinterpret_cast<int*>(planes + ((int64_t)p * rows_pad + row) * kpad + k4) = packed[p];
    }
}

// ---------------------------------------------------------------------------------------------- wgmma / cluster helpers
// TMA box load delivered to the same shared-memory offset (and signalling the same barrier offset) in every CTA of `mask`
__device__ __forceinline__ void tma_load_2d_mc(uint32_t smem_dst, const CUtensorMap* map, int c0, int c1, uint32_t bar, uint16_t mask) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(
            smem_dst),
        "l"(map), "r"(bar), "r"(c0), "r"(c1), "h"(mask)
        : "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// arrive on the barrier at shared-memory offset `bar` of CTA `cta` of the cluster (the own CTA included)
__device__ __forceinline__ void mbar_arrive_cta(uint32_t bar, uint32_t cta) {
    uint32_t remote;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(bar), "r"(cta));
    asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
}
// a consumed stage goes back to the producer of every CTA that wrote into it
template <int CL>
__device__ __forceinline__ void oz_release(uint32_t empty_bar) {
    if constexpr (CL == 1)
        mbar_arrive(empty_bar);
    else
        for (int r = 0; r < CL; ++r) mbar_arrive_cta(empty_bar, (uint32_t)r);
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving reads of accumulator registers above the wgmma.wait_group that completes them
template <int N>
__device__ __forceinline__ void wg_fence_regs(int (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+r"(d[i])::"memory");
}

#define OZ_R8(i) "+r"(d[i]), "+r"(d[i + 1]), "+r"(d[i + 2]), "+r"(d[i + 3]), "+r"(d[i + 4]), "+r"(d[i + 5]), "+r"(d[i + 6]), "+r"(d[i + 7])
#define OZ_R32(i) OZ_R8(i), OZ_R8(i + 8), OZ_R8(i + 16), OZ_R8(i + 24)
// D[64 x 64 NQ] += A[64 x 32] B[64 NQ x 32]^T, int8 x int8 -> int32, both operands K-major in shared memory; the
// accumulator of m64nN is N / 2 registers per thread (NQ = 1: the digit-plane products, NQ = 4: the peak probe).
template <int NQ>
__device__ __forceinline__ void wg_mma_i8(int* d, uint64_t adesc, uint64_t bdesc) {
    if constexpr (NQ == 1) {
        asm volatile(
            "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
            "wgmma.mma_async.sync.aligned.m64n64k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
            "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p;\n}\n"
            : OZ_R32(0)
            : "l"(adesc), "l"(bdesc), "r"(1));
    } else {
        static_assert(NQ == 4, "N = 64 or 256");
        asm volatile(
            "{\n.reg .pred p;\nsetp.ne.b32 p, %130, 0;\n"
            "wgmma.mma_async.sync.aligned.m64n256k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
            "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, "
            "%40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
            "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, "
            "%88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, "
            "%110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p;\n}\n"
            : OZ_R32(0), OZ_R32(32), OZ_R32(64), OZ_R32(96)
            : "l"(adesc), "l"(bdesc), "r"(1));
    }
}
#undef OZ_R32
#undef OZ_R8

// shared-memory matrix descriptor (sm_90 wgmma), K-major, 32-byte swizzle (rows of 32 B): 8-row groups are 256 B apart
__device__ __forceinline__ uint64_t oz_smem_desc(uint32_t saddr) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3fff);   // start address
    d |= (uint64_t)1 << 16;                   // leading byte offset (unused for swizzled K-major)
    d |= (uint64_t)(256 >> 4) << 32;          // stride byte offset
    d |= (uint64_t)3 << 62;                   // SWIZZLE_32B
    return d;
}
// exact int32 -> double without I2F.F64 (the conversion instruction has a low issue rate and would be the whole
// epilogue): 2^52 + 2^31 + v is assembled in the mantissa, the constant subtracted.
__device__ __forceinline__ double i32_to_f64(int v) {
    return __hiloint2double(0x43300000, v ^ 0x80000000) - 4503601774854144.0;
}
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

// The products of one stage for the weight classes LO..HI: A plane PP meets B planes Q = max(0, LO - PP) .. HI - PP, one
// m64n64 wgmma per pair into the accumulator of class PP + Q.  acc[32 (t - LO) + j] is element j of class t.  (One wide-N
// wgmma over the stacked B planes would cover several classes at once, but the register ranges of consecutive
// instructions would then overlap partially, and ptxas serialises such a chain.)
template <int LO, int HI, int PP, int Q>
__device__ __forceinline__ void oz_stage_mmas(int* acc, uint32_t a0, uint32_t b0) {
    if constexpr (PP <= HI) {
        constexpr int QQ = Q < LO - PP ? LO - PP : Q;
        wg_mma_i8<1>(acc + 32 * (PP + QQ - LO), oz_smem_desc(a0 + PP * OZ_A_TILE), oz_smem_desc(b0 + QQ * OZ_B_TILE));
        if constexpr (QQ < HI - PP)
            oz_stage_mmas<LO, HI, PP, QQ + 1>(acc, a0, b0);
        else
            oz_stage_mmas<LO, HI, PP + 1, 0>(acc, a0, b0);
    }
}

// k-blocks a tile of column pair / column tile `ty` runs over: all of them, or -- B lower triangular -- those up to
// the last row of B the tile (the CTA pair's tiles, which share the A stages) touches
__device__ __forceinline__ int oz_kb_count(const OzArgs& p, int CL, int ty) {
    if (!p.ktri) return p.kb_count;
    const int lim = ((CL * ty + CL) * OZ_BN + OZ_KB - 1) / OZ_KB;
    return lim < p.kb_count ? lim : p.kb_count;
}

// One pass of a consumer warpgroup over the k-blocks of a tile for the classes LO..HI, then the classes folded into the
// fp64 partial sum, smallest weight first (FIRST: the partial sum starts here).  `it` counts stages consumed by this CTA
// (shared with the producer's order).  The pass reads digit planes 0 .. HI.
template <int S, int CL, int LO, int HI, bool FIRST>
__device__ __forceinline__ void oz_consume_pass(const OzArgs& p, int kbn, uint32_t base, uint32_t full0, uint32_t empty0, int wg, uint32_t& it,
                                                double (&part)[32], long long& c_wait) {
    constexpr int NACC = 32 * (HI - LO + 1);
    constexpr int STAGE_BYTES = S * (OZ_A_TILE + OZ_B_TILE);
    constexpr int OZ_STAGES = oz_stages_for(S);
    const bool leader = (threadIdx.x & 127) == 0;
    int acc[NACC];
#pragma unroll
    for (int j = 0; j < NACC; ++j) acc[j] = 0;
    uint32_t prev = 0xffffffffu;
    for (int kb = 0; kb < kbn; ++kb, ++it) {
        const uint32_t s = it % OZ_STAGES, ph = (it / OZ_STAGES) & 1u;
        const long long f0 = p.prof ? clock64() : 0;
        mbar_wait(full0 + 8 * s, ph);
        if (p.prof) c_wait += clock64() - f0;
        const uint32_t st = base + s * STAGE_BYTES;
        wg_fence();
        oz_stage_mmas<LO, HI, 0, 0>(acc, st + wg * (OZ_A_TILE / 2), st + S * OZ_A_TILE);
        wg_commit();
        wg_wait<1>();   // the previous stage's products are done: its buffers go back to the producer(s)
        if (prev != 0xffffffffu && leader) oz_release<CL>(empty0 + 8 * prev);
        prev = s;
    }
    wg_wait<0>();
    wg_fence_regs(acc);
    if (prev != 0xffffffffu && leader) oz_release<CL>(empty0 + 8 * prev);
#pragma unroll
    for (int t = HI; t >= LO; --t) {
        const double w = __longlong_as_double((long long)(1023 - (12 + 8 * t)) << 52);
#pragma unroll
        for (int j = 0; j < 32; ++j) part[j] = fma(i32_to_f64(acc[32 * (t - LO) + j]), w, (FIRST && t == HI) ? 0.0 : part[j]);
    }
}

// the passes PASS .. oz_passes(S) - 1 of one tile
template <int S, int CL, int PASS>
__device__ __forceinline__ void oz_consume_passes(const OzArgs& p, int kbn, uint32_t base, uint32_t full0, uint32_t empty0, int wg,
                                                  uint32_t& it, double (&part)[32], long long& c_wait) {
    if constexpr (PASS < oz_passes(S)) {
        oz_consume_pass<S, CL, oz_pass_lo(S, PASS), oz_pass_hi(S, PASS), PASS == 0>(p, kbn, base, full0, empty0, wg, it, part, c_wait);
        oz_consume_passes<S, CL, PASS + 1>(p, kbn, base, full0, empty0, wg, it, part, c_wait);
    }
}

// Kernel organisation (persistent, one CTA per SM): 384 threads = two consumer warpgroups (rows 0-63 and 64-127 of the
// 128 x 64 tile; S class accumulators of m64n64 each would not fit the register file, so a tile is several passes over
// k, see oz_pass_hi, each folded into a register-resident fp64 partial sum) + one TMA producer warpgroup, which hands
// its registers to the consumers (setmaxnreg).  A stage is one 32-byte k-block of the pass's digit planes of A (128
// rows) and B (64 rows).
// CL = 2: the two CTAs of a cluster work on column tiles 2 j and 2 j + 1 of the same row block.  They need the same A
// digit planes, so each CTA fetches half of them and TMA multicasts every box into both shared memories.  A stage may be
// refilled only when BOTH CTAs have consumed it: the `empty` barriers count the arrivals of both CTAs' warpgroups.
template <int S, int CL>
__global__ void __launch_bounds__(OZ_THREADS, 1)
oz_mma_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB, const OzArgs p) {
    const uint32_t crank = CL == 2 ? cluster_ctarank() : 0u;
    const int tile_first = (int)blockIdx.x / CL, tile_step = (int)gridDim.x / CL;
    constexpr int STAGE_BYTES = S * (OZ_A_TILE + OZ_B_TILE);
    constexpr int OZ_STAGES = oz_stages_for(S);
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = (uint32_t)__cvta_generic_to_shared(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    const uint32_t bars = base + OZ_STAGES * STAGE_BYTES;  // full[OZ_STAGES], empty[OZ_STAGES]
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const uint32_t full0 = bars, empty0 = bars + 8 * OZ_STAGES;

    if (tid == 0) {
        for (int s = 0; s < OZ_STAGES; ++s) {
            mbar_init(full0 + 8 * s, 1);
            mbar_init(empty0 + 8 * s, 2 * CL);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (CL == 2) cluster_sync_all();   // the peer's barriers exist before anything is multicast or arrived at them

    if (warp >= 8) {
        // ------------------------------------------------------------ TMA producer; its registers go to the consumers
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
        if (warp == 8 && lane == 0) {
            uint32_t it = 0;
            long long m_empty = 0;
            const long long m_t0 = clock64();
            for (int tile = tile_first; tile < p.num_tiles; tile += tile_step) {
                const int2 tt = p.tile_list[tile];
                const int row0 = tt.x * OZ_BM, col0 = (CL * tt.y + (int)crank) * OZ_BN;
                const int kbn = oz_kb_count(p, CL, tt.y);
                for (int pass = 0; pass < oz_passes(S); ++pass) {
                    const int np = oz_pass_hi(S, pass) + 1;   // digit planes 0 .. hi
                    for (int kb = 0; kb < kbn; ++kb, ++it) {
                        const uint32_t s = it % OZ_STAGES, ph = (it / OZ_STAGES) & 1u;
                        const long long e0 = p.prof ? clock64() : 0;
                        mbar_wait(empty0 + 8 * s, ph ^ 1u);
                        if (p.prof) m_empty += clock64() - e0;
                        mbar_expect_tx(full0 + 8 * s, np * (OZ_A_TILE + OZ_B_TILE));   // bytes landing in THIS CTA's stage
                        const uint32_t st = base + s * STAGE_BYTES;
                        for (int q = 0; q < np; ++q) {
                            if (CL == 1)
                                tma_load_2d(st + q * OZ_A_TILE, &mapA, kb * OZ_KB, q * p.rowsA_pad + row0, full0 + 8 * s);
                            else if ((q < (np + 1) / 2) == (crank == 0))
                                tma_load_2d_mc(st + q * OZ_A_TILE, &mapA, kb * OZ_KB, q * p.rowsA_pad + row0, full0 + 8 * s, (uint16_t)3);
                            tma_load_2d(st + S * OZ_A_TILE + q * OZ_B_TILE, &mapB, kb * OZ_KB, q * p.rowsB_pad + col0, full0 + 8 * s);
                        }
                    }
                }
            }
            if (p.prof) {
                p.prof[8 * blockIdx.x + 5] = m_empty;              // producer: waiting for consumers to free a stage
                p.prof[8 * blockIdx.x + 6] = clock64() - m_t0;     // ... whole loop
            }
        }
    } else {
        // ------------------------------------------------------------ consumers: warpgroup wg owns rows 64 wg .. 64 wg + 63
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");
        const int wg = warp >> 2;
        uint32_t it = 0, tcount = 0;
        long long c_wait = 0, c_upd = 0;
        for (int tile = tile_first; tile < p.num_tiles; tile += tile_step, ++tcount) {
            const int2 tt = p.tile_list[tile];
            const int ti = tt.x, tj = CL * tt.y + (int)crank;
            const int kbn = oz_kb_count(p, CL, tt.y);
            double part[32];
            // rows of this thread in the accumulator layout: r0 and r0 + 8; columns 8 c + 2 (lane % 4) + {0, 1}, c = 0..7
            const int r0 = ti * OZ_BM + 64 * wg + 16 * (warp & 3) + (lane >> 2);
            const int c0 = tj * OZ_BN + 2 * (lane & 3);
            // pull this thread's part of the C tile towards L2 while the passes run
            if (p.debug == 0 && !p.overwrite && (lane & 3) == 0) {
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int c16 = 0; c16 < 4; ++c16) {
                        const int gr = r0 + 8 * h, gc = tj * OZ_BN + 16 * c16;
                        if (gr < p.m && gc < p.n && !(p.lower_only && gc > gr)) prefetch_l2(p.C + (int64_t)gr * p.ldc + gc);
                    }
            }
            oz_consume_passes<S, CL, 0>(p, kbn, base, full0, empty0, wg, it, part, c_wait);
            const long long t1 = clock64();
            if (p.debug == 0) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int gr = r0 + 8 * h;
                    if (gr >= p.m) continue;
                    const double sav = p.sa[gr] * p.alpha;
#pragma unroll
                    for (int c = 0; c < 8; ++c)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int gc = c0 + 8 * c + e;
                            if (gc < p.n && !(p.lower_only && gc > gr)) {
                                double* cp = p.C + (int64_t)gr * p.ldc + gc;
                                const double old = p.overwrite ? 0.0 : *cp;
                                *cp = fma(sav * p.sb[gc], part[4 * c + 2 * h + e], old);
                            }
                        }
                }
            }
            c_upd += clock64() - t1;
        }
        if (p.prof && tid == 0) {
            p.prof[8 * blockIdx.x + 0] = c_wait;   // consumers: waiting for TMA data
            p.prof[8 * blockIdx.x + 1] = c_upd;    // epilogue (C update)
            p.prof[8 * blockIdx.x + 3] = tcount;
        }
    }
    __syncthreads();
    if (CL == 2) cluster_sync_all();   // no arrival of mine may still be on its way to a peer that has exited
}

// ---------------------------------------------------------------------------------------------- peak probe
// The int8 tensor-pipe ceiling, measured instead of assumed: every CTA (one per SM, two warpgroups) issues `iters`
// back-to-back wgmma m64n256k32 s8 per warpgroup on operands that stay in shared memory (no TMA, no epilogue).
// ops = 2 * 64 * 256 * 32 per instruction.  What oz_mma_kernel can reach at most; its roofline denominator in bench.py.
constexpr int OZ_PEAK_THREADS = 256;
__global__ void __launch_bounds__(OZ_PEAK_THREADS, 1) oz_i8_peak_kernel(int iters, int* sink) {
    extern __shared__ uint8_t pk_raw[];
    const uint32_t raw = (uint32_t)__cvta_generic_to_shared(pk_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    uint8_t* gen = pk_raw + (base - raw);
    for (int i = threadIdx.x; i < (4096 + 8192) / 4; i += blockDim.x) reinterpret_cast<uint32_t*>(gen)[i] = 0x01010101u * (uint32_t)(i & 3);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes of the operands -> async proxy (MMA)
    __syncthreads();
    const int wg = threadIdx.x >> 7;
    const uint64_t ad = oz_smem_desc(base + 2048u * wg), bd = oz_smem_desc(base + 4096);
    int acc[128];
#pragma unroll
    for (int j = 0; j < 128; ++j) acc[j] = 0;
    for (int i = 0; i < iters; ++i) {
        wg_fence();
        wg_mma_i8<4>(acc, ad, bd);
        wg_commit();
        wg_wait<1>();
    }
    wg_wait<0>();
    wg_fence_regs(acc);
    if (sink && acc[0] == 0x7fffffff) sink[0] = acc[1];   // keeps the accumulators observable
}

// ---------------------------------------------------------------------------------------------- host side
static bool make_tmap_u8(CUtensorMap* map, const int8_t* base, int64_t rows_total, int64_t kpad, int box_rows) {
    PFN_tmapEncodeTiled enc = tmap_encoder();
    if (!enc) return false;
    cuuint64_t gdim[2] = {(cuuint64_t)kpad, (cuuint64_t)rows_total};
    cuuint64_t gstride[1] = {(cuuint64_t)kpad};
    cuuint32_t box[2] = {(cuuint32_t)OZ_KB, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    return enc(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, (void*)base, gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_32B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// C[m,n] += alpha * A[m,k] B[n,k]^T  (lower_only: j <= i, A == B allowed) through the int8 tensor cores
// Modes (OzMode): overwrite -- C = alpha A B^T, C not read (it may alias A's fp64 storage: the operands are copied to digit
// planes first); transB -- B is given transposed (element (j, kk) at B[kk * ldb + j]); ktri -- B is lower triangular.
// lower_only with m > n is the "trapezoid" of a factorisation with right-hand-side rows riding below the matrix: rows
// < n update j <= i only, the rows below update all n columns.
struct OzMode {
    bool overwrite = false, transB = false, ktri = false;
};
// One sliced operand: S digit planes [S][rows_pad][kpad] + the row scales.
struct OzOperand {
    const int8_t* planes = nullptr;
    const double* scale = nullptr;
    int64_t rows_pad = 0;
};

// slice `rows` rows of length k (source row r at src + rowmap128[r / 128] * ld + (r % 128) * ld when a row map is given -- a
// device array with one source row index per group of 128 rows, for operands gathered from block-cyclic storage --
// else at src + r * ld) into `planes` / `scale` (capacity checked by the caller)
template <int S>
static int oz_slice_launch(b2gp_ctx* ctx, cudaStream_t st, const double* src, int64_t ld, int64_t rows, int64_t k, DevBuf& planes,
                           DevBuf& scale, bool trans, const int64_t* rowmap128, OzOperand* out) {
    const int64_t kpad = round_up(k, OZ_KB), rp = round_up(rows, 128);
    RET_IF(ensure(ctx, planes, (size_t)S * rp * kpad));
    RET_IF(ensure(ctx, scale, (size_t)rp * 8));
    RET_IF(launch(ctx, PATH_OZ_SLICE, st, (unsigned)rp, 256, 0, oz_slice_kernel<S>, src, ld, (int)rows, (int)k, (int8_t*)planes.p, (int)rp,
                  (int)kpad, (double*)scale.p, trans ? 1 : 0, rowmap128));
    out->planes = (const int8_t*)planes.p;
    out->scale = (const double*)scale.p;
    out->rows_pad = rp;
    return B2GP_OK;
}

// the band-ordered tile list of an m x n (lower-only / trapezoid) product, cached per shape in `w`
static int oz_default_list(b2gp_ctx* ctx, cudaStream_t st, OzWork& w, int tiles_m, int tiles_n, bool lower_only, int CL,
                           const int2** list, int64_t* count) {
    // Tile order.  One round of the persistent loop runs sm_count consecutive list entries concurrently and, tiles
    // being equally long, in k-lockstep: if those tiles form a compact block of (row block, column block) pairs, each
    // operand block is fetched from HBM once per round and served to the other tiles from L2.  Bands of G row blocks,
    // column-major inside a band: a round covers ~G x (sm_count/G) tiles = G + sm_count/G distinct operand blocks.
    const int pairs_n = (tiles_n + CL - 1) / CL;   // list entries per row block: column tiles (CL = 1) or pairs of them
    OzTileList* tl = nullptr;
    for (auto& l : w.lists)
        if (l.tm == tiles_m && l.tn == tiles_n && l.lower == (lower_only ? 1 : 0) && l.cl == CL) tl = &l;
    if (!tl) {
        // one factorisation cycles through ~2 N / panel distinct shapes; they repeat from draw to draw
        tl = &w.lists[w.next_list];
        w.next_list = (w.next_list + 1) % OZ_LISTS;
        tl->host.clear();
        const int G = 8;
        for (int b0 = 0; b0 < tiles_m; b0 += G) {
            const int b1 = b0 + G < tiles_m ? b0 + G : tiles_m;
            // lower: row block ti owns column tiles 0 .. 2 ti + 1, i.e. pairs 0 .. ti
            const int last = lower_only ? (CL == 2 ? b1 - 1 : 2 * (b1 - 1) + 1) : pairs_n - 1;
            const int jmax = last < pairs_n - 1 ? last : pairs_n - 1;
            for (int tj = 0; tj <= jmax; ++tj)
                for (int ti = b0; ti < b1; ++ti)
                    if (!lower_only || tj <= (CL == 2 ? ti : 2 * ti + 1)) tl->host.push_back(make_int2(ti, tj));
        }
        tl->tm = tiles_m;
        tl->tn = tiles_n;
        tl->lower = lower_only ? 1 : 0;
        tl->cl = CL;
        tl->count = (int64_t)tl->host.size();
        // a list may still be in use by a kernel queued earlier on this stream: the copy is stream-ordered behind it
        RET_IF(ensure(ctx, tl->dev, tl->host.size() * sizeof(int2)));
        CUDA_TRY(ctx, cudaMemcpyAsync(tl->dev.p, tl->host.data(), tl->host.size() * sizeof(int2), cudaMemcpyHostToDevice, st));
    }
    *list = (const int2*)tl->dev.p;
    *count = tl->count;
    return B2GP_OK;
}

// C[m,n] (+)= alpha A B^T from sliced operands.  `list` (device, `count` entries of (row tile, column pair / tile)) overrides
// the default tile order: the distributed factorisation passes the staircase of a block-cyclic trailing matrix.
template <int S>
static int oz_mma_launch(b2gp_ctx* ctx, cudaStream_t st, OzWork& w, const OzOperand& oa, const OzOperand& ob, int64_t m, int64_t n,
                         int64_t k, double alpha, double* C, int64_t ldc, bool lower_only, OzMode mode, const int2* list, int64_t count) {
    const int64_t kpad = round_up(k, OZ_KB);
    CUtensorMap mapA, mapB;
    if (!make_tmap_u8(&mapA, oa.planes, (int64_t)S * oa.rows_pad, kpad, OZ_BM) || !make_tmap_u8(&mapB, ob.planes, (int64_t)S * ob.rows_pad, kpad, OZ_BN))
        return B2GP_ERR_UNSUPPORTED;
    OzArgs a;
    a.m = (int)m;
    a.n = (int)n;
    a.kb_count = (int)(kpad / OZ_KB);
    a.rowsA_pad = (int)oa.rows_pad;
    a.rowsB_pad = (int)ob.rows_pad;
    a.sa = oa.scale;
    a.sb = ob.scale;
    a.C = C;
    a.ldc = ldc;
    a.alpha = alpha;
    a.lower_only = lower_only ? 1 : 0;
    a.overwrite = mode.overwrite ? 1 : 0;
    a.ktri = mode.ktri ? 1 : 0;
    a.tiles_m = (int)ceil_div(m, OZ_BM);
    a.tiles_n = (int)ceil_div(n, OZ_BN);
    const int CL = (ctx->oz_cluster == 2) ? 2 : 1;
    if (!list) RET_IF(oz_default_list(ctx, st, w, a.tiles_m, a.tiles_n, lower_only, CL, &list, &count));
    if (count <= 0) return B2GP_OK;
    const int64_t tiles = count;
    a.num_tiles = (int)tiles;
    a.tile_list = list;
    a.prof = nullptr;
    if (w.prof.p) a.prof = (long long*)w.prof.p;
    a.debug = ctx->oz_debug;
    constexpr int smem_bytes = oz_stages_for(S) * S * (OZ_A_TILE + OZ_B_TILE) + 16 * oz_stages_for(S) + 1024;
    static_assert(smem_bytes <= 227 * 1024, "sm_90 opt-in shared memory per block");
    static PerDeviceOnce attr;
    if (attr.need(ctx->device)) {
        CUDA_TRY(ctx, cudaFuncSetAttribute(oz_mma_kernel<S, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
        CUDA_TRY(ctx, cudaFuncSetAttribute(oz_mma_kernel<S, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
        attr.done(ctx->device);
    }
    const int nsm = persist_sms(ctx);
    if (CL == 2) {
        const int ncl = nsm / 2;
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3((unsigned)(2 * (tiles < ncl ? tiles : ncl)));
        cfg.blockDim = dim3(OZ_THREADS);
        cfg.dynamicSmemBytes = smem_bytes;
        cfg.stream = st;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeClusterDimension;
        at[0].val.clusterDim.x = 2;
        at[0].val.clusterDim.y = 1;
        at[0].val.clusterDim.z = 1;
        cfg.attrs = at;
        cfg.numAttrs = 1;
        CUDA_TRY(ctx, cudaLaunchKernelEx(&cfg, oz_mma_kernel<S, 2>, mapA, mapB, a));
        return count_launch(ctx, PATH_OZ_MMA);
    }
    const int grid = (int)(tiles < nsm ? tiles : nsm);
    return launch(ctx, PATH_OZ_MMA, st, grid, OZ_THREADS, smem_bytes, oz_mma_kernel<S, 1>, mapA, mapB, a);
}

template <int S>
static int ozaki_gemm_nt(b2gp_ctx* ctx, cudaStream_t st, OzWork& w, int64_t m, int64_t n, int64_t k, double alpha, const double* A,
                         int64_t lda, const double* B, int64_t ldb, double* C, int64_t ldc, bool lower_only, OzMode mode = OzMode()) {
    if (m <= 0 || n <= 0 || k <= 0) return B2GP_OK;
    if (k > OZ_K_MAX) return B2GP_ERR_UNSUPPORTED;  // int32 accumulation bound (the dispatcher splits longer k)
    const bool same = (A == B && lda == ldb && n <= m && !mode.transB);   // B's rows are the first n rows of A: one set of planes
    OzOperand oa, ob;
    RET_IF(oz_slice_launch<S>(ctx, st, A, lda, m, k, w.planesA, w.scaleA, false, nullptr, &oa));
    if (same)
        ob = oa;
    else
        RET_IF(oz_slice_launch<S>(ctx, st, B, ldb, n, k, w.planesB, w.scaleB, mode.transB, nullptr, &ob));
    return oz_mma_launch<S>(ctx, st, w, oa, ob, m, n, k, alpha, C, ldc, lower_only, mode, nullptr, 0);
}

static int ozaki_dispatch(b2gp_ctx* ctx, cudaStream_t st, int64_t m, int64_t n, int64_t k, double alpha, const double* A, int64_t lda,
                          const double* B, int64_t ldb, double* C, int64_t ldc, bool lower_only, bool overwrite, bool transB, bool ktri) {
    Slot* sl = slot_of(ctx, st);
    OzWork* w = sl ? &sl->oz : &ctx->slots[0].oz;
    const int planes = oz_planes_for(ctx, st);
    for (int64_t k0 = 0; k0 < k; k0 += OZ_K_MAX) {
        const int64_t kc = k - k0 < OZ_K_MAX ? k - k0 : OZ_K_MAX;
        OzMode mode;
        mode.overwrite = overwrite && k0 == 0;      // later k-chunks accumulate onto the first
        mode.transB = transB;
        mode.ktri = ktri && k <= OZ_K_MAX;
        const double* Bk = transB ? B + k0 * ldb : B + k0;
        int rc;
        if (planes == 6)
            rc = ozaki_gemm_nt<6>(ctx, st, *w, m, n, kc, alpha, A + k0, lda, Bk, ldb, C, ldc, lower_only, mode);
        else
            rc = ozaki_gemm_nt<7>(ctx, st, *w, m, n, kc, alpha, A + k0, lda, Bk, ldb, C, ldc, lower_only, mode);
        if (rc != B2GP_OK) return rc;
    }
    return B2GP_OK;
}
