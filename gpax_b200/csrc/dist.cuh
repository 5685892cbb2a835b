// dist.cuh -- the multi-GPU forms of the path (SURVEY.md section 8e), inside the library: one process per GPU, NCCL over
// NVLink 5 / NVSwitch for the exchange steps, no torch / Python on the data path.
//
//   b2gp_dist_posterior          exact-GP posterior with k_XX distributed 2-D block-cyclically over a pr x pc process grid
//                                (config 4: N = 32768 on 8 GPUs as 2 x 4).  Replaces gpax/models/gp.py:253-277 at sizes
//                                where one GPU's 2 N^2 bytes or N^3/3 flops are too much.
//   b2gp_dist_sparse_posterior   N-sharded Nystrom / VFE posterior (config 5: N = 262144, M = 4096 on 4 GPUs): per-rank
//                                statistics of a shard, one all-reduce of the M x M matrix (gpax/models/sparse_gp.py:193-204).
//
// Layout of the block-cyclic factorisation.  Tiles are nb x nb.  Tile rows gi = 0 .. T-1 are k_XX, gi = T .. T+R-1 are
// the right-hand-side rows [k_pX; y^T] (the solve rides under the factorisation exactly as in potrf_tall); tile columns
// gj = 0 .. T-1.  Tile (gi, gj) lives on process (gi mod pr, gj mod pc) at local tile (gi / pr, gj / pc) of ONE row-major
// local matrix, so every local operation below is a plain strided GEMM.  Nothing is ever redistributed: the local
// matrix is generated in place from X by the Gram kernel.
//
// Right-looking step k (diagonal tile on process (k mod pr, k mod pc)):
//   (a) owner factors the nb x nb diagonal tile (fp64 leaves) and forms U = L_kk^{-T};
//   (b) U is broadcast down the owner's process COLUMN (column communicator);
//   (c) every process of that column solves its local rows of the panel, rows <- rows U: one int8 wgmma GEMM
//       (k = nb, overwrite, B transposed and k-triangular) -- the panel solve is spread over the pr processes;
//   (d) the solved rows are packed into this process row's slot of the panel buffer;
//   (e) each slot is broadcast along its process ROW (row communicator, root = column k mod pc), then
//   (f) all-gathered down every process COLUMN (column communicator): every process now holds the whole panel;
//   (g) trailing update of the local matrix, C -= P_rows P_cols^T: ONE int8 GEMM whose A operand is this process row's
//       slot, whose B operand gathers the panel tiles of this process's tile columns through a row map, and whose tile
//       list is the staircase gi >= gj of the block-cyclic lower triangle.
// Look-ahead, two kinds.  (i) (g) is split into the tile column of step k+1 (g1) and the rest (g2); the compute stream
// runs g1_k, then (c), (d) of step k+1, then g2_k, so the collectives (e), (f) of step k+1 -- on their own stream --
// overlap the bulk of step k's update.  (ii) Diagonal look-ahead: the tile (k+1, k) is broadcast along its process row
// AHEAD of the panel, right after the panel solve; the owner of diagonal tile k+1 applies it (D -= E E^T), factors the
// tile and forms U on a third stream while the panel of step k is still being exchanged and applied -- the 0.4 ms
// latency chain of the 128-wide leaves leaves the critical path, which becomes panel solve -> early tile -> (factor) ->
// U broadcast -> next panel solve.
#pragma once
#include <dlfcn.h>
#include <nccl.h>

#include <algorithm>

#include "common.cuh"

// ---------------------------------------------------------------------------------------------- NCCL, loaded at run time
// libb200gp.so does not link NCCL: single-GPU users need none, and a process that also runs torch must share torch's copy.
struct NcclApi {
    void* handle = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommSplit)(ncclComm_t, int, int, ncclComm_t*, ncclConfig_t*) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*Broadcast)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
    std::string error;
};

static NcclApi* nccl_api() {
    static NcclApi api;
    static std::once_flag once;
    std::call_once(once, [] {
        const char* env = getenv("B200GP_NCCL_LIB");
        const char* names[] = {env, "libnccl.so.2", "libnccl.so"};
        for (const char* n : names) {
            if (!n || !*n) continue;
            api.handle = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
            if (api.handle) break;
        }
        if (!api.handle) {
            api.error = "cannot load libnccl.so.2 (set B200GP_NCCL_LIB to its path)";
            return;
        }
#define B2GP_NCCL_SYM(field, name)                                                     \
    api.field = reinterpret_cast<decltype(api.field)>(dlsym(api.handle, name));        \
    if (!api.field) api.error = std::string("libnccl lacks ") + name;
        B2GP_NCCL_SYM(GetUniqueId, "ncclGetUniqueId")
        B2GP_NCCL_SYM(CommInitRank, "ncclCommInitRank")
        B2GP_NCCL_SYM(CommSplit, "ncclCommSplit")
        B2GP_NCCL_SYM(CommDestroy, "ncclCommDestroy")
        B2GP_NCCL_SYM(Broadcast, "ncclBroadcast")
        B2GP_NCCL_SYM(AllReduce, "ncclAllReduce")
        B2GP_NCCL_SYM(AllGather, "ncclAllGather")
        B2GP_NCCL_SYM(GroupStart, "ncclGroupStart")
        B2GP_NCCL_SYM(GroupEnd, "ncclGroupEnd")
        B2GP_NCCL_SYM(GetErrorString, "ncclGetErrorString")
#undef B2GP_NCCL_SYM
    });
    return &api;
}

#define NCCL_TRY(ctx, expr)                                                                                   \
    do {                                                                                                      \
        ncclResult_t r_ = (expr);                                                                             \
        if (r_ != ncclSuccess)                                                                                \
            return set_err((ctx), B2GP_ERR_CUDA, #expr, nccl_api()->GetErrorString(r_), __FILE__, __LINE__); \
    } while (0)

// ---------------------------------------------------------------------------------------------- block-cyclic index algebra
// (pure functions: exported through b2gp_dist_layout for the CPU tests)
struct BcGrid {
    int pr = 1, pc = 1, myrow = 0, mycol = 0;
    int64_t nb = 512, T = 0, R = 0;   // tile size, matrix tiles per side, right-hand-side tile rows
    int64_t rows_total() const { return T + R; }
    // local tile rows of process row r / tile columns of process column c
    int64_t lr(int r) const { return rows_total() > r ? (rows_total() - 1 - r) / pr + 1 : 0; }
    int64_t lc(int c) const { return T > c ? (T - 1 - c) / pc + 1 : 0; }
    // first local tile row of process row r whose global index exceeds k ( = number of its tile rows <= k)
    int64_t first_row_after(int64_t k, int r) const { return k >= r ? (k - r) / pr + 1 : 0; }
    int64_t first_col_after(int64_t k, int c) const { return k >= c ? (k - c) / pc + 1 : 0; }
    // rows of the panel of step k held by process row r, and the (uniform) slot size of the panel buffer
    int64_t panel_rows(int64_t k, int r) const { return (lr(r) - first_row_after(k, r)) * nb; }
    int64_t slot_rows(int64_t k) const {
        int64_t m = 0;
        for (int r = 0; r < pr; ++r) m = std::max(m, panel_rows(k, r));
        return m;
    }
};

// ---------------------------------------------------------------------------------------------- state
struct DistStep {             // per step k: staircase tile lists and the row map of the B operand (cached per problem shape)
    DevBuf g1, g2, bmap;
    int64_t n1 = 0, n2 = 0;
};
struct DistState {
    bool ready = false;
    int rank = 0, nranks = 1;
    BcGrid g;
    ncclComm_t world = nullptr, rowc = nullptr, colc = nullptr;
    cudaStream_t ms = nullptr, dq = nullptr;     // communication stream, diagonal-tile stream
    cudaEvent_t ev_u = nullptr, ev_ubc[2] = {nullptr, nullptr}, ev_chunk = nullptr, ev_comm[2] = {nullptr, nullptr}, ev_done = nullptr;
    cudaEvent_t ev_e = nullptr, ev_early[2] = {nullptr, nullptr}, ev_g2 = nullptr;
    DevBuf Aloc, PB[2], UB, EB, Xrows, Zcols, yloc, red, linv, updA, updB, updSA, updSB, wseg;
    std::vector<DistStep> steps;
    int64_t cache_T = -1, cache_R = -1, cache_nb = -1;
    int cache_cl = -1;
    double last_potrf_ms = 0.0, last_total_ms = 0.0;
    // the owner synchronises the device first; the buffers free themselves
    ~DistState() {
        for (cudaEvent_t e : {ev_u, ev_ubc[0], ev_ubc[1], ev_chunk, ev_comm[0], ev_comm[1], ev_done, ev_e, ev_early[0], ev_early[1], ev_g2})
            if (e) cudaEventDestroy(e);
        if (ms) cudaStreamDestroy(ms);
        if (dq) cudaStreamDestroy(dq);
        NcclApi* n = nccl_api();
        if (n->handle) {
            if (rowc) n->CommDestroy(rowc);
            if (colc) n->CommDestroy(colc);
            if (world) n->CommDestroy(world);
        }
    }
};

// diagonal term of k_XX on the diagonal tiles this process owns (gi = gi0 + t * step, t < count): K[i, i] += noise + jitter
__global__ void dist_diag_kernel(double* A, int64_t ld, int64_t nb, int pr, int pc, int64_t gi0, int64_t step, int64_t count,
                                 const double* __restrict__ theta, int d, double jitter) {
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= count * nb) return;
    const int64_t gi = gi0 + (idx / nb) * step, r = idx % nb;
    A[((gi / pr) * nb + r) * ld + (gi / pc) * nb + r] += theta[d + 1] + jitter;
}

// var[p] = k(x, x) + noise_p + jitter - nrm[p]; mean / var <- NaN when the factorisation failed
__global__ void dist_finish_kernel(double* mean, double* var, const double* nrm, int64_t P, int kind, int d, const double* theta,
                                   double noise_mult, double jitter, const int* info) {
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P) return;
    const bool bad = *info != 0;
    const double nan = __longlong_as_double(0x7ff8000000000000LL);
    if (var) var[p] = bad ? nan : (cov_self(kind, theta[d]) + (theta[d + 1] * noise_mult + jitter)) - nrm[p];
    if (bad) mean[p] = nan;
}
