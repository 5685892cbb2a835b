// common.cuh -- context, error handling, device buffers, kernel launches for libb200gp.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <atomic>

#include <cstdint>
#include <cstdio>
#include <cstring>
#include <memory>
#include <mutex>
#include <string>
#include <utility>
#include <vector>

#include "../../include/b200gp.h"

#define B2GP_MAX_STREAMS 16
#define B2GP_LEAF 128  // diagonal-block size of the factorisation (one CTA, shared memory)
#define B2GP_DRAW_BATCH_DEFAULT 4  // draws per lock-step group of a multi-draw posterior on the fp64 tall route (DESIGN.md 4.2)

// SM count of the largest device a context has been created on (grid_for's cap)
inline std::atomic<int> g_grid_sms{1};

// A device allocation that frees itself; ensure() grows it.  Move-only: one owner per pointer.
struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(DevBuf&& o) noexcept : p(o.p), cap(o.cap) {
        o.p = nullptr;
        o.cap = 0;
    }
    DevBuf& operator=(DevBuf&& o) noexcept {
        if (this != &o) {
            if (p) cudaFree(p);
            p = o.p;
            cap = o.cap;
            o.p = nullptr;
            o.cap = 0;
        }
        return *this;
    }
    ~DevBuf() {
        if (p) cudaFree(p);
    }
};

// Timing events handed out per call (per-stage timings, profiles), reused from call to call.
struct EventPool {
    std::vector<cudaEvent_t> ev;
    size_t next = 0;
    cudaEvent_t get() {
        if (next == ev.size()) {
            cudaEvent_t e;
            if (cudaEventCreate(&e) != cudaSuccess) return nullptr;
            ev.push_back(e);
        }
        return ev[next++];
    }
    void reset() { next = 0; }
    void destroy() {
        for (auto e : ev) cudaEventDestroy(e);
        ev.clear();
        next = 0;
    }
};

struct DistState;  // multi-GPU state (dist.cuh)

#define OZ_LISTS 192
// scratch of the int8-split (Ozaki) GEMM path, one per stream: digit planes, row scales, tile list
struct OzTileList {
    int tm = -1, tn = -1, lower = -1, cl = -1;
    int64_t count = 0;
    DevBuf dev;
    std::vector<int2> host;         // kept alive for the asynchronous upload
};
struct OzWork {
    DevBuf planesA, planesB, scaleA, scaleB, prof;
    OzTileList lists[OZ_LISTS];     // the (tiles_m, tiles_n, lower) shapes one factorisation cycles through
    int next_list = 0;
};

// One "slot" = the workspace of one posterior draw in flight.
struct Slot {
    cudaStream_t stream = nullptr;
    // k_XX / its factor L and the inverted diagonal blocks of L live in b2gp_ctx::post (posterior draw regions;
    // slot0_buffers for the single-slot entry points)
    DevBuf Vt;     // N-row scratch: host Gram staging (b2gp_posterior_gram), W^T (sparse paths), K^{-1} (likelihoods)
    DevBuf cov;    // P x ldC      posterior covariance / its factor
    DevBuf LinvC;  // inverted diagonal blocks of chol(cov)
    DevBuf misc;   // small scratch
    DevBuf panelU; // panel x panel scratch of the tall-panel factorisation: L_jj^{-T} of the current diagonal block
    OzWork oz;
    int oz_planes = 7;  // digit planes of the int8 path for the work queued on this slot when ctx->ozaki == -1 (auto)
    cudaEvent_t ev[8];
};

// Cumulative per-context counters of the kernels launched and the solver routes entered, in the order
// b2gp_debug_path_counts reports them.  The kernel counters are kept by launch() / count_launch(), the route counters by
// count_path() at the entry of the route.  They steer nothing: tests read them to prove which path a call took.
enum PathCounter {
    PATH_GEMM_NT = 0,   // gemm_nt_kernel launches (cp.async + DMMA), the 64x64 tail launch of the TMA kernel included
    PATH_GEMM_TMA,      // gemm_tma_kernel launches (persistent TMA + DMMA)
    PATH_OZ_MMA,        // oz_mma_kernel launches (int8 wgmma)
    PATH_OZ_SLICE,      // oz_slice_kernel launches (digit planes of one operand)
    PATH_TRSM_STRIP,    // trsm_strip_kernel launches
    PATH_POTRF_DIAG,    // potrf_diag_kernel launches (128-wide leaves)
    PATH_PANEL_SOLVE,   // panel_solve_all_rows calls
    PATH_TRSM_TALL,     // trsm_tall calls
    PATH_POTRF_TALL,    // factorisations that took potrf_tall on the int8 route (top-level entries, not its recursion)
    PATH_POTRF_TALL_FP64,  // factorisations that took potrf_tall on the fp64 DMMA route (ozaki = 0), top-level entries
    PATH_MLL_NNGP_GRAD,    // likelihood gradients that took the NNGP route (mll_nngp_grad_kernel, nngp.cuh), one per call
    PATH_MLL_GRAM_TRACE,   // likelihood gradients reduced against caller-supplied dK (mll_gram_trace_kernel), one per call
    PATH_MLL_BATCH_SMALL,  // b2gp_mll_batch calls that took the one-launch small route (mll_batch_small_kernel), one per call
    PATH_POTRF_TALL_BATCH, // lock-step groups of posterior draws factored by one batched potrf_tall (fp64 route), one per group
    PATH_MLL_DRAWS_BATCH,  // groups of likelihood draws b2gp_mll_draws ran in lock-step, one per group
    PATH_SPARSE_GRAM_TRACE,  // VFE-bound gradients reduced against caller-supplied blocks (sparse_gram_trace_kernel), one per call
    PATH_COUNT
};

struct b2gp_ctx {
    int device = 0;
    int sm_count = 0;
    int cc_major = 0, cc_minor = 0;
    size_t mem_bytes = 0;
    int n_streams = 2;
    int use_tma = 1;  // large GEMMs through the TMA / mbarrier persistent kernel (gemm_tma.cuh)
    int enqueue_threads = 1;  // queue the draws of a multi-draw posterior from one host thread per slot
    int big_grid = 0;        // CTAs of the persistent kernels (0 = one per SM); fewer leaves SMs for other streams' small kernels
    int oz_min_tiles = 0;  // smallest 128x64-tile count handed to the int8 path (set to the SM count at creation)
    int trsm_strip = 256;  // widest factor solved by the one-launch strip kernel (0: recurse down to the 128 leaves)
    int oz_cluster = 2;  // 2: CTA pairs (a cluster of 2) share the A digit planes by TMA multicast; 1: independent CTAs
    int panel = 1024;      // diagonal-block width of the tall-panel factorisation (potrf_tall); 0: recursive potrf_rec / trsm_rec only
    int tall_min = 2048;   // smallest N factored by potrf_tall on the int8 route
    int tall_min_fp64 = 8192;  // smallest N factored by potrf_tall on the fp64 route (ozaki = 0); DESIGN.md 4.2
    int oz_debug = 0;  // see OzArgs::debug (0 in production)
    int bnn_fused = 1;     // 1: BNN entry points take the fused kernels where the network fits (bnn.cuh); 0: layered route
    // draws of a multi-draw posterior factored in lock-step by one batched potrf_tall (fp64 tall route): 0 picks the
    // group size from the route (DESIGN.md 4.2), 1 factors every draw on its own, B >= 2 groups of B
    int draw_batch = 0;
    size_t smem_optin = 0; // opt-in dynamic shared memory per block of the device
    // 0: fp64 DMMA only; 6 / 7: large rank-k updates through the int8 wgmma path with that many base-256 digit planes
    // (46 / 54 bits per operand); -1: 6 or 7 per factorisation from a bound on cond(K), see oz_auto_planes().
    // Default 0: on H100 the int8 path is slower than DMMA (DESIGN.md section 5).
    int ozaki = 0;
    Slot slots[B2GP_MAX_STREAMS];
    cudaEvent_t ev_begin = nullptr, ev_end = nullptr, ev_a = nullptr, ev_b = nullptr;
    // staging for host-pointer entry points
    DevBuf d_in[8];
    DevBuf d_out[4];
    DevBuf d_info;
    DevBuf theta1;     // one-draw theta for b2gp_gram
    DevBuf potrf_buf;  // staging for host-pointer b2gp_potrf / trsm / gemm
    DevBuf gemm_buf[3];
    DevBuf eb[12];     // scratch of b2gp_sparse_elbo; [10], [11] stage the caller's blocks of the *_gram sparse entry points
    DevBuf f32_in[8];  // fp32 staging of the inputs / outputs of calls made with B2GP_FLAG_F32
    DevBuf f32_out[4];
    DevBuf mlp[4];     // b2gp_mlp_forward / b2gp_dkl_mll: staged X and yres | weights | activations | backward scratch
    std::vector<void*> user_allocs;  // b2gp_dev_alloc
    // factor bookkeeping for b2gp_trsm_lower (host-pointer mode keeps the factor resident)
    DevBuf last_linv;
    int64_t last_n = 0;
    // factor cache of slot 0 (host-pointer, single-draw calls): predict_in_batches / viGP chunk loops call the
    // posterior repeatedly with the same training set and theta; the reference re-inverts k_XX every time
    // (gp.py:319-322 -> gp.py:269-271), here the factor L and its inverted diagonal blocks are kept.
    struct {
        bool valid = false;
        int kind = -1, d = 0;
        int64_t N = 0;
        double jitter = 0.0;
        std::vector<double> theta;
        std::vector<char> X;   // raw bytes of the caller's training inputs (fp64 or fp32)
        int info = 0;
        int64_t U_nb = 0;      // > 0: `Ukeep` holds the explicit inverses of the factor's U_nb-wide diagonal blocks (potrf_tall)
    } fcache;
    DevBuf Ukeep;
    // posterior workspaces of the slots, one allocation: draw region q = [Linv | A (k_XX, then the rows under it) | panel
    // scratch] at q * stride doubles, so that a group of consecutive regions is one batch (posterior_impl); its front is
    // also slot 0's matrix for the other entry points (slot0_buffers)
    DevBuf post;
    int64_t cache_hits = 0;
    std::unique_ptr<DistState> dist;   // created by b2gp_dist_init, released by b2gp_dist_finalize or with the context
    b2gp_timing last{};                // what b2gp_last_timing reports
    EventPool pool;
    cudaEvent_t slot_done[B2GP_MAX_STREAMS] = {};
    cudaEvent_t inputs_ready = nullptr;
    std::atomic<int64_t> launches{0};  // kernels queued (draws may be queued from several host threads)
    std::atomic<int64_t> path[PATH_COUNT] = {};  // which kernels / routes the work took (b2gp_debug_path_counts)
    std::string err;
};

static inline void count_path(b2gp_ctx* ctx, int which) { ctx->path[which].fetch_add(1, std::memory_order_relaxed); }

static inline int set_err(b2gp_ctx* ctx, int code, const char* what, const char* detail, const char* file, int line) {
    char buf[512];
    snprintf(buf, sizeof buf, "%s: %s (%s:%d)", what, detail ? detail : "", file, line);
    if (ctx) {
        static std::mutex mu;  // draws of one call may be queued (and fail) on several host threads
        std::lock_guard<std::mutex> lock(mu);
        ctx->err = buf;
    }
    return code;
}

#define CUDA_TRY(ctx, expr)                                                                        \
    do {                                                                                           \
        cudaError_t e_ = (expr);                                                                   \
        if (e_ != cudaSuccess)                                                                     \
            return set_err((ctx), B2GP_ERR_CUDA, #expr, cudaGetErrorString(e_), __FILE__, __LINE__); \
    } while (0)

#define ARG_CHECK(ctx, cond)                                                                       \
    do {                                                                                           \
        if (!(cond)) return set_err((ctx), B2GP_ERR_ARG, "bad argument", #cond, __FILE__, __LINE__); \
    } while (0)

#define RET_IF(expr)                \
    do {                            \
        int r_ = (expr);            \
        if (r_ != B2GP_OK) return r_; \
    } while (0)

// Every kernel of the library is launched through launch() (or, for a cluster launch, by cudaLaunchKernelEx followed
// by count_launch()): the launch is checked where it is made, counted in ctx->launches (b2gp_timing::launches is the
// difference over a call) and, when `path` names a kernel counter, in ctx->path.
static inline int count_launch(b2gp_ctx* ctx, int path = -1) {
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_err(ctx, B2GP_ERR_CUDA, "kernel launch", cudaGetErrorString(e), __FILE__, __LINE__);
    ctx->launches++;
    if (path >= 0) count_path(ctx, path);
    return B2GP_OK;
}

template <typename... P, typename... A>
static int launch(b2gp_ctx* ctx, int path, cudaStream_t st, dim3 grid, dim3 block, size_t smem, void (*k)(P...), A&&... args) {
    k<<<grid, block, smem, st>>>(std::forward<A>(args)...);
    return count_launch(ctx, path);
}

template <typename... P, typename... A>
static int launch(b2gp_ctx* ctx, cudaStream_t st, dim3 grid, dim3 block, size_t smem, void (*k)(P...), A&&... args) {
    return launch(ctx, -1, st, grid, block, smem, k, std::forward<A>(args)...);
}

static inline int ensure(b2gp_ctx* ctx, DevBuf& b, size_t bytes) {
    if (b.cap >= bytes && b.p) return B2GP_OK;
    if (b.p) {
        CUDA_TRY(ctx, cudaFree(b.p));
        b.p = nullptr;
        b.cap = 0;
    }
    // round up so that slowly growing requests do not re-allocate every call
    size_t want = (bytes + ((size_t)1 << 20) - 1) & ~(((size_t)1 << 20) - 1);
    cudaError_t e = cudaMalloc(&b.p, want);
    if (e != cudaSuccess) {
        b.p = nullptr;
        return set_err(ctx, B2GP_ERR_NOMEM, "cudaMalloc", cudaGetErrorString(e), __FILE__, __LINE__);
    }
    b.cap = want;
    return B2GP_OK;
}

// Slot 0's factor matrix (a_bytes) and inverted diagonal blocks (linv_bytes) for the entry points that work on slot 0
// alone (likelihoods, sparse and distributed paths): the front of ctx->post, where the posterior keeps its draw
// regions, so that a fit and a prediction on one context share one allocation.  This overwrites a cached posterior
// factor: the callers drop the factor cache first.
static inline int slot0_buffers(b2gp_ctx* ctx, size_t a_bytes, size_t linv_bytes, double** A, double** Linv) {
    const size_t lb = (linv_bytes + 255) & ~(size_t)255;
    RET_IF(ensure(ctx, ctx->post, lb + a_bytes));
    *Linv = (double*)ctx->post.p;
    *A = (double*)((char*)ctx->post.p + lb);
    return B2GP_OK;
}

// cudaFuncSetAttribute is per device: a process may hold contexts on several devices (Context(device=1) next to
// the default one), so the "already opted in to large dynamic shared memory" memo is a bit per device.
struct PerDeviceOnce {
    std::atomic<uint64_t> mask{0};
    bool need(int dev) const { return ((mask.load(std::memory_order_acquire) >> (dev & 63)) & 1ull) == 0; }
    void done(int dev) { mask.fetch_or(1ull << (dev & 63), std::memory_order_release); }
};

static inline Slot* slot_of(b2gp_ctx* ctx, cudaStream_t st) {
    for (int i = 0; i < B2GP_MAX_STREAMS; ++i)
        if (ctx->slots[i].stream == st) return &ctx->slots[i];
    return nullptr;
}

// digit planes for the int8 GEMMs queued on stream `st`
static inline int oz_planes_for(b2gp_ctx* ctx, cudaStream_t st) {
    if (ctx->ozaki > 0) return ctx->ozaki;
    Slot* sl = slot_of(ctx, st);
    return sl ? sl->oz_planes : 7;
}

// Accuracy-aware plane count (DESIGN.md 4.6): the error the digit-plane GEMMs add to a posterior grows like
// cond(K) * 1.3e-16 with 46-bit operands (6 planes) and cond(K) * 3e-18 with 54-bit ones (7 planes); against the 1e-9
// parity bar 6 planes are safe while cond(K) <= 1e6.  cond(K) is bounded from the trace: lambda_max <= N k_scale +
// sigma^2 + jitter, lambda_min >= sigma^2 + jitter  (K = k(X, X) + (sigma^2 + jitter) I, k(x, x) = k_scale).
static inline int oz_auto_planes(double n, double k_scale, double noise, double jitter) {
    const double floor_ = noise + jitter;
    if (!(floor_ > 0.0) || !(k_scale > 0.0)) return 7;
    return (n * k_scale + floor_) / floor_ <= 1e6 ? 6 : 7;
}

// The draws of a batched launch: `n` draws whose operands (matrix, inverted diagonal blocks, panel scratch) all sit
// `stride` doubles apart; a kernel takes its draw from grid y or z (or its persistent tile index) and offsets every
// pointer by draw * stride.  n = 1 is one draw (stride unused).
struct Batch {
    int n = 1;
    int64_t stride = 0;
};

// CTAs a persistent (one CTA per SM) kernel should launch
static inline int persist_sms(b2gp_ctx* ctx) { return (ctx->big_grid > 0 && ctx->big_grid < ctx->sm_count) ? ctx->big_grid : ctx->sm_count; }

static inline int64_t round_up(int64_t x, int64_t m) { return (x + m - 1) / m * m; }
static inline int64_t ceil_div(int64_t x, int64_t m) { return (x + m - 1) / m; }
