// b200gp.cu -- C-ABI entry points of libb200gp.so (see include/b200gp.h for the contract and the
// reference lines each entry point replaces).  Host code here only orchestrates: workspace, streams,
// the order of kernel launches.  No torch, no JAX, no CPU fallback: every numerical result is
// produced by the sm_90a kernels in gram.cuh / gemm_dmma.cuh / potrf.cuh / posterior.cuh.
#include <algorithm>
#include <chrono>
#include <thread>

#include "common.cuh"
#include "gemm_dmma.cuh"
#include "gemm_tma.cuh"
#include "ozaki.cuh"
#include "gram.cuh"
#include "mll.cuh"
#include "posterior.cuh"
#include "grad.cuh"
#include "mtgp.cuh"
#include "potrf.cuh"
#include "sparse_elbo.cuh"
#include "acq.cuh"
#include "dist.cuh"
#include "dkl.cuh"
#include "nngp.cuh"
#include "bnn.cuh"
#include "mll_batch.cuh"

// ------------------------------------------------------------------------------------------ helpers
static inline bool dev_ptrs(unsigned flags) { return (flags & B2GP_FLAG_DEVICE_PTRS) != 0; }

struct CallTimer {
    b2gp_ctx* ctx;
    int64_t launches0;
    CallTimer(b2gp_ctx* c) : ctx(c), launches0(c->launches) {}
    std::chrono::steady_clock::time_point t_begin;
    int begin(cudaStream_t st) {
        t_begin = std::chrono::steady_clock::now();
        ctx->last = b2gp_timing{};
        ctx->pool.reset();
        CUDA_TRY(ctx, cudaEventRecord(ctx->ev_begin, st));
        return B2GP_OK;
    }
    // host time spent queueing work so far (call before any copy into pageable memory, which blocks the host)
    void mark_enqueued() {
        ctx->last.host_enqueue_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_begin).count();
    }
    int end(cudaStream_t st, b2gp_timing* out) {
        CUDA_TRY(ctx, cudaEventRecord(ctx->ev_end, st));
        if (ctx->last.host_enqueue_ms == 0.0) mark_enqueued();
        CUDA_TRY(ctx, cudaEventSynchronize(ctx->ev_end));
        float ms = 0.f;
        CUDA_TRY(ctx, cudaEventElapsedTime(&ms, ctx->ev_begin, ctx->ev_end));
        ctx->last.total_ms = ms;
        ctx->last.launches = ctx->launches - launches0;
        if (out) *out = ctx->last;
        return B2GP_OK;
    }
};


// ------------------------------------------------------------------------------------------ lifecycle
extern "C" int b2gp_version(void) { return B2GP_VERSION; }

extern "C" int b2gp_ctx_create(int device, b2gp_ctx** out) {
    if (!out) return B2GP_ERR_ARG;
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) return B2GP_ERR_CUDA;
    if (device < 0 || device >= ndev) return B2GP_ERR_ARG;
    if (cudaSetDevice(device) != cudaSuccess) return B2GP_ERR_CUDA;
    b2gp_ctx* ctx = new b2gp_ctx();
    ctx->device = device;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) {
        delete ctx;
        return B2GP_ERR_CUDA;
    }
    ctx->sm_count = prop.multiProcessorCount;
    ctx->oz_min_tiles = ctx->sm_count;
    for (int cur = g_grid_sms.load(); cur < ctx->sm_count && !g_grid_sms.compare_exchange_weak(cur, ctx->sm_count);) {
    }
    ctx->cc_major = prop.major;
    ctx->cc_minor = prop.minor;
    ctx->mem_bytes = prop.totalGlobalMem;
    ctx->smem_optin = prop.sharedMemPerBlockOptin;
    for (int i = 0; i < B2GP_MAX_STREAMS; ++i) {
        if (cudaStreamCreateWithFlags(&ctx->slots[i].stream, cudaStreamNonBlocking) != cudaSuccess) return B2GP_ERR_CUDA;
        for (int e = 0; e < 8; ++e) cudaEventCreate(&ctx->slots[i].ev[e]);
    }
    cudaEventCreate(&ctx->ev_begin);
    cudaEventCreate(&ctx->ev_end);
    cudaEventCreate(&ctx->ev_a);
    cudaEventCreate(&ctx->ev_b);
    for (int i = 0; i < B2GP_MAX_STREAMS; ++i) cudaEventCreateWithFlags(&ctx->slot_done[i], cudaEventDisableTiming);
    cudaEventCreateWithFlags(&ctx->inputs_ready, cudaEventDisableTiming);
    *out = ctx;
    return B2GP_OK;
}

// The device buffers (and the multi-GPU state, if b2gp_dist_finalize was not called) are released by `delete ctx`.
extern "C" int b2gp_ctx_destroy(b2gp_ctx* ctx) {
    if (!ctx) return B2GP_OK;
    cudaSetDevice(ctx->device);
    cudaDeviceSynchronize();
    for (Slot& s : ctx->slots) {
        for (int e = 0; e < 8; ++e) cudaEventDestroy(s.ev[e]);
        cudaStreamDestroy(s.stream);
    }
    for (cudaEvent_t e : {ctx->ev_begin, ctx->ev_end, ctx->ev_a, ctx->ev_b, ctx->inputs_ready}) cudaEventDestroy(e);
    for (cudaEvent_t e : ctx->slot_done) cudaEventDestroy(e);
    ctx->pool.destroy();
    for (void* p : ctx->user_allocs) cudaFree(p);
    delete ctx;
    return B2GP_OK;
}

static std::string g_null_err = "null context";
extern "C" const char* b2gp_last_error(const b2gp_ctx* ctx) { return ctx ? ctx->err.c_str() : g_null_err.c_str(); }

extern "C" int b2gp_set_option(b2gp_ctx* ctx, const char* key, int64_t value) {
    if (!ctx || !key) return B2GP_ERR_ARG;
    if (strcmp(key, "streams") == 0) {
        ARG_CHECK(ctx, value >= 1 && value <= B2GP_MAX_STREAMS);
        ctx->n_streams = (int)value;
        return B2GP_OK;
    }
    if (strcmp(key, "ozaki") == 0) {
        ARG_CHECK(ctx, value == -1 || value == 0 || value == 6 || value == 7);
        ctx->ozaki = (int)value;
        return B2GP_OK;
    }
    if (strcmp(key, "trsm_strip") == 0) {
        ARG_CHECK(ctx, value == 0 || value == 256 || value == 512 || value == 1024);
        ctx->trsm_strip = (int)value;
        return B2GP_OK;
    }
    if (strcmp(key, "oz_cluster") == 0) {
        ARG_CHECK(ctx, value == 1 || value == 2);
        ctx->oz_cluster = (int)value;
        return B2GP_OK;
    }
    if (strcmp(key, "enqueue_threads") == 0) {
        ctx->enqueue_threads = value != 0;
        return B2GP_OK;
    }
    if (strcmp(key, "big_grid") == 0) {
        ctx->big_grid = (int)value;
        return B2GP_OK;
    }
    if (strcmp(key, "oz_min_tiles") == 0) {
        ctx->oz_min_tiles = (int)value;
        return B2GP_OK;
    }
    if (strcmp(key, "panel") == 0) {   // diagonal-block width of the tall-panel factorisation; 0 = recursive scheme only
        ARG_CHECK(ctx, value == 0 || value == 128 || value == 256 || value == 512 || value == 1024);
        ctx->panel = (int)value;
        ctx->fcache.valid = false;
        return B2GP_OK;
    }
    if (strcmp(key, "tall_min") == 0) {
        ARG_CHECK(ctx, value >= 256);
        ctx->tall_min = (int)value;
        return B2GP_OK;
    }
    if (strcmp(key, "tall_min_fp64") == 0) {
        ARG_CHECK(ctx, value >= 256);
        ctx->tall_min_fp64 = (int)value;
        return B2GP_OK;
    }
    if (strcmp(key, "draw_batch") == 0) {   // tests and timing only: 0 = the route's group size, 1 = per-draw, B >= 2
        ARG_CHECK(ctx, value >= 0 && value <= B2GP_MAX_STREAMS);
        ctx->draw_batch = (int)value;
        return B2GP_OK;
    }
    if (strcmp(key, "bnn_fused") == 0) {   // tests and timing only: 0 puts b2gp_bnn_* on the layered route
        ARG_CHECK(ctx, value == 0 || value == 1);
        ctx->bnn_fused = (int)value;
        return B2GP_OK;
    }
    if (strcmp(key, "oz_debug") == 0) {   // timing experiments only: != 0 skips the C read-modify-write
        ARG_CHECK(ctx, value >= 0 && value <= 2);
        ctx->oz_debug = (int)value;
        return B2GP_OK;
    }
    if (strcmp(key, "tma") == 0) {
        ctx->use_tma = value ? 1 : 0;
        return B2GP_OK;
    }
    if (strcmp(key, "drop_factor_cache") == 0) {
        ctx->fcache.valid = false;
        return B2GP_OK;
    }
    return set_err(ctx, B2GP_ERR_ARG, "b2gp_set_option", "unknown key", __FILE__, __LINE__);
}

// every key of b2gp_set_option that has state ("drop_factor_cache" is an action, not a value)
extern "C" int b2gp_get_option(b2gp_ctx* ctx, const char* key, int64_t* value) {
    if (!ctx || !key || !value) return B2GP_ERR_ARG;
    const struct {
        const char* key;
        int v;
    } tab[] = {{"streams", ctx->n_streams},       {"ozaki", ctx->ozaki},         {"trsm_strip", ctx->trsm_strip},
               {"oz_cluster", ctx->oz_cluster},   {"enqueue_threads", ctx->enqueue_threads}, {"big_grid", ctx->big_grid},
               {"oz_min_tiles", ctx->oz_min_tiles}, {"panel", ctx->panel},       {"tall_min", ctx->tall_min},
               {"tall_min_fp64", ctx->tall_min_fp64}, {"bnn_fused", ctx->bnn_fused}, {"draw_batch", ctx->draw_batch},
               {"oz_debug", ctx->oz_debug},       {"tma", ctx->use_tma}};
    for (const auto& e : tab)
        if (strcmp(key, e.key) == 0) {
            *value = e.v;
            return B2GP_OK;
        }
    return set_err(ctx, B2GP_ERR_ARG, "b2gp_get_option", "unknown key", __FILE__, __LINE__);
}

extern "C" int b2gp_device_info(b2gp_ctx* ctx, int* sm_count, int* cc_major, int* cc_minor, size_t* mem_bytes) {
    if (!ctx) return B2GP_ERR_ARG;
    if (sm_count) *sm_count = ctx->sm_count;
    if (cc_major) *cc_major = ctx->cc_major;
    if (cc_minor) *cc_minor = ctx->cc_minor;
    if (mem_bytes) *mem_bytes = ctx->mem_bytes;
    return B2GP_OK;
}

extern "C" int64_t b2gp_debug_cache_hits(b2gp_ctx* ctx) { return ctx ? ctx->cache_hits : -1; }

// Development aid (not part of include/b200gp.h): the first n cumulative path counters of this context, in the order of
// PathCounter (common.cuh).  Returns how many there are.
extern "C" int b2gp_debug_path_counts(b2gp_ctx* ctx, int64_t* out, int n) {
    if (!ctx || (n > 0 && !out)) return B2GP_ERR_ARG;
    for (int i = 0; i < n && i < PATH_COUNT; ++i) out[i] = ctx->path[i].load(std::memory_order_relaxed);
    return PATH_COUNT;
}

extern "C" int b2gp_last_timing(b2gp_ctx* ctx, b2gp_timing* out) {
    if (!ctx || !out) return B2GP_ERR_ARG;
    *out = ctx->last;
    return B2GP_OK;
}

// ------------------------------------------------------------------------------------------ memory
extern "C" int b2gp_dev_alloc(b2gp_ctx* ctx, size_t bytes, void** dptr) {
    if (!ctx || !dptr) return B2GP_ERR_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    void* p = nullptr;
    cudaError_t e = cudaMalloc(&p, bytes ? bytes : 16);
    if (e != cudaSuccess) return set_err(ctx, B2GP_ERR_NOMEM, "cudaMalloc", cudaGetErrorString(e), __FILE__, __LINE__);
    ctx->user_allocs.push_back(p);
    *dptr = p;
    return B2GP_OK;
}

extern "C" int b2gp_dev_free(b2gp_ctx* ctx, void* dptr) {
    if (!ctx) return B2GP_ERR_ARG;
    if (!dptr) return B2GP_OK;
    auto& v = ctx->user_allocs;
    for (size_t i = 0; i < v.size(); ++i)
        if (v[i] == dptr) {
            v.erase(v.begin() + i);
            CUDA_TRY(ctx, cudaFree(dptr));
            return B2GP_OK;
        }
    return set_err(ctx, B2GP_ERR_ARG, "b2gp_dev_free", "pointer not owned by this ctx", __FILE__, __LINE__);
}

extern "C" int b2gp_host_alloc(b2gp_ctx* ctx, size_t bytes, void** hptr) {
    if (!ctx || !hptr) return B2GP_ERR_ARG;
    CUDA_TRY(ctx, cudaHostAlloc(hptr, bytes ? bytes : 16, cudaHostAllocDefault));
    return B2GP_OK;
}

extern "C" int b2gp_host_free(b2gp_ctx* ctx, void* hptr) {
    if (!ctx) return B2GP_ERR_ARG;
    if (hptr) CUDA_TRY(ctx, cudaFreeHost(hptr));
    return B2GP_OK;
}

extern "C" int b2gp_h2d(b2gp_ctx* ctx, void* dst, const void* src, size_t bytes) {
    if (!ctx) return B2GP_ERR_ARG;
    CUDA_TRY(ctx, cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice));
    return B2GP_OK;
}
extern "C" int b2gp_d2h(b2gp_ctx* ctx, void* dst, const void* src, size_t bytes) {
    if (!ctx) return B2GP_ERR_ARG;
    CUDA_TRY(ctx, cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost));
    return B2GP_OK;
}
extern "C" int b2gp_sync(b2gp_ctx* ctx) {
    if (!ctx) return B2GP_ERR_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    CUDA_TRY(ctx, cudaDeviceSynchronize());
    return B2GP_OK;
}

// stage a host array on the device (returns the device pointer) or pass a device pointer through
static int stage_in(b2gp_ctx* ctx, cudaStream_t st, DevBuf& buf, const void* src, size_t bytes, bool is_dev,
                    const double** out) {
    if (!src) {
        *out = nullptr;
        return B2GP_OK;
    }
    if (is_dev) {
        *out = (const double*)src;
        return B2GP_OK;
    }
    RET_IF(ensure(ctx, buf, bytes));
    CUDA_TRY(ctx, cudaMemcpyAsync(buf.p, src, bytes, cudaMemcpyHostToDevice, st));
    *out = (const double*)buf.p;
    return B2GP_OK;
}

// ---- fp32 I/O (B2GP_FLAG_F32): the reference's default precision is float32 (gpax/utils/utils.py:19-21), so callers hand
// over float arrays and expect float results.  Inputs are widened on the device right after the copy, outputs narrowed
// right before it (round to nearest); the Gram builds, the factorisation and the solves stay fp64 in between.
__global__ void cvt_f32_f64_kernel(double* __restrict__ dst, const float* __restrict__ src, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) dst[i] = (double)src[i];
}
__global__ void cvt_f64_f32_kernel(float* __restrict__ dst, int64_t ldd, const double* __restrict__ src, int64_t lds, int64_t rows,
                                   int64_t cols) {
    const int64_t total = rows * cols;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / cols, c = i % cols;
        dst[r * ldd + c] = (float)src[r * lds + c];
    }
}
static inline bool f32_io(unsigned flags) { return (flags & B2GP_FLAG_F32) != 0; }

// stage_in for `count` elements that are doubles, or floats when f32: the result is always a device array of doubles
static int stage_in_t(b2gp_ctx* ctx, cudaStream_t st, DevBuf& buf, DevBuf& tmp, const void* src, size_t count, bool is_dev, bool f32,
                      const double** out) {
    if (!f32) return stage_in(ctx, st, buf, src, count * 8, is_dev, out);
    if (!src) {
        *out = nullptr;
        return B2GP_OK;
    }
    const float* fsrc = (const float*)src;
    if (!is_dev) {
        RET_IF(ensure(ctx, tmp, count * 4));
        CUDA_TRY(ctx, cudaMemcpyAsync(tmp.p, src, count * 4, cudaMemcpyHostToDevice, st));
        fsrc = (const float*)tmp.p;
    }
    RET_IF(ensure(ctx, buf, count * 8));
    RET_IF(launch(ctx, st, grid_for((int64_t)count), 256, 0, cvt_f32_f64_kernel, (double*)buf.p, fsrc, (int64_t)count));
    *out = (const double*)buf.p;
    return B2GP_OK;
}

// A result of doubles [rows, cols] at `src` (device, leading dimension lds) -> the caller's array `dst` (leading dimension
// ldd): with f32 narrowed into the caller's float array (host or device); else copied back to the host array, or, for a
// device array, already in place (the result was written there).
static int store_out(b2gp_ctx* ctx, cudaStream_t st, DevBuf& tmp, void* dst, int64_t ldd, const double* src, int64_t lds, int64_t rows,
                     int64_t cols, bool is_dev, bool f32) {
    if (rows <= 0 || cols <= 0 || (is_dev && !f32)) return B2GP_OK;
    if (!f32) {
        if (ldd == cols && lds == cols)
            CUDA_TRY(ctx, cudaMemcpyAsync(dst, src, (size_t)rows * cols * 8, cudaMemcpyDeviceToHost, st));
        else
            CUDA_TRY(ctx, cudaMemcpy2DAsync(dst, (size_t)ldd * 8, src, (size_t)lds * 8, (size_t)cols * 8, (size_t)rows, cudaMemcpyDeviceToHost, st));
        return B2GP_OK;
    }
    float* fdst = (float*)dst;
    int64_t ldt = ldd;
    if (!is_dev) {
        RET_IF(ensure(ctx, tmp, (size_t)rows * cols * 4));
        fdst = (float*)tmp.p;
        ldt = cols;
    }
    RET_IF(launch(ctx, st, grid_for(rows * cols), 256, 0, cvt_f64_f32_kernel, fdst, ldt, src, lds, rows, cols));
    if (!is_dev)
        CUDA_TRY(ctx, cudaMemcpy2DAsync(dst, (size_t)ldd * 4, fdst, (size_t)ldt * 4, (size_t)cols * 4, (size_t)rows, cudaMemcpyDeviceToHost, st));
    return B2GP_OK;
}

// ------------------------------------------------------------------------------------------ gram
extern "C" int b2gp_gram(b2gp_ctx* ctx, int kind, const double* X, int64_t n, const double* Z, int64_t m, int d,
                         const double* lengthscale, double scale, double period, double diag_add, int same_xz, double* K,
                         int64_t ldk, unsigned flags) {
    if (!ctx) return B2GP_ERR_ARG;
    ARG_CHECK(ctx, kind >= 0 && kind <= B2GP_KERNEL_NNGP_RELU);
    ARG_CHECK(ctx, X && Z && K && lengthscale);
    ARG_CHECK(ctx, n >= 0 && m >= 0 && d >= 1 && d <= GRAM_MAX_D && ldk >= m);
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->slots[0].stream;
    CallTimer tm(ctx);
    RET_IF(tm.begin(st));
    // theta of a single "draw": lengthscale (always a host pointer: d values), scale, noise := diag_add, period
    double th[GRAM_MAX_D + 3];
    for (int k = 0; k < d; ++k) th[k] = lengthscale[k];
    th[d] = scale;
    th[d + 1] = diag_add;
    th[d + 2] = period;
    RET_IF(ensure(ctx, ctx->theta1, sizeof th));
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->theta1.p, th, (d + 3) * sizeof(double), cudaMemcpyHostToDevice, st));
    CUDA_TRY(ctx, cudaStreamSynchronize(st));  // th is a stack buffer
    const bool dev = dev_ptrs(flags), f32 = f32_io(flags);
    const double *dX, *dZ;
    RET_IF(stage_in_t(ctx, st, ctx->d_in[0], ctx->f32_in[0], X, (size_t)n * d, dev, f32, &dX));
    if (Z == X && (!dev || f32))
        dZ = dX;
    else
        RET_IF(stage_in_t(ctx, st, ctx->d_in[1], ctx->f32_in[1], Z, (size_t)m * d, dev, f32, &dZ));
    double* dK = K;
    int64_t ld = ldk;
    if (!dev || f32) {
        ld = round_up(m, 2);
        RET_IF(ensure(ctx, ctx->d_out[0], (size_t)n * ld * 8));
        dK = (double*)ctx->d_out[0].p;
    }
    const int lower = (flags & B2GP_FLAG_LOWER_ONLY) && same_xz && n == m;
    if (lower && (!dev || f32)) CUDA_TRY(ctx, cudaMemsetAsync(dK, 0, (size_t)n * ld * 8, st));
    RET_IF(launch_gram(ctx, st, kind, dX, n, dZ, m, d, (const double*)ctx->theta1.p, 1.0, 0.0, same_xz ? 1 : 0, lower, dK, ld));
    RET_IF(store_out(ctx, st, ctx->f32_out[0], K, ldk, dK, ld, n, m, dev, f32));
    RET_IF(tm.end(st, nullptr));
    ctx->last.gram_bytes = 8.0 * (double)n * (double)m + 8.0 * (double)(n + m) * d;
    return B2GP_OK;
}

// Multi-task Gram matrices (gpax/kernels/mtkernels.py:19-58 index_kernel, 61-125 MultitaskKernel):
//   K[i, j] = (k_data(x_i, z_j) + jitter [same point, same_xz]) * B[tX_i, tZ_j]  (+ noise_task[tX_i] + jitter on i == j when same_xz)
// -- the reference calls the data kernel with noise 0 but its usual diagonal rule, so k_data carries `jitter` where the two
// points coincide (mtkernels.py:103, 167); `group` consecutive rows are one data point (1, or the task count for the
// Kronecker form, whose jitter therefore lands on the whole T x T diagonal block).
// B = W W^T + diag(v) (T x T, formed by the caller: T^2 numbers).  The data kernel is the fused Gram kernel; the task factor
// is applied in place by one elementwise pass.  MultivariateKernel's Kronecker form (mtkernels.py:128-192) is the same
// thing on inputs repeated once per task with the task index cycling fastest (the shell does that).
__global__ void mt_task_kernel(double* K, int64_t ld, int64_t n, int64_t m, const int* __restrict__ tX, const int* __restrict__ tZ,
                               const double* __restrict__ B, int T, const double* __restrict__ noise_task, double jitter, int same_xz,
                               int group) {
    const int64_t total = n * m;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = idx / m, j = idx % m;
        double kd = K[i * ld + j];
        if (same_xz && i / group == j / group) kd += jitter;
        double v = kd * B[(int64_t)tX[i] * T + tZ[j]];
        if (same_xz && i == j) v += (noise_task ? noise_task[tX[i]] : 0.0) + jitter;
        K[i * ld + j] = v;
    }
}

extern "C" int b2gp_gram_multitask(b2gp_ctx* ctx, int kind, const double* X, const int* taskX, int64_t n, const double* Z,
                                   const int* taskZ, int64_t m, int d, const double* lengthscale, double scale, double period,
                                   const double* B, int T, const double* noise_task, double jitter, int same_xz, int group,
                                   double* K, int64_t ldk, unsigned flags) {
    if (!ctx) return B2GP_ERR_ARG;
    ARG_CHECK(ctx, kind >= 0 && kind <= B2GP_KERNEL_NNGP_RELU);
    ARG_CHECK(ctx, X && Z && taskX && taskZ && B && K && lengthscale);
    ARG_CHECK(ctx, n >= 1 && m >= 1 && T >= 1 && group >= 1 && d >= 1 && d <= GRAM_MAX_D && ldk >= m);
    ARG_CHECK(ctx, !(flags & (B2GP_FLAG_DEVICE_PTRS | B2GP_FLAG_F32)));      // host fp64 arrays (a callable-kernel building block)
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->slots[0].stream;
    CallTimer tm(ctx);
    RET_IF(tm.begin(st));
    double th[GRAM_MAX_D + 3];
    for (int k = 0; k < d; ++k) th[k] = lengthscale[k];
    th[d] = scale;
    th[d + 1] = 0.0;
    th[d + 2] = period;
    RET_IF(ensure(ctx, ctx->theta1, sizeof th));
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->theta1.p, th, (d + 3) * sizeof(double), cudaMemcpyHostToDevice, st));
    CUDA_TRY(ctx, cudaStreamSynchronize(st));
    const double *dX, *dZ, *dB, *dn = nullptr, *dtx, *dtz;
    RET_IF(stage_in(ctx, st, ctx->d_in[0], X, (size_t)n * d * 8, false, &dX));
    RET_IF(stage_in(ctx, st, ctx->d_in[1], Z, (size_t)m * d * 8, false, &dZ));
    RET_IF(stage_in(ctx, st, ctx->d_in[2], B, (size_t)T * T * 8, false, &dB));
    if (noise_task) RET_IF(stage_in(ctx, st, ctx->d_in[4], noise_task, (size_t)T * 8, false, &dn));
    RET_IF(stage_in(ctx, st, ctx->d_in[5], taskX, (size_t)n * 4, false, &dtx));
    RET_IF(stage_in(ctx, st, ctx->d_in[6], taskZ, (size_t)m * 4, false, &dtz));
    const int64_t ld = round_up(m, 2);
    RET_IF(ensure(ctx, ctx->d_out[0], (size_t)n * ld * 8));
    double* dK = (double*)ctx->d_out[0].p;
    RET_IF(launch_gram(ctx, st, kind, dX, n, dZ, m, d, (const double*)ctx->theta1.p, 0.0, 0.0, 0, 0, dK, ld));
    RET_IF(launch(ctx, st, grid_for(n * m), 256, 0, mt_task_kernel, dK, ld, n, m, (const int*)dtx, (const int*)dtz, dB, T, dn, jitter,
                  same_xz ? 1 : 0, group));
    CUDA_TRY(ctx, cudaMemcpy2DAsync(K, (size_t)ldk * 8, dK, (size_t)ld * 8, (size_t)m * 8, (size_t)n, cudaMemcpyDeviceToHost, st));
    return tm.end(st, nullptr);
}

// ------------------------------------------------------------------------------------------ potrf / trsm / gemm
extern "C" int b2gp_potrf(b2gp_ctx* ctx, int64_t n, double* A, int64_t lda, int* info, unsigned flags) {
    if (!ctx) return B2GP_ERR_ARG;
    ARG_CHECK(ctx, A && info && n >= 0 && lda >= n);
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->slots[0].stream;
    CallTimer tm(ctx);
    RET_IF(tm.begin(st));
    *info = 0;
    if (n == 0) return tm.end(st, nullptr);
    const bool dev = dev_ptrs(flags);
    double* dA = A;
    int64_t ld = lda;
    if (!dev) {
        ld = round_up(n, 2);
        RET_IF(ensure(ctx, ctx->potrf_buf, (size_t)n * ld * 8));
        dA = (double*)ctx->potrf_buf.p;
        CUDA_TRY(ctx, cudaMemcpy2DAsync(dA, (size_t)ld * 8, A, (size_t)lda * 8, (size_t)n * 8, (size_t)n, cudaMemcpyHostToDevice, st));
    }
    RET_IF(ensure(ctx, ctx->last_linv, (size_t)linv_bytes(n)));
    RET_IF(ensure(ctx, ctx->d_info, 64));
    CUDA_TRY(ctx, cudaMemsetAsync(ctx->d_info.p, 0, 8, st));
    RET_IF(potrf_auto(ctx, st, dA, ld, n, 0, (double*)ctx->last_linv.p, (int*)ctx->d_info.p));
    ctx->last_n = n;
    if (!dev) {
        // the strict upper triangle of the caller's array is documented as untouched: stage the factor on the
        // host and write back j <= i only
        std::vector<double> tmp((size_t)n * n);
        CUDA_TRY(ctx, cudaMemcpy2DAsync(tmp.data(), (size_t)n * 8, dA, (size_t)ld * 8, (size_t)n * 8, (size_t)n, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(ctx, cudaStreamSynchronize(st));
        for (int64_t i = 0; i < n; ++i) memcpy(A + i * lda, tmp.data() + i * n, (size_t)(i + 1) * 8);
    }
    CUDA_TRY(ctx, cudaMemcpyAsync(info, ctx->d_info.p, sizeof(int), cudaMemcpyDeviceToHost, st));
    RET_IF(tm.end(st, nullptr));
    ctx->last.flops = (double)n * (double)n * (double)n / 3.0;
    ctx->last.potrf_ms = ctx->last.total_ms;
    return B2GP_OK;
}

extern "C" int b2gp_trsm_lower(b2gp_ctx* ctx, int64_t n, int64_t nrhs, const double* L, int64_t ldl, double* B, int64_t ldb,
                               unsigned flags) {
    if (!ctx) return B2GP_ERR_ARG;
    ARG_CHECK(ctx, L && B && n >= 0 && nrhs >= 0 && ldl >= n && ldb >= n);
    if (ctx->last_n != n || !ctx->last_linv.p)
        return set_err(ctx, B2GP_ERR_ARG, "b2gp_trsm_lower", "call b2gp_potrf on this factor first (same ctx, same n)", __FILE__, __LINE__);
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->slots[0].stream;
    CallTimer tm(ctx);
    RET_IF(tm.begin(st));
    if (n == 0 || nrhs == 0) return tm.end(st, nullptr);
    const bool dev = dev_ptrs(flags);
    const double* dL = L;
    double* dB = B;
    int64_t ll = ldl, lb = ldb;
    if (!dev) {
        ll = round_up(n, 2);
        lb = ll;
        RET_IF(ensure(ctx, ctx->gemm_buf[0], (size_t)n * ll * 8));
        RET_IF(ensure(ctx, ctx->gemm_buf[1], (size_t)nrhs * lb * 8));
        CUDA_TRY(ctx, cudaMemcpy2DAsync(ctx->gemm_buf[0].p, (size_t)ll * 8, L, (size_t)ldl * 8, (size_t)n * 8, (size_t)n, cudaMemcpyHostToDevice, st));
        CUDA_TRY(ctx, cudaMemcpy2DAsync(ctx->gemm_buf[1].p, (size_t)lb * 8, B, (size_t)ldb * 8, (size_t)n * 8, (size_t)nrhs, cudaMemcpyHostToDevice, st));
        dL = (const double*)ctx->gemm_buf[0].p;
        dB = (double*)ctx->gemm_buf[1].p;
    }
    RET_IF(trsm_rec(ctx, st, dB, lb, nrhs, dL, ll, n, (const double*)ctx->last_linv.p));
    if (!dev)
        CUDA_TRY(ctx, cudaMemcpy2DAsync(B, (size_t)ldb * 8, dB, (size_t)lb * 8, (size_t)n * 8, (size_t)nrhs, cudaMemcpyDeviceToHost, st));
    RET_IF(tm.end(st, nullptr));
    ctx->last.flops = (double)n * (double)n * (double)nrhs;
    ctx->last.trsm_ms = ctx->last.total_ms;
    return B2GP_OK;
}

extern "C" int b2gp_gemm_nt(b2gp_ctx* ctx, int64_t m, int64_t n, int64_t k, double alpha, const double* A, int64_t lda,
                            const double* B, int64_t ldb, double beta, double* C, int64_t ldc, int lower_only, unsigned flags) {
    if (!ctx) return B2GP_ERR_ARG;
    ARG_CHECK(ctx, A && B && C && m >= 0 && n >= 0 && k >= 0 && lda >= k && ldb >= k && ldc >= n);
    ARG_CHECK(ctx, !lower_only || m >= n);   // m > n: lower triangle of the leading n x n block, all of the rows below it
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->slots[0].stream;
    CallTimer tm(ctx);
    RET_IF(tm.begin(st));
    const bool dev = dev_ptrs(flags);
    const double *dA = A, *dB = B;
    double* dC = C;
    int64_t la = lda, lb = ldb, lc = ldc;
    if (!dev) {
        la = lb = round_up(k > 0 ? k : 1, 2);
        lc = round_up(n > 0 ? n : 1, 2);
        RET_IF(ensure(ctx, ctx->gemm_buf[0], (size_t)(m + 1) * la * 8));
        RET_IF(ensure(ctx, ctx->gemm_buf[1], (size_t)(n + 1) * lb * 8));
        RET_IF(ensure(ctx, ctx->gemm_buf[2], (size_t)(m + 1) * lc * 8));
        if (m && k) CUDA_TRY(ctx, cudaMemcpy2DAsync(ctx->gemm_buf[0].p, (size_t)la * 8, A, (size_t)lda * 8, (size_t)k * 8, (size_t)m, cudaMemcpyHostToDevice, st));
        if (n && k) CUDA_TRY(ctx, cudaMemcpy2DAsync(ctx->gemm_buf[1].p, (size_t)lb * 8, B, (size_t)ldb * 8, (size_t)k * 8, (size_t)n, cudaMemcpyHostToDevice, st));
        if (m && n) CUDA_TRY(ctx, cudaMemcpy2DAsync(ctx->gemm_buf[2].p, (size_t)lc * 8, C, (size_t)ldc * 8, (size_t)n * 8, (size_t)m, cudaMemcpyHostToDevice, st));
        dA = (const double*)ctx->gemm_buf[0].p;
        dB = (A == B && lda == ldb && m == n) ? dA : (const double*)ctx->gemm_buf[1].p;
        dC = (double*)ctx->gemm_buf[2].p;
    }
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_a, st));
    RET_IF(gemm_nt(ctx, st, m, n, k, alpha, dA, la, dB, lb, beta, dC, lc, lower_only != 0));
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_b, st));
    if (!dev && m && n)
        CUDA_TRY(ctx, cudaMemcpy2DAsync(C, (size_t)ldc * 8, dC, (size_t)lc * 8, (size_t)n * 8, (size_t)m, cudaMemcpyDeviceToHost, st));
    RET_IF(tm.end(st, nullptr));
    float ms = 0.f;
    CUDA_TRY(ctx, cudaEventElapsedTime(&ms, ctx->ev_a, ctx->ev_b));
    ctx->last.epilogue_ms = ms;  // kernel-only time of the GEMM launch
    ctx->last.flops = (lower_only ? 1.0 : 2.0) * (double)m * (double)n * (double)k;
    return B2GP_OK;
}

// ------------------------------------------------------------------------------------------ posterior
namespace {
struct StageEvents {
    cudaEvent_t e[6];
};
}

// diag(A) += v   (per-point noise variances: mngp.py:96, hskgp.py:147); the draw of a batch is blockIdx.z (A `bstride`
// doubles apart, v `vstride` apart)
__global__ void add_diag_vec_kernel(double* A, int64_t ld, int64_t n, const double* __restrict__ v, int64_t bstride, int64_t vstride) {
    A += (int64_t)blockIdx.z * bstride;
    v += (int64_t)blockIdx.z * vstride;
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) A[i * ld + i] += v[i];
}

// The LCM covariance of MultiTaskGP / CoregGP (mtgp.cuh) in place of the single-task kernel: host arrays, task ids
// validated by the caller.  nullptr for every single-task entry.
struct MtDesc {
    const int* task_tr;    // [N]
    const int* task_new;   // [P] (posterior only)
    int group, T, L;
    const double* B;       // [S, L, T, T]
    const double* noise;   // [S, T]
};

// ---- caller-supplied Gram matrices (b2gp_mll_gram, b2gp_posterior_gram)
// The lower triangle of (K + K^T) / 2 into A (leading dimension lda).  A host K is first copied whole into `stage`.
static int gram_copyin(b2gp_ctx* ctx, cudaStream_t st, DevBuf& stage, const double* K, int64_t ldk, int64_t N, bool dev, double* A,
                       int64_t lda) {
    const double* src = K;
    int64_t lds = ldk;
    if (!dev) {
        lds = round_up(N, 8);
        RET_IF(ensure(ctx, stage, (size_t)N * lds * 8));
        CUDA_TRY(ctx, cudaMemcpy2DAsync(stage.p, (size_t)lds * 8, K, (size_t)ldk * 8, (size_t)N * 8, (size_t)N, cudaMemcpyHostToDevice, st));
        src = (const double*)stage.p;
    }
    const unsigned t = (unsigned)ceil_div(N, (int64_t)GCOPY_TILE);
    return launch(ctx, st, dim3(t, t), dim3(GCOPY_TILE, 8), 0, gram_copyin_kernel, src, lds, N, A, lda);
}

// b2gp_posterior_gram: the three Gram blocks of every draw come from the caller (host or device arrays, as `flags`):
// k_XX [N, N] (symmetrised on the copy-in), k_pX [P, N], k_pp [P, P] or only its diagonal [P] (kpp_diag); strides between
// draws in doubles, 0 = shared.
struct GramPost {
    const double* Kxx;
    int64_t kxx_stride;
    const double* Kpx;
    int64_t kpx_stride;
    const double* Kpp;
    int64_t kpp_stride;
    bool kpp_diag;
};

// The posterior with everything that may vary per draw: the training inputs (xtr_stride doubles between draws; 0 =
// shared), the test inputs (xnew_stride), the targets (yres_stride) and an optional vector of per-point noise variances
// added to the diagonal of k_XX (nv_stride between draws; 0 = shared).  b2gp_posterior is the all-shared special case.
// With B2GP_OUT_DMEAN / B2GP_OUT_DVAR (b2gp_posterior_grad and b2gp_posterior_multitask_grad only) the P*d derivative
// rows of grad.cuh (gram_dx_lcm_kernel, mtgp.cuh, for the LCM covariance) ride under [k_pX; y^T] through the same
// factorisation or solve, and dmean / dvar [S, P, d] are their row dots.
static int posterior_impl(b2gp_ctx* ctx, int kind, const double* Xtr, int64_t xtr_stride, int64_t N, const double* yres,
                          int64_t yres_stride, const double* Xnew, int64_t xnew_stride, int64_t P, int d, int64_t S,
                          const double* theta, const double* noise_vec, int64_t nv_stride, int noiseless, double jitter,
                          unsigned flags, double* mean, double* var, double* cov, const double* eps, int64_t n_samp,
                          double* y_sampled, int* info, b2gp_timing* timing, double* dmean_out = nullptr, double* dvar_out = nullptr,
                          const MtDesc* mt = nullptr, const GramPost* gp = nullptr) {
    if (!ctx) return B2GP_ERR_ARG;
    ARG_CHECK(ctx, kind >= 0 && kind <= B2GP_KERNEL_NNGP_RELU);
    const bool nngp = is_nngp(kind);   // NNGP: no multi-task form, no test-input gradient
    ARG_CHECK(ctx, !nngp || (!mt && !(flags & (B2GP_OUT_DMEAN | B2GP_OUT_DVAR))));
    ARG_CHECK(ctx, xtr_stride == 0 || xtr_stride >= N * d);
    ARG_CHECK(ctx, xnew_stride == 0 || xnew_stride >= P * d);
    ARG_CHECK(ctx, nv_stride == 0 || nv_stride >= N);
    ARG_CHECK(ctx, (gp || (Xtr && Xnew && theta)) && yres && info);
    ARG_CHECK(ctx, N >= 1 && P >= 1 && S >= 1 && d >= 1 && d <= GRAM_MAX_D);
    ARG_CHECK(ctx, yres_stride == 0 || yres_stride >= N);
    const bool want_mean = flags & B2GP_OUT_MEAN, want_var = flags & B2GP_OUT_VAR;
    const bool want_cov = flags & B2GP_OUT_COV, want_samp = flags & B2GP_OUT_SAMPLE;
    const bool want_dmean = flags & B2GP_OUT_DMEAN, want_dvar = flags & B2GP_OUT_DVAR;
    ARG_CHECK(ctx, !want_dmean || dmean_out);
    ARG_CHECK(ctx, !want_dvar || dvar_out);
    // rows of the slot's right-hand side block: [k_pX (P); y^T (1); D (G = P*d derivative rows, gradient calls only)]
    const int64_t G = (want_dmean || want_dvar) ? P * d : 0, R = P + 1 + G;
    ARG_CHECK(ctx, !want_mean || mean);
    ARG_CHECK(ctx, !want_var || var);
    ARG_CHECK(ctx, !want_cov || cov);
    ARG_CHECK(ctx, !want_samp || (eps && y_sampled && n_samp >= 1));
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    const bool dev = dev_ptrs(flags), f32 = f32_io(flags);
    if (nngp) {   // every draw's depth, before any work is queued
        std::vector<double> hth((size_t)S * (d + 3));
        if (dev)
            CUDA_TRY(ctx, cudaMemcpy(hth.data(), theta, hth.size() * 8, cudaMemcpyDeviceToHost));
        else
            memcpy(hth.data(), theta, hth.size() * 8);
        for (int64_t s = 0; s < S; ++s) RET_IF(nngp_check_depth(ctx, "b2gp_posterior", hth[(size_t)s * (d + 3)]));
    }
    const int nslots = (int)(S < ctx->n_streams ? S : ctx->n_streams);
    cudaStream_t st0 = ctx->slots[0].stream;
    CallTimer tm(ctx);
    RET_IF(tm.begin(st0));
    auto slot_stream = [&](int q) { return ctx->slots[q].stream; };

    // ---- inputs
    const int nth = mt ? mt->L * (d + 2) : d + 3;
    const double *dXtr, *dy, *dXnew, *dtheta, *deps = nullptr, *dnv = nullptr;
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_a, st0));
    // with B2GP_FLAG_F32 the data arrays (X, y, X_new, noise_vec, eps) are floats; theta stays double
    RET_IF(stage_in_t(ctx, st0, ctx->d_in[0], ctx->f32_in[0], Xtr, (size_t)(xtr_stride ? S * xtr_stride : N * d), dev, f32, &dXtr));
    RET_IF(stage_in_t(ctx, st0, ctx->d_in[1], ctx->f32_in[1], yres, (size_t)(yres_stride ? S * yres_stride : N), dev, f32, &dy));
    RET_IF(stage_in_t(ctx, st0, ctx->d_in[2], ctx->f32_in[2], Xnew, (size_t)(xnew_stride ? S * xnew_stride : P * d), dev, f32, &dXnew));
    if (noise_vec) RET_IF(stage_in_t(ctx, st0, ctx->d_in[6], ctx->f32_in[6], noise_vec, (size_t)(nv_stride ? S * nv_stride : N), dev, f32, &dnv));
    RET_IF(stage_in(ctx, st0, ctx->d_in[3], theta, (size_t)S * nth * 8, dev, &dtheta));
    if (want_samp) RET_IF(stage_in_t(ctx, st0, ctx->d_in[4], ctx->f32_in[4], eps, (size_t)S * n_samp * P, dev, f32, &deps));
    // NNGP: d+3 zeros, the theta of the zero prior the variance epilogue starts from
    const double* dzero = nullptr;
    std::vector<double> hzero;
    if (nngp || gp) {
        hzero.assign((size_t)d + 3, 0.0);
        RET_IF(stage_in(ctx, st0, ctx->d_in[5], hzero.data(), hzero.size() * 8, false, &dzero));
    }
    // multi-task: [B (S*L*T*T) | noise (S*T) | d+3 zeros] and the task ids [task_tr (N) | task_new (P)]
    const double* dmt = nullptr;
    const int* dtask = nullptr;
    std::vector<double> hmt;
    std::vector<int> htask;
    if (mt) {
        const size_t nb = (size_t)S * mt->L * mt->T * mt->T, nn = (size_t)S * mt->T;
        hmt.assign(nb + nn + d + 3, 0.0);
        memcpy(hmt.data(), mt->B, nb * 8);
        memcpy(hmt.data() + nb, mt->noise, nn * 8);
        htask.resize((size_t)(N + P));
        memcpy(htask.data(), mt->task_tr, (size_t)N * 4);
        memcpy(htask.data() + N, mt->task_new, (size_t)P * 4);
        RET_IF(stage_in(ctx, st0, ctx->d_in[5], hmt.data(), hmt.size() * 8, false, &dmt));
        const double* dt = nullptr;
        RET_IF(stage_in(ctx, st0, ctx->d_in[7], htask.data(), htask.size() * 4, false, &dt));
        dtask = (const int*)dt;
    }
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_b, st0));
    CUDA_TRY(ctx, cudaEventRecord(ctx->inputs_ready, st0));

    // ---- outputs
    double *dmean = mean, *dvar = var, *dcov = cov, *dsamp = y_sampled, *ddmean = dmean_out, *ddvar = dvar_out;
    if (!dev || f32) {
        if (want_mean) {
            RET_IF(ensure(ctx, ctx->d_out[0], (size_t)S * P * 8));
            dmean = (double*)ctx->d_out[0].p;
        }
        if (want_var) {
            RET_IF(ensure(ctx, ctx->d_out[1], (size_t)S * P * 8));
            dvar = (double*)ctx->d_out[1].p;
        }
        if (want_cov) {
            RET_IF(ensure(ctx, ctx->d_out[2], (size_t)S * P * P * 8));
            dcov = (double*)ctx->d_out[2].p;
        }
        if (want_samp) {
            RET_IF(ensure(ctx, ctx->d_out[3], (size_t)S * n_samp * P * 8));
            dsamp = (double*)ctx->d_out[3].p;
        }
        // a gradient call has no covariance or samples: their staging buffers take dmean / dvar
        if (want_dmean) {
            RET_IF(ensure(ctx, ctx->d_out[2], (size_t)S * P * d * 8));
            ddmean = (double*)ctx->d_out[2].p;
        }
        if (want_dvar) {
            RET_IF(ensure(ctx, ctx->d_out[3], (size_t)S * P * d * 8));
            ddvar = (double*)ctx->d_out[3].p;
        }
    }
    RET_IF(ensure(ctx, ctx->d_info, (size_t)2 * S * sizeof(int)));
    int* dinfo = (int*)ctx->d_info.p;
    CUDA_TRY(ctx, cudaMemsetAsync(dinfo, 0, (size_t)2 * S * sizeof(int), st0));

    // ---- per-slot workspaces
    // Draw region q of ctx->post = [Linv | A | panel scratch], regE doubles apart: the right-hand-side rows [k_pX; y^T]
    // live directly under k_XX in A (potrf_tall solves them with the factorisation's own panel GEMMs), and consecutive
    // regions form the batch of a group of draws.  Linv and k_XX do not move with P, so region 0 keeps the cached factor.
    const int64_t ldA = round_up(N, 8), ldV = ldA, ldC = round_up(P, 8);
    const bool need_cov = want_cov || want_samp;
    const bool tall = use_tall(ctx, N) || use_tall_fp64(ctx, N);
    const int64_t linvE = linv_bytes(N) / 8, aE = (N + R) * ldA;
    const int64_t regE = round_up(linvE + aE + (tall ? panel_scratch_elems(ctx, N < ctx->panel ? N : ctx->panel) : 0), 32);
    // Draws in lock-step groups of B (DESIGN.md 4.2): on the fp64 tall-panel route one batched potrf_tall factors a whole
    // group, every launch covering all its draws, and `ngs` groups are in flight on as many slot streams.  B = 1 is one
    // draw per group, every slot its own stream.  Group g runs on slot g % ngs, in regions (g % ngs) B .. + B - 1.  The
    // route's own choice keeps two groups in flight (one group leaves its diagonal chain exposed, DESIGN.md 5): B = 4
    // where the slots allow two groups of 4, fewer draws per group below that, and one draw per group (the per-draw
    // route) where even two groups of 2 do not fit.  S >= 2 rules out the factor cache (S = 1 calls only).
    int B = 1;
    if (use_tall_fp64(ctx, N) && S >= 2) {
        if (ctx->draw_batch == 0) {
            B = nslots / 2 < B2GP_DRAW_BATCH_DEFAULT ? nslots / 2 : B2GP_DRAW_BATCH_DEFAULT;
            if (B < 2) B = 1;
        } else {
            B = ctx->draw_batch < nslots ? ctx->draw_batch : nslots;
        }
    }
    const int ngs = nslots / B;
    const int64_t ngroups = ceil_div(S, (int64_t)B);
    {
        const size_t need = (size_t)ngs * B * regE * 8;   // the regions in use: ngs groups of B
        if (ctx->fcache.valid && ctx->fcache.N == N && ctx->post.p && ctx->post.cap < need) {
            // region 0 holds the cached factor and this call brings more test points than the one that made it:
            // grow the buffer AROUND the factor (a plain ensure() would free it and the reuse below would read garbage)
            DevBuf grown;
            RET_IF(ensure(ctx, grown, need));
            CUDA_TRY(ctx, cudaMemcpyAsync(grown.p, ctx->post.p, (size_t)(linvE + N * ldA) * 8, cudaMemcpyDeviceToDevice, st0));
            CUDA_TRY(ctx, cudaStreamSynchronize(st0));
            ctx->post = std::move(grown);
        }
        RET_IF(ensure(ctx, ctx->post, need));
    }
    for (int q = 0; q < ngs; ++q) {
        Slot& sl = ctx->slots[q];
        if (need_cov) RET_IF(ensure(ctx, sl.cov, (size_t)P * ldC * 8));
        if (want_samp) RET_IF(ensure(ctx, sl.LinvC, (size_t)linv_bytes(P)));
        if (!want_mean || ((mt || nngp || gp) && want_var)) RET_IF(ensure(ctx, sl.misc, (size_t)((mt || nngp || gp) ? 2 * P : P) * 8));
        if (gp && !dev) RET_IF(ensure(ctx, sl.Vt, (size_t)N * ldA * 8));   // a host k_XX is staged here before the copy-in
    }
    // inputs and the memset of dinfo were queued on st0: order the other streams behind them
    CUDA_TRY(ctx, cudaEventRecord(ctx->inputs_ready, st0));
    for (int q = 0; q < ngs; ++q)
        if (slot_stream(q) != st0) CUDA_TRY(ctx, cudaStreamWaitEvent(slot_stream(q), ctx->inputs_ready, 0));

    // host copy of theta: the accuracy-aware digit-plane count of the int8 path is chosen per draw (oz_auto_planes)
    std::vector<double> htheta;
    if (ctx->ozaki == -1 && !mt && !gp) {
        htheta.resize((size_t)S * nth);
        if (dev) {
            CUDA_TRY(ctx, cudaMemcpyAsync(htheta.data(), dtheta, (size_t)S * nth * 8, cudaMemcpyDeviceToHost, st0));
            CUDA_TRY(ctx, cudaStreamSynchronize(st0));
        } else {
            memcpy(htheta.data(), theta, (size_t)S * nth * 8);
        }
    }
    const double noise_mult_new = noiseless ? 0.0 : 1.0;  // gp.py:260-261
    const cudaMemcpyKind cpkind = dev ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;   // caller Gram blocks
    std::vector<StageEvents> sev;
    if (timing) sev.resize((size_t)S);

    // factor reuse (see b2gp_ctx::fcache): same kind / N / d / jitter / theta / training inputs as the previous
    // single-draw host-pointer call -> skip the Gram build and the factorisation
    // The cache is invalid for the whole duration of the call: any early return (allocation failure, launch error)
    // leaves it so, and it is re-validated -- together with the factor's `info` -- only after the call's work has
    // completed on the device (end of this function).
    bool reuse = false;
    const bool cacheable = (S == 1 && !dev && !noise_vec && !mt && !gp);
    if (cacheable) {
        auto& fc = ctx->fcache;
        const size_t xbytes = (size_t)N * d * (f32 ? 4 : 8);
        reuse = fc.valid && fc.kind == kind && fc.N == N && fc.d == d && fc.jitter == jitter && fc.X.size() == xbytes &&
                memcmp(fc.theta.data(), theta, (size_t)nth * 8) == 0 && memcmp(fc.X.data(), Xtr, xbytes) == 0;
        if (reuse) ctx->cache_hits++;
    }
    ctx->fcache.valid = false;
    // a cacheable call that factors by the tall-panel scheme also keeps the diagonal blocks' explicit inverses
    const bool keepU = cacheable && !reuse && use_tall(ctx, N);
    if (keepU) RET_IF(ensure(ctx, ctx->Ukeep, (size_t)ceil_div(N, (int64_t)ctx->panel) * ctx->panel * ctx->panel * 8));

    // One draw's work before (front) or after (!front) the factorisation of its group, queued on the group's stream, in
    // draw region `reg`.  Returns a B2GP_* code.
    auto enqueue_draw = [&](int64_t s, int gq, int64_t reg, bool front) -> int {
        Slot& sl = ctx->slots[gq];
        cudaStream_t st = sl.stream;
        double* Linv = (double*)ctx->post.p + reg * regE;
        double* A = Linv + linvE;
        double* Vt = A + N * ldA;
        const double* th = dtheta ? dtheta + s * nth : nullptr;
        const double* dXtr_s = dXtr + s * xtr_stride;
        const double* dXnew_s = dXnew + s * xnew_stride;
        // the P-side solve rides along with the factorisation (int8 or fp64 route of the tall-panel scheme)
        const bool fused_solve = !reuse && (use_tall(ctx, N) || use_tall_fp64(ctx, N));
        int* inf = dinfo + s;
        int* inf2 = dinfo + S + s;
        const int T = mt ? mt->T : 0, L = mt ? mt->L : 0, grp = mt ? mt->group : 0;
        const double* Bs = mt ? dmt + s * L * T * T : nullptr;
        const double* ns = mt ? dmt + (size_t)S * L * T * T + s * T : nullptr;
        const int *dtr = dtask, *dtn = mt ? dtask + N : nullptr;
        auto rhs_rows = [&]() -> int {
            // k_pX = kernel(X_new, X_train, params, jitter=0.0)  (gp.py:268); same-shape inputs add 0 there
            if (gp)
                CUDA_TRY(ctx, cudaMemcpy2DAsync(Vt, (size_t)ldV * 8, gp->Kpx + s * gp->kpx_stride, (size_t)N * 8, (size_t)N * 8, (size_t)P, cpkind, st));
            else if (mt)
                RET_IF(launch_gram_lcm(ctx, st, LCM_RECT, kind, dXnew_s, dtn, P, dXtr_s, dtr, N, d, T, L, grp, th, Bs, ns, 0.0, 0.0, Vt, ldV));
            else
                RET_IF(launch_gram(ctx, st, kind, dXnew_s, P, dXtr_s, N, d, th, 0.0, 0.0, 0, 0, Vt, ldV));
            CUDA_TRY(ctx, cudaMemcpyAsync(Vt + P * ldV, dy + (yres_stride ? s * yres_stride : 0), (size_t)N * 8, cudaMemcpyDeviceToDevice, st));
            if (G && mt)
                RET_IF(launch_gram_dx_lcm(ctx, st, kind, dXnew_s, dtn, P, dXtr_s, dtr, N, d, T, L, th, Bs, Vt + (P + 1) * ldV, ldV));
            else if (G)
                RET_IF(launch_gram_dx(ctx, st, kind, dXnew_s, P, dXtr_s, N, d, th, Vt + (P + 1) * ldV, ldV));
            return B2GP_OK;
        };
        if (front) {
            if (timing) {
                for (int e = 0; e < 6; ++e) sev[s].e[e] = ctx->pool.get();
                CUDA_TRY(ctx, cudaEventRecord(sev[s].e[0], st));
            }
            // factorisation and P-side solve: 6 or 7 digit planes from the trace bound on cond(K); covariance / sampling: 7.
            // The bound takes k(x, x) = k_scale, which an NNGP kernel does not satisfy: 7 there.
            sl.oz_planes = (htheta.empty() || noise_vec || mt || nngp) ? 7 : oz_auto_planes((double)N, htheta[s * nth + d], htheta[s * nth + d + 1], jitter);
            if (reuse) {
                if (timing) CUDA_TRY(ctx, cudaEventRecord(sev[s].e[1], st));
                return B2GP_OK;
            }
            // k_XX = kernel(X_train, X_train, params, noise, jitter)  (gp.py:269) -- lower triangle only
            if (gp)
                RET_IF(gram_copyin(ctx, st, sl.Vt, gp->Kxx + s * gp->kxx_stride, N, N, dev, A, ldA));
            else if (mt)
                RET_IF(launch_gram_lcm(ctx, st, LCM_LOWER, kind, dXtr_s, dtr, N, dXtr_s, dtr, N, d, T, L, grp, th, Bs, ns, 1.0, jitter, A, ldA));
            else
                RET_IF(launch_gram(ctx, st, kind, dXtr_s, N, dXtr_s, N, d, th, 1.0, jitter, 1, 1, A, ldA));
            if (dnv) RET_IF(launch(ctx, st, grid_for(N), 256, 0, add_diag_vec_kernel, A, ldA, N, dnv + s * nv_stride, (int64_t)0, (int64_t)0));
            if (fused_solve) RET_IF(rhs_rows());
            if (timing) CUDA_TRY(ctx, cudaEventRecord(sev[s].e[1], st));
            return B2GP_OK;
        }
        if (timing) CUDA_TRY(ctx, cudaEventRecord(sev[s].e[2], st));
        if (!fused_solve) RET_IF(rhs_rows());
        if (timing) CUDA_TRY(ctx, cudaEventRecord(sev[s].e[3], st));
        // [V^T; w^T] = [k_pX; y^T] L^{-T}
        if (!fused_solve) {
            if (reuse && ctx->fcache.U_nb > 0 && ctx->fcache.U_nb == ctx->panel && ctx->ozaki != 0)
                RET_IF(trsm_tall(ctx, st, Vt, ldV, R, A, ldA, N, (const double*)ctx->Ukeep.p, ctx->fcache.U_nb));
            else
                RET_IF(trsm_rec(ctx, st, Vt, ldV, R, A, ldA, N, Linv));
        }
        if (timing) CUDA_TRY(ctx, cudaEventRecord(sev[s].e[4], st));
        // mean / var
        double* mean_s = want_mean ? dmean + s * P : (double*)sl.misc.p;
        if (mt) {   // var = prior diagonal - |V^T[p,:]|^2: rowdot_kernel on a zero prior (a periodic kernel of scale 0), then the LCM diagonal
            const double* zero = dmt + (size_t)S * L * T * T + (size_t)S * T;
            if (want_mean || want_var || want_samp)
                RET_IF(launch(ctx, st, (unsigned)P, RD_THREADS, 0, rowdot_kernel, Vt, ldV, N, P, (int)B2GP_KERNEL_PERIODIC, d, zero, 0.0, 0.0, inf,
                              mean_s, want_var ? dvar + s * P : nullptr));
            if (want_var) {
                double* prior = (double*)sl.misc.p + P;
                RET_IF(launch_gram_lcm(ctx, st, LCM_DIAG, kind, dXnew_s, dtn, P, nullptr, nullptr, 0, d, T, L, grp, th, Bs, ns, noise_mult_new,
                                       jitter, prior, 1));
                RET_IF(launch(ctx, st, (unsigned)ceil_div(P, (int64_t)256), 256, 0, add_vec_kernel, dvar + s * P, (const double*)prior, P));
            }
        } else if (nngp || gp) {   // as the multi-task branch, with the prior diagonal k(x_p, x_p) + noise_p + jitter
            if (want_mean || want_var || want_samp)
                RET_IF(launch(ctx, st, (unsigned)P, RD_THREADS, 0, rowdot_kernel, Vt, ldV, N, P, (int)B2GP_KERNEL_PERIODIC, d, dzero, 0.0, 0.0,
                              inf, mean_s, want_var ? dvar + s * P : nullptr));
            if (want_var) {
                double* prior = (double*)sl.misc.p + P;
                if (gp)   // diag(k_pp): a strided copy of the full block's diagonal, or the caller's diagonal as it is
                    CUDA_TRY(ctx, cudaMemcpy2DAsync(prior, 8, gp->Kpp + s * gp->kpp_stride, (size_t)(gp->kpp_diag ? 1 : P + 1) * 8, 8, (size_t)P,
                                                    cpkind, st));
                else
                    RET_IF(launch(ctx, st, (unsigned)ceil_div(P, (int64_t)256), 256, 0, nngp_diag_kernel, dXnew_s, P, d, kind, th, noise_mult_new,
                                  jitter, prior));
                RET_IF(launch(ctx, st, (unsigned)ceil_div(P, (int64_t)256), 256, 0, add_vec_kernel, dvar + s * P, (const double*)prior, P));
            }
        } else if (want_mean || want_var || want_samp) {
            RET_IF(launch(ctx, st, (unsigned)P, RD_THREADS, 0, rowdot_kernel, Vt, ldV, N, P, kind, d, th, noise_mult_new, jitter, inf, mean_s,
                          want_var ? dvar + s * P : nullptr));
        }
        if (G)
            RET_IF(launch(ctx, st, (unsigned)P, RD_THREADS, 0, rowdot_grad_kernel, Vt, ldV, N, P, d, inf,
                          want_dmean ? ddmean + s * P * d : nullptr, want_dvar ? ddvar + s * P * d : nullptr));
        if (need_cov) {
            sl.oz_planes = 7;
            // cov = k_pp - V^T V  (gp.py:267, 272), lower tiles then mirrored -> exactly symmetric
            double* C = want_cov ? dcov + s * P * P : (double*)sl.cov.p;
            const int64_t ldc = want_cov ? P : ldC;
            if (gp)
                CUDA_TRY(ctx, cudaMemcpy2DAsync(C, (size_t)ldc * 8, gp->Kpp + s * gp->kpp_stride, (size_t)P * 8, (size_t)P * 8, (size_t)P, cpkind, st));
            else if (mt)
                RET_IF(launch_gram_lcm(ctx, st, LCM_LOWER, kind, dXnew_s, dtn, P, dXnew_s, dtn, P, d, T, L, grp, th, Bs, ns, noise_mult_new,
                                       jitter, C, ldc));
            else
                RET_IF(launch_gram(ctx, st, kind, dXnew_s, P, dXnew_s, P, d, th, noise_mult_new, jitter, 1, 1, C, ldc));
            RET_IF(gemm_nt(ctx, st, P, P, N, -1.0, Vt, ldV, Vt, ldV, 1.0, C, ldc, true));
            dim3 g2((unsigned)ceil_div(P, 32), (unsigned)ceil_div(P, 32)), b2(32, 32);
            RET_IF(launch(ctx, st, g2, b2, 0, mirror_lower_kernel, C, ldc, P));
            if (want_samp) {
                // y = mean + chol(cov) eps  (gp.py:292)
                double* CL = (double*)sl.cov.p;
                if (want_cov) RET_IF(launch(ctx, st, grid_for(P * P), 256, 0, copy2d_kernel, CL, ldC, C, ldc, P, P));
                RET_IF(potrf_rec(ctx, st, CL, ldC, P, (double*)sl.LinvC.p, inf2, 0));
                RET_IF(launch(ctx, st, g2, b2, 0, zero_upper_kernel, CL, ldC, P));
                double* Y = dsamp + s * n_samp * P;
                RET_IF(launch(ctx, st, grid_for(n_samp * P), 256, 0, bcast_rows_kernel, Y, P, n_samp, P, mean_s));
                RET_IF(gemm_nt(ctx, st, n_samp, P, P, 1.0, deps + s * n_samp * P, P, CL, ldC, 1.0, Y, P, false));
                RET_IF(launch(ctx, st, grid_for(n_samp * P), 256, 0, nan_if_bad_kernel, Y, P, n_samp, P, inf, inf2));
            }
            if (want_cov) RET_IF(launch(ctx, st, grid_for(P * P), 256, 0, nan_if_bad_kernel, C, ldc, P, P, inf, nullptr));
        }
        if (timing) CUDA_TRY(ctx, cudaEventRecord(sev[s].e[5], st));
        return B2GP_OK;
    };
    // One group: its draws' Gram blocks, the factorisation of all of them (with the P-side solve on the tall-panel route),
    // then their epilogues.
    auto enqueue_group = [&](int64_t g) -> int {
        const int gq = (int)(g % ngs);
        cudaStream_t st = slot_stream(gq);
        const int64_t s0 = g * B, reg0 = (int64_t)gq * B;
        const int nb = (int)(S - s0 < B ? S - s0 : B);
        double* Linv = (double*)ctx->post.p + reg0 * regE;
        double* A = Linv + linvE;
        for (int j = 0; j < nb; ++j) RET_IF(enqueue_draw(s0 + j, gq, reg0 + j, true));
        if (!reuse) {
            // factor instead of jnp.linalg.inv (gp.py:271); with the tall-panel scheme also [V^T; w^T] = [k_pX; y^T] L^{-T}
            if (tall) {
                for (int j = 0; j < nb; ++j) count_tall_entry(ctx, use_tall(ctx, N));
                if (nb > 1) count_path(ctx, (int)PATH_POTRF_TALL_BATCH);
                Batch bt;
                bt.n = nb;
                bt.stride = regE;
                RET_IF(potrf_tall(ctx, st, A + aE, A, ldA, N, R, Linv, dinfo + s0, 0, keepU ? (double*)ctx->Ukeep.p : nullptr, bt));
            } else {
                RET_IF(potrf_rec(ctx, st, A, ldA, N, Linv, dinfo + s0, 0));
            }
        } else {
            CUDA_TRY(ctx, cudaMemcpyAsync(dinfo + s0, &ctx->fcache.info, sizeof(int), cudaMemcpyHostToDevice, st));
        }
        for (int j = 0; j < nb; ++j) RET_IF(enqueue_draw(s0 + j, gq, reg0 + j, false));
        return B2GP_OK;
    };
    // A draw is ~1.4k launches at N=16384 and the driver lets the host run only ~1k launches ahead of the device, so a
    // single queueing thread feeds the slots one after the other and their streams barely overlap.  One host thread
    // per group slot keeps every stream's queue full (the slots share nothing but read-only inputs).
    if (ctx->enqueue_threads && ngs > 1 && ngroups > ngs && !timing) {
        std::vector<int> rcs((size_t)ngs, B2GP_OK);
        std::vector<std::thread> workers;
        for (int q = 0; q < ngs; ++q)
            workers.emplace_back([&, q] {
                if (cudaSetDevice(ctx->device) != cudaSuccess) {
                    rcs[q] = B2GP_ERR_CUDA;
                    return;
                }
                for (int64_t g = q; g < ngroups && rcs[q] == B2GP_OK; g += ngs) rcs[q] = enqueue_group(g);
            });
        for (auto& w : workers) w.join();
        for (int q = 0; q < ngs; ++q) RET_IF(rcs[q]);
    } else {
        for (int64_t g = 0; g < ngroups; ++g) RET_IF(enqueue_group(g));
    }
    tm.mark_enqueued();
    // ---- join the slots on stream 0
    for (int q = 0; q < ngs; ++q) {
        if (slot_stream(q) == st0) continue;
        CUDA_TRY(ctx, cudaEventRecord(ctx->slot_done[q], slot_stream(q)));
        CUDA_TRY(ctx, cudaStreamWaitEvent(st0, ctx->slot_done[q], 0));
    }
    cudaEvent_t ev_c = ctx->slots[0].ev[0], ev_d = ctx->slots[0].ev[1];
    CUDA_TRY(ctx, cudaEventRecord(ev_c, st0));
    std::vector<int> hinfo((size_t)2 * S);
    CUDA_TRY(ctx, cudaMemcpyAsync(hinfo.data(), dinfo, (size_t)2 * S * sizeof(int), cudaMemcpyDeviceToHost, st0));
    if (want_mean) RET_IF(store_out(ctx, st0, ctx->f32_out[0], mean, P, dmean, P, S, P, dev, f32));
    if (want_var) RET_IF(store_out(ctx, st0, ctx->f32_out[1], var, P, dvar, P, S, P, dev, f32));
    if (want_cov) RET_IF(store_out(ctx, st0, ctx->f32_out[2], cov, P, dcov, P, S * P, P, dev, f32));
    if (want_samp) RET_IF(store_out(ctx, st0, ctx->f32_out[3], y_sampled, P, dsamp, P, S * n_samp, P, dev, f32));
    if (want_dmean) RET_IF(store_out(ctx, st0, ctx->f32_out[2], dmean_out, P * d, ddmean, P * d, S, P * d, dev, f32));
    if (want_dvar) RET_IF(store_out(ctx, st0, ctx->f32_out[3], dvar_out, P * d, ddvar, P * d, S, P * d, dev, f32));
    CUDA_TRY(ctx, cudaEventRecord(ev_d, st0));
    RET_IF(tm.end(st0, nullptr));
    for (int q = 0; q < B2GP_MAX_STREAMS; ++q) ctx->slots[q].oz_planes = 7;   // other entry points: the conservative count
    for (int64_t s = 0; s < S; ++s) info[s] = hinfo[s] != 0 ? hinfo[s] : -hinfo[S + s];
    if (cacheable) {
        auto& fc = ctx->fcache;
        if (!reuse) {
            fc.kind = kind;
            fc.N = N;
            fc.d = d;
            fc.jitter = jitter;
            fc.theta.assign(theta, theta + nth);
            fc.X.assign((const char*)Xtr, (const char*)Xtr + (size_t)N * d * (f32 ? 4 : 8));
            fc.info = hinfo[0];
            fc.U_nb = keepU ? ctx->panel : 0;
        }
        fc.valid = true;
    }

    b2gp_timing& t = ctx->last;
    float ms = 0.f;
    CUDA_TRY(ctx, cudaEventElapsedTime(&ms, ctx->ev_a, ctx->ev_b));
    t.h2d_ms = ms;
    CUDA_TRY(ctx, cudaEventElapsedTime(&ms, ev_c, ev_d));
    t.d2h_ms = ms;
    if (timing) {
        // A group's draws queue their Gram blocks one after the other, then the group's factorisation, then their
        // epilogues: the factorisation is the span from the last draw's Gram end (e1) to the first draw's epilogue start
        // (e2), counted once, with the group's last draw.  B = 1: each draw's own e1 -> e2.
        for (int64_t s = 0; s < S; ++s) {
            float a = 0, b = 0, c = 0, e = 0, f = 0;
            cudaEventElapsedTime(&a, sev[s].e[0], sev[s].e[1]);
            if ((s + 1) % B == 0 || s + 1 == S) cudaEventElapsedTime(&b, sev[s].e[1], sev[s / B * B].e[2]);
            cudaEventElapsedTime(&c, sev[s].e[2], sev[s].e[3]);
            cudaEventElapsedTime(&e, sev[s].e[3], sev[s].e[4]);
            cudaEventElapsedTime(&f, sev[s].e[4], sev[s].e[5]);
            t.gram_ms += a + c;
            t.potrf_ms += b;
            t.trsm_ms += e;
            t.epilogue_ms += f;
        }
    }
    const double n = (double)N, p = (double)P;
    t.flops = (double)S * (n * n * n / 3.0 + n * n * (p + 1.0) + 4.0 * n * p + (need_cov ? n * p * p : 0.0));
    t.gram_bytes = (double)S * (8.0 * n * n / 2.0 + 8.0 * n * p + (need_cov ? 8.0 * p * p : 0.0));
    if (G) {   // the derivative rows: their solve and row dots, and the bytes gram_dx_kernel / gram_dx_lcm_kernel write
        t.flops += (double)S * (n * n * (double)G + 4.0 * n * (double)G);
        t.gram_bytes += (double)S * 8.0 * n * (double)G;
    }
    if (timing) *timing = t;
    return B2GP_OK;
}

extern "C" int b2gp_posterior(b2gp_ctx* ctx, int kind, const double* Xtr, int64_t N, const double* yres, int64_t yres_stride,
                              const double* Xnew, int64_t P, int d, int64_t S, const double* theta, int noiseless, double jitter,
                              unsigned flags, double* mean, double* var, double* cov, const double* eps, int64_t n_samp,
                              double* y_sampled, int* info, b2gp_timing* timing) {
    return posterior_impl(ctx, kind, Xtr, 0, N, yres, yres_stride, Xnew, 0, P, d, S, theta, nullptr, 0, noiseless, jitter,
                          flags & ~(unsigned)(B2GP_OUT_DMEAN | B2GP_OUT_DVAR), mean, var, cov, eps, n_samp, y_sampled, info, timing);
}

extern "C" int b2gp_posterior_batch(b2gp_ctx* ctx, int kind, const double* Xtr, int64_t xtr_stride, int64_t N, const double* yres,
                                    int64_t yres_stride, const double* Xnew, int64_t xnew_stride, int64_t P, int d, int64_t S,
                                    const double* theta, const double* noise_vec, int64_t noise_vec_stride, int noiseless,
                                    double jitter, unsigned flags, double* mean, double* var, double* cov, const double* eps,
                                    int64_t n_samp, double* y_sampled, int* info, b2gp_timing* timing) {
    return posterior_impl(ctx, kind, Xtr, xtr_stride, N, yres, yres_stride, Xnew, xnew_stride, P, d, S, theta, noise_vec,
                          noise_vec_stride, noiseless, jitter, flags & ~(unsigned)(B2GP_OUT_DMEAN | B2GP_OUT_DVAR), mean, var, cov,
                          eps, n_samp, y_sampled, info, timing);
}

// The posterior and its gradient w.r.t. the test inputs (grad.cuh); the derivative rows share the factorisation (or the
// cached factor) with [k_pX; y^T].  fp64 arrays only, shared inputs, no covariance or samples.
extern "C" int b2gp_posterior_grad(b2gp_ctx* ctx, int kind, const double* Xtr, int64_t N, const double* yres, int64_t yres_stride,
                                   const double* Xnew, int64_t P, int d, int64_t S, const double* theta, int noiseless, double jitter,
                                   unsigned flags, double* mean, double* var, double* dmean, double* dvar, int* info,
                                   b2gp_timing* timing) {
    if (!ctx) return B2GP_ERR_ARG;
    if (flags & (B2GP_FLAG_F32 | B2GP_OUT_COV | B2GP_OUT_SAMPLE))
        return set_err(ctx, B2GP_ERR_UNSUPPORTED, "b2gp_posterior_grad", "fp64 arrays, outputs mean / var / dmean / dvar only",
                       __FILE__, __LINE__);
    ARG_CHECK(ctx, kind >= 0 && kind <= 2);
    return posterior_impl(ctx, kind, Xtr, 0, N, yres, yres_stride, Xnew, 0, P, d, S, theta, nullptr, 0, noiseless, jitter, flags, mean,
                          var, nullptr, nullptr, 0, nullptr, info, timing, dmean, dvar);
}

extern "C" int b2gp_posterior_gram(b2gp_ctx* ctx, const double* Kxx, int64_t kxx_stride, int64_t N, const double* Kpx, int64_t kpx_stride,
                                   const double* Kpp, int64_t kpp_stride, int64_t P, int64_t S, const double* yres, int64_t yres_stride,
                                   unsigned flags, double* mean, double* var, double* cov, const double* eps, int64_t n_samp,
                                   double* y_sampled, int* info, b2gp_timing* timing) {
    if (!ctx) return B2GP_ERR_ARG;
    if (f32_io(flags)) return set_err(ctx, B2GP_ERR_UNSUPPORTED, "b2gp_posterior_gram", "fp64 arrays only", __FILE__, __LINE__);
    const bool diag = flags & B2GP_FLAG_KPP_DIAG;
    ARG_CHECK(ctx, !(flags & (B2GP_OUT_DMEAN | B2GP_OUT_DVAR)));
    ARG_CHECK(ctx, !diag || !(flags & (B2GP_OUT_COV | B2GP_OUT_SAMPLE)));
    ARG_CHECK(ctx, Kxx && Kpx && N >= 1 && P >= 1);
    ARG_CHECK(ctx, Kpp || !(flags & (B2GP_OUT_VAR | B2GP_OUT_COV | B2GP_OUT_SAMPLE)));
    ARG_CHECK(ctx, kxx_stride == 0 || kxx_stride >= N * N);
    ARG_CHECK(ctx, kpx_stride == 0 || kpx_stride >= P * N);
    ARG_CHECK(ctx, kpp_stride == 0 || kpp_stride >= (diag ? P : P * P));
    const GramPost gp{Kxx, kxx_stride, Kpx, kpx_stride, Kpp, kpp_stride, diag};
    return posterior_impl(ctx, B2GP_KERNEL_RBF, nullptr, 0, N, yres, yres_stride, nullptr, 0, P, 1, S, nullptr, nullptr, 0, 0, 0.0, flags,
                          mean, var, cov, eps, n_samp, y_sampled, info, timing, nullptr, nullptr, nullptr, &gp);
}

// the common checks of the two multi-task entries: limits, host fp64 arrays, task ids in [0, T) (so that no kernel can
// index B out of bounds) -- all before any launch
static int mt_check(b2gp_ctx* ctx, const char* who, int kind, unsigned flags, int d, int group, int T, int L, const int* task1,
                    int64_t n1, const int* task2, int64_t n2) {
    if (flags & (B2GP_FLAG_DEVICE_PTRS | B2GP_FLAG_F32))
        return set_err(ctx, B2GP_ERR_UNSUPPORTED, who, "host fp64 arrays only", __FILE__, __LINE__);
    ARG_CHECK(ctx, kind >= 0 && kind <= 2);
    ARG_CHECK(ctx, T >= 1 && T <= MT_MAX_T && L >= 1 && L <= MT_MAX_L && d >= 1 && d <= MLL_MAX_D && group >= 1);
    ARG_CHECK(ctx, task1 && n1 % group == 0 && (!task2 || n2 % group == 0));
    for (int64_t i = 0; i < n1; ++i)
        if (task1[i] < 0 || task1[i] >= T) return set_err(ctx, B2GP_ERR_ARG, who, "task id outside [0, T)", __FILE__, __LINE__);
    for (int64_t i = 0; task2 && i < n2; ++i)
        if (task2[i] < 0 || task2[i] >= T) return set_err(ctx, B2GP_ERR_ARG, who, "task id outside [0, T)", __FILE__, __LINE__);
    return B2GP_OK;
}

// MultiTaskGP / CoregGP.get_mvn_posterior / predict (gp.py:253-293 with the LCM kernel, mtkernels.py:197-233): the
// posterior of b2gp_posterior with the three Gram builds and the prior variance taken from gram_lcm_kernel.
extern "C" int b2gp_posterior_multitask(b2gp_ctx* ctx, int kind, const double* Xtr, const int* task_tr, int64_t N, const double* yres,
                                        int64_t yres_stride, const double* Xnew, const int* task_new, int64_t P, int d, int group, int T,
                                        int L, int64_t S, const double* theta, const double* B, const double* noise, int noiseless,
                                        double jitter, unsigned flags, double* mean, double* var, double* cov, const double* eps,
                                        int64_t n_samp, double* y_sampled, int* info, b2gp_timing* timing) {
    if (!ctx) return B2GP_ERR_ARG;
    ARG_CHECK(ctx, B && noise && task_new && N >= 1 && P >= 1);
    RET_IF(mt_check(ctx, "b2gp_posterior_multitask", kind, flags, d, group, T, L, task_tr, N, task_new, P));
    const MtDesc mt{task_tr, task_new, group, T, L, B, noise};
    return posterior_impl(ctx, kind, Xtr, 0, N, yres, yres_stride, Xnew, 0, P, d, S, theta, nullptr, 0, noiseless, jitter,
                          flags & ~(unsigned)(B2GP_OUT_DMEAN | B2GP_OUT_DVAR), mean, var, cov, eps, n_samp, y_sampled, info, timing,
                          nullptr, nullptr, &mt);
}

// The multi-task posterior and its gradient w.r.t. the test inputs: b2gp_posterior_multitask's call with the derivative
// rows of gram_dx_lcm_kernel (mtgp.cuh) solved alongside k_pX.  Host fp64 arrays, no covariance or samples.
extern "C" int b2gp_posterior_multitask_grad(b2gp_ctx* ctx, int kind, const double* Xtr, const int* task_tr, int64_t N,
                                             const double* yres, int64_t yres_stride, const double* Xnew, const int* task_new,
                                             int64_t P, int d, int group, int T, int L, int64_t S, const double* theta,
                                             const double* B, const double* noise, int noiseless, double jitter, unsigned flags,
                                             double* mean, double* var, double* dmean, double* dvar, int* info,
                                             b2gp_timing* timing) {
    if (!ctx) return B2GP_ERR_ARG;
    if (flags & (B2GP_FLAG_F32 | B2GP_FLAG_DEVICE_PTRS | B2GP_OUT_COV | B2GP_OUT_SAMPLE))
        return set_err(ctx, B2GP_ERR_UNSUPPORTED, "b2gp_posterior_multitask_grad",
                       "host fp64 arrays, outputs mean / var / dmean / dvar only", __FILE__, __LINE__);
    ARG_CHECK(ctx, B && noise && task_new && N >= 1 && P >= 1);
    RET_IF(mt_check(ctx, "b2gp_posterior_multitask_grad", kind, flags, d, group, T, L, task_tr, N, task_new, P));
    const MtDesc mt{task_tr, task_new, group, T, L, B, noise};
    return posterior_impl(ctx, kind, Xtr, 0, N, yres, yres_stride, Xnew, 0, P, d, S, theta, nullptr, 0, noiseless, jitter, flags, mean,
                          var, nullptr, nullptr, 0, nullptr, info, timing, dmean, dvar, &mt);
}

// ------------------------------------------------------------------------------------------ sparse posterior
// out[r, c] = in[c, r]
__global__ void transpose_kernel(double* __restrict__ out, int64_t ldo, const double* __restrict__ in, int64_t ldi,
                                 int64_t rows_in, int64_t cols_in) {
    __shared__ double tile[32][33];
    const int64_t c0 = (int64_t)blockIdx.x * 32, r0 = (int64_t)blockIdx.y * 32;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int64_t r = r0 + i, c = c0 + threadIdx.x;
        tile[i][threadIdx.x] = (r < rows_in && c < cols_in) ? in[r * ldi + c] : 0.0;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int64_t r = c0 + i, c = r0 + threadIdx.x;  // out coordinates
        if (r < cols_in && c < rows_in) out[r * ldo + c] = tile[threadIdx.x][i];
    }
}

// generic <row, w> and |row|^2 reductions: dot[p] = <R[p,:], w>, nrm[p] = |R[p,:]|^2.  The draw of a batch is blockIdx.z
// (R and the non-null w, dot and nrm `bstride` doubles apart).
__global__ void __launch_bounds__(RD_THREADS)
rowdot2_kernel(const double* __restrict__ R, int64_t ld, int64_t len, const double* __restrict__ w, double wscale,
               double* __restrict__ dot, double* __restrict__ nrm, int64_t bstride) {
    __shared__ double red1[RD_THREADS / 32], red2[RD_THREADS / 32];
    const int64_t boff = (int64_t)blockIdx.z * bstride;
    if (w) w += boff;
    if (dot) dot += boff;
    if (nrm) nrm += boff;
    const double* row = R + boff + (int64_t)blockIdx.x * ld;
    double s1 = 0.0, s2 = 0.0;
    for (int64_t k = threadIdx.x; k < len; k += RD_THREADS) {
        const double v = row[k];
        if (w) s1 = fma(v, w[k], s1);
        s2 = fma(v, v, s2);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        s1 += __shfl_xor_sync(0xffffffffu, s1, o);
        s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    }
    if ((threadIdx.x & 31) == 0) {
        red1[threadIdx.x >> 5] = s1;
        red2[threadIdx.x >> 5] = s2;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double a = 0.0, b = 0.0;
        for (int i = 0; i < RD_THREADS / 32; ++i) {
            a += red1[i];
            b += red2[i];
        }
        if (dot) dot[blockIdx.x] = a * wscale;
        if (nrm) nrm[blockIdx.x] = b;
    }
}

// var[p] = kdiag - q[p] + r[p];  NaN when the factorisations failed.  kss (caller-supplied blocks): kdiag = kss[p * kss_step]
__global__ void sparse_var_kernel(double* var, double* mean, const double* q, const double* r, int64_t P, int kind, int d,
                                  const double* theta, double noise_mult, double jitter, const int* info, const int* info2,
                                  const double* kss, int64_t kss_step) {
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P) return;
    const bool bad = (*info != 0) || (*info2 != 0);
    const double nan = __longlong_as_double(0x7ff8000000000000LL);
    if (var) {
        const double kd = kss ? kss[p * kss_step] : cov_self(kind, theta[d]) + (theta[d + 1] * noise_mult + jitter);
        var[p] = bad ? nan : (kd - q[p]) + r[p];
    }
    if (mean && bad) mean[p] = nan;
}

__global__ void scale_by_inv_noise_kernel(double* v, int64_t n, const double* theta, int d) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) v[i] = v[i] / theta[d + 1];
}

// The sparse GP's Gram blocks from the caller (b2gp_sparse_elbo_gram, b2gp_sparse_posterior_gram), host arrays or
// device arrays as `dev`: Kuu [M, M], factored as (Kuu + Kuu^T) / 2 with no jitter added (the caller's Kuu holds it, as
// the reference's kernel call adds it), Kuf [M, N]; posterior only: Kus [M, P] and Kss [P, P], or its diagonal [P]
// (kss_diag).  nullptr for the entry points that build the blocks with the fused kernels.
struct SparseGram {
    const double* Kuu;
    const double* Kuf;
    const double* Kus;
    const double* Kss;
    bool kss_diag, dev;
};

// Partial Nystrom statistics of a shard of the training set (all device pointers):
//   Luu = chol(Kuu + jitter I), W = Luu^{-1} K(Xu, Xtr_shard),  Kpart = W W^T / noise (lower),  cpart = W y / noise.
// Summed over shards these are the K (before "+ I") and W D^{-1} y of sparse_gp.py:198-204.  With `sg` Kuu and Kuf are
// the caller's (dXu, dXtr, dth, kind and jitter unused); host blocks are staged through ctx->eb[10] and sl.cov.
static int sparse_partial_dev(b2gp_ctx* ctx, Slot& sl, int kind, const double* dXu, int64_t M, const double* dXtr, int64_t N,
                              const double* dy, int d, const double* dth, double jitter, double noise_h, double* Luu, int64_t ldM,
                              double* LinvU, double* Kpart, int64_t ldk, double* cpart, int* dinfo, const SparseGram* sg = nullptr) {
    cudaStream_t st = sl.stream;
    const int64_t ldN = round_up(N, 8);
    RET_IF(ensure(ctx, sl.Vt, (size_t)N * ldM * 8));
    RET_IF(ensure(ctx, sl.cov, (size_t)M * ldN * 8));
    double* Wt = (double*)sl.Vt.p;
    double* W = (double*)sl.cov.p;
    // Kuu = kernel(Xu, Xu, params, **kwargs): noise defaults to 0, so the diagonal gets jitter only (sparse_gp.py:193)
    if (sg)
        RET_IF(gram_copyin(ctx, st, ctx->eb[10], sg->Kuu, M, M, sg->dev, Luu, ldM));
    else
        RET_IF(launch_gram(ctx, st, kind, dXu, M, dXu, M, d, dth, 0.0, jitter, 1, 1, Luu, ldM));
    RET_IF(potrf_auto(ctx, st, Luu, ldM, M, 0, LinvU, dinfo));                                  // sparse_gp.py:194
    // W^T = K_fu Luu^{-T}  (W = Luu^{-1} Kuf, sparse_gp.py:195-197), one training point per row
    if (sg) {   // Kuf^T; a host Kuf is staged in W, which is written only after the solve
        const double* src = sg->Kuf;
        int64_t lds = N;
        if (!sg->dev) {
            CUDA_TRY(ctx, cudaMemcpy2DAsync(W, (size_t)ldN * 8, sg->Kuf, (size_t)N * 8, (size_t)N * 8, (size_t)M, cudaMemcpyHostToDevice, st));
            src = W;
            lds = ldN;
        }
        RET_IF(launch(ctx, st, dim3((unsigned)ceil_div(N, 32), (unsigned)ceil_div(M, 32)), dim3(32, 8), 0, transpose_kernel, Wt, ldM, src, lds,
                      M, N));
    } else {
        RET_IF(launch_gram(ctx, st, kind, dXtr, N, dXu, M, d, dth, 0.0, 0.0, 0, 0, Wt, ldM));
    }
    RET_IF(trsm_rec(ctx, st, Wt, ldM, N, Luu, ldM, M, LinvU));   // tall right-hand sides: int8 panel GEMMs (potrf.cuh)
    RET_IF(launch(ctx, st, dim3((unsigned)ceil_div(M, 32), (unsigned)ceil_div(N, 32)), dim3(32, 8), 0, transpose_kernel, W, ldN, Wt, ldM, N, M));
    // W D^{-1} W^T with D = noise * 1  (sparse_gp.py:198-199).  Accumulated onto a zeroed matrix (beta = 1) so that the
    // product -- M^2 N flops, the bulk of the sparse posterior -- qualifies for the int8 wgmma path (k = N is split into
    // launches of <= 16384 by the dispatcher)
    CUDA_TRY(ctx, cudaMemsetAsync(Kpart, 0, (size_t)M * ldk * 8, st));
    RET_IF(gemm_nt(ctx, st, M, M, N, 1.0 / noise_h, W, ldN, W, ldN, 1.0, Kpart, ldk, true));
    // W D^{-1} y  (sparse_gp.py:203-204)
    return launch(ctx, st, (unsigned)M, RD_THREADS, 0, rowdot2_kernel, W, ldN, N, dy, 1.0 / noise_h, cpart, nullptr, (int64_t)0);
}

// Posterior from the summed statistics: K = Ksum + I, L = chol(K), then sparse_gp.py:206-217.  With `sg` Kus and Kss
// are the caller's (dXu, dXnew, dth, kind, noiseless and jitter unused: noise_p is inside Kss); host blocks are staged
// through ctx->eb[10] (Kus) and ctx->eb[11] (Kss).
static int sparse_finish_dev(b2gp_ctx* ctx, Slot& sl, int kind, const double* dXu, int64_t M, const double* Luu, int64_t ldM,
                             const double* LinvU, double* Kmat, int64_t ldk, double* LinvK, const double* cvec,
                             const double* dXnew, int64_t P, int d, const double* dth, int noiseless, double jitter,
                             bool want_var, bool want_cov, double* dmean, double* dvar, double* C, int64_t ldc, int* dinfo,
                             const SparseGram* sg = nullptr) {
    cudaStream_t st = sl.stream;
    RET_IF(ensure(ctx, sl.LinvC, (size_t)2 * (P + 1) * ldM * 8));
    RET_IF(ensure(ctx, sl.misc, (size_t)(2 * P + 16) * 8));
    double* Wst = (double*)sl.LinvC.p;          // P x ldM          Ws^T = K_su Luu^{-T}
    double* R = Wst + (P + 1) * ldM;            // (P+1) x ldM      rows 0..P-1: (L^{-1} Ws)^T; row P: L^{-1} c
    double* qv = (double*)sl.misc.p;            // |Ws^T[p]|^2
    double* rv = qv + P;                        // |R[p]|^2
    RET_IF(launch(ctx, st, grid_for(M), 256, 0, add_diag_kernel, Kmat, ldk, M, 1.0));           // sparse_gp.py:200
    RET_IF(potrf_auto(ctx, st, Kmat, ldk, M, 0, LinvK, dinfo + 1));                             // sparse_gp.py:201
    // Ws^T = K_su Luu^{-T}  (sparse_gp.py:206-207)
    const double* kss = nullptr;   // caller-supplied Kss on the device
    if (sg) {
        const double* kus = sg->Kus;
        if (!sg->dev) {
            RET_IF(ensure(ctx, ctx->eb[10], (size_t)M * P * 8));
            CUDA_TRY(ctx, cudaMemcpyAsync(ctx->eb[10].p, sg->Kus, (size_t)M * P * 8, cudaMemcpyHostToDevice, st));
            kus = (const double*)ctx->eb[10].p;
        }
        RET_IF(launch(ctx, st, dim3((unsigned)ceil_div(P, 32), (unsigned)ceil_div(M, 32)), dim3(32, 8), 0, transpose_kernel, Wst, ldM, kus,
                      P, M, P));
        kss = sg->Kss;
        if (kss && !sg->dev) {
            const size_t n = sg->kss_diag ? (size_t)P : (size_t)P * P;
            RET_IF(ensure(ctx, ctx->eb[11], n * 8));
            CUDA_TRY(ctx, cudaMemcpyAsync(ctx->eb[11].p, sg->Kss, n * 8, cudaMemcpyHostToDevice, st));
            kss = (const double*)ctx->eb[11].p;
        }
    } else {
        RET_IF(launch_gram(ctx, st, kind, dXnew, P, dXu, M, d, dth, 0.0, 0.0, 0, 0, Wst, ldM));
    }
    RET_IF(trsm_rec(ctx, st, Wst, ldM, P, Luu, ldM, M, LinvU));
    // pack = [c | Ws]; L^{-1} pack  (sparse_gp.py:208-212)
    RET_IF(launch(ctx, st, grid_for(P * M), 256, 0, copy2d_kernel, R, ldM, Wst, ldM, P, M));
    CUDA_TRY(ctx, cudaMemcpyAsync(R + P * ldM, cvec, (size_t)M * 8, cudaMemcpyDeviceToDevice, st));
    RET_IF(trsm_rec(ctx, st, R, ldM, P + 1, Kmat, ldk, M, LinvK));
    // mean = (L^{-1} c)^T (L^{-1} Ws)  (sparse_gp.py:213)
    RET_IF(launch(ctx, st, (unsigned)P, RD_THREADS, 0, rowdot2_kernel, R, ldM, M, R + P * ldM, 1.0, dmean, rv, (int64_t)0));
    RET_IF(launch(ctx, st, (unsigned)P, RD_THREADS, 0, rowdot2_kernel, Wst, ldM, M, nullptr, 1.0, nullptr, qv, (int64_t)0));
    RET_IF(launch(ctx, st, grid_for(P), 256, 0, sparse_var_kernel, want_var ? dvar : nullptr, dmean, qv, rv, P, kind, d, dth,
                  noiseless ? 0.0 : 1.0, jitter, dinfo, dinfo + 1, kss, (sg && !sg->kss_diag) ? P + 1 : (int64_t)1));
    if (want_cov) {
        // cov = Kss - Ws^T Ws + (L^{-1}Ws)^T (L^{-1}Ws)  (sparse_gp.py:215-217)
        if (sg)   // the lower triangle of (Kss + Kss^T) / 2
            RET_IF(launch(ctx, st, dim3((unsigned)ceil_div(P, (int64_t)GCOPY_TILE), (unsigned)ceil_div(P, (int64_t)GCOPY_TILE)),
                          dim3(GCOPY_TILE, 8), 0, gram_copyin_kernel, kss, P, P, C, ldc));
        else
            RET_IF(launch_gram(ctx, st, kind, dXnew, P, dXnew, P, d, dth, noiseless ? 0.0 : 1.0, jitter, 1, 1, C, ldc));
        RET_IF(gemm_nt(ctx, st, P, P, M, -1.0, Wst, ldM, Wst, ldM, 1.0, C, ldc, true));
        RET_IF(gemm_nt(ctx, st, P, P, M, 1.0, R, ldM, R, ldM, 1.0, C, ldc, true));
        RET_IF(launch(ctx, st, dim3((unsigned)ceil_div(P, 32), (unsigned)ceil_div(P, 32)), dim3(32, 32), 0, mirror_lower_kernel, C, ldc, P));
        RET_IF(launch(ctx, st, grid_for(P * P), 256, 0, nan_if_bad_kernel, C, ldc, P, P, dinfo, dinfo + 1));
    }
    return B2GP_OK;
}

// b2gp_sparse_posterior; with `sg` (b2gp_sparse_posterior_gram) the blocks are the caller's and the noise is `noise_g`
// (Xu, Xtr, Xnew, theta, kind, d, noiseless and jitter unused)
static int sparse_posterior_impl(b2gp_ctx* ctx, int kind, const double* Xu, int64_t M, const double* Xtr, int64_t N,
                                 const double* yres, const double* Xnew, int64_t P, int d, const double* theta, int noiseless,
                                 double jitter, unsigned flags, double* mean, double* var, double* cov, int* info,
                                 b2gp_timing* timing, double noise_g = 0.0, const SparseGram* sg = nullptr) {
    if (!ctx) return B2GP_ERR_ARG;
    ARG_CHECK(ctx, kind >= 0 && kind <= 2);
    ARG_CHECK(ctx, (sg || (Xu && Xtr && Xnew && theta)) && yres && info);
    ARG_CHECK(ctx, M >= 1 && N >= 1 && P >= 1 && d >= 1 && d <= GRAM_MAX_D);
    const bool want_mean = flags & B2GP_OUT_MEAN, want_var = flags & B2GP_OUT_VAR, want_cov = flags & B2GP_OUT_COV;
    ARG_CHECK(ctx, !want_mean || mean);
    ARG_CHECK(ctx, !want_var || var);
    ARG_CHECK(ctx, !want_cov || cov);
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    const bool dev = dev_ptrs(flags), f32 = f32_io(flags);
    Slot& sl = ctx->slots[0];
    cudaStream_t st = sl.stream;
    ctx->fcache.valid = false;
    CallTimer tm(ctx);
    RET_IF(tm.begin(st));
    const int nth = d + 3;
    const double *dXu = nullptr, *dXtr = nullptr, *dy, *dXnew = nullptr, *dth = nullptr;
    RET_IF(stage_in_t(ctx, st, ctx->d_in[1], ctx->f32_in[1], yres, (size_t)N, dev, f32, &dy));
    if (!sg) {
        RET_IF(stage_in_t(ctx, st, ctx->d_in[0], ctx->f32_in[0], Xtr, (size_t)N * d, dev, f32, &dXtr));
        RET_IF(stage_in_t(ctx, st, ctx->d_in[2], ctx->f32_in[2], Xnew, (size_t)P * d, dev, f32, &dXnew));
        RET_IF(stage_in(ctx, st, ctx->d_in[3], theta, (size_t)nth * 8, dev, &dth));
        RET_IF(stage_in_t(ctx, st, ctx->d_in[5], ctx->f32_in[5], Xu, (size_t)M * d, dev, f32, &dXu));
    }
    double noise_h = 0.0;
    if (sg) {
        noise_h = noise_g;
    } else if (dev) {
        CUDA_TRY(ctx, cudaMemcpyAsync(&noise_h, dth + d + 1, 8, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(ctx, cudaStreamSynchronize(st));
    } else {
        noise_h = theta[d + 1];
    }
    const int64_t ldM = round_up(M, 8), ldC = round_up(P, 8);
    double *slA = nullptr, *slLinv = nullptr;   // slot 0's matrix and inverted diagonal blocks
    RET_IF(slot0_buffers(ctx, (size_t)2 * M * ldM * 8, (size_t)2 * linv_bytes(M), &slA, &slLinv));
    RET_IF(ensure(ctx, ctx->d_out[0], (size_t)(2 * P + M + 16) * 8));
    if (want_cov && (!dev || f32)) RET_IF(ensure(ctx, ctx->d_out[2], (size_t)P * ldC * 8));
    RET_IF(ensure(ctx, ctx->d_info, 64));
    int* dinfo = (int*)ctx->d_info.p;
    CUDA_TRY(ctx, cudaMemsetAsync(dinfo, 0, 16, st));
    double* Luu = slA;
    double* Kmat = Luu + M * ldM;
    double* LinvU = slLinv;
    double* LinvK = LinvU + linv_bytes(M) / 8;
    double* mv = (double*)ctx->d_out[0].p;
    double* vv = mv + P;
    double* cvec = vv + P;
    RET_IF(sparse_partial_dev(ctx, sl, kind, dXu, M, dXtr, N, dy, d, dth, jitter, noise_h, Luu, ldM, LinvU, Kmat, ldM, cvec, dinfo, sg));
    const bool direct = dev && !f32;     // results written straight into the caller's (device, fp64) arrays
    double* dmean = (want_mean && direct) ? mean : mv;
    double* dvar = (want_var && direct) ? var : vv;
    double* C = direct ? cov : (double*)ctx->d_out[2].p;
    const int64_t ldc = direct ? P : ldC;
    RET_IF(sparse_finish_dev(ctx, sl, kind, dXu, M, Luu, ldM, LinvU, Kmat, ldM, LinvK, cvec, dXnew, P, d, dth, noiseless, jitter,
                             want_var, want_cov, dmean, dvar, C, ldc, dinfo, sg));
    if (want_cov) RET_IF(store_out(ctx, st, ctx->f32_out[2], cov, P, C, ldc, P, P, dev, f32));
    int hinfo[2] = {0, 0};
    CUDA_TRY(ctx, cudaMemcpyAsync(hinfo, dinfo, 2 * sizeof(int), cudaMemcpyDeviceToHost, st));
    if (want_mean) RET_IF(store_out(ctx, st, ctx->f32_out[0], mean, P, dmean, P, 1, P, dev, f32));
    if (want_var) RET_IF(store_out(ctx, st, ctx->f32_out[1], var, P, dvar, P, 1, P, dev, f32));
    RET_IF(tm.end(st, nullptr));
    info[0] = hinfo[0] != 0 ? hinfo[0] : -hinfo[1];
    const double m = (double)M, n = (double)N, p = (double)P;
    ctx->last.flops = 2.0 * m * m * m / 3.0 + 2.0 * m * m * n + 2.0 * m * m * (p + 1.0) + (want_cov ? 2.0 * m * p * p : 0.0);
    ctx->last.gram_bytes = 8.0 * (m * n + m * m / 2.0 + m * p);
    if (timing) *timing = ctx->last;
    return B2GP_OK;
}

extern "C" int b2gp_sparse_posterior(b2gp_ctx* ctx, int kind, const double* Xu, int64_t M, const double* Xtr, int64_t N,
                                     const double* yres, const double* Xnew, int64_t P, int d, const double* theta, int noiseless,
                                     double jitter, unsigned flags, double* mean, double* var, double* cov, int* info,
                                     b2gp_timing* timing) {
    return sparse_posterior_impl(ctx, kind, Xu, M, Xtr, N, yres, Xnew, P, d, theta, noiseless, jitter, flags, mean, var, cov, info, timing);
}

extern "C" int b2gp_sparse_posterior_gram(b2gp_ctx* ctx, const double* Kuu, int64_t M, const double* Kuf, int64_t N, const double* yres,
                                          double noise, const double* Kus, const double* Kss, int64_t P, unsigned flags, double* mean,
                                          double* var, double* cov, int* info, b2gp_timing* timing) {
    if (!ctx) return B2GP_ERR_ARG;
    if (f32_io(flags)) return set_err(ctx, B2GP_ERR_UNSUPPORTED, "b2gp_sparse_posterior_gram", "fp64 arrays only", __FILE__, __LINE__);
    const bool kss_diag = flags & B2GP_FLAG_KPP_DIAG;
    ARG_CHECK(ctx, !(kss_diag && (flags & B2GP_OUT_COV)));
    ARG_CHECK(ctx, Kss || !(flags & (B2GP_OUT_VAR | B2GP_OUT_COV)));
    ARG_CHECK(ctx, Kuu && Kuf && Kus);
    const SparseGram sg{Kuu, Kuf, Kus, Kss, kss_diag, dev_ptrs(flags)};
    return sparse_posterior_impl(ctx, B2GP_KERNEL_RBF, nullptr, M, nullptr, N, yres, nullptr, P, 1, nullptr, 0, 0.0, flags, mean, var, cov,
                                 info, timing, noise, &sg);
}

// ---- sharded sparse path (SURVEY.md section 8e, "N-sharded sparse GP"): each rank calls _partial on its shard of
// the training set, the M x M matrix and the M-vector are summed across ranks (NCCL all-reduce by the caller),
// every rank calls _finish.  All array pointers are DEVICE pointers; theta is a HOST pointer (d+3 values).
extern "C" int b2gp_sparse_partial(b2gp_ctx* ctx, int kind, const double* Xu, int64_t M, const double* Xtr, int64_t N,
                                   const double* yres, int d, const double* theta, double jitter, double* Kpart, int64_t ldk,
                                   double* cpart, int* info) {
    if (!ctx) return B2GP_ERR_ARG;
    ARG_CHECK(ctx, kind >= 0 && kind <= 2);
    ARG_CHECK(ctx, Xu && Xtr && yres && theta && Kpart && cpart && info);
    ARG_CHECK(ctx, M >= 1 && N >= 1 && d >= 1 && d <= GRAM_MAX_D && ldk >= M);
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    ctx->fcache.valid = false;
    Slot& sl = ctx->slots[0];
    cudaStream_t st = sl.stream;
    CallTimer tm(ctx);
    RET_IF(tm.begin(st));
    const double* dth;
    RET_IF(stage_in(ctx, st, ctx->d_in[3], theta, (size_t)(d + 3) * 8, false, &dth));
    const int64_t ldM = round_up(M, 8);
    double *slA = nullptr, *slLinv = nullptr;   // slot 0's matrix and inverted diagonal blocks
    RET_IF(slot0_buffers(ctx, (size_t)2 * M * ldM * 8, (size_t)2 * linv_bytes(M), &slA, &slLinv));
    RET_IF(ensure(ctx, ctx->d_info, 64));
    int* dinfo = (int*)ctx->d_info.p;
    CUDA_TRY(ctx, cudaMemsetAsync(dinfo, 0, 16, st));
    RET_IF(sparse_partial_dev(ctx, sl, kind, Xu, M, Xtr, N, yres, d, dth, jitter, theta[d + 1], slA, ldM,
                              slLinv, Kpart, ldk, cpart, dinfo));
    CUDA_TRY(ctx, cudaMemcpyAsync(info, dinfo, sizeof(int), cudaMemcpyDeviceToHost, st));
    return tm.end(st, nullptr);
}

extern "C" int b2gp_sparse_finish(b2gp_ctx* ctx, int kind, const double* Xu, int64_t M, double* Ksum, int64_t ldk,
                                  const double* csum, const double* Xnew, int64_t P, int d, const double* theta, int noiseless,
                                  double jitter, unsigned flags, double* mean, double* var, double* cov, int* info) {
    if (!ctx) return B2GP_ERR_ARG;
    ARG_CHECK(ctx, kind >= 0 && kind <= 2);
    ARG_CHECK(ctx, Xu && Ksum && csum && Xnew && theta && mean && info);
    ARG_CHECK(ctx, M >= 1 && P >= 1 && d >= 1 && d <= GRAM_MAX_D && ldk >= M);
    const bool want_var = flags & B2GP_OUT_VAR, want_cov = flags & B2GP_OUT_COV;
    ARG_CHECK(ctx, !want_var || var);
    ARG_CHECK(ctx, !want_cov || cov);
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    ctx->fcache.valid = false;
    Slot& sl = ctx->slots[0];
    cudaStream_t st = sl.stream;
    CallTimer tm(ctx);
    RET_IF(tm.begin(st));
    const double* dth;
    RET_IF(stage_in(ctx, st, ctx->d_in[3], theta, (size_t)(d + 3) * 8, false, &dth));
    const int64_t ldM = round_up(M, 8);
    double *slA = nullptr, *slLinv = nullptr;   // slot 0's matrix and inverted diagonal blocks
    RET_IF(slot0_buffers(ctx, (size_t)2 * M * ldM * 8, (size_t)2 * linv_bytes(M), &slA, &slLinv));
    RET_IF(ensure(ctx, ctx->d_info, 64));
    int* dinfo = (int*)ctx->d_info.p;
    CUDA_TRY(ctx, cudaMemsetAsync(dinfo, 0, 16, st));
    double* Luu = slA;
    double* LinvU = slLinv;
    double* LinvK = LinvU + linv_bytes(M) / 8;
    // Luu is rebuilt here (M^3/3 flops) so that _finish does not depend on ctx state left by _partial
    RET_IF(launch_gram(ctx, st, kind, Xu, M, Xu, M, d, dth, 0.0, jitter, 1, 1, Luu, ldM));
    RET_IF(potrf_rec(ctx, st, Luu, ldM, M, LinvU, dinfo, 0));
    RET_IF(sparse_finish_dev(ctx, sl, kind, Xu, M, Luu, ldM, LinvU, Ksum, ldk, LinvK, csum, Xnew, P, d, dth, noiseless, jitter,
                             want_var, want_cov, mean, var, cov, P, dinfo));
    int hinfo[2] = {0, 0};
    CUDA_TRY(ctx, cudaMemcpyAsync(hinfo, dinfo, 2 * sizeof(int), cudaMemcpyDeviceToHost, st));
    RET_IF(tm.end(st, nullptr));
    info[0] = hinfo[0] != 0 ? hinfo[0] : -hinfo[1];
    return B2GP_OK;
}

// ---- building blocks of the block-cyclic multi-GPU factorisation (device pointers only)
// Factor an n x n block and export its inverted 128x128 diagonal blocks (ceil(n/128) * 128*128 doubles) to Linv_out.
extern "C" int b2gp_potrf_inv(b2gp_ctx* ctx, int64_t n, double* A, int64_t lda, double* Linv_out, int* info) {
    if (!ctx) return B2GP_ERR_ARG;
    ARG_CHECK(ctx, A && Linv_out && info && n >= 1 && lda >= n);
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->slots[0].stream;
    CallTimer tm(ctx);
    RET_IF(tm.begin(st));
    RET_IF(ensure(ctx, ctx->d_info, 64));
    CUDA_TRY(ctx, cudaMemsetAsync(ctx->d_info.p, 0, 8, st));
    RET_IF(potrf_rec(ctx, st, A, lda, n, Linv_out, (int*)ctx->d_info.p, 0));
    CUDA_TRY(ctx, cudaMemcpyAsync(info, ctx->d_info.p, sizeof(int), cudaMemcpyDeviceToHost, st));
    return tm.end(st, nullptr);
}

// B (nrhs rows of length n) <- B L^{-T} with the inverted diagonal blocks supplied by the caller
extern "C" int b2gp_trsm_inv(b2gp_ctx* ctx, int64_t n, int64_t nrhs, const double* L, int64_t ldl, const double* Linv,
                             double* B, int64_t ldb) {
    if (!ctx) return B2GP_ERR_ARG;
    ARG_CHECK(ctx, L && Linv && B && n >= 1 && nrhs >= 0 && ldl >= n && ldb >= n);
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->slots[0].stream;
    CallTimer tm(ctx);
    RET_IF(tm.begin(st));
    RET_IF(trsm_rec(ctx, st, B, ldb, nrhs, L, ldl, n, Linv));
    return tm.end(st, nullptr);
}

// dot[r] (+)= scale * <R[r, 0:len), w>,  nrm[r] (+)= |R[r, 0:len)|^2   (either output may be NULL)
__global__ void accumulate_kernel(double* dst, const double* src, int64_t n, int accumulate) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = accumulate ? dst[i] + src[i] : src[i];
}
extern "C" int b2gp_rowdot(b2gp_ctx* ctx, int64_t rows, int64_t len, const double* R, int64_t ldr, const double* w,
                           double scale, double* dot, double* nrm, int accumulate) {
    if (!ctx) return B2GP_ERR_ARG;
    ARG_CHECK(ctx, R && rows >= 0 && len >= 0 && ldr >= len && (dot == nullptr || w != nullptr));
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->slots[0].stream;
    CallTimer tm(ctx);
    RET_IF(tm.begin(st));
    if (rows > 0) {
        RET_IF(ensure(ctx, ctx->slots[0].misc, (size_t)(2 * rows + 16) * 8));
        double* t1 = (double*)ctx->slots[0].misc.p;
        double* t2 = t1 + rows;
        RET_IF(launch(ctx, st, (unsigned)rows, RD_THREADS, 0, rowdot2_kernel, R, ldr, len, w, scale, dot ? t1 : nullptr, nrm ? t2 : nullptr, (int64_t)0));
        if (dot) RET_IF(launch(ctx, st, grid_for(rows), 256, 0, accumulate_kernel, dot, t1, rows, accumulate));
        if (nrm) RET_IF(launch(ctx, st, grid_for(rows), 256, 0, accumulate_kernel, nrm, t2, rows, accumulate));
    }
    return tm.end(st, nullptr);
}

extern "C" int b2gp_copy2d(b2gp_ctx* ctx, double* dst, int64_t ldd, const double* src, int64_t lds, int64_t rows, int64_t cols) {
    if (!ctx) return B2GP_ERR_ARG;
    ARG_CHECK(ctx, dst && src && rows >= 0 && cols >= 0 && ldd >= cols && lds >= cols);
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->slots[0].stream;
    if (rows && cols)
        CUDA_TRY(ctx, cudaMemcpy2DAsync(dst, (size_t)ldd * 8, src, (size_t)lds * 8, (size_t)cols * 8, (size_t)rows,
                                        cudaMemcpyDeviceToDevice, st));
    CUDA_TRY(ctx, cudaStreamSynchronize(st));
    return B2GP_OK;
}

// ------------------------------------------------------------------------------------------ fit side
// value and gradient (w.r.t. log lengthscale[d], log k_scale, log noise, log period) of the exact-GP log marginal
// likelihood -- see mll.cuh.  X[N,d], yres[N] host or device pointers (flags); theta is a HOST pointer (d+3);
// value, grad[d+3] and the optional alpha[N] = K^{-1} yres are HOST outputs.
// g[i] = 1/2 (alpha_i^2 - Kinv_ii): d log N(y; 0, K) / d K_ii, the gradient w.r.t. a per-point noise variance; the draw
// of a batch is blockIdx.z (every operand `bstride` doubles apart)
__global__ void mll_diag_grad_kernel(const double* __restrict__ alpha, const double* __restrict__ Kinv, int64_t ldk, int64_t n,
                                     double* __restrict__ g, int64_t bstride) {
    alpha += (int64_t)blockIdx.z * bstride;
    Kinv += (int64_t)blockIdx.z * bstride;
    g += (int64_t)blockIdx.z * bstride;
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) g[i] = 0.5 * (alpha[i] * alpha[i] - Kinv[i * ldk + i]);
}

// b2gp_mll_gram: K and its derivatives dK_j come from the caller instead of the fused Gram build and gradient reduction.
// K (leading dimension ldk) and every dK[j] (lddk) follow `flags`; dK is a host array of p pointers.
struct GramMll {
    const double* K;
    int64_t ldk;
    const double* const* dK;
    int64_t lddk, p;
};

// gout[j] = 1/2 sum_{a,b} W_ab dK_j[a, b] (mll_gram_trace_kernel, then the fixed-order column sums of mll_lcm_finish_kernel).
// Device dK: one launch over all p.  Host dK: streamed through the two N x ld buffers buf0 / buf1 -- the copy of dK_{j+1} on
// a second stream overlaps the reduction of dK_j, and the copy into a buffer waits for the reduction that last read it.
// `dptrs` is device scratch for max(p, 2) pointers.
static int mll_gram_trace(b2gp_ctx* ctx, cudaStream_t st, const GramMll& gm, bool dev, int tiles, const double* alpha,
                          const double* Kinv, int64_t ld, int64_t N, double* buf0, double* buf1, const double** dptrs, double* partial,
                          double* gout) {
    const int p = (int)gm.p;
    const dim3 grid((unsigned)tiles, (unsigned)tiles);
    count_path(ctx, (int)PATH_MLL_GRAM_TRACE);
    if (dev) {
        CUDA_TRY(ctx, cudaMemcpyAsync(dptrs, gm.dK, (size_t)p * sizeof(double*), cudaMemcpyHostToDevice, st));
        RET_IF(launch(ctx, st, grid, MLL_THREADS, 0, mll_gram_trace_kernel, alpha, Kinv, ld, N, (const double* const*)dptrs, gm.lddk, p, 0,
                      p, partial));
    } else {
        const double* bufs[2] = {buf0, buf1};
        CUDA_TRY(ctx, cudaMemcpyAsync(dptrs, bufs, sizeof bufs, cudaMemcpyHostToDevice, st));
        cudaStream_t cs = ctx->slots[1].stream;
        cudaEvent_t free_ev = ctx->pool.get(), cp[2] = {ctx->pool.get(), ctx->pool.get()}, red[2] = {ctx->pool.get(), ctx->pool.get()};
        ARG_CHECK(ctx, free_ev && cp[0] && cp[1] && red[0] && red[1]);
        CUDA_TRY(ctx, cudaEventRecord(free_ev, st));   // everything before (L^{-T} in buf0, the factor in buf1) is done with
        CUDA_TRY(ctx, cudaStreamWaitEvent(cs, free_ev, 0));
        for (int j = 0; j < p; ++j) {
            const int b = j & 1;
            if (j >= 2) CUDA_TRY(ctx, cudaStreamWaitEvent(cs, red[b], 0));
            CUDA_TRY(ctx, cudaMemcpy2DAsync((void*)bufs[b], (size_t)ld * 8, gm.dK[j], (size_t)gm.lddk * 8, (size_t)N * 8, (size_t)N,
                                            cudaMemcpyHostToDevice, cs));
            CUDA_TRY(ctx, cudaEventRecord(cp[b], cs));
            CUDA_TRY(ctx, cudaStreamWaitEvent(st, cp[b], 0));
            RET_IF(launch(ctx, st, grid, MLL_THREADS, 0, mll_gram_trace_kernel, alpha, Kinv, ld, N, (const double* const*)(dptrs + b), ld, 1, j,
                          p, partial));
            CUDA_TRY(ctx, cudaEventRecord(red[b], st));
        }
    }
    return launch(ctx, st, (unsigned)p, MLL_FIN_THREADS, 0, mll_lcm_finish_kernel, (const double*)partial, (int64_t)tiles * tiles, p, gout, (int64_t)0);
}

static int mll_impl(b2gp_ctx* ctx, int kind, const double* X, int64_t N, const double* yres, int d, const double* theta,
                    const double* noise_vec, double jitter, unsigned flags, double* value, double* grad, double* alpha_out,
                    double* grad_noise_vec, int* info, const MtDesc* mt = nullptr, double* grad_x_dev = nullptr,
                    const GramMll* gm = nullptr) {
    if (!ctx) return B2GP_ERR_ARG;
    ARG_CHECK(ctx, !grad_noise_vec || grad);
    ARG_CHECK(ctx, !gm || (!mt && !noise_vec && !grad_x_dev && kind == B2GP_KERNEL_RBF));
    ARG_CHECK(ctx, !grad_x_dev || (grad && !noise_vec && (!mt || kind != B2GP_KERNEL_PERIODIC)));
    ARG_CHECK(ctx, kind >= 0 && kind <= B2GP_KERNEL_NNGP_RELU);
    // NNGP: single task, no input gradient; no per-feature accumulator, so the Gram build's d <= 64 is the limit
    const bool nngp = is_nngp(kind);
    ARG_CHECK(ctx, !nngp || (!mt && !grad_x_dev));
    ARG_CHECK(ctx, (gm || (X && theta)) && yres && value && info);
    ARG_CHECK(ctx, N >= 1 && d >= 1 && d <= (nngp ? GRAM_MAX_D : MLL_MAX_D));
    if (nngp) RET_IF(nngp_check_depth(ctx, "b2gp_mll", theta[0]));
    const int depth = nngp ? (int)theta[0] : 0;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    ctx->fcache.valid = false;
    const bool dev = dev_ptrs(flags);
    Slot& sl = ctx->slots[0];
    cudaStream_t st = sl.stream;
    CallTimer tm(ctx);
    RET_IF(tm.begin(st));
    // multi-task: theta [L, d+2]; the gradient is [L, d+2] | [L, T, T] | [T] and the per-block partial sums of
    // mll_lcm_grad_kernel are nout wide, L blocks of tiles^2
    const int T = mt ? mt->T : 0, L = mt ? mt->L : 0;
    const int nth = mt ? L * (d + 2) : d + 3;
    const int ngrad = gm ? (int)gm->p : mt ? L * (d + 2) + L * T * T + T : nth, nout = d + 2 + T * T + T;
    const double *dX, *dy, *dth, *dnv = nullptr, *dmt = nullptr;
    const int* dtask = nullptr;
    std::vector<double> hmt;
    RET_IF(stage_in(ctx, st, ctx->d_in[0], X, (size_t)N * d * 8, dev, &dX));
    RET_IF(stage_in(ctx, st, ctx->d_in[1], yres, (size_t)N * 8, dev, &dy));
    RET_IF(stage_in(ctx, st, ctx->d_in[3], gm ? nullptr : theta, (size_t)nth * 8, false, &dth));
    if (noise_vec) RET_IF(stage_in(ctx, st, ctx->d_in[6], noise_vec, (size_t)N * 8, dev, &dnv));
    if (mt) {
        hmt.resize((size_t)L * T * T + T);
        memcpy(hmt.data(), mt->B, (size_t)L * T * T * 8);
        memcpy(hmt.data() + (size_t)L * T * T, mt->noise, (size_t)T * 8);
        RET_IF(stage_in(ctx, st, ctx->d_in[5], hmt.data(), hmt.size() * 8, false, &dmt));
        const double* dt = nullptr;
        RET_IF(stage_in(ctx, st, ctx->d_in[7], mt->task_tr, (size_t)N * 4, false, &dt));
        dtask = (const int*)dt;
    }
    const int64_t ld = round_up(N, 8);
    const int64_t tiles = ceil_div(N, MLL_TILE);
    double *slA = nullptr, *slLinv = nullptr;   // slot 0's matrix and inverted diagonal blocks
    RET_IF(slot0_buffers(ctx, (size_t)(N + 1) * ld * 8, (size_t)linv_bytes(N), &slA, &slLinv));
    RET_IF(ensure(ctx, ctx->d_info, 64));
    if (mt)
        RET_IF(ensure(ctx, sl.misc, (size_t)(3 * ld + 64 + L * tiles * tiles * nout + L * nout) * 8));
    else if (nngp)   // partials [tiles^2, 3] | self-chains [N, depth, 3]
        RET_IF(ensure(ctx, sl.misc, (size_t)(3 * ld + 64 + tiles * tiles * 3 + N * depth * 3) * 8));
    else if (gm)   // partials [tiles^2, p] | grad [p] | the device array of dK pointers [max(p, 2)]
        RET_IF(ensure(ctx, sl.misc, (size_t)(3 * ld + 64 + (tiles * tiles + 2) * gm->p + 2) * 8));
    else
        RET_IF(ensure(ctx, sl.misc, (size_t)(3 * ld + 64 + tiles * tiles * nth) * 8));
    int* dinfo = (int*)ctx->d_info.p;
    CUDA_TRY(ctx, cudaMemsetAsync(dinfo, 0, 8, st));
    double* A = slA;
    double* Linv = slLinv;
    double* w = A + N * ld;              // y rides under K as a right-hand-side row: L^{-1} y after the factorisation
    double* alpha = (double*)sl.misc.p + ld;   // K^{-1} y
    double* sc = alpha + ld;             // [0] sum log L_ii, [1] |w|^2, [8..8+nth) grad
    double* partial = sc + 64;
    double* gmt = partial + (size_t)L * tiles * tiles * nout;   // multi-task: per-latent column sums of the partials
    double* gdev = nullptr;              // caller-Gram mode: the gradient [p]
    if (gm)   // K staged through sl.cov, which takes L^{-T} only after the factorisation
        RET_IF(gram_copyin(ctx, st, sl.cov, gm->K, gm->ldk, N, dev, A, ld));
    else if (mt)
        RET_IF(launch_gram_lcm(ctx, st, LCM_LOWER, kind, dX, dtask, N, dX, dtask, N, d, T, L, mt->group, dth, dmt, dmt + (size_t)L * T * T, 1.0,
                               jitter, A, ld));
    else
        RET_IF(launch_gram(ctx, st, kind, dX, N, dX, N, d, dth, 1.0, jitter, 1, 1, A, ld));
    if (dnv)   // k + diag(measured_noise) / k + diag(exp(log_var)): mngp.py:96, hskgp.py:147
        RET_IF(launch(ctx, st, grid_for(N), 256, 0, add_diag_vec_kernel, A, ld, N, dnv, (int64_t)0, (int64_t)0));
    CUDA_TRY(ctx, cudaMemcpyAsync(w, dy, (size_t)N * 8, cudaMemcpyDeviceToDevice, st));
    // the scheme of the posterior (tall-panel int8 at N >= 2048); w = L^{-1} y falls out of the panel solves instead of
    // a separate chain of 2 N / 128 strip launches for one row
    RET_IF(potrf_auto(ctx, st, A, ld, N, 1, Linv, dinfo));
    RET_IF(launch(ctx, st, 1, 256, 0, logdiag_kernel, A, ld, N, sc, (int64_t)0));
    RET_IF(launch(ctx, st, 1, RD_THREADS, 0, rowdot2_kernel, w, ld, N, nullptr, 1.0, nullptr, sc + 1, (int64_t)0));
    if (grad || alpha_out) {
        RET_IF(ensure(ctx, sl.cov, (size_t)N * ld * 8));
        double* Bt = (double*)sl.cov.p;  // (L^{-1})^T
        RET_IF(launch(ctx, st, grid_for(N * N), 256, 0, set_identity_kernel, Bt, ld, N, (int64_t)0));
        RET_IF(trsm_rec(ctx, st, Bt, ld, N, A, ld, N, Linv));
        // alpha = L^{-T} w : alpha_i = <Bt[i,:], w>
        RET_IF(launch(ctx, st, (unsigned)N, RD_THREADS, 0, rowdot2_kernel, Bt, ld, N, w, 1.0, alpha, nullptr, (int64_t)0));
        if (grad) {
            RET_IF(ensure(ctx, sl.Vt, (size_t)N * ld * 8));
            double* Kinv = (double*)sl.Vt.p;
            // K^{-1} = L^{-T} L^{-1} accumulated onto zeros: beta = 1 is what the int8 tensor-core path takes (7 planes here)
            CUDA_TRY(ctx, cudaMemsetAsync(Kinv, 0, (size_t)N * ld * 8, st));
            RET_IF(gemm_nt(ctx, st, N, N, N, 1.0, Bt, ld, Bt, ld, 1.0, Kinv, ld, true));
            if (gm) {   // L^{-T} (sl.cov) and the factor (A) are free again: the staging buffers of host dK
                gdev = partial + tiles * tiles * gm->p;
                RET_IF(mll_gram_trace(ctx, st, *gm, dev, (int)tiles, alpha, Kinv, ld, N, Bt, A, (const double**)(gdev + gm->p), partial,
                                      gdev));
            } else if (mt) {
                RET_IF(launch(ctx, st, dim3((unsigned)tiles, (unsigned)tiles, (unsigned)L), MLL_THREADS, 0, mll_lcm_grad_kernel, dX, dtask, N,
                              d, kind, T, L, mt->group, dth, (const double*)dmt, (const double*)(dmt + (size_t)L * T * T), jitter,
                              (const double*)alpha, (const double*)Kinv, ld, partial));
                RET_IF(launch(ctx, st, (unsigned)(L * nout), MLL_FIN_THREADS, 0, mll_lcm_finish_kernel, (const double*)partial,
                              tiles * tiles, nout, gmt, (int64_t)0));
                if (grad_x_dev)   // d value / d X [N, d] of the LCM covariance on the device (dkl.cuh)
                    RET_IF(launch(ctx, st, (unsigned)ceil_div(N, DZ_ROWS), DZ_THREADS, 0, mll_lcm_dz_kernel, kind, dX, dtask, N, d, T, L,
                                  dth, (const double*)dmt, (const double*)alpha, (const double*)Kinv, ld, grad_x_dev));
            } else if (nngp) {   // nngp.cuh: self-chains, the cross chain per pair, fixed-order sums -> sc[8..11) = (var_w, noise, var_b)
                double* chain = partial + tiles * tiles * 3;
                if (depth > 0) RET_IF(launch(ctx, st, (unsigned)ceil_div(N, (int64_t)256), 256, 0, nngp_self_kernel, dX, N, d, kind, dth, chain, (int64_t)0));
                static PerDeviceOnce attr;
                if (attr.need(ctx->device)) {
                    CUDA_TRY(ctx, cudaFuncSetAttribute(mll_nngp_grad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                       (int)nngp_grad_smem(GRAM_MAX_D, NNGP_MAX_DEPTH)));
                    attr.done(ctx->device);
                }
                count_path(ctx, (int)PATH_MLL_NNGP_GRAD);
                RET_IF(launch(ctx, st, dim3((unsigned)tiles, (unsigned)tiles), NNGP_THREADS, nngp_grad_smem(d, depth),
                              mll_nngp_grad_kernel, dX, N, d, kind, dth, (const double*)chain, (const double*)alpha, (const double*)Kinv, ld,
                              partial, (int64_t)0));
                RET_IF(launch(ctx, st, 3u, MLL_FIN_THREADS, 0, mll_lcm_finish_kernel, (const double*)partial, tiles * tiles, 3, sc + 8, (int64_t)0));
            } else {
                RET_IF(launch(ctx, st, dim3((unsigned)tiles, (unsigned)tiles), MLL_THREADS, 0, mll_grad_kernel, dX, N, d, kind, dth, alpha, Kinv,
                              ld, partial, (int64_t)0));
                RET_IF(launch(ctx, st, 1, 32, 0, mll_finish_kernel, partial, tiles * tiles, nth, sc + 8, (int64_t)0));
                if (grad_x_dev)   // d value / d X [N, d] on the device (dkl.cuh)
                    RET_IF(launch(ctx, st, (unsigned)ceil_div(N, DZ_ROWS), DZ_THREADS, 0, mll_dz_kernel, kind, dX, N, d, dth,
                                  (const double*)alpha, (const double*)Kinv, ld, grad_x_dev));
            }
            if (grad_noise_vec) {
                RET_IF(launch(ctx, st, grid_for(N), 256, 0, mll_diag_grad_kernel, alpha, Kinv, ld, N, w, (int64_t)0));   // w is free again
                CUDA_TRY(ctx, cudaMemcpyAsync(grad_noise_vec, w, (size_t)N * 8, cudaMemcpyDeviceToHost, st));
            }
        }
    }
    double hsc[8 + MLL_MAX_D + 3];
    CUDA_TRY(ctx, cudaMemcpyAsync(hsc, sc, sizeof hsc, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(ctx, cudaMemcpyAsync(info, dinfo, sizeof(int), cudaMemcpyDeviceToHost, st));
    if (alpha_out) CUDA_TRY(ctx, cudaMemcpyAsync(alpha_out, alpha, (size_t)N * 8, cudaMemcpyDeviceToHost, st));
    std::vector<double> colsum(mt ? (size_t)L * nout : 0);
    if (grad && mt) CUDA_TRY(ctx, cudaMemcpyAsync(colsum.data(), gmt, colsum.size() * 8, cudaMemcpyDeviceToHost, st));
    if (gdev) CUDA_TRY(ctx, cudaMemcpyAsync(grad, gdev, (size_t)gm->p * 8, cudaMemcpyDeviceToHost, st));
    RET_IF(tm.end(st, nullptr));
    if (grad && mt) {   // grad_theta [L, d+2] | grad_B [L, T, T] (symmetrised) | grad_noise [T]  (mtgp.cuh)
        const int nth1 = d + 2;
        for (int q = 0; q < L; ++q) {
            const double* c = colsum.data() + (size_t)q * nout;
            for (int k = 0; k < nth1; ++k) grad[q * nth1 + k] = c[k];
            for (int a = 0; a < T; ++a)
                for (int b = 0; b < T; ++b)
                    grad[L * nth1 + (q * T + a) * T + b] = 0.5 * (c[nth1 + a * T + b] + c[nth1 + b * T + a]);
        }
        for (int t = 0; t < T; ++t) grad[L * nth1 + L * T * T + t] = colsum[nth1 + T * T + t];
    }
    *value = -0.5 * hsc[1] - hsc[0] - 0.5 * (double)N * 1.8378770664093453;  // log(2 pi)
    if (grad && nngp) {   // [0, d) depth slots: 0; d: log var_w; d+1: log noise; d+2: log var_b
        for (int k = 0; k < d; ++k) grad[k] = 0.0;
        for (int k = 0; k < 3; ++k) grad[d + k] = hsc[8 + k];
    } else if (grad && !mt && !gm) {
        for (int k = 0; k < nth; ++k) grad[k] = hsc[8 + k];
    }
    if (*info != 0) {
        *value = NAN;
        if (grad)
            for (int k = 0; k < ngrad; ++k) grad[k] = NAN;
        if (grad_noise_vec)
            for (int64_t i = 0; i < N; ++i) grad_noise_vec[i] = NAN;
    }
    ctx->last.flops = (double)N * N * N * (grad ? 1.0 / 3 + 1.0 + 1.0 : 1.0 / 3);
    return B2GP_OK;
}

extern "C" int b2gp_mll(b2gp_ctx* ctx, int kind, const double* X, int64_t N, const double* yres, int d, const double* theta,
                        double jitter, unsigned flags, double* value, double* grad, double* alpha_out, int* info) {
    return mll_impl(ctx, kind, X, N, yres, d, theta, nullptr, jitter, flags, value, grad, alpha_out, nullptr, info);
}

extern "C" int b2gp_mll_v(b2gp_ctx* ctx, int kind, const double* X, int64_t N, const double* yres, int d, const double* theta,
                          const double* noise_vec, double jitter, unsigned flags, double* value, double* grad, double* alpha_out,
                          double* grad_noise_vec, int* info) {
    return mll_impl(ctx, kind, X, N, yres, d, theta, noise_vec, jitter, flags, value, grad, alpha_out, grad_noise_vec, info);
}

extern "C" int b2gp_mll_gram(b2gp_ctx* ctx, const double* K, int64_t N, int64_t ldk, const double* yres, const double* const* dK,
                             int64_t lddk, int64_t p, unsigned flags, double* value, double* grad, double* alpha_out, int* info) {
    if (!ctx) return B2GP_ERR_ARG;
    if (f32_io(flags)) return set_err(ctx, B2GP_ERR_UNSUPPORTED, "b2gp_mll_gram", "fp64 arrays only", __FILE__, __LINE__);
    ARG_CHECK(ctx, K && N >= 1 && ldk >= N && p >= 0);
    const bool want_grad = grad && p > 0;
    if (want_grad) {
        ARG_CHECK(ctx, dK && lddk >= N);
        for (int64_t j = 0; j < p; ++j) ARG_CHECK(ctx, dK[j]);
    }
    const GramMll gm{K, ldk, dK, lddk, want_grad ? p : 0};
    return mll_impl(ctx, B2GP_KERNEL_RBF, nullptr, N, yres, 1, nullptr, nullptr, 0.0, flags, value, want_grad ? grad : nullptr, alpha_out,
                    nullptr, info, nullptr, nullptr, &gm);
}

// MultiTaskGP / CoregGP.model's likelihood (mtgp.py:147-167, corgp.py:66-98) with the LCM kernel and its gradient
extern "C" int b2gp_mll_multitask(b2gp_ctx* ctx, int kind, const double* X, const int* task, int64_t N, const double* yres, int d,
                                  int group, int T, int L, const double* theta, const double* B, const double* noise, double jitter,
                                  unsigned flags, double* value, double* grad_theta, double* grad_B, double* grad_noise,
                                  double* alpha_out, int* info) {
    if (!ctx) return B2GP_ERR_ARG;
    ARG_CHECK(ctx, B && noise && N >= 1);
    ARG_CHECK(ctx, (grad_theta != nullptr) == (grad_B != nullptr) && (grad_B != nullptr) == (grad_noise != nullptr));
    RET_IF(mt_check(ctx, "b2gp_mll_multitask", kind, flags, d, group, T, L, task, N, nullptr, 0));
    const MtDesc mt{task, nullptr, group, T, L, B, noise};
    std::vector<double> g;
    if (grad_theta) g.resize((size_t)L * (d + 2) + (size_t)L * T * T + T);
    RET_IF(mll_impl(ctx, kind, X, N, yres, d, theta, nullptr, jitter, flags, value, grad_theta ? g.data() : nullptr, alpha_out, nullptr,
                    info, &mt));
    if (grad_theta) {
        memcpy(grad_theta, g.data(), (size_t)L * (d + 2) * 8);
        memcpy(grad_B, g.data() + (size_t)L * (d + 2), (size_t)L * T * T * 8);
        memcpy(grad_noise, g.data() + (size_t)L * (d + 2) + (size_t)L * T * T, (size_t)T * 8);
    }
    return B2GP_OK;
}

// ------------------------------------------------------------------------------------------ likelihood draws in lock-step
// b2gp_mll_draws: S likelihoods on one X, draw s with theta[s] and its own or the shared yres, run as mll_impl's sequence in
// groups of B draws.  Each draw of a group owns one region of ctx->post, `stride` doubles apart, so that a single Batch
// offsets every operand of a launch:
//   [Linv | A ((N + 1) x ld: K, y under it) | Bt = L^{-T} | K^{-1} | panel scratch (tall route) | alpha | sc | partials |
//    NNGP self-chains | theta]
// sc is mll_impl's: [0] sum log L_ii, [1] |L^{-1} y|^2, [8 ..) the gradient.  Every kernel computes a draw exactly as its
// unbatched launch does, and every factorisation kernel gives the same bits whatever the batch (gemm_nt, potrf.cuh), so
// draw s returns b2gp_mll's bits on (theta[s], yres[s]) whatever S and the grouping.

// p[draw][0, n) = 0; the draw is blockIdx.y (`bstride` doubles apart)
__global__ void zero_batch_kernel(double* p, int64_t n, int64_t bstride) {
    p += (int64_t)blockIdx.y * bstride;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) p[i] = 0.0;
}

constexpr int MLLD_HS = 8 + MLL_MAX_D + 3;   // the scalars of sc read back per draw (mll_impl's hsc)

// Stage S vectors of N doubles, `stride` apart (0: one vector for every draw), as [S, N] in `buf`; `rows` holds the
// repeated host copy until the call's end
static int stage_rows(b2gp_ctx* ctx, cudaStream_t st, DevBuf& buf, std::vector<double>& rows, const double* src, int64_t stride,
                      int64_t S, int64_t N, const double** out) {
    if (stride != N) {
        rows.resize((size_t)S * N);
        for (int64_t s = 0; s < S; ++s) memcpy(rows.data() + s * N, src + s * stride, (size_t)N * 8);
        src = rows.data();
    }
    return stage_in(ctx, st, buf, src, (size_t)S * N * 8, false, out);
}

// b2gp_mll_draws and b2gp_mll_draws_v: noise_vec == nullptr is the plain likelihood, with no launch of the noise-vector form
static int mll_draws_impl(b2gp_ctx* ctx, const char* who, int kind, const double* X, int64_t N, const double* yres,
                          int64_t yres_stride, int d, int64_t S, const double* theta, const double* noise_vec, int64_t nv_stride,
                          double jitter, unsigned flags, double* value, double* grad, double* alpha_out, double* grad_noise_vec,
                          int* info) {
    if (!ctx) return B2GP_ERR_ARG;
    if (f32_io(flags) || dev_ptrs(flags)) return set_err(ctx, B2GP_ERR_UNSUPPORTED, who, "host fp64 arrays only", __FILE__, __LINE__);
    ARG_CHECK(ctx, kind >= 0 && kind <= B2GP_KERNEL_NNGP_RELU);
    const bool nngp = is_nngp(kind);
    ARG_CHECK(ctx, X && yres && theta && value && info);
    ARG_CHECK(ctx, N >= 1 && S >= 1 && d >= 1 && d <= (nngp ? GRAM_MAX_D : MLL_MAX_D));
    ARG_CHECK(ctx, yres_stride == 0 || yres_stride >= N);
    ARG_CHECK(ctx, !noise_vec || nv_stride == 0 || nv_stride >= N);
    ARG_CHECK(ctx, !grad_noise_vec || (noise_vec && grad));
    const int nth = d + 3;
    int depth = 0;   // NNGP: the deepest draw sizes the self-chains and the gradient kernel's shared memory
    if (nngp)
        for (int64_t s = 0; s < S; ++s) {
            RET_IF(nngp_check_depth(ctx, who, theta[s * nth]));
            depth = std::max(depth, (int)theta[s * nth]);
        }
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    ctx->fcache.valid = false;   // the regions overwrite slot 0's matrix
    Slot& sl = ctx->slots[0];
    cudaStream_t st = sl.stream;
    CallTimer tm(ctx);
    RET_IF(tm.begin(st));
    const int64_t ld = round_up(N, 8), tiles = ceil_div(N, MLL_TILE);
    const bool want_k = grad || alpha_out;
    const bool tall64 = use_tall_fp64(ctx, N);
    // region layout (doubles)
    const int64_t oA = linv_bytes(N) / 8, oBt = oA + (N + 1) * ld, oKi = oBt + (want_k ? N * ld : 0), oScr = oKi + (grad ? N * ld : 0);
    const int64_t oAl = oScr + (tall64 ? panel_scratch_elems(ctx, N < ctx->panel ? N : ctx->panel) : 0), oSc = oAl + ld, oPart = oSc + 64;
    const int64_t oCh = oPart + tiles * tiles * (nngp ? 3 : nth), oTh = oCh + (nngp ? N * depth * 3 : 0);
    const int64_t stride = round_up(oTh + nth, 32);
    // Group size.  The int8 route takes one draw at a time (its GEMMs and panel solves refuse batches).  Otherwise
    // draw_batch: 0 = as many draws as an eighth of the device memory holds, 1 = one draw per group, B >= 2 = groups of B.
    int64_t B = 1;
    if (ctx->ozaki == 0) {
        if (ctx->draw_batch == 0)
            B = std::max<int64_t>(1, (int64_t)(ctx->mem_bytes / 8) / (stride * 8));
        else
            B = ctx->draw_batch;
        B = std::min<int64_t>(std::min<int64_t>(B, S), 65535);
    }
    // inputs: X, theta [S, nth], yres and the noise vectors as [S, N] (a shared vector repeated), staged once
    std::vector<double> yrows, nvrows;
    const double *dX, *dy, *dth, *dnv = nullptr;
    RET_IF(stage_in(ctx, st, ctx->d_in[0], X, (size_t)N * d * 8, false, &dX));
    RET_IF(stage_rows(ctx, st, ctx->d_in[1], yrows, yres, yres_stride, S, N, &dy));
    RET_IF(stage_in(ctx, st, ctx->d_in[3], theta, (size_t)S * nth * 8, false, &dth));
    if (noise_vec) RET_IF(stage_rows(ctx, st, ctx->d_in[6], nvrows, noise_vec, nv_stride, S, N, &dnv));
    RET_IF(ensure(ctx, ctx->d_info, (size_t)S * sizeof(int)));
    RET_IF(ensure(ctx, ctx->d_out[0], (size_t)S * MLLD_HS * 8));
    if (alpha_out) RET_IF(ensure(ctx, ctx->d_out[1], (size_t)S * N * 8));
    if (grad_noise_vec) RET_IF(ensure(ctx, ctx->d_out[2], (size_t)S * N * 8));
    RET_IF(ensure(ctx, ctx->post, (size_t)B * stride * 8));
    int* dinfo = (int*)ctx->d_info.p;
    double* dsc = (double*)ctx->d_out[0].p;
    double* dal = (double*)ctx->d_out[1].p;
    double* dgnv = (double*)ctx->d_out[2].p;
    CUDA_TRY(ctx, cudaMemsetAsync(dinfo, 0, (size_t)S * sizeof(int), st));
    double* R = (double*)ctx->post.p;
    double *Linv = R, *A = R + oA, *w = A + N * ld, *Bt = R + oBt, *Kinv = R + oKi, *scr = R + oScr, *alpha = R + oAl, *sc = R + oSc,
           *partial = R + oPart, *chain = R + oCh, *th = R + oTh;
    if (nngp && grad) {
        static PerDeviceOnce attr;
        if (attr.need(ctx->device)) {
            CUDA_TRY(ctx, cudaFuncSetAttribute(mll_nngp_grad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               (int)nngp_grad_smem(GRAM_MAX_D, NNGP_MAX_DEPTH)));
            attr.done(ctx->device);
        }
    }
    for (int64_t g0 = 0; g0 < S; g0 += B) {
        const int nb = (int)std::min<int64_t>(B, S - g0);
        const Batch bt{nb, stride};
        const unsigned z = (unsigned)nb;
        count_path(ctx, (int)PATH_MLL_DRAWS_BATCH);
        RET_IF(launch(ctx, st, grid_for((int64_t)nb * nth), 256, 0, copy2d_kernel, th, stride, dth + g0 * nth, (int64_t)nth, (int64_t)nb,
                      (int64_t)nth));
        RET_IF(launch(ctx, st, grid_for((int64_t)nb * N), 256, 0, copy2d_kernel, w, stride, dy + g0 * N, N, (int64_t)nb, N));
        RET_IF(launch_gram(ctx, st, kind, dX, N, dX, N, d, th, 1.0, jitter, 1, 1, A, ld, bt));
        if (dnv)
            RET_IF(launch(ctx, st, dim3(grid_for(N), 1, z), 256, 0, add_diag_vec_kernel, A, ld, N, dnv + g0 * N, stride, N));
        if (nb == 1) {   // mll_impl's factorisation on every route
            RET_IF(potrf_auto(ctx, st, A, ld, N, 1, Linv, dinfo + g0));
        } else if (tall64) {   // fp64 tall-panel route, y riding below K
            for (int j = 0; j < nb; ++j) count_tall_entry(ctx, false);
            RET_IF(potrf_tall(ctx, st, scr, A, ld, N, 1, Linv, dinfo + g0, 0, nullptr, bt));
        } else {
            RET_IF(potrf_rec(ctx, st, A, ld, N, Linv, dinfo + g0, 0, bt));
            RET_IF(trsm_rec(ctx, st, w, ld, 1, A, ld, N, Linv, true, bt));
        }
        RET_IF(launch(ctx, st, dim3(1, 1, z), 256, 0, logdiag_kernel, (const double*)A, ld, N, sc, stride));
        RET_IF(launch(ctx, st, dim3(1, 1, z), RD_THREADS, 0, rowdot2_kernel, (const double*)w, ld, N, (const double*)nullptr, 1.0,
                      (double*)nullptr, sc + 1, stride));
        if (want_k) {
            RET_IF(launch(ctx, st, dim3(grid_for(N * N), z), 256, 0, set_identity_kernel, Bt, ld, N, stride));
            RET_IF(trsm_rec(ctx, st, Bt, ld, N, A, ld, N, Linv, true, bt));
            RET_IF(launch(ctx, st, dim3((unsigned)N, 1, z), RD_THREADS, 0, rowdot2_kernel, (const double*)Bt, ld, N, (const double*)w, 1.0,
                          alpha, (double*)nullptr, stride));
        }
        if (grad) {
            RET_IF(launch(ctx, st, dim3(grid_for(N * ld), z), 256, 0, zero_batch_kernel, Kinv, N * ld, stride));
            RET_IF(gemm_nt(ctx, st, N, N, N, 1.0, Bt, ld, Bt, ld, 1.0, Kinv, ld, true, bt));
            if (nngp) {
                if (depth > 0)
                    RET_IF(launch(ctx, st, dim3((unsigned)ceil_div(N, (int64_t)256), 1, z), 256, 0, nngp_self_kernel, dX, N, d, kind,
                                  (const double*)th, chain, stride));
                for (int j = 0; j < nb; ++j) count_path(ctx, (int)PATH_MLL_NNGP_GRAD);
                RET_IF(launch(ctx, st, dim3((unsigned)tiles, (unsigned)tiles, z), NNGP_THREADS, nngp_grad_smem(d, depth), mll_nngp_grad_kernel,
                              dX, N, d, kind, (const double*)th, (const double*)chain, (const double*)alpha, (const double*)Kinv, ld, partial,
                              stride));
                RET_IF(launch(ctx, st, dim3(3, 1, z), MLL_FIN_THREADS, 0, mll_lcm_finish_kernel, (const double*)partial, tiles * tiles, 3,
                              sc + 8, stride));
            } else {
                RET_IF(launch(ctx, st, dim3((unsigned)tiles, (unsigned)tiles, z), MLL_THREADS, 0, mll_grad_kernel, dX, N, d, kind,
                              (const double*)th, (const double*)alpha, (const double*)Kinv, ld, partial, stride));
                RET_IF(launch(ctx, st, dim3(1, 1, z), 32, 0, mll_finish_kernel, (const double*)partial, tiles * tiles, nth, sc + 8, stride));
            }
            if (grad_noise_vec)   // the draw's w row is free once alpha is formed
                RET_IF(launch(ctx, st, dim3(grid_for(N), 1, z), 256, 0, mll_diag_grad_kernel, (const double*)alpha, (const double*)Kinv, ld, N,
                              w, stride));
        }
        // the group's results leave the regions before the next group reuses them
        RET_IF(launch(ctx, st, grid_for((int64_t)nb * MLLD_HS), 256, 0, copy2d_kernel, dsc + g0 * MLLD_HS, (int64_t)MLLD_HS,
                      (const double*)sc, stride, (int64_t)nb, (int64_t)MLLD_HS));
        if (alpha_out)
            RET_IF(launch(ctx, st, grid_for((int64_t)nb * N), 256, 0, copy2d_kernel, dal + g0 * N, N, (const double*)alpha, stride,
                          (int64_t)nb, N));
        if (grad_noise_vec)
            RET_IF(launch(ctx, st, grid_for((int64_t)nb * N), 256, 0, copy2d_kernel, dgnv + g0 * N, N, (const double*)w, stride,
                          (int64_t)nb, N));
    }
    std::vector<double> hsc((size_t)S * MLLD_HS);
    CUDA_TRY(ctx, cudaMemcpyAsync(hsc.data(), dsc, hsc.size() * 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(ctx, cudaMemcpyAsync(info, dinfo, (size_t)S * sizeof(int), cudaMemcpyDeviceToHost, st));
    if (alpha_out) CUDA_TRY(ctx, cudaMemcpyAsync(alpha_out, dal, (size_t)S * N * 8, cudaMemcpyDeviceToHost, st));
    if (grad_noise_vec) CUDA_TRY(ctx, cudaMemcpyAsync(grad_noise_vec, dgnv, (size_t)S * N * 8, cudaMemcpyDeviceToHost, st));
    RET_IF(tm.end(st, nullptr));
    for (int64_t s = 0; s < S; ++s) {   // mll_impl's host epilogue, per draw
        const double* h = hsc.data() + s * MLLD_HS;
        value[s] = -0.5 * h[1] - h[0] - 0.5 * (double)N * 1.8378770664093453;  // log(2 pi)
        double* g = grad ? grad + s * nth : nullptr;
        if (g && nngp) {
            for (int k = 0; k < d; ++k) g[k] = 0.0;
            for (int k = 0; k < 3; ++k) g[d + k] = h[8 + k];
        } else if (g) {
            for (int k = 0; k < nth; ++k) g[k] = h[8 + k];
        }
        if (info[s] != 0) {
            value[s] = NAN;
            if (g)
                for (int k = 0; k < nth; ++k) g[k] = NAN;
            if (alpha_out)
                for (int64_t i = 0; i < N; ++i) alpha_out[s * N + i] = NAN;
            if (grad_noise_vec)
                for (int64_t i = 0; i < N; ++i) grad_noise_vec[s * N + i] = NAN;
        }
    }
    ctx->last.flops = (double)S * N * N * N * (grad ? 1.0 / 3 + 1.0 + 1.0 : 1.0 / 3);
    return B2GP_OK;
}

extern "C" int b2gp_mll_draws(b2gp_ctx* ctx, int kind, const double* X, int64_t N, const double* yres, int64_t yres_stride, int d,
                              int64_t S, const double* theta, double jitter, unsigned flags, double* value, double* grad,
                              double* alpha_out, int* info) {
    return mll_draws_impl(ctx, "b2gp_mll_draws", kind, X, N, yres, yres_stride, d, S, theta, nullptr, 0, jitter, flags, value, grad,
                          alpha_out, nullptr, info);
}

extern "C" int b2gp_mll_draws_v(b2gp_ctx* ctx, int kind, const double* X, int64_t N, const double* yres, int64_t yres_stride, int d,
                                int64_t S, const double* theta, const double* noise_vec, int64_t nv_stride, double jitter,
                                unsigned flags, double* value, double* grad, double* alpha_out, double* grad_noise_vec, int* info) {
    if (ctx && !noise_vec) return set_err(ctx, B2GP_ERR_ARG, "b2gp_mll_draws_v", "noise_vec is required", __FILE__, __LINE__);
    return mll_draws_impl(ctx, "b2gp_mll_draws_v", kind, X, N, yres, yres_stride, d, S, theta, noise_vec, nv_stride, jitter, flags, value,
                          grad, alpha_out, grad_noise_vec, info);
}

// ------------------------------------------------------------------------------------------ deep kernel learning (dkl.cuh)
// Layer l maps in[l] -> out[l] features; W_l [in, out] at woff[l] and b_l [out] at boff[l] of the params layout.
struct MlpShape {
    int L = 0;
    int64_t N = 0, d = 0, nparams = 0, max_in = 0, max_out = 0;
    std::vector<int64_t> in, out, woff, boff;
};

static int mlp_shape(b2gp_ctx* ctx, int64_t N, int64_t D, int n_layers, const int64_t* widths, int act, MlpShape& s) {
    ARG_CHECK(ctx, N >= 1 && D >= 1 && n_layers >= 0 && n_layers <= 64);
    ARG_CHECK(ctx, n_layers == 0 || (widths && (act == B2GP_ACT_RELU || act == B2GP_ACT_TANH)));
    s.L = n_layers;
    s.N = N;
    int64_t in = D, o = 0;
    for (int l = 0; l < n_layers; ++l) {
        ARG_CHECK(ctx, widths[l] >= 1 && widths[l] <= (1 << 16));
        s.in.push_back(in);
        s.out.push_back(widths[l]);
        s.woff.push_back(o);
        o += in * widths[l];
        s.boff.push_back(o);
        o += widths[l];
        s.max_in = std::max(s.max_in, in);
        s.max_out = std::max(s.max_out, widths[l]);
        in = widths[l];
    }
    s.d = in;
    s.nparams = o;
    return B2GP_OK;
}

// H[0] = X, H[l+1] = act(H[l] W_l + b_l) (no activation on the last layer), each [N, out_l] contiguous, in ctx->mlp[2]
// after the transposed weights W_l^T [out_l, in_l] that gemm_nt takes as its B operand.  dP: the weights on the device.
static int mlp_forward_dev(b2gp_ctx* ctx, cudaStream_t st, const MlpShape& s, int act, const double* dX, const double* dP,
                           std::vector<double*>& H) {
    std::vector<int64_t> hoff(s.L), toff(s.L);
    int64_t tot = 0;
    for (int l = 0; l < s.L; ++l) {
        toff[l] = tot;
        tot += round_up(s.out[l] * s.in[l], 8);
    }
    for (int l = 0; l < s.L; ++l) {
        hoff[l] = tot;
        tot += round_up(s.N * s.out[l], 8);
    }
    H.assign(s.L + 1, nullptr);
    H[0] = const_cast<double*>(dX);
    if (s.L == 0) return B2GP_OK;
    RET_IF(ensure(ctx, ctx->mlp[2], (size_t)tot * 8));
    double* base = (double*)ctx->mlp[2].p;
    for (int l = 0; l < s.L; ++l) {
        const int64_t in = s.in[l], out = s.out[l];
        double* Wt = base + toff[l];
        H[l + 1] = base + hoff[l];
        RET_IF(launch_transpose(ctx, st, dP + s.woff[l], out, in, out, Wt, in));
        RET_IF(gemm_nt(ctx, st, s.N, out, in, 1.0, H[l], in, Wt, in, 0.0, H[l + 1], out, false));
        RET_IF(launch(ctx, st, grid_for(s.N * out), 256, 0, mlp_bias_act_kernel, H[l + 1], out, s.N, (int)out,
                      (const double*)(dP + s.boff[l]), l + 1 < s.L ? act : (int)DKL_ACT_NONE));
    }
    return B2GP_OK;
}

extern "C" int b2gp_mlp_forward(b2gp_ctx* ctx, const double* X, int64_t N, int64_t D, int n_layers, const int64_t* widths, int act,
                                const double* params, int64_t S, int64_t params_stride, double* Z, unsigned flags) {
    if (!ctx) return B2GP_ERR_ARG;
    MlpShape s;
    RET_IF(mlp_shape(ctx, N, D, n_layers, widths, act, s));
    ARG_CHECK(ctx, X && Z && S >= 1 && !f32_io(flags));
    ARG_CHECK(ctx, n_layers == 0 || (params && params_stride >= s.nparams));
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    ctx->fcache.valid = false;
    cudaStream_t st = ctx->slots[0].stream;
    CallTimer tm(ctx);
    RET_IF(tm.begin(st));
    const double *dX, *dP = nullptr;
    RET_IF(stage_in(ctx, st, ctx->mlp[0], X, (size_t)N * D * 8, dev_ptrs(flags), &dX));
    if (n_layers > 0) RET_IF(stage_in(ctx, st, ctx->mlp[1], params, (size_t)((S - 1) * params_stride + s.nparams) * 8, false, &dP));
    std::vector<double*> H;
    for (int64_t m = 0; m < S; ++m) {
        RET_IF(mlp_forward_dev(ctx, st, s, act, dX, dP ? dP + m * params_stride : nullptr, H));
        CUDA_TRY(ctx, cudaMemcpyAsync(Z + m * N * s.d, H[s.L], (size_t)N * s.d * 8, cudaMemcpyDeviceToHost, st));
    }
    RET_IF(tm.end(st, nullptr));
    return B2GP_OK;
}

// The backward pass's scratch in ctx->mlp[3]: gz [N, d] | grad params | G ping-pong 2 x [N, max_out] | H_l^T [max_in, ldN]
// | G^T [max_out, ldN].  `tot` with the backward pass, `o_gp` (gz alone) without it.
struct MlpBack {
    int64_t ldN, o_gp, o_g0, o_g1, o_ht, o_gt, tot;
};

static MlpBack mlp_back_layout(const MlpShape& s) {
    MlpBack b;
    b.ldN = round_up(s.N, 8);
    b.o_gp = round_up(s.N * s.d, 8);
    b.o_g0 = b.o_gp + round_up(s.nparams, 8);
    b.o_g1 = b.o_g0 + round_up(s.N * s.max_out, 8);
    b.o_ht = b.o_g1 + round_up(s.N * s.max_out, 8);
    b.o_gt = b.o_ht + s.max_in * b.ldN;
    b.tot = b.o_gt + s.max_out * b.ldN;
    return b;
}

// The backward pass from gz = d value / dz (at base, the start of mlp[3]) to grad_params (HOST): per layer the bias
// gradient (column sum), the weight gradient H_l^T G (gemm_nt on the transposes) and, below the first layer, G W_l^T
// masked by the activation's derivative.
static int mlp_backward_dev(b2gp_ctx* ctx, cudaStream_t st, const MlpShape& s, const MlpBack& b, int act, const double* dP,
                            const std::vector<double*>& H, double* base, double* grad_params) {
    const int64_t N = s.N, ldN = b.ldN;
    double *gp = base + b.o_gp, *G0 = base + b.o_g0, *G1 = base + b.o_g1, *Ht = base + b.o_ht, *Gt = base + b.o_gt;
    double* G = base;   // d value / d (pre-activation output of layer l), [N, out_l]
    for (int l = s.L - 1; l >= 0; --l) {
        const int64_t in = s.in[l], out = s.out[l];
        RET_IF(launch(ctx, st, (unsigned)out, MLP_SUM_THREADS, 0, mlp_colsum_kernel, (const double*)G, out, N, gp + s.boff[l]));
        RET_IF(launch_transpose(ctx, st, H[l], in, N, in, Ht, ldN));
        RET_IF(launch_transpose(ctx, st, G, out, N, out, Gt, ldN));
        RET_IF(gemm_nt(ctx, st, in, out, N, 1.0, Ht, ldN, Gt, ldN, 0.0, gp + s.woff[l], out, false));
        if (l > 0) {
            double* Gn = G == G0 ? G1 : G0;
            RET_IF(gemm_nt(ctx, st, N, in, out, 1.0, G, out, dP + s.woff[l], out, 0.0, Gn, in, false));
            RET_IF(launch(ctx, st, grid_for(N * in), 256, 0, mlp_act_grad_kernel, Gn, in, (const double*)H[l], in, N, (int)in, act));
            G = Gn;
        }
    }
    CUDA_TRY(ctx, cudaMemcpyAsync(grad_params, gp, (size_t)s.nparams * 8, cudaMemcpyDeviceToHost, st));
    return B2GP_OK;
}

// b2gp_last_timing of a deep-kernel step reports the whole step: mll_impl's own timer covers only its part, so the call
// is bracketed by a second pair of events and its totals replace mll_impl's at the end
struct StepTimer {
    std::chrono::steady_clock::time_point t0;
    int64_t launches0 = 0;
    int begin(b2gp_ctx* ctx, cudaStream_t st) {
        t0 = std::chrono::steady_clock::now();
        launches0 = ctx->launches;
        CUDA_TRY(ctx, cudaEventRecord(ctx->ev_a, st));
        return B2GP_OK;
    }
    int end(b2gp_ctx* ctx, cudaStream_t st) {
        CUDA_TRY(ctx, cudaEventRecord(ctx->ev_b, st));
        CUDA_TRY(ctx, cudaEventSynchronize(ctx->ev_b));
        float ms = 0.f;
        CUDA_TRY(ctx, cudaEventElapsedTime(&ms, ctx->ev_a, ctx->ev_b));
        ctx->last.total_ms = ms;
        ctx->last.launches = ctx->launches - launches0;
        ctx->last.host_enqueue_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        return B2GP_OK;
    }
};

// viDKL / DKL's likelihood on z = MLP(X): forward pass, then mll_impl on z (the b2gp_mll route, with d value / dz from
// mll_dz_kernel), then the backward pass through the layers (mlp_backward_dev).
extern "C" int b2gp_dkl_mll(b2gp_ctx* ctx, int kind, const double* X, int64_t N, int64_t D, const double* yres, int n_layers,
                            const int64_t* widths, int act, const double* params, const double* theta, double jitter, unsigned flags,
                            double* value, double* grad_theta, double* grad_params, double* grad_z, int* info) {
    if (!ctx) return B2GP_ERR_ARG;
    MlpShape s;
    RET_IF(mlp_shape(ctx, N, D, n_layers, widths, act, s));
    ARG_CHECK(ctx, kind >= 0 && kind <= 2);
    ARG_CHECK(ctx, X && yres && theta && value && grad_theta && info && !f32_io(flags));
    ARG_CHECK(ctx, s.d <= MLL_MAX_D && (n_layers == 0 || params));
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    ctx->fcache.valid = false;
    cudaStream_t st = ctx->slots[0].stream;
    StepTimer tm;
    RET_IF(tm.begin(ctx, st));
    const bool dev = dev_ptrs(flags);
    const double *dX, *dy, *dP = nullptr;
    RET_IF(stage_in(ctx, st, ctx->mlp[0], X, (size_t)N * D * 8, dev, &dX));
    RET_IF(stage_in(ctx, st, ctx->d_in[1], yres, (size_t)N * 8, dev, &dy));
    if (n_layers > 0) RET_IF(stage_in(ctx, st, ctx->mlp[1], params, (size_t)s.nparams * 8, false, &dP));
    std::vector<double*> H;
    RET_IF(mlp_forward_dev(ctx, st, s, act, dX, dP, H));
    const bool back = grad_params && n_layers > 0;
    const MlpBack b = mlp_back_layout(s);
    RET_IF(ensure(ctx, ctx->mlp[3], (size_t)(back ? b.tot : b.o_gp) * 8));
    double* gz = (double*)ctx->mlp[3].p;
    const int64_t d = s.d;
    RET_IF(mll_impl(ctx, kind, H[s.L], N, dy, (int)d, theta, nullptr, jitter, B2GP_FLAG_DEVICE_PTRS, value, grad_theta, nullptr, nullptr,
                    info, nullptr, (grad_z || back) ? gz : nullptr));
    const int64_t ngp = grad_params ? s.nparams : 0;
    if (*info != 0) {
        for (int64_t i = 0; grad_z && i < N * d; ++i) grad_z[i] = NAN;
        for (int64_t i = 0; i < ngp; ++i) grad_params[i] = NAN;
    }
    if (grad_z && *info == 0) CUDA_TRY(ctx, cudaMemcpyAsync(grad_z, gz, (size_t)N * d * 8, cudaMemcpyDeviceToHost, st));
    if (back && *info == 0) RET_IF(mlp_backward_dev(ctx, st, s, b, act, dP, H, gz, grad_params));
    return tm.end(ctx, st);
}

// viDKL / DKL's posterior and its gradient w.r.t. the raw test inputs: embed X and Xnew per weight set (mlp_forward_dev,
// keeping the test points' hidden activations), posterior_impl on the embeddings with the derivative rows, then
// mlp_input_vjp_kernel pulls d mean / dz and d var / dz back through the network.  The embeddings go through host
// arrays into posterior_impl, exactly as b2gp_posterior receives b2gp_mlp_forward's output: the S = 1 factor cache keys
// on those bytes and on nothing else.  Everything besides posterior_impl works in ctx->mlp[0..3] on slot 0's stream
// (the forward GEMMs have beta = 0, so never the int8 route and its slot scratch) and leaves slot 0's matrix and Ukeep --
// the cached factor -- alone; unlike b2gp_mlp_forward this entry point therefore keeps the cache valid.
extern "C" int b2gp_dkl_posterior_grad(b2gp_ctx* ctx, int kind, const double* X, int64_t N, int64_t D, const double* yres,
                                       int64_t yres_stride, const double* Xnew, int64_t P, int n_layers, const int64_t* widths, int act,
                                       const double* params, int64_t S, int64_t params_stride, const double* theta, int noiseless,
                                       double jitter, unsigned flags, double* mean, double* var, double* dmean, double* dvar, int* info) {
    if (!ctx) return B2GP_ERR_ARG;
    if (flags & (B2GP_FLAG_F32 | B2GP_FLAG_DEVICE_PTRS | B2GP_OUT_COV | B2GP_OUT_SAMPLE))
        return set_err(ctx, B2GP_ERR_UNSUPPORTED, "b2gp_dkl_posterior_grad", "host fp64 arrays, outputs mean / var / dmean / dvar only",
                       __FILE__, __LINE__);
    ARG_CHECK(ctx, kind >= 0 && kind <= 2);
    MlpShape sx, sp;
    RET_IF(mlp_shape(ctx, N, D, n_layers, widths, act, sx));
    ARG_CHECK(ctx, P >= 1 && S >= 1);
    RET_IF(mlp_shape(ctx, P, D, n_layers, widths, act, sp));
    ARG_CHECK(ctx, X && Xnew && yres && theta && info && (n_layers == 0 || (params && params_stride >= sx.nparams)));
    ARG_CHECK(ctx, sx.d <= GRAM_MAX_D && D <= (int64_t)VJP_TILE * 65535);
    const unsigned outs = flags & (B2GP_OUT_MEAN | B2GP_OUT_VAR | B2GP_OUT_DMEAN | B2GP_OUT_DVAR);
    if (n_layers == 0)
        return b2gp_posterior_grad(ctx, kind, X, N, yres, yres_stride, Xnew, P, (int)D, S, theta, noiseless, jitter, outs, mean, var, dmean,
                                   dvar, info, nullptr);
    const bool want_dm = outs & B2GP_OUT_DMEAN, want_dv = outs & B2GP_OUT_DVAR;
    ARG_CHECK(ctx, (!want_dm || dmean) && (!want_dv || dvar));
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    const auto t0 = std::chrono::steady_clock::now();
    const int64_t launches0 = ctx->launches;
    cudaStream_t st = ctx->slots[0].stream;
    const int L = n_layers;
    const int64_t dz = sx.d;

    // ---- 1. inputs: [X | Xnew] in mlp[0], the S weight sets in mlp[1]
    const int64_t xoff = round_up(N * D, 8);
    RET_IF(ensure(ctx, ctx->mlp[0], (size_t)(xoff + P * D) * 8));
    double* dX = (double*)ctx->mlp[0].p;
    CUDA_TRY(ctx, cudaMemcpyAsync(dX, X, (size_t)N * D * 8, cudaMemcpyHostToDevice, st));
    CUDA_TRY(ctx, cudaMemcpyAsync(dX + xoff, Xnew, (size_t)P * D * 8, cudaMemcpyHostToDevice, st));
    const double* dP = nullptr;
    RET_IF(stage_in(ctx, st, ctx->mlp[1], params, (size_t)((S - 1) * params_stride + sx.nparams) * 8, false, &dP));

    // mlp[3]: the test points' hidden activations H_1 .. H_{L-1} per weight set (the layout mlp_forward_dev gives them) |
    // the cotangents [R][S, P, dz] | dX [S, R, P, D] | the kernel's G buffers when they do not fit in shared memory
    const int R = (want_dm ? 1 : 0) + (want_dv ? 1 : 0);
    int64_t hstride = 0, wmax = 0;
    for (int l = 0; l + 1 < L; ++l) hstride += round_up(P * sp.out[l], 8);
    for (int l = 0; l < L; ++l) wmax = std::max(wmax, sp.out[l]);
    const size_t smem = (size_t)2 * VJP_MAX_R * wmax * 8;
    const bool use_smem = smem <= VJP_SMEM_MAX;
    const dim3 grid((unsigned)(S * P), (unsigned)ceil_div(D, (int64_t)VJP_TILE));
    const int64_t o_cot = round_up(S * hstride, 8), o_dx = o_cot + round_up((int64_t)VJP_MAX_R * S * P * dz, 8);
    const int64_t o_g = o_dx + round_up((int64_t)S * R * P * D, 8);
    const int64_t tot = o_g + (use_smem || R == 0 ? 0 : (int64_t)grid.x * grid.y * 2 * VJP_MAX_R * wmax);
    RET_IF(ensure(ctx, ctx->mlp[3], (size_t)tot * 8));
    double* work = (double*)ctx->mlp[3].p;

    // ---- embeddings: the training set's and the test points' per weight set, on the host for posterior_impl
    std::vector<double> Ztr((size_t)S * N * dz), Zn((size_t)S * P * dz);
    std::vector<double*> H;
    for (int64_t m = 0; m < S; ++m) {
        const double* Pm = dP + m * params_stride;
        RET_IF(mlp_forward_dev(ctx, st, sp, act, dX + xoff, Pm, H));
        if (hstride > 0 && R > 0)
            CUDA_TRY(ctx, cudaMemcpyAsync(work + m * hstride, H[1], (size_t)hstride * 8, cudaMemcpyDeviceToDevice, st));
        CUDA_TRY(ctx, cudaMemcpyAsync(Zn.data() + m * P * dz, H[L], (size_t)P * dz * 8, cudaMemcpyDeviceToHost, st));
        RET_IF(mlp_forward_dev(ctx, st, sx, act, dX, Pm, H));
        CUDA_TRY(ctx, cudaMemcpyAsync(Ztr.data() + m * N * dz, H[L], (size_t)N * dz * 8, cudaMemcpyDeviceToHost, st));
    }
    CUDA_TRY(ctx, cudaStreamSynchronize(st));

    // ---- 2. the posterior and its gradient w.r.t. the embedding
    std::vector<double> dmz(want_dm ? (size_t)S * P * dz : 0), dvz(want_dv ? (size_t)S * P * dz : 0);
    const int64_t xs = S > 1 ? N * dz : 0, xns = S > 1 ? P * dz : 0;
    RET_IF(posterior_impl(ctx, kind, Ztr.data(), xs, N, yres, yres_stride, Zn.data(), xns, P, (int)dz, S, theta, nullptr, 0, noiseless,
                          jitter, outs, mean, var, nullptr, nullptr, 0, nullptr, info, nullptr, want_dm ? dmz.data() : nullptr,
                          want_dv ? dvz.data() : nullptr));

    // ---- 3. the pull-back to the raw inputs
    if (R > 0) {
        double* cot = work + o_cot;
        double* dXout = work + o_dx;
        const double* c0 = want_dm ? dmz.data() : dvz.data();
        CUDA_TRY(ctx, cudaMemcpyAsync(cot, c0, (size_t)S * P * dz * 8, cudaMemcpyHostToDevice, st));
        if (R > 1) CUDA_TRY(ctx, cudaMemcpyAsync(cot + S * P * dz, dvz.data(), (size_t)S * P * dz * 8, cudaMemcpyHostToDevice, st));
        VjpNet net{};
        net.L = L;
        net.R = R;
        net.width[0] = D;
        for (int l = 0; l < L; ++l) {
            net.width[l + 1] = sp.out[l];
            net.woff[l] = sp.woff[l];
        }
        RET_IF(launch(ctx, st, grid, VJP_THREADS, use_smem ? smem : 0, mlp_input_vjp_kernel, net, dP, params_stride,
                      (const double*)work, hstride, P, act, (const double*)cot, (const double*)(R > 1 ? cot + S * P * dz : nullptr),
                      dXout, use_smem ? (double*)nullptr : work + o_g, wmax));
        // dX [S, R, P, D]: row r of every weight set to its output
        const size_t row = (size_t)P * D * 8;
        if (want_dm) CUDA_TRY(ctx, cudaMemcpy2DAsync(dmean, row, dXout, R * row, row, (size_t)S, cudaMemcpyDeviceToHost, st));
        if (want_dv)
            CUDA_TRY(ctx, cudaMemcpy2DAsync(dvar, row, dXout + (R - 1) * P * D, R * row, row, (size_t)S, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(ctx, cudaStreamSynchronize(st));
    }
    for (int64_t m = 0; m < S; ++m) {
        if (info[m] == 0) continue;
        if (outs & B2GP_OUT_MEAN) std::fill(mean + m * P, mean + (m + 1) * P, (double)NAN);
        if (outs & B2GP_OUT_VAR) std::fill(var + m * P, var + (m + 1) * P, (double)NAN);
        if (want_dm) std::fill(dmean + m * P * D, dmean + (m + 1) * P * D, (double)NAN);
        if (want_dv) std::fill(dvar + m * P * D, dvar + (m + 1) * P * D, (double)NAN);
    }
    ctx->last.total_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    ctx->last.launches = ctx->launches - launches0;
    return B2GP_OK;
}

// vExactGP / UIGP: B independent likelihoods (mll_batch.cuh).  N <= B2GP_MLL_BATCH_SMALL_MAX_N: one launch of
// mll_batch_small_kernel, one CTA per member.  Larger N: mll_impl per member -- the b2gp_mll route and, with grad_x, the b2gp_dkl_mll(n_layers = 0)
// one (mll_dz_kernel), so each member's outputs are those calls' bits.
extern "C" int b2gp_mll_batch(b2gp_ctx* ctx, int kind, const double* X, int64_t N, const double* yres, int d, int64_t B,
                              const double* theta, double jitter, unsigned flags, double* value, double* grad, double* alpha_out,
                              double* grad_x, int* info) {
    if (!ctx) return B2GP_ERR_ARG;
    if (is_nngp(kind) || f32_io(flags) || dev_ptrs(flags))
        return set_err(ctx, B2GP_ERR_UNSUPPORTED, "b2gp_mll_batch", "RBF / Matern / Periodic, host fp64 arrays only", __FILE__, __LINE__);
    ARG_CHECK(ctx, kind >= 0 && kind <= B2GP_KERNEL_PERIODIC);
    ARG_CHECK(ctx, X && yres && theta && value && info && N >= 1 && B >= 1 && d >= 1 && d <= MLL_MAX_D);
    ARG_CHECK(ctx, !grad_x || grad);
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    const int nth = d + 3;
    if (N > B2GP_MLL_BATCH_SMALL_MAX_N) {
        cudaStream_t st = ctx->slots[0].stream;
        StepTimer tm;
        RET_IF(tm.begin(ctx, st));
        if (grad_x) RET_IF(ensure(ctx, ctx->mlp[3], (size_t)N * d * 8));
        double* gx = (double*)ctx->mlp[3].p;
        for (int64_t b = 0; b < B; ++b) {
            RET_IF(mll_impl(ctx, kind, X + b * N * d, N, yres + b * N, d, theta + b * nth, nullptr, jitter, 0, value + b,
                            grad ? grad + b * nth : nullptr, alpha_out ? alpha_out + b * N : nullptr, nullptr, info + b, nullptr,
                            grad_x ? gx : nullptr));
            if (grad_x && info[b] == 0) {
                CUDA_TRY(ctx, cudaMemcpyAsync(grad_x + b * N * d, gx, (size_t)N * d * 8, cudaMemcpyDeviceToHost, st));
                CUDA_TRY(ctx, cudaStreamSynchronize(st));
            }
        }
        RET_IF(tm.end(ctx, st));
    } else {
        ctx->fcache.valid = false;
        Slot& sl = ctx->slots[0];
        cudaStream_t st = sl.stream;
        CallTimer tm(ctx);
        RET_IF(tm.begin(st));
        count_path(ctx, (int)PATH_MLL_BATCH_SMALL);
        const double *dX, *dy, *dth;
        RET_IF(stage_in(ctx, st, ctx->d_in[0], X, (size_t)(B * N * d) * 8, false, &dX));
        RET_IF(stage_in(ctx, st, ctx->d_in[1], yres, (size_t)(B * N) * 8, false, &dy));
        RET_IF(stage_in(ctx, st, ctx->d_in[3], theta, (size_t)(B * nth) * 8, false, &dth));
        // outputs value [B] | grad [B, d+3] | alpha [B, N] | grad_x [B, N, d], then info [B]
        const int64_t o_g = B, o_a = o_g + B * nth, o_x = o_a + B * N, o_end = o_x + B * N * d;
        RET_IF(ensure(ctx, ctx->d_out[0], (size_t)o_end * 8 + (size_t)B * sizeof(int)));
        double* dout = (double*)ctx->d_out[0].p;
        int* dinfo = (int*)(dout + o_end);
        static PerDeviceOnce attr;
        if (attr.need(ctx->device)) {
            CUDA_TRY(ctx, cudaFuncSetAttribute(mll_batch_small_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, MLLB_SMEM));
            attr.done(ctx->device);
        }
        RET_IF(launch(ctx, st, (unsigned)B, PD_THREADS, MLLB_SMEM, mll_batch_small_kernel, kind, dX, (int)N, dy, d, dth, jitter, dout,
                      grad ? dout + o_g : nullptr, alpha_out ? dout + o_a : nullptr, grad_x ? dout + o_x : nullptr, dinfo));
        CUDA_TRY(ctx, cudaMemcpyAsync(value, dout, (size_t)B * 8, cudaMemcpyDeviceToHost, st));
        if (grad) CUDA_TRY(ctx, cudaMemcpyAsync(grad, dout + o_g, (size_t)(B * nth) * 8, cudaMemcpyDeviceToHost, st));
        if (alpha_out) CUDA_TRY(ctx, cudaMemcpyAsync(alpha_out, dout + o_a, (size_t)(B * N) * 8, cudaMemcpyDeviceToHost, st));
        if (grad_x) CUDA_TRY(ctx, cudaMemcpyAsync(grad_x, dout + o_x, (size_t)(B * N * d) * 8, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(ctx, cudaMemcpyAsync(info, dinfo, (size_t)B * sizeof(int), cudaMemcpyDeviceToHost, st));
        RET_IF(tm.end(st, nullptr));
    }
    for (int64_t b = 0; b < B; ++b) {   // a member without a factorisation: NaN outputs, whatever the route left there
        if (info[b] == 0) continue;
        value[b] = NAN;
        for (int k = 0; grad && k < nth; ++k) grad[b * nth + k] = NAN;
        for (int64_t i = 0; alpha_out && i < N; ++i) alpha_out[b * N + i] = NAN;
        for (int64_t i = 0; grad_x && i < N * d; ++i) grad_x[b * N * d + i] = NAN;
    }
    ctx->last.flops = (double)B * N * N * N * (grad ? 1.0 / 3 + 1.0 + 1.0 : 1.0 / 3);
    return B2GP_OK;
}

// viMTDKL's likelihood: the forward pass on the N points, z expanded to the N * group GP rows (point-major, one device
// copy per task slot), mll_impl on the rows with the LCM covariance (the b2gp_mll_multitask route, d value / dz from
// mll_lcm_dz_kernel), each point's rows summed in task order (group_sum_kernel), then the backward pass.
extern "C" int b2gp_mtdkl_mll(b2gp_ctx* ctx, int kind, const double* X, const int* task, int64_t N, int64_t D, const double* yres,
                              int group, int T, int L, int n_layers, const int64_t* widths, int act, const double* params,
                              const double* theta, const double* B, const double* noise, double jitter, unsigned flags,
                              double* value, double* grad_theta, double* grad_B, double* grad_noise, double* grad_params,
                              double* grad_z, int* info) {
    if (!ctx) return B2GP_ERR_ARG;
    MlpShape s;
    RET_IF(mlp_shape(ctx, N, D, n_layers, widths, act, s));
    ARG_CHECK(ctx, X && yres && theta && B && noise && value && grad_theta && grad_B && grad_noise && info);
    ARG_CHECK(ctx, group >= 1 && (n_layers == 0 || params));
    if (kind == B2GP_KERNEL_PERIODIC)
        return set_err(ctx, B2GP_ERR_UNSUPPORTED, "b2gp_mtdkl_mll", "RBF and Matern only (viMTDKL samples no period)", __FILE__,
                       __LINE__);
    const int64_t R = N * group;   // GP rows
    // task ids and limits before any launch; X and yres may be device pointers here, the arrays mt_check sees are host
    RET_IF(mt_check(ctx, "b2gp_mtdkl_mll", kind, flags & ~B2GP_FLAG_DEVICE_PTRS, (int)s.d, group, T, L, task, R, nullptr, 0));
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    ctx->fcache.valid = false;
    cudaStream_t st = ctx->slots[0].stream;
    StepTimer tm;
    RET_IF(tm.begin(ctx, st));
    const bool dev = dev_ptrs(flags);
    const double *dX, *dy, *dP = nullptr;
    RET_IF(stage_in(ctx, st, ctx->mlp[0], X, (size_t)N * D * 8, dev, &dX));
    RET_IF(stage_in(ctx, st, ctx->d_in[1], yres, (size_t)R * 8, dev, &dy));
    if (n_layers > 0) RET_IF(stage_in(ctx, st, ctx->mlp[1], params, (size_t)s.nparams * 8, false, &dP));
    std::vector<double*> H;
    RET_IF(mlp_forward_dev(ctx, st, s, act, dX, dP, H));
    const bool back = grad_params && n_layers > 0, want_z = grad_z || back;
    const int64_t d = s.d;
    // mlp[3]: the backward scratch (gz at its start), then z and d value / dz on the rows when group > 1
    const MlpBack b = mlp_back_layout(s);
    const int64_t o_rows = back ? b.tot : b.o_gp, nrow = group > 1 ? round_up(R * d, 8) : 0;
    RET_IF(ensure(ctx, ctx->mlp[3], (size_t)(o_rows + 2 * nrow) * 8));
    double* gz = (double*)ctx->mlp[3].p;
    const double* zr = H[s.L];
    double* gzr = gz;
    if (group > 1) {
        double* zrows = gz + o_rows;
        gzr = zrows + nrow;
        for (int t = 0; t < group; ++t)
            CUDA_TRY(ctx, cudaMemcpy2DAsync(zrows + t * d, (size_t)group * d * 8, H[s.L], (size_t)d * 8, (size_t)d * 8, (size_t)N,
                                            cudaMemcpyDeviceToDevice, st));
        zr = zrows;
    }
    const MtDesc mt{task, nullptr, group, T, L, B, noise};
    std::vector<double> g((size_t)L * (d + 2) + (size_t)L * T * T + T);
    RET_IF(mll_impl(ctx, kind, zr, R, dy, (int)d, theta, nullptr, jitter, B2GP_FLAG_DEVICE_PTRS, value, g.data(), nullptr, nullptr,
                    info, &mt, want_z ? gzr : nullptr));
    memcpy(grad_theta, g.data(), (size_t)L * (d + 2) * 8);
    memcpy(grad_B, g.data() + (size_t)L * (d + 2), (size_t)L * T * T * 8);
    memcpy(grad_noise, g.data() + (size_t)L * (d + 2) + (size_t)L * T * T, (size_t)T * 8);
    const int64_t ngp = grad_params ? s.nparams : 0;
    if (*info != 0) {
        for (int64_t i = 0; grad_z && i < N * d; ++i) grad_z[i] = NAN;
        for (int64_t i = 0; i < ngp; ++i) grad_params[i] = NAN;
    }
    if (want_z && group > 1 && *info == 0)
        RET_IF(launch(ctx, st, grid_for(N * d), 256, 0, group_sum_kernel, (const double*)gzr, N, (int)d, group, gz));
    if (grad_z && *info == 0) CUDA_TRY(ctx, cudaMemcpyAsync(grad_z, gz, (size_t)N * d * 8, cudaMemcpyDeviceToHost, st));
    if (back && *info == 0) RET_IF(mlp_backward_dev(ctx, st, s, b, act, dP, H, gz, grad_params));
    return tm.end(ctx, st);
}

// ------------------------------------------------------------------------------------------ Bayesian MLP (bnn.cuh)
static int bnn_optin(b2gp_ctx* ctx) {
    static PerDeviceOnce attr;
    if (attr.need(ctx->device)) {
        CUDA_TRY(ctx, cudaFuncSetAttribute(bnn_loglik_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)(ctx->smem_optin - 8 * BNN_THREADS)));
        CUDA_TRY(ctx, cudaFuncSetAttribute(bnn_predict_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ctx->smem_optin));
        CUDA_TRY(ctx, cudaFuncSetAttribute(bnn_predict_grad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ctx->smem_optin));
        attr.done(ctx->device);
    }
    return B2GP_OK;
}

// BNN's likelihood sum_{i,o} log N(y_io; z_io, sigma): two launches on the fused route, the DKL forward / backward pass
// around bnn_resid_kernel on the layered one.  Both leave sum r^2 in the slot after the parameter gradient.
extern "C" int b2gp_bnn_loglik(b2gp_ctx* ctx, const double* X, int64_t N, int64_t D, const double* y, int64_t O, int n_layers,
                               const int64_t* widths, int act, const double* params, double sigma, unsigned flags, double* value,
                               double* grad_sigma, double* grad_params) {
    if (!ctx) return B2GP_ERR_ARG;
    MlpShape s;
    RET_IF(mlp_shape(ctx, N, D, n_layers, widths, act, s));
    ARG_CHECK(ctx, X && y && params && value && grad_sigma && n_layers >= 1 && s.d == O && !f32_io(flags));
    ARG_CHECK(ctx, sigma > 0.0 && std::isfinite(sigma));
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    ctx->fcache.valid = false;
    cudaStream_t st = ctx->slots[0].stream;
    CallTimer tm(ctx);
    RET_IF(tm.begin(st));
    const bool dev = dev_ptrs(flags);
    const double *dX, *dy, *dP;
    RET_IF(stage_in(ctx, st, ctx->mlp[0], X, (size_t)N * D * 8, dev, &dX));
    RET_IF(stage_in(ctx, st, ctx->d_in[1], y, (size_t)N * O * 8, dev, &dy));
    RET_IF(stage_in(ctx, st, ctx->mlp[1], params, (size_t)s.nparams * 8, false, &dP));
    const double inv_s2 = 1.0 / (sigma * sigma);
    const size_t smem = ctx->bnn_fused ? bnn_fused_smem(D, n_layers, widths, true, ctx->smem_optin) : 0;
    const double* sums;   // [grad params | sum r^2] on the device
    if (smem) {
        RET_IF(bnn_optin(ctx));
        int per_sm = 0;
        CUDA_TRY(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, bnn_loglik_tile_kernel, BNN_THREADS, smem));
        const int64_t nblk = std::min<int64_t>(ceil_div(N, BNN_ROWS), (int64_t)ctx->sm_count * std::max(per_sm, 1));
        const int64_t ld = s.nparams + 1;
        RET_IF(ensure(ctx, ctx->mlp[3], (size_t)(nblk + 1) * ld * 8));
        double* partial = (double*)ctx->mlp[3].p;
        double* out = partial + nblk * ld;
        RET_IF(launch(ctx, st, (unsigned)nblk, BNN_THREADS, smem, bnn_loglik_tile_kernel, bnn_net(D, n_layers, widths), act, dX, dy,
                      N, dP, inv_s2, partial));
        RET_IF(launch(ctx, st, (unsigned)ceil_div(ld, 256), 256, 0, bnn_reduce_kernel, (const double*)partial, (int)nblk, (int)ld, out));
        if (grad_params) CUDA_TRY(ctx, cudaMemcpyAsync(grad_params, out, (size_t)s.nparams * 8, cudaMemcpyDeviceToHost, st));
        sums = out;
    } else {
        std::vector<double*> H;
        RET_IF(mlp_forward_dev(ctx, st, s, act, dX, dP, H));
        const MlpBack b = mlp_back_layout(s);
        RET_IF(ensure(ctx, ctx->mlp[3], (size_t)(b.tot + 1) * 8));
        double* base = (double*)ctx->mlp[3].p;
        double* r2 = base + b.tot;
        RET_IF(launch(ctx, st, 1, BNN_THREADS, 0, bnn_resid_kernel, (const double*)H[s.L], dy, N * O, inv_s2, base, r2));
        if (grad_params) RET_IF(mlp_backward_dev(ctx, st, s, b, act, dP, H, base, grad_params));
        sums = r2;
    }
    double r2sum = 0.0;
    CUDA_TRY(ctx, cudaMemcpyAsync(&r2sum, sums + (smem ? s.nparams : 0), 8, cudaMemcpyDeviceToHost, st));
    RET_IF(tm.end(st, nullptr));
    const double no = (double)N * (double)O;
    *value = -0.5 * r2sum * inv_s2 - no * (log(sigma) + 0.5 * log(2.0 * 3.141592653589793));
    *grad_sigma = r2sum * inv_s2 / sigma - no / sigma;
    return B2GP_OK;
}

// loc[s] = MLP(X; weight set s) and y_sampled[s] = loc[s] + sigma[s] * mean_k eps[s, k] for S weight sets: one launch on
// the fused route, the DKL forward pass and bnn_sample_kernel per draw on the layered one; one copy back either way.
extern "C" int b2gp_bnn_predict(b2gp_ctx* ctx, const double* X, int64_t P, int64_t D, int n_layers, const int64_t* widths, int act,
                                const double* params, int64_t S, int64_t params_stride, int64_t O, const double* sigma,
                                const double* eps, int64_t n, double* loc, double* y_sampled, unsigned flags) {
    if (!ctx) return B2GP_ERR_ARG;
    MlpShape s;
    RET_IF(mlp_shape(ctx, P, D, n_layers, widths, act, s));
    ARG_CHECK(ctx, X && params && loc && n_layers >= 1 && s.d == O && S >= 1 && params_stride >= s.nparams);
    ARG_CHECK(ctx, !eps || (sigma && y_sampled && n >= 1 && n <= (1 << 30)));
    ARG_CHECK(ctx, !f32_io(flags));
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    ctx->fcache.valid = false;
    cudaStream_t st = ctx->slots[0].stream;
    CallTimer tm(ctx);
    RET_IF(tm.begin(st));
    const int64_t PO = P * O;
    const double *dX, *dP, *dsig = nullptr, *deps = nullptr;
    RET_IF(stage_in(ctx, st, ctx->mlp[0], X, (size_t)P * D * 8, dev_ptrs(flags), &dX));
    RET_IF(stage_in(ctx, st, ctx->mlp[1], params, (size_t)((S - 1) * params_stride + s.nparams) * 8, false, &dP));
    if (eps) {
        RET_IF(stage_in(ctx, st, ctx->d_in[2], sigma, (size_t)S * 8, false, &dsig));
        RET_IF(stage_in(ctx, st, ctx->d_in[3], eps, (size_t)S * n * PO * 8, false, &deps));
    }
    const int64_t nout = round_up(S * PO, 8);
    RET_IF(ensure(ctx, ctx->d_out[0], (size_t)(eps ? 2 : 1) * nout * 8));
    double* dloc = (double*)ctx->d_out[0].p;
    double* dys = eps ? dloc + nout : nullptr;
    const size_t smem = ctx->bnn_fused ? bnn_fused_smem(D, n_layers, widths, false, ctx->smem_optin) : 0;
    if (smem) {
        RET_IF(bnn_optin(ctx));
        const BnnNet net = bnn_net(D, n_layers, widths);
        for (int64_t s0 = 0; s0 < S; s0 += 65535) {   // grid.y holds at most 65535 draws
            const dim3 grid((unsigned)ceil_div(P, BNN_ROWS), (unsigned)std::min<int64_t>(S - s0, 65535));
            RET_IF(launch(ctx, st, grid, BNN_THREADS, smem, bnn_predict_kernel, net, act, dX, P, dP, params_stride, dsig, deps, (int)n,
                          dloc, dys, s0));
        }
    } else {
        std::vector<double*> H;
        for (int64_t m = 0; m < S; ++m) {
            RET_IF(mlp_forward_dev(ctx, st, s, act, dX, dP + m * params_stride, H));
            RET_IF(launch(ctx, st, grid_for(PO), 256, 0, bnn_sample_kernel, (const double*)H[s.L], PO, m, dsig, deps, (int)n, dloc, dys));
        }
    }
    CUDA_TRY(ctx, cudaMemcpyAsync(loc, dloc, (size_t)S * PO * 8, cudaMemcpyDeviceToHost, st));
    if (eps) CUDA_TRY(ctx, cudaMemcpyAsync(y_sampled, dys, (size_t)S * PO * 8, cudaMemcpyDeviceToHost, st));
    RET_IF(tm.end(st, nullptr));
    return B2GP_OK;
}

// hidden activations the layered route of b2gp_bnn_predict_grad keeps at once (doubles, 1 GiB): draws are taken in
// chunks that stay under it
constexpr int64_t BNN_GRAD_KEEP = (int64_t)1 << 27;

// loc[s] = MLP(X; weight set s) for a one-output network and dloc[s, p, :] = d loc[s, p] / d X[p, :]: one launch per
// 65535 draws on the fused route (bnn_predict_grad_kernel); on the layered one the DKL forward pass per draw keeps the
// hidden activations of a chunk of draws and one mlp_input_vjp_kernel launch per chunk pulls the unit cotangent back.
extern "C" int b2gp_bnn_predict_grad(b2gp_ctx* ctx, const double* X, int64_t P, int64_t D, int n_layers, const int64_t* widths,
                                     int act, const double* params, int64_t S, int64_t params_stride, double* loc, double* dloc,
                                     unsigned flags) {
    if (!ctx) return B2GP_ERR_ARG;
    if (f32_io(flags)) return set_err(ctx, B2GP_ERR_UNSUPPORTED, "b2gp_bnn_predict_grad", "fp64 arrays only", __FILE__, __LINE__);
    MlpShape s;
    RET_IF(mlp_shape(ctx, P, D, n_layers, widths, act, s));
    ARG_CHECK(ctx, X && params && loc && dloc && n_layers >= 1 && s.d == 1 && S >= 1 && params_stride >= s.nparams);
    ARG_CHECK(ctx, D <= (int64_t)VJP_TILE * 65535);
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    ctx->fcache.valid = false;
    cudaStream_t st = ctx->slots[0].stream;
    CallTimer tm(ctx);
    RET_IF(tm.begin(st));
    const bool dev = dev_ptrs(flags);
    const double *dX, *dP;
    RET_IF(stage_in(ctx, st, ctx->mlp[0], X, (size_t)P * D * 8, dev, &dX));
    RET_IF(stage_in(ctx, st, ctx->mlp[1], params, (size_t)((S - 1) * params_stride + s.nparams) * 8, dev, &dP));
    const int64_t nloc = round_up(S * P, 8);
    RET_IF(ensure(ctx, ctx->d_out[0], (size_t)(nloc + S * P * D) * 8));
    double* dl = (double*)ctx->d_out[0].p;
    double* ddl = dl + nloc;
    std::vector<double> ones;   // the layered route's cotangents; alive until the copies that read it are done
    const size_t smem = ctx->bnn_fused ? bnn_fused_smem(D, n_layers, widths, false, ctx->smem_optin) : 0;
    if (smem) {
        RET_IF(bnn_optin(ctx));
        const BnnNet net = bnn_net(D, n_layers, widths);
        for (int64_t s0 = 0; s0 < S; s0 += 65535) {   // grid.y holds at most 65535 draws
            const dim3 grid((unsigned)ceil_div(P, BNN_ROWS), (unsigned)std::min<int64_t>(S - s0, 65535));
            RET_IF(launch(ctx, st, grid, BNN_THREADS, smem, bnn_predict_grad_kernel, net, act, dX, P, dP, params_stride, dl, ddl, s0));
        }
    } else {
        // mlp[3]: the hidden activations H_1 .. H_{L-1} of a chunk of draws (mlp_forward_dev's layout) | ones [chunk, P] |
        // the kernel's G buffers when they do not fit in shared memory
        const int L = n_layers;
        int64_t hstride = 0, wmax = 0;
        for (int l = 0; l + 1 < L; ++l) hstride += round_up(P * s.out[l], 8);
        for (int l = 0; l < L; ++l) wmax = std::max(wmax, s.out[l]);
        const int64_t chunk = std::min<int64_t>({S, std::max<int64_t>(1, BNN_GRAD_KEEP / std::max<int64_t>(hstride, 1)),
                                                 std::max<int64_t>(1, (int64_t)INT_MAX / P)});
        const size_t vsm = (size_t)2 * VJP_MAX_R * wmax * 8;
        const bool use_smem = vsm <= VJP_SMEM_MAX;
        const int64_t ntile = ceil_div(D, (int64_t)VJP_TILE);
        const int64_t o_one = round_up(chunk * hstride, 8), o_g = o_one + round_up(chunk * P, 8);
        RET_IF(ensure(ctx, ctx->mlp[3], (size_t)(o_g + (use_smem ? 0 : chunk * P * ntile * 2 * VJP_MAX_R * wmax)) * 8));
        double* work = (double*)ctx->mlp[3].p;
        ones.assign((size_t)chunk * P, 1.0);
        CUDA_TRY(ctx, cudaMemcpyAsync(work + o_one, ones.data(), (size_t)chunk * P * 8, cudaMemcpyHostToDevice, st));
        VjpNet net{};
        net.L = L;
        net.R = 1;
        net.width[0] = D;
        for (int l = 0; l < L; ++l) {
            net.width[l + 1] = s.out[l];
            net.woff[l] = s.woff[l];
        }
        std::vector<double*> H;
        for (int64_t c0 = 0; c0 < S; c0 += chunk) {
            const int64_t nc = std::min(chunk, S - c0);
            for (int64_t m = c0; m < c0 + nc; ++m) {
                RET_IF(mlp_forward_dev(ctx, st, s, act, dX, dP + m * params_stride, H));
                if (hstride > 0)
                    CUDA_TRY(ctx, cudaMemcpyAsync(work + (m - c0) * hstride, H[1], (size_t)hstride * 8, cudaMemcpyDeviceToDevice, st));
                CUDA_TRY(ctx, cudaMemcpyAsync(dl + m * P, H[L], (size_t)P * 8, cudaMemcpyDeviceToDevice, st));
            }
            const dim3 grid((unsigned)(nc * P), (unsigned)ntile);
            RET_IF(launch(ctx, st, grid, VJP_THREADS, use_smem ? vsm : 0, mlp_input_vjp_kernel, net, dP + c0 * params_stride,
                          params_stride, (const double*)work, hstride, P, act, (const double*)(work + o_one), (const double*)nullptr,
                          ddl + c0 * P * D, use_smem ? (double*)nullptr : work + o_g, wmax));
        }
    }
    CUDA_TRY(ctx, cudaMemcpyAsync(loc, dl, (size_t)S * P * 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(ctx, cudaMemcpyAsync(dloc, ddl, (size_t)S * P * D * 8, cudaMemcpyDeviceToHost, st));
    RET_IF(tm.end(st, nullptr));
    return B2GP_OK;
}

// b2gp_sparse_elbo_gram: the blocks and the directions to contract the bound's adjoints with come from the caller.
// blocks.Kuu / Kuf, kff_diag [N] and every direction block follow blocks.dev.  Direction j < p is (dKuu[j] [M, M],
// dKuf[j] [M, N], dkff[j] [N]); direction p + k, k < q, is (rKuu[k], rKuf[k]) and gives the row sums grad_rows[k, :].
// Each pointer array may be NULL, and so may each block in it (a zero block).
struct SparseElboGram {
    SparseGram blocks;
    const double* kff_diag;
    double noise;
    const double* const* dKuu;
    const double* const* dKuf;
    const double* const* dkff;
    int64_t p;
    const double* const* rKuu;
    const double* const* rKuf;
    int64_t q;
    double* grad;            // [p]
    double* grad_log_noise;  // [1]
    double* grad_rows;       // [q, M]
};

// The reverse pass of the bound contracted with the caller's directions: one sparse_gram_trace_kernel pass per block over
// the resident adjoints Gs (M x M, symmetric) and Guf (M x N), then the fixed-order sums of sparse_gram_finish_kernel.
// Device blocks: one launch over every direction.  Host blocks: streamed through ctx->eb[10] / eb[11] as in
// mll_gram_trace -- the copy of direction j+1 on a second stream overlaps the reduction of direction j, and the copy into a
// buffer waits for the reduction that last read it.  `rows` [(p+q), M], `ksum` [p+q], `gdev` [p], `dptrs` [3 (p+q)].
static int sparse_gram_trace(b2gp_ctx* ctx, cudaStream_t st, const SparseElboGram& g, int64_t M, int64_t N, const double* Gs,
                             int64_t ldgs, const double* Guf, int64_t ldguf, double gd, double* rows, double* ksum, double* gdev,
                             const double** dptrs) {
    const int64_t J = g.p + g.q;
    count_path(ctx, (int)PATH_SPARSE_GRAM_TRACE);
    if (J == 0) return B2GP_OK;
    auto blk = [&](int64_t j, int t) -> const double* {   // direction j's block t (0: Kuu, 1: Kuf, 2: kff) or NULL
        const double* const* arr = j < g.p ? (t == 0 ? g.dKuu : t == 1 ? g.dKuf : g.dkff) : (t == 0 ? g.rKuu : t == 1 ? g.rKuf : nullptr);
        return arr ? arr[j < g.p ? j : j - g.p] : nullptr;
    };
    const int64_t off[3] = {0, M * M, M * M + M * N}, len[3] = {M * M, M * N, N};
    std::vector<const double*> table((size_t)3 * J);
    if (g.blocks.dev) {
        for (int64_t j = 0; j < J; ++j)
            for (int t = 0; t < 3; ++t) table[3 * j + t] = blk(j, t);
        CUDA_TRY(ctx, cudaMemcpyAsync(dptrs, table.data(), table.size() * sizeof(double*), cudaMemcpyHostToDevice, st));
        RET_IF(launch(ctx, st, dim3((unsigned)(M + 1), (unsigned)J), SGT_THREADS, 0, sparse_gram_trace_kernel, Gs, ldgs, Guf, ldguf, M, N,
                      (const double* const*)dptrs, M, N, (int64_t)0, rows, ksum));
    } else {
        const size_t bytes = (size_t)(M * M + M * N + N) * 8;
        RET_IF(ensure(ctx, ctx->eb[10], bytes));
        RET_IF(ensure(ctx, ctx->eb[11], bytes));
        double* bufs[2] = {(double*)ctx->eb[10].p, (double*)ctx->eb[11].p};
        for (int64_t j = 0; j < J; ++j)
            for (int t = 0; t < 3; ++t) table[3 * j + t] = blk(j, t) ? bufs[j & 1] + off[t] : nullptr;
        CUDA_TRY(ctx, cudaMemcpyAsync(dptrs, table.data(), table.size() * sizeof(double*), cudaMemcpyHostToDevice, st));
        cudaStream_t cs = ctx->slots[1].stream;
        cudaEvent_t free_ev = ctx->pool.get(), cp[2] = {ctx->pool.get(), ctx->pool.get()}, red[2] = {ctx->pool.get(), ctx->pool.get()};
        ARG_CHECK(ctx, free_ev && cp[0] && cp[1] && red[0] && red[1]);
        CUDA_TRY(ctx, cudaEventRecord(free_ev, st));   // the staging of the caller's Kuu in eb[10] is done with
        CUDA_TRY(ctx, cudaStreamWaitEvent(cs, free_ev, 0));
        for (int64_t j = 0; j < J; ++j) {
            const int b = (int)(j & 1);
            if (j >= 2) CUDA_TRY(ctx, cudaStreamWaitEvent(cs, red[b], 0));
            for (int t = 0; t < 3; ++t)
                if (const double* src = blk(j, t))
                    CUDA_TRY(ctx, cudaMemcpyAsync(bufs[b] + off[t], src, (size_t)len[t] * 8, cudaMemcpyHostToDevice, cs));
            CUDA_TRY(ctx, cudaEventRecord(cp[b], cs));
            CUDA_TRY(ctx, cudaStreamWaitEvent(st, cp[b], 0));
            RET_IF(launch(ctx, st, dim3((unsigned)(M + 1), 1u), SGT_THREADS, 0, sparse_gram_trace_kernel, Gs, ldgs, Guf, ldguf, M, N,
                          (const double* const*)(dptrs + 3 * j), M, N, j, rows, ksum));
            CUDA_TRY(ctx, cudaEventRecord(red[b], st));
        }
    }
    if (g.p == 0) return B2GP_OK;
    return launch(ctx, st, (unsigned)ceil_div(g.p, (int64_t)128), 128, 0, sparse_gram_finish_kernel, (const double*)rows, M,
                  (const double*)ksum, gd, g.p, gdev);
}

// value and gradient of the VFE bound of the sparse GP (see sparse_elbo.cuh): d/dlog(lengthscale[d], k_scale, noise, period)
// in grad_theta[d+3] and d/dXu in grad_Xu[M,d], alpha_out[N] = (W^T W + noise I)^{-1} yres.  Xu, X, yres follow `flags`;
// theta is a HOST pointer; outputs are HOST.  With `g` the blocks and directions are the caller's (b2gp_sparse_elbo_gram):
// Xu, X, theta, kind, d and jitter are unused and the gradients go to g's outputs.
static int sparse_elbo_impl(b2gp_ctx* ctx, int kind, const double* Xu, int64_t M, const double* X, int64_t N, const double* yres,
                            int d, const double* theta, double jitter, unsigned flags, double* value, double* grad_theta,
                            double* grad_Xu, double* alpha_out, int* info, const SparseElboGram* g = nullptr) {
    if (!ctx) return B2GP_ERR_ARG;
    if (!g) {
        ARG_CHECK(ctx, kind >= 0 && kind <= 2);
        ARG_CHECK(ctx, Xu && X && theta && grad_theta && grad_Xu);
        ARG_CHECK(ctx, d >= 1 && d <= MLL_MAX_D);
    }
    ARG_CHECK(ctx, yres && value && info);
    ARG_CHECK(ctx, M >= 1 && N >= 1);
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    ctx->fcache.valid = false;
    const bool dev = dev_ptrs(flags);
    Slot& sl = ctx->slots[0];
    cudaStream_t st = sl.stream;
    CallTimer tm(ctx);
    RET_IF(tm.begin(st));
    const int nth = d + 3;
    const double noise = g ? g->noise : theta[d + 1], scale = g ? 0.0 : theta[d];
    const int64_t J = g ? g->p + g->q : 0;
    const double *dXu = nullptr, *dX = nullptr, *dy, *dth = nullptr, *dkff = nullptr;
    RET_IF(stage_in(ctx, st, ctx->d_in[1], yres, (size_t)N * 8, dev, &dy));
    if (g) {
        RET_IF(stage_in(ctx, st, ctx->d_in[2], g->kff_diag, (size_t)N * 8, dev, &dkff));
    } else {
        RET_IF(stage_in(ctx, st, ctx->d_in[0], X, (size_t)N * d * 8, dev, &dX));
        RET_IF(stage_in(ctx, st, ctx->d_in[3], theta, (size_t)nth * 8, false, &dth));
        RET_IF(stage_in(ctx, st, ctx->d_in[5], Xu, (size_t)M * d * 8, dev, &dXu));
    }
    const int64_t ldM = round_up(M, 8), ldN = round_up(N, 8);
    double *slA = nullptr, *slLinv = nullptr;   // slot 0's matrix and inverted diagonal blocks
    RET_IF(slot0_buffers(ctx, (size_t)2 * M * ldM * 8, (size_t)2 * linv_bytes(M), &slA, &slLinv));
    RET_IF(ensure(ctx, ctx->d_info, 64));
    for (int i = 0; i < 6; ++i) RET_IF(ensure(ctx, ctx->eb[i], (size_t)M * ldM * 8));
    RET_IF(ensure(ctx, ctx->eb[6], (size_t)N * ldM * 8));
    RET_IF(ensure(ctx, ctx->eb[7], (size_t)N * ldM * 8));
    RET_IF(ensure(ctx, ctx->eb[8], (size_t)M * ldN * 8));
    // tail after the 64 scalars: fused M x (d+3) partials | M x d grad_Xu;  caller blocks: rows [J, M] | ksum [J] |
    // grad [p] | the device table of 3 J direction pointers
    const int64_t tail = g ? J * M + J + g->p + 3 * J + 8 : M * (nth + d);
    RET_IF(ensure(ctx, ctx->eb[9], (size_t)(4 * ldM + 3 * ldN + 64 + tail) * 8));
    int* dinfo = (int*)ctx->d_info.p;
    CUDA_TRY(ctx, cudaMemsetAsync(dinfo, 0, 16, st));
    double* Luu = slA;
    double* Cm = Luu + M * ldM;
    double* LinvU = slLinv;
    double* LinvC = LinvU + linv_bytes(M) / 8;
    double *BtU = (double*)ctx->eb[0].p, *BtC = (double*)ctx->eb[1].p, *Cinv = (double*)ctx->eb[2].p;
    double *T1 = (double*)ctx->eb[3].p, *T2 = (double*)ctx->eb[4].p, *T3 = (double*)ctx->eb[5].p;
    double *E = (double*)ctx->eb[6].p, *GKuft = (double*)ctx->eb[7].p, *GKuf = (double*)ctx->eb[8].p;
    double* vec = (double*)ctx->eb[9].p;
    double *bvec = vec, *u = vec + ldM, *beta = vec + 2 * ldM, *tmpM = vec + 3 * ldM;
    double *tmpN = vec + 4 * ldM, *alpha = tmpN + ldN, *tmpN2 = alpha + ldN;
    double* scal = tmpN2 + ldN;          // [0] sum log LC_ii, [1] u'u, [2] y'y, [3] |W|_F^2, [4] tr(C^-1), [5] alpha'alpha,
                                         // [6] sum kff_diag (caller blocks), [8..] chain
    double* partial = scal + 64;         // M x (d+3)
    double* gXu = partial + M * nth;     // M x d
    dim3 b32(32, 32), gMM((unsigned)ceil_div(M, 32), (unsigned)ceil_div(M, 32));

    // forward pieces shared with the posterior: Luu, W (both layouts), W W^T / noise, W y / noise
    RET_IF(sparse_partial_dev(ctx, sl, kind, dXu, M, dX, N, dy, d, dth, jitter, noise, Luu, ldM, LinvU, Cm, ldM, bvec, dinfo,
                              g ? &g->blocks : nullptr));
    double* Wt = (double*)sl.Vt.p;
    double* W = (double*)sl.cov.p;
    RET_IF(launch(ctx, st, grid_for(M), 256, 0, add_diag_kernel, Cm, ldM, M, 1.0));
    RET_IF(potrf_rec(ctx, st, Cm, ldM, M, LinvC, dinfo + 1, 0));
    CUDA_TRY(ctx, cudaMemcpyAsync(u, bvec, (size_t)M * 8, cudaMemcpyDeviceToDevice, st));
    RET_IF(trsm_rec(ctx, st, u, ldM, 1, Cm, ldM, M, LinvC));
    RET_IF(launch(ctx, st, 1, 256, 0, logdiag_kernel, Cm, ldM, M, scal + 0, (int64_t)0));
    RET_IF(launch(ctx, st, 1, RD_THREADS, 0, rowdot2_kernel, u, ldM, M, nullptr, 1.0, nullptr, scal + 1, (int64_t)0));
    RET_IF(launch(ctx, st, 1, RD_THREADS, 0, rowdot2_kernel, dy, ldN, N, nullptr, 1.0, nullptr, scal + 2, (int64_t)0));
    RET_IF(launch(ctx, st, (unsigned)M, RD_THREADS, 0, rowdot2_kernel, W, ldN, N, nullptr, 1.0, nullptr, tmpM, (int64_t)0));
    RET_IF(launch(ctx, st, 1, 256, 0, vecsum_kernel, tmpM, M, scal + 3));
    if (g) RET_IF(launch(ctx, st, 1, 256, 0, vecsum_kernel, dkff, N, scal + 6));
    // C^{-1} = BtC BtC^T with BtC = (LC^{-1})^T, beta = C^{-1} b
    RET_IF(launch(ctx, st, grid_for(M * M), 256, 0, set_identity_kernel, BtC, ldM, M, (int64_t)0));
    RET_IF(trsm_rec(ctx, st, BtC, ldM, M, Cm, ldM, M, LinvC));
    RET_IF(launch(ctx, st, (unsigned)M, RD_THREADS, 0, rowdot2_kernel, BtC, ldM, M, u, 1.0, beta, tmpM, (int64_t)0));
    RET_IF(launch(ctx, st, 1, 256, 0, vecsum_kernel, tmpM, M, scal + 4));
    RET_IF(gemm_nt(ctx, st, M, M, M, 1.0, BtC, ldM, BtC, ldM, 0.0, Cinv, ldM, true));
    RET_IF(launch(ctx, st, gMM, b32, 0, mirror_lower_kernel, Cinv, ldM, M));
    // alpha = (y - W^T beta) / noise
    RET_IF(launch(ctx, st, (unsigned)N, RD_THREADS, 0, rowdot2_kernel, Wt, ldM, M, beta, 1.0, tmpN, nullptr, (int64_t)0));
    RET_IF(launch(ctx, st, grid_for(N), 256, 0, elbo_alpha_kernel, alpha, dy, tmpN, N, noise));
    RET_IF(launch(ctx, st, 1, RD_THREADS, 0, rowdot2_kernel, alpha, ldN, N, nullptr, 1.0, nullptr, scal + 5, (int64_t)0));
    // the clip of the trace term decides a coefficient of the reverse pass: fetch the scalars now
    double hs[8];
    CUDA_TRY(ctx, cudaMemcpyAsync(hs, scal, sizeof hs, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(ctx, cudaStreamSynchronize(st));
    double kd = scale;
    if (!g && kind == B2GP_KERNEL_MATERN52) {
        const double r = sqrt(1e-12), s5r = 2.23606797749979 * r;
        kd = scale * (1.0 + s5r) * exp(-s5r);
    }
    // sum_n Kff_nn - |W|_F^2: N k(x, x) for the fused kernels, the caller's diagonal otherwise
    const double T = (g ? hs[6] : (double)N * kd) - hs[3];
    const double coef = (T > 0.0) ? 1.0 : 0.0;
    // dELBO/dW^T = alpha beta^T + (coef W^T - W^T C^{-1}) / noise
    RET_IF(gemm_nt(ctx, st, N, M, M, 1.0, Wt, ldM, Cinv, ldM, 0.0, E, ldM, false));
    RET_IF(launch(ctx, st, grid_for(N * M), 256, 0, elbo_gw_kernel, E, ldM, Wt, ldM, alpha, beta, N, M, coef, noise));
    // dELBO/dKuf^T = (dELBO/dW^T) Luu^{-1}
    RET_IF(launch(ctx, st, grid_for(M * M), 256, 0, set_identity_kernel, BtU, ldM, M, (int64_t)0));
    RET_IF(trsm_rec(ctx, st, BtU, ldM, M, Luu, ldM, M, LinvU));
    RET_IF(gemm_nt(ctx, st, N, M, M, 1.0, E, ldM, BtU, ldM, 0.0, GKuft, ldM, false));
    RET_IF(launch(ctx, st, dim3((unsigned)ceil_div(M, 32), (unsigned)ceil_div(N, 32)), dim3(32, 8), 0, transpose_kernel, GKuf, ldN, GKuft, ldM,
                  N, M));
    // H^T = W G_Kuf^T; G_L = -tril(H); dELBO/dKuu = Luu^{-T} Phi(Luu^T G_L) Luu^{-1}
    RET_IF(gemm_nt(ctx, st, M, M, N, 1.0, W, ldN, GKuf, ldN, 0.0, T1, ldM, false));
    RET_IF(launch(ctx, st, gMM, b32, 0, tri_kernel, T2, ldM, T1, ldM, M, 1));                  // T2 = G_L^T = -triu(H^T)
    RET_IF(launch(ctx, st, gMM, b32, 0, tri_kernel, T3, ldM, Luu, ldM, M, 0));                 // T3 = tril(Luu)
    RET_IF(launch(ctx, st, gMM, dim3(32, 8), 0, transpose_kernel, T1, ldM, T3, ldM, M, M));    // T1 = Luu^T
    RET_IF(gemm_nt(ctx, st, M, M, M, 1.0, T1, ldM, T2, ldM, 0.0, T3, ldM, false));   // T3 = Luu^T G_L
    RET_IF(launch(ctx, st, gMM, b32, 0, tri_kernel, T2, ldM, T3, ldM, M, 2));                  // T2 = Phi(.)
    RET_IF(gemm_nt(ctx, st, M, M, M, 1.0, BtU, ldM, T2, ldM, 0.0, T1, ldM, false));  // T1 = BtU P^T
    RET_IF(gemm_nt(ctx, st, M, M, M, 1.0, BtU, ldM, T1, ldM, 0.0, T3, ldM, false));  // T3 = dELBO/dKuu
    RET_IF(launch(ctx, st, gMM, b32, 0, tri_kernel, T2, ldM, T3, ldM, M, 3));                  // T2 = T3 + T3^T
    double* rows = partial;              // caller blocks: [J, M] row sums | ksum [J] | grad [p] | direction table
    double* ksum = rows + J * M;
    double* gdev = ksum + J;
    if (g) {   // Gs = (T3 + T3^T) / 2, the adjoint of the symmetrised Kuu the factorisation reads; Guf = GKuf
        RET_IF(launch(ctx, st, gMM, b32, 0, tri_kernel, T1, ldM, T3, ldM, M, 4));
        RET_IF(sparse_gram_trace(ctx, st, *g, M, N, T1, ldM, GKuf, ldN, -coef / (2.0 * noise), rows, ksum, gdev,
                                 (const double**)(gdev + g->p)));
    } else {   // contract with the kernel derivatives
        RET_IF(launch(ctx, st, (unsigned)M, 256, 0, elbo_chain_kernel, kind, d, dth, dXu, (int)M, dX, N, GKuf, ldN, GKuf, ldN, 0, 0, partial, gXu));
        RET_IF(launch(ctx, st, (unsigned)M, 256, 0, elbo_chain_kernel, kind, d, dth, dXu, (int)M, dXu, M, T3, ldM, T2, ldM, 1, 1, partial, gXu));
        RET_IF(launch(ctx, st, 1, 32, 0, colsum_kernel, partial, M, nth, scal + 8));
    }
    double hs2[8 + MLL_MAX_D + 3];
    int hinfo[2] = {0, 0};
    CUDA_TRY(ctx, cudaMemcpyAsync(hs2, scal, sizeof hs2, cudaMemcpyDeviceToHost, st));
    if (g) {
        if (g->p) CUDA_TRY(ctx, cudaMemcpyAsync(g->grad, gdev, (size_t)g->p * 8, cudaMemcpyDeviceToHost, st));
        if (g->q) CUDA_TRY(ctx, cudaMemcpyAsync(g->grad_rows, rows + g->p * M, (size_t)(g->q * M) * 8, cudaMemcpyDeviceToHost, st));
    } else {
        CUDA_TRY(ctx, cudaMemcpyAsync(grad_Xu, gXu, (size_t)M * d * 8, cudaMemcpyDeviceToHost, st));
    }
    if (alpha_out) CUDA_TRY(ctx, cudaMemcpyAsync(alpha_out, alpha, (size_t)N * 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(ctx, cudaMemcpyAsync(hinfo, dinfo, sizeof hinfo, cudaMemcpyDeviceToHost, st));
    RET_IF(tm.end(st, nullptr));
    *info = hinfo[0] != 0 ? hinfo[0] : -hinfo[1];
    const double n = (double)N, m = (double)M;
    const double loglik = -0.5 * (n * 1.8378770664093453 + n * log(noise) + 2.0 * hs2[0] + hs2[2] / noise - hs2[1]);
    *value = loglik - 0.5 * (T > 0.0 ? T / noise : 0.0);
    const double trSinv = (n - m + hs2[4]) / noise;
    const double glog_noise = noise * (-0.5 * trSinv + 0.5 * hs2[5] + ((T > 0.0) ? 0.5 * T / (noise * noise) : 0.0));
    if (g) {
        if (g->grad_log_noise) *g->grad_log_noise = glog_noise;
    } else {
        for (int k = 0; k < nth; ++k) grad_theta[k] = hs2[8 + k];
        grad_theta[d] += (T > 0.0) ? -0.5 * n * kd / noise : 0.0;
        grad_theta[d + 1] = glog_noise;
    }
    if (*info != 0) {   // grad_Xu too: it was reduced from the failed factor and would otherwise come back finite
        *value = NAN;
        if (g) {
            for (int64_t k = 0; k < g->p; ++k) g->grad[k] = NAN;
            for (int64_t k = 0; k < g->q * M; ++k) g->grad_rows[k] = NAN;
            if (g->grad_log_noise) *g->grad_log_noise = NAN;
        } else {
            for (int k = 0; k < nth; ++k) grad_theta[k] = NAN;
            for (int64_t i = 0; i < M * d; ++i) grad_Xu[i] = NAN;
        }
        if (alpha_out)
            for (int64_t i = 0; i < N; ++i) alpha_out[i] = NAN;
    }
    return B2GP_OK;
}

extern "C" int b2gp_sparse_elbo(b2gp_ctx* ctx, int kind, const double* Xu, int64_t M, const double* X, int64_t N, const double* yres,
                                int d, const double* theta, double jitter, unsigned flags, double* value, double* grad_theta,
                                double* grad_Xu, int* info) {
    return b2gp_sparse_elbo_ex(ctx, kind, Xu, M, X, N, yres, d, theta, jitter, flags, value, grad_theta, grad_Xu, nullptr, info);
}

extern "C" int b2gp_sparse_elbo_ex(b2gp_ctx* ctx, int kind, const double* Xu, int64_t M, const double* X, int64_t N, const double* yres,
                                   int d, const double* theta, double jitter, unsigned flags, double* value, double* grad_theta,
                                   double* grad_Xu, double* alpha_out, int* info) {
    return sparse_elbo_impl(ctx, kind, Xu, M, X, N, yres, d, theta, jitter, flags, value, grad_theta, grad_Xu, alpha_out, info);
}

extern "C" int b2gp_sparse_elbo_gram(b2gp_ctx* ctx, const double* Kuu, int64_t M, const double* Kuf, int64_t N, const double* kff_diag,
                                     const double* yres, double noise, const double* const* dKuu, const double* const* dKuf,
                                     const double* const* dkff, int64_t p, const double* const* rKuu, const double* const* rKuf,
                                     int64_t q, unsigned flags, double* value, double* grad, double* grad_log_noise, double* grad_rows,
                                     double* alpha_out, int* info) {
    if (!ctx) return B2GP_ERR_ARG;
    if (f32_io(flags)) return set_err(ctx, B2GP_ERR_UNSUPPORTED, "b2gp_sparse_elbo_gram", "fp64 arrays only", __FILE__, __LINE__);
    ARG_CHECK(ctx, Kuu && Kuf && kff_diag && p >= 0 && q >= 0);
    ARG_CHECK(ctx, p == 0 || grad);
    ARG_CHECK(ctx, q == 0 || grad_rows);
    const SparseElboGram g{{Kuu, Kuf, nullptr, nullptr, false, dev_ptrs(flags)}, kff_diag, noise, dKuu, dKuf, dkff, p, rKuu, rKuf, q,
                           grad, grad_log_noise, grad_rows};
    return sparse_elbo_impl(ctx, B2GP_KERNEL_RBF, nullptr, M, nullptr, N, yres, 1, nullptr, 0.0, flags, value, nullptr, nullptr, alpha_out,
                            info, &g);
}

// ------------------------------------------------------------------------------------------ MVN sampling
// y[s, i, :] = mean[s, :] + chol(cov[s]) eps[s, i, :]  -- numpyro.distributions.MultivariateNormal(mean, cov).sample
// (call sites gpax/models/gp.py:292, gpax/models/hskgp.py via ExactGP._predict, gpax/acquisition/base_acq.py:221) for
// covariances the caller modified after the posterior call (VarNoiseGP adds the predicted noise to the diagonal).
extern "C" int b2gp_mvn_sample(b2gp_ctx* ctx, const double* mean, const double* cov, int64_t S, int64_t P, const double* eps,
                               int64_t n, double* y, int* info, unsigned flags) {
    if (!ctx) return B2GP_ERR_ARG;
    ARG_CHECK(ctx, mean && cov && eps && y && info && S >= 1 && P >= 1 && n >= 1);
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    const bool dev = dev_ptrs(flags);
    Slot& sl = ctx->slots[0];
    cudaStream_t st = sl.stream;
    CallTimer tm(ctx);
    RET_IF(tm.begin(st));
    const double *dmean, *dcov, *deps;
    RET_IF(stage_in(ctx, st, ctx->d_in[0], mean, (size_t)S * P * 8, dev, &dmean));
    RET_IF(stage_in(ctx, st, ctx->d_in[1], cov, (size_t)S * P * P * 8, dev, &dcov));
    RET_IF(stage_in(ctx, st, ctx->d_in[2], eps, (size_t)S * n * P * 8, dev, &deps));
    double* dy = y;
    if (!dev) {
        RET_IF(ensure(ctx, ctx->d_out[3], (size_t)S * n * P * 8));
        dy = (double*)ctx->d_out[3].p;
    }
    const int64_t ldC = round_up(P, 8);
    RET_IF(ensure(ctx, sl.cov, (size_t)P * ldC * 8));
    RET_IF(ensure(ctx, sl.LinvC, (size_t)linv_bytes(P)));
    RET_IF(ensure(ctx, ctx->d_info, (size_t)S * sizeof(int)));
    int* dinfo = (int*)ctx->d_info.p;
    CUDA_TRY(ctx, cudaMemsetAsync(dinfo, 0, (size_t)S * sizeof(int), st));
    double* CL = (double*)sl.cov.p;
    dim3 g2((unsigned)ceil_div(P, 32), (unsigned)ceil_div(P, 32)), b2(32, 32);
    for (int64_t s = 0; s < S; ++s) {
        RET_IF(launch(ctx, st, grid_for(P * P), 256, 0, copy2d_kernel, CL, ldC, dcov + s * P * P, P, P, P));
        RET_IF(potrf_rec(ctx, st, CL, ldC, P, (double*)sl.LinvC.p, dinfo + s, 0));
        RET_IF(launch(ctx, st, g2, b2, 0, zero_upper_kernel, CL, ldC, P));
        double* Y = dy + s * n * P;
        RET_IF(launch(ctx, st, grid_for(n * P), 256, 0, bcast_rows_kernel, Y, P, n, P, dmean + s * P));
        RET_IF(gemm_nt(ctx, st, n, P, P, 1.0, deps + s * n * P, P, CL, ldC, 1.0, Y, P, false));
        RET_IF(launch(ctx, st, grid_for(n * P), 256, 0, nan_if_bad_kernel, Y, P, n, P, dinfo + s, nullptr));
    }
    CUDA_TRY(ctx, cudaMemcpyAsync(info, dinfo, (size_t)S * sizeof(int), cudaMemcpyDeviceToHost, st));
    if (!dev) CUDA_TRY(ctx, cudaMemcpyAsync(y, dy, (size_t)S * n * P * 8, cudaMemcpyDeviceToHost, st));
    return tm.end(st, nullptr);
}

// ------------------------------------------------------------------------------------------ acquisition epilogues
// see include/b200gp.h; kernels in acq.cuh
extern "C" int b2gp_acq_moments(b2gp_ctx* ctx, int kind, const double* mean, const double* var, int64_t R, int64_t P, int have_best,
                                double best_f, double param, int maximize, double* out, unsigned flags) {
    if (!ctx) return B2GP_ERR_ARG;
    ARG_CHECK(ctx, kind >= ACQ_EI && kind <= ACQ_POI);
    ARG_CHECK(ctx, var && out && R >= 1 && P >= 1);
    ARG_CHECK(ctx, mean || kind == ACQ_UE);
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    const bool dev = dev_ptrs(flags);
    cudaStream_t st = ctx->slots[0].stream;
    CallTimer tm(ctx);
    RET_IF(tm.begin(st));
    const double *dmean, *dvar;
    RET_IF(stage_in(ctx, st, ctx->d_in[0], mean, (size_t)R * P * 8, dev, &dmean));
    RET_IF(stage_in(ctx, st, ctx->d_in[1], var, (size_t)R * P * 8, dev, &dvar));
    double* dout = out;
    if (!dev) {
        RET_IF(ensure(ctx, ctx->d_out[0], (size_t)R * P * 8));
        dout = (double*)ctx->d_out[0].p;
    }
    RET_IF(ensure(ctx, ctx->slots[0].misc, (size_t)(R + 16) * 8));
    double* dbest = (double*)ctx->slots[0].misc.p;
    if (kind == ACQ_EI || kind == ACQ_POI) {
        if (have_best) {
            std::vector<double> hb((size_t)R, best_f);
            CUDA_TRY(ctx, cudaMemcpyAsync(dbest, hb.data(), (size_t)R * 8, cudaMemcpyHostToDevice, st));
            CUDA_TRY(ctx, cudaStreamSynchronize(st));
        } else {
            RET_IF(launch(ctx, st, (unsigned)R, 256, 0, acq_best_kernel, dmean, P, P, maximize, dbest));
        }
    }
    RET_IF(launch(ctx, st, grid_for(R * P), 256, 0, acq_moments_kernel, kind, dmean, dvar, P, R, P, dbest, param, maximize, dout, P));
    if (!dev) CUDA_TRY(ctx, cudaMemcpyAsync(out, dout, (size_t)R * P * 8, cudaMemcpyDeviceToHost, st));
    return tm.end(st, nullptr);
}

extern "C" int b2gp_acq_samples(b2gp_ctx* ctx, int kind, const double* y, int64_t R, int64_t P, int have_best, double best_f,
                                double param, int maximize, double* out, double* mean_out, double* var_out, unsigned flags) {
    if (!ctx) return B2GP_ERR_ARG;
    ARG_CHECK(ctx, kind >= ACQ_EI && kind <= ACQ_POI);
    ARG_CHECK(ctx, y && out && R >= 1 && P >= 1);
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    const bool dev = dev_ptrs(flags);
    cudaStream_t st = ctx->slots[0].stream;
    CallTimer tm(ctx);
    RET_IF(tm.begin(st));
    const double* dy;
    RET_IF(stage_in(ctx, st, ctx->d_in[0], y, (size_t)R * P * 8, dev, &dy));
    RET_IF(ensure(ctx, ctx->d_out[0], (size_t)3 * P * 8));
    double* dm = (double*)ctx->d_out[0].p;
    double* dv = dm + P;
    double* dout = dev ? out : dv + P;
    RET_IF(ensure(ctx, ctx->slots[0].misc, 16 * 8));
    double* dbest = (double*)ctx->slots[0].misc.p;
    RET_IF(launch(ctx, st, (unsigned)ceil_div(P, 128), 128, 0, sample_moments_kernel, dy, R, P, dm, dv));
    if (kind == ACQ_EI || kind == ACQ_POI) {
        if (have_best) {
            CUDA_TRY(ctx, cudaMemcpyAsync(dbest, &best_f, 8, cudaMemcpyHostToDevice, st));
            CUDA_TRY(ctx, cudaStreamSynchronize(st));
        } else {
            RET_IF(launch(ctx, st, 1, 256, 0, acq_best_kernel, dm, P, P, maximize, dbest));
        }
    }
    RET_IF(launch(ctx, st, grid_for(P), 256, 0, acq_moments_kernel, kind, dm, dv, P, 1, P, dbest, param, maximize, dout, P));
    const cudaMemcpyKind kd = dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
    if (!dev) CUDA_TRY(ctx, cudaMemcpyAsync(out, dout, (size_t)P * 8, kd, st));
    if (mean_out) CUDA_TRY(ctx, cudaMemcpyAsync(mean_out, dm, (size_t)P * 8, kd, st));
    if (var_out) CUDA_TRY(ctx, cudaMemcpyAsync(var_out, dv, (size_t)P * 8, kd, st));
    return tm.end(st, nullptr);
}

// The knowledge gradient's rank-1 update on the device; diag_sub_v / nj_v (both or neither) give per-candidate values
static int kg_impl(b2gp_ctx* ctx, const double* mean, const double* cov, int64_t P, const double* ysim, int64_t n, double diag_sub,
                   double noise_plus_jitter, const double* diag_sub_v, const double* nj_v, int maximize, double* out, unsigned flags) {
    if (!ctx) return B2GP_ERR_ARG;
    ARG_CHECK(ctx, mean && cov && ysim && out && P >= 1 && n >= 1);
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    const bool dev = dev_ptrs(flags);
    cudaStream_t st = ctx->slots[0].stream;
    CallTimer tm(ctx);
    RET_IF(tm.begin(st));
    const double *dmean, *dcov, *dys, *dds = nullptr, *dnj = nullptr;
    RET_IF(stage_in(ctx, st, ctx->d_in[0], mean, (size_t)P * 8, dev, &dmean));
    RET_IF(stage_in(ctx, st, ctx->d_in[1], cov, (size_t)P * P * 8, dev, &dcov));
    RET_IF(stage_in(ctx, st, ctx->d_in[2], ysim, (size_t)n * P * 8, dev, &dys));
    if (diag_sub_v) {
        RET_IF(stage_in(ctx, st, ctx->d_in[3], diag_sub_v, (size_t)P * 8, dev, &dds));
        RET_IF(stage_in(ctx, st, ctx->d_in[4], nj_v, (size_t)P * 8, dev, &dnj));
    }
    double* dout = out;
    if (!dev) {
        RET_IF(ensure(ctx, ctx->d_out[0], (size_t)P * 8));
        dout = (double*)ctx->d_out[0].p;
    }
    RET_IF(ensure(ctx, ctx->slots[0].misc, 16 * 8));
    double* dbest = (double*)ctx->slots[0].misc.p;
    RET_IF(launch(ctx, st, 1, 256, 0, acq_best_kernel, dmean, P, P, maximize, dbest));
    if (diag_sub_v)
        RET_IF(launch(ctx, st, (unsigned)P, 256, 0, kg_kernel<true>, dmean, dcov, P, dys, (int)n, P, diag_sub, noise_plus_jitter, dds, dnj,
                      maximize, dbest, dout));
    else
        RET_IF(launch(ctx, st, (unsigned)P, 256, 0, kg_kernel<false>, dmean, dcov, P, dys, (int)n, P, diag_sub, noise_plus_jitter, dds, dnj,
                      maximize, dbest, dout));
    if (!dev) CUDA_TRY(ctx, cudaMemcpyAsync(out, dout, (size_t)P * 8, cudaMemcpyDeviceToHost, st));
    return tm.end(st, nullptr);
}

extern "C" int b2gp_kg(b2gp_ctx* ctx, const double* mean, const double* cov, int64_t P, const double* ysim, int64_t n,
                       double diag_sub, double noise_plus_jitter, int maximize, double* out, unsigned flags) {
    return kg_impl(ctx, mean, cov, P, ysim, n, diag_sub, noise_plus_jitter, nullptr, nullptr, maximize, out, flags);
}

extern "C" int b2gp_kg_v(b2gp_ctx* ctx, const double* mean, const double* cov, int64_t P, const double* ysim, int64_t n,
                         const double* diag_sub, const double* noise_plus_jitter, int maximize, double* out, unsigned flags) {
    if (!ctx) return B2GP_ERR_ARG;
    ARG_CHECK(ctx, diag_sub && noise_plus_jitter);
    return kg_impl(ctx, mean, cov, P, ysim, n, 0.0, 0.0, diag_sub, noise_plus_jitter, maximize, out, flags);
}

// ------------------------------------------------------------------------------------------ debug
// Development aid (not part of include/b200gp.h): run the leaf kernel on a device block with per-phase
// clock64 / globaltimer stamps.  prof_host receives 2*16 values (cycles, ns) per stamp.
extern "C" int b2gp_debug_leaf(b2gp_ctx* ctx, int n, double* A_dev, int64_t lda, double* linv_dev, long long* prof_host) {
    if (!ctx) return B2GP_ERR_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->slots[0].stream;
    RET_IF(ensure(ctx, ctx->d_info, 64 + 128 * 8));
    int* dinfo = (int*)ctx->d_info.p;
    long long* dprof = (long long*)((char*)ctx->d_info.p + 64);
    CUDA_TRY(ctx, cudaMemsetAsync(ctx->d_info.p, 0, 64 + 128 * 8, st));
    static PerDeviceOnce attr;
    if (attr.need(ctx->device)) {
        CUDA_TRY(ctx, cudaFuncSetAttribute(potrf_diag_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, PD_SMEM));
        attr.done(ctx->device);
    }
    RET_IF(launch(ctx, st, 1, PD_THREADS, PD_SMEM, potrf_diag_kernel, A_dev, lda, n, linv_dev, dinfo, 0, dprof, (int64_t)0));
    CUDA_TRY(ctx, cudaMemcpyAsync(prof_host, dprof, 64 * 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(ctx, cudaStreamSynchronize(st));
    return B2GP_OK;
}

// Development aid: time one GEMM/SYRK launch with an explicit tile configuration (device pointers).
extern "C" int b2gp_debug_gemm_cfg(b2gp_ctx* ctx, int cfg, int64_t m, int64_t n, int64_t k, const double* A, int64_t lda,
                                   const double* B, int64_t ldb, double* C, int64_t ldc, int lower, double* ms_out) {
    if (!ctx) return B2GP_ERR_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->slots[0].stream;
    GemmArgs a;
    a.m = (int)m; a.n = (int)n; a.k = (int)k; a.A = A; a.lda = lda; a.B = B; a.ldb = ldb; a.C = C; a.ldc = ldc;
    a.alpha = -1.0; a.beta = 1.0; a.lower_only = lower;
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_a, st));
    int rc = B2GP_ERR_ARG;
    switch (cfg) {
        case 0: rc = launch_gemm_cfg<128, 128, 2, 4, 4, 1>(ctx, st, a); break;
        case 1: rc = launch_gemm_cfg<128, 128, 4, 4, 4, 1>(ctx, st, a); break;
        case 2: rc = launch_gemm_cfg<128, 128, 2, 4, 3, 1>(ctx, st, a); break;
        case 3: rc = launch_gemm_cfg<128, 128, 4, 2, 4, 1>(ctx, st, a); break;
        case 4: rc = launch_gemm_cfg<128, 128, 2, 8, 4, 1>(ctx, st, a); break;
        case 5: rc = launch_gemm_cfg<128, 128, 4, 4, 3, 1>(ctx, st, a); break;
        // the latency-bound and lower-only configurations of gemm_nt
        case 6: rc = launch_gemm_cfg<32, 128, 1, 8, 3, 2>(ctx, st, a); break;
        case 7: rc = launch_gemm_cfg<64, 128, 2, 4, 3, 2>(ctx, st, a); break;
        case 8: rc = launch_gemm_cfg<64, 64, 2, 4, 4, 2>(ctx, st, a); break;
        default: break;
    }
    RET_IF(rc);
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_b, st));
    CUDA_TRY(ctx, cudaEventSynchronize(ctx->ev_b));
    float ms = 0.f;
    CUDA_TRY(ctx, cudaEventElapsedTime(&ms, ctx->ev_a, ctx->ev_b));
    *ms_out = ms;
    return B2GP_OK;
}

// Development aid: C[m,n] += alpha * A B^T through the int8 wgmma path (ozaki.cuh), device pointers, S = 6 or 7 digit planes.
extern "C" int b2gp_debug_ozaki(b2gp_ctx* ctx, int S, int64_t m, int64_t n, int64_t k, double alpha, const double* A, int64_t lda,
                                const double* B, int64_t ldb, double* C, int64_t ldc, int lower, double* ms_out) {
    if (!ctx) return B2GP_ERR_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->slots[0].stream;
    const size_t prof_bytes = (size_t)ctx->sm_count * 8 * sizeof(long long);   // [CTA][8], one CTA per SM at most
    RET_IF(ensure(ctx, ctx->slots[0].oz.prof, prof_bytes));
    CUDA_TRY(ctx, cudaMemsetAsync(ctx->slots[0].oz.prof.p, 0, prof_bytes, st));
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_a, st));
    int rc;
    if (S == 6)
        rc = ozaki_gemm_nt<6>(ctx, st, ctx->slots[0].oz, m, n, k, alpha, A, lda, B, ldb, C, ldc, lower != 0);
    else
        rc = ozaki_gemm_nt<7>(ctx, st, ctx->slots[0].oz, m, n, k, alpha, A, lda, B, ldb, C, ldc, lower != 0);
    RET_IF(rc);
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_b, st));
    CUDA_TRY(ctx, cudaEventSynchronize(ctx->ev_b));
    float ms = 0.f;
    CUDA_TRY(ctx, cudaEventElapsedTime(&ms, ctx->ev_a, ctx->ev_b));
    if (ms_out) *ms_out = ms;
    {
        std::vector<long long> h((size_t)ctx->sm_count * 8);
        CUDA_TRY(ctx, cudaMemcpy(h.data(), ctx->slots[0].oz.prof.p, prof_bytes, cudaMemcpyDeviceToHost));
        double w = 0, e = 0, t = 0, me = 0, mt = 0;
        for (int i = 0; i < ctx->sm_count; ++i) {
            w += h[8 * i]; e += h[8 * i + 1]; t += h[8 * i + 3];
            me += h[8 * i + 5]; mt += h[8 * i + 6];
        }
        if (t > 0 && getenv("B2GP_OZ_PROF"))
            fprintf(stderr, "[oz prof] per tile: consumers wait for TMA %.0f cyc, epilogue (C update) %.0f cyc; producer: total %.0f, "
                            "waits for a free stage %.0f; tiles %.0f, k-blocks/tile %lld\n",
                    w / t, e / t, mt / t, me / t, t, (long long)((k + 31) / 32));
    }
    return B2GP_OK;
}

// Development aid / roofline denominator: the measured int8 wgmma ceiling in TOP/s (see oz_i8_peak_kernel), best of `reps`.
extern "C" int b2gp_debug_i8_peak(b2gp_ctx* ctx, int iters, int reps, double* tops_out, double* ms_out) {
    if (!ctx || !tops_out || iters < 4 || reps < 1) return B2GP_ERR_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->slots[0].stream;
    const int smem = 200 * 1024;   // one CTA per SM
    static PerDeviceOnce attr;
    if (attr.need(ctx->device)) {
        CUDA_TRY(ctx, cudaFuncSetAttribute(oz_i8_peak_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        attr.done(ctx->device);
    }
    double best = 1e30;
    for (int r = 0; r < reps + 1; ++r) {
        CUDA_TRY(ctx, cudaEventRecord(ctx->ev_a, st));
        RET_IF(launch(ctx, st, ctx->sm_count, OZ_PEAK_THREADS, smem, oz_i8_peak_kernel, iters, nullptr));
        CUDA_TRY(ctx, cudaEventRecord(ctx->ev_b, st));
        CUDA_TRY(ctx, cudaEventSynchronize(ctx->ev_b));
        float ms = 0.f;
        CUDA_TRY(ctx, cudaEventElapsedTime(&ms, ctx->ev_a, ctx->ev_b));
        if (r > 0 && ms < best) best = ms;
    }
    *tops_out = 2.0 * 64 * 256 * 32 * (OZ_PEAK_THREADS / 128) * (double)iters * ctx->sm_count / (best * 1e-3) / 1e12;
    if (ms_out) *ms_out = best;
    return B2GP_OK;
}

// Development aid: the measured fp64 tensor ceiling in TFLOP/s of one DMMA shape (see dmma_peak_kernel; 0: m8n8k4,
// 1: m16n8k4, 2: m16n8k8, 3: m16n8k16), best of `reps`.
extern "C" int b2gp_debug_dmma_peak(b2gp_ctx* ctx, int shape, int iters, int reps, double* tflops_out, double* ms_out) {
    if (!ctx || !tflops_out || shape < 0 || shape > 3 || iters < 4 || reps < 1) return B2GP_ERR_ARG;
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->slots[0].stream;
    void (*const kern[4])(int, double*) = {dmma_peak_kernel<0>, dmma_peak_kernel<1>, dmma_peak_kernel<2>, dmma_peak_kernel<3>};
    double best = 1e30;
    for (int r = 0; r < reps + 1; ++r) {
        CUDA_TRY(ctx, cudaEventRecord(ctx->ev_a, st));
        RET_IF(launch(ctx, st, ctx->sm_count, DMMA_PEAK_THREADS, 0, kern[shape], iters, nullptr));
        CUDA_TRY(ctx, cudaEventRecord(ctx->ev_b, st));
        CUDA_TRY(ctx, cudaEventSynchronize(ctx->ev_b));
        float ms = 0.f;
        CUDA_TRY(ctx, cudaEventElapsedTime(&ms, ctx->ev_a, ctx->ev_b));
        if (r > 0 && ms < best) best = ms;
    }
    *tflops_out = 2.0 * dmma_peak_fma(shape) * DMMA_PEAK_ACC * (DMMA_PEAK_THREADS / 32) * (double)iters * ctx->sm_count / (best * 1e-3) / 1e12;
    if (ms_out) *ms_out = best;
    return B2GP_OK;
}

// ------------------------------------------------------------------------------------------ multi-GPU (dist.cuh)
extern "C" int b2gp_dist_unique_id(void* id128) {
    if (!id128) return B2GP_ERR_ARG;
    NcclApi* n = nccl_api();
    if (!n->handle || !n->error.empty()) return B2GP_ERR_UNSUPPORTED;
    static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
    ncclUniqueId id;
    if (n->GetUniqueId(&id) != ncclSuccess) return B2GP_ERR_CUDA;
    memcpy(id128, &id, 128);
    return B2GP_OK;
}

extern "C" int b2gp_dist_finalize(b2gp_ctx* ctx) {
    if (!ctx) return B2GP_ERR_ARG;
    if (ctx->dist) {
        cudaSetDevice(ctx->device);
        cudaDeviceSynchronize();
        ctx->dist.reset();
    }
    return B2GP_OK;
}

extern "C" int b2gp_dist_init(b2gp_ctx* ctx, const void* id128, int rank, int nranks, int grid_rows, int grid_cols) {
    if (!ctx) return B2GP_ERR_ARG;
    ARG_CHECK(ctx, id128 && nranks >= 1 && rank >= 0 && rank < nranks);
    ARG_CHECK(ctx, grid_rows >= 1 && grid_cols >= 1 && grid_rows * grid_cols == nranks);
    NcclApi* n = nccl_api();
    if (!n->handle || !n->error.empty())
        return set_err(ctx, B2GP_ERR_UNSUPPORTED, "b2gp_dist_init", n->error.c_str(), __FILE__, __LINE__);
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (ctx->dist) RET_IF(b2gp_dist_finalize(ctx));
    ctx->dist = std::make_unique<DistState>();
    DistState* ds = ctx->dist.get();
    ds->rank = rank;
    ds->nranks = nranks;
    ds->g.pr = grid_rows;
    ds->g.pc = grid_cols;
    ds->g.myrow = rank / grid_cols;     // row-major process grid
    ds->g.mycol = rank % grid_cols;
    ncclUniqueId id;
    memcpy(&id, id128, 128);
    NCCL_TRY(ctx, n->CommInitRank(&ds->world, nranks, id, rank));
    // row communicator: the pc processes of my grid row, ranked by column; column communicator: the pr processes of my
    // grid column, ranked by row
    NCCL_TRY(ctx, n->CommSplit(ds->world, ds->g.myrow, ds->g.mycol, &ds->rowc, nullptr));
    NCCL_TRY(ctx, n->CommSplit(ds->world, ds->g.mycol, ds->g.myrow, &ds->colc, nullptr));
    CUDA_TRY(ctx, cudaStreamCreateWithFlags(&ds->ms, cudaStreamNonBlocking));
    CUDA_TRY(ctx, cudaStreamCreateWithFlags(&ds->dq, cudaStreamNonBlocking));
    for (cudaEvent_t* e : {&ds->ev_u, &ds->ev_ubc[0], &ds->ev_ubc[1], &ds->ev_chunk, &ds->ev_comm[0], &ds->ev_comm[1], &ds->ev_done, &ds->ev_e,
                           &ds->ev_early[0], &ds->ev_early[1], &ds->ev_g2})
        CUDA_TRY(ctx, cudaEventCreateWithFlags(e, cudaEventDisableTiming));
    ds->ready = true;
    return B2GP_OK;
}

extern "C" int b2gp_dist_info(b2gp_ctx* ctx, int* rank, int* nranks, int* grid_rows, int* grid_cols) {
    if (!ctx) return B2GP_ERR_ARG;
    DistState* ds = ctx->dist.get();
    if (!ds || !ds->ready) return set_err(ctx, B2GP_ERR_ARG, "b2gp_dist_info", "call b2gp_dist_init first", __FILE__, __LINE__);
    if (rank) *rank = ds->rank;
    if (nranks) *nranks = ds->nranks;
    if (grid_rows) *grid_rows = ds->g.pr;
    if (grid_cols) *grid_cols = ds->g.pc;
    return B2GP_OK;
}

// Pure index algebra of the block-cyclic layout (no GPU, no NCCL): for the process at (row, col) of a pr x pc grid,
// out[0] = local tile rows, out[1] = local tile columns, out[2] = rows of the panel of step k it holds, out[3] = slot
// rows of the panel buffer at step k, out[4] = first local tile row after k, out[5] = first local tile column after k.
extern "C" int b2gp_dist_layout(int64_t T, int64_t R, int64_t nb, int pr, int pc, int row, int col, int64_t k, int64_t* out) {
    if (!out || T < 1 || R < 0 || nb < 1 || pr < 1 || pc < 1 || row < 0 || row >= pr || col < 0 || col >= pc || k < 0) return B2GP_ERR_ARG;
    BcGrid g;
    g.pr = pr;
    g.pc = pc;
    g.myrow = row;
    g.mycol = col;
    g.nb = nb;
    g.T = T;
    g.R = R;
    out[0] = g.lr(row);
    out[1] = g.lc(col);
    out[2] = g.panel_rows(k, row);
    out[3] = g.slot_rows(k);
    out[4] = g.first_row_after(k, row);
    out[5] = g.first_col_after(k, col);
    return B2GP_OK;
}

// staircase tile lists and B-operand row maps of every step, for the current grid / problem shape
static int dist_build_steps(b2gp_ctx* ctx, DistState* ds, cudaStream_t st, int CL) {
    const BcGrid& g = ds->g;
    if (ds->cache_T == g.T && ds->cache_R == g.R && ds->cache_nb == g.nb && ds->cache_cl == CL) return B2GP_OK;
    CUDA_TRY(ctx, cudaStreamSynchronize(st));   // lists of a previous shape may still be in use
    ds->steps.clear();
    ds->steps.resize((size_t)g.T);
    const int64_t nb = g.nb, t128 = nb / 128;          // 128-row groups per tile
    const int64_t colw = CL == 2 ? 128 : 64;           // columns covered by one list entry
    const int64_t ent_per_tile = nb / colw;
    for (int64_t k = 0; k < g.T; ++k) {
        DistStep& s = ds->steps[(size_t)k];
        const int64_t li0 = g.first_row_after(k, g.myrow), lj0 = g.first_col_after(k, g.mycol);
        const int64_t ntr = g.lr(g.myrow) - li0, ntc = g.lc(g.mycol) - lj0;    // local tile rows / columns of the trailing matrix
        if (ntr <= 0 || ntc <= 0) continue;
        // B operand: the panel tiles (gj, k) of my tile columns gj > k, found in slot gj % pr of the panel buffer
        const int64_t slot = g.slot_rows(k);
        std::vector<int64_t> bmap((size_t)(ntc * t128));
        for (int64_t c = 0; c < ntc; ++c) {
            const int64_t gj = (lj0 + c) * g.pc + g.mycol;
            const int r = (int)(gj % g.pr);
            const int64_t src = (int64_t)r * slot + (gj / g.pr - g.first_row_after(k, r)) * nb;
            for (int64_t q = 0; q < t128; ++q) bmap[(size_t)(c * t128 + q)] = src + q * 128;
        }
        RET_IF(ensure(ctx, s.bmap, bmap.size() * 8));
        CUDA_TRY(ctx, cudaMemcpyAsync(s.bmap.p, bmap.data(), bmap.size() * 8, cudaMemcpyHostToDevice, st));
        // staircase: 128-row tile ti of local tile row a (global gi) x column entry of local tile column c (global gj), gi >= gj
        std::vector<int2> l1, l2;
        const int64_t next_col = (k + 1 < g.T && (k + 1) % g.pc == g.mycol) ? (k + 1) / g.pc - lj0 : -1;   // local index (in the trailing matrix) of tile column k+1
        const int G = 8;
        const int64_t rows128 = ntr * t128;
        for (int64_t b0 = 0; b0 < rows128; b0 += G) {
            const int64_t b1 = std::min(b0 + G, rows128);
            for (int64_t c = 0; c < ntc; ++c) {
                const int64_t gj = (lj0 + c) * g.pc + g.mycol;
                for (int64_t e = 0; e < ent_per_tile; ++e)
                    for (int64_t ti = b0; ti < b1; ++ti) {
                        const int64_t gi = (li0 + ti / t128) * g.pr + g.myrow;
                        if (gi < gj) continue;
                        if (gi == k + 1 && gj == k + 1) continue;    // the next diagonal tile takes panel k on the diagonal stream (diag_factor)
                        (c == next_col ? l1 : l2).push_back(make_int2((int)ti, (int)(c * ent_per_tile + e)));
                    }
            }
        }
        s.n1 = (int64_t)l1.size();
        s.n2 = (int64_t)l2.size();
        if (s.n1) {
            RET_IF(ensure(ctx, s.g1, l1.size() * sizeof(int2)));
            CUDA_TRY(ctx, cudaMemcpyAsync(s.g1.p, l1.data(), l1.size() * sizeof(int2), cudaMemcpyHostToDevice, st));
        }
        if (s.n2) {
            RET_IF(ensure(ctx, s.g2, l2.size() * sizeof(int2)));
            CUDA_TRY(ctx, cudaMemcpyAsync(s.g2.p, l2.data(), l2.size() * sizeof(int2), cudaMemcpyHostToDevice, st));
        }
        CUDA_TRY(ctx, cudaStreamSynchronize(st));   // the host vectors die here
    }
    ds->cache_T = g.T;
    ds->cache_R = g.R;
    ds->cache_nb = g.nb;
    ds->cache_cl = CL;
    return B2GP_OK;
}

// Exact-GP posterior (mean + diagonal variance) with k_XX distributed over the process grid.  COLLECTIVE: every rank
// calls it with the same (replicated) inputs -- X, y, X_new and theta are a few hundred KB, only K is big.  HOST pointers.
extern "C" int b2gp_dist_posterior(b2gp_ctx* ctx, int kind, const double* Xtr, int64_t N, const double* yres, const double* Xnew,
                                   int64_t P, int d, const double* theta, int noiseless, double jitter, int64_t nb, unsigned flags,
                                   double* mean, double* var, int* info, b2gp_timing* timing) {
    if (!ctx) return B2GP_ERR_ARG;
    DistState* ds = ctx->dist.get();
    if (!ds || !ds->ready) return set_err(ctx, B2GP_ERR_ARG, "b2gp_dist_posterior", "call b2gp_dist_init first", __FILE__, __LINE__);
    ARG_CHECK(ctx, kind >= 0 && kind <= 2);
    ARG_CHECK(ctx, Xtr && yres && Xnew && theta && mean && info);
    ARG_CHECK(ctx, N >= 1 && P >= 1 && d >= 1 && d <= GRAM_MAX_D);
    ARG_CHECK(ctx, nb >= 128 && nb <= 1024 && nb % 128 == 0 && N % nb == 0);
    ARG_CHECK(ctx, !(flags & B2GP_FLAG_DEVICE_PTRS) && !(flags & (B2GP_OUT_COV | B2GP_OUT_SAMPLE)));
    const bool want_var = flags & B2GP_OUT_VAR;
    ARG_CHECK(ctx, !want_var || var);
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    NcclApi* nc = nccl_api();
    ctx->fcache.valid = false;
    Slot& sl = ctx->slots[0];
    cudaStream_t cs = sl.stream, ms = ds->ms;
    BcGrid& g = ds->g;
    g.nb = nb;
    g.T = N / nb;
    g.R = ceil_div(P + 1, nb);
    const int pr = g.pr, pc = g.pc, myrow = g.myrow, mycol = g.mycol;
    const int64_t T = g.T, Lr = g.lr(myrow), Lc = g.lc(mycol), ld = Lc * nb;
    const int CL = (ctx->oz_cluster == 2) ? 2 : 1;
    const int nth = d + 3;
    CallTimer tm(ctx);
    RET_IF(tm.begin(cs));
    RET_IF(dist_build_steps(ctx, ds, cs, CL));

    // ---- inputs: the rows / columns of X this process's tiles need, gathered on the host (a few hundred KB)
    std::vector<double> xr((size_t)(Lr * nb * d)), zc((size_t)std::max<int64_t>(Lc * nb * d, 1)), yl((size_t)std::max<int64_t>(Lc * nb, 1));
    for (int64_t li = 0; li < Lr; ++li) {
        const int64_t gi = li * pr + myrow;
        for (int64_t r = 0; r < nb; ++r) {
            const double* src;
            if (gi < T)
                src = Xtr + (gi * nb + r) * d;
            else {
                const int64_t p = (gi - T) * nb + r;
                src = Xnew + (p < P ? p : 0) * d;       // padding rows repeat a valid point; their results are never read
            }
            memcpy(&xr[(size_t)((li * nb + r) * d)], src, (size_t)d * 8);
        }
    }
    for (int64_t lj = 0; lj < Lc; ++lj) {
        const int64_t gj = lj * pc + mycol;
        memcpy(&zc[(size_t)(lj * nb * d)], Xtr + gj * nb * d, (size_t)(nb * d) * 8);
        memcpy(&yl[(size_t)(lj * nb)], yres + gj * nb, (size_t)nb * 8);
    }
    RET_IF(ensure(ctx, ds->Xrows, xr.size() * 8));
    RET_IF(ensure(ctx, ds->Zcols, zc.size() * 8));
    RET_IF(ensure(ctx, ds->yloc, yl.size() * 8));
    RET_IF(ensure(ctx, ctx->d_in[3], (size_t)nth * 8));
    RET_IF(ensure(ctx, ds->Aloc, (size_t)std::max<int64_t>(Lr * nb * ld, 1) * 8));
    RET_IF(ensure(ctx, ds->UB, (size_t)2 * nb * nb * 8));     // U of two consecutive steps
    RET_IF(ensure(ctx, ds->EB, (size_t)2 * nb * nb * 8));     // early tiles of two consecutive steps
    RET_IF(ensure(ctx, ds->linv, (size_t)linv_bytes(nb)));
    RET_IF(ensure(ctx, ds->red, (size_t)(4 * P + 64) * 8));
    RET_IF(ensure(ctx, ds->wseg, (size_t)std::max<int64_t>(ld, 1) * 8));
    const int64_t slot0 = g.slot_rows(0);
    for (int b = 0; b < 2; ++b) RET_IF(ensure(ctx, ds->PB[b], (size_t)std::max<int64_t>(pr * slot0 * nb, 1) * 8));
    RET_IF(ensure(ctx, ctx->d_info, 64));
    int* dinfo = (int*)ctx->d_info.p;
    CUDA_TRY(ctx, cudaMemcpyAsync(ds->Xrows.p, xr.data(), xr.size() * 8, cudaMemcpyHostToDevice, cs));
    CUDA_TRY(ctx, cudaMemcpyAsync(ds->Zcols.p, zc.data(), zc.size() * 8, cudaMemcpyHostToDevice, cs));
    CUDA_TRY(ctx, cudaMemcpyAsync(ds->yloc.p, yl.data(), yl.size() * 8, cudaMemcpyHostToDevice, cs));
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_in[3].p, theta, (size_t)nth * 8, cudaMemcpyHostToDevice, cs));
    CUDA_TRY(ctx, cudaMemsetAsync(dinfo, 0, 16, cs));
    CUDA_TRY(ctx, cudaStreamSynchronize(cs));   // the host staging vectors are pageable
    const double* dth = (const double*)ctx->d_in[3].p;
    double* A = (double*)ds->Aloc.p;
    // The block-cyclic factorisation has no fp64 trailing update to fall back to: every panel solve and update is an int8
    // GEMM, so ozaki == 0 (the library default) means "planes from the conditioning bound" here, like -1.
    sl.oz_planes = ctx->ozaki > 0 ? ctx->ozaki : oz_auto_planes((double)N, theta[d], theta[d + 1], jitter);

    // ---- the local matrix, generated in place: k(rows, columns) for every local tile, then the diagonal term and y
    if (Lr > 0 && Lc > 0) {
        RET_IF(launch_gram(ctx, cs, kind, (const double*)ds->Xrows.p, Lr * nb, (const double*)ds->Zcols.p, Lc * nb, d, dth, 0.0, 0.0, 0, 0, A, ld));
        int64_t gi0 = -1, step = 0, count = 0;
        for (int64_t gi = 0; gi < T; ++gi)
            if (gi % pr == myrow && gi % pc == mycol) {
                if (gi0 < 0)
                    gi0 = gi;
                else if (step == 0)
                    step = gi - gi0;
                ++count;
            }
        if (count > 0)
            RET_IF(launch(ctx, cs, grid_for(count * nb), 256, 0, dist_diag_kernel, A, ld, nb, pr, pc, gi0, step ? step : 1, count, dth, d, jitter));
        const int64_t gy = T + P / nb;                      // tile row holding the y^T right-hand side (global rhs row P)
        if (gy % pr == myrow)
            CUDA_TRY(ctx, cudaMemcpyAsync(A + ((gy / pr) * nb + P % nb) * ld, ds->yloc.p, (size_t)ld * 8, cudaMemcpyDeviceToDevice, cs));
    }
    cudaEvent_t ev_f0 = ctx->slots[0].ev[2], ev_f1 = ctx->slots[0].ev[3];
    CUDA_TRY(ctx, cudaEventRecord(ev_f0, cs));

    // optional phase profile (B2GP_DIST_PROF=1): CUDA events on the streams, summed per phase after the call
    const bool prof = getenv("B2GP_DIST_PROF") != nullptr;
    enum { PH_SLICE, PH_G1, PH_POTRF, PH_UWAIT, PH_PANEL, PH_G2, PH_COMMWAIT, PH_UBCAST, PH_ROWBCAST, PH_ALLGATHER, PH_EARLY, PH_N };
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> pev[PH_N];
    auto mark = [&](cudaStream_t s) -> cudaEvent_t {
        if (!prof) return nullptr;
        cudaEvent_t e = ctx->pool.get();
        cudaEventRecord(e, s);
        return e;
    };
    auto span = [&](int ph, cudaEvent_t a, cudaEvent_t b) {
        if (prof && a && b) pev[ph].emplace_back(a, b);
    };
    cudaStream_t dq = ds->dq;                         // the diagonal tiles are factored on their own stream, one step ahead
    double* UBs[2] = {(double*)ds->UB.p, (double*)ds->UB.p + nb * nb};
    double* EBs[2] = {(double*)ds->EB.p, (double*)ds->EB.p + nb * nb};
    auto diag_tile = [&](int64_t k) { return A + ((k / pr) * nb) * ld + (k / pc) * nb; };

    // ---- (a), (b) of step k on stream s: the owner folds in the tile (k, k-1) it received ahead of the panel
    // (`early`), factors the diagonal tile and forms U = L_kk^{-T}; every rank of the process column joins the broadcast
    // of U on the communication stream.  ev_ubc[k & 1] marks "U_k is here" for the panel solve.
    auto diag_factor = [&](int64_t k, cudaStream_t s, bool early) -> int {
        const int kr = (int)(k % pr), kc = (int)(k % pc);
        if (mycol != kc) return B2GP_OK;
        double* U = UBs[k & 1];
        if (myrow == kr) {
            cudaEvent_t p0 = mark(s);
            double* D = diag_tile(k);
            if (early) {   // D -= E E^T, E = L tile (k, k-1): from the early broadcast, or in place when this rank solved it itself
                const bool local = (pc == 1);
                const double* E = local ? A + (g.first_row_after(k - 1, myrow) * nb) * ld + ((k - 1) / pc) * nb : EBs[(k - 1) & 1];
                RET_IF(gemm_nt(ctx, s, nb, nb, nb, -1.0, E, local ? ld : nb, E, local ? ld : nb, 1.0, D, ld, true));
            }
            RET_IF(potrf_rec(ctx, s, D, ld, nb, (double*)ds->linv.p, dinfo, k * nb));
            RET_IF(launch(ctx, s, grid_for(nb * nb), 256, 0, set_identity_kernel, U, nb, nb, (int64_t)0));
            RET_IF(trsm_rec(ctx, s, U, nb, nb, D, ld, nb, (const double*)ds->linv.p));      // U = L_kk^{-T}
            span(PH_POTRF, p0, mark(s));
        }
        if (pr > 1) {
            CUDA_TRY(ctx, cudaEventRecord(ds->ev_u, s));
            CUDA_TRY(ctx, cudaStreamWaitEvent(ms, ds->ev_u, 0));
            cudaEvent_t m0 = mark(ms);
            NCCL_TRY(ctx, nc->Broadcast(U, U, (size_t)(nb * nb), ncclDouble, kr, ds->colc, ms));
            span(PH_UBCAST, m0, mark(ms));
            CUDA_TRY(ctx, cudaEventRecord(ds->ev_ubc[k & 1], ms));
        } else {
            CUDA_TRY(ctx, cudaEventRecord(ds->ev_ubc[k & 1], s));
        }
        return B2GP_OK;
    };
    // ---- (c) .. (f) of step k on the compute stream: panel solve once U is here, the tile (k+1, k) sent ahead to the owner
    // of the next diagonal tile (row communicator), pack, panel exchange
    auto panel_front_b = [&](int64_t k) -> int {
        const int kc = (int)(k % pc);
        const int64_t li0 = g.first_row_after(k, myrow), rows = g.panel_rows(k, myrow), slot = g.slot_rows(k);
        double* PBk = (double*)ds->PB[k & 1].p;
        double* rp = A + (li0 * nb) * ld + (k / pc) * nb;
        if (mycol == kc) {
            cudaEvent_t p1 = mark(cs);
            CUDA_TRY(ctx, cudaStreamWaitEvent(cs, ds->ev_ubc[k & 1], 0));
            cudaEvent_t p0 = mark(cs);
            span(PH_UWAIT, p1, p0);
            if (rows > 0) RET_IF(ozaki_dispatch(ctx, cs, rows, nb, nb, 1.0, rp, ld, UBs[k & 1], nb, rp, ld, false, true, true, true));
        }
        if (k + 1 < T && myrow == (int)((k + 1) % pr)) {      // my process row holds tile (k+1, k) -- the first tile of its panel rows
            if (pc > 1) {
                if (mycol == kc) RET_IF(launch(ctx, cs, grid_for(nb * nb), 256, 0, copy2d_kernel, EBs[k & 1], nb, rp, ld, nb, nb));
                CUDA_TRY(ctx, cudaEventRecord(ds->ev_e, cs));
                CUDA_TRY(ctx, cudaStreamWaitEvent(ms, ds->ev_e, 0));
                cudaEvent_t m0 = mark(ms);
                NCCL_TRY(ctx, nc->Broadcast(EBs[k & 1], EBs[k & 1], (size_t)(nb * nb), ncclDouble, kc, ds->rowc, ms));
                span(PH_EARLY, m0, mark(ms));
                CUDA_TRY(ctx, cudaEventRecord(ds->ev_early[k & 1], ms));
            } else {
                CUDA_TRY(ctx, cudaEventRecord(ds->ev_early[k & 1], cs));
            }
        }
        if (mycol == kc) {
            cudaEvent_t p0 = mark(cs);
            if (rows > 0) RET_IF(launch(ctx, cs, grid_for(rows * nb), 256, 0, copy2d_kernel, PBk + (int64_t)myrow * slot * nb, nb, rp, ld, rows, nb));
            span(PH_PANEL, p0, mark(cs));
        }
        if (slot > 0) {
            CUDA_TRY(ctx, cudaEventRecord(ds->ev_chunk, cs));
            CUDA_TRY(ctx, cudaStreamWaitEvent(ms, ds->ev_chunk, 0));
            double* mine = PBk + (int64_t)myrow * slot * nb;
            cudaEvent_t m0 = mark(ms);
            if (pc > 1) NCCL_TRY(ctx, nc->Broadcast(mine, mine, (size_t)(slot * nb), ncclDouble, kc, ds->rowc, ms));
            cudaEvent_t m1 = mark(ms);
            span(PH_ROWBCAST, m0, m1);
            if (pr > 1) NCCL_TRY(ctx, nc->AllGather(mine, PBk, (size_t)(slot * nb), ncclDouble, ds->colc, ms));
            span(PH_ALLGATHER, m1, mark(ms));
        }
        CUDA_TRY(ctx, cudaEventRecord(ds->ev_comm[k & 1], ms));
        return B2GP_OK;
    };
    // ---- diagonal look-ahead: tile j's last update (from panel j-1) and its factorisation run on the diagonal stream as
    // soon as the tile (j, j-1) has arrived and the compute stream has applied panels < j-1 to it (ev_g2)
    auto diag_ahead = [&](int64_t j) -> int {
        if (j >= T) return B2GP_OK;
        const bool in_col = mycol == (int)(j % pc), owner = in_col && myrow == (int)(j % pr);
        if (!in_col) return B2GP_OK;
        if (owner) {
            CUDA_TRY(ctx, cudaEventRecord(ds->ev_g2, cs));
            CUDA_TRY(ctx, cudaStreamWaitEvent(dq, ds->ev_g2, 0));
            CUDA_TRY(ctx, cudaStreamWaitEvent(dq, ds->ev_early[(j - 1) & 1], 0));
        }
        return diag_factor(j, dq, true);
    };
    OzOperand opA, opB;
    OzMode upd_mode;
    auto update_slices = [&](int64_t k) -> int {   // digit planes of the panel of step k for this process's rows and columns
        const DistStep& s = ds->steps[(size_t)k];
        const int64_t rows = g.panel_rows(k, myrow), cols = (Lc - g.first_col_after(k, mycol)) * nb, slot = g.slot_rows(k);
        if (rows <= 0 || cols <= 0 || s.n1 + s.n2 == 0) return B2GP_OK;
        const double* PBk = (const double*)ds->PB[k & 1].p;
        if (sl.oz_planes == 6) {
            RET_IF(oz_slice_launch<6>(ctx, cs, PBk + (int64_t)myrow * slot * nb, nb, rows, nb, ds->updA, ds->updSA, false, nullptr, &opA));
            RET_IF(oz_slice_launch<6>(ctx, cs, PBk, nb, cols, nb, ds->updB, ds->updSB, false, (const int64_t*)s.bmap.p, &opB));
        } else {
            RET_IF(oz_slice_launch<7>(ctx, cs, PBk + (int64_t)myrow * slot * nb, nb, rows, nb, ds->updA, ds->updSA, false, nullptr, &opA));
            RET_IF(oz_slice_launch<7>(ctx, cs, PBk, nb, cols, nb, ds->updB, ds->updSB, false, (const int64_t*)s.bmap.p, &opB));
        }
        return B2GP_OK;
    };
    auto update_part = [&](int64_t k, int part) -> int {   // (g1) / (g2) of step k
        const DistStep& s = ds->steps[(size_t)k];
        const int64_t cnt = part == 1 ? s.n1 : s.n2;
        if (cnt == 0) return B2GP_OK;
        const int64_t li0 = g.first_row_after(k, myrow), lj0 = g.first_col_after(k, mycol);
        const int64_t rows = g.panel_rows(k, myrow), cols = (Lc - lj0) * nb;
        double* C = A + (li0 * nb) * ld + lj0 * nb;
        const int2* list = (const int2*)(part == 1 ? s.g1.p : s.g2.p);
        if (sl.oz_planes == 6) return oz_mma_launch<6>(ctx, cs, sl.oz, opA, opB, rows, cols, nb, -1.0, C, ld, false, upd_mode, list, cnt);
        return oz_mma_launch<7>(ctx, cs, sl.oz, opA, opB, rows, cols, nb, -1.0, C, ld, false, upd_mode, list, cnt);
    };

    // ---- the factorisation (with the right-hand-side rows riding below).  Compute stream, step k: wait for panel k;
    // slices; g1 (tile column k+1 without its diagonal tile, which the diagonal stream owns); panel solve / early tile /
    // exchange of step k+1; g2; then hand tile k+2 to the diagonal stream.
    // the persistent int8 kernels leave a few SMs to the NCCL kernels and the diagonal-tile kernels running beside them
    const int big_grid_saved = ctx->big_grid;
    if (ctx->big_grid == 0) ctx->big_grid = ctx->sm_count - 16;
    CUDA_TRY(ctx, cudaEventRecord(ds->ev_g2, cs));
    CUDA_TRY(ctx, cudaStreamWaitEvent(dq, ds->ev_g2, 0));          // the diagonal stream starts behind the Gram build
    RET_IF(diag_factor(0, cs, false));
    RET_IF(panel_front_b(0));
    RET_IF(diag_ahead(1));
    for (int64_t k = 0; k < T; ++k) {
        cudaEvent_t q0 = mark(cs);
        CUDA_TRY(ctx, cudaStreamWaitEvent(cs, ds->ev_comm[k & 1], 0));
        cudaEvent_t q1 = mark(cs);
        span(PH_COMMWAIT, q0, q1);
        RET_IF(update_slices(k));
        cudaEvent_t q2 = mark(cs);
        span(PH_SLICE, q1, q2);
        RET_IF(update_part(k, 1));
        span(PH_G1, q2, mark(cs));
        if (k + 1 < T) RET_IF(panel_front_b(k + 1));
        cudaEvent_t q3 = mark(cs);
        RET_IF(update_part(k, 2));
        span(PH_G2, q3, mark(cs));
        RET_IF(diag_ahead(k + 2));
    }
    CUDA_TRY(ctx, cudaEventRecord(ds->ev_u, dq));                   // the compute stream ends behind the diagonal stream
    CUDA_TRY(ctx, cudaStreamWaitEvent(cs, ds->ev_u, 0));
    ctx->big_grid = big_grid_saved;
    CUDA_TRY(ctx, cudaEventRecord(ev_f1, cs));

    // ---- epilogue: mean[p] = <V[p, :], w>, var[p] = k(x,x) + noise_p + jitter - |V[p, :]|^2, summed over the process grid
    double* red = (double*)ds->red.p;        // [0, P): dot, [P, 2P): |V|^2
    CUDA_TRY(ctx, cudaMemsetAsync(red, 0, (size_t)(2 * P) * 8, cs));
    {
        const int64_t gy = T + P / nb;
        double* wseg = (double*)ds->wseg.p;
        if (gy % pr == myrow && Lc > 0)
            CUDA_TRY(ctx, cudaMemcpyAsync(wseg, A + ((gy / pr) * nb + P % nb) * ld, (size_t)ld * 8, cudaMemcpyDeviceToDevice, cs));
        if (pr > 1 && Lc > 0) {
            CUDA_TRY(ctx, cudaEventRecord(ds->ev_u, cs));
            CUDA_TRY(ctx, cudaStreamWaitEvent(ms, ds->ev_u, 0));
            NCCL_TRY(ctx, nc->Broadcast(wseg, wseg, (size_t)ld, ncclDouble, (int)(gy % pr), ds->colc, ms));
            CUDA_TRY(ctx, cudaEventRecord(ds->ev_ubc[0], ms));
            CUDA_TRY(ctx, cudaStreamWaitEvent(cs, ds->ev_ubc[0], 0));
        }
        for (int64_t li = 0; li < Lr && Lc > 0; ++li) {
            const int64_t gi = li * pr + myrow;
            if (gi < T) continue;
            const int64_t p0 = (gi - T) * nb, np = std::min<int64_t>(nb, P - p0);
            if (np <= 0) continue;
            RET_IF(launch(ctx, cs, (unsigned)np, RD_THREADS, 0, rowdot2_kernel, A + (li * nb) * ld, ld, ld, wseg, 1.0, red + p0, red + P + p0, (int64_t)0));
        }
        CUDA_TRY(ctx, cudaEventRecord(ds->ev_chunk, cs));
        CUDA_TRY(ctx, cudaStreamWaitEvent(ms, ds->ev_chunk, 0));
        NCCL_TRY(ctx, nc->AllReduce(red, red, (size_t)(2 * P), ncclDouble, ncclSum, ds->world, ms));
        NCCL_TRY(ctx, nc->AllReduce(dinfo, dinfo, 1, ncclInt, ncclMax, ds->world, ms));
        CUDA_TRY(ctx, cudaEventRecord(ds->ev_done, ms));
        CUDA_TRY(ctx, cudaStreamWaitEvent(cs, ds->ev_done, 0));
        RET_IF(launch(ctx, cs, grid_for(P), 256, 0, dist_finish_kernel, red, want_var ? red + 2 * P : nullptr, red + P, P, kind, d, dth,
                      noiseless ? 0.0 : 1.0, jitter, dinfo));
    }
    CUDA_TRY(ctx, cudaMemcpyAsync(mean, red, (size_t)P * 8, cudaMemcpyDeviceToHost, cs));
    if (want_var) CUDA_TRY(ctx, cudaMemcpyAsync(var, red + 2 * P, (size_t)P * 8, cudaMemcpyDeviceToHost, cs));
    CUDA_TRY(ctx, cudaMemcpyAsync(info, dinfo, sizeof(int), cudaMemcpyDeviceToHost, cs));
    RET_IF(tm.end(cs, nullptr));
    sl.oz_planes = 7;
    float ms_f = 0.f;
    CUDA_TRY(ctx, cudaEventElapsedTime(&ms_f, ev_f0, ev_f1));
    ctx->last.potrf_ms = ms_f;
    if (prof) {
        static const char* names[PH_N] = {"update slices", "g1 (next tile column)", "[diag stream] early update + potrf + U", "wait for U", "panel solve + pack",
                                          "g2 (rest of the update)", "wait for the panel exchange", "[comm stream] U broadcast",
                                          "[comm stream] panel row broadcast", "[comm stream] panel column all-gather",
                                          "[comm stream] early tile broadcast"};
        char line[2048];
        int off = snprintf(line, sizeof line, "[dist prof] rank %d (%d,%d) N=%lld nb=%lld factorisation %.2f ms:", ds->rank, myrow, mycol,
                           (long long)N, (long long)nb, ms_f);
        for (int ph = 0; ph < PH_N; ++ph) {
            double tot = 0.0;
            for (auto& pe : pev[ph]) {
                float f = 0.f;
                cudaEventElapsedTime(&f, pe.first, pe.second);
                tot += f;
            }
            if (off < (int)sizeof line) off += snprintf(line + off, sizeof line - off, " %s %.2f;", names[ph], tot);
        }
        fprintf(stderr, "%s\n", line);     // one write per rank: the ranks share a terminal
    }
    const double n = (double)N, p = (double)P;
    ctx->last.flops = n * n * n / 3.0 + n * n * (p + 1.0) + 4.0 * n * p;
    if (timing) *timing = ctx->last;
    return B2GP_OK;
}

// N-sharded sparse (Nystrom / VFE) posterior -- gpax/models/sparse_gp.py:173-223 with the training set split over the
// ranks (config 5).  COLLECTIVE, HOST pointers: every rank passes ITS shard (Xtr_shard[N_shard, d], y_shard) and the same
// Xu, X_new, theta.  Per rank: Luu, W = Luu^{-1} K(Xu, shard) and the statistics W W^T / noise, W y / noise
// (sparse_gp.py:193-199, 203-204 restricted to the shard); ONE in-library NCCL all-reduce of the M x M matrix and the
// M-vector; then the M x M Cholesky and the P-side solves replicated on every rank (sparse_gp.py:200-217).
extern "C" int b2gp_dist_sparse_posterior(b2gp_ctx* ctx, int kind, const double* Xu, int64_t M, const double* Xtr_shard,
                                          int64_t N_shard, const double* y_shard, const double* Xnew, int64_t P, int d,
                                          const double* theta, int noiseless, double jitter, unsigned flags, double* mean,
                                          double* var, int* info, b2gp_timing* timing) {
    if (!ctx) return B2GP_ERR_ARG;
    DistState* ds = ctx->dist.get();
    if (!ds || !ds->ready) return set_err(ctx, B2GP_ERR_ARG, "b2gp_dist_sparse_posterior", "call b2gp_dist_init first", __FILE__, __LINE__);
    ARG_CHECK(ctx, kind >= 0 && kind <= 2);
    ARG_CHECK(ctx, Xu && Xtr_shard && y_shard && Xnew && theta && mean && info);
    ARG_CHECK(ctx, M >= 1 && N_shard >= 1 && P >= 1 && d >= 1 && d <= GRAM_MAX_D);
    ARG_CHECK(ctx, !(flags & B2GP_FLAG_DEVICE_PTRS) && !(flags & (B2GP_OUT_COV | B2GP_OUT_SAMPLE)));
    const bool want_var = flags & B2GP_OUT_VAR;
    ARG_CHECK(ctx, !want_var || var);
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    NcclApi* nc = nccl_api();
    ctx->fcache.valid = false;
    Slot& sl = ctx->slots[0];
    cudaStream_t st = sl.stream, ms = ds->ms;
    CallTimer tm(ctx);
    RET_IF(tm.begin(st));
    const int nth = d + 3;
    const double *dXu, *dXtr, *dy, *dXnew, *dth;
    RET_IF(stage_in(ctx, st, ctx->d_in[0], Xtr_shard, (size_t)N_shard * d * 8, false, &dXtr));
    RET_IF(stage_in(ctx, st, ctx->d_in[1], y_shard, (size_t)N_shard * 8, false, &dy));
    RET_IF(stage_in(ctx, st, ctx->d_in[2], Xnew, (size_t)P * d * 8, false, &dXnew));
    RET_IF(stage_in(ctx, st, ctx->d_in[3], theta, (size_t)nth * 8, false, &dth));
    RET_IF(stage_in(ctx, st, ctx->d_in[5], Xu, (size_t)M * d * 8, false, &dXu));
    const int64_t ldM = round_up(M, 8);
    double *slA = nullptr, *slLinv = nullptr;   // slot 0's matrix and inverted diagonal blocks
    RET_IF(slot0_buffers(ctx, (size_t)(2 * M * ldM + ldM) * 8, (size_t)2 * linv_bytes(M), &slA, &slLinv));   // Luu | K (+ the M-vector right behind it: one all-reduce)
    RET_IF(ensure(ctx, ctx->d_out[0], (size_t)(2 * P + 16) * 8));
    RET_IF(ensure(ctx, ctx->d_info, 64));
    int* dinfo = (int*)ctx->d_info.p;
    CUDA_TRY(ctx, cudaMemsetAsync(dinfo, 0, 16, st));
    double* Luu = slA;
    double* Kmat = Luu + M * ldM;
    double* cvec = Kmat + M * ldM;
    double* LinvU = slLinv;
    double* LinvK = LinvU + linv_bytes(M) / 8;
    double* mv = (double*)ctx->d_out[0].p;
    double* vv = mv + P;
    cudaEvent_t e0 = sl.ev[2], e1 = sl.ev[3], e2 = sl.ev[4];
    CUDA_TRY(ctx, cudaEventRecord(e0, st));
    RET_IF(sparse_partial_dev(ctx, sl, kind, dXu, M, dXtr, N_shard, dy, d, dth, jitter, theta[d + 1], Luu, ldM, LinvU, Kmat, ldM, cvec, dinfo));
    CUDA_TRY(ctx, cudaEventRecord(e1, st));
    if (ds->nranks > 1) {
        CUDA_TRY(ctx, cudaEventRecord(ds->ev_chunk, st));
        CUDA_TRY(ctx, cudaStreamWaitEvent(ms, ds->ev_chunk, 0));
        NCCL_TRY(ctx, nc->AllReduce(Kmat, Kmat, (size_t)(M * ldM + M), ncclDouble, ncclSum, ds->world, ms));   // sparse_gp.py:199, 204 summed over shards
        NCCL_TRY(ctx, nc->AllReduce(dinfo, dinfo, 1, ncclInt, ncclMax, ds->world, ms));
        CUDA_TRY(ctx, cudaEventRecord(ds->ev_done, ms));
        CUDA_TRY(ctx, cudaStreamWaitEvent(st, ds->ev_done, 0));
    }
    CUDA_TRY(ctx, cudaEventRecord(e2, st));
    RET_IF(sparse_finish_dev(ctx, sl, kind, dXu, M, Luu, ldM, LinvU, Kmat, ldM, LinvK, cvec, dXnew, P, d, dth, noiseless, jitter, want_var,
                             false, mv, vv, nullptr, P, dinfo));
    int hinfo[2] = {0, 0};
    CUDA_TRY(ctx, cudaMemcpyAsync(hinfo, dinfo, 2 * sizeof(int), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(ctx, cudaMemcpyAsync(mean, mv, (size_t)P * 8, cudaMemcpyDeviceToHost, st));
    if (want_var) CUDA_TRY(ctx, cudaMemcpyAsync(var, vv, (size_t)P * 8, cudaMemcpyDeviceToHost, st));
    RET_IF(tm.end(st, nullptr));
    info[0] = hinfo[0] != 0 ? hinfo[0] : -hinfo[1];
    float f = 0.f;
    CUDA_TRY(ctx, cudaEventElapsedTime(&f, e0, e1));
    ctx->last.potrf_ms = f;          // per-rank statistics (Gram, Luu, W, W W^T)
    CUDA_TRY(ctx, cudaEventElapsedTime(&f, e1, e2));
    ctx->last.trsm_ms = f;           // the all-reduce
    const double m = (double)M, n = (double)N_shard * ds->nranks, p = (double)P;
    ctx->last.flops = 2.0 * m * m * m / 3.0 + 2.0 * m * m * n + 2.0 * m * m * (p + 1.0);
    if (timing) *timing = ctx->last;
    return B2GP_OK;
}
