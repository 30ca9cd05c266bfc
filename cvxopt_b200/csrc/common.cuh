// Shared device/host helpers for the cvxopt_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>
#include <atomic>
#include <mutex>
#include "../../include/cvxopt_b200.h"

namespace cvxb {

// ---- error plumbing ---------------------------------------------------------
void set_error(const char *fmt, ...);
extern std::atomic<unsigned long long> g_launches;   // kernels launched by this library
inline void count_launch(int n = 1) { g_launches.fetch_add((unsigned long long)n, std::memory_order_relaxed); }

// Function attributes (dynamic shared-memory opt-in ...) are PER DEVICE: a call site keeps one of
// these and sets its attributes the first time it runs on each device of the process.
struct DeviceOnce {
    std::atomic<unsigned long long> done{0};
    // returns the bit of the current device if its attributes are still to be set, else 0
    unsigned long long pending() {
        int d = 0;
        cudaGetDevice(&d);
        const unsigned long long bit = 1ull << (d & 63);
        return (done.load(std::memory_order_acquire) & bit) ? 0ull : bit;
    }
    void mark(unsigned long long bit) { done.fetch_or(bit, std::memory_order_release); }
};

#define CVXB_CUDA(expr)                                                            \
    do {                                                                           \
        cudaError_t _e = (expr);                                                   \
        if (_e != cudaSuccess) {                                                   \
            cvxb::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr,          \
                            cudaGetErrorString(_e));                               \
            return CVXB_E_CUDA;                                                    \
        }                                                                          \
    } while (0)

#define CVXB_TRY(expr)                                                             \
    do {                                                                           \
        int _r = (expr);                                                           \
        if (_r != 0) return _r;                                                    \
    } while (0)

#define CVXB_LAUNCH_CHECK()                                                        \
    do {                                                                           \
        cudaError_t _e = cudaGetLastError();                                       \
        if (_e != cudaSuccess) {                                                   \
            cvxb::set_error("%s:%d: kernel launch -> %s", __FILE__, __LINE__,      \
                            cudaGetErrorString(_e));                               \
            return CVXB_E_CUDA;                                                    \
        }                                                                          \
    } while (0)

// ---- scratch-buffer cache ----------------------------------------------------
// The cone / scaling entry points (cvxb_scale, cvxb_max_step, cvxb_update_scaling ...) need device temporaries per call;
// cudaMalloc + cudaFree cost far more than the kernels of a small call (cudaFree also synchronises the device).
// tmp_malloc / tmp_free keep
// freed blocks per device and hand them out again (best fit within +25 %); callers synchronise their stream before
// freeing, as they did for cudaFree.  The cache is bounded (CVXB_TMP_CACHE_MB, default 4096) and is dropped when a
// real allocation fails.
cudaError_t tmp_malloc_bytes(void **p, size_t bytes);
void tmp_free(void *p);
void tmp_cache_release();          // free every cached block of every device
template <class T> inline cudaError_t tmp_malloc(T **p, size_t bytes) { return tmp_malloc_bytes(reinterpret_cast<void **>(p), bytes); }

// n elements of device scratch from the cache, returned to it when the Scratch goes out of scope
template <class T> struct Scratch {
    T *p = nullptr;
    Scratch() = default;
    Scratch(const Scratch &) = delete;
    Scratch &operator=(const Scratch &) = delete;
    ~Scratch() { tmp_free(p); }
    int alloc(size_t n) {
        CVXB_CUDA(tmp_malloc(&p, (n ? n : 1) * sizeof(T)));
        return 0;
    }
};

// n doubles of a caller's buffer on the device: a host buffer (space == CVXB_HOST) is staged in scratch, a device
// pointer (CVXB_DEVICE) is used in place.  upload == false skips the host-to-device copy of output-only buffers.
struct Staged {
    double *dev = nullptr, *host = nullptr; size_t n = 0; bool owned = false;
    Staged() = default;
    Staged(const Staged &) = delete;
    Staged &operator=(const Staged &) = delete;
    ~Staged() { if (owned) tmp_free(dev); }
    int in(const double *src, size_t count, int space, cudaStream_t st, bool upload = true) {
        n = count; host = const_cast<double *>(src);
        if (space == CVXB_DEVICE) { dev = host; return 0; }
        CVXB_CUDA(tmp_malloc(&dev, (n ? n : 1) * sizeof(double)));
        owned = true;
        if (n && upload) CVXB_CUDA(cudaMemcpyAsync(dev, src, n * sizeof(double), cudaMemcpyHostToDevice, st));
        return 0;
    }
    int out(cudaStream_t st) {
        if (owned && n) CVXB_CUDA(cudaMemcpyAsync(host, dev, n * sizeof(double), cudaMemcpyDeviceToHost, st));
        return 0;
    }
};

// ---- long-lived device memory ---------------------------------------------------
// Bytes currently held by DevBufs, all devices together (cvxb_device_bytes).
extern std::atomic<unsigned long long> g_device_bytes;

// n elements of cudaMalloc memory owned by the handle (or workspace) it is a member of, freed with it.
template <class T> struct DevBuf {
    T *p = nullptr;
    size_t n = 0;
    DevBuf() = default;
    DevBuf(const DevBuf &) = delete;
    DevBuf &operator=(const DevBuf &) = delete;
    DevBuf(DevBuf &&o) noexcept : p(o.p), n(o.n) { o.p = nullptr; o.n = 0; }
    DevBuf &operator=(DevBuf &&o) noexcept {
        if (this != &o) { reset(); p = o.p; n = o.n; o.p = nullptr; o.n = 0; }
        return *this;
    }
    ~DevBuf() { reset(); }
    // Frees what it held, then allocates count elements.  An allocation that fails for lack of memory is tried
    // once more after the scratch-buffer cache is given back to the driver.  Leaves no CUDA error pending and no
    // error text: for callers that have a fallback.
    cudaError_t try_alloc(size_t count) {
        reset();
        const size_t bytes = count * sizeof(T);
        cudaError_t e = cudaMalloc(&p, bytes);
        if (e == cudaErrorMemoryAllocation) { cudaGetLastError(); tmp_cache_release(); e = cudaMalloc(&p, bytes); }
        if (e != cudaSuccess) { cudaGetLastError(); p = nullptr; return e; }
        n = count;
        g_device_bytes.fetch_add(bytes, std::memory_order_relaxed);
        return cudaSuccess;
    }
    // try_alloc; a failure returns CVXB_E_NOMEM (out of memory) or CVXB_E_CUDA with the error text set
    int alloc(size_t count) {
        const cudaError_t e = try_alloc(count);
        if (e == cudaSuccess) return 0;
        set_error("cudaMalloc(%zu bytes) -> %s", count * sizeof(T), cudaGetErrorString(e));
        return e == cudaErrorMemoryAllocation ? CVXB_E_NOMEM : CVXB_E_CUDA;
    }
    void reset() {
        if (!p) return;
        cudaFree(p);
        g_device_bytes.fetch_sub(n * sizeof(T), std::memory_order_relaxed);
        p = nullptr;
        n = 0;
    }
};

// CVXB_JACOBI_COOP (default on, =0 for one launch per round) allows a cooperative launch, and `ctas` CTAs of
// `threads` threads of `kernel` can be resident on the current device at once
bool coop_launch_fits(const void *kernel, int threads, long long ctas);

constexpr int kNumSMs = 132;       // H100 SXM
constexpr int NB = 128;            // Cholesky block size == GEMM tile edge

// ---- device helpers ---------------------------------------------------------
#ifdef __CUDACC__
// fp64 tensor-core MMA, Ampere shape: D(8x8) += A(8x4,row) * B(4x8,col).  SASS: DMMA.8x8x4.
// lane -> A[lane>>2][lane&3], B[k=lane&3][n=lane>>2], D[lane>>2][2*(lane&3)+{0,1}]
// Only for 8-wide tiles: on sm_90 it runs at half the fp64 tensor rate of dmma16x8x4 (128 against 256 flop per
// clock and SM, tools/dmma_rate).
__device__ __forceinline__ void dmma(double &d0, double &d1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                 : "+d"(d0), "+d"(d1)
                 : "d"(a), "d"(b));
}
// fp64 tensor-core MMA, sm_90 shape: D(16x8) += A(16x4,row) * B(4x8,col).  SASS: DMMA.16x8x4.
// lane -> A[lane>>2][lane&3] (a0), A[8+(lane>>2)][lane&3] (a1), B[k=lane&3][n=lane>>2],
//         D[lane>>2][2*(lane&3)+{0,1}] (d0,d1), D[8+(lane>>2)][2*(lane&3)+{0,1}] (d2,d3)
// so it is the two products dmma(d0,d1,a0,b) and dmma(d2,d3,a1,b) of 8-row blocks that share b, in one instruction
// (fragment map checked on the device by tools/dmma_rate).
__device__ __forceinline__ void dmma16x8x4(double &d0, double &d1, double &d2, double &d3, double a0, double a1,
                                           double b) {
    asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
                 : "+d"(d0), "+d"(d1), "+d"(d2), "+d"(d3)
                 : "d"(a0), "d"(a1), "d"(b));
}

__device__ __forceinline__ uint32_t smem_u32(const void *p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}
// 16-byte async copy global->shared, zero-filling (16 - src_bytes) trailing bytes.
__device__ __forceinline__ void cp_async16(void *smem, const void *gmem, int src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(smem)), "l"(gmem),
                 "r"(src_bytes));
}
__device__ __forceinline__ void cp_async8(void *smem, const void *gmem, int src_bytes) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(smem_u32(smem)), "l"(gmem),
                 "r"(src_bytes));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;" ::"n"(N));
}

// mbarrier ring of a producer / consumer pipeline: `full` barriers complete when their bulk / TMA copies have
// landed (expect_tx), `empty` ones when every consumer has arrived; waiters pass the parity of the phase they wait for
__device__ __forceinline__ void mbar_init(uint64_t *bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(smem_u32(bar)), "r"(parity)
        : "memory");
}
// contiguous global -> shared copy (16-byte aligned, multiple of 16 bytes) that completes `bytes` on bar
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
        ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}
// TMA box loads through a CUtensorMap kernel parameter (`map` is its generic address); the box lands in shared
// memory as the map's swizzle lays it out, elements outside the tensor are zero, and the whole box's bytes
// complete on bar
__device__ __forceinline__ void tma_load_1d(void *dst, const void *map, int c0, uint64_t *bar) {
    asm volatile(
        "cp.async.bulk.tensor.1d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2}], [%3];"
        ::"r"(smem_u32(dst)), "l"(map), "r"(c0), "r"(smem_u32(bar))
        : "memory");
}
__device__ __forceinline__ void tma_load_2d(void *dst, const void *map, int c0, int c1, uint64_t *bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
        ::"r"(smem_u32(dst)), "l"(map), "r"(c0), "r"(c1), "r"(smem_u32(bar))
        : "memory");
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_min(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
// Sum / min over the CTA (blockDim.x a multiple of 32), returned to every thread: warp reductions, then warp 0
// reduces the per-warp values.  sh holds 32 doubles of shared memory and is free again when the call returns.
__device__ __forceinline__ double block_sum(double v, double *sh) {
    v = warp_sum(v);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    __syncthreads();
    if (lane == 0) sh[warp] = v;
    __syncthreads();
    double t = (threadIdx.x < (blockDim.x >> 5)) ? sh[threadIdx.x] : 0.0;
    if (warp == 0) t = warp_sum(t);
    if (threadIdx.x == 0) sh[0] = t;
    __syncthreads();
    const double r = sh[0];
    __syncthreads();
    return r;
}
__device__ __forceinline__ double block_min(double v, double *sh) {
    v = warp_min(v);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    __syncthreads();
    if (lane == 0) sh[warp] = v;
    __syncthreads();
    double t = (threadIdx.x < (blockDim.x >> 5)) ? sh[threadIdx.x] : INFINITY;
    if (warp == 0) t = warp_min(t);
    if (threadIdx.x == 0) sh[0] = t;
    __syncthreads();
    const double r = sh[0];
    __syncthreads();
    return r;
}
__device__ __forceinline__ int ld_acquire(const int *p) {
    int v;
    asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release(int *p, int v) {
    asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
#endif

// ---- host-side kernels' launch API (device pointers, explicit stream) --------
struct GemmDesc {
    // C[r,c] = alpha * sum_k X[r,k] * w[k] * Y[c,k] + beta * D[r,c]      (col-major C/D)
    // X[r,k] = x_kmajor ? X[k + r*ldx] : X[r + k*ldx]; same for Y.
    int M = 0, N = 0, K = 0;
    const double *X = nullptr; int ldx = 0; bool x_kmajor = false;
    const double *Y = nullptr; int ldy = 0; bool y_kmajor = false;
    const double *w = nullptr;          // optional K-vector applied inside the contraction
    const double *D = nullptr; int ldd = 0;
    double *C = nullptr; int ldc = 0;
    double alpha = 1.0, beta = 0.0;
    bool lower_only = false;            // only tiles with r-tile >= c-tile (M == N)
    // tile-column window (look-ahead in the Cholesky): only c-tiles in [ct_begin, ct_end)
    int ct_begin = 0, ct_end = 1 << 30;
    // batching (blockIdx.z): element strides between consecutive problems
    int batch = 1;
    long long sX = 0, sY = 0, sW = 0, sD = 0, sC = 0;
    // split-K remainder workspace (>= kNumSMs * 128*128 doubles) or nullptr to disable
    double *splitk_ws = nullptr;
    // debug timeline (CVXB_TRACE): [0] = min CTA start, [1] = max CTA end (globaltimer ns)
    unsigned long long *trace = nullptr;
};
int dmma_gemm(const GemmDesc &g, cudaStream_t st);
size_t dmma_gemm_splitk_ws_doubles();   // workspace size for GemmDesc::splitk_ws
int dmma_gemm_tile_cols();              // width of a c tile (units of ct_begin / ct_end)

// ozaki_syrk.cu (opt-in): C(lower) = A' diag(d)^2 A + beta*D through int8 slices on wgmma
size_t ozaki_workspace_bytes(int n, int m, int S);
// CVXB_OZAKI (read when a handle is created): 0 or unset never, 1 for large problems, 2 always
int ozaki_mode();
// whether the SYRK of an m x n operand runs on the int8 slices (nine of them) under `mode`: 2 always, 1 when
// n >= 4096 and m >= 8192.  Keeps the slice workspace in `work`; when it does not fit, the answer is no (the
// DMMA kernel, which needs none, computes the same result), with no CUDA error pending and no error text.
bool ozaki_use(int mode, int n, int m, DevBuf<char> &work);
void ozaki_time_mma(cudaEvent_t a, cudaEvent_t b);   // events recorded around the MMA launches of this thread's next call
int ozaki_syrk(int n, int m, const double *A, long long lda, const double *d, const double *D,
               long long ldd, double beta, double *C, long long ldc, int S, int layout, void *work,
               cudaStream_t st);

// Cholesky (lower) of the n x n matrix A in place; inv receives the inverses of the
// NB x NB diagonal blocks of L (block j at inv + j*NB*NB, leading dimension NB).
// info (device int) = first non-positive pivot (1-based) or 0.
struct CholWork {
    cudaStream_t panel_stream = nullptr;   // high-priority: diagonal block, panel, next-panel update
    cudaStream_t trsm_stream = nullptr;    // high-priority: panel TRSM + next block column update
    cudaStream_t update_stream = nullptr;  // low-priority: near updates of the next group, grouped far updates
    cudaStream_t near_stream = nullptr;    // high-priority: near updates inside the group, panel transposes
    cudaEvent_t ev_end_t = nullptr, ev_end_n = nullptr;
    std::vector<cudaEvent_t> ev_dg, ev_tr, ev_c0, ev_na, ev_nb, ev_n;   // one per block step
    // CVXB_TRACE=1: per step {Dg, Tr, C0, near} x {start, end}; far update of the group ending at step j at
    // [8 * 2048 + 8 * j + 5], [.. + 6]
    DevBuf<unsigned long long> trace;
    struct GraphEntry {                    // captured factorisation, keyed by its arguments
        int n = 0, lda = 0, launches = 0;
        const void *A = nullptr, *inv = nullptr;
        cudaGraphExec_t exec = nullptr;
    };
    std::vector<GraphEntry> graphs;
    bool graph_failed = false;
    cudaEvent_t ev_start = nullptr, ev_end_p = nullptr, ev_end_u = nullptr;
    DevBuf<int> d_info;                    // device flag
    DevBuf<int> d_flags;                   // trsv progress flags (batch * ceil(n/NB) ints)
    DevBuf<double> splitk_ws;
    DevBuf<double> panel[2];               // out-of-place TRSM results (double-buffered)
    DevBuf<double> group[2];               // K-major copies of a group's panels (double-buffered by group)
    int panel_rows = 0;
    ~CholWork();                           // also right after a chol_work_create that failed part-way
};
int chol_work_create(CholWork &w);
int potrf_lower(int n, double *A, int lda, double *inv, CholWork &w, cudaStream_t st);
// b := L^{-T} L^{-1} b  (potrs with one right-hand side)
// batched variants: problem p uses L + p*sL, inv + p*sInv, b + p*sb
int potrs_lower(int n, const double *L, int ldl, const double *inv, double *b, CholWork &w,
                cudaStream_t st, int batch = 1, long long sL = 0, long long sInv = 0,
                long long sb = 0);
int trsv_lower(int n, const double *L, int ldl, const double *inv, double *b, bool trans,
               CholWork &w, cudaStream_t st, int batch = 1, long long sL = 0, long long sInv = 0,
               long long sb = 0);
int potrf_lower_batched(int n, double *A, int lda, long long sA, double *inv, long long sInv,
                        int batch, int *d_info, double *panel, int ldw, cudaStream_t st);
// B := L^{-1} B for the n x n Cholesky factor L (lower, ld ldl) with its diagonal-block inverses `inv`
// (potrf_lower's output); B is n x ncols (ld ldb), updated in place by blocked forward substitution (DMMA GEMMs).
// Batched: problem p uses L + p*sL, inv + p*sInv, B + p*sB.  Defined in kkt_api.cu.
int trsm_lower_left(int n, const double *L, long long ldl, const double *inv, double *B, long long ldb, int ncols,
                    cudaStream_t st, int batch = 1, long long sL = 0, long long sInv = 0, long long sB = 0);

// ---- device selection ----------------------------------------------------------
// CVXB_E_NOGPU unless `device` exists and is sm_90; selects it.
int check_device(int device);

// The entry points that take no cvxb_kkt / cvxb_batch handle (misc_solvers mirror, NT scaling, dense blocks)
// share one stream and one CholWork per device.  acquire() selects the device and holds its lock until the
// CallCtx goes out of scope, so calls on one device are serialised.  The lock is not recursive: such an entry
// point must not call another one.  Declare the CallCtx before the buffers it frees.
struct CallCtx {
    cudaStream_t st = nullptr;
    CholWork *cw = nullptr;
    std::unique_lock<std::mutex> lock;
    int acquire(int device);
};

}  // namespace cvxb
