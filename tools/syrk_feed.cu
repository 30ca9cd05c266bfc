// Operand-feed probe of the fp64 SYRK at the north-star shape: streams the operand panels of every lower tile of
// K = G' diag(w) G (G 16384 x 8192, K-major, the band order of gemm_dmma.cu's decode_tile) into shared memory
// with no DMMAs, so the time is what the L2 -> SM feed alone needs for one SYRK.
//
//   make tools/syrk_feed && tools/syrk_feed
//
//   (a) 128x64 tiles, 128 threads, two CTAs per SM, 3-stage cp.async ring, one __syncthreads per 16-wide k tile
//       (the feed of dmma_gemm_kernel<1,1,1>)
//   (b) 128x128 tiles, one CTA per SM, a producer warp issuing one 2D TMA box {16 k, 128 rows} per operand into a
//       6-stage mbarrier ring, 8 consumer warps releasing stages (the feed of syrk_tma_kernel)
//
// Each form reports GB/s moved from L2 into shared memory and the time of one SYRK's operand stream, beside the
// DMMA-bound time of the 1.1e12-flop SYRK at the measured clock (256 flop/clk/SM, tools/dmma_rate).  SM clock:
// clock64 over globaltimer deltas of every CTA.
#include <cuda_runtime.h>
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <algorithm>

#define CK(x)                                                                                     \
    do {                                                                                          \
        cudaError_t e_ = (x);                                                                     \
        if (e_ != cudaSuccess) {                                                                  \
            fprintf(stderr, "%s:%d: %s -> %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_)); \
            exit(1);                                                                              \
        }                                                                                         \
    } while (0)

constexpr int N = 8192, KD = 16384, BR = 128, BK = 16;

__device__ __forceinline__ uint32_t s32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void stamp(unsigned long long *t, int i, bool end) {
    unsigned long long g, c = clock64();
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g));
    t[4 * i + 2 * end] = g;
    t[4 * i + 2 * end + 1] = c;
}

// ---- (a) cp.async, 128x64 ----
constexpr int A_STAGES = 3, A_SK = BK + 4, A_ROWS = BR + 64;
__global__ void __launch_bounds__(128, 2) feed_cpasync(const double *X, const int2 *tiles, double *sink,
                                                        unsigned long long *t) {
    extern __shared__ __align__(16) double sa[];
    const int tid = threadIdx.x;
    if (tid == 0) stamp(t, blockIdx.x, false);
    const int2 tl = tiles[blockIdx.x];
    const int r0 = tl.x * BR, c0 = tl.y * 64;
    auto issue = [&](int kt) {
        double *st = sa + (kt % A_STAGES) * A_ROWS * A_SK;
#pragma unroll
        for (int j = 0; j < A_ROWS * BK / 2 / 128; ++j) {
            const int i = tid + j * 128, row = i >> 3, ch = i & 7;
            const double *src = X + (long long)(row < BR ? r0 + row : c0 + row - BR) * KD + kt * BK + ch * 2;
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s32(st + row * A_SK + ch * 2)), "l"(src));
        }
    };
    const int kts = KD / BK;
    double acc = 0.0;
    for (int s = 0; s < A_STAGES - 1; ++s) { issue(s); asm volatile("cp.async.commit_group;"); }
    for (int kt = 0; kt < kts; ++kt) {
        asm volatile("cp.async.wait_group %0;" ::"n"(A_STAGES - 2));
        __syncthreads();
        acc += sa[(kt % A_STAGES) * A_ROWS * A_SK + tid];
        if (kt + A_STAGES - 1 < kts) issue(kt + A_STAGES - 1);
        asm volatile("cp.async.commit_group;");
    }
    sink[blockIdx.x * 128 + tid] = acc;
    __syncthreads();
    if (tid == 0) stamp(t, blockIdx.x, true);
}

// ---- (b) TMA, 128x128 ----
constexpr int B_STAGES = 6, B_PANEL = BR * BK;
constexpr int B_SMEM = B_STAGES * 2 * B_PANEL * 8 + 2 * B_STAGES * 8 + 1024;
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t par) {
    asm volatile("{\n\t.reg .pred p;\n\tW_%=:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
                 "@!p bra W_%=;\n\t}" ::"r"(s32(bar)), "r"(par) : "memory");
}
__global__ void __launch_bounds__(288, 1) feed_tma(const __grid_constant__ CUtensorMap tm, const int2 *tiles,
                                                   double *sink, unsigned long long *t) {
    extern __shared__ unsigned char raw[];
    double *sm = reinterpret_cast<double *>(raw + ((1024u - (s32(raw) & 1023u)) & 1023u));
    uint64_t *full = reinterpret_cast<uint64_t *>(sm + B_STAGES * 2 * B_PANEL), *empty = full + B_STAGES;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid == 0) {
        stamp(t, blockIdx.x, false);
        for (int s = 0; s < B_STAGES; ++s) {
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(s32(full + s)));
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 8;" ::"r"(s32(empty + s)));
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const int2 tl = tiles[blockIdx.x];
    const int kts = KD / BK;
    if (warp == 8) {
        if (lane == 0) {
            for (int kt = 0; kt < kts; ++kt) {
                const int s = kt % B_STAGES;
                if (kt >= B_STAGES) mbar_wait(empty + s, (kt / B_STAGES - 1) & 1);
                asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s32(full + s)),
                             "r"(2 * B_PANEL * 8) : "memory");
                double *d = sm + s * 2 * B_PANEL;
                asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
                             " [%0], [%1, {%2, %3}], [%4];" ::"r"(s32(d)), "l"(&tm), "r"(kt * BK), "r"(tl.x * BR),
                             "r"(s32(full + s)) : "memory");
                asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
                             " [%0], [%1, {%2, %3}], [%4];" ::"r"(s32(d + B_PANEL)), "l"(&tm), "r"(kt * BK),
                             "r"(tl.y * BR), "r"(s32(full + s)) : "memory");
            }
        }
        return;
    }
    double acc = 0.0;
    for (int kt = 0; kt < kts; ++kt) {
        const int s = kt % B_STAGES;
        mbar_wait(full + s, (kt / B_STAGES) & 1);
        acc += sm[s * 2 * B_PANEL + tid * 8];
        __syncwarp();
        if (lane == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(s32(empty + s)) : "memory");
    }
    sink[blockIdx.x * 256 + tid] = acc;
    asm volatile("bar.sync 1, 256;");
    if (tid == 0) stamp(t, blockIdx.x, true);
}

// lower tiles (tr, tc) of c-tile width tcols in the band order of decode_tile (bands of `band` c tiles)
static std::vector<int2> band_order(int tcols, int band) {
    const int nTr = N / BR, nTc = N / tcols;
    auto first_tr = [&](int c) { return c * tcols / BR; };
    std::vector<int2> v;
    for (int c = 0; c < nTc; c += band) {
        const int cb_end = std::min(c + band, nTc);
        for (int r = first_tr(c); r < nTr; ++r) {
            const int cmax = std::min(cb_end - 1, (r * BR + BR - 1) / tcols);
            for (int cc = c; cc <= cmax; ++cc) v.push_back(make_int2(r, cc));
        }
    }
    return v;
}

int main() {
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    printf("device: %s, sm_%d%d, %d SMs\n", prop.name, prop.major, prop.minor, prop.multiProcessorCount);
    fflush(stdout);
    if (system("nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv,noheader") != 0)
        printf("nvidia-smi query failed\n");
    fflush(stdout);
    const int sms = prop.multiProcessorCount;
    double *X, *sink;
    CK(cudaMalloc(&X, (size_t)N * KD * sizeof(double)));
    CK(cudaMemset(X, 0, (size_t)N * KD * sizeof(double)));
    CK(cudaMalloc(&sink, (size_t)8192 * 256 * sizeof(double)));
    const double syrk_flop = (double)N * N * KD;         // n^2 K, the bench's SYRK count

    PFN_cuTensorMapEncodeTiled_v12000 enc = nullptr;
    cudaDriverEntryPointQueryResult q;
    CK(cudaGetDriverEntryPointByVersion("cuTensorMapEncodeTiled", (void **)&enc, 12000, cudaEnableDefault, &q));
    if (q != cudaDriverEntryPointSuccess || !enc) { printf("cuTensorMapEncodeTiled unavailable\n"); return 1; }
    CUtensorMap tm;
    const cuuint64_t dims[2] = {KD, N}, strides[1] = {(cuuint64_t)KD * 8};
    const cuuint32_t box[2] = {BK, BR}, es[2] = {1, 1};
    if (enc(&tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 2, X, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) !=
        CUDA_SUCCESS) { printf("tensor map encode failed\n"); return 1; }
    CK(cudaFuncSetAttribute(feed_cpasync, cudaFuncAttributeMaxDynamicSharedMemorySize, A_STAGES * A_ROWS * A_SK * 8));
    CK(cudaFuncSetAttribute(feed_tma, cudaFuncAttributeMaxDynamicSharedMemorySize, B_SMEM));

    for (int form = 0; form < 2; ++form) {
        const int tcols = form == 0 ? 64 : 128;
        std::vector<int2> tiles = band_order(tcols, 1024 / tcols);
        const int T = (int)tiles.size();
        int2 *dt; unsigned long long *ts;
        CK(cudaMalloc(&dt, T * sizeof(int2)));
        CK(cudaMalloc(&ts, (size_t)T * 4 * sizeof(unsigned long long)));
        CK(cudaMemcpy(dt, tiles.data(), T * sizeof(int2), cudaMemcpyHostToDevice));
        cudaEvent_t e0, e1;
        CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
        float best = 1e30f;
        for (int rep = 0; rep < 4; ++rep) {                // rep 0 warms up
            CK(cudaEventRecord(e0));
            if (form == 0) feed_cpasync<<<T, 128, A_STAGES * A_ROWS * A_SK * 8>>>(X, dt, sink, ts);
            else feed_tma<<<T, 288, B_SMEM>>>(tm, dt, sink, ts);
            CK(cudaEventRecord(e1));
            CK(cudaEventSynchronize(e1));
            CK(cudaGetLastError());
            float ms;
            CK(cudaEventElapsedTime(&ms, e0, e1));
            if (rep > 0) best = std::min(best, ms);
        }
        std::vector<unsigned long long> h((size_t)T * 4);
        CK(cudaMemcpy(h.data(), ts, h.size() * 8, cudaMemcpyDeviceToHost));
        double ns = 0, cyc = 0;
        for (int i = 0; i < T; ++i) { ns += (double)(h[4 * i + 2] - h[4 * i]); cyc += (double)(h[4 * i + 3] - h[4 * i + 1]); }
        const double mhz = cyc / ns * 1e3;
        const double bytes = (double)T * (BR + tcols) * KD * 8.0;
        const double dmma_ms = syrk_flop / (256.0 * sms * mhz * 1e6) * 1e3;
        printf("(%c) %s: %d tiles, %.1f GB from L2, %.2f ms = %.0f GB/s; SM clock %.0f MHz; "
               "DMMA-bound SYRK at that clock %.2f ms\n",
               'a' + form, form == 0 ? "128x64 cp.async, 2 CTAs/SM" : "128x128 TMA ring, 1 CTA/SM", T, bytes * 1e-9,
               best, bytes / (best * 1e-3) * 1e-9, mhz, dmma_ms);
        CK(cudaFree(dt)); CK(cudaFree(ts));
        CK(cudaEventDestroy(e0)); CK(cudaEventDestroy(e1));
    }
    CK(cudaFree(X)); CK(cudaFree(sink));
    return 0;
}
