// fp64 tensor-core shape probe for sm_90a: fragment layouts and issue rate of every mma.sync .f64 shape.
//
//   make tools/dmma_rate && tools/dmma_rate
//
// 1. Layout check: one warp multiplies small integer matrices (exact in fp64) with each of m8n8k4, m16n8k4,
//    m16n8k8 and m16n8k16, loading and storing the fragments by the maps written below; the host compares every
//    element of D = A B + C with a CPU product.  A pass pins the fragment maps the library's kernels rely on.
// 2. Rate: two 128-thread CTAs per SM (the occupancy of dmma_gemm_kernel), CH independent accumulator chains per
//    warp, timed with CUDA events over >= 200 ms; SM clocks from clock64() deltas inside the kernel.
//
// Fragment maps (g = lane / 4, t = lane % 4), with A M x K row-major, B K x 8 column-major, C/D M x 8:
//   A register i : A[g + 8 * (i % (M / 8))][t + 4 * (i / (M / 8))]
//   B register i : B[t + 4 * i][g]
//   D register i : D[g + 8 * (i / 2)][2 * t + i % 2]
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <vector>

#define CK(x)                                                                                     \
    do {                                                                                          \
        cudaError_t e_ = (x);                                                                     \
        if (e_ != cudaSuccess) {                                                                  \
            fprintf(stderr, "%s:%d: %s -> %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_)); \
            exit(1);                                                                              \
        }                                                                                         \
    } while (0)

template <int M, int K>
struct Shape {
    static constexpr int NA = M * K / 32, NB = K * 8 / 32, NC = M * 8 / 32;
    static constexpr double flop = 2.0 * M * 8 * K;
};

template <int M, int K>
__device__ __forceinline__ void mma(double (&d)[Shape<M, K>::NC], const double (&a)[Shape<M, K>::NA],
                                    const double (&b)[Shape<M, K>::NB]) {
    if constexpr (M == 8 && K == 4) {
        asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                     : "+d"(d[0]), "+d"(d[1])
                     : "d"(a[0]), "d"(b[0]));
    } else if constexpr (M == 16 && K == 4) {
        asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
                     : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
                     : "d"(a[0]), "d"(a[1]), "d"(b[0]));
    } else if constexpr (M == 16 && K == 8) {
        asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                     "{%0,%1,%2,%3};"
                     : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
                     : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
    } else {
        static_assert(M == 16 && K == 16, "unsupported shape");
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, "
                     "{%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, {%0,%1,%2,%3};"
                     : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
                     : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]),
                       "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
    }
}

// the fragment maps of the header
__host__ __device__ inline void a_pos(int M, int lane, int i, int &r, int &c) {
    r = lane / 4 + 8 * (i % (M / 8));
    c = lane % 4 + 4 * (i / (M / 8));
}
__host__ __device__ inline void b_pos(int lane, int i, int &k, int &n) { k = lane % 4 + 4 * i; n = lane / 4; }
__host__ __device__ inline void d_pos(int lane, int i, int &r, int &c) { r = lane / 4 + 8 * (i / 2); c = 2 * (lane % 4) + i % 2; }

// one warp: D = A B + C, fragments gathered from / scattered to row-major A (M x K), B (K x 8), C and D (M x 8)
template <int M, int K>
__global__ void layout_kernel(const double *A, const double *B, const double *C, double *D) {
    using S = Shape<M, K>;
    const int lane = threadIdx.x;
    double a[S::NA], b[S::NB], d[S::NC];
    for (int i = 0; i < S::NA; ++i) { int r, c; a_pos(M, lane, i, r, c); a[i] = A[r * K + c]; }
    for (int i = 0; i < S::NB; ++i) { int k, n; b_pos(lane, i, k, n); b[i] = B[k * 8 + n]; }
    for (int i = 0; i < S::NC; ++i) { int r, c; d_pos(lane, i, r, c); d[i] = C[r * 8 + c]; }
    mma<M, K>(d, a, b);
    for (int i = 0; i < S::NC; ++i) { int r, c; d_pos(lane, i, r, c); D[r * 8 + c] = d[i]; }
}

template <int M, int K, int CH>
__global__ void __launch_bounds__(128, 2) rate_kernel(double *out, long long *cycles, int iters, double seed) {
    using S = Shape<M, K>;
    double a[S::NA], b[S::NB], d[CH][S::NC];
    for (int i = 0; i < S::NA; ++i) a[i] = seed * (threadIdx.x + i);
    for (int i = 0; i < S::NB; ++i) b[i] = seed * (threadIdx.x - i);
    for (int c = 0; c < CH; ++c)
        for (int i = 0; i < S::NC; ++i) d[c][i] = 0.0;
    __syncthreads();
    const long long t0 = clock64();
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int c = 0; c < CH; ++c) mma<M, K>(d[c], a, b);
    }
    __syncthreads();
    const long long t1 = clock64();
    double s = 0.0;
    for (int c = 0; c < CH; ++c)
        for (int i = 0; i < S::NC; ++i) s += d[c][i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
    if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

template <int M, int K>
bool check_layout() {
    using S = Shape<M, K>;
    std::vector<double> A(M * K), B(K * 8), C(M * 8), D(M * 8), R(M * 8);
    unsigned s = 12345u + M * 100 + K;
    auto rnd = [&]() { s = s * 1664525u + 1013904223u; return (double)((int)((s >> 16) % 9) - 4); };
    for (auto &v : A) v = rnd();
    for (auto &v : B) v = rnd();
    for (auto &v : C) v = rnd();
    for (int r = 0; r < M; ++r)
        for (int c = 0; c < 8; ++c) {
            double v = C[r * 8 + c];
            for (int k = 0; k < K; ++k) v += A[r * K + k] * B[k * 8 + c];
            R[r * 8 + c] = v;
        }
    double *dA, *dB, *dC, *dD;
    CK(cudaMalloc(&dA, A.size() * 8)); CK(cudaMalloc(&dB, B.size() * 8));
    CK(cudaMalloc(&dC, C.size() * 8)); CK(cudaMalloc(&dD, D.size() * 8));
    CK(cudaMemcpy(dA, A.data(), A.size() * 8, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(dB, B.data(), B.size() * 8, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(dC, C.data(), C.size() * 8, cudaMemcpyHostToDevice));
    CK(cudaMemset(dD, 0xff, D.size() * 8));
    layout_kernel<M, K><<<1, 32>>>(dA, dB, dC, dD);
    CK(cudaGetLastError());
    CK(cudaMemcpy(D.data(), dD, D.size() * 8, cudaMemcpyDeviceToHost));
    int bad = 0;
    for (int i = 0; i < M * 8; ++i) bad += (D[i] != R[i]);
    printf("layout m%dn8k%d: %s (%d of %d elements differ)\n", M, K, bad ? "FAIL" : "pass", bad, M * 8);
    CK(cudaFree(dA)); CK(cudaFree(dB)); CK(cudaFree(dC)); CK(cudaFree(dD));
    return bad == 0;
}

template <int M, int K, int CH>
void rate(int sms) {
    using S = Shape<M, K>;
    const int ctas = 2 * sms;
    double *out; long long *cyc;
    CK(cudaMalloc(&out, ctas * 128 * sizeof(double)));
    CK(cudaMalloc(&cyc, ctas * sizeof(long long)));
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    auto run = [&](int iters) {
        CK(cudaEventRecord(e0));
        rate_kernel<M, K, CH><<<ctas, 128>>>(out, cyc, iters, 1e-3);
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
        CK(cudaGetLastError());
        float ms = 0.f;
        CK(cudaEventElapsedTime(&ms, e0, e1));
        return (double)ms;
    };
    run(1000);                                           // warm-up
    int iters = 20000;
    const double ms0 = run(iters);
    iters = (int)(iters * 200.0 / (ms0 > 1e-3 ? ms0 : 1e-3));   // ~200 ms of work
    if (iters < 1000) iters = 1000;
    const double ms = run(iters);
    std::vector<long long> c(ctas);
    CK(cudaMemcpy(c.data(), cyc, ctas * sizeof(long long), cudaMemcpyDeviceToHost));
    long long cmax = 0;
    for (long long v : c) cmax = v > cmax ? v : cmax;
    const double flop = S::flop * CH * iters * 4.0 * ctas;
    printf("rate m%2dn8k%-2d chains %2d: %7.2f TF/s  %6.1f flop/clk/SM  (%.1f ms, %.0f MHz from clock64)\n", M, K, CH,
           flop / (ms * 1e-3) * 1e-12, flop / ((double)cmax * sms), ms, (double)cmax / (ms * 1e3));
    CK(cudaFree(out)); CK(cudaFree(cyc));
    CK(cudaEventDestroy(e0)); CK(cudaEventDestroy(e1));
}

int main() {
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    printf("device: %s, sm_%d%d, %d SMs\n", prop.name, prop.major, prop.minor, prop.multiProcessorCount);
    fflush(stdout);
    if (system("nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv,noheader") != 0)
        printf("nvidia-smi query failed\n");
    fflush(stdout);
    bool ok = check_layout<8, 4>();
    ok &= check_layout<16, 4>();
    ok &= check_layout<16, 8>();
    ok &= check_layout<16, 16>();
    const int sms = prop.multiProcessorCount;
    rate<8, 4, 8>(sms);
    rate<8, 4, 16>(sms);
    rate<16, 4, 8>(sms);
    rate<16, 4, 16>(sms);
    rate<16, 8, 8>(sms);
    rate<16, 8, 16>(sms);
    rate<16, 16, 8>(sms);
    rate<16, 16, 16>(sms);
    return ok ? 0 : 1;
}
