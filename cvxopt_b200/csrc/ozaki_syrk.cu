// fp64 SYRK  C = A' diag(d)^2 A (+ H)  on the int8 tensor path (wgmma s8 x s8 -> s32, accumulators in
// registers) by error-free slicing (Ozaki scheme).  kkt_api.cu uses it for the 'l'-row SYRK when CVXB_OZAKI=2
// (the default fp64 DMMA kernel is faster on H100, see DESIGN.md).  Replaces the same reference call as the DMMA
// SYRK: blas.syrk(Gs, K, trans='T') in misc.kkt_chol.factor (misc.py:1275, blas.c:3039); the result is within
// 1e-15 * sum|terms| of an 80-bit evaluation (tests/test_i8_syrk_gpu.py).
//
// Arithmetic.  Column j of Gs = diag(d) A is written  Gs[k,j] = 2^e_j * sum_s q_s[k,j] 2^-(6+7s),
// q_s integers in [-64, 64] (round-to-nearest digits, radix 2^7, e_j from the column maximum), so
//   C[i,j] = 2^(e_i+e_j-12) * sum_d 2^(-7d) * ( sum_{s+t=d} q_s[:,i] . q_t[:,j] ),   d = 0 .. S-1.
// Every inner product is exact in int32 ((d+1) * 4096 * K < 2^31 for K <= 32768 rows per drain);
// levels d >= S are dropped (S = 9: 62 bits below the column maximum).  An output tile is 128 x 128 and
// its int32 accumulators live in the registers of two warpgroups (rows 0-63 / 64-127, 64 registers per
// level and thread), so a pass holds two levels and an output tile takes ceil(S/2) passes over K; inside a
// pass the two levels are combined exactly in fp64, scaled by powers of two and added to C.
//
// Data layout.  The slicing kernel writes the digits directly as the shared-memory image the MMA
// reads: a "unit" is the 128-column x 32-row (K) block of one slice, 4 KB, K-major with the 32-byte
// swizzle; units are ordered [column block][k step][slice] so that the first nS slices of one
// (block, k step) are one contiguous bulk copy, and two consecutive slices form the 256-row B operand of
// one m64n256k32 wgmma.  One CTA per 128x128 lower tile: warps 0-7 (two warpgroups) issue the wgmmas and
// run the epilogue, warp 8 is the producer (cp.async.bulk + mbarrier ring).
#include "common.cuh"
#include <cstdint>
#include <cstdlib>
#include <cmath>
#include <vector>
#include <algorithm>

namespace cvxb {

namespace {

constexpr int OZ_SMAX = 9;
constexpr int OZ_T = 128;                 // tile edge (rows and columns of C)
constexpr int OZ_KS = 32;                 // K rows per MMA (32 bytes of int8)
constexpr int OZ_UNIT = OZ_T * OZ_KS;     // 4096 B
constexpr int OZ_RING = 54;                // 4 KB units in the shared-memory ring (216 KB)
constexpr int OZ_MAXST = 8;                // most stages a pass may split the ring into
constexpr int OZ_MAXPASS = (OZ_SMAX + 1) / 2;
constexpr int OZ_SMEM = OZ_RING * OZ_UNIT + 1024 + 256;
constexpr int OZ_MMA_WARPS = 8;            // two warpgroups
constexpr int OZ_THREADS1 = 32 * OZ_MMA_WARPS + 32;     // + the producer warp
constexpr int OZ_KRANGE = 32768 / OZ_KS;  // k steps per drain (int32 overflow bound)

// byte offset of (row r of the unit = column of A, k byte kb) inside a 4 KB unit
__host__ __device__ inline int oz_unit_off(int layout, int r, int kb) {
    if (layout == 0)        // K-major, 32-byte swizzle: 16-byte chunk index ^= address bit 7
        return r * 32 + ((((kb >> 4) ^ (r >> 2)) & 1) << 4) + (kb & 15);
    // no swizzle, 8x16-byte core matrices: [row group][k chunk][row in group][16 B]
    return (r >> 3) * 256 + (kb >> 4) * 128 + (r & 7) * 16 + (kb & 15);
}

struct OzParams {
    const uint8_t *Q;          // units, [nblk][nk][S][4096]
    const double *cs;          // 2^e_j per column
    const double *D; long long ldd;
    double *C; long long ldc;
    double beta;
    int n, nblk, nk, S;
    int layout;                // 0: SW32; 1: none (core matrices 128 B apart along K, 256 B along rows)
    int npass;                 // level groups: pass ps accumulates levels pd0[ps] .. pd1[ps] (<= 2 of them)
    int pd0[OZ_MAXPASS], pd1[OZ_MAXPASS];
    const unsigned int *tiles; // (I << 16) | J per CTA, in launch order
    // split-K launch of the tail wave: CTA b works on tile b / nchunk over k steps [c*kper, (c+1)*kper), c = b % nchunk,
    // and writes its 128 x 128 partial (tile-local, column-major) to part + b * 128*128; oz_tail_reduce_kernel sums them
    int nchunk, kper;
    double *part;
    int kb2, kb5;              // k steps per ring stage for passes with <= 2 / <= 5 slices (ozaki_syrk sets 4 / 1)
};

// ---- wgmma (sm_90a): D(64 x N, registers of one warpgroup) += A(64 x 32, smem) * B(N x 32, smem)', int8 -> int32.
// Fragment of thread t (warp w = t/32 of the warpgroup, lane l): d[i] is row 16w + l/4 + 8*((i>>1)&1),
// column 8*(i>>2) + 2*(l%4) + (i&1); with N = 256, d[64 + i] is column 128 + that.
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accesses of the accumulators across a wgmma fence / wait
__device__ __forceinline__ void wg_fence_acc(uint32_t (&d)[64]) {
#pragma unroll
    for (int i = 0; i < 64; ++i) asm volatile("" : "+r"(d[i])::"memory");
}
__device__ __forceinline__ void wg_mma128(uint32_t (&d)[64], uint64_t da, uint64_t db) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p;\n\t}"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
        : "l"(da), "l"(db), "r"(1));
}
__device__ __forceinline__ void wg_mma256(uint32_t (&d0)[64], uint32_t (&d1)[64], uint64_t da, uint64_t db) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p;\n\t}"
        : "+r"(d0[0]), "+r"(d0[1]), "+r"(d0[2]), "+r"(d0[3]), "+r"(d0[4]), "+r"(d0[5]), "+r"(d0[6]), "+r"(d0[7]), "+r"(d0[8]), "+r"(d0[9]), "+r"(d0[10]), "+r"(d0[11]), "+r"(d0[12]), "+r"(d0[13]), "+r"(d0[14]), "+r"(d0[15]), "+r"(d0[16]), "+r"(d0[17]), "+r"(d0[18]), "+r"(d0[19]), "+r"(d0[20]), "+r"(d0[21]), "+r"(d0[22]), "+r"(d0[23]), "+r"(d0[24]), "+r"(d0[25]), "+r"(d0[26]), "+r"(d0[27]), "+r"(d0[28]), "+r"(d0[29]), "+r"(d0[30]), "+r"(d0[31]), "+r"(d0[32]), "+r"(d0[33]), "+r"(d0[34]), "+r"(d0[35]), "+r"(d0[36]), "+r"(d0[37]), "+r"(d0[38]), "+r"(d0[39]), "+r"(d0[40]), "+r"(d0[41]), "+r"(d0[42]), "+r"(d0[43]), "+r"(d0[44]), "+r"(d0[45]), "+r"(d0[46]), "+r"(d0[47]), "+r"(d0[48]), "+r"(d0[49]), "+r"(d0[50]), "+r"(d0[51]), "+r"(d0[52]), "+r"(d0[53]), "+r"(d0[54]), "+r"(d0[55]), "+r"(d0[56]), "+r"(d0[57]), "+r"(d0[58]), "+r"(d0[59]), "+r"(d0[60]), "+r"(d0[61]), "+r"(d0[62]), "+r"(d0[63]), "+r"(d1[0]), "+r"(d1[1]), "+r"(d1[2]), "+r"(d1[3]), "+r"(d1[4]), "+r"(d1[5]), "+r"(d1[6]), "+r"(d1[7]), "+r"(d1[8]), "+r"(d1[9]), "+r"(d1[10]), "+r"(d1[11]), "+r"(d1[12]), "+r"(d1[13]), "+r"(d1[14]), "+r"(d1[15]), "+r"(d1[16]), "+r"(d1[17]), "+r"(d1[18]), "+r"(d1[19]), "+r"(d1[20]), "+r"(d1[21]), "+r"(d1[22]), "+r"(d1[23]), "+r"(d1[24]), "+r"(d1[25]), "+r"(d1[26]), "+r"(d1[27]), "+r"(d1[28]), "+r"(d1[29]), "+r"(d1[30]), "+r"(d1[31]), "+r"(d1[32]), "+r"(d1[33]), "+r"(d1[34]), "+r"(d1[35]), "+r"(d1[36]), "+r"(d1[37]), "+r"(d1[38]), "+r"(d1[39]), "+r"(d1[40]), "+r"(d1[41]), "+r"(d1[42]), "+r"(d1[43]), "+r"(d1[44]), "+r"(d1[45]), "+r"(d1[46]), "+r"(d1[47]), "+r"(d1[48]), "+r"(d1[49]), "+r"(d1[50]), "+r"(d1[51]), "+r"(d1[52]), "+r"(d1[53]), "+r"(d1[54]), "+r"(d1[55]), "+r"(d1[56]), "+r"(d1[57]), "+r"(d1[58]), "+r"(d1[59]), "+r"(d1[60]), "+r"(d1[61]), "+r"(d1[62]), "+r"(d1[63])
        : "l"(da), "l"(db), "r"(1));
}

// shared-memory matrix descriptor: start address, leading / stride byte offsets, swizzle mode (bits 62-63, 3 = 32 B)
__device__ __forceinline__ uint64_t wg_desc(uint32_t saddr, uint64_t hi) { return hi | (uint64_t)((saddr >> 4) & 0x3FFFu); }

// One k step of a pass whose level range {D0} or {D0, D0+1} is known at compile time.  A slice s meets the B slices
// t = D0-s and D0+1-s, which sit back to back in shared memory: one m64n256k32 wgmma covers both levels (acc0 |
// acc1); at the edges of the range a single m64n128k32 one.
template <int D0, int D1>
__device__ __forceinline__ void oz_issue_step(uint32_t a0, uint32_t b0, uint64_t hi, uint32_t (&acc0)[64],
                                              uint32_t (&acc1)[64]) {
#pragma unroll
    for (int s = 0; s <= D1; ++s) {
        const uint64_t da = wg_desc(a0 + s * OZ_UNIT, hi);
        const int tlo = (D0 - s) > 0 ? (D0 - s) : 0, thi = D1 - s;
        const uint64_t db = wg_desc(b0 + tlo * OZ_UNIT, hi);
        if (thi > tlo) wg_mma256(acc0, acc1, da, db);
        else if (s + tlo == D0) wg_mma128(acc0, da, db);
        else wg_mma128(acc1, da, db);
    }
}

// k steps per ring stage: the passes with few slices hold little tensor work per k step, so they put several
// k steps behind one producer / consumer handshake
__device__ __forceinline__ int oz_kb(const OzParams &p, int nS) { return nS <= 2 ? p.kb2 : (nS <= 5 ? p.kb5 : 1); }

__global__ void __launch_bounds__(OZ_THREADS1, 1) oz_mma_kernel(OzParams p) {
    extern __shared__ uint8_t oz_smem_raw[];
    // warp index through a shuffle: the compiler then knows the role branches are warp-uniform (wgmma issue
    // inside a branch it thinks divergent is serialised)
    const int tid = threadIdx.x, warp = __shfl_sync(0xffffffffu, tid >> 5, 0), lane = tid & 31;
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(oz_smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem + OZ_RING * OZ_UNIT);
    uint64_t *full = bars, *empty = bars + OZ_MAXST;

    // lower-triangular tile (I >= J) of this CTA
    const bool split = p.nchunk > 1;
    const unsigned int tl = p.tiles[split ? blockIdx.x / p.nchunk : blockIdx.x];
    const int I = (int)(tl >> 16), J = (int)(tl & 0xFFFFu);
    const int kb = split ? (int)(blockIdx.x % p.nchunk) * p.kper : 0;
    const int ke = split ? min(p.nk, kb + p.kper) : p.nk;

    if (tid == 0) {
        for (int s = 0; s < OZ_MAXST; ++s) { mbar_init(full + s, 1); mbar_init(empty + s, OZ_MMA_WARPS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    const int S = p.S;
    const int npass = p.npass;
    const int nrange = (ke - kb + OZ_KRANGE - 1) / OZ_KRANGE;
    // Stage geometry of a pass: nS slices of A then nS slices of B per k step; the ring is cut into
    // as many such stages as fit (deeper prefetch for the passes that need few slices).

    if (warp == OZ_MMA_WARPS) {
        if (lane == 0) {
            // ===== producer: one bulk copy per operand per k step =====
            uint32_t filled = 0, epar = 0;               // per stage: ever filled / parity of its last release
            for (int rg = 0; rg < nrange; ++rg) {
                const int k0 = kb + rg * OZ_KRANGE, k1 = min(ke, k0 + OZ_KRANGE);
                for (int ps = 0; ps < npass; ++ps) {
                    const int nS = min(S, p.pd1[ps] + 1);
                    const int KB = oz_kb(p, nS);
                    const int nst = min(OZ_MAXST, OZ_RING / (2 * nS * KB));
                    const uint32_t bytes = (uint32_t)nS * OZ_UNIT;
                    // the new geometry overlaps the old stages: wait until every one of them is released
                    for (int s2 = 0; s2 < OZ_MAXST; ++s2)
                        if ((filled >> s2) & 1u) mbar_wait(empty + s2, (epar >> s2) & 1u);
                    int st = 0;
                    for (int kc = k0; kc < k1; kc += KB) {
                        const int kn = min(KB, k1 - kc);
                        if ((filled >> st) & 1u) { mbar_wait(empty + st, (epar >> st) & 1u); epar ^= 1u << st; }
                        else filled |= 1u << st;
                        mbar_expect_tx(full + st, 2 * bytes * (uint32_t)kn);
                        uint8_t *sa = smem + (size_t)st * 2 * bytes * KB;
                        for (int i = 0; i < kn; ++i, sa += 2 * bytes) {
                            bulk_g2s(sa, p.Q + ((size_t)I * p.nk + kc + i) * (size_t)S * OZ_UNIT, bytes, full + st);
                            bulk_g2s(sa + bytes, p.Q + ((size_t)J * p.nk + kc + i) * (size_t)S * OZ_UNIT, bytes, full + st);
                        }
                        if (++st == nst) st = 0;
                    }
                }
            }
        }
        return;
    }

    // ===== MMA warpgroups: warpgroup wg owns rows 64*wg .. 64*wg+63 of the tile =====
    const int wg = warp >> 2;
    const uint64_t hi = (p.layout == 0) ? ((uint64_t)(256 >> 4) << 32) | (1ull << 16) | (3ull << 62)
                                        : ((uint64_t)(256 >> 4) << 32) | ((uint64_t)(128 >> 4) << 16);
    const uint32_t sbase = smem_u32(smem);
    const int rl0 = 64 * wg + 16 * (warp & 3) + (lane >> 2);       // tile-local rows rl0, rl0 + 8
    const int cl0 = 2 * (lane & 3);                                // tile-local columns cl0 + 8*(i>>2) + (i&1)
    const int row0 = I * OZ_T + rl0;
    const double rsc[2] = {row0 < p.n ? p.cs[row0] : 0.0, row0 + 8 < p.n ? p.cs[row0 + 8] : 0.0};
    uint32_t cpar = 0;                                             // per stage: parity of its next fill
    int g = 0;                                                     // global pass counter
    for (int rg = 0; rg < nrange; ++rg) {
        const int k0 = kb + rg * OZ_KRANGE, k1 = min(ke, k0 + OZ_KRANGE);
        for (int ps = 0; ps < npass; ++ps, ++g) {
            const int d0 = p.pd0[ps], d1 = p.pd1[ps];
            const int nS = min(S, d1 + 1);
            const int KB = oz_kb(p, nS);
            const int nst = min(OZ_MAXST, OZ_RING / (2 * nS * KB));
            const uint32_t bytes = (uint32_t)nS * OZ_UNIT;
            const int code = d0 * 16 + d1;
            uint32_t acc0[64], acc1[64];
#pragma unroll
            for (int i = 0; i < 64; ++i) acc0[i] = acc1[i] = 0u;
            int st = 0, prev = -1;
            for (int kc = k0; kc < k1; kc += KB) {
                const int kn = min(KB, k1 - kc);
                mbar_wait(full + st, (cpar >> st) & 1u);
                cpar ^= 1u << st;
                wg_fence_acc(acc0); wg_fence_acc(acc1);
                wg_fence();
                for (int i = 0; i < kn; ++i) {
                    const uint32_t a0 = sbase + ((uint32_t)st * KB + (uint32_t)i) * 2u * bytes + (uint32_t)wg * (OZ_UNIT / 2);
                    const uint32_t b0 = sbase + ((uint32_t)st * KB + (uint32_t)i) * 2u * bytes + bytes;
#define OZ_CASE(D0, D1) \
    case (D0) * 16 + (D1): oz_issue_step<D0, D1>(a0, b0, hi, acc0, acc1); break;
                    switch (code) {
                        OZ_CASE(0, 0) OZ_CASE(0, 1) OZ_CASE(2, 2) OZ_CASE(2, 3) OZ_CASE(4, 4)
                        OZ_CASE(4, 5) OZ_CASE(6, 6) OZ_CASE(6, 7) OZ_CASE(8, 8)
                        default: break;
                    }
#undef OZ_CASE
                }
                wg_commit();
                wg_fence_acc(acc0); wg_fence_acc(acc1);
                wg_wait<1>();                            // the previous stage's wgmmas have read their operands
                if (prev >= 0 && lane == 0) mbar_arrive(empty + prev);
                prev = st;
                if (++st == nst) st = 0;
            }
            wg_wait<0>();
            wg_fence_acc(acc0); wg_fence_acc(acc1);
            if (prev >= 0 && lane == 0) mbar_arrive(empty + prev);

            // ===== epilogue: C (or the split-K partial tile) += 2^(-12 - 7 d1) (128 acc0 + acc1) * cs_i * cs_j =====
            const int nlev = d1 - d0 + 1;
            const double lsc = ldexp(1.0, -12 - 7 * (d0 + nlev - 1));
            const bool first = (g == 0);
            double *const part0 = split ? p.part + (size_t)blockIdx.x * (OZ_T * OZ_T) : nullptr;
#pragma unroll
            for (int i = 0; i < 64; ++i) {
                const int h = (i >> 1) & 1;
                const int rl = rl0 + 8 * h, cl = cl0 + 8 * (i >> 2) + (i & 1);
                const int row = I * OZ_T + rl, col = J * OZ_T + cl;
                double v = (double)(int)acc0[i];
                if (nlev > 1) v = fma(v, 128.0, (double)(int)acc1[i]);
                if (split) {
                    double *q = part0 + rl + (size_t)cl * OZ_T;
                    const double old = first ? 0.0 : *q;
                    *q = ((col < p.n) ? (v * lsc) * rsc[h] * p.cs[col] : 0.0) + old;
                } else if (row < p.n && col < p.n && col <= row) {
                    double *q = p.C + row + (size_t)col * p.ldc;
                    const double old = !first ? *q : (p.D ? p.beta * p.D[row + (size_t)col * p.ldd] : 0.0);
                    *q = (v * lsc) * rsc[h] * p.cs[col] + old;
                }
            }
        }
    }
}

// C tile = beta * D + sum of the nchunk partial tiles of the split-K tail launch (fixed order: deterministic)
__global__ void oz_tail_reduce_kernel(OzParams p, int ntail) {
    const int t = blockIdx.y;
    const unsigned int tl = p.tiles[t];
    const int I = (int)(tl >> 16), J = (int)(tl & 0xFFFFu);
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= OZ_T * OZ_T) return;
    const int r = e % OZ_T, c = e / OZ_T;
    const int row = I * OZ_T + r, col = J * OZ_T + c;
    if (row >= p.n || col >= p.n || col > row) return;
    double v = p.D ? p.beta * p.D[row + (size_t)col * p.ldd] : 0.0;
    const double *src = p.part + (size_t)t * p.nchunk * (OZ_T * OZ_T) + e;
    for (int ch = 0; ch < p.nchunk; ++ch) v += src[(size_t)ch * (OZ_T * OZ_T)];
    p.C[row + (size_t)col * p.ldc] = v;
}

// amax[j] = max_k |d[k] * A[k,j]|  ->  cs[j] = 2^e_j, sinv[j] = 64 * 2^-e_j
__global__ void oz_colscale_kernel(int m, int n, const double *A, long long lda, const double *d, double *cs, double *sinv) {
    __shared__ double sh[32];
    const int j = blockIdx.x;
    const double *a = A + (size_t)j * lda;
    double mx = 0.0;
    for (int k = threadIdx.x; k < m; k += blockDim.x) {
        double v = fabs((d ? d[k] : 1.0) * a[k]);
        if (!(v <= 1.7976931348623157e308)) v = INFINITY;      // NaN or Inf entry: poison the column (below)
        mx = fmax(mx, v);
    }
    for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = mx;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < (blockDim.x >> 5); ++w) mx = fmax(mx, sh[w]);
        int e = 0;
        if (mx > 0.0 && mx < INFINITY) frexp(mx, &e);         // mx = f * 2^e, f in [0.5, 1): |x| < 2^e
        // a non-finite entry makes row and column j of C NaN, as the fp64 kernel would (potrf then reports it)
        cs[j] = (mx < INFINITY) ? ldexp(1.0, e) : __longlong_as_double(0x7ff8000000000000LL);
        sinv[j] = (mx < INFINITY) ? ldexp(64.0, -e) : 0.0;
    }
}

// digits of column block cb, k step kc (one 128-column x 32-row block of Gs = 9 units).  The block is read with
// coalesced 256-byte rows (lane = k, one column per load instruction) into shared memory and sliced from there by one
// thread per column; reading it with one thread per column straight from global memory (32 distinct lines per load
// instruction) was several times slower.
__global__ void __launch_bounds__(OZ_T) oz_slice_kernel(int m, int n, const double *A, long long lda, const double *d,
                                                        const double *sinv, uint8_t *Q, int nk, int S, int layout) {
    __shared__ double tile[OZ_T][OZ_KS + 1];
    const int cb = blockIdx.y, kc = blockIdx.x, r = threadIdx.x, lane = r & 31, warp = r >> 5;
    {
        const int k = kc * OZ_KS + lane;
        const double dk = (k < m) ? (d ? d[k] : 1.0) : 0.0;
#pragma unroll 8
        for (int c = 0; c < 32; ++c) {
            const int cc = warp * 32 + c, j = cb * OZ_T + cc;
            double x = 0.0;
            if (j < n && k < m) x = dk * A[(size_t)j * lda + k];
            tile[cc][lane] = x;
        }
    }
    __syncthreads();
    const int j = cb * OZ_T + r;
    const double sc = (j < n) ? sinv[j] : 0.0;
    uint8_t *unit0 = Q + ((size_t)cb * nk + kc) * (size_t)S * OZ_UNIT;
    for (int half = 0; half < 2; ++half) {
        uint32_t pk[OZ_SMAX][4];
#pragma unroll
        for (int s = 0; s < OZ_SMAX; ++s) pk[s][0] = pk[s][1] = pk[s][2] = pk[s][3] = 0u;
#pragma unroll
        for (int e = 0; e < 16; ++e) {
            double x = tile[r][half * 16 + e] * sc;                          // |x| < 64 (0 outside the matrix)
#pragma unroll
            for (int s = 0; s < OZ_SMAX; ++s) {
                if (s < S) {
                    // round to nearest-even integer by adding 1.5 * 2^52 (|x| <= 8192 here): the sum's low mantissa word
                    // IS the integer in two's complement, so there is neither a FRND nor an F2I (both quarter rate) per
                    // digit: this kernel was bound by them
                    const double t = x + 6755399441055744.0;
                    const double q = t - 6755399441055744.0;               // == rint(x)
                    x = (x - q) * 128.0;                                   // exact
                    pk[s][e >> 2] |= ((uint32_t)__double2loint(t) & 0xFFu) << ((e & 3) * 8);
                }
            }
        }
        const int off = oz_unit_off(layout, r, half * 16);
#pragma unroll
        for (int s = 0; s < OZ_SMAX; ++s)
            if (s < S)
                *reinterpret_cast<uint4 *>(unit0 + (size_t)s * OZ_UNIT + off) = make_uint4(pk[s][0], pk[s][1], pk[s][2], pk[s][3]);
    }
}

}  // namespace

// C(lower) = A' diag(d)^2 A + beta * D.  A: m x n (lda), d: m (or nullptr).  work: ozaki_workspace_bytes.
// Levels are taken in pairs {0,1} {2,3} ... (two int32 accumulators per output element fit the register file).

// Optional timing of the MMA launches alone (without the two slicing kernels): the NEXT ozaki_syrk call of this thread
// records `a` before its first MMA launch and `b` after its last one (bench.py's roofline line via cvxb_kkt_syrk_mma_ms).
static thread_local cudaEvent_t g_oz_ev0 = nullptr, g_oz_ev1 = nullptr;
void ozaki_time_mma(cudaEvent_t a, cudaEvent_t b) { g_oz_ev0 = a; g_oz_ev1 = b; }

size_t ozaki_workspace_bytes(int n, int m, int S) {
    const size_t nblk = (n + OZ_T - 1) / OZ_T, nk = std::max(1, (m + OZ_KS - 1) / OZ_KS);
    return nblk * nk * (size_t)S * OZ_UNIT + 2 * (size_t)n * sizeof(double) + nblk * (nblk + 1) / 2 * sizeof(unsigned int) + 1024
           + (size_t)kNumSMs * OZ_T * OZ_T * sizeof(double) + 256;         // partial tiles of the split-K tail wave
}

int ozaki_mode() {
    const char *e = getenv("CVXB_OZAKI");
    return !e ? 0 : (e[0] == '0') ? 0 : (e[0] == '2') ? 2 : 1;
}

bool ozaki_use(int mode, int n, int m, DevBuf<char> &work) {
    if (!(mode == 2 || (mode == 1 && n >= 4096 && m >= 8192))) return false;
    // the slice workspace is ~1.125 x sizeof(A)
    const size_t need = ozaki_workspace_bytes(n, m, 9);
    return need <= work.n || work.try_alloc(need) == cudaSuccess;
}

int ozaki_syrk(int n, int m, const double *A, long long lda, const double *d, const double *D, long long ldd,
               double beta, double *C, long long ldc, int S, int layout, void *work, cudaStream_t st) {
    if (n <= 0) return 0;
    if (S < 1 || S > OZ_SMAX || !A || !C || !work || m < 0 || (layout != 0 && layout != 1)) {
        set_error("ozaki_syrk: bad arguments");
        return CVXB_E_ARG;
    }
    static DeviceOnce once;
    if (const unsigned long long bit = once.pending()) {
        CVXB_CUDA(cudaFuncSetAttribute(oz_mma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, OZ_SMEM));
        once.mark(bit);
    }
    const int nblk = (n + OZ_T - 1) / OZ_T, nk = std::max(1, (m + OZ_KS - 1) / OZ_KS);
    if (nblk > 65535) { set_error("ozaki_syrk: n too large"); return CVXB_E_ARG; }
    const long long tiles = (long long)nblk * (nblk + 1) / 2;
    double *cs = reinterpret_cast<double *>(work);
    double *sinv = cs + n;
    unsigned int *dtiles = reinterpret_cast<unsigned int *>(sinv + n);
    uint8_t *Q = reinterpret_cast<uint8_t *>(((uintptr_t)(dtiles + tiles) + 255) & ~uintptr_t(255));
    // launch order: bands of tile rows, column by column inside a band, so that the tiles in flight form a
    // compact block (few distinct operand streams -> L2 hits instead of HBM reads)
    // (rebuilt per call: a few microseconds, and no shared mutable state between threads / handles; the
    // pageable-source copy is staged before cudaMemcpyAsync returns)
    std::vector<unsigned int> order;
    order.reserve((size_t)tiles);
    const int band = 12;
    for (int r0 = 0; r0 < nblk; r0 += band) {
        const int r1 = std::min(nblk, r0 + band);
        for (int J = 0; J < r1; ++J)
            for (int I = std::max(r0, J); I < r1; ++I) order.push_back(((unsigned)I << 16) | (unsigned)J);
    }
    CVXB_CUDA(cudaMemcpyAsync(dtiles, order.data(), order.size() * sizeof(unsigned int), cudaMemcpyHostToDevice, st));
    oz_colscale_kernel<<<n, 256, 0, st>>>(m, n, A, lda, d, cs, sinv);
    count_launch();
    oz_slice_kernel<<<dim3(nk, nblk), OZ_T, 0, st>>>(m, n, A, lda, d, sinv, Q, nk, S, layout);
    count_launch();
    OzParams p;
    p.Q = Q; p.cs = cs; p.D = D; p.ldd = ldd; p.C = C; p.ldc = ldc; p.beta = beta;
    p.n = n; p.nblk = nblk; p.nk = nk; p.S = S; p.layout = layout; p.tiles = dtiles;
    p.nchunk = 1; p.kper = nk; p.part = nullptr;
    p.kb2 = 4; p.kb5 = 1;
    p.npass = 0;
    for (int d0 = 0; d0 < S; d0 += 2, ++p.npass) { p.pd0[p.npass] = d0; p.pd1[p.npass] = std::min(S - 1, d0 + 1); }
    cudaEvent_t tev0 = g_oz_ev0, tev1 = g_oz_ev1;
    g_oz_ev0 = g_oz_ev1 = nullptr;
    if (tev0) CVXB_CUDA(cudaEventRecord(tev0, st));
    // The last, partial wave of tiles (2080 = 15 x 132 + 100 at n = 8192) would leave SMs idle for a whole tile
    // time: when it fills at most half the SMs, its tiles are split along K over all SMs (partials + ordered
    // reduce).
    long long tmain = tiles;
    int ntail = (int)(tiles % kNumSMs), nchunk = 1;
    if (tiles > kNumSMs && ntail > 0 && ntail <= kNumSMs / 2) {
        nchunk = std::min(kNumSMs / ntail, nk);
        if (nchunk >= 2) tmain = tiles - ntail; else nchunk = 1;
    }
    if (tmain > 0) oz_mma_kernel<<<(unsigned)tmain, OZ_THREADS1, OZ_SMEM, st>>>(p);
    if (nchunk >= 2) {
        OzParams pt = p;
        pt.tiles = dtiles + tmain;
        pt.kper = (nk + nchunk - 1) / nchunk;
        pt.nchunk = (nk + pt.kper - 1) / pt.kper;                 // no empty chunk
        pt.part = reinterpret_cast<double *>(((uintptr_t)(Q + (size_t)nblk * nk * S * OZ_UNIT) + 255) & ~uintptr_t(255));
        oz_mma_kernel<<<(unsigned)(ntail * pt.nchunk), OZ_THREADS1, OZ_SMEM, st>>>(pt);
        oz_tail_reduce_kernel<<<dim3(OZ_T * OZ_T / 256, ntail), 256, 0, st>>>(pt, ntail);
        count_launch(2);
    }
    if (tev1) CVXB_CUDA(cudaEventRecord(tev1, st));
    count_launch();
    CVXB_LAUNCH_CHECK();
    return 0;
}

}  // namespace cvxb
