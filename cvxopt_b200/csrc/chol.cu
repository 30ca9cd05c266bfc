// Dense fp64 Cholesky (lower) + triangular solves for sm_90a.
//
// Replaces lapack.potrf / lapack.potrs as called by the reference KKT solver
// (reference src/python/misc.py:1282 and :1327; bindings src/C/lapack.c:1471, :1553).
//
// potrf_lower: right-looking blocked factorisation with NB = 128.
//   step j:  (1) potf2_inv   : one CTA factors the 128x128 diagonal block in shared
//                              memory and also produces its inverse (kept for the solves)
//            (2) panel TRSM  : L21 = A21 * inv(L11)'  as a DMMA GEMM (gemm_dmma.cu)
//            (3) trailing    : A22 -= L21 L21'  (lower tiles)
//   Look-ahead: the next block column of (3) runs on the high-priority panel stream together with (1),(2)
//   (dmma_gemm_kernel).  The rest of (3) is grouped by four panels: the columns inside the panel's group on a
//   high-priority stream (dmma_gemm_kernel, K = 128), the next group's columns per panel and everything beyond
//   as one K = 512 far update per group on the low-priority update stream (syrk_tma_kernel, from a K-major copy
//   of the group's panels), so the latency-bound panel work hides behind the throughput-bound updates.
//
// trsv_lower: blocked substitution that re-uses the diagonal-block inverses; one CTA
//   per 128-row block, progress published through acquire/release flags so that the
//   whole triangular solve is a single kernel (no per-block launches).
#include "common.cuh"
#include <cstdlib>

namespace cvxb {

namespace {

constexpr int PB = 8;                  // inner block width of the in-CTA factorisation
constexpr int SP = 12;                 // row stride (doubles) of the panel buffer: conflict-free frags
constexpr int LDM = NB + 4;            // column stride (doubles) of the shared-memory block
constexpr int POTF2_SMEM = (NB * LDM + NB * SP + 4 * 80) * 8;
constexpr int kGroup = 4;              // panels per far update of potrf_lower (K = 512)

// acc[cf][rf] -= sum_k Lt[c, k] Lt[r, k] over k = 0..127 for the tiles rf >= S_cf of each column
// fragment cf (Lt in shared memory, column-major with stride LDM; Ma/Mb already offset by lane).
// Column fragments 2mf and 2mf+1 go through one m16n8k4, so where only the first of the pair is live the
// second, strictly upper tile gets a product too; nothing reads an upper tile's accumulators.
template <int PAT>      // 0: every tile, 1: rf >= cf, 2: rf >= 4 + cf
__device__ __forceinline__ void sym_update(double (&acc)[4][8][2], const double *Ma, const double *Mb) {
#pragma unroll 2
    for (int kk = 0; kk < NB / 4; ++kk) {
        double a[4], bfr[8];
#pragma unroll
        for (int cf = 0; cf < 4; ++cf) a[cf] = -Ma[cf * 8 + kk * 4 * LDM];
#pragma unroll
        for (int rf = 0; rf < 8; ++rf) bfr[rf] = Mb[rf * 8 + kk * 4 * LDM];
#pragma unroll
        for (int mf = 0; mf < 2; ++mf)
#pragma unroll
            for (int rf = 0; rf < 8; ++rf) {
                if (PAT == 1 && rf < 2 * mf) continue;           // compile-time after unrolling
                if (PAT == 2 && rf < 4 + 2 * mf) continue;
                dmma16x8x4(acc[2 * mf][rf][0], acc[2 * mf][rf][1], acc[2 * mf + 1][rf][0], acc[2 * mf + 1][rf][1],
                           a[2 * mf], a[2 * mf + 1], bfr[rf]);
            }
    }
}

// Factor the jb x jb diagonal block at A (lower) in place, write inv(L) (NB x NB,
// ld NB, zero upper, identity padding beyond jb) to inv.
//
// The 128x128 block lives in REGISTERS as DMMA accumulator fragments (64 doubles per
// thread, same 8-warp 64x32 layout as the GEMM).  Right-looking with an 8-wide inner
// block: the owning warps drop the current 128x8 column block into shared memory,
// every warp re-derives the 8x8 Cholesky factor with shuffles (no CTA barrier for it),
// 128 row-threads do the 8-step substitution, then all warps apply the rank-8 update to
// their fragments with two DMMA k-steps per tile.  The inverse is then built in shared
// memory by recursive doubling (X21 = -X22 (L21 X11)) with DMMA tile products.
__global__ void __launch_bounds__(256, 1)
potf2_inv_kernel(double *A, long long lda, int jb, double *inv, double *invT, int *info, int joff,
                 long long sA, long long sInv, const double *Tprev, long long ldt,
                 const double *invprev, unsigned long long *trace) {
    extern __shared__ __align__(16) double sm[];
    if (trace && threadIdx.x == 0) {
        unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); trace[0] = t;
    }
#define CVXB_STAMP(SLOT)                                                                    \
    if (trace && threadIdx.x == 0) {                                                        \
        unsigned long long t_; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_));       \
        trace[8 * 2048 + (SLOT)] = t_;                                                      \
    }
    A += (long long)blockIdx.x * sA; inv += (long long)blockIdx.x * sInv;
    invT += (long long)blockIdx.x * sInv; info += blockIdx.x;
    double *M = sm;                    // NB x LDM, column-major
    double *P = M + NB * LDM;          // NB x SP, row-major panel
    double *Dw = P + NB * SP;          // 4 private copies of the 8x8 factor (+ reciprocal diagonal)
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    // Warp -> 64x32 fragment block.  Only the lower triangle is live, so the blocks carry very
    // different amounts of DMMA work; warps w and w+4 share an SM sub-partition, so pair a heavy
    // block with a light one: SMSP0 (1,0)+(0,2), SMSP1 (1,1)+(0,3), SMSP2 (1,2)+(0,1), SMSP3 (0,0)+(1,3)
    const int role = (0x72640531 >> (warp * 4)) & 7;     // role = wr + 2*wc, one nibble per warp
    const int wr = role & 1, wc = role >> 1;
    const int g4 = lane >> 2, t4 = lane & 3;

    double acc[4][8][2];
    // ---- optional prologue (look-ahead of the blocked factorisation): this diagonal block still
    // misses the previous step's update.  Tprev = A(j, j-1) before its TRSM, invprev = inv(L_{j-1,j-1}):
    //   Lt = Tprev * invprev'   (private copy of L(j, j-1)),   C -= Lt Lt'
    // so the chain of diagonal factorisations never waits for the full-width TRSM / update.
    if (Tprev != nullptr) {
#pragma unroll
        for (int cf = 0; cf < 4; ++cf)
#pragma unroll
            for (int rf = 0; rf < 8; ++rf) acc[cf][rf][0] = acc[cf][rf][1] = 0.0;
        const int kkmax = (wc + 1) * 8;                 // invprev[c, k] = 0 for k > c
        // Tprev (jb x 128) goes to shared memory M in one burst of async copies: read straight from global memory in
        // the k loop, the loop was a chain of L2 round trips (6 us for 0.5 MFLOP per warp)
        {
            const bool v16 = ((ldt & 1) == 0) && ((reinterpret_cast<uintptr_t>(Tprev) & 15) == 0);
            if (v16) {
                for (int q = tid; q < NB * NB / 2; q += 256) {
                    const int c = q >> 6, r = (q & 63) * 2;
                    const int nb = (r + 1 < jb) ? 16 : (r < jb ? 8 : 0);
                    cp_async16(M + r + c * LDM, nb ? Tprev + r + (long long)c * ldt : Tprev, nb);
                }
            } else {
                for (int q = tid; q < NB * NB; q += 256) {
                    const int c = q >> 7, r = q & 127;
                    cp_async8(M + r + c * LDM, (r < jb) ? Tprev + r + (long long)c * ldt : Tprev, (r < jb) ? 8 : 0);
                }
            }
            cp_async_commit();
        }
        const double *ip = invprev + (wc * 32 + g4) + t4 * NB;
        // first fragments of inv(L_prev) while the copies are in flight
        double a0[4];
#pragma unroll
        for (int cf = 0; cf < 4; ++cf) a0[cf] = ip[cf * 8];
        cp_async_wait<0>();
        __syncthreads();
        const double *tq = M + (wr * 64 + g4) + t4 * LDM;
#pragma unroll 2
        for (int kk = 0; kk < kkmax; ++kk) {
            double a[4], bfr[8];
#pragma unroll
            for (int cf = 0; cf < 4; ++cf) a[cf] = a0[cf];
            if (kk + 1 < kkmax) {
#pragma unroll
                for (int cf = 0; cf < 4; ++cf) a0[cf] = ip[cf * 8 + (kk + 1) * 4 * NB];
            }
#pragma unroll
            for (int rf = 0; rf < 8; ++rf) bfr[rf] = tq[rf * 8 + kk * 4 * LDM];
#pragma unroll
            for (int mf = 0; mf < 2; ++mf)
#pragma unroll
                for (int rf = 0; rf < 8; ++rf)
                    dmma16x8x4(acc[2 * mf][rf][0], acc[2 * mf][rf][1], acc[2 * mf + 1][rf][0],
                               acc[2 * mf + 1][rf][1], a[2 * mf], a[2 * mf + 1], bfr[rf]);
        }
        __syncthreads();                                // every warp is done reading Tprev from M
#pragma unroll
        for (int cf = 0; cf < 4; ++cf)
#pragma unroll
            for (int rf = 0; rf < 8; ++rf)
#pragma unroll
                for (int e = 0; e < 2; ++e)
                    M[(wr * 64 + rf * 8 + t4 * 2 + e) + (wc * 32 + cf * 8 + g4) * LDM] = acc[cf][rf][e];
    }
    CVXB_STAMP(0)
    // the block itself: straight into the fragment registers (identity padding beyond jb)
#pragma unroll
    for (int cf = 0; cf < 4; ++cf)
#pragma unroll
        for (int rf = 0; rf < 8; ++rf)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int r = wr * 64 + rf * 8 + t4 * 2 + e, c = wc * 32 + cf * 8 + g4;
                double v = (r == c) ? 1.0 : 0.0;
                if (r < jb && c < jb && r >= c) v = A[r + (long long)c * lda];
                acc[cf][rf][e] = v;
            }
    __syncthreads();
    CVXB_STAMP(4)
    if (Tprev != nullptr) {
        // which 8x8 tiles of this warp's 64x32 block touch the lower triangle depends only on
        // d = wc - 2*wr: all (d < 0), rf >= cf (d == 0), rf >= 4 + cf (d == 1), none (d > 1).
        // Static patterns keep the DMMA stream free of per-tile branches.
        const int d = wc - 2 * wr;
        const double *Ma = M + (wc * 32 + g4) + t4 * LDM;
        const double *Mb = M + (wr * 64 + g4) + t4 * LDM;
        if (d < 0) sym_update<0>(acc, Ma, Mb);
        else if (d == 0) sym_update<1>(acc, Ma, Mb);
        else if (d == 1) sym_update<2>(acc, Ma, Mb);
        __syncthreads();
    }
    CVXB_STAMP(1)
#pragma unroll 1
    for (int t = 0; t < NB / PB; ++t) {
      {
        const int c0 = t * PB;
        // 1. owners of column block t publish it: P[r][k] = C[r, c0 + k]
        //    (switch keeps the fragment index static without unrolling the whole step 4x)
        if (wc == (t >> 2)) {
#define CVXB_PUBLISH(CF)                                                          \
    _Pragma("unroll") for (int rf = 0; rf < 8; ++rf)                              \
        _Pragma("unroll") for (int e = 0; e < 2; ++e)                             \
            P[(wr * 64 + rf * 8 + t4 * 2 + e) * SP + g4] = acc[CF][rf][e];
            switch (t & 3) {
                case 0: CVXB_PUBLISH(0) break;
                case 1: CVXB_PUBLISH(1) break;
                case 2: CVXB_PUBLISH(2) break;
                default: CVXB_PUBLISH(3) break;
            }
#undef CVXB_PUBLISH
        }
        __syncthreads();
        // 2. 8x8 Cholesky of the diagonal block by a single lane; warps 0-3 pick the factor up from
        //    shared memory behind a 128-thread named barrier, warps 4-7 skip to the CTA barrier.
        if (warp == 0 && lane == 0) {
            // one lane, 36 registers, no shuffles: the critical path per pivot is one rsqrt, one
            // multiply and one FMA (the 32-lane shuffle version spent ~200 cycles per pivot)
            double a[PB][PB];
#pragma unroll
            for (int i = 0; i < PB; ++i)
#pragma unroll
                for (int k = 0; k <= i; ++k) a[i][k] = P[(c0 + i) * SP + k];
            bool bad = false;
#pragma unroll
            for (int j = 0; j < PB; ++j) {
                const double piv = a[j][j];
                if (!(piv > 0.0) && !bad) {
                    atomicCAS(info, 0, joff + c0 + j + 1);
                    bad = true;
                }
                const double rs = rsqrt(piv);
                a[j][j] = piv * rs;
                Dw[64 + j] = rs;
#pragma unroll
                for (int i = j + 1; i < PB; ++i) a[i][j] *= rs;
#pragma unroll
                for (int k = j + 1; k < PB; ++k)
#pragma unroll
                    for (int i = k; i < PB; ++i) a[i][k] -= a[i][j] * a[k][j];
            }
#pragma unroll
            for (int i = 0; i < PB; ++i)
#pragma unroll
                for (int k = 0; k < PB; ++k) Dw[i * 8 + k] = (k <= i) ? a[i][k] : 0.0;
        }
        if (warp < 4) asm volatile("bar.sync 1, 128;" ::: "memory");
        // 3. substitution on the rows below (one row per thread), zero rows above
        if (warp < 4) {
            const double *D = Dw;
            const int r = warp * 32 + lane;
            double x[PB];
            if (r >= c0 + PB) {
#pragma unroll
                for (int j = 0; j < PB; ++j) x[j] = P[r * SP + j];
#pragma unroll
                for (int j = 0; j < PB; ++j) {
                    double v = x[j];
#pragma unroll
                    for (int k = 0; k < j; ++k) v -= x[k] * D[j * 8 + k];
                    x[j] = v * D[64 + j];
                }
            } else if (r >= c0) {
#pragma unroll
                for (int j = 0; j < PB; ++j) x[j] = (j <= r - c0) ? D[(r - c0) * 8 + j] : 0.0;
            } else {
#pragma unroll
                for (int j = 0; j < PB; ++j) x[j] = 0.0;
            }
#pragma unroll
            for (int j = 0; j < PB; ++j) P[r * SP + j] = x[j];
        }
        __syncthreads();
        // 4. rank-8 update of the fragments right/below the block: C -= P P'.  Skipping is
        //    warp-uniform and coarse (whole warp / whole column fragment): per-tile tests put a
        //    branch in front of every DMMA and cost more than the few dead tiles they save.
        if (wr * 8 + 7 > t && wc * 4 + 3 > t) {
            double a[4][2], bfr[8][2];
#pragma unroll
            for (int kk = 0; kk < 2; ++kk) {
#pragma unroll
                for (int cf = 0; cf < 4; ++cf) a[cf][kk] = -P[(wc * 32 + cf * 8 + g4) * SP + kk * 4 + t4];
#pragma unroll
                for (int rf = 0; rf < 8; ++rf) bfr[rf][kk] = P[(wr * 64 + rf * 8 + g4) * SP + kk * 4 + t4];
            }
            // column fragments 2mf and 2mf+1 share one m16n8k4; when only the first is final (it is column
            // block t, published above) its accumulators take a product nobody reads
#pragma unroll
            for (int mf = 0; mf < 2; ++mf) {
                if (wc * 4 + 2 * mf + 1 <= t) continue;    // both column blocks already final
#pragma unroll
                for (int rf = 0; rf < 8; ++rf) {
                    dmma16x8x4(acc[2 * mf][rf][0], acc[2 * mf][rf][1], acc[2 * mf + 1][rf][0], acc[2 * mf + 1][rf][1],
                               a[2 * mf][0], a[2 * mf + 1][0], bfr[rf][0]);
                    dmma16x8x4(acc[2 * mf][rf][0], acc[2 * mf][rf][1], acc[2 * mf + 1][rf][0], acc[2 * mf + 1][rf][1],
                               a[2 * mf][1], a[2 * mf + 1][1], bfr[rf][1]);
                }
            }
        }
        // 5. the finished column block of L goes to shared M and to global memory
        for (int e = tid; e < NB * PB; e += 256) {
            const int r = e & (NB - 1), j = e >> 7;
            const double v = P[r * SP + j];
            M[r + (c0 + j) * LDM] = v;
            if (r >= c0 + j && r < jb && c0 + j < jb) A[r + (long long)(c0 + j) * lda] = v;
        }
        __syncthreads();
      }
    }

    CVXB_STAMP(2)
    // ---- inverse of L in shared memory ----
    // base: the 16 8x8 diagonal blocks, one per half-warp; lane (lane&15) < 8 owns column j
    {
        const int blk = warp * 2 + (lane >> 4);
        const int j = lane & 15;
        const int o = blk * PB;
        double x[PB];
        if (j < PB) {
#pragma unroll
            for (int i = 0; i < PB; ++i) {
                double v = (i == j) ? 1.0 : 0.0;
#pragma unroll
                for (int k = 0; k < i; ++k)
                    if (k >= j) v -= M[(o + i) + (o + k) * LDM] * x[k];
                x[i] = (i >= j) ? v / M[(o + i) + (o + i) * LDM] : 0.0;
            }
        }
        __syncwarp();
        if (j < PB) {
#pragma unroll
            for (int i = 0; i < PB; ++i) M[(o + i) + (o + j) * LDM] = x[i];
        }
    }
    __syncthreads();
    for (int s = PB; s < NB; s <<= 1) {
        const int sb = s / PB;                   // 8-blocks per side
        const int tp = sb * sb;                  // tiles per pair
        const int ntiles = (NB / (2 * s)) * tp;
        // phase 0: T = L21 * X11 -> stored in the (unused) upper block of the pair
        // phase 1: X21 = - X22 * T
        // each warp walks its tiles four at a time so four DMMA chains are in flight
#pragma unroll 1
        for (int phase = 0; phase < 2; ++phase) {
            for (int base = warp * 4; base < ntiles; base += 32) {
                double c[4][2];
                int oo[4], ti[4], tj[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int idx = min(base + u, ntiles - 1);
                    const int pr = idx / tp, loc = idx - pr * tp;
                    ti[u] = loc % sb; tj[u] = loc / sb; oo[u] = pr * 2 * s;
                    c[u][0] = c[u][1] = 0.0;
                }
                for (int kb = 0; kb < sb; ++kb) {
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        // X11 / X22 are lower triangular: skip the zero k blocks
                        const bool live = phase == 0 ? (kb >= tj[u]) : (kb <= ti[u]);
                        if (!live) continue;
                        const int o = oo[u];
#pragma unroll
                        for (int kk = 0; kk < 2; ++kk) {
                            const int k = kb * 8 + kk * 4 + t4;
                            double af, bf;
                            if (phase == 0) {
                                af = M[(o + s + ti[u] * 8 + g4) + (o + k) * LDM];
                                bf = M[(o + k) + (o + tj[u] * 8 + g4) * LDM];
                            } else {
                                af = M[(o + s + ti[u] * 8 + g4) + (o + s + k) * LDM];
                                bf = M[(o + k) + (o + s + tj[u] * 8 + g4) * LDM];
                            }
                            dmma(c[u][0], c[u][1], af, bf);
                        }
                    }
                }
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    if (base + u >= ntiles) continue;
                    const int o = oo[u];
                    if (phase == 0) {
                        M[(o + ti[u] * 8 + g4) + (o + s + tj[u] * 8 + t4 * 2) * LDM] = c[u][0];
                        M[(o + ti[u] * 8 + g4) + (o + s + tj[u] * 8 + t4 * 2 + 1) * LDM] = c[u][1];
                    } else {
                        M[(o + s + ti[u] * 8 + g4) + (o + tj[u] * 8 + t4 * 2) * LDM] = -c[u][0];
                        M[(o + s + ti[u] * 8 + g4) + (o + tj[u] * 8 + t4 * 2 + 1) * LDM] = -c[u][1];
                    }
                }
            }
            __syncthreads();
        }
    }
    CVXB_STAMP(3)
    for (int e = tid; e < NB * NB; e += 256) {
        int i = e & (NB - 1), k = e >> 7;
        inv[e] = (i >= k) ? M[i + k * LDM] : 0.0;
        invT[e] = (k >= i) ? M[k + i * LDM] : 0.0;     // invT[i + k*NB] = inv[k + i*NB]
    }
    if (trace && threadIdx.x == 0) {
        unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); trace[1] = t;
    }
}

// ---- blocked triangular solve with one right-hand side ------------------------
// forward:  L x = b ;  backward: L' x = b.   In place on b.  One CTA per 128-row block.
// flags[i] == epoch  <=>  x_i is final in b.
//
// Forward-progress assumption: CTA `bi` spins on the flags of the blocks it depends on, which are produced by
// CTAs with a SMALLER blockIdx.x (forward; the backward kernel reverses the block order so the same holds).  The
// hardware dispatches the CTAs of a grid in ascending linear block index, so a spinning CTA's producers are always
// resident or already finished; with at most ceil(n/128) CTAs per problem the whole grid is usually co-resident.
// CTA `bi` streams its block row (forward) / block column (backward) of L through a
// cp.async ring of 128x32 chunks that runs ahead of the dependency chain (L is static,
// only x arrives late), keeps inv(L_ii) in registers, and waits on the flag of block j
// only when it reaches that block's columns.  The critical path per block is then
// flag -> 128x128 smem GEMV -> 128x128 register GEMV -> flag.
constexpr int TR_CH = 32;                       // columns per ring chunk
constexpr int TR_R = 5;                         // ring depth
constexpr int TRSV_SMEM = (TR_R * NB * TR_CH + 4 * NB + 32 * 129) * 8;

template <bool TRANS, bool VEC>
__global__ void __launch_bounds__(256, 1)
trsv_kernel(int n, const double *__restrict__ L, long long ldl, const double *__restrict__ inv,
            const double *__restrict__ invT, double *b, int *flags, int epoch, long long sL,
            long long sInv, long long sb) {
    extern __shared__ __align__(16) double sm[];
    {   // batched: blockIdx.y selects the problem (blocks of one problem keep ascending order)
        const long long pb = blockIdx.y;
        L += pb * sL; inv += pb * sInv; invT += pb * sInv; b += pb * sb;
        flags += pb * ((n + NB - 1) / NB);
    }
    double *ring = sm;                          // TR_R x (32 cols x 128 rows), column-contiguous
    double *xs = ring + TR_R * NB * TR_CH;      // 128
    double *part = xs + NB;                     // 2 x 128
    double *tvec = part + 2 * NB;               // 128
    double *part2 = tvec + NB;                  // 32 x 129: per-lane column partials (backward)
    const int nblk = (n + NB - 1) / NB;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int bi = TRANS ? (nblk - 1 - (int)blockIdx.x) : (int)blockIdx.x;
    const int i0 = bi * NB;
    const int ni = min(NB, n - i0);
    const int r = tid & (NB - 1), half = tid >> 7;

    // inverse of the diagonal block -> registers (row r of inv, or row r of inv' for TRANS)
    double ireg[64];
    {
        const double *ip = (TRANS ? invT : inv) + (long long)bi * NB * NB + r + (long long)(half * 64) * NB;
#pragma unroll
        for (int k = 0; k < 64; ++k) ireg[k] = ip[k * NB];
    }

    // this block's right-hand side is input data nobody else writes: fetch it before the chain
    const double bown = (tid < ni) ? b[i0 + tid] : 0.0;
    const int nb_dep = TRANS ? (nblk - 1 - bi) : bi;         // blocks this CTA depends on
    const int nchunks = nb_dep * (NB / TR_CH);
    // chunk q -> (block j, column chunk cc)
    auto issue = [&](int q) {
        const int jj = q / (NB / TR_CH), cc = q % (NB / TR_CH);
        const int j = TRANS ? (nblk - 1 - jj) : jj;
        double *dst = ring + (q % TR_R) * (NB * TR_CH);
        const double *src;
        int nrows, ncols;
        if (!TRANS) { src = L + i0 + (long long)(j * NB + cc * TR_CH) * ldl; nrows = ni; ncols = TR_CH; }
        else { src = L + (long long)j * NB + (long long)(i0 + cc * TR_CH) * ldl; nrows = min(NB, n - j * NB); ncols = min(TR_CH, ni - cc * TR_CH); }
        if (VEC) {
#pragma unroll
            for (int it = 0; it < 8; ++it) {
                const int e = tid + it * 256;          // 2048 16-byte pieces
                const int c = e >> 6, rr = (e & 63) * 2;
                const int rem = nrows - rr;
                const int bytes = (c < ncols) ? (rem >= 2 ? 16 : (rem == 1 ? 8 : 0)) : 0;
                cp_async16(dst + c * NB + rr, bytes ? (src + rr + (long long)c * ldl) : L, bytes);
            }
        } else {
#pragma unroll
            for (int it = 0; it < 16; ++it) {
                const int e = tid + it * 256;
                const int c = e >> 7, rr = e & 127;
                const int bytes = (c < ncols && rr < nrows) ? 8 : 0;
                cp_async8(dst + c * NB + rr, bytes ? (src + rr + (long long)c * ldl) : L, bytes);
            }
        }
    };
#pragma unroll
    for (int q = 0; q < TR_R - 1; ++q) {
        if (q < nchunks) issue(q);
        cp_async_commit();
    }

    double acc = 0.0;           // forward: partial of row r over this thread's columns
    double accc[16];            // backward: per-lane partials of the warp's 16 columns
#pragma unroll
    for (int q = 0; q < 16; ++q) accc[q] = 0.0;

    for (int jj = 0; jj < nb_dep; ++jj) {
        const int j = TRANS ? (nblk - 1 - jj) : jj;
        if (tid == 0) while (ld_acquire(flags + j) != epoch) { }
        __syncthreads();
        if (tid < NB) xs[tid] = (j * NB + tid < n) ? __ldcg(b + j * NB + tid) : 0.0;
#pragma unroll
        for (int cc = 0; cc < NB / TR_CH; ++cc) {
            const int q = jj * (NB / TR_CH) + cc;
            cp_async_wait<TR_R - 2>();
            __syncthreads();
            {
                const int nq = q + TR_R - 1;
                if (nq < nchunks) issue(nq);
                cp_async_commit();
            }
            const double *ch = ring + (q % TR_R) * (NB * TR_CH);
            if (!TRANS) {
#pragma unroll
                for (int c = 0; c < 16; ++c)
                    acc += ch[(half * 16 + c) * NB + r] * xs[cc * TR_CH + half * 16 + c];
            } else {
                // warp w owns chunk columns w*4 .. w*4+3; lanes stride the 128 rows
#pragma unroll
                for (int qc = 0; qc < 4; ++qc) {
                    const double *col = ch + (warp * 4 + qc) * NB;
                    double a = 0.0;
#pragma unroll
                    for (int rr = 0; rr < 4; ++rr) a += col[lane + rr * 32] * xs[lane + rr * 32];
                    accc[cc * 4 + qc] += a;
                }
            }
        }
    }
    cp_async_wait<0>();
    __syncthreads();
    if (!TRANS) {
        part[half * NB + r] = acc;
        __syncthreads();
        if (tid < NB) tvec[tid] = (tid < ni) ? (bown - part[tid] - part[NB + tid]) : 0.0;
        __syncthreads();
    } else {
        // cross-lane reduction of the 16 column partials through shared memory (16 warp-shuffle
        // trees cost ~1.6 us on the critical path of every block step)
#pragma unroll
        for (int q = 0; q < 16; ++q) {
            const int c = (q >> 2) * TR_CH + warp * 4 + (q & 3);
            part2[lane * 129 + c] = accc[q];
        }
        __syncthreads();
        if (tid < NB) {
            double sacc = 0.0;
#pragma unroll 8
            for (int l = 0; l < 32; ++l) sacc += part2[l * 129 + tid];
            tvec[tid] = (tid < ni) ? (bown - sacc) : 0.0;
        }
        __syncthreads();
    }
    // x_i = inv_ii * t  (forward)  /  inv_ii' * t (backward): row r of the (transposed) inverse
    double a2 = 0.0;
#pragma unroll
    for (int k = 0; k < 64; ++k) a2 += ireg[k] * tvec[half * 64 + k];
    part[half * NB + r] = a2;
    __syncthreads();
    if (tid < ni) b[i0 + tid] = part[tid] + part[NB + tid];
    __threadfence();
    __syncthreads();
    if (tid == 0) st_release(flags + bi, epoch);
}

std::atomic<int> g_trsv_epoch{0};   // flags written by an earlier launch never equal a later epoch

// WT[k + r * ldt] = W[r + k * ldw] for r < rows, k < NB: a column-major panel to the K-major layout the TMA-fed
// update kernel reads.  32x32 tiles through shared memory, 32x8 threads.
__global__ void __launch_bounds__(256)
transpose_panel_kernel(const double *__restrict__ W, long long ldw, int rows, double *__restrict__ WT, long long ldt) {
    __shared__ double t[32][33];
    const int r0 = blockIdx.x * 32, k0 = blockIdx.y * 32, tx = threadIdx.x, ty = threadIdx.y;
#pragma unroll
    for (int i = ty; i < 32; i += 8)
        if (r0 + tx < rows) t[i][tx] = W[r0 + tx + (long long)(k0 + i) * ldw];
    __syncthreads();
#pragma unroll
    for (int i = ty; i < 32; i += 8)
        if (r0 + i < rows) WT[k0 + tx + (long long)(r0 + i) * ldt] = t[tx][i];
}

}  // namespace

int chol_work_create(CholWork &w) {
    int least = 0, greatest = 0;
    CVXB_CUDA(cudaDeviceGetStreamPriorityRange(&least, &greatest));
    CVXB_CUDA(cudaStreamCreateWithPriority(&w.panel_stream, cudaStreamNonBlocking, greatest));
    CVXB_CUDA(cudaStreamCreateWithPriority(&w.trsm_stream, cudaStreamNonBlocking, greatest));
    CVXB_CUDA(cudaStreamCreateWithPriority(&w.update_stream, cudaStreamNonBlocking, least));
    CVXB_CUDA(cudaStreamCreateWithPriority(&w.near_stream, cudaStreamNonBlocking, greatest));
    CVXB_CUDA(cudaEventCreateWithFlags(&w.ev_end_t, cudaEventDisableTiming));
    CVXB_CUDA(cudaEventCreateWithFlags(&w.ev_end_n, cudaEventDisableTiming));
    CVXB_CUDA(cudaEventCreateWithFlags(&w.ev_start, cudaEventDisableTiming));
    CVXB_CUDA(cudaEventCreateWithFlags(&w.ev_end_p, cudaEventDisableTiming));
    CVXB_CUDA(cudaEventCreateWithFlags(&w.ev_end_u, cudaEventDisableTiming));
    CVXB_TRY(w.d_info.alloc(1));
    CVXB_CUDA(cudaMemset(w.d_info.p, 0, sizeof(int)));
    CVXB_TRY(w.d_flags.alloc(4096));
    CVXB_CUDA(cudaMemset(w.d_flags.p, 0, 4096 * sizeof(int)));
    CVXB_TRY(w.splitk_ws.alloc(dmma_gemm_splitk_ws_doubles()));
    CVXB_CUDA(cudaFuncSetAttribute(potf2_inv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   POTF2_SMEM));
    CVXB_CUDA(cudaFuncSetAttribute(trsv_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, TRSV_SMEM));
    CVXB_CUDA(cudaFuncSetAttribute(trsv_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, TRSV_SMEM));
    CVXB_CUDA(cudaFuncSetAttribute(trsv_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, TRSV_SMEM));
    CVXB_CUDA(cudaFuncSetAttribute(trsv_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, TRSV_SMEM));
    return 0;
}

CholWork::~CholWork() {
    for (cudaStream_t s : {panel_stream, update_stream, trsm_stream, near_stream}) if (s) cudaStreamDestroy(s);
    for (auto &g : graphs) if (g.exec) cudaGraphExecDestroy(g.exec);
    for (cudaEvent_t e : {ev_end_t, ev_end_n, ev_start, ev_end_p, ev_end_u}) if (e) cudaEventDestroy(e);
    for (auto *v : {&ev_dg, &ev_tr, &ev_c0, &ev_na, &ev_nb, &ev_n})
        for (cudaEvent_t e : *v) cudaEventDestroy(e);
}

// Panels jb are grouped by q = jb / kGroup; group q's block columns are kGroup q .. kGroup q + kGroup - 1, and
// gq = kGroup (q + 1) is the first column of the next group.  Panel jb reaches block column c > jb exactly once:
//   c == jb + 1                       C0(jb)   on T  (K = 128, dmma_gemm_kernel)
//   jb + 2 <= c < gq                  Na(jb)   on N  near update inside the group (K = 128, dmma_gemm_kernel)
//   max(gq, jb + 2) <= c < gq + kGroup  Nb(jb)   on U  near update of the next group (K = 128, from the K-major copy)
//   c >= gq + kGroup                  F(q)     on U  far update, the whole group at once (K = kGroup * 128,
//                                                  syrk_tma_kernel), issued after the group's last panel
// (and the diagonal block (jb+1, jb+1) by the prologue of Dg(jb+1)).  F lags one group behind the chain: the
// columns of group q+1 get group q's panels from the small Nb updates, so the chain reaches F(q)'s first column
// only after factoring the whole of group q+1, while F(q) runs.
//
// Streams, per-step events:
//   D  (diag chain)   Dg(j): potf2_inv of block (j,j); for j>0 its prologue first applies panel j-1 to the block
//                     from the RAW tile A(j,j-1) and inv(j-1), so Dg(j-1) -> Dg(j) never waits for a full-width kernel.
//   T  (panel)        Tr(j): Wp = A(j+1:, j) inv(j)';  C0(j);  L(j:, j-1) copied from Wp back into A (after Dg(j)
//                     has consumed the raw tile).
//   N  (near)         Na(j), then the transpose of Wp's rows >= gq into slot j % kGroup of the group buffer.
//   U  (bulk)         Nb(j), and F(q) after Nb of the group's last panel.
// Ordering.  A writer of column c with panel p must follow every writer of c with a panel < p (read-modify-write of
// the same tiles); wait_col(s, c) orders stream s behind all updates of column c by panels <= c - 2, which is what
// Dg(c) (diagonal block, rows of the raw tile) and C0(c-1) need:
//   * Na(p) for p in c's group (p >= kGroup (c / kGroup)): N is in order, so ev_na[c-2] covers them;
//   * Nb(p) for p in the group before c's, and every F(q) with c >= its first column kGroup (q + 2): those F were
//     issued at steps <= kGroup (c / kGroup) - 5, so U runs them before Nb of the group before c's, and the wait
//     on ev_nb of the last such panel <= c - 2 covers both.  No wait is on an F that does not touch c, so the chain
//     never waits for the far update it is overlapping.
// The other orderings: Tr(j) rewrites panel[j & 1] after N's reads of step j-2 (ev_n[j-2]; the reads of T are in
// order).  Na(j) of a group's first panel follows Nb(j-1), which wrote the same columns (ev_nb[j-1]); the later
// Na of the group follow it on N.  Nb(j) follows the transpose (ev_n[j]) and, on U, F(q-1) (the previous panel's
// writer of its columns).  F(q) follows the group's transposes through Nb(j).  The group buffer of group q is
// rewritten by group q+2's transposes, each behind Tr -> Dg(c >= kGroup (q + 2)), which waited for an Nb queued
// after F(q).  Columns the chain leaves (c < j) are only read: the copy-back of L(j:, j-1) follows Dg(j) on T.
static int potrf_enqueue(int n, double *A, int lda, double *inv, CholWork &w, cudaStream_t st) {
    if (n <= 0) return 0;
    const int nblk = (n + NB - 1) / NB;
    if (w.panel_rows < n) {
        // captured graphs bake in the panel addresses and their leading dimension: drop them
        for (auto &g : w.graphs) if (g.exec) cudaGraphExecDestroy(g.exec);
        w.graphs.clear();
        for (DevBuf<double> &pb : w.panel) pb.reset();
        for (DevBuf<double> &gb : w.group) gb.reset();
        // two panel buffers (rows x NB): the TRSM result of step jb goes to panel[jb & 1], so it can be
        // written while the near updates of step jb-1 still read the other one; two group buffers
        // (kGroup NB x rows, K-major), group q's in group[q & 1] while the far update of group q-1 reads the other
        const int rows = (n + 1) & ~1;
        for (DevBuf<double> &pb : w.panel) CVXB_TRY(pb.alloc((size_t)rows * NB));
        for (DevBuf<double> &gb : w.group) CVXB_TRY(gb.alloc((size_t)rows * kGroup * NB));
        w.panel_rows = rows;
    }
    while ((int)w.ev_dg.size() < nblk) {
        cudaEvent_t e[6];
        for (int i = 0; i < 6; ++i) CVXB_CUDA(cudaEventCreateWithFlags(&e[i], cudaEventDisableTiming));
        w.ev_dg.push_back(e[0]); w.ev_tr.push_back(e[1]); w.ev_c0.push_back(e[2]);
        w.ev_na.push_back(e[3]); w.ev_nb.push_back(e[4]); w.ev_n.push_back(e[5]);
    }
    if (getenv("CVXB_TRACE") && !w.trace.p) CVXB_TRY(w.trace.alloc(8 * 4096));
    unsigned long long *trace = w.trace.p;
    if (trace) CVXB_CUDA(cudaMemsetAsync(trace, 0, 8 * 4096 * sizeof(unsigned long long), st));
    const int ldw = w.panel_rows;
    const int ldg = kGroup * NB;                             // leading dimension of a group buffer
    cudaStream_t D = w.panel_stream, T = w.trsm_stream, U = w.update_stream, N = w.near_stream;
    CVXB_CUDA(cudaMemsetAsync(w.d_info.p, 0, sizeof(int), st));
    CVXB_CUDA(cudaEventRecord(w.ev_start, st));
    for (cudaStream_t s : {D, T, U, N}) CVXB_CUDA(cudaStreamWaitEvent(s, w.ev_start, 0));
    // A22 -= X X' (lower) on block columns [lo, hi) and every row below, X = rows lo*NB.. of a K-wide panel
    auto update = [&](int lo, int hi, const double *X, int ldx, bool kmajor, int K, unsigned long long *tr,
                      cudaStream_t s) -> int {
        double *Acc = A + (long long)lo * NB * (1 + (long long)lda);
        GemmDesc u;
        u.M = n - lo * NB; u.N = (hi * NB < n ? hi * NB : n) - lo * NB; u.K = K;
        u.X = X; u.ldx = ldx; u.x_kmajor = kmajor;
        u.Y = X; u.ldy = ldx; u.y_kmajor = kmajor;
        u.D = Acc; u.ldd = lda; u.C = Acc; u.ldc = lda;
        u.alpha = -1.0; u.beta = 1.0; u.lower_only = true;
        u.trace = tr;
        return dmma_gemm(u, s);
    };
    auto wait_col = [&](cudaStream_t s, int c) -> int {
        const int p = c - 2, g0 = kGroup * (c / kGroup);
        if (p < 0) return 0;
        if (p >= g0) CVXB_CUDA(cudaStreamWaitEvent(s, w.ev_na[p], 0));
        if (g0 > 0) CVXB_CUDA(cudaStreamWaitEvent(s, w.ev_nb[p < g0 - 1 ? p : g0 - 1], 0));
        return 0;
    };
    for (int jb = 0; jb < nblk; ++jb) {
        const int j = jb * NB;
        const int wj = (n - j < NB) ? (n - j) : NB;
        const int m = n - j - wj;
        double *Ajj = A + j + (long long)j * lda;
        double *invj = inv + (long long)jb * NB * NB;
        double *invTj = inv + (long long)(nblk + jb) * NB * NB;
        double *Wp = w.panel[jb & 1].p;
        // ---- D: diagonal block.  Needs A(jb,jb) updated through panel jb-2 and the raw tile A(jb,jb-1)
        // (block column jb-1 complete through panel jb-2): C0(jb-2) and the updates of column jb.
        if (jb >= 2) CVXB_CUDA(cudaStreamWaitEvent(D, w.ev_c0[jb - 2], 0));
        CVXB_TRY(wait_col(D, jb));
        const double *Tprev = jb > 0 ? A + j + (long long)(j - NB) * lda : nullptr;
        const double *invprev = jb > 0 ? inv + (long long)(jb - 1) * NB * NB : nullptr;
        potf2_inv_kernel<<<1, 256, POTF2_SMEM, D>>>(Ajj, lda, wj, invj, invTj, w.d_info.p, j, 0, 0, Tprev,
                                                     lda, invprev, trace ? trace + 8 * jb : nullptr);
        count_launch();
        CVXB_LAUNCH_CHECK();
        CVXB_CUDA(cudaEventRecord(w.ev_dg[jb], D));
        // L(j:, j-1) goes back into A once Dg(jb) has consumed the raw tile; the copy rides on the
        // panel stream T behind this step's TRSM / column update
        auto copy_back_prev = [&]() -> int {
            if (jb == 0) return 0;
            const int jp = j - NB, mp = n - j;
            CVXB_CUDA(cudaMemcpy2DAsync(A + j + (long long)jp * lda, (size_t)lda * sizeof(double),
                                        w.panel[(jb - 1) & 1].p, (size_t)ldw * sizeof(double),
                                        (size_t)mp * sizeof(double), NB, cudaMemcpyDeviceToDevice, T));
            return 0;
        };
        if (m <= 0) {
            CVXB_CUDA(cudaStreamWaitEvent(T, w.ev_dg[jb], 0));
            CVXB_TRY(copy_back_prev());
            break;
        }
        double *A21 = Ajj + wj;
        double *A22 = A21 + (long long)wj * lda;
        // ---- T: panel TRSM as a GEMM with the block inverse (out of place) ----
        CVXB_CUDA(cudaStreamWaitEvent(T, w.ev_dg[jb], 0));
        // the panel buffer about to be overwritten was read on N two steps ago
        if (jb >= 2) CVXB_CUDA(cudaStreamWaitEvent(T, w.ev_n[jb - 2], 0));
        {
            GemmDesc g;
            g.M = m; g.N = wj; g.K = wj;
            g.X = A21; g.ldx = lda; g.x_kmajor = false;
            g.Y = invj; g.ldy = NB; g.y_kmajor = false;
            g.C = Wp; g.ldc = ldw;
            g.trace = trace ? trace + 8 * jb + 2 : nullptr;
            CVXB_TRY(dmma_gemm(g, T));
        }
        CVXB_CUDA(cudaEventRecord(w.ev_tr[jb], T));
        CVXB_TRY(wait_col(T, jb + 1));
        const int wn = (m < NB) ? m : NB;          // width of block column jb+1
        // ---- T: next block column, rows below its diagonal block ----
        if (m > wn) {
            GemmDesc c;
            c.M = m - wn; c.N = wn; c.K = wj;
            c.X = Wp + wn; c.Y = Wp;
            c.ldx = ldw; c.x_kmajor = false;
            c.ldy = ldw; c.y_kmajor = false;
            c.D = A22 + wn; c.ldd = lda; c.C = A22 + wn; c.ldc = lda;
            c.alpha = -1.0; c.beta = 1.0;
            c.trace = trace ? trace + 8 * jb + 4 : nullptr;
            CVXB_TRY(dmma_gemm(c, T));
        }
        CVXB_CUDA(cudaEventRecord(w.ev_c0[jb], T));
        CVXB_TRY(copy_back_prev());
        // ---- N: near update inside the group, then this panel's rows >= gq into the group buffer ----
        const int q = jb / kGroup, s = jb % kGroup, gq = kGroup * (q + 1);
        double *Wg = w.group[q & 1].p;
        unsigned long long *tr_near = trace ? trace + 8 * jb + 6 : nullptr;
        CVXB_CUDA(cudaStreamWaitEvent(N, w.ev_tr[jb], 0));
        if (s == 0 && jb > 0) CVXB_CUDA(cudaStreamWaitEvent(N, w.ev_nb[jb - 1], 0));
        {
            const int lo = jb + 2, hi = gq < nblk ? gq : nblk;
            if (lo < hi) CVXB_TRY(update(lo, hi, Wp + (lo - jb - 1) * NB, ldw, false, NB, tr_near, N));
        }
        CVXB_CUDA(cudaEventRecord(w.ev_na[jb], N));
        if (gq < nblk) {
            const int rows = n - gq * NB;
            transpose_panel_kernel<<<dim3((rows + 31) / 32, NB / 32), dim3(32, 8), 0, N>>>(
                Wp + (gq - jb - 1) * NB, ldw, rows, Wg + s * NB, ldg);
            count_launch();
            CVXB_LAUNCH_CHECK();
        }
        CVXB_CUDA(cudaEventRecord(w.ev_n[jb], N));
        // ---- U: near update of the next group's columns from the group buffer, and the far update ----
        if (gq < nblk) {
            CVXB_CUDA(cudaStreamWaitEvent(U, w.ev_n[jb], 0));
            const int lo = gq > jb + 2 ? gq : jb + 2, hi = gq + kGroup < nblk ? gq + kGroup : nblk;
            if (lo < hi) CVXB_TRY(update(lo, hi, Wg + s * NB + (long long)(lo - gq) * NB * ldg, ldg, true, NB, tr_near, U));
            CVXB_CUDA(cudaEventRecord(w.ev_nb[jb], U));
            if (s == kGroup - 1 && gq + kGroup < nblk)
                CVXB_TRY(update(gq + kGroup, nblk, Wg + (long long)kGroup * NB * ldg, ldg, true, kGroup * NB,
                                trace ? trace + 8 * 2048 + 8 * jb + 5 : nullptr, U));
        }
    }
    CVXB_CUDA(cudaEventRecord(w.ev_end_p, D));
    CVXB_CUDA(cudaEventRecord(w.ev_end_u, U));
    CVXB_CUDA(cudaEventRecord(w.ev_end_t, T));
    CVXB_CUDA(cudaEventRecord(w.ev_end_n, N));
    for (cudaEvent_t e : {w.ev_end_p, w.ev_end_u, w.ev_end_t, w.ev_end_n}) CVXB_CUDA(cudaStreamWaitEvent(st, e, 0));
    return 0;
}

// The ~450 launches / event operations of one factorisation are captured once per (n, A, lda,
// inv) into a CUDA graph (three-stream fork/join included) and replayed afterwards: dependent
// kernels then start without host-side launch latency, which is what the diagonal chain of
// small kernels is sensitive to.  First call with a new key runs eagerly (allocations, function
// attributes), the second one is captured; any capture failure falls back to eager launches.
int potrf_lower(int n, double *A, int lda, double *inv, CholWork &w, cudaStream_t st) {
    if (n <= 0) return 0;
    // replay removes ~450 host API calls per factorisation; large factorisations stay on the eager path because
    // graph kernel nodes do not keep the panel streams' priority over the bulk update (threshold chosen when the
    // kernels were tuned, not re-measured on H100)
    if (w.graph_failed || n > 4096) return potrf_enqueue(n, A, lda, inv, w, st);
    CholWork::GraphEntry *ent = nullptr;
    for (auto &g : w.graphs)
        if (g.n == n && g.A == A && g.lda == lda && g.inv == inv) { ent = &g; break; }
    if (ent && ent->exec) {
        CVXB_CUDA(cudaGraphLaunch(ent->exec, st));
        count_launch(ent->launches);
        return 0;
    }
    if (!ent) {                                        // first sight: eager, remember the key
        if (w.graphs.size() >= 4) {
            for (auto &g : w.graphs) if (g.exec) cudaGraphExecDestroy(g.exec);
            w.graphs.clear();
        }
        CholWork::GraphEntry g;
        g.n = n; g.A = A; g.lda = lda; g.inv = inv;
        w.graphs.push_back(g);
        return potrf_enqueue(n, A, lda, inv, w, st);
    }
    // second call with this key: capture
    const unsigned long long l0 = g_launches.load();
    if (cudaStreamBeginCapture(st, cudaStreamCaptureModeRelaxed) != cudaSuccess) {
        cudaGetLastError();
        w.graph_failed = true;
        return potrf_enqueue(n, A, lda, inv, w, st);
    }
    const int rc = potrf_enqueue(n, A, lda, inv, w, st);
    cudaGraph_t graph = nullptr;
    const cudaError_t ce = cudaStreamEndCapture(st, &graph);
    const int captured = (int)(g_launches.load() - l0);
    g_launches.fetch_sub((unsigned long long)captured);    // nothing has run yet
    if (rc != 0 || ce != cudaSuccess || !graph) {
        cudaGetLastError();
        if (graph) cudaGraphDestroy(graph);
        w.graph_failed = true;
        return potrf_enqueue(n, A, lda, inv, w, st);
    }
    cudaGraphExec_t exec = nullptr;
    if (cudaGraphInstantiate(&exec, graph, 0) != cudaSuccess || !exec) {
        cudaGetLastError();
        cudaGraphDestroy(graph);
        w.graph_failed = true;
        return potrf_enqueue(n, A, lda, inv, w, st);
    }
    cudaGraphDestroy(graph);
    ent->exec = exec;
    ent->launches = captured;
    CVXB_CUDA(cudaGraphLaunch(exec, st));
    count_launch(captured);
    return 0;
}

int trsv_lower(int n, const double *L, int ldl, const double *inv, double *b, bool trans,
               CholWork &w, cudaStream_t st, int batch, long long sL, long long sInv, long long sb) {
    if (n <= 0 || batch <= 0) return 0;
    const int nblk = (n + NB - 1) / NB;
    const size_t nflags = (size_t)nblk * batch;
    if (nflags > w.d_flags.n) {
        w.d_flags.reset();
        CVXB_TRY(w.d_flags.alloc(nflags));
        // on st: a plain cudaMemset runs on the legacy stream, which the non-blocking st does not wait for
        CVXB_CUDA(cudaMemsetAsync(w.d_flags.p, 0, nflags * sizeof(int), st));
    }
    const int epoch = g_trsv_epoch.fetch_add(1) + 1;
    const double *invT = inv + (long long)nblk * NB * NB;
    const bool vec = ((uintptr_t)L % 16 == 0) && (ldl % 2 == 0) && (batch == 1 || sL % 2 == 0);
    dim3 grid(nblk, batch);
#define TRSV_LAUNCH(T, V) trsv_kernel<T, V><<<grid, 256, TRSV_SMEM, st>>>(n, L, ldl, inv, invT, b, w.d_flags.p, epoch, sL, sInv, sb)
    if (trans) { if (vec) TRSV_LAUNCH(true, true); else TRSV_LAUNCH(true, false); }
    else       { if (vec) TRSV_LAUNCH(false, true); else TRSV_LAUNCH(false, false); }
#undef TRSV_LAUNCH
    count_launch();
    CVXB_LAUNCH_CHECK();
    return 0;
}

int potrs_lower(int n, const double *L, int ldl, const double *inv, double *b, CholWork &w,
                cudaStream_t st, int batch, long long sL, long long sInv, long long sb) {
    CVXB_TRY(trsv_lower(n, L, ldl, inv, b, false, w, st, batch, sL, sInv, sb));
    CVXB_TRY(trsv_lower(n, L, ldl, inv, b, true, w, st, batch, sL, sInv, sb));
    return 0;
}

namespace {
__global__ void copy2d_batched_kernel(const double *src, long long lds, long long ssrc, double *dst,
                                      long long ldd, long long sdst, int rows, int cols) {
    const long long pb = blockIdx.z;
    const int r = blockIdx.x * blockDim.x + threadIdx.x, c = blockIdx.y;
    if (r < rows && c < cols) dst[pb * sdst + r + (long long)c * ldd] = src[pb * ssrc + r + (long long)c * lds];
}
}  // namespace

// Batched Cholesky of `batch` independent n x n matrices (stride sA, inverse blocks stride
// sInv).  The batch itself fills the machine, so the steps run back to back on one stream
// (no look-ahead).  d_info: one int per problem.  panel: batch * ldw * NB doubles.
int potrf_lower_batched(int n, double *A, int lda, long long sA, double *inv, long long sInv,
                        int batch, int *d_info, double *panel, int ldw, cudaStream_t st) {
    if (n <= 0 || batch <= 0) return 0;
    const int nblk = (n + NB - 1) / NB;
    CVXB_CUDA(cudaMemsetAsync(d_info, 0, (size_t)batch * sizeof(int), st));
    const long long sW = (long long)ldw * NB;
    for (int jb = 0; jb < nblk; ++jb) {
        const int j = jb * NB;
        const int wj = (n - j < NB) ? (n - j) : NB;
        const int m = n - j - wj;
        double *Ajj = A + j + (long long)j * lda;
        double *invj = inv + (long long)jb * NB * NB;
        double *invTj = inv + (long long)(nblk + jb) * NB * NB;
        potf2_inv_kernel<<<batch, 256, POTF2_SMEM, st>>>(Ajj, lda, wj, invj, invTj, d_info, j, sA, sInv, nullptr, 0,
                                                        nullptr, nullptr);
        count_launch();
        CVXB_LAUNCH_CHECK();
        if (m <= 0) break;
        double *A21 = Ajj + wj;
        double *A22 = A21 + (long long)wj * lda;
        GemmDesc g;
        g.M = m; g.N = wj; g.K = wj;
        g.X = A21; g.ldx = lda; g.x_kmajor = false; g.sX = sA;
        g.Y = invj; g.ldy = NB; g.y_kmajor = false; g.sY = sInv;
        g.C = panel; g.ldc = ldw; g.sC = sW; g.batch = batch;
        CVXB_TRY(dmma_gemm(g, st));
        GemmDesc u;
        u.M = m; u.N = m; u.K = wj;
        u.X = panel; u.ldx = ldw; u.x_kmajor = false; u.sX = sW;
        u.Y = panel; u.ldy = ldw; u.y_kmajor = false; u.sY = sW;
        u.D = A22; u.ldd = lda; u.sD = sA; u.C = A22; u.ldc = lda; u.sC = sA;
        u.alpha = -1.0; u.beta = 1.0; u.lower_only = true; u.batch = batch;
        CVXB_TRY(dmma_gemm(u, st));
        dim3 cg((m + 255) / 256, wj, batch);
        copy2d_batched_kernel<<<cg, 256, 0, st>>>(panel, ldw, sW, A21, lda, sA, m, wj);
        count_launch();
        CVXB_LAUNCH_CHECK();
    }
    return 0;
}

}  // namespace cvxb
