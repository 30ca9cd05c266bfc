// fp64 tensor-core GEMM/SYRK for sm_90a.
//
//   C[r,c] = alpha * sum_k X[r,k] * w[k] * Y[c,k] + beta * D[r,c]
//
// This one kernel is the flop carrier of the whole KKT path:
//   * normal-equations assembly  K = H + G' diag(di^2) G        (X=Y=G, K-major, w=di^2,
//     lower tiles only; replaces scale(Gs)+blas.syrk+`K += H`,   reference misc.py:1268-1276)
//   * Cholesky panel TRSM  L21 = A21 * L11^{-T}                  (X=A21, Y=inv(L11), M-major)
//   * Cholesky next-column and in-group near updates A22 -= L21 L21'  (X=Y=L21, M-major, lower, K = 128)
//   * the 's'-cone congruences r' X r                            (batched general GEMMs)
//
// wgmma has no fp64 form, so the fp64 tensor path is warp-level mma.sync.  sm_90 runs the
// 16x8 shapes (DMMA.16x8x4/8/16) at 256 flop/clk/SM, the data-sheet 67 TF/s at 1.98 GHz, and
// the Ampere shape DMMA.8x8x4 at half that (tools/dmma_rate), so the kernel issues
// m16n8k4 (dmma16x8x4): same fragments as two m8n8k4, half the instructions.
// A 128x64x16 tile step moves 24 KB for 131072 FMAs, so operand traffic is small next to
// the tensor work; the design goal is to keep the DMMA pipe issuing:
//   * 128-thread CTAs (4 warps, 64x32 warp tiles, 64 accumulator doubles / thread),
//     TWO CTAs per SM so one CTA's barrier / prologue / epilogue bubbles are covered
//     by the other CTA's DMMAs
//   * 3-stage cp.async pipeline, padded shared-memory layouts that make every
//     fragment LDS.64 bank-conflict free
//   * fragments double-buffered in registers so the di^2 scaling DMULs of step kk+1
//     issue before the DMMAs of step kk (no DMUL->DMMA dependency stall)
//   * per-thread copy descriptors hoisted out of the k loop
//
// Single K-major lower-triangle SYRKs with 16-byte aligned operands and even leading dimensions (the KKT
// normal equations, A'A, Asct'Asct, cvxb_syrk_scaled, and the Cholesky's updates from its K-major group buffer: the
// far updates at K = 512 and the near updates of the next group at K = 128) run on syrk_tma_kernel instead: 128x128 tiles, one
// CTA per SM, operands fed by TMA through an mbarrier ring by a producer warpgroup (see its comment).  It keeps
// this kernel's warp tiles, fragments and k order, so the two agree bit for bit outside the split-K tail.
//
// MMA roles are swapped w.r.t. the matrix: the MMA "m" index runs over C's columns
// (Y operand), the "n" index over C's rows (X operand), so each thread's accumulator
// pair is two consecutive ROWS of a column-major C (one 16-byte access).  One m16n8k4
// covers the column fragments cf = 2mf and 2mf+1 (8 columns apart) of a row fragment.
#include "common.cuh"
#include <cuda.h>
#include <cudaTypedefs.h>

namespace cvxb {

namespace {

constexpr int BR = 128, BC = 64, BK = 16, STAGES = 3;
constexpr int THREADS = 128;
constexpr int SK = BK + 4;            // row stride (doubles) of a K-major operand tile  [idx][k]
constexpr int SMX = BR + 4;           // row stride of an M-major X tile [k][idx]  (132 = 4 mod 16)
constexpr int SMY = BC + 4;           // row stride of an M-major Y tile [k][idx]  (68  = 4 mod 16)
constexpr int X_STAGE = BR * SK;      // 2560 doubles >= 16*132
constexpr int Y_STAGE = BC * SK;      // 1280 doubles >= 16*68
constexpr int STAGE_DOUBLES = X_STAGE + Y_STAGE + BK;
constexpr int SMEM_BYTES = STAGES * STAGE_DOUBLES * 8;      // 92544 B -> 2 CTAs / SM
constexpr int TILE_ELEMS = BR * BC;
constexpr int CTAS_PER_WAVE = 2 * kNumSMs;
constexpr int SPLITK_WS_TILES = 4 * CTAS_PER_WAVE;   // split-K workspace capacity (tiles)

struct KParams {
    int M, N, K;
    const double *X; long long ldx;
    const double *Y; long long ldy;
    const double *w;
    const double *D; long long ldd;
    double *C; long long ldc;
    double alpha, beta;
    int lower_only;
    int ct_begin, ct_end;   // c-tile window in units of BC columns (already clipped)
    int nTr;                // number of r tiles
    long long sX, sY, sW, sD, sC;
    int full_tiles;         // units [0, full_tiles) are whole tiles
    int S;                  // splits per remainder tile (1 = none)
    int kchunk;             // K elements per split (multiple of BK)
    double *ws;
    int vec_c;              // C/D allow 16-byte accesses
    int stagger_ns;         // > 0: short-K launch, offset the second CTA of each SM by this much
    unsigned long long *trace;
    int band;               // > 0: band-major tile order (lower_only, long K), width in c tiles
};

// first r tile that intersects the lower triangle for c tile `tc` of width `tcols`
__device__ __host__ __forceinline__ int first_tr(int tc, int tcols) { return (tc * tcols) / BR; }

// unit t -> (r tile, c tile) for c tiles TC columns wide
template <int TC>
__device__ __forceinline__ void decode_tile(const KParams &p, int t, int &tr, int &tc) {
    int c = p.ct_begin;
    if (p.lower_only && p.band > 0) {
        // L2-friendly order for long-K launches: c tiles are grouped in bands of `band` columns
        // and a band is walked row tile by row tile, so the CTAs that run together share a
        // near-square set of operand panels (r01d: 11.3 GB of DRAM traffic for 1.6 GB of
        // operands with the column-major order, where every wave streams all of G).
        int cb_end;
        while (true) {
            cb_end = min(c + p.band, p.ct_end);
            int cnt = 0;
            for (int cc = c; cc < cb_end; ++cc) cnt += max(0, p.nTr - first_tr(cc, TC));
            if (t < cnt) break;
            t -= cnt;
            c = cb_end;
        }
        for (int r = first_tr(c, TC);; ++r) {
            const int cmax = min(cb_end - 1, (r * BR + BR - 1) / TC);   // last live c tile of this row
            const int cntr = cmax - c + 1;
            if (t < cntr) { tr = r; tc = c + t; return; }
            t -= cntr;
        }
    }
    if (p.lower_only) {
        while (true) {
            int cnt = p.nTr - first_tr(c, TC);
            if (t < cnt) break;
            t -= cnt;
            ++c;
        }
        tr = first_tr(c, TC) + t;
        tc = c;
    } else {
        tc = c + t / p.nTr;
        tr = t % p.nTr;
    }
}

// A thread's share of one operand tile copy.  Piece i of a thread sits at a fixed stride
// from piece 0 (rows advance for a K-major tile, k advances for an M-major tile), so the
// plan is a base pointer, a stride and two small integers; K advances by a pointer offset.
template <bool KMAJOR, bool VEC, int ROWS>
struct CopyPlan {
    static constexpr int W = VEC ? 2 : 1;                         // doubles per piece
    static constexpr int PER = KMAJOR ? BK / W : ROWS / W;        // pieces per row / per k
    static constexpr int NP = ROWS * BK / W / THREADS;            // pieces per thread
    static constexpr int DSTEP = THREADS / PER;                   // row (or k) step between pieces
    static constexpr int STRIDE_M = ROWS + 4;
    static constexpr int SSTEP = DSTEP * (KMAJOR ? SK : STRIDE_M);
    const double *g0;
    long long gstep;
    int s0, idx0, k0, cbytes;

    __device__ __forceinline__ void init(const double *src, long long ld, int nrows, int tid) {
        const int a = tid / PER, bq = (tid % PER) * W;
        if (KMAJOR) {
            idx0 = a; k0 = bq;
            g0 = src + k0 + (long long)idx0 * ld;
            s0 = idx0 * SK + k0;
            cbytes = 8 * W;                                        // k validity of a full tile
        } else {
            k0 = a; idx0 = bq;
            g0 = src + idx0 + (long long)k0 * ld;
            s0 = k0 * STRIDE_M + idx0;
            const int rem = nrows - idx0;
            cbytes = rem >= W ? 8 * W : (rem > 0 ? 8 * rem : 0);   // row validity (constant)
        }
        gstep = (long long)DSTEP * ld;
    }
    __device__ __forceinline__ void issue(double *sbase, const double *base, long long goff,
                                          int nrows, int kvalid) const {
        const double *g = g0 + goff;
        int kb = cbytes;
        if (KMAJOR && kvalid < BK) {                               // k tail (last tile only)
            const int rem = kvalid - k0;
            kb = rem >= W ? 8 * W : (rem > 0 ? 8 * rem : 0);
        }
#pragma unroll
        for (int i = 0; i < NP; ++i) {
            int bytes;
            if (KMAJOR) bytes = (idx0 + i * DSTEP < nrows) ? kb : 0;
            else        bytes = (k0 + i * DSTEP < kvalid) ? kb : 0;
            const double *gp = bytes ? g : base;
            if (VEC) cp_async16(sbase + s0 + i * SSTEP, gp, bytes);
            else     cp_async8(sbase + s0 + i * SSTEP, gp, bytes);
            g += gstep;
        }
    }
};

template <bool XK, bool YK, bool VEC>
__global__ void __launch_bounds__(THREADS, 2) dmma_gemm_kernel(const KParams p) {
    extern __shared__ __align__(16) double smem[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wr = warp & 1, wc = warp >> 1;
    const int g4 = lane >> 2, t4 = lane & 3;

    if (p.trace && tid == 0) {
        unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        atomicCAS(p.trace, 0ULL, t);   // first CTA to start
    }
    // ---- which unit am I? ----
    const int u = blockIdx.x;
    int tile, split = 0;
    if (u < p.full_tiles) {
        tile = u;
    } else {
        tile = p.full_tiles + (u - p.full_tiles) / p.S;
        split = (u - p.full_tiles) % p.S;
    }
    int tr, tc;
    decode_tile<BC>(p, tile, tr, tc);
    const bool is_split = (u >= p.full_tiles) && (p.S > 1);
    int kbeg = 0, kend = p.K;
    if (is_split) {
        kbeg = split * p.kchunk;
        kend = min(p.K, kbeg + p.kchunk);
    }
    const int r0 = tr * BR, c0 = tc * BC;
    const int nr = min(BR, p.M - r0), nc = min(BC, p.N - c0);

    const long long b = blockIdx.z;
    const double *X = p.X + b * p.sX;
    const double *Y = p.Y + b * p.sY;
    const double *w = p.w ? p.w + b * p.sW : nullptr;
    const bool has_w = (w != nullptr);

    // tile origins at k = kbeg
    const double *Xt = XK ? X + (long long)r0 * p.ldx + kbeg : X + r0 + (long long)kbeg * p.ldx;
    const double *Yt = YK ? Y + (long long)c0 * p.ldy + kbeg : Y + c0 + (long long)kbeg * p.ldy;
    const long long xstep = XK ? BK : (long long)BK * p.ldx;     // pointer advance per k tile
    const long long ystep = YK ? BK : (long long)BK * p.ldy;

    CopyPlan<XK, VEC, BR> px;
    CopyPlan<YK, VEC, BC> py;
    px.init(Xt, p.ldx, nr, tid);
    py.init(Yt, p.ldy, nc, tid);

    // Short-K launches (Cholesky trailing updates, K = 128): a tile's prologue/epilogue is as
    // long as half its main loop, and the two CTAs that share an SM start together and stay in
    // lock-step, so nothing overlaps (r01e profile: DMMA pipe 63 % busy).  (1) pull the D tile
    // towards L2 now, so the epilogue's read-modify-write does not pay DRAM latency four times;
    // (2) hold back the second CTA of every SM by half a tile so that one CTA's epilogue and
    // prologue run under the other's DMMAs from then on.
    if (p.stagger_ns > 0) {
        if (p.beta != 0.0 && p.D != nullptr && !is_split) {
            const double *Dt = p.D + b * p.sD + r0 + (long long)c0 * p.ldd;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int line = tid * 4 + i;               // 512 lines of 128 B in a 128x64 tile
                const int col = line >> 3, seg = line & 7;
                if (col < nc && seg * 16 < nr)
                    asm volatile("prefetch.global.L2 [%0];" ::"l"(Dt + seg * 16 + (long long)col * p.ldd));
            }
        }
        if (blockIdx.x >= (unsigned)kNumSMs && blockIdx.x < (unsigned)(2 * kNumSMs)) {
            unsigned long long t0, t1;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
            do {
                __nanosleep(256);
                asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
            } while (t1 - t0 < (unsigned long long)p.stagger_ns);
        }
    }

    double acc[4][8][2];
    // Read-modify-write launches with alpha = +-1 (the Cholesky trailing updates: C = D - X Y'): full interior tiles
    // start their accumulators from (beta/alpha) * D, loaded here straight into the fragment layout, so the loads
    // complete under the main loop and the epilogue is stores only.  (Staging D through shared memory after the main
    // loop cost a barrier, a 64 KB cp.async burst and its latency per tile: ~2 us of a ~10 us tile at K = 128.)
    const bool pre_d = p.vec_c && (nr == BR) && (nc == BC) && !(p.lower_only && (c0 + BC - 1 > r0)) && !is_split &&
                       p.beta != 0.0 && p.D != nullptr && (p.alpha == 1.0 || p.alpha == -1.0) && ((p.ldd & 1) == 0);
    if (pre_d) {
        const double sc = p.beta / p.alpha;
        const double *Dt = p.D + b * p.sD + r0 + (long long)c0 * p.ldd;
#pragma unroll
        for (int cf = 0; cf < 4; ++cf) {
            const int cl = wc * 32 + cf * 8 + g4;
#pragma unroll
            for (int rf = 0; rf < 8; ++rf) {
                const int rl = wr * 64 + rf * 8 + t4 * 2;
                const double2 dv = *reinterpret_cast<const double2 *>(Dt + rl + (long long)cl * p.ldd);
                acc[cf][rf][0] = sc * dv.x; acc[cf][rf][1] = sc * dv.y;
            }
        }
    } else {
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;
    }

    const int ktiles = (kend - kbeg + BK - 1) / BK;
    // lower-triangular outputs: a warp whose whole block is above the diagonal only helps with the
    // copies (matters for small n / batched SYRKs where a quarter of the tiles straddle the diagonal)
    const bool warp_idle = p.lower_only && (r0 + wr * 64 + 63 < c0 + wc * 32);

    auto load_stage = [&](int kt, int stage) {
        double *sx = smem + stage * STAGE_DOUBLES;
        double *sy = sx + X_STAGE;
        double *sw = sy + Y_STAGE;
        const int kvalid = min(BK, kend - kbeg - kt * BK);
        px.issue(sx, X, (long long)kt * xstep, nr, kvalid);
        py.issue(sy, Y, (long long)kt * ystep, nc, kvalid);
        if (has_w && tid < BK) {
            const int bytes = (tid < kvalid) ? 8 : 0;
            cp_async8(sw + tid, bytes ? (w + kbeg + kt * BK + tid) : w, bytes);
        }
    };

#pragma unroll
    for (int s = 0; s < STAGES - 1; ++s) {
        if (s < ktiles) load_stage(s, s);
        cp_async_commit();
    }

    // fragment offsets (doubles) inside a stage, for k = t4
    int xoff[8], yoff[4];
#pragma unroll
    for (int rf = 0; rf < 8; ++rf) {
        const int idx = wr * 64 + rf * 8 + g4;
        xoff[rf] = XK ? idx * SK + t4 : t4 * SMX + idx;
    }
#pragma unroll
    for (int cf = 0; cf < 4; ++cf) {
        const int idx = wc * 32 + cf * 8 + g4;
        yoff[cf] = X_STAGE + (YK ? idx * SK + t4 : t4 * SMY + idx);
    }
    constexpr int XKK = XK ? 4 : 4 * SMX;       // offset advance per kk step (4 k values)
    constexpr int YKK = YK ? 4 : 4 * SMY;

    for (int kt = 0; kt < ktiles; ++kt) {
        cp_async_wait<STAGES - 2>();
        __syncthreads();
        const double *st = smem + (kt % STAGES) * STAGE_DOUBLES;
        if (warp_idle) {            // this warp's 64x32 block lies strictly above the diagonal
            const int nk = kt + STAGES - 1;
            if (nk < ktiles) load_stage(nk, nk % STAGES);
            cp_async_commit();
            continue;
        }
        // fragments of kk = 0 first, so their latency overlaps the prefetch issue below
        double a[2][4], bf[2][8];
#pragma unroll
        for (int cf = 0; cf < 4; ++cf) a[0][cf] = st[yoff[cf]];
#pragma unroll
        for (int rf = 0; rf < 8; ++rf) bf[0][rf] = st[xoff[rf]];
        double wv = 1.0;
        if (has_w) wv = st[X_STAGE + Y_STAGE + t4];
        {
            const int nk = kt + STAGES - 1;
            if (nk < ktiles) load_stage(nk, nk % STAGES);
            cp_async_commit();
        }
        if (has_w) {
#pragma unroll
            for (int cf = 0; cf < 4; ++cf) a[0][cf] *= wv;
        }
#pragma unroll
        for (int kk = 0; kk < BK / 4; ++kk) {
            const int cur = kk & 1, nxt = cur ^ 1;
            if (kk + 1 < BK / 4) {
#pragma unroll
                for (int cf = 0; cf < 4; ++cf) a[nxt][cf] = st[yoff[cf] + (kk + 1) * YKK];
#pragma unroll
                for (int rf = 0; rf < 8; ++rf) bf[nxt][rf] = st[xoff[rf] + (kk + 1) * XKK];
                if (has_w) {
                    const double wn = st[X_STAGE + Y_STAGE + (kk + 1) * 4 + t4];
#pragma unroll
                    for (int cf = 0; cf < 4; ++cf) a[nxt][cf] *= wn;
                }
            }
#pragma unroll
            for (int mf = 0; mf < 2; ++mf)
#pragma unroll
                for (int rf = 0; rf < 8; ++rf)
                    dmma16x8x4(acc[2 * mf][rf][0], acc[2 * mf][rf][1], acc[2 * mf + 1][rf][0],
                               acc[2 * mf + 1][rf][1], a[cur][2 * mf], a[cur][2 * mf + 1], bf[cur][rf]);
        }
    }
    cp_async_wait<0>();

    // ---- epilogue ----
    if (is_split) {
        double *ws = p.ws + ((long long)(tile - p.full_tiles) * p.S + split) * TILE_ELEMS;
#pragma unroll
        for (int cf = 0; cf < 4; ++cf)
#pragma unroll
            for (int rf = 0; rf < 8; ++rf) {
                const int rl = wr * 64 + rf * 8 + t4 * 2;
                const int cl = wc * 32 + cf * 8 + g4;
                *reinterpret_cast<double2 *>(ws + rl + cl * BR) =
                    make_double2(acc[cf][rf][0], acc[cf][rf][1]);
            }
        return;
    }
    struct TraceEnd {
        unsigned long long *tr; int tid;
        __device__ ~TraceEnd() {
            if (tr && tid == 0) {
                unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
                atomicMax(tr + 1, t);
            }
        }
    } trace_end{p.trace, tid};
    double *C = p.C + b * p.sC;
    const double *D = p.D ? p.D + b * p.sD : nullptr;
    const bool diag = p.lower_only && (c0 + BC - 1 > r0);       // tile touches the diagonal
    const bool use_d = (p.beta != 0.0);
    const bool fast = p.vec_c && (nr == BR) && (nc == BC) && !diag;
    if (fast) {
        // full interior tile, 16-byte accesses
        if (pre_d) {
#pragma unroll
            for (int cf = 0; cf < 4; ++cf) {
                const long long c = c0 + wc * 32 + cf * 8 + g4;
#pragma unroll
                for (int rf = 0; rf < 8; ++rf) {
                    double2 v = make_double2(p.alpha * acc[cf][rf][0], p.alpha * acc[cf][rf][1]);
                    *reinterpret_cast<double2 *>(C + (r0 + wr * 64 + rf * 8 + t4 * 2) + c * p.ldc) = v;
                }
            }
            return;
        }
        if (use_d) {
            // read-modify-write epilogue: stage the whole D tile through the (now idle) pipeline
            // buffers with one burst of cp.async — a single memory round trip with coalesced
            // 1 KB column segments, instead of four dependent rounds of fragment-pattern loads
            constexpr int LDT = BR + 8;                     // 136: conflict-free 16-byte fragment reads
            static_assert(BC * LDT <= STAGES * STAGE_DOUBLES, "D tile must fit in the stage buffers");
            __syncthreads();                                // every warp is done with the stages
            const double *Dt = D + r0 + (long long)c0 * p.ldd;
#pragma unroll 8
            for (int i = 0; i < (BR * BC / 2) / THREADS; ++i) {
                const int q = tid + i * THREADS;            // 16-byte piece index
                const int col = q >> 6, rr = (q & 63) * 2;
                cp_async16(smem + col * LDT + rr, Dt + rr + (long long)col * p.ldd, 16);
            }
            cp_async_commit();
            cp_async_wait<0>();
            __syncthreads();
#pragma unroll
            for (int cf = 0; cf < 4; ++cf) {
                const int cl = wc * 32 + cf * 8 + g4;
#pragma unroll
                for (int rf = 0; rf < 8; ++rf) {
                    const int rl = wr * 64 + rf * 8 + t4 * 2;
                    const double2 dv = *reinterpret_cast<const double2 *>(smem + cl * LDT + rl);
                    double2 v = make_double2(p.alpha * acc[cf][rf][0] + p.beta * dv.x,
                                             p.alpha * acc[cf][rf][1] + p.beta * dv.y);
                    *reinterpret_cast<double2 *>(C + (r0 + rl) + (long long)(c0 + cl) * p.ldc) = v;
                }
            }
            return;
        }
#pragma unroll
        for (int cf = 0; cf < 4; ++cf) {
            const long long c = c0 + wc * 32 + cf * 8 + g4;
#pragma unroll
            for (int rf = 0; rf < 8; ++rf) {
                double2 v = make_double2(p.alpha * acc[cf][rf][0], p.alpha * acc[cf][rf][1]);
                *reinterpret_cast<double2 *>(C + (r0 + wr * 64 + rf * 8 + t4 * 2) + c * p.ldc) = v;
            }
        }
        return;
    }
    // edge / diagonal tiles: the 16 values of D a thread needs per column fragment are loaded as one batch
    // (C may alias D, so a load after a store cannot be hoisted: element-by-element this was 64 dependent round trips)
#pragma unroll
    for (int cf = 0; cf < 4; ++cf) {
        const int cl = wc * 32 + cf * 8 + g4;
        if (cl >= nc) continue;
        const long long c = c0 + cl;
        double dv[8][2];
#pragma unroll
        for (int rf = 0; rf < 8; ++rf) {
            const int rl = wr * 64 + rf * 8 + t4 * 2;
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const long long r = r0 + rl + e;
                const bool ok = use_d && (rl + e < nr) && !(diag && r < c);
                dv[rf][e] = ok ? D[r + c * p.ldd] : 0.0;
            }
        }
#pragma unroll
        for (int rf = 0; rf < 8; ++rf) {
            const int rl = wr * 64 + rf * 8 + t4 * 2;
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                if (rl + e >= nr) continue;
                const long long r = r0 + rl + e;
                if (diag && r < c) continue;
                double v = p.alpha * acc[cf][rf][e];
                if (use_d) v += p.beta * dv[rf][e];
                C[r + c * p.ldc] = v;
            }
        }
    }
}

// ---- K-major lower-triangle SYRK on 128x128 tiles: TMA-fed, warp-specialised ----
// One CTA per SM owns a 128x128 tile of C: warps 0-7 are the 2x4 grid of 64x32 warp tiles of dmma_gemm_kernel
// (same fragments, same k order, w applied to the column fragments, same pre_d start), so every element outside
// the split-K tail is bit-identical to the 128x64 kernel's; warps 8-11 are the producer warpgroup, which hands
// its registers to the consumers (setmaxnreg: 64 accumulators and two fragment sets per consumer thread do not fit
// the 168 registers a 9-warp CTA gets, because one SM sub-partition holds 3 of its warps).  Per 16-wide k tile it
// issues one 2D TMA box {16 k, 128 rows} per operand and a 1D box of w into a T_STAGES-deep mbarrier ring;
// consumers release a stage through its empty barrier, so the main loop has no CTA-wide barrier, and TMA's zero
// fill outside the tensor replaces CopyPlan's row and k-tail masking.  A 128x128 tile moves 256 operand rows
// per k for 2*128*128 flop (16 flop/B against 10.7 for 128x64), so a SYRK reads a third less from L2.
//
// Shared-memory map of an operand panel (128-byte swizzle): row r (a tile row of X, or column of Y) is 128 bytes
// = its 16 k values, and the 16-byte chunk c = k/2 of row r sits at chunk c ^ (r & 7).  A fragment load of one
// warp reads rows idx = 8j + g4 (g4 = lane/4) at k = 4kk + t4 (t4 = lane%4): lanes t4 < 2 read chunk 2kk and
// lanes t4 >= 2 chunk 2kk+1, which the eight g4 spread over all eight chunk positions, so each half-warp is
// one 128-byte wavefront (2 per load, the minimum for 256 bytes).  The double offset is
//   16 idx + 4 (kk ^ (g4 >> 1)) + 2 ((t4 >> 1) ^ (g4 & 1)) + (t4 & 1).
constexpr int TB = 128;                                  // tile edge (rows and columns of C)
constexpr int T_STAGES = 6;
constexpr int T_CONSUMERS = 8;                           // 2 x 4 warps of 64 x 32
constexpr int T_THREADS = 32 * (T_CONSUMERS + 4);        // + the producer warpgroup
constexpr int T_REGS_PRODUCER = 40, T_REGS_CONSUMER = 232;   // 128 * 40 + 256 * 232 <= 65536
constexpr int T_PANEL = TB * BK;                         // doubles of one operand panel (16 KB)
constexpr int T_SMEM = T_STAGES * (2 * T_PANEL + BK) * 8 + 2 * T_STAGES * 8 + 1024;   // + barriers, alignment
constexpr int T_TILE_ELEMS = TB * TB;
constexpr int T_WS_TILES = 4 * kNumSMs;                  // split-K workspace capacity (tiles)

__global__ void __launch_bounds__(T_THREADS, 1)
syrk_tma_kernel(const KParams p, const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmY,
                const __grid_constant__ CUtensorMap tmW) {
    extern __shared__ unsigned char t_smem_raw[];
    // 1024-byte aligned (the 128-byte swizzle repeats every 8 rows); offset from the array so that the compiler
    // keeps shared-memory loads
    double *sm = reinterpret_cast<double *>(t_smem_raw + ((1024u - (smem_u32(t_smem_raw) & 1023u)) & 1023u));
    double *sw = sm + T_STAGES * 2 * T_PANEL;            // w of stage s at sw + s * BK
    uint64_t *full = reinterpret_cast<uint64_t *>(sw + T_STAGES * BK), *empty = full + T_STAGES;
    // warp index through a shuffle, so the compiler knows the role branches are warp-uniform
    const int tid = threadIdx.x, warp = __shfl_sync(0xffffffffu, tid >> 5, 0), lane = tid & 31;

    const int u = blockIdx.x;
    int tile, split = 0;
    if (u < p.full_tiles) {
        tile = u;
    } else {
        tile = p.full_tiles + (u - p.full_tiles) / p.S;
        split = (u - p.full_tiles) % p.S;
    }
    int tr, tc;
    decode_tile<TB>(p, tile, tr, tc);
    const bool is_split = ((int)blockIdx.x >= p.full_tiles) && (p.S > 1);
    int kbeg = 0, kend = p.K;
    if (is_split) {
        kbeg = split * p.kchunk;
        kend = min(p.K, kbeg + p.kchunk);
    }
    const int r0 = tr * TB, c0 = tc * TB;
    const int nr = min(TB, p.M - r0), nc = min(TB, p.N - c0);
    const bool has_w = (p.w != nullptr);
    const int ktiles = (kend - kbeg + BK - 1) / BK;

    if (tid == 0) {
        for (int s = 0; s < T_STAGES; ++s) { mbar_init(full + s, 1); mbar_init(empty + s, T_CONSUMERS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp >= T_CONSUMERS) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(T_REGS_PRODUCER));
        if (warp == T_CONSUMERS && lane == 0) {
            // ===== producer: one box per operand (and one of w) per k tile =====
            const uint32_t bytes = (uint32_t)(2 * T_PANEL + (has_w ? BK : 0)) * 8u;
            for (int kt = 0; kt < ktiles; ++kt) {
                const int s = kt % T_STAGES;
                if (kt >= T_STAGES) mbar_wait(empty + s, (uint32_t)(kt / T_STAGES - 1) & 1u);
                mbar_expect_tx(full + s, bytes);
                const int k = kbeg + kt * BK;
                tma_load_2d(sm + s * 2 * T_PANEL, &tmX, k, r0, full + s);
                tma_load_2d(sm + s * 2 * T_PANEL + T_PANEL, &tmY, k, c0, full + s);
                if (has_w) tma_load_1d(sw + s * BK, &tmW, k, full + s);
            }
        }
        return;
    }

    // ===== consumers: warp (wr, wc) owns rows 64 wr .. +63 and columns 32 wc .. +31 of the tile =====
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(T_REGS_CONSUMER));
    const int wr = warp & 1, wc = warp >> 1;
    const int g4 = lane >> 2, t4 = lane & 3;
    double acc[4][8][2];
    const bool pre_d = p.vec_c && (nr == TB) && (nc == TB) && !(c0 + TB - 1 > r0) && !is_split &&
                       p.beta != 0.0 && p.D != nullptr && (p.alpha == 1.0 || p.alpha == -1.0) && ((p.ldd & 1) == 0);
    if (pre_d) {
        const double sc = p.beta / p.alpha;
        const double *Dt = p.D + r0 + (long long)c0 * p.ldd;
#pragma unroll
        for (int cf = 0; cf < 4; ++cf) {
            const int cl = wc * 32 + cf * 8 + g4;
#pragma unroll
            for (int rf = 0; rf < 8; ++rf) {
                const int rl = wr * 64 + rf * 8 + t4 * 2;
                const double2 dv = *reinterpret_cast<const double2 *>(Dt + rl + (long long)cl * p.ldd);
                acc[cf][rf][0] = sc * dv.x; acc[cf][rf][1] = sc * dv.y;
            }
        }
    } else {
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;
    }

    if (r0 + wr * 64 + 63 < c0 + wc * 32) {
        // this warp's 64x32 block lies strictly above the diagonal: it only takes part in the stage releases
        for (int kt = 0; kt < ktiles; ++kt) {
            const int s = kt % T_STAGES;
            mbar_wait(full + s, (uint32_t)(kt / T_STAGES) & 1u);
            __syncwarp();
            if (lane == 0) mbar_arrive(empty + s);
        }
    } else if (ktiles > 0) {
        // swizzled fragment offsets (see the address map above) at kk = 0; kk adds 4 (kk ^ q)
        const int q = g4 >> 1;
        const int lo = 2 * ((t4 >> 1) ^ (g4 & 1)) + (t4 & 1);
        const int xo = (wr * 64 + g4) * BK + lo;
        const int yo = T_PANEL + (wc * 32 + g4) * BK + lo;
        double a[2][4], bf[2][8];
        // fragments of step kk of stage s into buffer b (the column fragments scaled by w)
        auto load = [&](int s, int kk, int b) {
            const double *st = sm + s * 2 * T_PANEL + 4 * (kk ^ q);
#pragma unroll
            for (int cf = 0; cf < 4; ++cf) a[b][cf] = st[yo + cf * 8 * BK];
#pragma unroll
            for (int rf = 0; rf < 8; ++rf) bf[b][rf] = st[xo + rf * 8 * BK];
            if (has_w) {
                const double wv = sw[s * BK + kk * 4 + t4];
#pragma unroll
                for (int cf = 0; cf < 4; ++cf) a[b][cf] *= wv;
            }
        };
        mbar_wait(full, 0u);
        load(0, 0, 0);
        for (int kt = 0; kt < ktiles; ++kt) {
            const int s = kt % T_STAGES;
#pragma unroll
            for (int kk = 0; kk < BK / 4; ++kk) {
                const int cur = kk & 1, nxt = cur ^ 1;
                if (kk + 1 < BK / 4) load(s, kk + 1, nxt);
#pragma unroll
                for (int mf = 0; mf < 2; ++mf)
#pragma unroll
                    for (int rf = 0; rf < 8; ++rf)
                        dmma16x8x4(acc[2 * mf][rf][0], acc[2 * mf][rf][1], acc[2 * mf + 1][rf][0],
                                   acc[2 * mf + 1][rf][1], a[cur][2 * mf], a[cur][2 * mf + 1], bf[cur][rf]);
                if (kk + 1 == BK / 4 && kt + 1 < ktiles) {
                    // the next stage's first fragments load under this step's DMMAs
                    const int s1 = (kt + 1) % T_STAGES;
                    mbar_wait(full + s1, (uint32_t)((kt + 1) / T_STAGES) & 1u);
                    load(s1, 0, nxt);
                }
            }
            // every fragment of stage s is in registers (this tile's last DMMAs consumed them)
            __syncwarp();
            if (lane == 0) mbar_arrive(empty + s);
        }
    }

    // ---- epilogue (the expressions of dmma_gemm_kernel's, so that the results match it bit for bit) ----
    if (is_split) {
        double *ws = p.ws + ((long long)(tile - p.full_tiles) * p.S + split) * T_TILE_ELEMS;
#pragma unroll
        for (int cf = 0; cf < 4; ++cf)
#pragma unroll
            for (int rf = 0; rf < 8; ++rf) {
                const int rl = wr * 64 + rf * 8 + t4 * 2;
                const int cl = wc * 32 + cf * 8 + g4;
                *reinterpret_cast<double2 *>(ws + rl + cl * TB) = make_double2(acc[cf][rf][0], acc[cf][rf][1]);
            }
        return;
    }
    double *C = p.C;
    const double *D = p.D;
    const bool diag = (c0 + TB - 1 > r0);                 // tile touches the diagonal
    const bool use_d = (p.beta != 0.0);
    if (p.vec_c && (nr == TB) && (nc == TB) && !diag) {
        // full interior tile, 16-byte accesses
#pragma unroll
        for (int cf = 0; cf < 4; ++cf) {
            const int cl = wc * 32 + cf * 8 + g4;
#pragma unroll
            for (int rf = 0; rf < 8; ++rf) {
                const int rl = wr * 64 + rf * 8 + t4 * 2;
                double2 v;
                if (use_d && !pre_d) {
                    const double2 dv = *reinterpret_cast<const double2 *>(D + (r0 + rl) + (long long)(c0 + cl) * p.ldd);
                    v = make_double2(p.alpha * acc[cf][rf][0] + p.beta * dv.x,
                                     p.alpha * acc[cf][rf][1] + p.beta * dv.y);
                } else {
                    v = make_double2(p.alpha * acc[cf][rf][0], p.alpha * acc[cf][rf][1]);
                }
                *reinterpret_cast<double2 *>(C + (r0 + rl) + (long long)(c0 + cl) * p.ldc) = v;
            }
        }
        return;
    }
    // edge / diagonal tiles (C may alias D: a column fragment's D values are all loaded before it is stored)
#pragma unroll
    for (int cf = 0; cf < 4; ++cf) {
        const int cl = wc * 32 + cf * 8 + g4;
        if (cl >= nc) continue;
        const long long c = c0 + cl;
        double dv[8][2];
#pragma unroll
        for (int rf = 0; rf < 8; ++rf) {
            const int rl = wr * 64 + rf * 8 + t4 * 2;
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const long long r = r0 + rl + e;
                const bool ok = use_d && (rl + e < nr) && !(diag && r < c);
                dv[rf][e] = ok ? D[r + c * p.ldd] : 0.0;
            }
        }
#pragma unroll
        for (int rf = 0; rf < 8; ++rf) {
            const int rl = wr * 64 + rf * 8 + t4 * 2;
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                if (rl + e >= nr) continue;
                const long long r = r0 + rl + e;
                if (diag && r < c) continue;
                double v = p.alpha * acc[cf][rf][e];
                if (use_d) v += p.beta * dv[rf][e];
                C[r + c * p.ldc] = v;
            }
        }
    }
}

// sums the S split-K partials of the remainder tiles (BR x TC each) in a fixed order (deterministic)
template <int TC>
__global__ void __launch_bounds__(256) splitk_reduce_kernel(const KParams p) {
    constexpr int ELEMS = BR * TC;
    const int tile = p.full_tiles + blockIdx.x;
    int tr, tc;
    decode_tile<TC>(p, tile, tr, tc);
    const int r0 = tr * BR, c0 = tc * TC;
    const int nr = min(BR, p.M - r0), nc = min(TC, p.N - c0);
    const double *ws = p.ws + (long long)blockIdx.x * p.S * ELEMS;
    for (int e = blockIdx.y * blockDim.x + threadIdx.x; e < ELEMS; e += gridDim.y * blockDim.x) {
        const int rl = e % BR, cl = e / BR;
        if (rl >= nr || cl >= nc) continue;
        const long long r = r0 + rl, c = c0 + cl;
        if (p.lower_only && r < c) continue;
        double s = 0.0;
        for (int k = 0; k < p.S; ++k) s += ws[(long long)k * ELEMS + e];
        double v = p.alpha * s;
        if (p.beta != 0.0) v += p.beta * p.D[r + c * p.ldd];
        p.C[r + c * p.ldc] = v;
    }
}

template <bool XK, bool YK, bool VEC>
int launch_inst(const KParams &p, dim3 grid, cudaStream_t st) {
    static DeviceOnce once;              // per instantiation, per device
    if (const unsigned long long bit = once.pending()) {
        CVXB_CUDA(cudaFuncSetAttribute(dmma_gemm_kernel<XK, YK, VEC>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
        CVXB_CUDA(cudaFuncSetAttribute(dmma_gemm_kernel<XK, YK, VEC>,
                                       cudaFuncAttributePreferredSharedMemoryCarveout, 100));
        once.mark(bit);
    }
    dmma_gemm_kernel<XK, YK, VEC><<<grid, THREADS, SMEM_BYTES, st>>>(p);
    count_launch();
    CVXB_LAUNCH_CHECK();
    return 0;
}

// cuTensorMapEncodeTiled from the driver the runtime loaded (the library links the runtime only)
PFN_cuTensorMapEncodeTiled_v12000 tensor_map_encoder() {
    static PFN_cuTensorMapEncodeTiled_v12000 fn = [] {
        void *f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPointByVersion("cuTensorMapEncodeTiled", &f, 12000, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess) {
            cudaGetLastError();
            f = nullptr;
        }
        return reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(f);
    }();
    return fn;
}

// tensor map of a K-major operand (rows x K, row stride ld doubles) in boxes of {BK k, TB rows}, 128-byte swizzle;
// rank 1 (rows == 0): the K-vector w in boxes of BK
int encode_operand(CUtensorMap &m, const double *base, long long ld, int K, int rows) {
    PFN_cuTensorMapEncodeTiled_v12000 enc = tensor_map_encoder();
    if (!enc) {
        set_error("dmma_gemm: cuTensorMapEncodeTiled is not available from the driver");
        return CVXB_E_CUDA;
    }
    const cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
    const cuuint64_t strides[1] = {(cuuint64_t)ld * sizeof(double)};
    const cuuint32_t box[2] = {BK, TB};
    const cuuint32_t estr[2] = {1, 1};
    const CUresult r = enc(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, rows ? 2 : 1, const_cast<double *>(base), dims, strides,
                           box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                           rows ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                           CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("dmma_gemm: cuTensorMapEncodeTiled -> CUresult %d", (int)r);
        return CVXB_E_CUDA;
    }
    return 0;
}

int launch_tma(const KParams &p, dim3 grid, cudaStream_t st) {
    CUtensorMap tx, ty, tw;
    CVXB_TRY(encode_operand(tx, p.X, p.ldx, p.K, p.M));
    CVXB_TRY(encode_operand(ty, p.Y, p.ldy, p.K, p.N));
    if (p.w) CVXB_TRY(encode_operand(tw, p.w, 0, p.K, 0));
    else tw = tx;                                        // not read
    static DeviceOnce once;
    if (const unsigned long long bit = once.pending()) {
        CVXB_CUDA(cudaFuncSetAttribute(syrk_tma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, T_SMEM));
        once.mark(bit);
    }
    syrk_tma_kernel<<<grid, T_THREADS, T_SMEM, st>>>(p, tx, ty, tw);
    count_launch();
    CVXB_LAUNCH_CHECK();
    return 0;
}

}  // namespace

size_t dmma_gemm_splitk_ws_doubles() {
    const size_t a = (size_t)SPLITK_WS_TILES * TILE_ELEMS, b = (size_t)T_WS_TILES * T_TILE_ELEMS;
    return a > b ? a : b;
}
int dmma_gemm_tile_cols() { return BC; }

int dmma_gemm(const GemmDesc &g, cudaStream_t st) {
    if (g.M <= 0 || g.N <= 0) return 0;
    if (g.K < 0 || !g.X || !g.Y || !g.C) {
        set_error("dmma_gemm: bad arguments");
        return CVXB_E_ARG;
    }
    auto aligned = [](const void *ptr, long long ld) {
        return ((uintptr_t)ptr % 16 == 0) && (ld % 2 == 0);
    };
    const int nTc = (g.N + BC - 1) / BC;
    // single K-major lower-triangle SYRKs over the whole matrix run on the TMA kernel, which needs 16-byte aligned
    // operands and row strides; the rest (odd leading dimensions, batches, Cholesky updates) on dmma_gemm_kernel
    const bool tma = g.x_kmajor && g.y_kmajor && g.lower_only && g.batch == 1 && g.K > 0 && g.ct_begin <= 0 &&
                     g.ct_end >= nTc && aligned(g.X, g.ldx) && aligned(g.Y, g.ldy) && ((uintptr_t)g.w % 16 == 0);
    const int tcols = tma ? TB : BC;                     // c-tile width
    const int wave = tma ? kNumSMs : CTAS_PER_WAVE;      // resident CTAs
    KParams p;
    p.M = g.M; p.N = g.N; p.K = g.K;
    p.X = g.X; p.ldx = g.ldx; p.Y = g.Y; p.ldy = g.ldy; p.w = g.w;
    p.D = g.D; p.ldd = g.ldd; p.C = g.C; p.ldc = g.ldc;
    p.alpha = g.alpha; p.beta = (g.D ? g.beta : 0.0);
    p.lower_only = g.lower_only ? 1 : 0;
    p.nTr = (g.M + BR - 1) / BR;
    p.ct_begin = g.ct_begin < 0 ? 0 : g.ct_begin;
    p.ct_end = g.ct_end > nTc ? nTc : g.ct_end;
    if (p.ct_begin >= p.ct_end) return 0;
    if (tma) p.ct_end = (g.N + TB - 1) / TB;
    p.sX = g.sX; p.sY = g.sY; p.sW = g.sW; p.sD = g.sD; p.sC = g.sC;
    // bands of 1024 columns
    p.band = (p.lower_only && g.K >= 1024 && g.batch == 1) ? 1024 / tcols : 0;
    long long T = 0;
    if (p.lower_only) {
        for (int c = p.ct_begin; c < p.ct_end; ++c) {
            int cnt = p.nTr - first_tr(c, tcols);
            T += cnt > 0 ? cnt : 0;
        }
    } else {
        T = (long long)p.nTr * (p.ct_end - p.ct_begin);
    }
    if (T <= 0) return 0;
    // split-K of the remainder wave (deterministic: partials + ordered reduce)
    p.full_tiles = (int)T; p.S = 1; p.kchunk = g.K; p.ws = nullptr;
    if (g.splitk_ws && g.batch == 1 && g.K >= 1024) {
        // the tiles of the last, partial wave are split along K so that the tail costs
        // ceil(rem*S / wave) / S of a tile time instead of a whole one
        int full = (int)(T / wave) * wave;
        int rem = (int)T - full;
        if (rem > 0) {
            int maxS = g.K / 512;
            if (maxS > 18) maxS = 18;
            const int cap_units = tma ? T_WS_TILES : SPLITK_WS_TILES;   // workspace capacity in tiles
            int bestS = 1;
            double best = 1.0;
            for (int S = 2; S <= maxS; ++S) {
                if ((long long)rem * S > cap_units) break;
                const double cost = (double)((rem * S + wave - 1) / wave) / S;
                if (cost < best - 1e-9) { best = cost; bestS = S; }
            }
            if (bestS >= 2) {
                p.full_tiles = full;
                p.S = bestS;
                int kc = (g.K + bestS - 1) / bestS;
                p.kchunk = ((kc + BK - 1) / BK) * BK;
                p.ws = g.splitk_ws;
            }
        }
    }
    // short-K, multi-wave launches: half of a tile's shared main-loop time (two CTAs share the
    // DMMA pipe: ~2.1 us per 16-wide k step)
    p.stagger_ns = 0;
    p.trace = g.trace;
    if (!tma && g.K <= 512 && T > CTAS_PER_WAVE) p.stagger_ns = ((g.K + BK - 1) / BK) * 1050;
    const int rem_tiles = (int)T - p.full_tiles;
    const int units = p.full_tiles + rem_tiles * p.S;
    dim3 grid(units, 1, g.batch);
    const bool vec = aligned(g.X, g.ldx) && aligned(g.Y, g.ldy) &&
                     (g.batch == 1 || (g.sX % 2 == 0 && g.sY % 2 == 0));
    p.vec_c = aligned(g.C, g.ldc) && (!g.D || aligned(g.D, g.ldd)) &&
              (g.batch == 1 || (g.sC % 2 == 0 && g.sD % 2 == 0));
    int rc;
#define DISPATCH(XK, YK)                                                   \
    rc = vec ? launch_inst<XK, YK, true>(p, grid, st) : launch_inst<XK, YK, false>(p, grid, st)
    if (tma) rc = launch_tma(p, grid, st);
    else if (g.x_kmajor && g.y_kmajor) DISPATCH(true, true);
    else if (g.x_kmajor && !g.y_kmajor) DISPATCH(true, false);
    else if (!g.x_kmajor && g.y_kmajor) DISPATCH(false, true);
    else DISPATCH(false, false);
#undef DISPATCH
    if (rc) return rc;
    if (p.S > 1) {
        dim3 rg(rem_tiles, 8);
        if (tma) splitk_reduce_kernel<TB><<<rg, 256, 0, st>>>(p);
        else splitk_reduce_kernel<BC><<<rg, 256, 0, st>>>(p);
        count_launch();
        CVXB_LAUNCH_CHECK();
    }
    return 0;
}

}  // namespace cvxb
