// fp64 tensor-core GEMM/SYRK for sm_90a.
//
//   C[r,c] = alpha * sum_k X[r,k] * w[k] * Y[c,k] + beta * D[r,c]
//
// This one kernel is the flop carrier of the whole KKT path:
//   * normal-equations assembly  K = H + G' diag(di^2) G        (X=Y=G, K-major, w=di^2,
//     lower tiles only; replaces scale(Gs)+blas.syrk+`K += H`,   reference misc.py:1268-1276)
//   * Cholesky panel TRSM  L21 = A21 * L11^{-T}                  (X=A21, Y=inv(L11), M-major)
//   * Cholesky trailing update A22 -= L21 L21'                   (X=Y=L21, M-major, lower)
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
// MMA roles are swapped w.r.t. the matrix: the MMA "m" index runs over C's columns
// (Y operand), the "n" index over C's rows (X operand), so each thread's accumulator
// pair is two consecutive ROWS of a column-major C (one 16-byte access).  One m16n8k4
// covers the column fragments cf = 2mf and 2mf+1 (8 columns apart) of a row fragment.
#include "common.cuh"

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

// first r tile that intersects the lower triangle for c tile `tc`
__device__ __host__ __forceinline__ int first_tr(int tc) { return (tc * BC) / BR; }

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
            for (int cc = c; cc < cb_end; ++cc) cnt += max(0, p.nTr - first_tr(cc));
            if (t < cnt) break;
            t -= cnt;
            c = cb_end;
        }
        for (int r = first_tr(c);; ++r) {
            const int cmax = min(cb_end - 1, (r * BR + BR - 1) / BC);   // last live c tile of this row
            const int cntr = cmax - c + 1;
            if (t < cntr) { tr = r; tc = c + t; return; }
            t -= cntr;
        }
    }
    if (p.lower_only) {
        while (true) {
            int cnt = p.nTr - first_tr(c);
            if (t < cnt) break;
            t -= cnt;
            ++c;
        }
        tr = first_tr(c) + t;
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
    decode_tile(p, tile, tr, tc);
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

// sums the S split-K partials of the remainder tiles in a fixed order (deterministic)
__global__ void __launch_bounds__(256) splitk_reduce_kernel(const KParams p) {
    const int tile = p.full_tiles + blockIdx.x;
    int tr, tc;
    decode_tile(p, tile, tr, tc);
    const int r0 = tr * BR, c0 = tc * BC;
    const int nr = min(BR, p.M - r0), nc = min(BC, p.N - c0);
    const double *ws = p.ws + (long long)blockIdx.x * p.S * TILE_ELEMS;
    for (int e = blockIdx.y * blockDim.x + threadIdx.x; e < TILE_ELEMS; e += gridDim.y * blockDim.x) {
        const int rl = e % BR, cl = e / BR;
        if (rl >= nr || cl >= nc) continue;
        const long long r = r0 + rl, c = c0 + cl;
        if (p.lower_only && r < c) continue;
        double s = 0.0;
        for (int k = 0; k < p.S; ++k) s += ws[(long long)k * TILE_ELEMS + e];
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

}  // namespace

size_t dmma_gemm_splitk_ws_doubles() { return (size_t)SPLITK_WS_TILES * TILE_ELEMS; }
int dmma_gemm_tile_cols() { return BC; }

int dmma_gemm(const GemmDesc &g, cudaStream_t st) {
    if (g.M <= 0 || g.N <= 0) return 0;
    if (g.K < 0 || !g.X || !g.Y || !g.C) {
        set_error("dmma_gemm: bad arguments");
        return CVXB_E_ARG;
    }
    KParams p;
    p.M = g.M; p.N = g.N; p.K = g.K;
    p.X = g.X; p.ldx = g.ldx; p.Y = g.Y; p.ldy = g.ldy; p.w = g.w;
    p.D = g.D; p.ldd = g.ldd; p.C = g.C; p.ldc = g.ldc;
    p.alpha = g.alpha; p.beta = (g.D ? g.beta : 0.0);
    p.lower_only = g.lower_only ? 1 : 0;
    p.nTr = (g.M + BR - 1) / BR;
    const int nTc = (g.N + BC - 1) / BC;
    p.ct_begin = g.ct_begin < 0 ? 0 : g.ct_begin;
    p.ct_end = g.ct_end > nTc ? nTc : g.ct_end;
    if (p.ct_begin >= p.ct_end) return 0;
    p.sX = g.sX; p.sY = g.sY; p.sW = g.sW; p.sD = g.sD; p.sC = g.sC;
    p.band = (p.lower_only && g.K >= 1024 && g.batch == 1) ? 16 : 0;
    long long T = 0;
    if (p.lower_only) {
        for (int c = p.ct_begin; c < p.ct_end; ++c) {
            int cnt = p.nTr - first_tr(c);
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
        int full = (int)(T / CTAS_PER_WAVE) * CTAS_PER_WAVE;
        int rem = (int)T - full;
        if (rem > 0) {
            int maxS = g.K / 512;
            if (maxS > 18) maxS = 18;
            const int cap_units = SPLITK_WS_TILES;           // workspace capacity in tiles
            int bestS = 1;
            double best = 1.0;
            for (int S = 2; S <= maxS; ++S) {
                if ((long long)rem * S > cap_units) break;
                const double cost = (double)((rem * S + CTAS_PER_WAVE - 1) / CTAS_PER_WAVE) / S;
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
    if (g.K <= 512 && T > CTAS_PER_WAVE) p.stagger_ns = ((g.K + BK - 1) / BK) * 1050;
    const int rem_tiles = (int)T - p.full_tiles;
    const int units = p.full_tiles + rem_tiles * p.S;
    dim3 grid(units, 1, g.batch);
    auto aligned = [](const void *ptr, long long ld) {
        return ((uintptr_t)ptr % 16 == 0) && (ld % 2 == 0);
    };
    const bool vec = aligned(g.X, g.ldx) && aligned(g.Y, g.ldy) &&
                     (g.batch == 1 || (g.sX % 2 == 0 && g.sY % 2 == 0));
    p.vec_c = aligned(g.C, g.ldc) && (!g.D || aligned(g.D, g.ldd)) &&
              (g.batch == 1 || (g.sC % 2 == 0 && g.sD % 2 == 0));
    int rc;
#define DISPATCH(XK, YK)                                                   \
    rc = vec ? launch_inst<XK, YK, true>(p, grid, st) : launch_inst<XK, YK, false>(p, grid, st)
    if (g.x_kmajor && g.y_kmajor) DISPATCH(true, true);
    else if (g.x_kmajor && !g.y_kmajor) DISPATCH(true, false);
    else if (!g.x_kmajor && g.y_kmajor) DISPATCH(false, true);
    else DISPATCH(false, false);
#undef DISPATCH
    if (rc) return rc;
    if (p.S > 1) {
        dim3 rg(rem_tiles, 8);
        splitk_reduce_kernel<<<rg, 256, 0, st>>>(p);
        count_launch();
        CVXB_LAUNCH_CHECK();
    }
    return 0;
}

}  // namespace cvxb
