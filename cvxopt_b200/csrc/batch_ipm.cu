// Device-resident primal-dual interior-point method for a BATCH of independent dense QPs
//
//      minimize  1/2 x'P x + q'x    subject to  G x + s = h,  s in 'l' x 'q'[0] x ...,  A x = b
//
// run in lock-step, one problem per CTA-group, with per-problem convergence masks
// (BASELINE config 4; the reference has no batch API — its counterpart is a Python loop over
// solvers.coneqp).  The algorithm is a restatement of coneprog.coneqp (reference src/python/coneprog.py:1998-2547):
// same starting point (:2055-2106), residuals and stopping rule (:2169-2234), Nesterov-Todd scaling (misc.py:284-352),
// Mehrotra predictor/corrector with STEP 0.99 / EXPON 3 (:2357-2456), `refinement` steps of iterative refinement per
// Newton solve (:2330-2347) and scaling update (misc.py:439-573).  Every KKT solve is the same path as cvxb_kkt_*:
// SYRK, Cholesky, GEMV/TRSV — here batched over the problems through blockIdx.z / blockIdx.y.  Without 'q' cones
// di² is fused into the SYRK operand and W^{-T} G is never formed; with them each factorisation writes Gs = W^{-T} G.
// With p > 0 equality rows the reduced system is solved by kkt_chol2's elimination (misc.py:1352-1560): S = P + Gs'Gs
// (+ A'A for a problem whose S was singular at the start), S = L L', Asct = L^{-1} A', Kp = Asct'Asct = Lp Lp'.
// Nothing leaves the device between iterations except one int ("how many are done").
// A cone LP batch (no P: minimize c'x over the same constraints) runs coneprog.conelp (coneprog.py:31-1436) instead,
// through the same loop, solve<CONES, EQ, LP> with LP = true: the same factorisations, solves and refinement with the
// self-dual embedding's tau / kappa arithmetic around them.  Batches with 's' blocks (SDP = true) run either
// algorithm: cvxb_batch_create_sdp builds cone LPs, cvxb_batch_create_sdp_qp QPs.
#include "cone.cuh"
#include <algorithm>
#include <climits>
#include <cstdlib>
#include <vector>
#include <memory>
#include <type_traits>

using namespace cvxb;

namespace {

struct Scal {                       // per-problem scalars, device resident
    double resx0, resz0, gap, mu, sigma, eta, step, dsdz;
    double xPxq, xq, resx, resz, zrz, pcost, dcost, relgap, pres, dres;
    double resy0, resy, yry;          // equality rows: max(1, ||b||), ||A x - b||, y'(A x - b)
    int relgap_valid, done, iters, status;   // status: 0 running, 1 optimal, 2 maxiters, 3 singular
};

// The 'l' rows [0, ml) keep d / di / lmbda in the m-vectors; cone k occupies rows [qoff[k], qoff[k+1]) and its NT
// scaling W_k = beta_k (2 v_k v_k' - J) lives in the per-slot state row (misc.py:290-352).  'l' rows are spread over
// the threads of the CTA, 'q' cones over its warps: each warp runs cone.cuh's 'q' functions as a WarpTeam, and a pass
// that reads an entry another lane wrote follows a __syncwarp().  Kernels templated on CONES compile the cone loops out
// for batches without cones; those templated on EQ compile the equality rows out for batches without them.
struct Ptrs {
    int n, m, ml, nq, refinement;
    const double *q, *h;
    double *x, *s, *z, *rx, *rz, *dx, *ds, *dz, *lmbda, *lmbdasq, *d, *di, *di2, *ws3, *bzp;
    Scal *sc;
    const int *qoff;                 // nq + 1 row offsets; qoff[nq] = m
    long long L;                     // doubles per slot in the state row
    // inside a slot's row: v (sum q, indexed by row - ml) and beta (nq) with cones, the refinement vectors with
    // refinement > 0
    double *v, *beta, *wx, *wx2, *wz, *ws, *wz2, *ws2, *wz3;
    // equality rows (neq > 0): p-vectors of every slot, Kp's per-slot Cholesky info; wy, wy2 in the state row
    int neq;
    const double *beq;
    double *y, *ry, *dy, *aw, *wy, *wy2;   // aw: the 0/1 weight of A'A in S (1: S was singular at the start)
    const int *infop;
    // cone LP batches (cvxb_batch_create_lp): q holds c; lps is the LPScal at the end of a slot's state row;
    // x1 (n), y1 (p), z1 and th (m) are rebuilt every iteration
    double *lps, *x1, *y1, *z1, *th;
    // 's' blocks (cvxb_batch_create_sdp, cvxb_batch_create_sdp_qp).  Rows [mlq, m) of the m-vectors are the blocks,
    // unpacked (ms² rows each, column-major); bzp, th, z1 and Gs hold them packed in rows [mlq, mpk).  rw: the sdot
    // weight of each m-row (1 'l' / 'q' rows and diagonals, 2 strict lower, 0 strict upper); u2p: for each 's' row,
    // its packed row minus mlq.  sinfo: per block ms, unpacked row, packed row, offset in r / rti, offset in sigs.
    // r, rti, sigs and sigz are in the state row; spart holds 4 per-(slot, block) partial results of the block kernels
    int ns, mlq, mpk, mdg;
    const int *sinfo, *u2p;
    const double *rw;
    double *sr, *srti, *sigs, *sigz, *spart;
};
// per-problem scalars of conelp's self-dual embedding (coneprog.py:847, :1031-1047), in the state row so that they
// move with their slot
struct LPScal {
    double tau, kappa, dg, dgi, lg, lgsq;          // lg = lmbda[-1] = sqrt(tau kappa) in the scaled variables
    double rt, dtau, dkappa, wkappa3, tt, tk, z1sq;
    double wtau, wkappa, wtau2, wkappa2;           // refinement copies (coneprog.py:1201-1235)
};
__device__ __forceinline__ LPScal &lp_scal(const Ptrs &p, long long oc) {
    return *reinterpret_cast<LPScal *>(p.lps + oc);
}
// a loaded start (cvxb_batch_load_start) in problem order, laid out as x, y, s and z; nullptr: the key is absent
struct Warm {
    const double *x, *y, *s, *z;
};
#define PB_SETUP                                                                                       \
    const int b = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;                                      \
    const int lane = tid & 31, warp = tid >> 5, nwarp = nt >> 5;                                       \
    const long long on = (long long)b * p.n, om = (long long)b * p.m, oc = (long long)b * p.L;         \
    const long long oq = (long long)b * p.neq;                                                         \
    __shared__ double sh[32];                                                                          \
    Scal &S = p.sc[b];                                                                                 \
    const WarpTeam wt{lane};                                                                           \
    (void)lane; (void)warp; (void)nwarp; (void)on; (void)om; (void)oc; (void)oq; (void)sh; (void)S; (void)wt;
#define FOR_CONES(o, len)                                                  \
    for (int k_ = warp; k_ < p.nq; k_ += nwarp)                            \
        if (const int o = p.qoff[k_], len = p.qoff[k_ + 1] - p.qoff[k_]; true)
#define FOR_LANE(i, len) for (int i = lane; i < len; i += 32)

// value of m-row i (an 's' row when i >= mlq) of a vector whose 's' blocks are packed (bzp, z1)
__device__ __forceinline__ double unpacked(const Ptrs &p, const double *x, int i) {
    return i < p.mlq ? x[i] : x[p.mlq + p.u2p[i - p.mlq]] * (p.rw[i] == 1.0 ? 1.0 : M_SQRT1_2);
}

// starting point, part 1: rhs of [P G'; G -I][x; z] = [-q; h] with W = I   (coneprog.py:2055-2080): d = di = 1,
// v = e1 and beta = 1 for each cone.  EQ: y = b (the solve overwrites it, :2078-2081), aw = 0 (no A'A in S yet)
template <bool EQ, bool SDP = false> __global__ void k_init_rhs(Ptrs p) {
    PB_SETUP
    double nq = 0, nh = 0, nb = 0;
    if (SDP) {                                           // W = I: r = rti = I; snrm2(h) weighs the 's' rows
        for (int i = tid; i < p.m; i += nt) { const double v = p.h[om + i]; nh += p.rw[i] * v * v; }
        for (int k = 0; k < p.ns; ++k) {
            const int ms = p.sinfo[5 * k], ro = p.sinfo[5 * k + 3];
            for (int e = tid; e < ms * ms; e += nt) {
                const double v = (e % ms == e / ms) ? 1.0 : 0.0;
                p.sr[oc + ro + e] = v; p.srti[oc + ro + e] = v;
            }
        }
    }
    if (EQ) for (int i = tid; i < p.neq; i += nt) {
        const double v = p.beq[oq + i];
        p.y[oq + i] = v; p.aw[oq + i] = 0.0;
        nb += v * v;
    }
    for (int i = tid; i < p.n; i += nt) { double v = p.q[on + i]; p.dx[on + i] = -v; nq += v * v; }
    for (int i = tid; i < p.m; i += nt) {
        double v = p.h[om + i];
        p.dz[om + i] = v;
        p.d[om + i] = 1.0; p.di[om + i] = 1.0; p.di2[om + i] = 1.0;
        if (!SDP) nh += v * v;
    }
    double *v = p.v + oc - p.ml, *beta = p.beta + oc;
    FOR_CONES(o, len) {
        FOR_LANE(i, len) v[o + i] = (i == 0) ? 1.0 : 0.0;
        if (lane == 0) beta[k_] = 1.0;
    }
    nq = block_sum(nq, sh);
    nh = block_sum(nh, sh);
    if (EQ) nb = block_sum(nb, sh);
    if (tid == 0) {
        S.resx0 = fmax(1.0, sqrt(nq));                  // :1998
        S.resz0 = fmax(1.0, sqrt(nh));                  // :2000 (snrm2 == 2-norm for 'l' and 'q')
        if (EQ) S.resy0 = fmax(1.0, sqrt(nb));          // :1999
        S.done = 0; S.iters = 0; S.status = 0; S.sigma = 0; S.eta = 0; S.step = 0;
    }
}
// bzp = W^{-T} dz (the starting point's right-hand side): 'l' rows times di, each 'q' block times W_k^{-1}
__global__ void k_scale_bz(Ptrs p) {
    PB_SETUP
    const double *src = p.dz + om;
    double *dst = p.bzp + om;
    for (int i = tid; i < p.ml; i += nt) dst[i] = p.di[om + i] * src[i];
    const double *v = p.v + oc - p.ml, *beta = p.beta + oc;
    FOR_CONES(o, len) q_scale(wt, v + o, beta[k_], src + o, dst + o, len, true);
}
// starting point with 's' blocks, the part before k_s_eig_start reads s (coneprog.py:2083-2086): x = dx, z = the
// solve's bzp unpacked, s = -z
__global__ void k_init_sz(Ptrs p) {
    PB_SETUP
    for (int i = tid; i < p.n; i += nt) p.x[on + i] = p.dx[on + i];
    for (int i = tid; i < p.m; i += nt) {
        const double zv = unpacked(p, p.bzp + om, i);
        p.z[om + i] = zv; p.s[om + i] = -zv;
    }
}
// starting point, part 2 (coneprog.py:2083-2106, :2165): x = dx, z = bzp, s = -z, then e shifts on both, gap.
// SDP: k_init_sz has set x, z and s, and k_s_eig_start has left each block's smallest eigenvalues of s and z in
// spart; snrm2 and sdot weigh the 's' rows, and the shifts go to the blocks' diagonal rows
template <bool CONES, bool SDP = false> __global__ void k_init_point(Ptrs p) {
    PB_SETUP
    double *s = p.s + om, *z = p.z + om;
    const double *zn = p.bzp + om;                      // the solve leaves W uz in bzp
    double ns = 0, mins = INFINITY, minz = INFINITY;
    if (!SDP) for (int i = tid; i < p.n; i += nt) p.x[on + i] = p.dx[on + i];
    for (int i = tid; i < p.m; i += nt) {
        const double zv = SDP ? z[i] : zn[i];
        if (SDP) ns += p.rw[i] * zv * zv;
        else { z[i] = zv; s[i] = -zv; ns += zv * zv; }
        if (i < p.ml) { mins = fmin(mins, -zv); minz = fmin(minz, zv); }
    }
    if (CONES) FOR_CONES(o, len) {                      // s = -z: ||s1|| = ||z1||, s0 = -z0
        const double z0 = zn[o], mz = -q_max_step(wt, zn + o, len);
        mins = fmin(mins, -z0 - (z0 - mz));
        minz = fmin(minz, mz);
    }
    if (SDP && tid == 0) for (int k = 0; k < p.ns; ++k) {
        const double *q = p.spart + ((long long)b * p.ns + k) * 4;
        mins = fmin(mins, q[1]); minz = fmin(minz, q[2]);
    }
    ns = sqrt(block_sum(ns, sh));
    mins = block_min(mins, sh);
    minz = block_min(minz, sh);
    const double ts = -mins, tz = -minz;
    const double as = (ts >= -1e-8 * fmax(ns, 1.0)) ? 1.0 + ts : 0.0;
    const double az = (tz >= -1e-8 * fmax(ns, 1.0)) ? 1.0 + tz : 0.0;   // nrmz == nrms here
    for (int i = tid; i < p.ml; i += nt) { s[i] += as; z[i] += az; }
    if (CONES) for (int k = tid; k < p.nq; k += nt) { s[p.qoff[k]] += as; z[p.qoff[k]] += az; }
    if (SDP) for (int i = p.mlq + tid; i < p.m; i += nt) if (p.rw[i] == 1.0) { s[i] += as; z[i] += az; }
    if (CONES || SDP) __syncthreads();
    double gap = 0;
    for (int i = tid; i < p.m; i += nt) {
        if (SDP) gap += p.rw[i] * s[i] * z[i];
        else gap += s[i] * z[i];
    }
    gap = block_sum(gap, sh);
    if (tid == 0) S.gap = gap;
}
// a loaded start, part 1: x, y, s and z.  QP (coneqp's initvals, coneprog.py:2109-2149): the given keys, else x = y = 0
// and s = z = e.  LP (conelp's primalstart / dualstart, :689-740): x and s given or, without them, the W = I solve's x
// and s = -uz; z given (y given or 0) or, without it, the W = I solve's y and z = uz.  A given 's' block is read from
// its lower triangle and stored symmetric
template <bool CONES, bool EQ, bool LP, bool SDP = false> __global__ void k_warm_copy(Ptrs p, Warm w) {
    PB_SETUP
    const double *bz = p.bzp + om;                      // the W = I solve's uz (SDP: packed)
    if (w.x) for (int i = tid; i < p.n; i += nt) p.x[on + i] = w.x[on + i];
    else if (!LP) for (int i = tid; i < p.n; i += nt) p.x[on + i] = 0.0;
    if (EQ && (!LP || w.z)) for (int i = tid; i < p.neq; i += nt) p.y[oq + i] = w.y ? w.y[oq + i] : 0.0;
    auto fill = [&](double *v, const double *g, double sg) {
        for (int i = tid; i < p.ml; i += nt) v[i] = g ? g[om + i] : LP ? sg * bz[i] : 1.0;
        if (CONES) FOR_CONES(o, len) FOR_LANE(i, len)
            v[o + i] = g ? g[om + o + i] : LP ? sg * bz[o + i] : (i == 0 ? 1.0 : 0.0);
        if (SDP) for (int k = 0; k < p.ns; ++k) {
            const int ms = p.sinfo[5 * k], so = p.sinfo[5 * k + 1];
            for (int e = tid; e < ms * ms; e += nt) {
                const int r = e % ms, c = e / ms, lo = so + (r >= c ? e : c + r * ms);
                v[so + e] = g ? g[om + lo] : LP ? sg * unpacked(p, bz, so + e) : (r == c ? 1.0 : 0.0);
            }
        }
    };
    fill(p.s + om, w.s, -1.0);
    fill(p.z + om, w.z, 1.0);
}
// a loaded start, part 2 (coneprog.py:704-740, :842-857, :2128-2165): ts and tz (SDP: the blocks' smallest
// eigenvalues from k_s_eig_warm), bad[b] = 1 (2) when the given s (z) is not strictly inside the cone; a one-sided
// cone LP start shifts the other half by 1 + ts or 1 + tz; tau = kappa = 1, gap = sdot(s, z)
template <bool CONES, bool EQ, bool LP, bool SDP = false> __global__ void k_warm_point(Ptrs p, Warm w, int *bad) {
    PB_SETUP
    double *s = p.s + om, *z = p.z + om;
    double ns = 0, nz = 0, mins = INFINITY, minz = INFINITY;
    for (int i = tid; i < p.m; i += nt) {
        const double sv = s[i], zv = z[i], wr = SDP ? p.rw[i] : 1.0;
        ns += wr * sv * sv; nz += wr * zv * zv;
        if (i < p.ml) { mins = fmin(mins, sv); minz = fmin(minz, zv); }
    }
    if (CONES) FOR_CONES(o, len) {
        mins = fmin(mins, -q_max_step(wt, s + o, len));
        minz = fmin(minz, -q_max_step(wt, z + o, len));
    }
    if (SDP && tid == 0) for (int k = 0; k < p.ns; ++k) {
        const double *q = p.spart + ((long long)b * p.ns + k) * 4;
        mins = fmin(mins, q[1]); minz = fmin(minz, q[2]);
    }
    ns = sqrt(block_sum(ns, sh)); nz = sqrt(block_sum(nz, sh));
    mins = block_min(mins, sh); minz = block_min(minz, sh);
    const double ts = -mins, tz = -minz;
    if (tid == 0) bad[b] = (w.s && ts >= 0.0) ? 1 : (w.z && tz >= 0.0) ? 2 : 0;
    if (LP) {
        const double as = (!w.s && ts >= -1e-8 * fmax(ns, 1.0)) ? 1.0 + ts : 0.0;
        const double az = (!w.z && tz >= -1e-8 * fmax(nz, 1.0)) ? 1.0 + tz : 0.0;
        for (int i = tid; i < p.ml; i += nt) { s[i] += as; z[i] += az; }
        if (CONES) for (int k = tid; k < p.nq; k += nt) { s[p.qoff[k]] += as; z[p.qoff[k]] += az; }
        if (SDP) for (int i = p.mlq + tid; i < p.m; i += nt) if (p.rw[i] == 1.0) { s[i] += as; z[i] += az; }
        __syncthreads();
    }
    double gap = 0;
    for (int i = tid; i < p.m; i += nt) gap += (SDP ? p.rw[i] : 1.0) * s[i] * z[i];
    gap = block_sum(gap, sh);
    if (tid == 0) {
        S.gap = gap;
        if (LP) { LPScal &T = lp_scal(p, oc); T.tau = 1.0; T.kappa = 1.0; }
    }
}
// residuals, part 1: rx = q (then rx += P x by GEMV), rz = s - h; EQ: ry = b (then ry := A x - ry).
// LP: rx = 0, rz = s, ry = 0; the GEMVs then make them conelp's hrx = -A'y - G'z, hrz = s + G x, hry = A x (:861-896)
template <bool EQ, bool LP> __global__ void k_res_begin(Ptrs p) {
    PB_SETUP
    for (int i = tid; i < p.n; i += nt) p.rx[on + i] = LP ? 0.0 : p.q[on + i];
    for (int i = tid; i < p.m; i += nt) p.rz[om + i] = LP ? p.s[om + i] : p.s[om + i] - p.h[om + i];   // :2183-2184
    if (EQ) for (int i = tid; i < p.neq; i += nt) p.ry[oq + i] = LP ? 0.0 : p.beq[oq + i];           // :2177-2178
}
// f0 pieces once rx = P x + q   (:2172)
__global__ void k_res_dots(Ptrs p) {
    PB_SETUP
    double a = 0, c = 0;
    for (int i = tid; i < p.n; i += nt) { double xv = p.x[on + i]; a += xv * p.rx[on + i]; c += xv * p.q[on + i]; }
    a = block_sum(a, sh); c = block_sum(c, sh);
    if (tid == 0) { S.xPxq = a; S.xq = c; }
}
// statistics + stopping rule (:2175-2234); row-wise, so every cone row is treated alike.  EQ with m = 0 is coneqp's
// cdim == 0 branch (:2002-2040): the starting point is the solution, 'optimal' after 0 iterations, dcost = pcost.
// SDP: snrm2(rz) and sdot(z, rz) weigh the 's' rows (rw), so only their lower triangles count
template <bool EQ, bool SDP = false> __global__ void k_stats(Ptrs p, int iter, int maxiters, double abstol,
                                                             double reltol, double feastol, int *ndone, int *doneflags) {
    PB_SETUP
    double rx2 = 0, rz2 = 0, zrz = 0, ry2 = 0, yry = 0;
    for (int i = tid; i < p.n; i += nt) { double v = p.rx[on + i]; rx2 += v * v; }
    for (int i = tid; i < p.m; i += nt) {
        const double v = p.rz[om + i];
        if (SDP) { const double w = p.rw[i]; rz2 += w * v * v; zrz += w * p.z[om + i] * v; }
        else { rz2 += v * v; zrz += p.z[om + i] * v; }
    }
    if (EQ) for (int i = tid; i < p.neq; i += nt) { double v = p.ry[oq + i]; ry2 += v * v; yry += p.y[oq + i] * v; }
    rx2 = block_sum(rx2, sh); rz2 = block_sum(rz2, sh); zrz = block_sum(zrz, sh);
    if (EQ) { ry2 = block_sum(ry2, sh); yry = block_sum(yry, sh); }
    if (tid == 0) {
        if (!S.done) {
            const double f0 = 0.5 * (S.xPxq + S.xq);
            S.resx = sqrt(rx2); S.resz = sqrt(rz2); S.zrz = zrz;
            S.pcost = f0;
            if (EQ) { S.resy = sqrt(ry2); S.yry = yry; }
            S.dcost = EQ ? f0 + yry + zrz - S.gap : f0 + zrz - S.gap;
            if (EQ && p.m == 0) S.dcost = f0;
            if (S.pcost < 0.0) { S.relgap = S.gap / -S.pcost; S.relgap_valid = 1; }
            else if (S.dcost > 0.0) { S.relgap = S.gap / S.dcost; S.relgap_valid = 1; }
            else { S.relgap = 0.0; S.relgap_valid = 0; }
            S.pres = EQ ? fmax(S.resy / S.resy0, S.resz / S.resz0) : S.resz / S.resz0;
            S.dres = S.resx / S.resx0;
            const bool opt = (EQ && p.m == 0) || (S.pres <= feastol && S.dres <= feastol &&
                             (S.gap <= abstol || (S.relgap_valid && S.relgap <= reltol)));
            if (opt || iter == maxiters) {
                S.done = 1; S.iters = iter; S.status = opt ? 1 : 2;
            }
        }
        if (S.done) atomicAdd(ndone, 1);
        doneflags[b] = S.done;
    }
}

// ---- compaction of finished problems ----
// The lock-step loop launches every batched kernel over the first `Bact` slots.  When problems finish, each finished
// slot below the new active count trades places with an active slot from the tail: everything a problem owns between
// iterations (P, G, its 17 vectors, its scalars, its state row; K / inv / info / Gs are rebuilt every iteration) is
// swapped, so the active problems stay a contiguous prefix and finished ones keep their final iterates in the tail.
// ~6.3 MB per swap at n=512, m=1024, at most one swap per problem per solve.  With equality rows A and the NPV
// p-vectors (b y ry dy aw) move too; Asct / Kp / its inverses / infop are rebuilt every factorisation.
constexpr int NPV = 5;
struct SwapArgs {
    double *P, *G, *vecs; Scal *sc;
    long long sP, sG;
    int n, me, Btot;
    double *A, *pvecs;               // neq > 0 only
    long long sA;
    int neq;
};
__global__ void k_swap_slots(SwapArgs a, const int *pairs) {
    const int i = pairs[2 * blockIdx.y], j = pairs[2 * blockIdx.y + 1];
    const long long eP = a.sP, eG = a.sG, eN = 4LL * a.n, eM = 13LL * a.me, eS = (long long)(sizeof(Scal) / sizeof(double));
    const long long eA = a.neq ? a.sA : 0, eQ = (long long)NPV * a.neq;
    const long long total = eP + eG + eN + eM + eS + eA + eQ;
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
        double *x, *y;
        long long r = e;
        if (r < eP) { x = a.P + i * a.sP + r; y = a.P + j * a.sP + r; }
        else if ((r -= eP) < eG) { x = a.G + i * a.sG + r; y = a.G + j * a.sG + r; }
        else if ((r -= eG) < eN) {
            const long long arr = r / a.n, k = r % a.n;
            double *base = a.vecs + arr * (long long)a.Btot * a.n;
            x = base + (long long)i * a.n + k; y = base + (long long)j * a.n + k;
        } else if ((r -= eN) < eM) {
            const long long arr = r / a.me, k = r % a.me;
            double *base = a.vecs + 4LL * a.Btot * a.n + arr * (long long)a.Btot * a.me;
            x = base + (long long)i * a.me + k; y = base + (long long)j * a.me + k;
        } else if ((r -= eM) < eA) {
            x = a.A + i * a.sA + r; y = a.A + j * a.sA + r;
        } else if ((r -= eA) < eQ) {
            const long long arr = r / a.neq, k = r % a.neq;
            double *base = a.pvecs + arr * (long long)a.Btot * a.neq;
            x = base + (long long)i * a.neq + k; y = base + (long long)j * a.neq + k;
        } else {
            r -= eQ;
            x = reinterpret_cast<double *>(a.sc + i) + r; y = reinterpret_cast<double *>(a.sc + j) + r;
        }
        const double t = *x; *x = *y; *y = t;
    }
}
// swap rows i and j of a [slots x L] buffer for each pair
__global__ void k_swap_rows(double *a, long long L, const int *pairs) {
    const long long i = pairs[2 * blockIdx.y], j = pairs[2 * blockIdx.y + 1];
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < L; e += (long long)gridDim.x * blockDim.x) {
        const double t = a[i * L + e]; a[i * L + e] = a[j * L + e]; a[j * L + e] = t;
    }
}
// out[perm[slot], :] = in[slot, :]
__global__ void k_unpermute_rows(const double *in, double *out, const int *perm, int len) {
    const int slot = blockIdx.x;
    const double *src = in + (long long)slot * len;
    double *dst = out + (long long)perm[slot] * len;
    for (int k = threadIdx.x; k < len; k += blockDim.x) dst[k] = src[k];
}
static_assert(sizeof(Scal) % sizeof(double) == 0, "Scal is swapped as doubles");

// Gs = W^{-T} G, one warp per column (misc.py:1268-1271): 'l' rows times di, each 'q' block times W_k^{-1}
__global__ void k_build_gs(Ptrs p, const double *G, double *Gs, long long ldg, long long sG) {
    const int b = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
    const int j = blockIdx.x * nwarp + warp;
    if (j >= p.n) return;
    const long long off = (long long)b * sG + (long long)j * ldg;
    const double *g = G + off, *di = p.di + (long long)b * p.m;
    double *o = Gs + off;
    for (int i = lane; i < p.ml; i += 32) o[i] = di[i] * g[i];
    const double *v = p.v + (long long)b * p.L - p.ml, *beta = p.beta + (long long)b * p.L;
    for (int k = 0; k < p.nq; ++k) {
        const int r = p.qoff[k], len = p.qoff[k + 1] - r;
        q_scale(WarpTeam{lane}, v + r, beta[k], g + r, o + r, len, true);
    }
}
// NT scaling at iteration 0 (misc.py:284-352), lambda o lambda (misc.py:945-959), mu (coneprog.py:2357).
// di2 = di² is the SYRK's weight when W^{-T} G is not formed.  LP: conelp's dg, dgi and lmbdag at iteration 0, its
// lmbdasq[-1] and mu = ||lmbda||² / (1 + cdim) (coneprog.py:1031-1047, :1248)
template <bool CONES, bool LP = false, bool SDP = false> __global__ void k_scaling(Ptrs p, int first) {
    PB_SETUP
    if (S.done) return;
    double *l = p.lmbda + om, *lsq = p.lmbdasq + om;
    const double *s = p.s + om, *z = p.z + om;
    double ll = 0;
    for (int i = tid; i < p.ml; i += nt) {
        if (first) {
            const double d = sqrt(s[i] / z[i]), di = 1.0 / d;
            p.d[om + i] = d;
            p.di[om + i] = di;
            if (!CONES) p.di2[om + i] = di * di;
            l[i] = sqrt(s[i] * z[i]);
        }
        const double li2 = l[i] * l[i];
        lsq[i] = li2;
        if (LP) ll += li2;
    }
    double *v = p.v + oc - p.ml, *beta = p.beta + oc;
    if (CONES) FOR_CONES(o, len) {
        if (first) {
            q_nt_compute(wt, s + o, z + o, v + o, l + o, beta + k_, len);
            __syncwarp();
        }
        double nl = 0;
        FOR_LANE(i, len) nl += l[o + i] * l[o + i];
        nl = warp_sum(nl);
        const double l0 = l[o];
        FOR_LANE(i, len) lsq[o + i] = (i == 0) ? nl : 2.0 * l0 * l[o + i];
        if (LP && lane == 0) ll += nl;
    }
    // 's' blocks: lambda (k_s_nt_compute / k_s_update) on the diagonal rows, lmbdasq = lambda² there, 0 elsewhere
    if (SDP) for (int i = p.mlq + tid; i < p.m; i += nt)
        if (p.rw[i] == 1.0) { const double li2 = l[i] * l[i]; lsq[i] = li2; ll += li2; }
    if (LP) {
        ll = block_sum(ll, sh);
        if (tid == 0) {
            LPScal &T = lp_scal(p, oc);
            if (first) { T.dg = sqrt(T.kappa / T.tau); T.dgi = sqrt(T.tau / T.kappa); T.lg = sqrt(T.tau * T.kappa); }
            T.lgsq = T.lg * T.lg;
            S.mu = (ll + T.lgsq) / (1.0 + (SDP ? p.mdg : p.m)); S.sigma = 0.0;
        }
    } else if (tid == 0) {                           // SDP: the degree counts each block's order (:2357)
        S.mu = SDP ? S.gap / (p.ml + p.nq + (p.mdg - p.mlq)) : S.gap / (p.ml + p.nq);
        S.sigma = 0.0; S.eta = 0.0;
    }
}

// f4_no_ir before the solve (coneprog.py:2301-2309): s := lmbda o\ s; z := z - W's; bzp := W^{-T} z.
// 'l' row r (of the m-vectors), z and s in registers
__device__ __forceinline__ void f4_pre_row(const Ptrs &p, long long r, double &z, double &s) {
    s = s / p.lmbda[r];
    z = z - p.d[r] * s;
    p.bzp[r] = p.di[r] * z;
}
// cone k at rows [o, o + len) of slot b's z and s, one warp; bzp holds W's until it receives W^{-T} z
__device__ __forceinline__ void f4_pre_cone(const Ptrs &p, long long om, long long oc, int k, int o, int len,
                                            int lane, double *z, double *s) {
    const WarpTeam wt{lane};
    const double *v = p.v + oc - p.ml;
    double *t = p.bzp + om;
    q_sinv(wt, p.lmbda + om + o, s + o, len);
    __syncwarp();
    q_scale(wt, v + o, p.beta[oc + k], s + o, t + o, len, false);
    FOR_LANE(i, len) z[o + i] -= t[o + i];
    q_scale(wt, v + o, p.beta[oc + k], z + o, t + o, len, true);
}
// f4_no_ir after the solve (coneprog.py:2316), row r: z := W uz (the solve leaves it in bzp), s := s - z; returns z.
// Not for the rows of 's' blocks, which bzp holds packed (k_f4_post<EQ, true> unpacks them)
__device__ __forceinline__ double f4_post_row(const Ptrs &p, long long r, double &s) {
    const double z = p.bzp[r];
    s -= z;
    return z;
}

// right-hand side of the i-th Newton system (coneprog.py:2373-2399), a copy of it for the refinement (:2331-2335),
// then f4_no_ir's steps before the solve.  Cone rows are formed row-wise over the CTA; after a barrier the warp that
// owns a cone adds sigma mu to its entry 0 and runs the cone part.  EQ: dy = c ry (:2395-2397).
// LP: conelp's right-hand side (:1268-1298) and its refinement copy (:1212-1218), as f6_no_ir leaves them for the
// solve (:1154-1165): y := -y, and f4_no_ir's cone steps on (-bz, -bs).  That is coneqp's right-hand side with
// c = -1 + sigma and sigma mu in the corrector (i = 1) only; dx = -c rx keeps conelp's sign.  Negation is exact, so this
// is the reference's arithmetic.  Then dtau = (1 - sigma) rt and dkappa.
template <bool CONES, bool EQ, bool LP, bool SDP = false> __global__ void k_dir_rhs(Ptrs p, int i) {
    PB_SETUP
    const double sm = S.sigma * S.mu, c = -1.0 + (LP ? S.sigma : S.eta);
    const bool add_sm = !LP || i == 1;
    LPScal &T = lp_scal(p, oc);                          // LP only
    for (int k = tid; k < p.n; k += nt) {
        const double dx = (LP ? -c : c) * p.rx[on + k];
        p.dx[on + k] = dx;
        if (p.refinement) p.wx[oc + k] = dx;
    }
    if (EQ) for (int k = tid; k < p.neq; k += nt) {
        const double dy = c * p.ry[oq + k];
        p.dy[oq + k] = dy;
        if (p.refinement) p.wy[oc + k] = dy;
    }
    // row r: z = c rz, s = -ws3 (the Mehrotra correction, i = 1) - lmbda o lmbda (+ sigma mu where e is 1).  LP starts
    // from -0.0 so that s is conelp's -lmbdasq down to the sign of a zero
    auto rhs = [&](int r, bool e, double &z, double &s) {
        s = (i == 1) ? -p.ws3[om + r] : (LP ? -0.0 : 0.0);
        s -= p.lmbdasq[om + r];
        if (e && add_sm) s += sm;
        z = c * p.rz[om + r];
        if (p.refinement) { p.wz[oc + r] = z; p.ws[oc + r] = s; }
    };
#pragma unroll 1                                         // unrolled, the 'l'-only kernel needs more registers
    for (int k = tid; k < p.ml; k += nt) {
        double z, s;
        rhs(k, true, z, s);
        f4_pre_row(p, om + k, z, s);
        p.dz[om + k] = z; p.ds[om + k] = s;
    }
    if (SDP) for (int k = p.mlq + tid; k < p.m; k += nt) {   // e is the identity: sigma mu on the diagonal rows
        double z, s;
        rhs(k, p.rw[k] == 1.0, z, s);
        p.dz[om + k] = z; p.ds[om + k] = s;
    }
    if (CONES) {
        for (int k = p.ml + tid; k < (SDP ? p.mlq : p.m); k += nt) {
            double z, s;
            rhs(k, false, z, s);
            p.dz[om + k] = z; p.ds[om + k] = s;
        }
        __syncthreads();
        FOR_CONES(o, len) {
            if (lane == 0 && add_sm) { p.ds[om + o] += sm; if (p.refinement) p.ws[oc + o] += sm; }
            __syncwarp();
            f4_pre_cone(p, om, oc, k_, o, len, lane, p.dz + om, p.ds + om);
        }
    }
    if (LP && tid == 0) {
        T.dtau = -c * T.rt;
        T.dkappa = (i == 1) ? T.lgsq + (T.wkappa3 - sm) : T.lgsq;
        if (p.refinement) { T.wtau = T.dtau; T.wkappa = T.dkappa; }
    }
}
// f4_no_ir before the solve of a refinement step, on slot b's z and s at z + b*sz, s + b*ss
__global__ void k_f4_pre(Ptrs p, double *z, long long sz, double *s, long long ss) {
    PB_SETUP
    z += b * sz; s += b * ss;
    for (int i = tid; i < p.ml; i += nt) {
        double zv = z[i], sv = s[i];
        f4_pre_row(p, om + i, zv, sv);
        z[i] = zv; s[i] = sv;
    }
    FOR_CONES(o, len) f4_pre_cone(p, om, oc, k_, o, len, lane, z, s);
}
// f4_no_ir after a solve that refinement follows or that is a refinement step.  acc: the refinement step,
// (dx, dz, ds) += (x, z, s), and with EQ dy += wy2 (a refinement step's y is always wy2).  SDP: z is unpacked from
// bzp; a QP batch with 's' blocks also runs it after an unrefined solve, where k_s_dir_post reads its result
template <bool EQ, bool SDP = false>
__global__ void k_f4_post(Ptrs p, double *x, long long sx, double *z, long long sz, double *s, long long ss, int acc) {
    PB_SETUP
    x += b * sx; z += b * sz; s += b * ss;
    for (int i = tid; i < p.m; i += nt) {
        double sv = s[i], zv;
        if (SDP) { zv = unpacked(p, p.bzp + om, i); sv -= zv; }
        else zv = f4_post_row(p, om + i, sv);
        z[i] = zv; s[i] = sv;
        if (acc) { p.dz[om + i] += zv; p.ds[om + i] += sv; }
    }
    if (acc) for (int i = tid; i < p.n; i += nt) p.dx[on + i] += x[i];
    if (EQ && acc) for (int i = tid; i < p.neq; i += nt) p.dy[oq + i] += p.wy2[oc + i];
}
// refinement residual, the elementwise part of res() (coneprog.py:1930-1960): wx2 = wx, wz3 = W^{-1} dz,
// wz2 = wz - W' ds, ws2 = ws - lmbda o (dz + ds); EQ: wy2 = wy.  The P, A, A', G and G' products follow as
// batched GEMVs.  LP: conelp's res() (:599-631) adds the embedding's column ut (-c, b, h), ut = dtau / dg, to
// (wx2, wy2, wz2), and forms wtau2 = wtau + dg dkappa + c'dx + b'dy + h'wz3, wkappa2 = wkappa + lmbdag (dtau + dkappa).
template <bool EQ, bool LP, bool SDP = false> __global__ void k_res(Ptrs p) {
    PB_SETUP
    const double *l = p.lmbda + om, *dz = p.dz + om, *ds = p.ds + om, *h = p.h + om;
    const double ut = LP ? lp_scal(p, oc).dtau / lp_scal(p, oc).dg : 0.0;
    double cx = 0, by = 0, hz = 0;
    for (int i = tid; i < p.n; i += nt) {
        if (LP) {
            const double c = p.q[on + i];
            p.wx2[oc + i] = p.wx[oc + i] + (-ut) * c;
            cx += c * p.dx[on + i];
        } else p.wx2[oc + i] = p.wx[oc + i];
    }
    if (EQ) for (int i = tid; i < p.neq; i += nt) {
        if (LP) {
            const double bb = p.beq[oq + i];
            p.wy2[oc + i] = p.wy[oc + i] + ut * bb;
            by += bb * p.dy[oq + i];
        } else p.wy2[oc + i] = p.wy[oc + i];
    }
    double *wz3 = p.wz3 + oc, *wz2 = p.wz2 + oc, *ws2 = p.ws2 + oc;
    for (int i = tid; i < p.ml; i += nt) {
        const double w3 = p.di[om + i] * dz[i];
        wz3[i] = w3;
        double w = p.wz[oc + i];
        if (LP) { hz += h[i] * w3; w += ut * h[i]; }
        wz2[i] = w - p.d[om + i] * ds[i];
        ws2[i] = p.ws[oc + i] - l[i] * (dz[i] + ds[i]);
    }
    const double *v = p.v + oc - p.ml, *beta = p.beta + oc;
    FOR_CONES(o, len) {
        q_scale(wt, v + o, beta[k_], dz + o, wz3 + o, len, true);
        q_scale(wt, v + o, beta[k_], ds + o, wz2 + o, len, false);
        FOR_LANE(i, len) ws2[o + i] = ds[o + i] + dz[o + i];
        __syncwarp();
        q_sprod(wt, l + o, ws2 + o, ws2 + o, len);
        __syncwarp();
        FOR_LANE(i, len) {
            double w = p.wz[oc + o + i];
            if (LP) { hz += h[o + i] * wz3[o + i]; w += ut * h[o + i]; }
            wz2[o + i] = w - wz2[o + i];
            ws2[o + i] = p.ws[oc + o + i] - ws2[o + i];
        }
    }
    if (LP) {
        cx = block_sum(cx, sh); hz = block_sum(hz, sh);
        if (EQ) by = block_sum(by, sh);
        if (tid == 0) {
            LPScal &T = lp_scal(p, oc);
            if (SDP) for (int k = 0; k < p.ns; ++k) hz += p.spart[((long long)b * p.ns + k) * 4];   // k_s_res's h'wz3
            T.wtau2 = T.wtau + (T.dg * T.dkappa + cx + by + hz);
            T.wkappa2 = T.wkappa + T.lg * (T.dtau + T.dkappa);
        }
    }
}
// after the i-th direction: ds o dz, scale2 of ds and dz, step length, sigma (coneprog.py:2423-2456).
// f4_post: the solve has just run without refinement, so f4_no_ir's step after it is done here first.
// LP: conelp's dkappa dtau product, tt and tk in the step, sigma = (1 - step)^3 (coneprog.py:1302-1333)
template <bool CONES, bool LP = false, bool SDP = false> __global__ void k_dir_post(Ptrs p, int i, int f4_post) {
    PB_SETUP
    double *ds = p.ds + om, *dz = p.dz + om;
    const double *l = p.lmbda + om;
    double dsdz = 0, mins = INFINITY, minz = INFINITY;
#pragma unroll 1                                         // as in k_dir_rhs
    for (int k = tid; k < p.ml; k += nt) {
        double s = ds[k];
        const double z = f4_post ? f4_post_row(p, om + k, s) : dz[k];
        dsdz += s * z;
        if (i == 0) p.ws3[om + k] = s * z;
        const double ss = s / l[k], zs = z / l[k];
        ds[k] = ss; dz[k] = zs;
        mins = fmin(mins, ss); minz = fmin(minz, zs);
    }
    if (CONES && f4_post) {
        for (int k = p.ml + tid; k < p.m; k += nt) dz[k] = f4_post_row(p, om + k, ds[k]);
        __syncthreads();
    }
    if (CONES) FOR_CONES(o, len) {
        const double a = q_sprod(wt, dz + o, ds + o, i == 0 ? p.ws3 + om + o : nullptr, len);
        if (lane == 0) dsdz += a;
        __syncwarp();
        q_scale2(wt, l + o, ds + o, len, false);
        q_scale2(wt, l + o, dz + o, len, false);
        __syncwarp();
        mins = fmin(mins, -q_max_step(wt, ds + o, len));
        minz = fmin(minz, -q_max_step(wt, dz + o, len));
    }
    dsdz = block_sum(dsdz, sh);
    mins = block_min(mins, sh);
    minz = block_min(minz, sh);
    if (tid == 0) {
        if (SDP) for (int k = 0; k < p.ns; ++k) {        // k_s_dir_post: sdot(ds, dz) and the smallest eigenvalues
            const double *q = p.spart + ((long long)b * p.ns + k) * 4;
            dsdz += q[0]; mins = fmin(mins, q[1]); minz = fmin(minz, q[2]);
        }
        double t = fmax(0.0, fmax(-mins, -minz));
        if (LP) {
            LPScal &T = lp_scal(p, oc);
            if (i == 0) T.wkappa3 = T.dtau * T.dkappa;
            T.tt = -T.dtau / T.lg; T.tk = -T.dkappa / T.lg;
            t = fmax(t, fmax(T.tt, T.tk));
        }
        double step;
        if (t == 0.0) step = 1.0;
        else step = (i == 0) ? fmin(1.0, 1.0 / t) : fmin(1.0, 0.99 / t);
        S.step = step; S.dsdz = dsdz;
        if (i == 0 && LP) {
            const double v = 1.0 - step;
            S.sigma = v * v * v;
        } else if (i == 0) {
            const double v = fmin(1.0, fmax(0.0, 1.0 - step + dsdz / S.gap * step * step));
            S.sigma = v * v * v;
            S.eta = 0.0;
        }
    }
}
// x += step dx; ds, dz := e + step d; scale2 inverse; update_scaling (misc.py:439-573); s = W' lmbda,
// z = W^{-1} lmbda; gap (coneprog.py:2459-2547).  EQ: y += step dy (:2460); a singular Kp stops the problem too.
// LP: conelp's dg, lmbdag, tau, kappa and gap (coneprog.py:1405-1436); a singular factorisation returns the iterate
// divided by tau (:1078-1109)
template <bool CONES, bool EQ, bool LP = false, bool SDP = false>
__global__ void k_update(Ptrs p, const int *info, int iter) {
    PB_SETUP
    if (S.done) return;
    bool fail = false;                               // SDP: a block's Jacobi SVD did not converge (k_s_update)
    if (SDP) for (int k = 0; k < p.ns; ++k) fail |= p.spart[((long long)b * p.ns + k) * 4 + 3] != 0.0;
    if (fail || info[b] > 0 || (EQ && p.infop[b] > 0)) {   // non-positive pivot: "Terminated (singular KKT matrix)" (:2257-2275)
        if (LP) {
            const double ti = 1.0 / lp_scal(p, oc).tau;
            for (int k = tid; k < p.n; k += nt) p.x[on + k] *= ti;
            if (EQ) for (int k = tid; k < p.neq; k += nt) p.y[oq + k] *= ti;
            for (int k = tid; k < p.m; k += nt) { p.s[om + k] *= ti; p.z[om + k] *= ti; }
        }
        if (tid == 0) { S.done = 1; S.status = 3; S.iters = iter; }
        return;
    }
    const double step = S.step;
    for (int k = tid; k < p.n; k += nt) p.x[on + k] += step * p.dx[on + k];
    if (EQ) for (int k = tid; k < p.neq; k += nt) p.y[oq + k] += step * p.dy[oq + k];
    double *ds = p.ds + om, *dz = p.dz + om, *l = p.lmbda + om, *s = p.s + om, *z = p.z + om;
    double gap = 0;
    for (int k = tid; k < p.ml; k += nt) {
        const double lk = l[k];
        const double ss = sqrt((1.0 + step * ds[k]) * lk), sz = sqrt((1.0 + step * dz[k]) * lk);
        const double d = p.d[om + k] * ss / sz, di = 1.0 / d;
        const double ln = ss * sz;
        p.d[om + k] = d; p.di[om + k] = di;
        if (!CONES) p.di2[om + k] = di * di;
        l[k] = ln;
        s[k] = d * ln;
        z[k] = di * ln;
        gap += ln * ln;
    }
    double *v = p.v + oc - p.ml, *beta = p.beta + oc;
    if (CONES) FOR_CONES(o, len) {
        FOR_LANE(k, len) {
            ds[o + k] = step * ds[o + k] + (k == 0 ? 1.0 : 0.0);
            dz[o + k] = step * dz[o + k] + (k == 0 ? 1.0 : 0.0);
        }
        __syncwarp();
        q_scale2(wt, l + o, ds + o, len, true);
        q_scale2(wt, l + o, dz + o, len, true);
        __syncwarp();
        q_nt_update(wt, ds + o, dz + o, v + o, l + o, beta + k_, len);
        __syncwarp();
        // unscale with the new W and lambda
        const double bk = beta[k_];
        q_scale(wt, v + o, bk, l + o, s + o, len, false);
        q_scale(wt, v + o, bk, l + o, z + o, len, true);
        double g = 0;
        FOR_LANE(k, len) g += l[o + k] * l[o + k];
        g = warp_sum(g);
        if (lane == 0) gap += g;
    }
    if (SDP) {                                       // commit what k_s_update staged (every block succeeded)
        for (int k = p.mlq + tid; k < p.m; k += nt) {
            s[k] = ds[k]; z[k] = dz[k];
            if (p.rw[k] == 1.0) { const double lk = p.lmbdasq[om + k]; l[k] = lk; gap += lk * lk; }
        }
        for (int k = 0; k < p.ns; ++k) {
            const int ms = p.sinfo[5 * k], so = p.sinfo[5 * k + 1], ro = p.sinfo[5 * k + 3];
            for (int e = tid; e < ms * ms; e += nt) {
                p.sr[oc + ro + e] = p.d[om + so + e]; p.srti[oc + ro + e] = p.di[om + so + e];
            }
        }
    }
    gap = block_sum(gap, sh);
    if (LP) {
        if (tid == 0) {
            LPScal &T = lp_scal(p, oc);
            T.dg *= sqrt(1.0 - step * T.tk) / sqrt(1.0 - step * T.tt);
            T.dgi = 1.0 / T.dg;
            T.lg *= sqrt(1.0 - step * T.tt) * sqrt(1.0 - step * T.tk);
            T.kappa = T.lg / T.dgi; T.tau = T.lg * T.dgi;
            const double g = sqrt(gap) / T.tau;
            S.gap = g * g;
        }
    } else if (tid == 0) S.gap = gap;
}
// the S + A'A switch of kkt_chol2's first factorisation (misc.py:1421-1447), per problem: a slot whose S = P + Gs'Gs
// was singular at the start (info > 0) weights A'A by 1 in every later S
__global__ void k_switch(double *aw, const int *info, int neq) {
    const double w = info[blockIdx.x] > 0 ? 1.0 : 0.0;
    for (int k = threadIdx.x; k < neq; k += blockDim.x) aw[(long long)blockIdx.x * neq + k] = w;
}

// ---- cone LPs: coneprog.conelp (coneprog.py:31-1436) ----
// The kernels below are the arithmetic in which conelp's homogeneous self-dual embedding differs from coneqp; the
// scaling, the factorisation, the KKT solves, f4_no_ir's cone steps, the right-hand side, the refinement residual, the
// step length and the update are coneqp's kernels with LP = true.
// The primal start's solve has left uz in bzp: s = -uz (:698-701).  The dual start's right-hand side (-c, 0, 0):
// k_init_rhs put -c in dx, here y = 0 and bz = 0 (:724-728)
template <bool EQ, bool SDP = false> __global__ void k_lp_start_mid(Ptrs p) {
    PB_SETUP
    if (SDP) {
        for (int i = tid; i < p.m; i += nt) p.s[om + i] = -unpacked(p, p.bzp + om, i);
        __syncthreads();
        for (int i = tid; i < p.mpk; i += nt) p.bzp[om + i] = 0.0;
    } else
    for (int i = tid; i < p.m; i += nt) { p.s[om + i] = -p.bzp[om + i]; p.bzp[om + i] = 0.0; }
    if (EQ) for (int i = tid; i < p.neq; i += nt) p.y[oq + i] = 0.0;
}
// the starting point (:737-857): z from the dual start's solve, ts / tz, the "already optimal" return at iteration 0
// (:744-804), the shifts by 1 + ts and 1 + tz, tau = kappa = 1, gap
template <bool CONES, bool EQ, bool SDP = false> __global__ void k_lp_init_point(Ptrs p, double abstol, double reltol) {
    PB_SETUP
    double *s = p.s + om, *z = p.z + om;
    const double *zn = p.bzp + om, *h = p.h + om;
    double ns = 0, nz = 0, sz = 0, cx = 0, by = 0, hz = 0, mins = INFINITY, minz = INFINITY;
    for (int i = tid; i < p.n; i += nt) cx += p.q[on + i] * p.x[on + i];
    if (EQ) for (int i = tid; i < p.neq; i += nt) by += p.beq[oq + i] * p.y[oq + i];
    if (SDP) {
        // z unpacked from the solve's bzp; snrm2 / sdot weigh the 's' rows; the blocks' smallest eigenvalues come
        // from k_s_eig_start
        for (int i = tid; i < p.m; i += nt) {
            const double zv = unpacked(p, zn, i), sv = s[i], w = p.rw[i];
            z[i] = zv;
            ns += w * sv * sv; nz += w * zv * zv; sz += w * sv * zv; hz += w * h[i] * zv;
            if (i < p.ml) { mins = fmin(mins, sv); minz = fmin(minz, zv); }
        }
        if (tid == 0) for (int k = 0; k < p.ns; ++k) {
            const double *q = p.spart + ((long long)b * p.ns + k) * 4;
            mins = fmin(mins, q[1]); minz = fmin(minz, q[2]);
        }
    } else
    for (int i = tid; i < p.m; i += nt) {
        const double zv = zn[i], sv = s[i];
        z[i] = zv;
        ns += sv * sv; nz += zv * zv; sz += sv * zv; hz += h[i] * zv;
        if (i < p.ml) { mins = fmin(mins, sv); minz = fmin(minz, zv); }
    }
    if (CONES) FOR_CONES(o, len) {
        mins = fmin(mins, -q_max_step(wt, s + o, len));
        minz = fmin(minz, -q_max_step(wt, zn + o, len));
    }
    ns = sqrt(block_sum(ns, sh)); nz = sqrt(block_sum(nz, sh));
    sz = block_sum(sz, sh); cx = block_sum(cx, sh); hz = block_sum(hz, sh);
    if (EQ) by = block_sum(by, sh);
    mins = block_min(mins, sh); minz = block_min(minz, sh);
    const double ts = -mins, tz = -minz, dcost = -by - hz;
    const bool relv = cx < 0.0 || dcost > 0.0;
    const double relgap = cx < 0.0 ? sz / -cx : sz / dcost;
    if (ts <= 0 && tz <= 0 && (sz <= abstol || (relv && relgap <= reltol))) {
        if (tid == 0) {
            S.done = 1; S.status = 1; S.iters = 0; S.gap = sz;
            S.pcost = cx; S.dcost = -(by + hz);
        }
        return;
    }
    const double as = (ts >= -1e-8 * fmax(ns, 1.0)) ? 1.0 + ts : 0.0;
    const double az = (tz >= -1e-8 * fmax(nz, 1.0)) ? 1.0 + tz : 0.0;
    for (int i = tid; i < p.ml; i += nt) { s[i] += as; z[i] += az; }
    if (CONES) for (int k = tid; k < p.nq; k += nt) { s[p.qoff[k]] += as; z[p.qoff[k]] += az; }
    if (SDP) for (int i = p.mlq + tid; i < p.m; i += nt) if (p.rw[i] == 1.0) { s[i] += as; z[i] += az; }
    __syncthreads();
    double gap = 0;
    for (int i = tid; i < p.m; i += nt) gap += (SDP ? p.rw[i] : 1.0) * s[i] * z[i];
    gap = block_sum(gap, sh);
    if (tid == 0) {
        S.gap = gap;
        LPScal &T = lp_scal(p, oc);
        T.tau = 1.0; T.kappa = 1.0;
    }
}
// residuals, part 2, and the stopping rule (:864-1023): rx = hrx - c tau, ry = hry - b tau, rz = hrz - h tau, rt;
// optimal or maxiters divide the iterate by tau; a primal infeasibility certificate divides y and z by -h'z - b'y
// and x, s become NaN (the reference's None); a dual infeasibility certificate divides x and s by -c'x and y, z
// become NaN.  Status 4 primal infeasible, 5 dual infeasible.
template <bool EQ, bool SDP = false>
__global__ void k_lp_stats(Ptrs p, int iter, int maxiters, double abstol, double reltol, double feastol, int *ndone,
                           int *doneflags) {
    PB_SETUP
    __shared__ int act;
    __shared__ double fac;
    if (!S.done) {
        LPScal &T = lp_scal(p, oc);
        const double tau = T.tau;
        double hx = 0, rx2 = 0, hy = 0, ry2 = 0, hzz = 0, rz2 = 0, cx = 0, by = 0, hz = 0;
        for (int i = tid; i < p.n; i += nt) {
            const double v = p.rx[on + i], c = p.q[on + i], r = v + (-tau) * c;
            p.rx[on + i] = r;
            hx += v * v; rx2 += r * r; cx += c * p.x[on + i];
        }
        if (EQ) for (int i = tid; i < p.neq; i += nt) {
            const double v = p.ry[oq + i], bb = p.beq[oq + i], r = v + (-tau) * bb;
            p.ry[oq + i] = r;
            hy += v * v; ry2 += r * r; by += bb * p.y[oq + i];
        }
        for (int i = tid; i < p.m; i += nt) {
            const double v = p.rz[om + i], hh = p.h[om + i], r = v + (-tau) * hh;
            p.rz[om + i] = r;
            if (SDP) { const double w = p.rw[i]; hzz += w * v * v; rz2 += w * r * r; hz += w * hh * p.z[om + i]; }
            else { hzz += v * v; rz2 += r * r; hz += hh * p.z[om + i]; }
        }
        hx = block_sum(hx, sh); rx2 = block_sum(rx2, sh); cx = block_sum(cx, sh);
        hzz = block_sum(hzz, sh); rz2 = block_sum(rz2, sh); hz = block_sum(hz, sh);
        if (EQ) { hy = block_sum(hy, sh); ry2 = block_sum(ry2, sh); by = block_sum(by, sh); }
        if (tid == 0) {
            const double resx = sqrt(rx2) / tau, resy = sqrt(ry2) / tau, resz = sqrt(rz2) / tau;
            T.rt = T.kappa + cx + by + hz;
            S.resx = resx; S.resz = resz; S.resy = resy;
            S.pcost = cx / tau; S.dcost = -(by + hz) / tau;
            if (S.pcost < 0.0) { S.relgap = S.gap / -S.pcost; S.relgap_valid = 1; }
            else if (S.dcost > 0.0) { S.relgap = S.gap / S.dcost; S.relgap_valid = 1; }
            else { S.relgap = 0.0; S.relgap_valid = 0; }
            S.pres = EQ ? fmax(resy / S.resy0, resz / S.resz0) : resz / S.resz0;
            S.dres = resx / S.resx0;
            const bool pinf = hz + by < 0.0 && sqrt(hx) / S.resx0 / (-hz - by) <= feastol;
            const double dinfres = EQ ? fmax(sqrt(hy) / S.resy0, sqrt(hzz) / S.resz0) : sqrt(hzz) / S.resz0;
            const bool dinf = cx < 0.0 && dinfres / (-cx) <= feastol;
            const bool opt = S.pres <= feastol && S.dres <= feastol &&
                             (S.gap <= abstol || (S.relgap_valid && S.relgap <= reltol));
            act = 0;
            if (opt || iter == maxiters) { act = 1; fac = 1.0 / tau; S.status = opt ? 1 : 2; }
            else if (pinf) { act = 2; fac = 1.0 / (-hz - by); S.status = 4; S.pcost = NAN; S.dcost = 1.0; }
            else if (dinf) { act = 3; fac = 1.0 / (-cx); S.status = 5; S.pcost = -1.0; S.dcost = NAN; }
            if (act) { S.done = 1; S.iters = iter; }
        }
        __syncthreads();
        if (act) {
            const double f = fac, nan = NAN;
            const double fx = act == 2 ? nan : f, fy = act == 3 ? nan : f;
            for (int i = tid; i < p.n; i += nt) p.x[on + i] = act == 2 ? nan : p.x[on + i] * fx;
            if (EQ) for (int i = tid; i < p.neq; i += nt) p.y[oq + i] = act == 3 ? nan : p.y[oq + i] * fy;
            for (int i = tid; i < p.m; i += nt) {
                p.s[om + i] = act == 2 ? nan : p.s[om + i] * fx;
                p.z[om + i] = act == 3 ? nan : p.z[om + i] * fy;
            }
        }
    }
    if (tid == 0) {
        if (S.done) atomicAdd(ndone, 1);
        doneflags[b] = S.done;
    }
}
// the extra solve's right-hand side (:1066-1074): x1 = -c, y1 = b, z1 = h, and th = W^{-T} h (:1125-1128), which is
// also the solve's bzp
template <bool EQ> __global__ void k_lp_x1_rhs(Ptrs p) {
    PB_SETUP
    for (int i = tid; i < p.n; i += nt) p.x1[on + i] = -p.q[on + i];
    if (EQ) for (int i = tid; i < p.neq; i += nt) p.y1[oq + i] = p.beq[oq + i];
    const double *h = p.h + om;
    double *th = p.th + om, *bz = p.bzp + om;
    for (int i = tid; i < p.ml; i += nt) { const double t = p.di[om + i] * h[i]; th[i] = t; bz[i] = t; }
    const double *v = p.v + oc - p.ml, *beta = p.beta + oc;
    FOR_CONES(o, len) {
        q_scale(wt, v + o, beta[k_], h + o, th + o, len, true);
        __syncwarp();
        FOR_LANE(i, len) bz[o + i] = th[o + i];
    }
}
// (x1, y1, z1) *= dgi (:1075-1077); z1'z1 for f6_no_ir
template <bool EQ, bool SDP = false> __global__ void k_lp_x1_post(Ptrs p) {
    PB_SETUP
    const double dgi = lp_scal(p, oc).dgi;
    for (int i = tid; i < p.n; i += nt) p.x1[on + i] *= dgi;
    if (EQ) for (int i = tid; i < p.neq; i += nt) p.y1[oq + i] *= dgi;
    double a = 0;
    // SDP: z1 stays packed, so z1'z1 is its sdot
    for (int i = tid; i < (SDP ? p.mpk : p.m); i += nt) { const double v = dgi * p.bzp[om + i]; p.z1[om + i] = v; a += v * v; }
    a = block_sum(a, sh);
    if (tid == 0) lp_scal(p, oc).z1sq = a;
}
// f6_no_ir after the solve (:1180-1195): with the solve's (x, y) and uz in bzp, kappa := -bkappa / lmbdag,
// tau := dgi (btau - bkappa / tau + c'x + b'y + th'uz) / (1 + z1'z1), (x, y, z) += tau (x1, y1, z1), s := s - z,
// kappa -= tau.  acc = 0: the Newton solve, in place on (dx, dy, ds), z to dz, (btau, bkappa) = (dtau, dkappa).
// acc = 1: a refinement step on (wx2, wy2, ws2) with (wtau2, wkappa2), added to the direction (:1230-1235).
template <bool EQ, bool SDP = false>
__global__ void k_lp_f6_post(Ptrs p, double *x, long long sx, double *y, long long sy, double *s, long long ss, int acc) {
    PB_SETUP
    LPScal &T = lp_scal(p, oc);
    x += b * sx; s += b * ss;
    if (EQ) y += b * sy;
    const double *uz = p.bzp + om, *c = p.q + on, *x1 = p.x1 + on, *z1 = p.z1 + om, *th = p.th + om;
    const double tin = acc ? T.wtau2 : T.dtau, kin = acc ? T.wkappa2 : T.dkappa;
    double cx = 0, by = 0, tz = 0;
    for (int i = tid; i < p.n; i += nt) cx += c[i] * x[i];
    if (EQ) for (int i = tid; i < p.neq; i += nt) by += p.beq[oq + i] * y[i];
    for (int i = tid; i < (SDP ? p.mpk : p.m); i += nt) tz += th[i] * uz[i];   // SDP: packed, sdot(th, uz)
    cx = block_sum(cx, sh); tz = block_sum(tz, sh);
    if (EQ) by = block_sum(by, sh);
    double kap = -kin / T.lg;
    double tau = tin + kap / T.dgi;
    tau = T.dgi * (tau + cx + by + tz) / (1.0 + T.z1sq);
    for (int i = tid; i < p.n; i += nt) {
        const double v = x[i] + tau * x1[i];
        if (acc) p.dx[on + i] += v; else x[i] = v;
    }
    if (EQ) for (int i = tid; i < p.neq; i += nt) {
        const double v = y[i] + tau * p.y1[oq + i];
        if (acc) p.dy[oq + i] += v; else y[i] = v;
    }
    for (int i = tid; i < p.m; i += nt) {
        const double zv = SDP ? unpacked(p, uz, i) + tau * unpacked(p, z1, i) : uz[i] + tau * z1[i], sv = s[i] - zv;
        if (acc) { p.dz[om + i] += zv; p.ds[om + i] += sv; }
        else { p.dz[om + i] = zv; s[i] = sv; }
    }
    kap -= tau;
    if (tid == 0) {
        if (acc) { T.dtau += tau; T.dkappa += kap; }
        else { T.dtau = tau; T.dkappa = kap; }
    }
}

// ---- 's' blocks: one CTA of SB_T threads per (block, slot), grid (ns, Bact) ----
// A block of order ms <= CVXB_BATCH_SMAX is an ms x ms column-major matrix in shared memory.  The kernels read only
// the lower triangle of what they are given (the reference reads no more, misc_solvers.c scale / sdot), and write
// s, z, ds, dz and the refinement vectors with both triangles.  Per-block partial sums go to spart; the per-problem
// kernels add them up in block order.
constexpr int SB_T = 256, SMX = CVXB_BATCH_SMAX * CVXB_BATCH_SMAX, JAC_SWEEPS = 30;
#define SB_SETUP                                                                                       \
    const int k = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;                                       \
    const int ms = p.sinfo[5 * k], so = p.sinfo[5 * k + 1], sp = p.sinfo[5 * k + 2];                   \
    const int sro = p.sinfo[5 * k + 3], sgo = p.sinfo[5 * k + 4];                                      \
    const long long om = (long long)b * p.m, oc = (long long)b * p.L;                                  \
    Scal &S = p.sc[b];                                                                                 \
    (void)tid; (void)sp; (void)sro; (void)sgo; (void)om; (void)oc; (void)S;
#define SB_PART double *part = p.spart + ((long long)b * p.ns + k) * 4
#define SB_FOR(e, ms) for (int e = threadIdx.x; e < (ms) * (ms); e += SB_T)

// X := sym(lower triangle of the column-major block x)
__device__ void s_load(double *X, const double *x, int ms) {
    SB_FOR(e, ms) { const int i = e % ms, j = e / ms; X[e] = i >= j ? x[e] : x[j + i * ms]; }
    __syncthreads();
}
// X := the block unpacked from packed storage with sqrt(2) off-diagonals (misc.unpack)
__device__ void s_load_packed(double *X, const double *x, int ms) {
    SB_FOR(e, ms) {
        const int i = e % ms, j = e / ms, c = min(i, j), r = max(i, j);
        const double v = x[c * ms - c * (c - 1) / 2 + r - c];
        X[e] = i == j ? v : v * M_SQRT1_2;
    }
    __syncthreads();
}
// packed storage of X's lower triangle, off-diagonals times sqrt(2) (misc.pack / pack2)
__device__ void s_store_packed(double *x, const double *X, int ms) {
    SB_FOR(e, ms) {
        const int i = e % ms, j = e / ms;
        if (i >= j) x[j * ms - j * (j - 1) / 2 + i - j] = i == j ? X[e] : M_SQRT2 * X[e];
    }
}
// C := op(A) op(B).  The lanes of a warp take consecutive rows i.  With ta they would read A' at a stride of ms
// doubles, all in one bank when ms = 32, so each lane starts its sum at l = i (mod ms); it is never called with ta and
// tb both set, where that would move the conflict onto B.
__device__ void s_mm(double *C, const double *A, bool ta, const double *B, bool tb, int ms) {
    SB_FOR(e, ms) {
        const int i = e % ms, j = e / ms;
        double a = 0.0;
        int l = ta ? i : 0;
        for (int c = 0; c < ms; ++c, l = (l + 1 == ms) ? 0 : l + 1)
            a += (ta ? A[l + i * ms] : A[i + l * ms]) * (tb ? B[j + l * ms] : B[l + j * ms]);
        C[e] = a;
    }
    __syncthreads();
}
// C := A' X A (tr = true) or A X A' for symmetric X; T is scratch
__device__ void s_congr(double *C, const double *A, const double *X, double *T, bool tr, int ms) {
    s_mm(T, X, false, A, !tr, ms);
    s_mm(C, A, tr, T, false, ms);
}
// sdot's share of one block: diagonal once, strict lower triangle twice
__device__ double s_dot(const double *X, const double *Y, int ms, double *sh) {
    double a = 0.0;
    SB_FOR(e, ms) { const int i = e % ms, j = e / ms; if (i >= j) a += (i == j ? 1.0 : 2.0) * X[e] * Y[e]; }
    return block_sum(a, sh);
}
// in-CTA Cholesky X = L L' (lower, upper triangle zeroed); false for a non-positive pivot
__device__ bool s_chol(double *X, int ms) {
    __shared__ int ok;
    __syncthreads();                                  // every thread has read the previous call's ok
    if (threadIdx.x == 0) ok = 1;
    for (int j = 0; j < ms; ++j) {
        __syncthreads();
        if (threadIdx.x == 0) { const double d = X[j + j * ms]; if (!(d > 0.0)) ok = 0; X[j + j * ms] = sqrt(d); }
        __syncthreads();
        for (int i = j + 1 + threadIdx.x; i < ms; i += SB_T) X[i + j * ms] /= X[j + j * ms];
        __syncthreads();
        for (int e = threadIdx.x; e < ms * ms; e += SB_T) {
            const int i = e % ms, c = e / ms;
            if (c > j && i >= c) X[e] -= X[i + j * ms] * X[c + j * ms];
        }
    }
    __syncthreads();
    SB_FOR(e, ms) if (e % ms < e / ms) X[e] = 0.0;
    __syncthreads();
    return ok;
}
// SVD A = U diag(sig) V' of the block in A by cone.cuh's one-sided Jacobi (A := U, one warp per column pair, a column
// one element per lane); false when the sweeps ran out or a singular value is not positive
__device__ bool s_svd(double *A, double *V, double *sig, int ms) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    SB_FOR(e, ms) V[e] = (e % ms == e / ms) ? 1.0 : 0.0;
    __syncthreads();
    __shared__ int rot;
    const bool conv = jacobi_svd_cta(ms, A, V, JAC_SWEEPS, rot);
    __shared__ int ok;
    if (threadIdx.x == 0) ok = conv;
    __syncthreads();
    for (int j = warp; j < ms; j += SB_T / 32) {
        const double x = lane < ms ? A[j * ms + lane] : 0.0, nrm = sqrt(warp_sum(x * x));
        if (lane < ms) A[j * ms + lane] = x / nrm;
        if (lane == 0) { sig[j] = nrm; if (!(nrm > 0.0)) ok = 0; }
    }
    __syncthreads();
    return ok;
}
// eigendecomposition of the symmetric block in A = V diag(ev) V' by cone.cuh's two-sided Jacobi (jac_eig_cta, with
// jac_small_kernel's convergence rule); W is its second buffer, A and W are overwritten; false when the sweeps ran out
__device__ bool s_eig(double *A, double *W, double *V, double *ev, int ms, double *sh) {
    SB_FOR(e, ms) V[e] = (e % ms == e / ms) ? 1.0 : 0.0;
    __syncthreads();
    double *w0 = A, *w1 = W;
    const bool ok = jac_eig_cta<true>(w0, w1, V, ms, JAC_SWEEPS, sh, threadIdx.x, SB_T);
    for (int i = threadIdx.x; i < ms; i += SB_T) ev[i] = w0[i + i * ms];
    __syncthreads();
    return ok;
}
__device__ double s_min(const double *ev, int ms) {
    double t = INFINITY;
    for (int i = 0; i < ms; ++i) t = fmin(t, ev[i]);
    return t;
}
// write X (both triangles) to x
__device__ void s_store(double *x, const double *X, int ms) { SB_FOR(e, ms) x[e] = X[e]; }
__device__ __forceinline__ double s_lam(const Ptrs &p, long long om, int so, int ms, int i) {
    return p.lmbda[om + so + i * (ms + 1)];
}

// bzp := pack(W^{-T} z) = pack(rti' z rti) (mode 0; mode 1 also th := bzp, the x1 solve's W^{-T} h), or f4_no_ir's
// steps before the solve (mode 2): s := lmbda o\ s, z := z - W' s = z - r s r', bzp := pack(rti' z rti) (misc.py
// :1305-1307, coneprog.py :1154-1165).  z and s of slot b at z + b*sz, s + b*ss.
__global__ void __launch_bounds__(SB_T) k_s_wtz(Ptrs p, const double *z, long long sz, double *s, long long ss,
                                                int mode) {
    SB_SETUP
    __shared__ double R[SMX], X[SMX], Y[SMX], T[SMX];
    s_load(X, z + b * sz + so, ms);
    if (mode == 2) {
        double *sb = s + b * ss + so;
        s_load(Y, sb, ms);
        SB_FOR(e, ms) Y[e] /= 0.5 * (s_lam(p, om, so, ms, e % ms) + s_lam(p, om, so, ms, e / ms));
        __syncthreads();
        s_store(sb, Y, ms);
        SB_FOR(e, ms) R[e] = p.sr[oc + sro + e];
        __syncthreads();
        s_mm(T, Y, false, R, true, ms);
        s_mm(Y, R, false, T, false, ms);              // Y := r s r'
        SB_FOR(e, ms) X[e] -= Y[e];
        __syncthreads();
    }
    SB_FOR(e, ms) R[e] = p.srti[oc + sro + e];
    __syncthreads();
    s_congr(Y, R, X, T, true, ms);
    s_store_packed(p.bzp + om + sp, Y, ms);
    if (mode == 1) s_store_packed(p.th + om + sp, Y, ms);
}
// Gs = pack(W^{-T} G) for the 's' rows (misc.py:1267-1272): column j of Gs is pack(rti' mat(g_j) rti); grid.z
// splits the columns
__global__ void __launch_bounds__(SB_T) k_s_build_gs(Ptrs p, const double *G, double *Gs, long long ldg, long long sG) {
    SB_SETUP
    __shared__ double R[SMX], X[SMX], Y[SMX], T[SMX];
    SB_FOR(e, ms) R[e] = p.srti[oc + sro + e];
    __syncthreads();
    const int per = (p.n + gridDim.z - 1) / gridDim.z, j0 = blockIdx.z * per, j1 = min(p.n, j0 + per);
    for (int j = j0; j < j1; ++j) {
        const long long off = (long long)b * sG + (long long)j * ldg;
        s_load(X, G + off + so, ms);
        s_congr(Y, R, X, T, true, ms);
        s_store_packed(Gs + off + sp, Y, ms);
        __syncthreads();
    }
}
// NT scaling (misc.py:374-417): s = Ls Ls', z = Lz Lz', Lz' Ls = U diag(lambda) V',
// r = Lz^{-T} U diag(lambda)^{1/2}, rti = Lz U diag(lambda)^{-1/2}.  part[3] = 1 when a factorisation failed.
// ALL: every slot (the adjoint's scaling at the returned iterate); else the slots still running
template <bool ALL> __device__ __forceinline__ void s_nt_compute(const Ptrs &p) {
    SB_SETUP
    SB_PART;
    __shared__ double Ls[SMX], Lz[SMX], U[SMX], V[SMX], lam[CVXB_BATCH_SMAX];
    if (!ALL && S.done) return;
    s_load(Ls, p.s + om + so, ms);
    s_load(Lz, p.z + om + so, ms);
    bool ok = s_chol(Ls, ms);
    ok = s_chol(Lz, ms) && ok;
    s_mm(U, Lz, true, Ls, false, ms);
    ok = s_svd(U, V, lam, ms) && ok;
    // V := Lz^{-T} U (one column per thread), Ls := Lz U
    for (int c = threadIdx.x; c < ms; c += SB_T)
        for (int i = ms - 1; i >= 0; --i) {
            double a = U[i + c * ms];
            for (int l = i + 1; l < ms; ++l) a -= Lz[l + i * ms] * V[l + c * ms];
            V[i + c * ms] = a / Lz[i + i * ms];
        }
    __syncthreads();
    s_mm(Ls, Lz, false, U, false, ms);
    SB_FOR(e, ms) {
        const double a = sqrt(lam[e / ms]);
        p.sr[oc + sro + e] = V[e] * a;
        p.srti[oc + sro + e] = Ls[e] * (1.0 / a);
    }
    for (int i = threadIdx.x; i < ms; i += SB_T) p.lmbda[om + so + i * (ms + 1)] = ok ? lam[i] : NAN;
    if (tid == 0) part[3] = ok ? 0.0 : 1.0;        // a failed Cholesky or SVD stops the problem (k_update)
}
// at iteration 0
__global__ void __launch_bounds__(SB_T) k_s_nt_compute(Ptrs p) { s_nt_compute<false>(p); }
// the starting point's smallest eigenvalues (misc.max_step, coneprog.py:707, :737): s (unpacked), z (bzp, packed)
__global__ void __launch_bounds__(SB_T) k_s_eig_start(Ptrs p) {
    SB_SETUP
    SB_PART;
    __shared__ double A[SMX], W[SMX], V[SMX], ev[CVXB_BATCH_SMAX], sh[32];
    s_load(A, p.s + om + so, ms);
    const bool ok1 = s_eig(A, W, V, ev, ms, sh);
    const double m1 = s_min(ev, ms);
    s_load_packed(A, p.bzp + om + sp, ms);
    const bool ok2 = s_eig(A, W, V, ev, ms, sh);
    if (tid == 0) { part[1] = ok1 ? m1 : NAN; part[2] = ok2 ? s_min(ev, ms) : NAN; }
}
// k_s_eig_start for a loaded start, whose s and z are both unpacked (k_warm_copy)
__global__ void __launch_bounds__(SB_T) k_s_eig_warm(Ptrs p) {
    SB_SETUP
    SB_PART;
    __shared__ double A[SMX], W[SMX], V[SMX], ev[CVXB_BATCH_SMAX], sh[32];
    s_load(A, p.s + om + so, ms);
    const bool ok1 = s_eig(A, W, V, ev, ms, sh);
    const double m1 = s_min(ev, ms);
    s_load(A, p.z + om + so, ms);
    const bool ok2 = s_eig(A, W, V, ev, ms, sh);
    if (tid == 0) { part[1] = ok1 ? m1 : NAN; part[2] = ok2 ? s_min(ev, ms) : NAN; }
}
// the 's' rows of the refinement residual res() (coneprog.py:599-631): wz3 = W^{-1} dz = rti dz rti',
// wz2 = wz + ut h - W' ds = wz + ut h - r ds r', ws2 = ws - lmbda o (dz + ds); part[0] = sdot(h, wz3).
// A QP batch (LP = false) has no embedding: coneqp's res() (coneprog.py:1930-1960) is the same without ut and h'wz3
template <bool LP> __global__ void __launch_bounds__(SB_T) k_s_res(Ptrs p) {
    SB_SETUP
    SB_PART;
    __shared__ double R[SMX], X[SMX], Y[SMX], T[SMX], H[SMX], sh[32];
    const double ut = LP ? lp_scal(p, oc).dtau / lp_scal(p, oc).dg : 0.0;
    s_load(X, p.dz + om + so, ms);
    if (LP) s_load(H, p.h + om + so, ms);
    SB_FOR(e, ms) R[e] = p.srti[oc + sro + e];
    __syncthreads();
    s_congr(Y, R, X, T, false, ms);
    s_store(p.wz3 + oc + so, Y, ms);
    const double hz = LP ? s_dot(H, Y, ms, sh) : 0.0;
    s_load(Y, p.ds + om + so, ms);
    SB_FOR(e, ms) { R[e] = p.sr[oc + sro + e]; X[e] += Y[e]; }      // X := dz + ds
    __syncthreads();
    s_mm(T, Y, false, R, true, ms);
    s_mm(Y, R, false, T, false, ms);                                 // Y := W' ds = r ds r'
    SB_FOR(e, ms) {
        const int i = e % ms, j = e / ms, lo = i >= j ? e : j + i * ms;
        p.wz2[oc + so + e] = (LP ? p.wz[oc + so + lo] + ut * H[e] : p.wz[oc + so + lo]) - Y[e];
        p.ws2[oc + so + e] = p.ws[oc + so + lo] - 0.5 * (s_lam(p, om, so, ms, i) + s_lam(p, om, so, ms, j)) * X[e];
    }
    if (LP && tid == 0) part[0] = hz;
}
// after the i-th direction (coneprog.py:1302-1321): part[0] = sdot(ds, dz); i = 0: ws3 = ds o dz; ds and dz scaled
// by lambda^{-1/2} on both sides (scale2); part[1], part[2] their smallest eigenvalues; i = 1 also leaves the
// eigenvectors in ds and dz and the eigenvalues in sigs and sigz
__global__ void __launch_bounds__(SB_T) k_s_dir_post(Ptrs p, int i) {
    SB_SETUP
    SB_PART;
    __shared__ double Ds[SMX], Dz[SMX], V[SMX], T[SMX], ev[CVXB_BATCH_SMAX], sh[32];
    double *ds = p.ds + om + so, *dz = p.dz + om + so;
    s_load(Ds, ds, ms);
    s_load(Dz, dz, ms);
    const double dsdz = s_dot(Ds, Dz, ms, sh);
    if (i == 0) {
        s_mm(T, Ds, false, Dz, false, ms);
        SB_FOR(e, ms) p.ws3[om + so + e] = 0.5 * (T[e] + T[e / ms + (e % ms) * ms]);
    }
    SB_FOR(e, ms) {
        const double c = sqrt(s_lam(p, om, so, ms, e % ms)) * sqrt(s_lam(p, om, so, ms, e / ms));
        Ds[e] /= c; Dz[e] /= c;
    }
    __syncthreads();
    bool ok = s_eig(Ds, T, V, ev, ms, sh);
    const double m1 = s_min(ev, ms);
    if (i == 1) {
        s_store(ds, V, ms);
        for (int j = tid; j < ms; j += SB_T) p.sigs[oc + sgo + j] = ev[j];
    }
    __syncthreads();
    ok = s_eig(Dz, T, V, ev, ms, sh) && ok;
    if (i == 1) {
        s_store(dz, V, ms);
        for (int j = tid; j < ms; j += SB_T) p.sigz[oc + sgo + j] = ev[j];
    }
    if (tid == 0) { part[0] = dsdz; part[1] = ok ? m1 : NAN; part[2] = ok ? s_min(ev, ms) : NAN; }
}
// a cpl batch's unscaled steps of the 's' blocks (cvxprog.py:1031-1034): dz2 = W^{-1} dz = rti dz rti' and
// ds2 = W' ds = r ds r' (m-vectors, slot b at + b*m), from the scaled ds and dz before k_s_dir_post replaces them
__global__ void __launch_bounds__(SB_T) k_s_steps(Ptrs p, double *ds2, double *dz2) {
    SB_SETUP
    __shared__ double R[SMX], X[SMX], Y[SMX], T[SMX];
    if (S.done) return;
    s_load(X, p.dz + om + so, ms);
    SB_FOR(e, ms) R[e] = p.srti[oc + sro + e];
    __syncthreads();
    s_congr(Y, R, X, T, false, ms);
    s_store(dz2 + om + so, Y, ms);
    s_load(X, p.ds + om + so, ms);
    SB_FOR(e, ms) R[e] = p.sr[oc + sro + e];
    __syncthreads();
    s_congr(Y, R, X, T, false, ms);
    s_store(ds2 + om + so, Y, ms);
}
// after k_s_dir_post in a cpl batch: each block's eigenpairs of ds (sigs) and of dz (sigz) in ascending order, as
// max_step's syevd leaves them (misc.py:1046).  The update pairs sigs[i] with the i-th eigenvector, and after a resumed
// line search those come from different directions (cvxprog.py:1238-1261), so the order is part of the result.  NaN
// sorts last, so that the ranks are a permutation whatever the values
__global__ void __launch_bounds__(SB_T) k_s_sort(Ptrs p) {
    SB_SETUP
    __shared__ double V[SMX], ev[CVXB_BATCH_SMAX];
    __shared__ int rk[CVXB_BATCH_SMAX];
    if (S.done) return;
    for (int w = 0; w < 2; ++w) {
        double *x = (w ? p.dz : p.ds) + om + so, *sg = (w ? p.sigz : p.sigs) + oc + sgo;
        SB_FOR(e, ms) V[e] = x[e];
        for (int j = tid; j < ms; j += SB_T) ev[j] = sg[j];
        __syncthreads();
        for (int j = tid; j < ms; j += SB_T) {
            int r = 0;
            for (int i = 0; i < ms; ++i) {
                const double a = ev[i], c = ev[j];
                const bool na = isnan(a), nc = isnan(c);
                r += na != nc ? nc : (na || a == c) ? i < j : a < c;
            }
            rk[j] = r;
        }
        __syncthreads();
        SB_FOR(e, ms) x[e % ms + rk[e / ms] * ms] = V[e];
        for (int j = tid; j < ms; j += SB_T) sg[rk[j]] = ev[j];
        __syncthreads();
    }
}
// the update (coneprog.py:1365-1433, misc.py:592-634): Ls = diag(l)^{1/2} Qs diag(l)^{1/2} diag((1 + step sigs) / l)^{1/2},
// likewise Lz; r := r Ls V diag(lambda+)^{-1/2}, rti := rti Lz U diag(lambda+)^{-1/2} with Lz' Ls = U diag(lambda+) V';
// s = r diag(lambda+) r', z = rti diag(lambda+) rti'.  The results are staged in the block's rows of d (r), di (rti),
// ds (s), dz (z) and the diagonal rows of lmbdasq (lambda), which the 's' rows do not otherwise use at this point;
// k_update commits them only when every block of the problem succeeded, so a problem that stops keeps one
// iterate.  part[3] = 1 when the SVD failed (first: also when k_s_nt_compute failed, which skips the update).
template <bool EQ> __global__ void __launch_bounds__(SB_T) k_s_update(Ptrs p, const int *info, int first) {
    SB_SETUP
    SB_PART;
    __shared__ double M0[SMX], M1[SMX], M2[SMX], M3[SMX], M4[SMX], lam[CVXB_BATCH_SMAX];
    if (S.done || info[b] > 0 || (EQ && p.infop[b] > 0) || (first && part[3] != 0.0)) return;
    const double step = S.step;
    SB_FOR(e, ms) {
        const int i = e % ms, j = e / ms;
        const double li = s_lam(p, om, so, ms, i), lj = s_lam(p, om, so, ms, j), c = sqrt(li) * sqrt(lj);
        const double gs = (step * p.sigs[oc + sgo + j] + 1.0) / lj, gz = (step * p.sigz[oc + sgo + j] + 1.0) / lj;
        M2[e] = p.ds[om + so + e] * c * sqrt(gs);
        M3[e] = p.dz[om + so + e] * c * sqrt(gz);
        M0[e] = p.sr[oc + sro + e];
        M1[e] = p.srti[oc + sro + e];
    }
    __syncthreads();
    s_mm(M4, M0, false, M2, false, ms);           // r Ls
    s_mm(M0, M1, false, M3, false, ms);           // rti Lz
    s_mm(M1, M3, true, M2, false, ms);            // Lz' Ls = U diag(lambda+) V'
    const bool ok = s_svd(M1, M2, lam, ms);
    s_mm(M3, M4, false, M2, false, ms);           // r Ls V
    s_mm(M4, M0, false, M1, false, ms);           // rti Lz U
    if (tid == 0) part[3] = ok ? 0.0 : 1.0;
    if (!ok) return;
    SB_FOR(e, ms) {
        const double a = 1.0 / sqrt(lam[e / ms]);
        M3[e] *= a; M4[e] *= a;
        p.d[om + so + e] = M3[e]; p.di[om + so + e] = M4[e];
    }
    __syncthreads();
    SB_FOR(e, ms) {                               // lower triangle, mirrored: s and z are returned exactly symmetric
        const int i = e % ms, j = e / ms;
        if (i < j) continue;
        double a = 0.0, c = 0.0;
        for (int l = 0; l < ms; ++l) { a += M3[i + l * ms] * lam[l] * M3[j + l * ms]; c += M4[i + l * ms] * lam[l] * M4[j + l * ms]; }
        p.ds[om + so + e] = a; p.dz[om + so + e] = c;
        p.ds[om + so + j + i * ms] = a; p.dz[om + so + j + i * ms] = c;
    }
    for (int i = tid; i < ms; i += SB_T) p.lmbdasq[om + so + i * (ms + 1)] = lam[i];
}

// ---- geometric programs: cvxprog.gp -> cp -> cpl (cvxprog.py:1967-2155, :1746-1964, :556-1356) ----
// gp solves the epigraph problem of cp with cpl: the variable is (x, t), the objective t, the nonlinear rows are
// f0(x) - t, f1(x), ..., fmnl(x) with fi = log sum exp(Fi x + gi), and the 'l' rows G x <= h.  Every row is diagonally
// scaled.  The m-vectors hold rows [f1..fmnl; 'l'] (m = mnl + ml); the epigraph row f0 - t and t itself are scalars
// of GPScal.  The batch's G holds [Df[1:]; G] in rows [0, m) (the KKT operand kkt_chol2 scales by [dnli; di]) and F in
// rows [m, m + sum K); P holds H = sum_i z_i Fi'(diag(yi) - yi yi')Fi.  kktsolver_e (:1890-1943) eliminates t around
// one batch_solve.  Per-slot scalars and the relaxed line search's saved state live in the state row.
struct GPScal {
    double t, dt, s0, z0, ds0, dz0, ds20, dz20, l0, lsq0, d0, di0, rxt, rz0, a;   // epigraph row and t
    double wxt, wx2t, wz0, ws0, wz20, ws20, wz30;                                  // refinement copies
    double resznl, resx0, resznl0, pres0, th1, th2, th3, phi, dphi, relaxed, searching;
    double nt, ns0, nz0;                                                           // line-search trial
    // the saved state of a series of relaxed line searches (:1190-1215)
    double phi0, dphi0, gap0, step0, dsdz0, sigma0, eta0;
    double t0, dt0, s00, z00, ds00, dz00, ds200, dz200, l00, d00, di00, rxt0, rz00;
};
struct GPPtrs {
    int nK, sumK, mnl;
    long long ldg, sG, ldh, sH;
    const int *koff;                 // nK + 1 row offsets of the blocks Fi in F
    double *G;                       // per slot [Df[1:]; G; F], ld ldg
    // per slot, rebuilt every iteration: H's scaled rows (sum K x n, ld ldh) and their weights z_i, y = F x + g and
    // then the softmax, w = z_i y, f, grad f0, the unscaled steps ds2 / dz2 and the line search's trial point
    double *Hr, *hw, *yv, *wv, *fv, *gf0, *ds2, *dz2, *nx, *ny, *nz, *ns, *nrx;
    // in the state row: g (sum K), GPScal, and the saved vectors
    double *g, *gs, *x0, *dx0, *rx0, *y0, *dy0, *ry0, *s0, *z0, *ds0, *dz0, *ds20, *dz20, *l0, *d0, *di0, *rz0;
};
// the 'q' part of W that a cpl batch's relaxed line search saves with the rest (cvxprog.py:1196-1198): v (sum q) and
// beta (nq) in the state row, and with 's' blocks r and rti (sum s² each, :1199-1201).  A kernel's last argument, so
// that the GP and CP kernels' other arguments stay where they are
struct QSave {
    double *v0, *beta0, *r0, *rti0;
};
constexpr int GP_MAX_RELAXED = 8;
constexpr double GP_ALPHA = 0.01, GP_BETA = 0.5, GP_STEP = 0.99;
__device__ __forceinline__ GPScal &gp_scal(const GPPtrs &g, long long oc) {
    return *reinterpret_cast<GPScal *>(g.gs + oc);
}
#define GP_SETUP                                                                                       \
    PB_SETUP                                                                                           \
    GPScal &T = gp_scal(g, oc);                                                                        \
    const long long ok = (long long)b * g.sumK;                                                        \
    (void)T; (void)ok;

// the starting point (:556-570): x = 0, t = 0, y = 0, s = z = e, relaxed_iters = 0.  CONES: e is 1 at each cone's
// first row and 0 in the rest of it.  SDP: the identity in each 's' block (its diagonal rows)
template <bool CONES, bool SDP = false> __global__ void k_gp_init(Ptrs p, GPPtrs g) {
    GP_SETUP
    for (int i = tid; i < p.n; i += nt) p.x[on + i] = 0.0;
    for (int i = tid; i < p.neq; i += nt) p.y[oq + i] = 0.0;
    for (int i = tid; i < p.m; i += nt) {
        double e = !CONES || i < p.ml ? 1.0 : 0.0;
        if (SDP) e = i < p.ml || (i >= p.mlq && p.rw[i] == 1.0) ? 1.0 : 0.0;
        p.s[om + i] = e; p.z[om + i] = e;
    }
    if (CONES) {
        __syncthreads();
        for (int k = tid; k < p.nq; k += nt) { p.s[om + p.qoff[k]] = 1.0; p.z[om + p.qoff[k]] = 1.0; }
    }
    if (tid == 0) {
        T = GPScal{};
        T.s0 = 1.0; T.z0 = 1.0;
    }
}
// F(x) of gp (:2102-2153) for block i of slot b, grid (nK, Bact): yv holds F x on entry; y := softmax(F x + g),
// f_i = max + log sum exp, w = z_i y (z_i from z, or from the trial point's nz).  FULL: also Df_i = Fi' y (grad f0 or
// row i - 1 of G), H's rows sqrt(y_k)(F_k - Df_i) and their weights z_i.  trial: only slots still searching.
// ADJ (k_adj_gp_op, FULL): every slot, z_0 = 1, and neither w nor grad f0, which the adjoint does not read
template <bool FULL, bool ADJ> __device__ __forceinline__ void gp_eval_body(const Ptrs &p, const GPPtrs &g, int trial) {
    const int i = blockIdx.x, b = blockIdx.y, tid = threadIdx.x, nt = blockDim.x;
    const int lane = tid & 31, warp = tid >> 5, nwarp = nt >> 5;
    __shared__ double sh[32];
    const GPScal &T = gp_scal(g, (long long)b * p.L);
    if (!ADJ && (p.sc[b].done || (trial && T.searching == 0.0))) return;
    const int k0 = g.koff[i], K = g.koff[i + 1] - k0;
    const long long ok = (long long)b * g.sumK + k0;
    const double *F = g.G + (long long)b * g.sG + p.m + k0, *gv = g.g + (long long)b * p.L + k0;
    double *y = g.yv + ok;
    double mx = -INFINITY;
    for (int k = tid; k < K; k += nt) { const double v = y[k] + gv[k]; y[k] = v; mx = fmax(mx, v); }
    mx = -block_min(-mx, sh);
    double sum = 0.0;
    for (int k = tid; k < K; k += nt) { const double e = exp(y[k] - mx); y[k] = e; sum += e; }
    sum = block_sum(sum, sh);
    const double r = 1.0 / sum;
    const double *zs = trial ? g.nz : p.z;
    const double zi = i == 0 ? (ADJ ? 1.0 : trial ? T.nz0 : T.z0) : zs[(long long)b * p.m + i - 1];
    for (int k = tid; k < K; k += nt) {
        const double v = y[k] * r;
        y[k] = v;
        if (!ADJ) g.wv[ok + k] = zi * v;
        if (FULL) g.hw[ok + k] = zi;
    }
    if (tid == 0) g.fv[(long long)b * g.nK + i] = mx + log(sum);
    if (!FULL) return;
    __syncthreads();
    double *hr = g.Hr + (long long)b * g.sH + k0;
    for (int j = warp; j < p.n; j += nwarp) {           // one warp per column of Fi, its lanes down the rows
        const double *Fj = F + (long long)j * g.ldg;
        double a = 0.0;
        for (int k = lane; k < K; k += 32) a += Fj[k] * y[k];
        a = warp_sum(a);
        if (lane == 0) {
            if (i == 0) { if (!ADJ) g.gf0[(long long)b * p.n + j] = a; }
            else g.G[(long long)b * g.sG + (i - 1) + (long long)j * g.ldg] = a;
        }
        for (int k = lane; k < K; k += 32) hr[k + (long long)j * g.ldh] = sqrt(y[k]) * (Fj[k] - a);
    }
}
template <bool FULL> __global__ void k_gp_eval(Ptrs p, GPPtrs g, int trial) { gp_eval_body<FULL, false>(p, g, trial); }
// residuals, part 1 (:668-691): rx = 0 (the GEMVs add Df'znl + G'zl + A'y), rxt = 1 - z0; rz = s + f on the
// nonlinear rows, s - h on the 'l' rows (G x follows); rznl's epigraph row s0 + f0 - t; EQ: ry = b (A x - ry follows).
// Without the epigraph row (EPI false, a cpl batch): rx = c, and f has no objective entry
template <bool EQ, bool EPI = true> __global__ void k_gp_res_begin(Ptrs p, GPPtrs g) {
    GP_SETUP
    if (S.done) return;
    const double *f = g.fv + (long long)b * g.nK;
    for (int i = tid; i < p.n; i += nt) p.rx[on + i] = EPI ? 0.0 : p.q[on + i];
    for (int i = tid; i < p.m; i += nt)
        p.rz[om + i] = i < g.mnl ? p.s[om + i] + f[i + (EPI ? 1 : 0)] : p.s[om + i] - p.h[om + i];
    if (EQ) for (int i = tid; i < p.neq; i += nt) p.ry[oq + i] = p.beq[oq + i];
    if (EPI && tid == 0) { T.rxt = -T.z0 + 1.0; T.rz0 = T.s0 + (f[0] - T.t); }
}
// statistics and stopping rule (:693-755); iteration 0 fixes resx0, resznl0, pres0, dres0 and the merit weights.
// EPI false: pcost = c'x, and no epigraph row in gap, resx, resznl and dcost.  'q' rows are 'l' rows here: snrm2 and
// sdot are the 2-norm and the dot product on them.  SDP: they weigh the 's' rows (rw), so only the lower triangles count
template <bool EQ, bool EPI = true, bool SDP = false>
__global__ void k_gp_stats(Ptrs p, GPPtrs g, int iter, int maxiters, double abstol, double reltol, double feastol,
                           int *ndone, int *doneflags) {
    GP_SETUP
    if (!S.done) {
        double rx2 = 0, ry2 = 0, yry = 0, rn2 = 0, rl2 = 0, zrn = 0, zrl = 0, gap = 0, cx = 0;
        for (int i = tid; i < p.n; i += nt) {
            const double v = p.rx[on + i]; rx2 += v * v;
            if (!EPI) cx += p.q[on + i] * p.x[on + i];
        }
        if (EQ) for (int i = tid; i < p.neq; i += nt) { const double v = p.ry[oq + i]; ry2 += v * v; yry += p.y[oq + i] * v; }
        for (int i = tid; i < p.m; i += nt) {
            const double v = p.rz[om + i], zv = p.z[om + i];
            if (SDP) {
                const double w = p.rw[i];
                if (i < g.mnl) { rn2 += v * v; zrn += zv * v; } else { rl2 += w * v * v; zrl += w * zv * v; }
                gap += w * p.s[om + i] * zv;
                continue;
            }
            if (i < g.mnl) { rn2 += v * v; zrn += zv * v; } else { rl2 += v * v; zrl += zv * v; }
            gap += p.s[om + i] * zv;
        }
        rx2 = block_sum(rx2, sh); rn2 = block_sum(rn2, sh); rl2 = block_sum(rl2, sh);
        zrn = block_sum(zrn, sh); zrl = block_sum(zrl, sh); gap = block_sum(gap, sh);
        if (EQ) { ry2 = block_sum(ry2, sh); yry = block_sum(yry, sh); }
        if (!EPI) cx = block_sum(cx, sh);
        if (tid == 0) {
            if (EPI) gap += T.s0 * T.z0;
            const double resx = EPI ? sqrt(rx2 + T.rxt * T.rxt) : sqrt(rx2), resy = sqrt(ry2);
            const double resznl = EPI ? sqrt(rn2 + T.rz0 * T.rz0) : sqrt(rn2), reszl = sqrt(rl2);
            const double pcost = EPI ? T.t : cx;         // EPI: c'(x, t) with c = (0, 1)
            const double dcost = EPI ? pcost + yry + (zrn + T.z0 * T.rz0) + zrl - gap : pcost + yry + zrn + zrl - gap;
            S.pcost = pcost; S.dcost = dcost; S.gap = gap; S.resx = resx; S.resy = resy; S.resz = reszl;
            T.resznl = resznl;
            if (pcost < 0.0) { S.relgap = gap / -pcost; S.relgap_valid = 1; }
            else if (dcost > 0.0) { S.relgap = gap / dcost; S.relgap_valid = 1; }
            else { S.relgap = 0.0; S.relgap_valid = 0; }
            const double pres = sqrt(resy * resy + resznl * resznl + reszl * reszl);
            if (iter == 0) {
                T.resx0 = fmax(1.0, resx); T.resznl0 = fmax(1.0, resznl);
                T.pres0 = fmax(1.0, pres); S.resx0 = fmax(1.0, resx);          // dres0
                T.th1 = 1.0 / gap; T.th2 = 1.0 / T.resx0; T.th3 = 1.0 / T.resznl0;
            }
            S.pres = pres / T.pres0; S.dres = resx / S.resx0;
            const bool opt = S.pres <= feastol && S.dres <= feastol &&
                             (gap <= abstol || (S.relgap_valid && S.relgap <= reltol));
            if (opt || iter == maxiters) { S.done = 1; S.iters = iter; S.status = opt ? 1 : 2; }
        }
    }
    if (tid == 0) {
        if (S.done) atomicAdd(ndone, 1);
        doneflags[b] = S.done;
    }
}
// the scaling at iteration 0 (misc.py:compute_scaling, dnl and d alike) and lambda o lambda every iteration;
// di2 = di² is the SYRK's weight of [Df[1:]; G]
__global__ void k_gp_scaling(Ptrs p, GPPtrs g, int first) {
    GP_SETUP
    if (S.done) return;
    for (int i = tid; i <= p.m; i += nt) {
        const bool e = i == p.m;                         // the epigraph row
        double &l = e ? T.l0 : p.lmbda[om + i];
        if (first) {
            const double s = e ? T.s0 : p.s[om + i], z = e ? T.z0 : p.z[om + i];
            const double d = sqrt(s / z), di = 1.0 / d;
            if (e) { T.d0 = d; T.di0 = di; }
            else { p.d[om + i] = d; p.di[om + i] = di; p.di2[om + i] = di * di; }
            l = sqrt(s * z);
        }
        if (e) T.lsq0 = l * l; else p.lmbdasq[om + i] = l * l;
    }
    if (tid == 0) { S.sigma = 0.0; S.eta = 0.0; }       // :966
}
// the i-th Newton right-hand side (:978-1002), its refinement copy (:940-944) and f4_no_ir's steps before the solve
// (:868-876): s := lmbda o\ s, z := z - W's.  Then kktsolver_e's (:1933-1937): a = z[0], ux = bx + bt grad f0 (in dx),
// bzp = W^{-T} z[1:]
__global__ void k_gp_dir_rhs(Ptrs p, GPPtrs g) {
    GP_SETUP
    if (S.done) return;
    const double mu = S.gap / (p.m + 1), sm = S.sigma * mu, c = -1.0 + S.eta;
    const double dt = c * T.rxt;
    const bool ref = p.refinement > 0;
    for (int k = tid; k < p.n; k += nt) {
        const double v = c * p.rx[on + k];
        if (ref) p.wx[oc + k] = v;
        p.dx[on + k] = v + dt * g.gf0[on + k];
    }
    for (int k = tid; k < p.neq; k += nt) {
        const double v = c * p.ry[oq + k];
        p.dy[oq + k] = v;
        if (ref) p.wy[oc + k] = v;
    }
    for (int k = tid; k <= p.m; k += nt) {
        const bool e = k == p.m;
        double s = -(e ? T.lsq0 : p.lmbdasq[om + k]) + sm, z = c * (e ? T.rz0 : p.rz[om + k]);
        if (e) {
            if (ref) { T.ws0 = s; T.wz0 = z; T.wxt = dt; }
            s = s / T.l0; z = z - T.d0 * s;
            T.ds0 = s; T.a = z; T.dt = dt;
        } else {
            if (ref) { p.ws[oc + k] = s; p.wz[oc + k] = z; }
            s = s / p.lmbda[om + k]; z = z - p.d[om + k] * s;
            p.ds[om + k] = s; p.bzp[om + k] = p.di[om + k] * z;
        }
    }
}
// f4_no_ir's steps before a refinement solve, on (wx2, wx2t, wz2, ws2): as k_gp_dir_rhs's
__global__ void k_gp_f4_pre(Ptrs p, GPPtrs g) {
    GP_SETUP
    if (S.done) return;
    const double bt = T.wx2t;
    for (int k = tid; k < p.n; k += nt) p.wx2[oc + k] += bt * g.gf0[on + k];
    for (int k = tid; k <= p.m; k += nt) {
        if (k == p.m) {
            const double s = T.ws20 / T.l0;
            T.ws20 = s; T.a = T.wz20 - T.d0 * s;
        } else {
            const double s = p.ws2[oc + k] / p.lmbda[om + k], z = p.wz2[oc + k] - p.d[om + k] * s;
            p.ws2[oc + k] = s; p.bzp[om + k] = p.di[om + k] * z;
        }
    }
}
// after batch_solve (kktsolver_e :1938-1941, f4_no_ir :883): z[0] = -bt dnl[0], z[1:] = W uz, t = grad f0'ux +
// dnl[0]² bt - a, s := s - z.  acc = 0: the direction, in (dx, dt, dz, ds).  acc = 1: a refinement step on
// (wx2, wx2t, wz2, ws2), added to the direction (:953-956)
__global__ void k_gp_f4_post(Ptrs p, GPPtrs g, int acc) {
    GP_SETUP
    if (S.done) return;
    const double *ux = acc ? p.wx2 + oc : p.dx + on;
    double a = 0.0;
    for (int k = tid; k < p.n; k += nt) a += g.gf0[on + k] * ux[k];
    a = block_sum(a, sh);
    for (int k = tid; k < p.m; k += nt) {
        const double z = p.bzp[om + k];
        if (acc) {
            const double s = p.ws2[oc + k] - z;
            p.wz2[oc + k] = z; p.ws2[oc + k] = s;
            p.dz[om + k] += z; p.ds[om + k] += s;
        } else {
            p.dz[om + k] = z; p.ds[om + k] -= z;
        }
    }
    if (acc) {
        for (int k = tid; k < p.n; k += nt) p.dx[on + k] += ux[k];
        for (int k = tid; k < p.neq; k += nt) p.dy[oq + k] += p.wy2[oc + k];
    }
    if (tid == 0) {
        const double bt = acc ? T.wx2t : T.dt, d0 = T.d0;
        const double z0 = -bt * d0, t = a + d0 * d0 * bt - T.a;
        if (acc) {
            const double s0 = T.ws20 - z0;
            T.wz20 = z0; T.ws20 = s0; T.wx2t = t;
            T.dz0 += z0; T.ds0 += s0; T.dt += t;
        } else {
            T.dz0 = z0; T.ds0 -= z0; T.dt = t;
        }
    }
}
// refinement residual, the elementwise part of res() (:889-923): wx2 = wx - grad f0 wz3[0], wx2t = 2 wxt + wz3[0]
// (cp's H_e doubles v[1], :1812), wz3 = W^{-1} dz, wz2 = wz - W' ds (and the epigraph row's - (grad f0'dx - dt)),
// ws2 = ws - lmbda o (dz + ds); EQ: wy2 = wy.  The H, A, A', [Df[1:]; G] and its transpose products follow as GEMVs
__global__ void k_gp_res(Ptrs p, GPPtrs g) {
    GP_SETUP
    if (S.done) return;
    double a = 0.0;
    for (int k = tid; k < p.n; k += nt) a += g.gf0[on + k] * p.dx[on + k];
    a = block_sum(a, sh);
    const double w30 = T.di0 * T.dz0;
    for (int k = tid; k < p.n; k += nt) p.wx2[oc + k] = p.wx[oc + k] - g.gf0[on + k] * w30;
    for (int k = tid; k < p.neq; k += nt) p.wy2[oc + k] = p.wy[oc + k];
    for (int k = tid; k < p.m; k += nt) {
        const double dz = p.dz[om + k], ds = p.ds[om + k];
        p.wz3[oc + k] = p.di[om + k] * dz;
        p.wz2[oc + k] = p.wz[oc + k] - p.d[om + k] * ds;
        p.ws2[oc + k] = p.ws[oc + k] - p.lmbda[om + k] * (ds + dz);
    }
    if (tid == 0) {
        T.wz30 = w30;
        T.wx2t = w30 + (T.wxt + T.wxt);
        T.wz20 = (T.wz0 - (a - T.dt)) - T.d0 * T.ds0;
        T.ws20 = T.ws0 - T.l0 * (T.ds0 + T.dz0);
    }
}
// after the i-th direction (:1030-1078): dsdz, the unscaled steps dz2 = W^{-1} dz and ds2 = W' ds, scale2 of ds and
// dz, the step to the boundary, phi and its directional derivative; the problem starts its line search.  CONES: sdot
// is the dot product on the 'q' rows too; each cone's warp forms its dz2 = W^{-1} dz, ds2 = W' ds, scale2 and max_step.
// SDP: k_s_steps and k_s_dir_post have done the 's' rows, whose ds and dz now hold eigenvectors; their sdot and
// smallest eigenvalues come from spart
template <bool EPI = true, bool CONES = false, bool SDP = false> __global__ void k_gp_dir_post(Ptrs p, GPPtrs g, int i) {
    GP_SETUP
    if (S.done) return;
    double dsdz = 0, mins = INFINITY, minz = INFINITY;
    for (int k = tid; k < (SDP ? p.mlq : p.m); k += nt) {
        const double ds = p.ds[om + k], dz = p.dz[om + k], l = p.lmbda[om + k];
        dsdz += ds * dz;
        if (CONES && k >= p.ml) continue;
        g.dz2[om + k] = p.di[om + k] * dz; g.ds2[om + k] = p.d[om + k] * ds;
        const double ss = ds / l, zs = dz / l;
        p.ds[om + k] = ss; p.dz[om + k] = zs;
        mins = fmin(mins, ss); minz = fmin(minz, zs);
    }
    if (CONES) {
        __syncthreads();                                 // every row's ds dz is in dsdz before the cones scale them
        const double *v = p.v + oc - p.ml, *beta = p.beta + oc, *l = p.lmbda + om;
        double *ds = p.ds + om, *dz = p.dz + om;
        FOR_CONES(o, len) {
            q_scale(wt, v + o, beta[k_], dz + o, g.dz2 + om + o, len, true);
            q_scale(wt, v + o, beta[k_], ds + o, g.ds2 + om + o, len, false);
            __syncwarp();
            q_scale2(wt, l + o, ds + o, len, false);
            q_scale2(wt, l + o, dz + o, len, false);
            __syncwarp();
            mins = fmin(mins, -q_max_step(wt, ds + o, len));
            minz = fmin(minz, -q_max_step(wt, dz + o, len));
        }
    }
    dsdz = block_sum(dsdz, sh);
    mins = block_min(mins, sh);
    minz = block_min(minz, sh);
    if (tid == 0) {
        if (SDP) for (int k = 0; k < p.ns; ++k) {
            const double *q = p.spart + ((long long)b * p.ns + k) * 4;
            dsdz += q[0]; mins = fmin(mins, q[1]); minz = fmin(minz, q[2]);
        }
        if (EPI) {
            dsdz += T.ds0 * T.dz0;
            T.dz20 = T.di0 * T.dz0; T.ds20 = T.d0 * T.ds0;
            T.ds0 /= T.l0; T.dz0 /= T.l0;
            mins = fmin(mins, T.ds0); minz = fmin(minz, T.dz0);
        }
        const double t = fmax(0.0, fmax(-mins, -minz));
        S.step = t == 0.0 ? 1.0 : fmin(1.0, GP_STEP / t);
        S.dsdz = dsdz;
        T.phi = T.th1 * S.gap + T.th2 * S.resx + T.th3 * T.resznl;
        T.dphi = i == 0 ? -T.phi
                        : -T.th1 * (1 - S.sigma) * S.gap - T.th2 * (1 - S.eta) * S.resx - T.th3 * (1 - S.eta) * T.resznl;
        T.searching = 1.0;
    }
}
// the line search's trial point (:1127-1130): (x, t, y, z, s) + step (dx, dt, dy, dz2, ds2); nrx = 0 (the GEMVs add
// newDf'newznl + G'newzl + A'newy)
__global__ void k_gp_trial(Ptrs p, GPPtrs g) {
    GP_SETUP
    if (S.done || T.searching == 0.0) return;
    const double st = S.step;
    for (int k = tid; k < p.n; k += nt) { g.nx[on + k] = p.x[on + k] + st * p.dx[on + k]; g.nrx[on + k] = 0.0; }
    for (int k = tid; k < p.neq; k += nt) g.ny[oq + k] = p.y[oq + k] + st * p.dy[oq + k];
    for (int k = tid; k < p.m; k += nt) {
        g.nz[om + k] = p.z[om + k] + st * g.dz2[om + k];
        g.ns[om + k] = p.s[om + k] + st * g.ds2[om + k];
    }
    if (tid == 0) { T.nt = T.t + st * T.dt; T.nz0 = T.z0 + st * T.dz20; T.ns0 = T.s0 + st * T.ds20; }
}
// copies of the state a relaxed line search saves (:1190-1214) and a resumed one restores (:1239-1260); `dir`: the
// step vectors too (not on the restore after a singular KKT matrix, :790-813, which restores the residuals instead).
// CONES: W's v and beta too (:1196-1198); SDP: W's r and rti (:1199-1201); EPI: the epigraph row's scalars.  The 's'
// rows of the vectors come with the rest; sigs and sigz are not saved, as in the reference
template <bool EPI = true, bool CONES = false, bool SDP = false>
__device__ void gp_save(const Ptrs &p, const GPPtrs &g, const QSave &qs, int b, bool save, bool dir, bool res) {
    const int tid = threadIdx.x, nt = blockDim.x;
    const long long on = (long long)b * p.n, om = (long long)b * p.m, oc = (long long)b * p.L, oq = (long long)b * p.neq;
    auto cp = [save](double *live, double *kept) { if (save) *kept = *live; else *live = *kept; };
    for (int k = tid; k < p.n; k += nt) {
        cp(p.x + on + k, g.x0 + oc + k);
        if (dir) cp(p.dx + on + k, g.dx0 + oc + k);
        if (res) cp(p.rx + on + k, g.rx0 + oc + k);
    }
    for (int k = tid; k < p.neq; k += nt) {
        cp(p.y + oq + k, g.y0 + oc + k);
        if (dir) cp(p.dy + oq + k, g.dy0 + oc + k);
        if (res) cp(p.ry + oq + k, g.ry0 + oc + k);
    }
    for (int k = tid; k < p.m; k += nt) {
        cp(p.s + om + k, g.s0 + oc + k); cp(p.z + om + k, g.z0 + oc + k);
        cp(p.lmbda + om + k, g.l0 + oc + k);
        cp(p.d + om + k, g.d0 + oc + k); cp(p.di + om + k, g.di0 + oc + k);
        if (!save) p.di2[om + k] = p.di[om + k] * p.di[om + k];
        if (dir) {
            cp(p.ds + om + k, g.ds0 + oc + k); cp(p.dz + om + k, g.dz0 + oc + k);
            cp(g.ds2 + om + k, g.ds20 + oc + k); cp(g.dz2 + om + k, g.dz20 + oc + k);
        }
        if (res) cp(p.rz + om + k, g.rz0 + oc + k);
    }
    if (CONES) {
        for (int k = tid; k < p.m - p.ml; k += nt) cp(p.v + oc + k, qs.v0 + oc + k);
        for (int k = tid; k < p.nq; k += nt) cp(p.beta + oc + k, qs.beta0 + oc + k);
    }
    if (SDP) for (int k = 0; k < p.ns; ++k) {
        const int ms = p.sinfo[5 * k], ro = p.sinfo[5 * k + 3];
        for (int e = tid; e < ms * ms; e += nt) {
            cp(p.sr + oc + ro + e, qs.r0 + oc + ro + e); cp(p.srti + oc + ro + e, qs.rti0 + oc + ro + e);
        }
    }
    if (EPI && tid == 0) {
        GPScal &T = gp_scal(g, oc);
        cp(&T.t, &T.t0); cp(&T.s0, &T.s00); cp(&T.z0, &T.z00); cp(&T.l0, &T.l00); cp(&T.d0, &T.d00);
        cp(&T.di0, &T.di00);
        if (dir) { cp(&T.dt, &T.dt0); cp(&T.ds0, &T.ds00); cp(&T.dz0, &T.dz00); cp(&T.ds20, &T.ds200); cp(&T.dz20, &T.dz200); }
        if (res) { cp(&T.rxt, &T.rxt0); cp(&T.rz0, &T.rz00); }
    }
}
// the line search's decision for slot b (:1131-1261) once the GEMVs have formed newrx: newgap, newphi and cpl's
// relaxed-line-search state machine.  A problem still searching halves its step (or resumes the saved search) and
// counts itself in nsearch; a step that underflows to 0 ends the problem 'unknown' (status 3) on its iterate
template <bool EQ, bool EPI = true, bool CONES = false, bool SDP = false>
__global__ void k_gp_ls(Ptrs p, GPPtrs g, int i, int iter, int *nsearch, QSave qs) {
    GP_SETUP
    __shared__ int act;                                  // 1: save the state, 2: restore it
    if (S.done || T.searching == 0.0) return;
    const double *f = g.fv + (long long)b * g.nK;
    double rx2 = 0, rn2 = 0;
    for (int k = tid; k < p.n; k += nt) { const double v = g.nrx[on + k]; rx2 += v * v; }
    for (int k = tid; k < g.mnl; k += nt) { const double v = g.ns[om + k] + f[k + (EPI ? 1 : 0)]; rn2 += v * v; }
    rx2 = block_sum(rx2, sh); rn2 = block_sum(rn2, sh);
    if (tid == 0) {
        double nresx = sqrt(rx2), nresznl = sqrt(rn2);
        if (EPI) {
            const double rxt = -T.nz0 + 1.0, r0 = T.ns0 + (f[0] - T.nt);
            nresx = sqrt(rx2 + rxt * rxt); nresznl = sqrt(rn2 + r0 * r0);
        }
        const double step = S.step, gap = S.gap;
        const double ngap = (1.0 - (1.0 - S.sigma) * step) * gap + step * step * S.dsdz;
        const double nphi = T.th1 * ngap + T.th2 * nresx + T.th3 * nresznl;
        const int rel = (int)T.relaxed;
        bool back = true;
        act = 0;
        if (i == 0) {
            if (ngap <= (1.0 - GP_ALPHA * step) * gap &&
                ((0 <= rel && rel < GP_MAX_RELAXED) || nphi <= T.phi + GP_ALPHA * step * T.dphi)) {
                back = false;
                S.sigma = fmin(ngap / gap, pow(ngap / gap, 3.0));
                S.eta = 0.0;
            }
        } else if (rel == -1) {                          // standard; relaxed_iters stays -1 (:1178 compares)
            if (nphi <= T.phi + GP_ALPHA * step * T.dphi) back = false;
        } else if (rel == 0) {
            if (!(nphi <= T.phi + GP_ALPHA * step * T.dphi)) {
                T.phi0 = T.phi; T.dphi0 = T.dphi; T.gap0 = gap; T.step0 = step; T.dsdz0 = S.dsdz;
                T.sigma0 = S.sigma; T.eta0 = S.eta;
                T.relaxed = 1; act = 1;
            }
            back = false;
        } else if (rel < GP_MAX_RELAXED) {
            T.relaxed = nphi <= T.phi0 + GP_ALPHA * T.step0 * T.dphi0 ? 0 : rel + 1;
            back = false;
        } else if (nphi <= T.phi0 + GP_ALPHA * T.step0 * T.dphi0) {
            back = false; T.relaxed = 0;
        } else {                                         // resume the saved line search as a standard one
            T.phi = T.phi0; T.dphi = T.dphi0; S.gap = T.gap0; S.step = T.step0; S.dsdz = T.dsdz0;
            S.sigma = T.sigma0; S.eta = T.eta0;
            T.relaxed = -1; act = 2;
        }
        if (back && act == 0) S.step = step * GP_BETA;
        if (!back) T.searching = 0.0;
        else if (S.step == 0.0) { T.searching = 0.0; S.done = 1; S.status = 3; S.iters = iter; }
        else atomicAdd(nsearch, 1);
    }
    __syncthreads();
    if (act) gp_save<EPI, CONES, SDP>(p, g, qs, b, act == 1, true, act == 1);
}
// a singular KKT matrix after iteration 0 (:778-840): with 0 < relaxed_iters < 8 the problem restores the saved state
// (W, x, y, s, z, lmbda, the residuals, phi and gap) and is factored again (counted in nre); otherwise, or when the
// second factorisation fails too (second = 1), it ends 'unknown' (status 3) on its current iterate.  EPI false: mu
// follows the restored gap (:791), for k_dir_rhs; SDP: its degree counts each block's order
template <bool EQ, bool EPI = true, bool CONES = false, bool SDP = false>
__global__ void k_gp_singular(Ptrs p, GPPtrs g, const int *info, int iter, int second, int *nre, QSave qs) {
    GP_SETUP
    __shared__ int act;
    if (S.done || (info[b] <= 0 && !(EQ && p.infop[b] > 0))) return;
    if (tid == 0) {
        act = !second && T.relaxed > 0 && T.relaxed < GP_MAX_RELAXED;
        if (act) {
            T.phi = T.phi0; S.gap = T.gap0; T.relaxed = -1;
            if (!EPI) S.mu = SDP ? S.gap / (p.ml + p.nq + (p.mdg - p.mlq)) : S.gap / (p.ml + p.nq);
            atomicAdd(nre, 1);
        } else { S.done = 1; S.status = 3; S.iters = iter; }
    }
    __syncthreads();
    if (!act) return;
    gp_save<EPI, CONES, SDP>(p, g, qs, b, false, false, true);
    __syncthreads();
    double rx2 = 0, rn2 = 0;
    for (int k = tid; k < p.n; k += nt) { const double v = p.rx[on + k]; rx2 += v * v; }
    for (int k = tid; k < g.mnl; k += nt) { const double v = p.rz[om + k]; rn2 += v * v; }
    rx2 = block_sum(rx2, sh); rn2 = block_sum(rn2, sh);
    if (tid == 0) {
        if (EPI) { S.resx = sqrt(rx2 + T.rxt * T.rxt); T.resznl = sqrt(rn2 + T.rz0 * T.rz0); }
        else { S.resx = sqrt(rx2); T.resznl = sqrt(rn2); }
    }
}
// the update (:1264-1355): x, t, y += step d; ds, dz := e + step d; scale2 inverse; update_scaling with dnl and d
// alike; s = W' lmbda, z = W^{-1} lmbda; gap = lmbda'lmbda
__global__ void k_gp_update(Ptrs p, GPPtrs g) {
    GP_SETUP
    if (S.done) return;
    const double step = S.step;
    for (int k = tid; k < p.n; k += nt) p.x[on + k] += step * p.dx[on + k];
    for (int k = tid; k < p.neq; k += nt) p.y[oq + k] += step * p.dy[oq + k];
    double gap = 0.0;
    for (int k = tid; k <= p.m; k += nt) {
        const bool e = k == p.m;
        const double lk = e ? T.l0 : p.lmbda[om + k];
        const double ss = sqrt((1.0 + step * (e ? T.ds0 : p.ds[om + k])) * lk);
        const double sz = sqrt((1.0 + step * (e ? T.dz0 : p.dz[om + k])) * lk);
        const double d = (e ? T.d0 : p.d[om + k]) * ss / sz, di = 1.0 / d, ln = ss * sz;
        if (e) { T.d0 = d; T.di0 = di; T.l0 = ln; T.s0 = d * ln; T.z0 = di * ln; T.t += step * T.dt; }
        else {
            p.d[om + k] = d; p.di[om + k] = di; p.di2[om + k] = di * di; p.lmbda[om + k] = ln;
            p.s[om + k] = d * ln; p.z[om + k] = di * ln;
        }
        gap += ln * ln;
    }
    gap = block_sum(gap, sh);
    if (tid == 0) S.gap = gap;
}

// ---- convex programs: cvxprog.cp (:1359-1964) with the caller's F ----
// A CP batch is a GP batch without F (sum K = 0, nK = mnl + 1): the same epigraph problem, GPScal, state row and
// kernels, with f, Df and H written by the caller's callback (cvxb_cp_eval_fn) into per-slot buffers that the kernels
// below take into fv, gf0, G's rows [0, mnl) and P, where k_gp_eval writes them for a GP
struct CPPtrs {
    double *f, *Df, *H, *z;          // the callback's buffers, row-major per slot: nK, nK x n, n x n, nK
    const int *idx;                  // slot -> load index (the callback's `problem`)
    int *bad;                        // the smallest load index whose f at its iterate was not finite
    double *P;                       // the batch's P, ld ldp
    long long ldp, sP;
};
// Df'[z0; z[:mnl]] at column j of the slot's Df (nK x n, row-major)
__device__ __forceinline__ double cp_dfz(const double *Df, int n, int nK, double z0, const double *z, int j) {
    double a = z0 * Df[j];
    for (int i = 1; i < nK; ++i) a += z[i - 1] * Df[(long long)i * n + j];
    return a;
}
// a + Df'z[:nK] at column j of a cpl batch's Df (nK x n, row-major; no objective row)
__device__ __forceinline__ double cpl_dfz(const double *Df, int n, int nK, double a, const double *z, int j) {
    for (int i = 0; i < nK; ++i) a += z[i] * Df[(long long)i * n + j];
    return a;
}
// the z of a full evaluation, [z0; z[:mnl]] (EPI false: z[:mnl]), for every active slot
template <bool EPI = true> __global__ void k_cp_zpack(Ptrs p, GPPtrs g, CPPtrs c) {
    GP_SETUP
    double *zc = c.z + (long long)b * g.nK;
    if (EPI) for (int i = tid; i < g.nK; i += nt) zc[i] = i == 0 ? T.z0 : p.z[om + i - 1];
    else for (int i = tid; i < g.nK; i += nt) zc[i] = p.z[om + i];
}
// the callback's F at slot b's iterate (FULL) or trial point: f into fv.  FULL: a non-finite f recorded in bad,
// Df[0] into gf0, Df[1:] into G's rows [0, mnl) and H's lower triangle into P's, by 32 x 32 tiles through shared
// memory (H row-major, P column-major).  Trial, only the problems still searching: newrx's nonlinear part
// Df'[nz0; nz[:mnl]] into nrx (the GEMVs add G'newzl + A'newy).  EPI false (a cpl batch): Df is Df[:mnl], all of it
// goes into G, and newrx starts from c.  256 threads.
// ADJ (k_adj_cp_take, FULL): every slot, done or not; neither fv nor gf0, which the adjoint does not read; and
// flag[b] := 1 when f, Df or H's lower triangle has a non-finite entry, else 0
template <bool FULL, bool EPI, bool ADJ>
__device__ __forceinline__ void cp_take_body(const Ptrs &p, const GPPtrs &g, const CPPtrs &c, int *flag) {
    GP_SETUP
    if (!ADJ && (S.done || (!FULL && T.searching == 0.0))) return;
    const int n = p.n, nK = g.nK;
    const double *f = c.f + (long long)b * nK, *Df = c.Df + (long long)b * nK * n;
    if (!ADJ) for (int i = tid; i < nK; i += nt) g.fv[(long long)b * nK + i] = f[i];
    if (!FULL) {
        for (int j = tid; j < n; j += nt)
            g.nrx[on + j] = EPI ? cp_dfz(Df, n, nK, T.nz0, g.nz + om, j) : cpl_dfz(Df, n, nK, p.q[on + j], g.nz + om, j);
        return;
    }
    if (!ADJ && tid == 0) {
        bool fin = true;
        for (int i = 0; i < nK; ++i) fin = fin && isfinite(f[i]);
        if (!fin) atomicMin(c.bad, c.idx[b]);
    }
    if (EPI && !ADJ) for (int j = tid; j < n; j += nt) g.gf0[on + j] = Df[j];
    double *G = g.G + (long long)b * g.sG;
    for (long long e = tid; e < (long long)g.mnl * n; e += nt) {
        const long long i = e % g.mnl, j = e / g.mnl;
        G[i + j * g.ldg] = Df[(i + (EPI ? 1 : 0)) * n + j];
    }
    __shared__ double tile[32][33];
    const double *H = c.H + (long long)b * n * n;
    double *P = c.P + (long long)b * c.sP;
    const int tx = tid & 31, ty = tid >> 5, nb = (n + 31) / 32;
    for (int bj = 0; bj < nb; ++bj)
        for (int bi = bj; bi < nb; ++bi) {
            __syncthreads();
            for (int r = ty; r < 32; r += 8) {                 // rows of H, coalesced along them
                const int i = bi * 32 + r, j = bj * 32 + tx;
                if (i < n && j < n) tile[r][tx] = H[(long long)i * n + j];
            }
            __syncthreads();
            for (int q = ty; q < 32; q += 8) {                 // columns of P, coalesced down them
                const int i = bi * 32 + tx, j = bj * 32 + q;
                if (i < n && i >= j) P[i + (long long)j * c.ldp] = tile[tx][q];
            }
        }
    if (ADJ) {                                         // f, Df and H's lower triangle, read again in one flat pass
        bool fin = true;
        for (int i = tid; i < nK; i += nt) fin = fin && isfinite(f[i]);
        for (long long e = tid; e < (long long)nK * n; e += nt) fin = fin && isfinite(Df[e]);
        for (long long e = tid; e < (long long)n * n; e += nt) fin = fin && (e % n > e / n || isfinite(H[e]));
        const int bad = __syncthreads_or(!fin);
        if (tid == 0) flag[b] = bad ? 1 : 0;
    }
}
template <bool FULL, bool EPI = true> __global__ void __launch_bounds__(256) k_cp_take(Ptrs p, GPPtrs g, CPPtrs c) {
    cp_take_body<FULL, EPI, false>(p, g, c, nullptr);
}
// rx += Df'[z0; z[:mnl]] (EPI false: Df'z[:mnl]) at the iterates, from the callback's Df (after k_gp_res_begin; the
// GEMVs add G'zl + A'y)
template <bool EPI = true> __global__ void k_cp_rx(Ptrs p, GPPtrs g, CPPtrs c) {
    GP_SETUP
    if (S.done) return;
    const double *Df = c.Df + (long long)b * g.nK * p.n;
    for (int j = tid; j < p.n; j += nt)
        p.rx[on + j] += EPI ? cp_dfz(Df, p.n, g.nK, T.z0, p.z + om, j) : cpl_dfz(Df, p.n, g.nK, 0.0, p.z + om, j);
}
// a domain round's decision (:1052-1062) once the callback has evaluated F at the trial points x + step dx: a problem
// still searching whose f has a non-finite entry halves its step and counts itself in nsearch; a step that underflows
// to 0 ends the problem 'unknown' (status 3) on its iterate, as in k_gp_ls.  32 threads
__global__ void k_cp_dom(Ptrs p, GPPtrs g, CPPtrs c, int iter, int *nsearch) {
    GP_SETUP
    if (S.done || T.searching == 0.0) return;
    const double *f = c.f + (long long)b * g.nK;
    bool fin = true;
    for (int i = tid; i < g.nK; i += nt) fin = fin && isfinite(f[i]);
    fin = __all_sync(0xffffffffu, fin);
    if (tid == 0 && !fin) {
        S.step *= GP_BETA;
        if (S.step == 0.0) { T.searching = 0.0; S.done = 1; S.status = 3; S.iters = iter; }
        else atomicAdd(nsearch, 1);
    }
}

// ---- convex QCQPs: cp with f_i = x'P_i x / 2 + q_i'x + r_i (i = 0..mnl), evaluated by the library ----
// A QC batch is a CP batch whose F the library knows.  Per slot, G holds the stacked [P_0; ...; P_mnl] (symmetric,
// nK blocks of n rows) below the m rows of [Df[1:]; G], where a GP's F lies, so compaction moves them with the rest;
// gp_eval's GEMV forms u = [P_0 x; ...; P_mnl x] in yv.  q (nK x n) and then r (nK) sit in the state row where a GP's
// g does.  dom f is all of R^n: no domain rounds.
// f_i = x'(u_i / 2 + q_i) + r_i into fv at slot b's iterate (FULL) or trial point, one warp per i.  FULL: a non-finite
// f recorded in bad, Df_0 = u_0 + q_0 into gf0, Df_i = u_i + q_i into G's rows [0, mnl).  Trial, only the problems
// still searching: newrx's nonlinear part Df'[nz0; nz[:mnl]] into nrx (the GEMVs add G'newzl + A'newy).  256 threads
template <bool FULL> __global__ void __launch_bounds__(256) k_qc_eval(Ptrs p, GPPtrs g, CPPtrs c) {
    GP_SETUP
    if (S.done || (!FULL && T.searching == 0.0)) return;
    const int n = p.n, nK = g.nK;
    const double *u = g.yv + (long long)b * g.sumK, *qv = g.g + oc, *r = qv + g.sumK;
    const double *x = (FULL ? p.x : g.nx) + on;
    double *f = g.fv + (long long)b * nK;
    for (int i = warp; i < nK; i += nwarp) {
        const double *ui = u + (long long)i * n, *qi = qv + (long long)i * n;
        double a = 0.0;
        for (int k = lane; k < n; k += 32) a += x[k] * (0.5 * ui[k] + qi[k]);
        a = warp_sum(a);
        if (lane == 0) f[i] = a + r[i];
    }
    if (!FULL) {
        for (int j = tid; j < n; j += nt) {
            double a = T.nz0 * (u[j] + qv[j]);
            for (int i = 1; i < nK; ++i) a += g.nz[om + i - 1] * (u[(long long)i * n + j] + qv[(long long)i * n + j]);
            g.nrx[on + j] = a;
        }
    } else {
        for (int j = tid; j < n; j += nt) g.gf0[on + j] = u[j] + qv[j];
        double *G = g.G + (long long)b * g.sG;
        for (long long e = tid; e < (long long)g.mnl * n; e += nt) {
            const long long i = e % g.mnl, j = e / g.mnl;
            G[i + j * g.ldg] = u[(i + 1) * n + j] + qv[(i + 1) * n + j];
        }
        __syncthreads();
        if (tid == 0) {
            bool fin = true;
            for (int i = 0; i < nK; ++i) fin = fin && isfinite(f[i]);
            if (!fin) atomicMin(c.bad, c.idx[b]);
        }
    }
}
// rx += Df'[z0; z[:mnl]] at the iterates, from grad f0 and G's rows [0, mnl) as k_qc_eval<true> left them (after
// k_gp_res_begin; the GEMVs add G'zl + A'y)
__global__ void k_qc_rx(Ptrs p, GPPtrs g) {
    GP_SETUP
    if (S.done) return;
    const double *G = g.G + (long long)b * g.sG;
    for (int j = tid; j < p.n; j += nt) {
        double a = T.z0 * g.gf0[on + j];
        for (int i = 0; i < g.mnl; ++i) a += p.z[om + i] * G[i + (long long)j * g.ldg];
        p.rx[on + j] += a;
    }
}
// H = z0 P_0 + sum_i z_i P_i at the iterates into P's lower triangle, one 32 x 32 tile (bi >= bj) per CTA, grid
// (nb (nb + 1) / 2, Bact), 256 threads; each entry sums its nK terms in order.  MIRROR (refinement > 0, whose residual
// multiplies by all of H): the tile's transpose into the upper triangle too, through shared memory
template <bool MIRROR> __global__ void __launch_bounds__(256) k_qc_hessian(Ptrs p, GPPtrs g, CPPtrs c) {
    const int b = blockIdx.y, tid = threadIdx.x, tx = tid & 31, ty = tid >> 5;
    const int n = p.n, nb = (n + 31) / 32;
    int t = blockIdx.x, bj = 0;
    while (t >= nb - bj) { t -= nb - bj; ++bj; }
    const int bi = bj + t;
    const double z0 = gp_scal(g, (long long)b * p.L).z0, *z = p.z + (long long)b * p.m;
    const double *Ps = g.G + (long long)b * g.sG + p.m;
    double *P = c.P + (long long)b * c.sP;
    __shared__ double tile[32][33];
    const int i = bi * 32 + tx;
    for (int q = ty; q < 32; q += 8) {                   // columns of H, coalesced down them
        const int j = bj * 32 + q;
        if (i < n && j <= i) {
            const double *e = Ps + i + (long long)j * g.ldg;
            double a = z0 * e[0];
            for (int k = 1; k < g.nK; ++k) a += z[k - 1] * e[(long long)k * n];
            P[i + (long long)j * c.ldp] = a;
            if (MIRROR) tile[tx][q] = a;
        }
    }
    if (!MIRROR) return;
    __syncthreads();
    for (int q = ty; q < 32; q += 8) {                   // H(j, i) = H(i, j) for i > j, coalesced along j
        const int ii = bi * 32 + q, j = bj * 32 + tx;
        if (ii < n && j < ii) P[j + (long long)ii * c.ldp] = tile[q][tx];
    }
}

// ---- the adjoint of an 'l'-only QP batch's solution (cvxb_batch_adjoint) ----
// Differentiating P x + q + A'y + G'z = 0, A x = b, G x + s = h and s o z = 0 at the returned iterate gives the KKT
// matrix M = [P A' G'; A 0 0; G 0 -W'W], W'W = diag(s / z).  For a loss's gradients (gx, gy, gz) one reduced solve
// gives M [ux; uy; uz] = [gx; gy; gz], and then dL/dq = -ux, dL/db = uy, dL/dh = uz, dL/dP = -(ux x' + x ux') / 2,
// dL/dG = -(z ux' + uz x'), dL/dA = -(y ux' + uy x').  A problem whose results are not optimal, or whose adjoint
// factorisation failed, gets NaN in every output.
__device__ __forceinline__ bool adj_bad(const Ptrs &p, const int *info, int b) {
    return p.sc[b].status != 1 || info[b] > 0 || (p.neq > 0 && p.infop[b] > 0);
}
// slot b's right-hand side from problem perm[b]'s gradients (nullptr: zero): dx := gx, dy := gy, bzp := W^{-T} gz, with
// the scaling of the returned s and z: d = sqrt(s / z), di = 1 / d, di2 = z / s; and g in (rx, ry, rz) for the residual
__global__ void k_adj_rhs(Ptrs p, const double *gx, const double *gy, const double *gz, const int *perm) {
    const int b = blockIdx.x;
    const long long on = (long long)b * p.n, om = (long long)b * p.m, oq = (long long)b * p.neq, k = perm[b];
    for (int i = threadIdx.x; i < p.n; i += blockDim.x) p.dx[on + i] = p.rx[on + i] = gx ? gx[k * p.n + i] : 0.0;
    for (int i = threadIdx.x; i < p.neq; i += blockDim.x) p.dy[oq + i] = p.ry[oq + i] = gy ? gy[k * p.neq + i] : 0.0;
    for (int i = threadIdx.x; i < p.m; i += blockDim.x) {
        const double s = p.s[om + i], z = p.z[om + i], d = sqrt(s / z), di = 1.0 / d, g = gz ? gz[k * p.m + i] : 0.0;
        p.d[om + i] = d; p.di[om + i] = di; p.di2[om + i] = z / s;
        p.bzp[om + i] = di * g; p.rz[om + i] = g;
    }
}
// after the first solve: dz := uz = di o bzp (batch_solve leaves W uz in bzp)
__global__ void k_adj_uz(Ptrs p) {
    const long long om = (long long)blockIdx.x * p.m;
    for (int i = threadIdx.x; i < p.m; i += blockDim.x) p.dz[om + i] = p.di[om + i] * p.bzp[om + i];
}
// once the GEMVs have left rz = gz - G ux: rz += W'W uz, the residual's last block, and bzp := W^{-T} rz for the
// refinement solve
__global__ void k_adj_res(Ptrs p) {
    const long long om = (long long)blockIdx.x * p.m;
    for (int i = threadIdx.x; i < p.m; i += blockDim.x) {
        const double r = p.rz[om + i] + p.d[om + i] * p.d[om + i] * p.dz[om + i];
        p.bzp[om + i] = p.di[om + i] * r;
    }
}
// after the refinement solve (the correction in rx, ry and W duz in bzp): ux := dx + rx, uy := dy + ry and uz := dz +
// di o bzp, uz kept in bzp for k_adj_grad; ux, uy and uz into problem perm[b]'s rows of the outputs that are given
__global__ void k_adj_vecs(Ptrs p, double *ux, double *uy, double *uz, const int *perm, const int *info) {
    const int b = blockIdx.x;
    const long long on = (long long)b * p.n, om = (long long)b * p.m, oq = (long long)b * p.neq, k = perm[b];
    const bool bad = adj_bad(p, info, b);
    for (int i = threadIdx.x; i < p.n; i += blockDim.x) p.dx[on + i] += p.rx[on + i];
    for (int i = threadIdx.x; i < p.neq; i += blockDim.x) p.dy[oq + i] += p.ry[oq + i];
    for (int i = threadIdx.x; i < p.m; i += blockDim.x) {
        const double u = p.dz[om + i] + p.di[om + i] * p.bzp[om + i];
        p.bzp[om + i] = u;
        if (uz) uz[k * p.m + i] = bad ? NAN : u;
    }
    if (ux) for (int i = threadIdx.x; i < p.n; i += blockDim.x) ux[k * p.n + i] = bad ? NAN : p.dx[on + i];
    if (uy) for (int i = threadIdx.x; i < p.neq; i += blockDim.x) uy[k * p.neq + i] = bad ? NAN : p.dy[oq + i];
}
// o[c * rows + i] = f(i, c) for the nj columns c of a rows x nj column-major block, contiguous in memory: flat over the
// CTA, so that short columns keep every thread busy; (c, i) step by the CTA's stride without a division per entry
template <class F> __device__ __forceinline__ void adj_store(double *o, int rows, int nj, bool bad, F f) {
    const int qs = blockDim.x / rows, rs = blockDim.x % rows;
    int c = threadIdx.x / rows, i = threadIdx.x % rows;
    while (c < nj) {
        o[(long long)c * rows + i] = bad ? NAN : f(i, c);
        i += rs; c += qs;
        if (i >= rows) { i -= rows; ++c; }
    }
}
// dP, dG and dA (nullptr: not written) of problem perm[b] in one pass over columns [j0, j0 + ADJ_TJ), grid
// (ceil(n / ADJ_TJ), B): the tile's x_j and ux_j in shared memory, the row vectors read down the columns, and each
// matrix's tile stored as one contiguous run of its column-major layout
constexpr int ADJ_TJ = 32;
__global__ void __launch_bounds__(256) k_adj_grad(Ptrs p, double *dP, double *dG, double *dA, const int *perm,
                                                  const int *info) {
    const int b = blockIdx.y, j0 = blockIdx.x * ADJ_TJ, nj = min(ADJ_TJ, p.n - j0), n = p.n, m = p.m, pq = p.neq;
    const long long on = (long long)b * n, om = (long long)b * m, oq = (long long)b * pq, k = perm[b];
    const double *__restrict__ x = p.x + on, *__restrict__ ux = p.dx + on;
    const double *__restrict__ z = p.z + om, *__restrict__ uz = p.bzp + om;
    const double *__restrict__ y = p.y + oq, *__restrict__ uy = p.dy + oq;
    __shared__ double xs[ADJ_TJ], uxs[ADJ_TJ];
    if (threadIdx.x < nj) { xs[threadIdx.x] = x[j0 + threadIdx.x]; uxs[threadIdx.x] = ux[j0 + threadIdx.x]; }
    __syncthreads();
    const bool bad = adj_bad(p, info, b);
    // rounded products, no FMA: dP(i, j) and dP(j, i) are the same sum, so both triangles are bitwise symmetric
    if (dP) adj_store(dP + (k * n + j0) * n, n, nj, bad,
                      [&](int i, int c) { return -0.5 * __dadd_rn(__dmul_rn(ux[i], xs[c]), __dmul_rn(x[i], uxs[c])); });
    if (dG && m) adj_store(dG + (k * n + j0) * m, m, nj, bad,
                           [&](int i, int c) { return -(z[i] * uxs[c] + uz[i] * xs[c]); });
    if (dA && pq) adj_store(dA + (k * n + j0) * pq, pq, nj, bad,
                            [&](int i, int c) { return -(y[i] * uxs[c] + uy[i] * xs[c]); });
}

// ---- the adjoint of a cone QP or cone LP batch's solution (cvxb_batch_adjoint_cone) ----
// On the central path s o z = mu e, and its linearisation L(z) ds + L(s) dz = 0 gives ds = -L(z)^{-1} L(s) dz; s and z
// share a Jordan frame there, where L(z)^{-1} L(s) is the NT scaling's W'W.  So the adjoint is the 'l' one with W'W the
// NT scaling of the returned s and z, and a cone LP's is the same with P = 0.  The 'l' kernels above run on every row
// as before and these fix the cone rows around them: d = di = 0 there, so k_adj_res leaves 0 in those rows, and once
// stage 3 has zeroed them in bzp k_adj_vecs takes uz = dz.  'q' cones one per warp (W = beta (2 v v' - J), symmetric);
// 's' blocks in k_adj_s, with r and rti from k_adj_s_nt.
//   stage 0, after k_adj_rhs: each cone's scaling (v, beta; lmbda is scratch) and bzp := W^{-T} g; each 's' block of rz
//            := sym(g), which k_s_wtz then scales into bzp
//   stage 1, after k_adj_uz: dz := W^{-1} bzp; a failed 's' scaling (part[3]) sets info, so the problem gets NaN
//   stage 2, after k_adj_res: bzp := W^{-T} rz + W dz = W^{-T} (gz - G ux + W'W uz), the refinement's right-hand side
//   stage 3, after the refinement solve and k_adj_s: dz += W^{-1} bzp, then bzp := 0 on the cone rows
// ds is scratch throughout
__global__ void k_adj_cone(Ptrs p, int *info, int stage) {
    PB_SETUP
    double *rz = p.rz + om, *bzp = p.bzp + om, *dz = p.dz + om, *ds = p.ds + om;
    double *v = p.v + oc - p.ml, *beta = p.beta + oc;
    if (stage == 0) {
        for (int i = p.ml + tid; i < p.m; i += nt) { p.d[om + i] = 0.0; p.di[om + i] = 0.0; }
        for (int k = 0; k < p.ns; ++k) {
            const int ms = p.sinfo[5 * k], so = p.sinfo[5 * k + 1];
            for (int e = tid; e < ms * ms; e += nt) {
                const int i = e % ms, j = e / ms;
                if (i > j) {
                    const double a = 0.5 * (rz[so + e] + rz[so + j + i * ms]);
                    rz[so + e] = a; rz[so + j + i * ms] = a;
                }
            }
        }
        FOR_CONES(o, len) {
            q_nt_compute(wt, p.s + om + o, p.z + om + o, v + o, p.lmbda + om + o, beta + k_, len);
            __syncwarp();
            q_scale(wt, v + o, beta[k_], rz + o, bzp + o, len, true);
        }
    } else if (stage == 1) {
        FOR_CONES(o, len) q_scale(wt, v + o, beta[k_], bzp + o, dz + o, len, true);
        if (tid == 0)
            for (int k = 0; k < p.ns; ++k) if (p.spart[((long long)b * p.ns + k) * 4 + 3] != 0.0) info[b] = 1;
    } else if (stage == 2) {
        FOR_CONES(o, len) {
            q_scale(wt, v + o, beta[k_], rz + o, bzp + o, len, true);
            q_scale(wt, v + o, beta[k_], dz + o, ds + o, len, false);
            __syncwarp();
            FOR_LANE(i, len) bzp[o + i] += ds[o + i];
        }
    } else {
        FOR_CONES(o, len) {
            q_scale(wt, v + o, beta[k_], bzp + o, ds + o, len, true);
            __syncwarp();
            FOR_LANE(i, len) dz[o + i] += ds[o + i];
        }
        __syncthreads();
        for (int i = p.ml + tid; i < p.m; i += nt) bzp[i] = 0.0;
    }
}
// the NT scaling of every slot's returned s and z, done or not (k_s_nt_compute skips done slots)
__global__ void __launch_bounds__(SB_T) k_adj_s_nt(Ptrs p) { s_nt_compute<true>(p); }
// the 's' blocks of the adjoint, one CTA per (block, slot): mode 0 (after the first solve) dz := W^{-1} bzp =
// rti unpack(bzp) rti', mode 2 (after the refinement solve) dz += the same; mode 1 (after k_adj_res) bzp :=
// pack(W^{-T} rz + W dz) = pack(rti' rz rti + r' dz r).  dz is written from its lower triangle, so both of its
// triangles, and those of uz, dh and dG after it, hold the same values
__global__ void __launch_bounds__(SB_T) k_adj_s(Ptrs p, int mode) {
    SB_SETUP
    __shared__ double R[SMX], X[SMX], Y[SMX], T[SMX];
    if (mode == 1) {
        s_load(X, p.rz + om + so, ms);
        SB_FOR(e, ms) R[e] = p.srti[oc + sro + e];
        __syncthreads();
        s_congr(Y, R, X, T, true, ms);
        s_load(X, p.dz + om + so, ms);
        SB_FOR(e, ms) R[e] = p.sr[oc + sro + e];
        __syncthreads();
        s_congr(X, R, X, T, true, ms);
        SB_FOR(e, ms) Y[e] += X[e];
        __syncthreads();
        s_store_packed(p.bzp + om + sp, Y, ms);
        return;
    }
    s_load_packed(X, p.bzp + om + sp, ms);
    SB_FOR(e, ms) R[e] = p.srti[oc + sro + e];
    __syncthreads();
    s_congr(Y, R, X, T, false, ms);
    SB_FOR(e, ms) {
        const int i = e % ms, j = e / ms;
        const double u = Y[i >= j ? e : j + i * ms];
        p.dz[om + so + e] = mode == 2 ? p.dz[om + so + e] + u : u;
    }
}

// ---- the adjoint of a QCQP batch's solution (cvxb_batch_adjoint_qcqp) ----
// The same derivation with f_i(x) = x'P_i x / 2 + q_i'x + r_i: at the returned iterate, with the objective's multiplier
// z_0 = 1, the KKT matrix is the QP's with H = P_0 + sum_i znl_i P_i in place of P and [Df; G] in place of G, Df's rows
// (P_i x + q_i)'.  Row i of the constraint residual is f_i(x) + s_i, whose derivatives in q_i, r_i and P_i are x', 1
// and x x' / 2; so beyond the QP's gradients dL/dP_i = -(znl_i (ux x' + x ux') + uznl_i x x') / 2, dL/dq_i =
// -(znl_i ux + uznl_i x) and dL/dr_i = -uznl_i for i >= 1, and dL/dr_0 = 0.
// The operator at x, once gp_products has left u = [P_0 x; ...; P_mnl x] in yv: H into all of P (the refinement's P
// GEMV reads both triangles) and Df_i = u_i + q_i into G's rows [0, mnl), q from the slot's state row.  Thread e of a
// slot forms H's entry e and Df's entry e, grid (ceil(max(n², mnl n) / 256), B).  The stack is mirrored at load, so
// H(i, j) and H(j, i) are the same sum
__global__ void __launch_bounds__(256) k_adj_qc_op(Ptrs p, GPPtrs g, CPPtrs c) {
    const int b = blockIdx.y, n = p.n, mnl = g.mnl;
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const double *z = p.z + (long long)b * p.m;
    if (e < (long long)n * n) {
        const long long i = e % n, j = e / n;
        const double *pe = g.G + (long long)b * g.sG + p.m + i + j * g.ldg;
        double a = pe[0];
        for (int k = 1; k < g.nK; ++k) a += z[k - 1] * pe[(long long)k * n];
        c.P[(long long)b * c.sP + i + j * c.ldp] = a;
    }
    if (e < (long long)mnl * n) {
        const long long i = e % mnl, j = e / mnl;
        const double *u = g.yv + (long long)b * g.sumK, *qv = g.g + (long long)b * p.L;
        g.G[(long long)b * g.sG + i + j * g.ldg] = u[(i + 1) * n + j] + qv[(i + 1) * n + j];
    }
}
// o[(c nK + k) rows + i] = f(i, k, c) for the nj columns c of nK stacked rows x nj column-major blocks, contiguous in
// memory: adj_store with the block index k stepped alongside (c, i)
template <class F> __device__ __forceinline__ void adj_store_stack(double *o, int rows, int nK, int nj, bool bad, F f) {
    const int qs = blockDim.x / rows, rs = blockDim.x % rows, qc = qs / nK, qk = qs % nK;
    const int t = threadIdx.x / rows;
    int c = t / nK, k = t % nK, i = threadIdx.x % rows;
    while (c < nj) {
        o[((long long)c * nK + k) * rows + i] = bad ? NAN : f(i, k, c);
        i += rs; k += qk; c += qc;
        if (i >= rows) { i -= rows; ++k; }
        if (k >= nK) { k -= nK; ++c; }
    }
}
// dP's nK blocks, dq, dr, dG and dA (nullptr: not written) of problem perm[b] in one pass over columns [j0, j0 +
// ADJ_TJ), grid (ceil(n / ADJ_TJ), B), as k_adj_grad: dP per problem the (nK n) x n column-major stack, dq nK x n, dr
// nK (by the CTA of the first tile), dG over the 'l' rows only (rows mnl.. of z and uz)
__global__ void __launch_bounds__(256) k_adj_qc_grad(Ptrs p, GPPtrs g, double *dP, double *dq, double *dr, double *dG,
                                                     double *dA, const int *perm, const int *info) {
    const int b = blockIdx.y, j0 = blockIdx.x * ADJ_TJ, nj = min(ADJ_TJ, p.n - j0), n = p.n, m = p.m, pq = p.neq;
    const int nK = g.nK, ml = m - g.mnl;
    const long long on = (long long)b * n, om = (long long)b * m, oq = (long long)b * pq, k = perm[b];
    const double *__restrict__ x = p.x + on, *__restrict__ ux = p.dx + on;
    const double *__restrict__ z = p.z + om, *__restrict__ uz = p.bzp + om;
    const double *__restrict__ y = p.y + oq, *__restrict__ uy = p.dy + oq;
    __shared__ double xs[ADJ_TJ], uxs[ADJ_TJ];
    if (threadIdx.x < nj) { xs[threadIdx.x] = x[j0 + threadIdx.x]; uxs[threadIdx.x] = ux[j0 + threadIdx.x]; }
    __syncthreads();
    const bool bad = adj_bad(p, info, b);
    // rounded products, no FMA: every term is the same in (i, j) and (j, i), so each block is bitwise symmetric
    if (dP) adj_store_stack(dP + (k * n + j0) * nK * n, n, nK, nj, bad, [&](int i, int l, int c) {
        const double s = __dadd_rn(__dmul_rn(ux[i], xs[c]), __dmul_rn(x[i], uxs[c]));
        if (l == 0) return -0.5 * s;
        return -0.5 * __dadd_rn(__dmul_rn(z[l - 1], s), __dmul_rn(uz[l - 1], __dmul_rn(x[i], xs[c])));
    });
    if (dq)
        for (int e = threadIdx.x; e < nK * nj; e += blockDim.x) {
            const int l = e / nj, c = e % nj;
            dq[(k * nK + l) * n + j0 + c] = bad ? NAN : l == 0 ? -uxs[c] : -(z[l - 1] * uxs[c] + uz[l - 1] * xs[c]);
        }
    if (dr && blockIdx.x == 0)
        for (int l = threadIdx.x; l < nK; l += blockDim.x) dr[k * nK + l] = bad ? NAN : l == 0 ? 0.0 : -uz[l - 1];
    if (dG && ml) adj_store(dG + (k * n + j0) * ml, ml, nj, bad,
                            [&](int i, int c) { return -(z[g.mnl + i] * uxs[c] + uz[g.mnl + i] * xs[c]); });
    if (dA && pq) adj_store(dA + (k * n + j0) * pq, pq, nj, bad,
                            [&](int i, int c) { return -(y[i] * uxs[c] + uy[i] * xs[c]); });
}

// ---- the adjoint of a GP batch's solution (cvxb_batch_adjoint_gp) ----
// The QCQP's derivation with f_i(x) = lse(F_i x + g_i): at the returned iterate, with z_0 = 1, pi_i = softmax(F_i x +
// g_i) and Sigma_i = diag(pi_i) - pi_i pi_i', the KKT matrix has H = sum_i z_i F_i' Sigma_i F_i and Df's rows
// pi_i' F_i.  For a parameter t of f_i, dL/dt = -(z_i d_t(ux' grad f_i) + uz_i d_t f_i); with w_i = F_i ux and v_i =
// Sigma_i w_i = pi_i o (w_i - pi_i' w_i) that is dL/dg_i = -(z_i v_i + uz_i pi_i) and dL/dF_i = dL/dg_i x' -
// z_i pi_i ux', uz_0 = 0.  A monomial row (K_i = 1: pi = 1, Sigma = 0) gets the QP's dh and dG with h = -g.
// The operator at x, once gp_products has left F x in yv: k_gp_eval<true>'s body on every slot with z_0 = 1, so pi in
// yv, Df into G's rows [0, mnl), f into fv, and H's rows and their weights z_i in Hr and hw for gp_hessian
__global__ void k_adj_gp_op(Ptrs p, GPPtrs g) { gp_eval_body<true, true>(p, g, 0); }
// once the batched GEMV has left w = F ux in wv, grid (nK, B): block i of slot b reduces pi_i' w_i and replaces w_i by
// dL/dg_i in wv, stored into problem perm[b]'s row of dg (nullptr: not written), S = sum K per problem
__global__ void k_adj_gp_dg(Ptrs p, GPPtrs g, double *dg, const int *perm, const int *info) {
    const int i = blockIdx.x, b = blockIdx.y, tid = threadIdx.x, nt = blockDim.x;
    __shared__ double sh[32];
    const int k0 = g.koff[i], K = g.koff[i + 1] - k0;
    const long long ok = (long long)b * g.sumK + k0, om = (long long)b * p.m;
    const double *pi = g.yv + ok;
    double *w = g.wv + ok;
    double t = 0.0;
    for (int k = tid; k < K; k += nt) t += pi[k] * w[k];
    t = block_sum(t, sh);
    const double zi = i == 0 ? 1.0 : p.z[om + i - 1], uzi = i == 0 ? 0.0 : p.bzp[om + i - 1];
    const bool bad = adj_bad(p, info, b);
    double *o = dg ? dg + (long long)perm[b] * g.sumK + k0 : nullptr;
    for (int k = tid; k < K; k += nt) {
        const double v = -(zi * (pi[k] * (w[k] - t)) + uzi * pi[k]);
        w[k] = v;
        if (o) o[k] = bad ? NAN : v;
    }
}
// dF, dG and dA (nullptr: not written) of problem perm[b] over columns [j0, j0 + ADJ_TJ), grid (ceil(n / ADJ_TJ), B),
// as k_adj_grad: dF per problem the S x n column-major F of cvxb_batch_load_gp, row k dg_k x' - hw_k pi_k ux' from
// k_adj_gp_dg's dg in wv; dG over the 'l' rows only (rows mnl.. of z and uz)
__global__ void __launch_bounds__(256) k_adj_gp_grad(Ptrs p, GPPtrs g, double *dF, double *dG, double *dA,
                                                     const int *perm, const int *info) {
    const int b = blockIdx.y, j0 = blockIdx.x * ADJ_TJ, nj = min(ADJ_TJ, p.n - j0), n = p.n, m = p.m, pq = p.neq;
    const int S = g.sumK, ml = m - g.mnl;
    const long long on = (long long)b * n, om = (long long)b * m, oq = (long long)b * pq, ok = (long long)b * S;
    const long long k = perm[b];
    const double *__restrict__ x = p.x + on, *__restrict__ ux = p.dx + on;
    const double *__restrict__ z = p.z + om, *__restrict__ uz = p.bzp + om;
    const double *__restrict__ y = p.y + oq, *__restrict__ uy = p.dy + oq;
    const double *__restrict__ dgv = g.wv + ok, *__restrict__ pi = g.yv + ok, *__restrict__ hw = g.hw + ok;
    __shared__ double xs[ADJ_TJ], uxs[ADJ_TJ];
    if (threadIdx.x < nj) { xs[threadIdx.x] = x[j0 + threadIdx.x]; uxs[threadIdx.x] = ux[j0 + threadIdx.x]; }
    __syncthreads();
    const bool bad = adj_bad(p, info, b);
    if (dF) adj_store(dF + (k * n + j0) * S, S, nj, bad,
                      [&](int i, int c) { return dgv[i] * xs[c] - hw[i] * pi[i] * uxs[c]; });
    if (dG && ml) adj_store(dG + (k * n + j0) * ml, ml, nj, bad,
                            [&](int i, int c) { return -(z[g.mnl + i] * uxs[c] + uz[g.mnl + i] * xs[c]); });
    if (dA && pq) adj_store(dA + (k * n + j0) * pq, pq, nj, bad,
                            [&](int i, int c) { return -(y[i] * uxs[c] + uy[i] * xs[c]); });
}

// ---- the adjoint of a CP or cpl batch's solution (cvxb_batch_adjoint_cp) ----
// The QCQP's derivation with the caller's f: at the returned iterate, with zk = [1; znl] (cp's epigraph problem) or
// zk = znl (cpl), the KKT matrix has H = sum_i zk_i grad² f_i and Df's rows grad f_i' (i = 1..mnl), both from one call
// of the caller's F(x, zk); a cpl batch's cone rows get the cone adjoint's W'W.  For a parameter t of F, dL/dt =
// -d_t[ux' Df' zk + uk' f] with uk = [0; uznl] (cpl: uznl), which the caller forms from ux and uz; the library writes
// ux, uy, uz, dG and dA (k_adj_qc_grad without its P_i outputs).
// The z of that call on every slot (k_cp_zpack skips done slots, and after a solve every slot is done)
__global__ void k_adj_cp_zpack(Ptrs p, GPPtrs g, CPPtrs c, int epi) {
    const long long b = blockIdx.x;
    const double *z = p.z + b * p.m;
    double *zc = c.z + b * g.nK;
    for (int i = threadIdx.x; i < g.nK; i += blockDim.x) zc[i] = epi ? (i == 0 ? 1.0 : z[i - 1]) : z[i];
}
// the operator at x once the callback has run: Df into G's rows [0, mnl), H's lower triangle into P and each slot's
// non-finite flag into flag (cp_take_body<true, EPI, true>)
template <bool EPI> __global__ void __launch_bounds__(256) k_adj_cp_take(Ptrs p, GPPtrs g, CPPtrs c, int *flag) {
    cp_take_body<true, EPI, true>(p, g, c, flag);
}
// after the adjoint's last factorisation: a slot whose F(x, zk) was not finite fails it, so adj_bad gives it NaN
__global__ void k_adj_cp_flag(int *info, const int *flag, int B) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < B && flag[b]) info[b] = 1;
}

// ---- the tangent of a batch's solution (cvxb_batch_tangent, _qcqp, _gp, _cp) ----
// The adjoint's matrix M is symmetric, so the derivative of (x, y, z) along a data direction d is M^{-1} r(d): the
// same factorisation, solves and refinement as the adjoint with g = r.  r is the derivative of the KKT residual at the
// returned iterate with the sign that puts it on the right-hand side: rx = -d(grad_x L), ry = db - dA x, rz = dh -
// dG x, and on the nonlinear rows -d f_i.  The kernels below form r from the caller's d (problem order, nullptr: zero)
// and the slot's x, y and z, one CTA of TAN_T threads per slot, into problem perm[b]'s rows of rx, ry and rz; each
// matrix of d is read once, and no sum depends on the launch: the tangent is bit-identical across compaction and
// sub-batches.
constexpr int TAN_T = 256, TAN_RQ = 4, TAN_RC = 32 * TAN_RQ;   // threads, rows per lane, rows per chunk
// One pass over the rows x cols column-major matrix a (ld lda), chunks of TAN_RC rows, the warps over its columns:
// COLS: cs[j] += sum_i zf(i) a(i, j), the column sums by the lanes of warp j % nwarp (cs is global, and every pass
// gives column j to the same warp, so its updates need no fence between passes); ROWS: rowf(i, sum_j a(i, j) xs[j])
// once per row, the warps' partial sums added in warp order in part (TAN_RC doubles per warp).  a == nullptr is
// zero: rowf(i, 0) only.  Every thread of the CTA calls it; zf's values are read at the start of a chunk and rowf runs
// between two barriers, so rowf may overwrite what zf reads
template <bool COLS, bool ROWS, class Z, class R>
__device__ __forceinline__ void tan_pass(const double *__restrict__ a, long long lda, int rows, int cols,
                                         const double *xs, Z zf, double *cs, R rowf, double *part) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarp = blockDim.x >> 5;
    if (!a) {
        if (ROWS) {
            for (int i = tid; i < rows; i += blockDim.x) rowf(i, 0.0);
            __syncthreads();
        }
        return;
    }
    for (int r0 = 0; r0 < rows; r0 += TAN_RC) {
        double acc[TAN_RQ], zv[TAN_RQ];
#pragma unroll
        for (int q = 0; q < TAN_RQ; ++q) {
            const int i = r0 + lane + 32 * q;
            acc[q] = 0.0;
            zv[q] = COLS && i < rows ? zf(i) : 0.0;
        }
        for (int j = warp; j < cols; j += nwarp) {
            const double *aj = a + (long long)j * lda;
            const double xj = ROWS ? xs[j] : 0.0;
            double s = 0.0;
#pragma unroll
            for (int q = 0; q < TAN_RQ; ++q) {
                const int i = r0 + lane + 32 * q;
                if (i < rows) {
                    const double v = aj[i];
                    if (ROWS) acc[q] += v * xj;
                    if (COLS) s += zv[q] * v;
                }
            }
            if (COLS) {
                s = warp_sum(s);
                if (lane == 0) cs[j] += s;
            }
        }
        if (ROWS) {
#pragma unroll
            for (int q = 0; q < TAN_RQ; ++q) part[warp * TAN_RC + lane + 32 * q] = acc[q];
            __syncthreads();
            for (int t = tid; t < TAN_RC && r0 + t < rows; t += blockDim.x) {
                double v = 0.0;
                for (int w = 0; w < nwarp; ++w) v += part[w * TAN_RC + t];
                rowf(r0 + t, v);
            }
            __syncthreads();
        }
    }
}
// the caller's direction, problem order; which arrays a kind reads is its kernel's
struct TanIn {
    const double *dP, *dq, *dr, *dF, *dg, *tx, *tf, *dG, *dh, *dA, *db;
};
#define TAN_SETUP                                                                                      \
    const int b = blockIdx.x, tid = threadIdx.x, nt = blockDim.x, n = p.n, m = p.m, pq = p.neq;        \
    const long long k = perm[b];                                                                       \
    const double *x = p.x + (long long)b * n, *y = p.y + (long long)b * pq, *z = p.z + (long long)b * m; \
    double *rx = tx_ + k * n, *ry = ty_ + k * pq, *rz = tz_ + k * m;                                   \
    __shared__ double part[TAN_T / 32 * TAN_RC];                                                       \
    (void)y;
// the linear rows, shared by every kind once rx holds the rest of -rx: rx += dA'y + dG'zl, ry = db - dA x, rzl = dh -
// dG x over the ml = m - mnl rows of G (zl and rzl from row mnl of z and rz), then rx := -rx
__device__ __forceinline__ void tan_linear(const Ptrs &p, const TanIn &d, long long k, int mnl, const double *x,
                                           const double *y, const double *z, double *rx, double *ry, double *rz,
                                           double *part) {
    const int n = p.n, pq = p.neq, ml = p.m - mnl;
    if (pq) tan_pass<true, true>(d.dA ? d.dA + k * pq * n : nullptr, pq, pq, n, x, [&](int i) { return y[i]; }, rx,
                                 [&](int i, double t) { ry[i] = (d.db ? d.db[k * pq + i] : 0.0) - t; }, part);
    if (ml) tan_pass<true, true>(d.dG ? d.dG + k * ml * n : nullptr, ml, ml, n, x, [&](int i) { return z[mnl + i]; },
                                 rx, [&](int i, double t) { rz[mnl + i] = (d.dh ? d.dh[k * ml + i] : 0.0) - t; }, part);
    __syncthreads();
    for (int j = threadIdx.x; j < n; j += blockDim.x) rx[j] = -rx[j];
}
// QP, cone QP and cone LP (c in dq, dP nullptr): rx = -(sym(dP) x + dq + dA'y + dG'z)
__global__ void __launch_bounds__(TAN_T) k_tan_rhs(Ptrs p, TanIn d, double *tx_, double *ty_, double *tz_,
                                                   const int *perm) {
    TAN_SETUP
    for (int j = tid; j < n; j += nt) rx[j] = d.dq ? d.dq[k * n + j] : 0.0;
    __syncthreads();
    if (d.dP) tan_pass<true, true>(d.dP + k * n * n, n, n, n, x, [&](int i) { return 0.5 * x[i]; }, rx,
                                   [&](int i, double t) { rx[i] += 0.5 * t; }, part);
    tan_linear(p, d, k, 0, x, y, z, rx, ry, rz, part);
}
// QCQP, zk = [1; znl]: rx = -(sum_l zk_l (sym(dP_l) x + dq_l) + dA'y + dG'zl), rznl_l = -(x'dP_l x / 2 + dq_l'x +
// dr_l); dP per problem the (nK n) x n column-major stack, dq nK x n, dr nK
__global__ void __launch_bounds__(TAN_T) k_tan_rhs_qc(Ptrs p, GPPtrs g, TanIn d, double *tx_, double *ty_,
                                                      double *tz_, const int *perm) {
    TAN_SETUP
    const int nK = g.nK;
    __shared__ double sh[32];
    for (int j = tid; j < n; j += nt) {
        double a = 0.0;
        if (d.dq) {
            a = d.dq[k * nK * n + j];
            for (int l = 1; l < nK; ++l) a += z[l - 1] * d.dq[(k * nK + l) * n + j];
        }
        rx[j] = a;
    }
    __syncthreads();
    for (int l = 0; l < nK; ++l) {
        const double zl = l == 0 ? 1.0 : z[l - 1];
        double a = 0.0;                                  // this thread's share of x'dP_l x / 2 + dq_l'x
        if (d.dP) tan_pass<true, true>(d.dP + k * nK * n * n + (long long)l * n, (long long)nK * n, n, n, x,
                                       [&](int i) { return 0.5 * zl * x[i]; }, rx,
                                       [&](int i, double t) { rx[i] += 0.5 * zl * t; a += 0.5 * x[i] * t; }, part);
        if (l == 0) continue;
        if (d.dq) for (int i = tid; i < n; i += nt) a += d.dq[(k * nK + l) * n + i] * x[i];
        a = block_sum(a, sh);
        if (tid == 0) rz[l - 1] = -(a + (d.dr ? d.dr[k * nK + l] : 0.0));
    }
    tan_linear(p, d, k, g.mnl, x, y, z, rx, ry, rz, part);
}
// GP, pi_i = softmax(F_i x + g_i), w_i = dF_i x + dg_i, z_0 = 1: rx = -(sum_i z_i (dF_i'pi_i + F_i'Sigma_i w_i) +
// dA'y + dG'zl), rznl_i = -pi_i'w_i; dF per problem S x n column-major, dg S.  The slot's F x + g, pi, then z_i pi,
// w and z_i Sigma_i w_i in yv and wv (scratch that the adjoint and a solve rewrite before they read it)
__global__ void __launch_bounds__(TAN_T) k_tan_rhs_gp(Ptrs p, GPPtrs g, TanIn d, double *tx_, double *ty_,
                                                      double *tz_, const int *perm) {
    TAN_SETUP
    const int S = g.sumK, nK = g.nK;
    const double *Fb = g.G + (long long)b * g.sG + m, *gv = g.g + (long long)b * p.L;
    double *pi = g.yv + (long long)b * S, *w = g.wv + (long long)b * S;
    __shared__ double sh[32];
    auto none = [](int) { return 0.0; };
    tan_pass<false, true>(Fb, g.ldg, S, n, x, none, nullptr, [&](int r, double t) { pi[r] = t + gv[r]; }, part);
    for (int i = 0; i < nK; ++i) {                       // softmax per block, gp_eval_body's
        const int k0 = g.koff[i], K = g.koff[i + 1] - k0;
        const double zi = i == 0 ? 1.0 : z[i - 1];
        double mx = -INFINITY;
        for (int r = tid; r < K; r += nt) mx = fmax(mx, pi[k0 + r]);
        mx = -block_min(-mx, sh);
        double sum = 0.0;
        for (int r = tid; r < K; r += nt) { const double e = exp(pi[k0 + r] - mx); pi[k0 + r] = e; sum += e; }
        const double inv = 1.0 / block_sum(sum, sh);
        for (int r = tid; r < K; r += nt) { const double v = pi[k0 + r] * inv; pi[k0 + r] = v; w[k0 + r] = zi * v; }
    }
    for (int j = tid; j < n; j += nt) rx[j] = 0.0;
    __syncthreads();
    tan_pass<true, true>(d.dF ? d.dF + k * S * n : nullptr, S, S, n, x, [&](int r) { return w[r]; }, rx,
                         [&](int r, double t) { w[r] = t + (d.dg ? d.dg[k * S + r] : 0.0); }, part);
    for (int i = 0; i < nK; ++i) {                       // t_i = pi_i'w_i, then w := z_i Sigma_i w_i
        const int k0 = g.koff[i], K = g.koff[i + 1] - k0;
        const double zi = i == 0 ? 1.0 : z[i - 1];
        double t = 0.0;
        for (int r = tid; r < K; r += nt) t += pi[k0 + r] * w[k0 + r];
        t = block_sum(t, sh);
        if (i > 0 && tid == 0) rz[i - 1] = -t;
        for (int r = tid; r < K; r += nt) w[k0 + r] = zi * (pi[k0 + r] * (w[k0 + r] - t));
    }
    __syncthreads();
    tan_pass<true, false>(Fb, g.ldg, S, n, x, [&](int r) { return w[r]; }, rx, [](int, double) {}, part);
    tan_linear(p, d, k, g.mnl, x, y, z, rx, ry, rz, part);
}
// CP and cpl, from the caller's theta terms: rx = -(dc + tx + dA'y + dG'zl), rznl = -tf (tx n, tf mnl per problem)
__global__ void __launch_bounds__(TAN_T) k_tan_rhs_cp(Ptrs p, GPPtrs g, TanIn d, double *tx_, double *ty_,
                                                      double *tz_, const int *perm) {
    TAN_SETUP
    for (int j = tid; j < n; j += nt) rx[j] = (d.dq ? d.dq[k * n + j] : 0.0) + (d.tx ? d.tx[k * n + j] : 0.0);
    for (int i = tid; i < g.mnl; i += nt) rz[i] = d.tf ? -d.tf[k * g.mnl + i] : 0.0;
    __syncthreads();
    tan_linear(p, d, k, g.mnl, x, y, z, rx, ry, rz, part);
}

// the problem family of a batch: coneqp, conelp, gp, cp, cpl or a convex QCQP (cp with the library's F)
enum class Kind { QP, LP, GP, CP, CPL, QC };
}  // namespace

struct cvxb_batch {
    Kind kind = Kind::QP;
    // GP, CP, cpl and QC batches run the lock-step cpl (solve_cpl) with gq's per-slot state
    bool cpl_loop() const { return kind == Kind::GP || kind == Kind::CP || kind == Kind::CPL || kind == Kind::QC; }
    // CP and cpl batches evaluate the caller's F through cfn, which calls back to the host
    bool calls_back() const { return kind == Kind::CP || kind == Kind::CPL; }
    // CP, cpl and QC batches start from a loaded x0 and check that f is finite at the iterates
    bool from_x0() const { return calls_back() || kind == Kind::QC; }
    int device = 0, B = 0, n = 0, m = 0;
    long long ldg = 0, ldp = 0, ldk = 0;
    long long sG = 0, sP = 0, sK = 0, sInv = 0;
    int nblk = 0;
    DevBuf<double> P, G, K, inv, panel, gemv_ws;
    DevBuf<double> vecs;             // all n- and m-vectors
    double *q = nullptr, *h = nullptr;   // in vecs
    Ptrs p;                          // also holds the dims ('l' rows p.ml, p.nq cones) and p.refinement
    DevBuf<Scal> sc;
    DevBuf<int> d_info, d_ndone;
    DevBuf<int> d_done, d_pairs, d_perm;     // compaction: done flags, swap list, slot -> problem
    std::vector<int> perm;           // slot -> original problem index (identity unless the last solve compacted)
    bool permuted = false;
    int compact = 1;                 // CVXB_BATCH_COMPACT=0 disables
    int Bact = 0;                    // slots [0, Bact) are launched by the lock-step loop
    CholWork cw;
    cudaStream_t st = nullptr;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    bool loaded = false;
    bool solved = false;             // a cvxb_batch_solve completed since the last load (cvxb_batch_adjoint reads it)
    int iters_run = 0;
    int ls_rounds = 0;               // gp: line-search rounds of the last solve
    double solve_ms = 0;
    // single large problem: SYRK on the int8 tensor path (ozaki_syrk.cu), same rule as cvxb_kkt_factor
    // (ozaki_use) when B == 1 and there are no 'q' cones; ozaki_mode() at create
    int i8_mode = 0;
    int syrk_path = 0;
    DevBuf<char> oz_work;
    // 'q' cones (cvxb_batch_create_cones): rows [0, p.ml) are 'l', then the cones
    DevBuf<int> qoff;                // nq + 1 row offsets
    DevBuf<double> Gs;               // W^{-T} G per slot (ld ldg), rebuilt every factorisation; only with 'q' cones
    DevBuf<double> cst;              // per-slot state row (moves with its problem); empty without cones and refinement
    long long L = 0;
    // equality rows (cvxb_batch_create_eq, neq = p > 0), per problem: A (p x n, ld lda), Asct = L^{-1} A' (n x p,
    // ld ldas), Kp (p x p, ld ldkp) and its diagonal-block inverses, the NPV p-vectors b y ry dy aw, Kp's info
    int neq = 0;
    long long lda = 0, sA = 0, ldas = 0, sAs = 0, ldkp = 0, sKp = 0, sInvp = 0;
    DevBuf<double> A, Asct, Kp, invp, pvecs;
    DevBuf<int> d_infop;
    bool eq_loaded = false;          // cvxb_batch_load_eq since the last cvxb_batch_load
    bool switched = false;           // some problem of this solve factors S + A'A (its aw is 1)
    // cone LP batch (cvxb_batch_create_lp): no P; q holds c; lpv holds x1 (n), z1 and th (m), y1 (p) per slot
    DevBuf<double> lpv;
    // 's' blocks (cvxb_batch_create_sdp): p.ns blocks of positive order; Gs has mpk = cdim_pckd rows
    int mpk = 0;
    long long sums = 0, sums2 = 0;   // sum of the orders, of their squares
    DevBuf<int> sinfo, u2p;
    DevBuf<double> rw, spart;
    // the start (cvxb_batch_load_start): B * (n + p + 2 cdim) doubles in problem order, allocated on the first load;
    // warm_set until cvxb_batch_clear_start, warm's pointers into it for the given keys
    DevBuf<double> start;
    Warm warm{};
    bool warm_set = false;
    // geometric programs (cvxb_batch_create_gp): m = mnl + ml rows, G holds [Df[1:]; G; F] (ld ldg = m + sum K rounded
    // up to even), P holds H; gq's per-slot vectors live in gpv, H's scaled rows in gph, the block offsets in koff and
    // g, in problem order, in gpg (copied into the state row by each solve)
    GPPtrs gq{};
    DevBuf<double> gpv, gph, gpg;
    DevBuf<int> koff;
    long long glen = 0;              // gpg's doubles per problem: a GP's sum K, a QC batch's nK n + nK (q and r)
    // convex programs (cvxb_batch_create_cp): gq of a GP batch without F (sum K = 0, nK = mnl + 1); the callback's
    // buffers in cpv, x0 in problem order in cpx0, slot -> load index and the non-finite flag in cpi.  A QC batch
    // (cvxb_batch_create_qcqp) has cpx0 and cpi, and the GP batch's F rows and gpg for its P_i, q_i and r_i
    CPPtrs cq{};
    DevBuf<double> cpv, cpx0;
    DevBuf<int> cpi;
    cvxb_cp_eval_fn cfn = nullptr;
    void *cctx = nullptr;
    // cpl batches (cvxb_batch_create_cpl): a CP batch of cpl's own problem, without the epigraph row: nK = mnl, c in
    // q, 'q' cones after the 'l' rows; qs: the relaxed line search's saved v and beta with cones
    QSave qs{};
    ~cvxb_batch() {                  // synchronises the stream, then releases it and the events
        if (st) cudaStreamSynchronize(st);
        for (cudaEvent_t e : {e0, e1}) if (e) cudaEventDestroy(e);
        if (st) cudaStreamDestroy(st);
    }
};

namespace {

// The per-slot state row: v (sum q) | beta (nq) with cones, wx wx2 (n) | wz ws wz2 ws2 wz3 (m) | wy wy2 (p) with
// refinement, LPScal in a cone LP batch; every piece starts 16-byte aligned.  Reallocated when the layout changes: nothing in it outlives a solve.
int state_alloc(cvxb_batch *b) {
    Ptrs &p = b->p;
    auto ev = [](long long x) { return (x + 1) & ~1LL; };
    const long long sumq = b->m - p.ml, n2 = ev(b->n), m2 = ev(b->m), p2 = ev(b->neq);
    const long long cone = p.nq ? ev(sumq) + ev(p.nq) : 0, ref = p.refinement ? 2 * n2 + 5 * m2 + 2 * p2 : 0;
    const long long lps = b->kind == Kind::LP ? ev(sizeof(LPScal) / sizeof(double)) : 0;
    const long long sb = p.ns ? 2 * ev(b->sums2) + 2 * ev(b->sums) : 0;     // r rti (sum ms²) | sigs sigz (sum ms)
    // gp: g (glen: a GP's sum K, a QC batch's q and r) | GPScal | x0 dx0 rx0 (n) | y0 dy0 ry0 (p) | s0 z0 ds0 dz0 ds20
    // dz20 l0 d0 di0 rz0 (m), and with cones v0 (sum q) | beta0 (nq), with 's' blocks r0 rti0 (sum s²)
    const long long gpl = b->cpl_loop() ? ev(b->glen) + ev(sizeof(GPScal) / sizeof(double)) + 3 * n2 + 3 * p2 + 10 * m2 : 0;
    const long long qsv = gpl ? cone : 0, ssv = gpl && p.ns ? 2 * ev(b->sums2) : 0;
    const long long L = cone + sb + ref + lps + gpl + qsv + ssv;
    if (b->L == L) return 0;
    b->L = p.L = 0;
    b->cst.reset();
    p.v = p.beta = p.wx = p.wx2 = p.wz = p.ws = p.wz2 = p.ws2 = p.wz3 = p.wy = p.wy2 = p.lps = nullptr;
    p.sr = p.srti = p.sigs = p.sigz = nullptr;
    b->qs = QSave{};
    if (L == 0) return 0;
    CVXB_TRY(b->cst.alloc((size_t)b->B * L));
    CVXB_CUDA(cudaMemset(b->cst.p, 0, (size_t)b->B * L * sizeof(double)));
    b->L = p.L = L;
    double *r = b->cst.p;
    if (cone) { p.v = r; r += ev(sumq); p.beta = r; r += ev(p.nq); }
    if (sb) {
        p.sr = r; r += ev(b->sums2); p.srti = r; r += ev(b->sums2);
        p.sigs = r; r += ev(b->sums); p.sigz = r; r += ev(b->sums);
    }
    if (ref) {
        p.wx = r; r += n2; p.wx2 = r; r += n2;
        p.wz = r; r += m2; p.ws = r; r += m2; p.wz2 = r; r += m2; p.ws2 = r; r += m2; p.wz3 = r; r += m2;
        if (p2) { p.wy = r; r += p2; p.wy2 = r; r += p2; }
    }
    if (lps) p.lps = r;
    if (gpl) {
        GPPtrs &g = b->gq;
        g.g = r; r += ev(b->glen); g.gs = r; r += ev(sizeof(GPScal) / sizeof(double));
        for (double **v : {&g.x0, &g.dx0, &g.rx0}) { *v = r; r += n2; }
        for (double **v : {&g.y0, &g.dy0, &g.ry0}) { *v = r; r += p2; }
        for (double **v : {&g.s0, &g.z0, &g.ds0, &g.dz0, &g.ds20, &g.dz20, &g.l0, &g.d0, &g.di0, &g.rz0}) { *v = r; r += m2; }
    }
    if (qsv) { b->qs.v0 = r; r += ev(sumq); b->qs.beta0 = r; r += ev(p.nq); }
    if (ssv) { b->qs.r0 = r; r += ev(b->sums2); b->qs.rti0 = r; }
    return 0;
}

// Asct := L^{-1} A' (blocked forward substitution with S's diagonal-block inverses), Kp := Asct' Asct, Kp = Lp Lp'
// (misc.py:1464-1472).  Kp's per-slot info goes to d_infop.
int factor_kp(cvxb_batch *b) {
    cudaStream_t st = b->st;
    const int n = b->n, pq = b->neq, B = b->Bact;
    CVXB_TRY(transpose_copy(b->A.p, b->lda, b->Asct.p, b->ldas, pq, n, st, B, b->sA, b->sAs));
    CVXB_TRY(trsm_lower_left(n, b->K.p, b->ldk, b->inv.p, b->Asct.p, b->ldas, pq, st, B, b->sK, b->sInv, b->sAs));
    GemmDesc g;
    g.M = pq; g.N = pq; g.K = n;
    g.X = b->Asct.p; g.ldx = (int)b->ldas; g.x_kmajor = true; g.sX = b->sAs;
    g.Y = g.X; g.ldy = g.ldx; g.y_kmajor = true; g.sY = b->sAs;
    g.C = b->Kp.p; g.ldc = (int)b->ldkp; g.sC = b->sKp;
    g.lower_only = true; g.batch = B;
    if (b->B == 1) g.splitk_ws = b->cw.splitk_ws.p;
    CVXB_TRY(dmma_gemm(g, st));
    if (b->B == 1) {
        CVXB_TRY(potrf_lower(pq, b->Kp.p, (int)b->ldkp, b->invp.p, b->cw, st));
        CVXB_CUDA(cudaMemcpyAsync(b->d_infop.p, b->cw.d_info.p, sizeof(int), cudaMemcpyDeviceToDevice, st));
    } else {
        CVXB_TRY(potrf_lower_batched(pq, b->Kp.p, (int)b->ldkp, b->sKp, b->invp.p, b->sInvp, B, b->d_infop.p,
                                     b->panel.p, (pq + 1) & ~1, st));
    }
    return 0;
}

// K = P + Gs' Gs (+ A' diag(aw) A) with Gs = W^{-T} G (misc.py:1267-1282), then its Cholesky factor, then with
// equality rows (kp) Kp.  With 'q' cones Gs is formed; without, diag(di)² is applied inside the SYRK (w = di2), or
// by the int8 slicing for a single large problem.  A'A is added only while some problem is switched: aw = 0 adds
// exact zeros to the others.
int batch_factor(cvxb_batch *b, bool kp = true) {
    cudaStream_t st = b->st;
    const bool cones = b->p.nq > 0 || b->p.ns > 0;     // Gs = W^{-T} G is formed, mpk rows
    if (b->p.nq > 0 || (b->p.ns > 0 && b->p.mlq > 0)) {
        k_build_gs<<<dim3((b->n + 7) / 8, b->Bact), 256, 0, st>>>(b->p, b->G.p, b->Gs.p, b->ldg, b->sG);
        count_launch();
    }
    if (b->p.ns > 0) {
        k_s_build_gs<<<dim3(b->p.ns, b->Bact, (b->n + 15) / 16), SB_T, 0, st>>>(b->p, b->G.p, b->Gs.p, b->ldg, b->sG);
        count_launch();
    }
    // K = P + G' diag(di)^2 G from nine int8 slices per entry (fp64-accurate, ~1.8x the DMMA SYRK)
    const bool i8 = !cones && b->B == 1 && b->m > 0 && ozaki_use(b->i8_mode, b->n, b->m, b->oz_work);
    b->syrk_path = i8 ? 2 : 1;
    if (i8) {
        CVXB_TRY(ozaki_syrk(b->n, b->m, b->G.p, b->ldg, b->p.di, b->P.p, b->ldp, 1.0, b->K.p, b->ldk, 9, 0,
                            b->oz_work.p, st));
    } else {
        GemmDesc g;
        g.M = b->n; g.N = b->n; g.K = b->mpk;
        g.X = cones ? b->Gs.p : b->G.p; g.ldx = (int)b->ldg; g.x_kmajor = true; g.sX = b->sG;
        g.Y = g.X; g.ldy = (int)b->ldg; g.y_kmajor = true; g.sY = b->sG;
        if (!cones) { g.w = b->p.di2; g.sW = b->m; }
        g.D = b->P.p; g.ldd = (int)b->ldp; g.sD = b->sP; g.beta = 1.0;
        g.C = b->K.p; g.ldc = (int)b->ldk; g.sC = b->sK;
        g.lower_only = true; g.batch = b->Bact;
        if (b->B == 1) g.splitk_ws = b->cw.splitk_ws.p;
        CVXB_TRY(dmma_gemm(g, st));
    }
    if (b->switched) {
        GemmDesc g;
        g.M = b->n; g.N = b->n; g.K = b->neq;
        g.X = b->A.p; g.ldx = (int)b->lda; g.x_kmajor = true; g.sX = b->sA;
        g.Y = g.X; g.ldy = g.ldx; g.y_kmajor = true; g.sY = b->sA;
        g.w = b->p.aw; g.sW = b->neq;
        g.D = b->K.p; g.ldd = (int)b->ldk; g.sD = b->sK; g.beta = 1.0;
        g.C = b->K.p; g.ldc = (int)b->ldk; g.sC = b->sK;
        g.lower_only = true; g.batch = b->Bact;
        if (b->B == 1) g.splitk_ws = b->cw.splitk_ws.p;
        CVXB_TRY(dmma_gemm(g, st));
    }
    if (b->B == 1) {
        CVXB_TRY(potrf_lower(b->n, b->K.p, (int)b->ldk, b->inv.p, b->cw, st));
        CVXB_CUDA(cudaMemcpyAsync(b->d_info.p, b->cw.d_info.p, sizeof(int), cudaMemcpyDeviceToDevice, st));
    } else {
        CVXB_TRY(potrf_lower_batched(b->n, b->K.p, (int)b->ldk, b->sK, b->inv.p, b->sInv, b->Bact, b->d_info.p,
                                     b->panel.p, (b->n + 1) & ~1, st));
    }
    if (kp && b->neq > 0) CVXB_TRY(factor_kp(b));
    return 0;
}

// (x, y, bzp) := solution of the reduced KKT system; on entry x = bx (slot k at x + k*sx), y = by (slot k at
// y + k*sy, equality rows only), bzp = W^{-T} bz.  Gs is G with the weights di when it is not formed.
int batch_solve(cvxb_batch *b, double *x, long long sx, double *y = nullptr, long long sy = 0) {
    cudaStream_t st = b->st;
    const int n = b->n, m = b->m, B = b->Bact, pq = b->neq, mpk = b->mpk;
    const bool cones = b->p.nq > 0 || b->p.ns > 0;
    const double *A = cones ? b->Gs.p : b->G.p, *w = cones ? nullptr : b->p.di;
    const long long sw = w ? m : 0;
    // x := x + Gs' bzp
    GemvBatch gt; gt.batch = B; gt.sA = b->sG; gt.sw = sw; gt.sx = m; gt.sy = sx;
    CVXB_TRY(gemv_t(mpk, n, A, b->ldg, w, b->p.bzp, 1.0, 1.0, x, st, gt));
    if (pq == 0) {
        CVXB_TRY(potrs_lower(n, b->K.p, (int)b->ldk, b->inv.p, x, b->cw, st, B, b->sK, b->sInv, sx));
    } else {
        // kkt_chol2's elimination of the equality rows (misc.py:1526-1558)
        GemvBatch ga; ga.batch = B; ga.sA = b->sA; ga.sw = pq; ga.sx = sy; ga.sy = sx;
        if (b->switched)     // x += A' by for a switched problem (aw = 1), + 0 for the others
            CVXB_TRY(gemv_t(pq, n, b->A.p, b->lda, b->p.aw, y, 1.0, 1.0, x, st, ga));
        CVXB_TRY(trsv_lower(n, b->K.p, (int)b->ldk, b->inv.p, x, false, b->cw, st, B, b->sK, b->sInv, sx));
        GemvBatch gs; gs.batch = B; gs.sA = b->sAs; gs.sx = sx; gs.sy = sy;          // y := Asct' x - y
        CVXB_TRY(gemv_t(n, pq, b->Asct.p, b->ldas, nullptr, x, 1.0, -1.0, y, st, gs));
        CVXB_TRY(potrs_lower(pq, b->Kp.p, (int)b->ldkp, b->invp.p, y, b->cw, st, B, b->sKp, b->sInvp, sy));
        GemvBatch gy; gy.batch = B; gy.sA = b->sAs; gy.sx = sy; gy.sy = sx;          // x -= Asct y
        CVXB_TRY(gemv_n(n, pq, b->Asct.p, b->ldas, nullptr, y, -1.0, 1.0, x, b->gemv_ws.p, st, gy));
        CVXB_TRY(trsv_lower(n, b->K.p, (int)b->ldk, b->inv.p, x, true, b->cw, st, B, b->sK, b->sInv, sx));
    }
    // bzp := Gs x - bzp
    GemvBatch gn; gn.batch = B; gn.sA = b->sG; gn.sw = sw; gn.sx = sx; gn.sy = m;
    CVXB_TRY(gemv_n(mpk, n, A, b->ldg, w, x, 1.0, -1.0, b->p.bzp, b->gemv_ws.p, st, gn));
    return 0;
}

// the GEMVs of a refinement step's residual, res() (coneprog.py:1930-1952, :599-631; cvxprog.py:889-956):
// wx2 -= P dx + A' dy + G' wz3, wy2 -= A dx, wz2 -= G dx.  SDP: G' trisc(wz3) (misc.sgemv).  An LP has no P; in a GP,
// CP or cpl batch P holds H and G holds [Df; G]
template <bool EQ, bool LP, bool SDP> int refinement_gemvs(cvxb_batch *b) {
    cudaStream_t st = b->st;
    const int n = b->n, m = b->m, B = b->Bact, pq = b->neq;
    const Ptrs &p = b->p;
    const long long L = b->L;
    if (!LP) {
        GemvBatch gP; gP.batch = B; gP.sA = b->sP; gP.sx = n; gP.sy = L;
        CVXB_TRY(gemv_t(n, n, b->P.p, b->ldp, nullptr, p.dx, -1.0, 1.0, p.wx2, st, gP));
    }
    if (EQ) {
        GemvBatch ga; ga.batch = B; ga.sA = b->sA; ga.sx = pq; ga.sy = L;
        CVXB_TRY(gemv_t(pq, n, b->A.p, b->lda, nullptr, p.dy, -1.0, 1.0, p.wx2, st, ga));
    }
    if (m > 0) {
        GemvBatch gt; gt.batch = B; gt.sA = b->sG; gt.sx = L; gt.sy = L;
        CVXB_TRY(gemv_t(m, n, b->G.p, b->ldg, SDP ? p.rw : nullptr, p.wz3, -1.0, 1.0, p.wx2, st, gt));
    }
    if (EQ) {
        GemvBatch ga; ga.batch = B; ga.sA = b->sA; ga.sx = n; ga.sy = L;
        CVXB_TRY(gemv_n(pq, n, b->A.p, b->lda, nullptr, p.dx, -1.0, 1.0, p.wy2, b->gemv_ws.p, st, ga));
    }
    if (m > 0) {
        GemvBatch gn; gn.batch = B; gn.sA = b->sG; gn.sx = n; gn.sy = L;
        CVXB_TRY(gemv_n(m, n, b->G.p, b->ldg, nullptr, p.dx, -1.0, 1.0, p.wz2, b->gemv_ws.p, st, gn));
    }
    return 0;
}

// the i-th Newton direction: coneqp's f4 (coneprog.py:2288-2347) or, LP, conelp's f6 (:1211-1235) on the right-hand
// side, i.e. the unrefined solve and then `refinement` correction steps from the residual, followed by the step
// length and sigma
template <bool CONES, bool EQ, bool LP, bool SDP = false> int direction(cvxb_batch *b, int i) {
    cudaStream_t st = b->st;
    const int n = b->n, m = b->m, B = b->Bact, T = 256, pq = b->neq;
    const Ptrs &p = b->p;
    const long long L = b->L;
    const dim3 sg(p.ns, B);                          // SDP: one CTA per ('s' block, slot)
    k_dir_rhs<CONES, EQ, LP, SDP><<<B, T, 0, st>>>(p, i); count_launch();
    if (SDP) { k_s_wtz<<<sg, SB_T, 0, st>>>(p, p.dz, m, p.ds, m, 2); count_launch(); }
    CVXB_TRY(batch_solve(b, p.dx, n, p.dy, pq));
    // f4_no_ir's step after the solve: k_dir_post folds it in for an unrefined QP solve, except with 's' blocks, whose
    // rows k_s_dir_post reads before k_dir_post runs
    if (LP) { k_lp_f6_post<EQ, SDP><<<B, T, 0, st>>>(p, p.dx, n, p.dy, pq, p.ds, m, 0); count_launch(); }
    else if (p.refinement || SDP) { k_f4_post<EQ, SDP><<<B, T, 0, st>>>(p, p.dx, n, p.dz, m, p.ds, m, 0); count_launch(); }
    for (int r = 0; r < p.refinement; ++r) {
        // res(): its elementwise part, then the GEMVs
        if (SDP) { k_s_res<LP><<<sg, SB_T, 0, st>>>(p); count_launch(); }
        k_res<EQ, LP, SDP><<<B, T, 0, st>>>(p); count_launch();
        CVXB_TRY((refinement_gemvs<EQ, LP, SDP>(b)));
        k_f4_pre<<<B, T, 0, st>>>(p, p.wz2, L, p.ws2, L); count_launch();
        if (SDP) { k_s_wtz<<<sg, SB_T, 0, st>>>(p, p.wz2, L, p.ws2, L, 2); count_launch(); }
        CVXB_TRY(batch_solve(b, p.wx2, L, p.wy2, L));
        if (LP) k_lp_f6_post<EQ, SDP><<<B, T, 0, st>>>(p, p.wx2, L, p.wy2, L, p.ws2, L, 1);
        else k_f4_post<EQ, SDP><<<B, T, 0, st>>>(p, p.wx2, L, p.wz2, L, p.ws2, L, 1);
        count_launch();
    }
    if (SDP) { k_s_dir_post<<<sg, SB_T, 0, st>>>(p, i); count_launch(); }
    k_dir_post<CONES, LP, SDP><<<B, T, 0, st>>>(p, i, !LP && !SDP && p.refinement == 0); count_launch();
    return 0;
}

// swap the slots of each pair (disjoint pairs: one launch)
int swap_slots(cvxb_batch *b, const std::vector<int> &pairs) {
    const int np = (int)pairs.size() / 2;
    if (np == 0) return 0;
    CVXB_CUDA(cudaMemcpyAsync(b->d_pairs.p, pairs.data(), pairs.size() * sizeof(int), cudaMemcpyHostToDevice, b->st));
    SwapArgs a;
    a.P = b->P.p; a.G = b->G.p; a.vecs = b->vecs.p; a.sc = b->sc.p; a.sP = b->P.p ? b->sP : 0; a.sG = b->sG;
    a.n = b->n; a.me = b->m > 0 ? b->m : 1; a.Btot = b->B;
    a.A = b->A.p; a.pvecs = b->pvecs.p; a.sA = b->sA; a.neq = b->neq;
    k_swap_slots<<<dim3(96, np), 256, 0, b->st>>>(a, b->d_pairs.p);
    count_launch();
    if (b->cst.p) {
        k_swap_rows<<<dim3(8, np), 256, 0, b->st>>>(b->cst.p, b->L, b->d_pairs.p);
        count_launch();
    }
    // `pairs` is pageable host memory: the copy above is staged before cudaMemcpyAsync returns
    return 0;
}

// put every problem back into its own slot (a solve that compacted left them permuted)
int restore_order(cvxb_batch *b) {
    if (!b->permuted) return 0;
    std::vector<int> pr(2);
    for (int i = 0; i < b->B; ++i) {
        while (b->perm[i] != i) {
            const int j = b->perm[i];                // the problem in slot i belongs to slot j
            pr[0] = i; pr[1] = j;
            CVXB_TRY(swap_slots(b, pr));
            std::swap(b->perm[i], b->perm[j]);
        }
    }
    CVXB_CUDA(cudaStreamSynchronize(b->st));
    b->permuted = false;
    return 0;
}

// kkt_chol2's first factorisation (misc.py:1421-1447) once batch_factor(b, false) has factored S: a problem whose S is
// singular factors S + A'A from now on; then Kp.  Nothing to do without equality rows
template <bool EQ> int first_switch(cvxb_batch *b) {
    cudaStream_t st = b->st;
    const int B = b->Bact;
    if (EQ) {
        std::vector<int> info(B);
        CVXB_CUDA(cudaMemcpyAsync(info.data(), b->d_info.p, B * sizeof(int), cudaMemcpyDeviceToHost, st));
        CVXB_CUDA(cudaStreamSynchronize(st));
        for (int i = 0; i < B; ++i) b->switched |= info[i] > 0;
        if (b->switched) {
            k_switch<<<B, 256, 0, st>>>(b->p.aw, b->d_info.p, b->neq); count_launch();
            CVXB_TRY(batch_factor(b, false));
        }
        CVXB_TRY(factor_kp(b));
    }
    return 0;
}
// the starting point's factorisation with W = I, kkt_chol2's first
template <bool EQ> int start_factor(cvxb_batch *b) {
    CVXB_TRY(batch_factor(b, false));
    return first_switch<EQ>(b);
}

// the rank condition of the reference's ValueError for a singular KKT matrix: coneqp's "Rank(A) < p or Rank([P; A;
// G]) < n" (coneprog.py:2065-2067), without A "Rank([P; G]) < n"; conelp's (:680-700); cp's and cpl's (cvxprog.py)
const char *rank_text(Kind kind, bool eq) {
    switch (kind) {
    case Kind::QP: return eq ? "Rank(A) < p or Rank([P; A; G]) < n" : "Rank([P; G]) < n";
    case Kind::LP: return "Rank(A) < p or Rank([G; A]) < n";
    default: return "Rank(A) < p or Rank([H(x); A; Df(x); G]) < n";
    }
}

// a singular first factorisation is the reference's rank ValueError.  After a loaded start the first factorisation
// is iteration 0's (coneprog.py:2256-2259, :1078-1080), over the active slots
template <bool EQ> int start_check(cvxb_batch *b) {
    cudaStream_t st = b->st;
    const int B = b->Bact;
    std::vector<int> info(B), infop(EQ ? B : 0);
    CVXB_CUDA(cudaMemcpyAsync(info.data(), b->d_info.p, B * sizeof(int), cudaMemcpyDeviceToHost, st));
    if (EQ) CVXB_CUDA(cudaMemcpyAsync(infop.data(), b->d_infop.p, B * sizeof(int), cudaMemcpyDeviceToHost, st));
    CVXB_CUDA(cudaStreamSynchronize(st));
    for (int i = 0; i < B; ++i)
        if (info[i] > 0 || (EQ && infop[i] > 0)) {
            set_error("batch_solve: problem %d: %s (singular KKT matrix at the start)", b->perm[i],
                      rank_text(b->kind, EQ));
            return CVXB_E_ARG;
        }
    return 0;
}

// the starting point from a loaded start (coneqp :2109-2149, conelp :662-857).  A cone LP with one of primalstart and
// dualstart factors W = I and solves for the other half; coneqp and a cone LP with both skip the factorisation, so
// that iteration 0's is the first.  A given s or z not strictly inside the cone is CVXB_E_ARG naming the problem
template <bool CONES, bool EQ, bool LP, bool SDP> int warm_start(cvxb_batch *b) {
    cudaStream_t st = b->st;
    const int n = b->n, m = b->m, B = b->Bact, T = 256, pq = b->neq;
    const Ptrs &p = b->p;
    const Warm w = b->warm;
    if (LP && !(w.s && w.z)) {
        CVXB_TRY(start_factor<EQ>(b));
        if (!w.s) {                                                // primal start (0, b, h): s = -uz
            k_scale_bz<<<B, T, 0, st>>>(p); count_launch();
            if (SDP) { k_s_wtz<<<dim3(p.ns, B), SB_T, 0, st>>>(p, p.dz, m, nullptr, 0, 0); count_launch(); }
            CVXB_CUDA(cudaMemsetAsync(p.x, 0, (size_t)B * n * sizeof(double), st));
            CVXB_TRY(batch_solve(b, p.x, n, p.y, pq));
        } else {                                                   // dual start (-c, 0, 0): z = uz
            CVXB_CUDA(cudaMemsetAsync(p.bzp, 0, (size_t)B * m * sizeof(double), st));
            if (EQ) CVXB_CUDA(cudaMemsetAsync(p.y, 0, (size_t)B * pq * sizeof(double), st));
            CVXB_TRY(batch_solve(b, p.dx, n, p.y, pq));
        }
        CVXB_LAUNCH_CHECK();
        CVXB_TRY(start_check<EQ>(b));
    }
    k_warm_copy<CONES, EQ, LP, SDP><<<B, T, 0, st>>>(p, w); count_launch();
    if (SDP) { k_s_eig_warm<<<dim3(p.ns, B), SB_T, 0, st>>>(p); count_launch(); }
    k_warm_point<CONES, EQ, LP, SDP><<<B, T, 0, st>>>(p, w, b->d_info.p); count_launch();
    CVXB_LAUNCH_CHECK();
    std::vector<int> bad(B);
    CVXB_CUDA(cudaMemcpyAsync(bad.data(), b->d_info.p, B * sizeof(int), cudaMemcpyDeviceToHost, st));
    CVXB_CUDA(cudaStreamSynchronize(st));
    for (int i = 0; i < B; ++i)
        if (bad[i]) {
            set_error("batch_solve: problem %d: initial %c is not positive", i, bad[i] == 1 ? 's' : 'z');
            return CVXB_E_ARG;
        }
    return 0;
}

// finished slots below the new active count trade places with active slots from the tail; b->Bact becomes the
// number of active problems
int compact_slots(cvxb_batch *b, int B, int ndone, const std::vector<int> &flags, std::vector<int> &pairs) {
    const int nb = B - ndone;
    pairs.clear();
    int j = B - 1;
    for (int i = 0; i < nb; ++i) {
        if (!flags[i]) continue;
        while (flags[j]) --j;             // an active slot in [nb, B): there are as many as finished ones below nb
        pairs.push_back(i); pairs.push_back(j);
        std::swap(b->perm[i], b->perm[j]);
        --j;
    }
    CVXB_TRY(swap_slots(b, pairs));
    b->permuted = true;
    b->Bact = nb;
    return 0;
}

// one int of the device counter d_ndone, after the stream has drained
int read_count(cvxb_batch *b, int &v) {
    CVXB_CUDA(cudaMemcpyAsync(&v, b->d_ndone.p, sizeof(int), cudaMemcpyDeviceToHost, b->st));
    CVXB_CUDA(cudaStreamSynchronize(b->st));
    return 0;
}

// the lock-step loops' scaffold.  solve_begin: every slot active, no problem switched, zero per-slot scalars, and the
// timing starts
int solve_begin(cvxb_batch *b) {
    b->Bact = b->B;
    b->switched = false;
    b->ls_rounds = 0;
    CVXB_CUDA(cudaMemsetAsync(b->sc.p, 0, (size_t)b->B * sizeof(Scal), b->st));
    CVXB_CUDA(cudaEventRecord(b->e0, b->st));
    return 0;
}
// the done-poll once the stopping rule has counted the finished slots in d_ndone and flagged them in d_done: one sync
// reads both, and with bad also cq.bad (the first problem whose f is not finite; b->B for none).  Unless every active
// slot is done or bad names a problem, finished slots then leave the active range (compact_slots, b->Bact); moved
// says whether any slots traded places
int poll_done(cvxb_batch *b, std::vector<int> &flags, std::vector<int> &pairs, int &ndone, bool &moved,
              int *bad = nullptr) {
    const int B = b->Bact;
    moved = false;
    CVXB_CUDA(cudaMemcpyAsync(flags.data(), b->d_done.p, (size_t)B * sizeof(int), cudaMemcpyDeviceToHost, b->st));
    if (bad) CVXB_CUDA(cudaMemcpyAsync(bad, b->cq.bad, sizeof(int), cudaMemcpyDeviceToHost, b->st));
    CVXB_TRY(read_count(b, ndone));
    if (ndone >= B || ndone == 0 || (bad && *bad < b->B) || !b->compact || b->B == 1) return 0;
    CVXB_TRY(compact_slots(b, B, ndone, flags, pairs));
    moved = !pairs.empty();
    return 0;
}
// solve_end after `it` iterations: the results cover every slot again, and the solve's time
int solve_end(cvxb_batch *b, int it) {
    b->iters_run = it;
    b->Bact = b->B;
    CVXB_CUDA(cudaEventRecord(b->e1, b->st));
    CVXB_CUDA(cudaStreamSynchronize(b->st));
    float t = 0;
    cudaEventElapsedTime(&t, b->e0, b->e1);
    b->solve_ms = t;
    return 0;
}

// the lock-step IPM over the active slots; CONES: the batch has 'q' cones, EQ: equality rows.  LP: coneprog.conelp
// (coneprog.py:662-1436) on a batch without P: the self-dual embedding's tau and kappa, one more KKT solve per
// iteration for (x1, y1, z1), and infeasibility certificates
template <bool CONES, bool EQ, bool LP, bool SDP = false>
int solve(cvxb_batch *b, int maxiters, double abstol, double reltol, double feastol) {
    cudaStream_t st = b->st;
    const int n = b->n, m = b->m, T = 256, pq = b->neq;
    int B = b->B;                                 // active slots: shrinks as problems finish (compaction)
    const Ptrs &p = b->p;
    GemvBatch gP; gP.batch = B; gP.sA = b->sP; gP.sx = n; gP.sy = n;
    GemvBatch gGt; gGt.batch = B; gGt.sA = b->sG; gGt.sx = m; gGt.sy = n;
    GemvBatch gGn; gGn.batch = B; gGn.sA = b->sG; gGn.sx = n; gGn.sy = m;
    GemvBatch gAt; gAt.batch = B; gAt.sA = b->sA; gAt.sx = pq; gAt.sy = n;
    GemvBatch gAn; gAn.batch = B; gAn.sA = b->sA; gAn.sx = n; gAn.sy = pq;
    CVXB_TRY(solve_begin(b));
    // ---- starting point: W = I (coneqp :2055-2106, conelp :662-857) ----
    k_init_rhs<EQ, SDP><<<B, T, 0, st>>>(p); count_launch();  // dx = -q, y = b, dz = h, resx0 / resy0 / resz0
    // a loaded start (coneqp's cdim == 0 branch, :2002, ignores it); firstcall: iteration 0's factorisation is the first
    const bool warm = b->warm_set && m > 0, firstcall = warm && (!LP || (b->warm.s && b->warm.z));
    if (warm) CVXB_TRY((warm_start<CONES, EQ, LP, SDP>(b)));
    else {
        CVXB_TRY(start_factor<EQ>(b));
        k_scale_bz<<<B, T, 0, st>>>(p); count_launch();
        if (SDP) { k_s_wtz<<<dim3(p.ns, B), SB_T, 0, st>>>(p, p.dz, m, nullptr, 0, 0); count_launch(); }
        if (LP) {
            CVXB_CUDA(cudaMemsetAsync(p.x, 0, (size_t)B * n * sizeof(double), st));
            CVXB_TRY(batch_solve(b, p.x, n, p.y, pq));            // primal start: (0, b, h)
            k_lp_start_mid<EQ, SDP><<<B, T, 0, st>>>(p); count_launch();
            CVXB_TRY(batch_solve(b, p.dx, n, p.y, pq));           // dual start: (-c, 0, 0)
            if (SDP) { k_s_eig_start<<<dim3(p.ns, B), SB_T, 0, st>>>(p); count_launch(); }
            k_lp_init_point<CONES, EQ, SDP><<<B, T, 0, st>>>(p, abstol, reltol); count_launch();
        } else {
            CVXB_TRY(batch_solve(b, p.dx, n, p.y, pq));
            if (SDP) {
                k_init_sz<<<B, T, 0, st>>>(p); count_launch();
                k_s_eig_start<<<dim3(p.ns, B), SB_T, 0, st>>>(p); count_launch();
            }
            k_init_point<CONES, SDP><<<B, T, 0, st>>>(p); count_launch();
        }
        CVXB_LAUNCH_CHECK();
        CVXB_TRY(start_check<EQ>(b));
    }
    // residual GEMV signs: coneqp's rx = P x + q + A'y + G'z, ry = A x - b; conelp's hrx = -A'y - G'z, hry = A x
    const double sgn = LP ? -1.0 : 1.0;
    std::vector<int> flags(B), pairs;
    int it = 0;
    for (it = 0; it <= maxiters; ++it) {
        // residuals (coneqp :2169-2186, conelp :861-896)
        k_res_begin<EQ, LP><<<B, T, 0, st>>>(p); count_launch();
        if (!LP) {
            CVXB_TRY(gemv_t(n, n, b->P.p, b->ldp, nullptr, p.x, 1.0, 1.0, p.rx, st, gP));
            k_res_dots<<<B, T, 0, st>>>(p); count_launch();
        }
        if (EQ) {
            CVXB_TRY(gemv_t(pq, n, b->A.p, b->lda, nullptr, p.y, sgn, 1.0, p.rx, st, gAt));
            CVXB_TRY(gemv_n(pq, n, b->A.p, b->lda, nullptr, p.x, 1.0, -sgn, p.ry, b->gemv_ws.p, st, gAn));
        }
        if (m > 0) {                                              // SDP: G' trisc(z) (misc.sgemv)
            CVXB_TRY(gemv_t(m, n, b->G.p, b->ldg, SDP ? p.rw : nullptr, p.z, sgn, 1.0, p.rx, st, gGt));
            CVXB_TRY(gemv_n(m, n, b->G.p, b->ldg, nullptr, p.x, 1.0, 1.0, p.rz, b->gemv_ws.p, st, gGn));
        }
        CVXB_CUDA(cudaMemsetAsync(b->d_ndone.p, 0, sizeof(int), st));
        if (LP) k_lp_stats<EQ, SDP><<<B, T, 0, st>>>(p, it, maxiters, abstol, reltol, feastol, b->d_ndone.p, b->d_done.p);
        else k_stats<EQ, SDP><<<B, T, 0, st>>>(p, it, maxiters, abstol, reltol, feastol, b->d_ndone.p, b->d_done.p);
        count_launch();
        int ndone = 0;
        bool moved = false;
        CVXB_TRY(poll_done(b, flags, pairs, ndone, moved));
        if (ndone >= B) break;
        B = b->Bact;
        gP.batch = gGt.batch = gGn.batch = gAt.batch = gAn.batch = B;
        if (SDP && it == 0) { k_s_nt_compute<<<dim3(p.ns, B), SB_T, 0, st>>>(p); count_launch(); }
        k_scaling<CONES, LP, SDP><<<B, T, 0, st>>>(p, it == 0 ? 1 : 0); count_launch();
        if (firstcall && it == 0) {              // kkt_chol2's first call; still singular: the Rank ValueError
            CVXB_TRY(start_factor<EQ>(b));
            CVXB_TRY(start_check<EQ>(b));
        } else CVXB_TRY(batch_factor(b));
        if (LP) {
            // (x1, y1, z1) from (-c, b, h) (:1066-1077), th = W^{-T} h
            k_lp_x1_rhs<EQ><<<B, T, 0, st>>>(p); count_launch();
            if (SDP) { k_s_wtz<<<dim3(p.ns, B), SB_T, 0, st>>>(p, p.h, m, nullptr, 0, 1); count_launch(); }
            CVXB_TRY(batch_solve(b, p.x1, n, p.y1, pq));
            k_lp_x1_post<EQ, SDP><<<B, T, 0, st>>>(p); count_launch();
        }
        for (int i = 0; i < 2; ++i) CVXB_TRY((direction<CONES, EQ, LP, SDP>(b, i)));
        if (SDP) { k_s_update<EQ><<<dim3(p.ns, B), SB_T, 0, st>>>(p, b->d_info.p, it == 0); count_launch(); }
        k_update<CONES, EQ, LP, SDP><<<B, T, 0, st>>>(p, b->d_info.p, it); count_launch();
        CVXB_LAUNCH_CHECK();
    }
    return solve_end(b, it);
}

// ---- geometric programs: the lock-step cpl (cvxprog.py:622-1356) of gp's epigraph problem ----
// F(x) over the active slots at x (slot k at x + k*sx): yv = F x, then k_gp_eval (full: with Df, H's rows and weights).
// QC: yv = [P_0 x; ...; P_mnl x], then k_qc_eval (full: with Df; trial: with newrx's nonlinear part)
// yv = F x over the active slots (slot k at x + k*sx); QC: [P_0 x; ...; P_mnl x]
int gp_products(cvxb_batch *b, const double *x, long long sx) {
    const GPPtrs &g = b->gq;
    GemvBatch gf; gf.batch = b->Bact; gf.sA = g.sG; gf.sx = sx; gf.sy = g.sumK;
    return gemv_n(g.sumK, b->n, g.G + b->m, g.ldg, nullptr, x, 1.0, 0.0, g.yv, b->gemv_ws.p, b->st, gf);
}
int gp_eval(cvxb_batch *b, const double *x, long long sx, bool full, int trial) {
    const GPPtrs &g = b->gq;
    const int B = b->Bact;
    CVXB_TRY(gp_products(b, x, sx));
    if (b->kind == Kind::QC) {
        if (full) k_qc_eval<true><<<B, 256, 0, b->st>>>(b->p, g, b->cq);
        else k_qc_eval<false><<<B, 256, 0, b->st>>>(b->p, g, b->cq);
    } else if (full) k_gp_eval<true><<<dim3(g.nK, B), 256, 0, b->st>>>(b->p, g, trial);
    else k_gp_eval<false><<<dim3(g.nK, B), 256, 0, b->st>>>(b->p, g, trial);
    count_launch();
    return 0;
}
// r += Df'[z0; znl] + G' zl (+ A' y) (slot k's z at z + k*m).  GP: Df'[z0; znl] = F'(z_i y) from k_gp_eval's
// weights.  CP: at the iterates (full) k_cp_rx adds it; at trial points k_cp_take<false> has written it into r.
// QC: likewise k_qc_rx and k_qc_eval<false>.  SDP: G' trisc(zl) (misc.sgemv), the row weights rw on the 's' rows
template <bool EQ, bool EPI = true, bool SDP = false>
int gp_rx(cvxb_batch *b, const double *z, const double *y, double *r, bool full) {
    const GPPtrs &g = b->gq;
    const int B = b->Bact, n = b->n, m = b->m, ml = m - g.mnl;
    if (b->kind == Kind::GP) {
        GemvBatch gf; gf.batch = B; gf.sA = g.sG; gf.sx = g.sumK; gf.sy = n;
        CVXB_TRY(gemv_t(g.sumK, n, g.G + m, g.ldg, nullptr, g.wv, 1.0, 1.0, r, b->st, gf));
    } else if (full && b->kind == Kind::QC) {
        k_qc_rx<<<B, 256, 0, b->st>>>(b->p, g); count_launch();
    } else if (full) {
        k_cp_rx<EPI><<<B, 256, 0, b->st>>>(b->p, g, b->cq); count_launch();
    }
    if (ml > 0) {
        GemvBatch gl; gl.batch = B; gl.sA = g.sG; gl.sx = m; gl.sy = n;
        CVXB_TRY(gemv_t(ml, n, g.G + g.mnl, g.ldg, SDP ? b->p.rw + g.mnl : nullptr, z + g.mnl, 1.0, 1.0, r, b->st, gl));
    }
    if (EQ) {
        GemvBatch ga; ga.batch = B; ga.sA = b->sA; ga.sx = b->neq; ga.sy = n;
        CVXB_TRY(gemv_t(b->neq, n, b->A.p, b->lda, nullptr, y, 1.0, 1.0, r, b->st, ga));
    }
    return 0;
}
// H = sum_i z_i Fi'(diag(yi) - yi yi')Fi from k_gp_eval's rows (the reference's syrk with alpha = z[i], :2141-2150),
// lower triangle; mirrored when the refinement's residual multiplies by it, and always for the adjoint (mirror), whose
// refinement step multiplies by H whatever the solve's refinement setting
int gp_hessian(cvxb_batch *b, bool mirror = false) {
    const GPPtrs &g = b->gq;
    GemmDesc h;
    h.M = b->n; h.N = b->n; h.K = g.sumK;
    h.X = g.Hr; h.ldx = (int)g.ldh; h.x_kmajor = true; h.sX = g.sH;
    h.Y = g.Hr; h.ldy = (int)g.ldh; h.y_kmajor = true; h.sY = g.sH;
    h.w = g.hw; h.sW = g.sumK;
    h.C = b->P.p; h.ldc = (int)b->ldp; h.sC = b->sP;
    h.lower_only = true; h.batch = b->Bact;
    if (b->B == 1) h.splitk_ws = b->cw.splitk_ws.p;
    CVXB_TRY(dmma_gemm(h, b->st));
    if (mirror || b->p.refinement) CVXB_TRY(symmetrize_lower(b->n, b->P.p, b->ldp, b->Bact, b->sP, b->st));
    return 0;
}
// a QC batch's H = z0 P_0 + sum_i z_i P_i at the iterates, mirrored when the refinement's residual multiplies by it
int qc_hessian(cvxb_batch *b) {
    const int nb = (b->n + 31) / 32;
    const dim3 grid(nb * (nb + 1) / 2, b->Bact);
    if (b->p.refinement) k_qc_hessian<true><<<grid, 256, 0, b->st>>>(b->p, b->gq, b->cq);
    else k_qc_hessian<false><<<grid, 256, 0, b->st>>>(b->p, b->gq, b->cq);
    count_launch();
    return 0;
}
// the caller's F over the active slots at x (slot k at x + k*n); full: at the iterates, with z = [z0; z[:mnl]] and H
int cp_call(cvxb_batch *b, const double *x, bool full, const char *fn = "batch_solve") {
    const CPPtrs &c = b->cq;
    const int rc = b->cfn(b->cctx, b->Bact, full ? 1 : 0, x, full ? c.z : nullptr, c.idx, c.f, c.Df,
                          full ? c.H : nullptr, (void *)b->st);
    if (rc != 0) { set_error("%s: the evaluation callback returned %d", fn, rc); return CVXB_E_ARG; }
    return 0;
}
// F(x, z[:mnl]) at the iterates: f into fv, grad f0 into gf0, Df[1:] into G's rows [0, mnl); CP also H into P
// (GP forms H in gp_hessian).  EPI false (a cpl batch): Df[:mnl] into G's rows [0, mnl)
template <bool EPI = true> int cpl_eval_full(cvxb_batch *b) {
    if (!b->calls_back()) return gp_eval(b, b->p.x, b->n, true, 0);
    const int B = b->Bact;
    k_cp_zpack<EPI><<<B, 256, 0, b->st>>>(b->p, b->gq, b->cq); count_launch();
    CVXB_TRY(cp_call(b, b->p.x, true));
    k_cp_take<true, EPI><<<B, 256, 0, b->st>>>(b->p, b->gq, b->cq); count_launch();
    if (b->p.refinement) CVXB_TRY(symmetrize_lower(b->n, b->P.p, b->ldp, B, b->sP, b->st));
    return 0;
}
// F at the line search's trial points g.nx, for the problems still searching: f into fv; CP also newrx's nonlinear
// part into nrx (EPI false: c + Df'newznl)
template <bool EPI = true> int cpl_eval_trial(cvxb_batch *b) {
    if (!b->calls_back()) return gp_eval(b, b->gq.nx, b->n, false, 1);
    CVXB_TRY(cp_call(b, b->gq.nx, false));
    k_cp_take<false, EPI><<<b->Bact, 256, 0, b->st>>>(b->p, b->gq, b->cq); count_launch();
    return 0;
}
// slot -> load index for the callback, after a solve's start or a compaction
int cp_upload_idx(cvxb_batch *b) {
    CVXB_CUDA(cudaMemcpyAsync(b->cpi.p, b->perm.data(), (size_t)b->Bact * sizeof(int), cudaMemcpyHostToDevice, b->st));
    return 0;
}
// cp's backtracking into dom f after the i-th direction (:1052-1060): each round evaluates F at every searching
// problem's x + step dx (k_gp_trial) and halves the step of those whose f is not finite; one readback per round.
// dom f is convex, so the merit line search's shorter steps stay inside it
int cp_domain(cvxb_batch *b, int it) {
    cudaStream_t st = b->st;
    const int B = b->Bact;
    for (int left = 1; left > 0; b->ls_rounds++) {
        k_gp_trial<<<B, 256, 0, st>>>(b->p, b->gq); count_launch();
        CVXB_TRY(cp_call(b, b->gq.nx, false));
        CVXB_CUDA(cudaMemsetAsync(b->d_ndone.p, 0, sizeof(int), st));
        k_cp_dom<<<B, 32, 0, st>>>(b->p, b->gq, b->cq, it, b->d_ndone.p); count_launch();
        CVXB_LAUNCH_CHECK();
        CVXB_TRY(read_count(b, left));
    }
    return 0;
}
// the i-th Newton direction of cpl (:966-1045): right-hand side, kktsolver_e's solve and `refinement` steps from
// res() (:889-956), then the step to the boundary and the merit function's slope.  Without the epigraph row (EPI
// false) there is no t to eliminate, and cpl's f4 is coneqp's: the right-hand side is k_dir_rhs's without the
// Mehrotra term (its i = 0), then f4_no_ir around batch_solve and coneqp's refinement residual, 'q' cones included.
// SDP: the 's' blocks' parts of those are direction<..., SDP>'s (k_s_wtz, k_s_res, G' trisc(wz3)); then k_s_steps
// forms their dz2 and ds2, and k_s_dir_post their scale2 and max_step, which in cpl keeps the eigenvectors and
// eigenvalues after either direction (sigs is passed both times, :1042-1045), in syevd's order (k_s_sort)
template <bool EQ, bool EPI = true, bool CONES = false, bool SDP = false> int gp_direction(cvxb_batch *b, int i) {
    cudaStream_t st = b->st;
    const int n = b->n, m = b->m, B = b->Bact, T = 256, pq = b->neq;
    const Ptrs &p = b->p;
    const GPPtrs &g = b->gq;
    const long long L = b->L;
    const dim3 sg(p.ns, B);
    if (EPI) k_gp_dir_rhs<<<B, T, 0, st>>>(p, g);
    else k_dir_rhs<CONES, EQ, false, SDP><<<B, T, 0, st>>>(p, 0);
    count_launch();
    if (SDP) { k_s_wtz<<<sg, SB_T, 0, st>>>(p, p.dz, m, p.ds, m, 2); count_launch(); }
    CVXB_TRY(batch_solve(b, p.dx, n, p.dy, pq));
    if (EPI) k_gp_f4_post<<<B, T, 0, st>>>(p, g, 0);
    else k_f4_post<EQ, SDP><<<B, T, 0, st>>>(p, p.dx, n, p.dz, m, p.ds, m, 0);
    count_launch();
    for (int r = 0; r < p.refinement; ++r) {
        if (SDP) { k_s_res<false><<<sg, SB_T, 0, st>>>(p); count_launch(); }
        if (EPI) k_gp_res<<<B, T, 0, st>>>(p, g);
        else k_res<EQ, false, SDP><<<B, T, 0, st>>>(p);
        count_launch();
        CVXB_TRY((refinement_gemvs<EQ, false, SDP>(b)));     // with the epigraph row: G's rows are [Df[1:]; G]
        if (EPI) k_gp_f4_pre<<<B, T, 0, st>>>(p, g);
        else k_f4_pre<<<B, T, 0, st>>>(p, p.wz2, L, p.ws2, L);
        count_launch();
        if (SDP) { k_s_wtz<<<sg, SB_T, 0, st>>>(p, p.wz2, L, p.ws2, L, 2); count_launch(); }
        CVXB_TRY(batch_solve(b, p.wx2, L, p.wy2, L));
        if (EPI) k_gp_f4_post<<<B, T, 0, st>>>(p, g, 1);
        else k_f4_post<EQ, SDP><<<B, T, 0, st>>>(p, p.wx2, L, p.wz2, L, p.ws2, L, 1);
        count_launch();
    }
    if (SDP) {
        k_s_steps<<<sg, SB_T, 0, st>>>(p, g.ds2, g.dz2); count_launch();
        k_s_dir_post<<<sg, SB_T, 0, st>>>(p, 1); count_launch();
        k_s_sort<<<sg, SB_T, 0, st>>>(p); count_launch();
    }
    k_gp_dir_post<EPI, CONES, SDP><<<B, T, 0, st>>>(p, g, i); count_launch();
    return 0;
}
// the lock-step line search after the i-th direction (:1125-1261): each round evaluates F and newrx at every
// searching problem's trial point and takes its decision; one readback of the count still searching per round
template <bool EQ, bool EPI = true, bool CONES = false, bool SDP = false>
int gp_line_search(cvxb_batch *b, int i, int it) {
    cudaStream_t st = b->st;
    const int B = b->Bact, T = 256;
    const Ptrs &p = b->p;
    const GPPtrs &g = b->gq;
    for (int left = 1; left > 0; b->ls_rounds++) {
        k_gp_trial<<<B, T, 0, st>>>(p, g); count_launch();
        CVXB_TRY(cpl_eval_trial<EPI>(b));
        CVXB_TRY((gp_rx<EQ, EPI, SDP>(b, g.nz, g.ny, g.nrx, false)));
        CVXB_CUDA(cudaMemsetAsync(b->d_ndone.p, 0, sizeof(int), st));
        k_gp_ls<EQ, EPI, CONES, SDP><<<B, T, 0, st>>>(p, g, i, it, b->d_ndone.p, b->qs); count_launch();
        CVXB_LAUNCH_CHECK();
        CVXB_TRY(read_count(b, left));
    }
    return 0;
}
// K = H + [Df[1:]; G]' diag(di²) [Df[1:]; G] (+ A'A) factored from F(x) at the slots' iterates (a GP's H formed
// into P first, a QC batch's too; a CP's is there from cpl_eval_full)
int cpl_factor(cvxb_batch *b, bool first) {
    if (b->kind == Kind::GP) CVXB_TRY(gp_hessian(b));
    else if (b->kind == Kind::QC) CVXB_TRY(qc_hessian(b));
    return batch_factor(b, !first);
}
// the lock-step cpl of a GP or CP batch's epigraph problem (EPI) or of a cpl batch's own problem (EPI false, with 'q'
// cones when CONES).  A CP or cpl batch starts from its x0 and backtracks each step into dom f before the line search;
// it calls back to the host, so the loop is never captured into a graph.  A QC batch starts from its x0 too, and
// takes no domain rounds: its dom f is R^n, and the reference discards the values of its domain evaluation.  Without the epigraph row the scaling and
// the update are coneqp's (k_scaling, k_update: cpl's compute_scaling, ssqr, update_scaling and unscaling are
// coneqp's, and so is mu = gap / (mnl + ml + len(q)), :978).  SDP (a cpl batch with 's' blocks, which follow the 'q'
// rows): the 's' parts of those are the SDP QP batch's, with k_s_nt_compute before iteration 0's scaling, sdot /
// snrm2 / G' trisc(z) in the residuals and stopping rule, k_s_update before the update, and r, rti in the line
// search's saved state; mu's degree counts each block's order
template <bool EQ, bool EPI = true, bool CONES = false, bool SDP = false>
int solve_cpl(cvxb_batch *b, int maxiters, double abstol, double reltol, double feastol) {
    cudaStream_t st = b->st;
    const int n = b->n, m = b->m, T = 256, pq = b->neq;
    const Ptrs &p = b->p;
    const GPPtrs &g = b->gq;
    const int ml = m - g.mnl;
    const bool cb = b->calls_back(), x0 = b->from_x0();
    int B = b->B;
    CVXB_TRY(solve_begin(b));
    // every problem in its own slot (restore_order ran): g (a QC batch's q and r) into the state row, x0 into x
    if (b->glen)
        CVXB_CUDA(cudaMemcpy2DAsync(g.g, b->L * sizeof(double), b->gpg.p, b->glen * sizeof(double),
                                    b->glen * sizeof(double), B, cudaMemcpyDeviceToDevice, st));
    k_gp_init<CONES, SDP><<<B, T, 0, st>>>(p, g); count_launch();
    if (x0) {
        CVXB_CUDA(cudaMemcpyAsync(p.x, b->cpx0.p, (size_t)B * n * sizeof(double), cudaMemcpyDeviceToDevice, st));
        CVXB_TRY(cp_upload_idx(b));
        CVXB_CUDA(cudaMemsetAsync(b->cq.bad, 0x7f, sizeof(int), st));
    }
    std::vector<int> flags(B), pairs;
    int it = 0;
    for (it = 0; it <= maxiters; ++it) {
        // F(x, z[:mnl]) and the residuals (:627-691)
        CVXB_TRY(cpl_eval_full<EPI>(b));
        k_gp_res_begin<EQ, EPI><<<B, T, 0, st>>>(p, g); count_launch();
        CVXB_TRY((gp_rx<EQ, EPI, SDP>(b, p.z, p.y, p.rx, true)));
        if (EQ) {
            GemvBatch ga; ga.batch = B; ga.sA = b->sA; ga.sx = n; ga.sy = pq;
            CVXB_TRY(gemv_n(pq, n, b->A.p, b->lda, nullptr, p.x, 1.0, -1.0, p.ry, b->gemv_ws.p, st, ga));
        }
        if (ml > 0) {
            GemvBatch gl; gl.batch = B; gl.sA = g.sG; gl.sx = n; gl.sy = m;
            CVXB_TRY(gemv_n(ml, n, g.G + g.mnl, g.ldg, nullptr, p.x, 1.0, 1.0, p.rz + g.mnl, b->gemv_ws.p, st, gl));
        }
        CVXB_CUDA(cudaMemsetAsync(b->d_ndone.p, 0, sizeof(int), st));
        k_gp_stats<EQ, EPI, SDP><<<B, T, 0, st>>>(p, g, it, maxiters, abstol, reltol, feastol, b->d_ndone.p,
                                                  b->d_done.p);
        count_launch();
        int ndone = 0, bad = b->B;
        bool moved = false;
        CVXB_TRY(poll_done(b, flags, pairs, ndone, moved, x0 ? &bad : nullptr));
        if (bad < b->B) {                // the reference keeps its iterates inside dom f
            if (it == 0) set_error("batch_solve: problem %d: x0 not in the domain of f", bad);
            else set_error("batch_solve: problem %d: f is not finite at the iterate of iteration %d", bad, it);
            return CVXB_E_ARG;
        }
        if (ndone >= B) break;
        B = b->Bact;
        if (moved) {                     // F(x)'s per-slot results stay put
            if (x0) CVXB_TRY(cp_upload_idx(b));
            CVXB_TRY(cpl_eval_full<EPI>(b));
        }
        if (SDP && it == 0) { k_s_nt_compute<<<dim3(p.ns, B), SB_T, 0, st>>>(p); count_launch(); }
        if (EPI) k_gp_scaling<<<B, T, 0, st>>>(p, g, it == 0 ? 1 : 0);
        else k_scaling<CONES, false, SDP><<<B, T, 0, st>>>(p, it == 0 ? 1 : 0);
        count_launch();
        if (it == 0) {                   // kkt_chol2's first call; still singular: the Rank ValueError (:778-783)
            CVXB_TRY(cpl_factor(b, true));
            CVXB_TRY(first_switch<EQ>(b));
            CVXB_TRY(start_check<EQ>(b));
        } else {
            CVXB_TRY(cpl_factor(b, false));
            CVXB_CUDA(cudaMemsetAsync(b->d_ndone.p, 0, sizeof(int), st));
            k_gp_singular<EQ, EPI, CONES, SDP><<<B, T, 0, st>>>(p, g, b->d_info.p, it, 0, b->d_ndone.p, b->qs);
            count_launch();
            int nre = 0;
            CVXB_TRY(read_count(b, nre));
            if (nre > 0) {               // restored problems are factored again at their saved iterates (and W)
                CVXB_TRY(cpl_eval_full<EPI>(b));
                CVXB_TRY(cpl_factor(b, false));
                k_gp_singular<EQ, EPI, CONES, SDP><<<B, T, 0, st>>>(p, g, b->d_info.p, it, 1, b->d_ndone.p, b->qs);
                count_launch();
            }
        }
        for (int i = 0; i < 2; ++i) {
            CVXB_TRY((gp_direction<EQ, EPI, CONES, SDP>(b, i)));
            if (cb) CVXB_TRY(cp_domain(b, it));
            CVXB_TRY((gp_line_search<EQ, EPI, CONES, SDP>(b, i, it)));
        }
        // SDP: the step the line search left, with sigs and sigz of the last direction (not restored on a resume)
        if (SDP) { k_s_update<EQ><<<dim3(p.ns, B), SB_T, 0, st>>>(p, b->d_info.p, it == 0); count_launch(); }
        if (EPI) k_gp_update<<<B, T, 0, st>>>(p, g);
        else k_update<CONES, EQ, false, SDP><<<B, T, 0, st>>>(p, b->d_info.p, it);
        count_launch();
        CVXB_LAUNCH_CHECK();
    }
    return solve_end(b, it);
}

// dst[problem] = src[slot] for a [B x len] per-slot array, through the slot permutation (d_perm, uploaded by the
// caller) when the last solve compacted
int give_rows(cvxb_batch *b, double *dst, const double *src, int len, int space) {
    const cudaMemcpyKind kind = (space == CVXB_DEVICE) ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
    const size_t B = b->B;
    if (!b->permuted) { CVXB_CUDA(cudaMemcpy(dst, src, B * len * sizeof(double), kind)); return 0; }
    double *tmp = (space == CVXB_DEVICE) ? dst : nullptr;
    if (!tmp) CVXB_CUDA(tmp_malloc(&tmp, B * len * sizeof(double)));
    k_unpermute_rows<<<(unsigned)B, 256, 0, b->st>>>(src, tmp, b->d_perm.p, len);
    count_launch();
    cudaError_t e = cudaStreamSynchronize(b->st);
    if (e == cudaSuccess && tmp != dst) e = cudaMemcpy(dst, tmp, B * len * sizeof(double), kind);
    if (tmp != dst) tmp_free(tmp);
    CVXB_CUDA(e);
    return 0;
}

// every refusal of a creator's arguments, all before the device (fn names the creator): the sizes, the dims of the
// cone rows, which the mnl rows of f precede, and the rank checks before the first factorisation: coneqp's
// (coneprog.py:1962), conelp's (:572-573, with cdim_pckd), cp's and cpl's.  Counts G's rows: mlq 'l' and 'q' rows
// (mnl included), m = mlq + the 's' blocks' s², and mpk = mlq + their s (s + 1) / 2 (cdim_pckd)
int check_args(const char *fn, Kind kind, cvxb_batch **out, int nprob, int n, int p, int mnl, const cvxb_dims *dims,
               bool sdp, long long &mlq, long long &m, long long &mpk) {
    if (out) *out = nullptr;
    if (!out || nprob < 1 || n < 1 || mnl < 0 || !dims) {
        set_error("%s: bad sizes (nprob and n positive, mnl nonnegative, dims given)", fn);
        return CVXB_E_ARG;
    }
    if (p < 0) { set_error("%s: bad sizes (p must be nonnegative)", fn); return CVXB_E_ARG; }
    if (nprob > CVXB_BATCH_MAX) {
        set_error("%s: nprob = %d > %d (the problem index is a grid y/z coordinate)", fn, nprob, CVXB_BATCH_MAX);
        return CVXB_E_ARG;
    }
    if (dims->mnl != 0 || dims->ml < 0 || dims->nq < 0 || dims->ns < 0 || (dims->nq > 0 && !dims->q)) {
        set_error("%s: bad dims (mnl must be 0, ml and the cone counts nonnegative)", fn);
        return CVXB_E_ARG;
    }
    mlq = (long long)mnl + dims->ml;
    for (int k = 0; k < dims->nq; ++k) {
        if (dims->q[k] < 1) { set_error("%s: dims['q'][%d] = %d < 1", fn, k, dims->q[k]); return CVXB_E_ARG; }
        mlq += dims->q[k];
    }
    if (dims->ns > 0 && !sdp) { set_error("%s: 's' cones are not supported by the batch", fn); return CVXB_E_UNSUP; }
    if (dims->ns > 0 && !dims->s) { set_error("%s: dims has ns > 0 and no 's' orders", fn); return CVXB_E_ARG; }
    m = mpk = mlq;
    for (int k = 0; k < dims->ns; ++k) {
        const int s = dims->s[k];
        if (s < 0) { set_error("%s: dims['s'][%d] = %d < 0", fn, k, s); return CVXB_E_ARG; }
        if (s > CVXB_BATCH_SMAX) {
            set_error("%s: dims['s'][%d] = %d > %d, the largest 's' order of the batch", fn, k, s, CVXB_BATCH_SMAX);
            return CVXB_E_UNSUP;
        }
        m += (long long)s * s; mpk += (long long)s * (s + 1) / 2;
    }
    if (m > (1LL << 30)) { set_error("%s: too many rows", fn); return CVXB_E_ARG; }
    // deliberate for a cone LP; cpl's theta1 = 1 / gap0 (cvxprog.py:717) needs a row
    if (m == 0 && (kind == Kind::LP || kind == Kind::CPL)) {
        set_error("%s: no constraint rows (mnl + cdim = 0)", fn);
        return CVXB_E_ARG;
    }
    if (p > n || (kind == Kind::LP && p + mpk < n)) {
        set_error("%s: %s (p = %d, n = %d, cdim = %lld)", fn, rank_text(kind, true), p, n, mpk);
        return CVXB_E_ARG;
    }
    return 0;
}

// a batch of the given kind, once check_args has passed its arguments: QPs, or cone LPs (no P; q holds c), with the
// cones of dims ('l', 'q' and with sdp 's' blocks) and p equality rows; or a GP, CP or cpl batch, whose G begins with
// the mnl rows of Df (counted among the 'l' rows), f having nK = mnl + 1 rows with gp's and cp's epigraph row or nK =
// mnl (cpl).  K: a GP's term counts; the sum K rows of its F go below G's m rows, where a QC batch keeps its nK n
// rows of P_i.  Every buffer of the kind, then the state row
int create(cvxb_batch **out, const char *fn, Kind kind, int nprob, int n, int p, int mnl, const cvxb_dims *dims,
           bool sdp, int device, const int *K = nullptr) {
    long long mlq = 0, mm = 0, mpk = 0;
    CVXB_TRY(check_args(fn, kind, out, nprob, n, p, mnl, dims, sdp, mlq, mm, mpk));
    CVXB_TRY(check_device(device));
    const int m = (int)mm, ml = mnl + dims->ml, nK = kind == Kind::CPL ? mnl : mnl + 1;
    long long sumK = kind == Kind::QC ? (long long)nK * n : 0;        // QC: nK blocks P_i of n rows
    for (int i = 0; K && i < nK; ++i) sumK += K[i];
    std::unique_ptr<cvxb_batch> b(new cvxb_batch());
    b->kind = kind; b->device = device; b->B = nprob; b->n = n; b->m = m;
    b->i8_mode = ozaki_mode();
    b->ldg = ((m + sumK + 1) & ~1) > 2 ? ((m + sumK + 1) & ~1) : 2;
    b->ldp = b->ldk = (n + 1) & ~1;
    b->sG = b->ldg * n; b->sP = b->ldp * n; b->sK = b->ldk * n;
    b->nblk = (n + NB - 1) / NB;
    b->sInv = (long long)2 * b->nblk * NB * NB;
    const size_t B = nprob;
    CVXB_CUDA(cudaStreamCreateWithFlags(&b->st, cudaStreamNonBlocking));
    CVXB_CUDA(cudaEventCreate(&b->e0)); CVXB_CUDA(cudaEventCreate(&b->e1));
    CVXB_TRY(chol_work_create(b->cw));
    if (kind != Kind::LP) CVXB_TRY(b->P.alloc(B * b->sP));
    CVXB_TRY(b->G.alloc(B * b->sG));
    CVXB_TRY(b->K.alloc(B * b->sK));
    CVXB_TRY(b->inv.alloc(B * b->sInv));
    CVXB_TRY(b->panel.alloc(B * (size_t)((n + 1) & ~1) * NB));
    // GEMV workspace: G x (m rows), F x (sum K rows); with equality rows also A x (p rows) and Asct y (n rows)
    const size_t me = (size_t)(m > 0 ? m : 1);
    size_t ws = std::max(me, (size_t)sumK) * gemv_n_chunks(n);
    if (p > 0) ws = std::max({ws, (size_t)p * gemv_n_chunks(n), (size_t)n * gemv_n_chunks(p)});
    CVXB_TRY(b->gemv_ws.alloc(B * ws));
    // vectors: n-sized: q x rx dx ; m-sized: h s z rz ds dz lmbda lmbdasq d di di2 ws3 bzp
    const size_t nv = 4, mv = 13;
    CVXB_TRY(b->vecs.alloc(B * (nv * n + mv * me)));
    CVXB_CUDA(cudaMemset(b->vecs.p, 0, B * (nv * n + mv * me) * sizeof(double)));
    double *v = b->vecs.p;
    auto take = [&](size_t len) { double *r = v; v += B * len; return r; };
    Ptrs &q = b->p;
    q = Ptrs{};
    b->q = take(n); q.x = take(n); q.rx = take(n); q.dx = take(n);
    b->h = take(me); q.s = take(me); q.z = take(me); q.rz = take(me); q.ds = take(me);
    q.dz = take(me); q.lmbda = take(me); q.lmbdasq = take(me); q.d = take(me);
    q.di = take(me); q.di2 = take(me); q.ws3 = take(me); q.bzp = take(me);
    q.q = b->q; q.h = b->h; q.n = n; q.m = m; q.ml = ml;
    CVXB_TRY(b->sc.alloc(B));
    CVXB_CUDA(cudaMemset(b->sc.p, 0, B * sizeof(Scal)));
    q.sc = b->sc.p;
    CVXB_TRY(b->d_info.alloc(B));
    CVXB_TRY(b->d_ndone.alloc(1));
    CVXB_TRY(b->d_done.alloc(B));
    CVXB_TRY(b->d_pairs.alloc(2 * B));
    CVXB_TRY(b->d_perm.alloc(B));
    b->perm.resize(B);
    for (size_t i = 0; i < B; ++i) b->perm[i] = (int)i;
    if (const char *e = getenv("CVXB_BATCH_COMPACT")) b->compact = (e[0] == '0') ? 0 : 1;
    if (dims->nq > 0) {
        const int nq = dims->nq;
        std::vector<int> off(nq + 1, ml);
        for (int k = 0; k < nq; ++k) off[k + 1] = off[k] + dims->q[k];
        CVXB_TRY(b->qoff.alloc(nq + 1));
        CVXB_CUDA(cudaMemcpy(b->qoff.p, off.data(), (nq + 1) * sizeof(int), cudaMemcpyHostToDevice));
        CVXB_TRY(b->Gs.alloc(B * b->sG));
        q.nq = nq; q.qoff = b->qoff.p;
        q.refinement = 1;                         // the default with 'q' cones (coneprog.py:1862-1865)
    }
    b->mpk = (int)mpk;
    q.mlq = (int)mlq; q.mpk = (int)mpk; q.mdg = (int)mlq;
    if (mm > mlq) {                               // 's' blocks of positive order; order 0 adds no rows (:497-499)
        std::vector<int> info;
        std::vector<int> u2p(mm - mlq);
        std::vector<double> rw(m, 1.0);
        long long so = mlq, sp = 0, sro = 0, sgo = 0;
        for (int k = 0; k < dims->ns; ++k) {
            const int s = dims->s[k];
            if (s == 0) continue;
            info.insert(info.end(), {s, (int)so, (int)(mlq + sp), (int)sro, (int)sgo});
            for (int j = 0; j < s; ++j)
                for (int i = 0; i < s; ++i) {
                    const int r = std::max(i, j), c = std::min(i, j);
                    u2p[so - mlq + i + j * s] = (int)(sp + c * s - c * (c - 1) / 2 + r - c);
                    rw[so + i + j * s] = i == j ? 1.0 : (i > j ? 2.0 : 0.0);
                }
            so += (long long)s * s; sp += (long long)s * (s + 1) / 2; sro += (long long)s * s; sgo += s;
        }
        const int ns = (int)info.size() / 5;
        b->sums = sgo; b->sums2 = sro;
        CVXB_TRY(b->sinfo.alloc(info.size()));
        CVXB_CUDA(cudaMemcpy(b->sinfo.p, info.data(), info.size() * sizeof(int), cudaMemcpyHostToDevice));
        CVXB_TRY(b->u2p.alloc(u2p.size()));
        CVXB_CUDA(cudaMemcpy(b->u2p.p, u2p.data(), u2p.size() * sizeof(int), cudaMemcpyHostToDevice));
        CVXB_TRY(b->rw.alloc(rw.size()));
        CVXB_CUDA(cudaMemcpy(b->rw.p, rw.data(), rw.size() * sizeof(double), cudaMemcpyHostToDevice));
        CVXB_TRY(b->spart.alloc(B * ns * 4));
        CVXB_CUDA(cudaMemset(b->spart.p, 0, B * ns * 4 * sizeof(double)));
        if (!b->Gs.p) CVXB_TRY(b->Gs.alloc(B * b->sG));
        q.ns = ns; q.mdg = (int)(mlq + sgo);
        q.sinfo = b->sinfo.p; q.u2p = b->u2p.p; q.rw = b->rw.p; q.spart = b->spart.p;
        q.refinement = 1;                         // the default with 's' cones (coneprog.py:502-507)
    }
    if (p > 0) {
        b->neq = p;
        b->lda = b->ldkp = ((p + 1) & ~1) > 2 ? ((p + 1) & ~1) : 2;
        b->ldas = b->ldk;
        b->sA = b->lda * n; b->sAs = b->ldas * p; b->sKp = b->ldkp * p;
        b->sInvp = (long long)2 * ((p + NB - 1) / NB) * NB * NB;
        CVXB_TRY(b->A.alloc(B * b->sA));
        CVXB_CUDA(cudaMemset(b->A.p, 0, B * b->sA * sizeof(double)));
        CVXB_TRY(b->Asct.alloc(B * b->sAs));
        CVXB_TRY(b->Kp.alloc(B * b->sKp));
        CVXB_TRY(b->invp.alloc(B * b->sInvp));
        CVXB_TRY(b->pvecs.alloc(B * NPV * p));
        CVXB_CUDA(cudaMemset(b->pvecs.p, 0, B * NPV * p * sizeof(double)));
        CVXB_TRY(b->d_infop.alloc(B));
        CVXB_CUDA(cudaMemset(b->d_infop.p, 0, B * sizeof(int)));
        double *w = b->pvecs.p;
        q.neq = p;
        q.beq = w; q.y = w + B * p; q.ry = w + 2 * B * p; q.dy = w + 3 * B * p; q.aw = w + 4 * B * p;
        q.infop = b->d_infop.p;
    }
    if (kind == Kind::LP) {
        const size_t len = (size_t)n + 2 * (size_t)m + (size_t)p;
        CVXB_TRY(b->lpv.alloc(B * len));
        CVXB_CUDA(cudaMemset(b->lpv.p, 0, B * len * sizeof(double)));
        q.x1 = b->lpv.p; q.z1 = q.x1 + B * n; q.th = q.z1 + B * m; q.y1 = q.th + B * m;
    }
    GPPtrs &g = b->gq;
    if (b->cpl_loop()) {
        g.nK = nK; g.sumK = (int)sumK; g.mnl = mnl;
        g.ldg = b->ldg; g.sG = b->sG; g.G = b->G.p;
        // per slot: yv wv hw (sum K; a QC batch has no softmax weights: wv and hw empty) | fv (nK) | gf0 nx nrx (n) |
        // ny (p) | ds2 dz2 nz ns (m)
        const size_t sw = kind == Kind::GP ? sumK : 0;
        const size_t len = sumK + 2 * sw + nK + 3 * (size_t)n + p + 4 * (size_t)m;
        CVXB_TRY(b->gpv.alloc(B * len));
        CVXB_CUDA(cudaMemset(b->gpv.p, 0, B * len * sizeof(double)));
        v = b->gpv.p;
        g.yv = take(sumK); g.wv = take(sw); g.hw = take(sw); g.fv = take(nK);
        g.gf0 = take(n); g.nx = take(n); g.nrx = take(n); g.ny = take(p);
        g.ds2 = take(m); g.dz2 = take(m); g.nz = take(m); g.ns = take(m);
        q.refinement = m > 0 || b->from_x0() ? 1 : 0;     // cpl's default (cvxprog.py:422)
        // per problem, in problem order: a GP's g; a QC batch's q (nK x n), then r (nK)
        b->glen = kind == Kind::GP ? sumK : kind == Kind::QC ? sumK + nK : 0;
        if (b->glen) CVXB_TRY(b->gpg.alloc(B * b->glen));
    }
    if (kind == Kind::GP) {
        g.ldh = (sumK + 1) & ~1LL; g.sH = g.ldh * n;
        std::vector<int> off(nK + 1, 0);
        for (int i = 0; i < nK; ++i) off[i + 1] = off[i] + K[i];
        CVXB_TRY(b->koff.alloc(nK + 1));
        CVXB_CUDA(cudaMemcpy(b->koff.p, off.data(), (nK + 1) * sizeof(int), cudaMemcpyHostToDevice));
        g.koff = b->koff.p;
        CVXB_TRY(b->gph.alloc(B * g.sH));
        g.Hr = b->gph.p;
    }
    CPPtrs &c = b->cq;
    if (b->from_x0()) {                           // x0, the slot -> problem map and the non-finite flag
        CVXB_TRY(b->cpx0.alloc(B * (size_t)n));
        CVXB_TRY(b->cpi.alloc(B + 1));
        c.idx = b->cpi.p; c.bad = b->cpi.p + B;
        c.P = b->P.p; c.ldp = b->ldp; c.sP = b->sP;
    }
    if (b->calls_back()) {                        // the callback's buffers
        const size_t nn = n;
        // per slot: the callback's f, z (nK), Df (nK x n) and H (n x n)
        const size_t len = 2 * nK + nK * nn + nn * nn;
        CVXB_TRY(b->cpv.alloc(B * len));
        CVXB_CUDA(cudaMemset(b->cpv.p, 0, B * len * sizeof(double)));
        c.f = b->cpv.p; c.z = c.f + B * nK; c.Df = c.z + B * nK; c.H = c.Df + B * nK * nn;
    }
    CVXB_TRY(state_alloc(b.get()));
    *out = b.release();
    return 0;
}

// a fresh batch once its data is on the device: every problem in its own slot, A and b still to load
int load_done(cvxb_batch *b) {
    CVXB_CUDA(cudaStreamSynchronize(b->st));
    b->loaded = true;
    b->eq_loaded = false;
    b->solved = false;
    for (int i = 0; i < b->B; ++i) b->perm[i] = i;
    b->permuted = false;
    return 0;
}

// G, h and q (c) of every problem
int load_common(cvxb_batch *b, const double *q, const double *G, const double *h, cudaMemcpyKind kind) {
    const size_t B = b->B, n = b->n, m = b->m;
    // one strided 2-D copy per matrix operand: rows of the "matrix of columns" are the matrix columns
    if (m > 0) {
        CVXB_CUDA(cudaMemcpy2DAsync(b->G.p, b->ldg * sizeof(double), G, m * sizeof(double),
                                    m * sizeof(double), n * B, kind, b->st));
        CVXB_CUDA(cudaMemcpyAsync(const_cast<double *>(b->h), h, B * m * sizeof(double), kind, b->st));
    }
    CVXB_CUDA(cudaMemcpyAsync(const_cast<double *>(b->q), q, B * n * sizeof(double), kind, b->st));
    return load_done(b);
}

// the rows of a GP, CP or cpl batch after its own data: G below the mnl rows of Df, h in the 'l' and 'q' rows (0 on
// the nonlinear ones), q: c (a cpl batch), else 0 (c's x part in the epigraph problem)
int load_cpl_common(cvxb_batch *b, const double *G, const double *h, cudaMemcpyKind kind, const double *c = nullptr) {
    const size_t B = b->B, n = b->n, m = b->m, mnl = b->gq.mnl, ml = m - mnl;
    CVXB_CUDA(cudaMemsetAsync(const_cast<double *>(b->h), 0, B * (m ? m : 1) * sizeof(double), b->st));
    if (ml > 0) {
        CVXB_CUDA(cudaMemcpy2DAsync(b->G.p + mnl, b->ldg * sizeof(double), G, ml * sizeof(double),
                                    ml * sizeof(double), n * B, kind, b->st));
        CVXB_CUDA(cudaMemcpy2DAsync(const_cast<double *>(b->h) + mnl, m * sizeof(double), h, ml * sizeof(double),
                                    ml * sizeof(double), B, kind, b->st));
    }
    if (c) CVXB_CUDA(cudaMemcpyAsync(const_cast<double *>(b->q), c, B * n * sizeof(double), kind, b->st));
    else CVXB_CUDA(cudaMemsetAsync(const_cast<double *>(b->q), 0, B * n * sizeof(double), b->st));
    return load_done(b);
}

// fn(std::bool_constant<f>...) for the runtime flags f: each combination of the flags instantiates fn once, false
// before true with the last flag varying fastest (the order of the kernels in the object file follows it)
template <class Fn> int with_flags(Fn &&fn) { return fn(); }
template <class Fn, class... Rest> int with_flags(Fn &&fn, bool f, Rest... rest) {
    auto bind = [&](auto c) { return with_flags([&](auto... cs) { return fn(c, cs...); }, rest...); };
    if (!f) return bind(std::false_type{});
    return bind(std::true_type{});
}

}  // namespace

extern "C" {

int cvxb_batch_create(cvxb_batch **out, int nprob, int n, int m, int device) {
    cvxb_dims dims{};
    dims.ml = m;
    return create(out, "batch_create", Kind::QP, nprob, n, 0, 0, &dims, false, device);
}

int cvxb_batch_create_cones(cvxb_batch **out, int nprob, int n, const cvxb_dims *dims, int device) {
    return create(out, "batch_create_cones", Kind::QP, nprob, n, 0, 0, dims, false, device);
}

int cvxb_batch_create_eq(cvxb_batch **out, int nprob, int n, int p, const cvxb_dims *dims, int device) {
    return create(out, "batch_create_eq", Kind::QP, nprob, n, p, 0, dims, false, device);
}

int cvxb_batch_create_lp(cvxb_batch **out, int nprob, int n, int p, const cvxb_dims *dims, int device) {
    return create(out, "batch_create_lp", Kind::LP, nprob, n, p, 0, dims, false, device);
}

int cvxb_batch_create_sdp(cvxb_batch **out, int nprob, int n, int p, const cvxb_dims *dims, int device) {
    return create(out, "batch_create_sdp", Kind::LP, nprob, n, p, 0, dims, true, device);
}

int cvxb_batch_create_sdp_qp(cvxb_batch **out, int nprob, int n, int p, const cvxb_dims *dims, int device) {
    return create(out, "batch_create_sdp_qp", Kind::QP, nprob, n, p, 0, dims, true, device);
}

int cvxb_batch_create_gp(cvxb_batch **out, int nprob, int n, int nK, const int *K, int ml, int p, int device) {
    if (out) *out = nullptr;
    if (nK < 1 || !K) { set_error("batch_create_gp: bad sizes (nK >= 1 with K given)"); return CVXB_E_ARG; }
    long long sumK = 0;
    for (int i = 0; i < nK; ++i) {
        if (K[i] < 1) { set_error("batch_create_gp: K[%d] = %d < 1", i, K[i]); return CVXB_E_ARG; }
        sumK += K[i];
    }
    if (sumK + nK + ml > (1LL << 30)) { set_error("batch_create_gp: too many rows"); return CVXB_E_ARG; }
    cvxb_dims d{};
    d.ml = ml;
    return create(out, "batch_create_gp", Kind::GP, nprob, n, p, nK - 1, &d, false, device, K);
}

int cvxb_batch_create_cp(cvxb_batch **out, int nprob, int n, int mnl, int ml, int p, int device) {
    if (out) *out = nullptr;
    if ((long long)mnl + ml + 1 > (1LL << 30)) { set_error("batch_create_cp: too many rows"); return CVXB_E_ARG; }
    cvxb_dims d{};
    d.ml = ml;
    return create(out, "batch_create_cp", Kind::CP, nprob, n, p, mnl, &d, false, device);
}

int cvxb_batch_create_qcqp(cvxb_batch **out, int nprob, int n, int mnl, int ml, int p, int device) {
    if (out) *out = nullptr;
    // G's rows: [Df[1:]; G] and below them the nK = mnl + 1 blocks P_i of n rows, a GP's F with K = (n, ..., n);
    // create counts them
    if ((long long)mnl + ml + 1 + ((long long)mnl + 1) * (n > 0 ? n : 0) > (1LL << 30)) {
        set_error("batch_create_qcqp: too many rows");
        return CVXB_E_ARG;
    }
    cvxb_dims d{};
    d.ml = ml;
    return create(out, "batch_create_qcqp", Kind::QC, nprob, n, p, mnl, &d, false, device);
}

int cvxb_batch_create_cpl(cvxb_batch **out, int nprob, int n, int mnl, const cvxb_dims *dims, int p, int device) {
    return create(out, "batch_create_cpl", Kind::CPL, nprob, n, p, mnl, dims, false, device);
}

int cvxb_batch_create_sdp_cpl(cvxb_batch **out, int nprob, int n, int mnl, const cvxb_dims *dims, int p, int device) {
    return create(out, "batch_create_sdp_cpl", Kind::CPL, nprob, n, p, mnl, dims, true, device);
}

int cvxb_batch_set_cp_eval(cvxb_batch *b, cvxb_cp_eval_fn fn, void *ctx) {
    if (!b) { set_error("batch_set_cp_eval: batch is NULL"); return CVXB_E_ARG; }
    if (!b->calls_back()) { set_error("batch_set_cp_eval: not a CP batch (cvxb_batch_create_cp)"); return CVXB_E_ARG; }
    b->cfn = fn;
    b->cctx = ctx;
    return 0;
}

int cvxb_batch_set_refinement(cvxb_batch *b, int refinement) {
    if (!b || refinement < 0) { set_error("batch_set_refinement: refinement must be a nonnegative integer"); return CVXB_E_ARG; }
    CVXB_CUDA(cudaSetDevice(b->device));
    // a batch without constraint rows takes unrefined steps; a CP or QC batch always has cp's epigraph row
    b->p.refinement = b->m > 0 || b->from_x0() ? refinement : 0;
    CVXB_TRY(state_alloc(b));
    return 0;
}

void cvxb_batch_destroy(cvxb_batch *b) {
    if (!b) return;
    cudaSetDevice(b->device);
    delete b;
}

// P: nprob x (n x n, ld n) ; q: nprob x n ; G: nprob x (m x n column-major, ld m) ; h: nprob x m
int cvxb_batch_load(cvxb_batch *b, const double *P, const double *q, const double *G,
                    const double *h, int space) {
    if (!b || !P || !q || (b->m > 0 && (!G || !h))) { set_error("batch_load: NULL argument"); return CVXB_E_ARG; }
    if (b->kind == Kind::LP) { set_error("batch_load: a cone LP batch is loaded with cvxb_batch_load_lp"); return CVXB_E_ARG; }
    if (b->kind == Kind::GP) { set_error("batch_load: a GP batch is loaded with cvxb_batch_load_gp"); return CVXB_E_ARG; }
    if (b->calls_back()) { set_error("batch_load: a CP batch is loaded with cvxb_batch_load_cp"); return CVXB_E_ARG; }
    if (b->kind == Kind::QC) { set_error("batch_load: a QCQP batch is loaded with cvxb_batch_load_qcqp"); return CVXB_E_ARG; }
    CVXB_CUDA(cudaSetDevice(b->device));
    const cudaMemcpyKind kind = (space == CVXB_DEVICE) ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    const size_t n = b->n;
    CVXB_CUDA(cudaMemcpy2DAsync(b->P.p, b->ldp * sizeof(double), P, n * sizeof(double), n * sizeof(double),
                                n * b->B, kind, b->st));
    // only tril(P) is significant in the reference; make the resident copies symmetric
    CVXB_TRY(symmetrize_lower(b->n, b->P.p, b->ldp, b->B, b->sP, b->st));
    return load_common(b, q, G, h, kind);
}

int cvxb_batch_load_lp(cvxb_batch *b, const double *c, const double *G, const double *h, int space) {
    if (!b || !c || !G || !h) { set_error("batch_load_lp: NULL argument"); return CVXB_E_ARG; }
    if (b->kind != Kind::LP) { set_error("batch_load_lp: a QP, GP or CP batch is not a cone LP batch"); return CVXB_E_ARG; }
    CVXB_CUDA(cudaSetDevice(b->device));
    return load_common(b, c, G, h, (space == CVXB_DEVICE) ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice);
}

int cvxb_batch_load_gp(cvxb_batch *b, const double *F, const double *g, const double *G, const double *h, int space) {
    if (!b || !F || !g || (b->m > b->gq.mnl && (!G || !h))) { set_error("batch_load_gp: NULL argument"); return CVXB_E_ARG; }
    if (b->kind != Kind::GP) { set_error("batch_load_gp: not a GP batch (cvxb_batch_create_gp)"); return CVXB_E_ARG; }
    CVXB_CUDA(cudaSetDevice(b->device));
    const cudaMemcpyKind kind = (space == CVXB_DEVICE) ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    const size_t B = b->B, n = b->n, m = b->m, sK = b->gq.sumK;
    // F below the m rows of [Df[1:]; G]
    CVXB_CUDA(cudaMemcpy2DAsync(b->G.p + m, b->ldg * sizeof(double), F, sK * sizeof(double), sK * sizeof(double),
                                n * B, kind, b->st));
    CVXB_CUDA(cudaMemcpyAsync(b->gpg.p, g, B * sK * sizeof(double), kind, b->st));
    return load_cpl_common(b, G, h, kind);
}

int cvxb_batch_load_cp(cvxb_batch *b, const double *x0, const double *G, const double *h, int space) {
    if (!b || !x0 || (b->m > b->gq.mnl && (!G || !h))) { set_error("batch_load_cp: NULL argument"); return CVXB_E_ARG; }
    if (b->kind != Kind::CP) { set_error("batch_load_cp: not a CP batch (cvxb_batch_create_cp)"); return CVXB_E_ARG; }
    CVXB_CUDA(cudaSetDevice(b->device));
    const cudaMemcpyKind kind = (space == CVXB_DEVICE) ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    CVXB_CUDA(cudaMemcpyAsync(b->cpx0.p, x0, (size_t)b->B * b->n * sizeof(double), kind, b->st));
    return load_cpl_common(b, G, h, kind);
}

int cvxb_batch_load_cpl(cvxb_batch *b, const double *c, const double *x0, const double *G, const double *h, int space) {
    if (!b || !c || !x0 || (b->m > b->gq.mnl && (!G || !h))) { set_error("batch_load_cpl: NULL argument"); return CVXB_E_ARG; }
    if (b->kind != Kind::CPL) { set_error("batch_load_cpl: not a cpl batch (cvxb_batch_create_cpl)"); return CVXB_E_ARG; }
    CVXB_CUDA(cudaSetDevice(b->device));
    const cudaMemcpyKind kind = (space == CVXB_DEVICE) ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    CVXB_CUDA(cudaMemcpyAsync(b->cpx0.p, x0, (size_t)b->B * b->n * sizeof(double), kind, b->st));
    return load_cpl_common(b, G, h, kind, c);
}

int cvxb_batch_load_qcqp(cvxb_batch *b, const double *P, const double *q, const double *r, const double *x0,
                         const double *G, const double *h, int space) {
    if (!b || !P || !q || !r || (b->m > b->gq.mnl && (!G || !h))) { set_error("batch_load_qcqp: NULL argument"); return CVXB_E_ARG; }
    if (b->kind != Kind::QC) { set_error("batch_load_qcqp: not a QCQP batch (cvxb_batch_create_qcqp)"); return CVXB_E_ARG; }
    CVXB_CUDA(cudaSetDevice(b->device));
    const cudaMemcpyKind kind = (space == CVXB_DEVICE) ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    const size_t B = b->B, n = b->n, m = b->m, nK = b->gq.nK, S = b->gq.sumK, gl = b->glen;
    // [P_0; ...; P_mnl] below the m rows of [Df[1:]; G], each block mirrored from its lower triangle
    CVXB_CUDA(cudaMemcpy2DAsync(b->G.p + m, b->ldg * sizeof(double), P, S * sizeof(double), S * sizeof(double),
                                n * B, kind, b->st));
    for (size_t i = 0; i < nK; ++i) CVXB_TRY(symmetrize_lower(b->n, b->G.p + m + i * n, b->ldg, b->B, b->sG, b->st));
    // q and r in problem order, copied into the state row by each solve
    CVXB_CUDA(cudaMemcpy2DAsync(b->gpg.p, gl * sizeof(double), q, S * sizeof(double), S * sizeof(double), B, kind,
                                b->st));
    CVXB_CUDA(cudaMemcpy2DAsync(b->gpg.p + S, gl * sizeof(double), r, nK * sizeof(double), nK * sizeof(double), B,
                                kind, b->st));
    if (x0) CVXB_CUDA(cudaMemcpyAsync(b->cpx0.p, x0, B * n * sizeof(double), kind, b->st));
    else CVXB_CUDA(cudaMemsetAsync(b->cpx0.p, 0, B * n * sizeof(double), b->st));
    return load_cpl_common(b, G, h, kind);
}

int cvxb_batch_ls_rounds(cvxb_batch *b) { return b ? b->ls_rounds : CVXB_E_ARG; }

int cvxb_batch_load_eq(cvxb_batch *b, const double *A, const double *bvec, int space) {
    if (!b) { set_error("batch_load_eq: batch is NULL"); return CVXB_E_ARG; }
    if (b->neq == 0) return 0;
    if (!A || !bvec) { set_error("batch_load_eq: NULL argument"); return CVXB_E_ARG; }
    if (!b->loaded) { set_error("batch_load_eq: call cvxb_batch_load first"); return CVXB_E_ARG; }
    CVXB_CUDA(cudaSetDevice(b->device));
    CVXB_TRY(restore_order(b));                  // A and b are written to the problems' own slots
    const cudaMemcpyKind kind = (space == CVXB_DEVICE) ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    const size_t B = b->B, n = b->n, pq = b->neq;
    CVXB_CUDA(cudaMemcpy2DAsync(b->A.p, b->lda * sizeof(double), A, pq * sizeof(double), pq * sizeof(double),
                                n * B, kind, b->st));
    CVXB_CUDA(cudaMemcpyAsync(const_cast<double *>(b->p.beq), bvec, B * pq * sizeof(double), kind, b->st));
    CVXB_CUDA(cudaStreamSynchronize(b->st));
    b->eq_loaded = true;
    b->solved = false;
    return 0;
}

int cvxb_batch_load_start(cvxb_batch *b, const double *x, const double *s, const double *y, const double *z,
                          int space) {
    if (!b) { set_error("batch_load_start: batch is NULL"); return CVXB_E_ARG; }
    if (b->kind == Kind::GP) { set_error("batch_load_start: gp takes no starting point"); return CVXB_E_ARG; }
    if (b->calls_back()) { set_error("batch_load_start: cp and cpl start from the x0 of their load"); return CVXB_E_ARG; }
    if (b->kind == Kind::QC) { set_error("batch_load_start: qcqp starts from the x0 of its load"); return CVXB_E_ARG; }
    if (b->kind == Kind::LP && ((!x) != (!s) || (y && !z) || (!x && !z))) {
        set_error("batch_load_start: a cone LP start is x and s (primalstart), z with an optional y (dualstart), or "
                  "both");
        return CVXB_E_ARG;
    }
    CVXB_CUDA(cudaSetDevice(b->device));
    const size_t B = b->B, n = b->n, m = b->m, pq = b->neq;
    if (!b->start.p) CVXB_TRY(b->start.alloc(B * (n + pq + 2 * m)));
    double *x0 = b->start.p, *y0 = x0 + B * n, *s0 = y0 + B * pq, *z0 = s0 + B * m;
    const cudaMemcpyKind kind = (space == CVXB_DEVICE) ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    b->warm_set = false;                          // a failed copy leaves no start
    if (x) CVXB_CUDA(cudaMemcpyAsync(x0, x, B * n * sizeof(double), kind, b->st));
    if (y && pq) CVXB_CUDA(cudaMemcpyAsync(y0, y, B * pq * sizeof(double), kind, b->st));
    if (s && m) CVXB_CUDA(cudaMemcpyAsync(s0, s, B * m * sizeof(double), kind, b->st));
    if (z && m) CVXB_CUDA(cudaMemcpyAsync(z0, z, B * m * sizeof(double), kind, b->st));
    CVXB_CUDA(cudaStreamSynchronize(b->st));
    b->warm = Warm{x ? x0 : nullptr, (y && pq) ? y0 : nullptr, (s && m) ? s0 : nullptr, (z && m) ? z0 : nullptr};
    b->warm_set = true;
    return 0;
}

int cvxb_batch_clear_start(cvxb_batch *b) {
    if (!b) { set_error("batch_clear_start: batch is NULL"); return CVXB_E_ARG; }
    b->warm = Warm{};
    b->warm_set = false;
    return 0;
}

int cvxb_batch_solve(cvxb_batch *b, int maxiters, double abstol, double reltol, double feastol) {
    if (!b || !b->loaded) { set_error("batch_solve: load the problems first"); return CVXB_E_ARG; }
    if (b->neq > 0 && !b->eq_loaded) {
        set_error("batch_solve: the batch has p = %d equality rows: load A and b (cvxb_batch_load_eq) after "
                  "cvxb_batch_load", b->neq);
        return CVXB_E_ARG;
    }
    CVXB_CUDA(cudaSetDevice(b->device));
    b->solved = false;
    CVXB_TRY(restore_order(b));
    if (b->calls_back() && !b->cfn) { set_error("batch_solve: a CP batch needs its F (cvxb_batch_set_cp_eval)"); return CVXB_E_ARG; }
    // SDP: 's' blocks of positive order
    const bool sdp = b->p.ns > 0, lp = b->kind == Kind::LP, eq = b->neq > 0, cones = b->p.nq > 0;
    int rc = 0;
    if (b->kind == Kind::CPL)
        rc = with_flags([&](auto SDP, auto CONES, auto EQ) {
            return solve_cpl<EQ, false, CONES, SDP>(b, maxiters, abstol, reltol, feastol);
        }, sdp, cones, eq);
    else if (b->cpl_loop())                       // GP, CP, QC: the epigraph problem, 'l' rows only
        rc = eq ? solve_cpl<true>(b, maxiters, abstol, reltol, feastol)
                : solve_cpl<false>(b, maxiters, abstol, reltol, feastol);
    else
        rc = with_flags([&](auto SDP, auto LP, auto EQ, auto CONES) {
            return solve<CONES, EQ, LP, SDP>(b, maxiters, abstol, reltol, feastol);
        }, sdp, lp, eq, cones);
    b->solved = rc == 0;
    return rc;
}

namespace {
// the gradient outputs of an adjoint call (nullptr: not written); dq and dr are a QCQP batch's only, dF and dg a GP
// batch's
struct AdjGrads {
    double *dP = nullptr, *dq = nullptr, *dr = nullptr, *dG = nullptr, *dA = nullptr;
    double *dF = nullptr, *dg = nullptr;
};
// kkt_chol2's switch at the adjoint's factorisation (misc.py:1421-1447), once batch_factor has run: a problem whose
// S is singular there factors S + A'A, next to those the solve already switched.  Without P, at a converged iterate
// whose W'W spans many orders of magnitude, G' W^{-1} W^{-T} G is numerically singular when fewer than n rows are
// active, which a cone LP's vertex has with equality rows.  aw0: the solve's aw (slot order), for batch_adjoint to
// restore; empty when every factorisation succeeded and nothing changed
int adj_switch(cvxb_batch *b, std::vector<double> &aw0) {
    cudaStream_t st = b->st;
    const int B = b->B, pq = b->neq;
    std::vector<int> info(B);
    CVXB_CUDA(cudaMemcpyAsync(info.data(), b->d_info.p, B * sizeof(int), cudaMemcpyDeviceToHost, st));
    CVXB_CUDA(cudaStreamSynchronize(st));
    if (std::none_of(info.begin(), info.end(), [](int v) { return v > 0; })) return 0;
    aw0.resize((size_t)B * pq);
    CVXB_CUDA(cudaMemcpyAsync(aw0.data(), b->p.aw, aw0.size() * sizeof(double), cudaMemcpyDeviceToHost, st));
    CVXB_CUDA(cudaStreamSynchronize(st));
    for (int i = 0; i < B; ++i) info[i] = info[i] > 0 || aw0[(size_t)i * pq] != 0.0;   // k_switch's flags
    CVXB_CUDA(cudaMemcpyAsync(b->d_pairs.p, info.data(), B * sizeof(int), cudaMemcpyHostToDevice, st));
    k_switch<<<(unsigned)B, 256, 0, st>>>(b->p.aw, b->d_pairs.p, pq); count_launch();
    b->switched = true;
    return batch_factor(b);
}

// the adjoint of a solved QP, cone LP, QC or GP batch (the entry points check the kind and the solve): the right-hand
// side, for a QC or GP batch its operator at x (H in P, Df in G's rows [0, mnl)), the reduced solve, one refinement
// step on the full system, then ux, uy, uz and the gradients.  QC: dP is the (nK n) x n stack, dq nK x n, dr nK and dG
// ml x n per problem.  GP: dF is S x n, dg S and dG ml x n per problem; the call overwrites P, G's Df rows, yv, wv, Hr,
// hw and fv, all of which a solve rewrites before it reads them.  CP and cpl: the caller's F(x, zk) once, through the
// callback, on every slot in its caller-order index; dG is ml x n per problem (k_adj_qc_grad's), and the call
// overwrites P, G's Df rows, the callback's buffers, cpi and d_done (each slot's non-finite flag).  With 'q' cones or
// 's' blocks k_adj_cone and the 's' kernels fix the cone rows between the 'l' steps; a cone LP has no P (its entry
// point refuses dP)
int batch_adjoint(cvxb_batch *b, const double *gx, const double *gy, const double *gz, double *ux, double *uy,
                  double *uz, AdjGrads d, int space) {
    CVXB_CUDA(cudaSetDevice(b->device));
    cudaStream_t st = b->st;
    const bool qc = b->kind == Kind::QC, lp = b->kind == Kind::LP, gp = b->kind == Kind::GP;
    const bool cp = b->calls_back(), epi = b->kind == Kind::CP;
    const bool cones = b->p.nq > 0 || b->p.ns > 0, sdp = b->p.ns > 0;
    const size_t B = b->B, n = b->n, m = b->m, pq = b->neq, nK = qc ? b->gq.nK : 1;
    const size_t ml = qc || gp || cp ? m - b->gq.mnl : m, S = gp ? b->gq.sumK : 0;
    const Ptrs &p = b->p;
    const GPPtrs &g = b->gq;
    // host space: every given array staged on the device (inputs uploaded, outputs copied back); device: in place
    Staged s_gx, s_gy, s_gz, s_ux, s_uy, s_uz, s_dP, s_dq, s_dr, s_dG, s_dA, s_dF, s_dg;
    auto stage = [&](Staged &s, const double *a, size_t len, bool in) -> int {
        if (a && len) CVXB_TRY(s.in(a, B * len, space, st, in));
        return 0;
    };
    CVXB_TRY(stage(s_gx, gx, n, true)); CVXB_TRY(stage(s_gy, gy, pq, true)); CVXB_TRY(stage(s_gz, gz, m, true));
    CVXB_TRY(stage(s_ux, ux, n, false)); CVXB_TRY(stage(s_uy, uy, pq, false)); CVXB_TRY(stage(s_uz, uz, m, false));
    CVXB_TRY(stage(s_dP, d.dP, nK * n * n, false));
    if (qc) { CVXB_TRY(stage(s_dq, d.dq, nK * n, false)); CVXB_TRY(stage(s_dr, d.dr, nK, false)); }
    if (gp) { CVXB_TRY(stage(s_dF, d.dF, S * n, false)); CVXB_TRY(stage(s_dg, d.dg, S, false)); }
    CVXB_TRY(stage(s_dG, d.dG, ml * n, false));
    CVXB_TRY(stage(s_dA, d.dA, pq * n, false));
    b->Bact = b->B;
    CVXB_CUDA(cudaMemcpyAsync(b->d_perm.p, b->perm.data(), B * sizeof(int), cudaMemcpyHostToDevice, st));
    k_adj_rhs<<<(unsigned)B, 256, 0, st>>>(p, s_gx.dev, s_gy.dev, s_gz.dev, b->d_perm.p); count_launch();
    const dim3 sg(p.ns, (unsigned)B);                  // one CTA per ('s' block, slot)
    if (cones) { k_adj_cone<<<(unsigned)B, 256, 0, st>>>(p, b->d_info.p, 0); count_launch(); }
    if (sdp) {
        k_adj_s_nt<<<sg, SB_T, 0, st>>>(p); count_launch();
        k_s_wtz<<<sg, SB_T, 0, st>>>(p, p.rz, (long long)m, nullptr, 0, 0); count_launch();
    }
    if (qc) {
        CVXB_TRY(gp_products(b, p.x, n));
        const long long work = std::max(n * n, (size_t)b->gq.mnl * n);
        k_adj_qc_op<<<dim3((unsigned)((work + 255) / 256), (unsigned)B), 256, 0, st>>>(p, b->gq, b->cq);
        count_launch();
    }
    if (gp) {
        CVXB_TRY(gp_products(b, p.x, n));
        k_adj_gp_op<<<dim3((unsigned)g.nK, (unsigned)B), 256, 0, st>>>(p, g); count_launch();
        CVXB_TRY(gp_hessian(b, true));
    }
    if (cp) {                                            // F(x, zk): H, Df and the flags; P mirrored for the refinement
        CVXB_TRY(cp_upload_idx(b));
        k_adj_cp_zpack<<<(unsigned)B, 32, 0, st>>>(p, g, b->cq, epi ? 1 : 0); count_launch();
        CVXB_TRY(cp_call(b, p.x, true, "batch_adjoint_cp"));
        if (epi) k_adj_cp_take<true><<<(unsigned)B, 256, 0, st>>>(p, g, b->cq, b->d_done.p);
        else k_adj_cp_take<false><<<(unsigned)B, 256, 0, st>>>(p, g, b->cq, b->d_done.p);
        count_launch();
        CVXB_TRY(symmetrize_lower(b->n, b->P.p, b->ldp, b->Bact, b->sP, st));
    }
    CVXB_TRY(batch_factor(b));
    std::vector<double> aw0;                             // the solve's aw when adj_switch changed it
    const bool switched0 = b->switched;
    // a GP whose terms are all monomials is an LP, and S can be singular at its vertices as at a cone LP's; so can a
    // CP or cpl batch's, whose f the caller chooses
    if (pq && (lp || cones || gp || cp)) CVXB_TRY(adj_switch(b, aw0));
    if (cp) {
        k_adj_cp_flag<<<(unsigned)((B + 255) / 256), 256, 0, st>>>(b->d_info.p, b->d_done.p, (int)B);
        count_launch();
    }
    CVXB_TRY(batch_solve(b, p.dx, n, p.dy, pq));
    // one step of iterative refinement on the full KKT system: W'W spans many orders of magnitude at a converged
    // iterate, and the reduced solve alone loses digits to it.  r = g - M u, then u += M^{-1} r with the same factor
    const int Bi = (int)B, ni = (int)n, mi = (int)m, pi = (int)pq;
    k_adj_uz<<<(unsigned)B, 256, 0, st>>>(p); count_launch();
    // the info that k_adj_cone sets for a failed 's' scaling is the factorisation's, so it goes after batch_factor
    if (cones) { k_adj_cone<<<(unsigned)B, 256, 0, st>>>(p, b->d_info.p, 1); count_launch(); }
    if (sdp) { k_adj_s<<<sg, SB_T, 0, st>>>(p, 0); count_launch(); }
    if (!lp) {
        GemvBatch gP; gP.batch = Bi; gP.sA = b->sP; gP.sx = ni; gP.sy = ni;
        CVXB_TRY(gemv_t(ni, ni, b->P.p, b->ldp, nullptr, p.dx, -1.0, 1.0, p.rx, st, gP));
    }
    if (pq) {
        GemvBatch gt; gt.batch = Bi; gt.sA = b->sA; gt.sx = pi; gt.sy = ni;
        CVXB_TRY(gemv_t(pi, ni, b->A.p, b->lda, nullptr, p.dy, -1.0, 1.0, p.rx, st, gt));
        GemvBatch gn; gn.batch = Bi; gn.sA = b->sA; gn.sx = ni; gn.sy = pi;
        CVXB_TRY(gemv_n(pi, ni, b->A.p, b->lda, nullptr, p.dx, -1.0, 1.0, p.ry, b->gemv_ws.p, st, gn));
    }
    if (m) {                                           // 's' blocks: G' trisc(uz), the G the solver reads (rw)
        GemvBatch gt; gt.batch = Bi; gt.sA = b->sG; gt.sx = mi; gt.sy = ni;
        CVXB_TRY(gemv_t(mi, ni, b->G.p, b->ldg, p.rw, p.dz, -1.0, 1.0, p.rx, st, gt));
        GemvBatch gn; gn.batch = Bi; gn.sA = b->sG; gn.sx = ni; gn.sy = mi;
        CVXB_TRY(gemv_n(mi, ni, b->G.p, b->ldg, nullptr, p.dx, -1.0, 1.0, p.rz, b->gemv_ws.p, st, gn));
    }
    k_adj_res<<<(unsigned)B, 256, 0, st>>>(p); count_launch();
    if (p.nq) { k_adj_cone<<<(unsigned)B, 256, 0, st>>>(p, b->d_info.p, 2); count_launch(); }
    if (sdp) { k_adj_s<<<sg, SB_T, 0, st>>>(p, 1); count_launch(); }
    CVXB_TRY(batch_solve(b, p.rx, n, p.ry, pq));
    if (sdp) { k_adj_s<<<sg, SB_T, 0, st>>>(p, 2); count_launch(); }
    if (cones) { k_adj_cone<<<(unsigned)B, 256, 0, st>>>(p, b->d_info.p, 3); count_launch(); }
    k_adj_vecs<<<(unsigned)B, 256, 0, st>>>(p, s_ux.dev, s_uy.dev, s_uz.dev, b->d_perm.p, b->d_info.p);
    count_launch();
    const dim3 grid((unsigned)((n + ADJ_TJ - 1) / ADJ_TJ), (unsigned)B);
    if (gp) {
        if (s_dF.dev || s_dg.dev) {                      // w = F ux into wv (yv holds pi), then dg in its place
            GemvBatch gw; gw.batch = Bi; gw.sA = g.sG; gw.sx = ni; gw.sy = g.sumK;
            CVXB_TRY(gemv_n(g.sumK, ni, g.G + m, g.ldg, nullptr, p.dx, 1.0, 0.0, g.wv, b->gemv_ws.p, st, gw));
            k_adj_gp_dg<<<dim3((unsigned)g.nK, (unsigned)B), 256, 0, st>>>(p, g, s_dg.dev, b->d_perm.p,
                                                                           b->d_info.p);
            count_launch();
        }
        if (s_dF.dev || s_dG.dev || s_dA.dev) {
            k_adj_gp_grad<<<grid, 256, 0, st>>>(p, g, s_dF.dev, s_dG.dev, s_dA.dev, b->d_perm.p, b->d_info.p);
            count_launch();
        }
    } else if (s_dP.dev || s_dq.dev || s_dr.dev || s_dG.dev || s_dA.dev) {
        // CP and cpl: dG over rows mnl.. and dA only, whose formulas are the QC batch's
        if (qc || cp) k_adj_qc_grad<<<grid, 256, 0, st>>>(p, b->gq, s_dP.dev, s_dq.dev, s_dr.dev, s_dG.dev, s_dA.dev,
                                                    b->d_perm.p, b->d_info.p);
        else k_adj_grad<<<grid, 256, 0, st>>>(p, s_dP.dev, s_dG.dev, s_dA.dev, b->d_perm.p, b->d_info.p);
        count_launch();
    }
    CVXB_LAUNCH_CHECK();
    for (Staged *s : {&s_ux, &s_uy, &s_uz, &s_dP, &s_dq, &s_dr, &s_dG, &s_dA, &s_dF, &s_dg}) CVXB_TRY(s->out(st));
    if (!aw0.empty()) {                                  // the solver's state as the solve left it
        CVXB_CUDA(cudaMemcpyAsync(p.aw, aw0.data(), aw0.size() * sizeof(double), cudaMemcpyHostToDevice, st));
        b->switched = switched0;
    }
    CVXB_CUDA(cudaStreamSynchronize(st));
    return 0;
}

// the tangent of a solved batch along d (the entry points check the kind and the solve): r(d) into the outputs (a NULL
// output's part of r into temporary device memory), then batch_adjoint with g = r, which reads g before it writes u
int batch_tangent(cvxb_batch *b, TanIn d, double *dx, double *dy, double *dz, int space) {
    CVXB_CUDA(cudaSetDevice(b->device));
    cudaStream_t st = b->st;
    const bool qc = b->kind == Kind::QC, gp = b->kind == Kind::GP, cp = b->calls_back();
    const size_t B = b->B, n = b->n, m = b->m, pq = b->neq, nK = b->gq.nK, mnl = b->gq.mnl;
    const size_t ml = qc || gp || cp ? m - mnl : m, S = gp ? b->gq.sumK : 0;
    Staged s_dP, s_dq, s_dr, s_dF, s_dg, s_tx, s_tf, s_dG, s_dh, s_dA, s_db, s_dx, s_dy, s_dz;
    auto in = [&](Staged &s, const double *a, size_t len, const double *&o) -> int {
        o = nullptr;
        if (a && len) { CVXB_TRY(s.in(a, B * len, space, st)); o = s.dev; }
        return 0;
    };
    TanIn t{};
    const size_t sq = qc ? nK : 1;                       // P and q blocks per problem
    CVXB_TRY(in(s_dP, d.dP, sq * n * n, t.dP)); CVXB_TRY(in(s_dq, d.dq, sq * n, t.dq));
    if (qc) CVXB_TRY(in(s_dr, d.dr, nK, t.dr));
    if (gp) { CVXB_TRY(in(s_dF, d.dF, S * n, t.dF)); CVXB_TRY(in(s_dg, d.dg, S, t.dg)); }
    if (cp) { CVXB_TRY(in(s_tx, d.tx, n, t.tx)); CVXB_TRY(in(s_tf, d.tf, mnl, t.tf)); }
    CVXB_TRY(in(s_dG, d.dG, ml * n, t.dG)); CVXB_TRY(in(s_dh, d.dh, ml, t.dh));
    CVXB_TRY(in(s_dA, d.dA, pq * n, t.dA)); CVXB_TRY(in(s_db, d.db, pq, t.db));
    Scratch<double> tmp;                                 // r's parts whose outputs are NULL
    const size_t tn = (dx ? 0 : n) + (dy ? 0 : pq) + (dz ? 0 : m);
    if (tn) CVXB_TRY(tmp.alloc(B * tn));
    double *next = tmp.p;
    auto out = [&](Staged &s, double *a, size_t len, double *&o) -> int {
        if (!a) { o = next; next += B * len; return 0; }
        CVXB_TRY(s.in(a, B * len, space, st, false));
        o = s.dev;
        return 0;
    };
    double *rx, *ry, *rz;
    CVXB_TRY(out(s_dx, dx, n, rx)); CVXB_TRY(out(s_dy, dy, pq, ry)); CVXB_TRY(out(s_dz, dz, m, rz));
    CVXB_CUDA(cudaMemcpyAsync(b->d_perm.p, b->perm.data(), B * sizeof(int), cudaMemcpyHostToDevice, st));
    const Ptrs &p = b->p;
    if (qc) k_tan_rhs_qc<<<(unsigned)B, TAN_T, 0, st>>>(p, b->gq, t, rx, ry, rz, b->d_perm.p);
    else if (gp) k_tan_rhs_gp<<<(unsigned)B, TAN_T, 0, st>>>(p, b->gq, t, rx, ry, rz, b->d_perm.p);
    else if (cp) k_tan_rhs_cp<<<(unsigned)B, TAN_T, 0, st>>>(p, b->gq, t, rx, ry, rz, b->d_perm.p);
    else k_tan_rhs<<<(unsigned)B, TAN_T, 0, st>>>(p, t, rx, ry, rz, b->d_perm.p);
    count_launch();
    CVXB_LAUNCH_CHECK();
    CVXB_TRY(batch_adjoint(b, rx, ry, rz, dx ? rx : nullptr, dy ? ry : nullptr, dz ? rz : nullptr, AdjGrads{},
                           CVXB_DEVICE));
    for (Staged *s : {&s_dx, &s_dy, &s_dz}) CVXB_TRY(s->out(st));
    CVXB_CUDA(cudaStreamSynchronize(st));
    return 0;
}
}  // namespace

namespace {
// the checks every derivative entry point makes, in this order: a batch (b not NULL), of a kind the entry point
// differentiates (ok, else the refusal unsup), without an argument its kind lacks (bad, else the refusal arg), solved
// since its last load.  ok and bad are evaluated by the caller, so they test b before they read it
int deriv_checks(cvxb_batch *b, const char *what, bool ok, const char *unsup, bool bad = false,
                 const char *arg = nullptr) {
    if (!b) { set_error("%s: batch is NULL", what); return CVXB_E_ARG; }
    if (!ok) { set_error("%s: %s", what, unsup); return CVXB_E_UNSUP; }
    if (bad) { set_error("%s: %s", what, arg); return CVXB_E_ARG; }
    if (b->solved) return 0;
    set_error("%s: no completed cvxb_batch_solve since the last load", what);
    return CVXB_E_ARG;
}
const char *const QC_ONLY = "only QCQP batches (cvxb_batch_create_qcqp) are differentiated here";
const char *const GP_ONLY = "only GP batches (cvxb_batch_create_gp) are differentiated here";
const char *const CP_ONLY = "only CP and cpl batches (cvxb_batch_create_cp, _cpl, _sdp_cpl) are differentiated here";
const char *const CONE_ONLY = "only QP and cone LP batches are differentiated here";
bool qp_or_lp(const cvxb_batch *b) { return b && (b->kind == Kind::QP || b->kind == Kind::LP); }
bool lp_with_dP(const cvxb_batch *b, const double *dP) { return b && b->kind == Kind::LP && dP; }
}  // namespace

int cvxb_batch_adjoint(cvxb_batch *b, const double *gx, const double *gy, const double *gz, double *ux, double *uy,
                       double *uz, double *dP, double *dG, double *dA, int space) {
    CVXB_TRY(deriv_checks(b, "batch_adjoint", b && b->kind == Kind::QP && b->p.nq == 0 && b->p.ns == 0,
                          "only QP batches whose rows are all 'l' are differentiated"));
    return batch_adjoint(b, gx, gy, gz, ux, uy, uz, AdjGrads{dP, nullptr, nullptr, dG, dA}, space);
}

int cvxb_batch_adjoint_qcqp(cvxb_batch *b, const double *gx, const double *gy, const double *gz, double *ux,
                            double *uy, double *uz, double *dP, double *dq, double *dr, double *dG, double *dA,
                            int space) {
    CVXB_TRY(deriv_checks(b, "batch_adjoint_qcqp", b && b->kind == Kind::QC, QC_ONLY));
    return batch_adjoint(b, gx, gy, gz, ux, uy, uz, AdjGrads{dP, dq, dr, dG, dA}, space);
}

int cvxb_batch_adjoint_gp(cvxb_batch *b, const double *gx, const double *gy, const double *gz, double *ux, double *uy,
                          double *uz, double *dF, double *dg, double *dG, double *dA, int space) {
    CVXB_TRY(deriv_checks(b, "batch_adjoint_gp", b && b->kind == Kind::GP, GP_ONLY));
    AdjGrads d;
    d.dF = dF; d.dg = dg; d.dG = dG; d.dA = dA;
    return batch_adjoint(b, gx, gy, gz, ux, uy, uz, d, space);
}

int cvxb_batch_adjoint_cp(cvxb_batch *b, const double *gx, const double *gy, const double *gz, double *ux, double *uy,
                          double *uz, double *dG, double *dA, int space) {
    CVXB_TRY(deriv_checks(b, "batch_adjoint_cp", b && b->calls_back(), CP_ONLY));
    AdjGrads d;
    d.dG = dG; d.dA = dA;
    return batch_adjoint(b, gx, gy, gz, ux, uy, uz, d, space);
}

int cvxb_batch_adjoint_cone(cvxb_batch *b, const double *gx, const double *gy, const double *gz, double *ux,
                            double *uy, double *uz, double *dP, double *dG, double *dA, int space) {
    CVXB_TRY(deriv_checks(b, "batch_adjoint_cone", qp_or_lp(b), CONE_ONLY, lp_with_dP(b, dP),
                          "a cone LP has no P: dP must be NULL"));
    return batch_adjoint(b, gx, gy, gz, ux, uy, uz, AdjGrads{dP, nullptr, nullptr, dG, dA}, space);
}

int cvxb_batch_tangent(cvxb_batch *b, const double *dP, const double *dq, const double *dG, const double *dh,
                       const double *dA, const double *db, double *dx, double *dy, double *dz, int space) {
    CVXB_TRY(deriv_checks(b, "batch_tangent", qp_or_lp(b), CONE_ONLY, lp_with_dP(b, dP),
                          "a cone LP has no P: dP must be NULL"));
    TanIn d{};
    d.dP = dP; d.dq = dq; d.dG = dG; d.dh = dh; d.dA = dA; d.db = db;
    return batch_tangent(b, d, dx, dy, dz, space);
}

int cvxb_batch_tangent_qcqp(cvxb_batch *b, const double *dP, const double *dq, const double *dr, const double *dG,
                            const double *dh, const double *dA, const double *db, double *dx, double *dy, double *dz,
                            int space) {
    CVXB_TRY(deriv_checks(b, "batch_tangent_qcqp", b && b->kind == Kind::QC, QC_ONLY));
    TanIn d{};
    d.dP = dP; d.dq = dq; d.dr = dr; d.dG = dG; d.dh = dh; d.dA = dA; d.db = db;
    return batch_tangent(b, d, dx, dy, dz, space);
}

int cvxb_batch_tangent_gp(cvxb_batch *b, const double *dF, const double *dg, const double *dG, const double *dh,
                          const double *dA, const double *db, double *dx, double *dy, double *dz, int space) {
    CVXB_TRY(deriv_checks(b, "batch_tangent_gp", b && b->kind == Kind::GP, GP_ONLY));
    TanIn d{};
    d.dF = dF; d.dg = dg; d.dG = dG; d.dh = dh; d.dA = dA; d.db = db;
    return batch_tangent(b, d, dx, dy, dz, space);
}

int cvxb_batch_tangent_cp(cvxb_batch *b, const double *dc, const double *tx, const double *tf, const double *dG,
                          const double *dh, const double *dA, const double *db, double *dx, double *dy, double *dz,
                          int space) {
    CVXB_TRY(deriv_checks(b, "batch_tangent_cp", b && b->calls_back(), CP_ONLY, b && b->kind == Kind::CP && dc,
                          "a CP batch has no c (its objective is f_0): dc must be NULL"));
    TanIn d{};
    d.dq = dc; d.tx = tx; d.tf = tf; d.dG = dG; d.dh = dh; d.dA = dA; d.db = db;
    return batch_tangent(b, d, dx, dy, dz, space);
}

int cvxb_batch_results_y(cvxb_batch *b, double *y, int space) {
    if (!b || !y) { set_error("batch_results_y: NULL argument"); return CVXB_E_ARG; }
    if (b->neq == 0) return 0;
    CVXB_CUDA(cudaSetDevice(b->device));
    if (b->permuted)
        CVXB_CUDA(cudaMemcpy(b->d_perm.p, b->perm.data(), (size_t)b->B * sizeof(int), cudaMemcpyHostToDevice));
    return give_rows(b, y, b->p.y, b->neq, space);
}

int cvxb_batch_results(cvxb_batch *b, double *x, double *s, double *z, int *status, int *iters,
                       double *pobj, double *dobj, int space) {
    if (!b) { set_error("batch is NULL"); return CVXB_E_ARG; }
    CVXB_CUDA(cudaSetDevice(b->device));
    const size_t B = b->B;
    // slot -> problem (identity unless the solve compacted finished problems away)
    if (b->permuted) CVXB_CUDA(cudaMemcpy(b->d_perm.p, b->perm.data(), B * sizeof(int), cudaMemcpyHostToDevice));
    if (x) CVXB_TRY(give_rows(b, x, b->p.x, b->n, space));
    if (s && b->m) CVXB_TRY(give_rows(b, s, b->p.s, b->m, space));
    if (z && b->m) CVXB_TRY(give_rows(b, z, b->p.z, b->m, space));
    if (status || iters || pobj || dobj) {
        if (space == CVXB_DEVICE) { set_error("batch_results: scalars are returned to host memory only"); return CVXB_E_ARG; }
        std::vector<Scal> sc(B);
        CVXB_CUDA(cudaMemcpy(sc.data(), b->sc.p, B * sizeof(Scal), cudaMemcpyDeviceToHost));
        for (size_t slot = 0; slot < B; ++slot) {
            const size_t i = (size_t)b->perm[slot];
            if (status) status[i] = sc[slot].status;
            if (iters) iters[i] = sc[slot].iters;
            if (pobj) pobj[i] = sc[slot].pcost;
            if (dobj) dobj[i] = sc[slot].dcost;
        }
    }
    return 0;
}

// ---------------------------------------------------------------- the 's' block kernels on caller data
// A Ptrs with only what the kernels read: the block layout of cvxb_batch_create_sdp without 'l' and 'q' rows (mlq = 0),
// one Scal per problem (done, step), zero info and the caller's spart.  The launches are the solver's.
int cvxb_sblock_batched(int kernel, int mode, int batch, const cvxb_sblock_args *a, int device) {
    if (batch < 1 || batch > CVXB_BATCH_MAX) {
        set_error("sblock_batched: batch = %d outside 1..%d", batch, CVXB_BATCH_MAX);
        return CVXB_E_ARG;
    }
    if (!a || a->nblk < 1 || !a->orders || !a->spart) {
        set_error("sblock_batched: missing arguments, block orders or spart");
        return CVXB_E_ARG;
    }
    std::vector<int> info;
    long long so = 0, sp = 0, sgo = 0;
    for (int k = 0; k < a->nblk; ++k) {
        const int s = a->orders[k];
        if (s < 1 || s > CVXB_BATCH_SMAX) {
            set_error("sblock_batched: order %d of block %d outside 1..%d", s, k, CVXB_BATCH_SMAX);
            return CVXB_E_ARG;
        }
        info.insert(info.end(), {s, (int)so, (int)sp, (int)so, (int)sgo});
        so += (long long)s * s; sp += (long long)s * (s + 1) / 2; sgo += s;
    }
    if (a->m < so || a->L < so) {
        set_error("sblock_batched: m = %lld or L = %lld below the %lld rows of the blocks", a->m, a->L, so);
        return CVXB_E_ARG;
    }
    if (a->m > INT_MAX) {
        set_error("sblock_batched: m = %lld above %d (the solver keeps m in an int)", a->m, INT_MAX);
        return CVXB_E_ARG;
    }
    const bool lp = kernel == CVXB_SK_RES && mode == 1;
    const long long nlps = sizeof(LPScal) / sizeof(double);
    if (lp && a->L < nlps) {
        set_error("sblock_batched: L = %lld below the %lld doubles of the embedding's scalars", a->L, nlps);
        return CVXB_E_ARG;
    }
    int maxmode = 0;
    std::vector<const void *> need;
    switch (kernel) {
    case CVXB_SK_NT_COMPUTE: need = {a->s, a->z, a->r, a->rti, a->lmbda}; break;
    case CVXB_SK_UPDATE:
        maxmode = 1;
        need = {a->lmbda, a->sigs, a->sigz, a->ds, a->dz, a->r, a->rti, a->d, a->di, a->lmbdasq};
        break;
    case CVXB_SK_DIR_POST:
        maxmode = 1;
        need = {a->ds, a->dz, a->lmbda, mode == 0 ? a->ws3 : a->sigs, mode == 0 ? a->ws3 : a->sigz};
        break;
    case CVXB_SK_EIG_START: need = {a->s, a->bzp}; break;
    case CVXB_SK_EIG_WARM: need = {a->s, a->z}; break;
    case CVXB_SK_BUILD_GS:
        need = {a->rti, a->G, a->Gs};
        if (a->n < 1 || a->ldg < so || a->sG < a->ldg * a->n) {
            set_error("sblock_batched: build_gs needs n >= 1, ldg >= %lld, sG >= ldg * n", so);
            return CVXB_E_ARG;
        }
        break;
    case CVXB_SK_WTZ:
        maxmode = 2;
        need = {a->z, a->rti, a->bzp};
        if (mode == 1) need.push_back(a->th);
        if (mode == 2) need.insert(need.end(), {a->s, a->lmbda, a->r});
        break;
    case CVXB_SK_RES:
        maxmode = 1;
        need = {a->dz, a->ds, a->rti, a->r, a->wz, a->ws, a->lmbda, a->wz3, a->wz2, a->ws2};
        if (lp) need.push_back(a->h);
        break;
    default: set_error("sblock_batched: unknown kernel %d", kernel); return CVXB_E_ARG;
    }
    if (mode < 0 || mode > maxmode) {
        set_error("sblock_batched: mode %d outside 0..%d for kernel %d", mode, maxmode, kernel);
        return CVXB_E_ARG;
    }
    for (const void *q : need)
        if (!q) { set_error("sblock_batched: kernel %d mode %d is missing an operand", kernel, mode); return CVXB_E_ARG; }

    CallCtx ctx; CVXB_TRY(ctx.acquire(device));
    cudaStream_t st = ctx.st;
    const int ns = a->nblk;
    std::vector<Scal> sc(batch);                  // value-initialised: all zero
    for (int b = 0; b < batch; ++b) { sc[b].done = a->done ? a->done[b] : 0; sc[b].step = a->step; }
    std::vector<int> hinfo(batch, 0);
    if (a->info) std::copy(a->info, a->info + batch, hinfo.begin());
    Scratch<int> d_sinfo, d_info;
    Scratch<Scal> d_sc;
    Scratch<double> d_spart, d_lps;
    CVXB_TRY(d_sinfo.alloc(info.size()));
    CVXB_TRY(d_info.alloc(batch));
    CVXB_TRY(d_sc.alloc(batch));
    CVXB_TRY(d_spart.alloc((size_t)batch * ns * 4));
    CVXB_CUDA(cudaMemcpyAsync(d_sinfo.p, info.data(), info.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    CVXB_CUDA(cudaMemcpyAsync(d_info.p, hinfo.data(), batch * sizeof(int), cudaMemcpyHostToDevice, st));
    CVXB_CUDA(cudaMemcpyAsync(d_sc.p, sc.data(), batch * sizeof(Scal), cudaMemcpyHostToDevice, st));
    CVXB_CUDA(cudaMemcpyAsync(d_spart.p, a->spart, (size_t)batch * ns * 4 * sizeof(double), cudaMemcpyHostToDevice,
                              st));
    std::vector<double> lps;
    if (lp) {                                     // dtau / dg = ut for every problem
        lps.assign((size_t)batch * a->L, 0.0);
        for (int b = 0; b < batch; ++b) {
            LPScal *T = reinterpret_cast<LPScal *>(lps.data() + (size_t)b * a->L);
            T->dtau = a->ut; T->dg = 1.0;
        }
        CVXB_TRY(d_lps.alloc(lps.size()));
        CVXB_CUDA(cudaMemcpyAsync(d_lps.p, lps.data(), lps.size() * sizeof(double), cudaMemcpyHostToDevice, st));
    }
    Ptrs p{};
    p.n = a->n; p.m = (int)a->m; p.L = a->L; p.mlq = 0; p.mpk = (int)sp; p.mdg = (int)sgo; p.ns = ns;
    p.sinfo = d_sinfo.p; p.sc = d_sc.p; p.spart = d_spart.p; p.lps = d_lps.p;
    p.s = a->s; p.z = a->z; p.ds = a->ds; p.dz = a->dz; p.h = a->h; p.lmbda = a->lmbda; p.lmbdasq = a->lmbdasq;
    p.d = a->d; p.di = a->di; p.bzp = a->bzp; p.th = a->th; p.ws3 = a->ws3;
    p.sr = a->r; p.srti = a->rti; p.sigs = a->sigs; p.sigz = a->sigz;
    p.wz = a->wz; p.ws = a->ws; p.wz2 = a->wz2; p.ws2 = a->ws2; p.wz3 = a->wz3;
    const dim3 sg(ns, batch);
    switch (kernel) {
    case CVXB_SK_NT_COMPUTE: k_s_nt_compute<<<sg, SB_T, 0, st>>>(p); break;
    case CVXB_SK_UPDATE: k_s_update<false><<<sg, SB_T, 0, st>>>(p, d_info.p, mode); break;
    case CVXB_SK_DIR_POST: k_s_dir_post<<<sg, SB_T, 0, st>>>(p, mode); break;
    case CVXB_SK_EIG_START: k_s_eig_start<<<sg, SB_T, 0, st>>>(p); break;
    case CVXB_SK_EIG_WARM: k_s_eig_warm<<<sg, SB_T, 0, st>>>(p); break;
    case CVXB_SK_BUILD_GS:
        k_s_build_gs<<<dim3(ns, batch, (a->n + 15) / 16), SB_T, 0, st>>>(p, a->G, a->Gs, a->ldg, a->sG);
        break;
    case CVXB_SK_WTZ: k_s_wtz<<<sg, SB_T, 0, st>>>(p, a->z, a->m, a->s, a->m, mode); break;
    default:
        if (lp) k_s_res<true><<<sg, SB_T, 0, st>>>(p);
        else k_s_res<false><<<sg, SB_T, 0, st>>>(p);
    }
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess)
        e = cudaMemcpyAsync(a->spart, d_spart.p, (size_t)batch * ns * 4 * sizeof(double), cudaMemcpyDeviceToHost, st);
    const cudaError_t e2 = cudaStreamSynchronize(st);        // before the scratch goes back to the cache
    if (e == cudaSuccess) e = e2;
    if (e != cudaSuccess) { set_error("sblock_batched: %s", cudaGetErrorString(e)); return CVXB_E_CUDA; }
    return 0;
}

int cvxb_batch_syrk_path(cvxb_batch *b) { return b ? b->syrk_path : CVXB_E_ARG; }

int cvxb_batch_stats(cvxb_batch *b, double *solve_ms, int *iterations) {
    if (!b) return CVXB_E_ARG;
    if (solve_ms) *solve_ms = b->solve_ms;
    if (iterations) *iterations = b->iters_run;
    return 0;
}

}  // extern "C"
