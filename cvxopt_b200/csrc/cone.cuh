// Cone layout + Nesterov-Todd scaling kernels (device side of misc_solvers.scale/pack/...).
#pragma once
#include "common.cuh"
#include <vector>

namespace cvxb {

// Host + device description of a cone product  [mnl | l | q.. | s..]; owns its device arrays
struct ConeLayout {
    int mnl = 0, ml = 0, nq = 0, ns = 0;
    std::vector<int> q, s;
    int sumq = 0, sums = 0, sums2 = 0, sump = 0, maxs = 0;   // sums: sum of the 's' orders
    int cdim = 0, cdim_pckd = 0;
    // per-cone offsets (host)
    std::vector<int> q_off;    // row offset of q cone k in an (unpacked or packed) cone vector
    std::vector<int> v_off;    // offset in the concatenated v
    std::vector<int> s_off;    // unpacked row offset of s cone k
    std::vector<int> s_poff;   // packed row offset of s cone k
    std::vector<int> r_off;    // offset in the concatenated r / rti
    // device copies: [q sizes | q_off | v_off] and [s sizes | s_off | s_poff | r_off]
    int *d_q = nullptr, *d_qoff = nullptr, *d_voff = nullptr;
    int *d_s = nullptr, *d_soff = nullptr, *d_spoff = nullptr, *d_roff = nullptr;
    ConeLayout() = default;
    ConeLayout(const ConeLayout &) = delete;
    ConeLayout &operator=(const ConeLayout &) = delete;
    ~ConeLayout();
    int init(const cvxb_dims *dims);   // call once; what a failed init allocated is freed by the destructor
};

// Device-resident copy of the scaling W (flat mirror of the reference dict)
struct DevScaling {
    double *dnl = nullptr, *dnli = nullptr, *d = nullptr, *di = nullptr, *v = nullptr,
           *beta = nullptr, *r = nullptr, *rti = nullptr;
    double *di2 = nullptr;      // di .* di  (weight of the fused SYRK)
    double *store = nullptr;    // single allocation backing all of the above
    size_t total = 0;
    DevScaling() = default;
    DevScaling(const DevScaling &) = delete;
    DevScaling &operator=(const DevScaling &) = delete;
    ~DevScaling() { tmp_free(store); }
    int alloc(const ConeLayout &c);
    int upload(const ConeLayout &c, const cvxb_scaling *W, int space, cudaStream_t st);
    cvxb_scaling view() const;
};

// ---- vector / matrix scaling pieces (device pointers) ---------------------------
// rows [row0, row0+m) of the xr x xc matrix x (ld ldx): x[i,:] *= w[i]; out of place allowed
int scale_rows(const double *src, long long lds, double *dst, long long ldd, int m, int xc,
               const double *w, cudaStream_t st);
// all 'q' cones at once.  src/dst point at the FIRST q row of their matrices.
int scale_q(const ConeLayout &c, const DevScaling &W, const double *src, long long lds,
            double *dst, long long ldd, int xc, bool inverse, cudaStream_t st);
// 's' cones: dst_k = A' X A (form 1) or A X A' (form 2), A = r or rti, column by column.
// src points at the first 's' row (unpacked layout, ld lds); dst likewise (unpacked).
// work: >= 2 * maxs^2 * min(xc, chunk) doubles (see scale_s_chunk()).
int scale_s(const ConeLayout &c, const DevScaling &W, const double *src, long long lds,
            double *dst, long long ldd, int xc, int trans, int inverse, double *work,
            size_t work_doubles, cudaStream_t st);
// pack 's' blocks of xc columns: unpacked (src) -> packed lower with sqrt(2) off-diagonals.
// vector_mode reproduces misc_solvers.pack's rounding ((x/sqrt2)*sqrt2 on diagonals),
// otherwise pack2's (diagonal copied).  src/dst point at the first 's' row.
int pack_s(const ConeLayout &c, const double *src, long long lds, double *dst, long long ldd,
           int xc, bool vector_mode, cudaStream_t st);
int unpack_s(const ConeLayout &c, const double *src, long long lds, double *dst, long long ldd,
             int xc, cudaStream_t st);

// ---- GEMV (HBM-bound) -------------------------------------------------------------
// optional batching: problem b uses A + b*sA, w + b*sw, x + b*sx, y + b*sy
struct GemvBatch {
    int batch = 1;
    long long sA = 0, sw = 0, sx = 0, sy = 0;
};
// y[c] = alpha * sum_k A[k + c*lda] * (w ? w[k] : 1) * x[k] + beta * y[c],  c < ncols, k < nrows
int gemv_t(int nrows, int ncols, const double *A, long long lda, const double *w, const double *x,
           double alpha, double beta, double *y, cudaStream_t st,
           const GemvBatch &bs = GemvBatch());
// y[k] = alpha * (w ? w[k] : 1) * sum_c A[k + c*lda] x[c] + beta * y[k]
// ws: >= batch * nrows * gemv_n_chunks(ncols) doubles
int gemv_n_chunks(int ncols);
int gemv_n(int nrows, int ncols, const double *A, long long lda, const double *w, const double *x,
           double alpha, double beta, double *y, double *ws, cudaStream_t st,
           const GemvBatch &bs = GemvBatch());
// small elementwise helpers
int vec_mul(int n, const double *a, const double *b, double *out, cudaStream_t st);  // out = a.*b
int vec_axpby(int n, double alpha, const double *x, double beta, double *y, cudaStream_t st);
int symmetrize_lower(int n, double *A, long long lda, int batch, long long stride, cudaStream_t st);
// dst (cols x rows) = src' for src rows x cols; batched: problem p uses src + p*ssrc, dst + p*sdst
int transpose_copy(const double *src, long long lds, double *dst, long long ldd, int rows, int cols,
                   cudaStream_t st, int batch = 1, long long ssrc = 0, long long sdst = 0);

#ifdef __CUDACC__
// ---- 'q' cone algebra, one cone at a time ------------------------------------------------
// The single-problem kernels and the batch IPM share these.  Each function runs on the team of threads that owns one
// cone: a warp (the batch kernels, scale_q) or the whole CTA (the misc_solvers mirror and the NT scaling kernels).
// A pass gives thread `rank` the entries rank, rank + size, ..., or 1 + rank, 1 + rank + size, ... when entry 0 is
// handled apart, and rank 0 writes entry 0.  Entry-0 values every thread needs are read after the team's sums, and a
// function syncs before it overwrites what other threads read.  The two orders give an entry to different threads,
// so a caller syncs between two calls when the second reads what the first wrote.
struct WarpTeam {
    int rank;                                   // lane
    static constexpr int size = 32;
    __device__ __forceinline__ double sum(double v) const { return warp_sum(v); }
    __device__ __forceinline__ void sync() const { __syncwarp(); }
};
struct CtaTeam {
    int rank, size;                             // threadIdx.x, blockDim.x
    double *sh;                                 // block_sum's 32 doubles of shared memory
    __device__ __forceinline__ double sum(double v) const { return block_sum(v, sh); }
    __device__ __forceinline__ void sync() const { __syncthreads(); }
};
// Not unrolled: a cone seldom gives a thread more than one entry, and unrolled passes cost the batch kernels registers.
#define TEAM_FOR(i, t, i0, m) _Pragma("unroll 1") for (int i = (i0) + (t).rank; i < (m); i += (t).size)

// y := W x (inverse = false) or W^{-1} x, W = beta (2 v v' - J) (misc_solvers.c:144-183).  y may be x.
template <class Team>
__device__ __forceinline__ void q_scale(const Team &t, const double *v, double beta, const double *x, double *y, int m,
                                        bool inverse) {
    // w = v' x, with x0 negated first when applying the inverse (:166-170)
    double w = 0.0;
    TEAM_FOR(i, t, 0, m) {
        double xi = x[i];
        if (inverse && i == 0) xi = -xi;
        w += v[i] * xi;
    }
    const double tw = 2.0 * t.sum(w);
    const double b = inverse ? 1.0 / beta : beta;
    TEAM_FOR(i, t, 0, m) {
        double xi = x[i];
        // forward: x0 := -x0 before the rank-one update (:171); inverse: x0 was flipped twice
        if (!inverse && i == 0) xi = -xi;
        double yi = xi + v[i] * tw;           // dger (:172)
        if (inverse && i == 0) yi = -yi;      // (:174-175)
        y[i] = yi * b;                        // (:180-181)
    }
}

// x := H(lmbda^{1/2}) x (inverse = false) or H(lmbda^{-1/2}) x (misc_solvers.c:315-342)
template <class Team>
__device__ __forceinline__ void q_scale2(const Team &t, const double *l, double *x, int m, bool inverse) {
    double n2 = 0, dot = 0;
    TEAM_FOR(i, t, 1, m) { n2 += l[i] * l[i]; dot += l[i] * x[i]; }
    n2 = t.sum(n2); dot = t.sum(dot);
    const double nrm = sqrt(n2), l0 = l[0], x0 = x[0];
    const double a = sqrt(l0 + nrm) * sqrt(l0 - nrm);
    const double lx = inverse ? (l0 * x0 + dot) / a : (l0 * x0 - dot) / a;
    double b = (x0 + lx) / (l0 / a + 1.0) / a;
    if (!inverse) b = -b;
    const double sc = inverse ? a : 1.0 / a;
    t.sync();
    TEAM_FOR(i, t, 1, m) x[i] = (x[i] + b * l[i]) * sc;
    if (t.rank == 0) x[0] = lx * sc;
}

// out := y o x (misc_solvers.c:634-767); out may be x.  Returns y'x, the product's entry 0; with out == nullptr
// that is all it computes.
template <class Team>
__device__ __forceinline__ double q_sprod(const Team &t, const double *y, const double *x, double *out, int m) {
    double d = 0;
    TEAM_FOR(i, t, 0, m) d += y[i] * x[i];
    d = t.sum(d);
    if (!out) return d;
    const double y0 = y[0], x0 = x[0];
    t.sync();
    TEAM_FOR(i, t, 1, m) out[i] = y0 * x[i] + x0 * y[i];
    if (t.rank == 0) out[0] = d;
    return d;
}

// x := lmbda o\ x (misc_solvers.c:813-836)
template <class Team>
__device__ __forceinline__ void q_sinv(const Team &t, const double *l, double *x, int m) {
    double n2 = 0, d = 0;
    TEAM_FOR(i, t, 1, m) { n2 += l[i] * l[i]; d += x[i] * l[i]; }
    n2 = t.sum(n2); d = t.sum(d);
    const double nrm = sqrt(n2), l0 = l[0], x0 = x[0];
    const double a = (l0 + nrm) * (l0 - nrm);
    const double al1 = a / l0, al2 = d / l0 - x0, ia = 1.0 / a;
    t.sync();
    TEAM_FOR(i, t, 1, m) x[i] = (x[i] * al1 + al2 * l[i]) * ia;
    if (t.rank == 0) x[0] = (x0 * l0 - d) * ia;
}

// sqrt(x' J x) the way misc.jnrm2 evaluates it (misc.py:848-856): a = |x[1:]|, sqrt(x0 - a) * sqrt(x0 + a)
template <class Team>
__device__ __forceinline__ double q_jnrm2(const Team &t, const double *x, int m) {
    double n2 = 0.0;
    TEAM_FOR(i, t, 1, m) n2 += x[i] * x[i];
    const double a = sqrt(t.sum(n2));
    return sqrt(x[0] - a) * sqrt(x[0] + a);
}

// the cone's term of max_step, |x[1:]| - x0 (misc_solvers.c:1073-1085)
template <class Team>
__device__ __forceinline__ double q_max_step(const Team &t, const double *x, int m) {
    double n2 = 0;
    TEAM_FOR(i, t, 1, m) n2 += x[i] * x[i];
    return sqrt(t.sum(n2)) - x[0];
}

// NT scaling of the cone from s and z (misc.py:311-354): v, lmbda, and *beta = sqrt(a / b)
template <class Team>
__device__ __forceinline__ void q_nt_compute(const Team &t, const double *s, const double *z, double *v, double *lm,
                                             double *beta, int m) {
    const double aa = q_jnrm2(t, s, m), bb = q_jnrm2(t, z, m);
    double sz = 0.0;
    TEAM_FOR(i, t, 0, m) sz += s[i] * z[i];
    const double dot = t.sum(sz);
    const double cc = sqrt((dot / aa / bb + 1.0) / 2.0);
    // vk = 1/(2c) ( s/a + J z/b ),  then  v = (vk + e) / sqrt(2 (vk0 + 1))
    const double v0 = ((s[0] / aa) + (z[0] / bb)) / 2.0 / cc + 1.0;
    const double sc = 1.0 / sqrt(2.0 * v0);
    const double dd = 2.0 * cc + s[0] / aa + z[0] / bb;
    const double c1 = (cc + z[0] / bb) / dd / aa, c2 = (cc + s[0] / aa) / dd / bb, sab = sqrt(aa * bb);
    TEAM_FOR(i, t, 0, m) {
        if (i == 0) {
            v[0] = v0 * sc;
            lm[0] = cc * sab;
        } else {
            v[i] = ((s[i] / aa - z[i] / bb) / 2.0 / cc) * sc;
            lm[i] = (c1 * s[i] + c2 * z[i]) * sab;
        }
    }
    if (t.rank == 0) *beta = sqrt(aa / bb);
}

// NT scaling update of the cone (misc.py:504-573): s, z hold the new iterates in the current scaling and are
// normalised in place; v and lmbda are overwritten, *beta *= sqrt(a / b)
template <class Team>
__device__ __forceinline__ void q_nt_update(const Team &t, double *s, double *z, double *v, double *lm, double *beta,
                                            int m) {
    const double aa = q_jnrm2(t, s, m), bb = q_jnrm2(t, z, m);
    t.sync();                                   // every thread has read s[0] and z[0]
    double t1 = 0.0, t2 = 0.0, t3 = 0.0;
    TEAM_FOR(i, t, 0, m) {
        const double si = s[i] * (1.0 / aa), zi = z[i] * (1.0 / bb);
        s[i] = si; z[i] = zi;
        t1 += si * zi;
        t2 += v[i] * si;
        t3 += (i == 0 ? v[i] * zi : -v[i] * zi);     // jdot: v' J z
    }
    const double dot = t.sum(t1), vs = t.sum(t2), vz = t.sum(t3);
    t.sync();                                   // s[0] and z[0] are written
    const double cc = sqrt((1.0 + dot) / 2.0);
    const double vq = (vs + vz) / 2.0 / cc, vu = vs - vz;
    const double s0 = s[0], z0 = z[0], vk0 = v[0];
    const double wk0 = 2.0 * vk0 * vq - (s0 + z0) / 2.0 / cc;
    const double dd = (vk0 * vu - s0 / 2.0 + z0 / 2.0) / (wk0 + 1.0);
    const double sab = sqrt(aa * bb);
    // new v before its square root:  v := 2 (v'q) v - (J st/a + zt/b) / (2c)
    const double vn0 = 2.0 * vq * vk0 - s0 / 2.0 / cc - 0.5 / cc * z0 + 1.0;
    const double sc = 1.0 / sqrt(2.0 * vn0);
    t.sync();
    TEAM_FOR(i, t, 0, m) {
        const double vi = v[i], si = s[i], zi = z[i];
        if (i == 0) {
            lm[0] = cc * sab;
            v[0] = vn0 * sc;
        } else {
            lm[i] = (vi * (2.0 * (-dd * vq + 0.5 * vu)) + 0.5 * (1.0 - dd / cc) * si + 0.5 * (1.0 + dd / cc) * zi) * sab;
            v[i] = (2.0 * vq * vi + 0.5 / cc * si - 0.5 / cc * zi) * sc;
        }
    }
    if (t.rank == 0) *beta *= sqrt(aa / bb);
}

// ---- in-CTA Jacobi solvers for small blocks ---------------------------------------------------------------
// The single-problem kernels (cone_vec.cu jac_small_kernel, nt_scaling.cu jacobi_small_kernel) and the batch
// IPM's 's'-block kernels call the same bodies.
// Round-robin pairing of m2 (even) players: round r, slot t -> columns (p, q); an index >= m is a bye.
__device__ __forceinline__ void svd_pair(int m2, int r, int t, int &p, int &q) {
    const int n1 = m2 - 1;
    if (t == 0) { p = n1; q = r % n1; }
    else { p = (r + t) % n1; q = (r - t + n1) % n1; }
    if (p > q) { const int w = p; p = q; q = w; }
}
// Round r of the round-robin ("chess tournament") ordering on N (even) indices: N/2 disjoint pairs.
__device__ __forceinline__ void rr_pair(int N, int r, int k, int &p, int &q) {
    int a, b;
    if (k == 0) { a = N - 1; b = r; }
    else { a = (r + k) % (N - 1); b = (r - k + (N - 1)) % (N - 1); }
    p = min(a, b); q = max(a, b);
}

// rotation J = [c s; -s c] annihilating a_pq in J'[app apq; apq aqq]J;  t = tan of the angle
__device__ __forceinline__ void jac_rot(double app, double aqq, double apq, double &c, double &s, double &t) {
    if (apq == 0.0) { c = 1.0; s = 0.0; t = 0.0; return; }
    const double tau = (aqq - app) / (2.0 * apq);
    t = copysign(1.0, tau) / (fabs(tau) + sqrt(1.0 + tau * tau));     // tau*tau = inf -> t = 0
    c = 1.0 / sqrt(1.0 + t * t);
    s = t * c;
}

// One thread's share of a round: the 2x2 block (rows of pair I, columns of pair J) of
// dst = J'.src.J, and the same block of V := V.J.  Indices >= mk belong to the padding.
template <bool WITH_V>
__device__ __forceinline__ void jac_block(const double *src, double *dst, double *V, int mk, int N,
                                          int r, int I, int J) {
    int pi, qi, pj, qj;
    rr_pair(N, r, I, pi, qi);
    rr_pair(N, r, J, pj, qj);
    if (pi >= mk || pj >= mk) return;
    const bool vi = qi < mk, vj = qj < mk;
    double ci = 1, si = 0, ti = 0, cj = 1, sj = 0, tj = 0;
    if (vi) jac_rot(src[pi + (size_t)pi * mk], src[qi + (size_t)qi * mk], src[qi + (size_t)pi * mk], ci, si, ti);
    if (I == J) { cj = ci; sj = si; tj = ti; }
    else if (vj) jac_rot(src[pj + (size_t)pj * mk], src[qj + (size_t)qj * mk], src[qj + (size_t)pj * mk], cj, sj, tj);
    const double b00 = src[pi + (size_t)pj * mk];
    const double b01 = vj ? src[pi + (size_t)qj * mk] : 0.0;
    const double b10 = vi ? src[qi + (size_t)pj * mk] : 0.0;
    const double b11 = (vi && vj) ? src[qi + (size_t)qj * mk] : 0.0;
    double d00, d01, d10, d11;
    if (I == J) {
        d00 = b00 - ti * b10; d11 = b11 + ti * b10; d01 = 0.0; d10 = 0.0;
    } else {
        const double r00 = ci * b00 - si * b10, r01 = ci * b01 - si * b11;
        const double r10 = si * b00 + ci * b10, r11 = si * b01 + ci * b11;
        d00 = cj * r00 - sj * r01; d01 = sj * r00 + cj * r01;
        d10 = cj * r10 - sj * r11; d11 = sj * r10 + cj * r11;
    }
    dst[pi + (size_t)pj * mk] = d00;
    if (vj) dst[pi + (size_t)qj * mk] = d01;
    if (vi) dst[qi + (size_t)pj * mk] = d10;
    if (vi && vj) dst[qi + (size_t)qj * mk] = d11;
    if (WITH_V) {
        const double v00 = V[pi + (size_t)pj * mk];
        const double v01 = vj ? V[pi + (size_t)qj * mk] : 0.0;
        V[pi + (size_t)pj * mk] = cj * v00 - sj * v01;
        if (vj) V[pi + (size_t)qj * mk] = sj * v00 + cj * v01;
        if (vi) {
            const double v10 = V[qi + (size_t)pj * mk];
            const double v11 = vj ? V[qi + (size_t)qj * mk] : 0.0;
            V[qi + (size_t)pj * mk] = cj * v10 - sj * v11;
            if (vj) V[qi + (size_t)qj * mk] = sj * v10 + cj * v11;
        }
    }
}
// convergence of one block from its (off^2, total^2): at rounding level, or stagnating just above it
__host__ __device__ inline bool jac_done(double off2, double tot2, double prev_off2, int mk) {
    const double eps = 2.220446049250313e-16;
    if (!(off2 > eps * eps * (double)mk * tot2)) return off2 == off2;       // NaN never converges
    return off2 <= 1e-26 * tot2 && off2 >= 0.25 * prev_off2;
}

// Two-sided Jacobi sweeps on the symmetric mk x mk block in w0 (both triangles), ping-ponging with w1; V := V J when
// WITH_V; tid, nt: threadIdx.x, blockDim.x.  Needs blockDim.x >= (N/2)^2 with N = mk rounded up to even.  On return w0 points at the rotated block
// (eigenvalues on its diagonal, eigenvectors in the columns of V); false when max_sweeps ran out (jac_done).
template <bool WITH_V>
__device__ __forceinline__ bool jac_eig_cta(double *&w0, double *&w1, double *V, int mk, int max_sweeps, double *sh,
                                            int tid, int nt) {
    const int N = max(2, mk + (mk & 1)), h = N / 2;
    const int I = tid % h, J = tid / h;          // I fastest: rows of the column-major block
    double prev = 1e300;
    int sweep = 0;
    bool ok = false;
    for (;; ++sweep) {
        double off = 0, tot = 0;
        for (int e = tid; e < mk * mk; e += nt) {
            const double v = w0[e] * w0[e];
            tot += v;
            if (e % mk != e / mk) off += v;
        }
        off = block_sum(off, sh); tot = block_sum(tot, sh);
        if (jac_done(off, tot, prev, mk)) { ok = true; break; }
        if (sweep == max_sweeps) break;
        prev = off;
        for (int r = 0; r < N - 1; ++r) {
            if (J < h) jac_block<WITH_V>(w0, w1, V, mk, N, r, I, J);
            __syncthreads();
            double *t = w0; w0 = w1; w1 = t;
        }
    }
    return ok;
}

// One-sided Jacobi on the columns of the m x m block B (column-major, ld m), V := V J: one warp per column pair,
// until a sweep rotates nothing or maxsweeps have run (true: the former).  B and V are shared memory; the caller
// initialises V; rot is a shared int of the caller's.
__device__ __forceinline__ bool jacobi_svd_cta(int m, double *B, double *V, int maxsweeps, int &rot) {
    const int m2 = (m + 1) & ~1, npairs = m2 / 2;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarp = blockDim.x >> 5;
    for (int sweep = 0; sweep < maxsweeps; ++sweep) {
        if (threadIdx.x == 0) rot = 0;
        __syncthreads();
        for (int r = 0; r < m2 - 1; ++r) {
            for (int t = warp; t < npairs; t += nwarp) {        // one warp per pair
                int p, q;
                svd_pair(m2, r, t, p, q);
                if (q >= m) continue;
                double *bp = B + p * m, *bq = B + q * m;
                double a = 0.0, b = 0.0, g = 0.0;
                for (int i = lane; i < m; i += 32) { const double x = bp[i], y = bq[i]; a += x * x; b += y * y; g += x * y; }
                a = warp_sum(a); b = warp_sum(b); g = warp_sum(g);
                if (!(fabs(g) > (2.0 * 2.220446049250313e-16 * sqrt((double)m)) * sqrt(a * b)) || g == 0.0) continue;
                const double zeta = (b - a) / (2.0 * g);
                const double tt = (zeta >= 0.0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
                const double c = 1.0 / sqrt(1.0 + tt * tt), sn = c * tt;
                double *vp = V + p * m, *vq = V + q * m;
                for (int i = lane; i < m; i += 32) {
                    const double x = bp[i], y = bq[i];
                    bp[i] = c * x - sn * y; bq[i] = sn * x + c * y;
                    const double u = vp[i], w = vq[i];
                    vp[i] = c * u - sn * w; vq[i] = sn * u + c * w;
                }
                if (lane == 0) atomicAdd(&rot, 1);
            }
            __syncthreads();
        }
        const int done = (rot == 0);
        __syncthreads();
        if (done) break;
    }
    return rot == 0;
}
#endif

}  // namespace cvxb
