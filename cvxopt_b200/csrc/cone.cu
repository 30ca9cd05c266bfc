// Nesterov-Todd scaling, packing and the HBM-bound GEMVs of the KKT solve.
//
// Device restatement of the cone algebra that the reference keeps in
// src/C/misc_solvers.c: scale (:85-244), pack (:412-465), pack2 (:476-541),
// unpack (:552-601).  Arithmetic order inside each element follows the reference
// (e.g. the sign flips around the hyperbolic Householder update, the (x/sqrt2)*sqrt2
// rounding of `pack`), reductions use warp trees instead of BLAS loops.
#include "cone.cuh"

namespace cvxb {

// ------------------------------------------------------------------ layout
int ConeLayout::init(const cvxb_dims *dims) {
    if (!dims || dims->mnl < 0 || dims->ml < 0 || dims->nq < 0 || dims->ns < 0) {
        set_error("dims: negative dimension");
        return CVXB_E_ARG;
    }
    mnl = dims->mnl; ml = dims->ml; nq = dims->nq; ns = dims->ns;
    q.assign(dims->q, dims->q + nq);
    s.assign(dims->s, dims->s + ns);
    sumq = sums = sums2 = sump = maxs = 0;
    q_off.resize(nq); v_off.resize(nq); s_off.resize(ns); s_poff.resize(ns); r_off.resize(ns);
    for (int k = 0; k < nq; ++k) {
        if (q[k] < 1) { set_error("dims['q'] entries must be >= 1"); return CVXB_E_ARG; }
        q_off[k] = sumq; v_off[k] = sumq; sumq += q[k];
    }
    for (int k = 0; k < ns; ++k) {
        if (s[k] < 0) { set_error("dims['s'] entries must be >= 0"); return CVXB_E_ARG; }
        s_off[k] = sums2; s_poff[k] = sump; r_off[k] = sums2;
        sums += s[k]; sums2 += s[k] * s[k]; sump += s[k] * (s[k] + 1) / 2;
        if (s[k] > maxs) maxs = s[k];
    }
    cdim = mnl + ml + sumq + sums2;
    cdim_pckd = mnl + ml + sumq + sump;
    auto up = [&](int **dst, const std::vector<int> &h) -> int {
        if (h.empty()) { *dst = nullptr; return 0; }
        CVXB_CUDA(tmp_malloc(dst, h.size() * sizeof(int)));
        CVXB_CUDA(cudaMemcpy(*dst, h.data(), h.size() * sizeof(int), cudaMemcpyHostToDevice));
        return 0;
    };
    CVXB_TRY(up(&d_q, q)); CVXB_TRY(up(&d_qoff, q_off)); CVXB_TRY(up(&d_voff, v_off));
    CVXB_TRY(up(&d_s, s)); CVXB_TRY(up(&d_soff, s_off)); CVXB_TRY(up(&d_spoff, s_poff));
    CVXB_TRY(up(&d_roff, r_off));
    return 0;
}

ConeLayout::~ConeLayout() {
    for (int *p : {d_q, d_qoff, d_voff, d_s, d_soff, d_spoff, d_roff}) tmp_free(p);
}

// ------------------------------------------------------------------ scaling storage
int DevScaling::alloc(const ConeLayout &c) {
    total = (size_t)2 * c.mnl + (size_t)3 * c.ml + c.sumq + c.nq + (size_t)2 * c.sums2 + 8;
    CVXB_CUDA(tmp_malloc(&store, total * sizeof(double)));
    CVXB_CUDA(cudaMemset(store, 0, total * sizeof(double)));
    double *p = store;
    dnl = p; p += c.mnl; dnli = p; p += c.mnl;
    d = p; p += c.ml; di = p; p += c.ml; di2 = p; p += c.ml;
    v = p; p += c.sumq; beta = p; p += c.nq;
    r = p; p += c.sums2; rti = p; p += c.sums2;
    return 0;
}
cvxb_scaling DevScaling::view() const {
    cvxb_scaling w;
    w.dnl = dnl; w.dnli = dnli; w.d = d; w.di = di; w.v = v; w.beta = beta; w.r = r; w.rti = rti;
    return w;
}

namespace {
__global__ void square_kernel(int n, const double *a, double *out) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = a[i] * a[i];
}
}  // namespace

int DevScaling::upload(const ConeLayout &c, const cvxb_scaling *W, int space, cudaStream_t st) {
    if (!W) { set_error("scaling W is NULL"); return CVXB_E_ARG; }
    cudaMemcpyKind kind = (space == CVXB_DEVICE) ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    auto cp = [&](double *dst, const double *src, size_t n, const char *name) -> int {
        if (n == 0) return 0;
        if (!src) { set_error("scaling W: missing item '%s'", name); return CVXB_E_ARG; }
        CVXB_CUDA(cudaMemcpyAsync(dst, src, n * sizeof(double), kind, st));
        return 0;
    };
    CVXB_TRY(cp(dnl, W->dnl, c.mnl, "dnl")); CVXB_TRY(cp(dnli, W->dnli, c.mnl, "dnli"));
    CVXB_TRY(cp(d, W->d, c.ml, "d")); CVXB_TRY(cp(di, W->di, c.ml, "di"));
    CVXB_TRY(cp(v, W->v, c.sumq, "v")); CVXB_TRY(cp(beta, W->beta, c.nq, "beta"));
    CVXB_TRY(cp(r, W->r, c.sums2, "r")); CVXB_TRY(cp(rti, W->rti, c.sums2, "rti"));
    if (c.ml > 0) {
        square_kernel<<<(c.ml + 255) / 256, 256, 0, st>>>(c.ml, di, di2);
        count_launch();
        CVXB_LAUNCH_CHECK();
    }
    return 0;
}

// ------------------------------------------------------------------ kernels
namespace {

__global__ void scale_rows_kernel(const double *src, long long lds, double *dst, long long ldd,
                                  int m, int xc, const double *w) {
    // columns are strided over gridDim.y (capped at 65535 by the launch API; xc may exceed it)
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const double wi = w[i];
    for (long long j = blockIdx.y; j < xc; j += gridDim.y) dst[i + j * ldd] = src[i + j * lds] * wi;
}

// one warp per (cone, column)
__global__ void __launch_bounds__(128)
scale_q_kernel(const double *src, long long lds, double *dst, long long ldd, int xc,
               const int *q, const int *qoff, const int *voff, const double *vall,
               const double *betaall, int inverse) {
    const int k = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long j = (long long)blockIdx.x * 4 + warp;
    if (j >= xc) return;
    q_scale(WarpTeam{lane}, vall + voff[k], betaall[k], src + qoff[k] + j * lds, dst + qoff[k] + j * ldd, q[k],
            inverse);
}

__global__ void pack_s_kernel(const double *src, long long lds, double *dst, long long ldd,
                              const int *s, const int *soff, const int *spoff, int vector_mode, int xc) {
    const int k = blockIdx.z;
    const int ms = s[k];
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= ms * ms) return;
    const int i = e % ms, kk = e / ms;
    if (i < kk) return;
    const double sq2 = sqrt(2.0);
    const long long ip = (long long)kk * ms - (long long)kk * (kk - 1) / 2 + (i - kk);
    for (long long j = blockIdx.y; j < xc; j += gridDim.y) {
        double x = src[soff[k] + e + j * lds];
        double y;
        if (i == kk) y = vector_mode ? (x / sq2) * sq2 : x;   // misc_solvers.c:454,462 vs :531-532
        else y = x * sq2;
        dst[spoff[k] + ip + j * ldd] = y;
    }
}

__global__ void unpack_s_kernel(const double *src, long long lds, double *dst, long long ldd,
                                const int *s, const int *soff, const int *spoff, int xc) {
    const int k = blockIdx.z;
    const int ms = s[k];
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= ms * ms) return;
    const int i = e % ms, kk = e / ms;
    if (i < kk) return;
    const double a = 1.0 / sqrt(2.0);                        // misc_solvers.c:556
    const long long ip = (long long)kk * ms - (long long)kk * (kk - 1) / 2 + (i - kk);
    for (long long j = blockIdx.y; j < xc; j += gridDim.y) {
        double x = src[spoff[k] + ip + j * lds];
        dst[soff[k] + e + j * ldd] = (i == kk) ? x : x * a;
    }
}

// dst (ms x ms full, batch stride ms*ms) = symmetric completion of the lower triangle of
// src (ms x ms, ld ms, batch stride `sstride`).  32x32 tiles through shared memory.
__global__ void sym_copy_kernel(const double *src, long long sstride, double *dst, int ms) {
    __shared__ double t[32][33];
    const int nt = (ms + 31) / 32;
    // enumerate lower tiles
    int tl = blockIdx.x, ti = 0;
    while (tl >= ti + 1) { tl -= ti + 1; ++ti; }
    const int tj = tl;
    if (ti >= nt) return;
    const double *S = src + (long long)blockIdx.y * sstride;
    double *Dm = dst + (long long)blockIdx.y * ms * ms;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;   // 256 threads: 32 x 8
    for (int cc = ty; cc < 32; cc += 8) {
        int i = ti * 32 + tx, kk = tj * 32 + cc;
        double v = 0.0;
        if (i < ms && kk < ms) {
            if (i >= kk) v = S[i + (long long)kk * ms];
            else v = S[kk + (long long)i * ms];     // only on diagonal tiles
        }
        t[cc][tx] = v;
    }
    __syncthreads();
    for (int cc = ty; cc < 32; cc += 8) {
        int i = ti * 32 + tx, kk = tj * 32 + cc;
        if (i < ms && kk < ms) Dm[i + (long long)kk * ms] = t[cc][tx];
        if (ti != tj) {
            int i2 = tj * 32 + tx, k2 = ti * 32 + cc;   // transposed tile
            if (i2 < ms && k2 < ms) Dm[i2 + (long long)k2 * ms] = t[tx][cc];
        }
    }
}

// in-place: copy the strict lower triangle of A (n x n, ld lda) onto the upper one
__global__ void symmetrize_kernel(double *A, long long lda, int n, long long stride) {
    __shared__ double t[32][33];
    int tl = blockIdx.x, ti = 0;
    while (tl >= ti + 1) { tl -= ti + 1; ++ti; }
    const int tj = tl;
    double *M = A + (long long)blockIdx.y * stride;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    for (int cc = ty; cc < 32; cc += 8) {
        int i = ti * 32 + tx, kk = tj * 32 + cc;
        t[cc][tx] = (i < n && kk < n) ? M[i + (long long)kk * lda] : 0.0;
    }
    __syncthreads();
    for (int cc = ty; cc < 32; cc += 8) {
        int i2 = tj * 32 + tx, k2 = ti * 32 + cc;       // (row, col) of the mirrored element
        if (i2 < n && k2 < n && i2 < k2) M[i2 + (long long)k2 * lda] = t[tx][cc];
    }
}

// ---- GEMV-T: one warp per column; 16-byte loads, 8 in flight per lane
template <bool VEC, bool HAS_W>
__global__ void __launch_bounds__(256)
gemv_t_kernel(int nrows, int ncols, const double *__restrict__ A, long long lda,
              const double *__restrict__ w, const double *__restrict__ x, double alpha,
              double beta, double *y, GemvBatch bs) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long c = (long long)blockIdx.x * 8 + warp;
    if (c >= ncols) return;
    const long long pb = blockIdx.y;
    A += pb * bs.sA; x += pb * bs.sx; y += pb * bs.sy;
    if (HAS_W) w += pb * bs.sw;
    const double *a = A + c * lda;
    double s0 = 0, s1 = 0, s2 = 0, s3 = 0;
    int k = 0;
    if (VEC) {
        const double2 *a2 = reinterpret_cast<const double2 *>(a);
        const double2 *x2 = reinterpret_cast<const double2 *>(x);
        const double2 *w2 = reinterpret_cast<const double2 *>(w);
        const int n2 = nrows >> 1;
        int k2 = lane;
        for (; k2 + 96 < n2; k2 += 128) {
            double2 v0 = a2[k2], v1 = a2[k2 + 32], v2 = a2[k2 + 64], v3 = a2[k2 + 96];
            double2 u0 = x2[k2], u1 = x2[k2 + 32], u2 = x2[k2 + 64], u3 = x2[k2 + 96];
            if (HAS_W) {
                double2 q0 = w2[k2], q1 = w2[k2 + 32], q2 = w2[k2 + 64], q3 = w2[k2 + 96];
                u0.x *= q0.x; u0.y *= q0.y; u1.x *= q1.x; u1.y *= q1.y;
                u2.x *= q2.x; u2.y *= q2.y; u3.x *= q3.x; u3.y *= q3.y;
            }
            s0 += v0.x * u0.x; s0 += v0.y * u0.y;
            s1 += v1.x * u1.x; s1 += v1.y * u1.y;
            s2 += v2.x * u2.x; s2 += v2.y * u2.y;
            s3 += v3.x * u3.x; s3 += v3.y * u3.y;
        }
        for (; k2 < n2; k2 += 32) {
            double2 v0 = a2[k2], u0 = x2[k2];
            if (HAS_W) { double2 q0 = w2[k2]; u0.x *= q0.x; u0.y *= q0.y; }
            s0 += v0.x * u0.x; s0 += v0.y * u0.y;
        }
        k = n2 * 2 + lane;            // odd tail row (at most one)
    } else {
        k = lane;
    }
    for (; k < nrows; k += 32) s1 += a[k] * (HAS_W ? w[k] * x[k] : x[k]);
    double s = warp_sum((s0 + s1) + (s2 + s3));
    if (lane == 0) y[c] = (beta == 0.0) ? alpha * s : alpha * s + beta * y[c];
}

constexpr int GN_CH = 128;   // columns per chunk
__global__ void __launch_bounds__(256)
gemv_n_partial_kernel(int nrows, int ncols, const double *__restrict__ A, long long lda,
                      const double *__restrict__ x, double *ws, GemvBatch bs, long long sws) {
    __shared__ double xs[GN_CH];
    A += (long long)blockIdx.z * bs.sA; x += (long long)blockIdx.z * bs.sx;
    ws += (long long)blockIdx.z * sws;
    const int c0 = blockIdx.y * GN_CH;
    const int nc = min(GN_CH, ncols - c0);
    if (threadIdx.x < GN_CH) xs[threadIdx.x] = (threadIdx.x < nc) ? x[c0 + threadIdx.x] : 0.0;
    __syncthreads();
    const long long k = (long long)blockIdx.x * 256 + threadIdx.x;
    if (k >= nrows) return;
    const double *a = A + k + (long long)c0 * lda;
    double s0 = 0, s1 = 0, s2 = 0, s3 = 0;
    int c = 0;
    for (; c + 3 < nc; c += 4) {
        s0 += a[(long long)c * lda] * xs[c];
        s1 += a[(long long)(c + 1) * lda] * xs[c + 1];
        s2 += a[(long long)(c + 2) * lda] * xs[c + 2];
        s3 += a[(long long)(c + 3) * lda] * xs[c + 3];
    }
    for (; c < nc; ++c) s0 += a[(long long)c * lda] * xs[c];
    ws[(long long)blockIdx.y * nrows + k] = (s0 + s1) + (s2 + s3);
}
__global__ void gemv_n_reduce_kernel(int nrows, int nchunks, const double *ws, const double *w,
                                     double alpha, double beta, double *y, GemvBatch bs,
                                     long long sws) {
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nrows) return;
    ws += (long long)blockIdx.y * sws; y += (long long)blockIdx.y * bs.sy;
    if (w) w += (long long)blockIdx.y * bs.sw;
    double s = 0.0;
    for (int ch = 0; ch < nchunks; ++ch) s += ws[(long long)ch * nrows + k];
    if (w) s *= w[k];
    y[k] = (beta == 0.0) ? alpha * s : alpha * s + beta * y[k];
}

// dst (cols x rows, ld ldd) = src' where src is rows x cols (ld lds); 32x32 tiles through smem
__global__ void transpose_kernel(const double *src, long long lds, double *dst, long long ldd,
                                 int rows, int cols, long long ssrc, long long sdst) {
    __shared__ double t[32][33];
    src += blockIdx.z * ssrc; dst += blockIdx.z * sdst;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int r0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    for (int cc = ty; cc < 32; cc += 8) {
        int r = r0 + tx, c = c0 + cc;
        t[cc][tx] = (r < rows && c < cols) ? src[r + (long long)c * lds] : 0.0;
    }
    __syncthreads();
    for (int rr = ty; rr < 32; rr += 8) {
        int c = c0 + tx, r = r0 + rr;           // dst[c, r] = src[r, c]
        if (r < rows && c < cols) dst[c + (long long)r * ldd] = t[tx][rr];
    }
}

__global__ void vec_mul_kernel(int n, const double *a, const double *b, double *out) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = a[i] * b[i];
}
__global__ void vec_axpby_kernel(int n, double alpha, const double *x, double beta, double *y) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) y[i] = (beta == 0.0) ? alpha * x[i] : alpha * x[i] + beta * y[i];
}

}  // namespace

// ------------------------------------------------------------------ host wrappers
int scale_rows(const double *src, long long lds, double *dst, long long ldd, int m, int xc,
               const double *w, cudaStream_t st) {
    if (m <= 0 || xc <= 0) return 0;
    dim3 grid((m + 255) / 256, xc < 65535 ? xc : 65535);
    scale_rows_kernel<<<grid, 256, 0, st>>>(src, lds, dst, ldd, m, xc, w);
    count_launch();
    CVXB_LAUNCH_CHECK();
    return 0;
}

int scale_q(const ConeLayout &c, const DevScaling &W, const double *src, long long lds,
            double *dst, long long ldd, int xc, bool inverse, cudaStream_t st) {
    if (c.nq == 0 || xc <= 0) return 0;
    dim3 grid((xc + 3) / 4, c.nq);
    scale_q_kernel<<<grid, 128, 0, st>>>(src, lds, dst, ldd, xc, c.d_q, c.d_qoff, c.d_voff, W.v,
                                         W.beta, inverse ? 1 : 0);
    count_launch();
    CVXB_LAUNCH_CHECK();
    return 0;
}

int pack_s(const ConeLayout &c, const double *src, long long lds, double *dst, long long ldd,
           int xc, bool vector_mode, cudaStream_t st) {
    if (c.ns == 0 || xc <= 0 || c.maxs == 0) return 0;
    dim3 grid((c.maxs * c.maxs + 255) / 256, xc < 65535 ? xc : 65535, c.ns);
    pack_s_kernel<<<grid, 256, 0, st>>>(src, lds, dst, ldd, c.d_s, c.d_soff, c.d_spoff,
                                        vector_mode ? 1 : 0, xc);
    count_launch();
    CVXB_LAUNCH_CHECK();
    return 0;
}

int unpack_s(const ConeLayout &c, const double *src, long long lds, double *dst, long long ldd,
             int xc, cudaStream_t st) {
    if (c.ns == 0 || xc <= 0 || c.maxs == 0) return 0;
    dim3 grid((c.maxs * c.maxs + 255) / 256, xc < 65535 ? xc : 65535, c.ns);
    unpack_s_kernel<<<grid, 256, 0, st>>>(src, lds, dst, ldd, c.d_s, c.d_soff, c.d_spoff, xc);
    count_launch();
    CVXB_LAUNCH_CHECK();
    return 0;
}

int scale_s(const ConeLayout &c, const DevScaling &W, const double *src, long long lds,
            double *dst, long long ldd, int xc, int trans, int inverse, double *work,
            size_t work_doubles, cudaStream_t st) {
    if (c.ns == 0 || xc <= 0) return 0;
    // form 1: A' X A  for (N,N) with A=r and (T,I) with A=rti;  form 2: A X A' otherwise
    const bool inv = (inverse == 'I');
    const bool form1 = (!inv && trans == 'N') || (inv && trans == 'T');
    for (int k = 0; k < c.ns; ++k) {
        const int ms = c.s[k];
        if (ms == 0) continue;
        const long long m2 = (long long)ms * ms;
        const double *A = (inv ? W.rti : W.r) + c.r_off[k];
        long long chunk = (long long)(work_doubles / (2 * m2));
        if (chunk < 1) { set_error("scale_s: workspace too small"); return CVXB_E_NOMEM; }
        if (chunk > xc) chunk = xc;
        const int nt = (ms + 31) / 32;
        for (long long j0 = 0; j0 < xc; j0 += chunk) {
            const int nb = (int)((xc - j0 < chunk) ? (xc - j0) : chunk);
            double *Xf = work, *T = work + m2 * chunk;
            const double *sblk = src + c.s_off[k] + j0 * lds;
            double *dblk = dst + c.s_off[k] + j0 * ldd;
            dim3 g1(nt * (nt + 1) / 2, nb);
            sym_copy_kernel<<<g1, 256, 0, st>>>(sblk, lds, Xf, ms);
            count_launch();
            CVXB_LAUNCH_CHECK();
            GemmDesc a;   // T = X * A  (form 1)   or   T = X * A' (form 2)
            a.M = ms; a.N = ms; a.K = ms;
            a.X = Xf; a.ldx = ms; a.x_kmajor = false; a.sX = m2;
            a.Y = A; a.ldy = ms; a.y_kmajor = form1; a.sY = 0;
            a.C = T; a.ldc = ms; a.sC = m2; a.batch = nb;
            CVXB_TRY(dmma_gemm(a, st));
            GemmDesc b;   // dst = A' * T (form 1)  or  A * T (form 2); lower triangle only
            b.M = ms; b.N = ms; b.K = ms;
            b.X = A; b.ldx = ms; b.x_kmajor = form1; b.sX = 0;
            b.Y = T; b.ldy = ms; b.y_kmajor = true; b.sY = m2;
            b.C = dblk; b.ldc = ms; b.sC = ldd; b.batch = nb; b.lower_only = true;
            CVXB_TRY(dmma_gemm(b, st));
        }
    }
    return 0;
}

int gemv_t(int nrows, int ncols, const double *A, long long lda, const double *w, const double *x,
           double alpha, double beta, double *y, cudaStream_t st, const GemvBatch &bs) {
    if (ncols <= 0 || bs.batch <= 0) return 0;
    const bool vec = ((uintptr_t)A % 16 == 0) && (lda % 2 == 0) && ((uintptr_t)x % 16 == 0) &&
                     (!w || (uintptr_t)w % 16 == 0) &&
                     (bs.batch == 1 || (bs.sA % 2 == 0 && bs.sx % 2 == 0 && bs.sw % 2 == 0));
    dim3 grid((ncols + 7) / 8, bs.batch);
    if (vec) {
        if (w) gemv_t_kernel<true, true><<<grid, 256, 0, st>>>(nrows, ncols, A, lda, w, x, alpha, beta, y, bs);
        else   gemv_t_kernel<true, false><<<grid, 256, 0, st>>>(nrows, ncols, A, lda, w, x, alpha, beta, y, bs);
    } else {
        if (w) gemv_t_kernel<false, true><<<grid, 256, 0, st>>>(nrows, ncols, A, lda, w, x, alpha, beta, y, bs);
        else   gemv_t_kernel<false, false><<<grid, 256, 0, st>>>(nrows, ncols, A, lda, w, x, alpha, beta, y, bs);
    }
    count_launch();
    CVXB_LAUNCH_CHECK();
    return 0;
}

int gemv_n_chunks(int ncols) { return ncols <= 0 ? 1 : (ncols + GN_CH - 1) / GN_CH; }

int gemv_n(int nrows, int ncols, const double *A, long long lda, const double *w, const double *x,
           double alpha, double beta, double *y, double *ws, cudaStream_t st, const GemvBatch &bs) {
    if (nrows <= 0 || bs.batch <= 0) return 0;
    const int nch = gemv_n_chunks(ncols);
    const long long sws = (long long)nch * nrows;        // workspace per problem
    if (ncols > 0) {
        dim3 grid((nrows + 255) / 256, nch, bs.batch);
        gemv_n_partial_kernel<<<grid, 256, 0, st>>>(nrows, ncols, A, lda, x, ws, bs, sws);
        count_launch();
        CVXB_LAUNCH_CHECK();
    }
    dim3 rg((nrows + 255) / 256, bs.batch);
    gemv_n_reduce_kernel<<<rg, 256, 0, st>>>(nrows, ncols > 0 ? nch : 0, ws, w, alpha, beta, y, bs, sws);
    count_launch();
    CVXB_LAUNCH_CHECK();
    return 0;
}

int transpose_copy(const double *src, long long lds, double *dst, long long ldd, int rows, int cols,
                   cudaStream_t st, int batch, long long ssrc, long long sdst) {
    if (rows <= 0 || cols <= 0 || batch <= 0) return 0;
    dim3 grid((rows + 31) / 32, (cols + 31) / 32, batch);
    transpose_kernel<<<grid, 256, 0, st>>>(src, lds, dst, ldd, rows, cols, ssrc, sdst);
    count_launch();
    CVXB_LAUNCH_CHECK();
    return 0;
}

int vec_mul(int n, const double *a, const double *b, double *out, cudaStream_t st) {
    if (n <= 0) return 0;
    vec_mul_kernel<<<(n + 255) / 256, 256, 0, st>>>(n, a, b, out);
    count_launch();
    CVXB_LAUNCH_CHECK();
    return 0;
}
int vec_axpby(int n, double alpha, const double *x, double beta, double *y, cudaStream_t st) {
    if (n <= 0) return 0;
    vec_axpby_kernel<<<(n + 255) / 256, 256, 0, st>>>(n, alpha, x, beta, y);
    count_launch();
    CVXB_LAUNCH_CHECK();
    return 0;
}
int symmetrize_lower(int n, double *A, long long lda, int batch, long long stride,
                     cudaStream_t st) {
    if (n <= 1) return 0;
    const int nt = (n + 31) / 32;
    dim3 grid(nt * (nt + 1) / 2, batch);
    symmetrize_kernel<<<grid, 256, 0, st>>>(A, lda, n, stride);
    count_launch();
    CVXB_LAUNCH_CHECK();
    return 0;
}

}  // namespace cvxb
