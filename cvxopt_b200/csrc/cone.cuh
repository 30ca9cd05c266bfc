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

}  // namespace cvxb
