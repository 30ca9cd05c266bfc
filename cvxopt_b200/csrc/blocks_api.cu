// C ABI, part 2: dense building blocks on device pointers (the BLAS/LAPACK calls the
// reference path makes: blas.syrk blas.c:3039, lapack.potrf lapack.c:1471,
// lapack.potrs lapack.c:1553, blas.gemm blas.c:2602) and the misc_solvers mirror
// (src/C/misc_solvers.c:1155-1173) on flat buffers.  Also the per-device context (CallCtx, common.cuh)
// of every entry point that takes no handle.
#include "cone.cuh"
#include <map>
#include <memory>
#include <mutex>

using namespace cvxb;

namespace {
// check_device has passed and the stream and CholWork exist once ok is set
struct DevCtx {
    cudaStream_t st = nullptr;
    std::unique_ptr<CholWork> cw;
    bool ok = false;
    std::mutex mu;
};
// Contexts are created on first use and never destroyed: CUDA calls are not safe during static destruction.
// The map itself is guarded by g_ctx_mu.
std::map<int, DevCtx *> g_ctx;
std::mutex g_ctx_mu;
}  // namespace

int cvxb::CallCtx::acquire(int device) {
    DevCtx *c;
    {
        std::lock_guard<std::mutex> g(g_ctx_mu);
        DevCtx *&slot = g_ctx[device];
        if (!slot) slot = new DevCtx;
        c = slot;
    }
    lock = std::unique_lock<std::mutex>(c->mu);
    if (c->ok) {
        CVXB_CUDA(cudaSetDevice(device));
    } else {
        CVXB_TRY(check_device(device));
        if (!c->st) CVXB_CUDA(cudaStreamCreateWithFlags(&c->st, cudaStreamNonBlocking));
        c->cw.reset(new CholWork());      // frees what an earlier attempt that failed part-way created
        CVXB_TRY(chol_work_create(*c->cw));
        c->ok = true;
    }
    st = c->st;
    cw = c->cw.get();
    return 0;
}

extern "C" {

int cvxb_syrk_scaled(int n, int k, const double *A, int lda, const double *rowscale,
                     const double *H, int ldh, double *C, int ldc, int device) {
    CallCtx ctx; CVXB_TRY(ctx.acquire(device));
    GemmDesc g;
    g.M = n; g.N = n; g.K = k;
    g.X = A; g.ldx = lda; g.x_kmajor = true;
    g.Y = A; g.ldy = lda; g.y_kmajor = true;
    g.w = rowscale;
    g.D = H; g.ldd = ldh; g.beta = 1.0;
    g.C = C; g.ldc = ldc; g.lower_only = true; g.splitk_ws = ctx.cw->splitk_ws.p;
    CVXB_TRY(dmma_gemm(g, ctx.st));
    CVXB_CUDA(cudaStreamSynchronize(ctx.st));
    return 0;
}

int cvxb_syrk_scaled_i8(int n, int k, const double *A, int lda, const double *d, const double *H, int ldh,
                        double *C, int ldc, int slices, int device) {
    CallCtx ctx; CVXB_TRY(ctx.acquire(device));
    if (slices < 1 || slices > 9) { set_error("syrk_scaled_i8: slices must be 1..9"); return CVXB_E_ARG; }
    Scratch<char> work;
    if (work.alloc(ozaki_workspace_bytes(n, k, slices))) {
        cudaGetLastError();
        set_error("syrk_scaled_i8: out of device memory for the slice workspace");
        return CVXB_E_NOMEM;
    }
    int rc = ozaki_syrk(n, k, A, lda, d, H, ldh, 1.0, C, ldc, slices, 0, work.p, ctx.st);
    cudaError_t e = cudaStreamSynchronize(ctx.st);
    if (rc) return rc;
    if (e != cudaSuccess) { set_error("syrk_scaled_i8: %s", cudaGetErrorString(e)); return CVXB_E_CUDA; }
    return 0;
}

int cvxb_potrf(int n, double *A, int lda, double *work_inv, int device) {
    CallCtx ctx; CVXB_TRY(ctx.acquire(device));
    CVXB_TRY(potrf_lower(n, A, lda, work_inv, *ctx.cw, ctx.st));
    int info = 0;
    CVXB_CUDA(cudaMemcpyAsync(&info, ctx.cw->d_info.p, sizeof(int), cudaMemcpyDeviceToHost, ctx.st));
    CVXB_CUDA(cudaStreamSynchronize(ctx.st));
    if (info > 0) set_error("potrf: leading minor of order %d is not positive definite", info);
    return info;
}

int cvxb_potrs(int n, const double *L, int ldl, const double *inv, double *b, int device) {
    CallCtx ctx; CVXB_TRY(ctx.acquire(device));
    CVXB_TRY(potrs_lower(n, L, ldl, inv, b, *ctx.cw, ctx.st));
    CVXB_CUDA(cudaStreamSynchronize(ctx.st));
    return 0;
}

int cvxb_gemm(int transa, int transb, int m, int n, int k, double alpha, const double *A, int lda,
              const double *B, int ldb, double beta, double *C, int ldc, int device) {
    CallCtx ctx; CVXB_TRY(ctx.acquire(device));
    const bool ta = (transa == 'T' || transa == 't'), tb = (transb == 'T' || transb == 't');
    GemmDesc g;
    g.M = m; g.N = n; g.K = k;
    // X[r,kk] = op(A)[r,kk]: 'N' -> A[r + kk*lda] (M-major), 'T' -> A[kk + r*lda] (K-major)
    g.X = A; g.ldx = lda; g.x_kmajor = ta;
    // Y[c,kk] = op(B)[kk,c]: 'N' -> B[kk + c*ldb] (K-major), 'T' -> B[c + kk*ldb] (M-major)
    g.Y = B; g.ldy = ldb; g.y_kmajor = !tb;
    g.D = (beta != 0.0) ? C : nullptr; g.ldd = ldc; g.beta = beta;
    g.C = C; g.ldc = ldc; g.alpha = alpha;
    CVXB_TRY(dmma_gemm(g, ctx.st));
    CVXB_CUDA(cudaStreamSynchronize(ctx.st));
    return 0;
}

// ---------------------------------------------------------------- batched building blocks of the batch solver
// Problem b of every operand is at base + b * stride.  The arguments are checked before the device, as the batch
// constructors do.
static int batch_args(const char *what, int batch, int size0, int size1) {
    if (batch < 1 || batch > CVXB_BATCH_MAX) {
        set_error("%s: batch = %d outside 1..%d", what, batch, CVXB_BATCH_MAX);
        return CVXB_E_ARG;
    }
    if (size0 < 0 || size1 < 0) {
        set_error("%s: negative size", what);
        return CVXB_E_ARG;
    }
    return 0;
}
static int ld_arg(const char *what, const char *name, long long ld, int rows) {
    if (ld < (rows > 1 ? rows : 1)) {
        set_error("%s: %s = %lld < max(1, %d)", what, name, ld, rows);
        return CVXB_E_ARG;
    }
    return 0;
}

int cvxb_potrf_batched(int n, double *A, int lda, long long sA, double *work_inv, long long sInv, int batch,
                       int *info, int device) {
    CVXB_TRY(batch_args("potrf_batched", batch, n, 0));
    CVXB_TRY(ld_arg("potrf_batched", "lda", lda, n));
    CallCtx ctx; CVXB_TRY(ctx.acquire(device));
    Scratch<int> d_info;
    Scratch<double> panel;
    const int ldw = (n + 1) & ~1;
    CVXB_TRY(d_info.alloc(batch));
    CVXB_TRY(panel.alloc((size_t)batch * ldw * NB));
    int rc = potrf_lower_batched(n, A, lda, sA, work_inv, sInv, batch, d_info.p, panel.p, ldw, ctx.st);
    if (rc == 0 && n > 0) {
        const cudaError_t e = cudaMemcpyAsync(info, d_info.p, (size_t)batch * sizeof(int), cudaMemcpyDeviceToHost,
                                              ctx.st);
        if (e != cudaSuccess) { set_error("potrf_batched: %s", cudaGetErrorString(e)); rc = CVXB_E_CUDA; }
    } else if (rc == 0) {
        for (int b = 0; b < batch; ++b) info[b] = 0;
    }
    const cudaError_t e = cudaStreamSynchronize(ctx.st);        // before the scratch goes back to the cache
    if (rc) return rc;
    if (e != cudaSuccess) { set_error("potrf_batched: %s", cudaGetErrorString(e)); return CVXB_E_CUDA; }
    return 0;
}

int cvxb_trsv_batched(int n, const double *L, int ldl, long long sL, const double *inv, long long sInv, double *b,
                      long long sb, int trans, int batch, int device) {
    CVXB_TRY(batch_args("trsv_batched", batch, n, 0));
    CVXB_TRY(ld_arg("trsv_batched", "ldl", ldl, n));
    if (trans != 'N' && trans != 'T') { set_error("trsv_batched: trans must be 'N' or 'T'"); return CVXB_E_ARG; }
    CallCtx ctx; CVXB_TRY(ctx.acquire(device));
    CVXB_TRY(trsv_lower(n, L, ldl, inv, b, trans == 'T', *ctx.cw, ctx.st, batch, sL, sInv, sb));
    CVXB_CUDA(cudaStreamSynchronize(ctx.st));
    return 0;
}

int cvxb_trsm_batched(int n, const double *L, int ldl, long long sL, const double *inv, long long sInv, double *B,
                      int ldb, long long sB, int ncols, int batch, int device) {
    CVXB_TRY(batch_args("trsm_batched", batch, n, ncols));
    CVXB_TRY(ld_arg("trsm_batched", "ldl", ldl, n));
    CVXB_TRY(ld_arg("trsm_batched", "ldb", ldb, n));
    CallCtx ctx; CVXB_TRY(ctx.acquire(device));
    CVXB_TRY(trsm_lower_left(n, L, ldl, inv, B, ldb, ncols, ctx.st, batch, sL, sInv, sB));
    CVXB_CUDA(cudaStreamSynchronize(ctx.st));
    return 0;
}

int cvxb_syrk_batched(int n, int k, const double *A, int lda, long long sA, const double *w, long long sw,
                      const double *D, int ldd, long long sD, double *C, int ldc, long long sC, int batch,
                      int device) {
    CVXB_TRY(batch_args("syrk_batched", batch, n, k));
    CVXB_TRY(ld_arg("syrk_batched", "lda", lda, k));
    CVXB_TRY(ld_arg("syrk_batched", "ldc", ldc, n));
    if (D) CVXB_TRY(ld_arg("syrk_batched", "ldd", ldd, n));
    CallCtx ctx; CVXB_TRY(ctx.acquire(device));
    GemmDesc g;
    g.M = n; g.N = n; g.K = k;
    g.X = A; g.ldx = lda; g.x_kmajor = true; g.sX = sA;
    g.Y = A; g.ldy = lda; g.y_kmajor = true; g.sY = sA;
    g.w = w; g.sW = w ? sw : 0;
    g.D = D; g.ldd = D ? ldd : 0; g.sD = D ? sD : 0; g.beta = D ? 1.0 : 0.0;
    g.C = C; g.ldc = ldc; g.sC = sC;
    g.lower_only = true; g.batch = batch;
    // no split-K workspace: the result depends on the problem and the layout only
    CVXB_TRY(dmma_gemm(g, ctx.st));
    CVXB_CUDA(cudaStreamSynchronize(ctx.st));
    return 0;
}

int cvxb_gemv_batched(int trans, int nrows, int ncols, const double *A, int lda, long long sA, const double *w,
                      long long sw, const double *x, long long sx, double alpha, double beta, double *y,
                      long long sy, int batch, int device) {
    CVXB_TRY(batch_args("gemv_batched", batch, nrows, ncols));
    CVXB_TRY(ld_arg("gemv_batched", "lda", lda, nrows));
    if (trans != 'N' && trans != 'T') { set_error("gemv_batched: trans must be 'N' or 'T'"); return CVXB_E_ARG; }
    CallCtx ctx; CVXB_TRY(ctx.acquire(device));
    GemvBatch bs;
    bs.batch = batch; bs.sA = sA; bs.sw = w ? sw : 0; bs.sx = sx; bs.sy = sy;
    if (trans == 'T') {
        CVXB_TRY(gemv_t(nrows, ncols, A, lda, w, x, alpha, beta, y, ctx.st, bs));
        CVXB_CUDA(cudaStreamSynchronize(ctx.st));
        return 0;
    }
    Scratch<double> ws;
    CVXB_TRY(ws.alloc((size_t)batch * nrows * gemv_n_chunks(ncols)));
    const int rc = gemv_n(nrows, ncols, A, lda, w, x, alpha, beta, y, ws.p, ctx.st, bs);
    const cudaError_t e = cudaStreamSynchronize(ctx.st);        // before the workspace goes back to the cache
    if (rc) return rc;
    if (e != cudaSuccess) { set_error("gemv_batched: %s", cudaGetErrorString(e)); return CVXB_E_CUDA; }
    return 0;
}

// ---------------------------------------------------------------- misc_solvers mirror
int cvxb_scale(double *x, int xr, int xc, const cvxb_dims *dims, const cvxb_scaling *W, int trans,
               int inverse, int space) {
    CallCtx ctx; CVXB_TRY(ctx.acquire(0));
    cudaStream_t st = ctx.st;
    ConeLayout c;
    CVXB_TRY(c.init(dims));
    if (xr < c.cdim) { set_error("scale: x has fewer rows than the cone dimension"); return CVXB_E_ARG; }
    DevScaling S;
    CVXB_TRY(S.alloc(c));
    CVXB_TRY(S.upload(c, W, space, st));
    Staged X;
    CVXB_TRY(X.in(x, (size_t)xr * xc, space, st));
    const bool inv = (inverse == 'I');
    double *xd = X.dev;
    if (c.mnl) CVXB_TRY(scale_rows(xd, xr, xd, xr, c.mnl, xc, inv ? S.dnli : S.dnl, st));
    if (c.ml) CVXB_TRY(scale_rows(xd + c.mnl, xr, xd + c.mnl, xr, c.ml, xc, inv ? S.di : S.d, st));
    if (c.nq) CVXB_TRY(scale_q(c, S, xd + c.mnl + c.ml, xr, xd + c.mnl + c.ml, xr, xc, inv, st));
    Scratch<double> work;
    if (c.ns && c.maxs) {
        size_t per = (size_t)2 * c.maxs * c.maxs;
        size_t cols = (size_t)xc;
        size_t cap = (size_t)1 << 28;
        size_t want = per * cols;
        if (want > cap) want = (cap / per ? cap / per : 1) * per;
        CVXB_TRY(work.alloc(want));
        double *base = xd + c.mnl + c.ml + c.sumq;
        CVXB_TRY(scale_s(c, S, base, xr, base, xr, xc, trans, inverse, work.p, want, st));
    }
    CVXB_TRY(X.out(st));
    CVXB_CUDA(cudaStreamSynchronize(st));
    return 0;
}

static int pack_common(const double *x, double *y, const cvxb_dims *dims, int space, bool do_pack) {
    CallCtx ctx; CVXB_TRY(ctx.acquire(0));
    cudaStream_t st = ctx.st;
    ConeLayout c;
    CVXB_TRY(c.init(dims));
    const size_t nin = do_pack ? c.cdim : c.cdim_pckd, nout = do_pack ? c.cdim_pckd : c.cdim;
    Staged X, Y;
    CVXB_TRY(X.in(x, nin, space, st));
    CVXB_TRY(Y.in(y, nout, space, st));   // unpack leaves the strict upper triangles untouched
    const int nlq = c.mnl + c.ml + c.sumq;
    if (nlq) CVXB_CUDA(cudaMemcpyAsync(Y.dev, X.dev, (size_t)nlq * sizeof(double), cudaMemcpyDeviceToDevice, st));
    if (do_pack) CVXB_TRY(pack_s(c, X.dev + nlq, c.cdim, Y.dev + nlq, c.cdim_pckd, 1, true, st));
    else         CVXB_TRY(unpack_s(c, X.dev + nlq, c.cdim_pckd, Y.dev + nlq, c.cdim, 1, st));
    CVXB_TRY(Y.out(st));
    CVXB_CUDA(cudaStreamSynchronize(st));
    return 0;
}

int cvxb_pack(const double *x, double *y, const cvxb_dims *dims, int space) {
    return pack_common(x, y, dims, space, true);
}
int cvxb_unpack(const double *x, double *y, const cvxb_dims *dims, int space) {
    return pack_common(x, y, dims, space, false);
}

int cvxb_pack2(double *x, int xr, int xc, const cvxb_dims *dims, int space) {
    CallCtx ctx; CVXB_TRY(ctx.acquire(0));
    cudaStream_t st = ctx.st;
    ConeLayout c;
    CVXB_TRY(c.init(dims));
    if (c.ns == 0 || c.maxs == 0) return 0;
    Staged X;
    CVXB_TRY(X.in(x, (size_t)xr * xc, space, st));
    const int nlq = c.mnl + c.ml + c.sumq;
    // in place in the reference (rows compacted towards the top); go through a copy
    Scratch<double> tmp;
    CVXB_TRY(tmp.alloc((size_t)c.sump * xc));
    CVXB_TRY(pack_s(c, X.dev + nlq, xr, tmp.p, c.sump, xc, false, st));
    CVXB_CUDA(cudaMemcpy2DAsync(X.dev + nlq, (size_t)xr * sizeof(double), tmp.p,
                                (size_t)c.sump * sizeof(double), (size_t)c.sump * sizeof(double),
                                xc, cudaMemcpyDeviceToDevice, st));
    CVXB_TRY(X.out(st));
    CVXB_CUDA(cudaStreamSynchronize(st));
    return 0;
}

int cvxb_symm(double *x, int n, int space) {
    CallCtx ctx; CVXB_TRY(ctx.acquire(0));
    Staged X;
    CVXB_TRY(X.in(x, (size_t)n * n, space, ctx.st));
    CVXB_TRY(symmetrize_lower(n, X.dev, n, 1, 0, ctx.st));
    CVXB_TRY(X.out(ctx.st));
    CVXB_CUDA(cudaStreamSynchronize(ctx.st));
    return 0;
}

}  // extern "C"
