// misc.kkt_qr on the device (reference src/python/misc.py:1570-1699): KKT systems with a zero (1,1) block
//
//     [ 0   A'  G' ] [ux]   [bx]
//     [ A   0   0  ] [uy] = [by]          (conelp; the drivers' default for 'q'/'s' cones, coneprog.py:458-462)
//     [ G   0 -W'W ] [uz]   [bz]
//
// solved by two orthogonal factorisations instead of the normal equations:
//   once      A' = [Q1 Q2] [R1; 0]                 Householder reflectors (lapack.geqrf, misc.py:1603-1604), Q formed
//                                                   explicitly (n x n) so that later products are GEMM / GEMV
//   factor(W) Gs = pack(W^{-T} G);  [Gs1 Gs2] = Gs [Q1 Q2]   (lapack.ormqr :1619);   Gs2 = Q3 R3   (lapack.geqrf :1622)
//   solve     the reference's five steps (:1628-1697) with Q3, R3, Q, R1.
// The big factorisation Gs2 = Q3 R3 (cdim_pckd x (n-p)) is a Cholesky-QR with re-orthogonalisation: R from the
// Cholesky factor of Gs2'Gs2, Q = Gs2 R^-1, done twice (orthogonality ~eps when cond(Gs2) < 1e7); when the first
// Cholesky breaks down (cond(Gs2)^2 beyond 1/eps) it is restarted with the shift of Fukaya et al. (shifted
// Cholesky-QR3: s = 11 (m n + n(n+1)) eps |Gs2|_F^2, three passes).  Every flop is a DMMA GEMM / the blocked
// Cholesky of chol.cu; a Householder panel factorisation of a 131328 x 512 matrix would be a latency chain.
// Q3 is kept explicitly (as Q3', (n-p) x cdim_pckd) so that Q3'w and Q3 u are HBM-bound GEMVs.
#include "kkt_internal.cuh"
#include <cmath>

namespace cvxb {

namespace {

// Householder reflector k of the n x p matrix X (ld ldx): H = I - tau v v', v[k] = 1, v[k+1:] stored below the
// diagonal, H X[k:, k] = [beta; 0]   (dlarfg's conventions)
__global__ void __launch_bounds__(256) house_kernel(int n, int k, double *X, long long ldx, double *tau) {
    __shared__ double sh[32];
    double *x = X + (long long)k * ldx;
    double t = 0.0;
    for (int i = k + 1 + threadIdx.x; i < n; i += blockDim.x) t += x[i] * x[i];
    const double xn2 = block_sum(t, sh);
    const double alpha = x[k];
    if (xn2 == 0.0) { if (threadIdx.x == 0) tau[k] = 0.0; return; }
    const double beta = -copysign(sqrt(alpha * alpha + xn2), alpha);
    const double scal = 1.0 / (alpha - beta);
    __syncthreads();
    for (int i = k + 1 + threadIdx.x; i < n; i += blockDim.x) x[i] *= scal;
    if (threadIdx.x == 0) { tau[k] = (beta - alpha) / beta; x[k] = beta; }
}
// apply H_k (vector in column k of X below the diagonal) to columns [c0, c0 + gridDim.x) of T (rows k..n-1)
__global__ void __launch_bounds__(256) house_apply_kernel(int n, int k, const double *X, long long ldx, const double *tau,
                                                           double *T, long long ldt, int c0) {
    __shared__ double sh[32];
    const double tk = tau[k];
    if (tk == 0.0) return;
    const double *v = X + (long long)k * ldx;
    double *t = T + (long long)(c0 + blockIdx.x) * ldt;
    double a = 0.0;
    for (int i = k + 1 + threadIdx.x; i < n; i += blockDim.x) a += v[i] * t[i];
    const double wv = (block_sum(a, sh) + t[k]) * tk;
    __syncthreads();
    for (int i = k + 1 + threadIdx.x; i < n; i += blockDim.x) t[i] -= wv * v[i];
    if (threadIdx.x == 0) t[k] -= wv;
}
__global__ void identity_kernel(int n, double *Q, long long ld) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (long long)n * n) return;
    const int i = (int)(e % n), j = (int)(e / n);
    Q[i + (long long)j * ld] = (i == j) ? 1.0 : 0.0;
}
// R1 (p x p, ld p) = upper triangle of the first p rows of X
__global__ void extract_r_kernel(int p, const double *X, long long ldx, double *R) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= p * p) return;
    const int i = e % p, j = e / p;
    R[e] = (i <= j) ? X[i + (long long)j * ldx] : 0.0;
}
// x := R^{-1} x (trans 0) or R^{-T} x (trans 1), R p x p upper triangular; one CTA (lapack.trtrs with one
// right-hand side, misc.py:1637, :1690)
__global__ void __launch_bounds__(256) trsv_upper_small_kernel(int p, const double *R, double *x, int trans) {
    __shared__ double xj;
    if (!trans) {
        for (int j = p - 1; j >= 0; --j) {
            if (threadIdx.x == 0) { xj = x[j] / R[j + (long long)j * p]; x[j] = xj; }
            __syncthreads();
            for (int i = threadIdx.x; i < j; i += blockDim.x) x[i] -= R[i + (long long)j * p] * xj;
            __syncthreads();
        }
    } else {
        for (int j = 0; j < p; ++j) {
            if (threadIdx.x == 0) { xj = x[j] / R[j + (long long)j * p]; x[j] = xj; }
            __syncthreads();
            for (int i = j + 1 + threadIdx.x; i < p; i += blockDim.x) x[i] -= R[j + (long long)i * p] * xj;
            __syncthreads();
        }
    }
}
__global__ void sumsq_kernel(long long rows, int cols, const double *X, long long ld, double *out) {
    __shared__ double sh[32];
    double t = 0.0;
    const double *x = X + (long long)blockIdx.x * ld;
    for (long long i = threadIdx.x; i < rows; i += blockDim.x) t += x[i] * x[i];
    t = block_sum(t, sh);
    if (threadIdx.x == 0) atomicAdd(out, t);
}
__global__ void add_diag_kernel(int n, double *C, long long ld, const double *norm2, double factor) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) C[i + (long long)i * ld] += factor * norm2[0];
}
__global__ void axpy_kernel(int n, double a, const double *x, double *y) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) y[i] += a * x[i];
}
__global__ void axmy_kernel(int n, const double *x, double *y) {      // y := x - y
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) y[i] = x[i] - y[i];
}

}  // namespace

int kkt_qr_setup(cvxb_kkt *k) {
    const ConeLayout &c = k->cone;
    const int n = k->n, p = k->p, Kp = c.cdim_pckd;
    if (c.mnl) { set_error("kkt_qr: nonlinear rows are not part of this route (the reference's kkt_qr takes no mnl)"); return CVXB_E_ARG; }
    if (Kp < n - p) { set_error("kkt_qr: Rank([A; G]) < n (fewer cone rows than free variables)"); return CVXB_E_ARG; }
    auto q = std::make_unique<QrState>();
    cudaStream_t st = k->st;
    q->nq = n - p;
    const size_t nn = (size_t)(n > 0 ? n : 1);
    q->ldf = ((Kp + 1) & ~1) > 2 ? ((Kp + 1) & ~1) : 2;
    q->ldq = ((q->nq + 1) & ~1) > 2 ? ((q->nq + 1) & ~1) : 2;
    q->ldc = q->ldq;
    CVXB_TRY(q->GsF.alloc((size_t)q->ldf * nn));
    CVXB_TRY(q->Q3t.alloc((size_t)q->ldq * (Kp > 0 ? Kp : 1)));
    const int nbk = (q->nq + NB - 1) / NB + 1;
    for (int i = 0; i < 3; ++i) {
        CVXB_TRY(q->C[i].alloc((size_t)q->ldc * (q->nq > 0 ? q->nq : 1)));
        CVXB_TRY(q->inv[i].alloc((size_t)2 * nbk * NB * NB));
    }
    const size_t kp1 = (size_t)(Kp > 0 ? Kp : 1);
    CVXB_TRY(q->w.alloc(kp1));
    CVXB_TRY(q->u.alloc(kp1 > nn ? kp1 : nn));
    CVXB_TRY(q->vv.alloc(nn));
    CVXB_TRY(q->xt.alloc(nn));
    CVXB_TRY(q->norm2.alloc(1));
    {
        size_t a = nn * (size_t)gemv_n_chunks(Kp > n ? Kp : n), b = kp1 * (size_t)gemv_n_chunks(n);
        CVXB_TRY(q->ws.alloc(a > b ? a : b));
    }
    if (p > 0) {
        // A' = [Q1 Q2][R1; 0]: p Householder reflectors of the n x p matrix, then Q = H_0 ... H_{p-1} applied to I
        q->ldQ = (n + 1) & ~1;
        CVXB_TRY(q->Q.alloc((size_t)q->ldQ * nn));
        CVXB_TRY(q->R1.alloc((size_t)p * p));
        CVXB_TRY(q->tau.alloc((size_t)p));
        CVXB_TRY(q->GsQ.alloc((size_t)q->ldf * nn));
        DevBuf<double> QAbuf;                       // n x p
        const long long ldqa = (n + 1) & ~1;
        CVXB_TRY(QAbuf.alloc((size_t)ldqa * p));
        double *QA = QAbuf.p, *tau = q->tau.p;
        int rc = transpose_copy(k->Aeq.p, k->lda_eq, QA, ldqa, p, n, st);
        for (int j = 0; j < p && rc == 0; ++j) {
            house_kernel<<<1, 256, 0, st>>>(n, j, QA, ldqa, tau);
            if (j + 1 < p) house_apply_kernel<<<p - j - 1, 256, 0, st>>>(n, j, QA, ldqa, tau, QA, ldqa, j + 1);
            count_launch(2);
        }
        if (rc == 0) {
            identity_kernel<<<(unsigned)(((long long)n * n + 255) / 256), 256, 0, st>>>(n, q->Q.p, q->ldQ);
            for (int j = p - 1; j >= 0; --j) {
                // H_j touches rows j.. only and columns < j of the partial product are still unit vectors e_c with
                // c < j: apply to columns j .. n-1
                house_apply_kernel<<<n - j, 256, 0, st>>>(n, j, QA, ldqa, tau, q->Q.p, q->ldQ, j);
                count_launch();
            }
            extract_r_kernel<<<(p * p + 255) / 256, 256, 0, st>>>(p, QA, ldqa, q->R1.p);
            count_launch(2);
        }
        cudaError_t e = cudaStreamSynchronize(st);
        if (rc) return rc;
        if (e != cudaSuccess) { set_error("kkt_qr setup: %s", cudaGetErrorString(e)); return CVXB_E_CUDA; }
        CVXB_LAUNCH_CHECK();
    }
    k->qr = std::move(q);
    return 0;
}

int kkt_qr_factor(cvxb_kkt *k, const cvxb_scaling *Wp, int space) {
    QrState *q = k->qr.get();
    const ConeLayout &c = k->cone;
    const int n = k->n, p = k->p, Kp = c.cdim_pckd, nq = q->nq;
    cudaStream_t st = k->st;
    CVXB_CUDA(cudaEventRecord(k->e0, st));
    CVXB_TRY(k->W.upload(c, Wp, space, st));
    // ---- Gs = pack(W^{-T} G), every row materialised                            (misc.py:1614-1616)
    if (c.ml > 0) CVXB_TRY(scale_rows(k->G, k->ldg, q->GsF.p, q->ldf, c.ml, n, k->W.di, st));
    CVXB_TRY(kkt_scale_pack_G(k, q->GsF.p + c.ml, q->ldf));
    CVXB_CUDA(cudaEventRecord(k->e1, st));
    const double *Gs2 = q->GsF.p;
    if (p > 0) {                                   // [Gs1 Gs2] = Gs [Q1 Q2]          (:1619)
        GemmDesc g;
        g.M = Kp; g.N = n; g.K = n;
        g.X = q->GsF.p; g.ldx = (int)q->ldf; g.x_kmajor = false;
        g.Y = q->Q.p; g.ldy = (int)q->ldQ; g.y_kmajor = true;
        g.C = q->GsQ.p; g.ldc = (int)q->ldf;
        CVXB_TRY(dmma_gemm(g, st));
        Gs2 = q->GsQ.p + (long long)p * q->ldf;
    }
    int info = 0;
    if (nq > 0) {
        // ---- Gs2 = Q3 R3 by Cholesky-QR passes; Q3' is built in place in Q3t
        double *Q3t = q->Q3t.p, *norm2 = q->norm2.p;
        auto run = [&](bool shifted) -> int {
            q->npass = shifted ? 3 : 2;
            CVXB_TRY(transpose_copy(Gs2, q->ldf, Q3t, q->ldq, Kp, nq, st));
            if (shifted) {
                CVXB_CUDA(cudaMemsetAsync(norm2, 0, sizeof(double), st));
                sumsq_kernel<<<nq, 256, 0, st>>>(Kp, nq, Gs2, q->ldf, norm2);
                count_launch();
            }
            for (int ps = 0; ps < q->npass; ++ps) {
                double *C = q->C[ps].p, *inv = q->inv[ps].p;
                GemmDesc g;                        // C = B B'  (B = Q3t, nq x Kp), lower triangle
                g.M = nq; g.N = nq; g.K = Kp;
                g.X = Q3t; g.ldx = (int)q->ldq; g.x_kmajor = false;
                g.Y = Q3t; g.ldy = (int)q->ldq; g.y_kmajor = false;
                g.C = C; g.ldc = (int)q->ldc; g.lower_only = true; g.splitk_ws = k->cw.splitk_ws.p;
                CVXB_TRY(dmma_gemm(g, st));
                if (shifted && ps == 0) {
                    const double fac = 11.0 * ((double)Kp * nq + (double)nq * (nq + 1)) * 1.1102230246251565e-16;
                    add_diag_kernel<<<(nq + 255) / 256, 256, 0, st>>>(nq, C, q->ldc, norm2, fac);
                    count_launch();
                }
                CVXB_TRY(potrf_lower(nq, C, (int)q->ldc, inv, k->cw, st));
                CVXB_CUDA(cudaMemcpyAsync(&info, k->cw.d_info.p, sizeof(int), cudaMemcpyDeviceToHost, st));
                CVXB_CUDA(cudaStreamSynchronize(st));
                if (info > 0) return 0;
                CVXB_TRY(trsm_lower_left(nq, C, q->ldc, inv, Q3t, q->ldq, Kp, st));
            }
            return 0;
        };
        CVXB_TRY(run(false));
        if (info > 0) { info = 0; CVXB_TRY(run(true)); }
    }
    CVXB_CUDA(cudaEventRecord(k->e3, st));
    CVXB_CUDA(cudaStreamSynchronize(st));
    float t;
    cudaEventElapsedTime(&t, k->e0, k->e3); k->factor_ms = t;
    cudaEventElapsedTime(&t, k->e0, k->e1); k->br[0] = t;
    k->br[1] = 0; k->br[2] = 0;
    if (info > 0) {
        // Gs2 is numerically rank deficient: the reference's geqrf would return a singular R3 and trtrs raises
        set_error("kkt_qr: W^{-T} G Q2 is rank deficient (pivot %d)", info);
        return info;
    }
    return 0;
}

// on entry w = bzp = W^{-T} bz, packed (:1626-1627); on return it holds W*uz, packed, for kkt_unpack_z (:1675)
int kkt_qr_solve(cvxb_kkt *k, double *xd, double *yd) {
    const QrState *q = k->qr.get();
    const ConeLayout &c = k->cone;
    const int n = k->n, p = k->p, Kp = c.cdim_pckd, nq = q->nq;
    cudaStream_t st = k->st;
    const int T = 256;
    double *w = k->bzp.p;
    double *vv = q->vv.p, *xt = q->xt.p, *u = q->u.p, *ws = q->ws.p;
    const double *Q = q->Q.p, *R1 = q->R1.p, *GsQ = q->GsQ.p, *Q3t = q->Q3t.p;
    // vv := [Q1'bx; R3^{-T} Q2'bx]                                                (:1630-1633)
    if (p > 0) CVXB_TRY(gemv_t(n, n, Q, q->ldQ, nullptr, xd, 1.0, 0.0, vv, st));
    else CVXB_CUDA(cudaMemcpyAsync(vv, xd, (size_t)n * sizeof(double), cudaMemcpyDeviceToDevice, st));
    for (int ps = 0; ps < q->npass; ++ps)       // R3^{-T} = L_np^{-1} ... L_1^{-1}
        CVXB_TRY(trsv_lower(nq, q->C[ps].p, (int)q->ldc, q->inv[ps].p, vv + p, false, k->cw, st));
    if (p > 0) {
        // xt[:p] := R1^{-T} by;   w := w - Gs1 xt[:p]                             (:1636-1642)
        CVXB_CUDA(cudaMemcpyAsync(xt, yd, (size_t)p * sizeof(double), cudaMemcpyDeviceToDevice, st));
        trsv_upper_small_kernel<<<1, 256, 0, st>>>(p, R1, xt, 1);
        count_launch();
        CVXB_TRY(gemv_n(Kp, p, GsQ, q->ldf, nullptr, xt, -1.0, 1.0, w, ws, st));
    }
    // u := Q3'w + vv[p:]                                                          (:1646-1650)
    if (nq > 0) {
        CVXB_CUDA(cudaMemcpyAsync(u, vv + p, (size_t)nq * sizeof(double), cudaMemcpyDeviceToDevice, st));
        CVXB_TRY(gemv_n(nq, Kp, Q3t, q->ldq, nullptr, w, 1.0, 1.0, u, ws, st));
        // xt[p:] := R3^{-1} u = L_1^{-T} ... L_np^{-T} u                          (:1653-1655)
        CVXB_CUDA(cudaMemcpyAsync(xt + p, u, (size_t)nq * sizeof(double), cudaMemcpyDeviceToDevice, st));
        for (int ps = q->npass - 1; ps >= 0; --ps)
            CVXB_TRY(trsv_lower(nq, q->C[ps].p, (int)q->ldc, q->inv[ps].p, xt + p, true, k->cw, st));
    }
    // x := [Q1 Q2] xt                                                             (:1659)
    if (p > 0) CVXB_TRY(gemv_n(n, n, Q, q->ldQ, nullptr, xt, 1.0, 0.0, xd, ws, st));
    else CVXB_CUDA(cudaMemcpyAsync(xd, xt, (size_t)n * sizeof(double), cudaMemcpyDeviceToDevice, st));
    // W*uz (packed) := Q3 u - w, kept in bzp                                       (:1663-1665)
    if (nq > 0) CVXB_TRY(gemv_t(nq, Kp, Q3t, q->ldq, nullptr, u, 1.0, -1.0, w, st));
    else if (Kp > 0) { axmy_kernel<<<(Kp + T - 1) / T, T, 0, st>>>(Kp, u, w); count_launch(); }
    if (p > 0) {
        // y := R1^{-1} (Q1'bx - Gs1' (W uz))                                       (:1669-1673)
        CVXB_CUDA(cudaMemcpyAsync(yd, vv, (size_t)p * sizeof(double), cudaMemcpyDeviceToDevice, st));
        CVXB_TRY(gemv_t(Kp, p, GsQ, q->ldf, nullptr, w, -1.0, 1.0, yd, st));
        trsv_upper_small_kernel<<<1, 256, 0, st>>>(p, R1, yd, 0);
        count_launch();
    }
    CVXB_LAUNCH_CHECK();
    return 0;
}

}  // namespace cvxb
