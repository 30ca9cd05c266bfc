// Nesterov-Todd scaling on the device: misc.compute_scaling / misc.update_scaling of the reference
// (src/python/misc.py:250-419 and :422-634) for every cone type.
//
//   nonlinear + 'l' rows : elementwise (one thread per row)
//   'q' cones            : one CTA per cone: hyperbolic norms, the hyperbolic-Householder vector v, beta, lambda
//   's' cones            : Cholesky factors Ls, Lz of the two blocks (compute_scaling; update_scaling receives them),
//                          M = Lz' Ls (DMMA GEMM), SVD  M = U diag(lambda) V'  by one-sided (Hestenes) Jacobi with
//                          the round-robin parallel ordering, then   r = Ls V lambda^-1/2,  rti = Lz U lambda^-1/2
//                          (equal to the reference's  r = Lz^-T U lambda^1/2,  rti = Lz U lambda^-1/2  because
//                          Lz' Ls V = U lambda;  two GEMMs instead of a triangular solve), singular values sorted
//                          descending as LAPACK's gesvd returns them (:398, :611).
// The SVD replaces lapack.gesvd (src/C/lapack.c gesvd binding); blocks of order <= 48 run all sweeps inside one CTA
// (shared memory), larger ones one cooperative launch per sweep (grid barrier between the rounds of disjoint column pairs).
#include "cone.cuh"
#include <cooperative_groups.h>
#include <cmath>
#include <cstdlib>

using namespace cvxb;

namespace {

// ---------------------------------------------------------------- 'l' / nonlinear rows
// d = sqrt(s/z), di = 1/d, lambda = sqrt(s*z)                                   (misc.py:266-287)
__global__ void nt_l_compute_kernel(int m, const double *s, const double *z, double *d, double *di, double *lm) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const double sv = s[i], zv = z[i];
    const double dv = sqrt(sv / zv);
    d[i] = dv;
    di[i] = 1.0 / dv;
    lm[i] = sqrt(sv * zv);
}
// s := sqrt(s), z := sqrt(z), d := d*s/z, di = 1/d, lambda := s*z               (misc.py:450-468)
__global__ void nt_l_update_kernel(int m, double *s, double *z, double *d, double *di, double *lm) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const double ss = sqrt(s[i]), sz = sqrt(z[i]);
    s[i] = ss; z[i] = sz;
    const double dv = (d[i] * ss) / sz;
    d[i] = dv;
    di[i] = 1.0 / dv;
    lm[i] = ss * sz;
}

// ---------------------------------------------------------------- 'q' cones
// one CTA per cone                                                               (misc.py:311-354)
__global__ void nt_q_compute_kernel(const int *q, const int *qoff, const int *voff, int lam_base, const double *s,
                                    const double *z, double *vall, double *beta, double *lm) {
    __shared__ double sh[32];
    const int k = blockIdx.x;
    q_nt_compute(CtaTeam{(int)threadIdx.x, (int)blockDim.x, sh}, s + qoff[k], z + qoff[k], vall + voff[k],
                 lm + lam_base + voff[k], beta + k, q[k]);
}

// one CTA per cone; s, z hold the new iterates in the current scaling and are normalised in place   (misc.py:504-573)
__global__ void nt_q_update_kernel(const int *q, const int *qoff, const int *voff, int lam_base, double *s, double *z,
                                   double *vall, double *beta, double *lm) {
    __shared__ double sh[32];
    const int k = blockIdx.x;
    q_nt_update(CtaTeam{(int)threadIdx.x, (int)blockDim.x, sh}, s + qoff[k], z + qoff[k], vall + voff[k],
                lm + lam_base + voff[k], beta + k, q[k]);
}

// ---------------------------------------------------------------- 's' cones: helpers
// dst (m x m, ld m) = lower triangle of src (zero above the diagonal)
__global__ void tril_copy_kernel(int m, const double *src, double *dst) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= m * m) return;
    const int i = e % m, j = e / m;
    dst[e] = (i >= j) ? src[e] : 0.0;
}
__global__ void set_identity_kernel(int m, double *V) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= m * m) return;
    V[e] = (e % m == e / m) ? 1.0 : 0.0;
}


// One round of one-sided Jacobi: CTA t orthogonalises columns (p, q) of B and applies the same rotation to V.
__global__ void __launch_bounds__(128) jacobi_round_kernel(int m, int m2, int r, double *B, double *V, int *nrot) {
    __shared__ double sh[32];
    int p, q;
    svd_pair(m2, r, blockIdx.x, p, q);
    if (q >= m) return;                        // bye
    double *bp = B + (size_t)p * m, *bq = B + (size_t)q * m;
    double a = 0.0, b = 0.0, g = 0.0;
    for (int i = threadIdx.x; i < m; i += blockDim.x) {
        const double x = bp[i], y = bq[i];
        a += x * x; b += y * y; g += x * y;
    }
    a = block_sum(a, sh); b = block_sum(b, sh); g = block_sum(g, sh);
    // orthogonal to working accuracy: the computed dot product carries ~sqrt(m) eps |p||q| of rounding noise
    if (!(fabs(g) > (2.0 * 2.220446049250313e-16 * sqrt((double)m)) * sqrt(a * b)) || g == 0.0) return;
    const double zeta = (b - a) / (2.0 * g);
    const double tt = (zeta >= 0.0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
    const double c = 1.0 / sqrt(1.0 + tt * tt), sn = c * tt;
    double *vp = V + (size_t)p * m, *vq = V + (size_t)q * m;
    for (int i = threadIdx.x; i < m; i += blockDim.x) {
        const double x = bp[i], y = bq[i];
        bp[i] = c * x - sn * y; bq[i] = sn * x + c * y;
        const double u = vp[i], w = vq[i];
        vp[i] = c * u - sn * w; vq[i] = sn * u + c * w;
    }
    if (threadIdx.x == 0) atomicAdd(nrot, 1);
}

// A whole sweep (all m2 - 1 rounds) in one cooperative launch: CTA t handles pair t of every round, a grid barrier
// separates the rounds.  The per-round launches above cost ~25 us each at m = 512 (launch gap + three block
// reductions + two passes over four columns); here a round is one fused reduction, the two passes and the barrier.
__global__ void __launch_bounds__(128) jacobi_sweep_kernel(int m, int m2, double *B, double *V, int *nrot) {
    namespace cg = cooperative_groups;
    cg::grid_group grid = cg::this_grid();
    __shared__ double sh[3][4];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    int rotated = 0;
    for (int r = 0; r < m2 - 1; ++r) {
        int p, q;
        svd_pair(m2, r, blockIdx.x, p, q);
        if (q < m) {
            double *bp = B + (size_t)p * m, *bq = B + (size_t)q * m;
            double a = 0.0, b = 0.0, g = 0.0;
            for (int i = tid; i < m; i += 128) {
                const double x = bp[i], y = bq[i];
                a += x * x; b += y * y; g += x * y;
            }
            a = warp_sum(a); b = warp_sum(b); g = warp_sum(g);
            if (lane == 0) { sh[0][warp] = a; sh[1][warp] = b; sh[2][warp] = g; }
            __syncthreads();
            a = (sh[0][0] + sh[0][1]) + (sh[0][2] + sh[0][3]);
            b = (sh[1][0] + sh[1][1]) + (sh[1][2] + sh[1][3]);
            g = (sh[2][0] + sh[2][1]) + (sh[2][2] + sh[2][3]);
            __syncthreads();
            if ((fabs(g) > (2.0 * 2.220446049250313e-16 * sqrt((double)m)) * sqrt(a * b)) && g != 0.0) {
                const double zeta = (b - a) / (2.0 * g);
                const double tt = (zeta >= 0.0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
                const double c = 1.0 / sqrt(1.0 + tt * tt), sn = c * tt;
                double *vp = V + (size_t)p * m, *vq = V + (size_t)q * m;
                for (int i = tid; i < m; i += 128) {
                    const double x = bp[i], y = bq[i];
                    bp[i] = c * x - sn * y; bq[i] = sn * x + c * y;
                    const double u = vp[i], w = vq[i];
                    vp[i] = c * u - sn * w; vq[i] = sn * u + c * w;
                }
                rotated = 1;
            }
        }
        grid.sync();
    }
    if (rotated && tid == 0) atomicAdd(nrot, 1);
}

// Small blocks (m <= 48): the whole SVD iteration of one block inside one CTA, B and V in shared memory
// (2 m^2 doubles <= 36 KB), one warp per column pair.
__global__ void __launch_bounds__(256) jacobi_small_kernel(int m, double *Bg, double *Vg, int maxsweeps) {
    extern __shared__ double jsm[];
    double *B = jsm, *V = jsm + m * m;
    __shared__ int rot;
    for (int e = threadIdx.x; e < m * m; e += blockDim.x) { B[e] = Bg[e]; V[e] = (e % m == e / m) ? 1.0 : 0.0; }
    __syncthreads();
    jacobi_svd_cta(m, B, V, maxsweeps, rot);
    for (int e = threadIdx.x; e < m * m; e += blockDim.x) { Bg[e] = B[e]; Vg[e] = V[e]; }
}

// After convergence B = U diag(sigma): sigma[j] = |B[:,j]|, rank them descending (stable), and emit
//   U (columns sorted) into Uout, V (columns sorted) into Vout, sigma into sig.   One CTA per block.
__global__ void __launch_bounds__(256) svd_finish_kernel(int m, const double *B, const double *V, double *Uout,
                                                          double *Vout, double *sig, double *norms, int *perm) {
    __shared__ double sh[32];
    for (int j = 0; j < m; ++j) {               // column norms (m <= a few hundred: a serial loop of CTA reductions)
        double t = 0.0;
        for (int i = threadIdx.x; i < m; i += blockDim.x) { const double x = B[(size_t)j * m + i]; t += x * x; }
        t = block_sum(t, sh);
        if (threadIdx.x == 0) norms[j] = sqrt(t);
    }
    __syncthreads();
    for (int j = threadIdx.x; j < m; j += blockDim.x) {      // rank of column j in descending order
        const double nj = norms[j];
        int rank = 0;
        for (int k = 0; k < m; ++k) rank += (norms[k] > nj) || (norms[k] == nj && k < j);
        perm[rank] = j;
    }
    __syncthreads();
    for (int jj = 0; jj < m; ++jj) {
        const int j = perm[jj];
        const double nj = norms[j];
        const double inv = nj > 0.0 ? 1.0 / nj : 0.0;
        for (int i = threadIdx.x; i < m; i += blockDim.x) {
            Uout[(size_t)jj * m + i] = B[(size_t)j * m + i] * inv;
            Vout[(size_t)jj * m + i] = V[(size_t)j * m + i];
        }
        if (threadIdx.x == 0) sig[jj] = nj;
    }
}
// X[:, j] *= sigma[j]^(-1/2)
__global__ void colscale_rsqrt_kernel(int m, double *X, const double *sig) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= m * m) return;
    X[e] *= 1.0 / sqrt(sig[e / m]);
}
// dst = src' (m x m)
__global__ void transpose_small_kernel(int m, const double *src, double *dst) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= m * m) return;
    const int i = e % m, j = e / m;
    dst[(size_t)i * m + j] = src[e];
}

int gemm_mm(int transa, int transb, int m, const double *A, const double *B, double *C, cudaStream_t st) {
    GemmDesc g;
    g.M = m; g.N = m; g.K = m;
    g.X = A; g.ldx = m; g.x_kmajor = (transa == 'T');
    g.Y = B; g.ldy = m; g.y_kmajor = !(transb == 'T');
    g.C = C; g.ldc = m;
    return dmma_gemm(g, st);
}

// SVD of the m x m matrix in B (overwritten): U, V (columns sorted by descending singular value), sigma.
// work: B itself + Vw (m*m) + norms (m) + perm (m ints)
int svd_jacobi(int m, double *B, double *Vw, double *U, double *V, double *sig, double *norms, int *perm, int *d_cnt,
               cudaStream_t st) {
    if (m <= 0) return 0;
    const int T = 256, nb = (m * m + T - 1) / T;
    if (m <= 48) {
        jacobi_small_kernel<<<1, 256, 2 * (size_t)m * m * sizeof(double), st>>>(m, B, Vw, 30);
        count_launch();
        svd_finish_kernel<<<1, 256, 0, st>>>(m, B, Vw, U, V, sig, norms, perm);
        count_launch();
        CVXB_LAUNCH_CHECK();
        return 0;
    }
    set_identity_kernel<<<nb, T, 0, st>>>(m, Vw);
    count_launch();
    const int m2 = (m + 1) & ~1;
    // one cooperative launch per sweep when every pair's CTA can be resident at once, else one launch per round
    const bool coop = coop_launch_fits((const void *)jacobi_sweep_kernel, 128, m2 / 2);
    for (int sweep = 0; sweep < 30; ++sweep) {
        CVXB_CUDA(cudaMemsetAsync(d_cnt, 0, sizeof(int), st));
        if (coop) {
            int mm_ = m, m2_ = m2;
            void *args[] = {&mm_, &m2_, &B, &Vw, &d_cnt};
            CVXB_CUDA(cudaLaunchCooperativeKernel((const void *)jacobi_sweep_kernel, dim3(m2 / 2), dim3(128), args, 0, st));
            count_launch();
        } else {
            for (int r = 0; r < m2 - 1; ++r) {
                jacobi_round_kernel<<<m2 / 2, 128, 0, st>>>(m, m2, r, B, Vw, d_cnt);
                count_launch();
            }
        }
        CVXB_LAUNCH_CHECK();
        int cnt = 0;
        CVXB_CUDA(cudaMemcpyAsync(&cnt, d_cnt, sizeof(int), cudaMemcpyDeviceToHost, st));
        CVXB_CUDA(cudaStreamSynchronize(st));
        if (cnt == 0) break;
    }
    svd_finish_kernel<<<1, 256, 0, st>>>(m, B, Vw, U, V, sig, norms, perm);
    count_launch();
    CVXB_LAUNCH_CHECK();
    return 0;
}

// the 's' part shared by compute (need_chol) and update: blocks of s/z are overwritten
int nt_s_blocks(const ConeLayout &c, double *sS, double *zS, double *r, double *rti, double *lam_s,
                bool is_update, cudaStream_t st) {
    if (c.ns == 0) return 0;
    const size_t mm = (size_t)c.maxs * c.maxs;
    Scratch<double> t[7];
    Scratch<int> ti, tc;
    for (int i = 0; i < 7; ++i) CVXB_TRY(t[i].alloc(mm));
    CVXB_TRY(ti.alloc(c.maxs));
    CVXB_TRY(tc.alloc(1));
    double *Ls = t[0].p, *Lz = t[1].p, *M = t[2].p, *Vw = t[3].p, *U = t[4].p, *V = t[5].p, *tmp = t[6].p;
    Scratch<double> tn, tinv;
    CVXB_TRY(tn.alloc(c.maxs));
    const int nbk = (c.maxs + NB - 1) / NB + 1;
    CVXB_TRY(tinv.alloc((size_t)2 * nbk * NB * NB));
    Scratch<double> tpanel;
    const int ldw = (c.maxs + 1) & ~1;
    CVXB_TRY(tpanel.alloc((size_t)ldw * NB));
    Scratch<int> tinfo;
    CVXB_TRY(tinfo.alloc(1));
    int lam_off = 0;
    for (int k = 0; k < c.ns; ++k) {
        const int m = c.s[k];
        if (m == 0) continue;
        double *sk = sS + c.s_off[k], *zk = zS + c.s_off[k];
        double *rk = r + c.r_off[k], *rtk = rti + c.r_off[k];
        const int T = 256, nb = (m * m + T - 1) / T;
        if (!is_update) {
            // sk = Ls Ls', zk = Lz Lz'   (lapack.potrf, misc.py:386-391); strictly upper parts zeroed (:395-396)
            for (int w = 0; w < 2; ++w) {
                double *L = w ? Lz : Ls;
                tril_copy_kernel<<<nb, T, 0, st>>>(m, w ? zk : sk, L);
                count_launch();
                CVXB_TRY(potrf_lower_batched(m, L, m, 0, tinv.p, 0, 1, tinfo.p, tpanel.p, ldw, st));
                int info = 0;
                CVXB_CUDA(cudaMemcpyAsync(&info, tinfo.p, sizeof(int), cudaMemcpyDeviceToHost, st));
                CVXB_CUDA(cudaStreamSynchronize(st));
                if (info > 0) { set_error("compute_scaling: 's' block %d is not positive definite", k); return info; }
                tril_copy_kernel<<<nb, T, 0, st>>>(m, L, tmp);
                count_launch();
                CVXB_CUDA(cudaMemcpyAsync(L, tmp, (size_t)m * m * sizeof(double), cudaMemcpyDeviceToDevice, st));
            }
        } else {
            CVXB_CUDA(cudaMemcpyAsync(Ls, sk, (size_t)m * m * sizeof(double), cudaMemcpyDeviceToDevice, st));
            CVXB_CUDA(cudaMemcpyAsync(Lz, zk, (size_t)m * m * sizeof(double), cudaMemcpyDeviceToDevice, st));
        }
        // M = Lz' Ls;  M V = U diag(lambda)
        CVXB_TRY(gemm_mm('T', 'N', m, Lz, Ls, M, st));
        CVXB_TRY(svd_jacobi(m, M, Vw, U, V, lam_s + lam_off, tn.p, ti.p, tc.p, st));
        if (!is_update) {
            // r = Ls V lambda^-1/2,  rti = Lz U lambda^-1/2                         (= misc.py:402-414)
            CVXB_TRY(gemm_mm('N', 'N', m, Ls, V, rk, st));
            CVXB_TRY(gemm_mm('N', 'N', m, Lz, U, rtk, st));
        } else {
            // r := r Ls V lambda^-1/2,  rti := rti Lz U lambda^-1/2                 (misc.py:595-630)
            CVXB_TRY(gemm_mm('N', 'N', m, rk, Ls, tmp, st));
            CVXB_TRY(gemm_mm('N', 'N', m, tmp, V, rk, st));
            CVXB_TRY(gemm_mm('N', 'N', m, rtk, Lz, tmp, st));
            CVXB_TRY(gemm_mm('N', 'N', m, tmp, U, rtk, st));
            // side effect of the reference: U is left in sk, V' in zk (:611-613)
            CVXB_CUDA(cudaMemcpyAsync(sk, U, (size_t)m * m * sizeof(double), cudaMemcpyDeviceToDevice, st));
            transpose_small_kernel<<<nb, T, 0, st>>>(m, V, zk);
            count_launch();
        }
        colscale_rsqrt_kernel<<<nb, T, 0, st>>>(m, rk, lam_s + lam_off);
        colscale_rsqrt_kernel<<<nb, T, 0, st>>>(m, rtk, lam_s + lam_off);
        count_launch(2);
        CVXB_LAUNCH_CHECK();
        lam_off += m;
    }
    CVXB_CUDA(cudaStreamSynchronize(st));
    return 0;
}

}  // namespace

bool cvxb::coop_launch_fits(const void *kernel, int threads, long long ctas) {
    static const bool allowed = [] { const char *e = getenv("CVXB_JACOBI_COOP"); return !(e && e[0] == '0'); }();
    int dev = 0, can = 0, per_sm = 0, sms = 0;
    return allowed && cudaGetDevice(&dev) == cudaSuccess &&
           cudaDeviceGetAttribute(&can, cudaDevAttrCooperativeLaunch, dev) == cudaSuccess && can &&
           cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess &&
           cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, 0) == cudaSuccess &&
           (long long)per_sm * sms >= ctas;
}

extern "C" {

// misc.compute_scaling(s, z, lmbda, dims, mnl)  (misc.py:250-419).  s, z: cdim; lmbda: mnl + ml + sum q + sum s;
// W: writable arrays of the sizes of cvxb_scaling.  Nothing but W and lmbda is written.
int cvxb_compute_scaling(const double *s, const double *z, double *lmbda, const cvxb_dims *dims,
                         const cvxb_scaling *Wout, int space) {
    if (!s || !z || !lmbda || !dims || !Wout) { set_error("compute_scaling: NULL argument"); return CVXB_E_ARG; }
    CallCtx ctx; CVXB_TRY(ctx.acquire(0));
    cudaStream_t st = ctx.st;
    ConeLayout c;
    CVXB_TRY(c.init(dims));
    const int nl = c.mnl + c.ml, nlam = nl + c.sumq;
    Staged S, Z, L, Dnl, Dnli, D, Di, V, Beta, R, Rti;
    CVXB_TRY(S.in(s, c.cdim, space, st));
    CVXB_TRY(Z.in(z, c.cdim, space, st));
    CVXB_TRY(L.in(lmbda, (size_t)nlam + c.sums, space, st, false));
    CVXB_TRY(Dnl.in(Wout->dnl, c.mnl, space, st, false));
    CVXB_TRY(Dnli.in(Wout->dnli, c.mnl, space, st, false));
    CVXB_TRY(D.in(Wout->d, c.ml, space, st, false));
    CVXB_TRY(Di.in(Wout->di, c.ml, space, st, false));
    CVXB_TRY(V.in(Wout->v, c.sumq, space, st, false));
    CVXB_TRY(Beta.in(Wout->beta, c.nq, space, st, false));
    CVXB_TRY(R.in(Wout->r, c.sums2, space, st, false));
    CVXB_TRY(Rti.in(Wout->rti, c.sums2, space, st, false));
    const int T = 256;
    if (c.mnl > 0) { nt_l_compute_kernel<<<(c.mnl + T - 1) / T, T, 0, st>>>(c.mnl, S.dev, Z.dev, Dnl.dev, Dnli.dev, L.dev); count_launch(); }
    if (c.ml > 0) {
        nt_l_compute_kernel<<<(c.ml + T - 1) / T, T, 0, st>>>(c.ml, S.dev + c.mnl, Z.dev + c.mnl, D.dev, Di.dev, L.dev + c.mnl);
        count_launch();
    }
    if (c.nq > 0) {
        nt_q_compute_kernel<<<c.nq, 128, 0, st>>>(c.d_q, c.d_qoff, c.d_voff, nl, S.dev + nl, Z.dev + nl, V.dev,
                                                   Beta.dev, L.dev);
        count_launch();
    }
    CVXB_LAUNCH_CHECK();
    if (c.ns > 0) {
        // private copies of the 's' blocks (the inputs are const)
        Scratch<double> cs, cz;
        CVXB_TRY(cs.alloc(c.sums2));
        CVXB_TRY(cz.alloc(c.sums2));
        const size_t so = (size_t)nl + c.sumq;
        CVXB_CUDA(cudaMemcpyAsync(cs.p, S.dev + so, (size_t)c.sums2 * sizeof(double), cudaMemcpyDeviceToDevice, st));
        CVXB_CUDA(cudaMemcpyAsync(cz.p, Z.dev + so, (size_t)c.sums2 * sizeof(double), cudaMemcpyDeviceToDevice, st));
        CVXB_TRY(nt_s_blocks(c, cs.p, cz.p, R.dev, Rti.dev, L.dev + nlam, false, st));
    }
    CVXB_TRY(L.out(st)); CVXB_TRY(Dnl.out(st)); CVXB_TRY(Dnli.out(st)); CVXB_TRY(D.out(st)); CVXB_TRY(Di.out(st));
    CVXB_TRY(V.out(st)); CVXB_TRY(Beta.out(st)); CVXB_TRY(R.out(st)); CVXB_TRY(Rti.out(st));
    CVXB_CUDA(cudaStreamSynchronize(st));
    return 0;
}

// misc.update_scaling(W, lmbda, s, z)  (misc.py:422-634): W and lmbda are updated in place; s, z are overwritten
// as in the reference (square roots of the 'l' rows, normalised 'q' blocks, U / V' in the 's' blocks).
int cvxb_update_scaling(const cvxb_scaling *W, double *lmbda, double *s, double *z, const cvxb_dims *dims,
                        int space) {
    if (!s || !z || !lmbda || !dims || !W) { set_error("update_scaling: NULL argument"); return CVXB_E_ARG; }
    CallCtx ctx; CVXB_TRY(ctx.acquire(0));
    cudaStream_t st = ctx.st;
    ConeLayout c;
    CVXB_TRY(c.init(dims));
    const int nl = c.mnl + c.ml, nlam = nl + c.sumq;
    Staged S, Z, L, Dnl, Dnli, D, Di, V, Beta, R, Rti;
    CVXB_TRY(S.in(s, c.cdim, space, st));
    CVXB_TRY(Z.in(z, c.cdim, space, st));
    CVXB_TRY(L.in(lmbda, (size_t)nlam + c.sums, space, st));
    CVXB_TRY(Dnl.in(W->dnl, c.mnl, space, st));
    CVXB_TRY(Dnli.in(W->dnli, c.mnl, space, st, false));
    CVXB_TRY(D.in(W->d, c.ml, space, st));
    CVXB_TRY(Di.in(W->di, c.ml, space, st, false));
    CVXB_TRY(V.in(W->v, c.sumq, space, st));
    CVXB_TRY(Beta.in(W->beta, c.nq, space, st));
    CVXB_TRY(R.in(W->r, c.sums2, space, st));
    CVXB_TRY(Rti.in(W->rti, c.sums2, space, st));
    const int T = 256;
    if (c.mnl > 0) { nt_l_update_kernel<<<(c.mnl + T - 1) / T, T, 0, st>>>(c.mnl, S.dev, Z.dev, Dnl.dev, Dnli.dev, L.dev); count_launch(); }
    if (c.ml > 0) {
        nt_l_update_kernel<<<(c.ml + T - 1) / T, T, 0, st>>>(c.ml, S.dev + c.mnl, Z.dev + c.mnl, D.dev, Di.dev, L.dev + c.mnl);
        count_launch();
    }
    if (c.nq > 0) {
        nt_q_update_kernel<<<c.nq, 128, 0, st>>>(c.d_q, c.d_qoff, c.d_voff, nl, S.dev + nl, Z.dev + nl, V.dev, Beta.dev,
                                                  L.dev);
        count_launch();
    }
    CVXB_LAUNCH_CHECK();
    if (c.ns > 0) {
        const size_t so = (size_t)nl + c.sumq;
        CVXB_TRY(nt_s_blocks(c, S.dev + so, Z.dev + so, R.dev, Rti.dev, L.dev + nlam, true, st));
    }
    CVXB_TRY(S.out(st)); CVXB_TRY(Z.out(st)); CVXB_TRY(L.out(st));
    CVXB_TRY(Dnl.out(st)); CVXB_TRY(Dnli.out(st)); CVXB_TRY(D.out(st)); CVXB_TRY(Di.out(st));
    CVXB_TRY(V.out(st)); CVXB_TRY(Beta.out(st)); CVXB_TRY(R.out(st)); CVXB_TRY(Rti.out(st));
    CVXB_CUDA(cudaStreamSynchronize(st));
    return 0;
}

}  // extern "C"
