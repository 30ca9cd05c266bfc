// misc.kkt_ldl2 on the device (reference src/python/misc.py:1128-1210): the 2 x 2 system
//
//        K = [ H + GG' W^-1 W^-T GG   A' ]       (order N = n + p, lower triangle stored)
//            [ A                      0  ]
//
// factored as  P K P' = L D L'  with Bunch-Kaufman (partial) pivoting, D block diagonal with 1 x 1 and 2 x 2
// blocks — what lapack.sytrf computes (src/C/lapack.c:2282; the unblocked algorithm of LAPACK's dsytf2, lower
// case) — and solved by the forward / diagonal / backward sweeps of lapack.sytrs (src/C/lapack.c:2531, dsytrs).
// K is symmetric INDEFINITE (p negative eigenvalues), so the pivot search with row/column interchanges is what
// keeps the factorisation stable when S is singular or badly scaled; the assembly of S is the same fused-scaling
// SYRK as the Cholesky route.
//
// Kernels per elimination step (the pivot decisions are taken on the device, the host loop is uniform):
//   ldl_pivot_kernel  (1 CTA)  finishes the previous step (multipliers into the pivot columns, k advances), then
//                              searches column k, and if needed row/column imax, and chooses kp and the block size
//   ldl_swap_kernel            symmetric interchange of rows/columns kk and kp of the trailing matrix
//   ldl_mult_kernel            multipliers of the 1x1 / 2x2 pivot block for every trailing row
//   ldl_update_kernel (2-D)    rank-1 / rank-2 update of the trailing lower triangle
// This is a completeness route (memory-bound rank-1/2 updates, ~4 launches per column); the hot path of the
// library is the Cholesky route.  `kktreg` (the reference's kkt_ldl option, misc.py:1096-1098) adds +kktreg to the
// first n diagonal entries and -kktreg to the last p.
#include "kkt_internal.cuh"
#include <cmath>

namespace cvxb {

namespace {

// K2 =[S 0; A 0] (lower), diagonal regularisation
__global__ void ldl_build_kernel(int n, int p, const double *S, long long lds, const double *A, long long lda,
                                 double *K2, long long ld, double reg) {
    const int N = n + p;
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (long long)N * N) return;
    const int i = (int)(e % N), j = (int)(e / N);
    double v = 0.0;
    if (i >= j) {
        if (i < n) v = S[i + (long long)j * lds];
        else if (j < n) v = A[(i - n) + (long long)j * lda];
        if (i == j) v += (i < n) ? reg : -reg;
    }
    K2[i + (long long)j * ld] = v;
}

struct MaxIdx { double v; int i; };
__device__ __forceinline__ MaxIdx cta_argmax(double v, int i, double *shv, int *shi) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double ov = __shfl_xor_sync(0xffffffffu, v, o);
        const int oi = __shfl_xor_sync(0xffffffffu, i, o);
        if (ov > v || (ov == v && oi < i)) { v = ov; i = oi; }
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    __syncthreads();
    if (lane == 0) { shv[warp] = v; shi[warp] = i; }
    __syncthreads();
    if (warp == 0) {
        v = (lane < (blockDim.x >> 5)) ? shv[lane] : -1.0;
        i = (lane < (blockDim.x >> 5)) ? shi[lane] : 0x7fffffff;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const double ov = __shfl_xor_sync(0xffffffffu, v, o);
            const int oi = __shfl_xor_sync(0xffffffffu, i, o);
            if (ov > v || (ov == v && oi < i)) { v = ov; i = oi; }
        }
        if (lane == 0) { shv[0] = v; shi[0] = i; }
    }
    __syncthreads();
    MaxIdx r; r.v = shv[0]; r.i = shi[0];
    __syncthreads();
    return r;
}

// finish the pending step, then choose the pivot of the new step
__global__ void __launch_bounds__(512) ldl_pivot_kernel(int N, double *A, long long ld, int *ipiv, int *state,
                                                         const double *w1, const double *w2) {
    __shared__ double shv[32];
    __shared__ int shi[32];
    int k = state[0];
    if (state[4]) {                                    // multipliers of the previous step -> its columns
        const int ks = state[1];
        for (int i = k + ks + threadIdx.x; i < N; i += blockDim.x) {
            A[i + (long long)k * ld] = w1[i];
            if (ks == 2) A[i + (long long)(k + 1) * ld] = w2[i];
        }
        __syncthreads();
        k += ks;
    }
    if (k >= N) {
        if (threadIdx.x == 0) { state[0] = k; state[4] = 0; }
        return;
    }
    const double alpha = (1.0 + sqrt(17.0)) / 8.0;
    const double absakk = fabs(A[k + (long long)k * ld]);
    double v = -1.0; int vi = 0x7fffffff;
    for (int i = k + 1 + threadIdx.x; i < N; i += blockDim.x) {
        const double a = fabs(A[i + (long long)k * ld]);
        if (a > v) { v = a; vi = i; }
    }
    MaxIdx cm = cta_argmax(v, vi, shv, shi);
    const double colmax = (k + 1 < N) ? cm.v : 0.0;
    const int imax = cm.i;
    int kp = k, kstep = 1, info = 0;
    if (!(fmax(absakk, colmax) > 0.0)) {
        info = k + 1;                                  // exactly zero (or NaN) column: singular D
    } else if (absakk >= alpha * colmax) {
        kp = k;
    } else {
        // rowmax = largest off-diagonal entry of row / column imax of the trailing matrix
        double r = -1.0; int ri = 0;
        for (int j = k + threadIdx.x; j < imax; j += blockDim.x) r = fmax(r, fabs(A[imax + (long long)j * ld]));
        for (int i = imax + 1 + threadIdx.x; i < N; i += blockDim.x) r = fmax(r, fabs(A[i + (long long)imax * ld]));
        const double rowmax = cta_argmax(r, ri, shv, shi).v;
        if (absakk >= alpha * colmax * (colmax / rowmax)) kp = k;
        else if (fabs(A[imax + (long long)imax * ld]) >= alpha * rowmax) kp = imax;
        else { kp = imax; kstep = 2; }
    }
    if (threadIdx.x == 0) {
        state[0] = k; state[1] = kstep; state[2] = kp; state[4] = info ? 0 : 1;
        if (info && state[3] == 0) state[3] = info;
        if (kstep == 1) ipiv[k] = kp + 1;
        else { ipiv[k] = -(kp + 1); ipiv[k + 1] = -(kp + 1); }
        if (info) state[0] = k + 1;                    // skip the column (as dsytf2 does), nothing to eliminate
    }
}

// interchange rows and columns kk = k + kstep - 1 and kp in the trailing matrix A[k:, k:] (lower storage)
__global__ void ldl_swap_kernel(int N, double *A, long long ld, const int *state) {
    if (!state[4]) return;
    const int k = state[0], kstep = state[1], kp = state[2];
    const int kk = k + kstep - 1;
    if (kp == kk) return;
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    // rows below kp: columns kk and kp
    for (int i = kp + 1 + t; i < N; i += gridDim.x * blockDim.x) {
        const double a = A[i + (long long)kk * ld], b = A[i + (long long)kp * ld];
        A[i + (long long)kk * ld] = b; A[i + (long long)kp * ld] = a;
    }
    // between: A[kk+1 .. kp-1, kk]  <->  A[kp, kk+1 .. kp-1]
    for (int j = kk + 1 + t; j < kp; j += gridDim.x * blockDim.x) {
        const double a = A[j + (long long)kk * ld], b = A[kp + (long long)j * ld];
        A[j + (long long)kk * ld] = b; A[kp + (long long)j * ld] = a;
    }
    if (t == 0) {
        const double a = A[kk + (long long)kk * ld], b = A[kp + (long long)kp * ld];
        A[kk + (long long)kk * ld] = b; A[kp + (long long)kp * ld] = a;
        if (kstep == 2) {
            const double c = A[k + 1 + (long long)k * ld], d = A[kp + (long long)k * ld];
            A[k + 1 + (long long)k * ld] = d; A[kp + (long long)k * ld] = c;
        }
    }
}

// multipliers: 1x1  w1[i] = A[i,k] / A[k,k];   2x2 (dsytf2's formulas)  w1, w2 for the rows i >= k+2
__global__ void ldl_mult_kernel(int N, const double *A, long long ld, const int *state, double *w1, double *w2) {
    if (!state[4]) return;
    const int k = state[0], kstep = state[1];
    const int i = k + kstep + blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    if (kstep == 1) {
        const double r1 = 1.0 / A[k + (long long)k * ld];
        w1[i] = A[i + (long long)k * ld] * r1;
    } else {
        double d21 = A[k + 1 + (long long)k * ld];
        const double d11 = A[k + 1 + (long long)(k + 1) * ld] / d21;
        const double d22 = A[k + (long long)k * ld] / d21;
        const double tt = 1.0 / (d11 * d22 - 1.0);
        d21 = tt / d21;
        const double a = A[i + (long long)k * ld], b = A[i + (long long)(k + 1) * ld];
        w1[i] = d21 * (d11 * a - b);
        w2[i] = d21 * (d22 * b - a);
    }
}

// trailing update of the lower triangle: A[i,j] -= A[i,k] w1[j] (+ A[i,k+1] w2[j]),  i >= j >= k + kstep
__global__ void __launch_bounds__(256) ldl_update_kernel(int N, double *A, long long ld, const int *state,
                                                          const double *w1, const double *w2) {
    if (!state[4]) return;
    const int k = state[0], kstep = state[1];
    const int j0 = k + kstep;
    const int j = j0 + blockIdx.y * 8 + (threadIdx.x >> 5);          // 8 columns per CTA row, one warp each
    if (j >= N) return;
    const double wj1 = w1[j], wj2 = (kstep == 2) ? w2[j] : 0.0;
    const double *c1 = A + (long long)k * ld, *c2 = A + (long long)(k + 1) * ld;
    double *cj = A + (long long)j * ld;
    for (int i = j0 + blockIdx.x * 32 * 8 + (threadIdx.x & 31); i < N; i += gridDim.x * 32 * 8) {
#pragma unroll
        for (int u = 0; u < 8; ++u) {
            const int ii = i + u * 32;
            if (ii < N && ii >= j) {
                double v = cj[ii] - c1[ii] * wj1;
                if (kstep == 2) v -= c2[ii] * wj2;
                cj[ii] = v;
            }
        }
    }
}

// b := K^{-1} b from the factorisation (dsytrs, lower); one CTA
__global__ void __launch_bounds__(1024) ldl_solve_kernel(int N, const double *A, long long ld, const int *ipiv, double *b) {
    __shared__ double sh[32];
    __shared__ double bk0, bk1;
    // ---- L D y = b
    int k = 0;
    while (k < N) {
        if (ipiv[k] > 0) {
            const int kp = ipiv[k] - 1;
            if (threadIdx.x == 0) {
                if (kp != k) { const double t = b[k]; b[k] = b[kp]; b[kp] = t; }
                bk0 = b[k];
            }
            __syncthreads();
            const double m = bk0;
            for (int i = k + 1 + threadIdx.x; i < N; i += blockDim.x) b[i] -= A[i + (long long)k * ld] * m;
            if (threadIdx.x == 0) b[k] = m / A[k + (long long)k * ld];
            __syncthreads();
            k += 1;
        } else {
            const int kp = -ipiv[k] - 1;
            if (threadIdx.x == 0) {
                if (kp != k + 1) { const double t = b[k + 1]; b[k + 1] = b[kp]; b[kp] = t; }
                bk0 = b[k]; bk1 = b[k + 1];
            }
            __syncthreads();
            const double m0 = bk0, m1 = bk1;
            for (int i = k + 2 + threadIdx.x; i < N; i += blockDim.x)
                b[i] -= A[i + (long long)k * ld] * m0 + A[i + (long long)(k + 1) * ld] * m1;
            if (threadIdx.x == 0) {
                const double akm1k = A[k + 1 + (long long)k * ld];
                const double akm1 = A[k + (long long)k * ld] / akm1k, ak = A[k + 1 + (long long)(k + 1) * ld] / akm1k;
                const double denom = akm1 * ak - 1.0;
                const double bkm1 = m0 / akm1k, bk = m1 / akm1k;
                b[k] = (ak * bkm1 - bk) / denom;
                b[k + 1] = (akm1 * bk - bkm1) / denom;
            }
            __syncthreads();
            k += 2;
        }
    }
    // ---- L' x = y
    k = N - 1;
    while (k >= 0) {
        const int two = ipiv[k] < 0;
        double t0 = 0.0, t1 = 0.0;
        for (int i = k + 1 + threadIdx.x; i < N; i += blockDim.x) {
            const double bi = b[i];
            t0 += A[i + (long long)k * ld] * bi;
            if (two) t1 += A[i + (long long)(k - 1) * ld] * bi;
        }
        // CTA reductions
        t0 = warp_sum(t0); t1 = warp_sum(t1);
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        __syncthreads();
        if (lane == 0) sh[warp] = t0;
        __syncthreads();
        double s0 = (threadIdx.x < (blockDim.x >> 5)) ? sh[threadIdx.x] : 0.0;
        if (warp == 0) s0 = warp_sum(s0);
        __syncthreads();
        if (lane == 0) sh[warp] = t1;
        __syncthreads();
        double s1 = (threadIdx.x < (blockDim.x >> 5)) ? sh[threadIdx.x] : 0.0;
        if (warp == 0) s1 = warp_sum(s1);
        if (threadIdx.x == 0) {
            b[k] -= s0;
            if (two) b[k - 1] -= s1;
            const int kp = (two ? -ipiv[k] : ipiv[k]) - 1;
            if (kp != k) { const double t = b[k]; b[k] = b[kp]; b[kp] = t; }
        }
        __syncthreads();
        k -= two ? 2 : 1;
    }
}

}  // namespace

int kkt_ldl_setup(cvxb_kkt *k, double kktreg) {
    auto s = std::make_unique<LdlState>();
    s->N = k->n + k->p;
    s->kktreg = kktreg;
    s->ld = (s->N + 1) & ~1;
    if (s->ld < 2) s->ld = 2;
    const size_t NN = (size_t)(s->N > 0 ? s->N : 1);
    CVXB_TRY(s->K2.alloc((size_t)s->ld * NN));
    CVXB_TRY(s->ipiv.alloc(NN));
    CVXB_TRY(s->state.alloc(8));
    CVXB_TRY(s->w1.alloc(NN));
    CVXB_TRY(s->w2.alloc(NN));
    CVXB_TRY(s->u.alloc(NN));
    k->ldl = std::move(s);
    return 0;
}

int kkt_ldl_factor(cvxb_kkt *k) {
    const LdlState *s = k->ldl.get();
    const int n = k->n, p = k->p, N = s->N;
    cudaStream_t st = k->st;
    const long long ldk = kkt_ldk(k);
    double *K2 = s->K2.p, *w1 = s->w1.p, *w2 = s->w2.p;
    int *ipiv = s->ipiv.p, *state = s->state.p;
    ldl_build_kernel<<<(unsigned)(((long long)N * N + 255) / 256), 256, 0, st>>>(n, p, k->Kmat.p, ldk, k->Aeq.p,
                                                                               k->lda_eq, K2, s->ld, s->kktreg);
    count_launch();
    CVXB_CUDA(cudaMemsetAsync(state, 0, 8 * sizeof(int), st));
    for (int it = 0; it < N; ++it) {
        // after `it` completed steps k >= it: the trailing matrix has at most N - it - 1 rows beyond the pivot
        const int rem = N - it - 1;
        ldl_pivot_kernel<<<1, 512, 0, st>>>(N, K2, s->ld, ipiv, state, w1, w2);
        count_launch();
        if (rem <= 0) continue;
        int sb = (rem + 255) / 256; if (sb > 64) sb = 64;
        ldl_swap_kernel<<<sb, 256, 0, st>>>(N, K2, s->ld, state);
        ldl_mult_kernel<<<(rem + 255) / 256, 256, 0, st>>>(N, K2, s->ld, state, w1, w2);
        int gx = (rem + 255) / 256; if (gx > 32) gx = 32;
        dim3 grid(gx, (rem + 7) / 8);
        ldl_update_kernel<<<grid, 256, 0, st>>>(N, K2, s->ld, state, w1, w2);
        count_launch(3);
    }
    ldl_pivot_kernel<<<1, 512, 0, st>>>(N, K2, s->ld, ipiv, state, w1, w2);     // finish the last step
    count_launch();
    CVXB_LAUNCH_CHECK();
    // dsytrf's info > 0: D(info, info) is exactly zero -> the reference raises ArithmeticError
    CVXB_CUDA(cudaMemcpyAsync(k->cw.d_info.p, state + 3, sizeof(int), cudaMemcpyDeviceToDevice, st));
    return 0;
}

int kkt_ldl_solve(cvxb_kkt *k, double *xd, double *yd) {
    const LdlState *s = k->ldl.get();
    const int n = k->n, p = k->p, N = s->N;
    cudaStream_t st = k->st;
    double *u = s->u.p;
    CVXB_CUDA(cudaMemcpyAsync(u, xd, (size_t)n * sizeof(double), cudaMemcpyDeviceToDevice, st));
    CVXB_CUDA(cudaMemcpyAsync(u + n, yd, (size_t)p * sizeof(double), cudaMemcpyDeviceToDevice, st));
    ldl_solve_kernel<<<1, 1024, 0, st>>>(N, s->K2.p, s->ld, s->ipiv.p, u);
    count_launch();
    CVXB_LAUNCH_CHECK();
    CVXB_CUDA(cudaMemcpyAsync(xd, u, (size_t)n * sizeof(double), cudaMemcpyDeviceToDevice, st));
    CVXB_CUDA(cudaMemcpyAsync(yd, u + n, (size_t)p * sizeof(double), cudaMemcpyDeviceToDevice, st));
    return 0;
}

}  // namespace cvxb
