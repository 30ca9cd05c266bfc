// The O(cdim) cone algebra of the IPM side, mirror of src/C/misc_solvers.c:
//   scale2 (:256-401), sprod (:634-767), sinv (:775-878), trisc (:887-935), triusc (:940-986),
//   sdot (:991-1039), max_step (:1052-1153).
// One CTA walks the whole cone vector; reductions inside a 'q' cone / for sdot are block-wide.
// The 's' part of max_step (reference: dsyevr_ for the smallest eigenvalue, dsyevd_ when sigma is
// given, :1099-1150) is a parallel-order cyclic Jacobi eigensolver: every round applies N/2 disjoint
// plane rotations at once, one thread per 2x2 block of J'AJ, ping-ponging between two copies so a
// round is a single race-free pass.
#include "cone.cuh"
#include <cooperative_groups.h>
#include <vector>
#include <algorithm>
#include <cfloat>

using namespace cvxb;

namespace {

struct Cones {
    int nl;                     // mnl + ml
    int nq; const int *q;       // device arrays
    int ns; const int *s;
};

// x := H(lambda^{1/2}) x  or its inverse
__global__ void scale2_kernel(const double *lm, double *x, Cones c, int inverse) {
    __shared__ double sh[32];
    const int tid = threadIdx.x, nt = blockDim.x;
    for (int i = tid; i < c.nl; i += nt) x[i] = inverse ? x[i] * lm[i] : x[i] / lm[i];
    int m = c.nl;
    for (int k = 0; k < c.nq; ++k) {
        q_scale2(CtaTeam{tid, nt, sh}, lm + m, x + m, c.q[k], inverse);
        m += c.q[k];
        __syncthreads();
    }
    int ind2 = m;
    for (int k = 0; k < c.ns; ++k) {
        const int mk = c.s[k];
        for (int e = tid; e < mk * mk; e += nt) {
            const int i = e % mk, j = e / mk;
            const double cc = sqrt(lm[ind2 + i]) * sqrt(lm[ind2 + j]);
            x[m + e] = inverse ? x[m + e] * cc : x[m + e] / cc;
        }
        m += mk * mk; ind2 += mk;
    }
}

// x := y o x for the l / q blocks and the 's' blocks with diagonal y (diag == 'D')
__global__ void sprod_kernel(double *x, const double *y, Cones c, int diag_d) {
    __shared__ double sh[32];
    const int tid = threadIdx.x, nt = blockDim.x;
    for (int i = tid; i < c.nl; i += nt) x[i] *= y[i];
    int m = c.nl;
    for (int k = 0; k < c.nq; ++k) {
        q_sprod(CtaTeam{tid, nt, sh}, y + m, x + m, x + m, c.q[k]);
        m += c.q[k];
        __syncthreads();
    }
    if (!diag_d) return;
    int ind2 = m;
    for (int k = 0; k < c.ns; ++k) {
        const int mk = c.s[k];
        for (int e = tid; e < mk * mk; e += nt) {
            const int i = e % mk, j = e / mk;
            if (i >= j) x[m + e] *= 0.5 * (y[ind2 + i] + y[ind2 + j]);
        }
        m += mk * mk; ind2 += mk;
    }
}
// 's' blocks, full y: x_lower := 0.5 (T + T')  with T = sym(x) sym(y)
__global__ void sprod_s_finish_kernel(double *x, const double *T, int mk) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= mk * mk) return;
    const int i = e % mk, j = e / mk;
    if (i >= j) x[e] = 0.5 * (T[i + (long long)j * mk] + T[j + (long long)i * mk]);
}

__global__ void sinv_kernel(double *x, const double *y, Cones c) {
    __shared__ double sh[32];
    const int tid = threadIdx.x, nt = blockDim.x;
    for (int i = tid; i < c.nl; i += nt) x[i] /= y[i];
    int m = c.nl;
    for (int k = 0; k < c.nq; ++k) {
        q_sinv(CtaTeam{tid, nt, sh}, y + m, x + m, c.q[k]);
        m += c.q[k];
        __syncthreads();
    }
    int ind2 = m;
    for (int k = 0; k < c.ns; ++k) {
        const int mk = c.s[k];
        for (int e = tid; e < mk * mk; e += nt) {
            const int i = e % mk, j = e / mk;
            if (i >= j) x[m + e] /= 0.5 * (y[ind2 + i] + y[ind2 + j]);
        }
        m += mk * mk; ind2 += mk;
    }
}

// mode 0: trisc (upper := 0, strict lower *= 2); mode 1: triusc (strict lower *= 0.5)
__global__ void trisc_kernel(double *x, Cones c, int off, int mode) {
    int m = off;
    for (int k = 0; k < c.ns; ++k) {
        const int mk = c.s[k];
        for (int e = threadIdx.x; e < mk * mk; e += blockDim.x) {
            const int i = e % mk, j = e / mk;
            if (mode == 0) { if (i < j) x[m + e] = 0.0; else if (i > j) x[m + e] *= 2.0; }
            else if (i > j) x[m + e] *= 0.5;
        }
        m += mk * mk;
    }
}

__global__ void sdot_kernel(const double *x, const double *y, Cones c, int nlq, double *out) {
    __shared__ double sh[32];
    const int tid = threadIdx.x, nt = blockDim.x;
    double a = 0;
    for (int i = tid; i < nlq; i += nt) a += x[i] * y[i];
    int m = nlq;
    for (int k = 0; k < c.ns; ++k) {
        const int mk = c.s[k];
        for (int e = tid; e < mk * mk; e += nt) {
            const int i = e % mk, j = e / mk;
            if (i == j) a += x[m + e] * y[m + e];
            else if (i > j) a += 2.0 * x[m + e] * y[m + e];
        }
        m += mk * mk;
    }
    a = block_sum(a, sh);
    if (tid == 0) *out = a;
}

__global__ void max_step_kernel(const double *x, Cones c, double *out) {
    __shared__ double sh[32];
    const int tid = threadIdx.x, nt = blockDim.x;
    double t = -FLT_MAX;
    for (int i = tid; i < c.nl; i += nt) t = fmax(t, -x[i]);
    // block max through the sum helper's scratch: do a max-reduction by hand
    for (int o = 16; o > 0; o >>= 1) t = fmax(t, __shfl_xor_sync(0xffffffffu, t, o));
    __syncthreads();
    if ((tid & 31) == 0) sh[tid >> 5] = t;
    __syncthreads();
    t = -FLT_MAX;
    for (int w = 0; w < (nt >> 5); ++w) t = fmax(t, sh[w]);
    __syncthreads();
    int m = c.nl;
    for (int k = 0; k < c.nq; ++k) {
        t = fmax(t, q_max_step(CtaTeam{tid, nt, sh}, x + m, c.q[k]));
        m += c.q[k];
        __syncthreads();
    }
    if (tid == 0) *out = (m > 0) ? t : 0.0;
}


// The symmetric eigensolver for the 's' blocks (parallel-order cyclic Jacobi) is cone.cuh's jac_block / jac_eig_cta.

struct JacArgs {
    const double *x;        // first 's' row of the cone vector (lower triangles significant)
    double *w0, *w1, *V;    // three work copies, each sum(mk^2), same block offsets as x
    const int *s, *soff, *sigoff;
    double *sigma;          // sum(mk): eigenvalues, ascending inside each block
    double *xout;           // eigenvectors -> 's' blocks of x (nullptr: eigenvalues only)
    double *stats;          // 2 per block: off-diagonal and total squared Frobenius norms
    int *perm;              // sum(mk): rank of each unsorted eigenvalue
    int N;                  // padded (even) order shared by all blocks of the launch
};

__global__ void jac_init_kernel(JacArgs a) {
    const int k = blockIdx.y, mk = a.s[k];
    const size_t o = a.soff[k];
    for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < (size_t)mk * mk; e += (size_t)gridDim.x * blockDim.x) {
        const int i = (int)(e % mk), j = (int)(e / mk);
        a.w0[o + e] = (i >= j) ? a.x[o + e] : a.x[o + j + (size_t)i * mk];
        if (a.V) a.V[o + e] = (i == j) ? 1.0 : 0.0;
    }
}

template <bool WITH_V>
__global__ void jac_round_kernel(JacArgs a, int r, int flip) {
    const int k = blockIdx.z, mk = a.s[k];
    // I (the row pair) is the fast thread index: consecutive I are consecutive rows of the column-major blocks
    const int I = blockIdx.x * blockDim.x + threadIdx.x, J = blockIdx.y * blockDim.y + threadIdx.y;
    if (I >= a.N / 2 || J >= a.N / 2) return;
    const size_t o = a.soff[k];
    jac_block<WITH_V>((flip ? a.w1 : a.w0) + o, (flip ? a.w0 : a.w1) + o, a.V + (WITH_V ? o : 0), mk, a.N, r, I, J);
}

// A whole sweep (N - 1 rounds) in one cooperative launch, a grid barrier between rounds; the buffers swap every round,
// so the result of the sweep is in the buffer the sweep did NOT start from (N - 1 is odd).
template <bool WITH_V>
__global__ void __launch_bounds__(256) jac_sweep_kernel(JacArgs a, int flip) {
    namespace cg = cooperative_groups;
    cg::grid_group grid = cg::this_grid();
    const int k = blockIdx.z, mk = a.s[k];
    const int I = blockIdx.x * blockDim.x + threadIdx.x, J = blockIdx.y * blockDim.y + threadIdx.y;
    const bool live = I < a.N / 2 && J < a.N / 2;
    const size_t o = a.soff[k];
    for (int r = 0; r < a.N - 1; ++r) {
        if (live)
            jac_block<WITH_V>((flip ? a.w1 : a.w0) + o, (flip ? a.w0 : a.w1) + o, a.V + (WITH_V ? o : 0), mk, a.N, r, I, J);
        grid.sync();
        flip ^= 1;
    }
}

__global__ void jac_off_kernel(JacArgs a, int flip) {
    __shared__ double sh[32];
    const int k = blockIdx.x, mk = a.s[k];
    const double *S = (flip ? a.w1 : a.w0) + a.soff[k];
    double off = 0, tot = 0;
    for (size_t e = threadIdx.x; e < (size_t)mk * mk; e += blockDim.x) {
        const double v = S[e] * S[e];
        tot += v;
        if (e % mk != e / mk) off += v;
    }
    off = block_sum(off, sh); tot = block_sum(tot, sh);
    if (threadIdx.x == 0) { a.stats[2 * k] = off; a.stats[2 * k + 1] = tot; }
}

// eigenvalues = diagonal; rank them (stable), write sigma ascending
__global__ void jac_sort_kernel(JacArgs a, int flip) {
    const int k = blockIdx.x, mk = a.s[k];
    const double *S = (flip ? a.w1 : a.w0) + a.soff[k];
    for (int i = threadIdx.x; i < mk; i += blockDim.x) {
        const double di = S[i + (size_t)i * mk];
        int rank = 0;
        for (int j = 0; j < mk; ++j) {
            const double dj = S[j + (size_t)j * mk];
            rank += (dj < di) || (dj == di && j < i);
        }
        a.sigma[a.sigoff[k] + rank] = di;
        a.perm[a.sigoff[k] + i] = rank;
    }
}

__global__ void jac_vec_kernel(JacArgs a) {
    const int k = blockIdx.y, mk = a.s[k];
    const size_t o = a.soff[k];
    for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < (size_t)mk * mk; e += (size_t)gridDim.x * blockDim.x) {
        const int i = (int)(e % mk), j = (int)(e / mk);
        a.xout[o + i + (size_t)a.perm[a.sigoff[k] + j] * mk] = a.V[o + e];
    }
}


// All blocks of order <= 64: one CTA per block runs every sweep itself (block-level barriers only).
template <bool WITH_V>
__global__ void __launch_bounds__(1024) jac_small_kernel(JacArgs a, int max_sweeps, int *fail) {
    __shared__ double sh[32];
    const int k = blockIdx.x, mk = a.s[k];
    if (mk == 0) return;
    const size_t o = a.soff[k];
    double *w0 = a.w0 + o, *w1 = a.w1 + o, *V = WITH_V ? a.V + o : nullptr;
    const int tid = threadIdx.x, nt = blockDim.x;
    for (int e = tid; e < mk * mk; e += nt) {
        const int i = e % mk, j = e / mk;
        w0[e] = (i >= j) ? a.x[o + e] : a.x[o + j + (size_t)i * mk];
        if (WITH_V) V[e] = (i == j) ? 1.0 : 0.0;
    }
    __syncthreads();
    const bool ok = jac_eig_cta<WITH_V>(w0, w1, V, mk, max_sweeps, sh, tid, nt);
    if (!ok && tid == 0) atomicExch(fail, 1);
    for (int i = tid; i < mk; i += nt) {
        const double di = w0[i + (size_t)i * mk];
        int rank = 0;
        for (int j = 0; j < mk; ++j) {
            const double dj = w0[j + (size_t)j * mk];
            rank += (dj < di) || (dj == di && j < i);
        }
        a.sigma[a.sigoff[k] + rank] = di;
        if (WITH_V) a.perm[a.sigoff[k] + i] = rank;
    }
    if (WITH_V) {
        __syncthreads();
        for (int e = tid; e < mk * mk; e += nt) {
            const int i = e % mk, j = e / mk;
            a.xout[o + i + (size_t)a.perm[a.sigoff[k] + j] * mk] = V[e];
        }
    }
}

// t := max(t, -lambda_min) over the 's' blocks (sigma ascending per block)
__global__ void max_step_s_kernel(double *out, const double *sigma, const int *s, const int *sigoff,
                                  int ns, int any_lq) {
    double t = any_lq ? *out : -FLT_MAX;
    for (int k = 0; k < ns; ++k) if (s[k] > 0) t = fmax(t, -sigma[sigoff[k]]);
    *out = t;
}

Cones cones_of(const ConeLayout &c) { return Cones{c.mnl + c.ml, c.nq, c.d_q, c.ns, c.d_s}; }

}  // namespace

extern "C" {

int cvxb_scale2(const double *lmbda, double *x, const cvxb_dims *dims, int inverse, int space) {
    CallCtx ctx; CVXB_TRY(ctx.acquire(0));
    cudaStream_t st = ctx.st;
    ConeLayout c; CVXB_TRY(c.init(dims));
    Staged l, xb;
    CVXB_TRY(l.in(lmbda, (size_t)c.mnl + c.ml + c.sumq + c.sums, space, st));
    CVXB_TRY(xb.in(x, c.cdim, space, st));
    scale2_kernel<<<1, 256, 0, st>>>(l.dev, xb.dev, cones_of(c), inverse == 'I');
    count_launch(); CVXB_LAUNCH_CHECK();
    CVXB_TRY(xb.out(st));
    CVXB_CUDA(cudaStreamSynchronize(st));
    return 0;
}

int cvxb_sprod(double *x, const double *y, const cvxb_dims *dims, int diag, int space) {
    CallCtx ctx; CVXB_TRY(ctx.acquire(0));
    cudaStream_t st = ctx.st;
    ConeLayout c; CVXB_TRY(c.init(dims));
    const bool dd = (diag == 'D');
    size_t ny = dd ? (size_t)c.mnl + c.ml + c.sumq + c.sums : (size_t)c.cdim;
    Staged xb, yb;
    CVXB_TRY(xb.in(x, c.cdim, space, st));
    CVXB_TRY(yb.in(y, ny, space, st));
    sprod_kernel<<<1, 256, 0, st>>>(xb.dev, yb.dev, cones_of(c), dd ? 1 : 0);
    count_launch(); CVXB_LAUNCH_CHECK();
    if (!dd && c.ns > 0) {
        // 0.5 (A Y + Y A) with A = sym(x_k), Y = sym(y_k): T = A Y on the DMMA GEMM
        const int nlq = c.mnl + c.ml + c.sumq;
        for (int k = 0; k < c.ns; ++k) {
            const int mk = c.s[k];
            if (mk == 0) continue;
            const long long m2 = (long long)mk * mk;
            Scratch<double> tmp;
            CVXB_TRY(tmp.alloc(3 * m2));
            double *As = tmp.p, *Ys = tmp.p + m2, *T = tmp.p + 2 * m2;
            CVXB_CUDA(cudaMemcpyAsync(As, xb.dev + nlq + c.s_off[k], m2 * sizeof(double), cudaMemcpyDeviceToDevice, st));
            CVXB_CUDA(cudaMemcpyAsync(Ys, yb.dev + nlq + c.s_off[k], m2 * sizeof(double), cudaMemcpyDeviceToDevice, st));
            CVXB_TRY(symmetrize_lower(mk, As, mk, 1, 0, st));
            CVXB_TRY(symmetrize_lower(mk, Ys, mk, 1, 0, st));
            GemmDesc g;
            g.M = mk; g.N = mk; g.K = mk;
            g.X = As; g.ldx = mk; g.x_kmajor = false;
            g.Y = Ys; g.ldy = mk; g.y_kmajor = true;       // Y[c,k] = Ys[k, c]
            g.C = T; g.ldc = mk;
            CVXB_TRY(dmma_gemm(g, st));
            sprod_s_finish_kernel<<<(int)((m2 + 255) / 256), 256, 0, st>>>(xb.dev + nlq + c.s_off[k], T, mk);
            count_launch();
            CVXB_CUDA(cudaStreamSynchronize(st));    // before tmp is freed
        }
    }
    CVXB_TRY(xb.out(st));
    CVXB_CUDA(cudaStreamSynchronize(st));
    return 0;
}

int cvxb_sinv(double *x, const double *y, const cvxb_dims *dims, int space) {
    CallCtx ctx; CVXB_TRY(ctx.acquire(0));
    cudaStream_t st = ctx.st;
    ConeLayout c; CVXB_TRY(c.init(dims));
    Staged xb, yb;
    CVXB_TRY(xb.in(x, c.cdim, space, st));
    CVXB_TRY(yb.in(y, (size_t)c.mnl + c.ml + c.sumq + c.sums, space, st));
    sinv_kernel<<<1, 256, 0, st>>>(xb.dev, yb.dev, cones_of(c));
    count_launch(); CVXB_LAUNCH_CHECK();
    CVXB_TRY(xb.out(st));
    CVXB_CUDA(cudaStreamSynchronize(st));
    return 0;
}

static int trisc_common(double *x, const cvxb_dims *dims, int space, int mode) {
    CallCtx ctx; CVXB_TRY(ctx.acquire(0));
    cudaStream_t st = ctx.st;
    ConeLayout c; CVXB_TRY(c.init(dims));
    Staged xb;
    CVXB_TRY(xb.in(x, c.cdim, space, st));
    trisc_kernel<<<1, 256, 0, st>>>(xb.dev, cones_of(c), c.mnl + c.ml + c.sumq, mode);
    count_launch(); CVXB_LAUNCH_CHECK();
    CVXB_TRY(xb.out(st));
    CVXB_CUDA(cudaStreamSynchronize(st));
    return 0;
}
int cvxb_trisc(double *x, const cvxb_dims *dims, int space) { return trisc_common(x, dims, space, 0); }
int cvxb_triusc(double *x, const cvxb_dims *dims, int space) { return trisc_common(x, dims, space, 1); }

int cvxb_sdot(const double *x, const double *y, const cvxb_dims *dims, double *result, int space) {
    if (!result) { set_error("sdot: result is NULL"); return CVXB_E_ARG; }
    CallCtx ctx; CVXB_TRY(ctx.acquire(0));
    cudaStream_t st = ctx.st;
    ConeLayout c; CVXB_TRY(c.init(dims));
    Staged xb, yb;
    CVXB_TRY(xb.in(x, c.cdim, space, st));
    CVXB_TRY(yb.in(y, c.cdim, space, st));
    Scratch<double> d;
    CVXB_TRY(d.alloc(1));
    sdot_kernel<<<1, 256, 0, st>>>(xb.dev, yb.dev, cones_of(c), c.mnl + c.ml + c.sumq, d.p);
    count_launch();
    cudaError_t e = cudaMemcpyAsync(result, d.p, sizeof(double), cudaMemcpyDeviceToHost, st);
    cudaStreamSynchronize(st);
    if (e != cudaSuccess) { set_error("sdot: %s", cudaGetErrorString(e)); return CVXB_E_CUDA; }
    return 0;
}

// Eigen-decomposition of every 's' block of the device cone vector xs (first 's' row).
// sigma_dev: sum(mk) eigenvalues (ascending per block); with_vectors: the blocks of xs are
// overwritten by the eigenvectors (columns ordered like sigma), as dsyevd_ 'V' does in the reference.
static int sym_eig_blocks(const ConeLayout &c, double *xs, double *sigma_dev, const int *d_sigoff,
                          bool with_vectors, cudaStream_t st) {
    const int MAX_SWEEPS = 40;
    if (c.maxs == 0) return 0;
    const size_t m2 = (size_t)c.sums2;
    std::vector<double> hstats(2 * (size_t)c.ns), prev(c.ns, 1e300);
    Scratch<double> work, stats;
    Scratch<int> perm, fail;
    if (work.alloc((with_vectors ? 3 : 2) * m2) || stats.alloc(2 * (size_t)c.ns) || perm.alloc(c.sums) ||
        fail.alloc(1)) {
        cudaGetLastError();
        set_error("max_step: out of device memory for the eigensolver workspace");
        return CVXB_E_NOMEM;
    }
    JacArgs a;
    a.x = xs; a.w0 = work.p; a.w1 = work.p + m2; a.V = with_vectors ? work.p + 2 * m2 : nullptr;
    a.s = c.d_s; a.soff = c.d_soff; a.sigoff = d_sigoff;
    a.sigma = sigma_dev; a.xout = with_vectors ? xs : nullptr; a.stats = stats.p; a.perm = perm.p;
    a.N = std::max(2, c.maxs + (c.maxs & 1));
    const int h = a.N / 2;
    if (c.maxs <= 64) {
        CVXB_CUDA(cudaMemsetAsync(fail.p, 0, sizeof(int), st));
        const int nt = std::max(32, (h * h + 31) / 32 * 32);
        if (with_vectors) jac_small_kernel<true><<<c.ns, nt, 0, st>>>(a, MAX_SWEEPS, fail.p);
        else jac_small_kernel<false><<<c.ns, nt, 0, st>>>(a, MAX_SWEEPS, fail.p);
        count_launch();
        int hfail = 0;
        cudaError_t e = cudaMemcpyAsync(&hfail, fail.p, sizeof(int), cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) { set_error("max_step: %s", cudaGetErrorString(e)); return CVXB_E_CUDA; }
        if (hfail) { set_error("max_step: Jacobi eigensolver did not converge (non-finite input?)"); return 1; }
        return 0;
    }
    {
        const int gx = (int)std::min<size_t>(((size_t)c.maxs * c.maxs + 255) / 256, 1184);
        jac_init_kernel<<<dim3(gx, c.ns), 256, 0, st>>>(a);
        count_launch();
    }
    int flip = 0;
    bool ok = false;
    const void *sweep_fn = with_vectors ? (const void *)jac_sweep_kernel<true> : (const void *)jac_sweep_kernel<false>;
    const dim3 blk(16, 16), grd((h + 15) / 16, (h + 15) / 16, c.ns);
    // one cooperative launch per sweep when all its CTAs can be resident at once, else one launch per round
    const bool coop = coop_launch_fits(sweep_fn, 256, (long long)grd.x * grd.y * grd.z);
    for (int sweep = 0; sweep <= MAX_SWEEPS; ++sweep) {
        jac_off_kernel<<<c.ns, 256, 0, st>>>(a, flip);
        count_launch();
        cudaError_t e = cudaMemcpyAsync(hstats.data(), stats.p, hstats.size() * sizeof(double), cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) { set_error("max_step: %s", cudaGetErrorString(e)); return CVXB_E_CUDA; }
        ok = true;
        for (int k = 0; k < c.ns; ++k) {
            if (c.s[k] && !jac_done(hstats[2 * k], hstats[2 * k + 1], prev[k], c.s[k])) ok = false;
            prev[k] = hstats[2 * k];
        }
        if (ok || sweep == MAX_SWEEPS) break;
        if (coop) {
            void *args[] = {&a, &flip};
            if (cudaLaunchCooperativeKernel(sweep_fn, grd, blk, args, 0, st) != cudaSuccess) {
                set_error("max_step: cooperative launch failed: %s", cudaGetErrorString(cudaGetLastError()));
                return CVXB_E_CUDA;
            }
            count_launch();
            flip ^= 1;                                   // N - 1 (odd) buffer swaps
        } else {
            for (int r = 0; r < a.N - 1; ++r) {
                if (with_vectors) jac_round_kernel<true><<<grd, blk, 0, st>>>(a, r, flip);
                else jac_round_kernel<false><<<grd, blk, 0, st>>>(a, r, flip);
                count_launch();
                flip ^= 1;
            }
        }
    }
    if (!ok) { set_error("max_step: Jacobi eigensolver did not converge (non-finite input?)"); return 1; }
    jac_sort_kernel<<<c.ns, 256, 0, st>>>(a, flip);
    count_launch();
    if (with_vectors) {
        const int gx = (int)std::min<size_t>(((size_t)c.maxs * c.maxs + 255) / 256, 1184);
        jac_vec_kernel<<<dim3(gx, c.ns), 256, 0, st>>>(a);
        count_launch();
    }
    cudaError_t e = cudaGetLastError();
    cudaStreamSynchronize(st);                           // before the scratch is freed
    if (e != cudaSuccess) { set_error("max_step: %s", cudaGetErrorString(e)); return CVXB_E_CUDA; }
    return 0;
}

int cvxb_max_step(double *x, const cvxb_dims *dims, double *sigma, double *result, int space) {
    if (!result) { set_error("max_step: result is NULL"); return CVXB_E_ARG; }
    CallCtx ctx; CVXB_TRY(ctx.acquire(0));
    cudaStream_t st = ctx.st;
    ConeLayout c; CVXB_TRY(c.init(dims));
    const int nlq = c.mnl + c.ml + c.sumq;
    std::vector<int> sigoff(c.ns);
    for (int k = 0, o = 0; k < c.ns; ++k) { sigoff[k] = o; o += c.s[k]; }
    Staged xb;
    CVXB_TRY(xb.in(x, c.cdim, space, st));
    Scratch<double> d, dsig;
    Scratch<int> dsigoff;
    CVXB_TRY(d.alloc(1));
    max_step_kernel<<<1, 256, 0, st>>>(xb.dev, cones_of(c), d.p);
    count_launch();
    if (c.maxs > 0) {
        // 's' blocks: lambda_min of each block (reference dsyevr_ range 'I' 1..1, or dsyevd_ 'V' when
        // sigma is given: eigenvalues -> sigma, eigenvectors -> x; misc_solvers.c:1099-1150)
        if (dsig.alloc(c.sums) || dsigoff.alloc(c.ns) ||
            cudaMemcpyAsync(dsigoff.p, sigoff.data(), (size_t)c.ns * sizeof(int), cudaMemcpyHostToDevice, st) != cudaSuccess) {
            cudaGetLastError();
            set_error("max_step: device allocation failed");
            return CVXB_E_NOMEM;
        }
        CVXB_TRY(sym_eig_blocks(c, xb.dev + nlq, dsig.p, dsigoff.p, sigma != nullptr, st));
        max_step_s_kernel<<<1, 1, 0, st>>>(d.p, dsig.p, c.d_s, dsigoff.p, c.ns, nlq > 0);
        count_launch();
        if (sigma) {
            if (cudaMemcpyAsync(sigma, dsig.p, (size_t)c.sums * sizeof(double),
                                space == CVXB_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, st) != cudaSuccess) {
                set_error("max_step: copy of sigma failed");
                return CVXB_E_CUDA;
            }
            CVXB_TRY(xb.out(st));
        }
    }
    cudaError_t e = cudaMemcpyAsync(result, d.p, sizeof(double), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { set_error("max_step: %s", cudaGetErrorString(e)); return CVXB_E_CUDA; }
    return 0;
}

}  // extern "C"
