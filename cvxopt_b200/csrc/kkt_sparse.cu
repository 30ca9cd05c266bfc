// Sparse 'l' rows of G in the KKT factories (cvxb_kkt_create_sparse).
//
// The 'l' rows stay on the device twice: as CSR of G_l (for G x) and as CSR of G_l' (for G' y and the SYRK), so
// every product is a row-by-row sum with one owner per output and a fixed order: no atomics, the same bits on every
// run.  The pattern never changes, so the transpose and the SYRK's work partition are built once, at create.
//
// K := D + G_l' diag(w) G_l (lower) costs sum_k nnz(row k)^2 / 2 multiply-adds here, against ml n^2 / 2 for the
// dense SYRK; dense_wins picks the dense path when the sparse work is too large (DESIGN.md).
#include "cone.cuh"
#include "kkt_internal.cuh"
#include <algorithm>
#include <vector>

namespace cvxb {

namespace {
constexpr int SY_WARPS = 8;         // warps per CTA of the sparse SYRK
constexpr int SY_CHUNKS = kNumSMs * 64;   // column chunks: one per warp the SMs hold at once
constexpr int MV_LANES = 8;         // lanes per output row of the sparse GEMV
constexpr int MV_THREADS = 256;
// The dense SYRK takes over when sum_k nnz(row k)^2 > ml n^2 / kDenseRatio.  Measured on an H100 80GB HBM3 at 700 W
// (DESIGN.md, "Sparse G"): at n = 4096, ml = 65536 the two SYRKs take the same time at a ratio of about 1270.
constexpr double kDenseRatio = 1250.0;

// Warp w owns the columns [bnd[w], bnd[w+1]) of K.  For its column j it first writes D (or 0) into rows i >= j, then
// walks the entries G_kj of column j in order of k; for each, its lanes split the entries of row k from column j on,
// K[i, j] += (w_k G_kj) G_ki.  The columns in one row are distinct, so no two lanes write the same K[i, j], and
// __syncwarp orders one row's updates before the next's.
__global__ void __launch_bounds__(SY_WARPS * 32)
k_sparse_syrk(int n, int nchunk, const int *__restrict__ bnd, const long long *__restrict__ rowptr,
              const int *__restrict__ colind, const double *__restrict__ val, const long long *__restrict__ colptr,
              const int *__restrict__ rowind, const double *__restrict__ tval, const long long *__restrict__ tpos,
              const double *__restrict__ w, const double *__restrict__ D, long long ldd, double *K, long long ldk) {
    const int warp = blockIdx.x * SY_WARPS + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (warp >= nchunk) return;
    const unsigned full = 0xffffffffu;
    for (int j = bnd[warp]; j < bnd[warp + 1]; ++j) {
        double *Kj = K + (long long)j * ldk;
        if (D) {
            const double *Dj = D + (long long)j * ldd;
            for (int i = j + lane; i < n; i += 32) Kj[i] = Dj[i];
        } else {
            for (int i = j + lane; i < n; i += 32) Kj[i] = 0.0;
        }
        __syncwarp();
        const long long e1 = colptr[j + 1];
        for (long long e0 = colptr[j]; e0 < e1; e0 += 32) {
            // 32 entries of column j at a time, one per lane, then broadcast one by one
            const long long e = e0 + lane;
            double g = 0.0;
            long long qa = 0, qb = 0;
            if (e < e1) {
                const int kr = rowind[e];
                g = tval[e] * (w ? w[kr] : 1.0);
                qa = tpos[e];
                qb = rowptr[kr + 1];
            }
            const int cnt = (int)min(32LL, e1 - e0);
            for (int t = 0; t < cnt; ++t) {
                const double gt = __shfl_sync(full, g, t);
                const long long a = __shfl_sync(full, qa, t), b = __shfl_sync(full, qb, t);
                for (long long q = a + lane; q < b; q += 32) Kj[colind[q]] += gt * val[q];
                __syncwarp();
            }
        }
    }
}

// y[r] = alpha * (so ? so[r] : 1) * sum_q v[q] (si ? si[c] : 1) x[c] + beta * y[r],  c = idx[q], q in [ptr[r], ptr[r+1])
// MV_LANES lanes per row; their partial sums meet in a fixed shuffle tree.  beta == 0 does not read y.
__global__ void __launch_bounds__(MV_THREADS)
k_csr_mv(int rows, const long long *__restrict__ ptr, const int *__restrict__ idx, const double *__restrict__ v,
         const double *__restrict__ si, const double *__restrict__ so, const double *__restrict__ x, double alpha,
         double beta, double *__restrict__ y) {
    const long long r = ((long long)blockIdx.x * MV_THREADS + threadIdx.x) / MV_LANES;
    const int l = threadIdx.x % MV_LANES;
    double s = 0.0;
    if (r < rows)
        for (long long q = ptr[r] + l; q < ptr[r + 1]; q += MV_LANES) {
            const int c = idx[q];
            s += v[q] * (si ? si[c] * x[c] : x[c]);
        }
    for (int o = MV_LANES / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (r < rows && l == 0) {
        const double t = alpha * (so ? so[r] * s : s);
        y[r] = beta == 0.0 ? t : t + beta * y[r];
    }
}

// rows [r0, r0 + rows) of the dense G (ld ldg) from the CSR rows 0.. (one warp per row); G is zero on entry
__global__ void k_csr_scatter(int rows, const long long *__restrict__ ptr, const int *__restrict__ idx,
                              const double *__restrict__ v, double *G, long long ldg, int r0) {
    const long long r = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (r >= rows) return;
    for (long long q = ptr[r] + lane; q < ptr[r + 1]; q += 32) G[(r0 + r) + (long long)idx[q] * ldg] = v[q];
}

template <class T> int upload(DevBuf<T> &dst, const T *src, size_t count, cudaStream_t st) {
    CVXB_TRY(dst.alloc(count ? count : 1));
    if (count) CVXB_CUDA(cudaMemcpyAsync(dst.p, src, count * sizeof(T), cudaMemcpyHostToDevice, st));
    return 0;
}

bool dense_wins(double sparse_work, double ml, double n) { return sparse_work * kDenseRatio > ml * n * n; }
}  // namespace

int kkt_sparse_load(cvxb_kkt *k, const long long *rowptr, const int *colind, const double *val) {
    const ConeLayout &c = k->cone;
    const int n = k->n, ml = c.ml, r0 = c.mnl, rq = c.cdim - c.mnl - c.ml;
    const size_t nn = (size_t)(n > 0 ? n : 1);
    cudaStream_t st = k->st;
    k->sp.reset(new SparseL());
    SparseL &s = *k->sp;
    // the 'q' and 's' rows: dense, ld ldg, in Gown
    k->G = nullptr;
    k->ldg = (rq + 1) & ~1;
    if (k->ldg < 2) k->ldg = 2;
    std::vector<double> hq;
    if (rq > 0) {
        hq.assign((size_t)k->ldg * nn, 0.0);
        for (int i = 0; i < rq; ++i)
            for (long long q = rowptr[r0 + ml + i]; q < rowptr[r0 + ml + i + 1]; ++q)
                hq[i + (size_t)colind[q] * k->ldg] = val[q];
        CVXB_TRY(upload(k->Gown, hq.data(), hq.size(), st));
    }
    // the 'l' rows as CSR
    const long long base = rowptr[r0];
    s.nnz = rowptr[r0 + ml] - base;
    std::vector<long long> rp(ml + 1);
    double work = 0.0;
    for (int i = 0; i <= ml; ++i) rp[i] = rowptr[r0 + i] - base;
    for (int i = 0; i < ml; ++i) work += (double)(rp[i + 1] - rp[i]) * (double)(rp[i + 1] - rp[i]);
    CVXB_TRY(upload(s.rowptr, rp.data(), rp.size(), st));
    CVXB_TRY(upload(s.colind, colind + base, (size_t)s.nnz, st));
    CVXB_TRY(upload(s.val, val + base, (size_t)s.nnz, st));
    if (ml > 0 && dense_wins(work, ml, n)) {
        CVXB_CUDA(cudaStreamSynchronize(st));
        return kkt_sparse_densify(k);
    }
    // CSR of G_l' by a counting sort over the columns: rows come out in increasing order within each column
    std::vector<long long> cp(nn + 1, 0), tpos((size_t)s.nnz);
    std::vector<int> ri((size_t)s.nnz);
    std::vector<double> tv((size_t)s.nnz);
    for (long long q = 0; q < s.nnz; ++q) ++cp[colind[base + q] + 1];
    for (int j = 0; j < n; ++j) cp[j + 1] += cp[j];
    {
        std::vector<long long> next(cp.begin(), cp.end() - 1);
        for (int i = 0; i < ml; ++i)
            for (long long q = rp[i]; q < rp[i + 1]; ++q) {
                const long long e = next[colind[base + q]]++;
                ri[e] = i; tv[e] = val[base + q]; tpos[e] = q;
            }
    }
    // per-column work of the SYRK in warp steps: the column's fill, then per entry G_kj a broadcast and the row's
    // suffix from column j on; chunks of contiguous columns with equal shares of the total
    std::vector<double> cost(nn, 0.0);
    double total = 0.0;
    for (int j = 0; j < n; ++j) {
        double cj = (double)((n - j + 31) / 32);
        for (long long e = cp[j]; e < cp[j + 1]; ++e) cj += 2.0 + (double)((rp[ri[e] + 1] - tpos[e] + 31) / 32);
        cost[j] = cj;
        total += cj;
    }
    s.nchunk = std::max(1, std::min(n, SY_CHUNKS));
    std::vector<int> bnd(s.nchunk + 1, n);
    bnd[0] = 0;
    {
        int ch = 1;
        double acc = 0.0;
        for (int j = 0; j < n && ch < s.nchunk; ++j) {
            acc += cost[j];
            while (ch < s.nchunk && acc * s.nchunk >= total * ch) bnd[ch++] = j + 1;
        }
    }
    CVXB_TRY(upload(s.colptr, cp.data(), cp.size(), st));
    CVXB_TRY(upload(s.rowind, ri.data(), ri.size(), st));
    CVXB_TRY(upload(s.tval, tv.data(), tv.size(), st));
    CVXB_TRY(upload(s.tpos, tpos.data(), tpos.size(), st));
    CVXB_TRY(upload(s.bnd, bnd.data(), bnd.size(), st));
    CVXB_CUDA(cudaStreamSynchronize(st));       // before the host copies go out of scope
    return 0;
}

int kkt_sparse_densify(cvxb_kkt *k) {
    if (!k->sp) return 0;
    const ConeLayout &c = k->cone;
    const int n = k->n, rq = c.cdim - c.mnl - c.ml;
    const size_t nn = (size_t)(n > 0 ? n : 1);
    cudaStream_t st = k->st;
    long long ld = (c.cdim + 1) & ~1;
    if (ld < 2) ld = 2;
    DevBuf<double> G;
    CVXB_TRY(G.alloc((size_t)ld * nn));
    CVXB_CUDA(cudaMemsetAsync(G.p, 0, (size_t)ld * nn * sizeof(double), st));
    if (c.ml > 0 && k->sp->nnz > 0) {
        const long long threads = (long long)c.ml * 32;
        k_csr_scatter<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(c.ml, k->sp->rowptr.p, k->sp->colind.p,
                                                                        k->sp->val.p, G.p, ld, c.mnl);
        CVXB_LAUNCH_CHECK();
        count_launch();
    }
    if (rq > 0) CVXB_TRY(upload_matrix(G.p + c.mnl + c.ml, ld, k->Gown.p, k->ldg, rq, n, CVXB_DEVICE, st));
    CVXB_CUDA(cudaStreamSynchronize(st));
    k->Gown = std::move(G);
    k->G = k->Gown.p;
    k->ldg = ld;
    k->sp.reset();
    // the dense 'l' rows now go through gemv_n too
    if (k->gemv_ws.p && k->gemv_ws.n < kkt_gemv_ws_doubles(k)) CVXB_TRY(k->gemv_ws.alloc(kkt_gemv_ws_doubles(k)));
    return 0;
}

int kkt_sparse_syrk(cvxb_kkt *k, const double *D, long long ldd, const double *w, double *K, long long ldk) {
    const SparseL &s = *k->sp;
    if (k->n <= 0) return 0;
    const int ctas = (s.nchunk + SY_WARPS - 1) / SY_WARPS;
    k_sparse_syrk<<<ctas, SY_WARPS * 32, 0, k->st>>>(k->n, s.nchunk, s.bnd.p, s.rowptr.p, s.colind.p, s.val.p,
                                                     s.colptr.p, s.rowind.p, s.tval.p, s.tpos.p, w, D, ldd, K, ldk);
    CVXB_LAUNCH_CHECK();
    count_launch();
    return 0;
}

int kkt_sparse_mv(cvxb_kkt *k, bool trans, const double *w, const double *x, double alpha, double beta, double *y) {
    const SparseL &s = *k->sp;
    const int rows = trans ? k->n : k->cone.ml;
    if (rows <= 0) return 0;
    const long long threads = (long long)rows * MV_LANES;
    const unsigned ctas = (unsigned)((threads + MV_THREADS - 1) / MV_THREADS);
    if (trans)
        k_csr_mv<<<ctas, MV_THREADS, 0, k->st>>>(rows, s.colptr.p, s.rowind.p, s.tval.p, w, nullptr, x, alpha, beta,
                                                 y);
    else
        k_csr_mv<<<ctas, MV_THREADS, 0, k->st>>>(rows, s.rowptr.p, s.colind.p, s.val.p, nullptr, w, x, alpha, beta,
                                                 y);
    CVXB_LAUNCH_CHECK();
    count_launch();
    return 0;
}

}  // namespace cvxb
