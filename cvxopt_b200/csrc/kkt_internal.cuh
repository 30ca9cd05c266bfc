// Internal definition of the KKT factory handle shared by kkt_api.cu (Cholesky route, misc.kkt_chol / kkt_chol2),
// kkt_qr.cu (misc.kkt_qr) and kkt_ldl.cu (misc.kkt_ldl2).
#pragma once
#include "cone.cuh"
#include <memory>

using cvxb::ConeLayout;
using cvxb::DevScaling;
using cvxb::CholWork;
using cvxb::DevBuf;

namespace cvxb {
// state of the QR route (kkt_qr.cu)
struct QrState {
    int nq = 0;                 // n - p: columns of Gs2
    DevBuf<double> Q;           // n x n orthogonal factor of A' (p > 0)
    long long ldQ = 0;
    DevBuf<double> R1;          // p x p upper triangular (ld p)
    DevBuf<double> tau;
    DevBuf<double> GsF;         // cdim_pckd x n: Gs, then Gs [Q1 Q2] (p > 0: second buffer)
    DevBuf<double> GsQ;
    long long ldf = 0;
    DevBuf<double> Q3t;         // nq x cdim_pckd: Q3'
    long long ldq = 0;
    DevBuf<double> C[3], inv[3];
    long long ldc = 0;
    int npass = 2;
    DevBuf<double> w, u, vv, xt, ws, norm2;
};

// state of the LDL' route (kkt_ldl.cu)
struct LdlState {
    int N = 0;
    DevBuf<double> K2;          // N x N
    long long ld = 0;
    DevBuf<int> ipiv;           // LAPACK convention, 1-based, negative for 2x2 blocks
    DevBuf<int> state;          // [0] k  [1] kstep  [2] kp  [3] info  [4] pending (step to finish)
    DevBuf<double> w1, w2;      // multipliers of the current step
    DevBuf<double> u;           // N right-hand side
    double kktreg = 0.0;
};

// the 'l' rows of G kept sparse on the device (cvxb_kkt_create_sparse, kkt_sparse.cu).  Two copies of the pattern, so
// that G x and G' y both run as row-by-row sums, without atomics.
struct SparseL {
    long long nnz = 0;
    DevBuf<long long> rowptr;   // ml + 1: CSR of G_l
    DevBuf<int> colind;         // nnz, sorted within each row
    DevBuf<double> val;         // nnz
    DevBuf<long long> colptr;   // n + 1: CSR of G_l' (the CSC view of G_l)
    DevBuf<int> rowind;         // nnz, sorted within each column
    DevBuf<double> tval;        // nnz
    DevBuf<long long> tpos;     // nnz: index in val of the same entry, where the row's columns >= this one start
    DevBuf<int> bnd;            // nchunk + 1 column boundaries: warp w of the SYRK owns columns [bnd[w], bnd[w+1])
    int nchunk = 0;
};
}  // namespace cvxb

struct cvxb_kkt {
    int device = 0;
    int n = 0, p = 0;
    ConeLayout cone;
    const double *G = nullptr;   // cdim x n, rows [mnl, cdim) hold G (rows [0,mnl) belong to Df)
    DevBuf<double> Gown;         // backs G when it came from the host; a device G stays the caller's
    long long ldg = 0;
    // sparse 'l' rows (cvxb_kkt_create_sparse): G is unused, and Gown holds only the 'q' and 's' rows (ld ldg)
    std::unique_ptr<cvxb::SparseL> sp;
    DevBuf<double> Hres;         // resident H (symmetrised), or empty
    DevBuf<double> Hbuf;         // per-call H upload buffer (lazy)
    DevBuf<double> Kmat;         // n x n: normal equations, then its Cholesky factor (lower)
    DevBuf<double> inv;          // inverses of the diagonal blocks of L
    DevBuf<double> Gs;           // scaled+packed rows that are not 'l': [mnl | q | s packed] x n
    long long ldgs = 0;
    int nrest = 0;
    DevBuf<double> Gunp;         // unpacked scaled 's' rows (sums2 x n) — only when ns > 0
    DevBuf<double> Dfbuf;        // mnl x n upload buffer
    // equality constraints (p > 0), kkt_chol2-style elimination (reference misc.py:1464-1472):
    DevBuf<double> Aeq;          // p x n (ld lda_eq)
    long long lda_eq = 0;
    DevBuf<double> Asct;         // n x p: L^{-1} A'
    long long ldas = 0;
    DevBuf<double> Kp;           // p x p: Asct' Asct, then its Cholesky factor
    long long ldkp = 0;
    DevBuf<double> invp;         // diagonal-block inverses of chol(Kp)
    DevBuf<double> yd;           // p
    bool singular = false;       // first factorisation failed -> S += A'A from then on (misc.py:1433-1447)
    bool first_factor = true;
    DevScaling W;
    DevBuf<double> bzp, zin, zt, xv, yv;
    DevBuf<double> gemv_ws;
    DevBuf<double> swork;        // congruence workspace of the 's' rows
    CholWork cw;
    cudaStream_t st = nullptr;
    cudaEvent_t e0 = nullptr, e1 = nullptr, e2 = nullptr, e3 = nullptr, t0 = nullptr, t1 = nullptr;
    cudaEvent_t m0 = nullptr, m1 = nullptr;      // around the MMA launches of the int8-slice SYRK
    double mma_ms = 0.0;
    double factor_ms = 0, solve_ms = 0, br[3] = {0, 0, 0};
    bool factored = false;
    // SYRK of the 'l' rows on the int8 tensor path (ozaki_syrk.cu): ozaki_mode() at create; by default off: on
    // H100 the fp64 DMMA kernel is the faster of the two at every size measured (DESIGN.md).
    int i8_mode = 0;
    DevBuf<char> oz_work;
    int syrk_path = 0;           // kernel of the last factor's 'l'-row SYRK: 0 none, 1 fp64 DMMA, 2 int8 slices,
                                 // 3 sparse (kkt_sparse.cu)
    // factorisation route: 0 Cholesky of the reduced system (kkt_chol / kkt_chol2), 1 QR (kkt_qr), 2 LDL' of the
    // 2x2 system (kkt_ldl2).  Set once after create (cvxb_kkt_set_method), with the state of that route.
    int method = 0;
    std::unique_ptr<cvxb::QrState> qr;
    std::unique_ptr<cvxb::LdlState> ldl;
    ~cvxb_kkt();                 // synchronises the stream, then releases it and the events; the members free the rest
};


namespace cvxb {
int upload_matrix(double *dst, long long ldd, const double *src, long long lds, int rows, int cols, int space,
                  cudaStream_t st);
int xfer_vec(double *dst, const double *src, size_t n, int space, bool to_device, cudaStream_t st);
inline long long kkt_ldk(const cvxb_kkt *k) { long long l = (k->n + 1) & ~1; return l > 2 ? l : 2; }
int kkt_pack_bz(cvxb_kkt *k, const double *zd);      // k->bzp := pack(W^{-T} bz)
int kkt_unpack_z(cvxb_kkt *k, double *zd);           // z := unpack(k->bzp)
// the 'q' and 's' rows of pack(W^{-T} G): dst is where the first 'q' row goes (ld ldd), the packed 's' rows follow
// at dst + sumq
int kkt_scale_pack_G(cvxb_kkt *k, double *dst, long long ldd);
// route-specific factor / solve (kkt_qr.cu, kkt_ldl.cu); the solves work in place on device vectors, between
// cvxb_kkt_solve's kkt_pack_bz and kkt_unpack_z
int kkt_qr_factor(cvxb_kkt *k, const cvxb_scaling *W, int space);
int kkt_qr_solve(cvxb_kkt *k, double *xd, double *yd);
int kkt_qr_setup(cvxb_kkt *k);
// LDL' route: Kmat holds S (lower) on entry of factor; info (k->cw.d_info) = first exactly-zero pivot, 1-based
int kkt_ldl_factor(cvxb_kkt *k);
int kkt_ldl_solve(cvxb_kkt *k, double *xd, double *yd);
int kkt_ldl_setup(cvxb_kkt *k, double kktreg);
// first 'q' row of G (ld k->ldg); the 's' rows follow it
inline const double *kkt_G_qs(const cvxb_kkt *k) {
    return k->sp ? k->Gown.p : k->G + k->cone.mnl + k->cone.ml;
}
// sparse 'l' rows (kkt_sparse.cu).  kkt_sparse_load: rowptr/colind/val are the validated host CSR of all cdim rows;
// it keeps the 'l' rows sparse, or densifies them when the dense SYRK is the faster path.
int kkt_sparse_load(cvxb_kkt *k, const long long *rowptr, const int *colind, const double *val);
// turn a sparse handle into a dense one: rows [mnl, cdim) of a new dense G, on the device
int kkt_sparse_densify(cvxb_kkt *k);
// K (lower) := D + G_l' diag(w) G_l, D lower (ld ldd) or zero when D is NULL
int kkt_sparse_syrk(cvxb_kkt *k, const double *D, long long ldd, const double *w, double *K, long long ldk);
// y := alpha diag(w) G_l x + beta y (trans false, y has ml entries) or alpha G_l' diag(w) x + beta y (trans true,
// y has n entries); w may be NULL
int kkt_sparse_mv(cvxb_kkt *k, bool trans, const double *w, const double *x, double alpha, double beta, double *y);
// doubles of gemv_n workspace the handle needs
size_t kkt_gemv_ws_doubles(const cvxb_kkt *k);
}  // namespace cvxb
