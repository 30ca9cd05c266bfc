/*
 * cvxopt_b200 — C ABI of the H100-native KKT hot path of CVXOPT's cone solvers.
 *
 * Every entry point below is what a CVXOPT-side binding for this path would
 * bind (ctypes / CPython C-API; see INTEGRATION.md).  Plain pointers and sizes
 * only; no torch / Python types.  All matrices are fp64, column-major (the
 * layout of cvxopt's `matrix`, reference src/C/cvxopt.h:48-56), all index
 * arguments are 0-based element counts.
 *
 * Cone layout of every "cone vector" (reference src/python/coneprog.py:79-96):
 *   [ mnl nonlinear | ml 'l' | q[0] .. q[nq-1] 'q' blocks | s[0]^2 .. 's' blocks ]
 *   cdim      = mnl + ml + sum q + sum s^2        (unpacked, 's' blocks full col-major)
 *   cdim_pckd = mnl + ml + sum q + sum s(s+1)/2   (packed lower, off-diag * sqrt 2)
 *
 * Return codes (all int-returning functions):
 *    0   success
 *   >0   LAPACK-style `info`: leading minor of that order is not positive
 *        definite (the reference raises ArithmeticError for this,
 *        src/C/lapack.c:32-34) — Python layer raises ArithmeticError
 *   <0   CVXB_E_* below (bad argument / CUDA failure); cvxb_last_error() has text
 */
#ifndef CVXOPT_B200_H
#define CVXOPT_B200_H

#ifdef __cplusplus
extern "C" {
#endif

#define CVXB_E_ARG     (-1)   /* invalid argument (ValueError in the reference, misc.h:78-110) */
#define CVXB_E_CUDA    (-2)   /* CUDA runtime error */
#define CVXB_E_NOMEM   (-3)   /* allocation failure */
#define CVXB_E_NOGPU   (-4)   /* no usable sm_90 device: the product path has NO CPU fallback */
#define CVXB_E_UNSUP   (-5)   /* valid in the reference but not built on the device */

/* memory space of the pointers handed to a call */
#define CVXB_HOST   0
#define CVXB_DEVICE 1

typedef struct cvxb_kkt cvxb_kkt;     /* opaque: one kkt_chol factory instance  */
typedef struct cvxb_batch cvxb_batch; /* opaque: batch of independent dense QPs */

/* cone dimensions: mirror of the reference `dims` dict + mnl */
typedef struct {
    int mnl;          /* nonlinear rows (cvxprog), 0 for conelp/coneqp            */
    int ml;           /* dims['l']                                                 */
    int nq;           /* len(dims['q'])                                            */
    const int *q;     /* dims['q'][k]                                              */
    int ns;           /* len(dims['s'])                                            */
    const int *s;     /* dims['s'][k]                                              */
} cvxb_dims;

/* Nesterov-Todd scaling: flat mirror of the reference `W` dict
 * (src/python/coneprog.py:327-334, src/python/misc.py:45-56) */
typedef struct {
    const double *dnl, *dnli;   /* mnl each (may be NULL when mnl == 0)           */
    const double *d, *di;       /* ml each                                         */
    const double *v;            /* W['v'][0] | W['v'][1] | ...   (sum q)           */
    const double *beta;         /* nq                                              */
    const double *r, *rti;      /* W['r'][k] / W['rti'][k], s[k] x s[k] col-major,
                                   concatenated (sum s^2)                          */
} cvxb_scaling;

/* ---- library / device ---------------------------------------------------- */
const char *cvxb_last_error(void);
int  cvxb_device_count(void);                 /* sm_90 devices visible             */
int  cvxb_version(void);
/* number of kernels this library has launched since load (bench.py's gpu_launches) */
unsigned long long cvxb_launch_count(void);
/* bytes of device memory the library's handles and per-device workspaces hold right now (all devices); back to
 * its earlier value once a handle is destroyed.  The scratch-buffer cache of the calls without a handle is not
 * counted. */
unsigned long long cvxb_device_bytes(void);
/* cudaMalloc/cudaFree/cudaMemcpy shims so a ctypes-only host needs no CUDA binding */
int  cvxb_malloc(void **dptr, unsigned long long bytes);
int  cvxb_free(void *dptr);
int  cvxb_memcpy_h2d(void *dst, const void *src, unsigned long long bytes);
int  cvxb_memcpy_d2h(void *dst, const void *src, unsigned long long bytes);
int  cvxb_sync(void);

/* ---- kkt_chol factory:  replaces misc.kkt_chol(G, dims, A, mnl)
 *      reference src/python/misc.py:1213-1255.
 * G is cdim x n (rows mnl.. hold G; the mnl leading rows are Df, given per
 * factor call).  G is uploaded ONCE and stays resident in HBM.
 * space = CVXB_HOST: G/A are host pointers (copied); CVXB_DEVICE: device
 * pointers that are ADOPTED without copy (caller keeps them alive). */
int cvxb_kkt_create(cvxb_kkt **out, int n, int p, const cvxb_dims *dims,
                    const double *G, int ldg, const double *A, int lda,
                    int space, int device);
/* The same factory for a sparse G: cdim x n in CSR form with 0-based indices, rows [0, mnl) empty (they belong to
 * Df).  rowptr (cdim + 1 entries), colind and val (nnz each) are HOST arrays whatever `space` is; `space` applies to A.
 * The columns of each row must be sorted and distinct.  Every check is made before the device is touched: rowptr[0] != 0,
 * a decreasing rowptr, rowptr[cdim] != nnz, a column outside [0, n), unsorted or duplicate columns in a row, and
 * entries in rows [0, mnl) return CVXB_E_ARG with the fault named in cvxb_last_error().
 * The 'l' rows stay sparse on the device (a CSR copy and a CSR copy of their transpose) and their SYRK and GEMVs run
 * on sparse kernels; when sum over 'l' rows of nnz(row)^2 is too large against ml n^2 for that to pay, they are
 * densified once here and take the dense path (cvxb_kkt_syrk_path tells which).  The 'q' and 's' rows are kept dense.
 * Every other call works on this handle as on a dense one; route 1 (QR) densifies the 'l' rows first. */
int cvxb_kkt_create_sparse(cvxb_kkt **out, int n, int p, const cvxb_dims *dims, const long long *rowptr,
                           const int *colind, const double *val, long long nnz, const double *A, int lda,
                           int space, int device);
void cvxb_kkt_destroy(cvxb_kkt *k);

/* Factorisation route of this factory, chosen once right after cvxb_kkt_create:
 *   0  Cholesky of the reduced system           misc.kkt_chol / kkt_chol2   (misc.py:1213, :1352)  [default]
 *   1  QR:  A' = [Q1 Q2][R1; 0] (Householder, once), W^{-T} G Q2 = Q3 R3 per factor (Cholesky-QR with
 *      re-orthogonalisation, shifted when ill-conditioned)        misc.kkt_qr   (misc.py:1570-1699)
 *   2  LDL' with Bunch-Kaufman pivoting of the 2x2 system [H + Gs'Gs, A'; A, 0]   misc.kkt_ldl2 (misc.py:1128-1210);
 *      kktreg != 0 adds the reference's regularisation (misc.py:1096-1098 convention) to the diagonal.
 * Route 1 accepts no H / Df (zero (1,1) block, conelp). */
int cvxb_kkt_set_method(cvxb_kkt *k, int method, double kktreg);

/* Start a new solver run on the same factory (G, A, H stay resident): forgets the first-factorisation state
 * ("S singular on the first call -> S + A'A for the rest of the run", misc.py:1433-1447). */
int cvxb_kkt_reset(cvxb_kkt *k);

/* Make H (n x n, lower triangle significant) resident; later factor calls with
 * H == NULL and use_resident_H=1 add it.  coneqp passes the same P every
 * iteration (coneprog.py:1980-1981) — this avoids re-uploading n^2 doubles. */
int cvxb_kkt_set_H(cvxb_kkt *k, const double *H, int ldh, int space);

/* factor: replaces the closure `factor(W, H, Df)`  misc.py:1257-1282
 *   Gs = pack(W^{-T} [Df; G]);  K = Gs'Gs + H (lower);  K = L L'
 * W pointers live in `space`.  H/Df may be NULL.  use_resident_H: add the
 * matrix given to cvxb_kkt_set_H.  Returns info>0 on a non-positive pivot. */
int cvxb_kkt_factor(cvxb_kkt *k, const cvxb_scaling *W, const double *H, int ldh,
                    const double *Df, int lddf, int use_resident_H, int space);

/* solve: replaces the closure `solve(x, y, z)`  misc.py:1284-1345.
 * In place: (bx, by, bz) -> (ux, uy, W*uz).  x: n, y: p, z: cdim. */
int cvxb_kkt_solve(cvxb_kkt *k, double *x, double *y, double *z, int space);

/* read back pieces for tests: the Cholesky factor (n x n lower) */
int cvxb_kkt_get_L(cvxb_kkt *k, double *L_host, int ldl);
/* timing of the last factor/solve in ms (CUDA events on the library stream) */
int cvxb_kkt_last_ms(cvxb_kkt *k, double *factor_ms, double *solve_ms);
/* bracket a timed region with CUDA events on the library's launch stream (bench.py):
 * start records an event; stop records, synchronises and returns the elapsed ms */
int cvxb_kkt_timer_start(cvxb_kkt *k);
int cvxb_kkt_timer_stop(cvxb_kkt *k, double *ms);
/* debug (env CVXB_TRACE=1): globaltimer timeline of the last Cholesky, 8 values per block step:
 * {diag, trsm, next-column update, bulk update} x {start, end} in ns */
int cvxb_kkt_trace(cvxb_kkt *k, unsigned long long *out, int nsteps);
/* per-kernel-class CUDA-event breakdown of the last factor (syrk, potrf, scale) */
int cvxb_kkt_last_breakdown(cvxb_kkt *k, double *ms3);
/* which kernel computed the 'l'-row SYRK of the last factor: 0 none (ml == 0), 1 fp64 DMMA
 * (mma.sync.m16n8k4.f64, the default), 2 int8 slices on wgmma s8 (CVXB_OZAKI=2 always, =1 for large problems;
 * falls back to 1 when the slice workspace does not fit in device memory), 3 the sparse kernel of a
 * cvxb_kkt_create_sparse handle that kept its 'l' rows sparse */
int cvxb_kkt_syrk_path(cvxb_kkt *k);
/* int8-slice path only: CUDA-event time of the MMA launches of the last factor's SYRK, without the two slicing kernels
 * (0 on the DMMA path); bench.py's roofline line divides the int8 operations by this */
int cvxb_kkt_syrk_mma_ms(cvxb_kkt *k, double *ms);
/* QR route: Cholesky-QR passes of the last factor: 2 (plain, re-orthogonalised) or 3 (shifted, ill-conditioned) */
int cvxb_kkt_qr_passes(cvxb_kkt *k);

/* device-resident G / P operators for the function-valued G(x,y,alpha,beta,trans)
 * / P(x,y,alpha,beta) protocol of coneprog (coneprog.py:1682-1711):
 *   y := alpha*G*x + beta*y  (trans 'N')   or   y := alpha*G'*x + beta*y ('T')
 *   y := alpha*H*x + beta*y  (H symmetric, lower stored) */
int cvxb_kkt_gemv_G(cvxb_kkt *k, const double *x, double *y, double alpha, double beta,
                    int trans, int space);
int cvxb_kkt_symv_H(cvxb_kkt *k, const double *x, double *y, double alpha, double beta,
                    int space);
/* y := alpha*A*x + beta*y ('N') or alpha*A'*x + beta*y ('T') on the resident equality-constraint
 * matrix: the function-valued A(x, y, alpha, beta, trans) protocol (coneprog.py:1682-1711) */
int cvxb_kkt_gemv_A(cvxb_kkt *k, const double *x, double *y, double alpha, double beta,
                    int trans, int space);

/* The calls from here to cvxb_gemm take no handle.  The cone algebra and the NT scaling run on device 0, the dense
 * building blocks on their `device` argument, and calls on one device are serialised across host threads (each
 * call holds that device's one stream until it returns). */

/* ---- cone algebra: mirror of src/C/misc_solvers.c (12 entry points,
 * misc_solvers.c:1155-1173).  x is xr x xc column-major with leading
 * dimension xr; everything in place as in the reference. */
int cvxb_scale(double *x, int xr, int xc, const cvxb_dims *dims, const cvxb_scaling *W,
               int trans /*'N'|'T'*/, int inverse /*'N'|'I'*/, int space); /* misc_solvers.c:85  */
int cvxb_scale2(const double *lmbda, double *x, const cvxb_dims *dims, int inverse,
                int space);                                                  /* :256 */
int cvxb_pack(const double *x, double *y, const cvxb_dims *dims, int space); /* :412 */
int cvxb_pack2(double *x, int xr, int xc, const cvxb_dims *dims, int space); /* :476 */
int cvxb_unpack(const double *x, double *y, const cvxb_dims *dims, int space); /* :552 */
int cvxb_symm(double *x, int n, int space);                                  /* :610 */
int cvxb_sprod(double *x, const double *y, const cvxb_dims *dims, int diag, int space);  /* :634 */
int cvxb_sinv(double *x, const double *y, const cvxb_dims *dims, int space); /* :775 */
int cvxb_trisc(double *x, const cvxb_dims *dims, int space);                 /* :887 */
int cvxb_triusc(double *x, const cvxb_dims *dims, int space);                /* :940 */
int cvxb_sdot(const double *x, const double *y, const cvxb_dims *dims, double *result,
              int space);                                                    /* :991 */
/* sigma == NULL: x is read only.  sigma != NULL (sum of the 's' orders): the eigenvalues of every 's'
 * block go to sigma (ascending) and its eigenvectors overwrite the block of x (:1132-1136).
 * Returns 1 if the eigensolver does not converge (non-finite input). */
int cvxb_max_step(double *x, const cvxb_dims *dims, double *sigma, double *result,
                  int space);                                                /* :1052 */

/* ---- Nesterov-Todd scaling itself: misc.compute_scaling (src/python/misc.py:250-419) and
 * misc.update_scaling (:422-634) for every cone type.  `W` points at WRITABLE arrays laid out as in
 * cvxb_scaling (the const qualifiers of that struct are cast away for these two calls): compute_scaling fills
 * them, update_scaling updates them in place together with lmbda; update_scaling also overwrites s and z the
 * way the reference does.  lmbda has mnl + ml + sum q + sum s entries.  's' blocks: Cholesky + one-sided Jacobi
 * SVD on the device in place of lapack.potrf / lapack.gesvd; singular values in descending order.
 * Returns info > 0 if an 's' block is not positive definite (ArithmeticError in the reference). */
int cvxb_compute_scaling(const double *s, const double *z, double *lmbda, const cvxb_dims *dims,
                         const cvxb_scaling *W, int space);
int cvxb_update_scaling(const cvxb_scaling *W, double *lmbda, double *s, double *z,
                        const cvxb_dims *dims, int space);

/* ---- dense building blocks (the BLAS/LAPACK calls of the path, device pointers):
 * blas.syrk(trans='T') blas.c:3039 fused with the 'l' row scaling;
 * lapack.potrf lapack.c:1471; lapack.potrs lapack.c:1553. */
int cvxb_syrk_scaled(int n, int k, const double *A, int lda, const double *rowscale,
                     const double *H, int ldh, double *C, int ldc, int device);
/* The same SYRK, C(lower) = A' diag(d)^2 A + H, computed on the int8 tensor path by error-free
 * slicing (Ozaki scheme, `slices` = 1..9 radix-2^7 digits per entry; 9 reproduces fp64).  Note d, not
 * d^2 as in cvxb_syrk_scaled.  cvxb_kkt_factor uses it for the 'l' block when CVXB_OZAKI=2 (or =1 and large).
 * blas.syrk blas.c:3039. */
int cvxb_syrk_scaled_i8(int n, int k, const double *A, int lda, const double *d, const double *H,
                        int ldh, double *C, int ldc, int slices, int device);
/* work_inv: 2 * ceil(n/128) * 128*128 doubles — receives the inverses (and their
 * transposes) of the 128x128 diagonal blocks of L, consumed by cvxb_potrs */
int cvxb_potrf(int n, double *A, int lda, double *work_inv, int device);
int cvxb_potrs(int n, const double *L, int ldl, const double *inv, double *b, int device);
/* plain C = alpha * op(A) op(B) + beta*C on the DMMA kernel (tests / 's' congruence) */
int cvxb_gemm(int transa, int transb, int m, int n, int k, double alpha, const double *A,
              int lda, const double *B, int ldb, double beta, double *C, int ldc, int device);

/* ---- batched dense building blocks: the factorisation, solves and products the batch solver below runs on all of
 * its problems at once, exposed for tests and for callers that batch their own factorisations.  Device pointers,
 * column-major; problem b of an operand is at base + b * stride (strides in doubles).  batch outside
 * 1..CVXB_BATCH_MAX, a negative size, a leading dimension below max(1, rows) or an unknown trans is CVXB_E_ARG,
 * checked before the device.  Nothing is split or reduced across problems: a problem's result depends on its own
 * data and the layout only. */
/* n x n Cholesky (lower) of every problem in place; work_inv as for cvxb_potrf, per problem (stride sInv >=
 * 2 * ceil(n/128) * 128*128).  info (host, batch ints) receives LAPACK's info per problem; returns 0 or CVXB_E_*. */
int cvxb_potrf_batched(int n, double *A, int lda, long long sA, double *work_inv, long long sInv,
                       int batch, int *info, int device);
/* in place on b with cvxb_potrf_batched's factors: trans 'N' solves L x = b, 'T' solves L' x = b ('N' then 'T' is
 * potrs) */
int cvxb_trsv_batched(int n, const double *L, int ldl, long long sL, const double *inv, long long sInv,
                      double *b, long long sb, int trans, int batch, int device);
/* B := L^{-1} B in place, B n x ncols */
int cvxb_trsm_batched(int n, const double *L, int ldl, long long sL, const double *inv, long long sInv,
                      double *B, int ldb, long long sB, int ncols, int batch, int device);
/* lower triangle of C = A' diag(w) A + D, A k x n; w and D may be NULL, D may equal C */
int cvxb_syrk_batched(int n, int k, const double *A, int lda, long long sA, const double *w, long long sw,
                      const double *D, int ldd, long long sD, double *C, int ldc, long long sC,
                      int batch, int device);
/* A nrows x ncols.  trans 'T': y = alpha A' (w .* x) + beta y;  'N': y = alpha w .* (A x) + beta y.  w may be NULL;
 * beta = 0 does not read y */
int cvxb_gemv_batched(int trans, int nrows, int ncols, const double *A, int lda, long long sA,
                      const double *w, long long sw, const double *x, long long sx, double alpha,
                      double beta, double *y, long long sy, int batch, int device);

/* ---- batch of independent dense QPs (BASELINE config 4): one problem per
 * CTA-group, lock-step primal-dual IPM fully on device (oracle: a Python loop
 * over coneqp).  Problems are  min 1/2 x'P x + q'x  s.t.  G x + s = h, s in the
 * cone product  'l' x 'q'[0] x ... ; all problems share n and the dims.
 * cvxb_batch_create(.., m, ..) is dims = {'l': m}: G x <= h.
 * A batch with 'q' cones materialises Gs = W^{-T} G per problem (nprob * cdim * n
 * more doubles); an 'l'-only batch, with or without refinement, folds the 'l'
 * scaling into the SYRK and the GEMVs instead.
 * nprob is at most CVXB_BATCH_MAX: the batched kernels put the problem index in gridDim.y / gridDim.z, which
 * are limited to 65535.  A larger nprob is CVXB_E_ARG (checked before the device); split larger batches
 * (qp_batch's sub-batches do). */
#define CVXB_BATCH_MAX 65535
int cvxb_batch_create(cvxb_batch **out, int nprob, int n, int m, int device);
/* batch of  min 1/2 x'Px + q'x  s.t.  G x + s = h,  s in 'l' x 'q' cones  (B x coneqp, coneprog.py:1440).
 * dims->mnl != 0, a cone order q[k] < 1, nprob > CVXB_BATCH_MAX: CVXB_E_ARG; dims->ns > 0: CVXB_E_UNSUP. */
int cvxb_batch_create_cones(cvxb_batch **out, int nprob, int n, const cvxb_dims *dims, int device);
/* batch of  min 1/2 x'Px + q'x  s.t.  G x + s = h,  s in 'l' x 'q' cones,  A x = b  with p equality rows per
 * problem (B x coneqp(P, q, G, h, dims, A, b); kktsolver 'chol2' without 'q' cones, 'chol' with them: both
 * eliminate A through S = P + Gs'Gs, Asct = L^{-1} A', Kp = Asct'Asct, misc.py:1352-1560).  p = 0 is
 * cvxb_batch_create_cones.  p < 0 and the dims / nprob violations of cvxb_batch_create_cones are CVXB_E_ARG, and so
 * is p > n ("Rank(A) < p or Rank([P; A; G]) < n"), all checked before the device.  A problem whose S is singular at
 * the start factors S + A'A for the rest of the solve (misc.py:1421-1447); if that, or Kp, is singular at the start,
 * cvxb_batch_solve returns CVXB_E_ARG naming the problem.  Device memory per problem on top of the p = 0 batch, in
 * doubles: lda*n (A, lda = p rounded up to even, at least 2) + ldk*p (Asct, ldk = n rounded up to even) + lda*p (Kp)
 * + 2*ceil(p/128)*128^2 (Kp's diagonal-block inverses, even for small p) + 5p (b, y, ry, dy, A'A weight) + 2p
 * rounded up to even with refinement (wy, wy2), plus one int (Kp's info); all of it is counted by cvxb_device_bytes
 * and freed by cvxb_batch_destroy. */
int cvxb_batch_create_eq(cvxb_batch **out, int nprob, int n, int p, const cvxb_dims *dims, int device);
/* batch of cone LPs  min c'x  s.t.  G x + s = h,  s in 'l' x 'q' cones,  A x = b  with p equality rows per problem
 * (B x conelp(c, G, h, dims, A, b), coneprog.py:31-1436: the self-dual embedding with its infeasibility
 * certificates; kktsolver 'chol2' without 'q' cones, 'chol' with them; refinement 0 without 'q' cones, 1 with them).
 * Load it with cvxb_batch_load_lp (and cvxb_batch_load_eq when p > 0); every other cvxb_batch_* call serves both kinds
 * of batch.  CVXB_E_ARG, checked before the device: dims->mnl != 0, a cone order q[k] < 1, nprob > CVXB_BATCH_MAX,
 * p < 0, and, as conelp's "Rank(A) < p or Rank([G; A]) < n", p > n or p + cdim < n.  m = cdim = 0 is CVXB_E_ARG too:
 * a cone LP batch needs at least one cone row.  dims->ns > 0: CVXB_E_UNSUP.  A singular factorisation at the start
 * (W = I) makes cvxb_batch_solve return CVXB_E_ARG naming the problem.  Device memory per problem, in doubles: that of
 * the QP batch of the same n, cdim, p and dims without P's ldp*n (ldp = n rounded up to even), plus n + 2*cdim + p
 * (x1, z1, W^{-T} h, y1) and 18 scalars (tau, kappa and the rest of the embedding) in the per-problem state row; all
 * of it is counted by cvxb_device_bytes and freed by cvxb_batch_destroy. */
int cvxb_batch_create_lp(cvxb_batch **out, int nprob, int n, int p, const cvxb_dims *dims, int device);
/* the largest 's' order of a batch: one CTA holds a block's working matrices in shared memory */
#define CVXB_BATCH_SMAX 32
/* batch of cone LPs whose dims may hold 's' blocks as well as 'l' and 'q' cones: B x conelp(c, G, h, dims, A, b) with
 * kktsolver 'chol', the reference's solvers.sdp when dims is {'l': ml, 's': [...]}.  It refuses what
 * cvxb_batch_create_lp refuses, and, before the device: an order s[k] < 0 (CVXB_E_ARG), s[k] > CVXB_BATCH_SMAX
 * (CVXB_E_UNSUP), and conelp's rank check with the packed dimension, p > n or p + cdim_pckd < n (CVXB_E_ARG).  An
 * order-0 block adds no rows.  Every other cvxb_batch_* call serves it: G is cdim x n column-major with each 's'
 * block's rows unpacked (s[k]^2 rows, the block column-major), as the reference's G; only the lower triangle of each
 * 's' block of G and h is read.  cvxb_batch_results returns s and z with 's' blocks symmetric.  Refinement defaults
 * to 1.  Device memory per problem, in doubles: that of the cone LP batch of the same n, cdim and p, plus ldg*n for
 * Gs if dims has no 'q' cone, 2*sum(s^2) + 2*sum(s) (r, rti, and the eigenvalues sigs, sigz) each rounded up to even
 * in the state row, and 4 per block of partial sums; and, shared by the batch, cdim doubles of row weights and
 * cdim - ml - sum(q) + 5 ns ints of layout; all of it is counted by cvxb_device_bytes and freed by
 * cvxb_batch_destroy. */
int cvxb_batch_create_sdp(cvxb_batch **out, int nprob, int n, int p, const cvxb_dims *dims, int device);
/* batch of QPs  min 1/2 x'Px + q'x  s.t.  G x + s = h,  s in 'l' x 'q' x 's' cones,  A x = b  with p equality rows per
 * problem: B x coneqp(P, q, G, h, dims, A, b) with its default kktsolver ('chol' with 's' cones), each 's' order at
 * most CVXB_BATCH_SMAX.  It refuses, before the device, what cvxb_batch_create_eq refuses (CVXB_E_ARG: dims->mnl != 0,
 * a cone order q[k] < 1, nprob > CVXB_BATCH_MAX, p < 0, and coneqp's only rank check, p > n) and an order s[k] < 0
 * (CVXB_E_ARG) or s[k] > CVXB_BATCH_SMAX (CVXB_E_UNSUP); p + cdim_pckd < n is accepted, since P may have full rank.
 * Load it with cvxb_batch_load (and cvxb_batch_load_eq when p > 0), G and h laid out as for cvxb_batch_create_sdp;
 * results come back through cvxb_batch_results (s and z with symmetric 's' blocks) and cvxb_batch_results_y.  A
 * singular factorisation at the start makes cvxb_batch_solve return CVXB_E_ARG naming the problem.  Refinement
 * defaults to 1.  Device memory per problem, in doubles: that of the cvxb_batch_create_eq batch of the same n, cdim
 * (with the 's' blocks unpacked) and p, plus ldg*n for Gs if dims has no 'q' cone, 2*sum(s^2) + 2*sum(s) (r, rti,
 * sigs, sigz) each rounded up to even in the state row, and 4 per block of partial sums; and, shared by the batch,
 * cdim doubles of row weights and cdim - ml - sum(q) + 5 ns ints of layout; all of it is counted by
 * cvxb_device_bytes and freed by cvxb_batch_destroy.  Dims without an 's' block of positive order run exactly what
 * cvxb_batch_create_eq's batch runs. */
int cvxb_batch_create_sdp_qp(cvxb_batch **out, int nprob, int n, int p, const cvxb_dims *dims, int device);
/* ---- the batch solver's 's' block kernels on caller data, for tests: one launch of the kernel the solver runs, one
 * CTA per (block, problem), on blocks of the given orders laid out as in the solver without 'l' and 'q' rows.  Device
 * pointers; problem b of an m-vector operand is at base + b * m, of a state-row operand at base + b * L.  m-vectors
 * (s, z, ds, dz, h, lmbda, lmbdasq, d, di, ws3): the blocks one after another, each ms x ms column-major, lambda on a
 * block's diagonal rows; bzp and th hold the blocks packed (lower triangle by columns, off-diagonals times sqrt 2).
 * State rows: r, rti, wz, ws, wz2, ws2, wz3 at the blocks' unpacked offsets, sigs and sigz at sum of the earlier
 * orders.  G and Gs: column j of problem b at base + b * sG + j * ldg, rows as an m-vector (Gs packed).  Outputs the
 * solver stages come back staged: k_s_update's r in d, rti in di, s in ds, z in dz, lambda+ in lmbdasq's diagonal rows.
 * spart (host, batch * nblk * 4, problem-major) is uploaded before the launch and returned after it: per (problem,
 * block) sdot, the two smallest eigenvalues and the failure flag as the kernel leaves them.  done (host, batch ints)
 * and info (host, batch ints, k_s_update) may be NULL for all zero.  mode: k_s_update's `first`, k_s_dir_post's i,
 * k_s_wtz's mode (0, 1, 2), k_s_res's LP flag (1: ut = dtau / dg for every problem, needs L >= 17); 0 otherwise.
 * CVXB_E_ARG, before the device: batch outside 1..CVXB_BATCH_MAX, nblk < 1, an order outside 1..CVXB_BATCH_SMAX,
 * m or L below the blocks' rows, an unknown kernel or mode, or an operand the kernel reads or writes missing. */
#define CVXB_SK_NT_COMPUTE 0
#define CVXB_SK_UPDATE 1
#define CVXB_SK_DIR_POST 2
#define CVXB_SK_EIG_START 3
#define CVXB_SK_EIG_WARM 4
#define CVXB_SK_BUILD_GS 5
#define CVXB_SK_WTZ 6
#define CVXB_SK_RES 7
typedef struct {
    int nblk;
    const int *orders;                /* host, nblk */
    long long m, L;                   /* per-problem strides of the m-vector and the state-row operands */
    int n;                            /* columns of G (k_s_build_gs) */
    long long ldg, sG;
    double step;                      /* Scal.step of every problem (k_s_update) */
    double ut;                        /* k_s_res<true> */
    const int *done, *info;
    double *spart;
    double *s, *z, *ds, *dz, *h, *lmbda, *lmbdasq, *d, *di, *bzp, *th, *ws3;
    double *r, *rti, *sigs, *sigz, *wz, *ws, *wz2, *ws2, *wz3;
    const double *G;
    double *Gs;
} cvxb_sblock_args;
int cvxb_sblock_batched(int kernel, int mode, int batch, const cvxb_sblock_args *args, int device);
/* steps of iterative refinement per Newton solve; default 1 if dims has 'q' cones, else 0 (coneprog.py:1862-1865) */
int cvxb_batch_set_refinement(cvxb_batch *b, int refinement);
void cvxb_batch_destroy(cvxb_batch *b);
/* P: nprob x (n x n, ld n); q: nprob x n; G: nprob x (m x n column-major, ld m); h: nprob x m; m = cdim */
int cvxb_batch_load(cvxb_batch *b, const double *P, const double *q, const double *G,
                    const double *h, int space);
/* A: nprob x (p x n column-major, ld p); bvec: nprob x p.  Call it after every cvxb_batch_load of a batch with
 * p > 0 equality rows (cvxb_batch_solve refuses such a batch with CVXB_E_ARG until it is); a no-op when p = 0. */
int cvxb_batch_load_eq(cvxb_batch *b, const double *A, const double *bvec, int space);
/* cone LP batch only (cvxb_batch_load on it, and this call on a QP batch, are CVXB_E_ARG):
 * c: nprob x n; G: nprob x (m x n column-major, ld m); h: nprob x m; m = cdim */
int cvxb_batch_load_lp(cvxb_batch *b, const double *c, const double *G, const double *h, int space);
/* the starting point of the next solves (warm start): x nprob x n, y nprob x p, s and z nprob x cdim laid out as h
 * (an 's' block unpacked column-major, only its lower triangle read).  NULL: the key is absent.
 * QP batch: coneqp(..., initvals) with the given keys (coneprog.py:2109-2149); an absent x or y is 0, an absent s or
 * z is e (1 on the 'l' rows, on each 'q' cone's first row and on each 's' block's diagonal), so all NULL is the e
 * start.  Nothing is shifted, the W = I factorisation is skipped and iteration 0's factorisation is the first one:
 * kkt_chol2's S + A'A switch is decided there, and a KKT matrix still singular there makes cvxb_batch_solve return
 * CVXB_E_ARG naming the problem (Rank(A) < p or ...).  A batch without constraint rows (cdim = 0) ignores the start.
 * Cone LP batch: conelp(..., primalstart, dualstart) (coneprog.py:662-857): x and s together are primalstart, z with
 * an optional y is dualstart; x without s, s without x, y without z, or neither start is CVXB_E_ARG.  With one of the
 * two the W = I factorisation solves for the other half, which is shifted as conelp shifts it; with both, iteration 0's
 * factorisation is the first, as for a QP.
 * A given s or z that is not strictly inside the cone makes cvxb_batch_solve return CVXB_E_ARG with "problem %d:
 * initial s (z) is not positive".  The start is kept in the caller's problem order across solves and across
 * cvxb_batch_load*, until the next cvxb_batch_load_start or cvxb_batch_clear_start.  The first call allocates
 * nprob * (n + p + 2 cdim) doubles of device memory, counted by cvxb_device_bytes and freed by cvxb_batch_destroy. */
int cvxb_batch_load_start(cvxb_batch *b, const double *x, const double *s, const double *y, const double *z,
                          int space);
/* back to the cold start (the W = I start of coneqp and conelp); the start's memory stays with the handle */
int cvxb_batch_clear_start(cvxb_batch *b);
int cvxb_batch_solve(cvxb_batch *b, int maxiters, double abstol, double reltol, double feastol);
/* status: 1 optimal, 2 maximum iterations reached, 3 singular KKT matrix ('unknown' in the
 * reference for 2 and 3), and for cone LP batches 4 primal infeasible, 5 dual infeasible.  Where conelp returns None
 * the results hold NaN: x, s and the primal objective of a primal infeasible problem (its dual objective is 1, y and
 * z the certificate), y, z and the dual objective of a dual infeasible one (its primal objective is -1, x and s the
 * certificate).  x/s/z may be device pointers (space), scalars go to host memory. */
int cvxb_batch_results(cvxb_batch *b, double *x, double *s, double *z, int *status,
                       int *iters, double *pobj, double *dobj, int space);
/* y: nprob x p, the multipliers of A x = b in the caller's problem order (as x, s, z); nothing when p = 0 */
int cvxb_batch_results_y(cvxb_batch *b, double *y, int space);
/* Derivatives of the last solve's results with respect to the problem data, for a loss L with gradients gx = dL/dx
 * (nprob x n), gy = dL/dy (nprob x p) and gz = dL/dz (nprob x m).  At the returned iterate it solves
 *     [P A' G'; A 0 0; G 0 -W'W] [ux; uy; uz] = [gx; gy; gz],   W'W = diag(s / z),
 * with one more factorisation of the reduced KKT matrix and one step of iterative refinement on the full system, and
 * writes ux (nprob x n), uy (nprob x p), uz (nprob x m) and
 *     dP = -(ux x' + x ux') / 2   (n x n column-major per problem, both triangles: the gradient over symmetric P),
 *     dG = -(z ux' + uz x')        (m x n column-major per problem, as cvxb_batch_load's G),
 *     dA = -(y ux' + uy x')        (p x n column-major per problem, as cvxb_batch_load_eq's A);
 * dL/dq = -ux, dL/dh = uz and dL/db = uy.  Every array is in the caller's problem order and in `space`.  A NULL input
 * is zero; a NULL output is not written and its work is skipped.  A problem whose status is not 1 (optimal), or whose
 * KKT matrix has no Cholesky factor at that iterate, gets NaN in all its outputs.  The scaling comes from the returned
 * s and z alone, so the outputs are a function of the results; cvxb_batch_results is unchanged afterwards and a
 * re-solve computes the same results.  Each call factors again.
 * QP batches whose rows are all 'l' only (cvxb_batch_create, cvxb_batch_create_eq with dims {'l': m}); any other batch
 * is CVXB_E_UNSUP.  A batch without a completed cvxb_batch_solve since its last cvxb_batch_load or
 * cvxb_batch_load_eq is CVXB_E_ARG.  CVXB_DEVICE allocates nothing; CVXB_HOST stages each given array in temporary
 * device memory, at most nprob * (2 (n + p + m) + n (n + m + p)) doubles in all. */
int cvxb_batch_adjoint(cvxb_batch *b, const double *gx, const double *gy, const double *gz, double *ux, double *uy,
                       double *uz, double *dP, double *dG, double *dA, int space);
/* CUDA-event time of the last cvxb_batch_solve and the number of lock-step iterations run */
int cvxb_batch_stats(cvxb_batch *b, double *solve_ms, int *iterations);
/* kernel of the factorisations' SYRK in the last solve: 1 fp64 DMMA, 2 int8 slices (as cvxb_kkt_syrk_path) */
int cvxb_batch_syrk_path(cvxb_batch *b);
/* batch of geometric programs (B x solvers.gp, cvxprog.py:1967-2155, with its default kktsolver 'chol2'):
 *     minimize  log sum exp(F0 x + g0)  s.t.  log sum exp(Fi x + gi) <= 0 (i = 1..mnl),  G x <= h,  A x = b
 * with the block sizes K[0..nK-1] (mnl = nK - 1) shared by the batch, ml rows of G and p rows of A.  It runs cpl on
 * gp's epigraph problem (cp, :1746-1964) in lock-step, line search included.  CVXB_E_ARG, checked before the device:
 * nprob outside 1..CVXB_BATCH_MAX, n < 1, nK < 1, some K[i] < 1, ml < 0, p < 0, and gp's "Rank(A) < p" for p > n.
 * Load it with cvxb_batch_load_gp (and cvxb_batch_load_eq when p > 0); cvxb_batch_load, cvxb_batch_load_lp and
 * cvxb_batch_load_start on it are CVXB_E_ARG (gp takes no starting point).  Solve, set_refinement (default 1, as cpl),
 * results, results_y, stats and destroy are the other batches' calls: s and z have the mnl + ml rows [snl; sl] and
 * [znl; zl] (the epigraph row is dropped), the primal objective is t and the dual objective cpl's.  Status 1 optimal,
 * 2 maximum iterations, 3 singular KKT matrix or a line-search step that underflowed to 0 ('unknown' for 2 and 3).
 * A singular factorisation at iteration 0 makes cvxb_batch_solve return CVXB_E_ARG with "problem %d: Rank(A) < p or
 * Rank([H(x); A; Df(x); G]) < n".  Device memory per problem, with m = mnl + ml, S = sum K, ev() rounding up to even:
 * what cvxb_batch_create_eq's batch of the same n, p and dims {'l': m} holds with refinement 1, except that G is
 * ev(m + S) x n and the GEMV workspace holds max(m, S) rows, plus ev(S)*n (H's scaled rows), 4S + nK + 3n + p + 4m
 * (softmax, weights, f, grad f0, g, the unscaled steps and the line search's trial point) and ev(S) + 56 + 3 ev(n) +
 * 3 ev(p) + 10 ev(m) in the state row (g, the scalars and the line search's saved state); and, shared by the batch,
 * nK + 1 ints; all of it is counted by cvxb_device_bytes and freed by cvxb_batch_destroy. */
int cvxb_batch_create_gp(cvxb_batch **out, int nprob, int n, int nK, const int *K, int ml, int p, int device);
/* GP batch only: F nprob x (S x n column-major, ld S), g nprob x S, G nprob x (ml x n column-major, ld ml), h
 * nprob x ml; G and h may be NULL when ml = 0.  A and b come through cvxb_batch_load_eq. */
int cvxb_batch_load_gp(cvxb_batch *b, const double *F, const double *g, const double *G, const double *h, int space);
/* line-search rounds of the last solve of a GP or CP batch (every round evaluates F at every searching problem's trial
 * point; a CP batch's domain rounds count too); 0 for the other batches */
int cvxb_batch_ls_rounds(cvxb_batch *b);
/* batch of smooth convex programs (B x solvers.cp(F, G, h, dims={'l': ml}, A, b), cvxprog.py:1359-1964, with its
 * default kktsolver 'chol2'):
 *     minimize  f0(x)  s.t.  fk(x) <= 0 (k = 1..mnl),  G x <= h,  A x = b
 * with F evaluated by the caller (cvxb_batch_set_cp_eval).  It runs the GP batch's lock-step cpl on cp's epigraph
 * problem, starting from the loaded x0 with t = 0, y = 0 and s = z = e, and backtracks each direction's step into
 * dom f before the line search (:1052-1060).  CVXB_E_ARG, checked before the device: nprob outside
 * 1..CVXB_BATCH_MAX, n < 1, mnl < 0, ml < 0, p < 0, and cp's "Rank(A) < p" for p > n.  Load it with
 * cvxb_batch_load_cp (and cvxb_batch_load_eq when p > 0); cvxb_batch_load, load_lp, load_gp and load_start on it are
 * CVXB_E_ARG.  Solve, set_refinement (default 1, as cpl, also when mnl + ml = 0), results, results_y, stats,
 * ls_rounds and destroy are the GP batch's calls with its semantics: s and z are [snl; sl] and [znl; zl], the primal
 * objective is t, status 3 is a singular KKT matrix or a step that underflowed to 0 in the domain or merit line
 * search.  Solving without an evaluator is CVXB_E_ARG, as is a callback that returns non-zero ("the evaluation
 * callback returned %d"), a singular KKT matrix at iteration 0 ("problem %d: Rank(A) < p or Rank([H(x); A; Df(x);
 * G]) < n") and an f that is not finite at an iterate ("problem %d: x0 not in the domain of f" at iteration 0).
 * The solve calls back to the host, so it must not be captured into a CUDA graph.  Device memory per problem, with
 * m = mnl + ml, nf = mnl + 1 and ev() rounding up to even: what cvxb_batch_create_eq's batch of the same n, p and
 * dims {'l': m} holds with refinement 1, plus nf(n + 2) + n² (the callback's f, Df, z and H), nf + 3n + p + 4m (f,
 * grad f0, the unscaled steps and the line search's trial point), n (x0), 56 + 3 ev(n) + 3 ev(p) + 10 ev(m) in the
 * state row (the scalars and the line search's saved state) and one int (slot -> problem); and one int shared by the
 * batch; all of it is counted by cvxb_device_bytes and freed by cvxb_batch_destroy. */
int cvxb_batch_create_cp(cvxb_batch **out, int nprob, int n, int mnl, int ml, int p, int device);
/* CP batch only: x0 nprob x n (strictly inside dom f), G nprob x (ml x n column-major, ld ml), h nprob x ml; G and h
 * may be NULL when ml = 0.  A and b come through cvxb_batch_load_eq. */
int cvxb_batch_load_cp(cvxb_batch *b, const double *x0, const double *G, const double *h, int space);
/* F of a CP batch, called on the solving thread with k = the active problems (every evaluation covers all of them;
 * rows of problems that are not searching are evaluated and ignored).  Device buffers owned by the handle, row-major
 * per problem and problem-contiguous, nf = mnl + 1:
 *     x        k x n            in: the points (read only)
 *     z        k x nf           in, full evaluations only: [z0; znl] (read only)
 *     problem  k ints           in: the load index of each row (read only)
 *     f        k x nf           out: f(x); a row with a NaN or an infinite entry means x is not in dom f
 *     Df       k x nf x n       out: the rows of Df(x)
 *     H        k x n x n        out, full evaluations only: sum_i z_i grad² f_i(x), only its lower triangle is read
 * full = 1 at the iterates, where f must be finite; full = 0 (z and H NULL) at trial points.  stream is the batch's
 * cudaStream_t: the callback enqueues its work there and does not synchronise.  It must return 0, and the same
 * values for the same point.  fn = NULL clears the evaluator. */
typedef int (*cvxb_cp_eval_fn)(void *ctx, int k, int full, const double *x, const double *z, const int *problem,
                               double *f, double *Df, double *H, void *stream);
int cvxb_batch_set_cp_eval(cvxb_batch *b, cvxb_cp_eval_fn fn, void *ctx);
/* batch of cpl problems (B x solvers.cpl(c, F, G, h, dims, A, b), cvxprog.py:35-1356, with its default kktsolver):
 *     minimize  c'x  s.t.  fk(x) <= 0 (k = 1..mnl),  G x + s = h,  s in 'l' x 'q'[0] x ...,  A x = b
 * with F evaluated by the caller (cvxb_batch_set_cp_eval, nK = mnl: f, Df and z have no objective row).  It runs the
 * CP batch's lock-step cpl without the epigraph row, the 'q' rows after the 'l' rows, from the loaded x0 with y = 0
 * and s = z = e.  With 'q' cones the reference's default kktsolver is 'chol' (a QR of A' and a Cholesky of order
 * n - p); the batch keeps its 'chol2' elimination (S = H + Gs'Gs with Gs = W^{-T} [Df; G], S + A'A for a problem
 * whose S is singular at the start, then Kp), as the QP batch does with 'q' cones: both solve the same KKT system.
 * Refused before the device: CVXB_E_ARG for nprob outside 1..CVXB_BATCH_MAX, n < 1, mnl < 0, p < 0, dims NULL,
 * dims->mnl != 0, a negative count, a q[k] < 1, no constraint rows (mnl + cdim = 0) and cpl's "Rank(A) < p" for
 * p > n; CVXB_E_UNSUP for dims->ns > 0.  Load it with cvxb_batch_load_cpl (and cvxb_batch_load_eq when p > 0);
 * cvxb_batch_load, load_lp, load_gp, load_cp and load_start on it are CVXB_E_ARG.  Solve, set_refinement (default 1,
 * as cpl), results, results_y, stats, ls_rounds and destroy are the CP batch's calls with its semantics, except that
 * s and z are [snl; sl] and [znl; zl] with the 'q' rows in sl and zl, and the primal objective is c'x.  Device memory
 * per problem, with m = mnl + cdim and ev() rounding up to even: what cvxb_batch_create_eq's batch of the same n, p
 * and dims {'l': mnl + ml, 'q': q} holds with refinement 1, plus mnl(n + 2) + n² (the callback's f, Df, z and H),
 * mnl + 3n + p + 4m (f, the unscaled steps and the line search's trial point), n (x0), 56 + 3 ev(n) + 3 ev(p) +
 * 10 ev(m) in the state row (the scalars and the line search's saved state), ev(sum q) + ev(nq) more there with 'q'
 * cones (the saved v and beta), and one int (slot -> problem); and one int shared by the batch. */
int cvxb_batch_create_cpl(cvxb_batch **out, int nprob, int n, int mnl, const cvxb_dims *dims, int p, int device);
/* cpl batch only: c nprob x n, x0 nprob x n (strictly inside dom f), G nprob x (cdim x n column-major, ld cdim), h
 * nprob x cdim ('l' rows, then each 'q' cone); G and h may be NULL when cdim = 0.  A and b come through
 * cvxb_batch_load_eq. */
int cvxb_batch_load_cpl(cvxb_batch *b, const double *c, const double *x0, const double *G, const double *h, int space);
/* batch of cpl problems whose dims may hold 's' blocks (B x solvers.cpl(c, F, G, h, dims, A, b) with an LMI), each
 * 's' order at most CVXB_BATCH_SMAX:
 *     minimize  c'x  s.t.  fk(x) <= 0 (k = 1..mnl),  G x + s = h,  s in 'l' x 'q' x 's' cones,  A x = b
 * It refuses, before the device, what cvxb_batch_create_cpl refuses except dims->ns > 0, and an order s[k] < 0
 * (CVXB_E_ARG) or s[k] > CVXB_BATCH_SMAX (CVXB_E_UNSUP); the 's' rows count as constraint rows.  An order-0 block adds
 * no rows.  It is the cpl batch in every call: cvxb_batch_load_cpl (G and h rows: 'l', each 'q' cone, then each 's'
 * block unpacked, s[k]^2 rows column-major as the reference's G; only the lower triangle of an 's' block of G and h is
 * read), cvxb_batch_load_eq, set_cp_eval, solve, results (s and z with symmetric 's' blocks), results_y, stats,
 * ls_rounds and destroy.  It starts from s = z = e (the identity in each 's' block).  Device memory per problem, in
 * doubles, with S = sum(s^2) over the blocks and ev() rounding up to even: that of the cvxb_batch_create_cpl batch of
 * the same n, mnl and p with dims {'l': ml + S, 'q': q} (the same m = mnl + cdim rows), plus ldg*n for Gs if dims has
 * no 'q' cone, 2 ev(S) + 2 ev(sum s) (r, rti, sigs, sigz) and 2 ev(S) (the line search's saved r and rti) in the state
 * row, with 'q' cones 2 (ev(sum q + S) - ev(sum q)) more there (v and the saved v span the blocks' rows), and 4 per
 * block of partial sums; and, shared by the batch, m doubles of row weights and S + 5 nb ints of layout, nb the number
 * of blocks of positive order; all of it is counted by cvxb_device_bytes and freed by cvxb_batch_destroy.  Dims
 * without an 's' block of positive order run exactly what cvxb_batch_create_cpl's batch runs. */
int cvxb_batch_create_sdp_cpl(cvxb_batch **out, int nprob, int n, int mnl, const cvxb_dims *dims, int p, int device);
/* batch of convex QCQPs (B x solvers.cp(F, G, h, dims={'l': ml}, A, b) with its default kktsolver, F's functions
 * quadratic):
 *     minimize  f0(x)  s.t.  fi(x) <= 0 (i = 1..mnl),  G x <= h,  A x = b,   fi(x) = x'Pi x / 2 + qi'x + ri
 * with mnl, ml and p shared by the batch.  It is the CP batch with F evaluated by the library's own kernels: no
 * evaluator, no host callback, and no domain rounds (dom f is R^n).  Every Pi is the caller's promise to be positive
 * semidefinite; it is not checked.  mnl = 0 and P0 = 0 are allowed.  Refused before the device with CVXB_E_ARG: what
 * cvxb_batch_create_cp refuses, and (mnl + 1) n + mnl + ml + 1 > 2^30 ("too many rows").  Load it with
 * cvxb_batch_load_qcqp (and cvxb_batch_load_eq when p > 0); cvxb_batch_load, load_lp, load_gp, load_cp, load_cpl,
 * load_start and set_cp_eval on it are CVXB_E_ARG.  Solve, set_refinement (default 1), results, results_y, stats,
 * ls_rounds and destroy are the CP batch's calls with its semantics (status, s and z as [snl; sl] and [znl; zl], the
 * primal objective t, the rank error at iteration 0, "problem %d: x0 not in the domain of f" for a non-finite f at
 * x0).  Device memory per problem, in doubles, with m = mnl + ml, nK = mnl + 1, S = nK n and ev() rounding up to
 * even: what cvxb_batch_create_eq's batch of the same n, p and dims {'l': m} holds with refinement 1, except that G
 * is ev(m + S) x n (the stacked P0..Pmnl below [Df[1:]; G]) and the GEMV workspace holds max(m, S) rows, plus
 * S + nK + 3n + p + 4m (P x, f, grad f0, the unscaled steps and the line search's trial point), S + nK (q and r), n
 * (x0), ev(S + nK) + 56 + 3 ev(n) + 3 ev(p) + 10 ev(m) in the state row (q and r, the scalars and the line search's
 * saved state) and one int (slot -> problem); and one int shared by the batch; all of it is counted by
 * cvxb_device_bytes and freed by cvxb_batch_destroy. */
int cvxb_batch_create_qcqp(cvxb_batch **out, int nprob, int n, int mnl, int ml, int p, int device);
/* QCQP batch only: P nprob x ((mnl + 1) n x n column-major, ld (mnl + 1) n), the blocks P0..Pmnl stacked by rows,
 * only each block's lower triangle read; q nprob x (mnl + 1) x n (q0 first); r nprob x (mnl + 1); x0 nprob x n, or
 * NULL for 0; G nprob x (ml x n column-major, ld ml), h nprob x ml, NULL when ml = 0.  A and b come through
 * cvxb_batch_load_eq. */
int cvxb_batch_load_qcqp(cvxb_batch *b, const double *P, const double *q, const double *r, const double *x0,
                         const double *G, const double *h, int space);
/* Derivatives of a QCQP batch's last solve, cvxb_batch_adjoint's counterpart, for a loss L with gradients gx = dL/dx
 * (nprob x n), gy = dL/dy (nprob x p) and gz = dL/dz (nprob x m, m = mnl + ml, laid out as the results' [znl; zl]).
 * At the returned iterate, with the objective's multiplier z0 = 1, H = P0 + sum_i znl_i Pi, Df the mnl x n matrix of
 * rows (Pi x + qi)' (i = 1..mnl) and D = diag(s / z), it solves
 *     [H A' Df' G'; A 0 0 0; Df 0 -Dnl 0; G 0 0 -Dl] [ux; uy; uznl; uzl] = [gx; gy; gznl; gzl]
 * with one more factorisation of the reduced KKT matrix and one step of iterative refinement on the full system, and
 * writes ux (nprob x n), uy (nprob x p), uz = [uznl; uzl] (nprob x m) and the gradients dL/d(input):
 *     dP: per problem the (mnl + 1) n x n column-major stack of cvxb_batch_load_qcqp's P, both triangles of each
 *         block (the gradient over symmetric Pi, bitwise symmetric): dP0 = -(ux x' + x ux') / 2 and
 *         dPi = -(znl_i (ux x' + x ux') + uznl_i x x') / 2;
 *     dq: nprob x (mnl + 1) x n: dq0 = -ux, dqi = -(znl_i ux + uznl_i x);
 *     dr: nprob x (mnl + 1): dr0 = 0, dri = -uznl_i;
 *     dG = -(zl ux' + uzl x')  (ml x n column-major per problem, the 'l' rows only),
 *     dA = -(y ux' + uy x')    (p x n column-major per problem);
 * dL/dh = uzl and dL/db = uy.  Every array is in the caller's problem order and in `space`.  A NULL input is zero; a
 * NULL output is not written and its work is skipped: without dP, dq, dr, dG and dA the gradient kernel does not run.
 * A problem whose status is not 1 (optimal), or whose KKT matrix has no Cholesky factor at that iterate, gets NaN in
 * all its outputs, dr0 included.  The outputs are a function of the results and the data; cvxb_batch_results is
 * unchanged afterwards and a re-solve computes the same results.  QCQP batches only (cvxb_batch_create_qcqp): any
 * other batch is CVXB_E_UNSUP, and cvxb_batch_adjoint refuses a QCQP batch.  A batch without a completed
 * cvxb_batch_solve since its last cvxb_batch_load_qcqp or cvxb_batch_load_eq is CVXB_E_ARG.  CVXB_DEVICE allocates
 * nothing; CVXB_HOST stages each given array in temporary device memory, at most nprob * (2 (n + p + m) + nK n² +
 * nK n + nK + ml n + p n) doubles in all, nK = mnl + 1. */
int cvxb_batch_adjoint_qcqp(cvxb_batch *b, const double *gx, const double *gy, const double *gz, double *ux,
                            double *uy, double *uz, double *dP, double *dq, double *dr, double *dG, double *dA,
                            int space);
/* Derivatives of a cone QP or cone LP batch's last solve, cvxb_batch_adjoint's counterpart for batches with 'q' cones
 * and 's' blocks.  At the returned iterate it solves
 *     [P A' G'; A 0 0; G 0 -W'W] [ux; uy; uz] = [gx; gy; gz]
 * with W the Nesterov-Todd scaling of the returned s and z: diag(s / z) on the 'l' rows, W = beta (2 v v' - J) on a
 * 'q' cone, W'W(X) = r r' X r r' on an 's' block; P = 0 for a cone LP.  It factors the reduced KKT matrix once more,
 * takes one step of iterative refinement on the full system, and writes ux, uy, uz, dP, dG and dA with
 * cvxb_batch_adjoint's formulas and layouts: dL/dq (dL/dc) = -ux, dL/dh = uz, dL/db = uy.  This is the interior-point
 * linearisation at the returned iterate, exact on the central path; at a degenerate solution it is not the derivative
 * of the solution map.
 * 's' blocks: every 's' block of gz, uz and each column of dG is unpacked column-major, as the results' z, and the
 * pairing is the trace inner product, dL = sum over all unpacked entries of g * d.  Only the symmetric part
 * (gz + gz') / 2 of a gz block enters, so a gradient given on one triangle and its transpose give the same outputs.
 * Both triangles of uz's and dG's 's' blocks hold the same value, the gradient over symmetric matrices (as dP for P,
 * whose lower triangle alone is read), so a G whose 's' columns are built as X + X' gets the right gradient.
 * Accepts every QP batch (cvxb_batch_create, _cones, _eq, _sdp_qp) and every cone LP batch (cvxb_batch_create_lp,
 * _sdp); GP, CP, cpl and QCQP batches are CVXB_E_UNSUP.  dP must be NULL on a cone LP batch (CVXB_E_ARG).  A NULL
 * input is zero; a NULL output is not written and its work is skipped.  A problem whose status is not 1 (optimal: a
 * cone LP's infeasibility certificates included), whose KKT matrix has no Cholesky factor at that iterate, or whose
 * 's' scaling fails there (a block Cholesky factor or the SVD) gets NaN in all its outputs.  On a QP batch with 'l'
 * rows only it is cvxb_batch_adjoint, bit for bit.  cvxb_batch_results is unchanged afterwards and a re-solve
 * computes the same results.  A batch without a completed cvxb_batch_solve since its last load is CVXB_E_ARG.
 * CVXB_DEVICE allocates nothing; CVXB_HOST stages as cvxb_batch_adjoint does. */
int cvxb_batch_adjoint_cone(cvxb_batch *b, const double *gx, const double *gy, const double *gz, double *ux,
                            double *uy, double *uz, double *dP, double *dG, double *dA, int space);
/* Derivatives of a GP batch's last solve, cvxb_batch_adjoint_qcqp's counterpart, for a loss L with gradients gx =
 * dL/dx (nprob x n), gy = dL/dy (nprob x p) and gz = dL/dz (nprob x m, m = mnl + ml, laid out as the results' [znl;
 * zl]).  At the returned iterate, with the objective's multiplier z0 = 1, pi_i = softmax(Fi x + gi), Sigma_i =
 * diag(pi_i) - pi_i pi_i', H = sum_{i=0..mnl} z_i Fi' Sigma_i Fi, Df the mnl x n matrix of rows pi_i' Fi (i = 1..mnl)
 * and D = diag(s / z), it solves
 *     [H A' Df' G'; A 0 0 0; Df 0 -Dnl 0; G 0 0 -Dl] [ux; uy; uznl; uzl] = [gx; gy; gznl; gzl]
 * with one more factorisation of the reduced KKT matrix (S + A'A where S is singular there, as kkt_chol2 does) and one
 * step of iterative refinement on the full system, and writes ux (nprob x n), uy (nprob x p), uz = [uznl; uzl]
 * (nprob x m) and the gradients dL/d(input), with w_i = Fi ux, v_i = pi_i o (w_i - pi_i'w_i) and uz_0 = 0:
 *     dg: nprob x S (S = sum K), block i -(z_i v_i + uz_i pi_i);
 *     dF: per problem S x n column-major, ld S, as cvxb_batch_load_gp's F: block i dg_i x' - z_i pi_i ux';
 *     dG = -(zl ux' + uzl x')  (ml x n column-major per problem, the 'l' rows only),
 *     dA = -(y ux' + uy x')    (p x n column-major per problem);
 * dL/dh = uzl and dL/db = uy.  A monomial block (K_i = 1) gets exactly the QP adjoint's dG and dh of the row Fi x <= -gi.
 * Every array is in the caller's problem order and in `space`.  A NULL input is zero; a NULL output is not written and
 * its work is skipped: without dF, dg, dG and dA no gradient kernel runs.  A problem whose status is not 1 (optimal;
 * status 3 from a line-search step that underflowed included), or whose KKT matrix has no Cholesky factor at that
 * iterate, gets NaN in all its outputs.  The outputs are a function of the results and the data; cvxb_batch_results is
 * unchanged afterwards and a re-solve computes the same results.  GP batches only (cvxb_batch_create_gp): any other
 * batch is CVXB_E_UNSUP, and cvxb_batch_adjoint, _qcqp and _cone refuse a GP batch.  A batch without a completed
 * cvxb_batch_solve since its last cvxb_batch_load_gp or cvxb_batch_load_eq is CVXB_E_ARG.  CVXB_DEVICE allocates
 * nothing; CVXB_HOST stages each given array in temporary device memory, at most nprob * (2 (n + p + m) + S n + S +
 * ml n + p n) doubles in all. */
int cvxb_batch_adjoint_gp(cvxb_batch *b, const double *gx, const double *gy, const double *gz, double *ux, double *uy,
                          double *uz, double *dF, double *dg, double *dG, double *dA, int space);
/* Derivatives of a CP or cpl batch's last solve (cvxb_batch_create_cp, _cpl and _sdp_cpl: 'l', 'q' and 's' rows), for
 * a loss L with gradients gx = dL/dx (nprob x n), gy = dL/dy (nprob x p) and gz = dL/dz (nprob x m, m = mnl + ml,
 * laid out as the results' [znl; zl]).  At the returned iterate, with zk = [1; znl] for a CP batch (the objective's
 * multiplier z0 = 1, as the QCQP adjoint takes it) and zk = znl for a cpl batch, the batch's callback is called once
 * more, F(x, zk) on every problem, and gives H = sum_i zk_i grad² f_i and Df, the mnl x n matrix of rows grad f_i'
 * (i = 1..mnl).  With D = diag(s / z) on the nonlinear and 'l' rows and W'W the NT scaling of the returned s and z on
 * the 'q' and 's' rows (cvxb_batch_adjoint_cone's), it solves
 *     [H A' Df' G'; A 0 0 0; Df 0 -Dnl 0; G 0 0 -W'W] [ux; uy; uznl; uzl] = [gx; gy; gznl; gzl]
 * with one more factorisation of the reduced KKT matrix (S + A'A where S is singular there, as kkt_chol2 does) and one
 * step of iterative refinement on the full system, and writes ux (nprob x n), uy (nprob x p), uz = [uznl; uzl]
 * (nprob x m) and
 *     dG = -(zl ux' + uzl x')  (ml x n column-major per problem, the rows of G only),
 *     dA = -(y ux' + uy x')    (p x n column-major per problem);
 * dL/dh = uzl, dL/db = uy and, for a cpl batch, dL/dc = -ux.  An 's' block follows cvxb_batch_adjoint_cone: only the
 * symmetric part of gz's block enters, and both triangles of uz's and dG's block hold the same value.  For a
 * parameter t of F the caller forms dL/dt = -d_t[ux' Df(x; t)' zk + uk' f(x; t)] with uk = [0; uznl] (cpl: uznl),
 * x, z, ux and uz held constant, so uz's nonlinear rows are needed for that.  Every array is in the caller's problem
 * order and in `space`.  A NULL input is zero; a NULL output is not written: without dG and dA no gradient kernel
 * runs.  A problem whose status is not 1, whose F(x, zk) has a non-finite entry in f, Df or H's lower triangle, or
 * whose KKT matrix has no Cholesky factor at that iterate, gets NaN in all its outputs.  A callback that returns
 * nonzero makes the call CVXB_E_ARG, with the solver's state as the solve left it.  cvxb_batch_results is unchanged
 * afterwards and a re-solve computes the same results.  CP and cpl batches only: any other batch, a QCQP batch
 * included, is CVXB_E_UNSUP, and cvxb_batch_adjoint, _qcqp, _cone and _gp refuse CP and cpl batches.  A batch
 * without a completed cvxb_batch_solve since its last load is CVXB_E_ARG.  CVXB_DEVICE allocates nothing;
 * CVXB_HOST stages each given array in temporary device memory, at most nprob * (2 (n + p + m) + ml n + p n)
 * doubles in all. */
int cvxb_batch_adjoint_cp(cvxb_batch *b, const double *gx, const double *gy, const double *gz, double *ux, double *uy,
                          double *uz, double *dG, double *dA, int space);

/* Forward-mode derivatives (tangents) of a batch's last solve: how x, y and z move when the data move along a
 * direction d.  At the returned iterate, with the matrix M that the matching adjoint solves with (its scaling, H, Df
 * and D), they solve M [dx; dy; dz] = r(d) with the same factorisation, solves and refinement step as the adjoint,
 * and write dx (nprob x n), dy (nprob x p) and dz (nprob x m, on the nonlinear kinds [dznl; dzl] laid out as the
 * results' z).  With sym(X) = (X + X') / 2, r(d) is
 *     QP, cone QP and cone LP (P = 0, q = c):  rx = -(sym(dP) x + dq + dA'y + dG'z),  ry = db - dA x,  rz = dh - dG x;
 *     QCQP, zk = [1; znl]:  rx = -(sum_{i=0..mnl} zk_i (sym(dPi) x + dqi) + dA'y + dG'zl),
 *                           rznl_i = -(x'dPi x / 2 + dqi'x + dri),  ry and rzl as above;
 *     GP, z_0 = 1, pi_i = softmax(Fi x + gi), Sigma_i = diag(pi_i) - pi_i pi_i', w_i = dFi x + dgi:
 *                           rx = -(sum_{i=0..mnl} z_i (dFi'pi_i + Fi'Sigma_i w_i) + dA'y + dG'zl), rznl_i = -pi_i'w_i;
 *     CP and cpl:  rx = -(dc + tx + dA'y + dG'zl),  rznl = -tf,  with the caller's terms of F's parameters t at the
 *                  returned x, x and z held constant: tx = d_t[Df(x; t)' zk] dt (nprob x n) and tf = d_t[f_nl(x; t)] dt
 *                  (nprob x mnl), zk = [1; znl] for cp and znl for cpl; dc on a cpl batch only.
 * Every input has the layout of the matching load call, in the caller's problem order: P, G, A and F column-major per
 * problem, a QCQP's dP the (mnl + 1) n x n stack and dq (mnl + 1) x n, dG the rows of G only (ml rows on the
 * nonlinear kinds), a cone LP's dc in dq.  M is symmetric, so for every g, <g, (dx, dy, dz)> = <adjoint(g), d> with
 * the entrywise pairing of the adjoint's outputs with d, for any d: a non-symmetric dP, and 's' blocks of dh and of
 * dG's columns, enter through their symmetric parts, and dz's 's' blocks are symmetric.  The contract is the matching
 * adjoint's: a NULL input is zero and a NULL output is not written; a problem whose status is not 1, whose
 * factorisation fails there or (CP) whose F(x, zk) is not finite gets NaN in all its outputs; a failing callback makes
 * the call CVXB_E_ARG; cvxb_batch_results is unchanged afterwards and a re-solve computes the same results.
 * cvxb_batch_tangent takes every batch cvxb_batch_adjoint_cone takes (dP NULL on a cone LP, else CVXB_E_ARG);
 * _qcqp QCQP batches, _gp GP batches and _cp CP, cpl and sdp cpl batches (dc NULL on a CP batch, else CVXB_E_ARG).
 * Another kind is CVXB_E_UNSUP, and a batch without a completed cvxb_batch_solve since its last load CVXB_E_ARG.
 * r is formed in the outputs, so CVXB_DEVICE with dx, dy and dz given allocates nothing (a NULL output's part of r
 * takes temporary device memory); CVXB_HOST stages each given array in temporary device memory. */
int cvxb_batch_tangent(cvxb_batch *b, const double *dP, const double *dq, const double *dG, const double *dh,
                       const double *dA, const double *db, double *dx, double *dy, double *dz, int space);
int cvxb_batch_tangent_qcqp(cvxb_batch *b, const double *dP, const double *dq, const double *dr, const double *dG,
                            const double *dh, const double *dA, const double *db, double *dx, double *dy, double *dz,
                            int space);
int cvxb_batch_tangent_gp(cvxb_batch *b, const double *dF, const double *dg, const double *dG, const double *dh,
                          const double *dA, const double *db, double *dx, double *dy, double *dz, int space);
int cvxb_batch_tangent_cp(cvxb_batch *b, const double *dc, const double *tx, const double *tf, const double *dG,
                          const double *dh, const double *dA, const double *db, double *dx, double *dy, double *dz,
                          int space);

#ifdef __cplusplus
}
#endif
#endif /* CVXOPT_B200_H */
