"""Checks of fp64 dense kernels against an 80-bit long double evaluation of the same operation.

Each checker recomputes the exact-ish result in long double (64-bit mantissa, 2^11 times finer than fp64) and
compares the fp64 result with a deterministic rounding-error bound, so a failure means the kernel is wrong, not
unlucky.  Large operands are checked on sampled columns around the 128-wide block edges of the kernels.  Every
checker returns the largest error / bound it saw (1.0 is the bound) so that callers can report the margin."""
import numpy as np

EPS = 2.0 ** -53                  # unit roundoff of fp64
NB = 128                          # diagonal-block size of the Cholesky and the triangular solves
LD = np.longdouble


def block_edge_cols(n):
    """columns next to the 8- and 128-wide block edges, the middle and the last columns"""
    cand = {0, 1, 7, 8, 127, 128, 129, 255, 256, n // 2, n - 129, n - 128, n - 2, n - 1}
    return sorted(c for c in cand if 0 <= c < n)


def check_bound(err, bound):
    """max err / bound; a NaN or an err above bound fails"""
    bad = ~(err <= bound)
    if np.any(bad):
        i = np.flatnonzero(np.ravel(bad))[0]
        raise AssertionError("error %r above bound %r at flat index %d (%d entries over)"
                             % (float(np.ravel(err)[i]), float(np.ravel(bound)[i]), i, int(np.sum(bad))))
    with np.errstate(invalid="ignore", divide="ignore"):
        r = np.where(bound > 0, err / np.where(bound > 0, bound, 1), 0)
    return float(np.max(r)) if r.size else 0.0


def check_sums(got, ref, mag, nterms):
    """|got - ref| <= (nterms + 2) u mag entrywise: the bound of an fp64 sum of `nterms` products whose absolute
    values sum to `mag`, with a scaling and one more addition (ref, mag in long double)"""
    err = np.abs(np.asarray(got, dtype=LD) - ref)
    return check_bound(err, (nterms + 2) * EPS * mag)


def check_syrk(A, w, H, C, cols):
    """columns `cols` of the lower triangle of C = A' diag(w) A + H (A: k x n)"""
    k, n = A.shape
    Aw = A * (w[:, None] if w is not None else 1.0)        # fl(w * a) in fp64 first, like the kernels
    AL, AwL = A.astype(LD), Aw.astype(LD)
    worst = 0.0
    for j in cols:
        ref = AL[:, j:].T @ AwL[:, j]
        mag = np.abs(AL[:, j:]).T @ np.abs(AwL[:, j])
        if H is not None:
            ref = ref + H[j:, j].astype(LD)
            mag = mag + np.abs(H[j:, j]).astype(LD)
        worst = max(worst, check_sums(C[j:, j], ref, mag, k))
    return worst


def check_gemm(opA, opB, alpha, beta, C0, C, cols=None):
    """C = alpha op(A) op(B) + beta C0 on columns `cols` (all by default): the bound
    (k + 2) u (|alpha| |op(A)| |op(B)| + |beta| |C0|) per entry.  beta == 0 ignores C0 (BLAS: C0 may be NaN)."""
    k = opA.shape[1]
    cols = range(C.shape[1]) if cols is None else cols
    AL = opA.astype(LD)
    worst = 0.0
    for j in cols:
        b = opB[:, j].astype(LD)
        ref = LD(alpha) * (AL @ b) if k else np.zeros(C.shape[0], dtype=LD)
        mag = abs(LD(alpha)) * (np.abs(AL) @ np.abs(b)) if k else np.zeros(C.shape[0], dtype=LD)
        if beta != 0.0:
            ref = ref + LD(beta) * C0[:, j].astype(LD)
            mag = mag + abs(LD(beta)) * np.abs(C0[:, j]).astype(LD)
        worst = max(worst, check_sums(C[:, j], ref, mag, k))
    return worst


def diag_block_kappa(L):
    """largest 2-norm condition number of the 128 x 128 diagonal blocks of the lower triangular L"""
    n = L.shape[0]
    kap = 1.0
    for j in range(0, n, NB):
        B = np.tril(L[j:j + NB, j:j + NB])
        kap = max(kap, float(np.linalg.cond(B)))
    return kap


def check_potrf(A, L, cols, c=1.0, kappa=None):
    """Cholesky backward error on columns `cols`: |A - L L'| <= c (n + 2) u max(1, kappa) |L| |L'| entrywise in
    the lower triangle, kappa the largest condition number of L's diagonal blocks (default: computed).  For a
    plain Cholesky the bound without kappa holds (Higham, Thm 10.3: gamma_{n+1}); the blocked factorisation
    here forms the panel as A21 inv(L11)', whose residual carries kappa(L11).  Only L's lower triangle is read."""
    n = A.shape[0]
    L = np.tril(L)
    kap = max(1.0, diag_block_kappa(L) if kappa is None else kappa)
    LL = L.astype(LD)
    worst = 0.0
    for j in cols:
        Lr = LL[j:, :j + 1]
        lj = LL[j, :j + 1]
        ref = Lr @ lj
        mag = np.abs(Lr) @ np.abs(lj)
        err = np.abs(A[j:, j].astype(LD) - ref)
        worst = max(worst, check_bound(err, c * (n + 2) * EPS * kap * mag))
    return worst


def check_lower_only_written(before, after, off, n, lda):
    """flat buffers around an n x n matrix at element offset `off` with leading dimension lda: everything but the
    matrix's lower triangle (strict upper triangle, rows n..lda-1, the leading `off` elements) is bit-identical"""
    mask = np.ones(before.size, bool)
    for j in range(n):
        mask[off + j + j * lda:off + n + j * lda] = False
    same = np.asarray(before)[mask].view(np.uint64) == np.asarray(after)[mask].view(np.uint64)
    assert np.all(same), "%d elements outside the lower triangle changed" % int(np.sum(~same))


def backward_error(A, x, b):
    """||b - A x||_inf / (||A||_inf ||x||_inf + ||b||_inf) in long double"""
    AL = A.astype(LD)
    xl, bl = x.astype(LD), b.astype(LD)
    r = bl - AL @ xl
    nA = np.max(np.sum(np.abs(AL), axis=1))
    return float(np.max(np.abs(r)) / (nA * np.max(np.abs(xl)) + np.max(np.abs(bl))))


def check_potrs(A, x, b, kappa, c=1.0):
    """normwise backward error of a solve with A = L L' <= c (n + 2) u max(1, kappa); returns (error / bound, error).
    The residual is taken against A, so it includes the factorisation's own residual, whose bound check_potrf states
    as (n + 2) u max(1, kappa) |L| |L'|.  An earlier n u was below that and wrong for the smallest n: a 1 x 1 solve
    rounds the square root, the reciprocal and two products, and showed a backward error of 1.3 u."""
    n = A.shape[0]
    eta = backward_error(A, x, b)
    bound = c * (n + 2) * EPS * max(1.0, kappa)
    assert eta <= bound, (eta, bound)
    return eta / bound, eta


def check_trsv(L, x, b, trans, kappa, c=1.0):
    """triangular solve op(L) x = b (op(L) = L for 'N', L' for 'T'; only L's lower triangle is read): normwise
    backward error ||b - op(L) x||_inf / (||op(L)||_inf ||x||_inf + ||b||_inf) <= c n u max(1, kappa), kappa =
    diag_block_kappa(L).  The blocked solves form each block of x as inv(L_ii) t, so the residual carries kappa(L_ii)
    as in check_potrs.  Returns error / bound."""
    n = L.shape[0]
    Lt = np.tril(L)
    eta = backward_error(Lt.T if trans == "T" else Lt, x, b)
    bound = c * n * EPS * max(1.0, kappa)
    assert eta <= bound, (trans, eta, bound)
    return eta / bound


def check_trsm(L, X, B, kappa, c=1.0):
    """X = L^{-1} B column by column, each within check_trsv's bound; returns the largest error / bound"""
    return max((check_trsv(L, X[:, j], B[:, j], "N", kappa, c) for j in range(B.shape[1])), default=0.0)


def check_gemv(trans, A, w, x, alpha, beta, y0, y):
    """'T': y = alpha A' (w .* x) + beta y0 with fl(w .* x) formed in fp64 first, like the kernel: a sum of nrows
    products (nterms = nrows).  'N': y = alpha w .* (A x) + beta y0 with the weight applied after the sum of ncols
    products, one more rounding (nterms = ncols + 1).  Entrywise (nterms + 2) u (|alpha| |op(A)| |w x| + |beta| |y0|)
    (check_sums).  beta == 0 ignores y0 (it may be NaN).  Returns error / bound."""
    nrows, ncols = A.shape
    AL = A.astype(LD)
    if trans == "T":
        xw = x * w if w is not None else x                     # fp64 product, as the kernel forms it
        ref = LD(alpha) * (AL.T @ xw.astype(LD))
        mag = abs(LD(alpha)) * (np.abs(AL.T) @ np.abs(xw).astype(LD))
        nterms = nrows
    else:
        wl = w.astype(LD) if w is not None else LD(1)
        ref = LD(alpha) * wl * (AL @ x.astype(LD))
        mag = abs(LD(alpha)) * np.abs(wl) * (np.abs(AL) @ np.abs(x).astype(LD))
        nterms = ncols + 1
    if beta != 0.0:
        ref = ref + LD(beta) * y0.astype(LD)
        mag = mag + abs(LD(beta)) * np.abs(y0).astype(LD)
    return check_sums(y, ref, mag, nterms)


def check_qscale(v, beta, x, y, inverse):
    """y = W x (inverse False) or W^{-1} x for one second-order cone of order m, W = beta (2 v v' - J), J = diag(1, -1,
    .., -1), so W x = beta (2 v (v'x) - J x) and W^{-1} x = (1/beta) (2 J v (v' J x) - J x).  x may have several
    columns (m x xc).

    Bound, per entry i, to first order in u: the kernel forms s = v' (+-x) with an error of at most m u |v|'|x|, t = 2s
    exactly, fl(v_i t) (one rounding), fl(+-x_i + v_i t) (one), and the product with b = beta or fl(1/beta) (one, and
    one for fl(1/beta)).  With b the exact beta^{+-1} and M_i = |x_i| + 2 |v_i| |v|'|x|,
        |y_i - exact_i| <= (m + 4) u b M_i.
    Returns error / bound."""
    m = v.shape[0]
    X = x.reshape(m, -1).astype(LD)
    vl = v.astype(LD)
    J = -np.ones(m, dtype=LD)
    J[0] = 1
    Jx = X * J[:, None]
    b = LD(1) / LD(beta) if inverse else LD(beta)
    if inverse:
        ref = b * (2 * (J * vl)[:, None] * (vl @ Jx)[None, :] - Jx)
    else:
        ref = b * (2 * vl[:, None] * (vl @ X)[None, :] - Jx)
    mag = np.abs(X) + 2 * np.abs(vl)[:, None] * (np.abs(vl) @ np.abs(X))[None, :]
    err = np.abs(y.reshape(m, -1).astype(LD) - ref)
    return check_bound(err, (m + 4) * EPS * abs(b) * mag)
