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
    """normwise backward error of a solve with A = L L' <= c n u max(1, kappa); returns (error / bound, error)"""
    n = A.shape[0]
    eta = backward_error(A, x, b)
    bound = c * n * EPS * max(1.0, kappa)
    assert eta <= bound, (eta, bound)
    return eta / bound, eta
