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


# ---------------------------------------------------------------------------------- semidefinite ('s') blocks
# A block is an ms x ms matrix; the batch kernels read only its lower triangle.  ms <= 32, so the long double
# references below are plain cyclic Jacobi methods (numpy.linalg has no long double).
LD_EPS = LD(np.finfo(LD).eps)


def sym_lower(X):
    """the symmetric matrix whose lower triangle is X's"""
    L = np.tril(np.asarray(X))
    return L + np.tril(L, -1).T


def ld_chol(A):
    """lower Cholesky factor of the symmetric A (lower triangle read) in long double"""
    A = sym_lower(np.asarray(A, dtype=LD))
    n = A.shape[0]
    L = np.zeros_like(A)
    for j in range(n):
        d = A[j, j] - L[j, :j] @ L[j, :j]
        assert d > 0, "ld_chol: not positive definite"
        L[j, j] = np.sqrt(d)
        L[j + 1:, j] = (A[j + 1:, j] - L[j + 1:, :j] @ L[j, :j]) / L[j, j]
    return L


def _round_robin(n):
    """the n - 1 (n even) or n (n odd) rounds of disjoint pairs that together visit every pair (i, j) once"""
    m = n + n % 2
    idx = list(range(m))
    rounds = []
    for _ in range(m - 1):
        pr = [(idx[k], idx[m - 1 - k]) for k in range(m // 2)]
        pr = [(min(p, q), max(p, q)) for p, q in pr if p < n and q < n]
        if pr:
            rounds.append((np.array([p for p, _ in pr]), np.array([q for _, q in pr])))
        idx = [idx[0]] + [idx[-1]] + idx[1:-1]
    return rounds


def _rot(x, y):
    """(c, s) with t = sign(x) / (|x| + sqrt(x^2 + 1)) the smaller root of t^2 + 2 x t - 1 = 0"""
    big = np.abs(x) > LD(1e30)
    xs = np.where(big, LD(1), x)
    t = np.where(big, 1 / (2 * np.where(big, x, LD(1))), np.copysign(LD(1), xs) / (np.abs(xs) + np.sqrt(xs * xs + 1)))
    t = np.where(y, t, LD(0))
    c = 1 / np.sqrt(t * t + 1)
    return c, c * t


def ld_eigh(A, sweeps=100):
    """(w ascending, V) of the symmetric A (lower triangle read) by cyclic two-sided Jacobi in long double, the pairs
    of a sweep in round-robin order (each round rotates disjoint pairs at once), until the off-diagonal mass is below
    long double's epsilon times ||A||_F: the eigenvalues are then within about 1e-19 ||A|| of exact, far inside any
    fp64 bound"""
    A = sym_lower(np.asarray(A, dtype=LD)).copy()
    n = A.shape[0]
    V = np.eye(n, dtype=LD)
    nrm = np.sqrt(np.sum(A * A))
    rounds = _round_robin(n)
    for _ in range(sweeps + 1):
        if np.sqrt(np.sum(np.tril(A, -1) ** 2)) <= LD_EPS * nrm:
            break
        assert _ < sweeps, "ld_eigh: no convergence in %d sweeps" % sweeps
        for P, Q in rounds:
            apq = A[P, Q]
            nz = apq != 0
            th = (A[Q, Q] - A[P, P]) / (2 * np.where(nz, apq, LD(1)))
            c, s = _rot(th, nz)
            for M in (A, V):
                mp, mq = M[:, P].copy(), M[:, Q].copy()
                M[:, P], M[:, Q] = c * mp - s * mq, s * mp + c * mq
            ap, aq = A[P, :].copy(), A[Q, :].copy()
            A[P, :], A[Q, :] = c[:, None] * ap - s[:, None] * aq, s[:, None] * ap + c[:, None] * aq
            A[P, Q] = 0
            A[Q, P] = 0
    w = np.diag(A).copy()
    o = np.argsort(w)
    return w[o], V[:, o]


def ld_svdvals(M, sweeps=100):
    """singular values (ascending) of M by one-sided (Hestenes) Jacobi in long double: rotate column pairs until each
    pair is orthogonal to long double's epsilon; the column norms are then the singular values, each to high relative
    accuracy when M is a product of triangular factors (no squaring of the condition number)"""
    U = np.array(M, dtype=LD)
    rounds = _round_robin(U.shape[1])
    for _ in range(sweeps):
        rot = False
        for P, Q in rounds:
            a, b = np.sum(U[:, P] ** 2, axis=0), np.sum(U[:, Q] ** 2, axis=0)
            g = np.sum(U[:, P] * U[:, Q], axis=0)
            go = np.abs(g) > LD_EPS * np.sqrt(a * b)
            if not np.any(go):
                continue
            rot = True
            zeta = (b - a) / (2 * np.where(go, g, LD(1)))
            c, s = _rot(zeta, go)
            up, uq = U[:, P].copy(), U[:, Q].copy()
            U[:, P], U[:, Q] = c * up - s * uq, s * up + c * uq
        if not rot:
            break
    else:
        raise AssertionError("ld_svdvals: no convergence in %d sweeps" % sweeps)
    return np.sort(np.sqrt(np.sum(U * U, axis=0)))


def _finite(*xs):
    for x in xs:
        assert np.all(np.isfinite(np.asarray(x, dtype=float))), "NaN or Inf in a result"


def check_sym_eig(A, V, w, c=1.0, parts=None):
    """A = V diag(w) V' for the symmetric A (lower triangle read), n = order, u = fp64's unit roundoff, p = 2 n + 8:
      - |V'V - I| <= 4 c p u entrywise (see below for the 4);
      - ||A - V diag(w) V'||_F <= c (p + 2 sqrt(n)) u ||A||_F;
      - |w_i - w*_i| <= c p u ||A||_2 after sorting, w* the long double eigenvalues (ld_eigh).
    A backward-stable symmetric eigensolver returns the exact decomposition of A + E with ||E|| <= p(n) u ||A|| and V
    orthogonal to p(n) u, p(n) linear in n: one plane rotation or reflector per column and stage, each exact to a few u
    (Demmel and Veselic for Jacobi; Higham, section 19.3, for Householder tridiagonalisation), and Weyl's theorem moves
    each eigenvalue by at most ||E||_2.  p = 2 n + 8: LAPACK's dsyevd and dsyev reach 2.5 n u on |V'V - I| and 2.4 n u
    on the residual at n = 5, where the few roundings of each rotation dominate, and at most 27 u (orthogonality),
    22 u (residual) and 13 u (eigenvalues) at n = 16 and 32 on the inputs of test_sblock_checks_cpu.py.  (dsyevr, whose
    MRRR vectors are orthogonal only to a larger multiple, reaches 740 u at n = 32 and is not the reference here.)
    Two terms are Jacobi's own (k_s_dir_post, k_s_eig_*):
      - the orthogonality bound is four times wider: two-sided Jacobi builds V from n - 1 rotations per column in each
        of its 5 to 10 sweeps, several times the transformations LAPACK applies, each changing the column's norm and
        inner products by a few u (its V measures up to 1.15 p u at n = 5 and 9).  A loss of orthogonality cannot hide
        a wrong decomposition: the residual is taken with V as it is;
      - the residual's 2 sqrt(n) u ||A||_F is what Jacobi leaves by design: jac_done accepts a block at rounding level
        once its off-diagonal mass is at most 2 u sqrt(n) ||A||_F (off^2 <= eps^2 n tot^2 with eps = 2 u), and the
        returned diagonal drops that mass.
    The residual bound, at most 83 u at n = 32, is meant to catch a Jacobi method that stops with off-diagonal mass
    1e-13 ||A||_F, about 900 u, which is what jac_done's stagnation exit would leave, at every order up to 32.  A
    column of V paired with the wrong w fails the residual too.  `parts`, a dict, collects each check's
    error / bound under 'orth', 'res' and 'eig'.  Returns the largest error / bound."""
    n = A.shape[0]
    _finite(V, w)
    AL = sym_lower(np.asarray(A, dtype=LD))
    VL, wl = np.asarray(V, dtype=LD), np.asarray(w, dtype=LD)
    pu = c * (2 * n + 8) * EPS
    got = {"orth": check_bound(np.abs(VL.T @ VL - np.eye(n, dtype=LD)), np.full((n, n), 4 * pu))}
    nrmf = np.sqrt(np.sum(AL * AL))
    R = AL - (VL * wl) @ VL.T
    got["res"] = check_bound(np.array([np.sqrt(np.sum(R * R))]), np.array([(pu + c * 2 * np.sqrt(n) * EPS) * nrmf]))
    ws = ld_eigh(AL)[0]
    nrm2 = np.max(np.abs(ws))
    got["eig"] = check_bound(np.abs(np.sort(wl) - ws), np.full(n, pu * nrm2))
    if parts is not None:
        for k, v in got.items():
            parts[k] = max(parts.get(k, 0.0), v)
    return max(got.values())


def check_min_eig(A, got, c=1.0):
    """the smallest eigenvalue of the symmetric A (lower triangle read) within c (2 n + 8) u ||A||_2 (check_sym_eig's
    Weyl bound) of the long double one"""
    n = A.shape[0]
    _finite([got])
    ws = ld_eigh(A)[0]
    return check_bound(np.array([abs(LD(got) - ws[0])]), np.array([c * (2 * n + 8) * EPS * np.max(np.abs(ws))]))


def _kappa(L):
    return max(1.0, float(np.linalg.cond(np.asarray(L, dtype=float))))


def check_nt_scaling(s, z, r, rti, lam, c=1.0, extra=0.0):
    """the Nesterov-Todd scaling of one block (misc.compute_scaling): r' z r = diag(lam), rti' s rti = diag(lam),
    r' rti = I, and lam the singular values of Lz' Ls (s = Ls Ls', z = Lz Lz').  r is unique up to rotations inside
    equal lam, so these defining properties are what is checked, not r itself.  s and z: lower triangles read.

    Bounds, with n the order, kz = max(1, kappa_2(Lz)), ks = max(1, kappa_2(Ls)) of the long double factors and d_x the
    vector sqrt(diag(x)):
      - The factorisations: for an SPD x, |x_ij| <= d_i d_j and a Cholesky's backward error is |dx| <= (n + 1) u |L||L'|
        <= (n + 1) u d d' (Higham Thm 10.3; |L||L'|_ij <= ||L_i|| ||L_j|| = d_i d_j).  So x enters through d d'.
      - r' z r = diag(lam) holds in exact arithmetic for any orthogonal U (r = Lz^{-T} U diag(lam)^{1/2}), so its error
        is that of U's orthogonality, z's factorisation and the solve with Lz'.  The computed r solves (Lz' + E) r =
        U diag(lam)^{1/2} with |E| <= n u |Lz'|, so r' z r = diag(lam) - r' E' Lz' r - r' Lz E r + O(u^2): each of the
        two factors of r carries n u, z's factorisation (n + 1) u, the scaling by sqrt(lam) and the square roots of
        the pivots 3 u more, all on |r'| |Lz| |Lz'| |r| <= (|r|' d_z)(d_z' |r|); no kz, since the residual, not the
        solution, is compared:  |r' z r - diag(lam)| <= c (3 n + 4) u (|r|' d_z)(d_z' |r|).
      - rti' s rti = diag(lam) holds when Lz' Ls = U diag(lam) V' exactly; rti = Lz U diag(lam)^{-1/2} is a sum of n
        products on each side, the SVD's backward error is columnwise relative for a one-sided Jacobi SVD and
        normwise for LAPACK's, and s's factorisation adds (n + 1) u, so the same count:
        |rti' s rti - diag(lam)| <= c (3 n + 4) u (|rti|' d_s)(d_s' |rti|).
      - r' rti = I: here the solve's error E enters as r' E' Lz^{-1} rti, whose (i, j) entry is at most
        ||r_i|| ||E|| ||Lz^{-1}|| ||rti_j|| <= n u kz ||r_i|| ||rti_j|| (columns r_i, rti_j); with the products that
        form rti and the scalings, |r' rti - I| <= c (3 n + 4) u kz ||r_i|| ||rti_j||.
      `extra` is added to c (3 n + 4) u in these three bounds: check_nt_update passes the departure of the previous
      scaling from r0' rti0 = I, which the update inherits.
      - lam against the long double singular values sig* of Lz*' Ls*: lam_i^2 are the eigenvalues of Ls' z Ls, which s's
        and z's factorisation errors move by a relative (n + 1) u (ks^2 + kz^2), so lam_i by half of that; the SVD's
        backward error adds n u sig*_max, the square roots 4 u more:
            |lam_i - sig*_i| <= c (n + 4) u ((ks^2 + kz^2) sig*_i / 2 + sig*_max)  (sorted).
    Returns the largest error / bound."""
    n = s.shape[0]
    _finite(r, rti, lam)
    sL, zL = sym_lower(np.asarray(s, dtype=LD)), sym_lower(np.asarray(z, dtype=LD))
    Ls, Lz = ld_chol(sL), ld_chol(zL)
    ks, kz = _kappa(Ls), _kappa(Lz)
    rL, tL, lL = (np.asarray(x, dtype=LD) for x in (r, rti, lam))
    ar, at = np.abs(rL), np.abs(tL)
    dz, ds = np.sqrt(np.diag(zL)), np.sqrt(np.diag(sL))
    D = np.diag(lL)
    mz, ms_ = ar.T @ dz, at.T @ ds
    nu = c * (3 * n + 4) * EPS + extra
    worst = check_bound(np.abs(rL.T @ zL @ rL - D), nu * np.outer(mz, mz))
    worst = max(worst, check_bound(np.abs(tL.T @ sL @ tL - D), nu * np.outer(ms_, ms_)))
    cr, ct = np.sqrt(np.sum(ar * ar, axis=0)), np.sqrt(np.sum(at * at, axis=0))
    worst = max(worst, check_bound(np.abs(rL.T @ tL - np.eye(n, dtype=LD)), nu * kz * np.outer(cr, ct)))
    sig = ld_svdvals(Lz.T @ Ls)
    bound = c * (n + 4) * EPS * ((ks * ks + kz * kz) * sig / 2 + sig[-1])
    return max(worst, check_bound(np.abs(np.sort(lL) - sig), bound))


def nt_update_ld(r0, rti0, lam0, Qs, sigs, Qz, sigz, step):
    """long double s+ = r0 L^1/2 Qs (I + step Ss) Qs' L^1/2 r0' and z+ = rti0 L^1/2 Qz (I + step Sz) Qz' L^1/2 rti0'
    (misc.update_scaling on the eigendecompositions coneprog leaves in ds and dz), with |A| |A'| for A = r0 L^1/2 Qs
    (I + step Ss)^1/2 (and likewise for z) as their magnitudes"""
    out = []
    for W, Q, sg in ((r0, Qs, sigs), (rti0, Qz, sigz)):
        h = np.sqrt(np.asarray(lam0, dtype=LD))
        g = 1 + LD(step) * np.asarray(sg, dtype=LD)
        F = h[:, None] * np.asarray(Q, dtype=LD)
        WL = np.asarray(W, dtype=LD)
        A = WL @ F
        ref = (A * g) @ A.T
        mag = (np.abs(WL) @ (np.abs(F) * np.sqrt(np.abs(g)))) @ (np.abs(WL) @ (np.abs(F) * np.sqrt(np.abs(g)))).T
        out += [ref, mag]
    return out


def check_nt_update(r0, rti0, lam0, Qs, sigs, Qz, sigz, step, s, z, r, rti, lam, c=1.0):
    """k_s_update / misc.update_scaling for one block: the returned s and z equal nt_update_ld's s+ and z+ within
    check_sums' bound for 4 n + 4 terms (the kernel forms r0 Ls, Lz' Ls, its SVD, r0 Ls V and r lam r', each a sum of n
    products, and a few scalings: sqrt(l_i) sqrt(l_j) sqrt(g_j / l_j)); s and z are exactly symmetric; and the returned
    (r, rti, lam) are the NT scaling of s+ and z+ (check_nt_scaling with 2 c: r = r0 Ls V lam^{-1/2} and rti = rti0 Lz U
    lam^{-1/2} reach s+ and z+ through the old scaling as well as the new factors, two congruences where
    compute_scaling has one).  The update multiplies the old scaling without restoring r0' rti0 = I, so s+ and z+ reach
    (r, rti) through r0' rti0 = I + E0 as well: each of the two congruences in r' z+ r, rti' s+ rti and r' rti is off by
    at most ||E0||_2 relative, and check_nt_scaling gets extra = 2 ||E0||_2 (E0 measured in long double from the
    inputs), which is how errors of a chain of updates add up.  Returns the largest error / bound."""
    n = s.shape[0]
    _finite(s, z, r, rti, lam)
    assert np.array_equal(np.asarray(s), np.asarray(s).T) and np.array_equal(np.asarray(z), np.asarray(z).T), \
        "s or z not exactly symmetric"
    sp, msp, zp, mzp = nt_update_ld(r0, rti0, lam0, Qs, sigs, Qz, sigz, step)
    worst = check_sums(s, sp, msp, 4 * n + 4)
    worst = max(worst, check_sums(z, zp, mzp, 4 * n + 4))
    E0 = np.asarray(r0, dtype=LD).T @ np.asarray(rti0, dtype=LD) - np.eye(n, dtype=LD)
    e0 = float(np.linalg.norm(np.asarray(E0, dtype=float), 2))
    return max(worst, check_nt_scaling(sp.astype(float), zp.astype(float), r, rti, lam, 2 * c, extra=2 * e0))


def pack_ld(X):
    """misc.pack of one block: the lower triangle by columns, off-diagonals times sqrt(2)"""
    n = X.shape[0]
    out = []
    for j in range(n):
        col = np.asarray(X[j:, j])
        out.append(np.concatenate([col[:1], col[1:] * (np.sqrt(LD(2)) if col.dtype == LD else np.sqrt(2.0))]))
    return np.concatenate(out)


def unpack(x, n):
    """misc.unpack of one packed block (fp64): the symmetric matrix, off-diagonals divided by sqrt(2)"""
    X = np.zeros((n, n))
    k = 0
    for j in range(n):
        X[j, j] = x[k]
        X[j + 1:, j] = x[k + 1:k + n - j] / np.sqrt(2.0)
        k += n - j
    return sym_lower(X)


def check_congruence(A, X, got, trans, packed=False, plus=None, c=1.0):
    """got = A' X A (trans) or A X A' (+ plus, a long double (ref, mag) pair added to the result) for the symmetric X
    (lower triangle read), got packed (misc.pack, off-diagonals times sqrt 2: one more rounding) or the full matrix.
    check_sums with nterms = 2 n + 1 (two sums of n products, the sqrt 2) times c, on |A'| |X| |A|.  Returns the largest
    error / bound."""
    n = A.shape[0]
    AL, XL = np.asarray(A, dtype=LD), sym_lower(np.asarray(X, dtype=LD))
    if trans:
        ref, mag = AL.T @ XL @ AL, np.abs(AL).T @ np.abs(XL) @ np.abs(AL)
    else:
        ref, mag = AL @ XL @ AL.T, np.abs(AL) @ np.abs(XL) @ np.abs(AL).T
    if plus is not None:
        ref, mag = ref + plus[0], mag + plus[1]
    if packed:
        ref, mag = pack_ld(ref), pack_ld(mag)
    return check_sums(got, ref, mag, c * (2 * n + 1))
