"""The long-double checkers of tests/ld_check.py (used by the dense-kernel GPU tests) on LAPACK / BLAS results:
unmodified results pass, and results wrong by about 1e-12 relative in one entry, or written where they must not
be, fail.  This is what makes a passing GPU test mean something."""
import numpy as np
import pytest
import scipy.linalg.blas as blas
import scipy.linalg.lapack as lapack

from ld_check import (backward_error, block_edge_cols, check_gemm, check_gemv, check_lower_only_written, check_potrf,
                      check_potrs, check_qscale, check_trsm, check_trsv, diag_block_kappa)


def _spd(n, seed):
    rng = np.random.Generator(np.random.PCG64(seed))
    B = rng.standard_normal((n, n))
    return B @ B.T / n + np.eye(n)


def test_potrf_checker_passes_lapack_and_fails_a_perturbed_tile():
    n = 300
    A = _spd(n, 1)
    L, info = lapack.dpotrf(A, lower=1, clean=1)
    assert info == 0
    cols = block_edge_cols(n)
    kap = diag_block_kappa(L)
    assert check_potrf(A, L, cols, kappa=kap) < 0.1
    # one entry of an off-diagonal 128 x 128 tile, 1e-12 relative, in a sampled column
    for i, j in ((200, 0), (257, 129), (299, 150)):
        Lp = L.copy()
        Lp[i, j] *= 1 + 1e-12
        with pytest.raises(AssertionError):
            check_potrf(A, Lp, cols, kappa=kap)


def test_lower_only_checker_fails_a_touched_upper_triangle():
    n = 129
    A = _spd(n, 2)
    buf = np.asfortranarray(np.where(np.tri(n, dtype=bool), A, np.nan))   # strict upper triangle: NaN
    before = buf.ravel(order="F").copy()
    L, info = lapack.dpotrf(buf, lower=1, clean=0)      # LAPACK reads and writes the lower triangle only
    assert info == 0
    check_lower_only_written(before, L.ravel(order="F"), 0, n, n)
    Lc, _ = lapack.dpotrf(buf, lower=1, clean=1)        # clean=1 zeroes the upper triangle
    with pytest.raises(AssertionError):
        check_lower_only_written(before, Lc.ravel(order="F"), 0, n, n)
    # a padded buffer (offset 1, lda = n + 2): one write into row n fails
    lda = n + 2
    pad = np.full(1 + lda * n, np.nan)
    after = pad.copy()
    for j in range(n):
        after[1 + j + j * lda:1 + n + j * lda] = L[j:, j]
    check_lower_only_written(pad, after, 1, n, lda)
    after[1 + n + 5 * lda] = 0.0
    with pytest.raises(AssertionError):
        check_lower_only_written(pad, after, 1, n, lda)


def test_potrs_checker_passes_lapack_and_fails_a_wrong_solution():
    n = 300
    A = _spd(n, 3)
    L, _ = lapack.dpotrf(A, lower=1, clean=1)
    b = np.random.Generator(np.random.PCG64(4)).standard_normal(n)
    x, info = lapack.dpotrs(L, b, lower=1)
    assert info == 0
    kap = diag_block_kappa(L)
    ratio, eta = check_potrs(A, x, b, kap)
    assert ratio < 0.1 and eta == backward_error(A, x, b)
    x[37] *= 1 + 1e-9
    with pytest.raises(AssertionError):
        check_potrs(A, x, b, kap)


@pytest.mark.parametrize("k", [1, 17, 300])
def test_gemm_checker_passes_blas_and_fails_a_perturbed_entry(k):
    rng = np.random.Generator(np.random.PCG64(k))
    m, n = 129, 65
    A, B, C0 = rng.standard_normal((m, k)), rng.standard_normal((k, n)), rng.standard_normal((m, n))
    C = blas.dgemm(0.7, A, B, -0.3, np.asfortranarray(C0))
    check_gemm(A, B, 0.7, -0.3, C0, C)
    C[64, 31] *= 1 + (1e-12 if k < 300 else 1e-11)
    with pytest.raises(AssertionError):
        check_gemm(A, B, 0.7, -0.3, C0, C)
    # beta = 0: C0 is not read, NaN in it is fine; NaN in the result is not
    Cz = blas.dgemm(1.0, A, B)
    check_gemm(A, B, 1.0, 0.0, np.full((m, n), np.nan), Cz)
    Cz[3, 3] = np.nan
    with pytest.raises(AssertionError):
        check_gemm(A, B, 1.0, 0.0, None, Cz)


@pytest.mark.parametrize("trans", ["N", "T"])
def test_trsv_checker_passes_blas_and_fails_a_wrong_solution(trans):
    n = 300
    A = _spd(n, 5)
    L, _ = lapack.dpotrf(A, lower=1, clean=1)
    kap = diag_block_kappa(L)
    b = np.random.Generator(np.random.PCG64(6)).standard_normal(n)
    x = blas.dtrsv(L, b, lower=1, trans=int(trans == "T"))
    assert check_trsv(L, x, b, trans, kap) < 0.1
    # the strict upper triangle is not read: garbage there changes nothing
    assert check_trsv(L + np.triu(np.full((n, n), 1e3), 1), x, b, trans, kap) < 0.1
    for i in (0, 37, 128, n - 1):
        xp = x.copy()
        xp[i] *= 1 + 1e-9
        with pytest.raises(AssertionError):
            check_trsv(L, xp, b, trans, kap)
    # solving with the other triangle is caught
    with pytest.raises(AssertionError):
        check_trsv(L, blas.dtrsv(L, b, lower=1, trans=int(trans != "T")), b, trans, kap)


def test_trsm_checker_passes_blas_and_fails_a_perturbed_column():
    n, ncols = 257, 65
    A = _spd(n, 7)
    L, _ = lapack.dpotrf(A, lower=1, clean=1)
    kap = diag_block_kappa(L)
    B = np.random.Generator(np.random.PCG64(8)).standard_normal((n, ncols))
    X = blas.dtrsm(1.0, L, B, lower=1)
    assert check_trsm(L, X, B, kap) < 0.1
    for i, j in ((0, 0), (130, 31), (n - 1, ncols - 1)):
        Xp = X.copy()
        Xp[i, j] *= 1 + 1e-9
        with pytest.raises(AssertionError):
            check_trsm(L, Xp, B, kap)


def _gemv_ld(trans, A, w, x, alpha, beta, y0):
    """the exact result rounded once to fp64 (the weighted forms, which BLAS has no call for)"""
    LD = np.longdouble
    if trans == "T":
        xw = x * w if w is not None else x
        r = LD(alpha) * (A.astype(LD).T @ xw.astype(LD))
    else:
        r = LD(alpha) * (w.astype(LD) if w is not None else LD(1)) * (A.astype(LD) @ x.astype(LD))
    if beta != 0.0:
        r = r + LD(beta) * y0.astype(LD)
    return r.astype(np.float64)


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("trans", ["N", "T"])
def test_gemv_checker_passes_blas_and_fails_a_perturbed_entry(trans, weighted):
    rng = np.random.Generator(np.random.PCG64(9 + weighted))
    nrows, ncols = 129, 65
    A = rng.standard_normal((nrows, ncols))
    w = 10.0 ** rng.uniform(-4, 4, nrows) if weighted else None
    x = rng.standard_normal(nrows if trans == "T" else ncols)
    y0 = rng.standard_normal(ncols if trans == "T" else nrows)
    if weighted:
        y = _gemv_ld(trans, A, w, x, 0.7, -0.3, y0)
    else:
        y = blas.dgemv(0.7, A, x, -0.3, y0.copy(), trans=int(trans == "T"))
    assert check_gemv(trans, A, w, x, 0.7, -0.3, y0, y) < 0.5
    for i in np.argsort(-np.abs(y))[:3]:                # the largest entries: no cancellation to hide behind
        yp = y.copy()
        yp[i] *= 1 + 1e-12
        with pytest.raises(AssertionError):
            check_gemv(trans, A, w, x, 0.7, -0.3, y0, yp)
    # beta = 0: y0 is not read, NaN in it is fine; NaN in the result is not
    y1 = _gemv_ld(trans, A, w, x, -1.0, 0.0, None)
    check_gemv(trans, A, w, x, -1.0, 0.0, np.full(y0.size, np.nan), y1)
    y1[3] = np.nan
    with pytest.raises(AssertionError):
        check_gemv(trans, A, w, x, -1.0, 0.0, None, y1)


@pytest.mark.parametrize("inverse", [False, True])
def test_qscale_checker_passes_long_double_and_fails_a_perturbed_entry(inverse):
    rng = np.random.Generator(np.random.PCG64(11 + inverse))
    m, xc = 65, 4
    u = rng.standard_normal(m - 1)
    v = np.r_[np.sqrt(1.0 + u @ u), u]            # on the hyperboloid v' J v = 1
    beta = 7.3
    x = rng.standard_normal((m, xc))
    LD = np.longdouble
    J = np.r_[1.0, -np.ones(m - 1)].astype(LD)
    vl, X = v.astype(LD), x.astype(LD)
    if inverse:
        y = ((2 * (J * vl)[:, None] * (vl @ (X * J[:, None]))[None, :] - X * J[:, None]) / LD(beta)).astype(np.float64)
    else:
        y = (LD(beta) * (2 * vl[:, None] * (vl @ X)[None, :] - X * J[:, None])).astype(np.float64)
    assert check_qscale(v, beta, x, y, inverse) < 0.1
    # W and W^{-1} are inverses: the forward result is not the inverse one
    with pytest.raises(AssertionError):
        check_qscale(v, beta, x, y, not inverse)
    for i, j in ((0, 0), (1, 1), (m - 1, xc - 1)):
        yp = y.copy()
        yp[i, j] *= 1 + 1e-12
        with pytest.raises(AssertionError):
            check_qscale(v, beta, x, yp, inverse)
