"""The long-double checkers of tests/ld_check.py (used by the dense-kernel GPU tests) on LAPACK / BLAS results:
unmodified results pass, and results wrong by about 1e-12 relative in one entry, or written where they must not
be, fail.  This is what makes a passing GPU test mean something."""
import numpy as np
import pytest
import scipy.linalg.blas as blas
import scipy.linalg.lapack as lapack

from ld_check import (backward_error, block_edge_cols, check_gemm, check_lower_only_written, check_potrf,
                      check_potrs, diag_block_kappa)


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
