"""cvxb_potrf above 4096 (the eager path) against long double, where the trailing matrix is updated in groups of
four panels: block columns kGroup (q + 2) and beyond receive group q as one K = 512 update, the columns before them
per panel.  The sizes give 16 full groups (8192, 8193) and a last group with one panel (7850, 62 blocks); the
sampled columns sit at block edges reached only by per-panel updates (< 1024) and only by grouped ones."""
import numpy as np
import pytest
import scipy.linalg

from ld_check import NB, check_lower_only_written, check_potrf, diag_block_kappa

pytestmark = pytest.mark.gpu


def _lib():
    from cvxopt_b200 import _lib as L
    return L, L.load()


def _spd(n, seed):
    """symmetric Gaussian scaled to spectrum [-1, 1], plus 2 I: SPD, condition ~3, O(n^2) on the host"""
    rng = np.random.Generator(np.random.PCG64(seed))
    B = rng.standard_normal((n, n))
    return (B + B.T) / (2.0 * np.sqrt(2.0 * n)) + 2.0 * np.eye(n)


def _cols(n):
    cand = {0, 127, 128, 511, 512, 1023, 1024, 1151, 2047, 2048, 4095, 4096, 6143, 6144, n - 129, n - 128, n - 1}
    return sorted(c for c in cand if 0 <= c < n)


@pytest.mark.parametrize("n,lda", [(8192, 8192), (8192, 8195), (8193, 8193), (7850, 7851)])
def test_grouped_potrf_matches_long_double(n, lda):
    """L against long double on the sampled columns, NaN in the strict upper triangle and in rows n..lda-1 comes
    back bit for bit, work_inv is finite, and a second run gives the same bits"""
    import torch
    L, lib = _lib()
    A = _spd(n, n + lda)
    view = np.full((n, lda), np.nan)                    # column-major: view[c, r] = A[r, c]
    T = A.T.copy()
    T[np.tri(n, k=-1, dtype=bool)] = np.nan             # strict upper triangle of A
    view[:, :n] = T
    buf = view.ravel()
    nblk = (n + NB - 1) // NB
    dA = torch.from_numpy(buf).cuda()
    dinv = torch.full((2 * nblk * NB * NB,), float("nan"), dtype=torch.float64, device="cuda")
    assert lib.cvxb_potrf(n, dA.data_ptr(), lda, dinv.data_ptr(), 0) == 0, L.last_error()
    out = dA.cpu().numpy()
    assert np.all(np.isfinite(dinv.cpu().numpy()))
    dA.copy_(torch.from_numpy(buf))
    assert lib.cvxb_potrf(n, dA.data_ptr(), lda, dinv.data_ptr(), 0) == 0, L.last_error()
    assert np.array_equal(dA.cpu().numpy().view(np.uint64), out.view(np.uint64)), "L differs between runs"
    check_lower_only_written(buf, out, 0, n, lda)
    Lh = out.reshape(n, lda)[:, :n].T
    kap = diag_block_kappa(Lh)
    r = check_potrf(A, Lh, _cols(n), kappa=kap)
    print("\npotrf n=%d lda=%d: %.3g of the bound (kappa %.3g)" % (n, lda, r, kap))


@pytest.mark.parametrize("n", [8192, 7850])
def test_grouped_potrf_info_names_the_first_bad_minor(n):
    """A = L0 L0' with A[k,k] -= 2 L0[k,k]^2 returns k + 1 (LAPACK's info), for k in block columns that receive
    grouped updates (block 8 and beyond) and in the last column; a positive definite matrix afterwards returns 0"""
    import torch
    L, lib = _lib()
    S = _spd(n, 3 * n)
    L0 = scipy.linalg.cholesky(S, lower=True)
    nblk = (n + NB - 1) // NB
    dA = torch.empty(n * n, dtype=torch.float64, device="cuda")
    dinv = torch.empty(2 * nblk * NB * NB, dtype=torch.float64, device="cuda")
    for k in (8 * NB, 8 * NB + 77, 40 * NB + 127, n - 1):
        A = S.copy()
        A[k, k] -= 2.0 * L0[k, k] ** 2
        dA.copy_(torch.from_numpy(A.ravel(order="F")))
        got = lib.cvxb_potrf(n, dA.data_ptr(), n, dinv.data_ptr(), 0)
        assert got == k + 1, (k, got)
        assert ("order %d" % (k + 1)) in L.last_error()
    dA.copy_(torch.from_numpy(S.ravel(order="F")))
    assert lib.cvxb_potrf(n, dA.data_ptr(), n, dinv.data_ptr(), 0) == 0
