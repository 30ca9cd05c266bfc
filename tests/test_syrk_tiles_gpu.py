"""The fp64 SYRK C = A' diag(w) A + H (C-ABI cvxb_syrk_scaled) on its tile shapes: the 128x128 TMA kernel for even,
16-byte aligned leading dimensions, dmma_gemm_kernel for odd ones.  Checked against an 80-bit long double evaluation of
the same sums with the deterministic bound of an fp64 sum of K products, (K + 2) 2^-53 sum|terms|."""
import numpy as np
import pytest

from ld_check import check_syrk as _check                 # columns of C's lower triangle against long double

pytestmark = pytest.mark.gpu


def _run(n, k, lda, w, H, seed):
    """A (k x n, column-major, leading dimension lda) with the given w / H; returns (A, C) with C's lower triangle"""
    import torch
    from cvxopt_b200 import _lib
    lib = _lib.load()
    rng = np.random.Generator(np.random.PCG64(seed))
    A = rng.standard_normal((k, n))
    buf = np.full((n, lda), np.nan)
    buf[:, :k] = A.T                                       # column j of A at j * lda, padding never read
    dA = torch.from_numpy(buf).cuda()
    dw = torch.from_numpy(w.copy()).cuda() if w is not None else None
    dH = torch.from_numpy(np.ascontiguousarray(H.T)).cuda() if H is not None else None
    dC = torch.full((n, n), float("nan"), dtype=torch.float64, device="cuda")
    rc = lib.cvxb_syrk_scaled(n, k, dA.data_ptr(), lda, dw.data_ptr() if dw is not None else None,
                              dH.data_ptr() if dH is not None else None, n, dC.data_ptr(), n, 0)
    assert rc == 0, _lib.last_error()
    return A, dC.cpu().numpy().T


def _inputs(n, k, with_w, with_H, seed):
    rng = np.random.Generator(np.random.PCG64(seed + 7))
    w = np.exp(2.0 * rng.standard_normal(k)) if with_w else None
    H = None
    if with_H:
        B = rng.standard_normal((n, n))
        H = np.asfortranarray(B + B.T)
    return w, H


def _cols(n):
    if n <= 300:
        return range(n)
    return sorted({0, 1, 127, 128, 129, n // 2, n - 129, n - 128, n - 2, n - 1})


@pytest.mark.parametrize("k", [1, 15, 17, 1000, 4100])
@pytest.mark.parametrize("n", [1, 127, 129, 300, 1000])
def test_syrk_scaled_matches_long_double(n, k):
    lda = k + (1 if k % 2 else 2)                          # lda > k, even: the TMA kernel
    for with_w, with_H in ((True, True), (False, False)):
        w, H = _inputs(n, k, with_w, with_H, n + k)
        A, C = _run(n, k, lda, w, H, n * 31 + k)
        _check(A, w, H, C, _cols(n))


def test_syrk_scaled_mixed_w_h():
    for n, k, with_w, with_H in ((129, 17, True, False), (300, 1000, False, True)):
        w, H = _inputs(n, k, with_w, with_H, 3)
        A, C = _run(n, k, k, w, H, 4)
        _check(A, w, H, C, _cols(n))


def test_syrk_scaled_split_k_tail():
    """n = 2000: 136 lower 128x128 tiles on 132 SMs, so the last 4 tiles are split along K and reduced in order"""
    n, k = 2000, 2048
    w, H = _inputs(n, k, True, True, 11)
    A, C = _run(n, k, k, w, H, 12)
    _check(A, w, H, C, sorted({0, 5, 640, 1500, 1790, 1791, 1792, 1800, 1919, 1920, 1999}))


def test_syrk_scaled_odd_lda_fallback():
    """an odd leading dimension cannot be a TMA stride: dmma_gemm_kernel takes it, and without a split-K tail both
    kernels add the same products in the same order"""
    n, k = 300, 1000
    w, H = _inputs(n, k, True, True, 21)
    A, C = _run(n, k, k + 1, w, H, 22)
    _check(A, w, H, C, _cols(n))
    _, C2 = _run(n, k, k + 2, w, H, 22)
    il = np.tril_indices(n)
    assert np.array_equal(C[il], C2[il])


def test_syrk_scaled_device_bytes_unchanged():
    from cvxopt_b200 import _lib
    lib = _lib.load()
    w, H = _inputs(129, 1000, True, True, 31)
    _run(129, 1000, 1000, w, H, 32)                        # the per-device context exists from here on
    base = lib.cvxb_device_bytes()
    for n, k, lda in ((129, 1000, 1000), (300, 17, 18), (300, 1000, 1001), (2000, 2048, 2048)):
        w, H = _inputs(n, k, True, True, 33)
        _run(n, k, lda, w, H, 34)
    assert lib.cvxb_device_bytes() == base
