"""cvxb_potrf / cvxb_potrs / cvxb_gemm on device pointers against long double (tests/ld_check.py).

The Cholesky (potf2_inv_kernel, the panel TRSM as a GEMM with the diagonal-block inverse, the look-ahead trailing
update), the flag-chained triangular solves and the general dmma_gemm_kernel instantiations are checked
- on sizes around the 8- and 128-wide block edges, up to 4097 (one past the last size factored through a CUDA graph);
- with lda == n, an odd lda, an even lda > n and a base pointer that is 8- but not 16-byte aligned (the non-vector
  copy paths);
- with NaN in everything the call must neither read nor write (the strict upper triangle, rows n..lda-1, GEMM
  padding), which has to come back bit for bit;
- in the eager, graph-capture and graph-replay launch modes of potrf_lower, which must agree bit for bit.

Every check prints its largest error / bound (and LAPACK's, where it computes one) so that runs show the margin."""
import numpy as np
import pytest
import scipy.linalg.lapack as lapack

from ld_check import (EPS, NB, backward_error, block_edge_cols, check_bound, check_gemm, check_lower_only_written,
                      check_potrf, check_potrs, diag_block_kappa)

pytestmark = pytest.mark.gpu

SIZES = [1, 2, 7, 8, 9, 100, 127, 128, 129, 255, 256, 257, 385, 700, 1333, 4096, 4097]


def _lib():
    from cvxopt_b200 import _lib as L
    return L, L.load()


def _spd(n, seed):
    """well-conditioned SPD: B B'/n + I"""
    rng = np.random.Generator(np.random.PCG64(seed))
    B = rng.standard_normal((n, n))
    return B @ B.T / n + np.eye(n)


def _ipm(n, seed):
    """the late interior-point regime: P + G' diag(d)^2 G with d spanning 1e-4 .. 1e4"""
    rng = np.random.Generator(np.random.PCG64(seed))
    A0 = rng.standard_normal((n, n))
    G = rng.standard_normal((2 * n, n))
    d = 10.0 ** rng.uniform(-4, 4, 2 * n)
    Gd = G * d[:, None]
    S = A0.T @ A0 / n + np.eye(n) + Gd.T @ Gd
    return (S + S.T) / 2


def _poisoned(M, ld, off, lower_only):
    """flat host buffer: M (column-major, leading dimension ld) after `off` leading doubles, NaN everywhere else
    (and in M's strict upper triangle when lower_only)"""
    rows, cols = M.shape
    buf = np.full(off + ld * max(cols, 1), np.nan)
    view = buf[off:].reshape(max(cols, 1), ld)[:cols]
    if lower_only:
        il = np.tril_indices(rows, 0, cols)
        view[il[1], il[0]] = M[il]
    else:
        view[:, :rows] = M.T
    return buf


def _unpack(buf, off, ld, rows, cols):
    return buf[off:].reshape(max(cols, 1), ld)[:cols, :rows].T


def _variants(n):
    """(lda, offset in doubles): lda == n, odd lda, even lda > n, and an 8-byte aligned base with an even lda"""
    odd = n + 1 if n % 2 == 0 else n + 2
    even = n + 2 if n % 2 == 0 else n + 1
    return [(n, 0), (odd, 0), (even, 0), (even, 1)]


def _check_inv(inv, L, n):
    """work_inv: per diagonal block, inv(L_jj) (lower, identity-padded beyond the block's width) then, after all
    of them, the transposes; inv(L_jj) L_jj = I within the bound of a 128-term product times kappa(L_jj) (on the
    first two, the middle and the last two blocks)"""
    nblk = (n + NB - 1) // NB
    assert np.all(np.isfinite(inv))
    worst = 0.0
    for jb in range(nblk):
        X = inv[jb * NB * NB:(jb + 1) * NB * NB].reshape(NB, NB).T          # column-major NB x NB
        XT = inv[(nblk + jb) * NB * NB:(nblk + jb + 1) * NB * NB].reshape(NB, NB).T
        assert np.array_equal(XT, X.T), jb
        assert np.all(np.triu(X, 1) == 0), jb
        w = min(NB, n - jb * NB)
        if w < NB:
            pad = X.copy()
            pad[:w, :w] = 0
            assert np.array_equal(pad, np.diag(np.r_[np.zeros(w), np.ones(NB - w)])), jb
        if jb not in (0, 1, nblk // 2, nblk - 2, nblk - 1):
            continue
        Ljj = np.tril(L[jb * NB:jb * NB + w, jb * NB:jb * NB + w]).astype(np.longdouble)
        Xl = X[:w, :w].astype(np.longdouble)
        err = np.abs(Xl @ Ljj - np.eye(w, dtype=np.longdouble))
        kap = max(1.0, float(np.linalg.cond(np.tril(L[jb * NB:jb * NB + w, jb * NB:jb * NB + w]))))
        worst = max(worst, check_bound(err, (NB + 2) * EPS * kap * (np.abs(Xl) @ np.abs(Ljj))))
    return worst


def _potrs(lib, dL, off, n, lda, dinv, b):
    """solve with the factor and work_inv already on the device; L must come back bit-identical"""
    import torch
    before = dL.cpu().numpy()
    db = torch.from_numpy(b.copy()).cuda()
    assert lib.cvxb_potrs(n, dL.data_ptr() + 8 * off, lda, dinv.data_ptr(), db.data_ptr(), 0) == 0
    assert np.array_equal(dL.cpu().numpy().view(np.uint64), before.view(np.uint64)), "potrs modified L"
    return db.cpu().numpy()


def _lapack_ratios(A, cols, b):
    """LAPACK's dpotrf / dpotrs on the same input, measured by the same checkers (for the report only)"""
    Lr, info = lapack.dpotrf(A, lower=1, clean=1)
    assert info == 0
    kap = diag_block_kappa(Lr)
    x, info = lapack.dpotrs(Lr, b, lower=1)
    assert info == 0
    return check_potrf(A, Lr, cols, kappa=kap), backward_error(A, x, b) / (A.shape[0] * EPS * kap)


@pytest.mark.parametrize("n", SIZES)
def test_potrf_potrs_match_long_double(n):
    """every layout variant, each checked against long double; on lda == n the same matrix is factored in the
    eager, capture and replay modes (all eager beyond 4096) and must come out bit-identical (the schedule has no
    atomics and no split-K), then a second matrix goes through the replayed graph.  A1 is well-conditioned, A2 the
    interior-point regime up to n = 1333 (its Gram product is too slow on the host beyond) and another SPD matrix above."""
    import torch
    L, lib = _lib()
    cols = block_edge_cols(n)
    nblk = (n + NB - 1) // NB
    rng = np.random.Generator(np.random.PCG64(n))
    A1 = _spd(n, n)
    A2 = _ipm(n, n + 1) if n <= 1333 else _spd(n, n + 1)
    report = []
    keep = []                                   # distinct buffers for the whole test: distinct graph keys
    for vi, (lda, off) in enumerate(_variants(n)):
        dinv = torch.empty(2 * nblk * NB * NB, dtype=torch.float64, device="cuda")
        keep.append(dinv)
        buf1 = _poisoned(A1, lda, off, True)
        dA = torch.from_numpy(buf1).cuda()
        keep.append(dA)
        runs = []
        for mode in range(3 if vi == 0 else 1):
            dA.copy_(torch.from_numpy(buf1))
            dinv.fill_(float("nan"))
            rc = lib.cvxb_potrf(n, dA.data_ptr() + 8 * off, lda, dinv.data_ptr(), 0)
            assert rc == 0, (mode, L.last_error())
            runs.append((dA.cpu().numpy(), dinv.cpu().numpy()))
        for a, i in runs[1:]:                   # capture and replay (or, beyond 4096, eager again) == eager
            assert np.array_equal(a.view(np.uint64), runs[0][0].view(np.uint64)), "L differs between launch modes"
            assert np.array_equal(i.view(np.uint64), runs[0][1].view(np.uint64)), "work_inv differs between modes"
        out, inv = runs[0]
        check_lower_only_written(buf1, out, off, n, lda)
        Lh = _unpack(out, off, lda, n, n)
        kap = diag_block_kappa(Lh)
        r_f = check_potrf(A1, Lh, cols, kappa=kap)
        r_inv = _check_inv(inv, Lh, n)
        b = rng.standard_normal(n)
        r_s, eta = check_potrs(A1, _potrs(lib, dA, off, n, lda, dinv, b), b, kap)
        # a second matrix on the same key: the replayed graph on lda == n, the captured one otherwise
        buf2 = _poisoned(A2, lda, off, True)
        dA.copy_(torch.from_numpy(buf2))
        dinv.fill_(float("nan"))
        assert lib.cvxb_potrf(n, dA.data_ptr() + 8 * off, lda, dinv.data_ptr(), 0) == 0, L.last_error()
        out2, inv2 = dA.cpu().numpy(), dinv.cpu().numpy()
        check_lower_only_written(buf2, out2, off, n, lda)
        L2 = _unpack(out2, off, lda, n, n)
        kap2 = diag_block_kappa(L2)
        r_f2 = check_potrf(A2, L2, cols, kappa=kap2)
        _check_inv(inv2, L2, n)
        b2 = A2 @ rng.standard_normal(n)
        r_s2, eta2 = check_potrs(A2, _potrs(lib, dA, off, n, lda, dinv, b2), b2, kap2)
        line = ("potrf n=%d lda=%d off=%d: A1 %.3g (kappa %.3g), A2 %.3g (kappa %.3g), inv %.3g; "
                "potrs: A1 %.3g (eta %.2e), A2 %.3g (eta %.2e)" % (n, lda, off, r_f, kap, r_f2, kap2, r_inv,
                                                                   r_s, eta, r_s2, eta2))
        if vi == 0:
            lf, ls = _lapack_ratios(A1, cols, b)
            lf2, ls2 = _lapack_ratios(A2, cols, b2)
            line += "; LAPACK potrf A1 %.3g A2 %.3g, potrs A1 %.3g A2 %.3g" % (lf, lf2, ls, ls2)
        report.append(line)
    print("\n" + "\n".join(report))


@pytest.mark.parametrize("n", [300, 4097])
def test_potrf_info_names_the_first_bad_minor(n):
    """A = L0 L0' with A[k,k] -= 2 L0[k,k]^2: the k-th pivot is -L0[k,k]^2 and every earlier leading minor is
    positive, so LAPACK's info (and cvxb_potrf's return value) is k + 1.  The same buffer goes through the eager,
    capture and replay modes (n = 300); a positive definite matrix afterwards returns 0 (the replayed graph
    resets info)."""
    import torch
    L, lib = _lib()
    S = _spd(n, 7 * n)
    L0 = np.linalg.cholesky(S)
    nblk = (n + NB - 1) // NB
    dA = torch.empty(n * n, dtype=torch.float64, device="cuda")
    dinv = torch.empty(2 * nblk * NB * NB, dtype=torch.float64, device="cuda")
    for k in (0, 7, 8, 127, 128, 129, n - 1):
        A = S.copy()
        A[k, k] -= 2.0 * L0[k, k] ** 2
        _, want = lapack.dpotrf(A, lower=1)
        assert want == k + 1
        dA.copy_(torch.from_numpy(np.asfortranarray(A).ravel(order="F")))
        got = lib.cvxb_potrf(n, dA.data_ptr(), n, dinv.data_ptr(), 0)
        assert got == want, (k, got, want)
        assert ("order %d" % want) in L.last_error()
        dA.copy_(torch.from_numpy(S.ravel(order="F")))
        assert lib.cvxb_potrf(n, dA.data_ptr(), n, dinv.data_ptr(), 0) == 0


# (m, n, k, alpha, beta): m, n around the 128 x 64 tile, k around the 16-wide k step.  alpha = -1, beta = 1 is the
# read-modify-write form of the Cholesky updates (full interior tiles start their accumulators from C); beta = 0
# passes C filled with NaN, which must not be read
GEMM_CASES = [(1, 1, 1, 0.7, -0.3), (1, 300, 17, -1.0, 1.0), (300, 1, 1000, 1.3, 0.0), (63, 65, 3, 0.0, 0.8),
              (64, 64, 16, 1.0, 0.5), (65, 63, 17, 0.7, -0.3), (127, 129, 15, 1.3, 0.0), (128, 128, 4, -1.0, 1.0),
              (129, 127, 5, 1.0, 0.5), (64, 129, 0, 0.7, -0.3), (65, 64, 1, 0.0, 0.8), (300, 300, 1000, -1.0, 1.0),
              (129, 300, 16, 1.3, 0.0), (128, 64, 0, -1.0, 1.0), (300, 129, 1000, 0.7, -0.3),
              (256, 128, 17, 1.0, -1.0), (130, 70, 45, 0.7, -0.3), (257, 129, 300, 0.7, -0.3),
              (64, 200, 33, 0.7, -0.3), (100, 100, 100, 0.7, -0.3)]


def _ld(rows, vec, which):
    """leading dimension and base offset: even + aligned for the vector path; otherwise A gets an odd leading
    dimension and B and C an 8-byte aligned base"""
    if vec:
        return rows + 2 - rows % 2, 0
    if which == "A":
        return rows + 1 + rows % 2, 0
    return rows + 2 - rows % 2, 1


@pytest.mark.parametrize("vec", [True, False])
@pytest.mark.parametrize("tb", ["N", "T"])
@pytest.mark.parametrize("ta", ["N", "T"])
def test_gemm_matches_long_double(ta, tb, vec):
    """all 8 dmma_gemm_kernel<XK, YK, VEC> instantiations on edge shapes: per entry within
    (k + 2) u (|alpha| |op(A)| |op(B)| + |beta| |C0|); k = 0 gives exactly fl(beta C0); beta = 0 never reads C
    (NaN in, finite out); rows m..ldc-1 of C are not written"""
    import torch
    L, lib = _lib()
    rng = np.random.Generator(np.random.PCG64(ord(ta) * 7 + ord(tb) * 3 + vec))
    worst = 0.0
    for m, n, k, alpha, beta in GEMM_CASES:
        opA = rng.standard_normal((m, k))
        opB = rng.standard_normal((k, n))
        C0 = rng.standard_normal((m, n)) if beta != 0.0 else np.full((m, n), np.nan)
        Ast = opA.T if ta == "T" else opA                 # stored matrices
        Bst = opB.T if tb == "T" else opB
        lda, oa = _ld(Ast.shape[0], vec, "A")
        ldb, ob = _ld(Bst.shape[0], vec, "B")
        ldc, oc = _ld(m, vec, "C")
        lda, ldb = max(lda, 1), max(ldb, 1)
        ha = _poisoned(Ast, lda, oa, False) if k else np.full(oa + lda, np.nan)
        hb = _poisoned(Bst, ldb, ob, False) if k else np.full(ob + ldb, np.nan)
        hc = _poisoned(C0, ldc, oc, False)
        dA, dB, dC = (torch.from_numpy(h).cuda() for h in (ha, hb, hc))
        rc = lib.cvxb_gemm(ord(ta), ord(tb), m, n, k, alpha, dA.data_ptr() + 8 * oa, lda, dB.data_ptr() + 8 * ob,
                           ldb, beta, dC.data_ptr() + 8 * oc, ldc, 0)
        assert rc == 0, L.last_error()
        out = dC.cpu().numpy()
        C = _unpack(out, oc, ldc, m, n)
        mask = np.ones(out.size, bool)
        mask[oc:].reshape(n, ldc)[:, :m] = False
        assert np.array_equal(out[mask].view(np.uint64), hc[mask].view(np.uint64)), (m, n, k, "padding written")
        assert np.all(np.isfinite(C)), (m, n, k, alpha, beta)
        if k == 0:
            want = beta * C0 if beta != 0.0 else np.zeros((m, n))
            assert np.array_equal(C, want), (m, n, alpha, beta)
        cols = block_edge_cols(n) if n > 130 else None
        worst = max(worst, check_gemm(opA, opB, alpha, beta, C0, C, cols))
    print("\ngemm %s%s vec=%d: largest error / bound %.3g" % (ta, tb, vec, worst))
