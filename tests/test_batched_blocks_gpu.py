"""The batch solver's dense building blocks, problem by problem, against long double (tests/ld_check.py).

cvxb_potrf_batched, cvxb_trsv_batched, cvxb_trsm_batched, cvxb_syrk_batched and cvxb_gemv_batched run the code the
batch solver runs on all of its problems at once (potrf_lower_batched, the flag-chained trsv_kernel with the problem in
blockIdx.y, trsm_lower_left, the weighted batched dmma_gemm SYRK, gemv_t / gemv_n with GemvBatch strides).  Every
kernel is checked
- on each of four layouts: the batch solver's own (leading dimension = rows rounded up to even, stride = ld * cols),
  an odd leading dimension and odd stride (the non-vector copy paths), a gap between problems, and a base pointer that
  is 8- but not 16-byte aligned;
- with NaN in everything a call must neither read nor write (gaps, rows n..ld-1, strict upper triangles, vector
  padding), which has to come back bit for bit;
- on sampled problems (the first, the second, one in the middle, the last) and, for large operands, sampled columns;
- for cross-talk: a problem in slot j of a batch gives the same bits as in slot 0 of a batch of two with another
  neighbour (nothing in these paths is split or reduced across problems).
The 'q' rows of cvxb_scale (q_scale of cone.cuh, which the batch solver's k_build_gs runs too) are checked against
long double on the same terms.  Every check prints its largest error / bound."""
import numpy as np
import pytest
import scipy.linalg.lapack as lapack

from ld_check import (NB, block_edge_cols, check_gemv, check_potrf, check_potrs, check_qscale, check_syrk, check_trsm,
                      check_trsv, diag_block_kappa)
from test_dense_blocks_gpu import _check_inv, _ipm, _lib, _spd

pytestmark = pytest.mark.gpu

SIZES = [1, 2, 7, 8, 9, 127, 128, 129, 255, 256, 257, 385, 512]
LAYOUTS = ["solver", "odd", "gap", "unaligned"]
BATCH_MAX = 65535


class Lay:
    """`batch` column-major rows x cols operands in one flat device buffer: problem b at off + b * stride"""

    def __init__(self, kind, rows, cols, batch):
        ld = max(2, rows + rows % 2)
        stride, off = ld * cols, 0
        if kind == "odd":
            ld = rows + 1 - rows % 2                     # odd and >= rows
            stride = ld * cols + (1 - (ld * cols) % 2)   # odd
        elif kind == "gap":
            stride = ld * cols + 10
        elif kind == "unaligned":
            off = 1
        self.kind, self.rows, self.cols, self.batch = kind, rows, cols, batch
        self.ld, self.stride, self.off = ld, stride, off
        self.size = off + stride * (batch - 1) + ld * max(cols, 1) + 3

    def alloc(self):
        import torch
        return torch.full((self.size,), float("nan"), dtype=torch.float64, device="cuda")

    def view(self, buf):
        """(batch, cols, rows): view[b, c, r] is entry (r, c) of problem b"""
        import torch
        return torch.as_strided(buf, (self.batch, self.cols, self.ld), (self.stride, self.ld, 1),
                                self.off)[:, :, :self.rows]

    def ptr(self, buf):
        return buf.data_ptr() + 8 * self.off

    def put(self, M, lower=False):
        """a NaN-filled buffer holding M (batch x rows x cols); only the lower triangles when `lower`"""
        buf = self.alloc()
        v = self.view(buf)
        v.copy_(M.transpose(1, 2))
        if lower:
            v.masked_fill_(self._upper(), float("nan"))
        return buf

    def get(self, buf, b):
        return np.ascontiguousarray(self.view(buf)[b].cpu().numpy().T)

    def _upper(self):
        import torch
        return torch.ones(self.cols, self.rows, dtype=torch.bool, device="cuda").tril(-1)   # r < c

    def untouched(self, before, after, written, what):
        """everything outside the problems' operands (or their lower triangles, written == 'lower') is bit-identical;
        written == None: the whole buffer"""
        import torch
        diff = before.view(torch.int64) != after.view(torch.int64)
        if written is not None:
            v = self.view(diff)
            if written == "lower":
                v.masked_fill_(~self._upper(), False)
            else:
                v.fill_(False)
        bad = int(diff.sum())
        assert bad == 0, "%s: %d elements outside the operands changed (%s layout)" % (what, bad, self.kind)


def _samples(batch):
    return sorted({0, 1, batch // 2, batch - 1} & set(range(batch)))


def _spd_batch(n, batch, seed):
    """batch x n x n on the device: _spd for even problems, _ipm (d in 1e-4 .. 1e4) for odd ones, so that neighbours
    differ in scale; generated on the device with the same two recipes for large batches"""
    import torch
    if batch <= 3:
        return torch.from_numpy(np.stack([(_spd if b % 2 == 0 else _ipm)(n, seed + b) for b in range(batch)])).cuda()
    g = torch.Generator(device="cuda").manual_seed(seed)
    kw = dict(dtype=torch.float64, device="cuda", generator=g)
    out = torch.empty(batch, n, n, dtype=torch.float64, device="cuda")
    eye = torch.eye(n, dtype=torch.float64, device="cuda")
    Bm = torch.randn((batch + 1) // 2, n, n, **kw)
    out[0::2] = Bm @ Bm.mT / n + eye
    del Bm
    if batch > 1:
        no = batch // 2
        A0 = torch.randn(no, n, n, **kw)
        Gd = torch.randn(no, 2 * n, n, **kw) * 10.0 ** (torch.rand(no, 2 * n, 1, **kw) * 8 - 4)
        S = A0.mT @ A0 / n + eye + Gd.mT @ Gd
        out[1::2] = (S + S.mT) / 2
    return out


def _randn(shape, seed):
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(shape, dtype=torch.float64, device="cuda", generator=g)


def _rand(shape, seed):
    """uniform in [0, 1)"""
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.rand(shape, dtype=torch.float64, device="cuda", generator=g)


# The library runs on its own non-blocking stream, which does not wait for torch's: every call below is preceded by
# torch.cuda.synchronize() so that the operands torch wrote are complete.
def _bits_equal(a, b):
    return np.array_equal(np.asarray(a).view(np.uint64), np.asarray(b).view(np.uint64))


def _inputs_kept(before, after, what):
    """device buffers a call only reads come back bit for bit"""
    import torch
    for t0, t in zip(before, after):
        assert torch.equal(t0.view(torch.int64), t.view(torch.int64)), "%s wrote an input" % what


# ------------------------------------------------------------------------------------------ Cholesky + triangular solves
def _potrf(lib, L, M, kind):
    """factor the batch M (device, batch x n x n) on `kind`; returns (layout, A before, A after, inv, info)"""
    import torch
    batch, n = M.shape[0], M.shape[1]
    lay = Lay(kind, n, n, batch)
    nblk = (n + NB - 1) // NB
    sinv = 2 * nblk * NB * NB
    dA = lay.put(M, lower=True)
    before = dA.clone()
    dinv = torch.full((batch * sinv,), float("nan"), dtype=torch.float64, device="cuda")
    info = np.full(batch, -7, dtype=np.intc)
    torch.cuda.synchronize()
    rc = lib.cvxb_potrf_batched(n, lay.ptr(dA), lay.ld, lay.stride, dinv.data_ptr(), sinv, batch, info.ctypes.data, 0)
    assert rc == 0, L.last_error()
    return lay, before, dA, dinv, info


def _trsv(lib, L, lay, dA, dinv, rhs, trans, kind):
    """solve every problem's op(L) x = rhs (device, batch x n) in place ('NT': potrs); returns (vector layout, x)"""
    import torch
    batch, n = rhs.shape
    vl = Lay(kind, n, 1, batch)
    db = vl.put(rhs[:, :, None])
    bb, Lb = db.clone(), dA.clone()
    sinv = dinv.numel() // batch
    torch.cuda.synchronize()
    for t in trans:
        rc = lib.cvxb_trsv_batched(n, lay.ptr(dA), lay.ld, lay.stride, dinv.data_ptr(), sinv, vl.ptr(db), vl.stride,
                                   ord(t), batch, 0)
        assert rc == 0, L.last_error()
    lay.untouched(Lb, dA, None, "trsv (L)")
    vl.untouched(bb, db, "all", "trsv (b)")
    return vl, db


def _potrf_trsv_case(lib, L, n, batch, kind, seed):
    """one batch on one layout: potrf, then 'N', 'T' and 'NT' solves, checked on sampled problems"""
    M = _spd_batch(n, batch, seed)
    lay, before, dA, dinv, info = _potrf(lib, L, M, kind)
    assert np.all(info == 0), info
    lay.untouched(before, dA, "lower", "potrf")
    sinv = dinv.numel() // batch
    cols = block_edge_cols(n)
    rhs = _randn((batch, n), seed + 1)
    sols = {t: _trsv(lib, L, lay, dA, dinv, rhs, t, kind) for t in ("N", "T", "NT")}
    worst = dict(potrf=0.0, inv=0.0, N=0.0, T=0.0, NT=0.0)
    facs = {}
    for b in _samples(batch):
        A = M[b].cpu().numpy()
        Lh = lay.get(dA, b)
        facs[b] = Lh
        kap = diag_block_kappa(Lh)
        worst["potrf"] = max(worst["potrf"], check_potrf(A, Lh, cols, kappa=kap))
        worst["inv"] = max(worst["inv"], _check_inv(dinv[b * sinv:(b + 1) * sinv].cpu().numpy(), Lh, n))
        r = rhs[b].cpu().numpy()
        for t in ("N", "T"):
            vl, db = sols[t]
            worst[t] = max(worst[t], check_trsv(Lh, vl.get(db, b)[:, 0], r, t, kap))
        vl, db = sols["NT"]
        worst["NT"] = max(worst["NT"], check_potrs(A, vl.get(db, b)[:, 0], r, kap)[0])
    print("potrf/trsv n=%d batch=%d %s: potrf %.3g, inv %.3g, trsv N %.3g, T %.3g, potrs %.3g"
          % (n, batch, kind, worst["potrf"], worst["inv"], worst["N"], worst["T"], worst["NT"]))
    if batch >= 3:      # cross-talk: the middle problem in slot 0 of a batch of two, another neighbour in slot 1
        import torch
        j = batch // 2
        other = _spd_batch(n, 3, seed + 1000)[2 - j % 2]
        M2 = torch.stack([M[j], other])
        lay2, _, dA2, dinv2, info2 = _potrf(lib, L, M2, kind)
        assert np.all(info2 == 0)
        assert _bits_equal(lay2.get(dA2, 0), lay.get(dA, j)), "factor depends on the neighbours"
        assert _bits_equal(dinv2[:sinv].cpu().numpy(), dinv[j * sinv:(j + 1) * sinv].cpu().numpy()), "inverse"
        for t in ("N", "T", "NT"):
            vl2, db2 = _trsv(lib, L, lay2, dA2, dinv2, torch.stack([rhs[j], rhs[0]]), t, kind)
            vl, db = sols[t]
            assert _bits_equal(vl2.get(db2, 0), vl.get(db, j)), ("trsv depends on the neighbours", t)
    return lay, dA, dinv


@pytest.mark.parametrize("n", SIZES)
def test_potrf_trsv_batched_match_long_double(n):
    """each layout at batch 1 and 3 (and 64 at n = 129, 512): check_potrf with kappa and the work_inv contract per
    problem, info all zero, L and b bit-identical outside what a call writes; trsv 'N', 'T' and potrs on the factors"""
    L, lib = _lib()
    for batch in (1, 3) + ((64,) if n in (129, 512) else ()):
        for li, kind in enumerate(LAYOUTS):
            _potrf_trsv_case(lib, L, n, batch, kind, seed=1000 * n + 10 * batch + li)


def test_potrf_trsv_at_the_batch_solvers_shape():
    """B = 512 problems of n = 512 on the solver's layout: potrf_lower_batched and the 2048-CTA flag chain of the
    batched trsv that the batch solver runs every iteration"""
    L, lib = _lib()
    _potrf_trsv_case(lib, L, 512, 512, "solver", seed=4512)


@pytest.mark.parametrize("n", [257, 512])
def test_potrf_batched_info_per_problem(n):
    """B = 6, problems 1 and 4 not positive definite at leading minors k (built as in
    test_potrf_info_names_the_first_bad_minor): info[j] is LAPACK's info for every j, the good problems' factors and
    inverses are bit-identical to an all-good run of the same batch, and a clean run afterwards returns all zeros"""
    import torch
    L, lib = _lib()
    good = _spd_batch(n, 6, 77 * n)
    _, _, dA0, dinv0, info0 = _potrf(lib, L, good, "solver")
    assert np.all(info0 == 0)
    lay = Lay("solver", n, n, 6)
    sinv = dinv0.numel() // 6
    chol = {j: np.linalg.cholesky(good[j].cpu().numpy()) for j in (1, 4)}
    ks = [k for k in (0, 7, 8, 127, 128, 129, n - 1) if k < n]
    for i, k in enumerate(ks):
        M = good.clone()
        want = np.zeros(6, dtype=np.intc)
        for j, kk in ((1, k), (4, ks[(i + 3) % len(ks)])):
            A = good[j].cpu().numpy().copy()
            A[kk, kk] -= 2.0 * chol[j][kk, kk] ** 2
            want[j] = lapack.dpotrf(A, lower=1)[1]
            assert want[j] == kk + 1
            M[j] = torch.from_numpy(A).cuda()
        _, _, dA, dinv, info = _potrf(lib, L, M, "solver")
        assert np.array_equal(info, want), (k, info, want)
        for j in (0, 2, 3, 5):
            assert _bits_equal(lay.get(dA, j), lay.get(dA0, j)), (k, j, "factor of a good problem changed")
            assert _bits_equal(dinv[j * sinv:(j + 1) * sinv].cpu().numpy(),
                               dinv0[j * sinv:(j + 1) * sinv].cpu().numpy()), (k, j, "inverse of a good problem")
    _, _, dA, _, info = _potrf(lib, L, good, "solver")
    assert np.all(info == 0)
    assert _bits_equal(dA.cpu().numpy(), dA0.cpu().numpy())
    print("potrf_batched info n=%d: bad minors %s in problems 1 and 4 named, good problems bit-identical" % (n, ks))


# ------------------------------------------------------------------------------------------------------------ TRSM
def _trsm(lib, L, lay, dA, dinv, Bm, kind):
    import torch
    batch, n, ncols = Bm.shape
    bl = Lay(kind, n, ncols, batch)
    dB = bl.put(Bm)
    before, Lb = dB.clone(), dA.clone()
    torch.cuda.synchronize()
    rc = lib.cvxb_trsm_batched(n, lay.ptr(dA), lay.ld, lay.stride, dinv.data_ptr(), dinv.numel() // batch,
                               bl.ptr(dB), bl.ld, bl.stride, ncols, batch, 0)
    assert rc == 0, L.last_error()
    lay.untouched(Lb, dA, None, "trsm (L)")
    bl.untouched(before, dB, "all", "trsm (B)")
    return bl, dB


@pytest.mark.parametrize("kind", LAYOUTS)
@pytest.mark.parametrize("n", [1, 127, 128, 129, 257])
def test_trsm_batched_matches_long_double(n, kind):
    """B := L^{-1} B with ncols in {1, 2, 63, 64, 65, 130} (several column tiles of the in-place diagonal step) at batch
    1 and 3: check_trsm on sampled problems and block-edge columns, bit-identical padding, no cross-talk"""
    import torch
    L, lib = _lib()
    report = []
    for batch in (1, 3):
        M = _spd_batch(n, batch, 31 * n + batch)
        lay, _, dA, dinv, info = _potrf(lib, L, M, kind)
        assert np.all(info == 0)
        for ncols in (1, 2, 63, 64, 65, 130):
            Bm = _randn((batch, n, ncols), 7 * n + ncols + batch)
            bl, dB = _trsm(lib, L, lay, dA, dinv, Bm, kind)
            cols = block_edge_cols(ncols)
            worst = 0.0
            for b in _samples(batch):
                Lh = lay.get(dA, b)
                worst = max(worst, check_trsm(Lh, bl.get(dB, b)[:, cols], Bm[b].cpu().numpy()[:, cols],
                                              diag_block_kappa(Lh)))
            report.append("trsm n=%d ncols=%d batch=%d %s: %.3g" % (n, ncols, batch, kind, worst))
            if batch == 3:
                M2 = torch.stack([M[1], M[0]])
                lay2, _, dA2, dinv2, _ = _potrf(lib, L, M2, kind)
                bl2, dB2 = _trsm(lib, L, lay2, dA2, dinv2, torch.stack([Bm[1], Bm[2]]), kind)
                assert _bits_equal(bl2.get(dB2, 0), bl.get(dB, 1)), (n, ncols, "trsm depends on the neighbours")
    print("\n" + "\n".join(report))


# ------------------------------------------------------------------------------------------------------------ SYRK
def _syrk(lib, L, A, w, D, inplace, kind):
    """C(lower) = A' diag(w) A + D for the batch A (batch x k x n), w (batch x k) or None, D (batch x n x n) or None;
    returns (layout of C, C before, C after)"""
    import torch
    batch, k, n = A.shape
    al = Lay(kind, k, n, batch)
    dA = al.put(A)
    cl = Lay(kind, n, n, batch)
    wl = Lay(kind, k, 1, batch)
    dw = wl.put(w[:, :, None]) if w is not None else None
    dD = cl.put(D, lower=True) if D is not None else None
    dC = dD if inplace else cl.alloc()
    before = dC.clone()
    reads = [t for t in (dA, dw, dD) if t is not None and t is not dC]
    ins = [t.clone() for t in reads]
    torch.cuda.synchronize()
    rc = lib.cvxb_syrk_batched(n, k, al.ptr(dA), al.ld, al.stride, wl.ptr(dw) if dw is not None else None,
                               wl.stride, cl.ptr(dD) if dD is not None else None, cl.ld, cl.stride,
                               cl.ptr(dC), cl.ld, cl.stride, batch, 0)
    assert rc == 0, L.last_error()
    cl.untouched(before, dC, "lower", "syrk (C)")
    _inputs_kept(ins, reads, "syrk")
    return cl, before, dC


@pytest.mark.parametrize("kind", LAYOUTS)
@pytest.mark.parametrize("k", [0, 1, 3, 4, 17, 1024])
def test_syrk_batched_matches_long_double(k, kind):
    """w = NULL, w spanning 1e-8 .. 1e8 (di^2) and a 0/1 mask per problem (the batch solver's A'A switch: problem 0
    off, problem 1 on, problem 2 mixed); D = NULL, D apart from C and D == C.  check_syrk on sampled columns; k = 0
    gives C = D exactly; with w = 0 C comes back bit-identical to D (the other problems' K must not move when one
    problem switches); no cross-talk"""
    import torch
    L, lib = _lib()
    report = []
    for n, batch in ((9, 3), (129, 1), (257, 3)):
        A = _randn((batch, k, n), 100 * k + n)
        Dm = _randn((batch, n, n), 100 * k + n + 1)
        mask = torch.zeros((3, k), dtype=torch.float64, device="cuda")
        mask[1] = 1.0
        mask[2, 1::3] = 1.0
        ws = {"none": None, "wide": 10.0 ** (_rand((batch, k), 100 * k + n + 2) * 16 - 8), "mask": mask[:batch]}
        cols = block_edge_cols(n)
        for wname, w in ws.items():
            for dname in ("none", "apart", "inplace"):
                D = None if dname == "none" else Dm
                cl, before, dC = _syrk(lib, L, A, w, D, dname == "inplace", kind)
                worst = 0.0
                for b in _samples(batch):
                    Ah = A[b].cpu().numpy()
                    wh = w[b].cpu().numpy() if w is not None else None
                    Dh = Dm[b].cpu().numpy() if D is not None else None
                    Ch = cl.get(dC, b)
                    worst = max(worst, check_syrk(Ah, wh, Dh, Ch, cols))
                    low = np.tril(np.ones((n, n), bool))
                    if k == 0 or (w is not None and not wh.any()):
                        if Dh is not None:
                            assert _bits_equal(Ch[low], Dh[low]), (k, n, b, wname, dname, "C != D bit for bit")
                        else:
                            assert np.all(Ch[low] == 0.0), (k, n, b, wname, "C != 0")
                report.append("syrk n=%d k=%d batch=%d w=%s D=%s %s: %.3g" % (n, k, batch, wname, dname, kind, worst))
                if batch == 3:
                    sel = torch.tensor([1, 0], device="cuda")
                    cl2, _, dC2 = _syrk(lib, L, A[sel], w[sel] if w is not None else None,
                                        Dm[sel] if D is not None else None, dname == "inplace", kind)
                    assert _bits_equal(cl2.get(dC2, 0), cl.get(dC, 1)), (n, k, wname, dname, "cross-talk")
    print("\n" + "\n".join(report))


# ------------------------------------------------------------------------------------------------------------ GEMV
NROWS = [1, 2, 31, 32, 33, 255, 256, 257, 1023]
NCOLS = [0, 1, 127, 128, 129, 300]
ALPHAS = [1.0, -1.0, 0.7, 0.0]
BETAS = [1.0, -1.0, 0.0]


def _gemv(lib, L, trans, A, w, x, alpha, beta, y0, kind):
    """y = alpha op(A) (w) x + beta y0 for the batch; returns (y layout, y)"""
    import torch
    batch, nrows, ncols = A.shape
    al = Lay(kind, nrows, ncols, batch)
    dA = al.put(A)
    wl = Lay(kind, nrows, 1, batch)
    dw = wl.put(w[:, :, None]) if w is not None else None
    nx, ny = (nrows, ncols) if trans == "T" else (ncols, nrows)
    xl, yl = Lay(kind, nx, 1, batch), Lay(kind, ny, 1, batch)
    dx = xl.put(x[:, :, None])
    dy = yl.put(y0[:, :, None])
    reads = [t for t in (dA, dw, dx) if t is not None]
    before, ins = dy.clone(), [t.clone() for t in reads]
    torch.cuda.synchronize()
    rc = lib.cvxb_gemv_batched(ord(trans), nrows, ncols, al.ptr(dA), al.ld, al.stride,
                               wl.ptr(dw) if dw is not None else None, wl.stride, xl.ptr(dx), xl.stride,
                               alpha, beta, yl.ptr(dy), yl.stride, batch, 0)
    assert rc == 0, L.last_error()
    yl.untouched(before, dy, "all", "gemv (y)")
    _inputs_kept(ins, reads, "gemv")
    return yl, dy


def _gemv_case(lib, L, trans, nrows, ncols, alpha, beta, weighted, batch, kind, seed):
    import torch
    A = _randn((batch, nrows, ncols), seed)
    w = 10.0 ** (_rand((batch, nrows), seed + 4) * 8 - 4) if weighted else None
    nx, ny = (nrows, ncols) if trans == "T" else (ncols, nrows)
    x = _randn((batch, nx), seed + 1)
    y0 = _randn((batch, ny), seed + 2) if beta != 0.0 else torch.full((batch, ny), float("nan"), dtype=torch.float64,
                                                                       device="cuda")
    yl, dy = _gemv(lib, L, trans, A, w, x, alpha, beta, y0, kind)
    worst = 0.0
    for b in _samples(batch):
        yb = yl.get(dy, b)[:, 0]
        assert np.all(np.isfinite(yb))
        worst = max(worst, check_gemv(trans, A[b].cpu().numpy(), w[b].cpu().numpy() if weighted else None,
                                      x[b].cpu().numpy(), alpha, beta, y0[b].cpu().numpy(), yb))
    if batch >= 3:
        j = batch // 2
        sel = torch.tensor([j, 0], device="cuda")
        other = _randn((1, nrows, ncols), seed + 3)[0]
        A2 = torch.stack([A[j], other])
        yl2, dy2 = _gemv(lib, L, trans, A2, w[sel] if weighted else None, x[sel], alpha, beta, y0[sel], kind)
        assert _bits_equal(yl2.get(dy2, 0), yl.get(dy, j)), (trans, nrows, ncols, "gemv depends on the neighbours")
    return worst


@pytest.mark.parametrize("kind", LAYOUTS)
@pytest.mark.parametrize("trans", ["T", "N"])
def test_gemv_batched_matches_long_double(trans, kind):
    """every nrows x ncols pair (gemv_n's 128-column chunks, the odd tail row of the vector path); alpha, beta, w and
    batch in {1, 3, 512} cycle through the pairs; beta = 0 comes with NaN in y; check_gemv on sampled problems"""
    L, lib = _lib()
    worst, i = {}, 0
    for nrows in NROWS:
        for ncols in NCOLS:
            alpha, beta = ALPHAS[i % 4], BETAS[(i // 4) % 3]
            weighted = (i // 2) % 2 == 1
            batch = (1, 3, 512)[i % 3]
            r = _gemv_case(lib, L, trans, nrows, ncols, alpha, beta, weighted, batch, kind, seed=i)
            key = "w" if weighted else "-"
            worst[key] = max(worst.get(key, 0.0), r)
            i += 1
    print("\ngemv %s %s: largest error / bound %s" % (trans, kind, worst))


@pytest.mark.parametrize("trans", ["T", "N"])
def test_gemv_batched_at_the_batch_limit(trans):
    """batch = CVXB_BATCH_MAX at nrows = ncols = 8: the largest grid the batch kernels are launched with"""
    L, lib = _lib()
    for weighted, kind in ((False, "solver"), (True, "odd")):
        r = _gemv_case(lib, L, trans, 8, 8, 0.7, -1.0, weighted, BATCH_MAX, kind, seed=5)
        print("gemv %s batch=%d w=%d %s: %.3g" % (trans, BATCH_MAX, weighted, kind, r))


# ------------------------------------------------------------------------------------------------- 'q' scaling of G
QORDERS = [1, 2, 3, 31, 32, 33, 64, 65, 300]


@pytest.mark.parametrize("inverse", ["N", "I"])
@pytest.mark.parametrize("xc", [1, 4, 5, 1000])
def test_scale_q_rows_match_long_double(xc, inverse):
    """cvxb_scale on 5 'l' rows and cones of order 1 .. 300 (q_scale on a warp per cone and column, as k_build_gs
    forms Gs = W^{-T} G): 'q' rows against check_qscale with beta in 1e-3 .. 1e3 and v on the hyperboloid, 'l' rows
    exactly x * d (or di), and NaN rows cdim .. xr-1 untouched"""
    from cvxopt_b200 import misc_solvers as ms
    rng = np.random.Generator(np.random.PCG64(xc + (inverse == "I")))
    ml = 5
    vs, betas = [], []
    for m in QORDERS:
        u = rng.standard_normal(m - 1) * rng.uniform(0.1, 3.0)
        vs.append(np.r_[np.sqrt(1.0 + u @ u), u])
        betas.append(10.0 ** rng.uniform(-3, 3))
    d = 10.0 ** rng.uniform(-2, 2, ml)
    W = {"d": d, "di": 1.0 / d, "v": vs, "beta": betas, "r": [], "rti": []}
    cdim = ml + sum(QORDERS)
    xr = cdim + 3
    x = np.full((xr, xc), np.nan, order="F")
    x[:cdim] = rng.standard_normal((cdim, xc))
    x0 = x.copy(order="F")
    ms.scale(x, W, "N", inverse)
    assert _bits_equal(x[cdim:], x0[cdim:]), "rows beyond the cone dimension written"
    dl = W["di"] if inverse == "I" else d
    assert _bits_equal(x[:ml], x0[:ml] * dl[:, None]), "'l' rows"
    worst, o = 0.0, ml
    for v, beta in zip(vs, betas):
        m = v.size
        worst = max(worst, check_qscale(v, beta, x0[o:o + m], x[o:o + m], inverse == "I"))
        o += m
    print("\nscale q xc=%d inverse=%s: largest error / bound %.3g" % (xc, inverse, worst))
