"""`kktsolver` factories backed by the GPU library — host-side mirror of the
reference's KKT factories (reference src/python/misc.py:1213-1349, `kkt_chol`).

Usage with an unmodified CVXOPT (the plugin boundary, coneprog.py:323-344 /
1658-1679):

    from cvxopt import solvers
    import cvxopt_b200
    factor = cvxopt_b200.kkt_chol(G, dims, A, H=P)        # G, P uploaded once
    sol = solvers.coneqp(P, q, G, h, dims, kktsolver=lambda W: factor(W))

`factor(W, H=None, Df=None)` returns `solve(x, y, z)` which overwrites the
solver-owned vectors in place with (ux, uy, W*uz), exactly like the reference
closure.  Any object exposing the buffer protocol with fp64 column-major data
works (cvxopt.matrix, numpy F-ordered arrays); cvxopt itself is not imported.

G, A, H and Df may also be sparse: a cvxopt `spmatrix` (recognised by its `CCS`
and `size` attributes) or any scipy.sparse matrix.  The 'l' rows of G stay
sparse on the device; everything else is densified once (INTEGRATION.md §1).
"""
import ctypes as C
import sys

import numpy as np

from . import _lib


def _mat(a, name="matrix"):
    """fp64, column-major 2-D view (copy only if the layout requires it)."""
    arr = np.asarray(a)
    if arr.dtype != np.float64:
        if arr.dtype.kind in "iuf":
            arr = arr.astype(np.float64)
        else:
            raise TypeError("%s must be a real 'd' matrix" % name)
    if arr.ndim == 1:
        arr = arr.reshape(-1, 1)
    if arr.ndim != 2:
        raise TypeError("%s must be two-dimensional" % name)
    if not arr.flags.f_contiguous:
        arr = np.asfortranarray(arr)
    return arr


def is_sparse(a):
    """a cvxopt spmatrix (duck-typed: the package never imports cvxopt) or a scipy.sparse matrix"""
    if hasattr(a, "CCS") and hasattr(a, "size"):
        return True
    sps = sys.modules.get("scipy.sparse")      # a scipy.sparse matrix exists only once scipy.sparse is imported
    return sps is not None and sps.issparse(a)


def to_csr(a, name="matrix"):
    """spmatrix or scipy.sparse -> ((rows, cols), rowptr int64, colind int32, val float64), canonical CSR: columns
    sorted within each row, duplicate entries summed (in their order of appearance), explicit zeros kept."""
    if hasattr(a, "CCS") and hasattr(a, "size"):
        rows, cols = (int(k) for k in a.size)
        colptr, rowind, vals = a.CCS
        colptr = np.asarray(colptr, dtype=np.int64).ravel()
        r = np.asarray(rowind, dtype=np.int64).ravel()
        c = np.repeat(np.arange(cols, dtype=np.int64), np.diff(colptr))
        v = np.asarray(vals).ravel()
    else:
        coo = a.tocoo()
        rows, cols = (int(k) for k in coo.shape)
        r = np.asarray(coo.row, dtype=np.int64)
        c = np.asarray(coo.col, dtype=np.int64)
        v = np.asarray(coo.data)
    if v.dtype.kind not in "iuf":
        raise TypeError("%s must be a real 'd' matrix" % name)
    v = v.astype(np.float64)
    if r.size != v.size or c.size != v.size:
        raise TypeError("%s: inconsistent sparse storage" % name)
    if r.size and (r.min() < 0 or r.max() >= rows or c.min() < 0 or c.max() >= cols):
        raise TypeError("%s: an index is outside its %d x %d shape" % (name, rows, cols))
    order = np.lexsort((c, r))                   # stable: duplicates stay in their order of appearance
    r, c, v = r[order], c[order], v[order]
    if r.size:
        first = np.ones(r.size, dtype=bool)
        first[1:] = (r[1:] != r[:-1]) | (c[1:] != c[:-1])
        starts = np.flatnonzero(first)
        v = np.add.reduceat(v, starts)
        r, c = r[starts], c[starts]
    rowptr = np.zeros(rows + 1, dtype=np.int64)
    np.cumsum(np.bincount(r, minlength=rows), out=rowptr[1:])
    return (rows, cols), rowptr, np.ascontiguousarray(c, dtype=np.int32), np.ascontiguousarray(v)


def _dense(a, name="matrix"):
    """_mat, for sparse input too: a sparse matrix is densified"""
    if not is_sparse(a):
        return _mat(a, name)
    (rows, cols), rowptr, colind, val = to_csr(a, name)
    out = np.zeros((rows, cols), order="F")
    out[np.repeat(np.arange(rows), np.diff(rowptr)), colind] = val
    return out


def _vec_inplace(a, n, name):
    """writable fp64 view of a solver-owned vector of length n (no copy allowed)."""
    arr = np.asarray(a)
    if arr.dtype != np.float64 or arr.size != n:
        raise TypeError("%s must be a 'd' matrix of size (%d,1)" % (name, n))
    if n == 0:
        return np.zeros(1)          # nothing to read or write; keep a valid pointer
    flat = arr.reshape(-1, order="F") if arr.ndim > 1 else arr
    if not np.shares_memory(flat, arr) or not flat.flags.writeable or not flat.flags.c_contiguous:
        raise TypeError("%s must be a contiguous writable buffer" % name)
    return flat


def make_dims(dims, mnl=0):
    """reference `dims` dict -> (ctypes Dims, keep-alive tuple, cdim, cdim_pckd)"""
    if dims is None:
        raise TypeError("dims is required")
    ml = int(dims["l"])
    q = [int(k) for k in dims["q"]]
    s = [int(k) for k in dims["s"]]
    if ml < 0:
        raise TypeError("'dims['l']' must be a nonnegative integer")
    if any(k < 1 for k in q):
        raise TypeError("'dims['q']' must be a list of positive integers")
    if any(k < 0 for k in s):
        raise TypeError("'dims['s']' must be a list of nonnegative integers")
    qa = (C.c_int * max(1, len(q)))(*q)
    sa = (C.c_int * max(1, len(s)))(*s)
    d = _lib.Dims(int(mnl), ml, len(q), C.cast(qa, _lib.c_int_p), len(s), C.cast(sa, _lib.c_int_p))
    cdim = mnl + ml + sum(q) + sum(k * k for k in s)
    cdim_pckd = mnl + ml + sum(q) + sum(k * (k + 1) // 2 for k in s)
    return d, (qa, sa), cdim, cdim_pckd


def _flat(items, count, name):
    """concatenate a list of matrices (W['v'], W['r'], ...) into one fp64 vector"""
    if count == 0:
        return np.zeros(0)
    parts = [np.asarray(m, dtype=np.float64).reshape(-1, order="F") for m in items]
    out = np.concatenate(parts) if parts else np.zeros(0)
    if out.size != count:
        raise ValueError("W['%s'] has %d entries, expected %d" % (name, out.size, count))
    return np.ascontiguousarray(out)


def make_scaling(W, ml, q, s, mnl=0):
    """reference W dict -> (ctypes Scaling, keep-alive list)"""
    keep = []

    def ptr(a):
        keep.append(a)
        return a.ctypes.data if a.size else None

    try:
        d = _flat([W["d"]], ml, "d")
        di = _flat([W["di"]], ml, "di")
    except KeyError:
        raise KeyError("missing item W['d'] or W['di']")       # misc_solvers.c:134
    v = _flat(W["v"], sum(q), "v")
    beta = np.ascontiguousarray(np.array([float(b) for b in W["beta"]], dtype=np.float64))
    if beta.size != len(q):
        raise ValueError("W['beta'] has %d entries, expected %d" % (beta.size, len(q)))
    r = _flat(W["r"], sum(k * k for k in s), "r")
    rti = _flat(W["rti"], sum(k * k for k in s), "rti")
    if mnl:
        dnl = _flat([W["dnl"]], mnl, "dnl")
        dnli = _flat([W["dnli"]], mnl, "dnli")
    else:
        dnl = dnli = np.zeros(0)
    sc = _lib.Scaling(ptr(dnl), ptr(dnli), ptr(d), ptr(di), ptr(v), ptr(beta), ptr(r), ptr(rti))
    return sc, keep


class KKTChol:
    """One `kkt_chol` factory instance: G (and optionally H) resident in HBM."""

    METHODS = {"chol": 0, "qr": 1, "ldl2": 2}

    def __init__(self, G, dims, A=None, mnl=0, H=None, device=0, method="chol", kktreg=0.0):
        self._lib = _lib.load()
        self._h = C.c_void_p()
        # a sparse G keeps its 'l' rows sparse; the QR route needs the dense W^{-T} G and densifies all of G, as the
        # reference does
        sparse = is_sparse(G) and method != "qr"
        if sparse:
            gshape, rowptr, colind, val = to_csr(G, "G")
        else:
            Gm = _dense(G, "G")
            gshape = Gm.shape
        self.n = gshape[1]
        self.dims = {"l": int(dims["l"]), "q": [int(k) for k in dims["q"]],
                     "s": [int(k) for k in dims["s"]]}
        self.mnl = int(mnl)
        self._cd, self._keep, self.cdim, self.cdim_pckd = make_dims(self.dims, self.mnl)
        if A is None:
            p = 0
            Am = None
        else:
            Am = _dense(A, "A")
            p = Am.shape[0]
            if p and Am.shape[1] != self.n:
                raise TypeError("A must have %d columns" % self.n)
        self.p = p
        # the reference allocates Gs as (cdim, n) and copies G into rows mnl: (misc.py:1252,1270)
        if gshape[0] != self.cdim - self.mnl:
            raise TypeError("G must be a 'd' matrix of size (%d, %d)" % (self.cdim - self.mnl, self.n))
        Ap = Am.ctypes.data if (Am is not None and p) else None
        if sparse:
            # rows [0, mnl) of the factory's G belong to Df: empty rows of the CSR
            rowptr = np.ascontiguousarray(np.concatenate([np.zeros(self.mnl, dtype=np.int64), rowptr]))
            rc = self._lib.cvxb_kkt_create_sparse(
                C.byref(self._h), self.n, p, C.byref(self._cd), rowptr.ctypes.data,
                colind.ctypes.data if colind.size else None, val.ctypes.data if val.size else None,
                int(val.size), Ap, max(1, p), _lib.HOST, device)
        else:
            if self.mnl:
                full = np.zeros((self.cdim, self.n), order="F")
                full[self.mnl:, :] = Gm
                Gm = full
            rc = self._lib.cvxb_kkt_create(
                C.byref(self._h), self.n, p, C.byref(self._cd), Gm.ctypes.data, max(1, Gm.shape[0]),
                Ap, max(1, p), _lib.HOST, device)
        _lib.check(rc, "kkt_chol")
        self.method = method
        if method != "chol":
            _lib.check(self._lib.cvxb_kkt_set_method(self._h, self.METHODS[method], float(kktreg)),
                       "kkt_%s" % method)
        self._H_resident = None
        if H is not None:
            self.set_H(H)

    def reset(self):
        """start a new solver run on this factory: the reference builds a fresh kkt_chol2 closure per run, whose
        `F['firstcall']` / `F['singular']` state (misc.py:1395-1447) this clears"""
        _lib.check(self._lib.cvxb_kkt_reset(self._h), "reset")

    # -- resident H ---------------------------------------------------------
    def set_H(self, H):
        Hm = _dense(H, "H")
        if Hm.shape != (self.n, self.n):
            raise TypeError("H must be a 'd' matrix of size (%d, %d)" % (self.n, self.n))
        _lib.check(self._lib.cvxb_kkt_set_H(self._h, Hm.ctypes.data, max(1, self.n), _lib.HOST), "set_H")
        self._H_resident = H

    # -- factor(W, H, Df) -> solve ------------------------------------------
    def factor(self, W, H=None, Df=None):
        sc, keep = make_scaling(W, self.dims["l"], self.dims["q"], self.dims["s"], self.mnl)
        # H is None            -> add the resident H if the factory was given one
        # H is the resident H  -> no re-upload
        # any other H          -> uploaded for this call (cvxprog passes a fresh H every time)
        use_res = 0
        Hp, ldh = None, 1
        if H is None or H is self._H_resident:
            use_res = 1 if self._H_resident is not None else 0
        else:
            Hm = _dense(H, "H")
            if Hm.shape != (self.n, self.n):
                raise TypeError("H must be a 'd' matrix of size (%d, %d)" % (self.n, self.n))
            keep.append(Hm)
            Hp, ldh = Hm.ctypes.data, max(1, self.n)
        Dp, lddf = None, 1
        if self.mnl:
            if Df is None:
                raise TypeError("Df is required when mnl > 0")
            Dm = _dense(Df, "Df")
            if Dm.shape != (self.mnl, self.n):
                raise TypeError("Df must be a 'd' matrix of size (%d, %d)" % (self.mnl, self.n))
            keep.append(Dm)
            Dp, lddf = Dm.ctypes.data, max(1, self.mnl)
        rc = self._lib.cvxb_kkt_factor(self._h, C.byref(sc), Hp, ldh, Dp, lddf, use_res, _lib.HOST)
        _lib.check(rc, "factor")
        return self.solve

    def solve(self, x, y, z):
        xv = _vec_inplace(x, self.n, "x")
        zv = _vec_inplace(z, self.cdim, "z")
        yp = None
        if self.p:
            yp = _vec_inplace(y, self.p, "y").ctypes.data
        rc = self._lib.cvxb_kkt_solve(self._h, xv.ctypes.data, yp, zv.ctypes.data, _lib.HOST)
        _lib.check(rc, "solve")

    __call__ = factor

    # -- device-resident operators for function-valued G / P -----------------
    def G(self, x, y, alpha=1.0, beta=0.0, trans="N"):
        """y := alpha*G*x + beta*y (trans 'N') or alpha*G'*x + beta*y ('T') on the resident G
        (the function-valued G protocol, reference coneprog.py:1682-1711)."""
        m = self.cdim - self.mnl
        nx, ny = (m, self.n) if trans == "T" else (self.n, m)
        xv = np.ascontiguousarray(np.asarray(x, dtype=np.float64).reshape(-1, order="F"))
        yv = _vec_inplace(y, ny, "y")
        if xv.size != nx:
            raise TypeError("x must have %d entries" % nx)
        rc = self._lib.cvxb_kkt_gemv_G(self._h, xv.ctypes.data, yv.ctypes.data, float(alpha),
                                       float(beta), ord(trans), _lib.HOST)
        _lib.check(rc, "G operator")

    def A(self, x, y, alpha=1.0, beta=0.0, trans="N"):
        """y := alpha*A*x + beta*y ('N') or alpha*A'*x + beta*y ('T') on the resident equality-constraint
        matrix (function-valued A protocol, reference coneprog.py:1682-1711)."""
        if not self.p:
            raise ValueError("this factory was created without equality constraints")
        nx, ny = (self.p, self.n) if trans == "T" else (self.n, self.p)
        xv = np.ascontiguousarray(np.asarray(x, dtype=np.float64).reshape(-1, order="F"))
        yv = _vec_inplace(y, ny, "y")
        if xv.size != nx:
            raise TypeError("x must have %d entries" % nx)
        rc = self._lib.cvxb_kkt_gemv_A(self._h, xv.ctypes.data, yv.ctypes.data, float(alpha),
                                       float(beta), ord(trans), _lib.HOST)
        _lib.check(rc, "A operator")

    def P(self, x, y, alpha=1.0, beta=0.0):
        """y := alpha*H*x + beta*y on the resident H (function-valued P protocol)."""
        xv = np.ascontiguousarray(np.asarray(x, dtype=np.float64).reshape(-1, order="F"))
        yv = _vec_inplace(y, self.n, "y")
        rc = self._lib.cvxb_kkt_symv_H(self._h, xv.ctypes.data, yv.ctypes.data, float(alpha),
                                       float(beta), _lib.HOST)
        _lib.check(rc, "P operator")

    # -- raw-pointer entry points (device-resident callers: bench.py, the device IPM) ----
    def factor_ptr(self, d=0, di=0, v=0, beta=0, r=0, rti=0, dnl=0, dnli=0, H=0, ldh=1,
                   use_resident_H=True, space=_lib.DEVICE):
        """cvxb_kkt_factor with raw addresses (ints) living in `space`."""
        sc = _lib.Scaling(dnl or None, dnli or None, d or None, di or None, v or None,
                          beta or None, r or None, rti or None)
        rc = self._lib.cvxb_kkt_factor(self._h, C.byref(sc), H or None, ldh, None, 1,
                                       1 if use_resident_H else 0, space)
        _lib.check(rc, "factor")

    def solve_ptr(self, x, z, y=0, space=_lib.DEVICE):
        _lib.check(self._lib.cvxb_kkt_solve(self._h, x, y or None, z, space), "solve")

    def timer_start(self):
        _lib.check(self._lib.cvxb_kkt_timer_start(self._h), "timer")

    def timer_stop(self):
        ms = C.c_double()
        _lib.check(self._lib.cvxb_kkt_timer_stop(self._h, C.byref(ms)), "timer")
        return ms.value

    # -- introspection ---------------------------------------------------------
    def last_ms(self):
        f, s = C.c_double(), C.c_double()
        self._lib.cvxb_kkt_last_ms(self._h, C.byref(f), C.byref(s))
        return f.value, s.value

    def last_breakdown(self):
        b = (C.c_double * 3)()
        self._lib.cvxb_kkt_last_breakdown(self._h, b)
        out = {"syrk_ms": b[0], "potrf_ms": b[1], "scale_ms": b[2]}
        mm = C.c_double()
        self._lib.cvxb_kkt_syrk_mma_ms(self._h, C.byref(mm))
        if mm.value > 0:
            out["syrk_mma_ms"] = mm.value        # int8-slice path: the MMA launches alone (without slicing kernels)
        return out

    def syrk_path(self):
        """'none' | 'dmma' | 'int8' | 'sparse': the kernel that computed the last factor's 'l'-row SYRK"""
        return ("none", "dmma", "int8", "sparse")[self._lib.cvxb_kkt_syrk_path(self._h)]

    def qr_passes(self):
        """QR route: 2 = Cholesky-QR with re-orthogonalisation, 3 = the shifted variant took over"""
        return self._lib.cvxb_kkt_qr_passes(self._h)

    def get_L(self):
        L = np.zeros((self.n, self.n), order="F")
        _lib.check(self._lib.cvxb_kkt_get_L(self._h, L.ctypes.data, max(1, self.n)), "get_L")
        return np.tril(L)

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            self._lib.cvxb_kkt_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def kkt_chol(G, dims, A=None, mnl=0, H=None, device=0):
    """Drop-in for `misc.kkt_chol(G, dims, A, mnl)` (reference misc.py:1213).

    Returns `factor(W, H=None, Df=None)`; `factor` returns `solve(x, y, z)`.
    Extra keyword `H`: a constant Hessian block (coneqp's P) made resident once,
    so `factor(W)` / `factor(W, P)` do not re-upload n^2 doubles per iteration.
    """
    return KKTChol(G, dims, A, mnl, H, device)


def cpl_kktsolver(F, G, dims, A=None, mnl=0, device=0):
    """`kktsolver(x, z, W)` for `cvxprog.cpl` backed by the device KKT path: what cpl builds itself for
    kktsolver='chol' (reference cvxprog.py:526-537) with misc.kkt_chol replaced by this library:

        factor = kkt_chol(G, dims, A, mnl);  kktsolver(x, z, W) = factor(W, H, Df)  with f, Df, H = F(x, z)

    G is uploaded once; each call uploads the fresh dense H (n x n) and Df (mnl x n)."""
    factor = KKTChol(G, dims, A, mnl, None, device)

    def kktsolver(x, z, W):
        f, Df, H = F(x, z)
        return factor(W, H, Df)
    kktsolver.factory = factor
    return kktsolver


def cp_kktsolver(F, G, dims, A=None, mnl=0, device=0):
    """`kktsolver(x, z, W)` for `cvxprog.cp` (reference cvxprog.py:1876-1887): F's first row is the objective,
    so the nonlinear constraint block is Df[1:, :] and `mnl` counts the nonlinear CONSTRAINTS only."""
    factor = KKTChol(G, dims, A, mnl, None, device)

    def kktsolver(x, z, W):
        f, Df, H = F(x, z)
        return factor(W, H, Df[1:, :])
    kktsolver.factory = factor
    return kktsolver


def kkt_chol2(G, dims, A=None, mnl=0, H=None, device=0):
    """Drop-in for `misc.kkt_chol2(G, dims, A, mnl)` (reference misc.py:1352-1567), the drivers'
    default for problems with only 'l' constraints (coneprog.py:458-462, 1805-1809).

    S = H + GG' W^-1 W^-T GG = L L', K = A S^-1 A' = Lk Lk' (first-call fallback S += A'A when K
    is singular, :1433-1447): exactly the elimination KKTChol runs, with diag(di) fused into the
    SYRK operand load.  Same error as the reference for 'q'/'s' cones (:1384-1387)."""
    if dims["q"] or dims["s"]:
        raise ValueError("kktsolver option 'kkt_chol2' is implemented only for problems with no "
                         "second-order or semidefinite cone constraints")
    return KKTChol(G, dims, A, mnl, H, device)


def kkt_ldl2(G, dims, A=None, mnl=0, H=None, device=0):
    """Drop-in for `misc.kkt_ldl2(G, dims, A, mnl)` (reference misc.py:1128-1210): the 2x2 system

        [ H + GG' W^-1 W^-T GG   A' ] [ux]   [bx + GG' W^-1 W^-T bz]
        [ A                      0  ] [uy] = [by]

    factored as P K P' = L D L' with Bunch-Kaufman pivoting on the device (the algorithm of lapack.sytrf, which the
    reference calls at :1172; csrc/kkt_ldl.cu) and solved with the sweeps of lapack.sytrs (:1196).  With no
    equality constraints the reference itself uses potrf (:1173), and so does this factory."""
    return KKTChol(G, dims, A, mnl, H, device, method="ldl2")


def kkt_qr(G, dims, A=None, device=0):
    """Drop-in for `misc.kkt_qr(G, dims, A)` (reference misc.py:1570-1699), the drivers' default for conelp with
    second-order / semidefinite cones (coneprog.py:458-462): zero (1,1) block, equality constraints eliminated
    with a Householder QR of A' (done once here), reduced system solved through  W^{-T} G Q2 = Q3 R3  instead of
    the normal equations.  `factor(W)` takes no H / Df (as in the reference)."""
    return KKTChol(G, dims, A, 0, None, device, method="qr")
