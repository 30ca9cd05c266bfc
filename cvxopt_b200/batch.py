"""Batch of independent dense QPs solved in lock-step on the device (BASELINE config 4).

    minimize 1/2 x'P x + q'x   subject to   G x + s = h,  s in K,   A x = b

K is one 'l' cone of m rows by default, or dims = {'l': ml, 'q': [...]} shared by every problem, and so is the
number p of equality rows (none by default).
The per-problem algorithm is coneprog.coneqp (reference src/python/coneprog.py:1998-2547) with
default options — kktsolver='chol', or 'chol2' for 'l'-only problems with A; same start, stopping rule, Mehrotra
steps and iterative refinement — so every problem converges in the same number of iterations as
`solvers.coneqp(P, q, G, h, dims, A, b)` (for dims={'l': m}: `solvers.qp(P, q, G, h, A, b)`) does.
The reference has no batch API; its counterpart is a Python loop over those calls.

Cone LPs  minimize c'x  subject to  G x + s = h,  s in K,  A x = b  run coneprog.conelp (coneprog.py:31-1436) in the
same lock-step machinery (ConeLPBatch, conelp_batch): a Python loop over `solvers.conelp(c, G, h, dims, A, b)`
(`solvers.lp` for dims={'l': m}), with its infeasibility certificates.

Dims with 's' blocks (orders <= 32) run through SDPBatch / sdp_batch (conelp) and SDPQPBatch / coneqp_batch (coneqp).
cpl problems with 's' blocks (nonlinear constraints next to an LMI) run through SDPCPLBatch / sdp_cpl_batch.
"""
import ctypes as C

import numpy as np

from . import _lib

STATUS = {0: "running", 1: "optimal", 2: "unknown", 3: "unknown", 4: "primal infeasible", 5: "dual infeasible"}
DEFAULTS = dict(maxiters=100, abstol=1e-7, reltol=1e-6, feastol=1e-7)   # coneprog.py:436-456
BATCH_MAX = 65535        # CVXB_BATCH_MAX: problems per cvxb_batch handle
BATCH_SMAX = 32          # CVXB_BATCH_SMAX: the largest 's' order of a batch


def _batch_dims(dims, m=None):
    """dims -> (ctypes Dims or None, keep-alive, cdim).  None is {'l': m}.  's' cones are not built for the batch."""
    if dims is None:
        return None, None, m
    from . import kkt
    dims = {"l": dims.get("l", 0), "q": list(dims.get("q", [])), "s": list(dims.get("s", []))}
    d, keep, cdim, _ = kkt.make_dims(dims)
    if dims["s"]:
        raise NotImplementedError("the batch solver has no 's' cones")
    if m is not None and int(m) != cdim:
        raise TypeError("m = %d does not match the cone dimension %d of dims" % (int(m), cdim))
    return d, keep, cdim


def _stack(P, q, G, h):
    """-> contiguous (B,n,n), (B,n), (B,n,m) [= m x n column-major per problem], (B,m)"""
    P = np.ascontiguousarray(np.asarray(P, dtype=np.float64))
    q = np.ascontiguousarray(np.asarray(q, dtype=np.float64))
    G = np.asarray(G, dtype=np.float64)
    h = np.ascontiguousarray(np.asarray(h, dtype=np.float64))
    if P.ndim != 3 or P.shape[1] != P.shape[2]:
        raise TypeError("P must have shape (B, n, n)")
    B, n = P.shape[0], P.shape[1]
    if q.shape != (B, n):
        raise TypeError("q must have shape (B, n)")
    if G.ndim != 3 or G.shape[0] != B or G.shape[2] != n:
        raise TypeError("G must have shape (B, m, n)")
    m = G.shape[1]
    if h.shape != (B, m):
        raise TypeError("h must have shape (B, m)")
    # P is symmetric: its row-major image equals its column-major image as far as tril goes
    Pcm = np.ascontiguousarray(np.transpose(P, (0, 2, 1)))
    Gcm = np.ascontiguousarray(np.transpose(G, (0, 2, 1)))      # (B, n, m): column-major m x n
    return Pcm, q, Gcm, h, B, n, m


def _eq_rows(A, b, B, n):
    """p, the number of equality rows of A (B, p, n) and b (B, p); 0 when both are None.  The shape checks are
    coneqp's TypeErrors (coneprog.py:1910-1925)."""
    if A is None and b is None:
        return 0
    if A is None or b is None:
        raise TypeError("'A' and 'b' must be given together")
    A, b = np.asarray(A), np.asarray(b)
    if A.ndim != 3 or A.shape[0] != B or A.shape[2] != n:
        raise TypeError("'A' must have shape (B, p, %d) with B = %d" % (n, B))
    if b.shape != (B, A.shape[1]):
        raise TypeError("'b' must have shape (B, %d)" % A.shape[1])
    return A.shape[1]


def _stack_eq(A, b, B, n):
    """-> contiguous (B,n,p) [= p x n column-major per problem], (B,p), p; (None, None, 0) without A"""
    p = _eq_rows(A, b, B, n)
    if A is None:
        return None, None, 0
    Acm = np.ascontiguousarray(np.transpose(np.asarray(A, dtype=np.float64), (0, 2, 1)))
    return Acm, np.ascontiguousarray(np.asarray(b, dtype=np.float64)), p


def _start_arrays(start, B, n, p, m, what="initvals"):
    """a start dict with keys among x, s, y, z -> {key: contiguous float64 (B, len)}: x (B, n), y (B, p), s and z
    (B, cdim) laid out as h.  An unknown key or a wrong shape is a TypeError"""
    if not isinstance(start, dict):
        raise TypeError("'%s' must be a dictionary" % what)
    lens = {"x": n, "s": m, "y": p, "z": m}
    out = {}
    for key, v in start.items():
        if key not in lens:
            raise TypeError("'%s' has an unknown key %r" % (what, key))
        a = np.ascontiguousarray(np.asarray(v, dtype=np.float64))
        if a.shape != (B, lens[key]):
            raise TypeError("%s['%s'] must have shape (%d, %d)" % (what, key, B, lens[key]))
        out[key] = a
    return out


def _lp_start(primalstart, dualstart, B, n, p, m):
    """conelp's primalstart {'x', 's'} and dualstart {'z'[, 'y']} -> one _start_arrays dict, or None without either"""
    start = {}
    if primalstart is not None:
        if not isinstance(primalstart, dict) or set(primalstart) != {"x", "s"}:
            raise TypeError("'primalstart' must be a dictionary with keys 'x' and 's'")
        start.update(_start_arrays(primalstart, B, n, p, m, "primalstart"))
    if dualstart is not None:
        if not isinstance(dualstart, dict) or "z" not in dualstart or not set(dualstart) <= {"y", "z"}:
            raise TypeError("'dualstart' must be a dictionary with key 'z' and optionally 'y'")
        start.update(_start_arrays(dualstart, B, n, p, m, "dualstart"))
    return start or None


def _sdp_start(primalstart, dualstart, B, n, p, ml, ms):
    """sdp's primalstart {'x', 'sl', 'ss'} and dualstart {'zl', 'zs'[, 'y']} -> conelp's, 'ss' / 'zs' lists of
    (B, ms, ms) unpacked column-major after the 'l' rows as _sdp_args assembles hs"""
    def stack(d, lk, sk, what):
        if ml and lk not in d or ms and sk not in d:
            raise TypeError("'%s' must have the keys %s" % (what, ", ".join(repr(k) for k in
                                                                           ([lk] if ml else []) + ([sk] if ms else []))))
        parts = []
        if ml:
            v = np.asarray(d[lk], dtype=np.float64)
            if v.shape != (B, ml):
                raise TypeError("%s['%s'] must have shape (%d, %d)" % (what, lk, B, ml))
            parts.append(v)
        if ms:
            blocks = d[sk]
            if not isinstance(blocks, list) or len(blocks) != len(ms):
                raise TypeError("%s['%s'] must be a list of %d arrays" % (what, sk, len(ms)))
            for k, (v, o) in enumerate(zip(blocks, ms)):
                v = np.asarray(v, dtype=np.float64)
                if v.shape != (B, o, o):
                    raise TypeError("%s['%s'][%d] must have shape (%d, %d, %d)" % (what, sk, k, B, o, o))
                parts.append(v.transpose(0, 2, 1).reshape(B, -1))
        return np.concatenate(parts, axis=1) if parts else np.zeros((B, 0))
    ps = ds = None
    if primalstart is not None:
        if not isinstance(primalstart, dict) or "x" not in primalstart or not set(primalstart) <= {"x", "sl", "ss"}:
            raise TypeError("'primalstart' must be a dictionary with keys 'x', 'sl' and 'ss'")
        ps = {"x": primalstart["x"], "s": stack(primalstart, "sl", "ss", "primalstart")}
    if dualstart is not None:
        if not isinstance(dualstart, dict) or not set(dualstart) <= {"y", "zl", "zs"}:
            raise TypeError("'dualstart' must be a dictionary with keys 'zl', 'zs' and optionally 'y'")
        ds = {"z": stack(dualstart, "zl", "zs", "dualstart")}
        if "y" in dualstart:
            ds["y"] = dualstart["y"]
    return _lp_start(ps, ds, B, n, p, ml + sum(k * k for k in ms))


def _sdp_dims(dims, m=None):
    """_batch_dims for SDPBatch: dims may hold 's' blocks"""
    from . import kkt
    dims = {"l": dims.get("l", 0), "q": list(dims.get("q", [])), "s": list(dims.get("s", []))}
    d, keep, cdim, _ = kkt.make_dims(dims)
    if m is not None and int(m) != cdim:
        raise TypeError("m = %d does not match the cone dimension %d of dims" % (int(m), cdim))
    return d, keep, cdim


ADJOINT_KEYS = ("P", "q", "G", "h", "A", "b")
QCQP_ADJOINT_KEYS = ("P", "q", "r", "G", "h", "A", "b")
CONELP_ADJOINT_KEYS = ("c", "G", "h", "A", "b")
GP_ADJOINT_KEYS = ("F", "g", "G", "h", "A", "b")
CP_ADJOINT_KEYS = ("ux", "uznl", "G", "h", "A", "b")
CPL_ADJOINT_KEYS = CP_ADJOINT_KEYS + ("c",)


def _adjoint_args(gx, gy, gz, want, B, n, p, m, keys=ADJOINT_KEYS):
    """the gradients gx (B, n), gy (B, p), gz (B, m) as contiguous float64 arrays (None stays None) and `want` as a
    tuple of `keys`; a wrong shape or an unknown key is a TypeError"""
    want = tuple(want)
    unknown = [k for k in want if k not in keys]
    if unknown:
        raise TypeError("want: unknown keys %s; the keys are %s" % (unknown, keys))
    gs = []
    for name, a, k in (("gx", gx, n), ("gy", gy, p), ("gz", gz, m)):
        if a is not None:
            a = np.ascontiguousarray(np.asarray(a, dtype=np.float64))
            if a.shape != (B, k):
                raise TypeError("%s must have shape (%d, %d)" % (name, B, k))
        gs.append(a)
    return gs, want


def _tangent_in(B, named):
    """data directions `named` ((name, array or None, per-problem shape, axes to the library's layout or None)) ->
    contiguous float64 host arrays in the library's layouts (None stays None); a wrong shape or dtype is a TypeError"""
    out = []
    for name, a, shape, axes in named:
        if a is not None:
            a = np.asarray(a)
            if a.dtype.kind != "f":
                raise TypeError("%s must be a float array, not %s" % (name, a.dtype))
            if a.shape != (B,) + tuple(shape):
                raise TypeError("%s must have shape %s" % (name, (B,) + tuple(shape)))
            a = a.astype(np.float64, copy=False)
            a = np.ascontiguousarray(a if axes is None else a.transpose(axes))
        out.append(a)
    return out


def _ptrs(arrays):
    return [None if a is None else a.ctypes.data for a in arrays]


_T2 = (0, 2, 1)          # a (B, rows, n) matrix to rows x n column-major per problem

# Every derivative call takes its kind's own block, which each batch class declares as `_block`, and then this linear
# tail, which all kinds share.  An entry is (the tangent's name for it, its per-problem shape as load() takes it, from
# the batch's n, m, p, mnl and K, the axes to the library's layout or None, whether the adjoint writes dL/d(the name
# without its first letter) itself).  The tangent reads every entry in order; the adjoint writes ux, uy, uz, then the
# entries it writes in order, and its other keys come from ux, uy and uz by _FROM_U.  A QP is the case mnl = 0.
_TAIL = (("dG", lambda b: (b.m - b.mnl, b.n), _T2, True), ("dh", lambda b: (b.m - b.mnl,), None, False),
         ("dA", lambda b: (b.p, b.n), _T2, True), ("db", lambda b: (b.p,), None, False))

# the adjoint's gradients from its ux, uy and uz: key -> (which of the three, the gradient from it).  dL/dq = dL/dc =
# -ux, dL/db = uy, dL/dh = uz's rows after the mnl nonlinear ones, and the CP adjoint's ux and uznl (uz's first rows)
_FROM_U = {"q": (0, lambda u, mnl: -u), "c": (0, lambda u, mnl: -u), "ux": (0, lambda u, mnl: u),
           "b": (1, lambda u, mnl: u), "h": (2, lambda u, mnl: u[:, mnl:]), "uznl": (2, lambda u, mnl: u[:, :mnl])}


def _lib_shape(shape, axes):
    """a per-problem shape in the library's layout: the axes of the (B,) + shape array, None: as it is"""
    return shape if axes is None else tuple(((0,) + tuple(shape))[a] for a in axes[1:])


def _inverse(axes):
    """the axes back from the library's layout"""
    return tuple(axes.index(k) for k in range(len(axes)))


class QPBatch:
    """dims: the reference's cone dimensions dict ('l' and 'q' only); m must equal its cdim.  None: {'l': m}.
    p: equality rows A x = b per problem (load() then takes A (B, p, n) and b (B, p))."""
    _lp = False              # ConeLPBatch: a batch of cone LPs
    _sdp = False             # SDPBatch, SDPQPBatch: dims may hold 's' blocks
    mnl = 0                  # rows of nonlinear constraints before G's: none in a QP or cone LP
    _block = (("dP", lambda b: (b.n, b.n), _T2, True), ("dq", lambda b: (b.n,), None, False))

    def __init__(self, nprob, n, m, device=0, dims=None, p=0):
        if not isinstance(p, (int, np.integer)) or isinstance(p, bool):
            raise TypeError("p must be an integer")
        d, keep, cdim = (_sdp_dims if self._sdp else _batch_dims)(dims, m)
        self._lib = _lib.load()
        self._h = C.c_void_p()
        self.B, self.n, self.m, self.p = int(nprob), int(n), int(cdim), int(p)
        if d is None and (self._lp or self.p):
            d, keep, _ = _batch_dims({"l": self.m})
        if self._sdp:
            create = self._lib.cvxb_batch_create_sdp if self._lp else self._lib.cvxb_batch_create_sdp_qp
            rc = create(C.byref(self._h), self.B, self.n, self.p, C.byref(d), device)
        elif self._lp:
            rc = self._lib.cvxb_batch_create_lp(C.byref(self._h), self.B, self.n, self.p, C.byref(d), device)
        elif self.p:
            rc = self._lib.cvxb_batch_create_eq(C.byref(self._h), self.B, self.n, self.p, C.byref(d), device)
        elif d is None:
            rc = self._lib.cvxb_batch_create(C.byref(self._h), self.B, self.n, self.m, device)
        else:
            rc = self._lib.cvxb_batch_create_cones(C.byref(self._h), self.B, self.n, C.byref(d), device)
        del keep
        _lib.check(rc, "batch")
        self._refinement = None

    def _host_eq(self, A, b):
        """host A (B, p, n) and b (B, p) in the layout cvxb_batch_load_eq takes, checked against the batch's p"""
        Acm, bv, p = _stack_eq(A, b, self.B, self.n)
        if p != self.p:
            raise TypeError("A has %d rows; the batch was created with p = %d" % (p, self.p))
        return Acm, bv

    def _load_eq(self, A, b, space):
        """A and b after the problem data, nothing without equality rows: _host_eq's arrays, or raw addresses in
        `space` of p x n column-major blocks and p-vectors"""
        if not self.p:
            return
        if A is None or b is None:
            raise TypeError("the batch has p = %d equality rows: give A and b" % self.p)
        if isinstance(A, np.ndarray):
            A, b = A.ctypes.data, b.ctypes.data
        _lib.check(self._lib.cvxb_batch_load_eq(self._h, A, b, space), "batch_load_eq")

    def load(self, P, q, G, h, A=None, b=None):
        Pcm, q, Gcm, h, B, n, m = _stack(P, q, G, h)
        if (B, n, m) != (self.B, self.n, self.m):
            raise TypeError("problem shapes do not match the batch")
        Acm, bv = self._host_eq(A, b)
        rc = self._lib.cvxb_batch_load(self._h, Pcm.ctypes.data, q.ctypes.data, Gcm.ctypes.data,
                                       h.ctypes.data, _lib.HOST)
        _lib.check(rc, "batch_load")
        self._load_eq(Acm, bv, _lib.HOST)

    def load_ptr(self, P, q, G, h, space=_lib.DEVICE, A=None, b=None):
        """raw addresses of already laid-out buffers (device-resident callers); A: p x n column-major per problem"""
        _lib.check(self._lib.cvxb_batch_load(self._h, P, q, G, h, space), "batch_load")
        self._load_eq(A, b, space)

    def load_start(self, x=None, s=None, y=None, z=None):
        """the starting point of the next solves, kept until load_start or clear_start: coneqp's initvals on a QP batch
        (absent keys: x = y = 0, s = z = e), conelp's primalstart (x and s) and / or dualstart (z, optionally y) on a
        cone LP batch.  x (B, n), y (B, p), s and z (B, cdim) laid out as h; only the lower triangle of an 's' block is
        read"""
        given = {k: v for k, v in (("x", x), ("s", s), ("y", y), ("z", z)) if v is not None}
        a = _start_arrays(given, self.B, self.n, self.p, self.m)
        self.load_start_ptr(*(a[k].ctypes.data if k in a else None for k in "xsyz"), space=_lib.HOST)

    def load_start_ptr(self, x=None, s=None, y=None, z=None, space=_lib.DEVICE):
        """load_start from raw addresses in `space` of (B, n), (B, cdim), (B, p) and (B, cdim) arrays; None: absent"""
        _lib.check(self._lib.cvxb_batch_load_start(self._h, x, s, y, z, space), "batch_load_start")

    def clear_start(self):
        """back to the cold start"""
        _lib.check(self._lib.cvxb_batch_clear_start(self._h), "batch_clear_start")

    def solve(self, refinement=None, **options):
        """refinement: steps of iterative refinement per Newton solve (coneqp's option); None keeps the default
        (1 with 'q' cones, else 0)"""
        o = dict(DEFAULTS)
        o.update(options)
        if refinement is not None and refinement != self._refinement:
            if not isinstance(refinement, (int, np.integer)) or isinstance(refinement, bool) or refinement < 0:
                raise ValueError("refinement must be a nonnegative integer")
            _lib.check(self._lib.cvxb_batch_set_refinement(self._h, int(refinement)), "batch_set_refinement")
            self._refinement = refinement
        rc = self._lib.cvxb_batch_solve(self._h, int(o["maxiters"]), float(o["abstol"]),
                                        float(o["reltol"]), float(o["feastol"]))
        if rc == _lib.E_ARG and ("Rank(" in _lib.last_error() or "is not positive" in _lib.last_error()):
            raise ValueError(_lib.last_error())       # coneprog.py:2065-2067, :2130, :2144
        _lib.check(rc, "batch_solve")

    def results(self):
        B, n, m = self.B, self.n, self.m
        x, s, z = np.zeros((B, n)), np.zeros((B, m)), np.zeros((B, m))
        status = np.zeros(B, dtype=np.int32)
        iters = np.zeros(B, dtype=np.int32)
        pobj, dobj = np.zeros(B), np.zeros(B)
        rc = self._lib.cvxb_batch_results(self._h, x.ctypes.data, s.ctypes.data, z.ctypes.data,
                                          status.ctypes.data, iters.ctypes.data, pobj.ctypes.data,
                                          dobj.ctypes.data, _lib.HOST)
        _lib.check(rc, "batch_results")
        y = np.zeros((B, self.p))
        if self.p:
            _lib.check(self._lib.cvxb_batch_results_y(self._h, y.ctypes.data, _lib.HOST), "batch_results_y")
        return {"x": x, "y": y, "s": s, "z": z, "status": [STATUS[int(k)] for k in status],
                "status_code": status, "iterations": iters, "primal objective": pobj,
                "dual objective": dobj}

    def adjoint(self, gx, gy=None, gz=None, want=ADJOINT_KEYS):
        """derivatives of the last solve's results for a loss L with gradients gx = dL/dx (B, n), gy = dL/dy (B, p)
        and gz = dL/dz (B, m), None meaning zero (cvxb_batch_adjoint).  Returns host arrays for the keys in `want`:
        P (B, n, n, symmetric), q (B, n), G (B, m, n), h (B, m), A (B, p, n) and b (B, p), each dL/d(that input).
        A problem whose status is not 'optimal' gets NaN.  QP batches whose rows are all 'l' only: any other batch
        raises NotImplementedError, and a batch not solved since its last load raises ValueError."""
        return self._adjoint(self.adjoint_ptr, QPBatch._block, ADJOINT_KEYS, gx, gy, gz, want)

    def adjoint_ptr(self, gx=None, gy=None, gz=None, ux=None, uy=None, uz=None, dP=None, dG=None, dA=None,
                    space=_lib.DEVICE):
        """cvxb_batch_adjoint on raw addresses in `space`, laid out as include/cvxopt_b200.h states; None: NULL"""
        _lib.check(self._lib.cvxb_batch_adjoint(self._h, gx, gy, gz, ux, uy, uz, dP, dG, dA, space), "batch_adjoint")

    _cone_keys = ADJOINT_KEYS            # the keys adjoint_cone takes in `want` (a cone LP: CONELP_ADJOINT_KEYS)

    def adjoint_cone(self, gx, gy=None, gz=None, want=None):
        """adjoint's derivatives on any QP or cone LP batch, with 'q' cones and 's' blocks (cvxb_batch_adjoint_cone).
        gz (B, m) and the returned h (B, m) and G (B, m, n) are laid out as h, each 's' block unpacked column-major:
        only the symmetric part of gz's blocks enters, and the outputs' blocks hold the same value in both triangles.
        want: keys of ADJOINT_KEYS, of CONELP_ADJOINT_KEYS on a cone LP batch (c for q, no P); None: all of them."""
        keys = self._cone_keys
        return self._adjoint(self.adjoint_cone_ptr, QPBatch._block, keys, gx, gy, gz, keys if want is None else want)

    def adjoint_cone_ptr(self, gx=None, gy=None, gz=None, ux=None, uy=None, uz=None, dP=None, dG=None, dA=None,
                         space=_lib.DEVICE):
        """cvxb_batch_adjoint_cone on raw addresses in `space`, laid out as include/cvxopt_b200.h states; None: NULL"""
        _lib.check(self._lib.cvxb_batch_adjoint_cone(self._h, gx, gy, gz, ux, uy, uz, dP, dG, dA, space),
                   "batch_adjoint_cone")

    def tangent(self, dP=None, dq=None, dG=None, dh=None, dA=None, db=None):
        """forward-mode derivatives of the last solve's results along the data direction (dP, dq, dG, dh, dA, db) in
        load()'s shapes, None meaning zero (cvxb_batch_tangent): returns host arrays dx (B, n), dy (B, p) and dz
        (B, m), z's 's' blocks unpacked as h's.  A non-symmetric dP, and 's' blocks of dh and dG's columns, enter
        through their symmetric parts.  Every QP batch; a cone LP batch takes dc in place of dq and no dP.  A problem
        whose status is not 'optimal' gets NaN; a batch not solved since its last load raises ValueError."""
        return self._tangent(self.tangent_ptr, QPBatch._block, (dP, dq, dG, dh, dA, db))

    def tangent_ptr(self, dP=None, dq=None, dG=None, dh=None, dA=None, db=None, dx=None, dy=None, dz=None,
                    space=_lib.DEVICE):
        """cvxb_batch_tangent on raw addresses in `space`, laid out as include/cvxopt_b200.h states; None: NULL"""
        _lib.check(self._lib.cvxb_batch_tangent(self._h, dP, dq, dG, dh, dA, db, dx, dy, dz, space), "batch_tangent")

    def _adjoint(self, ptr, block, keys, gx, gy, gz, want):
        """the adjoint call `ptr` (an *_ptr) of the kind whose own block is `block`, with the gradients gx, gy, gz and
        `want` among `keys` -> {key: host array in load()'s layout}"""
        B = self.B
        gs, want = _adjoint_args(gx, gy, gz, want, B, self.n, self.p, self.m, keys)
        own = {name[1:]: (shape(self), axes) for name, shape, axes, writes in block + _TAIL if writes}
        us = [np.empty((B, w)) if any(_FROM_U[k][0] == i for k in want if k not in own) else None
              for i, w in enumerate((self.n, self.p, self.m))]
        outs = {k: np.empty((B,) + _lib_shape(*own[k])) for k in own if k in want}
        ptr(*_ptrs(gs + us + [outs.get(k) for k in own]), space=_lib.HOST)
        got = {k: v if own[k][1] is None else v.transpose(_inverse(own[k][1])) for k, v in outs.items()}
        return {k: np.ascontiguousarray(got[k] if k in got else _FROM_U[k][1](us[_FROM_U[k][0]], self.mnl))
                for k in want}

    def _tangent(self, ptr, block, dirs):
        """the tangent call `ptr` (a *_ptr) of the kind whose own block is `block` along dirs, the caller's arrays for
        block + _TAIL (None: zero) -> host dx (B, n), dy (B, p), dz (B, m)"""
        d = _tangent_in(self.B, [(name, a, shape(self), axes)
                                 for (name, shape, axes, _), a in zip(block + _TAIL, dirs)])
        out = [np.empty((self.B, w)) for w in (self.n, self.p, self.m)]
        ptr(*_ptrs(d + out), space=_lib.HOST)
        return tuple(out)

    def stats(self):
        ms, it = C.c_double(), C.c_int()
        self._lib.cvxb_batch_stats(self._h, C.byref(ms), C.byref(it))
        return {"solve_ms": ms.value, "lockstep_iterations": it.value,
                "syrk_path": ("none", "dmma", "int8")[self._lib.cvxb_batch_syrk_path(self._h)]}

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            self._lib.cvxb_batch_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _split(n, parts):
    base, extra = divmod(n, parts)
    out, lo = [], 0
    for r in range(parts):
        hi = lo + base + (1 if r < extra else 0)
        out.append((lo, hi))
        lo = hi
    return out


class QPBatchGroup:
    """`nsub` QPBatch objects over interleaved slices of one batch, solved CONCURRENTLY on their own CUDA streams
    (one host thread each; ctypes releases the GIL inside the library calls).  A lock-step batch alternates
    throughput-bound phases (batched SYRK / GEMV) with latency-bound ones (the chain of diagonal-block
    factorisations, the flag-chained triangular solves); with two or more sub-batches in flight the GPU runs one
    sub-batch's latency-bound phase under another's throughput-bound phase, and a sub-batch stops iterating as soon
    as ITS slowest problem is done.  Interleaved slices (problem i -> sub-batch i mod nsub) spread hard and easy
    problems evenly."""

    @staticmethod
    def _part():
        """the kind of batch each slice is (ConeLPBatchGroup: ConeLPBatch)"""
        return QPBatch

    def __init__(self, nprob, n, m, device=0, nsub=None, dims=None, p=0):
        if nsub is None:
            # a few sub-batches let the finished problems of one leave the lock-step loop early (counts chosen
            # when the kernels were tuned, not re-measured on H100; CVXB_BATCH_NSUB overrides)
            nsub = int(__import__("os").environ.get("CVXB_BATCH_NSUB", "0")) or (
                2 if nprob >= 256 else (max(1, min(8, nprob // 8)) if nprob >= 16 else 1))
        # one library batch holds at most BATCH_MAX problems (include/cvxopt_b200.h): larger batches take more parts
        self.nsub = max(1, min(int(nsub), nprob), -(-int(nprob) // BATCH_MAX))
        self.B, self.n, self.m, self.p = int(nprob), int(n), int(m), int(p)
        self.idx = [np.arange(r, self.B, self.nsub) for r in range(self.nsub)]
        self.parts = []
        eq = {"p": self.p} if self.p else {}
        try:
            for ix in self.idx:
                self.parts.append(self._part()(len(ix), n, m, device, dims, **eq))
        except BaseException:
            self.close()
            raise

    def load_ptr_sliced(self, loader):
        """loader(part_index, indices, QPBatch) loads one sub-batch (device-resident callers)"""
        for r, (ix, b) in enumerate(zip(self.idx, self.parts)):
            loader(r, ix, b)

    def load(self, P, q, G, h, A=None, b=None):
        self._load_sliced((P, q, G, h), A, b)

    def _load_sliced(self, data, A, b):
        """each part loads its slice of the per-problem arrays `data`, then of A and b"""
        data = [np.asarray(a) for a in data]
        if A is not None:
            A = np.asarray(A)
        if b is not None:
            b = np.asarray(b)
        for ix, part in zip(self.idx, self.parts):
            part.load(*(a[ix] for a in data), None if A is None else A[ix], None if b is None else b[ix])

    def load_start(self, x=None, s=None, y=None, z=None):
        """QPBatch.load_start on every part with its slice of the arrays"""
        given = {k: v for k, v in (("x", x), ("s", s), ("y", y), ("z", z)) if v is not None}
        a = _start_arrays(given, self.B, self.n, self.p, self.m)
        for ix, part in zip(self.idx, self.parts):
            part.load_start(**{k: v[ix] for k, v in a.items()})

    def clear_start(self):
        for part in self.parts:
            part.clear_start()

    def solve(self, **options):
        if self.nsub == 1:
            self.parts[0].solve(**options)
            return
        import threading
        errs = []

        def run(b):
            try:
                b.solve(**options)
            except BaseException as e:      # noqa: BLE001  re-raised on the calling thread
                errs.append(e)
        th = [threading.Thread(target=run, args=(b,)) for b in self.parts]
        for t in th:
            t.start()
        for t in th:
            t.join()
        if errs:
            raise errs[0]

    def results(self):
        B, n, m = self.B, self.n, self.m
        out = {"x": np.zeros((B, n)), "y": np.zeros((B, self.p)), "s": np.zeros((B, m)), "z": np.zeros((B, m)),
               "status_code": np.zeros(B, dtype=np.int32), "iterations": np.zeros(B, dtype=np.int32),
               "primal objective": np.zeros(B), "dual objective": np.zeros(B)}
        for ix, b in zip(self.idx, self.parts):
            r = b.results()
            for key in out:
                out[key][ix] = r[key]
        out["status"] = [STATUS[int(k)] for k in out["status_code"]]
        return out

    _adjoint_keys = ADJOINT_KEYS         # the keys each part's adjoint takes in `want`
    _cone_keys = ADJOINT_KEYS            # and its adjoint_cone

    def adjoint(self, gx, gy=None, gz=None, want=ADJOINT_KEYS):
        """QPBatch.adjoint on every part with its slice of the gradients, the results in problem order"""
        return self._adjoint_parts("adjoint", self._adjoint_keys, gx, gy, gz, want)

    def adjoint_cone(self, gx, gy=None, gz=None, want=None):
        """QPBatch.adjoint_cone on every part with its slice of the gradients, the results in problem order"""
        keys = self._cone_keys
        return self._adjoint_parts("adjoint_cone", keys, gx, gy, gz, keys if want is None else want)

    def _adjoint_parts(self, method, keys, gx, gy, gz, want):
        """the parts' adjoint `method` with their slices of the gradients, `want` among `keys` -> {key: array} in
        problem order"""
        gs, want = _adjoint_args(gx, gy, gz, want, self.B, self.n, self.p, self.m, keys)
        out = {}
        for ix, part in zip(self.idx, self.parts):
            r = getattr(part, method)(*(None if a is None else a[ix] for a in gs), want=want)
            for k, v in r.items():
                out.setdefault(k, np.empty((self.B,) + v.shape[1:]))[ix] = v
        return out

    def _tangent_parts(self, method, dirs):
        """the parts' `method` with their slices of the directions dirs -> dx, dy, dz in problem order"""
        dirs = [None if a is None else np.asarray(a) for a in dirs]
        if any(a is not None and (a.ndim < 1 or a.shape[0] != self.B) for a in dirs):
            raise TypeError("every direction must have leading dimension B = %d" % self.B)
        out = None
        for ix, part in zip(self.idx, self.parts):
            r = getattr(part, method)(*(None if a is None else a[ix] for a in dirs))
            if out is None:
                out = [np.empty((self.B,) + v.shape[1:]) for v in r]
            for o, v in zip(out, r):
                o[ix] = v
        return tuple(out)

    def tangent(self, dP=None, dq=None, dG=None, dh=None, dA=None, db=None):
        """QPBatch.tangent on every part with its slice of the direction, the results in problem order"""
        return self._tangent_parts("tangent", (dP, dq, dG, dh, dA, db))

    def stats(self):
        st = [b.stats() for b in self.parts]
        return {"solve_ms": max(s["solve_ms"] for s in st),
                "lockstep_iterations": max(s["lockstep_iterations"] for s in st),
                "lockstep_iterations_per_subbatch": [s["lockstep_iterations"] for s in st],
                "syrk_path": st[0]["syrk_path"], "nsub": self.nsub}

    def close(self):
        for b in self.parts:
            b.close()


class ConeLPBatch(QPBatch):
    """B cone LPs  min c'x  s.t.  G x + s = h,  s in K,  A x = b  (B x coneprog.conelp with default options, kktsolver
    'chol2' for 'l'-only problems, 'chol' with 'q' cones).  dims: 'l' and 'q' only, None is {'l': m}; m = cdim >= 1.
    p: equality rows per problem.  The constructor, solve / results / stats / close are QPBatch's;
    results()["status"] is one of 'optimal', 'primal infeasible', 'dual infeasible' or 'unknown', with NaN where
    conelp returns None."""
    _lp = True
    _cone_keys = CONELP_ADJOINT_KEYS
    _block = (QPBatch._block[0], ("dc", lambda b: (b.n,), None, False))      # P is never given: its address is NULL

    def load(self, c, G, h, A=None, b=None):
        c = np.ascontiguousarray(np.asarray(c, dtype=np.float64))
        h = np.ascontiguousarray(np.asarray(h, dtype=np.float64))
        G = np.asarray(G, dtype=np.float64)
        B, n, m = self.B, self.n, self.m
        if c.shape != (B, n) or G.shape != (B, m, n) or h.shape != (B, m):
            raise TypeError("problem shapes do not match the batch")
        Acm, bv = self._host_eq(A, b)
        Gcm = np.ascontiguousarray(np.transpose(G, (0, 2, 1)))
        _lib.check(self._lib.cvxb_batch_load_lp(self._h, c.ctypes.data, Gcm.ctypes.data, h.ctypes.data, _lib.HOST),
                   "batch_load_lp")
        self._load_eq(Acm, bv, _lib.HOST)

    def load_ptr(self, c, G, h, space=_lib.DEVICE, A=None, b=None):
        """raw addresses of already laid-out buffers: c (B, n), G m x n column-major per problem, h (B, m), A p x n
        column-major per problem, b (B, p)"""
        _lib.check(self._lib.cvxb_batch_load_lp(self._h, c, G, h, space), "batch_load_lp")
        self._load_eq(A, b, space)

    def tangent(self, dc=None, dG=None, dh=None, dA=None, db=None):
        """QPBatch.tangent along (dc, dG, dh, dA, db): a cone LP has no P"""
        return self._tangent(self.tangent_ptr, ConeLPBatch._block, (None, dc, dG, dh, dA, db))


class ConeLPBatchGroup(QPBatchGroup):
    """QPBatchGroup's interleaved sub-batches, solved concurrently, for cone LPs"""
    _cone_keys = CONELP_ADJOINT_KEYS

    @staticmethod
    def _part():
        return ConeLPBatch

    def load(self, c, G, h, A=None, b=None):
        self._load_sliced((c, G, h), A, b)

    def tangent(self, dc=None, dG=None, dh=None, dA=None, db=None):
        """ConeLPBatch.tangent on every part with its slice of the direction, the results in problem order"""
        return self._tangent_parts("tangent", (dc, dG, dh, dA, db))


def _lp_shapes(c, G, h, dims, A, b):
    """conelp's argument checks (coneprog.py:487-562) on the batch: -> B, n, cdim, p"""
    c, G, h = np.asarray(c), np.asarray(G), np.asarray(h)
    if c.ndim != 2:
        raise TypeError("'c' must have shape (B, n): one column per problem")
    B, n = c.shape
    if h.ndim != 2 or h.shape[0] != B:
        raise TypeError("'h' must have shape (B, cdim): one column per problem")
    cdim = h.shape[1] if dims is None else _batch_dims(dims)[2]
    if h.shape[1] != cdim:
        raise TypeError("'h' must be a 'd' matrix of size (%d,1)" % cdim)
    if G.ndim != 3 or G.shape != (B, cdim, n):
        raise TypeError("'G' must be a 'd' matrix of size (%d, %d)" % (cdim, n))
    if (A is None) != (b is None):
        raise TypeError("'A' and 'b' must be given together")
    p = 0
    if A is not None:
        A, b = np.asarray(A), np.asarray(b)
        if A.ndim != 3 or A.shape[0] != B or A.shape[2] != n:
            raise TypeError("'A' must be a 'd' matrix with %d columns " % n)
        p = A.shape[1]
        if b.shape != (B, p):
            raise TypeError("'b' must have length %d" % p)
    if p > n or p + cdim < n:
        raise ValueError("Rank(A) < p or Rank([G; A]) < n")          # coneprog.py:572-573
    return B, n, cdim, p


def conelp_batch(c, G, h, dims=None, A=None, b=None, device=0, nsub=None, primalstart=None, dualstart=None,
                 **options):
    """Solve B independent cone LPs on one GPU, each as solvers.conelp(c, G, h, dims, A, b) does.  c (B,n),
    G (B,cdim,n), h (B,cdim); optional A (B,p,n), b (B,p), given together.  dims: shared by every problem ('l' and
    'q' only); None is {'l': cdim}, i.e. solvers.lp.  nsub and the returned dict are qp_batch's; status is 'optimal',
    'primal infeasible', 'dual infeasible' or 'unknown', and entries the reference returns as None are NaN.
    primalstart {'x': (B,n), 's': (B,cdim)} and dualstart {'z': (B,cdim), 'y': (B,p) optional} are conelp's.
    options: maxiters, abstol, reltol, feastol, refinement (as conelp's)."""
    B, n, cdim, p = _lp_shapes(c, G, h, dims, A, b)
    start = _lp_start(primalstart, dualstart, B, n, p, cdim)
    return _run_group(ConeLPBatchGroup(B, n, cdim, device, nsub, dims, p), (c, G, h, A, b), options, start)


class SDPBatch(ConeLPBatch):
    """ConeLPBatch whose dims may hold 's' blocks of order <= 32 (cvxb_batch_create_sdp): B x conelp(c, G, h, dims, A,
    b) with kktsolver 'chol'.  load() takes conelp's stacked c (B, n), G (B, cdim, n), h (B, cdim), with each 's'
    block's rows unpacked column-major; only the lower triangle of an 's' block of G and h is read, and results()
    returns s and z with symmetric 's' blocks."""
    _sdp = True

    def __init__(self, nprob, n, dims, p=0, device=0):
        super().__init__(nprob, n, None, device, dims, p)


class SDPBatchGroup(ConeLPBatchGroup):
    """ConeLPBatchGroup of SDPBatch parts"""

    def __init__(self, nprob, n, dims, p=0, device=0, nsub=None):
        super().__init__(nprob, n, _sdp_dims(dims)[2], device, nsub, dims, p)

    @staticmethod
    def _part():
        return lambda nprob, n, m, device, dims, p=0: SDPBatch(nprob, n, dims, p, device)


def _sdp_args(c, Gl, hl, Gs, hs, A, b):
    """sdp's argument checks (coneprog.py:3846-3888) on the batch -> c, G, h, dims, A, b, ms as conelp takes them"""
    c = np.asarray(c, dtype=np.float64) if c is not None else None
    if c is None or c.ndim != 2:
        raise TypeError("'c' must be a dense column matrix")
    B, n = c.shape
    if n < 1:
        raise ValueError("number of variables must be at least 1")
    Gl = np.zeros((B, 0, n)) if Gl is None else np.asarray(Gl, dtype=np.float64)
    if Gl.ndim != 3 or Gl.shape[0] != B or Gl.shape[2] != n:
        raise TypeError("'Gl' must be a dense or sparse 'd' matrix with %d columns" % n)
    ml = Gl.shape[1]
    hl = np.zeros((B, 0)) if hl is None else np.asarray(hl, dtype=np.float64)
    if hl.shape != (B, ml):
        raise TypeError("'hl' must be a 'd' matrix of size (%d,1)" % ml)
    Gs = [] if Gs is None else Gs
    if not isinstance(Gs, list) or [G for G in Gs if np.ndim(G) != 3 or np.shape(G)[0] != B or np.shape(G)[2] != n]:
        raise TypeError("'Gs' must be a list of sparse or dense 'd' matrices with %d columns" % n)
    ms = [int(np.sqrt(np.shape(G)[1])) for G in Gs]
    a = [k for k in range(len(ms)) if ms[k] ** 2 != np.shape(Gs[k])[1]]
    if a:
        raise TypeError("the squareroot of the number of rows in 'Gs[%d]' is not an integer" % a[-1])
    hs = [] if hs is None else hs
    if not isinstance(hs, list) or len(hs) != len(ms) or [h for h in hs if np.ndim(h) != 3 or np.shape(h)[0] != B]:
        raise TypeError("'hs' must be a list of %d dense or sparse 'd' matrices" % len(ms))
    a = [k for k in range(len(ms)) if np.shape(hs[k])[1:] != (ms[k], ms[k])]
    if a:
        k = a[0]
        raise TypeError("hs[%d] has size (%d,%d).  Expected size is (%d,%d)."
                        % (k, np.shape(hs[k])[1], np.shape(hs[k])[2], ms[k], ms[k]))
    A = np.zeros((B, 0, n)) if A is None else np.asarray(A, dtype=np.float64)
    if A.ndim != 3 or A.shape[0] != B or A.shape[2] != n:
        raise TypeError("'A' must be a dense or sparse 'd' matrix with %d columns" % n)
    p = A.shape[1]
    b = np.zeros((B, 0)) if b is None else np.asarray(b, dtype=np.float64)
    if b.shape != (B, p):
        raise TypeError("'b' must be a dense matrix of size (%d,1)" % p)
    G = np.concatenate([Gl] + [np.asarray(G, dtype=np.float64) for G in Gs], axis=1)
    h = np.concatenate([hl] + [np.asarray(h, dtype=np.float64).transpose(0, 2, 1).reshape(B, -1) for h in hs], axis=1)
    if p > n or p + ml + sum(k * (k + 1) // 2 for k in ms) < n:
        raise ValueError("Rank(A) < p or Rank([G; A]) < n")          # conelp, coneprog.py:572-573
    return c, G, h, {"l": ml, "q": [], "s": ms}, A, b, ms


def sdp_batch(c, Gl=None, hl=None, Gs=None, hs=None, A=None, b=None, device=0, nsub=None, primalstart=None,
              dualstart=None, **options):
    """Solve B independent SDPs on one GPU, each as solvers.sdp(c, Gl, hl, Gs, hs, A, b, kktsolver='chol') does.
    c (B, n), Gl (B, ml, n), hl (B, ml), Gs a list of (B, ms², n), hs a list of (B, ms, ms), A (B, p, n), b (B, p);
    every 's' order at most 32.  Returns sdp's keys x, sl, ss (list of (B, ms, ms)), y, zl, zs, status, status_code,
    iterations, primal objective, dual objective, with conelp_batch's stats; NaN where sdp returns None.
    primalstart {'x', 'sl', 'ss'} and dualstart {'zl', 'zs', 'y'} are sdp's, in the shapes of x, hl, hs and b; 'sl' /
    'zl' are needed when ml > 0, 'ss' / 'zs' when there are 's' blocks, and 'y' is optional (0 without it).
    options: maxiters, abstol, reltol, feastol, refinement (as sdp's)."""
    c, G, h, dims, A, b, ms = _sdp_args(c, Gl, hl, Gs, hs, A, b)
    B, n = c.shape
    p = A.shape[1]
    start = _sdp_start(primalstart, dualstart, B, n, p, dims["l"], ms)
    out = _run_group(SDPBatchGroup(B, n, dims, p, device, nsub), (c, G, h, A if p else None, b if p else None),
                     options, start)
    ml = dims["l"]
    for key in ("s", "z"):
        v = out.pop(key)
        out[key + "l"] = v[:, :ml]
        blocks, o = [], ml
        for k in ms:
            blocks.append(v[:, o:o + k * k].reshape(B, k, k).transpose(0, 2, 1).copy())
            o += k * k
        out[key + "s"] = blocks
    return out


class SDPQPBatch(QPBatch):
    """QPBatch whose dims may hold 's' blocks of order <= 32 (cvxb_batch_create_sdp_qp): B x coneqp(P, q, G, h, dims,
    A, b).  load() takes QPBatch's P (B, n, n), q (B, n), G (B, cdim, n), h (B, cdim), with each 's' block's rows
    unpacked column-major; only the lower triangle of an 's' block of G and h is read, and results() returns s and z
    with symmetric 's' blocks."""
    _sdp = True

    def __init__(self, nprob, n, dims, p=0, device=0):
        super().__init__(nprob, n, None, device, dims, p)


class SDPQPBatchGroup(QPBatchGroup):
    """QPBatchGroup of SDPQPBatch parts"""

    def __init__(self, nprob, n, dims, p=0, device=0, nsub=None):
        super().__init__(nprob, n, _sdp_dims(dims)[2], device, nsub, dims, p)

    @staticmethod
    def _part():
        return lambda nprob, n, m, device, dims, p=0: SDPQPBatch(nprob, n, dims, p, device)


def coneqp_batch(P, q, G, h, dims, A=None, b=None, device=0, nsub=None, initvals=None, **options):
    """Solve B independent cone QPs on one GPU, each as solvers.coneqp(P, q, G, h, dims, A, b) does.  P (B,n,n),
    q (B,n), G (B,cdim,n), h (B,cdim); optional A (B,p,n), b (B,p), given together.  dims: shared by every problem,
    with 'l', 'q' and 's' (orders at most 32); each 's' block's rows of G and h are unpacked column-major, as the
    reference's G, and only their lower triangles are read.  nsub and the returned dict are qp_batch's; its s and z
    have symmetric 's' blocks.  initvals: qp_batch's.  options: maxiters, abstol, reltol, feastol, refinement (as
    coneqp's)."""
    _, _, _, _, B, n, m = _stack(P, q, G, h)
    _sdp_dims(dims, m)
    p = _eq_rows(A, b, B, n)
    if p > n:
        raise ValueError("Rank(A) < p or Rank([P; G; A]) < n")        # coneprog.py:1970-1971
    start = None if initvals is None else _start_arrays(initvals, B, n, p, m)
    return _run_group(SDPQPBatchGroup(B, n, dims, p, device, nsub), (P, q, G, h, A, b), options, start)


class GPBatch(QPBatch):
    """B geometric programs (cvxb_batch_create_gp): B x solvers.gp(K, F, g, G, h, A, b), cpl's lock-step iteration on
    gp's epigraph problem.  K (block sizes of F, mnl = len(K) - 1), ml rows of G and p rows of A are shared by the
    batch.  load() takes F (B, sum K, n), g (B, sum K), G (B, ml, n), h (B, ml) and, with p > 0, A (B, p, n), b (B, p).
    results()' s and z are [snl; sl] and [znl; zl] (mnl + ml columns); its primal objective is gp's t."""
    _block = (("dF", lambda b: (sum(b.K), b.n), _T2, True), ("dg", lambda b: (sum(b.K),), None, True))

    def __init__(self, nprob, n, K, ml, p=0, device=0):
        K = [int(k) for k in K]
        self._lib = _lib.load()
        self._h = C.c_void_p()
        self.B, self.n, self.K, self.p = int(nprob), int(n), K, int(p)
        self.mnl, self.ml = len(K) - 1, int(ml)
        self.m = self.mnl + self.ml
        karr = (C.c_int * max(1, len(K)))(*K)
        rc = self._lib.cvxb_batch_create_gp(C.byref(self._h), self.B, self.n, len(K), karr, self.ml, self.p, device)
        _lib.check(rc, "batch")
        self._refinement = None

    def load(self, F, g, G, h, A=None, b=None):
        B, n, S = self.B, self.n, sum(self.K)
        F = np.asarray(F, dtype=np.float64)
        g = np.ascontiguousarray(np.asarray(g, dtype=np.float64))
        G = np.zeros((B, 0, n)) if G is None else np.asarray(G, dtype=np.float64)
        h = np.zeros((B, 0)) if h is None else np.ascontiguousarray(np.asarray(h, dtype=np.float64))
        if F.shape != (B, S, n) or g.shape != (B, S) or G.shape != (B, self.ml, n) or h.shape != (B, self.ml):
            raise TypeError("problem shapes do not match the batch")
        Acm, bv = self._host_eq(A, b)
        Fcm = np.ascontiguousarray(np.transpose(F, (0, 2, 1)))
        Gcm = np.ascontiguousarray(np.transpose(G, (0, 2, 1)))
        self.load_ptr(Fcm.ctypes.data, g.ctypes.data, Gcm.ctypes.data if self.ml else None,
                      h.ctypes.data if self.ml else None, _lib.HOST, Acm, bv)

    def load_ptr(self, F, g, G, h, space=_lib.DEVICE, A=None, b=None):
        """cvxb_batch_load_gp on raw addresses in `space` (device-resident callers): F sum K x n column-major per
        problem, g, G ml x n column-major and h (None when ml = 0); A p x n column-major and b"""
        _lib.check(self._lib.cvxb_batch_load_gp(self._h, F, g, G, h, space), "batch_load_gp")
        self._load_eq(A, b, space)

    def adjoint_gp(self, gx, gy=None, gz=None, want=GP_ADJOINT_KEYS):
        """derivatives of the last solve's results for a loss L with gradients gx = dL/dx (B, n), gy = dL/dy (B, p)
        and gz = dL/dz (B, mnl + ml, laid out as [znl, zl]), None meaning zero (cvxb_batch_adjoint_gp).  Returns host
        arrays for the keys in `want`, each dL/d(that input) in load()'s layout: F (B, sum K, n), g (B, sum K),
        G (B, ml, n), h (B, ml), A (B, p, n) and b (B, p).  A problem whose status is not 'optimal' gets NaN.  A batch
        not solved since its last load raises ValueError."""
        return self._adjoint(self.adjoint_gp_ptr, GPBatch._block, GP_ADJOINT_KEYS, gx, gy, gz, want)

    def adjoint_gp_ptr(self, gx=None, gy=None, gz=None, ux=None, uy=None, uz=None, dF=None, dg=None, dG=None,
                       dA=None, space=_lib.DEVICE):
        """cvxb_batch_adjoint_gp on raw addresses in `space`, laid out as include/cvxopt_b200.h states; None: NULL"""
        _lib.check(self._lib.cvxb_batch_adjoint_gp(self._h, gx, gy, gz, ux, uy, uz, dF, dg, dG, dA, space),
                   "batch_adjoint_gp")

    def tangent_gp(self, dF=None, dg=None, dG=None, dh=None, dA=None, db=None):
        """forward-mode derivatives of the last solve's results along the direction (dF, dg, dG, dh, dA, db) in
        load()'s shapes, None meaning zero (cvxb_batch_tangent_gp): returns host arrays dx (B, n), dy (B, p) and dz
        (B, mnl + ml, laid out as [znl, zl]).  A problem whose status is not 'optimal' gets NaN"""
        return self._tangent(self.tangent_gp_ptr, GPBatch._block, (dF, dg, dG, dh, dA, db))

    def tangent_gp_ptr(self, dF=None, dg=None, dG=None, dh=None, dA=None, db=None, dx=None, dy=None, dz=None,
                       space=_lib.DEVICE):
        """cvxb_batch_tangent_gp on raw addresses in `space`, laid out as include/cvxopt_b200.h states; None: NULL"""
        _lib.check(self._lib.cvxb_batch_tangent_gp(self._h, dF, dg, dG, dh, dA, db, dx, dy, dz, space),
                   "batch_tangent_gp")

    def stats(self):
        out = super().stats()
        out["line_search_rounds"] = self._lib.cvxb_batch_ls_rounds(self._h)
        return out


class GPBatchGroup(QPBatchGroup):
    """QPBatchGroup's interleaved sub-batches, solved concurrently, for geometric programs"""

    def __init__(self, nprob, n, K, ml, p=0, device=0, nsub=None):
        self._K, self._ml = list(K), int(ml)
        super().__init__(nprob, n, len(K) - 1 + int(ml), device, nsub, None, p)

    def _part(self):
        return lambda nprob, n, m, device, dims, p=0: GPBatch(nprob, n, self._K, self._ml, p, device)

    def load(self, F, g, G, h, A=None, b=None):
        self._load_sliced((F, g, G, h), A, b)

    def tangent_gp(self, dF=None, dg=None, dG=None, dh=None, dA=None, db=None):
        """GPBatch.tangent_gp on every part with its slice of the direction, the results in problem order"""
        return self._tangent_parts("tangent_gp", (dF, dg, dG, dh, dA, db))

    def adjoint_gp(self, gx, gy=None, gz=None, want=GP_ADJOINT_KEYS):
        """GPBatch.adjoint_gp on every part with its slice of the gradients, the results in problem order"""
        return self._adjoint_parts("adjoint_gp", GP_ADJOINT_KEYS, gx, gy, gz, want)

    def stats(self):
        out = super().stats()
        out["line_search_rounds"] = max(b._lib.cvxb_batch_ls_rounds(b._h) for b in self.parts)
        return out


def _gp_args(K, F, g, G, h, A, b):
    """gp's argument checks (cvxprog.py:2056-2092) on the batch -> F, g, G, h, A, b with the defaults filled in"""
    if type(K) is not list or [k for k in K if type(k) is not int or k <= 0]:
        raise TypeError("'K' must be a list of positive integers")
    S = sum(K)
    F = np.asarray(F) if F is not None else None
    if F is None or F.ndim != 3 or F.shape[1] != S or F.dtype.kind != "f":
        raise TypeError("'F' must be a dense or sparse 'd' matrix with %d rows" % S)
    B, n = F.shape[0], F.shape[2]
    g = np.asarray(g) if g is not None else None
    if g is None or g.shape != (B, S) or g.dtype.kind != "f":
        raise TypeError("'g' must be a dene 'd' matrix of size (%d,1)" % S)
    G = np.zeros((B, 0, n)) if G is None else np.asarray(G)
    if G.ndim != 3 or G.shape[0] != B or G.shape[2] != n or G.dtype.kind != "f":
        raise TypeError("'G' must be a dense or sparse 'd' matrix with %d columns" % n)
    ml = G.shape[1]
    h = np.zeros((B, 0)) if h is None else np.asarray(h)
    if h.shape != (B, ml) or h.dtype.kind != "f":
        raise TypeError("'h' must be a dense 'd' matrix of size (%d,1)" % ml)
    A = np.zeros((B, 0, n)) if A is None else np.asarray(A)
    if A.ndim != 3 or A.shape[0] != B or A.shape[2] != n or A.dtype.kind != "f":
        raise TypeError("'A' must be a dense or sparse 'd' matrix with %d columns" % n)
    p = A.shape[1]
    b = np.zeros((B, 0)) if b is None else np.asarray(b)
    if b.shape != (B, p) or b.dtype.kind != "f":
        raise TypeError("'b' must be a dense 'd' matrix of size (%d,1)" % p)
    if p > n:
        raise ValueError("Rank(A) < p or Rank([H(x); A; Df(x); G]) < n")
    return F, g, G, h, A, b


def gp_batch(K, F, g, G=None, h=None, A=None, b=None, device=0, nsub=None, **options):
    """Solve B independent geometric programs on one GPU, each as solvers.gp(K, F, g, G, h, A, b) does:
    minimize log sum exp(F0 x + g0) s.t. log sum exp(Fi x + gi) <= 0, G x <= h, A x = b.  K (list of block sizes) is
    shared by the batch; F (B, sum K, n), g (B, sum K), G (B, ml, n), h (B, ml), A (B, p, n), b (B, p), the last four
    optional.  Returns gp's x, snl, sl, znl, zl, y, status ('optimal' or 'unknown'), iterations, primal objective and
    dual objective, with the batch's stats (solve_ms, lock-step iterations, line-search rounds).  nsub is qp_batch's.
    options: maxiters, abstol, reltol, feastol, refinement (as gp's)."""
    F, g, G, h, A, b = _gp_args(K, F, g, G, h, A, b)
    B, n, p, mnl = F.shape[0], F.shape[2], A.shape[1], len(K) - 1
    out = _run_group(GPBatchGroup(B, n, K, G.shape[1], p, device, nsub), (F, g, G, h, A if p else None,
                                                                           b if p else None), options)
    for key in ("s", "z"):
        v = out.pop(key)
        out[key + "nl"], out[key + "l"] = v[:, :mnl], v[:, mnl:]
    return out


class _DevArray:
    """a device buffer of the batch handle, for torch.as_tensor (__cuda_array_interface__, no copy)"""

    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {"data": (ptr, False), "shape": shape, "typestr": typestr, "version": 2}


def _calling_F(b, call, name, *args):
    """the library call call(b's handle, *args), which may run b's F: an exception F raised comes out unchanged, else
    the return code is checked (any batch: the library refuses the kinds without F)"""
    b._err = None
    rc = call(b._h, *args)
    err, b._err = b._err, None
    if err is not None:
        raise err
    _lib.check(rc, name)


class CPBatch(QPBatch):
    """B smooth convex programs (cvxb_batch_create_cp): B x solvers.cp(F, G, h, dims={'l': ml}, A, b), the GP batch's
    lock-step cpl on cp's epigraph problem with F evaluated by the caller's batched F on the device.  mnl, ml rows of
    G and p rows of A are shared by the batch.  load() takes x0 (B, n), G (B, ml, n), h (B, ml) and, with p > 0,
    A (B, p, n), b (B, p); set_F() takes cp_batch's F.  `index` is each problem's index in the caller's order, passed to
    F as idx.  results()' s and z are [snl; sl] and [znl; zl]; its primal objective is cp's t."""
    _epi = 1                 # rows of F's f and Df before the mnl: cp's objective (CPLBatch: none)
    # dc (a cpl batch only) and F's parameter terms tx and tf; the adjoint writes none of them
    _block = (("dc", lambda b: (b.n,), None, False), ("tx", lambda b: (b.n,), None, False),
              ("tf", lambda b: (b.mnl,), None, False))

    def __init__(self, nprob, n, mnl, ml, p=0, device=0, index=None):
        self._lib = _lib.load()
        self._h = C.c_void_p()
        self.B, self.n, self.p, self.device = int(nprob), int(n), int(p), int(device)
        self.mnl, self.ml = int(mnl), int(ml)
        self.m = self.mnl + self.ml
        self._nf = self.mnl + self._epi
        _lib.check(self._create(), "batch")
        self._refinement = None
        self.index = np.arange(self.B) if index is None else np.asarray(index)
        self._cb = None
        self._err = None

    def _create(self):
        return self._lib.cvxb_batch_create_cp(C.byref(self._h), self.B, self.n, self.mnl, self.ml, self.p, self.device)

    def load(self, x0, G, h, A=None, b=None):
        B, n = self.B, self.n
        x0 = np.ascontiguousarray(np.asarray(x0, dtype=np.float64))
        G = np.zeros((B, 0, n)) if G is None else np.asarray(G, dtype=np.float64)
        h = np.zeros((B, 0)) if h is None else np.ascontiguousarray(np.asarray(h, dtype=np.float64))
        if x0.shape != (B, n) or G.shape != (B, self.ml, n) or h.shape != (B, self.ml):
            raise TypeError("problem shapes do not match the batch")
        Acm, bv = self._host_eq(A, b)
        Gcm = np.ascontiguousarray(np.transpose(G, (0, 2, 1)))
        self.load_ptr(x0.ctypes.data, Gcm.ctypes.data if self.ml else None, h.ctypes.data if self.ml else None,
                      _lib.HOST, Acm, bv)

    def load_ptr(self, x0, G, h, space=_lib.DEVICE, A=None, b=None):
        """cvxb_batch_load_cp on raw addresses in `space` (device-resident callers): x0, G ml x n column-major and h
        (None when ml = 0); A p x n column-major and b"""
        _lib.check(self._lib.cvxb_batch_load_cp(self._h, x0, G, h, space), "batch_load_cp")
        self._load_eq(A, b, space)

    _cp_keys = CP_ADJOINT_KEYS           # the keys adjoint_cp takes in `want` (a cpl batch's add c)

    def adjoint_cp(self, gx, gy=None, gz=None, want=None):
        """derivatives of the last solve's results for a loss L with gradients gx = dL/dx (B, n), gy = dL/dy (B, p)
        and gz = dL/dz (B, mnl + ml, laid out as [znl, zl]), None meaning zero (cvxb_batch_adjoint_cp).  F is called
        once more, at the returned x.  Returns host arrays for the keys in `want` (None: all of them): the adjoint
        solution's ux (B, n) and uznl (B, mnl), which give a parameter t of F its dL/dt = -d_t[ux' Df' zk + uk' f]
        (zk = [1; znl] and uk = [0; uznl] here, znl and uznl on a cpl batch), and dL/d(input) in load()'s layout:
        G (B, ml, n), h (B, ml), A (B, p, n), b (B, p) and, on a cpl batch, c (B, n).  A problem whose status is not
        'optimal', or whose F(x, z) there is not finite, gets NaN.  An exception raised in F comes out unchanged; a
        batch not solved since its last load raises ValueError, and a QCQP batch NotImplementedError."""
        keys = self._cp_keys
        return self._adjoint(self.adjoint_cp_ptr, CPBatch._block, keys, gx, gy, gz, keys if want is None else want)

    def adjoint_cp_ptr(self, gx=None, gy=None, gz=None, ux=None, uy=None, uz=None, dG=None, dA=None,
                       space=_lib.DEVICE):
        """cvxb_batch_adjoint_cp on raw addresses in `space`, laid out as include/cvxopt_b200.h states; None: NULL.
        An exception raised in F comes out unchanged, as from solve()"""
        _calling_F(self, self._lib.cvxb_batch_adjoint_cp, "batch_adjoint_cp", gx, gy, gz, ux, uy, uz, dG, dA, space)

    def tangent_cp(self, dc=None, tx=None, tf=None, dG=None, dh=None, dA=None, db=None):
        """forward-mode derivatives of the last solve's results along dc (B, n, a cpl batch only), dG (B, ml, n), dh
        (B, ml), dA (B, p, n), db (B, p) and a direction dt of F's parameters t, which enters through tx = d_t[Df(x;
        t)' zk] dt (B, n) and tf = d_t[f_nl(x; t)] dt (B, mnl) at the returned x (zk = [1; znl], cpl: znl); None
        means zero (cvxb_batch_tangent_cp).  F is called once more, at the returned x.  Returns host arrays dx (B, n),
        dy (B, p) and dz (B, mnl + ml, laid out as [znl, zl]).  A problem whose status is not 'optimal', or whose
        F(x, z) there is not finite, gets NaN.  An exception raised in F comes out unchanged"""
        if dc is not None and self._epi:
            raise TypeError("a cp batch has no c: its objective is f_0, and F's parameters enter through tx and tf")
        return self._tangent(self.tangent_cp_ptr, CPBatch._block, (dc, tx, tf, dG, dh, dA, db))

    def tangent_cp_ptr(self, dc=None, tx=None, tf=None, dG=None, dh=None, dA=None, db=None, dx=None, dy=None,
                       dz=None, space=_lib.DEVICE):
        """cvxb_batch_tangent_cp on raw addresses in `space`, laid out as include/cvxopt_b200.h states; None: NULL.
        An exception raised in F comes out unchanged"""
        _calling_F(self, self._lib.cvxb_batch_tangent_cp, "batch_tangent_cp", dc, tx, tf, dG, dh, dA, db, dx, dy, dz,
                   space)

    def set_F(self, F):
        """F(x, idx=idx) -> (f, Df) and F(x, z, idx=idx) -> (f, Df, H), as cp_batch takes it.  The callback runs F on
        the batch's stream and copies what it returns into the handle's buffers; an exception in F is kept and
        re-raised by solve()"""
        import torch
        dev = torch.device("cuda", self.device)
        B, n, nf = self.B, self.n, self._nf
        gidx = torch.as_tensor(self.index, dtype=torch.int64, device=dev)
        views, streams = {}, {}

        def view(ptr, shape, typestr="<f8"):
            t = views.get((ptr, shape))
            if t is None:
                t = views[ptr, shape] = torch.as_tensor(_DevArray(ptr, (B,) + shape, typestr), device=dev)
            return t

        def check(v, shape, which, rows, cols):
            if not isinstance(v, torch.Tensor) or v.dtype != torch.float64 or tuple(v.shape) != shape or \
                    v.device != dev:
                raise TypeError("%s output argument of F() must be a 'd' matrix of size (%d,%d): a float64 tensor "
                                "of shape %s on %s" % (which, rows, cols, shape, dev))
            return v

        def cb(ctx, k, full, x, z, problem, f, Df, H, stream):
            try:
                st = streams.get(stream)
                if st is None:
                    st = streams[stream] = torch.cuda.ExternalStream(stream, device=dev)
                with torch.cuda.device(dev), torch.cuda.stream(st):
                    idx = gidx[view(problem, (), "<i4")[:k].long()]
                    X = view(x, (n,))[:k]
                    Z = (view(z, (nf,))[:k] if nf else X.new_zeros((k, 0))) if full else None
                    out = F(X, Z, idx=idx) if full else F(X, idx=idx)
                    if not isinstance(out, (tuple, list)) or len(out) != (3 if full else 2):
                        raise TypeError("F(x, z) must return (f, Df, H)" if full else "F(x) must return (f, Df)")
                    fv = check(out[0], (k, nf), "first", nf, 1)
                    Dfv = check(out[1], (k, nf, n), "second", nf, n)
                    if nf:
                        view(f, (nf,))[:k].copy_(fv)
                        view(Df, (nf, n))[:k].copy_(Dfv)
                    if full:
                        view(H, (n, n))[:k].copy_(check(out[2], (k, n, n), "third", n, n))
                return 0
            except BaseException as e:      # noqa: BLE001  re-raised by solve()
                self._err = e
                return 1
        self._cb = _lib.CP_EVAL_FN(cb)
        _lib.check(self._lib.cvxb_batch_set_cp_eval(self._h, C.cast(self._cb, C.c_void_p), None), "batch_set_cp_eval")

    def solve(self, refinement=None, **options):
        """QPBatch.solve; an exception raised in F comes out unchanged, and a problem named in an error is named by its
        index in the caller's order"""
        import re
        self._err = None
        try:
            super().solve(refinement, **options)
        except ValueError as e:
            err, self._err = self._err, None
            if err is not None:
                raise err
            k = re.search(r"problem (\d+):", str(e))
            if k is None:
                raise
            raise ValueError(str(e).replace(k.group(0), "problem %d:" % self.index[int(k.group(1))], 1)) from None

    def stats(self):
        out = super().stats()
        out["line_search_rounds"] = self._lib.cvxb_batch_ls_rounds(self._h)
        return out

    def close(self):
        super().close()
        self._cb = None


class CPBatchGroup(QPBatchGroup):
    """QPBatchGroup's interleaved sub-batches, solved concurrently, for convex programs.  Each sub-batch calls F from
    its own host thread; F holds the GIL, so evaluations of different sub-batches run one at a time while their CUDA
    work overlaps"""

    def __init__(self, nprob, n, mnl, ml, p=0, device=0, nsub=None):
        self._mnl, self._ml = int(mnl), int(ml)
        super().__init__(nprob, n, self._mnl + self._ml, device, nsub, None, p)
        for ix, part in zip(self.idx, self.parts):
            part.index = ix

    def _part(self):
        return lambda nprob, n, m, device, dims, p=0: CPBatch(nprob, n, self._mnl, self._ml, p, device)

    def set_F(self, F):
        for part in self.parts:
            part.set_F(F)

    def load(self, x0, G, h, A=None, b=None):
        self._load_sliced((x0, G, h), A, b)

    def tangent_cp(self, dc=None, tx=None, tf=None, dG=None, dh=None, dA=None, db=None):
        """CPBatch.tangent_cp on every part with its slice of the direction, the results in problem order"""
        return self._tangent_parts("tangent_cp", (dc, tx, tf, dG, dh, dA, db))

    def adjoint_cp(self, gx, gy=None, gz=None, want=None):
        """CPBatch.adjoint_cp on every part with its slice of the gradients, the results in problem order"""
        keys = self.parts[0]._cp_keys
        return self._adjoint_parts("adjoint_cp", keys, gx, gy, gz, keys if want is None else want)

    def stats(self):
        out = super().stats()
        out["line_search_rounds"] = max(b._lib.cvxb_batch_ls_rounds(b._h) for b in self.parts)
        return out


def _cp_args(F, G, h, dims, A, b):
    """cp's argument checks (cvxprog.py:1653-1728) on the batch -> mnl, x0, G, h, A, b with the defaults filled in"""
    try:
        mnl, x0 = F()
    except Exception:
        raise ValueError("function call 'F()' failed") from None
    if type(mnl) is not int or mnl < 0:
        raise TypeError("the first output of F() must be a nonnegative integer")
    if hasattr(x0, "detach"):
        x0 = x0.detach().cpu().numpy()
    x0 = np.asarray(x0)
    if x0.ndim != 2 or x0.dtype != np.float64:
        raise TypeError("'x0' must be a 'd' matrix with one column: a float64 array of shape (B, n)")
    B, n = x0.shape
    G, h, A, b = _cp_rows(B, n, G, h, dims, A, b)
    return mnl, x0, G, h, A, b


def _cp_rows(B, n, G, h, dims, A, b):
    """cp's checks of G, h, dims, A and b (cvxprog.py:1653-1728) for B problems with n variables -> G, h, A, b with the
    defaults filled in; 'q' and 's' cones raise NotImplementedError and p > n the Rank ValueError"""
    if dims is not None and (dims.get("q") or dims.get("s")):
        raise NotImplementedError("the CP batch takes 'l' inequalities only (dims without 'q' and 's' cones)")
    h = np.zeros((B, 0)) if h is None else np.asarray(h)
    if h.ndim != 2 or h.shape[0] != B or h.dtype.kind != "f":
        raise TypeError("'h' must be a 'd' matrix with one column")
    ml = h.shape[1] if not dims else int(dims.get("l", 0))
    if h.shape[1] != ml:
        raise TypeError("'h' must be a 'd' matrix of size (%d,1)" % ml)
    G = np.zeros((B, 0, n)) if G is None else np.asarray(G)
    if G.shape != (B, ml, n) or G.dtype.kind != "f":
        raise TypeError("'G' must be a 'd' matrix with size (%d, %d)" % (ml, n))
    A = np.zeros((B, 0, n)) if A is None else np.asarray(A)
    if A.ndim != 3 or A.shape[0] != B or A.shape[2] != n or A.dtype.kind != "f":
        raise TypeError("'A' must be a 'd' matrix with %d columns" % n)
    p = A.shape[1]
    b = np.zeros((B, 0)) if b is None else np.asarray(b)
    if b.ndim != 2 or b.shape[0] != B or b.dtype.kind != "f":
        raise TypeError("'b' must be a 'd' matrix with one column")
    if b.shape[1] != p:
        raise TypeError("'b' must have length %d" % p)
    if p > n:
        raise ValueError("Rank(A) < p or Rank([H(x); A; Df(x); G]) < n")
    return G, h, A, b


def cp_batch(F, G=None, h=None, dims=None, A=None, b=None, device=0, nsub=None, **options):
    """Solve B independent smooth convex programs on one GPU, each as solvers.cp(F, G, h, dims, A, b) does:
    minimize f0(x) s.t. fk(x) <= 0 (k = 1..mnl), G x <= h, A x = b.  F is batched, with float64 torch tensors on the
    device:
      F() -> (mnl, x0): mnl shared by the batch, x0 (B, n) strictly inside dom f (numpy array or tensor), called once;
      F(x, idx=idx) -> (f, Df): x (k, n) the points of k problems, idx (k,) int64 their indices in x0's order,
          f (k, mnl + 1), Df (k, mnl + 1, n).  A row of f with a NaN or an infinite entry means x is not in dom f;
          F must accept such points without raising;
      F(x, z, idx=idx) -> (f, Df, H): z (k, mnl + 1), H (k, n, n) = sum_i z_i grad² f_i(x), only its lower triangle
          read.
    F runs on the batch's CUDA stream and must return the same values for the same point.  G (B, ml, n), h (B, ml),
    A (B, p, n), b (B, p) are optional; dims, if given, is {'l': ml}.  Returns cp's x, snl, sl, znl, zl, y, status
    ('optimal' or 'unknown'), iterations, primal objective and dual objective, with the batch's stats (solve_ms,
    lock-step iterations, line-search rounds, nsub, solve_wall_ms).  nsub is qp_batch's.
    options: maxiters, abstol, reltol, feastol, refinement (as cp's)."""
    mnl, x0, G, h, A, b = _cp_args(F, G, h, dims, A, b)
    B, n, p = x0.shape[0], x0.shape[1], A.shape[1]
    grp = CPBatchGroup(B, n, mnl, G.shape[1], p, device, nsub)
    try:
        grp.set_F(F)
    except BaseException:
        grp.close()
        raise
    out = _run_group(grp, (x0, G, h, A if p else None, b if p else None), options)
    for key in ("s", "z"):
        v = out.pop(key)
        out[key + "nl"], out[key + "l"] = v[:, :mnl], v[:, mnl:]
    return out


class QCQPBatch(CPBatch):
    """B convex QCQPs (cvxb_batch_create_qcqp): B x solvers.cp(F, G, h, dims={'l': ml}, A, b) with f_i(x) = x'P_i x / 2
    + q_i'x + r_i (i = 0..mnl), the CP batch with F evaluated by the library's kernels (no set_F, no host callback).
    mnl, ml rows of G and p rows of A are shared by the batch.  load() takes P (B, mnl + 1, n, n), of which only each
    P_i's lower triangle is read, q (B, mnl + 1, n), r (B, mnl + 1), x0 (B, n) or None for 0, G (B, ml, n), h (B, ml)
    and, with p > 0, A (B, p, n), b (B, p).  results() are CPBatch's."""
    # P per problem the (mnl + 1) n x n column-major stack [P_0; ...; P_mnl]: column j holds P_0[:, j], P_1[:, j], ...
    _block = (("dP", lambda b: (b.mnl + 1, b.n, b.n), (0, 3, 1, 2), True),
              ("dq", lambda b: (b.mnl + 1, b.n), None, True), ("dr", lambda b: (b.mnl + 1,), None, True))

    def _create(self):
        return self._lib.cvxb_batch_create_qcqp(C.byref(self._h), self.B, self.n, self.mnl, self.ml, self.p,
                                                self.device)

    def load(self, P, q, r, x0, G, h, A=None, b=None):
        B, n, nK = self.B, self.n, self.mnl + 1
        P = np.asarray(P, dtype=np.float64)
        q = np.ascontiguousarray(np.asarray(q, dtype=np.float64))
        r = np.ascontiguousarray(np.asarray(r, dtype=np.float64))
        x0 = np.zeros((B, n)) if x0 is None else np.ascontiguousarray(np.asarray(x0, dtype=np.float64))
        G = np.zeros((B, 0, n)) if G is None else np.asarray(G, dtype=np.float64)
        h = np.zeros((B, 0)) if h is None else np.ascontiguousarray(np.asarray(h, dtype=np.float64))
        if P.shape != (B, nK, n, n) or q.shape != (B, nK, n) or r.shape != (B, nK) or x0.shape != (B, n) or \
                G.shape != (B, self.ml, n) or h.shape != (B, self.ml):
            raise TypeError("problem shapes do not match the batch")
        Acm, bv = self._host_eq(A, b)
        # per problem the (nK n) x n column-major stack [P_0; ...; P_mnl]: column j holds P_0[:, j], P_1[:, j], ...
        Pcm = np.ascontiguousarray(np.transpose(P, (0, 3, 1, 2)))
        Gcm = np.ascontiguousarray(np.transpose(G, (0, 2, 1)))
        self.load_ptr(Pcm.ctypes.data, q.ctypes.data, r.ctypes.data, x0.ctypes.data,
                      Gcm.ctypes.data if self.ml else None, h.ctypes.data if self.ml else None, _lib.HOST, Acm, bv)

    def load_ptr(self, P, q, r, x0, G, h, space=_lib.DEVICE, A=None, b=None):
        """cvxb_batch_load_qcqp on raw addresses in `space` (device-resident callers): P the (mnl + 1) n x n
        column-major stack per problem, q, r, x0 (None: 0), G ml x n column-major, h; A p x n column-major and b"""
        _lib.check(self._lib.cvxb_batch_load_qcqp(self._h, P, q, r, x0, G, h, space), "batch_load_qcqp")
        self._load_eq(A, b, space)

    def adjoint(self, gx, gy=None, gz=None, want=QCQP_ADJOINT_KEYS):
        """derivatives of the last solve's results for a loss L with gradients gx = dL/dx (B, n), gy = dL/dy (B, p)
        and gz = dL/dz (B, mnl + ml, laid out as [znl, zl]), None meaning zero (cvxb_batch_adjoint_qcqp).  Returns
        host arrays for the keys in `want`, each dL/d(that input) in load()'s layout: P (B, mnl + 1, n, n, each block
        symmetric), q (B, mnl + 1, n), r (B, mnl + 1), G (B, ml, n), h (B, ml), A (B, p, n) and b (B, p).  A problem
        whose status is not 'optimal' gets NaN.  A batch not solved since its last load raises ValueError."""
        return self._adjoint(self.adjoint_ptr, QCQPBatch._block, QCQP_ADJOINT_KEYS, gx, gy, gz, want)

    def adjoint_ptr(self, gx=None, gy=None, gz=None, ux=None, uy=None, uz=None, dP=None, dq=None, dr=None, dG=None,
                    dA=None, space=_lib.DEVICE):
        """cvxb_batch_adjoint_qcqp on raw addresses in `space`, laid out as include/cvxopt_b200.h states; None: NULL"""
        _lib.check(self._lib.cvxb_batch_adjoint_qcqp(self._h, gx, gy, gz, ux, uy, uz, dP, dq, dr, dG, dA, space),
                   "batch_adjoint_qcqp")

    def tangent(self, dP=None, dq=None, dr=None, dG=None, dh=None, dA=None, db=None):
        """forward-mode derivatives of the last solve's results along the direction (dP, dq, dr, dG, dh, dA, db) in
        load()'s shapes, None meaning zero (cvxb_batch_tangent_qcqp): returns host arrays dx (B, n), dy (B, p) and dz
        (B, mnl + ml, laid out as [znl, zl]).  A non-symmetric dP_i enters through its symmetric part.  A problem
        whose status is not 'optimal' gets NaN"""
        return self._tangent(self.tangent_ptr, QCQPBatch._block, (dP, dq, dr, dG, dh, dA, db))

    def tangent_ptr(self, dP=None, dq=None, dr=None, dG=None, dh=None, dA=None, db=None, dx=None, dy=None, dz=None,
                    space=_lib.DEVICE):
        """cvxb_batch_tangent_qcqp on raw addresses in `space`, laid out as include/cvxopt_b200.h states; None:
        NULL"""
        _lib.check(self._lib.cvxb_batch_tangent_qcqp(self._h, dP, dq, dr, dG, dh, dA, db, dx, dy, dz, space),
                   "batch_tangent_qcqp")


class QCQPBatchGroup(CPBatchGroup):
    """QPBatchGroup's interleaved sub-batches, solved concurrently on their own streams, for convex QCQPs; nothing
    calls back to the host, so the sub-batches never wait on each other"""

    _adjoint_keys = QCQP_ADJOINT_KEYS

    def _part(self):
        return lambda nprob, n, m, device, dims, p=0: QCQPBatch(nprob, n, self._mnl, self._ml, p, device)

    def load(self, P, q, r, x0, G, h, A=None, b=None):
        self._load_sliced((P, q, r, x0, G, h), A, b)

    def adjoint(self, gx, gy=None, gz=None, want=QCQP_ADJOINT_KEYS):
        """QCQPBatch.adjoint on every part with its slice of the gradients, the results in problem order"""
        return super().adjoint(gx, gy, gz, want)

    def tangent(self, dP=None, dq=None, dr=None, dG=None, dh=None, dA=None, db=None):
        """QCQPBatch.tangent on every part with its slice of the direction, the results in problem order"""
        return self._tangent_parts("tangent", (dP, dq, dr, dG, dh, dA, db))


def _qcqp_args(P, q, r, G, h, dims, A, b, x0):
    """qcqp_batch's checks: P, q, r and x0 with cp's wording, then _cp_rows' -> P, q, r, x0, G, h, A, b as float64
    arrays with the defaults filled in"""
    P = np.asarray(P)
    if P.ndim != 4 or P.shape[1] < 1 or P.shape[2] != P.shape[3] or P.shape[2] < 1 or P.dtype.kind != "f":
        raise TypeError("'P' must be a 'd' array of shape (B, mnl + 1, n, n)")
    B, nK, n = P.shape[:3]
    q = np.asarray(q)
    if q.shape != (B, nK, n) or q.dtype.kind != "f":
        raise TypeError("'q' must be a 'd' array of shape (%d, %d, %d)" % (B, nK, n))
    r = np.asarray(r)
    if r.shape != (B, nK) or r.dtype.kind != "f":
        raise TypeError("'r' must be a 'd' array of shape (%d, %d)" % (B, nK))
    x0 = np.zeros((B, n)) if x0 is None else np.asarray(x0)
    if x0.shape != (B, n) or x0.dtype.kind != "f":
        raise TypeError("'x0' must be a 'd' matrix with one column: a float64 array of shape (%d, %d)" % (B, n))
    G, h, A, b = _cp_rows(B, n, G, h, dims, A, b)
    f64 = [np.asarray(a, dtype=np.float64) for a in (P, q, r, x0, G, h, A, b)]
    return tuple(f64)


def qcqp_batch(P, q, r, G=None, h=None, dims=None, A=None, b=None, x0=None, device=0, nsub=None, **options):
    """Solve B independent convex QCQPs on one GPU, each as solvers.cp(F, G, h, dims, A, b) does with the quadratic F
    f_i(x) = x'P_i x / 2 + q_i'x + r_i, Df_i = (P_i x + q_i)', H = sum_i z_i P_i:
        minimize f_0(x) s.t. f_i(x) <= 0 (i = 1..mnl), G x <= h, A x = b.
    P (B, mnl + 1, n, n), only each P_i's lower triangle read (P_0 = 0 is a linear objective; every P_i positive
    semidefinite is the caller's promise), q (B, mnl + 1, n), r (B, mnl + 1); mnl = 0 is allowed.  G (B, ml, n),
    h (B, ml), A (B, p, n), b (B, p) and x0 (B, n, default 0; dom f is R^n) are optional; dims, if given, is
    {'l': ml}.  F is evaluated on the device by the library: nothing calls back to Python.  Returns cp_batch's dict:
    x, snl, sl, znl, zl, y, status ('optimal' or 'unknown'), iterations, primal objective and dual objective, with the
    batch's stats (solve_ms, lock-step iterations, line-search rounds, nsub, solve_wall_ms).  nsub is qp_batch's.
    options: maxiters, abstol, reltol, feastol, refinement (as cp's)."""
    P, q, r, x0, G, h, A, b = _qcqp_args(P, q, r, G, h, dims, A, b, x0)
    B, mnl, n, p = P.shape[0], P.shape[1] - 1, P.shape[2], A.shape[1]
    out = _run_group(QCQPBatchGroup(B, n, mnl, G.shape[1], p, device, nsub),
                     (P, q, r, x0, G, h, A if p else None, b if p else None), options)
    for key in ("s", "z"):
        v = out.pop(key)
        out[key + "nl"], out[key + "l"] = v[:, :mnl], v[:, mnl:]
    return out


class CPLBatch(CPBatch):
    """B cpl problems (cvxb_batch_create_cpl): B x solvers.cpl(c, F, G, h, dims, A, b) with 'l' and 'q' cones, the CP
    batch's lock-step cpl without the epigraph row.  mnl, dims and p are shared by the batch.  load() takes c (B, n),
    x0 (B, n), G (B, cdim, n), h (B, cdim) and, with p > 0, A (B, p, n), b (B, p); set_F() takes cpl_batch's F.
    results()' s and z are [snl; sl] and [znl; zl], the 'q' rows in sl and zl; its primal objective is c'x."""

    _epi = 0

    def __init__(self, nprob, n, mnl, dims, p=0, device=0, index=None):
        self._dims = (_sdp_dims if self._sdp else _batch_dims)(dims or {"l": 0})   # (ctypes dims, keep-alive, cdim)
        super().__init__(nprob, n, mnl, self._dims[2], p, device, index)      # ml: the rows of G and h

    def _create(self):
        create = self._lib.cvxb_batch_create_sdp_cpl if self._sdp else self._lib.cvxb_batch_create_cpl
        return create(C.byref(self._h), self.B, self.n, self.mnl, C.byref(self._dims[0]), self.p, self.device)

    def load(self, c, x0, G, h, A=None, b=None):
        B, n, cd = self.B, self.n, self.ml
        c = np.ascontiguousarray(np.asarray(c, dtype=np.float64))
        x0 = np.ascontiguousarray(np.asarray(x0, dtype=np.float64))
        G = np.zeros((B, 0, n)) if G is None else np.asarray(G, dtype=np.float64)
        h = np.zeros((B, 0)) if h is None else np.ascontiguousarray(np.asarray(h, dtype=np.float64))
        if c.shape != (B, n) or x0.shape != (B, n) or G.shape != (B, cd, n) or h.shape != (B, cd):
            raise TypeError("problem shapes do not match the batch")
        Acm, bv = self._host_eq(A, b)
        Gcm = np.ascontiguousarray(np.transpose(G, (0, 2, 1)))
        self.load_ptr(c.ctypes.data, x0.ctypes.data, Gcm.ctypes.data if cd else None, h.ctypes.data if cd else None,
                      _lib.HOST, Acm, bv)

    def load_ptr(self, c, x0, G, h, space=_lib.DEVICE, A=None, b=None):
        """cvxb_batch_load_cpl on raw addresses in `space` (device-resident callers): c, x0, G cdim x n column-major
        and h (None when cdim = 0); A p x n column-major and b"""
        _lib.check(self._lib.cvxb_batch_load_cpl(self._h, c, x0, G, h, space), "batch_load_cpl")
        self._load_eq(A, b, space)

    _cp_keys = CPL_ADJOINT_KEYS


class CPLBatchGroup(CPBatchGroup):
    """CPBatchGroup for cpl problems: interleaved CPLBatch sub-batches solved concurrently, F called with each
    sub-batch's idx"""

    _batch = CPLBatch        # the class of the sub-batches

    def __init__(self, nprob, n, mnl, dims, p=0, device=0, nsub=None):
        self._dims = dims
        cdim = (_sdp_dims if self._batch._sdp else _batch_dims)(dims or {"l": 0})[2]
        super().__init__(nprob, n, mnl, cdim, p, device, nsub)

    def _part(self):
        return lambda nprob, n, m, device, dims, p=0: self._batch(nprob, n, self._mnl, self._dims, p, device)

    def load(self, c, x0, G, h, A=None, b=None):
        self._load_sliced((c, x0, G, h), A, b)


def _cpl_args(c, F, G, h, dims, A, b, sdp=False):
    """cpl's argument checks (cvxprog.py:426-530) on the batch -> mnl, c, x0, G, h, dims, A, b with the defaults
    filled in; 's' cones raise NotImplementedError (unless sdp) and p > n the Rank ValueError, before anything is
    created.  cpl reads dims['q'] and dims['s'] (a missing key is its KeyError, :427, :472) and does not check their
    entries, which the batch needs: those are checked with coneprog's TypeErrors (coneprog.py:493-500)"""
    for key in ("q", "s"):
        if dims and key not in dims:
            raise KeyError(key)
    try:
        mnl, x0 = F()
    except Exception:
        raise ValueError("function call 'F()' failed") from None
    if type(mnl) is not int or mnl < 0:
        raise TypeError("the first output of F() must be a nonnegative integer")
    if hasattr(x0, "detach"):
        x0 = x0.detach().cpu().numpy()
    x0 = np.asarray(x0)
    if x0.ndim != 2 or x0.dtype != np.float64:
        raise TypeError("'x0' must be a 'd' matrix with one column: a float64 array of shape (B, n)")
    B, n = x0.shape
    if hasattr(c, "detach"):
        c = c.detach().cpu().numpy()
    c = np.asarray(c)
    if c.shape != (B, n) or c.dtype != np.float64:
        raise TypeError("'c' must be a 'd' matrix of size (%d,1)" % n)
    h = np.zeros((B, 0)) if h is None else np.asarray(h)
    if h.ndim != 2 or h.shape[0] != B or h.dtype.kind != "f":
        raise TypeError("'h' must be a 'd' matrix with 1 column")
    if not dims:
        dims = {"l": h.shape[1], "q": [], "s": []}
    if not isinstance(dims["l"], (int, np.integer)) or dims["l"] < 0:
        raise TypeError("'dims['l']' must be a nonnegative integer")
    if [k for k in dims["q"] if not isinstance(k, (int, np.integer)) or k < 1]:
        raise TypeError("'dims['q']' must be a list of positive integers")
    if [k for k in dims["s"] if not isinstance(k, (int, np.integer)) or k < 0]:
        raise TypeError("'dims['s']' must be a list of nonnegative integers")
    cdim = dims["l"] + sum(dims["q"]) + sum(k * k for k in dims["s"])
    if h.shape[1] != cdim:
        raise TypeError("'h' must be a 'd' matrix of size (%d,1)" % cdim)
    G = np.zeros((B, 0, n)) if G is None else np.asarray(G)
    if G.shape != (B, cdim, n) or G.dtype.kind != "f":
        raise TypeError("'G' must be a 'd' matrix with size (%d, %d)" % (cdim, n))
    A = np.zeros((B, 0, n)) if A is None else np.asarray(A)
    if A.ndim != 3 or A.shape[0] != B or A.shape[2] != n or A.dtype.kind != "f":
        raise TypeError("'A' must be a 'd' matrix with %d columns" % n)
    p = A.shape[1]
    b = np.zeros((B, 0)) if b is None else np.asarray(b)
    if b.ndim != 2 or b.shape[0] != B or b.dtype.kind != "f":
        raise TypeError("'b' must be a 'd' matrix with one column")
    if b.shape[1] != p:
        raise TypeError("'b' must have length %d" % p)
    if dims["s"] and not sdp:
        raise NotImplementedError("the cpl batch takes 'l' and 'q' cones only (dims without 's')")
    if p > n:
        raise ValueError("Rank(A) < p or Rank([H(x); A; Df(x); G]) < n")
    if mnl + cdim == 0:
        raise ValueError("cpl needs at least one constraint row (mnl + cdim = 0): its merit weight 1 / gap is undefined")
    return mnl, c, x0, G, h, dims, A, b


def cpl_batch(c, F, G=None, h=None, dims=None, A=None, b=None, device=0, nsub=None, **options):
    """Solve B independent convex problems with a linear objective on one GPU, each as solvers.cpl(c, F, G, h, dims,
    A, b) does with its default kktsolver: minimize c'x s.t. fk(x) <= 0 (k = 1..mnl), G x + s = h with s in the 'l' and
    'q' cones of dims, A x = b.  F is cp_batch's without the objective row:
      F() -> (mnl, x0): mnl shared by the batch (0 allowed), x0 (B, n) strictly inside dom f, called once;
      F(x, idx=idx) -> (f, Df): f (k, mnl), Df (k, mnl, n); a row of f with a NaN or an infinite entry means x is not
          in dom f (with mnl = 0, F is still called and dom f is everything);
      F(x, z, idx=idx) -> (f, Df, H): z (k, mnl), H (k, n, n) = sum_i z_i grad² f_i(x), only its lower triangle read
          (zero when mnl = 0).
    c (B, n), G (B, cdim, n), h (B, cdim), A (B, p, n), b (B, p); dims as cpl's, without 's' cones.  A nonlinear
    objective f0 goes in as its epigraph: add a variable t, minimise t, and make f0(x) - t the first row of f.
    Returns cpl's x, snl, sl, znl, zl, y, status, iterations, primal and dual objective, with the batch's stats
    (solve_ms, lock-step iterations, line-search rounds, nsub, solve_wall_ms).  nsub is qp_batch's.
    options: maxiters, abstol, reltol, feastol, refinement (as cpl's; refinement 1 by default)."""
    return _cpl_solve(c, F, G, h, dims, A, b, device, nsub, options, sdp=False)


class SDPCPLBatch(CPLBatch):
    """CPLBatch whose dims may hold 's' blocks of order <= 32 (cvxb_batch_create_sdp_cpl): B x solvers.cpl(c, F, G, h,
    dims, A, b).  load() takes CPLBatch's arguments, with each 's' block's rows of G and h unpacked column-major after
    the 'q' rows; only the lower triangle of an 's' block of G and h is read, and results() returns sl and zl with
    symmetric 's' blocks."""
    _sdp = True


class SDPCPLBatchGroup(CPLBatchGroup):
    """CPLBatchGroup of SDPCPLBatch parts"""
    _batch = SDPCPLBatch


def sdp_cpl_batch(c, F, G=None, h=None, dims=None, A=None, b=None, device=0, nsub=None, **options):
    """Solve B independent cpl problems with semidefinite cones on one GPU, each as solvers.cpl(c, F, G, h, dims, A, b)
    does: cpl_batch's arguments, F, options and returned dict, with dims that may hold 's' blocks (orders at most 32).
    Each 's' block's rows of G and h follow the 'q' rows, unpacked column-major as the reference's G, and only their
    lower triangles are read; the returned sl and zl have symmetric 's' blocks, as cpl returns them.  A nonlinear
    objective f0 goes in as its epigraph (a variable t, minimise t, f0(x) - t the first row of f): that is how a
    solvers.cp problem with an LMI is solved here."""
    return _cpl_solve(c, F, G, h, dims, A, b, device, nsub, options, sdp=True)


def _cpl_solve(c, F, G, h, dims, A, b, device, nsub, options, sdp):
    """cpl_batch (sdp false) and sdp_cpl_batch: the checks, the group, F, the solve and the returned dict"""
    mnl, c, x0, G, h, dims, A, b = _cpl_args(c, F, G, h, dims, A, b, sdp)
    B, n, p = x0.shape[0], x0.shape[1], A.shape[1]
    grp = (SDPCPLBatchGroup if sdp else CPLBatchGroup)(B, n, mnl, dims, p, device, nsub)
    try:
        grp.set_F(F)
    except BaseException:
        grp.close()
        raise
    out = _run_group(grp, (c, x0, G, h, A if p else None, b if p else None), options)
    for key in ("s", "z"):
        v = out.pop(key)
        out[key + "nl"], out[key + "l"] = v[:, :mnl], v[:, mnl:]
    return out


def _run_group(grp, data, options, start=None):
    """load `data` (and a start dict of load_start's keys) into the batch group, solve it timed, and return its results
    and stats; the group is closed"""
    try:
        grp.load(*data)
        if start is not None:
            grp.load_start(**start)
        import time
        t0 = time.perf_counter()
        grp.solve(**options)
        wall = (time.perf_counter() - t0) * 1e3
        out = grp.results()
        out.update(grp.stats())
        out["solve_wall_ms"] = wall
        return out
    finally:
        grp.close()


def qp_batch(P, q, G, h, A=None, b=None, device=0, nsub=None, dims=None, initvals=None, **options):
    """Solve B independent dense QPs on one GPU.  P (B,n,n), q (B,n), G (B,cdim,n), h (B,cdim); optional
    equality constraints A (B,p,n) x = b (B,p), given together.
    nsub: number of concurrently solved sub-batches (QPBatchGroup); default 4 (1 for tiny batches), and never fewer
    than ceil(B / 65535), the most problems one library batch holds.
    dims: cone dimensions shared by every problem ({'l': ml, 'q': [...]}); None is {'l': cdim}.
    initvals: coneqp's starting point {'x': (B,n), 's': (B,cdim), 'y': (B,p), 'z': (B,cdim)}, every key optional
    (x = y = 0 and s = z = e without it; {} is the e start); None is the default start.
    options: maxiters, abstol, reltol, feastol, refinement (as coneqp's)."""
    P = np.asarray(P)
    G = np.asarray(G)
    if P.ndim != 3 or G.ndim != 3:
        raise TypeError("P must have shape (B, n, n) and G (B, cdim, n)")
    _, _, cdim = _batch_dims(dims, G.shape[1])
    p = _eq_rows(A, b, P.shape[0], P.shape[1])
    start = None if initvals is None else _start_arrays(initvals, P.shape[0], P.shape[1], p, cdim)
    return _run_group(QPBatchGroup(P.shape[0], P.shape[1], cdim, device, nsub, dims, p), (P, q, G, h, A, b), options,
                      start)


# ---------------------------------------------------------------------------------------
# multi-GPU: problems are independent -> shard them across ranks, no data-path collective.
# One scatter of (P, q, G, h) from rank 0, one gather of (x, s, z, status, iters, objectives):
# point-to-point send/recv groups over the process group (NCCL over NVLink on GPUs: ncclSend/ncclRecv
# inside one group call; gloo in the CPU tests), exact shard sizes, nothing padded, and on GPUs nothing
# bounces through the host: shards land in device memory and QPBatch loads them from there.

def shard_bounds(nprob, world):
    """contiguous block partition: rank r owns [lo, hi)"""
    base, extra = divmod(nprob, world)
    bounds, lo = [], 0
    for r in range(world):
        hi = lo + base + (1 if r < extra else 0)
        bounds.append((lo, hi))
        lo = hi
    return bounds


def shard_indices(nprob, world, mode="interleaved"):
    """problem indices owned by each rank.  'interleaved': i -> rank i mod world (SURVEY.md §8e; spreads
    hard and easy problems evenly, which matters because a rank's lock-step loop runs until its slowest
    problem is done); 'contiguous': blocks (shard_bounds)."""
    if mode == "contiguous":
        return [np.arange(lo, hi) for lo, hi in shard_bounds(nprob, world)]
    return [np.arange(r, nprob, world) for r in range(world)]


def _p2p(ops):
    import torch.distributed as dist
    if ops:
        for w in dist.batch_isend_irecv(ops):
            w.wait()


def qp_batch_distributed(P, q, G, h, A=None, b=None, solver=None, group=None, sharding="interleaved", timings=None,
                         nsub=None, dims=None, **options):
    """Rank 0 passes the full batch (other ranks pass None); every rank returns its shard's results and
    rank 0 additionally gets the gathered batch, in the original problem order, under key 'all'.
    Every rank passes the same `dims` (and options); shards are (k, cdim, n).  Equality constraints A (B,p,n),
    b (B,p) travel with the other inputs and y comes back with x; a stand-in `solver` then receives A and b too.
    It takes no starting point: every shard starts cold (qp_batch's initvals is not forwarded).

    `timings` (dict, optional) receives scatter_ms / solve_ms / gather_ms of this rank, measured with
    device events on the current stream (wall clock on CPU)."""
    if "initvals" in options:
        raise TypeError("qp_batch_distributed takes no starting point (initvals)")
    import time
    import torch
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized():
        rank, world = dist.get_rank(group), dist.get_world_size(group)
        on_gpu = dist.get_backend(group) == "nccl"
    else:                                   # no process group: a one-rank "world", same code path
        rank, world, on_gpu = 0, 1, torch.cuda.is_available()
    dev = torch.device("cuda", torch.cuda.current_device()) if on_gpu else torch.device("cpu")
    f64 = torch.float64

    class _Clock:
        def __init__(self):
            self.t = {}
            self._open = None

        def start(self, name):
            if on_gpu:
                e = torch.cuda.Event(enable_timing=True); e.record()
            else:
                e = time.perf_counter()
            self._open = (name, e)

        def stop(self):
            name, e0 = self._open
            if on_gpu:
                e1 = torch.cuda.Event(enable_timing=True); e1.record(); e1.synchronize()
                self.t[name] = e0.elapsed_time(e1)
            else:
                self.t[name] = (time.perf_counter() - e0) * 1e3
    clk = _Clock()

    meta = torch.zeros(4, dtype=torch.int64, device=dev)
    full = None
    if rank == 0:
        # the batch in the layout QPBatch loads: column-major n x n / m x n / p x n per problem
        Pcm, qh, Gcm, hh, Btot, n, m = _stack(P, q, G, h)
        _batch_dims(dims, m)
        Acm, bh, p = _stack_eq(A, b, Btot, n)
        meta = torch.tensor([Btot, n, m, p], dtype=torch.int64, device=dev)
        arrays = (Pcm, qh, Gcm, hh) + ((Acm, bh) if p else ())
        full = [torch.from_numpy(a).to(dev) for a in arrays]                     # one H2D of the whole batch
    if world > 1:
        dist.broadcast(meta, 0, group=group)
    Btot, n, m, p = (int(v) for v in meta.tolist())
    owners = shard_indices(Btot, world, sharding)
    mine = owners[rank]
    k = len(mine)
    tails = [(n, n), (n,), (n, m), (m,)] + ([(n, p), (p,)] if p else [])

    # ---- setup (not data path): this rank's batch object = its device allocations ----
    local_dev = torch.cuda.current_device() if on_gpu else 0
    clk.start("setup_ms")
    bobj = QPBatchGroup(k, n, m, local_dev, nsub, dims, p) if (solver is None and k) else None
    clk.stop()

    # ---- scatter ----
    if on_gpu:
        torch.cuda.synchronize()
    clk.start("scatter_ms")
    if rank == 0:
        ops, keep = [], []
        shard = None
        for r in range(world):
            idx = torch.from_numpy(owners[r]).to(dev)
            parts = [t.index_select(0, idx) for t in full]            # contiguous copy of rank r's problems
            if r == 0:
                shard = parts
            elif len(owners[r]):
                keep.append(parts)
                ops += [dist.P2POp(dist.isend, t, r, group) for t in parts]
        _p2p(ops)
        del keep, full
    else:
        shard = [torch.empty((k,) + t, dtype=f64, device=dev) for t in tails]
        if k:
            _p2p([dist.P2POp(dist.irecv, t, 0, group) for t in shard])
    clk.stop()

    # ---- solve ----
    clk.start("solve_ms")
    if solver is not None:
        # stand-in (CPU tests): numpy in the public (B, m, n) layout
        Pn, qn, Gn, hn = (t.cpu().numpy() for t in shard[:4])
        eq = [np.transpose(shard[4].cpu().numpy(), (0, 2, 1)), shard[5].cpu().numpy()] if p else []
        res = solver(np.transpose(Pn, (0, 2, 1)), qn, np.transpose(Gn, (0, 2, 1)), hn, *eq) if k else None
        xs, ss, zs, ys = ((torch.from_numpy(np.ascontiguousarray(res[key])).to(dev) if k and d
                           else torch.zeros((k, d), dtype=f64, device=dev))
                          for key, d in (("x", n), ("s", m), ("z", m), ("y", p)))
        sc = torch.zeros((k, 4), dtype=f64, device=dev)
        if k:
            for j, key in enumerate(("status_code", "iterations", "primal objective", "dual objective")):
                sc[:, j] = torch.from_numpy(np.asarray(res[key], dtype=np.float64))
        stats = {}
    else:
        xs = torch.empty((k, n), dtype=f64, device=dev)
        ss = torch.empty((k, m), dtype=f64, device=dev)
        zs = torch.empty((k, m), dtype=f64, device=dev)
        ys = torch.empty((k, p), dtype=f64, device=dev)
        sc = torch.zeros((k, 4), dtype=f64, device=dev)
        stats = {}
        if k:
            b = bobj
            try:
                # shards are already in device memory: straight into the sub-batches, no host bounce
                keepalive = []

                def loader(r, ix, part):
                    it = torch.from_numpy(ix).to(dev)
                    sl = [t.index_select(0, it) for t in shard] if b.nsub > 1 else shard
                    keepalive.append(sl)
                    # the library copies on the sub-batch's own stream: the slices (written on torch's current
                    # stream) must be complete before it reads them
                    torch.cuda.current_stream().synchronize()
                    eq = (sl[4].data_ptr(), sl[5].data_ptr()) if p else ()
                    part.load_ptr(sl[0].data_ptr(), sl[1].data_ptr(), sl[2].data_ptr(), sl[3].data_ptr(), _lib.DEVICE,
                                  *eq)
                tw = time.perf_counter()
                b.load_ptr_sliced(loader)
                del keepalive
                clk.t["solve_load_wall_ms"] = (time.perf_counter() - tw) * 1e3
                tw = time.perf_counter()
                b.solve(**options)
                clk.t["solve_ipm_wall_ms"] = (time.perf_counter() - tw) * 1e3
                tw = time.perf_counter()
                for ix, part in zip(b.idx, b.parts):
                    kk = len(ix)
                    it = torch.from_numpy(ix).to(dev)
                    px = torch.empty((kk, n), dtype=f64, device=dev)
                    ps = torch.empty((kk, m), dtype=f64, device=dev)
                    pz = torch.empty((kk, m), dtype=f64, device=dev)
                    status = np.zeros(kk, dtype=np.int32); iters = np.zeros(kk, dtype=np.int32)
                    pobj, dobj = np.zeros(kk), np.zeros(kk)
                    lib = part._lib
                    torch.cuda.current_stream().synchronize()     # px/ps/pz may reuse blocks with work still queued
                    _lib.check(lib.cvxb_batch_results(part._h, px.data_ptr(), ps.data_ptr(), pz.data_ptr(), None, None,
                                                      None, None, _lib.DEVICE), "batch_results")
                    _lib.check(lib.cvxb_batch_results(part._h, None, None, None, status.ctypes.data, iters.ctypes.data,
                                                      pobj.ctypes.data, dobj.ctypes.data, _lib.HOST), "batch_results")
                    if p:
                        py = torch.empty((kk, p), dtype=f64, device=dev)
                        _lib.check(lib.cvxb_batch_results_y(part._h, py.data_ptr(), _lib.DEVICE), "batch_results_y")
                        ys.index_copy_(0, it, py)
                    xs.index_copy_(0, it, px); ss.index_copy_(0, it, ps); zs.index_copy_(0, it, pz)
                    sc.index_copy_(0, it, torch.from_numpy(np.stack(
                        [status.astype(np.float64), iters.astype(np.float64), pobj, dobj], axis=1)).to(dev))
                stats = b.stats()
                torch.cuda.synchronize()
                clk.t["solve_collect_wall_ms"] = (time.perf_counter() - tw) * 1e3
            except BaseException:
                b.close()
                raise
    del shard
    clk.stop()

    # ---- gather ----
    clk.start("gather_ms")
    local = [xs, ss, zs, sc] + ([ys] if p else [])
    widths = (n, m, m, 4) + ((p,) if p else ())
    gathered = None
    if rank == 0:
        outs = [torch.empty((Btot, d), dtype=f64, device=dev) for d in widths]
        ops, bufs = [], {}
        for r in range(1, world):
            kr = len(owners[r])
            if kr:
                bufs[r] = [torch.empty((kr, d), dtype=f64, device=dev) for d in widths]
                ops += [dist.P2POp(dist.irecv, t, r, group) for t in bufs[r]]
        _p2p(ops)
        bufs[0] = local
        for r, parts in bufs.items():
            idx = torch.from_numpy(owners[r]).to(dev)
            for o, t in zip(outs, parts):
                o.index_copy_(0, idx, t)
        gathered = [o.cpu().numpy() for o in outs]
    elif k:
        _p2p([dist.P2POp(dist.isend, t, 0, group) for t in local])
    clk.stop()
    if bobj is not None:
        bobj.close()          # device frees (tens of ms for GBs of buffers) stay outside the timed phases
    if timings is not None:
        timings.update(clk.t)

    scn = sc.cpu().numpy()
    res = {"x": xs.cpu().numpy(), "y": ys.cpu().numpy(), "s": ss.cpu().numpy(), "z": zs.cpu().numpy(),
           "status_code": scn[:, 0].astype(np.int32), "iterations": scn[:, 1].astype(np.int32),
           "primal objective": scn[:, 2].copy(), "dual objective": scn[:, 3].copy(), "indices": mine}
    res.update(stats)
    res["status"] = [STATUS[int(c)] for c in res["status_code"]]
    if rank == 0:
        g = gathered
        res["all"] = {"x": g[0], "y": g[4] if p else np.zeros((Btot, 0)), "s": g[1], "z": g[2],
                      "status_code": g[3][:, 0].astype(np.int64),
                      "iterations": g[3][:, 1].astype(np.int64), "primal objective": g[3][:, 2].copy(),
                      "dual objective": g[3][:, 3].copy(),
                      "status": [STATUS[int(c)] for c in g[3][:, 0]]}
    return res
