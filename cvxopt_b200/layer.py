"""The batched QP and QCQP solvers as torch autograd functions on CUDA float64 tensors (OptNet-style layers).

    x, y, z, status = qp_layer(P, q, G, h, A, b)   solves   minimize 1/2 x'P x + q'x  s.t.  G x <= h,  A x = b
    x, y, znl, zl, status = qcqp_layer(P, q, r, G, h, A, b)   solves   minimize f_0(x)  s.t.  f_i(x) <= 0 (i >= 1),
        G x <= h,  A x = b,   f_i(x) = x'P_i x / 2 + q_i'x + r_i

for B problems at once with qp_batch's and qcqp_batch's algorithms, and their backward runs the library's adjoint
(cvxb_batch_adjoint, cvxb_batch_adjoint_qcqp): one more factorisation and solve of the KKT system at the returned
iterate, then the gradients written by one kernel.  Nothing leaves the device.  The gradient of each P is the symmetric
one (the solvers read only lower triangles), so a P built as S + S' or from an expanded tensor gets the right gradient
from autograd.  A problem whose status is not optimal (status != 1) gets NaN gradients.
"""
import numpy as np
import torch
from torch.autograd.function import once_differentiable

from . import _lib
from .batch import QCQPBatchGroup, QPBatchGroup


def _typed(named):
    for name, t in named:
        if not isinstance(t, torch.Tensor):
            raise TypeError("%s must be a torch tensor" % name)
        if t.dtype != torch.float64:
            raise TypeError("%s must be float64, not %s" % (name, t.dtype))


def _constraint_rows(B, n, G, h, A, b):
    """the shapes of G (B, m, n) and h (B, m), and of A (B, p, n) and b (B, p) when given (None: no rows) -> m, p"""
    m = p = 0
    if G is not None:
        if G.dim() != 3 or G.shape[0] != B or G.shape[2] != n:
            raise TypeError("G must have shape (%d, m, %d)" % (B, n))
        m = G.shape[1]
        if tuple(h.shape) != (B, m):
            raise TypeError("h must have shape (%d, %d)" % (B, m))
    if A is not None:
        if A.dim() != 3 or A.shape[0] != B or A.shape[2] != n:
            raise TypeError("A must have shape (%d, p, %d)" % (B, n))
        p = A.shape[1]
        if tuple(b.shape) != (B, p):
            raise TypeError("b must have shape (%d, %d)" % (B, p))
    return m, p


def _dims(dims, m, layer):
    if dims is not None:
        if dims.get("q") or dims.get("s"):
            raise NotImplementedError("%s differentiates 'l' rows only: dims with 'q' or 's' cones" % layer)
        if int(dims.get("l", 0)) != m:
            raise TypeError("dims['l'] = %d does not match G's %d rows" % (int(dims.get("l", 0)), m))


def _on_device(named, P):
    for name, t in named:
        if t.device.type != "cuda":
            raise TypeError("%s must be a CUDA tensor" % name)
        if t.device != P.device:
            raise TypeError("%s is on %s, P on %s" % (name, t.device, P.device))


def _check(P, q, G, h, A, b, dims):
    """shapes, dtype and device of qp_layer's inputs, and dims: every refusal before any device work.  Returns B, n,
    m, p"""
    if (A is None) != (b is None):
        raise TypeError("'A' and 'b' must be given together")
    named = [("P", P), ("q", q), ("G", G), ("h", h)] + ([("A", A), ("b", b)] if A is not None else [])
    _typed(named)
    if P.dim() != 3 or P.shape[1] != P.shape[2]:
        raise TypeError("P must have shape (B, n, n)")
    B, n = P.shape[0], P.shape[1]
    if B < 1 or n < 1:
        raise TypeError("P must have shape (B, n, n) with B and n positive")
    if tuple(q.shape) != (B, n):
        raise TypeError("q must have shape (%d, %d)" % (B, n))
    m, p = _constraint_rows(B, n, G, h, A, b)
    _dims(dims, m, "qp_layer")
    _on_device(named, P)
    return B, n, m, p


def _check_qcqp(P, q, r, G, h, A, b, x0, dims):
    """qcqp_layer's _check.  Returns B, mnl, n, ml, p"""
    if (A is None) != (b is None):
        raise TypeError("'A' and 'b' must be given together")
    if (G is None) != (h is None):
        raise TypeError("'G' and 'h' must be given together")
    named = [("P", P), ("q", q), ("r", r)] + ([("G", G), ("h", h)] if G is not None else []) + \
        ([("A", A), ("b", b)] if A is not None else []) + ([("x0", x0)] if x0 is not None else [])
    _typed(named)
    if P.dim() != 4 or P.shape[2] != P.shape[3]:
        raise TypeError("P must have shape (B, mnl + 1, n, n)")
    B, nK, n = P.shape[0], P.shape[1], P.shape[2]
    if B < 1 or nK < 1 or n < 1:
        raise TypeError("P must have shape (B, mnl + 1, n, n) with B, mnl + 1 and n positive")
    if tuple(q.shape) != (B, nK, n):
        raise TypeError("q must have shape (%d, %d, %d)" % (B, nK, n))
    if tuple(r.shape) != (B, nK):
        raise TypeError("r must have shape (%d, %d)" % (B, nK))
    if x0 is not None and tuple(x0.shape) != (B, n):
        raise TypeError("x0 must have shape (%d, %d)" % (B, n))
    ml, p = _constraint_rows(B, n, G, h, A, b)
    _dims(dims, ml, "qcqp_layer")
    _on_device(named, P)
    return B, nK - 1, n, ml, p


def _rows(t, it):
    """t's rows `it` (None: all of t) as a contiguous tensor"""
    return (t if it is None else t.index_select(0, it)).contiguous()


def _solve(grp, data, load, options, dev, widths):
    """each part of grp loads its rows of `data` (name -> tensor in the library's layout) through load(part,
    addresses), the group solves, and the results come back in problem order.  widths: n, m, p.  Returns the parts'
    row indices on the device (None: all rows), x, s, z, y and the status codes"""
    B = grp.B
    n, m, p = widths
    its = [None if grp.nsub == 1 else torch.from_numpy(ix).to(dev) for ix in grp.idx]
    keep = []

    def loader(r, ix, part):
        sl = {k: _rows(t, its[r]) for k, t in data.items()}
        keep.append(sl)
        # the library reads on its own stream: torch's writes of the slices must be complete
        torch.cuda.current_stream(dev).synchronize()
        load(part, {k: t.data_ptr() for k, t in sl.items()})
    grp.load_ptr_sliced(loader)
    del keep
    grp.solve(**options)
    f64 = dict(dtype=torch.float64, device=dev)
    x, s, z, y = (torch.empty((B, k), **f64) for k in (n, m, m, p))
    status = np.zeros(B, dtype=np.int32)
    for it, ix, part in zip(its, grp.idx, grp.parts):
        k = len(ix)
        px, ps, pz, py = (torch.empty((k, w), **f64) for w in (n, m, m, p))
        st = np.zeros(k, dtype=np.int32)
        torch.cuda.current_stream(dev).synchronize()      # the new blocks may have torch work queued
        _lib.check(part._lib.cvxb_batch_results(part._h, px.data_ptr(), ps.data_ptr(), pz.data_ptr(), None,
                                                None, None, None, _lib.DEVICE), "batch_results")
        _lib.check(part._lib.cvxb_batch_results(part._h, None, None, None, st.ctypes.data, None, None, None,
                                                _lib.HOST), "batch_results")
        if p:
            _lib.check(part._lib.cvxb_batch_results_y(part._h, py.data_ptr(), _lib.DEVICE), "batch_results_y")
        status[ix] = st
        for full, pt in ((x, px), (s, ps), (z, pz), (y, py)):
            if it is None:
                full.copy_(pt)
            else:
                full.index_copy_(0, it, pt)
    return its, x, s, z, y, torch.from_numpy(status).to(dev)


def _keep(ctx, grp, its, needs):
    """the solved group stays on the device for backward when some input needs a gradient"""
    if any(needs):
        ctx.grp, ctx.its = grp, its
    else:
        grp.close()
    ctx.set_materialize_grads(False)


def _adjoint(ctx, grads, shapes, call, dev):
    """the adjoint of every part of the kept group with its rows of grads (gx, gy, gz; None: zero), into the outputs
    `shapes` (key -> per-problem shape) in problem order: call(part, gradient addresses, key -> output address).
    Frees the group"""
    grp, its = ctx.grp, ctx.its
    f64 = dict(dtype=torch.float64, device=dev)
    out = {k: torch.empty((grp.B,) + s, **f64) for k, s in shapes.items()}
    try:
        for it, part in zip(its, grp.parts):
            g = [None if t is None else _rows(t, it) for t in grads]
            o = out if it is None else {k: torch.empty((part.B,) + s, **f64) for k, s in shapes.items()}
            torch.cuda.current_stream(dev).synchronize()      # the slices are written, the new blocks free
            call(part, [None if t is None else t.data_ptr() for t in g], {k: t.data_ptr() for k, t in o.items()})
            if it is not None:
                for k, t in o.items():
                    out[k].index_copy_(0, it, t)
    finally:
        grp.close()
    return out


class _QPLayer(torch.autograd.Function):
    @staticmethod
    def forward(ctx, P, q, G, h, A, b, nsub, options):
        B, n, m, p = ctx.shapes = _check(P, q, G, h, A, b, options.pop("dims", None))
        dev = P.device
        # the layouts the library loads: P, G and A column-major per problem
        data = {"P": P.transpose(1, 2).contiguous(), "q": q.contiguous(), "G": G.transpose(1, 2).contiguous(),
                "h": h.contiguous()}
        if p:
            data.update(A=A.transpose(1, 2).contiguous(), b=b.contiguous())
        grp = QPBatchGroup(B, n, m, dev.index if dev.index is not None else torch.cuda.current_device(), nsub,
                           p=p)
        try:
            its, x, _, z, y, status = _solve(
                grp, data, lambda part, a: part.load_ptr(a["P"], a["q"], a["G"], a["h"], _lib.DEVICE,
                                                         a.get("A"), a.get("b")),
                options, dev, (n, m, p))
        except BaseException:
            grp.close()
            raise
        _keep(ctx, grp, its, ctx.needs_input_grad[:6])
        return x, y, z, status

    @staticmethod
    @once_differentiable
    def backward(ctx, gx, gy, gz, _gstatus):
        B, n, m, p = ctx.shapes
        need = dict(zip(("P", "q", "G", "h", "A", "b"), ctx.needs_input_grad[:6]))
        dev = gx.device if gx is not None else gz.device if gz is not None else gy.device
        # C's outputs ux, uy, uz, dP, dG, dA in problem order; the matrices column-major per problem
        shapes = {"q": (n,), "b": (p,), "h": (m,), "P": (n, n), "G": (n, m), "A": (n, p)}
        shapes = {k: s for k, s in shapes.items() if need[k] and (p or k not in ("b", "A"))}
        out = _adjoint(ctx, (gx, gy if p else None, gz if m else None), shapes,
                       lambda part, g, o: part.adjoint_ptr(*g, *(o.get(k) for k in ("q", "b", "h", "P", "G", "A")),
                                                           space=_lib.DEVICE), dev)
        f64 = dict(dtype=torch.float64, device=dev)
        grads = {"q": lambda t: -t, "b": lambda t: t, "h": lambda t: t}
        res = []
        for key in ("P", "q", "G", "h", "A", "b"):
            if key not in out:
                res.append(torch.zeros((B, 0) if key == "b" else (B, 0, n), **f64) if need[key] else None)
            elif key in grads:
                res.append(grads[key](out[key]))
            else:
                res.append(out[key].transpose(1, 2))
        return (*res, None, None)


class _QCQPLayer(torch.autograd.Function):
    @staticmethod
    def forward(ctx, P, q, r, G, h, A, b, x0, nsub, options):
        B, mnl, n, ml, p = ctx.shapes = _check_qcqp(P, q, r, G, h, A, b, x0, options.pop("dims", None))
        dev = P.device
        # the layouts the library loads: per problem P's (mnl + 1) n x n column-major stack, G and A column-major
        data = {"P": P.permute(0, 3, 1, 2).contiguous(), "q": q.contiguous(), "r": r.contiguous()}
        if x0 is not None:
            data["x0"] = x0.contiguous()
        if ml:
            data.update(G=G.transpose(1, 2).contiguous(), h=h.contiguous())
        if p:
            data.update(A=A.transpose(1, 2).contiguous(), b=b.contiguous())
        grp = QCQPBatchGroup(B, n, mnl, ml, p, dev.index if dev.index is not None else torch.cuda.current_device(),
                             nsub)
        try:
            its, x, _, z, y, status = _solve(
                grp, data, lambda part, a: part.load_ptr(a["P"], a["q"], a["r"], a.get("x0"), a.get("G"), a.get("h"),
                                                         _lib.DEVICE, a.get("A"), a.get("b")),
                options, dev, (n, mnl + ml, p))
        except BaseException:
            grp.close()
            raise
        _keep(ctx, grp, its, ctx.needs_input_grad[:7])
        return x, y, z[:, :mnl].clone(), z[:, mnl:].clone(), status

    @staticmethod
    @once_differentiable
    def backward(ctx, gx, gy, gznl, gzl, _gstatus):
        B, mnl, n, ml, p = ctx.shapes
        nK, m = mnl + 1, mnl + ml
        need = dict(zip(("P", "q", "r", "G", "h", "A", "b"), ctx.needs_input_grad[:7]))
        dev = next(t.device for t in (gx, gy, gznl, gzl) if t is not None)
        f64 = dict(dtype=torch.float64, device=dev)
        gz = None
        if m and (gznl is not None or gzl is not None):
            gz = torch.cat([torch.zeros((B, k), **f64) if t is None else t for t, k in ((gznl, mnl), (gzl, ml))], 1)
        # C's outputs uy, uz (h: its 'l' rows), dP, dq, dr, dG, dA in problem order; dP, dG, dA column-major
        shapes = {"b": (p,), "h": (m,), "P": (n, nK, n), "q": (nK, n), "r": (nK,), "G": (n, ml), "A": (n, p)}
        shapes = {k: s for k, s in shapes.items() if need[k] and (ml or k not in ("G", "h")) and
                  (p or k not in ("A", "b"))}
        out = _adjoint(ctx, (gx, gy if p else None, gz), shapes,
                       lambda part, g, o: part.adjoint_ptr(*g, None, *(o.get(k) for k in
                                                                       ("b", "h", "P", "q", "r", "G", "A")),
                                                           space=_lib.DEVICE), dev)
        view = {"P": lambda t: t.permute(0, 2, 3, 1), "h": lambda t: t[:, mnl:], "G": lambda t: t.transpose(1, 2),
                "A": lambda t: t.transpose(1, 2)}
        empty = {"G": (B, 0, n), "h": (B, 0), "A": (B, 0, n), "b": (B, 0)}
        res = []
        for key in ("P", "q", "r", "G", "h", "A", "b"):
            if key in out:
                res.append(view.get(key, lambda t: t)(out[key]))
            else:
                res.append(torch.zeros(empty[key], **f64) if need[key] else None)
        return (*res, None, None, None)


def qp_layer(P, q, G, h, A=None, b=None, nsub=None, **options):
    """Solve B dense QPs  minimize 1/2 x'P x + q'x  s.t.  G x <= h,  A x = b  on the GPU, differentiably.

    P (B, n, n), q (B, n), G (B, m, n), h (B, m), A (B, p, n) and b (B, p): CUDA float64 tensors on one device; A and
    b are optional and given together.  Returns (x, y, z, status_code): x (B, n), the multipliers y (B, p) of A x = b
    and z (B, m) of G x <= h, and the int32 status per problem (1 optimal, 2 maximum iterations, 3 singular).
    nsub: sub-batches solved concurrently, as qp_batch's.  options: maxiters, abstol, reltol, feastol, refinement, and
    dims ({'l': m} only: 'q' and 's' cones raise NotImplementedError).  Shape, dtype and device errors are TypeErrors
    raised before any device work.

    Backward (once: no double backward) returns dL/dP (symmetric), dL/dq, dL/dG, dL/dh, dL/dA and dL/db from the
    gradients of x, y and z, with NaN for problems whose status is not 1.  Inputs that need no gradient get none and
    cost nothing.  The solved batch is kept on the device from forward to backward, and freed by backward."""
    return _QPLayer.apply(P, q, G, h, A, b, nsub, dict(options))


def qcqp_layer(P, q, r, G=None, h=None, A=None, b=None, x0=None, nsub=None, **options):
    """Solve B convex QCQPs  minimize f_0(x)  s.t.  f_i(x) <= 0 (i = 1..mnl),  G x <= h,  A x = b,  with
    f_i(x) = x'P_i x / 2 + q_i'x + r_i,  on the GPU, differentiably (qcqp_batch's algorithm: solvers.cp's).

    P (B, mnl + 1, n, n), only each P_i's lower triangle read, q (B, mnl + 1, n), r (B, mnl + 1), G (B, ml, n),
    h (B, ml), A (B, p, n), b (B, p) and the start x0 (B, n, default 0): CUDA float64 tensors on one device; G and h,
    A and b are optional and given in pairs.  Returns (x, y, znl, zl, status_code): x (B, n), the multipliers y (B, p)
    of A x = b, znl (B, mnl) of f_i(x) <= 0 and zl (B, ml) of G x <= h, and the int32 status per problem (1 optimal).
    nsub: sub-batches solved concurrently, as qp_batch's.  options: maxiters, abstol, reltol, feastol, refinement, and
    dims ({'l': ml} only: 'q' and 's' cones raise NotImplementedError).  Shape, dtype and device errors are TypeErrors
    raised before any device work.

    Backward (once: no double backward) returns dL/dP (each block symmetric), dL/dq, dL/dr, dL/dG, dL/dh, dL/dA and
    dL/db from the gradients of x, y, znl and zl, with NaN for problems whose status is not 1; x0 gets none.  Inputs
    that need no gradient get none and cost nothing.  The solved batch is kept on the device from forward to backward,
    and freed by backward."""
    return _QCQPLayer.apply(P, q, r, G, h, A, b, x0, nsub, dict(options))
