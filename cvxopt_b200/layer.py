"""qp_layer: the batched QP solver as a torch autograd function on CUDA float64 tensors (an OptNet-style layer).

    x, y, z, status = qp_layer(P, q, G, h, A, b)   solves   minimize 1/2 x'P x + q'x  s.t.  G x <= h,  A x = b

for B problems at once with qp_batch's algorithm, and its backward runs the library's adjoint (cvxb_batch_adjoint):
one more factorisation and solve of the KKT system at the returned iterate, then the rank-2 gradients of P, G and A
written by one kernel.  Nothing leaves the device.  The gradient of P is the symmetric one (the solver reads only
its lower triangle), so P built as S + S' or from an expanded tensor gets the right gradient from autograd.  A
problem whose status is not optimal (status != 1) gets NaN gradients.
"""
import numpy as np
import torch
from torch.autograd.function import once_differentiable

from . import _lib
from .batch import QPBatchGroup


def _check(P, q, G, h, A, b, dims):
    """shapes, dtype and device of the inputs, and dims: every refusal before any device work.  Returns B, n, m, p"""
    if (A is None) != (b is None):
        raise TypeError("'A' and 'b' must be given together")
    named = [("P", P), ("q", q), ("G", G), ("h", h)] + ([("A", A), ("b", b)] if A is not None else [])
    for name, t in named:
        if not isinstance(t, torch.Tensor):
            raise TypeError("%s must be a torch tensor" % name)
        if t.dtype != torch.float64:
            raise TypeError("%s must be float64, not %s" % (name, t.dtype))
    if P.dim() != 3 or P.shape[1] != P.shape[2]:
        raise TypeError("P must have shape (B, n, n)")
    B, n = P.shape[0], P.shape[1]
    if B < 1 or n < 1:
        raise TypeError("P must have shape (B, n, n) with B and n positive")
    if tuple(q.shape) != (B, n):
        raise TypeError("q must have shape (%d, %d)" % (B, n))
    if G.dim() != 3 or G.shape[0] != B or G.shape[2] != n:
        raise TypeError("G must have shape (%d, m, %d)" % (B, n))
    m = G.shape[1]
    if tuple(h.shape) != (B, m):
        raise TypeError("h must have shape (%d, %d)" % (B, m))
    p = 0
    if A is not None:
        if A.dim() != 3 or A.shape[0] != B or A.shape[2] != n:
            raise TypeError("A must have shape (%d, p, %d)" % (B, n))
        p = A.shape[1]
        if tuple(b.shape) != (B, p):
            raise TypeError("b must have shape (%d, %d)" % (B, p))
    if dims is not None:
        if dims.get("q") or dims.get("s"):
            raise NotImplementedError("qp_layer differentiates 'l' rows only: dims with 'q' or 's' cones")
        if int(dims.get("l", 0)) != m:
            raise TypeError("dims['l'] = %d does not match G's %d rows" % (int(dims.get("l", 0)), m))
    for name, t in named:
        if t.device.type != "cuda":
            raise TypeError("%s must be a CUDA tensor" % name)
        if t.device != P.device:
            raise TypeError("%s is on %s, P on %s" % (name, t.device, P.device))
    return B, n, m, p


def _rows(t, it):
    """t's rows `it` (None: all of t) as a contiguous tensor"""
    return (t if it is None else t.index_select(0, it)).contiguous()


class _QPLayer(torch.autograd.Function):
    @staticmethod
    def forward(ctx, P, q, G, h, A, b, nsub, options):
        B, n, m, p = ctx.shapes = _check(P, q, G, h, A, b, options.pop("dims", None))
        dev = P.device
        # the layouts the library loads: P, G and A column-major per problem
        data = [P.transpose(1, 2).contiguous(), q.contiguous(), G.transpose(1, 2).contiguous(), h.contiguous()]
        if p:
            data += [A.transpose(1, 2).contiguous(), b.contiguous()]
        grp = QPBatchGroup(B, n, m, dev.index if dev.index is not None else torch.cuda.current_device(), nsub,
                           p=p)
        try:
            its = [None if grp.nsub == 1 else torch.from_numpy(ix).to(dev) for ix in grp.idx]
            keep = []

            def loader(r, ix, part):
                sl = [_rows(t, its[r]) for t in data]
                keep.append(sl)
                # the library reads on its own stream: torch's writes of the slices must be complete
                torch.cuda.current_stream(dev).synchronize()
                part.load_ptr(*(t.data_ptr() for t in sl[:4]), _lib.DEVICE,
                              *((sl[4].data_ptr(), sl[5].data_ptr()) if p else ()))
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
        except BaseException:
            grp.close()
            raise
        if any(ctx.needs_input_grad[:6]):
            ctx.grp, ctx.its = grp, its
        else:
            grp.close()
        ctx.set_materialize_grads(False)
        return x, y, z, torch.from_numpy(status).to(dev)

    @staticmethod
    @once_differentiable
    def backward(ctx, gx, gy, gz, _gstatus):
        B, n, m, p = ctx.shapes
        grp, its = ctx.grp, ctx.its
        need = dict(zip(("P", "q", "G", "h", "A", "b"), ctx.needs_input_grad[:6]))
        dev = gx.device if gx is not None else gz.device if gz is not None else gy.device
        f64 = dict(dtype=torch.float64, device=dev)
        # C's outputs ux, uy, uz, dP, dG, dA in problem order; the matrices column-major per problem
        shapes = {"q": (n,), "b": (p,), "h": (m,), "P": (n, n), "G": (n, m), "A": (n, p)}
        keys = [k for k in ("q", "b", "h", "P", "G", "A") if need[k] and (p or k not in ("b", "A"))]
        out = {k: torch.empty((B,) + shapes[k], **f64) for k in keys}
        try:
            for it, part in zip(its, grp.parts):
                k = part.B
                g = [None if t is None else _rows(t, it) for t in (gx, gy if p else None, gz if m else None)]
                o = out if it is None else {key: torch.empty((k,) + shapes[key], **f64) for key in keys}
                torch.cuda.current_stream(dev).synchronize()      # the slices are written, the new blocks free
                part.adjoint_ptr(*(None if t is None else t.data_ptr() for t in g),
                                 *(o[key].data_ptr() if key in o else None for key in ("q", "b", "h", "P", "G", "A")),
                                 space=_lib.DEVICE)
                if it is not None:
                    for key, t in o.items():
                        out[key].index_copy_(0, it, t)
        finally:
            grp.close()
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
