"""The batched QP and QCQP solvers as torch autograd functions on CUDA float64 tensors (OptNet-style layers).

    x, y, z, status = qp_layer(P, q, G, h, A, b)   solves   minimize 1/2 x'P x + q'x  s.t.  G x <= h,  A x = b
    x, y, znl, zl, status = qcqp_layer(P, q, r, G, h, A, b)   solves   minimize f_0(x)  s.t.  f_i(x) <= 0 (i >= 1),
        G x <= h,  A x = b,   f_i(x) = x'P_i x / 2 + q_i'x + r_i
    x, y, z, status = coneqp_layer(P, q, G, h, dims, A, b)   solves   minimize 1/2 x'P x + q'x  s.t.  G x + s = h,
        s in the cone of dims ('l', 'q', 's'),  A x = b;   conelp_layer(c, G, h, dims, A, b) the same with P = 0
    x, y, znl, zl, status = gp_layer(K, F, g, G, h, A, b)   solves   minimize lse(F_0 x + g_0)  s.t.
        lse(F_i x + g_i) <= 0 (i >= 1),  G x <= h,  A x = b   (a geometric program in log form)
    x, y, znl, zl, status = cp_layer(F, params, G, h, A, b)   solves   minimize f_0(x)  s.t.  f_i(x) <= 0 (i >= 1),
        G x <= h,  A x = b  with the caller's F(x; params);   cpl_layer(c, F, params, G, h, dims, A, b) minimises c'x
        with 'l', 'q' and 's' cones

for B problems at once with qp_batch's, qcqp_batch's, gp_batch's, cp_batch's and cpl_batch's algorithms, and their
backward runs the library's adjoint (cvxb_batch_adjoint, _qcqp, _cone, _gp, _cp): one more factorisation and solve of
the KKT system at the returned iterate, then the gradients written by one kernel.  Nothing leaves the device.  The
gradient of each P is the symmetric one (the solvers read only lower triangles), so a P built as S + S' or from an
expanded tensor gets the right gradient from autograd.  A problem whose status is not optimal (status != 1) gets NaN
gradients.

Every layer also has forward mode: under torch.autograd.forward_ad, dual inputs give dual x, y and z (znl and zl),
from the library's tangent (cvxb_batch_tangent, _qcqp, _gp, _cp), the same factorisation and solves as backward
with a right-hand side formed on the device from the input tangents.  A non-symmetric tangent of P enters through
its symmetric part.  In cp_layer and cpl_layer the params' tangents enter through one more call of F.  status carries
no tangent.
"""
import numpy as np
import torch
from torch.autograd.function import once_differentiable

from . import _lib
from .batch import (_FROM_U, _TAIL, BATCH_SMAX, ConeLPBatchGroup, CPBatch, CPBatchGroup, CPLBatchGroup, GPBatch,
                    GPBatchGroup, QCQPBatch, QCQPBatchGroup, QPBatch, QPBatchGroup, SDPBatchGroup, SDPCPLBatchGroup,
                    SDPQPBatchGroup, _inverse, _lib_shape)


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


def _on_device(named):
    """every tensor of `named` on one CUDA device, the first one's"""
    first, ref = named[0]
    for name, t in named:
        if t.device.type != "cuda":
            raise TypeError("%s must be a CUDA tensor" % name)
        if t.device != ref.device:
            raise TypeError("%s is on %s, %s on %s" % (name, t.device, first, ref.device))


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
    _on_device(named)
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
    _on_device(named)
    return B, nK - 1, n, ml, p


def _check_cone(P, q, G, h, dims, A, b):
    """coneqp_layer's and conelp_layer's _check (P None: a cone LP, q its c): every refusal before any device work.
    dims must count G's rows: 'l' + sum 'q' + sum of each 's' order squared.  Returns B, n, m, p"""
    if (A is None) != (b is None):
        raise TypeError("'A' and 'b' must be given together")
    qn = "c" if P is None else "q"
    named = ([] if P is None else [("P", P)]) + [(qn, q), ("G", G), ("h", h)] + \
        ([("A", A), ("b", b)] if A is not None else [])
    _typed(named)
    if q.dim() != 2 or q.shape[0] < 1 or q.shape[1] < 1:
        raise TypeError("%s must have shape (B, n) with B and n positive" % qn)
    B, n = q.shape
    if P is not None and tuple(P.shape) != (B, n, n):
        raise TypeError("P must have shape (%d, %d, %d)" % (B, n, n))
    m, p = _constraint_rows(B, n, G, h, A, b)
    _cone_dims(dims, m)
    _on_device(named)
    return B, n, m, p


def _cone_dims(dims, m):
    """the cone layers' and cpl_layer's dims, checked against the m rows of G and h -> dims with int entries"""
    if not isinstance(dims, dict) or not set(dims) <= {"l", "q", "s"}:
        raise TypeError("dims must be a dictionary with keys 'l', 'q' and 's'")
    if int(dims.get("l", 0)) < 0 or any(int(k) < 1 for k in dims.get("q", [])) or \
            any(not 0 <= int(k) <= BATCH_SMAX for k in dims.get("s", [])):
        raise TypeError("dims: 'l' must be nonnegative, each 'q' size at least 1, each 's' order in 0..%d" % BATCH_SMAX)
    dims = {"l": int(dims.get("l", 0)), "q": [int(k) for k in dims.get("q", [])],
            "s": [int(k) for k in dims.get("s", [])]}
    cdim = dims["l"] + sum(dims["q"]) + sum(k * k for k in dims["s"])
    if cdim != m:
        raise TypeError("dims has %d rows ('l' + sum 'q' + sum 's'²), G and h have %d" % (cdim, m))
    return dims


def _check_gp(K, F, g, G, h, A, b):
    """gp_layer's _check, K with gp_batch's message: every refusal before any device work.  Returns B, n, ml, p"""
    if type(K) is not list or not K or [k for k in K if type(k) is not int or k <= 0]:
        raise TypeError("'K' must be a list of positive integers")
    if (A is None) != (b is None):
        raise TypeError("'A' and 'b' must be given together")
    if (G is None) != (h is None):
        raise TypeError("'G' and 'h' must be given together")
    named = [("F", F), ("g", g)] + ([("G", G), ("h", h)] if G is not None else []) + \
        ([("A", A), ("b", b)] if A is not None else [])
    _typed(named)
    S = sum(K)
    if F.dim() != 3 or F.shape[1] != S or F.shape[0] < 1 or F.shape[2] < 1:
        raise TypeError("F must have shape (B, %d, n) with B and n positive (sum K = %d rows)" % (S, S))
    B, n = F.shape[0], F.shape[2]
    if tuple(g.shape) != (B, S):
        raise TypeError("g must have shape (%d, %d)" % (B, S))
    ml, p = _constraint_rows(B, n, G, h, A, b)
    _on_device(named)
    return B, n, ml, p


def _rows(t, it):
    """t's rows `it` (None: all of t) as a contiguous tensor"""
    return (t if it is None else t.index_select(0, it)).contiguous()


def _device(t):
    """the index of t's CUDA device"""
    return t.device.index if t.device.index is not None else torch.cuda.current_device()


def _layout(ts, block):
    """tensors ts in load()'s shapes, one per entry of block + _TAIL (block: a batch class's own block), as views in the
    library's layouts.  An absent or empty one (ml = 0, p = 0) is None: the library takes it as NULL"""
    return [None if t is None or not t.numel() else t if axes is None else t.permute(axes)
            for t, (_, _, axes, _) in zip(ts, block + _TAIL)]


def _solve(grp, data, load, options, dev, widths):
    """each part of grp loads its rows of `data` (tensors in the library's layouts, None: NULL) through load(part,
    *addresses), the group solves, and the results come back in problem order.  widths: n, m, p.  Returns the parts'
    row indices on the device (None: all rows), x, s, z, y and the status codes"""
    B = grp.B
    n, m, p = widths
    its = [None if grp.nsub == 1 else torch.from_numpy(ix).to(dev) for ix in grp.idx]
    keep = []

    def loader(r, ix, part):
        sl = [None if t is None else _rows(t, its[r]) for t in data]
        keep.append(sl)
        # the library reads on its own stream: torch's writes of the slices must be complete
        torch.cuda.current_stream(dev).synchronize()
        load(part, *(None if t is None else t.data_ptr() for t in sl))
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


def _keep(ctx, grp, its, needs, fw=False):
    """the solved group stays on the device for backward when some input needs a gradient, and for jvp when some
    input carries a forward-mode tangent (fw)"""
    if any(needs) or fw:
        ctx.grp, ctx.its = grp, its
    else:
        grp.close()
    ctx.set_materialize_grads(False)


def _forward(ctx, grp, data, load, options, needs, fw, F=None):
    """a layer's forward: the new group grp (F: its set_F, for cp and cpl) solves `data`, _layout's views made
    contiguous, each part loaded by load(part, *addresses), and stays on the device for backward (needs: the inputs'
    needs_input_grad) and jvp (fw); an error closes it.  ctx.shapes is (B, n, mnl, ml, p).  Returns x, y, z and the
    status codes"""
    B, n, mnl, ml, p = ctx.shapes
    try:
        if F is not None:
            grp.set_F(F)
        its, x, _, z, y, status = _solve(grp, [None if t is None else t.contiguous() for t in data], load, options,
                                         ctx.dev, (n, mnl + ml, p))
    except BaseException:
        grp.close()
        raise
    _keep(ctx, grp, its, needs, fw)
    return x, y, z, status


def _split(z, mnl):
    """z = [znl; zl] (or its tangent) as znl and zl, each a tensor of its own"""
    return z[:, :mnl].clone(), z[:, mnl:].clone()


def _has_tangent(*ts):
    """whether a tensor of ts carries a forward-mode tangent (torch.autograd.forward_ad)"""
    return any(isinstance(t, torch.Tensor) and torch.autograd.forward_ad.unpack_dual(t).tangent is not None
               for t in ts)


def _tangent(ctx, dirs, method, needs):
    """the tangent of every part of the kept group along its rows of dirs (tensors in the library's layouts, None:
    zero) by part.method (a tangent *_ptr), into dx, dy, dz in problem order.  Frees the group unless backward will
    need it (some input needs a gradient)"""
    B, n, mnl, ml, p = ctx.shapes
    grp, its = ctx.grp, ctx.its
    f64 = dict(dtype=torch.float64, device=ctx.dev)
    widths = (n, p, mnl + ml)
    out = [torch.empty((B, w), **f64) for w in widths]
    try:
        for it, part in zip(its, grp.parts):
            d = [None if t is None else _rows(t, it) for t in dirs]
            o = out if it is None else [torch.empty((part.B, w), **f64) for w in widths]
            torch.cuda.current_stream(ctx.dev).synchronize()      # the slices are written, the new blocks free
            getattr(part, method)(*(None if t is None else t.data_ptr() for t in d), *(t.data_ptr() for t in o),
                                  space=_lib.DEVICE)
            if it is not None:
                for full, t in zip(out, o):
                    full.index_copy_(0, it, t)
    finally:
        if not any(needs):
            grp.close()
    return out


def _adjoint(ctx, grads, shapes, method):
    """the adjoint of every part of the kept group with its rows of grads (gx, gy, gz; None: zero) by part.method (an
    adjoint *_ptr), into outputs of the per-problem `shapes` in the call's order (None: NULL) in problem order.  Frees
    the group"""
    grp, its = ctx.grp, ctx.its
    f64 = dict(dtype=torch.float64, device=ctx.dev)
    out = [None if s is None else torch.empty((grp.B,) + s, **f64) for s in shapes]
    try:
        for it, part in zip(its, grp.parts):
            g = [None if t is None else _rows(t, it) for t in grads]
            o = out if it is None else [None if s is None else torch.empty((part.B,) + s, **f64) for s in shapes]
            torch.cuda.current_stream(ctx.dev).synchronize()      # the slices are written, the new blocks free
            getattr(part, method)(*(None if t is None else t.data_ptr() for t in g + o), space=_lib.DEVICE)
            if it is not None:
                for full, t in zip(out, o):
                    if t is not None:
                        full.index_copy_(0, it, t)
    finally:
        grp.close()
    return out


def _grads(ctx, method, block, needs, gx, gy, gznl, gzl, theta=False):
    """a layer's backward: the gradients of its inputs, one per entry of block + _TAIL (needs: which need one), from
    those of x, y, znl and zl (None: zero) by the kept group's adjoint `method`, which writes ux, uy, uz and then the
    entries marked as written.  Those come as views in load()'s layouts, the others by _FROM_U; an empty input that
    needs a gradient gets zeros, one that needs none gets None.  With theta, ux and uznl follow for _theta_grads.
    Frees the group"""
    B, n, mnl, ml, p = ctx.shapes
    f64 = dict(dtype=torch.float64, device=ctx.dev)
    part = ctx.grp.parts[0]
    inputs = [(name[1:], (B,) + shape(part), axes, writes) for name, shape, axes, writes in block + _TAIL]
    want = {k for (k, s, _, _), nd in zip(inputs, needs) if nd and all(s)}
    want |= {"ux", "uznl"} if theta and mnl else {"ux"} if theta else set()
    own = [(k, s, axes) for k, s, axes, writes in inputs if writes]
    fromu = {_FROM_U[k][0] for k in want if k not in {k for k, _, _ in own}}
    shapes = [(w,) if i in fromu else None for i, w in enumerate((n, p, mnl + ml))]
    shapes += [_lib_shape(s[1:], axes) if k in want else None for k, s, axes in own]
    gz = None
    if mnl + ml and (gznl is not None or gzl is not None):
        gz = [torch.zeros((B, k), **f64) if t is None else t for t, k in ((gznl, mnl), (gzl, ml)) if k]
        gz = gz[0] if len(gz) == 1 else torch.cat(gz, 1)
    out = _adjoint(ctx, (gx, gy if p else None, gz), shapes, method)
    u, got = out[:3], dict(zip((k for k, _, _ in own), out[3:]))

    def from_u(k):
        return _FROM_U[k][1](u[_FROM_U[k][0]], mnl)
    res = []
    for (k, s, axes, writes), nd in zip(inputs, needs):
        if not nd:
            res.append(None)
        elif not all(s):
            res.append(torch.zeros(s, **f64))
        elif writes:
            res.append(got[k] if axes is None else got[k].permute(_inverse(axes)))
        else:
            res.append(from_u(k))
    if theta:
        res += [from_u("ux"), from_u("uznl") if mnl else torch.zeros((B, 0), **f64)]
    return res


def _load_qp(part, P, q, G, h, A, b):
    """a QP or cone LP part's load_ptr (a cone LP: P None)"""
    part.load_ptr(*((q, G, h) if P is None else (P, q, G, h)), _lib.DEVICE, A, b)


class _QPLayer(torch.autograd.Function):
    @staticmethod
    def forward(ctx, P, q, G, h, A, b, nsub, options):
        fw = options.pop("_fw")
        B, n, m, p = _check(P, q, G, h, A, b, options.pop("dims", None))
        ctx.shapes, ctx.dev = (B, n, 0, m, p), P.device
        data = _layout((P, q, G, h, A, b), QPBatch._block)
        grp = QPBatchGroup(B, n, m, _device(P), nsub, p=p)
        return _forward(ctx, grp, data, _load_qp, options, ctx.needs_input_grad[:6], fw)

    @staticmethod
    @once_differentiable
    def backward(ctx, gx, gy, gz, _gstatus):
        return (*_grads(ctx, "adjoint_ptr", QPBatch._block, ctx.needs_input_grad[:6], gx, gy, None, gz), None, None)

    @staticmethod
    def jvp(ctx, dP, dq, dG, dh, dA, db, _nsub, _options):
        dirs = _layout((dP, dq, dG, dh, dA, db), QPBatch._block)
        return (*_tangent(ctx, dirs, "tangent_ptr", ctx.needs_input_grad[:6]), None)


class _ConeLayer(torch.autograd.Function):
    # a cone LP: P None and q its c, in dq's place as the library takes it
    @staticmethod
    def forward(ctx, P, q, G, h, A, b, dims, nsub, options):
        fw = options.pop("_fw")
        B, n, m, p = _check_cone(P, q, G, h, dims, A, b)
        ctx.shapes, ctx.dev = (B, n, 0, m, p), q.device
        data = _layout((P, q, G, h, A, b), QPBatch._block)
        if P is not None:            # coneqp_batch's group
            grp = SDPQPBatchGroup(B, n, dims, p, _device(q), nsub)
        elif dims.get("s"):          # sdp_batch's
            grp = SDPBatchGroup(B, n, dims, p, _device(q), nsub)
        else:                        # conelp_batch's
            grp = ConeLPBatchGroup(B, n, m, _device(q), nsub, {"l": dims.get("l", 0), "q": dims.get("q", [])}, p)
        return _forward(ctx, grp, data, _load_qp, options, ctx.needs_input_grad[:6], fw)

    @staticmethod
    @once_differentiable
    def backward(ctx, gx, gy, gz, _gstatus):
        return (*_grads(ctx, "adjoint_cone_ptr", QPBatch._block, ctx.needs_input_grad[:6], gx, gy, None, gz), None,
                None, None)

    @staticmethod
    def jvp(ctx, dP, dq, dG, dh, dA, db, _dims, _nsub, _options):
        dirs = _layout((dP, dq, dG, dh, dA, db), QPBatch._block)
        return (*_tangent(ctx, dirs, "tangent_ptr", ctx.needs_input_grad[:6]), None)


class _QCQPLayer(torch.autograd.Function):
    @staticmethod
    def forward(ctx, P, q, r, G, h, A, b, x0, nsub, options):
        fw = options.pop("_fw")
        B, mnl, n, ml, p = _check_qcqp(P, q, r, G, h, A, b, x0, options.pop("dims", None))
        ctx.shapes, ctx.dev = (B, n, mnl, ml, p), P.device
        data = _layout((P, q, r, G, h, A, b), QCQPBatch._block) + [x0]
        grp = QCQPBatchGroup(B, n, mnl, ml, p, _device(P), nsub)
        x, y, z, status = _forward(
            ctx, grp, data, lambda part, P, q, r, G, h, A, b, x0: part.load_ptr(P, q, r, x0, G, h, _lib.DEVICE, A, b),
            options, ctx.needs_input_grad[:7], fw)
        return (x, y, *_split(z, mnl), status)

    @staticmethod
    @once_differentiable
    def backward(ctx, gx, gy, gznl, gzl, _gstatus):
        return (*_grads(ctx, "adjoint_ptr", QCQPBatch._block, ctx.needs_input_grad[:7], gx, gy, gznl, gzl), None,
                None, None)

    @staticmethod
    def jvp(ctx, dP, dq, dr, dG, dh, dA, db, _dx0, _nsub, _options):
        dirs = _layout((dP, dq, dr, dG, dh, dA, db), QCQPBatch._block)
        dx, dy, dz = _tangent(ctx, dirs, "tangent_ptr", ctx.needs_input_grad[:7])
        return (dx, dy, *_split(dz, ctx.shapes[2]), None)


class _GPLayer(torch.autograd.Function):
    @staticmethod
    def forward(ctx, K, F, g, G, h, A, b, nsub, options):
        fw = options.pop("_fw")
        B, n, ml, p = _check_gp(K, F, g, G, h, A, b)
        mnl = len(K) - 1
        ctx.shapes, ctx.dev = (B, n, mnl, ml, p), F.device
        data = _layout((F, g, G, h, A, b), GPBatch._block)
        grp = GPBatchGroup(B, n, K, ml, p, _device(F), nsub)
        x, y, z, status = _forward(
            ctx, grp, data, lambda part, F, g, G, h, A, b: part.load_ptr(F, g, G, h, _lib.DEVICE, A, b), options,
            ctx.needs_input_grad[1:7], fw)
        return (x, y, *_split(z, mnl), status)

    @staticmethod
    @once_differentiable
    def backward(ctx, gx, gy, gznl, gzl, _gstatus):
        return (None, *_grads(ctx, "adjoint_gp_ptr", GPBatch._block, ctx.needs_input_grad[1:7], gx, gy, gznl, gzl),
                None, None)

    @staticmethod
    def jvp(ctx, _dK, dF, dg, dG, dh, dA, db, _nsub, _options):
        dirs = _layout((dF, dg, dG, dh, dA, db), GPBatch._block)
        dx, dy, dz = _tangent(ctx, dirs, "tangent_gp_ptr", ctx.needs_input_grad[1:7])
        return (dx, dy, *_split(dz, ctx.shapes[2]), None)


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
    return _QPLayer.apply(P, q, G, h, A, b, nsub, dict(options, _fw=_has_tangent(P, q, G, h, A, b)))


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
    return _QCQPLayer.apply(P, q, r, G, h, A, b, x0, nsub,
                            dict(options, _fw=_has_tangent(P, q, r, G, h, A, b)))


def coneqp_layer(P, q, G, h, dims, A=None, b=None, nsub=None, **options):
    """Solve B cone QPs  minimize 1/2 x'P x + q'x  s.t.  G x + s = h,  s in C,  A x = b  on the GPU, differentiably
    (coneqp_batch's algorithm: solvers.coneqp's).

    P (B, n, n), q (B, n), G (B, m, n), h (B, m), A (B, p, n) and b (B, p): CUDA float64 tensors on one device; A and
    b are optional and given together.  dims: the cone C shared by every problem, {'l': ml, 'q': [...], 's': [...]}
    ('s' orders at most 32), with m = ml + sum 'q' + sum of the 's' orders squared.  G's and h's rows are the 'l' rows,
    each 'q' cone, then each 's' block unpacked column-major; only an 's' block's lower triangle is read.  Returns
    (x, y, z, status_code): x (B, n), y (B, p), z (B, m) laid out as h with symmetric 's' blocks, and the int32 status
    per problem (1 optimal).  nsub: sub-batches solved concurrently, as qp_batch's.  options: maxiters, abstol,
    reltol, feastol, refinement.  Shape, dtype, device and dims errors are TypeErrors raised before any device work.

    Backward (once: no double backward) returns dL/dP (symmetric), dL/dq, dL/dG, dL/dh, dL/dA and dL/db from the
    gradients of x, y and z (cvxb_batch_adjoint_cone), with NaN for problems whose status is not 1.  An 's' block of
    z's gradient enters through its symmetric part, and the 's' blocks of dL/dh and of each column of dL/dG are the
    gradient over symmetric matrices, the same value in both triangles: a G whose 's' columns are built as X + X' gets
    the right gradient from autograd.  The solved batch is kept on the device from forward to backward."""
    return _ConeLayer.apply(P, q, G, h, A, b, dims, nsub, dict(options, _fw=_has_tangent(P, q, G, h, A, b)))


def conelp_layer(c, G, h, dims, A=None, b=None, nsub=None, **options):
    """Solve B cone LPs  minimize c'x  s.t.  G x + s = h,  s in C,  A x = b  on the GPU, differentiably
    (conelp_batch's algorithm, sdp_batch's with 's' blocks: solvers.conelp's).

    c (B, n) and the rest as coneqp_layer's, which this is with P = 0.  Returns (x, y, z, status_code); a problem
    found infeasible (status 4 or 5) gets NaN gradients like any status other than 1.  Backward returns dL/dc, dL/dG,
    dL/dh, dL/dA and dL/db with coneqp_layer's conventions."""
    return _ConeLayer.apply(None, c, G, h, A, b, dims, nsub, dict(options, _fw=_has_tangent(c, G, h, A, b)))


def gp_layer(K, F, g, G=None, h=None, A=None, b=None, nsub=None, **options):
    """Solve B geometric programs in log form  minimize lse(F_0 x + g_0)  s.t.  lse(F_i x + g_i) <= 0 (i = 1..mnl),
    G x <= h,  A x = b,  lse(u) = log sum exp(u),  on the GPU, differentiably (gp_batch's algorithm: solvers.gp's).

    K: the block sizes of F shared by every problem, a list of mnl + 1 positive ints.  F (B, sum K, n), g (B, sum K),
    G (B, ml, n), h (B, ml), A (B, p, n), b (B, p): CUDA float64 tensors on one device; G and h, A and b are optional
    and given in pairs.  Returns (x, y, znl, zl, status_code): x (B, n), the multipliers y (B, p) of A x = b, znl
    (B, mnl) of the posynomial constraints and zl (B, ml) of G x <= h, and the int32 status per problem (1 optimal).
    nsub: sub-batches solved concurrently, as qp_batch's.  options: maxiters, abstol, reltol, feastol, refinement.
    Shape, dtype, device and K errors are TypeErrors raised before any device work.

    A log-log convex layer: a posynomial sum_k c_k prod_j u_j^F_kj with coefficients c > 0 in the variables u = exp(x)
    is lse(F x + log c), so the coefficients enter as g = torch.log(c) and autograd carries the gradient on to c:

        x, y, znl, zl, status = gp_layer(K, F, torch.log(c), G, h)
        u = torch.exp(x)

    Backward (once: no double backward) returns dL/dF, dL/dg, dL/dG, dL/dh, dL/dA and dL/db from the gradients of x,
    y, znl and zl (cvxb_batch_adjoint_gp), with NaN for problems whose status is not 1; K gets none.  Inputs that need
    no gradient get none and cost nothing.  The solved batch is kept on the device from forward to backward, and
    freed by backward."""
    return _GPLayer.apply(K, F, g, G, h, A, b, nsub, dict(options, _fw=_has_tangent(F, g, G, h, A, b)))


def _check_cp(F, params, c, G, h, dims, A, b, cpl):
    """cp_layer's and cpl_layer's _check (cpl: c given, dims with 'l', 'q' and 's'), F() called once: every refusal
    before any device work.  Returns B, n, mnl, ml, p, x0 (a contiguous float64 tensor on the inputs' device), the
    dims the group takes (None: 'l' rows only) and params as a tuple"""
    if not callable(F):
        raise TypeError("F must be callable")
    if not isinstance(params, (tuple, list)):
        raise TypeError("params must be a tuple of tensors")
    params = tuple(params)
    if (A is None) != (b is None):
        raise TypeError("'A' and 'b' must be given together")
    if (G is None) != (h is None):
        raise TypeError("'G' and 'h' must be given together")
    named = ([("c", c)] if cpl else []) + ([("G", G), ("h", h)] if G is not None else []) + \
        ([("A", A), ("b", b)] if A is not None else []) + [("params[%d]" % i, t) for i, t in enumerate(params)]
    _typed(named)
    try:
        mnl, x0 = F()
    except Exception:
        raise ValueError("function call 'F()' failed") from None
    if type(mnl) is not int or mnl < 0:
        raise TypeError("the first output of F() must be a nonnegative integer")
    if not isinstance(x0, torch.Tensor):
        x0 = torch.as_tensor(np.asarray(x0))
    if x0.dtype != torch.float64 or x0.dim() != 2 or x0.shape[0] < 1 or x0.shape[1] < 1:
        raise TypeError("x0, F()'s second output, must be a float64 tensor of shape (B, n) with B and n positive")
    B, n = x0.shape
    if cpl and tuple(c.shape) != (B, n):
        raise TypeError("c must have shape (%d, %d), as x0" % (B, n))
    for name, t in named:
        if name.startswith("params") and (t.dim() < 1 or t.shape[0] != B):
            raise TypeError("%s must have leading dimension B = %d" % (name, B))
    ml, p = _constraint_rows(B, n, G, h, A, b)
    gdims = None
    if not cpl:
        _dims(dims, ml, "cp_layer")
    else:
        gdims = _cone_dims({"l": ml} if dims is None else dims, ml)
    if p > n:
        raise ValueError("Rank(A) < p or Rank([H(x); A; Df(x); G]) < n")
    if cpl and mnl + ml == 0:
        raise ValueError("cpl needs at least one constraint row (mnl + cdim = 0): its merit weight 1 / gap is undefined")
    if named:
        _on_device(named)
    dev = named[0][1].device if named else x0.device
    if dev.type != "cuda":
        raise TypeError("x0 must be a CUDA tensor when no other tensor is given")
    return B, n, mnl, ml, p, x0.to(dev).contiguous(), gdims, params


class _CPLayer(torch.autograd.Function):
    # inputs: F, c (None: cp_layer), G, h, A, b, the checked shapes and dims, nsub, options, then the params one by one
    @staticmethod
    def forward(ctx, F, c, G, h, A, b, info, nsub, options, *params):
        B, n, mnl, ml, p, x0, dims = info
        fw = options.pop("_fw")
        ctx.shapes, ctx.dev, ctx.cpl = (B, n, mnl, ml, p), x0.device, c is not None
        # F sees the params detached
        det = tuple(t.detach() for t in params)

        def Fd(x=None, z=None, idx=None):
            return F(x, idx=idx, params=det) if z is None else F(x, z, idx=idx, params=det)
        data = _layout((c, G, h, A, b), CPBatch._block[:1]) + [x0]
        if c is None:
            grp = CPBatchGroup(B, n, mnl, ml, p, _device(x0), nsub)
        else:
            grp = (SDPCPLBatchGroup if dims["s"] else CPLBatchGroup)(B, n, mnl, dims, p, _device(x0), nsub)
        needs = ctx.needs_input_grad
        x, y, z, status = _forward(
            ctx, grp, data, lambda part, c, G, h, A, b, x0: part.load_ptr(*(() if c is None else (c,)), x0, G, h,
                                                                          _lib.DEVICE, A, b),
            options, needs[1:6] + needs[9:], fw, Fd)
        if any(needs[9:]) or fw:             # the theta call's point and multipliers, and the detached params
            ctx.F, ctx.params, ctx.x, ctx.znl = F, det, x.clone(), z[:, :mnl].clone()
        return (x, y, *_split(z, mnl), status)

    @staticmethod
    @once_differentiable
    def backward(ctx, gx, gy, gznl, gzl, _gstatus):
        needp = ctx.needs_input_grad[9:]
        theta = any(needp)
        g = _grads(ctx, "adjoint_cp_ptr", CPBatch._block[:1], ctx.needs_input_grad[1:6], gx, gy, gznl, gzl, theta)
        dparams = _theta_grads(ctx, *g[5:], ctx.cpl, needp) if theta else [None] * len(needp)
        return (None, *g[:5], None, None, None, *dparams)

    @staticmethod
    def jvp(ctx, _dF, dc, dG, dh, dA, db, _dinfo, _nsub, _options, *dparams):
        needs = ctx.needs_input_grad
        tx = tf = None
        if any(t is not None for t in dparams):
            tx, tf = _theta_tangents(ctx, dparams, ctx.cpl)
        dirs = _layout((dc, tx, tf, dG, dh, dA, db), CPBatch._block)
        dx, dy, dz = _tangent(ctx, dirs, "tangent_cp_ptr", needs[1:6] + needs[9:])
        return (dx, dy, *_split(dz, ctx.shapes[2]), None)


def _theta_tangents(ctx, dparams, cpl):
    """tx = d_theta[Df(x; theta)' zk] dtheta and tf = d_theta[f_nl(x; theta)] dtheta at the returned x, x and z held
    constant (zk = [1; znl], f_nl = f[:, 1:]; cpl: znl and f), from one call F(x, idx=arange(B), params=...): the
    directional derivative as the gradient in u of <J'u, dtheta>, J'u by reverse mode (a dual level cannot be opened
    inside jvp)"""
    x, znl = ctx.x, ctx.znl
    B = x.shape[0]
    zk = znl if cpl else torch.cat([torch.ones((B, 1), dtype=x.dtype, device=x.device), znl], 1)
    with torch.enable_grad():
        leaves = tuple(t.detach().requires_grad_(d is not None) for t, d in zip(ctx.params, dparams))
        f, Df = ctx.F(x, idx=torch.arange(B, device=x.device), params=leaves)[:2]
        outs = ((Df * zk[:, :, None]).sum(1), f if cpl else f[:, 1:])
        us = tuple(torch.zeros_like(o, requires_grad=True) for o in outs)
        wrt = [(t, d) for t, d in zip(leaves, dparams) if d is not None]
        diff = [o for o in outs if o.requires_grad]
        if not diff:                     # F uses none of the params with a tangent
            return torch.zeros_like(outs[0]), torch.zeros_like(outs[1])
        vjp = torch.autograd.grad([o for o in outs if o.requires_grad], [t for t, _ in wrt],
                                  [u for o, u in zip(outs, us) if o.requires_grad], create_graph=True,
                                  allow_unused=True)
        s = sum((g * d).sum() for g, (_, d) in zip(vjp, wrt) if g is not None)
        if not isinstance(s, torch.Tensor) or not s.requires_grad:
            return torch.zeros_like(outs[0]), torch.zeros_like(outs[1])
        got = torch.autograd.grad(s, us, allow_unused=True)
    return tuple((torch.zeros_like(o) if g is None else g).detach() for o, g in zip(outs, got))


def _theta_grads(ctx, ux, uznl, cpl, needp):
    """dL/dtheta = -d_theta[ux' Df(x; theta)' zk + uk' f(x; theta)] for the params that need it (zk = [1; znl], uk =
    [0; uznl]; cpl: znl and uznl), from one call F(x, idx=arange(B), params=...) with those params as fresh leaves"""
    x, znl = ctx.x, ctx.znl
    B = x.shape[0]
    if cpl:
        zk, uk = znl, uznl
    else:
        zk = torch.cat([torch.ones((B, 1), dtype=x.dtype, device=x.device), znl], 1)
        uk = torch.cat([torch.zeros((B, 1), dtype=x.dtype, device=x.device), uznl], 1)
    with torch.enable_grad():
        leaves = tuple(t.detach().requires_grad_(nd) for t, nd in zip(ctx.params, needp))
        f, Df = ctx.F(x, idx=torch.arange(B, device=x.device), params=leaves)[:2]
        phi = (Df * (zk[:, :, None] * ux[:, None, :])).sum() + (uk * f).sum()
        wrt = [t for t, nd in zip(leaves, needp) if nd]
        # phi depends on none of them when F uses none of the params that need a gradient, or when f and Df are
        # empty (a cpl problem with mnl = 0): every such param gets zeros
        got = iter(torch.autograd.grad(phi, wrt, allow_unused=True) if phi.requires_grad else [None] * len(wrt))
    out = []
    for t, nd in zip(leaves, needp):
        if not nd:
            out.append(None)
            continue
        g = next(got)
        out.append(torch.zeros_like(t) if g is None else -g)
    return out


def cp_layer(F, params=(), G=None, h=None, A=None, b=None, nsub=None, **options):
    """Solve B smooth convex programs  minimize f_0(x; theta)  s.t.  f_i(x; theta) <= 0 (i = 1..mnl),  G x <= h,
    A x = b  on the GPU, differentiably (cp_batch's algorithm: solvers.cp's), with f written by the caller in torch.

    F is cp_batch's F with one more keyword, the parameters theta:
      F() -> (mnl, x0): mnl shared by the batch, x0 (B, n) float64 strictly inside dom f; no gradient reaches x0;
      F(x, idx=idx, params=params) -> (f, Df): f (k, mnl + 1), Df (k, mnl + 1, n) at the k points x of the problems
          idx (int64 indices into the batch);
      F(x, z, idx=idx, params=params) -> (f, Df, H): also H (k, n, n) = sum_i z_i grad² f_i(x), lower triangle read.
    params: a tuple of CUDA float64 tensors with leading dimension B, which F indexes with idx.  G (B, ml, n),
    h (B, ml), A (B, p, n), b (B, p): CUDA float64 tensors on the params' device, optional and given in pairs.
    Returns (x, y, znl, zl, status_code) as qcqp_layer.  nsub: sub-batches solved concurrently, as qp_batch's.
    options: maxiters, abstol, reltol, feastol, refinement, and dims ({'l': ml} only: 'q' and 's' cones raise
    NotImplementedError).  Shape, dtype and device errors are TypeErrors raised before any device work.

    Backward (once: no double backward) runs cvxb_batch_adjoint_cp, which calls F(x, z) once more per sub-batch, and
    returns dL/dG, dL/dh, dL/dA, dL/db and, for a param that needs one, dL/dparam = -d_param[ux' Df' zk + uk' f] with
    zk = [1; znl] and uk = [0; uznl], from one more call F(x, idx=arange(B), params=...) under autograd; a param F does
    not use gets zeros.  Problems whose status is not 1 get NaN.  Inputs that need no gradient get none and cost
    nothing: without a param that needs one, F is not called for theta.  The solved batch is kept on the device from
    forward to backward, and freed by backward.  F must return the same values for the same point; it runs on the
    library's stream and may see its rows in any order."""
    dims = options.pop("dims", None)
    B, n, mnl, ml, p, x0, _, params = _check_cp(F, params, None, G, h, dims, A, b, False)
    return _CPLayer.apply(F, None, G, h, A, b, (B, n, mnl, ml, p, x0, None), nsub,
                          dict(options, _fw=_has_tangent(G, h, A, b, *params)), *params)


def cpl_layer(c, F, params=(), G=None, h=None, dims=None, A=None, b=None, nsub=None, **options):
    """Solve B convex problems  minimize c'x  s.t.  f_i(x; theta) <= 0 (i = 1..mnl),  G x + s = h,  s in C,  A x = b
    on the GPU, differentiably (cpl_batch's algorithm, sdp_cpl_batch's with 's' blocks: solvers.cpl's).

    F is cp_layer's without the objective row: f (k, mnl), Df (k, mnl, n), z (k, mnl).  c (B, n); G and h with dims
    {'l': ml, 'q': [...], 's': [...]} as coneqp_layer's ('s' orders at most 32, each block unpacked column-major, only
    its lower triangle read); dims None is {'l': rows of G}.  Returns (x, y, znl, zl, status_code), zl laid out as h
    with symmetric 's' blocks.  Backward returns dL/dc = -ux, dL/dG, dL/dh, dL/dA, dL/db with coneqp_layer's 's'
    conventions, and dL/dparam as cp_layer's with zk = znl and uk = uznl.  The rest is cp_layer's."""
    B, n, mnl, ml, p, x0, gdims, params = _check_cp(F, params, c, G, h, dims, A, b, True)
    return _CPLayer.apply(F, c, G, h, A, b, (B, n, mnl, ml, p, x0, gdims), nsub,
                          dict(options, _fw=_has_tangent(c, G, h, A, b, *params)), *params)
