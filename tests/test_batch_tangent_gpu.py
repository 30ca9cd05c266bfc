"""The batch tangents (cvxb_batch_tangent, _qcqp, _gp, _cp, the batches' tangent methods and the layers' forward mode)
on the device: a dense numpy solve of the KKT matrix at the batch's own returned iterate; duality with the adjoint,
<g, tangent(d)> = <adjoint(g), d> for non-symmetric d, on every kind; central differences of the batch's own
re-solves; the 's' convention; the NaN policy; bit-identity across sub-batches, compaction, spaces and repeated calls;
the zero direction; the refusals; and forward-mode AD through every layer."""

import numpy as np
import pytest

import cp_problems as cpp
import cpl_problems as cplp
from sdcpl_problems import sdcpl_batch_data
from test_batch_adjoint_gpu import _batch
from test_batch_conelp_gpu import lp_batch
from test_batch_cone_adjoint_gpu import _group as _cone_group
from test_batch_cp_adjoint_gpu import _cp_group, _cpl_group
from test_batch_eq_gpu import eq_batch
from test_batch_gp_adjoint_gpu import _data as _gp_data, _solved_group as _gp_group
from test_batch_qcqp_adjoint_gpu import _data as _qc_data, _solved_group as _qc_group
from test_batch_sdp_gpu import sdp_batch_data
from test_batch_sdqp_gpu import sdqp_batch_data
from qcqp_problems import sym

pytestmark = pytest.mark.gpu

DIMS = {"l": 6, "q": [4, 3], "s": [3, 2]}


def _rng_like(rng, arrays):
    return [None if a is None else rng.standard_normal(np.shape(a)) for a in arrays]


def _pair(a, b):
    """per-problem entrywise inner product of two (B, ...) arrays"""
    return (a * b).reshape(a.shape[0], -1).sum(1)


def _check_duality(t, g, adj, d, ok, tol=1e-8):
    """<g, (dx, dy, dz)> against sum over the keys of <adj[k], d[k]>, per optimal problem, relative to the terms' size"""
    lhs = sum(_pair(a, b) for a, b in zip(g, t))
    rhs = sum(_pair(adj[k], d[k]) for k in d)
    scale = sum(np.abs(a * b).reshape(a.shape[0], -1).sum(1) for a, b in zip(g, t)) + \
        sum(np.abs(adj[k] * d[k]).reshape(d[k].shape[0], -1).sum(1) for k in d)
    err = np.abs(lhs - rhs)[ok] / scale[ok]
    assert err.max() <= tol, err.max()
    return err.max()


def _grads(B, widths, seed):
    rng = np.random.default_rng(seed)
    return [rng.standard_normal((B, w)) for w in widths]


QP_CASES = [  # kind, B, n, dims, p
    ("qp", 9, 10, {"l": 14}, 3), ("qp", 7, 8, {"l": 12}, 0), ("qp", 7, 10, {"l": 8, "q": [4, 3]}, 2),
    ("sdqp", 9, 10, DIMS, 2), ("lp", 9, 10, {"l": 12, "q": [4, 3]}, 2), ("sdp", 9, 8, {"l": 6, "s": [1, 4]}, 2),
    ("sdp", 257, 6, {"l": 4, "s": [3]}, 0),
]


def _qp_data(kind, B, n, dims, p, seed):
    if kind == "sdqp":
        return sdqp_batch_data(B, n, dims, p, seed)
    if kind == "sdp":
        return sdp_batch_data(B, n, dims, p, seed)
    return (lp_batch if kind == "lp" else eq_batch)(B, n, dims, p, seed)


@pytest.mark.parametrize("kind,B,n,dims,p", QP_CASES)
def test_tangent_qp_and_cone_is_the_adjoints_transpose(kind, B, n, dims, p):
    data = list(_qp_data(kind, B, n, dims, p, 500))
    lp = kind in ("lp", "sdp")
    keys = ("c", "G", "h", "A", "b") if lp else ("P", "q", "G", "h", "A", "b")
    m = data[-3].shape[1]
    grp = _cone_group(tuple(data), dims, nsub=2)
    try:
        ok = grp.results()["status_code"] == 1
        d = dict(zip(keys, _rng_like(np.random.default_rng(3), data)))   # non-symmetric dP, dG and dh blocks
        if not p:
            d.pop("A"), d.pop("b")
        g = _grads(B, (n, p, m), 4)
        t = grp.tangent(**{"d" + k: v for k, v in d.items()})
        adj = grp.adjoint_cone(*g, want=tuple(d))
    finally:
        grp.close()
    assert ok.sum() >= max(1, 4 * B // 5)
    assert all(np.isfinite(a[ok]).all() for a in t)
    print("\n%s %s: duality %.1e" % (kind, dims, _check_duality(t, g, adj, d, ok)))


def test_tangent_qp_matches_dense_kkt_solve():
    """r of include/cvxopt_b200.h and M = [P A' G'; A 0 0; G 0 -diag(s / z)] at the returned iterate, solved densely"""
    for p in (3, 0):
        B, n, m = 12, 10, 16
        data = _batch(B, n, m, p, 510)
        grp = _cone_group(tuple(data), {"l": m}, nsub=1)
        try:
            res = grp.results()
            rng = np.random.default_rng(5)
            dP, dq, dG, dh, dA, db = _rng_like(rng, data)
            t = grp.tangent(dP, dq, dG, dh, dA if p else None, db if p else None)
        finally:
            grp.close()
        P, q, G, h, A, b = data
        x, y, s, z = (res[k] for k in ("x", "y", "s", "z"))
        for j in np.flatnonzero(res["status_code"] == 1):
            M = np.zeros((n + p + m, n + p + m))
            M[:n, :n] = P[j]
            M[n:n + p, :n], M[:n, n:n + p] = A[j], A[j].T
            M[n + p:, :n], M[:n, n + p:] = G[j], G[j].T
            M[n + p:, n + p:] = -np.diag(s[j] / z[j])
            rx = -(0.5 * (dP[j] + dP[j].T) @ x[j] + dq[j] + (dA[j].T @ y[j] if p else 0) + dG[j].T @ z[j])
            r = np.concatenate([rx, (db[j] - dA[j] @ x[j]) if p else np.zeros(0), dh[j] - dG[j] @ x[j]])
            D = 1.0 / np.sqrt(np.abs(M).max(axis=1))
            u = D * np.linalg.solve(D[:, None] * M * D, D * r)
            got = np.concatenate([t[0][j], t[1][j], t[2][j]])
            tol = max(1e-9, 10 * np.finfo(float).eps * np.linalg.cond(M))
            assert np.linalg.norm(got - u) <= tol * np.linalg.norm(u), (p, j)


def test_tangent_qp_matches_central_differences():
    """x(theta + eps d) - x(theta - eps d) from the batch's own re-solves at tolerances 1e-10, on the seeds whose
    solution has a strict-complementarity margin min max(s, z) of at least 2e-2 (test_batch_adjoint_gpu's)"""
    n, m, p = 12, 20, 3
    parts = [_batch(1, n, m, p, 4000 + seed) for seed in (0, 1, 4, 5, 7)]
    data = [np.concatenate([d[i] for d in parts]) for i in range(6)]
    B = data[0].shape[0]
    tight = dict(abstol=1e-10, reltol=1e-10, feastol=1e-10)
    d = _rng_like(np.random.default_rng(6), data)
    d[0] = d[0] + d[0].transpose(0, 2, 1)               # a perturbed P must stay symmetric
    grp = _cone_group(tuple(data), {"l": m}, nsub=1, **tight)
    try:
        res = grp.results()
        t = grp.tangent(*d)
    finally:
        grp.close()
    eps = 1e-5
    xs = []
    for sgn in (1, -1):
        g2 = _cone_group(tuple(a + sgn * eps * da for a, da in zip(data, d)), {"l": m}, nsub=1, **tight)
        try:
            xs.append(g2.results()["x"])
        finally:
            g2.close()
    fd = (xs[0] - xs[1]) / (2 * eps)
    assert (res["status_code"] == 1).all() and np.maximum(res["s"], res["z"]).min() > 2e-2
    for j in range(B):
        assert np.linalg.norm(fd[j] - t[0][j]) <= 1e-4 * np.linalg.norm(t[0][j]), j


def test_s_convention():
    """d and d' of each 's' block (of dh and of dG's columns) give the same tangent, and dz's blocks are symmetric"""
    B, n, p = 6, 10, 2
    data = sdqp_batch_data(B, n, DIMS, p, 530)
    grp = _cone_group(tuple(data), DIMS, nsub=1)
    rng = np.random.default_rng(7)
    dG, dh = rng.standard_normal(data[2].shape), rng.standard_normal(data[3].shape)
    dGt, dht = dG.copy(), dh.copy()
    o = DIMS["l"] + sum(DIMS["q"])
    for k in DIMS["s"]:
        blk = slice(o, o + k * k)
        dht[:, blk] = dh[:, blk].reshape(B, k, k).transpose(0, 2, 1).reshape(B, -1)
        dGt[:, blk] = dG[:, blk].reshape(B, k, k, n).transpose(0, 2, 1, 3).reshape(B, k * k, n)
        o += k * k
    try:
        t1 = grp.tangent(dG=dG, dh=dh)
        t2 = grp.tangent(dG=dGt, dh=dht)
    finally:
        grp.close()
    for a, b in zip(t1, t2):
        assert np.allclose(a, b, rtol=1e-10, atol=1e-12)
    o = DIMS["l"] + sum(DIMS["q"])
    for k in DIMS["s"]:
        Z = t1[2][:, o:o + k * k].reshape(B, k, k)
        assert np.allclose(Z, Z.transpose(0, 2, 1), rtol=1e-12, atol=1e-13)
        o += k * k


@pytest.mark.parametrize("kind", ["quad", "linear"])
def test_tangent_qcqp_is_the_adjoints_transpose(kind):
    d = _qc_data(12, 16, 3, 2, 4, kind, 540)
    B, nK, n = d["P"].shape[:3]
    ml, p = d["G"].shape[1], d["A"].shape[1]
    grp = _qc_group(d, nsub=2)
    try:
        ok = grp.results()["status_code"] == 1
        dd = dict(zip(("P", "q", "r", "G", "h", "A", "b"),
                      _rng_like(np.random.default_rng(8), [d[k] for k in ("P", "q", "r", "G", "h", "A", "b")])))
        dd["r"][:, 0] = 0.0                          # r_0 is the objective's constant: no effect, adjoint dr_0 = 0
        g = _grads(B, (n, p, nK - 1 + ml), 9)
        t = grp.tangent(**{"d" + k: v for k, v in dd.items()})
        adj = grp.adjoint(*g, want=tuple(dd))
    finally:
        grp.close()
    assert ok.sum() >= 4 * B // 5
    print("\nqcqp %s: duality %.1e" % (kind, _check_duality(t, g, adj, dd, ok)))


@pytest.mark.parametrize("K,p", [([32, 8, 8, 8], 0), ([16, 1, 8, 1], 2)])
def test_tangent_gp_is_the_adjoints_transpose(K, p):
    d = _gp_data(12, 16, K, 4, p, 550)
    B, S, n = d["F"].shape
    ml = d["G"].shape[1]
    grp = _gp_group(K, d, nsub=2)
    try:
        ok = grp.results()["status_code"] == 1
        keys = ("F", "g", "G", "h") + (("A", "b") if p else ())
        dd = dict(zip(keys, _rng_like(np.random.default_rng(10), [d[k] for k in keys])))
        g = _grads(B, (n, p, len(K) - 1 + ml), 11)
        t = grp.tangent_gp(**{"d" + k: v for k, v in dd.items()})
        adj = grp.adjoint_gp(*g, want=keys)
    finally:
        grp.close()
    assert ok.sum() >= 4 * B // 5
    print("\ngp K=%s: duality %.1e" % (K, _check_duality(t, g, adj, dd, ok)))


def _cp_duality(grp, B, n, p, mnl, ml, cpl, seed):
    """<g, tangent(d)> = <adjoint_cp(g), d>, with tx and tf paired with -ux and -uznl (dL/dtheta's formula)"""
    rng = np.random.default_rng(seed)
    ok = grp.results()["status_code"] == 1
    d = {"tx": rng.standard_normal((B, n)), "tf": rng.standard_normal((B, mnl)),
         "G": rng.standard_normal((B, ml, n)), "h": rng.standard_normal((B, ml))}
    if p:
        d.update(A=rng.standard_normal((B, p, n)), b=rng.standard_normal((B, p)))
    if cpl:
        d["c"] = rng.standard_normal((B, n))
    g = _grads(B, (n, p, mnl + ml), seed + 1)
    t = grp.tangent_cp(**{("d" + k if k not in ("tx", "tf") else k): v for k, v in d.items()})
    adj = grp.adjoint_cp(*g)
    adj = dict(adj, tx=-adj["ux"], tf=-adj["uznl"])
    assert ok.sum() >= 4 * B // 5
    return _check_duality(t, g, adj, d, ok)


@pytest.mark.parametrize("family,n,p,r", [("qcqp", 6, 0, 3), ("entropy", 10, 2, 4), ("centering", 8, 3, 0)])
def test_tangent_cp_is_the_adjoints_transpose(family, n, p, r):
    B = 8
    d = cpp.cp_batch_data(family, range(560, 560 + B), n, p, r)
    grp = _cp_group(family, d, nsub=2)
    try:
        print("\ncp %s: duality %.1e" % (family, _cp_duality(grp, B, n, p, cpp.MNL[family], d["G"].shape[1], False,
                                                             12)))
        with pytest.raises(TypeError, match="no c"):
            grp.tangent_cp(dc=np.zeros((B, n)))
    finally:
        grp.close()


@pytest.mark.parametrize("family,n,q,s,ml,p", [("socp", 8, [3, 4], [], 2, 1), ("lsecone", 7, [3], [], 1, 0),
                                              ("socp", 8, [3], [3, 2], 2, 0)])
def test_tangent_cpl_is_the_adjoints_transpose(family, n, q, s, ml, p):
    B = 6
    if s:
        d = sdcpl_batch_data(family, range(570, 570 + B), n, q, s, ml, p)
    else:
        d = cplp.cpl_batch_data(family, range(570, 570 + B), n, q, ml, p)
    grp = _cpl_group(family, d, nsub=2)
    try:
        print("\ncpl %s: duality %.1e" % (family, _cp_duality(grp, B, n, p, cplp.MNL[family], d["G"].shape[1], True,
                                                              14)))
    finally:
        grp.close()


def test_nan_policy_zero_direction_and_bit_identity(monkeypatch):
    """problems stopped before optimality get NaN rows; a zero direction gives zeros; the tangent is bit-identical
    across sub-batches, compaction, HOST / DEVICE spaces and repeated calls, and the results do not move"""
    import torch
    B, n, p = 9, 10, 2
    data = sdqp_batch_data(B, n, DIMS, p, 580)
    data[1] *= np.linspace(0.1, 30.0, B)[:, None]       # spread the iteration counts: compaction moves problems
    m = data[2].shape[1]
    d = _rng_like(np.random.default_rng(15), data)
    outs = []
    for compact, nsub in (("1", 1), ("0", 1), ("1", 3)):
        monkeypatch.setenv("CVXB_BATCH_COMPACT", compact)
        grp = _cone_group(tuple(data), DIMS, nsub=nsub)
        try:
            before = grp.results()
            outs.append(grp.tangent(*d))
            outs.append(grp.tangent(*d))
            zero = grp.tangent()
            after = grp.results()
        finally:
            grp.close()
        for k in ("x", "y", "s", "z"):
            assert np.array_equal(before[k], after[k])
        ok = before["status_code"] == 1
        assert ok.all()
        for a in zero:
            assert not np.any(a)
    for o in outs[1:]:
        for a, b in zip(o, outs[0]):
            assert np.array_equal(a, b)
    # DEVICE space through tangent_ptr on torch tensors
    monkeypatch.setenv("CVXB_BATCH_COMPACT", "1")
    grp = _cone_group(tuple(data), DIMS, nsub=1)
    dev = torch.device("cuda", 0)
    try:
        part = grp.parts[0]
        cm = [torch.from_numpy(np.ascontiguousarray(a.transpose(0, 2, 1) if a.ndim == 3 else a)).to(dev) for a in d]
        o = [torch.empty((B, w), dtype=torch.float64, device=dev) for w in (n, p, m)]
        torch.cuda.synchronize()
        part.tangent_ptr(*(t.data_ptr() for t in cm), *(t.data_ptr() for t in o))
        for a, b in zip(o, outs[0]):
            assert np.array_equal(a.cpu().numpy(), b)
        # NaN policy: stopped after 3 iterations, nothing is optimal
        grp.solve(maxiters=3)
        st = grp.results()["status_code"]
        t = grp.tangent(*d)
        for a in t:
            assert np.isnan(a[st != 1]).all()
    finally:
        grp.close()


def test_nan_rows_leave_the_others_bit_identical():
    """a primal infeasible problem gets NaN rows; the other problems' tangents equal those of a batch without it"""
    B, n, p = 8, 10, 0
    dims = {"l": 12, "q": [4, 3]}
    data = lp_batch(B, n, dims, p, 590, kinds={3: "pinf"})
    rng = np.random.default_rng(16)
    d = [rng.standard_normal(a.shape) for a in data[:3]]
    keep = np.array([j for j in range(B) if j != 3])
    g1 = _cone_group(tuple(data), dims, nsub=1)
    g2 = _cone_group(tuple(a[keep] for a in data), dims, nsub=1)
    try:
        st = g1.results()["status_code"]
        t1 = g1.tangent(*d)
        t2 = g2.tangent(*(a[keep] for a in d))
    finally:
        g1.close()
        g2.close()
    assert st[3] != 1
    for a, b in zip(t1, t2):
        assert np.isnan(a[3]).all()
        assert np.array_equal(a[keep], b)


def test_refuses_other_kinds():
    from cvxopt_b200 import GPBatch, QCQPBatch, QPBatch
    qp = QPBatch(2, 3, 4)
    qc = QCQPBatch(2, 3, 1, 2)
    gp = GPBatch(2, 3, [2, 2], 2)
    try:
        for obj, call in ((qc, "cvxb_batch_tangent"), (gp, "cvxb_batch_tangent"), (qp, "cvxb_batch_tangent_qcqp"),
                          (gp, "cvxb_batch_tangent_qcqp"), (qp, "cvxb_batch_tangent_gp"),
                          (qc, "cvxb_batch_tangent_gp"), (qp, "cvxb_batch_tangent_cp"),
                          (qc, "cvxb_batch_tangent_cp"), (gp, "cvxb_batch_tangent_cp")):
            from cvxopt_b200 import _lib
            nargs = 10 if call in ("cvxb_batch_tangent_qcqp", "cvxb_batch_tangent_cp") else 9
            assert getattr(obj._lib, call)(obj._h, *([None] * nargs), _lib.HOST) == _lib.E_UNSUP, (call, obj)
        with pytest.raises(ValueError, match="no completed"):     # not solved since the last load
            qp.tangent()
    finally:
        for o in (qp, qc, gp):
            o.close()


def _torch(arrays, dev=None):
    import torch
    dev = dev or torch.device("cuda", 0)
    return [None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in arrays]


def _fw(layer, primals, tangents, *args, **kw):
    """the layer's outputs' primal values and tangents under forward-mode AD"""
    import torch.autograd.forward_ad as fwAD
    with fwAD.dual_level():
        duals = [p if t is None else fwAD.make_dual(p, t) for p, t in zip(primals, tangents)]
        out = layer(*duals[:kw.pop("_split", len(duals))], *args, *duals[kw.pop("_rest", len(duals)):], **kw)
        return [fwAD.unpack_dual(o) for o in out]


def test_qp_layer_forward_ad_equals_group_tangent_and_pairs_with_backward():
    import torch
    import torch.autograd.forward_ad as fwAD
    from cvxopt_b200 import _lib, qp_layer
    B, n, m, p = 12, 8, 10, 2
    data = _batch(B, n, m, p, 600)
    d = _rng_like(np.random.default_rng(17), data)
    lib = _lib.load()
    before = lib.cvxb_device_bytes()
    t, dt = _torch(data), _torch(d)
    with fwAD.dual_level():
        out = qp_layer(*(fwAD.make_dual(a, b) for a, b in zip(t, dt)), nsub=3)
        got = [fwAD.unpack_dual(o).tangent for o in out[:3]]
        assert fwAD.unpack_dual(out[3]).tangent is None
    assert lib.cvxb_device_bytes() == before              # forward mode only: jvp freed the group
    grp = _cone_group(tuple(data), {"l": m}, nsub=3)
    try:
        want = grp.tangent(*d)
    finally:
        grp.close()
    for a, b in zip(got, want):
        assert np.array_equal(a.cpu().numpy(), b)
    # <g, jvp(d)> = <vjp(g), d> through the layer's own backward, with both modes on the same call
    g = _torch(_grads(B, (n, p, m), 18))
    leaves = [a.clone().requires_grad_() for a in t]
    with fwAD.dual_level():
        out = qp_layer(*(fwAD.make_dual(a, b) for a, b in zip(leaves, dt)))
        jv = [fwAD.unpack_dual(o).tangent for o in out[:3]]
        prim = [fwAD.unpack_dual(o).primal for o in out[:3]]
    vj = torch.autograd.grad(sum((a * b).sum() for a, b in zip(prim, g)), leaves)
    assert lib.cvxb_device_bytes() == before              # both modes: backward freed it
    lhs = sum((a * b).sum() for a, b in zip(g, jv))
    rhs = sum((a * b).sum() for a, b in zip(vj, dt))
    assert abs(float(lhs - rhs)) <= 1e-8 * float(sum((a * b).abs().sum() for a, b in zip(vj, dt)))
    x, y, z, _ = qp_layer(*leaves)                        # backward only
    torch.autograd.grad((x * g[0]).sum(), leaves[:2])
    assert lib.cvxb_device_bytes() == before


@pytest.mark.parametrize("lp", [False, True])
def test_cone_layers_forward_ad_and_side_stream(lp):
    import torch
    from cvxopt_b200 import _lib, conelp_layer, coneqp_layer
    B, n, p = 9, 10, 2
    data = sdp_batch_data(B, n, {"l": 6, "s": [1, 4]}, p, 610) if lp else sdqp_batch_data(B, n, DIMS, p, 610)
    dims = {"l": 6, "s": [1, 4]} if lp else DIMS
    d = _rng_like(np.random.default_rng(19), data)
    lib = _lib.load()
    before = lib.cvxb_device_bytes()

    def run(stream=None):
        with torch.cuda.stream(stream):
            k = 3 if lp else 4
            out = _fw(conelp_layer if lp else coneqp_layer, _torch(data), _torch(d), dims, _split=k, _rest=k, nsub=2)
            torch.cuda.synchronize()
        return [o.tangent for o in out[:3]]
    full = run()
    assert lib.cvxb_device_bytes() == before
    side = run(torch.cuda.Stream())
    for a, b in zip(side, full):
        assert torch.equal(a, b)
    grp = _cone_group(tuple(data), dims, nsub=2)
    try:
        want = grp.tangent(*d)
    finally:
        grp.close()
    for a, b in zip(full, want):
        assert np.array_equal(a.cpu().numpy(), b)


def test_qcqp_and_gp_layers_forward_ad_equal_group_tangents():
    from cvxopt_b200 import _lib, gp_layer, qcqp_layer
    lib = _lib.load()
    before = lib.cvxb_device_bytes()
    d = _qc_data(10, 12, 2, 2, 4, "quad", 620)
    keys = ("P", "q", "r", "G", "h", "A", "b")
    dd = _rng_like(np.random.default_rng(20), [d[k] for k in keys])
    out = _fw(qcqp_layer, _torch([d[k] for k in keys]), _torch(dd), nsub=2)
    grp = _qc_group(d, nsub=2)
    try:
        want = grp.tangent(*dd)
    finally:
        grp.close()
    mnl = d["P"].shape[1] - 1
    got = [out[0].tangent, out[1].tangent, np.concatenate([out[2].tangent.cpu().numpy(),
                                                           out[3].tangent.cpu().numpy()], 1)]
    for a, b in zip(got, want):
        assert np.array_equal(a if isinstance(a, np.ndarray) else a.cpu().numpy(), b)
    assert out[2].tangent.shape[1] == mnl
    K = [16, 4, 4]
    g = _gp_data(10, 8, K, 3, 2, 630)
    keys = ("F", "g", "G", "h", "A", "b")
    dg = _rng_like(np.random.default_rng(21), [g[k] for k in keys])
    out = _fw(lambda *a, **kw: gp_layer(K, *a, **kw), _torch([g[k] for k in keys]), _torch(dg), nsub=2)
    grp = _gp_group(K, g, nsub=2)
    try:
        want = grp.tangent_gp(*dg)
    finally:
        grp.close()
    got = [out[0].tangent.cpu().numpy(), out[1].tangent.cpu().numpy(),
           np.concatenate([out[2].tangent.cpu().numpy(), out[3].tangent.cpu().numpy()], 1)]
    for a, b in zip(got, want):
        assert np.array_equal(a, b)
    assert lib.cvxb_device_bytes() == before


def _qcqp_param_F(x0):
    """the convex QCQP f_i(x) = x'P_i x / 2 + q_i'x + r_i with (P, q, r) as F's params"""
    import torch

    def F(x=None, z=None, idx=None, params=()):
        if x is None:
            return 1, x0
        P, q, r = (t[idx] for t in params)
        Px = torch.einsum("bkij,bj->bki", P, x)
        f = 0.5 * (Px * x[:, None, :]).sum(2) + (q * x[:, None, :]).sum(2) + r
        Df = Px + q
        if z is None:
            return f, Df
        return f, Df, torch.einsum("bk,bkij->bij", z, P)
    return F


def test_cp_layer_theta_tangent_matches_qcqp_layer():
    """cp_layer on F(x; P, q, r) = the qcqp family: its forward-mode tangent in (P, q, r, G, h) equals qcqp_layer's"""
    import torch.autograd.forward_ad as fwAD
    from cvxopt_b200 import _lib, cp_layer, qcqp_layer
    lib = _lib.load()
    before = lib.cvxb_device_bytes()
    d = _qc_data(8, 6, 1, 0, 3, "quad", 640)
    rng = np.random.default_rng(22)
    Psym = sym(d["P"])
    dP = rng.standard_normal(Psym.shape)
    dP = dP + dP.transpose(0, 1, 3, 2)                   # F reads both triangles: a symmetric direction
    dq, dr, dG, dh = (rng.standard_normal(d[k].shape) for k in ("q", "r", "G", "h"))
    P, q, r, G, h, x0 = _torch([Psym, d["q"], d["r"], d["G"], d["h"], d["x0"]])
    tP, tq, tr, tG, th = _torch([dP, dq, dr, dG, dh])
    with fwAD.dual_level():
        params = tuple(fwAD.make_dual(a, b) for a, b in ((P, tP), (q, tq), (r, tr)))
        out = cp_layer(_qcqp_param_F(x0), params, fwAD.make_dual(G, tG), fwAD.make_dual(h, th), nsub=2)
        got = [fwAD.unpack_dual(o).tangent for o in out[:4]]
        ok = (out[4] == 1).cpu().numpy()
        out = qcqp_layer(*(fwAD.make_dual(a, b) for a, b in ((P, tP), (q, tq), (r, tr), (G, tG), (h, th))))
        want = [fwAD.unpack_dual(o).tangent for o in out[:4]]
        ok &= (out[4] == 1).cpu().numpy()
    assert ok.sum() >= 6
    worst = max(float(np.abs(a.cpu().numpy()[ok] - b.cpu().numpy()[ok]).max() /
                      max(1.0, np.abs(b.cpu().numpy()[ok]).max())) for a, b in zip(got, want) if a.shape[1])
    print("\ncp_layer theta tangent vs qcqp_layer: largest difference %.1e" % worst)
    assert worst <= 1e-6
    assert lib.cvxb_device_bytes() == before
