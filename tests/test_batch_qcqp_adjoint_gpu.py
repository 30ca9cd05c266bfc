"""The QCQP batch's adjoint (cvxb_batch_adjoint_qcqp, QCQPBatch.adjoint, qcqp_layer) on the device, on
tests/qcqp_problems.py's families: parity with a dense numpy solve of the KKT matrix at the batch's own returned
iterate, central differences of the reference's solvers.cp, the NaN policy, bit-identity across compaction,
sub-batches, spaces, repeated calls and the noise above each P_i's diagonal, the call contract and the torch layer."""

import numpy as np
import pytest

from qcqp_problems import qcqp_batch_data, ref_F, sym

pytestmark = pytest.mark.gpu

KEYS = ("P", "q", "r", "G", "h", "A", "b")


def _data(B, n, mnl, p, r, kind, seed):
    return qcqp_batch_data(range(seed, seed + B), n, mnl, p, r, kind)


def _dims(d):
    B, nK, n = d["P"].shape[:3]
    return B, n, nK - 1, d["G"].shape[1], d["A"].shape[1]


def _solved_group(d, nsub=None, **options):
    from cvxopt_b200 import QCQPBatchGroup
    B, n, mnl, ml, p = _dims(d)
    grp = QCQPBatchGroup(B, n, mnl, ml, p, 0, nsub)
    grp.load(d["P"], d["q"], d["r"], d["x0"], d["G"], d["h"], d["A"] if p else None, d["b"] if p else None)
    grp.solve(**options)
    return grp


def _grads(d, seed):
    B, n, mnl, ml, p = _dims(d)
    rng = np.random.default_rng(seed)
    return rng.standard_normal((B, n)), rng.standard_normal((B, p)), rng.standard_normal((B, mnl + ml))


def _oracle(d, res, g):
    """per problem, at the returned iterate with z_0 = 1: H = P_0 + sum znl_i P_i, Df's rows (P_i x + q_i)',
    M = [H A' Df' G'; A 0 0 0; Df 0 -Dnl 0; G 0 0 -Dl] with D = diag(s / z), u = M^{-1} g (equilibrated), the
    formulas of include/cvxopt_b200.h, and cond(M)"""
    B, n, mnl, ml, p = _dims(d)
    m = mnl + ml
    out = {k: [] for k in KEYS}
    cond = []
    for j in range(B):
        P = sym(d["P"][j])
        x, y, s, z = (np.asarray(res[k][j]) for k in ("x", "y", "s", "z"))
        znl = z[:mnl]
        H = P[0] + np.tensordot(znl, P[1:], 1)
        Gf = np.vstack([P[1:] @ x + d["q"][j][1:], d["G"][j]])
        A = d["A"][j]
        M = np.zeros((n + p + m, n + p + m))
        M[:n, :n] = H
        M[n:n + p, :n] = A
        M[:n, n:n + p] = A.T
        M[n + p:, :n] = Gf
        M[:n, n + p:] = Gf.T
        M[n + p:, n + p:] = -np.diag(s / z)
        D = 1.0 / np.sqrt(np.abs(M).max(axis=1))
        u = D * np.linalg.solve(D[:, None] * M * D, D * np.concatenate([g[0][j], g[1][j], g[2][j]]))
        ux, uy, uz = u[:n], u[n:n + p], u[n + p:]
        S = np.outer(ux, x) + np.outer(x, ux)
        zk, uk = np.concatenate([[1.0], znl]), np.concatenate([[0.0], uz[:mnl]])
        out["P"].append(np.array([-(zk[i] * S + uk[i] * np.outer(x, x)) / 2 for i in range(mnl + 1)]))
        out["q"].append(np.array([-(zk[i] * ux + uk[i] * x) for i in range(mnl + 1)]))
        out["r"].append(-uk)
        out["G"].append(-(np.outer(z[mnl:], ux) + np.outer(uz[mnl:], x)))
        out["h"].append(uz[mnl:])
        out["A"].append(-(np.outer(y, ux) + np.outer(uy, x)))
        out["b"].append(uy)
        cond.append(np.linalg.cond(M))
    return {k: np.array(v) for k, v in out.items()}, np.array(cond)


def _rel(a, b):
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


def _check_oracle(got, want, cond, rows=None):
    """every output within max(1e-9, 10 u cond(M)) relative of the oracle, per problem; returns the largest relative
    difference"""
    rows = range(len(cond)) if rows is None else rows
    worst = 0.0
    for j in rows:
        tol = max(1e-9, 10 * np.finfo(float).eps * cond[j])
        for k in got:
            dd = _rel(got[k][j], want[k][j])
            assert dd <= tol, (j, k, dd, cond[j])
            worst = max(worst, dd)
    return worst


SHAPES = [  # n, mnl, p, r, B, kind
    (16, 3, 2, 4, 12, "quad"),
    (16, 2, 2, 4, 16, "linear"),        # P_0 = 0
    (16, 0, 2, 4, 20, "quad"),          # mnl = 0
    (12, 0, 4, 0, 10, "deficient"),     # S + A'A
    (32, 2, 0, 8, 1, "quad"),           # B = 1
    (24, 8, 3, 6, 257, "quad"),         # several sub-batches, compaction
]


@pytest.mark.parametrize("n,mnl,p,r,B,kind", SHAPES)
def test_adjoint_matches_dense_kkt_solve(n, mnl, p, r, B, kind):
    d = _data(B, n, mnl, p, r, kind, 100)
    grp = _solved_group(d)
    try:
        res = grp.results()
        assert all(c == 1 for c in res["status_code"])
        g = _grads(d, 7)
        got = grp.adjoint(*g)
    finally:
        grp.close()
    assert got["P"].shape == (B, d["P"].shape[1], n, n)
    assert np.array_equal(got["P"], got["P"].transpose(0, 1, 3, 2))
    assert (got["r"][:, 0] == 0).all()
    want, cond = _oracle(d, res, g)
    worst = _check_oracle(got, want, cond)
    print("\nqcqp adjoint B=%d n=%d mnl=%d p=%d %s: largest relative difference %.1e, cond(M) up to %.1e"
          % (B, n, mnl, p, kind, worst, cond.max()))


def _loss(res, g):
    z = np.concatenate([np.array(res["znl"]).ravel(), np.array(res["zl"]).ravel()])
    return float(g[0] @ np.array(res["x"]).ravel() + g[1] @ np.array(res["y"]).ravel() + g[2] @ z)


# seeds whose reference solution has a strict-complementarity margin min max(s, z) of at least 2e-2, over the
# quadratic and the linear rows, so that no row changes from active to inactive within the perturbation; each has a
# quadratic constraint active, and the linear seeds two, so the terms through uznl carry the P_i, q_i and r_i gradients.
# At 1e-10 s / z spans 1e-15..1e15 and the reduced KKT matrix is conditioned badly enough that on other seeds of the
# family with that margin one refinement step leaves more than 1e-5 (quad 0: 4e-5, linear 3: 9e-5; DESIGN.md)
@pytest.mark.parametrize("kind,seed", [("quad", 7), ("quad", 8), ("quad", 13), ("linear", 0), ("linear", 1),
                                       ("linear", 15)])
def test_adjoint_matches_central_differences_of_cp(ref, kind, seed):
    from cvxopt import matrix, solvers
    n, mnl, p, r = 8, 2, 2, 3
    d = _data(1, n, mnl, p, r, kind, 7000 + seed)
    tight = dict(abstol=1e-10, reltol=1e-10, feastol=1e-10, show_progress=False)

    def cp(dd):
        kw = dict(G=matrix(dd["G"][0]), h=matrix(dd["h"][0]), A=matrix(dd["A"][0]), b=matrix(dd["b"][0]))
        res = solvers.cp(ref_F(dd, 0), options=tight, **kw)
        assert res["status"] == "optimal"
        return res
    base = cp(d)
    s = np.concatenate([np.array(base[k]).ravel() for k in ("snl", "sl")])
    z = np.concatenate([np.array(base[k]).ravel() for k in ("znl", "zl")])
    assert np.maximum(s, z).min() > 2e-2, "no strict complementarity: the active set could change"
    assert np.array(base["znl"]).max() > 2e-2, "no quadratic constraint is active"
    grp = _solved_group(d, nsub=1, abstol=1e-10, reltol=1e-10, feastol=1e-10)
    try:
        assert grp.results()["status_code"][0] == 1
        g = _grads(d, 50 + seed)
        grad = grp.adjoint(*g)
    finally:
        grp.close()
    rng = np.random.default_rng(60 + seed)
    S = rng.standard_normal((mnl + 1, n, n))
    dirs = {"P": S + S.transpose(0, 2, 1), "q": rng.standard_normal((mnl + 1, n)), "r": rng.standard_normal(mnl + 1),
            "G": rng.standard_normal((2 * n + r, n)), "h": rng.standard_normal(2 * n + r),
            "A": rng.standard_normal((p, n)), "b": rng.standard_normal(p)}
    eps = 1e-5

    def moved(sign):
        dd = {k: v.copy() for k, v in d.items()}
        for k in KEYS:
            # P: the symmetric matrices plus the symmetric step, lower triangles as the batch reads them
            dd[k][0] = (sym(d[k][0]) if k == "P" else d[k][0]) + sign * eps * dirs[k]
        return dd
    gl = [gi[0] for gi in g]
    fd = (_loss(cp(moved(1)), gl) - _loss(cp(moved(-1)), gl)) / (2 * eps)
    an = sum(float(np.sum(grad[k][0] * dirs[k])) for k in KEYS)
    assert abs(fd - an) <= 1e-5 * max(abs(fd), abs(an)), (fd, an)


def test_adjoint_nan_for_problems_that_are_not_optimal():
    d = _data(12, 16, 3, 2, 4, "quad", 300)
    g = _grads(d, 11)
    grp = _solved_group(d, nsub=1)
    try:
        full = grp.adjoint(*g)
        its = grp.results()["iterations"]
    finally:
        grp.close()
    assert its.min() < its.max()
    cut = int(its.min() + its.max()) // 2
    grp = _solved_group(d, nsub=1, maxiters=cut)
    try:
        res = grp.results()
        got = grp.adjoint(*g)
    finally:
        grp.close()
    ok = res["status_code"] == 1
    assert ok.any() and not ok.all()
    for k in KEYS:
        assert np.isnan(got[k][~ok]).all(), k
        assert np.isfinite(got[k][ok]).all(), k
        assert np.array_equal(got[k][ok], full[k][ok]), k


def _spread(seed=400):
    return _data(9, 20, 3, 3, 6, "quad", seed)


def test_adjoint_bit_identical_across_compaction_subbatches_and_noise(monkeypatch):
    d = _spread()
    g = _grads(d, 17)

    def run(nsub, dd=d):
        grp = _solved_group(dd, nsub=nsub)
        try:
            return grp.results(), grp.adjoint(*g)
        finally:
            grp.close()
    r1, a1 = run(1)
    assert len(set(r1["iterations"].tolist())) > 1
    monkeypatch.setenv("CVXB_BATCH_COMPACT", "0")
    r0, a0 = run(1)
    monkeypatch.delenv("CVXB_BATCH_COMPACT")
    noisy = dict(d)
    noisy["P"] = np.tril(d["P"]) + np.triu(np.random.default_rng(3).standard_normal(d["P"].shape), 1)
    rn, an = run(1, noisy)
    for k in KEYS:
        assert np.array_equal(a0[k], a1[k]), k
        assert np.array_equal(an[k], a1[k]), k
    r2, a2 = run(2)
    r4, a4 = run(4)
    # a problem whose results differ between the two splits ran alone at the end of a sub-batch
    same = [j for j in range(9) if all(np.array_equal(r2[k][j], r4[k][j]) for k in ("x", "y", "s", "z"))]
    assert len(same) >= 9 // 2
    for k in KEYS:
        assert np.array_equal(a2[k][same], a4[k][same]), k


def test_adjoint_spaces_repeats_results_and_resolve():
    import torch
    from cvxopt_b200 import QCQPBatch
    d = _spread(seed=500)
    B, n, mnl, ml, p = _dims(d)
    nK, m = mnl + 1, mnl + ml
    g = _grads(d, 19)
    qb = QCQPBatch(B, n, mnl, ml, p, 0)
    try:
        qb.load(d["P"], d["q"], d["r"], d["x0"], d["G"], d["h"], d["A"], d["b"])
        qb.solve()
        r0 = qb.results()
        host = qb.adjoint(*g)
        again = qb.adjoint(*g)
        dev = torch.device("cuda", 0)
        gd = [torch.from_numpy(a).to(dev) for a in g]
        outs = [torch.full(s, 7.0, dtype=torch.float64, device=dev)
                for s in ((B, n), (B, p), (B, m), (B, n, nK, n), (B, nK, n), (B, nK), (B, n, ml), (B, n, p))]
        torch.cuda.synchronize()
        qb.adjoint_ptr(*(t.data_ptr() for t in gd), *(t.data_ptr() for t in outs))
        o = [t.cpu().numpy() for t in outs]
        on_dev = {"b": o[1], "h": o[2][:, mnl:], "P": o[3].transpose(0, 2, 3, 1), "q": o[4], "r": o[5],
                  "G": o[6].transpose(0, 2, 1), "A": o[7].transpose(0, 2, 1)}
        r1 = qb.results()
        qb.solve()
        r2 = qb.results()
    finally:
        qb.close()
    assert np.array_equal(o[4][:, 0], -o[0])                  # dq_0 = -ux
    for k in KEYS:
        assert np.array_equal(host[k], again[k]), k
        assert np.array_equal(host[k], on_dev[k]), k
    for k in ("x", "y", "s", "z", "iterations", "status_code", "primal objective"):
        assert np.array_equal(r0[k], r1[k]), k
        assert np.array_equal(r0[k], r2[k]), k


def test_adjoint_call_contract():
    import cvxopt_b200
    import torch
    from cvxopt_b200 import QCQPBatch, QPBatch, _lib
    d = _data(5, 12, 2, 2, 3, "quad", 600)
    B, n, mnl, ml, p = _dims(d)
    nK = mnl + 1
    g = _grads(d, 23)
    qb = QCQPBatch(B, n, mnl, ml, p, 0)
    try:
        with pytest.raises(ValueError, match="no completed"):
            qb.adjoint(*g)                          # never loaded
        qb.load(d["P"], d["q"], d["r"], d["x0"], d["G"], d["h"], d["A"], d["b"])
        with pytest.raises(ValueError, match="no completed"):
            qb.adjoint(*g)
        qb.solve()
        with pytest.raises(NotImplementedError, match="'l'"):
            QPBatch.adjoint_ptr(qb)                 # cvxb_batch_adjoint still refuses a QCQP batch
        full = qb.adjoint(*g)
        zero = qb.adjoint(g[0], np.zeros((B, p)), np.zeros((B, mnl + ml)))
        null = qb.adjoint(g[0])
        for k in KEYS:
            assert np.array_equal(zero[k], null[k]), k
        # only the requested outputs, equal to the full call's; nothing past their ends is written
        dev = torch.device("cuda", 0)
        gd = [torch.from_numpy(a).to(dev) for a in g]
        guard = 4096
        uz = torch.full((B * (mnl + ml) + guard,), 7.0, dtype=torch.float64, device=dev)
        dr = torch.full((B * nK + guard,), 7.0, dtype=torch.float64, device=dev)
        torch.cuda.synchronize()
        c0 = cvxopt_b200.launch_count()
        qb.adjoint_ptr(*(t.data_ptr() for t in gd), uz=uz.data_ptr(), dr=dr.data_ptr())
        c1 = cvxopt_b200.launch_count()
        qb.adjoint_ptr(*(t.data_ptr() for t in gd), uz=uz.data_ptr())
        c2 = cvxopt_b200.launch_count()
        qb.adjoint(*g)
        c3 = cvxopt_b200.launch_count()
        qb.adjoint(*g, want=("P",))
        c4 = cvxopt_b200.launch_count()
        assert c1 - c0 == (c2 - c1) + 1, "the gradient kernel runs only for a gradient output"
        assert c3 - c2 == c1 - c0 and c4 - c3 == c1 - c0
        print("\nqcqp adjoint launches (B=%d, n=%d, mnl=%d, p=%d): %d" % (B, n, mnl, p, c1 - c0))
        u, rr = uz.cpu().numpy(), dr.cpu().numpy()
        assert (u[B * (mnl + ml):] == 7.0).all() and (rr[B * nK:] == 7.0).all()
        assert np.array_equal(u[:B * (mnl + ml)].reshape(B, -1)[:, mnl:], full["h"])
        assert np.array_equal(rr[:B * nK].reshape(B, nK), full["r"])
        only = qb.adjoint(*g, want=("q",))
        assert set(only) == {"q"} and np.array_equal(only["q"], full["q"])
        # a new load (problem data, then A and b) needs a new solve
        qb.load(d["P"], d["q"], d["r"], d["x0"], d["G"], d["h"], d["A"], d["b"])
        with pytest.raises(ValueError, match="no completed"):
            qb.adjoint(*g)
        qb.solve()
        qb._load_eq(np.ascontiguousarray(d["A"].transpose(0, 2, 1)), d["b"], _lib.HOST)
        with pytest.raises(ValueError, match="no completed"):
            qb.adjoint(*g)
    finally:
        qb.close()


def _refused(batch):
    from cvxopt_b200 import QCQPBatch
    with pytest.raises(NotImplementedError, match="QCQP"):
        QCQPBatch.adjoint_ptr(batch)
    batch.close()


def test_adjoint_refuses_other_batches():
    from cvxopt_b200 import CPBatch, CPLBatch, ConeLPBatch, GPBatch, QPBatch, SDPBatch, SDPQPBatch
    _refused(QPBatch(3, 5, 7, 0))
    _refused(ConeLPBatch(3, 5, 8, 0))
    _refused(GPBatch(3, 5, [2, 3], 4))
    _refused(CPBatch(3, 5, 1, 4))
    _refused(CPLBatch(3, 5, 1, {"l": 4}))
    _refused(SDPBatch(3, 5, {"l": 4, "s": [3]}))
    _refused(SDPQPBatch(3, 5, {"l": 4, "s": [3]}))


def _torch(d, keys, dev=None):
    import torch
    dev = dev or torch.device("cuda", 0)
    return [torch.from_numpy(np.ascontiguousarray(d[k])).to(dev) for k in keys]


def test_qcqp_layer_backward_equals_group_adjoint():
    import torch
    from cvxopt_b200 import qcqp_layer
    d = _data(24, 12, 3, 2, 4, "quad", 700)
    B, n, mnl, ml, p = _dims(d)
    g = _grads(d, 29)
    t = [x.requires_grad_() for x in _torch(d, KEYS)]
    x, y, znl, zl, status = qcqp_layer(*t, nsub=3)
    grp = _solved_group(d, nsub=3)
    try:
        res = grp.results()
        want = grp.adjoint(*g)
    finally:
        grp.close()
    assert np.array_equal(status.cpu().numpy(), res["status_code"])
    for k, v in (("x", x), ("y", y)):
        assert np.array_equal(v.detach().cpu().numpy(), res[k]), k
    assert np.array_equal(torch.cat([znl, zl], 1).detach().cpu().numpy(), res["z"])
    gx, gy, gz = (torch.from_numpy(a).cuda() for a in g)
    loss = (x * gx).sum() + (y * gy).sum() + (znl * gz[:, :mnl]).sum() + (zl * gz[:, mnl:]).sum()
    grads = torch.autograd.grad(loss, t)
    for k, v in zip(KEYS, grads):
        assert np.array_equal(v.cpu().numpy(), want[k]), k


def test_qcqp_layer_through_factored_and_expanded_inputs():
    import torch
    from cvxopt_b200 import qcqp_layer
    d = _data(6, 10, 2, 0, 4, "quad", 800)
    B, n, mnl, ml, p = _dims(d)
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(31)
    S = torch.from_numpy(rng.standard_normal((B, mnl + 1, n, n)) / np.sqrt(n)).to(dev).requires_grad_()
    q0 = torch.from_numpy(d["q"][0]).to(dev).requires_grad_()
    r0 = torch.from_numpy(d["r"][0] - 3.0).to(dev).requires_grad_()
    Gt, ht = _torch(d, ("G", "h"))
    P = S @ S.transpose(2, 3) + 0.1 * torch.eye(n, dtype=torch.float64, device=dev)
    x, y, znl, zl, status = qcqp_layer(P, q0.expand(B, mnl + 1, n), r0.expand(B, mnl + 1), Gt, ht)
    assert (status == 1).all()
    gx = torch.from_numpy(rng.standard_normal((B, n))).to(dev)
    gzn = torch.from_numpy(rng.standard_normal((B, mnl))).to(dev)
    gS, gq0, gr0 = torch.autograd.grad((x * gx).sum() + (znl * gzn).sum(), (S, q0, r0))
    dd = dict(d, P=P.detach().cpu().numpy(), q=np.broadcast_to(q0.detach().cpu().numpy(), (B, mnl + 1, n)).copy(),
              r=np.broadcast_to(r0.detach().cpu().numpy(), (B, mnl + 1)).copy())
    grp = _solved_group(dd, nsub=1)
    try:
        want = grp.adjoint(gx.cpu().numpy(), None, np.hstack([gzn.cpu().numpy(), np.zeros((B, ml))]),
                           want=("P", "q", "r"))
    finally:
        grp.close()
    Sn = S.detach().cpu().numpy()
    assert np.allclose(gS.cpu().numpy(), 2 * want["P"] @ Sn, rtol=1e-10, atol=1e-13)
    assert np.allclose(gq0.cpu().numpy(), want["q"].sum(axis=0), rtol=1e-10, atol=1e-13)
    assert np.allclose(gr0.cpu().numpy(), want["r"].sum(axis=0), rtol=1e-10, atol=1e-13)


def test_qcqp_layer_work_streams_and_memory():
    import cvxopt_b200
    import torch
    from cvxopt_b200 import _lib, qcqp_layer
    d = _data(12, 10, 2, 2, 3, "quad", 900)
    B, n, mnl, ml, p = _dims(d)
    g = [torch.from_numpy(a).cuda() for a in _grads(d, 37)]
    lib = _lib.load()
    before = lib.cvxb_device_bytes()

    def run(needs, stream=None):
        with torch.cuda.stream(stream):                  # None: torch's current stream
            t = _torch(d, KEYS)
            for x, need in zip(t, needs):
                x.requires_grad_(need)
            x, y, znl, zl, _ = qcqp_layer(*t, nsub=1)
            c0 = cvxopt_b200.launch_count()
            grads = torch.autograd.grad((x * g[0]).sum() + (y * g[1]).sum() + (znl * g[2][:, :mnl]).sum() +
                                        (zl * g[2][:, mnl:]).sum(), [a for a, need in zip(t, needs) if need])
            torch.cuda.synchronize()
        return grads, cvxopt_b200.launch_count() - c0
    full, c_full = run([True] * 7)
    assert lib.cvxb_device_bytes() == before
    vec, c_vec = run([False, False, False, False, True, False, True])
    assert c_vec == c_full - 1, "no gradient output, no gradient kernel"
    for a, b in zip(vec, (full[4], full[6])):
        assert torch.equal(a, b)
    side = torch.cuda.Stream()
    on_side, _ = run([True] * 7, side)
    for a, b in zip(on_side, full):
        assert torch.equal(a, b)
    # inputs without requires_grad: nothing is kept for backward, nothing stays on the device
    t = _torch(d, KEYS)
    x, *_ = qcqp_layer(*t, nsub=1)
    assert not x.requires_grad
    assert lib.cvxb_device_bytes() == before
