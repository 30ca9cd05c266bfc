"""The QP batch's adjoint (cvxb_batch_adjoint, QPBatch.adjoint, qp_layer) on the device: parity with a dense numpy
solve of the KKT matrix at the batch's own returned iterate, central differences of the reference's coneqp, the NaN
policy, the S + A'A switch, bit-identity across compaction, sub-batches, spaces and repeated calls, the call contract
and the torch layer."""

import numpy as np
import pytest

from test_batch_eq_gpu import _switch_batch, eq_batch

pytestmark = pytest.mark.gpu

KEYS = ("P", "q", "G", "h", "A", "b")


def _batch(B, n, m, p, seed):
    return eq_batch(B, n, {"l": m}, p, seed)


def _grads(B, n, p, m, seed):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((B, n)), rng.standard_normal((B, p)), rng.standard_normal((B, m))


def _oracle(data, res, g):
    """per problem: M = [P A' G'; A 0 0; G 0 -diag(s / z)] at the returned iterate, u = M^{-1} g, the formulas of
    include/cvxopt_b200.h, and cond(M)"""
    P, q, G, h, A, b = data
    x, y, s, z = (res[k] for k in ("x", "y", "s", "z"))
    B, n = x.shape
    m, p = s.shape[1], y.shape[1]
    out = {k: [] for k in KEYS}
    cond = []
    for j in range(B):
        M = np.zeros((n + p + m, n + p + m))
        M[:n, :n] = P[j]
        M[n:n + p, :n] = A[j]
        M[:n, n:n + p] = A[j].T
        M[n + p:, :n] = G[j]
        M[:n, n + p:] = G[j].T
        M[n + p:, n + p:] = -np.diag(s[j] / z[j])
        D = 1.0 / np.sqrt(np.abs(M).max(axis=1))         # equilibrated: the oracle's own error stays near u
        u = D * np.linalg.solve(D[:, None] * M * D, D * np.concatenate([g[0][j], g[1][j], g[2][j]]))
        ux, uy, uz = u[:n], u[n:n + p], u[n + p:]
        out["q"].append(-ux)
        out["b"].append(uy)
        out["h"].append(uz)
        out["P"].append(-0.5 * (np.outer(ux, x[j]) + np.outer(x[j], ux)))
        out["G"].append(-(np.outer(z[j], ux) + np.outer(uz, x[j])))
        out["A"].append(-(np.outer(y[j], ux) + np.outer(uy, x[j])))
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
            d = _rel(got[k][j], want[k][j])
            assert d <= tol, (j, k, d, cond[j])
            worst = max(worst, d)
    return worst


def _solved_group(data, nsub=None, **options):
    from cvxopt_b200 import QPBatchGroup
    P, q, G, h, A, b = data
    B, n, m, p = P.shape[0], P.shape[1], G.shape[1], A.shape[1]
    grp = QPBatchGroup(B, n, m, 0, nsub, p=p)
    grp.load(*data)
    grp.solve(**options)
    return grp


@pytest.mark.parametrize("B,n,m,p", [(1, 12, 30, 0), (7, 12, 30, 0), (33, 40, 80, 5), (257, 64, 128, 8)])
def test_adjoint_matches_dense_kkt_solve(B, n, m, p):
    data = _batch(B, n, m, p, 1000 * B + n)
    grp = _solved_group(data)
    try:
        res = grp.results()
        assert all(c == 1 for c in res["status_code"])
        g = _grads(B, n, p, m, 7)
        got = grp.adjoint(*g)
    finally:
        grp.close()
    want, cond = _oracle(data, res, g)
    assert np.array_equal(got["P"], got["P"].transpose(0, 2, 1))
    worst = _check_oracle(got, want, cond)
    print("\nadjoint B=%d n=%d m=%d p=%d: largest relative difference %.1e, cond(M) up to %.1e"
          % (B, n, m, p, worst, cond.max()))


def _loss(res, g):
    return sum(float(gi @ np.array(res[k]).ravel()) for gi, k in zip(g, ("x", "y", "z")))


# seeds whose reference solution has a strict-complementarity margin min max(s, z) of at least 2e-2.  At a smaller
# margin the two effects of a converged iterate meet: s / z of a weakly active row stays far from 0 or infinity at the
# default tolerances (seed 3, margin 2.7e-3: 1e-4 even in exact arithmetic), and at 1e-10 the reduced KKT matrix is
# conditioned badly enough that one refinement step leaves 6.5e-5 (seed 2, margin 8e-3)
@pytest.mark.parametrize("seed", [0, 1, 4, 5, 7])
def test_adjoint_matches_central_differences_of_coneqp(ref, seed):
    from cvxopt import matrix, solvers
    n, m, p = 12, 20, 3
    data = _batch(1, n, m, p, 4000 + seed)
    P, q, G, h, A, b = (a[0] for a in data)
    tight = dict(abstol=1e-10, reltol=1e-10, feastol=1e-10, show_progress=False)

    def coneqp(P, q, G, h, A, b):
        r = solvers.coneqp(matrix(P), matrix(q), matrix(G), matrix(h), None, matrix(A), matrix(b), options=tight)
        assert r["status"] == "optimal"
        return r
    base = coneqp(P, q, G, h, A, b)
    s, z = np.array(base["s"]).ravel(), np.array(base["z"]).ravel()
    assert np.maximum(s, z).min() > 2e-2, "no strict complementarity: the active set could change"
    # the batch at the same tolerances: at the default ones s / z of the returned iterate moves the derivative by
    # up to 2e-4 on these seeds
    grp = _solved_group(data, nsub=1, abstol=1e-10, reltol=1e-10, feastol=1e-10)
    try:
        assert grp.results()["status_code"][0] == 1
        g = _grads(1, n, p, m, 50 + seed)
        grad = grp.adjoint(*g)
    finally:
        grp.close()
    rng = np.random.default_rng(60 + seed)
    S = rng.standard_normal((n, n))
    d = {"P": S + S.T, "q": rng.standard_normal(n), "G": rng.standard_normal((m, n)), "h": rng.standard_normal(m),
         "A": rng.standard_normal((p, n)), "b": rng.standard_normal(p)}
    eps = 1e-5
    cur = dict(P=P, q=q, G=G, h=h, A=A, b=b)
    Lp = _loss(coneqp(**{k: cur[k] + eps * d[k] for k in KEYS}), [gi[0] for gi in g])
    Lm = _loss(coneqp(**{k: cur[k] - eps * d[k] for k in KEYS}), [gi[0] for gi in g])
    fd = (Lp - Lm) / (2 * eps)
    an = sum(float(np.sum(grad[k][0] * d[k])) for k in KEYS)
    assert abs(fd - an) <= 1e-5 * max(abs(fd), abs(an)), (fd, an)


def test_adjoint_nan_for_problems_that_are_not_optimal():
    B, n, m, p = 9, 30, 60, 4
    data = _batch(B, n, m, p, 5000)
    data[1] *= np.linspace(0.1, 30.0, B)[:, None]
    g = _grads(B, n, p, m, 11)
    grp = _solved_group(data, nsub=1)
    try:
        full = grp.adjoint(*g)
        its = grp.results()["iterations"]
    finally:
        grp.close()
    assert its.min() < its.max()
    cut = int(its.min() + its.max()) // 2
    grp = _solved_group(data, nsub=1, maxiters=cut)
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
        assert np.allclose(got[k][ok], full[k][ok], rtol=1e-12, atol=0), k
    want, cond = _oracle(data, res, g)
    _check_oracle(got, want, cond, rows=np.flatnonzero(ok))


def test_adjoint_with_the_s_plus_ata_switch():
    data, dims = _switch_batch()
    grp = _solved_group(data, nsub=1)
    try:
        res = grp.results()
        g = _grads(4, 64, 16, dims["l"], 13)
        got = grp.adjoint(*g)
    finally:
        grp.close()
    want, cond = _oracle(data, res, g)
    _check_oracle(got, want, cond)


def _spread(B=9, n=40, m=80, p=6, seed=5500):
    data = _batch(B, n, m, p, seed)
    data[1] *= np.linspace(0.1, 30.0, B)[:, None]
    return data


def test_adjoint_bit_identical_across_compaction_and_subbatches(monkeypatch):
    data = _spread()
    B, n, m, p = 9, 40, 80, 6
    g = _grads(B, n, p, m, 17)

    def run(nsub):
        grp = _solved_group(data, nsub=nsub)
        try:
            return grp.results(), grp.adjoint(*g)
        finally:
            grp.close()
    r1, a1 = run(1)
    assert len(set(r1["iterations"].tolist())) > 1
    monkeypatch.setenv("CVXB_BATCH_COMPACT", "0")
    r0, a0 = run(1)
    monkeypatch.delenv("CVXB_BATCH_COMPACT")
    for k in KEYS:
        assert np.array_equal(a0[k], a1[k]), k
    r2, a2 = run(2)
    r4, a4 = run(4)
    # a problem whose results differ between the two splits ran alone at the end of a sub-batch
    same = [j for j in range(B) if all(np.array_equal(r2[k][j], r4[k][j]) for k in ("x", "y", "s", "z"))]
    assert len(same) >= B // 2
    for k in KEYS:
        assert np.array_equal(a2[k][same], a4[k][same]), k


def test_adjoint_spaces_repeats_results_and_resolve():
    import torch
    from cvxopt_b200 import QPBatch
    data = _spread(seed=5600)
    P, q, G, h, A, b = data
    B, n, m, p = 9, 40, 80, 6
    g = _grads(B, n, p, m, 19)
    qb = QPBatch(B, n, m, 0, p=p)
    try:
        qb.load(*data)
        qb.solve()
        r0 = qb.results()
        host = qb.adjoint(*g)
        again = qb.adjoint(*g)
        dev = torch.device("cuda", 0)
        gd = [torch.from_numpy(a).to(dev) for a in g]
        outs = [torch.full(s, 7.0, dtype=torch.float64, device=dev)
                for s in ((B, n), (B, p), (B, m), (B, n, n), (B, n, m), (B, n, p))]
        torch.cuda.synchronize()
        qb.adjoint_ptr(*(t.data_ptr() for t in gd), *(t.data_ptr() for t in outs))
        o = [t.cpu().numpy() for t in outs]
        on_dev = {"q": -o[0], "b": o[1], "h": o[2], "P": o[3].transpose(0, 2, 1), "G": o[4].transpose(0, 2, 1),
                  "A": o[5].transpose(0, 2, 1)}
        r1 = qb.results()
        qb.solve()
        r2 = qb.results()
    finally:
        qb.close()
    for k in KEYS:
        assert np.array_equal(host[k], again[k]), k
        assert np.array_equal(host[k], on_dev[k]), k
    for k in ("x", "y", "s", "z", "iterations", "status_code", "primal objective"):
        assert np.array_equal(r0[k], r1[k]), k
        assert np.array_equal(r0[k], r2[k]), k


def test_adjoint_call_contract():
    import cvxopt_b200
    import torch
    from cvxopt_b200 import QPBatch, _lib
    B, n, m, p = 5, 20, 40, 3
    data = _batch(B, n, m, p, 5700)
    g = _grads(B, n, p, m, 23)
    qb = QPBatch(B, n, m, 0, p=p)
    try:
        with pytest.raises(ValueError, match="no completed"):
            qb.adjoint(*g)                          # loaded, never solved
        qb.load(*data)
        with pytest.raises(ValueError, match="no completed"):
            qb.adjoint(*g)
        qb.solve()
        full = qb.adjoint(*g)
        # NULL gy and gz are zero
        zero = qb.adjoint(g[0], np.zeros((B, p)), np.zeros((B, m)))
        null = qb.adjoint(g[0])
        for k in KEYS:
            assert np.array_equal(zero[k], null[k]), k
        # only the requested outputs, equal to the full call's; nothing past their ends is written
        dev = torch.device("cuda", 0)
        gd = [torch.from_numpy(a).to(dev) for a in g]
        guard = 4096
        ux = torch.full((B * n + guard,), 7.0, dtype=torch.float64, device=dev)
        dG = torch.full((B * m * n + guard,), 7.0, dtype=torch.float64, device=dev)
        torch.cuda.synchronize()
        c0 = cvxopt_b200.launch_count()
        qb.adjoint_ptr(*(t.data_ptr() for t in gd), ux=ux.data_ptr(), dG=dG.data_ptr())
        c1 = cvxopt_b200.launch_count()
        qb.adjoint_ptr(*(t.data_ptr() for t in gd), ux=ux.data_ptr())
        c2 = cvxopt_b200.launch_count()
        qb.adjoint(*g)
        c3 = cvxopt_b200.launch_count()
        qb.adjoint(*g)
        c4 = cvxopt_b200.launch_count()
        assert c1 - c0 == (c2 - c1) + 1, "the gradient kernel runs only for a matrix output"
        assert c3 - c2 == c1 - c0 and c4 - c3 == c1 - c0
        print("\nadjoint launches (B=%d, n=%d, p=%d): %d" % (B, n, p, c1 - c0))
        u, dg = ux.cpu().numpy(), dG.cpu().numpy()
        assert (u[B * n:] == 7.0).all() and (dg[B * m * n:] == 7.0).all()
        assert np.array_equal(-u[:B * n].reshape(B, n), full["q"])
        assert np.array_equal(dg[:B * m * n].reshape(B, n, m).transpose(0, 2, 1), full["G"])
        only = qb.adjoint(*g, want=("h",))
        assert set(only) == {"h"} and np.array_equal(only["h"], full["h"])
        # a new load (problem data, then A and b) needs a new solve
        qb.load(*data)
        with pytest.raises(ValueError, match="no completed"):
            qb.adjoint(*g)
        qb.solve()
        qb._load_eq(*(np.ascontiguousarray(data[4].transpose(0, 2, 1)), data[5]), _lib.HOST)
        with pytest.raises(ValueError, match="no completed"):
            qb.adjoint(*g)
    finally:
        qb.close()


def _refused(batch):
    with pytest.raises(NotImplementedError, match="'l'"):
        batch.adjoint_ptr()
    batch.close()


def test_adjoint_refuses_other_batches():
    from cvxopt_b200 import CPBatch, ConeLPBatch, GPBatch, QPBatch, SDPBatch, SDPQPBatch
    _refused(QPBatch(3, 5, 7, 0, dims={"l": 4, "q": [3]}))
    _refused(ConeLPBatch(3, 5, 8, 0))
    _refused(GPBatch(3, 5, [2, 3], 4))
    _refused(CPBatch(3, 5, 1, 4))
    _refused(SDPBatch(3, 5, {"l": 4, "s": [3]}))
    _refused(SDPQPBatch(3, 5, {"l": 4, "s": [3]}))


def _torch_data(data):
    import torch
    dev = torch.device("cuda", 0)
    return [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in data]


def test_qp_layer_backward_equals_group_adjoint():
    import torch
    from cvxopt_b200 import qp_layer
    B, n, m, p = 24, 16, 32, 4
    data = _batch(B, n, m, p, 5800)
    g = _grads(B, n, p, m, 29)
    t = [x.requires_grad_() for x in _torch_data(data)]
    x, y, z, status = qp_layer(*t, nsub=3)
    grp = _solved_group(data, nsub=3)
    try:
        res = grp.results()
        want = grp.adjoint(*g)
    finally:
        grp.close()
    assert np.array_equal(status.cpu().numpy(), res["status_code"])
    for k, v in (("x", x), ("y", y), ("z", z)):
        assert np.array_equal(v.detach().cpu().numpy(), res[k]), k
    gt = _torch_data(g)
    grads = torch.autograd.grad((x * gt[0]).sum() + (y * gt[1]).sum() + (z * gt[2]).sum(), t)
    for k, v in zip(KEYS, grads):
        assert np.allclose(v.cpu().numpy(), want[k], rtol=1e-12, atol=1e-14), k


def test_qp_layer_through_symmetric_and_expanded_inputs():
    import torch
    from cvxopt_b200 import qp_layer
    B, n, m = 6, 10, 24
    P, q, G, h, A, b = _batch(B, n, m, 0, 5900)
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(31)
    R = rng.standard_normal((B, n, n))
    S = torch.from_numpy(P / 2 + R - R.transpose(0, 2, 1)).to(dev).requires_grad_()     # not symmetric; S + S' = P
    q0 = torch.from_numpy(rng.standard_normal(n)).to(dev).requires_grad_()
    Gt, ht = (torch.from_numpy(a).to(dev) for a in (G, h))
    x, y, z, status = qp_layer(S + S.transpose(1, 2), q0.expand(B, n), Gt, ht)
    assert (status == 1).all()
    gx = torch.from_numpy(rng.standard_normal((B, n))).to(dev)
    gS, gq0 = torch.autograd.grad((x * gx).sum(), (S, q0))
    Pn = (S + S.transpose(1, 2)).detach().cpu().numpy()
    qn = np.broadcast_to(q0.detach().cpu().numpy(), (B, n))
    grp = _solved_group((Pn, qn, G, h, np.zeros((B, 0, n)), np.zeros((B, 0))), nsub=1)
    try:
        want = grp.adjoint(gx.cpu().numpy(), want=("P", "q"))
    finally:
        grp.close()
    assert np.allclose(gS.cpu().numpy(), want["P"] + want["P"].transpose(0, 2, 1), rtol=1e-10, atol=1e-13)
    assert np.allclose(gq0.cpu().numpy(), want["q"].sum(axis=0), rtol=1e-10, atol=1e-13)


def test_qp_layer_work_streams_and_memory():
    import cvxopt_b200
    import torch
    from cvxopt_b200 import _lib, qp_layer
    B, n, m, p = 12, 14, 28, 3
    data = _batch(B, n, m, p, 6000)
    g = _torch_data(_grads(B, n, p, m, 37))
    lib = _lib.load()
    before = lib.cvxb_device_bytes()

    def run(needs, stream=None):
        with torch.cuda.stream(stream):                  # None: torch's current stream
            t = _torch_data(data)
            for x, need in zip(t, needs):
                x.requires_grad_(need)
            x, y, z, _ = qp_layer(*t, nsub=1)
            c0 = cvxopt_b200.launch_count()
            grads = torch.autograd.grad((x * g[0]).sum() + (y * g[1]).sum() + (z * g[2]).sum(),
                                        [a for a, need in zip(t, needs) if need])
            torch.cuda.synchronize()
        return grads, cvxopt_b200.launch_count() - c0
    full, c_full = run([True] * 6)
    assert lib.cvxb_device_bytes() == before
    vec, c_vec = run([False, True, False, True, False, True])
    assert c_vec == c_full - 1, "no matrix output, no gradient kernel"
    for a, b in zip(vec, (full[1], full[3], full[5])):
        assert torch.equal(a, b)
    side = torch.cuda.Stream()
    on_side, _ = run([True] * 6, side)
    for a, b in zip(on_side, full):
        assert torch.equal(a, b)
    assert lib.cvxb_device_bytes() == before
