"""The GP batch's adjoint (cvxb_batch_adjoint_gp, GPBatch.adjoint_gp, gp_layer) on the device, on tests/gp_problems.py's
family: parity with a dense numpy solve of the KKT matrix at the batch's own returned iterate, central differences of
the reference's solvers.gp, monomial rows against the same rows in G, the NaN policy, bit-identity across compaction,
sub-batches, spaces and repeated calls, the call contract and the torch layer."""

import numpy as np
import pytest

from gp_problems import gp_batch_data, gp_problem

pytestmark = pytest.mark.gpu

KEYS = ("F", "g", "G", "h", "A", "b")


def _data(B, n, K, r, p, seed):
    return dict(zip(KEYS, gp_batch_data(range(seed, seed + B), n, K, r, p)))


def _solved_group(K, d, nsub=None, **options):
    from cvxopt_b200 import GPBatchGroup
    B, S, n = d["F"].shape
    ml, p = d["G"].shape[1], d["A"].shape[1]
    grp = GPBatchGroup(B, n, K, ml, p, 0, nsub)
    grp.load(d["F"], d["g"], d["G"], d["h"], d["A"] if p else None, d["b"] if p else None)
    grp.solve(**options)
    return grp


def _grads(K, d, seed):
    B, S, n = d["F"].shape
    rng = np.random.default_rng(seed)
    return (rng.standard_normal((B, n)), rng.standard_normal((B, d["A"].shape[1])),
            rng.standard_normal((B, len(K) - 1 + d["G"].shape[1])))


def _oracle(K, d, res, g):
    """per problem, at the returned iterate with z_0 = 1: pi_i = softmax(F_i x + g_i), H = sum z_i F_i' Sigma_i F_i,
    Df's rows pi_i' F_i, M = [H A' Df' G'; A 0 0 0; Df 0 -Dnl 0; G 0 0 -Dl] with D = diag(s / z), u = M^{-1} g
    (equilibrated), the formulas of include/cvxopt_b200.h, and cond(M)"""
    B, S, n = d["F"].shape
    mnl, p = len(K) - 1, d["A"].shape[1]
    off = np.concatenate([[0], np.cumsum(K)])
    out = {k: [] for k in KEYS}
    cond = []
    for j in range(B):
        F, gv, G, A = d["F"][j], d["g"][j], d["G"][j], d["A"][j]
        x, y, s, z = (np.asarray(res[k][j]) for k in ("x", "y", "s", "z"))
        zk = np.concatenate([[1.0], z[:mnl]])
        H = np.zeros((n, n))
        pis, Df = [], []
        for i in range(mnl + 1):
            Fi = F[off[i]:off[i + 1]]
            u = Fi @ x + gv[off[i]:off[i + 1]]
            pi = np.exp(u - u.max())
            pi /= pi.sum()
            pis.append(pi)
            H += zk[i] * Fi.T @ (np.diag(pi) - np.outer(pi, pi)) @ Fi
            if i:
                Df.append(pi @ Fi)
        Gf = np.vstack(Df + [G])
        m = Gf.shape[0]
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
        uk = np.concatenate([[0.0], uz[:mnl]])
        dg, dF = np.zeros(S), np.zeros((S, n))
        for i in range(mnl + 1):
            Fi, pi = F[off[i]:off[i + 1]], pis[i]
            w = Fi @ ux
            dgi = -(zk[i] * pi * (w - pi @ w) + uk[i] * pi)
            dg[off[i]:off[i + 1]] = dgi
            dF[off[i]:off[i + 1]] = np.outer(dgi, x) - zk[i] * np.outer(pi, ux)
        out["F"].append(dF)
        out["g"].append(dg)
        out["G"].append(-(np.outer(z[mnl:], ux) + np.outer(uz[mnl:], x)))
        out["h"].append(uz[mnl:])
        out["A"].append(-(np.outer(y, ux) + np.outer(uy, x)))
        out["b"].append(uy)
        cond.append(np.linalg.cond(M))
    return {k: np.array(v) for k, v in out.items()}, np.array(cond)


def _rel(a, b):
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


def _check_oracle(got, want, cond, rows=None):
    """every output within max(1e-9, 10 u cond(M)) relative of the oracle, per problem (rows: those problems only);
    returns the largest relative difference"""
    worst = 0.0
    for j in range(len(cond)) if rows is None else rows:
        tol = max(1e-9, 10 * np.finfo(float).eps * cond[j])
        for k in got:
            if got[k][j].size == 0:
                continue
            dd = _rel(got[k][j], want[k][j])
            assert dd <= tol, (j, k, dd, cond[j])
            worst = max(worst, dd)
    return worst


def _switch_data(B, switch, p=3):
    """test_batch_gp_gpu's switch batch: n = 4, K = [1, 2], G = [I; -I], p rows of A.  Where `switch`, G keeps only its
    e1 rows and f1's two rows are equal and zero in the last two columns, so S is singular at the start and the solve
    factors S + A'A for those problems"""
    d = _data(B, 4, [1, 2], 0, p, 200)
    for k in switch:
        d["G"][k, [1, 2, 3, 5, 6, 7]] = 0.0
        d["F"][k, 2] = d["F"][k, 1]
        d["F"][k, 1:, 2:] = 0.0
        d["g"][k, 1:] = np.log(0.25)
    return d


SHAPES = [  # n, K, r, p, B, ml = 0
    (16, [32, 8, 8, 8], 4, 0, 12, False),
    (32, [64] + [8] * 8, 8, 2, 16, False),      # p > 0
    (6, [32, 6, 6], 0, 0, 10, True),            # ml = 0
    (16, [32, 1, 8, 1], 4, 2, 9, False),        # monomial blocks among posynomials
    (32, [64] + [8] * 8, 8, 2, 1, False),       # B = 1: gp_hessian's split-K workspace
    (16, [32, 8, 8, 8], 4, 0, 257, False),      # several sub-batches, compaction
]


@pytest.mark.parametrize("n,K,r,p,B,noG", SHAPES)
def test_adjoint_matches_dense_kkt_solve(n, K, r, p, B, noG):
    d = _data(B, n, K, r, p, 100)
    if noG:
        d["G"], d["h"] = d["G"][:, :0], d["h"][:, :0]
    grp = _solved_group(K, d)
    try:
        res = grp.results()
        assert all(c == 1 for c in res["status_code"])
        g = _grads(K, d, 7)
        got = grp.adjoint_gp(*g)
    finally:
        grp.close()
    assert got["F"].shape == d["F"].shape and got["g"].shape == d["g"].shape
    assert got["G"].shape == d["G"].shape and got["h"].shape == d["h"].shape
    want, cond = _oracle(K, d, res, g)
    worst = _check_oracle(got, want, cond)
    print("\ngp adjoint B=%d n=%d K=%s p=%d: largest relative difference %.1e, cond(M) up to %.1e"
          % (B, n, K, p, worst, cond.max()))


def test_adjoint_matches_dense_kkt_solve_with_the_switch():
    """the switched problems 1 and 4 are optimal; 2 and 5 end unknown, as in the reference, and get NaN"""
    K = [1, 2]
    d = _switch_data(6, [1, 4])
    grp = _solved_group(K, d, nsub=1)
    try:
        res = grp.results()
        g = _grads(K, d, 9)
        got = grp.adjoint_gp(*g)
    finally:
        grp.close()
    ok = res["status_code"] == 1
    assert ok[[1, 4]].all()
    want, cond = _oracle(K, d, res, g)
    _check_oracle(got, want, cond, np.flatnonzero(ok))
    for k in KEYS:
        assert np.isnan(got[k][~ok]).all(), k


def test_adjoint_mirrors_h_without_refinement():
    """refinement 0 never mirrors H in the solve; the adjoint's refinement step multiplies by all of H"""
    K = [32, 8, 8, 8]
    d = _data(12, 16, K, 4, 2, 150)
    grp = _solved_group(K, d, nsub=1, refinement=0)
    try:
        res = grp.results()
        assert all(c == 1 for c in res["status_code"])
        g = _grads(K, d, 13)
        got = grp.adjoint_gp(*g)
    finally:
        grp.close()
    want, cond = _oracle(K, d, res, g)
    _check_oracle(got, want, cond)


def _loss(res, g):
    z = np.concatenate([np.array(res["znl"]).ravel(), np.array(res["zl"]).ravel()])
    return float(g[0] @ np.array(res["x"]).ravel() + g[1] @ np.array(res["y"]).ravel() + g[2] @ z)


def _m(v):
    from cvxopt import matrix
    return matrix(np.ascontiguousarray(v, dtype=np.float64))


# seeds whose reference solution has a strict-complementarity margin min max(s, z) of at least 0.1 over the
# posynomial and the linear rows, so that no row changes from active to inactive within the perturbation, and a
# posynomial constraint active (max znl >= 0.1), so the terms through uznl carry the F_i and g_i gradients.  At 1e-10
# s / z spans many orders of magnitude, and on three more seeds with such margins (12, 13, 14) one refinement step
# leaves the adjoint 2e-3, 1.5e-5 and 2.4e-5 from the central differences, though a dense solve at the reference's
# own solution agrees with them to 2e-9 there (DESIGN.md)
@pytest.mark.parametrize("seed", [1, 3, 4])
def test_adjoint_matches_central_differences_of_gp(ref, seed):
    from cvxopt import solvers
    n, K, r, p = 8, [6, 4, 4], 3, 2
    d = dict(zip(KEYS, (a[None] for a in gp_problem(7000 + seed, n, K, r, p))))
    tight = dict(abstol=1e-10, reltol=1e-10, feastol=1e-10, show_progress=False)

    def gp(dd):
        res = solvers.gp(list(K), *(_m(dd[k][0]) for k in KEYS), options=tight)
        assert res["status"] == "optimal"
        return res
    base = gp(d)
    s = np.concatenate([np.array(base[k]).ravel() for k in ("snl", "sl")])
    z = np.concatenate([np.array(base[k]).ravel() for k in ("znl", "zl")])
    assert np.maximum(s, z).min() > 0.1, "no strict complementarity: the active set could change"
    assert np.array(base["znl"]).max() > 0.1, "no posynomial constraint is active"
    grp = _solved_group(K, d, nsub=1, abstol=1e-10, reltol=1e-10, feastol=1e-10)
    try:
        assert grp.results()["status_code"][0] == 1
        g = _grads(K, d, 50 + seed)
        grad = grp.adjoint_gp(*g)
    finally:
        grp.close()
    rng = np.random.default_rng(60 + seed)
    dirs = {k: rng.standard_normal(d[k].shape[1:]) for k in KEYS}
    eps = 1e-5

    def moved(sign):
        return {k: d[k] + sign * eps * dirs[k][None] for k in KEYS}
    gl = [gi[0] for gi in g]
    fd = (_loss(gp(moved(1)), gl) - _loss(gp(moved(-1)), gl)) / (2 * eps)
    an = sum(float(np.sum(grad[k][0] * dirs[k])) for k in KEYS)
    assert abs(fd - an) <= 1e-5 * max(abs(fd), abs(an)), (fd, an)


def test_monomial_rows_match_the_same_rows_in_g():
    """K = [K0, 4, 1, 1] against K = [K0, 4] with the two monomial rows appended to G and h = -g: the same problem, so
    dF's monomial rows are dG's last rows and dg there is -dh, to 1e-6 relative at the default tolerances (at 1e-10
    the adjoint's own error, the one the central-difference seeds show, reaches 1e-4)"""
    n, K0, B = 8, 6, 8
    d = _data(B, n, [K0, 4], 3, 0, 7100)
    rng = np.random.default_rng(5)
    Fm = rng.standard_normal((B, 2, n))
    gm = np.log(np.full((B, 2), 0.5))
    dA = dict(d, F=np.concatenate([d["F"], Fm], 1), g=np.concatenate([d["g"], gm], 1))
    dB = dict(d, G=np.concatenate([d["G"], Fm], 1), h=np.concatenate([d["h"], -gm], 1))
    gx = rng.standard_normal((B, n))
    out = []
    for K, dd in (([K0, 4, 1, 1], dA), ([K0, 4], dB)):
        grp = _solved_group(K, dd, nsub=1)
        try:
            assert all(c == 1 for c in grp.results()["status_code"])
            out.append(grp.adjoint_gp(gx))
        finally:
            grp.close()
    a, b = out
    ml = d["G"].shape[1]
    diffs = (_rel(a["F"][:, K0 + 4:], b["G"][:, ml:]), _rel(a["g"][:, K0 + 4:], -b["h"][:, ml:]),
             _rel(a["G"], b["G"][:, :ml]), _rel(a["F"][:, :K0 + 4], b["F"]))
    print("\nmonomial rows in F against the same rows in G: relative differences %s" % ["%.1e" % v for v in diffs])
    assert max(diffs) <= 1e-6


def test_adjoint_nan_for_problems_that_are_not_optimal():
    K = [32, 8, 8, 8]
    d = _data(12, 16, K, 4, 2, 300)
    g = _grads(K, d, 11)
    grp = _solved_group(K, d, nsub=1)
    try:
        full = grp.adjoint_gp(*g)
        its = grp.results()["iterations"]
    finally:
        grp.close()
    assert its.min() < its.max()
    for cut in (1, int(its.min() + its.max()) // 2):
        grp = _solved_group(K, d, nsub=1, maxiters=cut)
        try:
            res = grp.results()
            got = grp.adjoint_gp(*g)
        finally:
            grp.close()
        ok = res["status_code"] == 1
        assert not ok.all() and (ok.any() or cut == 1)
        for k in KEYS:
            assert np.isnan(got[k][~ok]).all(), k
            assert np.isfinite(got[k][ok]).all(), k
            assert np.array_equal(got[k][ok], full[k][ok]), k


def test_adjoint_bit_identical_across_compaction_and_subbatches(monkeypatch):
    K = [32, 8, 8, 8]
    d = _data(9, 16, K, 4, 2, 400)
    g = _grads(K, d, 17)

    def run(nsub):
        grp = _solved_group(K, d, nsub=nsub)
        try:
            return grp.results(), grp.adjoint_gp(*g)
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
    same = [j for j in range(9) if all(np.array_equal(r2[k][j], r4[k][j]) for k in ("x", "y", "s", "z"))]
    assert len(same) >= 9 // 2
    for k in KEYS:
        assert np.array_equal(a2[k][same], a4[k][same]), k


def test_adjoint_spaces_repeats_results_and_resolve():
    import torch
    from cvxopt_b200 import GPBatch
    K = [32, 8, 8, 8]
    d = _data(9, 16, K, 4, 2, 500)
    B, S, n = d["F"].shape
    ml, p, mnl = d["G"].shape[1], d["A"].shape[1], len(K) - 1
    m = mnl + ml
    g = _grads(K, d, 19)
    gb = GPBatch(B, n, K, ml, p, 0)
    try:
        gb.load(*(d[k] for k in KEYS))
        gb.solve()
        r0 = gb.results()
        host = gb.adjoint_gp(*g)
        again = gb.adjoint_gp(*g)
        dev = torch.device("cuda", 0)
        gd = [torch.from_numpy(a).to(dev) for a in g]
        outs = [torch.full(s, 7.0, dtype=torch.float64, device=dev)
                for s in ((B, n), (B, p), (B, m), (B, n, S), (B, S), (B, n, ml), (B, n, p))]
        torch.cuda.synchronize()
        gb.adjoint_gp_ptr(*(t.data_ptr() for t in gd), *(t.data_ptr() for t in outs))
        o = [t.cpu().numpy() for t in outs]
        on_dev = {"b": o[1], "h": o[2][:, mnl:], "F": o[3].transpose(0, 2, 1), "g": o[4],
                  "G": o[5].transpose(0, 2, 1), "A": o[6].transpose(0, 2, 1)}
        r1 = gb.results()
        gb.solve()
        r2 = gb.results()
    finally:
        gb.close()
    for k in KEYS:
        assert np.array_equal(host[k], again[k]), k
        assert np.array_equal(host[k], on_dev[k]), k
    for k in ("x", "y", "s", "z", "iterations", "status_code", "primal objective", "dual objective"):
        assert np.array_equal(r0[k], r1[k]), k
        assert np.array_equal(r0[k], r2[k]), k


# launches of one adjoint call on the batch of test_adjoint_call_contract (5 problems, n = 12, K = [16, 4, 4],
# ml = 27, p = 2) with every output; without the matrix and dg outputs it saves the GEMV's two kernels, k_adj_gp_dg
# and k_adj_gp_grad
LAUNCHES = 46


def test_adjoint_call_contract():
    import cvxopt_b200
    import torch
    from cvxopt_b200 import GPBatch, QPBatch, QCQPBatch, _lib
    K = [16, 4, 4]
    d = _data(5, 12, K, 3, 2, 600)
    B, S, n = d["F"].shape
    ml, p, mnl = d["G"].shape[1], d["A"].shape[1], len(K) - 1
    g = _grads(K, d, 23)
    lib = _lib.load()
    before = lib.cvxb_device_bytes()
    gb = GPBatch(B, n, K, ml, p, 0)
    try:
        with pytest.raises(ValueError, match="no completed"):
            gb.adjoint_gp(*g)                       # never loaded
        gb.load(*(d[k] for k in KEYS))
        with pytest.raises(ValueError, match="no completed"):
            gb.adjoint_gp(*g)
        gb.solve()
        # the other adjoint entry points still refuse a GP batch
        with pytest.raises(NotImplementedError, match="'l'"):
            QPBatch.adjoint_ptr(gb)
        with pytest.raises(NotImplementedError, match="QP and cone LP"):
            QPBatch.adjoint_cone_ptr(gb)
        with pytest.raises(NotImplementedError, match="QCQP"):
            QCQPBatch.adjoint_ptr(gb)
        full = gb.adjoint_gp(*g)
        zero = gb.adjoint_gp(g[0], np.zeros((B, p)), np.zeros((B, mnl + ml)))
        null = gb.adjoint_gp(g[0])
        for k in KEYS:
            assert np.array_equal(zero[k], null[k]), k
        # only the requested outputs, equal to the full call's; nothing past their ends is written
        dev = torch.device("cuda", 0)
        gd = [torch.from_numpy(a).to(dev) for a in g]
        guard = 4096
        uz = torch.full((B * (mnl + ml) + guard,), 7.0, dtype=torch.float64, device=dev)
        dg = torch.full((B * S + guard,), 7.0, dtype=torch.float64, device=dev)
        dG = torch.full((B * n * ml + guard,), 7.0, dtype=torch.float64, device=dev)
        torch.cuda.synchronize()
        c0 = cvxopt_b200.launch_count()
        gb.adjoint_gp_ptr(*(t.data_ptr() for t in gd), uz=uz.data_ptr())
        c1 = cvxopt_b200.launch_count()
        gb.adjoint_gp_ptr(*(t.data_ptr() for t in gd), uz=uz.data_ptr(), dg=dg.data_ptr())
        c2 = cvxopt_b200.launch_count()
        gb.adjoint_gp_ptr(*(t.data_ptr() for t in gd), uz=uz.data_ptr(), dG=dG.data_ptr())
        c3 = cvxopt_b200.launch_count()
        gb.adjoint_gp(*g)
        c4 = cvxopt_b200.launch_count()
        assert c2 - c1 == (c1 - c0) + 3, "dg: the GEMV's two kernels and k_adj_gp_dg"
        assert c3 - c2 == (c1 - c0) + 1, "dG alone: k_adj_gp_grad"
        assert c4 - c3 == (c1 - c0) + 4, "every output: both"
        print("\ngp adjoint launches (B=%d, n=%d, K=%s, p=%d): %d" % (B, n, K, p, c4 - c3))
        if LAUNCHES is not None:
            assert c4 - c3 == LAUNCHES
        u, gg, GG = uz.cpu().numpy(), dg.cpu().numpy(), dG.cpu().numpy()
        assert (u[B * (mnl + ml):] == 7.0).all() and (gg[B * S:] == 7.0).all() and (GG[B * n * ml:] == 7.0).all()
        assert np.array_equal(u[:B * (mnl + ml)].reshape(B, -1)[:, mnl:], full["h"])
        assert np.array_equal(gg[:B * S].reshape(B, S), full["g"])
        assert np.array_equal(GG[:B * n * ml].reshape(B, n, ml).transpose(0, 2, 1), full["G"])
        only = gb.adjoint_gp(*g, want=("F",))
        assert set(only) == {"F"} and np.array_equal(only["F"], full["F"])
        # a new load (problem data, then A and b) needs a new solve
        gb.load(*(d[k] for k in KEYS))
        with pytest.raises(ValueError, match="no completed"):
            gb.adjoint_gp(*g)
        gb.solve()
        gb._load_eq(np.ascontiguousarray(d["A"].transpose(0, 2, 1)), d["b"], _lib.HOST)
        with pytest.raises(ValueError, match="no completed"):
            gb.adjoint_gp(*g)
    finally:
        gb.close()
    assert lib.cvxb_device_bytes() == before


def _refused(batch):
    from cvxopt_b200 import GPBatch
    with pytest.raises(NotImplementedError, match="GP"):
        GPBatch.adjoint_gp_ptr(batch)
    batch.close()


def test_adjoint_gp_refuses_other_batches():
    from cvxopt_b200 import CPBatch, CPLBatch, ConeLPBatch, QCQPBatch, QPBatch, SDPBatch, SDPQPBatch
    _refused(QPBatch(3, 5, 7, 0))
    _refused(ConeLPBatch(3, 5, 8, 0))
    _refused(CPBatch(3, 5, 1, 4))
    _refused(CPLBatch(3, 5, 1, {"l": 4}))
    _refused(QCQPBatch(3, 5, 1, 4))
    _refused(SDPBatch(3, 5, {"l": 4, "s": [3]}))
    _refused(SDPQPBatch(3, 5, {"l": 4, "s": [3]}))


def _torch(d, keys, dev=None):
    import torch
    dev = dev or torch.device("cuda", 0)
    return [torch.from_numpy(np.ascontiguousarray(d[k])).to(dev) for k in keys]


def test_gp_layer_backward_equals_group_adjoint():
    import torch
    from cvxopt_b200 import gp_layer
    K = [32, 8, 8, 8]
    d = _data(24, 16, K, 4, 2, 700)
    mnl = len(K) - 1
    g = _grads(K, d, 29)
    t = [x.requires_grad_() for x in _torch(d, KEYS)]
    x, y, znl, zl, status = gp_layer(K, *t, nsub=3)
    grp = _solved_group(K, d, nsub=3)
    try:
        res = grp.results()
        want = grp.adjoint_gp(*g)
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


def test_gp_layer_through_log_coefficients():
    """posynomial coefficients c > 0 enter as g = log(c): dL/dc = dL/dg / c, summed over a c shared by the batch"""
    import torch
    from cvxopt_b200 import gp_layer
    K = [16, 4, 4]
    d = _data(6, 8, K, 3, 0, 800)
    B = d["F"].shape[0]
    dev = torch.device("cuda", 0)
    c = torch.from_numpy(np.exp(d["g"])).to(dev).requires_grad_()
    c0 = torch.from_numpy(np.exp(d["g"][0])).to(dev).requires_grad_()
    F, G, h = _torch(d, ("F", "G", "h"))
    rng = np.random.default_rng(31)
    gx = torch.from_numpy(rng.standard_normal((B, 8))).to(dev)
    x, y, znl, zl, status = gp_layer(K, F, torch.log(c), G, h)
    assert (status == 1).all()
    (gc,) = torch.autograd.grad((x * gx).sum(), (c,))
    # the group solves the g the layer saw, log(c), bit for bit
    grp = _solved_group(K, dict(d, g=torch.log(c).detach().cpu().numpy()), nsub=1)
    try:
        want = grp.adjoint_gp(gx.cpu().numpy(), want=("g",))["g"]
    finally:
        grp.close()
    assert np.allclose(gc.cpu().numpy(), want / c.detach().cpu().numpy(), rtol=1e-14, atol=0)
    # one coefficient vector for the whole batch: its gradient is the sum over the problems
    g0 = torch.log(c0).detach().cpu().numpy()
    x, *_ = gp_layer(K, F, torch.log(c0).expand(B, -1), G, h)
    (gc0,) = torch.autograd.grad((x * gx).sum(), (c0,))
    grp = _solved_group(K, dict(d, g=np.broadcast_to(g0, d["g"].shape).copy()), nsub=1)
    try:
        want0 = grp.adjoint_gp(gx.cpu().numpy(), want=("g",))["g"]
    finally:
        grp.close()
    assert np.allclose(gc0.cpu().numpy(), want0.sum(axis=0) / c0.detach().cpu().numpy(), rtol=1e-12, atol=1e-15)


def test_gp_layer_work_streams_and_memory():
    import cvxopt_b200
    import torch
    from cvxopt_b200 import _lib, gp_layer
    K = [16, 4, 4]
    d = _data(12, 10, K, 3, 2, 900)
    mnl = len(K) - 1
    g = [torch.from_numpy(a).cuda() for a in _grads(K, d, 37)]
    lib = _lib.load()
    before = lib.cvxb_device_bytes()

    def run(needs, stream=None):
        with torch.cuda.stream(stream):                  # None: torch's current stream
            t = _torch(d, KEYS)
            for x, need in zip(t, needs):
                x.requires_grad_(need)
            x, y, znl, zl, _ = gp_layer(K, *t, nsub=1)
            c0 = cvxopt_b200.launch_count()
            grads = torch.autograd.grad((x * g[0]).sum() + (y * g[1]).sum() + (znl * g[2][:, :mnl]).sum() +
                                        (zl * g[2][:, mnl:]).sum(), [a for a, need in zip(t, needs) if need])
            torch.cuda.synchronize()
        return grads, cvxopt_b200.launch_count() - c0
    full, c_full = run([True] * 6)
    assert lib.cvxb_device_bytes() == before
    vec, c_vec = run([False, False, False, True, False, True])
    assert c_vec == c_full - 4, "no matrix and no dg output: no GEMV, no k_adj_gp_dg, no k_adj_gp_grad"
    for a, b in zip(vec, (full[3], full[5])):
        assert torch.equal(a, b)
    side = torch.cuda.Stream()
    on_side, _ = run([True] * 6, side)
    for a, b in zip(on_side, full):
        assert torch.equal(a, b)
    # inputs without requires_grad: nothing is kept for backward, nothing stays on the device
    t = _torch(d, KEYS)
    c0 = cvxopt_b200.launch_count()
    x, *_ = gp_layer(K, *t, nsub=1)
    assert not x.requires_grad
    assert lib.cvxb_device_bytes() == before
    assert cvxopt_b200.launch_count() > c0
