"""The cone adjoint (cvxb_batch_adjoint_cone, adjoint_cone, coneqp_layer, conelp_layer) on the device: parity with a
dense numpy solve of the KKT matrix at the batch's own returned iterate, with W'W from the reference's NT scaling;
central differences of the reference's coneqp and conelp; the 's' convention; identity with the 'l'-only adjoint; the
NaN policy; bit-identity across compaction, sub-batches, spaces and repeated calls; the call contract and the layers."""

import numpy as np
import pytest

from test_batch_conelp_gpu import lp_batch
from test_batch_eq_gpu import eq_batch
from test_batch_sdp_gpu import _full, sdp_batch_data
from test_batch_sdqp_gpu import sdqp_batch_data

pytestmark = pytest.mark.gpu

QP_KEYS = ("P", "q", "G", "h", "A", "b")
LP_KEYS = ("c", "G", "h", "A", "b")


def _grads(B, n, p, m, seed):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((B, n)), rng.standard_normal((B, p)), rng.standard_normal((B, m))


def _group(data, dims, nsub=None, **options):
    """the solved group of a QP (data P, q, G, h, A, b) or cone LP (c, G, h, A, b) batch, as coneqp_batch,
    conelp_batch and sdp_batch build it"""
    from cvxopt_b200 import ConeLPBatchGroup, QPBatchGroup, SDPBatchGroup, SDPQPBatchGroup
    dims = _full(dims)
    lp = len(data) == 5
    B, n, p = data[0].shape[0], data[-2].shape[2], data[-2].shape[1]
    m = data[-3].shape[1]
    if dims["s"]:
        grp = (SDPBatchGroup if lp else SDPQPBatchGroup)(B, n, dims, p, 0, nsub)
    else:
        grp = (ConeLPBatchGroup if lp else QPBatchGroup)(B, n, m, 0, nsub, dims, p)
    grp.load(*data)
    grp.solve(**options)
    return grp


def _packing(ref, dims):
    """pack and unpack of the reference's misc (the isometry between the trace inner product on 's' blocks and the
    Euclidean one on their packed lower triangles), on numpy vectors"""
    from cvxopt import matrix, misc
    cdim = dims["l"] + sum(dims["q"]) + sum(k * k for k in dims["s"])
    cpk = dims["l"] + sum(dims["q"]) + sum(k * (k + 1) // 2 for k in dims["s"])

    def pack(v):
        y = matrix(0.0, (cpk, 1))
        misc.pack(matrix(np.ascontiguousarray(v, dtype=float)), y, dims)
        return np.array(y).ravel()

    def unpack(v):                        # misc.unpack writes the lower triangles: mirror them
        y = matrix(0.0, (cdim, 1))
        misc.unpack(matrix(np.ascontiguousarray(v, dtype=float)), y, dims)
        y = np.array(y).ravel()
        o = dims["l"] + sum(dims["q"])
        for k in dims["s"]:
            M = np.tril(y[o:o + k * k].reshape(k, k, order="F"))
            y[o:o + k * k] = (M + np.tril(M, -1).T).reshape(-1, order="F")
            o += k * k
        return y
    return pack, unpack, cdim, cpk


def _sym(v, dims):
    """v with each 's' block replaced by its symmetric part"""
    v = np.array(v, dtype=float)
    o = dims["l"] + sum(dims["q"])
    for k in dims["s"]:
        M = v[o:o + k * k].reshape(k, k, order="F")
        v[o:o + k * k] = ((M + M.T) / 2).reshape(-1, order="F")
        o += k * k
    return v


def _oracle(ref, data, dims, x, y, s, z, g):
    """per problem: M = [P A' Gp'; A 0 0; Gp 0 -H] in the reference's packed coordinates at the iterate (x, y, s, z),
    Gp = pack(G), H = pack(W'W unpack(.)) with W from misc.compute_scaling and applied by misc.scale; u = M^{-1}
    [gx; gy; pack(sym(gz))], uz unpacked; the formulas of include/cvxopt_b200.h, and cond(M)"""
    from cvxopt import matrix, misc
    dims = _full(dims)
    lp = len(data) == 5
    G, A = data[-4], data[-2]
    B, n = x.shape
    p = y.shape[1]
    pack, unpack, cdim, cpk = _packing(ref, dims)
    out = {k: [] for k in (LP_KEYS if lp else QP_KEYS)}
    cond = []
    for j in range(B):
        W = misc.compute_scaling(matrix(s[j]), matrix(z[j]), matrix(0.0, (cdim, 1)), dims)
        H = np.zeros((cpk, cpk))
        for i in range(cpk):
            e = matrix(unpack(np.eye(cpk)[i]))
            misc.scale(e, W)
            misc.scale(e, W, trans="T")
            H[:, i] = pack(np.array(e).ravel())
        Gp = np.stack([pack(G[j][:, c]) for c in range(n)], axis=1)
        N = n + p + cpk
        M = np.zeros((N, N))
        if not lp:
            M[:n, :n] = data[0][j]
        M[n:n + p, :n] = A[j]
        M[:n, n:n + p] = A[j].T
        M[n + p:, :n] = Gp
        M[:n, n + p:] = Gp.T
        M[n + p:, n + p:] = -H
        D = 1.0 / np.sqrt(np.abs(M).max(axis=1))         # equilibrated: the oracle's own error stays near u
        rhs = np.concatenate([g[0][j], g[1][j], pack(_sym(g[2][j], dims))])
        u = D * np.linalg.solve(D[:, None] * M * D, D * rhs)
        ux, uy, uz = u[:n], u[n:n + p], unpack(u[n + p:])
        out["c" if lp else "q"].append(-ux)
        out["b"].append(uy)
        out["h"].append(uz)
        if not lp:
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


def _parity(ref, data, dims, seed, **options):
    grp = _group(data, dims, **options)
    try:
        res = grp.results()
        assert all(c == 1 for c in res["status_code"])
        B, n, m, p = grp.B, grp.n, grp.m, grp.p
        g = _grads(B, n, p, m, seed)
        got = grp.adjoint_cone(*g)
    finally:
        grp.close()
    want, cond = _oracle(ref, data, dims, res["x"], res["y"], res["s"], res["z"], g)
    worst = _check_oracle(got, want, cond)
    print("\nadjoint_cone dims=%s B=%d n=%d p=%d: largest relative difference %.1e, cond(M) up to %.1e"
          % (dims, B, n, p, worst, cond.max()))
    return got


PARITY = [
    ("qp", 7, 10, {"l": 8, "q": [4, 3]}, 0), ("qp", 33, 16, {"l": 12, "q": [5, 1, 3]}, 3),
    ("qp", 1, 10, {"l": 8, "q": [4]}, 2), ("sdqp", 9, 10, {"l": 6, "q": [4], "s": [3, 2]}, 2),
    ("lp", 9, 10, {"l": 24}, 3), ("lp", 9, 10, {"l": 12, "q": [4, 3]}, 2),
    ("sdp", 9, 8, {"l": 6, "s": [1, 4]}, 2), ("sdp", 257, 6, {"l": 4, "s": [3]}, 0),
]


@pytest.mark.parametrize("kind,B,n,dims,p", PARITY)
def test_adjoint_cone_matches_dense_kkt_solve(ref, kind, B, n, dims, p):
    seed = 100 * B + n
    data = {"qp": lambda: eq_batch(B, n, dims, p, seed), "sdqp": lambda: sdqp_batch_data(B, n, dims, p, seed),
            "lp": lambda: lp_batch(B, n, dims, p, seed), "sdp": lambda: sdp_batch_data(B, n, dims, p, seed)}[kind]()
    _parity(ref, data, dims, 7)


def test_adjoint_cone_through_the_s_plus_ata_switch(ref):
    """an LP batch whose problems 1 and 3 factor S + A'A (test_batch_conelp_gpu's construction)"""
    n, m, p = 64, 128, 16
    data = lp_batch(4, n, {"l": m}, p, 9000)
    c, G, h, A, b = data
    rng = np.random.Generator(np.random.PCG64(9100))
    for j in (1, 3):
        G[j][:, 48:] = 0.0
        x0, z0, y0 = rng.standard_normal(n), rng.uniform(0.5, 1.5, m), rng.standard_normal(p)
        h[j] = G[j] @ x0 + rng.uniform(0.5, 1.5, m)
        b[j] = A[j] @ x0
        c[j] = -(G[j].T @ z0 + A[j].T @ y0)
    _parity(ref, data, {"l": m}, 13, nsub=1)


def _margin(s, z, dims):
    """the smallest Jordan eigenvalue of s + z over the cones: 'l' rows, u0 - |u1| of each 'q' cone, and the
    eigenvalues of S + Z of each 's' block"""
    u = s + z
    lam = list(u[:dims["l"]])
    o = dims["l"]
    for k in dims["q"]:
        lam.append(u[o] - np.linalg.norm(u[o + 1:o + k]))
        o += k
    for k in dims["s"]:
        lam.extend(np.linalg.eigvalsh(u[o:o + k * k].reshape(k, k, order="F")))
        o += k * k
    return min(lam)


def _sym_direction(rng, shape, dims):
    """a random direction whose 's' rows are symmetric blocks (column by column for G)"""
    d = rng.standard_normal(shape)
    return _sym(d, dims) if d.ndim == 1 else np.stack([_sym(d[:, j], dims) for j in range(d.shape[1])], axis=1)


TIGHT = dict(abstol=1e-10, reltol=1e-10, feastol=1e-10)
DELTA = 1e-2         # the strict-complementarity margin a seed must have


def _central_differences(ref, data, dims, seed, solve, rtol=1e-4, **options):
    """the batch's adjoint against central differences of the reference's solve(**data) along a random direction"""
    dims = _full(dims)
    lp = len(data) == 5
    keys = LP_KEYS if lp else QP_KEYS
    cur = dict(zip(keys, (a[0] for a in data)))
    base = solve(**cur)
    s, z = np.array(base["s"]).ravel(), np.array(base["z"]).ravel()
    assert _margin(s, z, dims) > DELTA, "no strict complementarity: the active set could change"
    grp = _group(data, dims, nsub=1, **(options or TIGHT))
    try:
        assert grp.results()["status_code"][0] == 1
        n, m, p = grp.n, grp.m, grp.p
        g = _grads(1, n, p, m, 50 + seed)
        grad = grp.adjoint_cone(*g)
    finally:
        grp.close()
    rng = np.random.default_rng(60 + seed)
    d = {k: _sym_direction(rng, cur[k].shape, dims) if k in ("G", "h") else rng.standard_normal(cur[k].shape)
         for k in keys}
    if not lp:
        d["P"] = d["P"] + d["P"].T
    eps = 1e-5

    def loss(r):
        return sum(float(gi[0] @ np.array(r[k]).ravel()) for gi, k in zip(g, ("x", "y", "z")))
    fd = (loss(solve(**{k: cur[k] + eps * d[k] for k in keys})) -
          loss(solve(**{k: cur[k] - eps * d[k] for k in keys}))) / (2 * eps)
    an = sum(float(np.sum(grad[k][0] * d[k])) for k in keys)
    assert abs(fd - an) <= rtol * max(abs(fd), abs(an)), (fd, an)


def _ref_coneqp(dims):
    from cvxopt import matrix, solvers

    def solve(P, q, G, h, A, b):
        r = solvers.coneqp(matrix(P), matrix(q), matrix(G), matrix(h), _full(dims), matrix(A), matrix(b),
                           options=dict(TIGHT, show_progress=False))
        assert r["status"] == "optimal"
        return r
    return solve


SOCP = {"l": 6, "q": [4, 3]}


def _ref_conelp(dims):
    from cvxopt import matrix, solvers

    def solve(c, G, h, A, b):
        r = solvers.conelp(matrix(c), matrix(G), matrix(h), _full(dims), matrix(A), matrix(b), kktsolver="chol",
                           options=dict(TIGHT, show_progress=False))
        assert r["status"] == "optimal"
        return r
    return solve


def _slack(data, dims, lift=10.0):
    """h's cone rows lifted by `lift` (each 'q' cone's leading row, each 's' block's diagonal): at the solution s is
    inside every cone and z = 0 there, the cones' strictly complementary case that does not depend on centring"""
    dims = _full(dims)
    h = data[-3]
    o = dims["l"]
    for k in dims["q"]:
        h[:, o] += lift
        o += k
    for k in dims["s"]:
        h[:, o:o + k * k:k + 1] += lift
        o += k * k
    return data


# The tolerance of every central-difference test is 1e-4 relative: at a margin of 2e-2 (seed 0) one refinement step
# leaves 1.8e-5 at the batch's iterate (1e-9 at the reference's), the accuracy DESIGN.md records for the QP and QCQP
# adjoints.  The coneqp seeds are 0-5 less those with a 'q' cone whose s and z both lie on its boundary: there the
# derivative depends on how well centred the returned iterate is (W'W on the off-diagonal Peirce space is a ratio of
# the small eigenvalues), and seeds 2, 4 and 5 differ by 2.9e-1, 2.0e-2 and 5.9e-3 even at the reference's iterate
@pytest.mark.parametrize("seed", [0, 1, 3])
def test_adjoint_cone_matches_central_differences_of_coneqp(ref, seed):
    _central_differences(ref, eq_batch(1, 8, SOCP, 2, 4000 + seed), SOCP, seed, _ref_coneqp(SOCP))


# conelp on an 'l' LP (seeds 0-2; seed 3 does not reach 'optimal' at 1e-10 in the reference), and on an SOCP and an
# SDP whose cones are slack at the solution: of seeds 0-5 with h lifted, seed 1 of each leaves every cone inactive (z = 0
# there, checked below); in the others a cone stays active with s and z both on its boundary.  The batch's cone LPs
# stop at tolerances of 1e-8: at 1e-10 they end with a singular factorisation on these problems
LP_FD = [({"l": 14}, False, 4300), ({"l": 14}, False, 4301), ({"l": 14}, False, 4302),
         ({"l": 10, "q": [4, 3]}, True, 4101), ({"l": 10, "s": [3, 2]}, True, 4201)]


@pytest.mark.parametrize("dims,slack,seed", LP_FD)
def test_adjoint_cone_matches_central_differences_of_conelp(ref, dims, slack, seed):
    make = sdp_batch_data if dims.get("s") else lp_batch
    data = make(1, 6 if dims.get("s") else 8, dims, 0, seed)
    if slack:
        data = _slack(data, dims)
        z = np.array(_ref_conelp(dims)(*(a[0] for a in data))["z"]).ravel()
        assert np.abs(z[dims["l"]:]).max() < 1e-6, "a cone is active at the solution"
    _central_differences(ref, data, dims, seed % 100, _ref_conelp(dims), abstol=1e-8, reltol=1e-8, feastol=1e-8)


def _s_rows(dims):
    """(offset, order) of each 's' block's rows"""
    o = dims["l"] + sum(dims["q"])
    for k in dims["s"]:
        yield o, k
        o += k * k


@pytest.mark.parametrize("lp", [False, True])
def test_s_convention(lp):
    """gz given on an 's' block's upper triangle, its transpose and its symmetric part give the same outputs, bit for
    bit; the 's' blocks of dh and of each column of dG are exactly symmetric"""
    dims = {"l": 3, "q": [3], "s": [3, 1, 4]}
    B, n, p = 5, 8, 2
    data = sdp_batch_data(B, n, dims, p, 300) if lp else sdqp_batch_data(B, n, dims, p, 300)
    grp = _group(data, dims, nsub=1)
    try:
        m = grp.m
        gx, gy, gz = _grads(B, n, p, m, 41)
        up, lo, sym = gz.copy(), gz.copy(), gz.copy()
        for o, k in _s_rows(dims):
            M = gz[:, o:o + k * k].reshape(B, k, k).transpose(0, 2, 1)     # column-major blocks
            U = np.triu(M, 1) + np.einsum("bii->bi", M)[:, :, None] * np.eye(k)
            for v, X in ((up, U), (lo, U.transpose(0, 2, 1)), (sym, (U + U.transpose(0, 2, 1)) / 2)):
                v[:, o:o + k * k] = X.transpose(0, 2, 1).reshape(B, k * k)
        outs = [grp.adjoint_cone(gx, gy, v) for v in (up, lo, sym)]
    finally:
        grp.close()
    for k in outs[0]:
        assert np.array_equal(outs[0][k], outs[1][k]) and np.array_equal(outs[0][k], outs[2][k]), k
    for o, k in _s_rows(dims):
        h = outs[0]["h"][:, o:o + k * k].reshape(B, k, k)
        assert np.array_equal(h, h.transpose(0, 2, 1))
        G = outs[0]["G"][:, o:o + k * k, :].reshape(B, k, k, n)
        assert np.array_equal(G, G.transpose(0, 2, 1, 3))


def test_l_only_qp_batch_is_the_qp_adjoint_bit_for_bit():
    import cvxopt_b200
    from cvxopt_b200 import QPBatch
    B, n, m, p = 9, 20, 40, 3
    data = eq_batch(B, n, {"l": m}, p, 310)
    g = _grads(B, n, p, m, 43)
    qb = QPBatch(B, n, m, 0, p=p)
    try:
        qb.load(*data)
        qb.solve()
        c0 = cvxopt_b200.launch_count()
        a = qb.adjoint(*g)
        c1 = cvxopt_b200.launch_count()
        b = qb.adjoint_cone(*g)
        c2 = cvxopt_b200.launch_count()
    finally:
        qb.close()
    assert c1 - c0 == c2 - c1
    for k in QP_KEYS:
        assert np.array_equal(a[k], b[k]), k


def test_nan_for_problems_that_are_not_optimal_qp(ref):
    dims = {"l": 6, "q": [4], "s": [3]}
    B, n, p = 9, 10, 2
    data = sdqp_batch_data(B, n, dims, p, 320)
    data[1] *= np.linspace(0.1, 30.0, B)[:, None]
    grp = _group(data, dims, nsub=1)
    try:
        m = grp.m
        g = _grads(B, n, p, m, 47)
        full = grp.adjoint_cone(*g)
        its = grp.results()["iterations"]
    finally:
        grp.close()
    assert its.min() < its.max()
    grp = _group(data, dims, nsub=1, maxiters=int(its.min() + its.max()) // 2)
    try:
        res = grp.results()
        got = grp.adjoint_cone(*g)
    finally:
        grp.close()
    ok = res["status_code"] == 1
    assert ok.any() and not ok.all()
    for k in QP_KEYS:
        assert np.isnan(got[k][~ok]).all(), k
        assert np.isfinite(got[k][ok]).all(), k
        assert np.allclose(got[k][ok], full[k][ok], rtol=1e-12, atol=0), k
    want, cond = _oracle(ref, data, dims, res["x"], res["y"], res["s"], res["z"], g)
    _check_oracle(got, want, cond, rows=np.flatnonzero(ok))


@pytest.mark.parametrize("dims", [{"l": 8, "q": [4, 3]}, {"l": 12, "s": [3]}])
def test_nan_for_infeasible_lps(ref, dims):
    """optimal, primal-infeasible (status 4) and dual-infeasible (status 5) problems in one LP batch"""
    B, n, p = 6, 8, 2
    kinds = {1: "pinf", 4: "dinf"}
    data = (sdp_batch_data if dims.get("s") else lp_batch)(B, n, dims, p, 330, kinds)
    grp = _group(data, dims, nsub=1)
    try:
        res = grp.results()
        m = grp.m
        g = _grads(B, n, p, m, 53)
        got = grp.adjoint_cone(*g)
    finally:
        grp.close()
    assert res["status_code"][1] == 4 and res["status_code"][4] == 5
    ok = res["status_code"] == 1
    assert ok.sum() == B - 2
    for k in LP_KEYS:
        assert np.isnan(got[k][~ok]).all(), k
        assert np.isfinite(got[k][ok]).all(), k
    rows = np.flatnonzero(ok)
    want, cond = _oracle(ref, [a[rows] for a in data], dims, *(res[k][rows] for k in ("x", "y", "s", "z")),
                         [a[rows] for a in g])
    _check_oracle({k: v[rows] for k, v in got.items()}, want, cond)


DIMS = {"l": 6, "q": [4, 3], "s": [3, 2]}


def _spread(seed):
    B, n, p = 9, 10, 2
    data = sdqp_batch_data(B, n, DIMS, p, seed)
    data[1] *= np.linspace(0.1, 30.0, B)[:, None]
    return data


def test_bit_identical_across_compaction_and_subbatches(monkeypatch):
    data = _spread(340)
    B, n, p = 9, 10, 2
    m = data[3].shape[1]
    g = _grads(B, n, p, m, 59)

    def run(nsub):
        grp = _group(data, DIMS, nsub=nsub)
        try:
            return grp.results(), grp.adjoint_cone(*g)
        finally:
            grp.close()
    r1, a1 = run(1)
    assert len(set(r1["iterations"].tolist())) > 1
    monkeypatch.setenv("CVXB_BATCH_COMPACT", "0")
    r0, a0 = run(1)
    monkeypatch.delenv("CVXB_BATCH_COMPACT")
    for k in QP_KEYS:
        assert np.array_equal(a0[k], a1[k]), k
    r2, a2 = run(2)
    r4, a4 = run(4)
    # a problem whose results differ between the two splits ran alone at the end of a sub-batch
    same = [j for j in range(B) if all(np.array_equal(r2[k][j], r4[k][j]) for k in ("x", "y", "s", "z"))]
    assert len(same) >= B // 2
    for k in QP_KEYS:
        assert np.array_equal(a2[k][same], a4[k][same]), k


@pytest.mark.parametrize("lp", [False, True])
def test_spaces_repeats_results_and_resolve(lp):
    import torch
    from cvxopt_b200 import SDPBatch, SDPQPBatch
    B, n, p = 9, 10, 2
    data = sdp_batch_data(B, n, DIMS, p, 350) if lp else _spread(350)
    m = data[-3].shape[1]
    g = _grads(B, n, p, m, 61)
    qb = (SDPBatch if lp else SDPQPBatch)(B, n, DIMS, p)
    try:
        qb.load(*data)
        qb.solve()
        r0 = qb.results()
        host = qb.adjoint_cone(*g)
        again = qb.adjoint_cone(*g)
        dev = torch.device("cuda", 0)
        gd = [torch.from_numpy(a).to(dev) for a in g]
        outs = [torch.full(s, 7.0, dtype=torch.float64, device=dev)
                for s in ((B, n), (B, p), (B, m), (B, n, n), (B, n, m), (B, n, p))]
        torch.cuda.synchronize()
        ptrs = [t.data_ptr() for t in outs]
        if lp:
            ptrs[3] = None
        qb.adjoint_cone_ptr(*(t.data_ptr() for t in gd), *ptrs)
        o = [t.cpu().numpy() for t in outs]
        on_dev = {"c" if lp else "q": -o[0], "b": o[1], "h": o[2], "G": o[4].transpose(0, 2, 1),
                  "A": o[5].transpose(0, 2, 1)}
        if not lp:
            on_dev["P"] = o[3].transpose(0, 2, 1)
        r1 = qb.results()
        qb.solve()
        r2 = qb.results()
    finally:
        qb.close()
    for k in host:
        assert np.array_equal(host[k], again[k]), k
        assert np.array_equal(host[k], on_dev[k]), k
    for k in ("x", "y", "s", "z", "iterations", "status_code", "primal objective"):
        assert np.array_equal(r0[k], r1[k]), k
        assert np.array_equal(r0[k], r2[k]), k


def test_call_contract():
    import cvxopt_b200
    import torch
    from cvxopt_b200 import SDPBatch, _lib
    dims = {"l": 4, "q": [3], "s": [2]}
    B, n, p = 5, 6, 2
    data = sdp_batch_data(B, n, dims, p, 360)
    m = data[2].shape[1]
    g = _grads(B, n, p, m, 67)
    qb = SDPBatch(B, n, dims, p)
    try:
        with pytest.raises(ValueError, match="no completed"):
            qb.adjoint_cone(*g)                     # never loaded
        qb.load(*data)
        with pytest.raises(ValueError, match="no completed"):
            qb.adjoint_cone(*g)
        qb.solve()
        full = qb.adjoint_cone(*g)
        with pytest.raises(ValueError, match="no P"):
            qb.adjoint_cone_ptr(*(None,) * 6, dP=1, space=_lib.HOST)
        zero = qb.adjoint_cone(g[0], np.zeros((B, p)), np.zeros((B, m)))
        null = qb.adjoint_cone(g[0])
        for k in LP_KEYS:
            assert np.array_equal(zero[k], null[k]), k
        dev = torch.device("cuda", 0)
        gd = [torch.from_numpy(a).to(dev) for a in g]
        guard = 4096
        ux = torch.full((B * n + guard,), 7.0, dtype=torch.float64, device=dev)
        dG = torch.full((B * m * n + guard,), 7.0, dtype=torch.float64, device=dev)
        torch.cuda.synchronize()
        c0 = cvxopt_b200.launch_count()
        qb.adjoint_cone_ptr(*(t.data_ptr() for t in gd), ux=ux.data_ptr(), dG=dG.data_ptr())
        c1 = cvxopt_b200.launch_count()
        qb.adjoint_cone_ptr(*(t.data_ptr() for t in gd), ux=ux.data_ptr())
        c2 = cvxopt_b200.launch_count()
        assert c1 - c0 == (c2 - c1) + 1, "the gradient kernel runs only for a matrix output"
        print("\nadjoint_cone launches (B=%d, n=%d, p=%d, dims %s): %d" % (B, n, p, dims, c1 - c0))
        u, dg = ux.cpu().numpy(), dG.cpu().numpy()
        assert (u[B * n:] == 7.0).all() and (dg[B * m * n:] == 7.0).all()
        assert np.array_equal(-u[:B * n].reshape(B, n), full["c"])
        assert np.array_equal(dg[:B * m * n].reshape(B, n, m).transpose(0, 2, 1), full["G"])
        only = qb.adjoint_cone(*g, want=("h",))
        assert set(only) == {"h"} and np.array_equal(only["h"], full["h"])
        qb.load(*data)
        with pytest.raises(ValueError, match="no completed"):
            qb.adjoint_cone(*g)
    finally:
        qb.close()


def _refused(batch):
    with pytest.raises(NotImplementedError, match="QP and cone LP"):
        batch.adjoint_cone_ptr()
    batch.close()


def test_refuses_other_batches():
    from cvxopt_b200 import CPBatch, CPLBatch, GPBatch, QCQPBatch
    _refused(GPBatch(3, 5, [2, 3], 4))
    _refused(CPBatch(3, 5, 1, 4))
    _refused(CPLBatch(3, 5, 1, {"l": 4}))
    _refused(QCQPBatch(3, 5, 1, 4, 0, 0))


def _torch(data):
    import torch
    dev = torch.device("cuda", 0)
    return [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in data]


SOCP_LAYER = {"l": 8, "q": [4, 3]}


@pytest.mark.parametrize("dims", [DIMS, SOCP_LAYER])
@pytest.mark.parametrize("lp", [False, True])
def test_layer_backward_equals_group_adjoint(lp, dims):
    """with 's' blocks the layers run on SDPQPBatchGroup / SDPBatchGroup, without them on SDPQPBatchGroup /
    ConeLPBatchGroup"""
    import torch
    from cvxopt_b200 import conelp_layer, coneqp_layer
    B, n, p = 12, 8, 2
    if dims.get("s"):
        data = sdp_batch_data(B, n, dims, p, 370) if lp else sdqp_batch_data(B, n, dims, p, 370)
    else:
        data = lp_batch(B, n, dims, p, 370) if lp else eq_batch(B, n, dims, p, 370)
    m = data[-3].shape[1]
    g = _grads(B, n, p, m, 71)
    t = [x.requires_grad_() for x in _torch(data)]
    if lp:
        x, y, z, status = conelp_layer(*t[:3], dims, *t[3:], nsub=3)
    else:
        x, y, z, status = coneqp_layer(*t[:4], dims, *t[4:], nsub=3)
    grp = _group(data, dims, nsub=3)
    try:
        res = grp.results()
        want = grp.adjoint_cone(*g)
    finally:
        grp.close()
    assert np.array_equal(status.cpu().numpy(), res["status_code"])
    for k, v in (("x", x), ("y", y), ("z", z)):
        assert np.array_equal(v.detach().cpu().numpy(), res[k]), k
    gt = _torch(g)
    grads = torch.autograd.grad((x * gt[0]).sum() + (y * gt[1]).sum() + (z * gt[2]).sum(), t)
    for k, v in zip(LP_KEYS if lp else QP_KEYS, grads):
        assert np.allclose(v.cpu().numpy(), want[k], rtol=1e-12, atol=1e-14), k


def test_layer_through_s_columns_built_as_x_plus_xt():
    """G's 's' block columns built as X + X' from a free X: autograd's dX = dG + dG' of the symmetric gradient"""
    import torch
    from cvxopt_b200 import conelp_layer
    dims = {"l": 4, "s": [3]}
    B, n, p = 4, 6, 1
    c, G, h, A, b = sdp_batch_data(B, n, dims, p, 380)
    dev = torch.device("cuda", 0)
    Xn = G[:, 4:, :].reshape(B, 3, 3, n).transpose(0, 2, 1, 3) / 2      # column-major blocks: X[b, i, j, col]
    X = torch.from_numpy(np.ascontiguousarray(Xn)).to(dev).requires_grad_()
    Gl, ct, ht, At, bt = _torch((G[:, :4, :], c, h, A, b))
    Gs = (X + X.transpose(1, 2)).transpose(1, 2).reshape(B, 9, n)
    x, y, z, status = conelp_layer(ct, torch.cat([Gl, Gs], 1), ht, dims, At, bt)
    assert (status == 1).all()
    gx = torch.from_numpy(np.random.default_rng(73).standard_normal((B, n))).to(dev)
    gX, = torch.autograd.grad((x * gx).sum(), (X,))
    Gn = torch.cat([Gl, Gs], 1).detach().cpu().numpy()
    grp = _group((c, Gn, h, A, b), dims, nsub=1)
    try:
        want = grp.adjoint_cone(gx.cpu().numpy(), want=("G",))["G"][:, 4:, :].reshape(B, 3, 3, n)
    finally:
        grp.close()
    want = want.transpose(0, 2, 1, 3)                                   # X's index order
    assert np.allclose(gX.cpu().numpy(), want + want.transpose(0, 2, 1, 3), rtol=1e-10, atol=1e-13)


def test_layer_side_stream_and_memory():
    import torch
    from cvxopt_b200 import _lib, coneqp_layer
    B, n, p = 6, 8, 2
    data = sdqp_batch_data(B, n, DIMS, p, 390)
    m = data[3].shape[1]
    g = _torch(_grads(B, n, p, m, 79))
    lib = _lib.load()
    before = lib.cvxb_device_bytes()

    def run(stream=None):
        with torch.cuda.stream(stream):                  # None: torch's current stream
            t = [x.requires_grad_() for x in _torch(data)]
            x, y, z, _ = coneqp_layer(*t[:4], DIMS, *t[4:], nsub=1)
            grads = torch.autograd.grad((x * g[0]).sum() + (y * g[1]).sum() + (z * g[2]).sum(), t)
            torch.cuda.synchronize()
        return grads
    full = run()
    assert lib.cvxb_device_bytes() == before
    on_side = run(torch.cuda.Stream())
    for a, b in zip(on_side, full):
        assert torch.equal(a, b)
    assert lib.cvxb_device_bytes() == before
