"""The CP and cpl batches' adjoint (cvxb_batch_adjoint_cp, CPBatch.adjoint_cp, cp_layer, cpl_layer) on the device, on
tests/cp_problems.py's, cpl_problems.py's and sdcpl_problems.py's families: parity with a dense solve of the KKT matrix
at the batch's own returned iterate, a cross-check against the QCQP adjoint, central differences of the reference's
solvers.cp and solvers.cpl, the NaN policy, exceptions from F, bit-identity across compaction, sub-batches, spaces and
repeated calls, the call contract and the torch layers."""

import numpy as np
import pytest

import cp_problems as cpp
import cpl_problems as cplp
from sdcpl_problems import sdcpl_batch_data

pytestmark = pytest.mark.gpu


def _full(dims):
    return {"l": dims.get("l", 0), "q": list(dims.get("q", [])), "s": list(dims.get("s", []))}


def _cp_group(family, d, nsub=None, F=None, rowwise=False, **options):
    from cvxopt_b200 import CPBatchGroup
    B, n = d["x0"].shape
    ml, p = d["G"].shape[1], d["A"].shape[1]
    grp = CPBatchGroup(B, n, cpp.MNL[family], ml, p, 0, nsub)
    grp.set_F(F or cpp.torch_F(family, d["data"], d["x0"], rowwise=rowwise))
    grp.load(d["x0"], d["G"], d["h"], d["A"] if p else None, d["b"] if p else None)
    grp.solve(**options)
    return grp


def _cpl_group(family, d, nsub=None, F=None, **options):
    from cvxopt_b200 import CPLBatchGroup, SDPCPLBatchGroup
    B, n = d["x0"].shape
    p, dims = d["A"].shape[1], _full(d["dims"])
    grp = (SDPCPLBatchGroup if dims["s"] else CPLBatchGroup)(B, n, cplp.MNL[family], dims, p, 0, nsub)
    grp.set_F(F or cplp.torch_F(family, d["data"], d["x0"]))
    grp.load(d["c"], d["x0"], d["G"], d["h"], d["A"] if p else None, d["b"] if p else None)
    grp.solve(**options)
    return grp


def _grads(B, n, p, m, seed):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((B, n)), rng.standard_normal((B, p)), rng.standard_normal((B, m))


def _sym(v, dims):
    """v with each 's' block replaced by its symmetric part"""
    v = np.array(v, dtype=float)
    o = dims["l"] + sum(dims["q"])
    for k in dims["s"]:
        M = v[o:o + k * k].reshape(k, k, order="F")
        v[o:o + k * k] = ((M + M.T) / 2).reshape(-1, order="F")
        o += k * k
    return v


def _packing(dims):
    """the reference's misc.pack and misc.unpack on numpy vectors, unpack mirroring the lower triangles"""
    from cvxopt import matrix, misc
    cdim = dims["l"] + sum(dims["q"]) + sum(k * k for k in dims["s"])
    cpk = dims["l"] + sum(dims["q"]) + sum(k * (k + 1) // 2 for k in dims["s"])

    def pack(v):
        y = matrix(0.0, (cpk, 1))
        misc.pack(matrix(np.ascontiguousarray(v, dtype=float)), y, dims)
        return np.array(y).ravel()

    def unpack(v):
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


def _oracle(evaluate, epi, d, dims, mnl, res, g):
    """per problem, at the returned iterate: zk = [1; znl] (epi) or znl, H and Df from the family's numpy evaluator,
    M = [H A' Gf'; A 0 0; Gf 0 -W'W] in the reference's packed coordinates with Gf = [Df; G] and W the reference's
    NT scaling of the returned s and z over dims {'l': mnl + l, 'q', 's'}; u = M^{-1} [gx; gy; pack(sym(gz))] solved
    equilibrated; include/cvxopt_b200.h's formulas, and cond(M)"""
    from cvxopt import matrix, misc
    full = dict(dims, l=mnl + dims["l"])
    pack, unpack, cdim, cpk = _packing(full)
    B, n = res["x"].shape
    p = d["A"].shape[1]
    out = {k: [] for k in ("ux", "uznl", "G", "h", "A", "b", "c")}
    cond = []
    for j in range(B):
        x, y, s, z = (np.asarray(res[k][j]) for k in ("x", "y", "s", "z"))
        zk = np.concatenate([[1.0], z[:mnl]]) if epi else z[:mnl]
        _, Df, H = evaluate(j, x, zk)
        Gf = np.vstack([Df[1:] if epi else Df, d["G"][j]])
        W = misc.compute_scaling(matrix(s), matrix(z), matrix(0.0, (cdim, 1)), full)
        WW = np.zeros((cpk, cpk))
        for i in range(cpk):
            e = matrix(unpack(np.eye(cpk)[i]))
            misc.scale(e, W)
            misc.scale(e, W, trans="T")
            WW[:, i] = pack(np.array(e).ravel())
        Gp = np.stack([pack(Gf[:, c]) for c in range(n)], axis=1)
        N = n + p + cpk
        M = np.zeros((N, N))
        M[:n, :n] = H
        M[n:n + p, :n] = d["A"][j]
        M[:n, n:n + p] = d["A"][j].T
        M[n + p:, :n] = Gp
        M[:n, n + p:] = Gp.T
        M[n + p:, n + p:] = -WW
        D = 1.0 / np.sqrt(np.abs(M).max(axis=1))
        rhs = np.concatenate([g[0][j], g[1][j], pack(_sym(g[2][j], full))])
        u = D * np.linalg.solve(D[:, None] * M * D, D * rhs)
        ux, uy, uz = u[:n], u[n:n + p], unpack(u[n + p:])
        out["ux"].append(ux)
        out["c"].append(-ux)
        out["uznl"].append(uz[:mnl])
        out["h"].append(uz[mnl:])
        out["G"].append(-(np.outer(z[mnl:], ux) + np.outer(uz[mnl:], x)))
        out["A"].append(-(np.outer(y, ux) + np.outer(uy, x)))
        out["b"].append(uy)
        cond.append(np.linalg.cond(M))
    return {k: np.array(v) for k, v in out.items()}, np.array(cond)


def _rel(a, b):
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


def _check_oracle(got, want, cond, rows=None):
    """every output within max(1e-9, 10 u cond(M)) relative of the oracle, per problem; the largest difference"""
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


def _cp_eval(family, d):
    return lambda j, x, z: cpp._eval_np(family, {k: v[j] for k, v in d["data"].items()}, x, z)


def _cpl_eval(family, d):
    return lambda j, x, z: cplp._eval_np(family, {k: v[j] for k, v in d["data"].items()}, x, z)


CP_SHAPES = [  # family, n, p, r (-1: _one_slack_row), B, options
    ("centering", 8, 3, 0, 6, {}),               # mnl = 0, p > 0, ml = 0
    ("entropy", 10, 2, 4, 6, {}),
    ("qcqp", 6, 0, 3, 8, {}),
    ("logistic", 8, 0, -1, 8, {"refinement": 0}),  # refinement 0: P mirrored by the adjoint itself
    ("qcqp", 8, 0, 2, 1, {}),                    # B = 1
    ("qcqp", 4, 0, 2, 257, {}),                  # several sub-batches, compaction
]


def _one_slack_row(d, n, B):
    """one 'l' row x_1 <= 100, inactive at the solution.  Without it, the logistic family's ball constraint ends with
    s / z near 1e-15 at the default tolerances, where one refinement step leaves the reduced solve up to 2e-2 from the
    dense one (DESIGN.md, "Adjoint of the CP and cpl batches": more steps converge to it)"""
    return dict(d, G=np.tile(np.eye(n)[None, :1], (B, 1, 1)), h=np.full((B, 1), 100.0))


@pytest.mark.parametrize("family,n,p,r,B,options", CP_SHAPES)
def test_adjoint_cp_matches_dense_kkt_solve(ref, family, n, p, r, B, options):
    d = cpp.cp_batch_data(family, range(100, 100 + B), n, p, max(r, 0))
    if r < 0:
        d = _one_slack_row(d, n, B)
    mnl = cpp.MNL[family]
    grp = _cp_group(family, d, **options)
    try:
        res = grp.results()
        g = _grads(B, n, p, mnl + d["G"].shape[1], 7)
        got = grp.adjoint_cp(*g)
    finally:
        grp.close()
    ok = res["status_code"] == 1
    assert ok.sum() >= max(1, (4 * B) // 5)
    assert got["G"].shape == d["G"].shape and got["h"].shape == d["h"].shape and got["uznl"].shape == (B, mnl)
    want, cond = _oracle(_cp_eval(family, d), True, d, {"l": d["G"].shape[1], "q": [], "s": []}, mnl, res, g)
    worst = _check_oracle(got, want, cond, np.flatnonzero(ok))
    print("\ncp adjoint %s B=%d n=%d p=%d: largest relative difference %.1e, cond(M) up to %.1e"
          % (family, B, n, p, worst, cond[ok].max()))


CPL_SHAPES = [  # family, n, q, s, ml, p, B
    ("socp", 8, [3, 4], [], 2, 1, 6),
    ("logcone", 8, [3], [], 0, 0, 6),
    ("lsecone", 7, [3], [], 1, 0, 6),
    ("socp", 8, [3], [3, 2], 2, 0, 5),           # 's' blocks (sdp_cpl_batch)
]


@pytest.mark.parametrize("family,n,q,s,ml,p,B", CPL_SHAPES)
def test_adjoint_cpl_matches_dense_kkt_solve(ref, family, n, q, s, ml, p, B):
    if s:
        d = sdcpl_batch_data(family, range(100, 100 + B), n, q, s, ml, p)
    else:
        d = cplp.cpl_batch_data(family, range(100, 100 + B), n, q, ml, p)
    dims = _full(d["dims"])
    mnl = cplp.MNL[family]
    grp = _cpl_group(family, d)
    try:
        res = grp.results()
        g = _grads(B, n, p, mnl + d["G"].shape[1], 11)
        got = grp.adjoint_cp(*g)
    finally:
        grp.close()
    ok = res["status_code"] == 1
    assert ok.sum() >= max(1, (4 * B) // 5)
    assert np.array_equal(got["c"], -got["ux"])
    want, cond = _oracle(_cpl_eval(family, d), False, d, dims, mnl, res, g)
    worst = _check_oracle(got, want, cond, np.flatnonzero(ok))
    print("\ncpl adjoint %s B=%d n=%d dims=%s: largest relative difference %.1e, cond(M) up to %.1e"
          % (family, B, n, dims, worst, cond[ok].max()))


def _qcqp_param_F(x0, mnl=3):
    """the qcqp family's F with P, q and r as params"""
    def F(x=None, z=None, idx=None, params=()):
        if x is None:
            return mnl, x0
        return cpp.torch_F("qcqp", dict(zip(("P", "q", "r"), params)), x0)(x, z, idx=idx)
    return F


def _torch(*arrays):
    import torch
    return [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]


def test_cp_layer_matches_qcqp_layer():
    """cp_layer on the qcqp family's F, parameterised by (P, q, r), against qcqp_layer on the same data: the two solve
    the same problems by the same algorithm with F evaluated in torch and in the library's kernels, so they differ by
    rounding; the gradients agree to a tolerance set from the difference of the solutions"""
    import torch
    from cvxopt_b200 import cp_layer, qcqp_layer
    B, n, r = 8, 6, 3
    d = cpp.cp_batch_data("qcqp", range(200, 200 + B), n, 0, r)
    P, q, rr, G, h = _torch(d["data"]["P"], d["data"]["q"], d["data"]["r"], d["G"], d["h"])
    g = [torch.from_numpy(a).cuda() for a in _grads(B, n, 0, 3 + G.shape[1], 13)]

    def run(layer):
        t = [a.clone().requires_grad_() for a in (P, q, rr, G, h)]
        if layer == "cp":
            x, y, znl, zl, st = cp_layer(_qcqp_param_F(torch.from_numpy(d["x0"]).cuda()), tuple(t[:3]), t[3], t[4])
        else:
            x, y, znl, zl, st = qcqp_layer(*t)
        assert (st == 1).all()
        loss = (x * g[0]).sum() + (znl * g[2][:, :3]).sum() + (zl * g[2][:, 3:]).sum()
        gr = torch.autograd.grad(loss, t)
        return [a.detach().cpu().numpy() for a in (x, znl, zl)], [a.cpu().numpy() for a in gr]
    (xa, za, zla), ga = run("cp")
    (xb, zb, zlb), gb = run("qcqp")
    dsol = max(_rel(xa, xb), _rel(za, zb), _rel(zla, zlb))
    sym = lambda a: (a + a.transpose(0, 1, 3, 2)) / 2       # noqa: E731  qcqp_layer's dP is the symmetric one
    diffs = [_rel(sym(ga[0]), gb[0])] + [_rel(a, b) for a, b in zip(ga[1:], gb[1:])]
    tol = max(1e-6, 1e3 * dsol)
    print("\ncp_layer against qcqp_layer: solutions %.1e apart; gradients (P, q, r, G, h) %s, tolerance %.1e"
          % (dsol, ["%.1e" % v for v in diffs], tol))
    assert max(diffs) <= tol


def _margin(s, z):
    return float(np.maximum(s, z).min())


def _ref_cp(ref, family, data, x0, G, h, A, b):
    from cvxopt import matrix, solvers
    F = cpp.ref_F(family, {k: v[None] for k, v in data.items()}, 0, x0)
    kw = {}
    if G.shape[0]:
        kw.update(G=matrix(G), h=matrix(h))
    if A.shape[0]:
        kw.update(A=matrix(A), b=matrix(b))
    res = solvers.cp(F, options=dict(abstol=1e-10, reltol=1e-10, feastol=1e-10, show_progress=False), **kw)
    assert res["status"] == "optimal"
    return res


# seeds chosen by margin: min max(s, z) over the nonlinear and 'l' rows of the reference's solution at least 0.1, so
# that no row changes from active to inactive within the perturbation (qcqp seeds 7000-7009: 7001, 7003, 7005, 7006
# and 7008 qualify).  logistic seed 7002 (margin 1.13) missed by 5e-4: at 1e-10 its ball constraint's s / z is near
# 1e-16 and one refinement step does not recover the digits (DESIGN.md), so it is left out
CD_CASES = [("qcqp", 6, 0, 3, 7001), ("qcqp", 6, 0, 3, 7005)]


@pytest.mark.parametrize("family,n,p,r,seed", CD_CASES)
def test_adjoint_cp_matches_central_differences_of_cp(ref, family, n, p, r, seed):
    """dL/d(params, G, h) of cp_layer along one random direction against central differences of the reference's
    solvers.cp, with params the family's data (qcqp: P, q, r; logistic: the samples a)"""
    import torch
    from cvxopt_b200 import cp_layer
    pr = cpp.cp_problem(family, seed, n, p, r)
    keys = ("P", "q", "r") if family == "qcqp" else ("a",)
    mnl, ml = cpp.MNL[family], pr["G"].shape[0]
    base = _ref_cp(ref, family, pr["data"], pr["x0"], pr["G"], pr["h"], pr["A"], pr["b"])
    s = np.concatenate([np.array(base[k]).ravel() for k in ("snl", "sl")])
    z = np.concatenate([np.array(base[k]).ravel() for k in ("znl", "zl")])
    margin = _margin(s, z)
    assert margin >= 0.1, "seed %d: margin %.2e, the active set could change" % (seed, margin)
    gx, _, gz = (a[0] for a in _grads(1, n, 0, mnl + ml, 50 + seed))
    x0 = torch.from_numpy(pr["x0"][None]).cuda()
    other = {k: pr["data"][k][None] for k in pr["data"] if k not in keys}

    def F(x=None, zz=None, idx=None, params=()):
        if x is None:
            return mnl, x0
        return cpp.torch_F(family, dict(other, **dict(zip(keys, params))), x0)(x, zz, idx=idx)
    prm = [a.requires_grad_() for a in _torch(*(pr["data"][k][None] for k in keys))]
    G, h = [a.requires_grad_() for a in _torch(pr["G"][None], pr["h"][None])]
    x, y, znl, zl, st = cp_layer(F, tuple(prm), G, h, abstol=1e-10, reltol=1e-10, feastol=1e-10)
    assert int(st[0]) == 1
    gzt = torch.from_numpy(gz).cuda()
    loss = (x[0] * torch.from_numpy(gx).cuda()).sum() + (znl[0] * gzt[:mnl]).sum() + (zl[0] * gzt[mnl:]).sum()
    grads = [a[0].cpu().numpy() for a in torch.autograd.grad(loss, prm + [G, h])]
    rng = np.random.default_rng(60 + seed)
    names = list(keys) + ["G", "h"]
    arrays = [pr["data"][k] for k in keys] + [pr["G"], pr["h"]]
    dirs = [rng.standard_normal(a.shape) for a in arrays]
    if family == "qcqp":
        dirs[0] = dirs[0] + dirs[0].transpose(0, 2, 1)     # the P_i stay symmetric
    eps = 1e-5

    def loss_at(sign):
        moved = {k: a + sign * eps * dd for k, a, dd in zip(names, arrays, dirs)}
        data = dict({k: v[0] for k, v in other.items()}, **{k: moved[k] for k in keys})
        r_ = _ref_cp(ref, family, data, pr["x0"], moved["G"], moved["h"], pr["A"], pr["b"])
        zz = np.concatenate([np.array(r_["znl"]).ravel(), np.array(r_["zl"]).ravel()])
        return float(gx @ np.array(r_["x"]).ravel() + gz @ zz)
    fd = (loss_at(1) - loss_at(-1)) / (2 * eps)
    an = sum(float(np.sum(gg * dd)) for gg, dd in zip(grads, dirs))
    print("\ncp central differences %s seed %d (margin %.2f): fd %.10e adjoint %.10e" % (family, seed, margin, fd, an))
    assert abs(fd - an) <= 1e-5 * max(abs(fd), abs(an)), (fd, an)


def _central_differences(d, keys, solve, grad, g, eps=1e-5, seed=72):
    """the loss gx'x + gy'y + gz'z of solve(moved data) along one random direction of the data `keys`, by central
    differences, and the adjoint's directional derivative from grad"""
    rng = np.random.default_rng(seed)
    dirs = {k: rng.standard_normal(d[k].shape[1:]) for k in keys}

    def loss_at(sign):
        r_ = solve({k: d[k][0] + sign * eps * dirs[k] for k in keys})
        zz = np.concatenate([np.array(r_["znl"]).ravel(), np.array(r_["zl"]).ravel()])
        yy = np.array(r_["y"]).ravel() if g[1][0].size else np.zeros(0)
        return float(g[0][0] @ np.array(r_["x"]).ravel() + g[1][0] @ yy + g[2][0] @ zz)
    fd = (loss_at(1) - loss_at(-1)) / (2 * eps)
    an = sum(float(np.sum(grad[k][0] * dirs[k])) for k in keys)
    return fd, an


def _ref_margin(res, nrows):
    """min max(s, z) over the first nrows rows of [s; z] (nonlinear and 'l'), and the largest |z| on the cone rows"""
    s = np.concatenate([np.array(res[k]).ravel() for k in ("snl", "sl")])
    z = np.concatenate([np.array(res[k]).ravel() for k in ("znl", "zl")])
    return (_margin(s[:nrows], z[:nrows]) if nrows else np.inf), float(np.abs(z[nrows:]).max()) if z.size > nrows else 0.0


TIGHT = dict(abstol=1e-10, reltol=1e-10, feastol=1e-10)


# seeds chosen by margin as CD_CASES' (entropy 7000-7005 all qualify, 0.10 to 0.62; centering has no inequality rows)
@pytest.mark.parametrize("family,n,p,r,seed", [("entropy", 6, 2, 3, 7000), ("entropy", 6, 2, 3, 7002),
                                               ("centering", 6, 3, 0, 7000), ("centering", 6, 3, 0, 7001)])
def test_adjoint_cp_data_matches_central_differences_of_cp(ref, family, n, p, r, seed):
    """dL/d(G, h, A, b) of the CP batch along one random direction against central differences of solvers.cp"""
    from cvxopt import matrix, solvers
    d = cpp.cp_batch_data(family, [seed], n, p, r)
    mnl, ml = cpp.MNL[family], d["G"].shape[1]
    keys = ("G", "h", "A", "b") if ml else ("A", "b")

    def cp(dd):
        F = cpp.ref_F(family, d["data"], 0, d["x0"][0])
        kw = dict(A=matrix(dd["A"]), b=matrix(dd["b"]))
        if ml:
            kw.update(G=matrix(dd["G"]), h=matrix(dd["h"]))
        r_ = solvers.cp(F, options=dict(TIGHT, show_progress=False), **kw)
        assert r_["status"] == "optimal"
        return r_
    margin, _ = _ref_margin(cp({k: d[k][0] for k in keys}), mnl + ml)
    assert margin >= 0.1, "seed %d: margin %.2e, the active set could change" % (seed, margin)
    grp = _cp_group(family, d, nsub=1, **TIGHT)
    try:
        assert grp.results()["status_code"][0] == 1
        g = _grads(1, n, p, mnl + ml, 73 + seed)
        grad = grp.adjoint_cp(*g)
    finally:
        grp.close()
    fd, an = _central_differences(d, keys, cp, grad, g)
    print("\ncp central differences %s seed %d (margin %.2f): fd %.10e adjoint %.10e" % (family, seed, margin, fd, an))
    assert abs(fd - an) <= 1e-5 * max(abs(fd), abs(an)), (fd, an)


# seeds chosen by margin (at least 0.1 over the nonlinear and 'l' rows) with the cones slack at the reference's solution
# (|zl| < 1e-6 on the 'q' rows): lsecone 7000 and 7002 qualify, and 7001, 7003-7007 have active cones or margins from
# 0.011 to 0.052.  logcone 7000-7007 all qualify, but 7000 and 7003 missed by 4.5e-4 and 3.0e-4: their constraint
# -sum log x <= r ends strongly active, the known limit of one refinement step (DESIGN.md), so logcone is left out
@pytest.mark.parametrize("family,n,q,ml,p,seed", [("socp", 6, [3], 2, 1, 7100), ("lsecone", 5, [3], 1, 0, 7000),
                                                  ("lsecone", 5, [3], 1, 0, 7002)])
def test_adjoint_cpl_matches_central_differences_of_cpl(ref, family, n, q, ml, p, seed):
    """dL/d(c, G, h, A, b) of the cpl batch along one random direction against central differences of solvers.cpl,
    on problems whose cones are slack at the solution"""
    from cvxopt import matrix, solvers
    d = cplp.cpl_batch_data(family, [seed], n, q, ml, p)
    dims = _full(d["dims"])
    mnl = cplp.MNL[family]
    keys = ("c", "G", "h", "A", "b") if p else ("c", "G", "h")

    def cpl(dd):
        F = cplp.ref_F(family, d["data"], 0, d["x0"][0])
        kw = dict(A=matrix(dd["A"]), b=matrix(dd["b"])) if p else {}
        r_ = solvers.cpl(matrix(dd["c"]), F, matrix(dd["G"]), matrix(dd["h"]), dims,
                         options=dict(TIGHT, show_progress=False), **kw)
        assert r_["status"] == "optimal"
        return r_
    margin, cone_z = _ref_margin(cpl({k: d[k][0] for k in keys}), mnl + dims["l"])
    assert margin >= 0.1 and cone_z < 1e-6, "cones not slack or no margin"
    grp = _cpl_group(family, d, nsub=1, **TIGHT)
    try:
        assert grp.results()["status_code"][0] == 1
        g = _grads(1, n, p, mnl + d["G"].shape[1], 71)
        grad = grp.adjoint_cp(*g)
    finally:
        grp.close()
    fd, an = _central_differences(d, keys, cpl, grad, g)
    print("\ncpl central differences %s seed %d (margin %.2f): fd %.10e adjoint %.10e" % (family, seed, margin, fd, an))
    assert abs(fd - an) <= 1e-5 * max(abs(fd), abs(an)), (fd, an)


def test_adjoint_cp_nan_for_problems_that_are_not_optimal():
    family, B = "logistic", 10
    d = cpp.cp_batch_data(family, range(300, 300 + B), 8)
    g = _grads(B, 8, 0, 1, 17)
    grp = _cp_group(family, d, nsub=1)
    try:
        full = grp.adjoint_cp(*g)
        its = grp.results()["iterations"]
    finally:
        grp.close()
    assert its.min() < its.max()
    grp = _cp_group(family, d, nsub=1, maxiters=int(its.min() + its.max()) // 2)
    try:
        res = grp.results()
        got = grp.adjoint_cp(*g)
    finally:
        grp.close()
    ok = res["status_code"] == 1
    assert not ok.all() and ok.any() and (res["status_code"][~ok] == 2).all()
    for k in got:
        assert np.isnan(got[k][~ok]).all(), k
        assert np.isfinite(got[k][ok]).all(), k
        assert np.array_equal(got[k][ok], full[k][ok]), k


def _poisoned(F, problem, calls):
    """F whose (f, Df, H) rows of `problem` are NaN from the second full call on (the adjoint's, after a solve that
    converged in one full call per iteration is not assumed: calls['arm'] switches it on)"""
    def G(x=None, z=None, idx=None):
        out = F(x, z, idx=idx)
        if z is not None and calls.get("arm"):
            out = tuple(o.clone() for o in out)
            rows = (idx == problem).nonzero().flatten()
            out[2][rows, 0, 0] = float("nan")
        return out
    return G


def test_adjoint_cp_nan_for_a_non_finite_f_at_the_adjoint():
    family, B, n = "qcqp", 8, 6
    d = cpp.cp_batch_data(family, range(400, 400 + B), n, 0, 2)
    g = _grads(B, n, 0, 3 + d["G"].shape[1], 19)
    calls = {}
    grp = _cp_group(family, d, nsub=1, F=_poisoned(cpp.torch_F(family, d["data"], d["x0"]), 3, calls))
    try:
        assert (grp.results()["status_code"] == 1).all()
        clean = grp.adjoint_cp(*g)
        calls["arm"] = True
        got = grp.adjoint_cp(*g)
    finally:
        grp.close()
    for k in got:
        assert np.isnan(got[k][3]).all(), k
        rest = np.arange(B) != 3
        assert np.array_equal(got[k][rest], clean[k][rest]), k


def test_adjoint_cp_re_raises_exceptions_from_F():
    family, B, n = "qcqp", 6, 6
    d = cpp.cp_batch_data(family, range(500, 500 + B), n, 0, 2)
    F0 = cpp.torch_F(family, d["data"], d["x0"], rowwise=True)
    state = {}

    class Boom(Exception):
        pass

    def F(x=None, z=None, idx=None):
        if state.get("raise") and z is not None:
            raise Boom("from F")
        return F0(x, z, idx=idx)
    g = _grads(B, n, 0, 3 + d["G"].shape[1], 23)
    grp = _cp_group(family, d, nsub=1, F=F)
    try:
        r0 = grp.results()
        a0 = grp.adjoint_cp(*g)
        state["raise"] = True
        with pytest.raises(Boom, match="from F"):
            grp.adjoint_cp(*g)
        state["raise"] = False
        r1 = grp.results()
        a1 = grp.adjoint_cp(*g)
        grp.solve()
        r2 = grp.results()
    finally:
        grp.close()
    for k in ("x", "y", "s", "z", "status_code", "iterations", "primal objective", "dual objective"):
        assert np.array_equal(r0[k], r1[k]) and np.array_equal(r0[k], r2[k]), k
    for k in a0:
        assert np.array_equal(a0[k], a1[k]), k


def test_adjoint_cp_bit_identical_across_compaction_and_subbatches(monkeypatch):
    family, B, n = "qcqp", 9, 6
    d = cpp.cp_batch_data(family, range(600, 600 + B), n, 0, 3)
    g = _grads(B, n, 0, 3 + d["G"].shape[1], 29)

    def run(nsub):
        grp = _cp_group(family, d, nsub=nsub, rowwise=True)
        try:
            return grp.results(), grp.adjoint_cp(*g)
        finally:
            grp.close()
    r1, a1 = run(1)
    assert len(set(r1["iterations"].tolist())) > 1
    monkeypatch.setenv("CVXB_BATCH_COMPACT", "0")
    r0, a0 = run(1)
    monkeypatch.delenv("CVXB_BATCH_COMPACT")
    for k in a1:
        assert np.array_equal(a0[k], a1[k]), k
    r2, a2 = run(2)
    r3, a3 = run(3)
    # a problem whose results differ between the two splits ran alone at the end of a sub-batch
    same = [j for j in range(B) if all(np.array_equal(r2[k][j], r3[k][j]) for k in ("x", "y", "s", "z"))]
    assert len(same) >= B // 2
    for k in a1:
        assert np.array_equal(a2[k][same], a3[k][same]), k


def test_adjoint_cp_spaces_and_repeats():
    import torch
    from cvxopt_b200 import CPLBatch
    family, B, n, q, ml, p = "socp", 7, 8, [3, 4], 2, 1
    d = cplp.cpl_batch_data(family, range(700, 700 + B), n, q, ml, p)
    mnl, cd = cplp.MNL[family], d["G"].shape[1]
    m = mnl + cd
    g = _grads(B, n, p, m, 31)
    cb = CPLBatch(B, n, mnl, _full(d["dims"]), p, 0)
    try:
        cb.set_F(cplp.torch_F(family, d["data"], d["x0"]))
        cb.load(d["c"], d["x0"], d["G"], d["h"], d["A"], d["b"])
        cb.solve()
        host = cb.adjoint_cp(*g)
        again = cb.adjoint_cp(*g)
        dev = torch.device("cuda", 0)
        gd = [torch.from_numpy(a).to(dev) for a in g]
        outs = [torch.full(s, 7.0, dtype=torch.float64, device=dev)
                for s in ((B, n), (B, p), (B, m), (B, n, cd), (B, n, p))]
        torch.cuda.synchronize()
        cb.adjoint_cp_ptr(*(t.data_ptr() for t in gd), *(t.data_ptr() for t in outs))
        o = [t.cpu().numpy() for t in outs]
    finally:
        cb.close()
    on_dev = {"ux": o[0], "c": -o[0], "b": o[1], "uznl": o[2][:, :mnl], "h": o[2][:, mnl:],
              "G": o[3].transpose(0, 2, 1), "A": o[4].transpose(0, 2, 1)}
    for k in host:
        assert np.array_equal(host[k], again[k]), k
        assert np.array_equal(host[k], on_dev[k]), k


def test_adjoint_cp_call_contract():
    import cvxopt_b200
    import torch
    from cvxopt_b200 import CPBatch, GPBatch, QCQPBatch, QPBatch, _lib
    family, B, n, p, r = "entropy", 5, 10, 2, 4
    d = cpp.cp_batch_data(family, range(800, 800 + B), n, p, r)
    ml = d["G"].shape[1]
    m = ml
    g = _grads(B, n, p, m, 37)
    lib = _lib.load()
    before = lib.cvxb_device_bytes()
    cb = CPBatch(B, n, 0, ml, p, 0)
    try:
        cb.set_F(cpp.torch_F(family, d["data"], d["x0"]))
        with pytest.raises(ValueError, match="no completed"):
            cb.adjoint_cp(*g)
        cb.load(d["x0"], d["G"], d["h"], d["A"], d["b"])
        with pytest.raises(ValueError, match="no completed"):
            cb.adjoint_cp(*g)
        cb.solve()
        # the other adjoint entry points refuse a CP batch
        with pytest.raises(NotImplementedError, match="'l'"):
            QPBatch.adjoint_ptr(cb)
        with pytest.raises(NotImplementedError, match="QP and cone LP"):
            QPBatch.adjoint_cone_ptr(cb)
        with pytest.raises(NotImplementedError, match="QCQP"):
            QCQPBatch.adjoint_ptr(cb)
        with pytest.raises(NotImplementedError, match="GP"):
            GPBatch.adjoint_gp_ptr(cb)
        full = cb.adjoint_cp(*g)
        zero = cb.adjoint_cp(g[0], np.zeros((B, p)), np.zeros((B, m)))
        null = cb.adjoint_cp(g[0])
        for k in full:
            assert np.array_equal(zero[k], null[k]), k
        dev = torch.device("cuda", 0)
        gd = [torch.from_numpy(a).to(dev) for a in g]
        guard = 4096
        uz = torch.full((B * m + guard,), 7.0, dtype=torch.float64, device=dev)
        dG = torch.full((B * n * ml + guard,), 7.0, dtype=torch.float64, device=dev)
        torch.cuda.synchronize()
        c0 = cvxopt_b200.launch_count()
        cb.adjoint_cp_ptr(*(t.data_ptr() for t in gd), uz=uz.data_ptr())
        c1 = cvxopt_b200.launch_count()
        cb.adjoint_cp_ptr(*(t.data_ptr() for t in gd), uz=uz.data_ptr(), dG=dG.data_ptr())
        c2 = cvxopt_b200.launch_count()
        assert c2 - c1 == (c1 - c0) + 1, "dG: k_adj_qc_grad and nothing else"
        print("\ncp adjoint launches (B=%d, n=%d, ml=%d, p=%d): %d without dG and dA, %d with dG"
              % (B, n, ml, p, c1 - c0, c2 - c1))
        if LAUNCHES is not None:
            assert c2 - c1 == LAUNCHES
        u, GG = uz.cpu().numpy(), dG.cpu().numpy()
        assert (u[B * m:] == 7.0).all() and (GG[B * n * ml:] == 7.0).all()
        assert np.array_equal(u[:B * m].reshape(B, m), full["h"])
        assert np.array_equal(GG[:B * n * ml].reshape(B, n, ml).transpose(0, 2, 1), full["G"])
        only = cb.adjoint_cp(*g, want=("A",))
        assert set(only) == {"A"} and np.array_equal(only["A"], full["A"])
        cb.load(d["x0"], d["G"], d["h"], d["A"], d["b"])
        with pytest.raises(ValueError, match="no completed"):
            cb.adjoint_cp(*g)
    finally:
        cb.close()
    assert lib.cvxb_device_bytes() == before


# launches of one adjoint call with dG on test_adjoint_cp_call_contract's batch (5 entropy problems, n = 10, ml = 4,
# p = 2)
LAUNCHES = 42


def _refused(batch):
    from cvxopt_b200 import CPBatch
    with pytest.raises(NotImplementedError, match="CP and cpl"):
        CPBatch.adjoint_cp_ptr(batch)
    batch.close()


def test_adjoint_cp_refuses_other_batches():
    from cvxopt_b200 import ConeLPBatch, GPBatch, QCQPBatch, QPBatch
    _refused(QPBatch(3, 5, 7, 0))
    _refused(ConeLPBatch(3, 5, 8, 0))
    _refused(GPBatch(3, 5, [3, 2], 4))
    _refused(QCQPBatch(3, 5, 1, 4))
    # QCQPBatch.adjoint_cp exists by inheritance and is the entry point's refusal, not a second QCQP adjoint
    qb = QCQPBatch(3, 5, 1, 4)
    try:
        with pytest.raises(NotImplementedError, match="CP and cpl"):
            qb.adjoint_cp(np.zeros((3, 5)))
    finally:
        qb.close()


def _logistic_param_F(x0, counts=None):
    """the logistic family's F with the samples a as the param"""
    import torch

    def F(x=None, z=None, idx=None, params=()):
        if x is None:
            return 1, x0
        if counts is not None:
            counts["theta" if torch.is_grad_enabled() and params[0].requires_grad else
                   "xz" if z is not None else "x"] += 1
        a, y = params
        return cpp.torch_F("logistic", {"a": a, "y": y}, x0)(x, z, idx=idx)
    return F


def test_cp_layer_backward_equals_group_adjoint_and_theta_formula():
    import torch
    from cvxopt_b200 import cp_layer
    B, n = 12, 6
    d = cpp.cp_batch_data("logistic", range(900, 900 + B), n)
    x0 = torch.from_numpy(d["x0"]).cuda()
    a, y = _torch(d["data"]["a"], d["data"]["y"])
    a.requires_grad_()
    counts = {"x": 0, "xz": 0, "theta": 0}
    gx = torch.from_numpy(_grads(B, n, 0, 1, 41)[0]).cuda()
    gz = torch.from_numpy(_grads(B, n, 0, 1, 43)[2]).cuda()
    x, _, znl, zl, st = cp_layer(_logistic_param_F(x0, counts), (a, y), nsub=3)
    assert (st == 1).all()
    before = dict(counts)
    (ga,) = torch.autograd.grad((x * gx).sum() + (znl * gz).sum(), (a,))
    assert counts["xz"] - before["xz"] == 3 and counts["theta"] - before["theta"] == 1
    assert counts["x"] == before["x"]
    grp = _cp_group("logistic", d, nsub=3)
    try:
        res = grp.results()
        want = grp.adjoint_cp(gx.cpu().numpy(), None, gz.cpu().numpy(), want=("ux", "uznl"))
    finally:
        grp.close()
    assert np.array_equal(x.detach().cpu().numpy(), res["x"])
    # the theta formula by hand: -d_a [ux' Df' zk + uk' f]
    ux, uz = (torch.from_numpy(want[k]).cuda() for k in ("ux", "uznl"))
    zk = torch.cat([torch.ones((B, 1), dtype=torch.float64, device="cuda"), znl.detach()], 1)
    uk = torch.cat([torch.zeros((B, 1), dtype=torch.float64, device="cuda"), uz], 1)
    aa = a.detach().clone().requires_grad_()
    f, Df = cpp.torch_F("logistic", {"a": aa, "y": y}, x0)(x.detach(), idx=torch.arange(B, device="cuda"))
    (gw,) = torch.autograd.grad((Df * (zk[:, :, None] * ux[:, None, :])).sum() + (uk * f).sum(), (aa,))
    assert torch.allclose(ga, -gw, rtol=1e-12, atol=1e-14)
    # y is used by F and needs no gradient: no theta call at all without a param that needs one
    counts.update(x=0, xz=0, theta=0)
    x, *_ = cp_layer(_logistic_param_F(x0, counts), (a.detach(), y), nsub=1)
    assert not x.requires_grad and counts["theta"] == 0


def test_cp_layer_params_match_central_differences_of_its_forward():
    """the user's view: loss = cp_layer(F, (a,), G, h)[0].square().sum() with a logistic F and a.requires_grad_()
    gives finite gradients, equal to central differences of the layer's own forward"""
    import torch
    from cvxopt_b200 import cp_layer
    B, n = 4, 5
    d = cpp.cp_batch_data("logistic", range(1000, 1000 + B), n)
    x0 = torch.from_numpy(d["x0"]).cuda()
    a, y = _torch(d["data"]["a"], d["data"]["y"])
    G, h = _torch(np.tile(np.eye(n)[None], (B, 1, 1)), np.full((B, n), 0.3))
    a.requires_grad_()
    tight = dict(abstol=1e-11, reltol=1e-11, feastol=1e-11)
    loss = cp_layer(_logistic_param_F(x0), (a, y), G, h, **tight)[0].square().sum()
    loss.backward()
    assert torch.isfinite(a.grad).all()
    rng = np.random.default_rng(5)
    for _ in range(2):
        D = torch.from_numpy(rng.standard_normal(a.shape)).cuda()
        eps = 1e-5
        with torch.no_grad():
            lp = cp_layer(_logistic_param_F(x0), (a + eps * D, y), G, h, **tight)[0].square().sum()
            lm = cp_layer(_logistic_param_F(x0), (a - eps * D, y), G, h, **tight)[0].square().sum()
        fd = float((lp - lm) / (2 * eps))
        an = float((a.grad * D).sum())
        print("\ncp_layer d/da: fd %.10e adjoint %.10e" % (fd, an))
        assert abs(fd - an) <= 1e-6 * max(abs(fd), abs(an)), (fd, an)


def test_cpl_layer_with_s_blocks_and_an_unused_param():
    import torch
    from cvxopt_b200 import cpl_layer
    family, B, n, q, s, ml = "socp", 6, 8, [3], [3], 2
    d = sdcpl_batch_data(family, range(1100, 1100 + B), n, q, s, ml, 0)
    dims = _full(d["dims"])
    x0 = torch.from_numpy(d["x0"]).cuda()
    P, qv, c, G, h = _torch(d["data"]["P"], d["data"]["q"], d["c"], d["G"], d["h"])
    unused = torch.ones((B, 2), dtype=torch.float64, device="cuda", requires_grad=True)
    t = [v.requires_grad_() for v in (P, qv, c, G, h)]

    def F(x=None, z=None, idx=None, params=()):
        if x is None:
            return 2, x0
        return cplp.torch_F(family, {"P": params[0], "q": params[1]}, x0)(x, z, idx=idx)
    x, _, znl, zl, st = cpl_layer(t[2], F, (t[0], t[1], unused), t[3], t[4], dims)
    assert (st == 1).all()
    gx = torch.from_numpy(_grads(B, n, 0, 1, 47)[0]).cuda()
    grads = torch.autograd.grad((x * gx).sum(), t + [unused])
    assert all(torch.isfinite(v).all() for v in grads[:5])
    assert torch.equal(grads[5], torch.zeros_like(unused))
    grp = _cpl_group(family, d)
    try:
        want = grp.adjoint_cp(gx.cpu().numpy())
    finally:
        grp.close()
    for k, v in zip(("c", "G", "h"), grads[2:5]):
        assert np.array_equal(v.cpu().numpy(), want[k]), k


def test_cp_layer_work_streams_and_memory():
    import cvxopt_b200
    import torch
    from cvxopt_b200 import _lib, cp_layer
    family, B, n, p, r = "entropy", 8, 10, 2, 4
    d = cpp.cp_batch_data(family, range(1200, 1200 + B), n, p, r)
    F0 = cpp.torch_F(family, d["data"], d["x0"])

    def F(x=None, z=None, idx=None, params=()):
        return F0(x, z, idx=idx) if x is not None else F0()
    gx = torch.from_numpy(_grads(B, n, 0, 1, 53)[0]).cuda()
    lib = _lib.load()
    before = lib.cvxb_device_bytes()

    def run(needs, stream=None):
        with torch.cuda.stream(stream):
            t = _torch(d["G"], d["h"], d["A"], d["b"])
            for v, need in zip(t, needs):
                v.requires_grad_(need)
            x, *_ = cp_layer(F, (), *t, nsub=1)
            c0 = cvxopt_b200.launch_count()
            grads = torch.autograd.grad((x * gx).sum(), [v for v, need in zip(t, needs) if need])
            torch.cuda.synchronize()
        return grads, cvxopt_b200.launch_count() - c0
    full, c_full = run([True] * 4)
    assert lib.cvxb_device_bytes() == before
    vec, c_vec = run([False, True, False, True])
    assert c_vec == c_full - 1, "no matrix output: no k_adj_qc_grad"
    for u, v in zip(vec, (full[1], full[3])):
        assert torch.equal(u, v)
    on_side, _ = run([True] * 4, torch.cuda.Stream())
    for u, v in zip(on_side, full):
        assert torch.equal(u, v)
    t = _torch(d["G"], d["h"], d["A"], d["b"])
    x, *_ = cp_layer(F, (), *t, nsub=1)
    assert not x.requires_grad and lib.cvxb_device_bytes() == before


def test_layers_with_only_unused_params_and_with_mnl_zero():
    """a param that F never reads gets zeros when it is the only one that needs a gradient, on cp_layer and on a
    cpl_layer without nonlinear rows (mnl = 0: f and Df are empty), and the other gradients are the group's adjoint's"""
    import torch
    from cvxopt_b200 import cp_layer, cpl_layer
    B, n = 6, 8
    d = cpp.cp_batch_data("entropy", range(1300, 1300 + B), n, 2, 3)
    F0 = cpp.torch_F("entropy", d["data"], d["x0"])
    unused = torch.ones((B, 3), dtype=torch.float64, device="cuda", requires_grad=True)
    G, h, A, b = [v.requires_grad_() for v in _torch(d["G"], d["h"], d["A"], d["b"])]
    gx = torch.from_numpy(_grads(B, n, 0, 1, 59)[0]).cuda()
    x, _, _, _, st = cp_layer(lambda x=None, z=None, idx=None, params=(): F0(x, z, idx=idx) if x is not None else F0(),
                              (unused,), G, h, A, b)
    assert (st == 1).all()
    grads = torch.autograd.grad((x * gx).sum(), [unused, G, h, A, b])
    assert torch.equal(grads[0], torch.zeros_like(unused))
    grp = _cp_group("entropy", d)
    try:
        want = grp.adjoint_cp(gx.cpu().numpy())
    finally:
        grp.close()
    for k, v in zip(("G", "h", "A", "b"), grads[1:]):
        assert np.array_equal(v.cpu().numpy(), want[k]), k
    # cpl with mnl = 0: the conelp family (F returns empty f and Df, H = 0)
    e = cplp.cpl_batch_data("conelp", range(1400, 1400 + B), n, [3], 3, 0)
    E0 = cplp.torch_F("conelp", e["data"], e["x0"])
    c, Ge, he = [v.requires_grad_() for v in _torch(e["c"], e["G"], e["h"])]
    x, _, znl, _, st = cpl_layer(c, lambda x=None, z=None, idx=None, params=(): E0(x, z, idx=idx) if x is not None
                                 else E0(), (unused,), Ge, he, _full(e["dims"]))
    assert (st == 1).all() and znl.shape == (B, 0)
    grads = torch.autograd.grad((x * gx).sum(), [unused, c, Ge, he])
    assert torch.equal(grads[0], torch.zeros_like(unused))
    grp = _cpl_group("conelp", e)
    try:
        want = grp.adjoint_cp(gx.cpu().numpy())
    finally:
        grp.close()
    for k, v in zip(("c", "G", "h"), grads[1:]):
        assert np.array_equal(v.cpu().numpy(), want[k]), k


def test_adjoint_cp_strongly_active_constraint_refines_to_the_dense_solve(ref):
    """the case _one_slack_row steers the dense-solve test away from, checked for what it is: the logistic family
    without 'l' rows ends with its ball constraint's s / z near 1e-15, where the adjoint's one refinement step leaves
    some problems far from the dense solve (DESIGN.md's known limit).  The operator is the dense one: refinement steps
    taken here, residuals of the dense M with the adjoint itself as the inner solve, converge to the dense solution"""
    fam, n, B = "logistic", 8, 8
    d = cpp.cp_batch_data(fam, range(100, 100 + B), n)
    grp = _cp_group(fam, d, nsub=1)
    try:
        res = grp.results()
        assert (res["status_code"] == 1).all()
        g = _grads(B, n, 0, 1, 7)
        u = grp.adjoint_cp(*g, want=("ux", "uznl"))
        want, _ = _oracle(_cp_eval(fam, d), True, d, {"l": 0, "q": [], "s": []}, 1, res, g)
        first = max(_rel(u["ux"][j], want["ux"][j]) for j in range(B))
        for _ in range(3):
            rx, rz = np.zeros((B, n)), np.zeros((B, 1))
            for j in range(B):
                s, z = res["s"][j], res["z"][j]
                _, Df, H = cpp._eval_np(fam, {k: v[j] for k, v in d["data"].items()}, res["x"][j],
                                        np.array([1.0, z[0]]))
                rx[j] = g[0][j] - (H @ u["ux"][j] + Df[1:].T @ u["uznl"][j])
                rz[j] = g[2][j] - (Df[1:] @ u["ux"][j] - (s / z) * u["uznl"][j])
            du = grp.adjoint_cp(rx, None, rz, want=("ux", "uznl"))
            u = {k: u[k] + du[k] for k in u}
    finally:
        grp.close()
    last = max(_rel(u["ux"][j], want["ux"][j]) for j in range(B))
    print("\nlogistic without 'l' rows: s / z down to %.0e; ux from the dense solve %.1e after one refinement step, "
          "%.1e after three more" % ((res["s"] / res["z"]).min(), first, last))
    assert last <= 1e-6 and last < first
