"""Warm starts of the batch solvers (cvxb_batch_load_start: qp_batch / coneqp_batch's initvals, conelp_batch /
sdp_batch's primalstart and dualstart) against a Python loop over the reference's solvers.coneqp(..., initvals),
solvers.conelp(..., primalstart, dualstart) and solvers.sdp (oracle/_ref), given the same starts: converged solutions,
iterates, iteration 0's factorisation, the positivity checks, the re-solve use case and the batch mechanics."""
import os
import sys

import numpy as np
import pytest

from problems import cone_point
from test_batch_conelp_gpu import TOL, _rel
from test_batch_sdp_gpu import _full, _sym, sdp_batch_data
from test_batch_sdp_gpu import assert_matches as assert_lp_matches
from test_batch_sdqp_gpu import assert_matches as assert_qp_matches
from test_batch_sdqp_gpu import sdqp_batch_data

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
from batch_warm_bench import push_interior  # noqa: E402

pytestmark = pytest.mark.gpu

DIMS = [{"l": 30}, {"l": 10, "q": [4, 3]}, {"l": 6, "q": [3], "s": [4, 3]}]
N = 12


def cdim(dims):
    d = _full(dims)
    return d["l"] + sum(d["q"]) + sum(k * k for k in d["s"])


def make_start(B, n, p, dims, seed, keys):
    """x, y ~ N(0, 1), s and z strictly inside the cones; only `keys`"""
    rng = np.random.Generator(np.random.PCG64(seed))
    v = {"x": rng.standard_normal((B, n)), "y": rng.standard_normal((B, p)),
         "s": np.stack([cone_point(_full(dims), rng) for _ in range(B)]),
         "z": np.stack([cone_point(_full(dims), rng) for _ in range(B)])}
    return {k: v[k] for k in keys}


def _m(v):
    from cvxopt import matrix
    return matrix(np.ascontiguousarray(v, dtype=np.float64))


def ref_qp_loop(batch, dims, initvals, **options):
    from cvxopt import solvers
    P, q, G, h, A, b = batch
    out = []
    for k in range(P.shape[0]):
        iv = None if initvals is None else {key: _m(v[k]) for key, v in initvals.items()}
        eq = (_m(A[k]), _m(b[k])) if A.shape[1] else (None, None)
        out.append(solvers.coneqp(_m(P[k]), _m(q[k]), _m(G[k]), _m(h[k]), _full(dims), *eq, initvals=iv,
                                  options=dict(show_progress=False, **options)))
    return out


def ref_lp_loop(batch, dims, ps, ds, **options):
    from cvxopt import solvers
    c, G, h, A, b = batch
    d = _full(dims)
    kw = {"kktsolver": "chol"} if d["q"] or d["s"] else {}
    out = []
    for k in range(c.shape[0]):
        pk = None if ps is None else {key: _m(v[k]) for key, v in ps.items()}
        dk = None if ds is None else {key: _m(v[k]) for key, v in ds.items()}
        eq = (_m(A[k]), _m(b[k])) if A.shape[1] else (None, None)
        out.append(solvers.conelp(_m(c[k]), _m(G[k]), _m(h[k]), d, *eq, primalstart=pk, dualstart=dk,
                                  options=dict(show_progress=False, **options), **kw))
    return out


def qp_solve(batch, dims, initvals, nsub=None, **options):
    import cvxopt_b200
    P, q, G, h, A, b = batch
    eq = dict(A=A, b=b) if A.shape[1] else {}
    return cvxopt_b200.coneqp_batch(P, q, G, h, dims, nsub=nsub, initvals=initvals, **eq, **options)


def lp_solve(batch, dims, ps, ds, nsub=None, **options):
    from cvxopt_b200 import SDPBatchGroup, batch as bt
    c, G, h, A, b = batch
    B, n = c.shape
    p = A.shape[1]
    start = bt._lp_start(ps, ds, B, n, p, cdim(dims))
    return bt._run_group(SDPBatchGroup(B, n, dims, p, 0, nsub), (c, G, h, A if p else None, b if p else None),
                         options, start)


QP_KEYS = [("x", "s", "y", "z"), (), ("x",), ("s", "z"), ("y",)]


@pytest.mark.parametrize("dims", DIMS)
@pytest.mark.parametrize("p", [0, 3])
@pytest.mark.parametrize("keys", QP_KEYS)
def test_coneqp_initvals_match_coneqp(ref, dims, p, keys):
    if p == 0 and "y" in keys:
        keys = tuple(k for k in keys if k != "y")
        if not keys:
            pytest.skip("y only needs p > 0")
    batch = sdqp_batch_data(3, N, dims, p, 200 + 10 * p + len(keys), pkind="random")
    iv = make_start(3, N, p, dims, 300 + p, keys)
    got = qp_solve(batch, dims, iv)
    want = ref_qp_loop(batch, dims, iv)
    assert all(w["status"] == "optimal" for w in want), [w["status"] for w in want]
    assert_qp_matches(got, dims, want)


LP_CASES = ["primal", "dual", "both", "dual_no_y"]


def shift_inside(v, dims):
    """v + (1 + max(0, t)) e per problem, t the largest step of misc.max_step: conelp's own shift of its start"""
    d = _full(dims)
    out = v.copy()
    for k in range(v.shape[0]):
        t, o = [], d["l"]
        if d["l"]:
            t.append(-v[k, :d["l"]].min())
        for j in d["q"]:
            t.append(np.linalg.norm(v[k, o + 1:o + j]) - v[k, o])
            o += j
        for j in d["s"]:
            t.append(-np.linalg.eigvalsh(v[k, o:o + j * j].reshape(j, j, order="F")).min())
            o += j * j
        out[k:k + 1] = v[k:k + 1] + (push_interior(np.zeros((1, v.shape[1])), dims, 1.0) * (1.0 + max(0.0, *t)))
    return out


def lp_start(B, n, p, dims, seed, case, batch=None):
    """random starts; with `batch`, the primal start is x and s = h - G x shifted inside the cones"""
    v = make_start(B, n, p, dims, seed, ("x", "s", "y", "z"))
    if batch is not None:
        c, G, h, A, b = batch
        v["s"] = shift_inside(h - np.einsum("bij,bj->bi", G, v["x"]), dims)
    ps = {"x": v["x"], "s": v["s"]} if case in ("primal", "both") else None
    ds = None
    if case in ("dual", "both"):
        ds = {"y": v["y"], "z": v["z"]} if p else {"z": v["z"]}
    if case == "dual_no_y":
        ds = {"z": v["z"]}
    return ps, ds


@pytest.mark.parametrize("dims", DIMS)
@pytest.mark.parametrize("p", [0, 3])
@pytest.mark.parametrize("case", LP_CASES)
def test_conelp_starts_match_conelp(ref, dims, p, case):
    if case == "dual_no_y" and p == 0:
        pytest.skip("the same as 'dual' without equality rows")
    batch = sdp_batch_data(3, N, dims, p, 500 + 10 * p + LP_CASES.index(case))
    ps, ds = lp_start(3, N, p, dims, 600 + p, case, batch)
    got = lp_solve(batch, dims, ps, ds)
    want = ref_lp_loop(batch, dims, ps, ds)
    assert all(w["status"] == "optimal" for w in want), [w["status"] for w in want]
    if (case, p, dims) == ("primal", 3, DIMS[1]):
        # problem 1 ends at a gap of 8e-9.  One iteration before, the batch's elimination of the equality rows (kkt_chol2's)
        # finds Kp singular where the reference's 'chol' (QR of A') does not, and stops with status 3.  The start is
        # not involved: every iterate up to that one matches.
        k = want[1]["iterations"] - 1
        g, w = lp_solve(batch, dims, ps, ds, maxiters=k), ref_lp_loop(batch, dims, ps, ds, maxiters=k)
        for key in ("x", "y", "s", "z"):
            assert _rel(g[key][1], np.array(w[1][key]).ravel()) <= TOL, key
        assert got["status_code"][1] == 3
        keep = [0, 2]
        got = {key: (v[keep] if isinstance(v, np.ndarray) and v.ndim and v.shape[0] == 3 else
                     [v[j] for j in keep] if key == "status" else v) for key, v in got.items()}
        batch, want = [x[keep] for x in batch], [want[j] for j in keep]
    assert_lp_matches(got, batch, dims, want)


def test_wrappers_pass_the_starts(ref):
    """qp_batch, conelp_batch and sdp_batch hand their keywords to load_start as coneqp_batch does"""
    import cvxopt_b200
    dims, p = {"l": 10, "q": [4, 3]}, 2
    P, q, G, h, A, b = batch = sdqp_batch_data(3, N, dims, p, 800, pkind="random")
    iv = make_start(3, N, p, dims, 801, ("x", "z"))
    got = cvxopt_b200.qp_batch(P, q, G, h, A, b, dims=dims, initvals=iv)
    assert_qp_matches(got, dims, ref_qp_loop(batch, dims, iv))
    lb = sdp_batch_data(3, N, dims, p, 802)
    ps, ds = lp_start(3, N, p, dims, 803, "both")
    got = cvxopt_b200.conelp_batch(*lb[:3], dims=dims, A=lb[3], b=lb[4], primalstart=ps, dualstart=ds)
    assert_lp_matches(got, lb, dims, ref_lp_loop(lb, dims, ps, ds))
    sd = {"l": 4, "s": [3, 5]}
    c, Gf, hf, A, b = lb = sdp_batch_data(3, N, sd, 1, 804)
    v = make_start(3, N, 1, sd, 805, ("x", "s", "z"))
    blocks = lambda w: [w[:, 4:13].reshape(3, 3, 3).transpose(0, 2, 1), w[:, 13:].reshape(3, 5, 5).transpose(0, 2, 1)]
    Gs = [Gf[:, 4:13], Gf[:, 13:]]
    hs = [hf[:, 4:13].reshape(3, 3, 3).transpose(0, 2, 1), hf[:, 13:].reshape(3, 5, 5).transpose(0, 2, 1)]
    got = cvxopt_b200.sdp_batch(c, Gf[:, :4], hf[:, :4], Gs, hs, A, b, primalstart={"x": v["x"], "sl": v["s"][:, :4],
                                "ss": blocks(v["s"])}, dualstart={"zl": v["z"][:, :4], "zs": blocks(v["z"])})
    want = ref_lp_loop(lb, sd, {"x": v["x"], "s": v["s"]}, {"z": v["z"]})
    for k, w in enumerate(want):
        assert got["status"][k] == w["status"] and got["iterations"][k] == w["iterations"]
        np.testing.assert_allclose(got["x"][k], np.array(w["x"]).ravel(), rtol=1e-6, atol=1e-8)
        np.testing.assert_allclose(got["zl"][k], np.array(w["z"]).ravel()[:4], rtol=1e-5, atol=1e-7)


def test_iterates_match_after_1_2_3_iterations(ref):
    dims, p = {"l": 6, "q": [3], "s": [4, 3]}, 2
    qb = sdqp_batch_data(3, N, dims, p, 900, pkind="random")
    iv = make_start(3, N, p, dims, 901, ("x", "s", "y", "z"))
    lb = sdp_batch_data(3, N, dims, p, 902)
    ps, ds = lp_start(3, N, p, dims, 903, "both")
    worst = 0.0
    for k in (1, 2, 3):
        for got, want in ((qp_solve(qb, dims, iv, maxiters=k), ref_qp_loop(qb, dims, iv, maxiters=k)),
                          (lp_solve(lb, dims, ps, ds, maxiters=k), ref_lp_loop(lb, dims, ps, ds, maxiters=k))):
            for j, w in enumerate(want):
                assert w["iterations"] == k and got["iterations"][j] == k
                for key in ("x", "y", "s", "z"):
                    wv = np.array(w[key]).ravel()
                    d = _rel(got[key][j], _sym(wv, dims) if key in ("s", "z") else wv)
                    assert d <= TOL, (j, k, key, d)
                    worst = max(worst, d)
    print("\nwarm-started iterates: largest relative difference %.2e" % worst)


def test_start_at_an_optimum_ends_at_iteration_0(ref):
    """problem 1 starts from the reference's own solution and is 'optimal' after 0 iterations; it leaves the batch
    before the first factorisation while problems 0 and 2 iterate"""
    dims, p = {"l": 10, "q": [4, 3]}, 2
    batch = sdqp_batch_data(3, N, dims, p, 1000, pkind="random")
    cold = ref_qp_loop(batch, dims, None)
    iv = make_start(3, N, p, dims, 1001, ("x", "s", "y", "z"))
    for key in iv:
        iv[key][1] = np.array(cold[1][key]).ravel()
    want = ref_qp_loop(batch, dims, iv)
    assert want[1]["iterations"] == 0 and want[1]["status"] == "optimal"
    for nsub in (1, 3):
        got = qp_solve(batch, dims, iv, nsub=nsub)
        assert_qp_matches(got, dims, want)


def _switch_batch(seed, lp):
    """'l'-only problems with p = 4 whose G has zero columns 12..15 in problems 1 and 3, so that P + G'DG is singular
    at iteration 0 but S + A'A is not"""
    n, m, p = 16, 40, 4
    rng = np.random.Generator(np.random.PCG64(seed))
    B = 4
    G, A = rng.standard_normal((B, m, n)), rng.standard_normal((B, p, n))
    x0, s0, z0, y0 = (rng.standard_normal((B, n)), rng.uniform(0.5, 1.5, (B, m)), rng.uniform(0.5, 1.5, (B, m)),
                      rng.standard_normal((B, p)))
    for j in (1, 3):
        G[j][:, 12:] = 0.0
    h = np.einsum("bij,bj->bi", G, x0) + s0
    b = np.einsum("bij,bj->bi", A, x0)
    c = -(np.einsum("bji,bj->bi", G, z0) + np.einsum("bji,bj->bi", A, y0))
    if lp:
        return c, G, h, A, b
    P = np.zeros((B, n, n))
    for j in (0, 2):
        M = rng.standard_normal((n, n))
        P[j] = M @ M.T / n
    return P, c, G, h, A, b


def test_iteration_0_takes_the_s_plus_ata_switch(ref):
    """the reference's kkt_chol2 (solvers.qp / solvers.lp) switches to S + A'A where S is singular at its first call,
    which a loaded start makes iteration 0's"""
    dims = {"l": 40}
    qb = _switch_batch(1100, lp=False)
    for j in (1, 3):
        with pytest.raises(np.linalg.LinAlgError):
            np.linalg.cholesky(qb[2][j].T @ qb[2][j])
    for iv in ({}, make_start(4, 16, 4, dims, 1101, ("s", "z"))):
        want = ref_qp_loop(qb, dims, iv)
        assert all(w["status"] == "optimal" for w in want)
        assert_qp_matches(qp_solve(qb, dims, iv, nsub=1), dims, want)
    lb = _switch_batch(1102, lp=True)
    ps, ds = lp_start(4, 16, 4, dims, 1103, "both")
    want = ref_lp_loop(lb, dims, ps, ds)
    assert all(w["status"] == "optimal" for w in want)
    assert_lp_matches(lp_solve(lb, dims, ps, ds, nsub=1), lb, dims, want)


def test_singular_iteration_0_raises_the_rank_error():
    dims = {"l": 8, "s": [3]}
    P, q, G, h, A, b = sdqp_batch_data(3, 12, dims, 2, 1200, pkind="zero")
    G[1][:, 5] = 0.0                       # x[5] appears nowhere: every KKT matrix of problem 1 is singular
    A[1][:, 5] = 0.0
    with pytest.raises(ValueError, match=r"problem 1: Rank\(A\) < p or Rank\(\[P; A; G\]\) < n"):
        qp_solve((P, q, G, h, A, b), dims, {}, nsub=1)
    c, G, h, A, b = sdp_batch_data(3, 12, dims, 2, 1201)
    G[2][:, 5] = 0.0
    A[2][:, 5] = 0.0
    ps, ds = lp_start(3, 12, 2, dims, 1202, "both")
    with pytest.raises(ValueError, match=r"problem 2: Rank\(A\) < p or Rank\(\[G; A\]\) < n"):
        lp_solve((c, G, h, A, b), dims, ps, ds, nsub=1)


@pytest.mark.parametrize("row,what", [(3, "s"), (10, "z"), (20, "s"), (22, "z")])
def test_a_start_outside_the_cone_raises(row, what):
    """dims {'l': 10, 'q': [4, 3], 's': [4]}: row 3 is an 'l' row, 10 the first 'q' cone's head, 20 the 's' block's
    entry (3, 0) and 22 its diagonal entry (1, 1)"""
    dims = {"l": 10, "q": [4, 3], "s": [4]}
    qb = sdqp_batch_data(3, N, dims, 0, 1300, pkind="random")
    iv = make_start(3, N, 0, dims, 1301, ("s", "z"))
    iv[what][1][row] = -50.0
    with pytest.raises(ValueError, match="problem 1: initial %s is not positive" % what):
        qp_solve(qb, dims, iv, nsub=1)
    lb = sdp_batch_data(3, N, dims, 0, 1302)
    ps, ds = lp_start(3, N, 0, dims, 1303, "primal" if what == "s" else "dual")
    (ps or ds)[what][1][row] = -50.0
    with pytest.raises(ValueError, match="problem 1: initial %s is not positive" % what):
        lp_solve(lb, dims, ps, ds, nsub=1)


@pytest.mark.parametrize("dims,p", [({"l": 30}, 3), ({"l": 6, "q": [3], "s": [4, 3]}, 2)])
def test_resolve_from_the_previous_solution(ref, dims, p):
    """solve, perturb h by 1e-3 relative, and re-solve warm from the previous x, y and the pushed s, z"""
    qb = sdqp_batch_data(4, N, dims, p, 1400, pkind="random")
    first = qp_solve(qb, dims, None)
    rng = np.random.Generator(np.random.PCG64(1401))
    P, q, G, h, A, b = qb
    h2 = h * (1.0 + 1e-3 * rng.standard_normal(h.shape))
    qb2 = (P, q, G, h2, A, b)
    iv = {"x": first["x"], "s": push_interior(first["s"], dims), "z": push_interior(first["z"], dims)}
    if p:
        iv["y"] = first["y"]
    want = ref_qp_loop(qb2, dims, iv)
    assert all(w["status"] == "optimal" for w in want)
    assert_qp_matches(qp_solve(qb2, dims, iv), dims, want)
    lb = sdp_batch_data(4, N, dims, p, 1402)
    first = lp_solve(lb, dims, None, None)
    c, G, h, A, b = lb
    lb2 = (c, G, h * (1.0 + 1e-3 * rng.standard_normal(h.shape)), A, b)
    ps = {"x": first["x"], "s": push_interior(first["s"], dims)}
    ds = {"z": push_interior(first["z"], dims)}
    if p:
        ds["y"] = first["y"]
    want = ref_lp_loop(lb2, dims, ps, ds)
    assert all(w["status"] == "optimal" for w in want)
    assert_lp_matches(lp_solve(lb2, dims, ps, ds), lb2, dims, want)


def test_batch_mechanics(ref, monkeypatch):
    """compaction, sub-batches, a second solve, the upper triangles of s and z, clear_start and device memory"""
    import cvxopt_b200 as cb
    from cvxopt_b200 import SDPQPBatch, _lib
    dims, p, B, n = {"l": 6, "q": [4], "s": [5, 3]}, 2, 9, 14
    m = cdim(dims)
    qb = sdqp_batch_data(B, n, dims, p, 1500)
    qb[1] *= np.linspace(0.1, 30.0, B)[:, None]
    iv = make_start(B, n, p, dims, 1501, ("x", "s", "y", "z"))
    base = qp_solve(qb, dims, iv, nsub=1)
    assert len(set(base["iterations"].tolist())) > 1
    monkeypatch.setenv("CVXB_BATCH_COMPACT", "0")
    flat = qp_solve(qb, dims, iv, nsub=1)
    monkeypatch.delenv("CVXB_BATCH_COMPACT")
    three = qp_solve(qb, dims, iv, nsub=3)
    junk = {k: v.copy() for k, v in iv.items()}
    rng = np.random.default_rng(3)
    o = 10
    for k in (5, 3):
        up = o + np.nonzero(np.triu(np.ones((k, k), dtype=bool), 1).reshape(-1, order="F"))[0]
        for key in ("s", "z"):
            junk[key][:, up] = rng.standard_normal((B, len(up)))
        o += k * k
    upper = qp_solve(qb, dims, junk, nsub=1)
    for key in ("x", "y", "s", "z", "iterations", "primal objective", "dual objective"):
        np.testing.assert_array_equal(flat[key], base[key], err_msg=key)
        np.testing.assert_array_equal(upper[key], base[key], err_msg=key)
        np.testing.assert_allclose(three[key], base[key], rtol=0, atol=1e-12 * (1 + np.abs(base[key]).max()))
    assert_qp_matches(base, dims, ref_qp_loop(qb, dims, iv))

    lib = _lib.load()
    P, q, G, h, A, b = qb
    before = lib.cvxb_device_bytes()
    cold = SDPQPBatch(B, n, dims, p=p)
    cold.load(P, q, G, h, A, b)
    cold.solve()
    l0 = cb.launch_count()
    cold.solve()                           # a second solve: it first restores the slot order, as warm's below does
    cold_launches = cb.launch_count() - l0
    want = cold.results()
    warm = SDPQPBatch(B, n, dims, p=p)
    created = lib.cvxb_device_bytes()
    warm.load(P, q, G, h, A, b)
    warm.load_start(**iv)
    assert lib.cvxb_device_bytes() - created == 8 * B * (n + p + 2 * m)
    warm.solve()
    r1 = warm.results()
    warm.load(P, q, G, h, A, b)            # the start outlives a load
    warm.load_start_ptr(None, None, None, None, _lib.HOST)
    warm.load_start(**iv)                  # a second load_start allocates nothing
    assert lib.cvxb_device_bytes() - created == 8 * B * (n + p + 2 * m)
    warm.solve()
    r2 = warm.results()
    for key in ("x", "y", "s", "z", "iterations"):
        np.testing.assert_array_equal(r1[key], base[key], err_msg=key)
        np.testing.assert_array_equal(r2[key], base[key], err_msg=key)
    warm.clear_start()
    l0 = cb.launch_count()
    warm.solve()
    assert cb.launch_count() - l0 == cold_launches
    r3 = warm.results()
    for key in ("x", "y", "s", "z", "iterations", "status_code", "primal objective", "dual objective"):
        np.testing.assert_array_equal(r3[key], want[key], err_msg=key)
    warm.close()
    cold.close()
    assert lib.cvxb_device_bytes() == before
