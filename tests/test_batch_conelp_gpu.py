"""Cone LP batches (conelp_batch, csrc/batch_ipm.cu's solve<CONES, EQ, LP> with LP = true) against a Python loop over
the reference's solvers.conelp(c, G, h, dims, A, b) (oracle/_ref): default kktsolver ('chol2') for 'l'-only problems,
kktsolver='chol' with 'q' cones (the reference's default there is 'qr').  Converged solutions, iterates, infeasibility
certificates, the S + A'A switch, the start, and the batch mechanics."""
import ctypes as C

import numpy as np
import pytest

from problems import cone_point
from test_batch_cones_gpu import _full

pytestmark = pytest.mark.gpu

TOL = 1e-10          # relative 2-norm difference of x, y, s and z per problem at k = 1..3 iterations


def lp_problem(n, dims, p, seed, kind="feasible"):
    """G, A, x0 ~ N(0,1); h = G x0 + s0, b = A x0, c = -(G'z0 + A'y0) with s0, z0 strictly inside the cones.
    'pinf': the first cone row (or 'q' block) reads 0 x + s = -e, so z = e_0 certifies primal infeasibility.
    'dinf': G d = -t (t inside the cones), A d = 0 and c'd < 0 for a direction d, so the LP is unbounded below."""
    dims = _full(dims)
    rng = np.random.Generator(np.random.PCG64(seed))
    m = dims["l"] + sum(dims["q"])
    G = rng.standard_normal((m, n))
    A = rng.standard_normal((p, n))
    x0, y0 = rng.standard_normal(n), rng.standard_normal(p)
    s0, z0 = cone_point(dims, rng), cone_point(dims, rng)
    if kind == "dinf":
        d = rng.standard_normal(n)
        if p:
            d -= A.T @ np.linalg.solve(A @ A.T, A @ d)
        t = cone_point(dims, rng)
        G += np.outer(-t - G @ d, d) / (d @ d)
    h = G @ x0 + s0
    c = -(G.T @ z0 + A.T @ y0)
    if kind == "dinf":
        c -= (2.0 * (z0 @ t) / (d @ d) + 1.0) * d
    if kind == "pinf":
        rows = range(1) if dims["l"] else range(dims["l"], dims["l"] + dims["q"][0])
        for r in rows:
            G[r] = 0.0
            h[r] = -1.0 if r == rows[0] else 0.0
    return c, G, h, A, A @ x0


def lp_batch(B, n, dims, p, seed0, kinds=None):
    parts = [lp_problem(n, dims, p, seed0 + k, (kinds or {}).get(k, "feasible")) for k in range(B)]
    return [np.stack([x[i] for x in parts]) for i in range(5)]


def _rel(a, b):
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


def ref_conelp(c, G, h, dims, A, b, **options):
    from cvxopt import matrix, solvers
    options.setdefault("show_progress", False)
    dims = _full(dims)
    kw = {"kktsolver": "chol"} if dims["q"] else {}
    Am, bm = (matrix(A), matrix(b)) if A.shape[0] else (None, None)
    return solvers.conelp(matrix(c), matrix(G), matrix(h), dims, Am, bm, options=options, **kw)


def _solve(batch, dims, **kw):
    import cvxopt_b200
    c, G, h, A, b = batch
    eq = dict(A=A, b=b) if A.shape[1] else {}
    return cvxopt_b200.conelp_batch(c, G, h, dims=dims, **eq, **kw)


def _margin(v, dims):
    """smallest cone margin of v: min over 'l' entries and x0 - ||x1|| of each 'q' block"""
    dims = _full(dims)
    out = [v[:dims["l"]].min()] if dims["l"] else []
    o = dims["l"]
    for k in dims["q"]:
        out.append(v[o] - np.linalg.norm(v[o + 1:o + k]))
        o += k
    return min(out)


def assert_matches(got, batch, dims, want, certificates=True, obj_rtol=1e-8):
    c, G, h, A, b = batch
    for k, w in enumerate(want):
        assert got["status"][k] == w["status"], (k, got["status"][k], w["status"])
        assert got["iterations"][k] == w["iterations"], (k, got["iterations"][k], w["iterations"])
        st = w["status"]
        if st == "optimal":
            np.testing.assert_allclose(got["primal objective"][k], w["primal objective"], rtol=obj_rtol)
            np.testing.assert_allclose(got["dual objective"][k], w["dual objective"], rtol=obj_rtol)
        for key in ("x", "y", "s", "z"):
            if w[key] is None:
                assert np.isnan(got[key][k]).all(), (k, key)
                continue
            rtol, atol = (1e-6, 1e-8) if key in ("x", "y") else (1e-5, 1e-7)
            np.testing.assert_allclose(got[key][k], np.array(w[key]).ravel(), rtol=rtol, atol=atol, err_msg=key)
        if st == "primal infeasible":
            assert got["dual objective"][k] == 1.0 and np.isnan(got["primal objective"][k])
        if st == "dual infeasible":
            assert got["primal objective"][k] == -1.0 and np.isnan(got["dual objective"][k])
        if not certificates:
            continue
        x, y, s, z = (got[key][k] for key in ("x", "y", "s", "z"))
        if st == "primal infeasible":        # A'y + G'z = 0, h'z + b'y = -1, z in the cone
            scale = 1 + np.abs(G[k]).max() * np.abs(z).max()
            assert np.abs(A[k].T @ y + G[k].T @ z).max() <= 1e-6 * scale
            assert h[k] @ z + b[k] @ y == pytest.approx(-1.0, abs=1e-9)
            assert _margin(z, dims) >= -1e-8
        if st == "dual infeasible":          # c'x = -1, A x = 0, G x + s = 0, s in the cone
            scale = 1 + np.abs(G[k]).max() * np.abs(x).max()
            assert c[k] @ x == pytest.approx(-1.0, abs=1e-9)
            assert np.abs(A[k] @ x).max(initial=0.0) <= 1e-6 * scale
            assert np.abs(G[k] @ x + s).max() <= 1e-6 * scale
            assert _margin(s, dims) >= -1e-8


def ref_loop(batch, dims, **options):
    c, G, h, A, b = batch
    return [ref_conelp(c[k], G[k], h[k], dims, A[k], b[k], **options) for k in range(c.shape[0])]


CASES = [
    (4, 30, {"l": 80}, 0),                              # 'l' only, solvers.lp
    (3, 150, {"l": 0, "q": [4] * 40}, 0),               # 'q' only, two Cholesky blocks
    (2, 200, {"l": 64, "q": [1, 2, 300]}, 0),           # cones of order 1 and 2, one longer than a CTA
    (1, 257, {"l": 300}, 0),                            # B = 1: the unbatched Cholesky, three blocks
    (3, 129, {"l": 300}, 20),                           # with A
    (2, 60, {"l": 20, "q": [5, 1, 40]}, 10),            # cones with A
    (1, 100, {"l": 30, "q": [50, 40]}, 5),              # B = 1, cones with A
]


@pytest.mark.parametrize("B,n,dims,p", CASES)
def test_lp_batch_matches_conelp(ref, B, n, dims, p):
    batch = lp_batch(B, n, dims, p, 1000 * B + n + p)
    got = _solve(batch, dims)
    want = ref_loop(batch, dims)
    assert all(w["status"] == "optimal" for w in want)
    assert_matches(got, batch, dims, want)


@pytest.mark.parametrize("dims,p,B,options", [({"l": 300}, 0, 3, {}), ({"l": 300}, 20, 1, {}),
                                              ({"l": 20, "q": [5, 1, 140]}, 16, 3, {}),
                                              ({"l": 20, "q": [5, 1, 140]}, 0, 3, {"refinement": 0})])
def test_lp_iterates_match_conelp(ref, dims, p, B, options):
    batch = lp_batch(B, 129, dims, p, 3000 + p)
    worst = 0.0
    for k in (1, 2, 3):
        got = _solve(batch, dims, maxiters=k, **options)
        for j in range(B):
            c, G, h, A, b = (x[j] for x in batch)
            want = ref_conelp(c, G, h, dims, A, b, maxiters=k, **options)
            assert want["status"] == "unknown" and want["iterations"] == k, (j, k, want["status"])
            assert got["status"][j] == "unknown" and got["iterations"][j] == k, (j, k, got["status_code"][j])
            for key in ("x", "y", "s", "z"):
                d = _rel(got[key][j], np.array(want[key]).ravel())
                assert d <= TOL, (j, k, key, d)
                worst = max(worst, d)
    print("\nconelp iterates %s p=%d: largest relative difference %.2e" % (dims, p, worst))


@pytest.mark.parametrize("dims,n,p", [({"l": 60}, 20, 3), ({"l": 10, "q": [6, 8]}, 12, 2), ({"q": [9, 7, 9]}, 10, 0)])
def test_certificates_match_conelp(ref, dims, n, p):
    """one batch mixes feasible, primal infeasible and dual infeasible problems"""
    kinds = {1: "pinf", 2: "dinf", 4: "pinf", 5: "dinf"}
    batch = lp_batch(6, n, dims, p, 5000 + n, kinds)
    got = _solve(batch, dims, nsub=1)
    want = ref_loop(batch, dims)
    statuses = [w["status"] for w in want]
    assert statuses.count("primal infeasible") == 2 and statuses.count("dual infeasible") == 2, statuses
    assert_matches(got, batch, dims, want)
    assert list(got["status_code"][[1, 4]]) == [4, 4] and list(got["status_code"][[2, 5]]) == [5, 5]


def test_s_plus_ata_switch(ref):
    """problems 1 and 3: columns 48..63 of G are zero, so Gs'Gs is singular, but A's columns 48..63 are a random
    (invertible) 16 x 16 block, so [G; A] has full rank"""
    n, m, p = 64, 128, 16
    batch = lp_batch(4, n, {"l": m}, p, 9000)
    c, G, h, A, b = batch
    rng = np.random.Generator(np.random.PCG64(9100))
    for j in (1, 3):
        G[j][:, 48:] = 0.0
        x0, z0, y0 = rng.standard_normal(n), rng.uniform(0.5, 1.5, m), rng.standard_normal(p)
        h[j] = G[j] @ x0 + rng.uniform(0.5, 1.5, m)
        b[j] = A[j] @ x0
        c[j] = -(G[j].T @ z0 + A[j].T @ y0)
        with pytest.raises(np.linalg.LinAlgError):
            np.linalg.cholesky(G[j].T @ G[j])
    got = _solve(batch, {"l": m})
    assert_matches(got, batch, {"l": m}, ref_loop(batch, {"l": m}))


def test_singular_start_names_the_problem():
    n, m, p = 20, 40, 5
    c, G, h, A, b = lp_batch(4, n, {"l": m}, p, 9500)
    G[2][:, 5] = 0.0                       # x[5] appears nowhere: the KKT matrix with W = I is singular
    A[2][:, 5] = 0.0
    with pytest.raises(ValueError, match=r"problem 2: Rank\(A\) < p or Rank\(\[G; A\]\) < n"):
        _solve((c, G, h, A, b), None, nsub=1)


def test_optimal_at_the_start(ref):
    """c = 0 and G = [I; -I], h = 1: the primal start is x = 0, s = h, the dual start z = 0, so the reference returns
    'optimal' after 0 iterations (coneprog.py:744-804).  Problems 1 and 3 are ordinary LPs in the same batch."""
    n = 12
    batch = lp_batch(4, n, {"l": 2 * n}, 0, 9600)
    c, G, h, A, b = batch
    for j in (0, 2):
        c[j] = 0.0
        G[j] = np.vstack([np.eye(n), -np.eye(n)])
        h[j] = 1.0
    got = _solve(batch, None)
    want = ref_loop(batch, {"l": 2 * n})
    assert [w["iterations"] for w in want][0::2] == [0, 0]
    assert_matches(got, batch, {"l": 2 * n}, want)


@pytest.mark.parametrize("refinement", [0, 2])
def test_refinement_option(ref, refinement):
    dims = {"l": 15, "q": [6, 4, 9]}
    batch = lp_batch(4, 20, dims, 0, 7000)
    got = _solve(batch, dims, refinement=refinement)
    want = ref_loop(batch, dims, refinement=refinement)
    worst = max(abs(got["dual objective"][k] / w["dual objective"] - 1) for k, w in enumerate(want))
    print("\nrefinement=%d: largest relative difference of the dual objective %.2e" % (refinement, worst))
    # without refinement the last Newton steps of a cone LP are solved less accurately, by the reference as here:
    # one dual objective differed from the reference's by 4.6e-8 (relative) on an H100, while every iterate of the
    # first three matches to 1e-10 (test_lp_iterates_match_conelp), so the objectives get 1e-7 there
    assert_matches(got, batch, dims, want, obj_rtol=1e-7 if refinement == 0 else 1e-8)


def test_compaction_subbatches_resolve_and_memory(ref, monkeypatch):
    import cvxopt_b200
    from cvxopt_b200 import ConeLPBatch, _lib
    n, B, p = 40, 9, 5
    dims = {"l": 30, "q": [5, 8, 3]}
    batch = lp_batch(B, n, dims, p, 9900, {2: "pinf", 7: "dinf"})
    batch[0] *= np.linspace(0.1, 30.0, B)[:, None]          # spread the iteration counts: compaction swaps slots
    base = _solve(batch, dims, nsub=1)
    assert len(set(base["iterations"].tolist())) > 1
    monkeypatch.setenv("CVXB_BATCH_COMPACT", "0")
    flat = _solve(batch, dims, nsub=1)
    monkeypatch.delenv("CVXB_BATCH_COMPACT")
    three = _solve(batch, dims, nsub=3)
    for key in ("x", "y", "s", "z", "primal objective", "dual objective"):
        np.testing.assert_array_equal(flat[key], base[key], err_msg=key)
        np.testing.assert_allclose(three[key], base[key], rtol=0, atol=1e-12 * (1 + np.nanmax(np.abs(base[key]))))
    assert np.array_equal(three["iterations"], base["iterations"])
    assert_matches(base, batch, dims, ref_loop(batch, dims))
    lib = _lib.load()
    before = lib.cvxb_device_bytes()
    lb = ConeLPBatch(B, n, 46, 0, dims=dims, p=p)
    assert lib.cvxb_device_bytes() > before
    c, G, h, A, b = batch
    lb.load(c[::-1], G[::-1], h[::-1], A[::-1], b[::-1])
    lb.solve()
    lb.load(c, G, h, A, b)                                   # re-load, re-solve
    lb.solve()
    r1 = lb.results()
    lb.solve()
    r2 = lb.results()
    for key in ("x", "y", "s", "z", "iterations"):
        np.testing.assert_array_equal(r1[key], r2[key], err_msg=key)
        np.testing.assert_array_equal(r1[key], base[key], err_msg=key)
    # a QP load on the LP handle and an LP load on a QP handle are refused
    x = np.zeros(B * n * n)
    assert lib.cvxb_batch_load(lb._h, x.ctypes.data, x.ctypes.data, x.ctypes.data, x.ctypes.data, _lib.HOST) == _lib.E_ARG
    qb = cvxopt_b200.QPBatch(B, n, 46, 0, dims=dims)
    assert lib.cvxb_batch_load_lp(qb._h, x.ctypes.data, x.ctypes.data, x.ctypes.data, _lib.HOST) == _lib.E_ARG
    qb.close()
    lb.close()
    assert lib.cvxb_device_bytes() == before
    h0 = C.c_void_p()
    d, keep, _ = cvxopt_b200.batch._batch_dims(dims)
    assert lib.cvxb_batch_create_lp(C.byref(h0), B, n, p, C.byref(d), 0) == 0
    Gcm = np.ascontiguousarray(G.transpose(0, 2, 1))
    assert lib.cvxb_batch_load_lp(h0, c.ctypes.data, Gcm.ctypes.data, h.ctypes.data, _lib.HOST) == 0
    assert lib.cvxb_batch_solve(h0, 100, 1e-7, 1e-6, 1e-7) == _lib.E_ARG       # A and b were never loaded
    lib.cvxb_batch_destroy(h0)
    assert lib.cvxb_device_bytes() == before
