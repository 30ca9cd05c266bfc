"""SDP batches (SDPBatch, sdp_batch: csrc/batch_ipm.cu's solve<CONES, EQ, true, true>) against a Python loop over the
reference's solvers.conelp(c, G, h, dims, A, b, kktsolver='chol') and solvers.sdp (oracle/_ref): converged
solutions, iterates, certificates, the upper triangles of G and h, and the batch mechanics."""
import numpy as np
import pytest

from problems import cone_point, sgemv_t
from test_batch_conelp_gpu import TOL, _rel

pytestmark = pytest.mark.gpu


def _full(d):
    return {"l": d.get("l", 0), "q": list(d.get("q", [])), "s": list(d.get("s", []))}


def sdp_problem(n, dims, p, seed, kind="feasible"):
    """conelp data with symmetric 's' columns of G: h = G x0 + s0, b = A x0, c = -(G'z0 + A'y0) with s0, z0 strictly
    inside the cones.  'pinf': the first 's' block reads 0 x + s = -I, so z = I / tr certifies primal infeasibility.
    'dinf': G d = -t (t inside the cones), A d = 0 and c'd < 0."""
    dims = _full(dims)
    rng = np.random.Generator(np.random.PCG64(seed))
    m = dims["l"] + sum(dims["q"]) + sum(k * k for k in dims["s"])
    G = rng.standard_normal((m, n))
    o = dims["l"] + sum(dims["q"])
    for k in dims["s"]:
        for j in range(n):
            M = G[o:o + k * k, j].reshape(k, k, order="F")
            G[o:o + k * k, j] = ((M + M.T) / 2).reshape(-1, order="F")
        o += k * k
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
    c = -(sgemv_t(G, z0, dims) + A.T @ y0)
    if kind == "dinf":
        c -= (2.0 * (z0 @ t) / (d @ d) + 1.0) * d
    if kind == "pinf":
        o = dims["l"] + sum(dims["q"])
        k = dims["s"][0]
        G[o:o + k * k] = 0.0
        h[o:o + k * k] = -np.eye(k).reshape(-1)
    return c, G, h, A, A @ x0


def sdp_batch_data(B, n, dims, p, seed0, kinds=None):
    parts = [sdp_problem(n, dims, p, seed0 + k, (kinds or {}).get(k, "feasible")) for k in range(B)]
    return [np.stack([x[i] for x in parts]) for i in range(5)]


def ref_conelp(c, G, h, dims, A, b, **options):
    from cvxopt import matrix, solvers
    options.setdefault("show_progress", False)
    Am, bm = (matrix(A), matrix(b)) if A.shape[0] else (None, None)
    return solvers.conelp(matrix(c), matrix(G), matrix(h), _full(dims), Am, bm, options=options, kktsolver="chol")


def ref_loop(batch, dims, **options):
    c, G, h, A, b = batch
    return [ref_conelp(c[k], G[k], h[k], dims, A[k], b[k], **options) for k in range(c.shape[0])]


def _solve(batch, dims, nsub=None, **options):
    from cvxopt_b200 import SDPBatchGroup, batch as bt
    c, G, h, A, b = batch
    p = A.shape[1]
    return bt._run_group(SDPBatchGroup(c.shape[0], c.shape[1], dims, p, 0, nsub),
                         (c, G, h, A if p else None, b if p else None), options)


def _sym(v, dims):
    """v with every 's' block made symmetric from its lower triangle"""
    dims = _full(dims)
    v = v.copy()
    o = dims["l"] + sum(dims["q"])
    for k in dims["s"]:
        M = v[o:o + k * k].reshape(k, k, order="F")
        v[o:o + k * k] = (np.tril(M) + np.tril(M, -1).T).reshape(-1, order="F")
        o += k * k
    return v


def _min_eig(v, dims):
    dims = _full(dims)
    o = dims["l"] + sum(dims["q"])
    out = [v[:dims["l"]].min()] if dims["l"] else []
    for k in dims["s"]:
        out.append(np.linalg.eigvalsh(v[o:o + k * k].reshape(k, k, order="F")).min())
        o += k * k
    return min(out)


def assert_matches(got, batch, dims, want, obj_rtol=1e-8):
    for k, w in enumerate(want):
        assert got["status"][k] == w["status"], (k, got["status"][k], w["status"])
        assert got["iterations"][k] == w["iterations"], (k, got["iterations"][k], w["iterations"])
        if w["status"] == "optimal":
            np.testing.assert_allclose(got["primal objective"][k], w["primal objective"], rtol=obj_rtol)
            np.testing.assert_allclose(got["dual objective"][k], w["dual objective"], rtol=obj_rtol)
        for key in ("x", "y", "s", "z"):
            if w[key] is None:
                assert np.isnan(got[key][k]).all(), (k, key)
                continue
            want_v = np.array(w[key]).ravel()
            if key in ("s", "z"):
                want_v = _sym(want_v, dims)
            rtol, atol = (1e-6, 1e-8) if key in ("x", "y") else (1e-5, 1e-7)
            np.testing.assert_allclose(got[key][k], want_v, rtol=rtol, atol=atol, err_msg=key)


CASES = [
    (4, 20, {"s": [8]}, 0),
    (3, 1, {"l": 2, "s": [1]}, 0),                  # n = cdim_pckd would make the start the exact solution
    (3, 2, {"s": [2]}, 0),
    (3, 40, {"l": 20, "s": [3, 7, 16]}, 0),
    (2, 60, {"s": [32]}, 0),
    (3, 30, {"l": 10, "q": [5, 3], "s": [6, 9]}, 0),
    (1, 200, {"l": 40, "s": [16, 16]}, 0),
    (3, 30, {"l": 10, "s": [6, 5]}, 6),
]


@pytest.mark.parametrize("B,n,dims,p", CASES)
def test_sdp_batch_matches_conelp(ref, B, n, dims, p):
    batch = sdp_batch_data(B, n, dims, p, 100 * B + n + p)
    got = _solve(batch, dims)
    want = ref_loop(batch, dims)
    assert all(w["status"] == "optimal" for w in want), [w["status"] for w in want]
    assert_matches(got, batch, dims, want)


def test_order_one_block_where_the_start_is_the_solution(ref):
    """{'s': [1]} with n = 1: G is 1 x 1, so the primal start s = h - G (h / G) is zero up to rounding and the
    reference returns 'optimal' after 0 iterations when its rounding leaves s >= 0 (coneprog.py:756).  The batch's
    Cholesky solve multiplies by the inverse of the pivot where LAPACK divides, so its s may land on -1e-16 instead,
    and then it takes the ordinary iterations to the same solution.  The iteration count therefore cannot be
    required to match; the status and the solution are."""
    dims = {"s": [1]}
    batch = sdp_batch_data(3, 1, dims, 0, 301)
    got = _solve(batch, dims)
    want = ref_loop(batch, dims)
    for k, w in enumerate(want):
        assert w["status"] == "optimal" and got["status"][k] == "optimal"
        np.testing.assert_allclose(got["x"][k], np.array(w["x"]).ravel(), rtol=1e-6, atol=1e-8)
        np.testing.assert_allclose(got["primal objective"][k], w["primal objective"], rtol=1e-7, atol=1e-9)
    print("\n{'s': [1]}, n = 1: iterations", list(got["iterations"]), "reference", [w["iterations"] for w in want])


@pytest.mark.parametrize("refinement", [0, 2])
def test_sdp_refinement_option(ref, refinement):
    dims = {"l": 6, "s": [5, 4]}
    batch = sdp_batch_data(3, 15, dims, 0, 700)
    got = _solve(batch, dims, refinement=refinement)
    assert_matches(got, batch, dims, ref_loop(batch, dims, refinement=refinement), obj_rtol=1e-7)


@pytest.mark.parametrize("dims,p", [({"l": 8, "s": [6, 5]}, 0), ({"q": [4], "s": [7]}, 3)])
def test_sdp_iterates_match_conelp(ref, dims, p):
    batch = sdp_batch_data(3, 25, dims, p, 3100 + p)
    worst = 0.0
    for k in (1, 2, 3):
        got = _solve(batch, dims, maxiters=k)
        for j in range(3):
            c, G, h, A, b = (x[j] for x in batch)
            want = ref_conelp(c, G, h, dims, A, b, maxiters=k)
            assert want["iterations"] == k and got["iterations"][j] == k
            for key in ("x", "y", "s", "z"):
                w = np.array(want[key]).ravel()
                d = _rel(got[key][j], _sym(w, dims) if key in ("s", "z") else w)
                assert d <= TOL, (j, k, key, d)
                worst = max(worst, d)
    print("\nsdp iterates %s p=%d: largest relative difference %.2e" % (dims, p, worst))


def test_sdp_certificates(ref):
    dims = {"l": 4, "s": [5, 3]}
    kinds = {1: "pinf", 2: "dinf", 4: "pinf"}
    batch = sdp_batch_data(5, 8, dims, 0, 5100, kinds)
    got = _solve(batch, dims, nsub=1)
    want = ref_loop(batch, dims)
    statuses = [w["status"] for w in want]
    assert statuses.count("primal infeasible") == 2 and statuses.count("dual infeasible") == 1, statuses
    assert_matches(got, batch, dims, want)
    c, G, h, A, b = batch
    dims = _full(dims)
    for k in (1, 4):
        z = got["z"][k]
        assert np.abs(sgemv_t(G[k], z, dims)).max() <= 1e-6 * (1 + np.abs(G[k]).max() * np.abs(z).max())
        assert sgemv_t(h[k][:, None], z, dims)[0] == pytest.approx(-1.0, abs=1e-9)
        assert _min_eig(z, dims) >= -1e-8
    x, s = got["x"][2], got["s"][2]
    assert c[2] @ x == pytest.approx(-1.0, abs=1e-9)
    assert np.abs(G[2] @ x + s).max() <= 1e-6 * (1 + np.abs(G[2]).max() * np.abs(x).max())
    assert _min_eig(s, dims) >= -1e-8


def test_upper_triangles_are_not_read_and_results_are_symmetric(ref):
    dims = {"l": 5, "s": [4, 6]}
    batch = sdp_batch_data(3, 12, dims, 0, 6100)
    runs = []
    for fill in ("mirror", "zero", "junk"):
        c, G, h, A, b = (x.copy() for x in batch)
        o = 5
        rng = np.random.default_rng(1)
        for k in dims["s"]:
            up = np.triu(np.ones((k, k), dtype=bool), 1).reshape(-1, order="F")
            rows = o + np.nonzero(up)[0]
            if fill == "zero":
                G[:, rows] = 0.0
                h[:, rows] = 0.0
            elif fill == "junk":
                G[:, rows] = rng.standard_normal(G[:, rows].shape)
                h[:, rows] = rng.standard_normal(h[:, rows].shape)
            o += k * k
        runs.append(_solve((c, G, h, A, b), dims))
    for r in runs[1:]:
        for key in ("x", "s", "z", "iterations", "primal objective"):
            np.testing.assert_array_equal(r[key], runs[0][key], err_msg=key)
    for v in (runs[0]["s"], runs[0]["z"]):
        for j in range(3):
            np.testing.assert_array_equal(v[j], _sym(v[j], dims))


def test_sdp_batch_front_end_matches_solvers_sdp(ref):
    from cvxopt import matrix, solvers
    import cvxopt_b200
    dims = {"l": 6, "s": [4, 3]}
    c, G, h, A, b = sdp_batch_data(3, 10, dims, 0, 7100)
    Gl, hl = G[:, :6], h[:, :6]
    Gs = [G[:, 6:22], G[:, 22:31]]
    hs = [h[:, 6:22].reshape(3, 4, 4).transpose(0, 2, 1), h[:, 22:31].reshape(3, 3, 3).transpose(0, 2, 1)]
    got = cvxopt_b200.sdp_batch(c, Gl, hl, Gs, hs)
    for k in range(3):
        w = solvers.sdp(matrix(c[k]), matrix(Gl[k]), matrix(hl[k]), [matrix(g[k]) for g in Gs],
                        [matrix(np.ascontiguousarray(x[k])) for x in hs], kktsolver="chol",
                        options={"show_progress": False})
        assert got["status"][k] == w["status"] and got["iterations"][k] == w["iterations"]
        np.testing.assert_allclose(got["x"][k], np.array(w["x"]).ravel(), rtol=1e-6, atol=1e-8)
        np.testing.assert_allclose(got["sl"][k], np.array(w["sl"]).ravel(), rtol=1e-5, atol=1e-7)
        for j in range(2):
            Z = np.array(w["zs"][j])
            Z = np.tril(Z) + np.tril(Z, -1).T
            np.testing.assert_allclose(got["zs"][j][k], Z, rtol=1e-5, atol=1e-7)


def test_compaction_subbatches_resolve_and_memory(ref, monkeypatch):
    from cvxopt_b200 import SDPBatch, _lib
    dims = {"l": 6, "q": [4], "s": [5, 3]}
    B, n, p = 9, 14, 2
    batch = sdp_batch_data(B, n, dims, p, 9100, {3: "dinf"})
    batch[0] *= np.linspace(0.1, 30.0, B)[:, None]
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
    sb = SDPBatch(B, n, dims, p=p)
    assert lib.cvxb_device_bytes() > before
    c, G, h, A, b = batch
    sb.load(c, G, h, A, b)
    sb.solve()
    r1 = sb.results()
    sb.solve()
    r2 = sb.results()
    for key in ("x", "y", "s", "z", "iterations"):
        np.testing.assert_array_equal(r1[key], r2[key], err_msg=key)
        np.testing.assert_array_equal(r1[key], base[key], err_msg=key)
    sb.close()
    assert lib.cvxb_device_bytes() == before


def test_batches_without_s_blocks_launch_what_they_did_before():
    """Launches per solve of an 'l'-only cone LP batch, a cone LP batch with 'q' cones and an 'l'-only QP batch (three
    lock-step iterations, one sub-batch).  The counts are those of the library before 's' blocks were added: the 's'
    kernels launch only for a batch that has them."""
    import cvxopt_b200 as cb
    from problems import dense_qp
    from test_batch_conelp_gpu import lp_batch
    got = []
    for dims, n in (({"l": 40}, 20), ({"l": 20, "q": [5, 4]}, 20)):
        c, G, h, A, b = lp_batch(4, n, dims, 0, 77)
        l0 = cb.launch_count()
        cb.conelp_batch(c, G, h, dims=dims, nsub=1, maxiters=3)
        got.append(cb.launch_count() - l0)
    P, q, G, h = zip(*[dense_qp(16, 32, seed=k) for k in range(4)])
    l0 = cb.launch_count()
    cb.qp_batch(np.stack(P), np.stack(q), np.stack(G), np.stack(h), nsub=1, maxiters=3)
    got.append(cb.launch_count() - l0)
    assert got == [117, 187, 93]
