"""QP batches with 's' blocks (SDPQPBatch, coneqp_batch: csrc/batch_ipm.cu's solve<CONES, EQ, false, true>) against a
Python loop over the reference's solvers.coneqp(P, q, G, h, dims, A, b) with its default kktsolver ('chol' with 's'
cones) (oracle/_ref): converged solutions, iterates, refinement, maxiters, the singular start, the upper triangles of
G and h, the batch mechanics, and the launches of batches without 's' blocks."""
import numpy as np
import pytest

from test_batch_conelp_gpu import TOL, _rel
from test_batch_sdp_gpu import _full, _sym, sdp_problem

pytestmark = pytest.mark.gpu

P_KINDS = ("random", "lowrank", "zero")


def psd(n, kind, seed):
    """a PSD P: M M' / n with M n x n ('random') or n x max(1, n // 3) ('lowrank'), or 0"""
    rng = np.random.Generator(np.random.PCG64(seed))
    if kind == "zero":
        return np.zeros((n, n))
    M = rng.standard_normal((n, n if kind == "random" else max(1, n // 3)))
    return M @ M.T / n


def sdqp_batch_data(B, n, dims, p, seed0, kinds=None, pkind=None):
    """sdp_problem's data, c used as q, and problem k's P of kind pkind or P_KINDS[k % 3] -> P, q, G, h, A, b"""
    out = []
    for k in range(B):
        c, G, h, A, b = sdp_problem(n, dims, p, seed0 + k, (kinds or {}).get(k, "feasible"))
        out.append((psd(n, pkind or P_KINDS[k % 3], 7 * seed0 + k), c, G, h, A, b))
    return [np.stack([x[i] for x in out]) for i in range(6)]


def ref_coneqp(P, q, G, h, dims, A, b, **options):
    from cvxopt import matrix, solvers
    options.setdefault("show_progress", False)
    Am, bm = (matrix(A), matrix(b)) if A.shape[0] else (None, None)
    return solvers.coneqp(matrix(P), matrix(q), matrix(G), matrix(h), _full(dims), Am, bm, options=options)


def ref_loop(batch, dims, **options):
    return [ref_coneqp(*(x[k] for x in batch[:4]), dims, batch[4][k], batch[5][k], **options)
            for k in range(batch[0].shape[0])]


def _solve(batch, dims, nsub=None, **options):
    import cvxopt_b200
    P, q, G, h, A, b = batch
    eq = dict(A=A, b=b) if A.shape[1] else {}
    return cvxopt_b200.coneqp_batch(P, q, G, h, dims, nsub=nsub, **eq, **options)


def assert_matches(got, dims, want, obj_rtol=1e-8):
    for k, w in enumerate(want):
        assert got["status"][k] == w["status"], (k, got["status"][k], w["status"])
        assert got["iterations"][k] == w["iterations"], (k, got["iterations"][k], w["iterations"])
        if w["status"] == "optimal":
            np.testing.assert_allclose(got["primal objective"][k], w["primal objective"], rtol=obj_rtol)
            np.testing.assert_allclose(got["dual objective"][k], w["dual objective"], rtol=obj_rtol)
        for key in ("x", "y", "s", "z"):
            want_v = np.array(w[key]).ravel()
            if key in ("s", "z"):
                want_v = _sym(want_v, dims)
            rtol, atol = (1e-6, 1e-8) if key in ("x", "y") else (1e-5, 1e-7)
            np.testing.assert_allclose(got[key][k], want_v, rtol=rtol, atol=atol, err_msg=key)


CASES = [
    (3, 20, {"s": [8]}, 0),
    (3, 1, {"l": 2, "s": [1]}, 0),
    (3, 2, {"s": [2]}, 0),
    (3, 40, {"l": 20, "s": [3, 7, 16]}, 0),
    (2, 60, {"s": [32]}, 0),
    (3, 30, {"l": 10, "q": [5, 3], "s": [6, 9]}, 0),
    (1, 200, {"l": 40, "s": [16, 16]}, 0),
    (3, 30, {"l": 10, "s": [6, 5]}, 6),
    (3, 25, {"q": [4], "s": [7]}, 3),
]


@pytest.mark.parametrize("B,n,dims,p", CASES)
def test_coneqp_batch_matches_coneqp(ref, B, n, dims, p):
    batch = sdqp_batch_data(B, n, dims, p, 100 * B + n + p)
    got = _solve(batch, dims)
    want = ref_loop(batch, dims)
    assert all(w["status"] == "optimal" for w in want), [w["status"] for w in want]
    assert_matches(got, dims, want)


@pytest.mark.parametrize("dims,p", [({"l": 8, "s": [6, 5]}, 0), ({"q": [4], "s": [7]}, 3)])
def test_coneqp_batch_iterates_match_coneqp(ref, dims, p):
    batch = sdqp_batch_data(3, 25, dims, p, 3100 + p)
    worst = 0.0
    for k in (1, 2, 3):
        got = _solve(batch, dims, maxiters=k)
        want = ref_loop(batch, dims, maxiters=k)
        for j, w in enumerate(want):
            assert w["iterations"] == k and got["iterations"][j] == k
            for key in ("x", "y", "s", "z"):
                wv = np.array(w[key]).ravel()
                d = _rel(got[key][j], _sym(wv, dims) if key in ("s", "z") else wv)
                assert d <= TOL, (j, k, key, d)
                worst = max(worst, d)
    print("\nconeqp_batch iterates %s p=%d: largest relative difference %.2e" % (dims, p, worst))


@pytest.mark.parametrize("refinement", [0, 2])
def test_coneqp_batch_refinement_option(ref, refinement):
    """refinement = 0 takes f4_no_ir's step after the solve without a refinement kernel after it: the 's' rows of
    uz are then unpacked from the solve's packed bzp by k_f4_post"""
    dims = {"l": 6, "q": [3], "s": [5, 4]}
    batch = sdqp_batch_data(3, 15, dims, 2, 700)
    got = _solve(batch, dims, refinement=refinement)
    assert_matches(got, dims, ref_loop(batch, dims, refinement=refinement), obj_rtol=1e-7)


def test_infeasible_problem_ends_unknown_at_maxiters(ref):
    """coneqp has no infeasibility certificates: a problem whose first 's' block reads 0 x + s = -I runs to maxiters"""
    dims = {"l": 4, "s": [5, 3]}
    batch = sdqp_batch_data(3, 8, dims, 0, 5100, kinds={1: "pinf"}, pkind="random")
    got = _solve(batch, dims, nsub=1, maxiters=15)
    want = ref_loop(batch, dims, maxiters=15)
    assert [w["status"] for w in want] == ["optimal", "unknown", "optimal"], [w["status"] for w in want]
    assert want[1]["iterations"] == 15
    assert list(got["status"]) == ["optimal", "unknown", "optimal"]
    assert list(got["iterations"]) == [w["iterations"] for w in want]
    assert got["status_code"][1] == 2                          # maxiters, not a failed factorisation


def test_singular_start_names_the_problem():
    n, p, dims = 12, 2, {"l": 4, "s": [3]}
    P, q, G, h, A, b = sdqp_batch_data(3, n, dims, p, 9500, pkind="zero")
    G[1][:, 5] = 0.0                       # x[5] appears nowhere: the KKT matrix with W = I is singular
    A[1][:, 5] = 0.0
    with pytest.raises(ValueError, match=r"problem 1: Rank\(A\) < p or Rank\(\[P; A; G\]\) < n"):
        _solve((P, q, G, h, A, b), dims, nsub=1)


def test_upper_triangles_are_not_read_and_results_are_symmetric(ref):
    dims = {"l": 5, "s": [4, 6]}
    batch = sdqp_batch_data(3, 12, dims, 0, 6100)
    runs = []
    for fill in ("mirror", "zero", "junk"):
        P, q, G, h, A, b = (x.copy() for x in batch)
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
        runs.append(_solve((P, q, G, h, A, b), dims))
    for r in runs[1:]:
        for key in ("x", "s", "z", "iterations", "primal objective", "dual objective"):
            np.testing.assert_array_equal(r[key], runs[0][key], err_msg=key)
    for v in (runs[0]["s"], runs[0]["z"]):
        for j in range(3):
            np.testing.assert_array_equal(v[j], _sym(v[j], dims))
    assert_matches(runs[0], dims, ref_loop(batch, dims))


def test_compaction_subbatches_resolve_and_memory(ref, monkeypatch):
    from cvxopt_b200 import SDPQPBatch, _lib
    dims = {"l": 6, "q": [4], "s": [5, 3]}
    B, n, p = 9, 14, 2
    batch = sdqp_batch_data(B, n, dims, p, 9100)
    batch[1] *= np.linspace(0.1, 30.0, B)[:, None]
    base = _solve(batch, dims, nsub=1)
    assert len(set(base["iterations"].tolist())) > 1
    monkeypatch.setenv("CVXB_BATCH_COMPACT", "0")
    flat = _solve(batch, dims, nsub=1)
    monkeypatch.delenv("CVXB_BATCH_COMPACT")
    three = _solve(batch, dims, nsub=3)
    for key in ("x", "y", "s", "z", "primal objective", "dual objective"):
        np.testing.assert_array_equal(flat[key], base[key], err_msg=key)
        np.testing.assert_allclose(three[key], base[key], rtol=0, atol=1e-12 * (1 + np.abs(base[key]).max()))
    assert np.array_equal(flat["iterations"], base["iterations"])
    assert np.array_equal(three["iterations"], base["iterations"])
    assert_matches(base, dims, ref_loop(batch, dims))
    lib = _lib.load()
    before = lib.cvxb_device_bytes()
    sb = SDPQPBatch(B, n, dims, p=p)
    assert lib.cvxb_device_bytes() > before
    P, q, G, h, A, b = batch
    sb.load(P, q, G, h, A, b)
    sb.solve()
    r1 = sb.results()
    sb.solve()
    r2 = sb.results()
    for key in ("x", "y", "s", "z", "iterations"):
        np.testing.assert_array_equal(r1[key], r2[key], err_msg=key)
        np.testing.assert_array_equal(r1[key], base[key], err_msg=key)
    sb.close()
    assert lib.cvxb_device_bytes() == before


@pytest.mark.parametrize("dims,p", [({"l": 30}, 0), ({"l": 10, "q": [5, 3]}, 2), ({"l": 12, "s": [0]}, 0)])
def test_dims_without_s_blocks_run_the_qp_batch(dims, p):
    """coneqp_batch on dims without an 's' block of positive order is qp_batch, bit for bit and launch for launch"""
    import cvxopt_b200 as cb
    P, q, G, h, A, b = sdqp_batch_data(4, 10, dims, p, 4400, pkind="random")
    eq = dict(A=A, b=b) if p else {}
    qdims = {"l": dims["l"], "q": dims.get("q", [])}
    l0 = cb.launch_count()
    want = cb.qp_batch(P, q, G, h, dims=qdims, nsub=1, **eq)
    l1 = cb.launch_count()
    got = cb.coneqp_batch(P, q, G, h, dims, nsub=1, **eq)
    l2 = cb.launch_count()
    assert l2 - l1 == l1 - l0
    for key in ("x", "y", "s", "z", "iterations", "status_code", "primal objective", "dual objective"):
        np.testing.assert_array_equal(got[key], want[key], err_msg=key)


# per lock-step iteration: those of the same QP batch without its 's' blocks, plus per direction k_s_wtz twice,
# k_s_res and k_s_dir_post, and once k_s_build_gs and k_s_update
LAUNCHES_PER_ITERATION = 95


def test_launches_per_iteration_with_s_blocks():
    """Launches of one lock-step iteration of a QP batch with 'l', 'q' and 's' rows, p > 0, refinement 1 and one
    sub-batch: the difference between maxiters = 3 and maxiters = 2, where no problem finishes earlier"""
    import cvxopt_b200 as cb
    dims = {"l": 6, "q": [4], "s": [5, 3]}
    batch = sdqp_batch_data(4, 14, dims, 2, 8800, pkind="random")      # P > 0: 10 rows of G are enough without 's'
    counts = []
    for k in (2, 3):
        l0 = cb.launch_count()
        r = _solve(batch, dims, nsub=1, maxiters=k)
        counts.append(cb.launch_count() - l0)
        assert list(r["iterations"]) == [k] * 4
    P, q, G, h, A, b = batch
    base = []
    for k in (2, 3):                       # the same problems without their 's' rows, through qp_batch
        l0 = cb.launch_count()
        cb.qp_batch(P, q, G[:, :10], h[:, :10], A, b, nsub=1, dims={"l": 6, "q": [4]}, maxiters=k)
        base.append(cb.launch_count() - l0)
    print("\nlaunches per lock-step iteration of a QP batch with 's' blocks: %d, without them: %d"
          % (counts[1] - counts[0], base[1] - base[0]))
    assert counts[1] - counts[0] == LAUNCHES_PER_ITERATION
    assert (counts[1] - counts[0]) - (base[1] - base[0]) == 10

