"""Batched geometric programs (gp_batch, cvxb_batch_create_gp) against a Python loop over the reference's solvers.gp
(oracle/_ref), problem by problem: converged solutions and iteration counts, iterates after 1-3 iterations at
refinement 0-2, the relaxed line search's iteration counts, iteration 0's Rank error and S + A'A switch, and the batch
mechanics (compaction, re-solves, sub-batches, device memory, launches).  The reference's gp returns no iteration
count; it is counted by wrapping misc.update_scaling, which cpl calls once per completed iteration."""
import numpy as np
import pytest

from gp_problems import gp_batch_data

pytestmark = pytest.mark.gpu

KEYS = ("x", "snl", "sl", "znl", "zl", "y")


def _m(v):
    from cvxopt import matrix
    return matrix(np.ascontiguousarray(v, dtype=np.float64))


def ref_gp_loop(ref, K, data, **options):
    """solvers.gp over the batch: per problem its result dict and 'iterations'"""
    from cvxopt import misc, solvers
    F, g, G, h, A, b = data
    out = []
    orig = misc.update_scaling
    count = [0]

    def counted(*a, **k):
        count[0] += 1
        return orig(*a, **k)
    misc.update_scaling = counted
    try:
        for k in range(F.shape[0]):
            count[0] = 0
            eq = (_m(A[k]), _m(b[k])) if A.shape[1] else (None, None)
            Gk, hk = (_m(G[k]), _m(h[k])) if G.shape[1] else (None, None)
            r = solvers.gp(list(K), _m(F[k]), _m(g[k]), Gk, hk, *eq, options=dict(show_progress=False, **options))
            r = dict(r)
            r["iterations"] = count[0]
            out.append(r)
    finally:
        misc.update_scaling = orig
    return out


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64).ravel(), np.asarray(b, dtype=np.float64).ravel()
    if a.size == 0:
        return 0.0
    return np.linalg.norm(a - b) / max(1.0, np.linalg.norm(b))


def assert_matches(out, refs, vec_tol, obj_tol, iters=True):
    """status and iterations equal, vectors within vec_tol relative, objectives within obj_tol; -> largest error"""
    worst = 0.0
    for k, r in enumerate(refs):
        assert out["status"][k] == r["status"], (k, out["status"][k], r["status"])
        if iters:
            assert out["iterations"][k] == r["iterations"], (k, out["iterations"][k], r["iterations"])
        for key in KEYS:
            e = _rel(out[key][k], np.array(r[key]))
            worst = max(worst, e)
            assert e <= vec_tol, (k, key, e)
        for key in ("primal objective", "dual objective"):
            e = abs(out[key][k] - r[key]) / max(1.0, abs(r[key]))
            worst = max(worst, e)
            assert e <= obj_tol, (k, key, e)
    return worst


SHAPES = [  # n, K, r, p, B
    (16, [32, 8, 8, 8], 4, 0, 257),
    (32, [64] + [8] * 8, 8, 2, 24),
    (64, [128] + [16] * 8, 16, 4, 12),
    (16, [32], 4, 0, 16),               # mnl = 0
    (32, [64] + [8] * 8, 8, 2, 1),      # B = 1
]


@pytest.mark.parametrize("n,K,r,p,B", SHAPES)
def test_converged_parity(ref, n, K, r, p, B):
    import cvxopt_b200
    data = gp_batch_data(range(100, 100 + B), n, K, r, p)
    refs = ref_gp_loop(ref, K, data)
    F, g, G, h, A, b = data
    out = cvxopt_b200.gp_batch(K, F, g, G, h, A if p else None, b if p else None)
    assert_matches(out, refs, 1e-6, 1e-8)
    assert all(s == "optimal" for s in out["status"])


@pytest.mark.parametrize("refinement", [0, 1, 2])
@pytest.mark.parametrize("maxiters", [1, 2, 3])
def test_iterates(ref, maxiters, refinement):
    import cvxopt_b200
    n, K, r, p = 16, [32, 8, 8, 8], 4, 2
    data = gp_batch_data(range(8), n, K, r, p)
    refs = ref_gp_loop(ref, K, data, maxiters=maxiters, refinement=refinement)
    out = cvxopt_b200.gp_batch(K, *data, maxiters=maxiters, refinement=refinement)
    worst = assert_matches(out, refs, 1e-12, 1e-12)
    print("iterates maxiters=%d refinement=%d: largest relative error %.2e" % (maxiters, refinement, worst))


def test_relaxed_line_search_iteration_counts(ref):
    """n = 8, K = [4, 4, 4], only the box rows: seeds 6 and 29 enter relaxed_iters = -1 for good (:1178 compares)
    and take 45 and 44 iterations; every count equals the reference's"""
    import cvxopt_b200
    K = [4, 4, 4]
    data = gp_batch_data(range(40), 8, K, 0, 0)
    refs = ref_gp_loop(ref, K, data)
    out = cvxopt_b200.gp_batch(K, *data[:4])
    its = [r["iterations"] for r in refs]
    assert its[6] == 45 and its[29] == 44, (its[6], its[29])
    assert list(out["iterations"]) == its
    assert_matches(out, refs, 1e-6, 1e-8)


def _switch_batch(B, switch, p=3):
    """n = 4, K = [1, 2], G = [I; -I], p rows of A.  Where `switch`, G keeps only its e1 rows, f1's two rows are equal
    with equal g1 and zero in the last two columns: H = 0 exactly (K0 = 1 and equal rows), so S = H + Df1'Df1 + G'G
    has an exactly zero trailing 2 x 2 block at the start, and S + A'A has full rank"""
    F, g, G, h, A, b = gp_batch_data(range(200, 200 + B), 4, [1, 2], 0, p)
    for k in switch:
        G[k, [1, 2, 3, 5, 6, 7]] = 0.0
        F[k, 2] = F[k, 1]
        F[k, 1:, 2:] = 0.0
        g[k, 1:] = np.log(0.25)
    return F, g, G, h, A, b


def test_iteration0_switch_with_parity(ref):
    import cvxopt_b200
    data = _switch_batch(6, [1, 4])
    refs = ref_gp_loop(ref, [1, 2], data)
    out = cvxopt_b200.gp_batch([1, 2], *data)
    assert_matches(out, refs, 1e-6, 1e-8)


def test_iteration0_rank_error_names_the_problem(ref):
    """without A the singular S of problem 1 stays singular: gp's ValueError at iteration 0"""
    import cvxopt_b200
    from cvxopt import solvers
    F, g, G, h, A, b = _switch_batch(3, [1], p=0)
    with pytest.raises(ValueError, match="Rank"):
        solvers.gp([1, 2], _m(F[1]), _m(g[1]), _m(G[1]), _m(h[1]), options=dict(show_progress=False))
    for k in (0, 2):
        solvers.gp([1, 2], _m(F[k]), _m(g[k]), _m(G[k]), _m(h[k]), options=dict(show_progress=False, maxiters=1))
    with pytest.raises(ValueError, match=r"problem 1: Rank\(A\) < p or Rank\(\[H\(x\); A; Df\(x\); G\]\) < n"):
        cvxopt_b200.gp_batch([1, 2], F, g, G, h)


def _solve(data, K, **kw):
    import cvxopt_b200
    F, g, G, h, A, b = data
    return cvxopt_b200.gp_batch(K, F, g, G, h, A, b, **kw)


def _same(a, b):
    for key in KEYS + ("iterations", "primal objective", "dual objective"):
        assert np.array_equal(np.asarray(a[key]), np.asarray(b[key])), key
    assert list(a["status"]) == list(b["status"])


def test_layout_bit_identical(monkeypatch):
    """compaction off, a second solve of the same handle and other sub-batch counts give the same bits"""
    from cvxopt_b200 import GPBatch
    K = [32, 8, 8, 8]
    data = gp_batch_data(range(24), 16, K, 4, 2)
    base = _solve(data, K, nsub=1)
    for nsub in (2, 3):
        _same(base, _solve(data, K, nsub=nsub))
    monkeypatch.setenv("CVXB_BATCH_COMPACT", "0")
    _same(base, _solve(data, K, nsub=1))
    monkeypatch.delenv("CVXB_BATCH_COMPACT")
    bt = GPBatch(24, 16, K, 36, p=2)
    try:
        bt.load(*data)
        bt.solve()
        r1 = bt.results()
        bt.solve()
        r2 = bt.results()
    finally:
        bt.close()
    for key in ("x", "s", "z", "y", "iterations", "primal objective"):
        assert np.array_equal(r1[key], r2[key])
        assert np.array_equal(r1[key], np.concatenate([base["snl"], base["sl"]], 1) if key == "s" else
                              np.concatenate([base["znl"], base["zl"]], 1) if key == "z" else base[key])


def test_device_bytes_return_after_destroy():
    from cvxopt_b200 import GPBatch, _lib
    lib = _lib.load()
    before = lib.cvxb_device_bytes()
    bt = GPBatch(5, 16, [32, 8, 8, 8], 36, p=2)
    assert lib.cvxb_device_bytes() > before
    bt.load(*gp_batch_data(range(5), 16, [32, 8, 8, 8], 4, 2))
    bt.solve(refinement=2)
    bt.close()
    assert lib.cvxb_device_bytes() == before


def test_gp_batch_refuses_the_other_loads():
    from cvxopt_b200 import GPBatch, _lib
    lib = _lib.load()
    bt = GPBatch(2, 4, [3, 2], 2)
    try:
        d = np.zeros(64)
        assert lib.cvxb_batch_load(bt._h, d.ctypes.data, d.ctypes.data, d.ctypes.data, d.ctypes.data,
                                   _lib.HOST) == _lib.E_ARG
        assert lib.cvxb_batch_load_lp(bt._h, d.ctypes.data, d.ctypes.data, d.ctypes.data, _lib.HOST) == _lib.E_ARG
        assert lib.cvxb_batch_load_start(bt._h, None, None, None, None, _lib.HOST) == _lib.E_ARG
    finally:
        bt.close()


# launches of one lock-step iteration without the line search, and of one line-search round, for the batch below
# (8 problems, n = 16, K = [32, 8, 8, 8], r = 4, p = 0, refinement 1, compaction off): every iteration after the first
# runs the same kernels, and every round the same 7 (trial point, F x in two GEMV kernels, F, two GEMVs for newrx,
# decision)
PER_ITER, PER_ROUND = 56, 7


def test_launches_per_iteration(monkeypatch):
    import cvxopt_b200
    from cvxopt_b200 import GPBatch
    monkeypatch.setenv("CVXB_BATCH_COMPACT", "0")
    K = [32, 8, 8, 8]
    data = gp_batch_data(range(8), 16, K, 4, 0)
    counts = []
    for maxiters in (2, 3, 4):
        bt = GPBatch(8, 16, K, 36)
        try:
            bt.load(*data[:4])
            before = cvxopt_b200.launch_count()
            bt.solve(maxiters=maxiters)
            counts.append((cvxopt_b200.launch_count() - before, bt.stats()["line_search_rounds"]))
        finally:
            bt.close()
    d1 = counts[1][0] - counts[0][0] - PER_ROUND * (counts[1][1] - counts[0][1])
    d2 = counts[2][0] - counts[1][0] - PER_ROUND * (counts[2][1] - counts[1][1])
    print("launches (total, rounds) at maxiters 2, 3, 4:", counts, "per iteration:", d1, d2)
    assert d1 == d2
    if PER_ITER is not None:
        assert d1 == PER_ITER
