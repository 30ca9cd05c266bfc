"""Batched cpl problems (cpl_batch, cvxb_batch_create_cpl) against a Python loop over the reference's solvers.cpl
(oracle/_ref), problem by problem, on tests/cpl_problems.py's families: converged solutions and iteration counts,
iterates after 1-3 iterations at refinement 0-2, the backtracking into dom f, the relaxed line search with 'q' cones,
the Rank error, compaction, device memory and launches.  The reference's cpl returns no iteration count; it is counted
by wrapping misc.update_scaling, which cpl calls once per completed iteration."""
import numpy as np
import pytest

from cpl_problems import MNL, cpl_batch_data, ref_F, torch_F

pytestmark = pytest.mark.gpu

KEYS = ("x", "snl", "sl", "znl", "zl", "y")


def _m(v):
    from cvxopt import matrix
    return matrix(np.ascontiguousarray(v, dtype=np.float64))


def ref_cpl_loop(ref, family, d, calls=None, **options):
    """solvers.cpl over the batch: per problem its result dict and 'iterations'; calls['none'] counts F's None
    returns"""
    from cvxopt import misc, solvers
    out = []
    orig = misc.update_scaling
    count = [0]

    def counted(*a, **k):
        count[0] += 1
        return orig(*a, **k)
    misc.update_scaling = counted
    try:
        for k in range(d["x0"].shape[0]):
            count[0] = 0
            kw = {}
            if d["G"].shape[1]:
                kw.update(G=_m(d["G"][k]), h=_m(d["h"][k]))
            if d["A"].shape[1]:
                kw.update(A=_m(d["A"][k]), b=_m(d["b"][k]))
            r = dict(solvers.cpl(_m(d["c"][k]), ref_F(family, d["data"], k, d["x0"][k], calls), dims=d["dims"],
                                 options=dict(show_progress=False, **options), **kw))
            r["iterations"] = count[0]
            out.append(r)
    finally:
        misc.update_scaling = orig
    return out


def cpl_solve(family, d, seen=None, F=None, **kw):
    import cvxopt_b200
    F = F or torch_F(family, d["data"], d["x0"], 0, seen)
    p = d["A"].shape[1]
    return cvxopt_b200.cpl_batch(d["c"], F, d["G"] if d["G"].shape[1] else None, d["h"] if d["G"].shape[1] else None,
                                 d["dims"], d["A"] if p else None, d["b"] if p else None, **kw)


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64).ravel(), np.asarray(b, dtype=np.float64).ravel()
    if a.size == 0:
        return 0.0
    return np.linalg.norm(a - b) / max(1.0, np.linalg.norm(b))


def assert_matches(out, refs, vec_tol, obj_tol):
    """status and iterations equal, vectors within vec_tol relative, objectives within obj_tol; -> largest error"""
    worst = 0.0
    for k, r in enumerate(refs):
        assert out["status"][k] == r["status"], (k, out["status"][k], r["status"])
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


SHAPES = [  # family, n, q, ml, p, B
    ("socp", 16, [3, 5, 10], 4, 0, 24),     # mnl = 2, three cones of different lengths
    ("socp", 16, [3, 5, 10], 4, 3, 257),    # with A; several sub-batches, compaction
    ("logcone", 12, [4, 6], 0, 2, 20),      # 'q' cones only, restricted domain
    ("conelp", 10, [3, 7], 5, 0, 12),       # mnl = 0: H = 0
    ("socp", 16, [], 6, 0, 12),             # 'l' rows only
    ("conelp", 24, [8], 3, 2, 1),           # B = 1
]


@pytest.mark.parametrize("family,n,q,ml,p,B", SHAPES)
def test_converged_parity(ref, family, n, q, ml, p, B):
    d = cpl_batch_data(family, range(100, 100 + B), n, q, ml, p)
    refs = ref_cpl_loop(ref, family, d)
    out = cpl_solve(family, d)
    assert_matches(out, refs, 1e-6, 1e-8)
    assert all(s == "optimal" for s in out["status"])
    assert out["snl"].shape == (B, MNL[family]) and out["sl"].shape == (B, d["G"].shape[1])


@pytest.mark.parametrize("refinement", [0, 1, 2])
@pytest.mark.parametrize("maxiters", [1, 2, 3])
@pytest.mark.parametrize("family,n,q,ml,p", [("socp", 12, [3, 5], 2, 2), ("logcone", 10, [4], 0, 2),
                                             ("conelp", 8, [3], 3, 0)])
def test_iterates(ref, family, n, q, ml, p, maxiters, refinement):
    d = cpl_batch_data(family, range(8), n, q, ml, p)
    refs = ref_cpl_loop(ref, family, d, maxiters=maxiters, refinement=refinement)
    out = cpl_solve(family, d, maxiters=maxiters, refinement=refinement)
    worst = assert_matches(out, refs, 1e-12, 1e-12)
    print("iterates %s maxiters=%d refinement=%d: largest relative error %.2e" % (family, maxiters, refinement, worst))


def test_domain_backtracking(ref):
    """logcone's steps leave x > 0: the reference's F returns None there, and the batch's F sees non-finite rows in
    its domain rounds"""
    d = cpl_batch_data("logcone", range(20), 16, [3], 0, 0)
    calls, seen = {}, {}
    refs = ref_cpl_loop(ref, "logcone", d, calls)
    out = cpl_solve("logcone", d, seen)
    assert calls.get("none", 0) > 0 and seen.get("nonfinite", 0) > 0, (calls, seen)
    assert_matches(out, refs, 1e-6, 1e-8)
    print("logcone: reference None returns %d, batch evaluations with non-finite rows %d, rounds %d"
          % (calls["none"], seen["nonfinite"], out["line_search_rounds"]))


def _relaxed_trace(ref, family, d):
    """per problem of `d`: whether the reference's cpl entered a relaxed line search (relaxed_iters became 1, saving W
    with its v and beta) and whether it resumed one (8 -> -1, restoring them), read from cpl's locals"""
    import sys
    from cvxopt import solvers
    out = []
    for k in range(d["x0"].shape[0]):
        vals = []

        def local(frame, event, arg):
            r = frame.f_locals.get("relaxed_iters")
            if r is not None and (not vals or vals[-1] != r):
                vals.append(r)
            return local
        kw = dict(G=_m(d["G"][k]), h=_m(d["h"][k]))
        if d["A"].shape[1]:
            kw.update(A=_m(d["A"][k]), b=_m(d["b"][k]))
        sys.settrace(lambda frame, event, arg: local if frame.f_code.co_name == "cpl" else None)
        try:
            solvers.cpl(_m(d["c"][k]), ref_F(family, d["data"], k, d["x0"][k]), dims=d["dims"],
                        options=dict(show_progress=False), **kw)
        finally:
            sys.settrace(None)
        out.append((1 in vals, any(a == 8 and b == -1 for a, b in zip(vals, vals[1:]))))
    return out


def test_relaxed_line_search_with_cones(ref):
    """lsecone (a GP in cpl's epigraph form with a 'q' cone of length 3), 40 seeds: many problems enter a relaxed line
    search, which saves W with its 'q' part (v0, beta0 in the state row), and seeds 23 and 29 run 8 relaxed iterations
    without sufficient decrease and resume the saved search, which restores it.  Status, iteration counts and
    solutions are the reference's, problem by problem"""
    d = cpl_batch_data("lsecone", range(40), 9, [3], 0, 0)
    trace = _relaxed_trace(ref, "lsecone", d)
    entered = [k for k, t in enumerate(trace) if t[0]]
    resumed = [k for k, t in enumerate(trace) if t[1]]
    assert resumed == [23, 29], resumed
    refs = ref_cpl_loop(ref, "lsecone", d)
    out = cpl_solve("lsecone", d)
    assert_matches(out, refs, 1e-6, 1e-8)
    print("lsecone sweep: relaxed searches entered by %d problems, resumed by %s (iterations %s); all iterations %s"
          % (len(entered), resumed, [int(out["iterations"][k]) for k in resumed],
             [int(k) for k in out["iterations"]]))


def test_rank_error_names_the_problem(ref):
    d = cpl_batch_data("conelp", range(6), 8, [3], 3, 0)
    d["G"][4] = 0.0                              # problem 4: Rank([H; A; Df; G]) < n (H = 0, mnl = 0)
    with pytest.raises(ValueError, match="problem 4: Rank"):
        cpl_solve("conelp", d, nsub=2)


def _same(a, b):
    for key in KEYS + ("iterations", "primal objective", "dual objective"):
        assert np.array_equal(np.asarray(a[key]), np.asarray(b[key])), key
    assert list(a["status"]) == list(b["status"])


def test_compaction_resolves_and_nsub(monkeypatch):
    """the same bits with compaction on and off, across re-solves of one batch and under nsub"""
    import cvxopt_b200
    d = cpl_batch_data("logcone", range(24), 12, [4, 6], 0, 2)
    F = torch_F("logcone", d["data"], d["x0"])
    base = cpl_solve("logcone", d, F=F, nsub=1)
    monkeypatch.setenv("CVXB_BATCH_COMPACT", "0")
    _same(cpl_solve("logcone", d, F=F, nsub=1), base)
    monkeypatch.delenv("CVXB_BATCH_COMPACT")
    bt = cvxopt_b200.CPLBatch(24, 12, 1, d["dims"], 2)
    try:
        bt.set_F(F)
        bt.load(d["c"], d["x0"], d["G"], d["h"], d["A"], d["b"])
        for _ in range(2):
            bt.solve()
            r = bt.results()
            assert np.array_equal(r["x"], base["x"]) and np.array_equal(r["iterations"], base["iterations"])
    finally:
        bt.close()
    three = cpl_solve("logcone", d, F=F, nsub=3)
    assert three["nsub"] == 3
    assert list(three["status"]) == list(base["status"]) and np.array_equal(three["iterations"], base["iterations"])
    assert np.allclose(three["x"], base["x"], rtol=1e-12, atol=1e-12)


def _ev(x):
    return (x + 1) & ~1


def test_device_memory():
    """what the header states: the eq batch of the same n, p and dims {'l': mnl + ml, 'q': q} with refinement 1, plus
    the callback's buffers, the per-slot vectors, x0, the state row's extra part and the ints"""
    import ctypes as C
    from cvxopt_b200 import CPLBatch, _lib, kkt
    lib = _lib.load()
    B, n, mnl, p, ml, q = 5, 9, 2, 3, 4, [3, 6]
    m = mnl + ml + sum(q)
    before = lib.cvxb_device_bytes()
    bt = CPLBatch(B, n, mnl, {"l": ml, "q": q}, p)
    cpl = lib.cvxb_device_bytes() - before
    bt.close()
    d, keep, _, _ = kkt.make_dims({"l": mnl + ml, "q": q, "s": []})
    h = C.c_void_p()
    assert lib.cvxb_batch_create_eq(C.byref(h), B, n, p, C.byref(d), 0) == 0
    assert lib.cvxb_batch_set_refinement(h, 1) == 0
    eq = lib.cvxb_device_bytes() - before
    lib.cvxb_batch_destroy(h)
    extra = 8 * B * (mnl * (n + 2) + n * n + mnl + 3 * n + p + 4 * m + n
                     + 56 + 3 * _ev(n) + 3 * _ev(p) + 10 * _ev(m) + _ev(sum(q)) + _ev(len(q))) + 4 * (B + 1)
    assert cpl - eq == extra, (cpl - eq, extra)
    assert lib.cvxb_device_bytes() == before


def test_cpl_batch_refuses_the_other_loads():
    from cvxopt_b200 import CPLBatch, CPBatch, _lib
    lib = _lib.load()
    bt = CPLBatch(2, 4, 1, {"l": 2, "q": [3]})
    cp = CPBatch(2, 4, 1, 2)
    try:
        v = np.zeros(64)
        a = v.ctypes.data
        assert lib.cvxb_batch_load(bt._h, a, a, a, a, _lib.HOST) == _lib.E_ARG
        assert lib.cvxb_batch_load_lp(bt._h, a, a, a, _lib.HOST) == _lib.E_ARG
        assert lib.cvxb_batch_load_gp(bt._h, a, a, a, a, _lib.HOST) == _lib.E_ARG
        assert lib.cvxb_batch_load_cp(bt._h, a, a, a, _lib.HOST) == _lib.E_ARG
        assert lib.cvxb_batch_load_start(bt._h, None, None, None, None, _lib.HOST) == _lib.E_ARG
        assert lib.cvxb_batch_load_cpl(cp._h, a, a, a, a, _lib.HOST) == _lib.E_ARG
        bt.load(np.ones((2, 4)), np.ones((2, 4)), np.zeros((2, 5, 4)), np.ones((2, 5)))
        assert lib.cvxb_batch_solve(bt._h, 10, 1e-7, 1e-6, 1e-7) == _lib.E_ARG      # no evaluator
        assert "cvxb_batch_set_cp_eval" in _lib.last_error()
    finally:
        bt.close()
        cp.close()


class _Boom(Exception):
    pass


def test_errors_from_F():
    from cvxopt_b200 import _lib
    lib = _lib.load()
    before = lib.cvxb_device_bytes()
    d = cpl_batch_data("socp", range(20), 10, [3, 4], 2, 0)
    F = torch_F("socp", d["data"], d["x0"])
    boom, n_full = _Boom("from F"), [0]

    def raising(x=None, z=None, idx=None):
        if z is not None:
            n_full[0] += 1
            if n_full[0] == 3:
                raise boom
        return F(x, z, idx=idx)
    with pytest.raises(_Boom) as e:
        cpl_solve("socp", d, F=raising, nsub=2)
    assert e.value is boom
    assert lib.cvxb_device_bytes() == before

    def wrong(x=None, z=None, idx=None):
        r = F(x, z, idx=idx)
        return r if x is None else (r[0][:, :1],) + tuple(r[1:])
    with pytest.raises(TypeError, match="first output argument of F"):
        cpl_solve("socp", d, F=wrong)
    assert lib.cvxb_device_bytes() == before

    e = cpl_batch_data("logcone", range(20), 8, [3], 0, 0)
    e["x0"][13, 2] = -1.0
    with pytest.raises(ValueError, match="problem 13: x0 not in the domain of f"):
        cpl_solve("logcone", e, nsub=2)
    assert lib.cvxb_device_bytes() == before


# launches of one lock-step iteration of the 8-problem batch below with compaction off: its two directions, each
# followed by one domain round and one line-search round (4 rounds per iteration, also pinned)
CPL_PER_ITER, CPL_ROUNDS_PER_ITER = 102, 4


def test_launches_per_iteration(monkeypatch):
    """launches and line-search rounds per lock-step iteration (maxiters 2 -> 3 -> 4 on a batch whose problems all
    run past 4 iterations), pinned"""
    import cvxopt_b200
    monkeypatch.setenv("CVXB_BATCH_COMPACT", "0")
    d = cpl_batch_data("socp", range(8), 12, [3, 5], 2, 2)
    F = torch_F("socp", d["data"], d["x0"])
    counts, rounds = [], []
    for maxiters in (2, 3, 4):
        c0 = cvxopt_b200.launch_count()
        out = cpl_solve("socp", d, F=F, nsub=1, maxiters=maxiters)
        counts.append(cvxopt_b200.launch_count() - c0)
        rounds.append(out["line_search_rounds"])
    print("cpl launches at maxiters 2, 3, 4:", counts, "line-search rounds:", rounds)
    assert counts[1] - counts[0] == counts[2] - counts[1] == CPL_PER_ITER
    assert rounds[1] - rounds[0] == rounds[2] - rounds[1] == CPL_ROUNDS_PER_ITER
