"""Batched convex QCQPs (qcqp_batch, cvxb_batch_create_qcqp) against a Python loop over the reference's solvers.cp
(oracle/_ref) with the same quadratic F, problem by problem, on tests/qcqp_problems.py: converged solutions and
iteration counts, iterates after 1-3 iterations at refinement 0-2, cp_problems' qcqp family through both qcqp_batch and
cp_batch, a 40-seed sweep, the rank errors, compaction, re-solves, device memory and launches.  The reference's cp
returns no iteration count; it is counted by wrapping misc.update_scaling, which cpl calls once per completed
iteration."""
import ctypes as C
import sys

import numpy as np
import pytest

from qcqp_problems import qcqp_batch_data, ref_F

pytestmark = pytest.mark.gpu

KEYS = ("x", "snl", "sl", "znl", "zl", "y")


def _m(v):
    from cvxopt import matrix
    return matrix(np.ascontiguousarray(v, dtype=np.float64))


def ref_qcqp_loop(ref, d, relaxed=None, **options):
    """solvers.cp over the batch: per problem its result dict and 'iterations'.  relaxed: a list that gets, per
    problem, whether cpl entered a relaxed line search (its relaxed_iters went above 0)"""
    from cvxopt import cvxprog, misc, solvers
    out = []
    orig = misc.update_scaling
    count, seen = [0], [0]

    def counted(*a, **k):
        count[0] += 1
        return orig(*a, **k)

    def tracer(frame, event, arg):
        if frame.f_code is cvxprog.cpl.__code__:
            def local(fr, ev, a):
                if fr.f_locals.get("relaxed_iters", 0) > 0:
                    seen[0] = 1
                return local
            return local
        return None
    misc.update_scaling = counted
    try:
        for k in range(d["x0"].shape[0]):
            count[0] = seen[0] = 0
            kw = {}
            if d["G"].shape[1]:
                kw.update(G=_m(d["G"][k]), h=_m(d["h"][k]))
            if d["A"].shape[1]:
                kw.update(A=_m(d["A"][k]), b=_m(d["b"][k]))
            if relaxed is not None:
                sys.settrace(tracer)
            try:
                r = dict(solvers.cp(ref_F(d, k), options=dict(show_progress=False, **options), **kw))
            finally:
                sys.settrace(None)
            r["iterations"] = count[0]
            out.append(r)
            if relaxed is not None:
                relaxed.append(seen[0])
    finally:
        misc.update_scaling = orig
    return out


def qcqp_solve(d, **kw):
    import cvxopt_b200
    ml, p = d["G"].shape[1], d["A"].shape[1]
    return cvxopt_b200.qcqp_batch(d["P"], d["q"], d["r"], d["G"] if ml else None, d["h"] if ml else None, None,
                                  d["A"] if p else None, d["b"] if p else None, x0=d["x0"], **kw)


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


def _switches(d, kind):
    """deficient: every problem's S at iteration 0 (z0 P_0, no G rows) has no Cholesky factor in exact arithmetic, so
    the reference and the batch both switch to S + A'A"""
    if kind == "deficient":
        from qcqp_problems import sym
        for P in d["P"]:
            with pytest.raises(np.linalg.LinAlgError):
                np.linalg.cholesky(sym(P)[0])


SHAPES = [  # n, mnl, p, r, B, kind
    (16, 3, 0, 4, 12, "quad"),
    (16, 0, 2, 4, 20, "quad"),          # mnl = 0: a QP through cp's algorithm
    (24, 8, 3, 6, 257, "quad"),         # several sub-batches, compaction
    (32, 2, 0, 8, 1, "quad"),           # B = 1
    (16, 2, 2, 4, 16, "linear"),        # P_0 = 0
    (12, 0, 4, 0, 10, "deficient"),     # S singular at iteration 0: S + A'A
]


@pytest.mark.parametrize("n,mnl,p,r,B,kind", SHAPES)
def test_converged_parity(ref, n, mnl, p, r, B, kind):
    d = qcqp_batch_data(range(100, 100 + B), n, mnl, p, r, kind)
    _switches(d, kind)
    if kind == "quad" and p:                       # a start away from 0
        d["x0"] = np.random.Generator(np.random.PCG64(7)).uniform(-1.0, 1.0, d["x0"].shape)
    refs = ref_qcqp_loop(ref, d)
    out = qcqp_solve(d)
    worst = assert_matches(out, refs, 1e-6, 1e-8)
    assert all(s == "optimal" for s in out["status"])
    assert out["snl"].shape == (B, d["P"].shape[1] - 1) and out["sl"].shape == (B, d["G"].shape[1])
    print("converged %s n=%d mnl=%d p=%d B=%d: largest relative error %.2e" % (kind, n, mnl, p, B, worst))


@pytest.mark.parametrize("refinement", [0, 1, 2])
@pytest.mark.parametrize("maxiters", [1, 2, 3])
@pytest.mark.parametrize("n,mnl,p,r,kind", [(12, 3, 2, 4, "quad"), (12, 2, 2, 4, "linear"), (10, 0, 3, 0, "deficient")])
def test_iterates(ref, n, mnl, p, r, kind, maxiters, refinement):
    d = qcqp_batch_data(range(8), n, mnl, p, r, kind)
    _switches(d, kind)
    refs = ref_qcqp_loop(ref, d, maxiters=maxiters, refinement=refinement)
    out = qcqp_solve(d, maxiters=maxiters, refinement=refinement)
    worst = assert_matches(out, refs, 1e-12, 1e-12)
    print("iterates %s maxiters=%d refinement=%d: largest relative error %.2e" % (kind, maxiters, refinement, worst))


@pytest.mark.parametrize("maxiters", [2, 100])
def test_cp_family_through_qcqp_and_cp_batch(maxiters):
    """cp_problems' qcqp family: the library's F and cp_batch's torch F take the same iterations, to 1e-12"""
    import cvxopt_b200
    from cp_problems import cp_batch_data, torch_F
    d = cp_batch_data("qcqp", range(24), 16, 0, 4)
    D = d["data"]
    qc = cvxopt_b200.qcqp_batch(D["P"], D["q"], D["r"], d["G"], d["h"], x0=d["x0"], maxiters=maxiters)
    cp = cvxopt_b200.cp_batch(torch_F("qcqp", D, d["x0"]), d["G"], d["h"], maxiters=maxiters)
    assert list(qc["status"]) == list(cp["status"])
    assert np.array_equal(qc["iterations"], cp["iterations"])
    worst = 0.0
    for key in KEYS + ("primal objective", "dual objective"):
        for k in range(24):
            e = _rel(qc[key][k], cp[key][k])
            worst = max(worst, e)
            assert e <= 1e-12, (key, k, e)
    print("qcqp_batch vs cp_batch maxiters=%d: largest relative difference %.2e, iterations %s"
          % (maxiters, worst, np.bincount(qc["iterations"]).nonzero()[0].tolist()))


def test_seed_sweep(ref):
    """40 seeds: the reference's iteration count for every one; how many enter a relaxed line search is reported"""
    d = qcqp_batch_data(range(40), 16, 4, 2, 6)
    relaxed = []
    refs = ref_qcqp_loop(ref, d, relaxed)
    out = qcqp_solve(d)
    assert_matches(out, refs, 1e-6, 1e-8)
    print("sweep: iterations %s, %d of 40 problems enter a relaxed line search"
          % (out["iterations"].tolist(), sum(relaxed)))


def test_rank_errors_name_the_problem():
    import cvxopt_b200
    d = qcqp_batch_data(range(6), 8, 1, 2, 2)
    with pytest.raises(ValueError, match=r"Rank\(A\) < p or Rank\(\[H\(x\); A; Df\(x\); G\]\) < n"):
        cvxopt_b200.qcqp_batch(d["P"], d["q"], d["r"], d["G"], d["h"], A=np.zeros((6, 9, 8)), b=np.zeros((6, 9)))
    # problem 5: P_0 = P_1 = 0, no G rows, one row of A: S + A'A is singular at iteration 0
    e = qcqp_batch_data(range(6), 8, 1, 1, 0, "quad")
    e["P"][5] = 0.0
    e["G"], e["h"] = e["G"][:, :0], e["h"][:, :0]
    with pytest.raises(ValueError, match=r"problem 5: Rank\(A\) < p or Rank\(\[H\(x\); A; Df\(x\); G\]\) < n"):
        qcqp_solve(e, nsub=2)


def _same(a, b):
    for key in KEYS + ("iterations", "primal objective", "dual objective"):
        assert np.array_equal(np.asarray(a[key]), np.asarray(b[key])), key
    assert list(a["status"]) == list(b["status"])


def _alone(iters, nsub):
    """the problems that run alone at the end of their sub-batch (problem i is in sub-batch i mod nsub): the only one
    with its sub-batch's most iterations"""
    out = set()
    for r in range(nsub):
        sub = iters[r::nsub]
        if np.sum(sub == sub.max()) == 1:
            out.add(r + nsub * int(np.argmax(sub)))
    return out


def _same_but_alone(a, b, alone):
    """a and b: equal status and iterations, the same bits except for problems in `alone` (a single active slot takes
    the factorisation's single-matrix SYRK, which sums in another order), which agree to 1e-13; -> those that differ"""
    assert list(a["status"]) == list(b["status"]) and np.array_equal(a["iterations"], b["iterations"])
    moved = set()
    for key in KEYS + ("primal objective", "dual objective"):
        assert np.allclose(a[key], b[key], rtol=1e-13, atol=1e-15), key
        moved |= {k for k in range(len(a["status"])) if not np.array_equal(a[key][k], b[key][k])}
    assert moved <= alone, (sorted(moved), sorted(alone))
    return moved


def test_compaction_resolves_and_subbatches(monkeypatch):
    """compaction off, and four sub-batches instead of two: the same bits except for a problem that ran alone at the end
    of its sub-batch in either run; a re-solve of one batch object: the same bits"""
    import cvxopt_b200
    from cvxopt_b200 import QCQPBatch
    d = qcqp_batch_data(range(40), 12, 3, 2, 4)
    base = qcqp_solve(d, nsub=2)
    monkeypatch.setenv("CVXB_BATCH_COMPACT", "0")
    off = qcqp_solve(d, nsub=2)
    monkeypatch.delenv("CVXB_BATCH_COMPACT")
    assert list(off["status"]) == list(base["status"]) and np.array_equal(off["iterations"], base["iterations"])
    moved = _same_but_alone(off, base, _alone(base["iterations"], 2))
    print("compaction off: problems with other bits", sorted(moved))
    _same(qcqp_solve(d, nsub=2), base)
    s4 = qcqp_solve(d, nsub=4)
    moved = _same_but_alone(s4, base, _alone(base["iterations"], 2) | _alone(base["iterations"], 4))
    print("nsub 4 against nsub 2: problems with other bits", sorted(moved))
    bt = QCQPBatch(40, 12, 3, 28, p=2)
    try:
        bt.load(d["P"], d["q"], d["r"], d["x0"], d["G"], d["h"], d["A"], d["b"])
        bt.solve()
        r1 = bt.results()
        bt.solve()
        r2 = bt.results()
    finally:
        bt.close()
    for key in ("x", "s", "z", "y", "iterations", "primal objective", "dual objective"):
        assert np.array_equal(r1[key], r2[key]), key


def _ev(x):
    return (x + 1) & ~1


def test_device_bytes_match_the_header():
    """what cvxb_batch_create_eq's batch of the same n, p and dims {'l': m} holds with refinement 1, except G and the
    GEMV workspace, plus the QC batch's own buffers (include/cvxopt_b200.h)"""
    from cvxopt_b200 import QCQPBatch, _lib, kkt
    lib = _lib.load()
    B, n, mnl, ml, p = 5, 16, 2, 36, 2
    m, nK = mnl + ml, mnl + 1
    S = nK * n
    before = lib.cvxb_device_bytes()
    bt = QCQPBatch(B, n, mnl, ml, p=p)
    qc = lib.cvxb_device_bytes() - before
    d = qcqp_batch_data(range(B), n, mnl, p, ml - 2 * n)
    bt.load(d["P"], d["q"], d["r"], d["x0"], d["G"], d["h"], d["A"], d["b"])
    bt.solve(refinement=2)
    bt.close()
    assert lib.cvxb_device_bytes() == before
    dd, keep, _, _ = kkt.make_dims({"l": m, "q": [], "s": []})
    h = C.c_void_p()
    assert lib.cvxb_batch_create_eq(C.byref(h), B, n, p, C.byref(dd), 0) == 0
    assert lib.cvxb_batch_set_refinement(h, 1) == 0
    eq = lib.cvxb_device_bytes() - before
    lib.cvxb_batch_destroy(h)

    def ch(c):
        return max(1, -(-c // 128))

    def ldg(rows):
        return max(2, _ev(rows))
    ws_qc = max(max(m, S) * ch(n), p * ch(n), n * ch(p))
    ws_eq = max(m * ch(n), p * ch(n), n * ch(p))
    extra = 8 * B * ((ldg(m + S) - ldg(m)) * n + ws_qc - ws_eq + S + nK + 3 * n + p + 4 * m + S + nK + n
                     + _ev(S + nK) + 56 + 3 * _ev(n) + 3 * _ev(p) + 10 * _ev(m)) + 4 * (B + 1)
    assert qc - eq == extra, (qc - eq, extra)
    assert lib.cvxb_device_bytes() == before


def test_qcqp_batch_refuses_the_other_loads():
    from cvxopt_b200 import CPBatch, QCQPBatch, _lib
    lib = _lib.load()
    bt = QCQPBatch(2, 4, 1, 2)
    cp = CPBatch(2, 4, 1, 2)
    try:
        v = np.zeros(256)
        a = v.ctypes.data
        assert lib.cvxb_batch_load(bt._h, a, a, a, a, _lib.HOST) == _lib.E_ARG
        assert lib.cvxb_batch_load_lp(bt._h, a, a, a, _lib.HOST) == _lib.E_ARG
        assert lib.cvxb_batch_load_gp(bt._h, a, a, a, a, _lib.HOST) == _lib.E_ARG
        assert lib.cvxb_batch_load_cp(bt._h, a, a, a, _lib.HOST) == _lib.E_ARG
        assert lib.cvxb_batch_load_cpl(bt._h, a, a, a, a, _lib.HOST) == _lib.E_ARG
        assert lib.cvxb_batch_load_start(bt._h, None, None, None, None, _lib.HOST) == _lib.E_ARG
        assert lib.cvxb_batch_set_cp_eval(bt._h, None, None) == _lib.E_ARG
        assert lib.cvxb_batch_load_qcqp(cp._h, a, a, a, a, a, a, _lib.HOST) == _lib.E_ARG
        assert "not a QCQP batch" in _lib.last_error()
    finally:
        bt.close()
        cp.close()


# launches of one lock-step iteration without its line-search rounds, and of one round, for the 8-problem batch below
# (n = 16, mnl = 3, 36 'l' rows, p = 0, refinement 1, compaction off).  A round is k_gp_trial, P x (two GEMV kernels),
# k_qc_eval<false>, G'newzl and k_gp_ls.  The iteration: F at the iterate (two GEMV kernels and k_qc_eval<true>),
# k_qc_rx, the residual GEMVs and statistics, the scaling, k_qc_hessian and the factorisation, two directions
QC_PER_ITER, QC_PER_ROUND = 55, 6
# the CP batch's launches per lock-step iteration on cp_problems' qcqp family (8 problems, n = 16, r = 4), whose
# domain and line-search rounds are pinned too: two of each per iteration
CP_PER_ITER, CP_ROUNDS_PER_ITER = 66, 4


def test_launches_per_iteration(monkeypatch):
    """QC: launches per iteration and per line-search round, pinned.  GP and CP launch what they launched before"""
    import cvxopt_b200
    import test_batch_gp_gpu
    from cp_problems import cp_batch_data, torch_F
    test_batch_gp_gpu.test_launches_per_iteration(monkeypatch)
    monkeypatch.setenv("CVXB_BATCH_COMPACT", "0")
    d = qcqp_batch_data(range(8), 16, 3, 0, 4)
    counts = []
    for maxiters in (2, 3, 4):
        c0 = cvxopt_b200.launch_count()
        out = qcqp_solve(d, nsub=1, maxiters=maxiters)
        counts.append((cvxopt_b200.launch_count() - c0, out["line_search_rounds"]))
    d1 = counts[1][0] - counts[0][0] - QC_PER_ROUND * (counts[1][1] - counts[0][1])
    d2 = counts[2][0] - counts[1][0] - QC_PER_ROUND * (counts[2][1] - counts[1][1])
    print("QC launches (total, rounds) at maxiters 2, 3, 4:", counts, "per iteration:", d1, d2)
    assert d1 == d2
    if QC_PER_ITER is not None:
        assert d1 == QC_PER_ITER
    e = cp_batch_data("qcqp", range(8), 16, 0, 4)
    F = torch_F("qcqp", e["data"], e["x0"])
    counts, rounds = [], []
    for maxiters in (2, 3, 4):
        c0 = cvxopt_b200.launch_count()
        out = cvxopt_b200.cp_batch(F, e["G"], e["h"], nsub=1, maxiters=maxiters)
        counts.append(cvxopt_b200.launch_count() - c0)
        rounds.append(out["line_search_rounds"])
    print("CP launches at maxiters 2, 3, 4:", counts, "rounds:", rounds)
    assert counts[1] - counts[0] == counts[2] - counts[1]
    assert rounds[1] - rounds[0] == rounds[2] - rounds[1] == CP_ROUNDS_PER_ITER
    if CP_PER_ITER is not None:
        assert counts[1] - counts[0] == CP_PER_ITER


def _kernels(fn):
    """the names of the CUDA kernels that run during fn(), from torch.profiler"""
    import torch
    from torch.profiler import ProfilerActivity
    with torch.profiler.profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    from torch.autograd import DeviceType
    return {e.name for e in prof.events()
            if e.device_type == DeviceType.CUDA and not any(w in e.name for w in ("Memcpy", "Memset"))}


def _library_kernel(name):
    """every kernel of libcvxopt_b200 lives in namespace cvxb or in a file's anonymous namespace"""
    name = name[5:] if name.startswith("void ") else name
    return name.startswith(("cvxb::", "(anonymous namespace)::")) or "_ZN4cvxb" in name or "_GLOBAL__N_" in name


def test_F_is_never_called_back():
    """cp_problems' qcqp family: through cp_batch the profile holds F's torch kernels next to the library's; through
    qcqp_batch every kernel that runs is the library's, and the QC kernels are among them"""
    import cvxopt_b200
    from cp_problems import cp_batch_data, torch_F
    d = cp_batch_data("qcqp", range(8), 16, 0, 4)
    D = d["data"]
    F = torch_F("qcqp", D, d["x0"])
    cp = _kernels(lambda: cvxopt_b200.cp_batch(F, d["G"], d["h"], maxiters=3))
    qc = _kernels(lambda: cvxopt_b200.qcqp_batch(D["P"], D["q"], D["r"], d["G"], d["h"], maxiters=3))
    assert [k for k in cp if not _library_kernel(k)], sorted(cp)
    assert not [k for k in qc if not _library_kernel(k)], sorted(k for k in qc if not _library_kernel(k))
    assert any("k_qc_eval" in k for k in qc) and any("k_qc_hessian" in k for k in qc), sorted(qc)
