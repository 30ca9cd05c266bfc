"""Batched convex programs (cp_batch, cvxb_batch_create_cp) against a Python loop over the reference's solvers.cp
(oracle/_ref), problem by problem, on tests/cp_problems.py's four families: converged solutions and iteration counts,
iterates after 1-3 iterations at refinement 0-2, the backtracking into dom f, the idx contract, the errors, and the
launches of the other batches.  The reference's cp returns no iteration count; it is counted by wrapping
misc.update_scaling, which cpl calls once per completed iteration."""
import numpy as np
import pytest

from cp_problems import MNL, cp_batch_data, ref_F, torch_F

pytestmark = pytest.mark.gpu

KEYS = ("x", "snl", "sl", "znl", "zl", "y")


def _m(v):
    from cvxopt import matrix
    return matrix(np.ascontiguousarray(v, dtype=np.float64))


def ref_cp_loop(ref, family, d, calls=None, **options):
    """solvers.cp over the batch: per problem its result dict and 'iterations'; calls['none'] counts F's None returns"""
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
            r = dict(solvers.cp(ref_F(family, d["data"], k, d["x0"][k], calls), options=dict(show_progress=False,
                                                                                             **options), **kw))
            r["iterations"] = count[0]
            out.append(r)
    finally:
        misc.update_scaling = orig
    return out


def cp_solve(family, d, seen=None, F=None, **kw):
    import cvxopt_b200
    F = F or torch_F(family, d["data"], d["x0"], 0, seen)
    ml, p = d["G"].shape[1], d["A"].shape[1]
    return cvxopt_b200.cp_batch(F, d["G"] if ml else None, d["h"] if ml else None, None, d["A"] if p else None,
                                d["b"] if p else None, **kw)


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


SHAPES = [  # family, n, p, r, B
    ("centering", 16, 4, 0, 24),        # mnl = 0 and no inequality rows
    ("entropy", 16, 3, 4, 257),         # mnl = 0; several sub-batches, compaction
    ("qcqp", 16, 0, 4, 12),
    ("logistic", 16, 0, 0, 12),
    ("qcqp", 32, 0, 8, 1),              # B = 1
    ("entropy", 48, 4, 8, 20),
]


@pytest.mark.parametrize("family,n,p,r,B", SHAPES)
def test_converged_parity(ref, family, n, p, r, B):
    d = cp_batch_data(family, range(100, 100 + B), n, p, r)
    refs = ref_cp_loop(ref, family, d)
    out = cp_solve(family, d)
    assert_matches(out, refs, 1e-6, 1e-8)
    assert all(s == "optimal" for s in out["status"])
    assert out["snl"].shape == (B, MNL[family]) and out["sl"].shape == (B, d["G"].shape[1])


@pytest.mark.parametrize("refinement", [0, 1, 2])
@pytest.mark.parametrize("maxiters", [1, 2, 3])
@pytest.mark.parametrize("family,n,p,r", [("entropy", 16, 3, 4), ("qcqp", 12, 0, 4), ("centering", 16, 4, 0)])
def test_iterates(ref, family, n, p, r, maxiters, refinement):
    d = cp_batch_data(family, range(8), n, p, r)
    refs = ref_cp_loop(ref, family, d, maxiters=maxiters, refinement=refinement)
    out = cp_solve(family, d, maxiters=maxiters, refinement=refinement)
    worst = assert_matches(out, refs, 1e-12, 1e-12)
    print("iterates %s maxiters=%d refinement=%d: largest relative error %.2e" % (family, maxiters, refinement, worst))


@pytest.mark.parametrize("family,seeds", [("entropy", range(20)), ("centering", range(20))])
def test_domain_backtracking(ref, family, seeds):
    """seeds 4, 5, 10 and 17 of entropy and 3 of centering step out of x > 0: the reference's F returns None there,
    and the batch's F sees non-finite rows in its domain rounds"""
    d = cp_batch_data(family, seeds, 16, 3 if family == "entropy" else 4, 4 if family == "entropy" else 0)
    calls, seen = {}, {}
    refs = ref_cp_loop(ref, family, d, calls)
    out = cp_solve(family, d, seen)
    assert calls.get("none", 0) > 0 and seen.get("nonfinite", 0) > 0, (calls, seen)
    assert_matches(out, refs, 1e-6, 1e-8)
    print("%s: reference None returns %d, batch evaluations with non-finite rows %d, rounds %d"
          % (family, calls["none"], seen["nonfinite"], out["line_search_rounds"]))


def _same(a, b):
    for key in KEYS + ("iterations", "primal objective", "dual objective"):
        assert np.array_equal(np.asarray(a[key]), np.asarray(b[key])), key
    assert list(a["status"]) == list(b["status"])


def test_idx_contract(ref, monkeypatch):
    """qcqp's and logistic's F read their data by idx: parity problem by problem over three sub-batches with
    compaction, and the same results with compaction off.  Compaction can leave one problem running alone, and a
    single active slot takes the factorisation's single-matrix SYRK, which sums in another order: qcqp seed 319 is that
    last problem, and its x moves by an ulp.  The logistic batch below never runs one problem alone: the same bits"""
    d = cp_batch_data("qcqp", range(300, 324), 12, 0, 4)
    refs = ref_cp_loop(ref, "qcqp", d)
    F = torch_F("qcqp", d["data"], d["x0"], rowwise=True)
    base = cp_solve("qcqp", d, F=F, nsub=3)
    assert base["nsub"] == 3
    assert_matches(base, refs, 1e-6, 1e-8)
    monkeypatch.setenv("CVXB_BATCH_COMPACT", "0")
    off = cp_solve("qcqp", d, F=F, nsub=3)
    assert list(off["status"]) == list(base["status"]) and np.array_equal(off["iterations"], base["iterations"])
    for key in KEYS + ("primal objective", "dual objective"):
        assert np.allclose(off[key], base[key], rtol=1e-15, atol=1e-15), key
    e = cp_batch_data("logistic", range(24), 8)
    F = torch_F("logistic", e["data"], e["x0"])
    off = cp_solve("logistic", e, F=F, nsub=1)
    monkeypatch.delenv("CVXB_BATCH_COMPACT")
    _same(cp_solve("logistic", e, F=F, nsub=1), off)


class _Boom(Exception):
    pass


def test_errors_and_device_memory():
    from cvxopt_b200 import _lib
    lib = _lib.load()
    before = lib.cvxb_device_bytes()
    d = cp_batch_data("entropy", range(20), 16, 3, 4)
    F = torch_F("entropy", d["data"], d["x0"])
    boom, n_full = _Boom("from F"), [0]

    def raising(x=None, z=None, idx=None):
        if z is not None:
            n_full[0] += 1
            if n_full[0] == 3:
                raise boom
        return F(x, z, idx=idx)
    with pytest.raises(_Boom) as e:
        cp_solve("entropy", d, F=raising, nsub=2)
    assert e.value is boom
    assert lib.cvxb_device_bytes() == before

    def wrong(x=None, z=None, idx=None):
        r = F(x, z, idx=idx)
        return r if x is None else (r[0][:, :1].repeat(1, 2),) + tuple(r[1:])
    with pytest.raises(TypeError, match="first output argument of F"):
        cp_solve("entropy", d, F=wrong)
    assert lib.cvxb_device_bytes() == before

    bad = dict(d, x0=d["x0"].copy())
    bad["x0"][13, 2] = -1.0
    with pytest.raises(ValueError, match="problem 13: x0 not in the domain of f"):
        cp_solve("entropy", bad, nsub=2)
    assert lib.cvxb_device_bytes() == before


def test_cp_batch_refuses_the_other_loads():
    from cvxopt_b200 import CPBatch, _lib
    lib = _lib.load()
    bt = CPBatch(2, 4, 1, 2)
    try:
        v = np.zeros(64)
        assert lib.cvxb_batch_load(bt._h, v.ctypes.data, v.ctypes.data, v.ctypes.data, v.ctypes.data,
                                   _lib.HOST) == _lib.E_ARG
        assert lib.cvxb_batch_load_lp(bt._h, v.ctypes.data, v.ctypes.data, v.ctypes.data, _lib.HOST) == _lib.E_ARG
        assert lib.cvxb_batch_load_gp(bt._h, v.ctypes.data, v.ctypes.data, v.ctypes.data, v.ctypes.data,
                                      _lib.HOST) == _lib.E_ARG
        assert lib.cvxb_batch_load_start(bt._h, None, None, None, None, _lib.HOST) == _lib.E_ARG
        bt.load(np.ones((2, 4)), np.zeros((2, 2, 4)), np.ones((2, 2)))
        assert lib.cvxb_batch_solve(bt._h, 10, 1e-7, 1e-6, 1e-7) == _lib.E_ARG      # no evaluator
        assert "cvxb_batch_set_cp_eval" in _lib.last_error()
    finally:
        bt.close()


# launches of one lock-step QP iteration (8 problems, n = 16, 'l' rows 36, refinement 0, compaction off)
QP_PER_ITER = 25


def test_other_batches_launch_what_they_did(monkeypatch):
    """the GP batch's pinned launches per iteration and per line-search round, and the QP batch's per iteration"""
    import cvxopt_b200
    import test_batch_gp_gpu
    test_batch_gp_gpu.test_launches_per_iteration(monkeypatch)
    from problems import dense_qp
    monkeypatch.setenv("CVXB_BATCH_COMPACT", "0")
    P, q, G, h = (np.stack(a) for a in zip(*(dense_qp(16, 36, seed=s) for s in range(8))))
    counts = []
    for maxiters in (2, 3, 4):
        c0 = cvxopt_b200.launch_count()
        cvxopt_b200.qp_batch(P, q, G, h, nsub=1, maxiters=maxiters)
        counts.append(cvxopt_b200.launch_count() - c0)
    d1, d2 = counts[1] - counts[0], counts[2] - counts[1]
    print("QP launches at maxiters 2, 3, 4:", counts, "per iteration:", d1, d2)
    assert d1 == d2
    if QP_PER_ITER is not None:
        assert d1 == QP_PER_ITER
