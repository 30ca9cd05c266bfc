"""Batched cpl problems with semidefinite cones (sdp_cpl_batch, cvxb_batch_create_sdp_cpl) against a Python loop over
the reference's solvers.cpl (oracle/_ref), problem by problem, on tests/sdcpl_problems.py's families: converged
solutions and iteration counts, iterates after 1-3 iterations at refinement 0-2, the backtracking into dom f, the
relaxed line search with 's' blocks, cp's epigraph through the batch, the cpl batch's path without 's' blocks,
compaction, device memory and launches.  Iterations are counted as test_batch_cpl_gpu.py counts them."""
import numpy as np
import pytest

from cpl_problems import MNL, cpl_batch_data, torch_F
from sdcpl_problems import lmi_rows, sdcpl_batch_data
from test_batch_cpl_gpu import _m, _rel, _relaxed_trace, _same, cpl_solve, ref_cpl_loop

pytestmark = pytest.mark.gpu

TOL = 1e-10                      # the SDP suites' bar for iterates
KEYS = ("x", "snl", "sl", "znl", "zl", "y")
ALSO = ("iterations", "primal objective", "dual objective", "status")


def sdcpl_solve(family, d, seen=None, F=None, **kw):
    import cvxopt_b200
    F = F or torch_F(family, d["data"], d["x0"], 0, seen)
    p = d["A"].shape[1]
    return cvxopt_b200.sdp_cpl_batch(d["c"], F, d["G"] if d["G"].shape[1] else None,
                                     d["h"] if d["G"].shape[1] else None, d["dims"], d["A"] if p else None,
                                     d["b"] if p else None, **kw)


def assert_matches(out, refs, xy_tol, sz_tol, obj_tol):
    """status and iterations equal; x and y within xy_tol relative, s and z (symmetric 's' blocks in both) within
    sz_tol, objectives within obj_tol; -> largest error"""
    worst = 0.0
    for k, r in enumerate(refs):
        assert out["status"][k] == r["status"], (k, out["status"][k], r["status"])
        assert out["iterations"][k] == r["iterations"], (k, out["iterations"][k], r["iterations"])
        for key, tol in (("x", xy_tol), ("y", xy_tol), ("snl", sz_tol), ("sl", sz_tol), ("znl", sz_tol),
                         ("zl", sz_tol)):
            e = _rel(out[key][k], np.array(r[key]))
            worst = max(worst, e)
            assert e <= tol, (k, key, e)
        for key in ("primal objective", "dual objective"):
            e = abs(out[key][k] - r[key]) / max(1.0, abs(r[key]))
            worst = max(worst, e)
            assert e <= obj_tol, (k, key, e)
    return worst


def _symmetric_blocks(v, ml, s):
    o = ml
    for k in (k for k in s if k):
        blk = v[:, o:o + k * k].reshape(-1, k, k)
        assert np.array_equal(blk, blk.transpose(0, 2, 1))
        o += k * k


SHAPES = [  # family, n, q, s, ml, p, B, first seed
    ("socp", 12, [3], [4, 7], 3, 0, 16, 100),        # 'l' + 'q' + 's', mnl = 2
    ("socp", 10, [], [32], 2, 2, 257, 100),          # the largest order, with A; sub-batches, compaction
    ("logcone", 16, [3], [2], 0, 0, 20, 0),          # restricted domain: both backtrack into it
    ("conelp", 8, [3], [1, 0, 6], 2, 0, 12, 100),    # mnl = 0, an order-0 block
    ("socp", 14, [5], [8], 2, 1, 1, 100),            # B = 1
]


@pytest.mark.parametrize("family,n,q,s,ml,p,B,seed", SHAPES)
def test_converged_parity(ref, family, n, q, s, ml, p, B, seed):
    d = sdcpl_batch_data(family, range(seed, seed + B), n, q, s, ml, p)
    calls, seen = {}, {}
    refs = ref_cpl_loop(ref, family, d, calls)
    out = sdcpl_solve(family, d, seen)
    worst = assert_matches(out, refs, 1e-6, 1e-5, 1e-8)
    assert all(st == "optimal" for st in out["status"])
    assert out["snl"].shape == (B, MNL[family]) and out["sl"].shape == (B, d["G"].shape[1])
    cd = d["dims"]["l"] + sum(d["dims"]["q"])
    _symmetric_blocks(out["sl"], cd, s)
    _symmetric_blocks(out["zl"], cd, s)
    if family == "logcone":
        assert calls.get("none", 0) > 0 and seen.get("nonfinite", 0) > 0, (calls, seen)
    print("%s s=%s B=%d: largest relative error %.2e, reference None returns %d, rounds %d"
          % (family, s, B, worst, calls.get("none", 0), out["line_search_rounds"]))


@pytest.mark.parametrize("refinement", [0, 1, 2])
@pytest.mark.parametrize("maxiters", [1, 2, 3])
@pytest.mark.parametrize("family,n,q,s,ml,p", [("socp", 12, [3], [3, 5], 2, 2), ("logcone", 10, [4], [4], 0, 2),
                                               ("conelp", 8, [], [6], 3, 0)])
def test_iterates(ref, family, n, q, s, ml, p, maxiters, refinement):
    d = sdcpl_batch_data(family, range(8), n, q, s, ml, p)
    refs = ref_cpl_loop(ref, family, d, maxiters=maxiters, refinement=refinement)
    out = sdcpl_solve(family, d, maxiters=maxiters, refinement=refinement)
    worst = assert_matches(out, refs, TOL, TOL, TOL)
    print("iterates %s s=%s maxiters=%d refinement=%d: largest relative error %.2e"
          % (family, s, maxiters, refinement, worst))


def test_relaxed_line_search_with_s_blocks(ref):
    """lsecone (a GP in cpl's epigraph form) with a 'q' cone of length 3 and an 's' block of order 3, 40 seeds: many
    problems enter a relaxed line search, which saves W with its r and rti (r0, rti0 in the state row), and seed 23
    runs 8 relaxed iterations without sufficient decrease and resumes the saved search, which restores them (and the
    eigenvectors in ds, dz with the current direction's sigs, sigz, as the reference does).  Status, iteration counts
    and solutions are the reference's, problem by problem"""
    d = sdcpl_batch_data("lsecone", range(40), 9, [3], [3], 0, 0)
    trace = _relaxed_trace(ref, "lsecone", d)
    entered = [k for k, t in enumerate(trace) if t[0]]
    resumed = [k for k, t in enumerate(trace) if t[1]]
    assert resumed == [23] and len(entered) == 19, (resumed, entered)
    refs = ref_cpl_loop(ref, "lsecone", d)
    out = sdcpl_solve("lsecone", d)
    assert_matches(out, refs, 1e-6, 1e-5, 1e-8)
    print("lsecone s=[3] sweep: relaxed searches entered by %d problems, resumed by %s (iterations %s); all "
          "iterations %s" % (len(entered), resumed, [int(out["iterations"][k]) for k in resumed],
                             [int(k) for k in out["iterations"]]))


def test_epigraph_cp_with_an_lmi(ref):
    """min |x - a|² s.t. G x <= h and an LMI, as sdp_cpl_batch's epigraph (variable (x, t), minimise t, |x - a|² - t
    <= 0) against the reference's solvers.cp(F, G, h, dims) on the same problem; cp eliminates t with its own
    kktsolver, so the iteration counts are not compared"""
    import torch
    import cvxopt_b200
    from cvxopt import matrix, solvers
    B, n, ml, s = 12, 6, 4, [5]
    rng = np.random.Generator(np.random.PCG64(7))
    a = rng.standard_normal((B, n)) * 2.0
    Gl = rng.standard_normal((B, ml, n))
    hl = rng.uniform(0.5, 1.5, (B, ml))                  # x = 0 strictly feasible
    Gs, hs = zip(*[lmi_rows(k, n, s, "socp") for k in range(B)])
    G, h = np.concatenate([Gl, np.stack(Gs)], 1), np.concatenate([hl, np.stack(hs)], 1)
    dims = {"l": ml, "q": [], "s": s}
    x0 = np.zeros((B, n + 1))                           # cp's start: (x0, t = 0), cvxprog.py:1768
    at = torch.as_tensor(a, device="cuda")

    def F(x=None, z=None, idx=None):
        if x is None:
            return 1, x0
        r = x[:, :n] - at[idx]
        f = ((r * r).sum(1) - x[:, n])[:, None]
        Df = torch.cat([2.0 * r, -torch.ones_like(x[:, :1])], 1)[:, None, :]
        if z is None:
            return f, Df
        H = torch.zeros((x.shape[0], n + 1, n + 1), dtype=x.dtype, device=x.device)
        H[:, :n, :n] = 2.0 * z[:, 0, None, None] * torch.eye(n, dtype=x.dtype, device=x.device)
        return f, Df, H
    c = np.zeros((B, n + 1))
    c[:, n] = 1.0
    Ge = np.concatenate([G, np.zeros((B, G.shape[1], 1))], 2)
    out = cvxopt_b200.sdp_cpl_batch(c, F, Ge, h, dims)
    worst = 0.0
    for k in range(B):
        def Fk(x=None, z=None, k=k):
            if x is None:
                return 0, matrix(0.0, (n, 1))
            r = np.array(x).ravel() - a[k]
            f, Df = matrix([float(r @ r)]), matrix(2.0 * r[None, :])
            return (f, Df) if z is None else (f, Df, matrix(2.0 * z[0] * np.eye(n)))
        rr = solvers.cp(Fk, _m(G[k]), _m(h[k]), dims, options=dict(show_progress=False))
        assert rr["status"] == "optimal" and out["status"][k] == "optimal"
        e = _rel(out["x"][k, :n], np.array(rr["x"]))
        o = abs(out["primal objective"][k] - rr["primal objective"]) / max(1.0, abs(rr["primal objective"]))
        worst = max(worst, e, o)
        assert e <= 1e-6 and o <= 1e-7, (k, e, o)
    print("epigraph cp with an LMI: largest relative error %.2e" % worst)


@pytest.mark.parametrize("s", [[], [0, 0]])
def test_no_s_blocks_is_the_cpl_batch(s):
    """dims without an 's' block of positive order run cpl_batch's path: the same bits and the same launches"""
    import cvxopt_b200
    d = cpl_batch_data("socp", range(16), 12, [3, 5], 2, 2)
    F = torch_F("socp", d["data"], d["x0"])
    c0 = cvxopt_b200.launch_count()
    base = cpl_solve("socp", d, F=F, nsub=1)
    c1 = cvxopt_b200.launch_count()
    e = dict(d, dims=dict(d["dims"], s=s))
    out = sdcpl_solve("socp", e, F=F, nsub=1)
    c2 = cvxopt_b200.launch_count()
    _same(out, base)
    assert c2 - c1 == c1 - c0


def test_compaction_resolves_and_nsub(monkeypatch):
    """the same bits with compaction on and off, across re-solves of one batch and under nsub.  A lone active slot
    takes the single-matrix SYRK (test_batch_cpl_gpu.py): with compaction, the last problem to finish, when it is the
    only one left, and every problem of nsub > 1 are compared to 1e-12"""
    import cvxopt_b200
    d = sdcpl_batch_data("logcone", range(24), 12, [4], [3, 5], 0, 2)
    F = torch_F("logcone", d["data"], d["x0"])
    base = sdcpl_solve("logcone", d, F=F, nsub=1)
    monkeypatch.setenv("CVXB_BATCH_COMPACT", "0")
    off = sdcpl_solve("logcone", d, F=F, nsub=1)
    monkeypatch.delenv("CVXB_BATCH_COMPACT")
    it = np.asarray(base["iterations"])
    lone = np.flatnonzero(it == it.max()) if (it == it.max()).sum() == 1 else []
    rest = np.setdiff1d(np.arange(24), lone)
    _same({k: np.asarray(v)[rest] for k, v in off.items() if k in KEYS + ALSO},
          {k: np.asarray(v)[rest] for k, v in base.items() if k in KEYS + ALSO})
    for k in lone:
        assert off["status"][k] == base["status"][k] and off["iterations"][k] == base["iterations"][k]
        assert np.allclose(off["x"][k], base["x"][k], rtol=1e-12, atol=1e-12)
    bt = cvxopt_b200.SDPCPLBatch(24, 12, 1, d["dims"], 2)
    try:
        bt.set_F(F)
        bt.load(d["c"], d["x0"], d["G"], d["h"], d["A"], d["b"])
        for _ in range(2):
            bt.solve()
            r = bt.results()
            assert np.array_equal(r["x"], base["x"]) and np.array_equal(r["iterations"], base["iterations"])
            assert np.array_equal(r["z"][:, 1:], base["zl"])
    finally:
        bt.close()
    three = sdcpl_solve("logcone", d, F=F, nsub=3)
    assert three["nsub"] == 3
    assert list(three["status"]) == list(base["status"]) and np.array_equal(three["iterations"], base["iterations"])
    assert np.allclose(three["x"], base["x"], rtol=1e-12, atol=1e-12)


def _ev(x):
    return (x + 1) & ~1


@pytest.mark.parametrize("q,s", [([3, 6], [4, 0, 3]), ([], [5])])
def test_device_memory(q, s):
    """what the header states: the cpl batch of the same n, mnl, p with dims {'l': ml + sum s², 'q': q}, plus Gs
    without 'q' cones, v and the saved v over the 's' rows with them, r, rti, sigs, sigz, r0, rti0, the partial sums,
    the row weights and the layout ints"""
    from cvxopt_b200 import CPLBatch, SDPCPLBatch, _lib
    lib = _lib.load()
    B, n, mnl, p, ml = 5, 9, 2, 3, 4
    pos = [k for k in s if k]
    S1, S2, ns = sum(pos), sum(k * k for k in pos), len(pos)
    m = mnl + ml + sum(q) + S2
    before = lib.cvxb_device_bytes()
    bt = SDPCPLBatch(B, n, mnl, {"l": ml, "q": q, "s": s}, p)
    sd = lib.cvxb_device_bytes() - before
    bt.close()
    assert lib.cvxb_device_bytes() == before
    bt = CPLBatch(B, n, mnl, {"l": ml + S2, "q": q, "s": []}, p)
    cpl = lib.cvxb_device_bytes() - before
    bt.close()
    ldg = max(2, (m + 1) & ~1)
    state = 2 * _ev(S2) + 2 * _ev(S1) + 2 * _ev(S2)
    if q:
        state += 2 * (_ev(sum(q) + S2) - _ev(sum(q)))
    extra = 8 * B * (state + 4 * ns + (0 if q else ldg * n)) + 8 * m + 4 * (5 * ns + S2)
    assert sd - cpl == extra, (sd - cpl, extra)
    assert lib.cvxb_device_bytes() == before


# launches of one lock-step iteration of the 8-problem batch below with compaction off, and of the same batch without
# its 's' rows (CPL_PER_ITER_NO_S): the difference is, per direction, k_s_wtz, k_s_steps, k_s_dir_post and
# k_s_sort, plus k_s_res and k_s_wtz per refinement step (refinement 1: 6), and per iteration k_s_update and, without
# 'q' cones, k_build_gs and k_s_build_gs (the batch without cones does not form Gs): 2 * 6 + 1 + 2 = 15
SDCPL_PER_ITER, CPL_PER_ITER_NO_S = 116, 101


def test_launches_per_iteration(monkeypatch):
    """launches per lock-step iteration (maxiters 2 -> 3 -> 4 on a batch whose problems all run past 4 iterations),
    pinned, with and without the 's' block"""
    import cvxopt_b200
    monkeypatch.setenv("CVXB_BATCH_COMPACT", "0")
    d = sdcpl_batch_data("socp", range(8), 12, [], [6], 2, 2)
    e = cpl_batch_data("socp", range(8), 12, [], 2, 2)
    F = torch_F("socp", d["data"], d["x0"])
    per = {}
    for name, data, solve in (("s", d, sdcpl_solve), ("no s", e, cpl_solve)):
        counts, rounds = [], []
        for maxiters in (2, 3, 4):
            c0 = cvxopt_b200.launch_count()
            out = solve("socp", data, F=F, nsub=1, maxiters=maxiters)
            counts.append(cvxopt_b200.launch_count() - c0)
            rounds.append(out["line_search_rounds"])
        print("%s: launches at maxiters 2, 3, 4: %s, line-search rounds %s" % (name, counts, rounds))
        assert counts[1] - counts[0] == counts[2] - counts[1]
        assert rounds[1] - rounds[0] == rounds[2] - rounds[1] == 4
        per[name] = counts[1] - counts[0]
    assert (per["s"], per["no s"]) == (SDCPL_PER_ITER, CPL_PER_ITER_NO_S), per
    assert SDCPL_PER_ITER - CPL_PER_ITER_NO_S == 15
