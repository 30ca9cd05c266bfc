"""Equality constraints A x = b in the batch solver: qp_batch(P, q, G, h, A, b) against
solvers.coneqp(P, q, G, h, dims, A, b) (oracle/_ref, default kktsolver: 'chol2' for 'l'-only problems, 'chol' with
'q' cones) problem by problem, iterate by iterate and at convergence; the per-problem S + A'A switch; the start's
rank errors; p = 0 running exactly what a batch without A runs; compaction, sub-batches, re-solves and memory."""
import ctypes as C

import numpy as np
import pytest

from problems import cone_point
from test_batch_cones_gpu import _full

pytestmark = pytest.mark.gpu

TOL = 1e-10          # relative 2-norm difference of x, y, s and z per problem at k = 1..3 iterations


def eq_qp(n, dims, p, seed):
    """P = M'M/n + I; G, A, q, x0 ~ N(0,1); h = G x0 + s0 with s0 strictly inside the cones, b = A x0"""
    dims = _full(dims)
    rng = np.random.Generator(np.random.PCG64(seed))
    M = rng.standard_normal((n, n))
    P = M.T @ M / n + np.eye(n)
    q = rng.standard_normal(n)
    m = dims["l"] + sum(dims["q"])
    G = rng.standard_normal((m, n))
    x0 = rng.standard_normal(n)
    h = G @ x0 + cone_point(dims, rng)
    A = rng.standard_normal((p, n))
    return P, q, G, h, A, A @ x0


def eq_batch(B, n, dims, p, seed0):
    parts = [eq_qp(n, dims, p, seed0 + k) for k in range(B)]
    return [np.stack([x[i] for x in parts]) for i in range(6)]


def _rel(a, b):
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


def _coneqp(P, q, G, h, dims, A, b, **options):
    from cvxopt import matrix, solvers
    options.setdefault("show_progress", False)
    Gm = matrix(G) if G.shape[0] else matrix(0.0, (0, P.shape[0]))
    hm = matrix(h) if h.shape[0] else matrix(0.0, (0, 1))
    return solvers.coneqp(matrix(P), matrix(q), Gm, hm, _full(dims), matrix(A), matrix(b), options=options)


def _compare_iterates(batch, dims, batch_dims=None, ks=(1, 2, 3), tol=TOL, **options):
    import cvxopt_b200
    P, q, G, h, A, b = batch
    worst = 0.0
    for k in ks:
        got = cvxopt_b200.qp_batch(P, q, G, h, A, b, dims=batch_dims, maxiters=k, **options)
        for j in range(P.shape[0]):
            want = _coneqp(P[j], q[j], G[j], h[j], dims, A[j], b[j], maxiters=k, **options)
            assert want["status"] == "unknown" and want["iterations"] == k, (j, k, want["status"])
            assert got["status"][j] == "unknown" and got["iterations"][j] == k, (j, k, got["status_code"][j])
            for key in ("x", "y", "s", "z"):
                d = _rel(got[key][j], np.array(want[key]).ravel())
                assert d <= tol, (j, k, key, d)
                worst = max(worst, d)
    return worst


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("n,p", [(127, 1), (129, 1), (129, 127), (257, 1), (257, 127), (257, 129)])
def test_eq_iterates_match_coneqp(ref, n, p, B):
    """the 128-row block edges of both L (n) and Lp (p); B = 1 runs potrf_lower, B = 3 the batched kernels"""
    dims = {"l": 2 * n}
    worst = _compare_iterates(eq_batch(B, n, dims, p, 100 * n + 10 * p + B), dims)
    print("\neq iterates n=%d p=%d B=%d: largest relative difference %.2e" % (n, p, B, worst))


def test_eq_cone_iterates_match_coneqp(ref):
    dims = {"l": 20, "q": [5, 1, 140]}
    worst = _compare_iterates(eq_batch(3, 129, dims, 32, 7000), dims, batch_dims=dims)
    print("\neq iterates cones: largest relative difference %.2e" % worst)


def test_eq_l_refinement_iterates_match_coneqp(ref):
    dims = {"l": 258}
    worst = _compare_iterates(eq_batch(3, 129, dims, 32, 7100), dims, refinement=1)
    print("\neq iterates 'l' refinement=1: largest relative difference %.2e" % worst)


def _compare_converged(batch, dims, got, rtol=1e-8):
    P, q, G, h, A, b = batch
    for j in range(P.shape[0]):
        want = _coneqp(P[j], q[j], G[j], h[j], dims, A[j], b[j])
        assert want["status"] == "optimal" and got["status"][j] == "optimal", (j, got["status_code"][j])
        assert got["iterations"][j] == want["iterations"], (j, got["iterations"][j], want["iterations"])
        assert got["primal objective"][j] == pytest.approx(want["primal objective"], rel=rtol)
        for key in ("x", "y"):
            assert _rel(got[key][j], np.array(want[key]).ravel()) <= rtol, (j, key)


def test_eq_batch_converges_like_coneqp(ref):
    import cvxopt_b200
    n = 96
    dims = {"l": 2 * n}
    batch = eq_batch(16, n, dims, n // 4, 8000)
    got = cvxopt_b200.qp_batch(*batch)
    _compare_converged(batch, dims, got)


def _switch_batch():
    """problems 1 and 3: columns 48..63 of P and G are zero, so P + G'G is singular, but A's columns 48..63 are a
    random (invertible) 16 x 16 block, so [P; A; G] has full rank"""
    n, m, p = 64, 128, 16
    batch = eq_batch(4, n, {"l": m}, p, 9000)
    P, q, G, h, A, b = batch
    rng = np.random.Generator(np.random.PCG64(9100))
    for j in (1, 3):
        P[j][48:, :] = 0.0
        P[j][:, 48:] = 0.0
        G[j][:, 48:] = 0.0
        x0 = rng.standard_normal(n)
        h[j] = G[j] @ x0 + rng.uniform(0.5, 1.5, m)
        b[j] = A[j] @ x0
    return batch, {"l": m}


def test_eq_per_problem_switch_to_s_plus_ata(ref, monkeypatch):
    import cvxopt_b200
    batch, dims = _switch_batch()
    P = batch[0]
    for j in (1, 3):
        with pytest.raises(np.linalg.LinAlgError):
            np.linalg.cholesky(P[j] + batch[2][j].T @ batch[2][j])
    # S + A'A is worse conditioned than the random problems' S: x of a switched problem differed from coneqp's by
    # 1.2e-10 at k = 1 on an H100, so these iterates get 1e-9
    _compare_iterates(batch, dims, tol=1e-9)
    got = cvxopt_b200.qp_batch(*batch)
    _compare_converged(batch, dims, got)
    monkeypatch.setenv("CVXB_BATCH_COMPACT", "0")
    flat = cvxopt_b200.qp_batch(*batch)
    for key in ("x", "y", "s", "z"):
        assert np.array_equal(flat[key], got[key]), key


def test_eq_rank_errors_name_the_problem():
    """Rank(A) < p through a zero row, so Kp has an exactly zero pivot.  (With a repeated row the pivot is a rounding
    residue whose sign decides, in LAPACK's potrf as here: the reference raises for this fixture's repeated row, the
    H100's Cholesky left a tiny positive pivot.)"""
    import cvxopt_b200
    n, m, p = 20, 40, 5
    P, q, G, h, A, b = eq_batch(4, n, {"l": m}, p, 9500)
    A2, b2 = A.copy(), b.copy()
    A2[2][3] = 0.0                           # a zero row: Kp is singular
    b2[2][3] = 0.0
    with pytest.raises(ValueError, match=r"problem 2: Rank\(A\) < p"):
        cvxopt_b200.qp_batch(P, q, G, h, A2, b2, nsub=1)
    P3, G3, A3 = P.copy(), G.copy(), A.copy()
    P3[2][5, :] = P3[2][:, 5] = 0.0         # x[5] appears nowhere: P + G'G + A'A is singular
    G3[2][:, 5] = 0.0
    A3[2][:, 5] = 0.0
    with pytest.raises(ValueError, match=r"problem 2: Rank\(A\) < p"):
        cvxopt_b200.qp_batch(P3, q, G3, h, A3, b, nsub=1)


@pytest.mark.parametrize("cones", [False, True])
def test_p0_runs_what_a_batch_without_A_runs(cones):
    import cvxopt_b200
    dims = {"l": 20, "q": [5, 1, 40]} if cones else {"l": 120}
    n, B = 60, 5
    P, q, G, h, A, b = eq_batch(B, n, dims, 0, 9700)
    bd = dims if cones else None
    c0 = cvxopt_b200.launch_count()
    plain = cvxopt_b200.qp_batch(P, q, G, h, dims=bd, nsub=1)
    c1 = cvxopt_b200.launch_count()
    with0 = cvxopt_b200.qp_batch(P, q, G, h, A, b, dims=bd, nsub=1)
    c2 = cvxopt_b200.launch_count()
    assert A.shape == (B, 0, n) and with0["y"].shape == (B, 0) and plain["y"].shape == (B, 0)
    assert c2 - c1 == c1 - c0
    for key in ("x", "s", "z", "iterations", "primal objective"):
        assert np.array_equal(with0[key], plain[key]), key


def test_eq_compaction_subbatches_resolve_and_memory(ref, monkeypatch):
    import cvxopt_b200
    from cvxopt_b200 import QPBatch, _lib
    n, B, p = 80, 9, 20
    dims = {"l": 160}
    batch = eq_batch(B, n, dims, p, 9900)
    batch[1] *= np.linspace(0.1, 30.0, B)[:, None]          # spread the iteration counts: compaction swaps slots
    base = cvxopt_b200.qp_batch(*batch, nsub=1)
    assert len(set(base["iterations"].tolist())) > 1
    monkeypatch.setenv("CVXB_BATCH_COMPACT", "0")
    flat = cvxopt_b200.qp_batch(*batch, nsub=1)
    monkeypatch.delenv("CVXB_BATCH_COMPACT")
    three = cvxopt_b200.qp_batch(*batch, nsub=3)
    for key in ("x", "y", "s", "z"):
        assert np.array_equal(flat[key], base[key]), key
        assert np.abs(three[key] - base[key]).max() <= 1e-12 * (1 + np.abs(base[key]).max()), key
    assert np.array_equal(three["iterations"], base["iterations"])
    _compare_converged(batch, dims, base)
    lib = _lib.load()
    before = lib.cvxb_device_bytes()
    qb = QPBatch(B, n, 160, 0, p=p)
    assert lib.cvxb_device_bytes() > before
    P, q, G, h, A, b = batch
    qb.load(P, q, G, h, A, b)
    qb.solve()
    r1 = qb.results()
    qb.solve()
    r2 = qb.results()
    for key in ("x", "y", "s", "z", "iterations"):
        assert np.array_equal(r1[key], r2[key]), key
        assert np.array_equal(r1[key], base[key]), key
    qb.close()
    assert lib.cvxb_device_bytes() == before
    h0 = C.c_void_p()
    d, keep, _ = cvxopt_b200.batch._batch_dims({"l": 160})
    assert lib.cvxb_batch_create_eq(C.byref(h0), B, n, p, C.byref(d), 0) == 0
    Pcm, Gcm = (np.ascontiguousarray(X.transpose(0, 2, 1)) for X in (P, G))
    assert lib.cvxb_batch_load(h0, Pcm.ctypes.data, q.ctypes.data, Gcm.ctypes.data, h.ctypes.data, _lib.HOST) == 0
    assert lib.cvxb_batch_solve(h0, 100, 1e-7, 1e-6, 1e-7) == _lib.E_ARG       # A and b were never loaded
    assert "cvxb_batch_load_eq" in _lib.last_error()
    lib.cvxb_batch_destroy(h0)
    assert lib.cvxb_device_bytes() == before


def test_eq_without_inequalities_matches_coneqp(ref):
    """m = 0: coneqp's cdim == 0 branch, one KKT solve, 'optimal' after 0 iterations"""
    import cvxopt_b200
    n, p, B = 40, 10, 3
    P, q, G, h, A, b = eq_batch(B, n, {"l": 0}, p, 9950)
    got = cvxopt_b200.qp_batch(P, q, G, h, A, b)
    for j in range(B):
        want = _coneqp(P[j], q[j], G[j], h[j], {"l": 0}, A[j], b[j])
        assert want["status"] == "optimal" and want["iterations"] == 0
        assert got["status"][j] == "optimal" and got["iterations"][j] == 0
        assert got["primal objective"][j] == pytest.approx(want["primal objective"], rel=1e-12)
        assert got["dual objective"][j] == pytest.approx(want["dual objective"], rel=1e-12)
        for key in ("x", "y"):
            assert _rel(got[key][j], np.array(want[key]).ravel()) <= 1e-12, key
