"""Batch iterates before convergence: cvxopt_b200.qp_batch(..., maxiters=k) against solvers.coneqp(...,
kktsolver='chol', options={'maxiters': k}) (oracle/_ref) problem by problem, for k = 1..3 (coneqp refuses
maxiters = 0, coneprog.py:1785).

Both stop at the same point of the iteration (coneqp returns its current iterate when iters == MAXITERS,
coneprog.py:2212-2234), so status 'unknown', the iteration count and x, s, z must agree.  A converged solve hides
an inexact Newton direction or one wrong tile of one problem of a batch; an early iterate does not: every one of
the k directions computed so far went through the factorisation and the solves.  B = 1 runs the single
graph-replayed potrf_lower, B = 3 the batched Cholesky, GEMM, triangular solve and GEMV kernels; n spans one to
three 128-wide diagonal blocks with partial last blocks."""
import numpy as np
import pytest

from problems import dense_qp
from test_batch_cones_gpu import _full, cone_qp

pytestmark = pytest.mark.gpu

TOL = 1e-10          # relative 2-norm difference of x, s and z per problem


def _rel(a, b):
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


def _compare(P, q, G, h, dims, batch_dims):
    import cvxopt_b200
    from cvxopt import matrix, solvers
    worst = {}
    for k in (1, 2, 3):
        got = cvxopt_b200.qp_batch(P, q, G, h, dims=batch_dims, maxiters=k)
        dk = 0.0
        for p in range(P.shape[0]):
            want = solvers.coneqp(matrix(P[p]), matrix(q[p]), matrix(G[p]), matrix(h[p]), dims, kktsolver="chol",
                                  options={"maxiters": k, "show_progress": False})
            assert want["status"] == "unknown" and want["iterations"] == k, (p, k, want["status"])
            assert got["status_code"][p] == 2 and got["status"][p] == "unknown", (p, k, got["status_code"][p])
            assert got["iterations"][p] == k, (p, k, got["iterations"][p])
            for key in ("x", "s", "z"):
                d = _rel(got[key][p], np.array(want[key]).ravel())
                assert d <= TOL, (p, k, key, d)
                dk = max(dk, d)
        worst[k] = dk
    return worst


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("n", [127, 128, 129, 257])
def test_l_batch_iterates_match_coneqp(ref, n, B):
    m = 2 * n
    parts = [dense_qp(n, m, seed=1000 * n + 10 * B + p) for p in range(B)]
    P, q, G, h = (np.stack([x[i] for x in parts]) for i in range(4))
    worst = _compare(P, q, G, h, {"l": m, "q": [], "s": []}, None)
    print("\nbatch iterates 'l' n=%d B=%d: largest relative difference per k %s"
          % (n, B, ", ".join("%d: %.2e" % kv for kv in worst.items())))


def test_cone_batch_iterates_match_coneqp(ref):
    dims = {"l": 20, "q": [5, 1, 140]}
    n, B = 129, 3
    parts = [cone_qp(n, dims, 2000 + p) for p in range(B)]
    P, q, G, h = (np.stack([x[i] for x in parts]) for i in range(4))
    worst = _compare(P, q, G, h, _full(dims), dims)
    print("\nbatch iterates cones n=%d B=%d: largest relative difference per k %s"
          % (n, B, ", ".join("%d: %.2e" % kv for kv in worst.items())))


def test_batch_singular_start_names_the_problem():
    """problem 2 of a B = 4 batch has Rank([P; G]) < n: the batched Cholesky's per-problem info names it"""
    import cvxopt_b200
    n, m = 20, 40
    parts = [dense_qp(n, m, seed=3000 + p) for p in range(4)]
    P, q, G, h = (np.stack([x[i] for x in parts]) for i in range(4))
    P[2] = 0.0
    G[2, :, 5:] = 0.0              # x[5:] appears nowhere: the 6th pivot of P + G'G is exactly 0
    with pytest.raises(ValueError, match=r"problem 2: Rank"):
        cvxopt_b200.qp_batch(P, q, G, h, nsub=1)
