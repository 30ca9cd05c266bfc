"""Seeded convex QCQPs for the QCQP batch tests and tools/batch_qcqp_bench.py: numpy Generator(PCG64(seed)) only.

    f_i(x) = x'P_i x / 2 + q_i'x + r_i (i = 0..mnl),  minimize f_0 s.t. f_i <= 0, G x <= h, A x = b

Each P_i is stored with its lower triangle significant and noise above the diagonal, which the batch must not read;
`ref_F` is the reference's F for solvers.cp, built from the same lower triangles mirrored.
"""
import numpy as np

KINDS = ("quad", "linear", "deficient")


def qcqp_problem(seed, n, mnl, p=0, r=0, kind="quad"):
    """one problem drawn from PCG64(seed): a point xh ~ U(-0.5, 0.5) strictly feasible for every constraint;
    P_i = M M'/n + 0.1 I (i >= 1), q_i ~ N(0, 1), r_i = -(f_i(xh) without r_i) - U(0.5, 1.5); G = [I; -I; N(0, 1)
    (r rows)], h = [2 (2n entries); G_r xh + U(0.5, 1.5)]; A ~ N(0, 1) (p x n), b = A xh; x0 = 0.  The objective:
      quad:      P_0 = M M'/n + 0.1 I, q_0 ~ N(0, 1), r_0 = 0;
      linear:    P_0 = 0 (a linear objective over the box);
      deficient: P_0 = [M M'/(n - p) + 0.1 I, 0; 0, 0] with M (n - p) x (n - p): its last p rows and columns are
                 exactly zero, mnl and r are ignored (0) and there are no G rows.  S = P_0 at iteration 0 then has an
                 exactly zero pivot, so every Cholesky fails on it and the factorisation switches to S + A'A (p > 0);
                 [P_0; A] has full rank when A's last p columns do."""
    rng = np.random.Generator(np.random.PCG64(seed))
    if kind == "deficient":
        mnl, r = 0, 0
    nK = mnl + 1
    xh = rng.uniform(-0.5, 0.5, n)
    P, q, rr = np.zeros((nK, n, n)), rng.standard_normal((nK, n)), np.zeros(nK)
    for i in range(nK):
        if i == 0 and kind == "linear":
            continue
        if i == 0 and kind == "deficient":                        # p exactly zero rows and columns
            M = rng.standard_normal((n - p, n - p))
            P[i, :n - p, :n - p] = M @ M.T / (n - p) + 0.1 * np.eye(n - p)
            continue
        M = rng.standard_normal((n, n))
        P[i] = M @ M.T / n + 0.1 * np.eye(n)
    for i in range(1, nK):
        rr[i] = -(0.5 * xh @ P[i] @ xh + q[i] @ xh) - rng.uniform(0.5, 1.5)
    if kind == "deficient":
        G, h = np.zeros((0, n)), np.zeros(0)
    else:
        Gr = rng.standard_normal((r, n))
        G = np.vstack([np.eye(n), -np.eye(n), Gr])
        h = np.concatenate([np.full(2 * n, 2.0), Gr @ xh + rng.uniform(0.5, 1.5, r)])
    A = rng.standard_normal((p, n))
    b = A @ xh
    noise = np.triu(rng.standard_normal((nK, n, n)), 1)          # above the diagonal: never read
    return {"P": np.tril(P) + noise, "q": q, "r": rr, "x0": np.zeros(n), "G": G, "h": h, "A": A, "b": b}


def qcqp_batch_data(seeds, n, mnl, p=0, r=0, kind="quad"):
    """qcqp_problem over the seeds, stacked along a leading batch axis"""
    probs = [qcqp_problem(s, n, mnl, p, r, kind) for s in seeds]
    return {k: np.stack([d[k] for d in probs]) for k in probs[0]}


def sym(P):
    """the symmetric matrices whose lower triangles P's are"""
    L = np.tril(P)
    return L + np.swapaxes(np.tril(P, -1), -1, -2)


def ref_F(d, k):
    """solvers.cp's F for problem k of qcqp_batch_data's d"""
    from cvxopt import matrix
    P, q, r, x0 = sym(d["P"][k]), d["q"][k], d["r"][k], d["x0"][k]
    mnl = P.shape[0] - 1

    def F(x=None, z=None):
        if x is None:
            return mnl, matrix(np.asarray(x0, dtype=np.float64))
        x = np.array(x).ravel()
        Px = P @ x
        f = 0.5 * Px @ x + q @ x + r
        Df = Px + q
        if z is None:
            return matrix(f), matrix(Df)
        return matrix(f), matrix(Df), matrix(np.tensordot(np.array(z).ravel(), P, 1))
    return F
