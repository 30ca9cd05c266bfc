"""Seeded geometric programs for the GP batch tests and tools/batch_gp_bench.py: numpy Generator(PCG64(seed)) only."""
import numpy as np


def gp_problem(seed, n, K, r=0, p=0):
    """A geometric program for solvers.gp(K, F, g, G, h, A, b), drawn from PCG64(seed) in this order: F ~ N(0, 1)
    (sum K x n); g0 ~ N(0, 1) and, for each block i >= 1, g_i = log(0.5 w / sum w) with w ~ U(0.1, 1), so that x = 0 is
    strictly feasible; G = [I; -I; N(0, 1) (r x n)] and h = [5 (2n entries); U(0.5, 1.5) (r)]; A = 0.1 N(0, 1) (p x n)
    and b = 0."""
    rng = np.random.Generator(np.random.PCG64(seed))
    F = rng.standard_normal((sum(K), n))
    g = [rng.standard_normal(K[0])]
    for k in K[1:]:
        w = rng.uniform(0.1, 1.0, k)
        g.append(np.log(0.5 * w / w.sum()))
    g = np.concatenate(g)
    G = np.vstack([np.eye(n), -np.eye(n), rng.standard_normal((r, n))])
    h = np.concatenate([np.full(2 * n, 5.0), rng.uniform(0.5, 1.5, r)])
    A = 0.1 * rng.standard_normal((p, n))
    return F, g, G, h, A, np.zeros(p)


def gp_batch_data(seeds, n, K, r=0, p=0):
    """gp_problem over the seeds, stacked: F (B, sum K, n), g, G (B, 2n + r, n), h, A (B, p, n), b"""
    probs = [gp_problem(s, n, K, r, p) for s in seeds]
    return tuple(np.stack([q[j] for q in probs]) for j in range(6))
