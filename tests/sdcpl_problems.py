"""Seeded cpl problems with semidefinite cones for the sdp_cpl_batch tests and tools/batch_cpl_bench.py: each of
tests/cpl_problems.py's families with LMI rows appended after its 'l' and 'q' rows, numpy Generator(PCG64) only.

Block k of order sk is sum_j x_j A_jk <= S0_k + sum_j xf_j A_jk (the Loewner order), with A_jk = (M + M')/(2 sqrt(n))
symmetric, M ~ N(0, 1), S0_k = N N'/sk + I with N ~ N(0, 1), and xf the family's strictly feasible point (0, or 1 for
logcone), so xf stays strictly feasible and boundedness is the family's.  In G x + s = h the block's rows are
G[:, j] = vec(A_jk) and h = vec(S0_k + sum_j xf_j A_jk), unpacked column-major as the reference's G.  lsecone's LMI
leaves its epigraph variable t out (A_tk = 0).  The rows are linear, so F is the family's: cpl_problems.ref_F and
cpl_problems.torch_F serve unchanged.
"""
import numpy as np

from cpl_problems import cpl_batch_data


def lmi_rows(seed, n, s, family):
    """the 's' rows of G and h of one problem: (sum s² x n, sum s²), drawn from PCG64([seed, 1]) block by block"""
    rng = np.random.Generator(np.random.PCG64([seed, 1]))
    nx = n - 1 if family == "lsecone" else n
    xf = np.ones(nx) if family == "logcone" else np.zeros(nx)
    G, h = [np.zeros((0, n))], [np.zeros(0)]
    for k in s:
        if k == 0:
            continue
        M = rng.standard_normal((nx, k, k))
        A = (M + M.transpose(0, 2, 1)) / (2.0 * np.sqrt(n))
        N = rng.standard_normal((k, k))
        S0 = N @ N.T / k + np.eye(k)
        Gk = np.zeros((k * k, n))
        Gk[:, :nx] = A.transpose(0, 2, 1).reshape(nx, k * k).T          # column j = vec(A_j), column-major
        G.append(Gk)
        h.append((S0 + np.tensordot(xf, A, 1)).T.reshape(-1))
    return np.vstack(G), np.concatenate(h)


def sdcpl_batch_data(family, seeds, n, q, s, ml=0, p=0):
    """cpl_batch_data(family, seeds, n, q, ml, p) with the LMI rows of blocks of orders s appended to G and h;
    dims['s'] = s"""
    seeds = list(seeds)
    d = cpl_batch_data(family, seeds, n, q, ml, p)
    rows = [lmi_rows(seed, n, s, family) for seed in seeds]
    d["G"] = np.concatenate([d["G"], np.stack([r[0] for r in rows])], axis=1)
    d["h"] = np.concatenate([d["h"], np.stack([r[1] for r in rows])], axis=1)
    d["dims"] = dict(d["dims"], s=list(s))
    return d
