"""Sparse G against dense G in the single-problem KKT factory (kkt_chol), alternating the two factories on the same
seeded 'l'-only G and fresh scalings W, in one process:
  s4k      n = 4096, m = 65536, 8 entries per row
  s8k      n = 8192, m = 131072, 16 entries per row
  dense4k  n = 4096, m = 65536, 512 entries per row: above the density where the factory takes the dense SYRK
and a sweep at n = 4096, m = 65536 over the entries per row (--sweep) that puts the sparse SYRK's time next to the
dense one's, to place the crossover ratio R = m n^2 / sum_k nnz(row k)^2.
Per factory: factor ms and solve ms (CUDA events), the factor split by the existing breakdown events into the SYRK
(the sparse kernel alone on the sparse factory, the DMMA SYRK on the dense one), potrf and the scaling; the path the
factory took; the sparse kernel's useful bytes (K's lower triangle written once, both CSR copies read once) over its
time against the 3.35 TB/s HBM3 data-sheet bound; the largest relative difference between the two factories'
directions; the card name and power limit read in the same run.  One JSON line per shape."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12
SHAPES = {"s4k": (4096, 65536, 8), "s8k": (8192, 131072, 16), "dense4k": (4096, 65536, 512)}


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                       # noqa: BLE001
        return "unknown (%s)" % e


def make_G(n, m, per, seed):
    """m x n CSR, `per` distinct random columns per row, normal values"""
    import scipy.sparse as sps
    rng = np.random.Generator(np.random.PCG64(seed))
    cols = np.empty((m, per), dtype=np.int64)
    for r0 in range(0, m, 8192):                 # distinct columns per row: argpartition of random keys
        r1 = min(m, r0 + 8192)
        cols[r0:r1] = np.argpartition(rng.random((r1 - r0, n)), per - 1, axis=1)[:, :per]
    rows = np.repeat(np.arange(m), per)
    return sps.csr_matrix((rng.standard_normal(m * per), (rows, cols.ravel())), shape=(m, n))


def useful_bytes(G):
    """K's lower triangle written once; CSR (rowptr, colind, val) and the transposed copy (colptr, rowind, val,
    position) read once; the weights once"""
    m, n = G.shape
    return 8 * n * (n + 1) / 2 + G.nnz * (12 + 20) + 8 * (m + 1) + 8 * (n + 1) + 8 * m


def run_shape(name, n, m, per, reps):
    import cvxopt_b200
    G = make_G(n, m, per, seed=n + per)
    s = np.diff(G.indptr).astype(np.float64)
    work = float(np.sum(s * s))
    dims = {"l": m, "q": [], "s": []}
    fs = cvxopt_b200.kkt_chol(G, dims)
    Gd = G.T.toarray().T                         # Fortran order without a second copy
    fd = cvxopt_b200.kkt_chol(Gd, dims)
    del Gd
    rng = np.random.Generator(np.random.PCG64(7))
    rows = {"sparse": [], "dense": []}
    maxdiff = 0.0
    for rep in range(reps + 1):
        d = rng.uniform(0.5, 2.0, m)
        W = {"d": d, "di": 1.0 / d, "v": [], "beta": [], "r": [], "rti": []}
        x0, z0 = rng.standard_normal(n), rng.standard_normal(m)
        out = {}
        for key, f in (("sparse", fs), ("dense", fd)) if rep % 2 == 0 else (("dense", fd), ("sparse", fs)):
            x, z = x0.copy(), z0.copy()
            f(W)(x, None, z)
            fms, sms = f.last_ms()
            br = f.last_breakdown()
            out[key] = (x, z)
            if rep:                               # rep 0 is the warm-up
                rows[key].append(dict(factor_ms=fms, solve_ms=sms, syrk_ms=br["syrk_ms"], potrf_ms=br["potrf_ms"],
                                      scale_ms=br["scale_ms"]))
        for a, b in zip(out["sparse"], out["dense"]):
            maxdiff = max(maxdiff, float(np.linalg.norm(a - b) / np.linalg.norm(b)))
    med = lambda key, f: float(np.median([r[f] for r in rows[key]]))     # noqa: E731
    res = dict(shape=name, n=n, m=m, nnz=int(G.nnz), nnz_per_row=per, sparse_work=work,
               ratio_mn2_over_work=m * float(n) * n / work, path=fs.syrk_path(), dense_path=fd.syrk_path(),
               reps=reps, max_rel_diff=maxdiff)
    for key in ("sparse", "dense"):
        for f in ("factor_ms", "solve_ms", "syrk_ms", "potrf_ms", "scale_ms"):
            res["%s_%s" % (key, f)] = med(key, f)
    if fs.syrk_path() == "sparse":
        t = res["sparse_syrk_ms"] * 1e-3
        res["sparse_kernel_bytes"] = useful_bytes(G)
        res["sparse_kernel_GBps"] = useful_bytes(G) / t / 1e9
        res["sparse_kernel_frac_of_3.35TBps"] = useful_bytes(G) / t / HBM_BYTES_PER_S
        res["sparse_updates_per_s"] = float(np.sum(s * (s + 1) / 2)) / t
    fs.close()
    fd.close()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--shapes", default="s4k,s8k,dense4k")
    ap.add_argument("--sweep", default="32,64,128,160",
                    help="entries per row at n = 4096, m = 65536 for the crossover sweep ('' for none)")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    gpu = card()
    todo = [(s, *SHAPES[s]) for s in args.shapes.split(",") if s]
    todo += [("sweep%d" % int(p), 4096, 65536, int(p)) for p in args.sweep.split(",") if p]
    for name, n, m, per in todo:
        res = run_shape(name, n, m, per, args.reps)
        res["card"] = gpu
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
