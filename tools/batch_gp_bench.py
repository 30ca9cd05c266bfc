"""Batched geometric programs (gp_batch) on B = 512 seeded feasible GPs (tests/gp_problems.py's gp_problem, seeds
0..B-1) at two shapes:
  gp64   n = 64,  K = [128] + [16]*8,  r = 16, p = 4  (ml = 2n + r = 144);
  gp256  n = 256, K = [512] + [32]*16, r = 64, p = 8  (ml = 576).
A warm-up solve of each shape precedes the timed one.  Prints one JSON line per shape: solve_ms (CUDA events around
the solve), lock-step iterations, line-search rounds, kernel launches per lock-step iteration (line-search
rounds included, summed over the concurrent sub-batches), problems/s, status counts, and the card name and power limit
read in the same run.  With --ref K it also times the reference's solvers.gp (oracle/_ref) on the first K problems of
each shape, on the host, and reports its time per problem."""
import argparse
import collections
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

SHAPES = [("gp64", 64, [128] + [16] * 8, 16, 4), ("gp256", 256, [512] + [32] * 16, 64, 8)]


def ref_ms_per_problem(K, data, count):
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    from cvxopt import matrix, solvers
    F, g, G, h, A, b = data
    m = lambda v: matrix(np.ascontiguousarray(v, dtype=np.float64))     # noqa: E731
    t0 = time.perf_counter()
    for k in range(count):
        eq = (m(A[k]), m(b[k])) if A.shape[1] else (None, None)
        solvers.gp(list(K), m(F[k]), m(g[k]), m(G[k]), m(h[k]), *eq, options=dict(show_progress=False))
    return (time.perf_counter() - t0) * 1e3 / count


def main():
    import cvxopt_b200
    from batch_coneqp_bench import card
    from gp_problems import gp_batch_data
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=512)
    ap.add_argument("--ref", type=int, default=0, help="time the reference on the first K problems of each shape")
    ap.add_argument("--shapes", default="gp64,gp256")
    a = ap.parse_args()
    if cvxopt_b200.device_count() == 0:
        raise SystemExit("batch_gp_bench: no GPU visible")
    gpu = card()
    for name, n, K, r, p in SHAPES:
        if name not in a.shapes.split(","):
            continue
        data = gp_batch_data(range(a.B), n, K, r, p)
        cvxopt_b200.gp_batch(K, *data)                                  # warm-up
        before = cvxopt_b200.launch_count()
        out = cvxopt_b200.gp_batch(K, *data)
        launches = cvxopt_b200.launch_count() - before
        it = out["lockstep_iterations"]
        row = {"shape": name, "n": n, "K": [K[0], "%dx%d" % (len(K) - 1, K[1])], "r": r, "p": p, "B": a.B,
               "card": gpu, "solve_ms": round(out["solve_ms"], 2), "lockstep_iterations": it,
               "line_search_rounds": out["line_search_rounds"],
               "launches_per_iteration": round(launches / max(1, it), 1),
               "problems_per_s": round(a.B / out["solve_ms"] * 1e3, 1),
               "status": dict(collections.Counter(out["status"])),
               "iterations_min_max": [int(np.min(out["iterations"])), int(np.max(out["iterations"]))]}
        if a.ref:
            row["ref_host_ms_per_problem"] = round(ref_ms_per_problem(K, data, a.ref), 2)
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
