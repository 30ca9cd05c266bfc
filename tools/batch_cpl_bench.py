"""Batched cpl problems (cpl_batch) on B = 512 seeded feasible problems (tests/cpl_problems.py, seeds 0..B-1) at two
shapes of the socp family (mnl = 2 quadratic constraints, 'l' rows and second-order cones of different lengths):
  socp64   n = 64,  ml = 16, q = [3, 8, 16, 33], p = 4;
  socp256  n = 256, ml = 32, q = [5, 17, 64, 129], p = 8;
and, with semidefinite cones (sdp_cpl_batch on tests/sdcpl_problems.py's socp family with LMI rows):
  sdp64    n = 64,  ml = 16, q = [8], s = [16, 16];
  sdp128   n = 128, ml = 16, s = [32].
A warm-up solve of each shape precedes the timed one.  Prints one JSON line per shape: solve_ms (CUDA events around
the solve), lock-step iterations, line-search rounds (domain rounds included), launches per lock-step iteration (the
launches of both sub-batches, line-search rounds included, over the lock-step iterations), problems/s, status counts, F's calls and
their host time, and the card name and power limit read in the same run.  With --ref K it also times the
reference's solvers.cpl (oracle/_ref) on the first K problems of each shape, on the host, and reports its time per
problem."""
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

SHAPES = [("socp64", "socp", 64, [3, 8, 16, 33], 16, 4, []), ("socp256", "socp", 256, [5, 17, 64, 129], 32, 8, []),
          ("sdp64", "socp", 64, [8], 16, 0, [16, 16]), ("sdp128", "socp", 128, [], 16, 0, [32])]


def ref_ms_per_problem(family, d, count):
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    from cvxopt import matrix, solvers
    from cpl_problems import ref_F
    m = lambda v: matrix(np.ascontiguousarray(v, dtype=np.float64))     # noqa: E731
    t0 = time.perf_counter()
    for k in range(count):
        kw = dict(G=m(d["G"][k]), h=m(d["h"][k]))
        if d["A"].shape[1]:
            kw.update(A=m(d["A"][k]), b=m(d["b"][k]))
        solvers.cpl(m(d["c"][k]), ref_F(family, d["data"], k, d["x0"][k]), dims=d["dims"],
                    options=dict(show_progress=False), **kw)
    return (time.perf_counter() - t0) * 1e3 / count


def main():
    import cvxopt_b200
    from batch_coneqp_bench import card
    from cpl_problems import cpl_batch_data, torch_F
    from sdcpl_problems import sdcpl_batch_data
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=512)
    ap.add_argument("--ref", type=int, default=0, help="time the reference on the first K problems of each shape")
    ap.add_argument("--shapes", default="socp64,socp256")
    a = ap.parse_args()
    if cvxopt_b200.device_count() == 0:
        raise SystemExit("batch_cpl_bench: no GPU visible")
    gpu = card()
    for name, family, n, q, ml, p, s in SHAPES:
        if name not in a.shapes.split(","):
            continue
        d = sdcpl_batch_data(family, range(a.B), n, q, s, ml, p) if s else \
            cpl_batch_data(family, range(a.B), n, q, ml, p)
        solve = cvxopt_b200.sdp_cpl_batch if s else cvxopt_b200.cpl_batch
        args = (d["G"], d["h"], d["dims"], d["A"] if p else None, d["b"] if p else None)
        solve(d["c"], torch_F(family, d["data"], d["x0"]), *args)          # warm-up
        F, host = torch_F(family, d["data"], d["x0"]), [0.0, 0]

        def timed_F(x=None, z=None, idx=None):
            if x is None:
                return F()
            t0 = time.perf_counter()
            out = F(x, z, idx=idx)
            host[0] += time.perf_counter() - t0
            host[1] += 1
            return out
        l0 = cvxopt_b200.launch_count()
        out = solve(d["c"], timed_F, *args)
        launches = cvxopt_b200.launch_count() - l0
        row = {"shape": name, "family": family, "n": n, "q": q, "s": s, "ml": ml, "p": p, "B": a.B, "card": gpu,
               "solve_ms": round(out["solve_ms"], 2), "solve_wall_ms": round(out["solve_wall_ms"], 2),
               "lockstep_iterations": out["lockstep_iterations"], "line_search_rounds": out["line_search_rounds"],
               "launches_per_iteration": round(launches / max(1, out["lockstep_iterations"]), 1),
               "nsub": out["nsub"], "problems_per_s": round(a.B / out["solve_ms"] * 1e3, 1),
               "F_calls": host[1], "f_host_ms": round(host[0] * 1e3, 2),
               "status": dict(collections.Counter(out["status"])),
               "iterations_min_max": [int(np.min(out["iterations"])), int(np.max(out["iterations"]))]}
        if a.ref:
            row["ref_host_ms_per_problem"] = round(ref_ms_per_problem(family, d, a.ref), 2)
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
