"""Batched convex programs (cp_batch) on B = 512 seeded problems (tests/cp_problems.py, seeds 0..B-1) at two shapes:
  qcqp64      n = 64,  qcqp family (mnl = 3 quadratic constraints), r = 16 (ml = 2n + r = 144);
  entropy256  n = 256, entropy family (mnl = 0, domain x > 0), p = 8, r = 32.
A warm-up solve of each shape precedes the timed one.  Prints one JSON line per shape: solve_ms (CUDA events around
the solve), lock-step iterations, line-search rounds (domain rounds included), kernel launches per lock-step iteration
(summed over the concurrent sub-batches), problems/s, status counts, F's calls and the time inside F: its device time
from CUDA events recorded on the batch's stream around each call (f_device_share: the mean over sub-batches of that
time over solve_ms) and its host time (f_host_share: over the solve's wall time; evaluations hold the GIL, so they run
one at a time), and the card name and power limit read in the same run.  With --ref K it also times the reference's
solvers.cp (oracle/_ref) on the first K problems of each shape, on the host, and reports its time per problem."""
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

SHAPES = [("qcqp64", "qcqp", 64, 0, 16), ("entropy256", "entropy", 256, 8, 32)]


def ref_ms_per_problem(family, d, count):
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    from cvxopt import matrix, solvers
    from cp_problems import ref_F
    m = lambda v: matrix(np.ascontiguousarray(v, dtype=np.float64))     # noqa: E731
    t0 = time.perf_counter()
    for k in range(count):
        kw = {}
        if d["G"].shape[1]:
            kw.update(G=m(d["G"][k]), h=m(d["h"][k]))
        if d["A"].shape[1]:
            kw.update(A=m(d["A"][k]), b=m(d["b"][k]))
        solvers.cp(ref_F(family, d["data"], k, d["x0"][k]), options=dict(show_progress=False), **kw)
    return (time.perf_counter() - t0) * 1e3 / count


def timed(F):
    """F with CUDA events and a host clock around every call, kept per stream"""
    import torch
    rec = collections.defaultdict(list)
    host = [0.0, 0]

    def G(x=None, z=None, idx=None):
        if x is None:
            return F()
        st = torch.cuda.current_stream()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record(st)
        out = F(x, z, idx=idx)
        e1.record(st)
        host[0] += time.perf_counter() - t0
        host[1] += 1
        rec[st.cuda_stream].append((e0, e1))
        return out

    def report():
        torch.cuda.synchronize()
        dev = [sum(a.elapsed_time(b) for a, b in v) for v in rec.values()]
        return dev, host[0] * 1e3, host[1]
    return G, report


def main():
    import cvxopt_b200
    from batch_coneqp_bench import card
    from cp_problems import cp_batch_data, torch_F
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=512)
    ap.add_argument("--ref", type=int, default=0, help="time the reference on the first K problems of each shape")
    ap.add_argument("--shapes", default="qcqp64,entropy256")
    a = ap.parse_args()
    if cvxopt_b200.device_count() == 0:
        raise SystemExit("batch_cp_bench: no GPU visible")
    gpu = card()
    for name, family, n, p, r in SHAPES:
        if name not in a.shapes.split(","):
            continue
        d = cp_batch_data(family, range(a.B), n, p, r)
        args = (d["G"], d["h"], None, d["A"] if p else None, d["b"] if p else None)
        cvxopt_b200.cp_batch(torch_F(family, d["data"], d["x0"]), *args)          # warm-up
        F, report = timed(torch_F(family, d["data"], d["x0"]))
        before = cvxopt_b200.launch_count()
        out = cvxopt_b200.cp_batch(F, *args)
        launches = cvxopt_b200.launch_count() - before
        dev, host_ms, calls = report()
        it = out["lockstep_iterations"]
        row = {"shape": name, "family": family, "n": n, "p": p, "r": r, "B": a.B, "card": gpu,
               "solve_ms": round(out["solve_ms"], 2), "solve_wall_ms": round(out["solve_wall_ms"], 2),
               "lockstep_iterations": it, "line_search_rounds": out["line_search_rounds"], "nsub": out["nsub"],
               "launches_per_iteration": round(launches / max(1, it), 1),
               "problems_per_s": round(a.B / out["solve_ms"] * 1e3, 1),
               "F_calls": calls, "f_device_ms": [round(v, 2) for v in dev],
               "f_device_share": round(float(np.mean(dev)) / out["solve_ms"], 3),
               "f_host_ms": round(host_ms, 2), "f_host_share": round(host_ms / out["solve_wall_ms"], 3),
               "status": dict(collections.Counter(out["status"])),
               "iterations_min_max": [int(np.min(out["iterations"])), int(np.max(out["iterations"]))]}
        if a.ref:
            row["ref_host_ms_per_problem"] = round(ref_ms_per_problem(family, d, a.ref), 2)
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
