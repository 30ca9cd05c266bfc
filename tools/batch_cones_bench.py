"""Throughput of the batch solver with 'q' cones (csrc/batch_ipm.cu; Gs = W^{-T} G is materialised only with them).

Two workloads, each printed as one JSON line:
  cone4  512 problems, n = 512, {'l': 512, 'q': [16]*32} (cdim 1024, the m of BASELINE config 4), run alternately in
         the same process with config 4 itself ({'l': 1024}, di² fused into the SYRK): the difference is the cost of
         the cones at an equal G size.
  soc    256 problems, n = 256, {'l': 0, 'q': [8]*64}.
Both use one sub-batch (nsub=1), so solve_ms / lockstep_iterations is the time of one lock-step iteration.  With
oracle/_ref built, the reference loop over solvers.coneqp runs on the first 16 problems: its wall time and whether
the iteration counts agree.

    python tools/batch_cones_bench.py [--reps 2] [--workloads cone4,soc] [--nref 16]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from problems import cone_point, dense_qp  # noqa: E402


def full(dims):
    return {"l": dims.get("l", 0), "q": list(dims.get("q", [])), "s": []}


def cone_batch(B, n, dims, seed0):
    dims = full(dims)
    m = dims["l"] + sum(dims["q"])
    P, q, G, h = np.empty((B, n, n)), np.empty((B, n)), np.empty((B, m, n)), np.empty((B, m))
    for k in range(B):
        rng = np.random.Generator(np.random.PCG64(seed0 + k))
        A0 = rng.standard_normal((n, n))
        P[k] = A0.T @ A0 / n + np.eye(n)
        q[k] = rng.standard_normal(n)
        G[k] = rng.standard_normal((m, n))
        x0 = rng.standard_normal(n)
        h[k] = G[k] @ x0 + cone_point(dims, rng)
    return P, q, G, h


def l_batch(B, n, m, seed0):
    P, q, G, h = np.empty((B, n, n)), np.empty((B, n)), np.empty((B, m, n)), np.empty((B, m))
    for k in range(B):
        P[k], q[k], G[k], h[k] = dense_qp(n, m, seed=seed0 + k)
    return P, q, G, h


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[1] if len(out) > 1 else ""
    except (OSError, subprocess.SubprocessError):
        return ""


def run(batch, dims):
    import cvxopt_b200
    r = cvxopt_b200.qp_batch(*batch, nsub=1, dims=dims)
    B = len(r["iterations"])
    return {"solve_ms": r["solve_ms"], "lockstep_iterations": r["lockstep_iterations"],
            "ms_per_lockstep_iteration": r["solve_ms"] / max(1, r["lockstep_iterations"]),
            "total_iterations": int(np.sum(r["iterations"])), "problems_per_s": B / (r["solve_ms"] * 1e-3),
            "optimal": int(sum(s == "optimal" for s in r["status"]))}, r


def reference(batch, dims, got, nref):
    refdir = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.isdir(os.path.join(refdir, "cvxopt")) or nref <= 0:
        return {}
    sys.path.insert(0, refdir)
    from cvxopt import matrix, solvers
    solvers.options["show_progress"] = False
    P, q, G, h = batch
    k = min(nref, P.shape[0])
    t0 = time.perf_counter()
    its = [solvers.coneqp(matrix(P[i]), matrix(q[i]), matrix(G[i]), matrix(h[i]), full(dims),
                          kktsolver="chol")["iterations"] for i in range(k)]
    wall = (time.perf_counter() - t0) * 1e3
    return {"ref_problems": k, "ref_wall_ms": wall,
            "ref_iterations_agree": bool(list(its) == [int(v) for v in got["iterations"][:k]])}


def spread(vals):
    return {"min": min(vals), "median": float(np.median(vals)), "max": max(vals)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--workloads", default="cone4,soc")
    ap.add_argument("--nref", type=int, default=16)
    a = ap.parse_args()
    import cvxopt_b200
    if cvxopt_b200.device_count() == 0:
        raise SystemExit("no H100 visible: the batch solver has no CPU fallback")
    gpu = card()
    print("# card: name, power.limit, clocks.max.sm = %s" % gpu)
    for w in a.workloads.split(","):
        if w == "cone4":
            B, n, dims = 512, 512, {"l": 512, "q": [16] * 32}
            legs = [("cone", cone_batch(B, n, dims, 0), dims), ("l", l_batch(B, n, 1024, 0), None)]
        elif w == "soc":
            B, n, dims = 256, 256, {"l": 0, "q": [8] * 64}
            legs = [("cone", cone_batch(B, n, dims, 0), dims)]
        else:
            raise SystemExit("unknown workload %r" % w)
        for _, batch, d in legs:                         # warm-up on a slice: first launches, allocator
            run(tuple(x[:8] for x in batch), d)
        res = {name: [] for name, _, _ in legs}
        last = {}
        for _ in range(a.reps):                          # the legs alternate
            for name, batch, d in legs:
                st, r = run(batch, d)
                res[name].append(st)
                last[name] = r
        out = {"workload": w, "card": gpu, "nprob": B, "n": n, "dims": {"l": dims["l"], "q": dims["q"][:1] + ["x%d" % len(dims["q"])]},
               "reps": a.reps}
        for name in res:
            out[name] = {key: spread([s[key] for s in res[name]]) for key in res[name][0]}
        if "l" in res:
            c = out["cone"]["ms_per_lockstep_iteration"]["median"]
            l_ = out["l"]["ms_per_lockstep_iteration"]["median"]
            out["cone_over_l_per_iteration"] = c / l_
        out.update(reference(legs[0][1], dims, last["cone"], a.nref))
        print(json.dumps(out))
        sys.stdout.flush()


if __name__ == "__main__":
    main()
