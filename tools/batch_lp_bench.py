"""Throughput of the batched cone LP solver (conelp_batch: coneprog.conelp in lock-step, csrc/batch_ipm.cu).

Workloads, run alternately in one process, `--reps` times, one JSON line each:
  lp      512 dense LPs at config 4's shape (n = 512, {'l': 1024}), p = 0
  lp_eq   the same LPs with p = 64 equality rows through each problem's interior point
  socp    512 SOCPs, n = 512, {'l': 512, 'q': [16]*32}
  pinf    batch `lp` with every 20th problem (5 %) made primal infeasible, through conelp_batch
  pinf_qp the same batch through qp_batch with P = 0 (coneqp: no certificate, an infeasible problem runs until
          maxiters or a singular KKT matrix)
Problems: G, A ~ N(0,1), h = G x0 + s0, b = A x0, c = -(G'z0 + A'y0) with s0, z0 strictly inside the cones, so each
LP is feasible and bounded.  An infeasible problem's first row reads 0 x + s = -1.  One sub-batch (nsub=1), so
solve_ms / lockstep_iterations is the time of one lock-step iteration.  Each line gives solve_ms, the lock-step
iterations, ms and launches per lock-step iteration, problems/s, the status counts and the card read in the same run.

    python tools/batch_lp_bench.py [--reps 3] [--workloads lp,lp_eq,socp,pinf,pinf_qp] [--batch 512]
"""
import argparse
import json
import os
import subprocess
import sys
from collections import Counter

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from problems import cone_point  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    return out[1] if len(out) > 1 else ""


def lp_batch(B, n, dims, p, seed0, pinf_every=0):
    dims = {"l": dims.get("l", 0), "q": list(dims.get("q", [])), "s": []}
    m = dims["l"] + sum(dims["q"])
    c, G, h = np.empty((B, n)), np.empty((B, m, n)), np.empty((B, m))
    A, b = np.empty((B, p, n)), np.empty((B, p))
    for k in range(B):
        rng = np.random.Generator(np.random.PCG64(seed0 + k))
        G[k] = rng.standard_normal((m, n))
        A[k] = rng.standard_normal((p, n))
        x0, y0 = rng.standard_normal(n), rng.standard_normal(p)
        h[k] = G[k] @ x0 + cone_point(dims, rng)
        b[k] = A[k] @ x0
        c[k] = -(G[k].T @ cone_point(dims, rng) + A[k].T @ y0)
        if pinf_every and k % pinf_every == pinf_every - 1:
            G[k][0] = 0.0
            h[k][0] = -1.0
    return c, G, h, A, b


def run(name, batch, dims, p):
    import cvxopt_b200
    c, G, h, A, b = batch
    eq = dict(A=A[:, :p], b=b[:, :p]) if p else {}
    c0 = cvxopt_b200.launch_count()
    if name == "pinf_qp":
        B, n = c.shape
        r = cvxopt_b200.qp_batch(np.zeros((B, n, n)), c, G, h, dims=dims, nsub=1, **eq)
    else:
        r = cvxopt_b200.conelp_batch(c, G, h, dims=dims, nsub=1, **eq)
    launches = cvxopt_b200.launch_count() - c0
    it = max(1, r["lockstep_iterations"])
    return {"workload": name, "p": p, "solve_ms": r["solve_ms"], "lockstep_iterations": r["lockstep_iterations"],
            "ms_per_lockstep_iteration": r["solve_ms"] / it, "launches_per_lockstep_iteration": launches / it,
            "problems_per_s": c.shape[0] / (r["solve_ms"] * 1e-3), "total_iterations": int(np.sum(r["iterations"])),
            "status": dict(Counter(r["status"]))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--workloads", default="lp,lp_eq,socp,pinf,pinf_qp")
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--n", type=int, default=512)
    ap.add_argument("--m", type=int, default=1024)
    args = ap.parse_args()
    import cvxopt_b200
    if cvxopt_b200.device_count() == 0:
        raise SystemExit("batch_lp_bench: no H100 visible")
    B, n, m = args.batch, args.n, args.m
    ldims = {"l": m}
    sdims = {"l": m // 2, "q": [16] * (m // 32)}
    lp = lp_batch(B, n, ldims, 64, 0)
    soc = lp_batch(B, n, sdims, 0, 10 ** 5)
    pinf = lp_batch(B, n, ldims, 0, 0, pinf_every=20)
    work = {"lp": (lp, ldims, 0), "lp_eq": (lp, ldims, 64), "socp": (soc, sdims, 0),
            "pinf": (pinf, ldims, 0), "pinf_qp": (pinf, ldims, 0)}
    names = args.workloads.split(",")
    gpu = card()
    for name in names:                                  # warm-up: every shape once
        data, dims, p = work[name]
        run(name, tuple(x[:8] for x in data), dims, p)
    for rep in range(args.reps):
        for name in names:
            data, dims, p = work[name]
            res = run(name, data, dims, p)
            res.update({"rep": rep, "B": B, "n": n, "m": m, "card": gpu})
            print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
