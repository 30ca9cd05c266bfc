"""Cost of equality constraints A x = b in the batch solver (csrc/batch_ipm.cu, kkt_chol2's elimination).

The config 4 shape of BASELINE (512 problems, n = 512, {'l': 1024}) with p = 0, 64 and 256 equality rows per
problem, run alternately in one process, `--reps` times.  P, q, G, h are bench.py's config 4 problems
(tests/problems.dense_qp); A ~ N(0,1) and b = A x0 at dense_qp's own interior point x0, so every problem stays
strictly feasible.  One sub-batch (nsub=1), so solve_ms / lockstep_iterations is the time of one lock-step
iteration.  Each line also gives the launches per lock-step iteration and the card read in the same run.

    python tools/batch_eq_bench.py [--reps 3] [--ps 0,64,256] [--batch 512]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from problems import dense_qp  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    return out[1] if len(out) > 1 else ""


def eq_batch(B, n, m, pmax, seed0):
    """config 4's problems, plus pmax equality rows through each problem's x0 (the first p of them are used)"""
    P, q, G, h = np.empty((B, n, n)), np.empty((B, n)), np.empty((B, m, n)), np.empty((B, m))
    A, b = np.empty((B, pmax, n)), np.empty((B, pmax))
    for k in range(B):
        P[k], q[k], G[k], h[k] = dense_qp(n, m, seed=seed0 + k)
        rng = np.random.Generator(np.random.PCG64(seed0 + k))       # replays dense_qp's draws up to x0
        rng.standard_normal((n, n)); rng.standard_normal(n); rng.standard_normal((m, n))
        x0 = rng.standard_normal(n)
        A[k] = np.random.Generator(np.random.PCG64(10 ** 6 + seed0 + k)).standard_normal((pmax, n))
        b[k] = A[k] @ x0
    return P, q, G, h, A, b


def run(batch, p):
    import cvxopt_b200
    P, q, G, h, A, b = batch
    eq = (A[:, :p], b[:, :p]) if p else ()
    c0 = cvxopt_b200.launch_count()
    r = cvxopt_b200.qp_batch(P, q, G, h, *eq, nsub=1)
    launches = cvxopt_b200.launch_count() - c0
    it = max(1, r["lockstep_iterations"])
    return {"p": p, "solve_ms": r["solve_ms"], "lockstep_iterations": r["lockstep_iterations"],
            "ms_per_lockstep_iteration": r["solve_ms"] / it, "launches_per_lockstep_iteration": launches / it,
            "total_iterations": int(np.sum(r["iterations"])),
            "optimal": int(sum(s == "optimal" for s in r["status"]))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ps", default="0,64,256")
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--n", type=int, default=512)
    ap.add_argument("--m", type=int, default=1024)
    args = ap.parse_args()
    import cvxopt_b200
    if cvxopt_b200.device_count() == 0:
        raise SystemExit("batch_eq_bench: no H100 visible")
    ps = [int(v) for v in args.ps.split(",")]
    batch = eq_batch(args.batch, args.n, args.m, max(ps), 0)
    gpu = card()
    for p in ps:                                   # warm-up: every shape once
        run(tuple(x[:8] for x in batch), p)
    for rep in range(args.reps):
        for p in ps:
            res = run(batch, p)
            res.update({"rep": rep, "B": args.batch, "n": args.n, "m": args.m, "card": gpu})
            print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
