"""Batched cone QP solver with 's' blocks (coneqp_batch / SDPQPBatchGroup) on two shapes of B = 512 seeded feasible
problems: {'l': 64, 's': [16, 16]} with n = 128, and {'s': [32]} (the largest order) with n = 256.  G, h and q are
sdp_batch's data (tests/test_batch_sdp_gpu.sdp_problem, c used as q) and P = M M' / n + 1e-3 I with M n x n Gaussian.
Prints one JSON line per shape: solve_ms, lock-step iterations, ms and launches per lock-step iteration, problems/s,
and the card name and power limit read in the same run.  --ref K also times the host loop over the reference's
solvers.coneqp(P, q, G, h, dims) (default kktsolver, 'chol' with 's' cones) on the first K problems, as CPU time."""
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
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip()
    except Exception as e:          # noqa: BLE001
        return "unknown (%s)" % e


def p_matrices(B, n, seed):
    rng = np.random.Generator(np.random.PCG64(seed))
    M = rng.standard_normal((B, n, n))
    return M @ M.transpose(0, 2, 1) / n + 1e-3 * np.eye(n)


def main():
    import cvxopt_b200
    from cvxopt_b200 import SDPQPBatchGroup, batch as bt
    from test_batch_sdp_gpu import sdp_batch_data
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=512)
    ap.add_argument("--ref", type=int, default=0)
    a = ap.parse_args()
    if cvxopt_b200.device_count() == 0:
        raise SystemExit("batch_coneqp_bench: no GPU visible")
    for n, dims in ((128, {"l": 64, "s": [16, 16]}), (256, {"s": [32]})):
        q, G, h, _, _ = sdp_batch_data(a.B, n, dims, 0, 42)
        P = p_matrices(a.B, n, 43)
        data = (P, q, G, h, None, None)
        bt._run_group(SDPQPBatchGroup(a.B, n, dims), data, {})            # warm-up
        l0 = cvxopt_b200.launch_count()
        out = bt._run_group(SDPQPBatchGroup(a.B, n, dims), data, {})
        launches = cvxopt_b200.launch_count() - l0
        it = out["lockstep_iterations"]
        row = {"shape": dims, "n": n, "B": a.B, "card": card(), "solve_ms": out["solve_ms"],
               "lockstep_iterations": it, "ms_per_iteration": out["solve_ms"] / max(it, 1),
               "launches_per_iteration": launches / max(it, 1), "problems_per_s": a.B / out["solve_ms"] * 1e3,
               "optimal": int(sum(s == "optimal" for s in out["status"]))}
        if a.ref:
            from cvxopt import matrix, solvers
            full = {"l": dims.get("l", 0), "q": [], "s": dims["s"]}
            t0 = time.perf_counter()
            for k in range(a.ref):
                solvers.coneqp(matrix(P[k]), matrix(q[k]), matrix(G[k]), matrix(h[k]), full,
                               options={"show_progress": False})
            row["reference_coneqp_cpu_ms_per_problem"] = (time.perf_counter() - t0) * 1e3 / a.ref
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
