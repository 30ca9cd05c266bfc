"""Batched convex QCQPs: qcqp_batch (F evaluated by the library's kernels) against cp_batch with cp_problems' torch F
on the same B = 512 seeded problems, at two shapes:
  qcqp64   n = 64,  mnl = 3, r = 16, p = 0: batch_cp_bench.py's qcqp64 (tests/cp_problems.py's qcqp family);
  qcqp256  n = 256, mnl = 3, r = 32, p = 8: tests/qcqp_problems.py's quad family (P_i symmetrised for the torch F).
Each shape warms up both solvers, then alternates them --reps times.  One JSON line per shape and solver with every
rep's solve_ms (CUDA events around the solve), their median, lock-step iterations, line-search rounds, launches per
lock-step iteration (summed over the concurrent sub-batches), problems/s at the median, status counts, and the card
name and power limit read in the same run.  Then, per shape, one line from a separate profiled qcqp_batch run
(torch.profiler, maxiters 3 and compaction off, so that every iterate evaluation covers all B slots): the new kernels'
time, launches and, for k_qc_hessian, k_qc_eval<true> and k_qc_rx, the bytes they must move over their kernel time.
The P x GEMV runs in gemv_n's kernels, which the other GEMVs share: it is not separated."""
import argparse
import collections
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

SHAPES = [("qcqp64", 64, 3, 0, 16), ("qcqp256", 256, 3, 8, 32)]


def shape_data(name, B, n, mnl, p, r):
    """(P, q, r, G, h, A, b) for qcqp_batch and the torch F's data dict for cp_batch"""
    if name == "qcqp64":
        from cp_problems import cp_batch_data
        d = cp_batch_data("qcqp", range(B), n, p, r)
        D = d["data"]
        return (D["P"], D["q"], D["r"], d["G"], d["h"], None, None), D, d["x0"]
    from qcqp_problems import qcqp_batch_data, sym
    d = qcqp_batch_data(range(B), n, mnl, p, r)
    D = {"P": sym(d["P"]), "q": d["q"], "r": d["r"]}
    return (d["P"], d["q"], d["r"], d["G"], d["h"], d["A"], d["b"]), D, d["x0"]


def kernel_bytes(B, n, mnl, S):
    """bytes per launch over B active slots that each new kernel must read and write (8-byte doubles)"""
    nK = mnl + 1
    return {"k_qc_hessian": 8 * B * (nK * n * (n + 1) // 2 + n * n),     # lower triangles of P_i; H mirrored
            "k_qc_eval<true>": 8 * B * (2 * S + n + nK + n + mnl * n),    # u, q, x, r; grad f0 and Df[1:]
            "k_qc_rx": 8 * B * (nK * n + mnl + 2 * n)}                   # Df, z, rx read and written


def profile(cvxopt_b200, args, B, n, mnl):
    import torch
    from torch.profiler import ProfilerActivity
    os.environ["CVXB_BATCH_COMPACT"] = "0"
    try:
        with torch.profiler.profile(activities=[ProfilerActivity.CUDA]) as prof:
            out = cvxopt_b200.qcqp_batch(*args[:5], None, *args[5:], maxiters=3)
            torch.cuda.synchronize()
    finally:
        del os.environ["CVXB_BATCH_COMPACT"]
    nb = out["nsub"]
    per = kernel_bytes(B // nb, n, mnl, (mnl + 1) * n)
    rows = {}
    for e in prof.key_averages():
        for keys, tag in ((("k_qc_hessian",), "k_qc_hessian"), (("k_qc_evalILb1", "k_qc_eval<true>"), "k_qc_eval<true>"),
                          (("k_qc_evalILb0", "k_qc_eval<false>"), "k_qc_eval<false>"), (("k_qc_rx",), "k_qc_rx")):
            if any(k in e.key for k in keys):
                us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
                r = rows.setdefault(tag, {"launches": 0, "kernel_ms": 0.0})
                r["launches"] += e.count
                r["kernel_ms"] += us / 1e3
    for tag, r in rows.items():
        r["kernel_ms"] = round(r["kernel_ms"], 3)
        if tag in per and r["kernel_ms"] > 0:
            r["GB_per_s"] = round(per[tag] * r["launches"] / (r["kernel_ms"] * 1e-3) / 1e9, 1)
    return rows


def main():
    import cvxopt_b200
    from batch_coneqp_bench import card
    from cp_problems import torch_F
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=512)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--shapes", default="qcqp64,qcqp256")
    a = ap.parse_args()
    if cvxopt_b200.device_count() == 0:
        raise SystemExit("batch_qcqp_bench: no GPU visible")
    gpu = card()
    for name, n, mnl, p, r in SHAPES:
        if name not in a.shapes.split(","):
            continue
        args, D, x0 = shape_data(name, a.B, n, mnl, p, r)
        P, q, rr, G, h, A, b = args
        F = torch_F("qcqp", D, x0)

        def qc():
            return cvxopt_b200.qcqp_batch(P, q, rr, G, h, None, A, b, x0=x0)

        def cp():
            return cvxopt_b200.cp_batch(F, G, h, None, A, b)
        runs = {"qcqp_batch": qc, "cp_batch": cp}
        for fn in runs.values():
            fn()                                                      # warm-up
        res = collections.defaultdict(list)
        for _ in range(a.reps):
            for key, fn in runs.items():
                before = cvxopt_b200.launch_count()
                out = fn()
                res[key].append((out, cvxopt_b200.launch_count() - before))
        for key, rs in res.items():
            out, launches = rs[-1]
            ms = [round(o["solve_ms"], 2) for o, _ in rs]
            it = out["lockstep_iterations"]
            print(json.dumps({"shape": name, "solver": key, "n": n, "mnl": mnl, "p": p, "r": r, "B": a.B,
                              "card": gpu, "solve_ms": ms, "solve_ms_median": float(np.median(ms)),
                              "solve_wall_ms": [round(o["solve_wall_ms"], 2) for o, _ in rs],
                              "lockstep_iterations": it, "line_search_rounds": out["line_search_rounds"],
                              "nsub": out["nsub"], "launches_per_iteration": round(launches / max(1, it), 1),
                              "problems_per_s": round(a.B / float(np.median(ms)) * 1e3, 1),
                              "status": dict(collections.Counter(out["status"])),
                              "iterations_min_max": [int(np.min(out["iterations"])),
                                                     int(np.max(out["iterations"]))]}), flush=True)
        qc_x, cp_x = res["qcqp_batch"][-1][0]["x"], res["cp_batch"][-1][0]["x"]
        print(json.dumps({"shape": name, "card": gpu, "x_max_rel_diff_qcqp_vs_cp":
                          float(np.max(np.linalg.norm(qc_x - cp_x, axis=1) /
                                       np.maximum(1.0, np.linalg.norm(cp_x, axis=1)))),
                          "kernels": profile(cvxopt_b200, args, a.B, n, mnl)}), flush=True)


if __name__ == "__main__":
    main()
