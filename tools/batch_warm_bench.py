"""Warm-started re-solves of the batch solvers (cvxb_batch_load_start) on three shapes of B = 512 seeded problems:
  qp    config 4's shape, n = 512, {'l': 1024} QPs (batch_cones_bench's l_batch), through QPBatchGroup;
  socp  batch_cones_bench's SOC shape, n = 256, {'q': [8]*64} QPs (its cone_batch), through QPBatchGroup;
  sdp   batch_sdp_bench's first shape, n = 128, {'l': 64, 's': [16, 16]} cone LPs, through SDPBatchGroup.
Each batch is solved cold, then q (c) and h are perturbed by a seeded relative 1e-3 (x (1 + 1e-3 N(0, 1)) per entry),
and the perturbed batch is solved twice: cold, and warm from the first solution's x and y with s and z pushed into
the interior by push_interior (t = 1e-3).  A warm-up solve of each shape precedes the timed ones.  Prints one JSON line
per shape and leg: solve_ms, lock-step iterations, total iterations over the problems, problems/s, the optimal count,
and the card name and power limit read in the same run."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def push_interior(v, dims, t=1e-3):
    """v (B, cdim) + t max(1, max|v_k|) e for each problem k, e being 1 on the 'l' rows, on each 'q' cone's first row
    and on each 's' block's diagonal: a point of the closed cones moves strictly inside them"""
    d = {"l": dims.get("l", 0), "q": list(dims.get("q", [])), "s": list(dims.get("s", []))}
    rows = list(range(d["l"]))
    o = d["l"]
    for k in d["q"]:
        rows.append(o)
        o += k
    for k in d["s"]:
        rows += [o + i * (k + 1) for i in range(k)]
        o += k * k
    v = np.array(v, dtype=np.float64)
    v[:, rows] += (t * np.maximum(1.0, np.abs(v).max(axis=1)))[:, None]
    return v


def perturb(a, rng, eps=1e-3):
    return a * (1.0 + eps * rng.standard_normal(a.shape))


def main():
    import cvxopt_b200
    from batch_cones_bench import cone_batch, l_batch
    from batch_coneqp_bench import card
    from cvxopt_b200 import QPBatchGroup, SDPBatchGroup, batch as bt
    from test_batch_sdp_gpu import sdp_batch_data
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=512)
    a = ap.parse_args()
    if cvxopt_b200.device_count() == 0:
        raise SystemExit("batch_warm_bench: no GPU visible")
    gpu = card()
    B = a.B
    shapes = [("qp", 512, {"l": 1024}), ("socp", 256, {"l": 0, "q": [8] * 64}), ("sdp", 128, {"l": 64, "s": [16, 16]})]
    for name, n, dims in shapes:
        rng = np.random.Generator(np.random.PCG64(7))
        if name == "sdp":
            c, G, h, _, _ = sdp_batch_data(B, n, dims, 0, 42)
            group = lambda: SDPBatchGroup(B, n, dims)
            first = (c, G, h, None, None)
            second = (perturb(c, rng), G, perturb(h, rng), None, None)
        else:
            P, q, G, h = l_batch(B, n, 1024, 0) if name == "qp" else cone_batch(B, n, dims, 0)
            m = G.shape[1]
            group = lambda: QPBatchGroup(B, n, m, 0, None, dims)
            first = (P, q, G, h, None, None)
            second = (P, perturb(q, rng), G, perturb(h, rng), None, None)
        bt._run_group(group(), first, {})                                  # warm-up
        base = bt._run_group(group(), first, {})
        start = {"x": base["x"], "s": push_interior(base["s"], dims), "z": push_interior(base["z"], dims)}
        legs = [("first", first, None), ("perturbed_cold", second, None), ("perturbed_warm", second, start)]
        for leg, data, st in legs:
            out = base if leg == "first" else bt._run_group(group(), data, {}, st)
            row = {"shape": name, "dims": {k: (v if k != "q" else v[:1] + ["x%d" % len(v)]) for k, v in dims.items()},
                   "n": n, "B": B, "leg": leg, "card": gpu, "solve_ms": round(out["solve_ms"], 2),
                   "lockstep_iterations": out["lockstep_iterations"],
                   "total_iterations": int(np.sum(out["iterations"])),
                   "problems_per_s": round(B / out["solve_ms"] * 1e3, 1),
                   "optimal": int(sum(s == "optimal" for s in out["status"]))}
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
