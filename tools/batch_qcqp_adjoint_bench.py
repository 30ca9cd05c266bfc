"""The QCQP batch's adjoint (cvxb_batch_adjoint_qcqp) against a dense torch baseline, at two shapes of
tests/qcqp_problems.py's quad family:
  layer    B = 4096, n = 32,  mnl = 4, r = 16, p = 4  (a layer-sized batch);
  qcqp256  B = 512,  n = 256, mnl = 3, r = 32, p = 8  (tools/batch_qcqp_bench.py's qcqp256).
The problems are loaded into one QCQPBatch (nsub = 1) from device memory and solved.  Per rep: the solve's solve_ms
(CUDA events), then adjoint_ms, a host clock around one device-space cvxb_batch_adjoint_qcqp call with every output (the
call ends in a stream synchronise), then the torch baseline: the full (n + p + m)^2 KKT matrix per problem at the same
iterate (H = P_0 + sum znl_i P_i, Df's rows P_i x + q_i), batched torch.linalg.solve and the outer products, timed with
CUDA events on torch's stream.  After --reps reps, a separate torch.profiler run gives the gradient kernel's
(k_adj_qc_grad) own time and its achieved bytes/s: B (nK n^2 + nK n + nK + ml n + p n) 8 bytes written over its kernel
time, against the 3.35 TB/s HBM3 data-sheet bound.  One JSON line per shape, with the card name and power limit read in
the same run and the largest relative difference of the baseline's gradients from the adjoint's."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

SHAPES = {"layer": (4096, 32, 4, 4, 16), "qcqp256": (512, 256, 3, 8, 32)}    # B, n, mnl, p, r
HBM_BYTES_PER_S = 3.35e12


def torch_baseline(P, q, G, A, x, y, s, z, gx, gy, gz):
    """the dense KKT solve and outer products in torch, P the symmetric (B, nK, n, n): (dP, dq, dr, dG, dA, uy, uzl)"""
    import torch
    B, nK, n = P.shape[:3]
    mnl, m, p = nK - 1, s.shape[1], y.shape[1]
    N = n + p + m
    znl = z[:, :mnl]
    H = P[:, 0] + (znl[:, :, None, None] * P[:, 1:]).sum(1)
    Gf = torch.cat([(P[:, 1:] @ x[:, None, :, None])[..., 0] + q[:, 1:], G], 1)
    K = torch.zeros((B, N, N), dtype=P.dtype, device=P.device)
    K[:, :n, :n] = H
    K[:, n:n + p, :n] = A
    K[:, :n, n:n + p] = A.transpose(1, 2)
    K[:, n + p:, :n] = Gf
    K[:, :n, n + p:] = Gf.transpose(1, 2)
    K[:, n + p:, n + p:] = -torch.diag_embed(s / z)
    u = torch.linalg.solve(K, torch.cat([gx, gy, gz], 1))
    ux, uy, uz = u[:, :n], u[:, n:n + p], u[:, n + p:]
    o = lambda a, c: a[:, :, None] * c[:, None, :]          # noqa: E731  batched outer product
    zk = torch.cat([torch.ones((B, 1), dtype=P.dtype, device=P.device), znl], 1)
    uk = torch.cat([torch.zeros((B, 1), dtype=P.dtype, device=P.device), uz[:, :mnl]], 1)
    S, xx = o(ux, x) + o(x, ux), o(x, x)
    dP = -0.5 * (zk[:, :, None, None] * S[:, None] + uk[:, :, None, None] * xx[:, None])
    dq = -(zk[:, :, None] * ux[:, None] + uk[:, :, None] * x[:, None])
    dG = -(o(z[:, mnl:], ux) + o(uz[:, mnl:], x))
    dA = -(o(y, ux) + o(uy, x))
    return dP, dq, -uk, dG, dA, uy, uz[:, mnl:]


def main():
    import torch
    from torch.profiler import ProfilerActivity
    import cvxopt_b200
    from cvxopt_b200 import QCQPBatch, _lib
    from batch_coneqp_bench import card
    from qcqp_problems import qcqp_batch_data, sym
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--shapes", default="layer,qcqp256")
    a = ap.parse_args()
    if cvxopt_b200.device_count() == 0:
        raise SystemExit("batch_qcqp_adjoint_bench: no GPU visible")
    gpu = card()
    dev = torch.device("cuda", 0)
    f64 = dict(dtype=torch.float64, device=dev)
    for name in a.shapes.split(","):
        B, n, mnl, p, r = SHAPES[name]
        d = qcqp_batch_data(range(B), n, mnl, p, r)
        nK, ml = mnl + 1, d["G"].shape[1]
        m = mnl + ml
        Ps = torch.from_numpy(sym(d["P"])).to(dev)                          # symmetric, for the baseline
        q, G, A = (torch.from_numpy(d[k]).to(dev) for k in ("q", "G", "A"))
        data = [torch.from_numpy(np.ascontiguousarray(np.transpose(d["P"], (0, 3, 1, 2)))).to(dev), q,
                torch.from_numpy(d["r"]).to(dev), torch.from_numpy(d["x0"]).to(dev),
                G.transpose(1, 2).contiguous(), torch.from_numpy(d["h"]).to(dev)]
        eq = [A.transpose(1, 2).contiguous(), torch.from_numpy(d["b"]).to(dev)]
        del d
        gen = torch.Generator(device=dev).manual_seed(1)
        gx, gy, gz = (torch.randn((B, k), generator=gen, **f64) for k in (n, p, m))
        qb = QCQPBatch(B, n, mnl, ml, p, 0)
        x, y, s, z = (torch.empty((B, k), **f64) for k in (n, p, m, m))
        outs = [torch.empty(sh, **f64) for sh in ((B, n), (B, p), (B, m), (B, n, nK, n), (B, nK, n), (B, nK),
                                                  (B, n, ml), (B, n, p))]
        torch.cuda.synchronize()
        qb.load_ptr(*(t.data_ptr() for t in data), _lib.DEVICE, *(t.data_ptr() for t in eq))
        solve_ms, adjoint_ms, torch_ms = [], [], []
        for rep in range(a.reps + 1):                      # rep 0 warms up every path
            qb.solve()
            solve_ms.append(qb.stats()["solve_ms"])
            _lib.check(qb._lib.cvxb_batch_results(qb._h, x.data_ptr(), s.data_ptr(), z.data_ptr(), None, None, None,
                                                  None, _lib.DEVICE), "batch_results")
            _lib.check(qb._lib.cvxb_batch_results_y(qb._h, y.data_ptr(), _lib.DEVICE), "batch_results_y")
            t0 = time.perf_counter()
            qb.adjoint_ptr(gx.data_ptr(), gy.data_ptr(), gz.data_ptr(), *(t.data_ptr() for t in outs))
            adjoint_ms.append((time.perf_counter() - t0) * 1e3)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            base = torch_baseline(Ps, q, G, A, x, y, s, z, gx, gy, gz)
            e1.record()
            e1.synchronize()
            torch_ms.append(e0.elapsed_time(e1))
        status = np.zeros(B, dtype=np.int32)
        _lib.check(qb._lib.cvxb_batch_results(qb._h, None, None, None, status.ctypes.data, None, None, None,
                                              _lib.HOST), "batch_results")
        ok = torch.from_numpy(status == 1).to(dev)
        ours = (outs[3].permute(0, 2, 3, 1), outs[4], outs[5], outs[6].transpose(1, 2), outs[7].transpose(1, 2),
                outs[1], outs[2][:, mnl:])
        diff = max(float(((u - v)[ok].norm() / v[ok].norm().clamp_min(1e-300)).item()) if v.numel() else 0.0
                   for u, v in zip(ours, base))
        del base
        with torch.profiler.profile(activities=[ProfilerActivity.CUDA]) as prof:
            qb.adjoint_ptr(gx.data_ptr(), gy.data_ptr(), gz.data_ptr(), *(t.data_ptr() for t in outs))
            torch.cuda.synchronize()
        grad_ms = sum((getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0))
                      for e in prof.key_averages() if "k_adj_qc_grad" in e.key) / 1e3
        qb.close()
        written = 8 * B * (nK * n * n + nK * n + nK + ml * n + p * n)
        t = lambda v: [round(x, 3) for x in v[1:]]          # noqa: E731  the timed reps
        print(json.dumps({
            "shape": name, "B": B, "n": n, "mnl": mnl, "ml": ml, "p": p, "card": gpu, "reps": a.reps,
            "status_optimal": int((status == 1).sum()),
            "solve_ms": t(solve_ms), "adjoint_ms": t(adjoint_ms), "adjoint_ms_median": float(np.median(adjoint_ms[1:])),
            "torch_baseline_ms": t(torch_ms), "torch_baseline_ms_median": float(np.median(torch_ms[1:])),
            "grad_kernel_ms": round(grad_ms, 3), "grad_bytes_written": written,
            "grad_kernel_GB_per_s": round(written / (grad_ms * 1e-3) / 1e9, 1) if grad_ms else None,
            "grad_kernel_share_of_3.35TB_per_s": round(written / (grad_ms * 1e-3) / HBM_BYTES_PER_S, 3) if grad_ms
            else None,
            "max_rel_diff_torch_vs_adjoint": diff}), flush=True)
        del Ps, q, G, A, data, eq, outs
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
