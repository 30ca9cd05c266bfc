"""The QP batch's adjoint (cvxb_batch_adjoint) against what users write today in torch, at two shapes:
  config4  B = 512,  n = 512, m = 1024, p = 0  (BASELINE config 4's batch);
  layer    B = 8192, n = 32,  m = 64,   p = 8  (a layer-sized OptNet batch).
Seeded problems are built on the device (P = M M'/n + I, h = G x0 + U(0.5, 1.5), b = A x0), loaded into one QPBatch
(nsub = 1) from device memory and solved.  Per rep: the solve's solve_ms (CUDA events), then adjoint_ms, a host clock
around one device-space cvxb_batch_adjoint call with every output (the call ends in a stream synchronise), then the
torch baseline: the full (n + p + m)^2 KKT matrix per problem at the same iterate, batched torch.linalg.solve and the
outer products, timed with CUDA events on torch's stream.  After --reps reps, a separate torch.profiler run gives the
gradient kernel's (k_adj_grad) own time and its achieved bytes/s: B (n^2 + m n + p n) 8 bytes written over its kernel
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
sys.path.insert(0, os.path.join(ROOT, "tools"))

SHAPES = {"config4": (512, 512, 1024, 0), "layer": (8192, 32, 64, 8)}
HBM_BYTES_PER_S = 3.35e12


def problems(B, n, m, p, dev, seed=0):
    import torch
    g = torch.Generator(device=dev).manual_seed(seed)
    f64 = dict(dtype=torch.float64, device=dev)
    M = torch.randn((B, n, n), generator=g, **f64)
    P = M @ M.transpose(1, 2) / n + torch.eye(n, **f64)
    del M
    q = torch.randn((B, n), generator=g, **f64)
    G = torch.randn((B, m, n), generator=g, **f64)
    x0 = torch.randn((B, n, 1), generator=g, **f64)
    h = (G @ x0)[..., 0] + 0.5 + torch.rand((B, m), generator=g, **f64)
    A = torch.randn((B, p, n), generator=g, **f64)
    b = (A @ x0)[..., 0]
    return P, q, G, h, A, b


def torch_baseline(P, G, A, x, y, s, z, gx, gy, gz):
    """the dense KKT solve and outer products in torch: (dP, dG, dA, ux, uy, uz)"""
    import torch
    B, n = x.shape
    m, p = s.shape[1], y.shape[1]
    N = n + p + m
    K = torch.zeros((B, N, N), dtype=P.dtype, device=P.device)
    K[:, :n, :n] = P
    K[:, n:n + p, :n] = A
    K[:, :n, n:n + p] = A.transpose(1, 2)
    K[:, n + p:, :n] = G
    K[:, :n, n + p:] = G.transpose(1, 2)
    K[:, n + p:, n + p:] = -torch.diag_embed(s / z)
    u = torch.linalg.solve(K, torch.cat([gx, gy, gz], 1))
    ux, uy, uz = u[:, :n], u[:, n:n + p], u[:, n + p:]
    o = lambda a, c: a[:, :, None] * c[:, None, :]          # noqa: E731  batched outer product
    dP = -0.5 * (o(ux, x) + o(x, ux))
    dG = -(o(z, ux) + o(uz, x))
    dA = -(o(y, ux) + o(uy, x))
    return dP, dG, dA, ux, uy, uz


def main():
    import torch
    from torch.profiler import ProfilerActivity
    import cvxopt_b200
    from cvxopt_b200 import QPBatch, _lib
    from batch_coneqp_bench import card
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--shapes", default="config4,layer")
    a = ap.parse_args()
    if cvxopt_b200.device_count() == 0:
        raise SystemExit("batch_adjoint_bench: no GPU visible")
    gpu = card()
    dev = torch.device("cuda", 0)
    for name in a.shapes.split(","):
        B, n, m, p = SHAPES[name]
        P, q, G, h, A, b = problems(B, n, m, p, dev)
        data = [P.transpose(1, 2).contiguous(), q, G.transpose(1, 2).contiguous(), h]
        eq = [A.transpose(1, 2).contiguous(), b] if p else []
        f64 = dict(dtype=torch.float64, device=dev)
        gen = torch.Generator(device=dev).manual_seed(1)
        gx, gy, gz = (torch.randn((B, k), generator=gen, **f64) for k in (n, p, m))
        qb = QPBatch(B, n, m, 0, p=p)
        x, y, s, z = (torch.empty((B, k), **f64) for k in (n, p, m, m))
        outs = [torch.empty(sh, **f64) for sh in ((B, n), (B, p), (B, m), (B, n, n), (B, n, m), (B, n, p))]
        torch.cuda.synchronize()
        qb.load_ptr(*(t.data_ptr() for t in data), _lib.DEVICE, *(t.data_ptr() for t in eq))
        solve_ms, adjoint_ms, torch_ms = [], [], []
        for rep in range(a.reps + 1):                      # rep 0 warms up every path
            qb.solve()
            solve_ms.append(qb.stats()["solve_ms"])
            _lib.check(qb._lib.cvxb_batch_results(qb._h, x.data_ptr(), s.data_ptr(), z.data_ptr(), None, None, None,
                                                  None, _lib.DEVICE), "batch_results")
            if p:
                _lib.check(qb._lib.cvxb_batch_results_y(qb._h, y.data_ptr(), _lib.DEVICE), "batch_results_y")
            t0 = time.perf_counter()
            qb.adjoint_ptr(gx.data_ptr(), gy.data_ptr(), gz.data_ptr(), *(t.data_ptr() for t in outs))
            adjoint_ms.append((time.perf_counter() - t0) * 1e3)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            base = torch_baseline(P, G, A, x, y, s, z, gx, gy, gz)
            e1.record()
            e1.synchronize()
            torch_ms.append(e0.elapsed_time(e1))
        status = np.zeros(B, dtype=np.int32)
        _lib.check(qb._lib.cvxb_batch_results(qb._h, None, None, None, status.ctypes.data, None, None, None,
                                              _lib.HOST), "batch_results")
        ok = torch.from_numpy(status == 1).to(dev)
        ours = (outs[3].transpose(1, 2), outs[4].transpose(1, 2), outs[5].transpose(1, 2), outs[0], outs[1], outs[2])
        diff = max(float(((u - v)[ok].norm() / v[ok].norm().clamp_min(1e-300)).item()) if v.numel() else 0.0
                   for u, v in zip(ours, base))
        del base
        with torch.profiler.profile(activities=[ProfilerActivity.CUDA]) as prof:
            qb.adjoint_ptr(gx.data_ptr(), gy.data_ptr(), gz.data_ptr(), *(t.data_ptr() for t in outs))
            torch.cuda.synchronize()
        grad_ms = sum((getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0))
                      for e in prof.key_averages() if "k_adj_grad" in e.key) / 1e3
        qb.close()
        written = 8 * B * (n * n + m * n + p * n)
        t = lambda v: [round(x, 3) for x in v[1:]]          # noqa: E731  the timed reps
        print(json.dumps({
            "shape": name, "B": B, "n": n, "m": m, "p": p, "card": gpu, "reps": a.reps,
            "status_optimal": int((status == 1).sum()),
            "solve_ms": t(solve_ms), "adjoint_ms": t(adjoint_ms), "adjoint_ms_median": float(np.median(adjoint_ms[1:])),
            "torch_baseline_ms": t(torch_ms), "torch_baseline_ms_median": float(np.median(torch_ms[1:])),
            "grad_kernel_ms": round(grad_ms, 3), "grad_bytes_written": written,
            "grad_kernel_GB_per_s": round(written / (grad_ms * 1e-3) / 1e9, 1) if grad_ms else None,
            "grad_kernel_share_of_3.35TB_per_s": round(written / (grad_ms * 1e-3) / HBM_BYTES_PER_S, 3) if grad_ms
            else None,
            "max_rel_diff_torch_vs_adjoint": diff}), flush=True)
        del P, q, G, h, A, b, data, eq, outs
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
