"""The GP batch's adjoint (cvxb_batch_adjoint_gp) against a dense torch baseline, at two shapes of tests/gp_problems.py's
family:
  layer  B = 4096, n = 32,  K = [32] + [8]*4,    r = 16, p = 4  (a layer-sized batch, ml = 2n + r = 80);
  gp256  B = 512,  n = 256, K = [512] + [32]*16, r = 64, p = 8  (tools/batch_gp_bench.py's gp256, ml = 576).
The problems are loaded into one GPBatch (nsub = 1) from device memory and solved.  Per rep: the solve's solve_ms (CUDA
events), then adjoint_ms, a host clock around one device-space cvxb_batch_adjoint_gp call with every output (the call
ends in a stream synchronise), then the torch baseline: the full (n + p + m)^2 KKT matrix per problem at the same
iterate (pi_i = softmax(F_i x + g_i), H = sum z_i F_i' (diag(pi_i) - pi_i pi_i') F_i, Df's rows pi_i' F_i), batched
torch.linalg.solve and the gradient formulas, timed with CUDA events on torch's stream.  After --reps reps, a separate
torch.profiler run gives the gradient kernel's (k_adj_gp_grad) own time and its achieved bytes/s: B (S n + S + ml n +
p n) 8 bytes written (S = sum K; dg counted with it, though k_adj_gp_dg stores it) over its kernel time, against the
3.35 TB/s HBM3 data-sheet bound.  One JSON line per shape, with the card name and power limit read in the same run and
the largest relative difference of the baseline's gradients from the adjoint's."""
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

SHAPES = {"layer": (4096, 32, [32] + [8] * 4, 16, 4), "gp256": (512, 256, [512] + [32] * 16, 64, 8)}  # B, n, K, r, p
HBM_BYTES_PER_S = 3.35e12


def torch_baseline(K, F, g, G, A, x, y, s, z, gx, gy, gz):
    """the dense KKT solve and the gradient formulas in torch: (dF, dg, dG, dA, uy, uzl)"""
    import torch
    B, S, n = F.shape
    mnl, m, p = len(K) - 1, s.shape[1], y.shape[1]
    N = n + p + m
    one = torch.ones((B, 1), dtype=F.dtype, device=F.device)
    zk = torch.cat([one, z[:, :mnl]], 1)
    u = torch.bmm(F, x[:, :, None])[..., 0] + g
    H = torch.zeros((B, n, n), dtype=F.dtype, device=F.device)
    pis, Df, o = [], [], 0
    for i, k in enumerate(K):
        Fi = F[:, o:o + k]
        pi = torch.softmax(u[:, o:o + k], 1)
        d = (Fi.transpose(1, 2) @ pi[:, :, None])[..., 0]                  # F_i' pi_i
        H += zk[:, i, None, None] * (Fi.transpose(1, 2) @ (pi[:, :, None] * Fi) - d[:, :, None] * d[:, None, :])
        pis.append(pi)
        if i:
            Df.append(d[:, None, :])
        o += k
    Gf = torch.cat(Df + [G], 1)
    KK = torch.zeros((B, N, N), dtype=F.dtype, device=F.device)
    KK[:, :n, :n] = H
    KK[:, n:n + p, :n] = A
    KK[:, :n, n:n + p] = A.transpose(1, 2)
    KK[:, n + p:, :n] = Gf
    KK[:, :n, n + p:] = Gf.transpose(1, 2)
    KK[:, n + p:, n + p:] = -torch.diag_embed(s / z)
    sol = torch.linalg.solve(KK, torch.cat([gx, gy, gz], 1))
    ux, uy, uz = sol[:, :n], sol[:, n:n + p], sol[:, n + p:]
    uk = torch.cat([0 * one, uz[:, :mnl]], 1)
    w = torch.bmm(F, ux[:, :, None])[..., 0]
    dg, hp, o = [], [], 0
    for i, k in enumerate(K):
        pi, wi = pis[i], w[:, o:o + k]
        dg.append(-(zk[:, i, None] * pi * (wi - (pi * wi).sum(1, keepdim=True)) + uk[:, i, None] * pi))
        hp.append(zk[:, i, None] * pi)
        o += k
    dg, hp = torch.cat(dg, 1), torch.cat(hp, 1)
    out = lambda a, c: a[:, :, None] * c[:, None, :]          # noqa: E731  batched outer product
    dF = out(dg, x) - out(hp, ux)
    dG = -(out(z[:, mnl:], ux) + out(uz[:, mnl:], x))
    dA = -(out(y, ux) + out(uy, x))
    return dF, dg, dG, dA, uy, uz[:, mnl:]


def main():
    import torch
    from torch.profiler import ProfilerActivity
    import cvxopt_b200
    from cvxopt_b200 import GPBatch, _lib
    from batch_coneqp_bench import card
    from gp_problems import gp_batch_data
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--shapes", default="layer,gp256")
    a = ap.parse_args()
    if cvxopt_b200.device_count() == 0:
        raise SystemExit("batch_gp_adjoint_bench: no GPU visible")
    gpu = card()
    dev = torch.device("cuda", 0)
    f64 = dict(dtype=torch.float64, device=dev)
    for name in a.shapes.split(","):
        B, n, K, r, p = SHAPES[name]
        F, g, G, h, A, b = (torch.from_numpy(v).to(dev) for v in gp_batch_data(range(B), n, K, r, p))
        S, ml, mnl = sum(K), G.shape[1], len(K) - 1
        m = mnl + ml
        data = [F.transpose(1, 2).contiguous(), g, G.transpose(1, 2).contiguous(), h]
        eq = [A.transpose(1, 2).contiguous(), b]
        gen = torch.Generator(device=dev).manual_seed(1)
        gx, gy, gz = (torch.randn((B, k), generator=gen, **f64) for k in (n, p, m))
        gb = GPBatch(B, n, K, ml, p, 0)
        x, y, s, z = (torch.empty((B, k), **f64) for k in (n, p, m, m))
        outs = [torch.empty(sh, **f64) for sh in ((B, n), (B, p), (B, m), (B, n, S), (B, S), (B, n, ml), (B, n, p))]
        torch.cuda.synchronize()
        gb.load_ptr(*(t.data_ptr() for t in data), _lib.DEVICE, *(t.data_ptr() for t in eq))
        solve_ms, adjoint_ms, torch_ms = [], [], []
        for rep in range(a.reps + 1):                      # rep 0 warms up every path
            gb.solve()
            solve_ms.append(gb.stats()["solve_ms"])
            _lib.check(gb._lib.cvxb_batch_results(gb._h, x.data_ptr(), s.data_ptr(), z.data_ptr(), None, None, None,
                                                  None, _lib.DEVICE), "batch_results")
            _lib.check(gb._lib.cvxb_batch_results_y(gb._h, y.data_ptr(), _lib.DEVICE), "batch_results_y")
            t0 = time.perf_counter()
            gb.adjoint_gp_ptr(gx.data_ptr(), gy.data_ptr(), gz.data_ptr(), *(t.data_ptr() for t in outs))
            adjoint_ms.append((time.perf_counter() - t0) * 1e3)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            base = torch_baseline(K, F, g, G, A, x, y, s, z, gx, gy, gz)
            e1.record()
            e1.synchronize()
            torch_ms.append(e0.elapsed_time(e1))
        status = np.zeros(B, dtype=np.int32)
        _lib.check(gb._lib.cvxb_batch_results(gb._h, None, None, None, status.ctypes.data, None, None, None,
                                              _lib.HOST), "batch_results")
        ok = torch.from_numpy(status == 1).to(dev)
        ours = (outs[3].transpose(1, 2), outs[4], outs[5].transpose(1, 2), outs[6].transpose(1, 2), outs[1],
                outs[2][:, mnl:])
        diff = max(float(((u - v)[ok].norm() / v[ok].norm().clamp_min(1e-300)).item()) if v.numel() else 0.0
                   for u, v in zip(ours, base))
        del base
        with torch.profiler.profile(activities=[ProfilerActivity.CUDA]) as prof:
            gb.adjoint_gp_ptr(gx.data_ptr(), gy.data_ptr(), gz.data_ptr(), *(t.data_ptr() for t in outs))
            torch.cuda.synchronize()
        grad_ms = sum((getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0))
                      for e in prof.key_averages() if "k_adj_gp_grad" in e.key) / 1e3
        gb.close()
        written = 8 * B * (S * n + S + ml * n + p * n)
        t = lambda v: [round(x, 3) for x in v[1:]]          # noqa: E731  the timed reps
        print(json.dumps({
            "shape": name, "B": B, "n": n, "K": [K[0], "%dx%d" % (mnl, K[1])], "ml": ml, "p": p, "card": gpu,
            "reps": a.reps, "status_optimal": int((status == 1).sum()),
            "solve_ms": t(solve_ms), "adjoint_ms": t(adjoint_ms), "adjoint_ms_median": float(np.median(adjoint_ms[1:])),
            "torch_baseline_ms": t(torch_ms), "torch_baseline_ms_median": float(np.median(torch_ms[1:])),
            "grad_kernel_ms": round(grad_ms, 3), "grad_bytes_written": written,
            "grad_kernel_GB_per_s": round(written / (grad_ms * 1e-3) / 1e9, 1) if grad_ms else None,
            "grad_kernel_share_of_3.35TB_per_s": round(written / (grad_ms * 1e-3) / HBM_BYTES_PER_S, 3) if grad_ms
            else None,
            "max_rel_diff_torch_vs_adjoint": diff}), flush=True)
        del F, g, G, h, A, b, data, eq, outs
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
