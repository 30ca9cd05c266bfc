"""The batch tangents (cvxb_batch_tangent, _qcqp, _gp) next to the solve and the adjoint, at the adjoint benches' layer
shapes:
  qp      B = 8192, n = 32, m = 64, p = 8      (batch_adjoint_bench's layer; problems from its generator)
  socp    B = 4096, n = 32, 'l' 32, 8 x 'q' 4  (batch_cone_adjoint_bench's)
  sdp     B = 1024, n = 16, 'l' 16, 's' [8]    (batch_cone_adjoint_bench's)
  qcqp    B = 4096, n = 32, mnl = 4, p = 4     (batch_qcqp_adjoint_bench's layer)
  gp      B = 4096, n = 32, K = [32, 8 x 4]    (batch_gp_adjoint_bench's layer)
Per rep: the solve's solve_ms (CUDA events); adjoint_ms, a host clock around one device-space adjoint call with ux, uy
and uz only; tangent_ms, a host clock around one device-space tangent call along a seeded direction in every data
array (both calls end in a stream synchronise).  A separate torch.profiler run gives the right-hand-side kernel's
(k_tan_rhs*) own time, and its bytes read (the direction, x, y, z; the GP kernel also reads the batch's F twice and
g) over that time against the 3.35 TB/s HBM3 data-sheet bound.  On the qp shape a torch baseline builds the full
(n + p + m)^2 KKT matrix per problem at the same iterate and runs batched torch.linalg.solve on the tangent's
right-hand side formed in torch; the largest relative difference from the tangent is reported.  One JSON line per
shape, with the card name and power limit read in the same run."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

SHAPES = ("qp", "socp", "sdp", "qcqp", "gp")
HBM_BYTES_PER_S = 3.35e12


def _build(name, dev):
    """-> batch, widths (n, p, m), direction (device tensors in the library's layouts), tangent(outs) and
    adjoint(g, outs) calls, the bytes the RHS kernel reads, and for the qp shape the torch baseline's inputs"""
    import torch
    from cvxopt_b200 import GPBatch, QCQPBatch, QPBatch, SDPQPBatch, _lib
    f64 = dict(dtype=torch.float64, device=dev)
    gen = torch.Generator(device=dev).manual_seed(2)
    rnd = lambda *s: torch.randn(s, generator=gen, **f64)          # noqa: E731
    base = None
    if name == "qp":
        import batch_adjoint_bench as qa
        B, n, m, p = qa.SHAPES["layer"]
        P, q, G, h, A, b = qa.problems(B, n, m, p, dev)
        bt = QPBatch(B, n, m, 0, p=p)
        torch.cuda.synchronize()
        bt.load_ptr(P.transpose(1, 2).contiguous().data_ptr(), q.data_ptr(), G.transpose(1, 2).contiguous().data_ptr(),
                    h.data_ptr(), _lib.DEVICE, A.transpose(1, 2).contiguous().data_ptr(), b.data_ptr())
        d = [rnd(B, n, n), rnd(B, n), rnd(B, m, n), rnd(B, m), rnd(B, p, n), rnd(B, p)]
        lay = [d[0].transpose(1, 2).contiguous(), d[1], d[2].transpose(1, 2).contiguous(), d[3],
               d[4].transpose(1, 2).contiguous(), d[5]]
        tan, adj, widths = bt.tangent_ptr, bt.adjoint_cone_ptr, (n, p, m)
        base = (P, G, A, d)
    elif name in ("socp", "sdp"):
        import batch_cone_adjoint_bench as ca
        B, n, dims = ca.SHAPES[name]
        m, _ = ca.cdims(dims)
        P, q, G, h = ca.problems(B, n, dims, dev)
        bt = SDPQPBatch(B, n, dims) if dims["s"] else QPBatch(B, n, m, 0, dims=dims)
        data = [P.transpose(1, 2).contiguous(), q, G.transpose(1, 2).contiguous(), h]
        torch.cuda.synchronize()
        bt.load_ptr(*(t.data_ptr() for t in data), _lib.DEVICE)
        lay = [rnd(B, n, n), rnd(B, n), rnd(B, n, m), rnd(B, m), None, None]
        tan, adj, widths = bt.tangent_ptr, bt.adjoint_cone_ptr, (n, 0, m)
    elif name == "qcqp":
        import batch_qcqp_adjoint_bench as qq
        from qcqp_problems import qcqp_batch_data
        B, n, mnl, p, r = qq.SHAPES["layer"]
        dd = qcqp_batch_data(range(B), n, mnl, p, r)
        nK, ml = mnl + 1, dd["G"].shape[1]
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)   # noqa: E731
        bt = QCQPBatch(B, n, mnl, ml, p, 0)
        data = [t(np.transpose(dd["P"], (0, 3, 1, 2))), t(dd["q"]), t(dd["r"]), t(dd["x0"]),
                t(np.transpose(dd["G"], (0, 2, 1))), t(dd["h"])]
        eq = [t(np.transpose(dd["A"], (0, 2, 1))), t(dd["b"])]
        torch.cuda.synchronize()
        bt.load_ptr(*(a.data_ptr() for a in data), _lib.DEVICE, *(a.data_ptr() for a in eq))
        lay = [rnd(B, n, nK, n), rnd(B, nK, n), rnd(B, nK), rnd(B, n, ml), rnd(B, ml), rnd(B, n, p), rnd(B, p)]
        tan, adj, widths = bt.tangent_ptr, bt.adjoint_ptr, (n, p, mnl + ml)
    else:
        import batch_gp_adjoint_bench as ga
        from gp_problems import gp_batch_data
        B, n, K, r, p = ga.SHAPES["layer"]
        F, g, G, h, A, b = (torch.from_numpy(v).to(dev) for v in gp_batch_data(range(B), n, K, r, p))
        S, ml, mnl = sum(K), G.shape[1], len(K) - 1
        bt = GPBatch(B, n, K, ml, p, 0)
        data = [F.transpose(1, 2).contiguous(), g, G.transpose(1, 2).contiguous(), h]
        eq = [A.transpose(1, 2).contiguous(), b]
        torch.cuda.synchronize()
        bt.load_ptr(*(a.data_ptr() for a in data), _lib.DEVICE, *(a.data_ptr() for a in eq))
        lay = [rnd(B, n, S), rnd(B, S), rnd(B, n, ml), rnd(B, ml), rnd(B, n, p), rnd(B, p)]
        tan, adj, widths = bt.tangent_gp_ptr, bt.adjoint_gp_ptr, (n, p, mnl + ml)
    n, p, m = widths
    read = 8 * sum(a.numel() for a in lay if a is not None) + 8 * bt.B * (n + p + m)
    if name == "gp":
        read += 8 * bt.B * (2 * sum(K) * n + sum(K))
    ptrs = [None if a is None else a.data_ptr() for a in lay]

    def tangent(outs):
        tan(*ptrs, *(o.data_ptr() if o.numel() else None for o in outs))

    def adjoint(gs, outs):
        adj(*(v.data_ptr() if v.numel() else None for v in gs), *(o.data_ptr() if o.numel() else None for o in outs))
    return bt, widths, tangent, adjoint, read, base, lay


def torch_baseline(P, G, A, d, x, y, s, z):
    """the tangent in torch: the full KKT matrix at the iterate, r formed in torch, batched torch.linalg.solve"""
    import torch
    dP, dq, dG, dh, dA, db = d
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
    mv = lambda M, v: (M @ v[..., None])[..., 0]                     # noqa: E731
    mtv = lambda M, v: (M.transpose(1, 2) @ v[..., None])[..., 0]    # noqa: E731
    rx = -(0.5 * (mv(dP, x) + mtv(dP, x)) + dq + mtv(dA, y) + mtv(dG, z))
    u = torch.linalg.solve(K, torch.cat([rx, db - mv(dA, x), dh - mv(dG, x)], 1))
    return u[:, :n], u[:, n:n + p], u[:, n + p:]


def main():
    import torch
    from torch.profiler import ProfilerActivity
    import cvxopt_b200
    from cvxopt_b200 import _lib
    from batch_coneqp_bench import card
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    a = ap.parse_args()
    if cvxopt_b200.device_count() == 0:
        raise SystemExit("batch_tangent_bench: no GPU visible")
    gpu = card()
    dev = torch.device("cuda", 0)
    f64 = dict(dtype=torch.float64, device=dev)
    for name in a.shapes.split(","):
        bt, (n, p, m), tangent, adjoint, read, base, keep = _build(name, dev)
        B = bt.B
        gen = torch.Generator(device=dev).manual_seed(1)
        gs = [torch.randn((B, k), generator=gen, **f64) for k in (n, p, m)]
        touts = [torch.empty((B, k), **f64) for k in (n, p, m)]
        aouts = [torch.empty((B, k), **f64) for k in (n, p, m)]
        solve_ms, adjoint_ms, tangent_ms = [], [], []
        for rep in range(a.reps + 1):                      # rep 0 warms up every path
            bt.solve()
            solve_ms.append(bt.stats()["solve_ms"])
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            adjoint(gs, aouts)
            adjoint_ms.append((time.perf_counter() - t0) * 1e3)
            t0 = time.perf_counter()
            tangent(touts)
            tangent_ms.append((time.perf_counter() - t0) * 1e3)
        status = np.zeros(B, dtype=np.int32)
        _lib.check(bt._lib.cvxb_batch_results(bt._h, None, None, None, status.ctypes.data, None, None, None,
                                              _lib.HOST), "batch_results")
        diff = torch_ms = None
        if base is not None:
            x, y, s, z = (torch.empty((B, k), **f64) for k in (n, p, m, m))
            _lib.check(bt._lib.cvxb_batch_results(bt._h, x.data_ptr(), s.data_ptr(), z.data_ptr(), None, None, None,
                                                  None, _lib.DEVICE), "batch_results")
            _lib.check(bt._lib.cvxb_batch_results_y(bt._h, y.data_ptr(), _lib.DEVICE), "batch_results_y")
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            want = torch_baseline(*base, x, y, s, z)
            e1.record()
            e1.synchronize()
            torch_ms = e0.elapsed_time(e1)
            ok = torch.from_numpy(status == 1).to(dev)
            diff = max(float(((u - v)[ok].norm() / v[ok].norm().clamp_min(1e-300)).item()) if v.numel() else 0.0
                       for u, v in zip(touts, want))
            del want
        with torch.profiler.profile(activities=[ProfilerActivity.CUDA]) as prof:
            tangent(touts)
            torch.cuda.synchronize()
        rhs_ms = sum((getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0))
                     for e in prof.key_averages() if "k_tan_rhs" in e.key) / 1e3
        bt.close()
        t = lambda v: [round(x, 3) for x in v[1:]]          # noqa: E731  the timed reps
        print(json.dumps({
            "shape": name, "B": B, "n": n, "p": p, "m": m, "card": gpu, "reps": a.reps,
            "status_optimal": int((status == 1).sum()), "solve_ms": t(solve_ms),
            "adjoint_ms": t(adjoint_ms), "adjoint_ms_median": float(np.median(adjoint_ms[1:])),
            "tangent_ms": t(tangent_ms), "tangent_ms_median": float(np.median(tangent_ms[1:])),
            "rhs_kernel_ms": round(rhs_ms, 4), "rhs_bytes_read": read,
            "rhs_kernel_GB_per_s": round(read / (rhs_ms * 1e-3) / 1e9, 1) if rhs_ms else None,
            "rhs_kernel_share_of_3.35TB_per_s": round(read / (rhs_ms * 1e-3) / HBM_BYTES_PER_S, 3) if rhs_ms else None,
            "torch_baseline_ms": torch_ms, "max_rel_diff_torch_vs_tangent": diff}), flush=True)
        del keep, base
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
