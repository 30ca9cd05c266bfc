"""The CP and cpl batches' adjoint (cvxb_batch_adjoint_cp) against a dense torch baseline, at four shapes:
  logistic4096  B = 4096, n = 32, tests/cp_problems.py's logistic family (mnl = 1, ml = 0, p = 0): a layer-sized batch;
  qcqp64        B = 512,  n = 64, the qcqp family, r = 16 (tools/batch_cp_bench.py's qcqp64, mnl = 3, ml = 144);
  entropy256    B = 512,  n = 256, the entropy family, p = 8, r = 32 (batch_cp_bench.py's entropy256, mnl = 0);
  socp64        B = 512,  n = 64, tests/cpl_problems.py's socp, q = [3, 8, 16, 33], ml = 16, p = 4 (batch_cpl_bench's).
The problems are loaded into one CPBatch or CPLBatch (nsub = 1) from device memory and solved.  Per rep: the solve's
solve_ms, then adjoint_ms, a host clock around one device-space cvxb_batch_adjoint_cp call with every output (the call
ends in a stream synchronise), of which f_ms is the caller's F(x, z) inside it (CUDA events around the callback on the
batch's stream: not the library's time), then the torch baseline at the same iterate: H and Df from the same F, the
full (n + p + m)^2 KKT matrix per problem (socp64's cone rows with W'W = beta^2 (2 w w' - J) per 'q' cone), batched
torch.linalg.solve and the gradient formulas, timed with CUDA events on torch's stream (its F call included).  One JSON
line per shape, with the card name and power limit read in the same run and, over the optimal problems whose adjoint is
finite, each problem's relative difference from the baseline (the largest over the outputs of ||adjoint - baseline|| /
||baseline||): its maximum and median and the number of problems above 1e-6, and the number of optimal problems whose
adjoint is NaN."""
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

SHAPES = {  # kind, family, B, n, p, r (cp) or q, ml (cpl)
    "logistic4096": ("cp", "logistic", 4096, 32, 0, 0, None),
    "qcqp64": ("cp", "qcqp", 512, 64, 0, 16, None),
    "entropy256": ("cp", "entropy", 512, 256, 8, 32, None),
    "socp64": ("cpl", "socp", 512, 64, 4, 16, [3, 8, 16, 33]),
}


def soc_ww(s, z):
    """W'W = beta^2 (2 w w' - J) of the NT scaling of one 'q' cone's s and z, batched: (B, k, k)"""
    import torch
    J = torch.ones(s.shape[1], dtype=s.dtype, device=s.device)
    J[1:] = -1.0
    a = torch.sqrt((s * s * J).sum(1))
    b = torch.sqrt((z * z * J).sum(1))
    sb, zb = s / a[:, None], z / b[:, None]
    c = torch.sqrt((1.0 + (sb * zb).sum(1)) / 2.0)
    w = (sb + J * zb) / (2.0 * c[:, None])
    return (a / b)[:, None, None] * (2.0 * w[:, :, None] * w[:, None, :] - torch.diag(J))


def torch_baseline(F, epi, c, G, A, dims, x, y, s, z, gx, gy, gz):
    """H and Df from F at x, the dense KKT solve and the gradient formulas in torch: (ux, uy, uz, dG, dA)"""
    import torch
    B, n = x.shape
    p, m, mnl = y.shape[1], s.shape[1], s.shape[1] - G.shape[1]
    N = n + p + m
    zk = torch.cat([torch.ones((B, 1), dtype=x.dtype, device=x.device), z[:, :mnl]], 1) if epi else z[:, :mnl]
    _, Df, H = F(x, zk, idx=torch.arange(B, device=x.device))
    H = torch.tril(H) + torch.tril(H, -1).transpose(1, 2)
    Gf = torch.cat([Df[:, 1:] if epi else Df, G], 1)
    KK = torch.zeros((B, N, N), dtype=x.dtype, device=x.device)
    KK[:, :n, :n] = H
    KK[:, n:n + p, :n] = A
    KK[:, :n, n:n + p] = A.transpose(1, 2)
    KK[:, n + p:, :n] = Gf
    KK[:, :n, n + p:] = Gf.transpose(1, 2)
    lrows = mnl + dims["l"]
    KK[:, n + p:n + p + lrows, n + p:n + p + lrows] = -torch.diag_embed(s[:, :lrows] / z[:, :lrows])
    o = n + p + lrows
    for k in dims["q"]:
        KK[:, o:o + k, o:o + k] = -soc_ww(s[:, o - n - p:o - n - p + k], z[:, o - n - p:o - n - p + k])
        o += k
    sol = torch.linalg.solve(KK, torch.cat([gx, gy, gz], 1))
    ux, uy, uz = sol[:, :n], sol[:, n:n + p], sol[:, n + p:]
    out = lambda a, b: a[:, :, None] * b[:, None, :]          # noqa: E731  batched outer product
    dG = -(out(z[:, mnl:], ux) + out(uz[:, mnl:], x))
    dA = -(out(y, ux) + out(uy, x))
    return ux, uy, uz, dG, dA


def main():
    import torch
    import cvxopt_b200
    import cp_problems as cpp
    import cpl_problems as cplp
    from cvxopt_b200 import CPBatch, CPLBatch, _lib
    from batch_coneqp_bench import card
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    a = ap.parse_args()
    if cvxopt_b200.device_count() == 0:
        raise SystemExit("batch_cp_adjoint_bench: no GPU visible")
    gpu = card()
    dev = torch.device("cuda", 0)
    f64 = dict(dtype=torch.float64, device=dev)
    for name in a.shapes.split(","):
        kind, family, B, n, p, r, q = SHAPES[name]
        epi = kind == "cp"
        if epi:
            d = cpp.cp_batch_data(family, range(B), n, p, r)
            mnl, dims = cpp.MNL[family], {"l": d["G"].shape[1], "q": []}
            F0 = cpp.torch_F(family, d["data"], d["x0"])
        else:
            d = cplp.cpl_batch_data(family, range(B), n, q, r, p)
            mnl, dims = cplp.MNL[family], dict(d["dims"])
            F0 = cplp.torch_F(family, d["data"], d["x0"])
        ml = d["G"].shape[1]
        m = mnl + ml
        f_ms, events = [], []

        def F(x=None, z=None, idx=None):            # CUDA events around each evaluation on the calling stream
            if x is None:
                return F0()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = F0(x, z, idx=idx)
            e1.record()
            events.append((e0, e1))
            return out
        t = {k: torch.from_numpy(np.ascontiguousarray(d[k])).to(dev) for k in ("x0", "G", "h", "A", "b", "c")
             if k in d}
        Gcm, Acm = t["G"].transpose(1, 2).contiguous(), t["A"].transpose(1, 2).contiguous()
        gen = torch.Generator(device=dev).manual_seed(1)
        gx, gy, gz = (torch.randn((B, k), generator=gen, **f64) for k in (n, p, m))
        bt = CPBatch(B, n, mnl, ml, p, 0) if epi else CPLBatch(B, n, mnl, {**dims, "s": []}, p, 0)
        bt.set_F(F)
        x, y, s, z = (torch.empty((B, k), **f64) for k in (n, p, m, m))
        outs = [torch.empty(sh, **f64) for sh in ((B, n), (B, p), (B, m), (B, n, ml), (B, n, p))]
        torch.cuda.synchronize()
        G_, h_ = (Gcm.data_ptr(), t["h"].data_ptr()) if ml else (None, None)
        A_, b_ = (Acm.data_ptr(), t["b"].data_ptr()) if p else (None, None)
        if epi:
            bt.load_ptr(t["x0"].data_ptr(), G_, h_, _lib.DEVICE, A_, b_)
        else:
            bt.load_ptr(t["c"].data_ptr(), t["x0"].data_ptr(), G_, h_, _lib.DEVICE, A_, b_)
        solve_ms, adjoint_ms, torch_ms = [], [], []
        for rep in range(a.reps + 1):                      # rep 0 warms up every path
            bt.solve()
            solve_ms.append(bt.stats()["solve_ms"])
            _lib.check(bt._lib.cvxb_batch_results(bt._h, x.data_ptr(), s.data_ptr(), z.data_ptr(), None, None, None,
                                                  None, _lib.DEVICE), "batch_results")
            if p:
                _lib.check(bt._lib.cvxb_batch_results_y(bt._h, y.data_ptr(), _lib.DEVICE), "batch_results_y")
            events.clear()
            t0 = time.perf_counter()
            bt.adjoint_cp_ptr(gx.data_ptr(), gy.data_ptr(), gz.data_ptr(), *(o.data_ptr() for o in outs))
            adjoint_ms.append((time.perf_counter() - t0) * 1e3)
            f_ms.append(sum(e0.elapsed_time(e1) for e0, e1 in events))
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            base = torch_baseline(F0, epi, t.get("c"), t["G"], t["A"], dims, x, y, s, z, gx, gy, gz)
            e1.record()
            e1.synchronize()
            torch_ms.append(e0.elapsed_time(e1))
        status = np.zeros(B, dtype=np.int32)
        _lib.check(bt._lib.cvxb_batch_results(bt._h, None, None, None, status.ctypes.data, None, None, None,
                                              _lib.HOST), "batch_results")
        bt.close()
        ok = torch.from_numpy(status == 1).to(dev)
        ours = (outs[0], outs[1], outs[2], outs[3].transpose(1, 2), outs[4].transpose(1, 2))
        # problems whose adjoint factorisation failed get NaN (and the baseline may not be finite there either)
        fin = ok & torch.isfinite(ours[0]).all(1) & torch.isfinite(base[0]).all(1)
        # per problem: the largest over the outputs of ||ours - baseline|| / ||baseline||, each output flattened
        per = torch.zeros(B, **f64)
        for u, v in zip(ours, base):
            if v.numel():
                u2, v2 = u.reshape(B, -1), v.reshape(B, -1)
                per = torch.maximum(per, (u2 - v2).norm(dim=1) / v2.norm(dim=1).clamp_min(1e-300))
        per = per[fin].cpu().numpy()
        nonfinite = int((ok & ~torch.isfinite(ours[0]).all(1)).sum())
        del base
        tr = lambda v: [round(float(e), 3) for e in v[1:]]          # noqa: E731  the timed reps
        print(json.dumps({
            "shape": name, "family": family, "B": B, "n": n, "mnl": mnl, "ml": ml, "q": dims["q"], "p": p,
            "card": gpu, "reps": a.reps, "status_optimal": int((status == 1).sum()),
            "solve_ms": tr(solve_ms), "adjoint_ms": tr(adjoint_ms), "adjoint_ms_median": float(np.median(adjoint_ms[1:])),
            "f_ms_in_adjoint": tr(f_ms), "adjoint_minus_f_ms_median":
                float(np.median(np.array(adjoint_ms[1:]) - np.array(f_ms[1:]))),
            "torch_baseline_ms": tr(torch_ms), "torch_baseline_ms_median": float(np.median(torch_ms[1:])),
            "per_problem_rel_diff_max": float(per.max()) if per.size else None,
            "per_problem_rel_diff_median": float(np.median(per)) if per.size else None,
            "problems_rel_diff_above_1e-6": int((per > 1e-6).sum()), "optimal_with_nan_adjoint": nonfinite}),
            flush=True)
        del t, Gcm, Acm, outs
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
