"""The cone adjoint (cvxb_batch_adjoint_cone) against what users write today in torch, at two layer-sized shapes:
  socp  B = 4096, n = 32, dims {'l': 32, 'q': [4] * 8}   (QPBatch with second-order cones);
  sdp   B = 1024, n = 16, dims {'l': 16, 's': [8]}       (SDPQPBatch with one 's' block).
Seeded QPs are built on the device (P = M M'/n + I, G ~ N(0, 1) with symmetric 's' columns, h = G x0 + s0 with s0
strictly inside the cones), loaded into one batch (nsub = 1) from device memory and solved.  Per rep: the solve's
solve_ms (CUDA events), then adjoint_ms, a host clock around one device-space cvxb_batch_adjoint_cone call with every
output (the call ends in a stream synchronise), then the torch baseline, timed with CUDA events on torch's stream: W'W
built in torch from the returned s and z (diag(s / z), beta² (2 v v' - J)² per 'q' cone, X -> R X R per 's' block with
R = S^{1/2} (S^{1/2} Z S^{1/2})^{-1/2} S^{1/2}), the full KKT matrix in packed coordinates per problem, batched
torch.linalg.solve and the outer products.  After --reps reps, a separate torch.profiler run gives the gradient
kernel's (k_adj_grad) own time.  One JSON line per shape, with the card name and power limit read in the same run and
the largest relative difference of the baseline's gradients from the adjoint's over the optimal problems."""
import argparse
import json
import math
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

SHAPES = {"socp": (4096, 32, {"l": 32, "q": [4] * 8, "s": []}), "sdp": (1024, 16, {"l": 16, "q": [], "s": [8]})}


def cdims(dims):
    """m (unpacked rows) and the packed row count"""
    mlq = dims["l"] + sum(dims["q"])
    return mlq + sum(k * k for k in dims["s"]), mlq + sum(k * (k + 1) // 2 for k in dims["s"])


def pack_ops(dims, **f64):
    """Pk (packed x m): the lower triangle of each 's' block, off-diagonals times sqrt(2) (misc.pack); Uk (m x packed):
    its inverse onto symmetric blocks, both triangles (misc.unpack, mirrored)"""
    import torch
    m, cpk = cdims(dims)
    Pk, Uk = torch.zeros((cpk, m), **f64), torch.zeros((m, cpk), **f64)
    mlq = dims["l"] + sum(dims["q"])
    for i in range(mlq):
        Pk[i, i] = Uk[i, i] = 1.0
    o, op = mlq, mlq
    for k in dims["s"]:
        for j in range(k):
            for i in range(j, k):
                r = op + j * k - j * (j - 1) // 2 + i - j
                if i == j:
                    Pk[r, o + i + j * k] = Uk[o + i + j * k, r] = 1.0
                else:
                    Pk[r, o + i + j * k] = math.sqrt(2.0)
                    Uk[o + i + j * k, r] = Uk[o + j + i * k, r] = math.sqrt(0.5)
        o += k * k
        op += k * (k + 1) // 2
    return Pk, Uk


def transposed(dims, dev):
    """the row permutation that transposes each 's' block of an unpacked vector"""
    import torch
    m, _ = cdims(dims)
    t = list(range(m))
    o = dims["l"] + sum(dims["q"])
    for k in dims["s"]:
        for j in range(k):
            for i in range(k):
                t[o + i + j * k] = o + j + i * k
        o += k * k
    return torch.tensor(t, device=dev)


def problems(B, n, dims, dev, seed=0):
    import torch
    g = torch.Generator(device=dev).manual_seed(seed)
    f64 = dict(dtype=torch.float64, device=dev)
    m, _ = cdims(dims)
    M = torch.randn((B, n, n), generator=g, **f64)
    P = M @ M.transpose(1, 2) / n + torch.eye(n, **f64)
    q = torch.randn((B, n), generator=g, **f64)
    G = torch.randn((B, m, n), generator=g, **f64)
    parts = [0.5 + torch.rand((B, dims["l"]), generator=g, **f64)]
    for k in dims["q"]:
        u = torch.randn((B, k), generator=g, **f64)
        u[:, 0] = u[:, 1:].norm(dim=1) + 0.5 + torch.rand((B,), generator=g, **f64)
        parts.append(u)
    o = dims["l"] + sum(dims["q"])
    for k in dims["s"]:
        Gs = G[:, o:o + k * k, :].reshape(B, k, k, n)
        G[:, o:o + k * k, :] = ((Gs + Gs.transpose(1, 2)) / 2).reshape(B, k * k, n)
        R = torch.randn((B, k, k), generator=g, **f64)
        parts.append((R @ R.transpose(1, 2) / k + torch.eye(k, **f64)).reshape(B, k * k))
        o += k * k
    x0 = torch.randn((B, n, 1), generator=g, **f64)
    h = (G @ x0)[..., 0] + torch.cat(parts, 1)
    return P, q, G, h


def _psd_pow(X, e):
    """X^e of a batch of symmetric positive definite matrices"""
    import torch
    w, V = torch.linalg.eigh(X)
    return (V * w.pow(e)[:, None, :]) @ V.transpose(1, 2)


def wtw(s, z, dims, Pk, Uk):
    """W'W of the NT scaling of s and z in packed coordinates, (B, packed, packed)"""
    import torch
    B = s.shape[0]
    m, cpk = cdims(dims)
    H = torch.zeros((B, cpk, cpk), dtype=s.dtype, device=s.device)
    ml = dims["l"]
    idx = torch.arange(ml, device=s.device)
    H[:, idx, idx] = s[:, :ml] / z[:, :ml]
    o = ml
    for k in dims["q"]:
        sk, zk = s[:, o:o + k], z[:, o:o + k]
        a = (sk[:, 0] ** 2 - (sk[:, 1:] ** 2).sum(1)).sqrt()
        b = (zk[:, 0] ** 2 - (zk[:, 1:] ** 2).sum(1)).sqrt()
        c = (((sk * zk).sum(1) / (a * b) + 1.0) / 2.0).sqrt()
        w = sk / a[:, None]
        w = w + torch.cat([zk[:, :1], -zk[:, 1:]], 1) / b[:, None]
        w = w / (2.0 * c[:, None])
        v = w.clone()
        v[:, 0] += 1.0
        v = v / (2.0 * v[:, :1]).sqrt()
        J = torch.diag(torch.tensor([1.0] + [-1.0] * (k - 1), dtype=s.dtype, device=s.device))
        W = (a / b).sqrt()[:, None, None] * (2.0 * v[:, :, None] * v[:, None, :] - J)
        H[:, o:o + k, o:o + k] = W @ W
        o += k
    op = o
    for k in dims["s"]:
        S, Z = s[:, o:o + k * k].reshape(B, k, k).transpose(1, 2), z[:, o:o + k * k].reshape(B, k, k).transpose(1, 2)
        Sh = _psd_pow(S, 0.5)
        R = Sh @ _psd_pow(Sh @ Z @ Sh, -0.5) @ Sh                  # R Z R = S
        kron = (R[:, :, None, :, None] * R[:, None, :, None, :]).reshape(B, k * k, k * k)   # vec(R X R), col-major
        kp = k * (k + 1) // 2
        H[:, op:op + kp, op:op + kp] = Pk[op:op + kp, o:o + k * k] @ kron @ Uk[o:o + k * k, op:op + kp]
        o += k * k
        op += kp
    return H


def torch_baseline(P, G, x, s, z, gx, gz, dims, Pk, Uk):
    """the dense KKT solve and outer products in torch: (dP, dG, ux, uz)"""
    import torch
    B, n = x.shape
    _, cpk = cdims(dims)
    Gp = Pk @ G
    N = n + cpk
    K = torch.zeros((B, N, N), dtype=P.dtype, device=P.device)
    K[:, :n, :n] = P
    K[:, n:, :n] = Gp
    K[:, :n, n:] = Gp.transpose(1, 2)
    K[:, n:, n:] = -wtw(s, z, dims, Pk, Uk)
    gsym = Pk @ ((gz + gz[:, transposed(dims, gz.device)]) / 2)[..., None]      # pack(sym(gz))
    u = torch.linalg.solve(K, torch.cat([gx[..., None], gsym], 1))[..., 0]
    ux, uz = u[:, :n], (Uk @ u[:, n:, None])[..., 0]
    o = lambda a, c: a[:, :, None] * c[:, None, :]          # noqa: E731  batched outer product
    return -0.5 * (o(ux, x) + o(x, ux)), -(o(z, ux) + o(uz, x)), ux, uz


def main():
    import torch
    from torch.profiler import ProfilerActivity
    import cvxopt_b200
    from cvxopt_b200 import QPBatch, SDPQPBatch, _lib
    from batch_coneqp_bench import card
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--shapes", default="socp,sdp")
    a = ap.parse_args()
    if cvxopt_b200.device_count() == 0:
        raise SystemExit("batch_cone_adjoint_bench: no GPU visible")
    gpu = card()
    dev = torch.device("cuda", 0)
    f64 = dict(dtype=torch.float64, device=dev)
    for name in a.shapes.split(","):
        B, n, dims = SHAPES[name]
        m, _ = cdims(dims)
        P, q, G, h = problems(B, n, dims, dev)
        Pk, Uk = pack_ops(dims, **f64)
        data = [P.transpose(1, 2).contiguous(), q, G.transpose(1, 2).contiguous(), h]
        gen = torch.Generator(device=dev).manual_seed(1)
        gx, gz = (torch.randn((B, k), generator=gen, **f64) for k in (n, m))
        qb = SDPQPBatch(B, n, dims) if dims["s"] else QPBatch(B, n, m, 0, dims=dims)
        x, s, z = (torch.empty((B, k), **f64) for k in (n, m, m))
        outs = [torch.empty(sh, **f64) for sh in ((B, n), (B, m), (B, n, n), (B, n, m))]
        torch.cuda.synchronize()
        qb.load_ptr(*(t.data_ptr() for t in data), _lib.DEVICE)
        solve_ms, adjoint_ms, torch_ms = [], [], []
        for rep in range(a.reps + 1):                      # rep 0 warms up every path
            qb.solve()
            solve_ms.append(qb.stats()["solve_ms"])
            _lib.check(qb._lib.cvxb_batch_results(qb._h, x.data_ptr(), s.data_ptr(), z.data_ptr(), None, None, None,
                                                  None, _lib.DEVICE), "batch_results")
            t0 = time.perf_counter()
            qb.adjoint_cone_ptr(gx.data_ptr(), None, gz.data_ptr(), outs[0].data_ptr(), None, outs[1].data_ptr(),
                                outs[2].data_ptr(), outs[3].data_ptr())
            adjoint_ms.append((time.perf_counter() - t0) * 1e3)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            base = torch_baseline(P, G, x, s, z, gx, gz, dims, Pk, Uk)
            e1.record()
            e1.synchronize()
            torch_ms.append(e0.elapsed_time(e1))
        status = np.zeros(B, dtype=np.int32)
        _lib.check(qb._lib.cvxb_batch_results(qb._h, None, None, None, status.ctypes.data, None, None, None,
                                              _lib.HOST), "batch_results")
        ok = torch.from_numpy(status == 1).to(dev)
        ours = (outs[2].transpose(1, 2), outs[3].transpose(1, 2), outs[0], outs[1])
        diff = max(float(((u - v)[ok].norm() / v[ok].norm().clamp_min(1e-300)).item()) for u, v in zip(ours, base))
        del base
        with torch.profiler.profile(activities=[ProfilerActivity.CUDA]) as prof:
            qb.adjoint_cone_ptr(gx.data_ptr(), None, gz.data_ptr(), outs[0].data_ptr(), None, outs[1].data_ptr(),
                                outs[2].data_ptr(), outs[3].data_ptr())
            torch.cuda.synchronize()
        grad_ms = sum((getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0))
                      for e in prof.key_averages() if "k_adj_grad" in e.key) / 1e3
        qb.close()
        t = lambda v: [round(x, 3) for x in v[1:]]          # noqa: E731  the timed reps
        print(json.dumps({
            "shape": name, "B": B, "n": n, "dims": dims, "m": m, "card": gpu, "reps": a.reps,
            "status_optimal": int((status == 1).sum()),
            "solve_ms": t(solve_ms), "adjoint_ms": t(adjoint_ms), "adjoint_ms_median": float(np.median(adjoint_ms[1:])),
            "torch_baseline_ms": t(torch_ms), "torch_baseline_ms_median": float(np.median(torch_ms[1:])),
            "grad_kernel_ms": round(grad_ms, 3), "grad_bytes_written": 8 * B * (n * n + m * n),
            "max_rel_diff_torch_vs_adjoint": diff}), flush=True)
        del P, q, G, h, data, outs
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
