"""Seeded smooth convex programs for the CP batch tests and tools/batch_cp_bench.py: numpy Generator(PCG64(seed)) only.

Each family is written twice: `torch_F` is the batched F of cp_batch (float64 torch tensors, rows picked by idx), and
`ref_F` the per-problem F of the reference's solvers.cp (cvxopt matrices, evaluated in numpy).  Both return the same
f, Df and H = sum_i z_i grad² f_i; outside dom f the batched F returns non-finite rows and the reference's F None.

    centering  f0 = -sum log x,                                  A x = b             (mnl = 0, dom: x > 0)
    entropy    f0 = sum x log x,                                 A x = b, G x <= h   (mnl = 0, dom: x > 0)
    qcqp       fk = x'Pk x / 2 + qk'x + rk (k = 0..3),           G x <= h            (mnl = 3)
    logistic   f0 = sum_j log(1 + exp(-y_j a_j'x)) + lam/2 |x|², f1 = |x|² - rad²    (mnl = 1)
"""
import numpy as np

FAMILIES = ("centering", "entropy", "qcqp", "logistic")
MNL = {"centering": 0, "entropy": 0, "qcqp": 3, "logistic": 1}
LAM, RAD = 0.1, 1.0


def cp_problem(family, seed, n, p=0, r=0):
    """one problem of `family`, drawn from PCG64(seed) in the order the code below draws: a dict of its data arrays,
    x0 (strictly inside dom f), G (r' x n), h, A (p x n), b.
      centering: A = [1'; N(0, 1) (p - 1 rows)] (the first row keeps {x > 0, A x = b} bounded), b = A xh with
        xh ~ U(0.5, 1.5); x0 ~ U(0.05, 2) (far from A x = b, so that full steps leave x > 0 and the reference backtracks
        into its domain); no G.
      entropy: A = [1'; U(0, 1) (p - 1 rows)], xh ~ U(0.5, 1.5) / n, b = A xh; G ~ N(0, 1) (r x n), h = G xh + U(0.1, 1);
        x0 = 1 / n.
      qcqp: Pk = Mk Mk'/n + 0.1 I with Mk ~ N(0, 1), qk ~ N(0, 1), r0 = 0, rk = -U(0.5, 1.5) (x0 = 0 strictly feasible);
        G = [I; -I; N(0, 1) (r rows)], h = [2 (2n entries); U(0.5, 1.5) (r)].
      logistic: 2n samples a_j ~ N(0, 1) with labels y_j = sign(a_j'w + 0.5 N(0, 1)), w ~ N(0, 1); x0 = 0; no G."""
    rng = np.random.Generator(np.random.PCG64(seed))
    G, h, A, b = np.zeros((0, n)), np.zeros(0), np.zeros((0, n)), np.zeros(0)
    if family == "centering":
        A = np.vstack([np.ones((1, n)), rng.standard_normal((p - 1, n))])
        b = A @ rng.uniform(0.5, 1.5, n)
        data = {}
        x0 = rng.uniform(0.05, 2.0, n)
    elif family == "entropy":
        A = np.vstack([np.ones((1, n)), rng.uniform(0.0, 1.0, (p - 1, n))]) if p else A
        xh = rng.uniform(0.5, 1.5, n) / n
        b = A @ xh
        G = rng.standard_normal((r, n))
        h = G @ xh + rng.uniform(0.1, 1.0, r)
        data = {}
        x0 = np.full(n, 1.0 / n)
    elif family == "qcqp":
        P, q = [], []
        for _ in range(4):
            M = rng.standard_normal((n, n))
            P.append(M @ M.T / n + 0.1 * np.eye(n))
            q.append(rng.standard_normal(n))
        rr = np.concatenate([[0.0], -rng.uniform(0.5, 1.5, 3)])
        G = np.vstack([np.eye(n), -np.eye(n), rng.standard_normal((r, n))])
        h = np.concatenate([np.full(2 * n, 2.0), rng.uniform(0.5, 1.5, r)])
        data = {"P": np.stack(P), "q": np.stack(q), "r": rr}
        x0 = np.zeros(n)
    elif family == "logistic":
        a = rng.standard_normal((2 * n, n))
        w = rng.standard_normal(n)
        y = np.sign(a @ w + 0.5 * rng.standard_normal(2 * n))
        y[y == 0] = 1.0
        data = {"a": a, "y": y}
        x0 = np.zeros(n)
    else:
        raise ValueError(family)
    return {"data": data, "x0": x0, "G": G, "h": h, "A": A, "b": b}


def cp_batch_data(family, seeds, n, p=0, r=0):
    """cp_problem over the seeds, stacked: every array gets a leading batch axis"""
    probs = [cp_problem(family, s, n, p, r) for s in seeds]
    out = {k: np.stack([q[k] for q in probs]) for k in ("x0", "G", "h", "A", "b")}
    out["data"] = {k: np.stack([q["data"][k] for q in probs]) for k in probs[0]["data"]}
    return out


def _softplus(t):
    return np.log1p(np.exp(-np.abs(t))) + np.maximum(t, 0.0)


def _eval_np(family, d, x, z):
    """f, Df and (z given) H of one problem at x, in numpy; None outside dom f"""
    n = x.size
    if family in ("centering", "entropy"):
        if x.min() <= 0.0:
            return None
        lx = np.log(x)
        if family == "centering":
            f, Df, hd = np.array([-lx.sum()]), (-1.0 / x)[None, :], 1.0 / (x * x)
        else:
            f, Df, hd = np.array([x @ lx]), (lx + 1.0)[None, :], 1.0 / x
        return f, Df, None if z is None else np.diag(z[0] * hd)
    if family == "qcqp":
        Px = d["P"] @ x
        f = 0.5 * Px @ x + d["q"] @ x + d["r"]
        Df = Px + d["q"]
        return f, Df, None if z is None else np.tensordot(z, d["P"], 1)
    t = -d["y"] * (d["a"] @ x)
    s = 1.0 / (1.0 + np.exp(-t))                       # sigma(t)
    f = np.array([_softplus(t).sum() + 0.5 * LAM * x @ x, x @ x - RAD * RAD])
    Df = np.vstack([d["a"].T @ (-d["y"] * s) + LAM * x, 2.0 * x])
    if z is None:
        return f, Df, None
    H = z[0] * ((d["a"].T * (s * (1.0 - s))) @ d["a"] + LAM * np.eye(n)) + 2.0 * z[1] * np.eye(n)
    return f, Df, H


def ref_F(family, data, k, x0, calls=None):
    """the reference's F for problem k of cp_batch_data's `data` with starting point x0; calls['none'] counts the
    points it reports outside dom f"""
    from cvxopt import matrix
    d = {key: v[k] for key, v in data.items()}
    mnl = MNL[family]

    def F(x=None, z=None):
        if x is None:
            return mnl, matrix(np.asarray(x0, dtype=np.float64))
        r = _eval_np(family, d, np.array(x).ravel(), None if z is None else np.array(z).ravel())
        if r is None:
            if calls is not None:
                calls["none"] = calls.get("none", 0) + 1
            return None
        f, Df, H = r
        if z is None:
            return matrix(f), matrix(Df)
        return matrix(f), matrix(Df), matrix(H)
    return F


def torch_F(family, data, x0, device=0, seen=None, rowwise=False):
    """cp_batch's F over cp_batch_data's `data` and x0 (B, n); seen['nonfinite'] counts the evaluations that returned
    a non-finite row.  rowwise (qcqp): every sum is accumulated term by term in elementwise operations, so a row's bits
    do not depend on how many rows F is given (a batched matmul's may), and neither do the batch's results under
    compaction"""
    import torch
    dev = torch.device("cuda", device)
    D = {k: torch.as_tensor(v, dtype=torch.float64, device=dev) for k, v in data.items()}
    mnl = MNL[family]

    def F(x=None, z=None, idx=None):
        if x is None:
            return mnl, x0
        k, n = x.shape
        if family in ("centering", "entropy"):
            lx = torch.log(x)
            if family == "centering":
                f, Df, hd = -lx.sum(1, keepdim=True), (-1.0 / x)[:, None, :], 1.0 / (x * x)
            else:
                f, Df, hd = (x * lx).sum(1, keepdim=True), (lx + 1.0)[:, None, :], 1.0 / x
            H = None if z is None else torch.diag_embed(z[:, :1] * hd)
        elif family == "qcqp":
            P, q = D["P"][idx], D["q"][idx]                         # (k, 4, n, n), (k, 4, n)
            if rowwise:
                Px, xPx, qx = 0.0, 0.0, 0.0
                for j in range(n):
                    Px = Px + P[..., j] * x[:, None, None, j]
                for j in range(n):
                    xPx, qx = xPx + Px[..., j] * x[:, None, j], qx + q[..., j] * x[:, None, j]
                f = 0.5 * xPx + qx + D["r"][idx]
            else:
                Px = torch.einsum("kinj,kj->kin", P, x)
                f = 0.5 * (Px * x[:, None, :]).sum(2) + torch.einsum("kin,kn->ki", q, x) + D["r"][idx]
            Df = Px + q
            H = None
            if z is not None:
                H = z[:, 0, None, None] * P[:, 0]
                for i in range(1, 4):
                    H = H + z[:, i, None, None] * P[:, i]
        else:
            a, y = D["a"][idx], D["y"][idx]                          # (k, N, n), (k, N)
            t = -y * torch.einsum("kjn,kn->kj", a, x)
            s = 1.0 / (1.0 + torch.exp(-t))
            sp = torch.log1p(torch.exp(-t.abs())) + t.clamp(min=0.0)
            xx = (x * x).sum(1)
            f = torch.stack([sp.sum(1) + 0.5 * LAM * xx, xx - RAD * RAD], 1)
            Df = torch.stack([torch.einsum("kjn,kj->kn", a, -y * s) + LAM * x, 2.0 * x], 1)
            H = None
            if z is not None:
                eye = torch.eye(n, dtype=x.dtype, device=x.device)
                H = z[:, 0, None, None] * (torch.einsum("kjn,kj,kjm->knm", a, s * (1.0 - s), a) + LAM * eye) \
                    + 2.0 * z[:, 1, None, None] * eye
        if seen is not None and not bool(torch.isfinite(f).all()):
            seen["nonfinite"] = seen.get("nonfinite", 0) + 1
        return (f, Df) if z is None else (f, Df, H)
    return F
