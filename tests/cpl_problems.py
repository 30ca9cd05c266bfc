"""Seeded cpl problems (minimize c'x s.t. f(x) <= 0, G x + s = h with s in 'l' x 'q' cones, A x = b) for the cpl batch
tests and tools/batch_cpl_bench.py: numpy Generator(PCG64(seed)) only.

Each family is written twice: `torch_F` is the batched F of cpl_batch (float64 torch tensors, rows picked by idx), and
`ref_F` the per-problem F of the reference's solvers.cpl (cvxopt matrices, evaluated in numpy).  Both return the same
f, Df and H = sum_i z_i grad² f_i; outside dom f the batched F returns non-finite rows and the reference's F None.

    socp     f1 = |x|² - 4, f2 = x'P x / 2 + q'x - 1 (mnl = 2); 'l' rows G x <= h; cones |A_j x + b_j| <= c_j'x + d_j
    logcone  f1 = -sum log x - r (mnl = 1, dom: x > 0); cones |A_j x + b_j| <= c_j'x + d_j
    conelp   no f (mnl = 0, H = 0); 'l' rows G x <= h; the cone |x| <= 2 and cones |A_j x + b_j| <= c_j'x + d_j
    lsecone  a geometric program in cpl's epigraph form with cones: the variable is (u, t), minimise t s.t.
             lse(F0 u + g0) - t <= 0, lse(Fi u + gi) <= 0 (i = 1, 2; blocks of LSE_K rows), tests/gp_problems.py's box
             and 'l' rows on u, and cones |A_j u + b_j| <= c_j'u + d_j (mnl = 3)
"""
import numpy as np

from gp_problems import gp_problem

FAMILIES = ("socp", "logcone", "conelp", "lsecone")
MNL = {"socp": 2, "logcone": 1, "conelp": 0, "lsecone": 3}
LSE_K = (4, 4, 4)


def _cones(rng, n, q, x):
    """G and h rows of the cones |A_j x + b_j| <= c_j'x + d_j of lengths q: s_j = (c_j'x + d_j, A_j x + b_j) =
    h_j - G_j x, with d_j chosen so that x is strictly inside by U(0.5, 1.5)"""
    G, h = [], []
    for m in q:
        A = rng.standard_normal((m - 1, n)) / np.sqrt(n)
        b = rng.standard_normal(m - 1)
        c = rng.standard_normal(n) / np.sqrt(n)
        d = np.linalg.norm(A @ x + b) - c @ x + rng.uniform(0.5, 1.5)
        G.append(np.vstack([-c[None, :], -A]))
        h.append(np.concatenate([[d], b]))
    return (np.vstack(G), np.concatenate(h)) if q else (np.zeros((0, n)), np.zeros(0))


def cpl_problem(family, seed, n, q, ml=0, p=0):
    """one problem of `family` with cone lengths q, ml 'l' rows and p equality rows, drawn from PCG64(seed) in the
    order the code below draws: a dict of its data arrays, c, x0 (inside dom f), G, h (the 'l' rows, then the cones),
    A, b.  The 'l' rows are G ~ N(0, 1), h = G x + U(0.5, 1.5) at a strictly feasible x (x0, or 1 for logcone); A ~
    N(0, 1) with b = A x at the same x.
      socp: c ~ N(0, 1), P = M M'/n + 0.1 I with M ~ N(0, 1), q ~ N(0, 1) / 4; x0 = 0.
      logcone: c ~ U(0.5, 1.5), r = 1 (so x = 1 is strictly feasible); x0 ~ U(0.05, 2) (in dom f, far from A x = b:
        full steps leave x > 0, and the reference backtracks into its domain).
      conelp: c ~ N(0, 1); the cone (2, x) bounds x; x0 = 0.
      lsecone: n = len(u) + 1; F, g, the box and ml 'l' rows are gp_problem(seed, n - 1, LSE_K, ml)'s, A = 0.1 N(0, 1)
        (p x (n - 1)) and b = 0; the cones are drawn from PCG64(seed) at u = 0; c = e_t and x0 = 0 (cp's start)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    data = {}
    if family == "lsecone":
        F, g, Gl, hl, A, b = gp_problem(seed, n - 1, list(LSE_K), ml, p)
        Gq, hq = _cones(rng, n - 1, q, np.zeros(n - 1))
        G = np.hstack([np.vstack([Gl, Gq]), np.zeros((Gl.shape[0] + Gq.shape[0], 1))])
        return {"data": {"F": F, "g": g}, "c": np.eye(n)[n - 1], "x0": np.zeros(n), "G": G,
                "h": np.concatenate([hl, hq]), "A": np.hstack([A, np.zeros((p, 1))]), "b": b}
    if family == "socp":
        M = rng.standard_normal((n, n))
        data = {"P": M @ M.T / n + 0.1 * np.eye(n), "q": rng.standard_normal(n) / 4}
        c, x0, xf = rng.standard_normal(n), np.zeros(n), np.zeros(n)
    elif family == "logcone":
        data = {"r": np.array([1.0])}
        c, x0, xf = rng.uniform(0.5, 1.5, n), rng.uniform(0.05, 2.0, n), np.ones(n)
    elif family == "conelp":
        c, x0, xf = rng.standard_normal(n), np.zeros(n), np.zeros(n)
    else:
        raise ValueError(family)
    Gl = rng.standard_normal((ml, n))
    hl = Gl @ xf + rng.uniform(0.5, 1.5, ml)
    Gq, hq = _cones(rng, n, q, xf)
    if family == "conelp":
        Gq, hq = np.vstack([np.zeros((1, n)), -np.eye(n), Gq]), np.concatenate([[2.0], np.zeros(n), hq])
    A = rng.standard_normal((p, n))
    return {"data": data, "c": c, "x0": x0, "G": np.vstack([Gl, Gq]), "h": np.concatenate([hl, hq]), "A": A,
            "b": A @ xf}


def cpl_dims(family, n, q, ml=0):
    if family == "lsecone":
        ml += 2 * (n - 1)
    return {"l": ml, "q": ([n + 1] if family == "conelp" else []) + list(q), "s": []}


def cpl_batch_data(family, seeds, n, q, ml=0, p=0):
    """cpl_problem over the seeds, stacked: every array gets a leading batch axis; 'dims' the batch's dims"""
    probs = [cpl_problem(family, s, n, q, ml, p) for s in seeds]
    out = {k: np.stack([pr[k] for pr in probs]) for k in ("c", "x0", "G", "h", "A", "b")}
    out["data"] = {k: np.stack([pr["data"][k] for pr in probs]) for k in probs[0]["data"]}
    out["dims"] = cpl_dims(family, n, q, ml)
    return out


def _eval_np(family, d, x, z):
    """f, Df and (z given) H of one problem at x, in numpy; None outside dom f"""
    n = x.size
    if family == "socp":
        Px = d["P"] @ x
        f = np.array([x @ x - 4.0, 0.5 * Px @ x + d["q"] @ x - 1.0])
        Df = np.vstack([2.0 * x, Px + d["q"]])
        return f, Df, None if z is None else 2.0 * z[0] * np.eye(n) + z[1] * d["P"]
    if family == "lsecone":
        u, f, Df, H, o = x[:-1], np.zeros(3), np.zeros((3, n)), np.zeros((n, n)), 0
        for i, k in enumerate(LSE_K):
            Fi = d["F"][o:o + k]
            y = Fi @ u + d["g"][o:o + k]
            mx = y.max()
            e = np.exp(y - mx)
            w = e / e.sum()
            f[i] = mx + np.log(e.sum())
            Df[i, :-1] = w @ Fi
            if z is not None:
                H[:-1, :-1] += z[i] * (Fi.T @ (np.diag(w) - np.outer(w, w)) @ Fi)
            o += k
        f[0] -= x[-1]
        Df[0, -1] = -1.0
        return f, Df, None if z is None else H
    if family == "logcone":
        if x.min() <= 0.0:
            return None
        f = np.array([-np.log(x).sum() - d["r"][0]])
        return f, (-1.0 / x)[None, :], None if z is None else np.diag(z[0] / (x * x))
    return np.zeros(0), np.zeros((0, n)), None if z is None else np.zeros((n, n))


def ref_F(family, data, k, x0, calls=None):
    """the reference's F for problem k of cpl_batch_data's `data` with starting point x0; calls['none'] counts the
    points it reports outside dom f"""
    from cvxopt import matrix
    d = {key: v[k] for key, v in data.items()}
    mnl = MNL[family]

    def mat(a):
        a = np.asarray(a, dtype=np.float64)
        return matrix(a) if a.size else matrix(0.0, a.shape if a.ndim == 2 else (a.shape[0], 1))

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
            return mat(f), mat(Df)
        return mat(f), mat(Df), mat(H)
    return F


def torch_F(family, data, x0, device=0, seen=None):
    """cpl_batch's F over cpl_batch_data's `data` and x0 (B, n); seen['nonfinite'] counts the evaluations that returned
    a non-finite row"""
    import torch
    dev = torch.device("cuda", device)
    D = {k: torch.as_tensor(v, dtype=torch.float64, device=dev) for k, v in data.items()}
    mnl = MNL[family]

    def F(x=None, z=None, idx=None):
        if x is None:
            return mnl, x0
        k, n = x.shape
        H = None
        if family == "socp":
            P, q = D["P"][idx], D["q"][idx]
            Px = torch.einsum("knj,kj->kn", P, x)
            f = torch.stack([(x * x).sum(1) - 4.0, 0.5 * (Px * x).sum(1) + (q * x).sum(1) - 1.0], 1)
            Df = torch.stack([2.0 * x, Px + q], 1)
            if z is not None:
                eye = torch.eye(n, dtype=x.dtype, device=x.device)
                H = 2.0 * z[:, 0, None, None] * eye + z[:, 1, None, None] * P
        elif family == "lsecone":
            u, Fb, gb = x[:, :-1], D["F"][idx], D["g"][idx]
            fs, Ds, H, o = [], [], (x.new_zeros((k, n, n)) if z is not None else None), 0
            for i, K in enumerate(LSE_K):
                Fi = Fb[:, o:o + K]
                y = torch.einsum("kjn,kn->kj", Fi, u) + gb[:, o:o + K]
                w = torch.softmax(y, 1)
                fs.append(torch.logsumexp(y, 1))
                Ds.append(torch.einsum("kj,kjn->kn", w, Fi))
                if z is not None:
                    M = torch.diag_embed(w) - w[:, :, None] * w[:, None, :]
                    H[:, :-1, :-1] += z[:, i, None, None] * torch.einsum("kjn,kjl,klm->knm", Fi, M, Fi)
                o += K
            f = torch.stack(fs, 1)
            f[:, 0] -= x[:, -1]
            Df = torch.cat([torch.stack(Ds, 1), x.new_zeros((k, 3, 1))], 2)
            Df[:, 0, -1] = -1.0
        elif family == "logcone":
            f = -torch.log(x).sum(1, keepdim=True) - D["r"][idx]
            Df = (-1.0 / x)[:, None, :]
            if z is not None:
                H = torch.diag_embed(z[:, :1] / (x * x))
        else:
            f, Df = x.new_zeros((k, 0)), x.new_zeros((k, 0, n))
            if z is not None:
                H = x.new_zeros((k, n, n))
        if seen is not None and not bool(torch.isfinite(f).all()):
            seen["nonfinite"] = seen.get("nonfinite", 0) + 1
        return (f, Df) if z is None else (f, Df, H)
    return F
