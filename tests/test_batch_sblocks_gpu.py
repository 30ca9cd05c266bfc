"""The batch solver's semidefinite ('s') block kernels, block by block, against long double (tests/ld_check.py).

cvxb_sblock_batched launches the solver's own k_s_nt_compute, k_s_update, k_s_dir_post, k_s_eig_start, k_s_eig_warm,
k_s_build_gs, k_s_wtz and k_s_res on blocks laid out as in the solver.  Every kernel is checked
- on every order 1..32 (one problem holding all 32 blocks) and on problems of mixed blocks [1, 32, 5, 17, 32, 2];
- on batches of 1, 3 and 257 problems, sampled at the first, second, middle and last problem, and once at
  CVXB_BATCH_MAX problems of order 2;
- with NaN in everything a kernel must neither read nor write (the gap after each problem, other operands' rows, the
  strict upper triangle of every input it reads as a lower triangle), which has to come back bit for bit;
- for cross-talk (a problem in slot j gives the bits it gives in slot 0 of a batch of two), determinism (a second
  run gives the same bits) and exact symmetry where the solver relies on it;
- on the inputs where Jacobi and the NT algebra go wrong: late interior-point iterates (kappa(s), kappa(z) ~ 1e8,
  lambda clustered at sqrt(mu)), diagonal blocks (no rotation), identity and clusters a few ulps wide, rank one plus
  identity, indefinite directions.
Every check prints its largest error / bound."""
import ctypes

import numpy as np
import pytest

from ld_check import (LD, check_congruence, check_min_eig, check_nt_scaling, check_nt_update, check_sums,
                      check_sym_eig, pack_ld, sym_lower, unpack)

pytestmark = pytest.mark.gpu

BATCH_MAX = 65535
MIXED = [1, 32, 5, 17, 32, 2]
ALL = list(range(1, 33))
GAP = 5
M_OPS = ("s", "z", "ds", "dz", "h", "lmbda", "lmbdasq", "d", "di", "bzp", "th", "ws3")
L_OPS = ("r", "rti", "sigs", "sigz", "wz", "ws", "wz2", "ws2", "wz3")
FAMILIES = ["spd", "late", "diag", "cluster", "rank1"]


def _lib():
    from cvxopt_b200 import _lib as L
    return L, L.load()


def _samples(batch):
    return sorted({0, 1, batch // 2, batch - 1} & set(range(batch)))


class Layout:
    """the solver's 's' layout of `orders` without 'l' / 'q' rows, GAP NaN rows after each problem"""

    def __init__(self, orders, batch, n=1):
        self.orders, self.batch, self.n = list(orders), batch, n
        self.so, self.sp, self.sg = [], [], []
        so = sp = sg = 0
        for k in self.orders:
            self.so.append(so); self.sp.append(sp); self.sg.append(sg)
            so += k * k; sp += k * (k + 1) // 2; sg += k
        self.rows = so
        self.m = so + GAP
        self.L = max(so, 17) + GAP
        self.ldg = self.m
        self.sG = self.ldg * n + GAP

    def size(self, name):
        if name in ("G", "Gs"):
            return self.sG * self.batch
        return (self.m if name in M_OPS else self.L) * self.batch

    def stride(self, name):
        return self.m if name in M_OPS else self.L

    def nan(self, name):
        return np.full(self.size(name), np.nan)

    def blk(self, buf, name, b, k, col=0):
        """view of block k of problem b (column col of G / Gs) as an ms x ms column-major matrix"""
        ms = self.orders[k]
        o = (b * self.sG + col * self.ldg if name in ("G", "Gs") else b * self.stride(name)) + self.so[k]
        return buf[o:o + ms * ms].reshape(ms, ms, order="F")

    def pk(self, buf, name, b, k, col=0):
        ms = self.orders[k]
        o = (b * self.sG + col * self.ldg if name in ("G", "Gs") else b * self.stride(name)) + self.sp[k]
        return buf[o:o + ms * (ms + 1) // 2]

    def diag_idx(self, b, k):
        ms = self.orders[k]
        return b * self.m + self.so[k] + np.arange(ms) * (ms + 1)

    def sig(self, buf, b, k):
        o = b * self.L + self.sg[k]
        return buf[o:o + self.orders[k]]

    def mask(self, name, what):
        """True where a kernel may write: 'blk' whole blocks, 'pk' packed blocks, 'diag' diagonal rows, 'sig' the
        eigenvalue rows, 'gs' the packed blocks of every column of Gs"""
        mk = np.zeros(self.size(name), bool)
        for b in range(self.batch):
            for k, ms in enumerate(self.orders):
                if what == "blk":
                    self.blk(mk, name, b, k)[:] = True
                elif what == "pk":
                    self.pk(mk, name, b, k)[:] = True
                elif what == "diag":
                    mk[self.diag_idx(b, k)] = True
                elif what == "sig":
                    self.sig(mk, b, k)[:] = True
                elif what == "gs":
                    for j in range(self.n):
                        self.pk(mk, name, b, k, j)[:] = True
        return mk


WRITES = {   # kernel -> {operand: region it may write}
    "nt_compute": {"r": "blk", "rti": "blk", "lmbda": "diag"},
    "update": {"d": "blk", "di": "blk", "ds": "blk", "dz": "blk", "lmbdasq": "diag"},
    "dir_post0": {"ws3": "blk"},
    "dir_post1": {"ds": "blk", "dz": "blk", "sigs": "sig", "sigz": "sig"},
    "eig_start": {}, "eig_warm": {},
    "build_gs": {"Gs": "gs"},
    "wtz0": {"bzp": "pk"}, "wtz1": {"bzp": "pk", "th": "pk"}, "wtz2": {"bzp": "pk", "s": "blk"},
    "res0": {"wz3": "blk", "wz2": "blk", "ws2": "blk"}, "res1": {"wz3": "blk", "wz2": "blk", "ws2": "blk"},
}
KERNEL = {"nt_compute": 0, "update": 1, "dir_post": 2, "eig_start": 3, "eig_warm": 4, "build_gs": 5, "wtz": 6,
          "res": 7}


def run(lay, kernel, mode, ops, done=None, info=None, step=0.0, ut=0.0, spart=None, check_untouched=True):
    """launch `kernel` on host buffers `ops` (name -> flat array, copied to the device); returns (outputs, spart).
    Everything outside the regions WRITES allows comes back bit for bit."""
    import torch
    L, lib = _lib()
    dev = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in ops.items()}
    a = L.SblockArgs()
    orders = np.array(lay.orders, dtype=np.intc)
    a.nblk, a.orders, a.m, a.L = len(lay.orders), orders.ctypes.data, lay.m, lay.L
    a.n, a.ldg, a.sG, a.step, a.ut = lay.n, lay.ldg, lay.sG, step, ut
    d_arr = None if done is None else np.ascontiguousarray(done, dtype=np.intc)
    i_arr = None if info is None else np.ascontiguousarray(info, dtype=np.intc)
    a.done = None if d_arr is None else d_arr.ctypes.data
    a.info = None if i_arr is None else i_arr.ctypes.data
    sp = np.zeros(lay.batch * len(lay.orders) * 4) if spart is None else np.array(spart, dtype=float)
    a.spart = sp.ctypes.data
    for k, v in dev.items():
        setattr(a, k, v.data_ptr())
    torch.cuda.synchronize()
    rc = lib.cvxb_sblock_batched(KERNEL[kernel.rstrip("012")], mode, lay.batch, ctypes.byref(a), 0)
    assert rc == 0, L.last_error()
    out = {k: v.cpu().numpy() for k, v in dev.items()}
    if check_untouched:
        allowed = WRITES[kernel]
        for k in ops:
            diff = ops[k].view(np.uint64) != out[k].view(np.uint64)
            if k in allowed:
                diff &= ~lay.mask(k, allowed[k])
            assert not diff.any(), "%s wrote %d elements of %s outside its rows" % (kernel, int(diff.sum()), k)
    return out, sp.reshape(lay.batch, len(lay.orders), 4)


def _slot(lay, name):
    return lay.sG if name in ("G", "Gs") else lay.stride(name)


def same_bits_again_and_alone(lay, kernel, mode, ops, out, sp, **kw):
    """determinism: a second launch gives the same bits; cross-talk: each sampled problem j > 0 gives, in slot 0 of a
    batch of two (with problem 0 as its neighbour), the bits it gave in slot j"""
    again, sp2 = run(lay, kernel, mode, ops, check_untouched=False, **kw)
    assert all(_bits(out[k], again[k]) for k in out) and _bits(sp, sp2), "%s is not deterministic" % kernel
    two = Layout(lay.orders, 2, lay.n)
    for j in _samples(lay.batch)[1:]:
        ops2 = {nm: np.concatenate([v[j * _slot(lay, nm):(j + 1) * _slot(lay, nm)], v[:_slot(lay, nm)]])
                for nm, v in ops.items()}
        kw2 = dict(kw)
        if kw.get("spart") is not None:
            kw2["spart"] = np.concatenate([kw["spart"][j], kw["spart"][0]])
        out2, sp3 = run(two, kernel, mode, ops2, check_untouched=False, **kw2)
        for nm in out:
            st = _slot(lay, nm)
            assert _bits(out2[nm][:st], out[nm][j * st:(j + 1) * st]), ("cross-talk", kernel, nm, j)
        assert _bits(sp3[0], sp[j]), ("cross-talk in spart", kernel, j)


# ------------------------------------------------------------------------------------------------------------ inputs
def _rng(*seed):
    return np.random.default_rng(list(seed))


def _orth(n, rng):
    return np.linalg.qr(rng.standard_normal((n, n)))[0]


def spd_pair(n, fam, rng):
    """(s, z) of one block in the family `fam`"""
    if fam == "spd":
        B, C = rng.standard_normal((n, n)), rng.standard_normal((n, n))
        return B @ B.T / n + np.eye(n), C @ C.T / n + np.eye(n)
    if fam == "late":                      # s = Q diag(sig) Q', z = Q diag(mu / sig) Q' + a small perturbation
        Q, mu = _orth(n, rng), 1e-6
        sig = 10.0 ** rng.uniform(-8, 0, n)
        E = rng.standard_normal((n, n)) * 1e-5 * mu
        return sym_lower((Q * sig) @ Q.T), sym_lower((Q * (mu / sig)) @ Q.T + (E + E.T) / 2)
    if fam == "diag":
        return np.diag(rng.uniform(0.5, 2, n)), np.diag(rng.uniform(0.5, 2, n))
    if fam == "cluster":                   # identity and eigenvalues a few ulps apart
        Q = _orth(n, rng)
        w = 1.0 + np.arange(n) % 3 * 2 * np.finfo(float).eps
        return np.eye(n), sym_lower((Q * w) @ Q.T)
    q = rng.standard_normal(n)             # rank one plus identity
    return np.eye(n) + np.outer(q, q), np.eye(n) + 0.5 * np.outer(q[::-1], q[::-1])


def sym_input(n, fam, rng):
    """a symmetric (possibly indefinite) matrix for the eigen paths"""
    if fam == "spd":
        return sym_lower(rng.standard_normal((n, n)))       # indefinite
    s, z = spd_pair(n, fam, rng)
    return s if fam != "late" else s - 1e-9 * z


def _lower_only(M):
    """M with NaN in its strict upper triangle: the kernels read only the lower triangle"""
    X = np.array(M, dtype=float)
    X[np.triu_indices(X.shape[0], 1)] = np.nan
    return X


def _fam(b, k):
    return FAMILIES[(b + k) % len(FAMILIES)]


def fill(lay, names, gen, lower=()):
    """NaN buffers with block (b, k) of each name in `names` from gen(b, k, ms) -> dict name -> matrix"""
    ops = {nm: lay.nan(nm) for nm in names}
    for b in range(lay.batch):
        for k, ms in enumerate(lay.orders):
            for nm, M in gen(b, k, ms).items():
                if nm not in ops:
                    continue
                if nm == "lmbda" or nm == "lmbdasq":
                    ops[nm][lay.diag_idx(b, k)] = M
                elif nm in ("sigs", "sigz"):
                    lay.sig(ops[nm], b, k)[:] = M
                elif nm in ("bzp", "th"):
                    lay.pk(ops[nm], nm, b, k)[:] = M
                else:
                    lay.blk(ops[nm], nm, b, k)[:] = _lower_only(M) if nm in lower else M
    return ops


def _lam(lay, buf, b, k, name="lmbda"):
    return buf[name][lay.diag_idx(b, k)]


def _bits(a, b):
    return np.array_equal(np.asarray(a).view(np.uint64), np.asarray(b).view(np.uint64))


CONFIGS = [(ALL, 3), (MIXED, 1), (MIXED, 3), (MIXED, 257)]


def _ids(c):
    return "%s-b%d" % ("all" if c[0] == ALL else "mixed", c[1])


# ------------------------------------------------------------------------------------------------ k_s_nt_compute
def _nt_inputs(lay, seed):
    def gen(b, k, ms):
        s, z = spd_pair(ms, _fam(b, k), _rng(seed, b, k))
        return {"s": s, "z": z}
    ops = fill(lay, ("s", "z"), gen, lower=("s", "z"))
    for nm in ("r", "rti", "lmbda"):
        ops[nm] = lay.nan(nm)
    return ops


@pytest.mark.parametrize("cfg", CONFIGS, ids=_ids)
def test_nt_compute(cfg):
    orders, batch = cfg
    lay = Layout(orders, batch)
    ops = _nt_inputs(lay, 1)
    out, sp = run(lay, "nt_compute", 0, ops)
    worst = 0.0
    for b in _samples(batch):
        for k, ms in enumerate(orders):
            assert sp[b, k, 3] == 0.0
            s, z = sym_lower(lay.blk(ops["s"], "s", b, k)), sym_lower(lay.blk(ops["z"], "z", b, k))
            worst = max(worst, check_nt_scaling(s, z, lay.blk(out["r"], "r", b, k), lay.blk(out["rti"], "rti", b, k),
                                                 _lam(lay, out, b, k)))
    print("k_s_nt_compute %s: largest error / bound %.3g" % (_ids(cfg), worst))
    same_bits_again_and_alone(lay, "nt_compute", 0, ops, out, sp)


def test_nt_compute_crosstalk_and_skip_paths():
    """slot j against slot 0 of a batch of two; a non-PD block fails only its problem; done problems are untouched"""
    lay = Layout(MIXED, 257)
    ops = _nt_inputs(lay, 2)
    j = 200
    lay.blk(ops["z"], "z", j, 3)[2, 2] = -1.0              # not positive definite: block 3 of problem j fails
    done = np.zeros(257, int); done[7] = 1
    out, sp = run(lay, "nt_compute", 0, ops, done=done)
    assert sp[j, 3, 3] == 1.0 and np.all(np.isnan(_lam(lay, out, j, 3)))
    assert np.all(sp[np.arange(257) != j, :, 3] == 0) and np.all(sp[j, [0, 1, 2, 4, 5], 3] == 0)
    for k in range(len(MIXED)):
        for nm in ("r", "rti"):
            assert _bits(lay.blk(out[nm], nm, 7, k), lay.blk(ops[nm], nm, 7, k)), "done problem written"
        assert np.all(np.isnan(_lam(lay, out, 7, k)))
        if k != 3:
            assert np.all(np.isfinite(_lam(lay, out, j, k)))
    two = Layout(MIXED, 2)
    for slot in (1, 128, 256):
        ops2 = {nm: np.concatenate([v[slot * lay.stride(nm):(slot + 1) * lay.stride(nm)],
                                    v[0:lay.stride(nm)]]) for nm, v in ops.items()}
        out2, _ = run(two, "nt_compute", 0, ops2)
        for nm in ("r", "rti", "lmbda"):
            st = lay.stride(nm)
            assert _bits(out2[nm][:st], out[nm][slot * st:(slot + 1) * st]), ("cross-talk", nm, slot)


def test_nt_compute_batch_max():
    lay = Layout([2], BATCH_MAX)
    rng = _rng(3)
    A = rng.standard_normal((BATCH_MAX, 2, 2))
    S = A @ A.transpose(0, 2, 1) + np.eye(2)
    ops = {nm: lay.nan(nm) for nm in ("s", "z", "r", "rti", "lmbda")}
    for nm, M in (("s", S), ("z", S[::-1])):
        v = ops[nm].reshape(BATCH_MAX, lay.m)
        v[:, :4] = M.transpose(0, 2, 1).reshape(BATCH_MAX, 4)
        v[:, 2] = np.nan                                  # strict upper triangle
    out, sp = run(lay, "nt_compute", 0, ops, check_untouched=False)
    worst = 0.0
    for b in _samples(BATCH_MAX):
        worst = max(worst, check_nt_scaling(S[b], S[BATCH_MAX - 1 - b], lay.blk(out["r"], "r", b, 0),
                                            lay.blk(out["rti"], "rti", b, 0), _lam(lay, out, b, 0)))
    assert np.all(sp[:, 0, 3] == 0)
    print("k_s_nt_compute batch %d: largest error / bound %.3g" % (BATCH_MAX, worst))


# ------------------------------------------------------------------------------- k_s_dir_post, k_s_update (chained)
def _dir_inputs(lay, out, seed, lamname="lmbda"):
    """directions ds, dz with lambda^{-1/2} ds lambda^{-1/2} of 2-norm <= 1 (so 1 + step sig > 0 for step < 1)"""
    def gen(b, k, ms):
        rng = _rng(seed, b, k)
        h = np.sqrt(_lam(lay, out, b, k, lamname))
        res = {}
        for nm in ("ds", "dz"):
            X = sym_lower(rng.standard_normal((ms, ms)))
            X = X / max(np.abs(np.linalg.eigvalsh(X)).max(), 1e-300) * 0.9
            res[nm] = sym_lower(h[:, None] * X * h[None, :])
        return res
    return fill(lay, ("ds", "dz"), gen, lower=("ds", "dz"))


def _scaled(lay, ops, nm, b, k, lam):
    """what k_s_dir_post hands to the eigensolver: X_ij / (sqrt(l_i) sqrt(l_j)), in the kernel's fp64 operations"""
    X = sym_lower(lay.blk(ops[nm], nm, b, k))
    h = np.sqrt(lam)
    return X / (h[:, None] * h[None, :])


def _sdot(X, Y):
    """(sdot, its magnitude) of one block in long double: the diagonal once, the strict lower triangle twice"""
    n = X.shape[0]
    w = np.where(np.tri(n, dtype=bool), 2.0, 0.0) - np.eye(n)
    t = w * X.astype(LD) * Y.astype(LD)
    return np.sum(t), np.sum(np.abs(t))


def _check_dir_post(lay, ops, out, sp, mode, parts):
    worst = 0.0
    for b in _samples(lay.batch):
        for k, ms in enumerate(lay.orders):
            lam = _lam(lay, ops, b, k)
            Ds, Dz = sym_lower(lay.blk(ops["ds"], "ds", b, k)), sym_lower(lay.blk(ops["dz"], "dz", b, k))
            ref, mag = _sdot(Ds, Dz)
            worst = max(worst, check_sums(np.array([sp[b, k, 0]]), np.array([ref]), np.array([mag]), ms * ms))
            As, Az = _scaled(lay, ops, "ds", b, k, lam), _scaled(lay, ops, "dz", b, k, lam)
            if mode == 1:
                for nm, A, sg in (("ds", As, "sigs"), ("dz", Az, "sigz")):
                    V, w = lay.blk(out[nm], nm, b, k), lay.sig(out[sg], b, k)
                    worst = max(worst, check_sym_eig(A, V, w, parts=parts))
                assert sp[b, k, 1] == lay.sig(out["sigs"], b, k).min()
                assert sp[b, k, 2] == lay.sig(out["sigz"], b, k).min()
            else:
                W = lay.blk(out["ws3"], "ws3", b, k)
                assert _bits(W, W.T), "ws3 not exactly symmetric"
                DL, ZL = Ds.astype(LD), Dz.astype(LD)
                ref = (DL @ ZL + ZL @ DL) / 2
                mag = (np.abs(DL) @ np.abs(ZL) + np.abs(ZL) @ np.abs(DL)) / 2
                worst = max(worst, check_sums(W, ref, mag, ms + 1))
            worst = max(worst, check_min_eig(As, sp[b, k, 1]), check_min_eig(Az, sp[b, k, 2]))
    return worst


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("cfg", CONFIGS, ids=_ids)
def test_dir_post(cfg, mode):
    orders, batch = cfg
    lay = Layout(orders, batch)
    base, _ = run(lay, "nt_compute", 0, _nt_inputs(lay, 4))
    ops = _dir_inputs(lay, base, 5)
    ops["lmbda"] = base["lmbda"]
    ops.update({nm: lay.nan(nm) for nm in (("ws3",) if mode == 0 else ("sigs", "sigz"))})
    out, sp = run(lay, "dir_post%d" % mode, mode, ops)
    parts = {}
    worst = _check_dir_post(lay, ops, out, sp, mode, parts)
    # lambda = 1: a plain eigendecomposition of the families' (indefinite) blocks
    one = fill(lay, ("ds", "dz", "lmbda"), lambda b, k, ms: {
        "ds": sym_input(ms, _fam(b, k), _rng(6, b, k)), "dz": sym_input(ms, _fam(b + 1, k), _rng(7, b, k)),
        "lmbda": np.ones(ms)}, lower=("ds", "dz"))
    one.update({nm: lay.nan(nm) for nm in (("ws3",) if mode == 0 else ("sigs", "sigz"))})
    out1, sp1 = run(lay, "dir_post%d" % mode, mode, one)
    worst = max(worst, _check_dir_post(lay, one, out1, sp1, mode, parts))
    print("k_s_dir_post i=%d %s: largest error / bound %.3g%s" % (mode, _ids(cfg), worst, "".join(
        " (%s %.3g)" % kv for kv in sorted(parts.items()))))
    same_bits_again_and_alone(lay, "dir_post%d" % mode, mode, one, out1, sp1)


@pytest.mark.parametrize("cfg", [(ALL, 3), (MIXED, 257)], ids=_ids)
def test_update_chained(cfg):
    """the IPM's own sequence: k_s_nt_compute, then four rounds of k_s_dir_post(i = 1) and k_s_update, each update
    committed as the solver commits it (r := d, rti := di, lambda := lmbdasq's diagonal)"""
    orders, batch = cfg
    lay = Layout(orders, batch)
    st, _ = run(lay, "nt_compute", 0, _nt_inputs(lay, 8))
    worst = 0.0
    step = 0.95
    for it in range(4):
        dirs = _dir_inputs(lay, st, 20 + it)
        ops = {"ds": dirs["ds"], "dz": dirs["dz"], "lmbda": st["lmbda"], "sigs": lay.nan("sigs"),
               "sigz": lay.nan("sigz")}
        dp, _ = run(lay, "dir_post1", 1, ops)
        up = {"lmbda": st["lmbda"], "sigs": dp["sigs"], "sigz": dp["sigz"], "ds": dp["ds"], "dz": dp["dz"],
              "r": st["r"], "rti": st["rti"], "d": lay.nan("d"), "di": lay.nan("di"), "lmbdasq": lay.nan("lmbdasq")}
        out, sp = run(lay, "update", 0, up, step=step)
        assert np.all(sp[:, :, 3] == 0)
        if it == 0:
            same_bits_again_and_alone(lay, "update", 0, up, out, sp, step=step)
        for b in _samples(batch):
            for k, ms in enumerate(orders):
                g = lambda nm, o=out: lay.blk(o[nm], nm, b, k)
                worst = max(worst, check_nt_update(
                    lay.blk(st["r"], "r", b, k), lay.blk(st["rti"], "rti", b, k), _lam(lay, st, b, k),
                    lay.blk(dp["ds"], "ds", b, k), lay.sig(dp["sigs"], b, k),
                    lay.blk(dp["dz"], "dz", b, k), lay.sig(dp["sigz"], b, k), step,
                    g("ds"), g("dz"), g("d"), g("di"), _lam(lay, out, b, k, "lmbdasq")))
        new = {"r": lay.nan("r"), "rti": lay.nan("rti"), "lmbda": lay.nan("lmbda")}
        for b in range(batch):
            for k in range(len(orders)):
                lay.blk(new["r"], "r", b, k)[:] = lay.blk(out["d"], "d", b, k)
                lay.blk(new["rti"], "rti", b, k)[:] = lay.blk(out["di"], "di", b, k)
                new["lmbda"][lay.diag_idx(b, k)] = _lam(lay, out, b, k, "lmbdasq")
        st = new
        print("k_s_update %s round %d: largest error / bound %.3g" % (_ids(cfg), it, worst))
    # skip paths: done, info > 0 and first with a failed k_s_nt_compute leave the problem untouched
    done = np.zeros(batch, int); info = np.zeros(batch, int)
    done[0] = 1
    if batch > 1:
        info[batch - 1] = 3
    spin = np.zeros((batch, len(orders), 4))
    spin[batch // 2, :, 3] = 1.0 if batch > 2 else 0.0
    out2, sp2 = run(lay, "update", 1, up, done=done, info=info, step=step, spart=spin, check_untouched=False)
    skipped = {0, batch - 1} | ({batch // 2} if batch > 2 else set())
    for b in range(batch):
        for nm in ("d", "di", "ds", "dz"):
            same = _bits(out2[nm][b * lay.m:(b + 1) * lay.m], up[nm][b * lay.m:(b + 1) * lay.m])
            assert same == (b in skipped), (b, nm)


# ---------------------------------------------------------------------------------- k_s_eig_start, k_s_eig_warm
@pytest.mark.parametrize("cfg", CONFIGS + [([2], BATCH_MAX)], ids=lambda c: _ids(c) if c[1] != BATCH_MAX else "max")
@pytest.mark.parametrize("kernel", ["eig_start", "eig_warm"])
def test_eig_min(kernel, cfg):
    orders, batch = cfg
    lay = Layout(orders, batch)
    if batch == BATCH_MAX:
        rng = _rng(9)
        A = rng.standard_normal((batch, 2, 2))
        A = A + A.transpose(0, 2, 1)
        ops = {nm: lay.nan(nm) for nm in ("s", "z", "bzp")}
        for nm in ("s", "z"):
            ops[nm].reshape(batch, lay.m)[:, :4] = A.transpose(0, 2, 1).reshape(batch, 4)
        ops["bzp"].reshape(batch, lay.m)[:, :3] = np.stack([A[:, 0, 0], np.sqrt(2) * A[:, 1, 0], A[:, 1, 1]], 1)
        gen = lambda b, k: (A[b], A[b])
    else:
        def g(b, k, ms):
            X, Y = sym_input(ms, _fam(b, k), _rng(10, b, k)), sym_input(ms, _fam(b + 2, k), _rng(11, b, k))
            return {"s": X, "z": Y, "bzp": pack_ld(Y)}
        ops = fill(lay, ("s", "z", "bzp"), g, lower=("s", "z"))
        gen = lambda b, k: (sym_lower(lay.blk(ops["s"], "s", b, k)),
                            unpack(lay.pk(ops["bzp"], "bzp", b, k), orders[k]) if kernel == "eig_start"
                            else sym_lower(lay.blk(ops["z"], "z", b, k)))
    if kernel == "eig_start":
        del ops["z"]
    else:
        del ops["bzp"]
    out, sp = run(lay, kernel, 0, ops)
    if batch != BATCH_MAX:
        same_bits_again_and_alone(lay, kernel, 0, ops, out, sp)
    worst = 0.0
    for b in _samples(batch):
        for k in range(len(orders)):
            X, Y = gen(b, k)
            worst = max(worst, check_min_eig(X, sp[b, k, 1]), check_min_eig(Y, sp[b, k, 2]))
    print("k_s_%s %s: largest error / bound %.3g" % (kernel, _ids(cfg) if batch != BATCH_MAX else "max", worst))


# ----------------------------------------------------------------------------------------- k_s_build_gs, k_s_wtz
def _scaling(lay, seed):
    st, sp = run(lay, "nt_compute", 0, _nt_inputs(lay, seed))
    assert np.all(sp[:, :, 3] == 0)
    return st


@pytest.mark.parametrize("n", [1, 15, 16, 17, 100])
def test_build_gs(n):
    for orders, batch in ([MIXED, 3], [ALL, 1]) if n != 100 else ([MIXED, 3],):
        lay = Layout(orders, batch, n)
        st = _scaling(lay, 12)
        G = np.full(lay.size("G"), np.nan)
        rng = _rng(13, n)
        for b in range(batch):
            for j in range(n):
                for k, ms in enumerate(orders):
                    lay.blk(G, "G", b, k, j)[:] = _lower_only(rng.standard_normal((ms, ms)))
        ops = {"rti": st["rti"], "G": G, "Gs": np.full(lay.size("Gs"), np.nan)}
        out, sp = run(lay, "build_gs", 0, ops)
        same_bits_again_and_alone(lay, "build_gs", 0, ops, out, sp)
        worst = 0.0
        for b in _samples(batch):
            for j in sorted({0, 1, n // 2, 15, 16, n - 1} & set(range(n))):
                for k in range(len(orders)):
                    worst = max(worst, check_congruence(lay.blk(st["rti"], "rti", b, k), lay.blk(G, "G", b, k, j),
                                                        lay.pk(out["Gs"], "Gs", b, k, j), True, packed=True))
        print("k_s_build_gs n=%d %s: largest error / bound %.3g" % (n, _ids((orders, batch)), worst))


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("cfg", CONFIGS, ids=_ids)
def test_wtz(cfg, mode):
    orders, batch = cfg
    lay = Layout(orders, batch)
    st = _scaling(lay, 14)
    ops = fill(lay, ("z", "s"), lambda b, k, ms: {"z": sym_input(ms, _fam(b, k), _rng(15, b, k)),
                                                   "s": sym_input(ms, _fam(b + 1, k), _rng(16, b, k))},
               lower=("z", "s"))
    ops.update({"rti": st["rti"], "bzp": lay.nan("bzp")})
    if mode == 1:
        ops["th"] = lay.nan("th")
    if mode == 2:
        ops.update({"r": st["r"], "lmbda": st["lmbda"]})
    else:
        del ops["s"]
    out, sp = run(lay, "wtz%d" % mode, mode, ops)
    same_bits_again_and_alone(lay, "wtz%d" % mode, mode, ops, out, sp)
    worst = 0.0
    for b in _samples(batch):
        for k, ms in enumerate(orders):
            rti, Z = lay.blk(st["rti"], "rti", b, k), sym_lower(lay.blk(ops["z"], "z", b, k))
            got = lay.pk(out["bzp"], "bzp", b, k)
            if mode == 2:                           # s := lambda o\ s, then z - r s r'
                lam = _lam(lay, st, b, k)
                S1 = sym_lower(lay.blk(ops["s"], "s", b, k)) / (0.5 * (lam[:, None] + lam[None, :]))
                assert _bits(lay.blk(out["s"], "s", b, k), S1), "s := lambda o\\ s"
                r = lay.blk(st["r"], "r", b, k).astype(LD)
                X = Z.astype(LD) - r @ S1.astype(LD) @ r.T
                Xm = np.abs(Z).astype(LD) + np.abs(r) @ np.abs(S1).astype(LD) @ np.abs(r).T
                tl = rti.astype(LD)
                ref, mag = pack_ld(tl.T @ X @ tl), pack_ld(np.abs(tl).T @ Xm @ np.abs(tl))
                worst = max(worst, check_sums(got, ref, mag, 4 * ms + 3))
            else:
                worst = max(worst, check_congruence(rti, Z, got, True, packed=True))
            if mode == 1:
                assert _bits(lay.pk(out["th"], "th", b, k), got)
    print("k_s_wtz mode %d %s: largest error / bound %.3g" % (mode, _ids(cfg), worst))


# ------------------------------------------------------------------------------------------------------ k_s_res
@pytest.mark.parametrize("lp", [0, 1])
@pytest.mark.parametrize("cfg", CONFIGS, ids=_ids)
def test_res(cfg, lp):
    orders, batch = cfg
    lay = Layout(orders, batch)
    st = _scaling(lay, 17)
    ut = 0.37 if lp else 0.0

    def gen(b, k, ms):
        rng = _rng(18, b, k)
        return {nm: sym_lower(rng.standard_normal((ms, ms))) for nm in ("dz", "ds", "h", "wz", "ws")}
    ops = fill(lay, ("dz", "ds", "h", "wz", "ws"), gen, lower=("dz", "ds", "h", "wz", "ws"))
    ops.update({"rti": st["rti"], "r": st["r"], "lmbda": st["lmbda"]})
    ops.update({nm: lay.nan(nm) for nm in ("wz3", "wz2", "ws2")})
    if not lp:
        del ops["h"]
    out, sp = run(lay, "res%d" % lp, lp, ops, ut=ut)
    same_bits_again_and_alone(lay, "res%d" % lp, lp, ops, out, sp, ut=ut)
    worst = 0.0
    for b in _samples(batch):
        for k, ms in enumerate(orders):
            blk = lambda nm, o=ops: sym_lower(lay.blk(o[nm], nm, b, k))
            rti, r = lay.blk(st["rti"], "rti", b, k), lay.blk(st["r"], "r", b, k)
            W3 = lay.blk(out["wz3"], "wz3", b, k)
            worst = max(worst, check_congruence(rti, blk("dz"), W3, False))
            rl = r.astype(LD)
            Ds = blk("ds").astype(LD)
            H = blk("h").astype(LD) if lp else 0
            ref = blk("wz").astype(LD) + LD(ut) * H - rl @ Ds @ rl.T
            mag = np.abs(blk("wz")).astype(LD) + abs(LD(ut)) * np.abs(H) + np.abs(rl) @ np.abs(Ds) @ np.abs(rl).T
            worst = max(worst, check_sums(lay.blk(out["wz2"], "wz2", b, k), ref, mag, 2 * ms + 2))
            lam = _lam(lay, st, b, k).astype(LD)
            li = (lam[:, None] + lam[None, :]) / 2
            X = blk("dz").astype(LD) + Ds
            ref = blk("ws").astype(LD) - li * X
            mag = np.abs(blk("ws")).astype(LD) + li * (np.abs(blk("dz")).astype(LD) + np.abs(Ds))
            worst = max(worst, check_sums(lay.blk(out["ws2"], "ws2", b, k), ref, mag, 4))
            if lp:
                ref, mag = _sdot(blk("h"), W3)
                worst = max(worst, check_sums(np.array([sp[b, k, 0]]), np.array([ref]), np.array([mag]), ms * ms))
    print("k_s_res<%s> %s: largest error / bound %.3g" % ("true" if lp else "false", _ids(cfg), worst))
