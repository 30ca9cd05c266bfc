"""GPU parity tests of the KKT path through the C-ABI: cvxopt_b200.kkt_chol vs the
numpy oracle (oracle/kkt_oracle.py), which is itself pinned to the reference by
tests/test_oracle_vs_reference.py.  Tolerance: north_star's 1e-10 on the search
direction (relative, 2-norm)."""
import numpy as np
import pytest

import kkt_oracle as ko
from problems import cone_dim, dense_qp, random_scaling

pytestmark = pytest.mark.gpu
TOL = 1e-10


def relerr(a, b):
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


def packed(z, dims):
    _, _, _, _, cp = ko.cone_sizes(dims)
    out = np.zeros(cp)
    ko.pack(z.copy(), out, dims)
    return out


def run_case(dims, n, seed, with_H=True, resident=False, factors=1):
    """`factors` factorisations of one factory with different scalings W, each solve against the oracle: the
    handle's Cholesky runs eagerly the first time, is captured into a CUDA graph the second and replayed after"""
    import cvxopt_b200
    rng = np.random.Generator(np.random.PCG64(seed))
    K = cone_dim(dims)
    G = np.asfortranarray(rng.standard_normal((K, n)))
    H = None
    if with_H:
        B = rng.standard_normal((n, n))
        H = np.asfortranarray(B @ B.T / n + np.eye(n))
    fac = cvxopt_b200.kkt_chol(G, dims, None, H=H if resident else None)
    for f in range(factors):
        W, _ = random_scaling(dims, seed=seed + 1 + f)
        solve = fac(W) if (resident or H is None) else fac(W, H)
        f_or = ko.KktChol(G, dims).factor(W, H)
        for rep in range(2):
            x, z = rng.standard_normal(n), rng.standard_normal(K)
            xo, zo = x.copy(), z.copy()
            solve(x, None, z)
            f_or(xo, None, zo)
            assert relerr(x, xo) < TOL, (f, "x", relerr(x, xo))
            assert relerr(packed(z, dims), packed(zo, dims)) < TOL, (f, "z", relerr(packed(z, dims), packed(zo, dims)))
        L = fac.get_L()
        assert relerr(L, f_or.__self__.L) < 1e-9, f
    fac.close()


@pytest.mark.parametrize("n,m,seed", [(1, 1, 0), (3, 7, 1), (64, 100, 2), (200, 400, 3), (257, 391, 4), (513, 1100, 5)])
def test_l_cones(n, m, seed):
    run_case({"l": m, "q": [], "s": []}, n, seed, factors=4)


def test_l_cones_no_H():
    run_case({"l": 300, "q": [], "s": []}, 150, 7, with_H=False)


def test_l_cones_resident_H():
    run_case({"l": 300, "q": [], "s": []}, 150, 8, resident=True)


@pytest.mark.parametrize("q,n,seed", [([5], 4, 0), ([64] * 8, 128, 1), ([3, 1, 70, 33], 50, 2)])
def test_q_cones(q, n, seed):
    run_case({"l": 0, "q": q, "s": []}, n, seed, factors=4)


@pytest.mark.parametrize("s,n,seed", [([3], 4, 0), ([1, 10, 33], 40, 1), ([64], 48, 2), ([130], 20, 3)])
def test_s_cones(s, n, seed):
    run_case({"l": 0, "q": [], "s": s}, n, seed, factors=4)


def test_mixed_cones():
    run_case({"l": 37, "q": [9, 64, 2], "s": [5, 17]}, 90, 11, factors=4)
    run_case({"l": 5, "q": [4], "s": [3]}, 3, 12, with_H=False, factors=4)


@pytest.mark.parametrize("dims,n,p,with_H", [
    ({"l": 300, "q": [], "s": []}, 150, 20, True),
    ({"l": 40, "q": [9, 30], "s": [7]}, 60, 5, True),
    ({"l": 500, "q": [], "s": []}, 300, 130, False),       # p spans two 128-blocks
    ({"l": 20, "q": [], "s": []}, 50, 35, False),          # S singular -> S + A'A fallback
])
def test_equality_constraints(dims, n, p, with_H):
    """p > 0: (ux, uy, W uz) vs the oracle (which is pinned to the reference's QR-based kkt_chol)."""
    import cvxopt_b200
    rng = np.random.Generator(np.random.PCG64(77))
    K = cone_dim(dims)
    G = np.asfortranarray(rng.standard_normal((K, n)))
    A = np.asfortranarray(rng.standard_normal((p, n)))
    H = None
    if with_H:
        B = rng.standard_normal((n, n))
        H = np.asfortranarray(B @ B.T / n + np.eye(n))
    W, _ = random_scaling(dims, seed=8)
    fac = cvxopt_b200.kkt_chol(G, dims, A)
    solve = fac(W, H) if with_H else fac(W)
    f_or = ko.KktChol(G, dims, A).factor(W, H)
    for rep in range(2):
        x, y, z = rng.standard_normal(n), rng.standard_normal(p), rng.standard_normal(K)
        xo, yo, zo = x.copy(), y.copy(), z.copy()
        solve(x, y, z)
        f_or(xo, yo, zo)
        assert relerr(x, xo) < 1e-9, relerr(x, xo)
        assert relerr(y, yo) < 1e-9, relerr(y, yo)
        assert relerr(packed(z, dims), packed(zo, dims)) < 1e-9
    fac.close()


@pytest.mark.parametrize("name,dims,p", [("kkt_chol2", {"l": 90, "q": [], "s": []}, 0),
                                         ("kkt_chol2", {"l": 90, "q": [], "s": []}, 11),
                                         ("kkt_ldl2", {"l": 30, "q": [8, 5], "s": [6]}, 0),
                                         ("kkt_ldl2", {"l": 30, "q": [8, 5], "s": [6]}, 9)])
def test_chol2_and_ldl2_factory_names(name, dims, p):
    """cvxopt_b200.kkt_chol2 / kkt_ldl2 (misc.py:1352 / :1128): same call protocol, same solution as the
    oracle (pinned to the reference's kkt_chol2 / kkt_ldl2 by tests/test_oracle_vs_reference.py)."""
    import cvxopt_b200
    n = 45
    rng = np.random.Generator(np.random.PCG64(5))
    K = cone_dim(dims)
    G = np.asfortranarray(rng.standard_normal((K, n)))
    A = np.asfortranarray(rng.standard_normal((p, n))) if p else None
    B = rng.standard_normal((n, n))
    H = np.asfortranarray(B @ B.T / n + np.eye(n))
    W, _ = random_scaling(dims, seed=6)
    fac = getattr(cvxopt_b200, name)(G, dims, A)
    solve = fac(W, H)
    f_or = ko.KktChol(G, dims, A).factor(W, H)
    x, y, z = rng.standard_normal(n), rng.standard_normal(p), rng.standard_normal(K)
    xo, yo, zo = x.copy(), y.copy(), z.copy()
    solve(x, y if p else None, z)
    f_or(xo, yo if p else None, zo)
    assert relerr(x, xo) < 1e-9
    if p:
        assert relerr(y, yo) < 1e-9
    assert relerr(packed(z, dims), packed(zo, dims)) < 1e-9
    fac.close()
    with pytest.raises(ValueError):
        cvxopt_b200.kkt_chol2(G, {"l": 0, "q": [4], "s": []}, None)


def test_indefinite_raises_arithmetic_error():
    import cvxopt_b200
    n = 40
    dims = {"l": 10, "q": [], "s": []}
    rng = np.random.Generator(np.random.PCG64(0))
    G = np.asfortranarray(rng.standard_normal((10, n)))     # rank 10 < n and no H: singular
    W, _ = random_scaling(dims, 1)
    fac = cvxopt_b200.kkt_chol(G, dims)
    with pytest.raises(ArithmeticError):
        fac(W)
    H = -np.eye(n)
    with pytest.raises(ArithmeticError):
        fac(W, np.asfortranarray(H))


def test_ill_conditioned_scaling():
    """late-IPM regime: d spans 1e8 (SURVEY.md §7.3-4)"""
    import cvxopt_b200
    n, m = 120, 300
    P, q, G, h = dense_qp(n, m, seed=5)
    rng = np.random.Generator(np.random.PCG64(1))
    d = 10.0 ** rng.uniform(-4, 4, m)
    W = {"d": d, "di": 1.0 / d, "v": [], "beta": [], "r": [], "rti": []}
    dims = {"l": m, "q": [], "s": []}
    fac = cvxopt_b200.kkt_chol(G, dims, H=P)
    solve = fac(W)
    f_or = ko.KktChol(G, dims).factor(W, P)
    x, z = rng.standard_normal(n), rng.standard_normal(m)
    xo, zo = x.copy(), z.copy()
    solve(x, None, z)
    f_or(xo, None, zo)
    # both are backward-stable solves of a system with cond ~1e16*...; compare through the
    # KKT residual of each instead of against each other when conditioning is extreme
    assert relerr(x, xo) < 1e-6
    assert relerr(z, zo) < 1e-6


@pytest.mark.parametrize("dims", [{"l": 5, "q": [4, 9], "s": [3, 7]}, {"l": 0, "q": [], "s": [20]}, {"l": 11, "q": [], "s": []}])
def test_misc_solvers_mirror(dims):
    """cvxopt_b200.misc_solvers.{scale,pack,unpack,pack2,symm} vs the oracle restatement."""
    from cvxopt_b200 import misc_solvers as ms
    W, _ = random_scaling(dims, seed=4)
    rng = np.random.Generator(np.random.PCG64(5))
    K = cone_dim(dims)
    _, _, _, _, cp = ko.cone_sizes(dims)
    il = []
    off = dims["l"] + sum(dims["q"])
    mask = np.ones(K, bool)            # strict upper triangles of 's' blocks are not significant
    for k in dims["s"]:
        M = np.ones((k, k), bool)
        M[np.triu_indices(k, 1)] = False
        mask[off:off + k * k] = M.reshape(-1, order="F")
        off += k * k
    for trans in "NT":
        for inverse in "NI":
            x = np.asfortranarray(rng.standard_normal((K, 5)))
            xo = x.copy()
            ms.scale(x, W, trans, inverse)
            ko.scale(xo, W, trans, inverse)
            assert relerr(x[mask], xo[mask]) < 1e-12, (trans, inverse)
    x = rng.standard_normal(K)
    y, yo = np.zeros(cp), np.zeros(cp)
    ms.pack(x, y, dims)
    ko.pack(x, yo, dims)
    assert np.array_equal(y, yo)
    z, zo = rng.standard_normal(K), None
    zo = z.copy()
    ms.unpack(y, z, dims)
    ko.unpack(yo, zo, dims)
    assert np.array_equal(z, zo)
    X = np.asfortranarray(rng.standard_normal((K, 3)))
    Xo = X.copy()
    ms.pack2(X, dims)
    ko.pack2(Xo, dims)
    assert np.array_equal(X[:cp], Xo[:cp])
    S = rng.standard_normal(49)
    So = S.copy()
    ms.symm(S, 7)
    ko.symm(So, 7)
    assert np.array_equal(S, So)


@pytest.mark.parametrize("dims", [{"l": 6, "q": [4, 9, 1], "s": []}, {"l": 5, "q": [7], "s": [3, 8]}, {"l": 0, "q": [], "s": [20]}])
def test_misc_solvers_mirror_ipm_side(dims):
    """scale2 / sprod / sinv / sdot / max_step / trisc / triusc on the device vs the oracle."""
    from cvxopt_b200 import misc_solvers as ms
    from problems import cone_point
    rng = np.random.Generator(np.random.PCG64(15))
    K = cone_dim(dims)
    W, lm = random_scaling(dims, seed=9)
    mask = np.ones(K, bool)
    off = dims["l"] + sum(dims["q"])
    for k in dims["s"]:
        M = np.ones((k, k), bool); M[np.triu_indices(k, 1)] = False
        mask[off:off + k * k] = M.reshape(-1, order="F"); off += k * k
    for inv in "NI":
        x = cone_point(dims, rng); xo = x.copy()
        ms.scale2(lm, x, dims, inverse=inv); ko.scale2(lm, xo, dims, inverse=inv)
        assert relerr(x, xo) < 1e-13
    x, y = cone_point(dims, rng), cone_point(dims, rng); xo = x.copy()
    ms.sprod(x, y, dims); ko.sprod(xo, y, dims)
    assert relerr(x[mask], xo[mask]) < 1e-13
    x = cone_point(dims, rng); xo = x.copy()
    ms.sprod(x, lm, dims, diag="D"); ko.sprod(xo, lm, dims, diag="D")
    assert relerr(x[mask], xo[mask]) < 1e-13
    x = cone_point(dims, rng); xo = x.copy()
    ms.sinv(x, lm, dims); ko.sinv(xo, lm, dims)
    assert relerr(x[mask], xo[mask]) < 1e-13
    x, y = cone_point(dims, rng), cone_point(dims, rng)
    assert abs(ms.sdot(x, y, dims) - ko.sdot(x, y, dims)) <= 1e-12 * abs(ko.sdot(x, y, dims))
    for f, fo in ((ms.trisc, ko.trisc), (ms.triusc, ko.triusc)):
        x = rng.standard_normal(K); xo = x.copy()
        f(x, dims); fo(xo, dims)
        assert np.array_equal(x, xo)
    x = rng.standard_normal(K)
    assert abs(ms.max_step(x.copy(), dims) - ko.max_step(x.copy(), dims)) < 1e-12


@pytest.mark.parametrize("dims", [{"l": 3, "q": [4], "s": [3, 8, 0, 1, 2]},      # one CTA per block (order <= 64)
                                  {"l": 0, "q": [], "s": [64, 33]},
                                  {"l": 2, "q": [], "s": [70, 5, 0, 1]},           # one launch per Jacobi round
                                  {"l": 0, "q": [], "s": [129]},
                                  {"l": 1, "q": [], "s": [200, 130, 7]}])           # several CTAs per block and round
def test_max_step_s_blocks_jacobi_eigensolver(dims):
    """max_step on 's' blocks (misc_solvers.c:1099-1150): smallest eigenvalue without sigma (dsyevr_),
    all eigenvalues + eigenvectors with sigma (dsyevd_ 'V').  Eigenvalues agree with LAPACK to
    1e-12 * ||X||; the eigenvectors (unique only up to sign / rotation inside an eigenspace) are checked
    through orthonormality and the reconstruction Q diag(sigma) Q' = X."""
    from cvxopt_b200 import misc_solvers as ms
    rng = np.random.Generator(np.random.PCG64(33))
    K = cone_dim(dims)
    x = rng.standard_normal(K)
    x0 = x.copy()
    t = ms.max_step(x, dims)
    assert np.array_equal(x, x0)                      # without sigma x is not modified (:1139 copies)
    assert abs(t - ko.max_step(x0.copy(), dims)) < 1e-12 * max(1.0, np.abs(x0).max() * max(dims["s"]))
    ns = sum(dims["s"])
    sig = np.full(ns, np.nan); sigo = np.zeros(ns)
    xo = x0.copy()
    t2 = ms.max_step(x, dims, sigma=sig)
    to = ko.max_step(xo, dims, sigma=sigo)
    assert abs(t2 - to) < 1e-12 * max(1.0, np.abs(x0).max() * max(dims["s"]))
    nlq = dims["l"] + sum(dims["q"])
    assert np.array_equal(x[:nlq], x0[:nlq])
    off, o2 = nlq, 0
    for mk in dims["s"]:
        if mk:
            X = x0[off:off + mk * mk].reshape(mk, mk, order="F")
            X = np.tril(X) + np.tril(X, -1).T
            scale_ = np.linalg.norm(X)
            w = sig[o2:o2 + mk]
            assert np.all(np.diff(w) >= 0)
            assert np.abs(w - sigo[o2:o2 + mk]).max() < 1e-12 * scale_
            Q = x[off:off + mk * mk].reshape(mk, mk, order="F")
            assert np.abs(Q.T @ Q - np.eye(mk)).max() < 1e-12
            assert np.abs(Q @ np.diag(w) @ Q.T - X).max() < 1e-12 * scale_
        off += mk * mk; o2 += mk


def test_max_step_s_blocks_special_matrices():
    """already diagonal, zero, repeated eigenvalues, huge dynamic range, and a non-finite entry
    (the Jacobi sweeps cannot converge: ArithmeticError, like a LAPACK info > 0)."""
    from cvxopt_b200 import misc_solvers as ms
    for X in (np.eye(6), np.zeros((4, 4)), np.diag([1.0, 1, 2, 2, 2]), np.ones((6, 6)),
              np.diag([1e-200, 1.0, 1e200]), np.array([[1e300, 1e-300], [1e-300, -1e300]])):
        mk = X.shape[0]
        dims = {"l": 0, "q": [], "s": [mk]}
        sig = np.zeros(mk)
        x = X.reshape(-1, order="F").copy()
        t = ms.max_step(x, dims, sigma=sig)
        w = np.linalg.eigvalsh(X)
        assert np.abs(sig - w).max() <= 1e-13 * max(np.abs(w).max(), 1e-300)
        assert t == -sig[0]
    bad = np.eye(5); bad[3, 1] = np.nan
    with pytest.raises(ArithmeticError):
        ms.max_step(bad.reshape(-1, order="F").copy(), {"l": 0, "q": [], "s": [5]})


def open_factory(case, rng):
    """create, factor and solve one KKT factory of the kind `case`; returned still open"""
    import cvxopt_b200
    n, p, dims = 30, 5, {"l": 40, "q": [5, 8], "s": [4, 3]}
    if case in ("l", "ozaki2", "trace"):
        n, p, dims = 300, 0, {"l": 900, "q": [], "s": []}
    K = cone_dim(dims)
    G = np.asfortranarray(rng.standard_normal((K, n)))
    A = np.asfortranarray(rng.standard_normal((p, n))) if p else None
    B = rng.standard_normal((n, n))
    H = np.asfortranarray(B @ B.T / n + np.eye(n))
    W, _ = random_scaling(dims, 3)
    mnl = 0
    if case == "qs_A_H":
        f = cvxopt_b200.kkt_chol(G, dims, A, H=H)
        f.set_H(H)                      # the resident H a second time
        f(W)
        f(W, H.copy())                  # a per-call H: the lazily allocated upload buffer
    elif case == "mnl_Df":
        mnl = 3
        W = dict(W, dnl=rng.uniform(0.5, 2.0, mnl))
        W["dnli"] = 1.0 / W["dnl"]
        f = cvxopt_b200.kkt_chol(G, dims, A, mnl)
        f(W, H, np.asfortranarray(rng.standard_normal((mnl, n))))
    elif case == "qr_A":
        f = cvxopt_b200.kkt_qr(G, dims, A)
        f(W)
    elif case == "ldl2_A":
        f = cvxopt_b200.kkt_ldl2(G, dims, A)
        f(W, H)
    else:
        f = cvxopt_b200.kkt_chol(G, dims)
        f(W)
        assert f.syrk_path() == ("int8" if case == "ozaki2" else "dmma")
    f.solve(rng.standard_normal(n), rng.standard_normal(p) if p else None, rng.standard_normal(mnl + K))
    return f


def check_lifecycle(case, rng, monkeypatch):
    """20 create/factor/solve/close rounds of one kind of factory: cvxb_device_bytes() is above its baseline while the
    factory is open and back to it exactly after close(), and the card's free memory does not drift"""
    import torch
    from cvxopt_b200 import _lib
    lib = _lib.load()
    monkeypatch.delenv("CVXB_OZAKI", raising=False)
    monkeypatch.delenv("CVXB_TRACE", raising=False)
    if case == "ozaki2":
        monkeypatch.setenv("CVXB_OZAKI", "2")
    if case == "trace":
        monkeypatch.setenv("CVXB_TRACE", "1")
    free0 = torch.cuda.mem_get_info()[0]
    open_factory(case, rng).close()     # warm-up
    base = lib.cvxb_device_bytes()
    for _ in range(20):
        f = open_factory(case, rng)
        assert lib.cvxb_device_bytes() > base
        f.close()
        assert lib.cvxb_device_bytes() == base
    free1 = torch.cuda.mem_get_info()[0]
    assert free0 - free1 < 64 << 20, (free0, free1)


@pytest.mark.parametrize("case", ["qs_A_H", "mnl_Df", "qr_A", "ldl2_A", "ozaki2", "trace"])
def test_factory_lifecycle_frees_device_memory(case, monkeypatch):
    """every byte of device memory a factory holds is freed with it, for each route and each lazily allocated
    buffer (the per-call H upload, the int8-slice workspace with CVXB_OZAKI=2, the Cholesky timeline with
    CVXB_TRACE=1); the 'l'-only Cholesky case is test_no_cone_rows_and_handle_lifecycle's"""
    check_lifecycle(case, np.random.Generator(np.random.PCG64(2)), monkeypatch)


def test_no_cone_rows_and_handle_lifecycle(monkeypatch):
    """cdim == 0 (unconstrained QP step: K = H) and repeated create/destroy (no leaks, no stale state)."""
    import cvxopt_b200
    n = 70
    rng = np.random.Generator(np.random.PCG64(2))
    B = rng.standard_normal((n, n))
    H = np.asfortranarray(B @ B.T + np.eye(n))
    dims = {"l": 0, "q": [], "s": []}
    W = {"d": np.zeros(0), "di": np.zeros(0), "v": [], "beta": [], "r": [], "rti": []}
    fac = cvxopt_b200.kkt_chol(np.zeros((0, n), order="F"), dims)
    solve = fac(W, H)
    x = rng.standard_normal(n)
    x0 = x.copy()
    solve(x, None, np.zeros(0))
    assert relerr(x, np.linalg.solve(H, x0)) < 1e-11
    fac.close()
    check_lifecycle("l", rng, monkeypatch)
