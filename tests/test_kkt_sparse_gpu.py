"""Sparse G in the KKT factories, on the H100: the sparse factory against the dense factory on G.toarray(), the
sparse kernels' edge cases, bit-identical reruns, the G operator, the reference drivers end to end, the memory
held at a size where the dense G would not fit, and the choice between the sparse and the dense SYRK."""
import numpy as np
import pytest
import scipy.sparse as sps

from problems import cone_dim, cone_point, random_scaling

pytestmark = pytest.mark.gpu


def _rng(seed):
    return np.random.Generator(np.random.PCG64(seed))


def _sparse_rows(m, n, density, rng):
    """m x n CSR with about density * n entries per row (at least one per matrix), normal values"""
    nnz = max(1, int(round(density * m * n)))
    r = rng.integers(0, m, nnz)
    c = rng.integers(0, n, nnz)
    G = sps.coo_matrix((rng.standard_normal(nnz), (r, c)), shape=(m, n)).tocsr()
    G.sum_duplicates()
    return G


def _G(dims, n, density, seed):
    """sparse 'l' rows over dense 'q' rows and symmetric 's' columns: the layout a cone program's G has"""
    rng = _rng(seed)
    blocks = [_sparse_rows(dims["l"], n, density, rng)] if dims["l"] else []
    rest = cone_dim(dims) - dims["l"]
    if rest:
        D = rng.standard_normal((rest, n))
        off = sum(dims["q"])
        for k in dims["s"]:
            for j in range(n):
                M = D[off:off + k * k, j].reshape(k, k, order="F")
                D[off:off + k * k, j] = ((M + M.T) / 2).reshape(-1, order="F")
            off += k * k
        blocks.append(sps.csr_matrix(D))
    return sps.vstack(blocks, format="csr")


def _H(n, seed):
    B = _rng(seed).standard_normal((n, n))
    return np.asfortranarray(B @ B.T / n + np.eye(n))


def _relerr(a, b):
    return np.linalg.norm(np.ravel(a) - np.ravel(b)) / max(np.linalg.norm(np.ravel(b)), 1e-300)


def _solve_pair(fs, fd, W, n, p, cdim, seed, H=None, Df=None):
    """factor both with W, solve one right-hand side with both; the sparse result and the dense one"""
    rng = _rng(seed)
    x, z = rng.standard_normal(n), rng.standard_normal(cdim)
    y = rng.standard_normal(p) if p else np.zeros(0)
    out = []
    for f in (fs, fd):
        solve = f(W, H, Df) if (H is not None or Df is not None) else f(W)
        xx, yy, zz = x.copy(), y.copy(), z.copy()
        solve(xx, yy if p else None, zz)
        out.append((xx, yy, zz))
    return out


def _assert_close(pair, tol=1e-12):
    (xs, ys, zs), (xd, yd, zd) = pair
    assert _relerr(xs, xd) <= tol, _relerr(xs, xd)
    assert _relerr(zs, zd) <= tol, _relerr(zs, zd)
    if ys.size:
        assert _relerr(ys, yd) <= tol, _relerr(ys, yd)


DENSITIES = [1e-3, 1e-2, 0.2]


@pytest.mark.parametrize("density", DENSITIES)
@pytest.mark.parametrize("dims", [
    {"l": 3000, "q": [], "s": []},
    {"l": 2000, "q": [12, 7], "s": []},
    {"l": 1500, "q": [9], "s": [5, 3]},
])
def test_sparse_matches_dense_factory(dims, density):
    import cvxopt_b200
    n = 203
    G = _G(dims, n, density, seed=1)
    H = _H(n, 2)
    fs = cvxopt_b200.kkt_chol(G, dims, H=H)
    fd = cvxopt_b200.kkt_chol(np.asfortranarray(G.toarray()), dims, H=H)
    for it in range(3):                        # several factors, a fresh W each
        W, _ = random_scaling(dims, seed=10 + it)
        _assert_close(_solve_pair(fs, fd, W, n, 0, cone_dim(dims), seed=20 + it))
    assert fs.syrk_path() in ("sparse", "dmma")


@pytest.mark.parametrize("density", DENSITIES)
@pytest.mark.parametrize("factory", ["kkt_chol", "kkt_chol2", "kkt_ldl2"])
def test_sparse_with_equalities(factory, density):
    import cvxopt_b200
    n, p = 180, 23
    dims = {"l": 2500, "q": [], "s": []}
    G = _G(dims, n, density, seed=3)
    A = _rng(4).standard_normal((p, n))
    H = _H(n, 5)
    make = getattr(cvxopt_b200, factory)
    fs = make(G, dims, sps.csr_matrix(A), H=H)
    fd = make(np.asfortranarray(G.toarray()), dims, A, H=H)
    for it in range(3):
        W, _ = random_scaling(dims, seed=30 + it)
        _assert_close(_solve_pair(fs, fd, W, n, p, cone_dim(dims), seed=40 + it))


@pytest.mark.parametrize("density", DENSITIES)
def test_sparse_P_as_H(density):
    """a sparse P as the resident H and as a per-call H"""
    import cvxopt_b200
    n = 150
    dims = {"l": 1200, "q": [6], "s": []}
    G = _G(dims, n, density, seed=6)
    P = sps.random(n, n, density=0.05, random_state=np.random.RandomState(7), format="csc")
    P = (P @ P.T + sps.identity(n)).tocsc()
    Pd = np.asfortranarray(P.toarray())
    fs = cvxopt_b200.kkt_chol(G, dims, H=P)
    fd = cvxopt_b200.kkt_chol(np.asfortranarray(G.toarray()), dims, H=Pd)
    for it in range(3):
        W, _ = random_scaling(dims, seed=50 + it)
        _assert_close(_solve_pair(fs, fd, W, n, 0, cone_dim(dims), seed=60 + it))
    W, _ = random_scaling(dims, seed=59)
    _assert_close(_solve_pair(fs, fd, W, n, 0, cone_dim(dims), seed=61, H=P * 2.0))


@pytest.mark.parametrize("density", DENSITIES)
def test_sparse_nonlinear_rows_cp_kktsolver(density):
    """mnl > 0 through cp_kktsolver: F's Df (objective row dropped) and H per call, with the sparse G below them"""
    import cvxopt_b200
    n, mnl = 160, 4
    dims = {"l": 1800, "q": [5], "s": []}
    G = _G(dims, n, density, seed=8)
    rng = _rng(9)
    Df = rng.standard_normal((mnl + 1, n))
    H = _H(n, 10)

    def F(x=None, z=None):
        return None, Df, H
    ks_s = cvxopt_b200.cp_kktsolver(F, G, dims, None, mnl)
    ks_d = cvxopt_b200.cp_kktsolver(F, np.asfortranarray(G.toarray()), dims, None, mnl)
    cdim = mnl + cone_dim(dims)
    for it in range(3):
        W, _ = random_scaling(dims, seed=70 + it)
        dnl = _rng(80 + it).uniform(0.5, 2.0, mnl)
        W = dict(W, dnl=dnl, dnli=1.0 / dnl)
        x, z = rng.standard_normal(n), rng.standard_normal(cdim)
        res = []
        for ks in (ks_s, ks_d):
            xx, zz = x.copy(), z.copy()
            ks(None, None, W)(xx, None, zz)
            res.append((xx, np.zeros(0), zz))
        _assert_close(res)


def _edge_G(n, ml, rng, dense_row):
    """2 entries per row, an empty row (7), and either a fully dense row (11) or an empty column (5)"""
    rows, cols = [], []
    for i in range(ml):
        if i == 7:
            continue
        cs = np.arange(n) if (dense_row and i == 11) else rng.choice(n, 2, replace=False)
        rows.append(np.full(len(cs), i))
        cols.append(cs)
    rows, cols = np.concatenate(rows), np.concatenate(cols)
    if not dense_row:
        cols[cols == 5] = 6 if n > 6 else 0
    G = sps.csr_matrix((rng.standard_normal(rows.size), (rows, cols)), shape=(ml, n))
    G.sum_duplicates()
    return G


@pytest.mark.parametrize("dense_row", [True, False])
@pytest.mark.parametrize("n", [131, 77, 257])
def test_sparse_edge_cases(n, dense_row):
    """n a multiple of no tile size; an empty row; a fully dense row or an empty column"""
    import cvxopt_b200
    dims = {"l": 40000, "q": [], "s": []}
    G = _edge_G(n, dims["l"], _rng(n), dense_row)
    assert G.getnnz(axis=1)[7] == 0
    assert G.getnnz(axis=1)[11] == n if dense_row else G.getnnz(axis=0)[5] == 0
    H = _H(n, 11)
    fs = cvxopt_b200.kkt_chol(G, dims, H=H)
    fd = cvxopt_b200.kkt_chol(np.asfortranarray(G.toarray()), dims, H=H)
    W, _ = random_scaling(dims, seed=12)
    _assert_close(_solve_pair(fs, fd, W, n, 0, dims["l"], seed=13))
    assert fs.syrk_path() == "sparse"
    np.testing.assert_allclose(fs.get_L(), fd.get_L(), rtol=1e-12, atol=1e-13)


def test_sparse_single_nonzero():
    import cvxopt_b200
    n = 37
    dims = {"l": 50, "q": [], "s": []}
    G = sps.csr_matrix(([2.5], ([17], [29])), shape=(50, n))
    H = _H(n, 14)
    fs = cvxopt_b200.kkt_chol(G, dims, H=H)
    fd = cvxopt_b200.kkt_chol(np.asfortranarray(G.toarray()), dims, H=H)
    W, _ = random_scaling(dims, seed=15)
    _assert_close(_solve_pair(fs, fd, W, n, 0, dims["l"], seed=16))
    assert fs.syrk_path() == "sparse"


def test_sparse_bit_identical_reruns():
    import cvxopt_b200
    n, p = 240, 9
    dims = {"l": 4000, "q": [8], "s": [4]}
    G = _G(dims, n, 1e-2, seed=17)
    A = _rng(18).standard_normal((p, n))
    H = _H(n, 19)
    W, _ = random_scaling(dims, seed=20)
    runs = []
    for _ in range(2):
        f = cvxopt_b200.kkt_chol(G, dims, A, H=H)
        for rep in range(2):
            rng = _rng(21)
            x, y, z = rng.standard_normal(n), rng.standard_normal(p), rng.standard_normal(cone_dim(dims))
            f(W)(x, y, z)
            runs.append((x, y, z, f.get_L()))
        assert f.syrk_path() == "sparse"
    for r in runs[1:]:
        for a, b in zip(r, runs[0]):
            assert np.array_equal(a, b)


@pytest.mark.parametrize("trans", ["N", "T"])
def test_sparse_G_operator(trans):
    import cvxopt_b200
    n = 190
    dims = {"l": 2200, "q": [7], "s": [4]}
    G = _G(dims, n, 1e-2, seed=22)
    Gd = G.toarray()
    f = cvxopt_b200.kkt_chol(G, dims)
    rng = _rng(23)
    m = cone_dim(dims)
    nx, ny = (m, n) if trans == "T" else (n, m)
    for alpha, beta in [(1.0, 0.0), (-0.5, 2.0)]:
        x, y = rng.standard_normal(nx), rng.standard_normal(ny)
        want = alpha * (Gd.T @ x if trans == "T" else Gd @ x) + beta * y
        f.G(x, y, alpha, beta, trans)
        assert _relerr(y, want) < 1e-13


def _sparse_lp(n, ml, q, seed):
    """min c'x  s.t.  G x + s = h, s in 'l' x 'q': sparse rows, box rows, one dense 'q' block; strictly feasible"""
    rng = _rng(seed)
    Gl = sps.vstack([_sparse_rows(ml, n, 3.0 / n, rng), sps.identity(n), -sps.identity(n)], format="csr")
    dims = {"l": Gl.shape[0], "q": [q] if q else [], "s": []}
    G = sps.vstack([Gl, sps.csr_matrix(rng.standard_normal((q, n)))], format="csr") if q else Gl
    x0 = 0.1 * rng.standard_normal(n)
    s0, z0 = cone_point(dims, rng), cone_point(dims, rng)
    h = G @ x0 + s0
    c = -(G.T @ z0)
    return c, G.tocoo(), h, dims


def _spmatrix(ref, G):
    return ref.spmatrix(G.data.tolist(), G.row.tolist(), G.col.tolist(), G.shape)


def test_coneqp_sparse_G_matches_reference(ref):
    import cvxopt_b200
    from cvxopt import matrix, solvers
    n = 200
    c, G, h, dims = _sparse_lp(n, 600, 0, seed=24)
    P = _H(n, 25)
    Pm, qm, Gm, hm = matrix(P), matrix(c), _spmatrix(ref, G), matrix(h)
    f = cvxopt_b200.kkt_chol(Gm, dims, None, H=Pm)
    a = solvers.coneqp(Pm, qm, Gm, hm, dims, kktsolver=lambda W: f(W))
    b = solvers.coneqp(Pm, qm, Gm, hm, dims, kktsolver="chol")
    assert f.syrk_path() == "sparse"
    assert a["status"] == b["status"] == "optimal" and a["iterations"] == b["iterations"]
    np.testing.assert_allclose(a["primal objective"], b["primal objective"], rtol=1e-8)
    np.testing.assert_allclose(a["dual objective"], b["dual objective"], rtol=1e-8)
    np.testing.assert_allclose(np.array(a["x"]), np.array(b["x"]), rtol=1e-7, atol=1e-9)


def test_conelp_sparse_G_matches_reference(ref):
    import cvxopt_b200
    from cvxopt import matrix, solvers
    n = 200
    c, G, h, dims = _sparse_lp(n, 500, 6, seed=26)
    cm, Gm, hm = matrix(c), _spmatrix(ref, G), matrix(h)
    f = cvxopt_b200.kkt_chol(Gm, dims)
    a = solvers.conelp(cm, Gm, hm, dims, kktsolver=lambda W: f(W))
    b = solvers.conelp(cm, Gm, hm, dims, kktsolver="chol")
    assert f.syrk_path() == "sparse"
    assert a["status"] == b["status"] == "optimal" and a["iterations"] == b["iterations"]
    np.testing.assert_allclose(a["primal objective"], b["primal objective"], rtol=1e-8)
    np.testing.assert_allclose(a["dual objective"], b["dual objective"], rtol=1e-8)
    np.testing.assert_allclose(np.array(a["x"]), np.array(b["x"]), rtol=1e-7, atol=1e-9)


def test_sparse_memory_at_large_m():
    """n = 4096, m = 262144, 8 entries per row: the dense G alone would be 8.6 GB.  The factory holds K, the two
    CSR copies and the cone vectors: under 8 (2 n^2 + 3 nnz + 4 m) bytes, with 32 MB of slack for the fixed
    workspaces (the Cholesky's block inverses and split-K buffer)."""
    import cvxopt_b200
    from cvxopt_b200 import _lib
    n, m, per = 4096, 262144, 8
    rng = _rng(27)
    cols = np.stack([rng.choice(n, per, replace=False) for _ in range(64)])       # 64 row patterns, reused
    r = np.repeat(np.arange(m), per)
    c = cols[np.arange(m) % 64].ravel()
    c = (c + np.repeat(np.arange(m) // 64, per)) % n                              # shifted: every column is hit
    G = sps.csr_matrix((rng.standard_normal(m * per), (r, c)), shape=(m, n))
    nnz = G.nnz
    dims = {"l": m, "q": [], "s": []}
    lib = _lib.load()
    before = lib.cvxb_device_bytes()
    f = cvxopt_b200.kkt_chol(G, dims)
    W = {"d": rng.uniform(0.5, 2.0, m), "v": [], "beta": [], "r": [], "rti": []}
    W["di"] = 1.0 / W["d"]
    x, z = rng.standard_normal(n), rng.standard_normal(m)
    f(W)(x, None, z)
    grew = lib.cvxb_device_bytes() - before
    bound = 8 * (2 * n * n + 3 * nnz + 4 * m) + (32 << 20)
    assert f.syrk_path() == "sparse"
    assert grew < bound, (grew, bound)
    assert np.all(np.isfinite(x)) and np.all(np.isfinite(z))
    f.close()


def test_density_choice():
    """a dense-enough G goes the DMMA way and a sparse one the sparse way; both give the dense factory's directions"""
    import cvxopt_b200
    n = 256
    dims = {"l": 4000, "q": [], "s": []}
    H = _H(n, 28)
    W, _ = random_scaling(dims, seed=29)
    for density, path in [(0.5, "dmma"), (4.0 / n, "sparse")]:
        G = _G(dims, n, density, seed=30)
        fs = cvxopt_b200.kkt_chol(G, dims, H=H)
        fd = cvxopt_b200.kkt_chol(np.asfortranarray(G.toarray()), dims, H=H)
        _assert_close(_solve_pair(fs, fd, W, n, 0, dims["l"], seed=31))
        assert fs.syrk_path() == path


def test_kkt_qr_sparse_G():
    """kkt_qr densifies all of a sparse G, as the reference does: the same bits as the dense G; and the C ABI's QR route
    on a sparse handle (its 'l' rows densified by cvxb_kkt_set_method) gives the same directions"""
    import ctypes as C
    import cvxopt_b200
    from cvxopt_b200 import _lib
    from cvxopt_b200.kkt import make_dims, make_scaling, to_csr
    n = 60
    dims = {"l": 900, "q": [7], "s": []}
    G = _G(dims, n, 0.01, seed=32)             # sparse enough that the handle keeps its rows sparse
    W, _ = random_scaling(dims, seed=33)
    fs = cvxopt_b200.kkt_qr(G, dims)
    fd = cvxopt_b200.kkt_qr(np.asfortranarray(G.toarray()), dims)
    (xs, _, zs), (xd, _, zd) = _solve_pair(fs, fd, W, n, 0, cone_dim(dims), seed=34)
    assert np.array_equal(xs, xd) and np.array_equal(zs, zd)
    lib = _lib.load()
    cd, keep, cdim, _ = make_dims(dims)
    _, rowptr, colind, val = to_csr(G)
    h = C.c_void_p()
    _lib.check(lib.cvxb_kkt_create_sparse(C.byref(h), n, 0, C.byref(cd), rowptr.ctypes.data, colind.ctypes.data,
                                          val.ctypes.data, int(val.size), None, 1, _lib.HOST, 0), "create")
    try:
        assert lib.cvxb_kkt_syrk_path(h) == 0
        _lib.check(lib.cvxb_kkt_set_method(h, 1, 0.0), "set_method")
        sc, kw = make_scaling(W, dims["l"], dims["q"], dims["s"])
        _lib.check(lib.cvxb_kkt_factor(h, C.byref(sc), None, 1, None, 1, 0, _lib.HOST), "factor")
        rng = _rng(34)
        x, z = rng.standard_normal(n), rng.standard_normal(cdim)
        _lib.check(lib.cvxb_kkt_solve(h, x.ctypes.data, None, z.ctypes.data, _lib.HOST), "solve")
        assert _relerr(x, xd) < 1e-12 and _relerr(z, zd) < 1e-12
    finally:
        lib.cvxb_kkt_destroy(h)
