"""CPU-only: sparse G in the KKT factories.  The CSR converter, the argument checks of cvxb_kkt_create_sparse (made
before the device is touched), and what the sparse factory has to reproduce: the reference's own kkt_chol on a sparse
G against the oracle on the dense G."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sps

import kkt_oracle as ko
from problems import cone_dim, random_scaling


class SpStandIn:
    """The part of a cvxopt spmatrix the package reads: `size` and `CCS` (colptr, rowind, values)."""

    def __init__(self, rows, cols, colptr, rowind, vals):
        self.size = (rows, cols)
        self.CCS = (np.asarray(colptr, dtype=np.int64), np.asarray(rowind, dtype=np.int64),
                    np.asarray(vals, dtype=np.float64))


def _check_canonical(shape, rowptr, colind, val, dense):
    rows, cols = shape
    assert rowptr.dtype == np.int64 and colind.dtype == np.int32 and val.dtype == np.float64
    assert rowptr.shape == (rows + 1,) and rowptr[0] == 0 and rowptr[-1] == val.size == colind.size
    assert np.all(np.diff(rowptr) >= 0)
    for r in range(rows):
        assert np.all(np.diff(colind[rowptr[r]:rowptr[r + 1]]) > 0)      # sorted, no duplicates
    out = np.zeros((rows, cols))
    out[np.repeat(np.arange(rows), np.diff(rowptr)), colind] = val
    np.testing.assert_array_equal(out, dense)


def test_to_csr_scipy_formats():
    from cvxopt_b200.kkt import to_csr, _dense
    # duplicates (0,1) x2 and (3,2) x3, unsorted order, an explicit zero at (2,0), empty row 1 and empty column 3
    r = np.array([3, 0, 2, 3, 0, 3, 4])
    c = np.array([2, 1, 0, 2, 1, 2, 4])
    v = np.array([1.0, 2.0, 0.0, 0.5, -1.0, 0.25, 7.0])
    dense = np.zeros((5, 5))
    np.add.at(dense, (r, c), v)
    coo = sps.coo_matrix((v, (r, c)), shape=(5, 5))
    for m in (coo, coo.tocsr(), coo.tocsc(), sps.csr_matrix((v, (r, c)), shape=(5, 5))):
        shape, rowptr, colind, val = to_csr(m)
        assert shape == (5, 5)
        _check_canonical(shape, rowptr, colind, val, dense)
    shape, rowptr, colind, val = to_csr(coo)
    assert val.size == 4                        # (0,1), (2,0) kept although zero, (3,2), (4,4)
    assert list(colind) == [1, 0, 2, 4] and val[1] == 0.0
    assert val[0] == 1.0 and val[2] == 1.75     # duplicates summed
    np.testing.assert_array_equal(_dense(coo), dense)
    assert _dense(coo).flags.f_contiguous


def test_to_csr_spmatrix_standin():
    from cvxopt_b200.kkt import to_csr, is_sparse, _dense
    # 4 x 3, column-compressed; column 1 empty, row 2 empty, column 2 lists row 3 before row 0 and row 0 twice
    sp = SpStandIn(4, 3, [0, 2, 2, 5], [1, 3, 3, 0, 0], [1.0, 2.0, 3.0, 4.0, 0.0])
    assert is_sparse(sp) and not is_sparse(np.zeros((2, 2)))
    dense = np.zeros((4, 3))
    dense[1, 0], dense[3, 0], dense[3, 2], dense[0, 2] = 1.0, 2.0, 3.0, 4.0
    shape, rowptr, colind, val = to_csr(sp)
    assert shape == (4, 3)
    _check_canonical(shape, rowptr, colind, val, dense)
    np.testing.assert_array_equal(_dense(sp), dense)


def test_to_csr_empty():
    from cvxopt_b200.kkt import to_csr
    for m in (sps.csr_matrix((6, 4)), SpStandIn(6, 4, [0, 0, 0, 0, 0], [], [])):
        shape, rowptr, colind, val = to_csr(m)
        assert shape == (6, 4) and val.size == 0 and colind.size == 0
        assert np.array_equal(rowptr, np.zeros(7, dtype=np.int64))


def test_to_csr_refuses_complex_and_bad_indices():
    from cvxopt_b200.kkt import to_csr
    with pytest.raises(TypeError):
        to_csr(sps.csr_matrix(np.array([[1j, 0.0]])))
    with pytest.raises(TypeError):
        to_csr(SpStandIn(2, 2, [0, 1, 1], [5], [1.0]))


def _create(n, dims, rowptr, colind, val, nnz=None, mnl=0):
    from cvxopt_b200 import _lib
    from cvxopt_b200.kkt import make_dims
    lib = _lib.load()
    cd, keep, cdim, _ = make_dims(dims, mnl)
    rp = np.ascontiguousarray(rowptr, dtype=np.int64)
    ci = np.ascontiguousarray(colind, dtype=np.int32)
    v = np.ascontiguousarray(val, dtype=np.float64)
    h = C.c_void_p()
    rc = lib.cvxb_kkt_create_sparse(C.byref(h), n, 0, C.byref(cd), rp.ctypes.data, ci.ctypes.data if ci.size else None,
                                    v.ctypes.data if v.size else None, int(v.size if nnz is None else nnz),
                                    None, 1, _lib.HOST, 0)
    if rc == 0:
        lib.cvxb_kkt_destroy(h)
    return rc, _lib.last_error()


@pytest.mark.parametrize("case,rowptr,colind,nnz,mnl,msg", [
    ("rowptr0", [1, 2, 3], [0, 1, 2], 3, 0, "rowptr[0]"),
    ("monotone", [0, 2, 1], [0, 1], 1, 0, "not monotone"),
    ("end", [0, 1, 2], [0, 1], 3, 0, "differs from nnz"),
    ("col_neg", [0, 1, 2], [0, -1], 2, 0, "outside [0, n"),
    ("col_big", [0, 1, 2], [0, 3], 2, 0, "outside [0, n"),
    ("unsorted", [0, 2, 2], [2, 1], 2, 0, "unsorted"),
    ("duplicate", [0, 2, 2], [1, 1], 2, 0, "duplicate"),
    ("df_rows", [0, 1, 1, 1], [0], 1, 1, "mnl"),
])
def test_create_sparse_refusals(case, rowptr, colind, nnz, mnl, msg):
    """Every malformed CSR is refused with CVXB_E_ARG before the device: the same code with or without a GPU."""
    from cvxopt_b200 import _lib
    rc, err = _create(3, {"l": 2, "q": [], "s": []}, rowptr, colind, np.ones(len(colind)), nnz, mnl)
    assert rc == _lib.E_ARG, (case, rc, err)
    assert msg in err, (case, err)


def test_create_sparse_null_arguments():
    from cvxopt_b200 import _lib
    from cvxopt_b200.kkt import make_dims
    lib = _lib.load()
    cd, keep, _, _ = make_dims({"l": 2, "q": [], "s": []})
    h = C.c_void_p()
    assert lib.cvxb_kkt_create_sparse(C.byref(h), 3, 0, C.byref(cd), None, None, None, 0, None, 1, _lib.HOST, 0) \
        == _lib.E_ARG
    assert "rowptr is NULL" in _lib.last_error()
    rp = np.array([0, 1, 2], dtype=np.int64)
    assert lib.cvxb_kkt_create_sparse(C.byref(h), 3, 0, C.byref(cd), rp.ctypes.data, None, None, 2, None, 1,
                                      _lib.HOST, 0) == _lib.E_ARG
    assert "colind or val is NULL" in _lib.last_error()
    assert lib.cvxb_kkt_create_sparse(None, 3, 0, C.byref(cd), rp.ctypes.data, None, None, 0, None, 1,
                                      _lib.HOST, 0) == _lib.E_ARG


def test_factories_refuse_bad_sparse_shape():
    """A sparse G with the wrong number of rows is refused before the library is asked for a handle."""
    import cvxopt_b200
    with pytest.raises(TypeError, match="G must be"):
        cvxopt_b200.kkt_chol(sps.csr_matrix((5, 3)), {"l": 4, "q": [], "s": []})


def _sparse_G(K, n, density, seed):
    rng = np.random.Generator(np.random.PCG64(seed))
    G = sps.random(K, n, density=density, random_state=np.random.RandomState(seed), format="csc")
    G.data = rng.standard_normal(G.data.size)
    return G


@pytest.mark.parametrize("dims", [{"l": 30, "q": [], "s": []}, {"l": 12, "q": [5, 3], "s": [3]}])
def test_reference_sparse_kkt_chol_matches_oracle_dense(ref, dims):
    """The reference's misc.kkt_chol on an spmatrix G solves the system the oracle solves with the dense G: the
    result the sparse factory is held to."""
    from cvxopt import misc
    n = 9
    K = cone_dim(dims)
    Gs = _sparse_G(K, n, 0.3, seed=4).tocoo()
    Gd = np.asfortranarray(Gs.toarray())
    Gsp = ref.spmatrix(Gs.data.tolist(), Gs.row.tolist(), Gs.col.tolist(), (K, n))
    rng = np.random.Generator(np.random.PCG64(5))
    B = rng.standard_normal((n, n))
    H = np.asfortranarray(B @ B.T + np.eye(n))
    W, _ = random_scaling(dims, seed=6)
    f_or = ko.KktChol(Gd, dims).factor(W, H)
    m = ref.matrix
    Wr = {"d": m(W["d"]), "di": m(W["di"]), "v": [m(v) for v in W["v"]], "beta": list(W["beta"]),
          "r": [m(r) for r in W["r"]], "rti": [m(r) for r in W["rti"]]}
    f_ref = misc.kkt_chol(Gsp, dims, ref.matrix(0.0, (0, n)))(Wr, ref.matrix(H))
    x, z = rng.standard_normal(n), rng.standard_normal(K)
    xr, zr, yr = ref.matrix(x), ref.matrix(z), ref.matrix(0.0, (0, 1))
    f_or(x, None, z)
    f_ref(xr, yr, zr)
    np.testing.assert_allclose(x, np.array(xr).ravel(), rtol=1e-10, atol=1e-12)
    _, _, _, _, cp = ko.cone_sizes(dims)
    a, b = np.zeros(cp), np.zeros(cp)
    ko.pack(z, a, dims)
    ko.pack(np.array(zr).ravel(), b, dims)
    np.testing.assert_allclose(a, b, rtol=1e-10, atol=1e-12)
