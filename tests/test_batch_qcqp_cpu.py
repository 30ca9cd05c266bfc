"""QCQP batches without a GPU: qcqp_batch's argument errors (cp's wording for G, h, dims, A and b, raised before any
batch object exists), the refusal of 'q' and 's' cones, the up-front Rank ValueError for p > n, and
cvxb_batch_create_qcqp's and cvxb_batch_load_qcqp's refusals, each returned before the device."""
import ctypes as C

import numpy as np
import pytest

from qcqp_problems import qcqp_batch_data
from test_batch_conelp_cpu import _gpu_visible


def _no_device(*a, **k):
    raise AssertionError("device work before the argument checks")


@pytest.fixture
def no_groups(monkeypatch):
    from cvxopt_b200 import batch
    monkeypatch.setattr(batch, "QCQPBatchGroup", _no_device)


D = qcqp_batch_data([0, 1], 5, 2, p=2, r=3)


def _args(**kw):
    a = {k: D[k] for k in ("P", "q", "r", "G", "h", "A", "b", "x0")}
    a.update(kw)
    return a


P, q, r, X0, G, h, A, b = (D[k] for k in ("P", "q", "r", "x0", "G", "h", "A", "b"))
BAD = [
    dict(P=P[0]), dict(P=P[:, :, :, :-1]), dict(P=P[:, :0]), dict(P=P.astype(np.int64)), dict(P=None),
    dict(q=q[:, :-1]), dict(q=q[..., :-1]), dict(q=q.astype(np.int64)),
    dict(r=r[:, :-1]), dict(r=r[0]), dict(r=r.astype(np.int64)),
    dict(x0=X0[0]), dict(x0=X0[:, :-1]), dict(x0=X0.astype(np.int64)),
    dict(h=h[0]), dict(h=h.astype(np.int64)), dict(h=h[:, :-1]), dict(G=None), dict(G=G[:, :, :-1]), dict(G=G[0]),
    dict(dims={"l": 2}), dict(A=A[:, :, :-1]), dict(A=A[0]), dict(b=b[:, :-1]), dict(b=b[0]), dict(A=None),
]


@pytest.mark.parametrize("kw", BAD)
def test_qcqp_batch_type_errors(no_groups, kw):
    import cvxopt_b200
    with pytest.raises(TypeError):
        cvxopt_b200.qcqp_batch(**_args(**kw))


def test_qcqp_batch_rank_error_for_p_above_n(no_groups):
    import cvxopt_b200
    with pytest.raises(ValueError, match=r"Rank\(A\) < p or Rank\(\[H\(x\); A; Df\(x\); G\]\) < n"):
        cvxopt_b200.qcqp_batch(**_args(A=np.zeros((2, 6, 5)), b=np.zeros((2, 6))))


@pytest.mark.parametrize("dims", [{"l": 13, "q": [2], "s": []}, {"l": 13, "q": [], "s": [2]}])
def test_qcqp_batch_refuses_cones(no_groups, dims):
    import cvxopt_b200
    with pytest.raises(NotImplementedError):
        cvxopt_b200.qcqp_batch(**_args(dims=dims))


def test_qcqp_batch_defaults_reach_the_group(monkeypatch):
    """dims {'l': ml}, x0 = None and no A, b pass the checks: the group is the first thing created"""
    import cvxopt_b200
    from cvxopt_b200 import batch
    made = []

    def group(*a, **k):
        made.append(a)
        raise RuntimeError("group")
    monkeypatch.setattr(batch, "QCQPBatchGroup", group)
    with pytest.raises(RuntimeError, match="group"):
        cvxopt_b200.qcqp_batch(**_args(x0=None, A=None, b=None, dims={"l": 13, "q": [], "s": []}))
    assert made == [(2, 5, 2, 13, 0, 0, None)]


def _create(nprob, n, mnl, ml, p):
    from cvxopt_b200 import _lib
    lib = _lib.load()
    hd = C.c_void_p()
    return lib.cvxb_batch_create_qcqp(C.byref(hd), nprob, n, mnl, ml, p, 0), hd


@pytest.mark.parametrize("nprob,n,mnl,ml,p", [
    (0, 4, 1, 2, 0), (65536, 4, 1, 2, 0), (2, 0, 1, 2, 0), (2, 4, -1, 2, 0), (2, 4, 1, -1, 0), (2, 4, 1, 2, -1),
    (2, 4, 1, 2, 5), (2, 1 << 20, 1023, 0, 0), (2, 4, 1 << 30, 0, 0),
])
def test_create_qcqp_refusals_come_before_the_device_check(nprob, n, mnl, ml, p):
    from cvxopt_b200 import _lib
    rc, hd = _create(nprob, n, mnl, ml, p)
    assert rc == _lib.E_ARG
    assert hd.value is None
    assert "batch_create_qcqp" in _lib.last_error()


def test_qcqp_calls_refuse_a_null_handle():
    from cvxopt_b200 import _lib
    lib = _lib.load()
    v = np.zeros(8)
    a = v.ctypes.data
    assert lib.cvxb_batch_load_qcqp(None, a, a, a, a, a, a, _lib.HOST) == _lib.E_ARG
    assert "NULL argument" in _lib.last_error()


@pytest.mark.skipif(_gpu_visible(), reason="checks the no-GPU return code")
@pytest.mark.parametrize("nprob,n,mnl,ml,p", [(2, 4, 1, 2, 0), (1, 4, 0, 0, 4), (65535, 1, 3, 0, 0),
                                             (2, 1, (1 << 29) - 8, 0, 0)])     # no host buffer of mnl entries
def test_create_qcqp_without_gpu_reports_nogpu(nprob, n, mnl, ml, p):
    from cvxopt_b200 import _lib
    rc, hd = _create(nprob, n, mnl, ml, p)
    assert rc == _lib.E_NOGPU
    assert hd.value is None


def test_deficient_family_is_exactly_singular():
    """the deficient objective's last p rows and columns are exactly zero: a Cholesky of P_0 fails whatever its
    summation order, so a solve takes the S + A'A switch at iteration 0"""
    from qcqp_problems import qcqp_batch_data, sym
    for seeds, n, p in ((range(8), 10, 3), (range(100, 110), 12, 4)):
        d = qcqp_batch_data(seeds, n, 0, p, 0, "deficient")
        for P, A in zip(d["P"], d["A"]):
            P0 = sym(P)[0]
            assert not P0[n - p:].any() and not P0[:, n - p:].any()
            with pytest.raises(np.linalg.LinAlgError):
                np.linalg.cholesky(P0)
            assert np.linalg.matrix_rank(np.vstack([P0, A])) == n
