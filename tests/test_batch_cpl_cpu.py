"""cpl batches without a GPU: cpl_batch's argument errors (cvxprog.py:436-530) and its up-front Rank ValueError for
p > n, raised before any batch object exists, the refusal of 's' cones, and cvxb_batch_create_cpl's refusals, each
returned before CVXB_E_NOGPU."""
import ctypes as C

import numpy as np
import pytest

from cpl_problems import cpl_batch_data
from test_batch_conelp_cpu import _gpu_visible


def _no_device(*a, **k):
    raise AssertionError("device work before the argument checks")


@pytest.fixture
def no_groups(monkeypatch):
    from cvxopt_b200 import batch
    monkeypatch.setattr(batch, "CPLBatchGroup", _no_device)


D = cpl_batch_data("socp", [0, 1], 5, [3, 4], 2, 2)
c, X0, G, h, A, b, DIMS = D["c"], D["x0"], D["G"], D["h"], D["A"], D["b"], D["dims"]


def _F(mnl=2, x0=X0):
    def F(x=None, z=None, idx=None):
        if x is None:
            return mnl, x0
        raise AssertionError("F evaluated before the argument checks")
    return F


def _args(**kw):
    a = dict(c=c, F=_F(), G=G, h=h, dims=DIMS, A=A, b=b)
    a.update(kw)
    return a


BAD = [
    dict(F=_F(mnl=-1)), dict(F=_F(mnl=1.0)), dict(F=_F(x0=X0[0])), dict(F=_F(x0=X0.astype(np.float32))),
    dict(c=c[0]), dict(c=c[:, :-1]), dict(c=c.astype(np.float32)),
    dict(h=h[0]), dict(h=h.astype(np.int64)), dict(h=h[:, :-1]), dict(G=None), dict(G=G[:, :, :-1]), dict(G=G[0]),
    dict(dims={"l": 2, "q": [3], "s": []}), dict(A=A[:, :, :-1]), dict(A=A[0]), dict(b=b[:, :-1]),
    dict(b=b[0]), dict(A=None),
]


@pytest.mark.parametrize("kw", BAD)
def test_cpl_batch_type_errors(no_groups, kw):
    import cvxopt_b200
    with pytest.raises(TypeError):
        cvxopt_b200.cpl_batch(**_args(**kw))


@pytest.mark.parametrize("dims,match", [
    ({"l": -1, "q": [3, 4], "s": []}, r"'dims\['l'\]' must be a nonnegative integer"),
    ({"l": 2.0, "q": [3, 4], "s": []}, r"'dims\['l'\]' must be a nonnegative integer"),
    ({"l": 2, "q": [0, 7], "s": []}, r"'dims\['q'\]' must be a list of positive integers"),
    ({"l": 2, "q": [3, 4.0], "s": []}, r"'dims\['q'\]' must be a list of positive integers"),
    ({"l": 2, "q": [3, 4], "s": [-1]}, r"'dims\['s'\]' must be a list of nonnegative integers"),
])
def test_cpl_batch_dims_type_errors(no_groups, dims, match):
    import cvxopt_b200
    with pytest.raises(TypeError, match=match):
        cvxopt_b200.cpl_batch(**_args(dims=dims))


@pytest.mark.parametrize("dims", [{"l": 2, "q": [3, 4]}, {"l": 2, "s": []}])
def test_cpl_batch_missing_dims_key(no_groups, dims):
    """cpl reads dims['q'] and dims['s'] first (cvxprog.py:427): a missing key is its KeyError"""
    import cvxopt_b200
    with pytest.raises(KeyError):
        cvxopt_b200.cpl_batch(**_args(dims=dims))


def test_cpl_batch_rank_error_for_p_above_n(no_groups):
    import cvxopt_b200
    with pytest.raises(ValueError, match=r"Rank\(A\) < p or Rank\(\[H\(x\); A; Df\(x\); G\]\) < n"):
        cvxopt_b200.cpl_batch(**_args(A=np.zeros((2, 6, 5)), b=np.zeros((2, 6))))


def test_cpl_batch_F_call_failure(no_groups):
    import cvxopt_b200

    def F(x=None, z=None, idx=None):
        raise RuntimeError("no start")
    with pytest.raises(ValueError, match=r"function call 'F\(\)' failed"):
        cvxopt_b200.cpl_batch(**_args(F=F))


def test_cpl_batch_refuses_s_cones(no_groups):
    import cvxopt_b200
    dims = dict(DIMS, s=[2])
    with pytest.raises(NotImplementedError):
        cvxopt_b200.cpl_batch(**_args(dims=dims, G=np.zeros((2, 13, 5)), h=np.zeros((2, 13))))


def test_cpl_batch_refuses_no_rows(no_groups):
    import cvxopt_b200
    with pytest.raises(ValueError, match="at least one constraint row"):
        cvxopt_b200.cpl_batch(**_args(F=_F(mnl=0), G=None, h=None, dims=None))


def test_cpl_batch_accepts_q_dims_and_a_tensor_x0(monkeypatch):
    """dims with 'q' cones and a CPU tensor x0 pass the checks: the group is the first thing created"""
    import torch
    import cvxopt_b200
    from cvxopt_b200 import batch
    made = []

    def group(*a, **k):
        made.append(a)
        raise RuntimeError("group")
    monkeypatch.setattr(batch, "CPLBatchGroup", group)
    with pytest.raises(RuntimeError, match="group"):
        cvxopt_b200.cpl_batch(**_args(F=_F(x0=torch.as_tensor(X0))))
    assert made == [(2, 5, 2, DIMS, 2, 0, None)]


def _create(nprob, n, mnl, dims, p):
    from cvxopt_b200 import _lib, kkt
    lib = _lib.load()
    h = C.c_void_p()
    d, keep, _, _ = kkt.make_dims(dict({"l": 0, "q": [], "s": []}, **dims))
    return lib.cvxb_batch_create_cpl(C.byref(h), nprob, n, mnl, C.byref(d), p, 0), h


@pytest.mark.parametrize("nprob,n,mnl,dims,p", [
    (0, 4, 1, {"l": 2}, 0), (65536, 4, 1, {"l": 2}, 0), (2, 0, 1, {"l": 2}, 0), (2, 4, -1, {"l": 2}, 0),
    (2, 4, 1, {"l": 2}, -1), (2, 4, 1, {"l": 2, "q": [3]}, 5), (2, 4, 0, {"l": 0}, 0),
])
def test_create_cpl_refusals_come_before_the_device_check(nprob, n, mnl, dims, p):
    from cvxopt_b200 import _lib
    rc, h = _create(nprob, n, mnl, dims, p)
    assert rc == _lib.E_ARG
    assert h.value is None


def test_create_cpl_refuses_bad_dims_and_s_cones():
    from cvxopt_b200 import _lib
    lib = _lib.load()
    q = (C.c_int * 2)(3, 0)
    s = (C.c_int * 1)(2)
    for mnl_d, ml, nq, ns, code in [(1, 2, 0, 0, _lib.E_ARG), (0, -1, 0, 0, _lib.E_ARG), (0, 2, 2, 0, _lib.E_ARG),
                                    (0, 2, 1, 1, _lib.E_UNSUP)]:
        d = _lib.Dims(mnl_d, ml, nq, C.cast(q, _lib.c_int_p), ns, C.cast(s, _lib.c_int_p))
        h = C.c_void_p()
        assert lib.cvxb_batch_create_cpl(C.byref(h), 2, 4, 1, C.byref(d), 0, 0) == code
        assert h.value is None
    h = C.c_void_p()
    assert lib.cvxb_batch_create_cpl(C.byref(h), 2, 4, 1, None, 0, 0) == _lib.E_ARG
    assert h.value is None


def test_cpl_calls_refuse_a_null_handle():
    from cvxopt_b200 import _lib
    lib = _lib.load()
    assert lib.cvxb_batch_load_cpl(None, None, None, None, None, _lib.HOST) == _lib.E_ARG


@pytest.mark.skipif(_gpu_visible(), reason="checks the no-GPU return code")
@pytest.mark.parametrize("nprob,n,mnl,dims,p", [(2, 4, 1, {"l": 2, "q": [3, 5]}, 0), (1, 4, 0, {"q": [4]}, 4),
                                                (65535, 1, 3, {"l": 0}, 0)])
def test_create_cpl_without_gpu_reports_nogpu(nprob, n, mnl, dims, p):
    from cvxopt_b200 import _lib
    rc, h = _create(nprob, n, mnl, dims, p)
    assert rc == _lib.E_NOGPU
    assert h.value is None
