"""CP batches without a GPU: cp_batch's argument errors (cvxprog.py:1653-1728) and its up-front Rank ValueError for
p > n, raised before any batch object exists, the refusal of 'q' and 's' cones, and cvxb_batch_create_cp's refusals,
each returned before CVXB_E_NOGPU."""
import ctypes as C

import numpy as np
import pytest

from cp_problems import cp_batch_data
from test_batch_conelp_cpu import _gpu_visible


def _no_device(*a, **k):
    raise AssertionError("device work before the argument checks")


@pytest.fixture
def no_groups(monkeypatch):
    from cvxopt_b200 import batch
    monkeypatch.setattr(batch, "CPBatchGroup", _no_device)


D = cp_batch_data("entropy", [0, 1], 5, p=2, r=3)
X0, G, h, A, b = D["x0"], D["G"], D["h"], D["A"], D["b"]


def _F(mnl=0, x0=X0):
    def F(x=None, z=None, idx=None):
        if x is None:
            return mnl, x0
        raise AssertionError("F evaluated before the argument checks")
    return F


def _args(**kw):
    a = dict(F=_F(), G=G, h=h, A=A, b=b)
    a.update(kw)
    return a


BAD = [
    dict(F=_F(mnl=-1)), dict(F=_F(mnl=1.0)), dict(F=_F(x0=X0[0])), dict(F=_F(x0=X0.astype(np.float32))),
    dict(F=_F(x0=X0.astype(np.int64))),
    dict(h=h[0]), dict(h=h.astype(np.int64)), dict(h=h[:, :-1]), dict(G=None), dict(G=G[:, :, :-1]), dict(G=G[0]),
    dict(dims={"l": 2}), dict(A=A[:, :, :-1]), dict(A=A[0]), dict(b=b[:, :-1]), dict(b=b[0]), dict(A=None),
]


@pytest.mark.parametrize("kw", BAD)
def test_cp_batch_type_errors(no_groups, kw):
    import cvxopt_b200
    with pytest.raises(TypeError):
        cvxopt_b200.cp_batch(**_args(**kw))


def test_cp_batch_rank_error_for_p_above_n(no_groups):
    import cvxopt_b200
    with pytest.raises(ValueError, match=r"Rank\(A\) < p or Rank\(\[H\(x\); A; Df\(x\); G\]\) < n"):
        cvxopt_b200.cp_batch(**_args(A=np.zeros((2, 6, 5)), b=np.zeros((2, 6))))


def test_cp_batch_F_call_failure(no_groups):
    import cvxopt_b200

    def F(x=None, z=None, idx=None):
        raise RuntimeError("no start")
    with pytest.raises(ValueError, match=r"function call 'F\(\)' failed"):
        cvxopt_b200.cp_batch(**_args(F=F))


@pytest.mark.parametrize("dims", [{"l": 3, "q": [2], "s": []}, {"l": 3, "q": [], "s": [2]}])
def test_cp_batch_refuses_cones(no_groups, dims):
    import cvxopt_b200
    with pytest.raises(NotImplementedError):
        cvxopt_b200.cp_batch(**_args(dims=dims))


def test_cp_batch_accepts_l_dims_and_a_tensor_x0(monkeypatch):
    """dims {'l': ml} and a CPU tensor x0 pass the checks: the group is the first thing created"""
    import torch
    import cvxopt_b200
    from cvxopt_b200 import batch
    made = []

    def group(*a, **k):
        made.append(a)
        raise RuntimeError("group")
    monkeypatch.setattr(batch, "CPBatchGroup", group)
    with pytest.raises(RuntimeError, match="group"):
        cvxopt_b200.cp_batch(**_args(F=_F(x0=torch.as_tensor(X0)), dims={"l": 3, "q": [], "s": []}))
    assert made == [(2, 5, 0, 3, 2, 0, None)]


def _create(nprob, n, mnl, ml, p):
    from cvxopt_b200 import _lib
    lib = _lib.load()
    h = C.c_void_p()
    return lib.cvxb_batch_create_cp(C.byref(h), nprob, n, mnl, ml, p, 0), h


@pytest.mark.parametrize("nprob,n,mnl,ml,p", [
    (0, 4, 1, 2, 0), (65536, 4, 1, 2, 0), (2, 0, 1, 2, 0), (2, 4, -1, 2, 0), (2, 4, 1, -1, 0), (2, 4, 1, 2, -1),
    (2, 4, 1, 2, 5),
])
def test_create_cp_refusals_come_before_the_device_check(nprob, n, mnl, ml, p):
    from cvxopt_b200 import _lib
    rc, h = _create(nprob, n, mnl, ml, p)
    assert rc == _lib.E_ARG
    assert h.value is None


def test_cp_calls_refuse_a_null_handle():
    from cvxopt_b200 import _lib
    lib = _lib.load()
    assert lib.cvxb_batch_load_cp(None, None, None, None, _lib.HOST) == _lib.E_ARG
    assert lib.cvxb_batch_set_cp_eval(None, None, None) == _lib.E_ARG
    assert lib.cvxb_batch_ls_rounds(None) == _lib.E_ARG


@pytest.mark.skipif(_gpu_visible(), reason="checks the no-GPU return code")
@pytest.mark.parametrize("nprob,n,mnl,ml,p", [(2, 4, 1, 2, 0), (1, 4, 0, 0, 4), (65535, 1, 3, 0, 0)])
def test_create_cp_without_gpu_reports_nogpu(nprob, n, mnl, ml, p):
    from cvxopt_b200 import _lib
    rc, h = _create(nprob, n, mnl, ml, p)
    assert rc == _lib.E_NOGPU
    assert h.value is None
