"""GP batches without a GPU: gp_batch's TypeErrors (cvxprog.py:2056-2092) and its up-front Rank ValueError for p > n,
raised before any batch object exists, and cvxb_batch_create_gp's refusals, each returned before CVXB_E_NOGPU."""
import ctypes as C

import numpy as np
import pytest

from gp_problems import gp_batch_data
from test_batch_conelp_cpu import _gpu_visible


def _no_device(*a, **k):
    raise AssertionError("device work before the argument checks")


@pytest.fixture
def no_groups(monkeypatch):
    from cvxopt_b200 import batch
    monkeypatch.setattr(batch, "GPBatchGroup", _no_device)


K = [4, 3, 2]
F, g, G, h, A, b = gp_batch_data([0, 1], 5, K, r=1, p=2)


def _args(**kw):
    a = dict(K=K, F=F, g=g, G=G, h=h, A=A, b=b)
    a.update(kw)
    return a


BAD = [
    dict(K=(4, 3, 2)), dict(K=[4, 0, 2]), dict(K=[4, 3.0, 2]), dict(K=[4, True, 2]),
    dict(F=F[:, :-1]), dict(F=F[0]), dict(F=F.astype(np.int64)), dict(F=None),
    dict(g=g[:, :-1]), dict(g=g[0]), dict(g=None),
    dict(G=G[:, :, :-1]), dict(G=G[0]),
    dict(h=h[:, :-1]), dict(h=np.zeros((2, G.shape[1] + 1))), dict(G=None),
    dict(A=A[:, :, :-1]), dict(A=A[0]),
    dict(b=b[:, :-1]), dict(A=None),
]


@pytest.mark.parametrize("kw", BAD)
def test_gp_batch_type_errors(no_groups, kw):
    import cvxopt_b200
    with pytest.raises(TypeError):
        cvxopt_b200.gp_batch(**_args(**kw))


def test_gp_batch_rank_error_for_p_above_n(no_groups):
    import cvxopt_b200
    with pytest.raises(ValueError, match=r"Rank\(A\) < p or Rank\(\[H\(x\); A; Df\(x\); G\]\) < n"):
        cvxopt_b200.gp_batch(**_args(A=np.zeros((2, 6, 5)), b=np.zeros((2, 6))))


def _create(nprob, n, Kl, ml, p):
    from cvxopt_b200 import _lib
    lib = _lib.load()
    h = C.c_void_p()
    karr = (C.c_int * max(1, len(Kl)))(*Kl)
    rc = lib.cvxb_batch_create_gp(C.byref(h), nprob, n, len(Kl), karr, ml, p, 0)
    return rc, h


@pytest.mark.parametrize("nprob,n,Kl,ml,p", [
    (0, 4, [3], 2, 0), (65536, 4, [3], 2, 0), (2, 0, [3], 2, 0), (2, 4, [], 2, 0), (2, 4, [3, 0], 2, 0),
    (2, 4, [3, -1, 2], 2, 0), (2, 4, [3], -1, 0), (2, 4, [3], 2, -1), (2, 4, [3], 2, 5),
])
def test_create_gp_refusals_come_before_the_device_check(nprob, n, Kl, ml, p):
    from cvxopt_b200 import _lib
    rc, h = _create(nprob, n, Kl, ml, p)
    assert rc == _lib.E_ARG
    assert h.value is None


def test_gp_calls_refuse_a_null_handle():
    from cvxopt_b200 import _lib
    lib = _lib.load()
    assert lib.cvxb_batch_load_gp(None, None, None, None, None, _lib.HOST) == _lib.E_ARG
    assert lib.cvxb_batch_ls_rounds(None) == _lib.E_ARG


@pytest.mark.skipif(_gpu_visible(), reason="checks the no-GPU return code")
@pytest.mark.parametrize("nprob,n,Kl,ml,p", [(2, 4, [3], 2, 0), (1, 4, [3, 2, 2], 0, 4), (65535, 1, [1], 0, 0)])
def test_create_gp_without_gpu_reports_nogpu(nprob, n, Kl, ml, p):
    from cvxopt_b200 import _lib
    rc, h = _create(nprob, n, Kl, ml, p)
    assert rc == _lib.E_NOGPU
    assert h.value is None
