"""cpl batches with 's' blocks without a GPU: sdp_cpl_batch's argument errors, raised before any batch object exists,
its acceptance of 's' dims, the order-33 refusal from the create call, and cvxb_batch_create_sdp_cpl's refusals, each
returned before CVXB_E_NOGPU."""
import ctypes as C

import numpy as np
import pytest

from sdcpl_problems import sdcpl_batch_data
from test_batch_conelp_cpu import _gpu_visible
from test_batch_cpl_cpu import _F


def _no_device(*a, **k):
    raise AssertionError("device work before the argument checks")


@pytest.fixture
def no_groups(monkeypatch):
    from cvxopt_b200 import batch
    monkeypatch.setattr(batch, "SDPCPLBatchGroup", _no_device)


D = sdcpl_batch_data("socp", [0, 1], 5, [3, 4], [2, 3], 2, 2)
c, X0, G, h, A, b, DIMS = D["c"], D["x0"], D["G"], D["h"], D["A"], D["b"], D["dims"]


def _args(**kw):
    a = dict(c=c, F=_F(x0=X0), G=G, h=h, dims=DIMS, A=A, b=b)
    a.update(kw)
    return a


BAD = [
    dict(F=_F(mnl=-1, x0=X0)), dict(F=_F(mnl=1.0, x0=X0)), dict(F=_F(x0=X0[0])), dict(F=_F(x0=X0.astype(np.float32))),
    dict(c=c[0]), dict(c=c[:, :-1]), dict(c=c.astype(np.float32)),
    dict(h=h[0]), dict(h=h.astype(np.int64)), dict(h=h[:, :-1]), dict(G=None), dict(G=G[:, :, :-1]), dict(G=G[0]),
    dict(G=G[:, :-4]), dict(dims={"l": 2, "q": [3, 4], "s": [3, 2, 1]}), dict(dims={"l": 2, "q": [3, 4], "s": [2]}),
    dict(A=A[:, :, :-1]), dict(A=A[0]), dict(b=b[:, :-1]), dict(b=b[0]), dict(A=None),
]


@pytest.mark.parametrize("kw", BAD)
def test_sdp_cpl_batch_type_errors(no_groups, kw):
    """cpl_batch's TypeErrors on data with 's' rows, including dims whose 's' rows do not match G and h"""
    import cvxopt_b200
    with pytest.raises(TypeError):
        cvxopt_b200.sdp_cpl_batch(**_args(**kw))


@pytest.mark.parametrize("dims,match", [
    ({"l": 2, "q": [3, 4], "s": [-1, 3]}, r"'dims\['s'\]' must be a list of nonnegative integers"),
    ({"l": 2, "q": [3, 4], "s": [2, 3.0]}, r"'dims\['s'\]' must be a list of nonnegative integers"),
    ({"l": -1, "q": [3, 4], "s": [2, 3]}, r"'dims\['l'\]' must be a nonnegative integer"),
    ({"l": 2, "q": [0, 7], "s": [2, 3]}, r"'dims\['q'\]' must be a list of positive integers"),
])
def test_sdp_cpl_batch_dims_type_errors(no_groups, dims, match):
    import cvxopt_b200
    with pytest.raises(TypeError, match=match):
        cvxopt_b200.sdp_cpl_batch(**_args(dims=dims))


@pytest.mark.parametrize("dims", [{"l": 2, "q": [3, 4]}, {"l": 2, "s": [2, 3]}])
def test_sdp_cpl_batch_missing_dims_key(no_groups, dims):
    import cvxopt_b200
    with pytest.raises(KeyError):
        cvxopt_b200.sdp_cpl_batch(**_args(dims=dims))


def test_sdp_cpl_batch_rank_and_row_errors(no_groups):
    import cvxopt_b200
    with pytest.raises(ValueError, match=r"Rank\(A\) < p or Rank\(\[H\(x\); A; Df\(x\); G\]\) < n"):
        cvxopt_b200.sdp_cpl_batch(**_args(A=np.zeros((2, 6, 5)), b=np.zeros((2, 6))))
    with pytest.raises(ValueError, match="at least one constraint row"):
        cvxopt_b200.sdp_cpl_batch(**_args(F=_F(mnl=0, x0=X0), G=None, h=None, dims={"l": 0, "q": [], "s": [0]}))

    def F(x=None, z=None, idx=None):
        raise RuntimeError("no start")
    with pytest.raises(ValueError, match=r"function call 'F\(\)' failed"):
        cvxopt_b200.sdp_cpl_batch(**_args(F=F))


def test_sdp_cpl_batch_accepts_s_dims(monkeypatch):
    """dims with 's' blocks pass the checks: the group is the first thing created, with them"""
    import cvxopt_b200
    from cvxopt_b200 import batch
    made = []

    def group(*a, **k):
        made.append(a)
        raise RuntimeError("group")
    monkeypatch.setattr(batch, "SDPCPLBatchGroup", group)
    with pytest.raises(RuntimeError, match="group"):
        cvxopt_b200.sdp_cpl_batch(**_args())
    assert made == [(2, 5, 2, DIMS, 2, 0, None)]


def test_order_33_is_refused_by_the_create_call():
    """an order above 32 passes the Python checks and is refused by cvxb_batch_create_sdp_cpl (CVXB_E_UNSUP) before
    it looks for a device"""
    import cvxopt_b200
    d = sdcpl_batch_data("conelp", [0, 1], 4, [], [33], 1, 0)
    F = _F(mnl=0, x0=d["x0"])
    with pytest.raises(NotImplementedError, match=r"dims\['s'\]\[0\] = 33 > 32"):
        cvxopt_b200.sdp_cpl_batch(d["c"], F, d["G"], d["h"], d["dims"])


def _create(nprob, n, mnl, dims, p):
    from cvxopt_b200 import _lib, kkt
    lib = _lib.load()
    h = C.c_void_p()
    d, keep, _, _ = kkt.make_dims(dict({"l": 0, "q": [], "s": []}, **dims))
    return lib.cvxb_batch_create_sdp_cpl(C.byref(h), nprob, n, mnl, C.byref(d), p, 0), h


@pytest.mark.parametrize("nprob,n,mnl,dims,p", [
    (0, 4, 1, {"s": [2]}, 0), (65536, 4, 1, {"s": [2]}, 0), (2, 0, 1, {"s": [2]}, 0), (2, 4, -1, {"s": [2]}, 0),
    (2, 4, 1, {"s": [2]}, -1), (2, 4, 1, {"l": 2, "s": [3]}, 5), (2, 4, 0, {"l": 0, "s": [0, 0]}, 0),
])
def test_create_sdp_cpl_refusals_come_before_the_device_check(nprob, n, mnl, dims, p):
    from cvxopt_b200 import _lib
    rc, h = _create(nprob, n, mnl, dims, p)
    assert rc == _lib.E_ARG
    assert h.value is None


def test_create_sdp_cpl_refuses_bad_dims_and_orders():
    from cvxopt_b200 import _lib
    lib = _lib.load()
    q = (C.c_int * 2)(3, 0)
    for mnl_d, ml, nq, s, code in [(1, 2, 0, [2], _lib.E_ARG), (0, -1, 0, [2], _lib.E_ARG),
                                   (0, 2, 2, [2], _lib.E_ARG), (0, 2, 0, [2, -1], _lib.E_ARG),
                                   (0, 2, 1, [33], _lib.E_UNSUP), (0, 2, 0, [4, 40], _lib.E_UNSUP)]:
        sa = (C.c_int * len(s))(*s)
        d = _lib.Dims(mnl_d, ml, nq, C.cast(q, _lib.c_int_p), len(s), C.cast(sa, _lib.c_int_p))
        h = C.c_void_p()
        assert lib.cvxb_batch_create_sdp_cpl(C.byref(h), 2, 4, 1, C.byref(d), 0, 0) == code, (mnl_d, ml, nq, s)
        assert h.value is None
    d = _lib.Dims(0, 2, 0, C.cast(q, _lib.c_int_p), 1, None)              # ns > 0 without the orders
    h = C.c_void_p()
    assert lib.cvxb_batch_create_sdp_cpl(C.byref(h), 2, 4, 1, C.byref(d), 0, 0) == _lib.E_ARG
    assert lib.cvxb_batch_create_sdp_cpl(C.byref(h), 2, 4, 1, None, 0, 0) == _lib.E_ARG
    assert h.value is None


@pytest.mark.skipif(_gpu_visible(), reason="checks the no-GPU return code")
@pytest.mark.parametrize("nprob,n,mnl,dims,p", [(2, 4, 1, {"l": 2, "q": [3, 5], "s": [2, 0, 32]}, 0),
                                                (1, 4, 0, {"s": [4]}, 4), (3, 5, 2, {"s": [0]}, 1),
                                                (65535, 1, 3, {"l": 0, "s": [1]}, 0)])
def test_create_sdp_cpl_without_gpu_reports_nogpu(nprob, n, mnl, dims, p):
    from cvxopt_b200 import _lib
    rc, h = _create(nprob, n, mnl, dims, p)
    assert rc == _lib.E_NOGPU
    assert h.value is None
