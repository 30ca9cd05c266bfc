"""QP batches with 's' blocks without a GPU: cvxb_batch_create_sdp_qp's refusals, each returned before CVXB_E_NOGPU,
and coneqp_batch's TypeErrors and ValueError (coneprog.py:1880-1971) before any batch object exists."""
import ctypes as C

import numpy as np
import pytest

from test_batch_conelp_cpu import _dims, _gpu_visible


@pytest.mark.parametrize("nprob,n,p,dims,code", [
    (2, 4, 0, {"l": 6, "s": [33]}, "E_UNSUP"),      # above CVXB_BATCH_SMAX
    (65536, 4, 0, {"s": [3]}, "E_ARG"),             # nprob > CVXB_BATCH_MAX
    (2, 4, -1, {"s": [3]}, "E_ARG"),                # p < 0
    (2, 4, 5, {"s": [3]}, "E_ARG"),                 # p > n
    (2, 4, 0, {"q": [0], "s": [3]}, "E_ARG"),       # a 'q' order < 1
])
def test_create_sdp_qp_refusals_come_before_the_device_check(nprob, n, p, dims, code):
    from cvxopt_b200 import _lib
    lib = _lib.load()
    h = C.c_void_p()
    if dims.get("q") == [0]:                        # make_dims refuses it; the library must too
        d, keep = _dims({"q": [1], "s": [3]})
        q0 = (C.c_int * 1)(0)
        d.q = C.cast(q0, C.POINTER(C.c_int))
    else:
        d, keep = _dims(dims)
    assert lib.cvxb_batch_create_sdp_qp(C.byref(h), nprob, n, p, C.byref(d), 0) == getattr(_lib, code)
    assert h.value is None
    if code == "E_UNSUP":
        assert "32" in _lib.last_error()
    if p > n:
        assert "Rank(A) < p" in _lib.last_error()


def test_create_sdp_qp_refuses_mnl_and_negative_orders():
    from cvxopt_b200 import _lib
    lib = _lib.load()
    h = C.c_void_p()
    d, keep = _dims({"l": 4, "s": [3]})
    d.mnl = 1
    assert lib.cvxb_batch_create_sdp_qp(C.byref(h), 2, 4, 0, C.byref(d), 0) == _lib.E_ARG
    s = (C.c_int * 2)(3, -1)
    d, keep = _dims({"l": 4, "s": [3, 1]})
    d.s = C.cast(s, C.POINTER(C.c_int))
    assert lib.cvxb_batch_create_sdp_qp(C.byref(h), 2, 4, 0, C.byref(d), 0) == _lib.E_ARG
    assert "< 0" in _lib.last_error()
    assert h.value is None


@pytest.mark.parametrize("n,p,dims", [(4, 0, {"s": [2]}), (8, 1, {"l": 2, "s": [2]}), (50, 3, {"s": [3]})])
def test_create_sdp_qp_has_no_conelp_rank_check(n, p, dims):
    """p + cdim_pckd < n is a cone LP's rank condition (coneprog.py:572-573); coneqp has none, since P may have full
    rank.  Whatever the device, the constructor does not refuse these arguments."""
    from cvxopt_b200 import _lib
    lib = _lib.load()
    h = C.c_void_p()
    d, keep = _dims(dims)
    rc = lib.cvxb_batch_create_sdp_qp(C.byref(h), 2, n, p, C.byref(d), 0)
    if rc == 0:
        lib.cvxb_batch_destroy(h)
    assert rc in (0, _lib.E_NOGPU), (rc, _lib.last_error())


@pytest.mark.skipif(_gpu_visible(), reason="checks the no-GPU return code")
def test_create_sdp_qp_without_gpu_reports_nogpu():
    from cvxopt_b200 import _lib
    lib = _lib.load()
    h = C.c_void_p()
    d, keep = _dims({"l": 6, "q": [3], "s": [3, 0, 32]})
    assert lib.cvxb_batch_create_sdp_qp(C.byref(h), 2, 4, 1, C.byref(d), 0) == _lib.E_NOGPU
    assert h.value is None


def test_create_sdp_qp_is_exported():
    from cvxopt_b200 import exported_symbols
    assert "cvxb_batch_create_sdp_qp" in exported_symbols()


def test_coneqp_batch_argument_errors_before_the_device(monkeypatch):
    import cvxopt_b200
    from cvxopt_b200 import batch

    def no_device(*a, **k):
        raise AssertionError("device work before the argument checks")
    monkeypatch.setattr(batch, "SDPQPBatchGroup", no_device)
    rng = np.random.default_rng(0)
    B, n, dims = 3, 5, {"l": 4, "s": [3]}
    m = 13
    P, q = rng.standard_normal((B, n, n)), rng.standard_normal((B, n))
    G, h = rng.standard_normal((B, m, n)), rng.standard_normal((B, m))
    good = dict(P=P, q=q, G=G, h=h, dims=dims)
    for bad in (dict(P=P[0]), dict(P=P[:, :, :4]), dict(q=q[:, :4]), dict(q=q[:2]), dict(G=G[:, :, :4]),
                dict(G=G[:2]), dict(h=h[:, :12]), dict(G=G[:, :12], h=h[:, :12]),
                dict(dims={"l": 4, "s": [-1]}), dict(dims={"l": 4, "q": [0], "s": [3]}),
                dict(A=np.zeros((B, 1, 4)), b=np.zeros((B, 1))), dict(A=np.zeros((B, 1, n)), b=np.zeros((B, 2))),
                dict(A=np.zeros((B, 1, n))), dict(b=np.zeros((B, 1)))):
        args = dict(good)
        args.update(bad)
        with pytest.raises(TypeError):
            cvxopt_b200.coneqp_batch(**args)
    with pytest.raises(ValueError, match=r"Rank\(A\) < p"):
        cvxopt_b200.coneqp_batch(**good, A=np.zeros((B, 6, n)), b=np.zeros((B, 6)))
