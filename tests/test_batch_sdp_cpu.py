"""SDP batches without a GPU: cvxb_batch_create_sdp's refusals, each returned before CVXB_E_NOGPU, and sdp_batch's
TypeErrors and ValueError (coneprog.py:3846-3888, :572-573) before any batch object exists."""
import ctypes as C

import numpy as np
import pytest

from test_batch_conelp_cpu import _dims, _gpu_visible


@pytest.mark.parametrize("nprob,n,p,dims,code", [
    (2, 4, 0, {"l": 6, "s": [33]}, "E_UNSUP"),      # above CVXB_BATCH_SMAX
    (65536, 4, 0, {"s": [3]}, "E_ARG"),             # nprob > CVXB_BATCH_MAX
    (2, 4, -1, {"s": [3]}, "E_ARG"),                # p < 0
    (2, 4, 5, {"s": [3]}, "E_ARG"),                 # p > n
    (2, 4, 0, {"s": [2]}, "E_ARG"),                 # cdim = 4 >= n but cdim_pckd = 3 < n
    (2, 8, 1, {"l": 2, "s": [2]}, "E_ARG"),         # p + cdim_pckd < n
])
def test_create_sdp_refusals_come_before_the_device_check(nprob, n, p, dims, code):
    from cvxopt_b200 import _lib
    lib = _lib.load()
    h = C.c_void_p()
    d, keep = _dims(dims)
    assert lib.cvxb_batch_create_sdp(C.byref(h), nprob, n, p, C.byref(d), 0) == getattr(_lib, code)
    assert h.value is None
    if code == "E_UNSUP":
        assert "32" in _lib.last_error()
    if dims.get("s") == [2]:
        assert "Rank(A) < p or Rank([G; A]) < n" in _lib.last_error()


def test_create_sdp_refuses_mnl_and_negative_orders():
    from cvxopt_b200 import _lib
    lib = _lib.load()
    h = C.c_void_p()
    d, keep = _dims({"l": 4, "s": [3]})
    d.mnl = 1
    assert lib.cvxb_batch_create_sdp(C.byref(h), 2, 4, 0, C.byref(d), 0) == _lib.E_ARG
    s = (C.c_int * 2)(3, -1)
    d, keep = _dims({"l": 4, "s": [3, 1]})
    d.s = C.cast(s, C.POINTER(C.c_int))
    assert lib.cvxb_batch_create_sdp(C.byref(h), 2, 4, 0, C.byref(d), 0) == _lib.E_ARG
    assert "< 0" in _lib.last_error()


@pytest.mark.skipif(_gpu_visible(), reason="checks the no-GPU return code")
def test_create_sdp_without_gpu_reports_nogpu():
    from cvxopt_b200 import _lib
    lib = _lib.load()
    h = C.c_void_p()
    d, keep = _dims({"l": 6, "s": [3, 0, 32]})
    assert lib.cvxb_batch_create_sdp(C.byref(h), 2, 4, 1, C.byref(d), 0) == _lib.E_NOGPU


def test_create_sdp_is_exported():
    from cvxopt_b200 import exported_symbols
    assert "cvxb_batch_create_sdp" in exported_symbols()


def test_sdp_batch_argument_errors_before_the_device(monkeypatch):
    import cvxopt_b200
    from cvxopt_b200 import batch

    def no_device(*a, **k):
        raise AssertionError("device work before the argument checks")
    monkeypatch.setattr(batch, "SDPBatchGroup", no_device)
    rng = np.random.default_rng(0)
    B, n = 3, 5
    c, Gl, hl = rng.standard_normal((B, n)), rng.standard_normal((B, 4, n)), rng.standard_normal((B, 4))
    Gs, hs = [rng.standard_normal((B, 9, n))], [rng.standard_normal((B, 3, 3))]
    good = dict(c=c, Gl=Gl, hl=hl, Gs=Gs, hs=hs)
    for bad in (dict(c=c[0]), dict(Gl=Gl[:, :, :2]), dict(hl=hl[:, :3]), dict(Gs=Gs[0]), dict(Gs=[Gs[0][:, :8]]),
                dict(hs=hs + hs), dict(hs=[hs[0][:, :2]]), dict(Gs=[Gs[0][:2]]),
                dict(A=np.zeros((B, 1, 4)), b=np.zeros((B, 1))), dict(A=np.zeros((B, 1, n)), b=np.zeros((B, 2)))):
        args = dict(good)
        args.update(bad)
        with pytest.raises(TypeError):
            cvxopt_b200.sdp_batch(**args)
    with pytest.raises(ValueError, match=r"Rank\(A\) < p or Rank\(\[G; A\]\) < n"):
        cvxopt_b200.sdp_batch(**good, A=np.zeros((B, 6, n)), b=np.zeros((B, 6)))
    # cdim = 4 >= n = 4 but cdim_pckd = 3 < n
    with pytest.raises(ValueError, match=r"Rank\(A\) < p"):
        cvxopt_b200.sdp_batch(np.zeros((B, 4)), Gs=[np.zeros((B, 4, 4))], hs=[np.zeros((B, 2, 2))])
