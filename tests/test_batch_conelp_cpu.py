"""Cone LP batches without a GPU: cvxb_batch_create_lp's refusals, each returned before CVXB_E_NOGPU, and
conelp_batch's TypeErrors and ValueError (coneprog.py:487-573) before any batch object exists."""
import ctypes as C

import numpy as np
import pytest


def _gpu_visible():
    try:
        from cvxopt_b200 import _lib
        return _lib.load().cvxb_device_count() > 0
    except Exception:
        return False


def _dims(d):
    from cvxopt_b200 import kkt
    full = {"l": d.get("l", 0), "q": list(d.get("q", [])), "s": list(d.get("s", []))}
    dd, keep, _, _ = kkt.make_dims(full)
    return dd, keep


@pytest.mark.parametrize("nprob,n,p,dims,code", [
    (2, 4, -1, {"l": 6}, "E_ARG"),                  # p < 0
    (2, 4, 5, {"l": 6}, "E_ARG"),                   # p > n
    (2, 8, 1, {"l": 6}, "E_ARG"),                   # p + cdim < n
    (2, 4, 0, {"l": 0}, "E_ARG"),                   # m = 0
    (65536, 4, 0, {"l": 6}, "E_ARG"),               # nprob > CVXB_BATCH_MAX
    (0, 4, 0, {"l": 6}, "E_ARG"),
    (2, 0, 0, {"l": 6}, "E_ARG"),
    (2, 4, 0, {"l": 6, "s": [2]}, "E_UNSUP"),       # 's' cones
])
def test_create_lp_refusals_come_before_the_device_check(nprob, n, p, dims, code):
    from cvxopt_b200 import _lib
    lib = _lib.load()
    h = C.c_void_p()
    d, keep = _dims(dims)
    assert lib.cvxb_batch_create_lp(C.byref(h), nprob, n, p, C.byref(d), 0) == getattr(_lib, code)
    assert h.value is None
    if (n, p) in ((4, 5), (8, 1)):
        assert "Rank(A) < p or Rank([G; A]) < n" in _lib.last_error()


def test_create_lp_refuses_bad_dims_before_the_device_check():
    from cvxopt_b200 import _lib
    lib = _lib.load()
    h = C.c_void_p()
    d, keep = _dims({"l": 4, "q": [3]})
    d.mnl = 1
    assert lib.cvxb_batch_create_lp(C.byref(h), 2, 4, 0, C.byref(d), 0) == _lib.E_ARG
    q = (C.c_int * 2)(3, 0)                          # a 'q' order below 1
    d, keep = _dims({"l": 4, "q": [3, 1]})
    d.q = C.cast(q, C.POINTER(C.c_int))
    assert lib.cvxb_batch_create_lp(C.byref(h), 2, 4, 0, C.byref(d), 0) == _lib.E_ARG
    assert "< 1" in _lib.last_error()
    assert lib.cvxb_batch_create_lp(C.byref(h), 2, 4, 0, None, 0) == _lib.E_ARG


@pytest.mark.skipif(_gpu_visible(), reason="checks the no-GPU return code")
def test_create_lp_without_gpu_reports_nogpu():
    from cvxopt_b200 import _lib
    lib = _lib.load()
    h = C.c_void_p()
    d, keep = _dims({"l": 6, "q": [3]})
    assert lib.cvxb_batch_create_lp(C.byref(h), 2, 4, 1, C.byref(d), 0) == _lib.E_NOGPU


def test_load_lp_and_solve_refuse_a_null_handle():
    from cvxopt_b200 import _lib
    lib = _lib.load()
    x = np.zeros(4)
    assert lib.cvxb_batch_load_lp(None, x.ctypes.data, x.ctypes.data, x.ctypes.data, _lib.HOST) == _lib.E_ARG


def _lp(B=3, n=4, m=6, p=1, seed=0):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal((B, n)), rng.standard_normal((B, m, n)), rng.standard_normal((B, m)),
            rng.standard_normal((B, p, n)), rng.standard_normal((B, p)))


def test_conelp_batch_argument_errors_before_the_device(monkeypatch):
    import cvxopt_b200
    from cvxopt_b200 import batch

    def no_device(*a, **k):
        raise AssertionError("device work before the argument checks")
    monkeypatch.setattr(batch, "ConeLPBatchGroup", no_device)
    c, G, h, A, b = _lp()
    for bad in (dict(c=c[0]), dict(h=h[:, :5]), dict(G=G[:, :, :3]), dict(G=G[:2]), dict(G=G[0])):
        args = dict(c=c, G=G, h=h)
        args.update(bad)
        with pytest.raises(TypeError):
            cvxopt_b200.conelp_batch(**args)
    with pytest.raises(TypeError, match=r"size \(7,1\)"):
        cvxopt_b200.conelp_batch(c, G, h, dims={"l": 4, "q": [3]})
    for eq in (dict(A=A), dict(b=b), dict(A=A[:, :, :3], b=b), dict(A=A, b=b[:, :0]), dict(A=A[:2], b=b)):
        with pytest.raises(TypeError):
            cvxopt_b200.conelp_batch(c, G, h, **eq)
    with pytest.raises(NotImplementedError):
        cvxopt_b200.conelp_batch(c, G, h, dims={"l": 2, "s": [2]})
    # p > n and p + cdim < n: conelp's ValueError before the first factorisation
    A5, b5 = np.zeros((3, 5, 4)), np.zeros((3, 5))
    with pytest.raises(ValueError, match=r"Rank\(A\) < p or Rank\(\[G; A\]\) < n"):
        cvxopt_b200.conelp_batch(c, G, h, A=A5, b=b5)
    with pytest.raises(ValueError, match=r"Rank\(A\) < p"):
        cvxopt_b200.conelp_batch(np.zeros((3, 9)), np.zeros((3, 6, 9)), h, A=np.zeros((3, 2, 9)), b=np.zeros((3, 2)))


def test_status_codes_of_the_certificates():
    from cvxopt_b200 import batch
    assert batch.STATUS[4] == "primal infeasible" and batch.STATUS[5] == "dual infeasible"
    assert [batch.STATUS[k] for k in range(4)] == ["running", "optimal", "unknown", "unknown"]
