"""CPU-only: the C-ABI library loads and exports every symbol include/cvxopt_b200.h declares."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    txt = open(os.path.join(ROOT, "include", "cvxopt_b200.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(cvxb_[A-Za-z0-9_]+)\s*\(", txt)))


def test_library_exports_every_declared_symbol():
    import ctypes
    from cvxopt_b200 import _lib
    assert os.path.exists(_lib.LIB_PATH), "build with `make` (or __graft_entry__.build())"
    lib = ctypes.CDLL(_lib.LIB_PATH)
    syms = header_symbols()
    assert len(syms) >= 30
    for s in syms:
        assert hasattr(lib, s), "symbol %s declared in the header but not exported" % s
    # and the ctypes signature table covers exactly the header
    assert sorted(_lib.exported_symbols()) == syms


def test_no_cpu_fallback():
    """Without a GPU every compute entry point must fail loudly, never fall back."""
    import numpy as np
    import cvxopt_b200
    from cvxopt_b200 import _lib, misc_solvers as ms, scaling
    if cvxopt_b200.device_count() > 0:
        pytest.skip("a GPU is visible")
    with pytest.raises(RuntimeError):
        cvxopt_b200.kkt_chol(np.zeros((4, 2), order="F"), {"l": 4, "q": [], "s": []})
    # the entry points without a handle check for the device before they touch it
    dims = {"l": 2, "q": [3], "s": [2]}           # cdim 9, packed 8, lmbda 7
    W = {"d": np.ones(2), "di": np.ones(2), "v": [np.array([1.0, 0.0, 0.0])], "beta": [1.0],
         "r": [np.eye(2, order="F")], "rti": [np.eye(2, order="F")]}
    calls = [
        lambda: ms.scale(np.ones(9), W), lambda: ms.scale2(np.ones(7), np.ones(9), dims),
        lambda: ms.pack(np.ones(9), np.zeros(8), dims), lambda: ms.unpack(np.ones(8), np.zeros(9), dims),
        lambda: ms.pack2(np.ones(9), dims), lambda: ms.symm(np.ones(4), 2),
        lambda: ms.sprod(np.ones(9), np.ones(9), dims), lambda: ms.sinv(np.ones(9), np.ones(7), dims),
        lambda: ms.trisc(np.ones(9), dims), lambda: ms.triusc(np.ones(9), dims),
        lambda: ms.sdot(np.ones(9), np.ones(9), dims), lambda: ms.max_step(np.ones(9), dims),
        lambda: scaling.compute_scaling(np.ones(9), np.ones(9), np.zeros(7), dims),
        lambda: scaling.update_scaling(W, np.ones(7), np.ones(9), np.ones(9)),
    ]
    for call in calls:
        with pytest.raises(RuntimeError, match="no CUDA device available"):
            call()
    lib = _lib.load()
    a, c, inv = np.eye(2, order="F"), np.zeros((2, 2), order="F"), np.zeros(2 * 128 * 128)
    assert lib.cvxb_potrf(2, a.ctypes.data, 2, inv.ctypes.data, 0) == _lib.E_NOGPU
    assert "no CUDA device available" in _lib.last_error()
    assert lib.cvxb_gemm(ord("N"), ord("N"), 2, 2, 2, 1.0, a.ctypes.data, 2, a.ctypes.data, 2, 0.0,
                         c.ctypes.data, 2, 0) == _lib.E_NOGPU
    assert "no CUDA device available" in _lib.last_error()


def test_product_does_not_import_oracle():
    pkg = os.path.join(ROOT, "cvxopt_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dp, f)).read()
                assert "kkt_oracle" not in src and "oracle/_ref" not in src and "import cvxopt\n" not in src, f


def test_dims_validation():
    from cvxopt_b200.kkt import make_dims
    with pytest.raises(TypeError):
        make_dims({"l": -1, "q": [], "s": []})
    with pytest.raises(TypeError):
        make_dims({"l": 1, "q": [0], "s": []})
    d, keep, cdim, cp = make_dims({"l": 2, "q": [3], "s": [2, 3]})
    assert (cdim, cp) == (2 + 3 + 4 + 9, 2 + 3 + 3 + 6)


def test_batched_blocks_check_arguments_before_the_device():
    """the batched building blocks refuse a batch outside 1..CVXB_BATCH_MAX and an unknown trans with CVXB_E_ARG
    before they look for a device, and without a GPU fail with CVXB_E_NOGPU, never fall back"""
    import numpy as np
    import cvxopt_b200
    from cvxopt_b200 import _lib
    lib = _lib.load()
    a, inv = np.eye(2, order="F"), np.zeros(2 * 128 * 128)
    x, y = np.ones(2), np.zeros(2)
    info = np.zeros(1, dtype=np.intc)
    A, I, X, Y, P = a.ctypes.data, inv.ctypes.data, x.ctypes.data, y.ctypes.data, info.ctypes.data
    calls = {
        "potrf": lambda batch, tr: lib.cvxb_potrf_batched(2, A, 2, 4, I, 0, batch, P, 0),
        "trsv": lambda batch, tr: lib.cvxb_trsv_batched(2, A, 2, 4, I, 0, X, 2, tr, batch, 0),
        "trsm": lambda batch, tr: lib.cvxb_trsm_batched(2, A, 2, 4, I, 0, A, 2, 4, 2, batch, 0),
        "syrk": lambda batch, tr: lib.cvxb_syrk_batched(2, 2, A, 2, 4, None, 0, None, 0, 0, A, 2, 4, batch, 0),
        "gemv": lambda batch, tr: lib.cvxb_gemv_batched(tr, 2, 2, A, 2, 4, None, 0, X, 2, 1.0, 0.0, Y, 2, batch, 0),
    }
    for name, call in calls.items():
        for batch in (0, -1, 65535 + 1):
            assert call(batch, ord("N")) == _lib.E_ARG, (name, batch)
            assert "batch" in _lib.last_error(), name
        if name in ("trsv", "gemv"):
            assert call(1, ord("X")) == _lib.E_ARG, name
            assert "trans" in _lib.last_error(), name
    assert lib.cvxb_potrf_batched(-1, A, 2, 4, I, 0, 1, P, 0) == _lib.E_ARG
    assert lib.cvxb_gemv_batched(ord("T"), 2, -3, A, 2, 4, None, 0, X, 2, 1.0, 0.0, Y, 2, 1, 0) == _lib.E_ARG
    assert lib.cvxb_syrk_batched(2, 3, A, 2, 4, None, 0, None, 0, 0, A, 2, 4, 1, 0) == _lib.E_ARG   # lda < k
    if cvxopt_b200.device_count() > 0:
        pytest.skip("a GPU is visible")
    for name, call in calls.items():
        for batch in (1, 65535):
            assert call(batch, ord("T")) == _lib.E_NOGPU, (name, batch)
            assert "no CUDA device available" in _lib.last_error(), name
