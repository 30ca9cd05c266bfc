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


def test_sblock_kernels_check_arguments_before_the_device():
    """cvxb_sblock_batched refuses, with CVXB_E_ARG and before it looks for a device, a batch outside
    1..CVXB_BATCH_MAX, an order outside 1..CVXB_BATCH_SMAX, strides below the blocks' rows, an unknown kernel or mode
    and a missing operand; every kernel id with all its operands fails with CVXB_E_NOGPU without a GPU"""
    import ctypes
    import numpy as np
    import cvxopt_b200
    from cvxopt_b200 import _lib
    lib = _lib.load()
    buf = np.zeros(64)
    orders = np.array([2, 3], dtype=np.intc)
    spart = np.zeros(4 * 2 * 65535)

    def args(**kw):
        a = _lib.SblockArgs(nblk=2, orders=orders.ctypes.data, m=13, L=17, n=1, ldg=13, sG=13,
                            spart=spart.ctypes.data)
        for name in ("s", "z", "ds", "dz", "h", "lmbda", "lmbdasq", "d", "di", "bzp", "th", "ws3", "r", "rti",
                     "sigs", "sigz", "wz", "ws", "wz2", "ws2", "wz3", "G", "Gs"):
            setattr(a, name, buf.ctypes.data)
        for k, v in kw.items():
            setattr(a, k, v)
        return a

    def call(kernel=_lib.SK_NT_COMPUTE, mode=0, batch=1, **kw):
        return lib.cvxb_sblock_batched(kernel, mode, batch, ctypes.byref(args(**kw)), 0)

    for batch in (0, -1, 65536):
        assert call(batch=batch) == _lib.E_ARG and "batch" in _lib.last_error(), batch
    for bad in ([0, 3], [2, 33], [-1, 2]):
        o = np.array(bad, dtype=np.intc)
        assert call(orders=o.ctypes.data) == _lib.E_ARG and "order" in _lib.last_error(), bad
    assert call(nblk=0) == _lib.E_ARG
    assert call(orders=None) == _lib.E_ARG
    assert call(spart=None) == _lib.E_ARG
    assert lib.cvxb_sblock_batched(0, 0, 1, None, 0) == _lib.E_ARG
    assert call(m=12) == _lib.E_ARG and call(L=12) == _lib.E_ARG          # 4 + 9 rows
    assert call(m=2 ** 31) == _lib.E_ARG and "int" in _lib.last_error()
    assert call(kernel=_lib.SK_RES, mode=1, L=16) == _lib.E_ARG            # the embedding's scalars need 17
    assert call(kernel=8) == _lib.E_ARG and "kernel" in _lib.last_error()
    assert call(kernel=-1) == _lib.E_ARG
    modes = {_lib.SK_NT_COMPUTE: 0, _lib.SK_UPDATE: 1, _lib.SK_DIR_POST: 1, _lib.SK_EIG_START: 0,
             _lib.SK_EIG_WARM: 0, _lib.SK_BUILD_GS: 0, _lib.SK_WTZ: 2, _lib.SK_RES: 1}
    for kernel, top in modes.items():
        assert call(kernel=kernel, mode=top + 1) == _lib.E_ARG and "mode" in _lib.last_error(), kernel
        assert call(kernel=kernel, mode=-1) == _lib.E_ARG, kernel
    missing = [(_lib.SK_NT_COMPUTE, 0, "lmbda"), (_lib.SK_UPDATE, 0, "sigz"), (_lib.SK_DIR_POST, 0, "ws3"),
               (_lib.SK_DIR_POST, 1, "sigs"), (_lib.SK_EIG_START, 0, "bzp"), (_lib.SK_EIG_WARM, 0, "z"),
               (_lib.SK_BUILD_GS, 0, "Gs"), (_lib.SK_WTZ, 1, "th"), (_lib.SK_WTZ, 2, "r"), (_lib.SK_RES, 0, "wz3"),
               (_lib.SK_RES, 1, "h")]
    for kernel, mode, name in missing:
        assert call(kernel=kernel, mode=mode, **{name: None}) == _lib.E_ARG, (kernel, mode, name)
        assert "missing" in _lib.last_error()
    assert call(kernel=_lib.SK_BUILD_GS, n=0) == _lib.E_ARG
    assert call(kernel=_lib.SK_BUILD_GS, ldg=12) == _lib.E_ARG
    if cvxopt_b200.device_count() > 0:
        pytest.skip("a GPU is visible")
    for kernel, top in modes.items():
        for mode in range(top + 1):
            for batch in (1, 65535):
                assert call(kernel=kernel, mode=mode, batch=batch) == _lib.E_NOGPU, (kernel, mode, batch)
                assert "no CUDA device available" in _lib.last_error()
