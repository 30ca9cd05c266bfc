"""The GP batch's adjoint without a GPU: the exported entry point, its refusal of a NULL batch, the argument errors of
GPBatch.adjoint_gp / GPBatchGroup.adjoint_gp and of gp_layer, each raised before any device work, and the lazy
export."""
import ctypes as C

import numpy as np
import pytest


def _no_device(*a, **k):
    raise AssertionError("device work before the argument checks")


def test_adjoint_gp_is_exported():
    from cvxopt_b200 import _lib
    assert "cvxb_batch_adjoint_gp" in _lib.exported_symbols()
    assert hasattr(_lib.load(), "cvxb_batch_adjoint_gp")


def test_adjoint_gp_of_null_batch_is_e_arg():
    from cvxopt_b200 import _lib
    lib = _lib.load()
    assert lib.cvxb_batch_adjoint_gp(None, *([None] * 10), _lib.HOST) == _lib.E_ARG
    assert "NULL" in _lib.last_error()


class _Unbuilt:
    """a GPBatch / GPBatchGroup shell without a device batch: any library call fails the test"""
    def __getattr__(self, name):
        raise AssertionError("device work before the argument checks (%s)" % name)


def _shells(B=4, n=3, K=(5, 2, 3), ml=3, p=2):
    from cvxopt_b200 import GPBatch, GPBatchGroup
    gb = GPBatch.__new__(GPBatch)
    gb.B, gb.n, gb.K, gb.mnl, gb.ml, gb.p = B, n, list(K), len(K) - 1, ml, p
    gb.m = gb.mnl + ml
    gb._lib, gb._h = _Unbuilt(), C.c_void_p()
    grp = GPBatchGroup.__new__(GPBatchGroup)
    grp.B, grp.n, grp.m, grp.p, grp.nsub = B, n, len(K) - 1 + ml, p, 1
    grp.idx, grp.parts = [np.arange(B)], [_Unbuilt()]
    return gb, grp


BAD_ADJOINT = [
    (dict(gx=np.zeros((4, 2))), "gx must have shape"), (dict(gx=np.zeros(3)), "gx must have shape"),
    (dict(gy=np.zeros((4, 3))), "gy must have shape"), (dict(gz=np.zeros((4, 3))), "gz must have shape"),
    (dict(gz=np.zeros((3, 5))), "gz must have shape"),
    (dict(want=("F", "P")), "unknown keys"), (dict(want=("q",)), "unknown keys"), (dict(want=("znl",)), "unknown keys"),
]


@pytest.mark.parametrize("which", ["batch", "group"])
@pytest.mark.parametrize("case", range(len(BAD_ADJOINT)))
def test_adjoint_gp_argument_errors(which, case):
    gb, grp = _shells()
    kw, msg = BAD_ADJOINT[case]
    args = dict(gx=np.zeros((4, 3)))
    args.update(kw)
    with pytest.raises(TypeError, match=msg):
        (gb if which == "batch" else grp).adjoint_gp(**args)


def test_adjoint_gp_keys():
    from cvxopt_b200 import GPBatch
    from cvxopt_b200.batch import GP_ADJOINT_KEYS
    import inspect
    assert GP_ADJOINT_KEYS == ("F", "g", "G", "h", "A", "b")
    assert inspect.signature(GPBatch.adjoint_gp).parameters["want"].default == GP_ADJOINT_KEYS
    gb, _ = _shells()
    with pytest.raises(TypeError, match=r"the keys are \('F', 'g', 'G', 'h', 'A', 'b'\)"):
        gb.adjoint_gp(np.zeros((4, 3)), want=("P",))


def test_gp_batch_keeps_the_qp_adjoint_entry_points():
    """GPBatch adds adjoint_gp and overrides none of the QP batch's adjoint calls, whose refusals stay as they are"""
    from cvxopt_b200 import GPBatch, GPBatchGroup, QPBatch, QPBatchGroup
    for name in ("adjoint", "adjoint_ptr", "adjoint_cone", "adjoint_cone_ptr"):
        assert getattr(GPBatch, name) is getattr(QPBatch, name), name
    for name in ("adjoint", "adjoint_cone"):
        assert getattr(GPBatchGroup, name) is getattr(QPBatchGroup, name), name


def test_adjoint_gp_of_a_closed_batch_is_a_value_error():
    """a destroyed handle reaches the library as NULL: CVXB_E_ARG, raised as ValueError through _lib.check"""
    from cvxopt_b200 import GPBatch, _lib
    gb = GPBatch.__new__(GPBatch)
    gb.B, gb.n, gb.K, gb.mnl, gb.ml, gb.m, gb.p = 2, 3, [2, 1], 1, 2, 3, 0
    gb._lib, gb._h = _lib.load(), C.c_void_p()
    with pytest.raises(ValueError, match="batch_adjoint_gp"):
        gb.adjoint_gp(np.zeros((2, 3)))


def _layer_args(B=3, n=4, K=(5, 2, 3), ml=6, p=2):
    import torch
    rng = np.random.default_rng(0)
    t = lambda *s: torch.from_numpy(rng.standard_normal(s))     # noqa: E731  float64, on the CPU
    S = sum(K)
    return dict(K=list(K), F=t(B, S, n), g=t(B, S), G=t(B, ml, n), h=t(B, ml), A=t(B, p, n), b=t(B, p))


def _bad_layer_calls():
    import torch
    a = _layer_args()
    return [
        (dict(K=(5, 2, 3)), "'K' must be a list of positive integers"),
        (dict(K=[5, 0, 5]), "'K' must be a list of positive integers"),
        (dict(K=[5, 2.0, 3]), "'K' must be a list of positive integers"),
        (dict(K=[]), "'K' must be a list of positive integers"),
        (dict(K=[5, 2, 4]), "F must have shape"),
        (dict(F=a["F"][0]), "F must have shape"), (dict(F=a["F"][:, :, :0]), "F must have shape"),
        (dict(F=a["F"].float()), "F must be float64"), (dict(F=a["F"].numpy()), "F must be a torch tensor"),
        (dict(g=a["g"][:, :-1]), "g must have shape"), (dict(g=a["g"].to(torch.int64)), "g must be float64"),
        (dict(G=a["G"][:, :, :-1]), "G must have shape"), (dict(G=a["G"][0]), "G must have shape"),
        (dict(h=a["h"][:, :-1]), "h must have shape"),
        (dict(A=a["A"][:, :, :-1]), "A must have shape"), (dict(b=a["b"][:, :-1]), "b must have shape"),
        (dict(A=None), "given together"), (dict(b=None), "given together"),
        (dict(G=None), "given together"), (dict(h=None), "given together"),
        ({}, "must be a CUDA tensor"),                # every shape is right: the CPU tensors are refused last
    ]


@pytest.mark.parametrize("case", range(21))
def test_gp_layer_type_errors(monkeypatch, case):
    from cvxopt_b200 import layer
    monkeypatch.setattr(layer, "GPBatchGroup", _no_device)
    kw, msg = _bad_layer_calls()[case]
    a = _layer_args()
    a.update(kw)
    with pytest.raises(TypeError, match=msg):
        layer.gp_layer(**a)


def test_gp_layer_case_count():
    assert len(_bad_layer_calls()) == 21


def test_gp_layer_is_exported_lazily():
    import os
    import subprocess
    import sys
    import cvxopt_b200
    from cvxopt_b200.layer import gp_layer
    assert cvxopt_b200.gp_layer is gp_layer and "gp_layer" in cvxopt_b200.__all__
    # importing the package does not import torch; asking for the layer does
    code = ("import sys, cvxopt_b200; assert 'torch' not in sys.modules; cvxopt_b200.gp_layer; "
            "assert 'torch' in sys.modules")
    subprocess.run([sys.executable, "-c", code], check=True,
                   cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
