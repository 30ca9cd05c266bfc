"""The QCQP batch's adjoint without a GPU: the exported entry point, its refusal of a NULL batch, the argument errors of
QCQPBatch.adjoint / QCQPBatchGroup.adjoint and of qcqp_layer, each raised before any device work, and the lazy
export."""
import ctypes as C

import numpy as np
import pytest


def _no_device(*a, **k):
    raise AssertionError("device work before the argument checks")


def test_adjoint_qcqp_is_exported():
    from cvxopt_b200 import _lib
    assert "cvxb_batch_adjoint_qcqp" in _lib.exported_symbols()
    assert hasattr(_lib.load(), "cvxb_batch_adjoint_qcqp")


def test_adjoint_qcqp_of_null_batch_is_e_arg():
    from cvxopt_b200 import _lib
    lib = _lib.load()
    assert lib.cvxb_batch_adjoint_qcqp(None, *([None] * 11), _lib.HOST) == _lib.E_ARG
    assert "NULL" in _lib.last_error()


class _Unbuilt:
    """a QCQPBatch / QCQPBatchGroup shell without a device batch: any library call fails the test"""
    def __getattr__(self, name):
        raise AssertionError("device work before the argument checks (%s)" % name)


def _shells(B=4, n=3, mnl=2, ml=3, p=2):
    from cvxopt_b200 import QCQPBatch, QCQPBatchGroup
    qb = QCQPBatch.__new__(QCQPBatch)
    qb.B, qb.n, qb.mnl, qb.ml, qb.m, qb.p = B, n, mnl, ml, mnl + ml, p
    qb._lib, qb._h = _Unbuilt(), C.c_void_p()
    grp = QCQPBatchGroup.__new__(QCQPBatchGroup)
    grp.B, grp.n, grp.m, grp.p, grp.nsub = B, n, mnl + ml, p, 1
    grp.idx, grp.parts = [np.arange(B)], [_Unbuilt()]
    return qb, grp


BAD_ADJOINT = [
    (dict(gx=np.zeros((4, 2))), "gx must have shape"), (dict(gx=np.zeros(3)), "gx must have shape"),
    (dict(gy=np.zeros((4, 3))), "gy must have shape"), (dict(gz=np.zeros((4, 3))), "gz must have shape"),
    (dict(gz=np.zeros((3, 5))), "gz must have shape"),
    (dict(want=("P", "x")), "unknown keys"), (dict(want=("znl",)), "unknown keys"),
]


@pytest.mark.parametrize("which", ["batch", "group"])
@pytest.mark.parametrize("case", range(len(BAD_ADJOINT)))
def test_adjoint_argument_errors(which, case):
    qb, grp = _shells()
    kw, msg = BAD_ADJOINT[case]
    args = dict(gx=np.zeros((4, 3)))
    args.update(kw)
    with pytest.raises(TypeError, match=msg):
        (qb if which == "batch" else grp).adjoint(**args)


def test_qp_adjoint_keys_are_unchanged():
    """the QP batch still refuses 'r', and names its own keys"""
    from cvxopt_b200 import QPBatch
    qb = QPBatch.__new__(QPBatch)
    qb.B, qb.n, qb.m, qb.p = 4, 3, 5, 2
    qb._lib, qb._h = _Unbuilt(), C.c_void_p()
    with pytest.raises(TypeError, match=r"unknown keys \['r'\]; the keys are \('P', 'q', 'G', 'h', 'A', 'b'\)"):
        qb.adjoint(np.zeros((4, 3)), want=("r",))


def test_adjoint_of_a_closed_batch_is_a_value_error():
    """a destroyed handle reaches the library as NULL: CVXB_E_ARG, raised as ValueError through _lib.check"""
    from cvxopt_b200 import QCQPBatch, _lib
    qb = QCQPBatch.__new__(QCQPBatch)
    qb.B, qb.n, qb.mnl, qb.ml, qb.m, qb.p = 2, 3, 1, 2, 3, 0
    qb._lib, qb._h = _lib.load(), C.c_void_p()
    with pytest.raises(ValueError, match="batch_adjoint_qcqp"):
        qb.adjoint(np.zeros((2, 3)))


def _layer_args(B=3, n=4, mnl=2, ml=6, p=2):
    import torch
    rng = np.random.default_rng(0)
    t = lambda *s: torch.from_numpy(rng.standard_normal(s))     # noqa: E731  float64, on the CPU
    return dict(P=t(B, mnl + 1, n, n), q=t(B, mnl + 1, n), r=t(B, mnl + 1), G=t(B, ml, n), h=t(B, ml),
                A=t(B, p, n), b=t(B, p), x0=t(B, n))


def _bad_layer_calls():
    import torch
    a = _layer_args()
    return [
        (dict(P=a["P"][0]), "P must have shape"), (dict(P=a["P"][..., :-1]), "P must have shape"),
        (dict(P=a["P"][:, :0]), "P must have shape"),
        (dict(P=a["P"].float()), "P must be float64"), (dict(P=a["P"].numpy()), "P must be a torch tensor"),
        (dict(q=a["q"][:, :-1]), "q must have shape"), (dict(q=a["q"].to(torch.int64)), "q must be float64"),
        (dict(r=a["r"][:, :-1]), "r must have shape"), (dict(r=a["r"].numpy()), "r must be a torch tensor"),
        (dict(x0=a["x0"][:, :-1]), "x0 must have shape"), (dict(x0=a["x0"].float()), "x0 must be float64"),
        (dict(G=a["G"][:, :, :-1]), "G must have shape"), (dict(G=a["G"][0]), "G must have shape"),
        (dict(h=a["h"][:, :-1]), "h must have shape"),
        (dict(A=a["A"][:, :, :-1]), "A must have shape"), (dict(b=a["b"][:, :-1]), "b must have shape"),
        (dict(A=None), "given together"), (dict(b=None), "given together"),
        (dict(G=None), "given together"), (dict(h=None), "given together"),
        (dict(dims={"l": 5}), "does not match"),
        ({}, "must be a CUDA tensor"),                # every shape is right: the CPU tensors are refused last
    ]


@pytest.mark.parametrize("case", range(22))
def test_qcqp_layer_type_errors(monkeypatch, case):
    from cvxopt_b200 import layer
    monkeypatch.setattr(layer, "QCQPBatchGroup", _no_device)
    kw, msg = _bad_layer_calls()[case]
    a = _layer_args()
    a.update(kw)
    with pytest.raises(TypeError, match=msg):
        layer.qcqp_layer(**a)


def test_qcqp_layer_case_count():
    assert len(_bad_layer_calls()) == 22


@pytest.mark.parametrize("dims", [{"l": 6, "q": [2]}, {"l": 6, "s": [2]}])
def test_qcqp_layer_refuses_cones(monkeypatch, dims):
    from cvxopt_b200 import layer
    monkeypatch.setattr(layer, "QCQPBatchGroup", _no_device)
    with pytest.raises(NotImplementedError, match="qcqp_layer"):
        layer.qcqp_layer(**_layer_args(), dims=dims)


def test_qcqp_layer_is_exported_lazily():
    import os
    import subprocess
    import sys
    import cvxopt_b200
    from cvxopt_b200.layer import qcqp_layer
    assert cvxopt_b200.qcqp_layer is qcqp_layer and "qcqp_layer" in cvxopt_b200.__all__
    # importing the package does not import torch; asking for the layer does
    code = ("import sys, cvxopt_b200; assert 'torch' not in sys.modules; cvxopt_b200.qcqp_layer; "
            "assert 'torch' in sys.modules")
    subprocess.run([sys.executable, "-c", code], check=True,
                   cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
