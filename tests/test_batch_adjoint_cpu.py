"""The QP batch's adjoint without a GPU: the exported entry point, its refusal of a NULL batch, and the argument errors
of qp_layer and of QPBatch.adjoint / QPBatchGroup.adjoint, each raised before any device work."""
import ctypes as C

import numpy as np
import pytest


def _no_device(*a, **k):
    raise AssertionError("device work before the argument checks")


def test_adjoint_is_exported():
    from cvxopt_b200 import _lib
    assert "cvxb_batch_adjoint" in _lib.exported_symbols()
    assert hasattr(_lib.load(), "cvxb_batch_adjoint")


def test_adjoint_of_null_batch_is_e_arg():
    from cvxopt_b200 import _lib
    lib = _lib.load()
    assert lib.cvxb_batch_adjoint(None, *([None] * 9), _lib.HOST) == _lib.E_ARG
    assert "NULL" in _lib.last_error()


def _layer_args(B=3, n=4, m=6, p=2):
    import torch
    rng = np.random.default_rng(0)
    t = lambda *s: torch.from_numpy(rng.standard_normal(s))     # noqa: E731  float64, on the CPU
    return dict(P=t(B, n, n), q=t(B, n), G=t(B, m, n), h=t(B, m), A=t(B, p, n), b=t(B, p))


def _bad_layer_calls():
    import torch
    a = _layer_args()
    return [
        (dict(P=a["P"][0]), "P must have shape"), (dict(P=a["P"][:, :, :-1]), "P must have shape"),
        (dict(P=a["P"].float()), "P must be float64"), (dict(P=a["P"].numpy()), "P must be a torch tensor"),
        (dict(q=a["q"][:, :-1]), "q must have shape"), (dict(q=a["q"].to(torch.int64)), "q must be float64"),
        (dict(G=a["G"][:, :, :-1]), "G must have shape"), (dict(G=a["G"][0]), "G must have shape"),
        (dict(h=a["h"][:, :-1]), "h must have shape"),
        (dict(A=a["A"][:, :, :-1]), "A must have shape"), (dict(b=a["b"][:, :-1]), "b must have shape"),
        (dict(A=None), "given together"), (dict(b=None), "given together"),
        (dict(dims={"l": 5}), "does not match"),
        ({}, "must be a CUDA tensor"),                # every shape is right: the CPU tensors are refused last
    ]


@pytest.mark.parametrize("case", range(15))
def test_qp_layer_type_errors(monkeypatch, case):
    from cvxopt_b200 import layer
    monkeypatch.setattr(layer, "QPBatchGroup", _no_device)
    kw, msg = _bad_layer_calls()[case]
    a = _layer_args()
    a.update(kw)
    with pytest.raises(TypeError, match=msg):
        layer.qp_layer(**a)


@pytest.mark.parametrize("dims", [{"l": 6, "q": [2]}, {"l": 6, "s": [2]}])
def test_qp_layer_refuses_cones(monkeypatch, dims):
    from cvxopt_b200 import layer
    monkeypatch.setattr(layer, "QPBatchGroup", _no_device)
    with pytest.raises(NotImplementedError):
        layer.qp_layer(**_layer_args(), dims=dims)


def test_qp_layer_is_exported():
    import cvxopt_b200
    from cvxopt_b200.layer import qp_layer
    assert cvxopt_b200.qp_layer is qp_layer and "qp_layer" in cvxopt_b200.__all__


class _Unbuilt:
    """a QPBatch / QPBatchGroup shell without a device batch: any library call fails the test"""
    def __getattr__(self, name):
        raise AssertionError("device work before the argument checks (%s)" % name)


def _shells(B=4, n=3, m=5, p=2):
    from cvxopt_b200 import QPBatch, QPBatchGroup
    qb = QPBatch.__new__(QPBatch)
    qb.B, qb.n, qb.m, qb.p = B, n, m, p
    qb._lib, qb._h = _Unbuilt(), C.c_void_p()
    grp = QPBatchGroup.__new__(QPBatchGroup)
    grp.B, grp.n, grp.m, grp.p, grp.nsub = B, n, m, p, 1
    grp.idx, grp.parts = [np.arange(B)], [_Unbuilt()]
    return qb, grp


BAD_ADJOINT = [
    (dict(gx=np.zeros((4, 2))), "gx must have shape"), (dict(gx=np.zeros(3)), "gx must have shape"),
    (dict(gy=np.zeros((4, 3))), "gy must have shape"), (dict(gz=np.zeros((3, 5))), "gz must have shape"),
    (dict(want=("P", "x")), "unknown keys"),
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


def test_adjoint_check_of_a_closed_batch_is_a_value_error():
    """a destroyed handle reaches the library as NULL: CVXB_E_ARG, raised as ValueError through _lib.check"""
    from cvxopt_b200 import QPBatch, _lib
    qb = QPBatch.__new__(QPBatch)
    qb.B, qb.n, qb.m, qb.p = 2, 3, 4, 0
    qb._lib, qb._h = _lib.load(), C.c_void_p()
    with pytest.raises(ValueError, match="batch_adjoint"):
        qb.adjoint(np.zeros((2, 3)))
