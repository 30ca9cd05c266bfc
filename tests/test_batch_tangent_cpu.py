"""The batch tangents without a GPU: the exported entry points, their refusals before any device work (a NULL batch),
and the argument errors of QPBatch.tangent, ConeLPBatch.tangent, QCQPBatch.tangent, GPBatch.tangent_gp,
CPBatch.tangent_cp and their groups, each raised before any library call."""
import ctypes as C

import numpy as np
import pytest

ENTRY = ["cvxb_batch_tangent", "cvxb_batch_tangent_qcqp", "cvxb_batch_tangent_gp", "cvxb_batch_tangent_cp"]
NARGS = {"cvxb_batch_tangent": 9, "cvxb_batch_tangent_qcqp": 10, "cvxb_batch_tangent_gp": 9,
         "cvxb_batch_tangent_cp": 10}


@pytest.mark.parametrize("name", ENTRY)
def test_tangent_is_exported(name):
    from cvxopt_b200 import _lib
    assert name in _lib.exported_symbols()
    assert hasattr(_lib.load(), name)


@pytest.mark.parametrize("name", ENTRY)
def test_tangent_of_null_batch_is_e_arg(name):
    from cvxopt_b200 import _lib
    lib = _lib.load()
    assert getattr(lib, name)(None, *([None] * NARGS[name]), _lib.HOST) == _lib.E_ARG
    assert "NULL" in _lib.last_error()


class _Unbuilt:
    """a batch shell without a device batch: any library call fails the test"""
    def __getattr__(self, name):
        raise AssertionError("device work before the argument checks (%s)" % name)


def _shell(cls, **attrs):
    b = cls.__new__(cls)
    b.__dict__.update(attrs)
    b._lib, b._h = _Unbuilt(), C.c_void_p()
    return b


def _group(cls, part, B):
    grp = cls.__new__(cls)
    grp.B, grp.nsub, grp.idx, grp.parts = B, 1, [np.arange(B)], [part]
    return grp


B, N, M, P = 4, 3, 5, 2
BAD_QP = [
    (dict(dP=np.zeros((B, N, N + 1))), "dP must have shape"), (dict(dq=np.zeros((B, N + 1))), "dq must have shape"),
    (dict(dG=np.zeros((B, N, M))), "dG must have shape"), (dict(dh=np.zeros((B, M, 1))), "dh must have shape"),
    (dict(dA=np.zeros((B, P + 1, N))), "dA must have shape"), (dict(db=np.zeros((B, P + 1))), "db must have shape"),
    (dict(dq=np.zeros((B, N), dtype=np.int64)), "dq must be a float array"),
    (dict(dG=np.zeros((B, M, N), dtype=complex)), "dG must be a float array"),
]


@pytest.mark.parametrize("which", ["batch", "group"])
@pytest.mark.parametrize("case", range(len(BAD_QP)))
def test_qp_tangent_argument_errors(which, case):
    from cvxopt_b200 import QPBatch, QPBatchGroup
    qb = _shell(QPBatch, B=B, n=N, m=M, p=P)
    kw, msg = BAD_QP[case]
    obj = qb if which == "batch" else _group(QPBatchGroup, qb, B)
    with pytest.raises(TypeError, match=msg):
        obj.tangent(**kw)


def test_group_tangent_checks_the_leading_dimension():
    from cvxopt_b200 import QPBatch, QPBatchGroup
    grp = _group(QPBatchGroup, _shell(QPBatch, B=B, n=N, m=M, p=P), B)
    with pytest.raises(TypeError, match="leading dimension"):
        grp.tangent(dq=np.zeros((B + 1, N)))


def test_cone_lp_tangent_takes_dc_and_no_dp():
    from cvxopt_b200 import ConeLPBatch
    lb = _shell(ConeLPBatch, B=B, n=N, m=M, p=P)
    with pytest.raises(TypeError):
        lb.tangent(dP=np.zeros((B, N, N)))
    with pytest.raises(TypeError, match="dc must have shape"):
        lb.tangent(dc=np.zeros((B, N + 1)))


def test_qcqp_tangent_argument_errors():
    from cvxopt_b200 import QCQPBatch
    qb = _shell(QCQPBatch, B=B, n=N, m=2 + M, p=P, mnl=2, ml=M)
    for kw, msg in [(dict(dP=np.zeros((B, 3, N, N + 1))), "dP must have shape"),
                    (dict(dP=np.zeros((B, 2, N, N))), "dP must have shape"),
                    (dict(dq=np.zeros((B, 2, N))), "dq must have shape"), (dict(dr=np.zeros((B, 2))), "dr must"),
                    (dict(dG=np.zeros((B, M + 2, N))), "dG must have shape"), (dict(dh=np.zeros((B, M + 2))), "dh")]:
        with pytest.raises(TypeError, match=msg):
            qb.tangent(**kw)


def test_gp_tangent_argument_errors():
    from cvxopt_b200 import GPBatch, GPBatchGroup
    K = [4, 2, 3]
    gb = _shell(GPBatch, B=B, n=N, m=2 + M, p=P, mnl=2, ml=M, K=K)
    for obj in (gb, _group(GPBatchGroup, gb, B)):
        for kw, msg in [(dict(dF=np.zeros((B, 8, N))), "dF must have shape"), (dict(dg=np.zeros((B, 9, 1))), "dg"),
                        (dict(dG=np.zeros((B, M, N + 1))), "dG must have shape"),
                        (dict(dF=np.zeros((B, 9, N), dtype=np.int32)), "float array")]:
            with pytest.raises(TypeError, match=msg):
                obj.tangent_gp(**kw)


def test_cp_tangent_argument_errors():
    from cvxopt_b200 import CPBatch, CPLBatch
    cb = _shell(CPBatch, B=B, n=N, m=2 + M, p=P, mnl=2, ml=M, _epi=1)
    with pytest.raises(TypeError, match="no c"):
        cb.tangent_cp(dc=np.zeros((B, N)))
    for kw, msg in [(dict(tx=np.zeros((B, N + 1))), "tx must have shape"), (dict(tf=np.zeros((B, 3))), "tf must"),
                    (dict(dG=np.zeros((B, M + 2, N))), "dG must have shape"), (dict(db=np.zeros((B, 1))), "db")]:
        with pytest.raises(TypeError, match=msg):
            cb.tangent_cp(**kw)
    lb = _shell(CPLBatch, B=B, n=N, m=2 + M, p=P, mnl=2, ml=M)
    with pytest.raises(TypeError, match="dc must have shape"):
        lb.tangent_cp(dc=np.zeros((B, N + 1)))


def test_tangent_of_a_closed_batch_is_a_value_error():
    """a destroyed handle reaches the library as NULL: CVXB_E_ARG, raised as ValueError through _lib.check"""
    from cvxopt_b200 import QPBatch, _lib
    qb = QPBatch.__new__(QPBatch)
    qb.B, qb.n, qb.m, qb.p = 2, 3, 4, 0
    qb._lib, qb._h = _lib.load(), C.c_void_p()
    with pytest.raises(ValueError, match="batch_tangent"):
        qb.tangent(dq=np.zeros((2, 3)))


def test_layer_tangent_detection():
    """a forward-mode dual input is what makes the layers keep the solved group for jvp"""
    import torch
    import torch.autograd.forward_ad as fwAD
    from cvxopt_b200.layer import _has_tangent
    t = torch.zeros(2, 3, dtype=torch.float64)
    assert not _has_tangent(t, None, 3)
    with fwAD.dual_level():
        assert _has_tangent(None, fwAD.make_dual(t, torch.ones_like(t)))
        assert not _has_tangent(t)
