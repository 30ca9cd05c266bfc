"""The cone adjoint without a GPU: the exported entry point, its refusal of a NULL batch, the argument errors of
QPBatch.adjoint_cone / QPBatchGroup.adjoint_cone for the QP and the cone LP key sets, and every refusal of coneqp_layer
and conelp_layer, each raised before any device work."""
import ctypes as C

import numpy as np
import pytest


def _no_device(*a, **k):
    raise AssertionError("device work before the argument checks")


def test_adjoint_cone_is_exported():
    from cvxopt_b200 import _lib
    assert "cvxb_batch_adjoint_cone" in _lib.exported_symbols()
    assert hasattr(_lib.load(), "cvxb_batch_adjoint_cone")


def test_adjoint_cone_of_null_batch_is_e_arg():
    from cvxopt_b200 import _lib
    lib = _lib.load()
    assert lib.cvxb_batch_adjoint_cone(None, *([None] * 9), _lib.HOST) == _lib.E_ARG
    assert "NULL" in _lib.last_error()


class _Unbuilt:
    """a batch / group shell without a device batch: any library call fails the test"""
    def __getattr__(self, name):
        raise AssertionError("device work before the argument checks (%s)" % name)


def _shells(lp, B=4, n=3, m=5, p=2):
    from cvxopt_b200 import ConeLPBatch, ConeLPBatchGroup, QPBatch, QPBatchGroup
    cls, gcls = (ConeLPBatch, ConeLPBatchGroup) if lp else (QPBatch, QPBatchGroup)
    qb = cls.__new__(cls)
    qb.B, qb.n, qb.m, qb.p = B, n, m, p
    qb._lib, qb._h = _Unbuilt(), C.c_void_p()
    grp = gcls.__new__(gcls)
    grp.B, grp.n, grp.m, grp.p, grp.nsub = B, n, m, p, 1
    grp.idx, grp.parts = [np.arange(B)], [_Unbuilt()]
    return qb, grp


BAD_ADJOINT = [
    (dict(gx=np.zeros((4, 2))), "gx must have shape"), (dict(gx=np.zeros(3)), "gx must have shape"),
    (dict(gy=np.zeros((4, 3))), "gy must have shape"), (dict(gz=np.zeros((3, 5))), "gz must have shape"),
    (dict(want=("q", "x")), "unknown keys"),
]


@pytest.mark.parametrize("lp", [False, True])
@pytest.mark.parametrize("which", ["batch", "group"])
@pytest.mark.parametrize("case", range(len(BAD_ADJOINT)))
def test_adjoint_cone_argument_errors(lp, which, case):
    qb, grp = _shells(lp)
    kw, msg = BAD_ADJOINT[case]
    args = dict(gx=np.zeros((4, 3)))
    args.update(kw)
    with pytest.raises(TypeError, match=msg):
        (qb if which == "batch" else grp).adjoint_cone(**args)


@pytest.mark.parametrize("which", ["batch", "group"])
@pytest.mark.parametrize("lp, key", [(True, "P"), (True, "q"), (False, "c")])
def test_adjoint_cone_keys_follow_the_kind(which, lp, key):
    """a cone LP has c and no P; a QP has P and q and no c"""
    qb, grp = _shells(lp)
    with pytest.raises(TypeError, match="unknown keys"):
        (qb if which == "batch" else grp).adjoint_cone(np.zeros((4, 3)), want=(key,))


def test_adjoint_cone_keys():
    from cvxopt_b200 import SDPBatch, SDPBatchGroup, SDPQPBatch, SDPQPBatchGroup
    from cvxopt_b200.batch import ADJOINT_KEYS, CONELP_ADJOINT_KEYS
    assert CONELP_ADJOINT_KEYS == ("c", "G", "h", "A", "b")
    for cls in (SDPBatch, SDPBatchGroup):
        assert cls._cone_keys == CONELP_ADJOINT_KEYS
    for cls in (SDPQPBatch, SDPQPBatchGroup):
        assert cls._cone_keys == ADJOINT_KEYS


def test_adjoint_cone_of_a_closed_batch_is_a_value_error():
    """a destroyed handle reaches the library as NULL: CVXB_E_ARG, raised as ValueError through _lib.check"""
    from cvxopt_b200 import ConeLPBatch, _lib
    qb = ConeLPBatch.__new__(ConeLPBatch)
    qb.B, qb.n, qb.m, qb.p = 2, 3, 4, 0
    qb._lib, qb._h = _lib.load(), C.c_void_p()
    with pytest.raises(ValueError, match="batch_adjoint_cone"):
        qb.adjoint_cone(np.zeros((2, 3)))


DIMS = {"l": 2, "q": [3], "s": [2]}          # m = 2 + 3 + 4


def _layer_args(lp, B=3, n=4, p=2):
    import torch
    rng = np.random.default_rng(0)
    t = lambda *s: torch.from_numpy(rng.standard_normal(s))     # noqa: E731  float64, on the CPU
    a = dict(q=t(B, n), G=t(B, 9, n), h=t(B, 9), dims=dict(DIMS), A=t(B, p, n), b=t(B, p))
    if lp:
        a["c"] = a.pop("q")
    else:
        a["P"] = t(B, n, n)
    return a


def _bad_layer_calls(lp):
    import torch
    a = _layer_args(lp)
    qn = "c" if lp else "q"
    calls = [
        ({qn: a[qn][:, :-1]}, "P must have shape" if not lp else "G must have shape"),
        ({qn: a[qn][0]}, "%s must have shape" % qn), ({qn: a[qn].float()}, "%s must be float64" % qn),
        ({qn: a[qn].numpy()}, "%s must be a torch tensor" % qn),
        (dict(G=a["G"][:, :, :-1]), "G must have shape"), (dict(G=a["G"][0]), "G must have shape"),
        (dict(G=a["G"].to(torch.int64)), "G must be float64"),
        (dict(h=a["h"][:, :-1]), "h must have shape"),
        (dict(A=a["A"][:, :, :-1]), "A must have shape"), (dict(b=a["b"][:, :-1]), "b must have shape"),
        (dict(A=None), "given together"), (dict(b=None), "given together"),
        (dict(dims={"l": 2, "q": [3], "s": [3]}), "dims has 14 rows"), (dict(dims={"l": 9, "x": []}), "dims must"),
        (dict(dims=[9]), "dims must"),
        (dict(dims={"l": 2, "q": [3, 0], "s": [2]}), "each 'q' size"), (dict(dims={"l": 9, "s": [33]}), "'s' order in"),
        (dict(dims={"l": -1, "q": [6], "s": [2]}), "'l' must be nonnegative"),
        ({}, "must be a CUDA tensor"),                # every shape is right: the CPU tensors are refused last
    ]
    if not lp:
        calls += [(dict(P=a["P"][:, :, :-1]), "P must have shape"), (dict(P=a["P"].float()), "P must be float64")]
    return calls


@pytest.mark.parametrize("lp, case", [(False, i) for i in range(21)] + [(True, i) for i in range(19)])
def test_cone_layer_type_errors(monkeypatch, lp, case):
    from cvxopt_b200 import layer
    for g in ("SDPQPBatchGroup", "SDPBatchGroup", "ConeLPBatchGroup"):
        monkeypatch.setattr(layer, g, _no_device)
    kw, msg = _bad_layer_calls(lp)[case]
    a = _layer_args(lp)
    a.update(kw)
    with pytest.raises(TypeError, match=msg):
        (layer.conelp_layer if lp else layer.coneqp_layer)(**a)


def test_cone_layers_are_exported_lazily():
    import cvxopt_b200
    from cvxopt_b200.layer import conelp_layer, coneqp_layer
    assert cvxopt_b200.coneqp_layer is coneqp_layer and cvxopt_b200.conelp_layer is conelp_layer
    assert {"coneqp_layer", "conelp_layer"} <= set(cvxopt_b200.__all__)
