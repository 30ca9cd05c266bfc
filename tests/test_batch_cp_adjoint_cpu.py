"""The CP and cpl batches' adjoint without a GPU: the exported entry point, its refusal of a NULL batch, the argument
errors of CPBatch.adjoint_cp / CPBatchGroup.adjoint_cp and of cp_layer and cpl_layer, each raised before any device
work, and the lazy exports."""
import ctypes as C

import numpy as np
import pytest


def _no_device(*a, **k):
    raise AssertionError("device work before the argument checks")


def test_adjoint_cp_is_exported():
    from cvxopt_b200 import _lib
    assert "cvxb_batch_adjoint_cp" in _lib.exported_symbols()
    assert hasattr(_lib.load(), "cvxb_batch_adjoint_cp")


def test_adjoint_cp_of_null_batch_is_e_arg():
    from cvxopt_b200 import _lib
    lib = _lib.load()
    assert lib.cvxb_batch_adjoint_cp(None, *([None] * 8), _lib.HOST) == _lib.E_ARG
    assert "NULL" in _lib.last_error()


class _Unbuilt:
    """a batch or group shell without a device batch: any library call fails the test"""
    def __getattr__(self, name):
        raise AssertionError("device work before the argument checks (%s)" % name)


def _shells(cls_name, B=4, n=3, mnl=2, ml=3, p=2):
    import cvxopt_b200
    cls = getattr(cvxopt_b200, cls_name)
    gb = cls.__new__(cls)
    gb.B, gb.n, gb.mnl, gb.ml, gb.p = B, n, mnl, ml, p
    gb.m = mnl + ml
    gb._lib, gb._h, gb._err = _Unbuilt(), C.c_void_p(), None
    grp = getattr(cvxopt_b200, cls_name + "Group").__new__(getattr(cvxopt_b200, cls_name + "Group"))
    grp.B, grp.n, grp.m, grp.p, grp.nsub = B, n, mnl + ml, p, 1
    part = _Unbuilt()
    part.__dict__["_cp_keys"] = cls._cp_keys
    grp.idx, grp.parts = [np.arange(B)], [part]
    return gb, grp


BAD_ADJOINT = [
    (dict(gx=np.zeros((4, 2))), "gx must have shape"), (dict(gx=np.zeros(3)), "gx must have shape"),
    (dict(gy=np.zeros((4, 3))), "gy must have shape"), (dict(gz=np.zeros((4, 3))), "gz must have shape"),
    (dict(gz=np.zeros((3, 5))), "gz must have shape"),
    (dict(want=("G", "P")), "unknown keys"), (dict(want=("q",)), "unknown keys"), (dict(want=("znl",)), "unknown keys"),
    (dict(want=("uz",)), "unknown keys"),
]


@pytest.mark.parametrize("cls", ["CPBatch", "CPLBatch", "SDPCPLBatch"])
@pytest.mark.parametrize("which", ["batch", "group"])
@pytest.mark.parametrize("case", range(len(BAD_ADJOINT)))
def test_adjoint_cp_argument_errors(cls, which, case):
    gb, grp = _shells(cls)
    kw, msg = BAD_ADJOINT[case]
    args = dict(gx=np.zeros((4, 3)))
    args.update(kw)
    with pytest.raises(TypeError, match=msg):
        (gb if which == "batch" else grp).adjoint_cp(**args)


def test_adjoint_cp_keys():
    from cvxopt_b200 import CPBatch, CPLBatch, QCQPBatch, SDPCPLBatch
    from cvxopt_b200.batch import CP_ADJOINT_KEYS, CPL_ADJOINT_KEYS
    assert CP_ADJOINT_KEYS == ("ux", "uznl", "G", "h", "A", "b")
    assert CPL_ADJOINT_KEYS == CP_ADJOINT_KEYS + ("c",)
    assert CPBatch._cp_keys == CP_ADJOINT_KEYS and QCQPBatch._cp_keys == CP_ADJOINT_KEYS
    assert CPLBatch._cp_keys == CPL_ADJOINT_KEYS and SDPCPLBatch._cp_keys == CPL_ADJOINT_KEYS
    gb, _ = _shells("CPBatch")
    with pytest.raises(TypeError, match=r"the keys are \('ux', 'uznl', 'G', 'h', 'A', 'b'\)"):
        gb.adjoint_cp(np.zeros((4, 3)), want=("c",))


def test_cp_batches_keep_the_other_adjoint_entry_points():
    """the CP classes add adjoint_cp and load_ptr and override none of the other adjoint calls, whose refusals stay as
    they are; QCQPBatch's own adjoint stays the QCQP adjoint"""
    from cvxopt_b200 import CPBatch, CPBatchGroup, CPLBatch, QCQPBatch, QPBatch, QPBatchGroup
    for cls in (CPBatch, CPLBatch):
        for name in ("adjoint", "adjoint_ptr", "adjoint_cone", "adjoint_cone_ptr"):
            assert getattr(cls, name) is getattr(QPBatch, name), (cls, name)
    for name in ("adjoint", "adjoint_cone"):
        assert getattr(CPBatchGroup, name) is getattr(QPBatchGroup, name), name
    assert QCQPBatch.adjoint_cp is CPBatch.adjoint_cp and QCQPBatch.adjoint is not CPBatch.adjoint


def test_adjoint_cp_of_a_closed_batch_is_a_value_error():
    """a destroyed handle reaches the library as NULL: CVXB_E_ARG, raised as ValueError through _lib.check"""
    from cvxopt_b200 import CPBatch, _lib
    gb = CPBatch.__new__(CPBatch)
    gb.B, gb.n, gb.mnl, gb.ml, gb.m, gb.p = 2, 3, 1, 2, 3, 0
    gb._lib, gb._h, gb._err = _lib.load(), C.c_void_p(), None
    with pytest.raises(ValueError, match="batch_adjoint_cp"):
        gb.adjoint_cp(np.zeros((2, 3)))


def _F(B=3, n=4, mnl=1, x0=None):
    import torch
    x0 = torch.zeros((B, n), dtype=torch.float64) if x0 is None else x0

    def F(x=None, z=None, idx=None, params=()):
        if x is None:
            return mnl, x0
        raise AssertionError("F evaluated before the argument checks")
    return F


def _layer_args(B=3, n=4, ml=6, p=2, cpl=False):
    import torch
    rng = np.random.default_rng(0)
    t = lambda *s: torch.from_numpy(rng.standard_normal(s))     # noqa: E731  float64, on the CPU
    a = dict(F=_F(B, n), params=(t(B, n), t(B, 2, 2)), G=t(B, ml, n), h=t(B, ml), A=t(B, p, n), b=t(B, p))
    if cpl:
        a["c"] = t(B, n)
    return a


def _bad_layer_calls(cpl):
    import torch
    a = _layer_args(cpl=cpl)
    out = [
        (dict(F=None), TypeError, "F must be callable"),
        (dict(params=a["params"][0]), TypeError, "params must be a tuple"),
        (dict(params=(a["params"][0].float(),)), TypeError, r"params\[0\] must be float64"),
        (dict(params=(a["params"][0].numpy(),)), TypeError, r"params\[0\] must be a torch tensor"),
        (dict(params=(a["params"][0][:2],)), TypeError, r"params\[0\] must have leading dimension"),
        (dict(F=_F(mnl=-1)), TypeError, "nonnegative integer"),
        (dict(F=_F(mnl=1.0)), TypeError, "nonnegative integer"),
        (dict(F=_F(x0=torch.zeros((3, 4), dtype=torch.float32))), TypeError, "x0"),
        (dict(F=_F(x0=torch.zeros(4, dtype=torch.float64))), TypeError, "x0"),
        (dict(G=a["G"][:, :, :-1]), TypeError, "G must have shape"), (dict(G=a["G"][0]), TypeError, "G must have shape"),
        (dict(h=a["h"][:, :-1]), TypeError, "h must have shape"), (dict(h=a["h"].float()), TypeError, "h must be float64"),
        (dict(A=a["A"][:, :, :-1]), TypeError, "A must have shape"), (dict(b=a["b"][:, :-1]), TypeError, "b must have shape"),
        (dict(A=None), TypeError, "given together"), (dict(b=None), TypeError, "given together"),
        (dict(G=None), TypeError, "given together"), (dict(h=None), TypeError, "given together"),
        ({}, TypeError, "must be a CUDA tensor"),       # every shape is right: the CPU tensors are refused last
    ]
    if cpl:
        out += [
            (dict(c=a["c"][:, :-1]), TypeError, "c must have shape"), (dict(c=a["c"].numpy()), TypeError, "c must be"),
            (dict(dims={"l": 5}), TypeError, "dims has 5 rows"),
            (dict(dims={"l": 2, "q": [4]}), TypeError, "must be a CUDA tensor"),
            (dict(dims={"l": 2, "s": [2]}), TypeError, "must be a CUDA tensor"),
            (dict(dims={"l": 1, "q": [1], "s": [2]}), TypeError, "must be a CUDA tensor"),
            (dict(dims={"l": 2, "q": [0, 4]}), TypeError, "'q' size at least 1"),
            (dict(dims={"l": 6, "s": [40]}), TypeError, "'s' order in 0..32"),
            (dict(dims={"l": 6, "x": []}), TypeError, "keys 'l', 'q' and 's'"),
        ]
    else:
        out += [
            (dict(dims={"l": 5}), TypeError, r"dims\['l'\] = 5"),
            (dict(dims={"l": 2, "q": [4]}), NotImplementedError, "'l' rows only"),
            (dict(dims={"l": 2, "s": [2]}), NotImplementedError, "'l' rows only"),
        ]
    return out


@pytest.mark.parametrize("cpl,case", [(False, k) for k in range(23)] + [(True, k) for k in range(29)])
def test_cp_layer_argument_errors(monkeypatch, cpl, case):
    from cvxopt_b200 import layer
    for name in ("CPBatchGroup", "CPLBatchGroup", "SDPCPLBatchGroup"):
        monkeypatch.setattr(layer, name, _no_device)
    kw, exc, msg = _bad_layer_calls(cpl)[case]
    a = _layer_args(cpl=cpl)
    a.update(kw)
    with pytest.raises(exc, match=msg):
        (layer.cpl_layer if cpl else layer.cp_layer)(**a)


def test_cp_layer_case_counts():
    assert len(_bad_layer_calls(False)) == 23 and len(_bad_layer_calls(True)) == 29


def test_cp_layer_rank_and_empty_refusals(monkeypatch):
    """p > n is cp's Rank ValueError, and a cpl problem without rows cpl's, both before any device work"""
    import torch
    from cvxopt_b200 import layer
    for name in ("CPBatchGroup", "CPLBatchGroup", "SDPCPLBatchGroup"):
        monkeypatch.setattr(layer, name, _no_device)
    a = _layer_args(n=2, p=3)
    a["F"] = _F(n=2)
    with pytest.raises(ValueError, match="Rank"):
        layer.cp_layer(**a)
    c = torch.zeros((3, 4), dtype=torch.float64)
    with pytest.raises(ValueError, match="at least one constraint row"):
        layer.cpl_layer(c, _F(mnl=0))


@pytest.mark.parametrize("name", ["cp_layer", "cpl_layer"])
def test_cp_layers_are_exported_lazily(name):
    import os
    import subprocess
    import sys
    import cvxopt_b200
    from cvxopt_b200 import layer
    assert getattr(cvxopt_b200, name) is getattr(layer, name) and name in cvxopt_b200.__all__
    # importing the package does not import torch; asking for the layer does
    code = ("import sys, cvxopt_b200; assert 'torch' not in sys.modules; cvxopt_b200.%s; "
            "assert 'torch' in sys.modules" % name)
    subprocess.run([sys.executable, "-c", code], check=True,
                   cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _theta_ctx(F, params, B=3, n=4, mnl=1):
    import types
    import torch
    return types.SimpleNamespace(x=torch.linspace(-1, 1, B * n, dtype=torch.float64).reshape(B, n),
                                 znl=torch.full((B, mnl), 0.5, dtype=torch.float64), F=F, params=params)


@pytest.mark.parametrize("cpl", [False, True])
def test_theta_grads_of_params_that_f_does_not_use_are_zeros(cpl):
    """the parameters' backward on the host: a param F ignores gets zeros, also when it is the only one that needs a
    gradient (phi then has no graph at all), and so does every param of a cpl problem with mnl = 0 (f and Df empty)"""
    import torch
    from cvxopt_b200.layer import _theta_grads
    B, n = 3, 4
    w = torch.arange(1.0, B * n + 1, dtype=torch.float64).reshape(B, n)
    unused = torch.ones((B, 2), dtype=torch.float64)
    nf = 1 if cpl else 2

    def F(x, idx=None, params=()):                       # f_i = w'x for every row, params[0] unused
        return (params[1] * x).sum(1, keepdim=True).repeat(1, nf), params[1][:, None, :].repeat(1, nf, 1)
    ux = torch.linspace(0.5, 2.0, B * n, dtype=torch.float64).reshape(B, n)
    uz = torch.full((B, 1), 0.25, dtype=torch.float64)
    only_unused = _theta_grads(_theta_ctx(F, (unused, w)), ux, uz, cpl, (True, False))
    assert only_unused[1] is None and torch.equal(only_unused[0], torch.zeros_like(unused))
    both = _theta_grads(_theta_ctx(F, (unused, w)), ux, uz, cpl, (True, True))
    assert torch.equal(both[0], torch.zeros_like(unused))
    zk = torch.full((B, 1), 0.5, dtype=torch.float64)
    if cpl:
        want = -(zk * ux + uz * _theta_ctx(F, ()).x)
    else:
        want = -(ux + zk * ux + uz * _theta_ctx(F, ()).x)
    assert torch.allclose(both[1], want, rtol=1e-15, atol=1e-15)

    def F0(x, idx=None, params=()):                      # a cpl problem without nonlinear rows
        return x.new_zeros((B, 0)), x.new_zeros((B, 0, n))
    none = _theta_grads(_theta_ctx(F0, (w,), mnl=0), ux, uz[:, :0], True, (True,))
    assert torch.equal(none[0], torch.zeros_like(w))
