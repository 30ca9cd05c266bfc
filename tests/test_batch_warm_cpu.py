"""Warm starts without a GPU: the TypeErrors of qp_batch's and coneqp_batch's initvals, conelp_batch's and sdp_batch's
primalstart / dualstart, raised before any batch object exists, and the start calls of the C ABI on a NULL handle."""
import numpy as np
import pytest


def _no_device(*a, **k):
    raise AssertionError("device work before the argument checks")


@pytest.fixture
def no_groups(monkeypatch):
    from cvxopt_b200 import batch
    for name in ("QPBatchGroup", "SDPQPBatchGroup", "ConeLPBatchGroup", "SDPBatchGroup"):
        monkeypatch.setattr(batch, name, _no_device)


B, N, P_EQ = 3, 5, 2


def _qp(m=6):
    rng = np.random.default_rng(0)
    return dict(P=rng.standard_normal((B, N, N)), q=rng.standard_normal((B, N)), G=rng.standard_normal((B, m, N)),
                h=rng.standard_normal((B, m)), A=rng.standard_normal((B, P_EQ, N)), b=rng.standard_normal((B, P_EQ)))


BAD_INITVALS = [
    {"x": np.zeros((B, N + 1))}, {"x": np.zeros(N)}, {"s": np.zeros((B, 5))}, {"z": np.zeros((B + 1, 6))},
    {"y": np.zeros((B, P_EQ + 1))}, {"w": np.zeros((B, N))}, {"x": np.zeros((B, N)), "sl": np.zeros((B, 6))},
    [np.zeros((B, N))],
]


@pytest.mark.parametrize("initvals", BAD_INITVALS)
def test_qp_batch_initvals_type_errors(no_groups, initvals):
    import cvxopt_b200
    with pytest.raises(TypeError):
        cvxopt_b200.qp_batch(**_qp(), initvals=initvals)


@pytest.mark.parametrize("initvals", BAD_INITVALS)
def test_coneqp_batch_initvals_type_errors(no_groups, initvals):
    import cvxopt_b200
    args = _qp(m=6)
    args["G"], args["h"] = args["G"][:, :6], args["h"][:, :6]
    dims = {"l": 2, "s": [2]}                              # cdim = 2 + 4 = 6
    with pytest.raises(TypeError):
        cvxopt_b200.coneqp_batch(**args, dims=dims, initvals=initvals)


def _lp(m=6):
    rng = np.random.default_rng(1)
    return dict(c=rng.standard_normal((B, N)), G=rng.standard_normal((B, m, N)), h=rng.standard_normal((B, m)),
                A=rng.standard_normal((B, P_EQ, N)), b=rng.standard_normal((B, P_EQ)))


X, S, Y, Z = np.zeros((B, N)), np.ones((B, 6)), np.zeros((B, P_EQ)), np.ones((B, 6))


@pytest.mark.parametrize("start", [
    dict(primalstart={}), dict(primalstart={"x": X}), dict(primalstart={"s": S}),
    dict(primalstart={"x": X, "s": S, "z": Z}), dict(primalstart={"x": X[:, :4], "s": S}),
    dict(primalstart={"x": X, "s": S[:, :5]}), dict(primalstart=(X, S)),
    dict(dualstart={}), dict(dualstart={"y": Y}), dict(dualstart={"z": Z, "s": S}), dict(dualstart={"z": Z[:2]}),
    dict(dualstart={"z": Z, "y": Y[:, :1]}), dict(primalstart={"x": X, "s": S}, dualstart={"y": Y}),
])
def test_conelp_batch_start_type_errors(no_groups, start):
    import cvxopt_b200
    with pytest.raises(TypeError):
        cvxopt_b200.conelp_batch(**_lp(), **start)


def test_sdp_batch_start_type_errors(no_groups):
    import cvxopt_b200
    rng = np.random.default_rng(2)
    ml, ms = 2, [2, 3]
    c = rng.standard_normal((B, N))
    Gl, hl = rng.standard_normal((B, ml, N)), rng.standard_normal((B, ml))
    Gs = [rng.standard_normal((B, k * k, N)) for k in ms]
    hs = [np.stack([np.eye(k)] * B) for k in ms]
    A, b = rng.standard_normal((B, 1, N)), rng.standard_normal((B, 1))
    ss = [np.stack([np.eye(k)] * B) for k in ms]
    ok_p = {"x": X, "sl": np.ones((B, ml)), "ss": ss}
    ok_d = {"zl": np.ones((B, ml)), "zs": ss, "y": np.zeros((B, 1))}
    for start in (dict(primalstart={}), dict(primalstart={"x": X, "sl": np.ones((B, ml))}),
                  dict(primalstart={"sl": np.ones((B, ml)), "ss": ss}), dict(primalstart=dict(ok_p, s=S)),
                  dict(primalstart=dict(ok_p, ss=ss[:1])), dict(primalstart=dict(ok_p, ss=[ss[0], ss[0]])),
                  dict(primalstart=dict(ok_p, sl=np.ones((B, ml + 1)))), dict(dualstart={}),
                  dict(dualstart={"y": np.zeros((B, 1))}), dict(dualstart=dict(ok_d, zs=[z[:, :1] for z in ss])),
                  dict(dualstart=dict(ok_d, y=np.zeros((B, 2)))), dict(dualstart=dict(ok_d, z=Z)),
                  dict(primalstart=ok_p, dualstart=dict(ok_d, zl=None))):
        with pytest.raises(TypeError):
            cvxopt_b200.sdp_batch(c, Gl, hl, Gs, hs, A, b, **start)


def test_start_calls_on_a_null_handle():
    from cvxopt_b200 import _lib
    lib = _lib.load()
    x = np.zeros(4)
    assert lib.cvxb_batch_load_start(None, x.ctypes.data, None, None, None, _lib.HOST) == _lib.E_ARG
    assert lib.cvxb_batch_load_start(None, None, None, None, None, _lib.HOST) == _lib.E_ARG
    assert lib.cvxb_batch_clear_start(None) == _lib.E_ARG
    assert {"cvxb_batch_load_start", "cvxb_batch_clear_start"} <= set(_lib.exported_symbols())


def test_distributed_takes_no_start():
    import cvxopt_b200
    with pytest.raises(TypeError, match="initvals"):
        cvxopt_b200.batch.qp_batch_distributed(None, None, None, None, initvals={})
