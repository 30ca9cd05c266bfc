"""Equality constraints A x = b in the batch solver, without a GPU: argument checks that run before any device work,
the new C entry points' CVXB_E_ARG before CVXB_E_NOGPU, and y through the two-rank scatter / gather."""
import ctypes as C
import os
import socket

import numpy as np
import pytest


def _gpu_visible():
    try:
        from cvxopt_b200 import _lib
        return _lib.load().cvxb_device_count() > 0
    except Exception:
        return False


def _batch(B=3, n=5, m=7, p=2, seed=0):
    rng = np.random.default_rng(seed)
    M = rng.standard_normal((B, n, n))
    P = np.einsum("bij,bkj->bik", M, M) + np.eye(n)
    return (P, rng.standard_normal((B, n)), rng.standard_normal((B, m, n)), 10.0 + rng.standard_normal((B, m)),
            rng.standard_normal((B, p, n)), rng.standard_normal((B, p)))


def test_qp_batch_checks_A_and_b_before_the_device(monkeypatch):
    """shape errors are coneqp's TypeErrors and come before any batch object exists"""
    import cvxopt_b200
    from cvxopt_b200 import batch

    def no_device(*a, **k):
        raise AssertionError("device work before the argument checks")
    monkeypatch.setattr(batch, "QPBatchGroup", no_device)
    P, q, G, h, A, b = _batch()
    for bad in (dict(A=A), dict(b=b), dict(A=A[:, :, :4], b=b), dict(A=A[:2], b=b), dict(A=A, b=b[:, :1]),
                dict(A=A[0], b=b)):
        with pytest.raises(TypeError):
            cvxopt_b200.qp_batch(P, q, G, h, **bad)


def test_qpbatch_rejects_bad_p():
    from cvxopt_b200 import QPBatch
    with pytest.raises(TypeError):
        QPBatch(2, 5, 7, p=1.5)
    with pytest.raises(ValueError, match="p must be nonnegative"):
        QPBatch(2, 5, 7, p=-1)
    with pytest.raises(ValueError, match=r"Rank\(A\) < p"):
        QPBatch(2, 5, 7, p=6)


def test_create_eq_argument_errors_come_before_the_device_check():
    from cvxopt_b200 import _lib, kkt
    lib = _lib.load()
    h = C.c_void_p()
    d, keep, _, _ = kkt.make_dims({"l": 4, "q": [3], "s": []})
    assert lib.cvxb_batch_create_eq(C.byref(h), 2, 4, -1, C.byref(d), 0) == _lib.E_ARG
    assert lib.cvxb_batch_create_eq(C.byref(h), 2, 4, 5, C.byref(d), 0) == _lib.E_ARG
    assert "Rank(A) < p" in _lib.last_error()
    assert lib.cvxb_batch_create_eq(C.byref(h), 65536, 4, 2, C.byref(d), 0) == _lib.E_ARG
    assert "65535" in _lib.last_error()
    bad = _lib.Dims(mnl=1, ml=4)                 # the batch has no nonlinear rows
    assert lib.cvxb_batch_create_eq(C.byref(h), 2, 4, 2, C.byref(bad), 0) == _lib.E_ARG
    assert lib.cvxb_batch_create_eq(None, 2, 4, 2, C.byref(d), 0) == _lib.E_ARG
    assert lib.cvxb_batch_load_eq(None, None, None, _lib.HOST) == _lib.E_ARG
    assert lib.cvxb_batch_results_y(None, None, _lib.HOST) == _lib.E_ARG
    assert not h.value
    if not _gpu_visible():
        assert lib.cvxb_batch_create_eq(C.byref(h), 2, 4, 2, C.byref(d), 0) == _lib.E_NOGPU
        assert lib.cvxb_batch_create_eq(C.byref(h), 2, 4, 0, C.byref(d), 0) == _lib.E_NOGPU


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _standin_eq(P, q, G, h, A, b):
    """min 1/2 x'Px + q'x s.t. A x = b in closed form (the inequalities are slack): [P A'; A 0] [x; y] = [-q; b]"""
    B, n = q.shape
    p = b.shape[1]
    xs, ys = np.zeros((B, n)), np.zeros((B, p))
    for k in range(B):
        K = np.block([[P[k], A[k].T], [A[k], np.zeros((p, p))]])
        sol = np.linalg.solve(K, np.concatenate([-q[k], b[k]]))
        xs[k], ys[k] = sol[:n], sol[n:]
    s = h - np.einsum("bmn,bn->bm", G, xs)
    f = 0.5 * np.einsum("bn,bnk,bk->b", xs, P, xs) + np.einsum("bn,bn->b", q, xs)
    return {"x": xs, "y": ys, "s": s, "z": np.zeros_like(s), "status_code": np.ones(B, np.int32),
            "iterations": np.arange(B, dtype=np.int32), "primal objective": f, "dual objective": f}


def _worker(rank, world, port, nprob, ret):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from cvxopt_b200.batch import qp_batch_distributed
    P, q, G, h, A, b = _batch(nprob, 6, 9, 3, seed=11)
    args = (P, q, G, h, A, b) if rank == 0 else (None,) * 6
    res = qp_batch_distributed(*args, solver=_standin_eq)
    if rank == 0:
        want = _standin_eq(P, q, G, h, A, b)
        ret["ok"] = bool(np.allclose(res["all"]["x"], want["x"], rtol=1e-12, atol=1e-12)
                         and np.allclose(res["all"]["y"], want["y"], rtol=1e-12, atol=1e-12)
                         and res["all"]["y"].shape == (nprob, 3))
        ret["shard0"] = res["y"].shape
    dist.destroy_process_group()


@pytest.mark.parametrize("nprob", [7, 2])
def test_distributed_gathers_y_in_the_original_order(nprob):
    """rank 0 owns problems 0, 2, 4, ...: y comes back in problem order, next to x"""
    import torch.multiprocessing as mp
    mgr = mp.Manager()
    ret = mgr.dict()
    port = _free_port()
    ctx = mp.get_context("spawn")
    procs = [ctx.Process(target=_worker, args=(r, 2, port, nprob, ret)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(120)
        assert p.exitcode == 0
    assert ret["ok"]
    assert ret["shard0"] == ((nprob + 1) // 2, 3)
