"""The batch solver's limit of 65535 problems per library batch (CVXB_BATCH_MAX): the C entry points refuse
more before they look for a device, and QPBatchGroup splits larger batches into enough sub-batches."""
import ctypes as C

import numpy as np


def _gpu_visible():
    try:
        from cvxopt_b200 import _lib
        return _lib.load().cvxb_device_count() > 0
    except Exception:
        return False


def test_batch_create_rejects_more_than_65535_problems():
    """the batched kernels put the problem index in gridDim.y / .z (at most 65535); the size check comes before
    the device check, so it needs no GPU"""
    from cvxopt_b200 import _lib, kkt
    lib = _lib.load()
    h = C.c_void_p()
    assert lib.cvxb_batch_create(C.byref(h), 65536, 4, 8, 0) == _lib.E_ARG
    assert "65535" in _lib.last_error()
    d, keep, _, _ = kkt.make_dims({"l": 4, "q": [3], "s": []})
    assert lib.cvxb_batch_create_cones(C.byref(h), 65536, 4, C.byref(d), 0) == _lib.E_ARG
    assert "65535" in _lib.last_error()
    assert not h.value
    if not _gpu_visible():
        assert lib.cvxb_batch_create(C.byref(h), 65535, 4, 8, 0) == _lib.E_NOGPU
        assert lib.cvxb_batch_create_cones(C.byref(h), 65535, 4, C.byref(d), 0) == _lib.E_NOGPU


def test_batch_group_splits_past_the_limit(monkeypatch):
    """QPBatchGroup takes at least ceil(B / 65535) sub-batches, so qp_batch accepts any B"""
    from cvxopt_b200 import batch
    made = []

    class Fake:
        def __init__(self, nprob, n, m, device=0, dims=None):
            made.append(nprob)

        def close(self):
            pass
    monkeypatch.setattr(batch, "QPBatch", Fake)
    for B, nsub, want in ((65535, 1, 1), (65536, 1, 2), (131070, None, 2), (131071, None, 3), (200000, 2, 4),
                          (300, 5, 5), (3, 8, 3)):
        made.clear()
        g = batch.QPBatchGroup(B, 4, 8, nsub=nsub)
        assert g.nsub == want and len(made) == want, (B, nsub, g.nsub)
        assert sum(made) == B and max(made) <= 65535
        assert sorted(np.concatenate(g.idx).tolist()) == list(range(B))
