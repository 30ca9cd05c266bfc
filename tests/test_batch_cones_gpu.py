"""Batch solver with second-order cones (csrc/batch_ipm.cu) vs the reference: a Python loop over
solvers.coneqp(P, q, G, h, dims, kktsolver='chol') (oracle/_ref) on the same problems — same status and iteration
count per problem, objectives to rtol 1e-8, x / s / z to the tolerances of test_batch_gpu.py."""
import ctypes as C

import numpy as np
import pytest

from problems import cone_point


def _full(dims):
    return {"l": dims.get("l", 0), "q": list(dims.get("q", [])), "s": list(dims.get("s", []))}


def cone_qp(n, dims, seed):
    """P = A0'A0/n + I; G, q, x0 ~ N(0,1); h = G x0 + s0 with s0 strictly inside the cones"""
    dims = _full(dims)
    rng = np.random.Generator(np.random.PCG64(seed))
    A0 = rng.standard_normal((n, n))
    P = A0.T @ A0 / n + np.eye(n)
    q = rng.standard_normal(n)
    m = dims["l"] + sum(dims["q"])
    G = rng.standard_normal((m, n))
    x0 = rng.standard_normal(n)
    h = G @ x0 + cone_point(dims, rng)
    return P, q, G, h


def make_batch(B, n, dims, seed0=0):
    parts = [cone_qp(n, dims, seed0 + k) for k in range(B)]
    return tuple(np.stack([p[i] for p in parts]) for i in range(4))


def ref_loop(P, q, G, h, dims, refinement=None):
    from cvxopt import matrix, solvers
    kw = {}
    if refinement is not None:
        kw["options"] = {"refinement": refinement, "show_progress": False}
    return [solvers.coneqp(matrix(P[k]), matrix(q[k]), matrix(G[k]), matrix(h[k]), _full(dims), kktsolver="chol", **kw)
            for k in range(P.shape[0])]


def assert_matches(got, want):
    for k, w in enumerate(want):
        assert got["status"][k] == w["status"] == "optimal"
        assert got["iterations"][k] == w["iterations"], (k, list(got["iterations"]), [v["iterations"] for v in want])
        np.testing.assert_allclose(got["primal objective"][k], w["primal objective"], rtol=1e-8)
        np.testing.assert_allclose(got["dual objective"][k], w["dual objective"], rtol=1e-8)
        np.testing.assert_allclose(got["x"][k], np.array(w["x"]).ravel(), rtol=1e-6, atol=1e-8)
        np.testing.assert_allclose(got["s"][k], np.array(w["s"]).ravel(), rtol=1e-5, atol=1e-7)
        np.testing.assert_allclose(got["z"][k], np.array(w["z"]).ravel(), rtol=1e-5, atol=1e-7)


CASES = [
    (5, 30, {"l": 20, "q": [5, 3, 10]}),
    (3, 150, {"l": 0, "q": [4] * 40}),                # two Cholesky blocks, no 'l' rows
    (2, 200, {"l": 64, "q": [1, 2, 300]}),            # cones of order 1 and 2, one longer than a CTA
    (1, 257, {"l": 100, "q": [50] * 4}),              # B == 1: the unbatched Cholesky
]


@pytest.mark.gpu
@pytest.mark.parametrize("B,n,dims", CASES)
def test_cone_batch_matches_reference_loop(ref, B, n, dims):
    import cvxopt_b200
    P, q, G, h = make_batch(B, n, dims, seed0=20 * B + n)
    got = cvxopt_b200.qp_batch(P, q, G, h, dims=dims)
    assert got["syrk_path"] == "dmma"
    assert_matches(got, ref_loop(P, q, G, h, dims))


@pytest.mark.gpu
@pytest.mark.parametrize("refinement", [0, 2])
def test_cone_batch_refinement_option(ref, refinement):
    import cvxopt_b200
    dims = {"l": 15, "q": [6, 4, 9]}
    P, q, G, h = make_batch(4, 40, dims, seed0=70)
    got = cvxopt_b200.qp_batch(P, q, G, h, dims=dims, refinement=refinement)
    assert_matches(got, ref_loop(P, q, G, h, dims, refinement=refinement))


@pytest.mark.gpu
def test_l_only_batch_with_refinement_stays_fused(ref):
    """refinement on an 'l'-only batch keeps di² in the SYRK (Gs is not formed); the reference is solvers.qp with
    the option"""
    import cvxopt_b200
    from cvxopt import matrix, solvers
    from problems import dense_qp
    parts = [dense_qp(35, 80, seed=90 + k) for k in range(3)]
    P, q, G, h = (np.stack([p[i] for p in parts]) for i in range(4))
    got = cvxopt_b200.qp_batch(P, q, G, h, refinement=1)
    want = [solvers.qp(matrix(P[k]), matrix(q[k]), matrix(G[k]), matrix(h[k]), kktsolver="chol",
                       options={"refinement": 1, "show_progress": False}) for k in range(3)]
    assert_matches(got, want)


@pytest.mark.gpu
def test_l_dims_selects_the_l_path():
    """dims={'l': m} is the plain batch: the same kernels, the same bits"""
    import cvxopt_b200
    from cvxopt_b200 import _lib
    from problems import dense_qp
    lib = _lib.load()
    parts = [dense_qp(40, 90, seed=110 + k) for k in range(4)]
    P, q, G, h = (np.stack([p[i] for p in parts]) for i in range(4))
    c0 = lib.cvxb_launch_count()
    plain = cvxopt_b200.qp_batch(P, q, G, h)
    c1 = lib.cvxb_launch_count()
    withd = cvxopt_b200.qp_batch(P, q, G, h, dims={"l": 90})
    c2 = lib.cvxb_launch_count()
    assert c2 - c1 == c1 - c0
    for key in ("x", "s", "z", "primal objective", "dual objective"):
        np.testing.assert_array_equal(withd[key], plain[key])
    assert list(withd["iterations"]) == list(plain["iterations"])


def _mixed(B, n, dims, seed0):
    P, q, G, h = make_batch(B, n, dims, seed0=seed0)
    for k in range(0, B, 3):             # mixed difficulty, as in test_compaction_of_finished_problems
        q[k] *= 1e3
        h[k] *= 1e-2
    return P, q, G, h


@pytest.mark.gpu
def test_cone_batch_compaction(monkeypatch):
    import cvxopt_b200
    from cvxopt_b200.batch import QPBatch
    B, n, dims = 12, 40, {"l": 30, "q": [5, 8, 3]}
    P, q, G, h = _mixed(B, n, dims, seed0=130)
    monkeypatch.setenv("CVXB_BATCH_COMPACT", "0")
    plain = cvxopt_b200.qp_batch(P, q, G, h, nsub=1, dims=dims)
    monkeypatch.setenv("CVXB_BATCH_COMPACT", "1")
    b = QPBatch(B, n, 46, 0, dims=dims)
    try:
        b.load(P, q, G, h)
        b.solve()
        r1 = b.results()
        b.solve()
        r2 = b.results()
    finally:
        b.close()
    assert len(set(plain["iterations"])) > 1
    for r in (r1, r2):
        assert list(r["iterations"]) == list(plain["iterations"])
        assert list(r["status_code"]) == list(plain["status_code"])
        np.testing.assert_array_equal(r["x"], plain["x"])
        np.testing.assert_array_equal(r["z"], plain["z"])
        np.testing.assert_array_equal(r["primal objective"], plain["primal objective"])


@pytest.mark.gpu
def test_cone_subbatches_match_single_batch():
    import cvxopt_b200
    dims = {"l": 25, "q": [7, 7, 12]}
    P, q, G, h = make_batch(7, 50, dims, seed0=150)
    one = cvxopt_b200.qp_batch(P, q, G, h, nsub=1, dims=dims)
    three = cvxopt_b200.qp_batch(P, q, G, h, nsub=3, dims=dims)
    assert three["nsub"] == 3
    assert list(one["iterations"]) == list(three["iterations"])
    np.testing.assert_allclose(three["x"], one["x"], rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(three["primal objective"], one["primal objective"], rtol=1e-12)


@pytest.mark.gpu
@pytest.mark.parametrize("B", [3, 1])
def test_cone_batch_frees_its_device_memory(B, monkeypatch):
    from cvxopt_b200 import _lib
    from cvxopt_b200.batch import QPBatch
    lib = _lib.load()
    monkeypatch.setenv("CVXB_BATCH_COMPACT", "1")
    n, dims = 40, {"l": 20, "q": [6, 10]}
    P, q, G, h = _mixed(B, n, dims, seed0=173)      # iterations 8, 7, 9 at B = 3

    def run():
        b = QPBatch(B, n, 36, 0, dims=dims)
        b.load(P, q, G, h)
        b.solve()
        return b, b.results()

    b, _ = run()
    b.close()
    base = lib.cvxb_device_bytes()
    b, r = run()
    assert lib.cvxb_device_bytes() > base
    if B > 1:
        assert len(set(r["iterations"])) > 1
    b.close()
    assert lib.cvxb_device_bytes() == base


@pytest.mark.gpu
def test_cone_batch_rank_deficient_raises():
    import cvxopt_b200
    n, dims = 20, {"l": 2, "q": [3]}
    P = np.zeros((1, n, n))
    q = np.ones((1, n))
    G = np.random.default_rng(0).standard_normal((1, 5, n))
    h = np.ones((1, 5))
    h[0, 2] = 5.0
    with pytest.raises(ValueError):
        cvxopt_b200.qp_batch(P, q, G, h, dims=dims)


@pytest.mark.gpu
def test_cone_distributed_entry_matches_qp_batch():
    import cvxopt_b200
    dims = {"l": 10, "q": [4, 6]}
    P, q, G, h = make_batch(9, 30, dims, seed0=190)
    want = cvxopt_b200.qp_batch(P, q, G, h, nsub=2, dims=dims)
    got = cvxopt_b200.qp_batch_distributed(P, q, G, h, nsub=2, dims=dims)["all"]
    assert list(got["iterations"]) == list(want["iterations"])
    np.testing.assert_allclose(got["x"], want["x"], rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(got["z"], want["z"], rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(got["primal objective"], want["primal objective"], rtol=1e-12)


# ---- without a GPU ----

def _gpu_visible():
    from cvxopt_b200 import _lib
    try:
        return _lib.load().cvxb_device_count() > 0
    except Exception:
        return False


def test_create_cones_without_gpu_reports_nogpu():
    if _gpu_visible():
        pytest.skip("a GPU is visible")
    from cvxopt_b200 import _lib, kkt
    lib = _lib.load()
    d, keep, _, _ = kkt.make_dims({"l": 4, "q": [3, 2], "s": []})
    h = C.c_void_p()
    rc = lib.cvxb_batch_create_cones(C.byref(h), 2, 5, C.byref(d), 0)
    assert rc == _lib.E_NOGPU
    assert "no CUDA device available" in _lib.last_error()
    # argument errors come first
    dq = (C.c_int * 1)(0)
    bad = _lib.Dims(0, 4, 1, C.cast(dq, _lib.c_int_p), 0, C.cast(dq, _lib.c_int_p))
    assert lib.cvxb_batch_create_cones(C.byref(h), 2, 5, C.byref(bad), 0) == _lib.E_ARG
    mnl = _lib.Dims(1, 4, 0, C.cast(dq, _lib.c_int_p), 0, C.cast(dq, _lib.c_int_p))
    assert lib.cvxb_batch_create_cones(C.byref(h), 2, 5, C.byref(mnl), 0) == _lib.E_ARG
    ds = (C.c_int * 1)(2)
    sd = _lib.Dims(0, 4, 0, C.cast(dq, _lib.c_int_p), 1, C.cast(ds, _lib.c_int_p))
    assert lib.cvxb_batch_create_cones(C.byref(h), 2, 5, C.byref(sd), 0) == _lib.E_UNSUP
    assert lib.cvxb_batch_set_refinement(None, 1) == _lib.E_ARG


def test_qp_batch_argument_errors_without_gpu():
    if _gpu_visible():
        pytest.skip("a GPU is visible")
    import cvxopt_b200
    P, q, G, h = make_batch(2, 6, {"l": 3, "q": [3]}, seed0=5)
    with pytest.raises(TypeError):
        cvxopt_b200.qp_batch(P, q, G[:, :5], h[:, :5], dims={"l": 3, "q": [3]})
    with pytest.raises(NotImplementedError):
        cvxopt_b200.qp_batch(P, q, G, h, dims={"l": 2, "q": [], "s": [2]})
    with pytest.raises(TypeError):
        cvxopt_b200.qp_batch(P, q, G, h, dims={"l": 6, "q": [0]})
