"""cvxopt_b200._misc_solvers — the CPython extension mirroring cvxopt.misc_solvers (SURVEY.md §8b secondary
boundary; reference src/C/misc_solvers.c:1155-1173, src/C/cvxopt.h:93-132).

CPU part: the module imports next to the reference (import_cvxopt() finds the base_API capsule), exports the 12
functions with the reference's keyword lists, rejects bad arguments with the reference's exception types, and
fails loudly (RuntimeError) when asked to compute without a GPU.
GPU part: the 12 functions are swapped into cvxopt.misc and the UNMODIFIED solvers run to the reference's
iteration count with the reference's own kktsolver names ('chol', 'qr', 'ldl'); concurrent host threads get the
results of one thread."""
import numpy as np
import pytest

from problems import cone_lp, cone_point, dense_qp

NAMES = ["scale", "scale2", "pack", "pack2", "unpack", "symm", "sprod", "sinv", "trisc", "triusc", "sdot",
         "max_step"]
KWLISTS = {  # reference src/C/misc_solvers.c:98, 267, 418, 482, 558, 614, 645, 781, 893, 946, 997, 1060
    "scale": ["x", "W", "trans", "inverse"], "scale2": ["lmbda", "x", "dims", "mnl", "inverse"],
    "pack": ["x", "y", "dims", "mnl", "offsetx", "offsety"], "pack2": ["x", "dims", "mnl"],
    "unpack": ["x", "y", "dims", "mnl", "offsetx", "offsety"], "symm": ["x", "n", "offset"],
    "sprod": ["x", "y", "dims", "mnl", "diag"], "sinv": ["x", "y", "dims", "mnl"],
    "trisc": ["x", "dims", "offset"], "triusc": ["x", "dims", "offset"], "sdot": ["x", "y", "dims", "mnl"],
    "max_step": ["x", "dims", "mnl", "sigma"]}


def _ext(ref):
    import cvxopt_b200._misc_solvers as ms
    return ms


def test_extension_imports_and_mirrors_the_method_table(ref):
    ms = _ext(ref)
    import cvxopt.misc_solvers as ref_ms
    assert sorted(ms.__all__) == sorted(NAMES)
    for name in NAMES:
        assert callable(getattr(ms, name)) and callable(getattr(ref_ms, name))
        assert name + "(" in getattr(ms, name).__doc__


def test_extension_keyword_lists_and_error_types(ref):
    """every keyword of the reference's kwlist is accepted (the call then fails only for lack of a GPU or
    passes), an unknown keyword is a TypeError, a non-matrix argument is a TypeError."""
    ms = _ext(ref)
    from cvxopt import matrix
    import cvxopt_b200
    dims = {"l": 2, "q": [3], "s": [2]}
    x = matrix(1.0, (9, 1))
    lm = matrix(1.0, (5, 1))
    W = {"d": matrix(1.0, (2, 1)), "di": matrix(1.0, (2, 1)), "v": [matrix([1.0, 0.0, 0.0])], "beta": [1.0],
         "r": [matrix([1.0, 0.0, 0.0, 1.0], (2, 2))], "rti": [matrix([1.0, 0.0, 0.0, 1.0], (2, 2))]}
    calls = {
        "scale": dict(x=x, W=W, trans="N", inverse="N"),
        "scale2": dict(lmbda=lm, x=x, dims=dims, mnl=0, inverse="N"),
        "pack": dict(x=x, y=matrix(0.0, (8, 1)), dims=dims, mnl=0, offsetx=0, offsety=0),
        "pack2": dict(x=x, dims=dims, mnl=0),
        "unpack": dict(x=matrix(1.0, (8, 1)), y=matrix(0.0, (9, 1)), dims=dims, mnl=0, offsetx=0, offsety=0),
        "symm": dict(x=matrix(1.0, (4, 1)), n=2, offset=0),
        "sprod": dict(x=x, y=matrix(1.0, (9, 1)), dims=dims, mnl=0, diag="N"),
        "sinv": dict(x=x, y=lm, dims=dims, mnl=0),
        "trisc": dict(x=x, dims=dims, offset=0), "triusc": dict(x=x, dims=dims, offset=0),
        "sdot": dict(x=x, y=matrix(1.0, (9, 1)), dims=dims, mnl=0),
        "max_step": dict(x=x, dims=dims, mnl=0, sigma=None)}
    have_gpu = cvxopt_b200.device_count() > 0
    for name in NAMES:
        assert sorted(calls[name]) == sorted(KWLISTS[name])
        f = getattr(ms, name)
        if have_gpu:
            f(**calls[name])
        else:
            with pytest.raises(RuntimeError):         # no CPU fallback: loud failure, not a silent route
                f(**calls[name])
        with pytest.raises(TypeError):
            f(**dict(calls[name], no_such_keyword=1))
        bad = dict(calls[name])
        bad["x"] = [1.0, 2.0]
        with pytest.raises(TypeError):
            f(**bad)
    with pytest.raises(KeyError):                     # misc_solvers.c:134
        ms.scale(x, {"v": [], "beta": [], "r": [], "rti": []})
    with pytest.raises(TypeError):                    # buffer too short
        ms.pack(matrix(1.0, (3, 1)), matrix(0.0, (8, 1)), dims)


@pytest.fixture
def swapped(ref):
    """cvxopt.misc.<name> rebound to the extension for the duration of a test (misc.kkt_* and coneprog resolve
    misc.<name> at call time: misc.py:27-28 ..., coneprog.py:605 ...)"""
    ms = _ext(ref)
    from cvxopt import misc
    saved = {n: getattr(misc, n) for n in NAMES}
    for n in NAMES:
        setattr(misc, n, getattr(ms, n))
    try:
        yield ms
    finally:
        for n in NAMES:
            setattr(misc, n, saved[n])


def _solve_both(ref, run):
    from cvxopt import misc
    want = run()
    ms = _ext(ref)
    saved = {n: getattr(misc, n) for n in NAMES}
    import cvxopt_b200
    for n in NAMES:
        setattr(misc, n, getattr(ms, n))
    try:
        before = cvxopt_b200.launch_count()
        got = run()
        launched = cvxopt_b200.launch_count() - before
    finally:
        for n in NAMES:
            setattr(misc, n, saved[n])
    assert launched > 0
    return want, got


@pytest.mark.gpu
def test_unmodified_coneqp_chol_with_the_extension_swapped_in(ref):
    from cvxopt import matrix, solvers
    P, q, G, h = dense_qp(40, 90, seed=5)
    args = (matrix(P), matrix(q), matrix(G), matrix(h), {"l": 90, "q": [], "s": []})
    want, got = _solve_both(ref, lambda: solvers.coneqp(*args, kktsolver="chol"))
    assert want["status"] == got["status"] == "optimal" and want["iterations"] == got["iterations"]
    np.testing.assert_allclose(got["primal objective"], want["primal objective"], rtol=1e-8)
    np.testing.assert_allclose(np.array(got["x"]), np.array(want["x"]), rtol=1e-7, atol=1e-9)


@pytest.mark.gpu
@pytest.mark.parametrize("solver", ["chol", "qr", "ldl"])
def test_unmodified_sdp_and_socp_with_the_extension_swapped_in(ref, solver):
    """solvers.sdp / solvers.socp with the reference's own kktsolver names: every scale / pack / sprod / sinv /
    max_step (eigenvalues + eigenvectors of the 's' blocks) call goes to the GPU."""
    from cvxopt import matrix, solvers
    n = 9
    dims = {"l": 3, "q": [], "s": [5, 3]}
    c, G, h = cone_lp(n, dims, seed=21)
    Gm, hm = matrix(G), matrix(h)
    Gl, hl = Gm[:3, :], hm[:3]
    Gs = [Gm[3:28, :], Gm[28:37, :]]
    hs = [matrix(hm[3:28], (5, 5)), matrix(hm[28:37], (3, 3))]
    want, got = _solve_both(ref, lambda: solvers.sdp(matrix(c), Gl, hl, Gs, hs, kktsolver=solver))
    assert want["status"] == got["status"] == "optimal" and want["iterations"] == got["iterations"]
    np.testing.assert_allclose(got["primal objective"], want["primal objective"], rtol=1e-7)
    dims = {"l": 3, "q": [4, 6], "s": []}
    c, G, h = cone_lp(n, dims, seed=22)
    Gm, hm = matrix(G), matrix(h)
    Gq, hq = [Gm[3:7, :], Gm[7:13, :]], [hm[3:7], hm[7:13]]
    want, got = _solve_both(ref, lambda: solvers.socp(matrix(c), Gm[:3, :], hm[:3], Gq, hq, kktsolver=solver))
    assert want["status"] == got["status"] == "optimal" and want["iterations"] == got["iterations"]
    np.testing.assert_allclose(got["primal objective"], want["primal objective"], rtol=1e-7)


@pytest.mark.gpu
def test_concurrent_host_threads_get_single_thread_results():
    """The entry points without a handle share one stream per device and hold its lock for the whole call.  Two
    host threads calling cvxopt_b200.misc_solvers at once (ctypes releases the GIL, so the calls overlap in the
    library) must get, bit for bit, what the same calls give from one thread."""
    import threading
    from cvxopt_b200 import misc_solvers as ms
    dims = {"l": 5, "q": [4, 3], "s": [3, 70]}       # 70: the multi-launch Jacobi eigensolver of max_step

    def inputs(seed):
        rng = np.random.Generator(np.random.PCG64(seed))
        lam = [rng.uniform(0.5, 2.0, dims["l"])]
        lam += [np.concatenate([[2.0], rng.uniform(-0.5, 0.5, k - 1) / k]) for k in dims["q"]]
        lam += [rng.uniform(0.5, 2.0, k) for k in dims["s"]]
        return cone_point(dims, rng), cone_point(dims, rng), np.concatenate(lam)

    def calls(x, y, lam):
        out = []
        v = x.copy()
        ms.scale2(lam, v, dims)
        out.append(v)
        out.append(np.array([ms.sdot(x, y, dims)]))
        v = x.copy()
        ms.sprod(v, y, dims)
        out.append(v)
        v, sig = x.copy(), np.zeros(sum(dims["s"]))
        out += [np.array([ms.max_step(v, dims, sigma=sig)]), v, sig]
        return out

    data = [inputs(31), inputs(32)]                  # each thread its own inputs
    want = [calls(*d) for d in data]
    errors, start = [], threading.Barrier(2)

    def worker(t):
        try:
            start.wait()
            for it in range(40):
                got = calls(*data[t])
                for k, (g, w) in enumerate(zip(got, want[t])):
                    if g.tobytes() != w.tobytes():
                        errors.append("thread %d, iteration %d, result %d differs" % (t, it, k))
                        return
        except Exception as e:           # noqa: BLE001 - reported by the main thread
            errors.append("thread %d: %r" % (t, e))

    threads = [threading.Thread(target=worker, args=(t,)) for t in range(2)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
