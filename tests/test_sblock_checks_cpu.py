"""CPU: the long double checkers of the batch solver's 's' block kernels (tests/ld_check.py) pass the reference's own
fp64 results (misc.compute_scaling / misc.update_scaling of oracle/_ref, scipy.linalg.eigh, LAPACK gesvd, numpy's
products) and fail on each way a kernel could be subtly wrong: one entry off by 1e-12 relative, a touched upper
triangle, NaN, an eigenvector paired with the wrong eigenvalue, r with one column's sign flipped but rti not."""
import numpy as np
import pytest
import scipy.linalg

from ld_check import (check_congruence, check_min_eig, check_nt_scaling, check_nt_update, check_sym_eig, pack_ld,
                      sym_lower)

ORDERS = [1, 2, 5, 16, 32]


def _spd(n, rng):
    B = rng.standard_normal((n, n))
    return B @ B.T / n + np.eye(n)


def _late(n, rng, mu=1e-6):
    """an IPM-like late iterate: s = Q diag(sig) Q', z = Q diag(mu / sig) Q' plus a small symmetric perturbation"""
    Q = np.linalg.qr(rng.standard_normal((n, n)))[0]
    sig = 10.0 ** rng.uniform(-8, 0, n)
    E = rng.standard_normal((n, n)) * 1e-3 * mu
    s = (Q * sig) @ Q.T
    z = (Q * (mu / sig)) @ Q.T + (E + E.T) / 2 * 1e-2
    return sym_lower(s), sym_lower(z)


def _ref_scaling(ref, s, z):
    from cvxopt import matrix, misc
    n = s.shape[0]
    lam = matrix(0.0, (n, 1))
    W = misc.compute_scaling(matrix(s.reshape(-1, order="F")), matrix(z.reshape(-1, order="F")), lam,
                             {"l": 0, "q": [], "s": [n]})
    return np.array(W["r"][0]), np.array(W["rti"][0]), np.array(lam).ravel(), W


def _cases(n, seed):
    rng = np.random.default_rng(seed)
    return [(_spd(n, rng), _spd(n, rng)), _late(n, rng)]


@pytest.mark.parametrize("n", ORDERS)
def test_nt_scaling_passes_the_reference_and_fails_perturbations(ref, n):
    for late, (s, z) in enumerate(_cases(n, 10 + n)):
        r, rti, lam, _ = _ref_scaling(ref, s, z)
        m = check_nt_scaling(s, z, r, rti, lam)
        print("nt_scaling n=%d late=%d: %.3g" % (n, late, m))
        i = n // 2
        # on the late iterates (kappa(s), kappa(z) ~ 1e8) the smallest relative error detected is 1e-12 up to order 16
        # and 1e-11 at order 32, where kappa enters the lambda bound and the products' magnitudes outgrow the result
        d = 1e-11 if late and n > 16 else 1e-12
        bad_l = lam.copy(); bad_l[i] *= 1 + d
        bad_r = r.copy(); bad_r[np.argmax(np.abs(r[:, i])), i] *= 1 + d
        bad_t = rti.copy(); bad_t[np.argmax(np.abs(rti[:, i])), i] *= 1 + d
        nan_r = r.copy(); nan_r[0, -1] = np.nan
        for args in ((r, rti, bad_l), (bad_r, rti, lam), (r, bad_t, lam), (nan_r, rti, lam)):
            with pytest.raises(AssertionError):
                check_nt_scaling(s, z, *args)
        flip = r.copy(); flip[:, i] *= -1               # r' rti no longer I
        with pytest.raises(AssertionError):
            check_nt_scaling(s, z, flip, rti, lam)
        if n > 1 and abs(lam[0] - lam[-1]) > 1e-9 * lam.max():
            swap = lam.copy(); swap[[0, -1]] = swap[[-1, 0]]     # lambda out of step with r's columns
            with pytest.raises(AssertionError):
                check_nt_scaling(s, z, r, rti, swap)


@pytest.mark.parametrize("n", ORDERS)
def test_nt_update_passes_the_reference_and_fails_perturbations(ref, n):
    from cvxopt import matrix, misc
    rng = np.random.default_rng(20 + n)
    for late, (s0, z0) in enumerate(_cases(n, 30 + n)):
        r0, rti0, lam0, W = _ref_scaling(ref, s0, z0)
        step = 0.97
        Ds, Dz = rng.standard_normal((n, n)), rng.standard_normal((n, n))
        sigs, Qs = np.linalg.eigh(Ds + Ds.T)
        sigz, Qz = np.linalg.eigh(Dz + Dz.T)
        sigs, sigz = sigs / (2 * np.abs(sigs).max()), sigz / (2 * np.abs(sigz).max())   # 1 + step sig > 0
        Ls = np.sqrt(lam0)[:, None] * Qs * np.sqrt(1 + step * sigs)
        Lz = np.sqrt(lam0)[:, None] * Qz * np.sqrt(1 + step * sigz)
        lam = matrix(lam0.copy())
        misc.update_scaling(W, lam, matrix(Ls.reshape(-1, order="F")), matrix(Lz.reshape(-1, order="F")))
        r, rti, lam = np.array(W["r"][0]), np.array(W["rti"][0]), np.array(lam).ravel()
        s, z = sym_lower((r * lam) @ r.T), sym_lower((rti * lam) @ rti.T)
        args = (r0, rti0, lam0, Qs, sigs, Qz, sigz, step)
        m = check_nt_update(*args, s, z, r, rti, lam)
        print("nt_update n=%d late=%d: %.3g" % (n, late, m))
        i = n - 1
        # s+ and z+ are checked as sums, to 1e-12 on every family.  The new scaling is checked against them with the
        # inherited ||r0' rti0 - I|| added to its bound, and on the late iterates compute_scaling leaves that at about
        # kappa u ~ 1e-8: there the smallest relative error detected in r is 1e-12 up to order 5 and 1e-7 at 16 and 32,
        # in lambda 1e-11 at order 5, 1e-7 at 16 and 1e-6 at 32
        dr = 1e-7 if late and n >= 16 else 1e-12
        dl = ({5: 1e-11, 16: 1e-7, 32: 1e-6}.get(n, 1e-12)) if late else 1e-12
        bad = s.copy(); bad[i, i] *= 1 + 1e-12
        bad_r = r.copy(); bad_r[np.argmax(np.abs(r[:, 0])), 0] *= 1 + dr
        bad_l = lam.copy(); bad_l[0] *= 1 + dl
        upper = s.copy()
        if n > 1:
            upper[0, i] = np.nextafter(upper[0, i], np.inf)
        nan = z.copy(); nan[i, i] = np.nan
        for ss, zz, rr, ll in [(bad, z, r, lam), (s, nan, r, lam), (s, z, bad_r, lam), (s, z, r, bad_l)] + \
                ([(upper, z, r, lam)] if n > 1 else []):
            with pytest.raises(AssertionError):
                check_nt_update(*args, ss, zz, rr, rti, ll)
        flip = r.copy(); flip[:, 0] *= -1
        with pytest.raises(AssertionError):
            check_nt_update(*args, s, z, flip, rti, lam)


def _eig_inputs(n, rng):
    Q = np.linalg.qr(rng.standard_normal((n, n)))[0]
    w = np.ones(n); w[: n // 2] += 4 * np.finfo(float).eps      # a cluster a few ulps wide
    return [sym_lower(rng.standard_normal((n, n))),                # indefinite
            (Q * w) @ Q.T, np.eye(n) + np.outer(Q[:, 0], Q[:, 0]), np.diag(rng.standard_normal(n))]


@pytest.mark.parametrize("driver", ["evd", "ev"])
@pytest.mark.parametrize("n", ORDERS)
def test_sym_eig_passes_lapack_and_fails_perturbations(n, driver):
    rng = np.random.default_rng(40 + n)
    for A in _eig_inputs(n, rng):
        A = sym_lower((A + A.T) / 2)
        w, V = scipy.linalg.eigh(A, driver=driver)
        m = check_sym_eig(A, V, w)
        check_min_eig(A, w[0])
        print("sym_eig n=%d %s: %.3g" % (n, driver, m))
        scale = np.abs(w).max()
        bad_w = w.copy(); bad_w[-1] += 1e-12 * scale
        bad_v = V.copy(); bad_v[np.argmax(np.abs(V[:, 0])), 0] *= 1 + 1e-12
        nan_v = V.copy(); nan_v[-1, 0] = np.nan
        for VV, ww in ((V, bad_w), (bad_v, w), (nan_v, w)):
            with pytest.raises(AssertionError):
                check_sym_eig(A, VV, ww)
        with pytest.raises(AssertionError):
            check_min_eig(A, w[0] + 1e-12 * scale)
        if n > 1 and w[-1] - w[0] > 1e-6 * scale:
            with pytest.raises(AssertionError):                 # a column paired with the wrong eigenvalue
                check_sym_eig(A, V[:, ::-1], w)


@pytest.mark.parametrize("n", [2, 16, 27, 32])
def test_sym_eig_fails_a_jacobi_stopped_at_1e13_off_diagonal_mass(n):
    """what two-sided Jacobi returns when it stops with off-diagonal mass E, ||E||_F = 1e-13 ||A||_F (jac_done's
    stagnation exit): V and the diagonal, while A = V (diag(w) + E) V'.  check_sym_eig must refuse it at every order"""
    from ld_check import LD, ld_eigh
    rng = np.random.default_rng(60 + n)
    w0, V0 = ld_eigh(sym_lower(rng.standard_normal((n, n))))
    E = np.tril(rng.standard_normal((n, n)).astype(LD), -1)
    E = E + E.T
    D = np.diag(w0) + E * (LD(1e-13) * np.sqrt(np.sum(w0 * w0)) / np.sqrt(np.sum(E * E)))
    A = (V0 @ D @ V0.T).astype(float)
    V, w = V0.astype(float), w0.astype(float)
    parts = {}
    with pytest.raises(AssertionError):
        check_sym_eig(A, V, w, parts=parts)
    E[:] = 0                                                # the same without the residue passes
    check_sym_eig((V0 @ np.diag(w0) @ V0.T).astype(float), V, w)


@pytest.mark.parametrize("n", ORDERS)
def test_congruence_passes_fp64_and_fails_perturbations(n):
    rng = np.random.default_rng(50 + n)
    A, X = rng.standard_normal((n, n)), sym_lower(rng.standard_normal((n, n)))
    for trans in (True, False):
        Y = A.T @ X @ A if trans else A @ X @ A.T
        Yp = pack_ld(sym_lower(Y))
        m = max(check_congruence(A, X, sym_lower(Y), trans), check_congruence(A, X, Yp, trans, packed=True))
        print("congruence n=%d: %.3g" % (n, m))
        bad = Yp.copy(); bad[-1] *= 1 + 1e-12
        with pytest.raises(AssertionError):
            check_congruence(A, X, bad, trans, packed=True)
        nan = sym_lower(Y); nan[0, 0] = np.nan
        with pytest.raises(AssertionError):
            check_congruence(A, X, nan, trans)
        if n > 1:
            up = sym_lower(Y); up[0, n - 1] += 1e-12 * np.abs(Y).max()     # the full result's upper triangle
            with pytest.raises(AssertionError):
                check_congruence(A, X, up, trans)
