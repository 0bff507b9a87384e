"""CPU checks of the forward derivative's restatement (tests/solve_derivative_reference.py, DESIGN.md §3l): against
central differences of oracle solves, the pairing <g, J d> = <J' g, d> with the adjoint's restatement (unscaled and
scaled), independence of rho, sigma and the scaling, the half split of a Box row with l = u, and the C binding."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import cosmo_oracle as O
from tests import solve_adjoint_reference as SA
from tests import solve_derivative_reference as SD
from tests.test_solve_adjoint_cpu import _mixed_problem, _oracle

OUT = ("dx", "dy", "ds")


def _sym_direction(P, rng):
    """A symmetric direction of P on its stored pattern (both triangles move together)."""
    n = P.shape[0]
    S = rng.standard_normal((n, n))
    S = S + S.T
    return S[P.indices, np.repeat(np.arange(n), np.diff(P.indptr))], S


def _direction(P, A, m, rng):
    n = A.shape[1]
    dPx, _ = _sym_direction(P, rng)
    return dict(dPx=dPx, dq=rng.standard_normal(n), dAx=rng.standard_normal(A.nnz), db=rng.standard_normal(m),
                dl=rng.standard_normal(m), du=rng.standard_normal(m))


@pytest.mark.parametrize("seed", [0, 1])
def test_derivative_against_finite_differences(seed):
    P, q, A, b, cones = _mixed_problem(seed)
    m, n = A.shape
    r0 = _oracle(P, q, A, b, cones)
    warm = (r0.x, r0.s, r0.y)
    rng = np.random.default_rng(20 + seed)
    eps = 1e-6

    def fd(make):
        rp, rm = _oracle(*make(eps), warm=warm), _oracle(*make(-eps), warm=warm)
        return {"dx": (rp.x - rm.x) / (2 * eps), "dy": (rp.y - rm.y) / (2 * eps), "ds": (rp.s - rm.s) / (2 * eps)}

    def check(got, want):
        assert got["residual"] <= 1e-10
        for k in OUT:
            assert np.abs(got[k] - want[k]).max() <= 1e-5 * (1 + np.abs(want[k]).max()), (k, got[k], want[k])

    at = lambda **d: SD.unscaled(P, A, cones, r0.x, r0.s, r0.y, **d)
    dq = rng.standard_normal(n)
    check(at(dq=dq), fd(lambda e: (P, q + e * dq, A, b, cones)))
    db = rng.standard_normal(m)
    check(at(db=db), fd(lambda e: (P, q, A, b + e * db, cones)))
    dA = rng.standard_normal(A.nnz)
    check(at(dAx=dA), fd(lambda e: (P, q, sp.csc_matrix((A.data + e * dA, A.indices, A.indptr), shape=A.shape), b, cones)))
    dPx, S = _sym_direction(P, rng)
    check(at(dPx=dPx), fd(lambda e: (P + e * sp.csc_matrix(S), q, A, b, cones)))
    box = cones[1]
    for which in ("l", "u"):
        d = rng.standard_normal(box.dim)
        full = np.zeros(m)
        full[2:5] = d

        def make(e, which=which, d=d):
            l, u = box.l + (e * d if which == "l" else 0), box.u + (e * d if which == "u" else 0)
            return P, q, A, b, [cones[0], O.Box(l, u)] + cones[2:]
        check(at(**{"d" + which: full}), fd(make))


def _pairing(fwd, adj, g, d):
    lhs = sum(gk @ fwd[k] for gk, k in zip(g, OUT))
    rhs = sum(adj[k] @ d[k] for k in ("dPx", "dq", "dAx", "db", "dl", "du"))
    return lhs, rhs


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("rho", [0.1, 0.01])
def test_pairing_with_the_adjoint(seed, rho):
    P, q, A, b, cones = _mixed_problem(seed)
    m, n = A.shape
    r0 = _oracle(P, q, A, b, cones)
    rng = np.random.default_rng(30 + seed)
    for _ in range(3):
        g = (rng.standard_normal(n), rng.standard_normal(m), rng.standard_normal(m))
        d = _direction(P, A, m, rng)
        fwd = SD.unscaled(P, A, cones, r0.x, r0.s, r0.y, rho=rho, **d)
        adj = SA.unscaled(P, A, cones, r0.x, r0.s, r0.y, rho=rho, gx=g[0], gy=g[1], gs=g[2])
        lhs, rhs = _pairing(fwd, adj, g, d)
        assert abs(lhs - rhs) <= 1e-10 * (abs(lhs) + abs(rhs)), (lhs, rhs)


def _scaled(P, A, cones, r0, rng):
    """A Ruiz-like scaling of the mixed problem: scaled data, cones and point (cones scaled by one scalar)."""
    m, n = A.shape
    D = np.exp(rng.uniform(-0.5, 0.5, n))
    e = np.exp(rng.uniform(-0.5, 0.5))
    Ev = np.concatenate([np.exp(rng.uniform(-0.5, 0.5, 5)), np.full(m - 5, e)])
    c = 0.7
    Ps = sp.csc_matrix(c * sp.diags(D) @ P @ sp.diags(D))
    As = sp.csc_matrix(sp.diags(Ev) @ A @ sp.diags(D))
    box = cones[1]
    cs = [cones[0], O.Box(Ev[2:5] * box.l, Ev[2:5] * box.u)] + cones[2:]
    return Ps, As, cs, r0.x / D, Ev * r0.s, -c * r0.y / Ev, dict(D=D, E=Ev, c=c)


def test_pairing_with_the_adjoint_scaled():
    P, q, A, b, cones = _mixed_problem(0)
    m, n = A.shape
    r0 = _oracle(P, q, A, b, cones)
    rng = np.random.default_rng(4)
    Ps, As, cs, xs, ss, mus, sc = _scaled(P, A, cones, r0, rng)
    for _ in range(3):
        g = (rng.standard_normal(n), rng.standard_normal(m), rng.standard_normal(m))
        d = _direction(P, A, m, rng)
        fwd = SD.derivative(Ps, As, cs, xs, ss, mus, 0.1, **d, **sc)
        adj = SA.adjoint(Ps, As, cs, xs, ss, mus, 0.1, gx=g[0], gy=g[1], gs=g[2], **sc)
        lhs, rhs = _pairing(fwd, adj, g, d)
        assert abs(lhs - rhs) <= 1e-10 * (abs(lhs) + abs(rhs)), (lhs, rhs)


def test_independent_of_rho_sigma_and_scaling():
    P, q, A, b, cones = _mixed_problem(1)
    m, n = A.shape
    r0 = _oracle(P, q, A, b, cones)
    rng = np.random.default_rng(6)
    d = _direction(P, A, m, rng)
    a = SD.unscaled(P, A, cones, r0.x, r0.s, r0.y, rho=0.1, sigma=1e-6, **d)
    rho = np.where(np.arange(m) < 2, 100.0, 0.01)
    b_ = SD.unscaled(P, A, cones, r0.x, r0.s, r0.y, rho=rho, sigma=1e-3, **d)
    Ps, As, cs, xs, ss, mus, sc = _scaled(P, A, cones, r0, rng)
    s_ = SD.derivative(Ps, As, cs, xs, ss, mus, 0.1, **d, **sc)
    for k in OUT:
        np.testing.assert_allclose(a[k], b_[k], atol=1e-8 * (1 + np.abs(a[k]).max()))
        np.testing.assert_allclose(a[k], s_[k], atol=1e-8 * (1 + np.abs(a[k]).max()))


def test_box_row_with_equal_bounds():
    """min 1/2 |x|^2 + q'x with x0 fixed by a Box row l = u: moving both bounds moves x0 by their mean, and the pairing
    with the adjoint's half split holds."""
    P = sp.csc_matrix(np.eye(2))
    q = np.array([0.3, -0.2])
    A = sp.csc_matrix(np.array([[1.0, 0.0], [0.0, 1.0]]))
    b = np.zeros(2)
    cones = [O.Box(np.array([0.5, -1.0]), np.array([0.5, 1.0]))]
    r0 = _oracle(P, q, A, b, cones)
    assert abs(r0.s[0] - 0.5) <= 1e-9
    for dl, du in (([1.0, 0.0], [0.0, 0.0]), ([0.0, 0.0], [1.0, 0.0]), ([0.4, 0.0], [1.2, 0.0])):
        got = SD.unscaled(P, A, cones, r0.x, r0.s, r0.y, dl=np.array(dl), du=np.array(du))
        assert abs(got["ds"][0] - 0.5 * (dl[0] + du[0])) <= 1e-9, (dl, du, got["ds"])
        assert abs(got["dx"][0] + 0.5 * (dl[0] + du[0])) <= 1e-9   # x0 = b0 - s0
    rng = np.random.default_rng(8)
    g = (rng.standard_normal(2), rng.standard_normal(2), rng.standard_normal(2))
    d = dict(dPx=np.zeros(2), dq=np.zeros(2), dAx=np.zeros(2), db=np.zeros(2), dl=rng.standard_normal(2),
             du=rng.standard_normal(2))
    fwd = SD.unscaled(P, A, cones, r0.x, r0.s, r0.y, **d)
    adj = SA.unscaled(P, A, cones, r0.x, r0.s, r0.y, gx=g[0], gy=g[1], gs=g[2])
    lhs, rhs = _pairing(fwd, adj, g, d)
    assert abs(lhs - rhs) <= 1e-10 * (abs(lhs) + abs(rhs))


def test_binding():
    import cosmo_b200
    E = cosmo_b200.engine
    restype, argtypes = E._signatures()["cosmo_b200_solve_derivative"]
    assert restype == C.c_int and len(argtypes) == 12
    assert argtypes[1] == C.POINTER(E.SolveAdjointSettings) and argtypes[-1] == C.POINTER(C.c_double)
    assert all(a == C.c_void_p for a in argtypes[2:11])
    with open(__file__.replace("tests/test_solve_derivative_cpu.py", "include/cosmo_b200.h")) as f:
        assert ("int cosmo_b200_solve_derivative(cosmo_b200_handle* h, const cosmo_b200_solve_adjoint_settings* as, "
                "const double* dPx,\n                                const double* dq, const double* dAx, const double* db, "
                "const double* dl, const double* du,\n                                double* dx, double* dy, double* ds, "
                "double out[8]);") in f.read()
