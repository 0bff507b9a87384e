"""CPU checks of the solve adjoint's restatement (tests/solve_adjoint_reference.py, DESIGN.md §3k): the cone Jacobians
against central differences of the oracle's projections, the gradients against central differences of oracle solves,
their independence of rho, sigma and the scaling, agreement with the polish adjoint on a QP, and the C binding."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import cosmo_oracle as O
from tests import solve_adjoint_reference as SA


def _fd_jacobian(cones, w, h, eps=1e-7):
    def proj(v):
        v = v.copy()
        O.project(v, cones)
        return v
    return (proj(w + eps * h) - proj(w - eps * h)) / (2 * eps)


def _sym_svec(N, eigs, rng):
    Q, _ = np.linalg.qr(rng.standard_normal((N, N)))
    return Q @ np.diag(eigs) @ Q.T


@pytest.mark.parametrize("w", [
    [2.0, 0.3, -0.4, 0.5],        # inside: r <= t
    [-2.0, 0.3, -0.4, 0.5],       # polar: r <= -t
    [0.2, 0.9, -0.4, 0.5],        # the curved branch
    [0.3, -1.1],                  # dimension 2
    [-0.4, 0.7],
])
def test_soc_jacobian(w):
    w = np.array(w)
    cones = [O.SecondOrderCone(len(w))]
    rng = np.random.default_rng(0)
    for _ in range(3):
        h = rng.standard_normal(len(w))
        np.testing.assert_allclose(SA.dpi(w, cones, h), _fd_jacobian(cones, w, h), atol=1e-7)


@pytest.mark.parametrize("eigs", [[2.0, 1.0, -0.5, -1.5], [1.0, 1.0, -2.0, -2.0], [3.0, -1.0, -1.0, 0.5]])
@pytest.mark.parametrize("triangle", [True, False])
def test_psd_jacobian(eigs, triangle):
    rng = np.random.default_rng(1)
    N = len(eigs)
    W = _sym_svec(N, eigs, rng)
    if triangle:
        cones, w = [O.PsdConeTriangle(N * (N + 1) // 2)], SA._mat_to_tri(W)
    else:
        cones, w = [O.PsdCone(N * N)], W.reshape(-1, order="F")
    for _ in range(3):
        h = rng.standard_normal(len(w))
        J = SA.dpi(w, cones, h)
        np.testing.assert_allclose(J, _fd_jacobian(cones, w, h), atol=1e-6)
        g = rng.standard_normal(len(w))
        assert abs(g @ J - h @ SA.dpi(w, cones, g)) <= 1e-12 * (1 + abs(g @ J))   # symmetric


def _mixed_problem(seed):
    """Zero rows, Box rows (one bound active), a 4-dim SOC and a 3 x 3 PsdConeTriangle on 5 variables."""
    rng = np.random.default_rng(seed)
    n = 5
    G = rng.standard_normal((n, n))
    P = sp.csc_matrix(G @ G.T / n + 0.5 * np.eye(n))
    q = rng.standard_normal(n)
    cones = [O.ZeroSet(2), O.Box(np.array([-0.3, -1.0, -2.0]), np.array([0.2, 1.0, 2.0])), O.SecondOrderCone(4),
             O.PsdConeTriangle(6)]
    m = sum(c.dim for c in cones)
    A = sp.csc_matrix(rng.standard_normal((m, n)))
    s0 = np.concatenate([np.zeros(2), [0.0, 0.1, -0.5], [1.0, 0.2, 0.3, -0.1], SA._mat_to_tri(np.eye(3))])
    b = A @ (0.3 * rng.standard_normal(n)) + s0   # strictly feasible on the inequality rows
    return P, q, A, b, cones


def _oracle(P, q, A, b, cones, warm=None, **kw):
    st = O.Settings(eps_abs=1e-12, eps_rel=1e-12, max_iter=200000, kkt_solver="direct", scaling=0, **kw)
    r = O.solve(P, q, A, b, cones, st, *(warm or ()))
    assert r.status == "Solved", r.status
    return r


def _loss(r, g):
    return g[0] @ r.x + g[1] @ r.y + g[2] @ r.s


@pytest.mark.parametrize("seed", [0, 1])
def test_gradients_against_finite_differences(seed):
    P, q, A, b, cones = _mixed_problem(seed)
    m, n = A.shape
    r0 = _oracle(P, q, A, b, cones)
    rng = np.random.default_rng(10 + seed)
    g = (rng.standard_normal(n), rng.standard_normal(m), rng.standard_normal(m))
    got = SA.unscaled(P, A, cones, r0.x, r0.s, r0.y, gx=g[0], gy=g[1], gs=g[2])
    assert got["residual"] <= 1e-10
    warm = (r0.x, r0.s, r0.y)
    eps = 1e-6

    def fd(make):
        lp = _loss(_oracle(*make(eps), warm=warm), g)
        lm = _loss(_oracle(*make(-eps), warm=warm), g)
        return (lp - lm) / (2 * eps)

    for k in range(2):
        dq = rng.standard_normal(n)
        want = fd(lambda e: (P, q + e * dq, A, b, cones))
        assert abs(got["dq"] @ dq - want) <= 1e-5 * (1 + abs(want))
        db = rng.standard_normal(m)
        want = fd(lambda e: (P, q, A, b + e * db, cones))
        assert abs(got["db"] @ db - want) <= 1e-5 * (1 + abs(want))
        dA = rng.standard_normal(A.nnz)
        want = fd(lambda e: (P, q, sp.csc_matrix((A.data + e * dA, A.indices, A.indptr), shape=A.shape), b, cones))
        assert abs(got["dAx"] @ dA - want) <= 1e-5 * (1 + abs(want))
        S = rng.standard_normal((n, n))
        S = S + S.T
        dPx = S[P.indices, np.repeat(np.arange(n), np.diff(P.indptr))]
        want = fd(lambda e: (P + e * sp.csc_matrix(S), q, A, b, cones))
        assert abs(got["dPx"] @ dPx - want) <= 1e-5 * (1 + abs(want))
    # the Box bounds
    box = cones[1]
    for which in ("l", "u"):
        d = rng.standard_normal(box.dim)

        def make(e, which=which, d=d):
            l, u = box.l + (e * d if which == "l" else 0), box.u + (e * d if which == "u" else 0)
            return P, q, A, b, [cones[0], O.Box(l, u)] + cones[2:]
        want = fd(make)
        have = (got["dl"] if which == "l" else got["du"])[2:5] @ d
        assert abs(have - want) <= 1e-5 * (1 + abs(want))


def test_independent_of_rho_sigma_and_scaling():
    P, q, A, b, cones = _mixed_problem(0)
    m, n = A.shape
    r0 = _oracle(P, q, A, b, cones)
    rng = np.random.default_rng(3)
    g = dict(gx=rng.standard_normal(n), gy=rng.standard_normal(m), gs=rng.standard_normal(m))
    a = SA.unscaled(P, A, cones, r0.x, r0.s, r0.y, rho=0.1, sigma=1e-6, **g)
    rho = np.where(np.arange(m) < 2, 100.0, 0.01)   # equality rows at a larger rho, as the engine's rho vector
    b_ = SA.unscaled(P, A, cones, r0.x, r0.s, r0.y, rho=rho, sigma=1e-3, **g)
    for k in ("dq", "db", "dPx", "dAx", "dl", "du"):
        np.testing.assert_allclose(a[k], b_[k], atol=1e-8 * (1 + np.abs(a[k]).max()))
    # a Ruiz-like scaling: scaled data and point, the same unscaled gradients (cones scaled by one scalar)
    D = np.exp(rng.uniform(-0.5, 0.5, n))
    e = np.exp(rng.uniform(-0.5, 0.5))
    Ev = np.concatenate([np.exp(rng.uniform(-0.5, 0.5, 5)), np.full(m - 5, e)])
    c = 0.7
    Ps = sp.csc_matrix(c * sp.diags(D) @ P @ sp.diags(D))
    As = sp.csc_matrix(sp.diags(Ev) @ A @ sp.diags(D))
    box = cones[1]
    cs = [cones[0], O.Box(Ev[2:5] * box.l, Ev[2:5] * box.u)] + cones[2:]
    xs, ss, mus = r0.x / D, Ev * r0.s, -c * r0.y / Ev
    s_ = SA.adjoint(Ps, As, cs, xs, ss, mus, 0.1, D=D, E=Ev, c=c, **g)
    for k in ("dq", "db", "dPx", "dAx", "dl", "du"):
        np.testing.assert_allclose(a[k], s_[k], atol=1e-8 * (1 + np.abs(a[k]).max()))


def test_qp_agrees_with_polish_adjoint():
    """A strictly complementary QP: the fixed-point derivative equals the active-set one."""
    from tests import adjoint_reference as AR
    from tests import polish_reference as PR
    rng = np.random.default_rng(5)
    n = 4
    G = rng.standard_normal((n, n))
    P = sp.csc_matrix(G @ G.T + np.eye(n))
    q = rng.standard_normal(n)
    A = sp.csc_matrix(np.vstack([np.ones((1, n)), -np.eye(n)]))
    b = np.concatenate([[1.0], np.zeros(n)])          # sum x = 1, x >= 0
    cones = [O.ZeroSet(1), O.Nonnegatives(n)]
    r = _oracle(P, q, A, b, cones)
    assert np.all((r.s > 1e-6) | (-r.y > 1e-6) | (np.arange(n + 1) == 0))   # strictly complementary
    m = n + 1
    g = dict(gx=rng.standard_normal(n), gy=rng.standard_normal(m), gs=rng.standard_normal(m))
    mine = SA.unscaled(P, A, cones, r.x, r.s, r.y, **g)
    cls = np.array([PR.ZERO] + [PR.NONNEG] * n)
    kind = np.array([PR.EQUALITY] + [PR.LOWER if s < 1e-8 else PR.INACTIVE for s in r.s[1:]])
    theirs = AR.adjoint(P, A, cls, kind, r.x, r.y, refine_iter=10, **g)
    for k in ("dq", "db", "dPx", "dAx"):
        np.testing.assert_allclose(mine[k], theirs[k], atol=1e-7 * (1 + np.abs(theirs[k]).max()))


def test_binding():
    import cosmo_b200
    E = cosmo_b200.engine
    S = E.SolveAdjointSettings
    assert C.sizeof(S) == 32
    assert [(f, S.__dict__[f].offset) for f, _ in S._fields_] == [("tol", 0), ("max_iter", 8), ("restart", 12),
                                                                    ("kkt_tol", 16), ("reserved", 24)]
    restype, argtypes = E._signatures()["cosmo_b200_solve_adjoint"]
    assert restype == C.c_int and len(argtypes) == 12 and argtypes[1] == C.POINTER(S)
    assert E.SOLVE_ADJOINT_STATS[0] == "status" and len(E.SOLVE_ADJOINT_STATS) == 8
    with open(__file__.replace("tests/test_solve_adjoint_cpu.py", "include/cosmo_b200.h")) as f:
        assert "int cosmo_b200_solve_adjoint(cosmo_b200_handle* h, const cosmo_b200_solve_adjoint_settings* as" in f.read()
