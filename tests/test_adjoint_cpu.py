"""Derivatives of polished solutions without a GPU: the restatement of tests/adjoint_reference.py against central finite
differences of the polished solution map (oracle ADMM solve + the polish restatement), its linear solve against a
dense solve of K_A, the binding of cosmo_b200_adjoint and Model.adjoint's refusal before any polish."""
import numpy as np
import pytest
import scipy.sparse as sp

import cosmo_b200
from cosmo_b200 import engine as E
from oracle import cosmo_oracle as O
from tests import adjoint_reference as AR
from tests import golden_problems as G
from tests import polish_reference as R


def _cones_with_bounds(cones, l, u):
    """The cone list with the Box bounds taken from the m-vectors l, u."""
    out, off = [], 0
    for c in cones:
        if isinstance(c, O.Box):
            out.append(O.Box(l[off:off + c.dim].copy(), u[off:off + c.dim].copy()))
        else:
            out.append(c)
        off += c.dim
    return out


def _polished(P, q, A, b, cones):
    res = O.solve(P, q, A, b, cones, O.Settings(eps_abs=1e-8, eps_rel=1e-8, max_iter=20000))
    assert res.status == "Solved"
    cls, l, u = R.row_classes(cones)
    out = R.polish(P, q, A, b, cls, l, u, res.x, res.s, -res.y)
    assert out["status"] == 1
    return out


def _random_qp(seed):
    """A QP with ZeroSet, Nonnegatives and Box rows (one Box row with l = u) in set! form, through a feasible x0."""
    rng = np.random.default_rng(seed)
    n, mz, mn, mb = 8, 2, 6, 5
    B = rng.standard_normal((n, n)) * (rng.random((n, n)) < 0.4)
    P = sp.csc_matrix(B @ B.T + 0.5 * np.eye(n))
    x0 = rng.standard_normal(n)
    Az, An, Ab = (rng.standard_normal((k, n)) for k in (mz, mn, mb))
    bz = Az @ x0
    bn = An @ x0 + rng.uniform(0.0, 0.5, mn)
    bb = rng.standard_normal(mb)
    w = bb - Ab @ x0                                 # the slack of x0 in the Box rows
    l, u = w - rng.uniform(0.05, 0.5, mb), w + rng.uniform(0.05, 0.5, mb)
    l[0] = u[0] = w[0]
    A = sp.csc_matrix(np.vstack([Az, An, Ab]))
    b = np.concatenate([bz, bn, bb])
    q = 3.0 * rng.standard_normal(n)
    return P, q, A, b, [O.ZeroSet(mz), O.Nonnegatives(mn), O.Box(l, u)]


def _golden(builder):
    P, q, cons = builder()
    Pm, qm, A, b, cones = O.assemble(P, q, cons)
    return sp.csc_matrix(Pm), qm, sp.csc_matrix(A), b, cones


def _g2_strict():
    """G2 with q = (1, -1.5): as written (q = (1, -1)) its solution x = (0, 1) sits at u in the second row with a zero
    multiplier, a weakly active row where the map has only one-sided derivatives."""
    P, q, A, b, cones = _golden(G.g2_box_feasible)
    return P, np.array([1.0, -1.5]), A, b, cones


PROBLEMS = [("G1", lambda: _golden(G.g1_qp_box)), ("G2", _g2_strict),
            ("G12", lambda: _golden(G.g12_lp))] + [("qp%d" % s, lambda s=s: _random_qp(s)) for s in (0, 1, 2)]


def _loss(out, gx, gy, gs):
    return gx @ out["x"] + gy @ out["y"] + gs @ out["s"]


@pytest.mark.parametrize("name,make", PROBLEMS, ids=[p[0] for p in PROBLEMS])
def test_gradients_match_central_differences_of_the_polished_solution_map(name, make):
    P, q, A, b, cones = make()
    m, n = A.shape
    cls, l, u = R.row_classes(cones)
    base = _polished(P, q, A, b, cones)
    kind = base["kind"]
    # strict complementarity: the active set, and with it the map, is locally constant
    ineq = (kind == R.LOWER) | (kind == R.UPPER)
    assert np.all(np.abs(base["mu_p"][ineq]) > 1e-7)
    rng = np.random.default_rng(len(name) + n + m)
    gx, gy, gs = rng.standard_normal(n), rng.standard_normal(m), rng.standard_normal(m)
    g = AR.adjoint(P, A, cls, kind, base["x_p"], -base["mu_p"], gx, gy, gs)
    assert g["refine_residual"] <= 1e-12
    # random directions of q, b, P (symmetric, on its pattern), A (on its pattern) and the Box bounds
    pr, pc = P.indices, np.repeat(np.arange(n), np.diff(P.indptr))
    M = sp.csc_matrix((rng.standard_normal(P.nnz), P.indices, P.indptr), shape=P.shape)
    eP_sym = np.asarray((M + M.T)[pr, pc]).ravel() if P.nnz else np.zeros(0)
    dA = sp.csc_matrix(A, copy=True)
    dA.data = rng.standard_normal(A.nnz)
    box = cls == R.BOX
    dl = np.where(box & np.isfinite(l), rng.standard_normal(m), 0.0)
    du = np.where(box & np.isfinite(u), rng.standard_normal(m), 0.0)
    du = np.where(box & (l == u), dl, du)          # an equality row moves as one
    dirs = {"q": (np.zeros_like(P.data), rng.standard_normal(n), np.zeros(A.nnz), np.zeros(m), 0 * dl, 0 * du),
            "b": (np.zeros_like(P.data), np.zeros(n), np.zeros(A.nnz), rng.standard_normal(m), 0 * dl, 0 * du),
            "P": (eP_sym, np.zeros(n), np.zeros(A.nnz), np.zeros(m), 0 * dl, 0 * du),
            "A": (np.zeros_like(P.data), np.zeros(n), dA.data, np.zeros(m), 0 * dl, 0 * du),
            "bounds": (np.zeros_like(P.data), np.zeros(n), np.zeros(A.nnz), np.zeros(m), dl, du)}
    for what, (eP, eq, eA, eb, el, eu) in dirs.items():
        if not (np.any(eP) or np.any(eq) or np.any(eA) or np.any(eb) or np.any(el) or np.any(eu)):
            continue
        ana = g["dPx"] @ eP + g["dq"] @ eq + g["dAx"] @ eA + g["db"] @ eb + g["dl"] @ el + g["du"] @ eu
        eps = 1e-6
        vals = []
        for sgn in (1.0, -1.0):
            P2 = sp.csc_matrix((P.data + sgn * eps * eP, P.indices, P.indptr), shape=P.shape)
            A2 = sp.csc_matrix((A.data + sgn * eps * eA, A.indices, A.indptr), shape=A.shape)
            c2 = _cones_with_bounds(cones, l + sgn * eps * el, u + sgn * eps * eu)
            out = _polished(P2, q + sgn * eps * eq, A2, b + sgn * eps * eb, c2)
            assert np.array_equal(out["kind"], kind), what
            vals.append(_loss(out, gx, gy, gs))
        fd = (vals[0] - vals[1]) / (2 * eps)
        assert abs(fd - ana) <= 1e-6 * max(abs(ana), 1e-3), (what, fd, ana)


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_the_refined_solve_reaches_the_dense_solution_of_k_a(seed):
    rng = np.random.default_rng(seed)
    n, m = 30, 40
    B = sp.random(n, n, density=0.1, random_state=rng)
    P = sp.csc_matrix(B @ B.T + 0.1 * sp.identity(n))
    A = sp.csc_matrix(sp.random(m, n, density=0.15, random_state=rng) + sp.eye(m, n))
    kind = rng.choice([R.INACTIVE, R.LOWER, R.UPPER, R.EQUALITY], size=m, p=[0.6, 0.15, 0.1, 0.15]).astype(np.int8)
    act = np.flatnonzero(kind != R.INACTIVE)
    rx, rs = rng.standard_normal(n), rng.standard_normal(m)
    z = np.linalg.solve(AR.kkt_matrix(P, A, kind), np.concatenate([rx, rs[act]]))
    u, v, r = AR.solve(P, A, kind, rx, rs)
    assert np.linalg.norm(u - z[:n]) <= 1e-12 * np.linalg.norm(z)
    assert np.linalg.norm(v[act] - z[n:]) <= 1e-12 * np.linalg.norm(z)
    assert np.all(v[kind == R.INACTIVE] == 0.0) and r <= 1e-12 * np.abs(z).max()


def test_scaling_does_not_change_the_gradients():
    # the unscaled solution map does not depend on the scaling: the scaled path maps back to the same numbers
    P, q, A, b, cones = _random_qp(0)
    m, n = A.shape
    cls, l, u = R.row_classes(cones)
    base = _polished(P, q, A, b, cones)
    rng = np.random.default_rng(7)
    gx, gy, gs = rng.standard_normal(n), rng.standard_normal(m), rng.standard_normal(m)
    ref = AR.adjoint(P, A, cls, base["kind"], base["x_p"], -base["mu_p"], gx, gy, gs)
    D, Ev, c = rng.uniform(0.5, 2.0, n), rng.uniform(0.5, 2.0, m), 0.7
    Ps = c * sp.diags(D) @ P @ sp.diags(D)
    As = sp.diags(Ev) @ A @ sp.diags(D)
    got = AR.adjoint(sp.csc_matrix(Ps), sp.csc_matrix(As), cls, base["kind"], base["x_p"] / D, -c * base["mu_p"] / Ev,
                     gx, gy, gs, D=D, E=Ev, c=c)
    for k in ("dq", "db", "dPx", "dAx", "dl", "du"):
        assert np.allclose(got[k], ref[k], rtol=1e-10, atol=1e-12), k


def test_the_binding_names_the_entry_point():
    assert "cosmo_b200_adjoint" in E.SIGNATURES and "cosmo_b200_adjoint" in E.EXPORTS
    restype, argtypes = E.SIGNATURES["cosmo_b200_adjoint"]
    assert len(argtypes) == 12 and argtypes[1] is E.C.c_int32
    assert E.ADJOINT_STATS == ("status", "n_active", "n_weak", "refine_residual")


def test_model_adjoint_needs_a_polished_optimize():
    model = cosmo_b200.Model()
    P, q, cons = G.g2_box_feasible()
    model.set(sp.csc_matrix(P), q, sp.csc_matrix(-np.eye(2)), np.zeros(2), [cosmo_b200.Box([0.0, 0.0], [1.0, 1.0])])
    with pytest.raises(ValueError):
        model.adjoint(dx=np.ones(2))
