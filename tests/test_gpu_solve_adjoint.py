"""GPU tests of the derivatives of conic solutions through the fixed point of the iteration (cosmo_b200_solve_adjoint,
Engine.solve_adjoint, Model.solve_adjoint, autograd.solve_conic): the engine against the restatement of
tests/solve_adjoint_reference.py at the engine's own solution, finite differences through full engine re-solves,
independence of rho and alpha, agreement with the polish adjoint on a QP, host and device buffers, determinism and the
untouched next solve, statuses and refusals, and torch.autograd.gradcheck."""
import numpy as np
import pytest
import scipy.sparse as sp

import cosmo_b200
from cosmo_b200 import engine as E
from cosmo_b200 import model as M
from oracle.bridge import to_oracle_cones
from tests import solve_adjoint_reference as SA

pytestmark = pytest.mark.gpu

KEYS = ("dq", "db", "dPx", "dAx", "dl", "du")
TIGHT = dict(eps_abs=1e-11, eps_rel=1e-11, max_iter=200000)


def _engine(P, q, A, b, sets, kkt="DeviceLdlKKTSolver", scaling=0, dtype=np.float64, **kw):
    if kkt == "CGIndirectKKTSolver":
        kw.setdefault("tol_constant", 1e-9)   # inner solves accurate enough for the outer 1e-11
    st = cosmo_b200.Settings(kkt_solver=kkt, scaling=scaling, **{**TIGHT, **kw}).to_struct()
    return E.Engine(P, q, A, b, [M.set_tuple(S) for S in sets], st, dtype=dtype, equilibrate=scaling != 0)


def _problem(seed, n=12, n_soc=2, psd=(3, 3), square=False, big_psd=0):
    """ZeroSet, Box (one row clamped), SOC cones and PSD cones (PsdConeTriangle, or PsdCone with square) through a
    strictly feasible point; P positive definite so that the solution is unique."""
    rng = np.random.default_rng(seed)
    G = rng.standard_normal((n, n))
    P = sp.csc_matrix(np.triu(G @ G.T / n + 0.5 * np.eye(n)) + np.tril(G @ G.T / n + 0.5 * np.eye(n), -1))
    q = rng.standard_normal(n)
    sets, s0 = [cosmo_b200.ZeroSet(2)], [np.zeros(2)]
    sets.append(cosmo_b200.Box(np.array([-0.3, -1.0, -2.0]), np.array([0.2, 1.0, 2.0])))
    s0.append(np.array([0.0, 0.1, -0.5]))
    for _ in range(n_soc):
        sets.append(cosmo_b200.SecondOrderCone(4))
        s0.append(np.array([1.0, 0.2, 0.3, -0.1]))
    for N in list(psd) + ([big_psd] if big_psd else []):
        if square:
            sets.append(cosmo_b200.PsdCone(N * N))
            s0.append(np.eye(N).reshape(-1))
        else:
            sets.append(cosmo_b200.PsdConeTriangle(N * (N + 1) // 2))
            s0.append(SA._mat_to_tri(np.eye(N)))
    s0 = np.concatenate(s0)
    m = s0.size
    A = sp.csc_matrix(sp.random(m, n, density=0.5, random_state=seed) + sp.csc_matrix(
        (np.ones(min(m, n)), (np.arange(min(m, n)), np.arange(min(m, n)))), shape=(m, n)))
    b = A @ (0.3 * rng.standard_normal(n)) + s0
    return P, q, A, b, sets


def _grads(n, m, seed=5):
    rng = np.random.default_rng(seed)
    return rng.standard_normal(n), rng.standard_normal(m), rng.standard_normal(m)


def _reference(eng, P, A, sets, g):
    """The restatement at the engine's unscaled solution (rho is free at the fixed point)."""
    x, y, s = eng.solution(x=np.empty(eng.n), y=np.empty(eng.m), s=np.empty(eng.m))
    return SA.unscaled(P, A, to_oracle_cones(sets), x, s, y, gx=g[0], gy=g[1], gs=g[2])


def _rel(a, b):
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


def _bits(a):
    a = a.cpu().numpy() if hasattr(a, "cpu") else a
    return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


# ---------------------------------------------------------------------------
# 1. the engine against the restatement
# ---------------------------------------------------------------------------
CASES = {
    "soc_psd": dict(),
    "psd_batch": dict(n_soc=1, psd=(2, 3, 4, 5, 3, 2)),
    "square": dict(square=True, psd=(3,)),
    "large_psd": dict(n=30, n_soc=1, psd=(), big_psd=150),
}


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("scaling", [0, 10])
@pytest.mark.parametrize("kkt", ["DeviceLdlKKTSolver", "DeviceSupernodalKKTSolver", "CGIndirectKKTSolver"])
def test_engine_matches_the_restatement(kkt, scaling, case):
    P, q, A, b, sets = _problem(3, **CASES[case])
    eng = _engine(P, q, A, b, sets, kkt, scaling)
    assert eng.solve().status == "Solved"
    g = _grads(eng.n, eng.m)
    # the N = 150 cone makes (I - M') harder for GMRES(30): a longer Krylov space and a looser residual
    kw = dict(tol=1e-9, restart=100, max_iter=3000) if case == "large_psd" else {}
    got, st = eng.solve_adjoint(*g, **kw)
    assert st["status"] == 1 and st["residual"] <= kw.get("tol", 1e-10), st
    assert (st["inner_iterations"] > 0) == (kkt == "CGIndirectKKTSolver")
    want = _reference(eng, P, A, sets, g)
    for k, a in zip(KEYS, got):
        assert _rel(a, want[k]) <= 1e-6 or np.linalg.norm(want[k]) == 0 and np.abs(a).max() <= 1e-9, (k, _rel(a, want[k]))
    eng.close()


def test_fp32_matches_the_restatement():
    P, q, A, b, sets = _problem(4)
    eng = _engine(P, q, A, b, sets, dtype=np.float32, eps_abs=1e-6, eps_rel=1e-6)
    assert eng.solve().status == "Solved"
    g = _grads(eng.n, eng.m)
    got, st = eng.solve_adjoint(*g)
    assert st["status"] == 1, st
    want = _reference(eng, P, A, sets, g)
    for k, a in zip(KEYS[:4], got[:4]):
        assert _rel(a, want[k]) <= 1e-3, (k, _rel(a, want[k]))
    eng.close()


# ---------------------------------------------------------------------------
# 2. finite differences through full engine re-solves; 3. independence of rho and alpha
# ---------------------------------------------------------------------------
def test_finite_differences_through_engine_solves():
    P, q, A, b, sets = _problem(5)
    eng = _engine(P, q, A, b, sets)
    assert eng.solve().status == "Solved"
    g = _grads(eng.n, eng.m)
    (dq, db, dPx, dAx, dl, du), st = eng.solve_adjoint(*g)
    assert st["status"] == 1

    def loss(Px, q_, Ax, b_, sets_=sets):
        e = _engine(sp.csc_matrix((Px, P.indices, P.indptr), shape=P.shape), q_,
                    sp.csc_matrix((Ax, A.indices, A.indptr), shape=A.shape), b_, sets_)
        assert e.solve().status == "Solved"
        x, y, s = e.solution(x=np.empty(e.n), y=np.empty(e.m), s=np.empty(e.m))
        e.close()
        return g[0] @ x + g[1] @ y + g[2] @ s

    rng = np.random.default_rng(7)
    h = 1e-5
    dirs = [(rng.standard_normal(eng.n), 0), (rng.standard_normal(eng.m), 1), (rng.standard_normal(A.nnz), 2)]
    for d, which in dirs:
        args = [P.data, q, A.data, b]
        k = {0: 1, 1: 3, 2: 2}[which]
        plus, minus = list(args), list(args)
        plus[k], minus[k] = args[k] + h * d, args[k] - h * d
        fd = (loss(*plus) - loss(*minus)) / (2 * h)
        have = {0: dq, 1: db, 2: dAx}[which] @ d
        assert abs(have - fd) <= 1e-5 * max(1.0, abs(fd)), (which, have, fd)
    # a symmetric direction of P (both stored triangles move together) and the Box bounds through new engines
    S = rng.standard_normal((eng.n, eng.n))
    S = S + S.T
    dP = S[P.indices, np.repeat(np.arange(eng.n), np.diff(P.indptr))]
    fd = (loss(P.data + h * dP, q, A.data, b) - loss(P.data - h * dP, q, A.data, b)) / (2 * h)
    assert abs(dPx @ dP - fd) <= 1e-5 * max(1.0, abs(fd))
    box = sets[1]
    d = rng.standard_normal(3)
    for lo in (True, False):
        mk = lambda e: [sets[0], cosmo_b200.Box(box.l + (e * d if lo else 0), box.u + (0 if lo else e * d))] + sets[2:]
        fd = (loss(P.data, q, A.data, b, mk(h)) - loss(P.data, q, A.data, b, mk(-h))) / (2 * h)
        have = (dl if lo else du)[2:5] @ d
        assert abs(have - fd) <= 1e-5 * max(1.0, abs(fd)), (lo, have, fd)
    eng.close()


def test_independent_of_rho_and_alpha():
    P, q, A, b, sets = _problem(6)
    g = _grads(A.shape[1], A.shape[0])
    res = []
    for rho, alpha in ((0.1, 1.6), (0.01, 1.9)):
        eng = _engine(P, q, A, b, sets, rho=rho, alpha=alpha)
        assert eng.solve().status == "Solved"
        res.append(eng.solve_adjoint(*g)[0])
        eng.close()
    for k, a, c in zip(KEYS, *res):
        assert np.linalg.norm(a - c) <= 1e-7 * max(1.0, np.linalg.norm(a)), k


# ---------------------------------------------------------------------------
# 4. QPs: the polish adjoint
# ---------------------------------------------------------------------------
def test_qp_agrees_with_the_polish_adjoint():
    from tests.test_gpu_adjoint import _problem as qp
    P, q, A, b, sets = qp(100, 3)
    eng = _engine(P, q, A, b, sets)
    assert eng.solve().status == "Solved"
    g = _grads(eng.n, eng.m)
    mine, st = eng.solve_adjoint(*g)
    assert st["status"] == 1
    _, _, _, pst = eng.polish(x=np.empty(eng.n), y=np.empty(eng.m), s=np.empty(eng.m))
    assert pst["status"] == 1
    theirs, ast = eng.adjoint(*g, refine_iter=10)
    assert ast["status"] == 1
    for k, a, c in zip(KEYS, mine, theirs):
        assert np.linalg.norm(a - c) <= 1e-6 * max(1.0, np.linalg.norm(c)), (k, _rel(a, c))
    eng.close()


# ---------------------------------------------------------------------------
# 5. host and device buffers, determinism, the next solve
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("kkt", ["DeviceLdlKKTSolver", "CGIndirectKKTSolver"])
def test_buffers_determinism_and_next_solve(kkt):
    torch = pytest.importorskip("torch")
    P, q, A, b, sets = _problem(8)
    eng, twin = _engine(P, q, A, b, sets, kkt, 10), _engine(P, q, A, b, sets, kkt, 10)
    for e in (eng, twin):
        assert e.solve().status == "Solved"
    g = _grads(eng.n, eng.m)
    host1, st1 = eng.solve_adjoint(*g)
    host2, st2 = eng.solve_adjoint(*g)
    gd = [torch.tensor(a, device="cuda") for a in g]
    outs = [torch.empty(k, dtype=torch.float64, device="cuda") for k in (eng.n, eng.m, eng.nnzP, eng.nnzA, eng.m, eng.m)]
    eng.solve_adjoint(*gd, dq=outs[0], db=outs[1], dPx=outs[2], dAx=outs[3], dl=outs[4], du=outs[5])
    torch.cuda.synchronize()
    assert st1 == st2
    for a, c, d in zip(host1, host2, outs):
        assert np.array_equal(_bits(a), _bits(c)) and np.array_equal(_bits(a), _bits(d))
    # the next solve, from changed q, is the twin's bit for bit
    q2 = q + 0.01
    outs = []
    for e in (eng, twin):
        e.update_qb(q=q2)
        outs.append(e.solve())
    a, c = outs
    assert np.array_equal(_bits(a.x), _bits(c.x)) and np.array_equal(_bits(a.s), _bits(c.s))
    assert np.array_equal(_bits(a.mu), _bits(c.mu))
    assert a.obj_val == c.obj_val and a.iter == c.iter and np.array_equal(a.rho_updates, c.rho_updates)
    assert a.kkt_inner_iterations == c.kkt_inner_iterations
    eng.close()
    twin.close()


# ---------------------------------------------------------------------------
# 6. statuses and refusals
# ---------------------------------------------------------------------------
def test_statuses_and_refusals():
    P, q, A, b, sets = _problem(9, n_soc=1, psd=())
    eng = _engine(P, q, A, b, sets)
    with pytest.raises(E.EngineError) as e:
        eng.solve_adjoint()
    assert e.value.code == E.ERR_INVALID            # no solve yet
    assert eng.solve().status == "Solved"
    for bad in (dict(restart=0), dict(restart=201), dict(max_iter=0), dict(kkt_tol=0.0), dict(tol=-1.0)):
        with pytest.raises(E.EngineError) as e:
            eng.solve_adjoint(**bad)
        assert e.value.code == E.ERR_INVALID, bad
    g = _grads(eng.n, eng.m)
    out, st = eng.solve_adjoint(*g, max_iter=1)
    assert st["status"] == 0 and all(np.isnan(a).all() for a in out)
    eng.close()
    # an Exp cone: not applicable
    P = sp.csc_matrix(np.eye(3))
    A = sp.csc_matrix(-np.eye(3))
    eng = _engine(P, np.array([1.0, 1.0, 1.0]), A, np.zeros(3), [cosmo_b200.ExponentialCone()], eps_abs=1e-6,
                  eps_rel=1e-6)
    eng.solve()
    out, st = eng.solve_adjoint(*_grads(3, 3))
    assert st["status"] == -1 and all(np.isnan(a).all() for a in out)
    eng.close()
    # an infeasible solve: not applicable
    A = sp.csc_matrix(np.array([[1.0], [-1.0]]))
    eng = _engine(sp.csc_matrix((1, 1)), np.zeros(1), A, np.array([-1.0, -1.0]), [cosmo_b200.Nonnegatives(2)],
                  eps_abs=1e-5, eps_rel=1e-5)
    assert eng.solve().status == "Primal_infeasible"
    out, st = eng.solve_adjoint(np.ones(1))
    assert st["status"] == -1
    eng.close()


# ---------------------------------------------------------------------------
# 7. Model.solve_adjoint and gradcheck
# ---------------------------------------------------------------------------
def test_model_solve_adjoint():
    P, q, A, b, sets = _problem(10)
    model = cosmo_b200.Model(device=0)
    model.set(P, q, A, b, sets, cosmo_b200.Settings(kkt_solver="DeviceLdlKKTSolver", **TIGHT))
    with pytest.raises(ValueError):
        model.solve_adjoint()
    res = model.optimize()
    assert res.status == "Solved"
    g = _grads(A.shape[1], A.shape[0])
    d = model.solve_adjoint(*g)
    want = SA.unscaled(P, A, to_oracle_cones(sets), res.x, res.s, res.y, gx=g[0], gy=g[1], gs=g[2])
    assert d["stats"]["status"] == 1
    assert _rel(d["q"], want["dq"]) <= 1e-6 and _rel(d["A"].data, want["dAx"]) <= 1e-6


def test_gradcheck_of_solve_conic():
    torch = pytest.importorskip("torch")
    from cosmo_b200.autograd import solve_conic
    # min 1/2 |x|^2 + q'x  s.t.  |x[1:]| <= x0 + 1 (one SOC), x0 <= 2: the SOC on its boundary at the solution
    P = sp.csc_matrix(np.diag([1.0, 2.0, 1.5]))
    q = np.array([0.5, -3.0, 2.0])
    A = sp.csc_matrix(np.vstack([-np.eye(3), [[1.0, 0.0, 0.0]]]))
    b = np.array([1.0, 0.0, 0.0, 2.0])
    sets = [cosmo_b200.SecondOrderCone(3), cosmo_b200.Nonnegatives(1)]
    eng = _engine(P, q, A, b, sets, scaling=0, eps_abs=1e-12, eps_rel=1e-12)
    t = lambda a: torch.tensor(a, dtype=torch.float64, device="cuda", requires_grad=True)
    inputs = (t(P.data), t(q), t(A.data), t(b))
    x, y, s = solve_conic(eng, *inputs)
    r = np.linalg.norm(s[1:3].detach().cpu().numpy())
    assert abs(r - float(s[0])) <= 1e-9 and r > 0.1        # on the boundary, off the tip
    assert torch.autograd.gradcheck(lambda Px, q_, Ax, b_: solve_conic(eng, Px, q_, Ax, b_), inputs, eps=1e-6,
                                    atol=1e-5, rtol=1e-4)
    eng.close()
