"""GPU tests of the forward derivative of conic solutions through the fixed point of the iteration
(cosmo_b200_solve_derivative, Engine.solve_derivative, Model.solve_derivative, the forward mode of autograd.solve_conic):
the engine against the restatement of tests/solve_derivative_reference.py at the engine's own solution, the pairing
<g, J d> = <J' g, d> with Engine.solve_adjoint, finite differences through engine re-solves, fp32, host and device
buffers, determinism and the untouched next solve, statuses and refusals, Model.solve_derivative and
torch.autograd.gradcheck(check_forward_ad=True)."""
import numpy as np
import pytest
import scipy.sparse as sp

import cosmo_b200
from cosmo_b200 import engine as E
from oracle.bridge import to_oracle_cones
from tests import solve_derivative_reference as SD
from tests.test_gpu_solve_adjoint import CASES, TIGHT, _bits, _engine, _grads, _problem, _rel

pytestmark = pytest.mark.gpu

OUT = ("dx", "dy", "ds")
DIR = ("dPx", "dq", "dAx", "db", "dl", "du")
LARGE = dict(tol=1e-9, restart=100, max_iter=3000)   # the N = 150 cone, as the adjoint's tests solve it


def _direction(eng, P, seed=11):
    """A random direction of every input, symmetric in P (both stored triangles move together)."""
    rng = np.random.default_rng(seed)
    n, m = eng.n, eng.m
    S = rng.standard_normal((n, n))
    S = S + S.T
    dPx = S[P.indices, np.repeat(np.arange(n), np.diff(P.indptr))]
    return dict(dPx=dPx, dq=rng.standard_normal(n), dAx=rng.standard_normal(eng.nnzA), db=rng.standard_normal(m),
                dl=rng.standard_normal(m), du=rng.standard_normal(m))


def _reference(eng, P, A, sets, d):
    x, y, s = eng.solution(x=np.empty(eng.n), y=np.empty(eng.m), s=np.empty(eng.m))
    return SD.unscaled(P, A, to_oracle_cones(sets), x, s, y, **d)


def _close(a, want, bar):
    return _rel(a, want) <= bar or np.linalg.norm(want) == 0 and np.abs(a).max() <= 1e-9


# ---------------------------------------------------------------------------
# 1. the engine against the restatement; 2. the pairing with solve_adjoint
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("scaling", [0, 10])
@pytest.mark.parametrize("kkt", ["DeviceLdlKKTSolver", "DeviceSupernodalKKTSolver", "CGIndirectKKTSolver"])
def test_engine_matches_the_restatement(kkt, scaling, case):
    P, q, A, b, sets = _problem(3, **CASES[case])
    eng = _engine(P, q, A, b, sets, kkt, scaling)
    assert eng.solve().status == "Solved"
    d = _direction(eng, P)
    kw = LARGE if case == "large_psd" else {}
    got, st = eng.solve_derivative(**d, **kw)
    assert st["status"] == 1 and st["residual"] <= kw.get("tol", 1e-10), st
    assert (st["inner_iterations"] > 0) == (kkt == "CGIndirectKKTSolver")
    want = _reference(eng, P, A, sets, d)
    for k, a in zip(OUT, got):
        assert _close(a, want[k], 1e-6), (k, _rel(a, want[k]))
    eng.close()


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("scaling", [0, 10])
@pytest.mark.parametrize("kkt", ["DeviceLdlKKTSolver", "DeviceSupernodalKKTSolver", "CGIndirectKKTSolver"])
def test_pairing_with_solve_adjoint(kkt, scaling, case):
    P, q, A, b, sets = _problem(3, **CASES[case])
    eng = _engine(P, q, A, b, sets, kkt, scaling)
    assert eng.solve().status == "Solved"
    kw = LARGE if case == "large_psd" else {}
    for seed in (1, 2):
        g = _grads(eng.n, eng.m, seed=seed)
        d = _direction(eng, P, seed=20 + seed)
        jd, st = eng.solve_derivative(**d, **kw)
        jtg, ast = eng.solve_adjoint(*g, **kw)
        assert st["status"] == 1 and ast["status"] == 1, (st, ast)
        lhs = sum(gk @ v for gk, v in zip(g, jd))
        # the adjoint returns (dq, db, dPx, dAx, dl, du)
        rhs = sum(a @ d[k] for a, k in zip(jtg, ("dq", "db", "dPx", "dAx", "dl", "du")))
        scale = np.linalg.norm(np.concatenate(g)) * np.linalg.norm(np.concatenate(jd)) + \
            np.linalg.norm(np.concatenate(jtg)) * np.linalg.norm(np.concatenate([d[k] for k in DIR]))
        assert abs(lhs - rhs) <= 1e-8 * scale, (lhs, rhs, scale)
    eng.close()


# ---------------------------------------------------------------------------
# 3. finite differences through engine re-solves; 4. fp32
# ---------------------------------------------------------------------------
def test_finite_differences_through_engine_solves():
    P, q, A, b, sets = _problem(5)
    eng = _engine(P, q, A, b, sets)
    assert eng.solve().status == "Solved"

    def sol(Px, q_, Ax, b_, sets_=sets):
        e = _engine(sp.csc_matrix((Px, P.indices, P.indptr), shape=P.shape), q_,
                    sp.csc_matrix((Ax, A.indices, A.indptr), shape=A.shape), b_, sets_)
        assert e.solve().status == "Solved"
        out = e.solution(x=np.empty(e.n), y=np.empty(e.m), s=np.empty(e.m))
        e.close()
        return np.concatenate(out)

    d = _direction(eng, P, seed=7)
    h = 1e-5

    def check(fd, **dd):
        got, st = eng.solve_derivative(**dd)
        assert st["status"] == 1
        have = np.concatenate(got)
        assert np.abs(have - fd).max() <= 1e-5 * max(1.0, np.abs(fd).max()), (list(dd), np.abs(have - fd).max())

    base = dict(Px=P.data, q_=q, Ax=A.data, b_=b)
    for key, arg in (("dq", "q_"), ("db", "b_"), ("dAx", "Ax"), ("dPx", "Px")):
        plus, minus = dict(base), dict(base)
        plus[arg], minus[arg] = base[arg] + h * d[key], base[arg] - h * d[key]
        check((sol(**plus) - sol(**minus)) / (2 * h), **{key: d[key]})
    box = sets[1]
    for lo in (True, False):
        dv = d["dl" if lo else "du"][2:5]
        mk = lambda e: [sets[0], cosmo_b200.Box(box.l + (e * dv if lo else 0), box.u + (0 if lo else e * dv))] + sets[2:]
        fd = (sol(**base, sets_=mk(h)) - sol(**base, sets_=mk(-h))) / (2 * h)
        full = np.zeros(eng.m)
        full[2:5] = dv
        check(fd, **{"dl" if lo else "du": full})
    eng.close()


def test_fp32_matches_the_restatement():
    P, q, A, b, sets = _problem(4)
    eng = _engine(P, q, A, b, sets, dtype=np.float32, eps_abs=1e-6, eps_rel=1e-6)
    assert eng.solve().status == "Solved"
    d = _direction(eng, P)
    got, st = eng.solve_derivative(**d)
    assert st["status"] == 1, st
    want = _reference(eng, P, A, sets, d)
    for k, a in zip(OUT, got):
        assert _rel(a, want[k]) <= 1e-3, (k, _rel(a, want[k]))
    eng.close()


# ---------------------------------------------------------------------------
# 5. host and device buffers, determinism, the next solve, solve_adjoint untouched
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("kkt", ["DeviceLdlKKTSolver", "CGIndirectKKTSolver"])
def test_buffers_determinism_and_next_solve(kkt):
    torch = pytest.importorskip("torch")
    P, q, A, b, sets = _problem(8)
    eng, twin = _engine(P, q, A, b, sets, kkt, 10), _engine(P, q, A, b, sets, kkt, 10)
    for e in (eng, twin):
        assert e.solve().status == "Solved"
    g = _grads(eng.n, eng.m)
    d = _direction(eng, P)
    adj0, ast0 = eng.solve_adjoint(*g)
    host1, st1 = eng.solve_derivative(**d)
    host2, st2 = eng.solve_derivative(**d)
    dd = {k: torch.tensor(v, device="cuda") for k, v in d.items()}
    outs = [torch.empty(k, dtype=torch.float64, device="cuda") for k in (eng.n, eng.m, eng.m)]
    _, st3 = eng.solve_derivative(**dd, dx=outs[0], dy=outs[1], ds=outs[2])
    torch.cuda.synchronize()
    assert st1 == st2 == st3
    for a, c, o in zip(host1, host2, outs):
        assert np.array_equal(_bits(a), _bits(c)) and np.array_equal(_bits(a), _bits(o))
    adj1, ast1 = eng.solve_adjoint(*g)                 # the adjoint with a derivative in between
    assert ast0 == ast1
    for a, c in zip(adj0, adj1):
        assert np.array_equal(_bits(a), _bits(c))
    # the next solve, from changed q, is the twin's bit for bit
    q2 = q + 0.01
    res = []
    for e in (eng, twin):
        e.update_qb(q=q2)
        res.append(e.solve())
    a, c = res
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
        eng.solve_derivative()
    assert e.value.code == E.ERR_INVALID            # no solve yet
    assert eng.solve().status == "Solved"
    for bad in (dict(restart=0), dict(restart=201), dict(max_iter=0), dict(kkt_tol=0.0), dict(tol=-1.0)):
        with pytest.raises(E.EngineError) as e:
            eng.solve_derivative(**bad)
        assert e.value.code == E.ERR_INVALID, bad
    out, st = eng.solve_derivative(**_direction(eng, P), max_iter=1)
    assert st["status"] == 0 and all(np.isnan(a).all() for a in out)
    out, st = eng.solve_derivative()                   # the zero direction
    assert st["status"] == 1 and all((a == 0).all() for a in out)
    eng.close()
    # an Exp cone: not applicable
    P = sp.csc_matrix(np.eye(3))
    A = sp.csc_matrix(-np.eye(3))
    eng = _engine(P, np.array([1.0, 1.0, 1.0]), A, np.zeros(3), [cosmo_b200.ExponentialCone()], eps_abs=1e-6,
                  eps_rel=1e-6)
    eng.solve()
    out, st = eng.solve_derivative(dq=np.ones(3))
    assert st["status"] == -1 and all(np.isnan(a).all() for a in out)
    eng.close()
    # an infeasible solve: not applicable
    A = sp.csc_matrix(np.array([[1.0], [-1.0]]))
    eng = _engine(sp.csc_matrix((1, 1)), np.zeros(1), A, np.array([-1.0, -1.0]), [cosmo_b200.Nonnegatives(2)],
                  eps_abs=1e-5, eps_rel=1e-5)
    assert eng.solve().status == "Primal_infeasible"
    out, st = eng.solve_derivative(dq=np.ones(1))
    assert st["status"] == -1 and all(np.isnan(a).all() for a in out)
    eng.close()
    # a decomposed model (a banded max-cut SDP whose PSD cone splits into cliques)
    from tests.test_gpu_chordal_reverse import _c5_model
    model = _c5_model(200, dict(decompose=True, max_iter=50))
    model.optimize()
    assert model._dec is not None
    with pytest.raises(ValueError):
        model.solve_derivative(dq=np.ones(model.engine.n))


# ---------------------------------------------------------------------------
# 7. Model.solve_derivative; 8. forward-mode autograd
# ---------------------------------------------------------------------------
def test_model_solve_derivative():
    P, q, A, b, sets = _problem(10)
    model = cosmo_b200.Model(device=0)
    model.set(P, q, A, b, sets, cosmo_b200.Settings(kkt_solver="DeviceLdlKKTSolver", **TIGHT))
    with pytest.raises(ValueError):
        model.solve_derivative()
    res = model.optimize()
    assert res.status == "Solved"
    rng = np.random.default_rng(12)
    n, m = A.shape[1], A.shape[0]
    S = rng.standard_normal((n, n))
    dP = sp.csc_matrix(((S + S.T)[P.indices, np.repeat(np.arange(n), np.diff(P.indptr))], P.indices, P.indptr),
                       shape=P.shape)
    dA = sp.csc_matrix((rng.standard_normal(A.nnz), A.indices, A.indptr), shape=A.shape)
    dq, db = rng.standard_normal(n), rng.standard_normal(m)
    d = model.solve_derivative(dP=dP, dq=dq, dA=dA, db=db)
    assert d["stats"]["status"] == 1
    want = SD.unscaled(P, A, to_oracle_cones(sets), res.x, res.s, res.y, dPx=dP.data, dq=dq, dAx=dA.data, db=db)
    for k in ("x", "y", "s"):
        assert _rel(d[k], want["d" + k]) <= 1e-6, (k, _rel(d[k], want["d" + k]))


def _soc_problem():
    """The SOC problem of the adjoint's gradcheck: the cone on its boundary at the solution, P diagonal."""
    P = sp.csc_matrix(np.diag([1.0, 2.0, 1.5]))
    q = np.array([0.5, -3.0, 2.0])
    A = sp.csc_matrix(np.vstack([-np.eye(3), [[1.0, 0.0, 0.0]]]))
    b = np.array([1.0, 0.0, 0.0, 2.0])
    sets = [cosmo_b200.SecondOrderCone(3), cosmo_b200.Nonnegatives(1)]
    return P, q, A, b, sets


def test_gradcheck_forward_mode_of_solve_conic():
    torch = pytest.importorskip("torch")
    from cosmo_b200.autograd import solve_conic
    P, q, A, b, sets = _soc_problem()
    eng = _engine(P, q, A, b, sets, scaling=0, eps_abs=1e-12, eps_rel=1e-12)
    t = lambda a: torch.tensor(a, dtype=torch.float64, device="cuda", requires_grad=True)
    inputs = (t(P.data), t(q), t(A.data), t(b))
    assert torch.autograd.gradcheck(lambda Px, q_, Ax, b_: solve_conic(eng, Px, q_, Ax, b_), inputs, eps=1e-6,
                                    atol=1e-5, rtol=1e-4, check_forward_ad=True, check_backward_ad=False)
    # a forward_ad dual tensor: the tangent is Engine.solve_derivative's output bit for bit
    import torch.autograd.forward_ad as fwAD
    rng = np.random.default_rng(3)
    tang = [torch.tensor(rng.standard_normal(a.numel()), dtype=torch.float64, device="cuda") for a in inputs]
    with fwAD.dual_level():
        duals = [fwAD.make_dual(a.detach(), tt) for a, tt in zip(inputs, tang)]
        outs = solve_conic(eng, *duals)
        tangents = [fwAD.unpack_dual(o).tangent.clone() for o in outs]
    torch.cuda.synchronize()
    (dx, dy, ds), st = eng.solve_derivative(tang[0].cpu().numpy(), tang[1].cpu().numpy(), tang[2].cpu().numpy(),
                                            tang[3].cpu().numpy())
    assert st["status"] == 1
    for a, c in zip(tangents, (dx, dy, ds)):
        assert np.array_equal(_bits(a), _bits(c))
    eng.close()
