"""GPU tests of the derivatives through custom cones with the Jacobian hook (COSMO_B200_CUSTOM_HAS_JACOBIAN): the engine's
solve_adjoint and solve_derivative against the restatements of tests/solve_adjoint_reference.py and
tests/solve_derivative_reference.py at the engine's own solution, the same SOCP with SecondOrderCone and with the hooked
soc2_jac cones, the pairing of the two calls, finite differences through engine re-solves, fp32, the unchanged
status -1 of hookless types, determinism and the untouched next solve, the compile cache, and torch.autograd.gradcheck
of solve_conic in both modes.  The cones are those of tests/custom_cone_jacobians.py."""
import uuid

import numpy as np
import pytest
import scipy.sparse as sp

import cosmo_b200
from cosmo_b200 import model as M
from tests import custom_cone_jacobians as CJ
from tests import custom_cones as CC
from tests import solve_adjoint_reference as SA
from tests import solve_derivative_reference as SD
from tests.test_gpu_solve_adjoint import KEYS, _bits, _engine, _grads, _rel
from tests.test_gpu_solve_derivative import OUT, _close, _direction

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def restatement(monkeypatch):
    """the restatements' dpi with the Jacobians of the hooked cones"""
    CJ.install_restatement(monkeypatch)


def _problem(seed, cones, n=12, builtin=False):
    """ZeroSet, Box and the custom cones `cones` (name -> dims), plus a SecondOrderCone(4) and a 3 x 3 PsdConeTriangle
    with builtin, through a strictly feasible point; P positive definite"""
    rng = np.random.default_rng(seed)
    G = rng.standard_normal((n, n))
    P = sp.csc_matrix(np.triu(G @ G.T / n + 0.5 * np.eye(n)) + np.tril(G @ G.T / n + 0.5 * np.eye(n), -1))
    q = 3.0 * rng.standard_normal(n)
    sets = [cosmo_b200.ZeroSet(2), cosmo_b200.Box(np.array([-0.3, -1.0, -2.0]), np.array([0.2, 1.0, 2.0]))]
    s0 = [np.zeros(2), np.array([0.0, 0.1, -0.5])]
    if builtin:
        sets += [cosmo_b200.SecondOrderCone(4), cosmo_b200.PsdConeTriangle(6)]
        s0 += [np.array([1.0, 0.2, 0.3, -0.1]), SA._mat_to_tri(np.eye(3))]
    for name, dims in cones.items():
        for d in dims:
            if name == "nonpos":
                sets.append(M.CustomCone(CJ.nonpos_type(), d))
                s0.append(-0.5 * np.ones(d))
            elif name == "soc2":
                sets.append(M.CustomCone(CJ.soc2_type(), d))
                s0.append(np.concatenate([[1.0], 0.3 * rng.uniform(-1, 1, d - 1) / np.sqrt(d)]))
            else:
                sets.append(M.CustomCone(CJ.linf_type(), d, [2.0]))
                s0.append(np.concatenate([[2.0], 0.4 * rng.uniform(-1, 1, d - 1)]))
    s0 = np.concatenate(s0)
    m = s0.size
    A = sp.csc_matrix(sp.random(m, n, density=0.5, random_state=seed) + sp.csc_matrix(
        (np.ones(min(m, n)), (np.arange(min(m, n)), np.arange(min(m, n)))), shape=(m, n)))
    b = A @ (0.3 * rng.standard_normal(n)) + s0
    return P, q, A, b, sets


CASES = {
    "nonpos": dict(cones={"nonpos": (3, 1)}),
    "soc2": dict(cones={"soc2": (4, 5)}),
    "wlinf": dict(cones={"wlinf": (5, 300)}),
    "mixed": dict(cones={"nonpos": (2,), "soc2": (4,), "wlinf": (5,)}, builtin=True),
}
PLUGINS = ["DeviceLdlKKTSolver", "DeviceSupernodalKKTSolver", "CGIndirectKKTSolver"]


def _solution(eng):
    return eng.solution(x=np.empty(eng.n), y=np.empty(eng.m), s=np.empty(eng.m))


# ---------------------------------------------------------------------------
# 1. the engine against the restatements
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("scaling", [0, 10])
@pytest.mark.parametrize("kkt", PLUGINS)
def test_solve_adjoint_matches_the_restatement(kkt, scaling, case):
    P, q, A, b, sets = _problem(3, **CASES[case])
    eng = _engine(P, q, A, b, sets, kkt, scaling)
    assert eng.solve().status == "Solved"
    g = _grads(eng.n, eng.m)
    got, st = eng.solve_adjoint(*g)
    assert st["status"] == 1 and st["residual"] <= 1e-10, st
    x, y, s = _solution(eng)
    want = SA.unscaled(P, A, CJ.to_oracle(sets), x, s, y, gx=g[0], gy=g[1], gs=g[2])
    for k, a in zip(KEYS, got):
        assert _close(a, want[k], 1e-6), (k, _rel(a, want[k]))
    eng.close()


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("scaling", [0, 10])
@pytest.mark.parametrize("kkt", PLUGINS)
def test_solve_derivative_matches_the_restatement(kkt, scaling, case):
    P, q, A, b, sets = _problem(3, **CASES[case])
    eng = _engine(P, q, A, b, sets, kkt, scaling)
    assert eng.solve().status == "Solved"
    d = _direction(eng, P)
    got, st = eng.solve_derivative(**d)
    assert st["status"] == 1 and st["residual"] <= 1e-10, st
    x, y, s = _solution(eng)
    want = SD.unscaled(P, A, CJ.to_oracle(sets), x, s, y, **d)
    for k, a in zip(OUT, got):
        assert _close(a, want[k], 1e-6), (k, _rel(a, want[k]))
    eng.close()


def test_the_cases_reach_the_general_branches():
    """at the engine's solution of the wlinf and soc2 cases some cone is projected on its clipped / curved branch"""
    for case, name in (("wlinf", "wlinf_jac"), ("soc2", "soc2_jac")):
        P, q, A, b, sets = _problem(3, **CASES[case])
        eng = _engine(P, q, A, b, sets)
        assert eng.solve().status == "Solved"
        x, y, s = _solution(eng)
        ws, off, hit = s - y / 0.1, 5, False
        for S in sets[2:]:
            w = ws[off:off + S.dim]
            p = w.copy()
            CJ.NUMPY[name][0](p, S.params)
            hit = hit or (not np.allclose(p, w) and np.abs(p).max() > 1e-8)
            off += S.dim
        assert hit, case
        eng.close()


# ---------------------------------------------------------------------------
# 2. the built-in SOC and the hooked soc2 cone: one derivative
# ---------------------------------------------------------------------------
def _socp(kind):
    from tests.test_gpu_custom_cones import _socp as socp
    return socp(kind, seed=3)


@pytest.mark.parametrize("kkt", ["DeviceSupernodalKKTSolver", "CGIndirectKKTSolver"])
def test_builtin_and_hooked_soc_give_the_same_derivatives(kkt):
    res = []
    for kind in (None, CJ.soc2_type()):
        P, q, A, b, sets = _socp(kind)
        eng = _engine(P, q, A, b, sets, kkt, 10)
        assert eng.solve().status == "Solved"
        g = _grads(eng.n, eng.m)
        d = _direction(eng, P)
        adj, ast = eng.solve_adjoint(*g)
        der, dst = eng.solve_derivative(**d)
        assert ast["status"] == dst["status"] == 1, (ast, dst)
        res.append((adj, der))
        eng.close()
    (a0, d0), (a1, d1) = res
    for k, a, c in zip(KEYS, a0, a1):
        assert _close(c, a, 1e-6), (k, _rel(c, a))
    for k, a, c in zip(OUT, d0, d1):
        assert _close(c, a, 1e-6), (k, _rel(c, a))


# ---------------------------------------------------------------------------
# 3. the pairing; finite differences through engine re-solves; fp32
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("kkt", PLUGINS)
def test_pairing_of_the_two_calls(kkt):
    P, q, A, b, sets = _problem(3, **CASES["mixed"])
    eng = _engine(P, q, A, b, sets, kkt, 10)
    assert eng.solve().status == "Solved"
    g = _grads(eng.n, eng.m, seed=1)
    d = _direction(eng, P, seed=21)
    jd, st = eng.solve_derivative(**d)
    jtg, ast = eng.solve_adjoint(*g)
    assert st["status"] == 1 and ast["status"] == 1, (st, ast)
    lhs = sum(gk @ v for gk, v in zip(g, jd))
    rhs = sum(a @ d[k] for a, k in zip(jtg, KEYS))
    scale = np.linalg.norm(np.concatenate(g)) * np.linalg.norm(np.concatenate(jd)) + \
        np.linalg.norm(np.concatenate(jtg)) * np.linalg.norm(np.concatenate([d[k] for k in KEYS]))
    assert abs(lhs - rhs) <= 1e-8 * scale, (lhs, rhs, scale)
    eng.close()


def test_finite_differences_through_engine_solves():
    P, q, A, b, sets = _problem(5, **CASES["wlinf"])
    eng = _engine(P, q, A, b, sets)
    assert eng.solve().status == "Solved"
    g = _grads(eng.n, eng.m)
    (dq, db, dPx, dAx, _, _), st = eng.solve_adjoint(*g)
    assert st["status"] == 1

    def sol(Px, q_, Ax, b_):
        e = _engine(sp.csc_matrix((Px, P.indices, P.indptr), shape=P.shape), q_,
                    sp.csc_matrix((Ax, A.indices, A.indptr), shape=A.shape), b_, sets)
        assert e.solve().status == "Solved"
        out = np.concatenate(_solution(e))
        e.close()
        return out

    d = _direction(eng, P, seed=7)
    h = 1e-5
    base = dict(Px=P.data, q_=q, Ax=A.data, b_=b)
    grad = dict(dq=dq, db=db, dAx=dAx, dPx=dPx)
    gcat = np.concatenate(g)
    for key, arg in (("dq", "q_"), ("db", "b_"), ("dAx", "Ax"), ("dPx", "Px")):
        plus, minus = dict(base), dict(base)
        plus[arg], minus[arg] = base[arg] + h * d[key], base[arg] - h * d[key]
        fd = (sol(**plus) - sol(**minus)) / (2 * h)
        got, dst = eng.solve_derivative(**{key: d[key]})
        assert dst["status"] == 1
        have = np.concatenate(got)
        assert np.abs(have - fd).max() <= 1e-5 * max(1.0, np.abs(fd).max()), (key, np.abs(have - fd).max())
        assert abs(grad[key] @ d[key] - gcat @ fd) <= 1e-5 * max(1.0, abs(gcat @ fd)), key
    eng.close()


def test_fp32_matches_the_restatement():
    """every hook compiled for F32; the solve to 1e-5, which fp32 reaches on this problem"""
    P, q, A, b, sets = _problem(4, **CASES["mixed"])
    eng = _engine(P, q, A, b, sets, dtype=np.float32, eps_abs=1e-5, eps_rel=1e-5)
    assert eng.solve().status == "Solved"
    g = _grads(eng.n, eng.m)
    d = _direction(eng, P)
    adj, ast = eng.solve_adjoint(*g)
    der, dst = eng.solve_derivative(**d)
    assert ast["status"] == dst["status"] == 1, (ast, dst)
    x, y, s = _solution(eng)
    cones = CJ.to_oracle(sets)
    wa = SA.unscaled(P, A, cones, x, s, y, gx=g[0], gy=g[1], gs=g[2])
    wd = SD.unscaled(P, A, cones, x, s, y, **d)
    for k, a in zip(KEYS[:4], adj[:4]):
        assert _rel(a, wa[k]) <= 1e-3, (k, _rel(a, wa[k]))
    for k, a in zip(OUT, der):
        assert _rel(a, wd[k]) <= 1e-3, (k, _rel(a, wd[k]))
    eng.close()


# ---------------------------------------------------------------------------
# 4. what stays as it was: hookless types, determinism, the next solve, the compile cache
# ---------------------------------------------------------------------------
def test_hookless_types_are_not_applicable():
    P, q, A, b, _ = _problem(6, cones={"soc2": (4,), "nonpos": (3,)})
    hookless = [cosmo_b200.ZeroSet(2), cosmo_b200.Box(np.array([-0.3, -1.0, -2.0]), np.array([0.2, 1.0, 2.0])),
                M.CustomCone(CC.soc2_type(), 4), M.CustomCone(CC.nonpos_type(), 3)]
    mixed = hookless[:2] + [M.CustomCone(CJ.soc2_type(), 4), M.CustomCone(CJ.nonpos_type(jacobian=False), 3)]
    for sets in (hookless, mixed):
        eng = _engine(P, q, A, b, sets)
        assert eng.solve().status == "Solved"
        out, st = eng.solve_adjoint(*_grads(eng.n, eng.m))
        assert st["status"] == -1 and all(np.isnan(a).all() for a in out)
        out, st = eng.solve_derivative(**_direction(eng, P))
        assert st["status"] == -1 and all(np.isnan(a).all() for a in out)
        eng.close()


@pytest.mark.parametrize("kkt", ["DeviceLdlKKTSolver", "CGIndirectKKTSolver"])
def test_determinism_and_the_next_solve(kkt):
    P, q, A, b, sets = _problem(8, **CASES["mixed"])
    eng, twin = _engine(P, q, A, b, sets, kkt, 10), _engine(P, q, A, b, sets, kkt, 10)
    for e in (eng, twin):
        assert e.solve().status == "Solved"
    g = _grads(eng.n, eng.m)
    d = _direction(eng, P)
    a1, ast1 = eng.solve_adjoint(*g)
    d1, dst1 = eng.solve_derivative(**d)
    a2, ast2 = eng.solve_adjoint(*g)
    d2, dst2 = eng.solve_derivative(**d)
    assert ast1 == ast2 and dst1 == dst2 and ast1["status"] == dst1["status"] == 1
    for a, c in zip(a1 + d1, a2 + d2):
        assert np.array_equal(_bits(a), _bits(c))
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


def test_one_compilation_for_two_engines_of_a_hooked_type():
    base = CJ.linf_type()
    kind = M.CustomConeType(base.name, base.source + "\n// %s\n" % uuid.uuid4().hex, base.granularity, base.n_params,
                            jacobian=True)
    P, q, A, b, sets = _problem(9, cones={"wlinf": (5,)})
    sets = sets[:2] + [M.CustomCone(kind, 5, [2.0])]
    stats = []
    for _ in range(2):
        eng = _engine(P, q, A, b, sets)
        assert eng.solve().status == "Solved"
        assert eng.solve_adjoint(*_grads(eng.n, eng.m))[1]["status"] == 1
        stats.append(eng.custom_cone_stats())
        eng.close()
    assert (stats[0]["compilations"], stats[0]["cache_hits"]) == (1, 0)
    assert (stats[1]["compilations"], stats[1]["cache_hits"]) == (0, 1)


# ---------------------------------------------------------------------------
# 5. autograd.solve_conic
# ---------------------------------------------------------------------------
def test_gradcheck_of_solve_conic_with_a_hooked_cone():
    torch = pytest.importorskip("torch")
    from cosmo_b200.autograd import solve_conic
    from tests.test_gpu_solve_derivative import _soc_problem
    P, q, A, b, _ = _soc_problem()
    sets = [M.CustomCone(CJ.soc2_type(), 3), cosmo_b200.Nonnegatives(1)]
    eng = _engine(P, q, A, b, sets, scaling=0, eps_abs=1e-12, eps_rel=1e-12)
    t = lambda a: torch.tensor(a, dtype=torch.float64, device="cuda", requires_grad=True)
    inputs = (t(P.data), t(q), t(A.data), t(b))
    x, y, s = solve_conic(eng, *inputs)
    r = np.linalg.norm(s[1:3].detach().cpu().numpy())
    assert abs(r - float(s[0])) <= 1e-9 and r > 0.1        # on the boundary, off the tip
    assert torch.autograd.gradcheck(lambda Px, q_, Ax, b_: solve_conic(eng, Px, q_, Ax, b_), inputs, eps=1e-6,
                                    atol=1e-5, rtol=1e-4, check_forward_ad=True)
    eng.close()
