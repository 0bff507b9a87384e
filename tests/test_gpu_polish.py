"""GPU tests of solution polishing (cosmo_b200_polish, Engine.polish, Settings(polish=True)): the reference's known
answers, parity with the NumPy restatement of tests/polish_reference.py on the iterates read back from the same
engine, the state the handle keeps, the cases it does not apply to, rejection, refusals, device buffers, determinism,
fp32 and a degenerate LP.  Every case runs with both direct plugins; fp64 with scaling 0 and 10 unless stated."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp

import cosmo_b200
from cosmo_b200 import engine as E
from cosmo_b200 import model as M
from cosmo_b200.problems import _stratified_csc, _stratified_csr
from oracle import cosmo_oracle as O
from tests import golden_problems as G
from tests import polish_reference as R
from tests.gpu_helpers import U32

pytestmark = pytest.mark.gpu

PLUGINS = ["DeviceLdlKKTSolver", "DeviceSupernodalKKTSolver"]
SCALINGS = [0, 10]


def _to_mine(cons):
    out = []
    for c in cons:
        S = c.convex_set
        if isinstance(S, O.Box):
            S2 = cosmo_b200.Box(S.l, S.u)
        elif isinstance(S, (O.PowerCone, O.DualPowerCone)):
            S2 = getattr(cosmo_b200, type(S).__name__)(S.alpha)
        else:
            S2 = getattr(cosmo_b200, type(S).__name__)(S.dim)
        out.append(cosmo_b200.Constraint(c.A, c.b, S2))
    return out


def _model(builder, dtype=np.float64, **kw):
    P, q, cons = builder()
    model = cosmo_b200.Model(dtype=dtype)
    cosmo_b200.assemble(model, P, q, _to_mine(cons), cosmo_b200.Settings(**kw))
    return model


def _bits(a):
    a = a.cpu().numpy() if hasattr(a, "cpu") else a
    return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


def _outputs(eng):
    return np.empty(eng.n), np.empty(eng.m), np.empty(eng.m)


# ---------------------------------------------------------------------------
# 1. known answers
# ---------------------------------------------------------------------------
KNOWN = [("G1", G.g1_qp_nonneg, G.G1_X, G.G1_OBJ), ("G1b", G.g1_qp_box, G.G1_X, G.G1_OBJ),
         ("G2", G.g2_box_feasible, np.array([0.0, 1.0]), -0.5), ("G12", G.g12_lp, G.G12_X, G.G12_OBJ)]


@pytest.mark.parametrize("scaling", SCALINGS)
@pytest.mark.parametrize("kkt", PLUGINS)
@pytest.mark.parametrize("name,builder,x_star,obj_star", KNOWN, ids=[k[0] for k in KNOWN])
def test_known_answers(name, builder, x_star, obj_star, kkt, scaling):
    model = _model(builder, kkt_solver=kkt, scaling=scaling)
    res = model.optimize()
    assert res.status == "Solved" and res.polish == "Not_run"
    x, y, s, st = model.engine.polish(x=np.empty(len(x_star)), y=np.empty(model.m), s=np.empty(model.m))
    assert st["status"] == 1, st
    assert np.abs(x - x_star).max() <= 1e-9
    assert abs(st["obj_val"] - obj_star) <= 1e-9
    assert st["r_prim"] <= res.info.r_prim and st["r_dual"] <= res.info.r_dual


# ---------------------------------------------------------------------------
# 2. parity with the restatement on the engine's own iterates
# ---------------------------------------------------------------------------
def _qp_with_zero_block(n, m, density, seed, k):
    """random_sparse_qp plus k ZeroSet rows through its feasible point x0 (restated from the generator's rng stream)."""
    P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(n, m, density, seed=seed)
    rng = np.random.default_rng(seed)
    _stratified_csc(rng, m, n, max(1, int(round(density * m))))
    _stratified_csr(rng, n, n, 5)
    rng.uniform(0.1, 1.0, n)
    x0 = rng.standard_normal(n)
    assert np.all(A[: m // 2] @ x0 <= b[: m // 2])       # the generator's strictly feasible point
    Z = sp.random(k, n, density=0.02, random_state=np.random.default_rng(seed + 1), format="csc") + sp.eye(k, n)
    A2 = sp.vstack([Z, A], format="csc")
    b2 = np.concatenate([Z @ x0, b])
    return P, q, A2, b2, [cosmo_b200.ZeroSet(k)] + list(sets)


def _sets_rows(sets):
    return R.row_classes(O_cones(sets))


def O_cones(sets):
    from oracle.bridge import to_oracle_cones
    return to_oracle_cones(sets)


def _engine(P, q, A, b, sets, kkt, scaling, dtype=np.float64, **kw):
    st = cosmo_b200.Settings(kkt_solver=kkt, scaling=scaling, **kw).to_struct()
    return E.Engine(P, q, A, b, [M.set_tuple(S) for S in sets], st, dtype=dtype, equilibrate=scaling != 0)


def _scaled(eng, P, q, A, b, sets):
    D, Ev, c = eng.scaling()
    Dm, Em = sp.diags(D), sp.diags(Ev)
    cls, l, u = _sets_rows(sets)
    return (c * (Dm @ sp.csc_matrix(P) @ Dm), c * D * q, Em @ sp.csc_matrix(A) @ Dm, Ev * b, cls, Ev * l, Ev * u, D, Ev, c)


def _check_parity(eng, out, P, q, A, b, sets):
    """The engine's polish against the restatement on the same scaled iterates: the same verdict, counts, buffers and
    candidate residuals (a rejection hands back the unpolished solution on both sides)."""
    Ps, qs, As, bs, cls, ls, us, D, Ev, c = _scaled(eng, P, q, A, b, sets)
    ref = R.polish(Ps, qs, As, bs, cls, ls, us, out.x, out.s, out.mu, D=D, E=Ev, c=c)
    x, y, s, st = eng.polish(x=np.empty(eng.n), y=np.empty(eng.m), s=np.empty(eng.m))
    assert st["status"] == ref["status"]
    assert (st["n_lower"], st["n_upper"], st["n_equality"]) == (ref["n_lower"], ref["n_upper"], ref["n_equality"])
    for got, want in ((x, ref["x"]), (y, ref["y"]), (s, ref["s"])):
        assert np.linalg.norm(got - want) <= 1e-9 * max(np.linalg.norm(want), 1e-300)
    cand = R.residuals(Ps, qs, As, bs, ref["x_p"], ref["s_p"], ref["mu_p"], D, Ev, c)
    assert abs(st["r_prim"] - ref["r_prim"]) <= 1e-10 * (1 + cand[2])
    assert abs(st["r_dual"] - ref["r_dual"]) <= 1e-10 * (1 + cand[3])
    assert abs(st["obj_val"] - ref["obj_val"]) <= 1e-10 * max(1.0, abs(ref["obj_val"]))
    return st


@pytest.mark.parametrize("scaling", SCALINGS)
@pytest.mark.parametrize("kkt", PLUGINS)
@pytest.mark.parametrize("n", [200, 2000])
def test_parity_with_the_restatement(n, kkt, scaling):
    P, q, A, b, sets = _qp_with_zero_block(n, 2 * n, 20.0 / n, 3, n // 20)
    eng = _engine(P, q, A, b, sets, kkt, scaling)
    out = eng.solve()
    assert out.status == "Solved"
    st = _check_parity(eng, out, P, q, A, b, sets)
    assert st["n_equality"] >= n // 20 and st["n_lower"] + st["n_upper"] > 0
    # at n = 2000 without scaling the 1e-5 iterates can miss rows of the active set, and both sides reject alike
    assert st["status"] == 1 or (n == 2000 and scaling == 0)


@pytest.mark.parametrize("scaling", SCALINGS)
@pytest.mark.parametrize("kkt", PLUGINS)
def test_parity_after_update_q(kkt, scaling):
    P, q, cons = G.g14_update_qp()
    Pm, qm, A, b, cones = O.assemble(P, q, cons)
    sets = [cosmo_b200.Nonnegatives(A.shape[0])]
    eng = _engine(Pm, qm, A, b, sets, kkt, scaling)
    eng.solve()
    q2 = np.array([2.0, 3.0])
    eng.update_qb_original(q=q2)
    out = eng.solve()
    assert out.status == "Solved"
    assert _check_parity(eng, out, Pm, q2, A, b, sets)["status"] == 1


# ---------------------------------------------------------------------------
# 3. the handle is left as the solve left it
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("scaling", SCALINGS)
@pytest.mark.parametrize("kkt", PLUGINS)
def test_state_untouched(kkt, scaling):
    P, q, A, b, sets = _qp_with_zero_block(200, 400, 0.1, 5, 10)
    runs = []
    for polish in (True, False):
        eng = _engine(P, q, A, b, sets, kkt, scaling)
        eng.solve()
        if polish:
            eng.polish()
            eng.polish(x=np.empty(eng.n))
        runs.append(eng.solve())
    a, b_ = runs
    for f in ("x", "s", "mu"):
        assert np.array_equal(_bits(getattr(a, f)), _bits(getattr(b_, f))), f
    assert (a.iter, a.status) == (b_.iter, b_.status)
    assert np.array_equal(_bits(a.rho_updates), _bits(b_.rho_updates))


# ---------------------------------------------------------------------------
# 4. not applicable
# ---------------------------------------------------------------------------
def _sdp():
    return G.g4_small_sdp()


@pytest.mark.parametrize("kkt", PLUGINS)
@pytest.mark.parametrize("builder", [G.g3_hs21, _sdp, G.g15_exp_feasible, G.g2_box_primal_infeasible_1,
                                     G.g2_box_primal_infeasible_2, G.g2_box_dual_infeasible])
def test_not_applicable(builder, kkt):
    model = _model(builder, kkt_solver=kkt, max_iter=3000)
    res = model.optimize()
    eng = model.engine
    want = eng.solution(False, *_outputs(eng))
    got_x, got_y, got_s, st = eng.polish(x=np.empty(eng.n), y=np.empty(eng.m), s=np.empty(eng.m))
    assert st["status"] == -1, (res.status, st)
    assert (st["n_lower"], st["n_upper"], st["n_equality"]) == (0, 0, 0)
    assert all(np.isnan(st[k]) for k in ("r_prim", "r_dual", "obj_val", "refine_residual"))
    for g, w in zip((got_x, got_y, got_s), want):
        assert np.array_equal(_bits(g), _bits(w))


# ---------------------------------------------------------------------------
# 5. rejection
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("kkt", PLUGINS)
@pytest.mark.parametrize("case", ["g12", "qp"])
def test_rejection_follows_the_rule(case, kkt):
    if case == "g12":
        P, q, cons = G.g12_lp()
        P, q, A, b, cones = O.assemble(P, q, cons)
        sets = [cosmo_b200.Nonnegatives(A.shape[0])]
    else:
        P, q, A, b, sets = _qp_with_zero_block(200, 400, 0.1, 7, 10)
    eng = _engine(P, q, A, b, sets, kkt, 10, max_iter=2)
    out = eng.solve()
    assert out.status == "Max_iter_reached"
    Ps, qs, As, bs, cls, ls, us, D, Ev, c = _scaled(eng, P, q, A, b, sets)
    ref = R.polish(Ps, qs, As, bs, cls, ls, us, out.x, out.s, out.mu, D=D, E=Ev, c=c)
    cand = R.residuals(Ps, qs, As, bs, ref["x_p"], ref["s_p"], ref["mu_p"], D, Ev, c)
    x, y, s, st = eng.polish(x=np.empty(eng.n), y=np.empty(eng.m), s=np.empty(eng.m))
    assert st["status"] in (0, 1)
    if st["status"] == 1:
        assert st["r_prim"] <= max(out.r_prim, 10 * 2.0 ** -53 * (1 + cand[2]) * 1.001)
        assert st["r_dual"] <= max(out.r_dual, 10 * 2.0 ** -53 * (1 + cand[3]) * 1.001)
    else:
        worse = not (st["r_prim"] <= out.r_prim and st["r_dual"] <= out.r_dual)
        assert worse or np.isnan(st["r_prim"])
        for g, w in zip((x, y, s), eng.solution(False, *_outputs(eng))):
            assert np.array_equal(_bits(g), _bits(w))


# ---------------------------------------------------------------------------
# 6. refusals
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("kkt", ["CGIndirectKKTSolver", "MINRESIndirectKKTSolver"])
def test_indirect_plugins_are_refused(kkt):
    P, q, cons = G.g1_qp_box()
    Pm, qm, A, b, cones = O.assemble(P, q, cons)
    eng = _engine(Pm, qm, A, b, [cosmo_b200.Box(cones[0].l, cones[0].u)], kkt, 10)
    eng.solve()
    with pytest.raises(E.EngineError) as e:
        eng.polish()
    assert e.value.code == E.ERR_UNSUPPORTED


@pytest.mark.parametrize("kkt", PLUGINS)
def test_invalid_calls(kkt):
    P, q, cons = G.g1_qp_box()
    Pm, qm, A, b, cones = O.assemble(P, q, cons)
    eng = _engine(Pm, qm, A, b, [cosmo_b200.Box(cones[0].l, cones[0].u)], kkt, 10)
    with pytest.raises(E.EngineError) as e:
        eng.polish()                                    # no solve yet
    assert e.value.code == E.ERR_INVALID
    eng.solve()
    for kw in ({"delta": 0.0}, {"delta": -1e-6}, {"delta": float("nan")}, {"refine_iter": -1}, {"refine_iter": 101}):
        with pytest.raises(E.EngineError) as e:
            eng.polish(**kw)
        assert e.value.code == E.ERR_INVALID
    out = (C.c_double * 8)()
    bad = E.PolishSettings(1e-6, 3, 1)
    assert eng._lib.cosmo_b200_polish(eng._h, C.byref(bad), None, None, None, out) == E.ERR_INVALID
    eng.warm_start(x=np.zeros(eng.n))
    with pytest.raises(E.EngineError) as e:
        eng.polish()                                    # a warm start ends the solution
    assert e.value.code == E.ERR_INVALID


# ---------------------------------------------------------------------------
# 7. device buffers, 8. determinism
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("kkt", PLUGINS)
def test_device_buffers_and_determinism(kkt):
    torch = pytest.importorskip("torch")
    P, q, A, b, sets = _qp_with_zero_block(200, 400, 0.1, 9, 10)
    eng = _engine(P, q, A, b, sets, kkt, 10)
    eng.solve()
    hx, hy, hs, st1 = eng.polish(x=np.empty(eng.n), y=np.empty(eng.m), s=np.empty(eng.m))
    assert st1["status"] == 1
    dx, dy, ds = (torch.empty(k, dtype=torch.float64, device="cuda") for k in (eng.n, eng.m, eng.m))
    _, _, _, st2 = eng.polish(x=dx, y=dy, s=ds)
    torch.cuda.synchronize()
    for h, d in ((hx, dx), (hy, dy), (hs, ds)):
        assert np.array_equal(_bits(h), _bits(d))
    hx2, hy2, hs2, st3 = eng.polish(x=np.empty(eng.n), y=np.empty(eng.m), s=np.empty(eng.m))
    for a, b_ in ((hx, hx2), (hy, hy2), (hs, hs2)):
        assert np.array_equal(_bits(a), _bits(b_))
    for k in E.POLISH_STATS:
        assert np.array_equal(_bits(np.array([st1[k], st1[k]])), _bits(np.array([st2[k], st3[k]]))), k


# ---------------------------------------------------------------------------
# 9. fp32, 10. a degenerate LP
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("kkt", PLUGINS)
@pytest.mark.parametrize("builder", [G.g1_qp_nonneg, G.g12_lp])
def test_fp32_never_errors(builder, kkt):
    model = _model(builder, dtype=np.float32, kkt_solver=kkt)
    res = model.optimize()
    _, _, _, st = model.engine.polish(x=np.empty(model.engine.n))
    assert st["status"] in (0, 1)
    if st["status"] == 1:
        assert st["r_prim"] <= max(res.info.r_prim, 10 * U32 * (1 + 2 * res.info.max_norm_prim))
        assert st["r_dual"] <= max(res.info.r_dual, 10 * U32 * (1 + 2 * res.info.max_norm_dual))


def _degenerate_lp():
    # min x1 + x2 over x >= 0, x1 + x2 >= 0, x1 - x2 >= 0, x2 - x1 >= 0: five rows active at x* = 0, two variables
    A = np.array([[1.0, 0.0], [0.0, 1.0], [1.0, 1.0], [1.0, -1.0], [-1.0, 1.0]])
    return np.zeros((2, 2)), np.array([1.0, 1.0]), [O.Constraint(A, np.zeros(5), O.Nonnegatives(5))]


@pytest.mark.parametrize("scaling", SCALINGS)
@pytest.mark.parametrize("kkt", PLUGINS)
def test_degenerate_lp(kkt, scaling):
    model = _model(_degenerate_lp, kkt_solver=kkt, scaling=scaling)
    res = model.optimize()
    _, _, _, st = model.engine.polish(x=np.empty(2))
    assert st["status"] in (0, 1)
    if st["status"] == 1:
        assert np.isfinite(st["r_prim"]) and np.isfinite(st["r_dual"])
        assert st["r_prim"] <= max(res.info.r_prim, 1e-14) and st["r_dual"] <= max(res.info.r_dual, 1e-14)


# ---------------------------------------------------------------------------
# 11. Model level
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("scaling", SCALINGS)
def test_model_polish_and_the_next_solve(scaling):
    runs, models = [], []
    for polish in (True, False):
        model = _model(G.g12_lp, kkt_solver="DeviceLdlKKTSolver", scaling=scaling, polish=polish)
        first = model.optimize()
        model.update(q=np.array([1.0, 2.0, 3.0, 4.5]))
        runs.append((first, model.optimize()))
        models.append(model)
    (pol, nxt_p), (unp, nxt_u) = runs
    assert pol.polish == "Polished" and unp.polish == "Not_run" and "polish_time" in pol.times
    assert np.abs(pol.x - G.G12_X).max() <= 1e-9 and abs(pol.obj_val - G.G12_OBJ) <= 1e-9
    assert pol.status == unp.status and pol.iter == unp.iter
    assert pol.info.r_prim <= unp.info.r_prim and pol.info.r_dual <= unp.info.r_dual
    assert nxt_p.polish == "Polished"
    # the second solve starts from the ADMM iterates either way: bit for bit the same ADMM run
    assert nxt_p.iter == nxt_u.iter and nxt_p.status == nxt_u.status
    assert np.array_equal(_bits(nxt_p.info.rho_updates), _bits(nxt_u.info.rho_updates))
    for f in ("x", "s", "mu"):
        assert np.array_equal(_bits(getattr(models[0], f)), _bits(getattr(models[1], f))), f
    with pytest.raises(ValueError):
        _model(G.g12_lp, kkt_solver="DeviceLdlKKTSolver", polish=True).optimize(solution="device")
