"""GPU tests of the forward derivative of polished solutions (cosmo_b200_derivative, Engine.derivative,
Model.derivative, the jvp of autograd.solve_qp): the engine against the restatement of
tests/polish_derivative_reference.py on the engine's own polished point, the pairing with Engine.adjoint, directional
finite differences through full engine re-solves, dependent active rows, host and device buffers, determinism and
untouched state, refusals and statuses, and forward-mode torch.autograd.  Both direct plugins throughout; scaling 0
and 10 unless stated."""
import numpy as np
import pytest
import scipy.sparse as sp

import cosmo_b200
from cosmo_b200 import engine as E
from oracle import cosmo_oracle as O
from oracle.bridge import to_oracle_cones
from tests import adjoint_reference as AR
from tests import golden_problems as G
from tests import polish_derivative_reference as PD
from tests import polish_reference as R
from tests.gpu_helpers import U32
from tests.test_gpu_adjoint import PLUGINS, SCALINGS, _bits, _code, _engine, _fd_problem, _grads, _polish, _problem, _resolve

pytestmark = pytest.mark.gpu

OUT = ("dx", "dy", "ds")


def _direction(P, A, sets, seed):
    """A random direction of every input: P symmetric on its pattern, A on its pattern, the Box bounds where finite."""
    m, n = A.shape
    rng = np.random.default_rng(seed)
    pr, pc = P.indices, np.repeat(np.arange(n), np.diff(P.indptr))
    Msym = sp.csc_matrix((rng.standard_normal(P.nnz), P.indices, P.indptr), shape=P.shape)
    cls, l, u = R.row_classes(to_oracle_cones(sets))
    box = cls == R.BOX
    return dict(dPx=np.asarray((Msym + Msym.T)[pr, pc]).ravel(), dq=rng.standard_normal(n),
                dAx=rng.standard_normal(A.nnz), db=rng.standard_normal(m),
                dl=np.where(box & np.isfinite(l), rng.standard_normal(m), 0.0),
                du=np.where(box & np.isfinite(u), rng.standard_normal(m), 0.0))


def _scaled(eng, P, A, sets, out):
    """The engine's scaled data and its classification of the solve's (s, mu), as test_gpu_adjoint forms them."""
    D, Ev, c = eng.scaling()
    D, Ev = np.asarray(D, dtype=float), np.asarray(Ev, dtype=float)
    Ps = sp.csc_matrix(c * (sp.diags(D) @ P @ sp.diags(D)))
    As = sp.csc_matrix(sp.diags(Ev) @ A @ sp.diags(D))
    cls, l, u = R.row_classes(to_oracle_cones(sets))
    kind, _ = R.classify(cls, Ev * l, Ev * u, out.s.astype(float), out.mu.astype(float))
    return D, Ev, c, Ps, As, cls, kind


# ---------------------------------------------------------------------------
# 1. the engine against the restatement on its own polished point
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["fp64", "fp32"])
@pytest.mark.parametrize("scaling", SCALINGS)
@pytest.mark.parametrize("kkt", PLUGINS)
def test_engine_matches_the_restatement(kkt, scaling, dtype):
    P, q, A, b, sets = _problem(200, 3)
    eng = _engine(P, q, A, b, sets, kkt, scaling, dtype)
    out = eng.solve()
    assert out.status == "Solved"
    x, y, s, pst = eng.polish(x=np.empty(eng.n), y=np.empty(eng.m), s=np.empty(eng.m))
    d = _direction(P, A, sets, 8)
    got, st = eng.derivative(**d)
    assert st["status"] == pst["status"]
    if dtype == np.float32 and pst["status"] == 0:   # fp32 polishes may be rejected: then NaN, not derivatives
        assert all(np.all(np.isnan(g)) for g in got) and np.isnan(st["refine_residual"])
        return
    assert st["status"] == 1
    D, Ev, c, Ps, As, cls, kind = _scaled(eng, P, A, sets, out)
    active = kind != R.INACTIVE
    assert st["n_active"] == int(active.sum())
    ref = PD.derivative(Ps, As, cls, kind, x / D, c * y / Ev, **d, D=D, E=Ev, c=c)
    K = AR.kkt_matrix(Ps, As, kind)
    kappa = np.linalg.cond(K)
    if dtype == np.float64:
        # normwise backward error of the engine's (x~', y~') in the scaled system
        z = np.concatenate([got[0] / D, (c * got[1] / Ev)[active]])
        rhs = np.concatenate([ref["rx"], ref["rs"][active]])
        eta = np.abs(K @ z - rhs).max() / (np.abs(K).sum(axis=1).max() * np.abs(z).max() + np.abs(rhs).max())
        assert eta <= 1e-13, eta
        assert st["refine_residual"] <= 1e-10 * (1 + np.abs(rhs).max())
    tol = (1e-14 if dtype == np.float64 else 64 * U32) * kappa
    for k, g in zip(OUT, got):
        want = ref[k]
        assert np.linalg.norm(g - want) <= tol * np.linalg.norm(want), (k, np.linalg.norm(g - want) / np.linalg.norm(want), kappa)
    assert np.all(got[1][~active] == 0.0)
    # ds equals the bound direction on the active rows, up to the refinement residual
    want_s = PD.bound_direction(cls, kind, d["dl"], d["du"])
    assert np.abs(got[2] - want_s)[active].max() <= tol * max(1.0, np.abs(got[2]).max())


# ---------------------------------------------------------------------------
# 2. the pairing with Engine.adjoint on the same engine and point
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("scaling", SCALINGS)
@pytest.mark.parametrize("kkt", PLUGINS)
def test_pairing_with_the_adjoint(kkt, scaling):
    P, q, A, b, sets = _problem(200, 4)
    eng = _engine(P, q, A, b, sets, kkt, scaling)
    assert eng.solve().status == "Solved"
    _polish(eng)
    d = _direction(P, A, sets, 11)
    (dx, dy, ds), st = eng.derivative(**d)
    gx, gy, gs = _grads(eng.n, eng.m, 12)
    (dq, db, dPx, dAx, dl, du), sta = eng.adjoint(gx, gy, gs)
    assert st["status"] == sta["status"] == 1
    assert (st["n_active"], st["n_weak"]) == (sta["n_active"], sta["n_weak"])
    lhs = gx @ dx + gy @ dy + gs @ ds
    rhs = dPx @ d["dPx"] + dq @ d["dq"] + dAx @ d["dAx"] + db @ d["db"] + dl @ d["dl"] + du @ d["du"]
    assert abs(lhs - rhs) <= 1e-12 * (abs(lhs) + abs(rhs)), (lhs, rhs)


# ---------------------------------------------------------------------------
# 3. directional finite differences through full engine re-solves
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("scaling", SCALINGS)
@pytest.mark.parametrize("kkt", PLUGINS)
def test_directional_finite_differences(kkt, scaling):
    P, q, A, b, sets = _fd_problem()
    eng = _engine(P, q, A, b, sets, kkt, scaling)
    _resolve(eng, P.data, q, A.data, b)
    full = _direction(P, A, sets, 4)
    eps = 1e-6
    for what in ("dq", "db", "dPx", "dAx"):
        d = {k: (v if k == what else None) for k, v in full.items()}
        _resolve(eng, P.data, q, A.data, b)
        got, st = eng.derivative(**d)
        assert st["status"] == 1 and st["n_weak"] == 0
        z = lambda k: 0.0 if d[k] is None else d[k]
        sols = []
        for sgn in (1.0, -1.0):
            sols.append(_resolve(eng, P.data + sgn * eps * z("dPx"), q + sgn * eps * z("dq"), A.data + sgn * eps * z("dAx"),
                                 b + sgn * eps * z("db"))[:3])
        scale = max(1.0, max(np.abs(g).max() for g in got))
        for k, g, a, b_ in zip(OUT, got, *sols):
            fd = (a - b_) / (2 * eps)
            assert np.abs(fd - g).max() <= 1e-6 * scale, (what, k, np.abs(fd - g).max())


@pytest.mark.parametrize("scaling", SCALINGS)
@pytest.mark.parametrize("kkt", PLUGINS)
def test_dependent_rows_of_g1(kkt, scaling):
    # rows 0 and 3 are x1 + x2 <= 1 and -(x1 + x2) <= -1: dx and ds are unique, dy only through A_A' dy_A
    Pd, qd, cons = G.g1_qp_nonneg()
    P, q, A, b, cones = O.assemble(Pd, qd, cons)
    P, A = sp.csc_matrix(P), sp.csc_matrix(A)
    sets = [cosmo_b200.Nonnegatives(A.shape[0])]
    eng = _engine(P, q, A, b, sets, kkt, scaling)
    x, y, s, _ = _resolve(eng, P.data, q, A.data, b)
    assert np.abs(x - G.G1_X).max() <= 1e-9
    rng = np.random.default_rng(2)
    eb = np.zeros(A.shape[0]); eb[0], eb[3] = 1.0, -1.0
    pr, pc = P.indices, np.repeat(np.arange(2), np.diff(P.indptr))
    Msym = sp.csc_matrix((rng.standard_normal(P.nnz), P.indices, P.indptr), shape=P.shape)
    dirs = {"q": (None, rng.standard_normal(2), None), "P": (np.asarray((Msym + Msym.T)[pr, pc]).ravel(), None, None),
            "b": (None, None, eb)}
    eps = 1e-6
    for what, (eP, eq, eb_) in dirs.items():
        _resolve(eng, P.data, q, A.data, b)
        (dx, dy, ds), st = eng.derivative(dPx=eP, dq=eq, db=eb_)
        assert st["status"] == 1
        z = lambda a: 0.0 if a is None else a
        sols = [_resolve(eng, P.data + sgn * eps * z(eP), q + sgn * eps * z(eq), A.data, b + sgn * eps * z(eb_))
                for sgn in (1.0, -1.0)]
        fx = (sols[0][0] - sols[1][0]) / (2 * eps)
        fs = (sols[0][2] - sols[1][2]) / (2 * eps)
        fty = A.T @ ((sols[0][1] - sols[1][1]) / (2 * eps))
        assert np.abs(fx - dx).max() <= 1e-6 * max(1.0, np.abs(dx).max()), what
        assert np.abs(fs - ds).max() <= 1e-6 * max(1.0, np.abs(ds).max()), what
        assert np.abs(fty - A.T @ dy).max() <= 1e-6 * max(1.0, np.abs(A.T @ dy).max()), what


# ---------------------------------------------------------------------------
# 4. host and device buffers, determinism, untouched state
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("kkt", PLUGINS)
def test_host_and_cuda_arrays_and_repeated_calls_are_bit_identical(kkt):
    torch = pytest.importorskip("torch")
    P, q, A, b, sets = _problem(200, 5)
    eng = _engine(P, q, A, b, sets, kkt, 10)
    assert eng.solve().status == "Solved"
    _polish(eng)
    d = _direction(P, A, sets, 6)
    host1, st1 = eng.derivative(**d)
    host2, st2 = eng.derivative(**d)
    cuda = {k: torch.from_numpy(v).cuda() for k, v in d.items()}
    outs = [torch.empty(len(h), dtype=torch.float64, device="cuda") for h in host1]
    dev, st3 = eng.derivative(**cuda, dx=outs[0], dy=outs[1], ds=outs[2])
    torch.cuda.synchronize()
    for a, b_, c_ in zip(host1, host2, dev):
        assert np.array_equal(_bits(a), _bits(b_)) and np.array_equal(_bits(a), _bits(c_))
    assert st1 == st2 == st3
    # adjoint -> derivative -> adjoint: the adjoint's outputs do not move
    g = _grads(eng.n, eng.m)
    a1, sa1 = eng.adjoint(*g)
    eng.derivative(**d)
    a2, sa2 = eng.adjoint(*g)
    for u, v in zip(a1, a2):
        assert np.array_equal(_bits(u), _bits(v))
    assert sa1 == sa2


@pytest.mark.parametrize("kkt", PLUGINS)
def test_the_next_solve_is_the_solve_of_a_twin_that_never_ran_the_derivative(kkt):
    P, q, A, b, sets = _problem(200, 6)
    engs = [_engine(P, q, A, b, sets, kkt, 10) for _ in range(2)]
    for e in engs:
        assert e.solve().status == "Solved"
        _polish(e)
    engs[0].derivative(**_direction(P, A, sets, 7))
    sol0 = engs[0].solution(x=np.empty(engs[0].n), y=np.empty(engs[0].m), s=np.empty(engs[0].m))
    sol1 = engs[1].solution(x=np.empty(engs[1].n), y=np.empty(engs[1].m), s=np.empty(engs[1].m))
    for a, b_ in zip(sol0, sol1):
        assert np.array_equal(_bits(a), _bits(b_))
    q2 = q + 0.01
    D, _, c = engs[0].scaling()
    outs = []
    for e in engs:
        e.update_qb(q=c * D * q2)
        outs.append(e.solve())
    assert outs[0].iter == outs[1].iter
    for k in ("x", "s", "mu"):
        assert np.array_equal(getattr(outs[0], k), getattr(outs[1], k))


# ---------------------------------------------------------------------------
# 5. refusals and statuses
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("kkt", PLUGINS)
def test_no_polish_record_after_solve_update_or_reset(kkt):
    P, q, A, b, sets = _problem(200, 7)
    eng = _engine(P, q, A, b, sets, kkt, 0)
    dq = np.ones(eng.n)
    assert _code(lambda: eng.derivative(dq=dq)) == E.ERR_INVALID           # never polished
    for breaker in (lambda: eng.solve(), lambda: eng.update_qb(q=q), lambda: eng.reset(),
                    lambda: eng.update_matrices(P.data, A.data, q, b)):
        assert eng.solve().status == "Solved"
        _polish(eng)
        eng.derivative(dq=dq)
        breaker()
        assert _code(lambda: eng.derivative(dq=dq)) == E.ERR_INVALID
    assert eng.solve().status == "Solved"
    _polish(eng)
    assert _code(lambda: eng.derivative(dq=dq, refine_iter=101)) == E.ERR_INVALID
    assert _code(lambda: eng.derivative(dq=dq, refine_iter=-1)) == E.ERR_INVALID
    assert eng.derivative(dq=dq, refine_iter=100)[1]["status"] == 1


@pytest.mark.parametrize("kkt", ["CGIndirectKKTSolver", "MINRESIndirectKKTSolver"])
def test_indirect_plugins_are_refused(kkt):
    P, q, A, b, sets = _problem(200, 7)
    eng = _engine(P, q, A, b, sets, kkt, 0)
    eng.solve()
    assert _code(lambda: eng.derivative(dq=np.ones(eng.n))) == E.ERR_UNSUPPORTED


@pytest.mark.parametrize("kkt", PLUGINS)
def test_an_soc_row_gives_status_minus_one_and_nan(kkt):
    n = 3
    P = sp.identity(n, format="csc")
    q = np.array([1.0, -1.0, 0.5])
    A = sp.vstack([sp.identity(n), -sp.identity(n)], format="csc")
    b = np.array([1.0, 1.0, 1.0, 2.0, 0.0, 0.0])
    sets = [cosmo_b200.Nonnegatives(3), cosmo_b200.SecondOrderCone(3)]
    eng = _engine(P, q, A, b, sets, kkt, 0)
    eng.solve()
    _, _, _, pst = eng.polish(x=np.empty(n), y=np.empty(6), s=np.empty(6))
    assert pst["status"] == -1
    outs, st = eng.derivative(dq=np.ones(n))
    assert st["status"] == -1 and st["n_active"] == 0 and np.isnan(st["refine_residual"])
    assert all(np.all(np.isnan(o)) for o in outs)


@pytest.mark.parametrize("kkt", PLUGINS)
def test_the_weak_row_count(kkt):
    # G2 as written: x = (0, 1) sits at the upper bound of its second row with a zero multiplier.  Whether the polish
    # takes that row as active follows the sign of mu the solve leaves there; when it does, the row is weakly active.
    # Either way both calls count the active inequality rows whose polished multiplier is 0.
    P, q, cons = G.g2_box_feasible()
    Pm, qm, A, b, cones = O.assemble(P, q, cons)
    P, A = sp.csc_matrix(Pm), sp.csc_matrix(A)
    sets = [cosmo_b200.Box(cones[0].l, cones[0].u)]
    eng = _engine(P, qm, A, b, sets, kkt, 0)
    out = eng.solve()
    assert out.status == "Solved"
    x, y, s, _ = _polish(eng)
    cls, l, u = R.row_classes(cones)
    kind, _ = R.classify(cls, l, u, out.s.astype(float), out.mu.astype(float))
    weak = int((((kind == R.LOWER) | (kind == R.UPPER)) & (y == 0.0)).sum())
    (dx, dy, ds), st = eng.derivative(dq=np.array([1.0, 0.0]))
    _, sta = eng.adjoint(np.ones(2))
    assert st["status"] == 1 and st["n_active"] == int((kind != R.INACTIVE).sum()) and st["n_weak"] == weak
    assert (st["n_active"], st["n_weak"]) == (sta["n_active"], sta["n_weak"])


# ---------------------------------------------------------------------------
# 6. Model.derivative and torch.autograd
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("kkt", PLUGINS)
def test_model_derivative_in_update_coordinates(kkt):
    P, q, cons = G.g1_qp_box()
    model = cosmo_b200.Model()
    with pytest.raises(ValueError):
        model.derivative(dq=np.ones(2))
    box = cons[0].convex_set
    cosmo_b200.assemble(model, P, q, [cosmo_b200.Constraint(c.A, c.b, cosmo_b200.Box(c.convex_set.l, c.convex_set.u))
                                      for c in cons], cosmo_b200.Settings(kkt_solver=kkt, polish=True))
    res = model.optimize()
    assert res.polish == "Polished"
    rng = np.random.default_rng(3)
    P0, A0 = model.P0, model.A0
    dP = sp.csc_matrix((rng.standard_normal(P0.nnz), P0.indices, P0.indptr), shape=P0.shape)
    dP = sp.csc_matrix(dP + dP.T)
    dA = sp.csc_matrix((rng.standard_normal(A0.nnz), A0.indices, A0.indptr), shape=A0.shape)
    d = dict(dq=rng.standard_normal(2), db=rng.standard_normal(3), dl=rng.standard_normal(3), du=rng.standard_normal(3))
    got = model.derivative(dP=dP, dA=dA, **d)
    assert got["stats"]["status"] == 1
    m = A0.shape[0]
    cls, l, u = np.full(m, R.BOX, dtype=np.int8), np.asarray(box.l, dtype=float), np.asarray(box.u, dtype=float)
    kind, _ = R.classify(cls, l, u, res.s, -res.y)
    pr, pc = P0.indices, np.repeat(np.arange(P0.shape[1]), np.diff(P0.indptr))
    ar, ac = A0.indices, np.repeat(np.arange(A0.shape[1]), np.diff(A0.indptr))
    ref = PD.derivative(P0, A0, cls, kind, res.x, res.y, dPx=np.asarray(dP[pr, pc]).ravel(),
                        dAx=np.asarray(dA[ar, ac]).ravel(), **d)
    for k, key in zip(OUT, ("x", "y", "s")):
        assert np.allclose(got[key], ref[k], rtol=1e-9, atol=1e-10), (key, got[key], ref[k])
    model.update(q=np.array([1.0, 1.5]))
    with pytest.raises(ValueError):
        model.derivative(dq=np.ones(2))


def _gradcheck_problem():
    # test_gpu_adjoint's gradcheck problem: strictly complementary, x = (1/2, 1/2, 0), the bound on x3 active at a
    # multiplier of 2, P diagonal so that gradcheck can move each stored entry alone
    P = sp.csc_matrix(np.diag([2.0, 1.0, 1.5]))
    A = sp.csc_matrix(np.vstack([np.ones((1, 3)), -np.eye(3)]))
    q = np.array([-1.0, -0.5, 2.0])
    b = np.array([1.0, 0.0, 0.0, 0.0])
    sets = [cosmo_b200.ZeroSet(1), cosmo_b200.Nonnegatives(3)]
    return P, q, A, b, sets


def test_forward_mode_gradcheck_of_solve_qp():
    torch = pytest.importorskip("torch")
    from cosmo_b200.autograd import solve_qp
    P, q, A, b, sets = _gradcheck_problem()
    eng = _engine(P, q, A, b, sets, "DeviceLdlKKTSolver", 0)
    t = lambda a: torch.tensor(a, dtype=torch.float64, device="cuda", requires_grad=True)
    inputs = (t(P.data), t(q), t(A.data), t(b))
    assert torch.autograd.gradcheck(lambda Px, q_, Ax, b_: solve_qp(eng, Px, q_, Ax, b_), inputs, eps=1e-6, atol=1e-6,
                                    rtol=1e-5, check_forward_ad=True, check_backward_ad=False)


@pytest.mark.parametrize("kkt", PLUGINS)
def test_a_forward_ad_dual_equals_engine_derivative_bit_for_bit(kkt):
    torch = pytest.importorskip("torch")
    import torch.autograd.forward_ad as fwAD
    from cosmo_b200.autograd import solve_qp
    P, q, A, b, sets = _gradcheck_problem()
    eng = _engine(P, q, A, b, sets, kkt, 0)
    rng = np.random.default_rng(9)
    t = lambda a: torch.tensor(a, dtype=torch.float64, device="cuda")
    prim = [t(P.data), t(q), t(A.data), t(b)]
    tang = [t(rng.standard_normal(len(p))) for p in prim]
    with fwAD.dual_level():
        outs = solve_qp(eng, *(fwAD.make_dual(p, d) for p, d in zip(prim, tang)))
        jvp = [fwAD.unpack_dual(o).tangent.clone() for o in outs]
    torch.cuda.synchronize()
    (dx, dy, ds), st = eng.derivative(tang[0].cpu().numpy(), tang[1].cpu().numpy(), tang[2].cpu().numpy(),
                                      tang[3].cpu().numpy())
    assert st["status"] == 1
    for a, b_ in zip(jvp, (dx, dy, ds)):
        assert np.array_equal(_bits(a), _bits(b_))
