"""GPU tests of the derivatives of polished solutions (cosmo_b200_adjoint, Engine.adjoint, Model.adjoint,
autograd.solve_qp): the engine against the restatement of tests/adjoint_reference.py on the engine's own polished point,
directional finite differences through full engine re-solves, dependent active rows, host and device buffers,
determinism and untouched state, refusals and statuses, and torch.autograd.gradcheck.  Both direct plugins throughout;
scaling 0 and 10 unless stated."""
import numpy as np
import pytest
import scipy.sparse as sp

import cosmo_b200
from cosmo_b200 import engine as E
from cosmo_b200 import model as M
from oracle import cosmo_oracle as O
from oracle.bridge import to_oracle_cones
from tests import adjoint_reference as AR
from tests import golden_problems as G
from tests import polish_reference as R
from tests.gpu_helpers import U32
from tests.test_gpu_polish import _qp_with_zero_block

pytestmark = pytest.mark.gpu

PLUGINS = ["DeviceLdlKKTSolver", "DeviceSupernodalKKTSolver"]
SCALINGS = [0, 10]
KEYS = ("dq", "db", "dPx", "dAx", "dl", "du")


def _engine(P, q, A, b, sets, kkt, scaling, dtype=np.float64, **kw):
    st = cosmo_b200.Settings(kkt_solver=kkt, scaling=scaling, **kw).to_struct()
    return E.Engine(P, q, A, b, [M.set_tuple(S) for S in sets], st, dtype=dtype, equilibrate=scaling != 0)


def _problem(n, seed):
    """random_sparse_qp (Nonnegatives + Box rows) with n / 20 ZeroSet rows through its feasible point (the polish tests'
    problem)."""
    P, q, A, b, sets = _qp_with_zero_block(n, 2 * n, 20.0 / n, seed, n // 20)
    return sp.csc_matrix(P), q, sp.csc_matrix(A), b, sets


def _polish(eng):
    x, y, s, st = eng.polish(x=np.empty(eng.n), y=np.empty(eng.m), s=np.empty(eng.m))
    assert st["status"] == 1, st
    return x, y, s, st


def _grads(n, m, seed=5):
    rng = np.random.default_rng(seed)
    return rng.standard_normal(n), rng.standard_normal(m), rng.standard_normal(m)


def _bits(a):
    a = a.cpu().numpy() if hasattr(a, "cpu") else a
    return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


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
    gx, gy, gs = _grads(eng.n, eng.m)
    got, st = eng.adjoint(gx, gy, gs)
    assert st["status"] == pst["status"]
    if dtype == np.float32 and pst["status"] == 0:   # fp32 polishes may be rejected: then NaN, not gradients
        assert all(np.all(np.isnan(g)) for g in got)
        return
    assert st["status"] == 1
    # the restatement on the engine's scaled data and polished point, with the engine's classification
    D, Ev, c = eng.scaling()
    D, Ev = np.asarray(D, dtype=float), np.asarray(Ev, dtype=float)
    Ps = sp.csc_matrix(c * (sp.diags(D) @ P @ sp.diags(D)))
    As = sp.csc_matrix(sp.diags(Ev) @ A @ sp.diags(D))
    cls, l, u = R.row_classes(to_oracle_cones(sets))
    kind, _ = R.classify(cls, Ev * l, Ev * u, out.s.astype(float), out.mu.astype(float))
    active = kind != R.INACTIVE
    assert st["n_active"] == int(active.sum())
    ref = AR.adjoint(Ps, As, cls, kind, x / D, c * y / Ev, gx, gy, gs, D=D, E=Ev, c=c)
    K = AR.kkt_matrix(Ps, As, kind)
    assert K.shape[0] <= 3000
    kappa = np.linalg.cond(K)
    if dtype == np.float64:
        # normwise backward error of the engine's (u, v) in the scaled system
        ut = -got[0] / (c * D)
        vt = np.where(active, got[1] / Ev - gs / Ev, 0.0)
        rhs = np.concatenate([D * gx - As.T @ (gs / Ev), (Ev * gy / c)[active]])
        z = np.concatenate([ut, vt[active]])
        eta = np.abs(K @ z - rhs).max() / (np.abs(K).sum(axis=1).max() * np.abs(z).max() + np.abs(rhs).max())
        assert eta <= 1e-13, eta
        assert st["refine_residual"] <= 1e-10 * (1 + np.abs(rhs).max())
    tol = (1e-14 if dtype == np.float64 else 64 * U32) * kappa
    for k, g in zip(KEYS, got):
        want = ref[k]
        assert np.linalg.norm(g - want) <= tol * np.linalg.norm(want), (k, np.linalg.norm(g - want) / np.linalg.norm(want), kappa)
    # dl, du vanish off Box rows, and on Box rows that are not active
    box = cls == R.BOX
    assert np.all(got[4][~box] == 0.0) and np.all(got[5][~box] == 0.0)
    assert np.all(got[4][box & ~active] == 0.0) and np.all(got[5][box & ~active] == 0.0)


# ---------------------------------------------------------------------------
# 2. directional finite differences through full engine re-solves
# ---------------------------------------------------------------------------
def _fd_problem():
    P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(40, 80, 0.2, seed=11)
    return sp.csc_matrix(P), q, sp.csc_matrix(A), b, list(sets)


def _resolve(eng, Px, q, Ax, b):
    eng.update_matrices(Px, Ax, q, b)
    assert eng.solve().status == "Solved"
    return _polish(eng)


@pytest.mark.parametrize("scaling", SCALINGS)
@pytest.mark.parametrize("kkt", PLUGINS)
def test_directional_finite_differences(kkt, scaling):
    P, q, A, b, sets = _fd_problem()
    eng = _engine(P, q, A, b, sets, kkt, scaling)
    x, y, s, st0 = _resolve(eng, P.data, q, A.data, b)
    gx, gy, gs = _grads(eng.n, eng.m, 9)
    (dq, db, dPx, dAx, dl, du), st = eng.adjoint(gx, gy, gs)
    assert st["status"] == 1 and st["n_weak"] == 0
    rng = np.random.default_rng(4)
    pr, pc = P.indices, np.repeat(np.arange(P.shape[1]), np.diff(P.indptr))
    Msym = sp.csc_matrix((rng.standard_normal(P.nnz), P.indices, P.indptr), shape=P.shape)
    eP = np.asarray((Msym + Msym.T)[pr, pc]).ravel()
    dirs = {"q": (0 * P.data, rng.standard_normal(eng.n), 0 * A.data, 0 * b),
            "b": (0 * P.data, 0 * q, 0 * A.data, rng.standard_normal(eng.m)),
            "P": (eP, 0 * q, 0 * A.data, 0 * b),
            "A": (0 * P.data, 0 * q, rng.standard_normal(A.nnz), 0 * b)}
    eps = 1e-6
    for what, (eP_, eq, eA, eb) in dirs.items():
        ana = dPx @ eP_ + dq @ eq + dAx @ eA + db @ eb
        vals = []
        for sgn in (1.0, -1.0):
            xs, ys, ss, _ = _resolve(eng, P.data + sgn * eps * eP_, q + sgn * eps * eq, A.data + sgn * eps * eA,
                                     b + sgn * eps * eb)
            vals.append(gx @ xs + gy @ ys + gs @ ss)
        fd = (vals[0] - vals[1]) / (2 * eps)
        assert abs(fd - ana) <= 1e-6 * max(abs(ana), 1e-3), (what, fd, ana)


# ---------------------------------------------------------------------------
# 3. dependent active rows: G1's equality written as two inequalities
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("scaling", SCALINGS)
@pytest.mark.parametrize("kkt", PLUGINS)
def test_dependent_rows_of_g1(kkt, scaling):
    Pd, qd, cons = G.g1_qp_nonneg()
    P, q, A, b, cones = O.assemble(Pd, qd, cons)
    P, A = sp.csc_matrix(P), sp.csc_matrix(A)
    sets = [cosmo_b200.Nonnegatives(A.shape[0])]
    eng = _engine(P, q, A, b, sets, kkt, scaling)
    x, y, s, _ = _resolve(eng, P.data, q, A.data, b)
    assert np.abs(x - G.G1_X).max() <= 1e-9
    gx, gs = np.array([1.0, -2.0]), np.linspace(-1.0, 1.0, A.shape[0])
    (dq, db, dPx, dAx, dl, du), st = eng.adjoint(gx, None, gs)
    assert st["status"] == 1
    eps = 1e-6
    rng = np.random.default_rng(2)
    # rows 0 and 3 are x1 + x2 <= 1 and -(x1 + x2) <= -1: moving b along (e0 - e3) moves the equality
    eb = np.zeros(A.shape[0]); eb[0], eb[3] = 1.0, -1.0
    pr, pc = P.indices, np.repeat(np.arange(2), np.diff(P.indptr))
    Msym = sp.csc_matrix((rng.standard_normal(P.nnz), P.indices, P.indptr), shape=P.shape)
    dirs = {"q": (0 * P.data, rng.standard_normal(2), 0 * b), "P": (np.asarray((Msym + Msym.T)[pr, pc]).ravel(), 0 * q, 0 * b),
            "b": (0 * P.data, 0 * q, eb)}
    for what, (eP, eq, eb_) in dirs.items():
        ana = dPx @ eP + dq @ eq + db @ eb_
        vals = []
        for sgn in (1.0, -1.0):
            xs, _, ss, _ = _resolve(eng, P.data + sgn * eps * eP, q + sgn * eps * eq, A.data, b + sgn * eps * eb_)
            vals.append(gx @ xs + gs @ ss)
        fd = (vals[0] - vals[1]) / (2 * eps)
        assert abs(fd - ana) <= 1e-6 * max(abs(ana), 1e-3), (what, fd, ana)


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
    gx, gy, gs = _grads(eng.n, eng.m)
    host1, st1 = eng.adjoint(gx, gy, gs)
    host2, st2 = eng.adjoint(gx, gy, gs)
    cuda = lambda a: torch.from_numpy(a).cuda()
    outs = [torch.empty(len(h), dtype=torch.float64, device="cuda") for h in host1]
    dev, st3 = eng.adjoint(cuda(gx), cuda(gy), cuda(gs), dq=outs[0], db=outs[1], dPx=outs[2], dAx=outs[3], dl=outs[4],
                           du=outs[5])
    torch.cuda.synchronize()
    for a, b_, c_ in zip(host1, host2, dev):
        assert np.array_equal(_bits(a), _bits(b_)) and np.array_equal(_bits(a), _bits(c_))
    assert st1 == st2 == st3


@pytest.mark.parametrize("kkt", PLUGINS)
def test_the_next_solve_is_the_solve_of_a_twin_that_never_ran_the_adjoint(kkt):
    P, q, A, b, sets = _problem(200, 6)
    engs = [_engine(P, q, A, b, sets, kkt, 10) for _ in range(2)]
    for e in engs:
        assert e.solve().status == "Solved"
        _polish(e)
    gx, gy, gs = _grads(engs[0].n, engs[0].m)
    engs[0].adjoint(gx, gy, gs)
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
def _code(fn):
    with pytest.raises(E.EngineError) as e:
        fn()
    return e.value.code


@pytest.mark.parametrize("kkt", PLUGINS)
def test_no_polish_record_after_solve_update_or_reset(kkt):
    P, q, A, b, sets = _problem(200, 7)
    eng = _engine(P, q, A, b, sets, kkt, 0)
    g = _grads(eng.n, eng.m)
    assert _code(lambda: eng.adjoint(*g)) == E.ERR_INVALID           # never polished
    for breaker in (lambda: eng.solve(), lambda: eng.update_qb(q=q), lambda: eng.reset(),
                    lambda: eng.update_matrices(P.data, A.data, q, b)):
        assert eng.solve().status == "Solved"
        _polish(eng)
        eng.adjoint(*g)
        breaker()
        assert _code(lambda: eng.adjoint(*g)) == E.ERR_INVALID


@pytest.mark.parametrize("kkt", ["CGIndirectKKTSolver", "MINRESIndirectKKTSolver"])
def test_indirect_plugins_are_refused(kkt):
    P, q, A, b, sets = _problem(200, 7)
    eng = _engine(P, q, A, b, sets, kkt, 0)
    eng.solve()
    assert _code(lambda: eng.adjoint(*_grads(eng.n, eng.m))) == E.ERR_UNSUPPORTED


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
    outs, st = eng.adjoint(np.ones(n))
    assert st["status"] == -1 and st["n_active"] == 0 and np.isnan(st["refine_residual"])
    assert all(np.all(np.isnan(o)) for o in outs)


# ---------------------------------------------------------------------------
# 6. Model.adjoint and torch.autograd
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("kkt", PLUGINS)
def test_model_adjoint_in_update_coordinates(kkt):
    P, q, cons = G.g1_qp_box()
    model = cosmo_b200.Model()
    cosmo_b200.assemble(model, P, q, [cosmo_b200.Constraint(c.A, c.b, cosmo_b200.Box(c.convex_set.l, c.convex_set.u))
                                      for c in cons], cosmo_b200.Settings(kkt_solver=kkt, polish=True))
    res = model.optimize()
    assert res.polish == "Polished"
    g = model.adjoint(dx=np.array([1.0, 0.0]))
    assert g["stats"]["status"] == 1
    assert g["P"].shape == model.P0.shape and np.array_equal(g["P"].indices, model.P0.indices)
    assert g["A"].shape == model.A0.shape and np.array_equal(g["A"].indptr, model.A0.indptr)
    # x1 = 0.3 is fixed by the equality row x1 + x2 = 1 and the upper bound x2 <= 0.7: dx1 / dq = 0
    assert np.abs(g["q"]).max() <= 1e-12
    # set! form: s = (x1 + x2, x1, x2) in [l, u]; x2 sits at its upper bound 0.7 and x1 = 1 - x2, so d x1 / d u_3 = -1
    assert abs(g["u"][2] + 1.0) <= 1e-9 and g["u"][0] == g["l"][0]
    model.update(q=np.array([1.0, 1.5]))
    with pytest.raises(ValueError):
        model.adjoint(dx=np.ones(2))


def test_gradcheck_of_solve_qp():
    torch = pytest.importorskip("torch")
    from cosmo_b200.autograd import solve_qp
    # strictly complementary: x = argmin 1/2 x'Px + q'x over x1 + x2 + x3 = 1, x >= 0 is (1/2, 1/2, 0) with the bound
    # on x3 active at a multiplier of 2.  P is diagonal, so that gradcheck can move each stored entry alone.
    P = sp.csc_matrix(np.diag([2.0, 1.0, 1.5]))
    A = sp.csc_matrix(np.vstack([np.ones((1, 3)), -np.eye(3)]))
    q = np.array([-1.0, -0.5, 2.0])
    b = np.array([1.0, 0.0, 0.0, 0.0])
    sets = [cosmo_b200.ZeroSet(1), cosmo_b200.Nonnegatives(3)]
    eng = _engine(P, q, A, b, sets, "DeviceLdlKKTSolver", 0)
    t = lambda a: torch.tensor(a, dtype=torch.float64, device="cuda", requires_grad=True)
    inputs = (t(P.data), t(q), t(A.data), t(b))
    x, y, s = (t.detach() for t in solve_qp(eng, *inputs))
    assert abs(float(x.sum()) - 1.0) <= 1e-12 and abs(float(x[2])) <= 1e-12 and abs(float(x[0]) - 0.5) <= 1e-12
    assert torch.autograd.gradcheck(lambda Px, q_, Ax, b_: solve_qp(eng, Px, q_, Ax, b_), inputs, eps=1e-6, atol=1e-6,
                                    rtol=1e-5)
