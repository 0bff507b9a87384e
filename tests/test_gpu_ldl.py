"""GPU tests of the direct LDL' KKT plugin (kkt_solver = COSMO_B200_KKT_LDL, Settings(kkt_solver="DeviceLdlKKTSolver")):
the plugin-level solve against the oracle's direct KKT solve, iterate trajectories and solve-level parity with the
oracle's direct runs, the reference behaviours that need an exact KKT solve, errors and reproducibility."""
import numpy as np
import pytest
import scipy.sparse as sp

import cosmo_b200
from cosmo_b200 import engine as E
from oracle import cosmo_oracle as O
from oracle.bridge import to_oracle_cones
from tests import golden_problems as G
from tests.gpu_helpers import U32, _engine

pytestmark = pytest.mark.gpu

LDL = "DeviceLdlKKTSolver"
F32 = np.float32


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


def _solve_mine(builder, dtype=np.float64, **kw):
    P, q, cons = builder()
    model = cosmo_b200.Model(dtype=dtype)
    cosmo_b200.assemble(model, P, q, _to_mine(cons), cosmo_b200.Settings(kkt_solver=LDL, **kw))
    return cosmo_b200.optimize(model), model


def _oracle_kw(kw):
    kw = dict(kw)
    if kw.pop("accelerator", "EmptyAccelerator") == "AndersonAccelerator":
        kw["accelerator"] = "anderson"
    return kw


def _solve_oracle(builder, scale_q=1.0, scale_b=1.0, **kw):
    P, q, cons = builder()
    Pm, qm, A, b, cones = O.assemble(P, q, cons)
    return O.solve(Pm, qm * scale_q, A, b * scale_b, cones, O.Settings(**_oracle_kw(kw)))     # kkt_solver = "direct"


def _kkt(P, A, sigma, rho):
    n = P.shape[0]
    return sp.bmat([[sp.csc_matrix(P) + sigma * sp.identity(n), A.T], [A, -sp.diags(1.0 / rho)]], format="csc")


# ---------------------------------------------------------------------------
# plugin level
# ---------------------------------------------------------------------------
def _check_solves(eng, P, A, sigma, rng, bw_bar, fw_factor, dtype):
    rho = eng.rho_vec().astype(np.float64)
    Pd, Ad = (P.astype(np.float32).astype(np.float64), A.astype(np.float32).astype(np.float64)) if dtype == F32 else (P, A)
    K = _kkt(Pd, Ad, float(np.asarray(sigma, dtype=dtype)), rho)
    Kd = K.toarray()
    kappa = np.linalg.cond(Kd)
    direct = O.DirectKKT(Pd, Ad, float(np.asarray(sigma, dtype=dtype)), rho)
    worst_bw = worst_fw = 0.0
    for _ in range(3):
        r = rng.standard_normal(K.shape[0]).astype(dtype).astype(np.float64)
        x, inner = eng.kkt_solve(r)
        x = x.astype(np.float64)
        assert inner == 0
        bw = np.linalg.norm(r - K @ x, np.inf) / (np.linalg.norm(Kd, np.inf) * np.linalg.norm(x, np.inf) + np.linalg.norm(r, np.inf))
        ref = direct.solve(r)
        fw = np.linalg.norm(x - ref) / np.linalg.norm(ref)
        worst_bw, worst_fw = max(worst_bw, bw), max(worst_fw, fw / kappa)
    assert worst_bw <= bw_bar and worst_fw <= fw_factor, (worst_bw, worst_fw, kappa)
    return worst_bw, worst_fw


@pytest.mark.parametrize("dtype", [np.float64, F32], ids=["fp64", "fp32"])
@pytest.mark.parametrize("kind", ["qp", "portfolio", "psd"])
def test_kkt_solve_matches_the_direct_solve_after_rho_and_sigma_changes(kind, dtype):
    rng = np.random.default_rng(11)
    if kind == "qp":
        P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(300, 500, 0.02, seed=3)
    elif kind == "portfolio":
        P, q, A, b, sets = cosmo_b200.problems.portfolio_socp(200, 20, seed=1)
    else:
        P, q, A, b, sets = cosmo_b200.problems.closest_correlation_sdp(N=20)
    P, A = sp.csc_matrix(P), sp.csc_matrix(A)
    bw_bar, fw_bar = (1e-13, 1e-14) if dtype == np.float64 else (64 * U32, 64 * U32)
    eng = _engine(P, q, A, b, sets, dtype=dtype, kkt_solver=LDL, scaling=0)
    st0 = eng.ldl_stats()
    assert st0["N"] == P.shape[0] + A.shape[0] and st0["factorizations"] == 1 and st0["nnz_L"] > 0 and st0["levels"] >= 1
    _check_solves(eng, P, A, 1e-6, rng, bw_bar, fw_bar, dtype)
    assert eng.ldl_stats()["factorizations"] == 1 and eng.ldl_stats()["solve_nodes"] >= 2
    # update_rho! -> refactor! before the next solve
    new_rho = rng.uniform(0.01, 100.0, A.shape[0])
    eng.update_rho(new_rho, 3.0)
    _check_solves(eng, P, A, 1e-6, rng, bw_bar, fw_bar, dtype)
    assert eng.ldl_stats()["factorizations"] == 2
    # a sigma change through update_settings
    st = cosmo_b200.Settings(kkt_solver=LDL, scaling=0, sigma=1e-2).to_struct()
    eng.update_settings(st)
    _check_solves(eng, P, A, 1e-2, rng, bw_bar, fw_bar, dtype)
    assert eng.ldl_stats()["factorizations"] == 3
    eng.close()


# ---------------------------------------------------------------------------
# iterate trajectories against the oracle's direct run
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("scaling", [0, 10])
def test_w_trajectory_matches_the_oracle_direct_run(scaling):
    P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(40, 70, 0.15, seed=7)
    for k in (5, 45, 90):
        model = cosmo_b200.Model()       # scaling != 0: equilibrated on the device
        model.set(P, q, A, b, sets, cosmo_b200.Settings(kkt_solver=LDL, scaling=scaling, max_iter=k, eps_abs=1e-14,
                                                        eps_rel=1e-14, adaptive_rho_tolerance=1.5))
        res = model.optimize()
        ref = O.solve(P, q, A, b, to_oracle_cones(sets), O.Settings(scaling=scaling, max_iter=k, eps_abs=1e-14, eps_rel=1e-14,
                                                                    adaptive_rho_tolerance=1.5))
        w = model.engine.w()
        rel = np.linalg.norm(w - ref.w) / np.linalg.norm(ref.w)
        assert res.iter == ref.iter == k and rel <= 1e-9, (k, rel)
        assert np.allclose(res.info.rho_updates, ref.info.rho_updates, rtol=1e-9)
        if k == 90:
            assert len(ref.info.rho_updates) >= 2          # the trajectory crosses rho adaptations
        assert res.kkt_inner_iterations == 0


def test_c5_w_parity_with_the_oracle_direct_run():
    from cosmo_b200 import chordal
    rows, cols, wts = cosmo_b200.problems.banded_random_graph(2000, 3.0, 20, seed=1)
    P, q, A, b, sets = cosmo_b200.problems.maxcut_dual_sdp(2000, rows, cols, wts)
    P2, q2, A2, b2, sets2, info = chordal.decompose(P, q, A, b, sets, merge="parent_child")
    k = 20
    st = cosmo_b200.Settings(kkt_solver=LDL, scaling=0, adaptive_rho=False, max_iter=k, eps_abs=0.0, eps_rel=0.0)
    model = cosmo_b200.Model()
    model.set(P2, q2, A2, b2, sets2, st)
    model.optimize()
    ref = O.solve(P2, q2, A2, b2, to_oracle_cones(sets2), O.Settings(scaling=0, adaptive_rho=False, max_iter=k, eps_abs=0.0, eps_rel=0.0))
    w = model.engine.w()
    rel = float(np.max(np.abs(w - ref.w)) / np.max(np.abs(ref.w)))
    assert rel <= 1e-10, rel


# ---------------------------------------------------------------------------
# solve level: the reference's literal problems, statuses and iteration counts of the oracle's direct run
# ---------------------------------------------------------------------------
LITERAL = [("g1_qp_nonneg", G.g1_qp_nonneg, {}), ("g1_qp_box", G.g1_qp_box, {}), ("g2_box_feasible", G.g2_box_feasible, {}),
           ("g2_box_primal_infeasible_1", G.g2_box_primal_infeasible_1, {}),
           ("g2_box_primal_infeasible_2", G.g2_box_primal_infeasible_2, {}),
           ("g2_box_dual_infeasible", G.g2_box_dual_infeasible, dict(check_infeasibility=20, scaling=0)),
           ("g3_hs21", G.g3_hs21, {}), ("g4_small_sdp", G.g4_small_sdp, dict(check_termination=1)),
           ("g5_sigma_max_lmi", G.g5_sigma_max_lmi, {}), ("g6_chordal_sdp", G.g6_chordal_sdp, {}),
           ("g11_iteration_limit", G.g11_iteration_limit, dict(max_iter=2)), ("g12_lp", G.g12_lp, dict(eps_abs=1e-4, eps_rel=1e-5)),
           ("g13_lovasz_petersen", G.g13_lovasz_petersen, dict(eps_abs=1e-6, eps_rel=1e-6)),
           ("g17_complex_least_eigenvalue", G.g17_complex_least_eigenvalue, {})] + \
          [(g[0], g[1], g[5]) for g in G.G15_G16] + [(name, bld, {}) for name, bld, _ in G.INFEASIBILITY_PROBLEMS]


# On the infeasible and slowly converging problems the iteration at which a check first succeeds is not a continuous
# function of the data (tests/test_gpu_infeasibility.py): the oracle is run on the data and on q (1 +- 1e-15),
# b (1 +- 1e-15), b (1 +- 2e-15).  Where all seven runs agree, the engine must reproduce status and iteration count
# exactly; elsewhere its status must be one the oracle reaches.  Measured on one H100 80GB HBM3: g1_qp_nonneg with
# Anderson moves between 28 and 31 iterations in the oracle, primal_infeasible_3 between 163 and 172.
_PERTURB = ((1.0, 1.0), (1 + 1e-15, 1.0), (1 - 1e-15, 1.0), (1.0, 1 + 1e-15), (1.0, 1 - 1e-15), (1.0, 1 + 2e-15), (1.0, 1 - 2e-15))


# Measured on one H100 80GB HBM3: with default scaling the engine certifies primal_infeasible_3 at iteration 121, the
# oracle at 161 in all seven runs.  At scaling 0 both stop at 161.  The iterates agree to 1.7e-10 after 10 iterations
# and drift apart to 1.5e-4 by the first rho adaptation at iteration 40 (rho 19.68 against 19.80), so the two
# trajectories split on rounding.  The CG plugin splits the same way (561 against 641 at scaling 0).  The data
# perturbations of the protocol move the oracle by less than the difference between the two eigensolvers of the PSD
# projection, so the oracle looks stable here.
_PI3_DRIFT = pytest.mark.xfail(strict=True, reason="known: Primal_infeasible at 121 iterations against the oracle's 161 "
                                                   "(stable under the seven perturbations); the trajectories split on "
                                                   "rounding before the first rho adaptation")


def _literal_cases():
    out = []
    for name, builder, kw in LITERAL:
        for acc in ("EmptyAccelerator", "AndersonAccelerator"):
            if acc == "AndersonAccelerator" and name.endswith("large_psd"):
                continue          # the oracle does not decide it with acceleration (tests/golden_problems.py)
            marks = [_PI3_DRIFT] if (name, acc) == ("primal_infeasible_3", "EmptyAccelerator") else []
            out.append(pytest.param(builder, dict(kw, accelerator=acc), id="%s-%s" % (name, acc[:-11]), marks=marks))
    return out


@pytest.mark.parametrize("builder,kw", _literal_cases())
def test_literal_problems_match_the_oracle_direct_run(builder, kw):
    res, _ = _solve_mine(builder, **kw)
    ref = _solve_oracle(builder, **kw)
    if (res.status, res.iter) == (ref.status, ref.iter):
        if ref.status == "Solved":
            assert abs(res.obj_val - ref.obj_val) <= 1e-6 * max(1.0, abs(ref.obj_val)), (res.obj_val, ref.obj_val)
        return
    refs = [(ref.status, ref.iter)] + [(r.status, r.iter) for r in
                                       (_solve_oracle(builder, scale_q=sq, scale_b=sb, **kw) for sq, sb in _PERTURB[1:])]
    assert len(set(refs)) > 1 and res.status in {st for st, _ in refs}, (res.status, res.iter, refs)


# ---------------------------------------------------------------------------
# reference behaviours that need the exact KKT solve
# ---------------------------------------------------------------------------
def test_g6_at_eps_1e7_is_solved_in_75_iterations():
    from cosmo_b200 import chordal
    P, q, cons = G.g6_chordal_sdp()
    Pm, qm, A0, b0, cones0 = O.assemble(P, q, cons)
    P2, q2, A2, b2, sets2, info = chordal.decompose(Pm, qm, A0, b0, [cosmo_b200.PsdConeTriangle(45)], merge="none")
    model = cosmo_b200.Model()
    model.set(P2, q2, A2, b2, sets2, cosmo_b200.Settings(kkt_solver=LDL, eps_abs=1e-7, eps_rel=1e-7))
    res = model.optimize()
    ref = O.solve(P2, q2, A2, b2, to_oracle_cones(sets2), O.Settings(eps_abs=1e-7, eps_rel=1e-7))
    assert res.status == ref.status == "Solved" and res.iter == ref.iter == 75, (res.status, res.iter, ref.iter)
    assert abs(res.obj_val - ref.obj_val) < 1e-8


def test_warm_started_resolve_takes_fewer_iterations():
    """test/UnitTests/simple.jl:93-124 with the direct solver: res2.iter < res1.iter"""
    P, q, cons = G.g1_qp_nonneg()
    m1 = cosmo_b200.Model()
    cosmo_b200.assemble(m1, P, q, _to_mine(cons), cosmo_b200.Settings(kkt_solver=LDL, check_termination=1))
    r1 = m1.optimize()
    m2 = cosmo_b200.Model()
    cosmo_b200.assemble(m2, P, q, _to_mine(cons), cosmo_b200.Settings(kkt_solver=LDL, check_termination=1))
    rng = np.random.default_rng(0)
    m2.warm_start_primal(r1.x + 0.01 * rng.random(2))
    m2.warm_start_dual(r1.y + 0.01 * rng.random(6))
    r2 = m2.optimize()
    assert r1.status == r2.status == "Solved" and r2.iter < r1.iter, (r1.iter, r2.iter)


def test_complex_psd_solve_takes_the_oracle_direct_count():
    from tests.gpu_helpers import _hermitian_ws
    rng = np.random.default_rng(77)
    Nc = 60
    ws, H = _hermitian_ws(Nc, rng, "wigner")
    sets = [cosmo_b200.ComplexPsdConeTriangle(Nc * Nc)]
    eye = O.extract_upper_triangle_complex(np.eye(Nc, dtype=complex), np.sqrt(2.0))
    A = sp.csc_matrix(eye.reshape(-1, 1))
    P = sp.csc_matrix((1, 1))
    q = np.array([-1.0])
    model = cosmo_b200.Model()
    model.set(P, q, A, ws, sets, cosmo_b200.Settings(kkt_solver=LDL))
    res = model.optimize()
    ref = O.solve(P, q, A, ws, to_oracle_cones(sets), O.Settings())
    assert res.status == "Solved" == ref.status and res.iter == ref.iter, (res.iter, ref.iter)
    assert np.allclose(res.info.rho_updates, ref.info.rho_updates, rtol=1e-6)
    assert abs(res.x[0] - np.linalg.eigvalsh(H)[0]) < 1e-3 * abs(ref.x[0])


@pytest.mark.parametrize("scaling", [0, 10])
def test_obj_true_tol_1e8_is_reached(scaling):
    res, _ = _solve_mine(G.g1_qp_nonneg, scaling=scaling, obj_true=1.88, obj_true_tol=1e-8)
    ref = _solve_oracle(G.g1_qp_nonneg, scaling=scaling, obj_true=1.88, obj_true_tol=1e-8)
    assert res.status == "Solved" == ref.status and abs(res.obj_val - 1.88) <= 1e-8 and res.iter == ref.iter, \
        (res.status, res.iter, ref.iter, res.obj_val - 1.88)


# Measured on one H100 80GB HBM3: the direct solve does not rescue these fp32 runs.  pow_feasible ends at
# Max_iter_reached after 5000 iterations with r_prim 8.2e-2, r_dual 1.6e-2; pow_primal_infeasible at Max_iter_reached
# after 5000 with r_prim 0.63, r_dual 216.5; closest correlation N = 40 at Max_iter_reached after 5000 with
# r_prim 3.8e-6, r_dual 1.3e-4.  So the stall is not the inexact CG solve the fp32 xfails of test_gpu_float32.py
# name as the reason.
_FP32_POW = pytest.mark.xfail(strict=True, reason="known: Max_iter_reached after 5000 iterations in fp32 with the device "
                                                  "LDL' solve too (reference: solved in Float32 with QDLDL); not fixed yet")


@_FP32_POW
@pytest.mark.parametrize("name", ["pow_feasible", "pow_primal_infeasible"])
def test_float32_power_cone_problems_reach_the_reference_status(name):
    g = [g for g in G.G15_G16 if g[0] == name][0]
    res, _ = _solve_mine(g[1], dtype=F32, **g[5])
    assert res.status == g[2], (name, res.status, res.iter, res.info.r_prim, res.info.r_dual)
    if g[3] is not None:
        assert abs(res.obj_val - g[3]) < g[4], (name, res.obj_val)


@pytest.mark.xfail(strict=True, reason="known: Max_iter_reached after 5000 iterations in fp32 with the device LDL' solve "
                                      "(r_prim 3.8e-6, r_dual 1.3e-4; closestcorr.jl expects :Solved); not fixed yet")
def test_float32_closest_correlation_is_solved():
    N = 40
    P, q, A, b, sets = cosmo_b200.problems.closest_correlation_sdp(N=N, seed=12345)
    model = cosmo_b200.Model(dtype=F32)
    model.set(P, q, A, b, sets, cosmo_b200.Settings(kkt_solver=LDL))
    res = model.optimize()
    assert res.status == "Solved", (res.status, res.iter, res.info.r_prim, res.info.r_dual)
    X = np.zeros((N, N))
    iu = np.triu_indices(N)
    order = np.lexsort((iu[0], iu[1]))
    r, c = iu[0][order], iu[1][order]
    X[r, c] = np.where(r == c, res.x, res.x / np.sqrt(2))
    X = X + np.triu(X, 1).T
    assert np.max(np.abs(np.diag(X) - 1.0)) < 1e-3 and np.linalg.eigvalsh(X).min() > -1e-3


# ---------------------------------------------------------------------------
# errors and reproducibility
# ---------------------------------------------------------------------------
def test_nonconvex_objective_is_refused():
    n, m = 5, 3
    A = sp.csc_matrix(np.random.default_rng(1).standard_normal((m, n)))
    with pytest.raises(E.EngineError) as ei:
        _engine(-sp.identity(n, format="csc"), np.zeros(n), A, np.zeros(m), [cosmo_b200.Nonnegatives(m)], kkt_solver=LDL, scaling=0)
    assert ei.value.code == E.ERR_INVALID and "Objective function is not convex." in str(ei.value)


def test_sharded_handles_are_refused():
    P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(30, 40, 0.2, seed=0)
    eng = _engine(P, q, A, b, sets, kkt_solver=LDL)
    with pytest.raises(E.EngineError) as ei:
        eng.comm_init(2, 0, bytes(128))
    assert ei.value.code == E.ERR_UNSUPPORTED
    eng.close()


def test_two_fresh_handles_are_bitwise_equal():
    P, q, A, b, sets = cosmo_b200.problems.portfolio_socp(400, 40, seed=2)
    outs = []
    for _ in range(2):
        model = cosmo_b200.Model()
        model.set(P, q, A, b, sets, cosmo_b200.Settings(kkt_solver=LDL, max_iter=300))
        r = model.optimize()
        outs.append((r.x, r.s, r.y, r.iter))
    assert outs[0][3] == outs[1][3]
    for a, b_ in zip(outs[0][:3], outs[1][:3]):
        assert np.array_equal(a, b_)
