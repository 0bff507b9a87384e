"""GPU tests of the supernodal LDL' KKT plugin (kkt_solver = COSMO_B200_KKT_LDL_SUPERNODAL,
Settings(kkt_solver="DeviceSupernodalKKTSolver") or "MKLPardisoKKTSolver"): the plugin-level solve against the oracle's
direct KKT solve and against the simplicial plugin, both factorisation paths, iterate trajectories and solve-level parity
with the oracle's direct runs, the reference behaviours that need an exact KKT solve, errors and state."""
import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

import cosmo_b200
from cosmo_b200 import engine as E
from oracle import cosmo_oracle as O
from oracle.bridge import to_oracle_cones
from tests import golden_problems as G
from tests.gpu_helpers import U32, _engine
from tests.test_gpu_ldl import LITERAL, _PERTURB, _check_solves, _kkt, _oracle_kw, _to_mine

pytestmark = pytest.mark.gpu

SN = "DeviceSupernodalKKTSolver"
LDL = "DeviceLdlKKTSolver"
F32 = np.float32


def _solve_mine(builder, **kw):
    P, q, cons = builder()
    model = cosmo_b200.Model()
    cosmo_b200.assemble(model, P, q, _to_mine(cons), cosmo_b200.Settings(kkt_solver=SN, **kw))
    return cosmo_b200.optimize(model)


def _solve_oracle(builder, scale_q=1.0, scale_b=1.0, **kw):
    P, q, cons = builder()
    Pm, qm, A, b, cones = O.assemble(P, q, cons)
    return O.solve(Pm, qm * scale_q, A, b * scale_b, cones, O.Settings(**_oracle_kw(kw)))


def _problem(kind):
    if kind == "qp":
        return cosmo_b200.problems.random_sparse_qp(300, 500, 0.02, seed=3)
    if kind == "portfolio":
        return cosmo_b200.problems.portfolio_socp(200, 20, seed=1)
    return cosmo_b200.problems.closest_correlation_sdp(N=20)


# ---------------------------------------------------------------------------
# plugin level
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.float64, F32], ids=["fp64", "fp32"])
@pytest.mark.parametrize("kind", ["qp", "portfolio", "psd"])
def test_kkt_solve_matches_the_direct_solve_after_rho_and_sigma_changes(kind, dtype):
    rng = np.random.default_rng(11)
    P, q, A, b, sets = _problem(kind)
    P, A = sp.csc_matrix(P), sp.csc_matrix(A)
    bw_bar, fw_bar = (1e-13, 1e-14) if dtype == np.float64 else (64 * U32, 64 * U32)
    eng = _engine(P, q, A, b, sets, dtype=dtype, kkt_solver=SN, scaling=0)
    st0 = eng.ldl_stats()
    assert st0["N"] == P.shape[0] + A.shape[0] and st0["factorizations"] == 1 and st0["nnz_L"] > 0 and st0["levels"] >= 1
    sn = eng.ldl_sn_stats()
    assert sn["supernodes"] >= 1 and sn["small_path"] + sn["tiled_path"] == sn["supernodes"]
    _check_solves(eng, P, A, 1e-6, rng, bw_bar, fw_bar, dtype)
    assert eng.ldl_stats()["factorizations"] == 1 and eng.ldl_stats()["solve_nodes"] >= 2
    eng.update_rho(rng.uniform(0.01, 100.0, A.shape[0]), 3.0)
    _check_solves(eng, P, A, 1e-6, rng, bw_bar, fw_bar, dtype)
    assert eng.ldl_stats()["factorizations"] == 2
    eng.update_settings(cosmo_b200.Settings(kkt_solver=SN, scaling=0, sigma=1e-2).to_struct())
    _check_solves(eng, P, A, 1e-2, rng, bw_bar, fw_bar, dtype)
    assert eng.ldl_stats()["factorizations"] == 3
    eng.close()


def _kappa1(K):
    """1-norm condition number of the sparse K, the inverse's norm estimated through its LU"""
    lu = spla.splu(sp.csc_matrix(K))
    inv = spla.LinearOperator(K.shape, matvec=lu.solve, rmatvec=lambda v: lu.solve(v, trans="T"), dtype=np.float64)
    return spla.norm(K, 1) * spla.onenormest(inv)


def _agree_with_simplicial(P, q, A, b, sets, rng, dtype=np.float64):
    """the same right-hand sides through codes 4 and 3 on the same data: backward error of code 4 and the difference"""
    e4 = _engine(P, q, A, b, sets, dtype=dtype, kkt_solver=SN, scaling=0)
    e3 = _engine(P, q, A, b, sets, dtype=dtype, kkt_solver=LDL, scaling=0)
    K = _kkt(P, A, 1e-6, e4.rho_vec().astype(np.float64))
    kappa = _kappa1(K)
    Kinf = spla.norm(K, np.inf)
    worst_bw = worst_fw = 0.0
    for _ in range(3):
        r = rng.standard_normal(K.shape[0])
        x4, inner = e4.kkt_solve(r)
        x3, _ = e3.kkt_solve(r)
        assert inner == 0
        bw = np.linalg.norm(r - K @ x4, np.inf) / (Kinf * np.linalg.norm(x4, np.inf) + np.linalg.norm(r, np.inf))
        worst_bw = max(worst_bw, bw)
        worst_fw = max(worst_fw, np.linalg.norm(x4 - x3) / np.linalg.norm(x3) / kappa)
    return e4, e3, worst_bw, worst_fw


def test_tiled_path_on_the_portfolio_trailing_block():
    """portfolio n = 2000, k = 200: the 203-wide trailing supernode takes the tiled path, the rest the small path"""
    rng = np.random.default_rng(5)
    P, q, A, b, sets = cosmo_b200.problems.portfolio_socp(2000, 200, seed=1)
    P, A = sp.csc_matrix(P), sp.csc_matrix(A)
    e4, e3, bw, fw = _agree_with_simplicial(P, q, A, b, sets, rng)
    st = e4.ldl_sn_stats()
    assert st["small_path"] > 0 and st["tiled_path"] >= 1 and st["max_width"] == 203, st
    assert bw <= 1e-13 and fw <= 1e-14, (bw, fw)
    e4.close()
    e3.close()


def test_wide_tiled_supernode_is_reproducible_and_meets_the_backward_bar():
    """random QP n = 10 000, m = 20 000: a 9663-wide trailing supernode.  Its block columns launch sn_panel_kernel with
    up to 75 CTAs after the diagonal block's own launch, and its diagonal solves are wider than the solves' shared
    memory (8192 fp64 values), so they run in place.  A refactorisation with the same rho must give bitwise the same
    solve; the backward error is checked against the sparse K (the forward bar needs a condition number that a dense
    9663-wide fill makes too costly to estimate here)."""
    rng = np.random.default_rng(9)
    P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(10_000, 20_000, 0.0013, seed=0)
    P, A = sp.csc_matrix(P), sp.csc_matrix(A)
    eng = _engine(P, q, A, b, sets, kkt_solver=SN, scaling=0)
    st = eng.ldl_sn_stats()
    assert st["tiled_path"] >= 1 and st["max_width"] > 65536 // 8, st
    rho = eng.rho_vec().astype(np.float64)
    K = _kkt(P, A, 1e-6, rho)
    Kinf = spla.norm(K, np.inf)
    rs = [rng.standard_normal(K.shape[0]) for _ in range(2)]
    xs = []
    for r in rs:
        x, inner = eng.kkt_solve(r)
        bw = np.linalg.norm(r - K @ x, np.inf) / (Kinf * np.linalg.norm(x, np.inf) + np.linalg.norm(r, np.inf))
        assert inner == 0 and bw <= 1e-13, bw
        xs.append(x)
    eng.update_rho(rho, 0.1)                      # the same rho: a refactorisation that must reproduce the factor
    assert eng.ldl_stats()["factorizations"] == 1
    for r, x in zip(rs, xs):
        assert np.array_equal(eng.kkt_solve(r)[0], x)
    assert eng.ldl_stats()["factorizations"] == 2
    eng.close()


@pytest.mark.parametrize("kind", ["qp", "portfolio", "psd"])
def test_solves_agree_with_the_simplicial_plugin(kind):
    rng = np.random.default_rng(21)
    P, q, A, b, sets = _problem(kind)
    e4, e3, bw, fw = _agree_with_simplicial(sp.csc_matrix(P), q, sp.csc_matrix(A), b, sets, rng)
    assert bw <= 1e-13 and fw <= 1e-14, (bw, fw)
    e4.close()
    e3.close()


# ---------------------------------------------------------------------------
# iterate trajectories against the oracle's direct run
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("scaling", [0, 10])
def test_w_trajectory_matches_the_oracle_direct_run(scaling):
    P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(40, 70, 0.15, seed=7)
    for k in (5, 45, 90):
        model = cosmo_b200.Model()
        model.set(P, q, A, b, sets, cosmo_b200.Settings(kkt_solver=SN, scaling=scaling, max_iter=k, eps_abs=1e-14,
                                                        eps_rel=1e-14, adaptive_rho_tolerance=1.5))
        res = model.optimize()
        ref = O.solve(P, q, A, b, to_oracle_cones(sets), O.Settings(scaling=scaling, max_iter=k, eps_abs=1e-14, eps_rel=1e-14,
                                                                    adaptive_rho_tolerance=1.5))
        rel = np.linalg.norm(model.engine.w() - ref.w) / np.linalg.norm(ref.w)
        assert res.iter == ref.iter == k and rel <= 1e-9, (k, rel)
        assert np.allclose(res.info.rho_updates, ref.info.rho_updates, rtol=1e-9)
        if k == 90:
            assert len(ref.info.rho_updates) >= 2
        assert res.kkt_inner_iterations == 0


def test_c5_w_parity_with_the_oracle_direct_run():
    from cosmo_b200 import chordal
    rows, cols, wts = cosmo_b200.problems.banded_random_graph(2000, 3.0, 20, seed=1)
    P, q, A, b, sets = cosmo_b200.problems.maxcut_dual_sdp(2000, rows, cols, wts)
    P2, q2, A2, b2, sets2, info = chordal.decompose(P, q, A, b, sets, merge="parent_child")
    k = 20
    model = cosmo_b200.Model()
    model.set(P2, q2, A2, b2, sets2, cosmo_b200.Settings(kkt_solver=SN, scaling=0, adaptive_rho=False, max_iter=k,
                                                         eps_abs=0.0, eps_rel=0.0))
    model.optimize()
    ref = O.solve(P2, q2, A2, b2, to_oracle_cones(sets2), O.Settings(scaling=0, adaptive_rho=False, max_iter=k, eps_abs=0.0, eps_rel=0.0))
    w = model.engine.w()
    rel = float(np.max(np.abs(w - ref.w)) / np.max(np.abs(ref.w)))
    assert rel <= 1e-10, rel


# ---------------------------------------------------------------------------
# solve level: the literal problems under the seven-run protocol of test_gpu_ldl.py
# ---------------------------------------------------------------------------
# Measured on one H100 80GB HBM3: on these three cases the plugin reaches the oracle's status at another iteration,
# and all seven oracle runs agree on theirs.  The relative w distances after k iterations (same settings, max_iter = k)
# show rounding-size differences that the iteration amplifies, not a different KKT solve:
# * g1_qp_box with Anderson: w within 7.8e-16 of the oracle and 2.5e-15 of the simplicial plugin through k = 20, and
#   within 4.6e-16 of the oracle's at the stop; the termination test passes at 27 here and at 25 in the oracle.
# * primal_infeasible_3_soc: all three runs differ by 3e-8 to 1e-7 from k = 1 on (the simplicial plugin and the oracle
#   too); the first rho adaptation at 40 gives 21.10 here, 19.42 in the simplicial plugin, 20.69 in the oracle, and
#   the runs then certify at 121 here, 161 in both others.  On primal_infeasible_3 the roles swap: this plugin
#   certifies at 161 with the oracle, the simplicial plugin at 121 (its own xfail in test_gpu_ldl.py).
# * dual_infeasible_1 with Anderson: w within 3.3e-14 of the simplicial plugin at k = 5 (both 1.3e-6 from the oracle),
#   4.3e-5 at k = 10 and 0.8 at k = 40, while the simplicial plugin is 4.4e-5 from the oracle at k = 10; the oracle and
#   the simplicial plugin certify at 48, this run adapts rho to 5.3e-3 at 60 and certifies at 208.
_SPLIT = {("g1_qp_box", "AndersonAccelerator"): "Solved at 27 iterations against the oracle's 25",
          ("primal_infeasible_3_soc", "EmptyAccelerator"): "Primal_infeasible at 121 iterations against the oracle's 161",
          ("dual_infeasible_1", "AndersonAccelerator"): "Dual_infeasible at 208 iterations against the oracle's 48"}


def _literal_cases():
    out = []
    for name, builder, kw in LITERAL:
        for acc in ("EmptyAccelerator", "AndersonAccelerator"):
            if acc == "AndersonAccelerator" and name.endswith("large_psd"):
                continue
            why = _SPLIT.get((name, acc))
            marks = [pytest.mark.xfail(strict=True, reason="known: %s (stable under the seven perturbations); the "
                                                           "trajectories split on rounding" % why)] if why else []
            out.append(pytest.param(builder, dict(kw, accelerator=acc), id="%s-%s" % (name, acc[:-11]), marks=marks))
    return out


@pytest.mark.parametrize("builder,kw", _literal_cases())
def test_literal_problems_match_the_oracle_direct_run(builder, kw):
    res = _solve_mine(builder, **kw)
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
    model.set(P2, q2, A2, b2, sets2, cosmo_b200.Settings(kkt_solver=SN, eps_abs=1e-7, eps_rel=1e-7))
    res = model.optimize()
    ref = O.solve(P2, q2, A2, b2, to_oracle_cones(sets2), O.Settings(eps_abs=1e-7, eps_rel=1e-7))
    assert res.status == ref.status == "Solved" and res.iter == ref.iter == 75, (res.status, res.iter, ref.iter)
    assert abs(res.obj_val - ref.obj_val) < 1e-8


def test_warm_started_resolve_takes_fewer_iterations():
    P, q, cons = G.g1_qp_nonneg()
    m1 = cosmo_b200.Model()
    cosmo_b200.assemble(m1, P, q, _to_mine(cons), cosmo_b200.Settings(kkt_solver="MKLPardisoKKTSolver", check_termination=1))
    r1 = m1.optimize()
    m2 = cosmo_b200.Model()
    cosmo_b200.assemble(m2, P, q, _to_mine(cons), cosmo_b200.Settings(kkt_solver="MKLPardisoKKTSolver", check_termination=1))
    rng = np.random.default_rng(0)
    m2.warm_start_primal(r1.x + 0.01 * rng.random(2))
    m2.warm_start_dual(r1.y + 0.01 * rng.random(6))
    r2 = m2.optimize()
    assert r1.status == r2.status == "Solved" and r2.iter < r1.iter, (r1.iter, r2.iter)


# ---------------------------------------------------------------------------
# errors and state
# ---------------------------------------------------------------------------
def test_nonconvex_objective_is_refused():
    n, m = 5, 3
    A = sp.csc_matrix(np.random.default_rng(1).standard_normal((m, n)))
    with pytest.raises(E.EngineError) as ei:
        _engine(-sp.identity(n, format="csc"), np.zeros(n), A, np.zeros(m), [cosmo_b200.Nonnegatives(m)], kkt_solver=SN, scaling=0)
    assert ei.value.code == E.ERR_INVALID and "Objective function is not convex." in str(ei.value)


def test_sharded_handles_are_refused():
    P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(30, 40, 0.2, seed=0)
    eng = _engine(P, q, A, b, sets, kkt_solver=SN)
    with pytest.raises(E.EngineError) as ei:
        eng.comm_init(2, 0, bytes(128))
    assert ei.value.code == E.ERR_UNSUPPORTED
    eng.close()


def test_two_fresh_handles_are_bitwise_equal():
    P, q, A, b, sets = cosmo_b200.problems.portfolio_socp(400, 40, seed=2)
    outs = []
    for _ in range(2):
        model = cosmo_b200.Model()
        model.set(P, q, A, b, sets, cosmo_b200.Settings(kkt_solver=SN, max_iter=300))
        r = model.optimize()
        outs.append((r.x, r.s, r.y, r.iter))
    assert outs[0][3] == outs[1][3]
    for a, b_ in zip(outs[0][:3], outs[1][:3]):
        assert np.array_equal(a, b_)


def test_update_matrices_refactors_and_meets_the_bars():
    rng = np.random.default_rng(3)
    P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(300, 500, 0.02, seed=3)
    P, A = sp.csc_matrix(P), sp.csc_matrix(A)
    model = cosmo_b200.Model()
    model.set(P, q, A, b, sets, cosmo_b200.Settings(kkt_solver=SN, scaling=0, max_iter=50))
    model.optimize()
    eng = model.engine
    n_fact = eng.ldl_stats()["factorizations"]
    P2, A2 = P.copy(), A.copy()
    P2.data = P2.data * 1.5
    A2.data = A2.data * (1.0 + 0.1 * rng.standard_normal(A2.nnz))
    model.update(P=P2, A=A2)
    assert model.engine is eng and eng.ldl_stats()["factorizations"] == n_fact + 1
    _check_solves(eng, P2, A2, 1e-6, rng, 1e-13, 1e-14, np.float64)


def test_decompose_works_with_the_plugin():
    rows, cols, wts = cosmo_b200.problems.banded_random_graph(200, 3.0, 10, seed=1)
    P, q, A, b, sets = cosmo_b200.problems.maxcut_dual_sdp(200, rows, cols, wts)
    res = {}
    for solver in (SN, LDL):
        model = cosmo_b200.Model()
        model.set(P, q, A, b, sets, cosmo_b200.Settings(kkt_solver=solver, decompose=True, merge_strategy="ParentChildMerge"))
        res[solver] = model.optimize()
    assert res[SN].status == res[LDL].status == "Solved"
    assert abs(res[SN].obj_val - res[LDL].obj_val) <= 1e-6 * max(1.0, abs(res[LDL].obj_val))


def test_update_settings_switches_between_the_direct_plugins():
    rng = np.random.default_rng(8)
    P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(300, 500, 0.02, seed=3)
    P, A = sp.csc_matrix(P), sp.csc_matrix(A)
    eng = _engine(P, q, A, b, sets, kkt_solver=LDL, scaling=0)
    r = rng.standard_normal(P.shape[0] + A.shape[0])
    x3, _ = eng.kkt_solve(r)
    assert eng.ldl_sn_stats()["supernodes"] == 0
    eng.update_settings(cosmo_b200.Settings(kkt_solver=SN, scaling=0).to_struct())
    x4, inner = eng.kkt_solve(r)
    assert inner == 0 and eng.ldl_sn_stats()["supernodes"] > 0 and eng.ldl_stats()["factorizations"] == 1
    eng.update_settings(cosmo_b200.Settings(kkt_solver=LDL, scaling=0).to_struct())
    x3b, _ = eng.kkt_solve(r)
    assert np.array_equal(x3, x3b)
    assert np.linalg.norm(x4 - x3) <= 1e-10 * np.linalg.norm(x3)
    eng.update_settings(cosmo_b200.Settings(kkt_solver=SN, scaling=0).to_struct())
    _check_solves(eng, P, A, 1e-6, rng, 1e-13, 1e-14, np.float64)
    eng.close()
