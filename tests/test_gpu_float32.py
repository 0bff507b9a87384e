"""Model{Float32} on the device: every kernel of Engine<float> against a float64 reference of the same operation.

The data are drawn in fp64 and rounded to fp32; the fp64 oracle gets exactly those rounded values (`_round32`), so every
difference below is the kernel's own rounding.  Bars are stated in units of u32 = 2^-24 times the reduction length and
the natural scale of the operation (|M| |v| for products, |X|_F for projections)."""
import numpy as np
import pytest
import scipy.sparse as sp

import cosmo_b200
from cosmo_b200 import engine as E
from oracle import cosmo_oracle as O
from oracle.bridge import to_oracle_cones
from tests import golden_problems as G
from tests.gpu_helpers import U32, _engine, _hermitian_ws, _oracle_project, _project_engine, _psd_test_matrix, _round32, _tuples
from tests.test_gpu_parity import _ragged_matrix, _to_mine

pytestmark = pytest.mark.gpu
F32 = np.float32


def _csc32(M):
    M = sp.csc_matrix(M, dtype=np.float64)
    M.data = _round32(M.data)
    return M


def _spmv_bar(M, v):
    """per row: (k_row + 2) u32 (|M| |v|)_row, k_row = entries of the row"""
    k = np.diff(sp.csr_matrix(M).indptr)
    return (k + 2) * U32 * (abs(M) @ np.abs(v)) + 1e-300


def _check_spmv(eng, which, M, v):
    got = eng.spmv(which, v.astype(F32)).astype(np.float64)
    ref = M @ v
    assert got.dtype == np.float64 and np.all(np.abs(got - ref) <= _spmv_bar(M, v)), (which, float(np.max(np.abs(got - ref) / _spmv_bar(M, v))))


# ---------------------------------------------------------------------------
# SpMV: A x, A' y, P x
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("m,n", [(1, 1), (17, 9), (64, 257), (300, 131), (1000, 515)])
def test_spmv_ragged_float32(m, n):
    rng = np.random.default_rng(m * 1000 + n)
    A = _csc32(_ragged_matrix(rng, m, n))
    B = _ragged_matrix(rng, n, n)
    P = _csc32(B + B.T)
    eng = _engine(P, np.zeros(n), A, np.zeros(m), [cosmo_b200.Nonnegatives(m)], dtype=F32)
    x, y = _round32(rng.standard_normal(n)), _round32(rng.standard_normal(m))
    for which, M, v in ((0, A, x), (1, A.T, y), (2, P, x)):
        _check_spmv(eng, which, M, v)


@pytest.mark.parametrize("density", [0.002, 0.02, 0.2])
def test_spmv_lane_variants_float32(density):
    rng = np.random.default_rng(5)
    m, n = 3000, 1500
    A = _csc32(sp.random(m, n, density=density, random_state=rng, data_rvs=rng.standard_normal, format="csc"))
    B = sp.random(n, n, density=density, random_state=rng, data_rvs=rng.standard_normal, format="csc")
    P = _csc32(B + B.T)
    eng = _engine(P, np.zeros(n), A, np.zeros(m), [cosmo_b200.Nonnegatives(m)], dtype=F32)
    x, y = _round32(rng.standard_normal(n)), _round32(rng.standard_normal(m))
    for which, M, v in ((0, A, x), (1, A.T, y), (2, P, x)):
        _check_spmv(eng, which, M, v)


# fp32 windows hold 204800 / 4 = 51200 columns: 1, 2 and 3 windows; >= 24 entries per row segment so they are built
@pytest.mark.parametrize("m,n,per_row", [(400, 40000, 100), (400, 60000, 100), (2000, 120000, 150)])
def test_spmv_windowed_float32(m, n, per_row):
    rng = np.random.default_rng(m + n)
    rows = np.repeat(np.arange(m), per_row)
    cols = rng.integers(0, n, size=m * per_row)
    cols[:per_row] = rng.integers(0, 50, size=per_row)                      # row 0 lives in window 0 only
    cols[per_row:2 * per_row] = rng.integers(n - 50, n, size=per_row)       # row 1 lives in the last window only
    A = _csc32(sp.csc_matrix((rng.standard_normal(m * per_row), (rows, cols)), shape=(m, n)))
    P = sp.identity(n, format="csc")
    eng = _engine(P, np.zeros(n), A, np.zeros(m), [cosmo_b200.Nonnegatives(m)], dtype=F32, scaling=0)
    x, y = _round32(rng.standard_normal(n)), _round32(rng.standard_normal(m))
    for which, M, v in ((0, A, x), (1, A.T, y)):
        _check_spmv(eng, which, M, v)


# ---------------------------------------------------------------------------
# clamp cones and SOC
# ---------------------------------------------------------------------------
def test_clamp_cones_bit_exact_float32():
    rng = np.random.default_rng(3)
    l = _round32(rng.standard_normal(40) - 1.0)
    u = _round32(l + rng.random(40) * 2)
    l[3], u[5] = -np.inf, np.inf
    l[7] = u[7]
    l[9], u[9] = -np.inf, np.inf
    sets = [cosmo_b200.ZeroSet(9), cosmo_b200.Nonnegatives(33), cosmo_b200.Box(l, u)]
    eng = _project_engine(sets, dtype=F32)
    ws = (rng.standard_normal(82) * 3).astype(F32)
    ws[10] = np.nan                          # nonnegatives: NaN propagates through max(x, 0)
    ws[9 + 33 + 5] = 1e30
    got = eng.project(ws)
    want = np.concatenate([np.zeros(9, F32), np.where(np.isnan(ws[9:42]), ws[9:42], np.maximum(ws[9:42], F32(0))),
                           np.minimum(np.maximum(ws[42:], l.astype(F32)), u.astype(F32))])
    assert got.dtype == F32 and np.array_equal(got, want, equal_nan=True)


@pytest.mark.parametrize("dims", [(4, 4, 4), (1, 2, 9, 20000)])
def test_soc_float32(dims):
    rng = np.random.default_rng(len(dims))
    sets = [cosmo_b200.SecondOrderCone(d) for d in dims]
    if dims == (4, 4, 4):   # inside the cone, inside the polar cone, the generic case (test_soc_branches)
        ws = np.array([5.0, 1, 1, 1, -5.0, 1, 1, 1, 0.5, 1, 2, 2])
    else:
        ws = _round32(rng.standard_normal(sum(dims)))
    eng = _project_engine(sets, dtype=F32)
    got = eng.project(ws.astype(F32)).astype(np.float64)
    ref = _oracle_project(ws, sets)
    off = 0
    for d in dims:
        seg = slice(off, off + d)
        bar = 4.0 * (d + 2) * U32 * np.linalg.norm(ws[seg])
        assert np.linalg.norm(got[seg] - ref[seg]) <= bar, (d, float(np.linalg.norm(got[seg] - ref[seg]) / np.linalg.norm(ws[seg])))
        off += d


# ---------------------------------------------------------------------------
# exponential / power cones and their duals
# ---------------------------------------------------------------------------
@pytest.mark.xfail(strict=True, reason="known engine bug: for some points the fp32 search returns a point of the cone farther "
                                      "from v than the fp64 projection, e.g. Exp v = (-16.8, 0.95, -17.6) -> (-16.8, 0, 0) where "
                                      "(-16.8, 0.95, 2e-8) is feasible and closer: a failed search, not rounding; max error "
                                      "0.083 (1 + |v|); not fixed yet")
def test_project_exp_pow_cones_float32():
    # the fp32 engine searches in T = float with the same tolerances; the bar is the fp32 one of the issue: 1e-4 (1 + |v|)
    rng = np.random.default_rng(5)
    sets, pts = [], []
    special_exp = [(1.0, 2.0, 10.0), (-3.0, 0.0, 1.0), (1.0, -2.0, -3.0), (0.0, -1.0, -2.0), (-2.0, -3.0, 4.0), (-2.0, -3.0, -4.0)]
    for v in special_exp:
        sets.append(cosmo_b200.ExponentialCone()); pts.append(v)
    for v in [(2.0, 3.0, 1.0), (-1.0, -2.0, 0.5), (3.0, -2.0, 1e-9), (-3.0, 2.0, 0.0)]:
        sets.append(cosmo_b200.PowerCone(0.3)); pts.append(v)
    for i in range(400):
        a = 0.1 + 0.85 * rng.random()
        for S in (cosmo_b200.ExponentialCone(), cosmo_b200.DualExponentialCone(), cosmo_b200.PowerCone(a), cosmo_b200.DualPowerCone(a)):
            sets.append(S)
            pts.append(-25.0 + 50.0 * rng.random(3))
    ws = _round32(np.concatenate([np.asarray(v, dtype=float) for v in pts]))
    eng = _project_engine(sets, dtype=F32)
    got = eng.project(ws.astype(F32)).astype(np.float64)
    ref = _oracle_project(ws, sets)
    err = np.abs(got - ref).reshape(-1, 3).max(axis=1)
    scale = 1.0 + np.abs(ws).reshape(-1, 3).max(axis=1)
    print("MEAS exp/pow fp32 max err / (1 + |v|) = %.3e" % float((err / scale).max()))
    assert np.all(err <= 1e-4 * scale), float((err / scale).max())
    cones = to_oracle_cones(sets)
    mine = np.array([O.in_cone(got[3 * k:3 * k + 3], c, 1e-4) for k, c in enumerate(cones)])
    theirs = np.array([O.in_cone(ref[3 * k:3 * k + 3], c, 1e-4) for k, c in enumerate(cones)])
    print("MEAS exp/pow fp32 verdict mismatches = %d" % int(np.sum(mine != theirs)))
    assert np.sum(mine != theirs) <= 8 and mine.mean() > 0.99


# ---------------------------------------------------------------------------
# PSD: small-cone batch, tensor-core path, block Jacobi, Hermitian
# ---------------------------------------------------------------------------
def _check_psd32(eng, ws, sets, tag, level=None):
    """|Pi_gpu - Pi|_F / |X|_F no worse than the reference's fp32 route (the oracle fed the fp32 input, as ssyevr would be)
    and <= 1e-5; Pi = fp64 projection of the rounded input.  With `level`, only |Pi_gpu - Pi|_F / |X|_F <= level: the
    accuracy the fp32 Jacobi paths reach today, kept as a regression bar (the full bar is test_psd_jacobi_float32_full_bar)"""
    got = eng.project(ws.astype(F32)).astype(np.float64)
    truth = _oracle_project(ws, sets)
    ref32 = ws.astype(F32)
    O.project(ref32, to_oracle_cones(sets))
    off, errs = 0, []
    for S in sets:
        seg = slice(off, off + S.dim)
        nrm = np.linalg.norm(ws[seg]) + 1e-300
        errs.append((S.dim, np.linalg.norm(got[seg] - truth[seg]) / nrm, np.linalg.norm(ref32[seg].astype(np.float64) - truth[seg]) / nrm))
        off += S.dim
    print("MEAS psd32 %s worst gpu=%.2e worst ratio gpu/ref32=%.2f" % (tag, max(e[1] for e in errs), max(e[1] / e[2] for e in errs)))
    for dim, e_gpu, e_ref in errs:
        if level is not None:
            assert e_gpu <= level, (tag, dim, e_gpu, level)
        else:
            assert e_gpu <= max(2.0 * e_ref, 2e-7) and e_gpu <= 1e-5, (tag, dim, e_gpu, e_ref)


def _small_batch32(rng):
    sizes = list(range(1, 97))
    sets = [cosmo_b200.PsdConeTriangle(N * (N + 1) // 2) for N in sizes] + [cosmo_b200.PsdCone(N * N) for N in (3, 50, 96)]
    parts = [G._svec(_psd_test_matrix("wigner", N, rng)) for N in sizes]
    parts += [_psd_test_matrix("shifted", N, rng).reshape(-1, order="F") for N in (3, 50, 96)]
    return sets, _round32(np.concatenate(parts))


def test_project_psd_small_batch_float32():
    rng = np.random.default_rng(96)
    sets, ws = _small_batch32(rng)
    eng = _project_engine(sets, dtype=F32)
    _check_psd32(eng, ws, sets, "small", level=6e-5)          # measured worst over N = 1..96: 2.85e-5
    assert eng.psd_stats()["tc_projections"] == 0


@pytest.mark.parametrize("kind", ["wigner", "rank_deficient", "shifted", "zero", "admm_like", "graded"])
@pytest.mark.parametrize("N", [97, 200, 385])
def test_project_psd_tensor_core_path_float32_kinds(kind, N):
    rng = np.random.default_rng(2000 + N)
    X = _psd_test_matrix(kind, N, rng)
    sets = [cosmo_b200.PsdConeTriangle(N * (N + 1) // 2), cosmo_b200.PsdCone(N * N)]
    ws = _round32(np.concatenate([G._svec(X), X.reshape(-1, order="F")]))
    eng = _project_engine(sets, dtype=F32)
    _check_psd32(eng, ws, sets, kind)
    st = eng.psd_stats()
    assert st["tc_projections"] == 2 and st["tc_fallbacks"] == 0, st


@pytest.mark.parametrize("env", [("COSMO_B200_PSD_TC", "0"), ("COSMO_B200_TC_MAX_STEPS", "3")])
@pytest.mark.parametrize("N", [150, 257])
def test_project_psd_block_jacobi_float32(N, env, monkeypatch):
    monkeypatch.setenv(*env)
    rng = np.random.default_rng(3000 + N)
    X = _psd_test_matrix("wigner", N, rng)
    sets = [cosmo_b200.PsdConeTriangle(N * (N + 1) // 2)]
    ws = _round32(G._svec(X))
    eng = _project_engine(sets, dtype=F32)
    _check_psd32(eng, ws, sets, "block_jacobi", level=3e-4)   # measured: 5.8e-5 (N = 150), 1.37e-4 (N = 257)
    st = eng.psd_stats()
    assert st["tc_projections"] == 0 and st["tc_fallbacks"] == (1 if env[0] == "COSMO_B200_TC_MAX_STEPS" else 0), st


@pytest.mark.parametrize("Nc", [60, 100, 12])
def test_complex_psd_float32(Nc):
    rng = np.random.default_rng(4000 + Nc)
    ws, _ = _hermitian_ws(Nc, rng, "shifted")
    ws = _round32(ws)
    sets = [cosmo_b200.ComplexPsdConeTriangle(Nc * Nc)]
    eng = _project_engine(sets, dtype=F32)
    _check_psd32(eng, ws, sets, "complex", level=5e-6 if 2 * Nc <= 96 else None)   # small path, Nc = 12: measured 2.1e-6
    st = eng.psd_stats()
    assert st["tc_projections"] == (1 if 2 * Nc > 96 else 0) and st["tc_fallbacks"] == 0, st


@pytest.mark.xfail(strict=True, reason="known gap: the fp32 Jacobi paths miss the fp32 bar (worst 2.85e-5 small batch, 2.1e-6 "
                                      "complex Nc = 12 against 1.9e-8 for the oracle, 5.8e-5 / 1.37e-4 block Jacobi at N = 150 / "
                                      "257).  Neither a 64x smaller rotation threshold nor fp64 accumulation of the "
                                      "reconstruction changed these numbers; the cause is not found yet")
@pytest.mark.parametrize("path", ["small", "complex_small", "block_jacobi"])
def test_psd_jacobi_float32_full_bar(path, monkeypatch):
    rng = np.random.default_rng(96)
    if path == "small":
        sets, ws = _small_batch32(rng)
    elif path == "complex_small":
        sets, ws = [cosmo_b200.ComplexPsdConeTriangle(12 * 12)], _round32(_hermitian_ws(12, np.random.default_rng(4012), "shifted")[0])
    else:
        monkeypatch.setenv("COSMO_B200_PSD_TC", "0")
        N = 150
        sets, ws = [cosmo_b200.PsdConeTriangle(N * (N + 1) // 2)], _round32(G._svec(_psd_test_matrix("wigner", N, np.random.default_rng(3150))))
    _check_psd32(_project_engine(sets, dtype=F32), ws, sets, path)


# ---------------------------------------------------------------------------
# residuals, KKT solves, device Ruiz
# ---------------------------------------------------------------------------
def _small_qp32(seed=0, n=40, m=70):
    P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(n, m, 0.15, seed=seed)
    return _csc32(P), _round32(q), _csc32(A), _round32(b), sets


def test_residuals_float32():
    P, q, A, b, sets = _small_qp32(seed=4)
    m, n = A.shape
    eng = _engine(P, q, A, b, sets, dtype=F32, scaling=0)
    rng = np.random.default_rng(8)
    x, s, mu = _round32(rng.standard_normal(n)), _round32(rng.standard_normal(m)), _round32(rng.standard_normal(m))
    got = eng.residuals(x.astype(F32), s.astype(F32), mu.astype(F32))
    kA = np.diff(sp.csr_matrix(A).indptr).max()
    kD = np.diff(sp.csr_matrix(P).indptr).max() + np.diff(sp.csr_matrix(A.T).indptr).max() + 1
    ws = O.Workspace(P, q, A, b, to_oracle_cones(sets), O.Settings(scaling=0))
    ws.setup()
    ws.xv, ws.s, ws.mu = x, s, mu
    rp, rd = ws.calculate_residuals(False)             # |A x + s - b|_inf, |P x + q - A' mu|_inf
    sp_ = np.max(abs(A) @ np.abs(x) + np.abs(s) + np.abs(b))
    sd = np.max(abs(P) @ np.abs(x) + abs(A.T) @ np.abs(mu) + np.abs(q))
    assert abs(got[0] - rp) <= (kA + 2) * U32 * sp_ and abs(got[1] - rd) <= (kD + 2) * U32 * sd, (got[:2], rp, rd)
    cost = 0.5 * x @ (P @ x) + q @ x
    assert abs(got[4] - cost) <= (kD + n + 2) * U32 * (0.5 * np.abs(x) @ (abs(P) @ np.abs(x)) + np.abs(q) @ np.abs(x))


@pytest.mark.parametrize("name,kind", [("CG", "cg"), ("MINRESIndirectKKTSolver", "minres"),
                                       ("IndirectReducedKKTSolver:MINRES", "minres_reduced")])
def test_kkt_solve_float32(name, kind):
    # the fp32 solvers against the fp64 oracle solver of the same name on exactly the same (fp32-rounded) P, A, rho and
    # right-hand sides, with the same tolerance schedule and warm starts: both stop at the same inexact point up to
    # rounding, which the conditioning kappa of the system they iterate on amplifies.  Bar: 8 sqrt(n + m) kappa u32
    # relative.  After the schedule has tightened the solution must
    # also be that of the KKT system.
    P, q, A, b, sets = _small_qp32(seed=3, n=41, m=70)
    m, n = A.shape
    kw = {} if name == "CG" else dict(kkt_solver=name)
    eng = _engine(P, q, A, b, sets, dtype=F32, scaling=0, **kw)
    rho = eng.rho_vec().astype(np.float64)
    sigma = 1e-6
    oracle = O.make_kkt_solver(kind, P, A, sigma, rho.copy(), O.Settings())
    direct = O.DirectKKT(P, A, sigma, rho)
    K = (P + sigma * sp.identity(n) + A.T @ sp.diags(rho) @ A).toarray()
    if kind == "minres":
        K = np.block([[K - A.T @ sp.diags(rho) @ A, A.T.toarray()], [A.toarray(), -np.diag(1.0 / rho)]])
    kappa = np.linalg.cond(K)
    bar = 8.0 * np.sqrt(n + m) * kappa * U32
    rng = np.random.default_rng(2)
    worst = 0.0
    for k in range(6):
        rhs = _round32(rng.standard_normal(n + m))
        sol, inner = eng.kkt_solve(rhs.astype(F32))
        ref = oracle.solve(rhs)
        err = np.linalg.norm(sol.astype(np.float64) - ref) / np.linalg.norm(ref)
        worst = max(worst, err / (kappa * U32))
        assert abs(inner - oracle.inner_iterations[-1]) <= 1, (name, k, inner, oracle.inner_iterations[-1])
        assert err <= bar, (name, k, err, bar)
    for k in range(40):                  # the schedule tightens; both keep warm-starting from their own previous solution
        sol, _ = eng.kkt_solve(rhs.astype(F32))
        ref = oracle.solve(rhs)
        err = np.linalg.norm(sol.astype(np.float64) - ref) / np.linalg.norm(ref)
        worst = max(worst, err / (kappa * U32))
        assert err <= bar, (name, 6 + k, err, bar)
    # and the solution is that of the KKT system (1e-3 after 46 solves, as in test_minres_kkt_solve_matches_oracle)
    exact = direct.solve(rhs)
    err_exact = np.linalg.norm(sol.astype(np.float64) - exact)
    # measured worst over the 46 solves: err / (kappa u32) = 0.60 (CG), 0.46 (MINRES), 0.69 (reduced MINRES)
    print("MEAS kkt fp32 %s kappa=%.1f worst err/(kappa u32)=%.2f vs direct %.1e" % (name, kappa, worst, err_exact))
    assert err_exact <= 1e-3 * (1 + np.linalg.norm(sol)), (name, err_exact)


@pytest.mark.parametrize("prob", ["qp_box", "socp", "sdp"])
def test_device_ruiz_float32(prob):
    pr = cosmo_b200.problems
    if prob == "qp_box":
        P, q, A, b, sets = pr.random_sparse_qp(300, 500, 0.05, seed=0)
    elif prob == "socp":
        P, q, A, b, sets = pr.portfolio_socp(n=200, k=20, seed=2)
    else:
        P, q, A, b, sets = pr.closest_correlation_sdp(N=20, seed=7)
    P, q, A, b = _csc32(P), _round32(q), _csc32(A), _round32(b)
    st = cosmo_b200.Settings()
    eng = E.Engine(P, q, A, b, _tuples(sets), st.to_struct(), dtype=F32, equilibrate=True)
    D, Ev, c = eng.scaling()
    _, _, _, _, _, sm = O.scale_ruiz(P, q, A, b, to_oracle_cones(sets), O.Settings())
    errs = (np.max(np.abs(D - sm.D) / sm.D), np.max(np.abs(Ev - sm.E) / sm.E), abs(c - sm.c) / sm.c)
    print("MEAS ruiz fp32 %s D/E/c rel err = %.2e %.2e %.2e" % ((prob,) + errs))
    assert max(errs) <= 1e-5, errs


# ---------------------------------------------------------------------------
# solve level: the reference's Float32 unit tests (test/run_cosmo_tests.jl:9)
# ---------------------------------------------------------------------------
def _solve32(builder, **kw):
    P, q, cons = builder()
    model = cosmo_b200.Model(dtype=F32)
    cosmo_b200.assemble(model, P, q, _to_mine(cons), cosmo_b200.Settings(**kw))
    return cosmo_b200.optimize(model), model


@pytest.mark.parametrize("acc", ["EmptyAccelerator", "AndersonAccelerator"])
@pytest.mark.parametrize("builder", [G.g1_qp_nonneg, G.g1_qp_box])
def test_g1_float32(builder, acc):
    res, _ = _solve32(builder, eps_abs=1e-4, eps_rel=1e-4, accelerator=acc)       # simple.jl, qp-box.jl: 1e-3
    assert res.status == "Solved" and np.max(np.abs(res.x - G.G1_X)) < 1e-3 and abs(res.obj_val - G.G1_OBJ) < 1e-3


def test_g2_statuses_float32():
    assert abs(_solve32(G.g2_box_feasible)[0].obj_val + 0.5) < 1e-3
    assert _solve32(G.g2_box_primal_infeasible_1)[0].status == "Primal_infeasible"
    assert _solve32(G.g2_box_primal_infeasible_2)[0].status == "Primal_infeasible"
    assert _solve32(G.g2_box_dual_infeasible, check_infeasibility=20, scaling=0)[0].status == "Dual_infeasible"


_FP32_POW_STALL = pytest.mark.xfail(strict=True, reason="known: Max_iter_reached after 5000 iterations in fp32 (the reference "
                                                       "solves these in Float32 with its direct KKT solver); not fixed yet")


@pytest.mark.parametrize("name,builder,status,obj,atol,kw",
                         [pytest.param(*g, marks=_FP32_POW_STALL) if g[0] in ("pow_feasible", "pow_primal_infeasible") else g
                          for g in G.G15_G16], ids=[g[0] for g in G.G15_G16])
def test_g15_g16_float32(name, builder, status, obj, atol, kw):
    res, _ = _solve32(builder, **kw)
    assert res.status == status, (name, res.status, res.iter)
    if obj is not None:
        assert abs(res.obj_val - obj) < atol, (name, res.obj_val)


def test_g14_model_updates_float32():
    P, q, cons = G.g1_qp_nonneg()
    model = cosmo_b200.Model(dtype=F32)
    cosmo_b200.assemble(model, P, q, _to_mine(cons), cosmo_b200.Settings())
    model.optimize()
    model.update(q=np.array([2.0, 3.0]))
    r = model.optimize()
    assert abs(r.obj_val - 3.5) < 1e-3 and np.linalg.norm(r.x - [0.5, 0.5]) < 1e-3      # model_modifications.jl:41-43
    model = cosmo_b200.Model(dtype=F32)
    cosmo_b200.assemble(model, np.zeros((2, 2)), np.array([1.0, 1.0]),
                        cosmo_b200.Constraint(np.eye(2), np.array([-2.0, -3.0]), cosmo_b200.Nonnegatives),
                        cosmo_b200.Settings(check_termination=20))
    assert np.linalg.norm(model.optimize().x - [2.0, 3.0]) < 1e-3
    model.update(b=np.array([0.0, 1.0]))
    assert np.linalg.norm(model.optimize().x - [0.0, -1.0]) < 1e-3                      # :57-59


@pytest.mark.xfail(strict=True, reason="known: Max_iter_reached in fp32 at default settings (closestcorr.jl expects "
                                      ":Solved for Float32); not fixed yet")
def test_closest_correlation_float32():
    N = 40
    P, q, A, b, sets = cosmo_b200.problems.closest_correlation_sdp(N=N, seed=12345)
    model = cosmo_b200.Model(dtype=F32)
    model.set(P, q, A, b, sets, cosmo_b200.Settings())
    res = model.optimize()
    assert res.status == "Solved"
    X = np.zeros((N, N))
    iu = np.triu_indices(N)
    order = np.lexsort((iu[0], iu[1]))
    r, c = iu[0][order], iu[1][order]
    X[r, c] = np.where(r == c, res.x, res.x / np.sqrt(2))
    X = X + np.triu(X, 1).T
    assert np.max(np.abs(np.diag(X) - 1.0)) < 1e-3 and np.linalg.eigvalsh(X).min() > -1e-3   # closestcorr.jl:70-80
