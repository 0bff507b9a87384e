"""GPU parity tests: every call goes through the C ABI (ctypes -> libcosmo_b200.so)
and is compared with the CPU oracle on identical seeded inputs (SURVEY.md 8c
parity protocol).  Tolerances are stated per test."""
import os

import numpy as np
import pytest
import scipy.sparse as sp

import cosmo_b200
from cosmo_b200 import engine as E
from oracle import cosmo_oracle as O
from oracle.bridge import to_oracle_cones
from tests import golden_problems as G
from tests.gpu_helpers import _engine, _hermitian_ws, _psd_test_matrix, _tuples

pytestmark = pytest.mark.gpu


def _ragged_matrix(rng, m, n):
    """rows of length 0, 1, 2, 3, 5, ~n/3 and full: exercises head/body/tail peeling"""
    rows, cols, vals = [], [], []
    for i in range(m):
        k = [0, 1, 2, 3, 5, 7, n // 3, n][i % 8]
        k = min(k, n)
        c = np.sort(rng.choice(n, size=k, replace=False))
        rows += [i] * k
        cols += list(c)
        vals += list(rng.standard_normal(k))
    return sp.csc_matrix((vals, (rows, cols)), shape=(m, n))


# ---------------------------------------------------------------------------
# K1-K3: SpMV (kktsolver_indirect.jl:53-63 mul! calls)
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("m,n", [(1, 1), (17, 9), (64, 257), (300, 131), (1000, 515)])
def test_spmv_ragged(m, n):
    rng = np.random.default_rng(m * 1000 + n)
    A = _ragged_matrix(rng, m, n)
    B = _ragged_matrix(rng, n, n)
    P = sp.csc_matrix(B + B.T)
    eng = _engine(P, np.zeros(n), A, np.zeros(m), [cosmo_b200.Nonnegatives(m)])
    x = rng.standard_normal(n)
    y = rng.standard_normal(m)
    for which, M, v in ((0, A, x), (1, A.T, y), (2, P, x)):
        got = eng.spmv(which, v)
        ref = M @ v
        scale = np.abs(M) @ np.abs(v) + 1e-300
        assert np.max(np.abs(got - ref) / scale) < 1e-14, which  # summation order differs only


@pytest.mark.parametrize("density,lanes", [(0.002, 2), (0.02, 8), (0.2, 32)])
def test_spmv_lane_variants(density, lanes):
    rng = np.random.default_rng(5)
    m, n = 3000, 1500
    A = sp.random(m, n, density=density, random_state=rng, data_rvs=rng.standard_normal, format="csc")
    P = sp.identity(n, format="csc")
    eng = _engine(P, np.zeros(n), A, np.zeros(m), [cosmo_b200.Nonnegatives(m)])
    x, y = rng.standard_normal(n), rng.standard_normal(m)
    assert np.allclose(eng.spmv(0, x), A @ x, rtol=1e-12, atol=1e-12)
    assert np.allclose(eng.spmv(1, y), A.T @ y, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("m,n,per_row", [(400, 30000, 100), (30000, 400, 100), (3000, 60000, 300)])
def test_spmv_windowed_smem_path(m, n, per_row):
    """rows long enough for the column-windowed kernel (x slices staged in shared memory by TMA bulk
    copies): 1, 2 and 3 windows, rows with empty window segments, multi-step segments, fused P rows."""
    rng = np.random.default_rng(m + n)
    rows = np.repeat(np.arange(m), per_row)
    cols = rng.integers(0, n, size=m * per_row)
    cols[: per_row] = rng.integers(0, min(n, 50), size=per_row)        # row 0 lives in window 0 only
    A = sp.csc_matrix((rng.standard_normal(m * per_row), (rows, cols)), shape=(m, n))
    B = sp.random(n, n, density=3.0 / n, random_state=rng, format="csr") * 0.05
    P = sp.csc_matrix(B + B.T + sp.identity(n))          # diagonally dominant: well-conditioned reduced system
    eng = _engine(P, np.zeros(n), A, np.zeros(m), [cosmo_b200.Nonnegatives(m)], scaling=0)
    x, y = rng.standard_normal(n), rng.standard_normal(m)
    for which, M, v in ((0, A, x), (1, A.T, y)):
        got, ref = eng.spmv(which, v), M @ v
        scale = np.abs(M) @ np.abs(v) + 1e-300
        assert np.max(np.abs(got - ref) / scale) < 1e-14, which
    # the fused reduced-KKT operator (A' slab kernel + P rows + dot) through the CG solve
    rho = eng.rho_vec()
    ocg = O.IndirectReducedKKT(P, A, 1e-6, rho.copy(), "CG")
    for k in range(2):
        rhs = rng.standard_normal(n + m)
        sol, inner = eng.kkt_solve(rhs)
        ref = ocg.solve(rhs)
        assert abs(inner - ocg.inner_iterations[-1]) <= 1
        assert np.linalg.norm(sol - ref) <= 1e-8 * np.linalg.norm(ref)
    xr, sr, mur = rng.standard_normal(n), rng.standard_normal(m), rng.standard_normal(m)
    got = eng.residuals(xr, sr, mur)
    rp = np.max(np.abs(A @ xr + sr))
    rd = np.max(np.abs(P @ xr - A.T @ mur))
    assert np.isclose(got[0], rp, rtol=1e-12) and np.isclose(got[1], rd, rtol=1e-12)


def test_spmv_float32():
    rng = np.random.default_rng(6)
    m, n = 500, 300
    A = sp.random(m, n, density=0.1, random_state=rng, data_rvs=rng.standard_normal, format="csc")
    eng = _engine(sp.identity(n, format="csc"), np.zeros(n), A, np.zeros(m), [cosmo_b200.Nonnegatives(m)], dtype=np.float32)
    x = rng.standard_normal(n).astype(np.float32)
    ref = A.astype(np.float32) @ x
    assert np.allclose(eng.spmv(0, x), ref, rtol=2e-5, atol=2e-5)  # fp32 tolerance (Model{Float32})


# ---------------------------------------------------------------------------
# K5/K6: composite projection (convexset.jl:885-891)
# ---------------------------------------------------------------------------
def _composite(rng, psd_sizes=(1, 2, 5, 16), square=(3,), soc=(1, 2, 9, 20000)):
    sets = [cosmo_b200.ZeroSet(7), cosmo_b200.Nonnegatives(33)]
    l = rng.standard_normal(21) - 1.0
    u = l + rng.random(21) * 2
    l[3], u[5] = -np.inf, np.inf
    l[7] = u[7]
    sets.append(cosmo_b200.Box(l, u))
    sets += [cosmo_b200.SecondOrderCone(d) for d in soc]
    sets += [cosmo_b200.PsdCone(N * N) for N in square]
    sets += [cosmo_b200.PsdConeTriangle(N * (N + 1) // 2) for N in psd_sizes]
    return sets


def test_project_composite_matches_oracle():
    rng = np.random.default_rng(11)
    sets = _composite(rng)
    m = sum(S.dim for S in sets)
    n = 4
    A = sp.random(m, n, density=0.3, random_state=rng, format="csc")
    eng = _engine(sp.identity(n, format="csc"), np.zeros(n), A, np.zeros(m), sets)
    cones = to_oracle_cones(sets)
    for trial in range(3):
        ws = rng.standard_normal(m) * (10.0 ** trial)
        ws[3] = np.nan if trial == 2 else ws[3]          # NaN propagates through max(x, 0) like Julia
        ref = ws.copy()
        O.project(ref, cones)
        got = eng.project(ws)
        off = 0
        for S in sets:
            seg = slice(off, off + S.dim)
            if isinstance(S, (cosmo_b200.ZeroSet, cosmo_b200.Nonnegatives, cosmo_b200.Box)):
                assert np.array_equal(got[seg], ref[seg], equal_nan=True), type(S)     # bit-exact clamp cones
            elif isinstance(S, cosmo_b200.SecondOrderCone):
                assert np.allclose(got[seg], ref[seg], rtol=1e-14, atol=1e-14 * (1 + np.abs(ref[seg]).max()))
            else:  # PSD: |Pi_gpu - Pi_lapack|_F / |X|_F <= 1e-12
                nrm = np.linalg.norm(ws[seg]) + 1e-300
                assert np.linalg.norm(got[seg] - ref[seg]) / nrm < 1e-12, (type(S), S.dim)
            off += S.dim


def test_soc_branches():
    # convexset.jl:100-114: inside cone, inside polar cone, and the generic case
    sets = [cosmo_b200.SecondOrderCone(4)] * 3
    ws = np.array([5.0, 1, 1, 1, -5.0, 1, 1, 1, 0.5, 1, 2, 2])
    eng = _engine(sp.identity(1, format="csc"), np.zeros(1), sp.csc_matrix((12, 1)), np.zeros(12), sets)
    ref = ws.copy()
    O.project(ref, to_oracle_cones(sets))
    got = eng.project(ws)
    assert np.array_equal(got[:8], ref[:8])
    assert np.allclose(got[8:], ref[8:], rtol=1e-15)


def test_project_exp_pow_cones():
    # convexset.jl:510-532, 646-668, 784-789: the four projection cases of K_exp / K_pow and the Moreau
    # route of the dual cones.  The root searches stop at EXP_TOL / POW_TOL = 1e-8 (reference constants),
    # so CPU and GPU agree to that tolerance times the conditioning of the search, not to the last ulp:
    # asserted |diff| <= 1e-6 (1 + |v|); points that need no search (cases 1-3) are bit-exact.
    rng = np.random.default_rng(5)
    sets, pts = [], []
    special_exp = [(1.0, 2.0, 10.0), (-3.0, 0.0, 1.0),      # inside K_exp
                   (1.0, -2.0, -3.0), (0.0, -1.0, -2.0),      # -v in K_exp^* -> 0
                   (-2.0, -3.0, 4.0), (-2.0, -3.0, -4.0)]     # x, y < 0 -> (x, 0, max(z, 0))
    for v in special_exp:
        sets.append(cosmo_b200.ExponentialCone()); pts.append(v)
    special_pow = [(2.0, 3.0, 1.0), (-1.0, -2.0, 0.5), (3.0, -2.0, 1e-9), (-3.0, 2.0, 0.0)]
    for v in special_pow:
        sets.append(cosmo_b200.PowerCone(0.3)); pts.append(v)
    n_special = len(sets)
    for i in range(400):
        a = 0.1 + 0.85 * rng.random()
        for S in (cosmo_b200.ExponentialCone(), cosmo_b200.DualExponentialCone(), cosmo_b200.PowerCone(a),
                  cosmo_b200.DualPowerCone(a)):
            sets.append(S)
            pts.append(-25.0 + 50.0 * rng.random(3))    # test/UnitTests/sets.jl:87,97
    ws = np.concatenate([np.asarray(v, dtype=float) for v in pts])
    m = ws.size
    eng = _engine(sp.identity(1, format="csc"), np.zeros(1), sp.csc_matrix((m, 1)), np.zeros(m), sets)
    cones = to_oracle_cones(sets)
    ref = ws.copy()
    O.project(ref, cones)
    got = eng.project(ws)
    assert np.array_equal(got[:3 * n_special], ref[:3 * n_special])
    err = np.abs(got - ref).reshape(-1, 3).max(axis=1)
    scale = 1.0 + np.abs(ws).reshape(-1, 3).max(axis=1)
    assert np.all(err <= 1e-6 * scale), float((err / scale).max())
    # sets.jl:90,101 asks in_cone(Pi v, 1e-4) of 100 random points.  Of these 1600, four land where
    # y -> 0 makes y e^(x/y) ill-conditioned and the reference's own search misses that tolerance; the
    # GPU must reproduce the verdict of the CPU restatement point by point, misses included.
    mine = np.array([O.in_cone(got[3 * k:3 * k + 3], c, 1e-4) for k, c in enumerate(cones)])
    theirs = np.array([O.in_cone(ref[3 * k:3 * k + 3], c, 1e-4) for k, c in enumerate(cones)])
    assert np.array_equal(mine, theirs) and mine.mean() > 0.99


@pytest.mark.parametrize("N", [97, 130])
def test_project_psd_large_path(N):
    rng = np.random.default_rng(N)
    d = N * (N + 1) // 2
    sets = [cosmo_b200.PsdConeTriangle(d)]
    eng = _engine(sp.identity(1, format="csc"), np.zeros(1), sp.csc_matrix((d, 1)), np.zeros(d), sets)
    ws = rng.standard_normal(d)
    ref = ws.copy()
    O.project(ref, to_oracle_cones(sets))
    got = eng.project(ws)
    assert np.linalg.norm(got - ref) / np.linalg.norm(ws) < 1e-12


@pytest.mark.parametrize("kind", ["wigner", "rank_deficient", "shifted", "zero"])
def test_project_psd_tensor_core_path_n150(kind):
    # Pi_+(X) = (X + sign(X) X) / 2 with sign(X) by Newton-Schulz products; same bar as the eigensolver path
    rng = np.random.default_rng(21)
    N = 150
    B = rng.standard_normal((N, N))
    if kind == "wigner":
        X = (B + B.T) / 2
    elif kind == "rank_deficient":
        X = B[:, :20] @ B[:, :20].T - B[:, 20:30] @ B[:, 20:30].T
    elif kind == "shifted":
        X = (B + B.T) / 2 + 3.0 * np.eye(N)
    else:
        X = np.zeros((N, N))
    sets = [cosmo_b200.PsdConeTriangle(N * (N + 1) // 2), cosmo_b200.PsdCone(N * N)]
    ws = np.concatenate([G._svec(X), X.reshape(-1, order="F")])
    m = ws.size
    eng = _engine(sp.identity(1, format="csc"), np.zeros(1), sp.csc_matrix((m, 1)), np.zeros(m), sets)
    ref = ws.copy()
    O.project(ref, to_oracle_cones(sets))
    got = eng.project(ws)
    nrm = np.linalg.norm(ws) + 1e-300
    assert np.linalg.norm(got - ref) / nrm < 1e-12
    st = eng.psd_stats()
    assert st["tc_projections"] == 2 and st["tc_fallbacks"] == 0, st


# ---------------------------------------------------------------------------
# Tensor-core PSD path (csrc/tc_gemm.cuh, csrc/psd_tc.cuh): int8-sliced wgmma products + scaled Newton-Schulz
# ---------------------------------------------------------------------------
# N = 2000 / 2700: 136 / 253 upper-triangle tiles, more than the 132 SMs of an H100, so CTAs of the persistent kernel
# compute several tiles (ring position, phase and the reduction buffer carry over from tile to tile)
@pytest.mark.parametrize("N,slices,groups,bound", [(128, 8, 10, 2e-15), (200, 8, 10, 2e-15), (333, 8, 10, 2e-15), (333, 8, 8, 5e-15),
                                                   (333, 7, 7, 1e-12), (200, 6, 8, 1e-11), (200, 4, 6, 2e-7),
                                                   (2000, 8, 10, 2e-15), (2700, 8, 10, 2e-15)])
def test_tc_gemm_matches_dgemm(N, slices, groups, bound):
    # C = A B for commuting symmetric matrices; error measured against |A| |B| elementwise (the natural bound of a
    # row-scaled fixed-point product); one row is 1000x smaller than the rest (per-row exponents)
    rng = np.random.default_rng(N)
    Gm = rng.standard_normal((N, N))
    A = (Gm + Gm.T) / np.sqrt(2.0 * N)
    A[0, :] *= 1e-3
    A[:, 0] *= 1e-3
    B = A @ A
    B = (B + B.T) / 2
    got, _, fr = E.tc_gemm(A, B, slices=slices, groups=groups)
    ref = A @ B
    assert np.max(np.abs(got - ref) / (np.abs(A) @ np.abs(B))) < bound
    assert np.array_equal(got, got.T)                                   # mirrored store: exactly symmetric
    assert abs(fr[0] - np.sum(got * got)) <= 1e-12 * np.sum(got * got)  # fused |C|_F^2
    assert abs(fr[1] - np.sum((np.eye(N) - got) ** 2)) <= 1e-12 * np.sum((np.eye(N) - got) ** 2)


@pytest.mark.parametrize("kind", ["wigner", "rank_deficient", "shifted", "zero", "admm_like", "graded"])
@pytest.mark.parametrize("N", [200, 385])
def test_project_psd_tensor_core_path(kind, N):
    # same bar as the eigensolver path (SURVEY 8c-i: |Pi_gpu - Pi_lapack|_F / |X|_F <= 1e-12), triangle and square cone,
    # and the projection must really have come from the tensor-core path (no silent fallback)
    rng = np.random.default_rng(1000 + N)
    X = _psd_test_matrix(kind, N, rng)
    sets = [cosmo_b200.PsdConeTriangle(N * (N + 1) // 2), cosmo_b200.PsdCone(N * N)]
    ws = np.concatenate([G._svec(X), X.reshape(-1, order="F")])
    m = ws.size
    eng = _engine(sp.identity(1, format="csc"), np.zeros(1), sp.csc_matrix((m, 1)), np.zeros(m), sets)
    ref = ws.copy()
    O.project(ref, to_oracle_cones(sets))
    got = eng.project(ws)
    st = eng.psd_stats()
    assert st["tc_projections"] == 2 and st["tc_fallbacks"] == 0, st
    assert np.linalg.norm(got - ref) / (np.linalg.norm(ws) + 1e-300) < 1e-12, st


def test_project_psd_tensor_core_path_float32():
    # Model{Float32}: the oracle runs ssyevr (convexset.jl:163-165); the bar is the fp32 one of SURVEY 8c-i (1e-5).  The
    # reference's own fp32 path is only ~N eps32 accurate, so the engine (fp64 iterates inside) is also held against the
    # fp64 projection: it must not be worse than the reference's fp32 path.
    rng = np.random.default_rng(77)
    N = 256
    X = _psd_test_matrix("wigner", N, rng).astype(np.float32)
    sets = [cosmo_b200.PsdConeTriangle(N * (N + 1) // 2)]
    ws = G._svec(X.astype(np.float64)).astype(np.float32)
    m = ws.size
    eng = _engine(sp.identity(1, format="csc"), np.zeros(1), sp.csc_matrix((m, 1)), np.zeros(m), sets, dtype=np.float32)
    ref = ws.copy()
    O.project(ref, to_oracle_cones(sets))
    got = eng.project(ws)
    st = eng.psd_stats()
    assert st["tc_projections"] == 1 and st["tc_fallbacks"] == 0, st
    truth = ws.astype(np.float64)
    O.project(truth, to_oracle_cones(sets))
    nrm = np.linalg.norm(ws.astype(np.float64))
    err_engine = np.linalg.norm(got.astype(np.float64) - truth) / nrm
    err_ref32 = np.linalg.norm(ref.astype(np.float64) - truth) / nrm
    assert err_engine <= max(err_ref32, 2e-7), (err_engine, err_ref32)
    assert np.linalg.norm(got.astype(np.float64) - ref) / nrm < 1e-5 + err_ref32


def test_complex_psd_cone_projection_and_least_eigenvalue():
    # PsdConeTriangle{T, Complex{T}} (convexset.jl:344-360, 444-490): projection vs the Hermitian eigendecomposition of
    # the oracle at the real-PSD bar (1e-12), then least_eigenvalue.jl:33-39 (obj = 1 - sqrt 2 at 1e-4)
    rng = np.random.default_rng(9)
    sizes = [1, 2, 5, 12, 48]
    sets = [cosmo_b200.ComplexPsdConeTriangle(N * N) for N in sizes]
    parts = []
    for N in sizes:
        Z = rng.standard_normal((N, N)) + 1j * rng.standard_normal((N, N))
        parts.append(O.extract_upper_triangle_complex((Z + Z.conj().T) / 2 - 0.3 * np.eye(N), np.sqrt(2.0)))
    ws = np.concatenate(parts)
    m = ws.size
    eng = _engine(sp.identity(1, format="csc"), np.zeros(1), sp.csc_matrix((m, 1)), np.zeros(m), sets)
    ref = ws.copy()
    O.project(ref, to_oracle_cones(sets))
    got = eng.project(ws)
    off = 0
    for S in sets:
        seg = slice(off, off + S.dim)
        assert np.linalg.norm(got[seg] - ref[seg]) / (np.linalg.norm(ws[seg]) + 1e-300) < 1e-12, S.dim
        off += S.dim
    res, _ = _solve_mine(G.g17_complex_least_eigenvalue)
    ref = _solve_oracle(G.g17_complex_least_eigenvalue)
    assert res.status == "Solved" == ref.status and abs(res.obj_val - G.G17_OBJ) < 1e-4 + 1e-4 * abs(G.G17_OBJ)
    assert abs(res.iter - ref.iter) <= 25 and abs(res.obj_val - ref.obj_val) < 1e-5


def test_project_psd_batch_of_cliques():
    # many small cones in one launch (chordal-decomposition shape)
    rng = np.random.default_rng(3)
    sizes = rng.integers(2, 40, size=200)
    sets = [cosmo_b200.PsdConeTriangle(int(N * (N + 1) // 2)) for N in sizes]
    m = sum(S.dim for S in sets)
    eng = _engine(sp.identity(1, format="csc"), np.zeros(1), sp.csc_matrix((m, 1)), np.zeros(m), sets)
    ws = rng.standard_normal(m)
    ref = ws.copy()
    O.project(ref, to_oracle_cones(sets))
    got = eng.project(ws)
    assert np.linalg.norm(got - ref) / np.linalg.norm(ws) < 1e-12
    # idempotence: projecting a projected point changes nothing (size-independent property)
    again = eng.project(got)
    assert np.linalg.norm(again - got) / np.linalg.norm(got) < 1e-12


# ---------------------------------------------------------------------------
# P4a: reduced-KKT CG solve (kktsolver_indirect.jl:36-88)
# ---------------------------------------------------------------------------
def _small_qp(seed=0, n=40, m=70):
    return cosmo_b200.problems.random_sparse_qp(n, m, 0.15, seed=seed)


def test_kkt_solve_matches_oracle_and_direct():
    P, q, A, b, sets = _small_qp()
    m, n = A.shape
    eng = _engine(P, q, A, b, sets, scaling=0)
    rng = np.random.default_rng(2)
    rho = eng.rho_vec()
    ocg = O.IndirectReducedKKT(P, A, 1e-6, rho.copy(), "CG")
    direct = O.DirectKKT(P, A, 1e-6, rho)
    for k in range(6):
        rhs = rng.standard_normal(n + m)
        sol, inner = eng.kkt_solve(rhs)
        ref = ocg.solve(rhs)
        assert inner == ocg.inner_iterations[-1]                 # same tolerance schedule & stopping rule
        assert np.allclose(sol, ref, rtol=1e-9, atol=1e-9)
        # and both are inexact solves of the same KKT system (kktsolver.jl:104-109)
        tol = 1.0 / (k + 1) ** 1.5 / np.linalg.norm(rhs[:n] + A.T @ (rho * rhs[n:]))
        exact = direct.solve(rhs)
        assert np.linalg.norm(sol - exact) <= 1e3 * max(tol, 1e-12) * (1 + np.linalg.norm(exact))


@pytest.mark.parametrize("name,kind", [("MINRESIndirectKKTSolver", "minres"), ("IndirectReducedKKTSolver:MINRES", "minres_reduced")])
def test_minres_kkt_solve_matches_oracle(name, kind):
    # IndirectKKTSolver / IndirectReducedKKTSolver(:MINRES), kktsolver_indirect.jl:72-73, 123-162
    P, q, A, b, sets = _small_qp(seed=3, n=41, m=70)      # odd n: exercises the padded x2 offset
    m, n = A.shape
    eng = _engine(P, q, A, b, sets, scaling=0, kkt_solver=name)
    rho = eng.rho_vec()
    ref_solver = O.make_kkt_solver(kind, P, A, 1e-6, rho.copy(), O.Settings())
    direct = O.DirectKKT(P, A, 1e-6, rho)
    rng = np.random.default_rng(9)
    for k in range(5):
        rhs = rng.standard_normal(n + m)
        sol, inner = eng.kkt_solve(rhs)
        ref = ref_solver.solve(rhs)
        assert abs(inner - ref_solver.inner_iterations[-1]) <= 2
        assert np.linalg.norm(sol - ref) <= 1e-6 * (1 + np.linalg.norm(ref))
    # both converge to the direct solution when the tolerance schedule has tightened
    for k in range(40):
        sol, _ = eng.kkt_solve(rhs)
    assert np.linalg.norm(sol - direct.solve(rhs)) <= 1e-3 * (1 + np.linalg.norm(sol))


@pytest.mark.parametrize("name,kind", [("MINRESIndirectKKTSolver", "minres"), ("IndirectReducedKKTSolver:MINRES", "minres_reduced")])
def test_minres_solve_matches_oracle(name, kind):
    P, q, A, b, sets = _small_qp(seed=12)
    cones = to_oracle_cones(sets)
    ref = O.solve(P, q, A, b, cones, O.Settings(kkt_solver=kind, max_iter=300))
    model = cosmo_b200.Model()
    model.set(P, q, A, b, sets, cosmo_b200.Settings(kkt_solver=name, max_iter=300))
    res = model.optimize()
    # the reference's MINRES tolerance rule (abstol = tol_k / initial residual) makes the outer iteration plateau (see
    # tests/test_oracle_golden.py): both runs stop at max_iter.  Measured over three seeds (tests/run_minres_diffs.py):
    # |x - x_ref| <= 1e-10 and |obj - obj_ref| <= 2e-11 relative (full KKT), 1e-15 (reduced); bound 1e-8.
    assert res.status == ref.status and res.iter == ref.iter
    assert abs(res.obj_val - ref.obj_val) <= 1e-8 * max(1, abs(ref.obj_val))
    assert np.max(np.abs(res.x - ref.x)) <= 1e-8 * max(1, np.abs(ref.x).max())


def test_residuals_match_oracle():
    P, q, A, b, sets = _small_qp(seed=4)
    m, n = A.shape
    st = cosmo_b200.Settings()
    Ps, qs, As, bs, ss, D, Em, c = cosmo_b200.ruiz_equilibrate(P, q, A, b, sets, st)
    eng = E.Engine(Ps, qs, As, bs, _tuples(ss), st.to_struct(), D=D, E=Em, c=c)
    rng = np.random.default_rng(8)
    x, s, mu = rng.standard_normal(n), rng.standard_normal(m), rng.standard_normal(m)
    ws = O.Workspace(P, q, A, b, to_oracle_cones(sets), O.Settings())
    ws.setup()
    ws.xv, ws.s, ws.mu = x, s, mu
    for ign in (False, True):
        rp, rd = ws.calculate_residuals(ign)
        mp, md = ws.max_res_component_norm(ign)
        got = eng.residuals(x, s, mu, ign)
        assert np.allclose(got[:4], [rp, rd, mp, md], rtol=1e-11)
    assert np.isclose(eng.residuals(x, s, mu)[4], ws.calculate_cost(), rtol=1e-11)


# ---------------------------------------------------------------------------
# iterate-level parity (SURVEY 8c-ii): w trajectories vs the oracle
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("scaling", [0, 10])
def test_iterate_parity_first_iterations(scaling):
    P, q, A, b, sets = _small_qp(seed=7)
    cones = to_oracle_cones(sets)
    for iters in (1, 5, 40, 90):   # 40/80: rho adaptation + infeasibility checks are crossed
        ost = O.Settings(kkt_solver="cg", scaling=scaling, max_iter=iters, eps_abs=1e-14, eps_rel=1e-14)
        ref = O.solve(P, q, A, b, cones, ost)
        model = cosmo_b200.Model()
        model.set(P, q, A, b, sets, cosmo_b200.Settings(scaling=scaling, max_iter=iters, eps_abs=1e-14, eps_rel=1e-14))
        res = model.optimize()
        w = model.engine.w()
        assert res.iter == ref.iter == iters
        assert np.allclose(model.engine.rho_vec(), ref.rho_vec, rtol=1e-9)
        assert list(np.round(res.info.rho_updates, 9)) == list(np.round(ref.info.rho_updates, 9))
        assert np.linalg.norm(w - ref.w) / np.linalg.norm(ref.w) < 1e-8, iters
        assert np.allclose(res.x, ref.x, rtol=1e-7, atol=1e-9)
        assert np.allclose(res.s, ref.s, rtol=1e-7, atol=1e-9)
        assert np.allclose(res.y, ref.y, rtol=1e-7, atol=1e-9)
        assert np.isclose(res.info.r_prim, ref.info.r_prim, rtol=1e-6, atol=1e-12)
        assert np.isclose(res.info.r_dual, ref.info.r_dual, rtol=1e-6, atol=1e-12)


@pytest.mark.parametrize("scaling", [0, 10])
def test_accelerated_iterates_match_oracle(scaling):
    # Anderson acceleration (aa.cuh) against the oracle's restatement of the same method: the history update,
    # the QR least squares, the candidate, the safeguard decisions (two candidates are declined at iterations
    # 31-32 of this problem) and the memory restarts.  Measured agreement of w: 1e-13; asserted 1e-9.
    P, q, A, b, sets = _small_qp(seed=7)
    cones = to_oracle_cones(sets)
    for iters in (2, 5, 14, 33, 45):  # first update, first candidate, memory almost full, declined candidates, restarts
        ost = O.Settings(kkt_solver="cg", scaling=scaling, max_iter=iters, eps_abs=1e-14, eps_rel=1e-14, accelerator="anderson")
        ref = O.solve(P, q, A, b, cones, ost)
        model = cosmo_b200.Model()
        model.set(P, q, A, b, sets, cosmo_b200.Settings(scaling=scaling, max_iter=iters, eps_abs=1e-14, eps_rel=1e-14,
                                                        accelerator="AndersonAccelerator"))
        res = model.optimize()
        w = model.engine.w()
        # a declined candidate adds a safeguarding iteration inside the loop body, so the total can pass
        # max_iter by one (solver.jl:140: `while iter + safeguarding_iter < max_iter`)
        assert iters <= res.iter == ref.iter <= iters + 1 and res.safeguarding_iter == ref.safeguarding_iter
        assert np.linalg.norm(w - ref.w) / np.linalg.norm(ref.w) < 1e-9, iters
        assert np.allclose(res.x, ref.x, rtol=1e-5, atol=1e-7)


def test_engine_matches_committed_golden_iterates():
    # tests/golden/oracle_iterates.npz (generated by tests/golden/make_golden.py from the pinned oracle):
    # w after k iterations of plain and accelerated runs, without running the oracle here
    import os
    gold = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "oracle_iterates.npz"))
    P, q, A, b, sets = _small_qp(seed=7)
    for acc, name in (("empty", "EmptyAccelerator"), ("anderson", "AndersonAccelerator")):
        for scaling in (0, 10):
            for iters in (5, 14, 33):
                key = "qp40x70_seed7/%s/scaling%d/it%d" % (acc, scaling, iters)
                model = cosmo_b200.Model()
                model.set(P, q, A, b, sets, cosmo_b200.Settings(scaling=scaling, max_iter=iters, eps_abs=1e-14, eps_rel=1e-14,
                                                                accelerator=name))
                res = model.optimize()
                w = model.engine.w()
                assert [res.iter, res.safeguarding_iter] == gold[key + "/iter_sg"].tolist(), key
                assert np.linalg.norm(w - gold[key + "/w"]) / np.linalg.norm(gold[key + "/w"]) < 1e-8, key
    res, _ = _solve_mine(G.g1_qp_nonneg, scaling=0)
    assert res.iter == int(gold["g1_qp_nonneg/iter_obj"][0]) and abs(res.obj_val - gold["g1_qp_nonneg/iter_obj"][1]) < 1e-9
    assert np.allclose(res.x, gold["g1_qp_nonneg/x"], atol=1e-7) and np.allclose(res.s, gold["g1_qp_nonneg/s"], atol=1e-7)
    assert np.allclose(res.y, gold["g1_qp_nonneg/y"], atol=1e-6)
    res, _ = _solve_mine(G.g13_lovasz_petersen, eps_abs=1e-6, eps_rel=1e-6)
    assert abs(res.iter - int(gold["g13_lovasz_petersen/iter_obj"][0])) <= 25
    assert abs(res.obj_val - gold["g13_lovasz_petersen/iter_obj"][1]) < 1e-6
    res, _ = _solve_mine(G.g15_exp_feasible, eps_abs=1e-4, eps_rel=1e-4)
    assert abs(res.iter - int(gold["g15_exp_feasible/iter_obj"][0])) <= 25
    assert abs(res.obj_val - gold["g15_exp_feasible/iter_obj"][1]) < 1e-4 and np.allclose(res.x, gold["g15_exp_feasible/x"], atol=1e-3)


# ---------------------------------------------------------------------------
# solve-level parity on the reference's literal problems (SURVEY 8c G1..G14)
# ---------------------------------------------------------------------------
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


def _solve_mine(builder, **kw):
    P, q, cons = builder()
    model = cosmo_b200.Model()
    cosmo_b200.assemble(model, P, q, _to_mine(cons), cosmo_b200.Settings(**kw))
    return cosmo_b200.optimize(model), model


def _solve_oracle(builder, **kw):
    P, q, cons = builder()
    Pm, qm, A, b, cones = O.assemble(P, q, cons)
    return O.solve(Pm, qm, A, b, cones, O.Settings(kkt_solver="cg", **kw))


@pytest.mark.parametrize("builder", [G.g1_qp_nonneg, G.g1_qp_box])
@pytest.mark.parametrize("scaling", [0, 10])
def test_g1_simple_qp(builder, scaling):
    res, _ = _solve_mine(builder, scaling=scaling)
    ref = _solve_oracle(builder, scaling=scaling)
    assert res.status == "Solved" == ref.status
    assert np.max(np.abs(res.x - G.G1_X)) < 1e-3 and abs(res.obj_val - G.G1_OBJ) < 1e-3   # examples/qp.jl:41-44
    assert res.iter == ref.iter
    assert np.allclose(res.x, ref.x, atol=1e-7) and np.allclose(res.y, ref.y, atol=1e-6) and np.allclose(res.s, ref.s, atol=1e-7)


def test_g2_box_statuses():
    assert abs(_solve_mine(G.g2_box_feasible)[0].obj_val + 0.5) < 1e-5
    assert _solve_mine(G.g2_box_primal_infeasible_1)[0].status == "Primal_infeasible"
    assert _solve_mine(G.g2_box_primal_infeasible_2)[0].status == "Primal_infeasible"
    assert _solve_mine(G.g2_box_dual_infeasible, check_infeasibility=20, scaling=0)[0].status == "Dual_infeasible"
    assert _solve_mine(G.g2_box_dual_infeasible, check_infeasibility=40, scaling=10)[0].status == "Dual_infeasible"
    for bld, kw in ((G.g2_box_primal_infeasible_1, {}), (G.g2_box_dual_infeasible, dict(check_infeasibility=20, scaling=0))):
        assert _solve_mine(bld, **kw)[0].iter == _solve_oracle(bld, **kw).iter


def test_g3_hs21_with_soc_and_merging():
    res, model = _solve_mine(G.g3_hs21)
    ref = _solve_oracle(G.g3_hs21)
    assert [type(S).__name__ for S in model.sets0] == ["ZeroSet", "Nonnegatives", "Box", "Box", "SecondOrderCone"]
    assert res.status == "Solved" and abs(res.obj_val - G.G3_OBJ) < 1e-3 and np.max(np.abs(res.x - G.G3_X)) < 1e-3
    assert res.iter == ref.iter and np.allclose(res.x, ref.x, atol=1e-6)


def test_g12_lp():
    res, _ = _solve_mine(G.g12_lp, eps_abs=1e-4, eps_rel=1e-5)
    assert res.status == "Solved" and np.max(np.abs(res.x - G.G12_X)) < 1e-2 and abs(res.obj_val - G.G12_OBJ) < 1e-2


@pytest.mark.parametrize("name,builder,status,obj,atol,kw", G.G15_G16, ids=[g[0] for g in G.G15_G16])
def test_g15_g16_exp_pow_cone_problems(name, builder, status, obj, atol, kw):
    # test/UnitTests/exp_cone.jl, pow_cone.jl: the reference's expected statuses / objectives, and the oracle's
    # iterates (the projections agree to the 1e-8 search tolerance, so iteration counts may differ by one check)
    res, _ = _solve_mine(builder, **kw)
    ref = _solve_oracle(builder, **kw)
    assert res.status == status == ref.status
    assert abs(res.iter - ref.iter) <= 25
    if obj is not None:
        assert abs(res.obj_val - obj) < atol
        assert abs(res.obj_val - ref.obj_val) < 1e-4 and np.allclose(res.x, ref.x, atol=1e-3)


def test_g4_g5_g11_literal_problems():
    # G4 moi_wrapper.jl:39-106 (constraint primals 11 / 19 at 1e-3, check_termination = 1)
    res, _ = _solve_mine(G.g4_small_sdp, check_termination=1)
    ref = _solve_oracle(G.g4_small_sdp, check_termination=1)
    assert res.status == "Solved" == ref.status and abs(res.iter - ref.iter) <= 2
    assert abs(G.G4_A1 @ res.x - 11.0) < 1e-3 and abs(G.G4_A2 @ res.x - 19.0) < 1e-3
    assert np.allclose(res.x, ref.x, atol=1e-4)
    # G5 nuclear_norm_minimization.jl:31-40: t = sigma_max(Y) at 1e-3, the three inequalities hold
    res, _ = _solve_mine(G.g5_sigma_max_lmi)
    ref = _solve_oracle(G.g5_sigma_max_lmi)
    Y = res.x[1:].reshape(3, 3, order="F")
    assert res.status == "Solved" == ref.status and res.iter == ref.iter
    assert Y[1, 0] <= 4 + 1e-6 and Y[1, 1] >= 3 - 1e-6 and Y.sum() - 12.0 >= -1e-3
    assert abs(np.linalg.svd(Y, compute_uv=False).max() - res.x[0]) <= 1e-3 and abs(res.obj_val - ref.obj_val) < 1e-6
    # G11 moi_wrapper.jl:201-217: two iterations, ITERATION_LIMIT, rho never adapted
    res, _ = _solve_mine(G.g11_iteration_limit, max_iter=2)
    assert res.status == "Max_iter_reached" and res.iter == 2 and list(res.info.rho_updates) == [0.1]


def test_g6_chordal_sdp_through_the_clique_batch():
    # examples/chordal_decomposition.jl:7-23 with NoMerge: the documented cliques (docs/src/decomposition.md:43)
    # become five PsdConeTriangle blocks projected in one batched launch; optimum = the undecomposed optimum
    # (Agler), and the completed dual (complete_dual = true) is PSD.  Default tolerances first (both solve it), then
    # eps = 1e-7 (see below).
    from cosmo_b200 import chordal
    P, q, cons = G.g6_chordal_sdp()
    Pm, qm, A0, b0, cones0 = O.assemble(P, q, cons)
    sets0 = [cosmo_b200.PsdConeTriangle(45)]
    P2, q2, A2, b2, sets2, info = chordal.decompose(Pm, qm, A0, b0, sets0, merge="none")
    assert sorted(sorted(c.tolist()) for _, c in info.blocks[0]) == sorted(G.G6_CLIQUES)
    model = cosmo_b200.Model()
    model.set(P2, q2, A2, b2, sets2, cosmo_b200.Settings())
    dec = model.optimize()
    ref = O.solve(P2, q2, A2, b2, to_oracle_cones(sets2), O.Settings(kkt_solver="cg"))
    full = O.solve(Pm, qm, A0, b0, cones0, O.Settings(eps_abs=1e-7, eps_rel=1e-7))      # undecomposed, direct KKT
    assert dec.status == "Solved" == ref.status == full.status
    assert abs(dec.iter - ref.iter) <= 50 and abs(dec.obj_val - ref.obj_val) < 1e-4
    assert abs(dec.obj_val - full.obj_val) < 1e-3
    x, s, mu = chordal.reverse(info, dec.x, dec.s, -dec.y, complete_dual=True)
    assert np.allclose(x, full.x, atol=1e-3)
    assert np.linalg.eigvalsh(chordal._svec_to_mat(-mu, 9)).min() > -1e-3
    # eps = 1e-7 (the round-1 failure, root-caused): with the CG plugin the inexact KKT solves -- tolerance schedule
    # 1 / k^1.5 relative to |rhs|, kktsolver_indirect.jl:168-170 -- stall the residuals of this P = 0 problem near 1e-5.
    # Measured with the oracle on the CPU: CG -> Max_iter_reached after 5000 iterations (r_prim 1.04e-5, r_dual 1.95e-5,
    # also at eps = 1e-6), direct KKT solve -> Solved in 75 iterations.  The engine must agree with the CG oracle.
    tight = dict(eps_abs=1e-7, eps_rel=1e-7)
    model = cosmo_b200.Model()
    model.set(P2, q2, A2, b2, sets2, cosmo_b200.Settings(**tight))
    d7 = model.optimize()
    r7 = O.solve(P2, q2, A2, b2, to_oracle_cones(sets2), O.Settings(kkt_solver="cg", **tight))
    assert d7.status == r7.status == "Max_iter_reached" and d7.iter == r7.iter == 5000, (d7.status, d7.iter, r7.status, r7.iter)
    assert abs(d7.obj_val - r7.obj_val) < 1e-5 and d7.info.r_prim < 5e-5 and r7.info.r_prim < 5e-5, (d7.info.r_prim, r7.info.r_prim)
    # the same through the solver-level flags (Settings(decompose = true, merge_strategy, complete_dual))
    model = cosmo_b200.Model()
    cosmo_b200.assemble(model, P, q, _to_mine(cons), cosmo_b200.Settings(decompose=True, merge_strategy="NoMerge", complete_dual=True))
    res = model.optimize()
    assert res.status == "Solved" and res.iter == dec.iter and abs(res.obj_val - dec.obj_val) < 1e-9
    assert res.x.shape == (2,) and res.y.shape == (45,) and np.allclose(res.x, x, atol=1e-9) and np.allclose(res.y, -mu, atol=1e-9)


_AA_MINE = dict(accelerator="AndersonAccelerator")
_AA_REF = dict(accelerator="anderson")


@pytest.mark.parametrize("builder,x,obj,tol", [(G.g1_qp_nonneg, G.G1_X, G.G1_OBJ, 1e-3), (G.g1_qp_box, G.G1_X, G.G1_OBJ, 1e-3),
                                               (G.g12_lp, G.G12_X, G.G12_OBJ, 1e-2), (G.g3_hs21, G.G3_X, G.G3_OBJ, 1e-3),
                                               (G.g13_lovasz_petersen, None, G.G13_OBJ, 1e-3)])
def test_accelerated_solves_reach_the_reference_answers(builder, x, obj, tol):
    # the reference runs these with its default (accelerated) settings; the accelerated oracle is the comparison
    res, _ = _solve_mine(builder, **_AA_MINE)
    ref = _solve_oracle(builder, **_AA_REF)
    plain = _solve_oracle(builder)
    assert res.status == "Solved" == ref.status and abs(res.obj_val - obj) < tol
    if x is not None:
        assert np.max(np.abs(res.x - x)) < tol
    # with the inexact CG solves the accelerated trajectory is sensitive to rounding on the LP (P = 0): counts
    # are compared loosely, the answers tightly
    assert res.iter <= 1.5 * max(ref.iter, 25) + 30 and res.iter <= plain.iter + 1
    assert np.allclose(res.x, ref.x, atol=10 * tol)


def test_accelerated_statuses_and_exp_pow_problems():
    assert _solve_mine(G.g2_box_primal_infeasible_1, **_AA_MINE)[0].status == "Primal_infeasible"
    assert _solve_mine(G.g2_box_dual_infeasible, check_infeasibility=20, scaling=0, **_AA_MINE)[0].status == "Dual_infeasible"
    for name, builder, status, obj, atol, kw in G.G15_G16:
        res, _ = _solve_mine(builder, **kw, **_AA_MINE)
        assert res.status == status, name
        if obj is not None:
            assert abs(res.obj_val - obj) < atol, name


def test_accelerator_rho_adaption_limits():
    # AccelerationTests/max_rho_adaption.jl:21-36 with the accelerator on: exactly 2, then exactly 1 adaption
    res, _ = _solve_mine(G.g1_qp_nonneg, adaptive_rho_interval=25, adaptive_rho_max_adaptions=2, rho=1e-6, eps_abs=1e-6,
                         eps_rel=1e-4, **_AA_MINE)
    assert len(res.info.rho_updates) - 1 == 2
    res, _ = _solve_mine(G.g1_qp_nonneg, adaptive_rho_interval=25, adaptive_rho_max_adaptions=1, rho=1e-6, eps_abs=1e-4,
                         eps_rel=1e-4, **_AA_MINE)
    assert len(res.info.rho_updates) - 1 == 1


@pytest.mark.parametrize("scaling", [0, 10])
def test_g13_lovasz_petersen_sdp(scaling):
    res, _ = _solve_mine(G.g13_lovasz_petersen, scaling=scaling, eps_abs=1e-6, eps_rel=1e-6)
    ref = _solve_oracle(G.g13_lovasz_petersen, scaling=scaling, eps_abs=1e-6, eps_rel=1e-6)
    assert res.status == "Solved" and abs(res.obj_val - G.G13_OBJ) < 1e-3
    assert abs(res.obj_val - ref.obj_val) < 1e-6 and abs(res.iter - ref.iter) <= 25


def test_g14_model_updates_and_warm_start():
    P, q, cons = G.g1_qp_nonneg()
    model = cosmo_b200.Model()
    cosmo_b200.assemble(model, P, q, _to_mine(cons), cosmo_b200.Settings(check_termination=1))
    r1 = model.optimize()
    r2 = model.optimize()
    assert abs(r1.obj_val - r2.obj_val) <= 1e-3 and r2.iter <= r1.iter       # model_modifications.jl:29-31
    model = cosmo_b200.Model()
    cosmo_b200.assemble(model, P, q, _to_mine(cons), cosmo_b200.Settings())
    model.optimize()
    model.update(q=np.array([2.0, 3.0]))
    r = model.optimize()
    assert abs(r.obj_val - 3.5) < 1e-3 and np.linalg.norm(r.x - [0.5, 0.5]) < 1e-3   # :41-43
    model = cosmo_b200.Model()
    cosmo_b200.assemble(model, np.zeros((2, 2)), np.array([1.0, 1.0]),
                        cosmo_b200.Constraint(np.eye(2), np.array([-2.0, -3.0]), cosmo_b200.Nonnegatives),
                        cosmo_b200.Settings(check_termination=20))
    r = model.optimize()
    assert np.linalg.norm(r.x - [2.0, 3.0]) < 1e-3
    model.update(b=np.array([0.0, 1.0]))
    assert np.linalg.norm(model.optimize().x - [0.0, -1.0]) < 1e-4               # :57-59


# ---------------------------------------------------------------------------
# solve-level parity on the BASELINE problem families at oracle-sized instances
# ---------------------------------------------------------------------------
def _parity(P, q, A, b, sets, tol_x=1e-5, **kw):
    cones = to_oracle_cones(sets)
    ref = O.solve(P, q, A, b, cones, O.Settings(kkt_solver="cg", **kw))
    model = cosmo_b200.Model()
    model.set(P, q, A, b, sets, cosmo_b200.Settings(**kw))
    res = model.optimize()
    assert res.status == ref.status
    scale = max(1.0, np.abs(ref.x).max())
    assert abs(res.obj_val - ref.obj_val) <= 1e-6 * max(1.0, abs(ref.obj_val)) * 10
    assert np.max(np.abs(res.x - ref.x)) <= tol_x * scale
    assert np.max(np.abs(res.s - ref.s)) <= tol_x * max(1.0, np.abs(ref.s).max())
    assert np.max(np.abs(res.y - ref.y)) <= tol_x * max(1.0, np.abs(ref.y).max())
    return res, ref


@pytest.mark.parametrize("scaling", [0, 10])
def test_c2_random_sparse_qp_small(scaling):
    P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(2000, 4000, 0.01, seed=2)
    res, ref = _parity(P, q, A, b, sets, scaling=scaling)
    assert res.status == "Solved" and res.iter == ref.iter


def test_c3_portfolio_socp_small():
    P, q, A, b, sets = cosmo_b200.problems.portfolio_socp(n=400, k=40, seed=1)
    res, ref = _parity(P, q, A, b, sets, tol_x=1e-4, max_iter=3000)
    assert res.status == "Solved"


def test_c4_closest_correlation_small():
    P, q, A, b, sets = cosmo_b200.problems.closest_correlation_sdp(N=40, seed=12345)
    res, ref = _parity(P, q, A, b, sets, tol_x=1e-4)
    assert res.status == "Solved"
    N = 40
    X = np.zeros((N, N))
    iu = np.triu_indices(N)
    order = np.lexsort((iu[0], iu[1]))
    r, c = iu[0][order], iu[1][order]
    X[r, c] = np.where(r == c, res.x, res.x / np.sqrt(2))
    X = X + np.triu(X, 1).T
    assert np.max(np.abs(np.diag(X) - 1.0)) < 1e-4 and np.linalg.eigvalsh(X).min() > -1e-3   # closestcorr.jl:70-80


def test_float32_model_solves_g1():
    # Model{Float32} (test/run_cosmo_tests.jl:9); tolerance of the reference's own test: 1e-3
    P, q, cons = G.g1_qp_box()
    model = cosmo_b200.Model(dtype=np.float32)
    cosmo_b200.assemble(model, P, q, _to_mine(cons), cosmo_b200.Settings(eps_abs=1e-4, eps_rel=1e-4))
    res = model.optimize()
    assert res.status == "Solved" and np.max(np.abs(res.x - G.G1_X)) < 1e-3 and abs(res.obj_val - G.G1_OBJ) < 1e-3


def test_c5_maxcut_chordal_clique_batch():
    """config C5 at oracle size: dual MAXCUT SDP, host chordal decomposition, every clique a
    PsdConeTriangle projected in one batched launch; engine vs oracle on the SAME decomposed problem,
    and decomposed vs undecomposed optimum (Agler)."""
    from cosmo_b200 import chordal
    nv = 120
    rows, cols, w = cosmo_b200.problems.banded_random_graph(nv, 3.0, 6, seed=3)
    P, q, A, b, sets = cosmo_b200.problems.maxcut_dual_sdp(nv, rows, cols, w)
    P2, q2, A2, b2, sets2, info = chordal.decompose(P, q, A, b, sets, merge="parent_child")
    assert len(sets2) > 10
    res, ref = _parity(P2, q2, A2, b2, sets2, tol_x=1e-4, eps_abs=1e-6, eps_rel=1e-6)
    assert res.status == "Solved" and abs(res.iter - ref.iter) <= 25
    full = O.solve(P, q, A, b, to_oracle_cones(sets), O.Settings(kkt_solver="cg", eps_abs=1e-6, eps_rel=1e-6))
    assert abs(full.obj_val - res.obj_val) <= 1e-3 * max(1.0, abs(full.obj_val))
    x, s, mu = chordal.reverse(info, res.x, res.s, -res.y)
    assert np.max(np.abs(A @ x + s - b)) < 1e-3


def test_simple_statuses_and_warm_start():
    """test/UnitTests/simple.jl:58-124: Max_iter_reached (max_iter / huge check_termination),
    Time_limit_reached, warm start gives fewer iterations."""
    P, q, cons = G.g1_qp_nonneg()

    def run(**kw):
        model = cosmo_b200.Model()
        cosmo_b200.assemble(model, P, q, _to_mine(cons), cosmo_b200.Settings(**kw))
        return model, model.optimize()

    assert run(max_iter=20)[1].status == "Max_iter_reached"                     # :58-66
    assert run(check_termination=100000)[1].status == "Max_iter_reached"        # :70-80
    assert run(time_limit=0.2, check_termination=100000000, max_iter=10000000)[1].status == "Time_limit_reached"  # :82-90
    m1, r1 = run(check_termination=1)
    m2 = cosmo_b200.Model()
    cosmo_b200.assemble(m2, P, q, _to_mine(cons), cosmo_b200.Settings(check_termination=1))
    m2.warm_start_primal(r1.x)
    m2.warm_start_dual(r1.y)
    assert np.array_equal(m2.x, r1.x) and np.array_equal(m2.mu, -r1.y) and np.linalg.norm(m2.s - r1.s) < 1e-4   # :107-110
    rng = np.random.default_rng(0)
    m2.warm_start_primal(r1.x + 0.01 * rng.random(2))
    m2.warm_start_dual(r1.y + 0.01 * rng.random(6))
    r2 = m2.optimize()
    # the reference asserts res2.iter < res1.iter with its direct QDLDL solver (:118); with the inexact CG
    # solver a fresh handle restarts the tolerance schedule tol_k = 1/k^1.5, so only the statuses and the
    # solution are compared here
    assert r1.status == "Solved" and r2.status == "Solved" and np.max(np.abs(r2.x - r1.x)) < 1e-3
    with pytest.raises(ValueError):
        m2.warm_start_primal(rng.random(4))


def test_automatic_rho_interval_and_result_times():
    """settings.adaptive_rho_interval = 0 (solver.jl:244-256): the interval is fixed once the loop has run for
    adaptive_rho_fraction * setup_time, rounded to a multiple of check_termination; ResultTimes.proj_time / kkt_time
    (types.jl:26-41) are filled from device timers under verbose_timing."""
    P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(400, 700, 0.05, seed=3)
    model = cosmo_b200.Model()
    model.set(P, q, A, b, sets, cosmo_b200.Settings(adaptive_rho=True, adaptive_rho_interval=0, adaptive_rho_fraction=1e-9,
                                                    check_termination=25, verbose_timing=True, scaling=0))
    res = model.optimize()
    ref = O.solve(P, q, A, b, to_oracle_cones(sets), O.Settings(kkt_solver="cg", scaling=0, adaptive_rho_interval=25))
    assert res.status == "Solved"
    # with a vanishing fraction the rule fires at iteration 1: interval = max(round_multiple(1, 25), 25) = 25, i.e. the
    # run is the oracle's run with adaptive_rho_interval = 25
    assert res.iter == ref.iter and len(res.info.rho_updates) == len(ref.info.rho_updates)
    assert np.allclose(res.info.rho_updates, ref.info.rho_updates, rtol=1e-6)
    assert abs(res.obj_val - ref.obj_val) <= 1e-6 * max(1.0, abs(ref.obj_val))
    t = res.times
    assert t["proj_time"] > 0 and t["kkt_time"] > 0 and t["proj_time"] + t["kkt_time"] <= 1.05 * t["iter_time_device"]
    # never firing: fraction so large that the interval stays automatic -> no rho update at all
    model2 = cosmo_b200.Model()
    model2.set(P, q, A, b, sets, cosmo_b200.Settings(adaptive_rho=True, adaptive_rho_interval=0, adaptive_rho_fraction=1e9, scaling=0))
    res2 = model2.optimize()
    assert len(res2.info.rho_updates) == 1


@pytest.mark.parametrize("prob", ["qp_box", "socp", "sdp", "qp_wide"])
def test_device_ruiz_matches_oracle(prob):
    """scale_ruiz! on the device (csrc/ruiz.cuh; scaling.jl:21-116): unscaled data in, D / E / c and the scaled resident
    copies of A, A', P out -- against the oracle's restatement (which is pinned on the reference's known answers)."""
    pr = cosmo_b200.problems
    if prob == "qp_box":
        P, q, A, b, sets = pr.random_sparse_qp(300, 500, 0.05, seed=0)
    elif prob == "socp":
        P, q, A, b, sets = pr.portfolio_socp(n=200, k=20, seed=2)
    elif prob == "sdp":
        P, q, A, b, sets = pr.closest_correlation_sdp(N=20, seed=7)
    else:   # wide enough for the column-windowed slabs (ncols * 8 B > 200 KB)
        P, q, A, b, sets = pr.random_sparse_qp(30000, 4000, 0.002, seed=5)
    st = cosmo_b200.Settings()          # scaling = 10
    eng = E.Engine(P, q, A, b, _tuples(sets), st.to_struct(), equilibrate=True)   # unscaled data in, scale_ruiz! on the device
    D, Ev, c = eng.scaling()
    Ps, qs, As, bs, cones, sm = O.scale_ruiz(P, q, A, b, to_oracle_cones(sets), O.Settings())
    assert np.max(np.abs(D - sm.D) / sm.D) <= 1e-13
    assert np.max(np.abs(Ev - sm.E) / sm.E) <= 1e-13
    assert abs(c - sm.c) <= 1e-13 * sm.c
    rng = np.random.default_rng(1)
    x, y = rng.standard_normal(A.shape[1]), rng.standard_normal(A.shape[0])
    for which, got_in, ref in ((0, x, As @ x), (1, y, As.T @ y), (2, x, Ps @ x)):
        got = eng.spmv(which, got_in)
        assert np.max(np.abs(got - ref)) <= 1e-12 * max(1.0, np.max(np.abs(ref))), which
    # a full default-settings solve through the host mirror agrees with the oracle (status, iterations, solution)
    model = cosmo_b200.Model()
    model.set(P, q, A, b, sets, st)
    res = model.optimize()
    ref = O.solve(P, q, A, b, to_oracle_cones(sets), O.Settings(kkt_solver="cg"))
    assert res.status == ref.status and abs(res.iter - ref.iter) <= 25
    assert abs(res.obj_val - ref.obj_val) <= 1e-4 * max(1.0, abs(ref.obj_val))


def test_c4_closest_correlation_through_the_tensor_core_projection():
    """Config C4 at N = 256 (one PsdConeTriangle projected by psd_tc.cuh in every iteration), default settings incl. the
    device Ruiz scaling, run to Solved: status, iteration count, x / s / y and objective against the oracle (dsyevr),
    the closestcorr.jl:70-80 properties, and no fallback to block Jacobi in any of the projections."""
    N = 256
    P, q, A, b, sets = cosmo_b200.problems.closest_correlation_sdp(N=N, seed=12345)
    res, ref = _parity(P, q, A, b, sets, tol_x=1e-4)
    assert res.status == "Solved" and res.iter == ref.iter
    X = np.zeros((N, N))
    iu = np.triu_indices(N)
    order = np.lexsort((iu[0], iu[1]))
    r, c = iu[0][order], iu[1][order]
    X[r, c] = np.where(r == c, res.x, res.x / np.sqrt(2))
    X = X + np.triu(X, 1).T
    assert np.max(np.abs(np.diag(X) - 1.0)) < 1e-4 and np.linalg.eigvalsh(X).min() > -1e-3
    model = cosmo_b200.Model()
    model.set(P, q, A, b, sets, cosmo_b200.Settings())
    out = model.optimize()
    st = model.engine.psd_stats()
    assert st["tc_projections"] >= out.iter and st["tc_fallbacks"] == 0, st
    assert out.times["proj_time"] > 0.5 * out.times["iter_time_device"]      # the projection is the step here


def test_psd_tensor_core_large_and_fallback(monkeypatch):
    """N = 1500 (12 x 12 tiles, 78 in the upper triangle) at the LAPACK bar; then the fallback: with the step cap forced to
    3 the Newton-Schulz iteration cannot converge, the engine must fall back to block Jacobi and still be right."""
    rng = np.random.default_rng(5)
    N = 1500
    X = _psd_test_matrix("admm_like", N, rng)
    sets = [cosmo_b200.PsdConeTriangle(N * (N + 1) // 2)]
    ws = G._svec(X)
    eng = _engine(sp.identity(1, format="csc"), np.zeros(1), sp.csc_matrix((ws.size, 1)), np.zeros(ws.size), sets)
    ref = ws.copy()
    O.project(ref, to_oracle_cones(sets))
    got = eng.project(ws)
    st = eng.psd_stats()
    assert st["tc_projections"] == 1 and st["tc_fallbacks"] == 0, st
    assert np.linalg.norm(got - ref) / np.linalg.norm(ws) < 1e-12, st
    eng.close()
    monkeypatch.setenv("COSMO_B200_TC_MAX_STEPS", "3")
    N = 200
    X = _psd_test_matrix("wigner", N, rng)
    sets = [cosmo_b200.PsdConeTriangle(N * (N + 1) // 2)]
    ws = G._svec(X)
    eng = _engine(sp.identity(1, format="csc"), np.zeros(1), sp.csc_matrix((ws.size, 1)), np.zeros(ws.size), sets)
    ref = ws.copy()
    O.project(ref, to_oracle_cones(sets))
    got = eng.project(ws)
    st = eng.psd_stats()
    assert st["tc_projections"] == 0 and st["tc_fallbacks"] == 1, st
    assert np.linalg.norm(got - ref) / np.linalg.norm(ws) < 1e-12


def test_block_jacobi_non_convergence_is_a_numerical_error(monkeypatch):
    """tensor cores off and psd_max_sweeps = 1 on a Wigner matrix of side 150: block Jacobi misses the sweep cap, and
    project() and solve() fail with ERR_NUMERICAL, as the reference fails when LAPACK does not converge
    (convexset.jl:186)."""
    monkeypatch.setenv("COSMO_B200_PSD_TC", "0")
    N = 150
    ws = G._svec(_psd_test_matrix("wigner", N, np.random.default_rng(60)))
    sets = [cosmo_b200.PsdConeTriangle(N * (N + 1) // 2)]
    eng = _engine(sp.identity(1, format="csc"), np.zeros(1), sp.csc_matrix((ws.size, 1)), ws, sets, psd_max_sweeps=1)
    for call in (lambda: eng.project(ws), eng.solve):
        with pytest.raises(E.EngineError) as ei:
            call()
        assert ei.value.code == E.ERR_NUMERICAL, ei.value
        assert "block Jacobi eigensolver did not converge within psd_max_sweeps" in str(ei.value)
    eng.close()


@pytest.mark.parametrize("Nc,kind", [(49, "shifted"), (100, "wigner"), (100, "low_rank_plus_noise"), (193, "shifted")])
def test_complex_psd_cone_large_through_the_tensor_core_path(Nc, kind):
    """PsdConeTriangle{T, Complex{T}} beyond the shared-memory path (2 Nc > 96): the real embedding [[A, -B], [B, A]]
    goes through the same tensor-core projection as a real cone of side 2 Nc; against numpy's Hermitian eigh."""
    rng = np.random.default_rng(1000 + Nc)
    ws, H = _hermitian_ws(Nc, rng, kind)
    sets = [cosmo_b200.ComplexPsdConeTriangle(Nc * Nc)]
    eng = _engine(sp.identity(1, format="csc"), np.zeros(1), sp.csc_matrix((ws.size, 1)), np.zeros(ws.size), sets)
    got = eng.project(ws)
    st = eng.psd_stats()
    assert st["tc_projections"] == 1 and st["tc_fallbacks"] == 0, st
    ref = ws.copy()
    O.project(ref, to_oracle_cones(sets))
    lam, U = np.linalg.eigh(H)
    truth = O.extract_upper_triangle_complex((U * np.maximum(lam, 0.0)) @ U.conj().T, np.sqrt(2.0))
    assert np.linalg.norm(ref - truth) / np.linalg.norm(ws) < 1e-12          # the oracle is the Hermitian eigh
    assert np.linalg.norm(got - ref) / np.linalg.norm(ws) < 1e-12, st
    # idempotent, and the imaginary diagonal stays out of the picture
    again = eng.project(got)
    assert np.linalg.norm(again - got) / np.linalg.norm(ws) < 1e-12


def test_complex_psd_cone_large_block_jacobi_fallback_and_solve(monkeypatch):
    """the same cone through the fallback eigensolver (Newton-Schulz capped at 3 steps), and a solve: the least
    eigenvalue of a 60 x 60 Hermitian matrix as an SDP (least_eigenvalue.jl:33-39 at a size beyond the small path)."""
    rng = np.random.default_rng(77)
    Nc = 60
    ws, H = _hermitian_ws(Nc, rng, "wigner")
    sets = [cosmo_b200.ComplexPsdConeTriangle(Nc * Nc)]
    monkeypatch.setenv("COSMO_B200_TC_MAX_STEPS", "3")
    eng = _engine(sp.identity(1, format="csc"), np.zeros(1), sp.csc_matrix((ws.size, 1)), np.zeros(ws.size), sets)
    got = eng.project(ws)
    st = eng.psd_stats()
    assert st["tc_projections"] == 0 and st["tc_fallbacks"] == 1, st
    ref = ws.copy()
    O.project(ref, to_oracle_cones(sets))
    assert np.linalg.norm(got - ref) / np.linalg.norm(ws) < 1e-12
    eng.close()
    monkeypatch.delenv("COSMO_B200_TC_MAX_STEPS")
    # max t  s.t.  H - t I  in the Hermitian PSD cone:  x = t, minimise -t, A x + s = b with A = svec(I), b = svec(H)
    eye = O.extract_upper_triangle_complex(np.eye(Nc, dtype=complex), np.sqrt(2.0))
    A = sp.csc_matrix(eye.reshape(-1, 1))
    P = sp.csc_matrix((1, 1))
    q = np.array([-1.0])
    m1 = cosmo_b200.Model()
    m1.set(P, q, A, ws, sets, cosmo_b200.Settings())
    res = m1.optimize()
    # the engine's KKT solver is CG with the reference's tolerance schedule: the run to compare with is the oracle's CG
    # run (4725 iterations, 16 rho updates; with the direct solver the oracle needs 3100 -- a 1.3 % difference in the
    # first rho update is enough on this slowly converging problem)
    ref = O.solve(P, q, A, ws, to_oracle_cones(sets), O.Settings(kkt_solver="cg"))
    assert res.status == "Solved" == ref.status and res.iter == ref.iter
    assert np.allclose(res.info.rho_updates, ref.info.rho_updates, rtol=1e-6)
    assert abs(res.x[0] - ref.x[0]) < 1e-8 * abs(ref.x[0])
    assert abs(res.x[0] - np.linalg.eigvalsh(H)[0]) < 1e-3 * abs(ref.x[0])


@pytest.mark.parametrize("scaling", [0, 10])
def test_obj_true_joins_the_convergence_test(scaling):
    """settings.obj_true / obj_true_tol (residuals.jl:127-140): with a known optimal value the run only stops once the
    cost is within obj_true_tol of it as well -- the reference's examples/qp.jl (optimum 1.88)."""
    plain, _ = _solve_mine(G.g1_qp_nonneg, scaling=scaling)
    # (with the CG solver's inexact inner solves the cost stalls near 1e-7 of the optimum: 1e-6 is reachable, 1e-8 is not)
    for kw in (dict(obj_true=1.88, obj_true_tol=1e-3), dict(obj_true=1.88, obj_true_tol=1e-6),
               dict(obj_true=2.88, obj_true_tol=1e-3, max_iter=300)):
        res, _ = _solve_mine(G.g1_qp_nonneg, scaling=scaling, **kw)
        ref = _solve_oracle(G.g1_qp_nonneg, scaling=scaling, **kw)
        assert res.status == ref.status and res.iter == ref.iter, (kw, res.status, res.iter, ref.iter)
        assert abs(res.obj_val - ref.obj_val) < 1e-9
        if kw["obj_true"] == 1.88:
            assert res.status == "Solved" and abs(res.obj_val - 1.88) <= kw["obj_true_tol"]
    loose, _ = _solve_mine(G.g1_qp_nonneg, scaling=scaling, obj_true=1.88, obj_true_tol=1e-3)
    tight, _ = _solve_mine(G.g1_qp_nonneg, scaling=scaling, obj_true=1.88, obj_true_tol=1e-6)
    wrong, _ = _solve_mine(G.g1_qp_nonneg, scaling=scaling, obj_true=2.88, obj_true_tol=1e-3, max_iter=300)
    assert loose.iter == plain.iter and tight.iter > plain.iter and wrong.status == "Max_iter_reached" and wrong.iter == 300
