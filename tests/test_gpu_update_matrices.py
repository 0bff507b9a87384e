"""cosmo_b200_update_matrices: new values of P and A on the resident pattern leave the engine bit for bit where a new
engine with the new data would start.

Each case creates E1 with data D1, solves, updates it to D2 and solves again from a warm start w0; E2 is created with D2
and solves from the same w0.  Iterates, scalars, the operator products, the scaling and the rho vector must agree to
the bit.  Windowing both A and A' needs more than 25 600 fp64 columns (51 200 fp32) in each and at least 24 entries per
row segment; the setup report (COSMO_B200_SETUP_DEBUG) says which layout every slab got."""
import numpy as np
import pytest
import scipy.sparse as sp

import cosmo_b200
from cosmo_b200 import engine as E
from tests.gpu_helpers import _tuples
from tests.test_gpu_packed_slabs import PACKED, PLAIN, _assert_layout_rule, _count, _kernel_counts, _layouts, _ruiz_scaled

pytestmark = pytest.mark.gpu


def _new_values(P, A, seed, escapes=False):
    """the same pattern with new values: P = D P D for a positive diagonal D (still symmetric PSD), A Gaussian; with
    `escapes` 2 % of A's entries are tiny (~1e-30), outside the 14-binade window: the 9 B layout no longer pays"""
    rng = np.random.default_rng(seed)
    d = rng.uniform(0.5, 2.0, P.shape[0])
    P2, A2 = P.copy(), A.copy()
    P2.data = P.data * d[P.indices] * d[np.repeat(np.arange(P.shape[1]), np.diff(P.indptr))]
    A2.data = rng.standard_normal(A.nnz)
    if escapes:
        k = rng.choice(A.nnz, A.nnz // 50, replace=False)
        A2.data[k] *= 1e-30
    return P2, A2


def _problem(n, m, density, seed, escapes=False):
    P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(n, m, density, seed=seed)
    P.sort_indices()
    A.sort_indices()
    if escapes:
        P, A = _new_values(P, A, seed + 100, escapes=True)
    return P, q, A, b, sets


def _cone_problem(seed):
    """small (CSR-only) problem with Box + SOC + PSD rows"""
    rng = np.random.default_rng(seed)
    n, nb, nsoc, N = 40, 30, 12, 6
    npsd = N * (N + 1) // 2
    m = nb + nsoc + npsd
    A = sp.random(m, n, density=0.3, random_state=seed, data_rvs=rng.standard_normal, format="csc")
    B = sp.random(n, n, density=0.1, random_state=seed + 1, format="csr")
    P = (B @ B.T + sp.identity(n)).tocsc()
    P.sort_indices()
    A.sort_indices()
    q = rng.standard_normal(n)
    b = rng.standard_normal(m)
    sets = [cosmo_b200.Box(-np.ones(nb), np.ones(nb)), cosmo_b200.SecondOrderCone(nsoc), cosmo_b200.PsdConeTriangle(npsd)]
    return P, q, A, b, sets


def _settings(**kw):
    base = dict(scaling=0, max_iter=60, eps_abs=1e-12, eps_rel=1e-12)
    base.update(kw)
    return cosmo_b200.Settings(**base).to_struct()


def _create(P, q, A, b, sets, st, dtype, equilibrate):
    return E.Engine(P, q, A, b, _tuples(sets), st, dtype=dtype, equilibrate=equilibrate)


def _warm(n, m, dtype, seed=7):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal(n).astype(dtype), np.abs(rng.standard_normal(m)).astype(dtype),
            (0.1 * rng.standard_normal(m)).astype(dtype))


def _bits(v):
    return np.asarray(v).tobytes()


def _assert_same(e1, o1, e2, o2, seed=3):
    for f in ("x", "s", "mu"):
        assert _bits(getattr(o1, f)) == _bits(getattr(o2, f)), f
    assert _bits(np.float64(o1.obj_val)) == _bits(np.float64(o2.obj_val))
    assert (o1.iter, o1.status, o1.kkt_inner_iterations) == (o2.iter, o2.status, o2.kkt_inner_iterations)
    assert _bits(o1.rho_updates) == _bits(o2.rho_updates)
    rng = np.random.default_rng(seed)
    x, y = rng.standard_normal(e1.n), rng.standard_normal(e1.m)
    for which, v in ((0, x), (1, y), (2, x)):
        assert _bits(e1.spmv(which, v)) == _bits(e2.spmv(which, v)), which
    D1, E1, c1 = e1.scaling()
    D2, E2, c2 = e2.scaling()
    assert _bits(D1) == _bits(D2) and _bits(E1) == _bits(E2) and c1 == c2
    assert _bits(e1.rho_vec()) == _bits(e2.rho_vec())


def _update(eng, P2, q2, A2, b2, equilibrate):
    if equilibrate:
        eng.update_matrices(P2.data, A2.data, q2, b2)
    else:
        eng.update_matrices(P2.data, A2.data)


def _pair(D1, D2, st, dtype=np.float64, equilibrate=False, capfd=None):
    """(E1 updated D1 -> D2, its solve, E2 created with D2, its solve[, layouts reported by the update, by E2's create])"""
    P1, q1, A1, b1, sets = D1
    P2, q2, A2, b2, _ = D2
    e1 = _create(P1, q1, A1, b1, sets, st, dtype, equilibrate)
    e1.solve()
    if capfd is not None:
        capfd.readouterr()
    _update(e1, P2, q2, A2, b2, equilibrate)
    lay1 = _layouts(capfd) if capfd is not None else None
    w0 = _warm(e1.n, e1.m, dtype)
    e1.warm_start(*w0)
    o1 = e1.solve()
    e2 = _create(P2, q2, A2, b2, sets, st, dtype, equilibrate)
    lay2 = _layouts(capfd) if capfd is not None else None
    e2.warm_start(*w0)
    o2 = e2.solve()
    return e1, o1, e2, o2, lay1, lay2


def _assert_spmv_kernel(eng, layout, tmp_path):
    """the spmv_win_kernel instantiation of the layout runs, the other never does.  A torch.profiler capture can come
    back without the kernels of the window (see _kernel_counts), so a capture that misses both is taken again."""
    want, other = (PACKED, PLAIN) if layout == "9 B" else (PLAIN, PACKED)
    for attempt in range(3):
        try:
            counts = _kernel_counts(lambda: eng.spmv(0, np.ones(eng.n)), tmp_path)
        except AssertionError:          # an empty trace
            counts = {}
        if _count(counts, want) + _count(counts, other) > 0:
            break
    assert _count(counts, want) > 0 and _count(counts, other) == 0, counts


# (D1 escape-heavy, D2 escape-heavy, expected layouts after the update)
WINDOWED = {
    "packed": (False, False, "9 B"),
    "plain_10B": (True, True, "10 B"),
    "flip_to_10B": (False, True, "10 B"),
    "flip_to_9B": (True, False, "9 B"),
}


@pytest.mark.parametrize("case", list(WINDOWED))
def test_windowed_fp64_update_is_bit_identical(case, capfd, monkeypatch, tmp_path):
    esc1, esc2, layout = WINDOWED[case]
    monkeypatch.setenv("COSMO_B200_SETUP_DEBUG", "1")
    D1 = _problem(30000, 40000, 0.002, seed=4, escapes=esc1)
    P, q, A, b, sets = D1
    P2, A2 = _new_values(P, A, seed=5, escapes=esc2)
    e1, o1, e2, o2, lay1, lay2 = _pair(D1, (P2, q, A2, b, sets), _settings(), capfd=capfd)
    assert [l[0] for l in lay2] == [layout, layout], lay2
    assert lay1 == lay2                                    # layout, ebase and escape count as create chooses them
    _assert_same(e1, o1, e2, o2)
    _assert_spmv_kernel(e1, layout, tmp_path)
    e1.close()
    e2.close()


def test_windowed_fp32_update_is_bit_identical(capfd, monkeypatch):
    monkeypatch.setenv("COSMO_B200_SETUP_DEBUG", "1")
    D1 = _problem(60000, 60000, 0.001, seed=6)
    P, q, A, b, sets = D1
    P2, A2 = _new_values(P, A, seed=8)
    e1, o1, e2, o2, lay1, lay2 = _pair(D1, (P2, q, A2, b, sets), _settings(max_iter=40), dtype=np.float32, capfd=capfd)
    assert [l[0] for l in lay2] == ["6 B", "6 B"] and lay1 == lay2, (lay1, lay2)
    _assert_same(e1, o1, e2, o2)
    e1.close()
    e2.close()


def test_device_equilibration_update_is_bit_identical_on_scaled_slabs(capfd, monkeypatch):
    monkeypatch.setenv("COSMO_B200_SETUP_DEBUG", "1")
    D1 = _problem(30000, 40000, 0.002, seed=9)
    P, q, A, b, sets = D1
    P2, A2 = _new_values(P, A, seed=10)
    rng = np.random.default_rng(11)
    q2, b2 = rng.standard_normal(len(q)), b + rng.uniform(0.0, 0.5, len(b))
    e1, o1, e2, o2, lay1, lay2 = _pair(D1, (P2, q2, A2, b2, sets), _settings(scaling=10), equilibrate=True, capfd=capfd)
    D, Ev, _ = e2.scaling()
    _assert_layout_rule(_ruiz_scaled(A2, D, Ev), lay2)          # the slabs are filled from the scaled values
    assert lay1 == lay2, (lay1, lay2)
    assert not np.all(e1.scaling()[0] == 1.0)
    _assert_same(e1, o1, e2, o2)
    e1.close()
    e2.close()


@pytest.mark.parametrize("solver", ["MINRESIndirectKKTSolver", "DeviceLdlKKTSolver", "CGIndirectKKTSolver"])
def test_kkt_solvers_and_cones_update_is_bit_identical(solver):
    D1 = _cone_problem(1)
    P, q, A, b, sets = D1
    P2, A2 = _new_values(P, A, seed=2)
    e1, o1, e2, o2, _, _ = _pair(D1, (P2, q, A2, b, sets), _settings(kkt_solver=solver, max_iter=200))
    _assert_same(e1, o1, e2, o2)
    e1.close()
    e2.close()


def test_update_chain_returns_to_a_fresh_engine(capfd, monkeypatch):
    monkeypatch.setenv("COSMO_B200_SETUP_DEBUG", "1")
    P, q, A, b, sets = _problem(30000, 40000, 0.002, seed=14)
    P2, A2 = _new_values(P, A, seed=15, escapes=True)
    P3, A3 = _new_values(P, A, seed=16)
    st = _settings()
    e1 = _create(P, q, A, b, sets, st, np.float64, False)
    lay_fresh = _layouts(capfd)
    for Pk, Ak in ((P2, A2), (P3, A3), (P, A)):
        e1.solve()
        e1.update_matrices(Pk.data, Ak.data)
    assert _layouts(capfd)[-2:] == lay_fresh
    e2 = _create(P, q, A, b, sets, st, np.float64, False)
    w0 = _warm(e1.n, e1.m, np.float64)
    e1.warm_start(*w0)
    e2.warm_start(*w0)
    _assert_same(e1, e1.solve(), e2, e2.solve())
    e1.close()
    e2.close()


def test_errors_leave_the_engine_usable():
    P, q, A, b, sets = _cone_problem(3)
    st = _settings(max_iter=100)
    w0 = _warm(A.shape[1], A.shape[0], np.float64)
    ref = _create(P, q, A, b, sets, st, np.float64, False)
    ref.warm_start(*w0)
    o_ref = ref.solve()
    eng = _create(P, q, A, b, sets, st, np.float64, False)
    eng.warm_start(*w0)
    with pytest.raises(E.EngineError) as ei:
        eng.update_matrices(Ax=A.data[:-1])
    assert ei.value.code == E.ERR_INVALID
    _assert_same(eng, eng.solve(), ref, o_ref)
    eng.close()
    ref.close()
    # an equilibrating engine restarts Ruiz from the unscaled data: q and b must come along
    eq = _create(P, q, A, b, sets, _settings(scaling=10), np.float64, True)
    with pytest.raises(E.EngineError) as ei:
        eq.update_matrices(P.data, A.data)
    assert ei.value.code == E.ERR_INVALID
    eq.close()
    # the LDL' factorisation runs inside the update: a non-convex P fails like create does
    ldl = _create(P, q, A, b, sets, _settings(kkt_solver="DeviceLdlKKTSolver"), np.float64, False)
    with pytest.raises(E.EngineError) as ei:
        ldl.update_matrices(Px=-P.data)
    assert ei.value.code == E.ERR_INVALID and "not convex" in str(ei.value)
    ldl.close()


def test_model_update_matches_a_fresh_model():
    P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(300, 400, 0.05, seed=17)
    P2, A2 = _new_values(sp.csc_matrix(P), sp.csc_matrix(A), seed=18)
    q2 = np.random.default_rng(19).standard_normal(len(q))
    st = dict(max_iter=300)
    m1 = cosmo_b200.Model()
    m1.set(P, q, A, b, sets, cosmo_b200.Settings(**st))
    m1.optimize()
    x, s, mu = m1.x.copy(), m1.s.copy(), m1.mu.copy()
    engine = m1.engine
    m1.update(q=q2, P=P2, A=A2)
    assert m1.engine is engine
    r1 = m1.optimize()
    m2 = cosmo_b200.Model()
    m2.set(P2, q2, A2, b, sets, cosmo_b200.Settings(**st))
    m2.x[:], m2.s[:], m2.mu[:] = x, s, mu
    r2 = m2.optimize()
    for f in ("x", "y", "s"):
        assert _bits(getattr(r1, f)) == _bits(getattr(r2, f)), f
    assert (r1.obj_val, r1.iter, r1.status, r1.info.rho_updates) == (r2.obj_val, r2.iter, r2.status, r2.info.rho_updates)
    m1.empty_model()
    m2.empty_model()
