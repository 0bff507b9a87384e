"""The traditional transformation (compact_transformation = false) on the device: the reverse of
cosmo_b200_set_decomposition_noncompact against chordal.reverse, solves of the decomposed problem against the oracle,
and in-place updates of a traditionally decomposed model against a fresh one."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp

import cosmo_b200
from cosmo_b200 import chordal, engine as E
from oracle import cosmo_oracle as O
from oracle.bridge import to_oracle_cones
from tests import test_chordal_traditional_cpu as T

pytestmark = pytest.mark.gpu

M = cosmo_b200.model


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


def square_twin(A, b, N, off=0):
    """the PsdCone(N^2) form of a problem whose rows off.. are one PsdConeTriangle(N(N+1)/2): row i + N j takes the
    triangle row of (min, max), divided by sqrt 2 off the diagonal"""
    A = sp.csr_matrix(A)
    i, j = np.arange(N * N) % N, np.arange(N * N) // N
    lo, hi = np.minimum(i, j), np.maximum(i, j)
    src = off + hi * (hi + 1) // 2 + lo
    scale = np.where(i == j, 1.0, 1.0 / np.sqrt(2.0))
    rows = np.concatenate([np.arange(off), src, np.arange(off + N * (N + 1) // 2, A.shape[0])])
    sc = np.concatenate([np.ones(off), scale, np.ones(A.shape[0] - off - N * (N + 1) // 2)])
    return sp.csc_matrix(sp.diags(sc) @ A[rows]), sc * np.asarray(b)[rows]


def _maxcut(nv, square=False):
    rows, cols, w = cosmo_b200.problems.banded_random_graph(nv, 3.0, 20, seed=1)
    P, q, A, b, sets = cosmo_b200.problems.maxcut_dual_sdp(nv, rows, cols, w)
    if not square:
        return P, q, A, b, sets
    A, b = square_twin(A, b, nv)
    return P, q, A, b, [M.PsdCone(nv * nv)]


PROBLEMS = {
    "four_cone": T.four_cone_problem,
    "four_cone_triangle": lambda: T.four_cone_problem(triangle=True),
    "mixed": T.mixed_problem,
    "maxcut200": lambda: _maxcut(200),
    "maxcut200_square": lambda: _maxcut(200, square=True),
}


def _model(name, **settings):
    dtype = settings.pop("dtype", np.float64)
    model = cosmo_b200.Model(dtype=dtype)
    model.set(*PROBLEMS[name](), cosmo_b200.Settings(decompose=True, compact_transformation=False, **settings))
    return model


def test_square_twin_is_the_same_problem():
    P, q, A, b, sets = _maxcut(200)
    As, bs = square_twin(A, b, 200)
    x = np.random.default_rng(0).standard_normal(A.shape[1])
    v = b - A @ x
    X = O.populate_upper_triangle(v, 200, 1.0 / np.sqrt(2.0))
    X = np.triu(X) + np.triu(X, 1).T
    assert np.allclose((bs - As @ x).reshape(200, 200, order="F"), X, rtol=1e-13, atol=1e-13)


@pytest.mark.parametrize("name", sorted(PROBLEMS))
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("scaling", [0, 10])
def test_device_reverse_is_bit_identical(name, dtype, scaling):
    model = _model(name, scaling=scaling, dtype=dtype, max_iter=300)
    res = model.optimize()
    assert model._dec is not None and not model._dec.compact
    eng = model.engine
    d = chordal.decomposition_arrays(model._dec, eng.n, eng.m)
    assert d.traditional
    eng.set_decomposition(d)
    x, s, mu, stats = eng.reverse_decomposition(complete_dual=False)
    assert np.array_equal(_bits(x), _bits(res.x))
    assert np.array_equal(_bits(s), _bits(res.s))
    assert np.array_equal(_bits(mu), _bits(-res.y))
    assert stats["cones_completed"] == 0
    model.empty_model()


def _separator_kappa(y, info, d):
    """the largest condition number of a separator block of -mu, over the decomposed cones: two factorisations of it
    differ by about eps * kappa"""
    kappa = 1.0
    for k, c in zip(info.blocks, d.cones):
        S = info.sets_orig[k]
        seg = y[c.row_offset:c.row_offset + S.dim]
        Y0 = (seg.reshape(S.sqrt_dim, S.sqrt_dim, order="F") if isinstance(S, M.PsdCone)
              else chordal._svec_to_mat(seg, S.sqrt_dim))
        perm = np.argsort(c.new_of)
        kappa = max([kappa] + [np.linalg.cond(Y0[np.ix_(perm[c.idx[a0:a1]], perm[c.idx[a0:a1]])])
                               for lo, hi, a0, a1, k0, k1 in c.steps.tolist() if lo and hi > lo and a1 > a0])
    return kappa


@pytest.mark.parametrize("name", sorted(PROBLEMS))
def test_device_completion_matches_host(name):
    host = _model(name, complete_dual=True, max_iter=300)
    dev = _model(name, complete_dual=True, reverse_on_device=True, max_iter=300)
    rh, rd = host.optimize(), dev.optimize()
    assert rh.status == rd.status and rh.iter == rd.iter
    assert np.array_equal(_bits(rd.x), _bits(rh.x)) and np.array_equal(_bits(rd.s), _bits(rh.s))
    d = chordal.decomposition_arrays(host._dec, host.engine.n, host.engine.m)
    kappa = _separator_kappa(rh.y, host._dec, d)
    err = np.linalg.norm(rd.y - rh.y) / np.linalg.norm(rh.y)
    assert err <= 1e-12 * kappa, (err, kappa)
    if name in ("four_cone", "four_cone_triangle", "mixed"):
        # solved to the default tolerances: the completed square blocks are PSD
        for k in host._dec.blocks:
            S = host._dec.sets_orig[k]
            if isinstance(S, M.PsdCone):
                off = host._dec.cone_offsets[k]
                Y = rd.y[off:off + S.dim].reshape(S.sqrt_dim, S.sqrt_dim, order="F")
                assert np.array_equal(Y, Y.T) and np.linalg.eigvalsh(Y).min() > -1e-6
    host.empty_model()
    dev.empty_model()


def test_set_decomposition_paths():
    model = _model("mixed")
    model._setup()
    eng = model.engine
    d = chordal.decomposition_arrays(model._dec, eng.n, eng.m)
    # the compact entry point refuses the square layout, and a traditional map needs mu_src = NULL
    compact = chordal.DecompositionArrays(d.n_orig, d.m_orig, d.n, d.m, d.plain, d.row, d.s_ptr, d.s_src,
                                          d.s_src[d.s_ptr[1:] - 1], d.cones, traditional=False)
    with pytest.raises(E.EngineError) as ei:
        eng.set_decomposition(compact)
    assert ei.value.code == E.ERR_UNSUPPORTED
    keep = []
    cones = (E.CompletionStruct * len(d.cones))()
    for k, c in enumerate(d.cones):
        cones[k] = E.completion_struct(c, keep)
    bad = E.DecompositionStruct(d.n_orig, d.m_orig, d.n, d.m, len(d.plain), E._i64(d.plain, keep), len(d.row),
                                E._i64(d.row, keep), E._i64(d.s_ptr, keep), E._i64(d.s_src, keep),
                                E._i64(d.s_src[d.s_ptr[1:] - 1], keep), len(d.cones), C.cast(cones, C.c_void_p))
    assert eng._lib.cosmo_b200_set_decomposition_noncompact(eng._h, C.byref(bad)) == E.ERR_INVALID
    bad.mu_src = None
    bad.m = d.m + 1
    assert eng._lib.cosmo_b200_set_decomposition_noncompact(eng._h, C.byref(bad)) == E.ERR_INVALID
    bad.m = d.m
    assert eng._lib.cosmo_b200_set_decomposition_noncompact(eng._h, C.byref(bad)) == E.OK
    eng.set_decomposition(d)                              # the binding sizes the output buffers from the map it handed over
    eng.solve()
    x, s, mu, stats = eng.reverse_decomposition(complete_dual=True)
    assert stats["cones_completed"] == 4 and s.shape == mu.shape == (d.m_orig,)
    eng.set_decomposition(None)                           # cleared: no map is left
    with pytest.raises(E.EngineError) as ei:
        eng.reverse_decomposition()
    assert ei.value.code == E.ERR_INVALID
    model.empty_model()


@pytest.mark.parametrize("name", ["four_cone", "four_cone_triangle", "mixed"])
@pytest.mark.parametrize("solver", ["CGIndirectKKTSolver", "DeviceLdlKKTSolver"])
def test_solve_matches_the_oracle_on_the_decomposed_arrays(name, solver):
    P, q, A, b, sets = PROBLEMS[name]()
    P2, q2, A2, b2, sets2, info = chordal.decompose(P, q, A, b, sets, merge="clique_graph", compact=False)
    ref = O.solve(P2, q2, A2, b2, to_oracle_cones(sets2),
                  O.Settings(kkt_solver="cg") if solver == "CGIndirectKKTSolver" else O.Settings())
    model = _model(name, kkt_solver=solver)
    res = model.optimize()
    assert model.engine.n == A2.shape[1] and model.engine.m == A2.shape[0]
    assert res.status == ref.status == "Solved"
    assert res.iter == ref.iter, (res.iter, ref.iter)
    assert abs(res.obj_val - ref.obj_val) < 1e-6
    x, s, mu = chordal.reverse(info, ref.x, ref.s, -ref.y)
    assert np.abs(res.s - s).max() < 1e-5 and np.abs(res.x - x).max() < 1e-5
    model.empty_model()


def _maxcut_data(nv, seed):
    """the C5-type problem with new weights, column scales of A and a small diagonal P: the same pattern for every seed"""
    rows, cols, _ = cosmo_b200.problems.banded_random_graph(nv, 3.0, 20, seed=1)
    rng = np.random.default_rng(seed)
    w = rng.integers(1, 11, size=len(rows)).astype(np.float64)
    P, q, A, b, sets = cosmo_b200.problems.maxcut_dual_sdp(nv, rows, cols, w)
    A = sp.csc_matrix(A)
    A.sort_indices()
    A.data = A.data * rng.uniform(0.5, 2.0, A.nnz)
    P = sp.diags(rng.uniform(0.001, 0.01, nv), format="csc")
    return P, q * rng.uniform(0.9, 1.1, nv), A, b, sets


def _fresh(data, **st):
    dtype = st.pop("dtype", np.float64)
    model = cosmo_b200.Model(dtype=dtype)
    model.set(*data, cosmo_b200.Settings(decompose=True, compact_transformation=False, **st))
    return model


@pytest.mark.parametrize("nv,scaling,solver", [(200, 0, "CGIndirectKKTSolver"), (200, 10, "CGIndirectKKTSolver"),
                                               (200, 10, "DeviceLdlKKTSolver"), (2000, 0, "CGIndirectKKTSolver"),
                                               (2000, 10, "CGIndirectKKTSolver")])
def test_update_matches_a_fresh_model(nv, scaling, solver):
    D1, D2 = _maxcut_data(nv, 3), _maxcut_data(nv, 4)
    st = dict(scaling=scaling, kkt_solver=solver, max_iter=150)
    m1 = _fresh(D1, **st)
    m1.optimize()
    eng = m1.engine
    assert not m1._dec.compact and m1._fwd.b_uncovered.any()
    P2, q2, A2, b2, _ = D2
    m1.update(q=q2, b=b2, P=P2, A=A2)
    assert m1.engine is eng and m1._x2 is not None
    warm = (m1._x2.copy(), m1._s2.copy(), m1._mu2.copy())
    r1 = m1.optimize()
    m2 = _fresh(D2, **st)
    m2._setup()
    assert (m2.engine.n, m2.engine.m) == (eng.n, eng.m)
    assert np.array_equal(m2._fwd.a_src, m1._fwd.a_src) and np.array_equal(m2._fwd.b_src, m1._fwd.b_src)
    m2._x2, m2._s2, m2._mu2 = warm
    r2 = m2.optimize()
    for f in ("x", "s", "y"):
        assert np.array_equal(_bits(getattr(r1, f)), _bits(getattr(r2, f))), f
    assert (r1.status, r1.iter, r1.obj_val) == (r2.status, r2.iter, r2.obj_val)
    rng = np.random.default_rng(0)
    x, y = rng.standard_normal(eng.n), rng.standard_normal(eng.m)
    for which, v in ((0, x), (1, y), (2, x)):
        assert np.array_equal(_bits(eng.spmv(which, v)), _bits(m2.engine.spmv(which, v))), which
    m1.empty_model()
    m2.empty_model()


def test_nonzero_b_on_an_uncovered_row_rebuilds_the_engine():
    D1 = _maxcut_data(200, 3)
    model = _fresh(D1, max_iter=100)
    model.optimize()
    eng = model.engine
    b = D1[3].copy()
    b[np.nonzero(model._fwd.b_uncovered)[0][0]] = 1.0
    model.update(b=b)
    assert model.engine is None                           # the pattern changed: decomposed again at the next solve
    res = model.optimize()
    assert model.engine is not eng and model._dec is not None and not model._dec.compact
    assert res.s.shape == (len(b),)
    model.empty_model()
