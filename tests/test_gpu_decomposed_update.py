"""cosmo_b200_set_forward_map / cosmo_b200_update_matrices_original: new q, b, P and A of a chordally decomposed model go
to the live engine in the coordinates of the original problem and leave it bit for bit where a new engine on the
decomposed new data starts; the clique iterates stay as the warm start."""
import copy

import numpy as np
import pytest
import scipy.sparse as sp

import cosmo_b200
from cosmo_b200 import chordal, engine as E

pytestmark = pytest.mark.gpu


def _maxcut(nv, seed, graph_seed=1):
    """C5-type dual MAXCUT SDP on the banded graph of `graph_seed` with weights, a scaling of the columns of A and a small
    diagonal P drawn from `seed`: the same pattern for every seed"""
    rows, cols, _ = cosmo_b200.problems.banded_random_graph(nv, 3.0, 20, seed=graph_seed)
    rng = np.random.default_rng(seed)
    w = rng.integers(1, 11, size=len(rows)).astype(np.float64)
    P, q, A, b, sets = cosmo_b200.problems.maxcut_dual_sdp(nv, rows, cols, w)
    A = sp.csc_matrix(A)
    A.sort_indices()
    A.data = A.data * rng.uniform(0.5, 2.0, A.nnz)
    P = sp.diags(rng.uniform(0.001, 0.01, nv), format="csc")
    return P, q * rng.uniform(0.9, 1.1, nv), A, b, sets


def _model(data, **settings):
    dtype = settings.pop("dtype", np.float64)
    model = cosmo_b200.Model(dtype=dtype)
    model.set(*data, cosmo_b200.Settings(decompose=True, **settings))
    return model


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


def _assert_same_result(r1, r2):
    for f in ("x", "s", "y"):
        assert np.array_equal(_bits(getattr(r1, f)), _bits(getattr(r2, f))), f
    assert (r1.status, r1.iter, r1.obj_val, r1.kkt_inner_iterations) == (r2.status, r2.iter, r2.obj_val, r2.kkt_inner_iterations)
    assert r1.info.rho_updates == r2.info.rho_updates


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("solver", ["CGIndirectKKTSolver", "DeviceLdlKKTSolver"])
@pytest.mark.parametrize("scaling", [0, 10])
@pytest.mark.parametrize("nv", [200, 2000])
def test_update_matches_a_fresh_model(nv, scaling, solver, dtype):
    D1, D2 = _maxcut(nv, seed=3), _maxcut(nv, seed=4)
    st = dict(scaling=scaling, kkt_solver=solver, dtype=dtype, max_iter=150)
    m1 = _model(D1, **st)
    m1.optimize()
    eng = m1.engine
    P2, q2, A2, b2, _ = D2
    m1.update(q=q2, b=b2, P=P2, A=A2)
    assert m1.engine is eng and m1._x2 is not None                       # no rebuild, the clique iterates stay
    warm = (m1._x2.copy(), m1._s2.copy(), m1._mu2.copy())
    r1 = m1.optimize()
    m2 = _model(D2, **st)
    m2._setup()                                                          # same pattern, hence the same decomposition
    assert (m2.engine.n, m2.engine.m) == (eng.n, eng.m)
    assert np.array_equal(m2._fwd.a_src, m1._fwd.a_src) and np.array_equal(m2._fwd.b_src, m1._fwd.b_src)
    m2._x2, m2._s2, m2._mu2 = warm
    r2 = m2.optimize()
    _assert_same_result(r1, r2)
    rng = np.random.default_rng(0)
    x, y = rng.standard_normal(eng.n), rng.standard_normal(eng.m)
    for which, v in ((0, x), (1, y), (2, x)):                            # every resident copy of A and P
        assert np.array_equal(_bits(eng.spmv(which, v)), _bits(m2.engine.spmv(which, v))), which
    for a, b in zip(eng.scaling(), m2.engine.scaling()):
        assert np.array_equal(_bits(a), _bits(b))
    assert np.array_equal(_bits(eng.rho_vec()), _bits(m2.engine.rho_vec()))
    m1.empty_model()
    m2.empty_model()


def test_update_of_q_and_b_alone_keeps_rho_and_the_iterates():
    D1, D2 = _maxcut(200, seed=3), _maxcut(200, seed=4)
    m1 = _model(D1, scaling=10)
    m1.optimize()
    eng, rho = m1.engine, m1.engine.rho_vec()
    m1.update(q=D2[1], b=D2[3])
    assert m1.engine is eng and np.array_equal(eng.rho_vec(), rho) and m1._x2 is not None
    r1 = m1.optimize()
    fresh = _model((D1[0], D2[1], D1[2], D2[3], D1[4]), scaling=10).optimize()
    assert r1.status == fresh.status == "Solved" and abs(r1.obj_val - fresh.obj_val) <= 1e-3 * abs(fresh.obj_val)
    m1.empty_model()


def test_device_reverse_after_an_update_matches_the_host_reverse():
    D1, D2 = _maxcut(200, seed=3), _maxcut(200, seed=4)
    model = _model(D1, reverse_on_device=True, complete_dual=True, max_iter=300)
    model.optimize()
    eng = model.engine
    model.update(q=D2[1], b=D2[3], P=D2[0], A=D2[2])
    assert model.engine is eng
    with pytest.raises(E.EngineError) as ei:                             # the map stayed, but a reverse needs a solve first
        eng.reverse_decomposition()
    assert ei.value.code == E.ERR_INVALID and "no solve" in str(ei.value)
    res = model.optimize()
    x, s, mu = chordal.reverse(model._dec, model._x2, model._s2, model._mu2, complete_dual=True)
    assert np.array_equal(_bits(res.x), _bits(x)) and np.array_equal(_bits(res.s), _bits(s))
    d = chordal.decomposition_arrays(model._dec, eng.n, eng.m)
    assert np.array_equal(_bits(res.y[d.row]), _bits(-mu[d.row]))        # inside the cliques: the gathered values
    # the completed entries go through a factorisation of the separator blocks, as in test_gpu_chordal_reverse
    S = model.sets0[0]
    Y0 = chordal._svec_to_mat(-mu[:S.dim], S.sqrt_dim)
    c = d.cones[0]
    perm = np.argsort(c.new_of)
    kappa = max([np.linalg.cond(Y0[np.ix_(perm[c.idx[a0:a1]], perm[c.idx[a0:a1]])])
                 for lo, hi, a0, a1, k0, k1 in c.steps.tolist() if lo and hi > lo and a1 > a0] + [1.0])
    err = np.linalg.norm(res.y + mu) / np.linalg.norm(mu)
    assert err <= 1e-12 * kappa, (err, kappa)
    model.empty_model()


def test_warm_start_survives_the_update():
    nv = 2000
    D1 = _maxcut(nv, seed=3)
    P, q, A, b, sets = D1
    rng = np.random.default_rng(9)
    b2 = b * (1.0 + 1e-3 * rng.standard_normal(len(b)))                  # a small change of the weights
    A2 = A.copy()
    A2.data = A.data * (1.0 + 1e-3 * rng.standard_normal(A.nnz))
    model = _model(D1)
    first = model.optimize()
    model.update(b=b2, A=A2)
    warm = model.optimize()
    cold = _model((P, q, A2, b2, sets)).optimize()
    print("iterations: first solve %d, after the update from the kept clique iterates %d, cold fresh model %d"
          % (first.iter, warm.iter, cold.iter))
    assert first.status == warm.status == cold.status == "Solved"
    assert warm.iter < cold.iter
    assert abs(warm.obj_val - cold.obj_val) <= 1e-3 * abs(cold.obj_val)
    model.empty_model()


def _engine_pair(**settings):
    data = _maxcut(200, seed=3)
    ma, mb = _model(data, **settings), _model(data, **settings)
    ma._setup()
    mb._setup()
    return data, ma, mb


def _solve_from(eng, seed=7):
    rng = np.random.default_rng(seed)
    eng.warm_start(rng.standard_normal(eng.n), np.abs(rng.standard_normal(eng.m)), 0.1 * rng.standard_normal(eng.m))
    return eng.solve()


def test_refused_updates_change_nothing():
    (P, q, A, b, sets), ma, mb = _engine_pair(scaling=0, max_iter=100)
    eng, f = mb.engine, mb._fwd
    with pytest.raises(E.EngineError) as ei:
        eng.update_matrices_original(Ax=A.data[:-1] * 2.0, q=q * 2.0)
    assert ei.value.code == E.ERR_INVALID and "nnz" in str(ei.value)
    with pytest.raises(E.EngineError) as ei:
        eng.update_matrices_original(Px=np.ones(P.nnz + 1), Ax=A.data * 2.0)
    assert ei.value.code == E.ERR_INVALID
    bad_b = b.copy()
    bad_b[np.nonzero(f.b_uncovered)[0][:3]] = 1.0
    with pytest.raises(E.EngineError) as ei:
        eng.update_matrices_original(Px=P.data * 2.0, Ax=A.data * 2.0, q=q * 2.0, b=bad_b)
    assert ei.value.code == E.ERR_INVALID and "in 3 rows" in str(ei.value)
    o1, o2 = _solve_from(eng), _solve_from(ma.engine)
    for name in ("x", "s", "mu"):
        assert np.array_equal(_bits(getattr(o1, name)), _bits(getattr(o2, name))), name
    assert (o1.iter, o1.status, o1.obj_val) == (o2.iter, o2.status, o2.obj_val)
    # an equilibrating engine needs all four
    (P, q, A, b, sets), mc, md = _engine_pair(scaling=10, max_iter=100)
    with pytest.raises(E.EngineError) as ei:
        md.engine.update_matrices_original(Px=P.data, Ax=A.data)
    assert ei.value.code == E.ERR_INVALID and "equilibrating" in str(ei.value)
    # without a forward map
    md.engine.set_forward_map(None)
    with pytest.raises(E.EngineError) as ei:
        md.engine.update_matrices_original(Px=P.data, Ax=A.data, q=q, b=b)
    assert ei.value.code == E.ERR_INVALID and "no forward map" in str(ei.value)
    for m in (ma, mb, mc, md):
        m.empty_model()


def _map_mutations(f):
    k = np.nonzero(f.a_src >= 0)[0]
    r = np.nonzero(f.b_src != -1)[0]

    def put(attr, i, v):
        def g(m):
            a = np.array(getattr(m, attr))
            a[i] = v
            setattr(m, attr, a)
        return g

    return {
        "n": lambda m: setattr(m, "n", m.n + 1),
        "m": lambda m: setattr(m, "m", m.m - 1),
        "nnzA": lambda m: setattr(m, "a_src", m.a_src[:-1]),
        "n_orig_above_n": lambda m: setattr(m, "n_orig", m.n + 1),
        "a_src_too_large": put("a_src", k[0], f.nnzA_orig),
        "a_src_below_minus_two": put("a_src", k[0], -3),
        "a_source_used_twice": put("a_src", k[1], f.a_src[k[0]]),
        "a_source_not_used": put("a_src", k[0], -1),
        "b_src_too_large": put("b_src", r[0], f.m_orig),
        "b_clique_src_too_large": put("b_src", r[0], -2 - f.m_orig),
        "b_source_used_twice": put("b_src", r[1], f.b_src[r[0]]),
        "b_row_neither_used_nor_uncovered": put("b_src", r[0], -1),
        "b_row_used_and_uncovered": lambda m: setattr(m, "b_uncovered", np.ones_like(m.b_uncovered)),
    }


def test_set_forward_map_checks_every_index():
    data, ma, mb = _engine_pair(scaling=0, max_iter=100)
    eng, f = mb.engine, mb._fwd
    for what, mutate in _map_mutations(f).items():
        bad = copy.deepcopy(f)
        mutate(bad)
        with pytest.raises(E.EngineError) as ei:
            eng.set_forward_map(bad)
        assert ei.value.code == E.ERR_INVALID and "forward map" in str(ei.value), what
        with pytest.raises(E.EngineError):                               # a refused map leaves none behind
            eng.update_matrices_original(Ax=data[2].data)
    eng.set_forward_map(f)
    eng.update_matrices_original(Ax=data[2].data)
    o1, o2 = _solve_from(eng), _solve_from(ma.engine)
    assert np.array_equal(_bits(o1.x), _bits(o2.x)) and o1.iter == o2.iter
    ma.empty_model()
    mb.empty_model()
