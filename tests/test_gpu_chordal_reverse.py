"""The reverse of a chordal decomposition on the device (cosmo_b200_set_decomposition /
cosmo_b200_reverse_decomposition / cosmo_b200_psd_complete) against the host path (chordal.reverse,
chordal.psd_complete)."""
import numpy as np
import pytest
import scipy.linalg
import scipy.sparse as sp

import cosmo_b200
from cosmo_b200 import chordal, engine as E

pytestmark = pytest.mark.gpu


def _g6_model(settings):
    from tests import golden_problems as G
    A1, A2, B, c = G.g6_chordal_sdp_data()
    A = -np.column_stack([G._svec(A1), G._svec(A2)])
    model = cosmo_b200.Model(dtype=settings.pop("dtype", np.float64))
    model.assemble(np.zeros((2, 2)), c, [cosmo_b200.Constraint(A, G._svec(B), cosmo_b200.PsdConeTriangle(45))],
                   cosmo_b200.Settings(**settings))
    return model


def _c5_model(nv, settings):
    rows, cols, w = cosmo_b200.problems.banded_random_graph(nv, 3.0, 20, seed=1)
    P, q, A, b, sets = cosmo_b200.problems.maxcut_dual_sdp(nv, rows, cols, w)
    model = cosmo_b200.Model(dtype=settings.pop("dtype", np.float64))
    model.set(P, q, A, b, sets, cosmo_b200.Settings(**settings))
    return model


def _model(name, **settings):
    return _g6_model(settings) if name == "g6" else _c5_model(2000, settings)


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


@pytest.mark.parametrize("name", ["g6", "c5"])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("scaling", [0, 10])
def test_reverse_without_completion_is_bit_identical(name, dtype, scaling):
    # the host path of Model.optimize: D x, s / E, (E mu) / c in fp64, then chordal.reverse
    model = _model(name, decompose=True, scaling=scaling, dtype=dtype, max_iter=300 if name == "c5" else 5000)
    res = model.optimize()
    eng = model.engine
    with pytest.raises(E.EngineError) as ei:           # no map yet
        eng.reverse_decomposition()
    assert ei.value.code == E.ERR_INVALID
    eng.set_decomposition(chordal.decomposition_arrays(model._dec, eng.n, eng.m))
    x, s, mu, stats = eng.reverse_decomposition(complete_dual=False)
    assert np.array_equal(_bits(x), _bits(res.x))
    assert np.array_equal(_bits(s), _bits(res.s))
    assert np.array_equal(_bits(mu), _bits(-res.y))
    assert stats["cones_completed"] == 0 and stats["pinv_fallbacks"] == 0
    # a NULL buffer is skipped
    x1, s1, mu1, _ = eng.reverse_decomposition(x=False, mu=False)
    assert x1 is None and mu1 is None and np.array_equal(_bits(s1), _bits(s))


def _pattern(nv):
    if nv == 9:
        from tests import golden_problems as G
        cl = np.zeros((9, 9), dtype=bool)
        for c in G.G6_CLIQUES:
            cl[np.ix_(c, c)] = True
        r, c = np.nonzero(np.triu(cl, 1))
        return r, c
    rows, cols, _ = cosmo_b200.problems.banded_random_graph(nv, 3.0, 20, seed=nv)
    return np.asarray(rows), np.asarray(cols)


def _tree(nv):
    r, c = _pattern(nv)
    return chordal.clique_graph_merge(chordal.chordal_cliques(nv, r, c))


def _pd_on_cliques(tree, nv, kappa, seed):
    """a dense positive definite matrix of condition kappa, restricted to the cliques: every clique block is a principal
    submatrix of it, hence positive definite with condition <= kappa"""
    rng = np.random.default_rng(seed)
    Q, _ = np.linalg.qr(rng.standard_normal((nv, nv)))
    X = (Q * np.logspace(0, -np.log10(kappa), nv)) @ Q.T
    X = (X + X.T) / 2
    mask = np.zeros((nv, nv), dtype=bool)
    for c in tree.cliques:
        mask[np.ix_(c, c)] = True
    return np.where(mask, X, 0.0), mask


@pytest.mark.parametrize("nv,kappa", [(9, 1e3), (200, 1e3), (200, 1e6), (2000, 1e3)])
def test_psd_complete_matches_host(nv, kappa):
    tree = _tree(nv)
    Y, mask = _pd_on_cliques(tree, nv, kappa, seed=nv)
    sched = chordal.completion_schedule(tree, nv)
    got, stats = E.psd_complete(Y, sched)
    want = chordal.psd_complete(Y, tree)
    err = np.linalg.norm(got - want) / np.linalg.norm(want)
    assert err <= 1e-12 * kappa, err
    assert np.array_equal(_bits(got[mask]), _bits(Y[mask]))
    lam_min = scipy.linalg.eigh(got, eigvals_only=True, driver="evr", subset_by_index=[0, 0])[0]
    assert lam_min >= -1e-12 * np.linalg.norm(got), lam_min
    assert stats["pinv_fallbacks"] == 0 and stats["cones_completed"] == 1 and stats["workspace_bytes"] == 8 * nv * nv


def test_singular_separator_falls_back_to_the_pseudo_inverse():
    tree = _tree(200)
    Y, mask = _pd_on_cliques(tree, 200, 1e3, seed=5)
    sched = chordal.completion_schedule(tree, 200)
    # a vertex of a separator with an all-zero row and column: the separator block is singular (an exact zero pivot)
    seps = [v for t, k in enumerate(tree.sep) if tree.parent[t] >= 0 for v in k.tolist()]
    v = seps[len(seps) // 2]
    Y[v, :] = 0.0
    Y[:, v] = 0.0
    got, stats = E.psd_complete(Y, sched)
    want = chordal.psd_complete(Y, tree)
    assert stats["pinv_fallbacks"] >= 1
    assert np.linalg.norm(got - want) <= 1e-10 * np.linalg.norm(want)


@pytest.mark.parametrize("name", ["g6", "c5"])
def test_solve_with_completion_on_device_matches_host(name):
    host = _model(name, decompose=True, complete_dual=True)
    dev = _model(name, decompose=True, complete_dual=True, reverse_on_device=True)
    rh, rd = host.optimize(), dev.optimize()
    assert rh.status == rd.status and rh.iter == rd.iter
    assert np.array_equal(_bits(rd.x), _bits(rh.x)) and np.array_equal(_bits(rd.s), _bits(rh.s))
    # entries inside the cliques are the gathered values, bit for bit
    d = chordal.decomposition_arrays(host._dec, host.engine.n, host.engine.m)
    assert np.array_equal(_bits(rd.y[d.row]), _bits(rh.y[d.row]))
    # the completed entries: the dual of an SDP at its optimum is rank-deficient, so the separator blocks are
    # ill-conditioned and any two factorisations differ by about eps * cond(W[alpha, alpha])
    S = host.sets0[0]
    Y0 = chordal._svec_to_mat(rh.y[:S.dim], S.sqrt_dim)
    c = d.cones[0]
    perm = np.argsort(c.new_of)
    kappa = max([np.linalg.cond(Y0[np.ix_(perm[c.idx[a0:a1]], perm[c.idx[a0:a1]])])
                 for lo, hi, a0, a1, k0, k1 in c.steps.tolist() if lo and hi > lo and a1 > a0] + [1.0])
    err = np.linalg.norm(rd.y - rh.y) / np.linalg.norm(rh.y)
    assert err <= 1e-12 * kappa, (err, kappa)
    if name == "c5":
        # at eps = 1e-5 the clique blocks of C5's dual are slightly indefinite and nearly singular: the host completion
        # itself grows entries of order 1e64 there, so only agreement with it is required
        return
    Y = chordal._svec_to_mat(rd.y[:S.dim], S.sqrt_dim)
    lam_min = np.linalg.eigvalsh(Y).min()
    assert lam_min >= -1e-3 * max(1.0, np.abs(Y).max()), lam_min


def test_error_paths():
    model = _model("g6", decompose=True)
    model._setup()
    eng = model.engine
    d = chordal.decomposition_arrays(model._dec, eng.n, eng.m)
    eng.set_decomposition(d)
    with pytest.raises(E.EngineError) as ei:           # a map, but no solve since the engine was created
        eng.reverse_decomposition()
    assert ei.value.code == E.ERR_INVALID
    bad = chordal.decomposition_arrays(model._dec, eng.n, eng.m)
    bad.s_src = bad.s_src.copy()
    bad.s_src[0] = eng.m
    with pytest.raises(E.EngineError) as ei:
        eng.set_decomposition(bad)
    assert ei.value.code == E.ERR_INVALID
    sq = chordal.decomposition_arrays(model._dec, eng.n, eng.m)
    sq.cones[0].dim = sq.cones[0].N ** 2
    with pytest.raises(E.EngineError) as ei:
        eng.set_decomposition(sq)
    assert ei.value.code == E.ERR_UNSUPPORTED
    eng.solve()
    eng.set_decomposition(None)                        # cleared
    with pytest.raises(E.EngineError) as ei:
        eng.reverse_decomposition()
    assert ei.value.code == E.ERR_INVALID
    eng.set_decomposition(d)
    x, s, mu, _ = eng.reverse_decomposition(complete_dual=True)
    assert x.shape == (2,) and s.shape == mu.shape == (45,)
    eng.reset()                                        # reset forgets the solution
    with pytest.raises(E.EngineError) as ei:
        eng.reverse_decomposition()
    assert ei.value.code == E.ERR_INVALID
