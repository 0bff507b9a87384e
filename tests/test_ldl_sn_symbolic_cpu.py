"""CPU checks of the supernodal LDL' plugin's host analysis (cosmo_b200_ldl_sn_symbolic): a NumPy restatement of the
postorder, the supernode rule and the relaxed amalgamation over the output of the simplicial analysis
(cosmo_b200_ldl_symbolic), the stored pattern against the simplicial one, and the settings that select the plugin."""
import numpy as np
import pytest
import scipy.sparse as sp

import cosmo_b200
from cosmo_b200 import engine as E, sharding


def _relax_ok(w, zeros, stored):
    """the amalgamation rule of ldl_sn_symbolic.h (Ashcraft-Grimes relaxed supernodes, CHOLMOD's thresholds)"""
    if w > 256:
        return False
    z = zeros / stored if stored > 0 else 0.0
    return w <= 4 or (w <= 16 and z <= 0.8) or (w <= 48 and z <= 0.1) or z <= 0.05


def _restate(P, A):
    """(postordered perm, parent, colcount, supernode pointers) from cosmo_b200_ldl_symbolic's output"""
    perm0, parent0, cc0, _ = E.ldl_symbolic(P, A)
    N = perm0.size
    children = [[] for _ in range(N)]
    for j in range(N):
        if parent0[j] >= 0:
            children[parent0[j]].append(j)
    post = []
    for r in range(N):
        if parent0[r] >= 0:
            continue
        stack = [(r, 0)]
        while stack:
            j, k = stack.pop()
            if k < len(children[j]):
                stack.append((j, k + 1))
                stack.append((children[j][k], 0))
            else:
                post.append(j)
    post = np.array(post, dtype=np.int64)
    ipost = np.empty(N, dtype=np.int64)
    ipost[post] = np.arange(N)
    parent = np.where(parent0[post] >= 0, ipost[np.maximum(parent0[post], 0)], -1)
    cc = cc0[post]
    fund = [0] + [j + 1 for j in range(N - 1) if not (parent[j] == j + 1 and cc[j] == cc[j + 1] + 1)] + [N]
    sptr = [0]
    a, e = 0, fund[1]
    for f in range(1, len(fund) - 1):
        e2 = fund[f + 1]
        merge = parent[e - 1] == e
        if merge:
            w = e2 - a
            c = np.arange(a, e2)
            zeros = int(np.sum((e2 - 1 - c) + cc[e2 - 1] - cc[c]))
            merge = _relax_ok(w, zeros, w * (w - 1) // 2 + w * int(cc[e2 - 1]))
        if merge:
            e = e2
            continue
        sptr.append(e)
        a, e = e, e2
    sptr.append(N)
    return perm0[post], parent, cc, np.array(sptr), cc0


def _simplicial_pattern(P, A, perm):
    """strictly lower pattern of L by columns, in the numbering of `perm` (row subtrees of the permuted K)"""
    m, n = A.shape
    N = n + m
    K = sp.bmat([[sp.triu(sp.csc_matrix(P)) + sp.identity(n), None], [sp.csc_matrix(A), sp.identity(m)]], format="coo")
    ip = np.empty(N, dtype=np.int64)
    ip[perm] = np.arange(N)
    r, c = ip[K.row], ip[K.col]
    lo, hi = np.minimum(r, c), np.maximum(r, c)
    cols = [set() for _ in range(N)]
    for x, y in zip(lo.tolist(), hi.tolist()):
        if y > x:
            cols[x].add(y)
    return cols


def _check(P, A):
    P, A = sp.csc_matrix(P), sp.csc_matrix(A)
    perm, parent, _, sptr, cc0 = _restate(P, A)
    got_perm, got_sptr, got_spar, st = E.ldl_sn_symbolic(P, A)
    N = perm.size
    assert np.array_equal(got_perm, perm) and np.array_equal(got_sptr, sptr)            # the same partition
    # the engine's pivots are the simplicial ones renumbered: their simplicial column counts, read through the
    # engine's permutation, sum to the engine's nnz(L) and give its stored entries
    perm0 = E.ldl_symbolic(P, A)[0]
    pos0 = np.empty(N, dtype=np.int64)
    pos0[perm0] = np.arange(N)
    assert np.array_equal(np.sort(got_perm), np.arange(N))
    cc = cc0[pos0[got_perm]]
    assert st["nnz_L"] == int(cc0.sum())
    ns = got_sptr.size - 1
    assert st["supernodes"] == ns and st["max_width"] == int(np.max(np.diff(got_sptr)))
    snode_of = np.repeat(np.arange(ns), np.diff(got_sptr))
    stored = 0
    for s in range(ns):
        c0, c1 = got_sptr[s], got_sptr[s + 1]
        assert all(parent[j] == j + 1 for j in range(c0, c1 - 1))                         # an etree chain
        assert got_spar[s] == (snode_of[parent[c1 - 1]] if parent[c1 - 1] >= 0 else -1)
        w = c1 - c0
        st_s = w * (w - 1) // 2 + w * int(cc[c1 - 1])
        zeros = st_s - int(cc[c0:c1].sum())
        assert zeros >= 0
        fundamental = all(cc[j] == cc[j + 1] + 1 for j in range(c0, c1 - 1))
        assert fundamental or _relax_ok(w, zeros, st_s), (s, w, zeros, st_s)               # merges obey the rule
        if s > 0:                                                                            # no fundamental run split
            assert not (parent[c0 - 1] == c0 and cc[c0 - 1] == cc[c0] + 1), s
        stored += st_s
    assert st["stored"] == stored and st["explicit_zeros"] == stored - int(cc0.sum())
    level = np.zeros(ns, dtype=np.int64)
    for s in range(ns):
        if got_spar[s] >= 0:
            assert got_spar[s] > s
            level[got_spar[s]] = max(level[got_spar[s]], level[s] + 1)
    assert st["levels"] == (int(level.max()) + 1 if ns else 0)
    # the stored pattern {c+1..c1-1} u struct(L(:, c1-1)) contains the simplicial pattern
    cols = _simplicial_pattern(P, A, perm)
    Lc = [None] * N
    kids = [[] for _ in range(N)]
    for j in range(N):
        if parent[j] >= 0:
            kids[parent[j]].append(j)
    for j in range(N):
        s_ = set(cols[j])
        for k in kids[j]:
            s_ |= Lc[k]
        s_.discard(j)
        Lc[j] = s_
    assert [len(x) for x in Lc] == cc.tolist()
    for s in range(ns):
        c0, c1 = sptr[s], sptr[s + 1]
        top = Lc[c1 - 1]
        for c in range(c0, c1):
            assert Lc[c] <= set(range(c + 1, c1)) | top
    return st


def test_random_sparse_qp():
    P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(300, 500, 0.02, seed=3)
    _check(P, A)


def test_portfolio_socp():
    P, q, A, b, sets = cosmo_b200.problems.portfolio_socp(200, 20, seed=1)
    _check(P, A)


def test_closest_correlation_sdp():
    P, q, A, b, sets = cosmo_b200.problems.closest_correlation_sdp(N=20)
    _check(P, A)


def test_c5_decomposition():
    from cosmo_b200 import chordal
    rows, cols, w = cosmo_b200.problems.banded_random_graph(2000, 3.0, 20, seed=1)
    P, q, A, b, sets = cosmo_b200.problems.maxcut_dual_sdp(2000, rows, cols, w)
    P2, q2, A2, b2, sets2, info = chordal.decompose(P, q, A, b, sets, merge="parent_child")
    _check(P2, A2)


@pytest.mark.parametrize("seed", range(4))
def test_random_quasi_definite_patterns(seed):
    rng = np.random.default_rng(seed)
    n, m = int(rng.integers(1, 60)), int(rng.integers(0, 80))
    P = sp.random(n, n, density=rng.uniform(0, 0.2), random_state=rng, format="csc")
    A = sp.random(m, n, density=rng.uniform(0.01, 0.3), random_state=rng, format="csc")
    _check(P + P.T, A)


def test_portfolio_2000_200_counts():
    """The factor rows fill in to a dense trailing block, a chain of the elimination tree whose column counts fall by
    one per column: the rule makes it one supernode of width 203, where the simplicial plugin runs 203 levels.  The
    rest are 1999 supernodes of width 2 (a column with a leaf merged in by the relaxed rule) and 2001 of width 1."""
    P, q, A, b, sets = cosmo_b200.problems.portfolio_socp(2000, 200, seed=1)
    st = _check(P, A)
    assert st["simplicial_levels"] == 203
    assert (st["supernodes"], st["max_width"], st["levels"]) == PORTFOLIO_COUNTS, st


PORTFOLIO_COUNTS = (4001, 203, 3)


def test_settings_select_the_supernodal_plugin_and_sharding_refuses_it():
    for name in ("DeviceSupernodalKKTSolver", "MKLPardisoKKTSolver"):
        assert cosmo_b200.Settings(kkt_solver=name).to_struct().kkt_solver == E.KKT_LDL_SUPERNODAL == 4
    with pytest.raises(E.EngineError) as ei:
        cosmo_b200.Settings(kkt_solver="PardisoIndirectKKTSolver").to_struct()
    assert "DeviceSupernodalKKTSolver" in str(ei.value) and "MKLPardisoKKTSolver" in str(ei.value)
    P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(30, 40, 0.2, seed=0)
    shard = sharding.make_shard(P, q, A, b, sets, rank=0, world=2)
    for name in ("DeviceSupernodalKKTSolver", "MKLPardisoKKTSolver"):
        with pytest.raises(E.EngineError) as ei:
            sharding.create_engine(shard, cosmo_b200.Settings(kkt_solver=name), dist=object())
        assert ei.value.code == E.ERR_UNSUPPORTED


def test_symbolic_entry_validates_its_input():
    with pytest.raises(E.EngineError) as ei:
        E.ldl_sn_symbolic(sp.identity(3, format="csc"), sp.csc_matrix((2, 4)))
    assert ei.value.code == E.ERR_INVALID
