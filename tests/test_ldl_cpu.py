"""CPU checks of the direct LDL' KKT plugin: the host symbolic analysis (cosmo_b200_ldl_symbolic) against pure-Python
restatements, a NumPy model of the device factorisation and solves against SciPy's sparse LU, and the host-side
selection of the plugin."""
import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

import cosmo_b200
from cosmo_b200 import engine as E, sharding
from oracle import cosmo_oracle as O
from tests import golden_problems as G


def _kkt(P, A, sigma=1e-6, rho=None):
    m, n = A.shape
    rho = np.full(m, 0.1) if rho is None else rho
    return sp.bmat([[sp.csc_matrix(P) + sigma * sp.identity(n), A.T], [A, -sp.diags(1.0 / rho)]], format="csc")


def _permuted_pattern(P, A, perm):
    """lower triangle (with diagonal) of the permuted K pattern, as a list of row sets per column"""
    m, n = A.shape
    N = n + m
    Kpat = sp.bmat([[sp.triu(sp.csc_matrix(P)) + sp.identity(n), None], [sp.csc_matrix(A), sp.identity(m)]], format="coo")
    iperm = np.empty(N, dtype=np.int64)
    iperm[perm] = np.arange(N)
    r, c = iperm[Kpat.row], iperm[Kpat.col]
    lo, hi = np.minimum(r, c), np.maximum(r, c)
    cols = [set() for _ in range(N)]
    for a, b in zip(lo.tolist(), hi.tolist()):
        if b > a:
            cols[a].add(b)
    return cols


def _etree(cols, N):
    """Liu's elimination tree from the strictly lower pattern by columns (upper pattern by rows of the transpose)"""
    upper = [[] for _ in range(N)]
    for j in range(N):
        for i in cols[j]:
            upper[i].append(j)
    parent, anc = [-1] * N, [-1] * N
    for j in range(N):
        for i in upper[j]:
            while i != -1 and i < j:
                nxt = anc[i]
                anc[i] = j
                if nxt == -1:
                    parent[i] = j
                i = nxt
    return parent


def _symbolic(cols, parent, N):
    """struct(L_j) = struct(K_{>j, j}) u (children's structs minus j)"""
    Lc = [None] * N
    children = [[] for _ in range(N)]
    for j in range(N):
        if parent[j] >= 0:
            children[parent[j]].append(j)
    for j in range(N):
        s = set(cols[j])
        for c in children[j]:
            s |= Lc[c]
        s.discard(j)
        Lc[j] = s
    return Lc


def _check_analysis(P, A, nnz_bound=None):
    m, n = A.shape
    N = n + m
    perm, parent, colcount, level = E.ldl_symbolic(P, A)
    assert np.array_equal(np.sort(perm), np.arange(N))
    cols = _permuted_pattern(P, A, perm)
    par = _etree(cols, N)
    assert parent.tolist() == par
    Lc = _symbolic(cols, par, N)
    assert colcount.tolist() == [len(s) for s in Lc]
    # factorisation / forward solve: row i depends on the columns k of row i of L, all in earlier levels;
    # backward solve: column j depends on the rows of column j, all nearer the root
    depth = np.zeros(N, dtype=np.int64)
    for j in range(N - 1, -1, -1):
        depth[j] = 0 if par[j] < 0 else depth[par[j]] + 1
    for k in range(N):
        for i in Lc[k]:
            assert level[k] < level[i] and depth[i] < depth[k]
    if nnz_bound is not None:
        assert int(colcount.sum()) <= nnz_bound, (int(colcount.sum()), nnz_bound)
    return perm, int(colcount.sum())


GOLDEN = [G.g1_qp_nonneg, G.g1_qp_box, G.g2_box_feasible, G.g3_hs21, G.g4_small_sdp, G.g5_sigma_max_lmi, G.g6_chordal_sdp,
          G.g12_lp, G.g13_lovasz_petersen, G.g15_exp_feasible, G.g16_pow_feasible, G.g17_complex_least_eigenvalue]


@pytest.mark.parametrize("builder", GOLDEN, ids=lambda f: f.__name__)
def test_symbolic_analysis_on_the_golden_problems(builder):
    P, q, cons = builder()
    Pm, qm, A, b, cones = O.assemble(P, q, cons)
    _check_analysis(sp.csc_matrix(Pm), sp.csc_matrix(A))


@pytest.mark.parametrize("seed", range(6))
def test_symbolic_analysis_on_random_quasi_definite_patterns(seed):
    rng = np.random.default_rng(seed)
    n, m = int(rng.integers(1, 60)), int(rng.integers(0, 80))
    P = sp.random(n, n, density=rng.uniform(0, 0.2), random_state=rng, format="csc")
    P = P + P.T
    A = sp.random(m, n, density=rng.uniform(0.01, 0.3), random_state=rng, format="csc")
    _check_analysis(P, A)


def test_symbolic_analysis_on_c5_and_the_portfolio_fill():
    from cosmo_b200 import chordal
    rows, cols, w = cosmo_b200.problems.banded_random_graph(2000, 3.0, 20, seed=1)
    P, q, A, b, sets = cosmo_b200.problems.maxcut_dual_sdp(2000, rows, cols, w)
    P2, q2, A2, b2, sets2, info = chordal.decompose(P, q, A, b, sets, merge="parent_child")
    _check_analysis(sp.csc_matrix(P2), sp.csc_matrix(A2), nnz_bound=int(1.5 * 48_100))
    P, q, A, b, sets = cosmo_b200.problems.portfolio_socp(2000, 200, seed=1)
    _check_analysis(P, A, nnz_bound=int(1.5 * 232_302))


def _ldl_model(K, perm, parent, level):
    """NumPy restatement of ldl.cuh with its loop order: columns level by level, for column j the updates of the
    columns k of row j of L in ascending k, each over the rows >= j of column k; then the forward solve by rows,
    D^-1 and the backward solve by columns."""
    N = K.shape[0]
    Kp = K[perm][:, perm].tocsc()
    Kl = sp.tril(Kp).tocsc()
    Kl.sort_indices()
    cols = [set() for _ in range(N)]
    Kc = Kl.tocoo()
    for r, c in zip(Kc.row.tolist(), Kc.col.tolist()):
        if r > c:
            cols[c].add(r)
    Lc = _symbolic(cols, parent, N)
    Lrows = [sorted(s) for s in Lc]
    rowsL = [[] for _ in range(N)]
    for k in range(N):
        for i in Lrows[k]:
            rowsL[i].append(k)
    Lx = [dict() for _ in range(N)]
    d = np.zeros(N)
    order = sorted(range(N), key=lambda j: (level[j], j))
    w = np.zeros(N)
    for j in order:
        for e in range(Kl.indptr[j], Kl.indptr[j + 1]):
            w[Kl.indices[e]] = Kl.data[e]
        for k in rowsL[j]:                       # ascending
            f = Lx[k][j] * d[k]
            for i in [i for i in Lrows[k] if i >= j]:
                w[i] -= Lx[k][i] * f
        d[j] = w[j]
        for i in Lrows[j]:
            Lx[j][i] = w[i] / d[j]
            w[i] = 0.0
        w[j] = 0.0

    def solve(rhs):
        z = np.zeros(N)
        for i in sorted(range(N), key=lambda j: (level[j], j)):
            z[i] = rhs[perm[i]] - sum(Lx[k][i] * z[k] for k in rowsL[i])
        depth = np.zeros(N, dtype=np.int64)
        for j in range(N - 1, -1, -1):
            depth[j] = 0 if parent[j] < 0 else depth[parent[j]] + 1
        x = z.copy()
        for j in sorted(range(N), key=lambda j: (depth[j], j)):
            x[j] = z[j] / d[j] - sum(Lx[j][i] * x[i] for i in Lrows[j])
        out = np.empty(N)
        out[perm] = x
        return out
    return d, solve


@pytest.mark.parametrize("seed", range(4))
def test_level_scheduled_left_looking_model_matches_splu(seed):
    rng = np.random.default_rng(100 + seed)
    n, m = 40, 60
    F = sp.random(n, n, density=0.08, random_state=rng)
    P = (F @ F.T + sp.diags(rng.uniform(0, 1, n) * (rng.uniform(size=n) < 0.5))).tocsc()
    A = sp.random(m, n, density=0.06, random_state=rng, format="csc")
    rho = rng.uniform(0.01, 10.0, m)
    K = _kkt(P, A, 1e-6, rho)
    perm, parent, colcount, level = E.ldl_symbolic(P, A)
    d, solve = _ldl_model(K, perm, parent, level)
    assert int((d > 0).sum()) == n                       # the inertia check of the device factorisation
    r = rng.standard_normal(n + m)
    x = solve(r)
    ref = spla.splu(K).solve(r)
    assert np.linalg.norm(x - ref) <= 1e-13 * np.linalg.norm(ref), np.linalg.norm(x - ref) / np.linalg.norm(ref)


def test_settings_select_the_device_ldl_plugin_and_sharding_refuses_it():
    st = cosmo_b200.Settings(kkt_solver="DeviceLdlKKTSolver")
    assert st.to_struct().kkt_solver == E.KKT_LDL == 3
    with pytest.raises(E.EngineError) as ei:                  # the CPU plugin with AMD ordering stays refused
        cosmo_b200.Settings(kkt_solver="QdldlKKTSolver").to_struct()
    assert "DeviceLdlKKTSolver" in str(ei.value)
    P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(30, 40, 0.2, seed=0)
    shard = sharding.make_shard(P, q, A, b, sets, rank=0, world=2)
    with pytest.raises(E.EngineError) as ei:
        sharding.create_engine(shard, st, dist=object())
    assert ei.value.code == E.ERR_UNSUPPORTED


def test_symbolic_entry_validates_its_input():
    with pytest.raises(E.EngineError) as ei:
        E.ldl_symbolic(sp.identity(3, format="csc"), sp.csc_matrix((2, 4)))
    assert ei.value.code == E.ERR_INVALID
