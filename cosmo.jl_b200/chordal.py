"""Host-side chordal decomposition (SURVEY.md Appendix B) -- the producer of the clique batch.

Stays on the host like the reference's `src/chordal_decomposition/` (north-star);
what the GPU consumes is only the augmented `(P', q', A', b')`, the cone list with
one `PsdConeTriangle` per clique, and the row map used to sum the blocks back.

Restated (not ported) from the reference:
  * aggregate sparsity pattern of a PSD cone   chordal_decomposition.jl:100-115
  * chordal extension + elimination tree        trees.jl:634-642 (the reference calls QDLDL with an AMD
    ordering; neither is available here, so a minimum-degree elimination with explicit fill is used --
    any perfect elimination ordering gives a valid decomposition, only the clique set differs)
  * supernodes / cliques / clique tree          trees.jl:390-513 (Pothen-Sun rule: v joins a child's
    supernode iff |hadj(child)| = |hadj(v)| + 1)
  * merge strategy                              NoMerge; ParentChildMerge(t_fill, t_size) in two flavours --
    `parent_child` (bottom-up variant with the clique-size rule, the one the C5 measurements use) and
    `parent_child_reference` (the reference's top-down walk, clique_merging.jl:262-283, 641-648);
    `clique_graph` = CliqueGraphMerge, the reference default (reduced clique graph, complexity weights,
    permissible edges, clique tree rebuilt by Kruskal; clique_graph.jl, clique_merging.jl:34-67, 204-259, 305-600)
  * compact ("clique tree based") augmentation  transformations.jl:152-374: every clique becomes a
    PsdConeTriangle block; an entry (i,j) inside the separator of a clique gets a new variable with +1 in
    the clique's row and -1 in the parent's row of the same (i,j)
  * traditional augmentation                     transformations.jl:1-138 (compact_transformation = false):
    A' = [A H; 0 -I], b' = [b; 0] with one column of H per row of every clique block and of every kept cone; square
    PsdCone cones are decomposed too (clique blocks PsdCone(nc^2) over both triangles)
  * reverse_decomposition!                       chordal_decomposition.jl:129-213 (x truncated, s = sum of
    blocks, mu = block value; traditional: s = H s', mu = H mu' / overlap count)
  * psd_completion! / psd_complete!               chordal_decomposition.jl:215-311 (`complete_dual`): the entries
    of the dual matrix outside the pattern are chosen so that Y = -mat(mu) is positive semidefinite -- the
    maximum-determinant completion, clique by clique from the root of the clique tree
    (Vandenberghe & Andersen, Chordal Graphs and Semidefinite Optimization, alg. 10.2)
"""
from __future__ import annotations

import heapq
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import numpy as np
from sortedcontainers import SortedList
import scipy.sparse as sp

from . import model as M


def svec_index(i: int, j: int) -> int:
    """position of (i,j), i<=j (0-based), in the column-major upper triangle (convexset.jl:432-442)"""
    return j * (j + 1) // 2 + i


def svec_to_ij(k: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """inverse of svec_index (svec_to_mat, trees.jl:697-719)"""
    k = np.asarray(k, dtype=np.int64)
    j = ((np.sqrt(8.0 * k + 1.0) - 1.0) / 2.0).astype(np.int64)
    j = np.where((j + 1) * (j + 2) // 2 <= k, j + 1, j)
    j = np.where(j * (j + 1) // 2 > k, j - 1, j)
    return k - j * (j + 1) // 2, j


@dataclass
class CliqueTree:
    cliques: List[np.ndarray]          # sorted vertex lists
    parent: List[int]                  # -1 for roots
    sep: List[np.ndarray]              # clique ∩ parent clique (sorted)
    order: np.ndarray                  # elimination order used


def chordal_cliques(nv: int, rows: np.ndarray, cols: np.ndarray) -> CliqueTree:
    """Minimum-degree elimination with explicit fill -> maximal cliques and their tree."""
    adj: List[set] = [set() for _ in range(nv)]
    for a, b in zip(rows.tolist(), cols.tolist()):
        if a != b:
            adj[a].add(b)
            adj[b].add(a)
    heap = [(len(adj[v]), v) for v in range(nv)]
    heapq.heapify(heap)
    done = np.zeros(nv, dtype=bool)
    pos = np.empty(nv, dtype=np.int64)
    order: List[int] = []
    hadj: List[Optional[List[int]]] = [None] * nv
    while heap:
        d, v = heapq.heappop(heap)
        if done[v] or d != len(adj[v]):
            continue
        done[v] = True
        pos[v] = len(order)
        order.append(v)
        nb = list(adj[v])
        hadj[v] = nb
        for a in nb:
            adj[a].discard(v)
        for ia in range(len(nb)):      # fill: the higher neighbourhood becomes a clique
            a = nb[ia]
            sa = adj[a]
            for ib in range(ia + 1, len(nb)):
                b = nb[ib]
                if b not in sa:
                    sa.add(b)
                    adj[b].add(a)
        for a in nb:
            heapq.heappush(heap, (len(adj[a]), a))
        adj[v] = set()
    # elimination tree: parent = earliest-eliminated higher neighbour
    par = np.full(nv, -1, dtype=np.int64)
    for v in range(nv):
        if hadj[v]:
            par[v] = min(hadj[v], key=lambda u: pos[u])
    # Pothen-Sun supernodes
    absorbing_child = np.full(nv, -1, dtype=np.int64)
    for u in order:
        p = par[u]
        if p >= 0 and absorbing_child[p] < 0 and len(hadj[u]) == len(hadj[p]) + 1:
            absorbing_child[p] = u
    snode = np.full(nv, -1, dtype=np.int64)
    lowest: List[int] = []
    top: List[int] = []
    for v in order:
        c = absorbing_child[v]
        if c >= 0:
            snode[v] = snode[c]
            top[snode[v]] = v
        else:
            snode[v] = len(lowest)
            lowest.append(v)
            top.append(v)
    cliques, parent, seps = [], [], []
    for k, v in enumerate(lowest):
        cl = np.array(sorted([v] + list(hadj[v])), dtype=np.int64)
        cliques.append(cl)
        t = top[k]
        p = par[t]
        parent.append(int(snode[p]) if p >= 0 else -1)
    for k, cl in enumerate(cliques):
        if parent[k] < 0:
            seps.append(np.zeros(0, dtype=np.int64))
        else:
            seps.append(np.intersect1d(cl, cliques[parent[k]]))
    return CliqueTree(cliques, parent, seps, np.array(order, dtype=np.int64))


def parent_child_merge(tree: CliqueTree, t_fill: int = 8, t_size: int = 8) -> CliqueTree:
    """ParentChildMerge (clique_merging.jl:278-285, 641-648): children are merged into their parent
    when the fill-in (|C_par|-|sep|)(|C|-|sep|) <= t_fill or both supernodes are small."""
    n = len(tree.cliques)
    cl = [set(c.tolist()) for c in tree.cliques]
    parent = list(tree.parent)
    alive = [True] * n
    children: List[List[int]] = [[] for _ in range(n)]
    for k, p in enumerate(parent):
        if p >= 0:
            children[p].append(k)
    # visit children before parents
    depth = [0] * n
    for k in range(n):
        d, p = 0, parent[k]
        while p >= 0:
            d += 1
            p = parent[p]
        depth[k] = d
    for k in sorted(range(n), key=lambda i: -depth[i]):
        p = parent[k]
        if p < 0 or not alive[k]:
            continue
        while not alive[p]:
            p = parent[p]
        sep = len(cl[k] & cl[p])
        fill = (len(cl[p]) - sep) * (len(cl[k]) - sep)
        if fill <= t_fill or max(len(cl[k]) - sep, len(cl[p]) - sep) <= t_size:
            cl[p] |= cl[k]
            alive[k] = False
            for ch in children[k]:
                parent[ch] = p
                children[p].append(ch)
    idx = {k: i for i, k in enumerate([k for k in range(n) if alive[k]])}
    cliques, par2, seps = [], [], []
    for k in range(n):
        if not alive[k]:
            continue
        p = parent[k]
        while p >= 0 and not alive[p]:
            p = parent[p]
        c = np.array(sorted(cl[k]), dtype=np.int64)
        cliques.append(c)
        par2.append(idx[p] if p >= 0 else -1)
    for k, c in enumerate(cliques):
        seps.append(np.intersect1d(c, cliques[par2[k]]) if par2[k] >= 0 else np.zeros(0, dtype=np.int64))
    return CliqueTree(cliques, par2, seps, tree.order)


def _tree_from_sets(cl: List[set], parent: List[int], order: np.ndarray) -> CliqueTree:
    cliques = [np.array(sorted(c), dtype=np.int64) for c in cl]
    seps = [np.intersect1d(c, cliques[parent[k]]) if parent[k] >= 0 else np.zeros(0, dtype=np.int64)
            for k, c in enumerate(cliques)]
    return CliqueTree(cliques, list(parent), seps, order)


def _post_order(parent: List[int]) -> List[int]:
    """children before parents, roots last (post_order, trees.jl)"""
    n = len(parent)
    children: List[List[int]] = [[] for _ in range(n)]
    roots = []
    for k, p in enumerate(parent):
        (children[p] if p >= 0 else roots).append(k)
    out: List[int] = []
    for r in roots:
        stack = [(r, 0)]
        while stack:
            v, i = stack.pop()
            if i < len(children[v]):
                stack.append((v, i + 1))
                stack.append((children[v][i], 0))
            else:
                out.append(v)
    return out


def parent_child_merge_reference(tree: CliqueTree, t_fill: int = 8, t_size: int = 8, snd_post: Optional[List[int]] = None,
                                 return_log: bool = False):
    """ParentChildMerge exactly as the reference walks it (clique_merging.jl:98-106 initialise!, :262-283
    traverse / evaluate, :177-201 merge_child!, :295-303 update_strategy!): the supernode tree is traversed in
    descending topological order (root first); clique c is merged into its *current* parent when
        (|C_par| - |sep_c|) (|C_c| - |sep_c|) <= t_fill   or   max(|snd_c|, |snd_par|) <= t_size ,
    with snd = clique minus its separator.  A merge moves only the child's supernode into the parent's."""
    n = len(tree.cliques)
    sep = [set(x.tolist()) for x in tree.sep]
    snd = [set(c.tolist()) - sep[k] for k, c in enumerate(tree.cliques)]
    parent = list(tree.parent)
    children: List[set] = [set() for _ in range(n)]
    for k, p in enumerate(parent):
        if p >= 0:
            children[p].add(k)
    post = list(snd_post) if snd_post is not None else _post_order(parent)
    log_pairs, log_dec = [], []
    for ind in range(n - 2, -1, -1):             # clique_ind = length(snd) - 1 ... 1 (1-based)
        c = post[ind]
        par = parent[c]
        if par < 0:                               # a second root (disconnected pattern): nothing to merge into
            continue
        d_snd, d_sep = len(snd[c]), len(sep[c])
        p_snd, p_sep = len(snd[par]), len(sep[par])
        fill = ((p_snd + p_sep) - d_sep) * ((d_snd + d_sep) - d_sep)
        do_merge = fill <= t_fill or max(d_snd, p_snd) <= t_size
        log_pairs.append((par, c))
        log_dec.append(do_merge)
        if do_merge:                              # merge_child!
            snd[par] |= snd[c]
            snd[c] = set()
            sep[c] = set()
            for g in children[c]:
                parent[g] = par
            parent[c] = -2                        # removed
            children[par].discard(c)
            children[par] |= children[c]
            children[c] = set()
    alive = [k for k in range(n) if parent[k] != -2]
    idx = {k: i for i, k in enumerate(alive)}
    cl = [snd[k] | sep[k] for k in alive]
    par2 = [idx[parent[k]] if parent[k] >= 0 else -1 for k in alive]
    out = _tree_from_sets(cl, par2, tree.order)
    return (out, log_pairs, log_dec) if return_log else out


# ---- CliqueGraphMerge (the reference's default merge strategy) ------------------------------------------
def reduced_clique_graph(cliques: List[set], seps: List[set]) -> Tuple[List[int], List[int]]:
    """compute_reduced_clique_graph! (clique_graph.jl:19-49, Habib & Stacho): for every separator, largest
    first, the cliques that contain it form the separator graph H (an edge when two of them intersect in more
    than the separator); two such cliques get an edge of the reduced clique graph iff they lie in different
    connected components of H.  Returns (rows, cols) with row > col; separators that occur several times in
    `seps` contribute their edges several times (the reference then *adds* the duplicate weights)."""
    rows: List[int] = []
    cols: List[int] = []
    members: Dict[int, set] = {}
    for k, c in enumerate(cliques):
        for v in c:
            members.setdefault(v, set()).add(k)
    for separator in sorted(seps, key=len, reverse=True):      # sort! is stable, as is sorted()
        if not separator:
            # the empty separator of a root would link every pair of cliques from different connected components
            # of the pattern (O(p^2) edges of weight n1^3 + n2^3 - (n1+n2)^3 < 0 that can never be merged and never
            # make an edge impermissible); they are left out, so a disconnected pattern keeps a forest
            continue
        # cliques that contain the separator, in index order (inverted index instead of a scan over all cliques)
        holders = sorted((members[v] for v in separator), key=len)
        ind = sorted(set.intersection(*holders)) if holders else []
        H: Dict[int, List[int]] = {v: [] for v in ind}
        for a in range(len(ind)):
            for b_ in range(a + 1, len(ind)):
                ca, cb = ind[a], ind[b_]
                if (cliques[ca] & cliques[cb]) != separator:    # inter_equal, clique_graph.jl:113-131
                    H[ca].append(cb)
                    H[cb].append(ca)
        comp: Dict[int, int] = {}
        for v in ind:                                            # find_components (DFS)
            if v in comp:
                continue
            comp[v] = v
            stack = [v]
            while stack:
                u = stack.pop()
                for w in H[u]:
                    if w not in comp:
                        comp[w] = v
                        stack.append(w)
        for a in range(len(ind)):
            for b_ in range(a + 1, len(ind)):
                ca, cb = ind[a], ind[b_]
                if comp[ca] != comp[cb]:
                    rows.append(max(ca, cb))
                    cols.append(min(ca, cb))
    return rows, cols


def _complexity_weight(c_a: set, c_b: set) -> float:
    """ComplexityWeight: |Ca|^3 + |Cb|^3 - |Ca u Cb|^3 (clique_merging.jl:24-31, 395-405)"""
    return float(len(c_a) ** 3 + len(c_b) ** 3 - len(c_a | c_b) ** 3)


class CliqueGraph:
    """State of CliqueGraphMerge (clique_merging.jl:55-67): weighted edges of the reduced clique graph and the
    adjacency table.  Edges are keyed (row, col) with row > col and iterated in CSC order (col, then row), the
    order Julia's `findmax(edges.nzval)` / `findnz` see them in."""

    def __init__(self, cliques: List[set], seps: List[set]):
        self.snd = [set(c) for c in cliques]
        self.num = len(cliques)
        rows, cols = reduced_clique_graph(self.snd, [set(x) for x in seps])
        self.edges: Dict[Tuple[int, int], float] = {}
        for r, c in zip(rows, cols):                             # sparse(rows, cols, weights): duplicates add up
            self.edges[(r, c)] = self.edges.get((r, c), 0.0) + _complexity_weight(self.snd[r], self.snd[c])
        self.edges = {e: w for e, w in self.edges.items() if w != 0.0}
        # the candidate order of traverse(): weight descending, ties in CSC order (col, then row) -- kept incrementally
        self._ranked = SortedList((-w, e[1], e[0]) for e, w in self.edges.items())
        self.adj: Dict[int, set] = {k: set() for k in range(self.num)}
        for (r, c) in self.edges:
            self.adj[r].add(c)
            self.adj[c].add(r)
        self.log: List[Tuple[int, int, bool]] = []

    def _csc(self):
        return sorted(self.edges, key=lambda e: (e[1], e[0]))

    def permissible(self, edge) -> bool:                        # ispermissible, clique_graph.jl:149-158
        c1, c2 = edge
        for nb in self.adj[c1] & self.adj[c2]:
            if (self.snd[c1] & self.snd[nb]) != (self.snd[c2] & self.snd[nb]):
                return False
        return True

    def traverse(self):                                          # clique_merging.jl:242-259
        for (_, c, r) in self._ranked:                           # = sortperm(weights, rev = true), stable in CSC order
            if self.permissible((r, c)):
                return (r, c)
        return None

    def traverse_by_sorting(self):
        """the literal restatement (sort all edges at every call); kept as the cross-check of the incremental order"""
        order = self._csc()
        if not order:
            return None
        by_weight = sorted(order, key=lambda e: -self.edges[e])   # stable: ties keep CSC order
        for e in by_weight:
            if self.permissible(e):
                return e
        return None

    def _set_edge(self, key, w: float) -> None:
        old = self.edges.pop(key, None)
        if old is not None:
            self._ranked.remove((-old, key[1], key[0]))
        if w != 0.0:                                             # dropzeros!
            self.edges[key] = w
            self._ranked.add((-w, key[1], key[0]))

    def merge(self, edge) -> None:                              # merge_two_cliques! + update_strategy!
        c1, removed = edge
        self.snd[c1] |= self.snd[removed]
        self.snd[removed] = set()
        self.num -= 1
        neighbors = set(self.adj[c1])
        new_neighbors = self.adj[removed] - neighbors - {c1}
        for nb in (neighbors - {removed}) | new_neighbors:
            self._set_edge((max(c1, nb), min(c1, nb)), _complexity_weight(self.snd[c1], self.snd[nb]))
        for nb in self.adj[removed]:                           # every edge of `removed` (adj is a superset of edges)
            self._set_edge((max(removed, nb), min(removed, nb)), 0.0)
        self.adj[c1] |= new_neighbors
        for nb in new_neighbors:
            self.adj[nb].add(c1)
        for nb in self.adj[removed]:
            self.adj[nb].discard(removed)
        del self.adj[removed]

    def run(self) -> None:                                      # _merge_cliques!, clique_merging.jl:112-133
        while self.num > 1:
            cand = self.traverse()
            if cand is None:
                break
            do_merge = self.edges[cand] >= 0                    # evaluate, :286-293
            self.log.append((cand[0], cand[1], do_merge))
            if not do_merge:
                break
            self.merge(cand)

    def clique_tree(self, order: np.ndarray) -> CliqueTree:
        """clique_tree_from_graph! (clique_merging.jl:577-600): maximum-weight spanning tree of the clique
        graph under the weights |Ci & Cj| (Kruskal, :480-506), rooted at the clique that holds the vertex
        eliminated last (:532-550)."""
        alive = [k for k in range(len(self.snd)) if self.snd[k]]
        inter = {e: float(len(self.snd[e[0]] & self.snd[e[1]])) for e in self._csc()}
        edges_sorted = sorted(inter, key=lambda e: -inter[e])     # sortperm(V, rev = true), stable
        uf = {k: k for k in alive}

        def find(a):
            while uf[a] != a:
                uf[a] = uf[uf[a]]
                a = uf[a]
            return a

        mst: Dict[int, List[int]] = {k: [] for k in alive}
        found = 0
        for (r, c) in edges_sorted:
            if found >= len(alive) - 1:
                break
            ra, rb = find(r), find(c)
            if ra != rb:
                uf[ra] = rb
                mst[r].append(c)
                mst[c].append(r)
                found += 1
        parent = {k: -1 for k in alive}
        seen = set()
        last = int(order[-1]) if len(order) else -1
        roots = [k for k in alive if last in self.snd[k]][:1] + alive
        for r in roots:                                         # the pattern may be disconnected: several roots
            if r in seen:
                continue
            seen.add(r)
            stack = [r]
            while stack:
                u = stack.pop()
                for v in sorted(mst[u]):
                    if v not in seen:
                        seen.add(v)
                        parent[v] = u
                        stack.append(v)
        idx = {k: i for i, k in enumerate(alive)}
        return _tree_from_sets([self.snd[k] for k in alive], [idx[parent[k]] if parent[k] >= 0 else -1 for k in alive], order)


def clique_graph_merge(tree: CliqueTree) -> CliqueTree:
    """CliqueGraphMerge(edge_weight = ComplexityWeight()), the reference's default `merge_strategy`
    (settings.jl; clique_merging.jl:34-67, 147-166)."""
    g = CliqueGraph([set(c.tolist()) for c in tree.cliques], [set(x.tolist()) for x in tree.sep])
    g.run()
    return g.clique_tree(tree.order)


@dataclass
class DecompositionInfo:
    n_orig: int
    m_orig: int
    sets_orig: list
    # for every decomposed cone: list of (new_row_start, clique vertices)
    blocks: Dict[int, List[Tuple[int, np.ndarray]]] = field(default_factory=dict)
    row_map_plain: List[Tuple[int, int, int]] = field(default_factory=list)   # (old_start, new_start, dim)
    cone_offsets: Dict[int, int] = field(default_factory=dict)
    num_overlaps: int = 0
    clique_sizes: List[int] = field(default_factory=list)
    trees: Dict[int, "CliqueTree"] = field(default_factory=dict)   # clique tree of every decomposed cone
    # where the values of A' and b' come from (forward_arrays).  For every entry handed to the assembly of A', in that
    # order: its row, its column and its source -- the position in the CSR data of A, -1 for the constant +1.0 and -2 for
    # the constant -1.0 of an overlap column.  For every row of b' that takes a value of b: (row of b', row of b), and
    # whether it is a row of a clique block, where only the nonzero values of b are written (a -0.0 arrives as +0.0).
    a_rows: np.ndarray = field(default_factory=lambda: np.zeros(0, dtype=np.int64))
    a_cols: np.ndarray = field(default_factory=lambda: np.zeros(0, dtype=np.int64))
    a_src: np.ndarray = field(default_factory=lambda: np.zeros(0, dtype=np.int64))
    b_new: np.ndarray = field(default_factory=lambda: np.zeros(0, dtype=np.int64))
    b_old: np.ndarray = field(default_factory=lambda: np.zeros(0, dtype=np.int64))
    b_clique: np.ndarray = field(default_factory=lambda: np.zeros(0, dtype=bool))
    # the transformation: compact (clique tree based) or traditional (A' = [A H; 0 -I]); for the traditional one the
    # original row of every column of H (blocks and row_map_plain then point at row m_orig + column of the block's first
    # entry, and num_overlaps counts the columns of H)
    compact: bool = True
    h_rows: np.ndarray = field(default_factory=lambda: np.zeros(0, dtype=np.int64))


def _aggregate_pattern(A, b, off: int, S):
    """find_aggregate_sparsity + row_ind_to_matrix_indices (chordal_decomposition.jl:100-115, trees.jl:655-694): the (i, j)
    of every row of the cone at rows off.. that holds an entry of A or b, or None when the pattern with the diagonal
    flagged covers every row (a dense cone is kept, chordal_decomposition.jl:53-60).  A: CSR."""
    N, dim = S.sqrt_dim, S.dim
    # straight from the row pointers (slicing the CSR matrix would copy a 50-million-row cone: C5 has N = 10 000)
    ip = A.indptr
    a_rows = np.nonzero(ip[off + 1:off + dim + 1] - ip[off:off + dim])[0]
    nz_rows = np.unique(np.concatenate([a_rows, np.nonzero(b[off:off + dim])[0]]))
    v = np.arange(N, dtype=np.int64)
    if isinstance(S, M.PsdCone):                                # column-major: row i + N j
        ii, jj, diag_rows = nz_rows % N, nz_rows // N, v + N * v
    else:
        (ii, jj), diag_rows = svec_to_ij(nz_rows), v * (v + 1) // 2 + v
    if len(np.union1d(nz_rows, diag_rows)) >= dim:
        return None
    return ii, jj


def _merged(tree: CliqueTree, merge: str) -> CliqueTree:
    if merge == "parent_child":
        return parent_child_merge(tree)
    if merge == "parent_child_reference":
        return parent_child_merge_reference(tree)
    if merge == "clique_graph":
        return clique_graph_merge(tree)
    if merge != "none":
        raise ValueError("merge must be 'none', 'parent_child', 'parent_child_reference' or 'clique_graph'")
    return tree


def _clique_rows(S, c: np.ndarray) -> np.ndarray:
    """rows (cone-local) of the block of clique c, in the order of add_subblock_map! (transformations.jl:94-117): for a
    PsdCone all (vi, vj) column-major, for a PsdConeTriangle the upper triangle column-major"""
    c = np.asarray(c, dtype=np.int64)
    if isinstance(S, M.PsdCone):
        return (c[:, None] + S.sqrt_dim * c[None, :]).ravel(order="F")
    ai, bj = svec_to_ij(np.arange(len(c) * (len(c) + 1) // 2, dtype=np.int64))
    return c[bj] * (c[bj] + 1) // 2 + c[ai]


def decompose(P, q, A, b, sets, merge: str = "parent_child", min_dim: int = 3, compact: bool = True):
    """chordal_decomposition!(ws).  compact = True: the clique tree based transformation of PsdConeTriangle cones; square
    PsdCone cones stay whole (the reference defines it for triangles only, transformations.jl:267-268).  compact = False:
    the traditional transformation of both (_decompose_traditional).  Returns (P', q', A', b', sets', info)."""
    if not compact:
        return _decompose_traditional(P, q, A, b, sets, merge, min_dim)
    A = sp.csr_matrix(A)
    b = np.asarray(b, dtype=np.float64)
    m, n = A.shape
    info = DecompositionInfo(n, m, list(sets))
    rows_new: List[np.ndarray] = []
    cols_new: List[np.ndarray] = []
    vals_new: List[np.ndarray] = []
    src_new: List[np.ndarray] = []                               # source of every entry of vals_new (info.a_src)
    b_new: List[np.ndarray] = []
    b_map_new: List[np.ndarray] = []
    b_map_old: List[np.ndarray] = []
    b_map_clique: List[np.ndarray] = []
    sets_new = []
    row_ptr = 0
    n_new = n
    off = 0
    Acoo_by_row = A  # csr
    for k, S in enumerate(sets):
        dim = S.dim
        pattern = _aggregate_pattern(A, b, off, S) if isinstance(S, M.PsdConeTriangle) and S.sqrt_dim >= min_dim else None
        if pattern is not None:
            N = S.sqrt_dim
            ii, jj = pattern
            ip = A.indptr
            row_nnz = ip[off + 1:off + dim + 1] - ip[off:off + dim]
            a_rows = np.nonzero(row_nnz)[0]
        if pattern is None:
            sub = Acoo_by_row[off:off + dim].tocoo()
            rows_new.append(sub.row + row_ptr)
            cols_new.append(sub.col)
            vals_new.append(sub.data)
            src_new.append(np.arange(A.indptr[off], A.indptr[off + dim], dtype=np.int64))   # tocoo keeps the CSR order
            b_new.append(b[off:off + dim])
            b_map_new.append(np.arange(row_ptr, row_ptr + dim, dtype=np.int64))
            b_map_old.append(np.arange(off, off + dim, dtype=np.int64))
            b_map_clique.append(np.zeros(dim, dtype=bool))
            sets_new.append(S)
            info.row_map_plain.append((off, row_ptr, dim))
            row_ptr += dim
            off += dim
            continue
        tree = _merged(chordal_cliques(N, ii, jj), merge)
        # row offsets of the clique blocks
        starts = []
        for c in tree.cliques:
            starts.append(row_ptr)
            nc = len(c)
            row_ptr += nc * (nc + 1) // 2
        info.cone_offsets[k] = off
        info.trees[k] = tree
        info.blocks[k] = [(starts[t], tree.cliques[t]) for t in range(len(tree.cliques))]
        info.clique_sizes += [len(c) for c in tree.cliques]
        # owner (clique, local row) of every pattern entry; overlaps get +1/-1 columns
        owner: Dict[int, int] = {}
        for t, c in enumerate(tree.cliques):
            nc = len(c)
            in_sep = np.isin(c, tree.sep[t])
            loc = {int(v): a for a, v in enumerate(c)}
            par_t = tree.parent[t]
            par_loc = {int(v): a for a, v in enumerate(tree.cliques[par_t])} if par_t >= 0 else None
            ov_rows, ov_cols, ov_vals, ov_src = [], [], [], []
            for bj in range(nc):
                for ai in range(bj + 1):
                    gi, gj = int(c[ai]), int(c[bj])
                    new_row = starts[t] + svec_index(ai, bj)
                    if in_sep[ai] and in_sep[bj]:
                        pa, pb = par_loc[gi], par_loc[gj]
                        if pa > pb:
                            pa, pb = pb, pa
                        ov_rows += [new_row, starts[par_t] + svec_index(pa, pb)]
                        ov_cols += [n_new, n_new]
                        ov_vals += [1.0, -1.0]
                        ov_src += [-1, -2]
                        n_new += 1
                    else:
                        owner[svec_index(gi, gj)] = new_row
            if ov_rows:
                rows_new.append(np.array(ov_rows, dtype=np.int64))
                cols_new.append(np.array(ov_cols, dtype=np.int64))
                vals_new.append(np.array(ov_vals))
                src_new.append(np.array(ov_src, dtype=np.int64))
            sets_new.append(M.PsdConeTriangle(nc * (nc + 1) // 2))
        lo, hi = int(ip[off]), int(ip[off + dim])
        sub_row = np.repeat(a_rows, row_nnz[a_rows])             # cone-local row of every entry, CSR order
        mapped = np.array([owner[int(r)] for r in sub_row], dtype=np.int64) if hi > lo else np.zeros(0, dtype=np.int64)
        rows_new.append(mapped)
        cols_new.append(A.indices[lo:hi].astype(np.int64))
        vals_new.append(A.data[lo:hi].copy())
        src_new.append(np.arange(lo, hi, dtype=np.int64))
        b_map_new.append(np.fromiter(owner.values(), dtype=np.int64, count=len(owner)))
        b_map_old.append(off + np.fromiter(owner.keys(), dtype=np.int64, count=len(owner)))
        b_map_clique.append(np.ones(len(owner), dtype=bool))
        bseg = np.zeros(row_ptr - starts[0])
        nzb = np.nonzero(b[off:off + dim])[0]
        for r in nzb:
            bseg[owner[int(r)] - starts[0]] = b[off + r]
        b_new.append(bseg)
        off += dim
    info.num_overlaps = n_new - n
    rows_c = np.concatenate(rows_new) if rows_new else np.zeros(0, dtype=np.int64)
    cols_c = np.concatenate(cols_new) if cols_new else np.zeros(0, dtype=np.int64)
    vals_c = np.concatenate(vals_new) if vals_new else np.zeros(0)
    info.a_rows, info.a_cols = rows_c.astype(np.int64), cols_c.astype(np.int64)
    info.a_src = np.concatenate(src_new) if src_new else np.zeros(0, dtype=np.int64)
    info.b_new = np.concatenate(b_map_new) if b_map_new else np.zeros(0, dtype=np.int64)
    info.b_old = np.concatenate(b_map_old) if b_map_old else np.zeros(0, dtype=np.int64)
    info.b_clique = np.concatenate(b_map_clique) if b_map_clique else np.zeros(0, dtype=bool)
    A2 = sp.csc_matrix((vals_c, (rows_c, cols_c)), shape=(row_ptr, n_new))
    b2 = np.concatenate(b_new) if b_new else np.zeros(0)
    P2 = sp.block_diag([sp.csc_matrix(P), sp.csc_matrix((n_new - n, n_new - n))], format="csc")
    q2 = np.concatenate([np.asarray(q, dtype=np.float64), np.zeros(n_new - n)])
    return P2, q2, A2, b2, sets_new, info


def _decompose_traditional(P, q, A, b, sets, merge: str, min_dim: int):
    """find_decomposition_matrix! + augment_system! (transformations.jl:1-138): H has one column per row of a kept cone
    (the identity) and per entry of every clique block, each with a single +1.0 in the original row it copies, and
        A' = [A H; 0 -I],  b' = [b; 0],  P' = blockdiag(P, 0),  q' = [q; 0],
        sets' = ZeroSet(m), then every original cone or its cliques (PsdCone(nc^2) / PsdConeTriangle(nc(nc+1)/2)).
    Square PsdCone and PsdConeTriangle cones are decomposed; a cone whose clique tree has one clique is kept, as the
    reference does (chordal_decomposition.jl:64-69).  The one difference from the reference's [b; 0]: a row of a
    decomposed cone that lies in no clique gets +0.0 in b' (b is zero there, of either sign), so that new values mapped
    through forward_arrays, which writes +0.0 there, end where this decomposition of them ends."""
    A = sp.csr_matrix(A)
    b = np.asarray(b, dtype=np.float64)
    m, n = A.shape
    info = DecompositionInfo(n, m, list(sets), compact=False)
    h_rows: List[np.ndarray] = []
    sets_new = [M.ZeroSet(m)]
    covered = np.ones(m, dtype=bool)
    col, off = 0, 0
    for k, S in enumerate(sets):
        dim = S.dim
        tree = None
        if isinstance(S, (M.PsdConeTriangle, M.PsdCone)) and S.sqrt_dim >= min_dim:
            pattern = _aggregate_pattern(A, b, off, S)
            if pattern is not None:
                tree = _merged(chordal_cliques(S.sqrt_dim, *pattern), merge)
                if len(tree.cliques) == 1:
                    tree = None
        if tree is None:
            h_rows.append(np.arange(off, off + dim, dtype=np.int64))
            info.row_map_plain.append((off, m + col, dim))
            sets_new.append(S)
            col += dim
            off += dim
            continue
        info.cone_offsets[k] = off
        info.trees[k] = tree
        info.blocks[k] = []
        covered[off:off + dim] = False
        for c in tree.cliques:
            rows = off + _clique_rows(S, c)
            covered[rows] = True
            h_rows.append(rows)
            info.blocks[k].append((m + col, c))
            col += len(rows)
            nc = len(c)
            sets_new.append(M.PsdCone(nc * nc) if isinstance(S, M.PsdCone) else M.PsdConeTriangle(nc * (nc + 1) // 2))
        info.clique_sizes += [len(c) for c in tree.cliques]
        off += dim
    h = np.concatenate(h_rows) if h_rows else np.zeros(0, dtype=np.int64)
    nH = len(h)
    info.num_overlaps = nH
    info.h_rows = h
    # A in CSR order, then H (+1.0), then -I
    a_rows = np.repeat(np.arange(m, dtype=np.int64), np.diff(A.indptr))
    cols_h = n + np.arange(nH, dtype=np.int64)
    info.a_rows = np.concatenate([a_rows, h, m + np.arange(nH, dtype=np.int64)])
    info.a_cols = np.concatenate([A.indices.astype(np.int64), cols_h, cols_h])
    info.a_src = np.concatenate([np.arange(A.nnz, dtype=np.int64), np.full(nH, -1, dtype=np.int64),
                                 np.full(nH, -2, dtype=np.int64)])
    vals = np.concatenate([A.data, np.ones(nH), -np.ones(nH)])
    info.b_new = info.b_old = np.nonzero(covered)[0].astype(np.int64)
    info.b_clique = np.zeros(len(info.b_new), dtype=bool)
    A2 = sp.csc_matrix((vals, (info.a_rows, info.a_cols)), shape=(m + nH, n + nH))
    b2 = np.concatenate([np.where(covered, b, 0.0), np.zeros(nH)])
    P2 = sp.block_diag([sp.csc_matrix(P), sp.csc_matrix((nH, nH))], format="csc")
    q2 = np.concatenate([np.asarray(q, dtype=np.float64), np.zeros(nH)])
    return P2, q2, A2, b2, sets_new, info


def psd_complete(Y: np.ndarray, tree: CliqueTree, assume_symmetric: bool = False) -> np.ndarray:
    """psd_complete! (chordal_decomposition.jl:262-311): fill the entries of the symmetric matrix `Y` that lie
    outside the cliques of `tree` so that the result is positive semidefinite (given that every clique block
    is).  Cliques are visited parents first; for clique k with separator alpha = C_k & C_parent and residual
    nu = C_k minus alpha, the unknown entries between nu and eta = (vertices of the cliques visited so far) minus C_k are
        Y[eta, nu] = Y[eta, alpha] Y[alpha, alpha]^-1 Y[alpha, nu]
    (pseudo-inverse when the separator block is singular, as the reference's try/catch does).

    The vertices are renumbered in the order the traversal first meets them: the visited set is then a leading block,
    the residual of the current clique the next few indices, and the update is one product of a contiguous row block
    (rows of alpha are recomputed to themselves and restored, so known entries stay bit-identical)."""
    W = np.array(Y, dtype=np.float64)
    if not assume_symmetric:                 # the reference reads the upper triangle
        W = np.triu(W) + np.triu(W, 1).T
    N = W.shape[0]
    # traversal order (parents first) and the renumbering it induces
    order_k, new_of, residuals = _traversal(tree, N)
    perm = np.argsort(new_of)                              # perm[new] = old
    W = W[np.ix_(perm, perm)]
    seen = 0
    for k in order_k:
        nu_old = residuals[k]
        nn = len(nu_old)
        alpha_old = tree.sep[k] if tree.parent[k] >= 0 else np.zeros(0, dtype=np.int64)
        # the reference's nu = C_k minus alpha; vertices of alpha are always met before (they belong to the parent)
        lo, hi = seen, seen + nn                           # new indices of nu
        if seen and nn:
            if len(alpha_old):
                al = new_of[np.asarray(alpha_old, dtype=np.int64)]
                Waa = W[np.ix_(al, al)]
                Wan = W[al, lo:hi].copy()
                try:
                    Z = np.linalg.solve(Waa, Wan)
                    if not np.all(np.isfinite(Z)):
                        raise np.linalg.LinAlgError
                except np.linalg.LinAlgError:
                    Z = np.linalg.pinv(Waa) @ Wan
                blk = W[:seen, al] @ Z
                blk[al, :] = Wan                           # known entries (alpha x nu lies inside the clique) stay exact
            else:   # a new connected component: no coupling with what was completed before
                blk = np.zeros((seen, nn))
            # entries between nu and the OTHER members of its own clique are known as well: keep them
            c_new = new_of[np.asarray(tree.cliques[k], dtype=np.int64)]
            c_seen = c_new[c_new < seen]
            blk[c_seen, :] = W[c_seen, lo:hi]
            W[:seen, lo:hi] = blk
            W[lo:hi, :seen] = blk.T
        seen = hi
    inv = new_of                                           # old -> new
    return W[np.ix_(inv, inv)]


def _psd_complete_reference(Y: np.ndarray, tree: CliqueTree) -> np.ndarray:
    """the literal restatement (index sets per clique); kept as the cross-check of the renumbered version"""
    W = np.array(Y, dtype=np.float64)
    W = np.triu(W) + np.triu(W, 1).T
    ncl = len(tree.cliques)
    children: List[List[int]] = [[] for _ in range(ncl)]
    roots = []
    for k, p in enumerate(tree.parent):
        (children[p] if p >= 0 else roots).append(k)
    seen = np.zeros(W.shape[0], dtype=bool)
    stack = list(reversed(roots))
    while stack:
        k = stack.pop()
        c = tree.cliques[k]
        alpha = tree.sep[k] if tree.parent[k] >= 0 else np.zeros(0, dtype=np.int64)
        nu = np.setdiff1d(c, alpha)
        eta = np.nonzero(seen)[0]
        eta = np.setdiff1d(eta, c)
        if len(eta) and len(nu):
            if len(alpha):
                Waa = W[np.ix_(alpha, alpha)]
                Wan = W[np.ix_(alpha, nu)]
                try:
                    Z = np.linalg.solve(Waa, Wan)
                    if not np.all(np.isfinite(Z)):
                        raise np.linalg.LinAlgError
                except np.linalg.LinAlgError:
                    Z = np.linalg.pinv(Waa) @ Wan
                blk = W[np.ix_(eta, alpha)] @ Z
            else:
                blk = np.zeros((len(eta), len(nu)))
            W[np.ix_(eta, nu)] = blk
            W[np.ix_(nu, eta)] = blk.T
        seen[c] = True
        stack.extend(reversed(children[k]))
    return W


def _svec_to_mat(v: np.ndarray, N: int) -> np.ndarray:
    """populate_upper_triangle!(X, v, 1/sqrt 2) + symmetrise (convexset.jl:432-442).  The column-major upper triangle
    (0,0), (0,1), (1,1), (0,2) ... is the row-major lower triangle of the transpose: one masked assignment."""
    L = np.zeros((N, N))
    L[np.tri(N, dtype=bool)] = v
    d = np.diagonal(L).copy()
    X = L + L.T
    X *= 1.0 / np.sqrt(2.0)
    np.fill_diagonal(X, d)
    return X


def _mat_to_svec(X: np.ndarray) -> np.ndarray:
    """extract_upper_triangle!(X, v, sqrt 2) of a symmetric X: X[c, r] for r = 0.., c <= r, i.e. its row-major lower triangle"""
    N = X.shape[0]
    v = X[np.tri(N, dtype=bool)] * np.sqrt(2.0)
    j = np.arange(N, dtype=np.int64)
    v[j * (j + 1) // 2 + j] = np.diagonal(X)
    return v


def _traversal(tree: CliqueTree, N: int):
    """The clique order of `psd_complete` (parents first, children in order), its renumbering `new_of` (visited vertices
    form a leading block) and the residual of every clique."""
    ncl = len(tree.cliques)
    children: List[List[int]] = [[] for _ in range(ncl)]
    roots = []
    for k, p in enumerate(tree.parent):
        (children[p] if p >= 0 else roots).append(k)
    order_k: List[int] = []
    stack = list(reversed(roots))
    while stack:
        k = stack.pop()
        order_k.append(k)
        stack.extend(reversed(children[k]))
    new_of = np.full(N, -1, dtype=np.int64)
    nxt = 0
    residuals: Dict[int, np.ndarray] = {}
    for k in order_k:
        c = np.asarray(tree.cliques[k], dtype=np.int64)
        fresh = c[new_of[c] < 0]
        residuals[k] = fresh
        new_of[fresh] = np.arange(nxt, nxt + len(fresh))
        nxt += len(fresh)
    rest = np.nonzero(new_of < 0)[0]
    new_of[rest] = np.arange(nxt, nxt + len(rest))
    return order_k, new_of, residuals


@dataclass
class CompletionSchedule:
    """`psd_complete` of one N x N matrix as flat int64 arrays.  Step t (traversal order) completes the residual
    nu = new indices lo..hi-1 against the leading block 0..lo-1 (lo = hi of the step before, 0 for the first):
        W[r, nu] = W[r, alpha] Z,  W[alpha, alpha] Z = W[alpha, nu],   for every r < lo outside the clique,
    with alpha = idx[a0:a1] (the separator, new numbering) and idx[k0:k1] the clique's other members below lo, whose
    entries are known and stay as they are."""
    N: int
    row_offset: int            # first original row of the cone (0 for a bare matrix)
    dim: int                   # rows of the cone: N(N+1)/2 (PsdConeTriangle); N*N (PsdCone) in a traditional map only
    new_of: np.ndarray         # N: old vertex -> traversal position
    steps: np.ndarray          # (n_steps, 6): lo, hi, a0, a1, k0, k1
    idx: np.ndarray


@dataclass
class DecompositionArrays:
    """The map of `reverse` as flat int64 arrays (decomposition_arrays): plain rows are copied; an original row of a
    decomposed cone gets s = 0.0 + the clique rows s_src[s_ptr[i]:s_ptr[i+1]] in that order and mu = mu_src[i] (the
    last of them, the row the host loop writes last); rows in no clique stay 0.  A traditional map (s = H s') has no
    mu_src: mu = (0.0 + the same sum over mu') / the length of the list, and plain rows are 0.0 + the row."""
    n_orig: int
    m_orig: int
    n: int                     # decomposed problem
    m: int
    plain: np.ndarray          # (n_plain, 3): old_start, new_start, dim
    row: np.ndarray            # original rows of the decomposed cones, increasing
    s_ptr: np.ndarray          # len(row) + 1
    s_src: np.ndarray          # decomposed rows
    mu_src: np.ndarray         # len(row); empty in a traditional map
    cones: List[CompletionSchedule] = field(default_factory=list)
    traditional: bool = False  # the map of the traditional transformation (cosmo_b200_set_decomposition_noncompact)


def completion_schedule(tree: CliqueTree, N: int, row_offset: int = 0) -> CompletionSchedule:
    order_k, new_of, residuals = _traversal(tree, N)
    steps, idx = [], []
    seen = 0
    for k in order_k:
        nn = len(residuals[k])
        alpha = new_of[np.asarray(tree.sep[k], dtype=np.int64)] if tree.parent[k] >= 0 else np.zeros(0, dtype=np.int64)
        c_new = new_of[np.asarray(tree.cliques[k], dtype=np.int64)]
        other = c_new[(c_new < seen) & ~np.isin(c_new, alpha)]
        a0 = len(idx)
        idx.extend(alpha.tolist())
        k0 = len(idx)
        idx.extend(other.tolist())
        steps.append((seen, seen + nn, a0, k0, k0, len(idx)))
        seen += nn
    return CompletionSchedule(int(N), int(row_offset), int(N) * (int(N) + 1) // 2, new_of, np.array(steps, dtype=np.int64).reshape(-1, 6),
                              np.array(idx, dtype=np.int64))


def decomposition_arrays(info: DecompositionInfo, n: Optional[int] = None, m: Optional[int] = None) -> DecompositionArrays:
    """Flatten `info` for the device reverse (cosmo_b200_set_decomposition, or cosmo_b200_set_decomposition_noncompact
    for the traditional transformation).  n, m: size of the decomposed problem (default: what the blocks and row map
    imply)."""
    plain = np.array(info.row_map_plain, dtype=np.int64).reshape(-1, 3)
    orig_l, src_l = [], []
    cones = []
    m_imp = int((plain[:, 1] + plain[:, 2]).max()) if len(plain) else 0
    for k, blocks in info.blocks.items():                      # set order, then clique order: the host's loop
        S = info.sets_orig[k]
        off = info.cone_offsets[k]
        for start, c in blocks:
            rows = off + _clique_rows(S, c)
            orig_l.append(rows)
            src_l.append(start + np.arange(len(rows), dtype=np.int64))
            m_imp = max(m_imp, start + len(rows))
        sched = completion_schedule(info.trees[k], S.sqrt_dim, off)
        sched.dim = S.dim                                      # N*N for a PsdCone
        cones.append(sched)
    orig = np.concatenate(orig_l) if orig_l else np.zeros(0, dtype=np.int64)
    src = np.concatenate(src_l) if src_l else np.zeros(0, dtype=np.int64)
    perm = np.argsort(orig, kind="stable")                     # keeps the host's summation order within a row
    orig, src = orig[perm], src[perm]
    row, first, counts = np.unique(orig, return_index=True, return_counts=True)
    s_ptr = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    mu_src = src[s_ptr[1:] - 1] if len(row) and info.compact else np.zeros(0, dtype=np.int64)
    return DecompositionArrays(int(info.n_orig), int(info.m_orig), int(n if n is not None else info.n_orig + info.num_overlaps),
                               int(m if m is not None else m_imp), plain, row.astype(np.int64), s_ptr, src.astype(np.int64),
                               mu_src.astype(np.int64), cones, traditional=not info.compact)


def validate_schedule(c: CompletionSchedule, m_orig: Optional[int] = None, square_ok: bool = False) -> None:
    """The checks cosmo_b200_set_decomposition / cosmo_b200_psd_complete apply to a schedule: ValueError if one fails.
    square_ok: a schedule of a traditional map, where a cone may have the square PsdCone layout."""
    N = int(c.N)
    if N < 1:
        raise ValueError("schedule: N must be positive")
    square = c.dim == N * N and N > 1
    if m_orig is not None and square and not square_ok:
        raise NotImplementedError("schedule: the square PsdCone layout is not supported by the compact transformation")
    if m_orig is not None and ((not square and c.dim != N * (N + 1) // 2) or
                               not (0 <= c.row_offset and c.row_offset + c.dim <= m_orig)):
        raise ValueError("schedule: cone rows out of range")
    new_of = np.asarray(c.new_of)
    if new_of.shape != (N,) or not np.array_equal(np.sort(new_of), np.arange(N)):
        raise ValueError("schedule: new_of is not a permutation of 0..N-1")
    st = np.asarray(c.steps).reshape(-1, 6)
    idx = np.asarray(c.idx)
    lo_expect = 0
    for t, (lo, hi, a0, a1, k0, k1) in enumerate(st.tolist()):
        if lo != lo_expect or hi < lo or hi > N:
            raise ValueError("schedule: step %d does not continue the leading block" % t)
        if not (0 <= a0 <= a1 == k0 <= k1 <= len(idx)):
            raise ValueError("schedule: step %d index ranges are inconsistent" % t)
        known = idx[a0:k1]
        if len(known) and (known.min() < 0 or known.max() >= lo):
            raise ValueError("schedule: step %d refers to a vertex outside the leading block" % t)
        lo_expect = hi


def validate_decomposition_arrays(d: DecompositionArrays) -> None:
    """Every index in range and the maps consistent (the checks the C ABI applies): ValueError otherwise."""
    if min(d.n_orig, d.m_orig, d.n, d.m) < 0 or d.n_orig > d.n:
        raise ValueError("decomposition: bad dimensions")
    pl = np.asarray(d.plain).reshape(-1, 3)
    if len(pl) and ((pl < 0).any() or (pl[:, 0] + pl[:, 2] > d.m_orig).any() or (pl[:, 1] + pl[:, 2] > d.m).any()):
        raise ValueError("decomposition: plain rows out of range")
    row, s_ptr, s_src, mu_src = (np.asarray(a) for a in (d.row, d.s_ptr, d.s_src, d.mu_src))
    if len(row) and (row.min() < 0 or row.max() >= d.m_orig or (np.diff(row) <= 0).any()):
        raise ValueError("decomposition: rows out of range or not increasing")
    if s_ptr.shape != (len(row) + 1,) or s_ptr[0] != 0 or (np.diff(s_ptr) <= 0).any() or s_ptr[-1] != len(s_src):
        raise ValueError("decomposition: s_ptr is inconsistent")
    if len(s_src) and (s_src.min() < 0 or s_src.max() >= d.m):
        raise ValueError("decomposition: s_src out of range")
    if d.traditional:
        if len(mu_src):
            raise ValueError("decomposition: a traditional map has no mu_src (mu is the mean over s_src)")
    elif mu_src.shape != row.shape or (len(row) and not np.array_equal(mu_src, s_src[s_ptr[1:] - 1])):
        raise ValueError("decomposition: mu_src is not the last clique row of each row")
    cover = np.zeros(d.m_orig, dtype=np.int8)
    for old, _, dim in pl.tolist():
        cover[old:old + dim] += 1
    cover[row] += 1
    if (cover > 1).any():
        raise ValueError("decomposition: an original row is written twice")
    for c in d.cones:
        validate_schedule(c, d.m_orig, square_ok=d.traditional)


def reverse_from_arrays(d: DecompositionArrays, x2, s2, mu2):
    """`reverse(..., complete_dual=False)` replayed from the flat map (what the device gather pass computes)."""
    x = np.asarray(x2, dtype=np.float64)[:d.n_orig].copy()
    s = np.zeros(d.m_orig)
    mu = np.zeros(d.m_orig)
    s2 = np.asarray(s2, dtype=np.float64)
    mu2 = np.asarray(mu2, dtype=np.float64)
    zero = 0.0 if d.traditional else -0.0                    # -0.0 + v is v bit for bit; 0.0 + v makes a -0.0 +0.0
    for old, new, dim in np.asarray(d.plain).reshape(-1, 3).tolist():
        s[old:old + dim] = zero + s2[new:new + dim]
        mu[old:old + dim] = zero + mu2[new:new + dim]
    cnt = np.diff(d.s_ptr)

    def list_sum(v):
        acc = np.zeros(len(d.row))
        for t in range(int(cnt.max()) if len(cnt) else 0):   # position t of every row's list, in list order
            has = cnt > t
            acc[has] += v[d.s_src[d.s_ptr[:-1][has] + t]]
        return acc

    s[d.row] = list_sum(s2)
    if d.traditional:
        acc = list_sum(mu2)
        mu[d.row] = np.where(cnt > 1, acc / np.maximum(cnt, 1), acc)
    else:
        mu[d.row] = mu2[d.mu_src]
    return x, s, mu


@dataclass
class ForwardArrays:
    """Where the values of the decomposed problem come from (forward_arrays), as flat arrays.  A' in sorted CSC order:
    entry k is A.data[a_src[k]] (A in sorted CSC order), +1.0 for a_src[k] = -1, -1.0 for -2 (overlap columns).
    b'[i] = b[b_src[i]] for a plain row, 0.0 for b_src[i] = -1, and for a row of a clique block b_src[i] = -2 - r with r the
    row of b: b[r], where a zero of either sign arrives as +0.0 (`decompose` writes only the nonzero values there).
    q' = [q; 0] and P' = blockdiag(P, 0), whose stored values are P's in P's order: neither needs a map."""
    n_orig: int
    m_orig: int
    n: int                     # decomposed problem
    m: int
    nnzA_orig: int
    a_src: np.ndarray          # nnz(A')
    b_src: np.ndarray          # m
    b_uncovered: np.ndarray    # m_orig, uint8: 1 for a row of a decomposed cone that lies in no clique


def forward_arrays(info: DecompositionInfo, A0, n2: int, m2: int) -> ForwardArrays:
    """The value map of `decompose` as flat arrays (cosmo_b200_set_forward_map), from the row, column and source lists
    `decompose` assembled A' and b' from.  A0: the matrix `decompose` was given; n2, m2: size of the decomposed problem.
    A row of a decomposed cone outside every clique has no place in b': b must stay zero there (b_uncovered), or the
    aggregate pattern, and with it the decomposition, changes."""
    A0 = M._sorted_csc(A0)
    nnz0 = int(A0.nnz)
    # decompose() reads A row by row: CSR position -> sorted CSC position, by sending the positions through the same conversion
    tag = sp.csc_matrix((np.arange(1, nnz0 + 1, dtype=np.float64), A0.indices, A0.indptr), shape=A0.shape)
    csc_of_csr = sp.csr_matrix(tag).data.astype(np.int64) - 1
    src = np.array(info.a_src, dtype=np.int64)
    orig = src >= 0
    src[orig] = csc_of_csr[src[orig]]
    order = np.lexsort((info.a_rows, info.a_cols))             # sorted CSC order of A': by column, then row
    r, c = info.a_rows[order], info.a_cols[order]
    assert not np.any((np.diff(c) == 0) & (np.diff(r) == 0)), "two entries of A' share a position: the map is not one to one"
    a_src = src[order]
    assert np.array_equal(np.sort(a_src[a_src >= 0]), np.arange(nnz0)), "an entry of A is not used exactly once"
    b_src = np.full(int(m2), -1, dtype=np.int64)
    b_src[info.b_new] = np.where(info.b_clique, -2 - info.b_old, info.b_old)
    unc = np.ones(int(info.m_orig), dtype=np.uint8)
    unc[info.b_old] = 0
    f = ForwardArrays(int(info.n_orig), int(info.m_orig), int(n2), int(m2), nnz0, a_src, b_src, unc)
    validate_forward_arrays(f)
    return f


def validate_forward_arrays(f: ForwardArrays) -> None:
    """Every index in range, every entry of A used exactly once, every row of b used once or marked uncovered (the checks
    cosmo_b200_set_forward_map applies): ValueError otherwise."""
    if min(f.n_orig, f.m_orig, f.n, f.m, f.nnzA_orig) < 0 or f.n_orig > f.n:
        raise ValueError("forward map: bad dimensions")
    a_src, b_src, unc = np.asarray(f.a_src), np.asarray(f.b_src), np.asarray(f.b_uncovered)
    if b_src.shape != (f.m,) or unc.shape != (f.m_orig,) or a_src.ndim != 1:
        raise ValueError("forward map: an array has the wrong size")
    if len(a_src) and (a_src.min() < -2 or a_src.max() >= f.nnzA_orig):
        raise ValueError("forward map: a_src out of range")
    used = np.bincount(a_src[a_src >= 0], minlength=f.nnzA_orig)
    if (used != 1).any():
        raise ValueError("forward map: an entry of A is not used exactly once")
    b_row = np.where(b_src < -1, -2 - b_src, b_src)           # the source row; -1: none
    if len(b_row) and b_row.max() >= f.m_orig:
        raise ValueError("forward map: b_src out of range")
    used = np.bincount(b_row[b_row >= 0], minlength=f.m_orig)
    if (used + (unc != 0) != 1).any():
        raise ValueError("forward map: a row of b is used twice, or neither used nor marked uncovered")


def forward_values(f: ForwardArrays, Ax=None, q=None, b=None):
    """(A'.data, q', b') of the decomposed problem from values in the original coordinates (None stays None): what the
    device gather of cosmo_b200_update_matrices_original computes."""
    out = [None, None, None]
    if Ax is not None:
        Ax = np.asarray(Ax, dtype=np.float64) if f.nnzA_orig else np.zeros(1)
        out[0] = np.where(f.a_src >= 0, Ax[np.maximum(f.a_src, 0)], np.where(f.a_src == -1, 1.0, -1.0))
    if q is not None:
        out[1] = np.concatenate([np.asarray(q, dtype=np.float64), np.zeros(f.n - f.n_orig)])
    if b is not None:
        b = np.asarray(b, dtype=np.float64)
        b = b if f.m_orig else np.zeros(1)
        clique = b[np.maximum(-2 - f.b_src, 0)]
        out[2] = np.where(f.b_src >= 0, b[np.maximum(f.b_src, 0)], np.where((f.b_src == -1) | (clique == 0), 0.0, clique))
    return tuple(out)


def uncovered_rows(f: ForwardArrays, b) -> np.ndarray:
    """rows where `b` is nonzero although no clique holds them: such a b needs a new decomposition"""
    return np.nonzero((np.asarray(f.b_uncovered) != 0) & (np.asarray(b) != 0))[0]


def psd_complete_from_schedule(Y: np.ndarray, c: CompletionSchedule) -> np.ndarray:
    """`psd_complete(Y, tree, assume_symmetric=True)` replayed from the flat schedule."""
    new_of = np.asarray(c.new_of)
    perm = np.argsort(new_of)
    W = np.array(Y, dtype=np.float64)[np.ix_(perm, perm)]
    for lo, hi, a0, a1, k0, k1 in np.asarray(c.steps).reshape(-1, 6).tolist():
        if lo == 0 or hi == lo:
            continue
        al = c.idx[a0:a1]
        if len(al):
            Waa = W[np.ix_(al, al)]
            Wan = W[al, lo:hi]
            try:
                Z = np.linalg.solve(Waa, Wan)
                if not np.all(np.isfinite(Z)):
                    raise np.linalg.LinAlgError
            except np.linalg.LinAlgError:
                Z = np.linalg.pinv(Waa) @ Wan
            blk = W[:lo, al] @ Z
        else:
            blk = np.zeros((lo, hi - lo))
        known = c.idx[a0:k1]
        blk[known, :] = W[known, lo:hi]
        W[:lo, lo:hi] = blk
        W[lo:hi, :lo] = blk.T
    return W[np.ix_(new_of, new_of)]


def reverse(info: DecompositionInfo, x2, s2, mu2, complete_dual: bool = False):
    """reverse_decomposition! (chordal_decomposition.jl:129-213): x = x'[1:n]; s = sum of clique blocks;
    mu = the clique block's value (overlaps carry equal values at optimality).  With `complete_dual`
    (settings.complete_dual, :146) the entries of every decomposed dual matrix outside its cliques are
    filled by `psd_complete` so that y = -mu is in the PSD cone.
    The traditional transformation (info.compact False, chordal_decomposition.jl:136-168): s = H s'[m:] and
    mu = H mu'[m:] divided by each row's count of columns of H (rows in no clique: 0), H v summed as a sparse product
    sums, 0.0 + the copies in column order."""
    x = np.asarray(x2)[:info.n_orig].copy()
    if not info.compact:
        m, h = info.m_orig, info.h_rows
        s = np.zeros(m)
        mu = np.zeros(m)
        np.add.at(s, h, np.asarray(s2, dtype=np.float64)[m:m + len(h)])      # in index order: column order per row
        np.add.at(mu, h, np.asarray(mu2, dtype=np.float64)[m:m + len(h)])
        cnt = np.bincount(h, minlength=m)
        over = cnt > 1
        mu[over] /= cnt[over]
        if complete_dual:
            for k in info.blocks:
                _complete_cone(mu, info.sets_orig[k], info.cone_offsets[k], info.trees[k])
        return x, s, mu
    s = np.zeros(info.m_orig)
    mu = np.zeros(info.m_orig)
    for old, new, dim in info.row_map_plain:
        s[old:old + dim] = s2[new:new + dim]
        mu[old:old + dim] = mu2[new:new + dim]
    for k, blocks in info.blocks.items():
        off = info.cone_offsets[k]
        for start, c in blocks:
            nc = len(c)
            for bj in range(nc):
                gj = int(c[bj])
                gi = c[:bj + 1]
                orig = off + gj * (gj + 1) // 2 + gi
                seg = slice(start + svec_index(0, bj), start + svec_index(bj, bj) + 1)
                s[orig] += s2[seg]
                mu[orig] = mu2[seg]
        if complete_dual:
            _complete_cone(mu, info.sets_orig[k], off, info.trees[k])
    return x, s, mu


def _complete_cone(mu: np.ndarray, S, off: int, tree: CliqueTree) -> None:
    """complete!(mu, C, ...) of one decomposed cone at rows off.. (chordal_decomposition.jl:232-257), in place: a PsdCone
    from Symmetric(mat(-mu), :U), written back to all N^2 entries; a PsdConeTriangle from its scaled upper triangle."""
    N = S.sqrt_dim
    seg = slice(off, off + S.dim)
    if isinstance(S, M.PsdCone):
        Y = psd_complete((-mu[seg]).reshape(N, N, order="F"), tree)
        mu[seg] = -Y.ravel(order="F")
    else:
        Y = psd_complete(_svec_to_mat(-mu[seg], N), tree, assume_symmetric=True)
        mu[seg] = -_mat_to_svec(Y)
