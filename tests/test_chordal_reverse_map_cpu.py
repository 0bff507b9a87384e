"""The flat maps of the device reverse (chordal.decomposition_arrays): replayed in NumPy they must give exactly what
chordal.reverse and chordal.psd_complete give, and malformed maps must be refused."""
import copy

import numpy as np
import pytest
import scipy.sparse as sp

import cosmo_b200
from cosmo_b200 import chordal
from tests import golden_problems as G


def _g6():
    A1, A2, B, c = G.g6_chordal_sdp_data()
    A = sp.csc_matrix(-np.column_stack([G._svec(A1), G._svec(A2)]))
    return sp.csc_matrix((2, 2)), c, A, G._svec(B), [cosmo_b200.PsdConeTriangle(45)]


def _c5(nv):
    rows, cols, w = cosmo_b200.problems.banded_random_graph(nv, 3.0, 20, seed=1)
    return cosmo_b200.problems.maxcut_dual_sdp(nv, rows, cols, w)


def _mixed():
    # a Nonnegatives block, the G6 cone (decomposed) and a dense 3 x 3 cone (kept whole): plain rows on both sides
    P, q, A6, b6, _ = _g6()
    rng = np.random.default_rng(3)
    An = sp.csc_matrix(rng.standard_normal((4, 2)))
    Ad = sp.csc_matrix(rng.standard_normal((6, 2)))
    A = sp.vstack([An, A6, Ad], format="csc")
    b = np.concatenate([rng.standard_normal(4), b6, rng.standard_normal(6)])
    return P, q, A, b, [cosmo_b200.Nonnegatives(4), cosmo_b200.PsdConeTriangle(45), cosmo_b200.PsdConeTriangle(6)]


CASES = [("g6", m) for m in ("none", "parent_child_reference", "clique_graph")] + \
        [("c5_%d" % nv, m) for nv in (300, 2000) for m in ("none", "parent_child_reference", "clique_graph")] + \
        [("mixed", "clique_graph")]


def _problem(name):
    if name == "g6":
        return _g6()
    if name == "mixed":
        return _mixed()
    return _c5(int(name.split("_")[1]))


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


@pytest.mark.parametrize("name,merge", CASES)
def test_flat_map_reverse_is_bit_identical(name, merge):
    P, q, A, b, sets = _problem(name)
    P2, q2, A2, b2, sets2, info = chordal.decompose(P, q, A, b, sets, merge=merge)
    assert info.blocks
    d = chordal.decomposition_arrays(info, A2.shape[1], A2.shape[0])
    chordal.validate_decomposition_arrays(d)
    assert (d.n, d.m) == (A2.shape[1], A2.shape[0])
    if name == "mixed":
        assert len(d.plain) == 2 and len(d.cones) == 1
    rng = np.random.default_rng(7)
    # values of very different magnitude so that the summation order shows in the last bits
    x2 = rng.standard_normal(A2.shape[1]) * 10.0 ** rng.integers(-8, 8, A2.shape[1])
    s2 = rng.standard_normal(A2.shape[0]) * 10.0 ** rng.integers(-8, 8, A2.shape[0])
    mu2 = rng.standard_normal(A2.shape[0])
    want = chordal.reverse(info, x2, s2, mu2, complete_dual=False)
    got = chordal.reverse_from_arrays(d, x2, s2, mu2)
    for g, w in zip(got, want):
        assert np.array_equal(_bits(g), _bits(w))


def _pd_on_cliques(nv, rows, cols, seed):
    """diagonally dominant on the pattern: every clique block is positive definite"""
    rng = np.random.default_rng(seed)
    W = np.eye(nv) * 4.0
    W[rows, cols] = W[cols, rows] = rng.uniform(-0.5, 0.5, len(rows))
    return W


@pytest.mark.parametrize("nv,merge", [(9, "none"), (300, "clique_graph"), (2000, "clique_graph"), (2000, "parent_child_reference")])
def test_flat_schedule_matches_psd_complete(nv, merge):
    if nv == 9:
        P, q, A, b, sets = _g6()
        P2, q2, A2, b2, sets2, info = chordal.decompose(P, q, A, b, sets, merge=merge)
        tree = info.trees[0]
        cl = np.zeros((9, 9), dtype=bool)
        for c in tree.cliques:
            cl[np.ix_(c, c)] = True
        r, c = np.nonzero(np.triu(cl, 1))
        W = _pd_on_cliques(9, r, c, 0)
    else:
        rows, cols, _ = cosmo_b200.problems.banded_random_graph(nv, 3.0, 20, seed=1)
        rows, cols = np.asarray(rows), np.asarray(cols)
        tree = chordal.chordal_cliques(nv, rows, cols)
        tree = chordal.clique_graph_merge(tree) if merge == "clique_graph" else chordal.parent_child_merge_reference(tree)
        W = _pd_on_cliques(nv, rows, cols, 0)
    sched = chordal.completion_schedule(tree, W.shape[0])
    chordal.validate_schedule(sched)
    want = chordal.psd_complete(W, tree, assume_symmetric=True)
    got = chordal.psd_complete_from_schedule(W, sched)
    assert np.linalg.norm(got - want) <= 1e-13 * np.linalg.norm(want)


def _g6_arrays():
    P, q, A, b, sets = _mixed()
    P2, q2, A2, b2, sets2, info = chordal.decompose(P, q, A, b, sets, merge="none")
    return chordal.decomposition_arrays(info, A2.shape[1], A2.shape[0])


def _mutations():
    def set_(attr, fn):
        def f(d):
            setattr(d, attr, fn(np.array(getattr(d, attr))))
        return f

    def cone(attr, fn):
        def f(d):
            setattr(d.cones[0], attr, fn(np.array(getattr(d.cones[0], attr))))
        return f

    def bump(a, i, v):
        a.flat[i] += v
        return a

    return {
        "row_out_of_range": set_("row", lambda a: bump(a, len(a) - 1, 10 ** 6)),
        "rows_not_increasing": set_("row", lambda a: a[::-1].copy()),
        "row_in_plain_block": set_("row", lambda a: np.concatenate([[0], a[1:]])),
        "s_src_out_of_range": set_("s_src", lambda a: bump(a, 0, 10 ** 6)),
        "s_ptr_inconsistent": set_("s_ptr", lambda a: bump(a, 1, -1)),
        "mu_not_last_writer": set_("mu_src", lambda a: bump(a, 0, 1)),
        "plain_out_of_range": set_("plain", lambda a: bump(a, 2, 10 ** 6)),
        "new_of_not_a_permutation": cone("new_of", lambda a: np.zeros_like(a)),
        "step_breaks_leading_block": cone("steps", lambda a: bump(a, 6, 1)),
        "known_vertex_not_seen": cone("idx", lambda a: bump(a, len(a) - 1, 9)),
        "cone_rows_out_of_range": cone("row_offset", lambda a: a + 10 ** 6),
    }


@pytest.mark.parametrize("what", sorted(_mutations()))
def test_validator_rejects_malformed_maps(what):
    d = _g6_arrays()
    chordal.validate_decomposition_arrays(d)
    bad = copy.deepcopy(d)
    _mutations()[what](bad)
    with pytest.raises(ValueError):
        chordal.validate_decomposition_arrays(bad)


def test_validator_refuses_the_square_layout():
    d = _g6_arrays()
    d.cones[0].dim = d.cones[0].N ** 2
    with pytest.raises(NotImplementedError):
        chordal.validate_decomposition_arrays(d)
