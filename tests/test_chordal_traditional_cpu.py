"""The traditional transformation of a chordal decomposition (compact_transformation = false): A' = [A H; 0 -I],
b' = [b; 0], square PsdCone cones decomposed as well, the reverse s = H s', mu = H mu' / overlap count, and the flat
maps the device takes (decomposition_arrays with traditional = True, forward_arrays).  The solves run on the CPU oracle.

The problems restate the reference's DecompositionTests/chordal_decomposition_triangle.jl and psd_completion.jl with
NumPy data on their patterns."""
import copy
import os
import shutil
import subprocess

import numpy as np
import pytest
import scipy.sparse as sp

import cosmo_b200
from cosmo_b200 import chordal, engine as E, model as M
from oracle import cosmo_oracle as O
from oracle.bridge import to_oracle_cones

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SQRT2 = np.sqrt(2.0)


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


def _sym(rng, n):
    a = rng.random((n, n))
    return 0.5 * (a + a.T)


def _pos_def(rng, n, lo, hi):
    """generate_pos_def_matrix (COSMOTestUtils.jl:11-19)"""
    Q, _ = np.linalg.qr(rng.random((n, n)))
    X = (Q * (rng.random(n) * (hi - lo) + lo)) @ Q.T
    return 0.5 * (X + X.T)


def _svec(X):
    return O.extract_upper_triangle(X, SQRT2)


def four_cone_problem(triangle=False, seed=144545):
    """chordal_decomposition_triangle.jl:8-57: [PsdCone(16), ZeroSet(2), PsdCone(16), PsdCone(9)] with one variable;
    cones 1 and 3 have chordal patterns, cone 4 is dense.  triangle: the PsdConeTriangle twin (:75-97)."""
    rng = np.random.default_rng(seed)
    A1 = _sym(rng, 4)
    A1[0, 2] = A1[0, 3] = A1[2, 0] = A1[3, 0] = 0.0
    a2 = rng.random(2)
    A3 = _sym(rng, 4)
    A3[1, 3] = A3[3, 1] = A3[0, 2] = A3[2, 0] = A3[1, 2] = A3[2, 1] = 0.0
    A4 = _sym(rng, 3)
    S = [X + (np.linalg.eigvalsh(X)[0] + 1.0) * np.eye(len(X)) for X in (A1, A3, A4)]
    x = rng.random(1)
    a = np.concatenate([A1.ravel(order="F"), a2, A3.ravel(order="F"), A4.ravel(order="F")])
    b = a * x[0] + np.concatenate([S[0].ravel(order="F"), [0.0, 0.0], S[1].ravel(order="F"), S[2].ravel(order="F")])
    Y = [_pos_def(rng, 4, 0.1, 1.0), None, _pos_def(rng, 4, 0.1, 1.0), _pos_def(rng, 3, 0.1, 1.0)]
    y = np.concatenate([Y[0].ravel(order="F"), rng.random(2), Y[2].ravel(order="F"), Y[3].ravel(order="F")])
    q = -a @ y * np.ones(1)
    P = sp.csc_matrix((1, 1))
    if not triangle:
        return P, q, sp.csc_matrix(a[:, None]), b, [M.PsdCone(16), M.ZeroSet(2), M.PsdCone(16), M.PsdCone(9)]
    B1, B3, B4 = b[:16].reshape(4, 4, order="F"), b[18:34].reshape(4, 4, order="F"), b[34:].reshape(3, 3, order="F")
    at = np.concatenate([_svec(A1), a2, _svec(A3), _svec(A4)])
    bt = np.concatenate([_svec(B1), b[16:18], _svec(B3), _svec(B4)])
    return P, q, sp.csc_matrix(at[:, None]), bt, [M.PsdConeTriangle(10), M.ZeroSet(2), M.PsdConeTriangle(10),
                                                  M.PsdConeTriangle(6)]


def pattern_sdp(seed=144545):
    """feasible_sdp_with_pattern(rng, pattern2) (chordal_decomposition_triangle.jl:150-156, COSMOTestUtils.jl:93-123):
    one 9 x 9 PsdConeTriangle with a chordal pattern"""
    rng = np.random.default_rng(seed)
    pat = np.ones((9, 9))
    pat[0, 4:] = 0
    pat[1, 5:] = 0
    pat[2, 5:] = 0
    pat[3, 8] = 0
    pat = np.triu(pat) + np.triu(pat, 1).T
    S = np.where(pat != 0, _pos_def(rng, 9, 0.1, 2.0), 0.0)
    A1 = np.where(pat != 0, np.triu(rng.random((9, 9))), 0.0)
    A1 = np.triu(A1) + np.triu(A1, 1).T
    x = rng.random(1)
    b = A1.ravel(order="F") * x[0] + S.ravel(order="F")
    Y = _pos_def(rng, 9, 0.1, 1.0)
    q = -(A1.ravel(order="F") @ Y.ravel(order="F")) * np.ones(1)
    return (sp.csc_matrix((1, 1)), q, sp.csc_matrix(_svec(A1)[:, None]), _svec(b.reshape(9, 9, order="F")),
            [M.PsdConeTriangle(45)])


def completion_problem(seed=144545):
    """psd_completion.jl:13-33: one PsdCone(16) whose pattern splits into two cliques"""
    rng = np.random.default_rng(seed)
    A1 = _sym(rng, 4)
    A1[0, 2] = A1[0, 3] = A1[2, 0] = A1[3, 0] = 0.0
    S1 = np.where(A1 != 0, _pos_def(rng, 4, 0.1, 2.0), 0.0)
    x = rng.random(1)
    b = A1.ravel(order="F") * x[0] + S1.ravel(order="F")
    Y = _pos_def(rng, 4, 0.1, 1.0)
    q = -(A1.ravel(order="F") @ Y.ravel(order="F")) * np.ones(1)
    return sp.csc_matrix((1, 1)), q, sp.csc_matrix(A1.ravel(order="F")[:, None]), b, [M.PsdCone(16)]


def mixed_problem():
    """a Nonnegatives block, the four-cone problem's square cones and a triangle with a pattern: plain rows on both
    sides of every decomposed cone"""
    P, q, A, b, sets = four_cone_problem()
    Pt, qt, At, bt, setst = four_cone_problem(triangle=True)
    rng = np.random.default_rng(5)
    An = sp.csc_matrix(rng.standard_normal((3, 1)))
    A2 = sp.vstack([An, A, At], format="csc")
    b2 = np.concatenate([rng.standard_normal(3), b, bt])
    return P, q, A2, b2, [M.Nonnegatives(3)] + sets + setst


def solve(P, q, A, b, sets, info=None, complete_dual=False):
    """an oracle solve of (P, q, A, b, sets); with `info`, a decomposed problem reversed to the original coordinates"""
    r = O.solve(sp.csc_matrix(P), np.asarray(q), sp.csc_matrix(A), np.asarray(b), to_oracle_cones(sets), O.Settings())
    assert r.status == "Solved", r.status
    if info is None:
        return r.obj_val, r.x, r.s, r.y
    x, s, mu = chordal.reverse(info, r.x, r.s, -r.y, complete_dual=complete_dual)
    return r.obj_val, x, s, -mu


def _square_blocks(s):
    return s[:16].reshape(4, 4, order="F"), s[18:34].reshape(4, 4, order="F")


def _triangle_blocks(s):
    """Symmetric(populate_upper_triangle(...), :U) of both decomposable cones"""
    out = []
    for v in (s[:10], s[12:22]):
        U = O.populate_upper_triangle(v, 4, 1.0 / SQRT2)
        out.append(np.triu(U) + np.triu(U, 1).T)
    return out


def test_nomerge_cliques_and_augmented_problem():
    P, q, A, b, sets = four_cone_problem()
    P2, q2, A2, b2, sets2, info = chordal.decompose(P, q, A, b, sets, merge="none", compact=False)
    assert not info.compact
    assert [sorted(c.tolist()) for _, c in info.blocks[0]] == [[0, 1], [1, 2, 3]]
    assert [sorted(c.tolist()) for _, c in info.blocks[2]] == [[0, 1], [0, 3], [2, 3]]
    assert set(info.blocks) == {0, 2}                      # cone 4 is dense: kept whole
    assert [type(S).__name__ for S in sets2] == ["ZeroSet", "PsdCone", "PsdCone", "ZeroSet", "PsdCone", "PsdCone",
                                                 "PsdCone", "PsdCone"]
    assert [S.dim for S in sets2] == [43, 4, 9, 2, 4, 4, 4, 9]
    nH = sum(S.dim for S in sets2[1:])
    assert info.num_overlaps == nH and A2.shape == (43 + nH, 1 + nH) and b2.shape == (43 + nH,)
    # A' = [A H; 0 -I], one +1.0 per column of H in the row it copies
    D = A2.toarray()
    assert np.array_equal(D[:43, :1], A.toarray()) and np.array_equal(D[43:, 1:], -np.eye(nH)) and not D[43:, :1].any()
    H = D[:43, 1:]
    assert np.array_equal(H.sum(axis=0), np.ones(nH)) and np.array_equal(np.argmax(H, axis=0), info.h_rows)
    assert np.array_equal(P2.toarray(), np.zeros((1 + nH, 1 + nH))) and np.array_equal(q2, np.concatenate([q, np.zeros(nH)]))
    assert np.array_equal(b2, np.concatenate([b, np.zeros(nH)]))
    # both triangles of every clique block: row (1, 2) of the clique {1, 2, 3} (0-based) is entry (0, 1) and (1, 0)
    start, c = info.blocks[0][1]
    assert info.h_rows[start - 43:start - 43 + 9].tolist() == [i + 4 * j for j in c for i in c]


@pytest.mark.parametrize("compact", [True, False])
def test_triangle_decompositions_match_the_square_ones(compact):
    # chordal_decomposition_triangle.jl:164-175: undecomposed vs. decomposed, square vs. triangle
    P, q, A, b, sets = four_cone_problem()
    Pt, qt, At, bt, setst = four_cone_problem(triangle=True)
    o1, _, s1, _ = solve(P, q, A, b, sets)
    dec = chordal.decompose(P, q, A, b, sets, merge="clique_graph", compact=False)
    assert dec[5].blocks
    o2, _, s2, _ = solve(*dec[:5], info=dec[5])
    o3, _, s3, _ = solve(Pt, qt, At, bt, setst)
    dec = chordal.decompose(Pt, qt, At, bt, setst, merge="clique_graph", compact=compact)
    assert dec[5].blocks and dec[5].compact == compact
    o4, _, s4, _ = solve(*dec[:5], info=dec[5])
    assert abs(o1 - o2) < 1e-4 and abs(o1 - o3) < 1e-4 and abs(o2 - o4) < 1e-4
    for X1, X2, X3, X4 in zip(_square_blocks(s1), _square_blocks(s2), _triangle_blocks(s3), _triangle_blocks(s4)):
        assert np.abs(X1 - X2).max() < 1e-5 and np.abs(X2 - X3).max() < 1e-5 and np.abs(X3 - X4).max() < 1e-5


def test_reassembled_duals_satisfy_the_dual_equation():
    # chordal_decomposition_triangle.jl:150-187 (res5 - res7): A' y + q = 0 for the undecomposed problem and both
    # decompositions with complete_dual; the undecomposed dual is PSD
    P, q, A, b, sets = pattern_sdp()
    _, _, _, y5 = solve(P, q, A, b, sets)
    assert np.linalg.eigvalsh(O.populate_upper_triangle(y5, 9, 1.0 / SQRT2)).min() > -1e-6
    for compact in (True, False):
        dec = chordal.decompose(P, q, A, b, sets, merge="clique_graph", compact=compact)
        assert dec[5].blocks
        _, _, _, y = solve(*dec[:5], info=dec[5], complete_dual=True)
        assert np.abs(A.T @ y + q).max() < 1e-3
    assert np.abs(A.T @ y5 + q).max() < 1e-3


def test_square_psd_completion():
    # psd_completion.jl:36-58: NoMerge, complete_dual, the traditional transformation of a square cone
    P, q, A, b, sets = completion_problem()
    P2, q2, A2, b2, sets2, info = chordal.decompose(P, q, A, b, sets, merge="none", compact=False)
    assert [sorted(c.tolist()) for _, c in info.blocks[0]] == [[0, 1], [1, 2, 3]]
    _, _, _, y1 = solve(P, q, A, b, sets)
    _, _, s, y = solve(P2, q2, A2, b2, sets2, info=info, complete_dual=True)
    Y1 = y1.reshape(4, 4, order="F")
    Y = y.reshape(4, 4, order="F")
    assert np.linalg.eigvalsh(0.5 * (Y1 + Y1.T)).min() > -1e-6
    assert np.array_equal(Y, Y.T) and np.linalg.eigvalsh(Y).min() > -1e-6
    # the completion reads the upper triangle (Symmetric(mat(-mu), :U)) and only fills entries outside the cliques:
    # those inside are the mean of their clique copies
    _, _, _, y_raw = solve(P2, q2, A2, b2, sets2, info=info, complete_dual=False)
    inside = np.zeros((4, 4), dtype=bool)
    for _, c in info.blocks[0]:
        inside[np.ix_(c, c)] = True
    upper = inside & np.triu(np.ones((4, 4), dtype=bool))
    assert np.array_equal(_bits(Y[upper]), _bits(y_raw.reshape(4, 4, order="F")[upper]))
    assert not y_raw.reshape(4, 4, order="F")[~inside].any() and Y[~inside].all()


def _literal_reverse(info, x2, s2, mu2):
    """reverse_decomposition! + fill_dual_variables! (chordal_decomposition.jl:136-168) as written: s = H s'[m+1:end],
    mu = H mu'[m+1:end] divided by the number of ones in each row of H that has more than one"""
    m, nH = info.m_orig, len(info.h_rows)
    H = sp.csc_matrix((np.ones(nH), (info.h_rows, np.arange(nH))), shape=(m, nH))
    s = H @ s2[m:]
    mu = H @ mu2[m:]
    cnt = np.asarray(H.sum(axis=1)).ravel()
    mu[cnt > 1] = mu[cnt > 1] / cnt[cnt > 1]
    return x2[:info.n_orig].copy(), s, mu


CASES = [("four_cone", "none"), ("four_cone", "clique_graph"), ("four_cone_triangle", "none"),
         ("pattern_sdp", "none"), ("pattern_sdp", "clique_graph"), ("completion", "none"), ("mixed", "none"),
         ("mixed", "clique_graph"), ("c5_300", "clique_graph")]


def _problem(name):
    if name == "c5_300":
        rows, cols, w = cosmo_b200.problems.banded_random_graph(300, 3.0, 20, seed=1)
        return cosmo_b200.problems.maxcut_dual_sdp(300, rows, cols, w)
    return {"four_cone": four_cone_problem, "four_cone_triangle": lambda: four_cone_problem(triangle=True),
            "pattern_sdp": pattern_sdp, "completion": completion_problem, "mixed": mixed_problem}[name]()


def _iterates(A2, seed):
    """values of very different magnitude, so that the summation order shows in the last bits, and signed zeros"""
    rng = np.random.default_rng(seed)
    out = []
    for k in (A2.shape[1], A2.shape[0], A2.shape[0]):
        v = rng.standard_normal(k) * 10.0 ** rng.integers(-8, 8, k)
        v[rng.random(k) < 0.1] = -0.0
        out.append(v)
    return out


@pytest.mark.parametrize("name,merge", CASES)
def test_reverse_is_the_literal_h_product(name, merge):
    P, q, A, b, sets = _problem(name)
    P2, q2, A2, b2, sets2, info = chordal.decompose(P, q, A, b, sets, merge=merge, compact=False)
    assert info.blocks
    x2, s2, mu2 = _iterates(A2, 7)
    want = _literal_reverse(info, x2, s2, mu2)
    got = chordal.reverse(info, x2, s2, mu2)
    for g, w in zip(got, want):
        assert np.array_equal(_bits(g), _bits(w))
    # the flat map of the device replays it bit for bit
    d = chordal.decomposition_arrays(info, A2.shape[1], A2.shape[0])
    assert d.traditional and len(d.mu_src) == 0 and (d.n, d.m) == (A2.shape[1], A2.shape[0])
    chordal.validate_decomposition_arrays(d)
    for g, w in zip(chordal.reverse_from_arrays(d, x2, s2, mu2), want):
        assert np.array_equal(_bits(g), _bits(w))
    if name == "mixed":
        assert len(d.plain) == 5 and len(d.cones) == 4 and sorted(c.dim for c in d.cones) == [10, 10, 16, 16]
    # the completion schedules of square cones replay psd_complete on mat(-mu)
    for k, c in zip(info.blocks, d.cones):
        assert c.row_offset == info.cone_offsets[k] and c.dim == info.sets_orig[k].dim
        chordal.validate_schedule(c, info.m_orig, square_ok=True)


@pytest.mark.parametrize("name,merge", CASES)
def test_forward_map_reproduces_the_decomposition(name, merge):
    P, q, A, b, sets = _problem(name)
    b = b.copy()
    P2, q2, A2, b2, sets2, info = chordal.decompose(P, q, A, b, sets, merge=merge, compact=False)
    f = chordal.forward_arrays(info, A, A2.shape[1], A2.shape[0])
    A0 = M._sorted_csc(A)
    Ax, qx, bx = chordal.forward_values(f, A0.data, q, b)
    assert np.array_equal(_bits(Ax), _bits(M._sorted_csc(A2).data))
    assert np.array_equal(_bits(qx), _bits(q2)) and np.array_equal(_bits(bx), _bits(b2))
    # a_src: A's entries, then -1 for every entry of H and -2 for every entry of -I
    nH = info.num_overlaps
    assert np.count_nonzero(f.a_src == -1) == nH == np.count_nonzero(f.a_src == -2)
    # b_src: the identity on the first m rows except the uncovered ones, -1 below
    m = info.m_orig
    unc = f.b_uncovered.astype(bool)
    assert np.array_equal(f.b_src[:m][~unc], np.nonzero(~unc)[0]) and (f.b_src[:m][unc] == -1).all()
    assert (f.b_src[m:] == -1).all()
    if unc.any():
        # new values, with -0.0 where no clique holds the row: a fresh decomposition writes +0.0 there, as the map does
        rng = np.random.default_rng(3)
        Anew = A0.copy()
        Anew.data = rng.standard_normal(A0.nnz)
        bnew = rng.standard_normal(m)
        bnew[unc] = -0.0
        fresh = chordal.decompose(P, q, Anew, bnew, sets, merge=merge, compact=False)
        Ax, _, bx = chordal.forward_values(f, Anew.data, None, bnew)
        assert np.array_equal(_bits(Ax), _bits(M._sorted_csc(fresh[2]).data))
        assert np.array_equal(_bits(bx), _bits(fresh[3]))
        assert not len(chordal.uncovered_rows(f, bnew))
        bnew[np.nonzero(unc)[0][0]] = 1.0
        assert len(chordal.uncovered_rows(f, bnew)) == 1


def test_compact_transformation_keeps_square_cones():
    P, q, A, b, sets = four_cone_problem()
    P2, q2, A2, b2, sets2, info = chordal.decompose(P, q, A, b, sets, merge="none", compact=True)
    assert not info.blocks and info.compact
    assert (A2 != sp.csc_matrix(A)).nnz == 0 and np.array_equal(b2, b) and [type(S) for S in sets2] == [type(S) for S in sets]
    # the same problem through the model: compact_transformation = true leaves it undecomposed
    from tests.test_model_decompose_cpu import _OracleEngine
    _OracleEngine.instances.clear()
    orig = M._eng.Engine
    M._eng.Engine = _OracleEngine
    try:
        for compact in (True, False):
            model = cosmo_b200.Model()
            model.set(P, q, A, b, sets, cosmo_b200.Settings(scaling=0, decompose=True, merge_strategy="NoMerge",
                                                             compact_transformation=compact, complete_dual=True))
            res = model.optimize()
            assert res.status == "Solved" and res.s.shape == res.y.shape == (43,)
            assert (model._dec is None) == compact
            eng = _OracleEngine.instances[-1]
            assert eng.A.shape == ((43, 1) if compact else (43 + model._dec.num_overlaps, 1 + model._dec.num_overlaps))
            if not compact:
                # the traditional decomposition through the model: the reverse of chordal.reverse on its iterates
                assert isinstance(eng.cones[0], O.ZeroSet) and eng.cones[0].dim == 43
                Y = res.y[:16].reshape(4, 4, order="F")
                assert np.linalg.eigvalsh(Y).min() > -1e-6
    finally:
        M._eng.Engine = orig


def _traditional_arrays():
    P, q, A, b, sets = mixed_problem()
    P2, q2, A2, b2, sets2, info = chordal.decompose(P, q, A, b, sets, merge="none", compact=False)
    return chordal.decomposition_arrays(info, A2.shape[1], A2.shape[0])


def _mutations():
    def set_(attr, fn):
        def f(d):
            setattr(d, attr, fn(np.array(getattr(d, attr))))
        return f

    def cone(attr, fn, k=0):
        def f(d):
            setattr(d.cones[k], attr, fn(np.array(getattr(d.cones[k], attr))))
        return f

    def bump(a, i, v):
        a.flat[i] += v
        return a

    return {
        "mu_src_given": lambda d: setattr(d, "mu_src", d.s_src[d.s_ptr[1:] - 1].copy()),
        "row_out_of_range": set_("row", lambda a: bump(a, len(a) - 1, 10 ** 6)),
        "row_in_plain_block": set_("row", lambda a: np.concatenate([[0], a[1:]])),
        "s_src_out_of_range": set_("s_src", lambda a: bump(a, 0, 10 ** 6)),
        "s_ptr_inconsistent": set_("s_ptr", lambda a: bump(a, 1, -1)),
        "plain_out_of_range": set_("plain", lambda a: bump(a, 2, 10 ** 6)),
        "square_cone_rows_out_of_range": cone("row_offset", lambda a: a + 10 ** 6),
        "square_cone_bad_dim": cone("dim", lambda a: a - 1),
        "new_of_not_a_permutation": cone("new_of", lambda a: np.zeros_like(a)),
    }


@pytest.mark.parametrize("what", sorted(_mutations()))
def test_validator_rejects_malformed_traditional_maps(what):
    d = _traditional_arrays()
    chordal.validate_decomposition_arrays(d)
    bad = copy.deepcopy(d)
    _mutations()[what](bad)
    with pytest.raises(ValueError):
        chordal.validate_decomposition_arrays(bad)


def test_square_layout_belongs_to_the_traditional_map():
    d = _traditional_arrays()
    assert any(c.dim == c.N ** 2 for c in d.cones)
    compact = copy.deepcopy(d)
    compact.traditional = False
    compact.mu_src = compact.s_src[compact.s_ptr[1:] - 1]
    with pytest.raises(NotImplementedError):
        chordal.validate_decomposition_arrays(compact)


def test_entry_point_is_exported_and_declared(tmp_path):
    lib = E.load_library()
    assert "cosmo_b200_set_decomposition_noncompact" in E.EXPORTS and hasattr(lib, "cosmo_b200_set_decomposition_noncompact")
    assert lib.cosmo_b200_abi_version() == 4
    assert lib.cosmo_b200_set_decomposition_noncompact(None, None) == E.ERR_INVALID     # no handle
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "probe.c"
    src.write_text('#include <stdio.h>\n#include "cosmo_b200.h"\n'
                   "int main(void) {\n"
                   "  int (*fn)(cosmo_b200_handle*, const cosmo_b200_decomposition*) = cosmo_b200_set_decomposition_noncompact;\n"
                   '  printf("%d %d\\n", fn(NULL, NULL), COSMO_B200_ABI_VERSION);\n'
                   "  return 0;\n}\n")
    lib_path = lib._name
    exe = str(tmp_path / "probe")
    subprocess.run([cc, "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), lib_path,
                    "-Wl,-rpath," + os.path.dirname(lib_path), "-o", exe], check=True)
    out = subprocess.run([exe], check=True, capture_output=True, text=True).stdout.split()
    assert out == [str(E.ERR_INVALID), "4"]
