"""The forward value map of a chordal decomposition (chordal.forward_arrays): new values on the pattern a problem was
decomposed for, sent through the map, must be bit for bit what chordal.decompose makes of the new data; malformed maps
must be refused; and Model.update must keep the engine of a decomposed model exactly when the decomposition still
holds."""
import copy

import numpy as np
import pytest
import scipy.sparse as sp

import cosmo_b200
from cosmo_b200 import chordal, engine as E, model as M
from tests import golden_problems as G
from tests.oracle_engine import OracleEngine


def _g6():
    A1, A2, B, c = G.g6_chordal_sdp_data()
    A = sp.csc_matrix(-np.column_stack([G._svec(A1), G._svec(A2)]))
    return sp.csc_matrix((2, 2)), c, A, G._svec(B), [cosmo_b200.PsdConeTriangle(45)]


def _banded(nv, seed):
    rows, cols, w = cosmo_b200.problems.banded_random_graph(nv, 3.0, 20, seed=seed)
    return cosmo_b200.problems.maxcut_dual_sdp(nv, rows, cols, w)


def _mixed():
    # a Nonnegatives block before the decomposed G6 cone and a dense 3 x 3 cone (kept whole) after it; P is not empty
    _, q, A6, b6, _ = _g6()
    rng = np.random.default_rng(3)
    An = sp.csc_matrix(0.1 * rng.standard_normal((4, 2)))
    Ad = sp.csc_matrix(0.1 * rng.standard_normal((6, 2)))
    A = sp.vstack([An, A6, Ad], format="csc")
    b = np.concatenate([5.0 + rng.random(4), b6, G._svec(5.0 * np.eye(3))])     # the added rows are slack around the G6 optimum
    P = sp.csc_matrix(np.array([[2.0, 0.5], [0.5, 1.0]]))
    return P, q, A, b, [cosmo_b200.Nonnegatives(4), cosmo_b200.PsdConeTriangle(45), cosmo_b200.PsdConeTriangle(6)]


PROBLEMS = {"g6": _g6, "banded_300": lambda: _banded(300, 1), "banded_700": lambda: _banded(700, 5), "mixed": _mixed}
MERGES = ["none", "parent_child", "parent_child_reference", "clique_graph"]


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


def _new_values(P, q, A, b, seed):
    """new random values on the same pattern (stored entries of P and A, nonzero rows of b)"""
    rng = np.random.default_rng(seed)
    P2, A2 = sp.csc_matrix(P, copy=True), sp.csc_matrix(A, copy=True)
    A2.data = rng.standard_normal(A2.nnz) + 3.0 * np.sign(rng.standard_normal(A2.nnz))      # never zero
    P2.data = P2.data * rng.uniform(0.5, 2.0)
    b2 = np.where(b != 0, rng.uniform(0.5, 2.0, len(b)) * np.sign(rng.standard_normal(len(b))), 0.0)
    return P2, rng.standard_normal(len(q)), A2, b2


@pytest.mark.parametrize("merge", MERGES)
@pytest.mark.parametrize("name", sorted(PROBLEMS))
def test_forward_map_reproduces_decompose_on_new_values(name, merge):
    P, q, A, b, sets = PROBLEMS[name]()
    A = M._sorted_csc(A)
    P1, q1, A1, b1, sets1, info = chordal.decompose(P, q, A, b, sets, merge=merge)
    assert info.blocks
    f = chordal.forward_arrays(info, A, A1.shape[1], A1.shape[0])
    chordal.validate_forward_arrays(f)
    assert (f.n_orig, f.m_orig, f.n, f.m, f.nnzA_orig) == (A.shape[1], A.shape[0], A1.shape[1], A1.shape[0], A.nnz)
    assert A1.has_sorted_indices and len(f.a_src) == A1.nnz
    assert np.count_nonzero(f.a_src < 0) == 2 * info.num_overlaps
    for seed in (11, 12):
        Pn, qn, An, bn = _new_values(P, q, A, b, seed)
        P2, q2, A2, b2, sets2, info2 = chordal.decompose(Pn, qn, An, bn, sets, merge=merge)
        assert np.array_equal(A2.indptr, A1.indptr) and np.array_equal(A2.indices, A1.indices)   # same pattern, same map
        assert not len(chordal.uncovered_rows(f, bn))
        Ax, qf, bf = chordal.forward_values(f, An.data, qn, bn)
        assert np.array_equal(_bits(Ax), _bits(A2.data))
        assert np.array_equal(_bits(qf), _bits(q2))
        assert np.array_equal(_bits(bf), _bits(b2))
        P2 = M._sorted_csc(P2)                           # P' = blockdiag(P, 0): P's values in P's order, empty columns after
        Ps = M._sorted_csc(Pn)
        assert np.array_equal(_bits(P2.data), _bits(Ps.data)) and np.array_equal(P2.indices, Ps.indices)
        assert np.array_equal(P2.indptr[:Ps.shape[1] + 1], Ps.indptr) and np.all(P2.indptr[Ps.shape[1]:] == Ps.nnz)
    # the data the map was built from, too
    Ax, qf, bf = chordal.forward_values(f, A.data, q, b)
    assert np.array_equal(_bits(Ax), _bits(A1.data)) and np.array_equal(_bits(bf), _bits(b1)) and np.array_equal(_bits(qf), _bits(q1))


def _mixed_map():
    P, q, A, b, sets = _mixed()
    P1, q1, A1, b1, sets1, info = chordal.decompose(P, q, A, b, sets, merge="none")
    return chordal.forward_arrays(info, A, A1.shape[1], A1.shape[0]), b


def _mutations():
    def at(attr, i, v):
        def f(m):
            a = np.array(getattr(m, attr))
            a[i] = v
            setattr(m, attr, a)
        return f

    def first_source(m):                                # a second user of the source of the first mapped entry
        k = np.nonzero(m.a_src >= 0)[0]
        m.a_src = m.a_src.copy()
        m.a_src[k[1]] = m.a_src[k[0]]

    def b_twice(m):
        k = np.nonzero(m.b_src >= 0)[0]
        m.b_src = m.b_src.copy()
        m.b_src[k[1]] = m.b_src[k[0]]

    return {
        "a_src_too_large": at("a_src", 0, 10 ** 6),
        "a_src_below_minus_two": at("a_src", 0, -3),
        "a_source_used_twice": first_source,
        "a_source_dropped": lambda m: setattr(m, "a_src", np.where(m.a_src == 0, -1, m.a_src)),
        "b_src_too_large": at("b_src", 0, 10 ** 6),
        "b_source_used_twice": b_twice,
        "b_row_neither_used_nor_uncovered": lambda m: setattr(m, "b_src", np.where(m.b_src == m.b_src.max(), -1, m.b_src)),
        "b_row_used_and_uncovered": lambda m: setattr(m, "b_uncovered", np.ones_like(m.b_uncovered)),
        "b_src_wrong_size": lambda m: setattr(m, "b_src", m.b_src[:-1]),
        "b_uncovered_wrong_size": lambda m: setattr(m, "b_uncovered", m.b_uncovered[:-1]),
        "n_orig_above_n": lambda m: setattr(m, "n_orig", m.n + 1),
        "nnzA_orig_too_small": lambda m: setattr(m, "nnzA_orig", m.nnzA_orig - 1),
    }


@pytest.mark.parametrize("what", sorted(_mutations()))
def test_validator_rejects_malformed_maps(what):
    f, _ = _mixed_map()
    chordal.validate_forward_arrays(f)
    bad = copy.deepcopy(f)
    _mutations()[what](bad)
    with pytest.raises(ValueError):
        chordal.validate_forward_arrays(bad)


def test_b_outside_every_clique_is_flagged():
    f, b = _mixed_map()
    assert f.b_uncovered.sum() > 0 and not f.b_uncovered[:4].any() and not f.b_uncovered[-6:].any()   # plain rows are covered
    assert not len(chordal.uncovered_rows(f, b))
    r = int(np.nonzero(f.b_uncovered)[0][0])
    b2 = b.copy()
    b2[r] = 1e-300
    assert chordal.uncovered_rows(f, b2).tolist() == [r]
    b2[r] = np.nan
    assert chordal.uncovered_rows(f, b2).tolist() == [r]


class _ForwardEngine(OracleEngine):
    """the oracle stand-in with the two entry points of the forward map, replayed with chordal.forward_values"""
    log = []

    def set_forward_map(self, f):
        chordal.validate_forward_arrays(f)
        assert (f.n, f.m, len(f.a_src)) == (self.n, self.m, self.A.nnz) and self.A.has_sorted_indices
        self.fwd = f

    def update_matrices_original(self, Px=None, Ax=None, q=None, b=None):
        assert not len(chordal.uncovered_rows(self.fwd, b))
        Ax2, q2, b2 = chordal.forward_values(self.fwd, Ax, q, b)
        self.A = sp.csc_matrix((Ax2, self.A.indices, self.A.indptr), shape=self.A.shape)
        self.P = sp.csc_matrix((np.asarray(Px, dtype=float), self.P.indices, self.P.indptr), shape=self.P.shape)
        self.q, self.b = q2, b2
        _ForwardEngine.log.append("update_matrices_original")

    def update_qb(self, q=None, b=None):
        super().update_qb(q, b)
        _ForwardEngine.log.append("update_qb")


@pytest.fixture
def forward_engine(monkeypatch):
    _ForwardEngine.log = []
    monkeypatch.setattr(M._eng, "Engine", _ForwardEngine)
    return _ForwardEngine


def _model(P, q, A, b, sets):
    model = cosmo_b200.Model()
    model.set(P, q, A, b, sets, cosmo_b200.Settings(scaling=0, eps_abs=1e-7, eps_rel=1e-7, decompose=True, merge_strategy="NoMerge"))
    return model


def test_model_update_keeps_the_engine_while_the_decomposition_holds(forward_engine):
    P, q, A, b, sets = _mixed()
    model = _model(P, q, A, b, sets)
    assert model.optimize().status == "Solved"
    eng = model.engine
    assert model._fwd is eng.fwd and model._x2 is not None
    x2 = model._x2.copy()
    # new values of P and A (and q, b) on the pattern: the engine and the clique iterates stay
    A2 = A * 1.25                                       # A and b scaled alike: the feasible set stays
    q2, b2 = q * 1.1, b * 1.25
    model.update(q=q2, b=b2, P=P * 1.5, A=A2)
    assert model.engine is eng and forward_engine.log == ["update_matrices_original"]
    assert np.array_equal(model._x2, x2)
    P_, q_, A_, b_, _, _ = chordal.decompose(P * 1.5, q2, A2, b2, sets, merge="none")
    assert np.array_equal(_bits(eng.A.data), _bits(A_.data)) and np.array_equal(_bits(eng.b), _bits(b_))
    assert np.array_equal(_bits(eng.q), _bits(q_)) and np.array_equal(_bits(M._sorted_csc(eng.P).data), _bits(M._sorted_csc(P_).data))
    res = model.optimize()
    assert res.status == "Solved" and np.array_equal(eng._warm[0], x2)                # warm-started in clique coordinates
    fresh = _model(P * 1.5, q2, A2, b2, sets).optimize()
    assert abs(res.obj_val - fresh.obj_val) < 1e-5 and np.allclose(res.x, fresh.x, atol=1e-4)
    # q and b alone are mapped on the host and go through update_qb
    b3 = b2.copy()
    b3[:4] += 0.5
    model.update(b=b3)
    assert model.engine is eng and forward_engine.log[-1] == "update_qb" and model._x2 is not None
    assert np.array_equal(_bits(eng.b), _bits(chordal.decompose(P * 1.5, q2, A2, b3, sets, merge="none")[3]))
    assert model.optimize().status == "Solved"
    # a b that is nonzero where no clique reaches changes the pattern: rebuild at the next optimize!
    b4 = b3.copy()
    b4[int(np.nonzero(model._fwd.b_uncovered)[0][0])] = 0.25
    n_eng = len(OracleEngine.instances)
    model.update(b=b4)
    assert model.engine is None and model._x2 is None and model._fwd is None
    model.optimize()
    assert len(OracleEngine.instances) == n_eng + 1
    assert model.engine is not eng and model._fwd is not None
    # ... and so it does through update(P=, A=)
    b5 = b4.copy()
    b5[int(np.nonzero(model._fwd.b_uncovered)[0][0])] = 0.25
    model.update(b=b5, A=A2)
    assert model.engine is None and model._x2 is None


def test_engine_without_the_forward_map_is_rebuilt(monkeypatch):
    monkeypatch.setattr(M._eng, "Engine", OracleEngine)         # the plain stand-in cannot take a forward map
    P, q, A, b, sets = _mixed()
    model = _model(P, q, A, b, sets)
    model.optimize()
    assert model._fwd is None
    model.update(b=b * 1.0)
    assert model.engine is None and model._x2 is None


_PROBE = r"""
#include <stddef.h>
#include <stdio.h>
#include "cosmo_b200.h"
#define OFF(f) printf(#f " %zu\n", offsetof(cosmo_b200_forward_map, f))
int main(void) {
  printf("sizeof %zu\n", sizeof(cosmo_b200_forward_map));
  OFF(n_orig); OFF(m_orig); OFF(n); OFF(m); OFF(nnzA_orig); OFF(nnzA); OFF(a_src); OFF(b_src); OFF(b_uncovered);
  printf("abi %d %d\n", COSMO_B200_ABI_VERSION, cosmo_b200_abi_version());
  /* both entry points refuse a null handle before they read anything */
  printf("null_handle %d %d\n", cosmo_b200_set_forward_map(NULL, NULL),
         cosmo_b200_update_matrices_original(NULL, NULL, 0, NULL, 0, NULL, NULL));
  return 0;
}
"""


def test_c_layout_of_the_forward_map_matches_the_binding(tmp_path):
    import ctypes
    import os
    import shutil
    import subprocess
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib = E.load_library()
    assert {"cosmo_b200_set_forward_map", "cosmo_b200_update_matrices_original"} <= set(E.EXPORTS)
    assert lib.cosmo_b200_abi_version() == 4                     # additive: new symbols and one new struct
    src, exe = tmp_path / "forward_map_probe.c", str(tmp_path / "forward_map_probe")
    src.write_text(_PROBE)
    subprocess.run([cc, "-std=c99", "-Wall", "-Werror", "-I", os.path.join(root, "include"), str(src), lib._name,
                    "-Wl,-rpath," + os.path.dirname(lib._name), "-o", exe], check=True)
    vals = dict(line.split(" ", 1) for line in subprocess.run([exe], check=True, capture_output=True, text=True).stdout.splitlines())
    assert int(vals.pop("sizeof")) == ctypes.sizeof(E.ForwardMapStruct)
    assert vals.pop("abi") == "4 4" and vals.pop("null_handle") == "%d %d" % (E.ERR_INVALID, E.ERR_INVALID)
    assert sorted(vals) == sorted(n for n, _ in E.ForwardMapStruct._fields_)
    for name, off in vals.items():
        assert getattr(E.ForwardMapStruct, name).offset == int(off), name
