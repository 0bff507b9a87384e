"""Custom cones without a device: NVRTC compilation and the process-wide cache (cosmo_b200_custom_cone_compile), the
checks of a descriptor, the C layout of cosmo_b200_custom_cone, the model layer (sort order, marshalling, host Ruiz,
sharding, decomposition) and the reference's custom_cone.jl problems on the oracle."""
import ctypes
import os
import shutil
import subprocess
import uuid

import numpy as np
import pytest
import scipy.sparse as sp

import cosmo_b200
from cosmo_b200 import engine as E, model as M, sharding
from oracle import cosmo_oracle as O
from tests import custom_cones as CC

TYPES = [CC.nonpos_type, CC.soc2_type, CC.linf_type]


def _fresh(kind):
    """the same type with a source no other test compiled: a cache key of its own"""
    return M.CustomConeType(kind.name, kind.source + "\n// %s\n" % uuid.uuid4().hex, kind.granularity, kind.n_params,
                            kind.in_dual, kind.in_pol_recc)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("make", TYPES, ids=lambda f: f.__name__)
def test_every_test_cone_compiles_and_the_second_call_is_a_cache_hit(make, dtype):
    kind = _fresh(make())
    assert kind.compile(dtype) is True
    assert kind.compile(dtype) is False
    # an equal descriptor in other memory is the same type
    twin = M.CustomConeType(kind.name, str(kind.source), kind.granularity, kind.n_params, kind.in_dual, kind.in_pol_recc)
    assert twin.compile(dtype) is False


def test_compile_error_carries_the_nvrtc_log_with_the_users_line():
    src = "namespace broken {\ntemplate <typename T> __device__ void project(T* x, long long dim, const T* p, int lane, int width) {\n" \
          "  x[0] = ;\n}\n}\n"
    with pytest.raises(E.EngineError) as ei:
        M.CustomConeType("broken", src + "// %s\n" % uuid.uuid4().hex).compile()
    assert ei.value.code == E.ERR_INVALID
    assert "broken(3)" in str(ei.value) and "error" in str(ei.value)


@pytest.mark.parametrize("field,value", [("name", b"1abc"), ("name", b"a-b"), ("name", b""), ("name", b"cosmo_cone"),
                                         ("granularity", 3), ("granularity", -1), ("flags", 4), ("reserved", 1),
                                         ("n_params", -1)])
def test_bad_descriptors_are_refused(field, value):
    st = CC.soc2_type().struct()
    setattr(st, field, value)
    with pytest.raises(E.EngineError) as ei:
        E.custom_cone_compile(st)
    assert ei.value.code == E.ERR_INVALID


def test_missing_source_and_unknown_dtype_are_refused():
    lib = E.load_library()
    st = CC.soc2_type().struct()
    assert lib.cosmo_b200_custom_cone_compile(ctypes.byref(st), 7, None, 0) == E.ERR_INVALID
    st.source = None
    assert lib.cosmo_b200_custom_cone_compile(ctypes.byref(st), E.F64, None, 0) == E.ERR_INVALID
    assert lib.cosmo_b200_custom_cone_compile(None, E.F64, None, 0) == E.ERR_INVALID
    assert lib.cosmo_b200_custom_cone_stats(None, (ctypes.c_int64 * 4)()) == E.ERR_INVALID


_PROBE = r"""
#include <stddef.h>
#include <stdio.h>
#include "cosmo_b200.h"
#define OFF(f) printf(#f " %zu\n", offsetof(cosmo_b200_custom_cone, f))
int main(void) {
  printf("sizeof %zu\n", sizeof(cosmo_b200_custom_cone));
  OFF(name); OFF(source); OFF(granularity); OFF(n_params); OFF(flags); OFF(reserved);
  printf("abi %d %d\n", COSMO_B200_ABI_VERSION, cosmo_b200_abi_version());
  printf("set %zu\n", sizeof(cosmo_b200_set));
  printf("consts %d %d %d %d %d %d\n", COSMO_B200_CUSTOM, COSMO_B200_CUSTOM_THREAD, COSMO_B200_CUSTOM_WARP,
         COSMO_B200_CUSTOM_BLOCK, COSMO_B200_CUSTOM_HAS_IN_DUAL, COSMO_B200_CUSTOM_HAS_IN_POL_RECC);
  return 0;
}
"""


def test_c_layout_of_the_custom_cone_matches_the_binding(tmp_path):
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib = E.load_library()
    assert {"cosmo_b200_custom_cone_compile", "cosmo_b200_custom_cone_stats"} <= set(E.EXPORTS)
    src, exe = tmp_path / "custom_cone_probe.c", str(tmp_path / "custom_cone_probe")
    src.write_text(_PROBE)
    subprocess.run([cc, "-std=c99", "-Wall", "-Werror", "-I", os.path.join(root, "include"), str(src), lib._name,
                    "-Wl,-rpath," + os.path.dirname(lib._name), "-o", exe], check=True)
    vals = dict(line.split(" ", 1) for line in subprocess.run([exe], check=True, capture_output=True, text=True).stdout.splitlines())
    assert int(vals.pop("sizeof")) == ctypes.sizeof(E.CustomConeStruct)
    assert vals.pop("abi") == "4 4"                                 # additive: new symbols and one new struct
    assert int(vals.pop("set")) == ctypes.sizeof(E.SetStruct) == 48
    assert vals.pop("consts") == "%d %d %d %d %d %d" % (E.CUSTOM, E.CUSTOM_THREAD, E.CUSTOM_WARP, E.CUSTOM_BLOCK,
                                                        E.CUSTOM_HAS_IN_DUAL, E.CUSTOM_HAS_IN_POL_RECC)
    assert sorted(vals) == sorted(n for n, _ in E.CustomConeStruct._fields_)
    for name, off in vals.items():
        assert getattr(E.CustomConeStruct, name).offset == int(off), name


# ---- model layer ----------------------------------------------------------------
def test_custom_cones_sort_into_class_6_and_validate_their_parameters():
    kind = CC.linf_type()
    assert M._sort_sets(M.CustomCone(kind, 4, [2.0])) == 6
    with pytest.raises(ValueError):
        M.CustomCone(kind, 4)                       # n_params = 1
    with pytest.raises(ValueError):
        M.CustomConeType("x", "", granularity="grid")
    P, q, A, b, sets = CC.lp_problem(CC.nonpos_type())
    assert [type(S) for S in sets] == [M.ZeroSet, M.CustomCone]


class _Refuse(Exception):
    pass


def test_marshalling_of_custom_sets(monkeypatch):
    """u = the type's cosmo_b200_custom_cone, l = the parameters in the model's dtype, alpha = tol = max_iter = 0"""
    seen = {}
    real = E.load_library()

    class Lib:
        def __getattr__(self, name):
            return getattr(real, name)

        def cosmo_b200_create(self, h, prob, st):
            pr = prob._obj
            sets = ctypes.cast(pr.sets, ctypes.POINTER(E.SetStruct))
            for i in range(pr.n_sets):
                s = sets[i]
                rec = {"type": s.type, "dim": s.dim, "alpha": s.alpha, "tol": s.tol, "max_iter": s.max_iter}
                if s.type == E.CUSTOM:
                    cs = ctypes.cast(s.u, ctypes.POINTER(E.CustomConeStruct)).contents
                    rec.update(name=cs.name.decode(), source=cs.source.decode(), gran=cs.granularity, np=cs.n_params,
                               flags=cs.flags, reserved=cs.reserved)
                    rec["l"] = None if not s.l else np.ctypeslib.as_array(
                        ctypes.cast(s.l, ctypes.POINTER(ctypes.c_double if pr.dtype == E.F64 else ctypes.c_float)),
                        (cs.n_params,)).copy()
                seen.setdefault(pr.dtype, []).append(rec)
            raise _Refuse()

    monkeypatch.setattr(E, "_lib", Lib())
    soc2, linf = CC.soc2_type(), CC.linf_type()
    sets = [M.Nonnegatives(2), M.CustomCone(soc2, 3), M.CustomCone(linf, 4, [2.5])]
    m = sum(S.dim for S in sets)
    for dt in (np.float64, np.float32):
        with pytest.raises(_Refuse):
            E.Engine(sp.identity(1, format="csc"), np.zeros(1), sp.csc_matrix((m, 1)), np.zeros(m),
                     [M.set_tuple(S) for S in sets], E.default_settings(), dtype=dt)
    for dt, rec in seen.items():
        assert rec[0]["type"] == E.NONNEG
        r1, r2 = rec[1], rec[2]
        assert (r1["type"], r1["dim"], r1["name"], r1["gran"], r1["np"], r1["flags"], r1["l"]) == \
            (E.CUSTOM, 3, "soc2", E.CUSTOM_WARP, 0, E.CUSTOM_HAS_IN_DUAL | E.CUSTOM_HAS_IN_POL_RECC, None)
        assert r1["source"] == soc2.source and r1["reserved"] == 0
        assert (r2["type"], r2["dim"], r2["name"], r2["gran"], r2["np"], r2["flags"]) == (E.CUSTOM, 4, "wlinf", E.CUSTOM_BLOCK, 1, 0)
        assert r2["l"].tolist() == [2.5]
        for r in (r1, r2):
            assert r["alpha"] == r["tol"] == r["max_iter"] == 0
    assert set(seen) == {E.F64, E.F32}


def test_host_ruiz_gives_each_custom_cone_one_scaling():
    rng = np.random.default_rng(3)
    sets = [M.Nonnegatives(3), M.CustomCone(CC.soc2_type(), 4), M.CustomCone(CC.linf_type(), 5, [3.0])]
    m, n = 12, 6
    A = sp.random(m, n, density=0.6, random_state=4, format="csc") * 10.0 + sp.eye(m, n, format="csc")
    P = sp.eye(n, format="csc")
    q, b = rng.standard_normal(n), rng.standard_normal(m)
    _, _, _, _, _, D, Ecol, c = M.ruiz_equilibrate(P, q, A, b, sets, M.Settings())
    assert np.ptp(Ecol[3:7]) <= 1e-15 and np.ptp(Ecol[7:12]) <= 1e-15
    assert np.ptp(Ecol[0:3]) > 1e-3                 # the Nonnegatives rows keep their own scalings
    # exactly the rectification of a built-in cone on the same rows
    soc = [M.Nonnegatives(3), M.SecondOrderCone(4), M.SecondOrderCone(5)]
    _, _, _, _, _, D2, E2, c2 = M.ruiz_equilibrate(P, q, A, b, soc, M.Settings())
    assert np.array_equal(D, D2) and np.array_equal(Ecol, E2) and c == c2


def test_sharding_never_splits_a_custom_cone():
    kind = CC.soc2_type()
    sets = [M.Nonnegatives(5)] + [M.CustomCone(kind, d) for d in (7, 40, 3, 9)] + [M.ZeroSet(6)]
    m = sum(S.dim for S in sets)
    A = sp.random(m, 8, density=0.5, random_state=1, format="csc")
    for world in (2, 3, 4):
        parts = sharding.partition_rows(A, sets, world)
        for k, S in enumerate(sets):
            pieces = [(a, b) for part in parts for (kk, a, b) in part if kk == k]
            if isinstance(S, M.CustomCone):
                assert pieces == [(0, S.dim)], (world, k, pieces)
            assert sum(b - a for a, b in pieces) == S.dim


def test_decompose_passes_custom_cones_through_as_plain_blocks():
    from cosmo_b200 import chordal
    from tests import golden_problems as G
    kind = CC.soc2_type()
    # an arrow-pattern PSD constraint that the decomposition splits, followed by a custom cone
    N = 8
    rng = np.random.default_rng(5)
    rows, cols, vals = [], [], []
    tri = [(i, j) for j in range(N) for i in range(j + 1)]
    for r, (i, j) in enumerate(tri):
        if i == j or i == 0:
            rows.append(r); cols.append(r % 3); vals.append(rng.standard_normal())
    d = len(tri)
    A = sp.vstack([sp.csc_matrix((vals, (rows, cols)), shape=(d, 3)), sp.csc_matrix(rng.standard_normal((4, 3)))], format="csc")
    b = np.concatenate([np.where([i == j for i, j in tri], 1.0, 0.0), rng.standard_normal(4)])
    sets = [M.PsdConeTriangle(d), M.CustomCone(kind, 4)]
    P2, q2, A2, b2, sets2, info = chordal.decompose(sp.eye(3, format="csc"), np.ones(3), A, b, sets)
    assert info.blocks
    custom = [S for S in sets2 if isinstance(S, M.CustomCone)]
    assert len(custom) == 1 and custom[0] is sets[1]
    # the custom rows are the last rows of A2, unchanged
    assert np.array_equal(A2[-4:, :3].toarray(), A[-4:, :].toarray()) and np.array_equal(b2[-4:], b[-4:])


# ---- the reference's custom_cone.jl on the oracle -----------------------------------
@pytest.fixture
def oracle(monkeypatch):
    CC.install_oracle(monkeypatch)
    return O


def test_oracle_solves_the_nonpositives_lp(oracle):
    P, q, A, b, sets = CC.lp_problem(CC.nonpos_type())
    r = oracle.solve(P, q, A, b, CC.to_oracle(sets), oracle.Settings(kkt_solver="cg"))
    assert r.status == "Solved"
    assert abs(r.obj_val + 7.0) <= 1e-3


@pytest.mark.parametrize("hooks", [True, False])
def test_oracle_infeasibility_follows_the_hooks(oracle, hooks):
    kind = CC.nonpos_type(hooks)
    st = oracle.Settings(kkt_solver="cg", max_iter=2000)
    P, q, A, b, sets = CC.dual_infeasible_problem(kind)
    assert oracle.solve(P, q, A, b, CC.to_oracle(sets), st).status == ("Dual_infeasible" if hooks else "Max_iter_reached")
    P, q, A, b, sets = CC.primal_infeasible_problem(kind)
    assert oracle.solve(P, q, A, b, CC.to_oracle(sets), st).status == ("Primal_infeasible" if hooks else "Max_iter_reached")


def test_oracle_numpy_cones_match_their_definitions(oracle):
    rng = np.random.default_rng(7)
    v = rng.standard_normal(9) * 3
    x = v.copy()
    CC._linf_project(x, [2.0])
    # the projection is in the cone and v - x is in the polar (x is the nearest point): <v - x, x> = 0
    assert 2.0 * np.abs(x[1:]).max() <= x[0] * (1 + 1e-12)
    assert abs(np.dot(v - x, x)) <= 1e-10 * np.dot(v, v)
    y = v.copy()
    CC._soc_project(y, ())
    z = v.copy()
    O.project_cone(z, O.SecondOrderCone(9))
    assert np.array_equal(y, z)
