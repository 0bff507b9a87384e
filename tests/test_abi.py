"""CPU-side checks of the drop-in boundary: the shared library loads and exports
every symbol include/cosmo_b200.h declares; without a GPU the product path fails
loudly (no CPU fallback)."""
import ctypes
import os
import re

import numpy as np
import pytest

import cosmo_b200
from cosmo_b200 import engine as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "cosmo_b200.h")).read()
    return sorted(set(re.findall(r"\b(cosmo_b200_[a-z_0-9]+)\s*\(", src)))


def test_header_symbols_exported():
    lib = E.load_library()
    declared = _declared_symbols()
    assert len(declared) >= 20
    for name in declared:
        assert hasattr(lib, name), name
    assert sorted(E.EXPORTS) == declared
    assert lib.cosmo_b200_abi_version() == 4


def test_default_settings_match_reference():
    s = E.default_settings()  # src/settings.jl:101-139
    assert (s.rho, s.sigma, s.alpha) == (0.1, 1e-6, 1.6)
    assert (s.eps_abs, s.eps_rel, s.eps_prim_inf, s.eps_dual_inf) == (1e-5, 1e-5, 1e-4, 1e-4)
    assert (s.max_iter, s.check_termination, s.check_infeasibility, s.scaling) == (5000, 25, 40, 10)
    assert (s.adaptive_rho, s.adaptive_rho_interval, s.adaptive_rho_tolerance) == (1, 40, 5.0)
    assert (s.RHO_MIN, s.RHO_MAX, s.RHO_TOL, s.RHO_EQ_OVER_RHO_INEQ) == (1e-6, 1e6, 1e-4, 1e3)
    assert (s.tol_constant, s.tol_exponent) == (1.0, 1.5)


def test_struct_sizes():
    # keep the ctypes mirrors in sync with the C header layout
    assert ctypes.sizeof(E.CscStruct) == 40
    assert ctypes.sizeof(E.SetStruct) == 48
    assert ctypes.sizeof(E.ProblemStruct) == 16 + 16 + 80 + 16 + 16 + 32 + 8
    assert ctypes.sizeof(E.SettingsStruct) == 56 + 8 + 24 + 16 + 48 + 24 + 8 + 24 + 24 + 16   # ABI 3: adaptive_rho_fraction, setup_time, MAX_SCALING; ABI 4: obj_true, obj_true_tol
    assert ctypes.sizeof(E.ResultStruct) == 24 + 24 + 8 + 40 + 24 + 56 + 24


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(50, 100, 0.1, seed=0)
    m = cosmo_b200.Model()
    m.set(P, q, A, b, sets, cosmo_b200.Settings())
    with pytest.raises(cosmo_b200.EngineError) as ei:
        m.optimize()
    assert ei.value.code == E.ERR_CUDA and "no CPU fallback" in str(ei.value)


def test_host_mirror_assemble_matches_reference_ordering():
    # moi_wrapper.jl:266-271 / interface.jl:411-475: merge Zero & Nonneg, stable sort by type
    from tests import golden_problems as G
    from oracle import cosmo_oracle as O
    from oracle.bridge import to_oracle_cones
    P, q, cons = G.g3_hs21()
    Pm, qm, A, b, cones = O.assemble(P, q, cons)
    mine = [cosmo_b200.Constraint(c.A, c.b, _conv(c.convex_set)) for c in cons]
    m = cosmo_b200.Model()
    m.assemble(P, q, mine, cosmo_b200.Settings())
    assert [type(s).__name__ for s in m.sets0] == [type(c).__name__ for c in cones]
    assert np.array_equal(m.A0.toarray(), A.toarray()) and np.array_equal(m.b0, b)


def _conv(c):
    from oracle import cosmo_oracle as O
    from oracle.bridge import to_oracle_cones
    if isinstance(c, O.Box):
        return cosmo_b200.Box(c.l, c.u)
    return getattr(cosmo_b200, type(c).__name__)(c.dim)


def test_ruiz_matches_oracle():
    from oracle import cosmo_oracle as O
    from oracle.bridge import to_oracle_cones
    P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(60, 90, 0.2, seed=3)
    st = cosmo_b200.Settings()
    P1, q1, A1, b1, s1, D, Em, c = cosmo_b200.ruiz_equilibrate(P, q, A, b, sets, st)
    P2, q2, A2, b2, s2, sm = O.scale_ruiz(P, q, A, b, to_oracle_cones(sets), O.Settings())
    assert np.allclose(D, sm.D, rtol=1e-13) and np.allclose(Em, sm.E, rtol=1e-13) and abs(c - sm.c) < 1e-13 * abs(c)
    assert np.allclose(A1.toarray(), A2.toarray(), rtol=1e-12, atol=1e-14)
    assert np.allclose(P1.toarray(), P2.toarray(), rtol=1e-12, atol=1e-14)
    assert np.allclose(q1, q2, rtol=1e-12) and np.allclose(b1, b2, rtol=1e-12)
    assert np.allclose(s1[1].l, s2[1].l, rtol=1e-12) and np.allclose(s1[1].u, s2[1].u, rtol=1e-12)


def test_accelerator_settings_mapping_and_validation():
    import cosmo_b200
    from cosmo_b200 import engine as E
    st = cosmo_b200.Settings().to_struct()
    assert (st.accelerator, st.accelerator_mem, st.accelerator_min_mem, st.safeguard, st.safeguard_tol) == (E.ACC_EMPTY, 15, 3, 1, 2.0)
    st = cosmo_b200.Settings(accelerator="AndersonAccelerator", accelerator_mem=7, safeguard=False, safeguard_tol=3.0).to_struct()
    assert (st.accelerator, st.accelerator_mem, st.safeguard, st.safeguard_tol) == (E.ACC_ANDERSON, 7, 0, 3.0)
    with pytest.raises(ValueError):        # AndersonAccelerator(dim; mem <= 2) throws a DomainError in the package
        cosmo_b200.Settings(accelerator="AndersonAccelerator", accelerator_mem=2).to_struct()
    with pytest.raises(E.EngineError):
        cosmo_b200.Settings(accelerator="AndersonAccelerator", accelerator_mem=64).to_struct()
    with pytest.raises(E.EngineError):     # Type-I / rolling-memory variants are not implemented
        cosmo_b200.Settings(accelerator="AndersonAccelerator{Type1}").to_struct()
    d = E.default_settings()
    assert (d.accelerator, d.accelerator_mem, d.accelerator_min_mem, d.safeguard, d.safeguard_tol) == (0, 15, 3, 1, 2.0)


def test_c_header_layout_matches_ctypes_mirror(tmp_path):
    # compile a plain C program against include/cosmo_b200.h, link it with the shared library, and compare the
    # layout the C compiler sees with the ctypes structures the Python binding marshals
    import shutil
    import subprocess
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    lib_path = E.load_library()._name
    exe = str(tmp_path / "abi_probe")
    subprocess.run([cc, "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "abi_probe.c"),
                    lib_path, "-Wl,-rpath," + os.path.dirname(lib_path), "-o", exe], check=True)
    out = subprocess.run([exe], check=True, capture_output=True, text=True).stdout
    vals = {}
    for line in out.splitlines():
        k, _, v = line.partition(" ")
        vals[k] = v
    mirror = {"cosmo_b200_csc": E.CscStruct, "cosmo_b200_set": E.SetStruct, "cosmo_b200_problem": E.ProblemStruct,
              "cosmo_b200_settings": E.SettingsStruct, "cosmo_b200_result": E.ResultStruct}
    checked = 0
    for k, v in vals.items():
        if k.startswith("sizeof."):
            assert ctypes.sizeof(mirror[k[len("sizeof."):]]) == int(v), k
            checked += 1
        elif "." in k and k.split(".")[0] in mirror:
            st, field = k.split(".")
            assert getattr(mirror[st], field).offset == int(v), k
            checked += 1
    assert checked >= 35
    assert vals["abi"] == "4" and vals["defaults"] == "0.1 1e-06 1.6 5000 0 15 2"
    assert int(vals["create_null"]) == E.ERR_INVALID and "null" in vals["last_error"]
    assert vals["infeasibility_null"] == vals["lambda_max_null"] == "%d %d" % (E.ERR_INVALID, E.ERR_INVALID)


def _build_c_example(tmp_path):
    import shutil
    import subprocess
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    lib_path = E.load_library()._name
    exe = str(tmp_path / "solve_qp")
    subprocess.run([cc, "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "solve_qp.c"),
                    lib_path, "-Wl,-rpath," + os.path.dirname(lib_path), "-lm", "-o", exe], check=True)
    return exe


def test_c_example_builds_and_fails_loudly_without_a_gpu(tmp_path):
    # examples/solve_qp.c: the reference's examples/qp.jl through the C ABI from plain C
    import subprocess
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by the gpu-marked run of the same program")
    out = subprocess.run([_build_c_example(tmp_path)], capture_output=True, text=True)
    assert out.returncode == 3 and "no CPU fallback" in out.stdout     # arguments passed validation, then: no device


@pytest.mark.gpu
def test_c_example_solves_the_reference_qp(tmp_path):
    import subprocess
    out = subprocess.run([_build_c_example(tmp_path)], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.startswith("status 1 ")                              # COSMO_B200_SOLVED; x = (0.3, 0.7), obj 1.88 checked in C


def test_obj_true_settings_mapping_and_oracle_rule():
    # ABI 4: obj_true (NaN = off) / obj_true_tol reach the engine's settings; the oracle applies the rule of
    # residuals.jl:127-140 (a wrong value keeps the loop running, a tight tolerance costs iterations)
    import math
    from oracle import cosmo_oracle as O
    from tests import golden_problems as G
    d = E.default_settings()
    assert math.isnan(d.obj_true) and d.obj_true_tol == 1e-3
    st = cosmo_b200.Settings(obj_true=1.88, obj_true_tol=1e-6).to_struct()
    assert (st.obj_true, st.obj_true_tol) == (1.88, 1e-6) and math.isnan(cosmo_b200.Settings().to_struct().obj_true)
    P, q, cons = G.g1_qp_nonneg()
    Pm, qm, A, b, cones = O.assemble(P, q, cons)
    plain = O.solve(Pm, qm, A, b, cones, O.Settings())
    tight = O.solve(Pm, qm, A, b, cones, O.Settings(obj_true=1.88, obj_true_tol=1e-8))
    wrong = O.solve(Pm, qm, A, b, cones, O.Settings(obj_true=2.88, max_iter=200))
    assert plain.status == tight.status == "Solved" and tight.iter > plain.iter and abs(tight.obj_val - 1.88) <= 1e-8
    assert wrong.status == "Max_iter_reached" and wrong.iter == 200
