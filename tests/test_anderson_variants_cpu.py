"""The Anderson accelerator variants without a GPU: the CPU restatement of tests/anderson_variants.py against the
reference's acceleration tests and the algebra it states, the host settings and C ABI of cosmo_b200_set_accelerator,
and a dry run of tests/test_gpu_accelerators.py against the oracle stand-in."""
import inspect
import os
import shutil
import subprocess

import numpy as np
import pytest

import cosmo_b200
from cosmo_b200 import engine as E, model as M
from oracle import cosmo_oracle as O
from tests import anderson_variants as V
from tests import golden_problems as G
from tests.oracle_engine import OracleEngine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _g1():
    P, q, cons = G.g1_qp_nonneg()
    return O.assemble(P, q, cons)


@pytest.mark.parametrize("t,mem,reg", V.TYPES)
def test_every_variant_solves_the_reference_qp(t, mem, reg):
    # AccelerationTests/anderson_accelerator.jl:21-41: all 13 types reach :Solved on the literal QP
    res, ws = V.solve(*_g1(), O.Settings(accelerator="anderson"), **V.variant(t, mem, reg))
    assert res.status == "Solved" and abs(res.obj_val - G.G1_OBJ) < 1e-3 and np.max(np.abs(res.x - G.G1_X)) < 1e-3
    assert V.stats(ws)["accepted"] >= 1


@pytest.mark.parametrize("mem", ["RollingMemory", "RestartedMemory"])
def test_rho_adaptation_restarts_the_accelerator(mem):
    # AccelerationTests/adaptive_rho_acc_restarts.jl: Type2{NormalEquations}, mem 5, rho 1e-4, interval 23, no safeguard.
    # With RollingMemory every candidate of this restatement is accepted, so the adaptation keeps being postponed to a
    # non-accelerated iteration (solver.jl:284-292) and none happens: the reference's equality holds with 0 = 0.
    # RestartedMemory leaves non-accelerated iterations after each restart and adapts.
    res, ws = V.solve(*_g1(), O.Settings(accelerator="anderson", adaptive_rho_interval=23, rho=1e-4, safeguard=False,
                                         accelerator_mem=5), **V.variant("Type2{NormalEquations}", mem, "NoRegularizer"))
    assert V.stats(ws)["rho_restarts"] == len(ws.rho_updates) - 1
    if mem == "RestartedMemory":
        assert len(ws.rho_updates) - 1 >= 1 and res.status == "Solved"


def _history(aa, steps, seed=0, dim=40):
    """feed `steps` iterations of an affine contraction x <- K x + c; returns the accelerator after each update"""
    rng = np.random.default_rng(seed)
    K = rng.standard_normal((dim, dim)) * 0.2 / np.sqrt(dim)
    c = rng.standard_normal(dim)
    x = rng.standard_normal(dim)
    for k in range(steps):
        g = K @ x + c
        aa.update(g, x, k + 2)
        yield g
        x = g


@pytest.mark.parametrize("type1", [False, True])
@pytest.mark.parametrize("rolling", [False, True])
def test_gram_matrix_matches_the_window(type1, rolling):
    aa = V.NormalEquationsAccelerator(40, mem=6, min_mem=3, type1=type1, rolling=rolling)
    for k, g in enumerate(_history(aa, 20)):
        aa.accelerate(g.copy(), None, k + 2)
        l = min(aa.iter, aa.mem)
        A = aa.X if type1 else aa.F
        assert np.allclose(aa.M[:l, :l], A[:, :l].T @ aa.F[:, :l], rtol=1e-12, atol=1e-14), k
        if type1:   # G = X - F, stored as its own difference
            assert np.allclose(aa.G[:, :l], aa.X[:, :l] - aa.F[:, :l], atol=1e-12)


def test_type2_eta_is_the_least_squares_solution():
    aa = V.NormalEquationsAccelerator(40, mem=6)
    for k, g in enumerate(_history(aa, 6, seed=1)):
        g_acc = g.copy()
        aa.accelerate(g_acc, None, k + 2)
    l = min(aa.iter, aa.mem)
    eta = np.linalg.lstsq(aa.F[:, :l], aa.f, rcond=None)[0]
    kappa = np.linalg.cond(aa.F[:, :l])
    assert aa.success and np.linalg.norm(aa.eta[:l] - eta) <= 1e-13 * kappa ** 2 * (1 + np.linalg.norm(eta))
    assert np.allclose(g_acc, g - aa.G[:, :l] @ aa.eta[:l], atol=1e-12)


def test_type1_eta_solves_its_system():
    aa = V.NormalEquationsAccelerator(40, mem=6, type1=True)
    for k, g in enumerate(_history(aa, 6, seed=2)):
        aa.accelerate(g.copy(), None, k + 2)
    l = min(aa.iter, aa.mem)
    X, F = aa.X[:, :l], aa.F[:, :l]
    assert aa.success
    assert np.linalg.norm(X.T @ F @ aa.eta[:l] - X.T @ aa.f) <= 1e-10 * np.linalg.norm(X.T @ aa.f)


@pytest.mark.parametrize("type1", [False, True])
def test_regularised_system_has_the_stated_shift(type1):
    for reg in ("TikonovRegularizer", "FrobeniusNormRegularizer"):
        aa = V.NormalEquationsAccelerator(40, mem=5, type1=type1, regularizer=reg, lam=1e-3)
        for k, g in enumerate(_history(aa, 5, seed=3)):
            aa.accelerate(g.copy(), None, k + 2)
        l = min(aa.iter, aa.mem)
        A = aa.X[:, :l] if type1 else aa.F[:, :l]
        B = aa.F[:, :l]
        shift = 1e-3 if reg == "TikonovRegularizer" else 1e-3 * (np.sum(A * A) + np.sum(B * B))
        assert np.allclose(aa.system(l), A.T @ B + shift * np.eye(l), rtol=1e-12), reg


def test_lu_solve_rejections():
    assert V.lu_solve(np.zeros((3, 3)), np.ones(3)) is None                       # singular
    assert V.lu_solve(np.diag([1.0, np.nan, 1.0]), np.ones(3)) is None            # not finite
    assert V.lu_solve(np.diag([1e-5, 1.0]), np.ones(2)) is None                   # |eta| > 1e4
    M = np.array([[1e-3, 2.0], [3.0, 4.0]])
    assert np.allclose(V.lu_solve(M, np.array([1.0, 2.0])), np.linalg.solve(M, [1.0, 2.0]), rtol=1e-14)


def _candidates_per_iteration(var, **kw):
    counts = []
    ws = V.Workspace(*_g1(), O.Settings(accelerator="anderson", **kw), **var)
    res = ws.optimize(iter_callback=lambda it, w: counts.append((it, w.accelerator.num_accelerated_steps)))
    return res, ws, counts


@pytest.mark.parametrize("t", ["Type2{QRDecomp}", "Type1"])
def test_iter_activation_forms_no_candidate_before_k(t):
    k = 12
    var = V.variant(t, "RestartedMemory", "NoRegularizer", activation=("IterActivation", k))
    res, ws, counts = _candidates_per_iteration(var)
    assert V.stats(ws)["activated_at"] == k
    assert all(c == 0 for it, c in counts if it < k) and counts[-1][1] > 0 and res.status == "Solved"


@pytest.mark.parametrize("t", ["Type2{QRDecomp}", "Type2{NormalEquations}"])
def test_accuracy_activation_at_the_first_check_that_meets_it(t):
    tol = 1e-3
    # the plain run's termination checks: until activation the accelerated run follows it exactly
    checks = []
    ws0 = V.Workspace(*_g1(), O.Settings(accelerator="anderson", check_termination=5),
                      **V.variant(t, "RestartedMemory", "NoRegularizer", activation=("AccuracyActivation", 0.0)))
    conv = ws0.has_converged
    ws0.has_converged = lambda r: checks.append((ws0.accelerator.last_iter, r.r_prim < tol + tol * r.max_norm_prim and
                                                 r.r_dual < tol + tol * r.max_norm_dual)) or conv(r)
    ws0.optimize()
    first = next(it for it, ok in checks if ok)
    assert first > 1
    var = V.variant(t, "RestartedMemory", "NoRegularizer", activation=("AccuracyActivation", tol))
    res, ws, counts = _candidates_per_iteration(var, check_termination=5)
    assert V.stats(ws)["activated_at"] == first
    assert all(c == 0 for it, c in counts if it <= first) and res.status == "Solved"


# ---------------------------------------------------------------------------
# host settings and the C ABI
# ---------------------------------------------------------------------------
def test_settings_mapping_and_validation():
    assert cosmo_b200.Settings(accelerator="AndersonAccelerator").accelerator_struct() is None     # the default variant
    a = cosmo_b200.Settings(accelerator="AndersonAccelerator", accelerator_type="Type1", accelerator_memory="RollingMemory",
                            accelerator_regularizer="FrobeniusNormRegularizer", accelerator_lambda=1e-6,
                            accelerator_activation=("IterActivation", 7)).accelerator_struct()
    assert (a.type, a.memory, a.regularizer, a.lambda_, a.activation, a.start_iter) == \
        (E.AA_TYPE1, E.AA_ROLLING_MEMORY, E.AA_FROBENIUS, 1e-6, E.AA_ITER, 7)
    a = cosmo_b200.Settings(accelerator_activation=("AccuracyActivation", 1e-3)).accelerator_struct()
    assert (a.type, a.activation, a.start_accuracy) == (E.AA_TYPE2_QR, E.AA_ACCURACY, 1e-3)
    for t, mem, reg in V.TYPES:
        cosmo_b200.Settings(accelerator="AndersonAccelerator", **V.variant(t, mem, reg)).to_struct()
    for bad in (dict(accelerator_memory="RollingMemory"), dict(accelerator_regularizer="TikonovRegularizer"),
                dict(accelerator_type="Type3"), dict(accelerator_activation=("IterActivation",))):
        with pytest.raises(E.EngineError) as e:
            cosmo_b200.Settings(accelerator="AndersonAccelerator", **bad).to_struct()
        assert e.value.code == E.ERR_UNSUPPORTED
    with pytest.raises(E.EngineError) as e:
        cosmo_b200.Settings(accelerator="AndersonAccelerator", accelerator_type="Type1", accelerator_lambda=-1.0).to_struct()
    assert e.value.code == E.ERR_INVALID
    with pytest.raises(E.EngineError):
        cosmo_b200.Settings(accelerator="AndersonAccelerator{Type1}").to_struct()


def test_new_entry_points_are_exported():
    lib = E.load_library()
    for name in ("cosmo_b200_set_accelerator", "cosmo_b200_accelerator_stats"):
        assert name in E.EXPORTS and hasattr(lib, name)
    # no handle: refused with an error code
    assert lib.cosmo_b200_set_accelerator(None, None) == E.ERR_INVALID
    assert lib.cosmo_b200_accelerator_stats(None, (E.C.c_int64 * 6)()) == E.ERR_INVALID


def test_c_header_layout_of_the_accelerator_struct(tmp_path):
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "probe.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "cosmo_b200.h"\n'
                   '#define F(f) printf(#f " %zu\\n", offsetof(cosmo_b200_accelerator, f))\n'
                   'int main(void) { printf("sizeof %zu\\n", sizeof(cosmo_b200_accelerator)); F(type); F(memory);'
                   ' F(regularizer); F(activation); F(lambda); F(start_iter); F(start_accuracy);'
                   ' printf("null %d\\n", cosmo_b200_set_accelerator(NULL, NULL)); return 0; }\n')
    lib_path = E.load_library()._name
    exe = str(tmp_path / "probe")
    subprocess.run([cc, "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), lib_path,
                    "-Wl,-rpath," + os.path.dirname(lib_path), "-o", exe], check=True)
    out = dict(line.split() for line in subprocess.run([exe], check=True, capture_output=True, text=True).stdout.splitlines())
    S = E.AcceleratorStruct
    assert int(out["sizeof"]) == E.C.sizeof(S)
    for f in ("type", "memory", "regularizer", "activation", "start_iter", "start_accuracy"):
        assert int(out[f]) == getattr(S, f).offset, f
    assert int(out["lambda"]) == S.lambda_.offset
    assert int(out["null"]) == E.ERR_INVALID


# ---------------------------------------------------------------------------
# dry run of the GPU module against the oracle stand-in
# ---------------------------------------------------------------------------
_NAMES = {v: k for k, v in M.Settings._AA_TYPE.items()}, {v: k for k, v in M.Settings._AA_MEMORY.items()}, \
         {v: k for k, v in M.Settings._AA_REG.items()}


class VariantOracleEngine(OracleEngine):
    """the oracle stand-in with cosmo_b200_set_accelerator / cosmo_b200_accelerator_stats"""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.acc, self._stats = None, {k: 0 for k in E.ACCELERATOR_STATS}

    def set_accelerator(self, acc):
        self.acc = acc

    def accelerator_stats(self):
        return self._stats

    def solve(self):
        st, a = self.st, self.acc
        var = {}
        if a is not None:
            act = {E.AA_IMMEDIATE: "ImmediateActivation", E.AA_ITER: ("IterActivation", a.start_iter),
                   E.AA_ACCURACY: ("AccuracyActivation", a.start_accuracy)}[a.activation]
            var = V.variant(_NAMES[0][a.type], _NAMES[1][a.memory], _NAMES[2][a.regularizer], act, a.lambda_)
        ost = O.Settings(scaling=0, kkt_solver="cg", eps_abs=st.eps_abs, eps_rel=st.eps_rel, max_iter=st.max_iter, rho=st.rho,
                         check_termination=st.check_termination, check_infeasibility=st.check_infeasibility,
                         adaptive_rho=bool(st.adaptive_rho), adaptive_rho_interval=st.adaptive_rho_interval,
                         accelerator="anderson" if st.accelerator == E.ACC_ANDERSON else "empty",
                         accelerator_mem=st.accelerator_mem, safeguard=bool(st.safeguard), safeguard_tol=st.safeguard_tol)
        r, ws = V.solve(self.P, self.q, self.A, self.b, self.cones, ost, **var)
        if ws.accelerator is not None:
            self._stats = V.stats(ws)
        self._w, self._rho = r.w, r.rho_vec
        out = E.SolveOutput()
        out.x, out.s, out.mu = r.x, r.s, -r.y
        out.obj_val, out.iter, out.safeguarding_iter, out.status = r.obj_val, r.iter, r.safeguarding_iter, r.status
        out.r_prim, out.r_dual, out.max_norm_prim, out.max_norm_dual = r.info.r_prim, r.info.r_dual, 0.0, 0.0
        out.rho, out.rho_updates, out.times = 0.1, list(r.info.rho_updates), {"iter_time_device": 0.0}
        out.kkt_inner_iterations = out.kkt_multiplications = out.kernel_launches = 0
        return out


_DRY_MUST_PASS = {"test_every_variant_solves_the_reference_qp", "test_rho_adaptation_restarts_the_accelerator"}
_DRY = ["test_variant_iterates_match_oracle", "test_every_variant_solves_the_reference_qp",
        "test_variant_known_answers_and_statuses", "test_rho_adaptation_restarts_the_accelerator",
        "test_activation_matches_oracle", "test_dimension_below_memory", "test_float32_statuses"]


@pytest.mark.parametrize("name", _DRY)
def test_gpu_accelerator_test_body_runs_against_the_oracle_stand_in(name, monkeypatch):
    from tests.test_gpu_tests_dryrun_cpu import _calls
    monkeypatch.setattr(M._eng, "Engine", VariantOracleEngine)
    monkeypatch.setattr(E, "Engine", VariantOracleEngine)
    import tests.test_gpu_accelerators as T
    fn = getattr(T, name)
    kwargs = _calls(fn)
    if "monkeypatch" in inspect.signature(fn).parameters:
        kwargs["monkeypatch"] = monkeypatch
    try:
        fn(**kwargs)
    except AssertionError:
        # the stand-in skips the scaling and answers in float64; the tests that depend on neither must pass
        if name in _DRY_MUST_PASS:
            raise
