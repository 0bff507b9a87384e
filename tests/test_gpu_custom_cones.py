"""Custom cones on the device: the compiled projections against the oracle and against the built-in cones they
re-implement, the certificate hooks, the scaling, the updates, a decomposed model and the compile cache.

The test cones (tests/custom_cones.py): `nonpos` (one thread per cone, the reference's Nonpositives with its literal
hooks), `soc2` (one warp per cone, the second-order cone with both hooks) and `wlinf` (one block per cone, the weighted
l-infinity cone {(t, x) : w |x|_inf <= t}, w a parameter, projected by a block-wide bisection, no hooks).

Bars: `nonpos` is one comparison per entry, so it is bit-exact.  `soc2` differs from the built-in SOC kernel only in the
order of the sum of squares (a warp tree against the chunked, power-of-two-scaled sum), so its rows agree to a few
units of roundoff of |x|; `wlinf` sums in another order than the NumPy bisection, and its threshold agrees to 1e-12
relative.  A solve with `soc2` in place of SecondOrderCone follows the same trajectory up to those roundings: the same
status and iteration count, iterates within 1e-9 relative in fp64 and 2^10 units of fp32 roundoff in fp32."""
import uuid

import numpy as np
import pytest
import scipy.sparse as sp

import cosmo_b200
from cosmo_b200 import engine as E, model as M
from oracle import cosmo_oracle as O
from tests import custom_cones as CC
from tests.gpu_helpers import U32, U64, _engine, _project_engine, _tuples

pytestmark = pytest.mark.gpu


@pytest.fixture
def oracle(monkeypatch):
    CC.install_oracle(monkeypatch)
    return O


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.max(np.abs(a - b)) / max(1.0, np.max(np.abs(b)))) if b.size else 0.0


# ---- 1. projection parity -----------------------------------------------------------
def _mixed_sets():
    nonpos, soc2, linf = CC.nonpos_type(), CC.soc2_type(), CC.linf_type()
    builtin = [M.ZeroSet(3), M.Nonnegatives(5), M.Box(-np.ones(4), np.ones(4)), M.SecondOrderCone(6),
               M.PsdConeTriangle(10), M.ExponentialCone(), M.PowerCone(0.3)]
    custom = [M.CustomCone(nonpos, 7), M.CustomCone(soc2, 1), M.CustomCone(soc2, 5), M.CustomCone(soc2, 77),
              M.CustomCone(linf, 9, [2.0]), M.CustomCone(linf, 600, [0.5]), M.CustomCone(nonpos, 1),
              M.CustomCone(soc2, 40)]
    return builtin, custom


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_projection_parity_with_builtin_cones(oracle, seed):
    builtin, custom = _mixed_sets()
    sets = builtin + custom
    rng = np.random.default_rng(seed)
    m = sum(S.dim for S in sets)
    ws = rng.standard_normal(m) * 3.0
    mb = sum(S.dim for S in builtin)
    off = mb
    for S in custom:                # seed 0: inside the cone, 1: inside the polar, 2: the general branch
        if S.kind.name == "soc2" and S.dim > 1:
            nt = np.linalg.norm(ws[off + 1:off + S.dim])
            ws[off] = [5.0 * nt, -5.0 * nt, ws[off]][seed]
        off += S.dim
    eng = _project_engine(sets)
    got = eng.project(ws)
    ref = ws.copy()
    O.project(ref, CC.to_oracle(sets))
    # built-in rows: bit-identical to an engine that has no custom cone
    eng_b = _project_engine(builtin)
    assert np.array_equal(got[:mb], eng_b.project(ws[:mb]))
    off = mb
    for S in custom:
        g, r = got[off:off + S.dim], ref[off:off + S.dim]
        if S.kind.name == "nonpos":
            assert np.array_equal(g, r)
        elif S.kind.name == "soc2":
            assert np.max(np.abs(g - r)) <= 8 * S.dim * U64 * max(np.linalg.norm(ws[off:off + S.dim]), 1e-300), S.dim
        else:
            assert _rel(g, r) <= 1e-12, S.dim
        off += S.dim
    st = eng.custom_cone_stats()
    assert st["types"] == 3 and st["cones"] == len(custom)
    eng.close(); eng_b.close()


def test_projection_float32(oracle):
    _, custom = _mixed_sets()
    rng = np.random.default_rng(4)
    m = sum(S.dim for S in custom)
    ws = rng.standard_normal(m).astype(np.float32).astype(np.float64)
    eng = _project_engine(custom, dtype=np.float32)
    got = eng.project(ws).astype(np.float64)
    ref = ws.copy()
    O.project(ref, CC.to_oracle(custom))
    off = 0
    for S in custom:
        g, r = got[off:off + S.dim], ref[off:off + S.dim]
        if S.kind.name == "nonpos":
            assert np.array_equal(g, r)
        else:
            assert np.max(np.abs(g - r)) <= 16 * S.dim * U32 * max(np.abs(ws[off:off + S.dim]).max(), 1.0), S.kind.name
        off += S.dim


# ---- 2. the same solve with soc2 in place of SecondOrderCone ------------------------------
def _socp(kind=None, seed=0):
    rng = np.random.default_rng(seed)
    n = 30
    dims = [12, 9, 33, 1]
    sets = [M.Nonnegatives(10)] + [M.SecondOrderCone(d) if kind is None else M.CustomCone(kind, d) for d in dims]
    m = sum(S.dim for S in sets)
    A = sp.random(m, n, density=0.3, random_state=seed, format="csc") + sp.eye(m, n, format="csc")
    G = sp.random(n, n, density=0.1, random_state=seed + 1, format="csc")
    P = (G @ G.T + 0.1 * sp.eye(n)).tocsc()
    x0 = rng.standard_normal(n)
    s0 = np.concatenate([np.abs(rng.standard_normal(10))] +
                        [np.concatenate([[np.linalg.norm(v) + 1.0], v]) for v in (rng.standard_normal(d - 1) for d in dims)])
    return P, rng.standard_normal(n), A, A @ x0 + s0, sets


SOLVE_CASES = {"cg": {}, "ldl": {"kkt_solver": "DeviceLdlKKTSolver"}, "anderson": {"accelerator": "AndersonAccelerator"},
               "unscaled": {"scaling": 0}}


@pytest.mark.parametrize("case", sorted(SOLVE_CASES))
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_soc2_solves_like_the_builtin_soc(case, dtype):
    res = []
    for kind in (None, CC.soc2_type()):
        P, q, A, b, sets = _socp(kind)
        model = cosmo_b200.Model(dtype=dtype)
        model.set(P, q, A, b, sets, cosmo_b200.Settings(**SOLVE_CASES[case]))
        res.append(model.optimize())
    a, c = res
    bar = 1e-9 if dtype == np.float64 else 1024 * U32
    print("MEAS soc2 %s %s: %s/%d vs %s/%d, x %.2e s %.2e y %.2e" % (case, np.dtype(dtype).name, a.status, a.iter, c.status,
          c.iter, _rel(c.x, a.x), _rel(c.s, a.s), _rel(c.y, a.y)))
    assert a.status == c.status == "Solved" and a.iter == c.iter
    assert _rel(c.x, a.x) <= bar and _rel(c.s, a.s) <= bar and _rel(c.y, a.y) <= bar


# ---- 3. the reference's custom_cone.jl problems against the oracle ------------------------
_ST = dict(max_iter=2000, eps_abs=1e-5, eps_rel=1e-5)


@pytest.mark.parametrize("hooks", [True, False])
@pytest.mark.parametrize("problem", ["lp", "dual_infeasible", "primal_infeasible"])
def test_reference_problems_match_the_oracle(oracle, problem, hooks):
    P, q, A, b, sets = getattr(CC, problem + "_problem" if problem != "lp" else "lp_problem")(CC.nonpos_type(hooks))
    model = cosmo_b200.Model()
    model.set(P, q, A, b, sets, cosmo_b200.Settings(**_ST))
    res = model.optimize()
    ref = O.solve(P, q, A, b, CC.to_oracle(sets), O.Settings(kkt_solver="cg", accelerator="empty", **_ST))
    print("MEAS %s hooks=%s engine %s/%d oracle %s/%d" % (problem, hooks, res.status, res.iter, ref.status, ref.iter))
    expected = {"lp": "Solved", "dual_infeasible": "Dual_infeasible" if hooks else "Max_iter_reached",
                "primal_infeasible": "Primal_infeasible" if hooks else "Max_iter_reached"}[problem]
    assert res.status == ref.status == expected
    assert res.iter == ref.iter
    if problem == "lp":
        assert abs(res.obj_val + 7.0) <= 1e-3 and abs(res.obj_val - ref.obj_val) <= 1e-6


# ---- 4. the certificate hooks through cosmo_b200_infeasibility_test ----------------------
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_family_bit_16_follows_the_hooks_on_both_sides_of_the_tolerance(dtype):
    tol = 1e-4
    for hooks in (True, False):
        kind = CC.nonpos_type(hooks)
        sets = [M.CustomCone(kind, 2)]
        for second, certified in ((2 * tol, True), (0.5 * tol, False)):
            v = np.array([1.0, second])
            # primal rig: A = 0, b = 0, delta_y = -v: the cone test sees in_dual(-v) = all(v >= tol)
            eng = _engine(sp.identity(1, format="csc"), np.zeros(1), sp.csc_matrix((2, 1)), np.zeros(2), sets, dtype=dtype,
                          scaling=0, eps_prim_inf=tol, eps_dual_inf=tol)
            rec = eng.infeasibility_test(0, -v)
            assert rec["gate"] == 4 and bool(rec["families"] & E.FAMILY_CUSTOM) == (not (hooks and certified)), (hooks, second, rec)
            assert rec["verdict"] == int(hooks and certified)
            eng.close()
            # dual rig: A = I, P = 0, q = -v, delta_x = v: in_pol_recc(v) = all(v >= tol)
            eng = _engine(sp.csc_matrix((2, 2)), -v, sp.identity(2, format="csc"), np.zeros(2), sets, dtype=dtype,
                          scaling=0, eps_prim_inf=tol, eps_dual_inf=tol)
            rec = eng.infeasibility_test(1, v)
            assert rec["gate"] == 4 and bool(rec["families"] & E.FAMILY_CUSTOM) == (not (hooks and certified)), (hooks, second, rec)
            assert rec["verdict"] == int(hooks and certified)
            eng.close()


# ---- 5. scaling ------------------------------------------------------------------------
def test_device_ruiz_gives_each_custom_cone_one_scaling(oracle):
    builtin, custom = _mixed_sets()
    sets = builtin[:2] + custom
    rng = np.random.default_rng(8)
    m, n = sum(S.dim for S in sets), 25
    A = (sp.random(m, n, density=0.2, random_state=9, format="csc") * 20.0 + sp.eye(m, n, format="csc")).tocsc()
    P = sp.eye(n, format="csc") * 3.0
    q, b = rng.standard_normal(n), rng.standard_normal(m)
    eng = E.Engine(P, q, A, b, _tuples(sets), cosmo_b200.Settings(scaling=10).to_struct(), equilibrate=True)
    D, Ed, c = eng.scaling()
    *_, smat = O.scale_ruiz(P, q, A, b, CC.to_oracle(sets), O.Settings(scaling=10))
    assert _rel(D, smat.D) <= 1e-13 and _rel(Ed, smat.E) <= 1e-13 and abs(c - smat.c) <= 1e-13 * abs(smat.c)
    off = sum(S.dim for S in builtin[:2])
    for S in custom:
        assert np.ptp(Ed[off:off + S.dim]) <= 4 * U64 * Ed[off], S.dim
        off += S.dim
    eng.close()


# ---- 6. updates leave the engine as a fresh create does ---------------------------------
def _solve(eng):
    r = eng.solve()
    return r.status, r.iter, r.x.copy(), r.s.copy(), r.mu.copy()


def _same(a, b):
    assert a[:2] == b[:2] and all(np.array_equal(u, v) for u, v in zip(a[2:], b[2:])), (a[:2], b[:2])


@pytest.mark.parametrize("kkt", ["CGIndirectKKTSolver", "DeviceLdlKKTSolver"])
def test_updates_warm_start_and_reset_match_a_fresh_create(kkt):
    P0, q0, A0, b0, sets = _socp(CC.soc2_type(), seed=3)
    P1, q1, A1, b1, _ = _socp(CC.soc2_type(), seed=3)
    rng = np.random.default_rng(11)
    P1 = P1.copy(); A1 = A1.copy()
    P1.data = P1.data * (1.0 + 0.1 * rng.random(P1.nnz)); P1 = ((P1 + P1.T) / 2).tocsc()
    A1.data = A1.data * (1.0 + 0.1 * rng.random(A1.nnz))
    q1, b1 = q0 + 0.1 * rng.standard_normal(q0.size), b0 * 1.05
    P0 = ((P0 + P0.T) / 2).tocsc()
    P1.sort_indices(); P0.sort_indices()
    st = cosmo_b200.Settings(kkt_solver=kkt).to_struct()
    fresh = E.Engine(P1, q1, A1, b1, _tuples(sets), st)
    ref = _solve(fresh)
    fresh.reset()
    _same(_solve(fresh), ref)                                    # reset
    eng = E.Engine(P0, q0, A0, b0, _tuples(sets), st)
    _solve(eng)
    eng.update_matrices(P1.data, A1.data, q1, b1)
    _same(_solve(eng), ref)                                      # update_matrices
    eng2 = E.Engine(P1, q0, A1, b0, _tuples(sets), st)
    eng2.update_qb(q1, b1)
    _same(_solve(eng2), ref)                                     # update_qb before the first solve
    eng2.warm_start(np.zeros(P1.shape[0]), np.zeros(A1.shape[0]), np.zeros(A1.shape[0]))
    eng2.reset()
    _same(_solve(eng2), ref)                                     # warm start from zero, then reset
    for e in (fresh, eng, eng2):
        e.close()


# ---- 7. a decomposed model keeps its custom cones as plain blocks ---------------------------
def test_decomposed_model_with_a_custom_cone():
    rng = np.random.default_rng(12)
    N = 10
    tri = [(i, j) for j in range(N) for i in range(j + 1)]
    d = len(tri)
    n = 4
    rows, cols, vals = [], [], []
    for r, (i, j) in enumerate(tri):
        if i == j or i == 0 or i + 1 == j:
            for k in range(n):
                rows.append(r); cols.append(k); vals.append(rng.standard_normal())
    A_psd = sp.csc_matrix((vals, (rows, cols)), shape=(d, n))
    b_psd = np.array([5.0 if i == j else 0.0 for i, j in tri]) * np.sqrt(1.0)
    A_soc = sp.csc_matrix(np.vstack([np.zeros((1, n)), rng.standard_normal((5, n))]))
    b_soc = np.concatenate([[10.0], np.zeros(5)])
    A = sp.vstack([A_psd, A_soc], format="csc")
    b = np.concatenate([b_psd, b_soc])
    P, q = sp.eye(n, format="csc"), rng.standard_normal(n)
    out = {}
    for name, S in (("soc", M.SecondOrderCone(6)), ("soc2", M.CustomCone(CC.soc2_type(), 6))):
        for dec in (False, True):
            model = cosmo_b200.Model()
            model.set(P, q, A, b, [M.PsdConeTriangle(d), S], cosmo_b200.Settings(decompose=dec, merge_strategy="NoMerge"))
            out[name, dec] = model.optimize()
            if dec:
                assert model._dec is not None and model._dec.blocks
    for dec in (False, True):
        a, c = out["soc", dec], out["soc2", dec]
        assert a.status == c.status == "Solved" and a.iter == c.iter
        assert _rel(c.x, a.x) <= 1e-9 and _rel(c.y, a.y) <= 1e-9
    assert abs(out["soc2", True].obj_val - out["soc2", False].obj_val) <= 1e-4 * max(1.0, abs(out["soc2", False].obj_val))


# ---- 8. the compile cache -----------------------------------------------------------------
def test_two_engines_with_one_type_compile_once():
    base = CC.soc2_type()
    kind = M.CustomConeType("soc2", base.source + "// %s\n" % uuid.uuid4().hex, "warp", 0, True, True)
    twin = M.CustomConeType("soc2", str(kind.source), "warp", 0, True, True)
    sets = [M.CustomCone(kind, 4), M.CustomCone(twin, 6), M.CustomCone(CC.nonpos_type(), 3)]
    stats = []
    for _ in range(2):
        eng = _project_engine(sets)
        stats.append(eng.custom_cone_stats())
        eng.close()
    assert stats[0]["types"] == 2 and stats[0]["cones"] == 3     # equal descriptors are one type
    assert stats[0]["compilations"] + stats[0]["cache_hits"] == 2 and stats[0]["compilations"] >= 1
    assert stats[1] == {"types": 2, "cones": 3, "compilations": 0, "cache_hits": 2}


def test_create_refuses_missing_parameters_and_bad_descriptors():
    linf = CC.linf_type()
    tuples = [(E.CUSTOM, 4, None, linf)]                           # n_params = 1 but no parameters
    with pytest.raises(E.EngineError) as ei:
        E.Engine(sp.identity(1, format="csc"), np.zeros(1), sp.csc_matrix((4, 1)), np.zeros(4), tuples, E.default_settings())
    assert ei.value.code == E.ERR_INVALID
    bad = M.CustomConeType("soc2", CC.SOC2_SRC, "warp")
    bad.name = "not an identifier"
    bad._bytes = (b"not an identifier", bad._bytes[1])
    with pytest.raises(E.EngineError) as ei:
        _project_engine([M.CustomCone(bad, 3)])
    assert ei.value.code == E.ERR_INVALID
