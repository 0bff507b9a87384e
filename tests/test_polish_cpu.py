"""Solution polishing without a GPU: the restatement of tests/polish_reference.py (classification rule, convergence of
the refinement to the exact reduced KKT solution, the reference's known answers after an oracle ADMM solve), the
Settings that select it and the C layout of cosmo_b200_polish_settings against the ctypes binding."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

import cosmo_b200
from cosmo_b200 import engine as E
from oracle import cosmo_oracle as O
from tests import golden_problems as G
from tests import polish_reference as R

INF = np.inf


# ---------------------------------------------------------------------------
# step 1: the classification rule
# ---------------------------------------------------------------------------
def test_classification_covers_every_branch():
    cls = np.array([R.ZERO, R.NONNEG, R.NONNEG, R.NONNEG, R.BOX, R.BOX, R.BOX, R.BOX, R.BOX, R.BOX, R.BOX], dtype=np.int8)
    l = np.array([-INF, -INF, -INF, -INF, 0.0, 0.0, 0.0, 0.0, 2.0, -INF, 0.0])
    u = np.array([INF, INF, INF, INF, 1.0, 1.0, 1.0, 1.0, 2.0, INF, INF])
    s = np.array([5.0, 0.0, 0.0, 1e-3, 0.0, 1.0, 0.5, 0.0, 2.0, 3.0, 7.0])
    mu = np.array([3.0, -1.0, 0.0, -1e-4, -1e-2, 1e-2, 0.0, 0.0, -4.0, 1e3, 1e3])
    kind, sbar = R.classify(cls, l, u, s, mu)
    want = [R.EQUALITY,     # ZeroSet: always, sbar 0
            R.LOWER,        # 0 < 1
            R.INACTIVE,     # tie 0 < 0 is false
            R.INACTIVE,     # 1e-3 < 1e-4 is false
            R.LOWER,        # Box at l
            R.UPPER,        # Box at u: 1 - 1 < 1e-2
            R.INACTIVE,     # interior, mu = 0
            R.INACTIVE,     # s = l with mu = 0: a tie, not active
            R.EQUALITY,     # l = u
            R.INACTIVE,     # infinite bounds are never active, whatever mu
            R.INACTIVE]     # infinite u: u - s = inf
    assert kind.tolist() == want
    assert sbar.tolist() == [0.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 2.0, 0.0, 0.0]


def test_classification_prefers_the_lower_bound_and_ignores_nan():
    cls = np.array([R.BOX, R.BOX, R.NONNEG], dtype=np.int8)
    kind, sbar = R.classify(cls, np.array([0.0, 0.0, -INF]), np.array([1e-12, 1.0, INF]), np.array([0.0, np.nan, np.nan]),
                            np.array([-1.0, 1.0, -1.0]))
    assert kind.tolist() == [R.LOWER, R.INACTIVE, R.INACTIVE] and sbar[0] == 0.0


def test_row_classes_refuse_conic_sets():
    cls, l, u = R.row_classes([O.ZeroSet(1), O.Nonnegatives(2), O.Box(np.array([0.0]), np.array([1.0]))])
    assert cls.tolist() == [0, 1, 1, 2] and l[3] == 0.0 and u[3] == 1.0 and l[0] == -INF
    with pytest.raises(ValueError):
        R.row_classes([O.SecondOrderCone(3)])


# ---------------------------------------------------------------------------
# step 4: refinement converges to the exact reduced KKT solution
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_refinement_reaches_the_exact_reduced_kkt_solution(seed):
    rng = np.random.default_rng(seed)
    n, m = 40, 60
    B = sp.random(n, n, density=0.1, random_state=rng)
    P = sp.csc_matrix(B @ B.T + 0.1 * sp.identity(n))
    A = sp.csc_matrix(sp.random(m, n, density=0.15, random_state=rng) + sp.eye(m, n))
    q, b = rng.standard_normal(n), rng.standard_normal(m)
    kind = rng.choice([R.INACTIVE, R.LOWER, R.UPPER, R.EQUALITY], size=m, p=[0.55, 0.15, 0.15, 0.15]).astype(np.int8)
    sbar = np.where(kind == R.UPPER, 1.0, 0.0) * rng.uniform(0.5, 1.0, m)
    act = np.flatnonzero(kind != R.INACTIVE)
    assert len(act) < n
    Aa = A[act]
    Kex = sp.bmat([[P, Aa.T], [Aa, None]], format="csc")
    z = spla.splu(Kex).solve(np.concatenate([-q, (b - sbar)[act]]))
    x, nu, rref = R.refine(P, q, A, b, kind, sbar, delta=1e-6, refine_iter=3)
    assert np.linalg.norm(x - z[:n]) <= 1e-12 * np.linalg.norm(z[:n])
    assert np.linalg.norm(nu[act] - z[n:]) <= 1e-12 * np.linalg.norm(z[n:])
    assert np.all(nu[kind == R.INACTIVE] == 0.0)
    assert rref <= 1e-12 * (1 + np.abs(q).max() + np.abs(b).max())
    # without refinement the regularisation leaves an O(delta) error
    x0, _, r0 = R.refine(P, q, A, b, kind, sbar, delta=1e-6, refine_iter=0)
    assert r0 > rref


# ---------------------------------------------------------------------------
# the reference's known answers after an oracle ADMM solve at the default eps
# ---------------------------------------------------------------------------
KNOWN = [("G1", G.g1_qp_nonneg, G.G1_X, G.G1_OBJ), ("G1b", G.g1_qp_box, G.G1_X, G.G1_OBJ),
         ("G2", G.g2_box_feasible, np.array([0.0, 1.0]), -0.5), ("G12", G.g12_lp, G.G12_X, G.G12_OBJ)]


@pytest.mark.parametrize("name,builder,x_star,obj_star", KNOWN, ids=[k[0] for k in KNOWN])
def test_restatement_reproduces_the_known_answers(name, builder, x_star, obj_star):
    P, q, cons = builder()
    Pm, qm, A, b, cones = O.assemble(P, q, cons)
    res = O.solve(Pm, qm, A, b, cones, O.Settings())
    assert res.status == "Solved"
    assert np.abs(res.x - x_star).max() > 1e-9          # ADMM alone stops short of the exact answer
    cls, l, u = R.row_classes(cones)
    out = R.polish(Pm, qm, A, b, cls, l, u, res.x, res.s, -res.y)
    assert out["status"] == 1
    assert np.abs(out["x"] - x_star).max() <= 1e-9
    assert abs(out["obj_val"] - obj_star) <= 1e-9
    assert out["r_prim"] <= out["unpolished"][0] and out["r_dual"] <= out["unpolished"][1]


def test_a_wrong_active_set_is_rejected():
    # G12 after two iterations: the guess makes the candidate worse, and the restatement keeps the iterates
    P, q, cons = G.g12_lp()
    Pm, qm, A, b, cones = O.assemble(P, q, cons)
    res = O.solve(Pm, qm, A, b, cones, O.Settings(max_iter=2))
    cls, l, u = R.row_classes(cones)
    out = R.polish(Pm, qm, A, b, cls, l, u, res.x, res.s, -res.y)
    unp = out["unpolished"]
    cand = R.residuals(Pm, qm, A, b, out["x_p"], out["s_p"], out["mu_p"])
    u = 2.0 ** -53
    rule = cand[0] <= max(unp[0], 10 * u * (1 + cand[2])) and cand[1] <= max(unp[1], 10 * u * (1 + cand[3]))
    assert out["status"] == int(rule) and (out["r_prim"], out["r_dual"]) == cand[:2]
    if out["status"] == 0:
        assert np.array_equal(out["x"], res.x) and np.array_equal(out["y"], res.y)


# ---------------------------------------------------------------------------
# Settings and the binding
# ---------------------------------------------------------------------------
def test_settings_validation():
    st = cosmo_b200.Settings()
    assert (st.polish, st.polish_delta, st.polish_refine_iter) == (False, 1e-6, 3)
    for kkt in ("DeviceLdlKKTSolver", "DeviceSupernodalKKTSolver", "MKLPardisoKKTSolver"):
        cosmo_b200.Settings(polish=True, kkt_solver=kkt).to_struct()
    for kkt in ("CGIndirectKKTSolver", "MINRESIndirectKKTSolver", "IndirectReducedKKTSolver:MINRES"):
        with pytest.raises(E.EngineError) as e:
            cosmo_b200.Settings(polish=True, kkt_solver=kkt).to_struct()
        assert e.value.code == E.ERR_UNSUPPORTED
        cosmo_b200.Settings(polish=False, kkt_solver=kkt).to_struct()
    for bad in ({"polish_delta": 0.0}, {"polish_delta": -1e-6}, {"polish_delta": float("inf")}, {"polish_delta": float("nan")},
                {"polish_refine_iter": -1}, {"polish_refine_iter": 101}):
        with pytest.raises(E.EngineError) as e:
            cosmo_b200.Settings(polish=True, kkt_solver="DeviceLdlKKTSolver", **bad).to_struct()
        assert e.value.code == E.ERR_INVALID


def test_device_solution_with_polish_is_refused_before_the_solve():
    model = cosmo_b200.Model()
    P, q, cons = G.g1_qp_box()
    model.is_assembled = True
    model.settings = cosmo_b200.Settings(polish=True, kkt_solver="DeviceLdlKKTSolver")
    with pytest.raises(ValueError):
        model.optimize(solution="device")
    assert model.engine is None


_PROBE = r"""
#include <stddef.h>
#include <stdio.h>
#include "cosmo_b200.h"
#define OFF(f) printf(#f " %zu\n", offsetof(cosmo_b200_polish_settings, f))
int main(void) {
  double out[8];
  printf("sizeof %zu\n", sizeof(cosmo_b200_polish_settings));
  OFF(delta); OFF(refine_iter); OFF(reserved);
  printf("abi %d %d\n", COSMO_B200_ABI_VERSION, cosmo_b200_abi_version());
  /* a null handle or a null out is refused before anything is read */
  printf("null_handle %d %d\n", cosmo_b200_polish(NULL, NULL, NULL, NULL, NULL, out),
         cosmo_b200_polish(NULL, NULL, NULL, NULL, NULL, NULL));
  return 0;
}
"""


def test_c_layout_of_the_polish_settings_matches_the_binding(tmp_path):
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib = E.load_library()
    assert "cosmo_b200_polish" in E.EXPORTS
    assert lib.cosmo_b200_abi_version() == 4                     # additive: one new symbol and one new struct
    src, exe = tmp_path / "polish_probe.c", str(tmp_path / "polish_probe")
    src.write_text(_PROBE)
    subprocess.run([cc, "-std=c99", "-Wall", "-Werror", "-I", os.path.join(root, "include"), str(src), lib._name,
                    "-Wl,-rpath," + os.path.dirname(lib._name), "-o", exe], check=True)
    vals = dict(line.split(" ", 1) for line in subprocess.run([exe], check=True, capture_output=True, text=True).stdout.splitlines())
    assert int(vals.pop("sizeof")) == ctypes.sizeof(E.PolishSettings) == 16
    assert vals.pop("abi") == "4 4" and vals.pop("null_handle") == "%d %d" % (E.ERR_INVALID, E.ERR_INVALID)
    assert sorted(vals) == sorted(n for n, _ in E.PolishSettings._fields_)
    for name, off in vals.items():
        assert getattr(E.PolishSettings, name).offset == int(off), name
