"""The extended-precision Anderson restatement (tests/anderson_reference.py) pinned to the two fp64 restatements it
restates -- oracle.cosmo_oracle.AndersonAccelerator and tests/anderson_variants.NormalEquationsAccelerator -- on the
same sequences, and to exact rationals on small integer cases."""
from fractions import Fraction

import numpy as np
import pytest

from oracle import cosmo_oracle as O
from tests import anderson_reference as R
from tests import anderson_variants as V


def _fp64_run(dim, mem, min_mem, t, memory, reg, lam, g, x):
    """(formed, accepted, eta, candidate) of every step of the fp64 restatement"""
    if t == "Type2{QRDecomp}":
        aa = O.AndersonAccelerator(dim, mem, min_mem)
    else:
        aa = V.NormalEquationsAccelerator(dim, mem, min_mem, type1=t == "Type1", rolling=memory == "RollingMemory",
                                          regularizer=reg, lam=lam)
    out = []
    for k in range(g.shape[0]):
        init = aa.init_phase
        failed = sum(1 for e in aa.log if e[1] == "acc_failed")
        aa.update(g[k].copy(), x[k].copy(), k)
        l = 0 if init else min(aa.iter, aa.mem)
        cand = g[k].copy()
        aa.accelerate(cand, x[k], k)
        formed = aa.success or sum(1 for e in aa.log if e[1] == "acc_failed") > failed
        out.append((formed, aa.success, l, aa.eta[:l].copy(), cand))
    return out


@pytest.mark.parametrize("t,memory,reg", V.TYPES)
@pytest.mark.parametrize("dim,mem", [(40, 5), (4, 8), (30, 9)])
def test_matches_the_fp64_restatements(t, memory, reg, dim, mem):
    # every step's bookkeeping and verdict, and eta (physical order) and the candidate within 1e-13 kappa of the system
    # solved (a full-dimensional rolling window, dim = 4, is far less well conditioned than the designed 10)
    g, x = R.sequence(dim, 3 * mem + 2, kappa=10.0, seed=dim + mem, rank=min(mem, dim))
    ref = R.Reference(dim, mem, 3, t, memory, reg, 1e-8)
    steps = ref.run(g, x, solve_at=set())
    fp64 = _fp64_run(dim, mem, 3, t, memory, reg, 1e-8, g, x)
    for k, (formed, ok, l, eta, cand) in enumerate(fp64):
        ref = R.Reference(dim, mem, 3, t, memory, reg, 1e-8)     # analysis() reads the state after step k
        st = ref.run(g[:k + 1], x[:k + 1])[k]
        assert (st.formed, st.accepted, st.l, steps[k].l) == (formed, ok, l, l), (k, st.reason)
        if ok:
            e = np.array([float(v) for v in st.eta])
            tol = 1e-13 * ref.analysis(st)["kappa_sys"] * (1 + np.linalg.norm(e))
            assert np.linalg.norm(eta - e) <= tol, (k, np.linalg.norm(eta - e), tol)
            assert np.allclose(cand, st.cand, rtol=tol, atol=tol), k
    assert sum(f[1] for f in fp64) >= mem


def test_least_squares_minimiser_and_kappa():
    # Type2 with no shift: eta is the exact least-squares minimiser; kappa_F of a designed window; Type2 normal
    # equations square it
    g, x = R.sequence(50, 7, kappa=1e4, seed=3, rank=6)
    for t in ("Type2{QRDecomp}", "Type2{NormalEquations}"):
        ref = R.Reference(50, 6, 3, t)
        st = ref.run(g, x)[6]
        a = ref.analysis(st)
        assert st.l == 6 and 1e3 < a["kappa_F"] < 1e6
        if st.eta is not None:
            assert np.allclose([float(v) for v in st.eta], a["eta_ls"], rtol=1e-30, atol=1e-30 * np.linalg.norm(a["eta_ls"]))
        if t != "Type2{QRDecomp}":
            assert 0.5 * a["kappa_F"] ** 2 <= a["kappa_sys"] <= 50 * a["kappa_F"] ** 2


def _exact_design():
    F = np.array([[2.0, 1.0, 0.0], [0.0, 3.0, 1.0], [1.0, 0.0, 4.0], [0.0, 0.0, 0.0], [0.0, 0.0, 0.0]])
    G = np.array([[0.0, 0.0, 0.0], [0.0, 0.0, 0.0], [0.0, 0.0, 0.0], [1.0, 2.0, 0.0], [0.0, 1.0, 3.0]])
    f_last = np.array([5.0, -1.0, 2.0, 0.0, 0.0])
    return F, G, f_last


@pytest.mark.parametrize("t", ["Type2{QRDecomp}", "Type2{NormalEquations}", "Type1"])
def test_exact_rationals(t):
    # integer F, G, f: eta of the restatement equals the rational solution of the same system to 50 digits
    F, G, f_last = _exact_design()
    g, x = R.from_columns(F, G, f_last)
    ref = R.Reference(5, 5, 3, t)
    st = ref.run(g, x)[3]
    A = F + G if t == "Type1" else F
    M = [[int(v) for v in row] for row in (A.T @ F)]
    rhs = [int(v) for v in A.T @ f_last]
    want = R.exact_lu_eta(M, rhs)
    assert st.accepted and len(want) == 3
    for got, w in zip(st.eta, want):
        assert abs(Fraction(str(got)) - w) <= Fraction(1, 10 ** 45) * (1 + abs(w))
    cand = g[3] - G @ np.array([float(w) for w in want])
    assert np.allclose(st.cand, cand, rtol=1e-15, atol=1e-15)


def test_rejection_rules_and_memory_bookkeeping():
    # zero pivot from an exact duplicate (and the rest of the QR cycle), |eta| over 1e4, non-finite inputs, l < min_mem;
    # RestartedMemory restarts at mem, RollingMemory overwrites column iter mod mem
    F = np.zeros((6, 4))
    F[0, 0] = F[0, 1] = 4.0
    F[1, 2], F[2, 3] = 2.0, 1.0
    g, x = R.from_columns(F, np.zeros((6, 4)), np.array([1.0, 1.0, 1.0, 0.0, 0.0, 0.0]))
    for t in ("Type2{QRDecomp}", "Type2{NormalEquations}"):
        steps = R.Reference(6, 4, 3, t).run(g, x)
        assert [s.reason for s in steps] == [None, None, None, "zero_pivot", "zero_pivot"]
    F = np.diag([1.0, 1.0, 1.0])
    for target, reason in ((0.99e4, "accepted"), (1.01e4, "eta_norm")):
        g, x = R.from_columns(F, np.zeros((3, 3)), np.array([target, 0.0, 0.0]))
        assert R.Reference(3, 4, 3).run(g, x)[3].reason == reason
    g, x = R.sequence(10, 6, seed=1, rank=5)
    g[3, 2] = np.nan
    assert [s.reason for s in R.Reference(10, 8, 3).run(g, x)[3:]] == ["zero_pivot"] * 3
    assert [s.reason for s in R.Reference(10, 8, 3, "Type1").run(g, x)[3:]] == ["nonfinite_entry"] * 3
    g, x = R.sequence(10, 12, seed=2, rank=4)
    assert [s.j for s in R.Reference(10, 4, 3, "Type1", "RollingMemory").run(g, x)] == [-1] + [k % 4 for k in range(11)]
    rs = R.Reference(10, 4, 3).run(g, x)
    assert [s.l for s in rs] == [0, 1, 2, 3, 4, 1, 2, 3, 4, 1, 2, 3]
    assert [s.formed for s in R.Reference(10, 4, 5, "Type1").run(g, x)] == [False] * 12


def test_pivot_ties_pick_the_first_row():
    F = np.zeros((6, 3))
    F[0, 0] = 1.0
    F[0, 1], F[1, 1] = -2.0, 1.0
    F[0, 2], F[2, 2] = 2.0, 1.0
    g, x = R.from_columns(F, np.zeros((6, 3)), np.array([1.0, 3.0, -2.0, 0.0, 0.0, 0.0]))
    st = R.Reference(6, 5, 3, "Type2{NormalEquations}").run(g, x)[3]
    assert st.ties == 1 and st.pivots[0] == 1 and st.accepted
    assert [float(v) for v in st.eta] == pytest.approx([11.0, 3.0, -2.0], rel=1e-40)
