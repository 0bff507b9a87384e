"""Kernel parity of the device Anderson accelerator (csrc/aa.cuh through cosmo_b200_accelerator_probe) against the
extended-precision restatement of tests/anderson_reference.py: every variant of V.TYPES in fp64 and fp32, windows of 3
to 32 columns, dimensions below, at and past the 256-thread block and past the grid-stride wrap, both memories over
several wraps and restarts, and every rejection rule.

Error bars, set from the error analysis of each path before any device run (u the unit roundoff of T, l the window,
n_s the longest chain of additions in the device's two-stage sums over dim rows, rho >= 1 the rounding of the inputs:
f = x - g and the differences F, X are formed in T, and their exact perturbation -- known from the inputs by TwoSum --
over u |F|_2 (u |X|_F for X) is rho):
  * Type2{QRDecomp}, MGS without augmenting F by f.  The computed Q loses orthogonality by about u kappa, so Q'f
    carries an error of u kappa (|F| |eta| + |r|) and the back substitution multiplies it by |R^-1| = kappa / |F|:
        |d eta| <= C_QR l (n_s + l) u rho kappa^2 (|eta| + |r| / |F|_2).
    (A residual-only kappa^2 term, u (kappa + kappa^2 |r| / (|F| |eta|)), holds for the augmented MGS; without the
    augmentation the kappa^2 |eta| term is there at zero residual too, as a fp64 emulation of the MGS shows.)
  * Normal equations and Type1: M = A'B and rhs = A'f summed over dim rows (|dM| <= n_s u |A|_F |B|_F), the shift, and
    LU with partial pivoting (backward error l u |M_s|):
        |d eta| <= C_NE (n_s + l) u rho |M_s^-1|_F ((|A|_F |B|_F + shift) |eta| + |A|_F |f|).
  * The candidate g - G eta, G formed as differences of g:
        |d cand| <= |G|_F |d eta|_bar + (l + 3) u (|g| + |G|_F |eta|) (1 + sqrt(l) |eta|).
C_QR = C_NE = 1.  Where a bar exceeds a tenth of |eta|, or |eta| of the restatement lies within the bar of 1e4, the
type T cannot decide the candidate; such a step compares the bookkeeping only and counts as undecided.  The designed
edge cases below are all decided."""
import math

import numpy as np
import pytest
import scipy.sparse as sp

import cosmo_b200
from cosmo_b200 import engine as E
from tests import anderson_reference as R
from tests import anderson_variants as V

pytestmark = pytest.mark.gpu

U = {np.dtype(np.float64): 2.0 ** -53, np.dtype(np.float32): 2.0 ** -24}
K_BLOCK, K_MAX_GRID = 256, 132 * 8
C_QR = C_NE = 1.0
WORST = {}          # (path, dtype) -> worst measured error / bar, printed by test_report_worst_ratios


def _engine(dim, dtype=np.float64, t="Type2{QRDecomp}", memory="RestartedMemory", reg="NoRegularizer", mem=15, min_mem=3,
            lam=1e-8, safeguard_tol=2.0):
    """an engine whose operator variable has n + m = dim entries (n = 1), with the accelerator variant set"""
    m = dim - 1
    st = cosmo_b200.Settings(accelerator="AndersonAccelerator", accelerator_mem=mem, accelerator_min_mem=min_mem,
                             accelerator_type=t, accelerator_memory=memory, accelerator_regularizer=reg,
                             accelerator_lambda=lam, safeguard_tol=safeguard_tol)
    eng = E.Engine(sp.identity(1, format="csc"), np.zeros(1), sp.csc_matrix((m, 1)), np.zeros(m),
                   [cosmo_b200.model.set_tuple(cosmo_b200.Nonnegatives(m))], st.to_struct(), dtype=dtype)
    eng.set_accelerator(st.accelerator_struct())
    return eng


def _reference(dim, dtype, t, memory, reg, mem, min_mem=3, lam=1e-8):
    return R.Reference(dim, mem, min_mem, t, memory, reg, lam, dtype)


def _n_s(dim):
    grid = min(max(-(-dim // K_BLOCK), 1), K_MAX_GRID)
    return -(-dim // (K_BLOCK * grid)) + 17 + -(-grid // 32)


def _two_diff(a, b):
    """(fl(a - b), the exact error a - b - fl(a - b)) in the type of a and b (TwoSum)"""
    s = a - b
    bb = s - a
    return s, (a - (s - bb)) - (-b - bb)


def _input_rounding(g, x):
    """(max |df|, max |dF column|, max |dX column|): the exact perturbations of f = x - g and of the differences F and X
    that forming them in T causes, over the whole sequence, in float64"""
    with np.errstate(all="ignore"):
        f, ef = _two_diff(x, g)
        F, eF = _two_diff(f[1:], f[:-1])
        _, eX = _two_diff(x[1:], x[:-1])
    ef, eF, eX = (np.nan_to_num(e.astype(np.float64)) for e in (ef, eF, eX))
    dF = np.linalg.norm(eF, axis=1) + np.linalg.norm(ef[1:], axis=1) + np.linalg.norm(ef[:-1], axis=1)
    n = lambda e: float(np.max(e)) if e.size else 0.0
    return n(np.linalg.norm(ef, axis=1)), n(dF), n(np.linalg.norm(eX, axis=1))


def _bars(ref, st, a, dim, dtype, rnd):
    """(bar of |d eta|, bar of |d cand|) of the step, from the restatement's analysis `a` and the input rounding `rnd`"""
    u, l, ns = U[np.dtype(dtype)], st.l, _n_s(dim)
    eta = a["nrm_eta"]
    df, dF, dX = rnd
    if ref.type == "Type2{QRDecomp}":
        rho = max(1.0, (df + math.sqrt(l) * dF) / (u * a["nrm_F"]))
        b_eta = C_QR * l * (ns + l) * u * rho * a["kappa_F"] ** 2 * (eta + a["nrm_r"] / a["nrm_F"])
    else:
        rho = max(1.0, (df + math.sqrt(l) * dF) / (u * a["nrm_B"]), math.sqrt(l) * dX / (u * a["nrm_A"]))
        b_eta = C_NE * (ns + l) * u * rho * a["inv_sys"] * ((a["nrm_A"] * a["nrm_B"] + a["shift"]) * eta
                                                            + a["nrm_A"] * a["nrm_f"])
    b_cand = a["nrm_G"] * b_eta + (l + 3) * u * (a["nrm_g"] + a["nrm_G"] * eta) * (1.0 + math.sqrt(l) * eta)
    return b_eta, b_cand


def _path(t):
    return "QR" if t == "Type2{QRDecomp}" else ("Type1" if t == "Type1" else "NE")


def _compare(eng, ref, g, x, dtype, check=None, w_next=None):
    """probe and restatement on the same pairs; bookkeeping on every step, numbers on the steps of `check` (None:
    every formed step).  Returns (probe output, reference steps, number of decided steps)."""
    out = eng.accelerator_probe(g, x, w_next)
    steps = ref.run(g, x, solve_at=check)
    rnd = _input_rounding(g, x)
    decided = 0
    for k, st in enumerate(steps):
        assert (out["formed"][k], out["l"][k]) == (int(st.formed), st.l), (k, out["formed"][k], out["l"][k], st.formed, st.l)
        if st.l:
            assert out["j"][k] == st.j, (k, out["j"][k], st.j)
        if not out["accepted"][k]:
            assert np.array_equal(out["cand"][k].view(np.uint8), g[k].view(np.uint8)), k     # g bit for bit
            assert np.all(np.isnan(out["eta"][k]))
        if not st.formed or (check is not None and k not in check):
            continue
        if st.reason in ("nonfinite_entry", "zero_pivot", "nonfinite_pivot", "nonfinite_eta"):
            assert not out["accepted"][k], (k, st.reason)
            decided += 1
            continue
        a = ref.analysis(st)
        b_eta, b_cand = _bars(ref, st, a, ref.dim, dtype, rnd)
        nrm = a["nrm_eta"]
        if not (b_eta < 0.1 * nrm or b_eta < 1e-3) or abs(nrm - 1e4) <= b_eta:
            continue                                   # T cannot decide this candidate
        decided += 1
        assert bool(out["accepted"][k]) == st.accepted, (k, st.reason, nrm, b_eta)
        if not st.accepted:
            continue
        l = st.l
        eta_ref = np.array([float(e) for e in st.eta])
        e_eta = np.linalg.norm(out["eta"][k][:l] - eta_ref)
        e_cand = np.linalg.norm(out["cand"][k].astype(np.float64) - st.cand)
        assert np.all(np.isnan(out["eta"][k][l:]))
        assert e_eta <= b_eta and e_cand <= b_cand, (k, e_eta, b_eta, e_cand, b_cand, a["kappa_F"])
        key = (_path(ref.type), np.dtype(dtype).name)
        WORST[key] = max(WORST.get(key, (0.0, 0.0)), (e_eta / b_eta if b_eta else 0.0, a["kappa_sys"]))
    return out, steps, decided


# every mem of the issue and every dimension class: below the window (2, 5), at it, around one and two 256-row blocks
SHAPES = [(3, 2), (3, 5), (3, 3), (8, 255), (8, 8), (9, 256), (9, 257), (16, 16), (16, 255), (17, 257), (17, 5),
          (24, 256), (24, 24), (25, 257), (25, 25), (32, 255), (32, 32), (32, 256)]


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("t,memory,reg", V.TYPES)
def test_windows_and_dimensions(t, memory, reg, dtype):
    # 3 mem + 2 updates: a rolling window wraps three times, a restarted one restarts at mem and 2 mem (the restart
    # boundary at l = mem and l = mem + 1 = 1).  Numbers at the full window, one step past it and at the end.  Each
    # variant and type runs a third of SHAPES, so that every shape meets eight or nine of the 26.
    decided = 0
    off = V.TYPES.index((t, memory, reg)) + (1 if dtype == np.float32 else 0)
    shapes = [(i, s) for i, s in enumerate(SHAPES) if (i + off) % 3 == 0]
    for i, (mem, dim) in shapes:
        min_mem = 2 if dim == 2 else 3
        K = 3 * mem + 2
        eff = min(mem, dim)
        # twice as many directions as columns: each window of l random combinations is well conditioned (kappa of
        # a few) unless the window fills the whole space (dim <= mem)
        g, x = R.sequence(dim, K, kappa=1.0 if i % 2 else 10.0, dtype=dtype, seed=i, rank=min(2 * eff, dim))
        check = {eff, eff + 1, K - 1}
        eng = _engine(dim, dtype, t, memory, reg, mem, min_mem)
        out, steps, d = _compare(eng, _reference(dim, dtype, t, memory, reg, mem, min_mem), g, x, dtype, check)
        decided += d
        js = [s.j for s in steps if s.l]
        if memory == "RollingMemory":
            assert max(s.l for s in steps) == eff and js.count(0) >= 3, (mem, dim, js)
        else:
            assert sum(1 for k in range(1, len(steps)) if steps[k].l == 1 and steps[k - 1].l == eff) >= 2
        eng.close()
    # fp64 decides a step of every shape; in fp32 the worst-case bars of the wide windows exceed a tenth of |eta|
    assert decided >= (len(shapes) if dtype == np.float64 else 2), decided


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("kappa", [1.0, 1e3, 1e6, 1e10])
@pytest.mark.parametrize("t", ["Type2{QRDecomp}", "Type2{NormalEquations}", "Type1"])
def test_prescribed_condition(t, kappa, dtype):
    if kappa == 1e10 and dtype == np.float32:
        pytest.skip("kappa = 1e10 is beyond float32")
    dim, mem = 64, 8
    g, x = R.sequence(dim, mem + 1, kappa=kappa, dtype=dtype, seed=11, rank=mem)
    eng = _engine(dim, dtype, t, mem=mem)
    ref = _reference(dim, dtype, t, "RestartedMemory", "NoRegularizer", mem)
    out, steps, _ = _compare(eng, ref, g, x, dtype, check={mem})
    a = ref.analysis(steps[mem])
    assert 0.1 * kappa <= a["kappa_F"] <= 100 * kappa, a["kappa_F"]


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("t", ["Type2{QRDecomp}", "Type2{NormalEquations}", "Type1"])
def test_grid_stride_wrap(t, dtype):
    # dim > 2 kBlock kMaxGrid: every grid-stride loop of the aa kernels runs three rounds; the values sit on 1500 rows
    # spread over the whole range, the last one past the second wrap
    dim = 2 * K_BLOCK * K_MAX_GRID + 4099
    rows = np.unique(np.concatenate([np.linspace(0, dim - 1, 1497).astype(int), [dim - 1, dim - 2, 2 * K_BLOCK * K_MAX_GRID + 7]]))
    g, x = R.sequence(dim, 9, kappa=10.0, dtype=dtype, seed=3, rank=8, support=rows)
    eng = _engine(dim, dtype, t, mem=8)
    _, _, decided = _compare(eng, _reference(dim, dtype, t, "RestartedMemory", "NoRegularizer", 8), g, x, dtype, check={8})
    assert decided == 1


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("t,memory,reg", V.TYPES)
def test_min_mem_above_the_window(t, memory, reg, dtype):
    # l < min_mem forms no candidate: g comes back bit for bit
    g, x = R.sequence(40, 9, dtype=dtype, seed=5, rank=8)
    eng = _engine(40, dtype, t, memory, reg, mem=8, min_mem=6)
    out, steps, _ = _compare(eng, _reference(40, dtype, t, memory, reg, 8, 6), g, x, dtype)
    assert [int(v) for v in out["formed"]] == [0] * 6 + [1] * 3


def _dup_design(dtype, t):
    """columns 0 and 1 of F equal (2^3 e_0), column 2 = 2^3 e_1, the G differences on other rows (X = F + G, so X has
    the same duplicate); every value an integer, every sum exact"""
    dim = 12
    F = np.zeros((dim, 4))
    G = np.zeros((dim, 4))
    F[0, 0] = F[0, 1] = 8.0
    F[1, 2] = 8.0
    F[2, 3] = 4.0
    G[5, 0] = G[5, 1] = 2.0
    G[6, 2] = 3.0
    G[7, 3] = 1.0
    f_last = np.zeros(dim)
    f_last[:4] = [3.0, 5.0, 1.0, 2.0]
    return R.from_columns(F, G, f_last, dtype=dtype)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("t", ["Type2{QRDecomp}", "Type2{NormalEquations}", "Type1"])
def test_exact_duplicate_differences(t, dtype):
    # QR: R[1, 1] = 0 exactly, Q[:, 1] = 0/0, and every later candidate of the memory cycle is rejected.  Normal
    # equations: the Gram matrix is exactly singular, a zero pivot.  Then a restart clears it.
    g, x = _dup_design(dtype, t)
    g2, x2 = R.sequence(12, 6, dtype=dtype, seed=8, rank=4)
    g, x = np.concatenate([g, g2]), np.concatenate([x, x2])
    eng = _engine(12, dtype, t, mem=4)
    ref = _reference(12, dtype, t, "RestartedMemory", "NoRegularizer", 4)
    out, steps, _ = _compare(eng, ref, g, x, dtype)
    assert [s.reason for s in steps[3:5]] == ["zero_pivot", "zero_pivot"], [s.reason for s in steps]
    assert not out["accepted"][3] and not out["accepted"][4]
    if t == "Type2{QRDecomp}":
        assert not np.any(out["accepted"][3:5])
    assert out["accepted"][-1] or steps[-1].reason != "accepted"


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("t,memory,reg", V.TYPES)
@pytest.mark.parametrize("target", [0.99e4, 1.01e4])
def test_eta_norm_rule(t, memory, reg, dtype, target):
    # three orthogonal columns 2^k e_i, f = F eta* with eta* = (target, 0, 0): |eta| is target up to the shift's
    # relative 6e-8, far from the rule's 1e4 either way
    dim = 10
    F = np.zeros((dim, 3))
    G = np.zeros((dim, 3))
    F[0, 0], F[1, 1], F[2, 2] = 1.0, 2.0, 4.0
    G[5, 0], G[6, 1], G[7, 2] = 1.0, -1.0, 2.0
    f_last = np.zeros(dim)
    f_last[0] = target
    g, x = R.from_columns(F, G, f_last, dtype=dtype)
    eng = _engine(dim, dtype, t, memory, reg, mem=5)
    ref = _reference(dim, dtype, t, memory, reg, 5)
    out, steps, decided = _compare(eng, ref, g, x, dtype)
    assert steps[3].reason == ("accepted" if target < 1e4 else "eta_norm") and decided == 1
    assert bool(out["accepted"][3]) == (target < 1e4)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("t", ["Type2{QRDecomp}", "Type2{NormalEquations}", "Type1"])
@pytest.mark.parametrize("bad", [np.nan, np.inf])
def test_non_finite_inputs(t, dtype, bad):
    g, x = R.sequence(30, 8, dtype=dtype, seed=4, rank=6)
    g[4, 7] = bad                      # g of step 4: f_4, the columns of steps 4 and 5
    x[6, 2] = -bad                     # x of step 6
    eng = _engine(30, dtype, t, mem=10)
    out, steps, _ = _compare(eng, _reference(30, dtype, t, "RestartedMemory", "NoRegularizer", 10), g, x, dtype)
    assert all(s.reason not in (None, "accepted") for s in steps[4:])
    assert not np.any(out["accepted"][4:])


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_pivot_ties_of_opposite_sign(dtype):
    # M = F'F with M[1, 0] = -2, M[2, 0] = 2 above M[0, 0] = 1: a tie of opposite sign in the first pivot column
    dim = 8
    F = np.zeros((dim, 3))
    F[0, 0] = 1.0
    F[0, 1], F[1, 1] = -2.0, 1.0
    F[0, 2], F[2, 2] = 2.0, 1.0
    G = np.zeros((dim, 3))
    G[5, 0], G[6, 1], G[7, 2] = 1.0, 1.0, 1.0
    f_last = np.zeros(dim)
    f_last[:3] = [1.0, 3.0, -2.0]
    g, x = R.from_columns(F, G, f_last, dtype=dtype)
    for reg in ("NoRegularizer", "TikonovRegularizer"):
        eng = _engine(dim, dtype, "Type2{NormalEquations}", reg=reg, mem=5)
        ref = _reference(dim, dtype, "Type2{NormalEquations}", "RestartedMemory", reg, 5)
        out, steps, decided = _compare(eng, ref, g, x, dtype)
        assert steps[3].ties >= 1 and steps[3].pivots[0] == 1 and decided == 1 and out["accepted"][3]


def _orthogonal_f(dtype, scale):
    """f = scale on rows 0..31 (constant, so no difference sees it), history differences on rows 32..63 only, eta = 0"""
    dim = 64
    rng = np.random.default_rng(2)
    F = np.zeros((dim, 4))
    F[32:, :] = rng.integers(-4, 5, size=(32, 4))
    G = np.zeros((dim, 4))
    G[32:, :] = rng.integers(-3, 4, size=(32, 4))
    f_last = np.zeros(dim)
    f_last[:32] = float(dtype(scale))
    return R.from_columns(F, G, f_last, dtype=dtype)


@pytest.mark.parametrize("dtype,scale", [(np.float32, 1e19), (np.float32, 3e30), (np.float32, 1e-25),
                                         (np.float64, 1e160), (np.float64, 1e-170)])
def test_safeguard_norms_over_the_whole_range(dtype, scale):
    # |f|_2 far outside sqrt(max(T)) (or below sqrt(min(T))): a candidate whose f_acc = cand - w_next is 3 f must be
    # declined (the reference's norm(f, 2) rescales).  A plain sum of squares gives inf > 2 inf, false, and accepts it.
    t = "Type2{QRDecomp}"
    g, x = _orthogonal_f(dtype, scale)
    f = x.astype(np.float64) - g.astype(np.float64)
    for factor, declined in ((3.0, True), (1.5, False)):
        w_next = (g.astype(np.float64) - factor * f).astype(dtype)
        eng = _engine(64, dtype, t, mem=5)
        out = eng.accelerator_probe(g, x, w_next)
        assert out["accepted"][4] and np.array_equal(out["eta"][4][:4], np.zeros(4)), out["eta"][4]
        want_f = math.sqrt(32) * float(dtype(scale))
        assert abs(out["nrm_f"][4] / want_f - 1) < 1e-6, (out["nrm_f"][4], want_f)
        assert abs(out["nrm_f_acc"][4] / (factor * want_f) - 1) < 1e-6
        assert bool(out["declined"][4]) == declined, (factor, out["nrm_f"][4], out["nrm_f_acc"][4])


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("t", ["Type2{QRDecomp}", "Type2{NormalEquations}", "Type1"])
def test_overflowing_squares_never_accept_non_finite(t, dtype):
    # history differences near sqrt(max(T)) and above: the Gram sums overflow; the device rejects, never accepts a
    # non-finite candidate
    big = 1e30 if dtype == np.float32 else 1e200
    g, x = R.sequence(20, 6, dtype=np.float64, seed=9, rank=5)
    g, x = (g * big).astype(dtype), (x * big).astype(dtype)
    eng = _engine(20, dtype, t, mem=5)
    out = eng.accelerator_probe(g, x)
    for k in range(6):
        if out["accepted"][k]:
            assert np.all(np.isfinite(out["cand"][k])), k
        else:
            assert np.array_equal(out["cand"][k].view(np.uint8), g[k].view(np.uint8))
    assert not np.any(out["accepted"][4:])


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("t,memory,reg", [v for v in V.TYPES if v[2] != "TikonovRegularizer"])
def test_power_of_two_ladder_and_determinism(t, memory, reg, dtype):
    # inputs times 2^k: eta bit for bit, the candidate times 2^k exactly (Tikonov's lambda does not scale); two
    # identical probes agree bit for bit
    g, x = R.sequence(300, 12, kappa=10.0, dtype=dtype, seed=6, rank=8)
    eng = _engine(300, dtype, t, memory, reg, mem=8)
    base = eng.accelerator_probe(g, x)
    again = eng.accelerator_probe(g, x)
    for key in ("cand", "eta", "formed", "accepted", "l", "j"):
        b, a = np.ascontiguousarray(base[key]), np.ascontiguousarray(again[key])
        assert np.array_equal(b.view(np.uint8), a.view(np.uint8)), key
    assert base["accepted"].sum() >= 4
    for k in (-12, -3, 5, 20) if dtype == np.float32 else (-300, -7, 9, 400):
        s = np.ldexp(1.0, k)
        out = eng.accelerator_probe((g * s).astype(dtype), (x * s).astype(dtype))
        assert np.array_equal(out["accepted"], base["accepted"]), k
        assert np.array_equal(np.nan_to_num(out["eta"]), np.nan_to_num(base["eta"])), k
        assert np.array_equal(out["cand"], (base["cand"] * s).astype(dtype)), k


def test_probe_leaves_the_solve_state_untouched():
    P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(40, 60, 0.2, seed=1)
    st = cosmo_b200.Settings(accelerator="AndersonAccelerator", max_iter=60, eps_abs=1e-12, eps_rel=1e-12,
                             **V.variant("Type1", "RollingMemory", "NoRegularizer")).to_struct()
    tup = [cosmo_b200.model.set_tuple(S) for S in sets]
    one, two = E.Engine(P, q, A, b, tup, st), E.Engine(P, q, A, b, tup, st)
    for e in (one, two):
        e.set_accelerator(cosmo_b200.Settings(**V.variant("Type1", "RollingMemory", "NoRegularizer")).accelerator_struct())
    one.solve()
    two.solve()
    stats, w, rho = one.accelerator_stats(), one.w(), one.rho_vec()
    dim = one.n + one.m
    g, x = R.sequence(dim, 9, seed=2, rank=8)
    one.accelerator_probe(g, x, g[::-1].copy())
    assert one.accelerator_stats() == stats and stats["accepted"] > 0
    assert np.array_equal(one.w(), w) and np.array_equal(one.rho_vec(), rho)
    s1, s2 = one.solve(), two.solve()
    assert np.array_equal(s1.x, s2.x) and s1.iter == s2.iter and one.accelerator_stats() == two.accelerator_stats()


def test_report_worst_ratios():
    # runs last in this module: the worst |d eta| / bar of each path and type over the cases above
    import torch
    name = torch.cuda.get_device_name(0) if torch.cuda.is_available() else "?"
    for (path, dt), (ratio, kappa) in sorted(WORST.items()):
        print("worst |d eta| / bar: %-6s %-8s %.3e (kappa of the system %.1e) on %s" % (path, dt, ratio, kappa, name))
