"""Kernel parity of the infeasibility certificates (Engine<T>::primal_infeasible / dual_infeasible) against the
high-precision reference of tests/infeasibility_reference.py, through cosmo_b200_infeasibility_test and
cosmo_b200_psd_lambda_max, in fp64 and fp32.

Most cone tests use a "rig" whose gates are exact so that the cone kernels see exactly the vector v the test chose:
  * primal: A = 0, b = 0, delta_y = -2^s v  ->  A'dy = 0, the cone tests see -dy / |dy|_inf = v exactly;
  * dual: A = I, P = 0, q = -v, delta_x = 2^s v  ->  q'dx / |dx| = -|v|^2 / |v|_inf < -eps, P dx = 0, the cone tests
    see A dx / |dx|_inf = v exactly.
A leading Nonnegatives row holds -1, so |v|_inf = 1 and 1 / |delta| is a power of two.

Bars (u = 2^-53 in fp64, 2^-24 in fp32; every input is rounded to the engine's type first, see _round32):
  * |E dy|_inf, |D dx|_inf: bit-exact (one rounded product per entry, then a max);
  * SpMV-based gates: 1e-14 |M| |v| (fp64), 2 k u32 |M| |v| with k the longest row (fp32);
  * Box support sum: 1e-14 sum |terms| (fp64), m u32 sum |terms| (fp32); NaN where the reference is NaN;
  * lambda_max: 8 N u |X|_F, N the side that is diagonalized (2 Nc for a Hermitian cone).  Jacobi stops once every
    off-diagonal entry is below PsdEps<T> |X|_F = 2 u |X|_F, so the remaining off-diagonal part has 2-norm at most
    2 N u |X|_F and (Weyl) the largest diagonal entry is that close to lambda_max; the other 6 N u |X|_F cover the
    rounding of the rotations, which block Jacobi accumulates over more sweeps (measured on one H100 80GB HBM3: at
    most 66 u |X|_F on the shared-memory kernel, 855 u |X|_F = 3.3 N u |X|_F at N = 257 and 4.6 N u |X|_F at N = 97
    on block Jacobi);
  * verdicts: either verdict is accepted only where the reference margin is inside a band (SOC: (d + 2) u times the
    operands; PSD: the lambda_max bar; Exp/Pow: 32 u times the compared terms times (1 + |exponent argument|));
    outside it the verdict must equal the reference's.

The solve-level tests run the reference's InfeasibilityTests problems (tests/golden_problems.py) end to end.

Coverage is narrower than "everything" in places: lambda_max is checked at 18 sides between 1 and 257 (the small /
large boundary 96 / 97 included), not at every N; the CPU dry run executes a subset of these bodies against the
oracle stand-in (tests/test_gpu_tests_dryrun_cpu.py lists which).
"""
import math

import numpy as np
import pytest
import scipy.sparse as sp

import cosmo_b200
from cosmo_b200 import engine as E
from oracle import cosmo_oracle as O
from tests import golden_problems as G
from tests import infeasibility_reference as R
from tests.gpu_helpers import U32, U64, _psd_test_matrix, _round32
from tests.test_gpu_parity import _to_mine

pytestmark = pytest.mark.gpu
DTYPES = [np.float64, np.float32]
MEAS = {}


def _u(dtype):
    return U32 if np.dtype(dtype) == np.float32 else U64


def _cast(a, dtype):
    a = np.asarray(a, dtype=np.float64)
    return _round32(a) if np.dtype(dtype) == np.float32 else a


def _meas(key, val):
    MEAS[key] = max(MEAS.get(key, 0.0), float(val))
    print("MEAS %s %.3g" % (key, MEAS[key]))


def _settings(eps=2.0 ** -10, **kw):
    return cosmo_b200.Settings(eps_prim_inf=eps, eps_dual_inf=eps, scaling=0, **kw).to_struct()


class Rig:
    """engines whose gates are exact (module docstring); sets = engine tuples of the cones under test"""

    def __init__(self, sets, dtype=np.float64, eps=2.0 ** -10, **kw):
        self.sets = [(E.NONNEG, 1, None, None)] + list(sets)
        self.m = sum(int(t[1]) for t in self.sets)
        self.dtype, self.eps = dtype, eps
        st = _settings(eps, **kw)
        m = self.m
        self.pe = E.Engine(sp.csc_matrix((1, 1)), np.zeros(1), sp.csc_matrix((m, 1)), np.zeros(m), self.sets, st, dtype=dtype)
        self.de = E.Engine(sp.csc_matrix((m, m)), np.zeros(m), sp.identity(m, format="csc"), np.zeros(m), self.sets, st,
                           dtype=dtype)

    def full(self, v):
        v = _cast(v, self.dtype)
        assert v.size == self.m - 1 and np.max(np.abs(v), initial=0.0) <= 1.0
        return np.concatenate([[-1.0], v])

    def primal(self, v, s=0):
        return self.pe.infeasibility_test(0, -np.ldexp(self.full(v), s))

    def dual(self, v, s=0):
        vf = self.full(v)
        self.de.update_qb(q=-vf)
        return self.de.infeasibility_test(1, np.ldexp(vf, s))

    def lam(self, v):
        return self.pe.psd_lambda_max(self.full(v))

    def close(self):
        self.pe.close()
        self.de.close()


def _check_verdict(rec, fam, ok_ref, margin, band, where):
    got_ok = not (rec["families"] & fam)
    if abs(margin) > band:
        assert got_ok == ok_ref, (where, margin, band, rec)
    assert rec["gate"] == 4, (where, rec)


# ---- 1. gates, unscaled and scaled -----------------------------------------------------------------
def _gate_problem(dtype, rng, n=60, m=90):
    A = sp.random(m, n, 0.08, random_state=int(rng.integers(1 << 30)), format="lil")
    A[m - 10:, :] = 0                                     # ten empty rows: delta_y there has A'dy = 0
    A = sp.csc_matrix(A)
    A.data = _cast(A.data, dtype)
    B = sp.random(n, n, 0.05, random_state=int(rng.integers(1 << 30)))
    P = sp.csc_matrix(B @ B.T)
    P.data = _cast(P.data, dtype)
    q, b = _cast(rng.standard_normal(n), dtype), _cast(rng.standard_normal(m), dtype)
    return P, q, A, b


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("scaled", [False, True])
def test_gate_quantities_match_the_reference(dtype, scaled):
    rng = np.random.default_rng(11)
    P, q, A, b = _gate_problem(dtype, rng)
    m, n = A.shape
    D = _cast(rng.uniform(0.3, 3.0, n), dtype) if scaled else None
    Em = _cast(rng.uniform(0.3, 3.0, m), dtype) if scaled else None
    c = 0.7 if scaled else 1.0
    sets = [(E.NONNEG, m, None, None)]
    eng = E.Engine(P, q, A, b, sets, _settings(), D=D, E=Em, c=c, dtype=dtype)
    Dinv = None if D is None else _cast(1.0 / D, dtype)
    Einv = None if Em is None else _cast(1.0 / Em, dtype)
    u = _u(dtype)
    k = max(np.diff(sp.csc_matrix(A).indptr).max(), np.diff(sp.csr_matrix(P).indptr).max(), 16)
    bar = 1e-14 if dtype == np.float64 else 2 * k * u      # k: the longest row of A' and P, at least the depth of a reduction
    worst = 0.0
    for trial in range(6):
        dy = _cast(rng.standard_normal(m) * 10.0 ** rng.integers(-3, 4), dtype)
        got = eng.infeasibility_test(0, dy)
        ref = R.primal_gates(A, b, Em, Dinv, dy, 2.0 ** -10, dtype)
        assert got["norm"] == ref["norm"] and got["gate"] == ref["gate"] == 2, (got, ref)
        err = abs(got["gate2"] - ref["gate2"]) / ref["gate2_mag"]
        assert err <= bar, (trial, err, bar)
        worst = max(worst, err)
        dx = _cast(-q * 10.0 ** rng.integers(-2, 3) + 1e-3 * rng.standard_normal(n), dtype)
        got = eng.infeasibility_test(1, dx)
        ref = R.dual_gates(P, q, A, D, Dinv, Einv, c, dx, 2.0 ** -10, dtype)
        assert got["norm"] == ref["norm"] and got["gate"] == ref["gate"] >= 3, (got, ref)
        worst = max(worst, abs(got["gate2"] - ref["qdx"]) / ref["qdx_mag"], abs(got["gate3"] - ref["Pdx"]) / ref["Pdx_mag"])
        assert worst <= bar, (trial, worst, bar)
        # delta_y on the ten empty rows of A: A'dy = 0, the test reaches the cone tests and dy'b (b != 0)
        dy = np.zeros(m)
        dy[m - 10:] = _cast(rng.standard_normal(10), dtype)
        got = eng.infeasibility_test(0, dy)
        ref = R.primal_gates(A, b, Em, Dinv, dy, 2.0 ** -10, dtype)
        assert got["gate"] == ref["gate"] == 4 and got["gate2"] == ref["gate2"] == 0.0, (got, ref)
        err = abs(got["gate3"] - ref["dyt_b"]) / ref["dyt_b_mag"]
        assert err <= bar, (trial, err, bar, got, ref)
        worst = max(worst, err)
        cert = R.certificate(ref["v"], sets, 2.0 ** -10, primal=True)
        assert got["families"] == cert["families"] and got["verdict"] == int(cert["families"] == 0 and -ref["dyt_b"] <= 2.0 ** -10)
    _meas("gate_rel_err_%s_%s" % (np.dtype(dtype).name, "scaled" if scaled else "unscaled"), worst)
    eng.close()


@pytest.mark.parametrize("dtype", DTYPES)
def test_gates_reached_on_either_side_pin_E_D_and_c(dtype):
    """delta sits 2^-16 (relative) on either side of each gate; the gate reached must be the reference's.  E enters the
    primal norm, Dinv the A'dy gate, D the dual norm, c and D the q'dx and P dx gates, Einv the dual cone test (row 1
    lands at 1.5 tol with Einv and at 0.75 tol without it)."""
    n, m = 4, 4
    D = _cast([0.5, 2.0, 4.0, 0.25], dtype)
    Em = _cast([2.0, 0.5, 8.0, 1.0], dtype)
    c = 0.5
    eps = 2.0 ** -10
    A = sp.csc_matrix(np.diag(_cast([3.0, 1.5 * eps, 1.0, 1.0], dtype)))
    A = sp.csc_matrix(sp.vstack([A, sp.csc_matrix((1, n))]))       # row 4 is empty
    sets = [(E.NONNEG, m + 1, None, None)]
    f = 2.0 ** -16
    for side in (+1, -1):
        # primal: dy = (t, 0, 0, 0, 1): |E dy| = max(2 t, 1); gate 2 = |Dinv A'dy| = 3 t / 0.5 = 6 t
        t = _cast(eps / 6 * (1 + side * f), dtype)                # 2 t < 1: the norm is the empty row's 1
        P = sp.csc_matrix((n, n))
        eng = E.Engine(P, np.zeros(n), A, np.zeros(m + 1), sets, _settings(eps), D=D, E=np.append(Em, 1.0), c=c, dtype=dtype)
        got = eng.infeasibility_test(0, np.array([t, 0, 0, 0, 1.0]))
        assert got["norm"] == 1.0 and got["gate"] == (2 if side > 0 else 4), (side, got)
        # dual: dx = e_1 (D_1 = 2): norm 2; q'dx / (norm c) = q_1 / 1 -> gate 2 edge at q_1 = -eps
        q = np.zeros(n)
        q[1] = -eps * (1 - side * f)
        eng.update_qb(q=_cast(q, dtype))
        got = eng.infeasibility_test(1, np.array([0, 1.0, 0, 0]))
        assert got["norm"] == 2.0 and got["gate"] == (2 if side > 0 else 4), (side, got)   # P = 0 passes gate 3
        eng.close()
        # gate 3: P_11 = p: |Dinv P dx| / (norm c) = (p / 2) / 1 -> edge at p = 2 eps
        P = sp.csc_matrix(([2 * eps * (1 + side * f)], ([1], [1])), shape=(n, n))
        eng = E.Engine(P, _cast([0, -1.0, 0, 0], dtype), A, np.zeros(m + 1), sets, _settings(eps), D=D, E=np.append(Em, 1.0),
                       c=c, dtype=dtype)
        got = eng.infeasibility_test(1, np.array([0, 1.0, 0, 0]))
        assert got["gate"] == (3 if side > 0 else 4), (side, got)
        # the cone test of row 1 sees (Einv A dx / norm)_1 = 1.5 tol / 0.5 / 2 = 1.5 tol > tol (0.75 tol without Einv)
        if side < 0:
            assert got["families"] == E.FAMILY_ROWS, got
        eng.close()


# ---- 2. elementwise rows at the tolerance edge ---------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_rows_at_the_tolerance_edge(dtype):
    tol = 2.0 ** -10
    edge = [0.0, tol, -tol, np.nextafter(tol, 1), np.nextafter(tol, -1), -np.nextafter(tol, 1), 0.5, -0.5]
    if dtype == np.float32:
        edge = [0.0, tol, -tol, float(np.nextafter(np.float32(tol), np.float32(1))),
                float(np.nextafter(np.float32(tol), np.float32(0))), -float(np.nextafter(np.float32(tol), np.float32(1))), 0.5, -0.5]
    k = len(edge)
    l = np.array([-np.inf, -1.0, -2.0, -np.inf, 3.0, -1.0, -np.inf, -0.5])
    u = np.array([np.inf, 1.0, np.inf, 2.0, 3.0, np.inf, 4.0, 0.5])
    for typ in (E.ZERO, E.NONNEG, E.BOX):
        sets = [(typ, k, l if typ == E.BOX else None, u if typ == E.BOX else None)]
        rig = Rig(sets, dtype, tol)
        rs = [(R.BOX if typ == E.BOX else typ, k, l, u)]
        for perm in range(12):
            v = np.roll(edge, perm) if perm < k else np.random.default_rng(perm).permutation(edge)
            for which in (0, 1):
                got = rig.primal(v) if which == 0 else rig.dual(v)
                ref = R.certificate(v, rs, tol, primal=(which == 0))
                assert got["families"] == ref["families"], (typ, which, v, got, ref)
                if which == 0 and typ == E.BOX:
                    if math.isnan(ref["box_sum"]):
                        assert math.isnan(got["box_sum"]), (v, got)
                    elif math.isinf(ref["box_sum"]):
                        assert got["box_sum"] == ref["box_sum"], (v, got, ref)
                    else:
                        bar = 1e-14 if dtype == np.float64 else k * U32
                        assert abs(got["box_sum"] - ref["box_sum"]) <= bar * ref["box_mag"], (v, got, ref)
                    want = int(ref["families"] == 0 and ref["box_sum"] <= tol)
                    assert got["verdict"] == want, (v, got, ref)
        rig.close()


# ---- 3. second-order cones ---------------------------------------------------------------------
def _soc_point(d, margin_rel, rng, tol):
    t = rng.standard_normal(d - 1) if d > 1 else np.zeros(0)
    if d > 1:
        t /= 2 * np.linalg.norm(t)
    nrm = float(np.linalg.norm(t))
    v0 = tol - nrm * (1 + margin_rel) if d > 1 else tol - margin_rel      # margin = tol - v0 - nrm = nrm margin_rel
    return np.concatenate([[v0], t])


@pytest.mark.parametrize("dtype", DTYPES)
def test_soc_margins_dimensions_and_scale(dtype):
    tol = 2.0 ** -10
    u = _u(dtype)
    rng = np.random.default_rng(3)
    dims = [1, 2, 3, 4097, 8192, 8193]
    rig = Rig([(E.SOC, d, None, None) for d in dims], dtype, tol)
    smax = 900 if dtype == np.float64 else 100
    for k in range(1, 51, 3):
        for sign in (+1, -1):
            pts = [_soc_point(d, sign * 2.0 ** -k, rng, tol) for d in dims]
            for j, d in enumerate(dims):                       # one cone under test, the others well inside
                v = [pt if i == j else _soc_point(dd, 0.5, rng, tol) for i, (pt, dd) in enumerate(zip(pts, dims))]
                v = np.concatenate(v)
                vr = _cast(v, dtype)
                off = sum(dims[:j])
                ok, margin, nrm = R.soc_cert(vr[off:off + d], tol)
                band = (d + 2) * u * (nrm + abs(tol - vr[off]))
                for which in (0, 1):
                    first = None
                    for s in ((0, smax, 5 - smax // 100) if k % 9 == 1 else (0,)):
                        got = rig.primal(vr, s) if which == 0 else rig.dual(vr, s)
                        _check_verdict(got, E.FAMILY_SOC, ok, margin, band, (d, k, sign, which, s))
                        first = got["families"] if first is None else first
                        assert got["families"] == first, (d, k, sign, which, s)   # a power-of-two scaling is exact
                    # scaled below the tolerance the norm gate stops the test before any cone is looked at
                    got = rig.primal(vr, -smax) if which == 0 else rig.dual(vr, -smax)
                    assert got["gate"] == 1 and got["verdict"] == 0
    rig.close()


@pytest.mark.parametrize("dtype", DTYPES)
def test_soc_exact_boundary_points_are_certified(dtype):
    """|v[2:]| = tol - v[1] exactly (Pythagorean tails, scaled by powers of two): the reference certifies (<=)"""
    tol = 0.25
    rig = Rig([(E.SOC, 3, None, None), (E.SOC, 3, None, None)], dtype, tol)
    for e in range(0, 8):
        f = 2.0 ** -e
        v = np.array([tol - 5 * f / 8, 3 * f / 8, 4 * f / 8, tol - 13 * f / 16, 5 * f / 16, 12 * f / 16])
        for which in (0, 1):
            got = rig.primal(v) if which == 0 else rig.dual(v)
            assert got["families"] == 0 and got["verdict"] == 1, (e, which, got)
    # the issue's example: (-4.75, 3, 4) has tail norm 5 = tol - v0 (scaled into |v| <= 1)
    v = np.array([-4.75, 3.0, 4.0, -1.0, 0.0, 0.0]) / 8
    rig2 = Rig([(E.SOC, 3, None, None), (E.SOC, 3, None, None)], dtype, tol / 8)
    assert rig2.primal(v)["families"] == 0 and rig2.dual(v)["families"] == 0
    rig.close()
    rig2.close()


@pytest.mark.parametrize("dtype", DTYPES)
def test_soc_20000_with_an_all_zero_chunk(dtype):
    tol = 2.0 ** -10
    rng = np.random.default_rng(4)
    d = 20000
    rig = Rig([(E.SOC, d, None, None)], dtype, tol)
    for sign in (+1, -1):
        t = rng.standard_normal(d - 1) * 0.005
        t[8191:16383] = 0.0
        v0 = tol - np.linalg.norm(t) * (1 - sign * 2.0 ** -20)
        v = _cast(np.concatenate([[v0], t]), dtype)
        ok, margin, nrm = R.soc_cert(v, tol)
        band = (d + 2) * _u(dtype) * (nrm + abs(tol - v[0]))
        for which in (0, 1):
            got = rig.primal(v) if which == 0 else rig.dual(v)
            _check_verdict(got, E.FAMILY_SOC, ok, margin, band, (sign, which))
    rig.close()


# ---- 4. PSD lambda_max through the hook --------------------------------------------------------------
def _psd_vec(X, typ):
    N = X.shape[0]
    if typ == E.PSD_SQUARE:
        return X.reshape(-1, order="F")
    if typ == E.PSD_TRIANGLE:
        return np.concatenate([np.concatenate([X[:j, j] * math.sqrt(2.0), [X[j, j]]]) for j in range(N)])
    raise ValueError(typ)


def _lam_bar(N, X, dtype):
    return 8 * N * _u(dtype) * np.linalg.norm(X)


def _lam_case(typ, N, kind, rng):
    if typ == E.PSD_TRIANGLE_COMPLEX:
        Z = rng.standard_normal((N, N)) + 1j * rng.standard_normal((N, N))
        H = (Z + Z.conj().T) / 2
        from oracle.cosmo_oracle import extract_upper_triangle_complex
        return extract_upper_triangle_complex(H, math.sqrt(2.0)), N * N
    if kind == "cluster":
        Q, _ = np.linalg.qr(rng.standard_normal((N, N)))
        lam = np.concatenate([[1.0, 1.0 - 1e-12], rng.uniform(-1, 0.9, N - 2)])[:N]
        X = (Q * lam) @ Q.T
    else:
        X = _psd_test_matrix(kind, N, rng)
    X = (X + X.T) / 2
    if typ == E.PSD_SQUARE:   # a non-symmetric input: the lower triangle must not matter
        X = np.triu(X) + np.tril(rng.standard_normal((N, N)), -1)
    x = _psd_vec(X, typ)
    return x, x.size


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("typ", [E.PSD_TRIANGLE, E.PSD_SQUARE, E.PSD_TRIANGLE_COMPLEX])
def test_psd_lambda_max_small_and_large_paths(dtype, typ):
    rng = np.random.default_rng(20 + typ)
    if typ == E.PSD_TRIANGLE_COMPLEX:
        sizes = [1, 2, 3, 7, 16, 31, 48, 60]
    else:
        sizes = [1, 2, 3, 4, 5, 8, 13, 17, 31, 32, 33, 47, 64, 95, 96, 97, 150, 257]
    kinds = ["wigner", "graded", "rank_deficient", "cluster"]
    worst = {}
    for N in sizes:
        kind = kinds[N % len(kinds)] if N >= 4 else "wigner"
        x, dim = _lam_case(typ, N, kind, rng)
        x = _cast(x / np.max(np.abs(x)), dtype)
        rig = Rig([(typ, dim, None, None)], dtype)
        lam = rig.lam(x)
        ref_X = R.psd_matrix(x, typ)
        lam_ref = R.lambda_max(ref_X)
        side = 2 * N if (typ == E.PSD_TRIANGLE_COMPLEX and N > 1) else N
        err = abs(lam[0] - lam_ref)
        bar = _lam_bar(side, ref_X, dtype)
        assert err <= bar, (N, kind, lam[0], lam_ref, err, bar)
        path = "large" if side > 96 else "small"
        worst[path] = max(worst.get(path, 0.0), err / (_u(dtype) * np.linalg.norm(ref_X)))
        rig.close()
    for path, w in worst.items():
        _meas("lammax_err_in_u_fro_%s_%s_%s" % (np.dtype(dtype).name, typ, path), w)


@pytest.mark.parametrize("dtype", DTYPES)
def test_psd_lambda_max_homogeneity_ladder(dtype):
    """lambda_max(2^k v) = 2^k lambda_max(v) exactly: the prescaling by a power of two is exact on both paths"""
    rng = np.random.default_rng(31)
    ks = range(-1000, 901, 100) if dtype == np.float64 else range(-100, 101, 20)
    for N, typ in ((12, E.PSD_TRIANGLE), (6, E.PSD_SQUARE), (110, E.PSD_TRIANGLE)):
        x, dim = _lam_case(typ, N, "wigner", rng)
        x = _cast(x / np.max(np.abs(x)), dtype)
        sets = [(typ, dim, None, None)]
        st = _settings()
        eng = E.Engine(sp.csc_matrix((1, 1)), np.zeros(1), sp.csc_matrix((dim, 1)), np.zeros(dim), sets, st, dtype=dtype)
        base = eng.psd_lambda_max(x)[0]
        smallest = float(np.min(np.abs(x[x != 0]))) / 2       # a triangle's off-diagonal entries are multiplied by 1/sqrt 2
        tested = 0
        for k in ks:
            if math.ldexp(smallest, k) < np.finfo(dtype).tiny:
                continue                                      # subnormal inputs are not exact under scaling
            got = eng.psd_lambda_max(np.ldexp(x, k))[0]
            assert got == math.ldexp(base, k), (N, k, got, math.ldexp(base, k))
            tested += 1
        assert tested >= len(ks) - 2
        eng.close()


# ---- 5. PSD verdicts ---------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_psd_verdicts_at_the_tolerance(dtype):
    tol = 2.0 ** -10
    rng = np.random.default_rng(40)
    for N, typ in ((5, E.PSD_TRIANGLE), (4, E.PSD_SQUARE), (40, E.PSD_TRIANGLE), (100, E.PSD_TRIANGLE)):
        B = rng.standard_normal((N, N))
        X0 = (B + B.T) / 2
        X0 /= 2 * np.max(np.abs(np.linalg.eigvalsh(X0)))
        lam0 = np.linalg.eigvalsh(X0)[-1]
        x0 = _psd_vec(X0, typ)
        rig = Rig([(typ, x0.size, None, None)], dtype, tol)
        for k in range(1, 51, 4):
            for sign in (+1, -1):
                X = X0 + (tol * (1 + sign * 2.0 ** -k) - lam0) * np.eye(N)
                x = _cast(_psd_vec(X, typ), dtype)
                ok, margin, lam_ref, fro = R.psd_cert(x, typ, tol)
                for which in (0, 1):
                    got = rig.primal(x) if which == 0 else rig.dual(x)
                    _check_verdict(got, E.FAMILY_PSD, ok, margin, _lam_bar(N, R.psd_matrix(x, typ), dtype), (N, k, sign, which))
        rig.close()


def _nonsymmetric_square(N, flip, rng):
    """a square cone whose upper reflection and symmetrized matrix give opposite certificates at tol = 1/4 (the
    all-ones vector bounds lambda_max from below)"""
    L = np.tril(rng.uniform(0.9, 1.0, (N, N)), -1)
    X = -0.125 * np.eye(N)
    if flip:
        X = X + L.T - L           # upper reflection -I/8 + L + L.T: lambda_max >= -1/8 + 0.9 (N - 1); symmetrized -I/8
    else:
        X = X + L                 # upper reflection -I/8; symmetrized -I/8 + (L + L.T) / 2: lambda_max >= -1/8 + 0.45 (N - 1)
    return X.reshape(-1, order="F")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("N", [2, 9, 96, 97, 130])
def test_nonsymmetric_square_psd_certificate_reads_the_upper_triangle(dtype, N):
    tol = 0.25
    rng = np.random.default_rng(50 + N)
    for flip in (False, True):
        x = _cast(_nonsymmetric_square(N, flip, rng), dtype)
        ok, margin, lam_ref, _ = R.psd_cert(x, R.PSD_SQUARE, tol)
        Xs = x.reshape(N, N, order="F")
        lam_sym = np.linalg.eigvalsh((Xs + Xs.T) / 2)[-1]
        assert ok == (not flip) and (lam_sym < tol) == flip       # the two readings disagree
        rig = Rig([(E.PSD_SQUARE, N * N, None, None)], dtype, tol)
        lam = rig.lam(x)[0]
        assert abs(lam - lam_ref) <= _lam_bar(N, R.psd_matrix(x, R.PSD_SQUARE), dtype), (flip, lam, lam_ref, lam_sym)
        for which in (0, 1):
            got = rig.primal(x) if which == 0 else rig.dual(x)
            assert bool(got["families"] & E.FAMILY_PSD) == (not ok), (flip, which, got)
            assert got["verdict"] == int(ok), (flip, which, got)
        rig.close()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("N", [40, 150])
def test_unconverged_eigensolver_is_not_certified(N, dtype):
    """psd_max_sweeps = 1 on a matrix that needs more sweeps: the certificate says "not certified" and counts it,
    instead of ending the solve with an error; with the default cap the same point is certified"""
    rng = np.random.default_rng(60)
    B = rng.standard_normal((N, N))
    X = -np.eye(N) + 0.05 * (B + B.T) / np.sqrt(N)
    x = _psd_vec(X, E.PSD_TRIANGLE)
    x /= np.max(np.abs(x))
    for sweeps, certified in ((1, False), (30, True)):
        rig = Rig([(E.PSD_TRIANGLE, x.size, None, None)], dtype, 2.0 ** -10, psd_max_sweeps=sweeps)
        for which in (0, 1):
            got = rig.primal(x) if which == 0 else rig.dual(x)
            assert got["verdict"] == int(certified) and got["psd_unconverged"] == (0 if certified else 1), (sweeps, which, got)
        lam = rig.lam(x)[0]
        assert (lam == math.inf) == (not certified)
        rig.close()


# ---- 6. exponential / power cones --------------------------------------------------------------
def _c3_mag(typ, v, a):
    x, y, z = -v[0], -v[1], -v[2]
    with np.errstate(all="ignore"):
        if typ == E.EXP:
            arg = y / x if x != 0 else 0.0
            return (abs(x * math.exp(min(arg, 700))) + math.e * abs(z)) * (1 + abs(arg))
        if typ == E.DUAL_EXP:
            arg = x / y if y != 0 else 0.0
            return (abs(y * math.exp(min(arg, 700))) + abs(z)) * (1 + abs(arg))
        return abs(x) + abs(y) + abs(z)


def _c3_boundary_points(typ, a, rng):
    """points w on the boundary of the set that in_dual(-v) tests (w = -v), |w| <= 0.7"""
    ca = a ** a * (1 - a) ** (1 - a) if typ == E.POW else 1.0
    pts = []
    while len(pts) < 6:
        p, r = rng.uniform(0.1, 0.9), rng.uniform(-0.9, 0.9)
        if typ == E.EXP:          # K_exp*: -x e^(y/x) = e z, x < 0
            w = [-p, r, p * math.exp(-r / p) / math.e]
        elif typ == E.DUAL_EXP:   # K_exp: y e^(x/y) = z
            w = [r, p, p * math.exp(r / p)]
        elif typ == E.POW:        # K_pow*: s^a t^(1-a) = |w| a^a (1-a)^(1-a)
            t = rng.uniform(0.1, 0.9)
            w = [p, t, p ** a * t ** (1 - a) / ca * np.sign(r)]
        else:                     # K_pow: x^a y^(1-a) = |z|
            t = rng.uniform(0.1, 0.9)
            w = [p, t, p ** a * t ** (1 - a) * np.sign(r)]
        if np.max(np.abs(w)) <= 0.7:            # room for the shift of _c3_shift (at most tol + 1/8 / a^a (1-a)^(1-a))
            pts.append(np.array(w))
    return pts


def _c3_shift(typ, w, a, tol, delta):
    """move the boundary point w so that the reference's margin becomes delta (up to rounding)"""
    w = w.copy()
    if typ == E.EXP:              # margin = tol - (-x e^(y/x) - e z)
        w[2] += (delta - tol) / math.e
    elif typ == E.DUAL_EXP:       # margin = z + tol - y e^(x/y)
        w[2] += delta - tol
    elif typ == E.POW:            # margin = s^a t^(1-a) - |w| a^a (1-a)^(1-a) + tol
        w[2] = np.sign(w[2] or 1.0) * (abs(w[2]) + (tol - delta) / (a ** a * (1 - a) ** (1 - a)))
    else:                         # margin = x^a y^(1-a) - |z| + tol
        w[2] = np.sign(w[2] or 1.0) * (abs(w[2]) + tol - delta)
    return w


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("typ,a", [(E.EXP, 0.0), (E.DUAL_EXP, 0.0), (E.POW, 0.01), (E.POW, 0.3), (E.POW, 0.5),
                                   (E.POW, 0.99), (E.DUAL_POW, 0.3), (E.DUAL_POW, 0.99)])
def test_exp_pow_verdicts_near_the_boundary(dtype, typ, a):
    tol = 2.0 ** -10
    rng = np.random.default_rng(70 + typ)
    extra = {"alpha": a} if typ in (E.POW, E.DUAL_POW) else None
    rig = Rig([(typ, 3, None, None, extra)], dtype, tol)
    rtyp = {E.EXP: R.EXP, E.DUAL_EXP: R.DUAL_EXP, E.POW: R.POW, E.DUAL_POW: R.DUAL_POW}[typ]
    pts = [_c3_shift(typ, w, a, tol, sign * 2.0 ** -k) for w in _c3_boundary_points(typ, a, rng)
           for k in (3, 5, 10, 16, 20, 30, 45) for sign in (+1, -1)]
    if typ == E.EXP:              # x -> 0-: the edge between the two disjuncts of K_exp*
        pts += [np.array([-2.0 ** -e, 0.3, z]) for e in (8, 9, 10, 11, 12, 20, 40, 60) for z in (0.2, -tol, -2 * tol)]
    if typ == E.POW:              # the negative-base band of pow_in_dual: "not in the cone"
        pts += [np.array([s, 0.5, 0.0]) for s in (-tol / 2, -tol, -2 * tol)] + [np.array([0.5, s, 0.1]) for s in (-tol / 4, -tol)]
    worst_band = 0.0
    for w in pts:
        v = _cast(-w, dtype)
        ok, margin = R.c3_cert(v, rtyp, tol, a)
        band = 32 * _u(dtype) * (_c3_mag(typ, v, a) + tol)
        if abs(margin) <= band:
            worst_band = max(worst_band, abs(margin))
        for which in (0, 1):
            got = rig.primal(v) if which == 0 else rig.dual(v)
            _check_verdict(got, E.FAMILY_C3, ok, margin, band, (w, which))
    _meas("c3_in_band_margin_%s_%d" % (np.dtype(dtype).name, typ), worst_band)
    rig.close()


# ---- 7. one engine with every family ------------------------------------------------------------------
COMPOSITE_SETS = [(E.NONNEG, 3, None, None), (E.BOX, 3, np.array([-1.0, -2.0, -3.0]), np.array([1.0, np.inf, 3.0])),
                  (E.SOC, 3, None, None), (E.PSD_SQUARE, 9, None, None), (E.PSD_TRIANGLE, 6, None, None),
                  (E.PSD_TRIANGLE_COMPLEX, 4, None, None), (E.PSD_TRIANGLE, 5050, None, None),
                  (E.EXP, 3, None, None), (E.DUAL_EXP, 3, None, None), (E.POW, 3, None, None, {"alpha": 0.3}),
                  (E.DUAL_POW, 3, None, None, {"alpha": 0.6})]


def _composite_cases():
    """{name: (v, failing families)}: a base point inside every certificate, and for each family a point where only
    that family's cone fails"""
    tri100 = np.concatenate([np.concatenate([np.zeros(j), [-0.5]]) for j in range(100)])
    base = [np.full(3, -0.5), np.zeros(3), np.array([-1.0, 0.3, 0.4]), (-0.5 * np.eye(3)).reshape(-1),
            np.array([-0.5, 0, -0.5, 0, 0, -0.5]), np.array([-0.5, 0, -0.5, 0.0]), tri100,
            np.array([0.5, 0.0, -1.0]), np.array([0.0, -0.5, -1.0]), np.array([-0.5, -0.5, 0.0]), np.array([-0.5, -0.5, 0.0])]
    bad = {0: (np.array([-0.5, 0.5, -0.5]), E.FAMILY_ROWS), 2: (np.array([1.0, 0.3, 0.4]), E.FAMILY_SOC),
           3: (np.array([-0.5, 0, 0, 0, 0.5, 0, 0, 0, -0.5]), E.FAMILY_PSD), 4: (np.array([-0.5, 0, 0.5, 0, 0, -0.5]), E.FAMILY_PSD),
           5: (np.array([-0.5, 0, 0.5, 0.0]), E.FAMILY_PSD), 6: (-tri100, E.FAMILY_PSD),
           7: (np.array([-0.5, 0.0, -1.0]), E.FAMILY_C3), 8: (np.array([0.0, 0.5, -1.0]), E.FAMILY_C3),
           9: (np.array([0.5, -0.5, 0.0]), E.FAMILY_C3), 10: (np.array([-0.5, 0.5, 0.0]), E.FAMILY_C3)}
    cases = {"none": (np.concatenate(base), 0)}
    for i, (vb, fam) in bad.items():
        parts = list(base)
        parts[i] = vb
        cases["set%d" % i] = (np.concatenate(parts), fam)
    allbad = list(base)
    for i, (vb, _) in bad.items():
        allbad[i] = vb
    cases["all"] = (np.concatenate(allbad), E.FAMILY_ROWS | E.FAMILY_SOC | E.FAMILY_PSD | E.FAMILY_C3)
    return cases


@pytest.mark.parametrize("dtype", DTYPES)
def test_composite_bitmask_names_exactly_the_failing_family(dtype):
    tol = 2.0 ** -10
    rig = Rig(COMPOSITE_SETS, dtype, tol)
    rsets = [(t[0], t[1], t[2], t[3], t[4] if len(t) > 4 else None) for t in COMPOSITE_SETS]
    for name, (v, fam) in _composite_cases().items():
        for which in (0, 1):
            ref = R.certificate(v, rsets, tol, primal=(which == 0))
            assert ref["families"] == fam, (name, which, ref)
            got = rig.primal(v) if which == 0 else rig.dual(v)
            assert got["families"] == fam, (name, which, got)
            want = int(fam == 0 and (which == 1 or ref["box_sum"] <= tol))
            assert got["verdict"] == want, (name, which, got)
    rig.close()


# ---- 8. the reference's infeasible problems, end to end ---------------------------------------------------------
def _solve_cases():
    out = []
    for name, builder, expected in G.INFEASIBILITY_PROBLEMS:
        for acc in ("EmptyAccelerator", "AndersonAccelerator"):
            if acc == "AndersonAccelerator" and name.endswith("large_psd"):
                continue          # the oracle does not decide it with acceleration (tests/golden_problems.py)
            for scaling in (0, 10):
                out.append(((builder, expected, acc, scaling), "%s-%s-%d" % (name, acc[:-11], scaling)))
    return out


SOLVE_CASES = _solve_cases()


def _solve(builder, dtype=np.float64, **kw):
    P, q, cons = builder()
    model = cosmo_b200.Model(dtype=dtype)
    cosmo_b200.assemble(model, P, q, _to_mine(cons), cosmo_b200.Settings(max_iter=10000, eps_abs=1e-5, eps_rel=1e-5, **kw))
    return cosmo_b200.optimize(model)


def _solve_oracle(builder, acc, scaling, rel_q=0.0, rel_b=0.0):
    P, q, cons = builder()
    Pm, qm, A, b, cones = O.assemble(P, q, cons)
    return O.solve(Pm, qm * (1.0 + rel_q), A, b * (1.0 + rel_b), cones,
                   O.Settings(kkt_solver="cg", max_iter=10000, eps_abs=1e-5, eps_rel=1e-5, scaling=scaling,
                              accelerator="anderson" if acc == "AndersonAccelerator" else "empty"))


# On these diverging problems the iteration at which a check first certifies infeasibility is not a continuous function
# of the data: the oracle itself moves primal_infeasible_3 (EmptyAccelerator, scaling 0) from 641 to 3481 iterations
# when q is multiplied by 1 + 1e-15, and dual_infeasible_1 with AndersonAccelerator from Dual_infeasible at 57 to
# Max_iter_reached at 1 + 2e-15; primal_infeasible_2 (EmptyAccelerator, scaling 0) is stable under perturbations of q
# but moves from 441 to 401 when b is multiplied by 1 - 1e-15.  So the oracle is run on the data and on q (1 +- 1e-15),
# b (1 +- 1e-15), b (1 +- 2e-15): where all seven runs agree, the engine must reproduce status and iteration count
# exactly; elsewhere its status must be one the oracle reaches on those rounding-level perturbations.
_PERTURB = ((0.0, 0.0), (1e-15, 0.0), (-1e-15, 0.0), (0.0, 1e-15), (0.0, -1e-15), (0.0, 2e-15), (0.0, -2e-15))


@pytest.mark.parametrize("builder,expected,acc,scaling", [c for c, _ in SOLVE_CASES], ids=[i for _, i in SOLVE_CASES])
def test_reference_infeasible_problems_status_and_iterations(builder, expected, acc, scaling):
    """status (and, where the oracle's is stable, iteration count) of the oracle on the same data, and the status
    the reference's file asserts"""
    res = _solve(builder, accelerator=acc, scaling=scaling)
    refs = [(r.status, r.iter) for r in (_solve_oracle(builder, acc, scaling, eq, eb) for eq, eb in _PERTURB)]
    print("MEAS solve engine %s/%d oracle %s" % (res.status, res.iter, refs))
    assert any(st in expected for st, _ in refs), refs
    if len(set(refs)) == 1:
        assert (res.status, res.iter) == refs[0] and res.status in expected, (res.status, res.iter, refs)
    else:
        assert res.status in {st for st, _ in refs}, (res.status, res.iter, refs)


# measured on one H100 80GB HBM3: the fp32 engine reaches max_iter = 10000 on every primal-infeasible problem here
_FP32_PRIMAL_STALL = pytest.mark.xfail(strict=True, reason="known: the fp32 engine reaches Max_iter_reached (10000) where the "
                                                          "fp64 oracle reaches Primal_infeasible; not investigated yet")


@pytest.mark.parametrize("name,builder,expected",
                         [pytest.param(*g, marks=_FP32_PRIMAL_STALL) if g[0].startswith("primal_infeasible_")
                          and g[0] != "primal_infeasible_1" else g for g in G.INFEASIBILITY_PROBLEMS],
                         ids=[g[0] for g in G.INFEASIBILITY_PROBLEMS])
def test_reference_infeasible_problems_float32(name, builder, expected):
    """the fp32 engine reaches the infeasible status the fp64 oracle reaches (default scaling, no acceleration)"""
    ref = _solve_oracle(builder, "EmptyAccelerator", 10)
    res = _solve(builder, dtype=np.float32)
    assert ref.status in expected and res.status == ref.status, (name, res.status, ref.status, res.iter, ref.iter)
