"""Kernel parity tests for the device Ruiz equilibration (csrc/ruiz.cuh, Engine<T>::equilibrate) against the
extended-precision restatement of scale_ruiz! (tests/ruiz_reference.py), in fp64 and fp32.

Every result is read through the engine's existing readers: D, E, c from scaling(); the scaled A, A' and P entry by
entry as spmv(which, e_j) on unit vectors (a product with a unit vector is exact on every layout); b and q through the
residuals at chosen points; the scaled Box bounds as the projection of +-inf; the row classes through rho_vec().

Bars, from the arithmetic: the device takes weighted maxima of the unscaled data where the reference rescales the data on
every pass, so D, E and c differ from the restatement by reordered products only: 4 * scaling * u.  A scaled entry is
the data times c (D_i D_j) or E_i D_j, a few roundings more plus the error carried in D, E and c: 4 u + 3 times that
(_bars).  Each case prints its worst measured values next to the bars."""
import numpy as np
import pytest
import scipy.sparse as sp

import cosmo_b200
from cosmo_b200 import engine as E
from oracle import cosmo_oracle as O
from tests import ruiz_reference as R
from tests.gpu_helpers import U32, U64, _tuples

pytestmark = pytest.mark.gpu

DTYPES = [np.float64, np.float32]


def _u(dtype):
    return U64 if np.dtype(dtype) == np.float64 else U32


def _bars(dtype, scaling):
    scal = 4 * max(scaling, 1) * _u(dtype)
    return scal, 4 * _u(dtype) + 3 * scal


def _as_dtype(P, q, A, b, sets, dtype):
    """the data as an engine of `dtype` holds them (fp32: every value rounded once), in float64 arrays"""
    r = lambda a: np.asarray(a, dtype=np.float64).astype(dtype).astype(np.float64)
    P, A = sp.csc_matrix(P, copy=True), sp.csc_matrix(A, copy=True)
    P.sort_indices()
    A.sort_indices()
    P.data, A.data = r(P.data), r(A.data)
    sets = [cosmo_b200.Box(r(S.l), r(S.u)) if isinstance(S, cosmo_b200.Box) else S for S in sets]
    return P, r(q), A, r(b), sets


def _setup(P, q, A, b, sets, dtype, scaling=10):
    """(device engine, reference) for the data as `dtype` holds them"""
    P, q, A, b, sets = _as_dtype(P, q, A, b, sets, dtype)
    st = cosmo_b200.Settings(scaling=scaling).to_struct()
    eng = E.Engine(P, q, A, b, _tuples(sets), st, dtype=dtype, equilibrate=True)
    ref = R.scale_ruiz_ld(P, q, A, b, R.sets_to_oracle(sets), scaling=scaling, dtype=dtype)
    return eng, ref


def _read(eng, which, cols=None):
    """the columns `cols` (default all, in that order) of the resident scaled matrix, one unit vector each:
    0 -> A, 1 -> A', 2 -> P"""
    k = eng.m if which == 1 else eng.n
    cols = range(k) if cols is None else cols
    out = np.zeros((eng.m if which == 0 else eng.n, len(cols)), dtype=eng.dtype)
    e = np.zeros(k, dtype=eng.dtype)
    for t, j in enumerate(cols):
        e[j] = 1
        out[:, t] = eng.spmv(which, e)
        e[j] = 0
    return out


def _asymmetric_pairs(Pd):
    iu = np.triu_indices(Pd.shape[0], 1)
    return int(np.count_nonzero(Pd[iu] != Pd.T[iu])), iu[0].size


def _box_bounds(eng, sets):
    """the scaled Box bounds: Pi(+inf) and Pi(-inf) on the Box rows (0 on the others, which any cone accepts)"""
    box = np.zeros(eng.m, dtype=bool)
    off = 0
    for S in sets:
        box[off:off + S.dim] = isinstance(S, cosmo_b200.Box)
        off += S.dim
    w = np.where(box, np.inf, 0.0)
    return box, eng.project(-w)[box].astype(np.float64), eng.project(w)[box].astype(np.float64)


def _rho_classes(eng, st):
    """the class behind every entry of rho_vec (parameters.jl:17-49): 0 rho, 1 rho * RHO_EQ_OVER_RHO_INEQ, 2 RHO_MIN"""
    rv = eng.rho_vec().astype(np.float64)
    vals = np.array([st.rho, st.rho * st.RHO_EQ_OVER_RHO_INEQ, st.RHO_MIN])
    cls = np.argmin(np.abs(rv[:, None] - vals[None, :]) / vals[None, :], axis=1)
    assert np.allclose(rv, vals[cls], rtol=1e-6)
    return cls


def _ref_rho_classes(ref, sets, dtype, st):
    """classify_constraints! (setup.jl:75-85) on the reference's scaled b and Box bounds, rounded to the engine's type"""
    r = lambda a: np.asarray(a, dtype=np.float64).astype(dtype).astype(np.float64)
    big = st.COSMO_INFTY * st.MIN_SCALING
    b, l, u = r(ref.b), r(ref.l), r(ref.u)
    cls = np.zeros(ref.shape[0], dtype=int)
    off = 0
    for S in sets:
        s = slice(off, off + S.dim)
        if isinstance(S, cosmo_b200.ZeroSet):
            cls[s] = 1
        elif isinstance(S, cosmo_b200.Nonnegatives):
            cls[s] = np.where(b[s] > big, 2, 0)
        elif isinstance(S, cosmo_b200.Box):
            with np.errstate(invalid="ignore"):
                cls[s] = np.where((l[s] < -big) & (u[s] > big), 2, np.where(u[s] - l[s] < st.RHO_TOL, 1, 0))
        off += S.dim
    return cls


def _check(eng, ref, sets, dtype, scaling, label, read=True):
    """D, E, c, the scaled entries of A, A' and P (read=True), b, q, the Box bounds and the row classes against the
    reference; the read P must be exactly symmetric.  Returns the measured worst values."""
    D, Ev, c = eng.scaling()
    scal_bar, entry_bar = _bars(dtype, scaling)
    m, n = ref.shape
    errs = {"D": R.rel_err(D, ref.D), "E": R.rel_err(Ev, ref.E), "c": R.rel_err([c], [ref.c])}
    if read:
        Ad = R.dense(ref.A, (m, n))
        Pd = _read(eng, 2)
        errs.update(A=R.rel_err(_read(eng, 0), Ad), At=R.rel_err(_read(eng, 1), Ad.T), P=R.rel_err(Pd, R.dense(ref.P, (n, n))))
        asym, pairs = _asymmetric_pairs(Pd)
        assert asym == 0, "%s: %d of %d off-diagonal pairs of the scaled P are not symmetric" % (label, asym, pairs)
    # b: r_prim at x = 0, mu = 0, s = the reference's b is max_i |b_ref,i - b_i|; max_norm_prim at s = 0 is |b|_inf
    bref = np.asarray(ref.b, dtype=np.float64)
    zn, zm = np.zeros(n), np.zeros(m)
    r_b = eng.residuals(zn, bref, zm, ignore_scaling=True)
    r_0 = eng.residuals(zn, zm, zm, ignore_scaling=True)
    bmax = float(np.max(np.abs(bref))) if m else 0.0
    errs["b"] = r_b[0] / bmax if bmax else r_b[0]
    errs["|b|"] = abs(r_0[2] - bmax) / bmax if bmax else r_0[2]
    # q: r_dual at x = 0, mu = 0 is |q|_inf; the cost at a random x is (1/c)(x'Px / 2 + q'x)
    qmax = float(np.max(np.abs(ref.q))) if n else 0.0
    errs["|q|"] = abs(r_0[1] - qmax) / qmax if qmax else r_0[1]
    if read:
        x = np.random.default_rng(0).standard_normal(n).astype(dtype).astype(np.float64)
        Pref = R.dense(ref.P, (n, n))
        xl = x.astype(R.LD)
        want = (xl @ Pref @ xl / 2 + ref.q @ xl) / ref.c
        size = (np.abs(xl) @ np.abs(Pref) @ np.abs(xl) / 2 + np.abs(ref.q) @ np.abs(xl)) / ref.c
        cost = R.LD(eng.residuals(x, zm, zm, ignore_scaling=True)[4])
        errs["cost"] = float(abs(cost - want) / size) if size else 0.0
    box = ~np.isnan(ref.l)
    if box.any():
        _, lo, up = _box_bounds(eng, sets)
        for key, got, want in (("l", lo, ref.l[box]), ("u", up, ref.u[box])):
            inf = np.isinf(want)
            assert np.array_equal(got[inf], np.asarray(want[inf], dtype=np.float64)), (label, key)   # +-inf stays +-inf
            errs[key] = R.rel_err(got[~inf], want[~inf])
        st = cosmo_b200.Settings(scaling=scaling)
        assert np.array_equal(_rho_classes(eng, st), _ref_rho_classes(ref, sets, dtype, st)), label
    print("%s [%s]: worst %s; bars %.1e (D, E, c) / %.1e (entries, vectors)"
          % (label, np.dtype(dtype).name, {k: "%.1e" % v for k, v in errs.items()}, scal_bar, entry_bar))
    for k, v in errs.items():
        # the cost is a sum over n products: the device's summation adds up to n + 2 roundings to the entries' errors
        assert v <= (scal_bar if k in ("D", "E", "c") else entry_bar + (n + 2) * _u(dtype) if k == "cost" else entry_bar), \
            (label, k, v)
    return errs


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_clip_edges_at_the_first_pass(dtype):
    """scaling = 1: the norms are plain maxima of the data, so every scale is decidable bit for bit.  Columns 0-2 take
    their norms from P, 3-5 from A; rows and columns at exactly MIN keep it (scale 1/sqrt(MIN) = 100), one float below
    MIN gets the scale 1, above MAX is clipped to MAX, exactly MAX is kept."""
    T = np.dtype(dtype).type
    lo, hi = T(1e-4), T(1e4)
    below = np.nextafter(lo, T(0))
    n = m = 6
    P = sp.csc_matrix(np.diag([lo, below, 1e5, 1e-6, 1e-6, 1e-6]).astype(np.float64))
    Ad = np.zeros((m, n))
    Ad[0, 3], Ad[0, 0] = lo, 1e-6          # row 0: exactly MIN; column 3 (through A): exactly MIN
    Ad[1, 4], Ad[1, 1] = below, 1e-6       # row 1 and column 4 (through A): the float below MIN
    Ad[2, 5] = 1e5                         # row 2 and column 5 (through A): above MAX
    Ad[3, 5], Ad[3, 2] = hi, 1.0           # row 3: exactly MAX, kept
    Ad[4, 5] = 2e4                         # row 4: clipped to MAX, not 1 / sqrt(2e4)
    Ad[5, 2] = 0.5
    sets = [cosmo_b200.Nonnegatives(m)]
    eng, ref = _setup(P, np.ones(n), sp.csc_matrix(Ad), np.ones(m), sets, dtype, scaling=1)
    D, Ev, c = eng.scaling()
    inv = lambda v: np.float64(T(1) / np.sqrt(T(v)))
    clip = lambda v: np.where(v < lo, T(1), np.where(v > hi, hi, v)).astype(dtype)
    Dn = np.maximum(np.abs(P.toarray().astype(dtype)).max(0), np.abs(Ad.astype(dtype)).max(0))
    En = np.abs(Ad.astype(dtype)).max(1)
    want_D = (T(1) / np.sqrt(clip(Dn))).astype(np.float64)
    want_E = (T(1) / np.sqrt(clip(En))).astype(np.float64)
    assert np.array_equal(D, want_D), (D, want_D)
    assert np.array_equal(Ev, want_E), (Ev, want_E)
    assert D[0] == D[3] == inv(lo) and abs(inv(lo) - 100) <= 2 * _u(dtype) * 100
    assert D[1] == D[4] == 1.0 and D[2] == D[5] == inv(hi)
    assert Ev[0] == inv(lo) and Ev[1] == 1.0 and Ev[2] == Ev[3] == Ev[4] == inv(hi) and Ev[4] != inv(2e4)
    assert Ev[5] == inv(0.5)
    # the branches, as the restatement took them
    p = ref.passes[0]
    assert list(p["D_low"]) == [1, 4] and list(p["D_high"]) == [2, 5]
    assert list(p["E_low"]) == [1] and list(p["E_high"]) == [2, 4]
    assert np.array_equal(np.asarray(ref.D, dtype=np.float64), want_D) or R.rel_err(want_D, ref.D) <= _u(dtype)
    _check(eng, ref, sets, dtype, 1, "clip edges")


@pytest.mark.parametrize("dtype", DTYPES)
def test_zero_rows_and_columns_keep_the_scale_one(dtype):
    """an all-zero row of A (no entries), a row of stored zeros, an empty column of both P and A and a column of P
    without its diagonal entry: the zero norms take the scale 1 in every pass, the stored zeros stay zero"""
    rng = np.random.default_rng(4)
    n, m = 8, 9
    Pd = np.zeros((n, n))
    for i, j in ((0, 0), (1, 1), (2, 2), (3, 3), (4, 4), (7, 7), (0, 3), (2, 5), (4, 7), (1, 5)):
        Pd[i, j] = Pd[j, i] = rng.uniform(0.5, 3.0) * 10.0 ** rng.integers(-2, 3)
    # column 5: off-diagonal entries only; column 6: empty in P and A
    Ad = rng.standard_normal((m, n)) * 10.0 ** rng.uniform(-2, 2, (m, n))
    Ad[:, 6] = 0.0
    Ad[7, :] = 0.0
    Ad[8, :] = 0.0
    Ad[rng.random((m, n)) < 0.3] = 0.0
    r, k = np.nonzero(Ad)
    # row 8: stored zeros in columns 0 and 1
    A = sp.csc_matrix((np.r_[Ad[r, k], 0.0, 0.0], (np.r_[r, 8, 8], np.r_[k, 0, 1])), shape=(m, n))
    assert A.nnz == r.size + 2                         # the stored zeros are there
    sets = [cosmo_b200.ZeroSet(2), cosmo_b200.Nonnegatives(m - 2)]
    eng, ref = _setup(sp.csc_matrix(Pd), rng.standard_normal(n), A, rng.standard_normal(m), sets, dtype)
    D, Ev, c = eng.scaling()
    assert D[6] == 1.0 and Ev[7] == 1.0 and Ev[8] == 1.0, (D[6], Ev[7], Ev[8])
    for p in ref.passes:
        assert 6 in p["D_zero"] and 7 in p["E_zero"] and 8 in p["E_zero"]
    _check(eng, ref, sets, dtype, 10, "zero structure")


@pytest.mark.parametrize("case", ["lp", "q_zero", "lp_q_zero", "qp"])
@pytest.mark.parametrize("dtype", DTYPES)
def test_cost_scaling_guard(dtype, case):
    """the cost scaling runs only when mean(col norms of P) != 0 and |q|_inf != 0 (scaling.jl:82): c is exactly 1 for
    an LP, for q = 0 and for both; the QP is the control"""
    rng = np.random.default_rng(5)
    n, m = 30, 40
    P = R._sym_pattern(n, 0.2, rng, R._spread(-2, 2))
    if case.startswith("lp"):
        P = sp.csc_matrix((n, n))
    q = np.zeros(n) if case.endswith("q_zero") else R._spread(-2, 2)(n, rng)
    A = sp.csc_matrix(sp.random(m, n, density=0.2, random_state=rng) + sp.eye(m, n))
    sets = [cosmo_b200.Nonnegatives(m)]
    eng, ref = _setup(P, q, A, rng.standard_normal(m), sets, dtype)
    _, _, c = eng.scaling()
    if case == "qp":
        assert R.branch_count(ref, "cost") == 10 and c != 1.0
    else:
        assert R.branch_count(ref, "cost") == 0 and c == 1.0, c
    _check(eng, ref, sets, dtype, 10, "cost guard " + case)


@pytest.mark.parametrize("scaling", [1, 3, 10])
@pytest.mark.parametrize("dtype", DTYPES)
def test_dynamic_range_clips_in_every_pass(dtype, scaling):
    """entries over 1e-8 .. 1e8 and one of 3e12: norms below MIN in every pass, above MAX in the first three"""
    P, q, A, b, sets = R.problem_dynamic_range()
    eng, ref = _setup(P, q, A, b, sets, dtype, scaling=scaling)
    later = range(1, min(scaling, 3))
    for key in ("D_low", "E_low", "D_high", "E_high"):
        assert R.branch_count(ref, key, [0]) > 0, key
        if scaling > 1:
            assert R.branch_count(ref, key, later) > 0, key
    _check(eng, ref, sets, dtype, scaling, "dynamic range scaling=%d" % scaling)


@pytest.mark.parametrize("dtype", DTYPES)
def test_every_rectified_family(dtype):
    """SOC, PsdCone, PsdConeTriangle, ComplexPsdConeTriangle, Exp, DualExp, Pow, DualPow beside Zero, Nonnegatives and
    Box rows; one PSD triangle of 300 rows (> kBlock, the block reduction spans all warps).  On each rectified cone E is
    E (mean / E) as in the reference (E .*= Ework, scaling.jl:129-142): the cone's mean up to two roundings, so all its
    values lie within two ulps of each other; on the rows that are not rectified E varies."""
    P, q, A, b, sets = R.problem_every_rectified_family()
    eng, ref = _setup(P, q, A, b, sets, dtype)
    cones = R.sets_to_oracle(sets)
    assert ref.rectified == 9
    _, Ev, _ = eng.scaling()
    T = np.dtype(dtype).type
    off_mean = 0
    for rng, cone in zip(O.row_ranges(cones), cones):
        e = Ev[rng].astype(dtype)
        if isinstance(cone, O.SCALAR_SCALED_CONES):
            two_ulps = np.nextafter(np.nextafter(e.min(), T(np.inf)), T(np.inf))
            assert e.max() <= two_ulps, (type(cone).__name__, e.min(), e.max())
            off_mean += e.size - int(np.unique(e, return_counts=True)[1].max())
        elif cone.dim > 1:
            assert np.ptp(e) > 0, type(cone).__name__
    print("every rectified family [%s]: %d rows of rectified cones off their cone's most common E"
          % (np.dtype(dtype).name, off_mean))
    _check(eng, ref, sets, dtype, 10, "every rectified family")


@pytest.mark.parametrize("dtype", DTYPES)
def test_box_bounds_and_row_classes(dtype):
    """finite, +-inf, one-sided and equality bounds: l .*= E, u .*= E (convexset.jl:863-867), an infinite bound stays
    infinite, and the row classes behind rho_vec follow the scaled bounds -- including rows whose class the scaling
    changes (a bound across COSMO_INFTY * MIN_SCALING, a width across RHO_TOL)"""
    rng = np.random.default_rng(6)
    inf = np.inf
    l = np.array([-2.0, -inf, -4.0, -inf, 1.5, 0.0, -3e16, -3e16, -1e17, 2.0, -1.0, -5.0])
    u = np.array([3.0, 5.0, inf, inf, 1.5, 6e-5, 3e16, 3e16, 1e17, 2.00004, 1e-4, inf])
    nb = l.size
    n, m = 20, nb + 6
    sets = [cosmo_b200.Box(l, u), cosmo_b200.Nonnegatives(3), cosmo_b200.ZeroSet(3)]
    A = sp.random(m, n, density=0.4, random_state=rng, format="csr")
    A.data = R._spread(-1, 1)(A.data.size, rng)
    A = sp.csc_matrix(sp.diags(10.0 ** rng.uniform(-2, 2, m)) @ (A + sp.eye(m, n)))
    b = rng.standard_normal(m)
    b[nb] = 3e16                       # a Nonnegatives row near the loose threshold
    P = R._sym_pattern(n, 0.2, rng, R._spread(-1, 1))
    eng, ref = _setup(P, rng.standard_normal(n), A, b, sets, dtype)
    st = cosmo_b200.Settings()
    unscaled = _ref_rho_classes(R.scale_ruiz_ld(P, np.zeros(n), A, b, R.sets_to_oracle(sets), scaling=0, dtype=dtype),
                                sets, dtype, st)
    scaled = _ref_rho_classes(ref, sets, dtype, st)
    assert np.any(unscaled != scaled) and set(scaled[:nb]) == {0, 1, 2}, (unscaled, scaled)
    box, lo, up = _box_bounds(eng, sets)
    assert np.array_equal(lo[4], up[4])                                   # l = u stays an equality, bit for bit
    _check(eng, ref, sets, dtype, 10, "box bounds")


@pytest.mark.parametrize("dtype", DTYPES)
def test_long_rows_and_n_above_1024(dtype):
    """a row of A with 1500 entries and a column with 1600 (rows of A and A' longer than 32 and than 1024: the warp per
    row loops), n = 1500 > 1024 for the single-block ruiz_cost_kernel"""
    rng = np.random.default_rng(7)
    n, m = 1500, 1600
    A = sp.random(m, n, density=0.003, random_state=rng, format="lil")
    A[0, :] = R._spread(-3, 3)(n, rng)
    A[:, 0] = R._spread(-3, 3)(m, rng)[:, None]
    A = sp.csc_matrix(A + sp.eye(m, n))
    A.data = np.where(A.data == 0, 1.0, A.data)
    P = R._sym_pattern(n, 0.002, rng, R._spread(-2, 2))
    sets = [cosmo_b200.ZeroSet(100), cosmo_b200.Nonnegatives(m - 100)]
    eng, ref = _setup(P, R._spread(-2, 2)(n, rng), A, rng.standard_normal(m), sets, dtype)
    assert max(np.diff(sp.csr_matrix(A).indptr)) > 1024 and max(np.diff(A.indptr)) > 1024
    _check(eng, ref, sets, dtype, 10, "long rows, n = 1500")


@pytest.mark.parametrize("dtype", DTYPES)
def test_wide_qp_slabs_hold_the_scaled_values(dtype):
    """the wide QP of the oracle parity test (column-windowed slabs, packed in fp64): D, E, c, and the columns of A and
    rows of A' on both ends and around the middle of the column range, bit for bit those the reference rounds to"""
    P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(30000, 4000, 0.002, seed=5)
    eng, ref = _setup(P, q, A, b, sets, dtype)
    _check(eng, ref, sets, dtype, 10, "wide QP", read=False)
    m, n = ref.shape
    _, entry_bar = _bars(dtype, 10)
    Ar = sp.csc_matrix((np.asarray(ref.A[2], dtype=np.float64), (ref.A[0], ref.A[1])), shape=(m, n))
    Pr = sp.csc_matrix((np.asarray(ref.P[2], dtype=np.float64), (ref.P[0], ref.P[1])), shape=(n, n))
    cols = [0, 1, n // 2 - 1, n // 2, n - 1]
    rows = [0, 1, m // 2, m - 2, m - 1]
    errs = {"A": R.rel_err(_read(eng, 0, cols), Ar[:, cols].toarray()),
            "At": R.rel_err(_read(eng, 1, rows), Ar[rows, :].toarray().T),
            "P": R.rel_err(_read(eng, 2, cols), Pr[:, cols].toarray())}
    print("wide QP [%s]: sampled entries %s; bar %.1e" % (np.dtype(dtype).name, {k: "%.1e" % v for k, v in errs.items()},
                                                          entry_bar))
    assert max(errs.values()) <= entry_bar, errs


@pytest.mark.parametrize("dtype", DTYPES)
def test_scaled_P_is_symmetric(dtype):
    """the scaled P equals its transpose bit for bit (the reference symmetrizes it, scaling.jl:99): c D_i P_ij D_j
    rounded the same way on both sides of the diagonal, with D over many binades and c != 1"""
    P, q, A, b, sets = R.problem_symmetry()
    eng, ref = _setup(P, q, A, b, sets, dtype)
    _, _, c = eng.scaling()
    D = eng.scaling()[0]
    assert c != 1.0 and np.ptp(np.log2(D)) > 4
    Pd = _read(eng, 2)
    asym, pairs = _asymmetric_pairs(Pd)
    assert asym == 0, "%d of %d off-diagonal pairs of the scaled P are not symmetric" % (asym, pairs)
    _check(eng, ref, sets, dtype, 10, "symmetry")


@pytest.mark.parametrize("dtype", DTYPES)
def test_update_matrices_reproduces_a_fresh_engine(dtype):
    """update_matrices with new unscaled P, A, q, b on an equilibrating engine re-runs the equilibration: D, E, c, the
    scaled entries, b, q, the Box bounds and the row classes are bit for bit those of a new engine with these data"""
    P, q, A, b, sets = R.problem_every_rectified_family()
    P, q, A, b, sets = _as_dtype(P, q, A, b, sets, dtype)
    rng = np.random.default_rng(8)
    f = 10.0 ** rng.uniform(-3, 3, P.shape[0])
    P2 = P.copy()
    P2.data = P.data * (f[P.indices] * f[np.repeat(np.arange(P.shape[0]), np.diff(P.indptr))])   # exactly symmetric
    A2 = A.copy()
    A2.data = A.data * 10.0 ** rng.uniform(-3, 3, A.data.size)
    q2, b2 = 10.0 * rng.standard_normal(q.size), 0.1 * rng.standard_normal(b.size)
    P2, q2, A2, b2, _ = _as_dtype(P2, q2, A2, b2, sets, dtype)
    upd, _ = _setup(P, q, A, b, sets, dtype)
    upd.update_matrices(P2.data, A2.data, q2, b2)
    new, ref = _setup(P2, q2, A2, b2, sets, dtype)
    for a, b_ in zip(upd.scaling(), new.scaling()):
        assert np.array_equal(a, b_)
    for which in (0, 1, 2):
        assert np.array_equal(_read(upd, which), _read(new, which)), which
    m, n = upd.m, upd.n
    x = rng.standard_normal(n)
    for args in ((np.zeros(n), np.zeros(m), np.zeros(m)), (x, rng.standard_normal(m), rng.standard_normal(m))):
        assert upd.residuals(*args, ignore_scaling=True) == new.residuals(*args, ignore_scaling=True)
    assert np.array_equal(upd.rho_vec(), new.rho_vec())
    for got, want in zip(_box_bounds(upd, sets), _box_bounds(new, sets)):
        assert np.array_equal(got, want)
    _check(upd, ref, sets, dtype, 10, "update_matrices")
