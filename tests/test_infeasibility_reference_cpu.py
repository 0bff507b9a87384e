"""The high-precision reference of the infeasibility tests (tests/infeasibility_reference.py) checked against the
oracle's own predicates (in_dual, in_pol_recc, support_function) on random points whose margin is outside the band
the GPU tests use, so that the truth the kernels are held to is itself tested."""
import math

import numpy as np
import pytest

from oracle import cosmo_oracle as O
from tests import infeasibility_reference as R

U = 2.0 ** -53
TOL = 2.0 ** -10


def _band(scale, k=64):
    return k * U * max(scale, 1.0)


def test_soc_against_oracle():
    rng = np.random.default_rng(0)
    checked = 0
    for _ in range(400):
        d = int(rng.integers(2, 12))
        v = rng.standard_normal(d)
        v[0] = -np.linalg.norm(v[1:]) * (1 + 0.05 * rng.standard_normal()) + TOL
        ok, margin, nrm = R.soc_cert(v, TOL)
        if abs(margin) <= _band(nrm):
            continue
        assert ok == bool(O.in_pol_recc(v, O.SecondOrderCone(d), TOL)) == bool(O.in_dual(-v, O.SecondOrderCone(d), TOL))
        checked += 1
    assert checked > 300
    # an exact boundary point: tail norm 5 = tol - v0
    assert R.soc_cert(np.array([-4.75, 3.0, 4.0]), 0.25)[:2] == (True, 0.0)


@pytest.mark.parametrize("typ", [R.PSD_SQUARE, R.PSD_TRIANGLE, R.PSD_TRIANGLE_COMPLEX])
def test_psd_against_oracle(typ):
    rng = np.random.default_rng(1 + typ)
    checked = 0
    for N in (1, 2, 3, 5, 8, 13, 20):
        for _ in range(6):
            if typ == R.PSD_SQUARE:
                x = rng.standard_normal(N * N)               # not symmetric: the upper triangle decides
                cone = O.PsdCone(N * N)
            elif typ == R.PSD_TRIANGLE:
                x = rng.standard_normal(N * (N + 1) // 2)
                cone = O.PsdConeTriangle(x.size)
            else:
                x = rng.standard_normal(N * N)
                cone = O.ComplexPsdConeTriangle(N * N)
            X = R.psd_matrix(x, typ)
            x = x - (R.lambda_max(X) - TOL * (1 + 0.5 * rng.standard_normal())) * _identity_vec(N, typ)
            ok, margin, lam, fro = R.psd_cert(x, typ, TOL)
            if abs(margin) <= 8 * N * U * fro:
                continue
            assert ok == bool(O.in_pol_recc(x, cone, TOL)) == bool(O.in_dual(-x, cone, TOL)), (N, margin)
            checked += 1
    assert checked >= 30


def _identity_vec(N, typ):
    if typ == R.PSD_SQUARE:
        return np.eye(N).reshape(-1, order="F")
    e = np.zeros(N * (N + 1) // 2 if typ == R.PSD_TRIANGLE else N * N)
    k = 0
    for j in range(N):
        e[k + j] = 1.0
        k += j + 1
    return e


def test_square_psd_reads_the_upper_triangle():
    # the example of the symmetrization bug: upper reflection -I (certified), symmetrized matrix lambda_max = +1
    x = np.array([-1.0, 4.0, 0.0, -1.0])
    ok, margin, lam, _ = R.psd_cert(x, R.PSD_SQUARE, 0.25)
    assert ok and lam == -1.0
    assert O.in_pol_recc(x, O.PsdCone(4), 0.25)
    assert np.linalg.eigvalsh((x.reshape(2, 2, order="F") + x.reshape(2, 2)) / 2)[-1] == 1.0


def test_lambda_max_mpmath_matches_lapack():
    rng = np.random.default_rng(5)
    for N in (2, 7, R.MP_EIG_MAX_N):
        B = rng.standard_normal((N, N))
        X = (B + B.T) / 2
        assert abs(R.lambda_max(X) - np.linalg.eigvalsh(X)[-1]) <= 8 * N * U * np.linalg.norm(X)
        Z = B + 1j * rng.standard_normal((N, N))
        H = (Z + Z.conj().T) / 2
        assert abs(R.lambda_max(H) - np.linalg.eigvalsh(H)[-1]) <= 8 * N * U * np.linalg.norm(H)


@pytest.mark.parametrize("typ,alpha", [(R.EXP, 0.0), (R.DUAL_EXP, 0.0), (R.POW, 0.3), (R.DUAL_POW, 0.3),
                                       (R.POW, 0.01), (R.DUAL_POW, 0.99)])
def test_exp_pow_against_oracle(typ, alpha):
    rng = np.random.default_rng(10 + typ)
    cone = {R.EXP: O.ExponentialCone, R.DUAL_EXP: O.DualExponentialCone}[typ]() if typ in (R.EXP, R.DUAL_EXP) else \
        (O.PowerCone if typ == R.POW else O.DualPowerCone)(alpha)
    checked = 0
    for _ in range(600):
        v = rng.standard_normal(3) * 10.0 ** rng.integers(-3, 3)
        ok, margin = R.c3_cert(v, typ, TOL, alpha)
        if abs(margin) <= _band(float(np.max(np.abs(v))) * 8, 256):
            continue
        assert ok == bool(O.in_pol_recc(v, cone, TOL)) == bool(O.in_dual(-v, cone, TOL)), (v, margin)
        checked += 1
    assert checked > 400


def test_pow_negative_base_in_band_is_not_in_the_cone():
    # s in [-tol, 0): the reference raises a DomainError; defined as "not in the cone" on both sides
    assert R.pow_in_dual(-TOL / 2, 1.0, 0.0, 0.5, TOL) == (False, -math.inf)
    assert not O.in_dual(np.array([-TOL / 2, 1.0, 0.0]), O.PowerCone(0.5), TOL)


def test_box_support_against_oracle():
    rng = np.random.default_rng(3)
    for _ in range(50):
        k = int(rng.integers(1, 40))
        l = -np.abs(rng.standard_normal(k))
        u = np.abs(rng.standard_normal(k))
        y = rng.standard_normal(k)
        y[rng.random(k) < 0.2] = TOL
        s, mag = R.box_support(y, l, u, TOL)
        assert abs(s - O.support_function(y, O.Box(l, u), TOL)) <= k * U * mag
    l, u = np.array([-np.inf, -1.0, 2.0]), np.array([1.0, np.inf, 2.0])
    assert math.isnan(R.box_support(np.array([0.0, 0.0, 1.0]), l, u, TOL)[0])          # 0 * -inf
    assert math.isnan(O.support_function(np.array([0.0, 0.0, 1.0]), O.Box(l, u), TOL))
    s, _ = R.box_support(np.array([-0.5, 0.5, TOL]), np.array([-1.0, -1.0, 2.0]), np.array([1.0, 1.0, 2.0]), TOL)
    assert s == 0.5 + 0.5 + TOL * 2.0


def test_rows_against_oracle():
    rng = np.random.default_rng(4)
    for _ in range(200):
        k = int(rng.integers(1, 6))
        v = rng.choice([0.0, TOL, np.nextafter(TOL, 1), np.nextafter(TOL, -1), -TOL, -np.nextafter(TOL, 1)], k)
        assert R.rows_ok(v, R.NONNEG, TOL, primal=False) == O.in_pol_recc(v, O.Nonnegatives(k), TOL)
        assert R.rows_ok(v, R.NONNEG, TOL, primal=True) == (O.support_function(v, O.Nonnegatives(k), TOL) == 0.0)
        assert R.rows_ok(v, R.ZERO, TOL, primal=False) == O.in_pol_recc(v, O.ZeroSet(k), TOL)
        l = np.where(rng.random(k) < 0.5, -np.inf, -1.0)
        u = np.where(rng.random(k) < 0.5, np.inf, 1.0)
        assert R.rows_ok(v, R.BOX, TOL, l, u, primal=False) == O.in_pol_recc(v, O.Box(l, u), TOL)


def test_gates_against_oracle_formulas():
    import scipy.sparse as sp
    rng = np.random.default_rng(6)
    m, n = 30, 12
    A = sp.random(m, n, 0.3, random_state=7, format="csc") + sp.eye(m, n, format="csc")
    b = rng.standard_normal(m)
    Em, D = 2.0 ** rng.integers(-3, 4, m), 2.0 ** rng.integers(-3, 4, n)
    dy = rng.standard_normal(m)
    g = R.primal_gates(A, b, Em, 1.0 / D, dy, 1e-4)
    assert g["norm"] == O.scaled_norm(Em, dy, np.inf)
    assert g["gate"] == 2 and abs(g["gate2"] - np.max(np.abs((A.T @ dy) / D))) <= 4 * U * g["gate2_mag"]
    P = sp.csc_matrix((n, n))
    q = rng.standard_normal(n)
    dx = -q * 1e3
    h = R.dual_gates(P, q, A, D, 1.0 / D, 1.0 / Em, 1.0, dx, 1e-4)
    assert h["gate"] == 4 and h["Pdx"] == 0.0 and abs(h["qdx"] - q @ dx) <= 4 * U * h["qdx_mag"]
    assert np.all(np.abs(h["v"] - (A @ dx) / Em / h["norm"]) <= 16 * U * h["v_mag"])
