"""The double-double reference of the projection Jacobian (tests/projection_jacobian_reference.py), pinned without a GPU:
against mpmath at 50 digits (mp.eigsy) on small PSD cones and the SOC closed form, against central differences of the
oracle's projection, against the fp64 restatement solve_adjoint_reference.dpi (the yardstick of the GPU derivative
tests) on the cases the GPU tests use, and its matrix product against exact rational arithmetic."""
from fractions import Fraction

import mpmath as mp
import numpy as np
import pytest

from oracle import cosmo_oracle as O
from tests import projection_jacobian_reference as R
from tests import solve_adjoint_reference as SA
from tests.test_gpu_projection_jacobian import SOC_POINTS, SPECTRA, _antisym, _soc_point, _spectrum_case, _vec


def _mp_dpi_psd(w, h, N, triangle):
    """Dpi h of a real PSD cone at 50 digits, on the exact fp64 input"""
    mp.mp.dps = 50
    half = mp.mpf(1) / 2
    W, H = mp.matrix(N, N), mp.matrix(N, N)
    if triangle:
        r, c = R._svec_index(N)
        s2 = mp.sqrt(2)
        for k, (i, j) in enumerate(zip(r, c)):
            W[i, j] = W[j, i] = mp.mpf(w[k]) if i == j else mp.mpf(w[k]) / s2
            H[i, j] = H[j, i] = mp.mpf(h[k]) if i == j else mp.mpf(h[k]) / s2
    else:
        for i in range(N):
            for j in range(N):
                W[i, j] = (mp.mpf(w[j * N + i]) + mp.mpf(w[i * N + j])) * half
                H[i, j] = (mp.mpf(h[j * N + i]) + mp.mpf(h[i * N + j])) * half
    E, Q = mp.eigsy(W)
    C = Q.T * H * Q
    for i in range(N):
        for j in range(N):
            li, lj = E[i], E[j]
            if (li > 0) == (lj > 0):
                g = 1 if li > 0 else 0
            else:
                g = li / (li - lj) if li > 0 else lj / (lj - li)
            C[i, j] *= g
    X = Q * C * Q.T
    if triangle:
        return [X[i, j] if i == j else X[i, j] * mp.sqrt(2) for i, j in zip(*R._svec_index(N))]
    return [X[i, j] for j in range(N) for i in range(N)]


def _mp_err(o, ref):
    return max(abs(mp.mpf(float(o[0][k])) + mp.mpf(float(o[1][k])) - ref[k]) for k in range(len(ref)))


@pytest.mark.parametrize("triangle", [True, False], ids=["triangle", "square"])
@pytest.mark.parametrize("kind", ["wigner", "clusters", "rank", "tiny+", "tiny-", "positive"])
@pytest.mark.parametrize("N", [2, 5, 12])
def test_psd_against_mpmath(N, kind, triangle):
    rng = np.random.default_rng(N * 7 + len(kind))
    W, H = _spectrum_case(kind, N, rng)
    w = _vec(W, triangle)
    h = _vec(H, triangle) if triangle else _vec(H + _antisym(N, rng), False)
    o, kap, _, nh = R.psd_dd(w, h, N, triangle)
    err = _mp_err(o, _mp_dpi_psd(w, h, N, triangle))
    # clusters and exact zeros: the refinement resolves the split inside a cluster (a genuine u-sized split of the fp64
    # W, or the null space of the rank case) to fp64 accuracy only, which Gamma sees at first order
    tol = 1e-13 if kind in ("clusters", "rank") else 1e-25
    assert err <= tol * kap * max(nh, 1.0), (float(err), kap)


@pytest.mark.parametrize("d", [2, 3, 9, 40])
def test_soc_against_mpmath(d):
    mp.mp.dps = 50
    rng = np.random.default_rng(d)
    for kind in SOC_POINTS:
        w, h = _soc_point(kind, d, rng), rng.standard_normal(d)
        o = R.soc_dd(w, h)
        t, x = mp.mpf(w[0]), [mp.mpf(v) for v in w[1:]]
        r = mp.sqrt(sum(v * v for v in x))
        hm = [mp.mpf(v) for v in h]
        if r <= t:
            ref = hm
        elif r <= -t:
            ref = [mp.mpf(0)] * d
        else:
            dot = sum(a * b for a, b in zip(x, hm[1:]))
            ref = [(hm[0] + dot / r) / 2] + [(xi / r * hm[0] + (1 + t / r) * hi - (t / r) * xi * dot / r ** 2) / 2
                                           for xi, hi in zip(x, hm[1:])]
        assert _mp_err(o, ref) <= 1e-28 * (1 + np.abs(h).sum()), kind


def test_central_differences_of_the_oracle_projection():
    rng = np.random.default_rng(1)
    cones = [O.Nonnegatives(4), O.Box(np.array([-1.0, 0.0]), np.array([1.0, 2.0])), O.SecondOrderCone(5),
             O.PsdConeTriangle(10), O.PsdCone(9), O.ZeroSet(2)]
    X4 = rng.standard_normal((4, 4))
    X3 = rng.standard_normal((3, 3))
    w = np.concatenate([rng.standard_normal(4), [0.3, 3.0], _soc_point("generic", 5, rng), SA._mat_to_tri(X4 + X4.T),
                        (X3 + X3.T).reshape(-1), rng.standard_normal(2)])
    h = rng.standard_normal(w.size)
    got = R.dpi(w, cones, h)
    eps = 1e-6

    def proj(v):
        v = v.copy()
        O.project(v, cones)
        return v
    fd = (proj(w + eps * h) - proj(w - eps * h)) / (2 * eps)
    assert np.max(np.abs(got - fd)) <= 1e-8 * (1 + np.abs(h).max()), np.max(np.abs(got - fd))


@pytest.mark.parametrize("triangle", [True, False], ids=["triangle", "square"])
@pytest.mark.parametrize("N", [1, 2, 3, 31, 33, 64, 96, 97, 129])
def test_agrees_with_the_fp64_restatement(N, triangle):
    rng = np.random.default_rng(1000 * N + triangle)
    cone = O.PsdConeTriangle(N * (N + 1) // 2) if triangle else O.PsdCone(N * N)
    for kind in SPECTRA:
        W, H = _spectrum_case(kind, N, rng)
        w = _vec(W, triangle)
        h = _vec(H, triangle) if triangle else _vec(H + _antisym(N, rng), False)
        o, kap, _, nh = R.psd_dd(w, h, N, triangle)
        err = np.linalg.norm(R.value(o) - SA.dpi(w, [cone], h))
        assert err <= 1e-13 * kap * max(nh, 1e-300) * max(1.0, N / 10), (kind, err, kap)
    for d in (1, 2, 4, 8194):
        for kind in SOC_POINTS:
            w, h = _soc_point(kind, d, rng), rng.standard_normal(d)
            err = np.max(np.abs(R.value(R.soc_dd(w, h)) - SA.dpi(w, [O.SecondOrderCone(d)], h)))
            assert err <= 1e-13 * (1 + np.abs(h).max()), (d, kind, err)


def test_matmul_against_fractions():
    rng = np.random.default_rng(2)
    A = (rng.integers(-1000, 1000, (9, 9)) * 2.0 ** -7, rng.integers(-1000, 1000, (9, 9)) * 2.0 ** -70)
    B = (rng.integers(-2 ** 40, 2 ** 40, (9, 9)).astype(float), rng.integers(-9, 9, (9, 9)) * 2.0 ** -30)
    P = R.matmul(A, B)
    for i in range(9):
        for j in range(9):
            ex = sum((Fraction(A[0][i, k]) + Fraction(A[1][i, k])) * (Fraction(B[0][k, j]) + Fraction(B[1][k, j]))
                     for k in range(9))
            got = Fraction(P[0][i, j]) + Fraction(P[1][i, j])
            assert abs(got - ex) <= abs(ex) * Fraction(2) ** -100 + Fraction(2) ** -60, (i, j)


def test_kink_counts_and_the_scale_of_the_soc_reference():
    u = 2.0 ** -53
    b = R.kink_band(0.0, u)
    cones = [O.Nonnegatives(3), O.Box(np.array([0.0]), np.array([1.0])), O.SecondOrderCone(3)]
    w = np.array([b / 4, -4 * b, 1.0, 1.0 - 1e-17, 5.0, 3.0, 4.0])
    assert R.kink_counts(w, cones, u) == (2, 1, 0)
    # Dpi(2^k w)(2^j h) = 2^j Dpi(w) h, exactly, over the whole exponent range
    rng = np.random.default_rng(3)
    w, h = _soc_point("generic", 50, rng), rng.standard_normal(50)
    base = R.value(R.soc_dd(w, h))
    for k, j in ((-1000, -300), (900, 300), (0, 300)):
        assert np.array_equal(np.ldexp(R.value(R.soc_dd(np.ldexp(w, k), np.ldexp(h, j))), -j), base)
