"""Scale and shape edges of the projection kernels and of the int8-sliced product kernel.

* Homogeneity ladder: every projection is positively homogeneous, Pi(2^k w) = 2^k Pi(w), and multiplying by a power of two
  is exact, so 2^k Pi_oracle(w) is an exact reference at every scale whose inputs and outputs are normal numbers.
* Product kernel edges: one partial tile, tile boundaries, rows whose maximum is (just below) a power of two, zero rows,
  operands near both ends of the fp64 exponent range.
* Mixed shapes: cones of different N share the tensor-core workspace of one engine (sliced buffers, tensor maps, tile
  list, the l0 schedule); the small-kernel / tensor-core boundary N = 96 / 97."""
import numpy as np
import pytest

import cosmo_b200
from cosmo_b200 import engine as E
from tests import golden_problems as G
from tests.gpu_helpers import U32, _hermitian_ws, _oracle_project, _project_engine, _psd_test_matrix, _round32

pytestmark = pytest.mark.gpu


def _away_from_zero(w, floor):
    """nonzero entries no smaller than `floor` in magnitude: every entry of 2^k w stays zero or a normal number"""
    return np.where((np.abs(w) < floor) & (w != 0), np.where(w < 0, -floor, floor), w)


def _ladder_case(cone, rng):
    """(sets, w, env) of one cone type at unit scale"""
    if cone == "soc":
        d = 5000
        w = rng.standard_normal(d)
        w[0] = 0.5 * np.linalg.norm(w[1:])                   # generic branch: neither inside the cone nor its polar
        return [cosmo_b200.SecondOrderCone(d)], w, None
    if cone == "soc_chunks":
        # the tail is normed in chunks of 8192 entries; the first chunk is exactly zero, so it must not set the exponent
        # the other chunks are combined at (their squares would underflow against 2^0 at the small end of the ladder)
        d = 20000
        w = rng.standard_normal(d)
        w[1:8193] = 0.0
        w[0] = 0.5 * np.linalg.norm(w[1:])
        return [cosmo_b200.SecondOrderCone(d)], w, None
    if cone == "psd_small":
        N = 60
        return [cosmo_b200.PsdConeTriangle(N * (N + 1) // 2)], G._svec(_psd_test_matrix("wigner", N, rng)), None
    if cone == "psd_tc":
        N = 200
        X = _psd_test_matrix("wigner", N, rng)
        return [cosmo_b200.PsdConeTriangle(N * (N + 1) // 2)], G._svec(X), None
    if cone == "psd_block_jacobi":
        N = 150
        return [cosmo_b200.PsdCone(N * N)], _psd_test_matrix("wigner", N, rng).reshape(-1, order="F"), ("COSMO_B200_PSD_TC", "0")
    if cone == "psd_complex_small":
        return [cosmo_b200.ComplexPsdConeTriangle(12 * 12)], _hermitian_ws(12, rng, "shifted")[0], None
    if cone == "psd_complex_tc":
        return [cosmo_b200.ComplexPsdConeTriangle(60 * 60)], _hermitian_ws(60, rng, "shifted")[0], None
    raise ValueError(cone)


CONES = ["soc", "psd_small", "psd_tc", "psd_block_jacobi", "psd_complex_small", "psd_complex_tc", "soc_chunks"]
LADDER = {np.float64: [-1000, -600, -300, 0, 300, 600, 900], np.float32: [-100, -75, -40, 0, 40, 64, 100]}


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("cone", CONES)
def test_homogeneity_ladder(cone, dtype, monkeypatch):
    rng = np.random.default_rng(CONES.index(cone))
    sets, w, env = _ladder_case(cone, rng)
    if env:
        monkeypatch.setenv(*env)
    f32 = dtype == np.float32
    w = _away_from_zero(w, 2.0 ** -20)
    if f32:
        w = _round32(w)
    ref = _oracle_project(w, sets)                     # fp64 projection of exactly the input the kernel gets, at scale 1
    nrm = np.linalg.norm(w)
    # the bars of the unscaled tests: fp64 1e-14 (SOC) / 1e-12 (PSD) of |w|; fp32 (dim + 2) u32 (SOC) / 1e-5 (PSD)
    if cone in ("soc", "soc_chunks"):
        bar = 4.0 * (w.size + 2) * U32 if f32 else 1e-14
    elif cone == "psd_block_jacobi" and f32:
        bar = 2e-4      # block Jacobi in fp32: 5.8e-5 of |X|_F at N = 150 and scale 1 (test_gpu_float32.py, a known gap)
    elif cone == "psd_small" and f32:
        bar = 2e-5      # small-cone Jacobi in fp32 at N = 60: measured 1.10e-5 of |X|_F at every k (a known gap, as above)
    else:
        bar = 1e-5 if f32 else 1e-12
    eng = _project_engine(sets, dtype=dtype)
    for k in LADDER[dtype]:
        got = eng.project(np.ldexp(w, k).astype(dtype)).astype(np.float64)
        assert np.all(np.isfinite(got)), (cone, k)
        err = np.linalg.norm(np.ldexp(got, -k) - ref) / nrm
        assert err <= bar, (cone, k, err)
    st = eng.psd_stats()
    if cone in ("psd_tc", "psd_complex_tc"):   # a wrong answer counted as a tensor-core success would have failed above
        assert st["tc_projections"] == len(LADDER[dtype]) and st["tc_fallbacks"] == 0, st
    elif cone == "psd_block_jacobi":
        assert st["tc_projections"] == 0 and st["tc_fallbacks"] == 0, st


# ---------------------------------------------------------------------------
# product kernel (cosmo_b200_tc_gemm_test): C = A B, error relative to |A| |B| (test_tc_gemm_matches_dgemm)
# ---------------------------------------------------------------------------
def _edge_operands(N, rng):
    Gm = rng.standard_normal((N, N))
    A = (Gm + Gm.T) / np.sqrt(2.0 * N)
    np.fill_diagonal(A, np.clip(np.diag(A), -0.4, 0.4))
    A[0, 0] = 1.0                               # row maxima exactly a power of two ...
    A[1, 1] = -0.5
    A[2, 2] = 1.0 - 2.0 ** -53                  # ... and just below one: the leading digit is 64
    A[3, 3] = -(2.0 - 2.0 ** -52)
    return A


def _check_product(A, B, ref, scale_a=1.0, scale_b=1.0, bound=2e-15):
    got, _, _ = E.tc_gemm(A, B)
    got = got / (scale_a * scale_b) if scale_a * scale_b != 1.0 else got
    assert np.all(np.isfinite(got))
    err = np.max(np.abs(got - ref) / (np.abs(A / scale_a) @ np.abs(B / scale_b) + 1e-300))
    assert err < bound, err
    return got


@pytest.mark.parametrize("N", [97, 127, 129, 255, 256, 257])
def test_tc_gemm_tile_edges(N):
    rng = np.random.default_rng(N)
    A = _edge_operands(N, rng)
    B = A @ A
    B = (B + B.T) / 2
    got = _check_product(A, B, A @ B)
    assert np.array_equal(got, got.T)
    # block diagonal with an all-zero block: exactly zero rows / columns in both operands and in the product
    k = N // 2
    Z = A.copy()
    Z[k:, :] = 0.0
    Z[:, k:] = 0.0
    ZB = Z @ Z
    got = _check_product(Z, ZB, Z @ ZB)
    assert np.all(got[k:, :] == 0.0) and np.all(got[:, k:] == 0.0)


@pytest.mark.parametrize("N", [97, 256])
def test_tc_gemm_extreme_exponents(N):
    # every row is sliced relative to its own power-of-two scale, so the product is exact to 2^-7K of the row maxima over
    # the whole normal range; the references are computed at scale 1 and scaled by powers of two (exact)
    rng = np.random.default_rng(7 + N)
    A = _edge_operands(N, rng)
    B = A @ A
    B = (B + B.T) / 2
    ref = A @ B
    big, small = 2.0 ** 1000, 2.0 ** -1000
    _check_product(A * big, B * small, ref, big, small)
    tiny = 2.0 ** -1020
    _check_product(A, B * tiny, ref, 1.0, tiny)


# ---------------------------------------------------------------------------
# mixed shapes in one engine
# ---------------------------------------------------------------------------
def test_mixed_large_cone_shapes_share_the_workspace():
    # N = 250 and 200 share the padded size Np = 256: stale rows / columns of the larger cone would enter the K sum of the
    # smaller one if the padding were not cleared.  Three calls, since the l0 schedule carries over between calls.
    sizes = [130, 385, 250, 200, 256]
    sets = [cosmo_b200.PsdConeTriangle(N * (N + 1) // 2) for N in sizes] + [cosmo_b200.PsdCone(N * N) for N in sizes]
    eng = _project_engine(sets)
    rng = np.random.default_rng(11)
    kinds = ["wigner", "admm_like", "shifted"]
    for call in range(3):
        mats = [_psd_test_matrix(kinds[(call + i) % 3], N, rng) for i, N in enumerate(sizes + sizes)]
        ws = np.concatenate([G._svec(X) for X in mats[:5]] + [X.reshape(-1, order="F") for X in mats[5:]])
        got = eng.project(ws)
        ref = _oracle_project(ws, sets)
        off = 0
        for S in sets:
            seg = slice(off, off + S.dim)
            err = np.linalg.norm(got[seg] - ref[seg]) / (np.linalg.norm(ws[seg]) + 1e-300)
            assert err < 1e-12, (call, type(S).__name__, S.dim, err)
            off += S.dim
    st = eng.psd_stats()
    assert st["tc_projections"] == 3 * len(sets) and st["tc_fallbacks"] == 0, st


@pytest.mark.parametrize("N,tc", [(96, 0), (97, 1)])
def test_small_kernel_tensor_core_boundary(N, tc):
    rng = np.random.default_rng(N)
    sets = [cosmo_b200.PsdConeTriangle(N * (N + 1) // 2)]
    ws = G._svec(_psd_test_matrix("wigner", N, rng))
    eng = _project_engine(sets)
    got = eng.project(ws)
    assert np.linalg.norm(got - _oracle_project(ws, sets)) / np.linalg.norm(ws) < 1e-12
    st = eng.psd_stats()
    assert st["tc_projections"] == tc and st["tc_fallbacks"] == 0, st
