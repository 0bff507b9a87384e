"""The rho vector of the engine, bit for bit, against a NumPy statement of classify_constraints! (setup.jl:75-85;
convexset.jl:62-69, 831-842) and set_rho_vec! / apply_constraint_rho_scaling! (parameters.jl:3-49), applied to the b
and Box bounds the engine holds: the values as given, or T(E) * T(b) and T(E) * T(l), T(E) * T(u) after device
equilibration.  Each T value is widened to fp64 before it is compared or before u - l is formed, as the classification
of the engine does, so an fp32 b of 1e16 (10000000272564224 as a float) is loose against big = 1e16.

Every step that classifies rows is covered, for fp64 and fp32, with scaling 0 and with device equilibration: create;
update_qb(b) moving Nonnegatives rows across big in both directions, before and after a solve whose rho adapted (the
rho vector then takes the current rho, not settings.rho); update_matrices (with equilibration a new E, so new scaled b
and bounds); and update_settings with a new RHO_TOL, which takes effect at the next reset(), not before."""
import dataclasses

import numpy as np
import pytest
import scipy.sparse as sp

import cosmo_b200
from cosmo_b200 import engine as E
from cosmo_b200 import model as M
from tests import custom_cones as CC
from tests.gpu_helpers import _tuples

pytestmark = pytest.mark.gpu

INF = np.inf
B_NONNEG = np.array([2e16, 5e15, 1e16, 1.0, 0.0, 3.0])        # b of the Nonnegatives rows at create
B_NONNEG_SOLVE = np.array([1.0, 2.0, 0.5, 1.0, 0.0, 3.0])    # ... for the solve: x = 0 is feasible
B_NONNEG_AFTER = np.array([5e15, 2e16, 1e16, 3e16, 0.0, 3.0])  # ... after it
BOX_L = np.array([-INF, -2e16, 0.3, 1.0, 1.0, -INF, -1.0, -1.0])
BOX_U = np.array([INF, 2e16, 0.3, 1.0 + 5e-5, 1.0 + 2e-4, 1.0, INF, 1.0])
N_ZERO, N_SOC, N_PSD, N_CUSTOM = 3, 3, 6, 4
KIND_ZERO, KIND_NONNEG, KIND_BOX, KIND_OTHER = 0, 1, 2, 3


def _problem(seed=0):
    """Zero, Nonnegatives (b around big), Box (loose, tight and plain bounds), SOC, PSD and a custom cone; b is in the
    cones except on the Nonnegatives rows"""
    rng = np.random.default_rng(seed)
    sets = [M.ZeroSet(N_ZERO), M.Nonnegatives(B_NONNEG.size), M.Box(BOX_L, BOX_U), M.SecondOrderCone(N_SOC),
            M.PsdConeTriangle(N_PSD), M.CustomCone(CC.nonpos_type(), N_CUSTOM)]
    kind = np.concatenate([np.full(N_ZERO, KIND_ZERO), np.full(B_NONNEG.size, KIND_NONNEG),
                           np.full(BOX_L.size, KIND_BOX), np.full(N_SOC + N_PSD + N_CUSTOM, KIND_OTHER)])
    m, n = kind.size, 10
    A = sp.csc_matrix(rng.standard_normal((m, n)) * rng.uniform(0.1, 10.0, (m, 1)))
    P = sp.csc_matrix(np.diag(rng.uniform(0.5, 2.0, n)))
    q = rng.standard_normal(n)
    b = np.zeros(m)
    b[kind == KIND_NONNEG] = B_NONNEG
    b[kind == KIND_BOX] = np.clip(0.0, BOX_L, BOX_U)
    return P, q, A, b, sets, kind


def _expected(kind, b, l, u, st, rho, T):
    """the rho vector for the T values b, l, u (l, u read on Box rows only) the engine holds"""
    b, l, u = (np.asarray(v, dtype=T).astype(np.float64) for v in (b, l, u))
    big = st.COSMO_INFTY * st.MIN_SCALING
    cls = np.zeros(kind.size, dtype=np.int64)
    cls[kind == KIND_ZERO] = 1
    cls[(kind == KIND_NONNEG) & (b > big)] = 2
    with np.errstate(invalid="ignore"):
        box_loose = (l < -big) & (u > big)
        box_eq = ~box_loose & ((u - l) < st.RHO_TOL)
    cls[(kind == KIND_BOX) & box_loose] = 2
    cls[(kind == KIND_BOX) & box_eq] = 1
    r = T(rho)
    return np.where(cls == 2, T(st.RHO_MIN), np.where(cls == 1, r * T(st.RHO_EQ_OVER_RHO_INEQ), r)).astype(T)


def _bounds(kind):
    """the Box bounds as m-vectors (+-inf on the other rows)"""
    l, u = np.full(kind.size, -INF), np.full(kind.size, INF)
    l[kind == KIND_BOX], u[kind == KIND_BOX] = BOX_L, BOX_U
    return l, u


def _assert_bits(got, want, step):
    bad = np.flatnonzero(got.view(np.uint8).reshape(got.size, -1) != want.view(np.uint8).reshape(want.size, -1))
    assert got.dtype == want.dtype and bad.size == 0, (step, np.unique(bad), got, want)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("equilibrate", [False, True], ids=["scaling0", "device_ruiz"])
def test_rho_vector_follows_the_row_classes(dtype, equilibrate):
    T = np.dtype(dtype).type
    P, q, A, b, sets, kind = _problem()
    settings = cosmo_b200.Settings(scaling=10 if equilibrate else 0, max_iter=200, eps_abs=1e-12, eps_rel=1e-12,
                                   adaptive_rho_interval=5)
    eng = E.Engine(P, q, A, b, _tuples(sets), settings.to_struct(), dtype=dtype, equilibrate=equilibrate)

    def check(b, st, rho, step, b_scaled=True):
        """the rho vector for the b and Box bounds the engine holds: with device equilibration the bounds are always
        scaled by its E, b when it came through create or update_matrices (update_qb takes b as handed over)"""
        b, (l, u) = np.asarray(b, dtype=T), (np.asarray(v, dtype=T) for v in _bounds(kind))
        if equilibrate:
            e = eng.scaling()[1].astype(T)
            box = kind == KIND_BOX
            l[box], u[box] = e[box] * l[box], e[box] * u[box]
            if b_scaled:
                b = e * b
        got = eng.rho_vec()
        _assert_bits(got, _expected(kind, b, l, u, st, rho, T), step)
        return got

    def with_nonneg(v):
        out = b.copy()
        out[kind == KIND_NONNEG] = v
        return out

    try:
        rho0 = check(b, settings, settings.rho, "create")
        assert np.unique(rho0).size == 3, "every rho class is present"

        # Nonnegatives rows across big, loose -> active; the engine takes b as handed over (an equilibrating engine
        # expects it scaled)
        eng.update_qb(b=with_nonneg(B_NONNEG_SOLVE))
        check(with_nonneg(B_NONNEG_SOLVE), settings, settings.rho, "update_qb", b_scaled=False)
        out = eng.solve()
        assert len(out.rho_updates) > 1 and out.rho != settings.rho, "the solve adapted rho"
        check(with_nonneg(B_NONNEG_SOLVE), settings, out.rho, "solve", b_scaled=False)
        # active -> loose, and the vector takes the adapted rho
        eng.update_qb(b=with_nonneg(B_NONNEG_AFTER))
        check(with_nonneg(B_NONNEG_AFTER), settings, out.rho, "update_qb after an adapted solve", b_scaled=False)

        # new values of A: a new E when the engine equilibrates, the rows classified on the new scaled data, rho reset
        A2 = A.copy()
        A2.data = A.data * np.random.default_rng(5).uniform(0.2, 5.0, A.nnz)
        eng.update_matrices(Px=P.data, Ax=A2.data, q=q, b=b)
        check(b, settings, settings.rho, "update_matrices")

        # RHO_TOL is read when rows are classified: update_settings alone leaves the vector, reset() reclassifies
        settings2 = dataclasses.replace(settings, RHO_TOL=1e-2)
        eng.update_settings(settings2.to_struct())
        before = check(b, settings, settings.rho, "update_settings")
        eng.reset()
        after = check(b, settings2, settings2.rho, "reset with a new RHO_TOL")
        assert not np.array_equal(after, before), "the new RHO_TOL moved a Box row"
    finally:
        eng.close()
