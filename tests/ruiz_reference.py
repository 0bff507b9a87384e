"""scale_ruiz! (scaling.jl:21-116) restated in extended precision, literally as the reference runs it (tests only).

The data are rescaled on every pass, the norms are limited with clip(s, MIN, MAX, 1, MAX), the cost scaling runs under
the mean != 0 && |q|_inf != 0 guard, every cone of the oracle's SCALAR_SCALED_CONES gets one mean of E, P is symmetrized
at the end (scaling.jl:99, algebra.jl:215) and the Box bounds are scaled (convexset.jl:863-867).  The arithmetic is
np.longdouble (80-bit extended on x86, 64 significand bits): 11 more bits than fp64, so against the device's fp64 and fp32
results the reference's own rounding is negligible.  The matrices are kept as coordinate triplets so that the wide
problems of the tests fit.

scale_ruiz_ld also counts, pass by pass, which branch every norm took, so that a test can assert it reached the branch it
is named for: D_low / E_low (norm < MIN: scale 1, zero norms included), D_zero / E_zero, D_high / E_high (norm > MAX:
clipped), `cost` (whether the cost scaling ran) and `rectified` (the number of cones given one scalar)."""
from types import SimpleNamespace

import numpy as np
import scipy.sparse as sp

from oracle import cosmo_oracle as O

LD = np.longdouble


def _triplets(M):
    """(row, col, value) of a sparse matrix in CSC order, explicit zeros kept, values in extended precision"""
    M = sp.csc_matrix(M)
    col = np.repeat(np.arange(M.shape[1]), np.diff(M.indptr))
    return M.indices.astype(np.int64), col.astype(np.int64), np.asarray(M.data).astype(LD)


def _absmax(idx, val, size):
    out = np.zeros(size, dtype=LD)
    if val.size:
        np.maximum.at(out, idx, np.abs(val))
    return out


def _clip(s, lo, hi):
    """clip(s, MIN, MAX, one, MAX) (algebra.jl:5-7 with the arguments of scaling.jl:10-13)"""
    return np.where(s < lo, LD(1), np.where(s > hi, hi, s))


def _transpose_index(i, j, n):
    """k' with (i[k'], j[k']) = (j[k], i[k]) for every k; P must have a symmetric pattern"""
    key = i * n + j
    order = np.argsort(key, kind="stable")
    pos = np.searchsorted(key[order], j * n + i)
    if np.any(pos >= key.size) or np.any(key[order[np.minimum(pos, key.size - 1)]] != j * n + i):
        raise ValueError("P must store both triangles on a symmetric pattern")
    return order[pos]


def scale_ruiz_ld(P, q, A, b, cones, scaling=10, MIN_SCALING=1e-4, MAX_SCALING=1e4, dtype=np.float64):
    """scale_ruiz! in extended precision.  P (both triangles), q, A, b hold the values the engine sees (already rounded
    to `dtype`); `cones` are oracle cones.  MIN / MAX are taken in `dtype` like the engine's Settings{T}.  Returns a
    namespace with D, E, c, the scaled triplets P = (i, j, v) and A = (i, j, v), q, b, the scaled Box bounds l, u (NaN
    off the Box rows) and the branch counts `passes` (one dict per pass) and `rectified`."""
    T = np.dtype(dtype).type
    lo, hi = LD(T(MIN_SCALING)), LD(T(MAX_SCALING))
    A = sp.csc_matrix(A)
    m, n = A.shape
    pi, pj, pv = _triplets(P)
    ai, aj, av = _triplets(A)
    q = np.array(q, dtype=LD)
    b = np.array(b, dtype=LD)
    D, E, c = np.ones(n, dtype=LD), np.ones(m, dtype=LD), LD(1)
    passes = []
    for _ in range(scaling):
        Dw = np.maximum(_absmax(pj, pv, n), _absmax(aj, av, n))      # kkt_col_norms!, scaling.jl:3-8
        Ew = _absmax(ai, av, m)
        rec = {"D_low": np.nonzero(Dw < lo)[0], "D_zero": np.nonzero(Dw == 0)[0], "D_high": np.nonzero(Dw > hi)[0],
               "E_low": np.nonzero(Ew < lo)[0], "E_zero": np.nonzero(Ew == 0)[0], "E_high": np.nonzero(Ew > hi)[0]}
        Dw = LD(1) / np.sqrt(_clip(Dw, lo, hi))                        # limit_scaling!, inv_sqrt!
        Ew = LD(1) / np.sqrt(_clip(Ew, lo, hi))
        pv = Dw[pi] * pv * Dw[pj]                                      # scale_data!, scaling.jl:157-168
        av = Ew[ai] * av * Dw[aj]
        q = Dw * q
        b = Ew * b
        D = Dw * D
        E = Ew * E
        mean_col_norm_P = np.mean(_absmax(pj, pv, n)) if n else LD(0)
        inf_norm_q = np.max(np.abs(q)) if n else LD(0)
        rec["cost"] = bool(mean_col_norm_P != 0 and inf_norm_q != 0)
        if rec["cost"]:
            inf_norm_q = _clip(inf_norm_q, lo, hi)
            scale_cost = _clip(max(inf_norm_q, mean_col_norm_P), lo, hi)
            ctmp = LD(1) / scale_cost
            pv = pv * ctmp
            q = q * ctmp
            c = c * ctmp
        passes.append(rec)
    # rectify_set_scalings! (scaling.jl:129-142; convexset.jl:905-958): Ework = mean(E[cone]) ./ E[cone], E .*= Ework
    Ew = np.ones(m, dtype=LD)
    rectified = 0
    for rng, cone in zip(O.row_ranges(cones), cones):
        if isinstance(cone, O.SCALAR_SCALED_CONES) and cone.dim > 0:
            Ew[rng] = np.mean(E[rng]) / E[rng]
            rectified += 1
    if rectified:
        av = Ew[ai] * av
        b = Ew * b
        E = Ew * E
    # issymmetric(P) || symmetrize_full!(P)  (scaling.jl:99, algebra.jl:215-223)
    if pv.size:
        pv = (pv + pv[_transpose_index(pi, pj, n)]) / LD(2)
    # scale_sets! -> scale!(::Box) (scaling.jl:145-154, convexset.jl:863-867)
    l = np.full(m, np.nan, dtype=LD)
    u = np.full(m, np.nan, dtype=LD)
    for rng, cone in zip(O.row_ranges(cones), cones):
        if isinstance(cone, O.Box):
            l[rng] = np.asarray(cone.l, dtype=np.float64).astype(LD) * E[rng]
            u[rng] = np.asarray(cone.u, dtype=np.float64).astype(LD) * E[rng]
    return SimpleNamespace(D=D, E=E, c=c, P=(pi, pj, pv), A=(ai, aj, av), q=q, b=b, l=l, u=u, passes=passes,
                           rectified=rectified, shape=(m, n))


def dense(triplet, shape):
    """a scaled triplet as a dense extended-precision matrix (explicit zeros stay 0)"""
    i, j, v = triplet
    out = np.zeros(shape, dtype=LD)
    out[i, j] = v
    return out


def branch_count(ref, key, passes=None):
    """the number of indices that took branch `key` (D_low, D_zero, D_high, E_low, E_zero, E_high) over `passes`
    (an iterable of pass numbers, default all), or for key = 'cost' the number of passes whose cost scaling ran"""
    sel = range(len(ref.passes)) if passes is None else passes
    if key == "cost":
        return sum(int(ref.passes[k]["cost"]) for k in sel)
    return sum(ref.passes[k][key].size for k in sel)


def rel_err(got, ref):
    """max |got - ref| / |ref| over the entries with ref != 0; an entry with ref == 0 must be exactly 0 (else inf)"""
    got = np.asarray(got).astype(LD)
    ref = np.asarray(ref, dtype=LD)
    nz = ref != 0
    if np.any(got[~nz] != 0):
        return float("inf")
    if not np.any(nz):
        return 0.0
    return float(np.max(np.abs(got[nz] - ref[nz]) / np.abs(ref[nz])))


# ---------------------------------------------------------------------------------------------------------------------
# the test problems (cosmo_b200 sets; shared by the CPU check of this restatement and the device parity tests)
# ---------------------------------------------------------------------------------------------------------------------
def _sym_pattern(n, density, rng, mag=lambda k, rng: rng.standard_normal(k)):
    B = sp.random(n, n, density=density, random_state=rng, format="coo")
    B.data = mag(B.data.size, rng)
    S = sp.triu(B, 1)
    P = S + S.T + sp.diags(np.abs(mag(n, rng)) + 0.1)
    return sp.csc_matrix(P)


def _spread(lo_exp, hi_exp):
    """entries with magnitudes 10^U(lo_exp, hi_exp) and random signs"""
    return lambda k, rng: rng.choice([-1.0, 1.0], k) * 10.0 ** rng.uniform(lo_exp, hi_exp, k)


def problem_dynamic_range(seed=0, n=80, m=120):
    """P and A with entries over 1e-8 .. 1e8, four columns and four rows of entries below 1e-6 and one entry of 3e12:
    the norms below MIN recur in every pass, the one above MAX in the first three (3e12 -> 3e8 -> 3e4 -> 3)"""
    import cosmo_b200
    rng = np.random.default_rng(seed)
    P = _sym_pattern(n, 0.08, rng, _spread(-8, 8)).tolil()
    A = sp.random(m, n, density=0.08, random_state=rng, format="csc")
    A.data = _spread(-8, 8)(A.data.size, rng)
    A = sp.lil_matrix(A + sp.eye(m, n, format="csc"))
    tiny_cols, tiny_rows = rng.choice(np.arange(1, n), 4, replace=False), rng.choice(np.arange(1, m), 4, replace=False)
    for j in tiny_cols:
        P[j, :] = 0
        P[:, j] = 0
        P[j, j] = 1e-7
        for i in A[:, j].nonzero()[0]:
            A[i, j] = _spread(-8, -6)(1, rng)[0]
    for i in tiny_rows:
        for j in A[i, :].nonzero()[1]:
            A[i, j] = _spread(-8, -6)(1, rng)[0]
    A[0, 0] = 3e12
    P, A = sp.csc_matrix(P), sp.csc_matrix(A)
    P.eliminate_zeros()
    A.eliminate_zeros()
    q = _spread(-6, -4)(n, rng)
    b = _spread(-4, 4)(m, rng)
    return P, q, A, b, [cosmo_b200.ZeroSet(20), cosmo_b200.Nonnegatives(m - 20)]


def problem_every_rectified_family(seed=1, n=60):
    """every family the reference rectifies beside rows that it does not, and a PSD triangle of 300 rows (> kBlock)"""
    import cosmo_b200 as cb
    rng = np.random.default_rng(seed)
    sets = [cb.ZeroSet(3), cb.Nonnegatives(4), cb.Box(-np.ones(3), np.ones(3)), cb.SecondOrderCone(5), cb.PsdCone(9),
            cb.PsdConeTriangle(6), cb.ComplexPsdConeTriangle(9), cb.ExponentialCone(), cb.DualExponentialCone(),
            cb.PowerCone(0.3), cb.DualPowerCone(0.6), cb.Nonnegatives(2), cb.PsdConeTriangle(300)]
    m = sum(S.dim for S in sets)
    P = _sym_pattern(n, 0.1, rng, _spread(-2, 2))
    A = sp.random(m, n, density=0.15, random_state=rng, format="csc")
    A.data = _spread(-3, 3)(A.data.size, rng)
    A = sp.csc_matrix(A + sp.eye(m, n, format="csc"))
    return P, rng.standard_normal(n), A, rng.standard_normal(m), sets


def problem_symmetry(seed=3, n=200, m=150):
    """a dense-ish P whose scalings D spread over many binades and a cost scaling c != 1: the rounding order of
    c D_i P_ij D_j decides the last bit of about a third of the pairs"""
    import cosmo_b200
    rng = np.random.default_rng(seed)
    s = 10.0 ** rng.uniform(-3, 3, n)
    P = _sym_pattern(n, 0.3, rng)
    P.data *= s[P.indices] * s[np.repeat(np.arange(n), np.diff(P.indptr))]     # s_i s_j: P stays exactly symmetric
    A = sp.random(m, n, density=0.1, random_state=rng, format="csc")
    A.data = rng.standard_normal(A.data.size)
    q = 37.0 * rng.standard_normal(n)
    return P, q, sp.csc_matrix(A @ sp.diags(s)), rng.standard_normal(m), [cosmo_b200.Nonnegatives(m)]


def sets_to_oracle(sets):
    from oracle.bridge import to_oracle_cones
    return to_oracle_cones(sets)
