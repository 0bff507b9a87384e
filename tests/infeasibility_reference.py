"""High-precision truth for the individual operations of the infeasibility tests (infeasibility.jl,
convexset.jl), written from the reference's formulas and independent of the oracle's code: the oracle stays the
parity reference for whole solves, this module is the reference for each gate and each cone's certificate.

Precision:
  * every inequality that involves a computed quantity (a dot product, an SpMV, a norm, exp, pow, an eigenvalue) is
    evaluated with mpmath at 50 significant digits (``DPS``); products of two fp64 numbers are exact there;
  * the Box support function is the sum of the terms of convexset.jl:850-856 taken with ``math.fsum``;
  * lambda_max of a PSD cone comes from ``mpmath.eigsy`` / ``mpmath.eighe`` at 50 digits for sides up to
    ``MP_EIG_MAX_N`` and from LAPACK (``numpy.linalg.eigvalsh``, fp64, backward stable: error <= ~N u64 |A|_2) beyond,
    where mpmath is too slow; in fp64 that error can use a small share of the tests' lambda_max bar (8 N u |X|_F),
    in fp32 it is negligible;
  * comparisons of an input against a constant (x < 0, y == 0, |x| <= tol) are exact in floating point and are decided
    exactly.

Every certificate returns (ok, margin): ``margin`` is the signed distance of the fuzzy inequality from its bound
(ok <=> margin >= 0, or > 0 for the strict PSD test), combined over the disjuncts / conjuncts of the reference's
predicate with max / min, exact comparisons counting as +-inf.  A test may accept either device verdict only when
|margin| is inside the band it states; outside it the verdict must match exactly.

The vector a primal cone test sees is what the device computes before its cone kernels: ``normalized_primal``
reproduces the elementwise fp steps (scale by -1/|dy| in the engine's type), so that the truth is evaluated at the
device's exact operands.

Conventions of the reference kept here:
  * a PsdCone is read from its upper triangle (is_pos_def! -> cholesky!(Hermitian(X)), convexset.jl:324-336);
    PsdConeTriangle through populate_upper_triangle with 1/sqrt 2; the complex triangle as its Hermitian matrix;
  * a negative base inside the tol band of PowerCone's in_dual (convexset.jl:728-734) is a DomainError in the
    reference; it is defined here as "not in the cone".
"""
import math

import mpmath
import numpy as np

DPS = 50
MP_EIG_MAX_N = 12
ZERO, NONNEG, BOX, SOC, PSD_SQUARE, PSD_TRIANGLE, EXP, DUAL_EXP, POW, DUAL_POW, PSD_TRIANGLE_COMPLEX = range(11)
PSD_TYPES = (PSD_SQUARE, PSD_TRIANGLE, PSD_TRIANGLE_COMPLEX)
C3_TYPES = (EXP, DUAL_EXP, POW, DUAL_POW)
FAMILY_ROWS, FAMILY_SOC, FAMILY_PSD, FAMILY_C3 = 1, 2, 4, 8
INF = float("inf")


def _mp(x):
    return mpmath.mpf(float(x))


def unit_roundoff(dtype):
    return 2.0 ** -24 if np.dtype(dtype) == np.float32 else 2.0 ** -53


# ---- gates (infeasibility.jl) ------------------------------------------------------------------
def scaled_norm_inf(scale, v, dtype=np.float64):
    """|scale .* v|_inf with each product rounded once in ``dtype`` (what scaled_norm computes in T), so the result
    is exact and a kernel must reproduce it bit for bit; scale None = identity."""
    v = np.asarray(v, dtype=dtype)
    p = v if scale is None else np.asarray(scale, dtype=dtype) * v
    return float(np.max(np.abs(p))) if p.size else 0.0


def spmv(M, v):
    """(M v at 50 digits rounded to fp64, |M| |v|): the exact product and the magnitude an SpMV bar is relative to"""
    import scipy.sparse as sp
    M = sp.csr_matrix(M)
    out = np.zeros(M.shape[0])
    mag = np.zeros(M.shape[0])
    with mpmath.workdps(DPS):
        for i in range(M.shape[0]):
            lo, hi = M.indptr[i], M.indptr[i + 1]
            terms = [_mp(a) * _mp(v[j]) for a, j in zip(M.data[lo:hi], M.indices[lo:hi])]
            out[i] = float(mpmath.fsum(terms))
            mag[i] = float(mpmath.fsum([abs(t) for t in terms]))
    return out, mag


def dot(a, b):
    """(a'b at 50 digits, sum |a_i b_i|)"""
    with mpmath.workdps(DPS):
        terms = [_mp(x) * _mp(y) for x, y in zip(a, b)]
        return float(mpmath.fsum(terms)), float(mpmath.fsum([abs(t) for t in terms]))


def primal_gates(A, b, E, Dinv, dy, eps, dtype=np.float64):
    """is_primal_infeasible!'s gates: {norm, gate (1: |E dy| <= eps, 2: |Dinv A'dy| > eps |E dy|, 4: cone tests),
    gate2 = |Dinv A'dy|_inf, gate2_mag (its SpMV magnitude), v (the normalized -dy the cone tests see), dyt_b, dyt_b_mag}"""
    norm = scaled_norm_inf(E, dy, dtype)
    out = {"norm": norm, "gate": 1}
    if not norm > eps:
        return out
    Aty, mag = spmv(A.T, dy)
    d = np.ones(len(Aty)) if Dinv is None else np.asarray(Dinv, dtype=np.float64)
    out["gate2"] = float(np.max(np.abs(d * Aty))) if len(Aty) else 0.0
    out["gate2_mag"] = float(np.max(np.abs(d) * mag)) if len(Aty) else 0.0
    out["gate"] = 2
    if not out["gate2"] <= eps * norm:
        return out
    out["gate"] = 4
    v = normalized_primal(dy, norm, dtype)
    out["v"] = v
    out["dyt_b"], out["dyt_b_mag"] = dot(v, b)
    return out


def normalized_primal(dy, norm, dtype=np.float64):
    """dy .* (-1 / |E dy|_inf), rounded in ``dtype`` as the engine computes it"""
    T = np.dtype(dtype).type
    return (np.asarray(dy, dtype=dtype) * T(-1.0 / norm)).astype(np.float64)


def dual_gates(P, q, A, D, Dinv, Einv, c, dx, eps, dtype=np.float64):
    """is_dual_infeasible!'s gates: {norm, gate (1..4), qdx (q'dx), qdx_mag, Pdx (|Dinv P dx|_inf), Pdx_mag,
    v = Einv A dx / |D dx| (at 50 digits, rounded to fp64), v_mag}"""
    norm = scaled_norm_inf(D, dx, dtype)
    out = {"norm": norm, "gate": 1}
    out["qdx"], out["qdx_mag"] = dot(q, dx)
    if not norm > eps:
        return out
    out["gate"] = 2
    if not out["qdx"] / (norm * c) < -eps:
        return out
    out["gate"] = 3
    Pdx, mag = spmv(P, dx)
    d = np.ones(len(Pdx)) if Dinv is None else np.asarray(Dinv, dtype=np.float64)
    out["Pdx"] = float(np.max(np.abs(d * Pdx))) if len(Pdx) else 0.0
    out["Pdx_mag"] = float(np.max(np.abs(d) * mag)) if len(Pdx) else 0.0
    if not out["Pdx"] / (norm * c) <= eps:
        return out
    out["gate"] = 4
    Adx, mag = spmv(A, dx)
    e = np.ones(len(Adx)) if Einv is None else np.asarray(Einv, dtype=np.float64)
    out["v"] = e * Adx / norm
    out["v_mag"] = np.abs(e) * mag / norm
    return out


# ---- elementwise rows (convexset.jl:30-36, 76-82, 850-860) ------------------------------------------
def box_support(v, l, u, tol):
    """(sum of the convexset.jl:850-856 terms by math.fsum, sum |terms|); NaN when a term is 0 * inf"""
    terms = []
    for x, lo, hi in zip(v, l, u):
        with np.errstate(invalid="ignore"):
            terms.append(float(x) * float(hi) if (abs(x) > tol and x > 0) else float(x) * float(lo))
    if any(math.isnan(t) for t in terms):
        return float("nan"), float("nan")
    if any(math.isinf(t) for t in terms):
        return float(sum(terms)), INF
    return math.fsum(terms), math.fsum(abs(t) for t in terms)


def rows_ok(v, typ, tol, l=None, u=None, primal=True):
    """the row family's verdict on the rows of one Zero / Nonnegatives / Box set (exact comparisons)"""
    v = np.asarray(v, dtype=np.float64)
    if typ == NONNEG:
        return not np.any(v > tol)
    if primal:
        return True                      # Zero: in_dual is always true; Box: enters through its support function
    if typ == ZERO:
        return not np.any(np.abs(v) > tol)
    return not (np.any((np.asarray(u) == INF) & (v > tol)) or np.any((np.asarray(l) == -INF) & (v < -tol)))


# ---- second-order cone (convexset.jl:116-122) --------------------------------------------------
def soc_cert(v, tol):
    """-v in K* / v in the polar recession cone: |v[2:]|_2 <= tol - v[1]; margin = tol - v[1] - |v[2:]|"""
    with mpmath.workdps(DPS):
        nrm = mpmath.sqrt(mpmath.fsum([_mp(x) ** 2 for x in v[1:]]))
        margin = _mp(tol) - _mp(v[0]) - nrm
        return bool(margin >= 0), float(margin), float(nrm)


# ---- PSD cones ---------------------------------------------------------------------------------
def psd_side(typ, dim):
    if typ == PSD_SQUARE:
        return int(round(math.sqrt(dim)))
    if typ == PSD_TRIANGLE:
        return int(round((math.sqrt(8 * dim + 1) - 1) / 2))
    return int(round(math.sqrt(dim)))


def psd_matrix(x, typ):
    """the matrix the reference's certificate factorizes: the upper reflection of a PsdCone, populate_upper_triangle
    (1/sqrt 2) of a PsdConeTriangle, the Hermitian matrix of a complex triangle (convexset.jl:444-490)"""
    x = np.asarray(x, dtype=np.float64)
    N = psd_side(typ, x.size)
    if typ == PSD_SQUARE:
        X = x.reshape(N, N, order="F")
        U = np.triu(X)
        return U + np.triu(U, 1).T
    s = 1.0 / math.sqrt(2.0)
    if typ == PSD_TRIANGLE:
        X = np.zeros((N, N))
        k = 0
        for j in range(N):
            for i in range(j):
                X[i, j] = X[j, i] = s * x[k]
                k += 1
            X[j, j] = x[k]
            k += 1
        return X
    H = np.zeros((N, N), dtype=complex)
    k = 0
    for j in range(N):
        for i in range(j):
            H[i, j] = s * x[k]
            k += 1
        H[j, j] = x[k]
        k += 1
    for j in range(N):
        for i in range(j):
            H[i, j] += 1j * s * x[k]
            k += 1
    return np.triu(H) + np.triu(H, 1).conj().T


def lambda_max(X):
    """largest eigenvalue of a symmetric / Hermitian matrix: mpmath at 50 digits up to MP_EIG_MAX_N, LAPACK beyond"""
    N = X.shape[0]
    if N == 0:
        return -INF
    if N > MP_EIG_MAX_N:
        return float(np.linalg.eigvalsh(X)[-1])
    with mpmath.workdps(DPS):
        if np.iscomplexobj(X):
            M = mpmath.matrix([[mpmath.mpc(complex(X[i, j])) for j in range(N)] for i in range(N)])
            ev = mpmath.eighe(M, eigvals_only=True)
        else:
            M = mpmath.matrix([[_mp(X[i, j]) for j in range(N)] for i in range(N)])
            ev = mpmath.eigsy(M, eigvals_only=True)
        return float(max(ev[i] for i in range(N)))


def psd_cert(x, typ, tol):
    """-mat(v) + tol I positive definite <=> lambda_max(mat v) < tol; margin = tol - lambda_max (strict)"""
    X = psd_matrix(x, typ)
    lam = lambda_max(X)
    return bool(tol - lam > 0), tol - lam, lam, float(np.linalg.norm(X))


# ---- exponential / power cones (convexset.jl:600-612, 719-745, 780-781) ----------------------------
def _combine(disjuncts):
    """max over disjuncts of min over conjuncts (exact comparisons enter as +-inf)"""
    return max(min(c) for c in disjuncts)


def exp_in_cone(x, y, z, tol):
    """(y > 0 and y e^(x/y) <= z + tol) or (x <= tol and y == 0 and z >= -tol)"""
    with mpmath.workdps(DPS):
        X, Y, Z = _mp(x), _mp(y), _mp(z)
        d1 = [INF if y > 0 else -INF]
        if y > 0:
            d1.append(float(Z + _mp(tol) - Y * mpmath.exp(X / Y)))
        d2 = [INF if (x <= tol and y == 0.0 and z >= -tol) else -INF]
        m = _combine([d1, d2])
        return m >= 0, m


def exp_in_dual(x, y, z, tol):
    """(x < 0 and -x e^(y/x) - e z <= tol) or (|x| <= tol and y >= -tol and z >= -tol)"""
    with mpmath.workdps(DPS):
        X, Y, Z = _mp(x), _mp(y), _mp(z)
        d1 = [INF if x < 0 else -INF]
        if x < 0:
            d1.append(float(_mp(tol) - (-X * mpmath.exp(Y / X) - mpmath.e * Z)))
        d2 = [INF if (abs(x) <= tol and y >= -tol and z >= -tol) else -INF]
        m = _combine([d1, d2])
        return m >= 0, m


def pow_in_cone(x, y, z, a, tol):
    """x >= 0 and y >= 0 and x^a y^(1-a) >= |z| - tol"""
    if not (x >= 0 and y >= 0):
        return False, -INF
    with mpmath.workdps(DPS):
        A = _mp(a)
        m = float(_mp(x) ** A * _mp(y) ** (1 - A) - (abs(_mp(z)) - _mp(tol)))
        return m >= 0, m


def pow_in_dual(s, t, w, a, tol):
    """s >= -tol and t >= -tol and s^a t^(1-a) >= |w| a^a (1-a)^(1-a) - tol; a negative base in the band is
    "not in the cone" (a DomainError in the reference)"""
    if not (s >= -tol and t >= -tol) or s < 0 or t < 0:
        return False, -INF
    with mpmath.workdps(DPS):
        A = _mp(a)
        rhs = abs(_mp(w)) * A ** A * (1 - A) ** (1 - A) - _mp(tol)
        m = float(_mp(s) ** A * _mp(t) ** (1 - A) - rhs)
        return m >= 0, m


def c3_cert(v, typ, tol, alpha=0.0):
    """in_dual(-v) of the 3-d cone (support function and polar recession cone alike); the dual cones' in_dual is the
    primal cone's in_cone (convexset.jl:780)"""
    x, y, z = -float(v[0]), -float(v[1]), -float(v[2])
    if typ == EXP:
        return exp_in_dual(x, y, z, tol)
    if typ == DUAL_EXP:
        return exp_in_cone(x, y, z, tol)
    if typ == POW:
        return pow_in_dual(x, y, z, alpha, tol)
    return pow_in_cone(x, y, z, alpha, tol)


# ---- every family of a composite set --------------------------------------------------------------
def certificate(v, sets, tol, primal=True):
    """cone tests of is_primal_infeasible! (primal: v = -dy / |dy|) or is_dual_infeasible! (v = Einv A dx / |dx|) on
    the engine's set tuples (type, dim, l, u[, extra]).  Returns {"families": bitmask of failed families,
    "margins": {family: smallest margin}, "box_sum", "box_mag", "lam": [lambda_max per PSD cone]}."""
    fams, margins, lam = 0, {}, []
    box_terms_v, box_l, box_u = [], [], []
    off = 0
    for t in sets:
        typ, dim = int(t[0]), int(t[1])
        x = np.asarray(v[off:off + dim], dtype=np.float64)
        off += dim
        if typ in (ZERO, NONNEG, BOX):
            if typ == BOX and primal:
                box_terms_v.extend(x)
                box_l.extend(np.asarray(t[2], dtype=np.float64))
                box_u.extend(np.asarray(t[3], dtype=np.float64))
            elif not rows_ok(x, typ, tol, t[2], t[3], primal):
                fams |= FAMILY_ROWS
            continue
        if typ == SOC:
            ok, m, _ = soc_cert(x, tol)
            fam = FAMILY_SOC
        elif typ in PSD_TYPES:
            ok, m, lm, _ = psd_cert(x, typ, tol)
            lam.append(lm)
            fam = FAMILY_PSD
        else:
            alpha = (t[4] or {}).get("alpha", 0.0) if len(t) > 4 else 0.0
            ok, m = c3_cert(x, typ, tol, alpha)
            fam = FAMILY_C3
        margins[fam] = min(margins.get(fam, INF), m)
        if not ok:
            fams |= fam
    box_sum, box_mag = box_support(box_terms_v, box_l, box_u, tol) if box_terms_v else (0.0, 0.0)
    return {"families": fams, "margins": margins, "box_sum": box_sum, "box_mag": box_mag, "lam": lam}
