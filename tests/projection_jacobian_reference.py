"""An extended-precision reference of the projection Jacobian Dpi(w_s) h (cosmo_b200_project_jacobian, DESIGN.md §3k).

TEST INFRASTRUCTURE: the GPU tests compare the engine's sa_dpi with it, so it has to be more accurate than any kernel:
a failure then always points at the kernel.  tests/test_projection_jacobian_reference_cpu.py pins it against mpmath,
central differences of the oracle's projection and the fp64 restatement solve_adjoint_reference.dpi.

Arithmetic is double-double (a value is an unevaluated sum hi + lo of two doubles, about 106 bits), built from Dekker's
split and Knuth's TwoSum in vectorised NumPy: portable (np.longdouble differs between x86 and aarch64 hosts) and fast
enough for N = 257.  Products of double-double matrices are exact sums of fp64 matrix products of 21-bit slices (the
operands cut at per-row / per-column powers of two, so each slice product is exact in fp64 up to N = 2048).

  Rows       exact: h where w is strictly inside, 0 otherwise; 0 on ZeroSet rows.
  SOC        the closed form of DESIGN §3k in double-double on the exact input (w and h scaled by powers of two first).
  Real PSD   the fp64 eigh eigenpairs of mat(w) refined in double-double by Ogita-Aishima iterations (RefSyEv; pairs
             closer than the usual delta are orthonormalised only, and Dpi does not depend on the basis inside a cluster
             of one sign; eigenvalues within 1e-8 |W|_2 of each other are first rotated by an fp64 eigensolve of
             their block of Q'WQ less its mean, so the split inside such a cluster is only fp64 accurate),
             eigenvalues below 2^-80 |W|_2 taken as exact zeros, then Gamma, Q'HQ and Q (Gamma o .) Q'.
             A square cone is symmetrised first and last, as project! does.

Every cone's bar comes with its kappa = max(1, |W|_2 / min over pairs lam_i > 0 >= lam_j of (lam_i - lam_j))."""
import numpy as np

from oracle import cosmo_oracle as O

_SPLIT = 134217729.0                                   # 2^27 + 1
_RSQRT2 = (0.7071067811865476, -4.833646656726457e-17)  # 1 / sqrt 2 in double-double
_SQRT2 = (1.4142135623730951, -9.667293313452913e-17)
ZERO_EIG = 2.0 ** -80                                  # relative to |W|_2: an eigenvalue below it is an exact zero


# ---- double-double primitives: a value is a pair (hi, lo) of equal-shaped arrays -----------------------------------
def two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def fast_two_sum(a, b):
    s = a + b
    return s, b - (s - a)


def split(a):
    c = _SPLIT * a
    hi = c - (c - a)
    return hi, a - hi


def two_prod(a, b):
    p = a * b
    ah, al = split(a)
    bh, bl = split(b)
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def dd(a):
    a = np.asarray(a, dtype=np.float64)
    return a, np.zeros_like(a)


def add(x, y):
    s, e = two_sum(x[0], y[0])
    return fast_two_sum(s, e + x[1] + y[1])


def neg(x):
    return -x[0], -x[1]


def sub(x, y):
    return add(x, neg(y))


def mul(x, y):
    p, e = two_prod(x[0], y[0])
    return fast_two_sum(p, e + x[0] * y[1] + x[1] * y[0])


def div(x, y):
    q1 = x[0] / y[0]
    r = sub(x, mul(dd(q1), y))
    q2 = r[0] / y[0]
    r = sub(r, mul(dd(q2), y))
    return add(fast_two_sum(q1, q2), dd(r[0] / y[0]))


def sqrt(x):
    s = np.sqrt(x[0])
    with np.errstate(divide="ignore", invalid="ignore"):
        c = np.where(s > 0, sub(x, mul(dd(s), dd(s)))[0] / (2.0 * s), 0.0)
    return fast_two_sum(s, c)


def scale2(x, k):
    """x 2^k (exact)"""
    return np.ldexp(x[0], k), np.ldexp(x[1], k)


def total(x):
    """the sum of a 1-D double-double array, pairwise"""
    hi, lo = np.atleast_1d(x[0]).copy(), np.atleast_1d(x[1]).copy()
    if hi.size == 0:
        return 0.0, 0.0
    while hi.size > 1:
        if hi.size % 2:
            hi, lo = np.append(hi, 0.0), np.append(lo, 0.0)
        hi, lo = add((hi[0::2], lo[0::2]), (hi[1::2], lo[1::2]))
    return hi[0], lo[0]


def value(x):
    """hi + lo as one double"""
    return x[0] + x[1]


def _slices(x, axis, count=5, bits=21):
    """x = sum of the slices + O(2^-(count bits)) of the largest |x| along `axis`: each slice an integer of at most `bits`
    bits times a power of two per row (axis 1) or column (axis 0)"""
    hi, lo = x
    mx = np.max(np.abs(hi), axis=axis, keepdims=True)
    _, e = np.frexp(np.where(mx > 0, mx, 1.0))
    out = []
    for _ in range(count):
        S = np.ldexp(np.rint(np.ldexp(hi, bits - e)), e - bits)
        out.append(S)
        hi, lo = two_sum(hi - S, lo)
        e = e - bits
    return out


def matmul(A, B):
    """A B for double-double matrices: the exact fp64 products of their slices summed in double-double"""
    sa, sb = _slices(A, 1), _slices(B, 0)
    K = len(sa) - 1
    acc = None
    for k in range(K, -1, -1):                     # smallest terms first
        for i in range(k + 1):
            P = dd(sa[i] @ sb[k - i])
            acc = P if acc is None else add(acc, P)
    return acc


def transpose(A):
    return A[0].T.copy(), A[1].T.copy()


# ---- PSD ------------------------------------------------------------------------------------------------------------
def _svec_index(N):
    """(rows, cols) of the svec order: the upper triangle column by column"""
    iu = np.triu_indices(N)
    order = np.lexsort((iu[0], iu[1]))
    return iu[0][order], iu[1][order]


def psd_matrix(x, N, triangle):
    """mat(x) in double-double: the svec triangle unscaled by sqrt 2 off the diagonal, a square cone symmetrised"""
    x = np.asarray(x, dtype=np.float64)
    if triangle:
        r, c = _svec_index(N)
        off = r != c
        v = dd(x.copy())
        scaled = mul(dd(x[off]), (np.full(off.sum(), _RSQRT2[0]), np.full(off.sum(), _RSQRT2[1])))
        v[0][off], v[1][off] = scaled
        M = (np.zeros((N, N)), np.zeros((N, N)))
        for k in range(2):
            M[k][r, c] = v[k]
            M[k][c, r] = v[k]
        return M
    X = x.reshape(N, N, order="F")
    s = two_sum(X, X.T)
    return s[0] / 2.0, s[1] / 2.0


def psd_vector(M, triangle):
    """svec (sqrt 2 off the diagonal) or the column-major square of a symmetric double-double matrix"""
    if triangle:
        N = M[0].shape[0]
        r, c = _svec_index(N)
        v = (M[0][r, c].copy(), M[1][r, c].copy())
        off = r != c
        scaled = mul((v[0][off], v[1][off]), (np.full(off.sum(), _SQRT2[0]), np.full(off.sum(), _SQRT2[1])))
        v[0][off], v[1][off] = scaled
        return v
    return M[0].reshape(-1, order="F"), M[1].reshape(-1, order="F")


CLUSTER = 1e-8   # relative to |W|_2: eigenvalues this close are resolved inside their cluster first


def _resolve_clusters(X, S, lam, normA):
    """Rotate the columns of every cluster of nearly equal eigenvalues by the eigenvectors of its block of S = X'AX less
    its mean, formed in double-double: the split inside the cluster is then resolved to fp64 accuracy of its spread,
    and RefSyEv's corrections between its members stay small.  Returns (X, whether any cluster was rotated)."""
    order = np.argsort(lam, kind="stable")
    groups, cur = [], [order[0]]
    for a, b in zip(order[:-1], order[1:]):
        if lam[b] - lam[a] <= CLUSTER * normA:
            cur.append(b)
        else:
            groups.append(cur)
            cur = [b]
    groups.append(cur)
    rotated = False
    for g in groups:
        if len(g) < 2:
            continue
        g = np.array(g)
        Sc = (S[0][np.ix_(g, g)], S[1][np.ix_(g, g)])
        mean = np.mean(np.diag(Sc[0]))
        D = value(sub(Sc, dd(mean * np.eye(g.size))))
        _, V = np.linalg.eigh((D + D.T) / 2)
        Xc = matmul((X[0][:, g], X[1][:, g]), dd(V))
        X[0][:, g], X[1][:, g] = Xc
        rotated = True
    return X, rotated


def refsyev(A, iters=3):
    """Eigenpairs of the symmetric double-double matrix A: fp64 eigh, then `iters` Ogita-Aishima refinements.  Returns
    (lam, Q), both double-double, lam ascending."""
    N = A[0].shape[0]
    lam0, X = np.linalg.eigh(A[0])
    X = dd(X)
    I = dd(np.eye(N))
    normA = np.linalg.norm(A[0], 2)
    lam = dd(lam0)
    for _ in range(iters):
        XT = transpose(X)
        R = sub(I, matmul(XT, X))
        S = matmul(XT, matmul(A, X))
        X, rotated = _resolve_clusters(X, S, value(lam), normA)
        if rotated:
            XT = transpose(X)
            R = sub(I, matmul(XT, X))
            S = matmul(XT, matmul(A, X))
        lam = div((np.diag(S[0]).copy(), np.diag(S[1]).copy()), sub(dd(np.ones(N)), (np.diag(R[0]).copy(), np.diag(R[1]).copy())))
        Sv, Rv, lv = value(S), value(R), value(lam)
        Soff = Sv - np.diag(np.diag(Sv))
        delta = 2.0 * (np.linalg.norm(Soff, 2) + np.max(np.abs(np.diag(Sv) - lv)) + normA * np.linalg.norm(Rv, 2))
        delta = max(delta, ZERO_EIG * normA)     # the resolution of S and R: closer pairs stay one cluster
        gap = lv[None, :] - lv[:, None]                         # lam_j - lam_i
        sep = np.abs(gap) > delta
        with np.errstate(divide="ignore", invalid="ignore"):
            E = np.where(sep, (Sv + lv[None, :] * Rv) / np.where(sep, gap, 1.0), Rv / 2.0)
        X = add(X, matmul(X, dd(E)))
    order = np.argsort(value(lam), kind="stable")
    return (lam[0][order], lam[1][order]), (X[0][:, order], X[1][:, order])


def _snap(lam, normW):
    v = value(lam)
    z = np.abs(v) <= ZERO_EIG * normW
    return np.where(z, 0.0, lam[0]), np.where(z, 0.0, lam[1])


def gamma(lam):
    """Gamma_ij in double-double from double-double eigenvalues, in the branch forms of the kernels"""
    v = value(lam)
    N = v.size
    li = (np.repeat(lam[0][:, None], N, 1), np.repeat(lam[1][:, None], N, 1))
    lj = transpose(li)
    pi, pj = v[:, None] > 0, v[None, :] > 0
    mixed = pi != pj
    num = (np.where(pi, li[0], lj[0]), np.where(pi, li[1], lj[1]))          # lam_+
    den = sub(num, (np.where(pi, lj[0], li[0]), np.where(pi, lj[1], li[1])))  # lam_+ - lam_-
    den = (np.where(mixed, den[0], 1.0), np.where(mixed, den[1], 0.0))
    g = div(num, den)
    hi = np.where(mixed, g[0], np.where(pi & pj, 1.0, 0.0))
    lo = np.where(mixed, g[1], 0.0)
    return hi, lo


def kappa(lam, normW):
    """max(1, |W|_2 / min over pairs lam_i > 0 >= lam_j of (lam_i - lam_j))"""
    v = value(lam)
    pos, nonpos = v[v > 0], v[v <= 0]
    if pos.size == 0 or nonpos.size == 0 or normW == 0.0:
        return 1.0
    return max(1.0, normW / (pos.min() - nonpos.max()))


def psd_dd(w, h, N, triangle):
    """(Dpi h as double-double, kappa, lam as double-double, |H|_F) of one real PSD cone at w"""
    w, h = np.asarray(w, dtype=np.float64), np.asarray(h, dtype=np.float64)
    ew = _exponent(w)
    eh = _exponent(h)
    W = psd_matrix(np.ldexp(w, -ew), N, triangle)
    H = psd_matrix(np.ldexp(h, -eh), N, triangle)
    normW = np.linalg.norm(W[0], 2)
    lam, Q = refsyev(W)
    lam = _snap(lam, normW)
    C = matmul(transpose(Q), matmul(H, Q))
    C = mul(gamma(lam), C)
    X = matmul(Q, matmul(C, transpose(Q)))
    s = add(X, transpose(X))
    X = (s[0] / 2.0, s[1] / 2.0)
    out = scale2(psd_vector(X, triangle), eh)
    return out, kappa(lam, normW), scale2(lam, ew), np.ldexp(np.linalg.norm(H[0]), eh)


# ---- SOC ------------------------------------------------------------------------------------------------------------
def _exponent(x):
    """e with max |x| < 2^e (0 for a zero vector)"""
    mx = np.max(np.abs(x)) if np.size(x) else 0.0
    return int(np.frexp(mx)[1]) if mx > 0 else 0


def soc_dd(w, h):
    """Dpi h of one SOC (t, xbar) at w, double-double"""
    w, h = np.asarray(w, dtype=np.float64), np.asarray(h, dtype=np.float64)
    eh = _exponent(h)
    ws, hs = np.ldexp(w, -_exponent(w)), np.ldexp(h, -eh)
    t, x = ws[0], ws[1:]
    r = sqrt(total(two_prod(x, x)))
    rt = value(sub(r, dd(t)))                           # sign of r - t, exact enough to decide the branch
    rmt = value(add(r, dd(t)))                          # sign of r + t
    if rt <= 0.0:
        return scale2(dd(hs.copy()), eh)
    if rmt <= 0.0:
        return dd(np.zeros_like(h))
    d = total(two_prod(x, hs[1:]))
    dh = div(d, r)
    n = x.size
    rv = (np.full(n, r[0]), np.full(n, r[1]))
    xr = div(dd(x), rv)
    tr = div(dd(t), r)
    tr_v = (np.full(n, tr[0]), np.full(n, tr[1]))
    dh_v = (np.full(n, dh[0]), np.full(n, dh[1]))
    tail = add(add(mul(xr, dd(np.full(n, hs[0]))), mul(add(dd(np.ones(n)), tr_v), dd(hs[1:]))),
               neg(mul(mul(tr_v, xr), dh_v)))
    head = add(dd(hs[0]), dh)
    hi = np.concatenate([[head[0]], tail[0]]) / 2.0
    lo = np.concatenate([[head[1]], tail[1]]) / 2.0
    return scale2((hi, lo), eh)


# ---- every cone -----------------------------------------------------------------------------------------------------
def _psd_N(cone):
    if isinstance(cone, O.PsdConeTriangle):
        return int(round((np.sqrt(8 * cone.dim + 1) - 1) / 2))
    return int(round(np.sqrt(cone.dim)))


def _custom_jacobian(cone, w, h):
    ps = np.array(w, dtype=np.float64).copy()
    cone.project(ps, cone.params)
    return cone.jacobian(np.asarray(w, dtype=np.float64), ps, np.asarray(h, dtype=np.float64), cone.params)


def dpi(w, cones, h, info=None):
    """Dpi(w) h, cone by cone, rounded to fp64 from double-double.  `cones` are the oracle's cone objects; a custom cone
    with a NumPy `jacobian` (tests/custom_cone_jacobians.py) goes through it at Pi(w).  With `info` a list, one dict
    per cone is appended: its kind, rows and kappa (PSD)."""
    w, h = np.asarray(w, dtype=np.float64), np.asarray(h, dtype=np.float64)
    out = np.zeros_like(h)
    k = 0
    for cone in cones:
        d = cone.dim
        sl = slice(k, k + d)
        ws, hs = w[sl], h[sl]
        rec = {"rows": sl, "kappa": 1.0, "kind": type(cone).__name__}
        if isinstance(cone, O.ZeroSet):
            out[sl] = 0.0
        elif isinstance(cone, O.Nonnegatives):
            out[sl] = np.where(ws > 0, hs, 0.0)
        elif isinstance(cone, O.Box):
            out[sl] = np.where((ws > cone.l) & (ws < cone.u), hs, 0.0)
        elif isinstance(cone, O.SecondOrderCone):
            out[sl] = value(soc_dd(ws, hs))
        elif isinstance(cone, (O.PsdConeTriangle, O.PsdCone)):
            o, kap, _, _ = psd_dd(ws, hs, _psd_N(cone), isinstance(cone, O.PsdConeTriangle))
            out[sl] = value(o)
            rec["kappa"] = kap
        elif getattr(cone, "jacobian", None) is not None:
            out[sl] = _custom_jacobian(cone, ws, hs)
            rec["kind"] = "custom"
        else:
            raise TypeError("no Jacobian for %r" % (cone,))
        if info is not None:
            info.append(rec)
        k += d
    return out


# ---- bars and kink counts -------------------------------------------------------------------------------------------
def psd_bar(N, u, kap, normH):
    """|out - ref|_F of a PSD cone: 8 N u kappa |H|_F"""
    return 8.0 * N * u * kap * normH


def soc_bar(h, u):
    """|out - ref|_inf of a SOC: 64 u (|h_t| + |hbar|_2)"""
    h = np.asarray(h, dtype=np.float64)
    return 64.0 * u * (abs(h[0]) + np.linalg.norm(h[1:]))


def kink_band(a, u):
    """DESIGN's kink band 64 u (1 + |w_s|)"""
    return 64.0 * u * (1.0 + a)


def kink_counts(w, cones, u):
    """(rows, SOC cones, PSD cones) within the kink band: Nonnegatives |w| <= band(|w|), Box |w - l| or |w - u| <=
    band(|w|), SOC | |xbar| - |t| | <= band(max(|t|, |xbar|)), PSD an eigenvalue within band(max |w_s| of the cone)"""
    w = np.asarray(w, dtype=np.float64)
    rows = soc = psd = 0
    k = 0
    for cone in cones:
        ws = w[k:k + cone.dim]
        band = kink_band(np.abs(ws), u)
        if isinstance(cone, O.Nonnegatives):
            rows += int(np.sum(np.abs(ws) <= band))
        elif isinstance(cone, O.Box):
            with np.errstate(invalid="ignore"):
                rows += int(np.sum((np.abs(ws - cone.l) <= band) | (np.abs(ws - cone.u) <= band)))
        elif isinstance(cone, O.SecondOrderCone):
            t, r = abs(ws[0]), np.linalg.norm(ws[1:])
            soc += int(abs(r - t) <= kink_band(max(t, r), u))
        elif isinstance(cone, (O.PsdConeTriangle, O.PsdCone)):
            N = _psd_N(cone)
            tri = isinstance(cone, O.PsdConeTriangle)
            e = _exponent(ws)
            lam = np.ldexp(np.linalg.eigvalsh(value(psd_matrix(np.ldexp(ws, -e), N, tri))), e)
            psd += int(np.any(np.abs(lam) <= kink_band(np.max(np.abs(ws)), u)))
        k += cone.dim
    return rows, soc, psd
