"""An extended-precision restatement of the device Anderson accelerator (csrc/aa.cuh, cosmo_b200_accelerator_probe).

The definitions are those of oracle.cosmo_oracle.AndersonAccelerator (Type2{QRDecomp}) and
tests/anderson_variants.NormalEquationsAccelerator (Type2{NormalEquations}, Type1, the regularisers and both memories);
nothing here is new.  What differs is the arithmetic: every input value (the fp64 or fp32 g_k and x_k the device
receives) is taken exactly, so f = x - g and the history columns F, G, X are exact, and their inner products are formed
exactly in integers.  The l x l algebra then runs in mpmath at 50 significant digits:
  * Type2{QRDecomp}: the R of modified Gram-Schmidt on F, which in exact arithmetic is the Cholesky factor of F'F with a
    positive diagonal, the right-hand side Q'f = R^-T F'f and the back substitution R eta = Q'f.  A zero diagonal of R
    turns the Q column of that step into 0/0, as on the device: every later R column of the memory cycle is then NaN.
  * Type2{NormalEquations} and Type1: M = A'B with (A, B) = (F, F) or (X, F), rhs = A'f, in physical column order,
    the shift lambda (Tikonov) or lambda (|A|_F^2 + |B|_F^2) over the window (Frobenius), and LU with partial pivoting
    by the first largest |pivot|.  lambda is the value of the device's type T.
  * RestartedMemory starts again at column 0 when the memory is full, RollingMemory overwrites column iter mod mem.
  * The acceptance rules: no candidate while l < min_mem; rejected on a non-finite entry of the system (normal
    equations), a zero or non-finite pivot, a non-finite eta or |eta|_2 > 1e4.
Beside eta and the candidate g - G eta, each formed step reports the rule that rejected it, the exact least-squares
minimiser of |f - F eta|, the condition numbers of F[:, :l] and of the system solved, and the norms the error bars of
tests/test_gpu_anderson.py need.  Rows where every g_k and x_k is zero take no part in any sum, so they are skipped;
their candidate entries are zero."""
from fractions import Fraction
from operator import mul

import mpmath
import numpy as np

DPS = 50
TYPES = ("Type2{QRDecomp}", "Type2{NormalEquations}", "Type1")
REASONS = ("accepted", "nonfinite_entry", "zero_pivot", "nonfinite_pivot", "nonfinite_eta", "eta_norm")


def _ctx():
    ctx = mpmath.mp.clone()
    ctx.dps = DPS
    return ctx


def _to_ints(a):
    """(ints, E): the finite float array `a` as Python ints n with a = n 2^E exactly, one common E"""
    a = np.asarray(a, dtype=np.float64)
    m, e = np.frexp(a)
    mi = (m * 2.0 ** 53).astype(np.int64)
    e = e.astype(np.int64) - 53
    nz = mi != 0
    E = int(e[nz].min()) if nz.any() else 0
    sh = np.where(nz, e - E, 0)
    return [int(v) << int(s) for v, s in zip(mi.ravel(), sh.ravel())], E


class Step:
    """what one update + accelerate of the restatement gives"""
    formed = False
    accepted = False
    reason = None
    l = 0
    j = -1
    eta = None          # list of l mpf, physical column order
    cand = None         # float64 array of dim (the exact candidate rounded once)
    ties = 0            # pivot columns of the LU with two rows of equal largest |value|
    pivots = None       # pivot rows of the LU (normal equations)


class Reference:
    """the accelerator of one engine: dim, mem (before min(mem, dim)), min_mem and the variant, on inputs of `dtype`"""

    def __init__(self, dim, mem=15, min_mem=3, type="Type2{QRDecomp}", memory="RestartedMemory",
                 regularizer="NoRegularizer", lam=1e-8, dtype=np.float64):
        if mem <= 2:
            raise ValueError("Memory has to be bigger than two.")
        self.dim, self.mem, self.min_mem = dim, min(mem, max(dim, 1)), min_mem
        self.type, self.rolling, self.reg = type, memory == "RollingMemory", regularizer
        self.lam = float(np.dtype(dtype).type(lam))
        self.dtype = np.dtype(dtype)
        self.ctx = _ctx()

    # ---- one sequence -------------------------------------------------------------------------------------------
    def run(self, g, x, solve_at=None):
        """the steps of update(g[k], x[k]) + accelerate on K pairs (K x dim arrays of self.dtype values), from a
        restart.  `solve_at`: the steps whose system is solved (None: every formed step); the bookkeeping of the others
        (formed, l, j) is still given."""
        g = np.asarray(g, dtype=np.float64).reshape(-1, self.dim)
        x = np.asarray(x, dtype=np.float64).reshape(-1, self.dim)
        K = g.shape[0]
        rows = np.flatnonzero(np.any(g != 0, axis=0) | np.any(x != 0, axis=0))
        self.rows = rows
        gs, xs = g[:, rows], x[:, rows]
        fin_g, fin_x = np.isfinite(gs), np.isfinite(xs)
        gi, E = _to_ints(np.where(np.isfinite(np.concatenate([gs, xs])), np.concatenate([gs, xs]), 0.0))
        r = rows.size
        self.E = E
        G_int = [gi[k * r:(k + 1) * r] for k in range(K)]
        X_int = [gi[(K + k) * r:(K + k + 1) * r] for k in range(K)]
        self.bad_step = [not (np.all(fin_g[k]) and np.all(fin_x[k])) for k in range(K)]
        self._restart()
        out = []
        for k in range(K):
            f = [a - b for a, b in zip(X_int[k], G_int[k])]
            out.append(self._step(k, G_int[k], X_int[k], f, solve_at is None or k in solve_at))
        return out

    def _restart(self):
        m = self.mem
        self.iter, self.init = 0, True
        self.cols = [None] * m            # (F, G, X) int columns, physical order
        self.bad = [False] * m            # column holds a non-finite value
        self.AB = [[0] * m for _ in range(m)]   # exact <A_i, B_c> of the stored columns (A = X for Type1, else F; B = F)
        self.nA, self.nB = [0] * m, [0] * m
        self.R = [[None] * m for _ in range(m)]  # QR: R of the current memory cycle
        self.last = None
        self.poison = False               # QR: a zero or non-finite R diagonal earlier in this memory cycle

    def _dot(self, a, b):
        return sum(map(mul, a, b))

    def _mpf2(self, n):
        """the int inner product n (scaled by 2^(2E)) as an mpf"""
        return self.ctx.ldexp(self.ctx.mpf(n), 2 * self.E)

    def _a(self, c):
        return self.cols[c][2] if self.type == "Type1" else self.cols[c][0]

    def _step(self, k, g, x, f, solve):
        st = Step()
        bad_now = self.bad_step[k]
        if self.init:
            self.last = (g, x, f, bad_now)
            self.init = False
            return st
        j = self.iter % self.mem
        if not self.rolling and j == 0 and self.iter != 0:
            self.iter = 0
            self.poison = False
        gl, xl, fl, bad_last = self.last
        self.cols[j] = ([a - b for a, b in zip(f, fl)], [a - b for a, b in zip(g, gl)], [a - b for a, b in zip(x, xl)])
        self.bad[j] = bad_now or bad_last
        self.last = (g, x, f, bad_now)
        self.iter += 1
        if self.iter >= 2 * self.mem:
            self.iter -= self.mem
        l = min(self.iter, self.mem)
        st.l, st.j = l, j
        self.f, self.f_bad = f, bad_now
        for c in range(self.mem):        # row and column j of the exact Gram data (the window is [0, l))
            if self.cols[c] is None:
                continue
            self.AB[j][c] = self._dot(self._a(j), self.cols[c][0])
            self.AB[c][j] = self._dot(self._a(c), self.cols[j][0])
        self.nA[j] = self._dot(self._a(j), self._a(j))
        self.nB[j] = self._dot(self.cols[j][0], self.cols[j][0])
        if self.type == "Type2{QRDecomp}":
            self._qr_column(j)
        if l < max(self.min_mem, 1):
            return st
        st.formed = True
        if not solve:
            return st
        if self.type == "Type2{QRDecomp}":
            self._solve_qr(st, l)
        else:
            self._solve_ne(st, l)
        if st.accepted:
            st.cand = self._candidate(st.eta, l)
        return st

    # ---- Type2{QRDecomp} --------------------------------------------------------------------------------------
    def _qr_column(self, j):
        """column j of R (MGS in exact arithmetic = the Cholesky factor of F'F, positive diagonal).  A non-finite
        column or a zero diagonal poisons the rest of the memory cycle, as Q[:, j] = 0/0 does on the device."""
        ctx, R = self.ctx, self.R
        if self.poison or self.bad[j]:
            self.poison = True
            return
        for i in range(j):
            R[i][j] = (self._mpf2(self.AB[i][j]) - ctx.fsum(R[p][i] * R[p][j] for p in range(i))) / R[i][i]
        d = self._mpf2(self.AB[j][j]) - ctx.fsum(R[p][j] ** 2 for p in range(j))
        if d <= 0:
            self.poison = True
            R[j][j] = ctx.mpf(0)
            return
        R[j][j] = ctx.sqrt(d)

    def _solve_qr(self, st, l):
        ctx, R = self.ctx, self.R
        if self.poison:
            st.reason = "zero_pivot"       # a zero (or, from a non-finite column, NaN) diagonal stays in R[:l, :l]
            return
        if self.f_bad:
            st.reason = "nonfinite_eta"
            return
        rhs = [self._mpf2(self._dot(self.cols[c][0], self.f)) for c in range(l)]
        qtf = [ctx.mpf(0)] * l                 # R' qtf = F'f
        for i in range(l):
            qtf[i] = (rhs[i] - ctx.fsum(R[p][i] * qtf[p] for p in range(i))) / R[i][i]
        eta = [ctx.mpf(0)] * l
        for i in range(l - 1, -1, -1):
            eta[i] = (qtf[i] - ctx.fsum(R[i][p] * eta[p] for p in range(i + 1, l))) / R[i][i]
        self._accept(st, eta)

    # ---- Type2{NormalEquations}, Type1 ---------------------------------------------------------------------------
    def system(self, l):
        """(M + shift I, rhs, shift) of the window, mpf, physical order"""
        ctx = self.ctx
        M = [[self._mpf2(self.AB[i][c]) for c in range(l)] for i in range(l)]
        rhs = [self._mpf2(self._dot(self._a(c), self.f)) for c in range(l)]
        shift = ctx.mpf(0)
        if self.reg == "TikonovRegularizer":
            shift = ctx.mpf(self.lam)
        elif self.reg == "FrobeniusNormRegularizer":
            shift = ctx.mpf(self.lam) * self._mpf2(sum(self.nA[:l]) + sum(self.nB[:l]))
        for i in range(l):
            M[i][i] += shift
        return M, rhs, shift

    def _solve_ne(self, st, l):
        ctx = self.ctx
        if any(self.bad[:l]) or self.f_bad:
            st.reason = "nonfinite_entry"
            return
        S, b, _ = self.system(l)
        st.pivots = []
        for k in range(l):
            best, p = -1, k
            for r in range(k, l):
                v = abs(S[r][k])
                if v > best:
                    best, p = v, r
            st.ties += sum(1 for r in range(k, l) if r != p and abs(S[r][k]) == best and S[r][k] != S[p][k])
            st.pivots.append(p)
            if S[p][k] == 0:
                st.reason = "zero_pivot"
                return
            if p != k:
                S[k], S[p] = S[p], S[k]
                b[k], b[p] = b[p], b[k]
            for r in range(k + 1, l):
                fct = S[r][k] / S[k][k]
                S[r][k] = fct
                for c in range(k + 1, l):
                    S[r][c] -= fct * S[k][c]
                b[r] -= fct * b[k]
        eta = [ctx.mpf(0)] * l
        for i in range(l - 1, -1, -1):
            eta[i] = (b[i] - ctx.fsum(S[i][c] * eta[c] for c in range(i + 1, l))) / S[i][i]
        self._accept(st, eta)

    def _accept(self, st, eta):
        ctx = self.ctx
        if not all(ctx.isfinite(e) for e in eta):
            st.reason = "nonfinite_eta"
            return
        if ctx.sqrt(ctx.fsum(e * e for e in eta)) > 10000:
            st.reason = "eta_norm"
            st.eta = eta
            return
        st.accepted, st.reason, st.eta = True, "accepted", eta

    def _candidate(self, eta, l):
        """g - G eta over all dim rows, rounded once to float64"""
        ctx = self.ctx
        out = np.zeros(self.dim)
        gl = self.last[0]
        Gc = [self.cols[c][1] for c in range(l)]
        vals = []
        for i in range(len(self.rows)):
            v = ctx.ldexp(ctx.mpf(gl[i]), self.E) - ctx.fsum(ctx.ldexp(ctx.mpf(Gc[c][i]), self.E) * eta[c] for c in range(l))
            vals.append(float(v))
        out[self.rows] = vals
        return out

    # ---- what the error bars need --------------------------------------------------------------------------------
    def analysis(self, st):
        """for the step just run (formed, finite data): the exact least-squares minimiser of |f - F eta| (physical
        order), kappa_2 of F[:, :l] and of the system solved, and the norms of the error bars, as floats.  The norms of
        matrices are Frobenius norms (F also its 2-norm), the inverse of the system its Frobenius norm, a bound of the
        2-norm."""
        ctx, l = self.ctx, st.l
        F = [self.cols[c][0] for c in range(l)]
        FtF = ctx.matrix([[self._mpf2(self._dot(a, b)) for b in F] for a in F])
        Ftf = ctx.matrix([self._mpf2(self._dot(a, self.f)) for a in F])
        out = {}
        try:
            # the singular values of R (Cholesky of the exact F'F at 50 digits), rounded to fp64: their absolute error
            # is 1e-16 |F|, so kappa_F is resolved to a relative 1e-16 kappa_F
            Rf = np.array(ctx.cholesky(FtF).tolist(), dtype=float)
            sv = np.linalg.svd(Rf, compute_uv=False)
            out["kappa_F"], out["nrm_F"] = float(sv[0] / sv[-1]) if sv[-1] > 0 else np.inf, float(sv[0])
            out["eta_ls"] = [float(v) for v in ctx.cholesky_solve(FtF, Ftf)]
        except (ValueError, ZeroDivisionError):
            out["kappa_F"], out["nrm_F"], out["eta_ls"] = np.inf, float(ctx.sqrt(sum(FtF[i, i] for i in range(l)))), None
        nf2 = self._mpf2(self._dot(self.f, self.f))
        out["nrm_f"] = float(ctx.sqrt(nf2))
        out["nrm_A"] = float(ctx.sqrt(self._mpf2(sum(self.nA[:l]))))
        out["nrm_B"] = float(ctx.sqrt(self._mpf2(sum(self.nB[:l]))))
        out["nrm_G"] = float(ctx.sqrt(self._mpf2(sum(self._dot(self.cols[c][1], self.cols[c][1]) for c in range(l)))))
        out["nrm_g"] = float(ctx.sqrt(self._mpf2(self._dot(self.last[0], self.last[0]))))
        if st.eta is not None:
            eta = ctx.matrix(st.eta)
            out["nrm_eta"] = float(ctx.norm(eta))
            r2 = nf2 - 2 * (eta.T * Ftf)[0] + (eta.T * FtF * eta)[0]      # |f - F eta|^2
            out["nrm_r"] = float(ctx.sqrt(max(r2, 0)))
        if self.type != "Type2{QRDecomp}":
            M, _, shift = self.system(l)
            Mm = ctx.matrix(M)
            try:
                inv = ctx.inverse(Mm)
                out["inv_sys"] = float(ctx.mnorm(inv, "F"))
                out["kappa_sys"] = float(ctx.mnorm(Mm, "F") * out["inv_sys"])
            except ZeroDivisionError:
                out["inv_sys"] = out["kappa_sys"] = np.inf
            out["shift"] = float(shift)
        else:
            out["kappa_sys"] = out["kappa_F"]
        return out


def exact_lu_eta(M, rhs):
    """eta of M eta = rhs by LU with the first-largest pivot rule in exact rationals (M, rhs of ints or Fractions):
    None on a zero pivot.  The small cases of tests/test_anderson_reference_cpu.py pin the restatement to it."""
    S = [[Fraction(v) for v in row] for row in M]
    b = [Fraction(v) for v in rhs]
    l = len(b)
    for k in range(l):
        p = max(range(k, l), key=lambda r: (abs(S[r][k]), -r))
        if S[p][k] == 0:
            return None
        S[k], S[p] = S[p], S[k]
        b[k], b[p] = b[p], b[k]
        for r in range(k + 1, l):
            fct = S[r][k] / S[k][k]
            for c in range(k, l):
                S[r][c] -= fct * S[k][c]
            b[r] -= fct * b[k]
    eta = [Fraction(0)] * l
    for i in range(l - 1, -1, -1):
        eta[i] = (b[i] - sum(S[i][c] * eta[c] for c in range(i + 1, l))) / S[i][i]
    return eta


def sequence(dim, K, kappa=1.0, dtype=np.float64, seed=0, rank=None, support=None, resid=1e-3):
    """K pairs (g_k, x_k) (K x dim arrays of `dtype`) whose history differences F_j = f_j - f_{j-1} lie in the span of
    `rank` orthonormal directions scaled by logspace(0, -log10 kappa): every window of F has a condition number near
    kappa.  f_0 is orthogonal to that span with norm `resid` (the least-squares residual), the G differences are
    independent, x_k = f_k + g_k.  `support`: the rows that carry values (all by default); the others stay zero."""
    rng = np.random.default_rng(seed)
    rows = np.arange(dim) if support is None else np.asarray(support)
    d = rows.size
    r = max(1, min(rank or d, d))
    U, _ = np.linalg.qr(rng.standard_normal((d, d)))
    s = np.logspace(0, -np.log10(kappa), r) if r > 1 else np.ones(1)
    if K - 1 == r:      # the one full window: F = U S V' with V orthogonal, kappa(F) = kappa exactly before rounding
        V, _ = np.linalg.qr(rng.standard_normal((r, r)))
        D = np.concatenate([np.zeros((d, 1)), (U[:, :r] * s) @ V.T], axis=1)
    else:
        D = (U[:, :r] * s) @ rng.standard_normal((r, K))
    f0 = U[:, r:] @ rng.standard_normal(d - r) if r < d else np.zeros(d)
    if r < d:
        f0 *= resid / max(np.linalg.norm(f0), 1e-300)
    f = f0[:, None] + np.cumsum(D, axis=1)
    gg = rng.standard_normal((d, 1)) + np.cumsum(rng.standard_normal((d, K)), axis=1)
    g = np.zeros((K, dim), dtype=dtype)
    x = np.zeros((K, dim), dtype=dtype)
    g[:, rows] = gg.T.astype(dtype)
    x[:, rows] = (f + gg).T.astype(dtype)
    return g, x


def from_columns(F, G, f_last, g0=None, dtype=np.float64):
    """the pairs whose history differences are exactly the columns of F and G (dim x l) and whose last f is f_last,
    for integer-valued designs where every sum is exact: f_0 = f_last - sum F, g_0 = g0 (zero), x = f + g"""
    F, G = np.asarray(F, dtype=float), np.asarray(G, dtype=float)
    dim, l = F.shape
    f = np.asarray(f_last, dtype=float) - F.sum(axis=1)
    g = np.zeros(dim) if g0 is None else np.asarray(g0, dtype=float)
    gs, xs = [g.copy()], [f + g]
    for c in range(l):
        f, g = f + F[:, c], g + G[:, c]
        gs.append(g.copy())
        xs.append(f + g)
    out = np.array(gs).astype(dtype), np.array(xs).astype(dtype)
    assert np.array_equal(out[1].astype(float) - out[0].astype(float), np.array(xs) - np.array(gs)), "design not exact"
    return out
