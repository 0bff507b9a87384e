"""CPU restatement of the Anderson accelerator variants beside the default one (csrc/aa.cuh, cosmo_b200_set_accelerator).

COSMOAccelerators.jl is not part of the reference tree, so -- like oracle.cosmo_oracle.AndersonAccelerator -- this is
a restatement from the published methods and PARITY WITH THE PACKAGE IS UNPINNED:
  * Type2{NormalEquations}: type-II Anderson acceleration (Walker & Ni, "Anderson acceleration for fixed-point
    iterations", 2011) with the least squares min |f - F eta| solved through the normal equations F'F eta = F'f.
  * Type1: type-I Anderson acceleration X'F eta = X'f and its Frobenius-norm regularisation (Fu, Zhang & Boyd,
    "Anderson accelerated Douglas-Rachford splitting", 2020).
  * the safeguard, restarts on rho adaptation and the call sites: Garstka, Cannon & Goulart 2022 and
    accelerator_interface.jl:1-130, solver.jl:272-275, residuals.jl:129 of the reference.
Choices written down here (the engine makes the same ones):
  * f = x - g with g = w = T(w_prev), x = w_prev; history columns X_j = x - x_last, F_j = f - f_last, G_j = g - g_last,
    G stored as its own difference (not as X - F).  After a restart the first update only stores (x, g, f).
  * M = A'B with (A, B) = (F, F) for Type2{NormalEquations} and (X, F) for Type1, rhs = A'f, in physical column order.
    A new column j refreshes row j and column j of M against the current window of l = min(iter, mem) columns.
  * regularisers: Tikonov M + lambda I; FrobeniusNorm M + lambda (|A|_F^2 + |B|_F^2) I over the window.  The package
    default lambda is remembered as 1e-8 but unverified; 1e-8 is the value used (Settings.accelerator_lambda).
  * the system is solved by LU with partial pivoting (first row of largest |pivot|).  The candidate g - G eta is
    rejected when an entry of the system is not finite, a pivot is zero or not finite, eta is not finite or
    |eta|_2 > 1e4 (the rules of the QR variant), and when l < min_mem no candidate is formed.
  * RollingMemory overwrites column iter mod mem and never clears; RestartedMemory starts again at column 0 when the
    memory is full (logged as memory_full).  rho adaptation restarts every variant.
  * activation (accelerator_interface.jl:1-48): ImmediateActivation from iteration 2, IterActivation(k) once
    iter >= k (any k is accepted, as the reference's constructor never throws), AccuracyActivation(tol) after the first
    termination check with r_prim < tol + tol max_norm_prim and r_dual < tol + tol max_norm_dual.
"""
import numpy as np

from oracle import cosmo_oracle as O

# anderson_accelerator.jl:5-19, as (type, memory, regularizer) of cosmo_b200.Settings
TYPES = [(t, mem, reg) for t in ("Type1", "Type2{NormalEquations}") for reg in ("NoRegularizer", "TikonovRegularizer",
         "FrobeniusNormRegularizer") for mem in ("RollingMemory", "RestartedMemory")] + \
        [("Type2{QRDecomp}", "RestartedMemory", "NoRegularizer")]


def variant(t, mem, reg, activation="ImmediateActivation", lam=1e-8):
    """the Settings keywords of one AndersonAccelerator{Float64, t, mem, reg} with an activation reason"""
    return dict(accelerator_type=t, accelerator_memory=mem, accelerator_regularizer=reg, accelerator_lambda=lam,
                accelerator_activation=activation)


def lu_solve(M, rhs):
    """M eta = rhs by LU with partial pivoting; None when the candidate is rejected (see the module header)."""
    S = np.array(M, dtype=float)
    b = np.array(rhs, dtype=float)
    l = b.shape[0]
    if not (np.all(np.isfinite(S)) and np.all(np.isfinite(b))):
        return None
    for k in range(l):
        col = np.abs(S[k:, k])
        col = np.where(np.isnan(col), np.inf, col)
        p = k + int(np.argmax(col))
        piv = S[p, k]
        if piv == 0.0 or not np.isfinite(piv):
            return None
        if p != k:
            S[[k, p]] = S[[p, k]]
            b[[k, p]] = b[[p, k]]
        for r in range(k + 1, l):
            fct = S[r, k] / S[k, k]
            S[r, k] = fct
            S[r, k + 1:] -= fct * S[k, k + 1:]
            b[r] -= fct * b[k]
    eta = np.zeros(l)
    with np.errstate(all="ignore"):
        for i in range(l - 1, -1, -1):
            eta[i] = (b[i] - S[i, i + 1:] @ eta[i + 1:]) / S[i, i]
        nrm = np.linalg.norm(eta)
    if not np.isfinite(nrm) or nrm > 1e4:
        return None
    return eta


class NormalEquationsAccelerator:
    """AndersonAccelerator{T, Type2{NormalEquations} | Type1, RollingMemory | RestartedMemory, regularizer}(dim; mem)."""

    def __init__(self, dim, mem=15, min_mem=3, type1=False, rolling=False, regularizer="NoRegularizer", lam=1e-8):
        if mem <= 2:
            raise ValueError("Memory has to be bigger than two.")
        self.dim, self.mem, self.min_mem = dim, min(mem, dim), min_mem
        self.type1, self.rolling, self.regularizer, self.lam = type1, rolling, regularizer, lam
        self.X = np.zeros((dim, self.mem)) if type1 else None
        self.F = np.zeros((dim, self.mem))
        self.G = np.zeros((dim, self.mem))
        self.M = np.zeros((self.mem, self.mem))
        self.nrmA = np.zeros(self.mem)
        self.nrmB = np.zeros(self.mem)
        self.x_last, self.g_last = np.zeros(dim), np.zeros(dim)
        self.f, self.f_last = np.zeros(dim), np.zeros(dim)
        self.eta = np.zeros(self.mem)
        self.iter, self.j = 0, 0
        self.init_phase, self.fresh, self.success = True, False, False
        self.num_accelerated_steps = 0
        self.log = []

    def restart(self):
        self.iter = 0
        self.init_phase = True
        self.fresh = False

    def update(self, g, x, num_iter):
        self.f[:] = x - g
        if self.init_phase:
            self.x_last[:], self.g_last[:], self.f_last[:] = x, g, self.f
            self.init_phase, self.fresh = False, False
            return
        j = self.iter % self.mem
        if not self.rolling and j == 0 and self.iter != 0:
            self.iter = 0
            self.log.append((num_iter, "memory_full"))
        self.G[:, j] = g - self.g_last
        self.F[:, j] = self.f - self.f_last
        if self.type1:
            self.X[:, j] = x - self.x_last
        self.x_last[:], self.g_last[:], self.f_last[:] = x, g, self.f
        self.j = j
        self.iter += 1
        if self.iter >= 2 * self.mem:   # keeps iter mod mem and min(iter, mem)
            self.iter -= self.mem
        self.fresh = True

    def system(self, l):
        """(M + shift I)[0:l, 0:l] of the current window"""
        M = self.M[:l, :l].copy()
        if self.regularizer == "TikonovRegularizer":
            M += self.lam * np.eye(l)
        elif self.regularizer == "FrobeniusNormRegularizer":
            M += self.lam * (self.nrmA[:l].sum() + self.nrmB[:l].sum()) * np.eye(l)
        return M

    def accelerate(self, g, x, num_iter):
        self.success = False
        if not self.fresh:
            return
        self.fresh = False
        l, j = min(self.iter, self.mem), self.j
        A = self.X if self.type1 else self.F
        B = self.F
        self.M[:l, j] = A[:, :l].T @ B[:, j]
        self.M[j, :l] = A[:, j] @ B[:, :l]
        self.nrmA[j] = A[:, j] @ A[:, j]
        self.nrmB[j] = B[:, j] @ B[:, j]
        rhs = A[:, :l].T @ self.f
        if l < max(self.min_mem, 1):
            return
        eta = lu_solve(self.system(l), rhs)
        if eta is None:
            self.log.append((num_iter, "acc_failed"))
            return
        self.eta[:l] = eta
        g -= self.G[:, :l] @ eta
        self.num_accelerated_steps += 1
        self.success = True


class Activated:
    """An accelerator behind an activation reason: update!/accelerate! reach it only once it is active."""

    def __init__(self, aa, reason="ImmediateActivation"):
        self.aa = aa
        self.kind, self.arg = (reason, None) if isinstance(reason, str) else tuple(reason)
        self.active, self.activated_at, self.last_iter = False, 0, 0

    def __getattr__(self, name):
        return getattr(self.aa, name)

    def restart(self):
        self.aa.restart()

    def update(self, g, x, num_iter):   # acceleration_pre! -> check_activation!(ws, reason, num_iter)
        self.last_iter = num_iter
        if not self.active and ((self.kind == "ImmediateActivation" and num_iter >= 2) or
                                (self.kind == "IterActivation" and num_iter >= self.arg)):
            self.active, self.activated_at = True, num_iter
        if self.active:
            self.aa.update(g, x, num_iter)

    def accelerate(self, g, x, num_iter):
        if self.active:
            self.aa.accelerate(g, x, num_iter)

    def check_accuracy(self, r):        # has_converged -> check_activation!(ws, reason, r)
        if self.kind == "AccuracyActivation" and not self.active:
            tol = self.arg
            if r.r_prim < tol + tol * r.max_norm_prim and r.r_dual < tol + tol * r.max_norm_dual:
                self.active, self.activated_at = True, self.last_iter


class Workspace(O.Workspace):
    """The oracle workspace with an accelerator variant (keywords of `variant`) and its activation reason."""

    def __init__(self, P, q, A, b, cones, settings: O.Settings, **var):
        super().__init__(P, q, A, b, cones, settings)
        self.var = variant(*TYPES[-1]) if not var else dict(variant(*TYPES[-1]), **var)

    def setup(self):
        fresh = self.kkt is None
        super().setup()
        st, v = self.st, self.var
        if st.accelerator != "anderson":
            return
        if fresh:
            if v["accelerator_type"] == "Type2{QRDecomp}":
                aa = self.accelerator
            else:
                aa = NormalEquationsAccelerator(self.n + self.m, st.accelerator_mem, st.accelerator_min_mem,
                                                type1=v["accelerator_type"] == "Type1",
                                                rolling=v["accelerator_memory"] == "RollingMemory",
                                                regularizer=v["accelerator_regularizer"], lam=v["accelerator_lambda"])
            self.accelerator = Activated(aa, v["accelerator_activation"])
        self.accelerator.active = False     # ws.accelerator_active = false (setup.jl:47-49)
        self.accelerator_active = True      # the activation reason decides, inside Activated

    def has_converged(self, r):
        if isinstance(self.accelerator, Activated):
            self.accelerator.check_accuracy(r)
        return super().has_converged(r)


def stats(ws):
    """the counters of cosmo_b200_accelerator_stats, from the accelerator's log"""
    aa = ws.accelerator
    count = lambda ev: sum(1 for e in aa.log if e[1] == ev)
    return {"accepted": aa.num_accelerated_steps, "declined": count("acc_guarded_declined"), "rejected": count("acc_failed"),
            "rho_restarts": count("rho_adapted"), "memory_restarts": count("memory_full"), "activated_at": aa.activated_at}


def solve(P, q, A, b, cones, settings: O.Settings, x0=None, s0=None, y0=None, **var):
    """(Result, Workspace) of one accelerated oracle solve with the variant `var`"""
    ws = Workspace(P, q, A, b, cones, settings, **var)
    ws.warm_start(x0, s0, y0)
    return ws.optimize(), ws
