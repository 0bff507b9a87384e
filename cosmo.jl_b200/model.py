"""Host-side mirror of COSMO.jl's native API for the accelerated path.

Same names, argument meaning and error behaviour as the reference's
``COSMO.Model`` / ``COSMO.Constraint`` / ``assemble!`` / ``optimize!`` /
``warm_start_*!`` / ``update!`` (src/interface.jl, src/constraint.jl,
src/solver.jl:78-203), so that parity tests read like the reference's own.
Everything here is model building and the `setup!` / `reverse_scaling!` glue
that stays on the host in the reference too; the ADMM loop itself is
``cosmo_b200_solve`` in the CUDA library (engine.py).  Julia is not available in
this image, which is why this mirror is Python: INTEGRATION.md shows the
~100-line Julia shim that replaces it in a real deployment.
"""
from __future__ import annotations

import math
import time
from dataclasses import dataclass, field
from typing import List, Optional, Sequence, Tuple, Union

import numpy as np
import scipy.sparse as sp

from . import engine as _eng


# ---------------------------------------------------------------------------
# convex sets (src/convexset.jl)
# ---------------------------------------------------------------------------
class AbstractConvexSet:
    dim: int


class ZeroSet(AbstractConvexSet):
    """COSMO.ZeroSet(dim), convexset.jl:16-23."""
    code = _eng.ZERO

    def __init__(self, dim):
        if dim < 0:
            raise ValueError("dimension must be nonnegative")
        self.dim = int(dim)


class Nonnegatives(AbstractConvexSet):
    """COSMO.Nonnegatives(dim), convexset.jl:52-60."""
    code = _eng.NONNEG

    def __init__(self, dim):
        if dim < 0:
            raise ValueError("dimension must be nonnegative")
        self.dim = int(dim)


class Box(AbstractConvexSet):
    """COSMO.Box(l, u), convexset.jl:803-830."""
    code = _eng.BOX

    def __init__(self, l, u):
        self.l = np.array(l, dtype=np.float64).ravel()
        self.u = np.array(u, dtype=np.float64).ravel()
        if self.l.shape != self.u.shape:
            raise ValueError("bounds must be same length")
        bad = np.nonzero(self.l > self.u)[0]
        if bad.size:
            i = int(bad[0])
            raise ValueError("Box set: inconsistent lower/upper bounds specified at index i = %d: l[i] = %g, u[i] = %g"
                             % (i + 1, self.l[i], self.u[i]))
        self.dim = self.l.shape[0]


class SecondOrderCone(AbstractConvexSet):
    """COSMO.SecondOrderCone(dim), convexset.jl:92-98."""
    code = _eng.SOC

    def __init__(self, dim):
        if dim < 0:
            raise ValueError("dimension must be nonnegative")
        self.dim = int(dim)


class PsdCone(AbstractConvexSet):
    """COSMO.PsdCone(dim): vec of a square matrix, convexset.jl:271-284."""
    code = _eng.PSD_SQUARE

    def __init__(self, dim):
        if dim < 0:
            raise ValueError("dimension must be nonnegative")
        r = math.isqrt(dim)
        if r * r != dim:
            raise ValueError("dimension must be a square")
        self.dim, self.sqrt_dim = int(dim), r


class PsdConeTriangle(AbstractConvexSet):
    """COSMO.PsdConeTriangle(dim): scaled upper triangle, convexset.jl:362-377."""
    code = _eng.PSD_TRIANGLE

    def __init__(self, dim):
        if dim < 0:
            raise ValueError("dimension must be nonnegative")
        self.dim = int(dim)
        self.sqrt_dim = (math.isqrt(1 + 8 * dim) - 1) // 2
        if self.sqrt_dim * (self.sqrt_dim + 1) // 2 != dim:
            raise ValueError("dimension must be N(N+1)/2")


class ComplexPsdConeTriangle(AbstractConvexSet):
    """COSMO.PsdConeTriangle{T, Complex{T}}(dim), dim = N^2: Hermitian PSD matrices, real upper triangle (sqrt 2 scaled
    off the diagonal) followed by the imaginary parts of the strict upper triangle (convexset.jl:344-360)."""
    code = _eng.PSD_TRIANGLE_COMPLEX

    def __init__(self, dim):
        if dim < 0:
            raise ValueError("dimension must be nonnegative")
        self.dim = int(dim)
        self.sqrt_dim = math.isqrt(self.dim)
        if self.sqrt_dim * self.sqrt_dim != self.dim:
            raise ValueError("dimension must be a square")


class ExponentialCone(AbstractConvexSet):
    """COSMO.ExponentialCone(): cl{(x,y,z) | y > 0, y e^(x/y) <= z}, convexset.jl:497-507."""
    code = _eng.EXP
    dim = 3

    def __init__(self, dim=3, MAX_ITERS=100, EXP_TOL=1e-8):
        self.MAX_ITER, self.TOL = int(MAX_ITERS), float(EXP_TOL)


class DualExponentialCone(ExponentialCone):
    """COSMO.DualExponentialCone(), convexset.jl:749-758."""
    code = _eng.DUAL_EXP


class PowerCone(AbstractConvexSet):
    """COSMO.PowerCone(alpha): {(x,y,z) | x^a y^(1-a) >= |z|, x, y >= 0}, convexset.jl:625-636."""
    code = _eng.POW
    dim = 3

    def __init__(self, alpha, MAX_ITERS=20, POW_TOL=1e-8):
        if alpha <= 0 or alpha >= 1:
            raise ValueError("The exponent alpha of the power cone has to be in (0, 1).")
        self.alpha, self.MAX_ITER, self.TOL = float(alpha), int(MAX_ITERS), float(POW_TOL)


class DualPowerCone(PowerCone):
    """COSMO.DualPowerCone(alpha), convexset.jl:765-775."""
    code = _eng.DUAL_POW


class CustomConeType:
    """A user-defined cone type: the counterpart of `struct MyCone{T} <: COSMO.AbstractConvexCone{T}` with its
    `project!` (and optionally `in_dual` / `in_pol_recc`) methods, written as CUDA C++ device templates in namespace
    `name` (the contract is in include/cosmo_b200.h at COSMO_B200_CUSTOM).  The engine compiles it for sm_90a when an
    engine that uses it is created, once per process and dtype.  granularity: "thread" (one lane per cone), "warp"
    (32 lanes) or "block" (256 lanes); n_params: values per cone; in_dual / in_pol_recc: whether `source` defines the
    certificate hooks (without them the infeasibility checks never certify, as the reference's documentation says)."""
    _GRAN = {"thread": _eng.CUSTOM_THREAD, "warp": _eng.CUSTOM_WARP, "block": _eng.CUSTOM_BLOCK}

    def __init__(self, name: str, source: str, granularity: str = "warp", n_params: int = 0, in_dual: bool = False,
                 in_pol_recc: bool = False):
        if granularity not in self._GRAN:
            raise ValueError("granularity must be one of %s" % sorted(self._GRAN))
        self.name, self.source, self.granularity = str(name), str(source), granularity
        self.n_params, self.in_dual, self.in_pol_recc = int(n_params), bool(in_dual), bool(in_pol_recc)
        self._bytes = (self.name.encode(), self.source.encode())   # what struct() points to, alive with the type

    def struct(self) -> "_eng.CustomConeStruct":
        flags = (_eng.CUSTOM_HAS_IN_DUAL if self.in_dual else 0) | (_eng.CUSTOM_HAS_IN_POL_RECC if self.in_pol_recc else 0)
        return _eng.CustomConeStruct(self._bytes[0], self._bytes[1], self._GRAN[self.granularity], self.n_params, flags, 0)

    def compile(self, dtype=np.float64) -> bool:
        """Compile for `dtype` without a device (True: compiled now, False: found in the cache)."""
        return _eng.custom_cone_compile(self.struct(), dtype)


class CustomCone(AbstractConvexSet):
    """A cone of a CustomConeType, `dim` rows, with the type's n_params parameters (never scaled: scale! of a custom
    cone is a no-op in the reference)."""
    code = _eng.CUSTOM

    def __init__(self, kind: CustomConeType, dim, params=()):
        if dim < 0:
            raise ValueError("dimension must be nonnegative")
        self.kind, self.dim = kind, int(dim)
        self.params = np.array(params, dtype=np.float64).ravel()
        if self.params.size != kind.n_params:
            raise ValueError("the cone type %s takes %d parameters, got %d" % (kind.name, kind.n_params, self.params.size))


# cones whose rows may only be scaled by one common factor (rectify_scaling!, convexset.jl:952-957; a custom cone takes
# the reference's conservative fall-back, convexset.jl:952-953)
SCALAR_SCALED_CONES = (SecondOrderCone, PsdCone, PsdConeTriangle, ComplexPsdConeTriangle, ExponentialCone, PowerCone,
                       CustomCone)
# cones that cannot be split across ranks
ATOMIC_CONES = SCALAR_SCALED_CONES


def set_tuple(S):
    """The (type, dim, l, u[, params]) tuple `engine.Engine` marshals into a cosmo_b200_set."""
    if isinstance(S, (ExponentialCone, PowerCone)):
        return (S.code, 3, None, None, {"alpha": getattr(S, "alpha", 0.0), "max_iter": S.MAX_ITER, "tol": S.TOL})
    if isinstance(S, CustomCone):
        return (S.code, S.dim, S.params, S.kind)
    return (S.code, S.dim, getattr(S, "l", None), getattr(S, "u", None))


_SORT = (ZeroSet, Nonnegatives, Box, SecondOrderCone, PsdCone, PsdConeTriangle)


def _sort_sets(C) -> int:
    """sort_sets, interface.jl:466-475."""
    for k, T in enumerate(_SORT):
        if isinstance(C, T):
            return k + 1
    return 6


# ---------------------------------------------------------------------------
# Constraint (src/constraint.jl:47-108)
# ---------------------------------------------------------------------------
class Constraint:
    """``COSMO.Constraint(A, b, convex_set, dim=0, indices=None)``: A x + b in convex_set."""

    def __init__(self, A, b, convex_set, dim: int = 0, indices=None):
        if not sp.issparse(A):
            A = np.asarray(A, dtype=np.float64)
            if A.ndim == 0:
                A = A.reshape(1, 1)
            elif A.ndim == 1:
                A = A.reshape(-1, 1)
        A = sp.csr_matrix(A, dtype=np.float64)
        b = np.atleast_1d(np.asarray(b, dtype=np.float64)).ravel()
        if isinstance(convex_set, type):  # set passed as a type, constraint.jl:84-108
            if issubclass(convex_set, Box):
                raise ValueError("You can't create a constraint by passing the convex set as a type, if your "
                                 "convex set is a Box. Please pass an object.")
            convex_set = convex_set(A.shape[0])
        if A.shape[0] != b.shape[0]:
            raise ValueError("The dimensions of matrix A and vector b don't match.")
        if A.shape[0] != convex_set.dim:
            raise ValueError("The row dimension of A doesn't match the dimension of the constraint set.")
        if indices is not None:  # constraint.jl:66-72; (start, stop) 1-based inclusive like Julia's start:stop
            start, stop = int(indices[0]), int(indices[-1])
            if start < 1 or stop < start:
                raise ValueError("The index range for x has to be increasing and nonnegative.")
            if dim < stop:
                raise ValueError("The dimension of x must be equal or higher than the stop value of indices.")
            Ac = sp.lil_matrix((A.shape[0], dim))
            Ac[:, start - 1:stop] = A
            A = sp.csr_matrix(Ac)
        self.A, self.b, self.convex_set = A, b, convex_set


# ---------------------------------------------------------------------------
# Settings (src/settings.jl:61-155) and results (src/types.jl:26-112)
# ---------------------------------------------------------------------------
@dataclass
class Settings:
    rho: float = 0.1
    sigma: float = 1e-6
    alpha: float = 1.6
    eps_abs: float = 1e-5
    eps_rel: float = 1e-5
    eps_prim_inf: float = 1e-4
    eps_dual_inf: float = 1e-4
    max_iter: int = 5000
    verbose: bool = False
    verbose_timing: bool = False             # settings.jl:43: here it forces the device phase timers (proj_time, kkt_time)
    kkt_solver: str = "CGIndirectKKTSolver"   # the indirect family, "DeviceLdlKKTSolver" (direct LDL' on the device) or
    #                                          "DeviceSupernodalKKTSolver" / "MKLPardisoKKTSolver" (supernodal LDL')
    check_termination: int = 25
    check_infeasibility: int = 40
    scaling: int = 10
    MIN_SCALING: float = 1e-4
    MAX_SCALING: float = 1e4
    adaptive_rho: bool = True
    adaptive_rho_interval: int = 40           # 0: automatic (a fraction of the setup time, solver.jl:244-256)
    adaptive_rho_fraction: float = 0.4
    adaptive_rho_tolerance: float = 5.0
    adaptive_rho_max_adaptions: int = 2 ** 62
    RHO_MIN: float = 1e-6
    RHO_MAX: float = 1e6
    RHO_TOL: float = 1e-4
    RHO_EQ_OVER_RHO_INEQ: float = 1e3
    COSMO_INFTY: float = 1e20
    time_limit: float = 0.0
    obj_true: float = float("nan")            # residuals.jl:132-137: |obj_true - cost| <= obj_true_tol joins the convergence test
    obj_true_tol: float = 1e-3
    nearly_ratio: float = 100.0               # only read by is_primal/dual_nearly_feasible (the MOI layer, residuals.jl:119-125)
    tol_constant: float = 1.0
    tol_exponent: float = 1.5
    psd_max_sweeps: int = 30
    # "EmptyAccelerator" | "AndersonAccelerator" (settings.jl:136-138).  The AndersonAccelerator{T, type, memory,
    # regularizer} parameters and the activation reason (accelerator_interface.jl:1-48) follow; the defaults give the
    # reference's default AndersonAccelerator{T, Type2{QRDecomp}, RestartedMemory, NoRegularizer}, ImmediateActivation.
    accelerator: str = "EmptyAccelerator"
    accelerator_mem: int = 15
    accelerator_min_mem: int = 3
    accelerator_type: str = "Type2{QRDecomp}"             # | "Type2{NormalEquations}" | "Type1"
    accelerator_memory: str = "RestartedMemory"           # | "RollingMemory"
    accelerator_regularizer: str = "NoRegularizer"        # | "TikonovRegularizer" | "FrobeniusNormRegularizer"
    accelerator_lambda: float = 1e-8                      # regulariser weight
    accelerator_activation: Union[str, Tuple[str, float]] = "ImmediateActivation"   # | ("IterActivation", k) |
    #                                                                                   ("AccuracyActivation", tol)
    safeguard: bool = True
    safeguard_tol: float = 2.0
    # chordal decomposition of PsdConeTriangle and PsdCone constraints (settings.jl:50-53,129-135; host side, chordal.py).
    # The reference defaults to decompose = true with CliqueGraphMerge; here it is opt-in.
    decompose: bool = False
    merge_strategy: str = "CliqueGraphMerge"   # "NoMerge" | "ParentChildMerge" | "CliqueGraphMerge"
    complete_dual: bool = False
    compact_transformation: bool = True         # False: the traditional transformation A' = [A H; 0 -I], which also
    #                                             decomposes square PsdCone constraints
    # engine-specific: reverse the decomposition (reverse_scaling!, reverse_decomposition!, psd_completion!) on the
    # device from the iterates the solve left there, instead of chordal.reverse on the host
    reverse_on_device: bool = False

    _KKT = {"CGIndirectKKTSolver": _eng.KKT_CG, "MINRESIndirectKKTSolver": _eng.KKT_MINRES,
            "IndirectReducedKKTSolver:MINRES": _eng.KKT_MINRES_REDUCED, "DeviceLdlKKTSolver": _eng.KKT_LDL,
            "DeviceSupernodalKKTSolver": _eng.KKT_LDL_SUPERNODAL, "MKLPardisoKKTSolver": _eng.KKT_LDL_SUPERNODAL}
    _AA_TYPE = {"Type2{QRDecomp}": _eng.AA_TYPE2_QR, "Type2{NormalEquations}": _eng.AA_TYPE2_NORMAL, "Type1": _eng.AA_TYPE1}
    _AA_MEMORY = {"RestartedMemory": _eng.AA_RESTARTED_MEMORY, "RollingMemory": _eng.AA_ROLLING_MEMORY}
    _AA_REG = {"NoRegularizer": _eng.AA_NO_REGULARIZER, "TikonovRegularizer": _eng.AA_TIKONOV,
               "FrobeniusNormRegularizer": _eng.AA_FROBENIUS}

    def accelerator_struct(self) -> Optional["_eng.AcceleratorStruct"]:
        """The cosmo_b200_accelerator of these settings; None for the default variant (nothing to set).  Validates the
        combination: Type2{QRDecomp} with RollingMemory or a regulariser -> ERR_UNSUPPORTED, lambda < 0 -> ERR_INVALID."""
        for value, table, what in ((self.accelerator_type, self._AA_TYPE, "type"),
                                   (self.accelerator_memory, self._AA_MEMORY, "memory"),
                                   (self.accelerator_regularizer, self._AA_REG, "regularizer")):
            if value not in table:
                raise _eng.EngineError(_eng.ERR_UNSUPPORTED, "accelerator %s %r is not an AndersonAccelerator parameter" % (what, value))
        act = self.accelerator_activation
        kind, arg = (act, None) if isinstance(act, str) else (tuple(act) if len(act) == 2 else (None, None))
        if kind not in ("ImmediateActivation", "IterActivation", "AccuracyActivation") or (kind == "ImmediateActivation") != (arg is None):
            raise _eng.EngineError(_eng.ERR_UNSUPPORTED, "accelerator_activation %r is not an activation reason" % (act,))
        if not self.accelerator_lambda >= 0:
            raise _eng.EngineError(_eng.ERR_INVALID, "accelerator_lambda must be a non-negative number")
        a = _eng.AcceleratorStruct()
        a.type = self._AA_TYPE[self.accelerator_type]
        a.memory = self._AA_MEMORY[self.accelerator_memory]
        a.regularizer = self._AA_REG[self.accelerator_regularizer]
        a.lambda_ = float(self.accelerator_lambda)
        a.activation = {"ImmediateActivation": _eng.AA_IMMEDIATE, "IterActivation": _eng.AA_ITER,
                        "AccuracyActivation": _eng.AA_ACCURACY}[kind]
        a.start_iter = int(arg) if kind == "IterActivation" else 2
        a.start_accuracy = float(arg) if kind == "AccuracyActivation" else 0.0
        if a.type == _eng.AA_TYPE2_QR and a.memory != _eng.AA_RESTARTED_MEMORY:
            raise _eng.EngineError(_eng.ERR_UNSUPPORTED, "Type2{QRDecomp} with RollingMemory is not supported (no QR downdate)")
        if a.type == _eng.AA_TYPE2_QR and a.regularizer != _eng.AA_NO_REGULARIZER:
            raise _eng.EngineError(_eng.ERR_UNSUPPORTED, "Type2{QRDecomp} takes no regularizer")
        if a.type == _eng.AA_TYPE2_QR and a.activation == _eng.AA_IMMEDIATE:
            return None
        return a

    def to_struct(self) -> "_eng.SettingsStruct":
        if self.kkt_solver not in self._KKT:
            raise _eng.EngineError(_eng.ERR_UNSUPPORTED,
                                   "kkt_solver %r is not an engine plugin: the H100 engine implements CGIndirectKKTSolver, "
                                   "MINRESIndirectKKTSolver, for a direct LDL' factorisation as QdldlKKTSolver does, "
                                   "DeviceLdlKKTSolver and, for a supernodal one as MKLPardisoKKTSolver does, "
                                   "DeviceSupernodalKKTSolver (also selected as MKLPardisoKKTSolver)" % self.kkt_solver)
        if self.accelerator not in ("EmptyAccelerator", "AndersonAccelerator"):
            raise _eng.EngineError(_eng.ERR_UNSUPPORTED,
                                   "accelerator %r: the engine implements EmptyAccelerator and AndersonAccelerator "
                                   "(variant in accelerator_type / _memory / _regularizer)" % self.accelerator)
        if self.accelerator == "AndersonAccelerator":
            self.accelerator_struct()
            if self.accelerator_mem <= 2:
                raise ValueError("Memory has to be bigger than two.")      # AndersonAccelerator ctor (DomainError)
            if self.accelerator_mem > 32:
                raise _eng.EngineError(_eng.ERR_UNSUPPORTED, "accelerator_mem > 32 is not supported by the device accelerator")
        s = _eng.default_settings()
        for name in ("rho", "sigma", "alpha", "eps_abs", "eps_rel", "eps_prim_inf", "eps_dual_inf", "max_iter",
                     "check_termination", "check_infeasibility", "scaling", "adaptive_rho_interval",
                     "adaptive_rho_tolerance", "adaptive_rho_max_adaptions", "RHO_MIN", "RHO_MAX", "RHO_TOL",
                     "RHO_EQ_OVER_RHO_INEQ", "COSMO_INFTY", "MIN_SCALING", "time_limit", "tol_constant",
                     "tol_exponent", "psd_max_sweeps", "accelerator_mem", "accelerator_min_mem", "safeguard_tol",
                     "adaptive_rho_fraction", "MAX_SCALING", "obj_true", "obj_true_tol"):
            setattr(s, name, getattr(self, name))
        s.adaptive_rho = int(self.adaptive_rho)
        s.verbose = int(bool(self.verbose)) | (2 if self.verbose_timing else 0)
        s.kkt_solver = self._KKT[self.kkt_solver]
        s.accelerator = _eng.ACC_ANDERSON if self.accelerator == "AndersonAccelerator" else _eng.ACC_EMPTY
        s.safeguard = int(self.safeguard)
        return s


@dataclass
class ResultInfo:
    r_prim: float
    r_dual: float
    max_norm_prim: float
    max_norm_dual: float
    rho_updates: List[float]


@dataclass
class Result:
    x: np.ndarray
    y: np.ndarray
    s: np.ndarray
    obj_val: float
    iter: int
    safeguarding_iter: int
    status: str
    info: ResultInfo
    times: dict
    kkt_inner_iterations: int = 0
    kernel_launches: int = 0


# ---------------------------------------------------------------------------
# Ruiz equilibration (src/scaling.jl:21-116) -- host-side setup!, runs once
# ---------------------------------------------------------------------------
def _col_absmax(M: sp.csc_matrix, out: np.ndarray):
    if M.nnz:
        nz = np.diff(M.indptr) > 0
        mx = np.maximum.reduceat(np.abs(M.data), M.indptr[:-1][nz])
        out[nz] = np.maximum(out[nz], mx)
    return out


def _row_absmax(M: sp.csc_matrix, out: np.ndarray):
    if M.nnz:
        np.maximum.at(out, M.indices, np.abs(M.data))
    return out


def _limit(v, lo, hi):
    """limit_scaling!: clip(s, MIN, MAX, one, MAX) (scaling.jl:10-18, algebra.jl:5-7)."""
    return np.where(v < lo, 1.0, np.where(v > hi, hi, v))


def ruiz_equilibrate(P, q, A, b, sets, st: Settings):
    """scale_ruiz! on CSC arrays in place; returns (P, q, A, b, sets, D, E, c)."""
    P = sp.csc_matrix(P, dtype=np.float64, copy=True)
    A = sp.csc_matrix(A, dtype=np.float64, copy=True)
    q = np.array(q, dtype=np.float64)
    b = np.array(b, dtype=np.float64)
    m, n = A.shape
    D, E, c = np.ones(n), np.ones(m), 1.0
    colA = np.repeat(np.arange(n), np.diff(A.indptr))
    colP = np.repeat(np.arange(n), np.diff(P.indptr))

    def scale_data(Ds, Es):
        nonlocal q, b
        P.data *= Ds[P.indices] * Ds[colP]
        A.data *= Es[A.indices] * Ds[colA]
        q = Ds * q
        b = Es * b

    for _ in range(st.scaling):
        Dw = _col_absmax(A, _col_absmax(P, np.zeros(n)))
        Ew = _row_absmax(A, np.zeros(m))
        Dw = 1.0 / np.sqrt(_limit(Dw, st.MIN_SCALING, st.MAX_SCALING))
        Ew = 1.0 / np.sqrt(_limit(Ew, st.MIN_SCALING, st.MAX_SCALING))
        scale_data(Dw, Ew)
        D *= Dw
        E *= Ew
        mean_col_norm_P = float(np.mean(_col_absmax(P, np.zeros(n)))) if n else 0.0
        inf_norm_q = float(np.max(np.abs(q))) if n else 0.0
        if mean_col_norm_P != 0.0 and inf_norm_q != 0.0:
            inf_norm_q = float(_limit(inf_norm_q, st.MIN_SCALING, st.MAX_SCALING))
            scale_cost = float(_limit(max(inf_norm_q, mean_col_norm_P), st.MIN_SCALING, st.MAX_SCALING))
            ctmp = 1.0 / scale_cost
            P.data *= ctmp
            q = q * ctmp
            c *= ctmp
    # cones that only admit a scalar scaling (convexset.jl:905-958, 978-982)
    Ew = np.ones(m)
    changed = False
    off = 0
    for S in sets:
        if isinstance(S, SCALAR_SCALED_CONES) and S.dim > 0:
            seg = slice(off, off + S.dim)
            Ew[seg] = np.mean(E[seg]) / E[seg]
            changed = True
        off += S.dim
    if changed:
        scale_data(np.ones(n), Ew)
        E *= Ew
    new_sets, off = [], 0
    for S in sets:  # scale!(box, e), convexset.jl:863-867
        if isinstance(S, Box):
            e = E[off:off + S.dim]
            new_sets.append(Box(S.l * e, S.u * e))
        else:
            new_sets.append(S)
        off += S.dim
    return P, q, A, b, new_sets, D, E, c


def _sorted_csc(M) -> sp.csc_matrix:
    """M as a float64 CSC matrix with sorted row indices (a copy when they had to be sorted)."""
    M = sp.csc_matrix(M, dtype=np.float64)
    return M if M.has_sorted_indices else M.sorted_indices()


# ---------------------------------------------------------------------------
# Model (COSMO.Model = Workspace, src/types.jl:348-403)
# ---------------------------------------------------------------------------
class Model:
    def __init__(self, dtype=np.float64, device: int = 0):
        self.dtype = np.dtype(dtype)
        self.device = device
        self.is_assembled = False
        self.is_scaled = False
        self.engine: Optional[_eng.Engine] = None
        self.settings = Settings()
        self.times = {}
        self._dec = None          # chordal DecompositionInfo of the problem the engine holds (settings.decompose)
        self._x2 = None           # iterates of the decomposed problem (None: restart from self.x)
        self._fwd = None          # chordal.ForwardArrays the engine holds: original values -> decomposed problem
        self._q0 = self._b0 = None
        self._qb_on_device = [False, False]   # q0 / b0 came as CUDA arrays: the engine holds them (original_qb)
        self._solution_on_device = False      # optimize(solution="device"): x, s, mu live only in the engine

    # q0 and b0 after update(q=, b=) with CUDA arrays are read back from the engine only when something reads them
    @property
    def q0(self):
        if self._qb_on_device[0]:
            self._fetch_qb()
        return self._q0

    @q0.setter
    def q0(self, v):
        self._q0, self._qb_on_device[0] = v, False

    @property
    def b0(self):
        if self._qb_on_device[1]:
            self._fetch_qb()
        return self._b0

    @b0.setter
    def b0(self, v):
        self._b0, self._qb_on_device[1] = v, False

    def _fetch_qb(self):
        if not any(self._qb_on_device):
            return
        want = [np.empty(k) if dev else None for dev, k in zip(self._qb_on_device, (self.n, self.m))]
        q, b = self.engine.original_qb(*want)
        if q is not None:
            self.q0 = q
        if b is not None:
            self.b0 = b

    def _fetch_solution(self):
        """x, s, mu of a solve that left them on the device, to the host (before the engine loses them)."""
        if not self._solution_on_device:
            return
        self._solution_on_device = False
        x, y, s = self._device_solution(np.empty(self.n), np.empty(self.m), np.empty(self.m))
        self.x, self.s, self.mu = x, s, -y
        self._x2 = None   # the clique iterates stay in the engine: a decomposed model restarts from x

    def _device_solution(self, x, y, s):
        if self._dec is not None and not self.engine.n_orig:   # reverse on the device, with or without reverse_on_device
            from . import chordal as _chordal
            self.engine.set_decomposition(_chordal.decomposition_arrays(self._dec, len(self.D), len(self.E)))
        return self.engine.solution(self.settings.complete_dual, x, y, s)

    # assemble!(model, P, q, constraints; settings, x0, y0), interface.jl:30-77
    def assemble(self, P, q, constraints: Union[Constraint, Sequence[Constraint]], settings: Optional[Settings] = None,
                 x0=None, y0=None):
        if isinstance(constraints, Constraint):
            constraints = [constraints]
        cons = list(constraints)
        n = int(np.atleast_1d(np.asarray(q)).size)
        # merge_constraints!, interface.jl:411-460
        for T in (ZeroSet, Nonnegatives):
            idx = [i for i, c in enumerate(cons) if type(c.convex_set) is T]
            if len(idx) > 1:
                A = sp.vstack([cons[i].A for i in idx], format="csr")
                b = np.concatenate([cons[i].b for i in idx])
                cons = [c for i, c in enumerate(cons) if i not in idx] + [Constraint(A, b, T(A.shape[0]))]
        cons.sort(key=lambda c: _sort_sets(c.convex_set))
        for c in cons:  # check_A_dim
            if c.A.shape[1] != n:
                raise ValueError("The dimensions of a matrix A (m x %d) in one of the constraints is inconsistent "
                                 "with the dimension of P (%d)." % (c.A.shape[1], n))
        P = sp.csc_matrix(P, dtype=np.float64) if sp.issparse(P) else sp.csc_matrix(np.atleast_2d(np.asarray(P, dtype=np.float64)))
        if P.shape != (n, n):
            raise ValueError("Dimensions of P and q are inconsistent.")
        A = sp.vstack([-c.A for c in cons], format="csc") if cons else sp.csc_matrix((0, n))
        b = np.concatenate([c.b for c in cons]) if cons else np.zeros(0)
        self.set(P, np.asarray(q, dtype=np.float64).ravel(), A, b, [c.convex_set for c in cons], settings)
        if x0 is not None:
            self.warm_start_primal(x0)
        if y0 is not None:
            self.warm_start_dual(y0)

    # set!(model, P, q, A, b, convex_sets, settings), interface.jl:218-250: model form A x + s = b
    def set(self, P, q, A, b, convex_sets: Sequence[AbstractConvexSet], settings: Optional[Settings] = None):
        A = _sorted_csc(A)
        P = _sorted_csc(P)
        m, n = A.shape
        if sum(S.dim for S in convex_sets) != m:
            raise ValueError("set dimension is not m")
        if P.shape != (n, n) or len(q) != n or len(b) != m:
            raise ValueError("Dimensions of P, q, A, b are inconsistent.")
        self.P0, self.q0, self.A0, self.b0 = P, np.array(q, dtype=np.float64), A, np.array(b, dtype=np.float64)
        self.sets0 = list(convex_sets)
        self.m, self.n = m, n
        if settings is not None:
            self.settings = settings
        self.x = np.zeros(n)
        self.s = np.zeros(m)
        self.mu = np.zeros(m)
        self.is_assembled = True
        self.is_scaled = False
        self._dec = None
        self._x2 = None
        self._fwd = None
        self._solution_on_device = False
        if self.engine is not None:
            self.engine.close()
            self.engine = None

    # warm starts in unscaled coordinates, interface.jl:117-179
    def warm_start_primal(self, x0):
        x0 = np.asarray(x0, dtype=np.float64)
        if x0.shape != (self.n,):
            raise ValueError("Dimension of warm starting vector doesn't match the length of index range ind.")
        self._fetch_solution()
        self.x[:] = x0
        self.s[:] = self.b0 - self.A0 @ self.x   # s0 = b - A x0 (interface.jl:131-147)
        self._x2 = None                           # a decomposed model restarts from this point (see _setup)

    def warm_start_slack(self, s0):
        self._fetch_solution()
        self.s[:] = s0
        self._x2 = None

    def warm_start_dual(self, y0):
        y0 = np.asarray(y0, dtype=np.float64)
        if y0.shape != (self.m,):
            raise ValueError("Dimension of warm starting vector doesn't match the length of index range ind.")
        self._fetch_solution()
        self.mu[:] = -y0
        self._x2 = None

    # update!(model; q, b), interface.jl:187-211, extended by new values of P and A on the pattern given to set!.  The
    # new values go to the live engine, and the iterates of the model stay as the next warm start.  The reference
    # refuses to update a chordally decomposed model (interface.jl:192,204); here the values are mapped onto the
    # decomposed problem, and rho and the clique iterates stay, as update! keeps them.  q and b may be CUDA arrays
    # (__cuda_array_interface__, fp64): with a live engine and no new P or A they go to the engine without a host copy
    # (update_qb_original), else they are copied to the host first.
    def update(self, q=None, b=None, *, P=None, A=None):
        if not self.is_assembled:
            raise RuntimeError("Model has to be assembled once before one can start updating q or b.")
        if _eng.is_cuda_array(q) or _eng.is_cuda_array(b):
            for v, k, name in ((q, self.n, "q"), (b, self.m, "b")):
                if _eng.is_cuda_array(v) and tuple(v.__cuda_array_interface__["shape"]) != (k,):
                    raise ValueError("The dimension of %s, does not agree with the model dimension, %s." % (name, "nm"[name == "b"]))
            if P is None and A is None and self.engine is not None and (self._dec is None or self._fwd is not None):
                try:
                    self.engine.update_qb_original(q, b)
                except _eng.EngineError as e:
                    if e.code != _eng.ERR_INVALID or self._dec is None or b is None:
                        raise
                    # b is nonzero on a row no clique holds: the host route below drops the engine
                    pass
                else:
                    for k, v in enumerate((q, b)):
                        if v is not None:
                            self._qb_on_device[k] = True
                    return
            q, b = (None if v is None else _eng.to_host(v) for v in (q, b))
        new = {}
        for name, M, old in (("P", P, self.P0), ("A", A, self.A0)):
            if M is None:
                continue
            M = _sorted_csc(M)
            if M.shape != old.shape or not (np.array_equal(M.indptr, old.indptr) and np.array_equal(M.indices, old.indices)):
                raise ValueError("The sparsity pattern of %s differs from the one the model was set up with: use set! "
                                 "(Model.set) for a new pattern." % name)
            new[name] = M
        if q is not None:
            q = np.asarray(q, dtype=np.float64)
            if q.shape != (self.n,):
                raise ValueError("The dimension of q, does not agree with the model dimension, n.")
        if b is not None:
            b = np.asarray(b, dtype=np.float64)
            if b.shape != (self.m,):
                raise ValueError("The dimension of b, does not agree with the model dimension, m.")
        self.P0, self.A0 = new.get("P", self.P0), new.get("A", self.A0)
        if new:
            self._fetch_solution()   # new matrices reset the engine's iterates; the next solve warm-starts from the host
        if q is not None:
            self.q0 = q.copy()
        if b is not None:
            self.b0 = b.copy()
        if self.engine is None or (self._dec is not None and not self._decomposition_holds(b)):
            return
        if not new:
            # q and b alone, scaled on the host; a decomposed model maps them first, q' = [q; 0] and b' = b[b_src]
            q2, b2 = self.q0, self.b0
            if self._dec is not None:
                from . import chordal as _chordal
                _, q2, b2 = _chordal.forward_values(self._fwd, None, self.q0 if q is not None else None,
                                                    self.b0 if b is not None else None)
            self.engine.update_qb((self.D * q2) * self.c if q is not None else None,
                                  self.E * b2 if b is not None else None)
            return
        if self._dec is not None:
            # the values in the original coordinates go through the forward map on the device; all four, so that an
            # equilibrating engine can run Ruiz again
            self.engine.update_matrices_original(self.P0.data, self.A0.data, self.q0, self.b0)
        elif self._engine_equilibrates:
            # Ruiz runs again on the device from the unscaled data: every vector goes with the matrices
            self.engine.update_matrices(self.P0.data, self.A0.data, self.q0, self.b0)
        else:
            self.engine.update_matrices(new["P"].data if "P" in new else None, new["A"].data if "A" in new else None,
                                        q, b)
        if self._engine_equilibrates:
            self.D, self.E, self.c = self.engine.scaling()

    def _decomposition_holds(self, b) -> bool:
        """Can the live engine of a decomposed model take the new data?  Not without the forward map, and not when the new
        `b` is nonzero in a row of a decomposed cone that no clique holds: the aggregate sparsity pattern changes, so the
        engine is dropped and the next optimize! decomposes again (rho and the clique iterates restart)."""
        if self._fwd is not None:
            if b is None:
                return True
            from . import chordal as _chordal
            if not len(_chordal.uncovered_rows(self._fwd, b)):
                return True
        self._fetch_qb()          # what lives only in the engine goes to the host before it is closed
        self._fetch_solution()
        self._x2 = None
        self._fwd = None
        self.engine.close()
        self.engine = None
        return False

    # setup! (setup.jl:18-64): scaling + engine creation (the KKT "factorisation" analogue)
    def _setup(self):
        st = self.settings
        t0 = time.perf_counter()
        if self.engine is None:
            # chordal_decomposition!(ws), chordal_decomposition.jl:1-30 (before setup!, solver.jl:88-93)
            self._dec = None
            self._fwd = None
            P0, q0, A0, b0, sets0 = self.P0, self.q0, self.A0, self.b0, self.sets0
            if st.decompose:
                from . import chordal as _chordal
                merge = {"NoMerge": "none", "ParentChildMerge": "parent_child_reference",
                         "CliqueGraphMerge": "clique_graph"}.get(st.merge_strategy)
                if merge is None:
                    raise ValueError("unknown merge_strategy %r" % (st.merge_strategy,))
                P2, q2, A2, b2, sets2, info = _chordal.decompose(P0, q0, A0, b0, sets0, merge=merge,
                                                                 compact=st.compact_transformation)
                if info.blocks:                   # at least one cone was decomposed
                    self._dec = info
                    P0, q0, A0, b0, sets0 = P2, q2, A2, b2, sets2
                    self._x2 = np.concatenate([self.x, np.zeros(A2.shape[1] - self.n)])
                    self._s2, self._mu2 = np.zeros(A2.shape[0]), np.zeros(A2.shape[0])
            m2, n2 = A0.shape
            # scale_ruiz! runs on the device (csrc/ruiz.cuh): the engine ingests the unscaled data and hands D, E, c back
            # how the engine was created, not the settings of a later solve, decides what update(P=, A=) hands over
            self._engine_equilibrates = st.scaling != 0
            self.engine = _eng.Engine(P0, q0, A0, b0, [set_tuple(S) for S in sets0], st.to_struct(),
                                      dtype=self.dtype, device=self.device, equilibrate=self._engine_equilibrates)
            D, E, c = self.engine.scaling() if st.scaling != 0 else (np.ones(n2), np.ones(m2), 1.0)
            self.D, self.E, self.c = D, E, c
            if self._dec is not None and st.reverse_on_device:
                self.engine.set_decomposition(_chordal.decomposition_arrays(self._dec, n2, m2))
            if self._dec is not None and hasattr(self.engine, "set_forward_map"):
                # later updates of q, b, P and A keep this engine; an engine that cannot take the map is rebuilt instead
                self._fwd = _chordal.forward_arrays(self._dec, self.A0, n2, m2)
                self.engine.set_forward_map(self._fwd)
        else:
            self.engine.update_settings(st.to_struct())
        configure_accelerator(self.engine, st)
        # scale_variables! (scaling.jl:118-123)
        if self._solution_on_device:
            # the last solution never left the device: the same unscale / rescale round trip, in place
            self._solution_on_device = False
            self.engine.rescale_iterates()
        elif self._dec is not None:
            # The decomposed problem keeps its own iterates between solves.  A warm start given in the ORIGINAL
            # coordinates enters through x only (the clique copies of s and mu start from zero): the reference
            # re-allocates all variables after the decomposition (pre_allocate_variables!, chordal_decomposition.jl:29),
            # i.e. drops the warm start altogether, and cannot re-solve a decomposed model.
            if getattr(self, "_x2", None) is None:
                n2, m2 = len(self.D), len(self.E)
                self._x2 = np.concatenate([self.x, np.zeros(n2 - self.n)])
                self._s2, self._mu2 = np.zeros(m2), np.zeros(m2)
            self.engine.warm_start(self._x2 / self.D, self.E * self._s2, (self._mu2 / self.E) * self.c)
        else:
            self.engine.warm_start(self.x / self.D, self.E * self.s, (self.mu / self.E) * self.c)
        return time.perf_counter() - t0

    # optimize!(model), solver.jl:78-203.  solution="device" leaves the solution on the device: Result.x, .y, .s are
    # None, solution_into() writes it into caller arrays, and the next optimize starts from it without a host round trip.
    def optimize(self, solution: str = "host") -> Result:
        if not self.is_assembled:
            raise RuntimeError("The model has to be assembled! / set! before optimize!() can be called.")
        if solution not in ("host", "device"):
            raise ValueError("solution must be \"host\" or \"device\"")
        t0 = time.perf_counter()
        setup_time = self._setup()
        if self.settings.time_limit != 0 or (self.settings.adaptive_rho and self.settings.adaptive_rho_interval == 0):
            st = self.settings.to_struct()           # both rules count setup! (solver.jl:119,244-256,349)
            st.setup_time = setup_time
            self.engine.update_settings(st)
        out = self.engine.solve() if solution == "host" else self.engine.solve(copy_out=False)
        times = dict(out.times)
        times["setup_time"] = setup_time
        info = ResultInfo(out.r_prim, out.r_dual, out.max_norm_prim, out.max_norm_dual, list(out.rho_updates))
        if solution == "device":
            self._solution_on_device = True
            times["solver_time"] = time.perf_counter() - t0
            return Result(None, None, None, out.obj_val, out.iter, out.safeguarding_iter, out.status, info, times,
                          kkt_inner_iterations=out.kkt_inner_iterations, kernel_launches=out.kernel_launches)
        # reverse_scaling! (scaling.jl:170-179)
        x = self.D * out.x.astype(np.float64)
        s = out.s.astype(np.float64) / self.E
        mu = self.E * out.mu.astype(np.float64) / self.c
        if self._dec is not None:   # reverse_decomposition! (+ psd_completion!), chordal_decomposition.jl:129-151
            from . import chordal as _chordal
            self._x2, self._s2, self._mu2 = x.copy(), s.copy(), mu.copy()
            if self.settings.reverse_on_device:
                x, s, mu, _ = self.engine.reverse_decomposition(complete_dual=self.settings.complete_dual)
            else:
                x, s, mu = _chordal.reverse(self._dec, x, s, mu, complete_dual=self.settings.complete_dual)
        self.x, self.s, self.mu = x.copy(), s.copy(), mu.copy()
        times["solver_time"] = time.perf_counter() - t0
        return Result(x, -mu, s, out.obj_val, out.iter, out.safeguarding_iter, out.status, info, times,
                      kkt_inner_iterations=out.kkt_inner_iterations, kernel_launches=out.kernel_launches)

    def solution_into(self, x=None, y=None, s=None):
        """The last solution (x, y, s of Result, completed as settings.complete_dual asks) into caller fp64 arrays, CUDA
        (__cuda_array_interface__) or NumPy; None skips one.  After optimize(solution="device") it is reversed on the
        device straight into them (a decomposed model without reverse_on_device gets the device map for it)."""
        if self._solution_on_device:
            self._device_solution(x, y, s)
            return
        for dst, src in ((x, self.x), (y, -self.mu), (s, self.s)):
            if dst is not None:
                _eng.copy_into(dst, src)

    def empty_model(self):  # empty_model!, interface.jl:84-100
        if self.engine is not None:
            self.engine.close()
        self.__init__(self.dtype, self.device)


def configure_accelerator(engine, st: Settings):
    """Hand the Anderson variant of `st` to the engine (_make_accelerator!, setup.jl:10-14).  An engine that never ran
    a non-default variant is left alone; one that did is reset to the default."""
    acc = st.accelerator_struct() if st.accelerator == "AndersonAccelerator" else None
    if acc is not None or getattr(engine, "_custom_accelerator", False):
        engine.set_accelerator(acc)
        engine._custom_accelerator = acc is not None


def assemble(model: Model, P, q, constraints, settings: Optional[Settings] = None, x0=None, y0=None):
    """``assemble!(model, P, q, constraints; settings, x0, y0)``."""
    model.assemble(P, q, constraints, settings, x0, y0)


def optimize(model: Model) -> Result:
    """``COSMO.optimize!(model)``."""
    return model.optimize()
