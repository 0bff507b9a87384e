"""Custom cones with the Jacobian hook (COSMO_B200_CUSTOM_HAS_JACOBIAN), each defined twice: as CUDA C++ for the engine
(model.CustomConeType(..., jacobian=True)) and as NumPy functions for the oracle and the restatements of
tests/solve_adjoint_reference.py and tests/solve_derivative_reference.py, whose dpi `install_restatement` extends for
the duration of one test.

The cones are those of tests/custom_cones.py under new type names (so the types there stay as they are), each source
reopening its namespace to add `jacobian(w, s, h, dim, p, lane, width)`, which overwrites h with DPi(w) h:
  nonpos_jac (one thread per cone): h where w < 0, 0 elsewhere;
  soc2_jac   (one warp per cone):   the SOC Jacobian of the engine's built-in branch (solve_adjoint.cuh, sa_dpi_rows_kernel);
  wlinf_jac  (one block per cone): {(t, x) : c |x|_inf <= t}, c the parameter.  At a point w = (t0, x0) outside the cone
    and its polar, the projection clips x0 at the threshold r = s[0] / c; with C the clipped entries and k = |C|, r
    solves c^2 r - c t0 - sum_C (|x0_i| - r) = 0, so dr = (c h0 + sum_C sign(x0_i) h_i) / (c^2 + k) and
    DPi h = (c dr, h_i off C, sign(x0_i) dr on C): the identity off C plus a rank-one block, symmetric."""
import numpy as np

from cosmo_b200 import model as M
from oracle.bridge import to_oracle_cones
from tests import custom_cones as CC
from tests import solve_adjoint_reference as SA
from tests import solve_derivative_reference as SD

NONPOS_JAC = r"""
template <typename T> __device__ void jacobian(const T* w, const T* s, T* h, long long dim, const T* p, int lane, int width) {
  for (long long i = 0; i < dim; ++i) if (!(w[i] < T(0))) h[i] = T(0);
}
"""

SOC2_JAC = r"""
template <typename T> __device__ void jacobian(const T* w, const T* s, T* h, long long dim, const T* p, int lane, int width) {
  const T r = tail_norm(w, dim, lane, width);
  const T t = w[0];
  if (r <= t) return;
  if (r <= -t) {
    for (long long i = lane; i < dim; i += width) h[i] = T(0);
    return;
  }
  T d = T(0);
  for (long long i = 1 + lane; i < dim; i += width) d += w[i] * h[i];
  d = cosmo_cone::sum(d, width);
  const T h0 = h[0];
  cosmo_cone::sync(width);          // every lane has read h[0] before lane 0 overwrites it
  const T tr = t / r;
  for (long long i = 1 + lane; i < dim; i += width)
    h[i] = T(0.5) * (w[i] / r * h0 + (T(1) + tr) * h[i] - tr * w[i] * d / (r * r));
  if (lane == 0) h[0] = T(0.5) * (h0 + d / r);
}
"""

LINF_JAC = r"""
template <typename T> __device__ void jacobian(const T* w, const T* s, T* h, long long dim, const T* p, int lane, int width) {
  const T c = p[0], t0 = w[0];
  T amax = T(0);
  for (long long i = 1 + lane; i < dim; i += width) amax = fabs(w[i]) > amax ? fabs(w[i]) : amax;
  amax = cosmo_cone::max(amax, width);
  if (c * amax <= t0) return;                       // inside the cone: the identity
  const T r = s[0] / c;
  if (!(r > T(0))) {                                // projected to the origin
    for (long long i = lane; i < dim; i += width) h[i] = T(0);
    return;
  }
  T num = T(0), k = T(0);
  for (long long i = 1 + lane; i < dim; i += width)
    if (fabs(w[i]) > r) { num += w[i] > T(0) ? h[i] : -h[i]; k += T(1); }
  num = cosmo_cone::sum(num, width);
  k = cosmo_cone::sum(k, width);
  const T h0 = h[0];
  cosmo_cone::sync(width);
  const T dr = (c * h0 + num) / (c * c + k);
  for (long long i = 1 + lane; i < dim; i += width)
    if (fabs(w[i]) > r) h[i] = w[i] > T(0) ? dr : -dr;
  if (lane == 0) h[0] = c * dr;
}
"""


def _with_jacobian(src, name, new, jac):
    """`src` with its namespace renamed to `new`, reopened to add `jac`"""
    return src.replace("namespace %s {" % name, "namespace %s {" % new) + "namespace %s {\n%s}\n" % (new, jac)


NONPOS_SRC = _with_jacobian(CC.NONPOS_SRC, "nonpos", "nonpos_jac", NONPOS_JAC)
SOC2_SRC = _with_jacobian(CC.SOC2_SRC, "soc2", "soc2_jac", SOC2_JAC)
LINF_SRC = _with_jacobian(CC.LINF_SRC, "wlinf", "wlinf_jac", LINF_JAC)


def nonpos_type(jacobian=True):
    return M.CustomConeType("nonpos_jac", NONPOS_SRC, "thread", in_dual=True, in_pol_recc=True, jacobian=jacobian)


def soc2_type(jacobian=True):
    return M.CustomConeType("soc2_jac", SOC2_SRC, "warp", in_dual=True, in_pol_recc=True, jacobian=jacobian)


def linf_type(jacobian=True):
    return M.CustomConeType("wlinf_jac", LINF_SRC, "block", n_params=1, jacobian=jacobian)


TYPES = [nonpos_type, soc2_type, linf_type]


# ---- the Jacobians in NumPy: DPi(w) h, s = Pi(w) -------------------------------------------
def _nonpos_jacobian(w, s, h, p):
    return np.where(w < 0.0, h, 0.0)


def _soc_jacobian(w, s, h, p):
    t, xb = w[0], w[1:]
    r = np.linalg.norm(xb)
    if r <= t:
        return h.copy()
    if r <= -t:
        return np.zeros_like(h)
    d = xb @ h[1:]
    o = np.empty_like(h)
    o[0] = 0.5 * (h[0] + d / r)
    o[1:] = 0.5 * (xb / r * h[0] + (1 + t / r) * h[1:] - (t / r) * xb * d / r ** 2)
    return o


def _linf_jacobian(w, s, h, p):
    c, t0 = float(p[0]), w[0]
    a = np.abs(w[1:])
    if c * (a.max() if a.size else 0.0) <= t0:
        return h.copy()
    r = s[0] / c
    if not r > 0.0:
        return np.zeros_like(h)
    C = a > r
    sg = np.sign(w[1:])
    dr = (c * h[0] + (sg[C] * h[1:][C]).sum()) / (c * c + C.sum())
    o = h.copy()
    o[0] = c * dr
    o[1:][C] = sg[C] * dr
    return o


# name -> (project, in_dual, in_pol_recc, jacobian)
NUMPY = {
    "nonpos_jac": CC.NUMPY["nonpos"] + (_nonpos_jacobian,),
    "soc2_jac": CC.NUMPY["soc2"] + (_soc_jacobian,),
    "wlinf_jac": CC.NUMPY["wlinf"] + (_linf_jacobian,),
}


class OracleJacobianCone(CC.OracleCustomCone):
    """An oracle custom cone with a NumPy `jacobian(w, s, h, params)` (DPi(w) h, s = Pi(w)), which the restatements
    apply once install_restatement has run."""

    def __init__(self, dim, project, in_dual=None, in_pol_recc=None, jacobian=None, params=()):
        super().__init__(dim, project, in_dual, in_pol_recc, params)
        self.jacobian = jacobian


def to_oracle(sets):
    """The oracle's cones of `sets`: the types here as OracleJacobianCone (the Jacobian only when the type has the flag),
    the types of tests/custom_cones.py through its to_oracle, every other set through oracle.bridge."""
    out = []
    for S in sets:
        if isinstance(S, M.CustomCone) and S.kind.name in NUMPY:
            proj, dual, recc, jac = NUMPY[S.kind.name]
            out.append(OracleJacobianCone(S.dim, proj, dual if S.kind.in_dual else None,
                                          recc if S.kind.in_pol_recc else None, jac if S.kind.jacobian else None,
                                          S.params))
        elif isinstance(S, M.CustomCone):
            out.extend(CC.to_oracle([S]))
        else:
            out.extend(to_oracle_cones([S]))
    return out


def install_restatement(monkeypatch):
    """Extend the dpi of the restatements (solve_adjoint_reference.dpi, which solve_derivative_reference imports) for the
    duration of one test (pytest's monkeypatch undoes it): a cone with a NumPy `jacobian` goes through it at Pi(w)
    computed by its own projection, every other cone through the restatement's dpi as before."""
    dpi = SA.dpi

    def dpi_(w, cones, h):
        out = np.empty_like(h)
        k = 0
        for cone in cones:
            sl = slice(k, k + cone.dim)
            if getattr(cone, "jacobian", None) is not None:
                ps = w[sl].copy()
                cone.project(ps, cone.params)
                out[sl] = cone.jacobian(w[sl], ps, h[sl], cone.params)
            else:
                out[sl] = dpi(w[sl], [cone], h[sl])
            k += cone.dim
        return out

    monkeypatch.setattr(SA, "dpi", dpi_)
    monkeypatch.setattr(SD, "dpi", dpi_)
