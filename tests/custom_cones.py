"""The custom cones of the tests, each defined twice: as CUDA C++ for the engine (model.CustomConeType) and as NumPy
functions for the oracle.  `install_oracle` teaches the oracle's dispatch functions (project_cone, in_dual,
in_pol_recc and, through in_dual, support_function) and its Ruiz rectification about OracleCustomCone, the oracle's
counterpart of a custom cone, with the rule the engine follows: a type without a hook never certifies."""
import numpy as np

from cosmo_b200 import model as M
from oracle import cosmo_oracle as O
from oracle.bridge import to_oracle_cones

# The reference's example (docs/src/literate/custom_cone.jl): x .= min.(x, 0) and its literal certificate hooks
NONPOS_SRC = r"""
namespace nonpos {
template <typename T> __device__ void project(T* x, long long dim, const T* p, int lane, int width) {
  for (long long i = 0; i < dim; ++i) x[i] = x[i] > T(0) ? T(0) : x[i];
}
template <typename T> __device__ bool in_dual(const T* x, long long dim, T tol, const T* p, int lane, int width) {
  for (long long i = 0; i < dim; ++i) if (x[i] > -tol) return false;
  return true;
}
template <typename T> __device__ bool in_pol_recc(const T* x, long long dim, T tol, const T* p, int lane, int width) {
  for (long long i = 0; i < dim; ++i) if (x[i] < tol) return false;
  return true;
}
}
"""

# The second-order cone, one warp per cone (convexset.jl:100-122)
SOC2_SRC = r"""
namespace soc2 {
template <typename T> __device__ T tail_norm(const T* x, long long dim, int lane, int width) {
  T s = T(0);
  for (long long i = 1 + lane; i < dim; i += width) s += x[i] * x[i];
  return sqrt(cosmo_cone::sum(s, width));
}
template <typename T> __device__ void project(T* x, long long dim, const T* p, int lane, int width) {
  const T nx = tail_norm(x, dim, lane, width);
  const T t = x[0];
  cosmo_cone::sync(width);          // every lane has read x[0] before lane 0 overwrites it
  if (nx <= t) return;
  if (nx <= -t) {
    for (long long i = lane; i < dim; i += width) x[i] = T(0);
    return;
  }
  const T f = (nx + t) / (T(2) * nx);
  for (long long i = 1 + lane; i < dim; i += width) x[i] = f * x[i];
  if (lane == 0) x[0] = (nx + t) / T(2);
}
template <typename T> __device__ bool in_dual(const T* x, long long dim, T tol, const T* p, int lane, int width) {
  return tail_norm(x, dim, lane, width) <= tol + x[0];
}
template <typename T> __device__ bool in_pol_recc(const T* x, long long dim, T tol, const T* p, int lane, int width) {
  return tail_norm(x, dim, lane, width) <= tol - x[0];
}
}
"""

# {(t, x) : w |x|_inf <= t} with the weight w > 0 as the parameter, one block per cone.  For t = w s the nearest point
# has x = clip(x0, -s, s), and s >= 0 is the root of g(s) = w^2 s - w t0 - sum_i max(|x0_i| - s, 0) (increasing in s),
# found by bisection on [0, max(|x0|_inf, t0 / w)]; s = 0 (the origin) when g(0) >= 0.
LINF_SRC = r"""
namespace wlinf {
template <typename T> __device__ T excess(const T* x, long long dim, T s, int lane, int width) {
  T e = T(0);
  for (long long i = 1 + lane; i < dim; i += width) { const T a = fabs(x[i]) - s; e += a > T(0) ? a : T(0); }
  return cosmo_cone::sum(e, width);
}
template <typename T> __device__ void project(T* x, long long dim, const T* p, int lane, int width) {
  const T w = p[0], t0 = x[0];
  T amax = T(0);
  for (long long i = 1 + lane; i < dim; i += width) amax = fabs(x[i]) > amax ? fabs(x[i]) : amax;
  amax = cosmo_cone::max(amax, width);
  cosmo_cone::sync(width);
  if (w * amax <= t0) return;
  T lo = T(0), hi = amax > t0 / w ? amax : t0 / w;
  if (w * w * lo - w * t0 - excess(x, dim, lo, lane, width) >= T(0)) {
    hi = T(0);
  } else {
    for (int it = 0; it < 200; ++it) {
      const T mid = T(0.5) * (lo + hi);
      if (mid <= lo || mid >= hi) break;
      if (w * w * mid - w * t0 - excess(x, dim, mid, lane, width) < T(0)) lo = mid; else hi = mid;
    }
  }
  const T s = hi;
  cosmo_cone::sync(width);
  for (long long i = 1 + lane; i < dim; i += width) x[i] = x[i] > s ? s : (x[i] < -s ? -s : x[i]);
  if (lane == 0) x[0] = w * s;
}
}
"""


def nonpos_type(hooks=True):
    return M.CustomConeType("nonpos", NONPOS_SRC, "thread", in_dual=hooks, in_pol_recc=hooks)


def soc2_type(hooks=True):
    return M.CustomConeType("soc2", SOC2_SRC, "warp", in_dual=hooks, in_pol_recc=hooks)


def linf_type():
    return M.CustomConeType("wlinf", LINF_SRC, "block", n_params=1)


# ---- the same cones in NumPy ------------------------------------------------
def _nonpos_project(x, p):
    x[:] = np.where(x > 0.0, 0.0, x)


def _soc_project(x, p):
    O.project_cone(x, O.SecondOrderCone(x.shape[0]))


def _linf_project(x, p):
    w, t0 = float(p[0]), float(x[0])
    a = np.abs(x[1:])
    amax = float(a.max()) if a.size else 0.0
    if w * amax <= t0:
        return

    def g(s):
        return w * w * s - w * t0 - float(np.maximum(a - s, 0.0).sum())

    lo, hi = 0.0, max(amax, t0 / w)
    if g(0.0) >= 0.0:
        hi = 0.0
    else:
        for _ in range(200):
            mid = 0.5 * (lo + hi)
            if mid <= lo or mid >= hi:
                break
            if g(mid) < 0.0:
                lo = mid
            else:
                hi = mid
    x[1:] = np.clip(x[1:], -hi, hi)
    x[0] = w * hi


NUMPY = {
    "nonpos": (_nonpos_project, lambda x, tol, p: not np.any(x > -tol), lambda x, tol, p: not np.any(x < tol)),
    "soc2": (_soc_project, lambda x, tol, p: np.linalg.norm(x[1:]) <= tol + x[0],
             lambda x, tol, p: np.linalg.norm(x[1:]) <= tol - x[0]),
    "wlinf": (_linf_project, None, None),
}


class OracleCustomCone:
    """The oracle's custom cone: NumPy callables project(x, params) (in place), in_dual(x, tol, params) and
    in_pol_recc(x, tol, params) (None: the type does not define the hook)."""

    def __init__(self, dim, project, in_dual=None, in_pol_recc=None, params=()):
        self.dim = int(dim)
        self.project, self.in_dual, self.in_pol_recc = project, in_dual, in_pol_recc
        self.params = np.asarray(params, dtype=np.float64)


def install_oracle(monkeypatch):
    """Extend the oracle's dispatch for the duration of one test (pytest's monkeypatch undoes it)."""
    project_cone, in_dual, in_pol_recc = O.project_cone, O.in_dual, O.in_pol_recc

    def project_cone_(x, cone):
        if isinstance(cone, OracleCustomCone):
            cone.project(x, cone.params)
        else:
            project_cone(x, cone)

    def in_dual_(x, cone, tol):
        if isinstance(cone, OracleCustomCone):
            return cone.in_dual is not None and bool(cone.in_dual(x, tol, cone.params))
        return in_dual(x, cone, tol)

    def in_pol_recc_(x, cone, tol):
        if isinstance(cone, OracleCustomCone):
            return cone.in_pol_recc is not None and bool(cone.in_pol_recc(x, tol, cone.params))
        return in_pol_recc(x, cone, tol)

    monkeypatch.setattr(O, "project_cone", project_cone_)
    monkeypatch.setattr(O, "in_dual", in_dual_)
    monkeypatch.setattr(O, "in_pol_recc", in_pol_recc_)
    monkeypatch.setattr(O, "SCALAR_SCALED_CONES", O.SCALAR_SCALED_CONES + (OracleCustomCone,))


def to_oracle(sets):
    """bridge.to_oracle_cones that also translates model.CustomCone (through NUMPY, by type name)"""
    out = []
    for S in sets:
        if isinstance(S, M.CustomCone):
            proj, dual, recc = NUMPY[S.kind.name]
            out.append(OracleCustomCone(S.dim, proj, dual if S.kind.in_dual else None,
                                        recc if S.kind.in_pol_recc else None, S.params))
        else:
            out.extend(to_oracle_cones([S]))
    return out


# ---- the problems of the reference's custom_cone.jl, in model form A x + s = b, s in K ------------------------------
def _model_form(P, q, constraints):
    m = M.Model()
    m.assemble(P, q, constraints)
    return m.P0, m.q0, m.A0, m.b0, m.sets0


def lp_problem(kind):
    """maximise x1 + x2 + x3 s.t. x1 <= 3, x2 <= 2 (a Nonpositives constraint of `kind`), x1 + x3 = 5: objective -7"""
    c1 = M.Constraint(np.eye(2), [-3.0, -2.0], M.CustomCone(kind, 2), 3, (1, 2))
    c2 = M.Constraint(np.array([[1.0, 0.0, 1.0]]), [-5.0], M.ZeroSet(1))
    return _model_form(np.zeros((3, 3)), -np.ones(3), [c1, c2])


def dual_infeasible_problem(kind):
    """minimise x s.t. x - 3 in Nonpositives: unbounded below"""
    return _model_form(np.zeros((1, 1)), np.ones(1), [M.Constraint(np.ones((1, 1)), [-3.0], M.CustomCone(kind, 1))])


def primal_infeasible_problem(kind):
    """x + 1 in Nonpositives and x >= 0: no x"""
    return _model_form(np.zeros((1, 1)), np.ones(1), [M.Constraint(np.ones((1, 1)), [1.0], M.CustomCone(kind, 1)),
                                                      M.Constraint(np.ones((1, 1)), [0.0], M.Nonnegatives(1))])
