"""NumPy/SciPy restatement of the forward derivative of a polished solution (cosmo_b200_derivative, DESIGN.md §3j): the
Jacobian-vector product whose transpose tests/adjoint_reference.py states, through the same solve (scipy's splu of the
regularised K~ of the polish, then refinement against K_A).

TEST INFRASTRUCTURE: the CPU tests pin it against central finite differences of the polished solution map and against
the adjoint restatement (<g, J d> = <J' g, d>), the GPU tests compare the engine with it.  Conventions are the adjoint's:
A x + s = b, y = -mu; rows are described by (cls, l, u) as in polish_reference.  With the active set held fixed:
  K_A [dx; dy_A] = [-dq - dP x - dA' y; db_A - dsbar_A - dA_A x],  dy = 0 off A,  ds = db - dA x - A dx,
  dsbar = dl on lower-active Box rows, du on upper-active ones, (dl + du) / 2 on Box rows with l = u, 0 elsewhere."""
import numpy as np
import scipy.sparse as sp

from tests import adjoint_reference as AR
from tests import polish_reference as R


def bound_direction(cls, kind, dl, du):
    """dsbar of the module docstring (the transpose of the adjoint's dl / du split)."""
    box = cls == R.BOX
    return np.where(box & (kind == R.LOWER), dl,
                    np.where(box & (kind == R.UPPER), du, np.where(box & (kind == R.EQUALITY), 0.5 * (dl + du), 0.0)))


def derivative(P, A, cls, kind, x, y, dPx=None, dq=None, dAx=None, db=None, dl=None, du=None, delta=1e-6,
               refine_iter=3, D=None, E=None, c=1.0):
    """The engine's path: on the scaled data (P, A) of a scaling (D, E, c) (None: unscaled) with the scaled polished point
    (x, y = -mu_p) and the active set `kind`, along the unscaled direction (dPx and dAx in the CSC data order of P and A;
    None: zero).  Returns a dict of the unscaled dx, dy, ds plus the scaled "u", "v" (the solution of K_A), "rx", "rs"
    (its right-hand side) and "refine_residual"."""
    P, A = sp.csc_matrix(P), sp.csc_matrix(A)
    m, n = A.shape
    Dv = np.ones(n) if D is None else np.asarray(D, dtype=float)
    Ev = np.ones(m) if E is None else np.asarray(E, dtype=float)
    z = lambda a, k: np.zeros(k) if a is None else np.asarray(a, dtype=float)
    dPx, dAx, dq, db, dl, du = z(dPx, P.nnz), z(dAx, A.nnz), z(dq, n), z(db, m), z(dl, m), z(du, m)
    # the direction, scaled as the data are
    pr, pc = P.indices, np.repeat(np.arange(n), np.diff(P.indptr))
    ar, ac = A.indices, np.repeat(np.arange(n), np.diff(A.indptr))
    dPs = sp.csc_matrix((c * Dv[pr] * Dv[pc] * dPx, P.indices, P.indptr), shape=P.shape)
    dAs = sp.csc_matrix((Ev[ar] * Dv[ac] * dAx, A.indices, A.indptr), shape=A.shape)
    e = Ev * db - dAs @ x
    rx = -c * Dv * dq - dPs @ x - dAs.T @ y
    rs = np.where(kind != R.INACTIVE, e - bound_direction(cls, kind, Ev * dl, Ev * du), 0.0)
    u, v, r = AR.solve(P, A, kind, rx, rs, delta, refine_iter)
    ds = e - A @ u
    return {"dx": Dv * u, "dy": Ev * v / c, "ds": ds / Ev, "u": u, "v": v, "rx": rx, "rs": rs, "refine_residual": r}
