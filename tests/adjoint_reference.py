"""NumPy/SciPy restatement of the derivatives of a polished solution (cosmo_b200_adjoint, DESIGN.md §3j), on top of
tests/polish_reference.py: the same classification, scipy's splu of the same regularised K~, the same delta and
refinement steps.

TEST INFRASTRUCTURE: the CPU tests pin it against central finite differences of the polished solution map, the GPU
tests compare the engine with it.  Conventions are the engine's: A x + s = b, y = -mu; rows are described by (cls, l, u)
as in polish_reference.  With K_A = [P, A_A'; A_A, 0] and K_A [u; v] = [g_x - A' g_s; g_y on A], v = 0 off A:
  dq = -u,  db = v + g_s,  dP_ij = -(u_i x_j + x_i u_j) / 2,  dA_rj = -(y_r u_j + v_r x_j) - g_s,r x_j,
  dl = -v on lower-active Box rows, du = -v on upper-active ones, both -v / 2 on Box rows with l = u, 0 elsewhere."""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from tests import polish_reference as R


def solve(P, A, kind, rx, rs, delta=1e-6, refine_iter=3):
    """K_A [u; v] = [rx; rs on the active rows]: splu of K~ from z = 0, then refine_iter steps against K_A with v masked
    off the active rows.  Returns (u, v, |r|_inf after the last step)."""
    P, A = sp.csc_matrix(P), sp.csc_matrix(A)
    n = P.shape[0]
    active = kind != R.INACTIVE
    rs = np.where(active, rs, 0.0)
    lu = spla.splu(R.regularised_kkt(P, A, kind, delta))
    z = lu.solve(np.concatenate([rx, rs]))
    u, v = z[:n].copy(), np.where(active, z[n:], 0.0)
    for _ in range(refine_iter):
        ex, es = R.exact_residual(P, -rx, A, kind, rs, u, v)
        dz = lu.solve(np.concatenate([ex, es]))
        u = u + dz[:n]
        v = np.where(active, v + dz[n:], 0.0)
    ex, es = R.exact_residual(P, -rx, A, kind, rs, u, v)
    return u, v, max(np.abs(ex).max(initial=0.0), np.abs(es).max(initial=0.0))


def kkt_matrix(P, A, kind):
    """K_A as a dense matrix (for condition numbers)."""
    act = np.flatnonzero(kind != R.INACTIVE)
    Aa = sp.csc_matrix(A)[act]
    return sp.bmat([[sp.csc_matrix(P), Aa.T], [Aa, None]], format="csc").toarray()


def gradients(P, A, cls, kind, x, y, u, v, gs):
    """The formulas of the module docstring: dict of dq, db, dPx, dAx (the CSC data order of P and A), dl, du."""
    P, A = sp.csc_matrix(P), sp.csc_matrix(A)
    pr, pc = P.indices, np.repeat(np.arange(P.shape[1]), np.diff(P.indptr))
    ar, ac = A.indices, np.repeat(np.arange(A.shape[1]), np.diff(A.indptr))
    box = cls == R.BOX
    dl = np.where(box & (kind == R.LOWER), -v, 0.0)
    du = np.where(box & (kind == R.UPPER), -v, 0.0)
    eq = box & (kind == R.EQUALITY)
    dl = np.where(eq, -0.5 * v, dl)
    du = np.where(eq, -0.5 * v, du)
    return {"dq": -u, "db": v + gs, "dPx": -0.5 * (u[pr] * x[pc] + x[pr] * u[pc]),
            "dAx": -(y[ar] * u[ac] + v[ar] * x[ac]) - gs[ar] * x[ac], "dl": dl, "du": du}


def adjoint(P, A, cls, kind, x, y, gx=None, gy=None, gs=None, delta=1e-6, refine_iter=3, D=None, E=None, c=1.0):
    """The engine's path: on the scaled data (P, A) of a scaling (D, E, c) (None: unscaled) with the scaled polished point
    (x, y = -mu_p) and the active set `kind`, from the unscaled incoming gradients.  Returns the unscaled gradients (dict
    of gradients()) plus "u", "v" (scaled) and "refine_residual"."""
    P, A = sp.csc_matrix(P), sp.csc_matrix(A)
    m, n = A.shape
    Dv = np.ones(n) if D is None else np.asarray(D, dtype=float)
    Ev = np.ones(m) if E is None else np.asarray(E, dtype=float)
    gx = np.zeros(n) if gx is None else gx
    gy = np.zeros(m) if gy is None else gy
    gs = np.zeros(m) if gs is None else gs
    gs_t = gs / Ev
    rx = Dv * gx - A.T @ gs_t
    rs = np.where(kind != R.INACTIVE, Ev * gy / c, 0.0)
    u, v, r = solve(P, A, kind, rx, rs, delta, refine_iter)
    g = gradients(P, A, cls, kind, x, y, u, v, gs_t)
    pr, pc = P.indices, np.repeat(np.arange(n), np.diff(P.indptr))
    ar, ac = A.indices, np.repeat(np.arange(n), np.diff(A.indptr))
    out = {"dq": c * Dv * g["dq"], "db": Ev * g["db"], "dPx": c * (Dv[pr] * Dv[pc]) * g["dPx"],
           "dAx": Ev[ar] * Dv[ac] * g["dAx"], "dl": Ev * g["dl"], "du": Ev * g["du"]}
    out.update(u=u, v=v, refine_residual=r)
    return out
