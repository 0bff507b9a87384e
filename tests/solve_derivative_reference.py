"""NumPy/SciPy restatement of the forward derivative of a conic solution through the fixed point of the ADMM iteration
(cosmo_b200_solve_derivative, DESIGN.md §3l): the Jacobian-vector product whose transpose tests/solve_adjoint_reference.py
states.

TEST INFRASTRUCTURE: the CPU tests pin it against central finite differences of oracle solves and against the adjoint
restatement (<g, J d> = <J' g, d>), the GPU tests compare the engine with it.  Conventions are the adjoint's: A x + s = b,
y = -mu, cones as the oracle's cone objects.  In scaled coordinates, with w_s = s + mu / rho, Dpi = DPi(w_s) and
K = [P + sigma I, A'; A, -diag(1 / rho)], for the scaled direction (dP, dq, dA, db, dl, du):
  dPi = dl on Box rows with w_s <= l, du with w_s >= u, (dl + du) / 2 on those with l = u, 0 elsewhere,
  [x'; nu'] = K^-1 [-dq - dP x - dA' y; db - 2 dPi - dA x],  t = [x'; dPi - nu' / rho],
  (I - M) v = [v_x - a; v_s + b / rho - h],  h = Dpi v_s,  [a; b] = K^-1 [sigma v_x; v_s - 2 h],
  solve (I - M) w' = t (GMRES),  dx = w'_x,  ds = Dpi w'_s + dPi,  dy = -rho (w'_s - ds)."""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from tests.solve_adjoint_reference import box_bounds, dpi


def derivative(P, A, cones, x, s, mu, rho, sigma=1e-6, dPx=None, dq=None, dAx=None, db=None, dl=None, du=None, D=None,
               E=None, c=1.0, tol=1e-12, restart=30, maxiter=2000):
    """The engine's path on the scaled data (P, A, cones with scaled Box bounds) of a scaling (D, E, c) (None: unscaled)
    at the scaled point (x, s, mu) with the rho vector `rho`, along the unscaled direction (dPx and dAx in the CSC data
    order of P and A; None: zero).  Returns a dict of the unscaled derivatives dx, dy, ds plus "w", "t", "residual" and
    "apps"."""
    P, A = sp.csc_matrix(P), sp.csc_matrix(A)
    m, n = A.shape
    rho = np.broadcast_to(np.asarray(rho, dtype=float), (m,)).copy()
    Dv = np.ones(n) if D is None else np.asarray(D, dtype=float)
    Ev = np.ones(m) if E is None else np.asarray(E, dtype=float)
    z = lambda a, k: np.zeros(k) if a is None else np.asarray(a, dtype=float)
    dPx, dAx, dq, db, dl, du = z(dPx, P.nnz), z(dAx, A.nnz), z(dq, n), z(db, m), z(dl, m), z(du, m)
    # the direction, scaled as the data are
    pr, pc = P.indices, np.repeat(np.arange(n), np.diff(P.indptr))
    ar, ac = A.indices, np.repeat(np.arange(n), np.diff(A.indptr))
    dPs = sp.csc_matrix((c * Dv[pr] * Dv[pc] * dPx, P.indices, P.indptr), shape=P.shape)
    dAs = sp.csc_matrix((Ev[ar] * Dv[ac] * dAx, A.indices, A.indptr), shape=A.shape)
    dqs, dbs, dls, dus = c * Dv * dq, Ev * db, Ev * dl, Ev * du
    ws = s + mu / rho
    y = -mu
    l, ub, box = box_bounds(cones, m)
    lower, upper = box & (ws <= l), box & ~(ws <= l) & (ws >= ub)
    eq = box & (l == ub)
    dPi = np.where(eq & (lower | upper), 0.5 * (dls + dus), np.where(lower, dls, np.where(upper, dus, 0.0)))
    K = sp.bmat([[P + sigma * sp.identity(n), A.T], [A, sp.diags(-1.0 / rho)]], format="csc")
    lu = spla.splu(K)
    zt = lu.solve(np.concatenate([-dqs - dPs @ x - dAs.T @ y, dbs - 2 * dPi - dAs @ x]))
    t = np.concatenate([zt[:n], dPi - zt[n:] / rho])
    apps = [0]

    def op(v):
        apps[0] += 1
        h = dpi(ws, cones, v[n:])
        ab = lu.solve(np.concatenate([sigma * v[:n], v[n:] - 2 * h]))
        return np.concatenate([v[:n] - ab[:n], v[n:] + ab[n:] / rho - h])

    L = spla.LinearOperator((n + m, n + m), matvec=op, dtype=float)
    if np.linalg.norm(t) == 0:
        w = np.zeros(n + m)
    else:
        w, info = spla.gmres(L, t, rtol=tol, atol=0.0, restart=restart, maxiter=maxiter)
        assert info == 0, info
    res = np.linalg.norm(t - op(w)) / max(np.linalg.norm(t), 1e-300)
    dxs = w[:n]
    dss = dpi(ws, cones, w[n:]) + dPi
    dys = -rho * (w[n:] - dss)
    return {"dx": Dv * dxs, "ds": dss / Ev, "dy": Ev * dys / c, "w": w, "t": t, "residual": res, "apps": apps[0]}


def unscaled(P, A, cones, x, s, y, rho=0.1, sigma=1e-6, **kw):
    """derivative() of an unscaled problem at its solution (x, s, y): mu = -y, one rho for every row."""
    return derivative(P, A, cones, x, s, -np.asarray(y, dtype=float), rho, sigma, **kw)
