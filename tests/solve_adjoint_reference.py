"""NumPy/SciPy restatement of the derivatives of a conic solution through the fixed point of the ADMM iteration
(cosmo_b200_solve_adjoint, DESIGN.md §3k).

TEST INFRASTRUCTURE: the CPU tests pin it against central finite differences of the oracle's projections and solves,
the GPU tests compare the engine with it.  Conventions are the engine's: A x + s = b, y = -mu, cones as the oracle's
cone objects (tests use oracle.bridge.to_oracle_cones).  In scaled coordinates, with w_s = s + mu / rho, Dpi = DPi(w_s)
and K = [P + sigma I, A'; A, -diag(1 / rho)]:
  gw = [gx~; Dpi(gs~ + rho gy~) - rho gy~],   (I - M') lam = lam - [sigma a; b + Dpi(lam_s - 2 b)],
  [a; b] = K^-1 [lam_x; -lam_s / rho],   solve (I - M') lam = gw (GMRES),   [u; v] = K^-1 [lam_x; -lam_s / rho],
  dq = -u,  db = v,  dP_ij = -(u_i x_j + x_i u_j) / 2,  dA_rj = -(v_r x_j + y_r u_j),
  Box rows with w_s <= l: dl = lam_s - 2 v + gs~ + rho gy~, with w_s >= u the same in du, half each when l = u."""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from oracle import cosmo_oracle as O

SQRT2 = np.sqrt(2.0)


def _tri_to_mat(x, N):
    """svec (sqrt 2 scaled upper triangle, column by column) -> symmetric N x N matrix."""
    X = np.zeros((N, N))
    iu = np.triu_indices(N)
    order = np.lexsort((iu[0], iu[1]))          # column-major upper triangle
    r, c = iu[0][order], iu[1][order]
    v = np.where(r == c, x, x / SQRT2)
    X[r, c] = v
    X[c, r] = v
    return X


def _mat_to_tri(X):
    N = X.shape[0]
    iu = np.triu_indices(N)
    order = np.lexsort((iu[0], iu[1]))
    r, c = iu[0][order], iu[1][order]
    return np.where(r == c, X[r, c], SQRT2 * X[r, c])


def _psd_N(cone):
    if isinstance(cone, O.PsdConeTriangle):
        return int(round((np.sqrt(8 * cone.dim + 1) - 1) / 2))
    return int(round(np.sqrt(cone.dim)))


def gamma(lam):
    """Gamma_ij of the PSD Jacobian in its branch forms."""
    li, lj = lam[:, None], lam[None, :]
    pi, pj = li > 0, lj > 0
    G = np.where(pi & pj, 1.0, 0.0)
    with np.errstate(divide="ignore", invalid="ignore"):
        G = np.where(pi & ~pj, li / (li - lj), G)
        G = np.where(~pi & pj, lj / (lj - li), G)
    return G


def dpi(w, cones, h):
    """Dpi(w) h, cone by cone."""
    out = np.zeros_like(h)
    k = 0
    for cone in cones:
        d = cone.dim
        sl = slice(k, k + d)
        ws, hs = w[sl], h[sl]
        if isinstance(cone, O.ZeroSet):
            out[sl] = 0.0
        elif isinstance(cone, O.Nonnegatives):
            out[sl] = np.where(ws > 0, hs, 0.0)
        elif isinstance(cone, O.Box):
            out[sl] = np.where((ws > cone.l) & (ws < cone.u), hs, 0.0)
        elif isinstance(cone, O.SecondOrderCone):
            t, xb = ws[0], ws[1:]
            r = np.linalg.norm(xb)
            if r <= t:
                out[sl] = hs
            elif r <= -t:
                out[sl] = 0.0
            else:
                dot = xb @ hs[1:]
                o = np.empty(d)
                o[0] = 0.5 * (hs[0] + dot / r)
                o[1:] = 0.5 * (xb / r * hs[0] + (1 + t / r) * hs[1:] - (t / r) * xb * dot / r ** 2)
                out[sl] = o
        elif isinstance(cone, (O.PsdConeTriangle, O.PsdCone)):
            N = _psd_N(cone)
            tri = isinstance(cone, O.PsdConeTriangle)
            if tri:
                W, H = _tri_to_mat(ws, N), _tri_to_mat(hs, N)
            else:
                W, H = ws.reshape(N, N, order="F"), hs.reshape(N, N, order="F")
                W, H = (W + W.T) / 2, (H + H.T) / 2
            lam, Q = np.linalg.eigh(W)
            C = gamma(lam) * (Q.T @ H @ Q)
            X = Q @ C @ Q.T
            X = (X + X.T) / 2
            out[sl] = _mat_to_tri(X) if tri else X.reshape(-1, order="F")
        else:
            raise TypeError("no Jacobian for %r" % (cone,))
        k += d
    return out


def box_bounds(cones, m):
    l, u, box = np.full(m, -np.inf), np.full(m, np.inf), np.zeros(m, dtype=bool)
    k = 0
    for cone in cones:
        if isinstance(cone, O.Box):
            l[k:k + cone.dim], u[k:k + cone.dim], box[k:k + cone.dim] = cone.l, cone.u, True
        k += cone.dim
    return l, u, box


def adjoint(P, A, cones, x, s, mu, rho, sigma=1e-6, gx=None, gy=None, gs=None, D=None, E=None, c=1.0, tol=1e-12,
            restart=30, maxiter=2000):
    """The engine's path on the scaled data (P, A, cones with scaled Box bounds) of a scaling (D, E, c) (None: unscaled)
    at the scaled point (x, s, mu) with the rho vector `rho`, from the unscaled incoming gradients.  Returns a dict of
    the unscaled gradients dq, db, dPx, dAx (CSC data order), dl, du, plus "lam", "u", "v", "residual" and "apps"."""
    P, A = sp.csc_matrix(P), sp.csc_matrix(A)
    m, n = A.shape
    rho = np.broadcast_to(np.asarray(rho, dtype=float), (m,)).copy()
    Dv = np.ones(n) if D is None else np.asarray(D, dtype=float)
    Ev = np.ones(m) if E is None else np.asarray(E, dtype=float)
    gx = np.zeros(n) if gx is None else np.asarray(gx, dtype=float)
    gy = np.zeros(m) if gy is None else np.asarray(gy, dtype=float)
    gs = np.zeros(m) if gs is None else np.asarray(gs, dtype=float)
    gxt, gst, gyt = Dv * gx, gs / Ev, Ev * gy / c
    ws = s + mu / rho
    K = sp.bmat([[P + sigma * sp.identity(n), A.T], [A, sp.diags(-1.0 / rho)]], format="csc")
    lu = spla.splu(K)

    def kinv(lam):
        z = lu.solve(np.concatenate([lam[:n], -lam[n:] / rho]))
        return z[:n], z[n:]

    apps = [0]

    def op(lam):
        apps[0] += 1
        a, b = kinv(lam)
        return lam - np.concatenate([sigma * a, b + dpi(ws, cones, lam[n:] - 2 * b)])

    gw = np.concatenate([gxt, dpi(ws, cones, gst + rho * gyt) - rho * gyt])
    L = spla.LinearOperator((n + m, n + m), matvec=op, dtype=float)
    if np.linalg.norm(gw) == 0:
        lam = np.zeros(n + m)
    else:
        lam, info = spla.gmres(L, gw, rtol=tol, atol=0.0, restart=restart, maxiter=maxiter)
        assert info == 0, info
    res = np.linalg.norm(gw - op(lam)) / max(np.linalg.norm(gw), 1e-300)
    u, v = kinv(lam)
    y = -mu
    l, ub, box = box_bounds(cones, m)
    val = lam[n:] - 2 * v + gst + rho * gyt
    lower, upper = box & (ws <= l), box & ~(ws <= l) & (ws >= ub)
    eq = box & (l == ub)
    dl = np.where(eq & (lower | upper), 0.5 * val, np.where(lower, val, 0.0))
    du = np.where(eq & (lower | upper), 0.5 * val, np.where(upper, val, 0.0))
    pr, pc = P.indices, np.repeat(np.arange(n), np.diff(P.indptr))
    ar, ac = A.indices, np.repeat(np.arange(n), np.diff(A.indptr))
    dPt = -0.5 * (u[pr] * x[pc] + x[pr] * u[pc])
    dAt = -(v[ar] * x[ac] + y[ar] * u[ac])
    return {"dq": -c * Dv * u, "db": Ev * v, "dPx": c * Dv[pr] * Dv[pc] * dPt, "dAx": Ev[ar] * Dv[ac] * dAt,
            "dl": Ev * dl, "du": Ev * du, "lam": lam, "u": u, "v": v, "residual": res, "apps": apps[0]}


def unscaled(P, A, cones, x, s, y, rho=0.1, sigma=1e-6, **kw):
    """adjoint() of an unscaled problem at its solution (x, s, y): mu = -y, one rho for every row."""
    return adjoint(P, A, cones, x, s, -np.asarray(y, dtype=float), rho, sigma, **kw)
