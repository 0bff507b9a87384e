"""NumPy/SciPy restatement of solution polishing (cosmo_b200_polish, DESIGN.md §3i), steps 1-6 on the scaled data.

TEST INFRASTRUCTURE, like tests/infeasibility_reference.py: the CPU tests pin it against exact reduced-KKT solves and
the reference's known answers, the GPU tests compare the engine with it.  The regularised solve is scipy's splu of
K~ = [P + delta I, A'; A, -diag(1 / rho)].

Conventions are the engine's: A x + s = b with s in K, mu = rho (w_s - s), y = -mu, nu = -mu the second unknown of
the KKT system.  Rows are described by (cls, l, u): cls 0 ZeroSet, 1 Nonnegatives, 2 Box (l, u are only read on Box
rows)."""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from oracle import cosmo_oracle as O

ZERO, NONNEG, BOX = 0, 1, 2
INACTIVE, LOWER, UPPER, EQUALITY = 0, 1, 2, 3


def row_classes(cones):
    """(cls, l, u) of a list of oracle cones; ValueError for a set with no finite active set."""
    cls, lo, up = [], [], []
    for c in cones:
        if isinstance(c, O.ZeroSet):
            cls += [ZERO] * c.dim
        elif isinstance(c, O.Nonnegatives):
            cls += [NONNEG] * c.dim
        elif isinstance(c, O.Box):
            cls += [BOX] * c.dim
            lo += list(np.asarray(c.l, dtype=float))
            up += list(np.asarray(c.u, dtype=float))
            continue
        else:
            raise ValueError("polishing applies to ZeroSet, Nonnegatives and Box rows only, not %s" % type(c).__name__)
        lo += [-np.inf] * c.dim
        up += [np.inf] * c.dim
    return np.array(cls, dtype=np.int8), np.array(lo), np.array(up)


def classify(cls, l, u, s, mu):
    """Step 1: (kind, sbar) of every row."""
    m = len(cls)
    kind = np.zeros(m, dtype=np.int8)
    sbar = np.zeros(m)
    with np.errstate(invalid="ignore"):
        for i in range(m):
            if cls[i] == ZERO:
                kind[i] = EQUALITY
            elif cls[i] == NONNEG:
                if s[i] < -mu[i]:
                    kind[i] = LOWER
            elif cls[i] == BOX:
                if l[i] == u[i]:
                    kind[i], sbar[i] = EQUALITY, l[i]
                elif s[i] - l[i] < -mu[i]:
                    kind[i], sbar[i] = LOWER, l[i]
                elif u[i] - s[i] < mu[i]:
                    kind[i], sbar[i] = UPPER, u[i]
    return kind, sbar


def regularised_kkt(P, A, kind, delta):
    """Step 3: K~ with sigma = delta, rho = 1/delta on the active rows and delta elsewhere."""
    n = P.shape[0]
    active = kind != INACTIVE
    rho = np.where(active, 1.0 / delta, delta)
    return sp.bmat([[sp.csc_matrix(P) + delta * sp.identity(n), A.T], [A, -sp.diags(1.0 / rho)]], format="csc")


def exact_residual(P, q, A, kind, rhs, x, nu):
    """r^ - K_A z of the exact reduced system embedded in n + m rows (0 on the inactive rows)."""
    active = kind != INACTIVE
    rx = -q - (P @ x + A.T @ nu)
    rs = np.where(active, rhs - A @ x, 0.0)
    return rx, rs


def refine(P, q, A, b, kind, sbar, delta=1e-6, refine_iter=3, x0=None, nu0=None):
    """Steps 3-4: (x, nu, |r|_inf after the last step).  The regularised solve is centred at z0 = (x0, nu0) (zero when
    not given; the ADMM iterate in polish): K~ z = r^ + (K~ - K_A) z0 = [-q + delta x0; b - sbar - delta nu0 on the active
    rows, 0 elsewhere], the first refinement step from z0 written without a product."""
    n, m = P.shape[0], A.shape[0]
    active = kind != INACTIVE
    rhs = np.where(active, b - sbar, 0.0)
    x0 = np.zeros(n) if x0 is None else x0
    nu0 = np.zeros(m) if nu0 is None else np.where(active, nu0, 0.0)
    lu = spla.splu(regularised_kkt(P, A, kind, delta))
    z = lu.solve(np.concatenate([-q + delta * x0, rhs - delta * nu0]))
    x, nu = z[:n].copy(), np.where(active, z[n:], 0.0)
    for _ in range(refine_iter):
        rx, rs = exact_residual(P, q, A, kind, rhs, x, nu)
        dz = lu.solve(np.concatenate([rx, rs]))
        x = x + dz[:n]
        nu = np.where(active, nu + dz[n:], 0.0)
    rx, rs = exact_residual(P, q, A, kind, rhs, x, nu)
    return x, nu, max(np.abs(rx).max(initial=0.0), np.abs(rs).max(initial=0.0))


def project(w, cls, l, u):
    """Pi_K of the elementwise sets."""
    s = np.where(cls == NONNEG, np.maximum(w, 0.0), w)
    s = np.where(cls == BOX, np.minimum(np.maximum(w, l), u), s)
    return np.where(cls == ZERO, 0.0, s)


def candidate_mu(kind, nu):
    """Step 5: mu_p = -nu on the active rows, clipped into the normal cone of the row's set at sbar."""
    mu = -nu
    mu = np.where(kind == LOWER, np.minimum(mu, 0.0), mu)
    mu = np.where(kind == UPPER, np.maximum(mu, 0.0), mu)
    return np.where(kind == INACTIVE, 0.0, mu)


def residuals(P, q, A, b, x, s, mu, D=None, E=None, c=1.0):
    """compute_residuals (residuals.jl:30-96, 143-147): (r_prim, r_dual, max_norm_prim, max_norm_dual, obj), unscaled
    by E^-1 and c^-1 D^-1 when D and E are given."""
    Einv = 1.0 / E if E is not None else np.ones(len(b))
    Dc = (1.0 / D if D is not None else np.ones(len(q))) / c
    ax, px, atmu = A @ x, P @ x, A.T @ mu
    rp = np.abs(Einv * (ax + s - b)).max(initial=0.0)
    mp = max(np.abs(Einv * ax).max(initial=0.0), np.abs(Einv * s).max(initial=0.0), np.abs(Einv * b).max(initial=0.0))
    rd = np.abs(Dc * (px + q - atmu)).max(initial=0.0)
    md = max(np.abs(Dc * px).max(initial=0.0), np.abs(Dc * q).max(initial=0.0), np.abs(Dc * atmu).max(initial=0.0))
    return rp, rd, mp, md, (0.5 * x @ px + q @ x) / c


def polish(P, q, A, b, cls, l, u, x, s, mu, delta=1e-6, refine_iter=3, D=None, E=None, c=1.0, unit_roundoff=2.0 ** -53):
    """Steps 1-6 on the scaled data (P, q, A, b, l, u) and the scaled iterates (x, s, mu).  Returns a dict: status (1 or
    0), the counts, the candidate (x, s, mu, scaled), its residuals, the refinement residual and the accepted solution
    in the original coordinates (x, y, s) -- the candidate's on status 1, the iterates' otherwise."""
    P, A = sp.csc_matrix(P), sp.csc_matrix(A)
    kind, sbar = classify(cls, l, u, s, mu)
    xp, nu, rref = refine(P, q, A, b, kind, sbar, delta, refine_iter, x, -mu)
    sp_ = project(b - A @ xp, cls, l, u)
    mup = candidate_mu(kind, nu)
    cand = residuals(P, q, A, b, xp, sp_, mup, D, E, c)
    unp = residuals(P, q, A, b, x, s, mu, D, E, c)
    finite = all(np.isfinite(v) for v in cand) and np.isfinite(rref)
    ok = finite and cand[0] <= max(unp[0], 10 * unit_roundoff * (1 + cand[2])) and \
        cand[1] <= max(unp[1], 10 * unit_roundoff * (1 + cand[3]))
    X, S, MU = (xp, sp_, mup) if ok else (x, s, mu)
    Dv = D if D is not None else np.ones(len(q))
    Ev = E if E is not None else np.ones(len(b))
    return {"status": 1 if ok else 0, "n_lower": int((kind == LOWER).sum()), "n_upper": int((kind == UPPER).sum()),
            "n_equality": int((kind == EQUALITY).sum()), "kind": kind, "x_p": xp, "s_p": sp_, "mu_p": mup,
            "r_prim": cand[0], "r_dual": cand[1], "obj_val": cand[4], "refine_residual": rref, "unpolished": unp,
            "x": Dv * X, "y": -(Ev * MU) / c, "s": S / Ev}
