"""A stand-in for cosmo_b200.engine.Engine that answers with the CPU oracle (tests only).

It exists to exercise, without a GPU, the Python side of everything that normally talks to the CUDA engine: the host
glue of Model (scaling, decomposition, warm starts) and the bodies of the GPU tests themselves (so a typo in a GPU
test is found by the CPU run, not at the next GPU run).  It implements the part of the call surface those users need:
ctor, update_settings, warm_start, update_qb, update_matrices, project, project_jacobian, solve, w, rho_vec, scaling,
spmv, residuals, close, the infeasibility hooks infeasibility_test and psd_lambda_max, and set_accelerator with the
accelerator_probe hook."""
import numpy as np
import scipy.sparse as sp

from cosmo_b200 import engine as E
from oracle import cosmo_oracle as O

_PLAIN = {E.ZERO: O.ZeroSet, E.NONNEG: O.Nonnegatives, E.SOC: O.SecondOrderCone, E.PSD_SQUARE: O.PsdCone,
          E.PSD_TRIANGLE: O.PsdConeTriangle, E.PSD_TRIANGLE_COMPLEX: O.ComplexPsdConeTriangle}
_FAMILY = {O.ZeroSet: E.FAMILY_ROWS, O.Nonnegatives: E.FAMILY_ROWS, O.Box: E.FAMILY_ROWS, O.SecondOrderCone: E.FAMILY_SOC,
           O.PsdCone: E.FAMILY_PSD, O.PsdConeTriangle: E.FAMILY_PSD, O.ComplexPsdConeTriangle: E.FAMILY_PSD}


def cones_from_tuples(sets):
    out = []
    for t in sets:
        typ, dim, l, u = t[:4]
        extra = t[4] if len(t) > 4 and t[4] else {}
        if typ == E.BOX:
            out.append(O.Box(l, u))
        elif typ == E.EXP:
            out.append(O.ExponentialCone())
        elif typ == E.DUAL_EXP:
            out.append(O.DualExponentialCone())
        elif typ == E.POW:
            out.append(O.PowerCone(extra["alpha"]))
        elif typ == E.DUAL_POW:
            out.append(O.DualPowerCone(extra["alpha"]))
        else:
            out.append(_PLAIN[typ](dim))
    return out


class OracleEngine:
    instances = []

    def __init__(self, P, q, A, b, sets, settings=None, D=None, E=None, c=1.0, dtype=np.float64, device=0, julia_indexing=True,
                 equilibrate=False):
        self._args = (P, q, A, b, sets, settings, D, E, c, dtype, device, julia_indexing, equilibrate)
        self.P, self.q = sp.csc_matrix(P), np.array(q, dtype=float)
        self.A, self.b = sp.csc_matrix(A), np.array(b, dtype=float)
        self.m, self.n = self.A.shape
        self.dtype = np.dtype(dtype)
        self.cones = cones_from_tuples(sets)
        self.st = settings
        self.scaled = D is not None
        self._scal = (np.ones(self.n), np.ones(self.m), 1.0) if D is None else (np.array(D), np.array(E), float(c))
        if equilibrate and D is None and settings is not None and settings.scaling != 0:
            # like the engine: unscaled data + scaling requested -> equilibrate here (scale_ruiz!)
            ost = O.Settings(scaling=int(settings.scaling), MIN_SCALING=settings.MIN_SCALING, MAX_SCALING=settings.MAX_SCALING)
            Ps, qs, As, bs, cones, sm = O.scale_ruiz(self.P, self.q, self.A, self.b, self.cones, ost)
            Ps = sp.csc_matrix(Ps)
            Ps = sp.csc_matrix((Ps + Ps.T) / 2)      # symmetrize_full!, scaling.jl:99
            self.P, self.q, self.A, self.b, self.cones = Ps, qs, sp.csc_matrix(As), bs, cones
            self._scal = (sm.D, sm.E, sm.c)
            self.scaled = True
        self._w = self._rho = self._warm = None
        self._acc = None
        OracleEngine.instances.append(self)

    def scaling(self):
        return self._scal

    def psd_stats(self):
        return {"tc_projections": 0, "tc_fallbacks": 0}

    def update_settings(self, st):
        self.st = st

    def warm_start(self, x, s, mu):
        self._warm = (np.array(x), np.array(s), np.array(mu))

    def update_qb(self, q=None, b=None):
        if q is not None:
            self.q = np.array(q, dtype=float)
        if b is not None:
            self.b = np.array(b, dtype=float)

    def update_matrices(self, Px=None, Ax=None, q=None, b=None):
        """new values on the pattern of create: the stand-in is rebuilt from the new unscaled data"""
        P, q0, A, b0, *rest = self._args
        P, A = sp.csc_matrix(P, copy=True), sp.csc_matrix(A, copy=True)
        P.sort_indices()
        A.sort_indices()
        if Px is not None:
            P.data = np.array(Px, dtype=float)
        if Ax is not None:
            A.data = np.array(Ax, dtype=float)
        OracleEngine.instances.remove(self)
        self.__init__(P, q0 if q is None else q, A, b0 if b is None else b, *rest)

    def spmv(self, which, x):
        x = np.asarray(x, dtype=float)
        M = {0: self.A, 1: self.A.T, 2: self.P}[which]
        return (M @ x).astype(self.dtype)

    def residuals(self, x, s, mu, ignore_scaling=False):
        """(r_prim, r_dual, max_norm_prim, max_norm_dual, cost) of the resident (scaled) data, unscaled unless
        ignore_scaling, as cosmo_b200_residuals"""
        x, s, mu = (np.asarray(v, dtype=float) for v in (x, s, mu))
        D, Em, c = self._scal if not ignore_scaling else (np.ones(self.n), np.ones(self.m), 1.0)
        Ax, Px, Aty = self.A @ x, self.P @ x, self.A.T @ mu
        nrm = lambda v: float(np.max(np.abs(v))) if v.size else 0.0
        return (nrm((Ax + s - self.b) / Em), nrm((Px + self.q - Aty) / D / c), max(nrm(Ax / Em), nrm(s / Em), nrm(self.b / Em)),
                max(nrm(Px / D / c), nrm(Aty / D / c), nrm(self.q / D / c)), (0.5 * x @ Px + self.q @ x) / self._scal[2])

    def project(self, ws):
        out = np.array(ws, dtype=float).copy()
        O.project(out, self.cones)
        return out.astype(self.dtype)

    def project_jacobian(self, w_s, h, out=None):
        """Dpi(w_s) h from the double-double reference, with its kink counts (no eigensolve misses here)"""
        from tests import projection_jacobian_reference as R
        w = np.asarray(w_s, dtype=float)
        u = 2.0 ** -24 if self.dtype == np.float32 else 2.0 ** -53
        res = R.dpi(w, self.cones, np.asarray(h, dtype=float)).astype(self.dtype)
        if out is not None:
            out[:] = res
            res = out
        counts = dict(zip(E.PROJECT_JACOBIAN_STATS, R.kink_counts(w, self.cones, u) + (0,)))
        return res, counts

    def solve(self):
        st = self.st
        ost = O.Settings(scaling=0, kkt_solver="cg", eps_abs=st.eps_abs, eps_rel=st.eps_rel, max_iter=st.max_iter, rho=st.rho,
                         check_termination=st.check_termination, check_infeasibility=st.check_infeasibility,
                         adaptive_rho=bool(st.adaptive_rho), adaptive_rho_interval=st.adaptive_rho_interval,
                         adaptive_rho_max_adaptions=st.adaptive_rho_max_adaptions,
                         accelerator="anderson" if st.accelerator == E.ACC_ANDERSON else "empty",
                         accelerator_mem=st.accelerator_mem, safeguard=bool(st.safeguard), safeguard_tol=st.safeguard_tol)
        r = O.solve(self.P, self.q, self.A, self.b, self.cones, ost)
        self._w, self._rho = r.w, r.rho_vec
        out = E.SolveOutput()
        out.x, out.s, out.mu = r.x, r.s, -r.y
        out.obj_val, out.iter, out.safeguarding_iter, out.status = r.obj_val, r.iter, r.safeguarding_iter, r.status
        out.r_prim, out.r_dual, out.max_norm_prim, out.max_norm_dual = r.info.r_prim, r.info.r_dual, 0.0, 0.0
        out.rho, out.rho_updates, out.times = 0.1, list(r.info.rho_updates), {"iter_time_device": 0.0}
        out.kkt_inner_iterations = out.kkt_multiplications = out.kernel_launches = 0
        return out

    def set_accelerator(self, acc):
        self._acc = acc

    def accelerator_probe(self, g, x, w_next=None):
        """cosmo_b200_accelerator_probe through the two fp64 restatements: oracle.cosmo_oracle.AndersonAccelerator for
        Type2{QRDecomp}, tests/anderson_variants.NormalEquationsAccelerator for the others"""
        from cosmo_b200 import model as M
        from tests import anderson_variants as V
        names = lambda table, v: {i: k for k, i in table.items()}[v]
        a = self._acc
        t = "Type2{QRDecomp}" if a is None else names(M.Settings._AA_TYPE, a.type)
        memory = "RestartedMemory" if a is None else names(M.Settings._AA_MEMORY, a.memory)
        reg = "NoRegularizer" if a is None else names(M.Settings._AA_REG, a.regularizer)
        lam = 0.0 if a is None else float(self.dtype.type(a.lambda_))
        dim = self.n + self.m
        g = np.asarray(g, dtype=self.dtype).reshape(-1, dim)
        x = np.asarray(x, dtype=self.dtype).reshape(-1, dim)
        K = g.shape[0]
        if x.shape[0] != K:
            raise E.EngineError(E.ERR_INVALID, "g and x must hold the same number of vectors")
        if t == "Type2{QRDecomp}":
            aa = O.AndersonAccelerator(dim, self.st.accelerator_mem, self.st.accelerator_min_mem)
        else:
            aa = V.NormalEquationsAccelerator(dim, self.st.accelerator_mem, self.st.accelerator_min_mem,
                                              type1=t == "Type1", rolling=memory == "RollingMemory", regularizer=reg,
                                              lam=lam)
        out = {"cand": g.copy(), "eta": np.full((K, 32), np.nan), "formed": np.zeros(K, dtype=np.int64),
               "accepted": np.zeros(K, dtype=np.int64), "l": np.zeros(K, dtype=np.int64), "j": np.full(K, -1, dtype=np.int64)}
        sg = np.full((K, 3), np.nan)
        with np.errstate(all="ignore"):
            for k in range(K):
                gk, xk = g[k].astype(float), x[k].astype(float)
                init = aa.init_phase
                rejected = len([e for e in aa.log if e[1] == "acc_failed"])
                aa.update(gk, xk, k)
                j = aa.j if hasattr(aa, "j") else (aa.iter - 1) % aa.mem
                l = 0 if init else min(aa.iter, aa.mem)
                cand = gk.copy()
                aa.accelerate(cand, xk, k)
                formed = aa.success or len([e for e in aa.log if e[1] == "acc_failed"]) > rejected
                out["formed"][k], out["accepted"][k], out["l"][k] = formed, aa.success, l
                out["j"][k] = -1 if init else j
                if aa.success:
                    out["cand"][k] = cand.astype(self.dtype)
                    out["eta"][k, :l] = aa.eta[:l]
                if w_next is not None:
                    wn = np.asarray(w_next, dtype=self.dtype).reshape(K, dim)[k].astype(float)
                    nf, nacc = np.linalg.norm(aa.f), np.linalg.norm(out["cand"][k].astype(float) - wn)
                    sg[k] = (float(nacc > nf * self.st.safeguard_tol), nf, nacc)
        if w_next is not None:
            out.update(declined=sg[:, 0] == 1.0, nrm_f=sg[:, 1], nrm_f_acc=sg[:, 2])
        return out

    def accelerator_stats(self):
        return dict.fromkeys(E.ACCELERATOR_STATS, 0)

    def infeasibility_test(self, which, delta):
        """cosmo_b200_infeasibility_test through the oracle's scaled_norm / in_dual / in_pol_recc / support_function"""
        D, Em, c = self._scal
        eps = (self.st.eps_prim_inf if which == 0 else self.st.eps_dual_inf) if self.st is not None else 1e-4
        d = np.array(delta, dtype=float)
        rec = dict(zip(E.INFEASIBILITY_RECORD, [0, 1, np.nan, np.nan, np.nan, np.nan, 0, 0]))
        norm = O.scaled_norm(Em if which == 0 else D, d, np.inf)
        rec["norm"] = norm
        if which == 1:
            rec["gate2"] = float(self.q @ d)
        if not norm > eps:
            return rec
        rec["gate"] = 2
        if which == 0:
            rec["gate2"] = float(np.max(np.abs((self.A.T @ d) / D)))
            if not rec["gate2"] <= eps * norm:
                return rec
            v = d * (-1.0 / norm)
            rec["gate3"] = float(v @ self.b)
        else:
            if not rec["gate2"] / (norm * c) < -eps:
                return rec
            rec["gate"] = 3
            rec["gate3"] = float(np.max(np.abs((self.P @ d) / D)))
            if not rec["gate3"] / (norm * c) <= eps:
                return rec
            v = (self.A @ d) / Em / norm
        rec["gate"] = 4
        fams, box = 0, 0.0
        for rng, cone in zip(O.row_ranges(self.cones), self.cones):
            x = v[rng]
            if which == 0 and isinstance(cone, O.Box):
                box += O.support_function(x, cone, eps)
                continue
            ok = O.support_function(x, cone, eps) == 0.0 if which == 0 else O.in_pol_recc(x, cone, eps)
            if not ok:
                fams |= _FAMILY.get(type(cone), E.FAMILY_C3)
        rec["families"] = fams
        if which == 0:
            rec["box_sum"] = box
            rec["verdict"] = int((np.inf if fams else 0.0) + box - rec["gate3"] <= eps)
        else:
            rec["verdict"] = int(fams == 0)
        return rec

    def psd_lambda_max(self, v):
        """lambda_max of the upper reflection of every PSD cone (the matrix the oracle's _is_pos_def factorizes)"""
        lam = []
        for rng, cone in zip(O.row_ranges(self.cones), self.cones):
            if isinstance(cone, (O.PsdCone, O.PsdConeTriangle, O.ComplexPsdConeTriangle)):
                X = O._cone_matrix(np.array(v[rng], dtype=float), cone)
                U = np.triu(X)
                lam.append(float(np.linalg.eigvalsh(U + np.triu(U, 1).conj().T)[-1]))
        return np.array(lam)

    def w(self):
        return self._w

    def rho_vec(self):
        if self._rho is None and self.st is not None:     # before a solve: set_rho_vec! on the resident data
            ost = O.Settings(rho=self.st.rho, RHO_MIN=self.st.RHO_MIN, RHO_TOL=self.st.RHO_TOL,
                             RHO_EQ_OVER_RHO_INEQ=self.st.RHO_EQ_OVER_RHO_INEQ, COSMO_INFTY=self.st.COSMO_INFTY,
                             MIN_SCALING=self.st.MIN_SCALING)
            O.classify_constraints(self.cones, self.b, ost)
            rv = np.full(self.m, ost.rho)
            O.apply_constraint_rho_scaling(rv, self.cones, ost)
            return rv.astype(self.dtype)
        return self._rho

    def close(self):
        pass
