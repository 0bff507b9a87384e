"""CPU checks of the Jacobian hook of custom cones (COSMO_B200_CUSTOM_HAS_JACOBIAN, DESIGN.md §3g): the NumPy Jacobians
of tests/custom_cone_jacobians.py against central differences of their projections, the restatements of the solve
adjoint and the solve derivative with those cones against central differences of oracle solves and against each other,
and the NVRTC compilation of the hooked types (no device needed)."""
import uuid

import numpy as np
import pytest
import scipy.sparse as sp

from cosmo_b200 import engine as E
from cosmo_b200 import model as M
from oracle import cosmo_oracle as O
from tests import custom_cone_jacobians as CJ
from tests import custom_cones as CC
from tests import solve_adjoint_reference as SA
from tests import solve_derivative_reference as SD


@pytest.fixture
def oracle(monkeypatch):
    CC.install_oracle(monkeypatch)
    return O


@pytest.fixture(autouse=True)
def restatement(monkeypatch):
    """the restatements' dpi with the Jacobians of the hooked cones"""
    CJ.install_restatement(monkeypatch)


# ---- 1. the NumPy Jacobians ------------------------------------------------------------
def _points(name, rng):
    """points of each branch of the cone's projection, away from its kinks"""
    if name == "nonpos_jac":
        return [rng.standard_normal(7) for _ in range(3)]
    x = rng.standard_normal(6)
    r = np.linalg.norm(x[1:]) if name == "soc2_jac" else 2.0 * np.abs(x[1:]).max()
    # inside, in the polar, and the general branch (for wlinf two entries of x large: a clip of more than one entry)
    gen = x.copy()
    gen[0] = 0.3 * r
    if name == "wlinf_jac":
        gen[1], gen[2] = 3.0, -2.5
    return [np.concatenate([[2.0 * r], x[1:]]), np.concatenate([[-3.0 * r], x[1:]]), gen]


@pytest.mark.parametrize("name", sorted(CJ.NUMPY))
def test_numpy_jacobians_are_central_differences_of_the_projection_and_symmetric(name):
    proj, _, _, jac = CJ.NUMPY[name]
    p = np.array([2.0]) if name == "wlinf_jac" else np.zeros(0)
    rng = np.random.default_rng(0)

    def pi(v):
        v = v.copy()
        proj(v, p)
        return v

    for w in _points(name, rng):
        s = pi(w)
        for _ in range(3):
            h, g = rng.standard_normal(w.size), rng.standard_normal(w.size)
            eps = 1e-7
            fd = (pi(w + eps * h) - pi(w - eps * h)) / (2 * eps)
            J = jac(w, s, h, p)
            np.testing.assert_allclose(J, fd, atol=1e-6 * (1 + np.abs(fd).max()))
            assert abs(g @ J - h @ jac(w, s, g, p)) <= 1e-12 * (1 + abs(g @ J))


def test_the_general_branch_of_wlinf_clips_more_than_one_entry():
    """the general point of _points clips the two large entries, so the rank-one block has k = 2"""
    w = _points("wlinf_jac", np.random.default_rng(0))[2]
    s = w.copy()
    CC._linf_project(s, [2.0])
    r = s[0] / 2.0
    assert r > 0 and (np.abs(w[1:]) > r).sum() >= 2


# ---- 2. the restatements with hooked custom cones ----------------------------------------
def _problem(seed):
    """ZeroSet, Box (one bound active at the start point) and one cone of each hooked type on 6 variables, through a
    strictly feasible point; P positive definite"""
    rng = np.random.default_rng(seed)
    n = 6
    G = rng.standard_normal((n, n))
    P = sp.csc_matrix(G @ G.T / n + 0.5 * np.eye(n))
    q = 3.0 * rng.standard_normal(n)
    sets = [M.ZeroSet(1), M.Box(np.array([-0.3, -1.0]), np.array([0.2, 1.0])), M.CustomCone(CJ.nonpos_type(), 3),
            M.CustomCone(CJ.soc2_type(), 4), M.CustomCone(CJ.linf_type(), 5, [2.0])]
    s0 = np.concatenate([[0.0], [0.0, 0.1], -0.5 * np.ones(3), [1.0, 0.2, 0.3, -0.1], [2.0, 0.2, -0.3, 0.1, 0.4]])
    A = sp.csc_matrix(rng.standard_normal((s0.size, n)))
    b = A @ (0.3 * rng.standard_normal(n)) + s0
    return P, q, A, b, sets


def _solve(P, q, A, b, cones, warm=None):
    st = O.Settings(eps_abs=1e-12, eps_rel=1e-12, max_iter=200000, kkt_solver="direct", scaling=0)
    r = O.solve(P, q, A, b, cones, st, *(warm or ()))
    assert r.status == "Solved", r.status
    return r


@pytest.mark.parametrize("seed", [0, 1])
def test_restatements_against_central_differences_of_oracle_solves(oracle, seed):
    P, q, A, b, sets = _problem(seed)
    cones = CJ.to_oracle(sets)
    m, n = A.shape
    r0 = _solve(P, q, A, b, cones)
    rng = np.random.default_rng(10 + seed)
    g = (rng.standard_normal(n), rng.standard_normal(m), rng.standard_normal(m))
    adj = SA.unscaled(P, A, cones, r0.x, r0.s, r0.y, gx=g[0], gy=g[1], gs=g[2])
    assert adj["residual"] <= 1e-10
    warm = (r0.x, r0.s, r0.y)
    eps = 1e-6

    def fd(make):
        rp, rm = _solve(*make(eps), cones, warm=warm), _solve(*make(-eps), cones, warm=warm)
        return [(a - c) / (2 * eps) for a, c in zip((rp.x, rp.y, rp.s), (rm.x, rm.y, rm.s))]

    S = rng.standard_normal((n, n))
    S = S + S.T
    d = dict(dq=rng.standard_normal(n), db=rng.standard_normal(m), dAx=rng.standard_normal(A.nnz),
             dPx=S[P.indices, np.repeat(np.arange(n), np.diff(P.indptr))])
    makes = dict(dq=lambda e: (P, q + e * d["dq"], A, b), db=lambda e: (P, q, A, b + e * d["db"]),
                 dAx=lambda e: (P, q, sp.csc_matrix((A.data + e * d["dAx"], A.indices, A.indptr), shape=A.shape), b),
                 dPx=lambda e: (P + e * sp.csc_matrix(S), q, A, b))
    grad = dict(dq=adj["dq"], db=adj["db"], dAx=adj["dAx"], dPx=adj["dPx"])
    for k, make in makes.items():
        want = fd(make)
        jvp = SD.unscaled(P, A, cones, r0.x, r0.s, r0.y, **{k: d[k]})
        assert jvp["residual"] <= 1e-10
        for got, w in zip((jvp["dx"], jvp["dy"], jvp["ds"]), want):
            assert np.abs(got - w).max() <= 1e-5 * (1 + np.abs(w).max()), k
        lw = sum(gk @ w for gk, w in zip(g, want))
        assert abs(grad[k] @ d[k] - lw) <= 1e-5 * (1 + abs(lw)), k


def test_the_general_branches_are_exercised(oracle):
    """at the solution of _problem(0) the SOC and the l-infinity cone are on their curved / clipped branches and the
    Nonpositives cone has zero and negative rows, so the restatement above goes through every hook's interesting part"""
    P, q, A, b, sets = _problem(0)
    cones = CJ.to_oracle(sets)
    r = _solve(P, q, A, b, cones)
    ws = r.s - r.y / 0.1
    nonpos, soc, linf = ws[3:6], ws[6:10], ws[10:15]
    assert (nonpos < 0).any() or (nonpos > 0).any()
    for w, name in ((soc, "soc2_jac"), (linf, "wlinf_jac")):
        s = w.copy()
        CJ.NUMPY[name][0](s, [2.0])
        assert not np.allclose(s, w) and np.abs(s).max() > 1e-8, name


def test_pairing_of_the_restatements(oracle):
    """<g, J d> = <J' g, d> with the hooked cones at an oracle solution, unscaled and at a Ruiz-like scaling (one factor
    per cone, which leaves the custom cones as they are)"""
    P, q, A, b, sets = _problem(0)
    cones = CJ.to_oracle(sets)
    m, n = A.shape
    r = _solve(P, q, A, b, cones)
    rng = np.random.default_rng(4)
    g = dict(gx=rng.standard_normal(n), gy=rng.standard_normal(m), gs=rng.standard_normal(m))
    S = rng.standard_normal((n, n))
    d = dict(dPx=(S + S.T)[P.indices, np.repeat(np.arange(n), np.diff(P.indptr))], dq=rng.standard_normal(n),
             dAx=rng.standard_normal(A.nnz), db=rng.standard_normal(m), dl=rng.standard_normal(m),
             du=rng.standard_normal(m))
    D = np.exp(rng.uniform(-0.5, 0.5, n))
    Ev = np.concatenate([np.exp(rng.uniform(-0.5, 0.5, 3))] + [np.full(S_.dim, np.exp(rng.uniform(-0.5, 0.5)))
                                                               for S_ in sets[2:]])
    c = 0.7
    box = cones[1]
    scaled = (sp.csc_matrix(c * sp.diags(D) @ P @ sp.diags(D)), sp.csc_matrix(sp.diags(Ev) @ A @ sp.diags(D)),
              [cones[0], O.Box(Ev[1:3] * box.l, Ev[1:3] * box.u)] + cones[2:], r.x / D, Ev * r.s, -c * r.y / Ev,
              dict(D=D, E=Ev, c=c))
    for P_, A_, cs, x, s_, mu, kw in ((P, A, cones, r.x, r.s, -r.y, {}), scaled):
        jt = SA.adjoint(P_, A_, cs, x, s_, mu, 0.1, **g, **kw)
        jd = SD.derivative(P_, A_, cs, x, s_, mu, 0.1, **d, **kw)
        lhs = g["gx"] @ jd["dx"] + g["gy"] @ jd["dy"] + g["gs"] @ jd["ds"]
        rhs = sum(jt[k] @ d[k] for k in ("dq", "db", "dPx", "dAx", "dl", "du"))
        assert abs(lhs - rhs) <= 1e-9 * (1 + abs(lhs)), (lhs, rhs)
        # the scaling changes nothing but the coordinates
        want = SA.unscaled(P, A, cones, r.x, r.s, r.y, **g)
        for k in ("dq", "db", "dPx", "dAx"):
            np.testing.assert_allclose(jt[k], want[k], atol=1e-8 * (1 + np.abs(want[k]).max()))


# ---- 3. compilation -------------------------------------------------------------------
def _fresh(kind):
    return M.CustomConeType(kind.name, kind.source + "\n// %s\n" % uuid.uuid4().hex, kind.granularity, kind.n_params,
                            kind.in_dual, kind.in_pol_recc, kind.jacobian)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("make", CJ.TYPES, ids=lambda f: f.__name__)
def test_every_hooked_type_compiles(make, dtype):
    kind = _fresh(make())
    assert kind.struct().flags & E.CUSTOM_HAS_JACOBIAN
    assert kind.compile(dtype) is True
    assert kind.compile(dtype) is False
    # the same source without the flag is another type
    plain = M.CustomConeType(kind.name, kind.source, kind.granularity, kind.n_params, kind.in_dual, kind.in_pol_recc)
    assert plain.compile(dtype) is True


def test_a_flagged_source_without_the_hook_is_refused():
    src = CC.SOC2_SRC.replace("namespace soc2 {", "namespace soc2_nojac {") + "// %s\n" % uuid.uuid4().hex
    kind = M.CustomConeType("soc2_nojac", src, "warp", jacobian=True)
    with pytest.raises(E.EngineError) as ei:
        kind.compile()
    assert ei.value.code == E.ERR_INVALID
    assert "soc2_nojac" in str(ei.value) and "jacobian" in str(ei.value)
    # without the flag the same source compiles
    assert M.CustomConeType("soc2_nojac", src, "warp").compile() is True


def test_flag_values():
    assert E.CUSTOM_HAS_JACOBIAN == 8
    st = CJ.soc2_type().struct()
    assert st.flags == E.CUSTOM_HAS_IN_DUAL | E.CUSTOM_HAS_IN_POL_RECC | E.CUSTOM_HAS_JACOBIAN
    assert CJ.linf_type(jacobian=False).struct().flags == 0
    with open(__file__.replace("tests/test_custom_cone_jacobian_cpu.py", "include/cosmo_b200.h")) as f:
        assert "#define COSMO_B200_CUSTOM_HAS_JACOBIAN 8" in f.read()
