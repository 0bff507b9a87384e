"""CPU checks of the forward derivative of a polished solution (tests/polish_derivative_reference.py, DESIGN.md §3j):
against central differences of the polished solution map (oracle ADMM solves + the polish restatement), the pairing
<g, J d> = <J' g, d> with the adjoint's restatement (unscaled and scaled), independence of the scaling, ds = dsbar on
the active rows, the half split of a Box row with l = u, and the C binding."""
import numpy as np
import pytest
import scipy.sparse as sp

from cosmo_b200 import engine as E
from tests import adjoint_reference as AR
from tests import polish_derivative_reference as PD
from tests import polish_reference as R
from tests.test_adjoint_cpu import PROBLEMS, _cones_with_bounds, _polished, _random_qp

OUT = ("dx", "dy", "ds")


def _direction(P, A, cls, l, u, rng):
    """A random direction: P symmetric on its pattern, A on its pattern, the Box bounds where they are finite (an
    equality row's two bounds moving together, so that it stays one)."""
    m, n = A.shape
    pr, pc = P.indices, np.repeat(np.arange(n), np.diff(P.indptr))
    M = sp.csc_matrix((rng.standard_normal(P.nnz), P.indices, P.indptr), shape=P.shape)
    box = cls == R.BOX
    dl = np.where(box & np.isfinite(l), rng.standard_normal(m), 0.0)
    du = np.where(box & np.isfinite(u), rng.standard_normal(m), 0.0)
    du = np.where(box & (l == u), dl, du)
    return dict(dPx=np.asarray((M + M.T)[pr, pc]).ravel() if P.nnz else np.zeros(0), dq=rng.standard_normal(n),
                dAx=rng.standard_normal(A.nnz), db=rng.standard_normal(m), dl=dl, du=du)


def _only(d, key):
    return {k: (v if k == key else np.zeros_like(v)) for k, v in d.items()}


@pytest.mark.parametrize("name,make", PROBLEMS, ids=[p[0] for p in PROBLEMS])
def test_derivative_matches_central_differences_of_the_polished_solution_map(name, make):
    P, q, A, b, cones = make()
    m, n = A.shape
    cls, l, u = R.row_classes(cones)
    base = _polished(P, q, A, b, cones)
    kind = base["kind"]
    ineq = (kind == R.LOWER) | (kind == R.UPPER)
    assert np.all(np.abs(base["mu_p"][ineq]) > 1e-7)
    rng = np.random.default_rng(100 + len(name) + n + m)
    full = _direction(P, A, cls, l, u, rng)
    act = kind != R.INACTIVE
    for what in ("dPx", "dq", "dAx", "db", "bounds"):
        d = _only(full, what) if what != "bounds" else {k: (v if k in ("dl", "du") else np.zeros_like(v))
                                                       for k, v in full.items()}
        if not any(np.any(v) for v in d.values()):
            continue
        got = PD.derivative(P, A, cls, kind, base["x_p"], -base["mu_p"], **d)
        assert got["refine_residual"] <= 1e-12
        eps = 1e-6
        outs = []
        for sgn in (1.0, -1.0):
            P2 = sp.csc_matrix((P.data + sgn * eps * d["dPx"], P.indices, P.indptr), shape=P.shape)
            A2 = sp.csc_matrix((A.data + sgn * eps * d["dAx"], A.indices, A.indptr), shape=A.shape)
            c2 = _cones_with_bounds(cones, l + sgn * eps * d["dl"], u + sgn * eps * d["du"])
            out = _polished(P2, q + sgn * eps * d["dq"], A2, b + sgn * eps * d["db"], c2)
            assert np.array_equal(out["kind"], kind), what
            outs.append(out)
        fd = {k: (outs[0][k[1:]] - outs[1][k[1:]]) / (2 * eps) for k in OUT}
        scale = max(1.0, max(np.abs(got[k]).max(initial=0.0) for k in OUT))
        for k in OUT:
            # off the active rows y is 0 on both sides; the ADMM solve's tolerance bounds how well the FD resolves
            assert np.abs(fd[k] - got[k]).max(initial=0.0) <= 1e-5 * scale, (what, k)
        assert np.all(got["dy"][~act] == 0.0)


def _pairing(P, A, cls, kind, x, y, d, g, **scaling):
    fwd = PD.derivative(P, A, cls, kind, x, y, **d, **scaling)
    adj = AR.adjoint(P, A, cls, kind, x, y, g["dx"], g["dy"], g["ds"], **scaling)
    lhs = sum(g[k] @ fwd[k] for k in OUT)
    rhs = (adj["dPx"] @ d["dPx"] + adj["dq"] @ d["dq"] + adj["dAx"] @ d["dAx"] + adj["db"] @ d["db"]
           + adj["dl"] @ d["dl"] + adj["du"] @ d["du"])
    return lhs, rhs


@pytest.mark.parametrize("name,make", PROBLEMS, ids=[p[0] for p in PROBLEMS])
def test_pairing_with_the_adjoint_unscaled_and_scaled(name, make):
    P, q, A, b, cones = make()
    m, n = A.shape
    cls, l, u = R.row_classes(cones)
    base = _polished(P, q, A, b, cones)
    kind, x, y = base["kind"], base["x_p"], -base["mu_p"]
    rng = np.random.default_rng(200 + n + m)
    d = _direction(P, A, cls, l, u, rng)
    g = {k: rng.standard_normal(n if k == "dx" else m) for k in OUT}
    lhs, rhs = _pairing(P, A, cls, kind, x, y, d, g)
    assert abs(lhs - rhs) <= 1e-12 * (abs(lhs) + abs(rhs))
    # the same map on the scaled data of a scaling (D, E, c)
    D, Ev, c = rng.uniform(0.5, 2.0, n), rng.uniform(0.5, 2.0, m), 0.7
    Ps = sp.csc_matrix(c * sp.diags(D) @ P @ sp.diags(D))
    As = sp.csc_matrix(sp.diags(Ev) @ A @ sp.diags(D))
    lhs_s, rhs_s = _pairing(Ps, As, cls, kind, x / D, c * y / Ev, d, g, D=D, E=Ev, c=c)
    assert abs(lhs_s - rhs_s) <= 1e-12 * (abs(lhs_s) + abs(rhs_s))
    assert abs(lhs_s - lhs) <= 1e-10 * (abs(lhs) + abs(lhs_s))


def test_scaling_does_not_change_the_derivative():
    P, q, A, b, cones = _random_qp(0)
    m, n = A.shape
    cls, l, u = R.row_classes(cones)
    base = _polished(P, q, A, b, cones)
    rng = np.random.default_rng(7)
    d = _direction(P, A, cls, l, u, rng)
    ref = PD.derivative(P, A, cls, base["kind"], base["x_p"], -base["mu_p"], **d)
    D, Ev, c = rng.uniform(0.5, 2.0, n), rng.uniform(0.5, 2.0, m), 0.7
    Ps = sp.csc_matrix(c * sp.diags(D) @ P @ sp.diags(D))
    As = sp.csc_matrix(sp.diags(Ev) @ A @ sp.diags(D))
    got = PD.derivative(Ps, As, cls, base["kind"], base["x_p"] / D, -c * base["mu_p"] / Ev, **d, D=D, E=Ev, c=c)
    for k in OUT:
        assert np.allclose(got[k], ref[k], rtol=1e-10, atol=1e-12), k


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_ds_equals_the_bound_direction_on_the_active_rows(seed):
    P, q, A, b, cones = _random_qp(seed)
    cls, l, u = R.row_classes(cones)
    base = _polished(P, q, A, b, cones)
    kind = base["kind"]
    d = _direction(P, A, cls, l, u, np.random.default_rng(30 + seed))
    got = PD.derivative(P, A, cls, kind, base["x_p"], -base["mu_p"], **d)
    act = kind != R.INACTIVE
    want = PD.bound_direction(cls, kind, d["dl"], d["du"])
    assert np.abs(got["ds"][act] - want[act]).max() <= 1e-12 * max(1.0, np.abs(got["ds"]).max())


def test_half_split_of_a_box_row_with_l_equal_u():
    # the first Box row of _random_qp has l = u: the row is an equality at l, and its bound moves as (dl + du) / 2
    P, q, A, b, cones = _random_qp(0)
    m, n = A.shape
    cls, l, u = R.row_classes(cones)
    r = int(np.flatnonzero((cls == R.BOX) & (l == u))[0])
    base = _polished(P, q, A, b, cones)
    kind, x, y = base["kind"], base["x_p"], -base["mu_p"]
    assert kind[r] == R.EQUALITY
    dl, du = np.zeros(m), np.zeros(m)
    dl[r] = 1.0
    only_l = PD.derivative(P, A, cls, kind, x, y, dl=dl)
    both = PD.derivative(P, A, cls, kind, x, y, dl=dl, du=dl)
    assert np.isclose(only_l["ds"][r], 0.5, rtol=1e-12) and np.isclose(both["ds"][r], 1.0, rtol=1e-12)
    for k in OUT:
        assert np.allclose(2.0 * only_l[k], both[k], rtol=1e-12, atol=1e-14), k
    # the adjoint's dl, du of the row are each half of -v: the transpose of this split
    g = {"dx": np.zeros(n), "dy": np.zeros(m), "ds": np.zeros(m)}
    g["ds"][r] = 1.0
    adj = AR.adjoint(P, A, cls, kind, x, y, g["dx"], g["dy"], g["ds"])
    assert adj["dl"][r] == adj["du"][r]
    assert np.isclose(adj["dl"][r], only_l["ds"][r], rtol=1e-12)


def test_the_binding_names_the_entry_point():
    assert "cosmo_b200_derivative" in E.SIGNATURES and "cosmo_b200_derivative" in E.EXPORTS
    restype, argtypes = E.SIGNATURES["cosmo_b200_derivative"]
    assert len(argtypes) == 12 and argtypes[1] is E.C.c_int32
    assert argtypes[-1] == E.C.POINTER(E.C.c_double)
