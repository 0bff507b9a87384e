"""The extended-precision restatement of scale_ruiz! (tests/ruiz_reference.py) against the fp64 oracle (O.scale_ruiz,
itself pinned on the reference's known answers): the two must agree to the level of fp64 rounding on every problem the
device tests use, and the restatement's scaled P must be exactly symmetric (scaling.jl:99)."""
import numpy as np
import pytest
import scipy.sparse as sp

import cosmo_b200
from oracle import cosmo_oracle as O
from tests import ruiz_reference as R
from tests.gpu_helpers import U64


def _problems():
    pr = cosmo_b200.problems
    return {"qp_box": lambda: pr.random_sparse_qp(300, 500, 0.05, seed=0),
            "socp": lambda: pr.portfolio_socp(n=200, k=20, seed=2),
            "sdp": lambda: pr.closest_correlation_sdp(N=20, seed=7),
            "dynamic_range": R.problem_dynamic_range,
            "every_rectified_family": R.problem_every_rectified_family,
            "symmetry": R.problem_symmetry}


@pytest.mark.parametrize("scaling", [1, 3, 10])
@pytest.mark.parametrize("name", list(_problems()))
def test_restatement_matches_the_oracle(name, scaling):
    P, q, A, b, sets = _problems()[name]()
    cones = R.sets_to_oracle(sets)
    ref = R.scale_ruiz_ld(P, q, A, b, cones, scaling=scaling)
    Ps, qs, As, bs, ocones, sm = O.scale_ruiz(P, q, A, b, R.sets_to_oracle(sets), O.Settings(scaling=scaling))
    # the oracle rounds every product of every pass in fp64: D, E, c carry a few ulps per pass, the entries a few more
    bar = 4 * scaling * U64
    errs = {"D": R.rel_err(sm.D, ref.D), "E": R.rel_err(sm.E, ref.E), "c": R.rel_err([sm.c], [ref.c])}
    m, n = ref.shape
    Pd, Ad = R.dense(ref.P, (n, n)), R.dense(ref.A, (m, n))
    errs.update(P=R.rel_err(Ps.toarray(), Pd), A=R.rel_err(As.toarray(), Ad), q=R.rel_err(qs, ref.q), b=R.rel_err(bs, ref.b))
    box = ~np.isnan(ref.l)
    if box.any():
        ol = np.concatenate([np.full(S.dim, np.nan) if not isinstance(S, O.Box) else S.l for S in ocones])
        ou = np.concatenate([np.full(S.dim, np.nan) if not isinstance(S, O.Box) else S.u for S in ocones])
        fin = box & np.isfinite(ref.l)
        errs["l"] = R.rel_err(ol[fin], ref.l[fin])
        fin = box & np.isfinite(ref.u)
        errs["u"] = R.rel_err(ou[fin], ref.u[fin])
    print("%s scaling=%d: worst rel. error of the oracle vs the restatement %s (bar %.1e / %.1e)"
          % (name, scaling, {k: "%.1e" % v for k, v in errs.items()}, bar, 3 * bar + 4 * U64))
    for k in ("D", "E", "c"):
        assert errs[k] <= bar, (k, errs[k], bar)
    for k in set(errs) - {"D", "E", "c"}:
        assert errs[k] <= 3 * bar + 4 * U64, (k, errs[k])
    # symmetrize_full! leaves P exactly symmetric, whatever the rounding of the passes
    assert np.array_equal(Pd, Pd.T)


def test_restatement_branches_and_rectified_means():
    """the branch counts the device tests rely on, and one scalar of E per rectified cone"""
    P, q, A, b, sets = R.problem_dynamic_range()
    ref = R.scale_ruiz_ld(P, q, A, b, R.sets_to_oracle(sets), scaling=10)
    assert R.branch_count(ref, "D_low", range(1, 10)) > 0 and R.branch_count(ref, "D_high", range(1, 10)) > 0
    assert R.branch_count(ref, "E_low", range(1, 10)) > 0 and R.branch_count(ref, "E_high", range(1, 10)) > 0
    assert R.branch_count(ref, "cost") == 10
    P, q, A, b, sets = R.problem_every_rectified_family()
    cones = R.sets_to_oracle(sets)
    ref = R.scale_ruiz_ld(P, q, A, b, cones)
    assert ref.rectified == sum(isinstance(S, O.SCALAR_SCALED_CONES) for S in cones) == 9
    for rng, cone in zip(O.row_ranges(cones), cones):
        e = ref.E[rng]
        if isinstance(cone, O.SCALAR_SCALED_CONES):
            assert np.max(np.abs(e - e[0])) <= 4 * np.finfo(R.LD).eps * e[0]
        elif cone.dim > 1:
            assert np.ptp(e) > 0
    # an LP and a problem without q skip the cost scaling in every pass: c = 1
    for P0, q0 in ((sp.csc_matrix((A.shape[1], A.shape[1])), q), (P, np.zeros_like(q))):
        ref = R.scale_ruiz_ld(P0, q0, A, b, cones)
        assert R.branch_count(ref, "cost") == 0 and ref.c == 1
