"""The Anderson accelerator variants of anderson_accelerator.jl and the activation reasons on the device
(csrc/aa.cuh, cosmo_b200_set_accelerator), against the CPU restatement of tests/anderson_variants.py."""
import numpy as np
import pytest

import cosmo_b200
from oracle import cosmo_oracle as O
from oracle.bridge import to_oracle_cones
from tests import anderson_variants as V
from tests import golden_problems as G
from tests.test_gpu_parity import _small_qp, _to_mine

pytestmark = pytest.mark.gpu

_NEW = [t for t in V.TYPES if t[0] != "Type2{QRDecomp}"]
_TIGHT = dict(eps_abs=1e-14, eps_rel=1e-14)


def _mine(P, q, A, b, sets, **kw):
    model = cosmo_b200.Model()
    model.set(P, q, A, b, sets, cosmo_b200.Settings(accelerator="AndersonAccelerator", **kw))
    return model.optimize(), model


def _builder_mine(builder, **kw):
    P, q, cons = builder()
    model = cosmo_b200.Model()
    cosmo_b200.assemble(model, P, q, _to_mine(cons), cosmo_b200.Settings(accelerator="AndersonAccelerator", **kw))
    return model.optimize(), model


def _ref(P, q, A, b, sets, scaling=10, kkt_solver="cg", var=None, **kw):
    return V.solve(P, q, A, b, to_oracle_cones(sets), O.Settings(accelerator="anderson", scaling=scaling, kkt_solver=kkt_solver, **kw),
                   **(var or {}))


@pytest.mark.parametrize("t,mem,reg", V.TYPES)
@pytest.mark.parametrize("scaling", [0, 10])
def test_variant_iterates_match_oracle(t, mem, reg, scaling):
    # w after the first candidate (5), a full memory of 15 columns (20: a rolling wrap-around or a restart), declined
    # candidates (45) and, with rho = 1e-3 and interval 10, rho-adaptation restarts at iterations 18-33 (35) for every
    # variant but the rolling Type2 ones, whose accepted candidates postpone the adaptation past these runs.
    # Longer runs are not compared: a safeguard or |eta| decision that rounding tips the other way splits the
    # trajectories (the normal equations square the conditioning of F), as seen at 60 and 90 iterations.
    P, q, A, b, sets = _small_qp(seed=7)
    var = V.variant(t, mem, reg)
    runs = [(it, {}) for it in (5, 20, 45)] + [(35, dict(rho=1e-3, adaptive_rho_interval=10))]
    # measured worst: 2.5e-12 over the restarted and Type1 variants; the rolling Type2 window is never cleared and its
    # normal equations square an ill-conditioned F: up to 6.8e-9 at 35 iterations of the rho run with scaling 10
    bound = 1e-8 if (t, mem) == ("Type2{NormalEquations}", "RollingMemory") else 1e-9
    worst, seen = 0.0, {"declined": 0, "memory_restarts": 0}
    for iters, extra in runs:
        ref, ws = _ref(P, q, A, b, sets, scaling=scaling, var=var, max_iter=iters, **_TIGHT, **extra)
        res, model = _mine(P, q, A, b, sets, scaling=scaling, max_iter=iters, **_TIGHT, **extra, **var)
        w = model.engine.w()
        got, want = model.engine.accelerator_stats(), V.stats(ws)
        assert res.iter == ref.iter and res.safeguarding_iter == ref.safeguarding_iter, (iters, res.iter, ref.iter)
        assert got == want, (iters, got, want)
        err = np.linalg.norm(w - ref.w) / np.linalg.norm(ref.w)
        worst = max(worst, err)
        assert err < bound, (iters, err)
        for k in seen:
            seen[k] += got[k]
    assert seen["declined"] >= 1 and (seen["memory_restarts"] >= 1 or mem == "RollingMemory")
    print("worst relative |w - w_oracle|: %.2e" % worst)


@pytest.mark.parametrize("t,mem,reg", V.TYPES)
def test_every_variant_solves_the_reference_qp(t, mem, reg):
    # AccelerationTests/anderson_accelerator.jl:21-41
    res, _ = _builder_mine(G.g1_qp_nonneg, **V.variant(t, mem, reg))
    assert res.status == "Solved" and abs(res.obj_val - G.G1_OBJ) < 1e-3 and np.max(np.abs(res.x - G.G1_X)) < 1e-3


@pytest.mark.parametrize("t,mem,reg", [("Type1", "RollingMemory", "NoRegularizer"),
                                       ("Type2{NormalEquations}", "RestartedMemory", "TikonovRegularizer")])
def test_variant_known_answers_and_statuses(t, mem, reg):
    var = V.variant(t, mem, reg)
    for builder, x, obj, tol in ((G.g1_qp_nonneg, G.G1_X, G.G1_OBJ, 1e-3), (G.g1_qp_box, G.G1_X, G.G1_OBJ, 1e-3),
                                 (G.g12_lp, G.G12_X, G.G12_OBJ, 1e-2), (G.g13_lovasz_petersen, None, G.G13_OBJ, 1e-3)):
        res, _ = _builder_mine(builder, **var)
        assert res.status == "Solved" and abs(res.obj_val - obj) < tol, (builder.__name__, res.status, res.obj_val)
        if x is not None:
            assert np.max(np.abs(res.x - x)) < tol, builder.__name__
    assert _builder_mine(G.g2_box_feasible, **var)[0].status == "Solved"
    assert _builder_mine(G.g2_box_primal_infeasible_1, **var)[0].status == "Primal_infeasible"
    assert _builder_mine(G.g2_box_primal_infeasible_2, **var)[0].status == "Primal_infeasible"
    assert _builder_mine(G.g2_box_dual_infeasible, check_infeasibility=20, scaling=0, **var)[0].status == "Dual_infeasible"


@pytest.mark.parametrize("mem", ["RollingMemory", "RestartedMemory"])
def test_rho_adaptation_restarts_the_accelerator(mem):
    # AccelerationTests/adaptive_rho_acc_restarts.jl: one accelerator restart per rho adaption
    var = V.variant("Type2{NormalEquations}", mem, "NoRegularizer")
    res, model = _builder_mine(G.g1_qp_nonneg, adaptive_rho_interval=23, rho=1e-4, safeguard=False, accelerator_mem=5, **var)
    st = model.engine.accelerator_stats()
    assert st["rho_restarts"] == len(res.info.rho_updates) - 1
    if mem == "RestartedMemory":
        assert st["rho_restarts"] >= 1 and res.status == "Solved"


@pytest.mark.parametrize("t", ["Type2{QRDecomp}", "Type2{NormalEquations}"])
@pytest.mark.parametrize("activation", [("IterActivation", 30), ("IterActivation", 1), ("AccuracyActivation", 1e-2)])
def test_activation_matches_oracle(t, activation):
    # compared up to 15 iterations after the activation the oracle finds
    P, q, A, b, sets = _small_qp(seed=7)
    var = V.variant(t, "RestartedMemory", "NoRegularizer", activation=activation)
    act = V.stats(_ref(P, q, A, b, sets, var=var, max_iter=120, **_TIGHT)[1])["activated_at"]
    assert 0 < act <= 105
    ref, ws = _ref(P, q, A, b, sets, var=var, max_iter=act + 15, **_TIGHT)
    res, model = _mine(P, q, A, b, sets, max_iter=act + 15, **_TIGHT, **var)
    got, want = model.engine.accelerator_stats(), V.stats(ws)
    assert want["activated_at"] > 0 and got == want, (got, want)
    assert res.iter == ref.iter and res.safeguarding_iter == ref.safeguarding_iter
    assert np.linalg.norm(model.engine.w() - ref.w) / np.linalg.norm(ref.w) < 1e-9


@pytest.mark.parametrize("t,mem", [("Type1", "RollingMemory"), ("Type2{NormalEquations}", "RestartedMemory")])
def test_large_problem_full_memory(t, mem):
    # n + m = 1e6 at mem = 32: the Gram pass runs over many blocks and four chunks of 8 columns; 36 iterations fill the
    # window (l = 32), wrap it (rolling) or restart it (restarted).  Compared with the CPU restatement on the same data;
    # no safeguard and no rho adaptation, so that every candidate of both runs is formed from the same history.
    P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(300_000, 700_000, 4e-6, seed=5)
    var = V.variant(t, mem, "NoRegularizer")
    kw = dict(scaling=0, max_iter=36, accelerator_mem=32, safeguard=False, adaptive_rho=False, **_TIGHT)
    ref, ws = _ref(P, q, A, b, sets, var=var, **kw)
    res, model = _mine(P, q, A, b, sets, **kw, **var)
    got, want = model.engine.accelerator_stats(), V.stats(ws)
    assert got == want and want["accepted"] >= 25, (got, want)
    assert want["memory_restarts"] >= 1 or mem == "RollingMemory"
    w = model.engine.w()
    err = np.linalg.norm(w - ref.w) / np.linalg.norm(ref.w)
    print("n + m = 1e6, %s/%s: relative |w - w_oracle| = %.2e" % (t, mem, err))
    assert err < 1e-9, err


def test_dimension_below_memory():
    # dim = n + m = 10 < mem = 15: the history holds min(mem, dim) columns.  A full-dimensional window is nearly
    # singular, and rounding tips single safeguard decisions within 14 iterations (Type1, RollingMemory), so this
    # compares solves: status and answer of the oracle, and a memory that wrapped or restarted
    P, q, A, b, sets = _small_qp(seed=3, n=4, m=6)
    for t, mem, reg in _NEW:
        var = V.variant(t, mem, reg)
        ref, ws = _ref(P, q, A, b, sets, var=var, accelerator_mem=15)
        res, model = _mine(P, q, A, b, sets, accelerator_mem=15, **var)
        st = model.engine.accelerator_stats()
        assert res.status == ref.status == "Solved", (t, mem, reg, res.status, ref.status)
        assert np.max(np.abs(res.x - ref.x)) <= 1e-3 * max(1.0, np.abs(ref.x).max()), (t, mem, reg)
        assert st["accepted"] >= 1 and (st["memory_restarts"] >= 1 or mem == "RollingMemory"), (t, mem, reg, st)


# Measured on one H100 (float32, Type2{NormalEquations}, RestartedMemory, g2_box_primal_infeasible_1): accepted
# unregularised candidates extrapolate along the divergence ray to |w| = 1.59e7 (float64: 6.1e3, detected at iteration
# 162).  From there |w| * 2^-24 is about one, larger than the step of the ADMM iteration: w stops changing (|w| is the
# same after 1000 and 5000 iterations), every other candidate is rejected (420 -> 2420 rejections, accepted fixed at
# 66), so the postponed infeasibility checks do run -- and see no change.  The float32 iteration has stagnated.
_FP32_NE_INFEASIBLE = pytest.mark.xfail(strict=True, reason="known: Max_iter_reached in fp32 on qp-box.jl's first primal "
                                       "infeasible problem: w is extrapolated to |w| = 1.6e7 and the float32 iteration "
                                       "stagnates there")


@pytest.mark.parametrize("t,mem,builder,status", [
    (t, mem, builder, status) for t, mem in (("Type1", "RollingMemory"), ("Type2{NormalEquations}", "RestartedMemory"))
    for builder, status in ((G.g1_qp_nonneg, "Solved"), (G.g2_box_feasible, "Solved"))] + [
    ("Type1", "RollingMemory", G.g2_box_primal_infeasible_1, "Primal_infeasible"),
    pytest.param("Type2{NormalEquations}", "RestartedMemory", G.g2_box_primal_infeasible_1, "Primal_infeasible",
                 marks=_FP32_NE_INFEASIBLE)])
def test_float32_statuses(t, mem, builder, status):
    P, q, cons = builder()
    model = cosmo_b200.Model(dtype=np.float32)
    cosmo_b200.assemble(model, P, q, _to_mine(cons), cosmo_b200.Settings(accelerator="AndersonAccelerator", eps_abs=1e-4,
                                                                         eps_rel=1e-4, **V.variant(t, mem, "NoRegularizer")))
    res = model.optimize()
    assert res.status == status, (builder.__name__, res.status)
