"""torch.autograd for solves on the device: polished QPs and LPs (DESIGN.md §3j) and conic problems (§3k, §3l).

``solve_qp(engine, Px, q, Ax, b)`` puts new values of P, q, A and b into a live engine (``Engine.update_matrices``),
solves, polishes and returns the polished unscaled solution ``(x, y, s)`` as CUDA tensors; its backward pass is one
``Engine.adjoint`` and its forward-mode product (``torch.autograd.forward_ad``, ``gradcheck(check_forward_ad=True)``)
one ``Engine.derivative``, both into CUDA tensors.  Nothing leaves the device.

The engine is created by the caller with a direct KKT solver (DeviceLdlKKTSolver or DeviceSupernodalKKTSolver), on the
pattern of P and A, without host scaling (scaling 0, or ``equilibrate=True``), so that ``update_matrices`` takes the
unscaled data.  ``Px`` and ``Ax`` are the ``data`` arrays of P and A in sorted CSC order, all four inputs CUDA tensors of
the engine's dtype.  The Box bounds are not inputs of ``update_matrices`` and get no gradient here (``Engine.adjoint``
returns them).  The derivative is that of the polished solution map on its active set: exact where the active set is
stable, one-sided at weakly active rows.

The backward pass and the forward-mode product read the point and the factor the engine keeps from the last polish.
When the engine has run another ``solve_qp`` since this pass's forward (as ``torch.autograd.gradcheck`` does between
them), they first solve and polish this pass's data again; the solve is deterministic, so they differentiate the same
point.  Between a forward pass and its backward pass (or its forward-mode product) the engine must not be used other
than through ``solve_qp``.

``solve_conic(engine, Px, q, Ax, b)`` does the same for any solve the fixed-point derivatives cover, without a polish:
its backward pass is one ``Engine.solve_adjoint`` and its forward-mode product (``torch.autograd.forward_ad``,
``gradcheck(check_forward_ad=True)``) one ``Engine.solve_derivative``, both into CUDA tensors.  The ``torch.func``
transforms (``jvp``, ``jacfwd``, ``vmap``) are not supported: they need the ``setup_context`` form of the Function.
"""
import dataclasses
from typing import Callable

import torch

from .engine import EngineError


def _solve_and_polish(engine, Px, q, Ax, b):
    """update_matrices, solve and polish into new CUDA tensors; returns (x, y, s) and tags the engine with this call."""
    dev = q.device
    engine.set_caller_stream(torch.cuda.current_stream(dev).cuda_stream)
    engine.update_matrices(Px.detach().contiguous(), Ax.detach().contiguous(), q.detach().contiguous(),
                           b.detach().contiguous())
    engine.solve(copy_out=False)
    f64 = dict(dtype=torch.float64, device=dev)
    x, y, s = torch.empty(engine.n, **f64), torch.empty(engine.m, **f64), torch.empty(engine.m, **f64)
    _, _, _, st = engine.polish(x=x, y=y, s=s)
    if st["status"] != 1:
        raise EngineError(st["status"], "solve_qp: the solution could not be polished (status %d), so it has no "
                                        "derivative here" % st["status"])
    engine._solve_qp_call = getattr(engine, "_solve_qp_call", 0) + 1
    return x, y, s


def _solve(engine, Px, q, Ax, b):
    """update_matrices and solve, then the unscaled solution into new CUDA tensors; returns (x, y, s) and tags the engine
    with this call."""
    dev = q.device
    engine.set_caller_stream(torch.cuda.current_stream(dev).cuda_stream)
    engine.update_matrices(Px.detach().contiguous(), Ax.detach().contiguous(), q.detach().contiguous(),
                           b.detach().contiguous())
    out = engine.solve(copy_out=False)
    if out.status != "Solved":
        raise EngineError(0, "solve_conic: the solve ended %s, not Solved, so its solution has no derivative here"
                          % out.status)
    f64 = dict(dtype=torch.float64, device=dev)
    x, y, s = torch.empty(engine.n, **f64), torch.empty(engine.m, **f64), torch.empty(engine.m, **f64)
    engine.solution(x=x, y=y, s=s)
    engine._solve_conic_call = getattr(engine, "_solve_conic_call", 0) + 1
    return x, y, s


@dataclasses.dataclass(frozen=True)
class _Mode:
    """What solve_qp and solve_conic differ in: the forward solve, the engine attribute that counts its calls, the
    forward derivative (engine, options, direction, dx, dy, ds) and the adjoint (engine, options, gradients, dq, db, dPx,
    dAx), each returning the engine call's (outputs, stats), and the errors of those two when their status is not 1."""
    solve: Callable
    counter: str
    derivative: Callable
    adjoint: Callable
    derivative_error: str
    adjoint_error: str


def _at_forward_point(ctx):
    """ctx's engine, solved at the data of ctx's forward pass again when it has solved other data since, with the
    current stream as its caller stream; and the options of the fp64 output tensors."""
    eng, mode = ctx.engine, ctx.mode
    if getattr(eng, mode.counter) != ctx.call:   # the engine has solved other data since: this pass's point again
        mode.solve(eng, *ctx.saved_tensors)
        ctx.call = getattr(eng, mode.counter)
    eng.set_caller_stream(torch.cuda.current_stream(ctx.device).cuda_stream)
    return eng, dict(dtype=torch.float64, device=ctx.device)


class _Solve(torch.autograd.Function):
    @staticmethod
    def forward(ctx, mode, engine, options, Px, q, Ax, b):
        x, y, s = mode.solve(engine, Px, q, Ax, b)
        ctx.mode, ctx.engine, ctx.options, ctx.device = mode, engine, options, q.device
        ctx.call = getattr(engine, mode.counter)
        ctx.dtypes = (Px.dtype, q.dtype, Ax.dtype, b.dtype)
        ctx.save_for_backward(Px, q, Ax, b)
        ctx.save_for_forward(Px, q, Ax, b)
        return x, y, s

    @staticmethod
    def jvp(ctx, _mode, _engine, _options, tPx, tq, tAx, tb):
        eng, f64 = _at_forward_point(ctx)
        dx, dy, ds = torch.empty(eng.n, **f64), torch.empty(eng.m, **f64), torch.empty(eng.m, **f64)
        d = [None if t is None else t.detach().to(torch.float64).contiguous() for t in (tPx, tq, tAx, tb)]
        _, st = ctx.mode.derivative(eng, ctx.options, d, dx, dy, ds)
        if st["status"] != 1:
            raise EngineError(st["status"], ctx.mode.derivative_error % st["status"])
        return dx, dy, ds

    @staticmethod
    def backward(ctx, gx, gy, gs):
        eng, f64 = _at_forward_point(ctx)
        dq, db = torch.empty(eng.n, **f64), torch.empty(eng.m, **f64)
        dPx, dAx = torch.empty(eng.nnzP, **f64), torch.empty(eng.nnzA, **f64)
        g = [None if t is None else t.detach().to(torch.float64).contiguous() for t in (gx, gy, gs)]
        _, st = ctx.mode.adjoint(eng, ctx.options, g, dq, db, dPx, dAx)
        if st["status"] != 1:
            raise EngineError(st["status"], ctx.mode.adjoint_error % st["status"])
        tP, tq, tA, tb = ctx.dtypes
        return None, None, None, dPx.to(tP), dq.to(tq), dAx.to(tA), db.to(tb)


# dl and du: CUDA tensors for the polished adjoint, the NumPy arrays Engine.solve_adjoint allocates for the conic one
_QP = _Mode(
    _solve_and_polish, "_solve_qp_call",
    lambda eng, refine_iter, d, dx, dy, ds: eng.derivative(*d, refine_iter=refine_iter, dx=dx, dy=dy, ds=ds),
    lambda eng, refine_iter, g, dq, db, dPx, dAx: eng.adjoint(
        *g, refine_iter=refine_iter, dq=dq, db=db, dPx=dPx, dAx=dAx, dl=torch.empty_like(db), du=torch.empty_like(db)),
    "solve_qp: the derivative did not apply (status %d)", "solve_qp: the adjoint did not apply (status %d)")
_CONIC = _Mode(
    _solve, "_solve_conic_call",
    lambda eng, settings, d, dx, dy, ds: eng.solve_derivative(*d, dx=dx, dy=dy, ds=ds, **settings),
    lambda eng, settings, g, dq, db, dPx, dAx: eng.solve_adjoint(*g, dq=dq, db=db, dPx=dPx, dAx=dAx, **settings),
    "solve_conic: the solve derivative did not apply or converge (status %d)",
    "solve_conic: the solve adjoint did not apply or converge (status %d)")


def solve_qp(engine, Px, q, Ax, b, refine_iter=3):
    """The polished solution (x, y, s) of the engine's problem with the data (Px, q, Ax, b), differentiable with respect
    to all four (see the module docstring)."""
    return _Solve.apply(_QP, engine, refine_iter, Px, q, Ax, b)


def solve_conic(engine, Px, q, Ax, b, **adjoint_settings):
    """The solution (x, y, s) of the engine's problem with the data (Px, q, Ax, b), differentiable with respect to all four
    through Engine.solve_adjoint (DESIGN.md §3k): any cone but Exp/Pow, complex PSD and custom cones whose type has no
    Jacobian hook, any single-GPU KKT solver.  The engine is created as for solve_qp (on the pattern of P and A, without host scaling); the forward
    pass raises unless the solve ends Solved.  adjoint_settings (tol, max_iter, restart, kkt_tol) go to
    Engine.solve_adjoint and Engine.solve_derivative.  The derivative is that of the solution map at the solve's point,
    exact as the solve's tolerance goes to 0.  The engine rules of solve_qp apply: between a forward pass and its
    backward pass (or its forward-mode product) it is used only through solve_conic, and a derivative after other
    solves re-solves its own data first."""
    return _Solve.apply(_CONIC, engine, dict(adjoint_settings), Px, q, Ax, b)
