"""Receding-horizon MPC: a closed-loop episode of solve, apply, shift and re-solve, the loop of the reference's
cartpole and pendulum notebooks, as one library call.

Where every solve of the episode would run on the device loop (``solver._use_device_loop`` /
``_use_slew_device_loop``), the whole episode is one CUDA graph (``step.episode_raw``): the solves, the model steps
and the warm-start shifts run on the device, with no host read between control steps.  Anything else (Module costs,
opaque Module dynamics, ``verbose > 0``, a driver without conditional graph nodes) runs the same loop from Python over
``MPC.forward``; that host path steps the model with the kernels the device path uses, so the two agree bit for bit
wherever both apply.

With ``differentiable=True`` the episode's x and u carry gradients.  On the device path the forward also keeps each
solve's best iterate (``step.episode_raw(..., keep_plans=True)``) and the backward is one more library call
(``step.episode_backward_raw``), the closed loop's reverse sweep as one CUDA graph, with or without a slew-rate
penalty; the host path runs the same loop with autograd recording.
"""
import copy
from collections import namedtuple

import torch
from torch.autograd.function import once_differentiable

from . import solver
from ._lib import MpcB200Error
from .solver import CtrlPassthroughDynamics, LinDx, QuadCost, _mv

Episode = namedtuple("Episode", "x u costs info u_next")


def receding_horizon(ctrl, x_init, cost, dx, n_steps, differentiable=False):
    """Run `n_steps` control steps of receding-horizon MPC from `x_init` [B, n] with the solver `ctrl` (an ``MPC``,
    which supplies every solver option).  For k = 0 .. n_steps-1:

      * the plan: ``ctrl.forward(x_k, cost, dx)`` with ``u_init = w_k``; ``w_0`` is ``ctrl.u_init``, or zeros.  Every
        solve runs as with ``exit_unconverged=False, detach_unconverged=False`` (the notebooks' settings):
        ``ctrl``'s ``exit_unconverged``, ``detach_unconverged`` and ``backprop`` are not consulted;
      * the applied control: ``u_k = plan_u[0]``;
      * the next state, by the model itself: a known system (``CartpoleDx``, ``PendulumDx``) takes one step of its own
        dynamics, any other Module is called as ``dx(x_k, u_k)``, and ``LinDx`` takes its t = 0 slice,
        ``x_{k+1} = F_0 [x_k; u_k] + f_0``.  That is exact for a time-invariant system; a time-varying F is not
        shifted along the episode;
      * the next warm start: ``w_{k+1} = cat(plan_u[1:], 0)``, then ``w_{k+1}[-2] = w_{k+1}[-3]`` (the notebooks'
        rule, which needs T >= 3);
      * with ``ctrl.slew_rate_penalty``: solve k takes ``prev_ctrl = u_{k-1}``; solve 0 takes ``ctrl.prev_ctrl``, or
        zeros.

    Returns ``Episode(x, u, costs, info, u_next)``: x [n_steps+1, B, n] with x[0] = x_init, the applied controls u
    [n_steps, B, m], each solve's costs [n_steps, B], info int32 [n_steps, 2] (each solve's iterations, and iterations
    in which pnqp did not converge) and the warm start u_next [T, B, m] = w_{n_steps}.  A later call with
    ``ctrl.u_init = u_next`` (and ``ctrl.prev_ctrl = u[-1]`` under a slew-rate penalty) continues the same episode.
    pnqp warnings are printed as often as the solves would print them.

    ``differentiable=False`` (or grad mode off, or no input requires grad): every solve runs under
    ``torch.no_grad()`` and no output has a ``grad_fn``.  ``differentiable=True``: x and u carry gradients to
    ``x_init``, ``cost.C`` and ``cost.c`` (any shape ``MPC.forward`` takes), ``LinDx``'s F and f, and a known
    system's ``params``; costs, info and u_next carry none.  The gradient is exactly autograd's for the loop

        for k: _, plan_u, _ = ctrl'(x_k, cost, dx);  x_{k+1} = step(x_k, plan_u[0])

    with ``ctrl'`` = ``ctrl`` under ``exit_unconverged = detach_unconverged = False`` and ``u_init = w_k``: each solve
    contributes ``MPC.forward``'s differentiable tail (the KKT adjoint at its best iterate, with ``u_lower`` /
    ``u_upper`` as ``LQRStepFn.backward`` takes them; a known system's linearisation differentiated in its
    parameters, ``DynLinearize``), the model step its exact vector-Jacobian product in x_k, u_k and the parameters
    (``LinDx``: F[0], f[0]), and the warm starts w_k and ``prev_ctrl`` are held constant, as in the reference.
    Where the episode runs as one graph, with or without a slew-rate penalty, the backward is one more graph
    (``step.episode_backward_raw``); otherwise the host path's loop runs with autograd recording.  Under a slew-rate
    penalty each solve runs on the augmented state [u_{k-1}; x_k], and u_{k-1} is held constant there as the
    reference holds ``prev_ctrl``: no gradient flows through the previous control into the solve."""
    T, n, m = ctrl.T, ctrl.n_state, ctrl.n_ctrl
    if T < 3:
        raise MpcB200Error(f"a receding-horizon episode needs a horizon T >= 3 (the warm-start shift), got T={T}")
    if n_steps < 1:
        raise MpcB200Error(f"a receding-horizon episode needs n_steps >= 1, got {n_steps}")
    B = x_init.shape[0]
    cost = solver._expand_cost(cost, T, ctrl.n_batch if ctrl.n_batch is not None else B, n + m)
    w0 = _first_warm_start(ctrl, x_init)
    from .dynamics import params_scope
    if differentiable and torch.is_grad_enabled() and _requires_grad(x_init, cost, dx):
        with params_scope():
            if _takes_device_path(ctrl, x_init, cost, dx, w0):
                ep = _episode_device_grad(ctrl, x_init, cost, dx, n_steps, w0)
                if ep is not None:
                    return ep
            return _episode_host(ctrl, x_init, cost, dx, n_steps, w0)
    with torch.no_grad(), params_scope():     # a known system's CUDA parameters are read once per episode
        if _takes_device_path(ctrl, x_init, cost, dx, w0):
            ep = _episode_device(ctrl, x_init, cost, dx, n_steps, w0)
            if ep is not None:
                return ep
        return _episode_host(ctrl, x_init, cost, dx, n_steps, w0)


def _requires_grad(x_init, cost, dx):
    """Whether any input an episode differentiates in requires grad: x_init, a QuadCost's C and c (a Module cost's
    parameters), LinDx's F and f, or a Module's parameters and ``params``."""
    ts = [x_init]
    ts += [cost.C, cost.c] if isinstance(cost, QuadCost) else list(cost.parameters())
    if isinstance(dx, LinDx):
        ts += [dx.F, dx.f]
    else:
        ts += list(dx.parameters()) + [getattr(dx, "params", None)]
    return any(isinstance(t, torch.Tensor) and t.requires_grad for t in ts)


def _takes_device_path(ctrl, x_init, cost, dx, w0):
    """Whether the episode runs as one graph: exactly when each of its solves would take the device loop (T >= 3 is
    checked before).  Decided on tensor metadata alone."""
    return solver._use_device_loop(ctrl, x_init, cost, dx, w0) or \
        solver._use_slew_device_loop(ctrl, x_init, cost, dx, w0)


def shift_warm_start(plan_u):
    """The next solve's u_init from a plan [T, B, m]: cat(plan_u[1:], 0), then w[-2] = w[-3]."""
    w = torch.cat((plan_u[1:], torch.zeros_like(plan_u[:1])), 0)
    w[-2] = w[-3]
    return w


def _first_warm_start(ctrl, x_init):
    """w_0 [T, B, m]: ctrl.u_init ([T, m] expanded over the batch, or [T, B, m]) as MPC.forward takes it, or zeros."""
    T, B, m = ctrl.T, x_init.shape[0], ctrl.n_ctrl
    if ctrl.u_init is None:
        return torch.zeros(T, B, m, dtype=x_init.dtype, device=x_init.device)
    u = ctrl.u_init
    if u.ndimension() == 2:
        u = u.unsqueeze(1).expand(T, B, -1).clone()
    return u.to(dtype=x_init.dtype, device=x_init.device)


def _episode_device(ctrl, x_init, cost, dx, n_steps, w0):
    """The episode as one library call (step.episode_raw) on the problem MPC._ilqr_device stages, once; None when the
    driver refused the graph (nothing ran then)."""
    from . import step as _step
    T, m = ctrl.T, ctrl.n_ctrl
    n, x0, C, c, F, f, dyn = ctrl._device_problem(x_init, cost, dx)
    res = _step.episode_raw(n, m, T, n_steps, x0, C, c, F, f, w0, dyn=dyn, **ctrl._device_options())
    if res is None:
        solver._graph_cond_unavailable = True
        return None
    ctrl._print_pnqp_warnings(res["info"][:, 1].sum())      # the one host read, and only when they are printed
    x = res["x"][:, :, m:] if ctrl.slew_rate_penalty is not None else res["x"]
    return Episode(x, res["u"], res["costs"], res["info"], res["u_next"])


class _NoGraph(Exception):
    """The driver refused the episode's graph (nothing ran)."""


class EpisodeFn(torch.autograd.Function):
    """(x, u, costs, info, u_next) of a differentiable device episode: the forward is step.episode_raw with
    keep_plans, the backward one step.episode_backward_raw call.  One module-level Function (DESIGN.md section 3.2).
    `o` = (ctrl, dx, n_steps, w0); the known system's parameter values are the host numbers the forward took
    (params_scope) and the backward reuses them.  Under a slew-rate penalty the staged problem is the augmented one
    over [u_{k-1}; x] (MPC._device_problem): x is returned without its first m states, the backward pads dl_dx with
    m zeros in front, the sweep detaches those states (n_prev = m), and the gradients are cropped to the blocks of
    x_init, C, c, F and f inside the augmented ones (prev_ctrl and the warm starts get none).  Every tensor the
    backward reads (xs, us, the plans, the staged C, c,
    F, f and bounds) goes through save_for_backward, so an in-place edit of x or u before the backward raises, and the
    outputs do not keep themselves alive through ctx; ctx holds only the staged problem's metadata.  First order only:
    the backward is raw kernels."""

    @staticmethod
    def forward(ctx, o, x_init, C, c, F, f, params):
        from . import step as _step
        ctrl, dx, n_steps, w0 = o
        T, m = ctrl.T, ctrl.n_ctrl
        n, x0, C_, c_, F_, f_, dyn = ctrl._device_problem(x_init, QuadCost(C, c), dx)
        slew = ctrl.slew_rate_penalty is not None
        res = _step.episode_raw(n, m, T, n_steps, x0, C_, c_, F_, f_, w0, dyn=dyn, keep_plans=True,
                                n_prev=m if slew else 0, **ctrl._device_options())
        if res is None:
            raise _NoGraph()
        ctrl._print_pnqp_warnings(res["info"][:, 1].sum())
        s, ctx.n_steps, xs, us, plan_x, plan_u = res["saved"]
        ctx.save_for_backward(xs, us, plan_x, plan_u, s.C, s.c, s.F, s.f, s.u_lower, s.u_upper)
        ctx.problem = s._replace(C=None, c=None, F=None, f=None, u_lower=None, u_upper=None, u_zero_I=None)
        ctx.p_meta = (params.dtype, params.device) if params is not None else None
        ctx.mark_non_differentiable(res["costs"], res["info"], res["u_next"])
        x = res["x"][:, :, m:] if slew else res["x"]
        return x, res["u"], res["costs"], res["info"], res["u_next"]

    @staticmethod
    @once_differentiable
    def backward(ctx, dl_dx, dl_du, *_):
        from . import step as _step
        xs, us, plan_x, plan_u, C, c, F, f, lo, hi = ctx.saved_tensors
        s = ctx.problem._replace(C=C, c=c, F=F, f=f, u_lower=lo, u_upper=hi)
        n_steps, k = ctx.n_steps, s.n_prev
        if dl_dx is None:
            dl_dx = xs.new_zeros(n_steps + 1, s.dims.B, s.pad.n)
        elif k:                                   # the previous control's states: no gradient of their own
            dl_dx = torch.cat((dl_dx.new_zeros(n_steps + 1, s.dims.B, k), dl_dx), 2)
        if dl_du is None:
            dl_du = us.new_zeros(n_steps, s.dims.B, s.pad.m)
        dx_init, dC, dc, dF, df, dtheta = _step.episode_backward_raw((s, n_steps, xs, us, plan_x, plan_u), dl_dx,
                                                                     dl_du)
        if k:                                     # the blocks of x_init, C, c, F, f inside the augmented problem
            dx_init, dC, dc = dx_init[:, k:], dC[..., k:, k:], dc[..., k:]
            dF = dF[..., k:, k:] if dF is not None else None
            df = df[..., k:] if df is not None else None
        need = ctx.needs_input_grad
        dparams = None
        if dtheta is not None and need[6]:
            dparams = dtheta.sum(0).to(dtype=ctx.p_meta[0], device=ctx.p_meta[1])
        return (None, dx_init if need[1] else None, dC if need[2] else None, dc if need[3] else None,
                dF if need[4] else None, df if need[5] else None, dparams if need[6] else None)


def _episode_device_grad(ctrl, x_init, cost, dx, n_steps, w0):
    """The differentiable episode on the device path (EpisodeFn); None when the driver refused the graph."""
    F, f, params = None, None, None
    if isinstance(dx, LinDx):
        F, f = dx.F, dx.f
    else:
        params = getattr(dx, "params", None)
    try:
        x, u, costs, info, u_next = EpisodeFn.apply((ctrl, dx, n_steps, w0), x_init, cost.C, cost.c, F, f, params)
    except _NoGraph:
        solver._graph_cond_unavailable = True
        return None
    return Episode(x, u, costs, info, u_next)


def _episode_host(ctrl, x_init, cost, dx, n_steps, w):
    """The episode as a Python loop over MPC.forward, on a shallow copy of ctrl that takes each step's warm start.
    Differentiable where autograd records: the warm starts and prev_ctrl are held constant."""
    slew = ctrl.slew_rate_penalty is not None
    solve = copy.copy(ctrl)
    solve.exit_unconverged = solve.detach_unconverged = False
    xs, us, costs, infos = [x_init], [], [], []
    x, prev = x_init, ctrl.prev_ctrl
    for _ in range(n_steps):
        solve.u_init, solve.prev_ctrl = w, prev
        _, plan_u, plan_costs = solve(x, cost, dx)
        x = _model_step(solve, x, plan_u, cost, dx)
        w = shift_warm_start(plan_u.detach())
        if slew:
            prev = plan_u[0].detach()
        xs.append(x)
        us.append(plan_u[0])
        costs.append(plan_costs)
        infos.append(solve._solve_info.to(x_init.device))
    return Episode(torch.stack(xs), torch.stack(us), torch.stack(costs), torch.stack(infos), w)


def _model_step(solve, x, plan_u, cost, dx):
    """x_{k+1} from x_k and the plan, by the kernels the device path runs: a known system's rollout
    (dynamics.dyn_rollout_raw) or LinDx's (step.rollout_raw) over two steps, at t = 1; for a slew-rate penalty, that of
    the augmented problem over [u_{k-1}; x], cropped.  Differentiable through ModelStepFn.  Any other Module:
    dx(x_k, u_k)."""
    from .dynamics import DYN_LINEAR, dyn_rollout_raw, known_kind
    n, m = solve.n_state, solve.n_ctrl
    u2 = plan_u[:2].detach()
    xd = x.detach()
    lin = isinstance(dx, LinDx)
    own_kind, own_params = (DYN_LINEAR, None) if lin else known_kind(dx, n, m, x)
    if not lin and not own_kind:
        return dx(x, plan_u[0])
    if solve.slew_rate_penalty is not None and isinstance(cost, QuadCost):
        def value():
            F, f = (dx.F, dx.f) if lin else (None, None)
            _, _, _, F2, f2, _, x2 = solve._slew_augment(xd, cost.C, cost.c, F, f)
            if lin:
                return _lindx_step(n + m, m, x2, u2, F2, f2)[:, m:]
            kind, params = known_kind(CtrlPassthroughDynamics(dx), n + m, m, x2)
            return dyn_rollout_raw(kind, params, 2, x2, u2)[1][:, m:]
    elif lin:
        def value():
            return _lindx_step(n, m, xd, u2, dx.F, dx.f)
    else:
        def value():
            return dyn_rollout_raw(own_kind, own_params, 2, xd, u2)[1]
    if lin:
        return ModelStepFn.apply((value, DYN_LINEAR, None), x, plan_u[0], dx.F, dx.f, None)
    return ModelStepFn.apply((value, own_kind, own_params), x, plan_u[0], None, None, getattr(dx, "params", None))


class ModelStepFn(torch.autograd.Function):
    """The host path's model step x' = step(x, u) as one autograd node: the forward is `value()` (the kernels the
    device path runs, _model_step), the backward the step's exact vector-Jacobian product.  LinDx: x' = F[0] z + f[0]
    with z = [x; u], so dz = F[0]^T g, dF[0] = g z^T, df[0] = g.  A known system `kind` (the system itself, also
    under a slew-rate penalty, whose passthrough step is the system's step on x): [R S] = F[0] of
    dynamics.dyn_linearize_raw at T = 2, and d params = the VJP's `first` with df = g (x' depends on the parameters
    directly; the Jacobian is not differentiated).  An empty f (the reference's "no f") gets an empty gradient.
    `o` = (value, kind, kparams).  First order only."""

    @staticmethod
    def forward(ctx, o, x, u, F, f, params):
        value, kind, kparams = o
        ctx.kind, ctx.kparams = kind, kparams
        ctx.f_shape = f.shape if f is not None else None
        ctx.p_meta = (params.dtype, params.device) if params is not None else None
        ctx.save_for_backward(x, u, F)
        return value()

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        from .dynamics import DYN_LINEAR, dyn_linearize_raw, dyn_linearize_vjp_raw
        x, u, F = ctx.saved_tensors
        n = x.shape[1]
        need = ctx.needs_input_grad
        dF = df = dparams = None
        if ctx.kind == DYN_LINEAR:
            J = F[0].to(g.dtype)
            if need[3]:
                z = torch.cat((x, u), 1).to(g.dtype)
                dF = torch.zeros(F.shape, dtype=F.dtype, device=F.device)
                dF[0] = (g.unsqueeze(2) * z.unsqueeze(1)).to(F.dtype)
            if need[4] and ctx.f_shape is not None:
                df = torch.zeros(ctx.f_shape, dtype=g.dtype, device=g.device)
                if df.nelement() > 0:
                    df[0] = g
        else:
            x2, u2 = torch.stack((x, x)).detach(), torch.stack((u, u)).detach()
            J = dyn_linearize_raw(ctx.kind, ctx.kparams, 2, x2, u2)[0][0]
            if need[5] and ctx.p_meta is not None:
                first, _ = dyn_linearize_vjp_raw(ctx.kind, ctx.kparams, 2, x2, u2, torch.zeros_like(J).unsqueeze(0),
                                                 g.unsqueeze(0).contiguous())
                dparams = first[0].sum(0).to(dtype=ctx.p_meta[0], device=ctx.p_meta[1])
        dz = torch.einsum("bij,bi->bj", J, g)
        return None, dz[:, :n], dz[:, n:], dF, df, dparams


def _lindx_step(n, m, x, u2, F, f):
    """F_0 [x; u_0] + f_0: the rollout kernel over two steps where it takes the tensors (as solver.get_traj)."""
    f0 = f[:1] if f is not None and f.nelement() > 0 else None
    if x.is_cuda and x.dtype in (torch.float32, torch.float64) and F.dtype == x.dtype:
        from .step import rollout_raw
        return rollout_raw(n, m, 2, x, u2, F[:1], f0)[1]
    nx = _mv(F[0], torch.cat((x, u2[0]), 1))
    return nx + f0[0] if f0 is not None else nx
