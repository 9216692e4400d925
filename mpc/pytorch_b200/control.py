"""Receding-horizon MPC: a closed-loop episode of solve, apply, shift and re-solve, the loop of the reference's
cartpole and pendulum notebooks, as one library call.

Where every solve of the episode would run on the device loop (``solver._use_device_loop`` /
``_use_slew_device_loop``), the whole episode is one CUDA graph (``step.episode_raw``): the solves, the model steps
and the warm-start shifts run on the device, with no host read between control steps.  Anything else (Module costs,
opaque Module dynamics, ``verbose > 0``, a driver without conditional graph nodes) runs the same loop from Python over
``MPC.forward``; that host path steps the model with the kernels the device path uses, so the two agree bit for bit
wherever both apply.
"""
import copy
from collections import namedtuple

import torch

from . import solver
from ._lib import MpcB200Error
from .solver import CtrlPassthroughDynamics, LinDx, QuadCost, _mv

Episode = namedtuple("Episode", "x u costs info u_next")


def receding_horizon(ctrl, x_init, cost, dx, n_steps):
    """Run `n_steps` control steps of receding-horizon MPC from `x_init` [B, n] with the solver `ctrl` (an ``MPC``,
    which supplies every solver option).  For k = 0 .. n_steps-1:

      * the plan: ``ctrl.forward(x_k, cost, dx)`` with ``u_init = w_k``; ``w_0`` is ``ctrl.u_init``, or zeros.  Every
        solve runs under ``torch.no_grad()`` as with ``exit_unconverged=False, detach_unconverged=False`` (the
        notebooks' settings): ``ctrl``'s ``exit_unconverged``, ``detach_unconverged`` and ``backprop`` are not
        consulted, and no gradient flows through an episode;
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
    pnqp warnings are printed as often as the solves would print them."""
    T, n, m = ctrl.T, ctrl.n_state, ctrl.n_ctrl
    if T < 3:
        raise MpcB200Error(f"a receding-horizon episode needs a horizon T >= 3 (the warm-start shift), got T={T}")
    if n_steps < 1:
        raise MpcB200Error(f"a receding-horizon episode needs n_steps >= 1, got {n_steps}")
    B = x_init.shape[0]
    cost = solver._expand_cost(cost, T, ctrl.n_batch if ctrl.n_batch is not None else B, n + m)
    w0 = _first_warm_start(ctrl, x_init)
    from .dynamics import params_scope
    with torch.no_grad(), params_scope():     # a known system's CUDA parameters are read once per episode
        if _takes_device_path(ctrl, x_init, cost, dx, w0):
            ep = _episode_device(ctrl, x_init, cost, dx, n_steps, w0)
            if ep is not None:
                return ep
        return _episode_host(ctrl, x_init, cost, dx, n_steps, w0)


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


def _episode_host(ctrl, x_init, cost, dx, n_steps, w):
    """The episode as a Python loop over MPC.forward, on a shallow copy of ctrl that takes each step's warm start."""
    slew = ctrl.slew_rate_penalty is not None
    solve = copy.copy(ctrl)
    solve.exit_unconverged = solve.detach_unconverged = False
    xs, us, costs, infos = [x_init], [], [], []
    x, prev = x_init, ctrl.prev_ctrl
    for _ in range(n_steps):
        solve.u_init, solve.prev_ctrl = w, prev
        _, plan_u, plan_costs = solve(x, cost, dx)
        x = _model_step(solve, x, plan_u, cost, dx)
        w = shift_warm_start(plan_u)
        if slew:
            prev = plan_u[0]
        xs.append(x)
        us.append(plan_u[0])
        costs.append(plan_costs)
        infos.append(solve._solve_info.to(x_init.device))
    return Episode(torch.stack(xs), torch.stack(us), torch.stack(costs), torch.stack(infos), w)


def _model_step(solve, x, plan_u, cost, dx):
    """x_{k+1} from x_k and the plan, by the kernels the device path runs: a known system's rollout
    (dynamics.dyn_rollout_raw) or LinDx's (step.rollout_raw) over two steps, at t = 1; for a slew-rate penalty, that of
    the augmented problem over [u_{k-1}; x], cropped.  Any other Module: dx(x_k, u_k)."""
    from .dynamics import dyn_rollout_raw, known_kind
    n, m = solve.n_state, solve.n_ctrl
    u2 = plan_u[:2]
    if solve.slew_rate_penalty is not None and isinstance(cost, QuadCost):
        F, f = (dx.F, dx.f) if isinstance(dx, LinDx) else (None, None)
        _, _, _, F2, f2, _, x2 = solve._slew_augment(x, cost.C, cost.c, F, f)
        if isinstance(dx, LinDx):
            return _lindx_step(n + m, m, x2, u2, F2, f2)[:, m:]
        kind, params = known_kind(CtrlPassthroughDynamics(dx), n + m, m, x2)
        if kind:
            return dyn_rollout_raw(kind, params, 2, x2, u2)[1][:, m:]
        return dx(x, plan_u[0])
    if isinstance(dx, LinDx):
        return _lindx_step(n, m, x, u2, dx.F, dx.f)
    kind, params = known_kind(dx, n, m, x)
    if kind:
        return dyn_rollout_raw(kind, params, 2, x, u2)[1]
    return dx(x, plan_u[0])


def _lindx_step(n, m, x, u2, F, f):
    """F_0 [x; u_0] + f_0: the rollout kernel over two steps where it takes the tensors (as solver.get_traj)."""
    f0 = f[:1] if f is not None and f.nelement() > 0 else None
    if x.is_cuda and x.dtype in (torch.float32, torch.float64) and F.dtype == x.dtype:
        from .step import rollout_raw
        return rollout_raw(n, m, 2, x, u2, F[:1], f0)[1]
    nx = _mv(F[0], torch.cat((x, u2[0]), 1))
    return nx + f0[0] if f0 is not None else nx
