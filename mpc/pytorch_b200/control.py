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

An episode planned with a learned model (``NNDynamics`` on the kernels, ``mlp.episode_on_device``: no slew-rate
penalty, not time-varying, the network itself, a LinDx or a known system stepping the loop) is one graph of its own in
both directions (``mlp.episode_raw`` / ``mlp.episode_backward_raw``, NetEpisodeFn); the network's step there is its
rollout kernel, where the host path calls the Module.
"""
import copy
from collections import namedtuple

import torch
from torch.autograd.function import once_differentiable

from . import solver
from ._lib import MpcB200Error
from .solver import CtrlPassthroughDynamics, LinDx, QuadCost, _mv

Episode = namedtuple("Episode", "x u costs info u_next")


def receding_horizon(ctrl, x_init, cost, dx, n_steps, differentiable=False, plant=None, disturbance=None,
                     time_varying=False):
    """Run `n_steps` control steps of receding-horizon MPC from `x_init` [B, n] with the solver `ctrl` (an ``MPC``,
    which supplies every solver option).  For k = 0 .. n_steps-1:

      * the plan: ``ctrl.forward(x_k, cost, dx)`` with ``u_init = w_k``; ``w_0`` is ``ctrl.u_init``, or zeros.  Every
        solve runs as with ``exit_unconverged=False, detach_unconverged=False`` (the notebooks' settings):
        ``ctrl``'s ``exit_unconverged``, ``detach_unconverged`` and ``backprop`` are not consulted;
      * the applied control: ``u_k = plan_u[0]``;
      * the next state, by the model itself: a known system (``CartpoleDx``, ``PendulumDx``) takes one step of its own
        dynamics, any other Module is called as ``dx(x_k, u_k)``, and ``LinDx`` takes its t = 0 slice,
        ``x_{k+1} = F_0 [x_k; u_k] + f_0`` (with ``time_varying=False``; see below for a time-varying F);
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
    reference holds ``prev_ctrl``: no gradient flows through the previous control into the solve.

    ``plant``: what steps the loop, while every solve still plans with ``dx``.  None (or ``dx`` itself) is the model.
    Otherwise a ``LinDx`` (its t = 0 slice, as the model's LinDx step), a known system with its own ``params``,
    ``force_mag`` / ``max_torque`` and ``dt`` (its kind may differ from the model's), or any other Module, called as
    ``plant(x_k, u_k)``; it must map (n_state, n_ctrl) to n_state.  ``disturbance``: w [n_steps, B, n] in x_init's
    dtype and on its device, or None.  The loop is then

        for k: _, plan_u, _ = ctrl'(x_k, cost, dx);  x_{k+1} = plant(x_k, plan_u[0]) + w_k

    and ``Episode.x[k+1]`` is the disturbed state (under a slew-rate penalty the plant steps x, and solve k still takes
    ``prev_ctrl = u_{k-1}``).  Its gradient is autograd's for that loop: the model's parameters (``params``, or F and
    f) get the solves' part only, the plant's the plant steps' exact VJP (a known system's ``params`` the VJP's
    ``first``; a LinDx's F[0], f[0]: g z^T and g), ``disturbance`` gets dL/dx_{k+1} at step k, and a tensor that the
    model and the plant share gets the sum.  The episode runs as one graph when the model's episode would and the
    plant steps at the staged shape (a LinDx plant with F, f on the episode's device and dtype; a known plant whose
    state width is the staged one); otherwise (an opaque Module plant, say) the host path runs, stepping the plant
    with the kernels the graph uses and adding w_k, so the two agree bit for bit wherever both apply.

    ``time_varying=True``: every time-indexed input lies on the episode's time axis of L = n_steps + T - 1 slices,
    and solve k plans on the window of absolute times k .. k+T-1.  ``cost`` is a QuadCost with C [L, B, p, p] or
    [L, p, p] (or [p, p], expanded to L) and c [L, B, p] or [L, p] (or [p]); a LinDx model's F and f, and a LinDx
    plant's, have a leading axis of L - 1 or L; tensor bounds ``ctrl.u_lower`` / ``ctrl.u_upper`` are [L, B, m].
    ``u_zero_I``, ``delta_u``, a known system's ``params`` and ``disturbance`` are not windowed.  A time-invariant
    piece is passed as a stride-0 ``expand(L, ...)``.  The loop is
        for k: _, plan_u, _ = ctrl'(x_k, QuadCost(C[k:k+T], c[k:k+T]), LinDx(F[k:k+F_T], f[k:k+f_T]))
               x_{k+1} = step_k(x_k, plan_u[0])
    with F_T = T - (L - len(F)) (and f_T likewise), bounds [k:k+T], and the model's (or a LinDx plant's) step at
    slice k: x_{k+1} = F[k] [x_k; u_k] + f[k] (+ w_k).  Gradients are autograd's for that loop: dC, dc, dF and df
    are full length, element t summing every solve whose window holds t and, for F[k], f[k], the step at k.  A
    later call continues the episode with the axis from n_steps on (C[n_steps : n_steps + n2 + T - 1], ...).
    Wrong lengths, and a Module cost, raise MpcB200Error before anything runs."""
    T, n, m = ctrl.T, ctrl.n_state, ctrl.n_ctrl
    if T < 3:
        raise MpcB200Error(f"a receding-horizon episode needs a horizon T >= 3 (the warm-start shift), got T={T}")
    if n_steps < 1:
        raise MpcB200Error(f"a receding-horizon episode needs n_steps >= 1, got {n_steps}")
    B = x_init.shape[0]
    if plant is dx:
        plant = None
    _check_plant(plant, disturbance, x_init, n, m, n_steps)
    L = n_steps + T - 1 if time_varying else None
    if time_varying:
        _check_axis(ctrl, cost, dx, plant, L, B)
    if plant is None and disturbance is not None:
        plant = dx                        # the model steps the disturbed loop
    cost = solver._expand_cost(cost, L or T, ctrl.n_batch if ctrl.n_batch is not None else B, n + m)
    w0 = _first_warm_start(ctrl, x_init)
    from .dynamics import params_scope
    from .mlp import episode_on_device
    if differentiable and torch.is_grad_enabled() and _requires_grad(x_init, cost, dx, plant, disturbance):
        with params_scope():
            if _takes_device_path(ctrl, x_init, cost, dx, w0, plant):
                ep = _episode_device_grad(ctrl, x_init, cost, dx, n_steps, w0, plant, disturbance, L)
                if ep is not None:
                    return ep
            if episode_on_device(ctrl, x_init, cost, dx, w0, plant, time_varying, differentiable=True):
                ep = _episode_device_grad(ctrl, x_init, cost, dx, n_steps, w0, plant, disturbance)
                if ep is not None:
                    return ep
            return _episode_host(ctrl, x_init, cost, dx, n_steps, w0, plant, disturbance, L)
    with torch.no_grad(), params_scope():     # a known system's CUDA parameters are read once per episode
        if _takes_device_path(ctrl, x_init, cost, dx, w0, plant):
            ep = _episode_device(ctrl, x_init, cost, dx, n_steps, w0, plant, disturbance, L)
            if ep is not None:
                return ep
        if episode_on_device(ctrl, x_init, cost, dx, w0, plant, time_varying):
            ep = _episode_device(ctrl, x_init, cost, dx, n_steps, w0, plant, disturbance)
            if ep is not None:
                return ep
        return _episode_host(ctrl, x_init, cost, dx, n_steps, w0, plant, disturbance, L)


def _check_axis(ctrl, cost, dx, plant, L, B):
    """The inputs of a time-varying episode against its axis of L slices, before anything runs: a QuadCost whose C
    and c have L slices (or no time axis: [p, p], [p]); a LinDx model's or plant's F and f with L - 1 or L; tensor
    bounds [L, B, m]."""
    n, m = ctrl.n_state, ctrl.n_ctrl
    if not isinstance(cost, QuadCost):
        raise MpcB200Error("time_varying=True needs a QuadCost: a Module cost has no time axis")
    for name, t, flat in (("cost.C", cost.C, 2), ("cost.c", cost.c, 1)):
        if not isinstance(t, torch.Tensor) or (t.dim() != flat and (t.dim() not in (flat + 1, flat + 2) or
                                                                    t.shape[0] != L)):
            raise MpcB200Error(f"{name}: a time-varying episode needs {L} slices (n_steps + T - 1), got shape "
                               f"{tuple(t.shape) if isinstance(t, torch.Tensor) else t}")
    for who, d in (("dx", dx), ("plant", plant)):
        if not isinstance(d, LinDx):
            continue
        for name, t in (("F", d.F), ("f", d.f)):
            if isinstance(t, torch.Tensor) and t.nelement() > 0 and t.shape[0] not in (L - 1, L):
                raise MpcB200Error(f"{who}: a time-varying episode needs a LinDx {name} of {L - 1} or {L} slices, "
                                   f"got shape {tuple(t.shape)}")
    for name, b in (("u_lower", ctrl.u_lower), ("u_upper", ctrl.u_upper)):
        if isinstance(b, torch.Tensor) and tuple(b.shape) != (L, B, m):
            raise MpcB200Error(f"{name}: a time-varying episode needs tensor bounds of shape {(L, B, m)}, got "
                               f"{tuple(b.shape)}")


def _check_plant(plant, w, x_init, n, m, n_steps):
    """A plant's shapes against the model's (n_state, n_ctrl) and w's against the episode, before anything runs.  An
    opaque Module without n_state / n_ctrl is checked on its output at every step (_plant_step)."""
    if isinstance(plant, LinDx):
        F, f = plant.F, plant.f
        if not isinstance(F, torch.Tensor) or F.dim() < 3 or F.shape[0] < 1 or tuple(F.shape[-2:]) != (n, n + m):
            raise MpcB200Error(f"plant: a LinDx plant needs F [T, B, {n}, {n + m}], got "
                               f"{tuple(F.shape) if isinstance(F, torch.Tensor) else F}")
        if f is not None and f.nelement() > 0 and (f.dim() < 2 or f.shape[0] < 1 or f.shape[-1] != n):
            raise MpcB200Error(f"plant: a LinDx plant needs f [T, B, {n}], got {tuple(f.shape)}")
    elif plant is not None:
        dims = (getattr(plant, "n_state", n), getattr(plant, "n_ctrl", m))
        if dims != (n, m):
            raise MpcB200Error(f"plant: maps (n_state, n_ctrl) = {dims}, the model {(n, m)}")
    if w is not None:
        B = x_init.shape[0]
        if tuple(w.shape) != (n_steps, B, n) or w.dtype != x_init.dtype or w.device != x_init.device:
            raise MpcB200Error(f"disturbance: expected a {x_init.dtype} tensor of shape {(n_steps, B, n)} on "
                               f"{x_init.device}, got a {w.dtype} tensor of shape {tuple(w.shape)} on {w.device}")


def _requires_grad(x_init, cost, dx, plant=None, w=None):
    """Whether any input an episode differentiates in requires grad: x_init, a QuadCost's C and c (a Module cost's
    parameters), LinDx's F and f, or a Module's parameters and ``params``, of the model and of the plant; and w."""
    ts = [x_init, w]
    ts += [cost.C, cost.c] if isinstance(cost, QuadCost) else list(cost.parameters())
    for d in (dx, plant):
        if isinstance(d, LinDx):
            ts += [d.F, d.f]
        elif d is not None:
            ts += list(d.parameters()) + [getattr(d, "params", None)]
    return any(isinstance(t, torch.Tensor) and t.requires_grad for t in ts)


def _takes_device_path(ctrl, x_init, cost, dx, w0, plant=None):
    """Whether the episode runs as one graph: exactly when each of its solves would take the device loop (T >= 3 is
    checked before) and the plant, if any, steps at the staged shape (_plant_on_device).  Decided on tensor metadata
    alone, which a time-varying episode's full-length inputs share with its windows, so the same rule serves both.
    A learned model (NNDynamics) as model or plant never runs on this graph: mlp.episode_on_device decides whether an
    episode planned with one runs on its own (mlp.episode_raw), and otherwise the host path runs it."""
    from .mlp import _net
    if _net(dx)[0] is not None or _net(plant)[0] is not None:     # the episode's graph cannot step a network
        return False
    return (solver._use_device_loop(ctrl, x_init, cost, dx, w0) or
            solver._use_slew_device_loop(ctrl, x_init, cost, dx, w0)) and \
        (plant is None or _plant_on_device(ctrl, x_init, dx, plant))


def _plant_on_device(ctrl, x_init, dx, plant):
    """Whether the plant steps inside the episode's graph: a LinDx plant whose F (and f) are tensors of the episode's
    dtype and device (staged like the model's, _Pad; in a time-varying episode whole, its slice k copied per step), or
    a known system whose state width, n or n + m under a slew-rate penalty, is the staged one.  A known model always
    runs at its own width; a LinDx model where _pick_instance gives the exact shape or the large-shape kernels."""
    from .dynamics import DYN_LINEAR, known_kind
    from .step import _pick_instance
    n, m = ctrl.n_state, ctrl.n_ctrl
    if isinstance(plant, LinDx):
        ts = [plant.F] + ([plant.f] if plant.f is not None and plant.f.nelement() > 0 else [])
        return all(t.dtype == x_init.dtype and t.device == x_init.device for t in ts)
    if known_kind(plant, n, m, x_init)[0] == DYN_LINEAR:
        return False
    if not isinstance(dx, LinDx):
        return True
    n_aug = n + m if ctrl.slew_rate_penalty is not None else n
    return _pick_instance(n_aug, m, x_init.element_size(), DYN_LINEAR) == (n_aug, m)


def _plant_spec(ctrl, x_init, C, plant, F_p, f_p, whole=False):
    """The plant as step.episode_raw takes it, on the problem MPC._device_problem stages: (DYN_LINEAR, None, F, f) of
    a LinDx plant (under a slew-rate penalty its slice 0 alone, the one that steps, augmented as MPC._slew_augment
    augments F, f; with `whole`, a time-varying episode's, every slice), or (kind, params, None, None) of a known
    system (its passthrough kind under a slew-rate penalty)."""
    from .dynamics import DYN_CTRL_PASSTHROUGH, DYN_LINEAR, known_kind
    slew = ctrl.slew_rate_penalty is not None
    if isinstance(plant, LinDx):
        if slew:                          # [[0, 0, I], [0, F_p]] and [0; f_p] of the slices that step
            m = ctrl.n_ctrl
            F0 = F_p if whole else F_p[:1]
            Fu = F0.new_zeros(F0.shape[0], F0.shape[1], m, F0.shape[3] + m)
            Fu[..., F0.shape[3]:] = torch.eye(m, dtype=F0.dtype, device=F0.device)
            F_p = torch.cat((Fu, torch.cat((F0.new_zeros(*F0.shape[:3], m), F0), 3)), 2)
            if f_p is not None and f_p.nelement() > 0:
                f0 = f_p if whole else f_p[:1]
                f_p = torch.cat((f0.new_zeros(f0.shape[0], f0.shape[1], m), f0), 2)
        return DYN_LINEAR, None, F_p, f_p
    kind, params = known_kind(plant, ctrl.n_state, ctrl.n_ctrl, x_init)
    return (kind | DYN_CTRL_PASSTHROUGH if slew else kind), params, None, None


def _staged_w(ctrl, w):
    """w as the augmented problem takes it under a slew-rate penalty: m zeros in front (the previous control)."""
    if w is None or ctrl.slew_rate_penalty is None:
        return w
    return torch.cat((w.new_zeros(*w.shape[:2], ctrl.n_ctrl), w), 2)


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


def _dyn_inputs(d):
    """(F, f, params) of a model or plant, the inputs a differentiable episode takes its gradients in: a LinDx's F and
    f, another Module's ``params`` (None without them); all None for None."""
    if isinstance(d, LinDx):
        return d.F, d.f, None
    return None, None, getattr(d, "params", None)


def _run_episode(ctrl, x_init, C, c, dx, n_steps, w0, plant, F_p, f_p, w, L=None, keep_plans=False):
    """The episode as one library call on the problem MPC._device_problem stages, once: mlp.episode_raw for a learned
    model, else step.episode_raw; None when the driver refused the graph (nothing ran then).  F_p, f_p: a LinDx
    plant's; L: a time-varying episode's axis (episode_raw's window)."""
    from . import mlp, step
    T, m = ctrl.T, ctrl.n_ctrl
    n, x0, C_, c_, F_, f_, dyn = ctrl._device_problem(x_init, QuadCost(C, c), dx, T=L)
    if dyn is not None and dyn[0] == "mlp":
        return mlp.episode_raw(dx, n, m, T, n_steps, x0, C_, c_, w0, keep_plans=keep_plans, w=w,
                               plant=_net_plant_spec(ctrl, x_init, C, dx, plant, F_p, f_p), **ctrl._device_options())
    kw = {}
    if plant is not None:
        kw = dict(plant=_plant_spec(ctrl, x_init, C, plant, F_p, f_p, whole=L is not None), w=_staged_w(ctrl, w))
    return step.episode_raw(n, m, T, n_steps, x0, C_, c_, F_, f_, w0, dyn=dyn, keep_plans=keep_plans,
                            n_prev=m if ctrl.slew_rate_penalty is not None else 0, window=L, **kw,
                            **ctrl._device_options())


def _episode_device(ctrl, x_init, cost, dx, n_steps, w0, plant=None, w=None, L=None):
    """The episode as one library call (_run_episode); None when the driver refused the graph (nothing ran then)."""
    F_p, f_p, _ = _dyn_inputs(plant)
    res = _run_episode(ctrl, x_init, cost.C, cost.c, dx, n_steps, w0, plant, F_p, f_p, w, L)
    if res is None:
        solver._graph_cond_unavailable = True
        return None
    ctrl._print_pnqp_warnings(res["info"][:, 1].sum())      # the one host read, and only when they are printed
    x = res["x"][:, :, ctrl.n_ctrl:] if ctrl.slew_rate_penalty is not None else res["x"]
    return Episode(x, res["u"], res["costs"], res["info"], res["u_next"])


class _NoGraph(Exception):
    """The driver refused the episode's graph (nothing ran)."""


def _keep_for_backward(ctx, ctrl, res, F_p, f_p, plant_params, whole, *weights):
    """What a differentiable episode's backward reads, from the forward's res: every tensor (xs, us, the plans, the
    staged C, c, F, f, bounds and plant, `weights`) through save_for_backward, so an in-place edit before the backward
    raises and the outputs do not keep themselves alive through ctx; ctx holds only the staged problem's metadata and
    that of the plant's inputs.  The pnqp warnings are printed here, once."""
    ctrl._print_pnqp_warnings(res["info"][:, 1].sum())
    s, ctx.n_steps, xs, us, plan_x, plan_u = res["saved"]
    sp = s.plant
    ctx.save_for_backward(xs, us, plan_x, plan_u, s.C, s.c, s.F, s.f, s.u_lower, s.u_upper,
                          sp.F if sp is not None else None, sp.f if sp is not None else None, *weights)
    ctx.problem = s._replace(C=None, c=None, F=None, f=None, u_lower=None, u_upper=None, u_zero_I=None,
                             plant=sp._replace(F=None, f=None) if sp is not None else None)
    ctx.plant_meta = (F_p.shape if F_p is not None else None, f_p.shape if f_p is not None else None,
                      (plant_params.dtype, plant_params.device) if plant_params is not None else None, whole)
    ctx.mark_non_differentiable(res["costs"], res["info"], res["u_next"])


def _saved_for_backward(ctx, dl_dx, dl_du):
    """(saved as the backward raw call takes it, dl_dx, dl_du, weights) from _keep_for_backward's ctx: a missing
    gradient is zeros, and under a slew-rate penalty dl_dx gets zeros in front for the previous control's states."""
    xs, us, plan_x, plan_u, C, c, F, f, lo, hi, Fp, fp, *weights = ctx.saved_tensors    # raises after an in-place edit
    s = ctx.problem._replace(C=C, c=c, F=F, f=f, u_lower=lo, u_upper=hi)
    if s.plant is not None:
        s = s._replace(plant=s.plant._replace(F=Fp, f=fp))
    n_steps, k = ctx.n_steps, s.n_prev
    if dl_dx is None:
        dl_dx = xs.new_zeros(n_steps + 1, s.dims.B, s.pad.n)
    elif k:                                   # the previous control's states: no gradient of their own
        dl_dx = torch.cat((dl_dx.new_zeros(n_steps + 1, s.dims.B, k), dl_dx), 2)
    if dl_du is None:
        dl_du = us.new_zeros(n_steps, s.dims.B, s.pad.m)
    return (s, n_steps, xs, us, plan_x, plan_u), dl_dx, dl_du, weights


def _plant_grads(ctx, need, dF_p, df_p, dth_p):
    """The plant's gradients as its inputs take them, where `need` (F_p, f_p, params) asks for them: a LinDx plant's
    in slice 0 of F_p, f_p (whole in a time-varying episode, where slice k steps control step k), a known plant's
    params summed over the batch."""
    F_shape, f_shape, pp_meta, whole = ctx.plant_meta

    def placed(g, shape):
        if whole:
            return g
        out = g.new_zeros(shape)
        out[0] = g
        return out
    dFp = placed(dF_p, F_shape) if dF_p is not None and need[0] else None
    dfp = placed(df_p, f_shape) if df_p is not None and need[1] else None
    dpp = dth_p.sum(0).to(dtype=pp_meta[0], device=pp_meta[1]) if dth_p is not None and need[2] else None
    return dFp, dfp, dpp


class EpisodeFn(torch.autograd.Function):
    """(x, u, costs, info, u_next) of a differentiable device episode: the forward is step.episode_raw with
    keep_plans, the backward one step.episode_backward_raw call.  One module-level Function (DESIGN.md section 3.2).
    `o` = (ctrl, dx, n_steps, w0, plant, L); the known system's parameter values are the host numbers the forward took
    (params_scope) and the backward reuses them.  Under a slew-rate penalty the staged problem is the augmented one
    over [u_{k-1}; x] (MPC._device_problem): x is returned without its first m states, the backward pads dl_dx with
    m zeros in front, the sweep detaches those states (n_prev = m), and the gradients are cropped to the blocks of
    x_init, C, c, F and f inside the augmented ones (prev_ctrl and the warm starts get none).  The backward reads
    only what _keep_for_backward kept.  First order only: the backward is raw kernels.  `o[4]` a plant
    (receding_horizon's `plant`), or None: F_p, f_p (a LinDx plant's), plant_params (a known plant's) and w are then
    inputs too, and their gradients come from the plant sweep (step.episode_backward_raw), F_p's and f_p's in slice
    0 (_plant_grads).  `o[5]` a time-varying episode's axis L, or None: C, c, F, f, bounds and a LinDx plant's F_p,
    f_p are full length, and so are their gradients."""

    @staticmethod
    def forward(ctx, o, x_init, C, c, F, f, params, F_p=None, f_p=None, plant_params=None, w=None):
        ctrl, dx, n_steps, w0, plant, L = o
        res = _run_episode(ctrl, x_init, C, c, dx, n_steps, w0, plant, F_p, f_p, w, L, keep_plans=True)
        if res is None:
            raise _NoGraph()
        _keep_for_backward(ctx, ctrl, res, F_p, f_p, plant_params, L is not None)
        ctx.p_meta = (params.dtype, params.device) if params is not None else None
        m = ctrl.n_ctrl
        x = res["x"][:, :, m:] if ctrl.slew_rate_penalty is not None else res["x"]
        return x, res["u"], res["costs"], res["info"], res["u_next"]

    @staticmethod
    @once_differentiable
    def backward(ctx, dl_dx, dl_du, *_):
        from . import step as _step
        saved, dl_dx, dl_du, _ = _saved_for_backward(ctx, dl_dx, dl_du)
        out = _step.episode_backward_raw(saved, dl_dx, dl_du)
        dx_init, dC, dc, dF, df, dtheta = out[:6]
        dF_p, df_p, dth_p, dw = out[6:] if len(out) > 6 else (None, None, None, None)
        k = saved[0].n_prev
        if k:                                     # the blocks of x_init, C, c, F, f inside the augmented problem
            dx_init, dC, dc = dx_init[:, k:], dC[..., k:, k:], dc[..., k:]
            dF = dF[..., k:, k:] if dF is not None else None
            df = df[..., k:] if df is not None else None
            dF_p = dF_p[..., k:, k:] if dF_p is not None else None
            df_p = df_p[..., k:] if df_p is not None else None
            dw = dw[..., k:] if dw is not None else None
        need = ctx.needs_input_grad
        dparams = None
        if dtheta is not None and need[6]:
            dparams = dtheta.sum(0).to(dtype=ctx.p_meta[0], device=ctx.p_meta[1])
        return (None, dx_init if need[1] else None, dC if need[2] else None, dc if need[3] else None,
                dF if need[4] else None, df if need[5] else None, dparams,
                *_plant_grads(ctx, need[7:10], dF_p, df_p, dth_p), dw if dw is not None and need[10] else None)


def _net_plant_spec(ctrl, x_init, C, dx, plant, F_p=None, f_p=None):
    """The plant of an episode planned with a learned model as mlp.episode_raw takes it: None where the network itself
    steps the loop (plant None or dx), else _plant_spec's."""
    if plant is None or plant is dx:
        return None
    return _plant_spec(ctrl, x_init, C, plant, F_p, f_p)


class NetEpisodeFn(torch.autograd.Function):
    """(x, u, costs, info, u_next) of a differentiable episode planned with a learned model: the forward is
    mlp.episode_raw with keep_plans, the backward one mlp.episode_backward_raw call.  One module-level Function
    (DESIGN.md section 3.2).  `o` = (ctrl, dx, n_steps, w0, plant).  The inputs after o are x_init, C, c, a LinDx
    plant's F_p and f_p, a known plant's params, w, and the network's weights and biases in _layout's order W0 b0 W1
    b1 ...; dtheta of the sweep is split into views shaped like them.  The weights, like every tensor the backward
    reads, go through save_for_backward (_keep_for_backward), so an in-place edit of a weight before the backward
    raises; the staged problem holds the packed weights the forward ran with.  First order only: the backward is raw
    kernels.  costs, info and u_next carry no gradient."""

    @staticmethod
    def forward(ctx, o, x_init, C, c, F_p, f_p, plant_params, w, *weights):
        ctrl, dx, n_steps, w0, plant = o
        res = _run_episode(ctrl, x_init, C, c, dx, n_steps, w0, plant, F_p, f_p, w, keep_plans=True)
        if res is None:
            raise _NoGraph()
        _keep_for_backward(ctx, ctrl, res, F_p, f_p, plant_params, False, *weights)
        return res["x"], res["u"], res["costs"], res["info"], res["u_next"]

    @staticmethod
    @once_differentiable
    def backward(ctx, dl_dx, dl_du, *_):
        from .mlp import episode_backward_raw
        saved, dl_dx, dl_du, weights = _saved_for_backward(ctx, dl_dx, dl_du)
        dx_init, dC, dc, dtheta, dF_p, df_p, dth_p, dw = episode_backward_raw(saved, dl_dx, dl_du)
        need = ctx.needs_input_grad
        dweights, o = [], 0
        for p, want in zip(weights, need[8:]):
            dweights.append(dtheta[o:o + p.numel()].view(p.shape) if want else None)
            o += p.numel()
        return (None, dx_init if need[1] else None, dC if need[2] else None, dc if need[3] else None,
                *_plant_grads(ctx, need[4:7], dF_p, df_p, dth_p), dw if dw is not None and need[7] else None,
                *dweights)


def _episode_device_grad(ctrl, x_init, cost, dx, n_steps, w0, plant=None, w=None, L=None):
    """The differentiable episode on the device (NetEpisodeFn for a learned model, else EpisodeFn); None when the
    driver refused the graph."""
    from .models import NNDynamics
    plant_in = _dyn_inputs(plant) + (w,)
    try:
        if type(dx) is NNDynamics:
            weights = [t for fc in dx.fcs for t in (fc.weight, fc.bias)]
            out = NetEpisodeFn.apply((ctrl, dx, n_steps, w0, plant), x_init, cost.C, cost.c, *plant_in, *weights)
        else:
            out = EpisodeFn.apply((ctrl, dx, n_steps, w0, plant, L), x_init, cost.C, cost.c, *_dyn_inputs(dx),
                                  *plant_in)
    except _NoGraph:
        solver._graph_cond_unavailable = True
        return None
    return Episode(*out)


def _episode_host(ctrl, x_init, cost, dx, n_steps, w, plant=None, dist=None, L=None):
    """The episode as a Python loop over MPC.forward, on a shallow copy of ctrl that takes each step's warm start.
    Differentiable where autograd records: the warm starts and prev_ctrl are held constant.  A plant steps the loop
    in the model's place (_model_step applied to it), and dist[k] is added to its step.  L: a time-varying episode's
    axis; step k then solves and steps on its window (_window)."""
    slew = ctrl.slew_rate_penalty is not None
    solve = copy.copy(ctrl)
    solve.exit_unconverged = solve.detach_unconverged = False
    xs, us, costs, infos = [x_init], [], [], []
    x, prev = x_init, ctrl.prev_ctrl
    cost_k, dx_k, plant_k = cost, dx, plant
    for k in range(n_steps):
        solve.u_init, solve.prev_ctrl = w, prev
        if L is not None:
            cost_k, dx_k, plant_k = _window(ctrl, solve, cost, dx, plant, k, L)
        _, plan_u, plan_costs = solve(x, cost_k, dx_k)
        if plant_k is None:
            x = _model_step(solve, x, plan_u, cost_k, dx_k)
        else:
            x = _plant_step(solve, x, plan_u, cost_k, plant_k, dist[k] if dist is not None else None)
        w = shift_warm_start(plan_u.detach())
        if slew:
            prev = plan_u[0].detach()
        xs.append(x)
        us.append(plan_u[0])
        costs.append(plan_costs)
        infos.append(solve._solve_info.to(x_init.device))
    return Episode(torch.stack(xs), torch.stack(us), torch.stack(costs), torch.stack(infos), w)


def _window(ctrl, solve, cost, dx, plant, k, L):
    """Control step k of a time-varying episode on the host path: QuadCost(C[k:k+T], c[k:k+T]), a LinDx model's
    LinDx(F[k:k+F_T], f[k:k+f_T]) (F_T = T - (L - len(F))), tensor bounds [k:k+T] set on `solve`, and a LinDx
    plant's slice k (a plant that is the model steps with the model's window)."""
    T = ctrl.T

    def lin(d, n_keep):
        f = d.f
        if isinstance(f, torch.Tensor) and f.nelement() > 0:
            f = f[k:k + (n_keep - (L - f.shape[0]) if n_keep == T else n_keep)]
        return LinDx(d.F[k:k + (n_keep - (L - d.F.shape[0]) if n_keep == T else n_keep)], f)
    for name in ("u_lower", "u_upper"):
        b = getattr(ctrl, name)
        if isinstance(b, torch.Tensor):
            setattr(solve, name, b[k:k + T])
    dx_k = lin(dx, T) if isinstance(dx, LinDx) else dx
    if plant is dx:
        plant_k = dx_k
    else:
        plant_k = lin(plant, 1) if isinstance(plant, LinDx) else plant
    return QuadCost(cost.C[k:k + T], cost.c[k:k + T]), dx_k, plant_k


def _plant_step(solve, x, plan_u, cost, plant, w_k):
    """x_{k+1} = plant(x_k, u_k) + w_k on the host path: the plant stepped as _model_step steps the model (the
    kernels the device path runs, or a Module call), then w_k added."""
    nx = _model_step(solve, x, plan_u, cost, plant)
    if tuple(nx.shape) != tuple(x.shape):
        raise MpcB200Error(f"plant: returned a state of shape {tuple(nx.shape)} for x_k of shape {tuple(x.shape)}")
    return nx + w_k if w_k is not None else nx


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
