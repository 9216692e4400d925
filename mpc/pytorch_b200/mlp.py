"""A learned model (``models.NNDynamics``) on the device: the network's rollout, exact linearisation and the
split-mode LQR step's line search run as CUDA kernels (csrc/mlp.cu), and MPC.forward's iLQR loop as one CUDA graph
(``mpcb200_ilqr_mlp_*``).

``on_device`` decides which networks take the kernels: exactly ``NNDynamics`` (a subclass may override ``forward``),
at the solve's (n_state, n_ctrl), with every parameter a CUDA tensor of the solve's dtype on its device, and small
enough for the kernels' shared memory (``mpcb200_mlp_fits``).  Everything else keeps the Module path.  The weights are
packed into one buffer once per solve (``dynamics.params_scope``), so an in-place edit between solves is seen.

Only the linearisation depends on ``MPC.grad_method`` (ANALYTIC / AUTO_DIFF take ``linearize_raw``; FINITE_DIFF keeps
its central differences in torch, and with it the host loop).  The rollout (``get_traj``) and the split-mode step's line
search compute the same function under every grad_method, so they take the kernels whenever ``on_device`` holds.
MPC's differentiable tail (``linearize_dynamics(diff=True)``) takes ``linearize_diff``: ``MlpLinearize``, whose backward
is the VJP of the linearisation in the weights (``mpcb200_mlp_linearize_vjp_*``, DESIGN.md section 3.11).

A receding-horizon episode planned with the network runs as one graph in each direction where ``episode_on_device``
holds (``episode_raw``, ``episode_backward_raw``; ``mpcb200_episode_mlp_*``, DESIGN.md section 3.12).
"""
import ctypes

import torch

from . import _lib
from ._lib import MpcB200Error, _on_device, check, ptr, ptr_view, stream_handle
from .dynamics import _scope
from .models import NNDynamics


def _net(dx):
    """The NNDynamics a dynamics Module steps with, and its n_prev: (dx, 0), or (inner, m) for a CtrlPassthroughDynamics
    around one (the slew-rate augmented state [u_{t-1}; x]); (None, 0) for anything else."""
    if type(dx) is NNDynamics:
        return dx, 0
    from .solver import CtrlPassthroughDynamics
    if type(dx) is CtrlPassthroughDynamics and type(dx.dynamics) is NNDynamics:
        return dx.dynamics, dx.dynamics.n_ctrl
    return None, 0


def _layout(net):
    """(widths, W_off, b_off) of the packed parameter block: W0 b0 W1 b1 ..., each row-major as nn.Linear stores it."""
    widths = [net.fcs[0].in_features] + [fc.out_features for fc in net.fcs]
    W_off, b_off, o = [], [], 0
    for fc in net.fcs:
        W_off.append(o)
        o += fc.weight.numel()
        b_off.append(o)
        o += fc.bias.numel()
    return widths, W_off, b_off


def _record(net, n_prev, params):
    """The mpcb200_mlp record of `net` with parameter block address `params`."""
    widths, W_off, b_off = _layout(net)
    rec = _lib.Mlp(n_layers=len(net.fcs), activation=_lib.ACT[net.activation], passthrough=int(bool(net.passthrough)),
                   n_prev=int(n_prev), params=params)
    for i, w in enumerate(widths):
        rec.width[i] = int(w)
    for i, (wo, bo) in enumerate(zip(W_off, b_off)):
        rec.W_off[i], rec.b_off[i] = int(wo), int(bo)
    return rec


def record(dx, x):
    """(mpcb200_mlp record, parameter buffer) of the network `dx` steps with, for tensors like `x`; the buffer must
    outlive the calls.  Within one params_scope (one MPC.forward) the packed buffer is reused."""
    net, n_prev = _net(dx)
    epoch = getattr(_scope, "epoch", None) if getattr(_scope, "depth", 0) else None
    hit = getattr(net, "_mpcb200_mlp_cache", None)
    if epoch is None or hit is None or hit[0] != epoch or hit[1] != x.dtype:
        parts = [t.detach().reshape(-1) for fc in net.fcs for t in (fc.weight, fc.bias)]
        hit = (epoch, x.dtype, torch.cat(parts).to(x.dtype).contiguous())
        if epoch is not None:
            net._mpcb200_mlp_cache = hit
    buf = hit[2]
    return _record(net, n_prev, buf.data_ptr()), buf


def fits(net, n_prev, elem_size):
    """Whether the kernels take `net` with n_prev leading previous-control states (mpcb200_mlp_fits), from its widths
    alone."""
    if len(net.fcs) > 4 or net.activation not in _lib.ACT:
        return False
    return bool(_lib.lib().mpcb200_mlp_fits(ctypes.byref(_record(net, n_prev, 1)), int(elem_size)))


def on_device(dx, n, m, x):
    """Whether the network of `dx` (NNDynamics, or CtrlPassthroughDynamics around one) runs in the kernels for a solve
    of (n_state n, n_ctrl m) on tensors like `x`: its own (n_state, n_ctrl) is the solve's (the inner network's plus
    the previous control for the passthrough form), every parameter is a CUDA tensor of x's dtype on x's device, and
    it fits the kernels.  Decided on metadata alone."""
    net, n_prev = _net(dx)
    if net is None or not isinstance(x, torch.Tensor) or not x.is_cuda:
        return False
    if x.dtype not in (torch.float32, torch.float64):
        return False
    if (net.n_state + n_prev, net.n_ctrl) != (n, m) or net.fcs[0].in_features != net.n_state + net.n_ctrl:
        return False
    if net.fcs[-1].out_features != net.n_state:
        return False
    if any(not p.is_cuda or p.dtype != x.dtype or p.device != x.device for p in net.parameters()):
        return False
    return fits(net, n_prev, x.element_size())


def rollout_raw(dx, T, x_init, u):
    """get_traj(T, u, x_init, dx) in one kernel: x [T, B, n]."""
    from .step import _dense
    B, n = x_init.shape
    m = u.shape[2]
    dtype, dev = x_init.dtype, x_init.device
    rec, buf = record(dx, x_init)
    x0_, u_ = _dense(x_init, dtype), _dense(u, dtype)
    x = torch.empty(T, B, n, dtype=dtype, device=dev)
    fn = _lib.entry("mpcb200_mlp_rollout", dtype)
    with _on_device(dev):
        rc = fn(ctypes.byref(rec), B, T, n, m, ptr(x0_), ptr(u_), ptr(x), stream_handle(dev))
    check(rc, "mpcb200_mlp_rollout")
    return x


def linearize_raw(dx, T, x, u, rec=None, buf=None):
    """MPC.linearize_dynamics(x, u, dx, diff=False) in one kernel: F [T-1, B, n, n+m], f [T-1, B, n].  rec, buf: the
    record and packed buffer to run (default: record(dx, x))."""
    from .step import _dense
    _, B, n = x.shape
    m = u.shape[2]
    dtype, dev = x.dtype, x.device
    if rec is None:
        rec, buf = record(dx, x)
    x_, u_ = _dense(x, dtype), _dense(u, dtype)
    F = torch.empty(T - 1, B, n, n + m, dtype=dtype, device=dev)
    f = torch.empty(T - 1, B, n, dtype=dtype, device=dev)
    fn = _lib.entry("mpcb200_mlp_linearize", dtype)
    with _on_device(dev):
        rc = fn(ctypes.byref(rec), B, T, n, m, ptr(x_), ptr(u_), ptr(F), ptr(f), stream_handle(dev))
    check(rc, "mpcb200_mlp_linearize")
    return F, f


def vjp_workspace_bytes(dx, B, T, elem_size):
    """Bytes of mpcb200_mlp_linearize_vjp_*'s workspace for the network of `dx`; 0 when its VJP does not fit the
    kernel's shared memory (mpcb200_mlp_linearize_vjp_workspace_bytes, no device needed)."""
    net, n_prev = _net(dx)
    return int(_lib.lib().mpcb200_mlp_linearize_vjp_workspace_bytes(ctypes.byref(_record(net, n_prev, 1)), int(B),
                                                                     int(T), int(elem_size)))


def linearize_vjp_raw(dx, T, x, u, dF, df, rec=None, buf=None):
    """dtheta [n_params]: the gradient of sum(dF * F) + sum(df * f) for (F, f) = linearize_raw(dx, T, x, u) in the
    network's parameters, packed W0 b0 W1 b1 ... as _layout orders them; two kernels.  rec, buf: the record and
    packed buffer to differentiate at (default: record(dx, x))."""
    from .step import _dense
    _, B, n = x.shape
    m = u.shape[2]
    dtype, dev = x.dtype, x.device
    for name, t, shape in (("dF", dF, (T - 1, B, n, n + m)), ("df", df, (T - 1, B, n))):
        if tuple(t.shape) != shape:
            raise MpcB200Error(f"{name}: expected shape {shape}, got {tuple(t.shape)}")
    if rec is None:
        rec, buf = record(dx, x)
    nbytes = vjp_workspace_bytes(dx, B, T, x.element_size())
    if nbytes == 0:
        raise MpcB200Error("mpcb200_mlp_linearize_vjp: the network's VJP does not fit the kernel's shared memory")
    x_, u_, dF_, df_ = (_dense(t, dtype) for t in (x, u, dF, df))
    dtheta = torch.empty(buf.numel(), dtype=dtype, device=dev)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    fn = _lib.entry("mpcb200_mlp_linearize_vjp", dtype)
    with _on_device(dev):
        rc = fn(ctypes.byref(rec), B, T, n, m, ptr(x_), ptr(u_), ptr(dF_), ptr(df_), ptr(dtheta), ptr(ws), nbytes,
                stream_handle(dev))
    check(rc, "mpcb200_mlp_linearize_vjp")
    return dtheta


def _torch_linearize(dx, x, u):
    """(F, f) of linearize_raw by torch ops: the network and NNDynamics.grad_input at every (t, b), as
    MPC.linearize_dynamics's ANALYTIC tail forms them; differentiable in the weights under enable_grad."""
    net, n_prev = _net(dx)
    T, B, N = x.shape
    m = u.shape[2]
    xs, us = x[:-1].reshape(-1, N)[:, n_prev:], u[:-1].reshape(-1, m)
    R, S = net.grad_input(xs, us)
    f = net(xs, us) - (R @ xs.unsqueeze(2)).squeeze(2) - (S @ us.unsqueeze(2)).squeeze(2)
    F = torch.cat((R, S), 2)
    if n_prev:                  # the rows [0 0 I] and f 0 of the previous control, no column for it in the network's
        eye = torch.eye(n_prev, dtype=x.dtype, device=x.device).expand(xs.shape[0], -1, -1)
        top = torch.cat((torch.zeros(xs.shape[0], n_prev, N, dtype=x.dtype, device=x.device), eye), 2)
        F = torch.cat((top, torch.cat((torch.zeros_like(F[:, :, :n_prev]), F), 2)), 1)
        f = torch.cat((torch.zeros_like(f[:, :n_prev]), f), 1)
    return F.view(T - 1, B, N, N + m), f.view(T - 1, B, N)


class MlpLinearize(torch.autograd.Function):
    """(F, f) = linearize_raw(dx, T, x, u) along detached (x, u), differentiable in the network's parameter tensors
    (the inputs after dx, T, x, u, in _layout's order W0 b0 W1 b1 ...): the backward is mpcb200_mlp_linearize_vjp_*
    on the packed buffer the forward used.  The parameters are saved for backward, so an in-place edit between the
    two raises autograd's version-counter error.  Under create_graph the backward recomputes the VJP with torch ops
    (_torch_linearize), so higher-order gradients are those of the torch path.  One module-level Function (DESIGN.md
    section 3.2)."""

    @staticmethod
    def forward(ctx, dx, T, x, u, *params):
        rec, buf = record(dx, x)
        F, f = linearize_raw(dx, T, x, u, rec, buf)
        ctx.save_for_backward(*params)
        ctx.dx, ctx.T, ctx.rec, ctx.buf, ctx.x, ctx.u = dx, T, rec, buf, x, u
        return F, f

    @staticmethod
    def backward(ctx, dF, df):
        params = ctx.saved_tensors              # raises if a parameter was edited in place since the forward
        want = ctx.needs_input_grad[4:]
        if torch.is_grad_enabled():             # create_graph: the torch formula, differentiable again
            net, _ = _net(ctx.dx)
            live = [t for fc in net.fcs for t in (fc.weight, fc.bias)]
            wanted = [p for p, w in zip(live, want) if w]
            F, f = _torch_linearize(ctx.dx, ctx.x, ctx.u)
            g = iter(torch.autograd.grad((F * dF).sum() + (f * df).sum(), wanted, create_graph=True,
                                         allow_unused=True))
            grads = [next(g) if w else None for w in want]
            grads = [torch.zeros_like(p) if w and gi is None else gi for p, w, gi in zip(params, want, grads)]
        else:
            dtheta = linearize_vjp_raw(ctx.dx, ctx.T, ctx.x, ctx.u, dF, df, ctx.rec, ctx.buf)
            grads, o = [], 0
            for p, w in zip(params, want):
                grads.append(dtheta[o:o + p.numel()].view(p.shape) if w else None)
                o += p.numel()
        return (None, None, None, None, *grads)


def linearize_diff(dx, T, x, u):
    """(F, f) of linearize_raw as MPC's differentiable tail needs them, or None where the torch tail must form them:
    through MlpLinearize when autograd records and a parameter of the network requires grad, one linearize_raw
    launch and no graph when none does; None when its VJP does not fit the kernel (vjp_workspace_bytes 0).  x and u
    are detached (no gradient reaches the linearisation point)."""
    net, _ = _net(dx)
    params = [t for fc in net.fcs for t in (fc.weight, fc.bias)]
    x, u = x.detach(), u.detach()
    if not torch.is_grad_enabled() or not any(p.requires_grad for p in params):
        return linearize_raw(dx, T, x, u)
    if vjp_workspace_bytes(dx, x.shape[1], T, x.element_size()) == 0:
        return None
    return MlpLinearize.apply(dx, T, x, u, *params)


def step_raw(dx, n_state, n_ctrl, T, x_init, C, c, F, f, cur_x, cur_u, u_lower=None, u_upper=None, u_zero_I=None,
             delta_u=None, linesearch_decay=0.2, max_linesearch_iter=10):
    """The split-mode LQR step with the network as the true dynamics and QuadCost(C, c) as the true cost
    (mpcb200_mlp_step_*): the step kernel's gains, then the line search in one kernel.  Returns a dict like
    lqr_step_raw(..., want_du_first=True)'s: new_x, new_u, costs, alphas, du_first, qp_iters, free_mask, status."""
    from .step import _dense, _problem, _validate
    n, m = n_state, n_ctrl
    B = _validate(n, m, T, ("C", C, "TBpp"), ("c", c, "TBp"), ("x_init", x_init, "Bn"), ("current_x", cur_x, "TBn"),
                  ("current_u", cur_u, "TBm"), F=F, f=f, bounds=(u_lower, u_upper), u_zero_I=u_zero_I)
    dtype, dev = C.dtype, C.device
    s = _problem(n, m, T, B, dtype, dev, C, c, F, f, u_lower, u_upper, u_zero_I, delta_u, linesearch_decay,
                 max_linesearch_iter)
    pad, dims, N, M = s.pad, s.dims, s.pad.N, s.pad.M
    dims.do_rollout = 0
    rec, buf = record(dx, C)
    x0_, cx_, cu_ = pad.vec_n(_dense(x_init, dtype)), pad.vec_n(_dense(cur_x, dtype)), pad.vec_m(_dense(cur_u, dtype))
    new_x = torch.empty(T, B, N, dtype=dtype, device=dev)
    new_u = torch.empty(T, B, M, dtype=dtype, device=dev)
    costs = torch.empty(B, dtype=dtype, device=dev)
    alphas = torch.empty(B, dtype=dtype, device=dev)
    du_first = torch.empty(T, B, M, dtype=dtype, device=dev)
    qp_iters = torch.zeros(T, B, dtype=torch.int32, device=dev) if dims.bounds_kind else None
    free_mask = torch.empty(T, B, M, dtype=torch.uint8, device=dev)
    status = torch.empty(B, dtype=torch.int32, device=dev)
    nbytes = _lib.lib().mpcb200_mlp_step_workspace_bytes(ctypes.byref(dims), C.element_size())
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    fn = _lib.entry("mpcb200_mlp_step", dtype)
    with _on_device(dev):
        rc = fn(ctypes.byref(dims), ctypes.byref(s.params), ctypes.byref(rec), ptr_view(s.C), ptr_view(s.c),
                ptr_view(s.F), ptr_view(s.f), ptr(x0_), ptr(cx_), ptr(cu_), ptr(s.u_lower), ptr(s.u_upper),
                ptr(s.u_zero_I), ptr(new_x), ptr(new_u), ptr(costs), ptr(alphas), ptr(du_first), ptr(qp_iters),
                ptr(free_mask), ptr(status), ptr(ws), nbytes, stream_handle(dev))
    check(rc, "mpcb200_mlp_step")
    return {"new_x": pad.crop_n(new_x), "new_u": pad.crop_m(new_u), "costs": costs, "alphas": alphas,
            "du_first": pad.crop_m(du_first), "qp_iters": qp_iters, "free_mask": pad.crop_m(free_mask),
            "status": status}


def ilqr_raw(dx, n_state, n_ctrl, T, x_init, C, c, u_init, u_lower=None, u_upper=None, u_zero_I=None, delta_u=None,
             linesearch_decay=0.2, max_linesearch_iter=10, lqr_iter=10, not_improved_lim=5, eps=1e-7,
             best_cost_eps=1e-4):
    """step.ilqr_raw with the network of `dx` as the dynamics (mpcb200_ilqr_mlp_*): one CUDA graph of rollout,
    linearisation, step, line search, tracking and stop test.  Under a slew-rate penalty `dx` is the
    CtrlPassthroughDynamics and the problem the augmented one.  Same outputs; None without conditional graph nodes."""
    from .step import _dense, _problem, _validate
    n, m = n_state, n_ctrl
    B = _validate(n, m, T, ("C", C, "TBpp"), ("c", c, "TBp"), ("x_init", x_init, "Bn"), ("u_init", u_init, "TBm"),
                  bounds=(u_lower, u_upper), u_zero_I=u_zero_I, need_F=False)
    dtype, dev = C.dtype, C.device
    s = _problem(n, m, T, B, dtype, dev, C, c, None, None, u_lower, u_upper, u_zero_I, delta_u, linesearch_decay,
                 max_linesearch_iter)
    pad, dims, N, M = s.pad, s.dims, s.pad.N, s.pad.M
    rec, buf = record(dx, C)
    x0_, u0_ = pad.vec_n(_dense(x_init, dtype)), pad.vec_m(_dense(u_init, dtype))
    opts = _lib.IlqrOpts(lqr_iter=int(lqr_iter), not_improved_lim=int(not_improved_lim), m_ref=m, eps=float(eps),
                         best_cost_eps=float(best_cost_eps))
    nbytes = _lib.lib().mpcb200_ilqr_mlp_workspace_bytes(ctypes.byref(dims), ctypes.byref(opts), C.element_size())
    if nbytes == 0:
        raise MpcB200Error("mpcb200_ilqr_mlp: the problem has no workspace size (T < 2 or bad dimensions)")
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    best_x = torch.empty(T, B, N, dtype=dtype, device=dev)
    best_u = torch.empty(T, B, M, dtype=dtype, device=dev)
    costs = torch.empty(B, dtype=dtype, device=dev)
    fdn = torch.empty(B, dtype=dtype, device=dev)
    info = torch.empty(2, dtype=torch.int32, device=dev)
    fn = _lib.entry("mpcb200_ilqr_mlp", dtype)
    with _on_device(dev):
        rc = fn(ctypes.byref(dims), ctypes.byref(s.params), ctypes.byref(opts), ctypes.byref(rec), ptr_view(s.C),
                ptr_view(s.c), ptr(x0_), ptr(u0_), ptr(s.u_lower), ptr(s.u_upper), ptr(s.u_zero_I), ptr(best_x),
                ptr(best_u), ptr(costs), ptr(fdn), ptr(info), ptr(ws), nbytes, stream_handle(dev))
    if rc == _lib.ERR_NO_GRAPH_COND:
        return None
    check(rc, "mpcb200_ilqr_mlp")
    return {"x": pad.crop_n(best_x), "u": pad.crop_m(best_u), "costs": costs, "full_du_norm": fdn, "info": info}


def episode_on_device(ctrl, x_init, cost, dx, w0, plant=None, time_varying=False, differentiable=False):
    """Whether a receding-horizon episode planned with the learned model `dx` runs as one graph
    (mpcb200_episode_mlp_*, and with `differentiable` mpcb200_episode_backward_mlp_*): `dx` is exactly NNDynamics and
    every solve would take MPC.forward's device loop with it (solver._use_device_loop: the network on the kernels,
    ANALYTIC or AUTO_DIFF, a QuadCost, verbose <= 0, ...); no slew-rate penalty and not time-varying; the plant is None
    or `dx` itself (the network steps the loop), a LinDx of x_init's dtype and device, or a known system at its own
    (n_state, n_ctrl) where the episode runs unpadded; and, with `differentiable`, the network's linearisation VJP
    fits its kernel.  Decided on metadata alone."""
    from . import solver
    from .control import _plant_on_device
    from .dynamics import DYN_LINEAR
    from .step import _pick_instance
    if type(dx) is not NNDynamics or ctrl.slew_rate_penalty is not None or time_varying:
        return False
    if not solver._use_device_loop(ctrl, x_init, cost, dx, w0):
        return False
    if plant is not None and plant is not dx:
        if isinstance(plant, NNDynamics) or not _plant_on_device(ctrl, x_init, dx, plant):
            return False
        if not isinstance(plant, solver.LinDx):       # a known plant steps at its own width: the staged one
            n, m = ctrl.n_state, ctrl.n_ctrl
            if _pick_instance(n, m, x_init.element_size(), DYN_LINEAR) != (n, m):
                return False
    return not differentiable or vjp_workspace_bytes(dx, x_init.shape[0], ctrl.T, x_init.element_size()) > 0


def episode_raw(dx, n_state, n_ctrl, T, n_steps, x_init, C, c, u_init, u_lower=None, u_upper=None, u_zero_I=None,
                delta_u=None, linesearch_decay=0.2, max_linesearch_iter=10, lqr_iter=10, not_improved_lim=5, eps=1e-7,
                best_cost_eps=1e-4, plant=None, w=None, keep_plans=False):
    """step.episode_raw with the network of `dx` as the model every solve plans with (mpcb200_episode_mlp_*): each
    solve is ilqr_raw's graph, and without a plant the network steps the loop by its rollout kernel at T = 2,
    x_{k+1} = rollout_raw(dx, 2, x_k, plan_u[:2])[1] (+ w_k).  plant: (kind, params, F_p, f_p) as step.episode_raw
    takes it (a LinDx's slice 0, or a known system), or None; w [n_steps, B, n] or None.  The weights are packed once
    (record, within the caller's params_scope).  Returns step.episode_raw's dict; keep_plans adds "saved", what
    episode_backward_raw takes.  None when the driver has no conditional graph nodes (nothing was launched then).
    step._stage_episode stages the call."""
    from .step import _call, _episode_result, _stage_episode
    s, name, args, out = _stage_episode(n_state, n_ctrl, T, n_steps, x_init, C, c, None, None, u_init, u_lower, u_upper,
                                        u_zero_I, delta_u, linesearch_decay, max_linesearch_iter, lqr_iter,
                                        not_improved_lim, eps, best_cost_eps, keep_plans=keep_plans, plant=plant, w=w,
                                        net=dx)
    return _episode_result(_call(name, C.dtype, C.device, args), name, s, out)


def episode_backward_raw(saved, dl_dxs, dl_dus):
    """The reverse sweep of an episode run by episode_raw(..., keep_plans=True) in ONE library call
    (mpcb200_episode_backward_mlp_*): `saved` is that call's res["saved"], dl_dxs [n_steps+1, B, n] and dl_dus
    [n_steps, B, m] the gradients of its x and u.  Returns (dx_init [B, n], dC [T, B, p, p], dc [T, B, p], dtheta
    [n_params], dF_p [B, n, p], df_p [B, n], dtheta_p [B, NP_plant], dw [n_steps, B, n]): dtheta is the network's
    packed W0 b0 W1 b1 ... (_layout); the plant's outputs are None where the episode had no such plant (or no f), dw
    None where it added no w.  step._stage_episode_backward stages the call."""
    from .step import _call, _episode_grads, _stage_episode_backward
    name, args, out = _stage_episode_backward(saved, dl_dxs, dl_dus)
    check(_call(name, saved[2].dtype, saved[2].device, args), name)
    g = _episode_grads(saved[0], out)
    return g[:3] + g[5:]
