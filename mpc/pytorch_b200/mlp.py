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


def linearize_raw(dx, T, x, u):
    """MPC.linearize_dynamics(x, u, dx, diff=False) in one kernel: F [T-1, B, n, n+m], f [T-1, B, n]."""
    from .step import _dense
    _, B, n = x.shape
    m = u.shape[2]
    dtype, dev = x.dtype, x.device
    rec, buf = record(dx, x)
    x_, u_ = _dense(x, dtype), _dense(u, dtype)
    F = torch.empty(T - 1, B, n, n + m, dtype=dtype, device=dev)
    f = torch.empty(T - 1, B, n, dtype=dtype, device=dev)
    fn = _lib.entry("mpcb200_mlp_linearize", dtype)
    with _on_device(dev):
        rc = fn(ctypes.byref(rec), B, T, n, m, ptr(x_), ptr(u_), ptr(F), ptr(f), stream_handle(dev))
    check(rc, "mpcb200_mlp_linearize")
    return F, f


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
