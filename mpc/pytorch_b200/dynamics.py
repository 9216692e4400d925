"""Known nonlinear systems whose step function and exact Jacobians run inside the CUDA kernels
(SURVEY.md section 8(f) rank 2): drop-in stand-ins for the reference's example environments
``mpc.env_dx.cartpole.CartpoleDx`` (mpc/env_dx/cartpole.py:28-96) and ``mpc.env_dx.pendulum.PendulumDx``
(mpc/env_dx/pendulum.py:17-84, both the ``simple`` (g, m, l) and the five-parameter (g, m, l, d, b) form).

They are ordinary ``nn.Module`` dynamics - ``forward(x, u)`` is plain torch, so they work anywhere a Module
does - but they also carry ``mpcb200_kind`` / ``mpcb200_params()``.  ``MPC.forward`` recognises that and, on
CUDA tensors, replaces
  * ``util.get_traj``            (T-1 Python calls of the Module per iteration)        -> ``mpcb200_dyn_rollout``
  * ``MPC.linearize_dynamics``   ((T-1)*n_state autograd passes in AUTO_DIFF mode)     -> ``mpcb200_dyn_linearize``
  * its differentiable form in the solve's backward (autograd of those passes)      -> ``mpcb200_dyn_linearize_vjp``
  * the Module rollout of ``lqr_forward`` (reference mpc/lqr_step.py:224-225)          -> inside the step kernel
so that one iLQR iteration is three kernel launches plus the best-iterate bookkeeping.
"""
import contextlib
import ctypes
import itertools
import threading

import torch
from torch.nn import Module

from . import _lib
from ._lib import MpcB200Error, _on_device, check, ptr, stream_handle

# DYN_PENDULUM is PendulumDx(simple=True), DYN_PENDULUM_FULL PendulumDx(simple=False)
DYN_LINEAR, DYN_CARTPOLE, DYN_PENDULUM, DYN_PENDULUM_FULL = 0, 1, 2, 4
# OR'd into a known system's kind: that system under a slew-rate penalty, state [u_{t-1}; x]
# (solver.CtrlPassthroughDynamics), which the step runs on a dynamics-only kernel instance
DYN_CTRL_PASSTHROUGH = 16
DYN_KNOWN = (DYN_CARTPOLE, DYN_PENDULUM, DYN_PENDULUM_FULL)
# (n_state, n_ctrl) of each known system
DYN_DIMS = {DYN_CARTPOLE: (5, 1), DYN_PENDULUM: (3, 1), DYN_PENDULUM_FULL: (3, 1)}
DYN_DIMS.update({k | DYN_CTRL_PASSTHROUGH: (n + m, m) for k, (n, m) in DYN_DIMS.items()})
# number of learnable parameters of each system: the leading entries of its `params` tensor (mpcb200_params()[:NP])
DYN_NPARAMS = {DYN_CARTPOLE: 4, DYN_PENDULUM: 3, DYN_PENDULUM_FULL: 5}
# kinds whose step runs on a dynamics-only kernel instance of their own (csrc/dyn_instances.def), at exactly their
# (n_state, n_ctrl): the passthrough kinds, and the systems the (n, m) instances' line search has no branch for
DYN_OWN_INSTANCE = frozenset({DYN_PENDULUM_FULL} | {k | DYN_CTRL_PASSTHROUGH for k in DYN_KNOWN})

_scope = threading.local()      # depth and epoch of the enclosing params_scope() on this thread
_epochs = itertools.count(1)    # process-wide: two threads' scopes never share an epoch (the cache is per module)


@contextlib.contextmanager
def params_scope():
    """One solve (``MPC.forward``): inside it, CUDA parameter tensors of known systems are read back to the host
    once, not once per kernel launch (a device->host read per launch would serialise every iLQR iteration).
    Nested scopes share the outermost one's values.  Outside any scope every read is fresh, so a direct
    ``LQRStep`` call reads them once (its forward asks once)."""
    depth = getattr(_scope, "depth", 0)
    if depth == 0:
        _scope.epoch = next(_epochs)
    _scope.depth = depth + 1
    try:
        yield
    finally:
        _scope.depth = depth


def _host_values(owner, params):
    """Python floats of a (possibly CUDA, possibly learnable) parameter tensor, as ``forward`` would use them now.
    The kernels take the parameters by value.  CPU tensors are read on every call (free); CUDA tensors once per
    params_scope().  Tensor versions cannot tell whether the values changed: an edit through ``.data`` does not
    bump ``_version``, and a reassigned tensor may reuse the old one's storage."""
    if not params.is_cuda or getattr(_scope, "depth", 0) == 0:
        return tuple(float(v) for v in params.detach().cpu())
    hit = getattr(owner, "_mpcb200_host_cache", None)
    if hit is None or hit[0] != _scope.epoch or hit[1] is not params:
        hit = (_scope.epoch, params, tuple(float(v) for v in params.detach().cpu()))
        owner._mpcb200_host_cache = hit
    return hit[2]


class CartpoleDx(Module):
    """state = (x, dx, cos th, sin th, dth), one control (force, clamped to +-force_mag), semi-implicit Euler."""
    mpcb200_kind = DYN_CARTPOLE
    n_state, n_ctrl = 5, 1

    def __init__(self, params=None):
        super().__init__()
        # gravity, masscart, masspole, length
        self.params = torch.tensor((9.8, 1.0, 0.1, 0.5)) if params is None else params
        assert len(self.params) == 4
        self.force_mag = 100.0
        self.dt = 0.05
        self.lower, self.upper = -self.force_mag, self.force_mag
        self.goal_state = torch.tensor([0.0, 0.0, 1.0, 0.0, 0.0])
        self.goal_weights = torch.tensor([0.1, 0.1, 1.0, 1.0, 0.1])
        self.ctrl_penalty = 0.001
        self.mpc_eps = 1e-4
        self.linesearch_decay = 0.5
        self.max_linesearch_iter = 2

    def mpcb200_params(self):
        g, mc, mp, l = _host_values(self, self.params)
        return (g, mc, mp, l, float(self.force_mag), float(self.dt), 0.0, 0.0)

    def forward(self, state, u):
        single = state.dim() == 1
        if single:
            state, u = state.unsqueeze(0), u.unsqueeze(0)
        # pinned parameters are copied without a host synchronisation, which also lets torch.cuda.graph capture it
        g, mc, mp, l = self.params.to(state, non_blocking=self.params.is_pinned()).unbind()
        total, pml = mp + mc, mp * l
        force = u[:, 0].clamp(-self.force_mag, self.force_mag)
        pos, vel, c, s, om = state.unbind(1)
        th = torch.atan2(s, c)
        cart_in = (force + pml * om ** 2 * s) / total
        th_acc = (g * s - c * cart_in) / (l * (4.0 / 3.0 - mp * c ** 2 / total))
        acc = cart_in - pml * th_acc * c / total
        th2 = th + self.dt * om
        out = torch.stack((pos + self.dt * vel, vel + self.dt * acc, torch.cos(th2), torch.sin(th2),
                           om + self.dt * th_acc), 1)
        return out.squeeze(0) if single else out

    def get_true_obj(self):
        q = torch.cat((self.goal_weights, self.ctrl_penalty * torch.ones(self.n_ctrl)))
        p = torch.cat((-torch.sqrt(self.goal_weights) * self.goal_state, torch.zeros(self.n_ctrl)))
        return q, p


class PendulumDx(Module):
    """state = (cos th, sin th, dth), one control (torque, clamped to +-max_torque).  ``simple=True``: the
    reference's (g, m, l) parametrisation (kind DYN_PENDULUM).  ``simple=False``: its five-parameter form
    (g, m, l, d, b) with damping d and gravity bias b (kind DYN_PENDULUM_FULL), written as the reference writes it:
    d multiplies the wrapped angle atan2(sin th, cos th), and gravity acts through sin(th + b), not the state's
    sin th."""
    mpcb200_kind = DYN_PENDULUM
    n_state, n_ctrl = 3, 1

    def __init__(self, params=None, simple=True):
        super().__init__()
        self.simple = bool(simple)
        if not self.simple:
            self.mpcb200_kind = DYN_PENDULUM_FULL
        self.max_torque = 2.0
        self.dt = 0.05
        if params is None:
            params = torch.tensor((10.0, 1.0, 1.0) if self.simple else (10.0, 1.0, 1.0, 0.0, 0.0))
        self.params = params
        if self.simple:
            assert len(self.params) == 3
        elif len(self.params) != 5:
            raise ValueError(f"PendulumDx(simple=False) takes 5 params (g, m, l, d, b), got {len(self.params)}")
        self.goal_state = torch.tensor([1.0, 0.0, 0.0])
        self.goal_weights = torch.tensor([1.0, 1.0, 0.1])
        self.ctrl_penalty = 0.001
        self.lower, self.upper = -2.0, 2.0
        self.mpc_eps = 1e-3
        self.linesearch_decay = 0.2
        self.max_linesearch_iter = 5

    def mpcb200_params(self):
        if not self.simple:
            g, m, l, d, b = _host_values(self, self.params)
            return (g, m, l, d, b, float(self.max_torque), float(self.dt), 0.0)
        g, m, l = _host_values(self, self.params)
        return (g, m, l, 0.0, float(self.max_torque), float(self.dt), 0.0, 0.0)

    def forward(self, x, u):
        single = x.dim() == 1
        if single:
            x, u = x.unsqueeze(0), u.unsqueeze(0)
        tq = u.clamp(-self.max_torque, self.max_torque)[:, 0]
        c, s, om = x.unbind(1)
        th = torch.atan2(s, c)
        if not self.simple:
            g, m, l, d, b = self.params.to(x, non_blocking=self.params.is_pinned()).unbind()
            om2 = om + self.dt * (3.0 * g / (2.0 * l) * torch.sin(th + b) + 3.0 * tq / (m * l ** 2) - d * th)
            th2 = th + om2 * self.dt
            out = torch.stack((torch.cos(th2), torch.sin(th2), om2), 1)
            return out.squeeze(0) if single else out
        g, m, l = self.params.to(x, non_blocking=self.params.is_pinned()).unbind()
        om2 = om + self.dt * (3.0 * g / (2.0 * l) * s + 3.0 * tq / (m * l ** 2))
        th2 = th + om2 * self.dt
        out = torch.stack((torch.cos(th2), torch.sin(th2), om2), 1)
        return out.squeeze(0) if single else out

    def get_true_obj(self):
        q = torch.cat((self.goal_weights, self.ctrl_penalty * torch.ones(self.n_ctrl)))
        p = torch.cat((-torch.sqrt(self.goal_weights) * self.goal_state, torch.zeros(self.n_ctrl)))
        return q, p


def known_kind(dynamics, n_state, n_ctrl, ref_tensor):
    """(kind, params) if `dynamics` is a known system that can run in the kernels for these shapes / this tensor."""
    kind = getattr(dynamics, "mpcb200_kind", DYN_LINEAR)
    if kind == DYN_LINEAR or not ref_tensor.is_cuda or ref_tensor.dtype not in (torch.float32, torch.float64):
        return DYN_LINEAR, None
    if (n_state, n_ctrl) != (dynamics.n_state, dynamics.n_ctrl):
        return DYN_LINEAR, None
    return kind, tuple(dynamics.mpcb200_params())


def _dyn_array(params):
    return (ctypes.c_double * 8)(*params)


def _check_dyn_shapes(kind, T, what, x, x_shape, u):
    """The kernels index x and u by the system's own (n_state, 1): check the shapes before anything launches."""
    if kind not in DYN_DIMS:
        raise MpcB200Error(f"unknown dynamics kind {kind}")
    n, m = DYN_DIMS[kind]
    if int(T) < 1:
        raise MpcB200Error(f"T must be at least 1, got {T}")
    B = x.shape[-2] if x.dim() >= 2 else -1
    want_x = (B, n) if x_shape == "BN" else (T, B, n)
    if tuple(x.shape) != want_x or B < 1:
        raise MpcB200Error(f"{what}: expected shape {want_x} (n_state = {n}), got {tuple(x.shape)}")
    if tuple(u.shape) != (T, B, m):
        raise MpcB200Error(f"u: expected shape {(T, B, m)} (n_ctrl = {m}), got {tuple(u.shape)}")
    if x.dtype not in (torch.float32, torch.float64):
        raise MpcB200Error(f"unsupported dtype {x.dtype}")
    if u.device != x.device:
        raise MpcB200Error(f"u is on {u.device}, {what} on {x.device}")
    if not x.is_cuda:
        raise MpcB200Error("mpc.pytorch_b200 runs on CUDA tensors only (no CPU fallback)")
    return B, n, m


def dyn_rollout_raw(kind, params, T, x_init, u):
    """x = get_traj(T, u, x_init, dynamics) for a known system, ONE kernel (reference mpc/util.py:102-126)."""
    B, n, m = _check_dyn_shapes(kind, T, "x_init", x_init, "BN", u)
    dtype, dev = x_init.dtype, x_init.device
    x0 = x_init.detach().to(dtype).contiguous()
    u_ = u.detach().to(dtype).contiguous()
    x = torch.empty(T, B, n, dtype=dtype, device=dev)
    fn = _lib.entry("mpcb200_dyn_rollout", dtype)
    with _on_device(dev):
        rc = fn(kind, _dyn_array(params), B, T, ptr(x0), ptr(u_), ptr(x), stream_handle(dev))
    check(rc, "mpcb200_dyn_rollout")
    return x


def dyn_linearize_raw(kind, params, T, x, u):
    """(F[T-1,B,n,n+m], f[T-1,B,n]) = linearisation of a known system along (x, u), ONE kernel
    (reference MPC.linearize_dynamics, mpc/mpc.py:490-601)."""
    B, n, m = _check_dyn_shapes(kind, T, "x", x, "TBN", u)
    dtype, dev = x.dtype, x.device
    x_ = x.detach().to(dtype).contiguous()
    u_ = u.detach().to(dtype).contiguous()
    F = torch.empty(T - 1, B, n, n + m, dtype=dtype, device=dev)
    f = torch.empty(T - 1, B, n, dtype=dtype, device=dev)
    fn = _lib.entry("mpcb200_dyn_linearize", dtype)
    with _on_device(dev):
        rc = fn(kind, _dyn_array(params), B, T, ptr(x_), ptr(u_), ptr(F), ptr(f), stream_handle(dev))
    check(rc, "mpcb200_dyn_linearize")
    return F, f


def dyn_linearize_vjp_raw(kind, params, T, x, u, dF, df):
    """(first, second) [T-1, B, NP]: the vector-Jacobian product of dyn_linearize_raw(kind, params, T, x, u) in the
    system's learnable parameters theta = params[:NP] (DYN_NPARAMS), per (t, b), ONE kernel.  With z = [x; u],
    J = dx'/dz and f = x' - J z: first = sum_r df_r dx'_r/dtheta (J held constant), second = sum_rj (dF_rj - df_r z_j)
    dJ_rj/dtheta; their sum over (t, b) is the gradient of <dF, F> + <df, f>."""
    if kind not in DYN_NPARAMS:
        raise MpcB200Error(f"dyn_linearize_vjp_raw: kind {kind} is not a known system (passthrough kinds have no VJP)")
    n, m = DYN_DIMS[kind]
    B = x.shape[1] if x.dim() == 3 else -1
    dtype, dev = x.dtype, x.device
    for name, t, shape in (("dF", dF, (T - 1, B, n, n + m)), ("df", df, (T - 1, B, n))):
        if tuple(t.shape) != shape:
            raise MpcB200Error(f"{name}: expected shape {shape}, got {tuple(t.shape)}")
        if t.dtype != dtype or t.device != dev:
            raise MpcB200Error(f"{name} is {t.dtype} on {t.device}, x is {dtype} on {dev}")
    _check_dyn_shapes(kind, T, "x", x, "TBN", u)
    NP = DYN_NPARAMS[kind]
    x_, u_, dF_, df_ = (t.detach().contiguous() for t in (x, u.to(dtype), dF, df))
    first = torch.empty(T - 1, B, NP, dtype=dtype, device=dev)
    second = torch.empty(T - 1, B, NP, dtype=dtype, device=dev)
    fn = _lib.entry("mpcb200_dyn_linearize_vjp", dtype)
    with _on_device(dev):
        rc = fn(kind, _dyn_array(params), B, T, ptr(x_), ptr(u_), ptr(dF_), ptr(df_), ptr(first), ptr(second),
                stream_handle(dev))
    check(rc, "mpcb200_dyn_linearize_vjp")
    return first, second


class DynLinearize(torch.autograd.Function):
    """(F, f) = dyn_linearize_raw along detached (x, u), differentiable in the system's `params` tensor: the backward
    is the VJP kernel, summed over (t, b).  One module-level Function (DESIGN.md section 3.2): a class made per call
    would be a new Python type, and a new autograd node type, on every solve.  The forward reads nothing from the
    device: the parameter values are the host numbers the caller took from mpcb200_params()."""

    @staticmethod
    def forward(ctx, params, kind, kparams, T, x, u):
        F, f = dyn_linearize_raw(kind, kparams, T, x, u)
        ctx.save_for_backward(x, u)
        ctx.kind, ctx.kparams, ctx.T = kind, kparams, T
        ctx.p_dtype, ctx.p_device = params.dtype, params.device
        return F, f

    @staticmethod
    def backward(ctx, dF, df):
        x, u = ctx.saved_tensors
        first, second = dyn_linearize_vjp_raw(ctx.kind, ctx.kparams, ctx.T, x, u, dF, df)
        grad = (first + second).sum((0, 1))
        return grad.to(dtype=ctx.p_dtype, device=ctx.p_device), None, None, None, None, None


def linearize_known(dynamics, kind, kparams, T, x, u):
    """(F, f) of the known system `dynamics` (a kind of DYN_KNOWN) along (x, u), as MPC's differentiable
    tail needs it: through DynLinearize when autograd records and dynamics.params requires grad, otherwise one
    dyn_linearize_raw launch and no graph.  x and u are detached either way (no gradient reaches the linearisation
    point)."""
    params = getattr(dynamics, "params", None)
    if torch.is_grad_enabled() and isinstance(params, torch.Tensor) and params.requires_grad:
        return DynLinearize.apply(params, kind, kparams, T, x.detach(), u.detach())
    return dyn_linearize_raw(kind, kparams, T, x, u)
