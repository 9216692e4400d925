"""MPC: the outer iLQR loop around the CUDA LQR step (host side, device-resident state).

Mirrors the reference module ``mpc.MPC`` (mpc/mpc.py:58-337): identical constructor
keywords and defaults (:123-144), ``forward(x_init, cost, dx) -> (x, u, costs)`` (:184, :337),
``QuadCost`` / ``LinDx`` / ``GradMethods`` (:21-33), and the same error behaviour
(asserts, ``sys.exit(-1)`` on un-inferable shapes, printed warnings).

Differences are structural only: the best-iterate bookkeeping (reference :271-285, a Python
loop over the batch with one host sync per element) is a ``torch.where`` on the device and the
stop test costs ONE device->host read per iteration; every LQR step is a single CUDA kernel
(``step.LQRStep``).  Where the dynamics run in the kernels (``LinDx`` or a known system) and the cost
is a ``QuadCost``, the whole loop, bookkeeping and stop test included, runs as one CUDA graph with no
host read (``MPC._ilqr_device``, ``_use_device_loop``), computing bitwise what the host loop computes.
"""
import sys
from collections import namedtuple
from enum import Enum

import torch
from torch.autograd import Function
from torch.nn import Module

from .step import LQRStep

QuadCost = namedtuple("QuadCost", "C c", defaults=(None, None))
LinDx = namedtuple("LinDx", "F f", defaults=(None, None))


class GradMethods(Enum):
    AUTO_DIFF = 1
    FINITE_DIFF = 2
    ANALYTIC = 3
    ANALYTIC_CHECK = 4


def _detach(t):
    if t is None:
        return None
    return t.detach() if t.requires_grad else t


def _mv(A, x):
    return torch.matmul(A, x.unsqueeze(-1)).squeeze(-1)


def _expand_cost(cost, T, n_batch, p):
    """A QuadCost with C [p,p] / [T,p,p] and c [p] / [T,p] expanded to [T,B,p,p] and [T,B,p] (reference
    mpc/mpc.py:205-226); any other cost as it is."""
    if not isinstance(cost, QuadCost):
        return cost
    C, c = cost
    if C.ndimension() == 2:
        C = C.unsqueeze(0).unsqueeze(0).expand(T, n_batch, p, -1)
    elif C.ndimension() == 3:
        C = C.unsqueeze(1).expand(T, n_batch, p, -1)
    if c.ndimension() == 1:
        c = c.unsqueeze(0).unsqueeze(0).expand(T, n_batch, -1)
    elif c.ndimension() == 2:
        c = c.unsqueeze(1).expand(T, n_batch, -1)
    if C.ndimension() != 4 or c.ndimension() != 3:
        print("MPC Error: Unexpected QuadCost shape.")
        sys.exit(-1)
    return QuadCost(C, c)


def get_traj(T, u, x_init, dynamics):
    """Nominal rollout under the true dynamics (reference mpc/util.py:102-126), no graph."""
    with torch.no_grad():
        if isinstance(dynamics, Module):
            from .dynamics import known_kind, dyn_rollout_raw
            kind, kparams = known_kind(dynamics, x_init.shape[1], u.shape[2], x_init)
            if kind:                                          # one kernel instead of T-1 Module calls
                return dyn_rollout_raw(kind, kparams, T, _detach(x_init), _detach(u))
            from . import mlp
            if mlp.on_device(dynamics, x_init.shape[1], u.shape[2], x_init):
                return mlp.rollout_raw(dynamics, T, _detach(x_init), _detach(u))
        xs = [_detach(x_init)]
        if isinstance(dynamics, LinDx):
            F, f = _detach(dynamics.F), _detach(dynamics.f)
            if f is not None and f.nelement() > 0:
                assert f.shape == F.shape[:3]
            if x_init.is_cuda and x_init.dtype in (torch.float32, torch.float64) and F.dtype == x_init.dtype:
                from .step import rollout_raw                 # one kernel instead of T-1 bmm/cat/add launches
                return rollout_raw(x_init.shape[1], u.shape[2], T, _detach(x_init), _detach(u), F, f)
            for t in range(T - 1):
                nx = _mv(F[t], torch.cat((xs[t], u[t]), 1))
                if f is not None and f.nelement() > 0:
                    nx = nx + f[t]
                xs.append(nx)
        else:
            for t in range(T - 1):
                xs.append(dynamics(xs[t], u[t]).detach())
        return torch.stack(xs, 0)


def get_cost(T, u, cost, dynamics=None, x_init=None, x=None):
    """Total trajectory cost (reference mpc/util.py:129-153)."""
    assert x_init is not None or x is not None
    if x is None:
        x = get_traj(T, u, x_init, dynamics)
    tau = torch.cat((x, u), 2)
    if isinstance(cost, QuadCost):
        C, c = _detach(cost.C), _detach(cost.c)
        return (0.5 * (tau * _mv(C, tau)).sum(-1) + (tau * c).sum(-1)).sum(0)
    return torch.stack([cost(tau[t]) for t in range(T)], 0).sum(0)


class SlewRateCost(Module):
    """True cost of the slew-augmented problem (state = [u_{t-1}; x]); reference mpc/mpc.py:36-55."""

    def __init__(self, cost, slew_C, n_state, n_ctrl):
        super().__init__()
        self.cost, self.slew_C, self.n_state, self.n_ctrl = cost, slew_C, n_state, n_ctrl

    def forward(self, tau):
        inner = self.cost(tau[:, self.n_ctrl:])
        return inner + 0.5 * (tau * _mv(self.slew_C[0], tau)).sum(-1)

    def grad_input(self, x, u):
        raise NotImplementedError("Implement grad_input")


class CtrlPassthroughDynamics(Module):
    """Dynamics of the slew-augmented state [u_{t-1}; x] (reference mpc/dynamics.py:133-156).  Wrapping a known
    system (dynamics.CartpoleDx / PendulumDx, either form) it is one too, of kind inner | DYN_CTRL_PASSTHROUGH, so its
    rollout, linearisation and line-search rollout run in the kernels; any other Module keeps the Module path."""

    def __init__(self, dynamics):
        super().__init__()
        self.dynamics = dynamics
        from .dynamics import DYN_CTRL_PASSTHROUGH, DYN_KNOWN
        kind = getattr(dynamics, "mpcb200_kind", None)
        if kind in DYN_KNOWN:
            self.mpcb200_kind = kind | DYN_CTRL_PASSTHROUGH
            self.n_state, self.n_ctrl = dynamics.n_state + dynamics.n_ctrl, dynamics.n_ctrl
            self.mpcb200_params = dynamics.mpcb200_params      # the system's: its params_scope cache applies

    def forward(self, tilde_x, u):
        squeeze = tilde_x.dim() == 1
        if squeeze:
            tilde_x, u = tilde_x.unsqueeze(0), u.unsqueeze(0)
        m = u.size(1)
        nxt = torch.cat((u, self.dynamics(tilde_x[:, m:], u)), 1)
        return nxt.squeeze(0) if squeeze else nxt

    def grad_input(self, x, u):
        raise NotImplementedError("Implement grad_input")


class MPC(Module):
    """A differentiable box-constrained iLQR solver (drop-in for reference ``mpc.MPC``).

        min_{tau={x,u}} sum_t 0.5 tau_t^T C_t tau_t + c_t^T tau_t
            s.t. x_{t+1} = f(x_t, u_t),  x_0 = x_init,  u_lower <= u <= u_upper

    Arguments, defaults and semantics follow reference mpc/mpc.py:77-144 one for one.
    """

    def __init__(self, n_state, n_ctrl, T,
                 u_lower=None, u_upper=None,
                 u_zero_I=None,
                 u_init=None,
                 lqr_iter=10,
                 grad_method=GradMethods.ANALYTIC,
                 delta_u=None,
                 verbose=0,
                 eps=1e-7,
                 back_eps=1e-7,
                 n_batch=None,
                 linesearch_decay=0.2,
                 max_linesearch_iter=10,
                 exit_unconverged=True,
                 detach_unconverged=True,
                 backprop=True,
                 slew_rate_penalty=None,
                 prev_ctrl=None,
                 not_improved_lim=5,
                 best_cost_eps=1e-4):
        super().__init__()
        assert (u_lower is None) == (u_upper is None)
        assert max_linesearch_iter > 0
        self.n_state, self.n_ctrl, self.T = n_state, n_ctrl, T
        self.u_lower = u_lower if isinstance(u_lower, float) else _detach(u_lower)
        self.u_upper = u_upper if isinstance(u_upper, float) else _detach(u_upper)
        self.u_zero_I = _detach(u_zero_I)
        self.u_init = _detach(u_init)
        self.lqr_iter = lqr_iter
        self.grad_method = grad_method
        self.delta_u = delta_u
        self.verbose = verbose
        self.eps = eps
        self.back_eps = back_eps
        self.n_batch = n_batch
        self.linesearch_decay = linesearch_decay
        self.max_linesearch_iter = max_linesearch_iter
        self.exit_unconverged = exit_unconverged
        self.detach_unconverged = detach_unconverged
        self.backprop = backprop
        self.not_improved_lim = not_improved_lim
        self.best_cost_eps = best_cost_eps
        self.slew_rate_penalty = slew_rate_penalty
        self.prev_ctrl = prev_ctrl

    # ------------------------------------------------------------------------------------
    def forward(self, x_init, cost, dx):
        from .dynamics import params_scope
        with params_scope():            # a known system's CUDA parameters are read back once per solve
            return self._forward(x_init, cost, dx)

    def _forward(self, x_init, cost, dx):
        assert isinstance(cost, (QuadCost, Module, Function))
        assert isinstance(dx, (LinDx, Module, Function))
        T, n, m = self.T, self.n_state, self.n_ctrl

        if self.n_batch is not None:
            n_batch = self.n_batch
        elif isinstance(cost, QuadCost) and cost.C.ndimension() == 4:
            n_batch = cost.C.size(1)
        else:
            print("MPC Error: Could not infer batch size, pass in as n_batch")
            sys.exit(-1)

        cost = _expand_cost(cost, T, n_batch, n + m)

        assert x_init.ndimension() == 2 and x_init.size(0) == n_batch

        if self.u_init is None:
            u = torch.zeros(T, n_batch, m, dtype=x_init.dtype, device=x_init.device)
        else:
            u = self.u_init
            if u.ndimension() == 2:
                u = u.unsqueeze(1).expand(T, n_batch, -1).clone()
            u = u.to(dtype=x_init.dtype, device=x_init.device)

        if self.verbose > 0:
            print("Initial mean(cost): {:.4e}".format(
                torch.mean(get_cost(T, u, cost, dx, x_init=x_init)).item()))

        on_device = _use_device_loop(self, x_init, cost, dx, u) or _use_slew_device_loop(self, x_init, cost, dx, u)
        best = self._ilqr_device(x_init, cost, dx, u) if on_device else None
        if best is None:
            best = self._ilqr_host(x_init, cost, dx, u)
        x, u = best["x"], best["u"]
        full_du_norm = best["full_du_norm"]
        self._solve_info = best["info"]           # int32 [iterations, pnqp-unconverged iterations] (control.py)

        if isinstance(dx, LinDx):
            F, f = dx.F, dx.f
        else:
            F, f = self.linearize_dynamics(x, u, dx, diff=True)
        if isinstance(cost, QuadCost):
            C, c = cost.C, cost.c
        else:
            C, c, _ = self.approximate_cost(x, u, cost, diff=True)

        # the only differentiable call: identity forward, KKT-adjoint backward (reference :318-319)
        x, u = self.solve_lqr_subproblem(x_init, C, c, F, f, cost, dx, x, u, no_op_forward=True)

        if self.detach_unconverged:                         # reference :321-334
            if float(full_du_norm.max()) > self.eps:
                if self.exit_unconverged:
                    assert False
                if self.verbose >= 0:
                    print("LQR Warning: All examples did not converge to a fixed point.")
                    print("Detaching and *not* backpropping through the bad examples.")
                keep = (full_du_norm < self.eps).view(1, -1, 1)
                Ix = keep.expand_as(x).to(x.dtype)
                Iu = keep.expand_as(u).to(u.dtype)
                x = x * Ix + x.clone().detach() * (1. - Ix)
                u = u * Iu + u.clone().detach() * (1. - Iu)

        return (x, u, best["costs"])

    # ------------------------------------------------------------------------------------
    def _ilqr_device(self, x_init, cost, dx, u):
        """The iLQR iterations as one library call (mpcb200_ilqr_*): a CUDA graph whose conditional `while` node runs
        rollout, [linearisation,] step, best-iterate tracking and the stop test on the device, with the arithmetic of
        _ilqr_host.  No host read unless pnqp warnings are to be printed.  None when the driver has no conditional
        graph nodes (the caller then runs _ilqr_host)."""
        global _graph_cond_unavailable
        from . import step as _step
        T, m = self.T, self.n_ctrl
        n, x_init, C, c, F, f, dyn = self._device_problem(x_init, cost, dx)
        if dyn is not None and dyn[0] == "mlp":         # a learned model: mpcb200_ilqr_mlp_*
            from .mlp import ilqr_raw
            res = ilqr_raw(dyn[1], n, m, T, x_init, C, c, u, **self._device_options())
        else:
            res = _step.ilqr_raw(n, m, T, x_init, C, c, F, f, u, dyn=dyn, **self._device_options())
        if res is None:
            _graph_cond_unavailable = True
            return None
        self._print_pnqp_warnings(res["info"][1])          # the one host read: iterations with a pnqp warning
        x = res["x"][:, :, m:] if self.slew_rate_penalty is not None else res["x"]
        return {"x": x, "u": res["u"], "costs": res["costs"], "full_du_norm": res["full_du_norm"], "info": res["info"]}

    def _device_problem(self, x_init, cost, dx, T=None):
        """The problem of the device loop, staged once per solve (or episode): (n, x_init, C, c, F, f, dyn).  With a
        slew-rate penalty, the augmented problem over [u_{t-1}; x] (n = n_state + n_ctrl).  dyn = (kind, params) of a
        known system, with F = f = None; ("mlp", Module) for a learned model in the kernels (mlp.on_device; the Module
        a CtrlPassthroughDynamics under a slew-rate penalty), F = f = None; None for LinDx.  T: the length of C's time
        axis when it is not the solve's
        (a time-varying episode's, control.receding_horizon)."""
        n, m = self.n_state, self.n_ctrl
        C, c = cost.C, cost.c
        F, f = (dx.F, dx.f) if isinstance(dx, LinDx) else (None, None)
        if self.slew_rate_penalty is not None:
            _, C, c, F, f, _, x_init = self._slew_augment(x_init, C, c, F, f, T=T)
            if not isinstance(dx, LinDx):
                dx = CtrlPassthroughDynamics(dx)
            n = n + m
        if isinstance(dx, LinDx):
            dyn = None
        else:
            from .dynamics import known_kind
            from .mlp import on_device
            F = f = None
            dyn = ("mlp", dx) if on_device(dx, n, m, x_init) else known_kind(dx, n, m, x_init)
        return n, x_init, C, c, F, f, dyn

    def _device_options(self):
        """The solver options step.ilqr_raw / step.episode_raw take."""
        return dict(u_lower=self.u_lower, u_upper=self.u_upper, u_zero_I=self.u_zero_I, delta_u=self.delta_u,
                    linesearch_decay=self.linesearch_decay, max_linesearch_iter=self.max_linesearch_iter,
                    lqr_iter=self.lqr_iter, not_improved_lim=self.not_improved_lim, eps=self.eps,
                    best_cost_eps=self.best_cost_eps)

    def _print_pnqp_warnings(self, n_unconverged):
        """The pnqp warnings of a device-side solve: one per iteration counted in `n_unconverged` (a device scalar,
        read only when they are printed)."""
        if self.verbose >= 0 and self.u_lower is not None:
            for _ in range(int(n_unconverged)):
                print("[WARNING] pnqp warning: Did not converge")   # reference pnqp.py:81

    def _ilqr_host(self, x_init, cost, dx, u):
        """The iLQR iterations from Python: one host read per iteration for the stop test."""
        from .step import _host_reads
        T = self.T
        best = None
        n_not_improved = 0
        n_iter = n_unconverged = 0
        _host_reads.n_warned = 0                        # pnqp warnings LQRStep prints itself (verbose > 0)
        for i in range(self.lqr_iter):
            u = _detach(u)
            x = get_traj(T, u, x_init=x_init, dynamics=dx)
            if isinstance(dx, LinDx):
                F, f = dx.F, dx.f
            else:
                F, f = self.linearize_dynamics(x, u, dx, diff=False)
            if isinstance(cost, QuadCost):
                C, c = cost.C, cost.c
            else:
                C, c, _ = self.approximate_cost(x, u, cost, diff=False)

            defer = {} if self.verbose <= 0 else None       # step counters stay on the device unless they are printed
            x, u, n_total_qp_iter, costs, full_du_norm, mean_alphas = \
                self.solve_lqr_subproblem(x_init, C, c, F, f, cost, dx, x, u, _defer_host=defer)
            n_not_improved += 1
            assert x.ndimension() == 3 and u.ndimension() == 3

            # best-iterate tracking on the device (reference :271-285 semantics per element)
            if best is None:
                best = {"x": x, "u": u, "costs": costs, "full_du_norm": full_du_norm}
                flags = [full_du_norm.max(), torch.zeros_like(full_du_norm[0])]
            else:
                better = costs <= best["costs"] + self.best_cost_eps
                sel = better.view(1, -1, 1)
                best = {"x": torch.where(sel, x, best["x"]),
                        "u": torch.where(sel, u, best["u"]),
                        "costs": torch.where(better, costs, best["costs"]),
                        "full_du_norm": torch.where(better, full_du_norm, best["full_du_norm"])}
                flags = [full_du_norm.max(), better.any().to(full_du_norm.dtype)]
            if defer:
                flags.append(defer["unconverged"].to(full_du_norm.dtype))
            vals = torch.stack(flags).tolist()              # the one host sync of this iteration
            max_du, any_better = vals[0], vals[1]
            n_iter += 1
            n_unconverged += 1 if defer and vals[2] else 0
            if defer and vals[2] and self.verbose >= 0:
                print("[WARNING] pnqp warning: Did not converge")   # reference pnqp.py:81
            if any_better:
                n_not_improved = 0

            if self.verbose > 0:
                _table_log("lqr", (
                    ("iter", i),
                    ("mean(cost)", torch.mean(best["costs"]).item(), "{:.4e}"),
                    ("||full_du||_max", max_du, "{:.2e}"),
                    ("mean(alphas)", mean_alphas.item(), "{:.2e}"),
                    ("total_qp_iters", n_total_qp_iter),
                ))

            if max_du < self.eps or n_not_improved > self.not_improved_lim:   # reference :299-301
                break

        if best is not None:
            best["info"] = torch.tensor([n_iter, n_unconverged + _host_reads.n_warned], dtype=torch.int32)
        return best

    # ------------------------------------------------------------------------------------
    def solve_lqr_subproblem(self, x_init, C, c, F, f, cost, dynamics, x, u, no_op_forward=False,
                             _defer_host=None):
        from .step import _host_reads
        _host_reads.defer = _defer_host
        try:
            return self._solve_lqr_subproblem(x_init, C, c, F, f, cost, dynamics, x, u, no_op_forward)
        finally:
            _host_reads.defer = None

    def _solve_lqr_subproblem(self, x_init, C, c, F, f, cost, dynamics, x, u, no_op_forward=False):
        n, m, T = self.n_state, self.n_ctrl, self.T
        common = dict(T=T, u_lower=self.u_lower, u_upper=self.u_upper, u_zero_I=self.u_zero_I,
                      delta_u=self.delta_u, linesearch_decay=self.linesearch_decay,
                      max_linesearch_iter=self.max_linesearch_iter, delta_space=True,
                      back_eps=self.back_eps, no_op_forward=no_op_forward,
                      verbose=self.verbose)
        if self.slew_rate_penalty is None or isinstance(cost, Module):     # reference :341-361
            _lqr = LQRStep(n_state=n, n_ctrl=m, true_cost=cost, true_dynamics=dynamics,
                           current_x=x, current_u=u, **common)
            e = torch.empty(0, dtype=x_init.dtype, device=x_init.device)
            return _lqr(x_init, C, c, F, f if f is not None else e)

        # ---- slew-rate penalty: augment the state with the previous control (reference :362-445)
        n2 = n + m
        slew_C, C2, c2, F2, f2, prev_u, x_init2 = self._slew_augment(x_init, C, c, F, f)
        x2 = torch.cat((torch.cat((prev_u, _detach(u)[:-1])), x), 2)
        dyn2 = None if isinstance(dynamics, LinDx) else CtrlPassthroughDynamics(dynamics)
        if isinstance(dynamics, LinDx):
            dyn2 = LinDx(F2, f2 if f2.nelement() > 0 else None)
        true_cost2 = QuadCost(C2, c2) if isinstance(cost, QuadCost) else \
            SlewRateCost(cost, slew_C, n, m)
        _lqr = LQRStep(n_state=n2, n_ctrl=m, true_cost=true_cost2, true_dynamics=dyn2,
                       current_x=x2, current_u=u, **common)
        xo, *rest = _lqr(x_init2, C2, c2, F2, f2)
        return [xo[:, :, m:]] + list(rest)

    def _slew_augment(self, x_init, C, c, F, f, T=None):
        """The slew-rate augmented problem over the state [u_{t-1}; x] (reference :362-445): (slew_C, C2, c2, F2, f2,
        prev_u[1,B,m], x_init2).  F2 = [[0, 0, I], [0, F]] and f2 = [0; f] (empty without f); both None without F
        (a known system, which the kernels linearise in augmented form).  Differentiable in C, c, F, f and x_init.
        T: C's time axis when it is not the solve's (a time-varying episode's); each slice is augmented alike."""
        n, m = self.n_state, self.n_ctrl
        T = self.T if T is None else T
        B = C.size(1)
        n2, p2 = n + m, n + 2 * m
        kw = dict(dtype=C.dtype, device=C.device)
        gI = self.slew_rate_penalty * torch.eye(m, **kw)
        slew_C = torch.zeros(T, B, p2, p2, **kw)
        slew_C[:, :, :m, :m] = gI
        slew_C[:, :, -m:, :m] = -gI
        slew_C[:, :, :m, -m:] = -gI
        slew_C[:, :, -m:, -m:] = gI
        C2 = slew_C.clone()
        C2[:, :, m:, m:] += C
        c2 = torch.cat((torch.zeros(T, B, m, **kw), c), 2)
        F2 = f2 = None
        if F is not None:
            Fu = torch.zeros(F.shape[0], B, m, p2, **kw)
            Fu[:, :, :, n2:] = torch.eye(m, **kw)
            Fx = torch.cat((torch.zeros(F.shape[0], B, n, m, **kw), F), 3)
            F2 = torch.cat((Fu, Fx), 2)
            if f is not None and f.nelement() > 0:
                f2 = torch.cat((torch.zeros(f.shape[0], B, m, **kw), f), 2)
            else:
                f2 = torch.empty(0, **kw)
        if self.prev_ctrl is not None:
            prev_u = self.prev_ctrl
            while prev_u.ndimension() < 3:
                prev_u = prev_u.unsqueeze(0)
            prev_u = prev_u.detach().to(**kw)
            if prev_u.size(1) != B:
                prev_u = prev_u.expand(1, B, m)
        else:
            prev_u = torch.zeros(1, B, m, **kw)
        x_init2 = torch.cat((prev_u[0], x_init), 1)
        return slew_C, C2, c2, F2, f2, prev_u, x_init2

    # ------------------------------------------------------------------------------------
    def approximate_cost(self, x, u, Cf, diff=True):
        """Second-order expansion of a Module cost around (x,u) (reference :447-487)."""
        if self.slew_rate_penalty is not None:
            print("\nMPC Error: Using a non-convex cost with a slew rate penalty is not yet implemented.\n"
                  "The current implementation does not correctly do a line search.\n"
                  "More details: https://github.com/locuslab/mpc.pytorch/issues/12\n")
            sys.exit(-1)
        T, B = x.shape[0], x.shape[1]
        with torch.enable_grad():
            tau = torch.cat((x, u), dim=2).detach().reshape(T * B, -1).requires_grad_(True)
            costs = Cf(tau)
            grad = torch.autograd.grad(costs.sum(), tau, create_graph=True)[0]
            rows = [torch.autograd.grad(grad[:, i].sum(), tau, retain_graph=True,
                                        create_graph=diff)[0] for i in range(tau.shape[1])]
            H = torch.stack(rows, dim=-1)
            lin = grad - _mv(H, tau)
        p = tau.shape[1]
        H, lin, costs = H.view(T, B, p, p), lin.view(T, B, p), costs.view(T, B)
        if not diff:
            return H.detach(), lin.detach(), costs.detach()
        return H, lin, costs

    def _kernel_linearization(self, dynamics, x, diff):
        """(kind, params) when linearize_dynamics runs in the kernels, else (DYN_LINEAR, None): a known system under
        ANALYTIC or AUTO_DIFF at its own (n, m) on CUDA float32 / float64 tensors (dynamics.known_kind).  With diff,
        only a system itself, not a passthrough kind: the VJP kernel differentiates the systems' own parameters."""
        from .dynamics import DYN_CTRL_PASSTHROUGH, DYN_LINEAR, known_kind
        if self.grad_method not in (GradMethods.ANALYTIC, GradMethods.AUTO_DIFF):
            return DYN_LINEAR, None
        kind, kparams = known_kind(dynamics, self.n_state, self.n_ctrl, x)
        if diff and kind & DYN_CTRL_PASSTHROUGH:
            return DYN_LINEAR, None
        return kind, kparams

    def _mlp_on_device(self, dynamics, x):
        """Whether a learned model's network runs in the kernels here (mlp.on_device), under ANALYTIC or AUTO_DIFF."""
        from .mlp import on_device
        return self.grad_method in (GradMethods.ANALYTIC, GradMethods.AUTO_DIFF) and \
            on_device(dynamics, self.n_state, self.n_ctrl, x)

    def linearize_dynamics(self, x, u, dynamics, diff):
        """First-order expansion x' ~ F [x;u] + f of Module dynamics (reference :490-601),
        evaluated for all T-1 steps and the whole batch at once."""
        T, n, m = self.T, self.n_state, self.n_ctrl
        B = x.shape[1]
        kind, kparams = self._kernel_linearization(dynamics, x, diff)
        if not kind and self._mlp_on_device(dynamics, x):
            from .mlp import linearize_diff, linearize_raw
            if not diff:       # a network's exact Jacobians, one kernel
                return linearize_raw(dynamics, T, x.detach(), u.detach())
            Ff = linearize_diff(dynamics, T, x, u)     # differentiable in the weights through the VJP kernel
            if Ff is not None:
                return Ff
        if kind:               # exact Jacobians of a known system by forward-mode duals, one kernel
            from .dynamics import dyn_linearize_raw, linearize_known
            if diff:           # differentiable in the system's parameters through the VJP kernel
                return linearize_known(dynamics, kind, kparams, T, x, u)
            return dyn_linearize_raw(kind, kparams, T, x, u)
        xs = x[:-1].detach().reshape(-1, n)
        us = u[:-1].detach().reshape(-1, m)
        if self.grad_method == GradMethods.ANALYTIC:
            ctx = torch.enable_grad() if diff else torch.no_grad()
            with ctx:
                new_x = dynamics(xs, us)
                R, S = dynamics.grad_input(xs, us)
                f = new_x - _mv(R, xs) - _mv(S, us)
        elif self.grad_method in (GradMethods.AUTO_DIFF, GradMethods.ANALYTIC_CHECK):
            assert self.grad_method != GradMethods.ANALYTIC_CHECK, "ANALYTIC_CHECK is not maintained"
            with torch.enable_grad():
                xs_g, us_g = xs.requires_grad_(True), us.requires_grad_(True)
                new_x = dynamics(xs_g, us_g)
                Rr, Sr = [], []
                for jj in range(n):           # rows of the Jacobian; batch elements are independent
                    Rj, Sj = torch.autograd.grad(new_x[:, jj].sum(), [xs_g, us_g],
                                                 retain_graph=True, create_graph=diff)
                    Rr.append(Rj)
                    Sr.append(Sj)
                R, S = torch.stack(Rr, 1), torch.stack(Sr, 1)
                f = new_x - _mv(R, xs_g) - _mv(S, us_g)
        elif self.grad_method == GradMethods.FINITE_DIFF:
            h = 1e-4
            with torch.no_grad():
                new_x = dynamics(xs, us)
                cols = []
                for i in range(n):
                    e = torch.zeros_like(xs)
                    e[:, i] = h
                    cols.append((dynamics(xs + e, us) - dynamics(xs - e, us)) / (2 * h))
                R = torch.stack(cols, 2)
                cols = []
                for i in range(m):
                    e = torch.zeros_like(us)
                    e[:, i] = h
                    cols.append((dynamics(xs, us + e) - dynamics(xs, us - e)) / (2 * h))
                S = torch.stack(cols, 2)
                f = new_x - _mv(R, xs) - _mv(S, us)
        else:
            assert False
        F = torch.cat((R, S), 2).view(T - 1, B, n, n + m)
        f = f.view(T - 1, B, n)
        if not diff:
            F, f = F.detach(), f.detach()
        return F, f


_graph_cond_unavailable = False     # set once a driver without conditional graph nodes refused the device loop


def _use_device_loop(mpc, x_init, cost, dx, u):
    """Whether MPC.forward runs its iLQR iterations as one device-side graph (MPC._ilqr_device) rather than from
    Python (MPC._ilqr_host).  Decided on what the call shows without reading the device: the results are the same
    either way, so there is no user option.  Taken for CUDA float32/float64 tensors of one dtype, a QuadCost, LinDx
    dynamics, or a known system or a learned model in the kernels (mlp.on_device) linearised by ANALYTIC / AUTO_DIFF,
    no slew-rate penalty, verbose <= 0, lqr_iter >= 1, T >= 2 and a shape the step kernels take (an exact or
    zero-padded instance, or the large-shape kernels for LinDx)."""
    return mpc.slew_rate_penalty is None and _device_loop_takes(mpc, x_init, cost, dx, u, slew=False)


def _use_slew_device_loop(mpc, x_init, cost, dx, u):
    """_use_device_loop for a solve with a slew-rate penalty: the same conditions on the augmented problem over
    [u_{t-1}; x] (MPC._slew_augment).  LinDx runs it at the (n+m, m) instance _pick_instance gives (exact, padded or
    large); a known system runs its passthrough kind's dynamics-only instance.  prev_ctrl must be absent or a tensor on
    the solve's device."""
    if mpc.slew_rate_penalty is None:
        return False
    prev = mpc.prev_ctrl
    if prev is not None and (not isinstance(prev, torch.Tensor) or prev.device != x_init.device):
        return False
    return _device_loop_takes(mpc, x_init, cost, dx, u, slew=True)


def _device_loop_takes(mpc, x_init, cost, dx, u, slew):
    """The conditions the two device-loop predicates share; `slew`: on the augmented problem."""
    from .dynamics import DYN_CTRL_PASSTHROUGH, DYN_LINEAR
    from .step import _pick_instance
    from ._lib import MpcB200Error
    if _graph_cond_unavailable or mpc.verbose > 0 or mpc.lqr_iter < 1:
        return False
    if not isinstance(cost, QuadCost) or mpc.T < 2:
        return False
    dtype, dev = x_init.dtype, x_init.device
    if dtype not in (torch.float32, torch.float64) or not x_init.is_cuda:
        return False
    n, m = mpc.n_state, mpc.n_ctrl
    kind = DYN_LINEAR
    same = [cost.C, cost.c, u]
    if isinstance(dx, LinDx):
        if dx.F is None:
            return False
        same.append(dx.F)
        if dx.f is not None and dx.f.nelement() > 0:
            same.append(dx.f)
        known = False
    elif isinstance(dx, Module) and getattr(dx, "mpcb200_kind", DYN_LINEAR) != DYN_LINEAR:
        if mpc.grad_method not in (GradMethods.ANALYTIC, GradMethods.AUTO_DIFF):
            return False
        if (n, m) != (dx.n_state, dx.n_ctrl):
            return False
        kind = dx.mpcb200_kind | (DYN_CTRL_PASSTHROUGH if slew else 0)
        known = True
    elif mpc._mlp_on_device(dx, x_init):              # a learned model: the network's kernels around the step
        known = False
    else:
        return False
    same += [b for b in (mpc.u_lower, mpc.u_upper) if isinstance(b, torch.Tensor)]
    if any(not isinstance(t, torch.Tensor) or t.dtype != dtype or t.device != dev for t in same):
        return False
    if isinstance(mpc.u_zero_I, torch.Tensor) and mpc.u_zero_I.device != dev:
        return False
    n_aug = n + m if slew else n
    try:
        N, M = _pick_instance(n_aug, m, x_init.element_size(), kind)
    except MpcB200Error:
        return False
    return not known or (N, M) == (n_aug, m)


_seen_tables = []


def _table_log(tag, cols):
    """Markdown-ish iteration table (reference mpc/util.py:77-99)."""
    def row(cells):
        print("| " + " | ".join(cells) + " |")
    if tag not in _seen_tables:
        row([str(col[0]) for col in cols])
        _seen_tables.append(tag)
    row([col[2].format(col[1]) if len(col) == 3 else str(col[1]) for col in cols])
