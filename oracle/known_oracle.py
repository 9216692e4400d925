"""Float64 oracle of MPC.forward's iLQR loop and of the receding-horizon episode with a known system (CartpoleDx,
PendulumDx, PendulumDx(simple=False)) as the true dynamics: the reference's loop (mpc/mpc.py:244-301) with the
Module in its rollout (mpc/util.py:102-126), its AUTO_DIFF linearisation (mpc/mpc.py:538-592) and its line search
(mpc/lqr_step.py:224-225).

A known system is `step(x, u, theta)`, a CPU torch forward of states [B, n] and controls [B, m] with per-problem
parameters theta [B, NP] (gpu_harness.episode_known_step makes one from a module).  The loop is lqr_oracle.ilqr_loop,
which mlp_oracle.ilqr runs too; the Jacobians are autograd's, n grad calls per iteration over every (t, b) at once.

n_prev = m: the slew-rate form of the reference's CtrlPassthroughDynamics, state [u_{t-1}; x] stepped as
[u; step(x, u)] with the control as given (before the system's clamp), which is what the passthrough kinds of the
kernels step (DESIGN.md section 3.3).  Its cost is slew_oracle.slew_augment's."""
import torch

from . import lqr_oracle as lo
from .lqr_oracle import Episode, shift_warm_start
from .plant_oracle import plant_step
from .slew_oracle import slew_augment
from .window_oracle import _plant_at, _window


def passthrough(step, n_prev):
    """step of the augmented state [u_{t-1}; x]: [u; step(x, u, theta)] (n_prev = 0: step itself)."""
    if not n_prev:
        return step
    return lambda x, u, theta: torch.cat((u, step(x[:, n_prev:], u, theta)), 1)


def rollout(step, theta, x_init, u):
    """get_traj: x [T, B, n] from x_init under u [T, B, m]."""
    xs = [x_init]
    for t in range(u.shape[0] - 1):
        xs.append(step(xs[t], u[t], theta))
    return torch.stack(xs)


def linearize(step, theta, x, u):
    """F = [R S] [T-1, B, n, n+m] and f = x' - R x - S u [T-1, B, n] at (x[:-1], u[:-1]) by autograd: one grad call
    per state row over every (t, b) item at once."""
    T, B, n = x.shape
    m = u.shape[2]
    xs = x[:-1].reshape(-1, n).detach().requires_grad_(True)
    us = u[:-1].reshape(-1, m).detach().requires_grad_(True)
    nx = step(xs, us, theta.repeat(T - 1, 1))
    J = torch.stack([torch.cat(torch.autograd.grad(nx[:, r].sum(), (xs, us), retain_graph=r < n - 1), 1)
                     for r in range(n)], 1)
    f = nx.detach() - lo._mv(J, torch.cat((xs, us), 1).detach())
    return J.view(T - 1, B, n, n + m), f.view(T - 1, B, n)


def ilqr(n, m, T, x_init, C, c, step, theta, u_init=None, lqr_iter=10, eps=1e-7, not_improved_lim=5,
         best_cost_eps=1e-4, n_prev=0, **step_kw):
    """MPC.forward's iterations with QuadCost(C, c) and the known system `step` (parameters theta [B, NP]) as the true
    dynamics.  n is the (augmented) state count: with n_prev = m, x_init, C and c are the slew-rate problem's over
    [u_{t-1}; x] (slew_problem).  step_kw: lqr_step_forward's options (bounds, u_zero_I, delta_u, line search,
    coupled).  Returns (x, u, costs, iterations)."""
    dyn = passthrough(step, n_prev)
    return lo.ilqr_loop(n, m, T, x_init, C, c, lambda u: rollout(dyn, theta, x_init, u),
                        lambda x, u: linearize(dyn, theta, x, u), lambda x, u: dyn(x, u, theta), u_init=u_init,
                        lqr_iter=lqr_iter, eps=eps, not_improved_lim=not_improved_lim, best_cost_eps=best_cost_eps,
                        **step_kw)


def slew_problem(n, m, penalty, C, c, x_init, prev_ctrl=None):
    """(x_init~, C~, c~) of MPC(slew_rate_penalty=penalty, prev_ctrl=prev_ctrl): [u_{-1}; x_init] with u_{-1} =
    prev_ctrl or 0, and slew_augment's cost."""
    C2, c2, _, _ = slew_augment(n, m, penalty, C, c)
    prev = torch.zeros(x_init.shape[0], m, dtype=x_init.dtype) if prev_ctrl is None else prev_ctrl
    return torch.cat((prev, x_init), 1), C2, c2


def episode(n, m, T, n_steps, x_init, C, c, step, theta, plant=None, w=None, u_init=None, u_lower=None,
            u_upper=None, slew_rate_penalty=None, prev_ctrl=None, window=False, **kw):
    """The notebooks' loop on ilqr with the known system as the model: solve from x_k (under a slew-rate penalty from
    [u_{k-1}; x_k] on slew_problem's cost, u_{-1} = prev_ctrl or 0) with u_init = the warm start, apply u_k =
    plan_u[0], x_{k+1} = plant(x_k, u_k) + w[k], shift the warm start.  plant: None (the model steps), ("step", f,
    theta_p) or ("lin", F_p, f_p) as plant_oracle takes them; w [n_steps, B, n] or None.  window: C, c and tensor
    bounds lie on the episode's time axis of n_steps + T - 1 slices and control step k solves on slices k .. k+T-1
    (a LinDx plant steps its slice k), as window_oracle slices them.  kw: ilqr's other options.  Returns an Episode
    (plan_x augmented under a penalty)."""
    B = x_init.shape[0]
    L = C.shape[0]
    slew = slew_rate_penalty is not None
    ws = torch.zeros(T, B, m, dtype=C.dtype) if u_init is None else u_init
    prev = torch.zeros(B, m, dtype=C.dtype) if prev_ctrl is None else prev_ctrl.detach()
    x = x_init
    xs, us, costs, iters, plan_x, plan_u = [x_init], [], [], [], [], []
    for k in range(n_steps):
        at = (lambda t: _window(T, L, k, t)) if window else (lambda t: t)
        Ck, ck = at(C), at(c)
        if slew:
            xk, Ck, ck = slew_problem(n, m, slew_rate_penalty, Ck, ck, x, prev)
        else:
            xk = x
        bx, bu, bc, it = ilqr(n + m if slew else n, m, T, xk, Ck, ck, step, theta, u_init=ws,
                              u_lower=at(u_lower), u_upper=at(u_upper), n_prev=m if slew else 0, **kw)
        pk = _plant_at(plant, k) if window else plant
        x = step(x, bu[0], theta) if pk is None else plant_step(pk, None, None, x, bu[0])
        if w is not None:
            x = x + w[k]
        ws = shift_warm_start(bu)
        prev = bu[0]
        xs.append(x)
        us.append(bu[0])
        costs.append(bc)
        iters.append(it)
        plan_x.append(bx)
        plan_u.append(bu)
    return Episode(torch.stack(xs), torch.stack(us), torch.stack(costs), iters, torch.stack(plan_x),
                   torch.stack(plan_u), ws)
