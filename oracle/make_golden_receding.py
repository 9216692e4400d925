#!/usr/bin/env python3
"""Fixtures for receding-horizon episodes, from the REAL reference's own notebook loop.

Run with a checkout of locuslab/mpc.pytorch:   MPC_REFERENCE=<checkout> python oracle/make_golden_receding.py
Runs the control loop of the reference's cartpole and pendulum notebooks (examples/*.ipynb) on the unmodified
reference, CPU, float64: solve MPC(..., u_init=u_init, lqr_iter, eps, AUTO_DIFF, exit_unconverged=False,
detach_unconverged=False), apply nominal_actions[0], shift u_init = cat(nominal_actions[1:], 0) with
u_init[-2] = u_init[-3], step the plant.  Cases:
  cartpole       the cartpole notebook at B=4, T=25, 15 control steps;
  pendulum       the pendulum notebook (PendulumDx(params=(10, 1, 1), simple=True), swing-up cost), B=4, T=20;
  linear         a bounded LinDx loop (n=4, m=2, +-0.5, lqr_iter=10), plant F_0 tau + f_0 by util.bmv;
  pendulum_slew  the pendulum loop with a slew-rate penalty, prev_ctrl = the last applied control.
Stores the inputs, x, u, each solve's costs and iteration count as tests/golden/receding_<case>_f64.npz.  Round-off
guard: every episode is rerun from x_init perturbed by 1e-12 relative; its iteration counts must be identical and its
x, u within GUARD, so that no stored stop decision is decided by round-off.  GUARD is 1e-6, not tighter: solves that
stop at eps = 1e-2 amplify the perturbation over the closed loop, to up to 2e-7 in the pendulum episodes (with the
same iteration counts), which is still 50 times below the 1e-5 the fixtures are compared at.  Only numbers are stored.
"""
import contextlib
import io
import math
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from make_golden import load_reference, npz                    # noqa: E402
from make_golden_nn import load_ref_env                        # noqa: E402

B, STEPS = 4, 15
GUARD = 1e-6


def _uniform(shape, low, high):
    return torch.rand(shape) * (high - low) + low


def episode(rmpc, make, x0, cost, plant, steps, slew=False):
    """The notebooks' loop; returns x, u, costs, iteration counts."""
    iters = []
    real = rmpc.MPC.solve_lqr_subproblem

    def count(self, *a, **k):
        if not k.get("no_op_forward", False):
            iters[-1] += 1
        return real(self, *a, **k)
    rmpc.MPC.solve_lqr_subproblem = count
    try:
        x, u_init, prev = x0, None, None
        xs, us, costs = [x0], [], []
        for _ in range(steps):
            iters.append(0)
            with contextlib.redirect_stdout(io.StringIO()):
                _, actions, objs = make(u_init, prev)(x, cost, plant if not isinstance(plant, tuple) else plant[0])
            nxt = actions[0]
            u_init = torch.cat((actions[1:], torch.zeros(1, x.shape[0], actions.shape[2])), dim=0)
            u_init[-2] = u_init[-3]
            x = plant[1](x, nxt) if isinstance(plant, tuple) else plant(x, nxt)
            if slew:
                prev = nxt
            xs.append(x.detach())
            us.append(nxt.detach())
            costs.append(objs.detach())
    finally:
        rmpc.MPC.solve_lqr_subproblem = real
    return torch.stack(xs), torch.stack(us), torch.stack(costs), np.array(iters, dtype=np.int64)


def guarded(rmpc, make, x0, cost, plant, steps, slew=False):
    out = episode(rmpc, make, x0, cost, plant, steps, slew)
    again = episode(rmpc, make, x0 * (1 + 1e-12), cost, plant, steps, slew)
    assert np.array_equal(out[3], again[3]), (out[3], again[3])
    for a, b in zip(out[:2], again[:2]):
        assert float((a - b).abs().max()) < GUARD, float((a - b).abs().max())
    return out


def main():
    rmpc, _, _, rutil = load_reference()
    torch.set_default_dtype(torch.float64)
    GM = rmpc.GradMethods.AUTO_DIFF
    cp, pd = load_ref_env("cartpole"), load_ref_env("pendulum")

    def notebook_mpc(dx, T, **kw):
        return lambda u_init, prev: rmpc.MPC(
            dx.n_state, dx.n_ctrl, T, u_init=u_init, u_lower=dx.lower, u_upper=dx.upper, lqr_iter=50, verbose=0,
            exit_unconverged=False, detach_unconverged=False, linesearch_decay=dx.linesearch_decay,
            max_linesearch_iter=dx.max_linesearch_iter, grad_method=GM, eps=1e-2, prev_ctrl=prev, **kw)

    def common(dx, T):
        return dict(T=np.int64(T), n_steps=np.int64(STEPS), lqr_iter=np.int64(50), eps=np.float64(1e-2),
                    decay=np.float64(dx.linesearch_decay), ls_iter=np.int64(dx.max_linesearch_iter))

    # cartpole notebook
    dx = cp.CartpoleDx()
    T = 25
    torch.manual_seed(0)
    th, thdot = _uniform(B, -2 * math.pi, 2 * math.pi), _uniform(B, -.5, .5)
    x, xdot = _uniform(B, -0.5, 0.5), _uniform(B, -0.5, 0.5)
    x0 = torch.stack((x, xdot, torch.cos(th), torch.sin(th), thdot), dim=1)
    q, p = dx.get_true_obj()
    Q = torch.diag(q).unsqueeze(0).unsqueeze(0).repeat(T, B, 1, 1)
    pp = p.unsqueeze(0).repeat(T, B, 1)
    xs, us, cs, it = guarded(rmpc, notebook_mpc(dx, T), x0, rmpc.QuadCost(Q, pp), dx, STEPS)
    print("cartpole iterations", it.tolist())
    npz("receding_cartpole_f64", params=dx.params, x_init=x0, C=Q, c=pp, x=xs, u=us, costs=cs, iters=it,
        **common(dx, T))

    # pendulum notebook (swing-up), and with a slew-rate penalty
    dx = pd.PendulumDx(torch.tensor((10., 1., 1.)), simple=True)
    T = 20
    torch.manual_seed(0)
    th, thdot = _uniform(B, -(1 / 2) * math.pi, (1 / 2) * math.pi), _uniform(B, -1., 1.)
    x0 = torch.stack((torch.cos(th), torch.sin(th), thdot), dim=1)
    goal_weights, goal_state = torch.tensor((1., 1., 0.1)), torch.tensor((1., 0., 0.))
    q = torch.cat((goal_weights, 0.001 * torch.ones(dx.n_ctrl)))
    p = torch.cat((-torch.sqrt(goal_weights) * goal_state, torch.zeros(dx.n_ctrl)))
    Q = torch.diag(q).unsqueeze(0).unsqueeze(0).repeat(T, B, 1, 1)
    pp = p.unsqueeze(0).repeat(T, B, 1)
    xs, us, cs, it = guarded(rmpc, notebook_mpc(dx, T), x0, rmpc.QuadCost(Q, pp), dx, STEPS)
    print("pendulum iterations", it.tolist())
    npz("receding_pendulum_f64", params=dx.params, x_init=x0, C=Q, c=pp, x=xs, u=us, costs=cs, iters=it,
        **common(dx, T))
    penalty = 0.1
    xs, us, cs, it = guarded(rmpc, notebook_mpc(dx, T, slew_rate_penalty=penalty), x0, rmpc.QuadCost(Q, pp), dx,
                             STEPS, slew=True)
    print("pendulum slew iterations", it.tolist())
    npz("receding_pendulum_slew_f64", params=dx.params, x_init=x0, C=Q, c=pp, x=xs, u=us, costs=cs, iters=it,
        penalty=np.float64(penalty), **common(dx, T))

    # bounded LinDx; the plant is the model's t = 0 slice
    n, m, T, bound = 4, 2, 10, 0.5
    g = torch.Generator().manual_seed(5)
    L = torch.randn(T, B, n + m, n + m, generator=g) / (n + m) ** 0.5
    C = L @ L.transpose(-1, -2) + torch.eye(n + m)
    c = torch.randn(T, B, n + m, generator=g)
    A = 0.9 * torch.eye(n) + 0.2 * torch.randn(B, n, n, generator=g) / n ** 0.5
    F = torch.cat((A, torch.randn(B, n, m, generator=g) / n ** 0.5), -1).unsqueeze(0).repeat(T - 1, 1, 1, 1)
    f = 0.1 * torch.randn(T - 1, B, n, generator=g)
    x0 = 2.0 * torch.randn(B, n, generator=g)

    def make(u_init, prev):
        return rmpc.MPC(n, m, T, u_init=u_init, u_lower=-bound, u_upper=bound, lqr_iter=10, verbose=0,
                        exit_unconverged=False, detach_unconverged=False)

    def plant(x, u):
        return rutil.bmv(F[0], torch.cat((x, u), 1)) + f[0]
    xs, us, cs, it = guarded(rmpc, make, x0, rmpc.QuadCost(C, c), (rmpc.LinDx(F, f), plant), STEPS)
    print("linear iterations", it.tolist(), "on the bounds", int((us.abs() == bound).sum()), "of", us.numel())
    npz("receding_linear_f64", x_init=x0, C=C, c=c, F=F, f=f, x=xs, u=us, costs=cs, iters=it, T=np.int64(T),
        n_steps=np.int64(STEPS), lqr_iter=np.int64(10), eps=np.float64(1e-7), decay=np.float64(0.2),
        ls_iter=np.int64(10), bound=np.float64(bound))


if __name__ == "__main__":
    main()
