#!/usr/bin/env python3
"""Fixtures for differentiable receding-horizon episodes under a slew-rate penalty, from the REAL reference's own
notebook loop under autograd.

Run with a checkout of locuslab/mpc.pytorch:   MPC_REFERENCE=<checkout> python oracle/make_golden_receding_slew_grad.py
The loop is make_golden_receding_grad.py's (solve MPC(..., u_init=u_init, exit_unconverged=False,
detach_unconverged=False), apply nominal_actions[0], shift the warm start, step the plant), with
MPC(slew_rate_penalty=SLEW, prev_ctrl=the previous applied control): solve 0 takes the case's initial prev_ctrl (None:
the reference's zeros).  The reference detaches prev_ctrl itself (mpc/mpc.py:399-408), so the loss
sum(wx * x) + sum(wu * u) differentiates through each solve's augmented problem with the previous control held
constant.  Unmodified reference, CPU, float64, every input requiring grad.  Each solve's nominal_states /
nominal_actions are stored as plan_x [n_steps, T, B, n] (the system's states: the reference crops the augmented ones)
and plan_u [n_steps, T, B, m].

The reference's slew-rate branch takes no LinDx plant (it hands LQRStep true_dynamics=None for LinDx), so the linear
cases model LinDx(F0.expand(T-1, ...), f0.expand(T-1, ...)) as an affine Module x' = F0 [x; u] + f0 with
GradMethods.ANALYTIC and grad_input = (F0[:, :n], F0[:, n:]): its linearisation is F0 and f0 themselves, and the
gradient is LinDx's, summed over time (g_F [B, n, n+m], g_f [B, n]).

tests/golden/receding_grad_slew_f64.npz (keys prefixed by case; slew_rate_penalty SLEW):
  unbounded       LinDx n=4, m=2, B=4, T=10, 8 control steps (make_golden_receding_grad.problem()'s F[0], f[0], C, c,
                  x_init), prev_ctrl None;
  bounded         the same with u in [-0.5, 0.5] and a non-zero initial prev_ctrl, controls on the bounds;
  pendulum        PendulumDx(params=(10, 1, 1), simple=True), max_torque 2, GradMethods.AUTO_DIFF, B=4, T=10,
                  4 control steps, controls at the clamp;
  cartpole        CartpoleDx(params=(9.81, 1.3, 0.25, 0.8)), force_mag 6, otherwise as pendulum.
LinDx gradients g_x_init, g_C, g_c, g_F, g_f; known systems g_x_init, g_C, g_c, g_params (the reference's AUTO_DIFF
convention: its Jacobians are constants).  Round-off guard as make_golden_receding_grad.py's.  Only numbers are
stored.
"""
import contextlib
import io
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from make_golden import load_reference, npz                    # noqa: E402
from make_golden_nn import load_ref_env                         # noqa: E402
from make_golden_receding_grad import B, KB, KEPS, KITER, KNOWN, KSTEPS, KT, NAMES, KNAMES, STEPS, T, guarded, m, \
    n, problem                                                  # noqa: E402

SLEW = 0.1


def closed_loop(rmpc, make, leaves, problem_of, plant, steps, wx, wu, names, prev0):
    """The notebooks' loop under autograd with prev_ctrl = the previous applied control: (x, u, plan_x, plan_u,
    {name: gradient}, iterations per solve)."""
    iters = []
    real = rmpc.MPC.solve_lqr_subproblem

    def count(self, *a, **k):
        if not k.get("no_op_forward", False):
            iters[-1] += 1
        return real(self, *a, **k)
    rmpc.MPC.solve_lqr_subproblem = count
    try:
        x, u_init, prev = leaves["x_init"], None, prev0
        xs, us, px, pu = [x], [], [], []
        for _ in range(steps):
            iters.append(0)
            with contextlib.redirect_stdout(io.StringIO()):
                states, actions, _ = make(u_init, prev)(x, *problem_of(leaves))
            u_init = torch.cat((actions[1:], torch.zeros_like(actions[:1])), dim=0).detach()
            u_init[-2] = u_init[-3]
            prev = actions[0]
            x = plant(x, actions[0])
            xs.append(x)
            us.append(actions[0])
            px.append(states.detach())
            pu.append(actions.detach())
    finally:
        rmpc.MPC.solve_lqr_subproblem = real
    xs, us = torch.stack(xs), torch.stack(us)
    grads = torch.autograd.grad((wx * xs).sum() + (wu * us).sum(), [leaves[k] for k in names])
    return (xs.detach(), us.detach(), torch.stack(px), torch.stack(pu), dict(zip(names, grads)),
            np.array(iters, dtype=np.int64))


class Affine(torch.nn.Module):
    """x' = F0 [x; u] + f0 per problem (F0 [B, n, n+m], f0 [B, n]) for any batch of rows ordered (t, b)."""

    def __init__(self, F0, f0):
        super().__init__()
        self.F0, self.f0 = F0, f0

    def tiled(self, rows):
        r = rows // self.F0.shape[0]
        return self.F0.repeat(r, 1, 1), self.f0.repeat(r, 1)

    def forward(self, x, u):
        F0, f0 = self.tiled(x.shape[0])
        return (F0 @ torch.cat((x, u), 1).unsqueeze(2)).squeeze(2) + f0

    def grad_input(self, x, u):
        F0, _ = self.tiled(x.shape[0])
        return F0[:, :, :n], F0[:, :, n:]


def linear_run(rmpc, wx, wu, bound, prev0):
    kw = dict(u_lower=-bound, u_upper=bound) if bound is not None else {}

    def run(ins):
        leaves = {k: v.clone().requires_grad_(True) for k, v in ins.items()}
        dx = Affine(leaves["F"], leaves["f"])

        def make(u_init, prev):
            return rmpc.MPC(n, m, T, u_init=u_init, lqr_iter=10, verbose=0, exit_unconverged=False,
                            detach_unconverged=False, slew_rate_penalty=SLEW, prev_ctrl=prev,
                            grad_method=rmpc.GradMethods.ANALYTIC, **kw)
        return closed_loop(rmpc, make, leaves, lambda lv: (rmpc.QuadCost(lv["C"], lv["c"]), dx), dx, STEPS, wx, wu,
                           NAMES, prev0)
    return run


def known_case(rmpc, name):
    """A known system's slew-rate episode: (inputs, wx, wu, run, extra), the problem of make_golden_receding_grad's."""
    mod, ctor, params, attr, clamp = KNOWN[name]
    renv = load_ref_env(mod)
    cls = renv.CartpoleDx if name == "cartpole" else renv.PendulumDx
    dx0 = cls(params=torch.tensor(params), **ctor)
    ns, ms = dx0.n_state, dx0.n_ctrl
    g = torch.Generator().manual_seed(23 + len(name))
    q, p = dx0.get_true_obj()
    C = torch.diag(q).expand(KT, KB, ns + ms, ns + ms).contiguous()
    c = p.expand(KT, KB, ns + ms).contiguous()
    th = (torch.rand(KB, generator=g) * 2 - 1) * (3.0 if name == "cartpole" else 0.6)
    if name == "cartpole":
        x0 = torch.stack((torch.rand(KB, generator=g) - 0.5, torch.rand(KB, generator=g) - 0.5, th.cos(), th.sin(),
                          torch.rand(KB, generator=g) - 0.5), 1)
    else:
        x0 = torch.stack((th.cos(), th.sin(), torch.rand(KB, generator=g) - 0.5), 1)
    wx = torch.randn(KSTEPS + 1, KB, ns, generator=g)
    wu = torch.randn(KSTEPS, KB, ms, generator=g)
    inputs = dict(x_init=x0, C=C, c=c, params=torch.tensor(params))

    def run(ins):
        leaves = {k: v.clone().requires_grad_(True) for k, v in ins.items()}
        dx = cls(params=leaves["params"], **ctor)
        setattr(dx, attr, clamp)
        dx.lower, dx.upper = -clamp, clamp

        def make(u_init, prev):
            return rmpc.MPC(ns, ms, KT, u_init=u_init, u_lower=-clamp, u_upper=clamp, lqr_iter=KITER, verbose=0,
                            exit_unconverged=False, detach_unconverged=False, eps=KEPS,
                            linesearch_decay=dx.linesearch_decay, max_linesearch_iter=dx.max_linesearch_iter,
                            grad_method=rmpc.GradMethods.AUTO_DIFF, slew_rate_penalty=SLEW, prev_ctrl=prev)
        return closed_loop(rmpc, make, leaves, lambda lv: (rmpc.QuadCost(lv["C"], lv["c"]), dx), dx, KSTEPS, wx,
                           wu, KNAMES, None)
    return inputs, wx, wu, run, dict(ls_decay=np.float64(dx0.linesearch_decay),
                                     ls_iter=np.int64(dx0.max_linesearch_iter), clamp=np.float64(clamp))


def main():
    rmpc, _, _, _ = load_reference()
    torch.set_default_dtype(torch.float64)
    inputs, wx, wu = problem()
    inputs = dict(inputs, F=inputs["F"][0].clone(), f=inputs["f"][0].clone())
    prev_b = 0.4 * torch.randn(B, m, generator=torch.Generator().manual_seed(5))
    out = {}
    for name, bound, prev0 in (("unbounded", None, None), ("bounded", 0.5, prev_b)):
        xs, us, px, pu, g, iters = guarded(linear_run(rmpc, wx, wu, bound, prev0), inputs, name)
        on = int((us.abs() == bound).sum()) if bound is not None else 0
        print(name, "iterations", iters.tolist(), "controls on the bounds", on, "of", us.numel())
        if bound is not None:
            assert on > 0, name
        pre = name + "_"
        out.update({pre + k: v for k, v in inputs.items()})
        out.update({pre + "wx": wx, pre + "wu": wu, pre + "x": xs, pre + "u": us, pre + "iters": iters,
                    pre + "T": np.int64(T), pre + "n_steps": np.int64(STEPS), pre + "lqr_iter": np.int64(10),
                    pre + "eps": np.float64(1e-7), pre + "plan_x": px, pre + "plan_u": pu,
                    pre + "slew": np.float64(SLEW)})
        out.update({pre + "g_" + k: v for k, v in g.items()})
        if bound is not None:
            out[pre + "bound"] = np.float64(bound)
        if prev0 is not None:
            out[pre + "prev_ctrl"] = prev0
    for name in ("pendulum", "cartpole"):
        kin, kwx, kwu, run, extra = known_case(rmpc, name)
        xs, us, px, pu, g, iters = guarded(run, kin, name)
        clamp = float(extra["clamp"])
        print(name, "iterations", iters.tolist(), "plan controls at the clamp", int((pu.abs() == clamp).sum()), "of",
              pu.numel(), "applied", int((us.abs() == clamp).sum()), "of", us.numel())
        assert int((pu.abs() == clamp).sum()) > 0, name
        pre = name + "_"
        out.update({pre + k: v for k, v in kin.items()})
        out.update({pre + "wx": kwx, pre + "wu": kwu, pre + "x": xs, pre + "u": us, pre + "iters": iters,
                    pre + "plan_x": px, pre + "plan_u": pu, pre + "T": np.int64(KT), pre + "n_steps": np.int64(KSTEPS),
                    pre + "lqr_iter": np.int64(KITER), pre + "eps": np.float64(KEPS), pre + "slew": np.float64(SLEW)})
        out.update({pre + k: v for k, v in extra.items()})
        out.update({pre + "g_" + k: v for k, v in g.items()})
    npz("receding_grad_slew_f64", **out)


if __name__ == "__main__":
    main()
