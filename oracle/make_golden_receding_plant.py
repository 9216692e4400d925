#!/usr/bin/env python3
"""Fixtures for receding-horizon episodes closed on a plant other than the model, with additive disturbances, from the
REAL reference's own notebook loop under autograd.

Run with a checkout of locuslab/mpc.pytorch:   MPC_REFERENCE=<checkout> python oracle/make_golden_receding_plant.py
The loop is make_golden_receding_grad.py's (solve MPC(..., u_init=u_init, exit_unconverged=False,
detach_unconverged=False) with the MODEL, apply nominal_actions[0], shift the warm start), with the next state written
out as x_{k+1} = plant(x_k, u_k) + w_k, as the reference's examples/gym_pendulum_approximate.py closes the loop on the
environment rather than the model.  Under a slew-rate penalty each solve takes MPC(slew_rate_penalty=SLEW,
prev_ctrl=the previous applied control), which the reference detaches.  Unmodified reference, CPU, float64, every
input requiring grad (the model's, the plant's and w), loss sum(wx * x) + sum(wu * u).  Each solve's nominal_states /
nominal_actions are stored as plan_x [n_steps, T, B, n] and plan_u [n_steps, T, B, m].

tests/golden/receding_plant_f64.npz (keys prefixed by case):
  linear          LinDx model (make_golden_receding_grad.problem()'s x_init, C, c, F, f; n=4, m=2, B=4, T=10,
                  8 control steps) on the LinDx plant F_p [B, n, n+m] = F[0] (1 + 0.05 N), f_p [B, n] = f[0] + 0.02 N,
                  u in [-0.5, 0.5] (controls on the bounds), w = 0.05 N;
  pendulum        PendulumDx(params=(10, 1, 1), simple=True) model on PendulumDx(params=(10, 1, 1, 0.3, 0.2),
                  simple=False), max_torque 2 (the clamp binds), GradMethods.AUTO_DIFF, B=4, T=10, 4 control steps,
                  w = 0.02 N;
  cartpole        CartpoleDx(params=(9.81, 1.3, 0.25, 0.8)) model on CartpoleDx(params=(9.81, 1.35, 0.22, 0.78)),
                  force_mag 6, otherwise as pendulum;
  pendulum_slew   the pendulum case with slew_rate_penalty SLEW.
Gradients g_<input>: x_init, C, c, w and the model's F, f (LinDx) or params (the reference's AUTO_DIFF convention: its
Jacobians are constants), the plant's F_p, f_p or plant_params.  Round-off guard as make_golden_receding_grad.py's.
Only numbers are stored.
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
from make_golden_receding_grad import B, KB, KEPS, KITER, KNOWN, KSTEPS, KT, STEPS, T, guarded, m, n, \
    problem                                                     # noqa: E402

SLEW = 0.1
PLANTS = {"pendulum": ("pendulum", {"simple": False}, (10.0, 1.0, 1.0, 0.3, 0.2)),
          "cartpole": ("cartpole", {}, (9.81, 1.35, 0.22, 0.78))}


def closed_loop(rmpc, make, leaves, problem_of, plant, steps, wx, wu, names):
    """The loop under autograd with x_{k+1} = plant(x_k, u_k) + w_k: (x, u, plan_x, plan_u, {name: gradient},
    iterations per solve).  make(u_init, prev) builds solve k's MPC; prev is the previous applied control."""
    iters = []
    real = rmpc.MPC.solve_lqr_subproblem

    def count(self, *a, **k):
        if not k.get("no_op_forward", False):
            iters[-1] += 1
        return real(self, *a, **k)
    rmpc.MPC.solve_lqr_subproblem = count
    try:
        x, u_init, prev = leaves["x_init"], None, None
        xs, us, px, pu = [x], [], [], []
        for k in range(steps):
            iters.append(0)
            with contextlib.redirect_stdout(io.StringIO()):
                states, actions, _ = make(u_init, prev)(x, *problem_of(leaves))
            u_init = torch.cat((actions[1:], torch.zeros_like(actions[:1])), dim=0).detach()
            u_init[-2] = u_init[-3]
            prev = actions[0]
            x = plant(x, actions[0]) + leaves["w"][k]
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


def linear_case(rmpc, rutil):
    inputs, wx, wu = problem()
    g = torch.Generator().manual_seed(31)
    F0, f0 = inputs["F"][0], inputs["f"][0]
    inputs.update(F_p=F0 * (1 + 0.05 * torch.randn(F0.shape, generator=g)),
                  f_p=f0 + 0.02 * torch.randn(f0.shape, generator=g),
                  w=0.05 * torch.randn(STEPS, B, n, generator=g))
    names = ("x_init", "C", "c", "F", "f", "F_p", "f_p", "w")

    def run(ins):
        leaves = {k: v.clone().requires_grad_(True) for k, v in ins.items()}

        def make(u_init, prev):
            return rmpc.MPC(n, m, T, u_init=u_init, lqr_iter=10, verbose=0, exit_unconverged=False,
                            detach_unconverged=False, u_lower=-0.5, u_upper=0.5)
        return closed_loop(rmpc, make, leaves,
                           lambda lv: (rmpc.QuadCost(lv["C"], lv["c"]), rmpc.LinDx(lv["F"], lv["f"])),
                           lambda x, u: rutil.bmv(leaves["F_p"], torch.cat((x, u), 1)) + leaves["f_p"], STEPS, wx,
                           wu, names)
    return inputs, wx, wu, run, dict(T=np.int64(T), n_steps=np.int64(STEPS), lqr_iter=np.int64(10),
                                     eps=np.float64(1e-7), bound=np.float64(0.5))


def known_case(rmpc, name, slew):
    mod, ctor, params, attr, clamp = KNOWN[name]
    pmod, pctor, pparams = PLANTS[name]
    renv, penv = load_ref_env(mod), load_ref_env(pmod)
    cls = renv.CartpoleDx if name == "cartpole" else renv.PendulumDx
    pcls = penv.CartpoleDx if name == "cartpole" else penv.PendulumDx
    dx0 = cls(params=torch.tensor(params), **ctor)
    ns, ms = dx0.n_state, dx0.n_ctrl
    g = torch.Generator().manual_seed(41 + len(name))
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
    w = 0.02 * torch.randn(KSTEPS, KB, ns, generator=g)
    inputs = dict(x_init=x0, C=C, c=c, params=torch.tensor(params), plant_params=torch.tensor(pparams), w=w)
    names = ("x_init", "C", "c", "params", "plant_params", "w")

    def run(ins):
        leaves = {k: v.clone().requires_grad_(True) for k, v in ins.items()}
        dx = cls(params=leaves["params"], **ctor)
        pl = pcls(params=leaves["plant_params"], **pctor)
        for d in (dx, pl):
            setattr(d, attr, clamp)
            d.lower, d.upper = -clamp, clamp
        sl = dict(slew_rate_penalty=SLEW) if slew else {}

        def make(u_init, prev):
            return rmpc.MPC(ns, ms, KT, u_init=u_init, u_lower=-clamp, u_upper=clamp, lqr_iter=KITER, verbose=0,
                            exit_unconverged=False, detach_unconverged=False, eps=KEPS,
                            linesearch_decay=dx.linesearch_decay, max_linesearch_iter=dx.max_linesearch_iter,
                            grad_method=rmpc.GradMethods.AUTO_DIFF,
                            **(dict(sl, prev_ctrl=prev) if slew else {}))
        return closed_loop(rmpc, make, leaves, lambda lv: (rmpc.QuadCost(lv["C"], lv["c"]), dx), pl, KSTEPS, wx,
                           wu, names)
    extra = dict(ls_decay=np.float64(dx0.linesearch_decay), ls_iter=np.int64(dx0.max_linesearch_iter),
                 clamp=np.float64(clamp), T=np.int64(KT), n_steps=np.int64(KSTEPS), lqr_iter=np.int64(KITER),
                 eps=np.float64(KEPS))
    if slew:
        extra["slew"] = np.float64(SLEW)
    return inputs, wx, wu, run, extra


def main():
    rmpc, _, _, rutil = load_reference()
    torch.set_default_dtype(torch.float64)
    out = {}
    cases = [("linear", lambda: linear_case(rmpc, rutil)), ("pendulum", lambda: known_case(rmpc, "pendulum", False)),
             ("cartpole", lambda: known_case(rmpc, "cartpole", False)),
             ("pendulum_slew", lambda: known_case(rmpc, "pendulum", True))]
    for name, mk in cases:
        inputs, wx, wu, run, extra = mk()
        xs, us, px, pu, g, iters = guarded(run, inputs, name)
        bound = float(extra.get("clamp", extra.get("bound")))
        on = int((pu.abs() == bound).sum())
        print(name, "iterations", iters.tolist(), "plan controls on the bound", on, "of", pu.numel())
        assert on > 0, name
        pre = name + "_"
        out.update({pre + k: v for k, v in inputs.items()})
        out.update({pre + "wx": wx, pre + "wu": wu, pre + "x": xs, pre + "u": us, pre + "iters": iters,
                    pre + "plan_x": px, pre + "plan_u": pu})
        out.update({pre + k: v for k, v in extra.items()})
        out.update({pre + "g_" + k: v for k, v in g.items()})
    npz("receding_plant_f64", **out)


if __name__ == "__main__":
    main()
