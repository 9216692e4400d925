#!/usr/bin/env python3
"""Fixtures for receding-horizon episodes on a time-varying problem, from the REAL reference's own notebook loop under
autograd, with the slicing written out as a reference user writes it for a tracking problem or a time-varying model.

Run with a checkout of locuslab/mpc.pytorch:   MPC_REFERENCE=<checkout> python oracle/make_golden_receding_tv.py
Every time-indexed input lies on the episode's axis of L = n_steps + T - 1 slices.  Solve k is
MPC(..., u_init=the shifted warm start, exit_unconverged=False, detach_unconverged=False, u_lower/u_upper = the
bounds' slices [k:k+T] where they are tensors) on QuadCost(C[k:k+T], c[k:k+T]) and LinDx(F[k:k+T-1], f[k:k+T-1]) or
the known system; the next state is the model's step at slice k (F[k] [x; u] + f[k], or the system's own step) or a
LinDx plant's slice k, plus w[k].  Under a slew-rate penalty solve k takes prev_ctrl = the previous applied control,
which the reference detaches.  Unmodified reference, CPU, float64, every input requiring grad, loss
sum(wx * x) + sum(wu * u).  Each solve's nominal_states / nominal_actions are stored as plan_x [n_steps, T, B, n] and
plan_u [n_steps, T, B, m].

tests/golden/receding_tv_f64.npz (keys prefixed by case):
  linear         time-varying LinDx (n=4, m=2, B=3, T=6, 5 control steps, L=10) tracking a moving target, with
                 tensor bounds lo, hi [L, B, m] (controls on the bounds);
  pendulum       PendulumDx(params=(10, 1, 1)) tracking a goal angle 0.5 sin(0.3 t) (a time-varying c), max_torque 2
                 (the clamp binds), GradMethods.AUTO_DIFF, B=4, T=8, 4 control steps;
  cartpole       CartpoleDx(params=(9.81, 1.3, 0.25, 0.8)) moving its cart between set points 0 and 0.5, force_mag 6;
  pendulum_slew  the pendulum case with slew_rate_penalty SLEW (the penalty keeps its controls inside the clamp);
  linear_plant   the linear case's model, scalar bounds 0.5, on the time-varying LinDx plant F_p = F (1 + 0.05 N),
                 f_p = f + 0.02 N, with w = 0.05 N.
Gradients g_<input>: x_init, C, c, the model's F, f or params (the reference's AUTO_DIFF convention: its Jacobians
are constants), F_p, f_p and w.  Round-off guard as make_golden_receding_grad.py's.  Only numbers are stored.
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
from make_golden_receding_grad import KNOWN, guarded           # noqa: E402

SLEW = 0.1
SEED_PLANT = 59                     # seeds whose episodes pass the round-off guard
LB, LT, LSTEPS, LN, LM = 3, 6, 5, 4, 2
KB, KT, KSTEPS, KITER, KEPS = 4, 8, 4, 30, 1e-4


def closed_loop(rmpc, make, leaves, window, step_k, steps, wx, wu, names):
    """The windowed loop under autograd: make(k, u_init, prev) builds solve k's MPC, window(k) gives its cost and
    dynamics, step_k(k, x, u) the next state before w.  Returns (x, u, plan_x, plan_u, {name: gradient},
    iterations per solve)."""
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
                states, actions, _ = make(k, u_init, prev)(x, *window(k))
            u_init = torch.cat((actions[1:], torch.zeros_like(actions[:1])), dim=0).detach()
            u_init[-2] = u_init[-3]
            prev = actions[0]
            x = step_k(k, x, actions[0])
            if "w" in leaves:
                x = x + leaves["w"][k]
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


def linear_case(rmpc, rutil, with_plant):
    L = LSTEPS + LT - 1
    n, m, B, T = LN, LM, LB, LT
    g = torch.Generator().manual_seed(SEED_PLANT if with_plant else 53)
    R = torch.randn(L, B, n + m, n + m, generator=g) / (n + m) ** 0.5
    C = R @ R.transpose(-1, -2) + torch.eye(n + m)
    t = torch.arange(L, dtype=torch.float64)
    target = torch.sin(0.4 * t)[:, None, None] * torch.randn(1, B, n + m, generator=g)
    c = 0.3 * torch.randn(L, B, n + m, generator=g) - (C @ target.unsqueeze(-1)).squeeze(-1)
    A = 0.9 * torch.eye(n) + 0.1 * torch.randn(L - 1, B, n, n, generator=g) / n ** 0.5
    F = torch.cat((A, torch.randn(L - 1, B, n, m, generator=g) / n ** 0.5), 3)
    f = 0.1 * torch.randn(L - 1, B, n, generator=g)
    x0 = 2.0 * torch.randn(B, n, generator=g)
    wx, wu = torch.randn(LSTEPS + 1, B, n, generator=g), torch.randn(LSTEPS, B, m, generator=g)
    inputs = dict(x_init=x0, C=C, c=c, F=F, f=f)
    names = ["x_init", "C", "c", "F", "f"]
    extra = dict(T=np.int64(T), n_steps=np.int64(LSTEPS), lqr_iter=np.int64(10), eps=np.float64(1e-7))
    if with_plant:
        inputs.update(F_p=F * (1 + 0.05 * torch.randn(F.shape, generator=g)),
                      f_p=f + 0.02 * torch.randn(f.shape, generator=g), w=0.05 * torch.randn(LSTEPS, B, n, generator=g))
        names += ["F_p", "f_p", "w"]
        extra["bound"] = np.float64(0.5)
    else:
        lo = -0.2 - 0.4 * torch.rand(L, B, m, generator=g)
        inputs.update(lo=lo, hi=-lo + 0.1)

    def run(ins):
        leaves = {k: v.clone().requires_grad_(k not in ("lo", "hi")) for k, v in ins.items()}

        def make(k, u_init, prev):
            b = (dict(u_lower=leaves["lo"][k:k + T], u_upper=leaves["hi"][k:k + T]) if "lo" in leaves
                 else dict(u_lower=-0.5, u_upper=0.5))
            return rmpc.MPC(n, m, T, u_init=u_init, lqr_iter=10, verbose=0, exit_unconverged=False,
                            detach_unconverged=False, **b)

        def window(k):
            return (rmpc.QuadCost(leaves["C"][k:k + T], leaves["c"][k:k + T]),
                    rmpc.LinDx(leaves["F"][k:k + T - 1], leaves["f"][k:k + T - 1]))

        def step_k(k, x, u):
            Fs, fs = (leaves["F_p"], leaves["f_p"]) if with_plant else (leaves["F"], leaves["f"])
            return rutil.bmv(Fs[k], torch.cat((x, u), 1)) + fs[k]
        return closed_loop(rmpc, make, leaves, window, step_k, LSTEPS, wx, wu, names)
    return inputs, wx, wu, run, extra


def known_case(rmpc, name, slew):
    mod, ctor, params, attr, clamp = KNOWN[name]
    renv = load_ref_env(mod)
    cls = renv.CartpoleDx if name == "cartpole" else renv.PendulumDx
    dx0 = cls(params=torch.tensor(params), **ctor)
    ns, ms = dx0.n_state, dx0.n_ctrl
    L = KSTEPS + KT - 1
    g = torch.Generator().manual_seed(71 + len(name))
    q, p = dx0.get_true_obj()
    C = torch.diag(q).expand(L, KB, ns + ms, ns + ms).contiguous()
    t = torch.arange(L, dtype=torch.float64)
    goal = torch.zeros(L, KB, ns + ms)
    if name == "pendulum":
        ang = 0.5 * torch.sin(0.3 * t)
        goal[:, :, 0], goal[:, :, 1] = ang.cos()[:, None], ang.sin()[:, None]
    else:
        goal[:, :, 0] = (0.5 * (t >= L // 2).double())[:, None]
        goal[:, :, 2] = 1.0
    c = p.expand(L, KB, ns + ms) - (C @ goal.unsqueeze(-1)).squeeze(-1)
    th = (torch.rand(KB, generator=g) * 2 - 1) * (3.0 if name == "cartpole" else 0.6)
    if name == "cartpole":
        x0 = torch.stack((torch.rand(KB, generator=g) - 0.5, torch.rand(KB, generator=g) - 0.5, th.cos(), th.sin(),
                          torch.rand(KB, generator=g) - 0.5), 1)
    else:
        x0 = torch.stack((th.cos(), th.sin(), torch.rand(KB, generator=g) - 0.5), 1)
    wx = torch.randn(KSTEPS + 1, KB, ns, generator=g)
    wu = torch.randn(KSTEPS, KB, ms, generator=g)
    inputs = dict(x_init=x0, C=C, c=c, params=torch.tensor(params))
    names = ("x_init", "C", "c", "params")

    def run(ins):
        leaves = {k: v.clone().requires_grad_(True) for k, v in ins.items()}
        dx = cls(params=leaves["params"], **ctor)
        setattr(dx, attr, clamp)
        dx.lower, dx.upper = -clamp, clamp

        def make(k, u_init, prev):
            return rmpc.MPC(ns, ms, KT, u_init=u_init, u_lower=-clamp, u_upper=clamp, lqr_iter=KITER, verbose=0,
                            exit_unconverged=False, detach_unconverged=False, eps=KEPS,
                            linesearch_decay=dx.linesearch_decay, max_linesearch_iter=dx.max_linesearch_iter,
                            grad_method=rmpc.GradMethods.AUTO_DIFF,
                            **(dict(slew_rate_penalty=SLEW, prev_ctrl=prev) if slew else {}))
        return closed_loop(rmpc, make, leaves,
                           lambda k: (rmpc.QuadCost(leaves["C"][k:k + KT], leaves["c"][k:k + KT]), dx),
                           lambda k, x, u: dx(x, u), KSTEPS, wx, wu, names)
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
    cases = [("linear", lambda: linear_case(rmpc, rutil, False)),
             ("pendulum", lambda: known_case(rmpc, "pendulum", False)),
             ("cartpole", lambda: known_case(rmpc, "cartpole", False)),
             ("pendulum_slew", lambda: known_case(rmpc, "pendulum", True)),
             ("linear_plant", lambda: linear_case(rmpc, rutil, True))]
    for name, mk in cases:
        inputs, wx, wu, run, extra = mk()
        xs, us, px, pu, g, iters = guarded(run, inputs, name)
        if "clamp" in extra:
            on = int((pu.abs() == float(extra["clamp"])).sum())
        elif "lo" in inputs:
            T = int(extra["T"])
            on = sum(int(((pu[k] == inputs["lo"][k:k + T]) | (pu[k] == inputs["hi"][k:k + T])).sum())
                     for k in range(pu.shape[0]))
        else:
            on = int((pu.abs() == float(extra["bound"])).sum())
        print(name, "iterations", iters.tolist(), "plan controls on the bound", on, "of", pu.numel())
        assert on > 0 or name == "pendulum_slew", name
        pre = name + "_"
        out.update({pre + k: v for k, v in inputs.items()})
        out.update({pre + "wx": wx, pre + "wu": wu, pre + "x": xs, pre + "u": us, pre + "iters": iters,
                    pre + "plan_x": px, pre + "plan_u": pu})
        out.update({pre + k: v for k, v in extra.items()})
        out.update({pre + "g_" + k: v for k, v in g.items()})
    npz("receding_tv_f64", **out)


if __name__ == "__main__":
    main()
