#!/usr/bin/env python3
"""Fixtures for differentiable receding-horizon episodes, from the REAL reference's own notebook loop under autograd.

Run with a checkout of locuslab/mpc.pytorch:   MPC_REFERENCE=<checkout> python oracle/make_golden_receding_grad.py
Runs the notebooks' control loop (make_golden_receding.py's: solve MPC(..., u_init=u_init,
exit_unconverged=False, detach_unconverged=False), apply nominal_actions[0], shift u_init = cat(nominal_actions[1:], 0)
with u_init[-2] = u_init[-3], step the plant) on the unmodified reference, CPU, float64, with every input requiring
grad, and differentiates the fixed linear loss sum(wx * x) + sum(wu * u).  The reference detaches each u_init itself
(mpc/mpc.py:163).  Every case also stores each solve's nominal_states / nominal_actions (plan_x [n_steps, T, B, n],
plan_u [n_steps, T, B, m]): the points the reverse sweep linearises at, which oracle.receding_horizon_backward takes.

tests/golden/receding_grad_linear_f64.npz, both LinDx (n=4, m=2, B=4, T=10, 8 control steps), plant F_0 tau + f_0 by
util.bmv, gradients g_x_init, g_C, g_c, g_F, g_f:
  unbounded   no control bounds;
  bounded     u in [-0.5, 0.5], with controls on the bounds.
tests/golden/receding_grad_known_f64.npz, the reference's own systems with params requiring grad (GradMethods.AUTO_DIFF,
u_lower / u_upper = the system's clamp, which the controls reach; B=4, 4 control steps), plant dx(x, u), gradients
g_x_init, g_C, g_c, g_params:
  cartpole        CartpoleDx(params=(9.81, 1.3, 0.25, 0.8)), force_mag 6, T=10;
  pendulum        PendulumDx(params=(10, 1, 1), simple=True), max_torque 2, T=10;
  pendulum_full   PendulumDx(params=(10, 1, 1, 0.1, 0.05), simple=False), max_torque 2, T=10.
The reference's AUTO_DIFF linearisation takes its Jacobians without create_graph, so g_params is its convention: the
linearisation differentiates as x' alone (INTEGRATION.md section 2).  Each key is prefixed by its case.  Round-off guard
(make_golden_receding.py's, applied to the gradients too): every episode is rerun from x_init perturbed by 1e-12
relative; its iteration counts must be identical and its x, u, plans and gradients within GUARD relative to their
largest entry.  A rerun of this script must leave every array that receding_grad_linear_f64.npz held before it
bitwise unchanged.  Only numbers are stored.
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
from make_golden import GOLD, load_reference, npz              # noqa: E402
from make_golden_nn import load_ref_env                        # noqa: E402

B, T, n, m, STEPS = 4, 10, 4, 2, 8
GUARD = 1e-6
NAMES = ("x_init", "C", "c", "F", "f")


def problem():
    g = torch.Generator().manual_seed(7)
    L = torch.randn(T, B, n + m, n + m, generator=g) / (n + m) ** 0.5
    C = L @ L.transpose(-1, -2) + torch.eye(n + m)
    c = torch.randn(T, B, n + m, generator=g)
    A = 0.9 * torch.eye(n) + 0.2 * torch.randn(B, n, n, generator=g) / n ** 0.5
    F = torch.cat((A, torch.randn(B, n, m, generator=g) / n ** 0.5), -1).unsqueeze(0).repeat(T - 1, 1, 1, 1)
    f = 0.1 * torch.randn(T - 1, B, n, generator=g)
    x0 = 2.0 * torch.randn(B, n, generator=g)
    wx = torch.randn(STEPS + 1, B, n, generator=g)
    wu = torch.randn(STEPS, B, m, generator=g)
    return dict(x_init=x0, C=C, c=c, F=F, f=f), wx, wu


def differentiated(rmpc, rutil, inputs, wx, wu, bound):
    leaves = {k: v.clone().requires_grad_(True) for k, v in inputs.items()}
    kw = dict(u_lower=-bound, u_upper=bound) if bound is not None else {}

    def make(u_init):
        return rmpc.MPC(n, m, T, u_init=u_init, lqr_iter=10, verbose=0, exit_unconverged=False,
                        detach_unconverged=False, **kw)

    F, f = leaves["F"], leaves["f"]
    return closed_loop(rmpc, make, leaves, lambda lv: (rmpc.QuadCost(lv["C"], lv["c"]), rmpc.LinDx(F, f)),
                       lambda x, u: rutil.bmv(F[0], torch.cat((x, u), 1)) + f[0], STEPS, wx, wu, NAMES)


def closed_loop(rmpc, make, leaves, problem, plant, steps, wx, wu, names):
    """The notebooks' loop under autograd: (x, u, plan_x, plan_u, {name: gradient}, iterations per solve)."""
    iters = []
    real = rmpc.MPC.solve_lqr_subproblem

    def count(self, *a, **k):                  # iterations of each solve, as make_golden_receding.episode counts
        if not k.get("no_op_forward", False):
            iters[-1] += 1
        return real(self, *a, **k)
    rmpc.MPC.solve_lqr_subproblem = count
    try:
        x, u_init, xs, us, px, pu = leaves["x_init"], None, [leaves["x_init"]], [], [], []
        for _ in range(steps):
            iters.append(0)
            with contextlib.redirect_stdout(io.StringIO()):
                states, actions, _ = make(u_init)(x, *problem(leaves))
            u_init = torch.cat((actions[1:], torch.zeros_like(actions[:1])), dim=0).detach()
            u_init[-2] = u_init[-3]
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


def guarded(run, inputs, name):
    """run(inputs) and run(inputs with x_init * (1 + 1e-12)): the same iteration counts, and x, u, the plans and the
    gradients within GUARD relative."""
    out = run(inputs)
    again = run(dict(inputs, x_init=inputs["x_init"] * (1 + 1e-12)))
    assert np.array_equal(out[5], again[5]), (name, out[5], again[5])
    pairs = list(zip(("x", "u", "plan_x", "plan_u"), out[:4], again[:4]))
    pairs += [(k, out[4][k], again[4][k]) for k in out[4]]
    for what, a, b in pairs:
        err = float((a - b).abs().max()) / max(1.0, float(a.abs().max()))
        assert err < GUARD, (name, what, err)
    return out


# the known systems: (reference module name, constructor keywords, params, clamp attribute, clamp)
KNOWN = {"cartpole": ("cartpole", {}, (9.81, 1.3, 0.25, 0.8), "force_mag", 6.0),
         "pendulum": ("pendulum", {"simple": True}, (10.0, 1.0, 1.0), "max_torque", 2.0),
         "pendulum_full": ("pendulum", {"simple": False}, (10.0, 1.0, 1.0, 0.1, 0.05), "max_torque", 2.0)}
KB, KT, KSTEPS, KITER, KEPS = 4, 10, 4, 30, 1e-4
KNAMES = ("x_init", "C", "c", "params")


def known_case(rmpc, name):
    """A known system's episode: (inputs, wx, wu, run) with run(inputs) the reference's loop under autograd."""
    mod, ctor, params, attr, clamp = KNOWN[name]
    renv = load_ref_env(mod)
    dx0 = (renv.CartpoleDx if name == "cartpole" else renv.PendulumDx)(params=torch.tensor(params), **ctor)
    n, m = dx0.n_state, dx0.n_ctrl
    g = torch.Generator().manual_seed(11 + len(name))
    q, p = dx0.get_true_obj()
    C = torch.diag(q).expand(KT, KB, n + m, n + m).contiguous()
    c = p.expand(KT, KB, n + m).contiguous()
    th = (torch.rand(KB, generator=g) * 2 - 1) * (3.0 if name == "cartpole" else 0.6)
    if name == "cartpole":
        x0 = torch.stack((torch.rand(KB, generator=g) - 0.5, torch.rand(KB, generator=g) - 0.5, th.cos(), th.sin(),
                          torch.rand(KB, generator=g) - 0.5), 1)
    else:
        x0 = torch.stack((th.cos(), th.sin(), torch.rand(KB, generator=g) - 0.5), 1)
    wx = torch.randn(KSTEPS + 1, KB, n, generator=g)
    wu = torch.randn(KSTEPS, KB, m, generator=g)
    inputs = dict(x_init=x0, C=C, c=c, params=torch.tensor(params))

    def run(ins):
        leaves = {k: v.clone().requires_grad_(True) for k, v in ins.items()}
        dx = (renv.CartpoleDx if name == "cartpole" else renv.PendulumDx)(params=leaves["params"], **ctor)
        setattr(dx, attr, clamp)
        dx.lower, dx.upper = -clamp, clamp

        def make(u_init):
            return rmpc.MPC(n, m, KT, u_init=u_init, u_lower=-clamp, u_upper=clamp, lqr_iter=KITER, verbose=0,
                            exit_unconverged=False, detach_unconverged=False, eps=KEPS,
                            linesearch_decay=dx.linesearch_decay, max_linesearch_iter=dx.max_linesearch_iter,
                            grad_method=rmpc.GradMethods.AUTO_DIFF)
        return closed_loop(rmpc, make, leaves, lambda lv: (rmpc.QuadCost(lv["C"], lv["c"]), dx), dx, KSTEPS, wx,
                           wu, KNAMES)
    return inputs, wx, wu, run, dict(ls_decay=np.float64(dx0.linesearch_decay),
                                     ls_iter=np.int64(dx0.max_linesearch_iter), clamp=np.float64(clamp))


def main():
    rmpc, _, _, rutil = load_reference()
    torch.set_default_dtype(torch.float64)
    inputs, wx, wu = problem()
    old = dict(np.load(os.path.join(GOLD, "receding_grad_linear_f64.npz")))
    out = {}
    for name, bound in (("unbounded", None), ("bounded", 0.5)):
        xs, us, px, pu, g, iters = guarded(lambda ins: differentiated(rmpc, rutil, ins, wx, wu, bound), inputs, name)
        print(name, "iterations", iters.tolist(), "controls on the bounds", int((us.abs() == bound).sum())
              if bound is not None else 0, "of", us.numel())
        pre = name + "_"
        out.update({pre + k: v for k, v in inputs.items()})
        out.update({pre + "wx": wx, pre + "wu": wu, pre + "x": xs, pre + "u": us, pre + "iters": iters,
                    pre + "T": np.int64(T), pre + "n_steps": np.int64(STEPS), pre + "lqr_iter": np.int64(10),
                    pre + "eps": np.float64(1e-7), pre + "plan_x": px, pre + "plan_u": pu})
        out.update({pre + "g_" + k: v for k, v in g.items()})
        if bound is not None:
            out[pre + "bound"] = np.float64(bound)
    for k, v in old.items():                  # the arrays stored before the plans were added stay bitwise the same
        assert np.array_equal(np.asarray(out[k].detach() if torch.is_tensor(out[k]) else out[k]), v), k
    npz("receding_grad_linear_f64", **out)

    out = {}
    for name in KNOWN:
        inputs, kwx, kwu, run, extra = known_case(rmpc, name)
        xs, us, px, pu, g, iters = guarded(run, inputs, name)
        clamp = float(extra["clamp"])
        print(name, "iterations", iters.tolist(), "plan controls at the clamp", int((pu.abs() == clamp).sum()), "of",
              pu.numel(), "applied", int((us.abs() == clamp).sum()), "of", us.numel())
        assert int((pu.abs() == clamp).sum()) > 0, name
        pre = name + "_"
        out.update({pre + k: v for k, v in inputs.items()})
        out.update({pre + "wx": kwx, pre + "wu": kwu, pre + "x": xs, pre + "u": us, pre + "iters": iters,
                    pre + "plan_x": px, pre + "plan_u": pu, pre + "T": np.int64(KT), pre + "n_steps": np.int64(KSTEPS),
                    pre + "lqr_iter": np.int64(KITER), pre + "eps": np.float64(KEPS)})
        out.update({pre + k: v for k, v in extra.items()})
        out.update({pre + "g_" + k: v for k, v in g.items()})
    npz("receding_grad_known_f64", **out)


if __name__ == "__main__":
    main()
