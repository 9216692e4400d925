#!/usr/bin/env python3
"""Fixtures for differentiable receding-horizon episodes, from the REAL reference's own notebook loop under autograd.

Run with a checkout of locuslab/mpc.pytorch:   MPC_REFERENCE=<checkout> python oracle/make_golden_receding_grad.py
Runs the notebooks' control loop (make_golden_receding.py's: solve MPC(..., u_init=u_init,
exit_unconverged=False, detach_unconverged=False), apply nominal_actions[0], shift u_init = cat(nominal_actions[1:], 0)
with u_init[-2] = u_init[-3], step the plant F_0 tau + f_0 by util.bmv) on the unmodified reference, CPU, float64,
with x_init, C, c, F and f requiring grad, and differentiates the fixed linear loss sum(wx * x) + sum(wu * u).  The
reference detaches each u_init itself (mpc/mpc.py:163).  Cases, both LinDx (n=4, m=2, B=4, T=10, 8 control steps):
  unbounded   no control bounds;
  bounded     u in [-0.5, 0.5], with controls on the bounds.
Stores the inputs, the loss weights, x, u and the gradients g_x_init, g_C, g_c, g_F, g_f as
tests/golden/receding_grad_linear_f64.npz, each key prefixed by its case.  Round-off guard (make_golden_receding.py's,
applied to the gradients too): every episode is rerun from x_init perturbed by 1e-12 relative; its iteration counts
must be identical and its x, u and gradients within GUARD relative to their largest entry.  Only numbers are stored.
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

    def make(u_init, prev):
        return rmpc.MPC(n, m, T, u_init=u_init, lqr_iter=10, verbose=0, exit_unconverged=False,
                        detach_unconverged=False, **kw)

    F, f = leaves["F"], leaves["f"]
    iters = []
    real = rmpc.MPC.solve_lqr_subproblem

    def count(self, *a, **k):                  # iterations of each solve, as make_golden_receding.episode counts
        if not k.get("no_op_forward", False):
            iters[-1] += 1
        return real(self, *a, **k)
    rmpc.MPC.solve_lqr_subproblem = count
    try:
        x, u_init, xs, us = leaves["x_init"], None, [leaves["x_init"]], []
        for _ in range(STEPS):
            iters.append(0)
            with contextlib.redirect_stdout(io.StringIO()):
                _, actions, _ = make(u_init, None)(x, rmpc.QuadCost(leaves["C"], leaves["c"]), rmpc.LinDx(F, f))
            u_init = torch.cat((actions[1:], torch.zeros(1, B, m)), dim=0)
            u_init[-2] = u_init[-3]
            x = rutil.bmv(F[0], torch.cat((x, actions[0]), 1)) + f[0]
            xs.append(x)
            us.append(actions[0])
    finally:
        rmpc.MPC.solve_lqr_subproblem = real
    xs, us = torch.stack(xs), torch.stack(us)
    grads = torch.autograd.grad((wx * xs).sum() + (wu * us).sum(), [leaves[k] for k in NAMES])
    return xs.detach(), us.detach(), dict(zip(NAMES, grads)), np.array(iters, dtype=np.int64)


def main():
    rmpc, _, _, rutil = load_reference()
    torch.set_default_dtype(torch.float64)
    inputs, wx, wu = problem()
    out = {}
    for name, bound in (("unbounded", None), ("bounded", 0.5)):
        xs, us, g, iters = differentiated(rmpc, rutil, inputs, wx, wu, bound)
        moved = dict(inputs, x_init=inputs["x_init"] * (1 + 1e-12))
        xs2, us2, g2, iters2 = differentiated(rmpc, rutil, moved, wx, wu, bound)
        assert np.array_equal(iters, iters2), (iters, iters2)
        for what, a, b in [("x", xs, xs2), ("u", us, us2)] + [(k, g[k], g2[k]) for k in NAMES]:
            err = float((a - b).abs().max()) / max(1.0, float(a.abs().max()))
            assert err < GUARD, (name, what, err)
        print(name, "iterations", iters.tolist(), "controls on the bounds", int((us.abs() == bound).sum())
              if bound is not None else 0, "of", us.numel())
        pre = name + "_"
        out.update({pre + k: v for k, v in inputs.items()})
        out.update({pre + "wx": wx, pre + "wu": wu, pre + "x": xs, pre + "u": us, pre + "iters": iters,
                    pre + "T": np.int64(T), pre + "n_steps": np.int64(STEPS), pre + "lqr_iter": np.int64(10),
                    pre + "eps": np.float64(1e-7)})
        out.update({pre + "g_" + k: v for k, v in g.items()})
        if bound is not None:
            out[pre + "bound"] = np.float64(bound)
    npz("receding_grad_linear_f64", **out)


if __name__ == "__main__":
    main()
