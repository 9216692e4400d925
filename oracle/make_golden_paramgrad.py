#!/usr/bin/env python3
"""Fixtures for the parameter gradient of a known system, from the REAL reference.

Run with a checkout of locuslab/mpc.pytorch:   MPC_REFERENCE=<checkout> python oracle/make_golden_paramgrad.py
Solves MPC(n, 1, T) of the unmodified reference (mpc/mpc.py) with its own CartpoleDx and PendulumDx (mpc/env_dx/) at
the non-default physics of oracle/make_golden_nn.py (KNOWN_SYSTEMS), float64, AUTO_DIFF, with `params` requiring
grad, once without bounds and once with box bounds inside the clamp, and backpropagates a fixed linear loss
<wx, x> + <wu, u>.  Stores per regime
  x, u        the solution;
  x_lin       the states at which the reference's final linearize_dynamics(diff=True) linearised (it re-rolls the
              system out from x_init under u, mpc/mpc.py:538-592);
  df          the gradient that reached that call's f (a tensor hook on its output);
  grad        the reference's params.grad.
The reference takes R, S without create_graph, so its F carries no gradient and grad = sum_{t,b} df . dx'/dtheta at
(x_lin, u): the `first` output of the VJP kernel.  tests/golden/paramgrad_{cartpole,pendulum}_f64.npz; only numbers
are stored.
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
from make_golden_nn import KNOWN_SYSTEMS, _known_states, load_ref_env    # noqa: E402

B, T, LQR_ITER = 5, 8, 15


def main():
    rmpc, _, _, _ = load_reference()
    torch.set_default_dtype(torch.float64)
    seen = {}
    orig = rmpc.MPC.linearize_dynamics

    def hooked(self, x, u, dynamics, diff):
        F, f = orig(self, x, u, dynamics, diff)
        if diff:
            f.register_hook(lambda g: seen.__setitem__("df", g.detach().clone()))
        return F, f

    rmpc.MPC.linearize_dynamics = hooked
    for name, spec in KNOWN_SYSTEMS.items():
        renv = load_ref_env(name)
        n = 5 if name == "cartpole" else 3
        clamp = spec["clamp"][1]
        g = torch.Generator().manual_seed(51 if name == "cartpole" else 52)
        x0 = _known_states(name, B, g)
        probe = (renv.CartpoleDx if name == "cartpole" else renv.PendulumDx)(params=torch.tensor(spec["params"]))
        q, p = probe.get_true_obj()
        Q = torch.diag(q.double()).repeat(T, B, 1, 1)
        pp = p.double().repeat(T, B, 1)
        pp[..., n:] = 0.3 * clamp * (torch.rand(T, B, 1, generator=g) - 0.5)
        wx = torch.randn(T, B, n, generator=g)
        wu = torch.randn(T, B, 1, generator=g)
        out = dict(params=torch.tensor(spec["params"]), dt=np.float64(spec["dt"]), clamp=np.float64(clamp),
                   decay=np.float64(spec["decay"]), ls_iter=np.int64(spec["ls_iter"]), lqr_iter=np.int64(LQR_ITER),
                   x_init=x0, C=Q, c=pp, wx=wx, wu=wu)
        for tag, bound in (("unb", None), ("box", 0.8 * clamp)):
            params = torch.tensor(spec["params"]).requires_grad_(True)
            dx = (renv.CartpoleDx if name == "cartpole" else renv.PendulumDx)(params=params)
            dx.dt = spec["dt"]
            setattr(dx, spec["clamp"][0], clamp)
            kw = {} if bound is None else dict(u_lower=-bound, u_upper=bound)
            seen.clear()
            with contextlib.redirect_stdout(io.StringIO()):
                x, u, costs = rmpc.MPC(n, 1, T, lqr_iter=LQR_ITER, verbose=-1, exit_unconverged=False,
                                       detach_unconverged=False, linesearch_decay=spec["decay"],
                                       max_linesearch_iter=spec["ls_iter"], grad_method=rmpc.GradMethods.AUTO_DIFF,
                                       eps=1e-9, **kw)(x0, rmpc.QuadCost(Q, pp), dx)
            ((wx * x).sum() + (wu * u).sum()).backward()
            with torch.no_grad():
                x_lin = [x0]
                for t in range(T - 1):
                    x_lin.append(dx(x_lin[t], u[t]))
                x_lin = torch.stack(x_lin)
            beyond = int((u.abs() > clamp).sum())
            print(f"{name} {tag}: grad {params.grad.tolist()}, controls beyond the clamp {beyond} of {u.numel()}, "
                  f"max|x_lin - x| {float((x_lin - x).abs().max()):.2e}")
            out.update({f"x_{tag}": x, f"u_{tag}": u, f"x_lin_{tag}": x_lin, f"df_{tag}": seen["df"],
                        f"grad_{tag}": params.grad})
            if bound is not None:
                out[f"bound_{tag}"] = np.float64(bound)
        npz(f"paramgrad_{name}_f64", **out)
    rmpc.MPC.linearize_dynamics = orig


if __name__ == "__main__":
    main()
