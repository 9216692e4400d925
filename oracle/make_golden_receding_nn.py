#!/usr/bin/env python3
"""Fixtures for receding-horizon episodes planned with a learned model, from the REAL reference's own loop under
autograd: the model-based control loop of its examples/gym_pendulum_approximate.py, in which a network plans and the
network itself or the real system steps.

Run with a checkout of locuslab/mpc.pytorch:   MPC_REFERENCE=<checkout> python oracle/make_golden_receding_nn.py
The loop is make_golden_receding_plant.py's closed_loop (solve MPC(..., u_init=u_init, exit_unconverged=False,
detach_unconverged=False) with the reference's NNDynamics, GradMethods.ANALYTIC, apply nominal_actions[0], shift the
warm start) with x_{k+1} = step(x_k, u_k) + w_k.  Unmodified reference, CPU, float64, every input requiring grad,
loss sum(wx * x) + sum(wu * u).

tests/golden/receding_nn_f64.npz (keys prefixed by case):
  net        NNDynamics(3, 2, hidden [12, 10], sigmoid, passthrough) with seeded weights (scaled by 0.5), B=4, T=8,
             4 control steps, u in [-1, 1]; the network steps the loop, w = 0;
  pendulum   NNDynamics(3, 1, hidden [16], sigmoid, passthrough) planning for the reference's PendulumDx(params=(10, 1,
             1), simple=True), max_torque 2, which steps the loop, u in [-2, 2], B=4, T=10, 4 control steps,
             w = 0.02 N.
Per case: x_init, C, c, W<i>, b<i>, w, (params), wx, wu, x, u, plan_x, plan_u, iters, T, n_steps, lqr_iter, eps, bound,
and g_<input> for x_init, C, c, w, every W<i> and b<i> (and the plant's params).  Round-off guard as
make_golden_receding_grad.py's.  Only numbers are stored.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from make_golden import load_reference, npz                    # noqa: E402
from make_golden_nn import load_ref_env                         # noqa: E402
from make_golden_receding_grad import guarded                   # noqa: E402
from make_golden_receding_plant import closed_loop              # noqa: E402

CASES = {"net": dict(n=3, m=2, hidden=[12, 10], B=4, T=8, steps=4, bound=1.0, lqr_iter=10, eps=1e-4, seed=51),
         "pendulum": dict(n=3, m=1, hidden=[16], B=4, T=10, steps=4, bound=2.0, lqr_iter=10, eps=1e-4, seed=52)}


def case(rmpc, rdyn, name):
    cf = CASES[name]
    n, m, B, T, steps, bound = cf["n"], cf["m"], cf["B"], cf["T"], cf["steps"], cf["bound"]
    torch.manual_seed(cf["seed"])
    net0 = rdyn.NNDynamics(n, m, hidden_sizes=cf["hidden"], activation="sigmoid", passthrough=True).double()
    g = torch.Generator().manual_seed(cf["seed"])
    A = 0.3 * torch.randn(T, B, n + m, n + m, generator=g)
    C = A @ A.transpose(-1, -2) + torch.eye(n + m)
    c = torch.randn(T, B, n + m, generator=g)
    if name == "pendulum":
        th = (torch.rand(B, generator=g) * 2 - 1) * 0.6
        x0 = torch.stack((th.cos(), th.sin(), torch.rand(B, generator=g) - 0.5), 1)
        w = 0.02 * torch.randn(steps, B, n, generator=g)
    else:
        x0 = torch.randn(B, n, generator=g)
        w = torch.zeros(steps, B, n)
    wx = torch.randn(steps + 1, B, n, generator=g)
    wu = torch.randn(steps, B, m, generator=g)
    inputs = dict(x_init=x0, C=C, c=c, w=w)
    for i, fc in enumerate(net0.fcs):
        inputs[f"W{i}"], inputs[f"b{i}"] = 0.5 * fc.weight.detach().clone(), fc.bias.detach().clone()
    nl = len(net0.fcs)
    names = ["x_init", "C", "c", "w"] + [f"{k}{i}" for i in range(nl) for k in ("W", "b")]
    if name == "pendulum":
        inputs["params"] = torch.tensor((10.0, 1.0, 1.0))
        names.append("params")

    def run(ins):
        leaves = {k: v.clone().requires_grad_(True) for k, v in ins.items()}
        net = rdyn.NNDynamics(n, m, hidden_sizes=cf["hidden"], activation="sigmoid", passthrough=True).double()
        for i, fc in enumerate(net.fcs):           # the leaves themselves, so autograd reaches them
            del fc.weight, fc.bias
            fc.weight, fc.bias = leaves[f"W{i}"], leaves[f"b{i}"]
        net.Ws = [fc.weight for fc in net.fcs]     # grad_input reads the list taken at construction
        if name == "pendulum":
            penv = load_ref_env("pendulum")
            plant = penv.PendulumDx(params=leaves["params"], simple=True)
            plant.max_torque, plant.lower, plant.upper = bound, -bound, bound
        else:
            plant = net

        def make(u_init, prev):
            return rmpc.MPC(n, m, T, u_init=u_init, u_lower=-bound, u_upper=bound, lqr_iter=cf["lqr_iter"],
                            verbose=0, exit_unconverged=False, detach_unconverged=False, eps=cf["eps"],
                            grad_method=rmpc.GradMethods.ANALYTIC)
        return closed_loop(rmpc, make, leaves, lambda lv: (rmpc.QuadCost(lv["C"], lv["c"]), net), plant, steps, wx,
                           wu, names)
    extra = dict(T=np.int64(T), n_steps=np.int64(steps), lqr_iter=np.int64(cf["lqr_iter"]), eps=np.float64(cf["eps"]),
                 bound=np.float64(bound), n_layers=np.int64(nl))
    return inputs, wx, wu, run, extra


def main():
    rmpc, _, _, _ = load_reference()
    import ref_mpc.dynamics as rdyn
    torch.set_default_dtype(torch.float64)
    out = {}
    for name in CASES:
        inputs, wx, wu, run, extra = case(rmpc, rdyn, name)
        xs, us, px, pu, g, iters = guarded(run, inputs, name)
        print(name, "iterations", iters.tolist(), "plan controls on the bound",
              int((pu.abs() == float(extra["bound"])).sum()), "of", pu.numel())
        pre = name + "_"
        out.update({pre + k: v for k, v in inputs.items()})
        out.update({pre + "wx": wx, pre + "wu": wu, pre + "x": xs, pre + "u": us, pre + "iters": iters,
                    pre + "plan_x": px, pre + "plan_u": pu})
        out.update({pre + k: v for k, v in extra.items()})
        out.update({pre + "g_" + k: v for k, v in g.items()})
    npz("receding_nn_f64", **out)


if __name__ == "__main__":
    main()
