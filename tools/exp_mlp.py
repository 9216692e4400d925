#!/usr/bin/env python3
"""MPC.forward + .backward() with a learned model (NNDynamics), this tree against another built tree of the project
(--parent), alternated in worker processes (measure.alternate).  In this tree the iLQR iterations run as one CUDA
graph with the network's kernels (mpcb200_ilqr_mlp_*); a tree without them runs the network from Python.

  python tools/exp_mlp.py --parent TREE [--reps 3] [--rounds 2] [--out DIR]

Workloads (lqr_iter=50, eps=1e-2, ANALYTIC, a passthrough network with seeded weights, cost diag(Q) x + p;
loss = sum(x) + sum(u) backpropagated to the weights):
  fixture   B=4,   T=8,  (3, 2), [12, 10], +-0.6  (the reference fixtures' size)
  pendulum  B=16,  T=20, (3, 1), [100],    +-2    (the pendulum notebook's size)
  config2   B=128, T=25, (5, 1), [100],    +-100  (BASELINE config 2's size)
  float32, and the pendulum row again in float64.  Prints one JSON line per workload: median ms per forward +
backward for each tree, the iterations each ran, and the largest relative difference of x and u."""
import argparse
import json
import statistics
import sys

import measure

ROWS = {"fixture": (4, 8, 3, 2, [12, 10], 0.6, "float32"), "pendulum": (16, 20, 3, 1, [100], 2.0, "float32"),
        "config2": (128, 25, 5, 1, [100], 100.0, "float32"), "pendulum_f64": (16, 20, 3, 1, [100], 2.0, "float64")}


def case(name):
    import torch
    from mpc.pytorch_b200.models import NNDynamics
    from mpc.pytorch_b200.solver import MPC, GradMethods, QuadCost
    B, T, n, m, hidden, bound, dt = ROWS[name]
    dtype, dev = getattr(torch, dt), torch.device("cuda:0")
    torch.manual_seed(0)
    net = NNDynamics(n, m, hidden_sizes=hidden).to(dtype=dtype, device=dev)
    g = torch.Generator().manual_seed(1)
    q = torch.cat((torch.ones(n), 0.1 * torch.ones(m))).to(dtype)
    C = torch.diag(q).expand(T, B, n + m, n + m).contiguous().to(dev)
    c = (0.5 * torch.randn(T, B, n + m, generator=g)).to(dtype=dtype, device=dev)
    x0 = torch.randn(B, n, generator=g).to(dtype=dtype, device=dev)
    ctrl = MPC(n, m, T, u_lower=-bound, u_upper=bound, lqr_iter=50, eps=1e-2, verbose=-1,
               grad_method=GradMethods.ANALYTIC, exit_unconverged=False, detach_unconverged=False)
    return ctrl, x0, QuadCost(C, c), net


def worker(tree, out, save, reps):
    measure.enter(tree)
    import torch
    times, info, outputs = {}, {}, {}
    for name in ROWS:
        ctrl, x0, cost, net = case(name)

        def one():
            net.zero_grad()
            x, u, _ = ctrl(x0, cost, net)
            (x.sum() + u.sum()).backward()
            return x.detach(), u.detach()
        one()
        ts, (x, u) = measure.host_time(one, reps)
        times[name] = ts
        info[name] = {"iterations": int(ctrl._solve_info[0])}
        outputs[name] = {"x": x, "u": u, "dW0": net.fcs[0].weight.grad.detach()}
    measure.save(out, times, info, outputs if save else None)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=3)
    measure.add_arguments(ap, rounds=2)
    a = ap.parse_args()
    if a.worker:
        tree, out, save = a.worker
        return worker(tree, out, save == "1", a.reps)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    c = measure.card()
    arms = {k: (t, {}) for k, t in measure.trees(a.parent).items()}
    times, info, outs = measure.alternate(__file__, arms, a.rounds, ["--reps", str(a.reps)])
    rows = []
    for name in ROWS:
        row = {"workload": name, "dtype": ROWS[name][-1]}
        for arm in arms:
            row[f"{arm}_ms"] = round(1e3 * statistics.median(times[arm][name]), 2)
            row[f"{arm}_iterations"] = info[arm][name]["iterations"]
        if "parent" in arms:
            for k in ("x", "u", "dW0"):
                mine, theirs = outs["this"][name][k].double(), outs["parent"][name][k].double()
                row[f"{k}_max_rel_diff"] = float((mine - theirs).abs().max() / max(1e-30, float(theirs.abs().max())))
        rows.append(row)
        print(json.dumps(row), flush=True)
    measure.report(a.out, __file__, c, rows, {arm: times[arm] for arm in arms}, reps=a.reps, rounds=a.rounds)


if __name__ == "__main__":
    sys.exit(main())
