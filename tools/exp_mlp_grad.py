#!/usr/bin/env python3
"""The gradient to a learned model's weights: MPC.forward + loss.backward() with an NNDynamics, this tree against
another built tree of the project (--parent), alternated in worker processes (measure.alternate).  In this tree the
differentiable tail's linearisation is MlpLinearize, whose backward is the VJP kernel (mpcb200_mlp_linearize_vjp_*);
a tree without it builds the tail from grad_input under autograd and double-differentiates it.

  python tools/exp_mlp_grad.py --parent TREE [--reps 5] [--rounds 2] [--out DIR]

Workloads (lqr_iter=50, eps=1e-2, a passthrough network with seeded weights, cost diag(Q) x + p; loss = sum(x) +
sum(u) backpropagated to every weight and bias):
  fixture      B=4,    T=8,  (3, 2), [12, 10], +-0.6  (the reference fixtures' size)
  pendulum     B=16,   T=20, (3, 1), [100],    +-2    (the pendulum notebook's size)
  config2      B=128,  T=25, (5, 1), [100],    +-100  (BASELINE config 2's size)
  pendulum_f64 the pendulum row in float64
  pendulum_ad  the pendulum row under AUTO_DIFF
  large        B=1024, T=25, (5, 1), [100],    +-100
  float32 unless named.  Prints one JSON line per workload: the median ms of backward() alone (CUDA events around a
backward between two synchronisations) and of forward + backward for each tree, and the largest relative difference
of each parameter's gradient (|this - parent| max over max |parent|)."""
import argparse
import json
import statistics
import sys

import measure

ROWS = {"fixture": (4, 8, 3, 2, [12, 10], 0.6, "float32", "ANALYTIC"),
        "pendulum": (16, 20, 3, 1, [100], 2.0, "float32", "ANALYTIC"),
        "config2": (128, 25, 5, 1, [100], 100.0, "float32", "ANALYTIC"),
        "pendulum_f64": (16, 20, 3, 1, [100], 2.0, "float64", "ANALYTIC"),
        "pendulum_ad": (16, 20, 3, 1, [100], 2.0, "float32", "AUTO_DIFF"),
        "large": (1024, 25, 5, 1, [100], 100.0, "float32", "ANALYTIC")}


def case(name):
    import torch
    from mpc.pytorch_b200.models import NNDynamics
    from mpc.pytorch_b200.solver import MPC, GradMethods, QuadCost
    B, T, n, m, hidden, bound, dt, gm = ROWS[name]
    dtype, dev = getattr(torch, dt), torch.device("cuda:0")
    torch.manual_seed(0)
    net = NNDynamics(n, m, hidden_sizes=hidden).to(dtype=dtype, device=dev)
    g = torch.Generator().manual_seed(1)
    q = torch.cat((torch.ones(n), 0.1 * torch.ones(m))).to(dtype)
    C = torch.diag(q).expand(T, B, n + m, n + m).contiguous().to(dev)
    c = (0.5 * torch.randn(T, B, n + m, generator=g)).to(dtype=dtype, device=dev)
    x0 = torch.randn(B, n, generator=g).to(dtype=dtype, device=dev)
    ctrl = MPC(n, m, T, u_lower=-bound, u_upper=bound, lqr_iter=50, eps=1e-2, verbose=-1,
               grad_method=getattr(GradMethods, gm), exit_unconverged=False, detach_unconverged=False)
    return ctrl, x0, QuadCost(C, c), net


def worker(tree, out, save, reps):
    measure.enter(tree)
    import torch
    times, info, outputs = {}, {}, {}
    for name in ROWS:
        ctrl, x0, cost, net = case(name)
        bwd = []

        def one():
            net.zero_grad()
            x, u, _ = ctrl(x0, cost, net)
            loss = x.sum() + u.sum()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            loss.backward()
            e1.record()
            torch.cuda.synchronize()
            bwd.append(e0.elapsed_time(e1) / 1e3)
            return x.detach(), u.detach()
        one()
        bwd.clear()
        ts, _ = measure.host_time(one, reps)
        times[name + ":backward"] = bwd
        times[name + ":forward_backward"] = ts
        info[name] = {"iterations": int(ctrl._solve_info[0])}
        outputs[name] = {f"{k}{i}": getattr(fc, k).grad.detach() for i, fc in enumerate(net.fcs)
                         for k in ("weight", "bias")}
    measure.save(out, times, info, outputs if save else None)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=5)
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
        row = {"workload": name, "dtype": ROWS[name][6], "grad_method": ROWS[name][7]}
        for arm in arms:
            for part in ("backward", "forward_backward"):
                row[f"{arm}_{part}_ms"] = round(1e3 * statistics.median(times[arm][f"{name}:{part}"]), 3)
            row[f"{arm}_iterations"] = info[arm][name]["iterations"]
        if "parent" in arms:
            for k, mine in outs["this"][name].items():
                theirs = outs["parent"][name][k].double()
                row[f"d{k}_max_rel_diff"] = float((mine.double() - theirs).abs().max() /
                                                  max(1e-30, float(theirs.abs().max())))
        rows.append(row)
        print(json.dumps(row), flush=True)
    measure.report(a.out, __file__, c, rows, {arm: times[arm] for arm in arms}, reps=a.reps, rounds=a.rounds)


if __name__ == "__main__":
    sys.exit(main())
