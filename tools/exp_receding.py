#!/usr/bin/env python3
"""Receding-horizon episodes: a notebook-style Python loop of MPC.forward (each solve on the device loop, one graph
built per solve) against receding_horizon (one graph per episode), alternated in one process, outputs checked bitwise.

  python tools/exp_receding.py [--reps 5] [--steps 100] [--out DIR]

Episodes (float32, the notebooks' solver options: lqr_iter=50, eps=1e-2, AUTO_DIFF, bounds of the system):
  cartpole  B=8,   T=25  (the reference's cartpole notebook)
  pendulum  B=16,  T=20  (the reference's pendulum notebook, PendulumDx(params=(10, 1, 1)))
  config2   B=128, T=25  (cartpole at BASELINE config 2's size)
The loop is control._episode_host: per control step MPC.forward, the model step by the rollout kernel and the shift
of the warm start, as the notebooks do it.  Prints one JSON line per episode (ms per control step and per episode,
median over --reps alternated repetitions of measure.host_time, after one warm-up of each) and the card
(measure.card); with --out DIR, also writes them to DIR/exp_receding.json."""
import argparse
import json
import statistics

import torch

import measure
from mpc.pytorch_b200 import control
from mpc.pytorch_b200.dynamics import CartpoleDx, PendulumDx
from mpc.pytorch_b200.solver import MPC, GradMethods, QuadCost

DEV = torch.device("cuda:0")


def _case(name, B, T):
    sysdx = CartpoleDx() if name != "pendulum" else PendulumDx(params=torch.tensor((10.0, 1.0, 1.0)))
    n, m = sysdx.n_state, sysdx.n_ctrl
    q, p = sysdx.get_true_obj()
    Q = torch.diag(q).expand(T, B, n + m, n + m).contiguous().to(DEV)
    pp = p.expand(T, B, n + m).contiguous().to(DEV)
    g = torch.Generator().manual_seed(0)
    th = (torch.rand(B, generator=g) * 2 - 1) * (3.14159 if name != "pendulum" else 1.5708)
    if name == "pendulum":
        x0 = torch.stack((th.cos(), th.sin(), torch.rand(B, generator=g) * 2 - 1), 1)
    else:
        r = torch.rand(B, 3, generator=g) - 0.5
        x0 = torch.stack((r[:, 0], r[:, 1], th.cos(), th.sin(), r[:, 2]), 1)
    ctrl = MPC(n, m, T, u_lower=float(sysdx.lower), u_upper=float(sysdx.upper), lqr_iter=50, verbose=-1,
               linesearch_decay=sysdx.linesearch_decay, max_linesearch_iter=sysdx.max_linesearch_iter,
               grad_method=GradMethods.AUTO_DIFF, eps=1e-2, exit_unconverged=False, detach_unconverged=False)
    return ctrl, x0.to(DEV), QuadCost(Q, pp), sysdx


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--out", default=None, help="directory for exp_receding.json (default: print only)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    c = measure.card()
    rows = []
    for name, B, T in (("cartpole", 8, 25), ("pendulum", 16, 20), ("config2", 128, 25)):
        ctrl, x0, cost, dx = _case(name, B, T)
        w0 = control._first_warm_start(ctrl, x0)

        def loop():
            with torch.no_grad():
                return control._episode_host(ctrl, x0, cost, dx, a.steps, w0)

        def graph():
            return control.receding_horizon(ctrl, x0, cost, dx, a.steps)
        ref = measure.host_time(loop, 1)[1]            # warm-up of both
        got = measure.host_time(graph, 1)[1]
        same = all(torch.equal(getattr(got, k), getattr(ref, k).to(DEV)) for k in control.Episode._fields)
        t_loop, t_graph = [], []
        for _ in range(a.reps):                       # alternated
            t_loop += measure.host_time(loop, 1)[0]
            t_graph += measure.host_time(graph, 1)[0]
        ml, mg = statistics.median(t_loop), statistics.median(t_graph)
        row = dict(episode=name, B=B, T=T, steps=a.steps, bitwise_equal=same,
                   iterations=int(got.info[:, 0].sum()),
                   loop_ms_per_step=1e3 * ml / a.steps, graph_ms_per_step=1e3 * mg / a.steps,
                   loop_s=ml, graph_s=mg, speedup=ml / mg,
                   loop_s_all=t_loop, graph_s_all=t_graph)
        rows.append(row)
        print(json.dumps(row), flush=True)
    measure.report(a.out, __file__, c, rows, {r["episode"]: dict(loop_s=r["loop_s_all"], graph_s=r["graph_s_all"])
                                              for r in rows}, steps=a.steps, reps=a.reps)
    if not all(r["bitwise_equal"] for r in rows):
        raise SystemExit("receding_horizon differs from the loop")


if __name__ == "__main__":
    main()
