#!/usr/bin/env python3
"""Differentiable receding-horizon episodes: forward + .backward() on the device path (one graph for the episode,
one graph for its reverse sweep) against the host path (the Python loop of MPC.forward with autograd recording),
alternated in one process, gradients checked against each other.

  python tools/exp_receding_grad.py [--reps 5] [--steps 100] [--slew] [--out DIR]

Episodes (float32, the notebooks' solver options, as tools/exp_receding.py; x_init, C, c and the system's params
require grad; loss = sum(x) + sum(u)):
  cartpole  B=8,   T=25
  pendulum  B=16,  T=20
  config2   B=128, T=25  (cartpole at BASELINE config 2's size)
Prints one JSON line per episode (ms per episode for forward + backward, median over --reps alternated repetitions of
measure.host_time after one warm-up of each, the backward alone timed the same way, and the largest relative gradient
difference) and the card (measure.card); with --out DIR, also writes them to DIR/exp_receding_grad.json.
--slew: the same episodes with slew_rate_penalty = 0.1 (the augmented problem over [u_{k-1}; x]); each row also
records the plan bits of the device backward's last nested adjoint step (mpcb200_last_step_plan: 16 = the large-shape
kernels), and the output file is exp_receding_grad_slew.json."""
import argparse
import json
import statistics

import torch

import measure
from exp_receding import _case
from mpc.pytorch_b200 import _lib, control

DEV = torch.device("cuda:0")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--slew", action="store_true", help="slew_rate_penalty = 0.1 on every episode")
    ap.add_argument("--out", default=None, help="directory for exp_receding_grad.json (default: print only)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    c = measure.card()
    rows = []
    for name, B, T in (("cartpole", 8, 25), ("pendulum", 16, 20), ("config2", 128, 25)):
        ctrl, x0, cost, dx = _case(name, B, T)
        dx.params = dx.params.to(DEV)
        if a.slew:
            ctrl.slew_rate_penalty = 0.1

        def leaves():
            return [t.detach().clone().requires_grad_(True) for t in (x0, cost.C, cost.c, dx.params)]

        def forward(host):
            lv = leaves()
            dx.params = lv[3]
            if host:
                w0 = control._first_warm_start(ctrl, lv[0])
                from mpc.pytorch_b200.dynamics import params_scope
                with params_scope():
                    ep = control._episode_host(ctrl, lv[0], control.QuadCost(lv[1], lv[2]), dx, a.steps, w0)
            else:
                ep = control.receding_horizon(ctrl, lv[0], control.QuadCost(lv[1], lv[2]), dx, a.steps,
                                              differentiable=True)
            return lv, ep.x.sum() + ep.u.sum()

        def both(host):
            def run():
                lv, loss = forward(host)
                loss.backward()
                return [t.grad for t in lv]
            return run

        def backward_only(host):
            _, loss = forward(host)
            return measure.host_time(loss.backward, 1)[0]
        g_host = measure.host_time(both(True), 1)[1]          # warm-up of both
        g_dev = measure.host_time(both(False), 1)[1]
        plan = _lib.last_step_plan()
        rel = max(float((d - h).abs().max()) / max(1e-30, float(h.abs().max())) for d, h in zip(g_dev, g_host))
        t_host, t_dev, b_host, b_dev = [], [], [], []
        for _ in range(a.reps):                               # alternated
            t_host += measure.host_time(both(True), 1)[0]
            t_dev += measure.host_time(both(False), 1)[0]
            b_host += backward_only(True)
            b_dev += backward_only(False)
        mh, md = statistics.median(t_host), statistics.median(t_dev)
        row = dict(episode=name, B=B, T=T, steps=a.steps, max_rel_grad_diff=rel,
                   host_ms=1e3 * mh, device_ms=1e3 * md, speedup=mh / md,
                   host_backward_ms=1e3 * statistics.median(b_host), device_backward_ms=1e3 * statistics.median(b_dev),
                   host_s_all=t_host, device_s_all=t_dev)
        if a.slew:
            row.update(slew_rate_penalty=0.1, adjoint_plan=plan)
        rows.append(row)
        print(json.dumps(row), flush=True)
    measure.report(a.out, __file__.replace(".py", "_slew.py") if a.slew else __file__, c, rows, {r["episode"]: dict(host_s=r["host_s_all"], device_s=r["device_s_all"])
                                              for r in rows}, steps=a.steps, reps=a.reps)


if __name__ == "__main__":
    main()
