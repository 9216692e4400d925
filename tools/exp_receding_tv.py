#!/usr/bin/env python3
"""Receding-horizon episodes with a moving set point (a time-varying c on the episode's axis, time_varying=True):
the Python loop over MPC.forward with per-step slices (what a user writes without the window entries), the windowed
graph, and the time-invariant graph on the same sizes (its first window for every solve), so that the per-step window
copy shows as its own cost.  Forward alone, and forward + .backward(), alternated in one process.

  python tools/exp_receding_tv.py [--reps 5] [--steps 100] [--out DIR]

Episodes (float32, the notebooks' solver options, as tools/exp_receding.py; x_init, C and c require grad in the
timed backward; loss = sum(x) + sum(u)):
  cartpole  B=8,   T=25  the cart's set point steps from 0 to 0.5 half way along the axis
  pendulum  B=16,  T=20  the goal angle moves as 0.4 sin(0.1 t)
  config2   B=128, T=25  the cartpole case at BASELINE config 2's size
Prints one JSON line per episode: medians over --reps alternated repetitions of measure.host_time (ms per episode),
and whether the loop's and the windowed graph's x and u are bitwise equal; and the card (measure.card); with --out DIR,
also writes them to DIR/exp_receding_tv.json."""
import argparse
import json
import statistics

import torch

import measure
from exp_receding import _case
from mpc.pytorch_b200 import control
from mpc.pytorch_b200.dynamics import params_scope


def moving(name, cost, L):
    """C, c on the axis of L slices: C the notebook's (stride-0 over time), c = p - Q goal(t)."""
    C0, p = cost.C[0], cost.c[0]
    t = torch.arange(L, dtype=C0.dtype, device=C0.device)
    goal = torch.zeros(L, *p.shape, dtype=C0.dtype, device=C0.device)
    if name == "pendulum":
        ang = 0.4 * torch.sin(0.1 * t)
        goal[:, :, 0], goal[:, :, 1] = ang.cos()[:, None], ang.sin()[:, None]
    else:
        goal[:, :, 0] = (0.5 * (t > L / 2).to(C0.dtype))[:, None]
        goal[:, :, 2] = 1.0
    C = C0.expand(L, *C0.shape)
    c = p - (C @ goal.unsqueeze(-1)).squeeze(-1)
    return C, c


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--out", default=None, help="directory for exp_receding_tv.json (default: print only)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    c = measure.card()
    rows = []
    for name, B, T in (("cartpole", 8, 25), ("pendulum", 16, 20), ("config2", 128, 25)):
        ctrl, x0, cost, dx = _case(name, B, T)
        L = a.steps + T - 1
        C, cc = moving(name, cost, L)

        def episode(arm, grad):
            lv = [t.detach().clone().requires_grad_(grad) for t in (x0, C, cc)]
            cst = control.QuadCost(lv[1], lv[2])
            if arm == "loop":
                w0 = control._first_warm_start(ctrl, lv[0])
                with params_scope(), torch.set_grad_enabled(grad):
                    ep = control._episode_host(ctrl, lv[0], cst, dx, a.steps, w0, None, None, L)
            elif arm == "window":
                ep = control.receding_horizon(ctrl, lv[0], cst, dx, a.steps, differentiable=grad, time_varying=True)
            else:
                ep = control.receding_horizon(ctrl, lv[0], control.QuadCost(lv[1][:T], lv[2][:T]), dx, a.steps,
                                              differentiable=grad)
            return ep

        def timed(arm, grad):
            def run():
                ep = episode(arm, grad)
                if grad:
                    (ep.x.sum() + ep.u.sum()).backward()
                return ep
            return run
        arms = ("loop", "window", "ti")
        outs = {arm: measure.host_time(timed(arm, False), 1)[1] for arm in arms}     # warm-up of each
        for arm in arms:
            measure.host_time(timed(arm, True), 1)
        same = bool(torch.equal(outs["loop"].x, outs["window"].x) and torch.equal(outs["loop"].u, outs["window"].u))
        fw = {arm: [] for arm in arms}
        fb = {arm: [] for arm in arms}
        for _ in range(a.reps):                               # alternated
            for arm in arms:
                fw[arm] += measure.host_time(timed(arm, False), 1)[0]
                fb[arm] += measure.host_time(timed(arm, True), 1)[0]
        med = {f"{arm}_{kind}_ms": 1e3 * statistics.median(d[arm]) for arm in arms
               for kind, d in (("forward", fw), ("fwd_bwd", fb))}
        row = dict(episode=name, B=B, T=T, steps=a.steps, L=L, loop_window_bitwise=same, **med,
                   forward_speedup=med["loop_forward_ms"] / med["window_forward_ms"],
                   fwd_bwd_speedup=med["loop_fwd_bwd_ms"] / med["window_fwd_bwd_ms"],
                   window_over_ti_forward=med["window_forward_ms"] / med["ti_forward_ms"],
                   window_over_ti_fwd_bwd=med["window_fwd_bwd_ms"] / med["ti_fwd_bwd_ms"],
                   forward_s_all=fw, fwd_bwd_s_all=fb)
        rows.append(row)
        print(json.dumps({k: v for k, v in row.items() if not k.endswith("_all")}), flush=True)
    measure.report(a.out, __file__, c, rows, {r["episode"]: dict(forward_s=r["forward_s_all"],
                                                                 fwd_bwd_s=r["fwd_bwd_s_all"]) for r in rows},
                   steps=a.steps, reps=a.reps)


if __name__ == "__main__":
    main()
