#!/usr/bin/env python3
"""Differentiable receding-horizon episodes closed on a plant other than the model, with process disturbances:
forward + .backward() on the device path (one graph for the episode, one for its reverse sweep) against the host path
(the Python loop of MPC.forward, the plant stepped by the same kernels, autograd recording), alternated in one process,
gradients checked against each other.

  python tools/exp_receding_plant.py [--reps 5] [--steps 100] [--out DIR]

Episodes (float32, the notebooks' solver options, as tools/exp_receding.py; x_init, C, c, the model's and the plant's
params and w require grad; w = 0.01 N(0, 1), seeded; loss = sum(x) + sum(u)):
  pendulum  B=16,  T=20  PendulumDx() model on PendulumDx(simple=False, params=(10, 1, 1, 0.3, 0.2))
  cartpole  B=8,   T=25  CartpoleDx() model on CartpoleDx(params=(9.8, 1.2, 0.12, 0.55))
  config2   B=128, T=25  the cartpole pair at BASELINE config 2's size
Prints one JSON line per episode (ms per episode for forward + backward, median over --reps alternated repetitions of
measure.host_time after one warm-up of each, the backward alone timed the same way, and the largest relative gradient
difference) and the card (measure.card); with --out DIR, also writes them to DIR/exp_receding_plant.json."""
import argparse
import json
import statistics

import torch

import measure
from exp_receding import _case
from mpc.pytorch_b200 import control
from mpc.pytorch_b200.dynamics import CartpoleDx, PendulumDx, params_scope

DEV = torch.device("cuda:0")
PLANTS = {"pendulum": lambda: PendulumDx(params=torch.tensor((10.0, 1.0, 1.0, 0.3, 0.2)), simple=False),
          "cartpole": lambda: CartpoleDx(params=torch.tensor((9.8, 1.2, 0.12, 0.55))),
          "config2": lambda: CartpoleDx(params=torch.tensor((9.8, 1.2, 0.12, 0.55)))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--out", default=None, help="directory for exp_receding_plant.json (default: print only)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    c = measure.card()
    rows = []
    for name, B, T in (("pendulum", 16, 20), ("cartpole", 8, 25), ("config2", 128, 25)):
        ctrl, x0, cost, dx = _case(name, B, T)
        plant = PLANTS[name]()
        n = x0.shape[1]
        w = 0.01 * torch.randn(a.steps, B, n, generator=torch.Generator().manual_seed(1)).to(DEV)
        mparams, pparams = dx.params.to(DEV), plant.params.to(DEV)

        def leaves():
            return [t.detach().clone().requires_grad_(True) for t in (x0, cost.C, cost.c, mparams, pparams, w)]

        def forward(host):
            lv = leaves()
            dx.params, plant.params = lv[3], lv[4]
            cst = control.QuadCost(lv[1], lv[2])
            if host:
                w0 = control._first_warm_start(ctrl, lv[0])
                with params_scope():
                    ep = control._episode_host(ctrl, lv[0], cst, dx, a.steps, w0, plant, lv[5])
            else:
                ep = control.receding_horizon(ctrl, lv[0], cst, dx, a.steps, differentiable=True, plant=plant,
                                              disturbance=lv[5])
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
        rel = max(float((d - h).abs().max()) / max(1e-30, float(h.abs().max())) for d, h in zip(g_dev, g_host))
        t_host, t_dev, b_host, b_dev = [], [], [], []
        for _ in range(a.reps):                               # alternated
            t_host += measure.host_time(both(True), 1)[0]
            t_dev += measure.host_time(both(False), 1)[0]
            b_host += backward_only(True)
            b_dev += backward_only(False)
        mh, md = statistics.median(t_host), statistics.median(t_dev)
        row = dict(episode=name, B=B, T=T, steps=a.steps, plant=type(plant).__name__, max_rel_grad_diff=rel,
                   host_ms=1e3 * mh, device_ms=1e3 * md, speedup=mh / md,
                   host_backward_ms=1e3 * statistics.median(b_host), device_backward_ms=1e3 * statistics.median(b_dev),
                   host_s_all=t_host, device_s_all=t_dev)
        rows.append(row)
        print(json.dumps(row), flush=True)
    measure.report(a.out, __file__, c, rows, {r["episode"]: dict(host_s=r["host_s_all"], device_s=r["device_s_all"])
                                              for r in rows}, steps=a.steps, reps=a.reps)


if __name__ == "__main__":
    main()
