#!/usr/bin/env python3
"""Receding-horizon episodes planned with a learned model (NNDynamics): the device path (mpcb200_episode_mlp_* for the
episode, mpcb200_episode_backward_mlp_* for its reverse sweep) against the host path (the Python loop of MPC.forward,
the network stepped by its torch Module, autograd recording), alternated in one process, forward alone and
forward + .backward(), outputs and gradients checked against each other.

  python tools/exp_receding_mlp.py [--reps 3] [--steps 100] [--out DIR]

Episodes (float32, GradMethods.ANALYTIC, lqr_iter 10, seeded weights; x_init, C, c and every weight and bias require
grad; loss = sum(x) + sum(u)):
  fixtures  B=4,   T=8,  (n, m) = (3, 2), hidden [12, 10], the network steps the loop, u in [-1, 1]
  pendulum  B=16,  T=20, (3, 1), hidden [100], planning for the known pendulum (PendulumDx, params (10, 1, 1)), which
            steps the loop, u in [-2, 2] (the pendulum notebook's size)
  config2   B=128, T=25, (5, 1), hidden [100], the network steps the loop, u in [-1, 1] (BASELINE config 2's size)
Prints one JSON line per episode: ms per episode (median over --reps alternated repetitions of measure.host_time
after one warm-up of each) for the forward and for forward + backward on both paths, the largest relative difference
of x and of the gradients; and the card (measure.card).  With --out DIR, also writes DIR/exp_receding_mlp.json."""
import argparse
import contextlib
import json
import statistics

import torch

import measure
from mpc.pytorch_b200 import control, mlp
from mpc.pytorch_b200.dynamics import PendulumDx
from mpc.pytorch_b200.models import NNDynamics
from mpc.pytorch_b200.solver import MPC, GradMethods, QuadCost

DEV = torch.device("cuda:0")
CASES = (("fixtures", 4, 8, 3, 2, [12, 10], 1.0, False), ("pendulum", 16, 20, 3, 1, [100], 2.0, True),
         ("config2", 128, 25, 5, 1, [100], 1.0, False))


def _case(B, T, n, m, hidden, bound, pendulum, seed=0):
    torch.manual_seed(seed)
    net = NNDynamics(n, m, hidden_sizes=hidden).to(DEV)
    with torch.no_grad():
        for fc in net.fcs:
            fc.weight.mul_(0.5)
    g = torch.Generator().manual_seed(seed + 1)
    A = 0.3 * torch.randn(T, B, n + m, n + m, generator=g)
    C = (A @ A.transpose(-1, -2) + torch.eye(n + m)).to(DEV)
    c = torch.randn(T, B, n + m, generator=g).to(DEV)
    if pendulum:
        th = (torch.rand(B, generator=g) * 2 - 1) * 0.6
        x0 = torch.stack((th.cos(), th.sin(), torch.rand(B, generator=g) - 0.5), 1).to(DEV)
    else:
        x0 = torch.randn(B, n, generator=g).to(DEV)
    ctrl = MPC(n, m, T, u_lower=-bound, u_upper=bound, lqr_iter=10, verbose=-1, grad_method=GradMethods.ANALYTIC,
               exit_unconverged=False, detach_unconverged=False)
    plant = PendulumDx(params=torch.tensor((10.0, 1.0, 1.0), device=DEV)) if pendulum else None
    return ctrl, x0, C, c, net, plant


@contextlib.contextmanager
def host_path(on):
    """With `on`, mlp.episode_on_device refuses every episode, so receding_horizon runs its host loop."""
    real = mlp.episode_on_device
    if on:
        mlp.episode_on_device = lambda *a, **k: False
    try:
        yield
    finally:
        mlp.episode_on_device = real


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--out", default=None, help="directory for exp_receding_mlp.json (default: print only)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    c = measure.card()
    rows, runs = [], {}
    for name, B, T, n, m, hidden, bound, pendulum in CASES:
        ctrl, x0, C, cc, net, plant = _case(B, T, n, m, hidden, bound, pendulum)
        weights = [t for fc in net.fcs for t in (fc.weight, fc.bias)]

        def forward(host, grad):
            lv = [t.detach().clone().requires_grad_(grad) for t in (x0, C, cc)]
            for t in weights:
                t.requires_grad_(grad)
                t.grad = None
            with host_path(host):
                ep = control.receding_horizon(ctrl, lv[0], QuadCost(lv[1], lv[2]), net, a.steps,
                                              differentiable=grad, plant=plant)
            return lv, ep

        def fwd(host):
            return lambda: forward(host, False)[1].x

        def both(host):
            def run():
                lv, ep = forward(host, True)
                (ep.x.sum() + ep.u.sum()).backward()
                return [t.grad.clone() for t in lv + weights]
            return run
        x_h = measure.host_time(fwd(True), 1)[1]              # warm-up of each
        x_d = measure.host_time(fwd(False), 1)[1]
        g_h = measure.host_time(both(True), 1)[1]
        g_d = measure.host_time(both(False), 1)[1]
        rel_x = float((x_d - x_h).abs().max()) / max(1.0, float(x_h.abs().max()))
        rel_g = max(float((d - h).abs().max()) / max(1e-30, float(h.abs().max())) for d, h in zip(g_d, g_h))
        f_h, f_d, t_h, t_d = [], [], [], []
        for _ in range(a.reps):                               # alternated
            f_h += measure.host_time(fwd(True), 1)[0]
            f_d += measure.host_time(fwd(False), 1)[0]
            t_h += measure.host_time(both(True), 1)[0]
            t_d += measure.host_time(both(False), 1)[0]
        ms = lambda v: 1e3 * statistics.median(v)            # noqa: E731
        row = dict(episode=name, B=B, T=T, n=n, m=m, hidden=hidden, steps=a.steps, plant="pendulum" if pendulum else
                   "network", max_rel_x_diff=rel_x, max_rel_grad_diff=rel_g, host_forward_ms=ms(f_h),
                   device_forward_ms=ms(f_d), forward_speedup=ms(f_h) / ms(f_d), host_fwd_bwd_ms=ms(t_h),
                   device_fwd_bwd_ms=ms(t_d), fwd_bwd_speedup=ms(t_h) / ms(t_d))
        rows.append(row)
        runs[name] = dict(host_forward_s=f_h, device_forward_s=f_d, host_fwd_bwd_s=t_h, device_fwd_bwd_s=t_d)
        print(json.dumps(row), flush=True)
    measure.report(a.out, __file__, c, rows, runs, steps=a.steps, reps=a.reps)


if __name__ == "__main__":
    main()
