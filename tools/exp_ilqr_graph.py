"""MPC.forward per solve with the iLQR loop on the host (one host round trip per iteration) and on the device (one CUDA
graph with a conditional `while` node, mpcb200_ilqr_*), alternating, several runs each; host clock around a
synchronise.  Also reports the host time of the library call that builds, instantiates and launches the graph, the
iterations run, and checks in the same run that both loops give bitwise equal x, u and costs.

    python tools/exp_ilqr_graph.py [--reps 5] [--rounds 3]
"""
import argparse
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from mpc.pytorch_b200 import solver, step  # noqa: E402
from mpc.pytorch_b200.dynamics import CartpoleDx, PendulumDx  # noqa: E402
from mpc.pytorch_b200.solver import MPC, GradMethods, LinDx, QuadCost  # noqa: E402
from tests.cartpole import initial_states  # noqa: E402
from tests.helpers import gen_problem  # noqa: E402

DEV = torch.device("cuda:0")


def config2():
    """tools/exp_cartpole.py: cartpole B=128, T=25, +-100, <= 50 iterations, eps 1e-2, AUTO_DIFF, float32."""
    dx = CartpoleDx()
    B, T = 128, 25
    q, p = dx.get_true_obj()
    cost = QuadCost(torch.diag(q).expand(T, B, 6, 6).contiguous().to(DEV), p.expand(T, B, 6).contiguous().to(DEV))
    ctrl = MPC(5, 1, T, u_lower=dx.lower, u_upper=dx.upper, lqr_iter=50, verbose=-1, exit_unconverged=False,
               detach_unconverged=False, linesearch_decay=dx.linesearch_decay,
               max_linesearch_iter=dx.max_linesearch_iter, grad_method=GradMethods.AUTO_DIFF, eps=1e-2)
    return ctrl, initial_states(B, seed=0).to(DEV), cost, dx


def pendulum():
    dx = PendulumDx()
    B, T = 128, 20
    q, p = dx.get_true_obj()
    cost = QuadCost(torch.diag(q).expand(T, B, 4, 4).contiguous().to(DEV), p.expand(T, B, 4).contiguous().to(DEV))
    th = torch.linspace(-3.0, 3.0, B)
    x0 = torch.stack((th.cos(), th.sin(), torch.zeros(B)), 1).to(DEV)
    ctrl = MPC(3, 1, T, u_lower=dx.lower, u_upper=dx.upper, lqr_iter=50, verbose=-1, exit_unconverged=False,
               detach_unconverged=False, linesearch_decay=dx.linesearch_decay,
               max_linesearch_iter=dx.max_linesearch_iter, grad_method=GradMethods.AUTO_DIFF, eps=dx.mpc_eps)
    return ctrl, x0, cost, dx


def linear(B, T, bound, lqr_iter):
    C, c, F, f, x0 = [t.to(DEV) for t in gen_problem(0, B, T, 8, 2, torch.float32)]
    kw = dict(u_lower=-bound, u_upper=bound) if bound else {}
    ctrl = MPC(8, 2, T, lqr_iter=lqr_iter, verbose=-1, exit_unconverged=False, detach_unconverged=False, **kw)
    return ctrl, x0, QuadCost(C, c), LinDx(F, f)


WORKLOADS = {
    "config 2: cartpole B=128 T=25 <=50 it": config2,
    "pendulum B=128 T=20 <=50 it": pendulum,
    "LinDx (8,2) B=1024 T=20 +-0.25, 10 it (config-4 size)": lambda: linear(1024, 20, 0.25, 10),
    "LinDx (8,2) config 3 unbounded, 3 it": lambda: linear(128, 20, None, 3),
}


def run(ctrl, x0, cost, dx, device_loop, reps, call_times, iters):
    orig_pred, orig_raw = solver._use_device_loop, step.ilqr_raw

    def spy(*a, **k):
        t0 = time.perf_counter()
        res = orig_raw(*a, **k)
        call_times.append(time.perf_counter() - t0)
        iters.append(res["info"])
        return res
    solver._use_device_loop = (lambda *a: True) if device_loop else (lambda *a: False)
    step.ilqr_raw = spy
    try:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        with torch.no_grad():
            for _ in range(reps):
                out = ctrl(x0, cost, dx)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / reps, out
    finally:
        solver._use_device_loop, step.ilqr_raw = orig_pred, orig_raw


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    name = torch.cuda.get_device_name(DEV)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    print(f"device: {name}, power limit {power}; torch {torch.__version__}, CUDA {torch.version.cuda}")
    for label, make in WORKLOADS.items():
        ctrl, x0, cost, dx = make()
        assert solver._use_device_loop(ctrl, x0, cost, dx,
                                       torch.zeros(ctrl.T, x0.shape[0], ctrl.n_ctrl, device=DEV)), label
        _, host_out = run(ctrl, x0, cost, dx, False, 1, [], [])          # warm-up, and the bitwise check
        calls, iters = [], []
        _, dev_out = run(ctrl, x0, cost, dx, True, 1, calls, iters)
        same = all(torch.equal(a, b) for a, b in zip(host_out, dev_out))
        host_t, dev_t, calls = [], [], []
        for _ in range(args.rounds):
            host_t.append(run(ctrl, x0, cost, dx, False, args.reps, [], [])[0])
            dev_t.append(run(ctrl, x0, cost, dx, True, args.reps, calls, iters)[0])
        h, d = statistics.median(host_t), statistics.median(dev_t)
        it = int(iters[-1][0])
        print(f"{label}: host loop {h * 1e3:.2f} ms, device loop {d * 1e3:.2f} ms per solve "
              f"(x{h / d:.1f}); {it} iterations; graph build+instantiate+launch call {statistics.median(calls) * 1e3:.3f}"
              f" ms; runs host {[round(t * 1e3, 2) for t in host_t]} device {[round(t * 1e3, 2) for t in dev_t]}; "
              f"bitwise equal: {same}", flush=True)


if __name__ == "__main__":
    main()
