"""MPC.forward per solve with a slew-rate penalty: the iLQR loop on the host and on the device (one CUDA graph), and for
the known systems also today's route before the passthrough kind (the system wrapped as an opaque Module: split-mode
rollout, Module linearisation), alternating, several runs each; host clock around a synchronise.  Checks in the same
run that both loops give bitwise equal x, u and costs, prints the iterations each route ran in its last solve, and
the card name and power limit.

    python tools/exp_slew.py [--reps 5] [--rounds 3]
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
PENALTY = 0.1


class Opaque(torch.nn.Module):
    """The same physics without mpcb200_kind: the Module path the slew penalty took before."""

    def __init__(self, dx):
        super().__init__()
        self.dx = dx

    def forward(self, x, u):
        return self.dx(x, u)


def known(dx, n, B, T, x0, eps):
    q, p = dx.get_true_obj()
    cost = QuadCost(torch.diag(q).expand(T, B, n + 1, n + 1).contiguous().to(DEV),
                    p.expand(T, B, n + 1).contiguous().to(DEV))
    ctrl = MPC(n, 1, T, u_lower=dx.lower, u_upper=dx.upper, lqr_iter=50, verbose=-1, exit_unconverged=False,
               detach_unconverged=False, linesearch_decay=dx.linesearch_decay,
               max_linesearch_iter=dx.max_linesearch_iter, grad_method=GradMethods.AUTO_DIFF, eps=eps,
               slew_rate_penalty=PENALTY)
    return ctrl, x0.to(DEV), cost, dx


def config2():
    """config 2 (tools/exp_cartpole.py): cartpole B=128, T=25, +-100, <= 50 iterations, eps 1e-2, float32."""
    return known(CartpoleDx(), 5, 128, 25, initial_states(128, seed=0), 1e-2)


def pendulum():
    th = torch.linspace(-3.0, 3.0, 128)
    dx = PendulumDx()
    return known(dx, 3, 128, 20, torch.stack((th.cos(), th.sin(), torch.zeros(128)), 1), dx.mpc_eps)


def linear():
    C, c, F, f, x0 = [t.to(DEV) for t in gen_problem(0, 1024, 20, 8, 2, torch.float32)]
    ctrl = MPC(8, 2, 20, u_lower=-0.25, u_upper=0.25, lqr_iter=10, verbose=-1, exit_unconverged=False,
               detach_unconverged=False, slew_rate_penalty=PENALTY)
    return ctrl, x0, QuadCost(C, c), LinDx(F, f)


WORKLOADS = {
    "config 2 + slew: cartpole B=128 T=25 <=50 it": config2,
    "pendulum + slew: B=128 T=20 <=50 it": pendulum,
    "LinDx (8,2) + slew: B=1024 T=20 +-0.25, 10 it": linear,
}


def run(ctrl, x0, cost, dx, device_loop, reps):
    """(seconds per solve, outputs of the last solve, iterations of the last solve)."""
    orig, orig_raw, orig_sub = solver._use_slew_device_loop, step.ilqr_raw, MPC.solve_lqr_subproblem
    seen = {"info": None, "host": 0}

    def raw(*a, **k):
        res = orig_raw(*a, **k)
        seen["info"] = res["info"]
        return res

    def sub(self, *a, **k):
        if not k.get("no_op_forward", False):
            seen["host"] += 1
        return orig_sub(self, *a, **k)
    solver._use_slew_device_loop = orig if device_loop else (lambda *a: False)
    step.ilqr_raw, MPC.solve_lqr_subproblem = raw, sub
    try:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        with torch.no_grad():
            for _ in range(reps):
                seen["host"] = 0
                out = ctrl(x0, cost, dx)
        torch.cuda.synchronize()
        iters = int(seen["info"][0]) if device_loop else seen["host"]
        return (time.perf_counter() - t0) / reps, out, iters
    finally:
        solver._use_slew_device_loop, step.ilqr_raw, MPC.solve_lqr_subproblem = orig, orig_raw, orig_sub


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
        u0 = torch.zeros(ctrl.T, x0.shape[0], ctrl.n_ctrl, device=DEV)
        assert solver._use_slew_device_loop(ctrl, x0, cost, dx, u0), label
        routes = {"host loop": (dx, False), "device loop": (dx, True)}
        if not isinstance(dx, LinDx):
            routes["opaque Module (before)"] = (Opaque(dx), False)
        outs = {k: run(ctrl, x0, cost, d, dev, 1)[1] for k, (d, dev) in routes.items()}      # warm-up
        same = all(torch.equal(a, b) for a, b in zip(outs["host loop"], outs["device loop"]))
        times, iters = {k: [] for k in routes}, {}
        for _ in range(args.rounds):
            for k, (d, dev) in routes.items():
                t, _, iters[k] = run(ctrl, x0, cost, d, dev, args.reps)
                times[k].append(t)
        med = {k: statistics.median(v) for k, v in times.items()}
        d = med["device loop"]
        parts = [f"{k} {v * 1e3:.2f} ms (x{v / d:.1f} of device, {iters[k]} iterations)" for k, v in med.items()]
        runs = "; ".join(f"{k} {[round(t * 1e3, 2) for t in v]}" for k, v in times.items())
        print(f"{label}: " + ", ".join(parts) + f"; runs {runs}; bitwise equal host/device: {same}", flush=True)


if __name__ == "__main__":
    main()
