#!/usr/bin/env python3
"""MPC.forward per solve with the iLQR loop on the host (one host round trip per iteration) and on the device (one
CUDA graph with a conditional `while` node, mpcb200_ilqr_*), and for the known systems the same physics wrapped as an
opaque Module (measure.Opaque: autograd linearisation, torch rollout, host loop), the route they took before the
kernels knew them.

  python tools/exp_ilqr_loop.py [--slew] [--reps 5] [--rounds 3] [--out DIR]

Workloads (float32, under torch.no_grad()):
  config2   cartpole B=128, T=25, +-100, <=50 iterations, eps 1e-2, AUTO_DIFF (BASELINE config 2)
  pendulum  B=128, T=20, +-2, <=50 iterations
  config4   LinDx (8,2) at config-4 size: B=1024, T=20, +-0.25, lqr_iter=10
  config3   LinDx (8,2) B=128, T=20, unbounded, lqr_iter=3
--slew runs the same table with slew_rate_penalty=0.1.  Routes alternate in every round; a round times --reps
solves of each route (host clock, each solve ending in a device synchronise) and the route's time is the median of
the rounds' means.  Per workload it prints ms per solve for each route, the iterations of each route's last solve,
the median host time of the library call that builds, instantiates and launches the graph, and whether the host and
device loops give bitwise equal x, u and costs."""
import argparse
import json
import statistics
import time

import measure

PENALTY = 0.1


def workloads(dev, slew):
    import torch
    from mpc.pytorch_b200.dynamics import CartpoleDx, PendulumDx
    from mpc.pytorch_b200.solver import MPC, GradMethods, LinDx, QuadCost
    from tests.cartpole import initial_states
    from tests.helpers import gen_problem
    kw = dict(verbose=-1, exit_unconverged=False, detach_unconverged=False, slew_rate_penalty=PENALTY if slew else None)

    def known(dx, B, T, x0, eps):
        n = dx.n_state
        q, p = dx.get_true_obj()
        cost = QuadCost(torch.diag(q).expand(T, B, n + 1, n + 1).contiguous().to(dev),
                        p.expand(T, B, n + 1).contiguous().to(dev))
        ctrl = MPC(n, 1, T, u_lower=dx.lower, u_upper=dx.upper, lqr_iter=50, linesearch_decay=dx.linesearch_decay,
                   max_linesearch_iter=dx.max_linesearch_iter, grad_method=GradMethods.AUTO_DIFF, eps=eps, **kw)
        return ctrl, x0.to(dev), cost, dx

    def pendulum():
        th = torch.linspace(-3.0, 3.0, 128)
        dx = PendulumDx()
        return known(dx, 128, 20, torch.stack((th.cos(), th.sin(), torch.zeros(128)), 1), dx.mpc_eps)

    def linear(B, bound, lqr_iter):
        C, c, F, f, x0 = [t.to(dev) for t in gen_problem(0, B, 20, 8, 2, torch.float32)]
        box = dict(u_lower=-bound, u_upper=bound) if bound else {}
        return MPC(8, 2, 20, lqr_iter=lqr_iter, **box, **kw), x0, QuadCost(C, c), LinDx(F, f)

    return {"config2": lambda: known(CartpoleDx(), 128, 25, initial_states(128, seed=0), 1e-2),
            "pendulum": pendulum,
            "config4": lambda: linear(1024, 0.25, 10),
            "config3": lambda: linear(128, None, 3)}


def solve(ctrl, x0, cost, dx, device_loop, reps, calls):
    """Seconds of each of `reps` solves, the last solve's (x, u, costs) and its iterations; the host time of every
    mpcb200_ilqr call goes to `calls`."""
    import torch
    from mpc.pytorch_b200 import solver, step
    orig = solver._use_device_loop, solver._use_slew_device_loop, step.ilqr_raw, solver.MPC.solve_lqr_subproblem
    seen = {"info": None, "host": 0}

    def raw(*a, **k):
        t0 = time.perf_counter()
        res = orig[2](*a, **k)
        calls.append(time.perf_counter() - t0)
        seen["info"] = res["info"]
        return res

    def sub(self, *a, **k):                          # one LQR step per host iteration
        if not k.get("no_op_forward", False):
            seen["host"] += 1
        return orig[3](self, *a, **k)

    def one():
        seen["host"] = 0
        with torch.no_grad():
            return ctrl(x0, cost, dx)
    if not device_loop:
        solver._use_device_loop = solver._use_slew_device_loop = lambda *a: False
    step.ilqr_raw, solver.MPC.solve_lqr_subproblem = raw, sub
    try:
        ts, out = measure.host_time(one, reps)
    finally:
        solver._use_device_loop, solver._use_slew_device_loop, step.ilqr_raw, solver.MPC.solve_lqr_subproblem = orig
    return ts, out, int(seen["info"][0]) if device_loop else seen["host"]


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--slew", action="store_true", help=f"slew_rate_penalty={PENALTY}")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="directory for exp_ilqr_loop.json (default: print only)")
    a = ap.parse_args()
    import torch
    from mpc.pytorch_b200 import solver
    from mpc.pytorch_b200.solver import LinDx
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    dev = torch.device("cuda:0")
    c = measure.card()
    rows, runs = [], {}
    for w, make in workloads(dev, a.slew).items():
        ctrl, x0, cost, dx = make()
        u0 = torch.zeros(ctrl.T, x0.shape[0], ctrl.n_ctrl, device=dev)
        takes = solver._use_slew_device_loop if a.slew else solver._use_device_loop
        assert takes(ctrl, x0, cost, dx, u0), f"{w}: MPC.forward would not run the device loop"
        routes = {"host": (dx, False), "device": (dx, True)}
        if not isinstance(dx, LinDx):
            routes["opaque"] = (measure.Opaque(dx), False)
        calls = []
        outs = {k: solve(ctrl, x0, cost, d, dev_loop, 1, calls)[1] for k, (d, dev_loop) in routes.items()}  # warm-up
        same = all(torch.equal(p, q) for p, q in zip(outs["host"], outs["device"]))
        means, iters, calls = {k: [] for k in routes}, {}, []
        for _ in range(a.rounds):
            for k, (d, dev_loop) in routes.items():
                ts, _, iters[k] = solve(ctrl, x0, cost, d, dev_loop, a.reps, calls)
                means[k].append(statistics.fmean(ts))
        row = dict(workload=w, slew=a.slew, bitwise_equal_host_device=same,
                   graph_call_ms=round(1e3 * statistics.median(calls), 3))
        for k in routes:
            row[f"{k}_ms"] = round(1e3 * statistics.median(means[k]), 2)
            row[f"{k}_iterations"] = iters[k]
        rows.append(row)
        runs[w] = {k: [round(1e3 * t, 3) for t in v] for k, v in means.items()}
        print(json.dumps(row), flush=True)
    measure.report(a.out, __file__, c, rows, runs, reps=a.reps, rounds=a.rounds)
    if not all(r["bitwise_equal_host_device"] for r in rows):
        raise SystemExit("the device loop differs from the host loop")


if __name__ == "__main__":
    main()
