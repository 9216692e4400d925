#!/usr/bin/env python3
"""Parameter gradients of the known systems: MPC's differentiable tail through the VJP kernel (dynamics.DynLinearize)
against the torch autograd route, and MPC.forward + backward against another build of the project.

  python tools/exp_param_grad.py [--reps 7] [--parent TREE] [--out DIR]

Workloads (learnable `params` on the device, requires_grad; the loss is a fixed linear function of (x, u)):
  tail_known    config 2 size (cartpole B=128, T=25, float32): linearize_dynamics(diff=True) + backward, known system
  tail_opaque   the same with the physics wrapped as an opaque Module (torch AUTO_DIFF, create_graph: the old route)
  config2       cartpole B=128, T=25, bounds +-100, <=50 iterations, eps 1e-2, float32: MPC.forward + backward
  pendulum      the pendulum notebook's size, B=16, T=20, PendulumDx(params=(10, 1, 1)), bounds +-2, float32
  config2_f64   config2 in float64 (also gives d/dc and d/dx_init, to compare against TREE at rounding level)
  pendulum_full the pendulum notebook's size with the five-parameter PendulumDx(params=(10, 1, 1, 0.3, 0.2),
                simple=False), bounds +-2, float32: MPC.forward + backward, d/dparams of all five entries
  pendulum_full_opaque  the same with the physics wrapped as an opaque Module (torch rollout, AUTO_DIFF with
                create_graph, split-mode line search: the only route before the kernels knew this system)
Each tree runs in worker processes of its own, alternated (measure.alternate): this tree, TREE, this tree, ...  A
worker warms up once, then times --reps calls (measure.host_time); the first worker of each tree saves its outputs,
and the parent compares them (measure.compare, and the relative change of each gradient).  A tree that cannot
build a workload's system (PendulumDx(simple=False) raising NotImplementedError) leaves that workload out.  Prints one JSON line per
workload and the card (measure.card); with --out DIR, also writes DIR/exp_param_grad.json."""
import argparse
import json
import statistics

import measure

WORKLOADS = ("tail_known", "tail_opaque", "config2", "pendulum", "config2_f64", "pendulum_full",
             "pendulum_full_opaque")


def _worker(tree, out, save, reps):
    measure.enter(tree)
    import torch
    from mpc.pytorch_b200 import MPC, GradMethods, QuadCost
    from mpc.pytorch_b200.dynamics import CartpoleDx, PendulumDx
    dev = torch.device("cuda:0")

    def problem(name, dtype):
        B, T = (128, 25) if name == "cartpole" else (16, 20)
        g = torch.Generator().manual_seed(0)
        if name.startswith("pendulum"):
            full = name == "pendulum_full"
            params = torch.tensor((10.0, 1.0, 1.0, 0.3, 0.2) if full else (10.0, 1.0, 1.0), dtype=dtype,
                                  device=dev).requires_grad_(True)
            dx = PendulumDx(params=params, simple=not full)
            th = (torch.rand(B, generator=g, dtype=dtype) * 2 - 1) * 1.5708
            x0 = torch.stack((th.cos(), th.sin(), torch.rand(B, generator=g, dtype=dtype) * 2 - 1), 1)
        else:
            params = torch.tensor((9.8, 1.0, 0.1, 0.5), dtype=dtype, device=dev).requires_grad_(True)
            dx = CartpoleDx(params=params)
            th = (torch.rand(B, generator=g, dtype=dtype) * 2 - 1) * 3.14159
            r = torch.rand(B, 3, generator=g, dtype=dtype) - 0.5
            x0 = torch.stack((r[:, 0], r[:, 1], th.cos(), th.sin(), r[:, 2]), 1)
        n = dx.n_state
        q, p = dx.get_true_obj()
        Q = torch.diag(q).to(dtype).expand(T, B, n + 1, n + 1).contiguous().to(dev)
        c = p.to(dtype).expand(T, B, n + 1).contiguous().to(dev).requires_grad_(True)
        x0 = x0.to(dev).requires_grad_(True)
        wx = torch.randn(T, B, n, generator=g, dtype=dtype).to(dev)
        wu = torch.randn(T, B, 1, generator=g, dtype=dtype).to(dev)
        ctrl = MPC(n, 1, T, u_lower=float(dx.lower), u_upper=float(dx.upper), lqr_iter=50, verbose=-1,
                   linesearch_decay=dx.linesearch_decay, max_linesearch_iter=dx.max_linesearch_iter,
                   grad_method=GradMethods.AUTO_DIFF, eps=1e-2, exit_unconverged=False, detach_unconverged=False)
        return ctrl, dx, params, x0, Q, c, wx, wu

    def make(workload):
        dtype = torch.float64 if workload == "config2_f64" else torch.float32
        name = workload.replace("_opaque", "") if workload.startswith("pendulum") else "cartpole"
        ctrl, dx, params, x0, Q, c, wx, wu = problem(name, dtype)
        if workload.startswith("tail"):
            with torch.no_grad():
                x, u, _ = ctrl(x0, QuadCost(Q, c), dx)
            if workload == "tail_opaque":
                dx = measure.Opaque(dx)
            wF = torch.randn(x.shape[0] - 1, x.shape[1], x.shape[2], x.shape[2] + 1, generator=torch.Generator()
                             .manual_seed(1), dtype=dtype).to(dev)

            def run():
                F, f = ctrl.linearize_dynamics(x, u, dx, diff=True)
                g, = torch.autograd.grad((wF * F).sum() + (wx[:-1] * f).sum(), params)
                return {"F": F.detach(), "f": f.detach(), "grad_params": g}
            return run
        if workload == "pendulum_full_opaque":
            dx = measure.Opaque(dx)
        leaves = [params, c, x0] if dtype == torch.float64 else [params]

        def run():
            x, u, costs = ctrl(x0, QuadCost(Q, c), dx)
            grads = torch.autograd.grad((wx * x).sum() + (wu * u).sum(), leaves)
            res = {"x": x.detach(), "u": u.detach(), "costs": costs.detach()}
            res.update({f"grad_{k}": g for k, g in zip(("params", "c", "x_init"), grads)})
            return res
        return run

    times, saved = {}, {}
    for w in WORKLOADS:
        try:
            run = make(w)
        except NotImplementedError:
            continue
        run()                                           # warm-up
        times[w], saved[w] = measure.host_time(run, reps)
    measure.save(out, times, outputs=saved if save else None)


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / max(1e-300, float(b.double().abs().max())))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    measure.add_arguments(ap)
    a = ap.parse_args()
    if a.worker:
        return _worker(*a.worker[:2], a.worker[2] == "1", a.reps)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    c = measure.card()
    arms = {k: (tree, {}) for k, tree in measure.trees(a.parent).items()}
    times, _, outs = measure.alternate(__file__, arms, a.rounds, ["--reps", str(a.reps)])
    rows = []
    for w in WORKLOADS:
        if w not in times["this"]:
            continue
        row = dict(workload=w, this_ms=1e3 * statistics.median(times["this"][w]),
                   this_ms_all=[round(1e3 * t, 3) for t in times["this"][w]])
        if "parent" in arms and w in times["parent"]:
            row.update(parent_ms=1e3 * statistics.median(times["parent"][w]),
                       parent_ms_all=[round(1e3 * t, 3) for t in times["parent"][w]])
            row["speedup"] = row["parent_ms"] / row["this_ms"]
            mine, theirs = outs["this"][w], outs["parent"][w]
            row.update(measure.compare(mine, theirs))
            row.update({f"{k}_rel_change": _rel(mine[k], theirs[k]) for k in mine
                        if k not in ("x", "u", "costs")})
        rows.append(row)
        print(json.dumps(row), flush=True)
    print(f"tail: known system {rows[0]['this_ms']:.3f} ms, opaque Module {rows[1]['this_ms']:.3f} ms "
          f"(x{rows[1]['this_ms'] / rows[0]['this_ms']:.1f})")
    by = {r["workload"]: r["this_ms"] for r in rows}
    print(f"pendulum_full: kernels {by['pendulum_full']:.3f} ms, opaque Module {by['pendulum_full_opaque']:.3f} ms "
          f"(x{by['pendulum_full_opaque'] / by['pendulum_full']:.1f})")
    runs = {k: {w: [round(1e3 * t, 3) for t in ts] for w, ts in v.items()} for k, v in times.items()}
    measure.report(a.out, __file__, c, rows, runs, rounds=a.rounds, reps=a.reps)


if __name__ == "__main__":
    main()
