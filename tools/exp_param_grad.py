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
Each tree runs in worker processes of its own (the two builds share module names), alternated: this tree, TREE,
this tree, ...  A worker warms up once, then times --reps calls (host clock around work that ends in a device
synchronise) and saves its outputs; the parent compares x, u, costs (bitwise) and the gradients of the two trees.
Prints one JSON line per workload and the card's name and power limit, read in the same run; with --out DIR, also
writes DIR/exp_param_grad.json."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKLOADS = ("tail_known", "tail_opaque", "config2", "pendulum", "config2_f64")


def _worker(tree, reps, out):
    sys.path.insert(0, tree)
    import torch
    from mpc.pytorch_b200 import MPC, GradMethods, QuadCost
    from mpc.pytorch_b200.dynamics import CartpoleDx, PendulumDx
    dev = torch.device("cuda:0")

    def problem(name, dtype):
        B, T = (16, 20) if name == "pendulum" else (128, 25)
        g = torch.Generator().manual_seed(0)
        if name == "pendulum":
            params = torch.tensor((10.0, 1.0, 1.0), dtype=dtype, device=dev).requires_grad_(True)
            dx = PendulumDx(params=params)
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
        ctrl, dx, params, x0, Q, c, wx, wu = problem("pendulum" if workload == "pendulum" else "cartpole", dtype)
        if workload.startswith("tail"):
            with torch.no_grad():
                x, u, _ = ctrl(x0, QuadCost(Q, c), dx)
            if workload == "tail_opaque":
                inner = dx

                class Opaque(torch.nn.Module):
                    def forward(self, x, u):
                        return inner(x, u)
                dx = Opaque()
            wF = torch.randn(x.shape[0] - 1, x.shape[1], x.shape[2], x.shape[2] + 1, generator=torch.Generator()
                             .manual_seed(1), dtype=dtype).to(dev)

            def run():
                F, f = ctrl.linearize_dynamics(x, u, dx, diff=True)
                g, = torch.autograd.grad((wF * F).sum() + (wx[:-1] * f).sum(), params)
                return {"F": F.detach(), "f": f.detach(), "grad_params": g}
            return run
        leaves = [params, c, x0] if dtype == torch.float64 else [params]

        def run():
            x, u, costs = ctrl(x0, QuadCost(Q, c), dx)
            grads = torch.autograd.grad((wx * x).sum() + (wu * u).sum(), leaves)
            res = {"x": x.detach(), "u": u.detach(), "costs": costs.detach()}
            res.update({f"grad_{k}": g for k, g in zip(("params", "c", "x_init"), grads)})
            return res
        return run

    rows, saved = {}, {}
    for w in WORKLOADS:
        run = make(w)
        res = run()                                     # warm-up
        torch.cuda.synchronize()
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter()
            res = run()
            torch.cuda.synchronize()
            ts.append(time.perf_counter() - t0)
        rows[w] = ts
        saved.update({f"{w}/{k}": v.cpu() for k, v in res.items()})
    torch.save(saved, out + ".pt")
    with open(out + ".json", "w") as fh:
        json.dump(rows, fh)


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / max(1e-300, float(b.double().abs().max())))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--rounds", type=int, default=3, help="alternated worker processes per tree")
    ap.add_argument("--parent", default=None, help="another tree of the project, built, to compare against")
    ap.add_argument("--out", default=None, help="directory for exp_param_grad.json (default: print only)")
    ap.add_argument("--worker", nargs=2, metavar=("TREE", "OUT"), help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        return _worker(a.worker[0], a.reps, a.worker[1])
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    card = smi[0] if smi else torch.cuda.get_device_name(0)
    trees = {"this": ROOT}
    if a.parent:
        trees["parent"] = os.path.abspath(a.parent)
    times = {k: {w: [] for w in WORKLOADS} for k in trees}
    outs = {}
    with tempfile.TemporaryDirectory() as tmp:
        for r in range(a.rounds):
            for k, tree in trees.items():
                out = os.path.join(tmp, f"{k}{r}")
                subprocess.run([sys.executable, os.path.abspath(__file__), "--reps", str(a.reps), "--worker", tree,
                                out], check=True, cwd=tmp)
                with open(out + ".json") as fh:
                    for w, ts in json.load(fh).items():
                        times[k][w] += ts
                outs[k] = torch.load(out + ".pt")
    rows = []
    for w in WORKLOADS:
        row = dict(workload=w, this_ms=1e3 * statistics.median(times["this"][w]),
                   this_ms_all=[round(1e3 * t, 3) for t in times["this"][w]])
        if "parent" in trees:
            row.update(parent_ms=1e3 * statistics.median(times["parent"][w]),
                       parent_ms_all=[round(1e3 * t, 3) for t in times["parent"][w]])
            row["speedup"] = row["parent_ms"] / row["this_ms"]
            mine, theirs = outs["this"], outs["parent"]
            for key in sorted(k for k in mine if k.startswith(w + "/")):
                name = key.split("/", 1)[1]
                if name in ("x", "u", "costs"):
                    row[f"{name}_bitwise"] = bool(torch.equal(mine[key], theirs[key]))
                else:
                    row[f"{name}_rel_change"] = _rel(mine[key], theirs[key])
        rows.append(row)
        print(json.dumps(row), flush=True)
    if "tail_known" in times["this"]:
        print(f"tail: known system {rows[0]['this_ms']:.3f} ms, opaque Module {rows[1]['this_ms']:.3f} ms "
              f"(x{rows[1]['this_ms'] / rows[0]['this_ms']:.1f})")
    if a.out is not None:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "exp_param_grad.json"), "w") as fh:
            json.dump(dict(card=card, torch=torch.__version__, rows=rows), fh, indent=1)
    print("card:", card)


if __name__ == "__main__":
    main()
