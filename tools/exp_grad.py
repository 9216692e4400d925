#!/usr/bin/env python3
"""LQRStepFn.backward (the KKT adjoint through autograd) on this tree and, optionally, on another build of the project.

  python tools/exp_grad.py [--reps 30] [--rounds 3] [--parent TREE] [--out DIR]

Workloads: LQRStep(no_op_forward=True) at a fixed point (x, u) with u clamped to the box where there is one, so the
active set is not empty; the upstream gradients are fixed random tensors.
  config3       (8, 2) float32, B=4096, T=20, unbounded: the fused adjoint on both sides
  config3_box   the same with bounds +-0.25
  config5       (16, 4) float32, B=4096, T=50: past the generic kernel's KREDUCE switch (T = 23)
  padded_6_1    (6, 1) float32, B=4096, T=20, bounds +-0.25: zero padded to the (6, 2) instance
  padded_7_3    (7, 3) float64, B=1024, T=20, bounds +-0.25: zero padded to (7, 4), which the fused kernel does not take
  long_8_2      (8, 2) float64, B=256, T=700, bounds +-0.25: the gains of the masked step leave shared memory
  large_20_4    (20, 4) float64, B=256, T=10: no compiled instance, the large-shape kernels
Each tree runs in worker processes of its own (the two builds share module names), alternated: this tree, TREE, this
tree, ...  A worker warms up once, then times --reps calls (host clock around each call, which ends in a device
synchronise).  The first worker of each tree also saves its gradients and, for float32 workloads, the same backward
in float64 on the same (float32-rounded) inputs.  With --parent, each row says whether the gradients of the two trees
are bitwise equal and, where not, compares their difference with the bound two routes of one float32 input are held
to in the tests: 2 (4 |g32 - g64| + 1e-6 scale), with this tree's float64 backward standing in for the float64 oracle.
Prints one JSON line per workload and the card's name and power limit, read in the same run; with --out DIR, also
writes DIR/exp_grad.json."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# name: (n, m, T, B, dtype, box bound or None)
WORKLOADS = {
    "config3": (8, 2, 20, 4096, "float32", None),
    "config3_box": (8, 2, 20, 4096, "float32", 0.25),
    "config5": (16, 4, 50, 4096, "float32", None),
    "padded_6_1": (6, 1, 20, 4096, "float32", 0.25),
    "padded_7_3": (7, 3, 20, 1024, "float64", 0.25),
    "long_8_2": (8, 2, 700, 256, "float64", 0.25),
    "large_20_4": (20, 4, 10, 256, "float64", None),
}
NAMES = ("dx_init", "dC", "dc", "dF", "df")


def _inputs(n, m, T, B, bound, seed=0):
    """float64 CPU tensors of one workload: C = L L'/p + I, c, F = [0.9 I + noise, B], f, x_init, the point (x, u)
    and the upstream gradients."""
    import torch
    g = torch.Generator().manual_seed(seed)
    p = n + m
    rn = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)  # noqa: E731
    L = rn(T, B, p, p)
    C = L @ L.transpose(-1, -2) / p + torch.eye(p, dtype=torch.float64)
    F = torch.cat((0.9 * torch.eye(n, dtype=torch.float64) + 0.05 * rn(T - 1, B, n, n), 0.3 * rn(T - 1, B, n, m)), 3)
    u = 0.5 * rn(T, B, m)
    if bound is not None:
        u = u.clamp(-bound, bound)
    return dict(x_init=rn(B, n), C=C, c=rn(T, B, p), F=F, f=0.1 * rn(T - 1, B, n), x=rn(T, B, n), u=u,
                wx=rn(T, B, n), wu=rn(T, B, m))


def _worker(tree, reps, save, out):
    sys.path.insert(0, tree)
    import torch
    from mpc.pytorch_b200 import LQRStep, LinDx, QuadCost
    dev = torch.device("cuda:0")

    def backward(n, m, T, bound, P, dtype):
        d = {k: v.to(dtype).to(dev) for k, v in P.items()}
        lv = [d[k].requires_grad_(True) for k in ("x_init", "C", "c", "F", "f")]
        kw = {} if bound is None else dict(u_lower=-bound, u_upper=bound)
        fn = LQRStep(n, m, T, true_cost=QuadCost(lv[1], lv[2]), true_dynamics=LinDx(lv[3], lv[4]),
                     current_x=d["x"], current_u=d["u"], no_op_forward=True, **kw)
        xo, uo = fn(*lv)
        return lambda: torch.autograd.grad((xo, uo), lv, (d["wx"], d["wu"]), retain_graph=True)

    rows, saved = {}, {}
    for w, (n, m, T, B, dt, bound) in WORKLOADS.items():
        P = _inputs(n, m, T, B, bound)
        dtype = getattr(torch, dt)
        run = backward(n, m, T, bound, P, dtype)
        grads = run()                                     # warm-up
        torch.cuda.synchronize()
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter()
            run()
            torch.cuda.synchronize()
            ts.append(time.perf_counter() - t0)
        rows[w] = ts
        if save:
            saved.update({f"{w}/{k}": t.cpu() for k, t in zip(NAMES, grads)})
            if dtype == torch.float32:                    # the float64 yardstick on the same rounded inputs
                P32 = {k: v.float().double() for k, v in P.items()}
                saved.update({f"{w}/{k}64": t.cpu() for k, t in zip(NAMES, backward(n, m, T, bound, P32,
                                                                                    torch.float64)())})
        del run, grads
        torch.cuda.empty_cache()
    if save:
        torch.save(saved, out + ".pt")
    with open(out + ".json", "w") as fh:
        json.dump(rows, fh)


def _compare(w, mine, theirs):
    """bitwise equality of the two trees' gradients; where they differ, max |this - parent| / the routes' bound."""
    res = {}
    for k in NAMES:
        a, b = mine[f"{w}/{k}"], theirs[f"{w}/{k}"]
        res[f"{k}_bitwise"] = bool(a.shape == b.shape and bool((a == b).all()))
        if not res[f"{k}_bitwise"] and f"{w}/{k}64" in mine:
            g64 = mine[f"{w}/{k}64"]
            sc = max(1.0, float(g64.abs().max()))
            bound = 2 * (4 * float((a.double() - g64).abs().max()) + 1e-6 * sc)
            res[f"{k}_diff_over_bound"] = float((a.double() - b.double()).abs().max()) / bound
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3, help="alternated worker processes per tree")
    ap.add_argument("--parent", default=None, help="another tree of the project, built, to compare against")
    ap.add_argument("--out", default=None, help="directory for exp_grad.json (default: print only)")
    ap.add_argument("--worker", nargs=3, metavar=("TREE", "SAVE", "OUT"), help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        return _worker(a.worker[0], a.reps, a.worker[1] == "1", a.worker[2])
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
                                "1" if r == 0 else "0", out], check=True, cwd=tmp)
                with open(out + ".json") as fh:
                    for w, ts in json.load(fh).items():
                        times[k][w] += ts
                if r == 0:
                    outs[k] = torch.load(out + ".pt")
    rows = []
    for w in WORKLOADS:
        row = dict(workload=w, this_us=1e6 * statistics.median(times["this"][w]))
        if "parent" in trees:
            row.update(parent_us=1e6 * statistics.median(times["parent"][w]))
            row["speedup"] = row["parent_us"] / row["this_us"]
            row.update(_compare(w, outs["this"], outs["parent"]))
        rows.append(row)
        print(json.dumps(row), flush=True)
    if a.out is not None:
        os.makedirs(a.out, exist_ok=True)
        every = {k: {w: [round(1e6 * t, 2) for t in ts] for w, ts in v.items()} for k, v in times.items()}
        with open(os.path.join(a.out, "exp_grad.json"), "w") as fh:
            json.dump(dict(card=card, torch=torch.__version__, rounds=a.rounds, reps=a.reps,
                           this_us_all=every["this"], parent_us_all=every.get("parent", {}), rows=rows), fh, indent=1)
    print("card:", card)


if __name__ == "__main__":
    main()
