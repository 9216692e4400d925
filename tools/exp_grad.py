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
Each tree runs in worker processes of its own, alternated (measure.alternate): this tree, TREE, this tree, ...  A
worker warms up once, then times --reps calls (measure.host_time).  The first worker of each tree also saves its
gradients and, for float32 workloads, the same backward in float64 on the same (float32-rounded) inputs.  With
--parent, each row says whether the gradients of the two trees are bitwise equal and, where not, the largest
difference and its ratio to the bound two routes of one float32 input are held to in the tests:
2 (4 |g32 - g64| + 1e-6 scale), with this tree's float64 backward standing in for the float64 oracle.
Prints one JSON line per workload and the card (measure.card); with --out DIR, also
writes DIR/exp_grad.json."""
import argparse
import json
import statistics

import measure

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


def _worker(tree, out, save, reps):
    measure.enter(tree)
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

    times, saved = {}, {}
    for w, (n, m, T, B, dt, bound) in WORKLOADS.items():
        P = _inputs(n, m, T, B, bound)
        dtype = getattr(torch, dt)
        run = backward(n, m, T, bound, P, dtype)
        run()                                             # warm-up
        times[w], grads = measure.host_time(run, reps)
        if save:
            saved[w] = dict(zip(NAMES, grads))
            if dtype == torch.float32:                    # the float64 yardstick on the same rounded inputs
                P32 = {k: v.float().double() for k, v in P.items()}
                saved[w + "/f64"] = dict(zip(NAMES, backward(n, m, T, bound, P32, torch.float64)()))
        del run, grads
        torch.cuda.empty_cache()
    measure.save(out, times, outputs=saved if save else None)


def _compare(w, mine, theirs):
    """measure.compare of the two trees' gradients; where they differ, max |this - parent| / the routes' bound."""
    res = measure.compare(mine[w], theirs[w])
    for k in NAMES:
        if f"{k}_max_diff" in res and w + "/f64" in mine:
            a, g64 = mine[w][k], mine[w + "/f64"][k]
            sc = max(1.0, float(g64.abs().max()))
            bound = 2 * (4 * float((a.double() - g64).abs().max()) + 1e-6 * sc)
            res[f"{k}_diff_over_bound"] = res[f"{k}_max_diff"] / bound
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
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
        row = dict(workload=w, this_us=1e6 * statistics.median(times["this"][w]))
        if "parent" in arms:
            row.update(parent_us=1e6 * statistics.median(times["parent"][w]))
            row["speedup"] = row["parent_us"] / row["this_us"]
            row.update(_compare(w, outs["this"], outs["parent"]))
        rows.append(row)
        print(json.dumps(row), flush=True)
    runs = {k: {w: [round(1e6 * t, 2) for t in ts] for w, ts in v.items()} for k, v in times.items()}
    measure.report(a.out, __file__, c, rows, runs, rounds=a.rounds, reps=a.reps)


if __name__ == "__main__":
    main()
