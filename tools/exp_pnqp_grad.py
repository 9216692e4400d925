"""Cost of a gradient through the standalone pnqp: forward + backward with H, q, lower and upper requiring grad,
mpc.pnqp.pnqp (the pnqp kernel, then one mpcb200_pnqp_backward_* call) against the batch-coupled CPU oracle
(oracle.lqr_oracle.pnqp, coupled=True, the reference's control flow) run on the same GPU under autograd, which
differentiates through every iteration as the reference does.  (developer tool)

  python tools/exp_pnqp_grad.py [--reps 7] [--oracle-reps 3] [--batch 4096] [--sizes 2,8,32,128] [--out DIR]

Each row times forward + backward of sum(w * x) with CUDA events: two warm-up calls, then the median of --reps calls
(--oracle-reps for the oracle).  Inputs follow the pnqp generator of oracle/make_golden.py, cold start.  The card
(measure.card) is printed with the numbers; with --out DIR, the rows, every call's time and the card go to
DIR/exp_pnqp_grad.json.
"""
import argparse
import contextlib
import io
import statistics

import torch

import measure


def gen(B, n, dtype, dev):
    g = torch.Generator(device=dev).manual_seed(1000 * n + B)
    L = torch.randn(B, n, n, generator=g, device=dev, dtype=torch.float64)
    H = L @ L.transpose(1, 2) + 0.5 * torch.eye(n, device=dev, dtype=torch.float64)
    q = 2.0 * torch.randn(B, n, generator=g, device=dev, dtype=torch.float64)
    lo = -torch.rand(B, n, generator=g, device=dev, dtype=torch.float64)
    hi = torch.rand(B, n, generator=g, device=dev, dtype=torch.float64)
    w = torch.randn(B, n, generator=g, device=dev, dtype=torch.float64)
    return [t.to(dtype) for t in (H, q, lo, hi, w)]


def timed(fn, warmup, reps):
    """Milliseconds of each of `reps` calls after `warmup` calls, by CUDA events."""
    for _ in range(warmup):
        fn()
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--oracle-reps", type=int, default=3)
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--sizes", default="2,8,32,128")
    ap.add_argument("--out", default=None, help="directory for exp_pnqp_grad.json (default: print only)")
    args = ap.parse_args()
    from mpc.pnqp import pnqp
    from oracle import lqr_oracle as orc
    dev = torch.device("cuda:0")
    c = measure.card()
    rows, runs = [], {}
    B = args.batch
    print(f"{'dtype':>7} {'B':>5} {'n':>4} {'kernels ms':>11} {'oracle ms':>10} {'speed-up':>9}")
    for dtype in (torch.float32, torch.float64):
        for n in [int(s) for s in args.sizes.split(",")]:
            H, q, lo, hi, w = gen(B, n, dtype, dev)
            leaves = [t.clone().requires_grad_(True) for t in (H, q, lo, hi)]

            def ours():
                for t in leaves:
                    t.grad = None
                x = pnqp(*leaves, n_iter=20)[0]
                (w * x).sum().backward()

            def oracle():
                for t in leaves:
                    t.grad = None
                with torch.device(dev):     # the oracle makes its constants on the default device
                    x = orc.pnqp(*leaves, n_iter=20, coupled=True)[0]
                (w * x).sum().backward()

            with contextlib.redirect_stdout(io.StringIO()):            # fp32 iteration-cap warnings
                mine = timed(ours, 2, args.reps)
                theirs = timed(oracle, 1, args.oracle_reps)
            a, b = statistics.median(mine), statistics.median(theirs)
            name = str(dtype).replace("torch.", "")
            print(f"{name:>7} {B:5d} {n:4d} {a:11.3f} {b:10.2f} {b / a:9.1f}", flush=True)
            rows.append(dict(dtype=name, B=B, n=n, ms=a, oracle_ms=b))
            runs[f"{name},{B},{n}"] = dict(kernels=mine, oracle=theirs)
            del H, q, lo, hi, w, leaves
            torch.cuda.empty_cache()
    measure.report(args.out, __file__, c, rows, runs, reps=args.reps, oracle_reps=args.oracle_reps)


if __name__ == "__main__":
    main()
