"""Cost of the standalone pnqp (mpc.pnqp.pnqp) over batch size, QP size and precision.  (developer tool)

  python tools/exp_pnqp.py [--reps 7] [--batches 2,256,4096] [--sizes 8,9,16,32,64,100,128] [--out DIR]

Each row times the whole Python call (argument broadcast, output allocation, one kernel, the read of the
iteration counts) with CUDA events: two warm-up calls, then the median of --reps calls.  n = 8 runs the
thread-per-QP kernel, n > 8 the thread-block-per-QP kernel.  For the B = 2 rows the per-problem CPU oracle
(oracle/lqr_oracle.py, coupled=False) is timed on the same inputs as a baseline.  Inputs follow the pnqp
generator of oracle/make_golden.py.  The card (measure.card) is printed with the numbers; with --out DIR, the rows,
every call's time and the card go to DIR/exp_pnqp.json.
"""
import argparse
import contextlib
import io
import statistics
import time

import torch

import measure


def gen(B, n, dtype, dev):
    g = torch.Generator(device=dev).manual_seed(1000 * n + B)
    L = torch.randn(B, n, n, generator=g, device=dev, dtype=torch.float64)
    H = L @ L.transpose(1, 2) + 0.5 * torch.eye(n, device=dev, dtype=torch.float64)
    q = 2.0 * torch.randn(B, n, generator=g, device=dev, dtype=torch.float64)
    lo = -torch.rand(B, n, generator=g, device=dev, dtype=torch.float64)
    hi = torch.rand(B, n, generator=g, device=dev, dtype=torch.float64)
    return [t.to(dtype) for t in (H, q, lo, hi)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--batches", default="2,256,4096")
    ap.add_argument("--sizes", default="8,9,16,32,64,100,128")
    ap.add_argument("--out", default=None, help="directory for exp_pnqp.json (default: print only)")
    args = ap.parse_args()
    from mpc.pnqp import pnqp
    from oracle import lqr_oracle as orc
    dev = torch.device("cuda:0")
    c = measure.card()
    rows, runs = [], {}
    print(f"{'dtype':>7} {'B':>5} {'n':>4} {'iters':>5} {'ms/call':>9} {'QPs/s':>10} {'CPU oracle ms':>14}")
    for dtype in (torch.float32, torch.float64):
        for B in [int(b) for b in args.batches.split(",")]:
            for n in [int(s) for s in args.sizes.split(",")]:
                H, q, lo, hi = gen(B, n, dtype, dev)
                quiet = contextlib.redirect_stdout(io.StringIO())   # fp32 cap warnings
                with quiet:
                    for _ in range(2):
                        _, _, _, it = pnqp(H, q, lo, hi)
                    ms = []
                    for _ in range(args.reps):
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        pnqp(H, q, lo, hi)
                        e1.record()
                        e1.synchronize()
                        ms.append(e0.elapsed_time(e1))
                med = statistics.median(ms)
                cpu = ""
                if B == 2:
                    Hc, qc, lc, hc = (t.cpu() for t in (H, q, lo, hi))
                    tc = []
                    for _ in range(3):
                        t0 = time.perf_counter()
                        orc.pnqp(Hc, qc, lc, hc, n_iter=20, coupled=False)
                        tc.append(1e3 * (time.perf_counter() - t0))
                    cpu = f"{statistics.median(tc):.2f}"
                name = str(dtype).replace("torch.", "")
                print(f"{name:>7} {B:5d} {n:4d} {it:5d} {med:9.3f} {B / med * 1e3:10.3g} {cpu:>14}", flush=True)
                rows.append(dict(dtype=name, B=B, n=n, iters=it, ms=med, cpu_oracle_ms=float(cpu) if cpu else None))
                runs[f"{name},{B},{n}"] = ms
                del H, q, lo, hi
    torch.cuda.empty_cache()
    measure.report(args.out, __file__, c, rows, runs, reps=args.reps)


if __name__ == "__main__":
    main()
