"""Time the large-shape step kernel (csrc/lqr_large.cu) on the GPU: shapes without a compiled instance.

Per shape and dtype: device time per launch of mpcb200_lqr_step_* (CUDA events around blocks of launches, inputs
rotated over enough sets to exceed the 50 MB L2, unbounded, gains in Ks/ks), solves/s, the fraction of the HBM3 data
sheet bandwidth and of the fp32 FMA peak from bench.bytes_per_solve / bench.flops_per_solve (fp32 counts; f64 bytes
doubled), and the vectorised CPU oracle at the same shape on a small batch.  One context row times the instance kernel
at (16, 4), T = 50 against MPCB200_KERNEL=3 on the same inputs.  The card's name and power limit are read in the same
run.  Usage: python tools/exp_large.py [--quick]   (prints a markdown table and one JSON line)
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import bench  # noqa: E402
from mpc.pytorch_b200._lib import Dims, Params, check, entry, ptr  # noqa: E402
from mpc.pytorch_b200.step import large_limit, rollout_raw  # noqa: E402
from oracle import lqr_oracle as orc  # noqa: E402
from tests.helpers import gen_problem  # noqa: E402

DEV = torch.device("cuda:0")
L2_BYTES = 50 * 2 ** 20


def make_sets(B, T, n, m, dtype, nsets):
    sets = []
    for s in range(nsets):
        C, c, F, f, x0 = (t.to(DEV) for t in gen_problem(100 + s, B, T, n, m, dtype))
        u = torch.zeros(T, B, m, dtype=dtype, device=DEV)
        x = rollout_raw(n, m, T, x0, u, F, f)             # a feasible nominal trajectory, as in an iLQR iteration
        outs = [torch.empty(T, B, n, dtype=dtype, device=DEV), torch.empty(T, B, m, dtype=dtype, device=DEV)] + \
               [torch.empty(B, dtype=dtype, device=DEV) for _ in range(3)]
        gains = [torch.empty(T, B, m, n, dtype=dtype, device=DEV), torch.empty(T, B, m, dtype=dtype, device=DEV)]
        sets.append((C, c, F, f, x0, x, u, outs, gains))
    return sets


def launch(fn, dims, prm, s):
    C, c, F, f, x0, x, u, outs, gains = s
    rc = fn(ctypes.byref(dims), ctypes.byref(prm), ptr(C), ptr(c), ptr(F), ptr(f), ptr(x0), ptr(x), ptr(u), None, None,
            None, *[ptr(o) for o in outs], None, None, None, None, *[ptr(g) for g in gains], None)
    check(rc, "step")


def time_step(B, T, n, m, dtype, knob=None, blocks=5, per_block=10):
    es = 4 if dtype == torch.float32 else 8
    in_bytes = es * (T * (n + m) ** 2 + (T - 1) * n * (n + m)) * B
    nsets = max(2, -(-2 * L2_BYTES // in_bytes))
    sets = make_sets(B, T, n, m, dtype, nsets)
    dims = Dims(B=B, T=T, n=n, m=m, F_T=T - 1, has_f=1, max_ls_iter=10, pnqp_max_iter=20, do_rollout=1)
    prm = Params(ls_decay=0.2)
    fn = entry("mpcb200_lqr_step", dtype)
    old = os.environ.pop("MPCB200_KERNEL", None)
    if knob is not None:
        os.environ["MPCB200_KERNEL"] = knob
    try:
        for s in sets:                                    # warm-up: module load, attribute set, every input set
            launch(fn, dims, prm, s)
        torch.cuda.synchronize()
        times = []
        for _ in range(blocks):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(per_block):
                launch(fn, dims, prm, sets[i % nsets])
            e1.record()
            e1.synchronize()
            times.append(e0.elapsed_time(e1) * 1e3 / per_block)
    finally:
        os.environ.pop("MPCB200_KERNEL", None)
        if old is not None:
            os.environ["MPCB200_KERNEL"] = old
    return statistics.median(times), sets[0]


def cpu_oracle_rate(T, n, m, dtype, Bc=16):
    C, c, F, f, x0 = gen_problem(7, Bc, T, n, m, dtype)
    u = torch.zeros(T, Bc, m, dtype=dtype)
    x = orc.get_traj(T, u, x0, F, f)
    t0 = time.perf_counter()
    orc.lqr_step_forward(n, m, T, x0, C, c, F, f, x, u, coupled=False)
    return Bc / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="smaller batches (a rehearsal, not a measurement)")
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    nmax = large_limit(4, 4)
    shapes = [(20, 4, 4096, 50), (24, 8, 1024, 20), (48, 16, 1024, 20), (nmax, 4, 1024, 20)]
    rows = []
    for dtype in (torch.float32, torch.float64):
        es = 4 if dtype == torch.float32 else 8
        for n, m, B, T in shapes:
            if args.quick:
                B = min(B, 64)
            if n > large_limit(m, es):
                rows.append(dict(shape=f"({n},{m})", dtype=str(dtype)[6:], B=B, T=T, note="does not fit"))
                continue
            us, _ = time_step(B, T, n, m, dtype)
            byts = bench.bytes_per_solve(T, n, m) * es // 4
            fl = bench.flops_per_solve(T, n, m)
            rows.append(dict(shape=f"({n},{m})", dtype=str(dtype)[6:], B=B, T=T, us=round(us, 1),
                             solves_per_s=B / (us * 1e-6),
                             hbm_frac=round(byts * B / (us * 1e-6) / (bench.HBM_PEAK_GBS * 1e9), 4),
                             fma_frac=round(fl * B / (us * 1e-6) / 1e12 / bench.FP32_FMA_PEAK_TFLOPS, 4),
                             cpu_oracle_solves_per_s=round(cpu_oracle_rate(T, n, m, dtype), 1)))
    B = 64 if args.quick else 4096
    inst, s = time_step(B, 50, 16, 4, torch.float32)
    large, _ = time_step(B, 50, 16, 4, torch.float32, knob="3")
    context = dict(shape="(16,4)", dtype="float32", B=B, T=50, instance_us=round(inst, 1), large_us=round(large, 1))
    print(f"card: {card}; CPU oracle threads: {torch.get_num_threads()}")
    print("| shape | dtype | B | T | µs/launch | solves/s | of HBM | of fp32 FMA | CPU oracle solves/s |")
    print("|---|---|---|---|---|---|---|---|---|")
    for r in rows:
        if "note" in r:
            print(f"| {r['shape']} | {r['dtype']} | {r['B']} | {r['T']} | {r['note']} | | | | |")
        else:
            print(f"| {r['shape']} | {r['dtype']} | {r['B']} | {r['T']} | {r['us']} | {r['solves_per_s']:.3g} | "
                  f"{r['hbm_frac']} | {r['fma_frac']} | {r['cpu_oracle_solves_per_s']:.3g} |")
    print(f"| context (16,4) instance vs MPCB200_KERNEL=3 | float32 | {B} | 50 | {context['instance_us']} vs "
          f"{context['large_us']} | | | | |")
    print(json.dumps(dict(card=card, rows=rows, context=context, quick=args.quick)))


if __name__ == "__main__":
    main()
