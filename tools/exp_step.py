#!/usr/bin/env python3
"""Device time per launch of the LQR step (mpcb200_lqr_step_*) across arms: values of the MPCB200_KERNEL knob and/or
another build of the project.

  python tools/exp_step.py (--preset NAME | --case n,m,T,B[,dtype][,bound] ...) [--kernel 0,1,2,3] [--parent TREE]
                           [--riccati] [--cpu-oracle] [--rounds 3] [--out DIR]

A case is n,m,T,B with an optional dtype (float32, float64) and bound (a scalar box +-bound, or `tensor`: per-step
bounds drawn in (-0.52, -0.02) / (0.02, 0.52)).  Presets:
  config3, config3_box, config4, config5  the BASELINE configurations (DESIGN.md section 6)
  shapes   the generic and column-pair kernels over shapes and batches, the table behind PAIR_DEFAULT
           (lqr_step2.cuh): run with --kernel 1,2
  large    shapes without a compiled instance (lqr_large.cu), float32 and float64, and (16,4) at config 5's size,
           which has an instance: run with --kernel 0,3 to time the large-shape kernels there too
Each arm (--kernel value x this tree [and TREE]) runs in worker processes of its own, arms alternated in every round.
A worker times each case with bench.RawStepper / bench.time_launches: inputs from bench.gen_inputs (a feasible nominal
trajectory) rotated over enough sets to exceed the 50 MB L2, CUDA events around 5 blocks of launches, the median
block.  Gains go to Ks/ks where the library prefers it (mpcb200_step_prefers_workspace); --riccati times the Riccati
sweep alone (do_rollout = 0, gains in Ks/ks).  Per case and arm it prints us per launch (median over rounds), the plan
bits of the last launch (_lib.PLAN_*), the fractions of the HBM3 data-sheet bandwidth and of the fp32 FMA peak from
bench.bytes_per_solve / bench.flops_per_solve (float64 bytes doubled), and whether new_x, new_u, costs and alphas
(Ks, ks with --riccati) are bitwise equal to the first arm's.  --cpu-oracle adds the vectorised CPU oracle's
solves/s at the same shape on 16 problems."""
import argparse
import ctypes
import json
import statistics
import sys
import time

import measure

PRESETS = {
    "config3": ["8,2,20,4096", "8,2,20,65536"],
    "config3_box": ["8,2,20,4096,float32,0.25"],
    "config4": ["8,2,20,1024,float32,0.25", "8,2,20,1024,float32,tensor"],
    "config5": ["16,4,50,4096", "16,4,50,16384", "12,4,20,4096"],
    "shapes": ["16,4,50,4096", "16,4,50,16384", "16,4,50,4096,float32,0.25", "8,2,20,1024,float32,0.25",
               "8,2,20,16384", "8,4,20,4096", "12,4,30,4096", "4,2,20,4096", "6,2,25,128,float32,0.5",
               "2,2,10,4096"],
    "large": [f"{s},{dt}" for dt in ("float32", "float64")
              for s in ("20,4,50,4096", "24,8,20,1024", "48,16,20,1024", "max,4,20,1024")] + ["16,4,50,4096"],
}
OUTPUTS = ("new_x", "new_u", "costs", "alphas")


def parse_case(s):
    """(n, m, T, B, dtype name, bound) of `n,m,T,B[,dtype][,bound]`; n = `max`: the largest n_state the float32
    large-shape kernels take with this m (in float64 that case does not fit, and the row says so)."""
    f = s.split(",")
    if len(f) < 4 or len(f) > 6:
        raise argparse.ArgumentTypeError(f"case {s!r}: expected n,m,T,B[,dtype][,bound]")
    dtype = f[4] if len(f) > 4 else "float32"
    if dtype not in ("float32", "float64"):
        raise argparse.ArgumentTypeError(f"case {s!r}: dtype is float32 or float64")
    bound = None if len(f) < 6 else (f[5] if f[5] == "tensor" else float(f[5]))
    m = int(f[1])
    if f[0] == "max":
        from mpc.pytorch_b200.step import large_limit
        n = large_limit(m, 4)
    else:
        n = int(f[0])
    return n, m, int(f[2]), int(f[3]), dtype, bound


def name(case):
    n, m, T, B, dtype, bound = case
    return f"{n},{m},{T},{B},{dtype}" + ("" if bound is None else f",{bound}")


def _stepper(inp, case, riccati):
    """bench.RawStepper on `inp`, in the case's dtype, with its gains in Ks/ks where the library prefers it."""
    import torch
    import bench
    from mpc.pytorch_b200 import _lib
    n, m, T, B, dt, bound = case
    dtype, dev = getattr(torch, dt), inp["C"].device
    inp = {k: v.to(dtype) for k, v in inp.items()}
    tensor = None
    if bound == "tensor":
        g = torch.Generator(device=dev).manual_seed(7)
        tensor = (-0.5 * torch.rand(T, B, m, generator=g, device=dev, dtype=dtype) - 0.02,
                  0.5 * torch.rand(T, B, m, generator=g, device=dev, dtype=dtype) + 0.02)
    old = torch.get_default_dtype()
    torch.set_default_dtype(dtype)                  # RawStepper allocates its outputs in the default dtype
    try:
        st = bench.RawStepper(inp, B, T, n, m, bounds=None if tensor else bound, tensor_bounds=tensor)
    finally:
        torch.set_default_dtype(old)
    st.fn = _lib.entry("mpcb200_lqr_step", dtype)
    st.dims.do_rollout = 0 if riccati else 1
    st.Ks = st.ks = None
    if riccati or _lib.lib().mpcb200_step_prefers_workspace(ctypes.byref(st.dims), dtype.itemsize):
        st.Ks = torch.empty(T, B, m, n, dtype=dtype, device=dev)
        st.ks = torch.empty(T, B, m, dtype=dtype, device=dev)
    st.args[-3], st.args[-2] = _lib.ptr(st.Ks), _lib.ptr(st.ks)
    return st


def _worker(tree, out, save, cases, riccati):
    measure.enter(tree)
    import torch
    import bench
    from mpc.pytorch_b200 import _lib
    dev = torch.device("cuda:0")
    stream = torch.cuda.current_stream(dev)
    sh = ctypes.c_void_p(stream.cuda_stream)
    times, info, outputs = {}, {}, {}
    for case in cases:
        n, m, T, B, dt, bound = case
        nbytes = bench.bytes_per_solve(T, n, m, tensor_bounds=bound == "tensor") * B * (2 if dt == "float64" else 1)
        nsets = max(2, min(4, int(300e6 // nbytes) + 1))
        try:
            sts = [_stepper(bench.gen_inputs(100 + s, B, T, n, m, dev), case, riccati) for s in range(nsets)]
            _lib.check(sts[0].fn(*sts[0].args[:-1], sh), "step")     # a case the library refuses: say why
        except RuntimeError as e:
            info[name(case)] = dict(error=str(e))
            continue
        reps = max(10, min(400, int(2e10 // nbytes)))
        times[name(case)] = [bench.time_launches(sts, reps, stream, sh, blocks=5)]
        info[name(case)] = dict(plan=_lib.last_step_plan())
        sts[0](sh)
        torch.cuda.synchronize()
        if save:
            st = sts[0]
            outputs[name(case)] = dict(Ks=st.Ks, ks=st.ks) if riccati else {k: st.out[k] for k in OUTPUTS}
        del sts
        torch.cuda.empty_cache()
    measure.save(out, times, info, outputs if save else None)


def cpu_oracle_rate(case, Bc=16):
    """Solves/s of the vectorised CPU oracle at the case's shape on Bc problems."""
    import torch
    from oracle import lqr_oracle as orc
    from tests.helpers import gen_problem
    n, m, T, _, dt, _ = case
    dtype = getattr(torch, dt)
    C, c, F, f, x0 = gen_problem(7, Bc, T, n, m, dtype)
    u = torch.zeros(T, Bc, m, dtype=dtype)
    x = orc.get_traj(T, u, x0, F, f)
    t0 = time.perf_counter()
    orc.lqr_step_forward(n, m, T, x0, C, c, F, f, x, u, coupled=False)
    return Bc / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--preset", choices=sorted(PRESETS))
    ap.add_argument("--case", action="append", default=[], help="n,m,T,B[,dtype][,bound] (repeatable)")
    ap.add_argument("--kernel", default=None, help="comma-separated MPCB200_KERNEL values, one arm each")
    ap.add_argument("--riccati", action="store_true", help="the Riccati sweep alone (do_rollout = 0)")
    ap.add_argument("--cpu-oracle", action="store_true", help="also time the CPU oracle at each shape")
    measure.add_arguments(ap)
    a = ap.parse_args()
    specs = (PRESETS[a.preset] if a.preset else []) + a.case
    if not specs:
        ap.error("give --preset or --case")
    cases = [parse_case(s) for s in specs]
    args = [x for case in cases for x in ("--case", name(case))] + (["--riccati"] if a.riccati else [])
    if a.worker:
        return _worker(*a.worker[:2], a.worker[2] == "1", cases, a.riccati)
    import torch
    import bench
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    c = measure.card()
    knobs = a.kernel.split(",") if a.kernel else [None]
    arms = {t + ("" if k is None else f" k{k}"): (tree, {} if k is None else {"MPCB200_KERNEL": k})
            for t, tree in measure.trees(a.parent).items() for k in knobs}
    times, info, outs = measure.alternate(__file__, arms, a.rounds, args)
    first = next(iter(arms))
    rows = []
    for case in cases:
        n, m, T, B, dt, bound = case
        w = name(case)
        es_scale = 2 if dt == "float64" else 1
        row = dict(case=w)
        if a.cpu_oracle:
            row["cpu_oracle_solves_per_s"] = round(cpu_oracle_rate(case), 1)
        for arm in arms:
            r = dict(info[arm].get(w, {}))
            if w in times[arm]:
                us = statistics.median(times[arm][w])
                r.update(us=round(us, 2), solves_per_s=B / (us * 1e-6),
                         hbm_frac=round(bench.bytes_per_solve(T, n, m, tensor_bounds=bound == "tensor") * es_scale * B
                                        / (us * 1e-6) / (bench.HBM_PEAK_GBS * 1e9), 4),
                         fma_frac=round(bench.flops_per_solve(T, n, m) * B / (us * 1e-6) / 1e12
                                        / bench.FP32_FMA_PEAK_TFLOPS, 4))
                if arm != first and w in outs[first] and w in outs[arm]:
                    r.update(measure.compare(outs[arm][w], outs[first][w]))
            row[arm] = r
        rows.append(row)
        print(json.dumps(row), flush=True)
    measure.report(a.out, __file__, c, rows, times, rounds=a.rounds, riccati=a.riccati,
                   cpu_threads=torch.get_num_threads())


if __name__ == "__main__":
    sys.exit(main())
