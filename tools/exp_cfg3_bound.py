"""Is config 3 (T=20, n=8, m=2, fp32, unbounded) latency bound or throughput bound?  (developer tool)

Runs the step over a sweep of batch sizes and reports us per launch and us per busiest-SM problem slot: the
launch time over the number of problems the most loaded SM holds (ceil(CTAs / SMs) * problems per CTA).  The
generic kernel at (8, 2) fp32 puts 8 problems in a CTA (two consumer warps of 4 8-lane problems), so at B=4096 the
busiest SM holds 4 CTAs; at B=65536 an SM keeps as many resident as registers and shared memory allow and runs
waves of them.  If one warp's dependent chain set the time, the extra resident warps would hide it and the
per-slot time would fall; if an SM resource saturates already at B=4096, the per-slot time stays flat.

  python tools/exp_cfg3_bound.py [--riccati] [--batches 1024,4096,...] [--problems-per-cta 8] [--out DIR]

--riccati times the Riccati sweep alone (do_rollout = 0, gains written to Ks/ks).  The card (measure.card) and the
median SM clock under the load are printed with the numbers; with --out DIR they go to DIR/exp_cfg3_bound.json with
the rows.  Another build of the library is measured by running this script in that build's tree;
--problems-per-cta gives its CTA size, e.g. 6 for the earlier layout of 3 problems per warp and 2 consumer warps.
"""
import argparse
import ctypes
import math

import torch

import measure
import bench  # noqa: E402  (importable once measure has put the repository root on sys.path)

T, N, M = 20, 8, 2
PROBLEMS_PER_CTA = 8        # the generic kernel at (8, 2) f32: 2 consumer warps x 4 problems


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--riccati", action="store_true")
    ap.add_argument("--batches", default="1024,2048,4096,8192,16384,65536")
    ap.add_argument("--reps", type=int, default=0, help="launches per timed block (0: ~0.2 s of work)")
    ap.add_argument("--problems-per-cta", type=int, default=PROBLEMS_PER_CTA)
    ap.add_argument("--out", default=None, help="directory for exp_cfg3_bound.json (default: print only)")
    args = ap.parse_args()
    from mpc.pytorch_b200 import _lib
    dev = torch.device("cuda:0")
    stream = torch.cuda.current_stream(dev)
    sh = ctypes.c_void_p(stream.cuda_stream)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    c = measure.card()
    clk = bench.ClockSampler(0)
    clk.start()
    rows = []
    for B in [int(b) for b in args.batches.split(",")]:
        nsets = max(2, min(4, int(300e6 // (bench.bytes_per_solve(T, N, M) * B)) + 1))
        sts = [bench.RawStepper(bench.gen_inputs(100 + s, B, T, N, M, dev), B, T, N, M) for s in range(nsets)]
        if args.riccati:
            for st in sts:
                st.dims.do_rollout = 0
                st.Ks = torch.empty(T, B, M, N, device=dev)
                st.ks = torch.empty(T, B, M, device=dev)
                st.args[-3], st.args[-2] = _lib.ptr(st.Ks), _lib.ptr(st.ks)
        reps = args.reps or max(20, int(2e5 / max(1.0, 15.0 * B / 1024)))
        us = bench.time_launches(sts, reps, stream, sh, blocks=5)
        plan = _lib.last_step_plan()
        if not plan & _lib.PLAN_GENERIC:
            raise SystemExit(f"expected the generic kernel at (8, 2) f32, the plan was {plan}")
        w = args.problems_per_cta
        busiest = math.ceil(math.ceil(B / w) / sms) * w
        rows.append(dict(B=B, us=us, busiest_problems=busiest, us_per_slot=us / busiest))
        print(f"B={B:6d}  {us:9.1f} us/launch  busiest SM {busiest:4d} problems  {us / busiest:6.3f} us/slot",
              flush=True)
        del sts
        torch.cuda.empty_cache()
    load = clk.stop()
    print(f"median SM clock under load {load['sm_mhz']} MHz, throttle reasons {load['reasons']}; {sms} SMs; "
          f"{'Riccati only' if args.riccati else 'sweep + rollout'}")
    per_slot = {r["B"]: r["us_per_slot"] for r in rows}
    if 4096 in per_slot and 65536 in per_slot:
        print(f"per-slot time at B=4096 / B=65536: {per_slot[4096] / per_slot[65536]:.3f}")
    measure.report(args.out, __file__, c, rows, {r["B"]: [r["us"]] for r in rows}, clock=load, riccati=args.riccati,
                   problems_per_cta=args.problems_per_cta)


if __name__ == "__main__":
    main()
