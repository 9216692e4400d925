"""A/B timing of the generic (column per lane) and the column-pair step kernels (developer tool).
usage: python tools/exp_step2.py [B ...]   env MPCB200_KERNEL is set per arm by this script."""
import ctypes, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch, bench
dev = torch.device("cuda:0")
T, n, m = 20, 8, 2
Bs = [int(x) for x in sys.argv[1:]] or [4096, 65536]
sh = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def timeit(steppers, reps):
    for i in range(10):
        steppers[i % len(steppers)](sh)
    torch.cuda.synchronize()
    best = []
    for blk in range(5):
        e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
        e0.record()
        for i in range(reps):
            steppers[i % len(steppers)](sh)
        e1.record()
        torch.cuda.synchronize()
        best.append(e0.elapsed_time(e1) / reps * 1e3)
    return min(best), sorted(best)[len(best) // 2]


for B in Bs:
    nsets = 4 if B <= 8192 else 2
    sets = [bench.gen_inputs(3000 + s, B, T, n, m, dev) for s in range(nsets)]
    for box in (False, True):
        res = {}
        outs = {}
        for impl in ("1", "2"):
            os.environ["MPCB200_KERNEL"] = impl
            sts = [bench.RawStepper(s, B, T, n, m) for s in sets]
            if box:
                for st in sts:
                    st.dims.bounds_kind = 1
                    st.params.u_lo, st.params.u_hi = -0.25, 0.25
            res[impl] = timeit(sts, 40 if B <= 8192 else 10)
            sts[0](sh)
            torch.cuda.synchronize()
            outs[impl] = {k: v.clone() for k, v in sts[0].out.items()}
        d = max(float((outs["1"][k] - outs["2"][k]).abs().max()) for k in ("new_x", "new_u", "costs"))
        bps = bench.bytes_per_solve(T, n, m)
        print(f"B={B} box={box}: generic {res['1'][0]:.1f}/{res['1'][1]:.1f} us  pair {res['2'][0]:.1f}/{res['2'][1]:.1f} us (min/median)  "
              f"pair frac of HBM = {bps * B / (res['2'][0] * 1e-6) / 1e9 / bench.HBM_PEAK_GBS:.3f}  max|generic-pair| = {d:.2e}", flush=True)
