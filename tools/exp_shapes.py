"""Generic vs column-pair step kernel over shapes / batch sizes (developer tool): us per launch."""
import ctypes, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch, bench
dev = torch.device("cuda:0")
sh = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
CASES = [  # n, m, T, B, bounds
    (16, 4, 50, 4096, None), (16, 4, 50, 16384, None), (16, 4, 50, 4096, 0.25),
    (8, 2, 20, 1024, 0.25), (8, 2, 20, 16384, None), (8, 4, 20, 4096, None), (12, 4, 30, 4096, None),
    (4, 2, 20, 4096, None), (6, 2, 25, 128, 0.5), (2, 2, 10, 4096, None),
]
for (n, m, T, B, bounds) in CASES:
    bps = bench.bytes_per_solve(T, n, m)
    nsets = max(2, min(4, int(300e6 // (bps * B)) + 1))
    sets = [bench.gen_inputs(100 + s, B, T, n, m, dev) for s in range(nsets)]
    res = {}
    outs = {}
    for impl in ("1", "2"):
        os.environ["MPCB200_KERNEL"] = impl
        sts = [bench.RawStepper(s, B, T, n, m, bounds=bounds) for s in sets]
        try:
            res[impl] = bench.time_launches(sts, max(4, min(40, int(2e4 / max(1.0, bps * B / 2e6)))), torch.cuda.current_stream(dev), sh)
            sts[0](sh); torch.cuda.synchronize()
            outs[impl] = {k: v.clone() for k, v in sts[0].out.items()}
        except RuntimeError as e:
            res[impl] = float("nan"); print("  ", impl, e)
    d = max(float((outs["1"][k] - outs["2"][k]).abs().max()) for k in ("new_x", "new_u")) if len(outs) == 2 else float("nan")
    fl = bench.flops_per_solve(T, n, m) * B
    print(f"n={n} m={m} T={T} B={B} bounds={bounds}: generic {res['1']:.1f} us  pair {res['2']:.1f} us  "
          f"(pair: {bps * B / (res['2'] * 1e-6) / 1e9 / bench.HBM_PEAK_GBS:.3f} of HBM, {fl / (res['2'] * 1e-6) / 1e12 / bench.FP32_FMA_PEAK_TFLOPS:.3f} of fp32 FMA)  max|d|={d:.1e}", flush=True)
    del sets, sts
    torch.cuda.empty_cache()
