#!/usr/bin/env python3
"""Developer experiment: time the config-3 step kernel (device resident, rotating sets)."""
import ctypes, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench
B = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
bounded = len(sys.argv) > 2 and sys.argv[2] == "1"
dev = torch.device("cuda:0")
nsets = max(1, min(4, int(300e6 / (17128 * B)) + 1))
sets = [bench.gen_inputs(3000 + s, B, 20, 8, 2, dev) for s in range(nsets)]
st = [bench.RawStepper(s, B, 20, 8, 2) for s in sets]
if bounded:
    for s in st:
        s.dims.bounds_kind = 1
        s.params.u_lo, s.params.u_hi = -0.25, 0.25
sh = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
for i in range(40):
    st[i % nsets](sh)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
reps = 200
e0.record()
for i in range(reps):
    st[i % nsets](sh)
e1.record(); torch.cuda.synchronize()
us = e0.elapsed_time(e1) / reps * 1e3
print(f"lib={os.environ.get('MPCB200_LIB','default')[-20:]} dbg={os.environ.get('MPCB200_DEBUG','0')} B={B} bounded={bounded}: {us:.1f} us  {B/us:.2f} Msolves/s  {17128*B/us/1e3:.0f} GB/s ({17128*B/us/1e3/bench.HBM_PEAK_GBS*100:.1f}% of the HBM data-sheet peak)")
