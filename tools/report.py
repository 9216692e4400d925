#!/usr/bin/env python3
"""Per-config measurements (BASELINE.json configs 1-5) of the step kernel, device resident, + the
adjoint path and the cartpole MPC loop.  Prints a markdown table."""
import ctypes, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench
from mpc.pytorch_b200.step import lqr_step_raw, lqr_grad_raw

dev = torch.device("cuda:0")
PEAK = bench.HBM_PEAK_GBS


def time_step(B, T, n, m, bounds=None, reps=None):
    bps = bench.bytes_per_solve(T, n, m, tensor_bounds=(bounds == "tensor"))
    nsets = max(1, min(6, int(300e6 / (bps * B)) + 1))
    sets = [bench.gen_inputs(500 + s, B, T, n, m, dev) for s in range(nsets)]
    kw = {}
    if bounds == "tensor":
        kw = dict(u_lower=-0.5 * torch.rand(T, B, m, device=dev) - 0.02, u_upper=0.5 * torch.rand(T, B, m, device=dev) + 0.02)
    elif bounds is not None:
        kw = dict(u_lower=-bounds, u_upper=bounds)
    def run(s):
        return lqr_step_raw(n, m, T, s["x_init"], s["C"], s["c"], s["F"], s["f"], s["cur_x"], s["cur_u"], want_stats=False, **kw)
    for i in range(6):
        run(sets[i % nsets])
    torch.cuda.synchronize()
    reps = reps or max(10, min(200, int(2e9 / (bps * B))))
    e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
    e0.record()
    for i in range(reps):
        run(sets[i % nsets])
    e1.record(); torch.cuda.synchronize()
    us = e0.elapsed_time(e1) / reps * 1e3
    return us, B / us, bps * B / us / 1e3, bps


rows = []
for name, B, T, n, m, bounds in [
        ("1: TV-LQR example size", 1, 5, 3, 1, None),
        ("2-sized: cartpole LQR step", 128, 25, 5, 1, 100.0),
        ("3: random LTI (roofline run)", 4096, 20, 8, 2, None),
        ("3 with box +-0.25", 4096, 20, 8, 2, 0.25),
        ("3 at steady-state batch", 65536, 20, 8, 2, None),
        ("4: box pnqp, tensor bounds", 1024, 20, 8, 2, "tensor"),
        ("4 with scalar bounds +-0.25", 1024, 20, 8, 2, 0.25),
        ("5 shard (32768/8 per GPU)", 4096, 50, 16, 4, None),
        ("5 shard (32768/2 per GPU)", 16384, 50, 16, 4, None)]:
    us, msps, gbs, bps = time_step(B, T, n, m, bounds)
    rows.append((name, B, T, n, m, bounds, us, msps, gbs, bps))

print("| config | B,T,n,m | bounds | time/launch (us) | M solves/s | algorithmic GB/s | frac of %.0f GB/s | B/solve |" % PEAK)
print("|---|---|---|---|---|---|---|---|")
for name, B, T, n, m, bounds, us, msps, gbs, bps in rows:
    print(f"| {name} | {B},{T},{n},{m} | {bounds} | {us:.1f} | {msps:.2f} | {gbs:.0f} | {gbs / PEAK:.3f} | {bps} |")
print("\n(time/launch includes the Python/ctypes launch path of `lqr_step_raw`; small configs are launch bound.)")

# cartpole MPC (config 2 recipe), full iLQR: known system in the kernels vs the same physics as an opaque Module
from mpc import mpc
from mpc.env_dx.cartpole import CartpoleDx
from tests.cartpole import initial_states
B, T = 128, 25
dx = CartpoleDx()


class Opaque(torch.nn.Module):
    def forward(self, x, u):
        return dx(x, u)


x0 = initial_states(B, 0).to(dev)
q, p = dx.get_true_obj()
Q = torch.diag(q).repeat(T, B, 1, 1).to(dev)
pp = p.repeat(T, B, 1).to(dev)
print()
for name, dyn in (("known system: rollout, Jacobians and line search inside kernels", dx),
                  ("opaque nn.Module: autograd linearisation + torch rollout (round-1 path)", Opaque())):
    ctrl = mpc.MPC(5, 1, T, u_lower=-100.0, u_upper=100.0, lqr_iter=50, verbose=-1, exit_unconverged=False,
                   detach_unconverged=False, linesearch_decay=0.5, max_linesearch_iter=2,
                   grad_method=mpc.GradMethods.AUTO_DIFF, eps=1e-2)
    ctrl(x0, mpc.QuadCost(Q, pp), dyn)
    torch.cuda.synchronize(); t0 = time.perf_counter()
    for _ in range(3):
        ctrl(x0, mpc.QuadCost(Q, pp), dyn)
    torch.cuda.synchronize(); dt = (time.perf_counter() - t0) / 3
    print(f"cartpole MPC.forward (config 2: B=128, T=25, <=50 iLQR iterations, AUTO_DIFF), {name}: {dt * 1e3:.1f} ms -> "
          f"{B / dt:.0f} MPC-solves/s  (reference CPU, SURVEY section 6: 5.85 s, 22 MPC-solves/s)")
