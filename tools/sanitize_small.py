"""Tiny workload for compute-sanitizer (memcheck / racecheck / synccheck): every kernel + mode once."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from tests.helpers import gen_problem, nominal_controls
from mpc.pytorch_b200.step import lqr_step_raw, lqr_grad_raw
from mpc.pytorch_b200.solver import get_traj, LinDx
dev = torch.device("cuda:0")
for (B, T, n, m, dt) in [(13, 6, 8, 2, torch.float32), (7, 5, 3, 1, torch.float64), (5, 4, 16, 4, torch.float32)]:
    C, c, F, f, x0 = [t.to(dev) for t in gen_problem(1, B, T, n, m, dt)]
    u, ul, uu = nominal_controls(1, B, T, m, dt, 0.25)
    u = u.to(dev)
    x = get_traj(T, u, x0, LinDx(F, f))
    o = lqr_step_raw(n, m, T, x0, C, c, F, f, x, u, want_gains=True, want_du_first=True)
    o = lqr_step_raw(n, m, T, x0, C, c, F, f, x, u, u_lower=ul, u_upper=uu)
    I = (o["new_u"].abs() - 0.25).abs() <= 1e-8
    a = lqr_step_raw(n, m, T, torch.zeros_like(x0), C, -torch.cat((x, u), 2), F, None, torch.zeros_like(x), torch.zeros_like(u), u_zero_I=I)
    g = lqr_grad_raw(n, m, T, C, c, F, o["new_x"], o["new_u"], a["new_x"], a["new_u"], x, True)
    torch.cuda.synchronize()
from mpc.pnqp import pnqp
for (B, n, dt) in [(2, 100, torch.float64), (3, 128, torch.float32)]:    # one thread block per QP
    g = torch.Generator().manual_seed(n)
    L = torch.randn(B, n, n, generator=g, dtype=torch.float64)
    H = (L @ L.transpose(1, 2) + 0.5 * torch.eye(n, dtype=torch.float64)).to(dt).to(dev)
    q = (2.0 * torch.randn(B, n, generator=g, dtype=torch.float64)).to(dt).to(dev)
    pnqp(H, q, -torch.rand(B, n, generator=g).to(dt).to(dev), torch.rand(B, n, generator=g).to(dt).to(dev))
    torch.cuda.synchronize()
print("sanitize workload done")
