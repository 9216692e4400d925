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
# a shape without a compiled instance: the large-shape step (bounded, gains in Ks/ks) and, through autograd and then
# directly, mpcb200_lqr_adjoint_* (masked large step with its gains in the workspace + costate and outer-product
# kernels)
import ctypes
from mpc.pytorch_b200 import LQRStep, QuadCost, LinDx
from mpc.pytorch_b200._lib import Dims, Params, check, entry, lib, ptr
B, T, n, m, dt = 3, 4, 20, 5, torch.float64
C, c, F, f, x0 = [t.to(dev) for t in gen_problem(2, B, T, n, m, dt)]
u, ul, uu = nominal_controls(2, B, T, m, dt, 0.25)
u = u.to(dev)
x = get_traj(T, u, x0, LinDx(F, f))
lv = [t.clone().requires_grad_(True) for t in (x0, C, c, F, f)]
nx, nu = LQRStep(n, m, T, u_lower=ul, u_upper=uu, current_x=x, current_u=u, true_cost=QuadCost(lv[1], lv[2]),
                 true_dynamics=LinDx(lv[3], lv[4]))(*lv)[:2]
(nx.sum() + nu.sum()).backward()
dims = Dims(B=B, T=T, n=n, m=m, F_T=T - 1, has_f=1, bounds_kind=1, max_ls_iter=10, pnqp_max_iter=20, do_rollout=1)
nbytes = lib().mpcb200_adjoint_workspace_bytes(ctypes.byref(dims), 8)
ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
outs = [torch.empty_like(t) for t in (x0, C, c, F, f)]
ins = [C, c, F, nx.detach().contiguous(), nu.detach().contiguous(), torch.ones_like(x), torch.ones_like(u)]
check(entry("mpcb200_lqr_adjoint", dt)(ctypes.byref(dims), ctypes.byref(Params(u_lo=ul, u_hi=uu, ls_decay=0.2)),
                                       *[ptr(t) for t in ins], None, None, *[ptr(t) for t in outs], ptr(ws), nbytes,
                                       None), "adjoint")
torch.cuda.synchronize()
from mpc.pnqp import pnqp
for (B, n, dt) in [(2, 100, torch.float64), (3, 128, torch.float32)]:    # one thread block per QP
    g = torch.Generator().manual_seed(n)
    L = torch.randn(B, n, n, generator=g, dtype=torch.float64)
    H = (L @ L.transpose(1, 2) + 0.5 * torch.eye(n, dtype=torch.float64)).to(dt).to(dev)
    q = (2.0 * torch.randn(B, n, generator=g, dtype=torch.float64)).to(dt).to(dev)
    pnqp(H, q, -torch.rand(B, n, generator=g).to(dt).to(dev), torch.rand(B, n, generator=g).to(dt).to(dev))
    torch.cuda.synchronize()
# differentiable receding-horizon episodes: mpcb200_episode_plans_* and mpcb200_episode_backward_*, LinDx and pendulum
from mpc.pytorch_b200 import MPC
from mpc.pytorch_b200.dynamics import PendulumDx
from mpc.pytorch_b200.control import receding_horizon
B, T, n, m = 3, 4, 3, 2
C, c, F, f, x0 = [t.to(dev).requires_grad_(True) for t in gen_problem(3, B, T, n, m, torch.float32)]
ep = receding_horizon(MPC(n, m, T, u_lower=-0.3, u_upper=0.3, lqr_iter=3, verbose=-1), x0, QuadCost(C, c),
                      LinDx(F, f), 2, differentiable=True)
(ep.x.sum() + ep.u.sum()).backward()
pend = PendulumDx(params=torch.tensor((10.0, 1.0, 1.0), device=dev, requires_grad=True))
q, p = pend.get_true_obj()
x0 = torch.tensor([[1.0, 0.0, 0.1], [0.0, 1.0, -0.2]], device=dev, dtype=torch.float64, requires_grad=True)
ep = receding_horizon(MPC(3, 1, T, u_lower=-2.0, u_upper=2.0, lqr_iter=3, verbose=-1), x0,
                      QuadCost(torch.diag(q).double().to(dev), p.double().to(dev)), pend, 2, differentiable=True)
(ep.x.sum() + ep.u.sum()).backward()
torch.cuda.synchronize()
print("sanitize workload done")
