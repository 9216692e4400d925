#!/usr/bin/env python3
"""Fixtures for (n_state, n_ctrl) shapes without a compiled kernel instance (csrc/lqr_large.cu), from the REAL reference.

Run with a checkout of locuslab/mpc.pytorch:   MPC_REFERENCE=<checkout> python oracle/make_golden_large.py
Imports the unmodified reference under the alias ``ref_mpc`` (oracle/make_golden.py: load_reference), runs it in
float64 on CPU, asserts that oracle/lqr_oracle.py reproduces it, and stores inputs + the reference's outputs:
  large_slew_f64        MPC(16, 4, slew_rate_penalty=1.0) with box bounds, B=4, T=10 (the LQR step is (20, 4)), and
                        d u* / d c by the reference's autograd (one row per control entry);
  large_step_n14m7_f64  one unbounded LQRStep at (14, 7), forward and the gradients of a weighted loss;
  large_step_n24m8_f64  one LQRStep at (24, 8) with tensor bounds, run one problem at a time, so the stored outputs
                        have the per-problem pnqp control flow the kernels implement.
Only numbers are stored.
"""
import contextlib
import io
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from make_golden import close, gen_problem, load_reference, npz   # noqa: E402
import lqr_oracle as orc                                          # noqa: E402

F64 = torch.float64


def slew_augment(C, c, F, x0, prev, pen, n, m):
    """The (n+m, m) LQR problem the reference's slew-rate branch builds (mpc/mpc.py:362-445), state [u_{t-1}; x]."""
    T, B = C.shape[:2]
    p2 = n + 2 * m
    gI = pen * torch.eye(m, dtype=F64)
    C2 = torch.zeros(T, B, p2, p2, dtype=F64)
    C2[:, :, :m, :m] = gI
    C2[:, :, -m:, :m] = -gI
    C2[:, :, :m, -m:] = -gI
    C2[:, :, -m:, -m:] = gI
    C2[:, :, m:, m:] += C
    c2 = torch.cat((torch.zeros(T, B, m, dtype=F64), c), 2)
    F0 = torch.cat((torch.zeros(m, n + m, dtype=F64), torch.eye(m, dtype=F64)), 1).expand(T - 1, B, m, p2)
    F1 = torch.cat((torch.zeros(T - 1, B, n, m, dtype=F64), F), 3)
    F2 = torch.cat((F0, F1), 2).contiguous()
    return C2, c2, F2, torch.cat((prev, x0), 1)


def slew_case(rmpc):
    n, m, B, T, pen, bound = 16, 4, 4, 10, 1.0, 0.5
    C, c, F, _, x0 = gen_problem(401, B, T, n, m, F64)
    A, Bm = F[0, 0, :, :n].clone(), F[0, 0, :, n:].clone()      # one system for the batch (Module dynamics)
    F = torch.cat((A, Bm), 1).expand(T - 1, B, n, n + m).contiguous()
    prev = 0.2 * torch.randn(B, m, generator=torch.Generator().manual_seed(402), dtype=F64)

    class AffineDx(torch.nn.Module):   # the reference's slew branch needs Module dynamics (mpc/mpc.py:411-414)
        def forward(self, x, u):
            return x @ A.t() + u @ Bm.t()

    cl = c.clone().requires_grad_(True)
    with contextlib.redirect_stdout(io.StringIO()):
        xs, us, costs = rmpc.MPC(n, m, T, u_lower=-bound, u_upper=bound, lqr_iter=20, verbose=-1,
                                 exit_unconverged=False, detach_unconverged=False, slew_rate_penalty=pen,
                                 prev_ctrl=prev, eps=1e-9, grad_method=rmpc.GradMethods.AUTO_DIFF)(
            x0, rmpc.QuadCost(C, cl), AffineDx())
    uf = us.reshape(-1)
    rows = []
    with contextlib.redirect_stdout(io.StringIO()):
        for i in range(uf.numel()):
            rows.append(torch.autograd.grad(uf[i], cl, retain_graph=True)[0].reshape(-1))
    du_dc = torch.stack(rows)
    C2, c2, F2, x02 = slew_augment(C, c, F, x0, prev, pen, n, m)
    ox, ou, ocost, _ = orc.mpc_forward_lin(n + m, m, T, x02, C2, c2, F2, None, u_lower=-bound, u_upper=bound,
                                           lqr_iter=20, eps=1e-9, coupled=True)
    close(ou, us, 1e-10, "slew.u")
    close(ox[:, :, m:], xs, 1e-10, "slew.x")
    frac = float(((us.detach().abs() - bound).abs() <= 1e-8).double().mean())
    print(f"  large_slew_f64: fraction of clamped controls = {frac:.2f}, max|du/dc| = {float(du_dc.abs().max()):.3f}")
    npz("large_slew_f64", C=C, c=c, A=A, Bm=Bm, x_init=x0, prev_ctrl=prev, penalty=pen, bound=bound,
        lqr_iter=np.int64(20), x=xs, u=us, costs=costs, du_dc=du_dc)


def step_unbounded_case(rstep, rmpc, rutil):
    n, m, B, T = 14, 7, 3, 8
    C, c, F, f, x0 = gen_problem(411, B, T, n, m, F64)
    u = 0.1 * torch.randn(T, B, m, generator=torch.Generator().manual_seed(412), dtype=F64)
    x = rutil.get_traj(T, u, x0, rmpc.LinDx(F, f))
    leaves = [t.clone().requires_grad_(True) for t in (x0, C, c, F, f)]
    # one LQR step from the nominal (x, u) with the reference's own backward: MPC(lqr_iter=1, u_init=u) runs that
    # step, then differentiates its solution through the no-op LQRStep (mpc/mpc.py:318-337)
    with contextlib.redirect_stdout(io.StringIO()):
        nx, nu, costs = rmpc.MPC(n, m, T, u_init=u, lqr_iter=1, verbose=-1, exit_unconverged=False,
                                 detach_unconverged=False)(leaves[0], rmpc.QuadCost(leaves[1], leaves[2]),
                                                           rmpc.LinDx(leaves[3], leaves[4]))
    g = torch.Generator().manual_seed(413)
    wx = torch.randn(T, B, n, generator=g, dtype=F64)
    wu = torch.randn(T, B, m, generator=g, dtype=F64)
    with contextlib.redirect_stdout(io.StringIO()):
        grads = torch.autograd.grad((wx * nx).sum() + (wu * nu).sum(), leaves)
    o = orc.lqr_step_forward(n, m, T, x0, C, c, F, f, x, u, coupled=True)
    close(o.new_x, nx, 1e-10, "n14m7.x")
    close(o.new_u, nu, 1e-10, "n14m7.u")
    b = orc.lqr_step_backward(n, m, T, x0, C, c, F, f, nx.detach(), nu.detach(), wx, wu, coupled=True)
    for a, r, k in zip(b[:5], grads, ("dx_init", "dC", "dc", "dF", "df")):
        close(a, r, 1e-10, "n14m7." + k)
    npz("large_step_n14m7_f64", C=C, c=c, F=F, f=f, x_init=x0, cur_x=x, cur_u=u, new_x=nx, new_u=nu, costs=costs,
        wx=wx, wu=wu, dx_init=grads[0], dC=grads[1], dc=grads[2], dF=grads[3], df=grads[4])


def step_bounded_case(rstep, rmpc, rutil):
    n, m, B, T = 24, 8, 3, 6
    C, c, F, f, x0 = gen_problem(421, B, T, n, m, F64)
    g = torch.Generator().manual_seed(422)
    u = 0.1 * torch.randn(T, B, m, generator=g, dtype=F64)
    ul = -0.5 * torch.rand(T, B, m, generator=g, dtype=F64) - 0.05
    uu = 0.5 * torch.rand(T, B, m, generator=g, dtype=F64) + 0.05
    u = torch.maximum(torch.minimum(u, uu), ul)
    x = rutil.get_traj(T, u, x0, rmpc.LinDx(F, f))
    outs = []
    for i in range(B):                                        # one problem per call: per-problem pnqp semantics
        s = lambda t: t[:, i:i + 1]
        step = rstep.LQRStep(n, m, T, u_lower=s(ul), u_upper=s(uu), true_cost=rmpc.QuadCost(s(C), s(c)),
                             true_dynamics=rmpc.LinDx(s(F), s(f)), current_x=s(x), current_u=s(u))
        with contextlib.redirect_stdout(io.StringIO()):
            outs.append(step(x0[i:i + 1], s(C), s(c), s(F), s(f)))
    nx = torch.cat([o[0] for o in outs], 1)
    nu = torch.cat([o[1] for o in outs], 1)
    nqp = torch.cat([o[2] for o in outs])
    costs = torch.cat([o[3] for o in outs])
    o = orc.lqr_step_forward(n, m, T, x0, C, c, F, f, x, u, u_lower=ul, u_upper=uu, coupled=False)
    close(o.new_x, nx, 1e-10, "n24m8.x")
    close(o.new_u, nu, 1e-10, "n24m8.u")
    close(o.costs, costs, 1e-9, "n24m8.costs")
    frac = float(((nu - ul).abs() <= 1e-12).double().mean() + ((nu - uu).abs() <= 1e-12).double().mean())
    print(f"  large_step_n24m8_f64: fraction of clamped controls = {frac:.2f}, qp iterations {nqp.tolist()}")
    npz("large_step_n24m8_f64", C=C, c=c, F=F, f=f, x_init=x0, cur_x=x, cur_u=u, u_lower=ul, u_upper=uu,
        new_x=nx, new_u=nu, costs=costs, n_total_qp_iter=nqp)


def main():
    rmpc, rstep, _, rutil = load_reference()
    torch.set_default_dtype(F64)
    slew_case(rmpc)
    step_unbounded_case(rstep, rmpc, rutil)
    step_bounded_case(rstep, rmpc, rutil)


if __name__ == "__main__":
    main()
