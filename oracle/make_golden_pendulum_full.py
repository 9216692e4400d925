#!/usr/bin/env python3
"""Fixtures for the five-parameter pendulum, from the REAL reference.

Run with a checkout of locuslab/mpc.pytorch:   MPC_REFERENCE=<checkout> python oracle/make_golden_pendulum_full.py
Uses the unmodified reference's PendulumDx(params=(g, m, l, d, b), simple=False) (mpc/env_dx/pendulum.py:18-84),
CPU, float64, AUTO_DIFF, at non-default physics (PHYSICS: d != 0, b != 0, dt and max_torque changed, controls that
pass the clamp).  Writes, under tests/golden/ (only numbers are stored):
  known_step_pendulum_full_f64   one step on states at radii 0.3 / 1 / 3, theta at +-pi and near 0, controls at, one
                                 ulp inside and outside the clamp (step_next, R, S by autograd); a rollout and the
                                 reference's own AUTO_DIFF linearize_dynamics along it (roll_*); one LQRStep with the
                                 module as true dynamics, bounds inside the clamp ("in") and twice as wide ("wide");
  pendulum_full_ilqr_f64         MPC solves without bounds ("unb") and with box bounds ("box");
  known_slew_pendulum_full_f64   MPC solves with slew_rate_penalty and prev_ctrl, two bound regimes, as
                                 make_golden_slew.py stores them;
  paramgrad_pendulum_full_f64    params.grad of <wx, x> + <wu, u>, with x_lin and df, as make_golden_paramgrad.py
                                 stores them;
  receding_pendulum_full_f64     the pendulum notebook's control loop, as make_golden_receding.py runs it.
"""
import contextlib
import io
import math
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from make_golden import load_reference, npz                                   # noqa: E402
from make_golden_nn import _jacobians, _known_states, load_ref_env, maxdiff     # noqa: E402
from make_golden_receding import _uniform, guarded                              # noqa: E402

PHYSICS = dict(params=(9.1, 1.7, 0.6, 0.4, 0.25), dt=0.15, clamp=1.5, decay=0.35, ls_iter=6)
NOTEBOOK_PARAMS = (10.0, 1.0, 1.0, 0.3, 0.2)     # the receding-horizon episode: the notebook's physics plus d, b


def _model(renv, params=None):
    dx = renv.PendulumDx(params=torch.tensor(PHYSICS["params"]) if params is None else params, simple=False)
    dx.dt = PHYSICS["dt"]
    dx.max_torque = PHYSICS["clamp"]
    return dx


def _common():
    return dict(params=torch.tensor(PHYSICS["params"]), dt=np.float64(PHYSICS["dt"]),
                clamp=np.float64(PHYSICS["clamp"]), decay=np.float64(PHYSICS["decay"]),
                ls_iter=np.int64(PHYSICS["ls_iter"]))


def step_case(rmpc, rstep, renv):
    from oracle import lqr_oracle as orc
    from mpc.pytorch_b200.dynamics import PendulumDx
    ref = _model(renv)
    ours = PendulumDx(params=torch.tensor(PHYSICS["params"]), simple=False)
    ours.dt, ours.max_torque = PHYSICS["dt"], PHYSICS["clamp"]
    clamp = PHYSICS["clamp"]
    n, m, B, T = 3, 1, 7, 12
    p = n + m
    g = torch.Generator().manual_seed(64)
    xs = _known_states("pendulum", 24, g)
    edge = ((-1.0, 0.0), (-1.0, -0.0), (1.0, 0.0), (1.0, 1e-9), (1.0, -1e-9), (-2.5, 0.0))
    for k, (cv, sv) in enumerate(edge):
        xs[k, 0], xs[k, 1] = cv, sv
    ulp_in, ulp_out = np.nextafter(clamp, 0.0), np.nextafter(clamp, np.inf)
    us = torch.tensor((clamp, -clamp, ulp_in, -ulp_in, ulp_out, -ulp_out, 0.5 * clamp, -3.0 * clamp)).repeat(3)
    us = us.view(-1, 1)
    step_next, R, S = _jacobians(ref, xs, us)
    o_next, oR, oS = _jacobians(ours, xs, us)
    assert maxdiff(o_next, step_next) <= 1e-13 and maxdiff(oR, R) <= 1e-12 and maxdiff(oS, S) <= 1e-12
    # a rollout of the reference module and its AUTO_DIFF linearisation, as MPC.linearize_dynamics forms it
    Tr, Br = 9, 5
    rx0 = _known_states("pendulum", Br, g)
    ru = (torch.rand(Tr, Br, 1, generator=g) * 2 - 1) * 1.6 * clamp
    rx = [rx0]
    for t in range(Tr - 1):
        rx.append(ref(rx[t], ru[t]).detach())
    rx = torch.stack(rx)
    lin = rmpc.MPC(n, m, Tr, grad_method=rmpc.GradMethods.AUTO_DIFF)
    rF, rf = lin.linearize_dynamics(rx, ru, ref, diff=False)
    # one LQR step: nominal controls (some beyond the clamp), their rollout and its linearisation
    x0 = _known_states("pendulum", B, g)
    u = (torch.rand(T, B, 1, generator=g) * 2 - 1) * 1.2 * clamp
    x = [x0]
    for t in range(T - 1):
        x.append(ref(x[t], u[t]).detach())
    x = torch.stack(x)
    nx, Rl, Sl = _jacobians(ref, x[:-1].reshape(-1, n), u[:-1].reshape(-1, 1))
    F = torch.cat((Rl, Sl), 2).view(T - 1, B, n, p)
    f = (nx - torch.einsum("bij,bj->bi", Rl, x[:-1].reshape(-1, n))
         - torch.einsum("bij,bj->bi", Sl, u[:-1].reshape(-1, 1))).view(T - 1, B, n)
    Lc = torch.randn(T, B, p, p, generator=g) / p ** 0.5
    C = Lc @ Lc.transpose(-1, -2) + 0.5 * torch.eye(p)
    c = torch.randn(T, B, p, generator=g)
    c[..., :n] *= 20.0          # large requested moves: saturated controls and decaying line-search passes
    c[..., n:] = 0.0
    out = dict(_common(), step_x=xs, step_u=us, step_next=step_next, R=R, S=S, roll_x_init=rx0, roll_u=ru,
               roll_x=rx, roll_F=rF, roll_f=rf, x_init=x0, C=C, c=c, F=F, f=f, x=x, u=u)
    for tag, bound in (("in", 0.8 * clamp), ("wide", 2.0 * clamp)):
        with contextlib.redirect_stdout(io.StringIO()):
            nxr, nur, nqp, rcost, rfdn, ralpha = rstep.LQRStep(
                n, m, T, u_lower=-bound, u_upper=bound, linesearch_decay=PHYSICS["decay"],
                max_linesearch_iter=PHYSICS["ls_iter"], true_cost=rmpc.QuadCost(C, c), true_dynamics=ref,
                current_x=x, current_u=u)(x0, C, c, F, f)
        o = orc.lqr_step_forward(n, m, T, x0, C, c, F, f, x, u, u_lower=-bound, u_upper=bound,
                                 linesearch_decay=PHYSICS["decay"], max_linesearch_iter=PHYSICS["ls_iter"],
                                 coupled=True, dynamics=ours)
        for a, b in ((o.new_x, nxr), (o.new_u, nur), (o.costs, rcost), (o.full_du_norm, rfdn),
                     (o.mean_alphas, ralpha)):
            assert maxdiff(a, b) <= 1e-10 * max(1.0, float(b.abs().max())), (tag, maxdiff(a, b))
        beyond = float((nur.abs() > clamp).double().mean())
        print(f"step bounds {tag}: saturated {float((nur.abs() == bound).double().mean()):.2f}, beyond the clamp "
              f"{beyond:.2f}, mean alpha {float(ralpha):.3f}")
        if tag == "wide":
            assert beyond > 0, "the in-dynamics clamp must engage"
        assert float(ralpha) < 1.0, "the line search must decay some alphas"
        out.update({f"bound_{tag}": np.float64(bound), f"new_x_{tag}": nxr, f"new_u_{tag}": nur,
                    f"costs_{tag}": rcost, f"full_du_norm_{tag}": rfdn, f"mean_alpha_{tag}": ralpha,
                    f"n_qp_{tag}": float(nqp)})
    npz("known_step_pendulum_full_f64", **out)


def solve(rmpc, dx, x0, Q, pp, T, lqr_iter, **kw):
    with contextlib.redirect_stdout(io.StringIO()):
        return rmpc.MPC(3, 1, T, lqr_iter=lqr_iter, verbose=-1, exit_unconverged=False, detach_unconverged=False,
                        linesearch_decay=PHYSICS["decay"], max_linesearch_iter=PHYSICS["ls_iter"],
                        grad_method=rmpc.GradMethods.AUTO_DIFF, eps=1e-9, **kw)(x0, rmpc.QuadCost(Q, pp), dx)


def objective(dx, T, B, g, clamp):
    q, p = dx.get_true_obj()
    Q = torch.diag(q.double()).repeat(T, B, 1, 1)
    pp = p.double().repeat(T, B, 1)
    pp[..., 3:] = 0.3 * clamp * (torch.rand(T, B, 1, generator=g) - 0.5)       # some push on the controls
    return Q, pp


def ilqr_case(rmpc, renv):
    B, T, LQR_ITER = 6, 12, 15
    clamp = PHYSICS["clamp"]
    dx = _model(renv)
    g = torch.Generator().manual_seed(62)
    x0 = _known_states("pendulum", B, g)
    Q, pp = objective(dx, T, B, g, clamp)
    out = dict(_common(), lqr_iter=np.int64(LQR_ITER), x_init=x0, C=Q, c=pp)
    for tag, bound in (("unb", None), ("box", 0.8 * clamp)):
        kw = {} if bound is None else dict(u_lower=-bound, u_upper=bound)
        x, u, costs = solve(rmpc, dx, x0, Q, pp, T, LQR_ITER, **kw)
        print(f"ilqr {tag}: beyond the clamp {int((u.abs() > clamp).sum())} of {u.numel()}, mean cost "
              f"{float(costs.mean()):.4e}")
        out.update({f"x_{tag}": x, f"u_{tag}": u, f"costs_{tag}": costs})
        if bound is not None:
            out[f"bound_{tag}"] = np.float64(bound)
    assert bool((out["u_unb"].abs() > clamp).any()), "the unbounded solve must pass the clamp"
    npz("pendulum_full_ilqr_f64", **out)


def slew_case(rmpc, renv):
    PENALTY, B, T, LQR_ITER = 0.5, 6, 10, 12
    clamp = PHYSICS["clamp"]
    dx = _model(renv)
    g = torch.Generator().manual_seed(63)
    x0 = _known_states("pendulum", B, g)
    prev = torch.tensor((clamp, -clamp, np.nextafter(clamp, np.inf), -1.7 * clamp, 0.4 * clamp, 0.0))[:B].view(B, 1)
    Q, pp = objective(dx, T, B, g, clamp)
    out = dict(_common(), penalty=np.float64(PENALTY), lqr_iter=np.int64(LQR_ITER), x_init=x0, prev_ctrl=prev,
               C=Q, c=pp)
    for tag, bound in (("in", 0.8 * clamp), ("wide", 2.0 * clamp)):
        c = pp.clone().requires_grad_(True)
        with contextlib.redirect_stdout(io.StringIO()):
            x, u, costs = rmpc.MPC(3, 1, T, u_lower=-bound, u_upper=bound, lqr_iter=LQR_ITER, verbose=-1,
                                   exit_unconverged=False, detach_unconverged=False,
                                   linesearch_decay=PHYSICS["decay"], max_linesearch_iter=PHYSICS["ls_iter"],
                                   grad_method=rmpc.GradMethods.AUTO_DIFF, eps=1e-9, slew_rate_penalty=PENALTY,
                                   prev_ctrl=prev)(x0, rmpc.QuadCost(Q, c), dx)
        uf = u.reshape(-1)
        rows = [torch.autograd.grad(uf[i], c, retain_graph=True)[0].reshape(-1) for i in range(uf.numel())]
        print(f"slew bounds {tag}: on the bounds {int((u.abs() == bound).sum())} of {u.numel()}, beyond the clamp "
              f"{int((u.abs() > clamp).sum())}")
        out.update({f"bound_{tag}": np.float64(bound), f"x_{tag}": x, f"u_{tag}": u, f"costs_{tag}": costs,
                    f"du_dc_{tag}": torch.stack(rows)})
    npz("known_slew_pendulum_full_f64", **out)


def paramgrad_case(rmpc, renv):
    B, T, LQR_ITER = 5, 8, 15
    clamp = PHYSICS["clamp"]
    seen = {}
    orig = rmpc.MPC.linearize_dynamics

    def hooked(self, x, u, dynamics, diff):
        F, f = orig(self, x, u, dynamics, diff)
        if diff:
            f.register_hook(lambda gr: seen.__setitem__("df", gr.detach().clone()))
        return F, f

    g = torch.Generator().manual_seed(65)
    x0 = _known_states("pendulum", B, g)
    Q, pp = objective(_model(renv), T, B, g, clamp)
    wx = torch.randn(T, B, 3, generator=g)
    wu = torch.randn(T, B, 1, generator=g)
    out = dict(_common(), lqr_iter=np.int64(LQR_ITER), x_init=x0, C=Q, c=pp, wx=wx, wu=wu)
    rmpc.MPC.linearize_dynamics = hooked
    try:
        for tag, bound in (("unb", None), ("box", 0.8 * clamp)):
            params = torch.tensor(PHYSICS["params"]).requires_grad_(True)
            dx = _model(renv, params)
            kw = {} if bound is None else dict(u_lower=-bound, u_upper=bound)
            seen.clear()
            x, u, costs = solve(rmpc, dx, x0, Q, pp, T, LQR_ITER, **kw)
            ((wx * x).sum() + (wu * u).sum()).backward()
            with torch.no_grad():
                x_lin = [x0]
                for t in range(T - 1):
                    x_lin.append(dx(x_lin[t], u[t]))
                x_lin = torch.stack(x_lin)
            assert bool((params.grad != 0).all()), params.grad
            print(f"paramgrad {tag}: grad {params.grad.tolist()}, beyond the clamp {int((u.abs() > clamp).sum())}")
            out.update({f"x_{tag}": x, f"u_{tag}": u, f"x_lin_{tag}": x_lin, f"df_{tag}": seen["df"],
                        f"grad_{tag}": params.grad})
            if bound is not None:
                out[f"bound_{tag}"] = np.float64(bound)
    finally:
        rmpc.MPC.linearize_dynamics = orig
    npz("paramgrad_pendulum_full_f64", **out)


def receding_case(rmpc, renv):
    B, STEPS, T = 4, 15, 20
    dx = renv.PendulumDx(torch.tensor(NOTEBOOK_PARAMS), simple=False)
    torch.manual_seed(0)
    th, thdot = _uniform(B, -(1 / 2) * math.pi, (1 / 2) * math.pi), _uniform(B, -1., 1.)
    x0 = torch.stack((torch.cos(th), torch.sin(th), thdot), dim=1)
    q, p = dx.get_true_obj()
    Q = torch.diag(q).unsqueeze(0).unsqueeze(0).repeat(T, B, 1, 1)
    pp = p.unsqueeze(0).repeat(T, B, 1)

    def make(u_init, prev):
        return rmpc.MPC(3, 1, T, u_init=u_init, u_lower=dx.lower, u_upper=dx.upper, lqr_iter=50, verbose=0,
                        exit_unconverged=False, detach_unconverged=False, linesearch_decay=dx.linesearch_decay,
                        max_linesearch_iter=dx.max_linesearch_iter, grad_method=rmpc.GradMethods.AUTO_DIFF,
                        eps=1e-2, prev_ctrl=prev)
    xs, us, cs, it = guarded(rmpc, make, x0, rmpc.QuadCost(Q, pp), dx, STEPS)
    print("receding iterations", it.tolist())
    npz("receding_pendulum_full_f64", params=dx.params, x_init=x0, C=Q, c=pp, x=xs, u=us, costs=cs, iters=it,
        T=np.int64(T), n_steps=np.int64(STEPS), lqr_iter=np.int64(50), eps=np.float64(1e-2),
        decay=np.float64(dx.linesearch_decay), ls_iter=np.int64(dx.max_linesearch_iter))


def main():
    rmpc, rstep, _, _ = load_reference()
    torch.set_default_dtype(torch.float64)
    renv = load_ref_env("pendulum")
    step_case(rmpc, rstep, renv)
    ilqr_case(rmpc, renv)
    slew_case(rmpc, renv)
    paramgrad_case(rmpc, renv)
    receding_case(rmpc, renv)


if __name__ == "__main__":
    main()
