#!/usr/bin/env python3
"""Fixtures for the learned / affine dynamics modules (SURVEY.md section 8(f) rank 2), from the REAL reference.

Run with a checkout of locuslab/mpc.pytorch:   MPC_REFERENCE=<checkout> python oracle/make_golden_nn.py
Imports the unmodified reference under the alias ``ref_mpc`` (oracle/make_golden.py: load_reference), builds its
``NNDynamics`` / ``AffineDynamics`` (reference mpc/dynamics.py:15-131, :159-205) with seeded weights, and stores the
weights, one batched step, the analytic Jacobians ``grad_input`` and a short box-constrained iLQR solve with
``GradMethods.ANALYTIC`` as tests/golden/nn_dynamics_*.npz / affine_dynamics_f64.npz.  Only numbers are stored.
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
from make_golden import load_reference, npz          # noqa: E402


def main():
    rmpc, _, _, _ = load_reference()
    import ref_mpc.dynamics as rdyn
    torch.set_default_dtype(torch.float64)
    n, m, B, T = 3, 2, 4, 8
    p = n + m
    for act in ("sigmoid", "relu"):
        torch.manual_seed(7 if act == "sigmoid" else 8)
        net = rdyn.NNDynamics(n, m, hidden_sizes=[12, 10], activation=act, passthrough=True).double()
        with torch.no_grad():
            for fc in net.fcs:                       # O(1) Jacobians so the iLQR problem is non-trivial
                fc.weight.mul_(1.5)
        xs, us = torch.randn(9, n), torch.randn(9, m)
        nxt = net(xs, us)
        R, S = net.grad_input(xs, us)
        L = torch.randn(T, B, p, p) / p ** 0.5
        C = L @ L.transpose(-1, -2) + torch.eye(p)
        c = 0.5 * torch.randn(T, B, p)
        x0 = torch.randn(B, n)
        with contextlib.redirect_stdout(io.StringIO()):
            x, u, costs = rmpc.MPC(n, m, T, u_lower=-0.6, u_upper=0.6, lqr_iter=12, verbose=-1,
                                   grad_method=rmpc.GradMethods.ANALYTIC, exit_unconverged=False,
                                   detach_unconverged=False, eps=1e-6)(x0, rmpc.QuadCost(C, c), net)
        with contextlib.redirect_stdout(io.StringIO()):          # same problem without bounds: no QP tolerance involved
            xf, uf, cf = rmpc.MPC(n, m, T, lqr_iter=12, verbose=-1, grad_method=rmpc.GradMethods.ANALYTIC,
                                  exit_unconverged=False, detach_unconverged=False, eps=1e-6)(
                x0, rmpc.QuadCost(C, c), net)
        ws = {f"W{i}": fc.weight for i, fc in enumerate(net.fcs)}
        ws.update({f"b{i}": fc.bias for i, fc in enumerate(net.fcs)})
        npz(f"nn_dynamics_{act}_f64", step_x=xs, step_u=us, step_next=nxt, R=R, S=S, C=C, c=c, x_init=x0,
            x=x, u=u, costs=costs, x_free=xf, u_free=uf, costs_free=cf, n_layers=np.int64(len(net.fcs)), **ws)
        print(act, "clamped fraction", float((u.abs() == 0.6).double().mean()), "cost", float(costs.mean()))
    # affine dynamics: x' = A x + B u + c (one system shared by the batch)
    torch.manual_seed(9)
    A = 0.9 * torch.eye(n) + 0.2 * torch.randn(n, n)
    Bm = torch.randn(n, m)
    cc = 0.1 * torch.randn(n)
    aff = rdyn.AffineDynamics(A, Bm, cc)
    L = torch.randn(T, B, p, p) / p ** 0.5
    C = L @ L.transpose(-1, -2) + torch.eye(p)
    c = 0.5 * torch.randn(T, B, p)
    x0 = torch.randn(B, n)
    with contextlib.redirect_stdout(io.StringIO()):
        x, u, costs = rmpc.MPC(n, m, T, u_lower=-0.5, u_upper=0.5, lqr_iter=12, verbose=-1,
                               grad_method=rmpc.GradMethods.ANALYTIC, exit_unconverged=False,
                               detach_unconverged=False, eps=1e-6)(x0, rmpc.QuadCost(C, c), aff)
    npz("affine_dynamics_f64", A=A, B=Bm, c0=cc, C=C, c=c, x_init=x0, x=x, u=u, costs=costs)
    print("affine clamped fraction", float((u.abs() == 0.5).double().mean()))


if __name__ == "__main__":
    main()


def grad_cases():
    """d u* / d c and d u* / d (first-layer bias) of the iLQR solution through NNDynamics, with and without a
    slew-rate penalty, from the reference's own autograd (the quantities its tests
    test_lqr_backward_cost_nn_dynamics_module_constrained[_slew] compare with finite differences,
    tests/test_mpc.py:560-744).  Seeds are searched until the solution is strictly partially on the bounds."""
    rmpc, _, _, _ = load_reference()
    import ref_mpc.dynamics as rdyn
    torch.set_default_dtype(torch.float64)
    n, m, T, B = 2, 2, 3, 1
    p = n + m
    for tag, slew in (("nn_grad_f64", None), ("nn_grad_slew_f64", 1.0)):
        for seed in range(50):
            torch.manual_seed(seed)
            net = rdyn.NNDynamics(n, m, hidden_sizes=[10, 10], activation="sigmoid").double()
            Cf = 10.0 * torch.randn(T, B, p, p)
            C = (Cf.transpose(-1, -2) @ Cf).requires_grad_(True)
            c = (10.0 * torch.randn(T, B, p)).requires_grad_(True)
            x0 = torch.randn(B, n)
            with contextlib.redirect_stdout(io.StringIO()):
                x, u, _ = rmpc.MPC(n, m, T, u_lower=-1.0, u_upper=1.0, lqr_iter=40, verbose=-1,
                                   exit_unconverged=False, max_linesearch_iter=1, slew_rate_penalty=slew,
                                   grad_method=rmpc.GradMethods.ANALYTIC)(x0, rmpc.QuadCost(C, c), net)
            uf = u.reshape(-1)
            on = uf.abs() == 1.0
            if bool(on.any()) and bool((~on).any()):
                break
        else:
            raise RuntimeError("no seed with a partially active solution")
        rows_c, rows_b = [], []
        for i in range(uf.numel()):
            gc, gb = torch.autograd.grad(uf[i], [c, net.fcs[0].bias], retain_graph=True)
            rows_c.append(gc.reshape(-1))
            rows_b.append(gb.reshape(-1))
        ws = {f"W{i}": fc.weight for i, fc in enumerate(net.fcs)}
        ws.update({f"b{i}": fc.bias for i, fc in enumerate(net.fcs)})
        npz(tag, C=C, c=c, x_init=x0, x=x, u=u, du_dc=torch.stack(rows_c), du_db0=torch.stack(rows_b),
            n_layers=np.int64(len(net.fcs)), seed=np.int64(seed), **ws)
        print(tag, "seed", seed, "on bound", int(on.sum()), "of", uf.numel(),
              "max|du/dc|", float(torch.stack(rows_c).abs().max()), "max|du/db0|", float(torch.stack(rows_b).abs().max()))


if __name__ == "__main__" and os.environ.get("GOLDEN_NN_GRAD", "1") == "1":
    grad_cases()


def load_ref_env(modname):
    """Import ref_mpc.env_dx.<modname> (needs matplotlib at import time: stubbed; imports `mpc.util` by its absolute
    name: aliased to the reference only while importing)."""
    import importlib
    import types
    load_reference()
    for mod in ("matplotlib", "matplotlib.pyplot"):
        sys.modules.setdefault(mod, types.ModuleType(mod))
    sys.modules["matplotlib"].use = lambda *a, **k: None
    sys.modules["matplotlib"].pyplot = sys.modules["matplotlib.pyplot"]
    sys.modules["matplotlib.pyplot"].style = types.SimpleNamespace(use=lambda *a, **k: None)
    saved = {k: sys.modules.pop(k) for k in list(sys.modules) if k == "mpc" or k.startswith("mpc.")}
    sys.modules["mpc"] = sys.modules["ref_mpc"]
    sys.modules["mpc.util"] = sys.modules["ref_mpc.util"]
    try:
        env = importlib.import_module("ref_mpc.env_dx." + modname)
    finally:
        for k in [k for k in sys.modules if k == "mpc" or k.startswith("mpc.")]:
            del sys.modules[k]
        sys.modules.update(saved)
    return env


def pendulum_case():
    """Pendulum swing-up iLQR (reference mpc/env_dx/pendulum.py: `simple` model, bounds +-2, decay 0.2, 5 line-search
    iterations), B=16, T=20, float64, AUTO_DIFF Jacobians, 15 iterations: trajectories of the unmodified reference."""
    rmpc, _, _, _ = load_reference()
    rpen = load_ref_env("pendulum")
    torch.set_default_dtype(torch.float64)
    torch.manual_seed(3)
    B, T = 16, 20
    dx = rpen.PendulumDx(params=torch.tensor((10.0, 1.0, 1.0)))
    th = (torch.rand(B) * 2 - 1) * np.pi
    x0 = torch.stack((torch.cos(th), torch.sin(th), torch.rand(B) * 2 - 1), 1)
    q, p = dx.get_true_obj()
    Q = torch.diag(q.double()).repeat(T, B, 1, 1)
    pp = p.double().repeat(T, B, 1)
    with contextlib.redirect_stdout(io.StringIO()):
        x, u, costs = rmpc.MPC(3, 1, T, u_lower=dx.lower, u_upper=dx.upper, lqr_iter=15, verbose=-1,
                               exit_unconverged=False, detach_unconverged=False, linesearch_decay=dx.linesearch_decay,
                               max_linesearch_iter=dx.max_linesearch_iter, grad_method=rmpc.GradMethods.AUTO_DIFF,
                               eps=dx.mpc_eps)(x0, rmpc.QuadCost(Q, pp), dx)
    npz("pendulum_ilqr_f64", x_init=x0, q=q.double(), p=p.double(), x=x, u=u, costs=costs, lqr_iter=np.int64(15))
    print("pendulum: clamped fraction", float((u.abs() == 2.0).double().mean()), "mean cost", float(costs.mean()))


if __name__ == "__main__" and os.environ.get("GOLDEN_PENDULUM", "1") == "1":
    pendulum_case()


def _known_states(name, B, g):
    """States of a known system with the angle pair (r cos th, r sin th) at radii 0.3, 1 and 3, not only 1."""
    th = (torch.rand(B, generator=g) * 2 - 1) * 3.0
    r = torch.tensor((0.3, 1.0, 3.0)).repeat(B)[:B]
    rest = lambda s: (torch.rand(B, generator=g) - 0.5) * s
    if name == "cartpole":
        return torch.stack((rest(1.0), rest(1.0), r * torch.cos(th), r * torch.sin(th), rest(2.0)), 1)
    return torch.stack((r * torch.cos(th), r * torch.sin(th), rest(2.0)), 1)


def _jacobians(module, xs, us):
    """R = dx'/dx, S = dx'/du of module(xs, us) by autograd (what the reference's AUTO_DIFF linearisation does)."""
    xs = xs.clone().requires_grad_(True)
    us = us.clone().requires_grad_(True)
    nx = module(xs, us)
    rows = [torch.autograd.grad(nx[:, j].sum(), [xs, us], retain_graph=True) for j in range(nx.shape[1])]
    return nx.detach(), torch.stack([r[0] for r in rows], 1), torch.stack([r[1] for r in rows], 1)


# non-default physics of each known system: parameters, dt, control clamp, step options
KNOWN_SYSTEMS = {
    "cartpole": dict(params=(9.81, 1.3, 0.25, 0.8), dt=0.04, clamp=("force_mag", 7.5), decay=0.3, ls_iter=4,
                     u_weight=0.03),
    "pendulum": dict(params=(9.1, 1.7, 0.6), dt=0.15, clamp=("max_torque", 1.5), decay=0.35, ls_iter=6,
                     u_weight=1.0),
}


def known_step_cases():
    """One LQR step whose line search rolls out a known nonlinear system (reference
    LQRStep(..., true_dynamics=<env module>, true_cost=QuadCost), mpc/lqr_step.py:217-225) at non-default physics,
    linearised along a rollout of nominal controls, with one x_init off the unit circle.  Two bound regimes: scalar
    bounds inside the system's control clamp, and bounds twice as wide, so that the clamp inside the dynamics
    engages.  Asserts that oracle.lqr_step_forward(dynamics=<our module>) equals the reference to 1e-10 with the
    same saturated controls, and stores inputs, outputs, next states and autograd Jacobians of the reference module
    as tests/golden/known_step_{cartpole,pendulum}_f64.npz."""
    from oracle import lqr_oracle as orc
    from mpc.pytorch_b200.dynamics import CartpoleDx, PendulumDx
    rmpc, rstep, _, _ = load_reference()
    torch.set_default_dtype(torch.float64)
    ours_cls = {"cartpole": CartpoleDx, "pendulum": PendulumDx}
    for name, spec in KNOWN_SYSTEMS.items():
        renv = load_ref_env(name)
        ref_cls = renv.CartpoleDx if name == "cartpole" else renv.PendulumDx
        ref = ref_cls(params=torch.tensor(spec["params"]))
        ours = ours_cls[name](params=torch.tensor(spec["params"]))
        for mod in (ref, ours):
            mod.dt = spec["dt"]
            setattr(mod, spec["clamp"][0], spec["clamp"][1])
        clamp = spec["clamp"][1]
        n, m, B, T = ref.n_state, 1, 7, 12
        p = n + m
        g = torch.Generator().manual_seed(31 if name == "cartpole" else 32)
        # one-step fixture: states at three radii, theta at +-pi with both signs of sin = 0 and near 0, controls
        # at, one ulp inside and one ulp outside the clamp, and well inside / outside it
        xs = _known_states(name, 24, g)
        ic, is_ = (2, 3) if name == "cartpole" else (0, 1)
        edge = ((-1.0, 0.0), (-1.0, -0.0), (1.0, 0.0), (1.0, 1e-9), (1.0, -1e-9), (-2.5, 0.0))
        for k, (cv, sv) in enumerate(edge):
            xs[k, ic], xs[k, is_] = cv, sv
        ulp_in, ulp_out = np.nextafter(clamp, 0.0), np.nextafter(clamp, np.inf)
        us = torch.tensor((clamp, -clamp, ulp_in, -ulp_in, ulp_out, -ulp_out, 0.5 * clamp, -3.0 * clamp)).repeat(3)
        us = us.view(-1, 1)
        step_next, R, S = _jacobians(ref, xs, us)
        o_next, oR, oS = _jacobians(ours, xs, us)
        assert maxdiff(o_next, step_next) <= 1e-13 and maxdiff(oR, R) <= 1e-12 and maxdiff(oS, S) <= 1e-12, name
        # the LQR step: nominal controls (some beyond the clamp), their rollout and its linearisation
        x0 = _known_states(name, B, g)
        u = (torch.rand(T, B, 1, generator=g) * 2 - 1) * 1.2 * clamp
        xs_ = [x0]
        for t in range(T - 1):
            xs_.append(ref(xs_[t], u[t]).detach())
        x = torch.stack(xs_)
        nx, Rl, Sl = _jacobians(ref, x[:-1].reshape(-1, n), u[:-1].reshape(-1, 1))
        F = torch.cat((Rl, Sl), 2).view(T - 1, B, n, p)
        f = (nx - torch.einsum("bij,bj->bi", Rl, x[:-1].reshape(-1, n))
             - torch.einsum("bij,bj->bi", Sl, u[:-1].reshape(-1, 1))).view(T - 1, B, n)
        Lc = torch.randn(T, B, p, p, generator=g) / p ** 0.5
        C = Lc @ Lc.transpose(-1, -2) + 0.5 * torch.eye(p)
        c = torch.randn(T, B, p, generator=g)
        # large requested state moves: controls on the bounds and first line-search passes that are worse than the
        # nominal trajectory, so the nonlinear rollout is pinned over several passes (alpha decays)
        c[..., :n] *= 20.0
        c[..., n:] = 0.0
        C[..., n:, :] *= spec["u_weight"]
        C[..., :, n:] *= spec["u_weight"]
        out = dict(params=torch.tensor(spec["params"]), dt=np.float64(spec["dt"]), clamp=np.float64(clamp),
                   decay=np.float64(spec["decay"]), ls_iter=np.int64(spec["ls_iter"]), step_x=xs, step_u=us,
                   step_next=step_next, R=R, S=S, x_init=x0, C=C, c=c, F=F, f=f, x=x, u=u)
        for tag, bound in (("in", 0.8 * clamp), ("wide", 2.0 * clamp)):
            with contextlib.redirect_stdout(io.StringIO()):
                rx, ru, nqp, rcost, rfdn, ralpha = rstep.LQRStep(
                    n, m, T, u_lower=-bound, u_upper=bound, linesearch_decay=spec["decay"],
                    max_linesearch_iter=spec["ls_iter"], true_cost=rmpc.QuadCost(C, c), true_dynamics=ref,
                    current_x=x, current_u=u)(x0, C, c, F, f)
            o = orc.lqr_step_forward(n, m, T, x0, C, c, F, f, x, u, u_lower=-bound, u_upper=bound,
                                     linesearch_decay=spec["decay"], max_linesearch_iter=spec["ls_iter"],
                                     coupled=True, dynamics=ours)
            for a, b in ((o.new_x, rx), (o.new_u, ru), (o.costs, rcost), (o.full_du_norm, rfdn),
                         (o.mean_alphas, ralpha)):
                assert maxdiff(a, b) <= 1e-10 * max(1.0, float(b.abs().max())), (name, tag, maxdiff(a, b))
            assert float(o.n_total_qp_iter) == float(nqp), (name, tag)
            for side in (-bound, bound):
                assert torch.equal(o.new_u == side, ru == side), (name, tag, "active set")
            beyond = float((ru.abs() > clamp).double().mean())
            print(f"known step {name} bounds {tag}: saturated {float((ru.abs() == bound).double().mean()):.2f}, "
                  f"beyond the clamp {beyond:.2f}, mean alpha {float(ralpha):.3f}")
            if tag == "wide":
                assert beyond > 0, "the in-dynamics clamp must engage"
            assert float(ralpha) < 1.0, "the line search must decay some alphas"
            out.update({f"bound_{tag}": np.float64(bound), f"new_x_{tag}": rx, f"new_u_{tag}": ru,
                        f"costs_{tag}": rcost, f"full_du_norm_{tag}": rfdn, f"mean_alpha_{tag}": ralpha,
                        f"n_qp_{tag}": float(nqp)})
        npz(f"known_step_{name}_f64", **out)


def maxdiff(a, b):
    return float((torch.as_tensor(a).double() - torch.as_tensor(b).double()).abs().max())


if __name__ == "__main__" and os.environ.get("GOLDEN_KNOWN_STEP", "1") == "1":
    known_step_cases()
