#!/usr/bin/env python3
"""Generate tests/golden/*.npz from the REAL reference.

Run with a checkout of locuslab/mpc.pytorch:   MPC_REFERENCE=<checkout> python oracle/make_golden.py
It imports the unmodified reference package under the alias ``ref_mpc`` (so it
cannot collide with this repo's drop-in ``mpc`` package), runs it on seeded
inputs on CPU, checks that oracle/lqr_oracle.py (coupled=True) reproduces it,
and stores inputs + the reference's outputs as small .npz fixtures.  Tests only
ever read the fixtures; they never need the reference.

No reference source is copied: only its numerical outputs are stored.
"""
import contextlib
import importlib.util
import io
import os
import sys
import warnings
import zlib

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLD = os.path.join(ROOT, "tests", "golden")
REF = os.environ.get("MPC_REFERENCE")
sys.path.insert(0, ROOT)
warnings.filterwarnings("ignore")


def load_reference():
    if not REF:
        raise SystemExit("set MPC_REFERENCE to a checkout of locuslab/mpc.pytorch")
    spec = importlib.util.spec_from_file_location(
        "ref_mpc", os.path.join(REF, "mpc", "__init__.py"),
        submodule_search_locations=[os.path.join(REF, "mpc")])
    pkg = importlib.util.module_from_spec(spec)
    sys.modules["ref_mpc"] = pkg
    spec.loader.exec_module(pkg)
    import ref_mpc.mpc as rmpc          # noqa
    import ref_mpc.lqr_step as rstep    # noqa
    import ref_mpc.pnqp as rpnqp        # noqa
    import ref_mpc.util as rutil        # noqa
    return rmpc, rstep, rpnqp, rutil


def gen_problem(seed, B, T, n, m, dtype, time_varying=False, with_f=True):
    """Well-conditioned synthetic generator (SURVEY.md section 8d)."""
    g = torch.Generator().manual_seed(seed)
    p = n + m
    L = torch.randn(T, B, p, p, generator=g, dtype=torch.float64) / p ** 0.5
    C = L @ L.transpose(-1, -2) + torch.eye(p, dtype=torch.float64)
    c = torch.randn(T, B, p, generator=g, dtype=torch.float64)
    if time_varying:
        A = 0.9 * torch.eye(n, dtype=torch.float64) + 0.1 * torch.randn(T - 1, B, n, n, generator=g, dtype=torch.float64) / n ** 0.5
        Bm = torch.randn(T - 1, B, n, m, generator=g, dtype=torch.float64) / n ** 0.5
        F = torch.cat((A, Bm), -1)
    else:
        A = 0.9 * torch.eye(n, dtype=torch.float64) + 0.1 * torch.randn(B, n, n, generator=g, dtype=torch.float64) / n ** 0.5
        Bm = torch.randn(B, n, m, generator=g, dtype=torch.float64) / n ** 0.5
        F = torch.cat((A, Bm), -1).unsqueeze(0).repeat(T - 1, 1, 1, 1)
    f = 0.1 * torch.randn(T - 1, B, n, generator=g, dtype=torch.float64)
    x0 = torch.randn(B, n, generator=g, dtype=torch.float64)
    out = [t.to(dtype).contiguous() for t in (C, c, F, f, x0)]
    if not with_f:
        out[3] = None
    return out


def npz(name, **kw):
    arrs = {}
    for k, v in kw.items():
        if v is None:
            continue
        if torch.is_tensor(v):
            v = v.detach().cpu().numpy()
        arrs[k] = np.asarray(v)
    np.savez_compressed(os.path.join(GOLD, name + ".npz"), **arrs)
    print("wrote", name, {k: a.shape for k, a in arrs.items()})


def close(a, b, tol, what):
    d = float((a - b).abs().max()) if a.numel() else 0.0
    assert d <= tol, f"oracle != reference for {what}: max|d|={d:g} > {tol:g}"
    return d


def main():
    os.makedirs(GOLD, exist_ok=True)
    rmpc, rstep, rpnqp, rutil = load_reference()
    from oracle import lqr_oracle as orc

    # ---------------------------------------------------------------- pnqp
    for name, B, n, dtype, warm in [("pnqp_f64_cold", 6, 5, torch.float64, False),
                                    ("pnqp_f64_warm", 6, 4, torch.float64, True),
                                    ("pnqp_f32_cold", 5, 3, torch.float32, False),
                                    ("pnqp_f64_n1", 7, 1, torch.float64, False),
                                    ("pnqp_f64_n100", 2, 100, torch.float64, False)]:
        g = torch.Generator().manual_seed(zlib.crc32(name.encode()) % 1000 + 17)
        Lm = torch.randn(B, n, n, generator=g, dtype=torch.float64)
        H = (Lm @ Lm.transpose(1, 2) + 0.5 * torch.eye(n, dtype=torch.float64)).to(dtype)
        q = (2.0 * torch.randn(B, n, generator=g, dtype=torch.float64)).to(dtype)
        lo = (-torch.rand(B, n, generator=g, dtype=torch.float64)).to(dtype)
        hi = (torch.rand(B, n, generator=g, dtype=torch.float64)).to(dtype)
        x0 = (0.3 * torch.randn(B, n, generator=g, dtype=torch.float64)).to(dtype) if warm else None
        with contextlib.redirect_stdout(io.StringIO()):
            xr, _, Ifr, ir = rpnqp.pnqp(H, q, lo, hi, x_init=x0, n_iter=20)
        xo, _, Ifo, io_ = orc.pnqp(H, q, lo, hi, x_init=x0, n_iter=20, coupled=True)
        close(xo, xr, 1e-12 if dtype == torch.float64 else 1e-6, name + ".x")
        assert torch.equal(Ifo, Ifr.to(Ifo.dtype)), name + ".If"
        assert int(io_.max()) == int(ir), (name, io_, ir)
        npz(name, H=H, q=q, lower=lo, upper=hi, x_init=x0, x=xr, If=Ifr, n_iter=np.int64(ir))

    # ---------------------------------------------------------------- LQRStep forward
    cases = [
        # name, seed, B,T,n,m, dtype, bounds, delta_u, time_varying, with_f
        ("step_cfg1_f32", 101, 1, 5, 3, 1, torch.float32, None, None, True, True),
        ("step_unb_m2_f64", 102, 4, 6, 4, 2, torch.float64, None, None, False, True),
        ("step_unb_m2_f32", 103, 5, 7, 8, 2, torch.float32, None, None, False, False),
        ("step_box_scalar_f64", 104, 8, 8, 4, 2, torch.float64, 0.25, None, False, True),
        ("step_box_scalar_f32", 105, 8, 20, 8, 2, torch.float32, 0.25, None, False, True),
        ("step_box_tensor_f64", 106, 6, 6, 3, 4, torch.float64, "tensor", None, True, True),
        ("step_box_delta_f64", 107, 4, 6, 3, 2, torch.float64, 0.5, 0.1, False, True),
        ("step_box_m1_f64", 108, 6, 9, 5, 1, torch.float64, 0.3, None, False, False),
        ("step_box_n16m4_f32", 109, 3, 12, 16, 4, torch.float32, 0.25, None, False, True),
    ]
    for (name, seed, B, T, n, m, dtype, bounds, delta_u, tv, wf) in cases:
        C, c, F, f, x0 = gen_problem(seed, B, T, n, m, dtype, tv, wf)
        g = torch.Generator().manual_seed(seed + 7)
        u = (0.1 * torch.randn(T, B, m, generator=g, dtype=torch.float64)).to(dtype)
        if bounds is None:
            ul = uu = None
        elif bounds == "tensor":
            ul = (-0.5 * torch.rand(T, B, m, generator=g, dtype=torch.float64) - 0.05).to(dtype)
            uu = (0.5 * torch.rand(T, B, m, generator=g, dtype=torch.float64) + 0.05).to(dtype)
            u = torch.maximum(torch.minimum(u, uu), ul)
        else:
            ul, uu = -float(bounds), float(bounds)
            u = u.clamp(ul, uu)
        x = rutil.get_traj(T, u, x0, rmpc.LinDx(F, f))
        step = rstep.LQRStep(n, m, T, u_lower=ul, u_upper=uu, delta_u=delta_u,
                             true_cost=rmpc.QuadCost(C, c), true_dynamics=rmpc.LinDx(F, f),
                             current_x=x, current_u=u)
        with contextlib.redirect_stdout(io.StringIO()):
            nx, nu, nqp, costs, fdn, ma = step(x0, C, c, F, f if f is not None else torch.Tensor())
        o = orc.lqr_step_forward(n, m, T, x0, C, c, F, f, x, u, u_lower=ul, u_upper=uu,
                                 delta_u=delta_u, coupled=True)
        tol = 1e-10 if dtype == torch.float64 else 2e-5
        close(o.new_x, nx, tol, name + ".x"); close(o.new_u, nu, tol, name + ".u")
        close(o.costs, costs, tol * 50, name + ".costs")
        close(o.full_du_norm, fdn, tol * 10, name + ".fdn")
        close(o.mean_alphas, ma, 1e-12, name + ".alphas")
        if dtype == torch.float64:
            assert float(o.n_total_qp_iter) == float(nqp), (name, o.n_total_qp_iter, nqp)
        npz(name, C=C, c=c, F=F, f=f, x_init=x0, cur_x=x, cur_u=u,
            u_lower=ul, u_upper=uu, delta_u=delta_u,
            new_x=nx, new_u=nu, n_total_qp_iter=nqp, costs=costs, full_du_norm=fdn, mean_alphas=ma)

    # ---------------------------------------------------------------- MPC forward + autograd backward
    gcases = [
        ("grad_unb_f64", 201, 3, 5, 3, 2, None, 1),
        ("grad_box_f64", 202, 4, 6, 4, 2, 0.35, 12),
        ("grad_box_m1_f64", 203, 3, 5, 3, 1, 0.3, 12),
        ("grad_unb_m1_f64", 204, 2, 4, 2, 1, None, 1),
    ]
    for (name, seed, B, T, n, m, bounds, iters) in gcases:
        C, c, F, f, x0 = gen_problem(seed, B, T, n, m, torch.float64, True, True)
        leaves = [t.clone().requires_grad_(True) for t in (x0, C, c, F, f)]
        ul, uu = (None, None) if bounds is None else (-bounds, bounds)
        ctrl = rmpc.MPC(n, m, T, u_lower=ul, u_upper=uu, lqr_iter=iters, verbose=-1,
                        exit_unconverged=False, detach_unconverged=False, eps=1e-9, back_eps=1e-9)
        with contextlib.redirect_stdout(io.StringIO()):
            xs, us, costs = ctrl(leaves[0], rmpc.QuadCost(leaves[1], leaves[2]), rmpc.LinDx(leaves[3], leaves[4]))
        g = torch.Generator().manual_seed(seed + 3)
        wx = torch.randn(T, B, n, generator=g, dtype=torch.float64)
        wu = torch.randn(T, B, m, generator=g, dtype=torch.float64)
        loss = (wx * xs).sum() + (wu * us).sum()
        with contextlib.redirect_stdout(io.StringIO()):
            grads = torch.autograd.grad(loss, leaves)
        o = orc.lqr_step_backward(n, m, T, x0, C, c, F, f, xs.detach(), us.detach(), wx, wu,
                                  u_lower=ul, u_upper=uu, coupled=True)
        for a, b, nm in zip(o[:5], grads, ("dx_init", "dC", "dc", "dF", "df")):
            close(a, b, 1e-9, name + "." + nm)
        ox, ou, ocost, _ = orc.mpc_forward_lin(n, m, T, x0, C, c, F, f, u_lower=ul, u_upper=uu,
                                               lqr_iter=iters, eps=1e-9, coupled=True)
        close(ox, xs.detach(), 1e-9, name + ".mpc_x"); close(ou, us.detach(), 1e-9, name + ".mpc_u")
        if bounds is not None:
            frac = float(((us.detach().abs() - bounds).abs() <= 1e-8).double().mean())
            print(f"  {name}: fraction of clamped controls = {frac:.2f}")
        npz(name, C=C, c=c, F=F, f=f, x_init=x0, bound=bounds, lqr_iter=np.int64(iters),
            x=xs, u=us, costs=costs, wx=wx, wu=wu,
            dx_init=grads[0], dC=grads[1], dc=grads[2], dF=grads[3], df=grads[4])

    # ---------------------------------------------------------------- slew-rate penalty (reference mpc/mpc.py:362-445)
    # (the reference's slew branch only works with Module dynamics: for LinDx it passes true_dynamics=None, :411-414)
    class AffineDx(torch.nn.Module):
        def __init__(self, A, Bm):
            super().__init__()
            self.A, self.Bm = A, Bm

        def forward(self, x, u):
            return x @ self.A.t() + u @ self.Bm.t()

    for name, seed, B, T, n, m, pen, bounds, with_prev in [("slew_box_f64", 301, 3, 7, 3, 2, 0.5, 0.4, True),
                                                            ("slew_unb_f64", 302, 2, 6, 4, 2, 2.0, None, False)]:
        C, c, _, _, x0 = gen_problem(seed, B, T, n, m, torch.float64, False, True)
        g = torch.Generator().manual_seed(seed + 1)
        A = 0.9 * torch.eye(n, dtype=torch.float64) + 0.1 * torch.randn(n, n, generator=g, dtype=torch.float64) / n ** 0.5
        Bm = torch.randn(n, m, generator=g, dtype=torch.float64) / n ** 0.5
        prev = 0.2 * torch.randn(B, m, generator=g, dtype=torch.float64) if with_prev else None
        ul, uu = (None, None) if bounds is None else (-bounds, bounds)
        with contextlib.redirect_stdout(io.StringIO()):
            xs, us, costs = rmpc.MPC(n, m, T, u_lower=ul, u_upper=uu, lqr_iter=15, verbose=-1, exit_unconverged=False,
                                     detach_unconverged=False, slew_rate_penalty=pen, prev_ctrl=prev, eps=1e-9,
                                     grad_method=rmpc.GradMethods.AUTO_DIFF)(
                x0, rmpc.QuadCost(C, c), AffineDx(A, Bm))
        npz(name, C=C, c=c, A=A, Bm=Bm, x_init=x0, bound=bounds, penalty=pen, prev_ctrl=prev, x=xs, u=us, costs=costs)

    # ---------------------------------------------------------------- TV-LQR notebook trace
    # examples/Time Varying Linear-Quadratic Control.ipynb (cell 2); its recorded output
    # is the only golden output stored inside the reference tree.
    torch.manual_seed(0)
    B, n, m, T = 2, 3, 4, 5
    p = n + m
    C = torch.randn(T * B, p, p)
    C = torch.bmm(C, C.transpose(1, 2)).view(T, B, p, p)
    c = torch.randn(T, B, p)
    R = (torch.eye(n) + 0.2 * torch.randn(n, n)).repeat(T, B, 1, 1)
    S = torch.randn(T, B, n, m)
    F = torch.cat((R, S), dim=3)
    x0 = torch.randn(B, n)
    ul = -torch.rand(T, B, m)
    uu = torch.rand(T, B, m)
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        xs, us, costs = rmpc.MPC(n_state=n, n_ctrl=m, T=T, u_lower=ul, u_upper=uu, lqr_iter=20,
                                 verbose=1, backprop=False, exit_unconverged=False)(
            x0, rmpc.QuadCost(C, c), rmpc.LinDx(F))
    printed = buf.getvalue()
    mean_costs = []
    for line in printed.splitlines():
        if line.startswith("|") and "iter" not in line:
            mean_costs.append(float(line.split("|")[2]))
    notebook = [6.6806, 6.4417, 4.5778, 4.4537, 4.4527]        # ipynb:26-36
    for a, b in zip(mean_costs, notebook):
        assert abs(a - b) < 5e-4, (mean_costs, notebook)
    trace = []
    ox, ou, oc, _ = orc.mpc_forward_lin(n, m, T, x0, C, c, F, None, u_lower=ul, u_upper=uu,
                                        lqr_iter=20, coupled=True, trace=trace)
    close(ox, xs, 5e-4, "tvlqr.x"); close(ou, us, 5e-4, "tvlqr.u")
    npz("tvlqr_notebook_f32", C=C, c=c, F=F, x_init=x0, u_lower=ul, u_upper=uu,
        x=xs, u=us, costs=costs, mean_costs=np.array(mean_costs),
        notebook_mean_costs=np.array(notebook))
    # ---------------------------------------------------------------- cartpole iLQR (config 2 recipe, small)
    # reference CartpoleDx needs matplotlib at import time (mpc/env_dx/cartpole.py:18-21): stub it.
    import types
    for mod in ("matplotlib", "matplotlib.pyplot"):
        sys.modules.setdefault(mod, types.ModuleType(mod))
    sys.modules["matplotlib"].use = lambda *a, **k: None
    sys.modules["matplotlib"].pyplot = sys.modules["matplotlib.pyplot"]
    sys.modules["matplotlib.pyplot"].style = types.SimpleNamespace(use=lambda *a, **k: None)
    # the env module imports the package by its absolute name (`from mpc import util`):
    # alias the reference under that name only while it is being imported.
    saved = {k: sys.modules.pop(k) for k in list(sys.modules) if k == "mpc" or k.startswith("mpc.")}
    sys.modules["mpc"] = sys.modules["ref_mpc"]
    sys.modules["mpc.util"] = sys.modules["ref_mpc.util"]
    import ref_mpc.env_dx.cartpole as rcart
    for k in [k for k in sys.modules if k == "mpc" or k.startswith("mpc.")]:
        del sys.modules[k]
    sys.modules.update(saved)
    from tests.cartpole import Cartpole, initial_states
    dxr, mine = rcart.CartpoleDx(), Cartpole()
    B, T = 6, 12
    x0 = initial_states(B, seed=0)
    uu_ = torch.randn(B, 1)
    close(mine(x0, uu_), dxr(x0, uu_), 1e-6, "cartpole.step")
    q, p = dxr.get_true_obj()
    q2, p2 = Cartpole.objective()
    close(q2, q.data, 0, "cartpole.q"); close(p2, p.data, 0, "cartpole.p")
    Q = torch.diag(q.data).unsqueeze(0).unsqueeze(0).repeat(T, B, 1, 1)
    pp = p.data.unsqueeze(0).repeat(T, B, 1)
    # (the reference's FINITE_DIFF path raises for batched Module dynamics; AUTO_DIFF is what its notebooks use)
    for gm_name, gm in (("AUTO_DIFF", rmpc.GradMethods.AUTO_DIFF),):
        with contextlib.redirect_stdout(io.StringIO()):
            xs, us, costs = rmpc.MPC(5, 1, T, u_lower=dxr.lower, u_upper=dxr.upper, lqr_iter=8, verbose=-1,
                                     exit_unconverged=False, detach_unconverged=False,
                                     linesearch_decay=dxr.linesearch_decay,
                                     max_linesearch_iter=dxr.max_linesearch_iter,
                                     grad_method=gm, eps=1e-2)(x0, rmpc.QuadCost(Q, pp), dxr)
        npz("cartpole_" + gm_name.lower() + "_f32", x_init=x0, Q=Q, p=pp, x=xs, u=us, costs=costs)
    # ---------------------------------------------------------------- cartpole iLQR at BASELINE config 2 size
    # B=128, T=25, bounds +-100, decay .5, 2 line-search iterations, eps 1e-2 (examples/Cartpole Control.ipynb
    # cell 1 recipe).  float64 pins the algorithm to 1e-5; float32 is what the notebooks run.  lqr_iter is
    # capped at 20 (f64) / 10 (f32): the comparison is per-iterate, more iterations only amplify fp32 noise.
    if os.environ.get("GOLDEN_FULL", "1") == "1":
        B, T = 128, 25
        for tag, dtype, iters in (("f64", torch.float64, 20), ("f32", torch.float32, 10)):
            x0 = initial_states(B, seed=0).to(dtype)
            Q = torch.diag(q.data).to(dtype).unsqueeze(0).unsqueeze(0).repeat(T, B, 1, 1)
            pp = p.data.to(dtype).unsqueeze(0).repeat(T, B, 1)
            dxr_t = rcart.CartpoleDx(params=torch.tensor((9.8, 1.0, 0.1, 0.5), dtype=dtype))
            with contextlib.redirect_stdout(io.StringIO()):
                xs, us, costs = rmpc.MPC(5, 1, T, u_lower=dxr.lower, u_upper=dxr.upper, lqr_iter=iters, verbose=-1,
                                         exit_unconverged=False, detach_unconverged=False,
                                         linesearch_decay=dxr.linesearch_decay,
                                         max_linesearch_iter=dxr.max_linesearch_iter,
                                         grad_method=rmpc.GradMethods.AUTO_DIFF, eps=1e-2)(x0, rmpc.QuadCost(Q, pp), dxr_t)
            assert xs.dtype == dtype
            npz("cartpole_full_" + tag, x_init=x0, Q=Q[:1, :1], p=pp[:1, :1], x=xs, u=us, costs=costs,
                lqr_iter=np.int64(iters))
    print("all golden fixtures written; oracle == reference on every case")


if __name__ == "__main__":
    main()
