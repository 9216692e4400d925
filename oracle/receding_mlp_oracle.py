"""Float64 oracle of a receding-horizon episode planned with a learned model (NNDynamics), composed of mlp_oracle's
iLQR loop and network step, lqr_oracle's KKT adjoint and mlp_grad_oracle's linearisation VJP.  Pure CPU torch.

episode(): for k: plan = mlp_oracle.ilqr(x_k, u_init = w_k); x_{k+1} = step(x_k, plan_u[0]) + w_k, with step the
network (plant None) or a plant(x, u); w_{k+1} = lqr_oracle.shift_warm_start(plan_u).
backward(): autograd's gradient of sum(dl_dxs * xs) + sum(dl_dus * us) for that loop, each solve contributing
MPC.forward's differentiable tail at its plan (the adjoint on the network's linearisation, differentiated in the
weights), the warm starts held constant: lqr_oracle.receding_horizon_backward's sweep with the network's parts.
backward() runs in the dtype of its inputs: float64 for the oracle, float32 for the yardstick of float32 kernels."""
import torch

from . import lqr_oracle as lo
from . import mlp_grad_oracle as mgo
from . import mlp_oracle as mo


def episode(n, m, T, n_steps, x_init, C, c, layers, act, passthrough, plant=None, w=None, u_init=None, **ilqr_kw):
    """(xs [n_steps+1, B, n], us [n_steps, B, m], plan_x [n_steps, T, B, n], plan_u [n_steps, T, B, m], iterations
    per solve)."""
    B = x_init.shape[0]
    wk = torch.zeros(T, B, m, dtype=torch.float64) if u_init is None else u_init
    x, xs, us, px, pu, its = x_init, [x_init], [], [], [], []
    for k in range(n_steps):
        plan_x, plan_u, _, it = mo.ilqr(n, m, T, x, C, c, layers, act, passthrough, u_init=wk, **ilqr_kw)
        u = plan_u[0]
        x = mo.step(layers, act, passthrough, x, u) if plant is None else plant(x, u)
        if w is not None:
            x = x + w[k]
        wk = lo.shift_warm_start(plan_u)
        xs.append(x)
        us.append(u)
        px.append(plan_x)
        pu.append(plan_u)
        its.append(it)
    return torch.stack(xs), torch.stack(us), torch.stack(px), torch.stack(pu), its


def backward(n, m, T, C, c, layers, act, passthrough, xs, us, plan_x, plan_u, dl_dxs, dl_dus, u_lower=None,
             u_upper=None, plant=None, theta=None):
    """From GIVEN plans, states and controls.  plant None: the network steps, and its step's d<g, x'>/dtheta joins the
    weights' gradient; else plant(x, u, theta) with theta [B, NP] (or None) its parameters.  Returns a dict of
    dx_init, dC, dc, dlayers [(dW_i, db_i)], dw [n_steps, B, n] and, with theta, dtheta_plant."""
    n_steps, B = us.shape[0], us.shape[1]
    lay = [(W.detach().clone().requires_grad_(True), b.detach().clone().requires_grad_(True)) for W, b in layers]
    flat = [t for wb in lay for t in wb]
    dlay = [torch.zeros_like(t) for t in flat]
    th = theta.detach().clone().requires_grad_(True) if theta is not None else None
    dth = torch.zeros_like(th) if th is not None else None
    dC, dc = torch.zeros_like(C), torch.zeros_like(c)
    dw = torch.zeros(n_steps, B, n, dtype=C.dtype)
    g = dl_dxs[n_steps].clone()
    for k in range(n_steps - 1, -1, -1):
        dw[k] = g
        xl, ul = xs[k].detach().requires_grad_(True), us[k].detach().requires_grad_(True)
        if plant is None:
            gs = torch.autograd.grad((mo.step(lay, act, passthrough, xl, ul) * g).sum(), [xl, ul] + flat)
            gx, gu = gs[0], gs[1]
            dlay = [a + b for a, b in zip(dlay, gs[2:])]
        else:
            ins = [xl, ul] + ([th] if th is not None else [])
            gs = torch.autograd.grad((plant(xl, ul, th) * g).sum(), ins, allow_unused=True)
            gx, gu = gs[0], gs[1]
            if th is not None:
                dth += gs[2]
        Fk, fk = mo.linearize(layers, act, passthrough, plan_x[k], plan_u[k])
        dl_dx = torch.zeros(T, B, n, dtype=C.dtype)
        dl_du = torch.zeros(T, B, m, dtype=C.dtype)
        dl_du[0] = dl_dus[k] + gu
        dxk, dCk, dck, dFk, dfk, _, _ = lo.lqr_step_backward(n, m, T, plan_x[k][0], C, c, Fk, fk, plan_x[k],
                                                             plan_u[k], dl_dx, dl_du, u_lower=u_lower,
                                                             u_upper=u_upper, coupled=False)
        dC += dCk
        dc += dck
        gl = mgo.linearize_vjp(layers, act, passthrough, plan_x[k], plan_u[k], dFk, dfk)
        dlay = [a + b for a, b in zip(dlay, [t for wb in gl for t in wb])]
        g = dl_dxs[k] + gx + dxk
    out = dict(dx_init=g, dC=dC, dc=dc, dlayers=[(dlay[2 * i], dlay[2 * i + 1]) for i in range(len(layers))], dw=dw)
    if th is not None:
        out["dtheta_plant"] = dth
    return out
