"""Float64 oracle for receding-horizon episodes closed on a plant other than the model the solves plan with, with
additive process disturbances: x_{k+1} = plant(x_k, u_k) + w_k.  The episode (a LinDx model, as lqr_oracle's) and the
reverse sweep from given plans, with or without a slew-rate penalty.  Built on lqr_oracle's LQR step, adjoint and
iLQR loop and on slew_oracle's augmentation, which it leaves unchanged.  With the plant the model and no w, both
functions compute exactly what lqr_oracle's (no penalty) and slew_oracle's (a penalty) do, in the same order.

A plant is None (the model steps), ("lin", F_p, f_p) (F_p[0] [x; u] + f_p[0]; f_p None or empty: none) or
("step", step, theta_p) with step(x, u, theta_p) a CPU torch forward and theta_p [B, NP] its per-problem
parameters."""
import torch

from oracle.lqr_oracle import Episode, _mv, known_linearisation, lindx_step, lqr_step_backward, mpc_forward_lin, \
    shift_warm_start
from oracle.slew_oracle import slew_augment


def _has(t):
    return t is not None and t.nelement() > 0


def plant_step(plant, F, f, x, u):
    """x' of the plant (None: the LinDx model F, f) at (x, u), without w."""
    if plant is None:
        return lindx_step(F, f, x, u)
    if plant[0] == "lin":
        return lindx_step(plant[1], plant[2] if _has(plant[2]) else None, x, u)
    return plant[1](x, u, plant[2])


def receding_horizon_lin(n_state, n_ctrl, T, n_steps, x_init, C, c, F, f, plant=None, w=None, u_init=None,
                         slew_rate_penalty=None, prev_ctrl=None, **kw):
    """The notebooks' loop on mpc_forward_lin with the LinDx model (C, c, F, f): solve from x_k (under a slew-rate
    penalty from [u_{k-1}; x_k] on slew_augment's problem, u_{-1} = prev_ctrl or 0) with u_init = the warm start,
    apply u_k = plan_u[0], x_{k+1} = plant(x_k, u_k) + w[k] (w [n_steps, B, n] or None), shift the warm start.
    kw: mpc_forward_lin's options.  Returns an Episode (plan_x augmented under a penalty)."""
    n, m = n_state, n_ctrl
    B = C.shape[1]
    slew = slew_rate_penalty is not None
    if slew:
        C2, c2, F2, f2 = slew_augment(n, m, slew_rate_penalty, C, c, F, f)
    else:
        C2, c2, F2, f2 = C, c, F, f
    ws = torch.zeros(T, B, m, dtype=C.dtype) if u_init is None else u_init
    prev = torch.zeros(B, m, dtype=C.dtype) if prev_ctrl is None else prev_ctrl.detach()
    x = x_init
    xs, us, costs, iters, plan_x, plan_u = [x_init], [], [], [], [], []
    for k in range(n_steps):
        trace = []
        xk = torch.cat((prev, x), 1) if slew else x
        bx, bu, bc, _ = mpc_forward_lin(n + m if slew else n, m, T, xk, C2, c2, F2, f2, u_init=ws, trace=trace, **kw)
        x = plant_step(plant, F, f, x, bu[0])
        if w is not None:
            x = x + w[k]
        ws = shift_warm_start(bu)
        prev = bu[0]
        xs.append(x)
        us.append(bu[0])
        costs.append(bc)
        iters.append(len(trace))
        plan_x.append(bx)
        plan_u.append(bu)
    return Episode(torch.stack(xs), torch.stack(us), torch.stack(costs), iters, torch.stack(plan_x),
                   torch.stack(plan_u), ws)


def receding_horizon_backward(n_state, n_ctrl, T, C, c, F, f, xs, us, plan_x, plan_u, dl_dxs, dl_dus,
                              u_lower=None, u_upper=None, step=None, theta=None, full_linearisation=True,
                              coupled=False, slew_rate_penalty=None, prev_ctrl=None, plant=None):
    """The reverse sweep of an episode closed on `plant`, from GIVEN plans, states and controls: autograd's gradient
    of sum(dl_dxs * xs) + sum(dl_dus * us) for `for k: plan = ctrl'(x_k); x_{k+1} = plant(x_k, plan_u[k][0]) + w_k`.

    The model (LinDx F, f; or a known system: step(x, u, theta), theta [B, NP], F = f = None) gets only the solves'
    part: each adjoint (lqr_step_backward at its plan) and, for a known system, its linearisation's derivative
    (known_linearisation, `full_linearisation` as `full` there).  The plant gets the plant steps' direct part: a LinDx
    plant dF_p[0] += g z^T, df_p[0] += g; a step plant dtheta_plant += autograd of step(x_k, u_k, theta_p) in theta_p.
    dw[k] = g = dL/dx_{k+1}.  Under a slew-rate penalty each solve ran on slew_augment's problem over [u_{k-1}; x_k]
    with u_{k-1} held constant, as slew_oracle's sweep (plan_x augmented [n_steps, T, B, n+m] or the system's).
    plant None: the model steps, and its own step's part goes to the model, as lqr_oracle / slew_oracle give it.
    Returns a dict of dx_init, dC, dc, dF, df (LinDx model) or dtheta, dw [n_steps, B, n], and dF_p, df_p or
    dtheta_plant for a plant."""
    n, m = n_state, n_ctrl
    n_steps = us.shape[0]
    known = step is not None
    slew = slew_rate_penalty is not None
    mm = m if slew else 0
    dt = C.dtype
    has_f = _has(f)
    if known:
        theta = theta.detach().clone().requires_grad_(True)
    if slew:
        C2, c2, F2, f2 = slew_augment(n, m, slew_rate_penalty, C, c, F, f if has_f else None)
    dC, dc = torch.zeros_like(C), torch.zeros_like(c)
    dF = None if known else torch.zeros_like(F)
    df = torch.zeros_like(f) if has_f and not known else None
    dtheta = torch.zeros_like(theta) if known else None
    out = {}
    lin_p = plant is not None and plant[0] == "lin"
    if lin_p:
        Fp, fp = plant[1], plant[2] if _has(plant[2]) else None
        dF_p = out["dF_p"] = torch.zeros_like(Fp)
        df_p = out["df_p"] = torch.zeros_like(fp) if fp is not None else None
    elif plant is not None:
        pstep, ptheta = plant[1], plant[2].detach().clone().requires_grad_(True)
        dth_p = out["dtheta_plant"] = torch.zeros_like(ptheta)
    g = dl_dxs[n_steps].clone()
    B = g.shape[0]
    dw = out["dw"] = torch.zeros(n_steps, B, n, dtype=dt)
    prev = torch.zeros(B, m, dtype=dt) if prev_ctrl is None else prev_ctrl.detach()
    if slew and plan_x.shape[-1] == n:
        prevs = torch.cat((prev.unsqueeze(0), us[:-1]), 0)
        plan_x = torch.cat((torch.cat((prevs.unsqueeze(1), plan_u[:, :-1]), 1), plan_x), 3)
    for k in range(n_steps - 1, -1, -1):
        dw[k] = g
        xk, uk = xs[k], us[k]
        # the plant step's VJP (the model's own when plant is None)
        if plant is None and known:
            xl, ul = xk.detach().requires_grad_(True), uk.detach().requires_grad_(True)
            gx, gu, gth = torch.autograd.grad((step(xl, ul, theta) * g).sum(), (xl, ul, theta))
            dtheta += gth
        elif plant is None or lin_p:
            PF, Pf, PdF, Pdf = (F, f if has_f else None, dF, df) if plant is None else (Fp, fp, dF_p, df_p)
            z = torch.cat((xk, uk), 1)
            gz = _mv(PF[0].transpose(1, 2), g)
            gx, gu = gz[:, :n], gz[:, n:]
            PdF[0] += g.unsqueeze(2) * z.unsqueeze(1)
            if Pf is not None:
                Pdf[0] += g
        else:
            xl, ul = xk.detach().requires_grad_(True), uk.detach().requires_grad_(True)
            gx, gu, gth = torch.autograd.grad((pstep(xl, ul, ptheta) * g).sum(), (xl, ul, ptheta))
            dth_p += gth
        # the solve's adjoint at its plan
        if known:
            Fk, fk = known_linearisation(step, theta, plan_x[k][..., mm:], plan_u[k], full_linearisation)
            if slew:
                _, _, Fak, fak = slew_augment(n, m, slew_rate_penalty, C, c, Fk.detach(), fk.detach())
            else:
                Fak, fak = Fk, fk
        else:
            Fak, fak = (F2, f2) if slew else (F, f)
        dl_dx = torch.zeros(T, B, n + mm, dtype=dt)
        dl_du = torch.zeros(T, B, m, dtype=dt)
        dl_du[0] = dl_dus[k] + gu
        if slew:
            x0k = torch.cat((us[k - 1] if k > 0 else prev, xk), 1)
            Cs, cs = C2, c2
        else:
            x0k, Cs, cs = plan_x[k][0], C, c
        dxk, dCk, dck, dFk, dfk, _, _ = lqr_step_backward(
            n + mm, m, T, x0k, Cs, cs, Fak.detach(), fak.detach() if fak is not None else None, plan_x[k],
            plan_u[k], dl_dx, dl_du, u_lower=u_lower, u_upper=u_upper, coupled=coupled)
        if slew:
            dC += dCk[..., m:, m:]
            dc += dck[..., m:]
        else:
            dC += dCk
            dc += dck
        if known:
            if slew:
                dtheta += torch.autograd.grad((Fk * dFk[..., m:, m:]).sum() + (fk * dfk[..., m:]).sum(), theta)[0]
            else:
                dtheta += torch.autograd.grad((Fk * dFk).sum() + (fk * dfk).sum(), theta)[0]
        else:
            dF += dFk[..., m:, m:] if slew else dFk
            if has_f:
                df[:T - 1] += dfk[..., m:] if slew else dfk
        g = dl_dxs[k] + gx + (dxk[:, m:] if slew else dxk)     # under a penalty the previous control's part is dropped
    out.update(dx_init=g, dC=dC, dc=dc)
    if known:
        out["dtheta"] = dtheta
    else:
        out.update(dF=dF, df=df)
    return out
