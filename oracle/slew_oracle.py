"""Float64 oracle for receding-horizon episodes under a slew-rate penalty (mpc/mpc.py:362-445): the notebooks' closed
loop on the augmented problem over [u_{t-1}; x] and its reverse sweep, with the previous control held constant as the
reference holds prev_ctrl (:399-408).  Built on lqr_oracle's LQR step, adjoint and iLQR loop; its own augmentation
(slew_augment), so that it shares no code with the library's MPC._slew_augment.  Without a penalty both functions are
lqr_oracle's own."""
import torch

from oracle.lqr_oracle import (Episode, _mv, known_linearisation, lindx_step, lqr_step_backward, mpc_forward_lin,
                               receding_horizon_backward as _backward_plain, receding_horizon_lin as _episode_plain,
                               shift_warm_start)


def slew_augment(n_state, n_ctrl, slew_rate_penalty, C, c, F=None, f=None):
    """The slew-rate problem over the augmented state [u_{t-1}; x]: C~ = slew_C + C embedded at [m:, m:] with
    slew_C = penalty * [[I, 0, -I], [0, 0, 0], [-I, 0, I]], c~ = [0; c], F~ = [[0, 0, I], [0, F]] and f~ = [0; f]
    (None without f).  Differentiable in C, c, F, f; F None: (C~, c~, None, None)."""
    n, m = n_state, n_ctrl
    lead = C.shape[:-2]
    p2 = n + 2 * m
    gI = slew_rate_penalty * torch.eye(m, dtype=C.dtype)
    S = torch.zeros(*lead, p2, p2, dtype=C.dtype)
    S[..., :m, :m] = gI
    S[..., -m:, :m] = -gI
    S[..., :m, -m:] = -gI
    S[..., -m:, -m:] = gI
    C2 = S + torch.nn.functional.pad(C, (m, 0, m, 0))
    c2 = torch.cat((c.new_zeros(*c.shape[:-1], m), c), -1)
    if F is None:
        return C2, c2, None, None
    Fu = F.new_zeros(*F.shape[:-2], m, p2)
    Fu[..., n + m:] = torch.eye(m, dtype=F.dtype)
    F2 = torch.cat((Fu, torch.cat((F.new_zeros(*F.shape[:-1], m), F), -1)), -2)
    f2 = torch.cat((f.new_zeros(*f.shape[:-1], m), f), -1) if f is not None and f.nelement() > 0 else None
    return C2, c2, F2, f2


def receding_horizon_lin(n_state, n_ctrl, T, n_steps, x_init, C, c, F, f, u_init=None, slew_rate_penalty=None,
                         prev_ctrl=None, **kw):
    """lqr_oracle.receding_horizon_lin under a slew-rate penalty: each solve runs on the augmented problem
    (slew_augment) from [u_{k-1}; x_k], u_{-1} = prev_ctrl [B, m] or zeros; the plant is the system's own F[0] [x; u]
    + f[0].  Returns an Episode whose plan_x holds the augmented plans [n_steps, T, B, n+m]; x stays the system's
    state.  slew_rate_penalty None: lqr_oracle.receding_horizon_lin itself (prev_ctrl unused)."""
    if slew_rate_penalty is None:
        return _episode_plain(n_state, n_ctrl, T, n_steps, x_init, C, c, F, f, u_init=u_init, **kw)
    n, m = n_state, n_ctrl
    B = C.shape[1]
    C2, c2, F2, f2 = slew_augment(n, m, slew_rate_penalty, C, c, F, f)
    w = torch.zeros(T, B, m, dtype=C.dtype) if u_init is None else u_init
    prev = torch.zeros(B, m, dtype=C.dtype) if prev_ctrl is None else prev_ctrl.detach()
    x = x_init
    xs, us, costs, iters, plan_x, plan_u = [x_init], [], [], [], [], []
    for _ in range(n_steps):
        trace = []
        bx, bu, bc, _ = mpc_forward_lin(n + m, m, T, torch.cat((prev, x), 1), C2, c2, F2, f2, u_init=w, trace=trace,
                                        **kw)
        x = lindx_step(F, f, x, bu[0])
        w = shift_warm_start(bu)
        prev = bu[0]
        xs.append(x)
        us.append(bu[0])
        costs.append(bc)
        iters.append(len(trace))
        plan_x.append(bx)
        plan_u.append(bu)
    return Episode(torch.stack(xs), torch.stack(us), torch.stack(costs), iters, torch.stack(plan_x),
                   torch.stack(plan_u), w)


def receding_horizon_backward(n_state, n_ctrl, T, C, c, F, f, xs, us, plan_x, plan_u, dl_dxs, dl_dus,
                              u_lower=None, u_upper=None, step=None, theta=None, full_linearisation=True,
                              coupled=False, slew_rate_penalty=None, prev_ctrl=None):
    """lqr_oracle.receding_horizon_backward for an episode under a slew-rate penalty.  Each solve ran on the augmented
    problem over [u_{k-1}; x_k] (slew_augment; u_{-1} = prev_ctrl or 0).  plan_x holds its augmented plans
    [n_steps, T, B, n+m], or the system's [n_steps, T, B, n] (the reference's, augmented here with u_{k-1} and
    plan_u[k][:-1], which the passthrough copies); xs, us, dl_dxs, dl_dus and the returned gradients are the system's.

    The previous control is a constant (the reference detaches prev_ctrl, mpc/mpc.py:399-408): the part of each
    adjoint's dx_init for it is dropped.  The model step's VJP is the system's own (LinDx: F[0]^T g, dF[0] += g z^T,
    df[0] += g; a known system: autograd of step(x_k, u_k, theta)).  Each adjoint's dC~, dc~, dF~, df~ enter through
    their [m:, m:] / [m:] blocks; a known system's linearisation is the system's own along plan_x[..., m:]
    (known_linearisation, `full_linearisation` as `full` there), embedded as F~.  Returns a dict of dx_init, dC, dc,
    and dF, df (LinDx; df None without f) or dtheta [B, NP].  slew_rate_penalty None:
    lqr_oracle.receding_horizon_backward itself (prev_ctrl unused)."""
    if slew_rate_penalty is None:
        return _backward_plain(n_state, n_ctrl, T, C, c, F, f, xs, us, plan_x, plan_u, dl_dxs, dl_dus,
                               u_lower=u_lower, u_upper=u_upper, step=step, theta=theta,
                               full_linearisation=full_linearisation, coupled=coupled)
    n, m = n_state, n_ctrl
    n_steps = us.shape[0]
    known = step is not None
    dt = C.dtype
    has_f = f is not None and f.nelement() > 0
    if known:
        theta = theta.detach().clone().requires_grad_(True)
    C2, c2, F2, f2 = slew_augment(n, m, slew_rate_penalty, C, c, F, f if has_f else None)
    dC, dc = torch.zeros_like(C), torch.zeros_like(c)
    dF = None if known else torch.zeros_like(F)
    df = torch.zeros_like(f) if has_f and not known else None
    dtheta = torch.zeros_like(theta) if known else None
    g = dl_dxs[n_steps].clone()
    B = g.shape[0]
    prev = torch.zeros(B, m, dtype=dt) if prev_ctrl is None else prev_ctrl.detach()
    if plan_x.shape[-1] == n:
        prevs = torch.cat((prev.unsqueeze(0), us[:-1]), 0)
        plan_x = torch.cat((torch.cat((prevs.unsqueeze(1), plan_u[:, :-1]), 1), plan_x), 3)
    for k in range(n_steps - 1, -1, -1):
        xk, uk = xs[k], us[k]
        if known:
            xl, ul = xk.detach().requires_grad_(True), uk.detach().requires_grad_(True)
            gx, gu, gth = torch.autograd.grad((step(xl, ul, theta) * g).sum(), (xl, ul, theta))
            dtheta += gth
            Fk, fk = known_linearisation(step, theta, plan_x[k][..., m:], plan_u[k], full_linearisation)
            _, _, F2k, f2k = slew_augment(n, m, slew_rate_penalty, C, c, Fk.detach(), fk.detach())
        else:
            z = torch.cat((xk, uk), 1)
            gz = _mv(F[0].transpose(1, 2), g)
            gx, gu = gz[:, :n], gz[:, n:]
            dF[0] += g.unsqueeze(2) * z.unsqueeze(1)
            if has_f:
                df[0] += g
            F2k, f2k = F2, f2
        dl_dx = torch.zeros(T, B, n + m, dtype=dt)
        dl_du = torch.zeros(T, B, m, dtype=dt)
        dl_du[0] = dl_dus[k] + gu
        x2k = torch.cat((us[k - 1] if k > 0 else prev, xk), 1)
        dxk, dCk, dck, dFk, dfk, _, _ = lqr_step_backward(
            n + m, m, T, x2k, C2, c2, F2k.detach(), f2k.detach() if f2k is not None else None, plan_x[k], plan_u[k],
            dl_dx, dl_du, u_lower=u_lower, u_upper=u_upper, coupled=coupled)
        dC += dCk[..., m:, m:]
        dc += dck[..., m:]
        if known:
            dtheta += torch.autograd.grad((Fk * dFk[..., m:, m:]).sum() + (fk * dfk[..., m:]).sum(), theta)[0]
        else:
            dF += dFk[..., m:, m:]
            if has_f:
                df[:T - 1] += dfk[..., m:]
        g = dl_dxs[k] + gx + dxk[:, m:]        # dxk[:, :m], the previous control's part, is dropped
    out = dict(dx_init=g, dC=dC, dc=dc)
    if known:
        out["dtheta"] = dtheta
    else:
        out.update(dF=dF, df=df)
    return out
