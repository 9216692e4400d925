"""Float64 oracle for receding-horizon episodes on a time-varying problem (receding_horizon(..., time_varying=True)):
every time-indexed input lies on the episode's axis of L = n_steps + T - 1 slices, and control step k solves and
steps on its window.  Both functions are plant_oracle's, run one control step at a time on slices:

  C[k:k+T], c[k:k+T], F[k:k+F_T], f[k:k+f_T] (F_T = T - (L - len(F)), f_T likewise), tensor bounds [k:k+T], and a LinDx
  plant's slice k, ("lin", F_p[k:k+1], f_p[k:k+1]), which plant_oracle steps as its slice 0.

The sweep sums each step's slice gradients into the full-length ones at offset k, in the order k = n_steps-1 .. 0.
With n_steps = 1 the slices are the whole inputs and both functions are plant_oracle's (so lqr_oracle's and
slew_oracle's without a plant) bitwise.  plant_oracle, lqr_oracle and slew_oracle are unchanged.

whole: inputs handed whole to every control step instead of sliced, the forms of an episode whose window record
leaves their bit clear: "F" (a LinDx model's F, f: the solve's own [F_T] and [T-1|T], MPCB200_WIN_DYN clear; the
model steps with F[0], f[0]) and "plant" (a LinDx plant's F_p, f_p, of which slice 0 steps every control step,
MPCB200_WIN_PLANT clear).  Their gradients are then summed over the steps at offset 0, in the inputs' own shapes."""
import torch

from oracle import plant_oracle as porc
from oracle.lqr_oracle import Episode


def _has(t):
    return t is not None and t.nelement() > 0


def _window(T, L, k, t, width=None):
    """Slices k .. k+width-1 of a full-length input (width: T less the slices t lacks on the axis); scalars and None
    as they are."""
    if not isinstance(t, torch.Tensor) or t.nelement() == 0:
        return t
    w = T - (L - t.shape[0]) if width is None else width
    return t[k:k + w]


def _plant_at(plant, k, whole=False):
    """The plant of control step k: a LinDx plant's slice k (whole: the plant as it is); a step plant (or None) as it
    is."""
    if whole or plant is None or plant[0] != "lin":
        return plant
    return ("lin", plant[1][k:k + 1], plant[2][k:k + 1] if _has(plant[2]) else None)


def receding_horizon_tv(n_state, n_ctrl, T, n_steps, x_init, C, c, F, f, plant=None, w=None, u_init=None,
                        u_lower=None, u_upper=None, slew_rate_penalty=None, prev_ctrl=None, whole=(), **kw):
    """The windowed loop on plant_oracle.receding_horizon_lin with one control step per call: solve k on the window of
    C, c, F, f and the bounds from x_k with the shifted warm start (and prev_ctrl = u_{k-1} under a slew-rate
    penalty), then x_{k+1} = plant_k(x_k, u_k) + w[k].  kw: mpc_forward_lin's other options.  Returns an Episode."""
    L = C.shape[0]
    m = n_ctrl
    x, ws, prev = x_init, u_init, prev_ctrl
    xs, us, costs, iters, plan_x, plan_u = [x_init], [], [], [], [], []
    dyn = (lambda k, t: t) if "F" in whole else (lambda k, t: _window(T, L, k, t))  # noqa: E731
    for k in range(n_steps):
        ep = porc.receding_horizon_lin(
            n_state, m, T, 1, x, _window(T, L, k, C), _window(T, L, k, c), dyn(k, F), dyn(k, f),
            plant=_plant_at(plant, k, "plant" in whole), w=w[k:k + 1] if w is not None else None, u_init=ws,
            u_lower=_window(T, L, k, u_lower), u_upper=_window(T, L, k, u_upper),
            slew_rate_penalty=slew_rate_penalty, prev_ctrl=prev, **kw)
        x, ws, prev = ep.x[1], ep.u_next, ep.u[0]
        xs.append(x)
        us.append(ep.u[0])
        costs.append(ep.costs[0])
        iters += ep.iters
        plan_x.append(ep.plan_x[0])
        plan_u.append(ep.plan_u[0])
    return Episode(torch.stack(xs), torch.stack(us), torch.stack(costs), iters, torch.stack(plan_x),
                   torch.stack(plan_u), ws)


def receding_horizon_backward_tv(n_state, n_ctrl, T, C, c, F, f, xs, us, plan_x, plan_u, dl_dxs, dl_dus,
                                 u_lower=None, u_upper=None, step=None, theta=None, full_linearisation=True,
                                 coupled=False, slew_rate_penalty=None, prev_ctrl=None, plant=None, whole=()):
    """The reverse sweep of the windowed loop from GIVEN plans, states and controls: plant_oracle's sweep of one
    control step at a time, k = n_steps-1 .. 0, on step k's window, its plans and (dl_dxs[k], g_{k+1}), with
    prev_ctrl = u_{k-1} (u_{-1} = prev_ctrl).  The full-length dC [L], dc, dF, df and a LinDx plant's dF_p, df_p sum
    each step's slice gradients at offset k; dtheta and dtheta_plant sum over the steps; dw[k] and the carried g =
    dL/dx_k are step k's.  Returns plant_oracle's dict, with full-length gradients."""
    L, n_steps = C.shape[0], us.shape[0]
    lin_p = plant is not None and plant[0] == "lin"
    out = {"dC": torch.zeros_like(C), "dc": torch.zeros_like(c)}
    if step is None:
        out["dF"] = torch.zeros_like(F)
        out["df"] = torch.zeros_like(f) if _has(f) else None
    else:
        out["dtheta"] = torch.zeros_like(theta)
    if lin_p:
        out["dF_p"] = torch.zeros_like(plant[1])
        out["df_p"] = torch.zeros_like(plant[2]) if _has(plant[2]) else None
    elif plant is not None:
        out["dtheta_plant"] = torch.zeros_like(plant[2])
    out["dw"] = torch.zeros(n_steps, *xs.shape[1:], dtype=xs.dtype)
    g = dl_dxs[n_steps]
    dyn = (lambda k, t: t) if "F" in whole else (lambda k, t: _window(T, L, k, t))  # noqa: E731
    for k in range(n_steps - 1, -1, -1):
        prev = us[k - 1] if k > 0 else prev_ctrl
        kd, kp = 0 if "F" in whole else k, 0 if "plant" in whole else k
        r = porc.receding_horizon_backward(
            n_state, n_ctrl, T, _window(T, L, k, C), _window(T, L, k, c), dyn(k, F), dyn(k, f),
            xs[k:k + 2], us[k:k + 1], plan_x[k:k + 1], plan_u[k:k + 1], torch.stack((dl_dxs[k], g)),
            dl_dus[k:k + 1], u_lower=_window(T, L, k, u_lower), u_upper=_window(T, L, k, u_upper), step=step,
            theta=theta, full_linearisation=full_linearisation, coupled=coupled,
            slew_rate_penalty=slew_rate_penalty, prev_ctrl=prev, plant=_plant_at(plant, k, "plant" in whole))
        out["dC"][k:k + T] += r["dC"]
        out["dc"][k:k + T] += r["dc"]
        if step is None:
            out["dF"][kd:kd + r["dF"].shape[0]] += r["dF"]
            if out["df"] is not None:
                out["df"][kd:kd + r["df"].shape[0]] += r["df"]
        else:
            out["dtheta"] += r["dtheta"]
        if lin_p:
            out["dF_p"][kp:kp + r["dF_p"].shape[0]] += r["dF_p"]
            if out["df_p"] is not None:
                out["df_p"][kp:kp + r["df_p"].shape[0]] += r["df_p"]
        elif plant is not None:
            out["dtheta_plant"] += r["dtheta_plant"]
        out["dw"][k] = r["dw"][0]
        g = r["dx_init"]
    out["dx_init"] = g
    return out
