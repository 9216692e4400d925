"""Float64 oracle of a learned model, the reference's NNDynamics (mpc/dynamics.py:15-131): x' = [x +] MLP([x; u]) with
Linear layers, an activation after every layer but the last, and the exact input Jacobian by the chain rule, each
activation's slope taken from its output (sigmoid a(1-a), relu 1 where a > 0, elu 1 where a > 0 else a + 1).  Also the
iLQR loop of MPC.forward (mpc/mpc.py:244-301) with the network as the line search's true dynamics, built on
lqr_oracle.lqr_step_forward(..., dynamics=...).

A network is a list of (W [out, in], b [out]) float64 CPU tensors, an activation name and the passthrough flag.
n_prev = m: the slew-rate augmented state [u_{t-1}; x] of CtrlPassthroughDynamics, stepped as [u; step(x, u)].
"""
import torch

from . import lqr_oracle as lo

_ACT = {"sigmoid": torch.sigmoid, "relu": torch.relu, "elu": torch.nn.functional.elu}


def layers_of(net):
    """The (W, b) list of an nn.Module with `fcs` (NNDynamics), in float64 on the CPU."""
    return [(fc.weight.detach().double().cpu(), fc.bias.detach().double().cpu()) for fc in net.fcs]


def _slope(act, a):
    if act == "sigmoid":
        return a * (1.0 - a)
    if act == "relu":
        return (a > 0).to(a.dtype)
    return torch.where(a > 0, torch.ones_like(a), a + 1.0)


def _hidden(layers, act, z):
    hs = []
    for W, b in layers[:-1]:
        z = _ACT[act](z @ W.t() + b)
        hs.append(z)
    W, b = layers[-1]
    return hs, z @ W.t() + b


def step(layers, act, passthrough, x, u, n_prev=0):
    """x' of [B, n_prev + n] states and [B, m] controls."""
    xs = x[:, n_prev:]
    _, out = _hidden(layers, act, torch.cat((xs, u), 1))
    nxt = xs + out if passthrough else out
    return torch.cat((u[:, :n_prev], nxt), 1) if n_prev else nxt


def jacobian(layers, act, passthrough, x, u):
    """(R [B, n, n], S [B, n, m]) of the network's own state x [B, n] and control u [B, m]."""
    n = x.shape[1]
    hs, _ = _hidden(layers, act, torch.cat((x, u), 1))
    J = layers[-1][0].unsqueeze(0).expand(x.shape[0], -1, -1)
    for h, (W, _) in zip(reversed(hs), reversed(layers[:-1])):
        J = (J * _slope(act, h).unsqueeze(1)) @ W
    R, S = J[:, :, :n], J[:, :, n:]
    if passthrough:
        R = R + torch.eye(n, dtype=R.dtype)
    return R, S


def linearize(layers, act, passthrough, x, u, n_prev=0):
    """F [T-1, B, N, N+m] and f [T-1, B, N] of x [T, B, N] (N = n_prev + n), u [T, B, m]: [R S] and x' - R x - S u, and
    under n_prev the rows [0 0 I] (f 0) of the previous control."""
    T, B, N = x.shape
    m = u.shape[2]
    n = N - n_prev
    xs, us = x[:-1].reshape(-1, N), u[:-1].reshape(-1, m)
    R, S = jacobian(layers, act, passthrough, xs[:, n_prev:], us)
    nxt = step(layers, act, passthrough, xs, us, n_prev)[:, n_prev:]
    fs = nxt - lo._mv(R, xs[:, n_prev:]) - lo._mv(S, us)
    F = torch.zeros(xs.shape[0], N, N + m, dtype=x.dtype)
    f = torch.zeros(xs.shape[0], N, dtype=x.dtype)
    F[:, :n_prev, N:N + n_prev] = torch.eye(n_prev, dtype=x.dtype)
    F[:, n_prev:, n_prev:N] = R
    F[:, n_prev:, N:] = S
    f[:, n_prev:] = fs
    return F.view(T - 1, B, N, N + m), f.view(T - 1, B, N)


def rollout(layers, act, passthrough, x_init, u, n_prev=0):
    """get_traj (mpc/util.py:102-126): x [T, B, N]."""
    xs = [x_init]
    for t in range(u.shape[0] - 1):
        xs.append(step(layers, act, passthrough, xs[t], u[t], n_prev))
    return torch.stack(xs)


def ilqr(n, m, T, x_init, C, c, layers, act, passthrough, u_init=None, u_lower=None, u_upper=None, lqr_iter=10,
         eps=1e-7, not_improved_lim=5, best_cost_eps=1e-4, n_prev=0, **step_kw):
    """MPC.forward's iterations (mpc/mpc.py:244-301) with QuadCost(C, c) and the network: rollout, linearisation,
    lqr_step_forward with the network as the line search's dynamics, best-iterate tracking and the stop test.  n is
    the (augmented) state count.  The loop is lqr_oracle.ilqr_loop.  Returns (x, u, costs, iterations)."""
    return lo.ilqr_loop(n, m, T, x_init, C, c, lambda uu: rollout(layers, act, passthrough, x_init, uu, n_prev),
                        lambda x, uu: linearize(layers, act, passthrough, x, uu, n_prev),
                        lambda x, uu: step(layers, act, passthrough, x, uu, n_prev), u_init=u_init, lqr_iter=lqr_iter,
                        eps=eps, not_improved_lim=not_improved_lim, best_cost_eps=best_cost_eps, u_lower=u_lower,
                        u_upper=u_upper, **step_kw)
