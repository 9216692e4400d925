"""Shared test helpers that need no device: seeded problem generator (SURVEY.md section 8d), fixture loading, and
references and edits that CPU and GPU tests both use."""
import os

import numpy as np
import torch

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def gen_problem(seed, B, T, n, m, dtype, time_varying=False, with_f=True):
    """Well-conditioned LQR instance: C = LL'+I, LTI (or TV) A = 0.9I + 0.1 N/sqrt(n), B = N/sqrt(n)."""
    g = torch.Generator().manual_seed(seed)
    p = n + m
    f64 = torch.float64
    L = torch.randn(T, B, p, p, generator=g, dtype=f64) / p ** 0.5
    C = L @ L.transpose(-1, -2) + torch.eye(p, dtype=f64)
    c = torch.randn(T, B, p, generator=g, dtype=f64)
    if time_varying:
        A = 0.9 * torch.eye(n, dtype=f64) + 0.1 * torch.randn(T - 1, B, n, n, generator=g, dtype=f64) / n ** 0.5
        Bm = torch.randn(T - 1, B, n, m, generator=g, dtype=f64) / n ** 0.5
        F = torch.cat((A, Bm), -1)
    else:
        A = 0.9 * torch.eye(n, dtype=f64) + 0.1 * torch.randn(B, n, n, generator=g, dtype=f64) / n ** 0.5
        Bm = torch.randn(B, n, m, generator=g, dtype=f64) / n ** 0.5
        F = torch.cat((A, Bm), -1).unsqueeze(0).repeat(T - 1, 1, 1, 1)
    f = 0.1 * torch.randn(T - 1, B, n, generator=g, dtype=f64)
    x0 = torch.randn(B, n, generator=g, dtype=f64)
    out = [t.to(dtype).contiguous() for t in (C, c, F, f, x0)]
    if not with_f:
        out[3] = None
    return out


def nominal_controls(seed, B, T, m, dtype, bounds=None):
    """Returns (u, u_lower, u_upper); bounds: None | float | 'tensor'."""
    g = torch.Generator().manual_seed(seed + 7)
    u = (0.1 * torch.randn(T, B, m, generator=g, dtype=torch.float64)).to(dtype)
    if bounds is None:
        return u, None, None
    if bounds == "tensor":
        ul = (-0.5 * torch.rand(T, B, m, generator=g, dtype=torch.float64) - 0.05).to(dtype)
        uu = (0.5 * torch.rand(T, B, m, generator=g, dtype=torch.float64) + 0.05).to(dtype)
        return torch.maximum(torch.minimum(u, uu), ul), ul, uu
    return u.clamp(-float(bounds), float(bounds)), -float(bounds), float(bounds)


def load_golden(name):
    z = np.load(os.path.join(GOLD, name + ".npz"))
    out = {}
    for k in z.files:
        a = z[k]
        out[k] = torch.from_numpy(a) if a.ndim > 0 else a.item()
    return out


def scalar_or_tensor(v):
    return v if not torch.is_tensor(v) else v


def maxdiff(a, b):
    a = torch.as_tensor(a)
    b = torch.as_tensor(b)
    return float((a.detach().cpu().double() - b.detach().cpu().double()).abs().max()) if a.numel() else 0.0


def build_net(g, act):
    """NNDynamics(3, 2) with the weights of a make_golden_nn fixture."""
    from mpc.dynamics import NNDynamics
    nl = int(g["n_layers"])
    hidden = [g[f"W{i}"].shape[0] for i in range(nl - 1)]
    net = NNDynamics(3, 2, hidden_sizes=hidden, activation=act).double()
    with torch.no_grad():
        for i, fc in enumerate(net.fcs):
            fc.weight.copy_(g[f"W{i}"])
            fc.bias.copy_(g[f"b{i}"])
    return net


def condensed_box_lqr_scipy(C, c, F, f, x0, lo, hi):
    """Independent solution of one problem instance with scipy (stands in for cvxpy lqr_cp,
    reference tests/test_mpc.py:35-62): minimise the rolled-out cost over u in the box."""
    import numpy as np
    from scipy.optimize import minimize
    T, p = C.shape[0], C.shape[1]
    n = x0.shape[0]
    m = p - n
    C, c, F, f, x0 = (a.numpy() for a in (C, c, F, f, x0))

    def rollout(uflat):
        u = uflat.reshape(T, m)
        x = np.zeros((T, n))
        x[0] = x0
        for t in range(T - 1):
            x[t + 1] = F[t] @ np.concatenate((x[t], u[t])) + f[t]
        return x, u

    def cost(uflat):
        x, u = rollout(uflat)
        tau = np.concatenate((x, u), 1)
        return float(sum(0.5 * tau[t] @ C[t] @ tau[t] + c[t] @ tau[t] for t in range(T)))

    res = minimize(cost, np.zeros(T * m), method="L-BFGS-B", bounds=[(lo, hi)] * (T * m),
                   options=dict(maxiter=2000, ftol=1e-15, gtol=1e-10))
    x, u = rollout(res.x)
    return torch.from_numpy(x), torch.from_numpy(u)


def _edit_routes():
    """(label, edit(dx, new_values)) for every way a parameter tensor is commonly changed in place or replaced."""
    def opt_step(dx, v):
        opt = torch.optim.SGD([dx.params], lr=1.0)
        opt.zero_grad()
        dx.params.grad = (dx.params.detach() - v).clone()      # one SGD step lands exactly on v
        opt.step()

    def no_grad_copy(dx, v):
        with torch.no_grad():
            dx.params.copy_(v)

    def data_item(dx, v):
        for i in range(len(v)):
            dx.params.data[i] = float(v[i])

    def reassign(dx, v):
        dx.params = v.clone().to(dx.params.device).requires_grad_(dx.params.requires_grad)

    return [("optimizer step", opt_step), ("no_grad copy_", no_grad_copy), (".data[i] =", data_item),
            ("reassign", reassign)]


EDIT_ROUTES = _edit_routes()
