"""GPU: gradients of a known system's parameters (CartpoleDx / PendulumDx `params`) through the VJP kernel of the
in-kernel linearisation (mpcb200_dyn_linearize_vjp_*, dynamics.DynLinearize).

With z = [x; u], J = dx'/dz and f = x' - J z, the kernel writes per (t, b)
  first  = sum_r df_r dx'_r/dtheta                  (J held constant: the reference's whole gradient)
  second = sum_rj (dF_rj - df_r z_j) dJ_rj/dtheta   (what J's own dependence on theta adds)
and MPC's differentiable tail returns their sum over (t, b), the full derivative that torch autograd with
create_graph=True gives (INTEGRATION.md section 2).

Checked against float64 autograd of the module per (t, b), against central differences of the f64 linearisation
kernel, against the reference's params.grad (oracle/make_golden_paramgrad.py), end to end against the same physics
run as an opaque Module, and by learning the parameters back from perturbed values.  Tolerances: float64 1e-10
relative; float32 by the K32 rule of tests/gpu_harness.within."""
import pytest
import torch

from tests.gpu_harness import DEV, DT, F32, F64, PHYS, SYSTEMS, known_controls, known_module, known_states, within
from tests.helpers import load_golden, maxdiff

pytestmark = pytest.mark.gpu

NP = {"cartpole": 4, "pendulum": 3}


def _opaque(dx):
    class Opaque(torch.nn.Module):                      # hides mpcb200_kind: the torch AUTO_DIFF route
        def forward(self, x, u):
            return dx(x, u)
    return Opaque()


def _case(name, B, T, dtype, seed):
    """x [T,B,n] (angles across the atan2 cut, off the unit circle), u [T,B,1] (inside, at and one ulp either side of
    the clamp), random dF, df; float64 values rounded through dtype."""
    n = PHYS[name]["n"]
    g = torch.Generator().manual_seed(seed)
    x = torch.stack([known_states(name, B, seed + t) for t in range(T)]).to(dtype).double()
    u = known_controls(name, T, B, dtype, seed + 100).to(dtype).double()
    dF = torch.randn(T - 1, B, n, n + 1, generator=g, dtype=F64).to(dtype).double()
    df = torch.randn(T - 1, B, n, generator=g, dtype=F64).to(dtype).double()
    return x, u, dF, df


def autograd_vjp(name, x, u, dF, df, dtype):
    """(first, second) [T-1,B,NP] by torch autograd of the module in `dtype` on the CPU, one parameter column per
    (t, b) so that each item's gradient stays separate: the create_graph Jacobians contracted with dF, df."""
    T, B, n = x.shape
    N = (T - 1) * B
    base = torch.tensor(PHYS[name]["params"], dtype=dtype)
    P = base.view(-1, 1).expand(-1, N).clone().requires_grad_(True)    # unbind() gives one value per item
    dx = known_module(name, params=P)
    xs = x[:-1].reshape(N, n).to(dtype).requires_grad_(True)
    us = u[:-1].reshape(N, 1).to(dtype).requires_grad_(True)
    nx = dx(xs, us)
    rows = [torch.autograd.grad(nx[:, r].sum(), [xs, us], create_graph=True) for r in range(n)]
    J = torch.cat((torch.stack([a for a, _ in rows], 1), torch.stack([b for _, b in rows], 1)), 2)   # [N, n, n+1]
    z = torch.cat((xs, us), 1).detach()
    dF_, df_ = dF.reshape(N, n, n + 1).to(dtype), df.reshape(N, n).to(dtype)
    first, = torch.autograd.grad((df_ * nx).sum(), P, retain_graph=True)
    w = dF_ - df_.unsqueeze(2) * z.unsqueeze(1)
    second, = torch.autograd.grad((w * J).sum(), P)
    return first.t().reshape(T - 1, B, -1).double(), second.t().reshape(T - 1, B, -1).double()


def kernel_vjp(name, x, u, dF, df, dtype, dx=None):
    from mpc.pytorch_b200.dynamics import dyn_linearize_vjp_raw
    dx = known_module(name) if dx is None else dx
    T = x.shape[0]
    first, second = dyn_linearize_vjp_raw(dx.mpcb200_kind, dx.mpcb200_params(), T, *(t.to(dtype).to(DEV)
                                                                                      for t in (x, u, dF, df)))
    assert first.dtype == dtype and first.shape == (T - 1, x.shape[1], NP[name])
    return first.cpu(), second.cpu()


# ------------------------------------------------------------------------------------------------------------------
# the kernel per (t, b)
# ------------------------------------------------------------------------------------------------------------------
BT = [(1, 2), (7, 2), (300, 2), (1, 25), (7, 25), (300, 25)]


@pytest.mark.parametrize("B,T", BT, ids=[f"B{b}_T{t}" for b, t in BT])
@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("name", SYSTEMS)
def test_vjp_matches_autograd(name, dtype, B, T):
    x, u, dF, df = _case(name, B, T, dtype, 11 * B + T)
    first, second = kernel_vjp(name, x, u, dF, df, dtype)
    w64 = autograd_vjp(name, x, u, dF, df, F64)
    w32 = autograd_vjp(name, x, u, dF, df, F32) if dtype == F32 else (None, None)
    tag = f"{name} {DT[dtype]} B={B} T={T}"
    within(tag, "first", first, w64[0], w32[0], dtype, 1e-10)
    within(tag, "second", second, w64[1], w32[1], dtype, 1e-10)
    if B >= 7:   # the cases reach beyond the clamp, where a saturated control has no u column
        assert bool((u[:-1].abs() > PHYS[name]["clamp"]).any()), tag


@pytest.mark.parametrize("name", SYSTEMS)
def test_vjp_matches_finite_differences(name):
    """sum (first + second) against central differences in theta of <dF, F(theta)> + <df, f(theta)>, both from the
    float64 linearisation kernel: a check that does not go through autograd."""
    from mpc.pytorch_b200.dynamics import dyn_linearize_raw
    B, T = 7, 25
    x, u, dF, df = (t.to(DEV) for t in _case(name, B, T, F64, 5))
    dx = known_module(name)
    first, second = kernel_vjp(name, x, u, dF, df, F64, dx)
    got = (first + second).sum((0, 1))
    prm = list(dx.mpcb200_params())

    def objective(p):
        F, f = dyn_linearize_raw(dx.mpcb200_kind, p, T, x, u)
        return float((dF * F).sum() + (df * f).sum())
    fd = []
    for k in range(NP[name]):
        h = 1e-5 * abs(prm[k])
        hi, lo = list(prm), list(prm)
        hi[k] += h
        lo[k] -= h
        fd.append((objective(hi) - objective(lo)) / (2 * h))
    fd = torch.tensor(fd, dtype=F64)
    assert maxdiff(got, fd) <= 1e-6 * max(1.0, float(fd.abs().max())), f"{name}: {got.tolist()} vs {fd.tolist()}"
    assert float(second.sum((0, 1)).abs().max()) > 1e-3 * float(fd.abs().max()), "second must not be negligible"


@pytest.mark.parametrize("name", SYSTEMS)
def test_batch_independence(name):
    """Per-(t, b) outputs are bitwise the same whatever the problem's position in the batch and the batch size."""
    B, T = 300, 9
    x, u, dF, df = _case(name, B, T, F64, 3)
    for dtype in (F64, F32):
        big = kernel_vjp(name, x, u, dF, df, dtype)
        idx = torch.tensor([299, 0, 131, 7, 128, 64, 5])
        small = kernel_vjp(name, x[:, idx], u[:, idx], dF[:, idx], df[:, idx], dtype)
        for a, b in zip(big, small):
            assert torch.equal(a[:, idx], b), f"{name} {DT[dtype]}"


# ------------------------------------------------------------------------------------------------------------------
# the reference's gradient: `first` alone
# ------------------------------------------------------------------------------------------------------------------
def _fixture_module(name, g, params=None):
    from mpc.pytorch_b200.dynamics import CartpoleDx, PendulumDx
    dx = (CartpoleDx if name == "cartpole" else PendulumDx)(params=g["params"].clone() if params is None else params)
    dx.dt = g["dt"]
    setattr(dx, PHYS[name]["clamp_attr"], g["clamp"])
    return dx


@pytest.mark.parametrize("regime", ["unb", "box"])
@pytest.mark.parametrize("name", SYSTEMS)
def test_first_is_the_reference_gradient(name, regime):
    """At the reference's linearisation point and the df that reached its f, sum first equals the reference's
    params.grad; the repo's gradient is first + second (the documented convention difference)."""
    g = load_golden(f"paramgrad_{name}_f64")
    dx = _fixture_module(name, g)
    x, u, df = g[f"x_lin_{regime}"], g[f"u_{regime}"], g[f"df_{regime}"]
    dF = torch.zeros(*df.shape, df.shape[-1] + 1, dtype=F64)
    first, second = kernel_vjp(name, x, u, dF, df, F64, dx)
    want = g[f"grad_{regime}"]
    got = first.sum((0, 1))
    assert maxdiff(got, want) <= 1e-10 * max(1.0, float(want.abs().max())), f"{got.tolist()} vs {want.tolist()}"
    assert float(second.sum((0, 1)).abs().max()) > 1e-3 * float(want.abs().max())


# ------------------------------------------------------------------------------------------------------------------
# end to end: MPC.forward + backward
# ------------------------------------------------------------------------------------------------------------------
def _solve(name, dx, B, T, bounds, grad_method=None, slew=False, lqr_iter=20):
    from mpc.pytorch_b200 import MPC, QuadCost, GradMethods
    n = PHYS[name]["n"]
    q, p = known_module(name).get_true_obj()
    Q = torch.diag(q).double().expand(T, B, n + 1, n + 1).contiguous().to(DEV)
    pp = p.double().expand(T, B, n + 1).contiguous().to(DEV)
    kw = dict(u_lower=-bounds, u_upper=bounds, lqr_iter=lqr_iter, verbose=-1, exit_unconverged=False,
              detach_unconverged=False, linesearch_decay=0.3, max_linesearch_iter=4,
              grad_method=grad_method or GradMethods.AUTO_DIFF, eps=1e-9)
    if slew:
        kw.update(slew_rate_penalty=0.5, prev_ctrl=torch.linspace(-1, 1, B, dtype=F64, device=DEV).view(B, 1))
    x0 = known_states(name, B, 900 + B + T).to(DEV)
    return MPC(n, 1, T, **kw)(x0, QuadCost(Q, pp), dx)


def _loss(x, u):
    g = torch.Generator().manual_seed(4)
    wx = torch.randn(x.shape, generator=g, dtype=F64).to(DEV)
    wu = torch.randn(u.shape, generator=g, dtype=F64).to(DEV)
    return (wx * x).sum() + (wu * u).sum()


def _params(name, where):
    p = torch.tensor(PHYS[name]["params"], dtype=F32 if where == "f32" else F64)
    if where == "cuda":
        p = p.to(DEV)
    elif where == "pinned":
        p = p.pin_memory()
    return p.requires_grad_(True)


E2E = [("in", "cuda", False), ("wide", "cuda", False), ("in", "cpu", False), ("wide", "pinned", False),
       ("in", "f32", False), ("in", "cuda", True), ("wide", "cpu", True)]


@pytest.mark.parametrize("bounds,where,slew", E2E, ids=[f"{b}_{w}{'_slew' if s else ''}" for b, w, s in E2E])
@pytest.mark.parametrize("name", SYSTEMS)
def test_param_grad_equals_module_path(name, bounds, where, slew):
    """params.grad through the kernels equals the pre-change route (the same physics as an opaque Module: torch
    AUTO_DIFF with create_graph), and arrives in the dtype and on the device of params."""
    B, T = 13, 15
    bound = (0.8 if bounds == "in" else 2.0) * PHYS[name]["clamp"]
    params = _params(name, where)
    dx = known_module(name, params=params)
    dx.params = params                                  # known_module copies with .to(); keep the caller's tensor
    xa, ua, _ = _solve(name, dx, B, T, bound, slew=slew)
    ga, = torch.autograd.grad(_loss(xa, ua), params)
    xb, ub, _ = _solve(name, _opaque(dx), B, T, bound, slew=slew)
    gb, = torch.autograd.grad(_loss(xb, ub), params)
    assert ga.dtype == params.dtype and ga.device == params.device
    tag = f"{name} {bounds} {where} slew={slew}"
    assert maxdiff(ua, ub) < 1e-7 * max(1.0, float(ub.abs().max())), f"{tag}: u"
    tol = (1e-7 if where != "f32" else 1e-6) * max(1.0, float(gb.abs().max()))
    assert maxdiff(ga, gb) < tol, f"{tag}: {ga.tolist()} vs {gb.tolist()}"
    assert float(ga.abs().sum()) > 0, tag


@pytest.mark.parametrize("name", SYSTEMS)
def test_analytic_equals_auto_diff(name):
    """GradMethods.ANALYTIC with a known system returns and backpropagates, bitwise as AUTO_DIFF."""
    from mpc.pytorch_b200 import GradMethods
    out = []
    for gm in (GradMethods.ANALYTIC, GradMethods.AUTO_DIFF):
        params = _params(name, "cuda")
        dx = known_module(name, params=params, device=DEV)
        x, u, costs = _solve(name, dx, 9, 12, PHYS[name]["clamp"], grad_method=gm)
        g, = torch.autograd.grad(_loss(x, u), params)
        out.append((x.detach(), u.detach(), costs, g))
    for a, b in zip(*out):
        assert torch.equal(a, b), name


@pytest.mark.parametrize("name", SYSTEMS)
def test_no_graph_when_params_need_no_grad(name):
    """Under no_grad, and with params.requires_grad False, the tail is one linearisation launch and builds no graph;
    MPC.forward's outputs are bitwise those of a run whose params require grad."""
    from mpc.pytorch_b200 import MPC, _lib
    B, T = 6, 10
    n = PHYS[name]["n"]
    x = torch.stack([known_states(name, B, 60 + t) for t in range(T)]).to(DEV)
    u = known_controls(name, T, B, F64, 61).to(DEV)
    mpc = MPC(n, 1, T)
    ref = None
    for mode in ("grad", "no_grad", "frozen"):
        params = _params(name, "cuda")
        if mode == "frozen":
            params.requires_grad_(False)
        dx = known_module(name, params=params, device=DEV)
        with torch.no_grad() if mode == "no_grad" else torch.enable_grad():
            l0 = _lib.launch_count()
            F, f = mpc.linearize_dynamics(x, u, dx, diff=True)
            launches = _lib.launch_count() - l0
            sol = _solve(name, dx, B, T, PHYS[name]["clamp"])
        assert launches == 1, f"{name} {mode}: {launches} launches"
        assert (F.grad_fn is None and f.grad_fn is None) == (mode != "grad"), f"{name} {mode}"
        res = [t.detach() for t in (F, f) + tuple(sol)]
        if ref is None:
            ref = res
        for a, b in zip(res, ref):
            assert torch.equal(a, b), f"{name} {mode}"


# ------------------------------------------------------------------------------------------------------------------
# system identification: learn the physical parameters back by imitation
# ------------------------------------------------------------------------------------------------------------------
# Thresholds on final / initial imitation loss and final / initial relative parameter error, from one seeded run on an
# H100 80GB HBM3 (700 W power limit): cartpole loss 33.2 -> 2.39 (0.072), error 0.400 -> 0.049 (0.12); pendulum loss
# 3.92 -> 1.77 (0.45), error 0.346 -> 0.158 (0.46).  The pendulum's imitation loss sees only g / l and m l^2, so its
# perturbation (+g, +m, -l) moves both.
SYSID = {"pendulum": dict(sign=(1.0, 1.0, -1.0), steps=40, lr=0.01, loss=0.6, err=0.6),
         "cartpole": dict(sign=(1.0, -1.0, 1.0, -1.0), steps=40, lr=0.05, loss=0.15, err=0.25)}


@pytest.mark.parametrize("name", SYSTEMS)
def test_system_identification(name):
    """Parameters perturbed by +-20 % are learnt back by Adam (f64, log-parametrised) from an imitation loss on the
    controls of solves with the true parameters: the loss falls and the parameter error shrinks."""
    from mpc.pytorch_b200 import MPC, QuadCost, GradMethods
    cfg = SYSID[name]
    B, T = 16, 20
    n = PHYS[name]["n"]
    true = torch.tensor(PHYS[name]["params"], dtype=F64, device=DEV)
    sign = torch.tensor(cfg["sign"], dtype=F64, device=DEV)
    start = true * (1 + 0.2 * sign)
    dx = known_module(name, params=true, device=DEV)
    q, p = dx.get_true_obj()
    Q = torch.diag(q).double().expand(T, B, n + 1, n + 1).contiguous().to(DEV)
    pp = p.double().expand(T, B, n + 1).contiguous().to(DEV)
    x0 = known_states(name, B, 123).to(DEV)
    clamp = PHYS[name]["clamp"]

    def solve():
        return MPC(n, 1, T, u_lower=-clamp, u_upper=clamp, lqr_iter=15, verbose=-1, exit_unconverged=False,
                   detach_unconverged=False, grad_method=GradMethods.AUTO_DIFF, eps=1e-8)(x0, QuadCost(Q, pp), dx)
    with torch.no_grad():
        _, u_true, _ = solve()
    w = torch.zeros(NP[name], dtype=F64, device=DEV, requires_grad=True)
    opt = torch.optim.Adam([w], lr=cfg["lr"])
    losses, errs = [], []
    for _ in range(cfg["steps"]):
        dx.params = start * torch.exp(w)
        errs.append(float(((dx.params - true) / true).norm()))
        _, u, _ = solve()
        loss = ((u - u_true) ** 2).mean()
        losses.append(float(loss))
        opt.zero_grad()
        loss.backward()
        opt.step()
    print(f"{name}: loss {losses[0]:.4e} -> {losses[-1]:.4e}, parameter error {errs[0]:.4f} -> {errs[-1]:.4f}")
    assert losses[-1] < cfg["loss"] * losses[0], losses
    assert errs[-1] < cfg["err"] * errs[0], errs
