"""GPU: differentiable receding-horizon episodes.  With differentiable=True the forward outputs are bitwise those of
differentiable=False; the device path's backward (one mpcb200_episode_backward_* call) matches the host path's
autograd loop for x_init, the cost, LinDx's F and f and the known systems' parameters; both match a hand-written
MPC.forward loop and, for unbounded LinDx, central finite differences; the reference's own notebook loop under
autograd (float64 fixture) agrees; slew-rate penalties and Module costs are differentiable on the host path; the
backward makes no host read, is one library call, and keeps batch problems independent."""
import functools
import os

import numpy as np
import pytest
import torch

from mpc.pytorch_b200 import control, step
from mpc.pytorch_b200.control import receding_horizon
from mpc.pytorch_b200.dynamics import CartpoleDx, PendulumDx
from mpc.pytorch_b200.solver import MPC, GradMethods, LinDx, QuadCost
from tests.cartpole import initial_states
from tests.gpu_harness import DEV, F32, F64, maxdiff, within
from tests.helpers import gen_problem

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


# ------------------------------------------------------------------------------------------------------------------
# cases: make() builds fresh leaves, so every run differentiates its own copies
# ------------------------------------------------------------------------------------------------------------------
class Case:
    """An episode: ctrl() a fresh MPC, leaves() fresh inputs {name: tensor} (x0, C, c, F, f | params, those that
    require grad), problem(leaves) -> (x0, cost, dx)."""

    def __init__(self, ctrl, leaves, problem, steps):
        self.ctrl, self.leaves, self.problem, self.steps = ctrl, leaves, problem, steps


def _cast(dtype, ref32):
    """Inputs are generated in float64 and rounded to float32 for a float32 case, and for its float64 reference
    (ref32), so that both see the same numbers."""
    return lambda t: t.to(F32).to(dtype) if dtype == F32 or ref32 else t.to(dtype)


def linear_case(B, T, n, m, dtype, bounds="none", steps=4, seed=0, mask=False, f_T=None, expand_F=False,
                cost_shape=4, ref32=False):
    cast = _cast(dtype, ref32)
    C, c, F, f, x0 = gen_problem(seed, B, T, n, m, F64)
    F = 0.9 * F
    if f_T == T:
        f = torch.cat((f, f[-1:]), 0)
    C, c, F, f, x0 = (cast(t) for t in (C, c, F, f, x0))
    g = torch.Generator().manual_seed(seed + 1)
    kw = dict(lqr_iter=8, verbose=-1)
    if bounds == "scalar":
        kw.update(u_lower=-0.25, u_upper=0.25)
    elif bounds == "tensor_delta":
        lo = cast(-0.1 - 0.3 * torch.rand(T, B, m, generator=g, dtype=F64))
        kw.update(u_lower=lo.to(DEV), u_upper=(-lo + 0.05).to(DEV), delta_u=0.1)
    if mask:
        kw["u_zero_I"] = (torch.rand(T, B, m, generator=g) < 0.3).to(DEV)
    if cost_shape == 3:                      # [T, p, p] / [T, p]: MPC expands them over the batch
        C, c = C[:, 0], c[:, 0]
    base = dict(x0=x0, C=C, c=c, F=F[:1] if expand_F else F, f=f)

    def leaves():
        return {k: v.clone().to(DEV).requires_grad_(True) for k, v in base.items()}

    def problem(lv):
        Fv = lv["F"].expand(T - 1, B, n, n + m) if expand_F else lv["F"]
        return lv["x0"], QuadCost(lv["C"], lv["c"]), LinDx(Fv, lv["f"])
    return Case(lambda: MPC(n, m, T, **kw), leaves, problem, steps)


def known_case(name, B, T, dtype, steps=4, seed=0, lqr_iter=20, ref32=False):
    cast = _cast(dtype, ref32)
    mods = {"cartpole": lambda p: CartpoleDx(params=p), "pendulum": lambda p: PendulumDx(params=p),
            "pendulum_full": lambda p: PendulumDx(params=p, simple=False)}
    defaults = {"cartpole": (9.8, 1.0, 0.1, 0.5), "pendulum": (10.0, 1.0, 1.0),
                "pendulum_full": (10.0, 1.0, 1.0, 0.1, 0.05)}
    sysdx = mods[name](torch.tensor(defaults[name], dtype=torch.float64))
    n, m = sysdx.n_state, sysdx.n_ctrl
    q, p = sysdx.get_true_obj()
    Q = cast(torch.diag(q.double()).expand(T, B, n + m, n + m))
    pp = cast(p.double().expand(T, B, n + m))
    if name == "cartpole":
        x0 = cast(initial_states(B, seed=seed).double())
    else:
        th = torch.linspace(-1.5, 1.5, B, dtype=torch.float64) + 0.1 * seed
        x0 = cast(torch.stack((th.cos(), th.sin(), 0.1 * th), 1))
    base = dict(x0=x0, C=Q, c=pp)

    def leaves():
        lv = {k: v.clone().to(DEV).requires_grad_(True) for k, v in base.items()}
        lv["params"] = cast(torch.tensor(defaults[name], dtype=F64)).to(DEV).requires_grad_(True)
        return lv

    def problem(lv):
        return lv["x0"], QuadCost(lv["C"], lv["c"]), mods[name](lv["params"])

    def ctrl():
        return MPC(n, m, T, u_lower=float(sysdx.lower), u_upper=float(sysdx.upper), lqr_iter=lqr_iter, verbose=-1,
                   linesearch_decay=sysdx.linesearch_decay, max_linesearch_iter=sysdx.max_linesearch_iter,
                   grad_method=GradMethods.AUTO_DIFF, eps=1e-2)
    return Case(ctrl, leaves, problem, steps)


def loss_weights(steps, B, n, m, dtype, seed=5):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(steps + 1, B, n, generator=g, dtype=torch.float64).to(DEV, dtype),
            torch.randn(steps, B, m, generator=g, dtype=torch.float64).to(DEV, dtype))


def episode_grads(monkeypatch, case, path, differentiable=True, lv=None):
    """receding_horizon on `path` ("device": asserting one episode_backward_raw call; "host"), then the fixed linear
    loss backward.  Returns (episode, {leaf name: grad})."""
    lv = case.leaves() if lv is None else lv
    x0, cost, dx = case.problem(lv)
    calls = []
    with monkeypatch.context() as mp:
        if path == "device":
            real = step.episode_backward_raw

            def spy(*a, **k):
                calls.append(1)
                return real(*a, **k)
            mp.setattr(step, "episode_backward_raw", spy)
        else:
            mp.setattr(control, "_episode_device_grad", lambda *a: None)
        ep = receding_horizon(case.ctrl(), x0, cost, dx, case.steps, differentiable=differentiable)
        if not differentiable:
            return ep, None
        wx, wu = loss_weights(case.steps, x0.shape[0], ep.x.shape[2], ep.u.shape[2], ep.x.dtype)
        ((wx * ep.x).sum() + (wu * ep.u).sum()).backward()
    torch.cuda.synchronize()
    assert len(calls) == (1 if path == "device" else 0), f"{path}: {len(calls)} backward calls"
    return ep, {k: v.grad for k, v in lv.items()}


def check_grads(tag, got, want, dtype, w32=None, w64=None, tol64=1e-10):
    """float64: |got - want| <= tol64 x max|want|; float32: the `within` policy against the float64 host gradient
    w64 (got from the float32 host gradient w32 = want)."""
    worst = {}
    for k in want:
        if want[k] is None:
            assert got[k] is None, (tag, k)
            continue
        assert got[k] is not None and got[k].shape == want[k].shape, (tag, k)
        if dtype == F64:
            scale = max(1e-300, float(want[k].abs().max()))
            err = maxdiff(got[k], want[k])
            assert err <= tol64 * scale, f"{tag}: d{k} {err:.3e} > {tol64 * scale:.3e}"
            worst[k] = err / scale
        else:
            within(tag, f"d{k}", got[k].double(), w64[k].double(), w32[k].double(), F32,
                   scale=max(1.0, float(w64[k].abs().max())))
            worst[k] = maxdiff(got[k], w32[k]) / max(1e-30, float(w32[k].abs().max()))
    print(f"{tag}: max |device - host| / max|g| = " + ", ".join(f"{k} {v:.2e}" for k, v in worst.items()))


def device_vs_host(monkeypatch, make, dtype):
    """make(dtype, ref32=False) -> Case.  The device backward against the host path's autograd (float32: against the float64 host
    gradient on float32-rounded inputs, by `within`)."""
    case = make(dtype)
    ep_d, g_d = episode_grads(monkeypatch, case, "device")
    ep_h, g_h = episode_grads(monkeypatch, case, "host")
    assert torch.equal(ep_d.x, ep_h.x) and torch.equal(ep_d.u, ep_h.u)
    if dtype == F64:
        check_grads("f64", g_d, g_h, F64)
        return g_d
    _, g64 = episode_grads(monkeypatch, make(F64, ref32=True), "host")
    check_grads("f32", g_d, g_h, F32, w32=g_h, w64=g64)
    return g_d


# ------------------------------------------------------------------------------------------------------------------
# forward unchanged
# ------------------------------------------------------------------------------------------------------------------
P = functools.partial
FWD_CASES = {
    "lin_none": P(linear_case, 16, 8, 8, 2),
    "lin_scalar": P(linear_case, 16, 8, 8, 2, bounds="scalar"),
    "lin_tensor_delta": P(linear_case, 16, 8, 8, 2, bounds="tensor_delta"),
    "lin_mask": P(linear_case, 16, 8, 8, 2, mask=True),
    "lin_padded": P(linear_case, 12, 6, 6, 1, bounds="scalar", seed=3),
    "lin_large": P(linear_case, 12, 6, 20, 4, bounds="scalar", seed=3),
    "cartpole": P(known_case, "cartpole", 8, 12),
    "pendulum": P(known_case, "pendulum", 8, 12),
    "pendulum_full": P(known_case, "pendulum_full", 8, 12),
}


@pytest.mark.parametrize("dtype", [F32, F64])
@pytest.mark.parametrize("name", list(FWD_CASES))
def test_forward_bitwise_unchanged(monkeypatch, dtype, name):
    case = FWD_CASES[name](dtype)
    plain, _ = episode_grads(monkeypatch, case, "device", differentiable=False)
    ep, _ = episode_grads(monkeypatch, case, "device")
    assert plain.x.grad_fn is None and plain.u.grad_fn is None
    assert ep.x.grad_fn is not None and ep.u.grad_fn is not None
    for k in ("x", "u", "costs", "info", "u_next"):
        assert torch.equal(getattr(ep, k), getattr(plain, k)), k
        assert not getattr(ep, k).requires_grad or k in ("x", "u"), k


def test_no_graph_without_grad(monkeypatch):
    case = FWD_CASES["cartpole"](F32)
    lv = case.leaves()
    x0, cost, dx = case.problem({k: v.detach() for k, v in lv.items()})
    ep = receding_horizon(case.ctrl(), x0, cost, dx, 3, differentiable=True)
    assert ep.x.grad_fn is None
    x0, cost, dx = case.problem(lv)
    with torch.no_grad():
        ep = receding_horizon(case.ctrl(), x0, cost, dx, 3, differentiable=True)
    assert ep.x.grad_fn is None


# ------------------------------------------------------------------------------------------------------------------
# device backward against the host path's autograd
# ------------------------------------------------------------------------------------------------------------------
GRAD_CASES = dict(FWD_CASES)
GRAD_CASES.update({
    "lin_expand_F_cost3": P(linear_case, 16, 8, 8, 2, bounds="scalar", expand_F=True, cost_shape=3),
    "lin_fT": P(linear_case, 16, 8, 4, 2, f_T=8),
})


@pytest.mark.parametrize("dtype", [F32, F64])
@pytest.mark.parametrize("name", list(GRAD_CASES))
def test_device_backward_matches_host(monkeypatch, dtype, name):
    device_vs_host(monkeypatch, GRAD_CASES[name], dtype)


@pytest.mark.parametrize("edge", ["n_steps_1", "T_3", "B_1", "B_45"])
def test_edges(monkeypatch, edge):
    make = {"n_steps_1": P(linear_case, 16, 8, 8, 2, bounds="scalar", steps=1),
            "T_3": P(known_case, "pendulum", 8, 3),
            "B_1": P(known_case, "cartpole", 1, 10),
            "B_45": P(linear_case, 45, 6, 4, 2, bounds="scalar")}[edge]
    device_vs_host(monkeypatch, make, F64)


def test_large_batch_index_width(monkeypatch):
    device_vs_host(monkeypatch, P(linear_case, 4096, 5, 8, 2, bounds="scalar", steps=2), F64)


# ------------------------------------------------------------------------------------------------------------------
# the hand-written loop, finite differences, the reference
# ------------------------------------------------------------------------------------------------------------------
def user_loop(case, lv):
    """The loop a user writes: MPC.forward, then the model step in torch (LinDx F[0] z + f[0], or dx(x, u))."""
    x0, cost, dx = case.problem(lv)
    x, w, xs, us = x0, None, [x0], []
    for _ in range(case.steps):
        ctrl = case.ctrl()
        ctrl.u_init, ctrl.exit_unconverged, ctrl.detach_unconverged = w, False, False
        _, plan_u, _ = ctrl(x, cost, dx)
        u = plan_u[0]
        if isinstance(dx, LinDx):
            x = torch.einsum("bij,bj->bi", dx.F[0], torch.cat((x, u), 1)) + dx.f[0]
        else:
            x = dx(x, u)
        w = control.shift_warm_start(plan_u.detach())
        xs.append(x)
        us.append(u)
    return torch.stack(xs), torch.stack(us)


@pytest.mark.parametrize("name", ["lin_scalar", "lin_tensor_delta", "cartpole", "pendulum", "pendulum_full"])
def test_against_user_loop(monkeypatch, name):
    case = GRAD_CASES[name](F64)
    _, g_d = episode_grads(monkeypatch, case, "device")
    lv = case.leaves()
    x, u = user_loop(case, lv)
    wx, wu = loss_weights(case.steps, x.shape[1], x.shape[2], u.shape[2], F64)
    ((wx * x).sum() + (wu * u).sum()).backward()
    for k, v in lv.items():
        scale = float(v.grad.abs().max())
        err = maxdiff(g_d[k], v.grad)
        assert err <= 1e-8 * max(1.0, scale), f"{name}: d{k} {err:.3e}"


def test_finite_differences_unbounded_linear(monkeypatch):
    case = linear_case(4, 6, 3, 2, F64, steps=3, seed=4)
    _, g = episode_grads(monkeypatch, case, "device")
    base = {k: v.detach() for k, v in case.leaves().items()}
    wx, wu = loss_weights(case.steps, 4, 3, 2, F64)

    def loss(lv):
        with torch.no_grad():
            ep = receding_horizon(case.ctrl(), *case.problem(lv), case.steps)
        return float((wx * ep.x).sum() + (wu * ep.u).sum())
    h = 1e-6
    for name, idx in (("x0", (1, 2)), ("c", (2, 1, 4)), ("c", (0, 3, 0)), ("F", (0, 2, 1, 3)), ("F", (3, 0, 2, 0))):
        plus = {k: v.clone() for k, v in base.items()}
        minus = {k: v.clone() for k, v in base.items()}
        plus[name][idx] += h
        minus[name][idx] -= h
        fd = (loss(plus) - loss(minus)) / (2 * h)
        assert abs(fd - float(g[name][idx])) <= 1e-6 * max(1.0, abs(fd)), (name, idx, fd, float(g[name][idx]))


@pytest.mark.parametrize("name", ["unbounded", "bounded"])
def test_against_reference_fixture(monkeypatch, name):
    path = os.path.join(GOLD, "receding_grad_linear_f64.npz")
    g = dict(np.load(path))
    pre = name + "_"
    t = {k[len(pre):]: torch.from_numpy(v) for k, v in g.items() if k.startswith(pre) and v.dtype == np.float64}
    T, steps = int(g[pre + "T"]), int(g[pre + "n_steps"])
    n = t["F"].shape[2]
    m = t["F"].shape[3] - n
    kw = dict(lqr_iter=int(g[pre + "lqr_iter"]), verbose=-1, eps=float(g[pre + "eps"]))
    if pre + "bound" in g:
        kw.update(u_lower=-float(g[pre + "bound"]), u_upper=float(g[pre + "bound"]))
    base = dict(x0=t["x_init"], C=t["C"], c=t["c"], F=t["F"], f=t["f"])
    case = Case(lambda: MPC(n, m, T, **kw),
                lambda: {k: v.clone().to(DEV).requires_grad_(True) for k, v in base.items()},
                lambda lv: (lv["x0"], QuadCost(lv["C"], lv["c"]), LinDx(lv["F"], lv["f"])), steps)
    lv = case.leaves()
    x0, cost, dx = case.problem(lv)
    ep = receding_horizon(case.ctrl(), x0, cost, dx, steps, differentiable=True)
    ((t["wx"].to(DEV) * ep.x).sum() + (t["wu"].to(DEV) * ep.u).sum()).backward()
    # unbounded: the same solves, to rounding; bounded: pnqp's own accuracy (it stops at |dx| < 1e-4, and the
    # reference couples that test over the batch, INTEGRATION.md section 2, so a solve may take other iterations to the
    # same fixed point), with the same controls on the bounds
    iters = ep.info[:, 0].cpu().long().tolist()
    print(f"{name}: iterations {iters}, reference {g[pre + 'iters'].tolist()}")
    if name == "unbounded":
        assert iters == g[pre + "iters"].tolist(), f"{name}: iterations per solve"
    tol = 1e-8 if name == "unbounded" else 2e-4
    if name == "bounded":
        bound = float(g[pre + "bound"])
        assert torch.equal(ep.u.abs() == bound, t["u"].to(DEV).abs() == bound)
    errs = {"x": maxdiff(ep.x, t["x"].to(DEV)), "u": maxdiff(ep.u, t["u"].to(DEV))}
    for k, ref in (("x0", "g_x_init"), ("C", "g_C"), ("c", "g_c"), ("F", "g_F"), ("f", "g_f")):
        want = t[ref].to(DEV)
        errs["d" + k] = maxdiff(lv[k].grad, want) / max(1.0, float(want.abs().max()))
    print(f"{name}: " + ", ".join(f"{k} {v:.2e}" for k, v in errs.items()))
    assert all(v <= tol for v in errs.values()), errs


# ------------------------------------------------------------------------------------------------------------------
# host-only episodes: slew-rate penalties, Module costs
# ------------------------------------------------------------------------------------------------------------------
class QuadModule(torch.nn.Module):
    def __init__(self, Q, p):
        super().__init__()
        self.Q, self.p = torch.nn.Parameter(Q), torch.nn.Parameter(p)

    def forward(self, tau):
        return 0.5 * (tau * (tau @ self.Q)).sum(-1) + (tau * self.p).sum(-1)


def slew_user_loop(make, x0, cost, dx, steps):
    x, w, prev, xs, us = x0, None, None, [x0], []
    for _ in range(steps):
        ctrl = make()
        ctrl.u_init, ctrl.prev_ctrl, ctrl.exit_unconverged, ctrl.detach_unconverged = w, prev, False, False
        _, plan_u, _ = ctrl(x, cost, dx)
        u = plan_u[0]
        x = torch.einsum("bij,bj->bi", dx.F[0], torch.cat((x, u), 1)) + dx.f[0] if isinstance(dx, LinDx) \
            else dx(x, u)
        w, prev = control.shift_warm_start(plan_u.detach()), u.detach()
        xs.append(x)
        us.append(u)
    return torch.stack(xs), torch.stack(us)


@pytest.mark.parametrize("name", ["slew_linear", "slew_pendulum", "module_cost"])
def test_host_path_against_user_loop(name):
    steps = 3
    if name == "slew_linear":
        case = linear_case(8, 6, 4, 2, F64, bounds="scalar", steps=steps)
        lv = case.leaves()
        x0, cost, dx = case.problem(lv)
        make = lambda: MPC(4, 2, 6, u_lower=-0.25, u_upper=0.25, lqr_iter=8, verbose=-1,  # noqa: E731
                           slew_rate_penalty=0.3)
        leaves = lv
    elif name == "slew_pendulum":
        case = known_case("pendulum", 6, 8, F64, steps=steps)
        lv = case.leaves()
        x0, cost, dx = case.problem(lv)

        def make():
            c = case.ctrl()
            c.slew_rate_penalty = 0.5
            return c
        leaves = lv
    else:
        case = known_case("cartpole", 4, 8, F64, steps=steps)
        lv = case.leaves()
        x0, cost, dx = case.problem(lv)
        cost = QuadModule(cost.C[0, 0].detach().clone(), cost.c[0, 0].detach().clone())

        def make():
            c = case.ctrl()
            c.n_batch = 4
            return c
        leaves = {"x0": lv["x0"], "params": lv["params"], "Q": cost.Q, "p": cost.p}
    ep = receding_horizon(make(), x0, cost, dx, steps, differentiable=True)
    wx, wu = loss_weights(steps, ep.x.shape[1], ep.x.shape[2], ep.u.shape[2], F64)
    got = torch.autograd.grad((wx * ep.x).sum() + (wu * ep.u).sum(), list(leaves.values()), allow_unused=True)
    x, u = slew_user_loop(make, x0, cost, dx, steps)
    assert maxdiff(ep.x, x) <= 1e-9 and maxdiff(ep.u, u) <= 1e-9
    want = torch.autograd.grad((wx * x).sum() + (wu * u).sum(), list(leaves.values()), allow_unused=True)
    for k, a, b in zip(leaves, got, want):
        if b is None:
            assert a is None or float(a.abs().max()) == 0.0, k
            continue
        err = maxdiff(a, b)
        assert err <= 1e-8 * max(1.0, float(b.abs().max())), f"{name}: d{k} {err:.3e}"


# ------------------------------------------------------------------------------------------------------------------
# one call, no host read, batch independence
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["lin_scalar", "pendulum"])
def test_backward_no_host_read(monkeypatch, name):
    """The whole backward, a known system's parameter gradient (CUDA params that require grad) included, makes no
    host read: the forward reads the parameters once, before the checked region."""
    case = GRAD_CASES[name](F32)
    episode_grads(monkeypatch, case, "device")                 # library load, kernel set-up
    lv = case.leaves()
    x0, cost, dx = case.problem(lv)
    ep = receding_horizon(case.ctrl(), x0, cost, dx, case.steps, differentiable=True)
    loss = ep.x.sum() + ep.u.sum()
    torch.cuda.synchronize()
    from mpc.pytorch_b200 import _lib
    before = _lib.launch_count()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert _lib.launch_count() > before
    assert all(v.grad is not None and bool(torch.isfinite(v.grad).all()) for v in lv.values())
    if "params" in lv:
        assert lv["params"].grad.device == DEV and bool((lv["params"].grad != 0).any())


def _fixed_iterations(case, lqr_iter=4):
    """The case's solver with a fixed number of iterations per solve (eps = 0 never stops it, nor does the
    not-improved counter): the stop test is the one place the forward couples the batch."""
    def ctrl():
        c = case.ctrl()
        c.eps, c.not_improved_lim, c.lqr_iter = 0.0, 10 ** 6, lqr_iter
        return c
    return ctrl


def _raw_episode(ctrl, lv, case):
    x0, cost, dx = case.problem(lv)
    n, x0_, C, c, F, f, dyn = ctrl._device_problem(x0, cost, dx)
    return step.episode_raw(n, ctrl.n_ctrl, ctrl.T, case.steps, x0_, C, c, F, f, control._first_warm_start(ctrl, x0),
                            dyn=dyn, keep_plans=True, **ctrl._device_options())


@pytest.mark.parametrize("name", ["lin_scalar", "cartpole"])
def test_batch_independence(name):
    """Problem 0's episode and every per-problem gradient row (dx_init, dC, dc, dF, df, dtheta) are bitwise unchanged
    when the other problems' inputs (x0 rows, C and c slices) and loss weights change."""
    case = GRAD_CASES[name](F64)
    make = _fixed_iterations(case)
    lv = {k: v.detach() for k, v in case.leaves().items()}
    lv2 = {k: v.clone() for k, v in lv.items()}
    lv2["x0"][1:] = lv2["x0"][1:].flip(0) * 0.7
    lv2["C"][:, 1:] = lv2["C"][:, 1:] * 1.5
    lv2["c"][:, 1:] = -lv2["c"][:, 1:]
    r1, r2 = _raw_episode(make(), lv, case), _raw_episode(make(), lv2, case)
    assert torch.equal(r1["x"][:, 0], r2["x"][:, 0]) and torch.equal(r1["u"][:, 0], r2["u"][:, 0])
    assert not torch.equal(r1["x"][:, 1:], r2["x"][:, 1:])
    wx, wu = loss_weights(case.steps, r1["x"].shape[1], r1["x"].shape[2], r1["u"].shape[2], F64)
    wx2, wu2 = wx.clone(), wu.clone()
    wx2[:, 1:] = wx2[:, 1:].flip(1) * 3.0
    wu2[:, 1:] = -wu2[:, 1:]
    g1 = step.episode_backward_raw(r1["saved"], wx, wu)
    g2 = step.episode_backward_raw(r2["saved"], wx2, wu2)
    torch.cuda.synchronize()
    rows = [(g1[0][0], g2[0][0])] + [(a[:, 0], b[:, 0]) for a, b in zip(g1[1:5], g2[1:5]) if a is not None]
    if g1[5] is not None:
        rows.append((g1[5][0], g2[5][0]))
    for k, (a, b) in enumerate(rows):
        assert torch.equal(a, b), k
    assert not torch.equal(g1[0][1:], g2[0][1:])


@pytest.mark.parametrize("name", ["lin_scalar", "cartpole"])
def test_inplace_edit_before_backward_raises(name):
    """x and u are saved for the backward: editing them in place before it is an error, not a gradient at points the
    episode never visited."""
    case = GRAD_CASES[name](F64)
    for edit in (lambda ep: ep.u.clamp_(-0.1, 0.1), lambda ep: ep.x.mul_(2.0)):
        lv = case.leaves()
        ep = receding_horizon(case.ctrl(), *case.problem(lv), case.steps, differentiable=True)
        loss = (ep.x * 1.0).sum() + (ep.u * 1.0).sum()
        edit(ep)
        with pytest.raises(RuntimeError, match="inplace"):
            loss.backward()


@pytest.mark.parametrize("name", ["lin_scalar", "cartpole"])
def test_episode_freed_without_cyclic_gc(name):
    """No reference cycle through the autograd node: with the cyclic collector off, the episode's outputs die once the
    episode and its loss are dropped after the backward."""
    import gc
    import weakref
    case = GRAD_CASES[name](F64)
    gc.collect()
    gc.disable()
    try:
        lv = case.leaves()
        ep = receding_horizon(case.ctrl(), *case.problem(lv), case.steps, differentiable=True)
        refs = [weakref.ref(ep.x), weakref.ref(ep.u)]
        loss = ep.x.sum() + ep.u.sum()
        loss.backward()
        del ep, loss
        assert all(r() is None for r in refs)
    finally:
        gc.enable()


def test_first_order_only():
    """The backward is raw kernels: differentiating it again raises instead of returning first-order results."""
    case = GRAD_CASES["lin_scalar"](F64)
    lv = case.leaves()
    ep = receding_horizon(case.ctrl(), *case.problem(lv), case.steps, differentiable=True)
    g = torch.autograd.grad(ep.x.sum() + ep.u.sum(), lv["x0"], create_graph=True)[0]
    with pytest.raises(RuntimeError):
        g.sum().backward()


def test_empty_f(monkeypatch):
    """LinDx with an empty f (the reference's "no f") that requires grad: both paths differentiate, and agree."""
    case = GRAD_CASES["lin_scalar"](F64)
    base = case.leaves()
    grads = {}
    for path in ("device", "host"):
        lv = {k: v.detach().clone().requires_grad_(True) for k, v in base.items()}
        lv["f"] = torch.empty(0, dtype=F64, device=DEV, requires_grad=True)
        with monkeypatch.context() as mp:
            if path == "host":
                mp.setattr(control, "_episode_device_grad", lambda *a: None)
            ep = receding_horizon(case.ctrl(), lv["x0"], QuadCost(lv["C"], lv["c"]), LinDx(lv["F"], lv["f"]),
                                  case.steps, differentiable=True)
            (ep.x.sum() + ep.u.sum()).backward()
        assert lv["f"].grad is None or lv["f"].grad.numel() == 0
        grads[path] = {k: lv[k].grad for k in ("x0", "C", "c", "F")}
    for k in grads["host"]:
        scale = float(grads["host"][k].abs().max())
        assert maxdiff(grads["device"][k], grads["host"][k]) <= 1e-10 * max(1.0, scale), k


@pytest.mark.parametrize("name", ["lin_scalar", "pendulum_full"])
def test_backward_captured_in_caller_graph(name):
    """On a capturing stream the backward's nodes join the caller's graph, and replays match eager calls."""
    case = GRAD_CASES[name](F32)
    x0, cost, dx = case.problem({k: v.detach() for k, v in case.leaves().items()})
    ctrl = case.ctrl()
    n, x0_, C, c, F, f, dyn = ctrl._device_problem(x0, cost, dx)
    w0 = control._first_warm_start(ctrl, x0)
    res = step.episode_raw(n, ctrl.n_ctrl, ctrl.T, case.steps, x0_, C, c, F, f, w0, dyn=dyn, keep_plans=True,
                           **ctrl._device_options())
    wx, wu = loss_weights(case.steps, x0.shape[0], n, ctrl.n_ctrl, F32)
    static_x, static_u = wx.clone(), wu.clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step.episode_backward_raw(res["saved"], static_x, static_u)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step.episode_backward_raw(res["saved"], static_x, static_u)
    for gx, gu in ((2.0 * wx, wu.flip(0)), (-wx, 0.5 * wu)):
        static_x.copy_(gx)
        static_u.copy_(gu)
        graph.replay()
        want = step.episode_backward_raw(res["saved"], gx, gu)
        torch.cuda.synchronize()
        for a, b in zip(out, want):
            assert (a is None) == (b is None) and (a is None or torch.equal(a, b))
