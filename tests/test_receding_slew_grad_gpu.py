"""GPU: differentiable receding-horizon episodes under a slew-rate penalty.  The device path makes one
mpcb200_episode_backward_slew_* call per backward; its forward is bitwise that of differentiable=False; its gradients
match the host path's autograd loop (f64 <= 1e-10 of max|g|, f32 by `within`), the float64 oracle's slew sweep on the
device's own plans at every instance and adjoint route the sweep reaches, the reference's own loop (float64 fixture)
and, for unbounded LinDx, central finite differences; prev_ctrl carries no gradient; the backward makes no host read,
can be captured, keeps batch problems independent, refuses in-place edits of x or u and is first order only."""
import os

import numpy as np
import pytest
import torch

from mpc.pytorch_b200 import _lib, control, step
from mpc.pytorch_b200.control import receding_horizon
from mpc.pytorch_b200.solver import LinDx, QuadCost
from oracle import slew_oracle as orc
from tests.gpu_harness import DEV, F32, F64, episode_known_step, maxdiff
from tests.test_receding_grad_gpu import Case, check_grads, known_case, linear_case, loss_weights

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SLEW = 0.1


def slew(case, dtype, penalty=SLEW, prev=None):
    """The case with a slew-rate penalty; prev: the first solve's prev_ctrl [B, m] (None: zeros)."""
    def ctrl():
        c = case.ctrl()
        c.slew_rate_penalty = penalty
        c.prev_ctrl = None if prev is None else prev.to(DEV, dtype)
        return c
    return Case(ctrl, case.leaves, case.problem, case.steps)


def prev_ctrl(B, m, seed=3):
    return 0.3 * torch.randn(B, m, generator=torch.Generator().manual_seed(seed), dtype=F64)


def run(monkeypatch, case, path, lv=None, spy=None):
    """receding_horizon with differentiable=True on `path` ("device": one episode_backward_raw call on the slew entry;
    "host"), then the fixed linear loss backward.  Returns (episode, grads, saved, wx, wu, library kernels the
    backward launched)."""
    lv = case.leaves() if lv is None else lv
    x0, cost, dx = case.problem(lv)
    calls = []
    with monkeypatch.context() as mp:
        if path == "device":
            real = step.episode_backward_raw

            def spy_fn(saved, *a):
                calls.append(saved)
                return real(saved, *a)
            mp.setattr(step, "episode_backward_raw", spy_fn)
        else:
            mp.setattr(control, "_episode_device_grad", lambda *a: None)
        ep = receding_horizon(case.ctrl(), x0, cost, dx, case.steps, differentiable=True)
        wx, wu = loss_weights(case.steps, x0.shape[0], ep.x.shape[2], ep.u.shape[2], ep.x.dtype)
        before = _lib.launch_count()
        ((wx * ep.x).sum() + (wu * ep.u).sum()).backward()
    torch.cuda.synchronize()
    launches = _lib.launch_count() - before
    if path == "device":
        assert len(calls) == 1, f"{len(calls)} backward calls"
        assert calls[0][0].n_prev == ep.u.shape[2], "not the slew entry"
    else:
        assert not calls
    return ep, {k: v.grad for k, v in lv.items()}, (calls[0] if calls else None), wx, wu, launches


def lin(n, m, bounds="none", **kw):
    return lambda dtype, ref32=False: linear_case(6, 8, n, m, dtype, bounds=bounds, ref32=ref32, **kw)


CASES = {
    "lin42": (lin(4, 2), None),
    "lin42_prev": (lin(4, 2), 2),
    "lin52_pad": (lin(5, 2), None),
    "lin143_large": (lin(14, 3), 3),
    "lin42_scalar": (lin(4, 2, "scalar"), 2),
    "lin42_tensor_delta": (lin(4, 2, "tensor_delta"), 2),
    "lin42_mask": (lin(4, 2, mask=True), None),
    "lin42_fT": (lin(4, 2, f_T=8), 2),
    "lin42_expandF": (lin(4, 2, expand_F=True), None),
    "lin42_cost3": (lin(4, 2, cost_shape=3), 2),
    "cartpole": (lambda dtype, ref32=False: known_case("cartpole", 6, 8, dtype, ref32=ref32), 1),
    "pendulum": (lambda dtype, ref32=False: known_case("pendulum", 6, 8, dtype, ref32=ref32), None),
    "pendulum_full": (lambda dtype, ref32=False: known_case("pendulum_full", 6, 8, dtype, ref32=ref32), 1),
}


def make(name, dtype, ref32=False):
    mk, pm = CASES[name]
    base = mk(dtype, ref32=ref32)
    return slew(base, dtype, prev=None if pm is None else prev_ctrl(6, pm))


# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["lin42", "lin52_pad", "lin143_large", "cartpole", "pendulum", "pendulum_full"])
@pytest.mark.parametrize("dtype", [F32, F64])
def test_forward_bitwise_and_route(monkeypatch, name, dtype):
    """differentiable=True runs the same episode graph as differentiable=False, and its backward the slew entry."""
    case = make(name, dtype)
    lv = case.leaves()
    ep, _, _, _, _, _ = run(monkeypatch, case, "device", lv=lv)
    ep0 = receding_horizon(case.ctrl(), *case.problem(lv), case.steps, differentiable=False)
    assert torch.equal(ep.x.detach(), ep0.x) and torch.equal(ep.u.detach(), ep0.u)
    assert torch.equal(ep.costs, ep0.costs) and torch.equal(ep.u_next, ep0.u_next)


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("dtype", [F64, F32])
def test_device_against_host(monkeypatch, name, dtype):
    case = make(name, dtype)
    ep_d, g_d, _, _, _, _ = run(monkeypatch, case, "device")
    ep_h, g_h, _, _, _, _ = run(monkeypatch, case, "host")
    assert torch.equal(ep_d.x.detach(), ep_h.x.detach()) and torch.equal(ep_d.u.detach(), ep_h.u.detach())
    if dtype == F64:
        check_grads(f"{name} f64", g_d, g_h, F64)
    else:
        _, g64, _, _, _, _ = run(monkeypatch, make(name, F64, ref32=True), "host")
        check_grads(f"{name} f32", g_d, g_h, F32, w32=g_h, w64=g64)


def test_prev_ctrl_gets_no_gradient(monkeypatch):
    case = make("lin42", F64)
    prev = prev_ctrl(6, 2).to(DEV).requires_grad_(True)
    ctrl0 = case.ctrl

    def ctrl():
        c = ctrl0()
        c.prev_ctrl = prev
        return c
    _, g, _, _, _, _ = run(monkeypatch, Case(ctrl, case.leaves, case.problem, case.steps), "device")
    assert prev.grad is None and all(v is not None for v in g.values())


# ------------------------------------------------------------------------------------------------------------------
def oracle_grads(name, saved, wx, wu, n, m, prev):
    """The float64 oracle's slew sweep on the device's own plans, states and controls."""
    s, n_steps, xs, us, plan_x, plan_u = saved
    T, B = s.dims.T, s.dims.B
    cpu = lambda t: t.detach().to("cpu", F64)                 # noqa: E731
    xs_, us_ = cpu(xs[..., m:n + m]), cpu(us[..., :m])
    px, pu = cpu(plan_x[..., :n + m]), cpu(plan_u[..., :m])
    return xs_, us_, px, pu


@pytest.mark.parametrize("name", ["lin42_prev", "lin52_pad", "lin143_large", "lin42_tensor_delta", "cartpole",
                                  "pendulum", "pendulum_full"])
def test_device_against_oracle(monkeypatch, name):
    """f64 device gradients against the oracle's slew sweep on the device's own plans.  The adjoint's route, from the
    backward's launch count (gpu_harness.epgrad_launches): the fused column-pair kernel where the augmented shape has
    an instance ((6, 2), padded (7, 2) -> (8, 2), the pendulums' (4, 1)); the three-launch route where it has none
    (cartpole's (6, 1), (14, 3)'s (17, 3): the large-shape kernels)."""
    from tests.gpu_harness import epgrad_launches
    case = make(name, F64)
    lv = case.leaves()
    ep, g, saved, wx, wu, launches = run(monkeypatch, case, "device", lv=lv)
    ctrl = case.ctrl()
    n, m, T = ctrl.n_state, ctrl.n_ctrl, ctrl.T
    xs, us, px, pu = oracle_grads(name, saved, wx, wu, n, m, ctrl.prev_ctrl)
    cpu = lambda t: t.detach().to("cpu", F64) if isinstance(t, torch.Tensor) else t      # noqa: E731
    x0, cost, dx = case.problem({k: v.detach() for k, v in lv.items()})
    C, c = cost.C, cost.c
    if C.dim() == 3:
        C, c = C.unsqueeze(1).expand(T, xs.shape[1], *C.shape[1:]), c.unsqueeze(1).expand(T, xs.shape[1], -1)
    kw = dict(slew_rate_penalty=SLEW, prev_ctrl=cpu(ctrl.prev_ctrl), u_lower=cpu(ctrl.u_lower),
              u_upper=cpu(ctrl.u_upper))
    if ctrl.u_zero_I is not None:
        pytest.skip("u_zero_I is not an oracle backward option")
    if isinstance(dx, LinDx):
        out = orc.receding_horizon_backward(n, m, T, cpu(C), cpu(c), cpu(dx.F), cpu(dx.f), xs, us, px, pu, cpu(wx),
                                            cpu(wu), **kw)
        pairs = {"x0": out["dx_init"], "C": out["dC"], "c": out["dc"], "F": out["dF"], "f": out["df"]}
    else:
        mod = dx.__class__(params=cpu(dx.params), **({"simple": False} if name == "pendulum_full" else {}))
        B = xs.shape[1]
        out = orc.receding_horizon_backward(n, m, T, cpu(C), cpu(c), None, None, xs, us, px, pu, cpu(wx), cpu(wu),
                                            step=episode_known_step(mod), theta=cpu(dx.params).expand(B, -1),
                                            full_linearisation=True, **kw)
        pairs = {"x0": out["dx_init"], "C": out["dC"], "c": out["dc"], "params": out["dtheta"].sum(0)}
    worst = {}
    for k, want in pairs.items():
        got = cpu(g[k])
        scale = max(1e-300, float(want.abs().max()))
        worst[k] = maxdiff(got, want) / scale
        assert worst[k] <= 1e-9, (name, k, worst[k])
    known = not isinstance(dx, LinDx)
    route = "fused" if launches == epgrad_launches("fused", known) else "three-launch"
    print(f"{name}: N={saved[0].pad.N} M={saved[0].pad.M} launches={launches} route={route} "
          "max |device - oracle| / max|g| = " + ", ".join(f"{k} {v:.2e}" for k, v in worst.items()))
    assert launches in (epgrad_launches(r, known) for r in ("fused", "large")), launches
    if name in ("lin143_large", "cartpole"):
        assert route == "three-launch", (name, launches)


# ------------------------------------------------------------------------------------------------------------------
def _fixture():
    return {k: torch.from_numpy(v) for k, v in np.load(os.path.join(GOLD, "receding_grad_slew_f64.npz")).items()}


@pytest.mark.parametrize("case", ["unbounded", "bounded"])
def test_linear_against_reference(monkeypatch, case):
    """The reference's own loop (an affine Module plant, see the generator): x, u and every gradient."""
    z = _fixture()
    g = lambda k: z[case + "_" + k]                            # noqa: E731
    T, steps, n, m = int(g("T")), int(g("n_steps")), 4, 2
    B = g("x_init").shape[0]
    kw = dict(lqr_iter=int(g("lqr_iter")), eps=float(g("eps")), verbose=-1, slew_rate_penalty=float(g("slew")))
    if case + "_bound" in z:
        kw.update(u_lower=-float(g("bound")), u_upper=float(g("bound")))
    lv = {k: g(k).clone().to(DEV).requires_grad_(True) for k in ("x_init", "C", "c", "F", "f")}

    def ctrl():
        from mpc.pytorch_b200.solver import MPC
        c_ = MPC(n, m, T, **kw)
        c_.prev_ctrl = g("prev_ctrl").to(DEV) if case + "_prev_ctrl" in z else None
        return c_

    def problem(v):
        return v["x_init"], QuadCost(v["C"], v["c"]), LinDx(v["F"].expand(T - 1, B, n, n + m),
                                                             v["f"].expand(T - 1, B, n))
    calls = []
    real = step.episode_backward_raw
    monkeypatch.setattr(step, "episode_backward_raw", lambda *a: calls.append(1) or real(*a))
    ep = receding_horizon(ctrl(), *problem(lv), steps, differentiable=True)
    ((g("wx").to(DEV) * ep.x).sum() + (g("wu").to(DEV) * ep.u).sum()).backward()
    assert calls == [1]
    # unbounded: the same solves, to rounding; bounded: pnqp's own accuracy (test_receding_grad_gpu's policy), with the
    # same controls on the bounds
    tol = 1e-8 if case == "unbounded" else 2e-4
    if case == "unbounded":
        assert ep.info[:, 0].cpu().tolist() == g("iters").tolist()
    else:
        b = float(g("bound"))
        assert torch.equal(ep.u.detach().cpu().abs() == b, g("u").abs() == b)
    errs = {"x": maxdiff(ep.x.detach().cpu(), g("x")), "u": maxdiff(ep.u.detach().cpu(), g("u"))}
    errs.update({k: maxdiff(lv[k].grad.cpu(), g("g_" + k)) / max(1.0, float(g("g_" + k).abs().max())) for k in lv})
    print(case, {k: f"{v:.1e}" for k, v in errs.items()})
    assert max(errs.values()) <= tol, errs


@pytest.mark.parametrize("name", ["pendulum", "cartpole"])
def test_known_against_reference(monkeypatch, name):
    """dx_init, dC, dc against the reference's loop; dtheta against the oracle's full linearisation derivative."""
    from mpc.pytorch_b200.dynamics import CartpoleDx, PendulumDx
    from mpc.pytorch_b200.solver import MPC, GradMethods
    z = _fixture()
    g = lambda k: z[name + "_" + k]                            # noqa: E731
    T, steps = int(g("T")), int(g("n_steps"))
    clamp = float(g("clamp"))
    cls = CartpoleDx if name == "cartpole" else PendulumDx
    lv = {k: g(k).clone().to(DEV).requires_grad_(True) for k in ("x_init", "C", "c", "params")}
    dx = cls(params=lv["params"])
    if name == "cartpole":
        dx.force_mag = clamp
    else:
        dx.max_torque = clamp
    n = dx.n_state
    ctrl = MPC(n, 1, T, u_lower=-clamp, u_upper=clamp, lqr_iter=int(g("lqr_iter")), eps=float(g("eps")), verbose=-1,
               linesearch_decay=float(g("ls_decay")), max_linesearch_iter=int(g("ls_iter")),
               grad_method=GradMethods.AUTO_DIFF, slew_rate_penalty=float(g("slew")))
    calls = []
    real = step.episode_backward_raw
    monkeypatch.setattr(step, "episode_backward_raw", lambda *a: calls.append(a[0]) or real(*a))
    ep = receding_horizon(ctrl, lv["x_init"], QuadCost(lv["C"], lv["c"]), dx, steps, differentiable=True)
    ((g("wx").to(DEV) * ep.x).sum() + (g("wu").to(DEV) * ep.u).sum()).backward()
    assert len(calls) == 1
    # the solves stop at eps = 1e-4 and the kernels' Jacobians are exact where the reference's are autograd's: the
    # episodes agree to the solver's accuracy (the bounded LinDx policy, 2e-4)
    errs = {"x": maxdiff(ep.x.detach().cpu(), g("x")), "u": maxdiff(ep.u.detach().cpu(), g("u"))}
    errs.update({k: maxdiff(lv[k].grad.cpu(), g("g_" + k)) / max(1.0, float(g("g_" + k).abs().max()))
                 for k in ("x_init", "C", "c")})
    mod = cls(params=g("params").clone())
    B = g("x").shape[1]
    out = orc.receding_horizon_backward(n, 1, T, g("C"), g("c"), None, None, g("x"), g("u"), g("plan_x"),
                                        g("plan_u"), g("wx"), g("wu"), u_lower=-clamp, u_upper=clamp,
                                        step=episode_known_step(mod), theta=g("params").expand(B, -1),
                                        full_linearisation=True, slew_rate_penalty=float(g("slew")))
    errs["params"] = maxdiff(lv["params"].grad.cpu(), out["dtheta"].sum(0)) / max(1.0, float(
        out["dtheta"].sum(0).abs().max()))
    print(name, {k: f"{v:.1e}" for k, v in errs.items()})
    assert max(errs["x"], errs["u"]) <= 5e-4 and max(v for k, v in errs.items() if k not in "xu") <= 2e-4, errs


# ------------------------------------------------------------------------------------------------------------------
def test_finite_differences(monkeypatch):
    """Central differences in float64 of an unbounded LinDx slew episode in x_init, c, F and f.  The differentiated
    function is the loop with each solve's previous control held at the episode's own value (prev_ctrl, then u_{k-1}),
    which is what detaching it means; a perturbed prev_ctrl leaves the gradients of this affine episode in x_init, c
    and f unchanged."""
    from mpc.pytorch_b200.solver import MPC
    base = make("lin42_prev", F64)
    lv0 = {k: v.detach() for k, v in base.leaves().items()}
    ep, g, _, wx, wu, _ = run(monkeypatch, base, "device", lv={k: v.clone().requires_grad_(True)
                                                                for k, v in lv0.items()})
    ctrl0 = base.ctrl()
    prevs = [ctrl0.prev_ctrl] + [ep.u[k].detach() for k in range(base.steps - 1)]

    def loss(lv):
        x0, cost, dx = base.problem(lv)
        x, total = x0, float((wx[0] * x0).sum())
        with torch.no_grad():
            for k in range(base.steps):
                c = base.ctrl()
                c.prev_ctrl = prevs[k]
                _, plan_u, _ = c(x, cost, dx)
                u = plan_u[0]
                x = torch.einsum("bij,bj->bi", dx.F[0], torch.cat((x, u), 1)) + dx.f[0]
                total += float((wx[k + 1] * x).sum() + (wu[k] * u).sum())
        return total
    assert isinstance(ctrl0, MPC)
    gen = torch.Generator().manual_seed(9)
    h = 1e-6
    for k in ("x0", "c", "F", "f"):
        for _ in range(4):
            idx = tuple(int(torch.randint(0, s, (1,), generator=gen)) for s in lv0[k].shape)
            lp = {q: v.clone() for q, v in lv0.items()}
            lm = {q: v.clone() for q, v in lv0.items()}
            lp[k][idx] += h
            lm[k][idx] -= h
            fd = (loss(lp) - loss(lm)) / (2 * h)
            assert abs(fd - float(g[k][idx])) <= 1e-6 * max(1.0, abs(fd)), (k, idx, fd, float(g[k][idx]))
    other = slew(CASES["lin42_prev"][0](F64), F64, prev=prev_ctrl(6, 2, seed=8))
    _, g2, _, _, _, _ = run(monkeypatch, other, "device", lv={k: v.clone().requires_grad_(True)
                                                                 for k, v in lv0.items()})
    for k in ("x0", "c", "f"):
        assert maxdiff(g2[k], g[k]) <= 1e-9 * max(1.0, float(g[k].abs().max())), k


# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["lin42_scalar", "pendulum"])
def test_no_host_read(monkeypatch, name):
    case = make(name, F64)
    lv = case.leaves()
    ep = receding_horizon(case.ctrl(), *case.problem(lv), case.steps, differentiable=True)
    loss = ep.x.sum() + ep.u.sum()
    before = _lib.launch_count()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert _lib.launch_count() > before


def _raw(case, lv):
    ctrl = case.ctrl()
    x0, cost, dx = case.problem(lv)
    n, x0_, C, c, F, f, dyn = ctrl._device_problem(x0, cost, dx)
    return step.episode_raw(n, ctrl.n_ctrl, ctrl.T, case.steps, x0_, C, c, F, f, control._first_warm_start(ctrl, x0),
                            dyn=dyn, keep_plans=True, n_prev=ctrl.n_ctrl, **ctrl._device_options()), n, ctrl.n_ctrl


@pytest.mark.parametrize("name", ["lin42_scalar", "pendulum_full"])
def test_captured_in_caller_graph(name):
    case = make(name, F32)
    res, n, m = _raw(case, {k: v.detach() for k, v in case.leaves().items()})
    wx, wu = loss_weights(case.steps, res["x"].shape[1], n, m, F32)
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
    assert float(out[0][:, :m].abs().max()) == 0.0              # the previous control's part of dx_init


@pytest.mark.parametrize("name", ["lin42_scalar", "cartpole"])
def test_batch_independence(name):
    case = make(name, F64)
    ctrl0 = case.ctrl

    def ctrl():
        c = ctrl0()
        c.eps, c.not_improved_lim, c.lqr_iter = 0.0, 10 ** 6, 4
        return c
    case = Case(ctrl, case.leaves, case.problem, case.steps)
    lv = {k: v.detach() for k, v in case.leaves().items()}
    lv2 = {k: v.clone() for k, v in lv.items()}
    lv2["x0"][1:] = lv2["x0"][1:].flip(0) * 0.7
    lv2["C"][:, 1:] = lv2["C"][:, 1:] * 1.5
    lv2["c"][:, 1:] = -lv2["c"][:, 1:]
    (r1, n, m), (r2, _, _) = _raw(case, lv), _raw(case, lv2)
    assert torch.equal(r1["x"][:, 0], r2["x"][:, 0]) and torch.equal(r1["u"][:, 0], r2["u"][:, 0])
    wx, wu = loss_weights(case.steps, r1["x"].shape[1], n, m, F64)
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


@pytest.mark.parametrize("name", ["lin42_scalar", "cartpole"])
def test_inplace_edit_before_backward_raises(name):
    case = make(name, F64)
    for edit in (lambda ep: ep.u.clamp_(-0.1, 0.1), lambda ep: ep.x.mul_(2.0)):
        lv = case.leaves()
        ep = receding_horizon(case.ctrl(), *case.problem(lv), case.steps, differentiable=True)
        loss = (ep.x * 1.0).sum() + (ep.u * 1.0).sum()
        with pytest.raises(RuntimeError, match="inplace"):     # x is a view of the augmented states: at the edit
            edit(ep)
            loss.backward()


def test_first_order_only():
    case = make("lin42_scalar", F64)
    lv = case.leaves()
    ep = receding_horizon(case.ctrl(), *case.problem(lv), case.steps, differentiable=True)
    g = torch.autograd.grad(ep.x.sum() + ep.u.sum(), lv["x0"], create_graph=True)[0]
    with pytest.raises(RuntimeError):
        g.sum().backward()
