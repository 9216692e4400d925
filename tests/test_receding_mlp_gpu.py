"""GPU: receding-horizon episodes planned with a learned model as one CUDA graph (mpcb200_episode_mlp_*,
mpcb200_episode_backward_mlp_*; control.receding_horizon through mlp.episode_on_device).

Forwards are checked bitwise against a loop of MPC.forward and mlp.rollout_raw (or the plant's kernels), which runs
the same kernels on the same staged problem, and against the host path (the network stepped by its torch Module):
float64 within 1e-12 of max|x|; float32 within 1e-4 of max|x| on unbounded episodes, where the two differ only in the
model step's float32 rounding (torch's GEMM against the kernel's fixed-order sums, a few ulp per step), amplified by
at most the few solves and steps of the episode.  Gradients are checked against the host path's autograd (float64
1e-11 of max|g|; float32 2e-3 of max|g|, the same rounding carried through the adjoints), against central
differences, and against the reference's fixture.  Every output and workspace of the library calls starts at NaN
(poisoned)."""
import copy

import pytest
import torch

from mpc.pytorch_b200 import _lib, control, mlp as mlpmod, solver
from mpc.pytorch_b200.control import receding_horizon, shift_warm_start
from mpc.pytorch_b200.dynamics import PendulumDx, params_scope
from mpc.pytorch_b200.models import NNDynamics
from mpc.pytorch_b200.solver import MPC, GradMethods, LinDx, QuadCost
from tests.gpu_harness import DEV, F32, F64, maxdiff
from tests.test_mlp_gpu import poisoned

pytestmark = pytest.mark.gpu


def _net(n, m, hidden, act="sigmoid", passthrough=True, dtype=F64, seed=0):
    torch.manual_seed(seed)
    net = NNDynamics(n, m, hidden_sizes=hidden, activation=act, passthrough=passthrough).double()
    with torch.no_grad():
        for fc in net.fcs:
            fc.weight.mul_(0.5)
    return net.to(dtype=dtype, device=DEV)


def _problem(n, m, T, B, dtype, seed=1):
    g = torch.Generator().manual_seed(seed)
    p = n + m
    A = torch.randn(T, B, p, p, generator=g, dtype=F64) * 0.3
    C = A @ A.transpose(-1, -2) + torch.eye(p, dtype=F64)
    c = torch.randn(T, B, p, generator=g, dtype=F64)
    x0 = torch.randn(B, n, generator=g, dtype=F64)
    return [t.to(dtype=dtype, device=DEV) for t in (x0, C, c)]


def _ctrl(n, m, T, bound=None, **kw):
    box = {}
    if bound == "scalar":
        box = dict(u_lower=-0.8, u_upper=0.8)
    opts = dict(lqr_iter=8, verbose=-1, grad_method=GradMethods.ANALYTIC, exit_unconverged=False,
                detach_unconverged=False, eps=1e-8)
    opts.update(kw)
    return MPC(n, m, T, **box, **opts)


def _tensor_bounds(ctrl, T, B, m, dtype):
    g = torch.Generator().manual_seed(7)
    lo = -0.5 - torch.rand(T, B, m, generator=g, dtype=F64)
    ctrl.u_lower, ctrl.u_upper = lo.to(dtype=dtype, device=DEV), (-lo).to(dtype=dtype, device=DEV)


def _loop(ctrl, x0, cost, dx, n_steps, plant=None, w=None):
    """The episode as a loop of MPC.forward and the kernels the graph steps with: the network's rollout at T = 2, a
    LinDx plant's rollout, a known plant's (control._model_step); plans and warm starts as receding_horizon's."""
    solve = copy.copy(ctrl)
    x, wk = x0, control._first_warm_start(ctrl, x0)
    xs, us, costs, infos, px, pu = [x0], [], [], [], [], []
    with torch.no_grad(), params_scope():
        for k in range(n_steps):
            solve.u_init = wk
            plan_x, plan_u, plan_costs = solve(x, cost, dx)
            if plant is None or plant is dx:
                x = mlpmod.rollout_raw(dx, 2, x, plan_u[:2])[1]
            else:
                x = control._model_step(solve, x, plan_u, cost, plant)
            if w is not None:
                x = x + w[k]
            wk = shift_warm_start(plan_u)
            xs.append(x)
            us.append(plan_u[0])
            costs.append(plan_costs)
            infos.append(solve._solve_info.to(DEV))
            px.append(plan_x)
            pu.append(plan_u)
    return (torch.stack(xs), torch.stack(us), torch.stack(costs), torch.stack(infos), wk, torch.stack(px),
            torch.stack(pu))


def _device(ctrl, x0, cost, dx, n_steps, plant=None, w=None):
    """mlp.episode_raw(keep_plans=True) on the problem receding_horizon stages, poisoned."""
    n, m, T = ctrl.n_state, ctrl.n_ctrl, ctrl.T
    w0 = control._first_warm_start(ctrl, x0)
    with torch.no_grad(), params_scope(), poisoned():
        nn_, x0_, C, c, _, _, _ = ctrl._device_problem(x0, cost, dx)
        F_p, f_p = (plant.F, plant.f) if isinstance(plant, LinDx) else (None, None)
        spec = control._net_plant_spec(ctrl, x0, C, dx, plant, F_p, f_p)
        res = mlpmod.episode_raw(dx, nn_, m, T, n_steps, x0_, C, c, w0, plant=spec, w=w, keep_plans=True,
                                 **ctrl._device_options())
    s = res["saved"][0]
    return res, s.pad.crop_n(res["saved"][4]), s.pad.crop_m(res["saved"][5])


def _equal(a, b):
    return a.shape == b.shape and torch.equal(a, b)


FORWARD = [  # (n, m, hidden, act, passthrough, bound, delta_u)
    (3, 2, [12, 10], "sigmoid", True, None, None),
    (3, 2, [12], "relu", False, "scalar", None),
    (3, 2, [8, 8, 8], "elu", True, "tensor", None),
    (3, 2, [], "sigmoid", False, "scalar", 0.3),
    (5, 2, [16], "elu", True, None, None),          # padded to the (6, 2) instance
    (18, 5, [24], "sigmoid", True, "scalar", None),  # the large-shape kernels
]


@pytest.mark.parametrize("dtype", [F64, F32])
@pytest.mark.parametrize("case", FORWARD)
def test_forward_matches_a_loop(case, dtype):
    n, m, hidden, act, pt, bound, delta_u = case
    T, B, steps = 6, 4, 4
    dx = _net(n, m, hidden, act, pt, dtype)
    x0, C, c = _problem(n, m, T, B, dtype)
    ctrl = _ctrl(n, m, T, bound, delta_u=delta_u)
    if bound == "tensor":
        _tensor_bounds(ctrl, T, B, m, dtype)
    cost = QuadCost(C, c)
    res, plan_x, plan_u = _device(ctrl, x0, cost, dx, steps)
    xs, us, costs, infos, u_next, px, pu = _loop(ctrl, x0, cost, dx, steps)
    assert _equal(res["x"], xs) and _equal(res["u"], us) and _equal(res["costs"], costs)
    assert _equal(res["info"], infos) and _equal(res["u_next"], u_next)
    assert _equal(plan_x, px) and _equal(plan_u, pu)
    calls = []
    real = mlpmod.episode_raw
    mlpmod.episode_raw = lambda *a, **k: calls.append(1) or real(*a, **k)
    try:
        with poisoned():
            ep = receding_horizon(ctrl, x0, cost, dx, steps)
    finally:
        mlpmod.episode_raw = real
    assert calls and _equal(ep.x, xs) and _equal(ep.u, us) and _equal(ep.u_next, u_next)


def _pendulum(dtype):
    return PendulumDx(params=torch.tensor((10.0, 1.0, 1.0), dtype=dtype, device=DEV))


def _lindx_plant(n, m, B, dtype):
    g = torch.Generator().manual_seed(3)
    F = torch.cat((torch.eye(n, dtype=F64) + 0.05 * torch.randn(n, n, generator=g, dtype=F64),
                   0.1 * torch.randn(n, m, generator=g, dtype=F64)), 1).expand(1, B, n, n + m).clone()
    f = 0.02 * torch.randn(1, B, n, generator=g, dtype=F64)
    return LinDx(F.to(dtype=dtype, device=DEV), f.to(dtype=dtype, device=DEV))


def _w(steps, B, n, dtype):
    g = torch.Generator().manual_seed(4)
    return (0.01 * torch.randn(steps, B, n, generator=g, dtype=F64)).to(dtype=dtype, device=DEV)


@pytest.mark.parametrize("dtype", [F64, F32])
@pytest.mark.parametrize("plant", ["self", "lindx", "pendulum"])
def test_plant_forward_matches_a_loop(plant, dtype):
    n, m, T, B, steps = 3, 1, 6, 4, 4
    dx = _net(n, m, [16], "sigmoid", True, dtype)
    x0, C, c = _problem(n, m, T, B, dtype)
    p = {"self": dx, "lindx": _lindx_plant(n, m, B, dtype), "pendulum": _pendulum(dtype)}[plant]
    w = _w(steps, B, n, dtype)
    ctrl = _ctrl(n, m, T, "scalar")
    cost = QuadCost(C, c)
    res, plan_x, plan_u = _device(ctrl, x0, cost, dx, steps, p, w)
    xs, us, costs, infos, u_next, px, pu = _loop(ctrl, x0, cost, dx, steps, p, w)
    assert _equal(res["x"], xs) and _equal(res["u"], us) and _equal(res["costs"], costs)
    assert _equal(res["info"], infos) and _equal(res["u_next"], u_next)
    assert _equal(plan_x, px) and _equal(plan_u, pu)


def _host(monkeypatch, fn):
    with monkeypatch.context() as mp:
        mp.setattr(mlpmod, "episode_on_device", lambda *a, **k: False)
        return fn()


@pytest.mark.parametrize("dtype", [F64, F32])
def test_forward_matches_the_host_path(dtype, monkeypatch):
    n, m, T, B, steps = 3, 2, 8, 4, 5
    dx = _net(n, m, [12, 10], "sigmoid", True, dtype)
    x0, C, c = _problem(n, m, T, B, dtype)
    ctrl = _ctrl(n, m, T)
    cost = QuadCost(C, c)
    ep = receding_horizon(ctrl, x0, cost, dx, steps)
    eh = _host(monkeypatch, lambda: receding_horizon(ctrl, x0, cost, dx, steps))
    # the solves turn the model steps' last-bit differences into more in u and the costs: the floor is ten times what
    # the device episode itself makes of a relative change of x_init at the element type's resolution
    e2 = receding_horizon(ctrl, x0 * (1 + torch.finfo(dtype).eps), cost, dx, steps)
    tol = 1e-12 if dtype == F64 else 1e-4
    sc = max(1.0, float(eh.x.abs().max()))
    assert maxdiff(ep.x, eh.x) < tol * sc, maxdiff(ep.x, eh.x)
    assert maxdiff(ep.u, eh.u) < max(tol * sc, 10 * maxdiff(ep.u, e2.u)), (maxdiff(ep.u, eh.u), maxdiff(ep.u, e2.u))
    sc_c = max(1.0, float(eh.costs.abs().max()))
    assert maxdiff(ep.costs, eh.costs) < max(tol * sc_c, 10 * maxdiff(ep.costs, e2.costs))


def _grad_case(kind, dtype, bound="scalar"):
    n, m = (3, 1) if kind != "none2" else (3, 2)
    T, B, steps = 6, 4, 4
    dx = _net(n, m, [12, 10] if kind == "none2" else [16], "sigmoid", True, dtype)
    x0, C, c = _problem(n, m, T, B, dtype)
    plant = w = None
    if kind == "w":
        w = _w(steps, B, n, dtype)
    elif kind == "lindx":
        plant, w = _lindx_plant(n, m, B, dtype), _w(steps, B, n, dtype)
    elif kind == "pendulum":
        plant, w = _pendulum(dtype), _w(steps, B, n, dtype)
    return dx, x0, C, c, plant, w, _ctrl(n, m, T, bound), steps


def _leaves(dx, x0, C, c, plant, w):
    """Fresh leaves of every differentiable input and the loss weights; returns (run, leaves)."""
    lv = {"x0": x0.clone().requires_grad_(), "C": C.clone().requires_grad_(), "c": c.clone().requires_grad_()}
    for i, fc in enumerate(dx.fcs):
        fc.weight.requires_grad_(True)
        fc.bias.requires_grad_(True)
        lv[f"W{i}"], lv[f"b{i}"] = fc.weight, fc.bias
    p = plant
    if isinstance(plant, LinDx):
        lv["Fp"], lv["fp"] = plant.F.clone().requires_grad_(), plant.f.clone().requires_grad_()
        p = LinDx(lv["Fp"], lv["fp"])
    elif plant is not None:
        lv["params"] = plant.params.detach().clone().requires_grad_()
        p = PendulumDx(params=lv["params"])
    if w is not None:
        lv["w"] = w.clone().requires_grad_()
    return lv, p


def _grads(ctrl, dx, steps, lv, p, seed=5):
    for t in lv.values():
        t.grad = None
    ep = receding_horizon(ctrl, lv["x0"], QuadCost(lv["C"], lv["c"]), dx, steps, differentiable=True, plant=p,
                          disturbance=lv.get("w"))
    g = torch.Generator().manual_seed(seed)
    wx = torch.randn(ep.x.shape, generator=g, dtype=F64).to(ep.x)
    wu = torch.randn(ep.u.shape, generator=g, dtype=F64).to(ep.u)
    ((ep.x * wx).sum() + (ep.u * wu).sum()).backward()
    return ep, {k: t.grad.clone() for k, t in lv.items()}


@pytest.mark.parametrize("dtype", [F64, F32])
@pytest.mark.parametrize("kind", ["none", "none2", "w", "lindx", "pendulum"])
def test_gradients_match_the_host_path(kind, dtype, monkeypatch):
    dx, x0, C, c, plant, w, ctrl, steps = _grad_case(kind, dtype)
    lv, p = _leaves(dx, x0, C, c, plant, w)
    assert mlpmod.episode_on_device(ctrl, x0, QuadCost(C, c), dx, control._first_warm_start(ctrl, x0),
                                    p if p is not None else (dx if w is not None else None), differentiable=True)
    ep, gd = _grads(ctrl, dx, steps, lv, p)
    assert type(ep.x.grad_fn).__name__.startswith("NetEpisodeFn")
    _, gh = _host(monkeypatch, lambda: _grads(ctrl, dx, steps, lv, p))
    tol = 1e-11 if dtype == F64 else 2e-3
    for k in gh:
        sc = max(1e-30, float(gh[k].abs().max()))
        assert maxdiff(gd[k], gh[k]) <= tol * sc, (k, maxdiff(gd[k], gh[k]), sc)


def test_gradients_match_central_differences():
    """A small unbounded float64 episode whose solves run to convergence and keep their last iterate
    (best_cost_eps 0): the loss's gradient in x_init, c and one entry of each weight and bias against central
    differences of the device forward.  The network has one layer, so the model is affine, each solve is the LQR
    problem of its linearisation and MPC.forward's differentiable tail (which, as the reference's, leaves out the
    dynamics' second derivatives) is the exact derivative of the loop.  (A hidden layer's curvature, or a relu
    network's kinks, on which the solves' optima tend to settle, make the tail differ from the loop's derivative.)"""
    _, x0, C, c, plant, w, _, steps = _grad_case("none", F64, None)
    dx = _net(3, 1, [], "sigmoid", True, F64)
    ctrl = _ctrl(3, 1, 6, None, lqr_iter=100, eps=1e-12, not_improved_lim=100, best_cost_eps=0.0)
    lv, p = _leaves(dx, x0, C, c, plant, w)
    _, gd = _grads(ctrl, dx, steps, lv, p)
    gen = torch.Generator().manual_seed(5)
    ex = receding_horizon(ctrl, x0, QuadCost(C, c), dx, steps)
    wx = torch.randn(ex.x.shape, generator=gen, dtype=F64).to(DEV)
    wu = torch.randn(ex.u.shape, generator=gen, dtype=F64).to(DEV)

    def loss():
        with torch.no_grad():
            e = receding_horizon(ctrl, lv["x0"], QuadCost(lv["C"], lv["c"]), dx, steps)
        return float((e.x * wx).sum() + (e.u * wu).sum())
    h = 1e-6
    for k, idx in (("x0", (1, 0)), ("c", (2, 1, 3)), ("W0", (2, 3)), ("W0", (0, 1)), ("b0", (1,))):
        t = lv[k]
        with torch.no_grad():
            t[idx] += h
        up = loss()
        with torch.no_grad():
            t[idx] -= 2 * h
        dn = loss()
        with torch.no_grad():
            t[idx] += h
        fd = (up - dn) / (2 * h)
        assert abs(fd - float(gd[k][idx])) < 1e-6 * max(1.0, abs(fd)), (k, fd, float(gd[k][idx]))


def test_dtheta_is_bitwise_repeatable_and_captures():
    dx, x0, C, c, plant, w, ctrl, steps = _grad_case("w", F64)
    n, m, T = 3, 1, ctrl.T
    w0 = control._first_warm_start(ctrl, x0)
    with torch.no_grad(), params_scope():
        res = mlpmod.episode_raw(dx, n, m, T, steps, x0, C, c, w0, w=w, keep_plans=True, **ctrl._device_options())
        gx = torch.randn(steps + 1, x0.shape[0], n, dtype=F64, device=DEV)
        gu = torch.randn(steps, x0.shape[0], m, dtype=F64, device=DEV)
        with poisoned():
            a = mlpmod.episode_backward_raw(res["saved"], gx, gu)
            b = mlpmod.episode_backward_raw(res["saved"], gx, gu)
        s = torch.cuda.Stream()
        graph = torch.cuda.CUDAGraph()
        torch.cuda.synchronize()
        with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
            g_ = mlpmod.episode_backward_raw(res["saved"], gx, gu)
        graph.replay()
        graph.replay()
        torch.cuda.synchronize()
    for u, v, z in zip(a, b, g_):
        if u is not None:
            assert torch.equal(u, v) and torch.equal(u, z)


def test_batch_independence():
    """A problem's episode and gradients are bitwise the same alone and at another position of a batch."""
    dx, x0, C, c, plant, w, ctrl, steps = _grad_case("none", F64)
    ctrl = _ctrl(3, 1, 6, "scalar", eps=0.0, not_improved_lim=100)      # every solve runs all its iterations
    perm = torch.tensor([2, 0, 3, 1], device=DEV)
    full = _device(ctrl, x0, QuadCost(C, c), dx, steps)[0]
    for b in range(4):
        one = _device(ctrl, x0[b:b + 1], QuadCost(C[:, b:b + 1], c[:, b:b + 1]), dx, steps)[0]
        assert torch.equal(one["x"], full["x"][:, b:b + 1]) and torch.equal(one["u"], full["u"][:, b:b + 1])
    pm = _device(ctrl, x0[perm], QuadCost(C[:, perm], c[:, perm]), dx, steps)[0]
    assert torch.equal(pm["x"], full["x"][:, perm])
    gx = torch.randn(steps + 1, 4, 3, dtype=F64, device=DEV)
    gu = torch.randn(steps, 4, 1, dtype=F64, device=DEV)
    ga = mlpmod.episode_backward_raw(full["saved"], gx, gu)
    gp = mlpmod.episode_backward_raw(pm["saved"], gx[:, perm], gu[:, perm])
    assert torch.equal(gp[0], ga[0][perm]) and torch.equal(gp[1], ga[1][:, perm])


def test_in_place_weight_edit_raises_and_backward_reads_nothing():
    dx, x0, C, c, plant, w, ctrl, steps = _grad_case("none", F64)
    lv, p = _leaves(dx, x0, C, c, plant, w)
    ep = receding_horizon(ctrl, lv["x0"], QuadCost(lv["C"], lv["c"]), dx, steps, differentiable=True)
    with torch.no_grad():
        dx.fcs[0].weight.add_(0.0)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        ep.x.sum().backward()
    ep = receding_horizon(ctrl, lv["x0"], QuadCost(lv["C"], lv["c"]), dx, steps, differentiable=True)
    loss = ep.x.sum() + ep.u.sum()
    torch.cuda.synchronize()
    try:
        torch.cuda.set_sync_debug_mode("error")         # any host read (item, a device-to-host copy) raises
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert dx.fcs[0].weight.grad is not None and lv["x0"].grad is not None


def test_episode_is_freed_without_cyclic_gc():
    import gc
    import weakref
    dx, x0, C, c, plant, w, ctrl, steps = _grad_case("none", F64)
    lv, p = _leaves(dx, x0, C, c, plant, w)
    gc.disable()
    try:
        ep = receding_horizon(ctrl, lv["x0"], QuadCost(lv["C"], lv["c"]), dx, steps, differentiable=True)
        ref = weakref.ref(ep.x)
        del ep
        assert ref() is None
    finally:
        gc.enable()


def test_no_conditional_graph_falls_back_to_the_host_path(monkeypatch):
    dx, x0, C, c, plant, w, ctrl, steps = _grad_case("none", F64)
    monkeypatch.setattr(solver, "_graph_cond_unavailable", False)
    real = _lib.entry

    def refuse(name, dtype):
        if name == "mpcb200_episode_mlp":
            return lambda *a: _lib.ERR_NO_GRAPH_COND
        return real(name, dtype)
    monkeypatch.setattr(_lib, "entry", refuse)
    host = []
    monkeypatch.setattr(control, "_episode_host", lambda *a, **k: host.append(1) or "host")
    assert receding_horizon(ctrl, x0, QuadCost(C, c), dx, steps) == "host"
    assert host and solver._graph_cond_unavailable


@pytest.mark.parametrize("case", ["net", "pendulum"])
def test_device_episode_matches_the_reference_fixture(case):
    """tests/golden/receding_nn_f64.npz end to end: x, u and the gradients of sum(wx * x) + sum(wu * u) to x_init, C, c,
    w, every weight and bias (and the pendulum plant's params), to the reference's batched pnqp stopping rule (|dx| <
    1e-4 on these bounded solves): 2e-4 of max|x| on the trajectories, 2e-3 of max|g| on the gradients."""
    import os
    import numpy as np
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "receding_nn_f64.npz"))
    t = {k[len(case) + 1:]: torch.from_numpy(z[k]).to(DEV) for k in z.files if k.startswith(case + "_")}
    nl = int(t["n_layers"])
    n, m = t["x_init"].shape[1], t["u"].shape[2]
    T, steps, bound = int(t["T"]), int(t["n_steps"]), float(t["bound"])
    dx = NNDynamics(n, m, hidden_sizes=[t[f"W{i}"].shape[0] for i in range(nl - 1)]).to(dtype=F64, device=DEV)
    with torch.no_grad():
        for i, fc in enumerate(dx.fcs):
            fc.weight.copy_(t[f"W{i}"])
            fc.bias.copy_(t[f"b{i}"])
    ctrl = MPC(n, m, T, u_lower=-bound, u_upper=bound, lqr_iter=int(t["lqr_iter"]), eps=float(t["eps"]), verbose=-1,
               grad_method=GradMethods.ANALYTIC, exit_unconverged=False, detach_unconverged=False)
    plant = None
    if case == "pendulum":
        plant = PendulumDx(params=t["params"].clone())
        plant.max_torque = bound
    lv, p = _leaves(dx, t["x_init"], t["C"], t["c"], plant, t["w"])
    for k in lv:
        lv[k].grad = None
    ep = receding_horizon(ctrl, lv["x0"], QuadCost(lv["C"], lv["c"]), dx, steps, differentiable=True, plant=p,
                          disturbance=lv["w"])
    assert type(ep.x.grad_fn).__name__.startswith("NetEpisodeFn")
    ((ep.x * t["wx"]).sum() + (ep.u * t["wu"]).sum()).backward()
    tx, tg = 2e-4, 2e-3
    sc = max(1.0, float(t["x"].abs().max()))
    assert maxdiff(ep.x, t["x"]) < tx * sc and maxdiff(ep.u, t["u"]) < tx * sc
    names = {"x0": "x_init", "C": "C", "c": "c", "w": "w", "params": "params"}
    for k, v in lv.items():
        want = t["g_" + names.get(k, k)]
        assert maxdiff(v.grad, want) < tg * max(1.0, float(want.abs().max())), (k, maxdiff(v.grad, want))
