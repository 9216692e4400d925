"""GPU: receding-horizon episodes closed on a plant other than the model, x_{k+1} = plant(x_k, u_k) + w_k.  The
device path (mpcb200_episode_plant_*, then one mpcb200_episode_backward_plant_* call) is taken exactly where the plant
steps at the staged shape; its forward is bitwise the host path's and its gradients match the host path's autograd
loop (f64 <= 1e-10 of max|g|, f32 by `within`) for LinDx and known plants, known and LinDx models, with and without
w, bounds and a slew-rate penalty.  A separate plant equal to the model with w = 0 gives today's episode bitwise and
gradients that sum to today's; finite differences in w, the plant's F and the model's F agree; the backward makes no
host read, can be captured, keeps batch problems independent, refuses in-place edits and is first order only."""
import pytest
import torch

from mpc.pytorch_b200 import _lib, control, step
from mpc.pytorch_b200.control import receding_horizon
from mpc.pytorch_b200.dynamics import CartpoleDx, PendulumDx
from mpc.pytorch_b200.solver import LinDx
from tests.gpu_harness import DEV, F32, F64, maxdiff
from tests.test_receding_grad_gpu import _cast, check_grads, known_case, linear_case, loss_weights

pytestmark = pytest.mark.gpu

B, T, STEPS = 6, 8, 4
SLEW = 0.1
_ran_on_device = set()              # (plant form, slew, w) combinations the device path ran (test_zz_coverage)

SYSTEMS = {"pendulum": (lambda p: PendulumDx(params=p), (10.0, 1.0, 1.0)),
           "pendulum_full": (lambda p: PendulumDx(params=p, simple=False), (10.0, 1.0, 1.0, 0.3, 0.2)),
           "cartpole": (lambda p: CartpoleDx(params=p), (9.8, 1.2, 0.12, 0.55)),
           "pendulum_simple_other": (lambda p: PendulumDx(params=p), (9.0, 1.1, 0.9))}


class PCase:
    """A model case (tests.test_receding_grad_gpu.Case) with a plant and, optionally, a disturbance w."""

    def __init__(self, base, plant_leaves, make_plant, form, slew, with_w, n, dtype, ref32, seed=11):
        self.base, self.make_plant, self.form, self.slew, self.with_w = base, make_plant, form, slew, with_w
        self.steps = base.steps
        cast = _cast(dtype, ref32)
        g = torch.Generator().manual_seed(seed)
        self.extra = {k: cast(v) for k, v in plant_leaves.items()}
        if with_w:
            self.extra["w"] = cast(0.02 * torch.randn(base.steps, B, n, generator=g, dtype=F64))

    def ctrl(self):
        c = self.base.ctrl()
        if self.slew:
            c.slew_rate_penalty = SLEW
        return c

    def leaves(self):
        lv = self.base.leaves()
        lv.update({k: v.clone().to(DEV).requires_grad_(True) for k, v in self.extra.items()})
        return lv

    def problem(self, lv):
        x0, cost, dx = self.base.problem(lv)
        return x0, cost, dx, self.make_plant(lv), lv.get("w")


def _lin_plant_from(F, f, seed):
    """A perturbed copy of a LinDx model's F, f: the plant the controller's model approximates."""
    g = torch.Generator().manual_seed(seed)
    return {"Fp": F * (1 + 0.05 * torch.randn(F.shape, generator=g, dtype=F64)),
            "fp": f + 0.01 * torch.randn(f.shape, generator=g, dtype=F64)}


def make(name, dtype, slew=False, with_w=False, ref32=False):
    """name = "<model>/<plant>[/<bounds>]"."""
    model, plant = name.split("/")[:2]
    bounds = name.split("/")[2] if name.count("/") == 2 else "none"
    if model.startswith("lin"):
        n, m = {"lin42": (4, 2), "lin52": (5, 2), "lin182": (18, 2), "lin31": (3, 1), "lin51": (5, 1)}[model]
        base = linear_case(B, T, n, m, dtype, bounds=bounds, steps=STEPS, seed=2, ref32=ref32)
        raw = base.leaves()
        F, f = raw["F"].detach().double().cpu(), raw["f"].detach().double().cpu()
    else:
        base = known_case(model, B, T, dtype, steps=STEPS, ref32=ref32, lqr_iter=10)
        n, m = SYSTEMS[model][0](torch.tensor(SYSTEMS[model][1])).n_state, 1
    if plant == "lin":
        if model.startswith("lin"):
            pl = _lin_plant_from(F, f, 7)
        else:                                   # a linear plant for a known model: one slice, a stable map
            g = torch.Generator().manual_seed(8)
            Fp = torch.cat((0.97 * torch.eye(n, dtype=F64) + 0.02 * torch.randn(n, n, generator=g, dtype=F64),
                            0.05 * torch.randn(n, m, generator=g, dtype=F64)), 1)
            pl = {"Fp": Fp.expand(1, B, n, n + m).clone(), "fp": 0.01 * torch.randn(1, B, n, generator=g, dtype=F64)}
        form = "lin"

        def mk(lv):
            return LinDx(lv["Fp"], lv["fp"])
    else:
        ctor, vals = SYSTEMS[plant]
        pl = {"pparams": torch.tensor(vals, dtype=F64)}
        form = "known"

        def mk(lv):
            return ctor(lv["pparams"])
    return PCase(base, pl, mk, form, slew, with_w, n, dtype, ref32)


def run(monkeypatch, pc, path, lv=None):
    """receding_horizon(differentiable=True) on `path` ("device": one plant backward call; "host"), then the fixed
    linear loss backward.  Returns (episode, {leaf: grad})."""
    lv = pc.leaves() if lv is None else lv
    x0, cost, dx, plant, w = pc.problem(lv)
    calls = []
    with monkeypatch.context() as mp:
        if path == "device":
            real = step.episode_backward_raw

            def spy(saved, *a):
                calls.append(saved)
                return real(saved, *a)
            mp.setattr(step, "episode_backward_raw", spy)
        else:
            mp.setattr(control, "_episode_device_grad", lambda *a: None)
        ep = receding_horizon(pc.ctrl(), x0, cost, dx, pc.steps, differentiable=True, plant=plant, disturbance=w)
        wx, wu = loss_weights(pc.steps, x0.shape[0], ep.x.shape[2], ep.u.shape[2], ep.x.dtype)
        ((wx * ep.x).sum() + (wu * ep.u).sum()).backward()
    torch.cuda.synchronize()
    if path == "device":
        assert len(calls) == 1 and calls[0][0].plant is not None, "not the plant sweep"
        _ran_on_device.add((pc.form, pc.slew, pc.with_w))
    else:
        assert not calls
    return ep, {k: v.grad for k, v in lv.items()}


DEVICE_CASES = ["lin42/lin", "lin52/lin", "lin182/lin", "lin42/lin/scalar", "lin42/lin/tensor_delta",
                "pendulum/pendulum_full", "pendulum_full/pendulum_simple_other", "cartpole/cartpole", "pendulum/lin",
                "cartpole/lin", "lin31/pendulum", "lin51/cartpole", "lin31/pendulum_full"]
# (6, 1) LinDx (lin51 under a slew-rate penalty) pads to the (6, 2) instance: a known plant cannot step there
HOST_ONLY = {("lin51/cartpole", True)}


@pytest.mark.parametrize("with_w", [False, True])
@pytest.mark.parametrize("slew", [False, True])
@pytest.mark.parametrize("name", DEVICE_CASES)
def test_device_against_host_f64(monkeypatch, name, slew, with_w):
    pc = make(name, F64, slew, with_w)
    if (name, slew) in HOST_ONLY:
        lv = pc.leaves()
        x0, cost, dx, plant, w = pc.problem(lv)
        assert not control._plant_on_device(pc.ctrl(), x0, dx, plant)
        seen = []
        real = step.episode_raw
        monkeypatch.setattr(step, "episode_raw", lambda *a, **k: seen.append(1) or real(*a, **k))
        ep = receding_horizon(pc.ctrl(), x0, cost, dx, STEPS, differentiable=True, plant=plant, disturbance=w)
        (ep.x.sum() + ep.u.sum()).backward()
        assert not seen and all(bool(torch.isfinite(v.grad).all()) for v in lv.values())
        # against the float64 plant oracle's episode and sweep (the previous control and the warm starts held
        # constant, as the gradient defines them, which finite differences of the loop would not do)
        from oracle import plant_oracle as porc
        c = {k: v.detach().cpu() for k, v in lv.items()}
        ctrl = pc.ctrl()
        pl = ("step", _oracle_steps(name)[1], c["pparams"].expand(B, -1))
        args = (5, 1, T, c["C"], c["c"], c["F"], c["f"])
        ep_o = porc.receding_horizon_lin(5, 1, T, STEPS, c["x0"], c["C"], c["c"], c["F"], c["f"], plant=pl,
                                         w=c.get("w"), slew_rate_penalty=SLEW, lqr_iter=ctrl.lqr_iter, eps=ctrl.eps,
                                         coupled=False)
        assert maxdiff(ep.x.detach().cpu(), ep_o.x) <= 1e-9 * max(1.0, float(ep_o.x.abs().max()))
        want = porc.receding_horizon_backward(*args, ep_o.x, ep_o.u, ep_o.plan_x, ep_o.plan_u,
                                              torch.ones_like(ep_o.x), torch.ones_like(ep_o.u),
                                              slew_rate_penalty=SLEW, plant=pl)
        for key, w_ in (("x0", want["dx_init"]), ("C", want["dC"]), ("c", want["dc"]), ("F", want["dF"]),
                        ("f", want["df"]), ("pparams", want["dtheta_plant"].sum(0))) + \
                (("w", want["dw"]),) * with_w:
            err = maxdiff(lv[key].grad.cpu(), w_) / max(1.0, float(w_.abs().max()))
            assert err <= 1e-8, (key, err)
        return
    ep_d, g_d = run(monkeypatch, pc, "device")
    ep_h, g_h = run(monkeypatch, pc, "host")
    assert torch.equal(ep_d.x.detach(), ep_h.x.detach()) and torch.equal(ep_d.u.detach(), ep_h.u.detach())
    assert torch.equal(ep_d.costs, ep_h.costs)
    check_grads(f"{name} slew={slew} w={with_w} f64", g_d, g_h, F64)


@pytest.mark.parametrize("name,slew", [("lin42/lin", False), ("lin52/lin", True), ("pendulum/pendulum_full", False),
                                       ("lin31/pendulum", True), ("cartpole/lin", False)])
def test_device_against_host_f32(monkeypatch, name, slew):
    pc = make(name, F32, slew, True)
    ep_d, g_d = run(monkeypatch, pc, "device")
    ep_h, g_h = run(monkeypatch, pc, "host")
    assert torch.equal(ep_d.x.detach(), ep_h.x.detach()) and torch.equal(ep_d.u.detach(), ep_h.u.detach())
    _, g64 = run(monkeypatch, make(name, F64, slew, True, ref32=True), "host")
    check_grads(f"{name} slew={slew} f32", g_d, g_h, F32, w32=g_h, w64=g64)


def test_module_plant_takes_the_host_path(monkeypatch):
    """An opaque Module plant runs the host loop; its forward is the Module's own step plus w."""
    pc = make("lin42/lin", F64, with_w=True)
    lv = pc.leaves()
    x0, cost, dx, plant, w = pc.problem(lv)

    class Opaque(torch.nn.Module):
        def forward(self, x, u):
            return torch.einsum("bij,bj->bi", lv["Fp"][0], torch.cat((x, u), 1)) + lv["fp"][0]
    called = []
    monkeypatch.setattr(step, "episode_raw", lambda *a, **k: called.append(1))
    ep = receding_horizon(pc.ctrl(), x0, cost, dx, STEPS, differentiable=True, plant=Opaque(), disturbance=w)
    assert not called
    ep.x.sum().backward()
    assert lv["Fp"].grad is not None and lv["w"].grad is not None and lv["F"].grad is not None
    monkeypatch.undo()
    with torch.no_grad():
        ep_l = receding_horizon(pc.ctrl(), x0, cost, dx, STEPS, plant=LinDx(lv["Fp"], lv["fp"]), disturbance=w)
    assert maxdiff(ep.x.detach(), ep_l.x) <= 1e-12


@pytest.mark.parametrize("slew", [False, True])
@pytest.mark.parametrize("name", ["lin42", "lin52", "pendulum", "cartpole", "pendulum_full"])
def test_plant_equal_to_model_is_todays_episode(monkeypatch, name, slew):
    """A separate plant object equal to the model, with w = 0: today's x, u, costs, dx_init, dC and dc bitwise; the
    model's and the plant's parameter gradients sum to today's."""
    if name.startswith("lin"):
        base = linear_case(B, T, *{"lin42": (4, 2), "lin52": (5, 2)}[name], F64, steps=STEPS, seed=2)
    else:
        base = known_case(name, B, T, F64, steps=STEPS, lqr_iter=10)

    def ctrl():
        c = base.ctrl()
        c.slew_rate_penalty = SLEW if slew else None
        return c
    lv0 = base.leaves()
    x0, cost, dx = base.problem(lv0)
    ep0 = receding_horizon(ctrl(), x0, cost, dx, STEPS, differentiable=True)
    wx, wu = loss_weights(STEPS, B, ep0.x.shape[2], ep0.u.shape[2], F64)
    ((wx * ep0.x).sum() + (wu * ep0.u).sum()).backward()

    lv = base.leaves()
    x0, cost, dx = base.problem(lv)
    if isinstance(dx, LinDx):
        pF, pf = dx.F.detach().clone().requires_grad_(True), dx.f.detach().clone().requires_grad_(True)
        plant, ptensors = LinDx(pF, pf), {"F": pF, "f": pf}
    else:
        pp = dx.params.detach().clone().requires_grad_(True)
        plant, ptensors = type(dx)(params=pp, **({} if isinstance(dx, CartpoleDx) else {"simple": dx.simple})), \
            {"params": pp}
    w = torch.zeros(STEPS, B, x0.shape[1], dtype=F64, device=DEV, requires_grad=True)
    calls = []
    real = step.episode_backward_raw
    monkeypatch.setattr(step, "episode_backward_raw", lambda s, *a: calls.append(s) or real(s, *a))
    ep = receding_horizon(ctrl(), x0, cost, dx, STEPS, differentiable=True, plant=plant, disturbance=w)
    ((wx * ep.x).sum() + (wu * ep.u).sum()).backward()
    assert len(calls) == 1 and calls[0][0].plant is not None
    for a, b in ((ep.x, ep0.x), (ep.u, ep0.u), (ep.costs, ep0.costs)):
        assert torch.equal(a.detach(), b.detach())
    for k in ("x0", "C", "c"):
        assert torch.equal(lv[k].grad, lv0[k].grad), k
    worst = 0.0
    for k, t in ptensors.items():
        got, want = lv[k].grad + t.grad, lv0[k].grad
        scale = max(1e-300, float(want.abs().max()))
        worst = max(worst, maxdiff(got, want) / scale)
        assert maxdiff(got, want) <= 1e-12 * scale, k
    print(f"{name} slew={slew}: model + plant vs today's parameter gradient, max rel {worst:.2e}")
    assert torch.allclose(w.grad[-1], wx[-1])                     # dL/dx_{n_steps} is the loss weight alone


def test_disturbance_gradient_is_next_state_gradient(monkeypatch):
    """dL/dw_k = dL/dx_{k+1}: with a loss on x[k+1] alone, w's gradient at k is that loss's weight and the earlier
    ones are what flows back through the closed loop; x_init's gradient is then dL/dw_{-1} of the same sweep."""
    pc = make("lin42/lin", F64, with_w=True)
    lv = pc.leaves()
    x0, cost, dx, plant, w = pc.problem(lv)
    ep = receding_horizon(pc.ctrl(), x0, cost, dx, STEPS, differentiable=True, plant=plant, disturbance=w)
    gx = torch.zeros_like(ep.x)
    gx[2] = 1.0
    ep.x.backward(gx)
    assert torch.equal(lv["w"].grad[1], gx[2]) and bool((lv["w"].grad[2:] == 0).all())
    assert bool((lv["w"].grad[0] != 0).any())


# ------------------------------------------------------------------------------------------------------------------
def test_finite_differences_unbounded_linear():
    pc = make("lin42/lin", F64, with_w=True)
    lv = pc.leaves()
    x0, cost, dx, plant, w = pc.problem(lv)
    ep = receding_horizon(pc.ctrl(), x0, cost, dx, STEPS, differentiable=True, plant=plant, disturbance=w)
    wx, wu = loss_weights(STEPS, B, 4, 2, F64)
    ((wx * ep.x).sum() + (wu * ep.u).sum()).backward()
    base = {k: v.detach() for k, v in pc.leaves().items()}

    def loss(vals):
        with torch.no_grad():
            x0, cost, dx, plant, w = pc.problem(vals)
            e = receding_horizon(pc.ctrl(), x0, cost, dx, STEPS, plant=plant, disturbance=w)
        return float((wx * e.x).sum() + (wu * e.u).sum())
    h = 1e-6
    for name, idx in (("w", (0, 1, 2)), ("w", (2, 4, 0)), ("Fp", (0, 2, 1, 3)), ("Fp", (0, 0, 3, 5)),
                      ("fp", (0, 3, 1)), ("F", (0, 2, 1, 3)), ("F", (3, 0, 2, 0)), ("x0", (1, 2))):
        plus = {k: v.clone() for k, v in base.items()}
        minus = {k: v.clone() for k, v in base.items()}
        plus[name][idx] += h
        minus[name][idx] -= h
        fd = (loss(plus) - loss(minus)) / (2 * h)
        got = float(lv[name].grad[idx])
        assert abs(fd - got) <= 1e-6 * max(1.0, abs(fd)), (name, idx, fd, got)
    assert bool((lv["Fp"].grad[1:] == 0).all())                   # the plant steps with its slice 0 only


@pytest.mark.parametrize("name", ["lin42/lin", "pendulum/pendulum_full"])
def test_backward_no_host_read(monkeypatch, name):
    pc = make(name, F32, with_w=True)
    run(monkeypatch, pc, "device")                                 # library load, kernel set-up
    lv = pc.leaves()
    x0, cost, dx, plant, w = pc.problem(lv)
    ep = receding_horizon(pc.ctrl(), x0, cost, dx, STEPS, differentiable=True, plant=plant, disturbance=w)
    loss = ep.x.sum() + ep.u.sum()
    torch.cuda.synchronize()
    before = _lib.launch_count()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert _lib.launch_count() > before
    assert all(v.grad is not None and bool(torch.isfinite(v.grad).all()) for v in lv.values())


def test_pinned_plant_params_no_host_read(monkeypatch):
    """A known plant with pinned CPU parameters on a LinDx model: the whole episode, forward and backward, makes no
    host read (the parameters are read on the host, once, without a device synchronise)."""
    pc = make("lin31/pendulum_full", F32, with_w=True)
    run(monkeypatch, pc, "device")
    lv = pc.leaves()
    lv["pparams"] = lv["pparams"].detach().cpu().pin_memory()
    x0, cost, dx, plant, w = pc.problem(lv)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        ep = receding_horizon(pc.ctrl(), x0, cost, dx, STEPS, differentiable=True, plant=plant, disturbance=w)
        (ep.x.sum() + ep.u.sum()).backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert lv["w"].grad is not None and lv["F"].grad is not None


def _raw(pc, dtype=F32):
    """The plant episode's raw forward with plans (what EpisodeFn runs), on detached leaves."""
    lv = {k: v.detach() for k, v in pc.leaves().items()}
    x0, cost, dx, plant, w = pc.problem(lv)
    ctrl = pc.ctrl()
    n, x0_, C, c, F, f, dyn = ctrl._device_problem(x0, cost, dx)
    w0 = control._first_warm_start(ctrl, x0)
    Fp, fp = (plant.F, plant.f) if isinstance(plant, LinDx) else (None, None)
    with torch.no_grad():
        spec = control._plant_spec(ctrl, x0, cost.C, plant, Fp, fp)
    res = step.episode_raw(n, ctrl.n_ctrl, ctrl.T, pc.steps, x0_, C, c, F, f, w0, dyn=dyn, keep_plans=True,
                           n_prev=ctrl.n_ctrl if pc.slew else 0, plant=spec, w=control._staged_w(ctrl, w),
                           **ctrl._device_options())
    return res, n, ctrl.n_ctrl


@pytest.mark.parametrize("name", ["lin42/lin", "cartpole/cartpole"])
def test_backward_captured_in_caller_graph(name):
    pc = make(name, F32, with_w=True)
    res, n, m = _raw(pc)
    wx, wu = loss_weights(pc.steps, B, n, m, F32)
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
        assert len(out) == 10
        for a, b in zip(out, want):
            assert (a is None) == (b is None) and (a is None or torch.equal(a, b))


@pytest.mark.parametrize("name", ["lin42/lin", "pendulum/lin", "lin31/pendulum"])
def test_batch_independence(name):
    """Problem 0's episode and gradients do not depend on the other problems: with a fixed iteration count (the stop
    test mixes the batch), a batch whose other problems start elsewhere and see other disturbances gives problem 0
    bitwise the same results."""
    pc = make(name, F64, with_w=True)
    base_ctrl = pc.ctrl

    def fixed():
        c = base_ctrl()
        c.lqr_iter, c.eps, c.not_improved_lim = 4, 0.0, 1000
        return c
    pc.ctrl = fixed
    outs = []
    for perturb in (False, True):
        lv = pc.leaves()
        if perturb:
            with torch.no_grad():
                lv["x0"][1:] *= 1.01
                lv["w"][:, 1:] *= 1.5
        x0, cost, dx, plant, w = pc.problem(lv)
        ep = receding_horizon(pc.ctrl(), x0, cost, dx, STEPS, differentiable=True, plant=plant, disturbance=w)
        (ep.x[:, 0].sum() + ep.u[:, 0].sum()).backward()
        outs.append((ep, lv))
    (e0, l0), (e1, l1) = outs
    assert torch.equal(e0.x[:, 0], e1.x[:, 0]) and torch.equal(e0.u[:, 0], e1.u[:, 0])
    assert not torch.equal(e0.x[:, 1], e1.x[:, 1])
    assert torch.equal(l0["w"].grad[:, 0], l1["w"].grad[:, 0]) and torch.equal(l0["x0"].grad[0], l1["x0"].grad[0])


def test_poisoned_workspace_gives_same_gradients():
    """The sweep reads nothing it did not write: a workspace full of 0xFF gives bitwise the clean call's outputs."""
    pc = make("pendulum/pendulum_full", F64, slew=True, with_w=True)
    res, n, m = _raw(pc, F64)
    wx, wu = loss_weights(pc.steps, B, n, m, F64)
    clean = step.episode_backward_raw(res["saved"], wx, wu)
    real_empty = torch.empty

    def poisoned(*a, **k):
        t = real_empty(*a, **k)
        if t.dtype == torch.uint8:
            t.fill_(0xFF)
        return t
    torch.empty = poisoned
    try:
        dirty = step.episode_backward_raw(res["saved"], wx, wu)
    finally:
        torch.empty = real_empty
    torch.cuda.synchronize()
    for a, b in zip(clean, dirty):
        assert (a is None) == (b is None) and (a is None or torch.equal(a, b))


def test_inplace_edit_before_backward_raises():
    pc = make("lin42/lin", F64, with_w=True)
    lv = pc.leaves()
    x0, cost, dx, plant, w = pc.problem(lv)
    ep = receding_horizon(pc.ctrl(), x0, cost, dx, STEPS, differentiable=True, plant=plant, disturbance=w)
    loss = ep.x.sum()
    with torch.no_grad():
        ep.x.mul_(2.0)
    with pytest.raises(RuntimeError):
        loss.backward()


def test_first_order_only():
    pc = make("lin42/lin", F64, with_w=True)
    lv = pc.leaves()
    x0, cost, dx, plant, w = pc.problem(lv)
    ep = receding_horizon(pc.ctrl(), x0, cost, dx, STEPS, differentiable=True, plant=plant, disturbance=w)
    g = torch.autograd.grad(ep.x.sum() + ep.u.sum(), lv["w"], create_graph=True)[0]
    with pytest.raises(RuntimeError):
        g.sum().backward()


def test_forward_without_grad_runs_the_plant_graph(monkeypatch):
    """differentiable=False with a plant: one mpcb200_episode_plant_* graph, bitwise the differentiable forward."""
    pc = make("cartpole/lin", F64, slew=True, with_w=True)
    lv = pc.leaves()
    x0, cost, dx, plant, w = pc.problem(lv)
    seen = []
    real = step.episode_raw
    monkeypatch.setattr(step, "episode_raw", lambda *a, **k: seen.append(k.get("plant")) or real(*a, **k))
    with torch.no_grad():
        ep0 = receding_horizon(pc.ctrl(), x0, cost, dx, STEPS, plant=plant, disturbance=w)
    ep1 = receding_horizon(pc.ctrl(), x0, cost, dx, STEPS, differentiable=True, plant=plant, disturbance=w)
    assert len(seen) == 2 and all(s is not None for s in seen)
    assert torch.equal(ep0.x, ep1.x.detach()) and torch.equal(ep0.u, ep1.u.detach())


def test_zz_coverage():
    """Every plant form x slew-rate penalty x disturbance ran on the device path in this session."""
    want = {(form, slew, ww) for form in ("lin", "known") for slew in (False, True) for ww in (False, True)}
    missing = want - _ran_on_device
    assert not missing, f"never ran on the device: {sorted(missing)}"


# ------------------------------------------------------------------------------------------------------------------
# against the float64 plant oracle and the reference's own loop
# ------------------------------------------------------------------------------------------------------------------
def _oracle_steps(name):
    """The oracle's step(x, u, theta) of the case's model and plant: the project's CPU modules."""
    from tests.gpu_harness import episode_known_step
    model, plant = name.split("/")[:2]
    steps = []
    for sysname in (model, plant):
        if sysname in SYSTEMS:
            ctor, vals = SYSTEMS[sysname]
            steps.append(episode_known_step(ctor(torch.tensor(vals, dtype=F64))))
        else:
            steps.append(None)
    return steps


@pytest.mark.parametrize("slew", [False, True])
@pytest.mark.parametrize("name", ["lin42/lin", "lin52/lin", "lin42/lin/scalar", "pendulum/pendulum_full",
                                  "cartpole/cartpole", "lin31/pendulum", "pendulum/lin"])
def test_sweep_against_plant_oracle(name, slew):
    """The device sweep against the float64 plant oracle run on the device's own plans, states and controls."""
    from oracle import plant_oracle as porc
    pc = make(name, F64, slew, True)
    res, n_aug, m = _raw(pc, F64)
    k = m if slew else 0
    n = n_aug - k
    wx, wu = loss_weights(pc.steps, B, n, m, F64)
    gx = torch.cat((wx.new_zeros(pc.steps + 1, B, k), wx), 2)
    out = step.episode_backward_raw(res["saved"], gx, wu)
    dev = dict(zip(("dx_init", "dC", "dc", "dF", "df", "dtheta", "dF_p", "df_p", "dtheta_plant", "dw"), out))
    s, _, xs, us, plan_x, plan_u = res["saved"]
    lv = {kk: v.detach().cpu() for kk, v in pc.leaves().items()}
    cpu = lambda t: s.pad.crop_n(t).cpu() if t is not None else None           # noqa: E731
    xs_, us_ = cpu(xs)[..., k:], s.pad.crop_m(us).cpu()
    px, pu = cpu(plan_x), s.pad.crop_m(plan_u).cpu()
    ctrl = pc.ctrl()
    lo = hi = None
    if isinstance(ctrl.u_lower, float):
        lo, hi = ctrl.u_lower, ctrl.u_upper
    mstep, pstep = _oracle_steps(name)
    if mstep is None:
        F, f, theta = lv["F"], lv["f"], None
    else:
        F = f = None
        theta = lv["params"].expand(B, -1)
    plant = ("lin", lv["Fp"], lv["fp"]) if pc.form == "lin" else ("step", pstep, lv["pparams"].expand(B, -1))
    want = porc.receding_horizon_backward(n, m, T, lv["C"], lv["c"], F, f, xs_, us_, px, pu, wx.cpu(), wu.cpu(),
                                          u_lower=lo, u_upper=hi, step=mstep, theta=theta,
                                          slew_rate_penalty=SLEW if slew else None, plant=plant)
    worst = {}
    for key in want:
        got = dev[key]
        if got is None:
            assert want[key] is None, key
            continue
        got = got.cpu()
        if k:
            got = {"dx_init": lambda t: t[:, k:], "dC": lambda t: t[..., k:, k:], "dc": lambda t: t[..., k:],
                   "dF": lambda t: t[..., k:, k:], "df": lambda t: t[..., k:], "dF_p": lambda t: t[..., k:, k:],
                   "df_p": lambda t: t[..., k:], "dw": lambda t: t[..., k:]}.get(key, lambda t: t)(got)
        w = want[key]
        if key in ("dF_p", "df_p"):
            w = w[0]
        scale = max(1.0, float(w.abs().max()))
        worst[key] = maxdiff(got, w) / scale
        assert maxdiff(got, w) <= 1e-9 * scale, (key, worst[key])
    print(f"{name} slew={slew} vs plant oracle: " + ", ".join(f"{kk} {v:.1e}" for kk, v in worst.items()))


def test_linear_forward_against_oracle_episode():
    """Unbounded LinDx on a LinDx plant with w: the device episode is the oracle's, to rounding."""
    from oracle import plant_oracle as porc
    pc = make("lin42/lin", F64, with_w=True)
    lv = pc.leaves()
    x0, cost, dx, plant, w = pc.problem(lv)
    with torch.no_grad():
        ep = receding_horizon(pc.ctrl(), x0, cost, dx, STEPS, plant=plant, disturbance=w)
    c = {k: v.detach().cpu() for k, v in lv.items()}
    ctrl = pc.ctrl()
    want = porc.receding_horizon_lin(4, 2, T, STEPS, c["x0"], c["C"], c["c"], c["F"], c["f"],
                                     plant=("lin", c["Fp"], c["fp"]), w=c["w"], lqr_iter=ctrl.lqr_iter,
                                     eps=ctrl.eps)
    assert ep.info[:, 0].cpu().tolist() == want.iters
    for a, b in ((ep.x, want.x), (ep.u, want.u)):
        assert maxdiff(a.cpu(), b) <= 1e-9 * max(1.0, float(b.abs().max()))


@pytest.mark.parametrize("case", ["linear", "pendulum", "cartpole", "pendulum_slew"])
def test_against_reference_fixture(case):
    """The reference's own loop with the plant and + w_k written out (tests/golden/receding_plant_f64.npz), end to
    end through receding_horizon.  The solves bound their controls, so the tolerance is pnqp's own accuracy (2e-4,
    test_receding_grad_gpu's bounded case).  A known model's parameter gradient follows this project's convention
    (the linearisation's Jacobians differentiated) and the reference's does not: it is checked against the plant
    oracle with full_linearisation=True on the fixture's plans instead, which with False reproduces the fixture."""
    import os
    import numpy as np
    from oracle import plant_oracle as porc
    from mpc.pytorch_b200.solver import MPC, QuadCost, GradMethods
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "receding_plant_f64.npz"))
    pre = case + "_"
    t = {k[len(pre):]: torch.from_numpy(z[k]) for k in z.files
         if k.startswith(pre) and not (case == "pendulum" and k.startswith("pendulum_slew_"))}
    T_, steps = int(t["T"]), int(t["n_steps"])
    lv = {k: t[k].clone().to(DEV).requires_grad_(True)
          for k in ("x_init", "C", "c", "w", "F", "f", "F_p", "f_p", "params", "plant_params") if k in t}
    if case == "linear":
        n, m, b = 4, 2, float(t["bound"])
        ctrl = MPC(n, m, T_, u_lower=-b, u_upper=b, lqr_iter=int(t["lqr_iter"]), eps=float(t["eps"]), verbose=-1)
        dx = LinDx(lv["F"], lv["f"])
        plant = LinDx(lv["F_p"].unsqueeze(0), lv["f_p"].unsqueeze(0))
    else:
        sysname = case.split("_")[0]
        clamp = float(t["clamp"])
        if sysname == "cartpole":
            dx, plant = CartpoleDx(params=lv["params"]), CartpoleDx(params=lv["plant_params"])
            dx.force_mag = plant.force_mag = clamp
        else:
            dx, plant = PendulumDx(params=lv["params"]), PendulumDx(params=lv["plant_params"], simple=False)
            dx.max_torque = plant.max_torque = clamp
        n, m = dx.n_state, 1
        ctrl = MPC(n, m, T_, u_lower=-clamp, u_upper=clamp, lqr_iter=int(t["lqr_iter"]), eps=float(t["eps"]),
                   verbose=-1, linesearch_decay=float(t["ls_decay"]), max_linesearch_iter=int(t["ls_iter"]),
                   grad_method=GradMethods.AUTO_DIFF)
        if "slew" in t:
            ctrl.slew_rate_penalty = float(t["slew"])
    calls = []
    real = step.episode_backward_raw
    step.episode_backward_raw = lambda s, *a: calls.append(s) or real(s, *a)
    try:
        ep = receding_horizon(ctrl, lv["x_init"], QuadCost(lv["C"], lv["c"]), dx, steps, differentiable=True,
                              plant=plant, disturbance=lv["w"])
        ((t["wx"].to(DEV) * ep.x).sum() + (t["wu"].to(DEV) * ep.u).sum()).backward()
    finally:
        step.episode_backward_raw = real
    assert len(calls) == 1 and calls[0][0].plant is not None
    errs = {"x": maxdiff(ep.x, t["x"].to(DEV)) / max(1.0, float(t["x"].abs().max())),
            "u": maxdiff(ep.u, t["u"].to(DEV)) / max(1.0, float(t["u"].abs().max()))}
    for k in lv:
        if k == "params":
            continue
        want = t["g_" + k].to(DEV)
        errs["d" + k] = maxdiff(lv[k].grad, want) / max(1.0, float(want.abs().max()))
    if "params" in lv:
        B_ = t["x"].shape[1]
        mstep, pstep = _oracle_steps({"pendulum": "pendulum/pendulum_full", "cartpole": "cartpole/cartpole"}[
            case.split("_")[0]])
        want = porc.receding_horizon_backward(
            n, 1, T_, t["C"], t["c"], None, None, t["x"], t["u"], t["plan_x"], t["plan_u"], t["wx"], t["wu"],
            u_lower=-clamp, u_upper=clamp, step=mstep, theta=t["params"].expand(B_, -1),
            slew_rate_penalty=float(t["slew"]) if "slew" in t else None,
            plant=("step", pstep, t["plant_params"].expand(B_, -1)))["dtheta"].sum(0)
        errs["dparams (oracle, full)"] = maxdiff(lv["params"].grad.cpu(), want) / max(1.0, float(want.abs().max()))
    print(f"{case}: " + ", ".join(f"{k} {v:.2e}" for k, v in errs.items()))
    assert all(v <= 2e-4 for v in errs.values()), errs
