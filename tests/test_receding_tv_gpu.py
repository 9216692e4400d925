"""GPU: receding-horizon episodes on a time-varying cost and LinDx (receding_horizon(..., time_varying=True)).  Each
solve plans on its window of the episode's time axis; the device path (mpcb200_episode_window_*, then one
mpcb200_episode_backward_window_* call) copies each window on the device.  Its forward is bitwise the host path's,
which slices per step in Python; its float64 gradients match the host path's autograd loop to 1e-12 of max|g|.
With n_steps = 1, or inputs constant along the axis, the forward is bitwise the time-invariant episode's, and the
summed gradients match its gradients.  Central finite differences agree; the sweep makes no host read, can be
captured, keeps batch problems independent and is first order only."""
import pytest
import torch

from mpc.pytorch_b200 import step
from mpc.pytorch_b200._lib import MpcB200Error
from mpc.pytorch_b200.control import receding_horizon
from mpc.pytorch_b200.dynamics import CartpoleDx, PendulumDx
from mpc.pytorch_b200.solver import MPC, GradMethods, LinDx, QuadCost
from tests.gpu_harness import DEV, F32, F64, maxdiff
from tests.helpers import gen_problem

pytestmark = pytest.mark.gpu

SLEW = 0.1


class TV:
    """A time-varying episode: leaves {name: float64 CPU tensor} on the axis L = steps + T - 1, ctrl() a fresh MPC
    and problem(lv) -> (x0, cost, dx, plant, w)."""

    def __init__(self, n, m, T, B, steps, base, ctrl, problem):
        self.n, self.m, self.T, self.B, self.steps = n, m, T, B, steps
        self.base, self.ctrl, self.problem = base, ctrl, problem

    def leaves(self, dtype, grad=True):
        return {k: v.to(DEV, dtype).requires_grad_(grad) for k, v in self.base.items()}


def lin_tv(n, m, T, B, steps, bounds="none", slew=False, plant=False, with_w=False, f_full=False, F_full=False,
           seed=0, const=False):
    """A LinDx tracking problem: a target that moves along the axis (c), weights and dynamics that change over it.
    const: every input constant along the axis (one slice, expanded in problem())."""
    L = steps + T - 1
    C, c, F, f, x0 = gen_problem(seed, B, L + 1, n, m, F64, time_varying=True)
    F = 0.9 * F
    C, c, F, f = C[:L], c[:L], F[:L - (0 if F_full else 1)], f[:L - (0 if f_full else 1)]
    g = torch.Generator().manual_seed(seed + 3)
    t = torch.arange(L, dtype=F64)
    target = torch.sin(0.3 * t)[:, None, None] * torch.randn(1, B, n + m, generator=g, dtype=F64)
    c = c - (C @ target.unsqueeze(-1)).squeeze(-1)
    if const:
        C, c, F, f = C[:1], c[:1], F[:1], f[:1]
    base = dict(x0=x0, C=C, c=c, F=F, f=f)
    kw = dict(lqr_iter=8, verbose=-1)
    if bounds == "scalar":
        kw.update(u_lower=-0.3, u_upper=0.3)
    elif bounds == "tensor":
        lo = -0.15 - 0.3 * torch.rand(L, B, m, generator=g, dtype=F64)
        if const:
            lo = lo[:1]
        base.update(lo=lo, hi=-lo + 0.05)
    if plant:
        base.update(Fp=F * (1 + 0.05 * torch.randn(F.shape, generator=g, dtype=F64)),
                    fp=f + 0.01 * torch.randn(f.shape, generator=g, dtype=F64))
    if with_w:
        base["w"] = 0.02 * torch.randn(steps, B, n, generator=g, dtype=F64)
    ex = (lambda v, Lv: v.expand(Lv, *v.shape[1:])) if const else (lambda v, Lv: v)  # noqa: E731

    def ctrl(lv):
        k = dict(kw)
        if "lo" in lv:
            k.update(u_lower=ex(lv["lo"], L), u_upper=ex(lv["hi"], L))
        c_ = MPC(n, m, T, **k)
        if slew:
            c_.slew_rate_penalty = SLEW
        return c_

    def problem(lv):
        LF, Lf = F.shape[0] if not const else L - (0 if F_full else 1), L - (0 if f_full else 1)
        dx = LinDx(ex(lv["F"], LF), ex(lv["f"], Lf))
        pl = LinDx(ex(lv["Fp"], LF), ex(lv["fp"], Lf)) if plant else None
        return lv["x0"], QuadCost(ex(lv["C"], L), ex(lv["c"], L)), dx, pl, lv.get("w")
    return TV(n, m, T, B, steps, base, ctrl, problem)


KNOWN = {"pendulum": (lambda p: PendulumDx(params=p), (10.0, 1.0, 1.0)),
         "cartpole": (lambda p: CartpoleDx(params=p), (9.8, 1.0, 0.1, 0.5))}


def known_tv(name, T, B, steps, slew=False, plant=None, seed=0):
    """A known system tracking a moving reference: the goal angle (pendulum) or cart position (cartpole) moves along
    the axis, so c is time-varying; the clamp binds."""
    ctor, vals = KNOWN[name]
    sysdx = ctor(torch.tensor(vals, dtype=F64))
    n, m = sysdx.n_state, sysdx.n_ctrl
    L = steps + T - 1
    q, p = sysdx.get_true_obj()
    t = torch.arange(L, dtype=F64)
    C = torch.diag(q.double()).expand(L, B, n + m, n + m).clone()
    goal = torch.zeros(L, B, n + m, dtype=F64)
    if name == "pendulum":
        ang = 0.4 * torch.sin(0.2 * t)
        goal[:, :, 0], goal[:, :, 1] = ang.cos()[:, None], ang.sin()[:, None]
    else:
        goal[:, :, 0] = (0.5 * (t > L / 2).double())[:, None]
        goal[:, :, 2] = 1.0
    c = -(C @ goal.unsqueeze(-1)).squeeze(-1) + p.double()
    th = torch.linspace(-1.0, 1.0, B, dtype=F64) + 0.1 * seed
    if name == "pendulum":
        x0 = torch.stack((th.cos(), th.sin(), 0.1 * th), 1)
    else:
        x0 = torch.stack((0.1 * th, 0.05 * th, th.cos(), th.sin(), 0.1 * th), 1)
    base = dict(x0=x0, C=C, c=c, params=torch.tensor(vals, dtype=F64))
    if plant is not None:
        base["pparams"] = torch.tensor(plant, dtype=F64)

    def ctrl(lv):
        c_ = MPC(n, m, T, u_lower=float(sysdx.lower), u_upper=float(sysdx.upper), lqr_iter=10, verbose=-1,
                 linesearch_decay=sysdx.linesearch_decay, max_linesearch_iter=sysdx.max_linesearch_iter,
                 grad_method=GradMethods.AUTO_DIFF, eps=1e-2)
        if slew:
            c_.slew_rate_penalty = SLEW
        return c_

    def problem(lv):
        pl = ctor(lv["pparams"]) if "pparams" in lv else None
        return lv["x0"], QuadCost(lv["C"], lv["c"]), ctor(lv["params"]), pl, None
    return TV(n, m, T, B, steps, base, ctrl, problem)


def run(monkeypatch, case, path, dtype, differentiable=True, lv=None, tv=True):
    """receding_horizon(time_varying=tv) on `path` ("device": asserting the window entries ran; "host"), then a fixed
    linear loss backward when differentiable.  Returns (episode, {leaf: grad})."""
    lv = case.leaves(dtype, grad=differentiable) if lv is None else lv
    x0, cost, dx, plant, w = case.problem(lv)
    ctrl = case.ctrl(lv)
    windows = []
    with monkeypatch.context() as mp:
        if path == "device":
            real = step.episode_raw

            def spy(*a, **k):
                windows.append(k.get("window"))
                return real(*a, **k)
            mp.setattr(step, "episode_raw", spy)
        else:
            mp.setattr("mpc.pytorch_b200.control._takes_device_path", lambda *a, **k: False)
        ep = receding_horizon(ctrl, x0, cost, dx, case.steps, differentiable=differentiable, plant=plant,
                              disturbance=w, time_varying=tv)
        if path == "device":
            assert windows and all((x is not None) == tv for x in windows), windows
        grads = {}
        if differentiable:
            g = torch.Generator().manual_seed(5)
            wx = torch.randn(ep.x.shape, generator=g, dtype=F64).to(DEV, dtype)
            wu = torch.randn(ep.u.shape, generator=g, dtype=F64).to(DEV, dtype)
            ((ep.x * wx).sum() + (ep.u * wu).sum()).backward()
            grads = {k: (v.grad.clone() if v.grad is not None else None) for k, v in lv.items()}
    return ep, grads


def assert_same_forward(a, b, tag):
    for name in ("x", "u", "costs", "info", "u_next"):
        ta, tb = getattr(a, name), getattr(b, name)
        assert ta.shape == tb.shape and torch.equal(ta, tb), f"{tag}: {name} differs by {maxdiff(ta, tb)}"


def assert_close_grads(got, want, tag, tol=1e-12):
    for k, w in want.items():
        if w is None:
            assert got[k] is None or float(got[k].abs().max()) == 0.0, (tag, k)
            continue
        assert got[k] is not None and got[k].shape == w.shape, (tag, k)
        scale = max(1e-300, float(w.abs().max()))
        err = maxdiff(got[k], w)
        assert err <= tol * scale, f"{tag}: d{k} {err:.3e} > {tol * scale:.3e}"


LIN_CASES = {
    "lin42": dict(n=4, m=2),
    "lin42_scalar": dict(n=4, m=2, bounds="scalar"),
    "lin42_tensor": dict(n=4, m=2, bounds="tensor"),
    "lin42_full_Ff": dict(n=4, m=2, F_full=True, f_full=True),
    "lin52_pad_tensor": dict(n=5, m=2, bounds="tensor"),
    "lin52_pad_scalar": dict(n=5, m=2, bounds="scalar"),
    "lin182_large": dict(n=18, m=2, bounds="tensor"),
    "lin42_slew": dict(n=4, m=2, slew=True),
    "lin42_slew_tensor": dict(n=4, m=2, slew=True, bounds="tensor"),
    "lin42_plant": dict(n=4, m=2, plant=True, bounds="tensor"),
    "lin42_plant_w": dict(n=4, m=2, plant=True, with_w=True),
    "lin42_w": dict(n=4, m=2, with_w=True, bounds="scalar"),
    "lin42_plant_w_slew": dict(n=4, m=2, plant=True, with_w=True, slew=True),
    "lin52_pad_plant_w": dict(n=5, m=2, plant=True, with_w=True, bounds="tensor"),
}


@pytest.mark.parametrize("name", sorted(LIN_CASES))
@pytest.mark.parametrize("dtype", [F32, F64])
def test_lin_device_matches_host(monkeypatch, name, dtype):
    case = lin_tv(T=6, B=5, steps=4, **LIN_CASES[name])
    ep_d, g_d = run(monkeypatch, case, "device", dtype)
    ep_h, g_h = run(monkeypatch, case, "host", dtype)
    assert_same_forward(ep_d, ep_h, name)
    if dtype == F64:
        assert_close_grads(g_d, g_h, name)
    else:
        for k, w in g_h.items():
            if w is not None:
                scale = max(1.0, float(w.abs().max()))
                assert maxdiff(g_d[k], w) <= 2e-3 * scale, (name, k)


KNOWN_CASES = {"pendulum": dict(), "cartpole": dict(), "pendulum_slew": dict(slew=True),
               "pendulum_on_pendulum": dict(plant=(9.0, 1.1, 0.9))}


@pytest.mark.parametrize("name", sorted(KNOWN_CASES))
def test_known_device_matches_host(monkeypatch, name):
    case = known_tv(name.split("_")[0], T=8, B=4, steps=3, **KNOWN_CASES[name])
    ep_d, g_d = run(monkeypatch, case, "device", F64)
    ep_h, g_h = run(monkeypatch, case, "host", F64)
    assert_same_forward(ep_d, ep_h, name)
    assert_close_grads(g_d, g_h, name)


@pytest.mark.parametrize("name", ["lin42_tensor", "lin52_pad_tensor", "lin42_slew", "lin42_plant_w"])
def test_one_step_is_time_invariant(monkeypatch, name):
    """n_steps = 1: the axis is the solve's own, so the forward is bitwise time_varying=False's."""
    case = lin_tv(T=6, B=5, steps=1, **LIN_CASES[name])
    ep_tv, _ = run(monkeypatch, case, "device", F64, differentiable=False)
    ep_ti, _ = run(monkeypatch, case, "device", F64, differentiable=False, tv=False)
    assert_same_forward(ep_tv, ep_ti, name)


@pytest.mark.parametrize("name", ["lin42", "lin42_tensor", "lin52_pad_tensor", "lin42_slew", "lin42_plant_w"])
def test_constant_axis_is_time_invariant(monkeypatch, name):
    """Inputs constant along the axis (stride-0 expand): the forward is bitwise the time-invariant episode's, and the
    gradients, summed by autograd through the expand, match its gradients."""
    kw = dict(LIN_CASES[name])
    case = lin_tv(T=6, B=5, steps=4, const=True, **kw)
    ep_tv, g_tv = run(monkeypatch, case, "device", F64)

    ti = lin_tv(T=6, B=5, steps=4, const=True, **kw)
    T = 6

    def problem(lv):                      # the same leaves on the solve's own axis
        ex = lambda v, Lv: v.expand(Lv, *v.shape[1:])  # noqa: E731
        dx = LinDx(ex(lv["F"], T - 1), ex(lv["f"], T - 1))
        pl = LinDx(ex(lv["Fp"], 1), ex(lv["fp"], 1)) if "Fp" in lv else None
        return lv["x0"], QuadCost(ex(lv["C"], T), ex(lv["c"], T)), dx, pl, lv.get("w")
    ti.problem = problem
    base_ctrl = ti.ctrl

    def ctrl(lv):
        c_ = base_ctrl(lv)
        if "lo" in lv:
            c_.u_lower, c_.u_upper = lv["lo"].expand(T, *lv["lo"].shape[1:]), lv["hi"].expand(T, *lv["hi"].shape[1:])
        return c_
    ti.ctrl = ctrl
    ep_ti, g_ti = run(monkeypatch, ti, "device", F64, tv=False)
    assert_same_forward(ep_tv, ep_ti, name)
    assert_close_grads(g_tv, g_ti, name, tol=1e-11)


FD_CASES = {"lin42": (dict(), ("x0", "C", "c", "F", "f")),
            "lin42_slew": (dict(slew=True), ("x0", "C", "c", "F", "f")),
            "lin42_plant_w": (dict(plant=True, with_w=True), ("x0", "C", "c", "F", "f", "Fp", "fp", "w")),
            "lin42_plant_w_slew": (dict(plant=True, with_w=True, slew=True), ("C", "F", "Fp", "fp", "w"))}


@pytest.mark.parametrize("name", sorted(FD_CASES))
def test_finite_differences(monkeypatch, name):
    """Central differences of the windowed loop in float64, along random directions in each input: plain, under a
    slew-rate penalty (the augmented full-length gradients, with the previous control held as the reference holds
    prev_ctrl), and on a LinDx plant with w (the plant's dF[k], df[k])."""
    kw, keys = FD_CASES[name]
    case = lin_tv(4, 2, T=5, B=2, steps=3, seed=4, **kw)
    lv = case.leaves(F64)
    ep0, g = run(monkeypatch, case, "device", F64, lv=lv)
    gen = torch.Generator().manual_seed(9)
    gg = torch.Generator().manual_seed(5)
    wx = torch.randn(ep0.x.shape, generator=gg, dtype=F64).to(DEV)
    wu = torch.randn(ep0.u.shape, generator=gg, dtype=F64).to(DEV)
    T = case.T
    # under a slew-rate penalty the differentiated loop holds each solve's previous control at the episode's own
    # value (zeros, then u_{k-1}), which is what detaching it means; the problems are unbounded LinDx, so every
    # solve reaches its optimum whatever its warm start
    prevs = [None] + [ep0.u[k].detach() for k in range(case.steps - 1)]

    def loss(lv2):
        if not kw.get("slew"):
            ep, _ = run(monkeypatch, case, "device", F64, differentiable=False, lv=lv2)
            return float((ep.x * wx).sum() + (ep.u * wu).sum())
        x0, cost, dx, plant, w = case.problem(lv2)
        Fs, fs = (plant.F, plant.f) if plant is not None else (dx.F, dx.f)
        x, total = x0, float((wx[0] * x0).sum())
        with torch.no_grad():
            for k in range(case.steps):
                c_ = case.ctrl(lv2)
                c_.prev_ctrl = prevs[k]
                _, plan_u, _ = c_(x, QuadCost(cost.C[k:k + T], cost.c[k:k + T]),
                                  LinDx(dx.F[k:k + T - 1], dx.f[k:k + T - 1]))
                u = plan_u[0]
                x = torch.einsum("bij,bj->bi", Fs[k], torch.cat((x, u), 1)) + fs[k]
                if w is not None:
                    x = x + w[k]
                total += float((wx[k + 1] * x).sum() + (wu[k] * u).sum())
        return total
    for k in keys:
        d = torch.randn(lv[k].shape, generator=gen, dtype=F64).to(DEV)
        if k == "C":
            d = d + d.transpose(-1, -2)
        h = 1e-6
        lp = {n: v.detach() + (h * d if n == k else 0) for n, v in lv.items()}
        lm = {n: v.detach() - (h * d if n == k else 0) for n, v in lv.items()}
        fd = (loss(lp) - loss(lm)) / (2 * h)
        an = float((g[k] * d).sum())
        assert abs(fd - an) <= 1e-5 * max(1.0, abs(an)), (name, k, fd, an)


def test_errors_before_anything_runs():
    case = lin_tv(4, 2, T=6, B=3, steps=4, bounds="tensor")
    lv = case.leaves(F64, grad=False)
    x0, cost, dx, _, _ = case.problem(lv)
    ctrl = case.ctrl(lv)
    with pytest.raises(MpcB200Error, match="slices"):
        receding_horizon(ctrl, x0, QuadCost(cost.C[:-1], cost.c[:-1]), dx, 4, time_varying=True)
    with pytest.raises(MpcB200Error, match="LinDx F"):
        receding_horizon(ctrl, x0, cost, LinDx(dx.F[:-2], dx.f[:-2]), 4, time_varying=True)
    with pytest.raises(MpcB200Error, match="QuadCost"):
        receding_horizon(ctrl, x0, torch.nn.Linear(6, 1).to(DEV), dx, 4, time_varying=True)
    with pytest.raises(MpcB200Error, match="plant"):
        receding_horizon(ctrl, x0, cost, dx, 4, plant=LinDx(dx.F[:1], dx.f[:1]), time_varying=True)
    ctrl.u_lower = ctrl.u_lower[:6]
    with pytest.raises(MpcB200Error, match="u_lower"):
        receding_horizon(ctrl, x0, cost, dx, 4, time_varying=True)


def test_no_host_read_and_capture(monkeypatch):
    case = lin_tv(4, 2, T=6, B=5, steps=4, bounds="tensor", plant=True, with_w=True)
    lv = case.leaves(F64)
    ref, g_ref = run(monkeypatch, case, "device", F64, lv=lv)
    lv2 = case.leaves(F64)
    x0, cost, dx, plant, w = case.problem(lv2)
    ctrl = case.ctrl(lv2)
    gg = torch.Generator().manual_seed(5)
    wx = torch.randn(ref.x.shape, generator=gg, dtype=F64).to(DEV)
    wu = torch.randn(ref.u.shape, generator=gg, dtype=F64).to(DEV)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        ep = receding_horizon(ctrl, x0, cost, dx, case.steps, differentiable=True, plant=plant, disturbance=w,
                              time_varying=True)
        ((ep.x * wx).sum() + (ep.u * wu).sum()).backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert_same_forward(ep, ref, "sync")
    assert_close_grads({k: v.grad for k, v in lv2.items()}, g_ref, "sync", tol=0.0)

    # the forward captured inside a caller's graph, then replayed
    lv3 = case.leaves(F64, grad=False)
    x0, cost, dx, plant, w = case.problem(lv3)
    ctrl = case.ctrl(lv3)
    receding_horizon(ctrl, x0, cost, dx, case.steps, plant=plant, disturbance=w, time_varying=True)   # warm up
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        cap = receding_horizon(ctrl, x0, cost, dx, case.steps, plant=plant, disturbance=w, time_varying=True)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(cap.x, ref.x) and torch.equal(cap.u, ref.u)


def test_batch_independence(monkeypatch):
    """A problem's episode and gradients do not depend on the other problems of its batch."""
    case = lin_tv(4, 2, T=6, B=6, steps=4, bounds="tensor", plant=True, with_w=True)
    ep, g = run(monkeypatch, case, "device", F64)
    sub = lin_tv(4, 2, T=6, B=6, steps=4, bounds="tensor", plant=True, with_w=True)
    keep = [1, 4]
    sub.base = {k: (v[:, keep] if k not in ("x0",) and v.dim() >= 3 else (v[keep] if k == "x0" else v))
                for k, v in case.base.items()}
    lv = sub.leaves(F64)
    x0, cost, dx, plant, w = sub.problem(lv)
    ctrl = sub.ctrl(lv)
    ep2 = receding_horizon(ctrl, x0, cost, dx, sub.steps, differentiable=True, plant=plant, disturbance=w,
                           time_varying=True)
    assert torch.equal(ep2.x, ep.x[:, keep]) and torch.equal(ep2.u, ep.u[:, keep])
    gg = torch.Generator().manual_seed(5)
    wx = torch.randn(ep.x.shape, generator=gg, dtype=F64).to(DEV)[:, keep]
    wu = torch.randn(ep.u.shape, generator=gg, dtype=F64).to(DEV)[:, keep]
    ((ep2.x * wx).sum() + (ep2.u * wu).sum()).backward()
    for k in ("C", "c", "F", "f", "Fp", "fp", "w", "lo"):
        if lv[k].grad is None:
            continue
        want = g[k][keep] if k == "x0" else g[k][:, keep]
        assert maxdiff(lv[k].grad, want) <= 1e-12 * max(1.0, float(want.abs().max())), k


def test_first_order_only(monkeypatch):
    case = lin_tv(4, 2, T=6, B=3, steps=3)
    lv = case.leaves(F64)
    x0, cost, dx, _, _ = case.problem(lv)
    ep = receding_horizon(case.ctrl(lv), x0, cost, dx, case.steps, differentiable=True, time_varying=True)
    (gC,) = torch.autograd.grad(ep.x.sum(), lv["C"], create_graph=True)
    with pytest.raises(RuntimeError):
        torch.autograd.grad(gC.sum(), lv["C"])


# the window stage kernel's grid: epgrad_grid (csrc/episode_grad.cu) caps it at 4096 blocks of 256 threads
WINDOW_GRID_THREADS = 4096 * 256
# a batch whose window copy of C, T * B * (n + m)^2 elements, exceeds the capped grid
GRID_CASE = dict(T=4, n=4, m=2)
GRID_CASE["B"] = WINDOW_GRID_THREADS // (GRID_CASE["T"] * (GRID_CASE["n"] + GRID_CASE["m"]) ** 2) + 64


def test_second_grid_stride_pass(monkeypatch):
    """GRID_CASE: the stage kernel takes a second grid-stride pass; the device forward is bitwise the host path's."""
    T, n, m, B = GRID_CASE["T"], GRID_CASE["n"], GRID_CASE["m"], GRID_CASE["B"]
    case = lin_tv(n, m, T=T, B=B, steps=2, bounds="tensor", plant=True, with_w=True, seed=6)
    ep_d, g_d = run(monkeypatch, case, "device", F64)
    ep_h, g_h = run(monkeypatch, case, "host", F64)
    assert_same_forward(ep_d, ep_h, "grid")
    assert_close_grads(g_d, g_h, "grid")


def test_continuation(monkeypatch):
    """Two calls of 2 and 3 steps, the second given the axis from step 2 on and u_next, are the episode of 5."""
    case = lin_tv(4, 2, T=6, B=4, steps=5, bounds="scalar")
    lv = case.leaves(F64, grad=False)
    x0, cost, dx, _, _ = case.problem(lv)
    full = receding_horizon(case.ctrl(lv), x0, cost, dx, 5, time_varying=True)
    c1 = case.ctrl(lv)
    a = receding_horizon(c1, x0, QuadCost(cost.C[:7], cost.c[:7]), LinDx(dx.F[:6], dx.f[:6]), 2, time_varying=True)
    c2 = case.ctrl(lv)
    c2.u_init = a.u_next
    b = receding_horizon(c2, a.x[-1], QuadCost(cost.C[2:], cost.c[2:]), LinDx(dx.F[2:], dx.f[2:]), 3,
                         time_varying=True)
    assert torch.equal(torch.cat((a.x, b.x[1:])), full.x) and torch.equal(torch.cat((a.u, b.u)), full.u)


# ------------------------------------------------------------------------------------------------------------------
class _Poisoned:
    """torch for the step module, with every torch.empty filled: NaN (floating), -1 (int32) or 0xFF (bytes), so an
    output or workspace element the library does not write fails a comparison."""

    def __getattr__(self, name):
        return getattr(torch, name)

    @staticmethod
    def empty(*shape, **kw):
        t = torch.empty(*shape, **kw)
        return t.fill_(float("nan") if t.is_floating_point() else (255 if t.dtype == torch.uint8 else -1))


ORACLE_CASES = {"lin42_tensor": ("lin", dict(n=4, m=2, bounds="tensor")),
                "lin52_pad_tensor": ("lin", dict(n=5, m=2, bounds="tensor", F_full=True)),
                "lin42_slew_scalar": ("lin", dict(n=4, m=2, slew=True, bounds="scalar")),
                "lin42_plant_w": ("lin", dict(n=4, m=2, plant=True, with_w=True, bounds="tensor")),
                "lin42_w": ("lin", dict(n=4, m=2, with_w=True)),
                "pendulum": ("known", dict()), "cartpole": ("known", dict()),
                "pendulum_slew": ("known", dict(slew=True))}


@pytest.mark.parametrize("name", sorted(ORACLE_CASES))
def test_device_against_window_oracle(monkeypatch, name):
    """The device path, with every output and workspace poisoned before the calls, against the float64 window oracle
    (oracle/window_oracle.py) on the device's own plans: x from those plans through the model or plant, and every
    full-length gradient (dC, dc, dF, df, a plant's dF_p, df_p, dw) to 1e-10 of max|g|."""
    from oracle import window_oracle as wo
    from tests.gpu_harness import episode_known_step
    kind, kw = ORACLE_CASES[name]
    if kind == "lin":
        case = lin_tv(T=6, B=5, steps=4, seed=3, **kw)
    else:
        case = known_tv(name.split("_")[0], T=8, B=4, steps=3, **kw)
    saved = []
    real = step.episode_backward_raw

    def spy(s, *a):
        saved.append(s)
        return real(s, *a)
    monkeypatch.setattr(step, "episode_backward_raw", spy)
    monkeypatch.setattr(step, "torch", _Poisoned())
    lv = case.leaves(F64)
    ep, g = run(monkeypatch, case, "device", F64, lv=lv)
    monkeypatch.undo()
    assert len(saved) == 1 and saved[0][0].window is not None
    s, n_steps, _, _, plan_x, plan_u = saved[0]
    n, m, T = case.n, case.m, case.T
    ctrl = case.ctrl(lv)
    slew = ctrl.slew_rate_penalty
    cpu = {k: v.detach().cpu() for k, v in lv.items()}
    x, u = ep.x.detach().cpu(), ep.u.detach().cpu()
    px = plan_x.cpu()[..., :(n + m if slew else n)]
    pu = plan_u.cpu()[..., :m]
    gg = torch.Generator().manual_seed(5)
    wx = torch.randn(ep.x.shape, generator=gg, dtype=F64)
    wu = torch.randn(ep.u.shape, generator=gg, dtype=F64)
    assert torch.equal(pu[:, 0], u)
    if kind == "lin":
        Fs, fs = (cpu["Fp"], cpu["fp"]) if "Fp" in cpu else (cpu["F"], cpu["f"])
        plant = ("lin", cpu["Fp"], cpu["fp"]) if "Fp" in cpu else None
        bnd = (dict(u_lower=cpu["lo"], u_upper=cpu["hi"]) if "lo" in cpu else
               dict(u_lower=ctrl.u_lower, u_upper=ctrl.u_upper))
        xr = [x[0]]
        for k in range(n_steps):
            nx = (Fs[k] @ torch.cat((xr[-1], u[k]), 1).unsqueeze(-1)).squeeze(-1) + fs[k]
            xr.append(nx + cpu["w"][k] if "w" in cpu else nx)
        out = wo.receding_horizon_backward_tv(n, m, T, cpu["C"], cpu["c"], cpu["F"], cpu["f"], x, u, px, pu, wx, wu,
                                              slew_rate_penalty=slew, plant=plant if plant or "w" in cpu else None,
                                              **bnd)
        pairs = [("x0", "dx_init"), ("C", "dC"), ("c", "dc"), ("F", "dF"), ("f", "df"), ("Fp", "dF_p"),
                 ("fp", "df_p"), ("w", "dw")]
    else:
        mod = KNOWN[name.split("_")[0]][0](cpu["params"])
        mstep = episode_known_step(mod)
        theta = cpu["params"].expand(case.B, -1)
        xr = [x[0]]
        for k in range(n_steps):
            xr.append(mstep(xr[-1], u[k], theta).detach())
        out = wo.receding_horizon_backward_tv(n, m, T, cpu["C"], cpu["c"], None, None, x, u, px, pu, wx, wu,
                                              u_lower=ctrl.u_lower, u_upper=ctrl.u_upper, step=mstep, theta=theta,
                                              slew_rate_penalty=slew)
        out["dtheta"] = out["dtheta"].sum(0)
        pairs = [("x0", "dx_init"), ("C", "dC"), ("c", "dc"), ("params", "dtheta")]
    xr = torch.stack(xr)
    assert maxdiff(x, xr) <= 1e-12 * max(1.0, float(xr.abs().max())), name
    for leaf, key in pairs:
        if leaf not in cpu or out.get(key) is None:
            continue
        got, want = g[leaf].cpu(), out[key]
        assert bool(torch.isfinite(got).all()), (name, leaf)
        assert maxdiff(got, want) <= 1e-10 * max(1.0, float(want.abs().max())), (name, leaf, maxdiff(got, want))


FIXTURE_CASES = ["linear", "linear_plant", "pendulum", "cartpole", "pendulum_slew"]


@pytest.mark.parametrize("case", FIXTURE_CASES)
def test_against_reference_fixture(case):
    """The reference's own windowed loop (tests/golden/receding_tv_f64.npz), end to end through
    receding_horizon(time_varying=True, differentiable=True).  The solves bound their controls, so the tolerance is
    pnqp's own accuracy (2e-4, as the plant fixture's).  A known model's parameter gradient follows this project's
    convention (the linearisation's Jacobians differentiated), so it is checked against the window oracle with
    full_linearisation=True on the fixture's plans."""
    import os
    import numpy as np
    from oracle import window_oracle as wo
    from tests.gpu_harness import episode_known_step
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "receding_tv_f64.npz"))
    others = [c + "_" for c in FIXTURE_CASES if c != case and c.startswith(case)]
    t = {k[len(case) + 1:]: torch.from_numpy(z[k]) for k in z.files
         if k.startswith(case + "_") and not any(k.startswith(o) for o in others)}
    T_, steps = int(t["T"]), int(t["n_steps"])
    lv = {k: t[k].clone().to(DEV).requires_grad_(True)
          for k in ("x_init", "C", "c", "w", "F", "f", "F_p", "f_p", "params") if k in t}
    plant = None
    if case.startswith("linear"):
        n, m = 4, 2
        if "lo" in t:
            b = dict(u_lower=t["lo"].to(DEV), u_upper=t["hi"].to(DEV))
        else:
            b = dict(u_lower=-float(t["bound"]), u_upper=float(t["bound"]))
        ctrl = MPC(n, m, T_, lqr_iter=int(t["lqr_iter"]), eps=float(t["eps"]), verbose=-1, **b)
        dx = LinDx(lv["F"], lv["f"])
        if "F_p" in lv:
            plant = LinDx(lv["F_p"], lv["f_p"])
    else:
        clamp = float(t["clamp"])
        cls = CartpoleDx if case == "cartpole" else PendulumDx
        dx = cls(params=lv["params"])
        setattr(dx, "force_mag" if case == "cartpole" else "max_torque", clamp)
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
                              plant=plant, disturbance=lv.get("w"), time_varying=True)
        ((t["wx"].to(DEV) * ep.x).sum() + (t["wu"].to(DEV) * ep.u).sum()).backward()
    finally:
        step.episode_backward_raw = real
    assert len(calls) == 1 and calls[0][0].window is not None
    errs = {"x": maxdiff(ep.x, t["x"].to(DEV)) / max(1.0, float(t["x"].abs().max())),
            "u": maxdiff(ep.u, t["u"].to(DEV)) / max(1.0, float(t["u"].abs().max()))}
    for k in lv:
        if k == "params":
            continue
        want = t["g_" + k].to(DEV)
        errs["d" + k] = maxdiff(lv[k].grad, want) / max(1.0, float(want.abs().max()))
    if "params" in lv:
        B_ = t["x"].shape[1]
        mod = (CartpoleDx if case == "cartpole" else PendulumDx)()
        setattr(mod, "force_mag" if case == "cartpole" else "max_torque", clamp)
        want = wo.receding_horizon_backward_tv(
            n, 1, T_, t["C"], t["c"], None, None, t["x"], t["u"], t["plan_x"], t["plan_u"], t["wx"], t["wu"],
            u_lower=-clamp, u_upper=clamp, step=episode_known_step(mod), theta=t["params"].expand(B_, -1),
            slew_rate_penalty=float(t["slew"]) if "slew" in t else None)["dtheta"].sum(0)
        errs["dparams (oracle, full)"] = maxdiff(lv["params"].grad.cpu(), want) / max(1.0, float(want.abs().max()))
    print(f"{case}: " + ", ".join(f"{k} {v:.2e}" for k, v in errs.items()))
    assert all(v <= 2e-4 for v in errs.values()), errs
