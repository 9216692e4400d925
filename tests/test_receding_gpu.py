"""GPU: receding_horizon's device path (one mpcb200_episode_* call, one CUDA graph per episode) computes bitwise what
its host path computes - a Python loop over MPC.forward whose every solve takes the device loop - for LinDx (exact,
zero-padded and large shapes, every bound kind), the known systems, slew-rate penalties and the notebooks' full
sizes; it matches the reference's own notebook loop (float64 fixtures); episodes continue from u_next; the episode is
one graph that makes no host read; and Module costs or opaque dynamics take the host path."""
import os

import numpy as np
import pytest
import torch

from mpc.pytorch_b200 import _lib, control, step
from mpc.pytorch_b200.control import receding_horizon, shift_warm_start
from mpc.pytorch_b200.dynamics import CartpoleDx, PendulumDx
from mpc.pytorch_b200.solver import MPC, GradMethods, LinDx, QuadCost
from tests.cartpole import initial_states
from tests.gpu_harness import DEV
from tests.helpers import gen_problem

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FIELDS = ("x", "u", "costs", "info", "u_next")


def run(monkeypatch, make, x0, cost, dx, n_steps, device):
    """receding_horizon on the device path (asserting that it ran) or on the host path; outputs synchronised."""
    seen = {}
    with monkeypatch.context() as mp:
        if device:
            real = step.episode_raw

            def spy(*a, **k):
                seen["res"] = real(*a, **k)
                return seen["res"]
            mp.setattr(step, "episode_raw", spy)
        else:
            mp.setattr(control, "_episode_device", lambda *a: None)
        ep = receding_horizon(make(), x0, cost, dx, n_steps)
    assert (seen.get("res") is not None) == device, "the device path did not run"
    torch.cuda.synchronize()
    return ep


def same_on_both_paths(monkeypatch, make, x0, cost, dx, n_steps):
    host = run(monkeypatch, make, x0, cost, dx, n_steps, False)
    dev = run(monkeypatch, make, x0, cost, dx, n_steps, True)
    for k in FIELDS:
        a, b = getattr(dev, k), getattr(host, k)
        assert a.shape == b.shape and a.dtype == b.dtype, (k, a.shape, b.shape, a.dtype, b.dtype)
        assert torch.equal(a, b.to(a.device)), f"{k}: {float((a.double() - b.double().to(a.device)).abs().max()):.3e}"
    assert bool((dev.info[:, 0] >= 1).all())
    return dev


def _linear(B, T, n, m, dtype, seed=0):
    C, c, F, f, x0 = gen_problem(seed, B, T, n, m, dtype)
    return [t.to(DEV) for t in (C, c, 0.9 * F, f, x0)]


def _linear_kw(case, T, B, m, dtype):
    kw = dict(lqr_iter=8, verbose=-1)
    g = torch.Generator().manual_seed(1)
    if case == "scalar":
        kw.update(u_lower=-0.25, u_upper=0.25)
    if case == "tensor_delta":
        lo = -0.1 - 0.3 * torch.rand(T, B, m, generator=g, dtype=dtype)
        kw.update(u_lower=lo.to(DEV), u_upper=(-lo + 0.05).to(DEV), delta_u=0.1)
    if case == "zero_mask":
        kw.update(u_zero_I=(torch.rand(T, B, m, generator=g) < 0.3).to(DEV))
    return kw


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("case", ["none", "scalar", "tensor_delta", "zero_mask"])
def test_linear_8_2(monkeypatch, dtype, case):
    B, T, n, m = 16, 8, 8, 2
    C, c, F, f, x0 = _linear(B, T, n, m, dtype)
    kw = _linear_kw(case, T, B, m, dtype)
    same_on_both_paths(monkeypatch, lambda: MPC(n, m, T, **kw), x0, QuadCost(C, c), LinDx(F, f), 6)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("n,m", [(6, 1), (20, 4)])          # zero-padded instance, large-shape kernels
def test_linear_padded_and_large(monkeypatch, dtype, n, m):
    B, T = 12, 6
    C, c, F, f, x0 = _linear(B, T, n, m, dtype, seed=3)
    for kw in (dict(), dict(u_lower=-0.3, u_upper=0.3)):
        same_on_both_paths(monkeypatch, lambda: MPC(n, m, T, lqr_iter=6, verbose=-1, **kw), x0, QuadCost(C, c),
                           LinDx(F, f), 5)


def _system(name, B, T, dtype, seed=0):
    sysdx = CartpoleDx() if name == "cartpole" else PendulumDx()
    n, m = sysdx.n_state, sysdx.n_ctrl
    q, p = sysdx.get_true_obj()
    Q = torch.diag(q).expand(T, B, n + m, n + m).contiguous().to(DEV, dtype)
    pp = p.expand(T, B, n + m).contiguous().to(DEV, dtype)
    if name == "cartpole":
        x0 = initial_states(B, seed=seed).to(DEV, dtype)
    else:
        th = torch.linspace(-1.5, 1.5, B, dtype=torch.float64)
        x0 = torch.stack((th.cos(), th.sin(), 0.1 * th), 1).to(DEV, dtype)
    return sysdx, x0, QuadCost(Q, pp)


def _notebook_mpc(sysdx, T, lqr_iter=50, verbose=-1, **kw):
    """The solver options of the reference's notebooks."""
    return lambda: MPC(sysdx.n_state, sysdx.n_ctrl, T, u_lower=float(sysdx.lower), u_upper=float(sysdx.upper),
                       lqr_iter=lqr_iter, verbose=verbose, linesearch_decay=sysdx.linesearch_decay,
                       max_linesearch_iter=sysdx.max_linesearch_iter, grad_method=GradMethods.AUTO_DIFF, eps=1e-2,
                       **kw)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("name", ["cartpole", "pendulum"])
def test_known_systems(monkeypatch, dtype, name):
    sysdx, x0, cost = _system(name, 8, 12, dtype)
    same_on_both_paths(monkeypatch, _notebook_mpc(sysdx, 12, 20), x0, cost, sysdx, 8)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_slew_known_system(monkeypatch, dtype):
    sysdx, x0, cost = _system("pendulum", 8, 10, dtype)
    prev = torch.linspace(-1.0, 1.0, 8, dtype=dtype, device=DEV).view(8, 1)
    for p in (None, prev):
        same_on_both_paths(monkeypatch, _notebook_mpc(sysdx, 10, 15, slew_rate_penalty=0.5, prev_ctrl=p), x0, cost,
                           sysdx, 6)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_slew_linear(monkeypatch, dtype):
    B, T, n, m = 12, 8, 8, 2
    C, c, F, f, x0 = _linear(B, T, n, m, dtype, seed=7)
    prev = 0.1 * torch.ones(B, m, dtype=dtype, device=DEV)
    same_on_both_paths(monkeypatch, lambda: MPC(n, m, T, u_lower=-0.3, u_upper=0.3, lqr_iter=8, verbose=-1,
                                                slew_rate_penalty=0.3, prev_ctrl=prev),
                       x0, QuadCost(C, c), LinDx(F, f), 5)


def test_cartpole_notebook_size(monkeypatch):
    """The cartpole notebook: B=8, T=25, 100 control steps, lqr_iter=50, eps=1e-2."""
    sysdx, x0, cost = _system("cartpole", 8, 25, torch.float32)
    same_on_both_paths(monkeypatch, _notebook_mpc(sysdx, 25), x0, cost, sysdx, 100)


def test_pendulum_notebook_size(monkeypatch):
    """The pendulum notebook: PendulumDx((10, 1, 1)), B=16, T=20, 100 control steps."""
    sysdx, x0, cost = _system("pendulum", 16, 20, torch.float32)
    same_on_both_paths(monkeypatch, _notebook_mpc(sysdx, 20), x0, cost, sysdx, 100)


def test_config2_size(monkeypatch):
    """BASELINE config 2's solve (cartpole, B=128, T=25) as an episode of 20 control steps."""
    sysdx, x0, cost = _system("cartpole", 128, 25, torch.float32, seed=2)
    same_on_both_paths(monkeypatch, _notebook_mpc(sysdx, 25), x0, cost, sysdx, 20)


# ------------------------------------------------------------------------------------------------------------------
# the reference's own notebook loop (tests/golden/receding_*_f64.npz, oracle/make_golden_receding.py)
# ------------------------------------------------------------------------------------------------------------------
def _fixture_case(name):
    g = dict(np.load(os.path.join(GOLD, f"receding_{name}_f64.npz")))
    t = {k: torch.from_numpy(v).to(DEV) for k, v in g.items() if v.dtype == np.float64}
    T, steps = int(g["T"]), int(g["n_steps"])
    opts = dict(lqr_iter=int(g["lqr_iter"]), verbose=-1, eps=float(g["eps"]),
                linesearch_decay=float(g["decay"]), max_linesearch_iter=int(g["ls_iter"]))
    if "bound" in g:
        opts.update(u_lower=-float(g["bound"]), u_upper=float(g["bound"]))
    if "penalty" in g:
        opts.update(slew_rate_penalty=float(g["penalty"]))
    if name == "linear":
        n, m = t["F"].shape[2], t["F"].shape[3] - t["F"].shape[2]
        dx = LinDx(t["F"], t["f"])
    else:
        dx = (CartpoleDx if name == "cartpole" else PendulumDx)(params=torch.from_numpy(g["params"]))
        n, m = dx.n_state, dx.n_ctrl
        opts.update(u_lower=float(dx.lower), u_upper=float(dx.upper), grad_method=GradMethods.AUTO_DIFF)
    return g, t, MPC(n, m, T, **opts), QuadCost(t["C"], t["c"]), dx, steps


@pytest.mark.parametrize("name", ["cartpole", "pendulum", "linear", "pendulum_slew"])
def test_against_reference_notebook_loop(monkeypatch, name):
    g, t, ctrl, cost, dx, steps = _fixture_case(name)
    ep = run(monkeypatch, lambda: ctrl, t["x_init"], cost, dx, steps, True)
    assert ep.info[:, 0].cpu().long().tolist() == g["iters"].tolist(), f"{name}: iterations per solve"
    # x and costs to 1e-5; the controls at pnqp's own accuracy (it stops at |dx| < 1e-4, and the reference couples
    # that test over the batch, INTEGRATION.md section 2), as tests/test_dynamics_gpu.py compares the pendulum solve,
    # with the set of controls on the bounds exactly
    for k, tol in (("x", 1e-5), ("costs", 1e-5), ("u", 2e-4)):
        err = float((getattr(ep, k) - t[k]).abs().max())
        assert err <= tol * max(1.0, float(t[k].abs().max())), f"{name}: {k} {err:.3e}"
    bound = float(ctrl.u_upper)
    assert torch.equal(ep.u.abs() == bound, t["u"].abs() == bound), f"{name}: controls on the bounds"


# ------------------------------------------------------------------------------------------------------------------
# continuation, one graph, no host read, routing
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["linear", "slew_pendulum"])
def test_continuation(case):
    if case == "linear":
        B, T, n, m = 16, 8, 8, 2
        C, c, F, f, x0 = _linear(B, T, n, m, torch.float64, seed=9)
        cost, dx = QuadCost(C, c), LinDx(F, f)
        make = lambda **o: MPC(n, m, T, u_lower=-0.3, u_upper=0.3, lqr_iter=8, verbose=-1, **o)  # noqa: E731
    else:
        dx, x0, cost = _system("pendulum", 8, 10, torch.float64)
        make = lambda **o: _notebook_mpc(dx, 10, 15, slew_rate_penalty=0.5, **o)()  # noqa: E731
    slew = case != "linear"
    whole = receding_horizon(make(), x0, cost, dx, 7)
    first = receding_horizon(make(), x0, cost, dx, 3)
    more = dict(u_init=first.u_next, **(dict(prev_ctrl=first.u[-1]) if slew else {}))
    second = receding_horizon(make(**more), first.x[-1], cost, dx, 4)
    torch.cuda.synchronize()
    assert torch.equal(whole.x, torch.cat((first.x, second.x[1:])))
    assert torch.equal(whole.u, torch.cat((first.u, second.u)))
    assert torch.equal(whole.costs, torch.cat((first.costs, second.costs)))
    assert torch.equal(whole.info, torch.cat((first.info, second.info)))
    assert torch.equal(whole.u_next, second.u_next)


def test_one_graph_per_episode():
    B, T, n, m = 16, 8, 8, 2
    C, c, F, f, x0 = _linear(B, T, n, m, torch.float32, seed=11)
    ctrl = MPC(n, m, T, u_lower=-0.3, u_upper=0.3, lqr_iter=8, verbose=-1)
    counts = []
    for steps in (1, 100, 1):
        before = _lib.launch_count()
        ep = receding_horizon(ctrl, x0, QuadCost(C, c), LinDx(F, f), steps)
        counts.append(_lib.launch_count() - before)
        torch.cuda.synchronize()
        assert bool((ep.info[:, 0] >= 1).all()), ep.info[:, 0].tolist()
    assert counts[0] == counts[1] == counts[2], counts


def test_no_host_read_linear():
    B, T, n, m = 16, 8, 8, 2
    C, c, F, f, x0 = _linear(B, T, n, m, torch.float32, seed=13)
    ctrl = MPC(n, m, T, u_lower=-0.3, u_upper=0.3, lqr_iter=8, verbose=-1)
    cost, dx = QuadCost(C, c), LinDx(F, f)
    receding_horizon(ctrl, x0, cost, dx, 5)                   # library load and kernel set-up
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        receding_horizon(ctrl, x0, cost, dx, 5)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    _capture_matches_eager(ctrl, cost, dx, [x0, 0.5 * x0, x0.flip(0)], 5)


def test_capture_known_system():
    # pinned CPU parameters: nothing to read back, and nothing a capture cannot copy
    sysdx = CartpoleDx(params=torch.tensor((9.8, 1.0, 0.1, 0.5)).pin_memory())
    _, x0, cost = _system("cartpole", 16, 15, torch.float32)
    _capture_matches_eager(_notebook_mpc(sysdx, 15, 20)(), cost, sysdx,
                           [x0, x0.flip(0), initial_states(16, seed=3).to(DEV)], 6)


def _capture_matches_eager(ctrl, cost, dx, x0s, steps):
    static_x0 = x0s[0].clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        receding_horizon(ctrl, static_x0, cost, dx, steps)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = receding_horizon(ctrl, static_x0, cost, dx, steps)
    for x0 in x0s[1:]:
        static_x0.copy_(x0)
        graph.replay()
        want = receding_horizon(ctrl, x0, cost, dx, steps)
        torch.cuda.synchronize()
        for k in FIELDS:
            assert torch.equal(getattr(out, k), getattr(want, k)), k


def _notebook_loop(make, x0, cost, dx, steps):
    """The notebooks' loop, written out."""
    u_init, x, xs, us = None, x0, [x0], []
    for _ in range(steps):
        _, actions, _ = make(u_init)(x, cost, dx)
        u_init = torch.cat((actions[1:], torch.zeros_like(actions[:1])), dim=0)
        u_init[-2] = u_init[-3]
        x = dx(x, actions[0])
        xs.append(x)
        us.append(actions[0])
    return torch.stack(xs).detach(), torch.stack(us).detach()


class _QuadModule(torch.nn.Module):
    """0.5 tau' Q tau + p' tau as a Module cost."""

    def __init__(self, Q, p):
        super().__init__()
        self.Q, self.p = Q, p

    def forward(self, tau):
        return 0.5 * (tau * (tau @ self.Q)).sum(-1) + (tau * self.p).sum(-1)


class _Opaque(torch.nn.Module):
    """A cartpole the kernels do not know: no mpcb200_kind."""

    def __init__(self):
        super().__init__()
        self.inner = CartpoleDx()

    def forward(self, x, u):
        return self.inner(x, u)


@pytest.mark.parametrize("case", ["module_cost", "opaque_dynamics"])
def test_routing_to_host_path(monkeypatch, case):
    B, T, steps = 4, 10, 4
    sysdx, x0, cost = _system("cartpole", B, T, torch.float64)
    dx = _Opaque() if case == "opaque_dynamics" else sysdx
    if case == "module_cost":
        cost = _QuadModule(cost.C[0, 0], cost.c[0, 0])
    opts = dict(u_lower=sysdx.lower, u_upper=sysdx.upper, lqr_iter=10, verbose=-1, n_batch=B,
                linesearch_decay=sysdx.linesearch_decay, max_linesearch_iter=sysdx.max_linesearch_iter,
                grad_method=GradMethods.AUTO_DIFF, eps=1e-2, exit_unconverged=False, detach_unconverged=False)
    called = []
    monkeypatch.setattr(step, "episode_raw", lambda *a, **k: called.append(1))
    ep = receding_horizon(MPC(5, 1, T, **opts), x0, cost, dx, steps)
    assert not called
    x, u = _notebook_loop(lambda w: MPC(5, 1, T, u_init=w, **opts), x0, cost, dx, steps)
    if case == "opaque_dynamics":          # the same solves and the same Module step: bit for bit
        assert torch.equal(ep.x, x) and torch.equal(ep.u, u)
    else:                                  # the model step runs in the kernel, the notebook's in torch
        assert float((ep.x - x).abs().max()) < 1e-9 and float((ep.u - u).abs().max()) < 1e-9
    assert ep.info.shape == (steps, 2) and bool((ep.info[:, 0] >= 1).all())


def test_pnqp_warnings_match(monkeypatch, capsys):
    sysdx, x0, cost = _system("cartpole", 16, 15, torch.float32)
    make = _notebook_mpc(sysdx, 15, 20, verbose=0)
    run(monkeypatch, make, x0, cost, sysdx, 5, False)
    host_out = capsys.readouterr().out
    run(monkeypatch, make, x0, cost, sysdx, 5, True)
    assert capsys.readouterr().out == host_out


def test_warm_start_rule_on_device():
    plan = torch.randn(7, 3, 2, device=DEV)
    w = shift_warm_start(plan)
    assert torch.equal(w[:5], plan[1:6]) and torch.equal(w[5], plan[5]) and bool((w[6] == 0).all())
