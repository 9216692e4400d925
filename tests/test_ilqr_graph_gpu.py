"""GPU: MPC.forward's iLQR loop as one device-side CUDA graph (mpcb200_ilqr_*) computes bitwise what the host loop
computes - x, u, costs, the iteration count, the printed pnqp warnings and the gradients of .backward() - for LinDx
problems (exact, zero-padded and large shapes, time-invariant inputs, every bound kind) and the known systems; the
solve makes no host read, so torch.cuda.graph captures it and its replays equal eager solves."""
import pytest
import torch

from mpc.pytorch_b200 import solver
from mpc.pytorch_b200.dynamics import CartpoleDx, PendulumDx
from mpc.pytorch_b200.solver import MPC, GradMethods, LinDx, QuadCost
from tests.cartpole import initial_states
from tests.gpu_harness import DEV, same_on_both_loops, solve_on
from tests.helpers import gen_problem

pytestmark = pytest.mark.gpu


def _linear(B, T, n, m, dtype, seed=0):
    C, c, F, f, x0 = gen_problem(seed, B, T, n, m, dtype)
    return [t.to(DEV) for t in (C, c, F, f, x0)]


BOUNDS = ("none", "scalar", "tensor", "delta_u", "zero_mask", "u_init_2d", "u_init_3d")


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("case", BOUNDS)
def test_linear_8_2(monkeypatch, dtype, case):
    B, T, n, m = 64, 12, 8, 2
    C, c, F, f, x0 = _linear(B, T, n, m, dtype)
    kw = dict(lqr_iter=10, verbose=-1, exit_unconverged=False, detach_unconverged=False)
    g = torch.Generator().manual_seed(1)
    if case in ("scalar", "delta_u", "u_init_2d", "u_init_3d"):
        kw.update(u_lower=-0.25, u_upper=0.25)
    if case == "tensor":
        lo = -0.1 - 0.3 * torch.rand(T, B, m, generator=g, dtype=dtype)
        kw.update(u_lower=lo.to(DEV), u_upper=(-lo + 0.05).to(DEV))
    if case == "delta_u":
        kw.update(delta_u=0.1)
    if case == "zero_mask":
        kw.update(u_zero_I=(torch.rand(T, B, m, generator=g) < 0.3).to(DEV))
    if case == "u_init_2d":
        kw.update(u_init=(0.1 * torch.randn(T, m, generator=g, dtype=dtype)).to(DEV))
    if case == "u_init_3d":
        kw.update(u_init=(0.1 * torch.randn(T, B, m, generator=g, dtype=dtype)).to(DEV))
    same_on_both_loops(monkeypatch, lambda: MPC(n, m, T, **kw), x0, QuadCost(C, c), LinDx(F, f))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("n,m", [(6, 1), (20, 4)])          # zero-padded instance, large-shape kernels
def test_linear_padded_and_large(monkeypatch, dtype, n, m):
    B, T = 32, 10
    C, c, F, f, x0 = _linear(B, T, n, m, dtype, seed=3)
    for bounds in ({}, dict(u_lower=-0.3, u_upper=0.3)):
        same_on_both_loops(monkeypatch, lambda: MPC(n, m, T, lqr_iter=8, verbose=-1, exit_unconverged=False,
                                       detach_unconverged=False, **bounds), x0, QuadCost(C, c), LinDx(F, f))


def test_linear_time_invariant_inputs(monkeypatch):
    B, T, n, m = 48, 10, 8, 2
    C, c, F, f, x0 = _linear(B, T, n, m, torch.float32, seed=5)
    C2, c1 = C[0, 0], c[0, 0]                                   # expanded over time and batch by MPC
    F_lti = F[0].unsqueeze(0).expand(T - 1, B, n, n + m)         # stride 0 over time
    same_on_both_loops(monkeypatch, lambda: MPC(n, m, T, u_lower=-0.2, u_upper=0.2, lqr_iter=6, verbose=-1,
                                                n_batch=B, exit_unconverged=False, detach_unconverged=False),
          x0, QuadCost(C2, c1), LinDx(F_lti, None))


@pytest.mark.parametrize("B", [1, 257])
def test_linear_batch_sizes(monkeypatch, B):
    T, n, m = 9, 8, 2
    C, c, F, f, x0 = _linear(B, T, n, m, torch.float32, seed=B)
    same_on_both_loops(monkeypatch, lambda: MPC(n, m, T, u_lower=-0.25, u_upper=0.25, lqr_iter=10, verbose=-1,
                                                exit_unconverged=False, detach_unconverged=False),
                       x0, QuadCost(C, c), LinDx(F, f))


def test_stop_reasons(monkeypatch):
    B, T, n, m = 32, 10, 8, 2
    C, c, F, f, x0 = _linear(B, T, n, m, torch.float64, seed=7)
    cost, dx = QuadCost(C, c), LinDx(F, f)
    base = dict(u_lower=-0.25, u_upper=0.25, verbose=-1, exit_unconverged=False, detach_unconverged=False)

    def iters(**o):
        return same_on_both_loops(monkeypatch, lambda: MPC(n, m, T, **base, **o), x0, cost, dx)[0].iters

    # by eps: a loose tolerance ends the loop before lqr_iter
    assert iters(lqr_iter=30, eps=1e-3) < 30
    # by not_improved_lim: no iteration ever counts as an improvement
    assert iters(lqr_iter=30, eps=0.0, best_cost_eps=-1e9, not_improved_lim=2) == 3
    # at lqr_iter
    assert iters(lqr_iter=4, eps=0.0) == 4
    assert iters(lqr_iter=1) == 1


def _system_problem(sysdx, B, T, dtype):
    n, m = sysdx.n_state, sysdx.n_ctrl
    q, p = sysdx.get_true_obj()
    Q = torch.diag(q).expand(T, B, n + m, n + m).contiguous().to(DEV, dtype)
    pp = p.expand(T, B, n + m).contiguous().to(DEV, dtype)
    if isinstance(sysdx, CartpoleDx):
        x0 = initial_states(B, seed=0).to(DEV, dtype)
    else:
        th = torch.linspace(-3.0, 3.0, B, dtype=torch.float64)
        x0 = torch.stack((th.cos(), th.sin(), torch.zeros(B, dtype=torch.float64)), 1).to(DEV, dtype)
    return x0, QuadCost(Q, pp)


def _system_mpc(sysdx, T, lqr_iter, verbose=-1):
    return lambda: MPC(sysdx.n_state, sysdx.n_ctrl, T, u_lower=float(sysdx.lower), u_upper=float(sysdx.upper),
                       lqr_iter=lqr_iter, verbose=verbose, exit_unconverged=False, detach_unconverged=False,
                       linesearch_decay=sysdx.linesearch_decay, max_linesearch_iter=sysdx.max_linesearch_iter,
                       grad_method=GradMethods.AUTO_DIFF, eps=sysdx.mpc_eps)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("system", ["cartpole", "pendulum"])
def test_known_systems(monkeypatch, dtype, system):
    sysdx = CartpoleDx() if system == "cartpole" else PendulumDx()
    B, T = 32, 15
    x0, cost = _system_problem(sysdx, B, T, dtype)
    assert same_on_both_loops(monkeypatch, _system_mpc(sysdx, T, 20), x0, cost, sysdx)[0].iters >= 2


def test_config2_cartpole_full_size(monkeypatch):
    """BASELINE config 2: cartpole, B=128, T=25, bounds +-100, <= 50 iterations, eps 1e-2, AUTO_DIFF."""
    sysdx = CartpoleDx()
    B, T = 128, 25
    x0, cost = _system_problem(sysdx, B, T, torch.float32)
    make = lambda: MPC(5, 1, T, u_lower=sysdx.lower, u_upper=sysdx.upper, lqr_iter=50, verbose=-1,  # noqa: E731
                       exit_unconverged=False, detach_unconverged=False, linesearch_decay=sysdx.linesearch_decay,
                       max_linesearch_iter=sysdx.max_linesearch_iter, grad_method=GradMethods.AUTO_DIFF, eps=1e-2)
    assert same_on_both_loops(monkeypatch, make, x0, cost, sysdx)[0].iters >= 2


def test_pnqp_warnings_match(monkeypatch, capsys):
    sysdx = CartpoleDx()
    B, T = 64, 20
    x0, cost = _system_problem(sysdx, B, T, torch.float32)
    make = _system_mpc(sysdx, T, 30, verbose=0)
    solve_on(monkeypatch, make, x0, cost, sysdx, False)
    host_out = capsys.readouterr().out
    solve_on(monkeypatch, make, x0, cost, sysdx, True)
    dev_out = capsys.readouterr().out
    assert dev_out == host_out
    # and on a bounded LinDx problem whose QPs get the default 20 pnqp iterations
    C, c, F, f, x0 = _linear(64, 12, 8, 2, torch.float32, seed=11)
    make = lambda: MPC(8, 2, 12, u_lower=-0.05, u_upper=0.05, lqr_iter=10, verbose=0,  # noqa: E731
                       exit_unconverged=False, detach_unconverged=False)
    solve_on(monkeypatch, make, x0, QuadCost(C, c), LinDx(F, f), False)
    host_out = capsys.readouterr().out
    solve_on(monkeypatch, make, x0, QuadCost(C, c), LinDx(F, f), True)
    assert capsys.readouterr().out == host_out


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_gradients_match(monkeypatch, dtype):
    B, T, n, m = 16, 8, 8, 2
    base = _linear(B, T, n, m, dtype, seed=13)
    grads = []
    for device_loop in (False, True):
        C, c, F, f, x0 = [t.clone().requires_grad_(True) for t in base]
        with monkeypatch.context() as mp:
            if not device_loop:
                mp.setattr(solver, "_use_device_loop", lambda *a: False)
            ctrl = MPC(n, m, T, u_lower=-0.25, u_upper=0.25, lqr_iter=10, verbose=-1, exit_unconverged=False,
                       detach_unconverged=False)
            x, u, _ = ctrl(x0, QuadCost(C, c), LinDx(F, f))
            (x.square().sum() + u.sum()).backward()
        grads.append([t.grad for t in (C, c, F, f, x0)])
    for a, b in zip(*grads):
        assert torch.equal(a, b), float((a - b).abs().max())


def _capture_matches_eager(ctrl, cost, dx, x0s):
    static_x0 = x0s[0].clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):                               # warm-up outside the capture, as torch advises
        ctrl(static_x0, cost, dx)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = ctrl(static_x0, cost, dx)
    for x0 in x0s[1:]:
        static_x0.copy_(x0)
        graph.replay()
        want = ctrl(x0, cost, dx)
        torch.cuda.synchronize()
        for a, b in zip(out, want):
            assert torch.equal(a, b), float((a - b).abs().max())


def test_cuda_graph_capture_linear():
    B, T, n, m = 32, 10, 8, 2
    C, c, F, f, x0 = _linear(B, T, n, m, torch.float32, seed=17)
    ctrl = MPC(n, m, T, u_lower=-0.25, u_upper=0.25, lqr_iter=10, verbose=-1, exit_unconverged=False,
               detach_unconverged=False)
    u0 = torch.zeros(T, B, m, device=DEV)
    assert solver._use_device_loop(ctrl, x0, QuadCost(C, c), LinDx(F, f), u0)
    _capture_matches_eager(ctrl, QuadCost(C, c), LinDx(F, f), [x0, 0.5 * x0, x0.flip(0)])


def test_cuda_graph_capture_cartpole():
    # CPU parameters: nothing to read back.  Pinned, because the differentiable tail of MPC.forward evaluates the
    # Module itself, and torch copies only pinned host memory inside a capture.
    sysdx = CartpoleDx(params=torch.tensor((9.8, 1.0, 0.1, 0.5)).pin_memory())
    B, T = 32, 15
    x0, cost = _system_problem(sysdx, B, T, torch.float32)
    ctrl = _system_mpc(sysdx, T, 20)()
    _capture_matches_eager(ctrl, cost, sysdx, [x0, x0.flip(0), initial_states(B, seed=3).to(DEV)])


def test_eager_device_loop_makes_no_host_sync():
    B, T, n, m = 32, 10, 8, 2
    C, c, F, f, x0 = _linear(B, T, n, m, torch.float32, seed=19)
    ctrl = MPC(n, m, T, u_lower=-0.25, u_upper=0.25, lqr_iter=10, verbose=-1, exit_unconverged=False,
               detach_unconverged=False)
    with torch.no_grad():                                       # first calls: library load and kernel set-up
        ctrl(x0, QuadCost(C, c), LinDx(F, f))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        with torch.no_grad():
            ctrl(x0, QuadCost(C, c), LinDx(F, f))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
