"""GPU: a learned model's kernels (csrc/mlp.cu) against the float64 oracle (oracle/mlp_oracle.py), and MPC.forward
with an NNDynamics on the device loop (mpcb200_ilqr_mlp_*) against the host loop, the reference's fixtures and its
own batch.  Every output buffer of a direct call starts at NaN, so an element a kernel does not write fails.

Tolerances: float64 1e-12 relative for the network's rollout and Jacobians (sums in another order than torch's);
float32 under gpu_harness.within (a float32 evaluation of the oracle sets the scale).  The line search and the loops
are compared at the step's own tolerance (gpu_harness.tol_for)."""
import contextlib
import ctypes

import pytest
import torch

from mpc.pytorch_b200 import _lib, mlp as mlpmod, solver
from mpc.pytorch_b200._lib import _on_device, stream_handle
from mpc.pytorch_b200.models import NNDynamics
from mpc.pytorch_b200.solver import MPC, CtrlPassthroughDynamics, GradMethods, QuadCost
from mpc.pytorch_b200.step import reference_full_du_norm
from oracle import lqr_oracle as lo
from oracle import mlp_oracle as mo
from tests.gpu_harness import F32, F64, tol_for, within
from tests.helpers import build_net, load_golden, maxdiff

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
ACTS = ("sigmoid", "relu", "elu")


def _network(n, m, hidden, act, passthrough, seed):
    torch.manual_seed(seed)
    net = NNDynamics(n, m, hidden_sizes=hidden, activation=act, passthrough=passthrough).double()
    with torch.no_grad():
        for fc in net.fcs:
            fc.weight.mul_(1.5)
    return net


def _states(seed, T, B, n, m):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(T, B, n, generator=g, dtype=torch.float64), torch.randn(T, B, m, generator=g,
                                                                               dtype=torch.float64)


def _nan(*shape, dtype):
    return torch.full(shape, float("nan"), dtype=dtype, device=DEV)


GRID = [((), "sigmoid", True), ((12,), "relu", False), ((100,), "elu", True), ((12, 100), "sigmoid", False),
        ((12, 12, 12), "relu", True), ((256,), "sigmoid", True), ((100, 12), "elu", False), ((256,), "relu", False)]


@pytest.mark.parametrize("dtype", [F64, F32])
@pytest.mark.parametrize("pad", [(0, 0), (2, 1)])
@pytest.mark.parametrize("hidden,act,passthrough", GRID)
def test_rollout_and_linearisation_match_the_oracle(hidden, act, passthrough, pad, dtype):
    n, m, T, B = 4, 2, 6, 37                       # B: not a multiple of a CTA's warps
    net = _network(n, m, hidden, act, passthrough, seed=len(hidden) * 7 + len(act))
    layers = mo.layers_of(net)
    if dtype == F32:
        layers = [(W.float().double(), b.float().double()) for W, b in layers]
    xs, us = _states(3, T, B, n, m)
    xs, us = xs.to(dtype).double(), us.to(dtype).double()
    want_x = mo.rollout(layers, act, passthrough, xs[0], us)
    want_F, want_f = mo.linearize(layers, act, passthrough, xs, us)
    w32 = None
    if dtype == F32:
        l32 = [(W.float(), b.float()) for W, b in layers]
        w32 = (mo.rollout(l32, act, passthrough, xs[0].float(), us.float()),
               *mo.linearize(l32, act, passthrough, xs.float(), us.float()))
    N, M = n + pad[0], m + pad[1]
    net_d = net.to(dtype=dtype, device=DEV)
    rec, buf = mlpmod.record(net_d, torch.empty(0, dtype=dtype, device=DEV))
    x0 = torch.zeros(B, N, dtype=dtype, device=DEV)
    x0[:, :n] = xs[0].to(dtype)
    u_ = torch.zeros(T, B, M, dtype=dtype, device=DEV)
    u_[:, :, :m] = us.to(dtype)
    x_ = torch.zeros(T, B, N, dtype=dtype, device=DEV)
    x_[:, :, :n] = xs.to(dtype)
    xo, Fo, fo = _nan(T, B, N, dtype=dtype), _nan(T - 1, B, N, N + M, dtype=dtype), _nan(T - 1, B, N, dtype=dtype)
    sfx = "f64" if dtype == F64 else "f32"
    L = _lib.lib()
    with _on_device(DEV):
        assert getattr(L, "mpcb200_mlp_rollout_" + sfx)(ctypes.byref(rec), B, T, N, M, _lib.ptr(x0), _lib.ptr(u_),
                                                        _lib.ptr(xo), stream_handle(DEV)) == 0
        assert getattr(L, "mpcb200_mlp_linearize_" + sfx)(ctypes.byref(rec), B, T, N, M, _lib.ptr(x_), _lib.ptr(u_),
                                                          _lib.ptr(Fo), _lib.ptr(fo), stream_handle(DEV)) == 0
    torch.cuda.synchronize()
    xo, Fo, fo = xo.cpu(), Fo.cpu(), fo.cpu()
    assert not xo[:, :, n:].any() and not fo[:, :, n:].any() and not Fo[:, :, n:].any()    # padding written as 0
    assert not Fo[:, :, :, n:N].any() and not Fo[:, :, :, N + m:].any()
    got_F = torch.cat((Fo[:, :, :n, :n], Fo[:, :, :n, N:N + m]), 3)
    tag = f"{hidden} {act} pt={passthrough} pad={pad}"
    for what, got, w64, i in (("x", xo[:, :, :n], want_x, 0), ("F", got_F, want_F, 1), ("f", fo[:, :, :n], want_f, 2)):
        within(tag, what, got, w64, None if w32 is None else w32[i].double(), dtype, tol64=1e-12)


def _ls_case(seed, T, B, n, m, mode, n_prev=0):
    """A step problem around a rolled-out nominal trajectory of a strongly curved network (weights x 8, nominal controls
    of unit scale), so that the full step (alpha = 1) overshoots for several problems and the line search backtracks
    (float64): (net, layers, kw, x0, C, c, x, u)."""
    torch.manual_seed(seed)
    net = NNDynamics(n - n_prev, m, hidden_sizes=(12,), activation="sigmoid").double()
    with torch.no_grad():
        for fc in net.fcs:
            fc.weight.mul_(8.0)
    layers = mo.layers_of(net)
    g = torch.Generator().manual_seed(seed)
    p = n + m
    Lc = torch.randn(T, B, p, p, generator=g, dtype=torch.float64) / p ** 0.5
    C = Lc @ Lc.transpose(-1, -2) + 0.5 * torch.eye(p, dtype=torch.float64)
    c = 2.0 * torch.randn(T, B, p, generator=g, dtype=torch.float64)
    x0 = torch.randn(B, n, generator=g, dtype=torch.float64)
    u = torch.randn(T, B, m, generator=g, dtype=torch.float64)
    kw = {}
    if mode in ("box", "boxD"):
        kw = dict(u_lower=-1.5, u_upper=1.5)
        u = u.clamp(-1.5, 1.5)
    if mode == "tensor":
        lo_ = -0.5 - torch.rand(T, B, m, generator=g, dtype=torch.float64)
        kw = dict(u_lower=lo_, u_upper=lo_ + 2.0)
        u = torch.maximum(torch.minimum(u, lo_ + 2.0), lo_)
    if mode == "boxD":
        kw["delta_u"] = 0.8
    if mode == "mask":
        kw = dict(u_zero_I=(torch.rand(T, B, m, generator=g) < 0.3).to(torch.float64))
    x = mo.rollout(layers, "sigmoid", True, x0, u, n_prev)
    return net, layers, kw, x0, C, c, x, u


@contextlib.contextmanager
def poisoned():
    """torch.empty fills what it returns: NaN for floating tensors, every bit set otherwise (a byte workspace then reads
    as NaN), so an output or workspace element a kernel does not write before reading fails the comparison."""
    real = torch.empty

    def empty(*a, **k):
        t = real(*a, **k)
        return t.fill_(float("nan")) if t.is_floating_point() else t.fill_(255 if t.dtype == torch.uint8 else -1)
    torch.empty = empty
    try:
        yield
    finally:
        torch.empty = real


@pytest.mark.parametrize("decay", [0.5, 0.3])
@pytest.mark.parametrize("max_ls", [1, 3, 10])
@pytest.mark.parametrize("mode", ["free", "box", "tensor", "boxD", "mask"])
@pytest.mark.parametrize("n_prev", [0, 2])
def test_line_search_matches_the_oracle(max_ls, mode, n_prev, decay):
    """mpcb200_mlp_step_* against lqr_step_forward with the network as the rollout's dynamics, on problems whose full
    step is worse for several problems: alpha decays per problem while the cost is worse, for at most max_ls passes,
    and a last pass still worse ends with alpha /= decay (the reference's lqr_step.py:252)."""
    T, B, m = 10, 48, 2
    n = 3 + n_prev
    net, layers, kw, x0, C, c, x, u = _ls_case(5, T, B, n, m, mode, n_prev)
    F, f = mo.linearize(layers, "sigmoid", True, x, u, n_prev)
    trace = []
    want = lo.lqr_step_forward(n, m, T, x0, C, c, F, f, x, u, dynamics=lambda a, b: mo.step(
        layers, "sigmoid", True, a, b, n_prev), max_linesearch_iter=max_ls, linesearch_decay=decay, ls_trace=trace,
        coupled=False, **kw)
    # the case exercises what it is meant to: repeat passes, decayed alphas, and problems still worse at the limit
    worse = [int((t > 0).sum()) for t in trace]
    assert worse[0] > 0, worse
    if max_ls > 1:
        assert len(trace) >= 2 and bool((want.alphas < 1).any()), worse
    if max_ls == 1 or (mode == "mask" and (max_ls == 3 or decay == 0.3)):
        assert len(trace) == max_ls and worse[-1] > 0, worse      # ends on the limit with problems still worse
    net_d = net.to(DEV)
    dx = CtrlPassthroughDynamics(net_d) if n_prev else net_d
    d = {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in kw.items()}
    with poisoned():
        got = mlpmod.step_raw(dx, n, m, T, x0.to(DEV), C.to(DEV), c.to(DEV), F.to(DEV), f.to(DEV), x.to(DEV),
                              u.to(DEV), max_linesearch_iter=max_ls, linesearch_decay=decay, **d)
    bounded = "u_lower" in kw
    tol = 2e-6 if bounded else tol_for(F64, False)["xu"]    # bounded: pnqp's stopping rule, per problem vs batched
    sc = max(1.0, float(want.new_x.abs().max()))
    assert maxdiff(got["new_u"], want.new_u) < tol * sc and maxdiff(got["new_x"], want.new_x) < tol * sc
    assert maxdiff(got["costs"], want.costs) < tol * max(1.0, float(want.costs.abs().max()))
    assert maxdiff(reference_full_du_norm(got["du_first"]), want.full_du_norm) < tol * sc
    if bounded:
        assert maxdiff(got["alphas"], want.alphas) < 1e-12
        lo_, hi_ = kw["u_lower"], kw["u_upper"]
        on = (want.new_u == lo_) | (want.new_u == hi_)
        gu = got["new_u"].cpu()
        assert torch.equal(on, (gu == lo_) | (gu == hi_))
    else:
        assert torch.equal(got["alphas"].cpu(), want.alphas)       # the same decisions and the same arithmetic
    if n_prev:
        assert torch.equal(got["new_x"][1:, :, :n_prev].cpu(), got["new_u"][:-1].cpu())


def _solve(g, net, bound, eps=1e-6, lqr_iter=12, host=False, **kw):
    T = g["C"].shape[0]
    box = {} if bound is None else dict(u_lower=-bound, u_upper=bound)
    ctrl = MPC(3, 2, T, **box, lqr_iter=lqr_iter, verbose=-1, grad_method=GradMethods.ANALYTIC,
               exit_unconverged=False, detach_unconverged=False, eps=eps, **kw)
    x0, cost = g["x_init"].to(DEV), QuadCost(g["C"].to(DEV), g["c"].to(DEV))
    if host:
        T, B = ctrl.T, x0.shape[0]
        from mpc.pytorch_b200.dynamics import params_scope
        with params_scope(), torch.no_grad():
            best = ctrl._ilqr_host(x0, cost, net, torch.zeros(T, B, 2, dtype=x0.dtype, device=DEV))
        return best["x"], best["u"], best["costs"], int(best["info"][0])
    assert solver._use_device_loop(ctrl, x0, cost, net, torch.zeros(T, x0.shape[0], 2, device=DEV, dtype=x0.dtype))
    with torch.no_grad(), poisoned():
        x, u, costs = ctrl(x0, cost, net)
    return x, u, costs, int(ctrl._solve_info[0])


class TorchNet(NNDynamics):
    """NNDynamics by another name: MPC runs it as any Module (its forward and grad_input in torch, the line search in
    step.rollout_split), the path every NNDynamics took before the kernels."""


def _torch_copy(net):
    t = TorchNet(net.n_state, net.n_ctrl, hidden_sizes=[fc.out_features for fc in net.fcs[:-1]],
                 activation=net.activation, passthrough=net.passthrough).to(dtype=net.fcs[0].weight.dtype, device=DEV)
    t.load_state_dict(net.state_dict())
    return t


@pytest.mark.parametrize("act", ["sigmoid", "relu"])
@pytest.mark.parametrize("bound", [None, 0.6])
def test_device_loop_matches_the_torch_host_loop(act, bound, monkeypatch):
    """The device loop (mpcb200_ilqr_mlp_*) against the host loop with the network in torch: get_traj's Module calls,
    grad_input and rollout_split, none of the network's kernels.  eps = 0 and a large not_improved_lim, so both run
    all lqr_iter iterations.  Unbounded to 1e-10 of max|x| (float64), or to ten times what the solve itself makes of
    a 1e-15 relative change of x_init where that is more: the sigmoid fixture's 12 iterations turn it into 4e-10 of x
    and 7e-9 of u in the float64 oracle alone, so no two implementations that sum in different orders agree closer.
    Bounded at pnqp's stopping rule with the same controls on the bounds."""
    g = load_golden(f"nn_dynamics_{act}_f64")
    net = build_net(g, act).to(DEV)
    kw = dict(eps=0.0, lqr_iter=12, not_improved_lim=100)
    xd, ud, cd, itd = _solve(g, net, bound, **kw)
    for name in ("rollout_raw", "linearize_raw", "step_raw", "ilqr_raw"):
        monkeypatch.setattr(mlpmod, name, lambda *a, _n=name, **k: pytest.fail(f"the torch path ran mlp.{_n}"))
    xh, uh, ch, ith = _solve(g, _torch_copy(net), bound, host=True, **kw)
    assert itd == ith == 12
    sc = max(1.0, float(xh.abs().max()))
    if bound is None:
        tol_x = tol_u = 1e-10 * sc
        layers = mo.layers_of(net)
        tol_c = 1e-10 * max(1.0, float(ch.abs().max()))
        one = [mo.ilqr(3, 2, g["C"].shape[0], x0, g["C"], g["c"], layers, act, True, **kw)[:3]
               for x0 in (g["x_init"], g["x_init"] * (1 + 1e-15))]
        tol_x = max(tol_x, 10 * maxdiff(one[0][0], one[1][0]))
        tol_u = max(tol_u, 10 * maxdiff(one[0][1], one[1][1]))
        tol_c = max(tol_c, 10 * maxdiff(one[0][2], one[1][2]))
    else:
        tol_x = tol_u = 2e-4 * sc
        tol_c = 1e-5 * max(1.0, float(ch.abs().max()))
    assert maxdiff(xd, xh) < tol_x and maxdiff(ud, uh) < tol_u, (maxdiff(xd, xh), tol_x, maxdiff(ud, uh), tol_u)
    assert maxdiff(cd, ch) < tol_c, (maxdiff(cd, ch), tol_c)
    if bound is not None:
        assert torch.equal(ud.abs() == bound, uh.abs() == bound)


@pytest.mark.parametrize("act", ["sigmoid", "relu"])
def test_device_loop_matches_the_reference_fixture(act):
    g = load_golden(f"nn_dynamics_{act}_f64")
    net = build_net(g, act).to(DEV)
    x, u, costs, _ = _solve(g, net, 0.6)
    sc = max(1.0, float(g["x"].abs().max()))
    assert maxdiff(u, g["u"]) < 2e-4 and maxdiff(x, g["x"]) < 2e-4 * sc
    assert maxdiff(costs, g["costs"]) < 1e-5 * max(1.0, float(g["costs"].abs().max()))
    x, u, costs, _ = _solve(g, net, None)
    sc = max(1.0, float(g["x_free"].abs().max()))
    assert maxdiff(u, g["u_free"]) < 1e-7 * sc and maxdiff(x, g["x_free"]) < 1e-7 * sc


def test_slew_gradients_through_the_device_forward():
    """nn_grad_slew_f64: d u* / d c through MPC.forward whose iterations ran on mpcb200_ilqr_mlp_* (n_prev = m)."""
    from mpc.dynamics import NNDynamics as Net
    g = load_golden("nn_grad_slew_f64")
    nl = int(g["n_layers"])
    net = Net(2, 2, hidden_sizes=[g[f"W{i}"].shape[0] for i in range(nl - 1)], activation="sigmoid").double()
    with torch.no_grad():
        for i, fc in enumerate(net.fcs):
            fc.weight.copy_(g[f"W{i}"])
            fc.bias.copy_(g[f"b{i}"])
    net = net.to(DEV)
    T = g["C"].shape[0]
    c = g["c"].to(DEV).requires_grad_(True)
    ctrl = MPC(2, 2, T, u_lower=-1.0, u_upper=1.0, lqr_iter=40, verbose=-1, exit_unconverged=False,
               max_linesearch_iter=1, slew_rate_penalty=1.0, grad_method=GradMethods.ANALYTIC)
    x0, cost = g["x_init"].to(DEV), QuadCost(g["C"].to(DEV), c)
    assert solver._use_slew_device_loop(ctrl, x0, cost, net, torch.zeros(T, 1, 2, dtype=x0.dtype, device=DEV))
    calls = []
    orig = mlpmod.ilqr_raw

    def spy(*a, **k):
        calls.append(1)
        return orig(*a, **k)
    mlpmod.ilqr_raw = spy
    try:
        x, u, _ = ctrl(x0, cost, net)
    finally:
        mlpmod.ilqr_raw = orig
    assert calls
    assert maxdiff(u, g["u"]) < 2e-4
    uf = u.reshape(-1)
    rows = [torch.autograd.grad(uf[i], c, retain_graph=True)[0].reshape(-1) for i in range(uf.numel())]
    Jc = torch.stack(rows)
    assert maxdiff(Jc, g["du_dc"]) < 2e-3 * float(g["du_dc"].abs().max())


def test_batch_independence_and_capture():
    """A problem's solve is bitwise the same alone and at any position of a batch; the loop runs inside a caller's
    CUDA graph capture with no host read."""
    g = load_golden("nn_dynamics_sigmoid_f64")
    net = build_net(g, "sigmoid").to(DEV)
    T = g["C"].shape[0]
    opts = dict(u_lower=-0.6, u_upper=0.6, lqr_iter=12, verbose=-1, exit_unconverged=False, detach_unconverged=False,
                eps=0.0, not_improved_lim=100)     # every solve runs all 12 iterations, whatever its batch
    ctrl = MPC(3, 2, T, **opts)
    x0, C, c = g["x_init"].to(DEV), g["C"].to(DEV), g["c"].to(DEV)
    with torch.no_grad(), poisoned():
        x, u, _ = ctrl(x0, QuadCost(C, c), net)
        perm = torch.tensor([2, 0, 3, 1], device=DEV)
        xp, up, _ = ctrl(x0[perm], QuadCost(C[:, perm], c[:, perm]), net)
        assert torch.equal(xp, x[:, perm]) and torch.equal(up, u[:, perm])
        for b in range(4):
            one = MPC(3, 2, T, **opts)
            x1, u1, _ = one(x0[b:b + 1], QuadCost(C[:, b:b + 1], c[:, b:b + 1]), net)
            assert int(one._solve_info[0]) == int(ctrl._solve_info[0]) == 12
            assert torch.equal(x1, x[:, b:b + 1]) and torch.equal(u1, u[:, b:b + 1])
    from mpc.pytorch_b200.mlp import ilqr_raw
    u0 = torch.zeros(T, 4, 2, dtype=x0.dtype, device=DEV)
    kw = dict(u_lower=-0.6, u_upper=0.6, lqr_iter=12, eps=1e-6)
    ref = ilqr_raw(net, 3, 2, T, x0, C, c, u0, **kw)
    s = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            res = ilqr_raw(net, 3, 2, T, x0, C, c, u0, **kw)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(res["x"], ref["x"]) and torch.equal(res["u"], ref["u"])


def test_graph_refused_falls_back_to_the_host_loop(monkeypatch):
    g = load_golden("nn_dynamics_sigmoid_f64")
    net = build_net(g, "sigmoid").to(DEV)
    monkeypatch.setattr(mlpmod, "ilqr_raw", lambda *a, **k: None)
    monkeypatch.setattr(solver, "_graph_cond_unavailable", False)
    T = g["C"].shape[0]
    ctrl = MPC(3, 2, T, lqr_iter=12, verbose=-1, exit_unconverged=False, detach_unconverged=False, eps=1e-6)
    with torch.no_grad():
        x, u, _ = ctrl(g["x_init"].to(DEV), QuadCost(g["C"].to(DEV), g["c"].to(DEV)), net)
    assert solver._graph_cond_unavailable
    monkeypatch.setattr(solver, "_graph_cond_unavailable", False)
    sc = max(1.0, float(g["x_free"].abs().max()))
    assert maxdiff(u, g["u_free"]) < 1e-7 * sc
