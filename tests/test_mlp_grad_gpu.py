"""GPU: the gradient of a learned model's linearisation in its weights (mpcb200_mlp_linearize_vjp_*, csrc/mlp.cu)
against the float64 oracle (oracle/mlp_grad_oracle.py), its bitwise repeatability, and MPC.forward + backward() to
every weight and bias through MlpLinearize against the torch tail and the reference's fixtures.  Every output and the
workspace of a direct call start at NaN, so an element a kernel does not write fails.

Tolerances (DESIGN.md section 3.11): float64 1e-11 of max|dtheta|; float32 2e-4 of max|dtheta| (the inputs are
rounded through float32 first, so only the kernel's float32 arithmetic is measured)."""
import ctypes

import pytest
import torch

from mpc.pytorch_b200 import _lib, mlp as mlpmod
from mpc.pytorch_b200._lib import _on_device, stream_handle
from mpc.pytorch_b200.models import NNDynamics
from mpc.pytorch_b200.solver import MPC, GradMethods, QuadCost
from oracle import mlp_grad_oracle as mgo
from oracle import mlp_oracle as mo
from tests.gpu_harness import F32, F64
from tests.helpers import load_golden, maxdiff

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")

# (widths, B, T) with more items than slots and more slots than the VJP kernel's warps (test_mlp_grad_cpu.py)
GRID_CASE = ((6, 12, 4), 700, 5)


def _network(n, m, hidden, act, passthrough, seed, dtype=F64):
    torch.manual_seed(seed)
    net = NNDynamics(n, m, hidden_sizes=hidden, activation=act, passthrough=passthrough).double()
    with torch.no_grad():
        for fc in net.fcs:
            fc.weight.mul_(1.5)
        if act == "relu" and hidden:             # a hidden unit whose pre-activation is exactly 0 at every item
            net.fcs[0].weight[0].zero_()
            net.fcs[0].bias[0] = 0.0
    return net.to(dtype).double()


def _nan(*shape, dtype):
    return torch.full(shape, float("nan"), dtype=dtype, device=DEV)


def _inputs(seed, T, B, N, M, dtype):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g, dtype=F64).to(dtype)       # noqa: E731
    return r(T, B, N), r(T, B, M), r(T - 1, B, N, N + M), r(T - 1, B, N)


def _call(net, n_prev, B, T, N, M, x, u, dF, df, dtype, stream=None):
    """dtheta of mpcb200_mlp_linearize_vjp_* on inputs already on the device, with a NaN workspace and output."""
    buf = torch.cat([t.detach().reshape(-1) for fc in net.fcs for t in (fc.weight, fc.bias)]).to(DEV, dtype)
    rec = mlpmod._record(net, n_prev, buf.data_ptr())
    nbytes = _lib.lib().mpcb200_mlp_linearize_vjp_workspace_bytes(ctypes.byref(rec), B, T, buf.element_size())
    assert nbytes > 0
    ws = torch.full((nbytes // buf.element_size(),), float("nan"), dtype=dtype, device=DEV)
    out = _nan(buf.numel(), dtype=dtype)
    sfx = "f64" if dtype == F64 else "f32"
    st = stream if stream is not None else torch.cuda.current_stream(DEV)
    with _on_device(DEV), torch.cuda.stream(st):
        rc = getattr(_lib.lib(), "mpcb200_mlp_linearize_vjp_" + sfx)(
            ctypes.byref(rec), B, T, N, M, _lib.ptr(x), _lib.ptr(u), _lib.ptr(dF), _lib.ptr(df), _lib.ptr(out),
            _lib.ptr(ws), nbytes, stream_handle(DEV))
    assert rc == 0
    return out, (rec, buf, ws, nbytes)


def _want(net, act, pt, n_prev, n, m, x, u, dF, df):
    """The oracle's dtheta on the network's own block of the staged inputs, packed W0 b0 W1 b1 ..."""
    N = n_prev + n
    xs, us = x[:, :, :N].double().cpu(), u[:, :, :m].double().cpu()
    Nst = x.shape[2]
    dF_ = torch.cat((dF[:, :, :N, :N], dF[:, :, :N, Nst:Nst + m]), 3).double().cpu()
    g = mgo.linearize_vjp(mo.layers_of(net), act, pt, xs, us, dF_, df[:, :, :N].double().cpu(), n_prev)
    return torch.cat([t.reshape(-1) for wb in g for t in wb])


GRID = [((), "sigmoid", True), ((12,), "relu", False), ((31,), "elu", True), ((33,), "sigmoid", False),
        ((12, 100), "relu", True), ((12, 12, 12), "elu", False), ((100, 12, 40), "sigmoid", True),
        ((256,), "sigmoid", True), ((256,), "relu", False), ((64, 256), "elu", True)]


@pytest.mark.parametrize("dtype", [F64, F32])
@pytest.mark.parametrize("pad", [(0, 0, 0), (2, 1, 0), (0, 0, 2)])
@pytest.mark.parametrize("hidden,act,passthrough", GRID)
def test_vjp_matches_the_oracle(hidden, act, passthrough, pad, dtype):
    """pad = (extra states, extra controls, n_prev): padded N > n and M > m and the previous-control rows, with
    non-zero cotangents everywhere, padding included."""
    n, m, T, B = 4, 2, 5, 37
    n_prev = pad[2]
    net = _network(n, m, hidden, act, passthrough, seed=len(hidden) * 7 + len(act), dtype=dtype)
    N, M = n_prev + n + pad[0], m + pad[1]
    x, u, dF, df = (t.to(DEV) for t in _inputs(3, T, B, N, M, dtype))
    if n_prev:
        x[1:, :, :n_prev] = u[:-1, :, :m]
    got, _ = _call(net, n_prev, B, T, N, M, x, u, dF, df, dtype)
    want = _want(net, act, passthrough, n_prev, n, m, x, u, dF, df)
    sc = float(want.abs().max())
    err = maxdiff(got.cpu(), want)
    assert err <= (1e-11 if dtype == F64 else 2e-4) * sc, (err, sc)


@pytest.mark.parametrize("dtype", [F64, F32])
def test_grid_case_second_item_per_slot_and_second_slot_per_warp(dtype):
    widths, B, T = GRID_CASE
    n, m = widths[-1], widths[0] - widths[-1]
    net = _network(n, m, tuple(widths[1:-1]), "sigmoid", True, seed=11, dtype=dtype)
    x, u, dF, df = (t.to(DEV) for t in _inputs(5, T, B, n, m, dtype))
    got, _ = _call(net, 0, B, T, n, m, x, u, dF, df, dtype)
    want = _want(net, "sigmoid", True, 0, n, m, x, u, dF, df)
    sc = float(want.abs().max())
    assert maxdiff(got.cpu(), want) <= (1e-11 if dtype == F64 else 2e-4) * sc


@pytest.mark.parametrize("dtype", [F64, F32])
def test_bitwise_repeatable_across_calls_graphs_and_streams(dtype):
    widths, B, T = GRID_CASE
    n, m = widths[-1], widths[0] - widths[-1]
    net = _network(n, m, (40,), "elu", True, seed=3, dtype=dtype)
    x, u, dF, df = (t.to(DEV) for t in _inputs(9, T, B, n, m, dtype))
    a, (rec, buf, ws, nbytes) = _call(net, 0, B, T, n, m, x, u, dF, df, dtype)
    b, _ = _call(net, 0, B, T, n, m, x, u, dF, df, dtype)
    s2 = torch.cuda.Stream(DEV)
    c, _ = _call(net, 0, B, T, n, m, x, u, dF, df, dtype, stream=s2)
    torch.cuda.synchronize()
    assert torch.equal(a, b) and torch.equal(a, c)
    out = _nan(buf.numel(), dtype=dtype)
    ws.fill_(float("nan"))
    fn = getattr(_lib.lib(), "mpcb200_mlp_linearize_vjp_" + ("f64" if dtype == F64 else "f32"))
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream(DEV)
    torch.cuda.synchronize()
    with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
        assert fn(ctypes.byref(rec), B, T, n, m, _lib.ptr(x), _lib.ptr(u), _lib.ptr(dF), _lib.ptr(df), _lib.ptr(out),
                  _lib.ptr(ws), nbytes, stream_handle(DEV)) == 0
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, a)


def test_t1_writes_zero():
    net = _network(3, 2, (12,), "sigmoid", True, seed=1)
    x, u = torch.zeros(1, 4, 3, dtype=F64, device=DEV), torch.zeros(1, 4, 2, dtype=F64, device=DEV)
    e = torch.zeros(1, dtype=F64, device=DEV)
    got, _ = _call(net, 0, 4, 1, 3, 2, x, u, e, e, F64)
    torch.cuda.synchronize()
    assert not got.any()


# ------------------------------------------------------------------------------------------------------------------
# MPC.forward + backward() to every weight and bias
# ------------------------------------------------------------------------------------------------------------------
def _mpc_case(act, gm, bound, slew, dtype=F64, seed=0, B=4, T=8, n=3, m=2, hidden=(12, 10)):
    torch.manual_seed(seed)
    net = NNDynamics(n, m, hidden_sizes=hidden, activation=act).to(DEV, dtype)
    g = torch.Generator().manual_seed(seed)
    p = n + m
    Lc = torch.randn(T, B, p, p, generator=g, dtype=F64) / p ** 0.5
    C = (Lc @ Lc.transpose(-1, -2) + torch.eye(p, dtype=F64)).to(DEV, dtype)
    c = torch.randn(T, B, p, generator=g, dtype=F64).to(DEV, dtype)
    x0 = torch.randn(B, n, generator=g, dtype=F64).to(DEV, dtype)
    box = {} if bound is None else dict(u_lower=-bound, u_upper=bound)
    ctrl = MPC(n, m, T, **box, lqr_iter=8, verbose=-1, exit_unconverged=False, detach_unconverged=False,
               grad_method=gm, slew_rate_penalty=slew)
    return net, ctrl, x0, QuadCost(C, c)


def _grads(net, ctrl, x0, cost, create_graph=False):
    x, u, _ = ctrl(x0, cost, net)
    loss = (x ** 2).sum() + (u * torch.linspace(0.5, 1.5, u.shape[-1], device=DEV, dtype=u.dtype)).sum()
    params = [t for fc in net.fcs for t in (fc.weight, fc.bias)]
    g = torch.autograd.grad(loss, params, create_graph=create_graph)
    return x.detach(), u.detach(), g


def _torch_tail(monkeypatch):
    monkeypatch.setattr(mlpmod, "linearize_diff", lambda *a, **k: None)


@pytest.mark.parametrize("gm", [GradMethods.ANALYTIC, GradMethods.AUTO_DIFF])
@pytest.mark.parametrize("bound", [None, 0.6])
@pytest.mark.parametrize("slew", [None, 0.5])
def test_mpc_gradients_match_the_torch_tail(gm, bound, slew, monkeypatch):
    net, ctrl, x0, cost = _mpc_case("sigmoid", gm, bound, slew)
    calls = []
    orig = mlpmod.MlpLinearize.apply
    monkeypatch.setattr(mlpmod.MlpLinearize, "apply", lambda *a: calls.append(1) or orig(*a))
    xk, uk, gk = _grads(net, ctrl, x0, cost)
    assert calls
    _torch_tail(monkeypatch)
    xt, ut, gt = _grads(net, ctrl, x0, cost)
    assert torch.equal(xk, xt) and torch.equal(uk, ut)
    sc = max(float(t.abs().max()) for t in gt)
    assert sc > 0
    for a, b in zip(gk, gt):
        assert maxdiff(a, b) <= 1e-12 * sc, (maxdiff(a, b), sc)


@pytest.mark.parametrize("act", ["relu", "elu"])
def test_mpc_gradients_match_the_torch_tail_other_activations(act, monkeypatch):
    net, ctrl, x0, cost = _mpc_case(act, GradMethods.ANALYTIC, 0.6, None, seed=2)
    _, _, gk = _grads(net, ctrl, x0, cost)
    _torch_tail(monkeypatch)
    _, _, gt = _grads(net, ctrl, x0, cost)
    sc = max(float(t.abs().max()) for t in gt)
    for a, b in zip(gk, gt):
        assert maxdiff(a, b) <= 1e-12 * sc


@pytest.mark.parametrize("name,slew", [("nn_grad_f64", None), ("nn_grad_slew_f64", 1.0)])
def test_reference_fixture_du_db0(name, slew):
    """d u* / d b0 through MPC.forward, whose differentiable tail ran MlpLinearize, against the reference's autograd."""
    from mpc.dynamics import NNDynamics as Net
    g = load_golden(name)
    nl = int(g["n_layers"])
    net = Net(2, 2, hidden_sizes=[g[f"W{i}"].shape[0] for i in range(nl - 1)], activation="sigmoid").double()
    with torch.no_grad():
        for i, fc in enumerate(net.fcs):
            fc.weight.copy_(g[f"W{i}"])
            fc.bias.copy_(g[f"b{i}"])
    net = net.to(DEV)
    T = g["C"].shape[0]
    ctrl = MPC(2, 2, T, u_lower=-1.0, u_upper=1.0, lqr_iter=40, verbose=-1, exit_unconverged=False,
               max_linesearch_iter=1, slew_rate_penalty=slew, grad_method=GradMethods.ANALYTIC)
    calls = []
    orig = mlpmod.MlpLinearize.apply
    mlpmod.MlpLinearize.apply = lambda *a: calls.append(1) or orig(*a)
    try:
        x, u, _ = ctrl(g["x_init"].to(DEV), QuadCost(g["C"].to(DEV), g["c"].to(DEV)), net)
    finally:
        mlpmod.MlpLinearize.apply = orig
    assert calls
    b0 = net.fcs[0].bias
    uf = u.reshape(-1)
    J = torch.stack([torch.autograd.grad(uf[i], b0, retain_graph=True)[0].reshape(-1) for i in range(uf.numel())])
    want = g["du_db0"].reshape(J.shape)
    assert maxdiff(J, want) < 2e-3 * float(want.abs().max())


def test_second_order_gradient_matches_the_torch_tail(monkeypatch):
    net, ctrl, x0, cost = _mpc_case("sigmoid", GradMethods.ANALYTIC, None, None, seed=6)

    def second():
        _, _, g = _grads(net, ctrl, x0, cost, create_graph=True)
        s = sum((t ** 2).sum() for t in g)
        return torch.autograd.grad(s, net.fcs[0].weight)[0]
    a = second()
    _torch_tail(monkeypatch)
    b = second()
    assert maxdiff(a, b) <= 1e-12 * float(b.abs().max())


def test_editing_a_weight_in_place_between_forward_and_backward_raises():
    net, ctrl, x0, cost = _mpc_case("sigmoid", GradMethods.ANALYTIC, 0.6, None, seed=8)
    x, u, _ = ctrl(x0, cost, net)
    with torch.no_grad():
        net.fcs[1].weight.add_(0.1)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        (x.sum() + u.sum()).backward()


def test_grad_disabled_builds_no_graph(monkeypatch):
    net, ctrl, x0, cost = _mpc_case("sigmoid", GradMethods.ANALYTIC, 0.6, None, seed=9)
    monkeypatch.setattr(mlpmod.MlpLinearize, "apply", lambda *a: pytest.fail("MlpLinearize under no_grad"))
    with torch.no_grad():
        x, u, _ = ctrl(x0, cost, net)
    assert not x.requires_grad and not u.requires_grad
