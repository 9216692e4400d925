"""CPU: the gradient of a learned model's linearisation in its weights.  The float64 oracle
(oracle/mlp_grad_oracle.py) against central differences of mlp_oracle.linearize and against the closed form the VJP
kernel computes (reverse over forward with matrix tangents, DESIGN.md section 3.11); mpcb200_mlp_linearize_vjp_*'s
workspace formula, fit and status codes without a device; and which linearisations MPC's differentiable tail sends
through the kernel, decided on tensor metadata alone (FakeTensor CUDA tensors: no device, no kernel)."""
import ctypes
import os
import re

import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode

from mpc.pytorch_b200 import _lib, mlp as mlpmod
from mpc.pytorch_b200._lib import Mlp
from mpc.pytorch_b200.models import NNDynamics
from mpc.pytorch_b200.solver import MPC, GradMethods
from oracle import mlp_grad_oracle as mgo
from oracle import mlp_oracle as mo

ACTS = ("sigmoid", "relu", "elu")


def _layers(widths, seed, scale=0.8):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(b, a, generator=g, dtype=torch.float64) * scale,
             torch.randn(b, generator=g, dtype=torch.float64) * 0.3) for a, b in zip(widths[:-1], widths[1:])]


def _case(widths, seed, n_prev=0, T=3, B=4):
    n, p = widths[-1], widths[0]
    m = p - n
    g = torch.Generator().manual_seed(seed + 100)
    x = torch.randn(T, B, n_prev + n, generator=g, dtype=torch.float64)
    u = torch.randn(T, B, m, generator=g, dtype=torch.float64)
    N = n_prev + n
    dF = torch.randn(T - 1, B, N, N + m, generator=g, dtype=torch.float64)
    df = torch.randn(T - 1, B, N, generator=g, dtype=torch.float64)
    return x, u, dF, df


def _loss(layers, act, pt, x, u, dF, df, n_prev=0):
    F, f = mo.linearize(layers, act, pt, x, u, n_prev)
    return float((F * dF).sum() + (f * df).sum())


@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("widths", [(5, 3), (5, 7, 3), (4, 9, 6, 2)])
def test_oracle_is_central_differences_of_the_linearisation(act, widths):
    layers = _layers(widths, seed=len(widths))
    x, u, dF, df = _case(widths, 1)
    got = mgo.linearize_vjp(layers, act, True, x, u, dF, df)
    g = torch.Generator().manual_seed(7)
    for _ in range(3):
        v = [(torch.randn(W.shape, generator=g, dtype=torch.float64), torch.randn(b.shape, generator=g,
                                                                                  dtype=torch.float64))
             for W, b in layers]
        h = 1e-6
        plus = [(W + h * a, b + h * c) for (W, b), (a, c) in zip(layers, v)]
        minus = [(W - h * a, b - h * c) for (W, b), (a, c) in zip(layers, v)]
        fd = (_loss(plus, act, True, x, u, dF, df) - _loss(minus, act, True, x, u, dF, df)) / (2 * h)
        dot = sum(float((dW * a).sum() + (db * c).sum()) for (dW, db), (a, c) in zip(got, v))
        assert abs(fd - dot) < 1e-6 * max(1.0, abs(dot)), (fd, dot)


def _act_curv(act, h):
    if act == "sigmoid":
        return h * (1 - h) * (1 - 2 * h)
    if act == "relu":
        return torch.zeros_like(h)
    return torch.where(h > 0, torch.zeros_like(h), h + 1)


def closed_form(layers, act, x, u, dF, df, n_prev=0):
    """The kernel's formula per item (t, b), summed: forward h_{i+1} = act(W_i h_i + b_i), T_{i+1} = diag(act') W_i T_i
    from h_0 = z, T_0 = I; reverse from G^ = dJ - df z^T with A_i = W_i T_i."""
    N = dF.shape[2]
    n, p = layers[-1][0].shape[0], layers[0][0].shape[1]
    m = p - n
    z = torch.cat((x[:-1, :, n_prev:], u[:-1]), 2).reshape(-1, p)
    dFi = dF.reshape(-1, N, dF.shape[3])[:, n_prev:]
    dJ = torch.cat((dFi[:, :, n_prev:N], dFi[:, :, N:N + m]), 2)
    dfi = df.reshape(-1, N)[:, n_prev:]
    G = dJ - dfi.unsqueeze(2) * z.unsqueeze(1)
    L = len(layers)
    hs, Ts, As = [z], [torch.eye(p, dtype=z.dtype).expand(z.shape[0], p, p)], []
    for W, b in layers[:-1]:
        h = mo._ACT[act](hs[-1] @ W.t() + b)
        A = W @ Ts[-1]
        As.append(A)
        hs.append(h)
        Ts.append(mo._slope(act, h).unsqueeze(2) * A)
    W = layers[-1][0]
    out = [None] * L
    out[-1] = ((G @ Ts[-1].transpose(1, 2) + dfi.unsqueeze(2) * hs[-1].unsqueeze(1)).sum(0), dfi.sum(0))
    Tb, hb = W.t() @ G, dfi @ W
    for i in range(L - 2, -1, -1):
        W, h = layers[i][0], hs[i + 1]
        s = mo._slope(act, h)
        Ab = s.unsqueeze(2) * Tb
        ab = hb * s + (Tb * As[i]).sum(2) * _act_curv(act, h)
        out[i] = ((Ab @ Ts[i].transpose(1, 2) + ab.unsqueeze(2) * hs[i].unsqueeze(1)).sum(0), ab.sum(0))
        Tb, hb = W.t() @ Ab, ab @ W
    return out


@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("widths", [(5, 3), (5, 7, 3), (5, 40, 9, 3), (6, 40, 12, 40, 4)])
@pytest.mark.parametrize("pt,n_prev", [(True, 0), (False, 0), (True, 2)])
def test_oracle_is_the_closed_form(act, widths, pt, n_prev):
    layers = _layers(widths, seed=len(widths) + 3)
    if n_prev:
        n_prev = widths[0] - widths[-1]
    x, u, dF, df = _case(widths, 2, n_prev)
    want = mgo.linearize_vjp(layers, act, pt, x, u, dF, df, n_prev)
    got = closed_form(layers, act, x, u, dF, df, n_prev)
    for (gW, gb), (wW, wb) in zip(got, want):
        sc = max(1.0, float(wW.abs().max()))
        assert float((gW - wW).abs().max()) < 1e-12 * sc and float((gb - wb).abs().max()) < 1e-12 * sc


# ------------------------------------------------------------------------------------------------------------------
# workspace, fit and status codes, without a device
# ------------------------------------------------------------------------------------------------------------------
FAKE = 1 << 20          # a non-NULL, 256-byte aligned address that is never dereferenced: every call below fails first
LIMIT = 227 * 1024
SRC = os.path.join(os.path.dirname(__file__), "..", "mpc", "pytorch_b200", "csrc")


def _const(name):
    with open(os.path.join(SRC, "mlp.cuh")) as fh:
        m = re.search(rf"constexpr (?:long long|int) {name} = (\d+)(?:ll << (\d+))?;", fh.read())
    return int(m.group(1)) << int(m.group(2) or 0)


def _rec(widths=(5, 100, 3), act=0, n_prev=0, params=FAKE):
    r = Mlp(n_layers=len(widths) - 1, activation=act, passthrough=1, n_prev=n_prev, params=params)
    o = 0
    for i, w in enumerate(widths):
        r.width[i] = w
    for i in range(len(widths) - 1):
        r.W_off[i] = o
        o += widths[i + 1] * widths[i]
        r.b_off[i] = o
        o += widths[i + 1]
    return r


def _nparams(widths):
    return sum(widths[i + 1] * (widths[i] + 1) for i in range(len(widths) - 1))


def slots(items, n_params):
    """G: the slot count, a function of the item and parameter counts alone."""
    return max(1, min(items, _const("kMlpVjpMaxSlots"), max(1, _const("kMlpVjpSlotElems") // n_params)))


def _vjp_smem(widths, esz, warps=1):
    """An mbarrier, the parameters, and one slice per warp: z, the hidden outputs, their tangents [w_i, p], two
    adjoint buffers [maxw, p] and two [maxw]."""
    p, maxw, hidden = widths[0], max(widths), sum(widths[1:-1])
    per_warp = (p + hidden + hidden * p + 2 * maxw * p + 2 * maxw + 3) // 4 * 4
    return 16 + (_nparams(widths) * esz + 15) // 16 * 16 + warps * per_warp * esz


def _ws(widths, B, T, esz, **kw):
    return _lib.lib().mpcb200_mlp_linearize_vjp_workspace_bytes(ctypes.byref(_rec(widths, **kw)), B, T, esz)


def _want_ws(widths, B, T, esz):
    if _vjp_smem(widths, esz) > LIMIT:
        return 0
    return (slots((T - 1) * B, _nparams(widths)) * _nparams(widths) * esz + 255) // 256 * 256


@pytest.mark.parametrize("esz", [4, 8])
def test_workspace_is_the_documented_formula(esz):
    for widths in [(5, 3), (5, 100, 3), (6, 12, 12, 12, 5), (6, 256, 5), (20, 256, 256, 4)]:
        for B, T in [(1, 2), (4, 5), (1024, 25), (300, 9), (7, 1)]:
            assert _ws(widths, B, T, esz) == _want_ws(widths, B, T, esz), (widths, B, T)
    assert slots(0, 10) == 1 and slots(5, 10) == 5 and slots(10 ** 6, 10) == _const("kMlpVjpMaxSlots")
    assert slots(10 ** 6, 1 << 24) == 1 and slots(10 ** 6, 10 ** 5) == (1 << 23) // 10 ** 5


@pytest.mark.parametrize("esz", [4, 8])
def test_a_width_256_network_at_the_edge_of_the_fit(esz):
    """(p, 256, 4): the widest input that fits, with the formula checked on both sides of the edge; a network that the
    forward kernels take but whose VJP does not fit gets 0."""
    widths = lambda p: (p, 256, 4)                   # noqa: E731
    p = max(q for q in range(5, 257) if _vjp_smem(widths(q), esz) <= LIMIT)
    assert p < 256
    assert _ws(widths(p), 8, 6, esz) > 0 and _ws(widths(p + 1), 8, 6, esz) == 0
    assert _lib.lib().mpcb200_mlp_fits(ctypes.byref(_rec(widths(p + 1))), esz) == 1
    assert _ws((64, 256, 4), 8, 6, esz) == 0
    assert _lib.lib().mpcb200_mlp_fits(ctypes.byref(_rec((64, 256, 4))), esz) == 1


def test_workspace_refuses_malformed_arguments():
    assert _ws((5, 100, 3), 4, 5, 2) == 0
    assert _ws((5, 100, 3), 0, 5, 4) == 0 and _ws((5, 100, 3), 4, 0, 4) == 0
    assert _ws((5, 100, 3), 4, 5, 4, act=3) == 0
    assert _ws((5, 100, 3), 4, 5, 4, n_prev=1) == 0
    assert _lib.lib().mpcb200_mlp_linearize_vjp_workspace_bytes(None, 4, 5, 4) == 0


def _vjp(rec, B=4, T=5, N=3, M=2, ptrs=None, ws_bytes=1 << 30, sfx="f32"):
    if ptrs is None:
        ptrs = [FAKE] * 6
    fn = getattr(_lib.lib(), "mpcb200_mlp_linearize_vjp_" + sfx)
    return fn(None if rec is None else ctypes.byref(rec), B, T, N, M, *ptrs, ws_bytes, None)


@pytest.mark.parametrize("sfx", ["f32", "f64"])
def test_status_codes(sfx):
    r = _rec()
    assert _vjp(None, sfx=sfx) == 1
    assert _vjp(_rec(act=7), sfx=sfx) == 2
    assert _vjp(_rec(n_prev=1), sfx=sfx) == 2
    for k in range(6):                                      # x u dF df dtheta workspace
        ptrs = [FAKE] * 6
        ptrs[k] = None
        assert _vjp(r, ptrs=ptrs, sfx=sfx) == 1, k
    assert _vjp(r, B=0, sfx=sfx) == 2 and _vjp(r, T=0, sfx=sfx) == 2
    assert _vjp(r, N=2, sfx=sfx) == 2 and _vjp(r, M=1, sfx=sfx) == 2 and _vjp(r, N=3 + 17, sfx=sfx) == 2
    esz = 4 if sfx == "f32" else 8
    need = _ws((5, 100, 3), 4, 5, esz)
    assert need > 0
    assert _vjp(r, ws_bytes=need - 1, sfx=sfx) == 2
    assert _vjp(r, ptrs=[FAKE] * 5 + [FAKE + 16], ws_bytes=need, sfx=sfx) == 2
    assert _vjp(_rec((64, 256, 4)), N=4, M=60, sfx=sfx) == 4             # the forward fits, the VJP does not


def test_grid_cases_reach_a_second_item_per_slot_and_a_second_slot_per_warp():
    """The GPU module's grid case: more items than slots (a slot sums several items), and more slots than the VJP
    kernel's CTAs hold warps (a warp serves several slots); 8 warps per CTA for its small network."""
    from tests.test_mlp_grad_gpu import GRID_CASE
    widths, B, T = GRID_CASE
    items, G = (T - 1) * B, slots((T - 1) * B, _nparams(widths))
    assert items > G > _const("kMlpVjpMaxCtas") * 8
    assert _vjp_smem(widths, 8, warps=8) <= LIMIT


# ------------------------------------------------------------------------------------------------------------------
# routing of MPC's differentiable tail
# ------------------------------------------------------------------------------------------------------------------
T, B = 6, 3


@pytest.fixture
def fake():
    with FakeTensorMode(allow_non_fake_inputs=True) as mode:
        yield mode


def _on(net, dtype=torch.float32, device="cuda"):
    for fc in net.fcs:          # fresh parameters (FakeTensor CUDA ones inside `fake`)
        fc.weight = torch.nn.Parameter(torch.zeros(fc.weight.shape, dtype=dtype, device=device))
        fc.bias = torch.nn.Parameter(torch.zeros(fc.bias.shape, dtype=dtype, device=device))
    return net


@pytest.fixture
def route(monkeypatch):
    """Which path linearize_dynamics(diff=True) took: "vjp" (MlpLinearize), "raw" (one linearize_raw launch) or
    "torch" (the torch tail, which returns real tensors)."""
    monkeypatch.setattr(mlpmod.MlpLinearize, "apply", lambda *a: "vjp")
    monkeypatch.setattr(mlpmod, "linearize_raw", lambda *a, **k: "raw")

    def run(ctrl, net, n, m, grad=True, device="cuda"):
        x = torch.zeros(T, B, n, device=device)
        u = torch.zeros(T, B, m, device=device)
        with torch.set_grad_enabled(grad):
            out = ctrl.linearize_dynamics(x, u, net, diff=True)
        return out if isinstance(out, str) else "torch"
    return run


def test_the_tail_takes_the_vjp_kernel(fake, route):
    for gm in (GradMethods.ANALYTIC, GradMethods.AUTO_DIFF):
        for act in ACTS:
            net = _on(NNDynamics(3, 2, hidden_sizes=(12,), activation=act))
            assert route(MPC(3, 2, T, grad_method=gm), net, 3, 2) == "vjp"
    net = _on(NNDynamics(3, 2, hidden_sizes=(12,)))
    for p in net.parameters():
        p.requires_grad_(False)
    net.fcs[1].bias.requires_grad_(True)                                       # one parameter is enough
    assert route(MPC(3, 2, T), net, 3, 2) == "vjp"


def test_each_disqualifier_keeps_the_torch_tail(fake, route):
    net = _on(NNDynamics(3, 2, hidden_sizes=(12,)))
    assert route(MPC(3, 2, T, grad_method=GradMethods.FINITE_DIFF), net, 3, 2) == "torch"

    class Sub(NNDynamics):
        pass
    assert route(MPC(3, 2, T), _on(Sub(3, 2, hidden_sizes=(12,))), 3, 2) == "torch"       # a subclass
    cpu = _on(NNDynamics(3, 2, hidden_sizes=(12,)), device="cpu")
    assert route(MPC(3, 2, T), cpu, 3, 2, device="cpu") == "torch"                    # CPU tensors
    assert route(MPC(3, 2, T), net, 3, 2, grad=False) == "raw"                 # grad disabled: no graph
    frozen = _on(NNDynamics(3, 2, hidden_sizes=(12,)))
    for p in frozen.parameters():
        p.requires_grad_(False)
    assert route(MPC(3, 2, T), frozen, 3, 2) == "raw"                          # no parameter requires grad
    big = _on(NNDynamics(4, 60, hidden_sizes=(256,)))                          # the forward fits, the VJP does not
    assert mlpmod.on_device(big, 4, 60, torch.zeros(B, 4, device="cuda"))
    assert mlpmod.vjp_workspace_bytes(big, B, T, 4) == 0
    assert route(MPC(4, 60, T), big, 4, 60) == "torch"
