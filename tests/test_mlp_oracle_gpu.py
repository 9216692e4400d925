"""GPU: a learned model's kernels (csrc/mlp.cu), its device iLQR loop (mpcb200_ilqr_mlp_*) and its episodes
(mpcb200_episode_mlp_*, mpcb200_episode_backward_mlp_*) against the float64 oracle (oracle/mlp_oracle.py,
oracle/receding_mlp_oracle.py) where those kernels can go wrong:

  * A. the rollout and linearisation at every batch position of three launch shapes (8 warps per CTA, an odd count
    in 3-7, and the 1 warp of the widest network mpcb200_mlp_fits accepts), each with a batch past 1024 CTAs so that
    warps take a second grid-stride item, the staged problem padded to the largest the warp slice is sized for
    (p_max = n_prev + width[0] + 16), n_prev 0 and m, widths on both sides of mlp_layer's split / per-lane choice,
    T = 1, and parameter blocks that take each path of stage_params (bulk copy, bulk + thread-copied tail, threads
    alone below 16 bytes and at a misaligned pointer); the split-mode line search over activations, depths, n_prev,
    bounds, decays and pass limits in float64 and float32, on batches that mix one-pass, backtracking and
    worse-at-the-limit problems, with time-invariant and time-strided costs;
  * B. the device loop at every step plan its body records (do_rollout = 0: generic and pair kernels with gains in
    shared memory or in Ks/ks past the switch horizons found on the device, the large-shape kernels), its inputs
    (tensor bounds, delta_u, u_zero_I, the slew-rate passthrough form, a time-invariant cost through MPC.forward) and
    a batch past 1024 x 8 problems; test_zz_mlp_loop_plan_coverage fails if a reachable plan never ran in the loop;
  * C. episodes at B = 512, T = 6, where the VJP's slots take a second item: the forward against the oracle's step
    and iLQR applied to the device's own states and plans, the reverse sweep against receding_mlp_oracle.backward.

Launch shapes (warps per CTA, grid passes) come from the fit formula (`smem_bytes`, mlp_smem_bytes in mlp.cu) and the
device's shared_memory_per_block_optin, never from constants.  Every output and workspace of a direct call starts
as NaN.  Tolerances: float64 1e-12 relative for the network's rollout and Jacobians; the step's own (tol_for) for
the line search and loops; float32 under gpu_harness.within against the oracle run in float32."""
import ctypes
import functools

import pytest
import torch

from mpc.pytorch_b200 import _lib, mlp as mlpmod
from mpc.pytorch_b200._lib import _on_device, stream_handle
from mpc.pytorch_b200.models import NNDynamics
from mpc.pytorch_b200.solver import MPC, CtrlPassthroughDynamics, GradMethods, QuadCost
from oracle import lqr_oracle as lo
from oracle import mlp_oracle as mo
from oracle import receding_mlp_oracle as rmo
from tests.gpu_harness import (DT, F32, F64, INSTANCES, LS_MARGIN, MAX, MID, ONE, ORACLE_TMAX, PAIR_SHAPES,
                               check_loop_departures, on_bounds,
                               kernel_env, layout_batches, ls_classes, ls_layout, misaligned, plan,
                               plan_str, pool_size, probe_step, rollout_passes, round_through, staged, switches,
                               tol_for, within)
from tests.helpers import maxdiff

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
ESZ = {F32: 4, F64: 8}
MAX_CTAS, MAX_WARPS, SLACK = 1024, 8, 16      # mlp_prepare's grid cap, mlp_warps' start, MPCB200_MLP_PAD_SLACK


# ------------------------------------------------------------------------------------------------------------------
# the launch shape, from the fit formula (mlp_shape / mlp_smem_bytes / mlp_warps / mlp_prepare in csrc/mlp.cu)
# ------------------------------------------------------------------------------------------------------------------
def widths_of(n, m, hidden):
    return (n + m, *hidden, n)


def n_params(widths):
    return sum(widths[i + 1] * (widths[i] + 1) for i in range(len(widths) - 1))


def per_warp(widths, n_prev=0):
    """Elements of one warp's shared-memory slice: the larger of the linearisation's forward pass and two Jacobian
    blocks, and the rollout / line search's two activation buffers and staged problem (p_max)."""
    L, ns, maxw = len(widths) - 1, widths[-1], max(widths)
    lin = widths[0] + sum(widths[1:-1]) + ns + (2 * ns * maxw if L > 1 else 0)
    ls = 2 * maxw + p_max(widths, n_prev)
    return (max(lin, ls) + 3) // 4 * 4


def p_max(widths, n_prev=0):
    return n_prev + widths[0] + SLACK


def smem_bytes(widths, esz, n_prev=0, warps=1):
    return 16 + (n_params(widths) * esz + 15) // 16 * 16 + warps * per_warp(widths, n_prev) * esz


def launch_warps(widths, esz, n_prev, items, optin):
    w = MAX_WARPS
    while w > 1 and (w > items or smem_bytes(widths, esz, n_prev, w) > optin):
        w -= 1
    return w


def grid_passes(items, warps):
    """Grid-stride passes of the busiest warp: items over (CTAs x warps), the CTAs capped at 1024."""
    ctas = min(MAX_CTAS, -(-items // warps))
    return -(-items // (ctas * warps))


def record_of(widths, act=0, passthrough=1, n_prev=0, params=1 << 20):
    """An mpcb200_mlp record of packed W0 b0 W1 b1 ... (the default params address is never dereferenced)."""
    r = _lib.Mlp(n_layers=len(widths) - 1, activation=act, passthrough=passthrough, n_prev=n_prev, params=params)
    o = 0
    for i, w in enumerate(widths):
        r.width[i] = w
    for i in range(len(widths) - 1):
        r.W_off[i] = o
        o += widths[i + 1] * widths[i]
        r.b_off[i] = o
        o += widths[i + 1]
    return r


def fits(widths, esz, n_prev=0):
    return bool(_lib.lib().mpcb200_mlp_fits(ctypes.byref(record_of(widths, n_prev=n_prev)), esz))


EDGE_NM = (4, 2)


@functools.lru_cache(maxsize=None)
def edge_hidden(esz, n_prev=0, nm=EDGE_NM):
    """The widest h of a (n+m, h, h, n) network that mpcb200_mlp_fits accepts, by bisection."""
    n, m = nm
    lo_, hi = 1, 256
    assert fits(widths_of(n, m, (lo_, lo_)), esz, n_prev) and not fits(widths_of(n, m, (hi, hi)), esz, n_prev)
    while hi - lo_ > 1:
        mid = (lo_ + hi) // 2
        if fits(widths_of(n, m, (mid, mid)), esz, n_prev):
            lo_ = mid
        else:
            hi = mid
    return lo_


def odd_hidden(esz, optin):
    """The widest (n+m, h, h, n) network that runs an odd warp count in 3..7 per CTA at this opt-in."""
    n, m = EDGE_NM
    for h in range(256, 0, -1):
        w = launch_warps(widths_of(n, m, (h, h)), esz, 0, 1 << 30, optin)
        if w in (3, 5, 7):
            return h
    raise AssertionError("no network width runs an odd warp count")


def optin():
    return torch.cuda.get_device_properties(DEV).shared_memory_per_block_optin


# (name, n, m, hidden, act, passthrough, n_prev); hidden None: sized at run time from the device's opt-in
SHAPES = [("small", 4, 2, (32,), "sigmoid", True, 0), ("small_prev", 4, 2, (32, 12), "relu", False, 2),
          ("odd", 4, 2, None, "elu", True, 0), ("edge", 4, 2, None, "sigmoid", True, 0),
          ("edge_prev", 4, 2, None, "relu", False, 2)]
PAD = (10, 6)                                   # N, M padding: N + M = p_max exactly
GRID_T = 3                                      # (T - 1) * B linearisation items


def shape_hidden(name, hidden, dtype, n_prev):
    if hidden is not None:
        return hidden
    esz = ESZ[dtype]
    h = odd_hidden(esz, optin()) if name == "odd" else edge_hidden(esz, n_prev)
    return (h, h)


def grid_batches(W):
    """layout_batches over a pool coprime to W, and one batch past 1024 CTAs of W warps: every warp takes a second
    grid-stride item."""
    K = pool_size(W)
    return K, layout_batches(1, W, K) + [MAX_CTAS * W + W + 1]


# ------------------------------------------------------------------------------------------------------------------
# direct calls
# ------------------------------------------------------------------------------------------------------------------
def _nan(*shape, dtype):
    return torch.full(shape, float("nan"), dtype=dtype, device=DEV)


def _call(name, rec, dtype, *args):
    L = _lib.lib()
    with _on_device(DEV):
        rc = getattr(L, f"mpcb200_mlp_{name}_{DT[dtype]}")(ctypes.byref(rec), *args, stream_handle(DEV))
    assert rc == 0, f"mpcb200_mlp_{name}: {L.mpcb200_strerror(rc)}"


def direct(rec, dtype, B, T, N, M, x, u):
    """(x from the rollout of x[0], F, f of the linearisation at x, u) of device tensors x [T, B, N], u [T, B, M]."""
    xo, Fo, fo = _nan(T, B, N, dtype=dtype), _nan(max(T - 1, 1), B, N, N + M, dtype=dtype), \
        _nan(max(T - 1, 1), B, N, dtype=dtype)
    x0 = x[0].contiguous()
    _call("rollout", rec, dtype, B, T, N, M, _lib.ptr(x0), _lib.ptr(u), _lib.ptr(xo))
    _call("linearize", rec, dtype, B, T, N, M, _lib.ptr(x), _lib.ptr(u), _lib.ptr(Fo), _lib.ptr(fo))
    torch.cuda.synchronize()
    return xo.cpu(), Fo.cpu(), fo.cpu()


def _net(n, m, hidden, act, passthrough, seed, scale=1.5):
    torch.manual_seed(seed)
    net = NNDynamics(n, m, hidden_sizes=list(hidden), activation=act, passthrough=passthrough).double()
    with torch.no_grad():
        for fc in net.fcs:
            fc.weight.mul_(scale)
    return net


def _layers(net, dtype):
    return [(round_through(W, dtype), round_through(b, dtype)) for W, b in mo.layers_of(net)]


def direct_oracle(layers, act, pt, n_prev, n, m, x, u, N, M):
    """The oracle's rollout of x[0] and linearisation at (x, u), at the staged shape: x[0] as given (padding
    included), 0 in every padded state after it, F and f embedded at [N, N+M] with zeros around them."""
    T, K = x.shape[:2]
    Nn = n_prev + n
    dt = x.dtype
    xs = torch.zeros(T, K, N, dtype=dt)
    xs[:, :, :Nn] = mo.rollout(layers, act, pt, x[0, :, :Nn], u[:, :, :m], n_prev)
    xs[0] = x[0]
    F0, f0 = mo.linearize(layers, act, pt, x[:, :, :Nn], u[:, :, :m], n_prev)
    F = torch.zeros(T - 1, K, N, N + M, dtype=dt)
    F[..., :Nn, :Nn] = F0[..., :Nn]
    F[..., :Nn, N:N + m] = F0[..., Nn:]
    f = torch.zeros(T - 1, K, N, dtype=dt)
    f[..., :Nn] = f0
    return xs, F, f


def pool_inputs(K, T, N, M, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    x = round_through(torch.randn(T, K, N, generator=g, dtype=F64), dtype)
    u = round_through(torch.randn(T, K, M, generator=g, dtype=F64), dtype)
    return x, u


def check_direct(tag, got, pool64, pool32, idx, dtype, T):
    for i, what in enumerate(("x", "F", "f")):
        if T == 1 and i:
            continue
        w64 = pool64[i][:, idx]
        w32 = None if pool32 is None else pool32[i][:, idx].double()
        g = got[i] if i == 0 else got[i][:T - 1]
        within(tag, what, g, w64, w32, dtype, tol64=1e-12)
        zero = (w64 == 0)
        assert bool((g[zero] == 0).all()), f"{tag}: {what} not exactly 0 in padding or structural zeros"


def run_grid(tag, net, act, pt, n_prev, dtype, batches, K, pad=PAD, T=GRID_T, seed=11):
    n, m = net.n_state, net.n_ctrl
    widths = widths_of(n, m, [fc.out_features for fc in net.fcs[:-1]])
    N, M = n_prev + n + pad[0], m + pad[1]
    layers = _layers(net, dtype)
    x, u = pool_inputs(K, T, N, M, dtype, seed)
    pool64 = direct_oracle(layers, act, pt, n_prev, n, m, x, u, N, M)
    pool32 = None
    if dtype == F32:
        pool32 = direct_oracle([(W.float(), b.float()) for W, b in layers], act, pt, n_prev, n, m, x.float(),
                               u.float(), N, M)
    net_d = net.to(dtype=dtype, device=DEV)
    dxm = CtrlPassthroughDynamics(net_d) if n_prev else net_d
    rec, buf = mlpmod.record(dxm, torch.empty(0, dtype=dtype, device=DEV))
    assert N + M == p_max(widths, n_prev) or pad != PAD
    for B in batches:
        idx = torch.arange(B) % K
        xd, ud = x[:, idx].to(DEV, dtype).contiguous(), u[:, idx].to(DEV, dtype).contiguous()
        got = direct(rec, dtype, B, T, N, M, xd, ud)
        check_direct(f"{tag} B={B}", got, pool64, pool32, idx, dtype, T)
    return widths


# ------------------------------------------------------------------------------------------------------------------
# A. direct kernels at every batch position and launch shape
# ------------------------------------------------------------------------------------------------------------------
LAUNCH_REPORT = {}


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("shape", SHAPES, ids=[s[0] for s in SHAPES])
def test_rollout_and_linearisation_grid_stride_at_each_launch_shape(shape, dtype):
    """Every batch of layout_batches(1, W, K) and one past 1024 x W problems, at the warps per CTA the launcher picks
    (from the fit formula and the device's opt-in), the staged problem at p_max."""
    name, n, m, hidden, act, pt, n_prev = shape
    hidden = shape_hidden(name, hidden, dtype, n_prev)
    widths = widths_of(n, m, hidden)
    esz = ESZ[dtype]
    assert fits(widths, esz, n_prev)
    W = launch_warps(widths, esz, n_prev, 1 << 30, optin())
    if name == "small" or name == "small_prev":
        assert W == MAX_WARPS
    elif name == "odd":
        assert W in (3, 5, 7)
    else:
        assert W == 1 and not fits(widths_of(n, m, (hidden[0] + 1,) * 2), esz, n_prev)
    K, batches = grid_batches(W)
    big = batches[-1]
    assert grid_passes(big, W) == 2 and grid_passes((GRID_T - 1) * big, W) >= 2
    net = _net(n, m, hidden, act, pt, seed=len(name))
    run_grid(f"{name} {hidden} {DT[dtype]} W={W}", net, act, pt, n_prev, dtype, batches, K)
    LAUNCH_REPORT[(name, DT[dtype])] = dict(hidden=hidden, warps=W, batch=big,
                                            rollout_passes=grid_passes(big, W),
                                            linearize_passes=grid_passes((GRID_T - 1) * big, W))
    print(name, DT[dtype], LAUNCH_REPORT[(name, DT[dtype])])


# networks with layers on both sides of mlp_layer's split / per-lane choice: output widths 1, 31, 32, 33, 64 behind
# an input of 256, and a 256-wide layer behind a narrow input
WIDTH_NETS = [(4, 2, (256, k)) for k in (1, 31, 32, 33, 64)] + [(k, 2, (256,)) for k in (1, 20)]


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("n,m,hidden", WIDTH_NETS, ids=[f"n{c[0]}_{'x'.join(map(str, c[2]))}" for c in WIDTH_NETS])
def test_rollout_and_linearisation_at_layer_width_switches(n, m, hidden, dtype):
    widths = widths_of(n, m, hidden)
    W = launch_warps(widths, ESZ[dtype], 0, 1 << 30, optin())
    K = pool_size(W)
    net = _net(n, m, hidden, "sigmoid", True, seed=n + len(hidden))
    run_grid(f"{hidden} n={n} {DT[dtype]}", net, "sigmoid", True, 0, dtype, [2 * W + 1], K)


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("n_prev", [0, 2])
def test_horizon_one_rollout_writes_x0_and_linearisation_writes_nothing(n_prev, dtype):
    n, m, B = 4, 2, 19
    net = _net(n, m, (16,), "elu", True, seed=3).to(dtype=dtype, device=DEV)
    dxm = CtrlPassthroughDynamics(net) if n_prev else net
    rec, buf = mlpmod.record(dxm, torch.empty(0, dtype=dtype, device=DEV))
    N, M = n_prev + n + 3, m + 1
    x0 = torch.randn(B, N, dtype=dtype, device=DEV)
    u = torch.randn(1, B, M, dtype=dtype, device=DEV)
    xo, F, f = _nan(1, B, N, dtype=dtype), _nan(2, B, N, N + M, dtype=dtype), _nan(2, B, N, dtype=dtype)
    before = _lib.launch_count()
    _call("rollout", rec, dtype, B, 1, N, M, _lib.ptr(x0), _lib.ptr(u), _lib.ptr(xo))
    mid = _lib.launch_count()
    _call("linearize", rec, dtype, B, 1, N, M, _lib.ptr(x0), _lib.ptr(u), _lib.ptr(F), _lib.ptr(f))
    torch.cuda.synchronize()
    assert mid - before == 1 and _lib.launch_count() == mid
    assert torch.equal(xo[0], x0)
    assert bool(F.isnan().all()) and bool(f.isnan().all())


# (n, m, hidden): n_params x 4 and x 8 a multiple of 16 (bulk copy alone); odd n_params (bulk copy and a tail in both
# dtypes); 3 parameters (f32: 12 bytes, no bulk copy at all; f64: 16 bytes of bulk and an 8-byte tail)
STAGING = [(4, 2, (32,)), (3, 2, (8,)), (1, 1, ())]


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("n,m,hidden", STAGING, ids=["bulk", "bulk_tail", "tiny"])
def test_parameter_staging_paths_are_bitwise_equal(n, m, hidden, dtype, monkeypatch):
    """The same network from an aligned block and from one 4 (f32) or 8 (f64) bytes off 16-byte alignment, whose
    whole block the threads copy: rollout, linearisation and the split-mode step bitwise equal, and within tolerance
    of the oracle.  B is past 1024 CTAs, so every CTA stages the block and every warp then takes a second item."""
    widths = widths_of(n, m, hidden)
    esz = ESZ[dtype]
    tail = (n_params(widths) * esz) % 16
    assert tail == {(4, 2, (32,)): 0, (3, 2, (8,)): (12 if esz == 4 else 8), (1, 1, ()): (12 if esz == 4 else 8)}[
        (n, m, hidden)]
    net = _net(n, m, hidden, "sigmoid", True, seed=7)
    W = launch_warps(widths, esz, 0, 1 << 30, optin())
    B, T = MAX_CTAS * W + W + 1, 5
    K = pool_size(W)
    assert grid_passes(B, W) == 2
    run_grid(f"staging {hidden} {DT[dtype]}", net, "sigmoid", True, 0, dtype, [B], K, pad=(0, 0), T=T)
    LAUNCH_REPORT[("staging_" + "x".join(map(str, widths)), DT[dtype])] = dict(
        warps=W, batch=B, rollout_step_passes=grid_passes(B, W), linearize_passes=grid_passes((T - 1) * B, W))
    net_d = net.to(dtype=dtype, device=DEV)
    x, u = pool_inputs(B, T, n, m, dtype, 5)
    xd, ud = x.to(DEV, dtype), u.to(DEV, dtype)
    C, c = _cost(2, T, B, n + m)
    Cd, cd = C.to(DEV, dtype), c.to(DEV, dtype)
    F, f = mlpmod.linearize_raw(net_d, T, xd, ud)

    def everything():
        with poisoned_empty():
            r = [mlpmod.rollout_raw(net_d, T, xd[0], ud), *mlpmod.linearize_raw(net_d, T, xd, ud)]
            s = mlpmod.step_raw(net_d, n, m, T, xd[0], Cd, cd, F, f, xd, ud, max_linesearch_iter=4)
        torch.cuda.synchronize()
        return r + [s[k] for k in ("new_x", "new_u", "costs", "alphas", "du_first")]
    aligned = everything()
    real = mlpmod.record

    def shifted(dx, x_):
        rec, buf = real(dx, x_)
        assert buf.data_ptr() % 16 == 0
        mis = misaligned(buf)
        assert mis.data_ptr() % 16 == esz
        return mlpmod._record(dx, 0, mis.data_ptr()), mis
    monkeypatch.setattr(mlpmod, "record", shifted)
    moved = everything()
    for k, (a, b) in enumerate(zip(aligned, moved)):
        assert torch.equal(a, b), f"output {k} differs between the aligned and the misaligned parameter block"
        assert not bool(a.isnan().any()), f"output {k} not written"


# ------------------------------------------------------------------------------------------------------------------
# A.5 the split-mode line search
# ------------------------------------------------------------------------------------------------------------------
def poisoned_empty():
    from tests.test_mlp_gpu import poisoned
    return poisoned()


def _cost(seed, T, B, p):
    g = torch.Generator().manual_seed(seed)
    Lc = torch.randn(T, B, p, p, generator=g, dtype=F64) / p ** 0.5
    C = Lc @ Lc.transpose(-1, -2) + 0.5 * torch.eye(p, dtype=F64)
    c = 2.0 * torch.randn(T, B, p, generator=g, dtype=F64)
    return C, c


LS_MODES = ("free", "box", "tensor", "boxD", "mask")
LS_ACTS = ("sigmoid", "relu", "elu")
LS_HIDDEN = ((), (12,), (12, 12), (12, 12, 12))
LS_T, LS_M, LS_N = 6, 2, 3
LS_POOL = 480


def ls_matrix():
    """A covering set of the line search's options: every value of every option appears, each dtype with each
    activation, depth, mode and pass limit."""
    out = []
    for i in range(30):
        out.append(dict(dtype=(F64, F32)[i % 2], act=LS_ACTS[(i // 2) % 3], hidden=LS_HIDDEN[(i // 2) % 4],
                        n_prev=(0, LS_M)[(i // 4) % 2], mode=LS_MODES[i % 5], decay=(0.5, 0.3)[(i // 3) % 2],
                        max_ls=(1, 3, 10)[(i // 5) % 3], seed=400 + i))
    return out


LS_CASES = ls_matrix()


def ls_case_id(c):
    return (f"{DT[c['dtype']]}_{c['act']}_L{len(c['hidden']) + 1}_p{c['n_prev']}_{c['mode']}_d{c['decay']}"
            f"_ls{c['max_ls']}")


@functools.lru_cache(maxsize=4)
def ls_pool(dtype, act, hidden, n_prev, mode, decay, max_ls, seed, K=LS_POOL, T=LS_T, n_in=LS_N, m=LS_M,
            net_scale=None):
    """K float64 step problems around nominals that make the line search backtrack (four families by k % 4, as
    gpu_harness.ls_nominal: 0 a rolled-out nominal, 1 its controls perturbed after the rollout, 2 and 3 its states
    perturbed and pulled down their stage cost's gradient, so that no rollout reaches the nominal's cost), inputs
    rounded through dtype.  Returns (net, layers, P, kw, o64, first64, o32, first32, cls): cls per candidate, -1
    where it is not kept (a pass within LS_MARGIN of the old cost, a worse-at-the-limit problem whose last pass
    equals its first, a float32 oracle that decides otherwise)."""
    n = n_in + n_prev
    net = _net(n_in, m, hidden, act, True, seed, scale=net_scale or ls_scale(act, hidden))
    layers = _layers(net, dtype)
    g = torch.Generator().manual_seed(seed)
    C, c = _cost(seed, T, K, n + m)
    x0 = torch.randn(K, n, generator=g, dtype=F64)
    fam = torch.arange(K) % 4
    u = torch.randn(T, K, m, generator=g, dtype=F64) * (0.3 + 1.7 * torch.rand(1, K, 1, generator=g, dtype=F64))
    kw = {}
    if mode in ("box", "boxD"):
        kw = dict(u_lower=-1.5, u_upper=1.5)
        u = u.clamp(-1.5, 1.5)
    elif mode == "tensor":
        lo_ = -0.5 - torch.rand(T, K, m, generator=g, dtype=F64)
        kw = dict(u_lower=lo_, u_upper=lo_ + 2.0)
        u = torch.maximum(torch.minimum(u, lo_ + 2.0), lo_)
    if mode == "boxD":
        kw["delta_u"] = 0.8
    if mode == "mask":
        kw["u_zero_I"] = torch.rand(T, K, m, generator=g) < 0.3
    x0, u, C, c = (round_through(t, dtype) for t in (x0, u, C, c))
    x = mo.rollout(layers, act, True, x0, u, n_prev)
    later = (torch.arange(T) >= 1).view(T, 1, 1)
    du = 0.3 * torch.randn(T, K, m, generator=g, dtype=F64)
    u1 = torch.where((fam == 1).view(1, K, 1) & later, u + du, u)
    if "u_lower" in kw:
        lo_, hi = (torch.as_tensor(kw[k], dtype=F64).expand_as(u) for k in ("u_lower", "u_upper"))
        u1 = torch.minimum(torch.maximum(u1, lo_), hi)
    u = round_through(u1, dtype)
    noise = torch.randn(T, K, n, generator=g, dtype=F64)
    pull = 6.0 * torch.rand(K, generator=g, dtype=F64)
    pert = (fam >= 2).view(1, K, 1) & later
    x = torch.where(pert, x + noise, x)
    grad = torch.einsum("tbij,tbj->tbi", C[..., :n, :], torch.cat((x, u), 2)) + c[..., :n]
    x = torch.where(pert, x - pull.view(1, K, 1) * grad / grad.norm(dim=2, keepdim=True).clamp_min(1e-12), x)
    x = round_through(x, dtype)
    F, f = mo.linearize(layers, act, True, x, u, n_prev)
    F, f = round_through(F, dtype), round_through(f, dtype)
    P = dict(x0=x0, C=C, c=c, F=F, f=f, x=x, u=u)
    kw = {k: round_through(v, dtype) for k, v in kw.items()}
    kw.update(linesearch_decay=decay, max_linesearch_iter=max_ls)
    o64, trace, first64 = ls_oracle(n, m, T, P, kw, layers, act, n_prev)
    cls = ls_classes(trace)
    old = o64.costs - trace[-1]
    counted = torch.arange(trace.shape[0]).view(-1, 1) < rollout_passes(trace).view(1, -1)
    ok = ((trace.abs() >= LS_MARGIN * old.abs().clamp_min(1.0)) | ~counted).all(0)
    if max_ls > 1:
        ok &= (cls != MAX) | ((first64 - o64.new_u).abs().amax((0, 2)) > 1e-6)
    o32 = first32 = None
    if dtype == F32:
        l32 = [(W.float(), b.float()) for W, b in layers]
        lo32 = lambda t: t.float() if torch.is_tensor(t) and t.is_floating_point() else t  # noqa: E731
        o32, t32, first32 = ls_oracle(n, m, T, {k: lo32(v) for k, v in P.items()}, {k: lo32(v) for k, v in kw.items()},
                                      l32, act, n_prev)
        ok &= (ls_classes(t32) == cls) & (rollout_passes(t32) == rollout_passes(trace))
    return net, layers, P, kw, o64, first64, o32, first32, torch.where(ok, cls, -1)


def ls_scale(act, hidden):
    """Weight scale of the line-search networks: curved enough that full steps overshoot (sigmoid layers saturate,
    so deep sigmoid networks take more), mild enough that a deep relu / elu network's float32 round-off flips no
    kink the float32 oracle does not flip too."""
    if len(hidden) <= 1:
        return 4.0
    return 8.0 if act == "sigmoid" else 2.5


def ls_oracle(n, m, T, P, kw, layers, act, n_prev):
    trace, first = [], []
    o = lo.lqr_step_forward(n, m, T, *[P[k] for k in ("x0", "C", "c", "F", "f", "x", "u")], coupled=False,
                            dynamics=lambda a, b: mo.step(layers, act, True, a, b, n_prev), ls_trace=trace,
                            first_u=first, **kw)
    return o, torch.stack(trace), first[0]


def ls_select(cls, layout):
    """Pool indices realising a class layout; a class the pool lacks is replaced by the next of MID, MAX, ONE."""
    have = {c: (cls == c).nonzero()[:, 0].tolist() for c in (ONE, MID, MAX)}
    order = {ONE: (ONE, MID, MAX), MID: (MID, MAX, ONE), MAX: (MAX, MID, ONE)}
    seen = {ONE: 0, MID: 0, MAX: 0}
    idx = []
    for c in layout:
        c = next(d for d in order[c] if have[d])
        idx.append(have[c][seen[c] % len(have[c])])
        seen[c] += 1
    return torch.tensor(idx)


def ls_batch_layout(B):
    """One problem per warp: ls_layout's one-problem-per-CTA cycle ONE, MAX, MID, so that neighbouring warps, the
    first warps of neighbouring CTAs (8 per CTA, coprime to 3) and a warp's grid-stride items (1024 x 8 apart,
    also coprime to 3) hold problems of different pass counts."""
    return ls_layout(B, 1, 1)


def _rows(v, idx):
    if not torch.is_tensor(v) or v.dim() == 0:
        return v
    return v[idx] if v.dim() <= 2 else v[:, idx]


def run_ls(pool, n_prev, idx, dtype, C_view=None, c_view=None, nm=None):
    """mpcb200_mlp_step_* on the pool problems idx (poisoned); C_view, c_view: device views to hand over instead
    of the dense C, c; nm: the staged (n, m) when it is not the network's."""
    net, layers, P, kw, *_ = pool
    n, m = nm or (LS_N + n_prev, LS_M)
    d = lambda t: t.to(DEV, dtype) if torch.is_tensor(t) and t.is_floating_point() else (  # noqa: E731
        t.to(DEV) if torch.is_tensor(t) else t)
    Pd = {k: d(_rows(v, idx)) for k, v in P.items()}
    opts = {k: d(_rows(v, idx)) for k, v in kw.items()}
    net_d = net.to(dtype=dtype, device=DEV)
    dxm = CtrlPassthroughDynamics(net_d) if n_prev else net_d
    C = Pd["C"] if C_view is None else C_view
    c = Pd["c"] if c_view is None else c_view
    with poisoned_empty():
        r = mlpmod.step_raw(dxm, n, m, LS_T, Pd["x0"], C, c, Pd["F"], Pd["f"], Pd["x"], Pd["u"], **opts)
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in r.items() if v is not None}


def check_ls(tag, r, pool, idx, dtype):
    _, _, P, kw, o64, first64, o32, first32, cls = pool
    sel = lambda o, k: None if o is None else _rows(getattr(o, k), idx)  # noqa: E731
    bounded = "u_lower" in kw
    if dtype == F64:
        tol = 2e-6 if bounded else tol_for(F64, False)["xu"]      # bounded: pnqp's stopping rule
        sc = max(1.0, float(sel(o64, "new_x").abs().max()))
        for k in ("new_x", "new_u"):
            assert maxdiff(r[k], sel(o64, k)) < tol * sc, f"{tag}: {k} {maxdiff(r[k], sel(o64, k)):.3e}"
        assert maxdiff(r["costs"], sel(o64, "costs")) < tol * max(1.0, float(sel(o64, "costs").abs().max())), tag
        du = _rows(P["u"], idx) - _rows(first64, idx)
        assert maxdiff(r["du_first"], du) < tol * sc, f"{tag}: du_first"
        if bounded:
            assert maxdiff(r["alphas"], sel(o64, "alphas")) < 1e-12, f"{tag}: alphas"
        else:
            assert torch.equal(r["alphas"], sel(o64, "alphas")), f"{tag}: alphas"
    else:
        sc = max(1.0, float(sel(o64, "new_x").abs().max()), float(sel(o64, "new_u").abs().max()))
        for k in ("new_x", "new_u"):
            within(tag, k, r[k], sel(o64, k), sel(o32, k).double(), dtype, scale=sc)
        within(tag, "costs", r["costs"], sel(o64, "costs"), sel(o32, "costs").double(), dtype)
        u = _rows(P["u"], idx)
        within(tag, "du_first", r["du_first"], u - _rows(first64, idx), u - _rows(first32, idx).double(), dtype,
               scale=sc)
        w32, w64 = sel(o32, "alphas"), sel(o64, "alphas")
        same = (w32.double() - w64).abs() <= 1e-6
        assert bool(same.all()), f"{tag}: the float32 oracle decides a kept problem otherwise"
        assert torch.equal(r["alphas"], w32), f"{tag}: alphas {r['alphas']} vs {w32}"
    if "u_zero_I" in kw:
        assert bool((r["new_u"][_rows(kw["u_zero_I"], idx)] == 0).all()), f"{tag}: masked controls"


def _ls_args(c):
    return (c["dtype"], c["act"], c["hidden"], c["n_prev"], c["mode"], c["decay"], c["max_ls"], c["seed"])


LS_B = 3 * MAX_WARPS + 4                         # three CTAs of 8 warps and a partial one


@pytest.mark.parametrize("case", LS_CASES, ids=[ls_case_id(c) for c in LS_CASES])
def test_line_search_matches_the_oracle_on_mixed_pass_counts(case):
    dtype = case["dtype"]
    pool = ls_pool(*_ls_args(case))
    cls = pool[-1]
    idx = ls_select(cls, ls_batch_layout(LS_B))
    assert len(set(cls[idx].tolist())) >= (2 if case["max_ls"] == 1 else 3), cls[idx]
    r = run_ls(pool, case["n_prev"], idx, dtype)
    check_ls(ls_case_id(case), r, pool, idx, dtype)


LS_LAYOUT_CASES = [LS_CASES[0], LS_CASES[11]]      # f64 and f32, each with a tensor box or none


@pytest.mark.parametrize("case", LS_LAYOUT_CASES, ids=[ls_case_id(c) for c in LS_LAYOUT_CASES])
def test_line_search_cost_layouts_are_bitwise_equal(case):
    """A time-invariant C, c (stride 0 over time) and a C, c that is every other slice of a [2T, ...] tensor (a
    positive time stride) give the dense call's outputs bit for bit."""
    dtype = case["dtype"]
    pool = ls_pool(*_ls_args(case))
    idx = ls_select(pool[-1], ls_batch_layout(LS_B))
    _, _, P, *_ = pool
    C, c = _rows(P["C"], idx), _rows(P["c"], idx)
    # time invariant: every slice is slice 0, dense for the reference call
    ti = list(pool)
    ti[2] = dict(P, C=P["C"][:1].expand_as(P["C"]).contiguous(), c=P["c"][:1].expand_as(P["c"]).contiguous())
    dense = run_ls(ti, case["n_prev"], idx, dtype)
    C0, c0 = C[:1].to(DEV, dtype), c[:1].to(DEV, dtype)
    Cv, cv = C0.expand(LS_T, *C0.shape[1:]), c0.expand(LS_T, *c0.shape[1:])
    assert staged(Cv, dtype)[1] == -1 and staged(cv, dtype)[1] == -1
    got = run_ls(ti, case["n_prev"], idx, dtype, Cv, cv)
    for k in dense:
        assert torch.equal(got[k], dense[k]), f"time-invariant cost: {k}"
    # every other slice of [2T, B, ...]
    dense = run_ls(pool, case["n_prev"], idx, dtype)
    C2 = torch.zeros(2 * LS_T, *C.shape[1:], dtype=dtype, device=DEV)
    c2 = torch.zeros(2 * LS_T, *c.shape[1:], dtype=dtype, device=DEV)
    C2[::2], c2[::2] = C.to(DEV, dtype), c.to(DEV, dtype)
    C2[1::2], c2[1::2] = float("nan"), float("nan")
    assert staged(C2[::2], dtype)[1] > 0 and staged(c2[::2], dtype)[1] > 0
    got = run_ls(pool, case["n_prev"], idx, dtype, C2[::2], c2[::2])
    for k in dense:
        assert torch.equal(got[k], dense[k]), f"time-strided cost: {k}"
    check_ls(ls_case_id(case), dense, pool, idx, dtype)


@pytest.mark.parametrize("mode", ["free", "box"])
@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
def test_line_search_fills_the_warp_slice_at_p_max(dtype, mode):
    """The line search's slice holds two activation buffers and the staged X and U; with a network that has no hidden
    layer that is the larger term of per_warp, and with N + M = p_max it is used to its last element.  The network
    (n, m) = (3, 1) runs in the (16, 4) instance's step: N + M = 20 = n_prev + width[0] + 16.  States past the
    network's are 0 after every step, the padded controls are penalised by C = I and reach nothing; the oracle solves
    the same padded problem with the network as the dynamics of its first 3 states.  B spans four CTAs of 8 warps, so
    a slice too short by a few elements would overlap the next warp's activations while it runs."""
    n0, m0, N, M = 3, 1, 16, 4
    widths = widths_of(n0, m0, ())
    assert N + M == p_max(widths) and per_warp(widths) == 2 * max(widths) + p_max(widths)
    pool = ls_pool(dtype, "elu", (), 0, mode, 0.5, 10, 490, n_in=n0, m=m0)
    net, layers, P0, kw0, *_ = pool
    idx = ls_select(pool[-1], ls_batch_layout(LS_B))
    B, T = LS_B, LS_T
    P0 = {k: _rows(v, idx) for k, v in P0.items()}
    P = dict(x0=torch.zeros(B, N, dtype=F64), x=torch.zeros(T, B, N, dtype=F64), u=torch.zeros(T, B, M, dtype=F64),
             C=torch.eye(N + M, dtype=F64).repeat(T, B, 1, 1), c=torch.zeros(T, B, N + M, dtype=F64),
             F=torch.zeros(T - 1, B, N, N + M, dtype=F64), f=torch.zeros(T - 1, B, N, dtype=F64))
    P["x0"][:, :n0], P["x"][..., :n0], P["u"][..., :m0] = P0["x0"], P0["x"], P0["u"]
    sel = list(range(n0)) + [N + j for j in range(m0)]
    P["C"][..., torch.tensor(sel)[:, None], torch.tensor(sel)[None, :]] = P0["C"]
    P["c"][..., torch.tensor(sel)] = P0["c"]
    P["F"][..., :n0, :n0], P["F"][..., :n0, N:N + m0], P["f"][..., :n0] = P0["F"][..., :n0], P0["F"][..., n0:], P0["f"]
    kw = {k: v for k, v in kw0.items()}

    def dyn(lay):
        def step(x, u):
            out = torch.zeros_like(x)
            out[:, :n0] = mo.step(lay, "elu", True, x[:, :n0], u[:, :m0])
            return out
        return step
    trace, first = [], []
    o64 = lo.lqr_step_forward(N, M, T, *[P[k] for k in ("x0", "C", "c", "F", "f", "x", "u")], coupled=False,
                              dynamics=dyn(layers), ls_trace=trace, first_u=first, **kw)
    assert len(set(ls_classes(torch.stack(trace)).tolist())) == 3
    o32 = first32 = None
    if dtype == F32:
        f32 = lambda t: t.float() if torch.is_tensor(t) and t.is_floating_point() else t  # noqa: E731
        first32 = []
        o32 = lo.lqr_step_forward(N, M, T, *[f32(P[k]) for k in ("x0", "C", "c", "F", "f", "x", "u")],
                                  coupled=False, dynamics=dyn([(W.float(), b.float()) for W, b in layers]),
                                  first_u=first32, **{k: f32(v) for k, v in kw.items()})
        first32 = first32[0]
    padded = (net, layers, P, kw, o64, first[0], o32, first32, None)
    every = torch.arange(B)
    r = run_ls(padded, 0, every, dtype, nm=(N, M))
    check_ls(f"p_max {DT[dtype]} {mode}", r, padded, every, dtype)


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
def test_line_search_horizon_one(dtype):
    pool = ls_pool(dtype, "sigmoid", (12,), 0, "free", 0.5, 3, 470, K=24, T=1)
    net, layers, P, kw, o64, first64, o32, first32, cls = pool
    idx = torch.arange(24)
    n, m = LS_N, LS_M
    d = lambda t: t.to(DEV, dtype)  # noqa: E731
    net_d = net.to(dtype=dtype, device=DEV)
    F = torch.empty(0, 24, n, n + m, dtype=dtype, device=DEV)
    with poisoned_empty():
        r = mlpmod.step_raw(net_d, n, m, 1, d(P["x0"]), d(P["C"]), d(P["c"]), F, None, d(P["x"]), d(P["u"]),
                            linesearch_decay=0.5, max_linesearch_iter=3)
    torch.cuda.synchronize()
    r = {k: v.cpu() for k, v in r.items() if v is not None}
    assert torch.equal(r["new_x"][0], P["x0"].to(dtype))
    check_ls(f"T=1 {DT[dtype]}", r, pool, idx, dtype)


@pytest.mark.parametrize("which", ["small_f64", "small_f32", "edge_f64"])
def test_line_search_grid_stride_items_start_afresh(which):
    """A batch past 1024 CTAs (8 warps each for the small network, 1 for the widest one), so that each warp runs a
    second problem after one of another pass count: its alpha, cost and staged state must start afresh."""
    dtype = F32 if which.endswith("f32") else F64
    if which.startswith("edge"):
        h = edge_hidden(ESZ[dtype], 0, (LS_N, LS_M))
        hidden, K = (h, h), 96
        W = launch_warps(widths_of(LS_N, LS_M, hidden), ESZ[dtype], 0, 1 << 30, optin())
        assert W == 1
    else:
        hidden, W, K = (12,), MAX_WARPS, LS_POOL
    B = MAX_CTAS * W + W + 1
    assert grid_passes(B, W) == 2
    pool = ls_pool(dtype, "sigmoid", hidden, 0, "free", 0.5, 10, 480, K=K)
    idx = ls_select(pool[-1], ls_batch_layout(B))
    assert len(set(pool[-1][idx].tolist())) == 3
    # a warp's two items hold different pass counts wherever the layout allows
    r = run_ls(pool, 0, idx, dtype)
    check_ls(f"grid {which} B={B} W={W}", r, pool, idx, dtype)
    LAUNCH_REPORT[("linesearch_" + which, DT[dtype])] = dict(hidden=hidden, warps=W, batch=B,
                                                             passes=grid_passes(B, W))
    print(which, LAUNCH_REPORT[("linesearch_" + which, DT[dtype])])


# ------------------------------------------------------------------------------------------------------------------
# B. the device loop against mlp_oracle.ilqr at every step plan
# ------------------------------------------------------------------------------------------------------------------
LOOP_SEEN = {}                      # dtype -> step plans run inside the MLP loop
LOOP_DEPARTED = []
LOOP_HIDDEN = (16,)


def loop_plan_name(p):
    if p == _lib.PLAN_LARGE:
        return "large"
    assert not p & _lib.PLAN_KREDUCE, plan_str(p)
    return ("generic" if p & _lib.PLAN_GENERIC else "pair") + ("_smem" if p & _lib.PLAN_GAINS_SMEM else "_ks")


def loop_net(n, m, seed, n_prev=0):
    """A sigmoid network without passthrough and weights x 0.5: x' = W1 sigmoid(W0 z + b0) + b1, so every state of
    any rollout stays within sum |W1| + |b1| of 0, however long the horizon."""
    return _net(n - n_prev, m, LOOP_HIDDEN, "sigmoid", False, seed, scale=0.5)


@functools.lru_cache(maxsize=4)
def loop_case(seed, B, T, n, m, dtype, mode, lqr_iter=3, n_prev=0, time_invariant=False):
    """(net, P, kw, opts, o64, o32|None): a bounded-state network, a PD cost, and the oracle's loop with eps = 0 and
    not_improved_lim > lqr_iter, so every problem runs lqr_iter iterations whatever its batch."""
    net = loop_net(n, m, seed, n_prev)
    layers = _layers(net, dtype)
    C, c = _cost(seed, 1 if time_invariant else T, B, n + m)
    if time_invariant:
        C, c = C.expand(T, *C.shape[1:]).contiguous(), c.expand(T, *c.shape[1:]).contiguous()
    c = 0.5 * c
    g = torch.Generator().manual_seed(seed + 1)
    x0 = torch.randn(B, n, generator=g, dtype=F64)
    kw = {}
    if mode == "box":
        kw = dict(u_lower=-0.5, u_upper=0.5)
    elif mode in ("tensor", "boxD"):
        kw = dict(u_lower=-0.2 - 0.6 * torch.rand(T, B, m, generator=g, dtype=F64),
                  u_upper=0.2 + 0.6 * torch.rand(T, B, m, generator=g, dtype=F64))
        if mode == "boxD":
            kw["delta_u"] = 0.3
    elif mode == "mask":
        kw["u_zero_I"] = torch.rand(T, B, m, generator=g) < 0.3
    P = {k: round_through(v, dtype) for k, v in dict(C=C, c=c, x0=x0).items()}
    kw = {k: round_through(v, dtype) for k, v in kw.items()}
    opts = dict(lqr_iter=lqr_iter, eps=0.0, not_improved_lim=lqr_iter + 1)
    o64 = mo.ilqr(n, m, T, P["x0"], P["C"], P["c"], layers, "sigmoid", False, n_prev=n_prev, coupled=False, **kw,
                  **opts)
    o32 = None
    if dtype == F32:
        f = lambda t: t.float() if torch.is_tensor(t) and t.is_floating_point() else t  # noqa: E731
        o32 = mo.ilqr(n, m, T, f(P["x0"]), f(P["C"]), f(P["c"]), [(W.float(), b.float()) for W, b in layers],
                      "sigmoid", False, u_init=torch.zeros(T, B, m), n_prev=n_prev, coupled=False,
                      **{k: f(v) for k, v in kw.items()}, **opts)
    bound = float(layers[-1][0].abs().sum(1).max()) + float(layers[-1][1].abs().max())
    assert float(o64[0][1:, :, n_prev:].abs().max()) <= bound + 1e-12, "a state left the network's range"

    def sensitive(tol):
        """[B]: the problems whose float64 oracle loop moves by more than tol in x or u, or changes its controls on
        a bound, when C is scaled by 1 +- 1e-15 (float64 round-off): round-off decides their paths."""
        lay64 = _layers(net, dtype)
        moved = torch.zeros(B, dtype=torch.bool)
        for s_ in (1 + 1e-15, 1 - 1e-15):
            o = mo.ilqr(n, m, T, P["x0"], P["C"] * s_, P["c"], lay64, "sigmoid", False, n_prev=n_prev, coupled=False,
                        **kw, **opts)
            moved |= torch.maximum((o[0] - o64[0]).abs().amax((0, 2)), (o[1] - o64[1]).abs().amax((0, 2))) > tol
            if "u_lower" in kw:
                moved |= (on_bounds(o[1], kw) != on_bounds(o64[1], kw)).any(3).any(1).any(0)
        return moved
    return net, P, kw, opts, o64, o32, sensitive


def run_mlp_loop(net, n, m, T, P, kw, opts, dtype, impl=None, n_prev=0, idx=None):
    d = lambda t: t.to(DEV, dtype) if torch.is_tensor(t) and t.is_floating_point() else (  # noqa: E731
        t.to(DEV) if torch.is_tensor(t) else t)
    P = {k: _rows(v, idx) for k, v in P.items()} if idx is not None else P
    kw = {k: _rows(v, idx) for k, v in kw.items()} if idx is not None else kw
    net_d = net.to(dtype=dtype, device=DEV)
    dxm = CtrlPassthroughDynamics(net_d) if n_prev else net_d
    B = P["x0"].shape[0]
    u0 = torch.zeros(T, B, m, dtype=dtype, device=DEV)
    with kernel_env(impl), poisoned_empty():
        res = mlpmod.ilqr_raw(dxm, n, m, T, d(P["x0"]), d(P["C"]), d(P["c"]), u0, **{k: d(v) for k, v in kw.items()},
                              **opts)
        p = _lib.last_step_plan()
    assert res is not None, "the driver has no conditional graph nodes"
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in res.items()}, p


def check_mlp_loop(tag, r, case, dtype, idx=None):
    """x, u and costs per problem against the oracle under gpu_harness.check_loop_departures (at (16, 4) T = 101 and
    (18, 5) with tensor bounds, 5 of 8 and 7 of 16 problems depart where the oracle's own loop moves, by up to 1e-4),
    and the iteration count."""
    _, P, kw, opts, o64, o32, sensitive = case
    LOOP_DEPARTED.append(check_loop_departures(tag, r, o64, o32, kw, opts["lqr_iter"], sensitive, dtype, idx)[:3])
    assert int(r["info"][0]) == opts["lqr_iter"], f"{tag}: {int(r['info'][0])} iterations"


@functools.lru_cache(maxsize=None)
def earliest(which, dtype):
    """(n, m, T*) of the instance whose `which` switch (generic_riccati or pair_nofit, probed with do_rollout =
    False, the loop body's step) comes first within ORACLE_TMAX; None if none has it."""
    cands = []
    for n, m in (INSTANCES if which == "generic_riccati" else PAIR_SHAPES):
        Ts = switches(n, m, dtype)[which]
        if Ts is not None and 3 <= Ts <= ORACLE_TMAX:
            cands.append((Ts, n + m, n, m))
    if not cands:
        return None
    Ts, _, n, m = min(cands)
    return n, m, Ts


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("which", ["generic_riccati", "pair_nofit"])
def test_mlp_loop_plans_at_switch(which, dtype):
    """The MLP loop just below and at the switch: the forced kernel's plan is asserted from the switch, the default
    dispatch's from a probe of the loop body's step (do_rollout = False, gains buffers given), and every run is
    compared with the oracle."""
    pick = earliest(which, dtype)
    if pick is None:
        pytest.skip(f"no instance has a {which} switch within T <= {ORACLE_TMAX}")
    n, m, Ts = pick
    impl = 1 if which == "generic_riccati" else 2
    for k, T in enumerate((Ts - 1, Ts)):
        mode = ("free", "tensor")[k]
        # float32: one iteration; at these horizons later iterations compare costs of hundreds of stages that
        # differ by less than float32 resolves, so round-off would decide their line searches
        case = loop_case(1500 + k + 10 * impl, 8, T, n, m, dtype, mode, lqr_iter=3 if dtype == F64 else 1)
        for im in (impl, None):
            want = plan(impl == 1, T < Ts) if im == impl else probe_step(n, m, dtype, T, None, True, False)
            tag = f"{which} n{n}m{m} {DT[dtype]} T={T} (T*={Ts}) {mode} MPCB200_KERNEL={im}"
            r, p = run_mlp_loop(case[0], n, m, T, *case[1:4], dtype, im)
            assert p == want, f"{tag}: plan {plan_str(p)}, expected {plan_str(want)}"
            LOOP_SEEN.setdefault(dtype, set()).add(loop_plan_name(p))
            check_mlp_loop(tag, r, case, dtype)


# (n, m, impl, mode, n_prev, staged (N, M)): the large-shape kernel forced at an instance, a shape no instance covers,
# a shape padded to an instance ((5, 3) -> (7, 4)); tensor bounds, delta_u and u_zero_I; the slew-rate passthrough
# form, padded ((5, 2) -> (6, 2)) and exact
LOOP_CASES = [(3, 2, 3, "box", 0, (3, 2)), (18, 5, None, "tensor", 0, (18, 5)), (5, 3, None, "boxD", 0, (7, 4)),
              (3, 2, None, "mask", 0, (3, 2)), (4, 2, None, "tensor", 0, (4, 2)), (5, 2, None, "box", 2, (6, 2)),
              (6, 2, None, "mask", 2, (6, 2))]


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("n,m,impl,mode,n_prev,staged_nm", LOOP_CASES,
                         ids=[f"n{c[0]}m{c[1]}_k{c[2]}_{c[3]}_p{c[4]}" for c in LOOP_CASES])
def test_mlp_loop_inputs_and_shapes(n, m, impl, mode, n_prev, staged_nm, dtype):
    """The loop's plan is the one the step records at the staged instance with do_rollout = False and gains buffers
    (probe_step), and the large-shape kernels wherever they were asked for or no instance covers the shape."""
    from mpc.pytorch_b200.step import _pick_instance
    T, B = 10, 16
    assert _pick_instance(n, m, ESZ[dtype]) == staged_nm
    case = loop_case(1600 + n + 7 * m + n_prev, B, T, n, m, dtype, mode, n_prev=n_prev)
    r, p = run_mlp_loop(case[0], n, m, T, *case[1:4], dtype, impl, n_prev)
    want = probe_step(*staged_nm, dtype, T, impl, True, False)
    tag = f"n{n}m{m} {mode} n_prev={n_prev} {DT[dtype]} MPCB200_KERNEL={impl}"
    assert p == want, f"{tag}: plan {plan_str(p)}, expected {plan_str(want)}"
    assert (p == _lib.PLAN_LARGE) == (impl == 3 or (n, m) == (18, 5)), f"{tag}: plan {plan_str(p)}"
    LOOP_SEEN.setdefault(dtype, set()).add(loop_plan_name(p))
    check_mlp_loop(tag, r, case, dtype)
    if n_prev:
        assert torch.equal(r["x"][1:, :, :n_prev], r["u"][:-1]), f"{tag}: previous controls"


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
def test_mlp_loop_time_invariant_cost_through_mpc_forward(dtype):
    n, m, T, B = 3, 2, 10, 12
    case = loop_case(1700, B, T, n, m, dtype, "box", time_invariant=True)
    net, P, kw, opts, o64, o32, _ = case
    net_d = net.to(dtype=dtype, device=DEV)
    C0, c0 = P["C"][:1].to(DEV, dtype), P["c"][:1].to(DEV, dtype)
    cost = QuadCost(C0.expand(T, *C0.shape[1:]), c0.expand(T, *c0.shape[1:]))
    ctrl = MPC(n, m, T, u_lower=kw["u_lower"], u_upper=kw["u_upper"], lqr_iter=opts["lqr_iter"], eps=0.0,
               not_improved_lim=opts["not_improved_lim"], verbose=-1, grad_method=GradMethods.ANALYTIC,
               exit_unconverged=False, detach_unconverged=False)
    calls = []
    real = mlpmod.ilqr_raw
    mlpmod.ilqr_raw = lambda *a, **k: calls.append(a[5].stride(0)) or real(*a, **k)
    try:
        with torch.no_grad(), poisoned_empty():
            x, u, costs = ctrl(P["x0"].to(DEV, dtype), cost, net_d)
    finally:
        mlpmod.ilqr_raw = real
    assert calls == [0], calls                   # the device loop ran, on the stride-0 (time-invariant) cost
    r = dict(x=x.cpu(), u=u.cpu(), costs=costs.cpu(), info=ctrl._solve_info.cpu())
    check_mlp_loop(f"time-invariant cost {DT[dtype]}", r, case, dtype)


FULL_B = MAX_CTAS * MAX_WARPS + 2 * MAX_WARPS + 3     # every rollout / line-search warp takes a second problem


def full_samples(B, W=MAX_WARPS):
    """First and last problem of a CTA, of the first and second grid pass and of the batch (one problem per warp)."""
    span = MAX_CTAS * W
    s = {0, W - 1, W, 2 * W - 1, span - 1, span, span + W - 1, B - 1, B - 2}
    return sorted(b for b in s if 0 <= b < B)


def test_mlp_loop_full_size_batch():
    """B past 1024 x 8 problems: the rollout and line search take two grid-stride passes inside the graph.  The
    batch tiles a pool of K problems (K coprime to 8), so the oracle solves K problems; sampled rows are compared
    with it, and each solved alone gives its row bit for bit."""
    n, m, T, dtype = 3, 2, 6, F32
    K = pool_size(MAX_WARPS, MAX_CTAS * MAX_WARPS)
    case = loop_case(1800, K, T, n, m, dtype, "free")
    net, P, kw, opts, o64, o32, _ = case
    idx = torch.arange(FULL_B) % K
    r, _ = run_mlp_loop(net, n, m, T, P, kw, opts, dtype, idx=idx)
    assert grid_passes(FULL_B, MAX_WARPS) == 2
    samples = torch.tensor(full_samples(FULL_B))
    sub = {k: (v[:, samples] if v.dim() == 3 else v[samples]) if k != "info" else v for k, v in r.items()}
    check_mlp_loop(f"full size B={FULL_B}", sub, case, dtype, idx=idx[samples])
    for b in samples.tolist():
        one, _ = run_mlp_loop(net, n, m, T, P, kw, opts, dtype, idx=idx[b:b + 1])
        assert torch.equal(one["x"], r["x"][:, b:b + 1]) and torch.equal(one["u"], r["u"][:, b:b + 1]), b


def test_zz_mlp_loop_plan_coverage():
    if not LOOP_SEEN:
        pytest.skip("no MLP loop test of this module ran")
    missing = []
    for dtype in (F64, F32):
        need = {"large"}
        if earliest("generic_riccati", dtype) is not None:
            need |= {"generic_smem", "generic_ks"}
        if earliest("pair_nofit", dtype) is not None:
            need |= {"pair_smem", "pair_ks"}
        seen = LOOP_SEEN.get(dtype, set())
        print(f"{DT[dtype]}: switches generic_riccati {earliest('generic_riccati', dtype)} pair_nofit "
              f"{earliest('pair_nofit', dtype)}; plans run in the MLP loop {sorted(seen)}")
        missing += [f"{DT[dtype]} {p}" for p in sorted(need - seen)]
    print(f"problems departing from the oracle: {sum(a for _, a, _ in LOOP_DEPARTED)} of "
          f"{sum(b for _, _, b in LOOP_DEPARTED)} compared, in {sum(a > 0 for _, a, _ in LOOP_DEPARTED)} of "
          f"{len(LOOP_DEPARTED)} loops:", [(t, a, b) for t, a, b in LOOP_DEPARTED if a])
    for k, v in sorted(LAUNCH_REPORT.items()):
        print("launch shape", k, v)
    assert not missing, "plans never run inside the MLP loop: " + ", ".join(missing)


# ------------------------------------------------------------------------------------------------------------------
# C. episodes at batch scale
# ------------------------------------------------------------------------------------------------------------------
EP_N, EP_M, EP_T, EP_B, EP_STEPS, EP_HIDDEN = 3, 1, 6, 512, 4, (16,)


def _ep_plant(kind, dtype):
    from tests.test_receding_mlp_gpu import _lindx_plant, _pendulum
    if kind == "lindx":
        return _lindx_plant(EP_N, EP_M, EP_B, dtype)
    if kind == "pendulum":
        return _pendulum(dtype)
    return None


@functools.lru_cache(maxsize=2)
def episode_run(kind, dtype):
    from tests.test_receding_mlp_gpu import _device, _net as ep_net, _problem, _w
    dx = ep_net(EP_N, EP_M, list(EP_HIDDEN), "sigmoid", True, dtype)
    x0, C, c = _problem(EP_N, EP_M, EP_T, EP_B, dtype)
    plant = _ep_plant(kind, dtype)
    w = _w(EP_STEPS, EP_B, EP_N, dtype)
    ctrl = MPC(EP_N, EP_M, EP_T, u_lower=-0.8, u_upper=0.8, lqr_iter=4, verbose=-1, grad_method=GradMethods.ANALYTIC,
               exit_unconverged=False, detach_unconverged=False, eps=0.0, not_improved_lim=10)
    res, plan_x, plan_u = _device(ctrl, x0, QuadCost(C, c), dx, EP_STEPS, plant if plant is not None else dx, w)
    return dx, x0, C, c, plant, w, ctrl, res, plan_x, plan_u


def _plant_step(kind, plant, dtype):
    """The oracle's x' = plant(x, u, theta) on CPU tensors of dtype (theta None: the plant's own parameters)."""
    if kind == "lindx":
        F, f = plant.F.cpu().to(dtype), plant.f.cpu().to(dtype)
        n, p = EP_N, EP_N + EP_M

        def lin(x, u, th=None):
            if th is None:
                return lo.lindx_step(F, f, x, u)
            Fb = th[:, :n * p].view(-1, n, p)
            return (Fb @ torch.cat((x, u), 1).unsqueeze(2)).squeeze(2) + th[:, n * p:]
        return lin
    from mpc.pytorch_b200.dynamics import PendulumDx
    mod = PendulumDx(params=plant.params.detach().cpu().to(dtype))

    def pend(x, u, th=None):
        if th is not None:
            mod.params = th.t()
        return mod(x, u)
    return pend


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("kind", ["self", "lindx", "pendulum"])
def test_episode_forward_applies_the_oracle_step_to_the_device_plans(kind, dtype):
    """Every applied control is its plan's first control, every next state the oracle's step (the network, the
    LinDx plant or the pendulum) of the device's own state and control plus w_k; a sample of the plans is the
    oracle's iLQR (eps = 0, so its solve does not depend on the rest of the batch) from the device's state and
    the shifted warm start."""
    dx, x0, C, c, plant, w, ctrl, res, plan_x, plan_u = episode_run(kind, dtype)
    xs, us = res["x"].cpu().double(), res["u"].cpu().double()
    pu = plan_u.cpu().double()
    assert torch.equal(res["u"].cpu(), plan_u[:, 0].cpu()), "applied controls are not the plans' first"
    layers = _layers(dx, dtype)
    wc = w.cpu().double()
    steps = []
    for ld in ((layers, None),) + ((([(W.float(), b.float()) for W, b in layers]), torch.float32),) * (dtype == F32):
        lay, d32 = ld
        cast = (lambda t: t) if d32 is None else (lambda t: t.float())
        if kind == "self":
            nxt = torch.stack([mo.step(lay, "sigmoid", True, cast(xs[k]), cast(us[k])) for k in range(EP_STEPS)])
        else:
            stp = _plant_step(kind, plant, F64 if d32 is None else torch.float32)
            nxt = torch.stack([stp(cast(xs[k]), cast(us[k])) for k in range(EP_STEPS)])
        steps.append((nxt + cast(wc)).double())
    within(f"episode {kind} {DT[dtype]}", "x_{k+1}", xs[1:], steps[0], steps[1] if dtype == F32 else None, dtype,
           tol64=1e-12)
    assert int(res["info"][:, 0].min()) == int(res["info"][:, 0].max()) == ctrl.lqr_iter
    if dtype == F32:
        return
    # a sample of the plans against the oracle's iLQR on that step's problem
    Cc, cc = C.cpu(), c.cpu()
    for b in (0, 255, 256, EP_B - 1):
        for k in (0, EP_STEPS - 1):
            wk = torch.zeros(EP_T, 1, EP_M, dtype=F64) if k == 0 else lo.shift_warm_start(pu[k - 1][:, b:b + 1])
            ox, ou, _, _ = mo.ilqr(EP_N, EP_M, EP_T, xs[k][b:b + 1], Cc[:, b:b + 1], cc[:, b:b + 1], layers,
                                   "sigmoid", True, u_init=wk, u_lower=-0.8, u_upper=0.8, lqr_iter=ctrl.lqr_iter,
                                   eps=0.0, not_improved_lim=10, coupled=False)
            sc = max(1.0, float(ox.abs().max()))
            assert maxdiff(plan_x[k][:, b:b + 1].cpu(), ox) < 2e-6 * sc, (b, k, maxdiff(plan_x[k][:, b:b + 1].cpu(), ox))
            assert maxdiff(pu[k][:, b:b + 1], ou) < 2e-6 * sc, (b, k)


def _vjp_slots(items, nparams):
    from tests.test_mlp_grad_cpu import slots
    return slots(items, nparams)


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("kind", ["self", "lindx", "pendulum"])
def test_episode_reverse_sweep_matches_the_oracle_and_repeats(kind, dtype):
    """The reverse sweep on the device's own plans against receding_mlp_oracle.backward: dx_init, dC, dc, dtheta,
    the plant's gradients and dw.  float64 within 1e-11 of each gradient's max; float32 under `within`, against the
    oracle run in float32 on the same float32 plans, weights and upstream gradients.  dtheta bitwise equal across
    two calls.  (T-1) x B = 2560 linearisation items over min(2560, 2048) VJP slots: slots take a second item."""
    dx, x0, C, c, plant, w, ctrl, res, plan_x, plan_u = episode_run(kind, dtype)
    nparams = n_params(widths_of(EP_N, EP_M, EP_HIDDEN))
    G = _vjp_slots((EP_T - 1) * EP_B, nparams)
    assert 1 < G < (EP_T - 1) * EP_B
    g = torch.Generator().manual_seed(9)
    gx = round_through(torch.randn(EP_STEPS + 1, EP_B, EP_N, generator=g, dtype=F64), dtype)
    gu = round_through(torch.randn(EP_STEPS, EP_B, EP_M, generator=g, dtype=F64), dtype)
    with torch.no_grad(), poisoned_empty():
        a = mlpmod.episode_backward_raw(res["saved"], gx.to(DEV, dtype), gu.to(DEV, dtype))
        b = mlpmod.episode_backward_raw(res["saved"], gx.to(DEV, dtype), gu.to(DEV, dtype))
    torch.cuda.synchronize()
    assert torch.equal(a[3], b[3]), "dtheta differs between two calls"
    layers = _layers(dx, dtype)
    theta = None
    if kind == "lindx":
        theta = torch.cat((plant.F[0].cpu().reshape(EP_B, -1), plant.f[0].cpu()), 1).double()
    elif kind == "pendulum":
        theta = plant.params.detach().cpu().double().view(1, -1).expand(EP_B, -1).contiguous()

    def oracle(odt):
        cast = lambda t: None if t is None else t.cpu().to(odt)  # noqa: E731
        stp = None if kind == "self" else _plant_step(kind, plant, odt)
        o = rmo.backward(EP_N, EP_M, EP_T, cast(C), cast(c), [(cast(W), cast(bb)) for W, bb in layers], "sigmoid",
                         True, cast(res["x"]), cast(res["u"]), cast(plan_x), cast(plan_u), cast(gx), cast(gu),
                         u_lower=-0.8, u_upper=0.8, plant=stp, theta=cast(theta))
        out = {"dx_init": o["dx_init"], "dC": o["dC"], "dc": o["dc"], "dw": o["dw"],
               "dtheta": torch.cat([t.reshape(-1) for wb in o["dlayers"] for t in wb])}
        p = EP_N + EP_M
        if kind == "lindx":
            out["dF_plant"] = o["dtheta_plant"][:, :EP_N * p].reshape(EP_B, EP_N, p)
            out["df_plant"] = o["dtheta_plant"][:, EP_N * p:]
        elif kind == "pendulum":
            out["dtheta_plant"] = o["dtheta_plant"]
        return {k: v.double() for k, v in out.items()}
    o64 = oracle(F64)
    o32 = oracle(torch.float32) if dtype == F32 else None
    got = {"dx_init": a[0], "dC": a[1], "dc": a[2], "dtheta": a[3], "dF_plant": a[4], "df_plant": a[5],
           "dtheta_plant": a[6], "dw": a[7]}
    for name, want in o64.items():
        g_ = got[name].cpu().double()
        if dtype == F64:
            sc = max(1e-30, float(want.abs().max()))
            err = maxdiff(g_, want)
            assert err <= 1e-11 * sc, f"{kind}: {name} |device - oracle| = {err:.3e}, max|g| = {sc:.3e}"
        else:
            within(f"episode backward {kind} f32", name, g_, want, o32[name], dtype)
