"""GPU: a slew-rate penalty on the device.  The control-passthrough kind of the known systems (state [u_{t-1}; x]) in
the rollout and linearisation kernels and in the dynamics-only step instances, against CtrlPassthroughDynamics(module)
and the float64 oracle; and MPC.forward with slew_rate_penalty on the device loop, bitwise against the host loop, for
the known systems and for LinDx at exact, zero-padded and large augmented shapes."""
import ctypes

import pytest
import torch

from mpc.pytorch_b200 import _lib, step
from mpc.pytorch_b200.dynamics import dyn_linearize_raw, dyn_rollout_raw
from mpc.pytorch_b200.solver import MPC, CtrlPassthroughDynamics, GradMethods, LinDx, QuadCost
from oracle import lqr_oracle as orc
from tests.gpu_harness import (BT, DEV, F32, F64, PHYS, SYSTEMS, check_alphas, check_clamps, check_pnqp,
                               check_trajectory, known_controls, known_module, known_states, linearise, rollout,
                               run_step, same_on_both_loops, solve_on, within)
from tests.helpers import gen_problem, load_golden, maxdiff

pytestmark = pytest.mark.gpu


def _augknown_states(name, B, T, dtype, seed):
    """[B, n+1] passthrough states (previous control, then the system's edge states) and [T, B, 1] controls."""
    u = known_controls(name, T, B, dtype, seed)
    prev = known_controls(name, 1, B, dtype, seed + 5)[0]
    return torch.cat((prev, known_states(name, B, seed)), 1), u


# ------------------------------------------------------------------------------------------------------------------
# rollout and linearisation
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,T", BT, ids=[f"B{b}_T{t}" for b, t in BT])
@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("name", SYSTEMS)
def test_passthrough_rollout_matches_module(name, dtype, B, T):
    """Every step of the passthrough rollout against CtrlPassthroughDynamics(module) from the kernel's own state;
    the first M states of each next state are the control exactly as given, before the system's clamp."""
    pt = CtrlPassthroughDynamics(known_module(name))
    x0, u = _augknown_states(name, B, T, dtype, 10 + B + T)
    x0, u = x0.to(dtype), u.to(dtype)
    x = dyn_rollout_raw(pt.mpcb200_kind, pt.mpcb200_params(), T, x0.to(DEV), u.to(DEV)).cpu()
    assert x.shape == (T, B, pt.n_state) and x.dtype == dtype
    assert torch.equal(x[0], x0)
    if T == 1:
        return
    assert torch.equal(x[1:, :, :1], u[:-1])
    pt32 = CtrlPassthroughDynamics(known_module(name, params=torch.tensor(PHYS[name]["params"], dtype=F32)))
    xs, us = x[:-1].reshape(-1, pt.n_state).double(), u[:-1].reshape(-1, 1).double()
    w64 = pt(xs, us).view(T - 1, B, -1)
    w32 = pt32(xs.float(), us.float()).view(T - 1, B, -1) if dtype == F32 else None
    within(f"{name} B={B} T={T}", "rollout", x[1:], w64, w32, dtype, 1e-12)


@pytest.mark.parametrize("B,T", BT, ids=[f"B{b}_T{t}" for b, t in BT])
@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("name", SYSTEMS)
def test_passthrough_linearisation_matches_autograd(name, dtype, B, T):
    """F~, f~ of the linearisation kernel against autograd of CtrlPassthroughDynamics(module) at states off the unit
    circle, theta edges, previous and current controls at / one ulp either side of the clamp; and bitwise the blocks
    MPC._slew_augment assembles from the system's own linearisation kernel."""
    dx = known_module(name)
    pt = CtrlPassthroughDynamics(dx)
    n = pt.n_state
    prm = pt.mpcb200_params()
    x = torch.stack([_augknown_states(name, B, 1, dtype, 30 + t)[0] for t in range(T)]).to(dtype)
    u = known_controls(name, T, B, dtype, 40 + B + T).to(dtype)
    F, f = dyn_linearize_raw(pt.mpcb200_kind, prm, T, x.to(DEV), u.to(DEV))
    assert F.shape == (T - 1, B, n, n + 1) and f.shape == (T - 1, B, n)
    if T == 1:
        assert F.numel() == 0 and f.numel() == 0
        return
    pt32 = CtrlPassthroughDynamics(known_module(name, params=torch.tensor(PHYS[name]["params"], dtype=F32)))
    Fw, fw = linearise(pt, x.to(F64), u.to(F64))
    F32w, f32w = linearise(pt32, x.to(F32), u.to(F32)) if dtype == F32 else (None, None)
    tag = f"{name} B={B} T={T}"
    within(tag, "F", F.cpu(), Fw, F32w, dtype, 1e-11)
    within(tag, "f", f.cpu(), fw, f32w, dtype, 1e-11)
    Fi, fi = dyn_linearize_raw(dx.mpcb200_kind, prm, T, x[..., 1:].contiguous().to(DEV), u.to(DEV))
    ctrl = MPC(dx.n_state, 1, T, slew_rate_penalty=1.0)
    C = torch.zeros(T, B, n, n, dtype=dtype, device=DEV)          # the system's own (n_state + 1)^2
    _, _, _, F2, f2, _, _ = ctrl._slew_augment(x[0, :, 1:].to(DEV), C, C[..., 0], Fi, fi)
    assert torch.equal(F, F2) and torch.equal(f, f2)


# ------------------------------------------------------------------------------------------------------------------
# the fused step on the dynamics-only instances
# ------------------------------------------------------------------------------------------------------------------
def _step_case(name, B, T, bounds, seed, calm=False):
    """A float64 passthrough LQR step around a module rollout, and the oracle's step with the module as dynamics.
    `calm`: the system starts near its resting angle with small controls, so that long horizons stay bounded."""
    g = torch.Generator().manual_seed(seed)
    pt = CtrlPassthroughDynamics(known_module(name))
    clamp = PHYS[name]["clamp"]
    x0, u = _augknown_states(name, B, T, F64, seed)
    x0[:, 0] *= 0.2
    u = u * 0.2
    if calm:
        th = torch.pi + 0.4 * (torch.rand(B, generator=g, dtype=F64) - 0.5)
        ic, is_ = (3, 4) if name == "cartpole" else (1, 2)
        x0[:, ic], x0[:, is_] = torch.cos(th), torch.sin(th)
        u = u * 0.5
    x = rollout(pt, x0, u)
    n = x.shape[2]
    p = n + 1
    F, f = linearise(pt, x, u)
    L = torch.randn(T, B, p, p, generator=g, dtype=F64) / p ** 0.5
    C = L @ L.transpose(-1, -2) + 0.5 * torch.eye(p, dtype=F64)
    c = torch.randn(T, B, p, generator=g, dtype=F64)
    c[..., n:] *= 0.2 * clamp
    kw = dict(linesearch_decay=0.3, max_linesearch_iter=4)
    if bounds == "scalar":
        kw.update(u_lower=-0.8 * clamp, u_upper=0.8 * clamp)
    elif bounds == "wide":
        kw.update(u_lower=-2.0 * clamp, u_upper=2.0 * clamp)
    P = dict(x0=x0, C=C, c=c, F=F, f=f, x=x, u=u)
    o = orc.lqr_step_forward(n, 1, T, x0, C, c, F, f, x, u, coupled=False, dynamics=pt, **kw)
    return P, kw, o


def _kernel_step(name, T, P, kw, monkeypatch):
    """lqr_step_raw with the passthrough kind (alphas, free sets, pnqp counts) and LQRStep with
    true_dynamics=CtrlPassthroughDynamics(known) (its outputs; split mode must not run)."""
    pt = CtrlPassthroughDynamics(known_module(name))
    n = pt.n_state
    r, plan = run_step(n, 1, T, P, kw, want_gains=False, dyn=(pt.mpcb200_kind, pt.mpcb200_params()))

    def no_split(*a, **k):
        raise AssertionError("split-mode rollout ran")
    monkeypatch.setattr(step, "rollout_split", no_split)
    C, c, F, f = (P[k].to(DEV) for k in ("C", "c", "F", "f"))
    nx, nu, _, costs, _, _ = step.LQRStep(n, 1, T, true_cost=QuadCost(C, c), true_dynamics=pt,
                                          current_x=P["x"].to(DEV), current_u=P["u"].to(DEV), **kw)(
        P["x0"].to(DEV), C, c, F, f)
    for k, v in (("new_x", nx), ("new_u", nu), ("costs", costs)):
        assert torch.equal(v.cpu(), r[k]), k
    return r, plan


def _check_step(tag, r, P, kw, o):
    check_alphas(tag, r, o, None)
    check_trajectory(tag, r, P["u"], o, None, F64)
    check_pnqp(tag, r, o, kw)
    check_clamps(tag, r, o, kw)


# problems per CTA of the dynamics-only instances in float64: (6, 1) W = 4, (4, 1) W = 6; the bulk path needs B even
STEP_BATCHES = [("cartpole", 13), ("cartpole", 14), ("pendulum", 13), ("pendulum", 20)]


@pytest.mark.parametrize("bounds", [None, "scalar", "wide"])
@pytest.mark.parametrize("name,B", STEP_BATCHES, ids=[f"{s}_B{b}" for s, b in STEP_BATCHES])
def test_passthrough_step_matches_oracle(name, B, bounds, monkeypatch):
    T = 12
    P, kw, o = _step_case(name, B, T, bounds, 300 + B)
    r, plan = _kernel_step(name, T, P, kw, monkeypatch)
    tag = f"{name} B={B} {bounds}"
    assert plan & _lib.PLAN_GENERIC, f"{tag}: plan {plan}"
    _check_step(tag, r, P, kw, o)


def _gain_switch(kind, n, esz):
    L = _lib.lib()
    for T in range(2, 4096):
        d = _lib.Dims(B=1, T=T, n=n, m=1, F_T=T - 1, dynamics_kind=kind, max_ls_iter=1, pnqp_max_iter=1,
                      do_rollout=1)
        if L.mpcb200_step_prefers_workspace(ctypes.byref(d), esz):
            return T
    return None


@pytest.mark.parametrize("name", SYSTEMS)
def test_passthrough_step_on_both_sides_of_the_gain_store_switch(name, monkeypatch):
    pt = CtrlPassthroughDynamics(known_module(name))
    Ts = _gain_switch(pt.mpcb200_kind, pt.n_state, 8)
    assert Ts is not None and 2 < Ts <= 1024, Ts
    for T in (Ts - 1, Ts):
        P, kw, o = _step_case(name, 6, T, "scalar", 800 + T, calm=True)
        r, plan = _kernel_step(name, T, P, kw, monkeypatch)
        tag = f"{name} T={T} (switch {Ts})"
        assert plan & _lib.PLAN_GENERIC, tag
        assert bool(plan & _lib.PLAN_GAINS_SMEM) == (T < Ts), f"{tag}: plan {plan}"
        _check_step(tag, r, P, kw, o)


# ------------------------------------------------------------------------------------------------------------------
# MPC.forward with a slew-rate penalty: device loop vs host loop
# ------------------------------------------------------------------------------------------------------------------
def _same_full_du_norm(tag, dev, host):
    """full_du_norm, which the device loop sums in another order (DESIGN section 3.5): 1e-12 (float64) / 1e-5
    (float32) relative."""
    a, b = dev.full_du_norm, host.full_du_norm
    rtol = 1e-12 if a.dtype == F64 else 1e-5
    assert torch.allclose(a, b, rtol=rtol, atol=0), f"{tag}: full_du_norm {float((a - b).abs().max())}"


def _known_problem(name, B, T):
    dx = known_module(name, params=torch.tensor(PHYS[name]["params"], dtype=F64, device=DEV).requires_grad_(True),
                 device=DEV)
    n = dx.n_state
    q, p = dx.get_true_obj()
    Q = torch.diag(q).double().expand(T, B, n + 1, n + 1).contiguous().to(DEV).requires_grad_(True)
    pp = p.double().expand(T, B, n + 1).contiguous().to(DEV).requires_grad_(True)
    return dx, Q, pp, known_states(name, B, 40 + B).to(DEV)


KNOWN_CASES = [("in", None, None), ("wide", None, None), ("in", 0.3, None), ("in", None, "m"), ("wide", 0.5, "Bm")]


@pytest.mark.parametrize("bounds,delta,prev", KNOWN_CASES, ids=[f"{b}_du{d}_prev{p}" for b, d, p in KNOWN_CASES])
@pytest.mark.parametrize("name", SYSTEMS)
def test_known_system_slew_device_loop_equals_host_loop(name, bounds, delta, prev, monkeypatch):
    B, T = 24, 15
    clamp = PHYS[name]["clamp"]
    dx, Q, pp, x0 = _known_problem(name, B, T)
    b = (0.8 if bounds == "in" else 2.0) * clamp
    g = torch.Generator().manual_seed(7)
    pc = {None: None, "m": torch.tensor([0.3 * clamp], dtype=F64),
          "Bm": (torch.rand(B, 1, generator=g, dtype=F64) - 0.5) * clamp}[prev]
    kw = dict(u_lower=-b, u_upper=b, lqr_iter=8, verbose=-1, exit_unconverged=False, detach_unconverged=False,
              linesearch_decay=0.3, max_linesearch_iter=4, grad_method=GradMethods.AUTO_DIFF, eps=1e-9,
              slew_rate_penalty=0.5, prev_ctrl=None if pc is None else pc.to(DEV),
              delta_u=None if delta is None else delta * clamp)
    make = lambda: MPC(dx.n_state, 1, T, **kw)
    cost = QuadCost(Q, pp)
    tag = f"{name} {bounds} delta {delta} prev {prev}"
    dev, host = same_on_both_loops(monkeypatch, make, x0, cost, dx, grads=(Q, pp, dx.params))
    _same_full_du_norm(tag, dev, host)
    assert float(dev.grads[2].abs().max()) > 0, f"{tag}: no gradient reaches the system parameters"

    class Opaque(torch.nn.Module):                      # hides mpcb200_kind: today's Module path (split mode)
        def forward(self, xx, uu):
            return dx(xx, uu)
    x, u, costs = make()(x0, QuadCost(Q.detach(), pp.detach()), Opaque())
    for k, (p, q) in enumerate(((x, dev.x), (u, dev.u))):
        assert maxdiff(p, q) < 1e-7 * max(1.0, float(p.abs().max())), f"{tag}: opaque module {k}"
    assert maxdiff(costs, dev.costs) < 1e-8 * max(1.0, float(costs.abs().max())), f"{tag}: opaque costs"


@pytest.mark.parametrize("name", SYSTEMS)
def test_known_system_slew_follows_parameter_edits(name, monkeypatch):
    B, T = 9, 12
    dx, Q, pp, x0 = _known_problem(name, B, T)
    kw = dict(u_lower=-2.0 * PHYS[name]["clamp"], u_upper=2.0 * PHYS[name]["clamp"], lqr_iter=4, verbose=-1,
              exit_unconverged=False, detach_unconverged=False, slew_rate_penalty=0.2,
              grad_method=GradMethods.AUTO_DIFF)
    make = lambda: MPC(dx.n_state, 1, T, **kw)
    cost = QuadCost(Q.detach(), pp.detach())
    first = solve_on(monkeypatch, make, x0, cost, dx, True)
    with torch.no_grad():
        dx.params.mul_(1.2)
    dev, host = same_on_both_loops(monkeypatch, make, x0, cost, dx)
    _same_full_du_norm(f"{name} after an edit", dev, host)
    assert not torch.equal(first.x, dev.x)


# ------------------------------------------------------------------------------------------------------------------
# LinDx with a slew-rate penalty
# ------------------------------------------------------------------------------------------------------------------
LIN_SHAPES = [(3, 4), (8, 2), (16, 4)]      # augmented (7, 4) exact, (10, 2) padded to (12, 4), (20, 4) large
LIN_CASES = ["scalar", "tensor", "zero_mask"]


@pytest.mark.parametrize("case", LIN_CASES)
@pytest.mark.parametrize("dtype", [F32, F64], ids=["f32", "f64"])
@pytest.mark.parametrize("n,m", LIN_SHAPES, ids=[f"{n}x{m}" for n, m in LIN_SHAPES])
def test_lindx_slew_device_loop_equals_host_loop(n, m, dtype, case, monkeypatch):
    B, T = 40, 10
    C, c, F, f, x0 = [t.to(DEV) for t in gen_problem(5, B, T, n, m, dtype)]
    g = torch.Generator().manual_seed(3)
    kw = dict(lqr_iter=8, verbose=-1, exit_unconverged=False, detach_unconverged=False, slew_rate_penalty=0.7,
              prev_ctrl=(0.2 * torch.randn(B, m, generator=g, dtype=F64)).to(DEV))
    if case == "scalar":
        kw.update(u_lower=-0.3, u_upper=0.3)
    elif case == "tensor":
        lo = -0.1 - 0.3 * torch.rand(T, B, m, generator=g, dtype=dtype)
        kw.update(u_lower=lo.to(DEV), u_upper=(-lo + 0.05).to(DEV))
    else:
        kw.update(u_zero_I=(torch.rand(T, B, m, generator=g) < 0.3).to(DEV))
    Cl, cl = C.requires_grad_(True), c.requires_grad_(True)
    make = lambda: MPC(n, m, T, **kw)
    dev, host = same_on_both_loops(monkeypatch, make, x0, QuadCost(Cl, cl), LinDx(F, f), grads=(Cl, cl))
    _same_full_du_norm(f"({n},{m}) {dtype} {case}", dev, host)


@pytest.mark.parametrize("name", ["slew_box_f64", "slew_unb_f64"])
def test_slew_fixtures_as_lindx_on_the_device_loop(name, monkeypatch):
    """The reference's slew solves (oracle/make_golden.py) posed as LinDx([A, Bm]): the device loop, under the
    tolerances of test_mpc_gpu.py::test_slew_rate_matches_reference_fixture."""
    g = load_golden(name)
    T, B, p = g["C"].shape[:3]
    n = g["x_init"].shape[1]
    m = p - n
    bound = g.get("bound")
    kw = {} if bound is None else dict(u_lower=-float(bound), u_upper=float(bound))
    prev = g["prev_ctrl"].to(DEV) if "prev_ctrl" in g else None
    F = torch.cat((g["A"], g["Bm"]), 1).expand(T - 1, B, n, p).to(DEV)
    make = lambda: MPC(n, m, T, lqr_iter=15, verbose=-1, exit_unconverged=False, detach_unconverged=False,
                       slew_rate_penalty=float(g["penalty"]), prev_ctrl=prev, eps=1e-9, **kw)
    x, u, costs = solve_on(monkeypatch, make, g["x_init"].to(DEV), QuadCost(g["C"].to(DEV), g["c"].to(DEV)),
                           LinDx(F), True)[:3]
    tol = 2e-4 if bound is not None else 1e-8
    assert maxdiff(u, g["u"]) < tol and maxdiff(x, g["x"]) < tol
    assert maxdiff(costs, g["costs"]) < 10 * tol * max(1.0, float(g["costs"].abs().max()))


@pytest.mark.parametrize("bounds", ["in", "wide"])
@pytest.mark.parametrize("name", SYSTEMS)
def test_known_system_slew_matches_reference_fixture(name, bounds, monkeypatch):
    """The reference's own MPC(slew_rate_penalty, prev_ctrl) with its CartpoleDx / PendulumDx (float64, AUTO_DIFF,
    oracle/make_golden_slew.py), against the device loop with the known system in the kernels.  Bounds inside the
    system's clamp and twice as wide (the copied controls then go beyond it), prev_ctrl at, inside and beyond the clamp.
    Tolerances of the known-system fixture tests: costs 1e-7 relative, x and u at pnqp's accuracy (2e-4 x scale; the
    reference couples pnqp's termination over the batch), the saturated controls exactly, and d u* / d c as
    test_models_gpu.py's gradient fixtures (2e-3 x scale)."""
    from mpc.pytorch_b200.dynamics import CartpoleDx, PendulumDx
    g = load_golden(f"known_slew_{name}_f64")
    T, B = g["C"].shape[:2]
    dx = (CartpoleDx if name == "cartpole" else PendulumDx)(params=g["params"].to(DEV))
    dx.dt = float(g["dt"])
    setattr(dx, PHYS[name]["clamp_attr"], float(g["clamp"]))
    n, b = dx.n_state, float(g[f"bound_{bounds}"])
    ctrl = MPC(n, 1, T, u_lower=-b, u_upper=b, lqr_iter=int(g["lqr_iter"]), verbose=-1, exit_unconverged=False,
               detach_unconverged=False, linesearch_decay=float(g["decay"]), max_linesearch_iter=int(g["ls_iter"]),
               grad_method=GradMethods.AUTO_DIFF, eps=1e-9, slew_rate_penalty=float(g["penalty"]),
               prev_ctrl=g["prev_ctrl"].to(DEV))
    C, x0 = g["C"].to(DEV), g["x_init"].to(DEV)
    c = g["c"].to(DEV).requires_grad_(True)
    x, u, costs = solve_on(monkeypatch, lambda: ctrl, x0, QuadCost(C, c), dx, True)[:3]
    wx, wu, wc = g[f"x_{bounds}"], g[f"u_{bounds}"], g[f"costs_{bounds}"]
    tag = f"{name} bounds {bounds}"
    rel = (costs.detach().cpu() - wc).abs() / wc.abs().clamp_min(1.0)
    assert float(rel.max()) < 1e-7, f"{tag}: costs {float(rel.max()):.3e}"
    assert maxdiff(u, wu) < 2e-4 * max(1.0, float(wu.abs().max())), f"{tag}: u {maxdiff(u, wu):.3e}"
    assert maxdiff(x, wx) < 2e-4 * max(1.0, float(wx.abs().max())), f"{tag}: x {maxdiff(x, wx):.3e}"
    assert torch.equal(u.detach().abs().cpu() == b, wu.abs() == b), f"{tag}: saturated controls"
    uf = u.reshape(-1)
    rows = torch.stack([torch.autograd.grad(uf[i], c, retain_graph=True)[0].reshape(-1).cpu()
                        for i in range(uf.numel())])
    want = g[f"du_dc_{bounds}"]
    sc = float(want.abs().max())
    assert maxdiff(rows, want) < 2e-3 * sc, f"{tag}: du/dc {maxdiff(rows, want):.3e} (scale {sc:.3e})"


def test_lindx_slew_solve_makes_no_host_read_and_captures():
    # (3, 4) augments to the exact (7, 4) instance: staging a zero-padded instance indexes on the device
    B, T, n, m = 32, 10, 3, 4
    C, c, F, f, x0 = [t.to(DEV) for t in gen_problem(9, B, T, n, m, F32)]
    make = lambda: MPC(n, m, T, u_lower=-0.3, u_upper=0.3, lqr_iter=6, verbose=-1, exit_unconverged=False,
                       detach_unconverged=False, slew_rate_penalty=0.5, prev_ctrl=torch.zeros(B, m, device=DEV))
    want = make()(x0, QuadCost(C, c), LinDx(F, f))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        with torch.no_grad():
            got = make()(x0, QuadCost(C, c), LinDx(F, f))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        make()(x0, QuadCost(C, c), LinDx(F, f))             # warm-up on the side stream, as torch.cuda.graph wants
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        cap = make()(x0, QuadCost(C, c), LinDx(F, f))
    graph.replay()
    torch.cuda.synchronize()
    for a, b, k in zip(want, got, "xuc"):
        assert torch.equal(a, b), k
    for a, b, k in zip(want, cap, "xuc"):
        assert torch.equal(a, b), k
