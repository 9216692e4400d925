"""GPU: a slew-rate penalty on the device.  The control-passthrough kind of the known systems (state [u_{t-1}; x]) in
the rollout and linearisation kernels and in the dynamics-only step instances, against CtrlPassthroughDynamics(module)
and the float64 oracle; and MPC.forward with slew_rate_penalty on the device loop, bitwise against the host loop, for
the known systems and for LinDx at exact, zero-padded and large augmented shapes."""
import ctypes

import pytest
import torch

from mpc.pytorch_b200 import _lib, solver, step
from mpc.pytorch_b200.dynamics import dyn_linearize_raw, dyn_rollout_raw
from mpc.pytorch_b200.solver import MPC, CtrlPassthroughDynamics, GradMethods, LinDx, QuadCost
from oracle import lqr_oracle as orc
from tests.helpers import gen_problem, load_golden, maxdiff
from tests.test_known_systems_gpu import BT, PHYS, SYSTEMS, _controls, _jac, _module, _states, _within

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
F64, F32 = torch.float64, torch.float32


def _aug_states(name, B, T, dtype, seed):
    """[B, n+1] passthrough states (previous control, then the system's edge states) and [T, B, 1] controls."""
    u = _controls(name, T, B, dtype, seed)
    prev = _controls(name, 1, B, dtype, seed + 5)[0]
    return torch.cat((prev, _states(name, B, seed)), 1), u


# ------------------------------------------------------------------------------------------------------------------
# rollout and linearisation
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,T", BT, ids=[f"B{b}_T{t}" for b, t in BT])
@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("name", SYSTEMS)
def test_passthrough_rollout_matches_module(name, dtype, B, T):
    """Every step of the passthrough rollout against CtrlPassthroughDynamics(module) from the kernel's own state;
    the first M states of each next state are the control exactly as given, before the system's clamp."""
    pt = CtrlPassthroughDynamics(_module(name))
    x0, u = _aug_states(name, B, T, dtype, 10 + B + T)
    x0, u = x0.to(dtype), u.to(dtype)
    x = dyn_rollout_raw(pt.mpcb200_kind, pt.mpcb200_params(), T, x0.to(DEV), u.to(DEV)).cpu()
    assert x.shape == (T, B, pt.n_state) and x.dtype == dtype
    assert torch.equal(x[0], x0)
    if T == 1:
        return
    assert torch.equal(x[1:, :, :1], u[:-1])
    pt32 = CtrlPassthroughDynamics(_module(name, params=torch.tensor(PHYS[name]["params"], dtype=F32)))
    xs, us = x[:-1].reshape(-1, pt.n_state).double(), u[:-1].reshape(-1, 1).double()
    w64 = pt(xs, us).view(T - 1, B, -1)
    w32 = pt32(xs.float(), us.float()).view(T - 1, B, -1) if dtype == F32 else None
    _within(f"{name} B={B} T={T} rollout", x[1:], w64, w32, dtype, 1e-12)


@pytest.mark.parametrize("B,T", BT, ids=[f"B{b}_T{t}" for b, t in BT])
@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("name", SYSTEMS)
def test_passthrough_linearisation_matches_autograd(name, dtype, B, T):
    """F~, f~ of the linearisation kernel against autograd of CtrlPassthroughDynamics(module) at states off the unit
    circle, theta edges, previous and current controls at / one ulp either side of the clamp; and bitwise the blocks
    MPC._slew_augment assembles from the system's own linearisation kernel."""
    dx = _module(name)
    pt = CtrlPassthroughDynamics(dx)
    n = pt.n_state
    prm = pt.mpcb200_params()
    x = torch.stack([_aug_states(name, B, 1, dtype, 30 + t)[0] for t in range(T)]).to(dtype)
    u = _controls(name, T, B, dtype, 40 + B + T).to(dtype)
    F, f = dyn_linearize_raw(pt.mpcb200_kind, prm, T, x.to(DEV), u.to(DEV))
    assert F.shape == (T - 1, B, n, n + 1) and f.shape == (T - 1, B, n)
    if T == 1:
        assert F.numel() == 0 and f.numel() == 0
        return
    xs, us = x[:-1].reshape(-1, n), u[:-1].reshape(-1, 1)
    pt32 = CtrlPassthroughDynamics(_module(name, params=torch.tensor(PHYS[name]["params"], dtype=F32)))

    def lin(mod, dt):
        nx, R, S = _jac(mod, xs.to(dt), us.to(dt))
        fw = nx - torch.einsum("bij,bj->bi", R, xs.to(dt)) - torch.einsum("bij,bj->bi", S, us.to(dt))
        return torch.cat((R, S), 2).view(T - 1, B, n, n + 1), fw.view(T - 1, B, n)
    Fw, fw = lin(pt, F64)
    F32w, f32w = lin(pt32, F32) if dtype == F32 else (None, None)
    tag = f"{name} B={B} T={T}"
    _within(f"{tag} F", F.cpu(), Fw, F32w, dtype, 1e-11)
    _within(f"{tag} f", f.cpu(), fw, f32w, dtype, 1e-11)
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
    pt = CtrlPassthroughDynamics(_module(name))
    clamp = PHYS[name]["clamp"]
    x0, u = _aug_states(name, B, T, F64, seed)
    x0[:, 0] *= 0.2
    u = u * 0.2
    if calm:
        th = torch.pi + 0.4 * (torch.rand(B, generator=g, dtype=F64) - 0.5)
        ic, is_ = (3, 4) if name == "cartpole" else (1, 2)
        x0[:, ic], x0[:, is_] = torch.cos(th), torch.sin(th)
        u = u * 0.5
    xs = [x0]
    for t in range(T - 1):
        xs.append(pt(xs[t], u[t]))
    x = torch.stack(xs)
    n = x.shape[2]
    p = n + 1
    nx, R, S = _jac(pt, x[:-1].reshape(-1, n), u[:-1].reshape(-1, 1))
    F = torch.cat((R, S), 2).view(T - 1, B, n, p)
    f = (nx - torch.einsum("bij,bj->bi", R, x[:-1].reshape(-1, n))
         - torch.einsum("bij,bj->bi", S, u[:-1].reshape(-1, 1))).view(T - 1, B, n)
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
    pt = CtrlPassthroughDynamics(_module(name))
    n = pt.n_state
    d = lambda t: t.to(DEV) if torch.is_tensor(t) else t
    r = step.lqr_step_raw(n, 1, T, *[d(P[k]) for k in ("x0", "C", "c", "F", "f", "x", "u")],
                          dyn=(pt.mpcb200_kind, pt.mpcb200_params()), **{k: d(v) for k, v in kw.items()})
    plan = _lib.last_step_plan()

    def no_split(*a, **k):
        raise AssertionError("split-mode rollout ran")
    monkeypatch.setattr(step, "rollout_split", no_split)
    C, c, F, f = (d(P[k]) for k in ("C", "c", "F", "f"))
    nx, nu, _, costs, _, _ = step.LQRStep(n, 1, T, true_cost=QuadCost(C, c), true_dynamics=pt,
                                          current_x=d(P["x"]), current_u=d(P["u"]), **kw)(d(P["x0"]), C, c, F, f)
    assert torch.equal(nx, r["new_x"]) and torch.equal(nu, r["new_u"]) and torch.equal(costs, r["costs"])
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in r.items() if v is not None}, plan


def _check_step(tag, r, o, bounded):
    assert torch.equal(r["alphas"], o.alphas), f"{tag}: alphas {r['alphas']} vs {o.alphas}"
    sc = max(1.0, float(o.new_x.abs().max()), float(o.new_u.abs().max()))
    for k in ("new_x", "new_u"):
        err = maxdiff(r[k], getattr(o, k))
        assert err <= 1e-9 * sc, f"{tag}: {k} {err:.3e}"
    assert maxdiff(r["costs"], o.costs) <= 1e-9 * max(1.0, float(o.costs.abs().max())), tag
    assert torch.equal(r["free_mask"].bool(), o.free_masks), f"{tag}: free sets"
    if bounded:
        assert torch.equal(r["qp_iters"].long(), o.qp_iters), f"{tag}: pnqp iterations"


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
    _check_step(tag, r, o, bounds is not None)


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
    pt = CtrlPassthroughDynamics(_module(name))
    Ts = _gain_switch(pt.mpcb200_kind, pt.n_state, 8)
    assert Ts is not None and 2 < Ts <= 1024, Ts
    for T in (Ts - 1, Ts):
        P, kw, o = _step_case(name, 6, T, "scalar", 800 + T, calm=True)
        r, plan = _kernel_step(name, T, P, kw, monkeypatch)
        tag = f"{name} T={T} (switch {Ts})"
        assert plan & _lib.PLAN_GENERIC, tag
        assert bool(plan & _lib.PLAN_GAINS_SMEM) == (T < Ts), f"{tag}: plan {plan}"
        _check_step(tag, r, o, True)


# ------------------------------------------------------------------------------------------------------------------
# MPC.forward with a slew-rate penalty: device loop vs host loop
# ------------------------------------------------------------------------------------------------------------------
def _run(monkeypatch, make, x0, cost, dx, device_loop, grads=()):
    """(x, u, costs, full_du_norm, gradients of (x.sum() + u.sum()) w.r.t. `grads`) on the chosen loop."""
    seen = {}
    with monkeypatch.context() as mp:
        if device_loop:
            assert solver._use_slew_device_loop(make(), x0, cost, dx, _u0(make(), x0))
            real = step.ilqr_raw

            def spy(*a, **k):
                seen["res"] = real(*a, **k)
                return seen["res"]
            mp.setattr(step, "ilqr_raw", spy)
        else:
            mp.setattr(solver, "_use_slew_device_loop", lambda *a: False)
        real_host = MPC._ilqr_host

        def host(self, *a, **k):
            seen["best"] = real_host(self, *a, **k)
            return seen["best"]
        mp.setattr(MPC, "_ilqr_host", host)
        x, u, costs = make()(x0, cost, dx)
    assert ("res" in seen) == device_loop and ("best" in seen) != device_loop
    fdn = seen["res"]["full_du_norm"] if device_loop else seen["best"]["full_du_norm"]
    gs = torch.autograd.grad(x.sum() + u.sum(), grads) if grads else ()
    torch.cuda.synchronize()
    return x, u, costs, fdn, gs


def _u0(ctrl, x0):
    return torch.zeros(ctrl.T, x0.shape[0], ctrl.n_ctrl, dtype=x0.dtype, device=x0.device)


def _bitwise(tag, a, b):
    """x, u, costs and the gradients bit for bit; full_du_norm, which the device loop sums in another order (DESIGN
    section 3.5), to 1e-12 (float64) / 1e-5 (float32) relative."""
    for k, (p, q) in enumerate(zip(a[:3], b[:3])):
        assert p.shape == q.shape and torch.equal(p, q), f"{tag}: output {k} {float((p - q).abs().max()):.3e}"
    rtol = 1e-12 if a[3].dtype == F64 else 1e-5
    assert torch.allclose(a[3], b[3], rtol=rtol, atol=0), f"{tag}: full_du_norm {float((a[3] - b[3]).abs().max())}"
    for k, (p, q) in enumerate(zip(a[4], b[4])):
        assert torch.equal(p, q), f"{tag}: gradient {k} {float((p - q).abs().max()):.3e}"


def _known_problem(name, B, T):
    dx = _module(name, params=torch.tensor(PHYS[name]["params"], dtype=F64, device=DEV).requires_grad_(True),
                 device=DEV)
    n = dx.n_state
    q, p = dx.get_true_obj()
    Q = torch.diag(q).double().expand(T, B, n + 1, n + 1).contiguous().to(DEV).requires_grad_(True)
    pp = p.double().expand(T, B, n + 1).contiguous().to(DEV).requires_grad_(True)
    return dx, Q, pp, _states(name, B, 40 + B).to(DEV)


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
    dev = _run(monkeypatch, make, x0, cost, dx, True, grads=(Q, pp, dx.params))
    host = _run(monkeypatch, make, x0, cost, dx, False, grads=(Q, pp, dx.params))
    tag = f"{name} {bounds} delta {delta} prev {prev}"
    _bitwise(tag, dev, host)
    assert float(dev[4][2].abs().max()) > 0, f"{tag}: no gradient reaches the system parameters"

    class Opaque(torch.nn.Module):                      # hides mpcb200_kind: today's Module path (split mode)
        def forward(self, xx, uu):
            return dx(xx, uu)
    x, u, costs = make()(x0, QuadCost(Q.detach(), pp.detach()), Opaque())
    for k, (p, q) in enumerate(((x, dev[0]), (u, dev[1]))):
        assert maxdiff(p, q) < 1e-7 * max(1.0, float(p.abs().max())), f"{tag}: opaque module {k}"
    assert maxdiff(costs, dev[2]) < 1e-8 * max(1.0, float(costs.abs().max())), f"{tag}: opaque costs"


@pytest.mark.parametrize("name", SYSTEMS)
def test_known_system_slew_follows_parameter_edits(name, monkeypatch):
    B, T = 9, 12
    dx, Q, pp, x0 = _known_problem(name, B, T)
    kw = dict(u_lower=-2.0 * PHYS[name]["clamp"], u_upper=2.0 * PHYS[name]["clamp"], lqr_iter=4, verbose=-1,
              exit_unconverged=False, detach_unconverged=False, slew_rate_penalty=0.2,
              grad_method=GradMethods.AUTO_DIFF)
    make = lambda: MPC(dx.n_state, 1, T, **kw)
    cost = QuadCost(Q.detach(), pp.detach())
    first = _run(monkeypatch, make, x0, cost, dx, True)
    with torch.no_grad():
        dx.params.mul_(1.2)
    dev = _run(monkeypatch, make, x0, cost, dx, True)
    host = _run(monkeypatch, make, x0, cost, dx, False)
    _bitwise(f"{name} after an edit", dev, host)
    assert not torch.equal(first[0], dev[0])


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
    dev = _run(monkeypatch, make, x0, QuadCost(Cl, cl), LinDx(F, f), True, grads=(Cl, cl))
    host = _run(monkeypatch, make, x0, QuadCost(Cl, cl), LinDx(F, f), False, grads=(Cl, cl))
    _bitwise(f"({n},{m}) {dtype} {case}", dev, host)


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
    x, u, costs, _, _ = _run(monkeypatch, make, g["x_init"].to(DEV), QuadCost(g["C"].to(DEV), g["c"].to(DEV)),
                             LinDx(F), True)
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
    assert solver._use_slew_device_loop(ctrl, x0, QuadCost(C, c), dx, _u0(ctrl, x0))
    ran = []
    real = step.ilqr_raw
    monkeypatch.setattr(step, "ilqr_raw", lambda *a, **k: ran.append(1) or real(*a, **k))
    x, u, costs = ctrl(x0, QuadCost(C, c), dx)
    assert ran == [1]
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
