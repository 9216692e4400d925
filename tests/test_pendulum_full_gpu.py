"""GPU: the five-parameter pendulum, PendulumDx(simple=False) (kind DYN_PENDULUM_FULL), in the kernels.

  1. rollout and exact Jacobians against the torch module (float64 CPU) and the reference's AUTO_DIFF F, f;
  2. the parameter VJP (all five parameters) against autograd, central differences and the reference's params.grad;
  3. the fused LQR step on its dynamics-only instance against the float64 oracle and the opaque-Module route, with
     repeated line-search passes, a saturating clamp, and both sides of the gain-store switch;
  4. MPC.forward: device loop bitwise equal to the host loop, and against the reference's solves (bounded, unbounded,
     slew-rate penalty) and its receding-horizon episode;
  5. params.grad end to end against the opaque Module with create_graph;
  6. system identification of damping and gravity bias.

Physics: oracle/make_golden_pendulum_full.py's (g, m, l, d, b) = (9.1, 1.7, 0.6, 0.4, 0.25), dt 0.15, clamp 1.5.
Tolerances follow tests/test_known_systems_gpu.py: float64 next states 1e-12, Jacobians 1e-11, the fused step 1e-9 with
alphas, free sets and pnqp iteration counts bit exact; float32 by the K32 rule of tests/gpu_harness.within."""
import functools
import os

import numpy as np
import pytest
import torch

from oracle import lqr_oracle as orc
from tests.gpu_harness import (DEV, DT, F32, F64, check_alphas, check_clamps, check_pnqp, check_trajectory, decays,
                               f32_compared, linearise, round_through, rollout, run_step, same_on_both_loops, within)
from tests.helpers import load_golden, maxdiff

pytestmark = pytest.mark.gpu

PARAMS, DT_, CLAMP = (9.1, 1.7, 0.6, 0.4, 0.25), 0.15, 1.5
RADII = (0.3, 1.0, 3.0)


def module(params=None, device="cpu"):
    from mpc.pytorch_b200.dynamics import PendulumDx
    p = torch.tensor(PARAMS, dtype=F64) if params is None else params
    dx = PendulumDx(params=p.to(device), simple=False)
    dx.dt, dx.max_torque = DT_, CLAMP
    return dx


def opaque(dx):
    class Opaque(torch.nn.Module):                      # hides mpcb200_kind: the torch Module route
        def forward(self, x, u):
            return dx(x, u)
    return Opaque()


def states(B, seed):
    """float64 [B, 3]: angle pair at radii 0.3 / 1 / 3, the first rows at theta = +-pi (both signs of sin = 0) and
    near 0."""
    g = torch.Generator().manual_seed(seed)
    th = (torch.rand(B, generator=g, dtype=F64) * 2 - 1) * 3.0
    r = torch.tensor(RADII, dtype=F64).repeat(B)[:B]
    x = torch.stack((r * th.cos(), r * th.sin(), (torch.rand(B, generator=g, dtype=F64) - 0.5) * 2.0), 1)
    edge = ((-1.0, 0.0), (-1.0, -0.0), (-0.3, 0.0), (-3.0, -0.0), (1.0, 1e-9), (1.0, -1e-9), (3.0, 0.0))
    for k, (cv, sv) in enumerate(edge[:B]):
        x[k, 0], x[k, 1] = cv, sv
    return x


def controls(T, B, dtype, seed):
    """float64 [T, B, 1] in +-1.5 clamp; the last rows of every time step at, one ulp (of dtype) inside and one
    outside the clamp."""
    g = torch.Generator().manual_seed(seed)
    u = (torch.rand(T, B, 1, generator=g, dtype=F64) * 2 - 1) * 1.5 * CLAMP
    npd = np.float64 if dtype == F64 else np.float32
    inn, out = float(np.nextafter(npd(CLAMP), npd(0))), float(np.nextafter(npd(CLAMP), npd(np.inf)))
    e = torch.tensor((CLAMP, -CLAMP, inn, -inn, out, -out), dtype=F64)
    k = min(B, len(e))
    u[:, -k:, 0] = e[:k]
    return u


# ------------------------------------------------------------------------------------------------------------------
# 1. rollout and exact Jacobians
# ------------------------------------------------------------------------------------------------------------------
BT = [(1, 1), (127, 11), (128, 2), (129, 11), (300, 40), (4097, 3)]


@pytest.mark.parametrize("B,T", BT, ids=[f"B{b}_T{t}" for b, t in BT])
@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
def test_rollout_matches_module(dtype, B, T):
    from mpc.pytorch_b200.dynamics import dyn_rollout_raw
    dx = module()
    x0, u = states(B, 10 + B + T).to(dtype), controls(T, B, dtype, 20 + B + T).to(dtype)
    x = dyn_rollout_raw(dx.mpcb200_kind, dx.mpcb200_params(), T, x0.to(DEV), u.to(DEV)).cpu()
    assert x.shape == (T, B, 3) and x.dtype == dtype and torch.equal(x[0], x0)
    if T == 1:
        return
    xs, us = x[:-1].reshape(-1, 3).double(), u[:-1].reshape(-1, 1).double()
    w64 = dx(xs, us).view(T - 1, B, -1)
    w32 = module(torch.tensor(PARAMS, dtype=F32))(xs.float(), us.float()).view(T - 1, B, -1) if dtype == F32 else None
    within(f"{DT[dtype]} B={B} T={T}", "rollout", x[1:], w64, w32, dtype, 1e-12)


@pytest.mark.parametrize("B,T", BT, ids=[f"B{b}_T{t}" for b, t in BT])
@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
def test_jacobians_match_autograd(dtype, B, T):
    """Unclamped, clamped and exactly-at-the-bound controls: S is exactly 0 beyond the clamp, non-zero at it."""
    from mpc.pytorch_b200.dynamics import dyn_linearize_raw
    dx = module()
    x = torch.stack([states(B, 30 + t) for t in range(T)]).to(dtype)
    u = controls(T, B, dtype, 40 + B + T).to(dtype)
    F, f = dyn_linearize_raw(dx.mpcb200_kind, dx.mpcb200_params(), T, x.to(DEV), u.to(DEV))
    F, f = F.cpu(), f.cpu()
    assert F.shape == (T - 1, B, 3, 4) and f.shape == (T - 1, B, 3)
    if T == 1:
        return
    F64w, f64w = linearise(dx, x.double(), u.double())
    F32w, f32w = linearise(module(torch.tensor(PARAMS, dtype=F32)), x.float(), u.float()) if dtype == F32 else \
        (None, None)
    tag = f"{DT[dtype]} B={B} T={T}"
    within(tag, "F", F, F64w, F32w, dtype, 1e-11)
    within(tag, "f", f, f64w, f32w, dtype, 1e-11)
    out = u[:-1, :, 0].double().abs() > CLAMP
    assert bool((F[..., 3][out] == 0).all()) and bool((F[..., 3][~out].abs().sum(-1) > 0).all()), tag


def test_linearisation_matches_reference_fixture():
    """The reference's own AUTO_DIFF linearize_dynamics along its rollout (float64)."""
    from mpc.pytorch_b200.dynamics import dyn_linearize_raw, dyn_rollout_raw
    g = load_golden("known_step_pendulum_full_f64")
    dx = module(g["params"])
    dx.dt, dx.max_torque = float(g["dt"]), float(g["clamp"])
    T = g["roll_u"].shape[0]
    x = dyn_rollout_raw(dx.mpcb200_kind, dx.mpcb200_params(), T, g["roll_x_init"].to(DEV), g["roll_u"].to(DEV))
    assert maxdiff(x, g["roll_x"]) <= 1e-12
    F, f = dyn_linearize_raw(dx.mpcb200_kind, dx.mpcb200_params(), T, g["roll_x"].to(DEV), g["roll_u"].to(DEV))
    assert maxdiff(F, g["roll_F"]) <= 1e-11 * max(1.0, float(g["roll_F"].abs().max()))
    assert maxdiff(f, g["roll_f"]) <= 1e-11 * max(1.0, float(g["roll_f"].abs().max()))


# ------------------------------------------------------------------------------------------------------------------
# 2. the parameter VJP
# ------------------------------------------------------------------------------------------------------------------
def _vjp_case(B, T, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.stack([states(B, seed + t) for t in range(T)]).to(dtype).double()
    u = controls(T, B, dtype, seed + 100).to(dtype).double()
    dF = torch.randn(T - 1, B, 3, 4, generator=g, dtype=F64).to(dtype).double()
    df = torch.randn(T - 1, B, 3, generator=g, dtype=F64).to(dtype).double()
    return x, u, dF, df


def _autograd_vjp(x, u, dF, df, dtype=F64):
    """(first, second) [T-1, B, 5] by autograd of the module in dtype, one parameter column per (t, b)."""
    T, B, n = x.shape
    N = (T - 1) * B
    P = torch.tensor(PARAMS, dtype=dtype).view(-1, 1).expand(-1, N).clone().requires_grad_(True)
    dx = module(P)
    x, u, dF, df = (t.to(dtype) for t in (x, u, dF, df))
    xs = x[:-1].reshape(N, n).clone().requires_grad_(True)
    us = u[:-1].reshape(N, 1).clone().requires_grad_(True)
    nx = dx(xs, us)
    rows = [torch.autograd.grad(nx[:, r].sum(), [xs, us], create_graph=True) for r in range(n)]
    J = torch.cat((torch.stack([a for a, _ in rows], 1), torch.stack([b for _, b in rows], 1)), 2)
    z = torch.cat((xs, us), 1).detach()
    dF_, df_ = dF.reshape(N, n, n + 1), df.reshape(N, n)
    first, = torch.autograd.grad((df_ * nx).sum(), P, retain_graph=True)
    second, = torch.autograd.grad(((dF_ - df_.unsqueeze(2) * z.unsqueeze(1)) * J).sum(), P)
    return first.t().reshape(T - 1, B, 5).double(), second.t().reshape(T - 1, B, 5).double()


def _kernel_vjp(dx, x, u, dF, df, dtype=F64):
    from mpc.pytorch_b200.dynamics import dyn_linearize_vjp_raw
    first, second = dyn_linearize_vjp_raw(dx.mpcb200_kind, dx.mpcb200_params(), x.shape[0],
                                          *(t.to(dtype).to(DEV) for t in (x, u, dF, df)))
    assert first.shape == (x.shape[0] - 1, x.shape[1], 5) and first.dtype == dtype
    return first.cpu(), second.cpu()


@pytest.mark.parametrize("B,T", [(7, 2), (300, 9)], ids=["B7_T2", "B300_T9"])
def test_vjp_matches_autograd_and_finite_differences(B, T):
    from mpc.pytorch_b200.dynamics import dyn_linearize_raw
    x, u, dF, df = _vjp_case(B, T, F64, 11 * B + T)
    dx = module()
    first, second = _kernel_vjp(dx, x, u, dF, df)
    w1, w2 = _autograd_vjp(x, u, dF, df)
    within(f"B={B} T={T}", "first", first, w1, None, F64, 1e-10)
    within(f"B={B} T={T}", "second", second, w2, None, F64, 1e-10)
    got = (first + second).sum((0, 1))
    prm = list(dx.mpcb200_params())
    xd, ud, dFd, dfd = (t.to(DEV) for t in (x, u, dF, df))

    def objective(p):
        F, f = dyn_linearize_raw(dx.mpcb200_kind, p, T, xd, ud)
        return float((dFd * F).sum() + (dfd * f).sum())
    fd = []
    for k in range(5):
        h = 1e-5 * abs(prm[k])
        hi, lo = list(prm), list(prm)
        hi[k] += h
        lo[k] -= h
        fd.append((objective(hi) - objective(lo)) / (2 * h))
    fd = torch.tensor(fd, dtype=F64)
    assert maxdiff(got, fd) <= 1e-6 * max(1.0, float(fd.abs().max())), f"{got.tolist()} vs {fd.tolist()}"
    assert bool((got.abs() > 0).all())


def test_vjp_f32_matches_autograd():
    x, u, dF, df = _vjp_case(129, 6, F32, 5)
    first, second = _kernel_vjp(module(), x, u, dF, df, F32)
    w1, w2 = _autograd_vjp(x, u, dF, df)
    f1, f2 = _autograd_vjp(x, u, dF, df, F32)
    within("f32", "first", first, w1, f1, F32)
    within("f32", "second", second, w2, f2, F32)


@pytest.mark.parametrize("regime", ["unb", "box"])
def test_first_is_the_reference_gradient(regime):
    g = load_golden("paramgrad_pendulum_full_f64")
    dx = module(g["params"])
    dx.dt, dx.max_torque = float(g["dt"]), float(g["clamp"])
    x, u, df = g[f"x_lin_{regime}"], g[f"u_{regime}"], g[f"df_{regime}"]
    dF = torch.zeros(*df.shape, df.shape[-1] + 1, dtype=F64)
    first, _ = _kernel_vjp(dx, x, u, dF, df)
    want = g[f"grad_{regime}"]
    assert maxdiff(first.sum((0, 1)), want) <= 1e-10 * max(1.0, float(want.abs().max())), regime


# ------------------------------------------------------------------------------------------------------------------
# 3. the fused step on the dynamics-only instance
# ------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=8)
def step_case(B, T, dtype, bounds, ls_iter, decay, seed, calm=False):
    """Inputs (float64 rounded through dtype), the float64 oracle with its line-search trace, the float32 oracle;
    as tests/test_known_systems_gpu.step_case builds them for the simple pendulum."""
    dx = module()
    g = torch.Generator().manual_seed(seed)
    x0 = states(B, seed)
    if calm:
        th = torch.pi + 0.4 * (torch.rand(B, generator=g, dtype=F64) - 0.5)
        x0[:, 0], x0[:, 1] = th.cos(), th.sin()
    x0 = round_through(x0, dtype)
    u = round_through((torch.rand(T, B, 1, generator=g, dtype=F64) * 2 - 1) * (0.1 if calm else 0.8) * CLAMP, dtype)
    x = round_through(rollout(dx, x0, u), dtype)
    F, f = linearise(dx, x, u)
    L = torch.randn(T, B, 4, 4, generator=g, dtype=F64) / 2.0
    C = L @ L.transpose(-1, -2) + 0.5 * torch.eye(4, dtype=F64)
    c = torch.randn(T, B, 4, generator=g, dtype=F64)
    if calm:
        c[..., 3:] *= 0.2 * CLAMP
    else:
        c[..., :3] *= 20.0
        c[..., 3:] = 0.0
    F, f, C, c = (round_through(v, dtype) for v in (F, f, C, c))
    kw = dict(linesearch_decay=decay, max_linesearch_iter=ls_iter)
    if bounds == "scalar":
        kw.update(u_lower=-0.8 * CLAMP, u_upper=0.8 * CLAMP)
    elif bounds == "wide":
        kw.update(u_lower=-2.0 * CLAMP, u_upper=2.0 * CLAMP)
    P = dict(x0=x0, C=C, c=c, F=F, f=f, x=x, u=u)
    trace = []
    o64 = orc.lqr_step_forward(3, 1, T, x0, C, c, F, f, x, u, coupled=False, dynamics=dx, ls_trace=trace, **kw)
    o32 = None
    if dtype == F32:
        lo32 = lambda v: v.float() if torch.is_tensor(v) and v.is_floating_point() else v  # noqa: E731
        o32 = orc.lqr_step_forward(3, 1, T, *[lo32(P[k]) for k in ("x0", "C", "c", "F", "f", "x", "u")],
                                   coupled=False, dynamics=module(torch.tensor(PARAMS, dtype=F32)), **kw)
    return P, kw, o64, torch.stack(trace), o32


def _run_step(T, case, dtype):
    dx = module()
    return run_step(3, 1, T, case[0], case[1], dtype, dyn=(dx.mpcb200_kind, dx.mpcb200_params()))


def check_step(tag, r, case, dtype):
    P, kw, o64, trace, o32 = case
    keep = torch.ones(P["x0"].shape[0], dtype=torch.bool)
    if dtype == F32:
        keep = f32_compared(case)
        assert int((~keep).sum()) <= max(1, len(keep) // 8), f"{tag}: too many problems left out"
        d = kw["linesearch_decay"]
        assert torch.equal(decays(r["alphas"], d)[keep], decays(o64.alphas, d)[keep]), f"{tag}: line search"
        assert int((r["status"] & ~1).max()) == 0, tag
    else:
        check_alphas(tag, r, o64, None)
        check_pnqp(tag, r, o64, kw)
        check_clamps(tag, r, o64, kw)
    check_trajectory(tag, r, P["u"], o64, o32, dtype, keep)


STEP_OPTS = [(None, 10, 0.2), ("scalar", 1, 0.2), ("wide", 2, 0.35), ("scalar", 6, 0.35)]


@pytest.mark.parametrize("bounds,ls_iter,decay", STEP_OPTS, ids=[f"{b}_ls{i}_d{d}" for b, i, d in STEP_OPTS])
@pytest.mark.parametrize("dtype,B", [(F64, 20), (F64, 21), (F32, 21)], ids=["f64_B20", "f64_B21", "f32_B21"])
def test_fused_step_matches_oracle(dtype, B, bounds, ls_iter, decay):
    """The step kernel's line search runs the five-parameter pendulum: it matches the oracle with dynamics=<module>
    and differs from the same step with the simple pendulum's physics."""
    from mpc.pytorch_b200 import _lib
    T = 15
    case = step_case(B, T, dtype, bounds, ls_iter, decay, 500 + B)
    r, plan = _run_step(T, case, dtype)
    tag = f"{DT[dtype]} B={B} {bounds} ls={ls_iter} decay={decay}"
    assert plan & _lib.PLAN_GENERIC, f"{tag}: plan {plan}"
    check_step(tag, r, case, dtype)


def test_fused_step_cases_exercise_the_line_search_and_the_clamp():
    for bounds, ls_iter, decay in STEP_OPTS:
        decayed = worse_first = beyond = 0
        for dtype, B in ((F64, 20), (F64, 21)):
            _, _, o64, trace, _ = step_case(B, 15, dtype, bounds, ls_iter, decay, 500 + B)
            decayed += int((o64.alphas < 1).sum())
            worse_first += int((trace[0] > 0).sum())
            beyond += int((o64.new_u.abs() > CLAMP).sum())
        assert (decayed if ls_iter > 1 else worse_first) > 0, f"{bounds}: the line search never engages"
        if bounds == "wide":
            assert beyond > 0, "no control beyond the clamp"


def test_fused_step_equals_opaque_module_route():
    """LQRStep with the known system (in-kernel line search) against the same physics as an opaque Module (the
    split-mode route: the rollout in torch between kernel calls)."""
    from mpc.pytorch_b200 import LQRStep, LinDx, QuadCost
    B, T = 21, 15
    P, kw, o64, _, _ = step_case(B, T, F64, "scalar", 6, 0.35, 521)
    dx = module(device=DEV)
    d = {k: v.to(DEV) for k, v in P.items()}
    out = []
    for true_dx in (dx, opaque(dx)):
        step = LQRStep(3, 1, T, u_lower=kw["u_lower"], u_upper=kw["u_upper"], linesearch_decay=kw["linesearch_decay"],
                       max_linesearch_iter=kw["max_linesearch_iter"], true_cost=QuadCost(d["C"], d["c"]),
                       true_dynamics=true_dx, current_x=d["x"], current_u=d["u"])
        out.append([t.detach().cpu() for t in step(d["x0"], d["C"], d["c"], d["F"], d["f"])[:2]])
    for a, b, w in zip(out[0], out[1], (o64.new_x, o64.new_u)):
        sc = max(1.0, float(w.abs().max()))
        assert maxdiff(a, b) <= 1e-9 * sc and maxdiff(a, w) <= 1e-9 * sc


def _gain_switch(esz):
    """First horizon at which the step of the kind keeps its gains in Ks/ks (the library's own answer)."""
    import ctypes
    from mpc.pytorch_b200 import _lib
    from mpc.pytorch_b200.dynamics import DYN_PENDULUM_FULL
    for T in range(2, 4096):
        d = _lib.Dims(B=1, T=T, n=3, m=1, F_T=T - 1, dynamics_kind=DYN_PENDULUM_FULL, max_ls_iter=1,
                      pnqp_max_iter=1, do_rollout=1)
        if _lib.lib().mpcb200_step_prefers_workspace(ctypes.byref(d), esz):
            return T
    return None


def test_fused_step_on_both_sides_of_the_gain_store_switch():
    from mpc.pytorch_b200 import _lib
    B = 13
    Ts = _gain_switch(8)
    assert Ts is not None and 2 < Ts <= 1024, Ts
    for T in (Ts - 1, Ts):
        case = step_case(B, T, F64, "scalar", 4, 0.3, 700 + T, calm=True)
        r, plan = _run_step(T, case, F64)
        tag = f"f64 B={B} T={T} (switch {Ts})"
        assert plan & _lib.PLAN_GENERIC, tag
        assert bool(plan & _lib.PLAN_GAINS_SMEM) == (T < Ts), f"{tag}: plan {plan}"
        check_step(tag, r, case, F64)


def test_column_pair_kernel_is_refused():
    """MPCB200_KERNEL=2 forces the column-pair kernel, which has no in-kernel dynamics: UNSUPPORTED_DIMS."""
    from mpc.pytorch_b200._lib import MpcB200Error
    case = step_case(20, 15, F64, "scalar", 1, 0.2, 520)
    dx = module()
    with pytest.raises(MpcB200Error, match=r"\[3\]"):
        run_step(3, 1, 15, case[0], case[1], F64, impl=2, dyn=(dx.mpcb200_kind, dx.mpcb200_params()))


# ------------------------------------------------------------------------------------------------------------------
# 4. MPC.forward
# ------------------------------------------------------------------------------------------------------------------
def _mpc(T, lqr_iter=15, **kw):
    from mpc.pytorch_b200 import MPC, GradMethods
    opts = dict(lqr_iter=lqr_iter, verbose=-1, exit_unconverged=False, detach_unconverged=False,
                linesearch_decay=0.35, max_linesearch_iter=6, grad_method=GradMethods.AUTO_DIFF, eps=1e-9)
    opts.update(kw)
    return lambda: MPC(3, 1, T, **opts)


def _cost(B, T, dtype):
    from mpc.pytorch_b200 import QuadCost
    q, p = module().get_true_obj()
    Q = torch.diag(q).to(dtype).expand(T, B, 4, 4).contiguous().to(DEV)
    c = p.to(dtype).expand(T, B, 4).contiguous().to(DEV).requires_grad_(True)
    return QuadCost(Q, c), c


@pytest.mark.parametrize("slew", [False, True], ids=["plain", "slew"])
@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
def test_device_loop_equals_host_loop(monkeypatch, dtype, slew):
    """x, u, costs and the gradients in c, x_init and params, bit for bit."""
    B, T = 9, 12
    params = torch.tensor(PARAMS, dtype=dtype, device=DEV).requires_grad_(True)
    dx = module(params)
    dx.params = params
    cost, c = _cost(B, T, dtype)
    x0 = states(B, 3).to(dtype).to(DEV).requires_grad_(True)
    kw = dict(u_lower=-2.0 * CLAMP, u_upper=2.0 * CLAMP)
    if slew:
        kw.update(slew_rate_penalty=0.5, prev_ctrl=torch.linspace(-2, 2, B, dtype=dtype, device=DEV).view(B, 1))
    same_on_both_loops(monkeypatch, _mpc(T, **kw), x0, cost, dx, grads=(c, x0, params))


def _fixture_solve(g, x0, Q, c, kw):
    from mpc.pytorch_b200 import QuadCost
    dx = module(g["params"].to(DEV))
    dx.dt, dx.max_torque = float(g["dt"]), float(g["clamp"])
    return _mpc(Q.shape[0], int(g["lqr_iter"]), linesearch_decay=float(g["decay"]),
                max_linesearch_iter=int(g["ls_iter"]), **kw)()(x0.to(DEV), QuadCost(Q.to(DEV), c.to(DEV)), dx)


@pytest.mark.parametrize("regime", ["unb", "box"])
def test_mpc_matches_reference_solves(regime):
    g = load_golden("pendulum_full_ilqr_f64")
    kw = {} if regime == "unb" else dict(u_lower=-float(g["bound_box"]), u_upper=float(g["bound_box"]))
    x, u, costs = _fixture_solve(g, g["x_init"], g["C"], g["c"], kw)
    for k, got, tol in (("x", x, 1e-7), ("u", u, 1e-6), ("costs", costs, 1e-7)):
        want = g[f"{k}_{regime}"]
        assert maxdiff(got, want) <= tol * max(1.0, float(want.abs().max())), f"{regime}: {k} {maxdiff(got, want)}"


@pytest.mark.parametrize("regime", ["in", "wide"])
def test_mpc_matches_reference_slew_solves(regime):
    """The tolerances of tests/test_slew_gpu.py's known-system fixtures: costs 1e-7 relative, x and u at pnqp's
    accuracy (2e-4 x scale; the reference couples pnqp's termination over the batch), saturated controls exactly."""
    g = load_golden("known_slew_pendulum_full_f64")
    b = float(g[f"bound_{regime}"])
    kw = dict(u_lower=-b, u_upper=b, slew_rate_penalty=float(g["penalty"]), prev_ctrl=g["prev_ctrl"].to(DEV))
    x, u, costs = _fixture_solve(g, g["x_init"], g["C"], g["c"], kw)
    wx, wu, wc = g[f"x_{regime}"], g[f"u_{regime}"], g[f"costs_{regime}"]
    rel = (costs.detach().cpu() - wc).abs() / wc.abs().clamp_min(1.0)
    assert float(rel.max()) < 1e-7, f"{regime}: costs {float(rel.max()):.3e}"
    assert maxdiff(u, wu) < 2e-4 * max(1.0, float(wu.abs().max())), f"{regime}: u {maxdiff(u, wu):.3e}"
    assert maxdiff(x, wx) < 2e-4 * max(1.0, float(wx.abs().max())), f"{regime}: x {maxdiff(x, wx):.3e}"
    assert torch.equal(u.detach().abs().cpu() == b, wu.abs() == b), f"{regime}: saturated controls"


def test_receding_horizon_graph_equals_host_and_reference(monkeypatch):
    """The episode as one CUDA graph, bitwise the host episode; against the reference's notebook loop."""
    from tests.test_receding_gpu import FIELDS, run
    from mpc.pytorch_b200 import MPC, GradMethods, QuadCost
    from mpc.pytorch_b200.dynamics import PendulumDx
    g = dict(np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden",
                                  "receding_pendulum_full_f64.npz")))
    t = {k: torch.from_numpy(v).to(DEV) for k, v in g.items() if v.dtype == np.float64}
    dx = PendulumDx(params=torch.from_numpy(g["params"]), simple=False)
    make = lambda: MPC(3, 1, int(g["T"]), u_lower=float(dx.lower), u_upper=float(dx.upper),  # noqa: E731
                       lqr_iter=int(g["lqr_iter"]), verbose=-1, eps=float(g["eps"]),
                       linesearch_decay=float(g["decay"]), max_linesearch_iter=int(g["ls_iter"]),
                       grad_method=GradMethods.AUTO_DIFF)
    cost = QuadCost(t["C"], t["c"])
    steps = int(g["n_steps"])
    host = run(monkeypatch, make, t["x_init"], cost, dx, steps, False)
    ep = run(monkeypatch, make, t["x_init"], cost, dx, steps, True)
    for k in FIELDS:
        a, b = getattr(ep, k), getattr(host, k)
        assert torch.equal(a, b.to(a.device)), k
    assert ep.info[:, 0].cpu().long().tolist() == g["iters"].tolist(), "iterations per solve"
    for k, tol in (("x", 1e-5), ("costs", 1e-5), ("u", 2e-4)):
        err = float((getattr(ep, k) - t[k]).abs().max())
        assert err <= tol * max(1.0, float(t[k].abs().max())), f"{k} {err:.3e}"
    assert torch.equal(ep.u.abs() == dx.upper, t["u"].abs() == dx.upper)


# ------------------------------------------------------------------------------------------------------------------
# 5. params.grad end to end
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bounds,where,slew", [("in", "cuda", False), ("wide", "cuda", False), ("wide", "cpu", False),
                                               ("in", "f32", False), ("in", "cuda", True)],
                         ids=["in_cuda", "wide_cuda", "wide_cpu", "in_f32", "in_cuda_slew"])
def test_param_grad_equals_module_path(bounds, where, slew):
    """All five entries of params.grad through the kernels equal the opaque Module's, differentiated with
    create_graph (the full derivative, INTEGRATION.md section 2)."""
    from mpc.pytorch_b200 import QuadCost
    B, T = 13, 15
    bound = (0.8 if bounds == "in" else 2.0) * CLAMP
    params = torch.tensor(PARAMS, dtype=F32 if where == "f32" else F64)
    params = (params.to(DEV) if where != "cpu" else params).requires_grad_(True)
    dx = module(params)
    dx.params = params
    q, p = dx.get_true_obj()
    Q = torch.diag(q).double().expand(T, B, 4, 4).contiguous().to(DEV)
    pp = p.double().expand(T, B, 4).contiguous().to(DEV)
    kw = dict(u_lower=-bound, u_upper=bound)
    if slew:
        kw.update(slew_rate_penalty=0.5, prev_ctrl=torch.linspace(-1, 1, B, dtype=F64, device=DEV).view(B, 1))
    x0 = states(B, 900 + B + T).to(DEV)
    gen = torch.Generator().manual_seed(4)
    wx, wu = torch.randn(T, B, 3, generator=gen, dtype=F64).to(DEV), torch.randn(T, B, 1, generator=gen, dtype=F64)
    res = []
    for d in (dx, opaque(dx)):
        x, u, _ = _mpc(T, 20, linesearch_decay=0.3, max_linesearch_iter=4, **kw)()(x0, QuadCost(Q, pp), d)
        gr, = torch.autograd.grad((wx * x).sum() + (wu.to(DEV) * u).sum(), params)
        res.append((u.detach(), gr))
    (ua, ga), (ub, gb) = res
    assert ga.dtype == params.dtype and ga.device == params.device and ga.shape == (5,)
    tag = f"{bounds} {where} slew={slew}"
    assert maxdiff(ua, ub) < 1e-7 * max(1.0, float(ub.abs().max())), f"{tag}: u"
    tol = (1e-7 if where != "f32" else 1e-6) * max(1.0, float(gb.abs().max()))
    assert maxdiff(ga, gb) < tol, f"{tag}: {ga.tolist()} vs {gb.tolist()}"
    assert bool((ga != 0).all()), f"{tag}: {ga.tolist()}"


# ------------------------------------------------------------------------------------------------------------------
# 6. system identification of damping and gravity bias
# ------------------------------------------------------------------------------------------------------------------
# Thresholds on final / initial imitation loss and final / initial relative error of (d, b), from one seeded run on
# an H100 80GB HBM3 (700 W power limit): loss 2.00 -> 0.912 (0.46), error 0.707 -> 0.271 (0.38).  The imitation loss
# of these solves is not smooth in (d, b) (saturated controls, 15 iLQR iterations), so it falls unevenly.
SYSID = dict(steps=40, lr=0.03, loss=0.6, err=0.5)


def test_system_identification():
    """g, m, l known; d and b start 50 % off and are learnt back by Adam from an imitation loss on the controls of
    solves with the true parameters (f64), from states on the unit circle within 1 rad of upright: the loss falls
    and the error of (d, b) shrinks."""
    from mpc.pytorch_b200 import MPC, GradMethods, QuadCost
    B, T = 16, 20
    true = torch.tensor(PARAMS, dtype=F64, device=DEV)
    dx = module(true, device=DEV)
    q, p = dx.get_true_obj()
    Q = torch.diag(q).double().expand(T, B, 4, 4).contiguous().to(DEV)
    pp = p.double().expand(T, B, 4).contiguous().to(DEV)
    g = torch.Generator().manual_seed(123)
    th = (torch.rand(B, generator=g, dtype=F64) * 2 - 1) * 1.0
    x0 = torch.stack((th.cos(), th.sin(), torch.rand(B, generator=g, dtype=F64) - 0.5), 1).to(DEV)

    def solve():
        return MPC(3, 1, T, u_lower=-CLAMP, u_upper=CLAMP, lqr_iter=15, verbose=-1, exit_unconverged=False,
                   detach_unconverged=False, grad_method=GradMethods.AUTO_DIFF, eps=1e-8)(x0, QuadCost(Q, pp), dx)
    with torch.no_grad():
        _, u_true, _ = solve()
    db = torch.tensor((PARAMS[3] * 1.5, PARAMS[4] * 0.5), dtype=F64, device=DEV).requires_grad_(True)
    opt = torch.optim.Adam([db], lr=SYSID["lr"])
    losses, errs = [], []
    for _ in range(SYSID["steps"]):
        dx.params = torch.cat((true[:3], db))
        errs.append(float(((db.detach() - true[3:]) / true[3:]).norm()))
        _, u, _ = solve()
        loss = ((u - u_true) ** 2).mean()
        losses.append(float(loss))
        opt.zero_grad()
        loss.backward()
        opt.step()
    print(f"pendulum_full: loss {losses[0]:.4e} -> {losses[-1]:.4e}, (d, b) error {errs[0]:.4f} -> {errs[-1]:.4f}")
    assert losses[-1] < SYSID["loss"] * losses[0], losses
    assert errs[-1] < SYSID["err"] * errs[0], errs
