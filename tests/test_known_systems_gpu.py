"""GPU: the known-system kernels against float64 references - the rollout and exact-Jacobian kernels against the
plain-torch modules (tests/test_known_systems_cpu.py pins those to the reference), the fused LQR step's in-kernel
line-search rollout against oracle.lqr_step_forward(dynamics=<module>), and MPC.forward against the same physics
run as an opaque nn.Module.

Every case uses non-default physics (parameters, dt and control clamp), states whose angle pair (r cos th, r sin th)
is off the unit circle (radius 0.3 or 3 for the pendulum; 0.3 or 2 for the cartpole, whose th_acc denominator
l (4/3 - mp c^2 / (mp + mc)) vanishes near |c| = 2.9 at these parameters), theta at +-pi with both signs of
sin = 0 and near 0, and controls at, one ulp inside and one ulp outside the clamp.

Tolerances.  float64: next states to 1e-12 x scale, Jacobians to 1e-11 x scale; the fused step to 1e-9 x scale with
alphas, free sets and pnqp iteration counts bit exact.  float32: the kernel's error against the float64 truth must
stay within K32 = 4 times the error of the same computation run in float32 on the CPU, plus 1e-6 x scale.

Batch layouts of the generic step kernel (StepCfg in csrc/lqr_step.cuh, bulk_ok in csrc/api.cu).  A CTA holds
W problems, PPW per warp: (5,1) has PPW = 5 and W = 10 (f64) / 20 (f32); (3,1) has PPW = 8 and W = 8.  The bulk
(TMA) load path needs B*n*size and B*m*size to be multiples of 16 bytes (B even in f64, B a multiple of 4 in f32);
the last CTA's count is then aligned too, since W is a multiple of 2 (f64) / 4 (f32).  Otherwise every tile is
copied by the producer warp's lanes."""
import functools

import pytest
import torch

from oracle import lqr_oracle as orc
from tests.gpu_harness import (BT, DEV, DT, F32, F64, PHYS, SYSTEMS, angle_cols, check_alphas, check_clamps, check_pnqp,
                               check_trajectory, decays, f32_compared, first_true, jacobians, known_controls,
                               known_module, known_states, linearise, probe_step, round_through, rollout, run_step,
                               within)
from tests.helpers import EDIT_ROUTES, maxdiff

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------------------------
# rollout and exact Jacobians
# ------------------------------------------------------------------------------------------------------------------
BT = [(1, 1), (1, 200), (127, 11), (128, 2), (129, 11), (300, 200), (4097, 11), (4097, 2)]


@pytest.mark.parametrize("B,T", BT, ids=[f"B{b}_T{t}" for b, t in BT])
@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("name", SYSTEMS)
def test_rollout_matches_module(name, dtype, B, T):
    """Every step of the kernel rollout against the module's step from the kernel's own state (float64 CPU); the
    first state is the caller's x_init, copied exactly; several CTAs of 128 threads and a partial last one."""
    from mpc.pytorch_b200.dynamics import dyn_rollout_raw
    dx = known_module(name)
    x0 = known_states(name, B, 10 + B + T).to(dtype)
    u = known_controls(name, T, B, dtype, 20 + B + T).to(dtype)
    x = dyn_rollout_raw(dx.mpcb200_kind, dx.mpcb200_params(), T, x0.to(DEV), u.to(DEV)).cpu()
    assert x.shape == (T, B, dx.n_state) and x.dtype == dtype
    assert torch.equal(x[0], x0)
    if T == 1:
        return
    xs, us = x[:-1].reshape(-1, dx.n_state).double(), u[:-1].reshape(-1, 1).double()
    w64 = dx(xs, us).view(T - 1, B, -1)
    w32 = dx(xs.float(), us.float()).view(T - 1, B, -1) if dtype == F32 else None
    within(f"{name} {DT[dtype]} B={B} T={T}", "rollout", x[1:], w64, w32, dtype, 1e-12)


@pytest.mark.parametrize("B,T", BT, ids=[f"B{b}_T{t}" for b, t in BT])
@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("name", SYSTEMS)
def test_jacobians_match_autograd(name, dtype, B, T):
    """F = [R S] and f = x' - R x - S u of the linearisation kernel against float64 autograd of the module, at
    states off the unit circle, theta edges and controls at / one ulp either side of the clamp."""
    from mpc.pytorch_b200.dynamics import dyn_linearize_raw
    dx = known_module(name)
    n = dx.n_state
    x = torch.stack([known_states(name, B, 30 + t) for t in range(T)]).to(dtype)
    u = known_controls(name, T, B, dtype, 40 + B + T).to(dtype)
    F, f = dyn_linearize_raw(dx.mpcb200_kind, dx.mpcb200_params(), T, x.to(DEV), u.to(DEV))
    F, f = F.cpu(), f.cpu()
    assert F.shape == (T - 1, B, n, n + 1) and f.shape == (T - 1, B, n)
    if T == 1:
        assert F.numel() == 0 and f.numel() == 0
        return
    F64w, f64w = linearise(dx, x.to(F64), u.to(F64))
    F32w, f32w = linearise(dx, x.to(F32), u.to(F32)) if dtype == F32 else (None, None)
    tag = f"{name} {DT[dtype]} B={B} T={T}"
    within(tag, "F", F, F64w, F32w, dtype, 1e-11)
    within(tag, "f", f, f64w, f32w, dtype, 1e-11)
    clamp = PHYS[name]["clamp"]
    out = u[:-1, :, 0].double().abs() > clamp
    assert bool((F[..., n][out] == 0).all()), f"{tag}: S must be exactly 0 beyond the clamp"
    assert bool((F[..., n][~out].abs().sum(-1) > 0).all()), f"{tag}: S vanished inside / at the clamp"


# ------------------------------------------------------------------------------------------------------------------
# the fused LQR step: line-search rollout of the known system inside the step kernel
# ------------------------------------------------------------------------------------------------------------------
# (scale of the linear state cost, scale of the control row / column of C) of the step cases: the step asks for
# large state moves, so that the first line-search pass of the nonlinear rollout is often worse than the nominal
# trajectory and alpha decays.  The cartpole's control authority dt / (mc + mp) is small: its control weight is
# lowered too, or every step stays where the linearisation is accurate.
PUSH = {"cartpole": (20.0, 0.03), "pendulum": (20.0, 1.0)}


@functools.lru_cache(maxsize=8)
def step_case(name, B, T, dtype, bounds, ls_iter, decay, seed, calm=False):
    """Inputs (float64, rounded through dtype), the float64 oracle and its line-search trace, the float32 oracle.
    The nominal controls are random; x is their nonlinear rollout and F, f its float64 linearisation.
    calm: hanging start (theta near pi), small nominal controls and linear cost - for long horizons, where the
    upright-pendulum rollout of random controls amplifies round-off past any fixed tolerance."""
    dx = known_module(name)
    n, p, clamp = dx.n_state, dx.n_state + 1, PHYS[name]["clamp"]
    g = torch.Generator().manual_seed(seed)
    x0 = known_states(name, B, seed)
    if calm:
        th = torch.pi + 0.4 * (torch.rand(B, generator=g, dtype=F64) - 0.5)
        ic, is_ = angle_cols(name)
        x0[:, ic], x0[:, is_] = torch.cos(th), torch.sin(th)
    x0 = round_through(x0, dtype)
    u = round_through((torch.rand(T, B, 1, generator=g, dtype=F64) * 2 - 1) * (0.1 if calm else 0.8) * clamp, dtype)
    x = round_through(rollout(dx, x0, u), dtype)
    F, f = linearise(dx, x, u)
    L = torch.randn(T, B, p, p, generator=g, dtype=F64) / p ** 0.5
    C = L @ L.transpose(-1, -2) + 0.5 * torch.eye(p, dtype=F64)
    c = torch.randn(T, B, p, generator=g, dtype=F64)
    if calm:
        c[..., n:] *= 0.2 * clamp
    else:
        x_lin, u_weight = PUSH[name]
        c[..., :n] *= x_lin
        c[..., n:] = 0.0
        C[..., n:, :] *= u_weight
        C[..., :, n:] *= u_weight
    F, f, C, c = (round_through(v, dtype) for v in (F, f, C, c))
    kw = dict(linesearch_decay=decay, max_linesearch_iter=ls_iter)
    if bounds == "scalar":
        kw.update(u_lower=-0.8 * clamp, u_upper=0.8 * clamp)
    elif bounds == "wide":                        # wider than the clamp inside the dynamics
        kw.update(u_lower=-2.0 * clamp, u_upper=2.0 * clamp)
    elif bounds in ("tensor", "delta"):
        lo = -clamp * (0.3 + 1.7 * torch.rand(T, B, 1, generator=g, dtype=F64))
        hi = clamp * (0.3 + 1.7 * torch.rand(T, B, 1, generator=g, dtype=F64))
        kw.update(u_lower=round_through(lo, dtype), u_upper=round_through(hi, dtype))
        u = torch.maximum(torch.minimum(u, kw["u_upper"]), kw["u_lower"])
        if bounds == "delta":
            kw["delta_u"] = 0.4 * clamp
    P = dict(x0=x0, C=C, c=c, F=F, f=f, x=x, u=u)
    trace = []
    o64 = orc.lqr_step_forward(n, 1, T, x0, C, c, F, f, x, u, coupled=False, dynamics=dx, ls_trace=trace, **kw)
    o32 = None
    if dtype == F32:
        lo32 = lambda v: v.float() if torch.is_tensor(v) and v.is_floating_point() else v  # noqa: E731
        dx32 = known_module(name, params=torch.tensor(PHYS[name]["params"], dtype=F32))
        o32 = orc.lqr_step_forward(n, 1, T, *[lo32(P[k]) for k in ("x0", "C", "c", "F", "f", "x", "u")],
                                   coupled=False, dynamics=dx32, **{k: lo32(v) for k, v in kw.items()})
    return P, kw, o64, torch.stack(trace), o32


def _run_step(name, T, case, dtype):
    dx = known_module(name)
    return run_step(dx.n_state, 1, T, case[0], case[1], dtype, dyn=(dx.mpcb200_kind, dx.mpcb200_params()))


def check_step(tag, r, case, dtype):
    """float64: 1e-9 x scale, alphas / free sets / pnqp iterations bit exact.  float32: the same line-search
    decisions (number of decays) as the float64 oracle and alphas to 1e-6, except at near-ties; those problems
    leave the trajectory comparison."""
    P, kw, o64, trace, o32 = case
    keep = torch.ones(P["x0"].shape[0], dtype=torch.bool)
    if dtype == F32:
        keep = f32_compared(case)
        out = int((~keep).sum())
        assert out <= max(1, len(keep) // 8), f"{tag}: {out} of {len(keep)} problems left out"
        decay = kw["linesearch_decay"]
        assert torch.equal(decays(r["alphas"], decay)[keep], decays(o64.alphas, decay)[keep]), \
            f"{tag}: line-search decisions {r['alphas']} vs {o64.alphas}"
        assert maxdiff(r["alphas"][keep], o64.alphas[keep]) <= 1e-6, f"{tag}: alphas"
        assert int((r["status"] & ~1).max()) == 0, tag
    else:
        check_alphas(tag, r, o64, None)
        check_pnqp(tag, r, o64, kw)
        check_clamps(tag, r, o64, kw)
    check_trajectory(tag, r, P["u"], o64, o32, dtype, keep)
    # the gains also on the scale of the trajectory: these systems' gains can be 14x larger than x and u
    sc = max(1.0, float(o64.new_x.abs().max()), float(o64.new_u.abs().max()))
    for k in ("Ks", "ks"):
        within(tag, k, r[k][:, keep], getattr(o64, k)[:, keep], None if o32 is None else getattr(o32, k)[:, keep],
               dtype, scale=sc)


def _layout(name, B, dtype):
    """(problems per CTA, bulk load path) of the generic step kernel, from the rules in the module docstring."""
    n = PHYS[name]["n"]
    W = {("cartpole", F64): 10, ("cartpole", F32): 20, ("pendulum", F64): 8, ("pendulum", F32): 8}[(name, dtype)]
    sz = 8 if dtype == F64 else 4
    return W, (B * sz) % 16 == 0 and (B * n * sz) % 16 == 0


# (system, dtype, B, bulk path): every B leaves a partial last warp and a partial last CTA
STEP_BATCHES = [("cartpole", F64, 22, True), ("cartpole", F64, 13, False), ("cartpole", F32, 44, True),
                ("cartpole", F32, 43, False), ("pendulum", F64, 20, True), ("pendulum", F64, 21, False),
                ("pendulum", F32, 20, True), ("pendulum", F32, 21, False)]
# (bounds, max_linesearch_iter, decay)
STEP_OPTS = [(None, 10, 0.2), ("scalar", 1, 0.2), ("wide", 2, 0.35), ("tensor", 10, 0.35), ("delta", 2, 0.2)]


@pytest.mark.parametrize("bounds,ls_iter,decay", STEP_OPTS, ids=[f"{b}_ls{i}_d{d}" for b, i, d in STEP_OPTS])
@pytest.mark.parametrize("name,dtype,B,bulk", STEP_BATCHES,
                         ids=[f"{s}_{DT[d]}_B{b}" for s, d, b, _ in STEP_BATCHES])
def test_fused_step_matches_oracle(name, dtype, B, bulk, bounds, ls_iter, decay):
    from mpc.pytorch_b200 import _lib
    W, is_bulk = _layout(name, B, dtype)
    ppw = 5 if name == "cartpole" else 8
    assert is_bulk == bulk and B % W != 0 and (B % W) % ppw != 0
    T = 15
    case = step_case(name, B, T, dtype, bounds, ls_iter, decay, 500 + B)
    r, plan = _run_step(name, T, case, dtype)
    tag = f"{name} {DT[dtype]} B={B} T={T} {bounds} ls={ls_iter} decay={decay}"
    assert plan & _lib.PLAN_GENERIC, f"{tag}: plan {plan}"
    check_step(tag, r, case, dtype)


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("name", SYSTEMS)
def test_fused_step_cases_exercise_the_line_search_and_the_clamp(name, dtype):
    """The step cases above are not vacuous, for each system and dtype, over the batches they use: in every bound
    regime with more than one line-search pass some compared problems end with a decayed alpha; with one pass
    (where alpha is restored at the end) some first passes are worse than the nominal; with bounds wider than the
    clamp some controls go beyond it, where the dynamics see the clamped value."""
    for bounds, ls_iter, decay in STEP_OPTS:
        decayed = worse_first = beyond = 0
        for s, d, B, _ in STEP_BATCHES:
            if (s, d) != (name, dtype):
                continue
            case = step_case(name, B, 15, dtype, bounds, ls_iter, decay, 500 + B)
            _, _, o64, trace, _ = case
            keep = f32_compared(case) if dtype == F32 else torch.ones(B, dtype=torch.bool)
            decayed += int((o64.alphas[keep] < 1).sum())
            worse_first += int((trace[0][keep] > 0).sum())
            beyond += int((o64.new_u.abs() > PHYS[name]["clamp"]).sum())
        tag = f"{name} {DT[dtype]} {bounds}"
        assert (decayed if ls_iter > 1 else worse_first) > 0, f"{tag}: the line search never engages"
        if bounds == "wide":
            assert beyond > 0, f"{tag}: no control beyond the clamp"


@functools.lru_cache(maxsize=None)
def _gain_switch(n, dtype):
    """First horizon at which the generic kernel (known-system instance (n, 1)) keeps its gains in Ks/ks."""
    from mpc.pytorch_b200 import _lib
    return first_true(lambda T: not probe_step(n, 1, dtype, T, 1, True) & _lib.PLAN_GAINS_SMEM)


@pytest.mark.parametrize("name", SYSTEMS)
def test_fused_step_on_both_sides_of_the_gain_store_switch(name):
    """float64, one horizon below and one at the switch where the gains leave shared memory for the caller's
    Ks/ks buffer (found on the device): the plan says so, and both match the oracle."""
    from mpc.pytorch_b200 import _lib
    n, B = PHYS[name]["n"], 13
    Ts = _gain_switch(n, F64)
    assert Ts is not None and 2 < Ts <= 1024, Ts
    for T in (Ts - 1, Ts):
        case = step_case(name, B, T, F64, "scalar", 4, 0.3, 700 + T, calm=True)
        r, plan = _run_step(name, T, case, F64)
        tag = f"{name} f64 B={B} T={T} (switch {Ts})"
        assert plan & _lib.PLAN_GENERIC, tag
        assert bool(plan & _lib.PLAN_GAINS_SMEM) == (T < Ts), f"{tag}: plan {plan}"
        check_step(tag, r, case, F64)


# ------------------------------------------------------------------------------------------------------------------
# MPC.forward: the known system (three kernels per iteration) against the same physics as an opaque Module
# ------------------------------------------------------------------------------------------------------------------
def _mpc_pair(dx, x0, B, T, bounds, lqr_iter=6):
    from mpc.pytorch_b200 import MPC, QuadCost, GradMethods

    class Opaque(torch.nn.Module):                      # hides mpcb200_kind: the generic Module path
        def forward(self, x, u):
            return dx(x, u)

    n = dx.n_state
    q, p = dx.get_true_obj()
    Q = torch.diag(q).double().expand(T, B, n + 1, n + 1).contiguous().to(DEV)
    pp = p.double().expand(T, B, n + 1).contiguous().to(DEV)
    kw = dict(u_lower=-bounds, u_upper=bounds, lqr_iter=lqr_iter, verbose=-1, exit_unconverged=False,
              detach_unconverged=False, linesearch_decay=0.3, max_linesearch_iter=4,
              grad_method=GradMethods.AUTO_DIFF, eps=1e-9)
    a = MPC(n, 1, T, **kw)(x0.to(DEV), QuadCost(Q, pp), dx)
    b = MPC(n, 1, T, **kw)(x0.to(DEV), QuadCost(Q, pp), Opaque())
    return a, b


def _assert_mpc_equal(tag, a, b):
    (xa, ua, ca), (xb, ub, cb) = a, b
    assert maxdiff(ua, ub) < 1e-7 * max(1.0, float(ub.abs().max())), f"{tag}: u {maxdiff(ua, ub):.3e}"
    assert maxdiff(xa, xb) < 1e-7 * max(1.0, float(xb.abs().max())), f"{tag}: x {maxdiff(xa, xb):.3e}"
    assert maxdiff(ca, cb) < 1e-8 * max(1.0, float(cb.abs().max())), f"{tag}: costs {maxdiff(ca, cb):.3e}"


MPC_CASES = [(1, 100), (13, 25), (300, 2), (300, 25)]


@pytest.mark.parametrize("bounds", ["in", "wide"])
@pytest.mark.parametrize("B,T", MPC_CASES, ids=[f"B{b}_T{t}" for b, t in MPC_CASES])
@pytest.mark.parametrize("name", SYSTEMS)
def test_mpc_known_system_equals_module_path(name, B, T, bounds):
    dx = known_module(name)
    clamp = PHYS[name]["clamp"]
    x0 = known_states(name, B, 900 + B + T)
    a, b = _mpc_pair(dx, x0, B, T, (0.8 if bounds == "in" else 2.0) * clamp)
    _assert_mpc_equal(f"{name} B={B} T={T} bounds {bounds}", a, b)


# ------------------------------------------------------------------------------------------------------------------
# parameters changed in place between solves
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", SYSTEMS)
def test_kernels_follow_parameter_edits_between_solves(name):
    """CUDA parameters edited between solves by an optimizer step, a no_grad copy_, .data[i] = and reassignment:
    after each edit the kernel rollout and Jacobians equal the module's own forward and autograd, and MPC.forward
    with the known system equals the same physics run as an opaque Module."""
    from mpc.pytorch_b200.dynamics import dyn_linearize_raw, dyn_rollout_raw
    dx = known_module(name, params=torch.tensor(PHYS[name]["params"], dtype=F64, device=DEV).requires_grad_(True),
                 device=DEV)
    B, T = 9, 12
    x0 = known_states(name, B, 77)
    u = known_controls(name, T, B, F64, 78)
    base = torch.tensor(PHYS[name]["params"], dtype=F64)
    for k, (route, edit) in enumerate(EDIT_ROUTES):
        _mpc_pair(dx, x0, B, T, 2.0 * PHYS[name]["clamp"], lqr_iter=2)      # a solve before the edit
        edit(dx, (base * (1.0 + 0.15 * (k + 1))).to(DEV))
        prm = dx.mpcb200_params()
        assert prm[:len(base)] == tuple(float(v) for v in dx.params.detach().cpu()), route
        x = dyn_rollout_raw(dx.mpcb200_kind, prm, T, x0.to(DEV), u.to(DEV))
        want = dx(x[:-1].reshape(-1, dx.n_state), u[:-1].reshape(-1, 1).to(DEV)).view(T - 1, B, -1)
        assert maxdiff(x[1:], want) <= 1e-12 * max(1.0, float(want.abs().max())), f"{route}: rollout"
        F, f = dyn_linearize_raw(dx.mpcb200_kind, prm, T, x, u.to(DEV))
        _, R, S = jacobians(dx, x[:-1].reshape(-1, dx.n_state).detach(), u[:-1].reshape(-1, 1).to(DEV))
        Fw = torch.cat((R, S), 2).view(T - 1, B, dx.n_state, -1)
        assert maxdiff(F, Fw) <= 1e-11 * max(1.0, float(Fw.abs().max())), f"{route}: Jacobians"
        a, b = _mpc_pair(dx, x0, B, T, 2.0 * PHYS[name]["clamp"], lqr_iter=3)
        _assert_mpc_equal(f"{name} after {route}", a, b)
