"""GPU: receding-horizon episodes (mpcb200_episode_plans_*) and their reverse sweep (mpcb200_episode_backward_*)
against the float64 oracle (orc.receding_horizon_lin, orc.receding_horizon_backward).

Every LinDx case runs the device episode through the C ABI (gpu_harness.abi_episode), then checks
  * the forward: x, u, costs, info, u_next and each solve's best iterate (plan_x, plan_u) against the oracle's
    notebook loop with per-problem pnqp.  The stop test is off (eps = 0, a huge not_improved_lim, a fixed lqr_iter),
    so the solves keep every problem independent, and the per-problem departure rule of test_ilqr_oracle_gpu
    applies: in bounded cases at most one problem in four may leave the tolerance (round-off decides some problems'
    pnqp paths).  One case per dtype keeps the default stop rule;
  * the backward: the device sweep against the oracle's sweep run on the device's OWN plans, xs and us (upcast to
    float64), so forward round-off never reaches the backward check.  float64: within 1e-9 x max(1, max|g|); float32:
    the `within` policy, with the oracle's sweep run in float32 on the same plans as the yardstick;
  * the step plan the solve recorded, and the adjoint's route in the sweep's body (adjoint_route): by the backward's
    launch count, derived from epgrad_record (init, stage and accumulate kernels, 3; a known system's linearisation
    and its VJP, 2; the fused route's prep + column-pair kernel, 2, or any three-launch route's prep, fill_zero,
    masked step and 2 gradient kernels, 5), and by the plan its nested step recorded (check_route).

Cases: LinDx at every compiled instance and a padded shape, with batch tails and batches whose grid-stride loops take
several passes; every step plan of the solve on both sides of its switch horizon (tests/gpu_harness.pick_switch);
every adjoint route of the sweep's body; the input forms (bounds, u_zero_I, F_T, f, a time-invariant F and a
time-invariant cost, which reach the library as stride-0 views over time); the known systems, whose sweep is checked
against the oracle's per-problem parameter gradient and whose forward for consistency (check_known_forward) and end to
end against the reference's fixture (tests/test_known_oracle_gpu.py compares it with oracle/known_oracle.py's
episode); and poisoned workspaces, where
every workspace byte and output starts at 0xFF and the results must be bitwise those of an unpoisoned call.
test_zz_coverage fails if a plan or route never ran."""
import functools
import os

import numpy as np
import pytest
import torch

from oracle import lqr_oracle as orc
from tests.gpu_harness import (DEV, DT, F32, F64, INSTANCES, PAIR_SHAPES, SWITCH_PLANS, abi_episode,
                               abi_episode_backward, check_episode_forward, episode_device_inputs, episode_known_inputs,
                               episode_known_module, episode_known_step, episode_linear_inputs, epgrad_launches,
                               kernel_env, loop_plan, pick_switch, plan_name, plan_str, switches, within)
from tests.helpers import maxdiff

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FWD_SEEN = {}                       # dtype -> step plans run inside the episode
ROUTES_SEEN = {}                    # dtype -> adjoint routes run inside the sweep
ERRS = {}                           # (dtype, what) -> largest observed error relative to max(1, max|want|)
DEPARTED = {}                       # dtype -> [(departing problems, compared problems)]


def _f32(t):
    return t.float() if torch.is_tensor(t) and t.is_floating_point() else t


def _note(dtype, what, err):
    ERRS[(dtype, what)] = max(ERRS.get((dtype, what), 0.0), err)


# ------------------------------------------------------------------------------------------------------------------
# cases
# ------------------------------------------------------------------------------------------------------------------
def loss_weights(n_steps, B, n, m, seed):
    g = torch.Generator().manual_seed(seed + 7)
    return torch.randn(n_steps + 1, B, n, generator=g, dtype=F64), torch.randn(n_steps, B, m, generator=g, dtype=F64)


def fixed_opts(lqr_iter):
    """The stop test off: every solve runs lqr_iter iterations, so no problem's path depends on another's."""
    return dict(lqr_iter=lqr_iter, eps=0.0, not_improved_lim=10 ** 6)


def run_device(n, m, T, n_steps, P, kw, opts, dtype, impl, dyn=None, poison=False):
    d = lambda t: t.to(DEV, dtype) if torch.is_tensor(t) and t.is_floating_point() else \
        (t.to(DEV) if torch.is_tensor(t) else t)  # noqa: E731
    u0 = torch.zeros(T, P["x0"].shape[0], m, dtype=dtype, device=DEV)
    with kernel_env(impl):
        return abi_episode(n, m, T, n_steps, *episode_device_inputs(P, dtype), u0, **{k: d(v) for k, v in kw.items()},
                           **opts, dyn=dyn, poison=poison)


def check_forward(tag, r, o64, o32, kw, dtype, several):
    """gpu_harness.check_episode_forward: x, u, costs, info, u_next and the plans against the oracle's, problem by
    problem; its largest error and departures recorded for test_zz_coverage."""
    err, n_dep, n_cmp = check_episode_forward(tag, r, o64, o32, kw, dtype, several)
    DEPARTED.setdefault(dtype, []).append((n_dep, n_cmp))
    _note(dtype, "forward x/u/u_next/plans", err)


GNAMES = ("dx_init", "dC", "dc", "dF", "df", "dtheta")


def oracle_sweep(n, m, T, P, kw, saved, wx, wu, dtype, step=None, theta=None):
    """The oracle's sweep on the device's own plans, xs and us: float64, and float32 for a float32 case."""
    s, _, xs, us, plan_x, plan_u = saved
    pad = s.pad
    got = [pad.crop_n(xs).cpu(), pad.crop_m(us).cpu(), pad.crop_n(plan_x).cpu(), pad.crop_m(plan_u).cpu()]
    lo, hi = kw.get("u_lower"), kw.get("u_upper")

    def run(cast):
        c = lambda t: cast(t) if torch.is_tensor(t) else t  # noqa: E731
        F = P.get("F")
        return orc.receding_horizon_backward(
            n, m, T, c(P["C"]).contiguous(), c(P["c"]).contiguous(), None if F is None else c(F).contiguous(),
            None if P.get("f") is None else c(P["f"]), *[c(t) for t in got], c(wx), c(wu), u_lower=c(lo),
            u_upper=c(hi), step=step, theta=None if theta is None else c(theta))
    o64 = run(lambda t: t.double())
    o32 = run(lambda t: t.float()) if dtype == F32 else None
    return o64, o32


def check_backward(tag, g, o64, o32, dtype):
    for name, got in zip(GNAMES, g):
        want = o64.get(name)
        if want is None:
            assert got is None, f"{tag}: {name} returned"
            continue
        got = got.cpu()
        assert got.shape == want.shape, f"{tag}: {name} shape {tuple(got.shape)} vs {tuple(want.shape)}"
        assert bool(torch.isfinite(got).all()), f"{tag}: {name} not finite"
        within(tag, name, got, want, None if o32 is None else o32[name], dtype)
        _note(dtype, "backward", maxdiff(got, want) / max(1.0, float(want.abs().max())))


def adjoint_route(N, M, T, B, dtype, impl):
    """The route the adjoint takes in the sweep's body at the staged (N, M) (api.cu adjoint_impl, adj_layout):
      large        the large-shape kernels' three-launch route (no instance, or MPCB200_KERNEL=3);
      three_gains  the nested step keeps its gains in the workspace's Ks/ks slice: from the instance's gain-store
                   switch on (gains_in_workspace, the generic kernel's switch of gpu_harness.switches);
      three_shape  no fused kernel: not a pair shape, or MPCB200_KERNEL=1;
      three_align  a pair shape whose time strides are not all 16-byte multiples;
      three_smem   a pair shape past the fused kernel's shared-memory limit (the adjoint's switch);
      fused        prep + the fused column-pair kernel.
    check_route pins each route by the launch count and by the plan the nested step recorded."""
    if impl == 3 or (N, M) not in INSTANCES:
        return "large"
    sw = switches(N, M, dtype)
    if sw["generic"] is not None and T >= sw["generic"]:
        return "three_gains"
    if (N, M) not in PAIR_SHAPES or impl == 1:
        return "three_shape"
    p = N + M
    if not all(B * k * dtype.itemsize % 16 == 0 for k in (p * p, p, N * p, N, M)):
        return "three_align"
    return "three_smem" if sw["adjoint"] is not None and T >= sw["adjoint"] else "fused"


def check_route(tag, route, launches, plan, known=False):
    """The backward's launch count (epgrad_launches) and the nested step's plan: the column-pair kernel with gains in
    shared memory on the fused route, the large-shape kernels on the large one, no gains in shared memory on
    three_gains, gains in shared memory on the other three-launch routes."""
    L = plan_flags()
    assert launches == epgrad_launches(route, known), f"{tag}: {launches} launches, {route} route expected"
    if route == "large":
        ok = plan == L.PLAN_LARGE
    elif route == "fused":
        ok = bool(plan & L.PLAN_PAIR) and bool(plan & L.PLAN_GAINS_SMEM)
    else:
        ok = plan != L.PLAN_LARGE and bool(plan & L.PLAN_GAINS_SMEM) == (route != "three_gains")
    assert ok, f"{tag}: the adjoint's nested step ran {plan_str(plan)} on the {route} route"


def plan_flags():
    from mpc.pytorch_b200 import _lib
    return _lib


def check_poisoned(tag, clean, fwd_args, wx, wu):
    """Both calls again with every workspace byte and output at 0xFF: every output finite and bitwise the same."""
    r, _, _ = run_device(*fwd_args, poison=True)
    for k in ("x", "u", "costs", "info", "u_next"):
        a = r[k]
        assert not a.is_floating_point() or bool(torch.isfinite(a).all()), f"{tag} poisoned: {k} not finite"
        assert torch.equal(a, clean[0][k]), f"{tag} poisoned: {k} differs"
    for i, k in enumerate(("plan_x", "plan_u")):
        assert torch.equal(r["saved"][4 + i], clean[0]["saved"][4 + i]), f"{tag} poisoned: {k} differs"
    g, _, _ = abi_episode_backward(clean[0]["saved"], wx, wu, poison=True)
    for name, a, b in zip(GNAMES, g, clean[1]):
        if a is None:
            continue
        assert bool(torch.isfinite(a).all()), f"{tag} poisoned: {name} not finite"
        assert torch.equal(a, b), f"{tag} poisoned: {name} differs by {float((a - b).abs().max()):.3e}"


def run_case(tag, n, m, T, B, dtype, n_steps, mode, impl=None, seed=0, lqr_iter=3, fixed=True, want_plan=None,
             want_route=None, poison=False, best_cost_eps=1e-4, **forms):
    """One LinDx episode: forward and backward against the oracle, the plan, the route and the launch count.  A
    time-invariant input must reach the library with time stride 0."""
    P, kw = episode_linear_inputs(seed, B, T, n, m, dtype, mode, **forms)
    opts = fixed_opts(lqr_iter) if fixed else dict(lqr_iter=lqr_iter, eps={F64: 1e-7, F32: 1e-4}[dtype])
    opts["best_cost_eps"] = best_cost_eps
    okw = dict(kw, **opts)
    o64 = orc.receding_horizon_lin(n, m, T, n_steps, P["x0"], P["C"].contiguous(), P["c"].contiguous(),
                                   P["F"].contiguous(), P["f"], coupled=False, **okw)
    o32 = None
    if dtype == F32:
        o32 = orc.receding_horizon_lin(n, m, T, n_steps, *[_f32(P[k]).contiguous() if P[k] is not None else None
                                                           for k in ("x0", "C", "c", "F", "f")], coupled=False,
                                       **{k: _f32(v) for k, v in okw.items()})
    fwd_args = (n, m, T, n_steps, P, kw, opts, dtype, impl)
    r, _, plan = run_device(*fwd_args)
    tag = f"{tag} n{n}m{m} {DT[dtype]} B={B} T={T} steps={n_steps} {mode} MPCB200_KERNEL={impl}"
    name = plan_name(plan, impl, n, m, dtype)
    if want_plan is not None:
        assert name == want_plan, f"{tag}: plan {plan_str(plan)} ({name}), expected {want_plan}"
    FWD_SEEN.setdefault(dtype, set()).add(name)
    s = r["saved"][0]
    for k in P["time_invariant"]:
        ts = getattr(s.dims, k + "_tstride")
        assert ts == -1, f"{tag}: {k} staged with time stride {ts}, not as time invariant"
    check_forward(tag, r, o64, o32, kw, dtype, fixed and (lqr_iter > 1 or n_steps > 1))
    wx, wu = loss_weights(n_steps, B, n, m, seed)
    with kernel_env(impl):
        g, launches, adj_plan = abi_episode_backward(r["saved"], wx.to(DEV, dtype), wu.to(DEV, dtype))
    route = adjoint_route(s.pad.N, s.pad.M, T, B, dtype, impl)
    if want_route is not None:
        assert route == want_route, f"{tag}: the case is meant for the {want_route} route, the rule gives {route}"
    check_route(tag, route, launches, adj_plan)
    ROUTES_SEEN.setdefault(dtype, set()).add(route)
    b64, b32 = oracle_sweep(n, m, T, P, kw, r["saved"], wx, wu, dtype)
    check_backward(tag, g, b64, b32, dtype)
    if poison:
        with kernel_env(impl):
            check_poisoned(tag, (r, g), fwd_args, wx.to(DEV, dtype), wu.to(DEV, dtype))
    return r, g


# ------------------------------------------------------------------------------------------------------------------
# every compiled instance and a padded shape, batch tails, T = 3
# ------------------------------------------------------------------------------------------------------------------
SHAPES = INSTANCES + [(6, 1)]                     # (6, 1) runs zero padded at (6, 2)


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("n,m", SHAPES, ids=[f"n{n}m{m}" for n, m in SHAPES])
def test_every_instance(n, m, dtype):
    """B = 1, unbounded or with u_zero_I (a bounded problem may be the one in four whose pnqp path round-off decides,
    and B = 1 would then leave nothing to compare), and a batch tail (257 = one past a 256-thread block) with bounds
    scalar, tensor or tensor + delta_u; n_steps 1, 2 and 5, T = 3 and 6."""
    k = SHAPES.index((n, m)) + (dtype == F32)
    for j, (B, modes) in enumerate(((1, ("plain", "mask")), (257, ("box", "tensor", "boxT")))):
        run_case("instance", n, m, (3, 6)[(k + j) % 2], B, dtype, (1, 2, 5)[(k + j) % 3], modes[k % len(modes)],
                 seed=100 + 10 * k + j, lqr_iter=2)


GRID = [((16, 4), F64, 3, 22000), ((4, 2), F32, 3, 9800)]


@pytest.mark.parametrize("shape,dtype,T,B", GRID, ids=["n16m4_f64_stage_and_accum", "n4m2_f32_accum"])
def test_grid_stride_passes(shape, dtype, T, B):
    """Batches past epgrad_grid's 4096-block cap: T B (n+m)^2 > 2^20 takes several grid-stride passes in the init
    and accumulate kernels, and at (16, 4) T B max(n, m) > 2^20 in the stage kernel too."""
    n, m = shape
    assert T * B * (n + m) ** 2 > 4096 * 256
    if shape == (16, 4):
        assert T * B * max(n, m) > 4096 * 256
    run_case("grid", n, m, T, B, dtype, 2, "box", seed=300, lqr_iter=1)


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
def test_default_stop_rule(dtype):
    """The default stop rule (eps, not_improved_lim) couples the batch through its stop decision; the oracle's loop
    decides on the same batch-wide norm."""
    run_case("default stop", 8, 2, 10, 16, dtype, 3, "plain", seed=310, lqr_iter=10, fixed=False)


# ------------------------------------------------------------------------------------------------------------------
# every step plan inside the episode, on both sides of its switch horizon; the large-shape kernels
# ------------------------------------------------------------------------------------------------------------------
GROUPS = list(SWITCH_PLANS)


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("group", GROUPS)
def test_plans_at_switch(group, dtype):
    """Episodes just below and at the switch horizon T* of the solve's step plan, under the default dispatch and
    each kernel forced; the plan recorded in the solve is asserted.  The first run at T* also runs poisoned."""
    pick = pick_switch(group, dtype)
    if pick is None:
        pytest.skip(f"no instance has a {group} switch of the loop's step within the oracle's horizons")
    n, m, Ts, impls = pick
    gi = GROUPS.index(group)
    for k, T in enumerate((Ts - 1, Ts)):
        for j, impl in enumerate(impls):
            want = loop_plan(n, m, dtype, T, impl)
            if want is None:
                continue
            run_case(f"{group} (T*={Ts})", n, m, T, 8, dtype, 1 + k, ("box", "plain", "boxT")[(gi + k + j) % 3],
                     impl,
                     seed=400 + 10 * gi + k, lqr_iter=2, want_plan=plan_name(want, impl, n, m, dtype),
                     poison=k == 1 and j == 0)


LARGE = [(20, 4, None, "boxT"), (8, 2, 3, "box"), (16, 4, 3, "plain")]


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("n,m,impl,mode", LARGE, ids=[f"n{c[0]}m{c[1]}_k{c[2]}_{c[3]}" for c in LARGE])
def test_large_shape_kernels(n, m, impl, mode, dtype):
    """A shape without an instance, and MPCB200_KERNEL=3 at instances: the large step in the solve, the large
    three-launch adjoint in the sweep."""
    run_case("large", n, m, 6, 5, dtype, 2, mode, impl, seed=500 + n, lqr_iter=2, want_plan="large",
             want_route="large", poison=impl is None)


# ------------------------------------------------------------------------------------------------------------------
# every adjoint route inside the sweep's body
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
def test_route_fused(dtype):
    run_case("fused", 8, 2, 6, 8, dtype, 3, "tensor", seed=600, want_route="fused", poison=True)


def test_route_three_launch_by_alignment():
    """f32 (n, 2) at an odd B: time strides that are no 16-byte multiple."""
    run_case("3-launch by alignment", 4, 2, 6, 7, F32, 3, "box", seed=610, want_route="three_align", poison=True)


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
def test_route_three_launch_by_gains(dtype):
    """From the adjoint's switch on, the nested step keeps its gains in the workspace's Ks/ks slice and the adjoint
    takes the three-launch route; the solve's step runs past the generic kernel's switch too.  This is where a short
    adjoint slice of the sweep's workspace would overwrite the staged plan behind it.  The second episode keeps each
    solve's first iterate as its best (best_cost_eps = -1e9), so the best iterate must survive two more iterations
    whose step writes its gains into the solve's Ks/ks workspace."""
    n, m = 16, 4
    sw = switches(n, m, dtype)
    assert sw["adjoint"] is not None and sw["generic"] is not None
    T = max(sw["adjoint"], sw["generic"])
    run_case("3-launch by gains", n, m, T, 8, dtype, 2, "box", seed=620, lqr_iter=2, want_route="three_gains",
             poison=True)
    run_case("3-launch by gains, first iterate best", n, m, T, 8, dtype, 2, "plain", seed=621, lqr_iter=3,
             want_route="three_gains", best_cost_eps=-1e9)


# ------------------------------------------------------------------------------------------------------------------
# input forms
# ------------------------------------------------------------------------------------------------------------------
FORMS_T = 8
FORMS = {"F_T_T": dict(F_T=FORMS_T), "f_none": dict(f_T="none"), "f_T": dict(f_T="T"),
         "expand_F": dict(time_invariant=("F",)), "cost_time_invariant": dict(time_invariant=("C", "c")),
         "expand_F_T": dict(time_invariant=("F",), F_T=FORMS_T)}


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("form", list(FORMS))
def test_input_forms(form, dtype):
    """F with T slices (the episode accepts them), f absent or of T slices, a time-invariant F (a stride-0 view over
    time, also with T slices: the stage kernel, the nested step and the adjoint read one slice, and dF comes back per
    slice) and a time-invariant cost C, c (stride 0 over time); bounds none, scalar, tensor, tensor + delta_u and
    u_zero_I."""
    i = list(FORMS).index(form)
    run_case(form, 8, 2, FORMS_T, 12, dtype, 3, ("box", "tensor", "boxT", "mask", "plain", "box")[i], seed=700 + i,
             poison=True, **FORMS[form])


def test_F_T_equal_T_gives_zero_last_slice():
    """F with T slices: dF's last slice never enters the episode and comes back exactly zero."""
    _, g = run_case("F_T=T zero slice", 4, 2, 5, 6, F64, 2, "box", seed=720, poison=True, F_T=5)
    assert bool((g[3][-1] == 0).all())


# ------------------------------------------------------------------------------------------------------------------
# the known systems: the sweep against the oracle's, per problem
# ------------------------------------------------------------------------------------------------------------------
KNOWN = ["cartpole", "pendulum", "pendulum_full"]


def check_known_forward(tag, r, mod, theta, clamp, dtype):
    """What a known-system episode's forward must satisfy without an iLQR oracle: the applied control is the plan's
    first, inside the clamp; each plan starts at its x_k; the model step and each plan's rollout are the module's
    own step (the CPU torch forward, float64, and float32 as the `within` yardstick) from the device's previous
    state; u_next is the last plan shifted."""
    xs, us, plan_x, plan_u = [t.cpu() for t in r["saved"][2:]]
    S, T = plan_u.shape[:2]
    assert torch.equal(us, plan_u[:, 0]) and torch.equal(r["u"].cpu(), us), f"{tag}: applied controls"
    assert torch.equal(plan_x[:, 0], xs[:-1]), f"{tag}: each plan starts at its x_k"
    assert bool((plan_u.abs() <= clamp).all()), f"{tag}: a control beyond the clamp"
    w = r["u_next"].cpu()
    assert torch.equal(w[:-2], plan_u[-1, 1:-1]) and torch.equal(w[-2], w[-3]) and bool((w[-1] == 0).all())
    step = episode_known_step(mod)
    for what, x, u, nxt in (("model step", xs[:-1], us, xs[1:]),
                            ("plan rollout", plan_x[:, :-1], plan_u[:, :-1], plan_x[:, 1:])):
        lead = x.shape[:-2]
        flat = lambda t: t.reshape(-1, t.shape[-1])  # noqa: E731
        th = theta.repeat(int(np.prod(lead)), 1)
        w64 = step(flat(x).double(), flat(u).double(), th).view(nxt.shape)
        w32 = step(flat(x).float(), flat(u).float(), th.float()).view(nxt.shape) if dtype == F32 else None
        within(tag, what, nxt, w64, w32, dtype)


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("B", [1, 7, 300])
@pytest.mark.parametrize("name", KNOWN)
def test_known_systems(name, B, dtype):
    """The known system's sweep (stage kernel's model-step VJP, linearisation, three-launch adjoint, linearisation
    VJP) against the oracle's on the device's own plans; dtheta per problem.  Controls reach the clamp.  The forward
    is checked here for consistency (check_known_forward: the model step and the plans' rollouts) and end to end
    against the reference (test_known_against_reference_fixture); tests/test_known_oracle_gpu.py checks its plans
    against known_oracle's iLQR loop."""
    T, n_steps, seed = 10, 3, 800 + B + KNOWN.index(name)
    mod, n, m, P, kw, dyn, theta = episode_known_inputs(name, B, T, dtype, seed)
    opts = dict(fixed_opts(4), linesearch_decay=mod.linesearch_decay, max_linesearch_iter=mod.max_linesearch_iter)
    fwd_args = (n, m, T, n_steps, P, kw, opts, dtype, None)
    r, _, _ = run_device(*fwd_args, dyn=dyn)
    tag = f"{name} {DT[dtype]} B={B}"
    check_known_forward(tag, r, mod, theta.expand(B, -1), kw["u_upper"], dtype)
    plans_u = r["saved"][5].cpu()
    assert bool((plans_u.abs() == kw["u_upper"]).any()), f"{name}: no control reaches the clamp"
    wx, wu = loss_weights(n_steps, B, n, m, seed)
    g, launches, adj_plan = abi_episode_backward(r["saved"], wx.to(DEV, dtype), wu.to(DEV, dtype))
    check_route(tag, adjoint_route(n, m, T, B, dtype, None), launches, adj_plan, known=True)
    ROUTES_SEEN.setdefault(dtype, set()).add(adjoint_route(n, m, T, B, dtype, None))
    b64, b32 = oracle_sweep(n, m, T, P, kw, r["saved"], wx, wu, dtype, step=episode_known_step(mod),
                            theta=theta.expand(B, -1))
    check_backward(tag, g, b64, b32, dtype)
    if B == 7:
        r2, _, _ = run_device(*fwd_args, dyn=dyn, poison=True)
        for k in ("x", "u", "costs", "info", "u_next"):
            assert torch.equal(r2[k], r[k]), f"{name} poisoned: {k}"
        g2, _, _ = abi_episode_backward(r["saved"], wx.to(DEV, dtype), wu.to(DEV, dtype), poison=True)
        for nm, a, b in zip(GNAMES, g2, g):
            assert a is None or (bool(torch.isfinite(a).all()) and torch.equal(a, b)), f"{name} poisoned: {nm}"


@pytest.mark.parametrize("name", KNOWN)
def test_known_against_reference_fixture(name):
    """receding_horizon(..., differentiable=True).backward() on the reference's own known-system episode
    (oracle/make_golden_receding_grad.py): x, u and the gradients of x_init, C and c at the bounded tolerance of
    test_receding_grad_gpu.test_against_reference_fixture (pnqp's own accuracy).  The reference's params.grad
    differentiates its linearisation with the Jacobians held constant; this project's adds their derivative
    (INTEGRATION.md section 2), so params.grad is compared with the reference's plus that term, which the oracle
    computes on the reference's plans."""
    from mpc.pytorch_b200.control import receding_horizon
    from mpc.pytorch_b200.solver import MPC, GradMethods, QuadCost
    z = np.load(os.path.join(GOLD, "receding_grad_known_f64.npz"))
    pre = name + "_"
    t = {k[len(pre):]: torch.from_numpy(z[k]) for k in z.files
         if k.startswith(pre) and not (name == "pendulum" and k.startswith("pendulum_full_"))}
    T, steps, clamp = int(t["T"]), int(t["n_steps"]), float(t["clamp"])
    mod, _ = episode_known_module(name)
    lv = {k: t[k].clone().to(DEV).requires_grad_(True) for k in ("x_init", "C", "c", "params")}
    mod.params = lv["params"]
    if name == "cartpole":
        mod.force_mag = clamp
    else:
        mod.max_torque = clamp
    n, m = mod.n_state, mod.n_ctrl
    ctrl = MPC(n, m, T, u_lower=-clamp, u_upper=clamp, lqr_iter=int(t["lqr_iter"]), eps=float(t["eps"]), verbose=-1,
               linesearch_decay=float(t["ls_decay"]), max_linesearch_iter=int(t["ls_iter"]),
               grad_method=GradMethods.AUTO_DIFF)
    ep = receding_horizon(ctrl, lv["x_init"], QuadCost(lv["C"], lv["c"]), mod, steps, differentiable=True)
    ((t["wx"].to(DEV) * ep.x).sum() + (t["wu"].to(DEV) * ep.u).sum()).backward()
    tol = 2e-4
    errs = {"x": maxdiff(ep.x, t["x"].to(DEV)), "u": maxdiff(ep.u, t["u"].to(DEV))}
    ref_mod, _ = episode_known_module(name)
    if name == "cartpole":
        ref_mod.force_mag = clamp
    else:
        ref_mod.max_torque = clamp
    B = t["x"].shape[1]
    args = (n, m, T, t["C"], t["c"], None, None, t["x"], t["u"], t["plan_x"], t["plan_u"], t["wx"], t["wu"])
    kw = dict(u_lower=-clamp, u_upper=clamp, step=episode_known_step(ref_mod), theta=t["params"].expand(B, -1))
    full = orc.receding_horizon_backward(*args, **kw)
    const = orc.receding_horizon_backward(*args, full_linearisation=False, **kw)
    assert maxdiff(const["dtheta"].sum(0), t["g_params"]) <= 1e-10 * float(t["g_params"].abs().max())
    want = {"x_init": t["g_x_init"], "C": t["g_C"], "c": t["g_c"],
            "params": t["g_params"] + full["dtheta"].sum(0) - const["dtheta"].sum(0)}
    for k, w in want.items():
        errs["d" + k] = maxdiff(lv[k].grad, w.to(DEV)) / max(1.0, float(w.abs().max()))
    print(f"{name}: " + ", ".join(f"{k} {v:.2e}" for k, v in errs.items()))
    assert all(v <= tol for v in errs.values()), errs


# ------------------------------------------------------------------------------------------------------------------
# coverage (runs last)
# ------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _needed_plans(dtype):
    need = {"large"}
    for group, plans in SWITCH_PLANS.items():
        if pick_switch(group, dtype) is not None:
            need |= set(plans)
    return need


def test_zz_coverage():
    if not FWD_SEEN:
        pytest.skip("no episode test of this module ran")
    missing = []
    for dtype in (F64, F32):
        seen, routes = FWD_SEEN.get(dtype, set()), ROUTES_SEEN.get(dtype, set())
        print(f"{DT[dtype]}: step plans run in the episode {sorted(seen)}; adjoint routes run in the sweep "
              f"{sorted(routes)}")
        missing += [f"{DT[dtype]} plan {p}" for p in sorted(_needed_plans(dtype) - seen)]
        need_routes = {"fused", "three_shape", "three_gains", "large"} | ({"three_align"} if dtype == F32 else set())
        missing += [f"{DT[dtype]} route {r}" for r in sorted(need_routes - routes)]
    for (dtype, what), v in sorted(ERRS.items(), key=lambda kv: (DT[kv[0][0]], kv[0][1])):
        print(f"{DT[dtype]} {what}: largest error {v:.3e} of max(1, max|want|)")
    for dtype, v in DEPARTED.items():
        print(f"{DT[dtype]}: problems departing from the oracle {sum(a for a, _ in v)} of {sum(b for _, b in v)} "
              f"compared, in {sum(a > 0 for a, _ in v)} of {len(v)} runs")
    assert not missing, "never run: " + ", ".join(missing)
