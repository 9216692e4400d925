"""GPU: the known systems' device iLQR loop and episodes against the float64 oracle of that loop
(oracle/known_oracle.py).  The loop is step.ilqr_raw(..., dyn=(kind, params)): one CUDA graph of rollout ->
dyn_linearize -> step with the in-kernel line search -> track -> stop, the known-system branch of api.cu's
ilqr_record.  Its kinds: CartpoleDx (5, 1), PendulumDx (3, 1), PendulumDx(simple=False) on its dynamics-only (3, 1)
instance, and each of them under a slew-rate penalty, the passthrough kinds at (6, 1) and (4, 1).

Rules (those of test_ilqr_oracle_gpu and test_mlp_oracle_gpu): every output and workspace starts as NaN; the stop test
is off (eps = 0, not_improved_lim > lqr_iter) except in one case per dtype, which keeps the default rule and must
match the oracle's iteration count; float64 within 1e-9 x scale, float32 by `within` against the oracle run in
float32 (the pendulum kinds unbounded or masked in float32: F32_PENDULUM_BOUNDS); a problem may depart only under
gpu_harness.check_loop_departures' rule.  Trajectories stay where round-off
is not amplified: the module's own cost around its target (with a small push on the control), moderate dt and
known_states' initial states (radii 0.3, 1 and 3, the theta edge rows).

Cases: every kind in both dtypes; every step plan the loop body records on both sides of each kind's gain-store
switch (found on the device by mpcb200_step_prefers_workspace with the kind, as the loop's layout asks it);
MPCB200_KERNEL = 1, 2, 3 with every kind; bounds none, inside, at and twice the clamp, tensor, tensor + delta_u and
u_zero_I; line searches of 1, 2 and 10 passes with two decays at default and other physics; a time-invariant cost
through MPC.forward; batch layouts with partial warps and CTAs on the bulk and per-lane load paths; a pool batch whose
track and stop kernels take two grid-stride passes; and episodes with the model stepping, a slew-rate penalty and a
known plant with and without w, and a time-varying window with tensor bounds (episodes in float64: in float32 the
episode's bounds sit at the clamp, where the float32 yardstick departs as above).  test_zz_known_loop_plan_coverage fails if a reachable plan never ran."""
import ctypes
import functools

import pytest
import torch

from mpc.pytorch_b200 import _lib
from mpc.pytorch_b200.dynamics import (DYN_CARTPOLE, DYN_CTRL_PASSTHROUGH, DYN_PENDULUM, DYN_PENDULUM_FULL,
                                       CartpoleDx, PendulumDx)
from oracle import known_oracle as ko
from tests.gpu_harness import (DEV, DT, F32, F64, ORACLE_TMAX, TMAX, check_episode_forward, check_loop_departures,
                               episode_known_step, first_true, kernel_env, known_states, layout_batches, on_bounds,
                               plan, plan_str, pool_size, round_through, run_loop, step_layout)

pytestmark = pytest.mark.gpu

# name: (kind, n, module constructor options, other physics: params, dt, clamp)
SYSTEMS = {"cartpole": (DYN_CARTPOLE, 5, {}, ((9.81, 1.3, 0.25, 0.8), 0.05, 7.5)),
           "pendulum": (DYN_PENDULUM, 3, {}, ((9.1, 1.7, 0.6), 0.1, 1.5)),
           "pendulum_full": (DYN_PENDULUM_FULL, 3, dict(simple=False), ((9.1, 1.7, 0.6, 0.4, 0.25), 0.1, 1.5))}
DEFAULT_PARAMS = {"cartpole": (9.8, 1.0, 0.1, 0.5), "pendulum": (10.0, 1.0, 1.0),
                  "pendulum_full": (10.0, 1.0, 1.0, 0.1, 0.05)}
KINDS = [(name, slew) for slew in (0, 1) for name in SYSTEMS]
KIND_IDS = [f"{name}{'_slew' if slew else ''}" for name, slew in KINDS]
SLEW = 0.5
DTYPES = (F64, F32)
# bound forms of the pendulum kinds in float32: with a box, the float32 oracle (the yardstick) lands controls on a bound
# where the float64 one does not on nearly every problem (bounds inside the clamp: 11 to 13 of 13 problems at T = 12),
# so the departure rule has nothing left to compare; unbounded and masked, it leaves none.  Cartpole and its
# passthrough kind run every bound form in float32.
F32_PENDULUM_BOUNDS = ("none", "mask")


# systems whose float32 loop is compared at its switch horizon: over the 576 to 887 steps of the pendulums' float32
# switches, the float32 oracle's one iteration leaves the float64 one by more than 1e-4 of the scale on every problem
# (an undamped swing's phase error grows with the horizon), so only cartpole (T* = 214) keeps problems to compare
F32_SWITCH_SYSTEMS = ("cartpole",)


def f32_bounds(name, bounds, dtype):
    """The bound form a case runs in dtype (F32_PENDULUM_BOUNDS)."""
    if dtype == F32 and name != "cartpole" and bounds not in F32_PENDULUM_BOUNDS:
        return "none"
    return bounds
SEEN = {}                           # dtype -> {(kind name, plan name)} run in the loop
DEPARTED = []                       # (tag, departing, compared, largest error)
SWITCHES = {}                       # (kind name, dtype) -> switch horizon


def kind_name(name, slew):
    return name + ("_slew" if slew else "")


def module(name, physics="other"):
    """(module, float64 parameter row, clamp) of a known system at its default or other physics.  "undamped": the
    other physics without the five-parameter pendulum's damping d, whose term d atan2(sin, cos) jumps where a swing
    passes +-pi, so that long horizons do not amplify round-off there."""
    kind, n, extra, (params, dt, clamp) = SYSTEMS[name]
    ctor = CartpoleDx if kind == DYN_CARTPOLE else PendulumDx
    if physics == "default":
        params = DEFAULT_PARAMS[name]
    elif physics == "undamped" and name == "pendulum_full":
        params = params[:3] + (0.0,) + params[4:]
    p = torch.tensor(params, dtype=F64)
    mod = ctor(params=p, **extra)
    if physics != "default":
        mod.dt = dt
        setattr(mod, "force_mag" if kind == DYN_CARTPOLE else "max_torque", clamp)
    clamp = float(mod.force_mag if kind == DYN_CARTPOLE else mod.max_torque)
    return mod, p, clamp


BOUNDS = ("none", "in", "at", "wide", "tensor", "tensorD", "mask")


@functools.lru_cache(maxsize=8)
def loop_case(name, slew, B, T, dtype, bounds, seed, lqr_iter=3, physics="other", decay=0.5, max_ls=4,
              stop_rule=False, time_invariant=False, calm=False):
    """A known system's solve: (mod, N, P, kw, opts, dyn, o64, o32|None, sensitive).  The module's own cost with a
    small push on the control, known_states' initial states; under a slew-rate penalty (slew = 1) the passthrough
    problem of slew_problem from a previous control inside the clamp.  time_invariant: the push is the same at every
    time step, so C and c are.  calm: angles within 0.5 of the target, so that long horizons never reach the wrapped
    angle's jump at +-pi (PendulumDx(simple=False) damps atan2(sin, cos)).  Inputs in float64 rounded through dtype."""
    mod, p, clamp = module(name, physics)
    kind, n = SYSTEMS[name][:2]
    dyn = (kind | (DYN_CTRL_PASSTHROUGH if slew else 0), mod.mpcb200_params())
    g = torch.Generator().manual_seed(seed)
    q, pp = mod.get_true_obj()
    C = torch.diag(q.double()).expand(T, B, n + 1, n + 1).contiguous()
    c = pp.double().expand(T, B, n + 1).contiguous()
    push = 0.0 if calm else 0.3 * clamp
    c[..., n:] = push * (torch.rand(1 if time_invariant else T, B, 1, generator=g, dtype=F64) - 0.5)
    x0 = known_states("cartpole" if name == "cartpole" else "pendulum", B, seed)
    if calm:
        th = 0.5 * (2 * torch.rand(B, generator=g, dtype=F64) - 1)
        ic = 2 if name == "cartpole" else 0
        x0[:, ic], x0[:, ic + 1] = th.cos(), th.sin()
    if slew:
        prev = 0.6 * clamp * (torch.rand(B, 1, generator=g, dtype=F64) - 0.5)
        x0, C, c = ko.slew_problem(n, 1, SLEW, C, c, x0, prev)
    kw = {}
    if bounds in ("in", "at", "wide"):
        b = {"in": 0.8, "at": 1.0, "wide": 2.0}[bounds] * clamp
        kw = dict(u_lower=-b, u_upper=b)
    elif bounds in ("tensor", "tensorD"):
        kw = dict(u_lower=-clamp * (0.3 + 1.2 * torch.rand(T, B, 1, generator=g, dtype=F64)),
                  u_upper=clamp * (0.3 + 1.2 * torch.rand(T, B, 1, generator=g, dtype=F64)))
        if bounds == "tensorD":
            kw["delta_u"] = 0.4 * clamp
    elif bounds == "mask":
        kw["u_zero_I"] = torch.rand(T, B, 1, generator=g) < 0.3
    C, c, x0 = (round_through(t, dtype) for t in (C, c, x0))
    kw = {k: round_through(v, dtype) for k, v in kw.items()}
    N = n + slew
    opts = dict(lqr_iter=lqr_iter, eps=0.0, not_improved_lim=lqr_iter + 1, linesearch_decay=decay,
                max_linesearch_iter=max_ls)
    if stop_rule:
        opts.update(eps=1e-7, not_improved_lim=5)
    step = episode_known_step(module(name, physics)[0])        # it sets its module's params per call

    def oracle(cast, Cs=C):
        return ko.ilqr(N, 1, T, cast(x0), cast(Cs), cast(c), step, cast(p).expand(B, -1),
                       u_init=torch.zeros(T, B, 1, dtype=cast(x0).dtype), n_prev=slew, coupled=False,
                       **{k: cast(v) if torch.is_tensor(v) and v.is_floating_point() else v for k, v in kw.items()},
                       **opts)
    o64 = oracle(lambda t: t)
    o32 = oracle(lambda t: t.float()) if dtype == F32 else None

    def sensitive(tol):
        """[B]: problems whose float64 oracle loop moves by more than tol, or changes its controls on a bound, when C
        is scaled by 1 +- 1e-15."""
        moved = torch.zeros(B, dtype=torch.bool)
        for s_ in (1 + 1e-15, 1 - 1e-15):
            o = oracle(lambda t: t, C * s_)
            moved |= torch.maximum((o[0] - o64[0]).abs().amax((0, 2)), (o[1] - o64[1]).abs().amax((0, 2))) > tol
            if "u_lower" in kw:
                moved |= (on_bounds(o[1], kw) != on_bounds(o64[1], kw)).any(3).any(1).any(0)
        return moved
    return mod, N, dict(x0=x0, C=C, c=c, F=None, f=None), kw, opts, dyn, o64, o32, sensitive


def take(case, idx):
    """P, kw of a case's batch rows idx."""
    _, _, P, kw = case[:4]
    B = P["x0"].shape[0]
    rows = lambda t: t.index_select(0 if t.dim() == 2 and t.shape[0] == B else 1, idx) \
        if torch.is_tensor(t) else t  # noqa: E731
    return {k: rows(v) for k, v in P.items()}, {k: rows(v) for k, v in kw.items()}


def run(case, T, dtype, impl=None, idx=None):
    """step.ilqr_raw with the case's known kind, every output and workspace NaN before the call: (outputs, plan)."""
    from tests.test_mlp_gpu import poisoned
    _, N, P, kw, opts, dyn = case[:6]
    if idx is not None:
        P, kw = take(case, idx)
    P = dict(P, u0=torch.zeros(T, P["x0"].shape[0], 1, dtype=F64))
    with poisoned():
        return run_loop(N, 1, T, P, kw, dict(opts, dyn=dyn), dtype, impl)


def check(tag, r, case, dtype, idx=None):
    o64, o32, sensitive = case[6:]
    rep = check_loop_departures(tag, r, o64, o32, case[3], case[4]["lqr_iter"], sensitive, dtype, idx)
    DEPARTED.append(rep)
    want = o64[3] if o32 is None else o32[3]
    assert int(r["info"][0]) == want, f"{tag}: {int(r['info'][0])} iterations, the oracle {want}"
    if case[5][0] & DYN_CTRL_PASSTHROUGH:
        assert torch.equal(r["x"][1:, :, :1], r["u"][:-1]), f"{tag}: carried previous controls"


@functools.lru_cache(maxsize=None)
def gain_switch(kind, N, dtype, knob=None):
    """First horizon at which the step of `kind` at (N, 1) keeps its gains in Ks/ks (the loop's layout then hands it
    Ks/ks); None if not within TMAX."""
    L = _lib.lib()

    def ws(T):
        d = _lib.Dims(B=1, T=T, n=N, m=1, F_T=T - 1, has_f=1, dynamics_kind=kind, max_ls_iter=1, pnqp_max_iter=1,
                      do_rollout=1)
        with kernel_env(knob):
            return bool(L.mpcb200_step_prefers_workspace(ctypes.byref(d), 8 if dtype == F64 else 4))
    if ws(2):
        return 2
    return first_true(ws, 2, TMAX)


def plan_name(p):
    if p & _lib.PLAN_PAIR:
        return "pair" + ("_smem" if p & _lib.PLAN_GAINS_SMEM else "_ks")
    assert p & _lib.PLAN_GENERIC, plan_str(p)
    return "generic" + ("_smem" if p & _lib.PLAN_GAINS_SMEM else "_ks")


def seen(name, slew, dtype, p):
    SEEN.setdefault(dtype, set()).add((kind_name(name, slew), plan_name(p)))


# ------------------------------------------------------------------------------------------------------------------
# every kind, the stop rule, the switch
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=[DT[d] for d in DTYPES])
@pytest.mark.parametrize("name,slew", KINDS, ids=KIND_IDS)
def test_every_kind(name, slew, dtype):
    T, B = 12, 13
    case = loop_case(name, slew, B, T, dtype, f32_bounds(name, "in", dtype), 100 + 3 * slew + len(name))
    r, p = run(case, T, dtype)
    kind, N = case[5][0], case[1]
    Ts = gain_switch(kind, N, dtype)
    assert p == plan(True, Ts is None or T < Ts), f"plan {plan_str(p)}"
    seen(name, slew, dtype, p)
    check(f"{kind_name(name, slew)} {DT[dtype]}", r, case, dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=[DT[d] for d in DTYPES])
def test_default_stop_rule(dtype):
    """eps = 1e-7 and not_improved_lim = 5 over up to 30 iterations: the device stops where the oracle stops (16
    iterations in float64)."""
    T, B = 15, 16
    case = loop_case("cartpole", 0, B, T, dtype, "in", 150, lqr_iter=30, physics="default", decay=0.2, max_ls=5,
                     stop_rule=True)
    r, _ = run(case, T, dtype)
    assert 1 < case[6][3] < 30, case[6][3]
    check(f"stop rule {DT[dtype]}", r, case, dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=[DT[d] for d in DTYPES])
@pytest.mark.parametrize("name,slew", KINDS, ids=KIND_IDS)
def test_plans_at_switch(name, slew, dtype):
    """Just below and at the kind's gain-store switch: gains in shared memory, then in the loop's Ks/ks, from calm
    initial states (loop_case) and without the damping term of the five-parameter pendulum (module): over hundreds of
    steps its swings reach +-pi, where that term jumps, and the damped float64 oracle itself then moves by up to 18
    under a 1e-15 relative change of x_init (test_known_oracle_cpu checks it).  float32 runs one iteration: at these
    horizons later iterations compare costs of hundreds of stages that differ by less than float32 resolves, so
    round-off would decide their line searches.  A float32 run would take one iteration: at these horizons later iterations compare
    costs of hundreds of stages that differ by less than float32 resolves, so round-off would decide their line
    searches."""
    kind, n = SYSTEMS[name][:2]
    N = n + slew
    k = kind | (DYN_CTRL_PASSTHROUGH if slew else 0)
    Ts = gain_switch(k, N, dtype)
    SWITCHES[(kind_name(name, slew), DT[dtype])] = Ts
    if Ts is None or Ts > ORACLE_TMAX:
        pytest.skip(f"no gain-store switch within T <= {ORACLE_TMAX} (T* = {Ts})")
    if dtype == F32 and name not in F32_SWITCH_SYSTEMS:
        pytest.skip(f"float32 at T* = {Ts}: the float32 yardstick leaves every problem (F32_SWITCH_SYSTEMS)")
    for i, T in enumerate((Ts - 1, Ts)):
        if T < 2:
            continue
        case = loop_case(name, slew, 8, T, dtype, f32_bounds(name, ("in", "tensor")[i], dtype), 200 + i,
                         lqr_iter=3 if dtype == F64 else 1, calm=True, physics="undamped")
        r, p = run(case, T, dtype)
        tag = f"{kind_name(name, slew)} {DT[dtype]} T={T} (T*={Ts})"
        assert p == plan(True, T < Ts), f"{tag}: plan {plan_str(p)}"
        seen(name, slew, dtype, p)
        check(tag, r, case, dtype)


# ------------------------------------------------------------------------------------------------------------------
# the developer knob
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("knob", [1, 2, 3])
@pytest.mark.parametrize("name,slew", KINDS, ids=KIND_IDS)
def test_kernel_knob(name, slew, knob):
    """MPCB200_KERNEL with a known kind.  1 records the default plan.  2 asks for the column-pair kernel, which has no
    in-kernel dynamics: the loop is refused with MPCB200_ERR_UNSUPPORTED_DIMS.  3: mpcb200_step_prefers_workspace
    answers Ks/ks at every horizon for cartpole and pendulum (gains_in_workspace asks runs_large of (n, m)), so the
    loop hands the step Ks/ks, but the generic instance that runs a known kind keeps its gains in shared memory below
    its own switch: the plan is the default one, and the results match the oracle.  The dynamics-only instances keep
    their own switch."""
    from mpc.pytorch_b200.step import ilqr_raw
    T, dtype = 10, F64
    case = loop_case(name, slew, 9, T, dtype, "in", 300 + knob)
    kind, N = case[5][0], case[1]
    tag = f"{kind_name(name, slew)} MPCB200_KERNEL={knob}"
    if knob == 2:
        _, _, P, kw, opts, dyn = case[:6]
        d = lambda t: t.to(DEV, dtype) if torch.is_tensor(t) and t.is_floating_point() else t  # noqa: E731
        with kernel_env(2), pytest.raises(_lib.MpcB200Error, match=r"\[3\]"):
            ilqr_raw(N, 1, T, d(P["x0"]), d(P["C"]), d(P["c"]), None, None, torch.zeros(T, 9, 1, dtype=dtype,
                     device=DEV), **{k: d(v) for k, v in kw.items()}, **opts, dyn=dyn)
        return
    r, p = run(case, T, dtype, knob)
    own = bool(slew) or name == "pendulum_full"
    assert (gain_switch(kind, N, dtype, knob) == 2) == (knob == 3 and not own), f"{tag}: workspace answer"
    Ts = gain_switch(kind, N, dtype)
    assert p == plan(True, Ts is None or T < Ts), f"{tag}: plan {plan_str(p)}"
    seen(name, slew, dtype, p)
    check(tag, r, case, dtype)


# ------------------------------------------------------------------------------------------------------------------
# inputs and line searches
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=[DT[d] for d in DTYPES])
@pytest.mark.parametrize("bounds", BOUNDS)
def test_inputs(bounds, dtype):
    """Bounds none (only the clamp inside the dynamics), inside, at and twice the clamp (S is exactly 0 beyond it),
    tensor bounds, tensor bounds + delta_u and u_zero_I, each on every system in turn and its passthrough kind."""
    T, B = 10, 12
    i = BOUNDS.index(bounds)
    for name in SYSTEMS:
        if f32_bounds(name, bounds, dtype) != bounds:
            continue
        slew = (i + len(name)) % 2
        case = loop_case(name, slew, B, T, dtype, bounds, 400 + i)
        if bounds == "wide":
            clamp = module(name)[2]
            assert bool((case[6][1].abs() > clamp).any()), "no control passes the clamp"
        r, p = run(case, T, dtype)
        seen(name, slew, dtype, p)
        check(f"{kind_name(name, slew)} {bounds} {DT[dtype]}", r, case, dtype)


LS = [(1, 0.5), (2, 0.5), (10, 0.5), (1, 0.2), (2, 0.2), (10, 0.2)]


def ls_args(j, max_ls, decay, dtype):
    """(physics, bounds) of test_line_search's system j (cartpole, pendulum): the physics alternate with the case."""
    name = ("cartpole", "pendulum")[j]
    return ("default", "other")[(j + LS.index((max_ls, decay))) % 2], f32_bounds(name, "in", dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=[DT[d] for d in DTYPES])
@pytest.mark.parametrize("max_ls,decay", LS, ids=[f"ls{a}_d{b}" for a, b in LS])
def test_line_search(max_ls, decay, dtype):
    """max_linesearch_iter 1, 2 and 10 with two decays, at the default and other physics, dt and clamp."""
    T, B = 15, 16
    for j, name in enumerate(("cartpole", "pendulum")):
        physics, bounds = ls_args(j, max_ls, decay, dtype)
        case = loop_case(name, 0, B, T, dtype, bounds, 500 + max_ls, lqr_iter=4, physics=physics, decay=decay,
                         max_ls=max_ls)
        r, p = run(case, T, dtype)
        seen(name, 0, dtype, p)
        check(f"{name} {physics} ls={max_ls} decay={decay} {DT[dtype]}", r, case, dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=[DT[d] for d in DTYPES])
def test_time_invariant_cost_through_mpc_forward(dtype):
    """MPC.forward on a QuadCost of expanded (time-invariant) C, c: the loop receives stride-0 C and c and the known
    kind, and matches the oracle."""
    from mpc.pytorch_b200 import step as S
    from mpc.pytorch_b200.solver import MPC, GradMethods, QuadCost
    from tests.test_mlp_gpu import poisoned
    T, B = 10, 12
    case = loop_case("pendulum", 0, B, T, dtype, f32_bounds("pendulum", "in", dtype), 600, time_invariant=True)
    _, N, P, kw, opts = case[:5]
    C0, c0 = (P[k][:1].to(DEV, dtype) for k in ("C", "c"))
    cost = QuadCost(C0.expand(T, *C0.shape[1:]), c0.expand(T, *c0.shape[1:]))
    mod_d = module("pendulum")[0]
    mod_d.params = mod_d.params.to(DEV, dtype)
    ctrl = MPC(N, 1, T, u_lower=kw.get("u_lower"), u_upper=kw.get("u_upper"), lqr_iter=opts["lqr_iter"], eps=0.0,
               not_improved_lim=opts["not_improved_lim"], linesearch_decay=opts["linesearch_decay"],
               max_linesearch_iter=opts["max_linesearch_iter"], verbose=-1, grad_method=GradMethods.ANALYTIC,
               exit_unconverged=False, detach_unconverged=False)
    calls = []
    real = S.ilqr_raw
    S.ilqr_raw = lambda *a, **k: calls.append((a[4].stride(0), a[5].stride(0), k.get("dyn"))) or real(*a, **k)
    try:
        with torch.no_grad(), poisoned():
            x, u, costs = ctrl(P["x0"].to(DEV, dtype), cost, mod_d)
    finally:
        S.ilqr_raw = real
    assert len(calls) == 1 and calls[0][:2] == (0, 0) and calls[0][2][0] == DYN_PENDULUM, calls
    r = dict(x=x.cpu(), u=u.cpu(), costs=costs.cpu(), info=ctrl._solve_info.cpu())
    check(f"time-invariant cost {DT[dtype]}", r, case, dtype)


# ------------------------------------------------------------------------------------------------------------------
# batch layouts
# ------------------------------------------------------------------------------------------------------------------
def layout_of(name, slew, dtype):
    """(problems per warp, per CTA) of the generic step kernel at the kind's instance (StepCfg)."""
    n = SYSTEMS[name][1] + slew
    return step_layout("generic", n, 1, dtype)


def layout_Bs(name, slew, dtype):
    """layout_batches of the kind's step layout, B = 1, 127, 128, 129, and W + 2, 2 W + ppw + 2: partial CTAs at
    an even B (bulk loads where B n elements make a 16-byte span) as well as odd ones (per-lane loads)."""
    ppw, W = layout_of(name, slew, dtype)
    return sorted(set(layout_batches(ppw, W)) | {1, 127, 128, 129, W + 2, 2 * W + ppw + 2})


@pytest.mark.parametrize("dtype", DTYPES, ids=[DT[d] for d in DTYPES])
@pytest.mark.parametrize("name,slew", [("cartpole", 0), ("pendulum", 0), ("pendulum_full", 1)],
                         ids=["cartpole", "pendulum", "pendulum_full_slew"])
def test_batch_layouts(name, slew, dtype):
    """B = 1, 127, 128, 129 (the 128-thread dynamics kernels) and the step kernel's layout batches: partial, full and
    overfull warps and CTAs, odd B (per-lane loads: B n elements are not a 16-byte span) and even B (bulk loads)."""
    ppw, W = layout_of(name, slew, dtype)
    Bs = layout_Bs(name, slew, dtype)
    T = 8
    for B in Bs:
        case = loop_case(name, slew, B, T, dtype, f32_bounds(name, "in", dtype), 700 + B)
        r, p = run(case, T, dtype)
        seen(name, slew, dtype, p)
        check(f"{kind_name(name, slew)} B={B} (warp {ppw}, CTA {W}) {DT[dtype]}", r, case, dtype)


GRID_CAP = 4096 * 256               # ilqr_grid: at most 4096 blocks of 256 threads per pass


def test_pool_batch_takes_two_grid_passes():
    """B tiles a pool of K problems (K coprime to every layout): the track kernel's T B N items and the stop
    kernel's B problems take two grid-stride passes.  Sampled rows against the oracle; each sampled problem solved
    alone gives its row bit for bit."""
    name, slew, T, dtype = "pendulum", 0, 10, F64
    ppw, W = layout_of(name, slew, dtype)
    K = pool_size(ppw, W, 128, 256)
    N = SYSTEMS[name][1]
    B = GRID_CAP // (T * N) + 2 * W + 1
    assert GRID_CAP < T * B * N < 2 * GRID_CAP
    case = loop_case(name, slew, K, T, dtype, "tensor", 800)
    idx = torch.arange(B) % K
    r, p = run(case, T, dtype, idx=idx)
    seen(name, slew, dtype, p)
    samples = torch.tensor(sorted({0, W - 1, W, 127, 128, GRID_CAP // (T * N), B - 2, B - 1}))
    sub = {k: (v[:, samples] if v.dim() == 3 else v[samples]) if k != "info" else v for k, v in r.items()}
    check(f"pool B={B} K={K}", sub, case, dtype, idx=idx[samples])
    for b in samples.tolist():
        one, _ = run(case, T, dtype, idx=idx[b:b + 1])
        assert torch.equal(one["x"], r["x"][:, b:b + 1]) and torch.equal(one["u"], r["u"][:, b:b + 1]), b


# ------------------------------------------------------------------------------------------------------------------
# episodes with a known model
# ------------------------------------------------------------------------------------------------------------------
EPISODES = [("cartpole", "none", False, False), ("pendulum", "none", False, False),
            ("pendulum_full", "none", False, False), ("cartpole", "none", False, True),
            ("pendulum", "none", False, True), ("pendulum_full", "none", False, True),
            ("pendulum", "pendulum_full", False, False), ("pendulum", "pendulum_full", True, False),
            ("cartpole", "cartpole", False, False), ("cartpole", "cartpole", True, False)]


@pytest.mark.parametrize("B", [1, 7, 300])
@pytest.mark.parametrize("model,plant,with_w,slew", EPISODES,
                         ids=[f"{a}_{b}{'_w' if c else ''}{'_slew' if d else ''}" for a, b, c, d in EPISODES])
def test_episode(model, plant, with_w, slew, B):
    """Episodes of 4 control steps, T = 8, with the model stepping, a slew-rate penalty, and a known plant with and
    without w, against known_oracle.episode (x, u, costs, info, u_next and the plans), and
    test_receding_plant_oracle_gpu.check_known_forward (the plant step plus w and the plans' rollouts)."""
    from tests import test_receding_plant_oracle_gpu as rp
    n = SYSTEMS[model][1]
    T, n_steps, dtype = 8, 4, F64
    c = rp.Case(n, 1, T, B, dtype, n_steps, "box", plant, with_w, slew, 900 + B + len(model) + 3 * slew,
                model=model)
    opts = dict(lqr_iter=3, eps=0.0, not_improved_lim=10 ** 6)
    r, _, _ = rp.device_call(c, opts=opts)
    tag = f"{c.form}{' w' if with_w else ''} B={B}"
    rp.check_known_forward(tag, c, r)
    o64 = ko.episode(n, 1, T, n_steps, c.P["x0"], c.P["C"], c.P["c"], c.mstep, c.theta, plant=c.oracle_plant(),
                     w=c.w, u_init=torch.zeros(T, B, 1, dtype=F64), slew_rate_penalty=rp.SLEW if slew else None,
                     prev_ctrl=c.prev, coupled=False, **c.kw, **opts)
    rr = dict(r, x=r["x"][..., 1:] if slew else r["x"])
    err, n_dep, n_cmp = check_episode_forward(tag, rr, o64, None, c.kw, dtype, True)
    DEPARTED.append((f"episode {tag}", n_dep, n_cmp, err))


@pytest.mark.parametrize("B", [1, 7, 300])
@pytest.mark.parametrize("name", ["cartpole", "pendulum"])
def test_window_episode(name, B):
    """A time-varying episode (episode_raw(..., window=L), mpcb200_episode_window_*) with a known model: C, c (a
    control push that changes with time) and tensor bounds on the episode's axis of L = n_steps + T - 1 slices, each
    control step solving on its window, against known_oracle.episode(window=True).  Every output and workspace starts
    as NaN.  check_episode_forward compares applied controls with each solve's bound at its t = 0, which for a window
    is slice k: the bounds it is handed are [1, n_steps, B, 1] so that its slice 0 holds them."""
    from mpc.pytorch_b200.step import episode_raw
    from tests.test_mlp_gpu import poisoned
    T, n_steps, dtype = 8, 4, F64
    L = n_steps + T - 1
    mod, p, clamp = module(name)
    n = SYSTEMS[name][1]
    g = torch.Generator().manual_seed(960 + B)
    q, pp = mod.get_true_obj()
    C = torch.diag(q.double()).expand(L, B, n + 1, n + 1).contiguous()
    c = pp.double().expand(L, B, n + 1).contiguous()
    c[..., n:] = 0.3 * clamp * (torch.rand(L, B, 1, generator=g, dtype=F64) - 0.5)
    x0 = known_states("cartpole" if name == "cartpole" else "pendulum", B, 960 + B)
    th = 2 * torch.rand(B, generator=g, dtype=F64) - 1
    ic = 2 if name == "cartpole" else 0
    x0[:, ic], x0[:, ic + 1] = th.cos(), th.sin()
    lo = -clamp * (0.3 + 1.2 * torch.rand(L, B, 1, generator=g, dtype=F64))
    hi = clamp * (0.3 + 1.2 * torch.rand(L, B, 1, generator=g, dtype=F64))
    opts = dict(lqr_iter=3, eps=0.0, not_improved_lim=10 ** 6, linesearch_decay=0.5, max_linesearch_iter=4)
    dyn = (SYSTEMS[name][0], mod.mpcb200_params())
    d = lambda t: t.to(DEV, dtype)  # noqa: E731
    with poisoned():
        r = episode_raw(n, 1, T, n_steps, d(x0), d(C), d(c), None, None, torch.zeros(T, B, 1, dtype=dtype, device=DEV),
                        u_lower=d(lo), u_upper=d(hi), dyn=dyn, keep_plans=True, window=L, **opts)
    assert r is not None, "the driver has no conditional graph nodes"
    torch.cuda.synchronize()
    o64 = ko.episode(n, 1, T, n_steps, x0, C, c, episode_known_step(module(name)[0]), p.expand(B, -1),
                     u_init=torch.zeros(T, B, 1, dtype=F64), u_lower=lo, u_upper=hi, window=True, coupled=False,
                     **opts)
    assert bool((o64.u.abs() >= torch.minimum(-lo[:n_steps], hi[:n_steps])).any()), "no applied control on a bound"
    kw = dict(u_lower=lo[:n_steps].unsqueeze(0), u_upper=hi[:n_steps].unsqueeze(0))
    err, n_dep, n_cmp = check_episode_forward(f"window {name} B={B}", r, o64, None, kw, dtype, True)
    DEPARTED.append((f"window {name} B={B}", n_dep, n_cmp, err))


# ------------------------------------------------------------------------------------------------------------------
# coverage (runs last)
# ------------------------------------------------------------------------------------------------------------------
def test_zz_known_loop_plan_coverage():
    if not SEEN:
        pytest.skip("no loop test of this module ran")
    missing = []
    for dtype in DTYPES:
        got = SEEN.get(dtype, set())
        for name, slew in KINDS:
            kind, n = SYSTEMS[name][:2]
            k = kind | (DYN_CTRL_PASSTHROUGH if slew else 0)
            Ts = gain_switch(k, n + slew, dtype)
            at_switch = Ts is not None and Ts <= ORACLE_TMAX and (dtype == F64 or name in F32_SWITCH_SYSTEMS)
            need = {"generic_smem"} | ({"generic_ks"} if at_switch else set())
            missing += [f"{DT[dtype]} {kind_name(name, slew)} {p}" for p in sorted(need - {p for kn, p in got
                                                                                          if kn == kind_name(name, slew)})]
            print(f"{DT[dtype]} {kind_name(name, slew)}: gain-store switch T* = {Ts}")
    worst = max((e for *_, e in DEPARTED), default=0.0)
    print(f"largest x/u error of the compared problems, relative to max(1, max|x|, max|u|): {worst:.3e}")
    print(f"problems departing from the oracle: {sum(a for _, a, _, _ in DEPARTED)} of "
          f"{sum(b for _, _, b, _ in DEPARTED)} compared, in {sum(a > 0 for _, a, _, _ in DEPARTED)} of "
          f"{len(DEPARTED)} runs:", [(t, a, b) for t, a, b, _ in DEPARTED if a])
    assert not missing, "plans never run inside the known-system loop: " + ", ".join(missing)
