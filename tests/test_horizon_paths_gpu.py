"""Horizon-dependent kernel paths against the oracle.

Both step kernels change code path with the horizon T, chosen at launch from shared-memory arithmetic:
  * generic kernel: the gains K_t, k_t of all T steps stay in shared memory, or go through the caller's Ks/ks
    (too long for shared memory, or - for one-problem-per-warp shapes with n a power of two - the KREDUCE rollout,
    where lane i reads column i of K_t and K dx is summed by a butterfly);
  * column-pair kernel: the same choice, with the gains moved out early once the store is "crowded"; when the
    store does not fit and there is no buffer it refuses, and the default dispatch runs the generic kernel;
  * KKT adjoint: the fused pair kernel (2 launches) while d tau of all T steps fits shared memory and the masked
    step would keep its gains there, else the in-library masked step + costate + outer-product kernels (4 launches),
    whose masked step keeps its gains in the workspace where a step with Ks/ks would; LQRStepFn.backward is that one
    library call for every shape.
The switch horizons are found on the device by bisection (mpcb200_last_step_plan for step paths, launch counts for
adjoint routes), never hard-coded, and every comparison asserts the plan that ran, so a retuned constant cannot
silently drop a path: test_zz_coverage_table fails if any instance x dtype misses an applicable path.

Tolerances: float64 1e-9 x scale, active sets / clamp masks / pnqp iteration counts bit exact.  float32 over long
horizons: the kernel's error against the float64 oracle must stay within 4x the error of the oracle itself run in
float32 (on the same float32-rounded inputs) plus 1e-6 x scale.  Inputs come from tests.helpers.gen_problem with
F *= 0.9, so trajectories stay O(1) at T ~ 900."""
import ctypes

import pytest
import torch

from oracle import lqr_oracle as orc
from tests.gpu_harness import (DT, F32, F64, INSTANCES, KREDUCE_SHAPES, ORACLE_TMAX, PAIR_SHAPES, abi_grad,
                               adjoint_case, autograd_backward, check_adjoint, check_alphas, check_clamps, check_pnqp,
                               check_routes_agree, check_trajectory, kernel_env, linear_step_case, plan as _plan,
                               plan_str as _plan_str, run_abi_adjoint, run_step, switches, to_dev, within)
from tests.helpers import gen_problem, maxdiff

pytestmark = pytest.mark.gpu
COVERAGE = {}                       # (n, m, dtype) -> {what: set of plans / launch counts seen}


def _L():
    from mpc.pytorch_b200 import _lib
    return _lib


def _seen(n, m, dtype, what, value):
    COVERAGE.setdefault((n, m, dtype), {}).setdefault(what, set()).add(value)


def check_step(tag, r, case, dtype):
    P, kw, o64, o32 = case
    if "alphas" in r:
        check_alphas(tag, r, o64, o32)
    check_trajectory(tag, r, P["u"], o64, o32, dtype)
    check_pnqp(tag, r, o64, kw)
    check_clamps(tag, r, o64, kw)
    assert not bool((r["status"] & 1).any()), f"{tag}: pnqp flagged unconverged"


def _modes(dtype, k):
    """Mode rotation: float64 cases cycle through every mode; float32 cases (compared against the float32 oracle
    as yardstick, where a round-off-decided pnqp stop would make the yardstick meaningless) use the unbounded ones."""
    ms = ("box", "mask", "boxD", "plain") if dtype == F64 else ("mask", "plain")
    return ms[k % len(ms)]


def _B(n, m, dtype):
    """Two warps of problems plus a tail; odd (unaligned spans: no bulk TMA) for the float64 generic-only shapes."""
    if dtype == F64 and (n, m) not in PAIR_SHAPES:
        return 9
    ppw = 32 // ((n + m) // 2) if (n, m) in PAIR_SHAPES else max(1, 32 // (n + m))
    return ((2 * ppw + 2 + 3) // 4) * 4 if ppw < 8 else 12


PARAMS = [(n, m, d) for (n, m) in INSTANCES for d in (F64, F32)]
PIDS = [f"n{n}m{m}_{DT[d]}" for n, m, d in PARAMS]
PAIR_PARAMS = [p for p in PARAMS if p[:2] in PAIR_SHAPES]
PAIR_PIDS = [f"n{n}m{m}_{DT[d]}" for n, m, d in PAIR_PARAMS]


def test_instance_list_is_complete():
    assert sorted(_L().supported_pairs()) == sorted(INSTANCES)


# ------------------------------------------------------------------------------------------------------------------
# generic kernel: both sides of the gain-store switch (rollout and Riccati-only)
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,m,dtype", PARAMS, ids=PIDS)
def test_generic_gain_store_switch(n, m, dtype):
    sw = switches(n, m, dtype)
    kred = (n, m) in KREDUCE_SHAPES
    B = _B(n, m, dtype)
    for leg, Ts, rollout in (("rollout", sw["generic"], True), ("riccati", sw["generic_riccati"], False)):
        assert Ts is not None and Ts <= ORACLE_TMAX, (leg, Ts)
        for k, T in enumerate((Ts - 1, Ts)):
            if T < 1:
                continue
            mode = _modes(dtype, n + m + k)
            case = linear_step_case(100 + n * 10 + m, B, T, n, m, dtype, mode)
            r, plan = run_step(n, m, T, *case[:2], dtype, impl=1, do_rollout=rollout)
            want = _plan(True, T < Ts, kred and rollout and T >= Ts)
            tag = f"generic {leg} n{n}m{m} {DT[dtype]} T={T} B={B} {mode}"
            assert plan == want, f"{tag}: plan {_plan_str(plan)}, expected {_plan_str(want)}"
            _seen(n, m, dtype, f"generic_{leg}", plan)
            check_step(tag, r, case, dtype)


KREDUCE_CASES = [(F64, "plain"), (F64, "box"), (F64, "mask"), (F32, "plain"), (F32, "mask")]


@pytest.mark.parametrize("dtype,mode", KREDUCE_CASES, ids=[f"{DT[d]}_{md}" for d, md in KREDUCE_CASES])
def test_generic_kreduce_long_horizon(dtype, mode):
    """KREDUCE at T=300: every row of Ks / ks and the rollout against the oracle."""
    n, m, T, B = 16, 4, 300, 5
    case = linear_step_case(400, B, T, n, m, dtype, mode)
    r, plan = run_step(n, m, T, *case[:2], dtype, impl=1)
    assert plan == _plan(True, False, True), _plan_str(plan)
    _seen(n, m, dtype, "generic_rollout", plan)
    check_step(f"kreduce {DT[dtype]} T={T} {mode}", r, case, dtype)


def _long_default(n, m, T, dtype, mode, B, kernel):
    """Default dispatch far past every gain-store switch: the gains round-trip through the caller's Ks/ks."""
    case = linear_step_case(40, B, T, n, m, dtype, mode)
    r, plan = run_step(n, m, T, *case[:2], dtype)
    assert plan == _plan(kernel == "generic", False), _plan_str(plan)
    check_step(f"long default n{n}m{m} {DT[dtype]} T={T} {mode}", r, case, dtype)


def test_gains_spill_to_global_for_long_horizons():
    """(8,2) float64, T=700, scalar bounds, default dispatch: too long for the shared-memory gain store, so the
    generic kernel round-trips K, k through the caller's buffer (the plan says so), and matches the oracle."""
    _long_default(8, 2, 700, F64, "box", 20, "generic")


# (n, m, T, dtype, mode, B, kernel the default dispatch picks)
LONG_DEFAULT = [(8, 4, 700, F32, "mask", 12, "pair"), (2, 2, 700, F64, "boxD", 12, "pair")]


@pytest.mark.parametrize("n,m,T,dtype,mode,B,kernel", LONG_DEFAULT,
                         ids=["n8m4_T700_f32_mask", "n2m2_T700_f64_boxT"])
def test_long_horizon_default_dispatch(n, m, T, dtype, mode, B, kernel):
    """Default dispatch far past every gain-store switch on pair-kernel shapes."""
    _long_default(n, m, T, dtype, mode, B, kernel)


# ------------------------------------------------------------------------------------------------------------------
# column-pair kernel
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,m,dtype", PAIR_PARAMS, ids=PAIR_PIDS)
def test_pair_crowded_switch(n, m, dtype):
    """At the crowded switch: the same inputs with the gains in Ks/ks (want_gains) and in shared memory."""
    sw = switches(n, m, dtype)
    Ts = sw["pair"]
    assert Ts is not None and Ts < sw["pair_nofit"]
    B = _B(n, m, dtype)
    for k, T in enumerate((Ts - 1, Ts)):
        if T < 1:
            continue
        mode = _modes(dtype, n + m + k + 1)
        case = linear_step_case(200 + n * 10 + m, B, T, n, m, dtype, mode)
        tag = f"pair crowded n{n}m{m} {DT[dtype]} T={T} B={B} {mode}"
        r1, p1 = run_step(n, m, T, *case[:2], dtype, impl=2, want_gains=True)
        assert p1 == _plan(False, T < Ts), f"{tag}: plan {_plan_str(p1)}"
        check_step(tag + " want_gains", r1, case, dtype)
        # without a buffer below the generic kernel's switch the gains stay in shared memory
        r0, p0 = run_step(n, m, T, *case[:2], dtype, impl=2, want_gains=False)
        ws = sw["generic"] is not None and T >= sw["generic"]         # lqr_step_raw passes Ks/ks anyway
        assert p0 == _plan(False, not (ws and T >= Ts)), f"{tag}: plan {_plan_str(p0)}"
        _seen(n, m, dtype, "pair_rollout", p1)
        _seen(n, m, dtype, "pair_rollout", p0)
        sc = max(1.0, float(r1["new_x"].abs().max()), float(r1["new_u"].abs().max()))
        d = max(maxdiff(r0[k2], r1[k2]) for k2 in ("new_x", "new_u", "costs"))
        _seen(n, m, dtype, "pair smem vs Ks bit-identical", d == 0.0)
        assert d <= (1e-12 if dtype == F64 else 1e-6) * sc, f"{tag}: smem vs Ks gains differ by {d:.3e}"
        check_step(tag + " gains in smem", r0, case, dtype)


@pytest.mark.parametrize("n,m,dtype", PAIR_PARAMS, ids=PAIR_PIDS)
def test_pair_long_horizon_and_no_fit(n, m, dtype):
    """Just below the pair kernel's shared-memory limit with the gains in Ks/ks; at the limit without a buffer the
    default dispatch falls back to the generic kernel and a forced pair kernel refuses; Riccati-only on both sides."""
    from mpc.pytorch_b200.step import lqr_step_raw
    sw = switches(n, m, dtype)
    Tn = sw["pair_nofit"]
    assert Tn is not None and Tn <= ORACLE_TMAX
    B = _B(n, m, dtype)
    seed = 300 + n * 10 + m
    mode = _modes(dtype, n + m + 2)
    below = linear_step_case(seed, B, Tn - 1, n, m, dtype, mode)
    tag = f"pair long n{n}m{m} {DT[dtype]} T={Tn - 1} B={B} {mode}"
    r, plan = run_step(n, m, Tn - 1, *below[:2], dtype, impl=2, want_gains=True)
    assert plan == _plan(False, False), f"{tag}: plan {_plan_str(plan)}"
    _seen(n, m, dtype, "pair_rollout", plan)
    check_step(tag, r, below, dtype)
    r, plan = run_step(n, m, Tn - 1, *below[:2], dtype, impl=2, do_rollout=False)
    assert plan == _plan(False, True), f"{tag} riccati: plan {_plan_str(plan)}"
    _seen(n, m, dtype, "pair_riccati", plan)
    check_step(tag + " riccati", r, below, dtype)

    at = linear_step_case(seed, B, Tn, n, m, dtype, mode)
    tag = f"pair no-fit n{n}m{m} {DT[dtype]} T={Tn} B={B} {mode}"
    r, plan = run_step(n, m, Tn, *at[:2], dtype, impl=2, do_rollout=False)
    assert plan == _plan(False, False), f"{tag} riccati: plan {_plan_str(plan)}"
    _seen(n, m, dtype, "pair_riccati", plan)
    check_step(tag + " riccati", r, at, dtype)
    if sw["generic"] is not None and Tn >= sw["generic"]:
        return          # lqr_step_raw passes Ks/ks at this horizon: no bufferless call to fall back from
    r, plan = run_step(n, m, Tn, *at[:2], dtype, impl=None, want_gains=False)
    assert plan == _plan(True, True), f"{tag} fallback: plan {_plan_str(plan)}"
    _seen(n, m, dtype, "pair_fallback", plan)
    check_step(tag + " fallback", r, at, dtype)
    P = {k: to_dev(v, dtype) for k, v in at[0].items()}
    kw = {k: to_dev(v, dtype) for k, v in at[1].items()}
    with kernel_env(2), pytest.raises(_L().MpcB200Error, match=r"\[4\]"):
        lqr_step_raw(n, m, Tn, P["x0"], P["C"], P["c"], P["F"], P["f"], P["x"], P["u"], **kw)
    assert _L().last_step_plan() == 0
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------------------
# KKT adjoint routes
# ------------------------------------------------------------------------------------------------------------------
ADJ_BOUNDS = (None, "box", "tensor")


def _prefers_workspace(n, m, T, dtype):
    from mpc.pytorch_b200._lib import Dims
    d = Dims(B=1, T=T, n=n, m=m, F_T=T - 1)
    return bool(_L().lib().mpcb200_step_prefers_workspace(ctypes.byref(d), dtype.itemsize))


def _adjoint_switch(n, m, dtype, check_plan):
    """Fused just below the adjoint's switch horizon, in-library 3-launch route at it, both against the oracle's
    adjoint; check_plan(tag, T, launches, plan) checks the nested step's plan."""
    Ta = switches(n, m, dtype)["adjoint"]
    assert Ta is not None and Ta <= ORACLE_TMAX
    B = _B(n, m, dtype)
    for k, T in enumerate((Ta - 1, Ta)):
        bounds = ADJ_BOUNDS[(n + m + k) % 3]
        with_f = (n + k) % 3 != 0
        case = adjoint_case(600 + n * 10 + m, B, T, n, m, dtype, bounds, with_f)
        got, launches = run_abi_adjoint(n, m, T, case, dtype)
        tag = f"adjoint n{n}m{m} {DT[dtype]} T={T} B={B} bounds={bounds} f={with_f}"
        assert launches == (2 if T < Ta else 4), f"{tag}: {launches} launches"
        check_plan(tag, T, launches, _L().last_step_plan())
        _seen(n, m, dtype, "adjoint_launches", launches)
        check_adjoint(tag, got, case, dtype)


# the KREDUCE shape's adjoint switches at the horizon where its masked step starts to keep the gains in Ks/ks
SWITCH_PARAMS = [p for p in PAIR_PARAMS if p[:2] not in KREDUCE_SHAPES]
SWITCH_PIDS = [f"n{n}m{m}_{DT[d]}" for n, m, d in SWITCH_PARAMS]
KREDUCE_PARAMS = [p for p in PAIR_PARAMS if p[:2] in KREDUCE_SHAPES]
KREDUCE_PIDS = [f"n{n}m{m}_{DT[d]}" for n, m, d in KREDUCE_PARAMS]


@pytest.mark.parametrize("n,m,dtype", SWITCH_PARAMS, ids=SWITCH_PIDS)
def test_adjoint_fused_to_three_launch_switch(n, m, dtype):
    """Fused just below the fit limit, in-library 3-launch route at it, both against the oracle's adjoint."""
    def check_plan(tag, T, launches, plan):
        # the nested masked step (fused or not) keeps its gains in shared memory: it has no Ks/ks buffer
        assert plan & _L().PLAN_GAINS_SMEM, f"{tag}: {_plan_str(plan)}"
    _adjoint_switch(n, m, dtype, check_plan)


@pytest.mark.parametrize("n,m,dtype", KREDUCE_PARAMS, ids=KREDUCE_PIDS)
def test_adjoint_switch_moves_gains_to_workspace(n, m, dtype):
    """(16,4): the adjoint leaves the fused kernel where its masked step starts to prefer Ks/ks (the KREDUCE switch),
    although the fused kernel would fit; there the 3-launch route's masked step keeps its gains in the workspace.
    Both sides against the oracle's adjoint."""
    def check_plan(tag, T, launches, plan):
        gains_ws = _prefers_workspace(n, m, T, dtype)
        assert gains_ws == (launches == 4), f"{tag}: prefers Ks/ks {gains_ws}, {launches} launches"
        assert bool(plan & _L().PLAN_GAINS_SMEM) != gains_ws, f"{tag}: {_plan_str(plan)}, Ks/ks given: {gains_ws}"
    _adjoint_switch(n, m, dtype, check_plan)


ROUTE_SHAPES = [(2, 2), (4, 2), (8, 2), (8, 4), (12, 4), (16, 4), (5, 1), (3, 4)]


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("n,m", ROUTE_SHAPES, ids=[f"n{n}m{m}" for n, m in ROUTE_SHAPES])
def test_adjoint_routes_agree_at_short_horizon(n, m, dtype):
    """One input per shape: fused route (default) and in-library 3-launch route (generic kernel forced) agree with
    each other and with the oracle."""
    T, B = 9, _B(n, m, dtype)
    bounds = ADJ_BOUNDS[(n + m) % 3]
    with_f = n % 2 == 0
    case = adjoint_case(700 + n * 10 + m, B, T, n, m, dtype, bounds, with_f)
    tag = f"routes n{n}m{m} {DT[dtype]} T={T} bounds={bounds} f={with_f}"
    g3, l3 = run_abi_adjoint(n, m, T, case, dtype, impl=1)
    assert l3 == 4, f"{tag}: {l3} launches"
    check_adjoint(tag + " 3-launch", g3, case, dtype)
    _seen(n, m, dtype, "adjoint_launches", l3)
    if (n, m) in PAIR_SHAPES:
        g2, l2 = run_abi_adjoint(n, m, T, case, dtype)
        assert l2 == 2, f"{tag}: {l2} launches"
        check_adjoint(tag + " fused", g2, case, dtype)
        _seen(n, m, dtype, "adjoint_launches", l2)
        check_routes_agree(tag + " fused vs 3-launch", g2, g3, case, dtype)


@pytest.mark.parametrize("dtype", [F32, F64], ids=["f32", "f64"])
def test_config5_backward_takes_three_launch_route(dtype):
    """(16,4) T=50 (config 5), past the generic kernel's KREDUCE switch: LQRStepFn.backward is the one library call,
    which takes the 3-launch route with the masked step's gains in the workspace (faster there than the fused kernel,
    which would fit this horizon); it agrees with the route the generic kernel gives."""
    n, m, T, B = 16, 4, 50, 5
    case = adjoint_case(800, B, T, n, m, dtype, "box", True)
    tag = f"config5 backward {DT[dtype]}"
    got, launches = autograd_backward(n, m, T, *case[:2], dtype)
    # (the step plan is per host thread, and autograd runs this backward on its own device thread)
    assert launches == 4, f"{tag}: {launches} launches, not the 3-launch route"
    _seen(n, m, dtype, "adjoint_launches", 4)
    check_adjoint(tag + " autograd", got, case, dtype)
    three, l3 = run_abi_adjoint(n, m, T, case, dtype, impl=1)
    assert l3 == 4, l3
    check_adjoint(tag + " 3-launch", three, case, dtype)
    check_routes_agree(tag + " default vs generic 3-launch", got, three, case, dtype)


# (n, m, T, dtype, B, launches of the one library call): a padded shape that runs fused ((6,1) -> (6,2)), and two
# horizons whose nested step keeps its gains in the workspace: past the gain store's size, and config 5 in float32
BACKWARD_CASES = [(6, 1, 9, F64, 7, 2), (8, 2, 700, F64, 6, 4), (16, 4, 50, F32, 5, 4)]


@pytest.mark.parametrize("n,m,T,dtype,B,launches", BACKWARD_CASES,
                         ids=[f"n{n}m{m}_T{T}_{DT[d]}" for n, m, T, d, _, _ in BACKWARD_CASES])
def test_backward_is_one_library_call(n, m, T, dtype, B, launches):
    """LQRStepFn.backward against the oracle's adjoint, as one mpcb200_lqr_adjoint_* call of the expected launch
    count; the same call made on this thread (lqr_adjoint_raw) gives the same gradients and shows the nested step's
    gain store."""
    from mpc.pytorch_b200.step import lqr_adjoint_raw
    case = adjoint_case(1000 + n * 10 + m + T, B, T, n, m, dtype, "box", True)
    P, kw = case[:2]
    tag = f"backward n{n}m{m} T={T} {DT[dtype]}"
    got, l_auto = autograd_backward(n, m, T, P, kw, dtype)
    assert l_auto == launches, f"{tag}: {l_auto} launches"
    check_adjoint(tag, got, case, dtype)
    d = lambda t: to_dev(t, dtype)  # noqa: E731
    raw = lqr_adjoint_raw(n, m, T, d(P["C"]), d(P["c"]), d(P["F"]), d(P["x"]), d(P["u"]), d(P["wx"]), d(P["wu"]),
                          kw["u_lower"], kw["u_upper"], True)
    plan = _L().last_step_plan()
    torch.cuda.synchronize()
    for i, name in enumerate(("dx_init", "dC", "dc", "dF", "df")):
        assert torch.equal(raw[i].cpu(), got[i]), f"{tag}: {name} autograd vs lqr_adjoint_raw"
    if launches == 4:
        assert _prefers_workspace(n, m, T, dtype) and not plan & _L().PLAN_GAINS_SMEM, f"{tag}: {_plan_str(plan)}"


@pytest.mark.parametrize("with_F", [False, True], ids=["F_none", "F_given"])
def test_backward_single_step(with_F):
    """T = 1 with F = None (the forward pass takes it, so the backward must: no dF) and with F given (T slices, whose
    dF slice is zero): LQRStepFn.backward against the oracle's adjoint, one fused library call."""
    n, m, T, B, dtype = 8, 2, 1, 6, F64
    C, c, F, _, x0 = gen_problem(1100, B, 2, n, m, F64)
    g = torch.Generator().manual_seed(1100)
    x, u = torch.randn(T, B, n, generator=g, dtype=F64), 0.1 * torch.randn(T, B, m, generator=g, dtype=F64)
    P = dict(x0=x0, C=C[:1], c=c[:1], F=F[:1], x=x, u=u, wx=torch.randn(T, B, n, generator=g, dtype=F64),
             wu=torch.randn(T, B, m, generator=g, dtype=F64))
    F_orc = P["F"] if with_F else torch.zeros(0, B, n, n + m, dtype=F64)
    ref = orc.lqr_step_backward(n, m, T, x0, P["C"], P["c"], F_orc, None, x, u, P["wx"], P["wu"], coupled=False)
    got, launches = autograd_backward(n, m, T, P, {}, dtype, keys=("x0", "C", "c", "F") if with_F else
                                       ("x0", "C", "c"))
    assert launches == 2, launches
    for i, name in enumerate(("dx_init", "dC", "dc", "dF")):
        if name == "dF" and not with_F:
            continue
        within("T=1", name, got[i], ref[i], None, dtype)


# ------------------------------------------------------------------------------------------------------------------
# mpcb200_lqr_grad_* (the costate workspace is required)
# ------------------------------------------------------------------------------------------------------------------
GRAD_CASES = [(8, 2, 9, F64), (8, 2, 300, F64), (5, 1, 9, F64), (5, 1, 300, F32), (16, 4, 12, F32), (16, 4, 250, F64)]


@pytest.mark.parametrize("n,m,T,dtype", GRAD_CASES, ids=[f"n{n}m{m}_T{T}_{DT[d]}" for n, m, T, d in GRAD_CASES])
def test_grad_two_kernels_match_oracle(n, m, T, dtype):
    """The two gradient kernels (costates through the workspace, then the outer products), fed the costate inputs of
    a solved problem (the oracle's adjoint solution dx, du), against the oracle's outer products."""
    case = adjoint_case(900 + n + T, 12, T, n, m, dtype, "box", True)
    P, _, ref64, ref32 = case
    dx, du = ref64[5], ref64[6]
    d = lambda t: to_dev(t, dtype)  # noqa: E731
    two, launches = abi_grad(n, m, T, *[d(P[k]) for k in ("C", "c", "F", "x", "u")], d(dx), d(du), d(P["wx"]))
    assert launches == 2, launches
    tag = f"grad n{n}m{m} T={T} {DT[dtype]}"
    for i, name in enumerate(("dx_init", "dC", "dc", "dF", "df")):
        # float32: the kernel is fed float32-rounded dx, du, so the yardstick is the float32 oracle's own adjoint
        within(f"{tag} two kernels", name, two[i], ref64[i], ref32[i] if ref32 is not None else None, dtype)


# ------------------------------------------------------------------------------------------------------------------
# coverage: every instance x dtype reached every applicable path (runs last)
# ------------------------------------------------------------------------------------------------------------------
def test_zz_coverage_table():
    if not COVERAGE:
        pytest.skip("no path test of this module ran")
    rows, missing = [], []
    for n, m, dtype in PARAMS:
        cov = COVERAGE.get((n, m, dtype), {})
        sw = switches(n, m, dtype)
        need = {"generic_rollout": {_plan(True, True), _plan(True, False, (n, m) in KREDUCE_SHAPES)},
                "generic_riccati": {_plan(True, True), _plan(True, False)}}
        if (n, m) in PAIR_SHAPES:
            need["pair_rollout"] = {_plan(False, False), _plan(False, True)}
            need["pair_riccati"] = {_plan(False, True), _plan(False, False)}
            need["adjoint_launches"] = {2, 4}
            if sw["generic"] is None or sw["pair_nofit"] < sw["generic"]:
                need["pair_fallback"] = {_plan(True, True)}
        for k, v in need.items():
            if not v <= cov.get(k, set()):
                missing.append(f"n{n}m{m} {DT[dtype]} {k}: missing {sorted(v - cov.get(k, set()))}")
        fmt = lambda k: ", ".join(sorted(str(p) if k == "adjoint_launches" else _plan_str(p)
                                         for p in cov.get(k, ()))) or "-"
        rows.append(f"| ({n},{m}) {DT[dtype]} | {sw['generic']} | {sw['generic_riccati']} | {sw['pair']} | "
                    f"{sw['pair_nofit']} | {sw['adjoint']} | {fmt('generic_rollout')} | {fmt('pair_rollout')} | "
                    f"{fmt('pair_fallback')} | {fmt('adjoint_launches')} |")
    print("\n| instance | T* generic | T* generic Riccati-only | T* pair (Ks) | T* pair no-fit | T* adjoint 3-launch "
          "| generic plans | pair plans | pair fallback | adjoint launches |\n|" + "---|" * 10)
    print("\n".join(rows))
    ident = {k: v for k, v in COVERAGE.items() if "pair smem vs Ks bit-identical" in v}
    print("pair kernel, gains in smem vs Ks bit-identical:",
          {f"n{n}m{m}_{DT[d]}": sorted(v["pair smem vs Ks bit-identical"]) for (n, m, d), v in ident.items()})
    assert not missing, "\n".join(missing)
