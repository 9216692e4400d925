"""GPU: the line-search repeat passes of the linear-dynamics step kernels against the float64 oracle.

A step's rollout runs again, with alpha times decay, while any problem of the batch is worse than its nominal cost,
up to max_ls passes; a problem still worse after the last pass divides its alpha by decay once (reference
lqr_step.py:164-261).  Each kernel repeats a pass its own way: the generic kernel votes in a 32-slot ring in shared
memory and its producer warp re-streams every tile; the column-pair kernel decides per warp with __any_sync and
restarts the warp's own tile stream; the large-shape kernels acquire their 1 or 2 stages again.  du_first and
full_du_norm keep the values of the first pass.

The cases come from tests.gpu_harness.line_search_case: per batch position a chosen class (one pass; backtracked,
then better; worse on every pass), laid out by ls_layout so that every warp and CTA mixes them, and the first problem
of every warp and, in even CTAs of several warps, all of warp 0 take one pass.  tests/test_line_search_cpu.py checks
on the CPU that the cases below hold every class where it can exist.

Tolerances: float64 within 1e-9 x scale of the oracle with alphas, free sets, pnqp iteration counts and the controls
on a bound bit exact; float32 within 4x the error of the oracle itself run in float32 on the same float32-rounded
inputs plus 1e-6 x scale, with the float64 oracle's line-search decisions (near-ties and problems where the float32
oracle decides differently left out, at most one in eight)."""
import pytest
import torch

from oracle import lqr_oracle as orc
from tests.gpu_harness import (DT, F32, F64, MAX, ONE, check_alphas, check_clamps, check_pnqp, check_trajectory,
                               decays, f32_compared, line_search_case, ls_layout, plan as _plan,
                               plan_str as _plan_str, run_loop, run_step, same_on_both_loops, step_layout, switches,
                               to_dev)
from tests.helpers import maxdiff

pytestmark = pytest.mark.gpu


def _L():
    from mpc.pytorch_b200 import _lib
    return _lib


# (kernel, n, m, dtype, T, B, mode, max_ls, decay, MPCB200_KERNEL); kernel is the mapping that runs at the shape's
# instance (padded (3, 3) and (6, 1) run at (3, 4) and (6, 2)).  Odd B takes the generic kernel's copy path instead
# of the bulk loads (the column-pair kernel needs the bulk loads: 16-byte aligned spans).
LS_CASES = [
    ("generic", 5, 1, F64, 7, 23, "box", 10, 0.2, 1),
    ("generic", 5, 1, F32, 5, 40, "boxT", 40, 0.9, 1),
    ("generic", 8, 2, F64, 4, 12, "boxD", 10, 0.5, 1),
    ("generic", 8, 2, F32, 7, 21, "boxM", 40, 0.35, 1),
    ("generic", 8, 2, F32, 3, 24, "mask", 2, 0.9, 1),
    ("generic", 3, 4, F64, 5, 15, "plain", 10, 0.2, 1),
    ("generic", 16, 4, F64, 2, 7, "box", 3, 0.5, 1),
    ("pair", 4, 2, F64, 5, 23, "boxT", 10, 0.2, 2),
    ("pair", 4, 2, F32, 4, 30, "box", 40, 0.9, 2),
    ("pair", 8, 2, F32, 4, 12, "box", 10, 0.5, 2),
    ("pair", 8, 4, F64, 7, 13, "boxD", 3, 0.5, 2),
    ("pair", 8, 4, F32, 3, 10, "mask", 1, 0.2, 2),
    ("pair", 16, 4, F64, 5, 8, "plain", 10, 0.35, 2),
    ("pair", 16, 4, F32, 1, 9, "boxM", 2, 0.2, 2),
    ("large", 17, 1, F64, 5, 4, "box", 10, 0.5, None),
    ("large", 20, 4, F32, 7, 5, "boxT", 40, 0.9, None),
    ("large", 24, 8, F64, 3, 4, "boxD", 3, 0.2, None),
    ("large", 8, 2, F64, 7, 5, "mask", 10, 0.2, 3),
    ("generic", 3, 3, F64, 4, 9, "boxT", 10, 0.2, None),
    ("generic", 6, 1, F32, 5, 11, "plain", 10, 0.9, None),
    # the 4-stage ring of the column-pair kernel (Step2Cfg::S = 4 for tiles up to 6 KB) at every residue of T mod 4,
    # T < S included, where a repeat pass restarts fewer stages than the ring holds; the generic kernel at T = 1
    ("pair", 4, 2, F32, 1, 20, "boxM", 10, 0.5, 2),
    ("pair", 8, 4, F32, 2, 12, "box", 10, 0.2, 2),
    ("pair", 4, 2, F32, 5, 20, "boxT", 10, 0.9, 2),
    ("pair", 8, 4, F32, 6, 12, "boxD", 10, 0.5, 2),
    ("generic", 8, 2, F32, 1, 16, "boxM", 10, 0.2, 1),
]
INSTANCE_OF = {(3, 3): (3, 4), (6, 1): (6, 2)}


def case_id(c):
    kernel, n, m, dtype, T, B, mode, max_ls, decay, impl = c
    return f"{kernel}_n{n}m{m}_{DT[dtype]}_T{T}_B{B}_{mode}_ls{max_ls}_d{decay}" + (f"_k{impl}" if impl else "")


def build_case(kernel, n, m, dtype, T, B, mode, max_ls, decay, seed=0, K=None, shifted=False):
    """The line_search_case of one row of LS_CASES (K candidates: 192, or 96 for the large shapes)."""
    K = K or (96 if n > 16 else 192)
    ppw, W = step_layout(kernel, *INSTANCE_OF.get((n, m), (n, m)), dtype)
    return line_search_case(1000 + seed + 37 * n + 11 * m + T, T, n, m, dtype, mode, max_ls, decay,
                            ls_layout(B, ppw, W), K, shifted)


def _kernel_plan(kernel):
    return {"generic": _L().PLAN_GENERIC, "pair": _L().PLAN_PAIR, "large": _L().PLAN_LARGE}[kernel]


def check_ls_step(tag, r, case, dtype):
    """A step that backtracks against the oracle: alphas (float64 bit exact; float32 the same decisions), new_x,
    new_u, costs of the last pass, du_first and full_du_norm of the first, Ks, ks; float64 also free sets, pnqp
    iterations, status and the controls on a bound."""
    P, kw, o64, o32 = case.P, case.kw, case.o64, case.o32
    keep = None
    if dtype == F32:
        keep = f32_compared(case)
        out = int((~keep).sum())
        assert out <= max(1, len(keep) // 8), f"{tag}: {out} of {len(keep)} problems left out"
        d = kw["linesearch_decay"]
        assert torch.equal(decays(r["alphas"], d)[keep], decays(o64.alphas, d)[keep]), \
            f"{tag}: line-search decisions {r['alphas'].tolist()} vs {o64.alphas.tolist()}"
        check_alphas(tag, r, o64, o32, keep)
        assert int((r["status"] & ~1).max()) == 0, f"{tag}: status {r['status'].tolist()}"
    else:
        check_alphas(tag, r, o64, None)
        check_pnqp(tag, r, o64, kw)
        check_clamps(tag, r, o64, kw)
        assert not bool((r["status"] & 1).any()), f"{tag}: pnqp flagged unconverged"
    check_trajectory(tag, r, P["u"], o64, o32, dtype, keep, first=(case.first64, case.first32))


@pytest.mark.parametrize("c", LS_CASES, ids=[case_id(c) for c in LS_CASES])
def test_repeat_passes_match_oracle(c):
    kernel, n, m, dtype, T, B, mode, max_ls, decay, impl = c
    case = build_case(*c[:9])
    r, plan = run_step(n, m, T, case.P, case.kw, dtype, impl=impl, want_du_first=True)
    tag = case_id(c)
    assert plan & _kernel_plan(kernel), f"{tag}: plan {plan}"
    check_ls_step(tag, r, case, dtype)


# (kernel, n, m, dtype, T, B, mode, max_ls, decay, MPCB200_KERNEL)
SHIFT_CASES = [("generic", 5, 1, F64, 6, 23, "box", 10, 0.5, 1), ("generic", 8, 2, F32, 5, 16, "plain", 10, 0.2, 1),
               ("pair", 8, 4, F64, 5, 13, "boxT", 10, 0.2, 2), ("pair", 4, 2, F32, 3, 20, "mask", 3, 0.5, 2),
               ("large", 20, 4, F64, 4, 5, "boxD", 10, 0.35, None)]


@pytest.mark.parametrize("c", SHIFT_CASES, ids=[case_id(c) for c in SHIFT_CASES])
def test_nominal_from_a_shifted_initial_state(c):
    """current_x[0] != x_init: every kernel feeds back x_init - current_x[0] from t = 0, as the oracle does (the
    reference starts its rollout from dx = 0 instead; DESIGN.md section 4).  These nominals often stay worse on every
    pass."""
    kernel, n, m, dtype, T, B, mode, max_ls, decay, impl = c
    case = build_case(*c[:9], shifted=True)
    assert bool((case.P["x"][0] != case.P["x0"]).any(1).any()), "no nominal starts away from x_init"
    r, plan = run_step(n, m, T, case.P, case.kw, dtype, impl=impl, want_du_first=True)
    assert plan & _kernel_plan(kernel), f"{case_id(c)}: plan {plan}"
    check_ls_step(case_id(c) + " shifted", r, case, dtype)


# ------------------------------------------------------------------------------------------------------------------
# both sides of each gain-store switch (found on the device), and KREDUCE
# ------------------------------------------------------------------------------------------------------------------
# (kernel, n, m, dtype, mode, max_ls, decay, switch)
SWITCH_CASES = [("generic", 5, 1, F64, "box", 10, 0.5, "generic"), ("generic", 8, 2, F64, "mask", 40, 0.2, "generic"),
                ("generic", 16, 4, F64, "plain", 10, 0.9, "generic"), ("pair", 4, 2, F64, "boxD", 10, 0.35, "pair"),
                ("pair", 8, 4, F32, "plain", 2, 0.5, "pair"), ("pair", 16, 4, F64, "boxM", 10, 0.2, "pair")]


@pytest.mark.parametrize("c", SWITCH_CASES, ids=[f"{k}_n{n}m{m}_{DT[d]}_{md}" for k, n, m, d, md, *_ in SWITCH_CASES])
def test_repeat_passes_on_both_sides_of_the_gain_switch(c):
    """Gains in shared memory below the switch, in Ks/ks at it (generic (16, 4): KREDUCE at and above 12 steps in
    float64, where the gain store moves out of shared memory)."""
    kernel, n, m, dtype, mode, max_ls, decay, which = c
    Ts = switches(n, m, dtype)[which]
    assert Ts is not None and Ts <= 900, Ts
    impl = 1 if kernel == "generic" else 2
    B = 2 * step_layout(kernel, n, m, dtype)[1] + 1
    for T in (Ts - 1, Ts):
        if T < 1:
            continue
        case = build_case(kernel, n, m, dtype, T, B, mode, max_ls, decay, seed=T, K=48)
        r, plan = run_step(n, m, T, case.P, case.kw, dtype, impl=impl, want_gains=True, want_du_first=True)
        tag = f"{kernel} n{n}m{m} {DT[dtype]} T={T} (switch {Ts}) {mode}"
        kred = kernel == "generic" and (n, m) == (16, 4) and T >= Ts
        want = _plan(kernel == "generic", T < Ts, kred)
        assert plan == want, f"{tag}: plan {_plan_str(plan)}, expected {_plan_str(want)}"
        assert bool((case.classes != ONE).any()), f"{tag}: no problem backtracks"
        check_ls_step(tag, r, case, dtype)


def test_kreduce_repeat_passes():
    """Generic (16, 4) float32 past its KREDUCE horizon: lane i reads column i of K_t in every repeat pass."""
    n, m, T = 16, 4, 30
    case = build_case("generic", n, m, F32, T, 7, "boxT", 10, 0.5, K=64)
    r, plan = run_step(n, m, T, case.P, case.kw, F32, impl=1, want_du_first=True)
    assert plan == _plan(True, False, True), _plan_str(plan)
    check_ls_step("kreduce f32 T=30", r, case, F32)


def test_largest_shapes_one_stage():
    """The largest accepted (n, 4) per dtype, where only one tile stage fits shared memory (the two-stage layout
    needs a whole stage more than the one-stage layout of n + 1, which does not fit)."""
    from mpc.pytorch_b200.step import large_limit
    for dtype in (F64, F32):
        n = large_limit(4, 8 if dtype == F64 else 4)
        case = build_case("large", n, 4, dtype, 3, 3, "box", 10, 0.5, K=24)
        r, plan = run_step(n, 4, 3, case.P, case.kw, dtype, want_du_first=True)
        assert plan == _L().PLAN_LARGE
        check_ls_step(f"large n{n}m4 {DT[dtype]}", r, case, dtype)


# ------------------------------------------------------------------------------------------------------------------
# batch independence: passes forced by a neighbour change nothing
# ------------------------------------------------------------------------------------------------------------------
BITS = {F32: torch.int32, F64: torch.int64}
# (kernel, n, m, dtype, T, B, mode, max_ls, decay, MPCB200_KERNEL)
ALONE_CASES = [("generic", 8, 2, F32, 5, 19, "boxT", 10, 0.5, 1), ("pair", 8, 2, F64, 4, 13, "box", 40, 0.9, 2),
               ("pair", 16, 4, F32, 3, 7, "boxD", 10, 0.2, None), ("large", 20, 4, F64, 4, 5, "mask", 10, 0.35, None)]


@pytest.mark.parametrize("c", ALONE_CASES, ids=[case_id(c) for c in ALONE_CASES])
def test_outputs_equal_the_problem_solved_alone(c):
    kernel, n, m, dtype, T, B, mode, max_ls, decay, impl = c
    case = build_case(*c[:9])
    assert {ONE, MAX} <= set(case.classes.tolist()), case.classes
    r, plan = run_step(n, m, T, case.P, case.kw, dtype, impl=impl, want_gains=True, want_du_first=True)
    assert plan & _kernel_plan(kernel), f"{case_id(c)}: plan {plan}"
    for b in range(B):
        idx = torch.tensor([b])
        one = lambda v: v.index_select(0 if v.dim() == 2 and v.shape[0] == B else 1, idx) \
            if torch.is_tensor(v) else v  # noqa: E731
        a, plan1 = run_step(n, m, T, {k: one(v) for k, v in case.P.items()}, {k: one(v) for k, v in case.kw.items()},
                            dtype, impl=impl, want_gains=True, want_du_first=True)
        assert plan1 == plan, f"{case_id(c)}: problem {b} alone ran plan {plan1}, the batch {plan}"
        for k, v in a.items():
            got = r[k].index_select(0 if r[k].dim() == 1 else 1, idx)
            bits = (lambda t: t.view(BITS[t.dtype]) if t.is_floating_point() else t)
            assert torch.equal(bits(got), bits(v)), f"{case_id(c)}: {k} of problem {b} differs from it solved alone"


# ------------------------------------------------------------------------------------------------------------------
# the device iLQR loop with non-default line-search settings
# ------------------------------------------------------------------------------------------------------------------
# (n, m, T, B, mode, max_ls, decay)
LOOP_CASES = [(8, 2, 6, 24, "box", 4, 0.5), (4, 2, 5, 20, "boxT", 40, 0.9), (20, 4, 4, 5, "box", 3, 0.35)]


def loop_case(n, m, T, B, mode, max_ls, decay, seed=5):
    """An unstable bounded problem (F x 1.6, nominal from u = 0) and the float64 oracle's loop with its trace."""
    from tests.helpers import gen_problem
    C, c, F, f, x0 = gen_problem(seed + n, B, T, n, m, F64)
    F = F * 1.6
    g = torch.Generator().manual_seed(seed)
    kw = dict(u_lower=-0.1, u_upper=0.1)
    if mode == "boxT":
        kw = dict(u_lower=-0.05 - 0.2 * torch.rand(T, B, m, generator=g, dtype=F64),
                  u_upper=0.05 + 0.2 * torch.rand(T, B, m, generator=g, dtype=F64))
    P = dict(C=C, c=c, F=F, f=f, x0=x0, u0=torch.zeros(T, B, m, dtype=F64))
    opts = dict(lqr_iter=8, eps=1e-7, not_improved_lim=5, best_cost_eps=1e-4)
    trace = []
    x, u, costs, fdn = orc.mpc_forward_lin(n, m, T, x0, C, c, F, f, u_init=P["u0"], coupled=False, trace=trace,
                                           linesearch_decay=decay, max_linesearch_iter=max_ls, **kw, **opts)
    return P, kw, opts, dict(x=x, u=u, costs=costs, fdn=fdn, iters=len(trace), trace=trace)


@pytest.mark.parametrize("impl", [None, 1, 2, 3], ids=["default", "k1", "k2", "k3"])
@pytest.mark.parametrize("c", LOOP_CASES, ids=[f"n{c[0]}m{c[1]}_{c[4]}_ls{c[5]}_d{c[6]}" for c in LOOP_CASES])
def test_device_loop_with_line_search_settings(c, impl):
    n, m, T, B, mode, max_ls, decay = c
    if impl == 2 and (n % 2 or m % 2 or n + m > 32):
        pytest.skip("no column-pair mapping at this shape")
    if impl in (1, 2) and (n, m) == (20, 4):
        pytest.skip("no compiled instance at this shape")
    P, kw, opts, o = loop_case(*c)
    r, plan = run_loop(n, m, T, P, kw, dict(opts, linesearch_decay=decay, max_linesearch_iter=max_ls), F64, impl)
    tag = f"loop n{n}m{m} {mode} ls={max_ls} decay={decay} impl={impl}"
    if impl == 3 or (n, m) == (20, 4):
        assert plan == _L().PLAN_LARGE, f"{tag}: plan {plan}"
    elif impl in (1, 2):
        assert plan & _kernel_plan("generic" if impl == 1 else "pair"), f"{tag}: plan {plan}"
    sc = max(1.0, float(o["x"].abs().max()), float(o["u"].abs().max()))
    assert int(r["info"][0]) == o["iters"], f"{tag}: {int(r['info'][0])} iterations, the oracle ran {o['iters']}"
    for k in ("x", "u"):
        assert maxdiff(r[k], o[k]) <= 1e-9 * sc, f"{tag}: {k} differs by {maxdiff(r[k], o[k]):.3e}"
    assert maxdiff(r["costs"], o["costs"]) <= 1e-9 * max(1.0, float(o["costs"].abs().max())), f"{tag}: costs"
    assert maxdiff(r["full_du_norm"], o["fdn"]) <= 1e-6 * sc, f"{tag}: full_du_norm"


def test_mpc_forward_device_loop_equals_host_loop_at_40_passes(monkeypatch):
    from mpc.pytorch_b200 import MPC, LinDx, QuadCost
    n, m, T, B = 8, 2, 6, 24
    P, kw, _, o = loop_case(n, m, T, B, "box", 40, 0.5, seed=9)
    assert any(t["mean_alphas"] < 1 for t in o["trace"]), "the oracle's loop never backtracks"
    d = {k: to_dev(v) for k, v in P.items()}
    same_on_both_loops(monkeypatch, lambda: MPC(n, m, T, lqr_iter=8, verbose=-1, exit_unconverged=False,
                                                detach_unconverged=False, linesearch_decay=0.5,
                                                max_linesearch_iter=40, **kw),
                       d["x0"], QuadCost(d["C"], d["c"]), LinDx(d["F"], d["f"]))
