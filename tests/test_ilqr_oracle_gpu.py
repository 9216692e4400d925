"""GPU: the device-side iLQR loop of MPC.forward (mpcb200_ilqr_*, csrc/ilqr.cuh) against the float64 oracle's loop
(orc.mpc_forward_lin with per-problem pnqp): x, u, costs, the best iterate's full_du_norm and the iteration count.

  * every step plan the loop body can record (generic kernel with gains in shared memory / in the Ks/ks workspace /
    KREDUCE, pair kernel with gains in shared memory / in the workspace, the pair kernel's fallback to the generic
    kernel, the large-shape kernels), on both sides of each switch horizon, which is bisected on the device with the
    probes of tests/test_horizon_paths_gpu.py and never hard-coded; test_zz_loop_plan_coverage fails if a plan that
    exists was never run inside the loop;
  * full-size batches (config 3, config 4, the config-5 shard), where the bookkeeping kernels' grid-stride loops take
    several passes, and the device loop against the host loop at B=65536;
  * the three stop reasons at B > 256, and the full_du_norm that decides MPC.forward's exit_unconverged assert and
    which problems detach_unconverged detaches;
  * u_zero_I, alone and with a tensor box, at an exact and at a zero-padded control dimension.

Tolerances, per problem.  float64: x and u within 1e-9 x scale, costs within 1e-9 relative, the controls sitting on
a bound bit for bit, the iteration count equal to the oracle's.  float32: x and u within 4x the largest error of the
oracle itself run in float32 on the same float32-rounded inputs, plus 1e-6 x scale, and the iteration count equal to
the float32 oracle's; problems where the float32 oracle leaves the float64 one (other bound sets, or x, u off by more
than 1e-4 x scale) are left out.  In bounded loops of more than one iteration at most one problem in four may miss
these bounds (check_loop says why: round-off decides some problems' pnqp paths, the oracle's own loop included).
float32 cases stop at eps = 1e-4, above the float32 round-off of a converged iterate's norm (~1e-6), so that no stop
decision is made by round-off.  full_du_norm, on the rows of the batch-mixing norm that hold no left-out problem:
float64 within 1e-6 relative plus 1e-12 x scale (a converged iterate's norm is round-off, ~1e-15), float32 within 4x
the float32 oracle's error plus 1e-6 x scale; test_zz_loop_plan_coverage prints the largest errors observed."""
import functools
import math

import pytest
import torch

from oracle import lqr_oracle as orc
from tests.gpu_harness import (DEV, DT, F32, F64, ORACLE_TMAX, SWITCH_PLANS, loop_plan, pick_switch, plan as _plan,
                               plan_name as _plan_name, plan_str as _plan_str, round_through, run_loop,
                               same_on_both_loops, within)
from tests.helpers import gen_problem, maxdiff

pytestmark = pytest.mark.gpu
EPS = {F64: 1e-7, F32: 1e-4}        # the stop tolerance of each dtype's cases (MPC's default in float64)
FDN_ERR = {}                        # (dtype, what) -> observed |full_du_norm - oracle| (or device - host), per run
LOOP_SEEN = {}                      # dtype -> step plans run inside the loop
DEPARTED = {}                       # dtype -> [(problems departing from the oracle, problems compared)]


def _L():
    from mpc.pytorch_b200 import _lib
    return _lib


# ------------------------------------------------------------------------------------------------------------------
# problems, the oracle's loop, the device loop
# ------------------------------------------------------------------------------------------------------------------
def _f32(t):
    return t.float() if torch.is_tensor(t) and t.is_floating_point() else t


def _oracle(n, m, T, P, kw, opts):
    trace = []
    x, u, costs, fdn = orc.mpc_forward_lin(n, m, T, P["x0"], P["C"], P["c"], P["F"], P["f"], u_init=P["u0"],
                                           coupled=False, trace=trace, **kw, **opts)
    return dict(x=x, u=u, costs=costs, fdn=fdn, iters=len(trace), trace=trace)


@functools.lru_cache(maxsize=2)
def loop_case(seed, B, T, n, m, dtype, mode, lqr_iter, eps, not_improved_lim=5, best_cost_eps=1e-4):
    """Inputs (float64, rounded through dtype), options and the oracle's loop: (P, kw, opts, o64, o32|None).
    mode: plain | box (+-0.25) | tensor (tensor box) | boxT (tensor box + delta_u) | mask (u_zero_I) |
    maskT (u_zero_I + tensor box)."""
    C, c, F, f, x0 = gen_problem(seed, B, T, n, m, F64)
    F = F * 0.9                     # trajectories stay O(1) over long horizons
    g = torch.Generator().manual_seed(seed + 1)
    kw = {}
    if mode == "box":
        kw = dict(u_lower=-0.25, u_upper=0.25)
    if mode in ("tensor", "boxT", "maskT"):
        kw = dict(u_lower=-0.5 * torch.rand(T, B, m, generator=g, dtype=F64) - 0.05,
                  u_upper=0.5 * torch.rand(T, B, m, generator=g, dtype=F64) + 0.05)
    if mode == "boxT":
        kw["delta_u"] = 0.125
    if mode in ("mask", "maskT"):
        kw["u_zero_I"] = torch.rand(T, B, m, generator=g) < 0.3
    P = {k: round_through(v, dtype) for k, v in dict(C=C, c=c, F=F, f=f, x0=x0).items()}
    P["u0"] = torch.zeros(T, B, m, dtype=F64)
    kw = {k: round_through(v, dtype) for k, v in kw.items()}
    opts = dict(lqr_iter=lqr_iter, eps=eps, not_improved_lim=not_improved_lim, best_cost_eps=best_cost_eps)
    o64 = _oracle(n, m, T, P, kw, opts)
    o32 = None
    if dtype == F32:
        o32 = _oracle(n, m, T, {k: _f32(v) for k, v in P.items()}, {k: _f32(v) for k, v in kw.items()}, opts)
    return P, kw, opts, o64, o32


# ------------------------------------------------------------------------------------------------------------------
# comparisons
# ------------------------------------------------------------------------------------------------------------------
def _on_bounds(u, kw):
    """[2, T, B, m]: which controls sit on the lower / upper bound."""
    lo, hi = (kw[k] if torch.is_tensor(kw[k]) else torch.full_like(u, kw[k]) for k in ("u_lower", "u_upper"))
    return torch.stack((u.double() == lo.double(), u.double() == hi.double()))


def _same_per_problem(a, b):
    return (a == b).all(3).all(1).all(0)


def _err_per_problem(a, b):
    """max |a - b| over x or u of each problem ([T, B, k] -> [B])."""
    return (a.double() - b.double()).abs().amax((0, 2))


def rows_holding(problems, T, m):
    """The rows of the batch-mixing full_du_norm (du [T,m,B] viewed as [B, T*m]) that hold an element of these
    problems' du: problem bb at (t, j) is flat element (t*m + j)*B + bb."""
    B = problems.shape[0]
    rows = torch.zeros(B, dtype=torch.bool)
    tj = torch.arange(T * m)
    for bb in problems.nonzero()[:, 0].tolist():
        rows[(tj * B + bb) // (T * m)] = True
    return rows


def check_fdn(tag, got, w64, w32, dtype, scale):
    """The best iterate's full_du_norm (the reference's batch-mixing norm) against the oracle's."""
    err = (got.double() - w64).abs()
    FDN_ERR.setdefault((dtype, "abs"), []).append(float(err.max()))
    if dtype == F64:
        bad = err > 1e-6 * w64.abs() + 1e-12 * scale
        assert not bool(bad.any()), (f"{tag}: full_du_norm differs in {int(bad.sum())} problems, e.g. kernel "
                                     f"{float(got[bad][0]):.6e} oracle {float(w64[bad][0]):.6e}")
    else:
        bound = 4 * maxdiff(w32, w64) + 1e-6 * max(1.0, float(w64.abs().max()))
        assert float(err.max()) <= bound, f"{tag}: full_du_norm |kernel - oracle| = {float(err.max()):.3e} > {bound:.3e}"


def check_loop(tag, r, case, dtype):
    """x, u, costs, full_du_norm, controls on a bound and the iteration count of one device loop against the oracle.

    A problem "departs" where its x or u misses the tolerance or its controls on a bound differ from the oracle's.
    Only bounded loops of more than one iteration may have departing problems, at most one in four: there pnqp's
    |dx| >= 1e-4 stop, its iteration cap and its Armijo test on nearly cancelling differences decide some problems'
    paths by round-off, so a perturbation of C at float64 round-off (1e-15 relative) moves the oracle's own loop too
    (2 of 8 problems by 3.3e-5 in x at (16,4) T=11 +-0.25, 25 of 300 by up to 2e-7 at (8,2) T=10 +-0.25), and the host
    loop departs exactly where the device loop does.  float32 problems where the float32 oracle itself departs from
    the float64 one (x or u off by more than 1e-4 x scale, or other bound sets) are left out.  full_du_norm is
    compared on the rows that hold no left-out or departing problem's du."""
    P, kw, opts, o64, o32 = case
    T, B, m = o64["u"].shape
    bounded = "u_lower" in kw
    sc = max(1.0, float(o64["x"].abs().max()), float(o64["u"].abs().max()))
    err_k = torch.maximum(_err_per_problem(r["x"], o64["x"]), _err_per_problem(r["u"], o64["u"]))
    out = torch.zeros(B, dtype=torch.bool)                  # left out: the float32 yardstick itself departs
    if o32 is None:
        tol = 1e-9 * sc
    else:
        err_32 = torch.maximum(_err_per_problem(o32["x"], o64["x"]), _err_per_problem(o32["u"], o64["u"]))
        out = err_32 > 1e-4 * sc
        if bounded:
            out |= ~_same_per_problem(_on_bounds(o32["u"], kw), _on_bounds(o64["u"], kw))
        assert not bool(out.all()), f"{tag}: no comparable problem"
        tol = 4 * float(err_32[~out].max()) + 1e-6 * sc
    dep = err_k > tol
    if bounded:
        dep |= ~_same_per_problem(_on_bounds(r["u"], kw), _on_bounds(o64["u"], kw))
    dep &= ~out
    n_dep, n_cmp = int(dep.sum()), int((~out).sum())
    DEPARTED.setdefault(dtype, []).append((n_dep, n_cmp))
    allowed = max(1, n_cmp // 4) if bounded and o64["iters"] > 1 else 0
    assert n_dep <= allowed, (f"{tag}: {n_dep} of {n_cmp} problems depart from the oracle (allowed {allowed}), "
                              f"largest x/u error {float(err_k[~out].max()):.3e}, tolerance {tol:.3e}")
    keep = ~(out | dep)
    assert bool(keep.any()), f"{tag}: no comparable problem"
    sel = lambda o, k: None if o is None else (o[k][:, keep] if o[k].dim() == 3 else o[k][keep])  # noqa: E731
    within(tag, "costs", sel(r, "costs"), sel(o64, "costs"), sel(o32, "costs"), dtype)
    rows = ~rows_holding(out | dep, T, m)
    if bool(rows.any()):
        g = lambda o: None if o is None else o["fdn"][rows]  # noqa: E731
        check_fdn(tag, r["full_du_norm"][rows], g(o64), g(o32), dtype, sc)
    want = (o64 if dtype == F64 else o32)["iters"]
    assert int(r["info"][0]) == want, f"{tag}: {int(r['info'][0])} iterations, the oracle ran {want}"
    assert int(r["info"][1]) == 0 or bounded, tag
    if "u_zero_I" in kw:
        assert bool((r["u"][kw["u_zero_I"]] == 0).all()), f"{tag}: masked controls"


# ------------------------------------------------------------------------------------------------------------------
# (a) every step plan the loop body can record, on both sides of its switch horizon
# ------------------------------------------------------------------------------------------------------------------
MODES = ("plain", "box", "boxT")
GROUPS = list(SWITCH_PLANS)


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("group", GROUPS)
def test_loop_plans_at_switch(group, dtype):
    """Short loops (B=16, 3 iterations) just below and at the switch horizon, under the default dispatch and each
    kernel forced; the plan recorded in the loop body is asserted, and every run is compared with the oracle."""
    pick = pick_switch(group, dtype)
    if pick is None:
        pytest.skip(f"no instance has a {group} switch of the loop's step within T <= {ORACLE_TMAX}")
    n, m, Ts, impls = pick
    gi = GROUPS.index(group)
    for k, T in enumerate((Ts - 1, Ts)):
        mode = MODES[(gi + k) % len(MODES)]
        case = loop_case(1100 + 10 * gi + k, 16, T, n, m, dtype, mode, 3, EPS[dtype])
        for impl in impls:
            want = loop_plan(n, m, dtype, T, impl)
            if want is None:
                continue
            tag = f"{group} n{n}m{m} {DT[dtype]} T={T} (T*={Ts}) {mode} MPCB200_KERNEL={impl}"
            r, plan = run_loop(n, m, T, *case[:3], dtype, impl)
            assert plan == want, f"{tag}: plan {_plan_str(plan)}, expected {_plan_str(want)}"
            LOOP_SEEN.setdefault(dtype, set()).add(_plan_name(plan, impl, n, m, dtype))
            check_loop(tag, r, case, dtype)


LARGE_CASES = [(20, 4, None, "boxT"), (8, 2, 3, "box"), (16, 4, 3, "plain")]


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("n,m,impl,mode", LARGE_CASES, ids=[f"n{c[0]}m{c[1]}_k{c[2]}_{c[3]}" for c in LARGE_CASES])
def test_loop_large_shape_kernels(n, m, impl, mode, dtype):
    """The large-shape kernels inside the loop: a shape without an instance, and MPCB200_KERNEL=3 at instances."""
    T = 10
    case = loop_case(1200 + n + m, 8, T, n, m, dtype, mode, 3, EPS[dtype])
    r, plan = run_loop(n, m, T, *case[:3], dtype, impl)
    assert plan == _L().PLAN_LARGE, _plan_str(plan)
    LOOP_SEEN.setdefault(dtype, set()).add("large")
    check_loop(f"large n{n}m{m} {DT[dtype]} {mode} MPCB200_KERNEL={impl}", r, case, dtype)


# ------------------------------------------------------------------------------------------------------------------
# (b) full-size batches, every problem against the oracle; device loop vs host loop at B=65536
# ------------------------------------------------------------------------------------------------------------------
# (name, n, m, B, T, mode, lqr_iter); float32, the default stop rule at eps = 1e-4
FULL = [("config3", 8, 2, 4096, 20, "plain", 4), ("config3_box", 8, 2, 4096, 20, "box", 5),
        ("config4_tensor", 8, 2, 1024, 20, "tensor", 5), ("config5_shard_box", 16, 4, 4096, 50, "box", 3)]


@pytest.mark.parametrize("name,n,m,B,T,mode,lqr_iter", FULL, ids=[c[0] for c in FULL])
def test_full_size_loop_vs_oracle(name, n, m, B, T, mode, lqr_iter):
    case = loop_case(3100 + FULL.index((name, n, m, B, T, mode, lqr_iter)), B, T, n, m, F32, mode, lqr_iter,
                     EPS[F32])
    r, plan = run_loop(n, m, T, *case[:3], F32)
    tag = f"{name} B={B} T={T} {mode} plan {_plan_str(plan)}"
    print(tag, "iterations", int(r["info"][0]), "track-kernel passes", math.ceil(T * B * max(n, m) / (4096 * 256)))
    check_loop(tag, r, case, F32)


def test_full_size_config5_shard_runs_kreduce():
    """The config-5 shard with the generic kernel forced: KREDUCE inside the loop, with a multi-pass track kernel."""
    n, m, B, T = 16, 4, 4096, 50
    assert T * B * max(n, m) > 4096 * 256
    case = loop_case(3103, B, T, n, m, F32, "box", 3, EPS[F32])
    r, plan = run_loop(n, m, T, *case[:3], F32, impl=1)
    assert plan == _plan(True, False, True), _plan_str(plan)
    LOOP_SEEN.setdefault(F32, set()).add("generic_kreduce")
    check_loop(f"config5 shard generic kernel B={B}", r, case, F32)


def test_device_loop_matches_host_loop_at_65536(monkeypatch):
    """(8,2) f32 B=65536 T=20 +-0.25: each stop-kernel thread walks 256 problems and the track kernel's grid wraps
    ten times.  The host loop keeps the best iterate with torch.where and reduces with torch: bitwise equal x, u,
    costs and iteration count, and full_du_norm equal up to its summation order."""
    from mpc.pytorch_b200.solver import MPC, LinDx, QuadCost
    B, T, n, m = 65536, 20, 8, 2
    C, c, F, f, x0 = [t.to(DEV) for t in gen_problem(3200, B, T, n, m, F32)]
    kw = dict(u_lower=-0.25, u_upper=0.25, lqr_iter=5, verbose=-1, exit_unconverged=False, detach_unconverged=False)
    dev, _ = same_on_both_loops(monkeypatch, lambda: MPC(n, m, T, **kw), x0, QuadCost(C, c), LinDx(F, f))
    assert dev.iters >= 2
    ctrl = MPC(n, m, T, **kw)
    u0 = torch.zeros(T, B, m, device=DEV)
    host = ctrl._ilqr_host(x0, QuadCost(C, c), LinDx(F, f), u0)
    dev = ctrl._ilqr_device(x0, QuadCost(C, c), LinDx(F, f), u0)
    a, b = dev["full_du_norm"].double(), host["full_du_norm"].double()
    rel = float(((a - b).abs() / b.abs().clamp_min(1e-30)).max())
    FDN_ERR.setdefault((F32, "device vs host rel"), []).append(rel)
    assert rel <= 1e-5, rel        # a sum of T*m = 40 squares of the same values, in another order


# ------------------------------------------------------------------------------------------------------------------
# (c) the three stop reasons at B > 256, float64
# ------------------------------------------------------------------------------------------------------------------
STOP_B, STOP_T = 300, 10


def test_stop_by_eps():
    """eps inside a >= 10x gap of the oracle's per-iteration max norms (run with eps = 0): the loop stops at the
    first iteration below it, before lqr_iter, and no norm lies within 3x of eps."""
    n, m, lqr_iter = 8, 2, 12
    mx = [t["full_du_max"] for t in loop_case(3300, STOP_B, STOP_T, n, m, F64, "box", lqr_iter, 0.0)[3]["trace"]]
    s = sorted(mx)
    eps = stop = None
    for _, i in sorted(((s[i + 1] / s[i], i) for i in range(len(s) - 1) if s[i] >= 1e-11 and s[i + 1] >= 10 * s[i]),
                       reverse=True):
        e = math.sqrt(s[i] * s[i + 1])
        j = next(j for j, v in enumerate(mx) if v < e) + 1
        if 2 <= j < lqr_iter:
            eps, stop = e, j
            break
    assert eps is not None, mx
    case = loop_case(3300, STOP_B, STOP_T, n, m, F64, "box", lqr_iter, eps)
    assert case[3]["iters"] == stop, (case[3]["iters"], stop, mx)
    r, _ = run_loop(n, m, STOP_T, *case[:3], F64)
    check_loop(f"eps stop B={STOP_B} eps={eps:.2e}", r, case, F64)


def test_stop_by_not_improved_lim():
    """No iteration after the first improves (best_cost_eps = -1e9): the loop stops after not_improved_lim + 1
    iterations and returns the first iterate, with that iterate's full_du_norm, while the latest iterate is carried."""
    n, m = 8, 2
    case = loop_case(3301, STOP_B, STOP_T, n, m, F64, "tensor", 10, 0.0, not_improved_lim=2, best_cost_eps=-1e9)
    assert case[3]["iters"] == 3
    r, _ = run_loop(n, m, STOP_T, *case[:3], F64)
    check_loop(f"not_improved_lim stop B={STOP_B}", r, case, F64)
    first = loop_case(3301, STOP_B, STOP_T, n, m, F64, "tensor", 1, 0.0)[3]
    assert torch.equal(case[3]["fdn"], first["fdn"])          # the oracle's best iterate is its first one


def test_stop_at_lqr_iter():
    n, m = 8, 2
    case = loop_case(3302, STOP_B, STOP_T, n, m, F64, "boxT", 4, 0.0, not_improved_lim=4)
    assert case[3]["iters"] == 4
    r, _ = run_loop(n, m, STOP_T, *case[:3], F64)
    check_loop(f"lqr_iter cap B={STOP_B}", r, case, F64)


# ------------------------------------------------------------------------------------------------------------------
# (d) full_du_norm decides MPC.forward's exit_unconverged assert and what detach_unconverged detaches
# ------------------------------------------------------------------------------------------------------------------
def _gap_eps(norms):
    """An eps at the geometric middle of the widest gap of the sorted norms whose neighbours are both >= 1e-11 (far
    above float64 round-off of a norm, ~1e-15) and differ by >= 3x, so that each lies >= 1.7x from eps: no keep /
    detach decision is made by round-off.  (The seeded problem below has no wider gap than 4.2x above 1e-11.)"""
    s = sorted(norms)
    gaps = [(s[i + 1] / s[i], i) for i in range(len(s) - 1) if s[i] >= 1e-11 and s[i + 1] >= 3 * s[i]]
    assert gaps, s
    i = max(gaps)[1]
    return math.sqrt(s[i] * s[i + 1])


def _grads(monkeypatch, base, ctrl_kw, device_loop):
    from mpc.pytorch_b200 import solver
    from mpc.pytorch_b200.solver import MPC, LinDx, QuadCost
    n, m, T = 8, 2, base[0].shape[0]
    C, c, F, f, x0 = [t.clone().requires_grad_(True) for t in base]
    with monkeypatch.context() as mp:
        if not device_loop:
            mp.setattr(solver, "_use_device_loop", lambda *a: False)
        x, u, _ = MPC(n, m, T, **ctrl_kw)(x0, QuadCost(C, c), LinDx(F, f))
        (x.square().sum() + u.sum()).backward()
    return [t.grad for t in (C, c, F, f, x0)]


def test_full_du_norm_decides_exit_and_detach(monkeypatch):
    from mpc.pytorch_b200.solver import MPC, LinDx, QuadCost
    n, m, T, B = 8, 2, 12, 64
    C, c, F, f, x0 = gen_problem(3, B, T, n, m, F64)
    box = dict(u_lower=-1.0, u_upper=1.0)
    P = dict(C=C, c=c, F=F, f=f, x0=x0, u0=torch.zeros(T, B, m, dtype=F64))
    o0 = _oracle(n, m, T, P, box, dict(lqr_iter=10, eps=0.0))
    eps = _gap_eps(o0["fdn"].tolist())
    o = _oracle(n, m, T, P, box, dict(lqr_iter=10, eps=eps))
    assert o["iters"] == o0["iters"] == 10
    keep = o["fdn"] < eps
    assert 0 < int(keep.sum()) < B

    # the device loop's full_du_norm: the oracle's, and the host loop's up to summation order
    d = [t.to(DEV) for t in (C, c, F, f, x0)]
    rc, _ = run_loop(n, m, T, P, box, dict(lqr_iter=10, eps=eps))
    check_loop(f"detach case eps={eps:.2e}", rc, (P, box, dict(lqr_iter=10, eps=eps), o, None), F64)
    # the keep / detach decision of every problem whose norm row holds no departing problem is the oracle's
    err = torch.maximum(_err_per_problem(rc["x"], o["x"]), _err_per_problem(rc["u"], o["u"]))
    clean = ~rows_holding(err > 1e-9 * max(1.0, float(o["x"].abs().max()), float(o["u"].abs().max())), T, m)
    assert torch.equal((rc["full_du_norm"] < eps)[clean], keep[clean])
    keep = rc["full_du_norm"] < eps                  # what MPC.forward decides from
    assert 0 < int(keep.sum()) < B
    ctrl = MPC(n, m, T, lqr_iter=10, eps=eps, **box)
    host = ctrl._ilqr_host(d[4], QuadCost(d[0], d[1]), LinDx(d[2], d[3]), P["u0"].to(DEV))
    a, b = rc["full_du_norm"], host["full_du_norm"].cpu()
    assert torch.equal(rc["x"], host["x"].cpu()) and torch.equal(rc["u"], host["u"].cpu())
    assert float(((a - b).abs() / b.abs().clamp_min(1e-300)).max()) <= 1e-12     # summation order only

    # exit_unconverged (default True): asserts with this eps, not with one above every problem's norm
    with pytest.raises(AssertionError):
        MPC(n, m, T, lqr_iter=10, eps=eps, **box)(d[4], QuadCost(d[0], d[1]), LinDx(d[2], d[3]))
    eps_hi = 10 * float(o0["fdn"].max())
    o_hi = _oracle(n, m, T, P, box, dict(lqr_iter=10, eps=eps_hi))
    assert float(o_hi["fdn"].max()) < eps_hi
    MPC(n, m, T, lqr_iter=10, eps=eps_hi, **box)(d[4], QuadCost(d[0], d[1]), LinDx(d[2], d[3]))

    # detach_unconverged: the converged problems' gradients are those of an undetached solve, the others are zero
    kw = dict(lqr_iter=10, eps=eps, exit_unconverged=False, verbose=-1, **box)
    g_det = _grads(monkeypatch, d, dict(kw, detach_unconverged=True), True)
    g_all = _grads(monkeypatch, d, dict(kw, detach_unconverged=False), True)
    g_host = _grads(monkeypatch, d, dict(kw, detach_unconverged=True), False)
    kd = keep.to(DEV)
    for name, gd, ga, gh in zip(("C", "c", "F", "f", "x_init"), g_det, g_all, g_host):
        bdim = 0 if name == "x_init" else 1
        assert torch.equal(gd, gh), f"{name}: device and host loop gradients differ"
        assert torch.equal(gd.index_select(bdim, kd.nonzero()[:, 0]), ga.index_select(bdim, kd.nonzero()[:, 0])), name
        assert bool((gd.index_select(bdim, (~kd).nonzero()[:, 0]) == 0).all()), f"{name}: a detached problem's gradient"
        assert bool((ga.index_select(bdim, (~kd).nonzero()[:, 0]) != 0).any()), name


# ------------------------------------------------------------------------------------------------------------------
# (e) u_zero_I, alone and with a tensor box, at an exact and a zero-padded control dimension
# ------------------------------------------------------------------------------------------------------------------
# (n, m, mode, lqr_iter, not_improved_lim, best_cost_eps): the mask-only cases keep their first iterate as the best
# (best_cost_eps = -1e9), so the returned full_du_norm is that of a full step, not round-off
MASK_CASES = [(8, 2, "mask", 5, 1, -1e9), (8, 2, "maskT", 4, 5, 1e-4), (3, 3, "mask", 5, 1, -1e9),
              (3, 3, "maskT", 4, 5, 1e-4)]


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("n,m,mode,lqr_iter,nil,bce", MASK_CASES,
                         ids=[f"n{c[0]}m{c[1]}_{c[2]}" for c in MASK_CASES])
def test_masked_controls_vs_oracle(n, m, mode, lqr_iter, nil, bce, dtype):
    B, T = 16, 10
    case = loop_case(3400 + 10 * n + m, B, T, n, m, dtype, mode, lqr_iter, EPS[dtype], nil, bce)
    r, _ = run_loop(n, m, T, *case[:3], dtype)
    check_loop(f"n{n}m{m} {mode} {DT[dtype]}", r, case, dtype)


# ------------------------------------------------------------------------------------------------------------------
# coverage: every plan the loop body can record ran inside the loop (runs last)
# ------------------------------------------------------------------------------------------------------------------
def test_zz_loop_plan_coverage():
    if not LOOP_SEEN:
        pytest.skip("no loop test of this module ran")
    missing = []
    for dtype in (F64, F32):
        need = {"large"}
        for group, plans in SWITCH_PLANS.items():
            if pick_switch(group, dtype) is not None:
                need |= set(plans)
        seen = LOOP_SEEN.get(dtype, set())
        print(f"{DT[dtype]}: switches", {g: pick_switch(g, dtype) for g in SWITCH_PLANS}, "plans run in the loop",
              sorted(seen))
        missing += [f"{DT[dtype]} {p}" for p in sorted(need - seen)]
        if need != {"large"} | {p for ps in SWITCH_PLANS.values() for p in ps}:
            print(f"{DT[dtype]}: plans without an instance that reaches them:",
                  sorted({p for ps in SWITCH_PLANS.values() for p in ps} - need))
    for (dtype, what), v in sorted(FDN_ERR.items(), key=lambda kv: (DT[kv[0][0]], kv[0][1])):
        print(f"full_du_norm {DT[dtype]} {what}: max observed {max(v):.3e} over {len(v)} runs")
    for dtype, v in DEPARTED.items():
        print(f"{DT[dtype]}: problems departing from the oracle {sum(a for a, _ in v)} of {sum(b for _, b in v)} "
              f"compared, in {sum(a > 0 for a, _ in v)} of {len(v)} runs")
    assert not missing, "plans never run inside the loop: " + ", ".join(missing)
