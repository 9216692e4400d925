"""Horizon-dependent kernel paths against the oracle.

Both step kernels change code path with the horizon T, chosen at launch from shared-memory arithmetic:
  * generic kernel: the gains K_t, k_t of all T steps stay in shared memory, or go through the caller's Ks/ks
    (too long for shared memory, or - for one-problem-per-warp shapes with n a power of two - the KREDUCE rollout,
    where lane i reads column i of K_t and K dx is summed by a butterfly);
  * column-pair kernel: the same choice, with the gains moved out early once the store is "crowded"; when the
    store does not fit and there is no buffer it refuses, and the default dispatch runs the generic kernel;
  * KKT adjoint: the fused pair kernel (2 launches) while d tau of all T steps fits shared memory, else the
    in-library masked step + costate + outer-product kernels (4 launches); LQRStepFn.backward takes the Python
    multi-call route (3 launches) where lqr_adjoint_raw declines the shape.
The switch horizons are found on the device by bisection (mpcb200_last_step_plan for step paths, launch counts for
adjoint routes), never hard-coded, and every comparison asserts the plan that ran, so a retuned constant cannot
silently drop a path: test_zz_coverage_table fails if any instance x dtype misses an applicable path.

Tolerances: float64 1e-9 x scale, active sets / clamp masks / pnqp iteration counts bit exact.  float32 over long
horizons: the kernel's error against the float64 oracle must stay within 4x the error of the oracle itself run in
float32 (on the same float32-rounded inputs) plus 1e-6 x scale.  Inputs come from tests.helpers.gen_problem with
F *= 0.9, so trajectories stay O(1) at T ~ 900."""
import contextlib
import ctypes
import functools
import os

import pytest
import torch

from oracle import lqr_oracle as orc
from tests.helpers import gen_problem, maxdiff, nominal_controls

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
F32, F64 = torch.float32, torch.float64
INSTANCES = [(1, 1), (2, 1), (2, 2), (3, 1), (3, 2), (3, 4), (4, 1), (4, 2), (4, 4), (5, 1), (6, 2), (7, 4), (8, 1),
             (8, 2), (8, 4), (12, 4), (16, 4)]
PAIR_SHAPES = [s for s in INSTANCES if s[0] % 2 == 0 and s[1] % 2 == 0]
KREDUCE_SHAPES = {(16, 4)}          # one problem per warp, n a power of two
TMAX = 1024                         # switches are searched in [1, TMAX]
ORACLE_TMAX = 900                   # oracle comparisons at switches up to this horizon
PROBE_B = 8                         # one warp of every mapping; 16-byte aligned spans for every shape and dtype
DT = {F32: "f32", F64: "f64"}
COVERAGE = {}                       # (n, m, dtype) -> {what: set of plans / launch counts seen}


def _L():
    from mpc.pytorch_b200 import _lib
    return _lib


def _plan_str(p):
    L = _L()
    if p == 0:
        return "none"
    s = "generic" if p & L.PLAN_GENERIC else "pair"
    s += "/smem" if p & L.PLAN_GAINS_SMEM else "/Ks"
    return s + ("+kreduce" if p & L.PLAN_KREDUCE else "")


def _seen(n, m, dtype, what, value):
    COVERAGE.setdefault((n, m, dtype), {}).setdefault(what, set()).add(value)


@contextlib.contextmanager
def _kernel(impl):
    """MPCB200_KERNEL: None default dispatch, 1 generic, 2 column pair."""
    old = os.environ.pop("MPCB200_KERNEL", None)
    if impl is not None:
        os.environ["MPCB200_KERNEL"] = str(impl)
    try:
        yield
    finally:
        os.environ.pop("MPCB200_KERNEL", None)
        if old is not None:
            os.environ["MPCB200_KERNEL"] = old


# ------------------------------------------------------------------------------------------------------------------
# finding the switches on the device
# ------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=2)
def _probe_inputs(n, m, dtype):
    p = n + m
    C = torch.eye(p, dtype=dtype, device=DEV).expand(TMAX, PROBE_B, p, p).contiguous()
    c = torch.ones(TMAX, PROBE_B, p, dtype=dtype, device=DEV)
    F = torch.cat((0.9 * torch.eye(n, dtype=dtype, device=DEV), torch.ones(n, m, dtype=dtype, device=DEV) / p), 1)
    F = F.expand(TMAX, PROBE_B, n, p).contiguous()
    x = torch.zeros(TMAX, PROBE_B, n, dtype=dtype, device=DEV)
    u = torch.zeros(TMAX, PROBE_B, m, dtype=dtype, device=DEV)
    return C, c, F, x, u


def _probe_step(n, m, dtype, T, impl, want_gains, do_rollout=True):
    """Plan of one step launch at horizon T; 0 if the library refused it for lack of shared memory."""
    from mpc.pytorch_b200.step import lqr_step_raw
    C, c, F, x, u = _probe_inputs(n, m, dtype)
    with _kernel(impl):
        try:
            lqr_step_raw(n, m, T, x[0], C[:T], c[:T], F[:T - 1], None, x[:T], u[:T], do_rollout=do_rollout,
                         want_gains=want_gains, want_stats=False)
        except _L().MpcB200Error as e:
            if "[4]" in str(e):
                return 0
            raise
        return _L().last_step_plan()


def _probe_adjoint(n, m, dtype, T):
    """Launches of one mpcb200_lqr_adjoint_* call at horizon T: 2 fused, 4 in-library 3-launch route, 0 if the
    masked generic step does not fit shared memory either (callers then take the multi-call route)."""
    C, c, F, x, u = _probe_inputs(n, m, dtype)
    try:
        _, launches = _abi_adjoint(n, m, T, C[:T], c[:T], F[:T - 1], x[:T], u[:T], x[:T], u[:T], None, None, False)
    except _L().MpcB200Error as e:
        if "[4]" in str(e):
            return 0
        raise
    return launches


def _first_true(pred, lo=0, hi=TMAX):
    """Smallest T in (lo, hi] with pred(T), pred monotone and pred(lo) False; None if pred(hi) is False."""
    if hi <= lo or not pred(hi):
        return None
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if pred(mid):
            hi = mid
        else:
            lo = mid
    return hi


@functools.lru_cache(maxsize=None)
def switches(n, m, dtype):
    """First horizon of each non-default side (None: not below TMAX / not applicable to the shape).
      generic          generic kernel with a Ks/ks buffer: gains leave shared memory
      generic_riccati  generic kernel, Riccati sweep only: gains no longer fit shared memory
      pair             pair kernel with a Ks/ks buffer: gains leave shared memory ("crowded" or not fitting)
      pair_nofit       pair kernel, Riccati sweep only: gains no longer fit shared memory
      adjoint          mpcb200_lqr_adjoint_*: fused kernel -> in-library 3-launch route"""
    L = _L()
    out = dict(
        generic=_first_true(lambda T: not _probe_step(n, m, dtype, T, 1, True) & L.PLAN_GAINS_SMEM),
        generic_riccati=_first_true(lambda T: not _probe_step(n, m, dtype, T, 1, True, False) & L.PLAN_GAINS_SMEM),
        pair=None, pair_nofit=None, adjoint=None)
    if (n, m) in PAIR_SHAPES:
        out["pair"] = _first_true(lambda T: not _probe_step(n, m, dtype, T, 2, True) & L.PLAN_GAINS_SMEM)
        out["pair_nofit"] = _first_true(lambda T: not _probe_step(n, m, dtype, T, 2, True, False) & L.PLAN_GAINS_SMEM)
        out["adjoint"] = _first_true(lambda T: _probe_adjoint(n, m, dtype, T) != 2)
    for k, v in out.items():
        _seen(n, m, dtype, "T*:" + k, v)
    return out


# ------------------------------------------------------------------------------------------------------------------
# problems, library calls, comparisons
# ------------------------------------------------------------------------------------------------------------------
def _round(t, dtype):
    """float32 cases: every input is rounded to float32 once, so kernel and oracle see the same numbers."""
    return t.to(dtype).double() if torch.is_tensor(t) and t.is_floating_point() and dtype == F32 else t


@functools.lru_cache(maxsize=4)
def step_case(seed, B, T, n, m, dtype, mode, with_f=True):
    """Inputs (float64, rounded through dtype) and the oracle: (P, kw, o64, o32|None).
    mode: plain | mask (u_zero_I) | box (scalar bounds) | boxT (tensor bounds + delta_u)."""
    C, c, F, f, x0 = gen_problem(seed, B, T, n, m, F64, with_f=with_f)
    F = F * 0.9
    u, ul, uu = nominal_controls(seed, B, T, m, F64, {"box": 0.25, "boxT": "tensor"}.get(mode))
    kw = {}
    if mode in ("box", "boxT"):
        kw = dict(u_lower=_round(ul, dtype), u_upper=_round(uu, dtype))
    if mode == "boxT":
        kw["delta_u"] = 0.125
    if mode == "mask":
        kw["u_zero_I"] = torch.rand(T, B, m, generator=torch.Generator().manual_seed(seed)) < 0.3
    C, c, F, f, x0, u = (_round(t, dtype) for t in (C, c, F, f, x0, u))
    x = _round(orc.get_traj(T, u, x0, F, f), dtype)
    P = dict(C=C, c=c, F=F, f=f, x0=x0, x=x, u=u)
    o64 = orc.lqr_step_forward(n, m, T, x0, C, c, F, f, x, u, coupled=False, **kw)
    o32 = None
    if dtype == F32:
        lo = lambda t: t.float() if torch.is_tensor(t) and t.is_floating_point() else t
        o32 = orc.lqr_step_forward(n, m, T, lo(x0), lo(C), lo(c), lo(F), lo(f), lo(x), lo(u), coupled=False,
                                   **{k: lo(v) for k, v in kw.items()})
    return P, kw, o64, o32


def _step(n, m, T, P, kw, dtype, impl=None, want_gains=True, do_rollout=True):
    """lqr_step_raw on the device; returns (outputs on the CPU, plan)."""
    from mpc.pytorch_b200.step import lqr_step_raw
    d = lambda t: t.to(device=DEV, dtype=dtype if t.is_floating_point() else t.dtype) if torch.is_tensor(t) else t
    with _kernel(impl):
        o = lqr_step_raw(n, m, T, d(P["x0"]), d(P["C"]), d(P["c"]), d(P["F"]), d(P["f"]), d(P["x"]), d(P["u"]),
                         do_rollout=do_rollout, want_gains=want_gains, **{k: d(v) for k, v in kw.items()})
        plan = _L().last_step_plan()
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in o.items() if v is not None}, plan


def _close(tag, what, got, w64, w32, dtype, scale=None):
    if scale is None:
        scale = max(1.0, float(w64.abs().max()))
    err = maxdiff(got, w64)
    bound = 1e-9 * scale if dtype == F64 else 4 * maxdiff(w32, w64) + 1e-6 * scale
    assert err <= bound, f"{tag}: {what} |kernel - oracle| = {err:.3e} > {bound:.3e}"


def check_step(tag, r, case, dtype, rollout=True):
    P, kw, o64, o32 = case
    g = lambda o, k: getattr(o, k) if o is not None else None
    bounded = "u_lower" in kw
    if rollout:
        sc = max(1.0, float(o64.new_x.abs().max()), float(o64.new_u.abs().max()))
        for k in ("new_x", "new_u"):
            _close(tag, k, r[k], g(o64, k), g(o32, k), dtype, sc)
        _close(tag, "costs", r["costs"], o64.costs, g(o32, "costs"), dtype)
        if o32 is None:
            assert torch.equal(r["alphas"], o64.alphas), f"{tag}: alphas"
        else:          # float32: the same line-search decisions wherever the float32 oracle makes the float64 ones
            same = (o32.alphas.double() - o64.alphas).abs() <= 1e-6
            assert torch.equal(r["alphas"][same], o32.alphas[same]), f"{tag}: alphas"
    if "Ks" in r:
        _close(tag, "Ks", r["Ks"], o64.Ks, g(o32, "Ks"), dtype)
        _close(tag, "ks", r["ks"], o64.ks, g(o32, "ks"), dtype)
    assert int((r["status"] & ~1).max()) == 0, tag
    assert not bool((r["status"] & 1).any()), f"{tag}: pnqp flagged unconverged"
    assert torch.equal(r["free_mask"].bool(), o64.free_masks), f"{tag}: free sets"
    if bounded:
        assert torch.equal(r["qp_iters"].long(), o64.qp_iters), f"{tag}: pnqp iterations"
        if rollout and "delta_u" not in kw:
            lo, hi = kw["u_lower"], kw["u_upper"]
            assert torch.equal(r["new_u"].double() == lo, o64.new_u == lo), f"{tag}: lower clamp mask"
            assert torch.equal(r["new_u"].double() == hi, o64.new_u == hi), f"{tag}: upper clamp mask"
    if rollout and "u_zero_I" in kw:
        assert bool((r["new_u"][kw["u_zero_I"]] == 0).all()), f"{tag}: masked controls"


def _modes(dtype, k):
    """Mode rotation: float64 cases cycle through every mode; float32 cases (compared against the float32 oracle
    as yardstick, where a round-off-decided pnqp stop would make the yardstick meaningless) use the unbounded ones."""
    ms = ("box", "mask", "boxT", "plain") if dtype == F64 else ("mask", "plain")
    return ms[k % len(ms)]


def _plan(generic, smem, kreduce=False):
    L = _L()
    return ((L.PLAN_GENERIC if generic else L.PLAN_PAIR) | (L.PLAN_GAINS_SMEM if smem else 0)
            | (L.PLAN_KREDUCE if kreduce else 0))


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
            case = step_case(100 + n * 10 + m, B, T, n, m, dtype, mode)
            r, plan = _step(n, m, T, case[0], case[1], dtype, impl=1, do_rollout=rollout)
            want = _plan(True, T < Ts, kred and rollout and T >= Ts)
            tag = f"generic {leg} n{n}m{m} {DT[dtype]} T={T} B={B} {mode}"
            assert plan == want, f"{tag}: plan {_plan_str(plan)}, expected {_plan_str(want)}"
            _seen(n, m, dtype, f"generic_{leg}", plan)
            check_step(tag, r, case, dtype, rollout)


KREDUCE_CASES = [(F64, "plain"), (F64, "box"), (F64, "mask"), (F32, "plain"), (F32, "mask")]


@pytest.mark.parametrize("dtype,mode", KREDUCE_CASES, ids=[f"{DT[d]}_{md}" for d, md in KREDUCE_CASES])
def test_generic_kreduce_long_horizon(dtype, mode):
    """KREDUCE at T=300: every row of Ks / ks and the rollout against the oracle."""
    n, m, T, B = 16, 4, 300, 5
    case = step_case(400, B, T, n, m, dtype, mode)
    r, plan = _step(n, m, T, case[0], case[1], dtype, impl=1)
    assert plan == _plan(True, False, True), _plan_str(plan)
    _seen(n, m, dtype, "generic_rollout", plan)
    check_step(f"kreduce {DT[dtype]} T={T} {mode}", r, case, dtype)


def _long_default(n, m, T, dtype, mode, B, kernel):
    """Default dispatch far past every gain-store switch: the gains round-trip through the caller's Ks/ks."""
    case = step_case(40, B, T, n, m, dtype, mode)
    r, plan = _step(n, m, T, case[0], case[1], dtype)
    assert plan == _plan(kernel == "generic", False), _plan_str(plan)
    check_step(f"long default n{n}m{m} {DT[dtype]} T={T} {mode}", r, case, dtype)


def test_gains_spill_to_global_for_long_horizons():
    """(8,2) float64, T=700, scalar bounds, default dispatch: too long for the shared-memory gain store, so the
    generic kernel round-trips K, k through the caller's buffer (the plan says so), and matches the oracle."""
    _long_default(8, 2, 700, F64, "box", 20, "generic")


# (n, m, T, dtype, mode, B, kernel the default dispatch picks)
LONG_DEFAULT = [(8, 4, 700, F32, "mask", 12, "pair"), (2, 2, 700, F64, "boxT", 12, "pair")]


@pytest.mark.parametrize("n,m,T,dtype,mode,B,kernel", LONG_DEFAULT,
                         ids=[f"n{c[0]}m{c[1]}_T{c[2]}_{DT[c[3]]}_{c[4]}" for c in LONG_DEFAULT])
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
        case = step_case(200 + n * 10 + m, B, T, n, m, dtype, mode)
        tag = f"pair crowded n{n}m{m} {DT[dtype]} T={T} B={B} {mode}"
        r1, p1 = _step(n, m, T, case[0], case[1], dtype, impl=2, want_gains=True)
        assert p1 == _plan(False, T < Ts), f"{tag}: plan {_plan_str(p1)}"
        check_step(tag + " want_gains", r1, case, dtype)
        # without a buffer below the generic kernel's switch the gains stay in shared memory
        r0, p0 = _step(n, m, T, case[0], case[1], dtype, impl=2, want_gains=False)
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
    below = step_case(seed, B, Tn - 1, n, m, dtype, mode)
    tag = f"pair long n{n}m{m} {DT[dtype]} T={Tn - 1} B={B} {mode}"
    r, plan = _step(n, m, Tn - 1, below[0], below[1], dtype, impl=2, want_gains=True)
    assert plan == _plan(False, False), f"{tag}: plan {_plan_str(plan)}"
    _seen(n, m, dtype, "pair_rollout", plan)
    check_step(tag, r, below, dtype)
    r, plan = _step(n, m, Tn - 1, below[0], below[1], dtype, impl=2, do_rollout=False)
    assert plan == _plan(False, True), f"{tag} riccati: plan {_plan_str(plan)}"
    _seen(n, m, dtype, "pair_riccati", plan)
    check_step(tag + " riccati", r, below, dtype, rollout=False)

    at = step_case(seed, B, Tn, n, m, dtype, mode)
    tag = f"pair no-fit n{n}m{m} {DT[dtype]} T={Tn} B={B} {mode}"
    r, plan = _step(n, m, Tn, at[0], at[1], dtype, impl=2, do_rollout=False)
    assert plan == _plan(False, False), f"{tag} riccati: plan {_plan_str(plan)}"
    _seen(n, m, dtype, "pair_riccati", plan)
    check_step(tag + " riccati", r, at, dtype, rollout=False)
    if sw["generic"] is not None and Tn >= sw["generic"]:
        return          # lqr_step_raw passes Ks/ks at this horizon: no bufferless call to fall back from
    r, plan = _step(n, m, Tn, at[0], at[1], dtype, impl=None, want_gains=False)
    assert plan == _plan(True, True), f"{tag} fallback: plan {_plan_str(plan)}"
    _seen(n, m, dtype, "pair_fallback", plan)
    check_step(tag + " fallback", r, at, dtype)
    P = {k: (v.to(DEV, dtype) if torch.is_tensor(v) else v) for k, v in at[0].items()}
    kw = {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in at[1].items()}
    kw = {k: (v.to(dtype) if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in kw.items()}
    with _kernel(2), pytest.raises(_L().MpcB200Error, match=r"\[4\]"):
        lqr_step_raw(n, m, Tn, P["x0"], P["C"], P["c"], P["F"], P["f"], P["x"], P["u"], **kw)
    assert _L().last_step_plan() == 0
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------------------
# KKT adjoint routes
# ------------------------------------------------------------------------------------------------------------------
def _abi_adjoint(n, m, T, C, c, F, new_x, new_u, dl_dx, dl_du, lo, hi, with_f):
    """mpcb200_lqr_adjoint_* through the C ABI (device tensors); returns (dx_init, dC, dc, dF, df|None), launches."""
    L = _L()
    from mpc.pytorch_b200._lib import Dims, Params, check, ptr, stream_handle
    dtype, B, p = C.dtype, C.shape[1], n + m
    kind = 0 if lo is None else (1 if isinstance(lo, float) else 2)
    dims = Dims(B=B, T=T, n=n, m=m, F_T=T - 1, has_f=int(with_f), bounds_kind=kind, max_ls_iter=10,
                pnqp_max_iter=20, do_rollout=1)
    prm = Params(u_lo=lo if kind == 1 else 0.0, u_hi=hi if kind == 1 else 0.0, delta_u=0.0, ls_decay=0.2)
    esz = C.element_size()
    nbytes = L.lib().mpcb200_adjoint_workspace_bytes(ctypes.byref(dims), esz)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    out = [torch.empty(B, n, dtype=dtype, device=DEV), torch.empty(T, B, p, p, dtype=dtype, device=DEV),
           torch.empty(T, B, p, dtype=dtype, device=DEV), torch.empty(T - 1, B, n, p, dtype=dtype, device=DEV),
           torch.empty(T - 1, B, n, dtype=dtype, device=DEV) if with_f else None]
    fn = L.lib().mpcb200_lqr_adjoint_f32 if dtype == F32 else L.lib().mpcb200_lqr_adjoint_f64
    before = L.launch_count()
    rc = fn(ctypes.byref(dims), ctypes.byref(prm), ptr(C), ptr(c), ptr(F), ptr(new_x), ptr(new_u), ptr(dl_dx),
            ptr(dl_du), ptr(lo if kind == 2 else None), ptr(hi if kind == 2 else None), *[ptr(t) for t in out],
            ptr(ws), nbytes, stream_handle(DEV))
    check(rc, "mpcb200_lqr_adjoint")
    torch.cuda.synchronize()
    return out, L.launch_count() - before


@functools.lru_cache(maxsize=4)
def adjoint_case(seed, B, T, n, m, dtype, bounds, with_f):
    """A solved problem (one oracle step from u = 0, so box bounds leave an active set), upstream gradients,
    and the oracle's adjoint in float64 (and float32): (P, kw, ref64, ref32|None)."""
    C, c, F, f, x0 = gen_problem(seed, B, T, n, m, F64, with_f=with_f)
    F = F * 0.9
    g = torch.Generator().manual_seed(seed)
    kw = {}
    if bounds == "box":
        kw = dict(u_lower=-0.25, u_upper=0.25)
    elif bounds == "tensor":
        kw = dict(u_lower=_round(-0.5 * torch.rand(T, B, m, generator=g, dtype=F64) - 0.05, dtype),
                  u_upper=_round(0.5 * torch.rand(T, B, m, generator=g, dtype=F64) + 0.05, dtype))
    C, c, F, f, x0 = (_round(t, dtype) for t in (C, c, F, f, x0))
    u = torch.zeros(T, B, m, dtype=F64)
    o = orc.lqr_step_forward(n, m, T, x0, C, c, F, f, orc.get_traj(T, u, x0, F, f), u, coupled=False, **kw)
    x, u = _round(o.new_x, dtype), _round(o.new_u, dtype)
    wx = _round(torch.randn(T, B, n, generator=g, dtype=F64), dtype)
    wu = _round(torch.randn(T, B, m, generator=g, dtype=F64), dtype)
    P = dict(C=C, c=c, F=F, f=f, x0=x0, x=x, u=u, wx=wx, wu=wu)
    ref64 = orc.lqr_step_backward(n, m, T, x0, C, c, F, f, x, u, wx, wu, coupled=False, **kw)
    ref32 = None
    if dtype == F32:
        lo = lambda t: t.float() if torch.is_tensor(t) else t
        ref32 = orc.lqr_step_backward(n, m, T, lo(x0), lo(C), lo(c), lo(F), lo(f), lo(x), lo(u), lo(wx), lo(wu),
                                      coupled=False, **{k: lo(v) for k, v in kw.items()})
    return P, kw, ref64, ref32


def _run_abi_adjoint(n, m, T, case, dtype, impl=None):
    P, kw, _, _ = case
    d = lambda t: t.to(DEV, dtype) if torch.is_tensor(t) else t
    with _kernel(impl):
        out, launches = _abi_adjoint(n, m, T, d(P["C"]), d(P["c"]), d(P["F"]), d(P["x"]), d(P["u"]), d(P["wx"]),
                                     d(P["wu"]), d(kw.get("u_lower")), d(kw.get("u_upper")), P["f"] is not None)
    return [t.cpu() if t is not None else None for t in out], launches


def check_adjoint(tag, got, case, dtype):
    _, _, ref64, ref32 = case
    for i, name in enumerate(("dx_init", "dC", "dc", "dF", "df")):
        if got[i] is None:
            assert ref64[i].numel() == 0, f"{tag}: {name} missing"
            continue
        _close(tag, name, got[i], ref64[i], ref32[i] if ref32 is not None else None, dtype)


def check_routes_agree(tag, a, b, case, dtype):
    """Two adjoint routes on one input: float64 within 1e-9 x scale of each other; float32 within the sum of their
    float32 yardsticks (each is checked against the oracle on its own)."""
    _, _, ref64, ref32 = case
    for i, name in enumerate(("dx_init", "dC", "dc", "dF", "df")):
        if a[i] is None:
            continue
        sc = max(1.0, float(ref64[i].abs().max()))
        err = maxdiff(a[i], b[i])
        bound = 1e-9 * sc if dtype == F64 else 2 * (4 * maxdiff(ref32[i], ref64[i]) + 1e-6 * sc)
        assert err <= bound, f"{tag}: {name} routes differ by {err:.3e} > {bound:.3e}"


ADJ_BOUNDS = (None, "box", "tensor")


@pytest.mark.parametrize("n,m,dtype", PAIR_PARAMS, ids=PAIR_PIDS)
def test_adjoint_fused_to_three_launch_switch(n, m, dtype):
    """Fused just below the fit limit, in-library 3-launch route at it, both against the oracle's adjoint."""
    Ta = switches(n, m, dtype)["adjoint"]
    assert Ta is not None and Ta <= ORACLE_TMAX
    B = _B(n, m, dtype)
    for k, T in enumerate((Ta - 1, Ta)):
        bounds = ADJ_BOUNDS[(n + m + k) % 3]
        with_f = (n + k) % 3 != 0
        case = adjoint_case(600 + n * 10 + m, B, T, n, m, dtype, bounds, with_f)
        got, launches = _run_abi_adjoint(n, m, T, case, dtype)
        tag = f"adjoint n{n}m{m} {DT[dtype]} T={T} B={B} bounds={bounds} f={with_f}"
        assert launches == (2 if T < Ta else 4), f"{tag}: {launches} launches"
        # the nested masked step (fused or not) keeps its gains in shared memory: it has no Ks/ks buffer
        assert _L().last_step_plan() & _L().PLAN_GAINS_SMEM, f"{tag}: {_plan_str(_L().last_step_plan())}"
        _seen(n, m, dtype, "adjoint_launches", launches)
        check_adjoint(tag, got, case, dtype)


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
    g3, l3 = _run_abi_adjoint(n, m, T, case, dtype, impl=1)
    assert l3 == 4, f"{tag}: {l3} launches"
    check_adjoint(tag + " 3-launch", g3, case, dtype)
    _seen(n, m, dtype, "adjoint_launches", l3)
    if (n, m) in PAIR_SHAPES:
        g2, l2 = _run_abi_adjoint(n, m, T, case, dtype)
        assert l2 == 2, f"{tag}: {l2} launches"
        check_adjoint(tag + " fused", g2, case, dtype)
        _seen(n, m, dtype, "adjoint_launches", l2)
        check_routes_agree(tag + " fused vs 3-launch", g2, g3, case, dtype)


@pytest.mark.parametrize("dtype", [F32, F64], ids=["f32", "f64"])
def test_config5_backward_takes_multicall_route(dtype):
    """(16,4) T=50 (config 5): LQRStepFn.backward sends this shape to the Python multi-call route (the fit test asks
    the generic kernel, whose KREDUCE preference says no), although the fused adjoint fits; all three routes agree."""
    from mpc.pytorch_b200 import LQRStep, QuadCost, LinDx
    n, m, T, B = 16, 4, 50, 5
    case = adjoint_case(800, B, T, n, m, dtype, "box", True)
    P, kw = case[:2]
    lv = [P[k].to(DEV, dtype).requires_grad_(True) for k in ("x0", "C", "c", "F", "f")]
    fn = LQRStep(n, m, T, true_cost=QuadCost(lv[1], lv[2]), true_dynamics=LinDx(lv[3], lv[4]),
                 current_x=P["x"].to(DEV, dtype), current_u=P["u"].to(DEV, dtype), no_op_forward=True, **kw)
    xo, uo = fn(*lv)
    before = _L().launch_count()
    grads = torch.autograd.grad((xo, uo), lv, (P["wx"].to(DEV, dtype), P["wu"].to(DEV, dtype)))
    torch.cuda.synchronize()
    tag = f"config5 backward {DT[dtype]}"
    # (the step plan is per host thread, and autograd runs this backward on its own device thread)
    assert _L().launch_count() - before == 3, f"{tag}: not the multi-call route"
    _seen(n, m, dtype, "adjoint_launches", 3)
    multi = [t.cpu() for t in grads[:5]]
    check_adjoint(tag + " multi-call", multi, case, dtype)
    fused, l2 = _run_abi_adjoint(n, m, T, case, dtype)
    three, l3 = _run_abi_adjoint(n, m, T, case, dtype, impl=1)
    assert (l2, l3) == (2, 4), (l2, l3)
    check_adjoint(tag + " fused", fused, case, dtype)
    check_adjoint(tag + " 3-launch", three, case, dtype)
    check_routes_agree(tag + " multi-call vs fused", multi, fused, case, dtype)
    check_routes_agree(tag + " multi-call vs 3-launch", multi, three, case, dtype)


# ------------------------------------------------------------------------------------------------------------------
# mpcb200_lqr_grad_* with and without a workspace
# ------------------------------------------------------------------------------------------------------------------
def _abi_grad(n, m, T, P, dx, du, dtype, with_f, workspace):
    L = _L()
    from mpc.pytorch_b200._lib import Dims, check, ptr, stream_handle
    ins = [P["C"], P["c"], P["F"], P["x"], P["u"], dx, du, P["wx"]]
    ins = [t.to(DEV, dtype).contiguous() for t in ins]             # kept alive across the call
    B, p = P["C"].shape[1], n + m
    dims = Dims(B=B, T=T, n=n, m=m, F_T=T - 1, has_f=int(with_f), max_ls_iter=1, pnqp_max_iter=1)
    out = [torch.empty(B, n, dtype=dtype, device=DEV), torch.empty(T, B, p, p, dtype=dtype, device=DEV),
           torch.empty(T, B, p, dtype=dtype, device=DEV), torch.empty(T - 1, B, n, p, dtype=dtype, device=DEV),
           torch.empty(T - 1, B, n, dtype=dtype, device=DEV) if with_f else None]
    ws = torch.empty(2 * T * B * n, dtype=dtype, device=DEV) if workspace else None
    fn = L.lib().mpcb200_lqr_grad_f32 if dtype == F32 else L.lib().mpcb200_lqr_grad_f64
    before = L.launch_count()
    rc = fn(ctypes.byref(dims), *[ptr(t) for t in ins], *[ptr(t) for t in out], ptr(ws), stream_handle(DEV))
    check(rc, "mpcb200_lqr_grad")
    torch.cuda.synchronize()
    return [t.cpu() if t is not None else None for t in out], L.launch_count() - before


GRAD_CASES = [(8, 2, 9, F64), (8, 2, 300, F64), (5, 1, 9, F64), (5, 1, 300, F32), (16, 4, 12, F32), (16, 4, 250, F64)]


@pytest.mark.parametrize("n,m,T,dtype", GRAD_CASES, ids=[f"n{n}m{m}_T{T}_{DT[d]}" for n, m, T, d in GRAD_CASES])
def test_grad_without_workspace_matches_two_kernel_path(n, m, T, dtype):
    """The one-kernel gradient (workspace NULL) and the two-kernel one, fed the costate inputs of a solved problem
    (the oracle's adjoint solution dx, du), against the oracle's outer products."""
    case = adjoint_case(900 + n + T, 12, T, n, m, dtype, "box", True)
    P, _, ref64, ref32 = case
    dx, du = ref64[5], ref64[6]
    one, l1 = _abi_grad(n, m, T, P, dx, du, dtype, True, False)
    two, l2 = _abi_grad(n, m, T, P, dx, du, dtype, True, True)
    assert (l1, l2) == (1, 2), (l1, l2)
    tag = f"grad n{n}m{m} T={T} {DT[dtype]}"
    for i, name in enumerate(("dx_init", "dC", "dc", "dF", "df")):
        sc = max(1.0, float(ref64[i].abs().max()))
        if dtype == F64:
            _close(tag + " one kernel", name, one[i], ref64[i], None, dtype)
            _close(tag + " two kernels", name, two[i], ref64[i], None, dtype)
        else:
            # the kernel is fed float32-rounded dx, du: the yardstick is the float32 oracle's own adjoint
            for got, nm in ((one, "one kernel"), (two, "two kernels")):
                err, bound = maxdiff(got[i], ref64[i]), 4 * maxdiff(ref32[i], ref64[i]) + 1e-6 * sc
                assert err <= bound, f"{tag} {nm}: {name} {err:.3e} > {bound:.3e}"
        d = maxdiff(one[i], two[i])
        assert d <= (1e-12 if dtype == F64 else 1e-6) * sc, f"{tag}: one vs two kernels, {name}: {d:.3e}"
        _seen(n, m, dtype, "grad one vs two kernels bit-identical", d == 0.0)


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
    gid = {k: v for k, v in COVERAGE.items() if "grad one vs two kernels bit-identical" in v}
    print("grad one vs two kernels bit-identical:",
          {f"n{n}m{m}_{DT[d]}": sorted(v["grad one vs two kernels bit-identical"]) for (n, m, d), v in gid.items()})
    assert not missing, "\n".join(missing)
