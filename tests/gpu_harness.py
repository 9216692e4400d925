"""What the GPU test modules share: device plumbing, the two tolerance policies, case builders, the checks of a step
against the oracle, the device probes of the kernels' switch horizons, the runner that solves an MPC on the
device loop or the host loop, and the raw call and float64 check of the standalone pnqp.

Tolerance policies (DESIGN section 4):
  * `within`: float64 within tol64 x scale of the float64 oracle; float32 within K32 = 4 times the error of the
    oracle itself run in float32 on the same float32-rounded inputs (`round_through`), plus 1e-6 x scale;
  * `tol_for`: the fixed SURVEY.md section 8c tolerances, for cases whose inputs are generated in their own dtype.

Importing this module touches no device: the library is loaded when a function that needs it runs."""
import contextlib
import ctypes
import functools
import math
import os
from collections import namedtuple

import numpy as np
import torch

from oracle import lqr_oracle as orc
from tests.helpers import gen_problem, maxdiff, nominal_controls

DEV = torch.device("cuda:0")
F32, F64 = torch.float32, torch.float64
DT = {F32: "f32", F64: "f64"}
K32 = 4


def _L():
    from mpc.pytorch_b200 import _lib
    return _lib


# ------------------------------------------------------------------------------------------------------------------
# device plumbing
# ------------------------------------------------------------------------------------------------------------------
def to_dev(t, dtype=None):
    """t on DEV, floating-point tensors cast to dtype when one is given; anything but a tensor is returned as is."""
    if not torch.is_tensor(t):
        return t
    return t.to(DEV, dtype if dtype is not None and t.is_floating_point() else t.dtype)


@contextlib.contextmanager
def kernel_env(impl):
    """MPCB200_KERNEL: None default dispatch, 1 generic, 2 column pair, 3 large-shape kernels."""
    old = os.environ.pop("MPCB200_KERNEL", None)
    if impl is not None:
        os.environ["MPCB200_KERNEL"] = str(impl)
    try:
        yield
    finally:
        os.environ.pop("MPCB200_KERNEL", None)
        if old is not None:
            os.environ["MPCB200_KERNEL"] = old


def run_step(n, m, T, P, kw=None, dtype=None, impl=None, want_gains=True, **opts):
    """lqr_step_raw on the device for the problem P (x0, C, c, F, f, x, u), with the problem's options kw (bounds,
    u_zero_I, delta_u, line search) and the call's opts (do_rollout, want_du_first, dyn); returns (outputs on the
    CPU, step plan)."""
    from mpc.pytorch_b200.step import lqr_step_raw
    d = lambda t: to_dev(t, dtype)  # noqa: E731
    with kernel_env(impl):
        o = lqr_step_raw(n, m, T, *[d(P[k]) for k in ("x0", "C", "c", "F", "f", "x", "u")],
                         want_gains=want_gains, **{k: d(v) for k, v in (kw or {}).items()}, **opts)
        plan = _L().last_step_plan()
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in o.items() if v is not None}, plan


def run_loop(n, m, T, P, kw, opts, dtype=None, impl=None):
    """step.ilqr_raw on the device from P (x0, C, c, F, f, u0); returns (outputs on the CPU, the plan of the step
    recorded in the loop body)."""
    from mpc.pytorch_b200.step import ilqr_raw
    d = lambda t: to_dev(t, dtype)  # noqa: E731
    with kernel_env(impl):
        res = ilqr_raw(n, m, T, *[d(P[k]) for k in ("x0", "C", "c", "F", "f", "u0")],
                       **{k: d(v) for k, v in kw.items()}, **opts)
        plan = _L().last_step_plan()
    assert res is not None, "the driver has no conditional graph nodes"
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in res.items()}, plan


def staged(t, dtype):
    """(tensor, mpcb200_dims time-stride field) of a [T, B, ...] input as the shim stages it (step._time_strided):
    dense and misaligned contiguous views stay as they are, stride-0 and 16-byte time strides keep their stride.
    None and empty tensors: (None, 0)."""
    from mpc.pytorch_b200.step import _time_strided
    if t is None or t.numel() == 0:
        return None, 0
    return _time_strided(t, dtype)


def _grad_buffers(T, B, n, m, F_T, want_df, dtype, poison):
    """dx_init, dC, dc, dF [F_T slices], df [T-1 slices] or None: empty, or all NaN when `poison`."""
    p = n + m
    make = (lambda *s: torch.full(s, float("nan"), dtype=dtype, device=DEV)) if poison else \
        (lambda *s: torch.empty(s, dtype=dtype, device=DEV))
    return [make(B, n), make(T, B, p, p), make(T, B, p), make(F_T, B, n, p), make(T - 1, B, n) if want_df else None]


def abi_adjoint(n, m, T, C, c, F, new_x, new_u, dl_dx, dl_du, lo=None, hi=None, with_f=True, F_T=None, poison=False):
    """mpcb200_lqr_adjoint_* through the C ABI on device tensors; lo, hi None, floats or tensors.  C, c and F keep
    their time strides (stride 0, or a 16-byte multiple) and every tensor its storage offset, as the shim hands them
    over.  F_T: time slices of F and dF (default T - 1).  poison: every output starts as NaN, so an element the call
    does not write fails any comparison; with_f False then still hands over a NaN df buffer (has_f = 0), which must
    come back untouched.  Returns ([dx_init, dC, dc, dF, df or None] on the CPU, kernel launches)."""
    L = _L()
    dtype, B = C.dtype, C.shape[1]
    F_T = T - 1 if F_T is None else F_T
    assert F is None and F_T == 0 or F.shape[0] == F_T, "F must hold F_T time slices"
    kind = 0 if lo is None else (1 if isinstance(lo, float) else 2)
    (C_, tsC), (c_, tsc), (F_, tsF) = staged(C, dtype), staged(c, dtype), staged(F, dtype)
    dims = L.Dims(B=B, T=T, n=n, m=m, F_T=F_T, has_f=int(with_f), bounds_kind=kind, max_ls_iter=10,
                  pnqp_max_iter=20, do_rollout=1, C_tstride=tsC, c_tstride=tsc, F_tstride=tsF)
    prm = L.Params(u_lo=lo if kind == 1 else 0.0, u_hi=hi if kind == 1 else 0.0, delta_u=0.0, ls_decay=0.2)
    nbytes = L.lib().mpcb200_adjoint_workspace_bytes(ctypes.byref(dims), C.element_size())
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    ins = [t.contiguous() for t in (new_x, new_u, dl_dx, dl_du)]         # alive until the sync
    ins += [lo.contiguous() if kind == 2 else None, hi.contiguous() if kind == 2 else None]
    out = _grad_buffers(T, B, n, m, F_T, with_f or poison, dtype, poison)
    df = out[4]
    if not with_f:
        out[4] = None
    before = L.launch_count()
    rc = L.entry("mpcb200_lqr_adjoint", dtype)(ctypes.byref(dims), ctypes.byref(prm), L.ptr_view(C_), L.ptr_view(c_),
                                               L.ptr_view(F_), *[L.ptr(t) for t in ins + out[:4]], L.ptr(df),
                                               L.ptr(ws), nbytes, L.stream_handle(DEV))
    L.check(rc, "mpcb200_lqr_adjoint")
    torch.cuda.synchronize()
    if not with_f and df is not None:
        assert bool(df.isnan().all()), "mpcb200_lqr_adjoint wrote df although has_f = 0"
    return [t.cpu() if t is not None else None for t in out], L.launch_count() - before


def abi_grad(n, m, T, C, c, F, new_x, new_u, dx, du, dl_dx, with_df=True, F_T=None, poison=False):
    """mpcb200_lqr_grad_* (costates through the workspace, then the outer products) through the C ABI on device
    tensors, C, c and F staged as abi_adjoint stages them; F_T and poison as there (without df the df pointer is
    NULL: the kernels take has_df from it).  Returns ([dx_init, dC, dc, dF, df or None] on the CPU, launches)."""
    L = _L()
    dtype, B = C.dtype, C.shape[1]
    F_T = T - 1 if F_T is None else F_T
    assert F is None and F_T == 0 or F.shape[0] == F_T, "F must hold F_T time slices"
    (C_, tsC), (c_, tsc), (F_, tsF) = staged(C, dtype), staged(c, dtype), staged(F, dtype)
    dims = L.Dims(B=B, T=T, n=n, m=m, F_T=F_T, has_f=int(with_df), max_ls_iter=1, pnqp_max_iter=1,
                  C_tstride=tsC, c_tstride=tsc, F_tstride=tsF)
    ins = [t.contiguous() for t in (new_x, new_u, dx, du, dl_dx)]
    out = _grad_buffers(T, B, n, m, F_T, with_df, dtype, poison)
    ws = torch.empty(2 * T * B * n, dtype=dtype, device=DEV)
    before = L.launch_count()
    rc = L.entry("mpcb200_lqr_grad", dtype)(ctypes.byref(dims), L.ptr_view(C_), L.ptr_view(c_), L.ptr_view(F_),
                                            *[L.ptr(t) for t in ins + out], L.ptr(ws), L.stream_handle(DEV))
    L.check(rc, "mpcb200_lqr_grad")
    torch.cuda.synchronize()
    return [t.cpu() if t is not None else None for t in out], L.launch_count() - before


def abi_rollout(n, m, T, F, f, x0, u, poison=False):
    """mpcb200_rollout_* through the C ABI on device tensors: x [T, B, n] on the CPU.  F [T-1 or T, B, n, n+m] (None
    or empty at T = 1) and f [T-1, B, n] (None or empty: no f) are staged as abi_adjoint stages them; poison: x starts
    as NaN."""
    L = _L()
    dtype, B = x0.dtype, x0.shape[0]
    (F_, tsF), (f_, tsf) = staged(F, dtype), staged(f, dtype)
    dims = L.Dims(B=B, T=T, n=n, m=m, F_T=F.shape[0] if F is not None else T - 1, has_f=int(f_ is not None),
                  max_ls_iter=1, pnqp_max_iter=1, F_tstride=tsF, f_tstride=tsf)
    x = torch.full((T, B, n), float("nan") if poison else 0.0, dtype=dtype, device=DEV)
    ins = [x0.contiguous(), u.contiguous()]
    rc = L.entry("mpcb200_rollout", dtype)(ctypes.byref(dims), L.ptr_view(F_), L.ptr_view(f_),
                                           *[L.ptr(t) for t in ins], L.ptr(x), L.stream_handle(DEV))
    L.check(rc, "mpcb200_rollout")
    torch.cuda.synchronize()
    return x.cpu()


def misaligned(t):
    """A contiguous copy of t that starts one element into its allocation, so data_ptr() % 16 != 0: the shim hands it
    to the kernels unchanged (a contiguous tensor is never copied), and the library picks its copy path for it."""
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
    v = buf[1:].view(t.shape)
    v.copy_(t)
    return v


# ------------------------------------------------------------------------------------------------------------------
# tolerance policies
# ------------------------------------------------------------------------------------------------------------------
def round_through(t, dtype):
    """float32 cases: every input is rounded to float32 once, so kernel and oracle see the same numbers."""
    return t.to(dtype).double() if torch.is_tensor(t) and t.is_floating_point() and dtype == F32 else t


def within(tag, what, got, w64, w32, dtype, tol64=1e-9, scale=None):
    """float64: |got - w64| <= tol64 x scale; float32: <= K32 |w32 - w64| + 1e-6 x scale.  scale defaults to
    max(1, |w64|)."""
    if scale is None:
        scale = max(1.0, float(w64.abs().max())) if w64.numel() else 1.0
    err = maxdiff(got, w64)
    bound = tol64 * scale if dtype == F64 else K32 * maxdiff(w32, w64) + 1e-6 * scale
    assert err <= bound, f"{tag}: {what} |kernel - oracle| = {err:.3e} > {bound:.3e}"


def tol_for(dtype, bounded):
    """SURVEY.md section 8c: float64 1e-9 on x, u and costs; float32 4e-5 (unbounded) or 2e-4 (bounded: pnqp stops
    at |dx| < 1e-4) on x, u and 3e-4 on costs."""
    if dtype == F64:
        return dict(xu=1e-9, cost=1e-9)
    return dict(xu=2e-4 if bounded else 4e-5, cost=3e-4)


# ------------------------------------------------------------------------------------------------------------------
# case builders
# ------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=8)
def linear_step_case(seed, B, T, n, m, dtype, mode, with_f=True, F_T=None):
    """LinDx step inputs (float64, rounded through dtype) and the oracle's step: (P, kw, o64, o32|None).
    mode: plain | mask (u_zero_I) | box (scalar bounds) | boxT (tensor bounds) | boxD (tensor bounds + delta_u).
    F_T=T: F carries T time slices."""
    C, c, F, f, x0 = gen_problem(seed, B, T, n, m, F64, with_f=with_f)
    F = F * 0.9                         # trajectories stay O(1) over long horizons
    if F_T == T:
        F = torch.cat((F, F[-1:]), 0) if T > 1 else gen_problem(seed, B, 2, n, m, F64)[2] * 0.9
    u, ul, uu = nominal_controls(seed, B, T, m, F64, {"box": 0.25, "boxT": "tensor", "boxD": "tensor"}.get(mode))
    kw = {}
    if mode.startswith("box"):
        kw = dict(u_lower=round_through(ul, dtype), u_upper=round_through(uu, dtype))
    if mode == "boxD":
        kw["delta_u"] = 0.125
    if mode == "mask":
        kw["u_zero_I"] = torch.rand(T, B, m, generator=torch.Generator().manual_seed(seed)) < 0.3
    C, c, F, f, x0, u = (round_through(t, dtype) for t in (C, c, F, f, x0, u))
    x = round_through(orc.get_traj(T, u, x0, F, f), dtype)
    P = dict(C=C, c=c, F=F, f=f, x0=x0, x=x, u=u)
    return (P, kw) + oracle_steps(n, m, T, P, kw, dtype)


def oracle_steps(n, m, T, P, kw, dtype, **opts):
    """The oracle's step on P in float64 and, for float32 cases, in float32 (the yardstick): (o64, o32|None)."""
    args = [P[k] for k in ("x0", "C", "c", "F", "f", "x", "u")]
    o64 = orc.lqr_step_forward(n, m, T, *args, coupled=False, **kw, **opts)
    if dtype != F32:
        return o64, None
    lo = lambda t: t.float() if torch.is_tensor(t) and t.is_floating_point() else t  # noqa: E731
    return o64, orc.lqr_step_forward(n, m, T, *map(lo, args), coupled=False, **{k: lo(v) for k, v in kw.items()},
                                     **opts)


LS_MARGIN = 1e-4                    # least |cost - oldcost| / max(1, |oldcost|) of a kept problem in every pass
ONE, MID, MAX = 0, 1, 2             # line-search classes: one pass; backtracked, then better; worse on every pass
LsCase = namedtuple("LsCase", "P kw o64 trace o32 first64 first32 classes")


def rollout_passes(trace):
    """Rollout passes each problem ran, from the oracle's ls_trace [passes, B] (cost - oldcost of every pass): up to
    its first pass that is not worse, else all of them (the batch loop ran to max_ls)."""
    better = trace <= 0
    return torch.where(better.any(0), better.to(torch.int64).argmax(0) + 1, trace.shape[0])


def ls_classes(trace):
    """ONE, MID or MAX per problem (a problem of class MAX ends worse than its nominal and restores alpha)."""
    p = rollout_passes(trace)
    worse_end = trace.gather(0, (p - 1).view(1, -1))[0] > 0
    return torch.where(worse_end, MAX, torch.where(p == 1, ONE, MID))


def _ls_oracle(n, m, T, P, kw, lo=None):
    """The per-problem oracle's step with its line-search trace and first-pass controls: (o, trace, first_u)."""
    lo = lo or (lambda t: t)
    trace, first = [], []
    o = orc.lqr_step_forward(n, m, T, *[lo(P[k]) for k in ("x0", "C", "c", "F", "f", "x", "u")], coupled=False,
                             ls_trace=trace, first_u=first, **{k: lo(v) for k, v in kw.items()})
    return o, torch.stack(trace), first[0]


def ls_nominal(seed, K, T, n, m, mode, shifted=False):
    """K float64 problems whose nominal (x, u) makes the line search backtrack, four families by index k % 4:
    0 unstable dynamics (F x 1.5-2, its 4/T-th power beyond T = 4) with the nominal rolled out from x0; 1 nominal controls
    perturbed at t >= 1 (0.3 N(0, 1), kept in the box) after the state was rolled out; 2, 3 a nominal state perturbed
    at t >= 1 (N(0, 1)) and pulled down the gradient of its stage cost by up to 6, so that its cost lies between the
    costs of the rollout's passes.  These nominals start at x0 (x[0] = x_init).  shifted: family 1 is instead a
    consistent nominal rolled out from a shifted initial state x0 + N(0, 1), so x[0] != x_init (DESIGN.md section 4:
    the step's feedback then acts on x_init - x[0] from t = 0).  mode: plain | box (+-0.1) | boxT (tensor box) | boxD
    (tensor box + delta_u) | mask (u_zero_I) | boxM (+-0.1 and u_zero_I)."""
    C, c, F, f, x0 = gen_problem(seed, K, T, n, m, F64)
    g = torch.Generator().manual_seed(seed + 13)
    fam = torch.arange(K) % 4
    s = 1.5 + 0.5 * torch.rand(K, generator=g, dtype=F64)
    scale = torch.where(fam == 0, s ** min(1.0, 4.0 / T), torch.full_like(s, 0.9))
    F = F * scale.view(1, K, 1, 1)
    u, ul, uu = nominal_controls(seed, K, T, m, F64, {"box": 0.1, "boxM": 0.1, "boxT": "tensor",
                                                      "boxD": "tensor"}.get(mode))
    x = orc.get_traj(T, u, x0, F, f)
    later = (torch.arange(T) >= 1).view(T, 1, 1)
    du = 0.3 * torch.randn(T, K, m, generator=g, dtype=F64)
    if shifted:
        delta = torch.randn(K, n, generator=torch.Generator().manual_seed(seed + 17), dtype=F64)
        x = orc.get_traj(T, u, x0 + delta * (fam == 1).view(K, 1), F, f)
    else:
        u = torch.where((fam == 1).view(1, K, 1) & later, u + du, u)
    if ul is not None:
        lo, hi = (torch.as_tensor(v, dtype=F64).expand_as(u) for v in (ul, uu))
        u = torch.minimum(torch.maximum(u, lo), hi)
    noise = torch.randn(T, K, n, generator=g, dtype=F64)
    pull = 6.0 * torch.rand(K, generator=g, dtype=F64)
    pert = (fam >= 2).view(1, K, 1) & later
    x = torch.where(pert, x + noise, x)
    grad = torch.einsum("tbij,tbj->tbi", C[..., :n, :], torch.cat((x, u), 2)) + c[..., :n]
    x = torch.where(pert, x - pull.view(1, K, 1) * grad / grad.norm(dim=2, keepdim=True).clamp_min(1e-12), x)
    kw = {}
    if mode.startswith("box"):
        kw = dict(u_lower=ul, u_upper=uu)
    if mode == "boxD":
        kw["delta_u"] = 0.125
    if mode in ("mask", "boxM"):
        kw["u_zero_I"] = torch.rand(T, K, m, generator=g) < 0.3
    return dict(C=C, c=c, F=F, f=f, x0=x0, x=x, u=u), kw


def _take(v, idx, B):
    """Batch elements idx of an input: [B, ...] (x0) or [T, B, ...]; scalars as they are."""
    if not torch.is_tensor(v):
        return v
    return v.index_select(0 if v.dim() == 2 and v.shape[0] == B else 1, idx)


@functools.lru_cache(maxsize=8)
def _ls_pool(seed, K, T, n, m, dtype, mode, max_ls, decay, shifted=False):
    """The candidates of line_search_case: inputs rounded through dtype, and per candidate its class, or -1 where it
    is not kept (a comparison within LS_MARGIN, a MAX problem whose final pass equals its first, or a float32 oracle
    that decides differently)."""
    P, kw = ls_nominal(seed, K, T, n, m, mode, shifted)
    P = {k: round_through(v, dtype) for k, v in P.items()}
    kw = {k: round_through(v, dtype) for k, v in kw.items()}
    kw.update(linesearch_decay=decay, max_linesearch_iter=max_ls)
    o, trace, first = _ls_oracle(n, m, T, P, kw)
    cls = ls_classes(trace)
    old = o.costs - trace[-1]
    counted = torch.arange(trace.shape[0]).view(-1, 1) < rollout_passes(trace).view(1, -1)
    ok = ((trace.abs() >= LS_MARGIN * old.abs().clamp_min(1.0)) | ~counted).all(0)
    if max_ls > 1:
        ok &= (cls != MAX) | ((first - o.new_u).abs().amax((0, 2)) > 1e-6)
    if dtype == F32:
        _, t32, _ = _ls_oracle(n, m, T, P, kw, lambda t: t.float() if torch.is_tensor(t) and t.is_floating_point()
                               else t)
        ok &= (ls_classes(t32) == cls) & (rollout_passes(t32) == rollout_passes(trace))
    return P, kw, torch.where(ok, cls, -1)


def line_search_case(seed, T, n, m, dtype, mode, max_ls, decay, layout, K=192, shifted=False):
    """A batch with a chosen line-search class at each position (`layout`: a sequence of ONE / MID / MAX), drawn from
    K seeded candidates (ls_nominal, `shifted` as there) classified by the float64 oracle.  The kernels and the oracle solve every
    problem on its own, so a candidate keeps its class wherever it is placed; the oracle is rerun on the batch and
    must agree.  A class the candidates lack is replaced by the next of MID, MAX, ONE that they have.  Returns an
    LsCase: inputs P, options kw, float64 oracle o64 with its line-search trace, float32 oracle o32|None, the
    first-pass controls of both, and the classes."""
    P, kw, pool = _ls_pool(seed, K, T, n, m, dtype, mode, max_ls, decay, shifted)
    have = {c: (pool == c).nonzero()[:, 0].tolist() for c in (ONE, MID, MAX)}
    order = {ONE: (ONE, MID, MAX), MID: (MID, MAX, ONE), MAX: (MAX, MID, ONE)}
    seen = {ONE: 0, MID: 0, MAX: 0}
    idx = []
    for c in layout:
        c = next(d for d in order[c] if have[d])
        idx.append(have[c][seen[c] % len(have[c])])
        seen[c] += 1
    idx = torch.tensor(idx)
    Bp = pool.shape[0]
    P = {k: _take(v, idx, Bp) for k, v in P.items()}
    kw = {k: _take(v, idx, Bp) for k, v in kw.items()}
    o64, trace, first64 = _ls_oracle(n, m, T, P, kw)
    classes = ls_classes(trace)
    assert torch.equal(classes, pool[idx]), "the oracle classifies a batch element unlike its candidate"
    o32 = first32 = None
    if dtype == F32:
        o32, _, first32 = _ls_oracle(n, m, T, P, kw, lambda t: t.float() if torch.is_tensor(t) and
                                     t.is_floating_point() else t)
    return LsCase(P, kw, o64, trace, o32, first64, first32, classes)


def step_layout(kernel, n, m, dtype):
    """(problems per warp, problems per CTA) of a step kernel at the (n, m) it runs: StepCfg (lqr_step.cuh) for
    the generic kernel, Step2Cfg (lqr_step2.cuh) for the column-pair kernel, one problem per CTA for the large-shape
    kernels."""
    if kernel == "large":
        return 1, 1
    if kernel == "pair":
        ppw = 32 // ((n + m) // 2)
        return ppw, ppw
    sz = 8 if dtype == F64 else 4
    lanes = n if (n, m, dtype) == (8, 2, F32) else n + m
    ppw = 32 // lanes
    span_ok = lambda nw: (nw * ppw * m * sz) % 16 == 0 and (nw * ppw * n * sz) % 16 == 0  # noqa: E731
    nw = 2 if lanes == n else 1 if span_ok(1) else 2 if span_ok(2) else 4
    return ppw, nw * ppw


def grad_layout(n, m):
    """(problems per warp, problems per CTA) of the gradient kernels (GradCfg, lqr_grad.cuh): n+m lanes per problem,
    four warps per CTA.  The outer-product kernel masks its flat stores by the problems of its warp group."""
    ppw = 32 // (n + m)
    return ppw, 4 * ppw


def rollout_layout(n):
    """(problems per warp, problems per CTA) of the LinDx rollout kernel (RolloutCfg, lqr_rollout.cuh): n lanes per
    problem, four warps per CTA."""
    ppw = 32 // n
    return ppw, 4 * ppw


def pool_size(*layout):
    """Smallest pool of at least 3 problems whose size is coprime to every given warp / CTA size: batch element b is
    pool problem b % K, so neighbouring warps and CTAs hold different problems, and a kernel that reads another
    batch element's operands reads another problem."""
    return next(k for k in range(3, 64) if all(math.gcd(k, s) == 1 for s in layout))


def layout_batches(ppw, W, K=None):
    """Batch sizes that put problems at every warp and CTA position and end in every kind of tail: one problem, a
    partial, full and just-overfull warp, a CTA short by one, full and overfull by one, two CTAs and a warp and one
    more.  With a pool of K: also K CTAs and a warp and one more, so that every pool problem sits at every position
    of a full CTA."""
    out = {1, ppw - 1, ppw, ppw + 1, W - 1, W, W + 1, 2 * W + ppw + 1}
    if K is not None:
        out.add(K * W + ppw + 1)
    return sorted(b for b in out if b >= 1)


def batch_rows(v, idx):
    """Batch elements idx of an input or an oracle output: [B, n] along dim 0, [T, B, ...] along dim 1; floats and
    empty tensors as they are."""
    if not torch.is_tensor(v) or v.numel() == 0:
        return v
    return v.index_select(0 if v.dim() == 2 else 1, idx)


def ls_layout(B, ppw, W):
    """Classes by batch position.  The first problem of every warp takes one pass, and so does all of warp 0 in
    even CTAs of several warps: a repeat decided by that problem or that warp alone would stop too early.  The other
    positions cycle through MAX, MID, ONE; the tail CTA keeps its warp 0 in the cycle.  With one problem per CTA the
    cycle is ONE, MAX, MID."""
    out = []
    for b in range(B):
        q, w, cta = b % ppw, (b % W) // ppw, b // W
        if W == 1:
            out.append((ONE, MAX, MID)[b % 3])
        elif q == 0 or (w == 0 and W > ppw and cta % 2 == 0 and (cta + 1) * W < B):
            out.append(ONE)
        else:
            out.append((MAX, MID, ONE)[(q - 1 + cta) % 3])
    if B > 1:
        out[-1] = MAX                   # the tail CTA always holds a problem that backtracks
    return tuple(out)


def rollout(module, x0, u):
    """[T, B, n]: x0 rolled out through module under the controls u [T, B, m]."""
    xs = [x0]
    for t in range(u.shape[0] - 1):
        xs.append(module(xs[t], u[t]))
    return torch.stack(xs)


def jacobians(module, xs, us):
    """(next, R, S) of module(xs, us) by autograd."""
    xs = xs.clone().requires_grad_(True)
    us = us.clone().requires_grad_(True)
    nx = module(xs, us)
    rows = [torch.autograd.grad(nx[:, j].sum(), [xs, us], retain_graph=True) for j in range(nx.shape[1])]
    return nx.detach(), torch.stack([r[0] for r in rows], 1), torch.stack([r[1] for r in rows], 1)


def linearise(module, x, u):
    """F = [R S] [T-1, B, n, n+m] and f = x' - R x - S u [T-1, B, n] of module at (x[:-1], u[:-1]), by autograd."""
    T, B, n = x.shape
    m = u.shape[2]
    xs, us = x[:-1].reshape(-1, n), u[:-1].reshape(-1, m)
    nx, R, S = jacobians(module, xs, us)
    f = nx - torch.einsum("bij,bj->bi", R, xs) - torch.einsum("bij,bj->bi", S, us)
    return torch.cat((R, S), 2).view(T - 1, B, n, n + m), f.view(T - 1, B, n)


# known systems with non-default physics: parameters, dt, control clamp
PHYS = {
    "cartpole": dict(params=(9.81, 1.3, 0.25, 0.8), dt=0.1, clamp_attr="force_mag", clamp=7.5, n=5),
    "pendulum": dict(params=(9.1, 1.7, 0.6), dt=0.15, clamp_attr="max_torque", clamp=1.5, n=3),
}
RADII = {"cartpole": (0.3, 1.0, 2.0), "pendulum": (0.3, 1.0, 3.0)}
SYSTEMS = tuple(PHYS)
BT = [(1, 1), (1, 200), (127, 11), (128, 2), (129, 11), (300, 200), (4097, 11), (4097, 2)]


def known_module(name, params=None, device="cpu"):
    from mpc.pytorch_b200.dynamics import CartpoleDx, PendulumDx
    ph = PHYS[name]
    p = torch.tensor(ph["params"], dtype=F64) if params is None else params
    dx = (CartpoleDx if name == "cartpole" else PendulumDx)(params=p.to(device))
    dx.dt = ph["dt"]
    setattr(dx, ph["clamp_attr"], ph["clamp"])
    return dx


def angle_cols(name):
    return (2, 3) if name == "cartpole" else (0, 1)


def known_states(name, B, seed):
    """float64 [B, n]: random states, angle pair at the RADII; the first rows hold the theta edge cases."""
    g = torch.Generator().manual_seed(seed)
    n = PHYS[name]["n"]
    x = (torch.rand(B, n, generator=g, dtype=F64) - 0.5) * 2.0
    th = (torch.rand(B, generator=g, dtype=F64) * 2 - 1) * 3.0
    r0, _, r1 = RADII[name]
    r = torch.tensor(RADII[name], dtype=F64).repeat(B)[:B]
    ic, is_ = angle_cols(name)
    x[:, ic], x[:, is_] = r * torch.cos(th), r * torch.sin(th)
    edge = ((-1.0, 0.0), (-1.0, -0.0), (-r0, 0.0), (-r1, -0.0), (1.0, 1e-9), (1.0, -1e-9), (r1, 0.0))
    for k, (cv, sv) in enumerate(edge[:B]):
        x[k, ic], x[k, is_] = cv, sv
    return x


def _clamp_edges(clamp, dtype):
    """u at the clamp, one ulp (of dtype) inside and outside it, both signs."""
    npd = np.float64 if dtype == F64 else np.float32
    c = npd(clamp)
    inn, out = float(np.nextafter(c, npd(0))), float(np.nextafter(c, npd(np.inf)))
    return (clamp, -clamp, inn, -inn, out, -out)


def known_controls(name, T, B, dtype, seed):
    """float64 [T, B, 1] in +-1.5 clamp; the edge values are spread over the first rows of every time step."""
    g = torch.Generator().manual_seed(seed + 1)
    clamp = PHYS[name]["clamp"]
    u = (torch.rand(T, B, 1, generator=g, dtype=F64) * 2 - 1) * 1.5 * clamp
    e = torch.tensor(_clamp_edges(clamp, dtype), dtype=F64)
    k = min(B, len(e))
    u[:, -k:, 0] = e[:k]                  # the last rows: the first rows hold the theta edges
    return u


# ------------------------------------------------------------------------------------------------------------------
# checks of one step against the oracle, over the problems `keep` (all by default)
# ------------------------------------------------------------------------------------------------------------------
def _cols(t, keep):
    if t is None or keep is None:
        return t
    return t[:, keep] if t.dim() >= 2 else t[keep]


def decays(alphas, decay):
    """Number of decays behind each alpha (alpha = decay ** decays): the line-search decisions, free of the
    dtype's rounding of decay ** decays."""
    return torch.round(torch.log(alphas.double()) / math.log(decay)).long()


def f32_compared(case):
    """float32 cases (P, kw, o64, trace, o32, ...): the problems whose line-search decisions the comparison may
    demand.  Left out are near-ties (|cost - oldcost| within 1e-5 relative in any pass of the float64 oracle:
    round-off may decide that comparison either way) and problems where the float32 oracle, the yardstick, decides
    differently."""
    P, kw, o64, trace, o32 = case[:5]
    old = o64.costs - trace[-1]
    tie = (trace.abs() <= 1e-5 * old.abs().clamp_min(1.0)).any(0)
    decay = kw["linesearch_decay"]
    return ~tie & (decays(o32.alphas, decay) == decays(o64.alphas, decay))


def check_alphas(tag, r, o64, o32, keep=None):
    """float64: alphas bit exact; float32: the float32 oracle's alphas wherever it makes the float64 oracle's
    line-search decisions."""
    got, w64 = _cols(r["alphas"], keep), _cols(o64.alphas, keep)
    if o32 is None:
        assert torch.equal(got, w64), f"{tag}: alphas {got} vs {w64}"
    else:
        w32 = _cols(o32.alphas, keep)
        same = (w32.double() - w64).abs() <= 1e-6
        assert torch.equal(got[same], w32[same]), f"{tag}: alphas"


def check_trajectory(tag, r, u, o64, o32, dtype, keep=None, first=None):
    """The outputs r holds, under `within`: new_x and new_u (on one scale), costs, Ks and ks; with du_first, the
    first full step u - new_u and its per-problem norm full_du_norm.  `first`: the new_u of the oracles' first
    line-search pass (float64, float32|None) where the line search backtracks; by default their final new_u.  A
    Riccati-only step holds the gains alone."""
    g = lambda o, k: None if o is None else _cols(getattr(o, k), keep)  # noqa: E731
    if "new_x" in r:
        sc = max(1.0, float(g(o64, "new_x").abs().max()), float(g(o64, "new_u").abs().max()))
        for k in ("new_x", "new_u"):
            within(tag, k, _cols(r[k], keep), g(o64, k), g(o32, k), dtype, scale=sc)
        within(tag, "costs", _cols(r["costs"], keep), g(o64, "costs"), g(o32, "costs"), dtype)
    if "du_first" in r:
        u = _cols(u, keep)
        f64, f32 = first if first is not None else (o64.new_u, None if o32 is None else o32.new_u)
        du = lambda f: None if f is None else u - _cols(f, keep)  # noqa: E731
        norm = lambda d: None if d is None else d.pow(2).sum((0, 2)).sqrt()  # noqa: E731
        within(tag, "du_first", _cols(r["du_first"], keep), du(f64), du(f32), dtype, scale=sc)
        within(tag, "full_du_norm", _cols(r["full_du_norm"], keep), norm(du(f64)), norm(du(f32)), dtype, scale=sc)
    if "Ks" in r:
        within(tag, "Ks", _cols(r["Ks"], keep), g(o64, "Ks"), g(o32, "Ks"), dtype)
        within(tag, "ks", _cols(r["ks"], keep), g(o64, "ks"), g(o32, "ks"), dtype)


def check_pnqp(tag, r, o, kw, keep=None):
    """pnqp against the oracle's o: no status bit but the cap flag, the cap flag only where the oracle's QP hits the
    cap, free sets bit exact, with bounds the iteration counts, and masked controls exactly zero."""
    assert int((r["status"] & ~1).max()) == 0, f"{tag}: status {r['status'].tolist()}"
    assert torch.equal(_cols(r["free_mask"].bool(), keep), _cols(o.free_masks, keep)), f"{tag}: free sets"
    bounded = kw.get("u_lower") is not None
    if bounded:
        capped = (o.qp_iters == 19).any(0)
        flagged = _cols((r["status"] & 1).bool() & ~capped, keep)
        assert not bool(flagged.any()), f"{tag}: pnqp flagged problems whose oracle QPs converged"
        assert torch.equal(_cols(r["qp_iters"].long(), keep), _cols(o.qp_iters, keep)), f"{tag}: pnqp iterations"
    if "new_u" in r and kw.get("u_zero_I") is not None:
        assert bool((r["new_u"][kw["u_zero_I"]] == 0).all()), f"{tag}: masked controls"


def check_clamps(tag, r, o, kw, keep=None):
    """Bounded steps without delta_u: the controls on each bound bit exact."""
    if "new_u" not in r or kw.get("u_lower") is None or kw.get("delta_u") is not None:
        return
    for side in ("u_lower", "u_upper"):
        b = kw[side] if torch.is_tensor(kw[side]) else torch.full_like(o.new_u, kw[side])
        assert torch.equal(_cols(r["new_u"].double() == b.double(), keep),
                           _cols(o.new_u.double() == b.double(), keep)), f"{tag}: {side} clamp mask"


def on_bounds(u, kw, sel=lambda t: t):
    """[2, T, B, m]: which controls u [T, B, m] sit on the lower / upper bound; tensor bounds go through sel (the
    batch rows u holds)."""
    lo_, hi = (sel(kw[k]) if torch.is_tensor(kw[k]) else torch.full_like(u.double(), kw[k]) for k in ("u_lower",
                                                                                                    "u_upper"))
    return torch.stack((u.double() == lo_.double(), u.double() == hi.double()))


def check_loop_departures(tag, r, o64, o32, kw, lqr_iter, sensitive, dtype, idx=None):
    """x, u and costs of a device iLQR loop per problem against the oracle's loop (x, u, costs, iterations), under
    test_ilqr_oracle_gpu.check_loop's rule.  A problem departs where its x or u misses the tolerance (float64 1e-9 x
    scale; float32 4x the float32 oracle's own error plus 1e-6 x scale), or where its controls on a bound differ from
    the oracle's.  Only bounded loops of more than one iteration may have departing problems, at most one in four:
    pnqp's |dx| >= 1e-4 stop decides some problems' paths by round-off.  Where more depart, each one beyond that
    allowance must be a problem whose float64 oracle loop itself moves under a 1e-15 relative change of C
    (sensitive(tol) -> [B] of the oracle's batch).  float32 problems the float32 oracle itself departs on are left out.
    Costs of the rest by `within`; under u_zero_I the masked controls exactly 0.  idx: the oracle's batch rows that
    r holds.  Returns (tag, departing problems, compared problems, largest x / u error of the kept problems relative
    to the scale)."""
    sel = (lambda t: t) if idx is None else (lambda t: t[idx] if t.dim() == 1 else t[:, idx])
    x64, u64, c64 = (sel(t) for t in o64[:3])
    B = x64.shape[1]
    bounded = "u_lower" in kw
    sc = max(1.0, float(x64.abs().max()), float(u64.abs().max()))
    per = lambda a, b: (a.double() - b.double()).abs().amax((0, 2))  # noqa: E731
    differ = lambda a, b: (on_bounds(a, kw, sel) != on_bounds(b, kw, sel)).any(3).any(1).any(0)  # noqa: E731
    err = torch.maximum(per(r["x"], x64), per(r["u"], u64))
    out = torch.zeros(B, dtype=torch.bool)
    if o32 is None:
        tol = tol_for(F64, False)["xu"] * sc
    else:
        x32, u32 = sel(o32[0]), sel(o32[1])
        e32 = torch.maximum(per(x32, x64), per(u32, u64))
        out = e32 > 1e-4 * sc
        if bounded:
            out |= differ(u32, u64)
        assert not bool(out.all()), f"{tag}: no comparable problem"
        tol = 4 * float(e32[~out].max()) + 1e-6 * sc
    dep = err > tol
    if bounded:
        dep |= differ(r["u"], u64)
    dep &= ~out
    n_dep, n_cmp = int(dep.sum()), int((~out).sum())
    report = (tag, n_dep, n_cmp)
    allowed = max(1, n_cmp // 4) if bounded and lqr_iter > 1 else 0
    unexplained = n_dep
    if n_dep > allowed and allowed > 0 and o32 is None:
        unexplained = int((dep & ~sel(sensitive(tol))).sum())
        report = (tag + f" ({n_dep - unexplained} the oracle's own round-off moves)", n_dep, n_cmp)
    assert unexplained <= allowed, (f"{tag}: {n_dep} of {n_cmp} depart, {unexplained} of them where the oracle is "
                                    f"not round-off sensitive (allowed {allowed}), max err {float(err.max()):.3e} "
                                    f"tolerance {tol:.3e}")
    keep = ~(out | dep)
    within(tag, "costs", r["costs"][keep], c64[keep], None if o32 is None else sel(o32[2])[keep].double(), dtype)
    if "u_zero_I" in kw:
        mask = kw["u_zero_I"] if idx is None else kw["u_zero_I"][:, idx]
        assert bool((r["u"][mask] == 0).all()), f"{tag}: masked controls"
    return report + (float(err[keep].max()) / sc,)


@functools.lru_cache(maxsize=16)
def adjoint_case(seed, B, T, n, m, dtype, bounds, with_f, F_T=None):
    """A solved problem (one oracle step from u = 0, so box bounds leave an active set), upstream gradients,
    and the oracle's adjoint in float64 (and float32): (P, kw, ref64, ref32|None).  F_T=T: F carries T time slices
    (the oracle's dF then ends in a zero slice)."""
    C, c, F, f, x0 = gen_problem(seed, B, T, n, m, F64, with_f=with_f)
    F = F * 0.9
    if F_T == T:
        F = torch.cat((F, F[-1:]), 0) if T > 1 else gen_problem(seed, B, 2, n, m, F64)[2] * 0.9
    g = torch.Generator().manual_seed(seed)
    kw = {}
    if bounds == "box":
        kw = dict(u_lower=-0.25, u_upper=0.25)
    elif bounds == "tensor":
        kw = dict(u_lower=round_through(-0.5 * torch.rand(T, B, m, generator=g, dtype=F64) - 0.05, dtype),
                  u_upper=round_through(0.5 * torch.rand(T, B, m, generator=g, dtype=F64) + 0.05, dtype))
    C, c, F, f, x0 = (round_through(t, dtype) for t in (C, c, F, f, x0))
    u = torch.zeros(T, B, m, dtype=F64)
    o = orc.lqr_step_forward(n, m, T, x0, C, c, F, f, orc.get_traj(T, u, x0, F, f), u, coupled=False, **kw)
    x, u = round_through(o.new_x, dtype), round_through(o.new_u, dtype)
    wx = round_through(torch.randn(T, B, n, generator=g, dtype=F64), dtype)
    wu = round_through(torch.randn(T, B, m, generator=g, dtype=F64), dtype)
    P = dict(C=C, c=c, F=F, f=f, x0=x0, x=x, u=u, wx=wx, wu=wu)
    ref64 = orc.lqr_step_backward(n, m, T, x0, C, c, F, f, x, u, wx, wu, coupled=False, **kw)
    ref32 = None
    if dtype == F32:
        lo = lambda t: t.float() if torch.is_tensor(t) else t  # noqa: E731
        ref32 = orc.lqr_step_backward(n, m, T, lo(x0), lo(C), lo(c), lo(F), lo(f), lo(x), lo(u), lo(wx), lo(wu),
                                      coupled=False, **{k: lo(v) for k, v in kw.items()})
    return P, kw, ref64, ref32


def run_abi_adjoint(n, m, T, case, dtype, impl=None, F_T=None, poison=False):
    """abi_adjoint on the problem of an adjoint_case (with df where it has f) under MPCB200_KERNEL=impl."""
    P, kw, _, _ = case
    d = lambda t: to_dev(t, dtype)  # noqa: E731
    with kernel_env(impl):
        return abi_adjoint(n, m, T, d(P["C"]), d(P["c"]), d(P["F"]), d(P["x"]), d(P["u"]), d(P["wx"]), d(P["wu"]),
                           d(kw.get("u_lower")), d(kw.get("u_upper")), P["f"] is not None, F_T, poison)


def check_adjoint(tag, got, case, dtype):
    _, _, ref64, ref32 = case
    for i, name in enumerate(("dx_init", "dC", "dc", "dF", "df")):
        if got[i] is None:
            assert ref64[i].numel() == 0, f"{tag}: {name} missing"
            continue
        within(tag, name, got[i], ref64[i], ref32[i] if ref32 is not None else None, dtype)


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


def autograd_backward(n, m, T, P, kw, dtype, keys=("x0", "C", "c", "F", "f")):
    """LQRStepFn.backward through autograd (no_op_forward at the solution P["x"], P["u"]) with respect to P[keys]
    (F and f are None when not in keys): ([dx_init, dC, dc, dF, df] on the CPU, None where not asked, library
    launches)."""
    from mpc.pytorch_b200 import LQRStep, QuadCost, LinDx
    lv = [P[k].to(DEV, dtype).requires_grad_(True) for k in keys]
    F, f = (dict(zip(keys, lv)).get(k) for k in ("F", "f"))
    fn = LQRStep(n, m, T, true_cost=QuadCost(lv[1], lv[2]), true_dynamics=LinDx(F, f),
                 current_x=P["x"].to(DEV, dtype), current_u=P["u"].to(DEV, dtype), no_op_forward=True,
                 **{k: to_dev(v, dtype) for k, v in kw.items()})
    xo, uo = fn(lv[0], lv[1], lv[2], F, f)
    before = _L().launch_count()
    grads = torch.autograd.grad((xo, uo), lv, (P["wx"].to(DEV, dtype), P["wu"].to(DEV, dtype)))
    torch.cuda.synchronize()
    return [g.cpu() for g in grads] + [None] * (5 - len(grads)), _L().launch_count() - before


def check_step_fixed(tag, r, o, kw, dtype):
    """A step under the fixed tolerances of `tol_for` (on the scale of new_x), alphas bit exact.  float32 bounded
    cases may flag one problem whose QP stopped at the cap because its |dx| < 1e-4 test is decided by round-off
    (tests/test_step_gpu.py explains); that problem leaves the pnqp comparison."""
    bounded = kw.get("u_lower") is not None
    tol = tol_for(dtype, bounded)
    scale = max(1.0, float(o.new_x.abs().max()))
    for k in ("new_x", "new_u", "Ks", "ks"):
        assert maxdiff(r[k], getattr(o, k)) <= tol["xu"] * scale, f"{tag}: {k}"
    assert maxdiff(r["costs"], o.costs) <= tol["cost"] * max(1.0, float(o.costs.abs().max())), f"{tag}: costs"
    assert maxdiff(r["alphas"], o.alphas) == 0.0, f"{tag}: alphas"
    flagged = (r["status"] & 1) != 0
    if dtype == F64 or not bounded:
        assert not bool(flagged.any()), f"{tag}: pnqp flagged unconverged"
    else:
        assert int(flagged.sum()) <= 1 and bool((r["qp_iters"][:, flagged] == 19).any(0).all()), f"{tag}: cap flag"
    check_pnqp(tag, r, o, kw, keep=~flagged)
    check_clamps(tag, r, o, kw, keep=~flagged)
    if bounded:
        lo, hi = (kw[k] if torch.is_tensor(kw[k]) else torch.full_like(o.new_u, kw[k]) for k in ("u_lower", "u_upper"))
        assert bool(((r["new_u"] >= lo) & (r["new_u"] <= hi)).all()), f"{tag}: controls outside the bounds"


# ------------------------------------------------------------------------------------------------------------------
# the kernels' switch horizons, found on the device
# ------------------------------------------------------------------------------------------------------------------
INSTANCES = [(1, 1), (2, 1), (2, 2), (3, 1), (3, 2), (3, 4), (4, 1), (4, 2), (4, 4), (5, 1), (6, 2), (7, 4), (8, 1),
             (8, 2), (8, 4), (12, 4), (16, 4)]
PAIR_SHAPES = [s for s in INSTANCES if s[0] % 2 == 0 and s[1] % 2 == 0]
KREDUCE_SHAPES = {(16, 4)}          # one problem per warp, n a power of two
TMAX = 1024                         # switches are searched in [1, TMAX]
ORACLE_TMAX = 900                   # oracle comparisons at switches up to this horizon
PROBE_B = 8                         # one warp of every mapping; 16-byte aligned spans for every shape and dtype


def plan_str(p):
    L = _L()
    if p == 0:
        return "none"
    s = "generic" if p & L.PLAN_GENERIC else "pair"
    s += "/smem" if p & L.PLAN_GAINS_SMEM else "/Ks"
    return s + ("+kreduce" if p & L.PLAN_KREDUCE else "")


def plan(generic, smem, kreduce=False):
    L = _L()
    return ((L.PLAN_GENERIC if generic else L.PLAN_PAIR) | (L.PLAN_GAINS_SMEM if smem else 0)
            | (L.PLAN_KREDUCE if kreduce else 0))


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


def probe_step(n, m, dtype, T, impl, want_gains, do_rollout=True):
    """Plan of one step launch at horizon T; 0 if the library refused it for lack of shared memory."""
    from mpc.pytorch_b200.step import lqr_step_raw
    C, c, F, x, u = _probe_inputs(n, m, dtype)
    with kernel_env(impl):
        try:
            lqr_step_raw(n, m, T, x[0], C[:T], c[:T], F[:T - 1], None, x[:T], u[:T], do_rollout=do_rollout,
                         want_gains=want_gains, want_stats=False)
        except _L().MpcB200Error as e:
            if "[4]" in str(e):
                return 0
            raise
        return _L().last_step_plan()


def probe_adjoint(n, m, dtype, T):
    """Launches of one mpcb200_lqr_adjoint_* call at horizon T: 2 fused, 4 in-library 3-launch route, 0 if the
    library refused it for lack of shared memory."""
    C, c, F, x, u = _probe_inputs(n, m, dtype)
    try:
        _, launches = abi_adjoint(n, m, T, C[:T], c[:T], F[:T - 1], x[:T], u[:T], x[:T], u[:T], with_f=False)
    except _L().MpcB200Error as e:
        if "[4]" in str(e):
            return 0
        raise
    return launches


def first_true(pred, lo=0, hi=TMAX):
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
        generic=first_true(lambda T: not probe_step(n, m, dtype, T, 1, True) & L.PLAN_GAINS_SMEM),
        generic_riccati=first_true(lambda T: not probe_step(n, m, dtype, T, 1, True, False) & L.PLAN_GAINS_SMEM),
        pair=None, pair_nofit=None, adjoint=None)
    if (n, m) in PAIR_SHAPES:
        out["pair"] = first_true(lambda T: not probe_step(n, m, dtype, T, 2, True) & L.PLAN_GAINS_SMEM)
        out["pair_nofit"] = first_true(lambda T: not probe_step(n, m, dtype, T, 2, True, False) & L.PLAN_GAINS_SMEM)
        out["adjoint"] = first_true(lambda T: probe_adjoint(n, m, dtype, T) != 2)
    return out


@functools.lru_cache(maxsize=None)
def _pair_default(n, m, dtype):
    """Whether the default dispatch runs the column-pair kernel at this instance (asked of the device)."""
    return bool(probe_step(n, m, dtype, 2, None, False) & _L().PLAN_PAIR)


def loop_plan(n, m, dtype, T, impl):
    """The plan the loop body's step records at horizon T under MPCB200_KERNEL=impl; None where the step refuses.
    The loop hands the step a Ks/ks workspace from the generic kernel's switch horizon on (mpcb200_ilqr_workspace
    asks mpcb200_step_prefers_workspace); below it the gains must fit shared memory."""
    L = _L()
    if impl == 3 or (n, m) not in INSTANCES:
        return L.PLAN_LARGE
    sw = switches(n, m, dtype)
    ws = sw["generic"] is not None and T >= sw["generic"]
    if impl == 2 or (impl is None and _pair_default(n, m, dtype)):
        if ws:
            return plan(False, sw["pair"] is None or T < sw["pair"])
        if sw["pair_nofit"] is None or T < sw["pair_nofit"]:
            return plan(False, True)
        if impl == 2:
            return None                 # the pair kernel refuses: no workspace and the gains do not fit
    return plan(True, not ws, ws and (n, m) in KREDUCE_SHAPES)


def plan_name(p, impl, n, m, dtype):
    """The loop's step plan p by name: refused, large, pair_smem, pair_ks, pair_fallback (the generic kernel with
    gains in shared memory where the default dispatch would run the pair kernel), generic_smem, generic_kreduce,
    generic_ks."""
    L = _L()
    if p is None:
        return "refused"
    if p == L.PLAN_LARGE:
        return "large"
    if p & L.PLAN_PAIR:
        return "pair_smem" if p & L.PLAN_GAINS_SMEM else "pair_ks"
    if p & L.PLAN_GAINS_SMEM:
        return "pair_fallback" if impl is None and _pair_default(n, m, dtype) else "generic_smem"
    return "generic_kreduce" if p & L.PLAN_KREDUCE else "generic_ks"


SWITCH_PLANS = {"generic": ("generic_smem", "generic_ks"), "kreduce": ("generic_smem", "generic_kreduce"),
                "pair": ("pair_smem", "pair_ks"), "fallback": ("pair_smem", "pair_fallback")}


@functools.lru_cache(maxsize=None)
def pick_switch(group, dtype, augmentable=False):
    """(n, m, T*, impls) of the instance whose `group` switch of the loop's step plan comes first, None if no
    instance has it within ORACLE_TMAX.  Below T* the loop runs SWITCH_PLANS[group][0], from T* on [1].
    augmentable: only instances with n > m, the slew-rate augmented shapes of the systems (n - m, m)."""
    cands = []
    for n, m in INSTANCES:
        if augmentable and n <= m:
            continue
        sw = switches(n, m, dtype)
        pair = (n, m) in PAIR_SHAPES
        impls = (None, 1, 2) if pair else (None, 1)
        Ts, impl = None, 1
        if group == "generic" and (n, m) not in KREDUCE_SHAPES:
            Ts = sw["generic"]
        elif group == "kreduce" and (n, m) in KREDUCE_SHAPES:
            Ts = sw["generic"]
        elif group == "pair" and pair and sw["generic"] is not None and sw["pair"] is not None:
            Ts, impl = max(sw["generic"], sw["pair"]), 2
        elif group == "fallback" and pair and sw["pair_nofit"] is not None and _pair_default(n, m, dtype):
            if sw["generic"] is None or sw["pair_nofit"] < sw["generic"]:
                Ts, impl, impls = sw["pair_nofit"], None, (None, 1)
        if Ts is None or Ts < 3 or Ts > ORACLE_TMAX:
            continue
        below, at = (plan_name(loop_plan(n, m, dtype, T, impl), impl, n, m, dtype) for T in (Ts - 1, Ts))
        if (below, at) == SWITCH_PLANS[group]:
            cands.append((Ts, n + m, n, m, impls))
    if not cands:
        return None
    Ts, _, n, m, impls = min(cands)
    return n, m, Ts, impls


# ------------------------------------------------------------------------------------------------------------------
# receding-horizon episodes through the library's own staging (step._stage_episode, step._stage_episode_backward)
# ------------------------------------------------------------------------------------------------------------------
def _owned(poison, *shape, dtype):
    """A caller-owned buffer: every byte 0xFF when `poison` (NaN in float32 and float64, -1 in int32), else empty."""
    t = torch.empty(shape, dtype=dtype, device=DEV)
    if poison:
        t.view(torch.uint8).fill_(255)
    return t


def _owned_alloc(poison, nan_outputs):
    """The staging's alloc hook: the workspace (the one byte buffer) _owned when `poison`, every output when `poison`
    or `nan_outputs`."""
    return lambda shape, dtype: _owned(poison or (nan_outputs and dtype != torch.uint8), *shape, dtype=dtype)


def abi_episode(n, m, T, n_steps, x_init, C, c, F, f, u_init, u_lower=None, u_upper=None, u_zero_I=None,
                delta_u=None, linesearch_decay=0.2, max_linesearch_iter=10, lqr_iter=10, not_improved_lim=5,
                eps=1e-7, best_cost_eps=1e-4, dyn=None, poison=False, n_prev=0, plant=None, w=None,
                nan_outputs=False, window=None):
    """step.episode_raw(..., keep_plans=True): the call its staging makes (step._stage_episode: mpcb200_episode_plans_*,
    mpcb200_episode_plant_* with a plant or w, mpcb200_episode_window_* with window = L, the time-varying episode
    whose inputs lie on the axis of L slices), with caller-owned outputs and workspace.  poison: every workspace
    byte and every output starts at 0xFF, so a kernel that reads an element nothing wrote reads NaN (or info -1);
    nan_outputs: the outputs alone start at 0xFF, so an element the call does not write comes back NaN (or -1).
    n_prev: a slew-rate penalty's augmented problem, recorded in the staged problem for abi_episode_backward.  plant
    ("lin", F_p, f_p) of a LinDx plant (f_p None: none) or (kind, params) of a known one, and w [n_steps, B, n] (plant
    None with w: the model steps, disturbed).  Returns (res, launches, plan): res as episode_raw's dict, "saved"
    included, launches the library kernels the call recorded, plan mpcb200_last_step_plan() after it (the step plan of
    the solve)."""
    from mpc.pytorch_b200 import step as S
    from mpc.pytorch_b200.dynamics import DYN_LINEAR
    L = _L()
    if plant is not None:
        plant = (DYN_LINEAR, None, plant[1], plant[2]) if plant[0] == "lin" else (plant[0], plant[1], None, None)
    s, name, args, out = S._stage_episode(
        n, m, T, n_steps, x_init, C, c, F, f, u_init, u_lower, u_upper, u_zero_I, delta_u, linesearch_decay,
        max_linesearch_iter, lqr_iter, not_improved_lim, eps, best_cost_eps, dyn=dyn, keep_plans=True, n_prev=n_prev,
        plant=plant, w=w, window=window, alloc=_owned_alloc(poison, nan_outputs))
    before = L.launch_count()
    rc = S._call(name, C.dtype, DEV, args)
    launches, p = L.launch_count() - before, L.last_step_plan()
    torch.cuda.synchronize()
    res = S._episode_result(rc, name, s, out)
    assert res is not None, "the driver has no conditional graph nodes"
    return res, launches, p


def abi_episode_backward(saved, dl_dxs, dl_dus, poison=False, nan_outputs=False):
    """step.episode_backward_raw: the call its staging makes (step._stage_episode_backward:
    mpcb200_episode_backward_plant_* when the staged problem records a plant, mpcb200_episode_backward_slew_* when it
    records n_prev > 0, else mpcb200_episode_backward_*), with caller-owned outputs and workspace, poison as in
    abi_episode.  Returns ((dx_init, dC, dc, dF, df, dtheta) as episode_backward_raw returns them, and for a plant
    four more: dF_p [B, n, p], df_p [B, n] (None without the plant's f), dtheta_p [B, NP_plant] and dw
    [n_steps, B, n] (None without w); launches, plan): plan is the nested step's, recorded in the sweep's body.  Under
    a slew-rate penalty every size is the augmented problem's."""
    from mpc.pytorch_b200 import step as S
    L = _L()
    name, args, out = S._stage_episode_backward(saved, dl_dxs, dl_dus, alloc=_owned_alloc(poison, nan_outputs))
    before = L.launch_count()
    rc = S._call(name, saved[2].dtype, DEV, args)
    L.check(rc, name)
    launches, p = L.launch_count() - before, L.last_step_plan()
    torch.cuda.synchronize()
    g = S._episode_grads(saved[0], out)
    return (g if saved[0].plant is not None else g[:6]), launches, p


def _episode_per_problem(a, b):
    """max |a - b| per problem of [S, B, k] tensors -> [B]."""
    return (a.double() - b.double()).abs().amax((0, 2))


def _episode_on_bounds(u, kw):
    """[2, S, B, m]: which applied controls u [S, B, m] sit on the lower / upper bound (each solve's bound at t = 0)."""
    at0 = lambda b: b[0] if torch.is_tensor(b) else b  # noqa: E731
    return torch.stack([u.double() == torch.as_tensor(at0(kw[k]), dtype=F64) for k in ("u_lower", "u_upper")])


def check_episode_forward(tag, r, o64, o32, kw, dtype, several):
    """x, u, costs, info, u_next and the plans of the device episode against the oracle's, problem by problem, under
    test_ilqr_oracle_gpu.check_loop's rule.  A problem departs where its x, u, u_next, plan_x or plan_u misses the
    tolerance, or where its applied controls on a bound differ from the oracle's bit for bit.  The plans' later
    controls are held to the value tolerance only: they are T times as many pnqp end points, whose landing exactly on
    a bound or within 1e-8 of it round-off decides often enough that a bitwise rule over every plan left more than
    one problem in four at (3,2), (6,2) and (8,2) with 5 control steps and tensor bounds.  Only bounded episodes of
    more than one solve iteration (`several`: lqr_iter > 1, or more than one control step, whose solves start from
    states and warm starts that carry the earlier solves' round-off) may have departing problems, at most one in
    four: there pnqp's |dx| >= 1e-4 stop and its Armijo test decide some problems' paths by round-off.  float32
    problems whose float32 oracle departs from the float64 one are left out.  costs by the `within` policy over the
    rest.  Returns (largest x / u / u_next / plan error of the problems kept, relative to max(1, max|x|, max|u|),
    departing problems, compared problems)."""
    x, u = r["x"].cpu(), r["u"].cpu()
    B = x.shape[1]
    bounded = "u_lower" in kw
    sc = max(1.0, float(o64.x.abs().max()), float(o64.u.abs().max()))
    s, _, _, _, plan_x, plan_u = r["saved"]
    got = (x, u, r["u_next"].cpu(), s.pad.crop_n(plan_x).cpu(), s.pad.crop_m(plan_u).cpu())

    def per_problem(a, o):              # x, u, u_next and each solve's best iterate (the sweep's linearisation points)
        e = [_episode_per_problem(a[i], w) for i, w in enumerate((o.x, o.u, o.u_next))]
        e += [(a[i].double() - w.double()).abs().amax((0, 1, 3)) for i, w in ((3, o.plan_x), (4, o.plan_u))]
        return torch.stack(e).amax(0)

    def bounds_differ(a, b):            # [B]: a problem's applied controls on a bound differ
        return (_episode_on_bounds(a, kw) != _episode_on_bounds(b, kw)).any(3).any(1).any(0)
    err = per_problem(got, o64)
    out = torch.zeros(B, dtype=torch.bool)
    if o32 is None:
        tol = 1e-9 * sc
    else:
        e32 = per_problem((o32.x, o32.u, o32.u_next, o32.plan_x, o32.plan_u), o64)
        out = e32 > 1e-4 * sc
        if bounded:
            out |= bounds_differ(o32.u, o64.u)
        assert not bool(out.all()), f"{tag}: no comparable problem"
        tol = 4 * float(e32[~out].max()) + 1e-6 * sc
    dep = err > tol
    if bounded:
        dep |= bounds_differ(u, o64.u)
    dep &= ~out
    n_dep, n_cmp = int(dep.sum()), int((~out).sum())
    allowed = max(1, n_cmp // 4) if bounded and several else 0
    assert n_dep <= allowed, (f"{tag}: {n_dep} of {n_cmp} problems depart from the oracle (allowed {allowed}), "
                              f"largest x/u/u_next/plan error {float(err[~out].max()):.3e}, tolerance {tol:.3e}")
    keep = ~(out | dep)
    assert bool(keep.any()), f"{tag}: no comparable problem"
    within(tag, "costs", r["costs"].cpu()[:, keep], o64.costs[:, keep],
           None if o32 is None else o32.costs[:, keep], dtype)
    want = o64.iters if o32 is None else o32.iters
    assert r["info"][:, 0].cpu().tolist() == want, f"{tag}: iterations {r['info'][:, 0].tolist()} vs {want}"
    if "u_zero_I" in kw:
        assert bool((u[:, kw["u_zero_I"][0]] == 0).all()), f"{tag}: masked controls"
    return float(err[keep].max()) / sc, n_dep, n_cmp


def episode_linear_inputs(seed, B, T, n, m, dtype, mode, F_T=None, f_T="T-1", time_invariant=(), L=None):
    """A LinDx episode's inputs, float64 rounded through dtype, and the solver's problem options: (P, kw).
    mode: plain | box (+-0.25) | tensor (tensor box) | boxT (tensor box + delta_u) | mask (u_zero_I).  F_T = T: F has
    T slices; f_T: "none", "T-1" or "T" slices of f.  time_invariant: names among "F", "C", "c" whose slices all
    equal slice 0; P holds them dense (what the oracle takes), and P["time_invariant"] names them, so that
    episode_device_inputs hands them over as stride-0 views over time made on the device.
    L: a time-varying episode's axis (episode_raw(..., window=L)): C, c and tensor bounds have L slices, F and f L-1
    (L with F_T = T, f_T = "T"), each slice its own (F too); u_zero_I stays the solve's [T, B, m]."""
    Ta = T if L is None else L
    C, c, F, f, x0 = gen_problem(seed, B, Ta, n, m, F64, time_varying=L is not None)
    F = 0.9 * F
    g = torch.Generator().manual_seed(seed + 1)
    if F_T == T:
        F = torch.cat((F, F[-1:]), 0)
    if f_T == "T":
        f = torch.cat((f, f[-1:]), 0)
    elif f_T == "none":
        f = None
    P = dict(C=C, c=c, F=F, f=f, x0=x0)
    for k in time_invariant:
        P[k] = P[k][:1].expand(P[k].shape).contiguous()
    kw = {}
    if mode == "box":
        kw = dict(u_lower=-0.25, u_upper=0.25)
    elif mode in ("tensor", "boxT"):
        kw = dict(u_lower=-0.5 * torch.rand(Ta, B, m, generator=g, dtype=F64) - 0.05,
                  u_upper=0.5 * torch.rand(Ta, B, m, generator=g, dtype=F64) + 0.05)
        if mode == "boxT":
            kw["delta_u"] = 0.125
    elif mode == "mask":
        kw["u_zero_I"] = torch.rand(T, B, m, generator=g) < 0.3
    P = {k: round_through(v, dtype) for k, v in P.items()}
    P["time_invariant"] = tuple(time_invariant)
    kw = {k: round_through(v, dtype) for k, v in kw.items()}
    return P, kw


def episode_device_inputs(P, dtype):
    """x0, C, c, F, f of an episode_linear_inputs problem on DEV in dtype.  A time-invariant input is slice 0 moved
    to the device and expanded there (a copy of an expanded tensor, .to() included, is dense), so the shim stages it
    with time stride 0 (MPCB200_TIME_INVARIANT)."""
    out = []
    for k in ("x0", "C", "c", "F", "f"):
        t = P[k]
        if t is not None and k in P.get("time_invariant", ()):
            t = to_dev(t[:1], dtype).expand(t.shape)
        else:
            t = to_dev(t, dtype)
        out.append(t)
    return out


def epgrad_launches(route, known, window=False):
    """Library kernels an mpcb200_episode_backward_* call records (api.cu epgrad_record): the init, stage and
    accumulate kernels; a known system's linearisation and its VJP; the adjoint: prep + fused column-pair kernel, or
    prep, fill_zero, masked step and the two gradient kernels on every three-launch route.  window
    (mpcb200_episode_backward_window_*): one more, the body's window_stage_kernel."""
    return 3 + (2 if known else 0) + (2 if route == "fused" else 5) + (1 if window else 0)


def episode_window_bounds(kw, n_steps):
    """kw for check_episode_forward on a time-varying episode: each solve's t = 0 bound is slice k of a windowed
    tensor bound [L, B, m], so a tensor bound becomes [1, n_steps, B, m] (its slice 0 holds solve k's at k); scalar
    bounds and the other options as they are."""
    return {k: v[:n_steps].unsqueeze(0) if k in ("u_lower", "u_upper") and torch.is_tensor(v) else v
            for k, v in kw.items()}


def episode_known_module(name):
    """(module, clamp) of the episodes' known systems: cartpole (params (9.81, 1.3, 0.25, 0.8), force_mag 6),
    pendulum ((10, 1, 1)) and the five-parameter pendulum ((10, 1, 1, 0.1, 0.05)), max_torque 2; float64 params, as
    oracle/make_golden_receding_grad.py builds the reference's."""
    from mpc.pytorch_b200.dynamics import CartpoleDx, PendulumDx
    if name == "cartpole":
        mod = CartpoleDx(params=torch.tensor((9.81, 1.3, 0.25, 0.8), dtype=F64))
        mod.force_mag = 6.0
    elif name == "pendulum":
        mod = PendulumDx(params=torch.tensor((10.0, 1.0, 1.0), dtype=F64))
    else:
        mod = PendulumDx(params=torch.tensor((10.0, 1.0, 1.0, 0.1, 0.05), dtype=F64), simple=False)
    clamp = mod.force_mag if name == "cartpole" else mod.max_torque
    return mod, float(clamp)


def episode_known_step(mod):
    """The oracle's step(x, u, theta): the module's CPU torch forward with per-problem parameters theta [B, NP]."""
    def step(x, u, theta):
        mod.params = theta.t()
        return mod(x, u)
    return step


def episode_known_inputs(name, B, T, dtype, seed):
    """A known system's episode: (module, n, m, P, bounds at the clamp, dyn = (kind, params), theta [NP]).  The
    module's own cost; states with the angle pair on the unit circle."""
    from mpc.pytorch_b200.dynamics import DYN_NPARAMS
    mod, clamp = episode_known_module(name)
    n, m = mod.n_state, mod.n_ctrl
    q, p = mod.get_true_obj()
    g = torch.Generator().manual_seed(seed)
    th = (torch.rand(B, generator=g, dtype=F64) * 2 - 1) * (3.0 if name == "cartpole" else 1.0)
    if name == "cartpole":
        x0 = torch.stack((torch.rand(B, generator=g, dtype=F64) - 0.5, torch.rand(B, generator=g, dtype=F64) - 0.5,
                          th.cos(), th.sin(), torch.rand(B, generator=g, dtype=F64) - 0.5), 1)
    else:
        x0 = torch.stack((th.cos(), th.sin(), torch.rand(B, generator=g, dtype=F64) - 0.5), 1)
    P = dict(C=torch.diag(q.double()).expand(T, B, n + m, n + m).contiguous(),
             c=p.double().expand(T, B, n + m).contiguous(), x0=x0, F=None, f=None)
    P = {k: round_through(v, dtype) for k, v in P.items()}
    dyn = (mod.mpcb200_kind, mod.mpcb200_params())
    theta = torch.tensor(dyn[1][:DYN_NPARAMS[mod.mpcb200_kind]], dtype=F64)
    return mod, n, m, P, dict(u_lower=-clamp, u_upper=clamp), dyn, theta


# ------------------------------------------------------------------------------------------------------------------
# MPC.forward on the device loop or on the host loop
# ------------------------------------------------------------------------------------------------------------------
Solve = namedtuple("Solve", "x u costs full_du_norm iters grads")


def solve_on(monkeypatch, make, x0, cost, dx, device_loop, grads=()):
    """make()(x0, cost, dx) on the device loop (asserting that its predicate, _use_device_loop or, for a slew-rate
    penalty, _use_slew_device_loop, picks it) or on the host loop, asserting that the chosen loop ran.  The gradients
    are those of x.sum() + u.sum() with respect to `grads`."""
    from mpc.pytorch_b200 import solver, step
    from mpc.pytorch_b200.solver import MPC
    ctrl = make()
    pred = "_use_device_loop" if ctrl.slew_rate_penalty is None else "_use_slew_device_loop"
    seen = {"host_iters": 0}
    with monkeypatch.context() as mp:
        if device_loop:
            u0 = torch.zeros(ctrl.T, x0.shape[0], ctrl.n_ctrl, dtype=x0.dtype, device=x0.device)
            assert getattr(solver, pred)(ctrl, x0, cost, dx, u0)
            real = step.ilqr_raw

            def spy(*a, **k):
                seen["res"] = real(*a, **k)
                return seen["res"]
            mp.setattr(step, "ilqr_raw", spy)
        else:
            mp.setattr(solver, pred, lambda *a: False)
            real_sub = MPC.solve_lqr_subproblem

            def count(self, *a, **k):
                if not k.get("no_op_forward", False):
                    seen["host_iters"] += 1
                return real_sub(self, *a, **k)
            mp.setattr(MPC, "solve_lqr_subproblem", count)
        real_host = MPC._ilqr_host

        def host(self, *a, **k):
            seen["best"] = real_host(self, *a, **k)
            return seen["best"]
        mp.setattr(MPC, "_ilqr_host", host)
        x, u, costs = make()(x0, cost, dx)
    assert ("res" in seen) == device_loop and ("best" in seen) != device_loop
    fdn = seen["res"]["full_du_norm"] if device_loop else seen["best"]["full_du_norm"]
    iters = int(seen["res"]["info"][0]) if device_loop else seen["host_iters"]
    gs = torch.autograd.grad(x.sum() + u.sum(), grads) if grads else ()
    torch.cuda.synchronize()
    return Solve(x, u, costs, fdn, iters, gs)


def same_on_both_loops(monkeypatch, make, x0, cost, dx, grads=()):
    """The host loop, then the device loop: x, u, costs, the iteration count and the gradients bit for bit.
    Returns (device, host) solves."""
    host = solve_on(monkeypatch, make, x0, cost, dx, False, grads)
    dev = solve_on(monkeypatch, make, x0, cost, dx, True, grads)
    for k, (a, b) in enumerate(zip(dev[:3], host[:3])):
        assert a.shape == b.shape and a.dtype == b.dtype, f"output {k}"
        assert torch.equal(a, b), f"output {k} {float((a - b).abs().max()):.3e}"
    assert dev.iters == host.iters >= 1, (dev.iters, host.iters)
    for k, (a, b) in enumerate(zip(dev.grads, host.grads)):
        assert torch.equal(a, b), f"gradient {k} {float((a - b).abs().max()):.3e}"
    return dev, host


# ------------------------------------------------------------------------------------------------------------------
# the standalone pnqp (csrc/pnqp.cu: one thread per QP for n <= 8, one thread block per QP above)
# ------------------------------------------------------------------------------------------------------------------
PNQP_ITER = 20


def gen_qp(seed, B, n):
    """The pnqp generator of oracle/make_golden.py: H = LL' + I/2, q ~ 2N(0,1), bounds in (-1,0) and (0,1),
    x_init ~ 0.3N(0,1); float64."""
    g = torch.Generator().manual_seed(seed)
    L = torch.randn(B, n, n, generator=g, dtype=F64)
    H = L @ L.transpose(1, 2) + 0.5 * torch.eye(n, dtype=F64)
    q = 2.0 * torch.randn(B, n, generator=g, dtype=F64)
    lo = -torch.rand(B, n, generator=g, dtype=F64)
    hi = torch.rand(B, n, generator=g, dtype=F64)
    x0 = 0.3 * torch.randn(B, n, generator=g, dtype=F64)
    return H, q, lo, hi, x0


def pnqp_raw(H, q, lo, hi, x0=None, n_iter=PNQP_ITER):
    """mpcb200_pnqp_* on dense [B,n] inputs: (x, H_free, If, iters, status) per problem, on the CPU."""
    B, n, _ = H.shape
    dt = H.dtype
    ins = [t.to(DEV).contiguous() for t in (H, q, lo.expand(B, n), hi.expand(B, n))]
    x0d = x0.to(DEV).contiguous() if x0 is not None else None
    x = torch.empty(B, n, dtype=dt, device=DEV)
    Hf = torch.empty(B, n, n, dtype=dt, device=DEV)
    If = torch.empty(B, n, dtype=torch.uint8, device=DEV)
    iters = torch.empty(B, dtype=torch.int32, device=DEV)
    status = torch.empty(B, dtype=torch.int32, device=DEV)
    lib = _L()
    fn = lib.entry("mpcb200_pnqp", dt)
    with lib._on_device(DEV):
        rc = fn(B, n, *[lib.ptr(t) for t in ins], lib.ptr(x0d), n_iter, lib.ptr(x), lib.ptr(Hf), lib.ptr(If),
                lib.ptr(iters), lib.ptr(status), lib.stream_handle(DEV))
    assert rc == 0, lib.lib().mpcb200_strerror(rc)
    torch.cuda.synchronize()
    return x.cpu(), Hf.cpu(), If.cpu(), iters.cpu().long(), status.cpu()


def check_qp_f64(got, want, tag):
    """float64 pnqp_raw outputs `got` against the oracle's (x, H_free, If, iters) `want`: x within
    1e-9 * max(1, |x|_inf), H_free within 1e-12, free sets and iteration counts exact."""
    x, Hf, If, iters, status = got
    xo, Ho, Ifo, ito = want
    scale = max(1.0, float(xo.abs().max()))
    assert maxdiff(x, xo) <= 1e-9 * scale, f"{tag}: x differs by {maxdiff(x, xo):.3g}"
    assert torch.equal(If.bool(), Ifo.bool()), f"{tag}: free set"
    assert torch.equal(iters, ito), f"{tag}: iterations {iters.tolist()} vs {ito.tolist()}"
    assert maxdiff(Hf, Ho) <= 1e-12, f"{tag}: H_free"
