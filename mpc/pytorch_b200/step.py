"""LQRStep: one box-constrained LQR step as a torch.autograd.Function over the C ABI.

Mirrors the reference factory ``LQRStep(...)`` (mpc/lqr_step.py:22-38, 409): same
keyword names, defaults, call signature ``(x_init, C, c, F, f)``, return arity and
shapes, and the same gradient tuple ``(dx_init, dC, dc, dF, df)`` (:407).  The
arithmetic runs in csrc/lqr_step.cuh and csrc/lqr_grad.cuh.
"""
import collections
import ctypes
import os
import threading

import torch
from torch.autograd import Function
from torch.nn import Module

from . import _lib
from ._lib import Dims, Params, MpcB200Error, _on_device, check, ptr, ptr_view, stream_handle
from .dynamics import DYN_CTRL_PASSTHROUGH, DYN_DIMS, DYN_LINEAR, DYN_NPARAMS, DYN_OWN_INSTANCE

PNQP_MAX_ITER = 20  # reference passes n_iter=20 (mpc/lqr_step.py:137)

# MPC's loop sets `_host_reads.defer` to a dict around its LQRStep calls: the per-step pnqp counters then stay
# on the device (no .item() per step) and MPC reads them with its own stop-test scalars.  Without it, a step that
# prints a pnqp warning counts it in `_host_reads.n_warned`, which MPC's loop resets per solve.  Thread local; the
# LQRStep(...) signature itself stays the reference's.
_host_reads = threading.local()


def _is_empty(t):
    return t is None or t.nelement() == 0


def _dense(t, dtype=None):
    """Dense, detached, right-dtype view of `t` (no copy and no new tensor object when it already is)."""
    if t is None:
        return None
    if dtype is not None and t.dtype != dtype:
        t = t.to(dtype)
    if t.requires_grad:
        t = t.detach()
    return t if t.is_contiguous() else t.contiguous()


def _validate(n, m, T, *named, F=None, f=None, bounds=(None, None), u_zero_I=None, dyn_kind=None, need_F=True):
    """Check, on tensor metadata alone, the tensors a raw call hands to the kernels; returns the batch size B.
    The kernels read raw device pointers: a wrong dtype, shape or device would be an out-of-bounds access, so fail
    here like the reference's indexing / eclamp size asserts would.  `named`: (name, tensor or None, layout), the
    layout one of "TBpp", "TBp", "TBn", "TBm", "Bn" (p = n+m).  The first tensor leads: the outputs are allocated in
    its dtype, and it fixes B and the device.  F [T-1|T,B,n,p] and f [T-1|T,B,n] may be absent or empty (F only for
    T = 1); tensor bounds and u_zero_I are [T,B,m].  `dyn_kind`: the call runs that known system's dynamics in the
    kernel, which needs the exact (n, m) instance _pick_instance gives that kind.  `need_F=False`: the call linearises
    a known system itself and takes no F."""
    lead_name, lead, lead_layout = named[0]
    if lead.dtype not in (torch.float32, torch.float64):
        raise MpcB200Error(f"unsupported dtype {lead.dtype}")
    if lead.dim() != len(lead_layout):
        raise MpcB200Error(f"{lead_name}: expected shape [{','.join(lead_layout)}], got {tuple(lead.shape)}")
    B, p = lead.shape[lead_layout.index("B")], n + m
    shape_of = {"TBpp": (T, B, p, p), "TBp": (T, B, p), "TBn": (T, B, n), "TBm": (T, B, m), "Bn": (B, n)}
    checked = []
    for name, t, layout in named:
        if t is not None:
            if t.shape != shape_of[layout]:
                raise MpcB200Error(f"{name}: expected shape {shape_of[layout]}, got {tuple(t.shape)}")
            checked.append((name, t))
    for name, t, shape in (("F", F, (B, n, p)), ("f", f, (B, n))):
        if not _is_empty(t):
            if t.shape[1:] != shape or t.shape[0] not in (T - 1, T):
                raise MpcB200Error(f"{name}: expected shape (T-1 or T, {', '.join(map(str, shape))}), "
                                   f"got {tuple(t.shape)}")
            checked.append((name, t))
    if _is_empty(F) and T > 1 and need_F:
        raise MpcB200Error("F is required for T > 1")
    u_lower, u_upper = bounds
    if (u_lower is None) != (u_upper is None):
        raise MpcB200Error("u_lower and u_upper must be given together")
    for name, t in (("u_lower", u_lower), ("u_upper", u_upper), ("u_zero_I", u_zero_I)):
        if isinstance(t, torch.Tensor):
            if t.shape != shape_of["TBm"]:
                raise MpcB200Error(f"{name}: expected shape {shape_of['TBm']}, got {tuple(t.shape)}")
            checked.append((name, t))
    if dyn_kind is not None and _pick_instance(n, m, lead.element_size(), dyn_kind) != (n, m):
        raise MpcB200Error("in-kernel dynamics need an exact (n_state, n_ctrl) kernel instance")
    dev = lead.device
    for name, t in checked:
        if t.device != dev:
            raise MpcB200Error(f"{name}: expected a tensor on {dev}, got {t.device}")
    if not lead.is_cuda:
        raise MpcB200Error("mpc.pytorch_b200 runs on CUDA tensors only (no CPU fallback)")
    return B


def _bounds(u_lower, u_upper, shape, dtype, dev, padded=False):
    """(kind, s_lo, s_hi, lo_t, hi_t) of the kernels' control box: none (0), two scalars (1) or two `shape` tensors
    (2).  A padded problem always takes tensors, which the caller widens: its padded controls get their own box."""
    if u_lower is None:
        return 0, 0.0, 0.0, None, None
    if isinstance(u_lower, float) and isinstance(u_upper, float) and not padded:
        return 1, u_lower, u_upper, None, None
    lo_t, hi_t = [torch.full(shape, b, dtype=dtype, device=dev) if isinstance(b, float) else _dense(b, dtype)
                  for b in (u_lower, u_upper)]
    return 2, 0.0, 0.0, lo_t, hi_t


def _time_strided(t, dtype):
    """(tensor, mpcb200_dims time-stride field) for a [T, B, ...] input WITHOUT materialising views whose
    [B, ...] slices are contiguous: dense -> 0; stride-0 over time (`x.unsqueeze(0).expand(T, ...)`, an LTI
    `F`, reference mpc/mpc.py:205-226) -> MPCB200_TIME_INVARIANT; any other 16-byte aligned time stride -> it.
    Everything else (batch-expanded, transposed, ...) is copied to a dense tensor, as before."""
    if t.dtype != dtype:
        t = t.to(dtype)
    if t.requires_grad:
        t = t.detach()
    if t.is_contiguous():
        return t, 0
    if t.dim() >= 2 and t.shape[0] > 0 and t[0].is_contiguous():
        st0 = t.stride(0)
        if st0 == 0:
            return t, -1
        if st0 > 0 and (st0 * t.element_size()) % 16 == 0:
            return t, st0
    return t.contiguous(), 0


# ----------------------------------------------------------------------------------------------
# padding to a compiled (n,m) instance (compatibility path for shapes without an exact kernel)
# ----------------------------------------------------------------------------------------------
_pairs_cache = None
_pick_cache = {}
_smem_fits_cache = {}


def _pick_instance(n, m, elem_size=4, kind=DYN_LINEAR):
    """The (N, M) kernel shape an (n, m) problem runs at: the smallest compiled instance that covers it (zero padded),
    else (n, m) itself on the large-shape kernels if they fit it in `elem_size`-byte elements.  A dynamics `kind` with
    a dynamics-only instance (DYN_OWN_INSTANCE: every passthrough kind, and DYN_PENDULUM_FULL) runs that instance,
    which exists at exactly that kind's (n, m) only."""
    if kind in DYN_OWN_INSTANCE or kind & DYN_CTRL_PASSTHROUGH:
        if DYN_DIMS.get(kind) != (n, m):
            raise MpcB200Error(f"dynamics kind {kind} has no kernel instance at (n_state={n}, n_ctrl={m})")
        return n, m
    key = (n, m, elem_size)
    hit = _pick_cache.get(key)
    if hit is not None:
        return hit
    hit = _pick_instance_uncached(n, m, elem_size)
    _pick_cache[key] = hit
    return hit


def _large_fits(n, m, elem_size):
    dims = Dims(B=1, T=1, n=n, m=m, F_T=0)
    return bool(_lib.lib().mpcb200_step_large_fits(ctypes.byref(dims), elem_size))


def large_limit(m, elem_size):
    """The largest n_state the large-shape kernels take with n_ctrl = m (0: none)."""
    n = 0
    while _large_fits(n + 1, m, elem_size):
        n += 1
    return n


def _pick_instance_uncached(n, m, elem_size=4):
    global _pairs_cache
    if _pairs_cache is None:
        _pairs_cache = _lib.supported_pairs()
    if (n, m) in _pairs_cache:
        return n, m
    cands = [(N + M, N, M) for (N, M) in _pairs_cache if N >= n and M >= m]
    if cands:
        _, N, M = min(cands)
        return N, M
    if _large_fits(n, m, elem_size):
        return n, m
    dtype = {4: "float32", 8: "float64"}.get(elem_size, f"{elem_size}-byte elements")
    nmax = large_limit(m, elem_size)
    limit = f"n_state <= {nmax} for n_ctrl={m}" if nmax else f"no n_state for n_ctrl={m}"
    raise MpcB200Error(
        f"(n_state={n}, n_ctrl={m}) exceeds every compiled kernel instance {_pairs_cache} and the shared-memory "
        f"limit of the large-shape kernel in {dtype} ({limit}, 227 KB per problem)")


class _Pad:
    """Embeds an (n,m) problem in an (N,M) one: padded states are 0 with zero dynamics/cost;
    padded controls get unit cost, zero linear term, no effect on the dynamics and bounds
    [-1,1], so they stay at 0, free, and contribute nothing to any output."""

    def __init__(self, n, m, N, M, device):
        self.n, self.m, self.N, self.M = n, m, N, M
        self.active = (N, M) != (n, m)
        self.idx = (torch.cat((torch.arange(n, device=device), N + torch.arange(m, device=device)))
                    if self.active else None)

    def mat_pp(self, C):          # [..., p, p] -> [..., P, P]
        out = C.new_zeros(*C.shape[:-2], self.N + self.M, self.N + self.M)
        out[..., self.idx[:, None], self.idx[None, :]] = C
        if self.M > self.m:
            d = torch.arange(self.N + self.m, self.N + self.M, device=C.device)
            out[..., d, d] = 1.0
        return out

    def vec_p(self, c):           # [..., p] -> [..., P]
        out = c.new_zeros(*c.shape[:-1], self.N + self.M)
        out[..., self.idx] = c
        return out

    def mat_np(self, F):          # [..., n, p] -> [..., N, P]
        out = F.new_zeros(*F.shape[:-2], self.N, self.N + self.M)
        out[..., : self.n, self.idx] = F
        return out

    # an exact instance (or None) passes through unchanged
    def vec_n(self, x):           # [..., n] -> [..., N]
        if not self.active or x is None:
            return x
        out = x.new_zeros(*x.shape[:-1], self.N)
        out[..., : self.n] = x
        return out

    def vec_m(self, u, fill=0.0):  # [..., m] -> [..., M], padded controls = fill
        if not self.active or u is None:
            return u
        out = u.new_full((*u.shape[:-1], self.M), fill)
        out[..., : self.m] = u
        return out

    def stage(self, t, dtype, widen):
        """(tensor, mpcb200_dims time-stride field) of a [T, B, ...] input (C, c, F, f); (None, 0) when it is absent
        or empty.  An exact instance keeps the time stride (_time_strided); a padded one reads a dense `widen` copy."""
        if t is None or t.nelement() == 0:
            return None, 0
        if not self.active:
            return _time_strided(t, dtype)
        return widen(_dense(t, dtype)), 0

    # the inverse of the widening, for outputs (None stays None)
    def crop_n(self, x):          # [..., N] -> [..., n]
        return x[..., : self.n] if self.active and x is not None else x

    def crop_m(self, u):          # [..., M] -> [..., m]
        return u[..., : self.m] if self.active and u is not None else u

    def crop_mn(self, K):         # [..., M, N] -> [..., m, n]
        return K[..., : self.m, : self.n] if self.active and K is not None else K

    def crop_p(self, c):          # [..., P] -> [..., p]
        return c[..., self.idx] if self.active else c

    def crop_pp(self, C):         # [..., P, P] -> [..., p, p]
        return C[..., self.idx[:, None], self.idx[None, :]] if self.active else C

    def crop_np(self, F):         # [..., N, P] -> [..., n, p]
        return F[..., : self.n, self.idx] if self.active and F is not None else F


# n_prev: an episode's slew-rate augmentation, the leading states that hold the previous control (0: none); plant: the
# _StagedPlant of an episode closed on a plant other than the model (None: the model steps it)
# window: the mpcb200_window record of a time-varying episode (episode_raw(..., window=L)), whose C, c, F, f and
# bounds are then the staged full-length inputs (the solve's own where the record does not window them)
# net: (mpcb200_mlp record, packed weights) of an episode planned with a learned model (mlp.episode_raw); disturbed:
# w was added to the network's own step (no plant: a staged plant records its own)
_Problem = collections.namedtuple("_Problem", "pad C c F f u_lower u_upper u_zero_I dims params n_prev plant window "
                                  "net disturbed", defaults=(0, None, None, None, False))
# rec: the mpcb200_plant record; F, f: a LinDx plant's slice 0 at the problem's (padded) sizes [B, N, N+M], [B, N]
# (f None without one), or in a time-varying episode its whole staged F_p, f_p; disturbed: w was added to its step
_StagedPlant = collections.namedtuple("_StagedPlant", "rec F f disturbed")


def _stage_plant(pad, plant, dtype, B, n, m, win=None):
    """The plant of episode_raw as the kernels take it (_StagedPlant, without w): (DYN_LINEAR, None, F_p, f_p) with
    F_p [T', B, n, n+m] and f_p [T', B, n] (or None / empty) of which slice 0 steps, widened like the model (_Pad); or
    (kind, params, None, None) of a known system (its passthrough kind under a slew-rate penalty), whose own (n, m)
    must be the staged instance's.  `win`: the mpcb200_window record of a time-varying episode, whose LinDx plant has
    F_p, f_p [L-1|L, B, ...] staged whole (slice k steps control step k; MPCB200_WIN_PLANT set in `win`).  Checked on
    metadata before anything runs."""
    kind, params, F_p, f_p = plant
    rec = _lib.Plant(kind=int(kind))
    if kind != DYN_LINEAR:
        if DYN_DIMS.get(kind) != (pad.N, pad.M):
            raise MpcB200Error(f"a plant of dynamics kind {kind} steps (n_state, n_ctrl) = {DYN_DIMS.get(kind)}, "
                               f"but the episode runs at {(pad.N, pad.M)}")
        for i, v in enumerate(params):
            rec.dyn[i] = float(v)
        return _StagedPlant(rec, None, None, False)
    lead = "T'" if win is None else f"{win.L - 1} or {win.L}"
    for name, t, shape in (("plant F", F_p, (B, n, n + m)), ("plant f", f_p, (B, n))):
        if name == "plant F" and t is None:
            raise MpcB200Error("a LinDx plant needs F")
        if not _is_empty(t) and (t.dim() != len(shape) + 1 or tuple(t.shape[1:]) != shape or
                                 (t.shape[0] < 1 if win is None else t.shape[0] not in (win.L - 1, win.L))):
            raise MpcB200Error(f"{name}: expected shape ({lead}, {', '.join(map(str, shape))}), got {tuple(t.shape)}")
    if win is not None:
        win.on |= _lib.WIN_PLANT
        Fp, win.Fp_tstride = pad.stage(F_p, dtype, pad.mat_np)
        fp, win.fp_tstride = pad.stage(f_p, dtype, pad.vec_n)
        rec.has_f = int(fp is not None)
        return _StagedPlant(rec, Fp, fp, False)
    F0 = _dense(F_p[:1], dtype)
    F0 = (pad.mat_np(F0) if pad.active else F0)[0].contiguous()
    f0 = None
    if not _is_empty(f_p):
        f0 = pad.vec_n(_dense(f_p[0], dtype)).contiguous()
        rec.has_f = 1
    return _StagedPlant(rec, F0, f0, False)


def _problem(n, m, T, B, dtype, dev, C=None, c=None, F=None, f=None, u_lower=None, u_upper=None, u_zero_I=None,
             delta_u=None, linesearch_decay=0.2, max_linesearch_iter=10, dyn=None):
    """A raw call's (n, m) problem as the kernels take it, at the instance it runs at (_pick_instance): the _Pad;
    C, c, F, f staged by _Pad.stage; the tensor bounds and u_zero_I (as a uint8 mask) widened for padded controls;
    and the Dims / Params of a step with a rollout, time strides included.  lqr_step_raw and ilqr_raw make the same
    call, so the iLQR graph hands each kernel what a host loop of raw calls hands it.  A call whose Dims differ sets
    those fields on the returned `dims`; the caller densifies and widens its x / u (_dense, _Pad.vec_n / vec_m)."""
    N, M = _pick_instance(n, m, dtype.itemsize, dyn[0] if dyn is not None else DYN_LINEAR)
    pad = _Pad(n, m, N, M, dev)
    (C_, tsC), (c_, tsc) = pad.stage(C, dtype, pad.mat_pp), pad.stage(c, dtype, pad.vec_p)
    (F_, tsF), (f_, tsf) = pad.stage(F, dtype, pad.mat_np), pad.stage(f, dtype, pad.vec_n)
    kind, s_lo, s_hi, lo_t, hi_t = _bounds(u_lower, u_upper, (T, B, m), dtype, dev, pad.active)
    zmask = (u_zero_I != 0).to(torch.uint8).contiguous() if u_zero_I is not None else None
    dims = Dims(B=B, T=T, n=N, m=M, F_T=F_.shape[0] if F_ is not None else T - 1, has_f=int(f_ is not None),
                bounds_kind=kind, has_zero_mask=int(zmask is not None), has_delta_u=int(delta_u is not None),
                max_ls_iter=int(max_linesearch_iter), pnqp_max_iter=PNQP_MAX_ITER, do_rollout=1,
                dynamics_kind=int(dyn[0]) if dyn is not None else 0,
                C_tstride=tsC, c_tstride=tsc, F_tstride=tsF, f_tstride=tsf)
    params = Params(u_lo=float(s_lo), u_hi=float(s_hi), delta_u=float(delta_u) if delta_u is not None else 0.0,
                    ls_decay=float(linesearch_decay))
    if dyn is not None:
        for i, v in enumerate(dyn[1]):
            params.dyn[i] = float(v)
    return _Problem(pad, C_, c_, F_, f_, pad.vec_m(lo_t, -1.0), pad.vec_m(hi_t, 1.0), pad.vec_m(zmask, 0),
                    dims, params)


def _grad_outputs(T, B, N, M, F, f_T, want_df, dtype, dev):
    """The (dx_init, dC, dc, dF, df) buffers the gradient kernels fill: dF like the staged F (None without one), df
    only when `want_df`, with f's leading dimension `f_T` (default T-1); the kernels write its slices < T-1, so a T-th
    slice (full-length f) is zeroed here."""
    P = N + M
    dx_init = torch.empty(B, N, dtype=dtype, device=dev)
    dC = torch.empty(T, B, P, P, dtype=dtype, device=dev)
    dc = torch.empty(T, B, P, dtype=dtype, device=dev)
    dF = torch.empty(F.shape[0], B, N, P, dtype=dtype, device=dev) if F is not None else None
    f_T = T - 1 if f_T is None else f_T
    df = torch.empty(f_T, B, N, dtype=dtype, device=dev) if want_df else None
    if want_df and f_T == T:
        df[T - 1].zero_()
    return dx_init, dC, dc, dF, df


# ----------------------------------------------------------------------------------------------
# raw calls (dense CUDA tensors in, fresh CUDA tensors out)
# ----------------------------------------------------------------------------------------------
def lqr_step_raw(n_state, n_ctrl, T, x_init, C, c, F, f, cur_x, cur_u,
                 u_lower=None, u_upper=None, u_zero_I=None, delta_u=None,
                 linesearch_decay=0.2, max_linesearch_iter=10, do_rollout=True,
                 want_gains=False, want_stats=True, want_du_first=False, dyn=None):
    """Run the step kernel.  Returns a dict of device tensors:
    new_x,new_u,costs,full_du_norm,alphas (do_rollout) and, on request, Ks,ks,qp_iters,
    free_mask,status."""
    n, m = n_state, n_ctrl
    B = _validate(n, m, T, ("C", C, "TBpp"), ("c", c, "TBp"), ("x_init", x_init, "Bn"), ("current_x", cur_x, "TBn"),
                  ("current_u", cur_u, "TBm"), F=F, f=f, bounds=(u_lower, u_upper), u_zero_I=u_zero_I,
                  dyn_kind=dyn[0] if dyn is not None else None)
    dtype, dev = C.dtype, C.device
    s = _problem(n, m, T, B, dtype, dev, C, c, F, f, u_lower, u_upper, u_zero_I, delta_u, linesearch_decay,
                 max_linesearch_iter, dyn)
    pad, dims, N, M = s.pad, s.dims, s.pad.N, s.pad.M
    dims.do_rollout = int(bool(do_rollout))
    x0_, cx_, cu_ = pad.vec_n(_dense(x_init, dtype)), pad.vec_n(_dense(cur_x, dtype)), pad.vec_m(_dense(cur_u, dtype))

    out = {}
    new_x = new_u = costs = fdn = alphas = None
    if do_rollout:
        new_x = torch.empty(T, B, N, dtype=dtype, device=dev)
        new_u = torch.empty(T, B, M, dtype=dtype, device=dev)
        costs = torch.empty(B, dtype=dtype, device=dev)
        fdn = torch.empty(B, dtype=dtype, device=dev)
        alphas = torch.empty(B, dtype=dtype, device=dev)
    du_first = None
    if do_rollout and want_du_first:
        du_first = torch.empty(T, B, M, dtype=dtype, device=dev)
    qp_iters = free_mask = status = None
    if want_stats:
        qp_iters = torch.zeros(T, B, dtype=torch.int32, device=dev) if dims.bounds_kind else None
        free_mask = torch.empty(T, B, M, dtype=torch.uint8, device=dev)
        status = torch.empty(B, dtype=torch.int32, device=dev)
    Ks = ks = None
    need_gains = want_gains or not do_rollout
    if not need_gains:
        # long horizons do not fit shared memory: the kernel then keeps gains in a caller buffer
        # the library's answer also depends on the MPCB200_KERNEL developer knob (3: the large kernels everywhere)
        key = (N, M, T, C.element_size(), os.environ.get("MPCB200_KERNEL"))
        fits = _smem_fits_cache.get(key)
        if fits is None:
            fits = not _lib.lib().mpcb200_step_prefers_workspace(ctypes.byref(dims), C.element_size())
            _smem_fits_cache[key] = fits
        need_gains = not fits
    if need_gains:
        Ks = torch.empty(T, B, M, N, dtype=dtype, device=dev)
        ks = torch.empty(T, B, M, dtype=dtype, device=dev)
    fn = _lib.entry("mpcb200_lqr_step", dtype)
    with _on_device(dev):
        rc = fn(ctypes.byref(dims), ctypes.byref(s.params), ptr_view(s.C), ptr_view(s.c), ptr_view(s.F),
                ptr_view(s.f), ptr(x0_), ptr(cx_), ptr(cu_), ptr(s.u_lower), ptr(s.u_upper), ptr(s.u_zero_I),
                ptr(new_x), ptr(new_u), ptr(costs), ptr(fdn), ptr(alphas), ptr(du_first), ptr(qp_iters),
                ptr(free_mask), ptr(status), ptr(Ks), ptr(ks), stream_handle(dev))
    check(rc, "mpcb200_lqr_step")
    if do_rollout:
        out.update(new_x=pad.crop_n(new_x), new_u=pad.crop_m(new_u), costs=costs, full_du_norm=fdn, alphas=alphas)
        if du_first is not None:
            out["du_first"] = pad.crop_m(du_first)
    if Ks is not None:
        out.update(Ks=pad.crop_mn(Ks), ks=pad.crop_m(ks))
    if want_stats:
        out.update(qp_iters=qp_iters, free_mask=pad.crop_m(free_mask), status=status)
    return out


def ilqr_raw(n_state, n_ctrl, T, x_init, C, c, F, f, u_init, u_lower=None, u_upper=None, u_zero_I=None,
             delta_u=None, linesearch_decay=0.2, max_linesearch_iter=10, lqr_iter=10, not_improved_lim=5, eps=1e-7,
             best_cost_eps=1e-4, dyn=None):
    """The iLQR iterations of MPC.forward (reference mpc/mpc.py:244-301) in ONE library call: a CUDA graph that runs
    rollout, [linearisation,] step, best-iterate tracking and the stop test until the stop test ends it, without a
    host read.  The dynamics are LinDx(F, f), or the known system `dyn` = (kind, params) with F = f = None.  The
    problem is staged once per solve, by the _problem call lqr_step_raw makes, so every kernel gets the values
    lqr_step_raw and rollout_raw would hand it per call.  Returns a dict of device tensors x, u, costs, full_du_norm
    (the best iterate) and info = int32 [iterations run, iterations with an unconverged pnqp]; None when the driver
    has no conditional graph nodes (nothing was launched then)."""
    n, m = n_state, n_ctrl
    B = _validate(n, m, T, ("C", C, "TBpp"), ("c", c, "TBp"), ("x_init", x_init, "Bn"), ("u_init", u_init, "TBm"),
                  F=F, f=f, bounds=(u_lower, u_upper), u_zero_I=u_zero_I,
                  dyn_kind=dyn[0] if dyn is not None else None, need_F=dyn is None)
    dtype, dev = C.dtype, C.device
    s = _problem(n, m, T, B, dtype, dev, C, c, F, f, u_lower, u_upper, u_zero_I, delta_u, linesearch_decay,
                 max_linesearch_iter, dyn)
    pad, dims, N, M = s.pad, s.dims, s.pad.N, s.pad.M
    x0_, u0_ = pad.vec_n(_dense(x_init, dtype)), pad.vec_m(_dense(u_init, dtype))
    opts = _lib.IlqrOpts(lqr_iter=int(lqr_iter), not_improved_lim=int(not_improved_lim), m_ref=m, eps=float(eps),
                         best_cost_eps=float(best_cost_eps))
    nbytes = _lib.lib().mpcb200_ilqr_workspace_bytes(ctypes.byref(dims), ctypes.byref(opts), C.element_size())
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    best_x = torch.empty(T, B, N, dtype=dtype, device=dev)
    best_u = torch.empty(T, B, M, dtype=dtype, device=dev)
    costs = torch.empty(B, dtype=dtype, device=dev)
    fdn = torch.empty(B, dtype=dtype, device=dev)
    info = torch.empty(2, dtype=torch.int32, device=dev)
    fn = _lib.entry("mpcb200_ilqr", dtype)
    with _on_device(dev):
        rc = fn(ctypes.byref(dims), ctypes.byref(s.params), ctypes.byref(opts), ptr_view(s.C), ptr_view(s.c),
                ptr_view(s.F), ptr_view(s.f), ptr(x0_), ptr(u0_), ptr(s.u_lower), ptr(s.u_upper), ptr(s.u_zero_I),
                ptr(best_x), ptr(best_u), ptr(costs), ptr(fdn), ptr(info), ptr(ws), nbytes, stream_handle(dev))
    if rc == _lib.ERR_NO_GRAPH_COND:
        return None
    check(rc, "mpcb200_ilqr")
    return {"x": pad.crop_n(best_x), "u": pad.crop_m(best_u), "costs": costs, "full_du_norm": fdn, "info": info}


def episode_raw(n_state, n_ctrl, T, n_steps, x_init, C, c, F, f, u_init, u_lower=None, u_upper=None, u_zero_I=None,
                delta_u=None, linesearch_decay=0.2, max_linesearch_iter=10, lqr_iter=10, not_improved_lim=5, eps=1e-7,
                best_cost_eps=1e-4, dyn=None, keep_plans=False, n_prev=0, plant=None, w=None, window=None):
    """A receding-horizon episode of n_steps control steps in ONE library call (mpcb200_episode_*): each step solves
    the problem from the current state as ilqr_raw does (u_init = the warm start), applies the plan's first control,
    steps the model (LinDx: F[0] [x; u] + f[0]; a known system `dyn`: one step of it) and shifts the warm start
    (cat(u[1:], 0), then w[-2] = w[-3]).  The problem is staged once per episode by the _problem call ilqr_raw makes.
    u_init None: zeros.  Returns a dict of device tensors x [n_steps+1, B, n], u [n_steps, B, m], costs
    [n_steps, B], info int32 [n_steps, 2] and u_next [T, B, m]; None when the driver has no conditional graph nodes
    or no conditional node inside another's body (nothing was launched then).  keep_plans: the call is
    mpcb200_episode_plans_*, and the dict also holds "saved", what episode_backward_raw takes: the staged problem and
    the padded xs, us and each solve's best iterate plan_x [n_steps, T, B, N], plan_u [n_steps, T, B, M].
    n_prev > 0: the problem is a slew-rate penalty's augmented one over [u_{k-1}; x_k] and its first n_prev states
    are the previous control; the staged problem records it, so episode_backward_raw detaches them.
    plant (mpcb200_episode_plant_*): what steps the loop instead of the model, (DYN_LINEAR, None, F_p, f_p) for a
    LinDx's t = 0 slice or (kind, params, None, None) for a known system (_stage_plant); w [n_steps, B, n]: added to
    each step, x_{k+1} = plant(x_k, u_k) + w_k (under a slew-rate penalty its first n_prev entries are the caller's
    zeros).  Either one takes that entry; the staged problem records the plant for episode_backward_raw.
    window = L (mpcb200_episode_window_*): a time-varying episode whose inputs lie on its time axis of
    L = n_steps + T - 1 slices (_window_problem).  _stage_episode stages the call."""
    s, name, args, out = _stage_episode(n_state, n_ctrl, T, n_steps, x_init, C, c, F, f, u_init, u_lower, u_upper,
                                        u_zero_I, delta_u, linesearch_decay, max_linesearch_iter, lqr_iter,
                                        not_improved_lim, eps, best_cost_eps, dyn=dyn, keep_plans=keep_plans,
                                        n_prev=n_prev, plant=plant, w=w, window=window)
    return _episode_result(_call(name, C.dtype, C.device, args), name, s, out)


def _stage_episode(n, m, T, n_steps, x_init, C, c, F, f, u_init, u_lower=None, u_upper=None, u_zero_I=None,
                   delta_u=None, linesearch_decay=0.2, max_linesearch_iter=10, lqr_iter=10, not_improved_lim=5,
                   eps=1e-7, best_cost_eps=1e-4, dyn=None, keep_plans=False, n_prev=0, plant=None, w=None,
                   window=None, net=None, alloc=None):
    """An episode's call as episode_raw (or, with `net`, mlp.episode_raw) makes it, staged but not made: (s, name,
    args, out).  s: the staged problem, which records n_prev, the plant, the window, the network and whether w was
    added; name: the entry (mpcb200_episode, _plans with keep_plans, _plant with a plant or w, _window with `window`,
    _mlp with `net`); args: its arguments in the header's order, a tensor standing for its device pointer (_call);
    out: (xs, us, costs, info, u_next, plan_x, plan_u), plan_x, plan_u None without keep_plans.  Every buffer, the
    workspace included, comes from alloc(shape, dtype) (default torch.empty on the inputs' device).
    net: the NNDynamics (or CtrlPassthroughDynamics) every solve plans with, F = f = dyn = None; without a plant the
    network steps the loop, and w is added to its step."""
    if T < 3 or n_steps < 1:
        raise MpcB200Error(f"an episode needs T >= 3 and n_steps >= 1, got T={T}, n_steps={n_steps}")
    if window is None:
        B = _validate(n, m, T, ("C", C, "TBpp"), ("c", c, "TBp"), ("x_init", x_init, "Bn"), ("u_init", u_init, "TBm"),
                      F=F, f=f, bounds=(u_lower, u_upper), u_zero_I=u_zero_I,
                      dyn_kind=dyn[0] if dyn is not None else None, need_F=dyn is None and net is None)
        s = _problem(n, m, T, B, C.dtype, C.device, C, c, F, f, u_lower, u_upper, u_zero_I, delta_u, linesearch_decay,
                     max_linesearch_iter, dyn)
    else:
        s = _window_problem(n, m, T, n_steps, window, x_init, C, c, F, f, u_init, u_lower, u_upper, u_zero_I, delta_u,
                            linesearch_decay, max_linesearch_iter, dyn)
    pad, dims, N, M, B = s.pad, s.dims, s.pad.N, s.pad.M, s.dims.B
    dtype, dev = C.dtype, C.device
    if net is not None:
        from .mlp import record
        net = record(net, C)
    x0_, u0_ = pad.vec_n(_dense(x_init, dtype)), pad.vec_m(_dense(u_init, dtype))
    if plant is None and w is not None and net is None:      # the model steps, disturbed
        plant = (DYN_LINEAR, None, F, f) if dyn is None else (dyn[0], dyn[1], None, None)
    sp = _stage_plant(pad, plant, dtype, B, n, m, s.window) if plant is not None else None
    w_ = None
    if w is not None:
        if tuple(w.shape) != (n_steps, B, n) or w.dtype != dtype or w.device != dev:
            raise MpcB200Error(f"w: expected a {dtype} tensor of shape {(n_steps, B, n)} on {dev}, got a "
                               f"{w.dtype} tensor of shape {tuple(w.shape)} on {w.device}")
        w_ = pad.vec_n(_dense(w, dtype)).contiguous()
        if sp is not None:
            sp = sp._replace(disturbed=True)
    s = s._replace(n_prev=int(n_prev), plant=sp, net=net, disturbed=w is not None and sp is None)
    opts = _lib.IlqrOpts(lqr_iter=int(lqr_iter), not_improved_lim=int(not_improved_lim), m_ref=m, eps=float(eps),
                         best_cost_eps=float(best_cost_eps))
    lib, esz = _lib.lib(), C.element_size()
    prec = ctypes.byref(sp.rec) if sp is not None else None
    if net is not None:
        name, recs = "mpcb200_episode_mlp", [ctypes.byref(net[0]), prec]
        nbytes = lib.mpcb200_episode_mlp_workspace_bytes(ctypes.byref(dims), ctypes.byref(opts), recs[0], esz)
        if nbytes == 0:
            raise MpcB200Error("mpcb200_episode_mlp: the episode has no workspace size (the network does not fit, or "
                               "bad dimensions)")
    elif s.window is not None:
        name, recs = "mpcb200_episode_window", [ctypes.byref(s.window), prec]
        nbytes = lib.mpcb200_episode_window_workspace_bytes(ctypes.byref(dims), ctypes.byref(opts), recs[0], esz)
    else:
        name = ("mpcb200_episode_plant" if sp is not None else
                "mpcb200_episode_plans" if keep_plans else "mpcb200_episode")
        recs = [prec] if sp is not None else []
        nbytes = lib.mpcb200_episode_workspace_bytes(ctypes.byref(dims), ctypes.byref(opts), esz)
    if alloc is None:
        def alloc(shape, dt):
            return torch.empty(shape, dtype=dt, device=dev)
    ws = alloc((nbytes,), torch.uint8)
    xs, us = alloc((n_steps + 1, B, N), dtype), alloc((n_steps, B, M), dtype)
    costs, info, u_next = alloc((n_steps, B), dtype), alloc((n_steps, 2), torch.int32), alloc((T, B, M), dtype)
    plan_x = plan_u = None
    if keep_plans:
        plan_x, plan_u = alloc((n_steps, T, B, N), dtype), alloc((n_steps, T, B, M), dtype)
    model = [s.C, s.c] if net is not None else [s.C, s.c, s.F, s.f]
    plant_in = [] if not recs else [sp.F if sp is not None else None, sp.f if sp is not None else None, w_]
    plans = [plan_x, plan_u] if name != "mpcb200_episode" else []
    args = [ctypes.byref(dims), ctypes.byref(s.params), ctypes.byref(opts), *recs, int(n_steps), *model, *plant_in,
            x0_, u0_, s.u_lower, s.u_upper, s.u_zero_I, xs, us, costs, info, u_next, *plans, ws, nbytes,
            stream_handle(dev)]
    return s, name, args, (xs, us, costs, info, u_next, plan_x, plan_u)


def _call(name, dtype, dev, args):
    """The status of the library entry `name` for `dtype` called with `args` on `dev`, each tensor in `args` passed as
    its device pointer (ptr_view: the staging made it dense, or validated its time stride)."""
    fn = _lib.entry(name, dtype)
    with _on_device(dev):
        return fn(*[ptr_view(a) if isinstance(a, torch.Tensor) else a for a in args])


def _episode_result(rc, name, s, out):
    """episode_raw's dict from the status of the call _stage_episode staged and its outputs; None when the driver has
    no conditional graph nodes.  "saved" where the plans were kept."""
    if rc == _lib.ERR_NO_GRAPH_COND:
        return None
    check(rc, name)
    xs, us, costs, info, u_next, plan_x, plan_u = out
    pad = s.pad
    res = {"x": pad.crop_n(xs), "u": pad.crop_m(us), "costs": costs, "info": info, "u_next": pad.crop_m(u_next)}
    if plan_x is not None:
        res["saved"] = (s, us.shape[0], xs, us, plan_x, plan_u)
    return res


def _window_problem(n, m, T, n_steps, L, x_init, C, c, F, f, u_init, u_lower, u_upper, u_zero_I, delta_u,
                    linesearch_decay, max_linesearch_iter, dyn):
    """The staged problem of a time-varying episode (episode_raw(..., window=L), mpcb200_episode_window_*).
    C [L, B, p, p], c [L, B, p], a LinDx model's F [L-1|L, B, n, p] and f [L-1|L, B, n], tensor bounds [L, B, m] and a
    LinDx plant's F_p, f_p [L-1|L, ...] lie on the episode's axis, L = n_steps + T - 1; u_init and u_zero_I are the
    solve's [T, B, m].  Solve k plans on slices k .. k+T-1 (F: k .. k+F_T-1, F_T = T - (L - len(F))), and control
    step k steps with slice k of a LinDx model or plant.  The per-solve problem is _problem's on the first window (its
    Dims, _Pad and widened u_zero_I); the full-length inputs are staged once, by the same _Pad widening, into its C, c,
    F, f and bounds, and the library copies each window on the device (the mpcb200_window record `window`)."""
    if L != n_steps + T - 1:
        raise MpcB200Error(f"window: a time-varying episode of {n_steps} steps at T={T} has an axis of "
                           f"{n_steps + T - 1} slices, got {L}")
    B = _validate(n, m, L, ("C", C, "TBpp"), ("c", c, "TBp"), ("x_init", x_init, "Bn"), F=F, f=f,
                  bounds=(u_lower, u_upper), dyn_kind=dyn[0] if dyn is not None else None, need_F=dyn is None)
    dtype, dev = C.dtype, C.device
    for name, t in (("u_init", u_init), ("u_zero_I", u_zero_I)):
        if t is not None and tuple(t.shape) != (T, B, m):
            raise MpcB200Error(f"{name}: expected shape {(T, B, m)}, got {tuple(t.shape)}")
    F_T = None if _is_empty(F) else T - (L - F.shape[0])

    def first(b):                         # the first window of a tensor bound
        return b[:T] if isinstance(b, torch.Tensor) else b
    s = _problem(n, m, T, B, dtype, dev, C[:T], c[:T], F[:F_T] if F_T else None, None if _is_empty(f) else f[:T - 1],
                 first(u_lower), first(u_upper), u_zero_I, delta_u, linesearch_decay, max_linesearch_iter, dyn)
    pad = s.pad
    rec = _lib.Window(L=int(L), on=_lib.WIN_COST)
    C_, rec.C_tstride = pad.stage(C, dtype, pad.mat_pp)
    c_, rec.c_tstride = pad.stage(c, dtype, pad.vec_p)
    F_, f_ = s.F, s.f
    if dyn is None:
        rec.on |= _lib.WIN_DYN
        F_, rec.F_tstride = pad.stage(F, dtype, pad.mat_np)
        f_, rec.f_tstride = pad.stage(f, dtype, pad.vec_n)
    lo_, hi_ = s.u_lower, s.u_upper
    if isinstance(u_lower, torch.Tensor) or isinstance(u_upper, torch.Tensor):
        rec.on |= _lib.WIN_BOUNDS
        _, _, _, lo_t, hi_t = _bounds(u_lower, u_upper, (L, B, m), dtype, dev, pad.active)
        lo_, hi_ = pad.vec_m(lo_t, -1.0).contiguous(), pad.vec_m(hi_t, 1.0).contiguous()
    return s._replace(C=C_, c=c_, F=F_, f=f_, u_lower=lo_, u_upper=hi_, window=rec)


def episode_backward_raw(saved, dl_dxs, dl_dus):
    """The reverse sweep of an episode run by episode_raw(..., keep_plans=True) in ONE library call
    (mpcb200_episode_backward_*): `saved` is that call's res["saved"], dl_dxs [n_steps+1, B, n] and dl_dus
    [n_steps, B, m] the gradients of its x and u.  Returns (dx_init [B, n], dC [T, B, p, p], dc [T, B, p], dF, df,
    dtheta): LinDx dF like the staged F's [F_T, B, n, p] and df like its f (None without f), dtheta None; a known
    system dF = df = None and dtheta [B, NP], one row per problem (the caller sums over b, as DynLinearize does).
    A slew-rate episode (the staged problem's n_prev > 0) runs mpcb200_episode_backward_slew_*: every size is the
    augmented problem's, and the first n_prev states of each augmented state get no gradient (dx_init[:, :n_prev] = 0);
    the caller crops the gradients to the system's own blocks.
    An episode closed on a plant (the staged problem's plant) runs mpcb200_episode_backward_plant_* and returns four
    more: dF_p [B, n, p] and df_p [B, n] (a LinDx plant's slice 0; df_p None without f), dtheta_p [B, NP_plant] (a
    known plant) and dw [n_steps, B, n] (None when no w was added); dF, df or dtheta are then the solves' part only.
    A time-varying episode (episode_raw(..., window=L)) runs mpcb200_episode_backward_window_*: dC, dc, dF, df and a
    windowed LinDx plant's dF_p, df_p are full length, with zero slices up to their inputs' lengths (slices no step
    reads).  _stage_episode_backward stages the call."""
    name, args, out = _stage_episode_backward(saved, dl_dxs, dl_dus)
    check(_call(name, saved[2].dtype, saved[2].device, args), name)
    g = _episode_grads(saved[0], out)
    return g if saved[0].plant is not None else g[:6]


def _stage_episode_backward(saved, dl_dxs, dl_dus, alloc=None):
    """The reverse sweep's call as episode_backward_raw (or mlp.episode_backward_raw) makes it, staged but not made:
    (name, args, out).  The entry is the network's (mpcb200_episode_backward_mlp) for an episode planned with one,
    else the window's, the plant's (a plant or w), the slew-rate penalty's (n_prev > 0) or the plain one; args and
    alloc as _stage_episode's.  out: the padded (dx_init, dC, dc, dF, df, dtheta, dF_p, df_p, dtheta_p, dw), None
    where the entry writes no such output: dF, df a LinDx model's (df with f, T-1 slices); dtheta a known system's
    [B, NP] or the network's [n_params]; dF_p, df_p a LinDx plant's, dtheta_p [B, NP_plant] a known plant's; dw where
    w was added.  dC, dc and df lie on a time-varying episode's axis of L slices, and so do a windowed LinDx plant's
    dF_p, df_p [L-1, B, ...]."""
    s, n_steps, xs, us, plan_x, plan_u = saved
    pad, dims, sp, win, net = s.pad, s.dims, s.plant, s.window, s.net
    B, N, P, k = dims.B, pad.N, pad.N + pad.M, int(s.n_prev)
    L = win.L if win is not None else dims.T          # the cost's time axis
    dtype, dev = xs.dtype, xs.device
    gx_, gu_ = pad.vec_n(_dense(dl_dxs, dtype)), pad.vec_m(_dense(dl_dus, dtype))
    lib, esz = _lib.lib(), xs.element_size()
    prec = ctypes.byref(sp.rec) if sp is not None else None
    if net is not None:
        name, head = "mpcb200_episode_backward_mlp", [ctypes.byref(net[0]), prec, int(n_steps)]
        nbytes = lib.mpcb200_episode_backward_mlp_workspace_bytes(ctypes.byref(dims), head[0], prec, esz)
        if nbytes == 0:
            raise MpcB200Error("mpcb200_episode_backward_mlp: the episode has no workspace size (the network's VJP "
                               "does not fit, or bad dimensions)")
    elif win is not None:
        name, head = "mpcb200_episode_backward_window", [ctypes.byref(win), prec, int(n_steps), k]
        nbytes = lib.mpcb200_episode_backward_window_workspace_bytes(ctypes.byref(dims), k, head[0], prec, esz)
    elif sp is not None:
        name, head = "mpcb200_episode_backward_plant", [prec, int(n_steps), k]
        nbytes = lib.mpcb200_episode_backward_plant_workspace_bytes(ctypes.byref(dims), k, prec, esz)
    elif k:
        name, head = "mpcb200_episode_backward_slew", [int(n_steps), k]
        nbytes = lib.mpcb200_episode_backward_slew_workspace_bytes(ctypes.byref(dims), k, esz)
    else:
        name, head = "mpcb200_episode_backward", [int(n_steps)]
        nbytes = lib.mpcb200_episode_backward_workspace_bytes(ctypes.byref(dims), esz)
    if alloc is None:
        def alloc(shape, dt):
            return torch.empty(shape, dtype=dt, device=dev)

    def n_params(kind):
        return DYN_NPARAMS[kind & ~DYN_CTRL_PASSTHROUGH]
    dx_init, dC, dc = alloc((B, N), dtype), alloc((L, B, P, P), dtype), alloc((L, B, P), dtype)
    dF = df = dtheta = None
    if net is not None:
        dtheta = alloc((net[1].numel(),), dtype)
    elif dims.dynamics_kind == DYN_LINEAR:
        dF = alloc((s.F.shape[0], B, N, P), dtype)
        df = alloc((L - 1, B, N), dtype) if dims.has_f else None
    else:
        dtheta = alloc((B, n_params(dims.dynamics_kind)), dtype)
    lin_plant = sp is not None and sp.rec.kind == DYN_LINEAR
    lead = (L - 1,) if win is not None and win.on & _lib.WIN_PLANT else ()
    dF_p = alloc((*lead, B, N, P), dtype) if lin_plant else None
    df_p = alloc((*lead, B, N), dtype) if lin_plant and sp.rec.has_f else None
    dth_p = alloc((B, n_params(sp.rec.kind)), dtype) if sp is not None and not lin_plant else None
    dw = alloc((n_steps, B, N), dtype) if s.disturbed or (sp is not None and sp.disturbed) else None
    ws = alloc((nbytes,), torch.uint8)
    plant_sweep = net is not None or win is not None or sp is not None
    args = [ctypes.byref(dims), ctypes.byref(s.params), *head, s.C, s.c, *([] if net is not None else [s.F]),
            *([sp.F if sp is not None else None] if plant_sweep else []), s.u_lower, s.u_upper, xs, us, plan_x, plan_u,
            gx_, gu_, dx_init, dC, dc, *([] if net is not None else [dF, df]), dtheta,
            *([dF_p, df_p, dth_p, dw] if plant_sweep else []), ws, nbytes, stream_handle(dev)]
    return name, args, (dx_init, dC, dc, dF, df, dtheta, dF_p, df_p, dth_p, dw)


def _episode_grads(s, out):
    """The ten gradients of a reverse sweep's outputs (_stage_episode_backward) as the staged problem's inputs take
    them: cropped to its own (n, m), and df (and a windowed LinDx plant's dF_p, df_p) zero-extended to the staged
    input's length, the slices no step reads."""
    dx_init, dC, dc, dF, df, dtheta, dF_p, df_p, dth_p, dw = out
    pad, sp = s.pad, s.plant

    def full(g, t):
        if g is None or t is None or t.shape[0] == g.shape[0]:
            return g
        return torch.cat((g, g.new_zeros(t.shape[0] - g.shape[0], *g.shape[1:])), 0)
    df = full(df, s.f)
    if s.window is not None and s.window.on & _lib.WIN_PLANT:
        dF_p, df_p = full(dF_p, sp.F), full(df_p, sp.f)
    return (pad.crop_n(dx_init), pad.crop_pp(dC), pad.crop_p(dc), pad.crop_np(dF), pad.crop_n(df), dtheta,
            pad.crop_np(dF_p), pad.crop_n(df_p), dth_p, pad.crop_n(dw))


def lqr_grad_raw(n_state, n_ctrl, T, C, c, F, new_x, new_u, dx, du, dl_dx, want_df, f_T=None):
    """Run the gradient-assembly kernel; returns (dx_init, dC, dc, dF, df|None)."""
    n, m = n_state, n_ctrl
    B = _validate(n, m, T, ("C", C, "TBpp"), ("c", c, "TBp"), ("new_x", new_x, "TBn"), ("new_u", new_u, "TBm"),
                  ("dx", dx, "TBn"), ("du", du, "TBm"), ("dl_dx", dl_dx, "TBn"), F=F)
    dtype, dev = C.dtype, C.device
    s = _problem(n, m, T, B, dtype, dev, C, c, F)
    pad, dims, N, M = s.pad, s.dims, s.pad.N, s.pad.M
    dims.has_f, dims.max_ls_iter, dims.pnqp_max_iter, dims.do_rollout = int(want_df), 1, 1, 0
    nx_, nu_ = pad.vec_n(_dense(new_x, dtype)), pad.vec_m(_dense(new_u, dtype))
    dx_, du_, r_ = pad.vec_n(_dense(dx, dtype)), pad.vec_m(_dense(du, dtype)), pad.vec_n(_dense(dl_dx, dtype))
    dx_init, dC, dc, dF, df = _grad_outputs(T, B, N, M, s.F, f_T, want_df, dtype, dev)
    fn = _lib.entry("mpcb200_lqr_grad", dtype)
    ws = torch.empty(2 * T * B * N, dtype=dtype, device=dev)     # costates: enables the two-kernel path
    with _on_device(dev):
        rc = fn(ctypes.byref(dims), ptr_view(s.C), ptr_view(s.c), ptr_view(s.F), ptr(nx_), ptr(nu_), ptr(dx_),
                ptr(du_), ptr(r_), ptr(dx_init), ptr(dC), ptr(dc), ptr(dF), ptr(df), ptr(ws), stream_handle(dev))
    check(rc, "mpcb200_lqr_grad")
    return pad.crop_n(dx_init), pad.crop_pp(dC), pad.crop_p(dc), pad.crop_np(dF), pad.crop_n(df)


_ws_cache = threading.local()


def _workspace(nbytes, dev):
    """Scratch buffer for the one-call adjoint, reused per (thread, device, stream): the library call is
    stream ordered, so consecutive backward passes on one stream can share it."""
    key = (dev, torch.cuda.current_stream(dev).cuda_stream)
    store = getattr(_ws_cache, "store", None)
    if store is None:
        store = _ws_cache.store = {}
    buf = store.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = store[key] = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    return buf


_adj_plans = {}


def lqr_adjoint_raw(n_state, n_ctrl, T, C, c, F, new_x, new_u, dl_dx, dl_du, u_lower, u_upper, want_df, f_T=None,
                    validated=False):
    """LQRStepFn.backward in ONE library call (mpcb200_lqr_adjoint_*: active set, nested masked step, costates and
    outer products; the library picks the kernels for the shape and horizon); returns (dx_init, dC, dc, dF|None,
    df|None).  The problem is staged as _problem stages it (a shape without an exact instance runs zero padded) and
    the outputs are cropped as lqr_grad_raw crops them.  `validated`: the tensors are the ones LQRStepFn.forward
    checked and saved plus autograd's gradients of its outputs (shapes follow), so the checks are not repeated on the
    backward path."""
    n, m = n_state, n_ctrl
    if not validated:
        _validate(n, m, T, ("C", C, "TBpp"), ("c", c, "TBp"), ("new_x", new_x, "TBn"), ("new_u", new_u, "TBm"),
                  ("dl_dx", dl_dx, "TBn"), ("dl_du", dl_du, "TBm"), F=F, bounds=(u_lower, u_upper))
    dtype, dev = C.dtype, C.device
    B = C.shape[1]
    esz = C.element_size()
    if _pick_instance(n, m, esz) == (n, m) and not _is_empty(F):
        # an exact instance, staged as _problem stages it, with the entry point, the ctypes structs and the workspace
        # size built once per signature (they depend only on the key)
        kind, s_lo, s_hi, lo_t, hi_t = _bounds(u_lower, u_upper, (T, B, m), dtype, dev)
        (C_, tsC), (c_, tsc), (F_, tsF) = _time_strided(C, dtype), _time_strided(c, dtype), _time_strided(F, dtype)
        key = (n, m, T, B, F.shape[0], esz, kind, s_lo, s_hi, bool(want_df), tsC, tsc, tsF,
               os.environ.get("MPCB200_KERNEL"))
        plan = _adj_plans.get(key)
        if plan is None:
            s = _problem(n, m, T, B, dtype, dev, C, c, F, None, u_lower, u_upper)   # for its Dims / Params
            if len(_adj_plans) > 256:
                _adj_plans.clear()
            plan = _adj_plans[key] = _adj_plan(s, want_df, dtype)
    else:
        s = _problem(n, m, T, B, dtype, dev, C, c, F, None, u_lower, u_upper)
        C_, c_, F_, lo_t, hi_t = s.C, s.c, s.F, s.u_lower, s.u_upper
        plan = _adj_plan(s, want_df, dtype)
    fn, pad, dims_ref, params_ref, nbytes = plan[:5]
    nx_, nu_ = pad.vec_n(_dense(new_x, dtype)), pad.vec_m(_dense(new_u, dtype))
    gx_, gu_ = pad.vec_n(_dense(dl_dx, dtype)), pad.vec_m(_dense(dl_du, dtype))
    dx_init, dC, dc, dF, df = _grad_outputs(T, B, pad.N, pad.M, F_, f_T, want_df, dtype, dev)
    ws = _workspace(nbytes, dev)
    with _on_device(dev):
        rc = fn(dims_ref, params_ref, ptr_view(C_), ptr_view(c_), ptr_view(F_), ptr(nx_), ptr(nu_), ptr(gx_),
                ptr(gu_), ptr(lo_t), ptr(hi_t), ptr(dx_init), ptr(dC), ptr(dc), ptr(dF), ptr(df), ptr(ws),
                nbytes, stream_handle(dev))
    check(rc, "mpcb200_lqr_adjoint")
    return pad.crop_n(dx_init), pad.crop_pp(dC), pad.crop_p(dc), pad.crop_np(dF), pad.crop_n(df)


def _adj_plan(s, want_df, dtype):
    """(entry point, _Pad, Dims ref, Params ref, workspace bytes, Dims, Params) of an adjoint call of the staged
    problem `s`; the last two keep the structs the refs point to alive."""
    dims, params = s.dims, s.params
    dims.has_f = int(want_df)
    nbytes = _lib.lib().mpcb200_adjoint_workspace_bytes(ctypes.byref(dims), dtype.itemsize)
    fn = _lib.entry("mpcb200_lqr_adjoint", dtype)
    return fn, s.pad, ctypes.byref(dims), ctypes.byref(params), nbytes, dims, params


def rollout_raw(n_state, n_ctrl, T, x_init, u, F, f=None):
    """x = get_traj(T, u, x_init, LinDx(F, f)) in ONE kernel (reference mpc/util.py:102-126)."""
    n, m = n_state, n_ctrl
    B = _validate(n, m, T, ("x_init", x_init, "Bn"), ("u", u, "TBm"), F=F, f=f)
    dtype, dev = x_init.dtype, x_init.device
    s = _problem(n, m, T, B, dtype, dev, F=F, f=f)
    s.dims.max_ls_iter = s.dims.pnqp_max_iter = 1
    x0_, u_ = s.pad.vec_n(_dense(x_init, dtype)), s.pad.vec_m(_dense(u, dtype))
    x = torch.empty(T, B, s.pad.N, dtype=dtype, device=dev)
    fn = _lib.entry("mpcb200_rollout", dtype)
    with _on_device(dev):
        rc = fn(ctypes.byref(s.dims), ptr_view(s.F), ptr_view(s.f), ptr(x0_), ptr(u_), ptr(x), stream_handle(dev))
    check(rc, "mpcb200_rollout")
    return s.pad.crop_n(x)


# ----------------------------------------------------------------------------------------------
# split-mode rollout for nn.Module dynamics / costs (cannot run inside the kernel)
# ----------------------------------------------------------------------------------------------
def _bound_at(v, t):
    return v if isinstance(v, float) else v[t]


def _clamp_assign(x, lo, hi):
    lo = torch.as_tensor(lo, dtype=x.dtype, device=x.device).expand_as(x)
    hi = torch.as_tensor(hi, dtype=x.dtype, device=x.device).expand_as(x)
    x = torch.where(x < lo, lo, x)          # util.eclamp order (reference mpc/util.py:64-68): lower, then upper
    return torch.where(x > hi, hi, x)


def _stage_cost(true_cost, tau, t):
    from .solver import QuadCost
    if isinstance(true_cost, QuadCost):
        Ct, ct = true_cost.C[t], true_cost.c[t]
        return 0.5 * (tau * torch.einsum("bij,bj->bi", Ct, tau)).sum(1) + (tau * ct).sum(1)
    return true_cost(tau)


def _step_dynamics(true_dynamics, x, u, t):
    from .solver import LinDx
    if isinstance(true_dynamics, LinDx):
        nx = torch.einsum("bij,bj->bi", true_dynamics.F[t], torch.cat((x, u), 1))
        if not _is_empty(true_dynamics.f):
            nx = nx + true_dynamics.f[t]
        return nx
    with torch.no_grad():
        return true_dynamics(x, u)


def rollout_split(T, x_init, cur_x, cur_u, Ks, ks, true_cost, true_dynamics,
                  u_lower, u_upper, u_zero_I, delta_u, decay, max_iter):
    """lqr_forward (reference mpc/lqr_step.py:164-261) with gains from the Riccati kernel and an
    arbitrary true model, as batched torch ops on the device."""
    B = x_init.shape[0]
    with torch.no_grad():
        old = 0
        for t in range(T):
            old = old + _stage_cost(true_cost, torch.cat((cur_x[t], cur_u[t]), 1), t)
        alphas = torch.ones(B, dtype=x_init.dtype, device=x_init.device)
        full_du_norm = None
        cost = None
        it = 0
        while it < max_iter and (cost is None or bool((cost > old).any())):
            xs, us = [x_init], []
            cost = 0
            for t in range(T):
                u = torch.einsum("bij,bj->bi", Ks[t], xs[t] - cur_x[t]) + cur_u[t] \
                    + alphas.unsqueeze(1) * ks[t]
                if u_zero_I is not None:
                    u = torch.where(u_zero_I[t].bool(), torch.zeros_like(u), u)
                if u_lower is not None:
                    lo, hi = _bound_at(u_lower, t), _bound_at(u_upper, t)
                    if delta_u is not None:
                        lo = torch.maximum(cur_u[t] - delta_u,
                                           torch.as_tensor(lo, dtype=u.dtype, device=u.device).expand_as(u))
                        hi = torch.minimum(cur_u[t] + delta_u,
                                           torch.as_tensor(hi, dtype=u.dtype, device=u.device).expand_as(u))
                    u = _clamp_assign(u, lo, hi)
                us.append(u)
                if t < T - 1:
                    xs.append(_step_dynamics(true_dynamics, xs[t], u, t))
                cost = cost + _stage_cost(true_cost, torch.cat((xs[t], u), 1), t)
            new_x, new_u = torch.stack(xs), torch.stack(us)
            if full_du_norm is None:
                full_du_norm = (cur_u - new_u).transpose(1, 2).reshape(B, -1).norm(2, 1)
            worse = cost > old
            alphas = torch.where(worse, alphas * decay, alphas)
            it += 1
        alphas = torch.where(cost > old, alphas / decay, alphas)
    return new_x, new_u, cost, full_du_norm, alphas


def reference_full_du_norm(du_first):
    """full_du_norm exactly as the reference forms it (mpc/lqr_step.py:244-245): the [T,B,m]
    difference is transposed to [T,m,B] and VIEWED as [B, T*m] before the row norm, so for
    B > 1 each entry mixes batch elements.  MPC's stop test / printed table depend on it."""
    B = du_first.shape[1]
    return du_first.transpose(1, 2).reshape(B, -1).norm(2, 1)


def _mlp_on_device(dx, n, m, x):
    from .mlp import on_device
    return isinstance(dx, Module) and on_device(dx, n, m, x)


def _same_storage(a, b):
    if a is None or b is None:
        return _is_empty(a) and _is_empty(b)
    return a.data_ptr() == b.data_ptr() and a.shape == b.shape and a.stride() == b.stride()


# ----------------------------------------------------------------------------------------------
# the autograd node
# ----------------------------------------------------------------------------------------------
class LQRStepFn(Function):
    """The autograd node behind LQRStep(...).  ONE class for every call (the reference builds a new Function
    class per call, mpc/lqr_step.py:275; the Python class creation alone costs more than the kernels at
    config 3): the closure arguments travel as the first, non-tensor argument `o`."""
    @staticmethod
    def forward(ctx, o, x_init, C, c, F, f=None):
        from .solver import QuadCost, LinDx
        from .dynamics import known_kind
        ctx.o = o
        if o.no_op_forward:                                   # reference :278-282
            # nothing is computed here, but backward hands these tensors to the kernels as raw pointers:
            # check them now, at the call site, once
            _validate(o.n_state, o.n_ctrl, o.T, ("C", C, "TBpp"), ("c", c, "TBp"), ("x_init", x_init, "Bn"),
                      ("current_x", o.current_x, "TBn"), ("current_u", o.current_u, "TBm"), F=F, f=f,
                      bounds=(o.u_lower, o.u_upper))
            ctx.save_for_backward(x_init, C, c, F, f, o.current_x, o.current_u)
            return o.current_x, o.current_u
        assert o.delta_space                                  # reference :284,298
        assert o.current_x is not None and o.current_u is not None
        assert not (o.delta_u is not None and o.u_lower is None)   # reference :195

        quad_same = (isinstance(o.true_cost, QuadCost) and _same_storage(o.true_cost.C, C)
                     and _same_storage(o.true_cost.c, c))
        fused = (quad_same and isinstance(o.true_dynamics, LinDx)
                 and _same_storage(o.true_dynamics.F, F)
                 and (_same_storage(o.true_dynamics.f, f)
                      or (_is_empty(o.true_dynamics.f) and _is_empty(f))))
        dyn = None
        if quad_same and not fused and isinstance(o.true_dynamics, Module):
            kind, kparams = known_kind(o.true_dynamics, o.n_state, o.n_ctrl, C)
            if kind:                       # a known system: its step function runs inside the kernel
                dyn, fused = (kind, kparams), True
        if fused:
            res = lqr_step_raw(o.n_state, o.n_ctrl, o.T, x_init, C, c, F, f, o.current_x, o.current_u,
                               u_lower=o.u_lower, u_upper=o.u_upper, u_zero_I=o.u_zero_I, delta_u=o.delta_u,
                               linesearch_decay=o.linesearch_decay,
                               max_linesearch_iter=o.max_linesearch_iter, do_rollout=True,
                               want_du_first=True, dyn=dyn)
            new_x, new_u = res["new_x"], res["new_u"]
            costs, alphas = res["costs"], res["alphas"]
            fdn = reference_full_du_norm(res["du_first"])
        elif quad_same and _mlp_on_device(o.true_dynamics, o.n_state, o.n_ctrl, C):
            # a learned model: the step's gains, then the network's line search in one kernel (mpcb200_mlp_step_*)
            from .mlp import step_raw
            res = step_raw(o.true_dynamics, o.n_state, o.n_ctrl, o.T, x_init, C, c, F, f, o.current_x, o.current_u,
                           u_lower=o.u_lower, u_upper=o.u_upper, u_zero_I=o.u_zero_I, delta_u=o.delta_u,
                           linesearch_decay=o.linesearch_decay, max_linesearch_iter=o.max_linesearch_iter)
            new_x, new_u, costs, alphas = res["new_x"], res["new_u"], res["costs"], res["alphas"]
            fdn = reference_full_du_norm(res["du_first"])
        else:
            assert o.true_cost is not None and o.true_dynamics is not None
            res = lqr_step_raw(o.n_state, o.n_ctrl, o.T, x_init, C, c, F, f, o.current_x, o.current_u,
                               u_lower=o.u_lower, u_upper=o.u_upper, u_zero_I=o.u_zero_I, delta_u=o.delta_u,
                               do_rollout=False)
            new_x, new_u, costs, fdn, alphas = rollout_split(
                o.T, x_init.detach(), o.current_x.detach(), o.current_u.detach(), res["Ks"], res["ks"],
                o.true_cost, o.true_dynamics, o.u_lower, o.u_upper, o.u_zero_I, o.delta_u,
                o.linesearch_decay, o.max_linesearch_iter)
        if o.u_lower is not None and o._defer_host is not None:
            # MPC's loop: no host read per step; the counters stay on the device and MPC reads them
            # together with its own stop-test scalars (one sync per iteration)
            o._defer_host["n_qp"] = (1 + res["qp_iters"].max(dim=1).values).sum()
            o._defer_host["unconverged"] = (res["status"] & 1).any()
            n_qp = float("nan")
        elif o.u_lower is not None:
            # reference: sum_t (1 + i_t) with one batched pnqp per step (:140)
            per_t = 1 + res["qp_iters"].max(dim=1).values
            if o.verbose > 1:                                   # reference :138-139, one line per time step
                for v in reversed(per_t.tolist()):              # the sweep runs t = T-1 .. 0
                    print("  + n_qp_iter: ", v)
            n_qp = float(per_t.sum().item())
            if o.verbose >= 0 and bool((res["status"] & 1).any()):
                print("[WARNING] pnqp warning: Did not converge")   # reference pnqp.py:81
                _host_reads.n_warned = getattr(_host_reads, "n_warned", 0) + 1
        else:
            n_qp = 0.0
        ctx.save_for_backward(x_init, C, c, F, f, new_x, new_u)
        return new_x, new_u, torch.Tensor([n_qp]), costs, fdn, alphas.mean()

    @staticmethod
    def backward(ctx, dl_dx, dl_du, temp=None, temp2=None, temp3=None, temp4=None):
        o = ctx.o
        x_init, C, c, F, f, new_x, new_u = ctx.saved_tensors
        if dl_dx is None:
            dl_dx = torch.zeros_like(new_x)
        if dl_du is None:
            dl_du = torch.zeros_like(new_u)
        want_df = not _is_empty(f)
        dx_init, dC, dc, dF, df = lqr_adjoint_raw(o.n_state, o.n_ctrl, o.T, C, c, F, new_x, new_u, dl_dx, dl_du,
                                                  o.u_lower, o.u_upper, want_df, f_T=f.shape[0] if want_df else None,
                                                  validated=True)
        if df is None:                                       # reference :402 (empty tensor)
            df = torch.zeros_like(f) if f is not None else None
        return None, dx_init, dC, dc, dF, df


# ----------------------------------------------------------------------------------------------
# the factory (reference mpc/lqr_step.py:22-38)
# ----------------------------------------------------------------------------------------------
def LQRStep(n_state,
            n_ctrl,
            T,
            u_lower=None,
            u_upper=None,
            u_zero_I=None,
            delta_u=None,
            linesearch_decay=0.2,
            max_linesearch_iter=10,
            true_cost=None,
            true_dynamics=None,
            delta_space=True,
            current_x=None,
            current_u=None,
            verbose=0,
            back_eps=1e-3,
            no_op_forward=False):
    """A single step of the box-constrained iLQR solver (drop-in for the reference factory).

    Returns a callable ``(x_init, C, c, F, f=None)`` giving
    ``(new_x[T,B,n], new_u[T,B,m], n_total_qp_iter (CPU float [1]), costs[B],
    full_du_norm[B], mean_alphas (0-d))`` - or ``(current_x, current_u)`` when
    ``no_op_forward`` - differentiable w.r.t. ``x_init, C, c, F, f``.
    """
    from types import SimpleNamespace
    o = SimpleNamespace(n_state=n_state, n_ctrl=n_ctrl, T=T, u_lower=u_lower, u_upper=u_upper, u_zero_I=u_zero_I,
                        delta_u=delta_u, linesearch_decay=linesearch_decay, max_linesearch_iter=max_linesearch_iter,
                        true_cost=true_cost, true_dynamics=true_dynamics, delta_space=delta_space,
                        current_x=current_x, current_u=current_u, verbose=verbose, back_eps=back_eps,
                        no_op_forward=no_op_forward, _defer_host=getattr(_host_reads, "defer", None))

    def apply(x_init, C, c, F, f=None):
        return LQRStepFn.apply(o, x_init, C, c, F, f)
    return apply

