"""GPU: time-varying receding-horizon episodes (mpcb200_episode_window_*) and their reverse sweep
(mpcb200_episode_backward_window_*) against the float64 oracle (oracle/window_oracle.py, known_oracle.episode).

Every time-indexed input lies on the episode's axis of L = n_steps + T - 1 slices, and solve k plans on slices
k .. k+T-1 of it; the library copies each window into workspace buffers (window_stage_kernel) and sums each sweep
step's gradients into the full-length outputs at offset k.  Every case runs both entries through the C ABI
(gpu_harness.abi_episode(window=L), abi_episode_backward) with every output at NaN (or 0xFF) before the call, so an
element no kernel writes fails (the slices past the last window included, which must be exactly 0), and checks
  * the forward of a LinDx model: x, u, costs, info, u_next and each solve's best iterate against
    window_oracle.receding_horizon_tv, problem by problem, under gpu_harness.check_episode_forward's rule (at most one
    problem in four departs, only in bounded episodes of several solve iterations), each solve's t = 0 bound being
    slice k of a windowed bound (episode_window_bounds).  The stop test is off (eps = 0, a fixed lqr_iter) except in
    one case per dtype.  A known model's forward against known_oracle.episode(window=True) in float64; in float32 for
    consistency (test_receding_plant_oracle_gpu.check_known_forward);
  * the sweep: every output (dx_init, dC, dc, dF, df, dtheta, dF_p, df_p, dtheta_p, dw) against
    window_oracle.receding_horizon_backward_tv run on the device's OWN xs, us and plans upcast to float64.  float64
    within 1e-9 x max(1, max|g|); float32 by the `within` policy, the oracle's float32 sweep on the same plans the
    yardstick.  Under a slew-rate penalty the first n_prev = m entries of dx_init and dw must be exactly 0;
  * the step plan the solve recorded, and the adjoint route of the sweep's body by its launch count (one more than the
    time-invariant sweep's: the window's stage kernel) and the plan its nested step recorded.  Under a window the
    solve's time strides are the dense staging buffers', so the 16-byte rule of adjoint_route applies to those.

Cases: every compiled instance (and padded, large shapes); the window input forms, with the staged record's time
strides asserted; every step plan on both sides of its switch (where the window buffers follow a larger episode
workspace); every adjoint route; slew-rate windows at every augmented instance; known models and plants; grid-stride
passes of every window loop in a pool layout; the forms only the C ABI reaches (a longer axis, a LinDx model or plant
whose window bit is clear); poisoned workspaces.  test_zz_coverage fails if, per dtype, the forward never ran a step
plan or the sweep an adjoint route, or if a window form never ran."""
import functools

import pytest
import torch

from mpc.pytorch_b200.dynamics import DYN_CTRL_PASSTHROUGH
from oracle import known_oracle as ko
from oracle import window_oracle as wo
from oracle.slew_oracle import slew_augment
from tests import test_receding_oracle_gpu as ro
from tests import test_receding_plant_oracle_gpu as pm
from tests.gpu_harness import (DEV, DT, F32, F64, INSTANCES, PAIR_SHAPES, SWITCH_PLANS, abi_episode,
                               abi_episode_backward, check_episode_forward, episode_known_inputs, episode_known_step,
                               episode_linear_inputs, episode_window_bounds, epgrad_launches, kernel_env, loop_plan,
                               pick_switch, plan_name, plan_str, pool_size, round_through, switches, within)
from tests.helpers import maxdiff

pytestmark = pytest.mark.gpu
SLEW = pm.SLEW
GRID_CAP = 4096 * 256               # epgrad_grid: at most 4096 blocks of 256 threads per pass
SEEN = set()                        # ("plan" | "route", dtype, name) and ("form", name)
ERRS = {}                           # (dtype, what) -> largest error relative to max(1, max|want|)
DEPARTED = {}                       # dtype -> [(departing problems, compared problems)]
GNAMES = pm.GNAMES
# the batch dimension of each output; a windowed LinDx plant's dF_p, df_p lie on the axis
BATCH_DIM = dict(dx_init=0, dC=1, dc=1, dF=1, df=1, dtheta=0, dF_p=1, df_p=1, dtheta_plant=0, dw=1)
KNOWN_OPTS = dict(lqr_iter=3, eps=0.0, not_improved_lim=10 ** 6, linesearch_decay=0.5, max_linesearch_iter=4)


def _note(dtype, what, err):
    ERRS[(dtype, what)] = max(ERRS.get((dtype, what), 0.0), err)


def _lib():
    from mpc.pytorch_b200 import _lib as L
    return L


# ------------------------------------------------------------------------------------------------------------------
# cases
# ------------------------------------------------------------------------------------------------------------------
class Case:
    """One time-varying episode: the system (n, m), its inputs on the axis L = n_steps + T - 1 rounded through dtype
    (episode_linear_inputs(L=L), or a known model's with a control push that changes along the axis), the plant, w and
    the previous control under a slew-rate penalty.
    plant: "none" (the model steps), "self" (the model steps, through the plant form: w alone), "lin" (a perturbed copy
    of the model's F, f along the axis, Lp = L-1 or L slices by Fp_T), "lin_nof" (the same without f), "lin_ti" (one
    slice for every step, a stride-0 view over the axis), or a known system's name.
    strided: names among C, c, F, f handed over with a positive time stride (every other slice of a [2 len, ...]
    tensor); P["time_invariant"] names inputs handed over as stride-0 views over the axis."""

    def __init__(self, n, m, T, B, dtype, n_steps, mode, plant="none", with_w=False, slew=False, seed=0, model=None,
                 Fp_T="L-1", strided=(), **forms):
        self.n, self.m, self.T, self.B, self.dtype, self.n_steps = n, m, T, B, dtype, n_steps
        self.mode, self.plant, self.with_w, self.slew, self.model = mode, plant, with_w, slew, model
        self.L = L = n_steps + T - 1
        self.strided, self.whole = tuple(strided), ()
        g = torch.Generator().manual_seed(seed + 3)
        if model is None:
            self.P, self.kw = episode_linear_inputs(seed, B, T, n, m, dtype, mode, L=L, **forms)
            self.dyn = self.mstep = self.theta = None
        else:
            mod, n_, m_, P, kw, dyn, theta = episode_known_inputs(model, B, L, dtype, seed)
            assert (n_, m_) == (n, m)
            push = 0.3 * kw["u_upper"] * (torch.rand(L, B, m, generator=g, dtype=F64) - 0.5)
            P["c"] = round_through(P["c"] + torch.cat((torch.zeros(L, B, n, dtype=F64), push), 2), dtype)
            P["time_invariant"] = ()
            self.P, self.kw, self.dyn = P, kw, dyn
            self.mstep, self.theta = episode_known_step(mod), theta.expand(B, -1)
        F, f = self.P["F"], self.P["f"]
        self.Fp = self.fp = None
        if plant in ("lin", "lin_nof", "lin_ti"):
            Lp = L - 1 if Fp_T == "L-1" else L
            if F is None:                   # a known model: a stable linear plant of its shape along the axis
                F = torch.cat((0.97 * torch.eye(n, dtype=F64) + 0.02 * torch.randn(Lp, B, n, n, generator=g,
                                                                                    dtype=F64),
                               0.05 * torch.randn(Lp, B, n, m, generator=g, dtype=F64)), 3)
            F = torch.cat((F, F[-1:]), 0) if F.shape[0] < Lp else F[:Lp]
            Fp = F * (1 + 0.05 * torch.randn(F.shape, generator=g, dtype=F64))
            fp = 0.01 * torch.randn(Lp, B, n, generator=g, dtype=F64)
            if f is not None:
                fp = fp + (torch.cat((f, f[-1:]), 0) if f.shape[0] < Lp else f[:Lp])
            if plant == "lin_ti":
                Fp, fp = Fp[:1].expand(Fp.shape).contiguous(), fp[:1].expand(fp.shape).contiguous()
            self.Fp = round_through(Fp, dtype)
            self.fp = None if plant == "lin_nof" else round_through(fp, dtype)
        self.pkind = self.pstep = self.ptheta = None
        if plant in pm.KNOWN:
            self.pkind, pmod = pm.known_plant_module(plant)
            self.pparams = pmod.mpcb200_params()
            self.pstep = episode_known_step(pmod)
            self.ptheta = pmod.params.double().expand(B, -1)
        self.w = round_through(0.02 * torch.randn(n_steps, B, n, generator=g, dtype=F64), dtype) if with_w else None
        self.prev = round_through(0.3 * torch.randn(B, m, generator=g, dtype=F64), dtype) if slew else None

    @property
    def lin_plant(self):
        return self.plant in ("lin", "lin_nof", "lin_ti")

    def oracle_plant(self, cast=lambda t: t):
        if self.lin_plant:
            return ("lin", cast(self.Fp), None if self.fp is None else cast(self.fp))
        if self.plant in pm.KNOWN:
            return ("step", self.pstep, cast(self.ptheta))
        return None

    def take(self, idx):
        """The case with batch elements idx (a pool layout: element b is problem idx[b])."""
        c = object.__new__(Case)
        c.__dict__.update(self.__dict__)
        B = self.B
        rows = lambda t: t.index_select(0 if t.dim() == 2 and t.shape[0] == B else 1, idx) \
            if torch.is_tensor(t) else t  # noqa: E731
        c.P = {k: rows(v) if k != "time_invariant" else v for k, v in self.P.items()}
        c.kw = {k: rows(v) for k, v in self.kw.items()}
        for k in ("Fp", "fp", "w"):
            setattr(c, k, None if getattr(self, k) is None else rows(getattr(self, k)))
        for k in ("prev", "theta", "ptheta"):
            setattr(c, k, None if getattr(self, k) is None else getattr(self, k).index_select(0, idx))
        c.B = idx.numel()
        return c


def _strided(t, dev):
    """t [len, ...] as every other slice of a [2 len, ...] tensor on dev: a positive time stride of 2 slices."""
    big = torch.zeros(2 * t.shape[0], *t.shape[1:], dtype=t.dtype, device=dev)
    big[::2] = t.to(dev)
    return big[::2]


def window_inputs(c, dev=DEV):
    """The case's x_init, C, c, F, f, plant and w as the episode takes them on `dev`, in its dtype: under a slew-rate
    penalty the augmented problem (slew_augment on the whole axis, the float32 oracle's own rounding), x_init
    [prev; x0], a LinDx plant's F~, f~ and [0; w]; a time-invariant input a stride-0 view over the axis made on dev,
    a strided one every other slice of a larger tensor (_strided)."""
    m, dt = c.m, c.dtype
    P = c.P
    x0, C, c_, F, f = (None if P[k] is None else P[k].to(dt) for k in ("x0", "C", "c", "F", "f"))
    Fp, fp, w = (None if t is None else t.to(dt) for t in (c.Fp, c.fp, c.w))
    if c.slew:
        if Fp is not None:
            Fp, fp = slew_augment(c.n, m, SLEW, C[:Fp.shape[0]], c_[:Fp.shape[0]], Fp, fp)[2:]
        C, c_, F, f = slew_augment(c.n, m, SLEW, C, c_, F, f)
        x0 = torch.cat((c.prev.to(dt), x0), 1)
        w = None if w is None else torch.cat((w.new_zeros(*w.shape[:2], m), w), 2)
    ins = []
    for k, t in (("x0", x0), ("C", C), ("c", c_), ("F", F), ("f", f)):
        if t is None:
            ins.append(None)
        elif k in P["time_invariant"]:
            ins.append(t[:1].to(dev).expand(t.shape))
        elif k in c.strided:
            ins.append(_strided(t, dev))
        else:
            ins.append(t.to(dev))
    plant = None
    if Fp is not None:
        if c.plant == "lin_ti":
            plant = ("lin", Fp[:1].to(dev).expand(Fp.shape), None if fp is None else fp[:1].to(dev).expand(fp.shape))
        else:
            plant = ("lin", Fp.to(dev), None if fp is None else fp.to(dev))
    elif c.pkind is not None:
        plant = (c.pkind | (DYN_CTRL_PASSTHROUGH if c.slew else 0), c.pparams)
    w_dev = w.to(dev) if w is not None and (c.with_w or c.plant == "self") else None
    return ins, plant, w_dev


def device_call(c, impl=None, opts=None, poison=False):
    """abi_episode(window=L) on the case; every output starts at NaN (info -1), the workspace too when `poison`."""
    m, dt = c.m, c.dtype
    ins, plant, w_dev = window_inputs(c)
    dyn = None
    if c.dyn is not None:
        dyn = (c.dyn[0] | (DYN_CTRL_PASSTHROUGH if c.slew else 0), c.dyn[1])
    u0 = torch.zeros(c.T, c.B, m, dtype=dt, device=DEV)
    kw = {k: (v.to(DEV, dt) if v.is_floating_point() else v.to(DEV)) if torch.is_tensor(v) else v
          for k, v in c.kw.items()}
    n = c.n + (m if c.slew else 0)
    with kernel_env(impl):
        return abi_episode(n, m, c.T, c.n_steps, *ins, u0, **kw, **opts, dyn=dyn, poison=poison,
                           n_prev=m if c.slew else 0, plant=plant, w=w_dev, nan_outputs=True, window=c.L)


def _cast(cast):
    return lambda t: cast(t) if torch.is_tensor(t) and t.is_floating_point() else t  # noqa: E731


def oracle_forward(c, opts):
    """The window oracle's episode (a known model: known_oracle.episode(window=True)) in float64, and in float32 for a
    float32 LinDx case (the yardstick)."""
    P = c.P
    okw = dict(c.kw, **opts)

    def run(cast):
        cc = _cast(cast)
        if c.model is not None:
            return ko.episode(c.n, c.m, c.T, c.n_steps, cc(P["x0"]), cc(P["C"]), cc(P["c"]), c.mstep, cc(c.theta),
                              plant=c.oracle_plant(cast), w=cc(c.w), u_init=torch.zeros(c.T, c.B, c.m, dtype=F64),
                              slew_rate_penalty=SLEW if c.slew else None, prev_ctrl=cc(c.prev), window=True,
                              coupled=False, **{k: cc(v) for k, v in okw.items()})
        return wo.receding_horizon_tv(
            c.n, c.m, c.T, c.n_steps, *[None if P[k] is None else cc(P[k]).contiguous()
                                        for k in ("x0", "C", "c", "F", "f")],
            plant=c.oracle_plant(cast), w=cc(c.w), slew_rate_penalty=SLEW if c.slew else None,
            prev_ctrl=cc(c.prev), coupled=False, whole=c.whole, **{k: cc(v) for k, v in okw.items()})
    o64 = run(lambda t: t.double())
    o32 = run(lambda t: t.float()) if c.dtype == F32 and c.model is None else None
    return o64, o32


def oracle_sweep(c, saved, wx, wu):
    """The window oracle's sweep on the device's own xs, us and plans (plan_x augmented under a penalty): float64, and
    float32 for a float32 case."""
    s, _, xs, us, plan_x, plan_u = saved
    k = c.m if c.slew else 0
    got = [s.pad.crop_n(xs).cpu()[..., k:], s.pad.crop_m(us).cpu(), s.pad.crop_n(plan_x).cpu(),
           s.pad.crop_m(plan_u).cpu()]
    P = c.P

    def run(cast):
        cc = _cast(cast)
        return wo.receding_horizon_backward_tv(
            c.n, c.m, c.T, cc(P["C"]).contiguous(), cc(P["c"]).contiguous(),
            None if P["F"] is None else cc(P["F"]).contiguous(), cc(P["f"]), *[cc(t) for t in got], cc(wx), cc(wu),
            u_lower=cc(c.kw.get("u_lower")), u_upper=cc(c.kw.get("u_upper")), step=c.mstep, theta=cc(c.theta),
            slew_rate_penalty=SLEW if c.slew else None, prev_ctrl=cc(c.prev), plant=c.oracle_plant(cast),
            whole=c.whole)
    o64 = run(lambda t: t.double())
    o32 = run(lambda t: t.float()) if c.dtype == F32 else None
    return o64, o32


def device_grads(c, g):
    """The sweep's outputs by oracle name, on the CPU, cropped to the system's blocks under a slew-rate penalty
    (whose detached entries of dx_init and dw must be exactly 0).  plant "self": the plant form returns the model's
    own step part in dF_p, df_p on the axis; the oracle gives it to dF, df at the same slices, so they are added."""
    out = {k: (None if t is None else t.cpu()) for k, t in zip(GNAMES, g)}
    if c.slew:
        k = c.m
        for name in ("dx_init", "dw"):
            if out.get(name) is not None:
                assert bool((out[name][..., :k] == 0).all()), f"{name}: the previous control's entries are not 0"
        crop = {"dx_init": lambda t: t[..., k:], "dC": lambda t: t[..., k:, k:], "dc": lambda t: t[..., k:],
                "dF": lambda t: t[..., k:, k:], "df": lambda t: t[..., k:], "dF_p": lambda t: t[..., k:, k:],
                "df_p": lambda t: t[..., k:], "dw": lambda t: t[..., k:]}
        out = {name: (crop[name](t) if t is not None and name in crop else t) for name, t in out.items()}
    if c.plant == "self":
        dfp = out.pop("df_p")
        out["dF"] = out["dF"] + out.pop("dF_p")
        out["df"] = None if out["df"] is None else out["df"] + dfp
    return out


def check_backward(tag, c, g, o64, o32):
    got = device_grads(c, g)
    want_keys = {k: v for k, v in o64.items() if v is not None}
    if not (c.with_w or c.plant == "self"):
        want_keys.pop("dw")             # the oracle's dw is dL/dx_{k+1}; the device writes it only for an added w
    for name, t in got.items():
        if name not in want_keys:
            assert t is None, f"{tag}: {name} returned, the oracle has none"
    for name, want in want_keys.items():
        a = got.get(name)
        assert a is not None, f"{tag}: {name} missing"
        w32 = None if o32 is None else o32[name]
        if name in ("dF_p", "df_p") and "plant" in c.whole:
            want, w32 = want[0], None if w32 is None else w32[0]
        assert a.shape == want.shape, f"{tag}: {name} shape {tuple(a.shape)} vs {tuple(want.shape)}"
        assert bool(torch.isfinite(a).all()), f"{tag}: {name} not finite"
        within(tag, name, a, want, w32, c.dtype)
        _note(c.dtype, "backward", maxdiff(a, want) / max(1.0, float(want.abs().max())))


def check_forward(tag, c, r, o64, o32, several):
    """A LinDx model (and a known one in float64): check_episode_forward on the system's states, each solve's t = 0
    bound its slice k; a known model in float32: the plant module's consistency check."""
    if c.model is not None and c.dtype == F32:
        pm.check_known_forward(tag, c, r)
        return
    r = dict(r, x=r["x"][..., c.m:] if c.slew else r["x"])
    err, n_dep, n_cmp = check_episode_forward(tag, r, o64, o32, episode_window_bounds(c.kw, c.n_steps), c.dtype,
                                              several)
    DEPARTED.setdefault(c.dtype, []).append((n_dep, n_cmp))
    _note(c.dtype, "forward x/u/u_next/plans", err)


def check_route(tag, route, launches, plan, known):
    """The windowed sweep's launch count (epgrad_launches(window=True)) and its nested step's plan, by
    test_receding_oracle_gpu.check_route's rule."""
    L = _lib()
    want = epgrad_launches(route, known, window=True)
    assert launches == want, f"{tag}: {launches} launches, {want} on the {route} route"
    if route == "large":
        ok = plan == L.PLAN_LARGE
    elif route == "fused":
        ok = bool(plan & L.PLAN_PAIR) and bool(plan & L.PLAN_GAINS_SMEM)
    else:
        ok = plan != L.PLAN_LARGE and bool(plan & L.PLAN_GAINS_SMEM) == (route != "three_gains")
    assert ok, f"{tag}: the adjoint's nested step ran {plan_str(plan)} on the {route} route"


def check_strides(tag, c, s):
    """The staged window record's time strides: 0 for a dense input, -1 for a stride-0 view, the view's own stride
    for a strided one; the bounds staged dense."""
    rec = s.window
    N, M = s.pad.N, s.pad.M
    P_, B = N + M, c.B
    slice_ = dict(C=B * P_ * P_, c=B * P_, F=B * N * P_, f=B * N)
    for k in ("C", "c", "F", "f"):
        if c.P[k] is None or (k in ("F", "f") and c.model is not None):
            continue
        want = -1 if k in c.P["time_invariant"] else 2 * slice_[k] if k in c.strided else 0
        got = getattr(rec, k + "_tstride")
        assert got == want, f"{tag}: {k} staged with time stride {got}, expected {want}"
    assert rec.lo_tstride == rec.hi_tstride == 0
    if c.lin_plant and "plant" not in c.whole:
        want = -1 if c.plant == "lin_ti" else 0
        assert rec.Fp_tstride == want, f"{tag}: plant F staged with time stride {rec.Fp_tstride}"


def loss_weights(c, seed):
    """dl_dx [n_steps+1, B, n], dl_du; and as the device takes them (m zeros in front under a slew-rate penalty)."""
    wx, wu = ro.loss_weights(c.n_steps, c.B, c.n, c.m, seed)
    wx, wu = round_through(wx, c.dtype), round_through(wu, c.dtype)
    gx = torch.cat((wx.new_zeros(*wx.shape[:2], c.m), wx), 2) if c.slew else wx
    return wx, wu, gx.to(DEV, c.dtype), wu.to(DEV, c.dtype)


def check_poisoned(tag, c, clean, g_clean, impl, opts, gx, gu):
    """Both calls again with every workspace byte and output at 0xFF: every output finite and bitwise the same."""
    r, _, _ = device_call(c, impl, opts, poison=True)
    for k in ("x", "u", "costs", "info", "u_next"):
        a = r[k]
        assert not a.is_floating_point() or bool(torch.isfinite(a).all()), f"{tag} poisoned: {k} not finite"
        assert torch.equal(a, clean[k]), f"{tag} poisoned: {k} differs"
    for i in (4, 5):
        assert torch.equal(r["saved"][i], clean["saved"][i]), f"{tag} poisoned: plans differ"
    with kernel_env(impl):
        g, _, _ = abi_episode_backward(clean["saved"], gx, gu, poison=True)
    for name, a, b in zip(GNAMES, g, g_clean):
        assert (a is None) == (b is None), f"{tag} poisoned: {name}"
        if a is not None:
            assert bool(torch.isfinite(a).all()), f"{tag} poisoned: {name} not finite"
            assert torch.equal(a, b), f"{tag} poisoned: {name} differs by {float((a - b).abs().max()):.3e}"


def opts_for(c, lqr_iter, fixed):
    if c.model is not None:
        return dict(KNOWN_OPTS)
    opts = ro.fixed_opts(lqr_iter) if fixed else dict(lqr_iter=lqr_iter, eps={F64: 1e-7, F32: 1e-4}[c.dtype])
    opts["best_cost_eps"] = 1e-4
    return opts


def run(tag, c, impl=None, seed=0, lqr_iter=2, fixed=True, want_plan=None, want_route=None, poison=False, form=None):
    """One episode and its sweep through the window entries, checked against the oracle; plan, route, launches and
    the staged record's time strides."""
    opts = opts_for(c, lqr_iter, fixed)
    N_aug = c.n + (c.m if c.slew else 0)
    tag = (f"{tag} n{c.n}m{c.m} {DT[c.dtype]} B={c.B} T={c.T} steps={c.n_steps} {c.mode} plant={c.plant} "
           f"w={c.with_w} slew={c.slew} model={c.model} MPCB200_KERNEL={impl}")
    r, _, plan = device_call(c, impl, opts)
    s = r["saved"][0]
    assert s.window is not None and s.window.L == c.L, f"{tag}: not the window entry"
    check_strides(tag, c, s)
    name = None
    if c.model is None:
        name = plan_name(plan, impl, N_aug, c.m, c.dtype)
        if want_plan is not None:
            assert name == want_plan, f"{tag}: plan {plan_str(plan)} ({name}), expected {want_plan}"
        SEEN.add(("plan", c.dtype, name))
    several = fixed and (lqr_iter > 1 or c.n_steps > 1)
    o64, o32 = oracle_forward(c, opts)
    check_forward(tag, c, r, o64, o32, several or c.model is not None)
    wx, wu, gx, gu = loss_weights(c, seed)
    with kernel_env(impl):
        g, launches, adj_plan = abi_episode_backward(r["saved"], gx, gu, nan_outputs=True)
    route = ro.adjoint_route(s.pad.N, s.pad.M, c.T, c.B, c.dtype, impl)
    if want_route is not None:
        assert route == want_route, f"{tag}: the case is meant for the {want_route} route, the rule gives {route}"
    check_route(tag, route, launches, adj_plan, known=c.model is not None)
    SEEN.add(("route", c.dtype, route))
    if form is not None:
        SEEN.add(("form", form))
    b64, b32 = oracle_sweep(c, r["saved"], wx, wu)
    check_backward(tag, c, g, b64, b32)
    if poison:
        check_poisoned(tag, c, r, g, impl, opts, gx, gu)
    return r, g


# ------------------------------------------------------------------------------------------------------------------
# every compiled instance, padded and large shapes; slew-rate windows at every augmented instance
# ------------------------------------------------------------------------------------------------------------------
SHAPES = INSTANCES + [(6, 1), (5, 2), (20, 4)]


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("n,m", SHAPES, ids=[f"n{n}m{m}" for n, m in SHAPES])
def test_every_instance(n, m, dtype):
    """B = 1 (scalar bounds or u_zero_I) and a batch tail of 257 (windowed tensor bounds with delta_u); n_steps 1, 2
    and 3; C, c and F all vary along the axis; the model steps, or a windowed LinDx plant with w does.  Scalar bounds
    on 257-problem tails over 3 control steps left the forward rule by round-off: 81 of 257 problems departed at
    (16, 4) in float64 (pnqp end points and line-search decisions), and at (5, 1) in float32 the kept problems' costs
    missed the float32 yardstick (2.8e-4 against 9.3e-5), as the plant module found over 5 steps; plain tensor
    bounds and scalar bounds at several problems run in test_window_forms (B = 12) and the route cases (B = 8)."""
    k = SHAPES.index((n, m)) + (dtype == F32)
    for j, (B, modes) in enumerate(((1, ("box", "mask")), (257, ("boxT",)))):
        plant = ("none", "lin")[(k + j) % 2]
        c = Case(n, m, (3, 6)[(k + j) % 2], B, dtype, (1, 2, 3)[(k + j) % 3], modes[k % len(modes)], plant,
                 plant != "none", seed=3000 + 10 * k + j)
        run("instance", c, seed=3000 + k)


SLEW_SYSTEMS = pm.SLEW_SYSTEMS


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("n,m", SLEW_SYSTEMS, ids=[f"n{n}m{m}" for n, m in SLEW_SYSTEMS])
def test_slew_every_instance(n, m, dtype):
    """The augmented shape (n + m, m) under a slew-rate penalty: B = 1 with the model stepping (unbounded, scalar
    bounds or u_zero_I), and B = 33 on a windowed LinDx plant with w (windowed tensor bounds with delta_u: with scalar
    bounds 9 of 33 float64 problems departed at (12, 4) by up to 3.2e-8, by round-off); a non-zero previous
    control."""
    k = SLEW_SYSTEMS.index((n, m)) + (dtype == F32)
    for j, (B, modes, plant) in enumerate(((1, ("plain", "box", "mask"), "none"), (33, ("boxT",), "lin"))):
        c = Case(n, m, (3, 6)[(k + j) % 2], B, dtype, (1, 2, 3)[(k + j) % 3], modes[k % len(modes)], plant,
                 plant != "none", True, seed=3100 + 10 * k + j)
        run("slew instance", c, seed=3100 + k)


# ------------------------------------------------------------------------------------------------------------------
# the window input forms
# ------------------------------------------------------------------------------------------------------------------
# name -> (mode, Case keywords)
FORMS = {
    "F_L-1": ("box", dict()),                                   # F, f with L-1 slices (F_T = T-1)
    "F_L": ("plain", dict(F_T="T")),                            # F with L slices (F_T = T)
    "f_none": ("box", dict(f_T="none")),
    "f_L": ("plain", dict(f_T="T")),
    "F_time_invariant": ("box", dict(time_invariant=("F",))),   # C windowed, F stride 0 with WIN_DYN set
    "c_time_invariant": ("plain", dict(time_invariant=("c",))),
    "strided": ("box", dict(strided=("C", "c", "F", "f"))),     # a positive time stride: not copied dense
    "bounds": ("tensor", dict()),
    "bounds_delta_u": ("boxT", dict()),
    "u_zero_I": ("mask", dict()),
    "plant_L-1": ("box", dict(plant="lin", with_w=True)),
    "plant_L": ("plain", dict(plant="lin", with_w=True, Fp_T="L")),
    "plant_nof": ("tensor", dict(plant="lin_nof", with_w=True)),
    "plant_time_invariant": ("box", dict(plant="lin_ti", with_w=True)),
    "w": ("plain", dict(plant="self", with_w=True)),
    "w_plant": ("boxT", dict(plant="lin", with_w=True, f_T="none")),
}


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("form", list(FORMS))
def test_window_forms(form, dtype):
    """Each window input form at (4, 2), B = 12, T = 6, 3 control steps (the staged record's time strides
    asserted)."""
    i = list(FORMS).index(form)
    mode, kw = FORMS[form]
    kw = dict(kw)
    if kw.get("F_T") == "T":
        kw["F_T"] = 6
    c = Case(4, 2, 6, 12, dtype, 3, mode, seed=3200 + 10 * i, **kw)
    run(f"form {form}", c, seed=3200 + i, lqr_iter=3, form=form, poison=i == 0)


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
def test_default_stop_rule(dtype):
    """The default stop rule (eps > 0): the oracle's loop decides on the same batch-wide norm.  A slew-rate window
    on a LinDx plant with w."""
    c = Case(4, 2, 8, 16, dtype, 3, "plain", "lin", True, True, seed=3300)
    run("default stop", c, seed=3300, lqr_iter=10, fixed=False, form="default stop")


# ------------------------------------------------------------------------------------------------------------------
# every step plan on both sides of its switch; every adjoint route
# ------------------------------------------------------------------------------------------------------------------
GROUPS = list(SWITCH_PLANS)


def switch_cases(pick, group_index):
    """(T, impl, slew, n_steps, poison) of a plan group's switch pick (N, M, T*, impls): just below and at T*, under
    every dispatch that applies, alternating the model stepping (the system (N, M)) and a slew-rate window (the
    system (N - M, M)); the first run at T* poisoned."""
    N, M, Ts, impls = pick
    out = []
    for k, T in enumerate((Ts - 1, Ts)):
        for j, impl in enumerate(impls):
            out.append((T, impl, (group_index + k + j) % 2 == 1, 1 + k, k == 1 and j == 0))
    return out


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("group", GROUPS)
def test_plans_at_switch(group, dtype):
    """Just below and at the switch horizon T* of the solve's step plan, under the default dispatch and each kernel
    forced; past a gain-store switch the window buffers follow the larger episode and sweep workspaces."""
    pick = pick_switch(group, dtype, augmentable=True)
    if pick is None:
        pytest.skip(f"no instance with n > m has a {group} switch of the loop's step within the oracle's horizons")
    N, M, Ts, _ = pick
    gi = GROUPS.index(group)
    for T, impl, slew, n_steps, poison in switch_cases(pick, gi):
        want = loop_plan(N, M, dtype, T, impl)
        if want is None:
            continue
        mode = "plain" if slew else ("box", "plain", "boxT")[gi % 3]
        c = Case(N - M if slew else N, M, T, 8, dtype, n_steps, mode, seed=3400 + 10 * gi + T % 7, slew=slew)
        run(f"{group} (T*={Ts})", c, impl, seed=3400 + gi, want_plan=plan_name(want, impl, N, M, dtype),
            poison=poison)


# (n, m, MPCB200_KERNEL, mode): no instance at (20, 4); knob 3 at instances
LARGE = [(20, 4, None, "boxT"), (8, 2, 3, "box"), (16, 4, 3, "plain")]


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("n,m,impl,mode", LARGE, ids=[f"n{c[0]}m{c[1]}_k{c[2]}" for c in LARGE])
def test_large_shape_kernels(n, m, impl, mode, dtype):
    c = Case(n, m, 6, 5, dtype, 2, mode, "lin", True, seed=3500 + n)
    run("large", c, impl, seed=3500, want_plan="large", want_route="large", poison=impl is None)


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
def test_route_fused(dtype):
    c = Case(8, 2, 6, 8, dtype, 3, "tensor", "lin", True, seed=3600)
    run("fused", c, seed=3600, lqr_iter=3, want_route="fused", poison=True)


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
def test_route_three_launch_by_shape(dtype):
    """(8, 2) under MPCB200_KERNEL=1: no fused kernel; (8, 1) by default: not a pair shape."""
    c = Case(8, 2, 6, 8, dtype, 2, "box", seed=3610)
    run("3-launch by knob", c, 1, seed=3610, want_route="three_shape", poison=True)
    c = Case(8, 1, 6, 8, dtype, 2, "boxT", "lin", True, seed=3611)
    run("3-launch by shape", c, seed=3611, want_route="three_shape")


def test_route_three_launch_by_alignment():
    """f32 (4, 2) at B = 7: the dense staging buffers' time strides are no 16-byte multiple (B p 4 bytes)."""
    assert (4, 2) in PAIR_SHAPES and (7 * 6 * 4) % 16 != 0
    c = Case(4, 2, 6, 7, F32, 3, "box", "lin", True, seed=3620)
    run("3-launch by alignment", c, seed=3620, lqr_iter=3, want_route="three_align", poison=True)
    c = Case(2, 2, 6, 7, F32, 2, "plain", slew=True, seed=3621)
    run("3-launch by alignment (slew)", c, seed=3621, want_route="three_align")


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
def test_route_three_launch_by_gains(dtype):
    """(16, 4) from the instance's gain-store switch on: the nested step keeps its gains in the workspace, and the
    window buffers follow the larger sweep workspace."""
    sw = switches(16, 4, dtype)
    assert sw["adjoint"] is not None and sw["generic"] is not None
    T = max(sw["adjoint"], sw["generic"])
    c = Case(16, 4, T, 8, dtype, 2, "box", "lin", True, seed=3630)
    run("3-launch by gains", c, seed=3630, want_route="three_gains", poison=True)


# ------------------------------------------------------------------------------------------------------------------
# known models and plants on windows
# ------------------------------------------------------------------------------------------------------------------
KNOWN_CASES = [(name, B, slew) for name in ("cartpole", "pendulum", "pendulum_full")
               for B, slew in ((1, False), (300, False), (7, True))]


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("name,B,slew", KNOWN_CASES, ids=[f"{a}_B{b}{'_slew' if s else ''}" for a, b, s in KNOWN_CASES])
def test_known_models(name, B, slew, dtype):
    """A known model on a window of C, c (a control push along the axis), with the clamp: the sweep's dtheta per
    problem; the passthrough kind under a slew-rate penalty."""
    n = 5 if name == "cartpole" else 3
    c = Case(n, 1, 8, B, dtype, 3, "clamp", seed=3700 + B + slew, slew=slew, model=name)
    run(f"known {name}", c, seed=3700, form=f"known {name}" + (" slew" if slew else ""), poison=B == 7)


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("name", ["pendulum", "cartpole"])
def test_known_plant_on_windowed_model(name, dtype):
    """Pendulum (3, 1) and cartpole (5, 1) plants on a windowed LinDx model of their shape, with w."""
    n = 5 if name == "cartpole" else 3
    c = Case(n, 1, 8, 9, dtype, 3, "plain", name, True, seed=3800 + n)
    run(f"{name} plant", c, seed=3800, lqr_iter=3, form=f"{name} plant")


# ------------------------------------------------------------------------------------------------------------------
# grid-stride passes past epgrad_grid's cap: a pool of K problems, element b is pool problem b mod K
# ------------------------------------------------------------------------------------------------------------------
# name -> (n, m, T, n_steps, B, plant): (4, 2) at B = 180 000, B P = 1 080 000 > 2^20
GRID = {"model_step": dict(n=4, m=2, T=3, n_steps=2, B=180_000, plant="none"),
        "plant_step": dict(n=4, m=2, T=3, n_steps=2, B=180_000, plant="lin")}


def grid_loops(name):
    """Items of each window loop a grid case targets, and whether its grid is capped: the window copy (grid by its
    largest input, C: T B P^2), the init's full-length zeroing (grid by L B P^2, dC), the accumulate (grid by T B P^2,
    its dC loop) and the windowed LinDx stage, of the model or of the plant (grid by T B max(N, M), loop over B P)."""
    g = GRID[name]
    N, M, T, B = g["n"], g["m"], g["T"], g["B"]
    P, L = N + M, g["n_steps"] + g["T"] - 1
    return {"window copy": (T * B * P * P, T * B * P * P > GRID_CAP),
            "init zeroing": (L * B * P * P, L * B * P * P > GRID_CAP),
            "accumulate": (T * B * P * P, T * B * P * P > GRID_CAP),
            ("plant stage" if g["plant"] != "none" else "model stage"): (B * P, T * B * max(N, M) > GRID_CAP)}


def grid_pool(name):
    """(K, idx): the pool size, coprime to the 256-thread block, to N and to P, and the pool problem of each
    element."""
    g = GRID[name]
    K = pool_size(256, g["n"], g["n"] + g["m"])
    return K, torch.arange(g["B"]) % K


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("name", list(GRID))
def test_grid_stride_passes(name, dtype):
    """Windowed tensor bounds, T = 3, 2 control steps, w on the plant: every copy bitwise its pool problem (x, u,
    plans, every gradient), the pool against the oracle."""
    g = GRID[name]
    K, idx = grid_pool(name)
    pool = Case(g["n"], g["m"], g["T"], K, dtype, g["n_steps"], "tensor", g["plant"], g["plant"] != "none",
                seed=3900)
    c = pool.take(idx)
    opts = dict(ro.fixed_opts(1), best_cost_eps=1e-4)
    r, _, plan = device_call(c, None, opts)
    wx, wu, _, _ = loss_weights(pool, 3900)
    gx, gu = wx.index_select(1, idx).to(DEV, dtype), wu.index_select(1, idx).to(DEV, dtype)
    grads, launches, adj_plan = abi_episode_backward(r["saved"], gx, gu, nan_outputs=True)
    s = r["saved"][0]
    route = ro.adjoint_route(s.pad.N, s.pad.M, c.T, c.B, dtype, None)
    check_route(name, route, launches, adj_plan, False)
    SEEN.add(("plan", dtype, plan_name(plan, None, s.pad.N, s.pad.M, dtype)))
    SEEN.add(("route", dtype, route))
    SEEN.add(("form", f"grid {name}"))
    di = idx.to(DEV)

    def copies(what, t, dim):
        ref = t.narrow(dim, 0, K).index_select(dim, di)
        assert torch.equal(t, ref), f"{name}: {what} of a copy differs from its pool problem"
    for k, dim in (("x", 1), ("u", 1), ("costs", 1)):
        copies(k, r[k], dim)
    for i in (2, 3):
        copies(("xs", "us")[i - 2], r["saved"][i], 1)
    for i in (4, 5):
        copies(("plan_x", "plan_u")[i - 4], r["saved"][i], 2)
    for gname, t in zip(GNAMES, grads):
        if t is not None:
            copies(gname, t, BATCH_DIM[gname])
    cut = lambda t, dim: t.narrow(dim, 0, K)  # noqa: E731
    rp = {k: cut(r[k], 1) for k in ("x", "u", "costs", "u_next")}
    rp["info"] = r["info"]
    saved = (s, r["saved"][1], cut(r["saved"][2], 1), cut(r["saved"][3], 1), cut(r["saved"][4], 2),
             cut(r["saved"][5], 2))
    rp["saved"] = saved
    o64, o32 = oracle_forward(pool, opts)
    check_forward(f"grid {name}", pool, rp, o64, o32, True)
    b64, b32 = oracle_sweep(pool, saved, wx, wu)
    gp = [None if t is None else cut(t, BATCH_DIM[k]) for k, t in zip(GNAMES, grads)]
    check_backward(f"grid {name}", pool, gp, b64, b32)


# ------------------------------------------------------------------------------------------------------------------
# the forms only the C ABI reaches: the Python staging, then the record and pointers edited
# ------------------------------------------------------------------------------------------------------------------
EXTRA = 3                           # slices past n_steps + T - 1 on the longer axis


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
def test_longer_axis(monkeypatch, dtype):
    """L = n_steps + T - 1 + 3: staged as an episode of n_steps + 3 steps, then called for n_steps.  The forward is
    bitwise the exact-L call's, the rows of steps it does not run stay untouched; the sweep's trailing slices are
    exactly 0 and its other slices bitwise the exact-L call's.  A windowed LinDx plant with w."""
    from mpc.pytorch_b200 import step as S
    n_steps = 2
    longc = Case(4, 2, 6, 10, dtype, n_steps + EXTRA, "tensor", "lin", True, seed=4000)
    exact = longc.take(torch.arange(10))
    L = n_steps + 6 - 1
    exact.n_steps, exact.L = n_steps, L
    cut = lambda t, k: None if t is None else t[:k]  # noqa: E731
    exact.P = {k: (v if k in ("x0", "time_invariant") or v is None else v[:L - (longc.L - v.shape[0])])
               for k, v in longc.P.items()}
    exact.kw = {k: cut(v, L) if torch.is_tensor(v) else v for k, v in longc.kw.items()}
    exact.Fp, exact.fp, exact.w = cut(longc.Fp, L - 1), cut(longc.fp, L - 1), cut(longc.w, n_steps)
    opts = opts_for(exact, 2, True)
    r0, _, _ = device_call(exact, None, opts)
    real = S._call

    def call_n_steps(name, dt, dev, args):     # the staged n_steps + 3 -> n_steps
        assert args[5] == n_steps + EXTRA
        return real(name, dt, dev, args[:5] + [n_steps] + args[6:])
    with monkeypatch.context() as mp:
        mp.setattr(S, "_call", call_n_steps)
        r1, _, _ = device_call(longc, None, opts)
    for k, k_rows in (("x", n_steps + 1), ("u", n_steps), ("costs", n_steps), ("info", n_steps)):
        assert torch.equal(r1[k][:k_rows], r0[k]), f"longer axis: {k} differs from the exact-L call's"
        rest = r1[k][k_rows:]
        assert bool(rest.isnan().all()) if rest.is_floating_point() else bool((rest == -1).all()), \
            f"longer axis: {k} written past n_steps"
    assert torch.equal(r1["u_next"], r0["u_next"])
    s1 = r1["saved"]
    saved = (s1[0], n_steps, s1[2][:n_steps + 1], s1[3][:n_steps], s1[4][:n_steps], s1[5][:n_steps])
    for i in (4, 5):
        assert torch.equal(saved[i], r0["saved"][i]), "longer axis: plans differ"
    _, _, gx, gu = loss_weights(exact, 4000)
    g0, _, _ = abi_episode_backward(r0["saved"], gx, gu, nan_outputs=True)
    g1, launches, plan = abi_episode_backward(saved, gx, gu, nan_outputs=True)
    check_route("longer axis", ro.adjoint_route(4, 2, 6, 10, dtype, None), launches, plan, False)
    for name, a, b in zip(GNAMES, g1, g0):
        assert (a is None) == (b is None), name
        if a is None:
            continue
        if a.shape == b.shape:
            assert torch.equal(a, b), f"longer axis: {name} differs from the exact-L call's"
            continue
        k = b.shape[0]
        assert a.shape[0] == k + EXTRA, f"longer axis: {name} has {a.shape[0]} slices"
        assert torch.equal(a[:k], b), f"longer axis: {name} differs from the exact-L call's"
        assert bool((a[k:] == 0).all()), f"longer axis: {name}'s trailing slices are not 0"
    SEEN.add(("form", "longer axis"))


def _raw_backward(saved, gx, gu):
    """The windowed sweep's raw outputs (the staging's padded buffers, every one at NaN before the call), without
    _episode_grads' zero-extension to the staged inputs' lengths."""
    from mpc.pytorch_b200 import step as S
    from tests.gpu_harness import _owned_alloc
    L = _lib()
    name, args, out = S._stage_episode_backward(saved, gx, gu, alloc=_owned_alloc(False, True))
    before = L.launch_count()
    L.check(S._call(name, saved[2].dtype, DEV, args), name)
    launches, p = L.launch_count() - before, L.last_step_plan()
    torch.cuda.synchronize()
    return out, launches, p


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("form", ["model", "plant"])
def test_window_bit_clear(monkeypatch, form, dtype):
    """model: a LinDx model with MPCB200_WIN_DYN clear, a stationary model under a windowed cost: F [F_T], f [T-1]
    handed to every solve and step, dF, df of the solve's own F_T, T-1 slices.  plant: a LinDx plant with
    MPCB200_WIN_PLANT clear: slice 0 steps every control step, dF_p [B, n, p].  The Python staging, then the record's
    bit cleared and the pointers set to the whole inputs; against window_oracle(whole=...)."""
    from mpc.pytorch_b200 import step as S
    L_ = _lib()
    T, n_steps, B = 6, 3, 10
    c = Case(4, 2, T, B, dtype, n_steps, "tensor", "lin" if form == "plant" else "none", form == "plant",
             seed=4100 + (form == "plant"))
    c.whole = ("F",) if form == "model" else ("plant",)
    if form == "model":
        c.P = dict(c.P, F=c.P["F"][:T - 1].clone(), f=c.P["f"][:T - 1].clone())
        real_wp = S._window_problem

        def window_problem(n, m, T_, n_steps_, L, x_init, C, c_, F, f, *a):
            axis = lambda t: torch.cat((t, t.new_zeros(L - 1 - t.shape[0], *t.shape[1:])), 0)  # noqa: E731
            s = real_wp(n, m, T_, n_steps_, L, x_init, C, c_, axis(F), axis(f), *a)
            s.window.on &= ~L_.WIN_DYN
            return s._replace(F=F.contiguous(), f=f.contiguous())
        mp_target = ("_window_problem", window_problem)
    else:
        c.Fp, c.fp = c.Fp[:1].clone(), c.fp[:1].clone()
        real_sp = S._stage_plant

        def stage_plant(pad, plant, dtype_, B_, n, m, win=None):
            kind, params, F_p, f_p = plant
            sp = real_sp(pad, (kind, params, F_p.expand(win.L - 1, *F_p.shape[1:]),
                               f_p.expand(win.L - 1, *f_p.shape[1:])), dtype_, B_, n, m, win)
            win.on &= ~L_.WIN_PLANT
            return sp._replace(F=F_p[0].contiguous(), f=f_p[0].contiguous())
        mp_target = ("_stage_plant", stage_plant)
    opts = opts_for(c, 2, True)
    with monkeypatch.context() as mp:
        mp.setattr(S, *mp_target)
        r, _, plan = device_call(c, None, opts)
    s = r["saved"][0]
    bit = L_.WIN_DYN if form == "model" else L_.WIN_PLANT
    assert not s.window.on & bit and s.window.on & L_.WIN_COST
    SEEN.add(("plan", dtype, plan_name(plan, None, 4, 2, dtype)))
    o64, o32 = oracle_forward(c, opts)
    check_forward(f"bit clear {form}", c, r, o64, o32, True)
    wx, wu, gx, gu = loss_weights(c, 4100)
    out, launches, adj_plan = _raw_backward(r["saved"], gx, gu)
    route = ro.adjoint_route(4, 2, T, B, dtype, None)
    check_route(f"bit clear {form}", route, launches, adj_plan, False)
    g = list(out)
    if form == "model":
        df = out[4]
        assert df.shape[0] == c.L - 1 and bool(df[T - 1:].isnan().all()), "df written past the solve's T-1 slices"
        g[4] = df[:T - 1]
        assert g[3].shape[0] == T - 1
    else:
        assert g[6].dim() == 3 and g[7].dim() == 2, "the plant's dF_p, df_p are not [B, ...]"
    b64, b32 = oracle_sweep(c, r["saved"], wx, wu)
    check_backward(f"bit clear {form}", c, g, b64, b32)
    SEEN.add(("form", f"{form} bit clear"))


# ------------------------------------------------------------------------------------------------------------------
# coverage (runs last)
# ------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _needed_plans(dtype):
    need = {"large"}
    for group, plans in SWITCH_PLANS.items():
        if pick_switch(group, dtype, augmentable=True) is not None:
            need |= set(plans)
    return need


NEEDED_FORMS = (set(FORMS) | {"default stop", "longer axis", "model bit clear", "plant bit clear",
                              "pendulum plant", "cartpole plant", "grid model_step", "grid plant_step"}
                | {f"known {a}" + (" slew" if s else "") for a, _, s in KNOWN_CASES})


def test_zz_coverage():
    if not SEEN:
        pytest.skip("no episode test of this module ran")
    missing = []
    for dtype in (F64, F32):
        plans = {x[2] for x in SEEN if x[:2] == ("plan", dtype)}
        routes = {x[2] for x in SEEN if x[:2] == ("route", dtype)}
        print(f"{DT[dtype]}: window step plans {sorted(plans)}; windowed sweep adjoint routes {sorted(routes)}")
        missing += [f"{DT[dtype]} plan {p}" for p in sorted(_needed_plans(dtype) - plans)]
        need_routes = {"fused", "three_shape", "three_gains", "large"}
        if dtype == F32:
            need_routes.add("three_align")
        missing += [f"{DT[dtype]} route {r}" for r in sorted(need_routes - routes)]
    forms = {x[1] for x in SEEN if x[0] == "form"}
    missing += [f"form {f}" for f in sorted(NEEDED_FORMS - forms)]
    for (dtype, what), v in sorted(ERRS.items(), key=lambda kv: (DT[kv[0][0]], kv[0][1])):
        print(f"{DT[dtype]} {what}: largest error {v:.3e} of max(1, max|want|)")
    for dtype, v in DEPARTED.items():
        print(f"{DT[dtype]}: problems departing from the oracle {sum(a for a, _ in v)} of {sum(b for _, b in v)} "
              f"compared, in {sum(a > 0 for a, _ in v)} of {len(v)} runs")
    assert not missing, "never run: " + ", ".join(missing)
