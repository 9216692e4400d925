"""GPU: receding-horizon episodes closed on a plant other than the model, with additive disturbances
(mpcb200_episode_plant_*, mpcb200_episode_backward_plant_*), and the slew-rate episode's reverse sweep
(mpcb200_episode_backward_slew_*), against the float64 oracle (oracle/plant_oracle.py).

Every case runs the device episode through the C ABI (gpu_harness.abi_episode, abi_episode_backward) with every output
at NaN (or 0xFF) before the call, so an element no kernel writes fails, and checks
  * the forward of a LinDx model: x, u, costs, info, u_next and each solve's best iterate against
    plant_oracle.receding_horizon_lin, problem by problem, under test_receding_oracle_gpu.check_forward's departure
    rule (at most one problem in four, only in bounded episodes of several solve iterations).  The stop test is off
    (eps = 0, a fixed lqr_iter) except in one case per dtype.  A known model has no iLQR oracle: its forward is checked
    for consistency (check_known_forward: applied controls, the plant step plus w, the plans' rollouts);
  * the sweep: every output (dx_init, dC, dc, dF, df, dtheta, dF_plant, df_plant, dtheta_plant, dw) against
    plant_oracle.receding_horizon_backward run on the device's OWN xs, us and plans upcast to float64.  float64 within
    1e-9 x max(1, max|g|); float32 by the `within` policy, the oracle's float32 sweep on the same plans the yardstick.
    Under a slew-rate penalty every size is the augmented problem's, and the first n_prev = m entries of dx_init and
    dw (the previous control, detached) must be exactly 0;
  * the step plan the solve recorded and the adjoint route of the sweep's body, by the launch count and the plan the
    nested step recorded (test_receding_oracle_gpu.adjoint_route, check_route).

Cases: the slew sweep at every instance reachable as an augmented shape; plant episodes at every instance with the
bound kinds, plant forms, known plants, known on known, and the passthrough plant kinds; every step plan on both sides
of its switch and every adjoint route, inside both sweeps; batches whose grid-stride loops take two passes (a pool
layout: batch element b is pool problem b mod K, every copy checked bitwise against its pool problem, the pool against
the oracle); the input forms; poisoned workspaces; and the invariant that the carried previous control is the applied
control, disturbance or not.  test_zz_coverage fails if, per dtype, an entry never ran a step plan or an adjoint
route, or if a plant form never ran; it does not ask for every combination of the four."""
import functools

import pytest
import torch

from mpc.pytorch_b200.dynamics import DYN_CARTPOLE, DYN_CTRL_PASSTHROUGH, DYN_PENDULUM, DYN_PENDULUM_FULL
from oracle import plant_oracle as porc
from oracle.slew_oracle import slew_augment
from tests import test_receding_oracle_gpu as ro
from tests.gpu_harness import (DEV, DT, F32, F64, INSTANCES, SWITCH_PLANS, abi_episode, abi_episode_backward,
                               check_episode_forward, episode_known_inputs, episode_known_step, episode_linear_inputs,
                               kernel_env, loop_plan, pick_switch, plan_name, plan_str, pool_size, round_through,
                               switches, within)
from tests.helpers import maxdiff

pytestmark = pytest.mark.gpu
SLEW = 0.1
GRID_CAP = 4096 * 256               # epgrad_grid / ilqr_grid: at most 4096 blocks of 256 threads per pass
SEEN = set()                        # ("plan" | "route", entry, dtype, name) and ("form", form)
ERRS = {}                           # (dtype, what) -> largest error relative to max(1, max|want|)
DEPARTED = {}                       # dtype -> [(departing problems, compared problems)]

# known systems as models and plants: (dynamics kind, constructor, parameters)
KNOWN = {"pendulum": (DYN_PENDULUM, dict(), (10.0, 1.0, 1.0)),
         "pendulum_full": (DYN_PENDULUM_FULL, dict(simple=False), (10.0, 1.0, 1.0, 0.3, 0.2)),
         "cartpole": (DYN_CARTPOLE, dict(), (9.8, 1.2, 0.12, 0.55))}
GNAMES = ("dx_init", "dC", "dc", "dF", "df", "dtheta", "dF_p", "df_p", "dtheta_plant", "dw")
BATCH_DIM = dict(dx_init=0, dC=1, dc=1, dF=1, df=1, dtheta=0, dF_p=0, df_p=0, dtheta_plant=0, dw=1)


def _note(dtype, what, err):
    ERRS[(dtype, what)] = max(ERRS.get((dtype, what), 0.0), err)


def _f32(t):
    return t.float() if torch.is_tensor(t) and t.is_floating_point() else t


def known_plant_module(name):
    from mpc.pytorch_b200.dynamics import CartpoleDx, PendulumDx
    kind, extra, vals = KNOWN[name]
    ctor = CartpoleDx if kind == DYN_CARTPOLE else PendulumDx
    return kind, ctor(params=torch.tensor(vals, dtype=F64), **extra)


# ------------------------------------------------------------------------------------------------------------------
# cases
# ------------------------------------------------------------------------------------------------------------------
class Case:
    """One episode: the system (n, m), its inputs rounded through dtype (float64 values, P and kw as
    episode_linear_inputs makes them, or a known model's), the plant form, w, the previous control under a slew-rate
    penalty.  plant: "none" (the model steps), "self" (the model steps, through the plant entry: w alone), "lin"
    (a perturbed copy of F[0], f[0]), "lin_nof" (the same without f), or a known system's name."""

    def __init__(self, n, m, T, B, dtype, n_steps, mode, plant, with_w, slew, seed, model=None, **forms):
        self.n, self.m, self.T, self.B, self.dtype, self.n_steps = n, m, T, B, dtype, n_steps
        self.mode, self.plant, self.with_w, self.slew, self.model = mode, plant, with_w, slew, model
        g = torch.Generator().manual_seed(seed + 3)
        if model is None:
            self.P, self.kw = episode_linear_inputs(seed, B, T, n, m, dtype, mode, **forms)
            self.dyn = self.mstep = self.theta = None
        else:
            mod, n_, m_, P, kw, dyn, theta = episode_known_inputs(model, B, T, dtype, seed)
            assert (n_, m_) == (n, m)
            P["time_invariant"] = ()
            self.P, self.kw, self.dyn = P, kw, dyn
            self.mstep, self.theta = episode_known_step(mod), theta.expand(B, -1)
        F, f = self.P["F"], self.P["f"]
        self.Fp = self.fp = None
        if plant in ("lin", "lin_nof"):
            if F is None:                   # a known model: a stable linear plant of its shape
                F = torch.cat((0.97 * torch.eye(n, dtype=F64) + 0.02 * torch.randn(n, n, generator=g, dtype=F64),
                               0.05 * torch.randn(n, m, generator=g, dtype=F64)), 1).expand(1, B, n, n + m)
            Fp = F[:1] * (1 + 0.05 * torch.randn(F[:1].shape, generator=g, dtype=F64))
            self.Fp = round_through(Fp, dtype)
            if plant == "lin":
                fp = 0.01 * torch.randn(1, B, n, generator=g, dtype=F64)
                self.fp = round_through(fp + (f[:1] if f is not None else 0), dtype)
        self.pkind = self.pstep = self.ptheta = None
        if plant in KNOWN:
            self.pkind, pmod = known_plant_module(plant)
            self.pparams = pmod.mpcb200_params()
            self.pstep = episode_known_step(pmod)
            self.ptheta = pmod.params.double().expand(B, -1)
        self.w = round_through(0.02 * torch.randn(n_steps, B, n, generator=g, dtype=F64), dtype) if with_w else None
        self.prev = round_through(0.3 * torch.randn(B, m, generator=g, dtype=F64), dtype) if slew else None

    @property
    def entry(self):
        return "plant" if self.plant != "none" or self.with_w else "slew"

    @property
    def form(self):
        if self.model is not None:
            return f"{self.model}/{self.plant}" + ("/slew" if self.slew else "")
        return self.plant

    def oracle_plant(self, cast=lambda t: t):
        if self.plant in ("lin", "lin_nof"):
            return ("lin", cast(self.Fp), None if self.fp is None else cast(self.fp))
        if self.plant in KNOWN:
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


def _dev(t, dtype):
    if not torch.is_tensor(t):
        return t
    return t.to(DEV, dtype) if t.is_floating_point() else t.to(DEV)


def device_call(c, impl=None, opts=None, poison=False):
    """abi_episode on the case: under a slew-rate penalty the augmented problem (slew_augment in the case's dtype, the
    float32 oracle's own rounding), x_init [prev; x0], a LinDx plant's F~, f~ and [0; w]; a time-invariant input a
    stride-0 view over time made on the device.  Every output starts at NaN (info -1), the workspace too when
    `poison`."""
    m, dt = c.m, c.dtype
    P = c.P
    x0, C, c_, F, f = (None if P[k] is None else P[k].to(dt) for k in ("x0", "C", "c", "F", "f"))
    Fp, fp, w = (None if t is None else t.to(dt) for t in (c.Fp, c.fp, c.w))
    n = c.n
    if c.slew:
        if Fp is not None:
            Fp, fp = slew_augment(c.n, m, SLEW, C[:1], c_[:1], Fp, fp)[2:]
        C, c_, F, f = slew_augment(c.n, m, SLEW, C, c_, F, f)
        x0 = torch.cat((c.prev.to(dt), x0), 1)
        w = None if w is None else torch.cat((w.new_zeros(*w.shape[:2], m), w), 2)
        n = c.n + m
    ins = []
    for k, t in (("x0", x0), ("C", C), ("c", c_), ("F", F), ("f", f)):
        ins.append(_dev(t[:1], dt).expand(t.shape) if t is not None and k in P["time_invariant"] else _dev(t, dt))
    plant = None
    if Fp is not None:
        plant = ("lin", _dev(Fp, dt), _dev(fp, dt))
    elif c.pkind is not None:
        plant = (c.pkind | (DYN_CTRL_PASSTHROUGH if c.slew else 0), c.pparams)
    dyn = None
    if c.dyn is not None:
        dyn = (c.dyn[0] | (DYN_CTRL_PASSTHROUGH if c.slew else 0), c.dyn[1])
    w_dev = _dev(w, dt) if c.with_w or c.plant == "self" else None
    u0 = torch.zeros(c.T, c.B, m, dtype=dt, device=DEV)
    with kernel_env(impl):
        return abi_episode(n, m, c.T, c.n_steps, *ins, u0, **{k: _dev(v, dt) for k, v in c.kw.items()}, **opts,
                           dyn=dyn, poison=poison, n_prev=m if c.slew else 0, plant=plant, w=w_dev,
                           nan_outputs=True)


def oracle_forward(c, opts):
    """plant_oracle's episode in float64, and in float32 for a float32 case (the yardstick)."""
    okw = dict(c.kw, **opts)
    P = c.P

    def run(cast):
        return porc.receding_horizon_lin(
            c.n, c.m, c.T, c.n_steps, *[None if P[k] is None else cast(P[k]).contiguous()
                                        for k in ("x0", "C", "c", "F", "f")],
            plant=c.oracle_plant(cast), w=None if c.w is None else cast(c.w),
            slew_rate_penalty=SLEW if c.slew else None, prev_ctrl=None if c.prev is None else cast(c.prev),
            coupled=False, **{k: cast(v) if torch.is_tensor(v) and v.is_floating_point() else v
                              for k, v in okw.items()})
    o64 = run(lambda t: t.double())
    o32 = run(_f32) if c.dtype == F32 else None
    return o64, o32


def oracle_sweep(c, saved, wx, wu):
    """plant_oracle's sweep on the device's own xs, us and plans (plan_x augmented under a penalty): float64, and
    float32 for a float32 case."""
    s, _, xs, us, plan_x, plan_u = saved
    k = c.m if c.slew else 0
    got = [s.pad.crop_n(xs).cpu()[..., k:], s.pad.crop_m(us).cpu(), s.pad.crop_n(plan_x).cpu(),
           s.pad.crop_m(plan_u).cpu()]
    P = c.P

    def run(cast):
        cc = lambda t: cast(t) if torch.is_tensor(t) else t  # noqa: E731
        return porc.receding_horizon_backward(
            c.n, c.m, c.T, cc(P["C"]).contiguous(), cc(P["c"]).contiguous(),
            None if P["F"] is None else cc(P["F"]).contiguous(), cc(P["f"]), *[cc(t) for t in got], cc(wx), cc(wu),
            u_lower=cc(c.kw.get("u_lower")), u_upper=cc(c.kw.get("u_upper")), step=c.mstep,
            theta=None if c.theta is None else cc(c.theta), slew_rate_penalty=SLEW if c.slew else None,
            prev_ctrl=None if c.prev is None else cc(c.prev), plant=c.oracle_plant(cast))
    o64 = run(lambda t: t.double())
    o32 = run(_f32) if c.dtype == F32 else None
    return o64, o32


def device_grads(c, g):
    """The device sweep's outputs by oracle name, on the CPU, cropped to the system's blocks under a slew-rate
    penalty (whose detached entries of dx_init and dw must be exactly 0).  plant "self": the plant entry gives the
    model's own step part in dF_p, df_p; the oracle gives it to dF[0], df[0], so they are added there."""
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
        dF, df = out["dF"].clone(), None if out["df"] is None else out["df"].clone()
        dF[0] += out.pop("dF_p")
        dfp = out.pop("df_p")
        if df is not None:
            df[0] += dfp
        out.update(dF=dF, df=df)
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
        if name in ("dF_p", "df_p"):
            want, w32 = want[0], None if w32 is None else w32[0]
        assert a.shape == want.shape, f"{tag}: {name} shape {tuple(a.shape)} vs {tuple(want.shape)}"
        assert bool(torch.isfinite(a).all()), f"{tag}: {name} not finite"
        within(tag, name, a, want, w32, c.dtype)
        _note(c.dtype, f"backward {name}", maxdiff(a, want) / max(1.0, float(want.abs().max())))


def check_forward(tag, c, r, o64, o32, several):
    """gpu_harness.check_episode_forward on the system's states (the augmented state's previous control dropped under
    a slew-rate penalty); its largest error and departures recorded for test_zz_coverage."""
    r = dict(r, x=r["x"][..., c.m:] if c.slew else r["x"])
    err, n_dep, n_cmp = check_episode_forward(tag, r, o64, o32, c.kw, c.dtype, several)
    DEPARTED.setdefault(c.dtype, []).append((n_dep, n_cmp))
    _note(c.dtype, "forward x/u/u_next/plans", err)


def check_known_forward(tag, c, r):
    """A known model's episode without an iLQR oracle: applied controls are the plans' first, within the clamp; each
    plan starts at its x_k; x_{k+1} = plant(x_k, u_k) + w_k and each plan's rollout is the model's step (CPU torch
    forward in float64, float32 the yardstick); under a slew-rate penalty x_{k+1}[:m] is u_k bitwise."""
    s, _, xs, us, plan_x, plan_u = r["saved"]
    xs, us, plan_x, plan_u = [t.cpu() for t in (xs, us, plan_x, plan_u)]
    k = c.m if c.slew else 0
    assert torch.equal(us, plan_u[:, 0]), f"{tag}: applied controls"
    assert torch.equal(plan_x[:, 0], xs[:-1]), f"{tag}: each plan starts at its x_k"
    assert bool((plan_u.abs() <= c.kw["u_upper"]).all()), f"{tag}: a control beyond the clamp"
    if c.slew:
        assert torch.equal(xs[1:, :, :k], us), f"{tag}: the carried previous control is not u_k"
    flat = lambda t: t.reshape(-1, t.shape[-1])  # noqa: E731

    def cmp(what, step, theta, x, u, nxt, add=None):
        th = theta.repeat(flat(x).shape[0] // theta.shape[0], 1)
        w64 = step(flat(x).double(), flat(u).double(), th.double()).view(nxt.shape)
        w32 = step(flat(x).float(), flat(u).float(), th.float()).view(nxt.shape) if c.dtype == F32 else None
        if add is not None:
            w64 = w64 + add.double()
            w32 = None if w32 is None else w32 + add.float()
        within(tag, what, nxt, w64, w32, c.dtype)
    if c.pstep is not None:
        cmp("plant step + w", c.pstep, c.ptheta, xs[:-1, :, k:], us, xs[1:, :, k:], c.w)
    cmp("plan rollout", c.mstep, c.theta, plan_x[:, :-1, :, k:], plan_u[:, :-1], plan_x[:, 1:, :, k:])


def check_poisoned(tag, c, clean, g_clean, impl, opts, wx, wu):
    """Both calls again with every workspace byte and output at 0xFF: every output finite and bitwise the same."""
    r, _, _ = device_call(c, impl, opts, poison=True)
    for k in ("x", "u", "costs", "info", "u_next"):
        a = r[k]
        assert not a.is_floating_point() or bool(torch.isfinite(a).all()), f"{tag} poisoned: {k} not finite"
        assert torch.equal(a, clean[k]), f"{tag} poisoned: {k} differs"
    for i in (4, 5):
        assert torch.equal(r["saved"][i], clean["saved"][i]), f"{tag} poisoned: plans differ"
    with kernel_env(impl):
        g, _, _ = abi_episode_backward(clean["saved"], wx, wu, poison=True)
    for name, a, b in zip(GNAMES, g, g_clean):
        assert (a is None) == (b is None), f"{tag} poisoned: {name}"
        if a is not None:
            assert bool(torch.isfinite(a).all()), f"{tag} poisoned: {name} not finite"
            assert torch.equal(a, b), f"{tag} poisoned: {name} differs by {float((a - b).abs().max()):.3e}"


def loss_weights(c, seed):
    """dl_dx [n_steps+1, B, n], dl_du; and as the device takes them (m zeros in front under a slew-rate penalty)."""
    wx, wu = ro.loss_weights(c.n_steps, c.B, c.n, c.m, seed)
    wx, wu = round_through(wx, c.dtype), round_through(wu, c.dtype)
    gx = torch.cat((wx.new_zeros(*wx.shape[:2], c.m), wx), 2) if c.slew else wx
    return wx, wu, gx.to(DEV, c.dtype), wu.to(DEV, c.dtype)


def record(c, name, route):
    """Coverage: the case's entry ran step plan `name` (None: a known model's) and adjoint route `route`."""
    if name is not None:
        SEEN.add(("plan", c.entry, c.dtype, name))
    SEEN.add(("route", c.entry, c.dtype, route))
    SEEN.add(("form", c.form))
    return name


def run(tag, c, impl=None, seed=0, lqr_iter=2, fixed=True, want_plan=None, want_route=None, poison=False,
        best_cost_eps=1e-4):
    """One episode and its sweep through the C ABI, checked against the oracle; the plan, route and launch count."""
    if c.model is not None:
        opts = dict(ro.fixed_opts(lqr_iter), linesearch_decay=0.2, max_linesearch_iter=10)
    else:
        opts = ro.fixed_opts(lqr_iter) if fixed else dict(lqr_iter=lqr_iter, eps={F64: 1e-7, F32: 1e-4}[c.dtype])
    opts["best_cost_eps"] = best_cost_eps
    N_aug = c.n + (c.m if c.slew else 0)
    tag = (f"{tag} n{c.n}m{c.m} {DT[c.dtype]} B={c.B} T={c.T} steps={c.n_steps} {c.mode} plant={c.plant} "
           f"w={c.with_w} slew={c.slew} MPCB200_KERNEL={impl}")
    r, _, plan = device_call(c, impl, opts)
    s = r["saved"][0]
    name = None
    if c.model is None:
        name = plan_name(plan, impl, N_aug, c.m, c.dtype)
        if want_plan is not None:
            assert name == want_plan, f"{tag}: plan {plan_str(plan)} ({name}), expected {want_plan}"
        for k in c.P["time_invariant"]:
            ts = getattr(s.dims, k + "_tstride")
            assert ts == -1, f"{tag}: {k} staged with time stride {ts}, not as time invariant"
        o64, o32 = oracle_forward(c, opts)
        check_forward(tag, c, r, o64, o32, fixed and (lqr_iter > 1 or c.n_steps > 1))
    else:
        check_known_forward(tag, c, r)
    wx, wu, gx, gu = loss_weights(c, seed)
    with kernel_env(impl):
        g, launches, adj_plan = abi_episode_backward(r["saved"], gx, gu, nan_outputs=True)
    assert len(g) == (10 if c.entry == "plant" else 6), f"{tag}: {len(g)} outputs"
    route = ro.adjoint_route(s.pad.N, s.pad.M, c.T, c.B, c.dtype, impl)
    if want_route is not None:
        assert route == want_route, f"{tag}: the case is meant for the {want_route} route, the rule gives {route}"
    ro.check_route(tag, route, launches, adj_plan, known=c.model is not None)
    record(c, name, route)
    b64, b32 = oracle_sweep(c, r["saved"], wx, wu)
    check_backward(tag, c, g, b64, b32)
    if poison:
        check_poisoned(tag, c, r, g, impl, opts, gx, gu)
    return r, g


# ------------------------------------------------------------------------------------------------------------------
# the slew sweep at every instance reachable as an augmented shape; plant episodes at every instance
# ------------------------------------------------------------------------------------------------------------------
# systems (n, m) whose augmented (n + m, m) is a compiled instance; (5, 1) -> (6, 1) runs zero padded at (6, 2), so
# n_prev = 1 < dims->m; (16, 4) -> (20, 4) has no instance (the large-shape kernels)
SLEW_SYSTEMS = [(N - M, M) for N, M in INSTANCES if N > M] + [(5, 1), (16, 4)]
PLANT_SHAPES = INSTANCES + [(6, 1), (20, 4)]


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("n,m", SLEW_SYSTEMS, ids=[f"n{n}m{m}" for n, m in SLEW_SYSTEMS])
def test_slew_every_instance(n, m, dtype):
    """B = 1 (unbounded or u_zero_I) and a batch tail of 257 (bounds scalar or tensor + delta_u); n_steps 1, 2 and 3,
    not test_receding_oracle_gpu's 1, 2 and 5; a non-zero previous control.  Bounded batch tails over 5 control steps
    of a slew-rate or plant episode leave the forward rule by round-off, not by a wrong kernel (the sweep, checked on
    the device's own plans, stays within its tolerance there): with tensor bounds without delta_u up to 37% of the
    problems departed in float64, each by at most 4e-8 (pnqp end points that round-off puts on or off a bound), and
    with scalar bounds in float32 the kept problems' costs missed the float32 yardstick (7.7e-4 against 8.4e-5 at
    (5, 1) on a plant, 5.3e-4 against 6.7e-5 at (3, 1) under a penalty).  Tensor bounds without delta_u run in
    test_plant_forms and test_input_forms instead (B = 12, 2 or 3 control steps)."""
    k = SLEW_SYSTEMS.index((n, m)) + (dtype == F32)
    for j, (B, modes) in enumerate(((1, ("plain", "mask")), (257, ("box", "boxT")))):
        c = Case(n, m, (3, 6)[(k + j) % 2], B, dtype, (1, 2, 3)[(k + j) % 3], modes[k % len(modes)], "none", False,
                 True, seed=1000 + 10 * k + j)
        run("slew instance", c, seed=1000 + k)


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("n,m", PLANT_SHAPES, ids=[f"n{n}m{m}" for n, m in PLANT_SHAPES])
def test_plant_every_instance(n, m, dtype):
    """A LinDx model on a perturbed LinDx plant (with and without the plant's f), with w: B = 1 and 257, the bound
    kinds as in test_slew_every_instance."""
    k = PLANT_SHAPES.index((n, m)) + (dtype == F32)
    for j, (B, modes) in enumerate(((1, ("plain", "mask")), (257, ("box", "boxT")))):
        c = Case(n, m, (3, 6)[(k + j) % 2], B, dtype, (1, 2, 3)[(k + j) % 3], modes[k % len(modes)],
                 ("lin", "lin_nof")[(k + j) % 2], True, False, seed=1100 + 10 * k + j)
        run("plant instance", c, seed=1100 + k)


PLANT_FORMS = {"lin": dict(), "lin_nof": dict(), "model_nof": dict(f_T="none"), "both_nof": dict(f_T="none"),
               "self": dict()}


@pytest.mark.parametrize("slew", [False, True], ids=["plain", "slew"])
@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("form", list(PLANT_FORMS))
def test_plant_forms(form, dtype, slew):
    """The plant's f present and absent, on a model with and without f; and the model itself disturbed (plant None,
    w given), whose step part the plant entry returns in the plant's outputs."""
    i = list(PLANT_FORMS).index(form)
    plant = {"model_nof": "lin", "both_nof": "lin_nof"}.get(form, form)
    c = Case(4, 2, 6, 12, dtype, 3, ("box", "tensor", "boxT", "plain", "mask")[i], plant, True, slew,
             seed=1200 + 10 * i + slew, **PLANT_FORMS[form])
    SEEN.add(("form", "plant " + form))
    run(f"plant form {form}", c, seed=1200 + i)


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("name,slew", [("pendulum", False), ("pendulum", True), ("cartpole", False)])
def test_known_plant_on_linear_model(name, slew, dtype):
    """Pendulum (3, 1) and cartpole (5, 1) plants on a LinDx model of their shape, with w; the pendulum's
    passthrough kind under a slew-rate penalty at (4, 1).  (Cartpole's augmented (6, 1) runs zero padded at (6, 2),
    where a known plant cannot step.)  The plant's clamp binds."""
    n = 5 if name == "cartpole" else 3
    c = Case(n, 1, 8, 9, dtype, 3, "plain", name, True, slew, seed=1300 + n + slew)
    run(f"{name} plant", c, seed=1300, lqr_iter=3)


KNOWN_PAIRS = [("pendulum", "pendulum_full", 1), ("pendulum", "pendulum_full", 7), ("pendulum", "pendulum_full", 300),
               ("cartpole", "cartpole", 7)]


@pytest.mark.parametrize("slew", [False, True], ids=["plain", "slew"])
@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("model,plant,B", KNOWN_PAIRS, ids=[f"{a}_on_{b}_B{B}" for a, b, B in KNOWN_PAIRS])
def test_known_on_known(model, plant, B, dtype, slew):
    """A known model on a known plant with other parameters, with w: the plant's parameter gradient per problem.
    Pendulum on the five-parameter pendulum at B = 7 is the first batch whose plant parameter part (5 per problem)
    overflows a slot sized by the model's 3 in float64 (test_receding_plant_oracle_cpu)."""
    n = 5 if model == "cartpole" else 3
    c = Case(n, 1, 8, B, dtype, 3, "clamp", plant, True, slew, seed=1400 + B + slew, model=model)
    r, _ = run(f"{model} on {plant}", c, seed=1400, lqr_iter=4, poison=B == 7)
    if not slew:                        # the slew-rate penalty keeps cartpole's controls inside its clamp
        assert bool((r["saved"][5].abs() == c.kw["u_upper"]).any()), "no control reaches the clamp"


# ------------------------------------------------------------------------------------------------------------------
# every step plan on both sides of its switch; the large-shape kernels; every adjoint route
# ------------------------------------------------------------------------------------------------------------------
GROUPS = list(SWITCH_PLANS)


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("group", GROUPS)
def test_plans_at_switch(group, dtype):
    """Both entries just below and at the switch horizon T* of the solve's step plan, under the default dispatch
    and each kernel forced, at the first instance with n > m that has the switch (the slew entry runs the system
    (n - m, m)); the first run at T* of each entry also runs poisoned."""
    pick = pick_switch(group, dtype, augmentable=True)
    if pick is None:
        pytest.skip(f"no instance with n > m has a {group} switch of the loop's step within the oracle's horizons")
    N, M, Ts, impls = pick
    gi = GROUPS.index(group)
    for k, T in enumerate((Ts - 1, Ts)):
        for j, impl in enumerate(impls):
            want = loop_plan(N, M, dtype, T, impl)
            if want is None:
                continue
            for e, slew in enumerate((False, True)):
                mode = "plain" if slew else ("box", "plain", "boxT")[(gi + k + j) % 3]
                c = Case(N - M if slew else N, M, T, 8, dtype, 1 + k, mode, "none" if slew else "lin", not slew,
                         slew, seed=1500 + 10 * gi + 2 * k + e)
                run(f"{group} (T*={Ts})", c, impl, seed=1500 + gi, want_plan=plan_name(want, impl, N, M, dtype),
                    poison=k == 1 and j == 0)


# (system n, m, slew, MPCB200_KERNEL, mode): no instance at (20, 4); knob 3 at instances, where a LinDx plant's step
# runs the large-shape rollout too
LARGE = [(20, 4, False, None, "boxT"), (16, 4, True, None, "box"), (8, 2, False, 3, "box"), (6, 2, True, 3, "plain"),
         (16, 4, False, 3, "plain"), (12, 4, True, 3, "tensor")]


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("n,m,slew,impl,mode", LARGE, ids=[f"n{c[0]}m{c[1]}_{'slew' if c[2] else 'plant'}_k{c[3]}"
                                                           for c in LARGE])
def test_large_shape_kernels(n, m, slew, impl, mode, dtype):
    c = Case(n, m, 6, 5, dtype, 2, mode, "none" if slew else "lin", not slew, slew, seed=1600 + n + slew)
    run("large", c, impl, seed=1600, want_plan="large", want_route="large", poison=impl is None)


ENTRIES = [False, True]


@pytest.mark.parametrize("slew", ENTRIES, ids=["plant", "slew"])
@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
def test_route_fused(dtype, slew):
    c = Case(6 if slew else 8, 2, 6, 8, dtype, 3, "tensor", "none" if slew else "lin", not slew, slew, seed=1700)
    run("fused", c, seed=1700, lqr_iter=3, want_route="fused", poison=True)


@pytest.mark.parametrize("slew", ENTRIES, ids=["plant", "slew"])
def test_route_three_launch_by_alignment(slew):
    """f32 (4, 2) at B = 7: time strides that are no 16-byte multiple."""
    c = Case(2 if slew else 4, 2, 6, 7, F32, 3, "box", "none" if slew else "lin", not slew, slew, seed=1710)
    run("3-launch by alignment", c, seed=1710, lqr_iter=3, want_route="three_align", poison=True)


@pytest.mark.parametrize("slew", ENTRIES, ids=["plant", "slew"])
@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
def test_route_three_launch_by_gains(dtype, slew):
    """(16, 4) from the instance's gain-store switch on: the nested step keeps its gains in the workspace."""
    sw = switches(16, 4, dtype)
    assert sw["adjoint"] is not None and sw["generic"] is not None
    T = max(sw["adjoint"], sw["generic"])
    c = Case(12 if slew else 16, 4, T, 8, dtype, 2, "box", "none" if slew else "lin", not slew, slew, seed=1720)
    run("3-launch by gains", c, seed=1720, want_route="three_gains", poison=True)


# ------------------------------------------------------------------------------------------------------------------
# grid-stride loops past epgrad_grid's cap: a pool of K problems, element b is pool problem b mod K
# ------------------------------------------------------------------------------------------------------------------
# name -> (system n, m, slew, plant, w, T, B, {loop: items per pass-1 grid thread ... the loops the case targets})
GRID = {
    # the detach mask of the carried gradient g over B N items, N = 6 not a power of two
    "slew_detach": dict(n=4, m=2, slew=True, plant="none", w=False, T=3, B=180_000),
    # dw, g (B N) and the LinDx plant's dF (B N P) under the plant entry's detach mask
    "plant_lin_w": dict(n=4, m=2, slew=True, plant="lin", w=True, T=3, B=180_000),
    # the known plant's dtheta (B NP) and the one-thread-per-problem stage loop (B)
    "plant_pendulum": dict(n=3, m=1, slew=False, plant="pendulum", w=True, T=3, B=GRID_CAP + 77),
}


def grid_loops(name):
    """Items of the loops each grid case targets, and whether each loop's grid is capped (its items / 256 blocks
    exceed 4096): the init / accumulate kernels size their grid by T B P^2, the stage kernel by T B max(N, M)."""
    g = GRID[name]
    N, M = g["n"] + (g["m"] if g["slew"] else 0), g["m"]
    P, B, T = N + M, g["B"], g["T"]
    capped_acc = T * B * P * P > GRID_CAP
    loops = {"g": (B * N, capped_acc)}
    if g["w"]:
        loops["dw"] = (B * N, capped_acc)
    if g["plant"] in ("lin", "lin_nof"):
        loops["plant dF"] = (B * N * P, capped_acc)
    if g["plant"] in KNOWN:
        loops["plant dtheta"] = (B * KNOWN_NP[g["plant"]], capped_acc)
        loops["stage"] = (B, T * B * max(N, M) > GRID_CAP)
    return N, loops


KNOWN_NP = {"pendulum": 3, "pendulum_full": 5, "cartpole": 4}


def grid_pool(name):
    """(K, idx): the pool size, coprime to the 256-thread block and to N, and the pool problem of each element."""
    N, _ = grid_loops(name)
    K = pool_size(256, N)
    return K, torch.arange(GRID[name]["B"]) % K


@pytest.mark.parametrize("name", list(GRID))
def test_grid_stride_passes(name):
    """float32, T = 3, n_steps 2: every copy bitwise its pool problem (x, u, plans, every gradient), the pool against
    the oracle."""
    g = GRID[name]
    K, idx = grid_pool(name)
    pool = Case(g["n"], g["m"], g["T"], K, F32, 2, "plain", g["plant"], g["w"], g["slew"], seed=1800)
    c = pool.take(idx)
    opts = dict(ro.fixed_opts(1), best_cost_eps=1e-4)
    r, _, plan = device_call(c, None, opts)
    wx, wu, _, _ = loss_weights(pool, 1800)
    gx = wx.index_select(1, idx)
    gx = torch.cat((gx.new_zeros(*gx.shape[:2], c.m), gx), 2) if c.slew else gx
    gu = wu.index_select(1, idx).to(DEV, F32)
    grads, launches, adj_plan = abi_episode_backward(r["saved"], gx.to(DEV, F32), gu, nan_outputs=True)
    s = r["saved"][0]
    route = ro.adjoint_route(s.pad.N, s.pad.M, c.T, c.B, F32, None)
    ro.check_route(name, route, launches, adj_plan)
    record(c, plan_name(plan, None, s.pad.N, s.pad.M, F32), route)
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
    # the pool problems against the oracle
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
# input forms, the default stop rule, the carried previous control
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("slew", ENTRIES, ids=["plant", "slew"])
@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("form", list(ro.FORMS))
def test_input_forms(form, dtype, slew):
    """test_receding_oracle_gpu.FORMS through the plant entry (a LinDx plant, w) and through the slew entry: F with
    T slices, f absent or of T slices, a time-invariant F and cost (stride 0 over time, asserted), u_zero_I."""
    i = list(ro.FORMS).index(form)
    c = Case(6 if slew else 8, 2, ro.FORMS_T, 12, dtype, 2, ("box", "tensor", "boxT", "mask", "plain", "box")[i],
             "none" if slew else "lin", not slew, slew, seed=1900 + 10 * i + slew, **ro.FORMS[form])
    run(form, c, seed=1900 + i, lqr_iter=3, poison=i == 0)


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
def test_default_stop_rule(dtype):
    """The default stop rule couples the batch through its stop decision; the oracle's loop decides on the same
    batch-wide norm.  A slew-rate episode on a LinDx plant with w."""
    c = Case(6, 2, 10, 16, dtype, 3, "plain", "lin", True, True, seed=2000)
    run("default stop", c, seed=2000, lqr_iter=10, fixed=False)


@pytest.mark.parametrize("plant", ["lin", "pendulum_full"])
def test_carried_control_is_the_applied_one(monkeypatch, plant):
    """receding_horizon under a slew-rate penalty with a disturbance: the augmented state's previous-control block
    x_{k+1}[:m] is bitwise u_k.  w reaches the plant's states only."""
    from mpc.pytorch_b200 import step
    from mpc.pytorch_b200.control import receding_horizon
    from mpc.pytorch_b200.dynamics import PendulumDx
    from mpc.pytorch_b200.solver import MPC, LinDx, QuadCost
    B, T, steps = 9, 8, 4
    if plant == "lin":
        n, m = 4, 2
        C, c_, F, f, x0 = (t.to(DEV) for t in episode_linear_inputs(2100, B, T, n, m, F64, "box")[0].values()
                           if torch.is_tensor(t))
        dx, pl = LinDx(F, f), LinDx(F[:1] * 1.02, f[:1] + 0.01)
        ctrl = MPC(n, m, T, u_lower=-0.25, u_upper=0.25, lqr_iter=3, verbose=-1)
    else:
        n, m = 3, 1
        mod, _, _, P, kw, _, _ = episode_known_inputs("pendulum", B, T, F64, 2100)
        C, c_, x0 = P["C"].to(DEV), P["c"].to(DEV), P["x0"].to(DEV)
        dx, pl = mod, known_plant_module("pendulum_full")[1]
        ctrl = MPC(n, m, T, u_lower=kw["u_lower"], u_upper=kw["u_upper"], lqr_iter=4, verbose=-1)
    ctrl.slew_rate_penalty = SLEW
    ctrl.prev_ctrl = 0.1 * torch.ones(B, m, dtype=F64, device=DEV)
    w = 0.05 * torch.randn(steps, B, n, generator=torch.Generator().manual_seed(2101), dtype=F64).to(DEV)
    seen = []
    real = step.episode_raw
    monkeypatch.setattr(step, "episode_raw", lambda *a, **k: seen.append(real(*a, **k)) or seen[-1])
    ep = receding_horizon(ctrl, x0, QuadCost(C, c_), dx, steps, plant=pl, disturbance=w)
    assert len(seen) == 1, "the episode did not run as one graph"
    xs, us = seen[0]["x"], seen[0]["u"]
    assert xs.shape[2] == n + m
    assert torch.equal(xs[1:, :, :m], us), "the carried previous control is not the applied control"
    assert torch.equal(xs[0, :, :m], ctrl.prev_ctrl)
    assert torch.equal(ep.x, xs[:, :, m:])
    SEEN.add(("form", "carried control " + plant))


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


NEEDED_FORMS = ({"none", "lin", "lin_nof", "self", "pendulum", "cartpole"}
                | {f"plant {f}" for f in PLANT_FORMS}
                | {f"{a}/{b}" + s for a, b, _ in KNOWN_PAIRS for s in ("", "/slew")}
                | {"carried control lin", "carried control pendulum_full"})


def test_zz_coverage():
    if not SEEN:
        pytest.skip("no episode test of this module ran")
    missing = []
    for dtype in (F64, F32):
        for entry in ("plant", "slew"):
            plans = {x[3] for x in SEEN if x[:3] == ("plan", entry, dtype)}
            routes = {x[3] for x in SEEN if x[:3] == ("route", entry, dtype)}
            print(f"{DT[dtype]} {entry}: step plans {sorted(plans)}; adjoint routes {sorted(routes)}")
            missing += [f"{DT[dtype]} {entry} plan {p}" for p in sorted(_needed_plans(dtype) - plans)]
            need_routes = {"fused", "three_shape", "three_gains", "large"}
            if dtype == F32:
                need_routes.add("three_align")
            missing += [f"{DT[dtype]} {entry} route {r}" for r in sorted(need_routes - routes)]
    forms = {x[1] for x in SEEN if x[0] == "form"}
    missing += [f"plant form {f}" for f in sorted(NEEDED_FORMS - forms)]
    for (dtype, what), v in sorted(ERRS.items(), key=lambda kv: (DT[kv[0][0]], kv[0][1])):
        print(f"{DT[dtype]} {what}: largest error {v:.3e} of max(1, max|want|)")
    for dtype, v in DEPARTED.items():
        print(f"{DT[dtype]}: problems departing from the oracle {sum(a for a, _ in v)} of {sum(b for _, b in v)} "
              f"compared, in {sum(a > 0 for a, _ in v)} of {len(v)} runs")
    assert not missing, "never run: " + ", ".join(missing)
