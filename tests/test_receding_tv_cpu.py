"""CPU: time-varying episodes.  The C ABI of mpcb200_episode_window_* and mpcb200_episode_backward_window_* returns
its status codes before touching a device, and their workspaces are the episode's (sweep's) layout followed by one
256-byte aligned buffer per windowed input; receding_horizon(..., time_varying=True) rejects a short axis, a Module
cost, a plant or bounds on the wrong axis before anything runs; the GPU module's large case reaches the window
kernel's second grid-stride pass; and the float64 window oracle (oracle/window_oracle.py), fed the reference's own
plans, reproduces the reference's windowed loop (tests/golden/receding_tv_f64.npz), is lqr_oracle's / slew_oracle's /
plant_oracle's bitwise at n_steps = 1, and their time-invariant episode for inputs constant along the axis.  No
kernel is launched here."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from mpc.pytorch_b200 import _lib
from mpc.pytorch_b200._lib import Dims, IlqrOpts, MpcB200Error, Params, Plant, Window
from mpc.pytorch_b200.control import receding_horizon
from mpc.pytorch_b200.dynamics import CartpoleDx, PendulumDx
from mpc.pytorch_b200.solver import MPC, LinDx, QuadCost
from oracle import lqr_oracle as orc
from oracle import plant_oracle as porc
from oracle import slew_oracle as sorc
from oracle import window_oracle as wo
from tests.gpu_harness import episode_known_step

NULL, BAD, NO_DEVICE = 1, 2, 6      # a well-formed call gets as far as looking for a device
# With a device present a well-formed call would capture and launch on the fake addresses below, so those calls are
# made only where there is none; the refusals, which return before any device work, are checked everywhere.
WELL_FORMED_CHECKED = not torch.cuda.is_available()
FAKE = 1 << 20                      # a 256-byte aligned address the checks never dereference
FW_NAMES = ("C", "c", "F", "f", "F_plant", "f_plant", "w", "x_init", "u_init", "u_lower", "u_upper", "u_zero_I",
            "xs", "us", "costs", "info", "u_next", "plan_x", "plan_u")
BW_NAMES = ("C", "c", "F", "F_plant", "u_lower", "u_upper", "xs", "us", "plan_x", "plan_u", "dl_dxs", "dl_dus",
            "dx_init", "dC", "dc", "dF", "df", "dtheta", "dF_plant", "df_plant", "dtheta_plant", "dw")


def dims(B=8, T=6, n=6, m=2, kind=0, has_f=1, bounds_kind=0):
    return Dims(B=B, T=T, n=n, m=m, F_T=T - 1, has_f=has_f, bounds_kind=bounds_kind, max_ls_iter=10,
                pnqp_max_iter=20, do_rollout=1, dynamics_kind=kind)


def opts(m=2):
    return IlqrOpts(lqr_iter=5, not_improved_lim=5, m_ref=m, eps=1e-7, best_cost_eps=1e-4)


def window(L=9, on=_lib.WIN_COST | _lib.WIN_DYN):
    return Window(L=L, on=on)


def forward(d, w, n_steps=4, pl=None, null=(), nbytes=None, esz=4):
    L = _lib.lib()
    if nbytes is None:
        nbytes = L.mpcb200_episode_window_workspace_bytes(ctypes.byref(d), ctypes.byref(opts(d.m)),
                                                          ctypes.byref(w) if w is not None else None, esz)
    ptrs = [None if k in null or k in ("w", "plan_x", "plan_u", "u_zero_I") or
            (k in ("F_plant", "f_plant") and pl is None) or (k in ("u_lower", "u_upper") and d.bounds_kind == 0)
            else FAKE for k in FW_NAMES]
    fn = L.mpcb200_episode_window_f32 if esz == 4 else L.mpcb200_episode_window_f64
    return fn(ctypes.byref(d), ctypes.byref(Params()), ctypes.byref(opts(d.m)),
              ctypes.byref(w) if w is not None else None, ctypes.byref(pl) if pl is not None else None, n_steps,
              *ptrs, FAKE, nbytes, None)


def backward(d, w, n_steps=4, n_prev=0, pl=None, null=(), nbytes=None):
    L = _lib.lib()
    prec = ctypes.byref(pl) if pl is not None else None
    if nbytes is None:
        nbytes = L.mpcb200_episode_backward_window_workspace_bytes(ctypes.byref(d), n_prev, ctypes.byref(w), prec, 4)
    skip = {"dtheta", "dF_plant", "df_plant", "dtheta_plant", "dw", "F_plant"} if pl is None else {"dtheta"}
    ptrs = [None if k in null or k in skip or (k in ("u_lower", "u_upper") and d.bounds_kind == 0) or
            (k == "df_plant" and pl is not None and not pl.has_f) else FAKE for k in BW_NAMES]
    return L.mpcb200_episode_backward_window_f32(ctypes.byref(d), ctypes.byref(Params()), ctypes.byref(w), prec,
                                                 n_steps, n_prev, *ptrs, FAKE, nbytes, None)


def well_formed(call):
    """A call that passes every argument check: NO_DEVICE without a device; not made with one."""
    if WELL_FORMED_CHECKED:
        assert call() == NO_DEVICE


def test_forward_status_codes():
    d = dims()
    well_formed(lambda: forward(d, window()))
    assert forward(d, None) == NULL
    assert forward(d, window(L=8)) == BAD                         # L < n_steps + T - 1
    well_formed(lambda: forward(d, window(L=10)))                 # a longer axis covers the episode
    assert forward(d, window(on=_lib.WIN_DYN)) == BAD             # the cost must be windowed
    assert forward(d, window(on=_lib.WIN_COST | 16)) == BAD       # unknown bit
    assert forward(d, window(on=_lib.WIN_COST | _lib.WIN_BOUNDS)) == BAD      # no tensor bounds
    well_formed(lambda: forward(dims(bounds_kind=2), window(on=_lib.WIN_COST | _lib.WIN_BOUNDS)))
    assert forward(d, window(on=_lib.WIN_COST | _lib.WIN_PLANT)) == BAD       # no LinDx plant
    well_formed(lambda: forward(d, window(on=_lib.WIN_COST | _lib.WIN_PLANT), pl=Plant(kind=0, has_f=1)))
    assert forward(d, window(), null=("C",)) == NULL
    assert forward(d, window(), null=("f",)) == NULL
    assert forward(d, window(), null=("xs",)) == NULL
    w = window()
    w.F_tstride = -2
    assert forward(d, w) == BAD
    assert forward(d, window(), nbytes=1024) == BAD


def test_backward_status_codes():
    d = dims()
    well_formed(lambda: backward(d, window()))
    assert backward(d, window(L=8)) == BAD
    assert backward(d, window(), null=("dC",)) == NULL
    assert backward(d, window(), null=("F",)) == NULL
    assert backward(d, window(), n_prev=-1) == BAD
    well_formed(lambda: backward(d, window(on=_lib.WIN_COST | _lib.WIN_DYN | _lib.WIN_PLANT),
                                 pl=Plant(kind=0, has_f=1)))
    assert backward(d, window(), nbytes=1024) == BAD


def up256(v):
    return (v + 255) // 256 * 256


@pytest.mark.parametrize("esz", [4, 8])
@pytest.mark.parametrize("on", [1, 3, 7, 15])
def test_workspace_formula(esz, on):
    """The window buffers follow the episode's (sweep's) workspace: T slices of C, c and the bounds, F_T of F, T of
    f (T-1 are read), one of a plant's F and f."""
    L = _lib.lib()
    B, T, n, m = 8, 6, 6, 2
    d = dims(B, T, n, m, bounds_kind=2 if on & 4 else 0)
    p = n + m
    w = window(on=on)
    extra = up256(T * B * p * p * esz) + up256(T * B * p * esz)
    if on & _lib.WIN_DYN:
        extra += up256((T - 1) * B * n * p * esz) + up256(T * B * n * esz)
    if on & _lib.WIN_BOUNDS:
        extra += 2 * up256(T * B * m * esz)
    if on & _lib.WIN_PLANT:
        extra += up256(B * n * p * esz) + up256(B * n * esz)
    base = L.mpcb200_episode_workspace_bytes(ctypes.byref(d), ctypes.byref(opts()), esz)
    assert L.mpcb200_episode_window_workspace_bytes(ctypes.byref(d), ctypes.byref(opts()), ctypes.byref(w), esz) == \
        base + extra
    pl = Plant(kind=0, has_f=1)
    base_bw = L.mpcb200_episode_backward_plant_workspace_bytes(ctypes.byref(d), 0, ctypes.byref(pl), esz)
    assert L.mpcb200_episode_backward_window_workspace_bytes(ctypes.byref(d), 0, ctypes.byref(w), ctypes.byref(pl),
                                                             esz) == base_bw + extra


def _case(L=9, B=3, n=4, m=2):
    g = torch.Generator().manual_seed(0)
    C = torch.eye(n + m, dtype=torch.float64).expand(L, B, n + m, n + m)
    c = torch.randn(L, B, n + m, generator=g, dtype=torch.float64)
    F = 0.1 * torch.randn(L - 1, B, n, n + m, generator=g, dtype=torch.float64)
    f = torch.zeros(L - 1, B, n, dtype=torch.float64)
    return torch.zeros(B, n, dtype=torch.float64), QuadCost(C, c), LinDx(F, f)


def test_shape_errors_before_anything_runs():
    """CPU tensors: a well-formed call would reach the kernels and refuse the device; every shape error comes
    first."""
    x0, cost, dx = _case()
    ctrl = MPC(4, 2, 6, lqr_iter=2, verbose=-1)
    with pytest.raises(MpcB200Error, match="slices"):
        receding_horizon(ctrl, x0, QuadCost(cost.C[:-1], cost.c[:-1]), dx, 4, time_varying=True)
    with pytest.raises(MpcB200Error, match="slices"):
        receding_horizon(ctrl, x0, QuadCost(cost.C, cost.c[:-1]), dx, 4, time_varying=True)
    with pytest.raises(MpcB200Error, match="LinDx F"):
        receding_horizon(ctrl, x0, cost, LinDx(dx.F[:-1], dx.f[:-1]), 4, time_varying=True)
    with pytest.raises(MpcB200Error, match="QuadCost"):
        receding_horizon(ctrl, x0, torch.nn.Linear(6, 1).double(), dx, 4, time_varying=True)
    with pytest.raises(MpcB200Error, match="plant"):
        receding_horizon(ctrl, x0, cost, dx, 4, plant=LinDx(dx.F[:1], dx.f[:1]), time_varying=True)
    ctrl.u_lower, ctrl.u_upper = -torch.ones(6, 3, 2, dtype=torch.float64), torch.ones(6, 3, 2, dtype=torch.float64)
    with pytest.raises(MpcB200Error, match="u_lower"):
        receding_horizon(ctrl, x0, cost, dx, 4, time_varying=True)


def test_grid_case_reaches_second_pass():
    """The GPU module's GRID_CASE: its window copy of C has more elements than the capped grid has threads, and that
    cap is the one epgrad_grid launches with."""
    from tests.test_receding_tv_gpu import GRID_CASE, WINDOW_GRID_THREADS
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "mpc", "pytorch_b200", "csrc",
                            "episode_grad.cu")).read()
    cap = re.search(r"static unsigned epgrad_grid\(size_t items\) \{.*?g > (\d+) \? (\d+) : g", src, re.S)
    block = re.search(r"window_stage_kernel<R><<<epgrad_grid\(items\), (\d+), 0, stream>>>", src)
    assert cap and block and cap.group(1) == cap.group(2)
    assert WINDOW_GRID_THREADS == int(cap.group(1)) * int(block.group(1))
    T, n, m, B = GRID_CASE["T"], GRID_CASE["n"], GRID_CASE["m"], GRID_CASE["B"]
    assert T * B * (n + m) ** 2 > WINDOW_GRID_THREADS


# ------------------------------------------------------------------------------------------------------------------
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
KNOWN_SYS = {"pendulum": (PendulumDx, "max_torque"), "cartpole": (CartpoleDx, "force_mag")}


def fixture(case):
    z = np.load(os.path.join(GOLD, "receding_tv_f64.npz"))
    pre = case + "_"
    others = [c + "_" for c in ("pendulum_slew", "linear_plant") if c != case and c.startswith(case)]
    return {k[len(pre):]: torch.from_numpy(z[k]) for k in z.files
            if k.startswith(pre) and not any(k.startswith(o) for o in others)}


def rel(a, b):
    return float((a - b).abs().max()) / max(1.0, float(b.abs().max()))


def known_step(case, t):
    cls, attr = KNOWN_SYS[case.split("_")[0]]
    mod = cls()
    setattr(mod, attr, float(t["clamp"]))
    return episode_known_step(mod)


@pytest.mark.parametrize("case", ["linear", "linear_plant"])
def test_linear_against_reference(case):
    """The window oracle's episode (its own solves) and its sweep on the reference's plans reproduce the reference's
    windowed loop: tensor bounds on the axis (linear), a time-varying LinDx plant with w (linear_plant)."""
    t = fixture(case)
    T, n_steps = int(t["T"]), int(t["n_steps"])
    if "lo" in t:
        bounds = dict(u_lower=t["lo"], u_upper=t["hi"])
    else:
        bounds = dict(u_lower=-float(t["bound"]), u_upper=float(t["bound"]))
    plant = ("lin", t["F_p"], t["f_p"]) if "F_p" in t else None
    ep = wo.receding_horizon_tv(4, 2, T, n_steps, t["x_init"], t["C"], t["c"], t["F"], t["f"], plant=plant,
                                w=t.get("w"), lqr_iter=int(t["lqr_iter"]), eps=float(t["eps"]), coupled=True, **bounds)
    assert ep.iters == t["iters"].tolist()
    errs = {"x": rel(ep.x, t["x"]), "u": rel(ep.u, t["u"]), "plan_x": rel(ep.plan_x, t["plan_x"]),
            "plan_u": rel(ep.plan_u, t["plan_u"])}
    out = wo.receding_horizon_backward_tv(4, 2, T, t["C"], t["c"], t["F"], t["f"], t["x"], t["u"], t["plan_x"],
                                          t["plan_u"], t["wx"], t["wu"], plant=plant, **bounds)
    for k, o in (("x_init", "dx_init"), ("C", "dC"), ("c", "dc"), ("F", "dF"), ("f", "df"), ("F_p", "dF_p"),
                 ("f_p", "df_p"), ("w", "dw")):
        if "g_" + k in t:
            errs[k] = rel(out[o], t["g_" + k])
    print(case, {k: f"{v:.1e}" for k, v in errs.items()})
    assert max(errs.values()) <= 1e-10, errs


@pytest.mark.parametrize("case", ["pendulum", "cartpole", "pendulum_slew"])
def test_known_against_reference(case):
    """A known system tracking a moving reference: x from the reference's plans through the system's step, and the
    sweep (the reference's convention for the parameters: constant Jacobians, full_linearisation=False)."""
    t = fixture(case)
    T, clamp = int(t["T"]), float(t["clamp"])
    B, n = t["x"].shape[1], t["x"].shape[2]
    step = known_step(case, t)
    theta = t["params"].expand(B, -1)
    x = [t["x_init"]]
    for k in range(t["u"].shape[0]):
        x.append(step(x[-1], t["plan_u"][k][0], theta).detach())
    assert torch.equal(t["plan_u"][:, 0], t["u"])
    errs = {"x": rel(torch.stack(x), t["x"])}
    out = wo.receding_horizon_backward_tv(
        n, 1, T, t["C"], t["c"], None, None, t["x"], t["u"], t["plan_x"], t["plan_u"], t["wx"], t["wu"],
        u_lower=-clamp, u_upper=clamp, step=step, theta=theta, full_linearisation=False,
        slew_rate_penalty=float(t["slew"]) if "slew" in t else None)
    errs.update({"x_init": rel(out["dx_init"], t["g_x_init"]), "C": rel(out["dC"], t["g_C"]),
                 "c": rel(out["dc"], t["g_c"]), "params": rel(out["dtheta"].sum(0), t["g_params"])})
    print(case, {k: f"{v:.1e}" for k, v in errs.items()})
    assert max(errs.values()) <= 1e-10, errs


def _same(a, b):
    if isinstance(a, dict):
        return set(k for k in a if a[k] is not None) <= set(b) and all(
            a[k] is None or torch.equal(a[k], b[k]) for k in a)
    return all((u == v) if isinstance(u, list) else torch.equal(u, v) for u, v in zip(a, b))


def test_one_step_is_the_existing_oracles():
    """n_steps = 1: the window is the whole axis, and the window oracle is lqr_oracle's, slew_oracle's and
    plant_oracle's episode and sweep bitwise."""
    t = fixture("linear_plant")
    T, b = int(t["T"]), float(t["bound"])
    C, c, F, f = t["C"][:T], t["c"][:T], t["F"][:T - 1], t["f"][:T - 1]
    kw = dict(u_lower=-b, u_upper=b, lqr_iter=10, eps=1e-7, coupled=True)
    args = (4, 2, T, 1, t["x_init"], C, c, F, f)
    wx, wu = t["wx"][:2], t["wu"][:1]
    for slew in (None, 0.1):
        prev = torch.full((3, 2), 0.2, dtype=torch.float64) if slew else None
        skw = dict(slew_rate_penalty=slew, prev_ctrl=prev) if slew else {}
        ref = (sorc if slew else orc).receding_horizon_lin(*args, **skw, **kw)
        got = wo.receding_horizon_tv(*args, **skw, **kw)
        assert _same(ref, got), slew
        bargs = (4, 2, T, C, c, F, f, ref.x, ref.u, ref.plan_x, ref.plan_u, wx, wu)
        r1 = (sorc if slew else orc).receding_horizon_backward(*bargs, u_lower=-b, u_upper=b, **skw)
        r2 = wo.receding_horizon_backward_tv(*bargs, u_lower=-b, u_upper=b, **skw)
        assert _same(r1, r2), slew
        plant = ("lin", t["F_p"][:1], t["f_p"][:1])
        p1 = porc.receding_horizon_lin(*args, plant=plant, w=t["w"][:1], **skw, **kw)
        p2 = wo.receding_horizon_tv(*args, plant=plant, w=t["w"][:1], **skw, **kw)
        assert _same(p1, p2), slew
        pargs = (4, 2, T, C, c, F, f, p1.x, p1.u, p1.plan_x, p1.plan_u, wx, wu)
        q1 = porc.receding_horizon_backward(*pargs, u_lower=-b, u_upper=b, plant=plant, **skw)
        q2 = wo.receding_horizon_backward_tv(*pargs, u_lower=-b, u_upper=b, plant=plant, **skw)
        assert _same(q1, q2), slew
    z = fixture("pendulum")
    T = int(z["T"])
    B = z["x"].shape[1]
    step = known_step("pendulum", z)
    kargs = (3, 1, T, z["C"][:T], z["c"][:T], None, None, z["x"][:2], z["u"][:1], z["plan_x"][:1], z["plan_u"][:1],
             z["wx"][:2], z["wu"][:1])
    kkw = dict(u_lower=-2.0, u_upper=2.0, step=step, theta=z["params"].expand(B, -1), full_linearisation=False)
    assert _same(orc.receding_horizon_backward(*kargs, **kkw), wo.receding_horizon_backward_tv(*kargs, **kkw))
    assert _same(sorc.receding_horizon_backward(*kargs, slew_rate_penalty=0.1, **kkw),
                 wo.receding_horizon_backward_tv(*kargs, slew_rate_penalty=0.1, **kkw))


def test_constant_axis_is_the_time_invariant_oracle():
    """Inputs constant along L: the window oracle's episode is plant_oracle's time-invariant one bitwise, and its
    full-length gradients summed over L are the time-invariant gradients to rounding."""
    t = fixture("linear_plant")
    T, b, n_steps = int(t["T"]), float(t["bound"]), int(t["n_steps"])
    L = n_steps + T - 1
    C0, c0, F0, f0 = t["C"][:1], t["c"][:1], t["F"][:1], t["f"][:1]
    plant = ("lin", t["F_p"][:1], t["f_p"][:1])
    kw = dict(u_lower=-b, u_upper=b, lqr_iter=10, eps=1e-7, coupled=True)
    ti = porc.receding_horizon_lin(4, 2, T, n_steps, t["x_init"], C0.expand(T, -1, -1, -1), c0.expand(T, -1, -1),
                                   F0.expand(T - 1, -1, -1, -1), f0.expand(T - 1, -1, -1), plant=plant, w=t["w"], **kw)
    ex = (lambda v, n: v.expand(n, *v.shape[1:]))  # noqa: E731
    wplant = ("lin", ex(t["F_p"][:1], L - 1), ex(t["f_p"][:1], L - 1))
    tv = wo.receding_horizon_tv(4, 2, T, n_steps, t["x_init"], ex(C0, L), ex(c0, L), ex(F0, L - 1), ex(f0, L - 1),
                                plant=wplant, w=t["w"], **kw)
    assert _same(ti, tv)
    r1 = porc.receding_horizon_backward(4, 2, T, C0.expand(T, -1, -1, -1), c0.expand(T, -1, -1),
                                        F0.expand(T - 1, -1, -1, -1), f0.expand(T - 1, -1, -1), ti.x, ti.u,
                                        ti.plan_x, ti.plan_u, t["wx"], t["wu"], u_lower=-b, u_upper=b, plant=plant)
    r2 = wo.receding_horizon_backward_tv(4, 2, T, ex(C0, L), ex(c0, L), ex(F0, L - 1), ex(f0, L - 1), ti.x, ti.u,
                                         ti.plan_x, ti.plan_u, t["wx"], t["wu"], u_lower=-b, u_upper=b, plant=wplant)
    for k in ("dC", "dc", "dF", "df", "dF_p", "df_p"):
        assert rel(r2[k].sum(0), r1[k].sum(0)) <= 1e-12, k
    for k in ("dx_init", "dw"):
        assert rel(r2[k], r1[k]) <= 1e-12, k
