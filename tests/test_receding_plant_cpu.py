"""CPU: episodes closed on a plant other than the model.  The C ABI of mpcb200_episode_plant_* and
mpcb200_episode_backward_plant_* returns its status codes before touching a device, and the backward's workspace is
the sweep's layout with the stage's parameter buffer sized by the plant; receding_horizon rejects a plant or a
disturbance of the wrong shape before anything runs; the float64 plant oracle, fed the reference's own plans,
reproduces the reference's episode and gradients (tests/golden/receding_plant_f64.npz), and without a plant it is
lqr_oracle's / slew_oracle's bitwise.  No kernel is launched here."""
import ctypes
import os

import numpy as np
import pytest
import torch

from mpc.pytorch_b200 import _lib
from mpc.pytorch_b200._lib import Dims, IlqrOpts, MpcB200Error, Params, Plant
from mpc.pytorch_b200.control import receding_horizon
from mpc.pytorch_b200.dynamics import CartpoleDx, PendulumDx
from mpc.pytorch_b200.solver import MPC, LinDx, QuadCost
from oracle import lqr_oracle as orc
from oracle import plant_oracle as porc
from oracle import slew_oracle as sorc
from tests.gpu_harness import episode_known_step

NULL, BAD, NO_DEVICE = 1, 2, 6      # a well-formed call gets as far as looking for a device
FAKE = 1 << 20                      # a 256-byte aligned address the checks never dereference
BW_NAMES = ("C", "c", "F", "F_plant", "u_lower", "u_upper", "xs", "us", "plan_x", "plan_u", "dl_dxs", "dl_dus",
            "dx_init", "dC", "dc", "dF", "df", "dtheta", "dF_plant", "df_plant", "dtheta_plant", "dw")
FW_NAMES = ("C", "c", "F", "f", "F_plant", "f_plant", "w", "x_init", "u_init", "u_lower", "u_upper", "u_zero_I",
            "xs", "us", "costs", "info", "u_next", "plan_x", "plan_u")


def dims(B=8, T=6, n=6, m=2, kind=0, has_f=1, bounds_kind=0):
    return Dims(B=B, T=T, n=n, m=m, F_T=T - 1, has_f=has_f, bounds_kind=bounds_kind, max_ls_iter=10,
                pnqp_max_iter=20, do_rollout=1, dynamics_kind=kind)


def plant(kind=0, has_f=1):
    return Plant(kind=kind, has_f=has_f)


def ws_bytes(d, n_prev, pl, esz=4):
    return _lib.lib().mpcb200_episode_backward_plant_workspace_bytes(ctypes.byref(d), n_prev, ctypes.byref(pl), esz)


def backward(d, pl, n_prev=0, n_steps=3, nbytes=None, workspace=FAKE, f64=False, **null):
    ptrs = [None if null.get(k) else FAKE for k in BW_NAMES]
    nbytes = ((ws_bytes(d, n_prev, pl) if pl is not None else 0) or 1 << 30) if nbytes is None else nbytes
    L = _lib.lib()
    fn = L.mpcb200_episode_backward_plant_f64 if f64 else L.mpcb200_episode_backward_plant_f32
    return fn(ctypes.byref(d), ctypes.byref(Params()), ctypes.byref(pl) if pl is not None else None, n_steps, n_prev,
              *ptrs, workspace, nbytes, None)


def forward(d, pl, n_steps=3, nbytes=1 << 30, workspace=FAKE, f64=False, **null):
    ptrs = [None if null.get(k) else FAKE for k in FW_NAMES]
    opts = IlqrOpts(lqr_iter=5, not_improved_lim=5, m_ref=d.m, eps=1e-7, best_cost_eps=1e-4)
    L = _lib.lib()
    fn = L.mpcb200_episode_plant_f64 if f64 else L.mpcb200_episode_plant_f32
    return fn(ctypes.byref(d), ctypes.byref(Params()), ctypes.byref(opts),
              ctypes.byref(pl) if pl is not None else None, n_steps, *ptrs, workspace, nbytes, None)


def test_plant_forward_status_codes():
    assert forward(dims(), None) == NULL
    for k in ("x_init", "xs", "us", "costs", "info", "u_next"):
        assert forward(dims(), plant(), **{k: True}) == NULL, k
    assert forward(dims(), plant(), F_plant=True) == NULL
    assert forward(dims(), plant(has_f=1), f_plant=True) == NULL
    assert forward(dims(), plant(), plan_x=True) == NULL                   # both plans or neither
    assert forward(dims(T=2), plant()) == BAD and forward(dims(), plant(), n_steps=0) == BAD
    assert forward(dims(), plant(kind=2)) == BAD                             # pendulum steps (3, 1), not (6, 2)
    assert forward(dims(n=3, m=1), plant(kind=1)) == BAD                     # cartpole steps (5, 1)
    assert forward(dims(n=3, m=1), plant(kind=18)) == BAD                    # a passthrough pendulum steps (4, 1)
    assert forward(dims(n=3, m=1), plant(kind=3)) == BAD                     # no such system
    assert forward(dims(), plant(), nbytes=16) == BAD                        # the episode's workspace
    assert forward(dims(), plant(), workspace=FAKE + 16) == BAD
    assert forward(dims(), plant(), plan_x=True, plan_u=True, w=True) == NO_DEVICE
    assert forward(dims(n=3, m=1, kind=2), plant(kind=4), F=True, f=True, F_plant=True, f_plant=True) == NO_DEVICE


def test_plant_backward_null_pointers():
    assert backward(dims(), None) == NULL
    for k in ("C", "c", "xs", "us", "plan_x", "plan_u", "dl_dxs", "dl_dus", "dx_init", "dC", "dc", "F_plant",
              "dF_plant"):
        assert backward(dims(), plant(), **{k: True}) == NULL, k
        assert backward(dims(), plant(), f64=True, **{k: True}) == NULL, k
    assert backward(dims(), plant(has_f=1), df_plant=True) == NULL
    assert backward(dims(), plant(has_f=0), df_plant=True) == NO_DEVICE
    assert backward(dims(), plant(), dw=True) == NO_DEVICE                   # dw is optional
    assert backward(dims(n=3, m=1), plant(kind=2), dtheta_plant=True) == NULL
    assert backward(dims(n=3, m=1, kind=2), plant(kind=4), dtheta=True) == NULL


def test_plant_backward_bad_dims():
    assert backward(dims(T=2), plant()) == BAD and backward(dims(), plant(), n_steps=0) == BAD
    assert backward(dims(), plant(), n_prev=-1) == BAD
    for kind, n in ((1, 5), (2, 3), (4, 3)):
        assert backward(dims(n=n, m=1), plant(kind=kind)) == NO_DEVICE, kind
        assert ws_bytes(dims(n=n, m=1), 0, plant(kind=kind)) > 0, kind
        assert backward(dims(n=n + 1, m=1), plant(kind=kind)) == BAD, kind   # not the plant's own shape
        assert ws_bytes(dims(n=n + 1, m=1), 0, plant(kind=kind)) == 0, kind
        assert backward(dims(n=n + 1, m=1), plant(kind=kind | 16), n_prev=1) == NO_DEVICE, kind   # slew
        assert backward(dims(n=n + 1, m=1), plant(kind=kind), n_prev=1) == BAD, kind        # system under slew
        assert backward(dims(n=n, m=1), plant(kind=kind | 16)) == BAD, kind                 # passthrough w/o slew
    assert backward(dims(n=4, m=2), plant(kind=18), n_prev=2) == BAD        # n_prev is the system's n_ctrl


def test_plant_backward_workspace_formula():
    """plant = LinDx or a system with the model's parameter count: the model's own sweep layout; a known plant with
    another parameter count changes only the stage's [B, NP] buffer."""
    L = _lib.lib()
    for esz in (4, 8):
        for d in (dims(), dims(n=3, m=1, kind=2), dims(n=5, m=1, kind=1)):
            base = L.mpcb200_episode_backward_workspace_bytes(ctypes.byref(d), esz)
            pk = d.dynamics_kind if d.dynamics_kind else 0
            assert ws_bytes(d, 0, plant(kind=pk), esz) == base
        d = dims(n=3, m=1, kind=2)                                           # pendulum model (NP 3)
        base = L.mpcb200_episode_backward_workspace_bytes(ctypes.byref(d), esz)
        up = lambda b: (b + 255) // 256 * 256                                 # noqa: E731
        assert ws_bytes(d, 0, plant(kind=4), esz) == base - up(8 * 3 * esz) + up(8 * 5 * esz)
        assert ws_bytes(d, 0, plant(kind=0), esz) == base - up(8 * 3 * esz)
        ds = dims(n=4, m=1, kind=18)
        slew = L.mpcb200_episode_backward_slew_workspace_bytes(ctypes.byref(ds), 1, esz)
        assert ws_bytes(ds, 1, plant(kind=18), esz) == slew
    d = dims()
    need = ws_bytes(d, 0, plant())
    assert need > 0 and need % 256 == 0
    assert backward(d, plant(), nbytes=need - 1) == BAD
    assert backward(d, plant(), nbytes=need, workspace=FAKE + 16) == BAD


# ------------------------------------------------------------------------------------------------------------------
def _episode_args(n=3, m=1, B=2, T=5):
    ctrl = MPC(n, m, T, lqr_iter=3, verbose=-1)
    C = torch.eye(n + m, dtype=torch.float64).expand(T, B, n + m, n + m)
    c = torch.zeros(T, B, n + m, dtype=torch.float64)
    F = torch.randn(T - 1, B, n, n + m, dtype=torch.float64)
    return ctrl, torch.zeros(B, n, dtype=torch.float64), QuadCost(C, c), LinDx(F)


@pytest.mark.parametrize("bad", ["lin_rows", "lin_cols", "lin_f", "known", "module", "w_shape", "w_dtype"])
def test_plant_shape_errors_before_anything_runs(bad):
    """The checks run on metadata alone, so CPU tensors reach them: no device is needed to see the error."""
    ctrl, x0, cost, dx = _episode_args()
    B, n, m = 2, 3, 1
    plant, w = None, None
    if bad == "lin_rows":
        plant = LinDx(torch.zeros(1, B, n + 1, n + m + 1, dtype=torch.float64))
    elif bad == "lin_cols":
        plant = LinDx(torch.zeros(1, B, n, n, dtype=torch.float64))
    elif bad == "lin_f":
        plant = LinDx(torch.zeros(1, B, n, n + m, dtype=torch.float64), torch.zeros(1, B, n + 1, dtype=torch.float64))
    elif bad == "known":
        plant = CartpoleDx()
    elif bad == "module":
        class Wide(torch.nn.Module):
            n_state, n_ctrl = 3, 2
        plant = Wide()
    elif bad == "w_shape":
        w = torch.zeros(4, B, n, dtype=torch.float64)
    else:
        w = torch.zeros(3, B, n, dtype=torch.float32)
    with pytest.raises(MpcB200Error):
        receding_horizon(ctrl, x0, cost, dx, 3, plant=plant, disturbance=w)


def test_pendulum_plant_shape_accepted_by_check():
    from mpc.pytorch_b200.control import _check_plant
    _check_plant(PendulumDx(simple=False), torch.zeros(3, 2, 3), torch.zeros(2, 3), 3, 1, 3)


# ------------------------------------------------------------------------------------------------------------------
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SYSTEMS = {"pendulum": (lambda: PendulumDx(simple=True), lambda: PendulumDx(simple=False), "max_torque"),
           "cartpole": (CartpoleDx, CartpoleDx, "force_mag")}


def fixture(case):
    z = np.load(os.path.join(GOLD, "receding_plant_f64.npz"))
    pre = case + "_"
    return {k[len(pre):]: torch.from_numpy(z[k]) for k in z.files
            if k.startswith(pre) and not (case == "pendulum" and k.startswith("pendulum_slew_"))}


def rel(a, b):
    return float((a - b).abs().max()) / max(1.0, float(b.abs().max()))


def known_steps(case, t):
    """The oracle's model and plant step functions for a known-system case: the project's CPU modules, clamped as the
    fixture's systems were."""
    sysname = case.split("_")[0]
    model_cls, plant_cls, attr = SYSTEMS[sysname]
    model, plant = model_cls(), plant_cls()
    for mod in (model, plant):
        setattr(mod, attr, float(t["clamp"]))
    return episode_known_step(model), episode_known_step(plant)


def test_linear_sweep_and_episode_against_reference():
    t = fixture("linear")
    T, n_steps, b = int(t["T"]), int(t["n_steps"]), float(t["bound"])
    n, m = 4, 2
    plant = ("lin", t["F_p"].unsqueeze(0), t["f_p"].unsqueeze(0))
    ep = porc.receding_horizon_lin(n, m, T, n_steps, t["x_init"], t["C"], t["c"], t["F"], t["f"], plant=plant,
                                   w=t["w"], u_lower=-b, u_upper=b, lqr_iter=int(t["lqr_iter"]), eps=float(t["eps"]),
                                   coupled=True)
    assert ep.iters == t["iters"].tolist()
    assert rel(ep.x, t["x"]) <= 1e-10 and rel(ep.u, t["u"]) <= 1e-10
    assert rel(ep.plan_x, t["plan_x"]) <= 1e-10 and rel(ep.plan_u, t["plan_u"]) <= 1e-10
    out = porc.receding_horizon_backward(n, m, T, t["C"], t["c"], t["F"], t["f"], t["x"], t["u"], t["plan_x"],
                                         t["plan_u"], t["wx"], t["wu"], u_lower=-b, u_upper=b, plant=plant)
    errs = {"x_init": rel(out["dx_init"], t["g_x_init"]), "C": rel(out["dC"], t["g_C"]),
            "c": rel(out["dc"], t["g_c"]), "F": rel(out["dF"], t["g_F"]), "f": rel(out["df"], t["g_f"]),
            "F_p": rel(out["dF_p"][0], t["g_F_p"]), "f_p": rel(out["df_p"][0], t["g_f_p"]),
            "w": rel(out["dw"], t["g_w"])}
    print("linear", {k: f"{v:.1e}" for k, v in errs.items()})
    assert max(errs.values()) <= 1e-10, errs


@pytest.mark.parametrize("case", ["pendulum", "cartpole", "pendulum_slew"])
def test_known_sweep_against_reference(case):
    """A known model on a known plant of other parameters (the clamp binding), with w: the reference's convention for
    the model's parameters (constant Jacobians, full_linearisation=False)."""
    t = fixture(case)
    T, clamp = int(t["T"]), float(t["clamp"])
    B, n = t["x"].shape[1], t["x"].shape[2]
    step, pstep = known_steps(case, t)
    out = porc.receding_horizon_backward(
        n, 1, T, t["C"], t["c"], None, None, t["x"], t["u"], t["plan_x"], t["plan_u"], t["wx"], t["wu"],
        u_lower=-clamp, u_upper=clamp, step=step, theta=t["params"].expand(B, -1), full_linearisation=False,
        slew_rate_penalty=float(t["slew"]) if "slew" in t else None,
        plant=("step", pstep, t["plant_params"].expand(B, -1)))
    errs = {"x_init": rel(out["dx_init"], t["g_x_init"]), "C": rel(out["dC"], t["g_C"]),
            "c": rel(out["dc"], t["g_c"]), "params": rel(out["dtheta"].sum(0), t["g_params"]),
            "plant_params": rel(out["dtheta_plant"].sum(0), t["g_plant_params"]), "w": rel(out["dw"], t["g_w"])}
    print(case, {k: f"{v:.1e}" for k, v in errs.items()})
    assert max(errs.values()) <= 1e-10, errs
    assert bool((t["plan_u"].abs() == clamp).any()) and float(t["g_plant_params"].abs().max()) > 0


def test_oracle_is_lqr_and_slew_oracle_without_a_plant():
    """Plant None (the model steps) and no w: lqr_oracle's episode and sweep, and slew_oracle's under a penalty,
    bitwise."""
    t = fixture("linear")
    T, b = int(t["T"]), float(t["bound"])
    kw = dict(u_lower=-b, u_upper=b, lqr_iter=10, eps=1e-7, coupled=True)
    args = (4, 2, T, 3, t["x_init"], t["C"], t["c"], t["F"], t["f"])
    for slew in (None, 0.1):
        prev = torch.full((4, 2), 0.2, dtype=torch.float64) if slew else None
        if slew:
            a = sorc.receding_horizon_lin(*args, slew_rate_penalty=slew, prev_ctrl=prev, **kw)
        else:
            a = orc.receding_horizon_lin(*args, **kw)
        p = porc.receding_horizon_lin(*args, slew_rate_penalty=slew, prev_ctrl=prev, **kw)
        for u, v in zip(a, p):
            assert (u == v) if isinstance(u, list) else torch.equal(u, v)
        bargs = (4, 2, T, t["C"], t["c"], t["F"], t["f"], a.x, a.u, a.plan_x, a.plan_u, t["wx"][:4], t["wu"][:3])
        if slew:
            r1 = sorc.receding_horizon_backward(*bargs, u_lower=-b, u_upper=b, slew_rate_penalty=slew, prev_ctrl=prev)
        else:
            r1 = orc.receding_horizon_backward(*bargs, u_lower=-b, u_upper=b)
        r2 = porc.receding_horizon_backward(*bargs, u_lower=-b, u_upper=b, slew_rate_penalty=slew, prev_ctrl=prev)
        assert all(torch.equal(r1[k], r2[k]) for k in r1), slew
    # a known model: the model's own step, theta's split as before
    z = fixture("pendulum")
    B = z["x"].shape[1]
    step, _ = known_steps("pendulum", z)
    kargs = (3, 1, int(z["T"]), z["C"], z["c"], None, None, z["x"], z["u"], z["plan_x"], z["plan_u"], z["wx"],
             z["wu"])
    kkw = dict(u_lower=-2.0, u_upper=2.0, step=step, theta=z["params"].expand(B, -1), full_linearisation=False)
    r1 = orc.receding_horizon_backward(*kargs, **kkw)
    r2 = porc.receding_horizon_backward(*kargs, **kkw)
    assert all(torch.equal(r1[k], r2[k]) for k in r1)
    r1 = sorc.receding_horizon_backward(*kargs, slew_rate_penalty=0.1, **kkw)
    r2 = porc.receding_horizon_backward(*kargs, slew_rate_penalty=0.1, **kkw)
    assert all(torch.equal(r1[k], r2[k]) for k in r1)
