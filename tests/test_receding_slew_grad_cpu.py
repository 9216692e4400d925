"""CPU: the slew-rate episode backward's C ABI (mpcb200_episode_backward_slew_*) returns its status codes before
touching a device and sizes its workspace by the sweep's layout; the float64 oracle's slew sweep, fed the reference's
own plans, reproduces the reference's gradients (tests/golden/receding_grad_slew_f64.npz); and the slew oracle without
a penalty is lqr_oracle's own.  No kernel is launched here."""
import ctypes
import os

import numpy as np
import pytest
import torch

from mpc.pytorch_b200 import _lib
from mpc.pytorch_b200._lib import Dims, Params
from oracle import lqr_oracle as orc
from oracle import slew_oracle as sorc

OK, NULL, BAD = 0, 1, 2
FAKE = 1 << 20                      # a 256-byte aligned address the checks never dereference
GOLD = os.path.join(os.path.dirname(__file__), "golden")
NAMES = ("C", "c", "F", "u_lower", "u_upper", "xs", "us", "plan_x", "plan_u", "dl_dxs", "dl_dus", "dx_init", "dC",
         "dc", "dF", "df", "dtheta")


def dims(B=8, T=6, n=6, m=2, kind=0, has_f=1, F_T=None, bounds_kind=0):
    return Dims(B=B, T=T, n=n, m=m, F_T=T - 1 if F_T is None else F_T, has_f=has_f, bounds_kind=bounds_kind,
                max_ls_iter=10, pnqp_max_iter=20, do_rollout=1, dynamics_kind=kind)


def ws_bytes(d, n_prev, esz=4):
    return _lib.lib().mpcb200_episode_backward_slew_workspace_bytes(ctypes.byref(d), n_prev, esz)


def backward(d, n_prev, n_steps=3, nbytes=None, workspace=FAKE, f64=False, **null):
    ptrs = [None if null.get(k) else FAKE for k in NAMES]
    nbytes = (ws_bytes(d, n_prev) or 1 << 30) if nbytes is None else nbytes
    fn = _lib.lib().mpcb200_episode_backward_slew_f64 if f64 else _lib.lib().mpcb200_episode_backward_slew_f32
    return fn(ctypes.byref(d), ctypes.byref(Params()), n_steps, n_prev, *ptrs, workspace, nbytes, None)


def test_slew_backward_null_pointers():
    L = _lib.lib()
    assert L.mpcb200_episode_backward_slew_f32(None, ctypes.byref(Params()), 3, 2, *([FAKE] * 17), FAKE, 1 << 30,
                                               None) == NULL
    for k in ("C", "c", "xs", "us", "plan_x", "plan_u", "dl_dxs", "dl_dus", "dx_init", "dC", "dc"):
        assert backward(dims(), 2, **{k: True}) == NULL, k
        assert backward(dims(), 2, f64=True, **{k: True}) == NULL, k
    assert backward(dims(), 2, workspace=None) == NULL
    assert backward(dims(), 2, F=True) == NULL and backward(dims(), 2, dF=True) == NULL
    assert backward(dims(), 2, df=True) == NULL
    assert backward(dims(kind=18, n=4, m=1), 1, dtheta=True) == NULL
    assert backward(dims(bounds_kind=2), 2, u_lower=True) == NULL


def test_slew_backward_bad_dims():
    assert backward(dims(T=2), 2) == BAD and backward(dims(T=3), 2, n_steps=0) == BAD
    assert backward(dims(B=0), 2) == BAD
    for n_prev in (0, -1, 3):                                      # 1 <= n_prev <= m
        assert ws_bytes(dims(), n_prev) == 0 and backward(dims(), n_prev) == BAD, n_prev
    d = dims(n=2, m=2)                                              # n_prev < n
    assert ws_bytes(d, 2) == 0 and backward(d, 2) == BAD
    assert ws_bytes(dims(n=3, m=2), 2) > 0
    for kind, n in ((1, 5), (2, 3), (4, 3)):                         # the systems themselves: the plain entry's
        d = dims(kind=kind, n=n, m=1)
        assert ws_bytes(d, 1) == 0 and backward(d, 1) == BAD, kind
    for kind, n in ((17, 6), (18, 4), (20, 4)):
        assert ws_bytes(dims(kind=kind, n=n, m=1), 1) > 0, kind
        assert backward(dims(kind=kind, n=n + 1, m=1), 1) == BAD, kind        # not the dynamics-only shape
        assert backward(dims(kind=kind, n=n, m=2), 1) == BAD, kind
        assert backward(dims(kind=kind, n=n, m=2), 2) == BAD, kind
    assert backward(dims(kind=16, n=4, m=1), 1) == BAD                # a passthrough flag without a system


def test_slew_backward_workspace_checks():
    d = dims()
    need = ws_bytes(d, 2)
    assert need > 0 and need % 256 == 0
    assert backward(d, 2, nbytes=need - 1) == BAD
    assert backward(d, 2, nbytes=need, workspace=FAKE + 16) == BAD


def up256(v):
    return (v + 255) // 256 * 256


@pytest.mark.parametrize("kind,n,NP", [(0, 6, 0), (0, 17, 0), (17, 6, 4), (18, 4, 3), (20, 4, 5)])
@pytest.mark.parametrize("esz", [4, 8])
@pytest.mark.parametrize("B,T,has_f,F_T", [(8, 6, 1, 5), (33, 3, 0, 3)])
def test_slew_backward_workspace_formula(kind, n, NP, esz, B, T, has_f, F_T):
    m = 1 if kind else 2 if n == 6 else 3
    d = dims(B=B, T=T, n=n, m=m, kind=kind, has_f=has_f, F_T=F_T)
    p = n + m
    da = dims(B=B, T=T, n=n, m=m, has_f=has_f, F_T=F_T)
    if kind:
        da.F_T, da.has_f = T - 1, 1
    adj = _lib.lib().mpcb200_adjoint_workspace_bytes(ctypes.byref(da), esz)
    TB, T1B = T * B, (T - 1) * B
    pieces = [TB * n, TB * m, TB * n, TB * m, B * n, B * NP, B * n, TB * p * p, TB * p, da.F_T * B * n * p,
              T1B * n if da.has_f else 0]
    pieces = [adj] + [v * esz for v in pieces]
    if kind:
        pieces += [T1B * n * p * esz, T1B * n * esz, T1B * NP * esz, T1B * NP * esz]
    pieces.append(16)
    want = sum(up256(v) for v in pieces)
    assert ws_bytes(d, m, esz) == want
    if not kind:                                      # the same layout as the plain entry's for LinDx
        assert _lib.lib().mpcb200_episode_backward_workspace_bytes(ctypes.byref(d), esz) == want


# ---------------------------------------------------------------------------------------------- the oracle
def _gold():
    return dict(np.load(os.path.join(GOLD, "receding_grad_slew_f64.npz")))


def _t(z, k):
    return torch.from_numpy(z[k])


def _lin_inputs(z, case):
    """The case's problem as LinDx(F0.expand, f0.expand) over T-1 slices (the fixture's affine Module)."""
    g = lambda k: _t(z, case + "_" + k)                      # noqa: E731
    T, n_steps = int(z[case + "_T"]), int(z[case + "_n_steps"])
    F = g("F").unsqueeze(0).expand(T - 1, *g("F").shape)
    f = g("f").unsqueeze(0).expand(T - 1, *g("f").shape)
    kw = {}
    if case + "_bound" in z:
        b = float(z[case + "_bound"])
        kw = dict(u_lower=torch.full((T, g("x_init").shape[0], 2), -b, dtype=torch.float64),
                  u_upper=torch.full((T, g("x_init").shape[0], 2), b, dtype=torch.float64))
    prev = g("prev_ctrl") if case + "_prev_ctrl" in z else None
    return g, T, n_steps, F, f, kw, prev


def _rel(a, b):
    return float((a - b).abs().max()) / max(1.0, float(b.abs().max()))


@pytest.mark.parametrize("case", ["unbounded", "bounded"])
def test_oracle_slew_sweep_linear_against_reference(case):
    z = _gold()
    g, T, n_steps, F, f, kw, prev = _lin_inputs(z, case)
    n, m = 4, 2
    out = sorc.receding_horizon_backward(n, m, T, g("C"), g("c"), F, f, g("x"), g("u"), g("plan_x"), g("plan_u"),
                                        g("wx"), g("wu"), slew_rate_penalty=float(z[case + "_slew"]), prev_ctrl=prev,
                                        **kw)
    errs = {"x_init": _rel(out["dx_init"], g("g_x_init")), "C": _rel(out["dC"], g("g_C")),
            "c": _rel(out["dc"], g("g_c")), "F": _rel(out["dF"].sum(0), g("g_F")),
            "f": _rel(out["df"].sum(0), g("g_f"))}
    print(case, {k: f"{v:.1e}" for k, v in errs.items()})
    assert max(errs.values()) < 1e-10, errs


@pytest.mark.parametrize("case", ["unbounded", "bounded"])
def test_oracle_slew_episode_against_reference(case):
    """The oracle's slew episode reproduces the reference's x, u, plans and iteration counts."""
    z = _gold()
    g, T, n_steps, F, f, kw, prev = _lin_inputs(z, case)
    ep = sorc.receding_horizon_lin(4, 2, T, n_steps, g("x_init"), g("C"), g("c"), F, f, lqr_iter=10, eps=1e-7,
                                  slew_rate_penalty=float(z[case + "_slew"]), prev_ctrl=prev, coupled=True, **kw)
    assert ep.iters == z[case + "_iters"].tolist()
    assert _rel(ep.x, g("x")) < 1e-10 and _rel(ep.u, g("u")) < 1e-10
    assert _rel(ep.plan_x[..., 2:], g("plan_x")) < 1e-10 and _rel(ep.plan_u, g("plan_u")) < 1e-10


@pytest.mark.parametrize("name", ["pendulum", "cartpole"])
def test_oracle_slew_sweep_known_against_reference(name):
    """Known systems: dx_init, dC, dc and, with the reference's constant Jacobians (full_linearisation=False), dtheta."""
    from tests.gpu_harness import episode_known_module, episode_known_step
    z = _gold()
    g = lambda k: _t(z, name + "_" + k)                      # noqa: E731
    T, clamp = int(z[name + "_T"]), float(z[name + "_clamp"])
    mod, _ = episode_known_module(name)
    assert torch.equal(mod.params, g("params"))
    B, n = g("x").shape[1], g("x").shape[2]
    out = sorc.receding_horizon_backward(n, 1, T, g("C"), g("c"), None, None, g("x"), g("u"), g("plan_x"),
                                        g("plan_u"), g("wx"), g("wu"), u_lower=-clamp, u_upper=clamp,
                                        step=episode_known_step(mod), theta=g("params").expand(B, -1),
                                        full_linearisation=False, slew_rate_penalty=float(z[name + "_slew"]))
    errs = {"x_init": _rel(out["dx_init"], g("g_x_init")), "C": _rel(out["dC"], g("g_C")),
            "c": _rel(out["dc"], g("g_c")), "params": _rel(out["dtheta"].sum(0), g("g_params"))}
    print(name, {k: f"{v:.1e}" for k, v in errs.items()})
    assert max(errs.values()) < 1e-10, errs
    assert float(g("g_C").abs().max()) > 0


def test_oracle_without_penalty_unchanged():
    """The slew oracle without a penalty (prev_ctrl then unused) is lqr_oracle's episode and sweep, bitwise."""
    z = dict(np.load(os.path.join(GOLD, "receding_grad_linear_f64.npz")))
    g = lambda k: torch.from_numpy(z["bounded_" + k])       # noqa: E731
    T, n_steps, b = int(z["bounded_T"]), 3, float(z["bounded_bound"])
    kw = dict(u_lower=-b, u_upper=b, lqr_iter=10, eps=1e-7, coupled=True)
    a = orc.receding_horizon_lin(4, 2, T, n_steps, g("x_init"), g("C"), g("c"), g("F"), g("f"), **kw)
    b_ = sorc.receding_horizon_lin(4, 2, T, n_steps, g("x_init"), g("C"), g("c"), g("F"), g("f"),
                                  slew_rate_penalty=None, prev_ctrl=torch.ones(4, 2, dtype=torch.float64), **kw)
    for u, v in zip(a, b_):
        assert (u == v) if isinstance(u, list) else torch.equal(u, v)
    lo = torch.full((T, 4, 2), -b, dtype=torch.float64)
    args = (4, 2, T, g("C"), g("c"), g("F"), g("f"), a.x, a.u, a.plan_x, a.plan_u, g("wx")[:n_steps + 1],
            g("wu")[:n_steps])
    r1 = orc.receding_horizon_backward(*args, u_lower=lo, u_upper=-lo)
    r2 = sorc.receding_horizon_backward(*args, u_lower=lo, u_upper=-lo, slew_rate_penalty=None,
                                        prev_ctrl=torch.ones(4, 2, dtype=torch.float64))
    assert r1.keys() == r2.keys() and all(torch.equal(r1[k], r2[k]) for k in r1)
