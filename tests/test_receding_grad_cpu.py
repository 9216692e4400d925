"""CPU: the C ABI of differentiable episodes - mpcb200_episode_plans_* and mpcb200_episode_backward_* return their
status codes for NULL pointers, bad dims and small or misaligned workspaces before touching a device, and
mpcb200_episode_backward_workspace_bytes follows its layout.  No kernel is launched here."""
import ctypes

import pytest

from mpc.pytorch_b200 import _lib
from mpc.pytorch_b200._lib import Dims, IlqrOpts, Params

OK, NULL, BAD = 0, 1, 2
FAKE = 1 << 20                      # a 256-byte aligned address the checks never dereference
KNOWN = {1: (5, 1, 4), 2: (3, 1, 3), 4: (3, 1, 5)}      # kind: (n, m, learnable parameters)


def dims(B=8, T=6, n=4, m=2, kind=0, has_f=1, F_T=None, bounds_kind=0):
    if kind:
        n, m = KNOWN.get(kind, (n, m))[:2]
    return Dims(B=B, T=T, n=n, m=m, F_T=T - 1 if F_T is None else F_T, has_f=has_f, bounds_kind=bounds_kind,
                max_ls_iter=10, pnqp_max_iter=20, do_rollout=1, dynamics_kind=kind)


def ws_bytes(d, esz=4):
    return _lib.lib().mpcb200_episode_backward_workspace_bytes(ctypes.byref(d), esz)


def backward(d, n_steps=3, nbytes=None, workspace=FAKE, **null):
    """mpcb200_episode_backward_f32 with every pointer FAKE except the names in `null`."""
    names = ("C", "c", "F", "u_lower", "u_upper", "xs", "us", "plan_x", "plan_u", "dl_dxs", "dl_dus", "dx_init", "dC",
             "dc", "dF", "df", "dtheta")
    ptrs = [None if null.get(k) else FAKE for k in names]
    nbytes = ws_bytes(d) if nbytes is None else nbytes
    return _lib.lib().mpcb200_episode_backward_f32(ctypes.byref(d), ctypes.byref(Params()), n_steps, *ptrs,
                                                   workspace, nbytes, None)


def test_backward_null_pointers():
    L = _lib.lib()
    assert L.mpcb200_episode_backward_f32(None, ctypes.byref(Params()), 3, *([FAKE] * 17), FAKE, 1 << 30, None) == NULL
    for k in ("C", "c", "xs", "us", "plan_x", "plan_u", "dl_dxs", "dl_dus", "dx_init", "dC", "dc"):
        assert backward(dims(), **{k: True}) == NULL, k
    assert backward(dims(), workspace=None) == NULL
    assert backward(dims(), F=True) == NULL and backward(dims(), dF=True) == NULL     # LinDx needs F and dF
    assert backward(dims(), df=True) == NULL                                         # ... and df with f
    assert backward(dims(kind=2), dtheta=True) == NULL                               # a known system: dtheta
    assert backward(dims(bounds_kind=2), u_lower=True) == NULL                       # tensor bounds


def test_backward_bad_dims():
    assert backward(dims(T=2)) == BAD and backward(dims(T=3), n_steps=0) == BAD
    assert backward(dims(B=0), nbytes=1 << 30) == BAD
    assert backward(dims(F_T=3)) == BAD                                              # F_T must be T-1 or T
    assert backward(dims(bounds_kind=3), nbytes=1 << 30) == BAD
    d = dims(kind=2)
    d.n = 4
    assert backward(d, nbytes=1 << 30) == BAD                                        # not the system's shape
    d = dims(kind=18, n=4, m=1)                                                      # a slew-rate passthrough kind
    assert ws_bytes(d) == 0 and backward(d, nbytes=1 << 30) == BAD


def test_backward_workspace_checks():
    d = dims()
    need = ws_bytes(d)
    assert need > 0 and need % 256 == 0
    assert backward(d, nbytes=need - 1) == BAD
    assert backward(d, nbytes=need, workspace=FAKE + 16) == BAD                      # 256-byte alignment


def up256(v):
    return (v + 255) // 256 * 256


@pytest.mark.parametrize("kind", [0, 1, 2, 4])
@pytest.mark.parametrize("esz", [4, 8])
@pytest.mark.parametrize("B,T,has_f,F_T", [(8, 6, 1, 5), (33, 3, 0, 3), (1, 10, 1, 10)])
def test_backward_workspace_formula(kind, esz, B, T, has_f, F_T):
    d = dims(B=B, T=T, kind=kind, has_f=has_f, F_T=F_T)
    n, m, p = d.n, d.m, d.n + d.m
    da = dims(B=B, T=T, kind=kind, has_f=has_f, F_T=F_T)
    if kind:                                     # each step's adjoint takes the dense linearisation [T-1, ...]
        da.F_T, da.has_f = T - 1, 1
    da.dynamics_kind = 0
    adj = _lib.lib().mpcb200_adjoint_workspace_bytes(ctypes.byref(da), esz)
    NP = KNOWN[kind][2] if kind else 0
    TB, T1B = T * B, (T - 1) * B
    pieces = [adj, TB * n, TB * m, TB * n, TB * m, B * n, B * NP, B * n, TB * p * p, TB * p, da.F_T * B * n * p,
              T1B * n if da.has_f else 0]
    pieces = [pieces[0]] + [v * esz for v in pieces[1:]]
    if kind:
        pieces += [T1B * n * p * esz, T1B * n * esz, T1B * NP * esz, T1B * NP * esz]
    pieces.append(16)                            # the sweep's state
    assert ws_bytes(d, esz) == sum(up256(v) for v in pieces)


def test_plans_null_pointers():
    L = _lib.lib()
    d = dims()
    opts = IlqrOpts(lqr_iter=5, not_improved_lim=5, m_ref=2, eps=1e-7, best_cost_eps=1e-4)
    nbytes = L.mpcb200_episode_workspace_bytes(ctypes.byref(d), ctypes.byref(opts), 4)
    args = [FAKE] * 14
    for which in (0, 1):
        plans = [FAKE, FAKE]
        plans[which] = None
        assert L.mpcb200_episode_plans_f32(ctypes.byref(d), ctypes.byref(Params()), ctypes.byref(opts), 3, *args,
                                           *plans, FAKE, nbytes, None) == NULL
    d.T = 2
    assert L.mpcb200_episode_plans_f32(ctypes.byref(d), ctypes.byref(Params()), ctypes.byref(opts), 3, *args,
                                       FAKE, FAKE, FAKE, 1 << 30, None) == BAD
