"""CPU: the episode entry points (mpcb200_episode_*) refuse malformed arguments with status codes before they touch a
device and size their workspace without one; receding_horizon picks its device or host path on tensor metadata alone
(FakeTensor CUDA tensors here: no device, no kernel) and refuses horizons and step counts its warm-start rule cannot
take; the host path's warm-start rule is the notebooks' expression."""
import ctypes

import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode

from mpc.pytorch_b200 import _lib, control, solver
from mpc.pytorch_b200._lib import Dims, IlqrOpts, MpcB200Error, Params
from mpc.pytorch_b200.control import receding_horizon, shift_warm_start
from mpc.pytorch_b200.dynamics import DYN_CARTPOLE, CartpoleDx, PendulumDx
from mpc.pytorch_b200.solver import MPC, GradMethods, LinDx, QuadCost


def _dims(B=4, T=5, n=8, m=2, **kw):
    return Dims(B=B, T=T, n=n, m=m, F_T=T - 1, has_f=0, bounds_kind=0, has_zero_mask=0, has_delta_u=0,
                max_ls_iter=10, pnqp_max_iter=20, do_rollout=1, **kw)


def _opts(**kw):
    o = dict(lqr_iter=10, not_improved_lim=5, m_ref=2, eps=1e-7, best_cost_eps=1e-4)
    o.update(kw)
    return IlqrOpts(**o)


FAKE = 1 << 20          # a non-NULL, 256-byte aligned address that is never dereferenced: every call below fails first


def _call(dims, opts, n_steps=3, ptrs=None, ws_bytes=1 << 30, fn="mpcb200_episode_f32"):
    p = Params(u_lo=0, u_hi=0, delta_u=0, ls_decay=0.2)
    if ptrs is None:
        ptrs = [FAKE] * 15    # C c F f x_init u_init u_lower u_upper u_zero_I xs us costs info u_next workspace
    return getattr(_lib.lib(), fn)(ctypes.byref(dims) if dims is not None else None, ctypes.byref(p),
                                   ctypes.byref(opts) if opts is not None else None, n_steps, *ptrs, ws_bytes, None)


def _without(k):
    ptrs = [FAKE] * 15
    ptrs[k] = None
    return ptrs


def test_argument_errors_are_status_codes():
    d, o = _dims(), _opts()
    assert _call(None, o) == 1                                  # NULL dims
    assert _call(d, None) == 1                                  # NULL options
    for k in (0, 1, 4, 9, 10, 11, 12, 13, 14):                  # C c x_init xs us costs info u_next workspace
        assert _call(d, o, ptrs=_without(k)) == 1, k
        assert _call(d, o, ptrs=_without(k), fn="mpcb200_episode_f64") == 1, k
    assert _call(d, o, ptrs=_without(2)) == 1                   # F of a LinDx problem
    assert _call(_dims(T=2), o) == 2                            # the warm-start shift needs T >= 3
    assert _call(d, o, n_steps=0) == 2
    assert _call(d, o, n_steps=-1) == 2
    assert _call(d, _opts(lqr_iter=0)) == 2                     # the solve's own checks
    assert _call(d, _opts(m_ref=3)) == 2
    assert _call(_dims(dynamics_kind=DYN_CARTPOLE), o) == 2
    need = _lib.lib().mpcb200_episode_workspace_bytes(ctypes.byref(d), ctypes.byref(o), 4)
    assert _call(d, o, ws_bytes=need - 1) == 2                  # a short workspace
    ptrs = [FAKE] * 14 + [FAKE + 16]
    assert _call(d, o, ptrs=ptrs, ws_bytes=need) == 2           # a workspace that is not 256-byte aligned


def _up256(v):
    return (v + 255) // 256 * 256


@pytest.mark.parametrize("esz", [4, 8])
@pytest.mark.parametrize("shape", [dict(B=4, T=5, n=8, m=2), dict(B=33, T=25, n=5, m=1, dynamics_kind=DYN_CARTPOLE),
                                   dict(B=7, T=9, n=20, m=4)])
def test_workspace_is_the_solve_plus_the_episode_buffers(esz, shape):
    L, o = _lib.lib(), _opts(m_ref=shape["m"])
    d = _dims(**shape)
    solve = L.mpcb200_ilqr_workspace_bytes(ctypes.byref(d), ctypes.byref(o), esz)
    B, T, n, m = shape["B"], shape["T"], shape["n"], shape["m"]
    extra = (_up256(T * B * n * esz) + _up256(T * B * m * esz) + 2 * _up256(B * esz) + _up256(8)   # best x, u, costs, fdn, info
             + _up256(B * n * esz) + _up256(T * B * m * esz) + _up256(2 * B * n * esz) + _up256(16))  # state warm traj counter
    assert solve > 0
    assert L.mpcb200_episode_workspace_bytes(ctypes.byref(d), ctypes.byref(o), esz) == solve + extra
    assert L.mpcb200_episode_workspace_bytes(None, ctypes.byref(o), esz) == 0
    assert L.mpcb200_episode_workspace_bytes(ctypes.byref(d), ctypes.byref(o), 2) == 0


# ------------------------------------------------------------------------------------------------------------------
# routing
# ------------------------------------------------------------------------------------------------------------------
T, B = 6, 3


def _problem(n=8, m=2, dtype=torch.float32, device="cuda"):
    C = torch.zeros(T, B, n + m, n + m, dtype=dtype, device=device)
    c = torch.zeros(T, B, n + m, dtype=dtype, device=device)
    F = torch.zeros(T - 1, B, n, n + m, dtype=dtype, device=device)
    f = torch.zeros(T - 1, B, n, dtype=dtype, device=device)
    x0 = torch.zeros(B, n, dtype=dtype, device=device)
    u = torch.zeros(T, B, m, dtype=dtype, device=device)
    return QuadCost(C, c), LinDx(F, f), x0, u


def _device(ctrl, cost, dx, x0, u):
    return control._takes_device_path(ctrl, x0, cost, dx, u)


@pytest.fixture
def fake():
    with FakeTensorMode(allow_non_fake_inputs=True) as mode:
        yield mode


def test_device_path_for_what_the_device_loop_takes(fake):
    cost, dx, x0, u = _problem()
    assert _device(MPC(8, 2, T), cost, dx, x0, u)
    assert _device(MPC(8, 2, T, u_lower=-1.0, u_upper=1.0, delta_u=0.5), cost, dx, x0, u)
    assert _device(MPC(8, 2, T, slew_rate_penalty=0.1), cost, dx, x0, u)
    assert _device(MPC(6, 1, T), *_problem(6, 1))
    assert _device(MPC(20, 4, T), *_problem(20, 4))
    for sysdx, (n, m) in ((CartpoleDx(), (5, 1)), (PendulumDx(), (3, 1))):
        cost, _, x0, u = _problem(n, m)
        assert _device(MPC(n, m, T, grad_method=GradMethods.AUTO_DIFF), cost, sysdx, x0, u)
        assert _device(MPC(n, m, T, slew_rate_penalty=0.5), cost, sysdx, x0, u)


def test_host_path_for_everything_else(fake, monkeypatch):
    cost, dx, x0, u = _problem()
    assert not _device(MPC(8, 2, T, verbose=1), cost, dx, x0, u)
    assert not _device(MPC(8, 2, T), torch.nn.Linear(10, 1), dx, x0, u)       # a Module cost
    assert not _device(MPC(8, 2, T), cost, torch.nn.Linear(10, 8), x0, u)     # opaque dynamics
    assert not _device(MPC(8, 2, T), cost, dx, x0.double(), u)
    assert not _device(MPC(8, 2, T, slew_rate_penalty=0.1, prev_ctrl=torch.zeros(B, 2)), cost, dx, x0, u)
    monkeypatch.setattr(solver, "_graph_cond_unavailable", True)
    assert not _device(MPC(8, 2, T), cost, dx, x0, u)


def test_cpu_tensors_take_the_host_path():
    assert not _device(MPC(8, 2, T), *_problem(device="cpu"))


def test_horizon_and_step_count_are_checked_first(fake):
    cost, dx, x0, _ = _problem()
    for t in (1, 2):
        with pytest.raises(MpcB200Error, match="T >= 3"):
            receding_horizon(MPC(8, 2, t), x0, cost, dx, 5)
    for steps in (0, -3):
        with pytest.raises(MpcB200Error, match="n_steps"):
            receding_horizon(MPC(8, 2, T), x0, cost, dx, steps)


@pytest.mark.parametrize("shape", [(3, 1, 1), (25, 8, 1), (10, 4, 3)])
def test_warm_start_rule_is_the_notebooks(shape):
    g = torch.Generator().manual_seed(0)
    plan = torch.randn(*shape, generator=g, dtype=torch.float64)
    T_, n_batch, n_ctrl = shape
    u_init = torch.cat((plan[1:], torch.zeros(1, n_batch, n_ctrl, dtype=torch.float64)), dim=0)
    u_init[-2] = u_init[-3]
    assert torch.equal(shift_warm_start(plan), u_init)
