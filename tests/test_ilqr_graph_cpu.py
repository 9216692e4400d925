"""CPU: the device-side iLQR loop (mpcb200_ilqr_*) refuses malformed arguments with status codes before it touches a
device, sizes its workspace without one, and MPC.forward's choice between the device loop and the host loop is made on
tensor metadata alone (FakeTensor CUDA tensors here: no device, no kernel)."""
import ctypes

import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode

from mpc.pytorch_b200 import _lib, solver
from mpc.pytorch_b200._lib import Dims, IlqrOpts, Params
from mpc.pytorch_b200.dynamics import DYN_CARTPOLE, CartpoleDx, PendulumDx
from mpc.pytorch_b200.solver import MPC, GradMethods, LinDx, QuadCost


def _dims(B=4, T=5, n=8, m=2, F_T=None, **kw):
    return Dims(B=B, T=T, n=n, m=m, F_T=T - 1 if F_T is None else F_T, has_f=0, bounds_kind=0, has_zero_mask=0,
                has_delta_u=0, max_ls_iter=10, pnqp_max_iter=20, do_rollout=1, **kw)


def _opts(**kw):
    o = dict(lqr_iter=10, not_improved_lim=5, m_ref=2, eps=1e-7, best_cost_eps=1e-4)
    o.update(kw)
    return IlqrOpts(**o)


FAKE = 1 << 20          # a non-NULL, 256-byte aligned address that is never dereferenced: every call below fails first


def _call(dims, opts, ptrs=None, ws_bytes=0, fn="mpcb200_ilqr_f32"):
    p = Params(u_lo=0, u_hi=0, delta_u=0, ls_decay=0.2)
    if ptrs is None:
        ptrs = [FAKE] * 15             # C c F f x_init u_init u_lower u_upper u_zero_I best_x best_u costs fdn info ws
    return getattr(_lib.lib(), fn)(ctypes.byref(dims) if dims is not None else None, ctypes.byref(p),
                                   ctypes.byref(opts) if opts is not None else None, *ptrs, ws_bytes, None)


def test_argument_errors_are_status_codes():
    d, o = _dims(), _opts()
    assert _call(None, o) == 1                                  # NULL dims
    assert _call(d, None) == 1                                  # NULL options
    assert _call(d, o, ptrs=[None] * 15) == 1                   # NULL tensors
    no_ws = [FAKE] * 14 + [None]
    assert _call(d, o, ptrs=no_ws, fn="mpcb200_ilqr_f64") == 1
    assert _call(d, _opts(lqr_iter=0)) == 2                     # lqr_iter < 1
    assert _call(d, _opts(m_ref=3)) == 2                        # m_ref > m
    assert _call(d, _opts(m_ref=0)) == 2
    assert _call(_dims(F_T=2), o) == 2
    # a known system with the wrong (n_state, n_ctrl)
    assert _call(_dims(dynamics_kind=DYN_CARTPOLE), _opts()) == 2
    assert _call(_dims(n=5, m=1, dynamics_kind=DYN_CARTPOLE), _opts(m_ref=1)) == 2   # valid, but no workspace
    # a workspace smaller than mpcb200_ilqr_workspace_bytes
    need = _lib.lib().mpcb200_ilqr_workspace_bytes(ctypes.byref(d), ctypes.byref(o), 4)
    assert _call(d, o, ws_bytes=need - 1) == 2
    assert b"12.3" in _lib.lib().mpcb200_strerror(_lib.ERR_NO_GRAPH_COND)


def test_workspace_size_grows_with_batch_and_horizon():
    L = _lib.lib()
    o = _opts()

    def size(esz=4, **kw):
        return L.mpcb200_ilqr_workspace_bytes(ctypes.byref(_dims(**kw)), ctypes.byref(o), esz)

    base = size(B=16, T=10)
    assert base > 0
    assert size(B=32, T=10) > base and size(B=16, T=20) > base
    assert size(8, B=16, T=10) > base
    assert L.mpcb200_ilqr_workspace_bytes(None, ctypes.byref(o), 4) == 0
    assert L.mpcb200_ilqr_workspace_bytes(ctypes.byref(_dims()), ctypes.byref(o), 2) == 0
    # a known system also keeps its linearisation there
    kd = _dims(n=5, m=1, dynamics_kind=DYN_CARTPOLE)
    ld = _dims(n=5, m=1)
    assert L.mpcb200_ilqr_workspace_bytes(ctypes.byref(kd), ctypes.byref(o), 4) > \
        L.mpcb200_ilqr_workspace_bytes(ctypes.byref(ld), ctypes.byref(o), 4)


# ------------------------------------------------------------------------------------------------------------------
# the predicate
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


def _decide(ctrl, cost, dx, x0, u):
    return solver._use_device_loop(ctrl, x0, cost, dx, u)


@pytest.fixture
def fake():
    with FakeTensorMode(allow_non_fake_inputs=True) as mode:
        yield mode


def test_predicate_takes_linear_and_known_systems(fake):
    cost, dx, x0, u = _problem()
    assert _decide(MPC(8, 2, T), cost, dx, x0, u)
    assert _decide(MPC(8, 2, T, u_lower=-1.0, u_upper=1.0, delta_u=0.5), cost, dx, x0, u)
    lo = torch.full((T, B, 2), -1.0, device="cuda")
    assert _decide(MPC(8, 2, T, u_lower=lo, u_upper=-lo, u_zero_I=torch.zeros(T, B, 2, device="cuda")),
                   cost, dx, x0, u)
    assert _decide(MPC(8, 2, T), cost, LinDx(dx.F, None), x0, u)
    cost64, dx64, x064, u64 = _problem(dtype=torch.float64)
    assert _decide(MPC(8, 2, T), cost64, dx64, x064, u64)
    assert _decide(MPC(6, 1, T), *_problem(6, 1))                      # zero-padded instance
    assert _decide(MPC(20, 4, T), *_problem(20, 4))                    # large-shape kernels
    for sysdx, (n, m) in ((CartpoleDx(), (5, 1)), (PendulumDx(), (3, 1))):
        cost, _, x0, u = _problem(n, m)
        for gm in (GradMethods.ANALYTIC, GradMethods.AUTO_DIFF):
            assert _decide(MPC(n, m, T, grad_method=gm), cost, sysdx, x0, u)
        assert not _decide(MPC(n, m, T, grad_method=GradMethods.FINITE_DIFF), cost, sysdx, x0, u)


def test_predicate_turns_down_everything_else(fake):
    cost, dx, x0, u = _problem()
    ctrl = MPC(8, 2, T)
    assert not _decide(MPC(8, 2, T, slew_rate_penalty=0.1), cost, dx, x0, u)
    assert not _decide(MPC(8, 2, T, verbose=1), cost, dx, x0, u)
    assert _decide(MPC(8, 2, T, verbose=-1), cost, dx, x0, u)
    assert not _decide(MPC(8, 2, T, lqr_iter=0), cost, dx, x0, u)
    assert not _decide(MPC(8, 2, 1), cost, dx, x0, u)                  # T = 1
    # dtype / device
    assert not _decide(ctrl, cost, dx, x0.double(), u)
    assert not _decide(ctrl, QuadCost(cost.C.double(), cost.c), dx, x0, u)
    assert not _decide(ctrl, cost, LinDx(dx.F.double(), dx.f), x0, u)
    assert not _decide(ctrl, cost, dx, x0, u.double())
    h16 = _problem(dtype=torch.float16)
    assert not _decide(ctrl, *h16)
    assert not _decide(MPC(8, 2, T, u_lower=torch.zeros(T, B, 2, dtype=torch.float64, device="cuda"),
                           u_upper=torch.ones(T, B, 2, dtype=torch.float64, device="cuda")), cost, dx, x0, u)
    assert not _decide(MPC(8, 2, T, u_zero_I=torch.zeros(T, B, 2)), cost, dx, x0, u)    # mask on the CPU
    # cost and dynamics kinds
    assert not _decide(ctrl, torch.nn.Linear(10, 1), dx, x0, u)
    assert not _decide(ctrl, cost, torch.nn.Linear(10, 8), x0, u)
    assert not _decide(ctrl, cost, LinDx(None, None), x0, u)
    # a known system of another shape than the problem's
    assert not _decide(MPC(8, 2, T), cost, CartpoleDx(), x0, u)
    # (n_state, n_ctrl) beyond every kernel
    assert not _decide(MPC(300, 2, T), *_problem(300, 2))


def test_predicate_turns_down_cpu_tensors():
    cost, dx, x0, u = _problem(device="cpu")
    assert not _decide(MPC(8, 2, T), cost, dx, x0, u)


def test_predicate_remembers_a_driver_without_conditional_nodes(fake, monkeypatch):
    cost, dx, x0, u = _problem()
    monkeypatch.setattr(solver, "_graph_cond_unavailable", True)
    assert not _decide(MPC(8, 2, T), cost, dx, x0, u)
