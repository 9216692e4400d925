"""CPU: a slew-rate penalty on the device.  The control-passthrough kind of a known system in the C ABI (status codes
before any launch, workspace sizing, the instance list), CtrlPassthroughDynamics as a known system, and MPC.forward's
choice of the device loop for slew solves, made on tensor metadata alone (FakeTensor CUDA tensors: no device)."""
import ctypes

import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode

from mpc.pytorch_b200 import _lib, solver
from mpc.pytorch_b200._lib import Dims, IlqrOpts, Params
from mpc.pytorch_b200.dynamics import (DYN_CARTPOLE, DYN_CTRL_PASSTHROUGH, DYN_LINEAR, DYN_PENDULUM, CartpoleDx,
                                       PendulumDx, known_kind)
from mpc.pytorch_b200.solver import MPC, CtrlPassthroughDynamics, GradMethods, LinDx, QuadCost

CP, PP = DYN_CARTPOLE | DYN_CTRL_PASSTHROUGH, DYN_PENDULUM | DYN_CTRL_PASSTHROUGH
FAKE = 1 << 20          # a non-NULL, 256-byte aligned address that is never dereferenced: every call below fails first


def _dims(B=4, T=5, n=6, m=1, **kw):
    return Dims(B=B, T=T, n=n, m=m, F_T=T - 1, has_f=0, bounds_kind=0, has_zero_mask=0, has_delta_u=0,
                max_ls_iter=10, pnqp_max_iter=20, do_rollout=1, **kw)


def _opts():
    return IlqrOpts(lqr_iter=10, not_improved_lim=5, m_ref=1, eps=1e-7, best_cost_eps=1e-4)


def _ilqr(dims, ptrs=None, ws_bytes=0):
    p = Params(u_lo=0, u_hi=0, delta_u=0, ls_decay=0.2)
    ptrs = [FAKE] * 15 if ptrs is None else ptrs
    return _lib.lib().mpcb200_ilqr_f64(ctypes.byref(dims), ctypes.byref(p), ctypes.byref(_opts()), *ptrs, ws_bytes,
                                       None)


def _step(dims, ptrs=None):
    p = Params(u_lo=0, u_hi=0, delta_u=0, ls_decay=0.2)
    ptrs = [FAKE] * 21 if ptrs is None else ptrs
    return _lib.lib().mpcb200_lqr_step_f64(ctypes.byref(dims), ctypes.byref(p), *ptrs, None)


def _dyn(fn, kind, ptrs):
    dyn = (ctypes.c_double * 8)(*([1.0] * 8))
    return getattr(_lib.lib(), fn)(kind, dyn, 4, 5, *ptrs, None)


def test_passthrough_kind_argument_errors_are_status_codes():
    ws = _lib.lib().mpcb200_ilqr_workspace_bytes
    for kind, (n, m) in ((CP, (6, 1)), (PP, (4, 1))):
        # the flagged kind at any other (n, m) than the system's n+1, 1
        for bad in ((n - 1, m), (n + 1, m), (n, 2)):
            d = _dims(n=bad[0], m=bad[1], dynamics_kind=kind)
            assert _ilqr(d) == 2
            assert ws(ctypes.byref(d), ctypes.byref(_opts()), 8) == 0
            assert _step(d) in (2, 3)
        good = _dims(n=n, m=m, dynamics_kind=kind)
        assert _ilqr(good) == 2                                  # valid, but no workspace
        assert _ilqr(good, ptrs=[None] * 15) == 1                # NULL tensors
        assert _step(good, ptrs=[None] * 21) == 1
        # the rollout and linearisation calls take the kind, and check their pointers first
        assert _dyn("mpcb200_dyn_rollout_f64", kind, [None] * 3) == 1
        assert _dyn("mpcb200_dyn_linearize_f64", kind, [None] * 4) == 1
    # the flag on DYN_LINEAR, or on an unknown system, is no kind
    for kind in (DYN_CTRL_PASSTHROUGH, DYN_CTRL_PASSTHROUGH | 3):
        for n in (1, 4, 6):
            d = _dims(n=n, dynamics_kind=kind)
            assert _ilqr(d) == 2
            assert _step(d) in (2, 3)
            assert ws(ctypes.byref(d), ctypes.byref(_opts()), 8) == 0
        assert _dyn("mpcb200_dyn_rollout_f64", kind, [FAKE] * 3) == 2
        assert _dyn("mpcb200_dyn_linearize_f64", kind, [FAKE] * 4) == 2


def test_passthrough_workspace_holds_the_augmented_linearisation():
    L, o = _lib.lib(), _opts()

    def size(esz, **kw):
        return L.mpcb200_ilqr_workspace_bytes(ctypes.byref(_dims(B=64, T=20, **kw)), ctypes.byref(o), esz)
    for kind, sys_kind, n in ((CP, DYN_CARTPOLE, 6), (PP, DYN_PENDULUM, 4)):
        for esz in (4, 8):
            flagged = size(esz, n=n, dynamics_kind=kind)
            assert flagged > size(esz, n=n)                                  # LinDx at the same (n, m)
            assert flagged > size(esz, n=n - 1, dynamics_kind=sys_kind)      # the system without the passthrough


def test_dynamics_only_instances_are_not_listed():
    pairs = _lib.supported_pairs()
    assert (6, 1) not in pairs
    assert not _lib.lib().mpcb200_supported(6, 1)
    # the step asks for its gain store by the dynamics kind: (6, 1) exists only for the passthrough cartpole
    d = _dims(T=20, dynamics_kind=CP)
    assert _lib.lib().mpcb200_step_smem_bytes(ctypes.byref(d), 8) > 0
    assert _lib.lib().mpcb200_step_smem_bytes(ctypes.byref(_dims(T=20)), 8) == 0


def test_step_picks_the_dynamics_instance_only_for_its_kind():
    from mpc.pytorch_b200.step import _pick_instance
    from mpc.pytorch_b200._lib import MpcB200Error
    assert _pick_instance(6, 1, 8, CP) == (6, 1)
    assert _pick_instance(4, 1, 4, PP) == (4, 1)
    assert _pick_instance(6, 1, 8) != (6, 1)                 # LinDx (6, 1) pads as before
    with pytest.raises(MpcB200Error):
        _pick_instance(5, 1, 8, CP)
    with pytest.raises(MpcB200Error):
        _pick_instance(6, 1, 8, PP)


# ------------------------------------------------------------------------------------------------------------------
# CtrlPassthroughDynamics as a known system
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def fake():
    with FakeTensorMode(allow_non_fake_inputs=True) as mode:
        yield mode


def test_passthrough_of_a_known_system_is_known():
    with FakeTensorMode(allow_non_fake_inputs=True):
        t = torch.zeros(3, 6, dtype=torch.float64, device="cuda")
        t4, t4f = t[:, :4], t[:, :4].float()
    cart = CartpoleDx(params=torch.tensor((9.0, 1.5, 0.2, 0.7), dtype=torch.float64))
    wrapped = CtrlPassthroughDynamics(cart)
    kind, params = known_kind(wrapped, 6, 1, t)
    assert kind == CP and params == tuple(cart.mpcb200_params())
    assert (wrapped.n_state, wrapped.n_ctrl) == (6, 1)
    assert known_kind(wrapped, 5, 1, t)[0] == DYN_LINEAR              # the inner shape is not the wrapper's
    pend = CtrlPassthroughDynamics(PendulumDx())
    assert known_kind(pend, 4, 1, t4)[0] == PP
    assert known_kind(pend, 4, 1, t4f)[0] == PP
    # an opaque inner Module keeps the Module path
    opaque = CtrlPassthroughDynamics(torch.nn.Linear(6, 5))
    assert known_kind(opaque, 6, 1, t) == (DYN_LINEAR, None)
    assert not hasattr(opaque, "mpcb200_kind") and not hasattr(opaque, "mpcb200_params")
    # and a CPU tensor is not the kernels'
    assert known_kind(wrapped, 6, 1, torch.zeros(3, 6, dtype=torch.float64))[0] == DYN_LINEAR


def test_passthrough_parameters_follow_the_inner_system():
    cart = CartpoleDx()
    wrapped = CtrlPassthroughDynamics(cart)
    with torch.no_grad():
        cart.params[0] = 7.5
    assert wrapped.mpcb200_params() == cart.mpcb200_params()
    assert wrapped.mpcb200_params()[0] == 7.5


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
    return solver._use_slew_device_loop(ctrl, x0, cost, dx, u)


def test_slew_predicate_takes_linear_and_known_systems(fake):
    for n, m in ((3, 4), (8, 2), (16, 4), (6, 1)):           # exact, padded, large and padded augmented shapes
        cost, dx, x0, u = _problem(n, m)
        assert _decide(MPC(n, m, T, slew_rate_penalty=0.1), cost, dx, x0, u)
        assert _decide(MPC(n, m, T, slew_rate_penalty=0.1, u_lower=-1.0, u_upper=1.0, delta_u=0.5), cost, dx, x0, u)
        assert _decide(MPC(n, m, T, slew_rate_penalty=0.1), cost, LinDx(dx.F, None), x0, u)
        assert _decide(MPC(n, m, T, slew_rate_penalty=0.1, verbose=-1), *_problem(n, m, torch.float64))
    lo = torch.full((T, B, 2), -1.0, device="cuda")
    assert _decide(MPC(8, 2, T, slew_rate_penalty=0.1, u_lower=lo, u_upper=-lo,
                       u_zero_I=torch.zeros(T, B, 2, device="cuda")), *_problem())
    for prev in (torch.zeros(2, device="cuda"), torch.zeros(B, 2, device="cuda"),
                 torch.zeros(B, 2, dtype=torch.float64, device="cuda")):
        assert _decide(MPC(8, 2, T, slew_rate_penalty=0.1, prev_ctrl=prev), *_problem())
    for sysdx, (n, m) in ((CartpoleDx(), (5, 1)), (PendulumDx(), (3, 1))):
        cost, _, x0, u = _problem(n, m)
        for gm in (GradMethods.ANALYTIC, GradMethods.AUTO_DIFF):
            assert _decide(MPC(n, m, T, grad_method=gm, slew_rate_penalty=0.1), cost, sysdx, x0, u)
            assert _decide(MPC(n, m, T, grad_method=gm, slew_rate_penalty=0.1, u_lower=-1.0, u_upper=1.0,
                               prev_ctrl=torch.zeros(B, 1, device="cuda")), cost, sysdx, x0, u)
        assert not _decide(MPC(n, m, T, grad_method=GradMethods.FINITE_DIFF, slew_rate_penalty=0.1), cost, sysdx,
                           x0, u)
    # the slew predicate leaves unpenalised solves to _use_device_loop, and the other way round
    assert not _decide(MPC(8, 2, T), *_problem())
    assert not solver._use_device_loop(MPC(8, 2, T, slew_rate_penalty=0.1), _problem()[2], *_problem()[:2],
                                       _problem()[3])


def test_slew_predicate_turns_down_everything_else(fake):
    cost, dx, x0, u = _problem()

    def ctrl(**kw):
        return MPC(8, 2, T, slew_rate_penalty=0.1, **kw)
    assert not _decide(ctrl(verbose=1), cost, dx, x0, u)
    assert not _decide(ctrl(lqr_iter=0), cost, dx, x0, u)
    assert not _decide(MPC(8, 2, 1, slew_rate_penalty=0.1), cost, dx, x0, u)       # T = 1
    assert not _decide(ctrl(), cost, dx, x0.double(), u)
    assert not _decide(ctrl(), QuadCost(cost.C.double(), cost.c), dx, x0, u)
    assert not _decide(ctrl(), cost, LinDx(dx.F.double(), dx.f), x0, u)
    assert not _decide(ctrl(), *_problem(dtype=torch.float16))
    assert not _decide(ctrl(u_zero_I=torch.zeros(T, B, 2)), cost, dx, x0, u)       # mask on the CPU
    assert not _decide(ctrl(prev_ctrl=torch.zeros(B, 2)), cost, dx, x0, u)         # prev_ctrl on the CPU
    assert not _decide(ctrl(prev_ctrl=[0.0, 0.0]), cost, dx, x0, u)
    assert not _decide(ctrl(), torch.nn.Linear(10, 1), dx, x0, u)                   # a Module cost
    assert not _decide(ctrl(), cost, torch.nn.Linear(10, 8), x0, u)                 # opaque dynamics
    assert not _decide(ctrl(), cost, CtrlPassthroughDynamics(torch.nn.Linear(10, 8)), x0, u)
    assert not _decide(ctrl(), cost, LinDx(None, None), x0, u)
    assert not _decide(ctrl(), cost, CartpoleDx(), x0, u)                           # another shape than the problem's
    assert not _decide(MPC(300, 2, T, slew_rate_penalty=0.1), *_problem(300, 2))    # beyond every kernel
    # a known system already wrapped has no instance one slew level up
    cost5, _, x05, u5 = _problem(6, 1)
    assert not _decide(MPC(6, 1, T, slew_rate_penalty=0.1), cost5, CtrlPassthroughDynamics(CartpoleDx()), x05, u5)


def test_slew_predicate_turns_down_cpu_tensors_and_a_driver_without_conditional_nodes(monkeypatch):
    assert not _decide(MPC(8, 2, T, slew_rate_penalty=0.1), *_problem(device="cpu"))
    with FakeTensorMode(allow_non_fake_inputs=True):
        monkeypatch.setattr(solver, "_graph_cond_unavailable", True)
        assert not _decide(MPC(8, 2, T, slew_rate_penalty=0.1), *_problem())
