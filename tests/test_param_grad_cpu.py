"""CPU: which linearisations of MPC's differentiable tail take the parameter-VJP kernel (dynamics.DynLinearize), the
argument errors of dyn_linearize_vjp_raw, and the exported symbols.  No kernel is launched here."""
import types

import pytest
import torch


def _cuda_like(dtype=torch.float64):
    """What known_kind looks at of the solve's tensor: a CUDA tensor of `dtype`, without a device."""
    return types.SimpleNamespace(is_cuda=True, dtype=dtype)


def _route(dx, grad_method, diff, ref, n=None):
    from mpc.pytorch_b200 import MPC
    n = dx.n_state if n is None else n
    return MPC(n, 1, 5, grad_method=grad_method)._kernel_linearization(dx, ref, diff)[0]


@pytest.mark.parametrize("diff", [True, False])
def test_known_systems_route_to_the_kernels_under_analytic_and_auto_diff(diff):
    from mpc.pytorch_b200 import GradMethods
    from mpc.pytorch_b200.dynamics import DYN_CARTPOLE, DYN_PENDULUM, CartpoleDx, PendulumDx
    for dx, kind in ((CartpoleDx(), DYN_CARTPOLE), (PendulumDx(), DYN_PENDULUM)):
        for gm in (GradMethods.ANALYTIC, GradMethods.AUTO_DIFF):
            assert _route(dx, gm, diff, _cuda_like()) == kind
            assert _route(dx, gm, diff, _cuda_like(torch.float32)) == kind
        assert _route(dx, GradMethods.FINITE_DIFF, diff, _cuda_like()) == 0          # the torch code as it is
        assert _route(dx, GradMethods.AUTO_DIFF, diff, torch.zeros(1, dtype=torch.float64)) == 0     # CPU tensors
        assert _route(dx, GradMethods.AUTO_DIFF, diff, _cuda_like(torch.float16)) == 0
        assert _route(dx, GradMethods.AUTO_DIFF, diff, _cuda_like(), n=dx.n_state + 1) == 0        # other (n, m)


def test_opaque_modules_and_passthrough_kinds_keep_the_torch_tail():
    from mpc.pytorch_b200 import GradMethods
    from mpc.pytorch_b200.dynamics import DYN_CARTPOLE, DYN_CTRL_PASSTHROUGH, CartpoleDx
    from mpc.pytorch_b200.solver import CtrlPassthroughDynamics
    dx = CartpoleDx()

    class Opaque(torch.nn.Module):
        n_state, n_ctrl = 5, 1

        def forward(self, x, u):
            return dx(x, u)
    assert _route(Opaque(), GradMethods.AUTO_DIFF, True, _cuda_like()) == 0
    wrapped = CtrlPassthroughDynamics(dx)
    assert _route(wrapped, GradMethods.AUTO_DIFF, False, _cuda_like()) == DYN_CARTPOLE | DYN_CTRL_PASSTHROUGH
    assert _route(wrapped, GradMethods.AUTO_DIFF, True, _cuda_like()) == 0


def test_the_function_is_taken_only_when_params_need_a_gradient(monkeypatch):
    """linearize_known: DynLinearize when autograd records and params requires grad, else one plain launch."""
    from mpc.pytorch_b200 import dynamics
    calls = []
    monkeypatch.setattr(dynamics, "dyn_linearize_raw", lambda *a: calls.append("raw") or (None, None))
    monkeypatch.setattr(dynamics.DynLinearize, "apply", lambda *a: calls.append("function") or (None, None))
    x, u = torch.zeros(3, 2, 3), torch.zeros(3, 2, 1)
    learn = dynamics.PendulumDx(params=torch.tensor((10.0, 1.0, 1.0), requires_grad=True))
    frozen = dynamics.PendulumDx()
    kp = learn.mpcb200_params()
    dynamics.linearize_known(learn, dynamics.DYN_PENDULUM, kp, 3, x, u)
    dynamics.linearize_known(frozen, dynamics.DYN_PENDULUM, kp, 3, x, u)
    with torch.no_grad():
        dynamics.linearize_known(learn, dynamics.DYN_PENDULUM, kp, 3, x, u)
    assert calls == ["function", "raw", "raw"]


def test_vjp_raw_argument_errors():
    from mpc.pytorch_b200._lib import MpcB200Error
    from mpc.pytorch_b200.dynamics import (DYN_CARTPOLE, DYN_CTRL_PASSTHROUGH, DYN_LINEAR, DYN_PENDULUM,
                                           PendulumDx, dyn_linearize_vjp_raw)
    kp = PendulumDx().mpcb200_params()
    T, B = 4, 2
    x, u = torch.zeros(T, B, 3, dtype=torch.float64), torch.zeros(T, B, 1, dtype=torch.float64)
    dF, df = torch.zeros(T - 1, B, 3, 4, dtype=torch.float64), torch.zeros(T - 1, B, 3, dtype=torch.float64)
    cases = [
        ((DYN_PENDULUM | DYN_CTRL_PASSTHROUGH, kp, T, x, u, dF, df), "passthrough"),
        ((DYN_LINEAR, kp, T, x, u, dF, df), "not a known system"),
        ((DYN_CARTPOLE, kp, T, x, u, dF, df), "dF: expected shape (3, 2, 5, 6)"),
        ((DYN_PENDULUM, kp, T, x, u, dF[:, :, :, :3], df), "dF: expected shape"),
        ((DYN_PENDULUM, kp, T, x, u, dF, df[:-1]), "df: expected shape"),
        ((DYN_PENDULUM, kp, T, x, u, dF.float(), df), "dF is torch.float32"),
        ((DYN_PENDULUM, kp, T, x, u[:, :1], dF, df), "u: expected shape"),
        ((DYN_PENDULUM, kp, T, x, u, dF, df), "CUDA tensors only"),
    ]
    for args, msg in cases:
        with pytest.raises(MpcB200Error, match=msg.replace("(", r"\(").replace(")", r"\)")):
            dyn_linearize_vjp_raw(*args)


def test_vjp_symbols_are_exported():
    from mpc.pytorch_b200 import _lib
    for sym in ("mpcb200_dyn_linearize_vjp_f32", "mpcb200_dyn_linearize_vjp_f64"):
        assert sym in _lib.EXPORTED_SYMBOLS
        assert hasattr(_lib.lib(), sym)
