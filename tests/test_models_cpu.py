"""Learned / affine dynamics modules (mpc.dynamics drop-in path) vs fixtures of the reference's modules
(oracle/make_golden_nn.py) and vs autograd.  Module arithmetic only - no solver call, so it runs without a GPU."""
import pytest
import torch

from tests.helpers import build_net, load_golden


@pytest.mark.parametrize("act", ["sigmoid", "relu"])
def test_nn_dynamics_step_and_jacobians_match_reference(act):
    g = load_golden(f"nn_dynamics_{act}_f64")
    net = build_net(g, act)
    x, u = g["step_x"], g["step_u"]
    assert float((net(x, u) - g["step_next"]).abs().max()) < 1e-14
    R, S = net.grad_input(x, u)
    assert float((R - g["R"]).abs().max()) < 1e-14 and float((S - g["S"]).abs().max()) < 1e-14
    assert net(x[0], u[0]).shape == (3,)                      # 1-d inputs (reference :58-63, :76-77)
    R1, S1 = net.grad_input(x[0], u[0])
    assert R1.shape == (3, 3) and S1.shape == (3, 2)


@pytest.mark.parametrize("act,passthrough", [("sigmoid", True), ("relu", False), ("elu", True)])
def test_nn_dynamics_grad_input_is_the_autograd_jacobian(act, passthrough):
    from mpc.dynamics import NNDynamics
    torch.manual_seed(3)
    net = NNDynamics(4, 2, hidden_sizes=[9, 7, 5], activation=act, passthrough=passthrough).double()
    x, u = torch.randn(6, 4, dtype=torch.float64), torch.randn(6, 2, dtype=torch.float64)
    R, S = net.grad_input(x, u)
    Jx, Ju = torch.autograd.functional.jacobian(lambda a, b: net(a, b).sum(0), (x, u))
    assert float((Jx.permute(1, 0, 2) - R).abs().max()) < 1e-13
    assert float((Ju.permute(1, 0, 2) - S).abs().max()) < 1e-13
    # differentiable in the weights (what learning the dynamics through the controller needs)
    (R.sum() + S.sum()).backward()
    assert all(fc.weight.grad is not None for fc in net.fcs[:-1])


def test_affine_dynamics():
    from mpc.dynamics import AffineDynamics, CtrlPassthroughDynamics
    g = load_golden("affine_dynamics_f64")
    dx = AffineDynamics(g["A"], g["B"], g["c0"])
    x, u = torch.randn(5, 3, dtype=torch.float64), torch.randn(5, 2, dtype=torch.float64)
    want = x @ g["A"].t() + u @ g["B"].t() + g["c0"]
    assert torch.allclose(dx(x, u), want, atol=1e-14) and torch.allclose(dx(x[0], u[0]), want[0], atol=1e-14)
    R, S = dx.grad_input(x, u)
    assert R.shape == (5, 3, 3) and torch.equal(R[2], g["A"]) and torch.equal(S[4], g["B"])
    aug = CtrlPassthroughDynamics(dx)                            # state [u_prev; x] (reference :133-156)
    out = aug(torch.cat((u, x), 1), 2 * u)
    assert torch.equal(out[:, :2], 2 * u) and torch.equal(out[:, 2:], dx(x, 2 * u))


def test_nn_dynamics_pickles():
    """The reference makes its MLP picklable by hand (mpc/dynamics.py:39-54); a plain Module round-trips as is."""
    import io
    from mpc.dynamics import NNDynamics
    torch.manual_seed(1)
    net = NNDynamics(3, 1, hidden_sizes=[8], activation="relu", passthrough=False)
    buf = io.BytesIO()
    torch.save(net, buf)
    buf.seek(0)
    net2 = torch.load(buf, weights_only=False)
    x, u = torch.randn(4, 3), torch.randn(4, 1)
    assert torch.equal(net(x, u), net2(x, u)) and net2.activation == "relu" and net2.passthrough is False
