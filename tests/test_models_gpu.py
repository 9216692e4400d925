"""iLQR through learned / affine dynamics with GradMethods.ANALYTIC (grad_input Jacobians, reference
mpc/mpc.py:495-524) vs trajectories of the unmodified reference (oracle/make_golden_nn.py), float64.

Tolerance: these are box-constrained solves, so the comparison is at pnqp's own accuracy - the reference stops its
batched QP when the slowest element has |dx| < 1e-4 while the kernels stop per problem (INTEGRATION.md section 2);
SURVEY.md section 8(c) policy: x, u to 2e-4, costs (second order in that difference) to 1e-5 relative, and the set
of controls sitting on a bound exactly."""
TOL_XU, TOL_COST = 2e-4, 1e-5
import pytest
import torch

from tests.helpers import build_net, load_golden, maxdiff

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def solve(g, dx, bound):
    from mpc.pytorch_b200 import MPC, QuadCost, GradMethods
    T = g["C"].shape[0]
    kw = {} if bound is None else dict(u_lower=-bound, u_upper=bound)
    ctrl = MPC(3, 2, T, **kw, lqr_iter=12, verbose=-1, grad_method=GradMethods.ANALYTIC,
               exit_unconverged=False, detach_unconverged=False, eps=1e-6)
    return ctrl(g["x_init"].to(DEV), QuadCost(g["C"].to(DEV), g["c"].to(DEV)), dx)


@pytest.mark.parametrize("act", ["sigmoid", "relu"])
def test_mpc_nn_dynamics_analytic_matches_reference(act):
    g = load_golden(f"nn_dynamics_{act}_f64")
    x, u, costs = solve(g, build_net(g, act).to(DEV), 0.6)
    sc = max(1.0, float(g["x"].abs().max()))
    assert maxdiff(u, g["u"]) < TOL_XU and maxdiff(x, g["x"]) < TOL_XU * sc
    assert maxdiff(costs, g["costs"]) < TOL_COST * max(1.0, float(g["costs"].abs().max()))
    assert torch.equal(u.abs().cpu() == 0.6, g["u"].abs() == 0.6)        # same controls on the bounds


@pytest.mark.parametrize("act", ["sigmoid", "relu"])
def test_mpc_nn_dynamics_unbounded_matches_reference_tightly(act):
    """No bounds, so no QP stopping tolerance: 12 iLQR iterations through the network agree to round-off."""
    g = load_golden(f"nn_dynamics_{act}_f64")
    x, u, costs = solve(g, build_net(g, act).to(DEV), None)
    sc = max(1.0, float(g["x_free"].abs().max()))
    assert maxdiff(u, g["u_free"]) < 1e-7 * sc and maxdiff(x, g["x_free"]) < 1e-7 * sc
    assert maxdiff(costs, g["costs_free"]) < 1e-9 * max(1.0, float(g["costs_free"].abs().max()))


def test_mpc_affine_dynamics_analytic_matches_reference():
    from mpc.dynamics import AffineDynamics
    g = load_golden("affine_dynamics_f64")
    dx = AffineDynamics(g["A"].to(DEV), g["B"].to(DEV), g["c0"].to(DEV))
    x, u, costs = solve(g, dx, 0.5)
    assert maxdiff(u, g["u"]) < TOL_XU and maxdiff(x, g["x"]) < TOL_XU * max(1.0, float(g["x"].abs().max()))
    assert maxdiff(costs, g["costs"]) < TOL_COST * max(1.0, float(g["costs"].abs().max()))
    assert torch.equal(u.abs().cpu() == 0.5, g["u"].abs() == 0.5)


def test_nn_dynamics_gradient_flows_to_the_weights():
    """d loss / d weights through the controller (the reference's imitation-learning use, README): the final
    differentiable LQR step sees F, f built from grad_input under autograd."""
    from mpc.pytorch_b200 import MPC, QuadCost, GradMethods
    g = load_golden("nn_dynamics_sigmoid_f64")
    net = build_net(g, "sigmoid").to(DEV)
    T = g["C"].shape[0]
    ctrl = MPC(3, 2, T, lqr_iter=12, verbose=-1, grad_method=GradMethods.ANALYTIC, exit_unconverged=False,
               detach_unconverged=False, eps=1e-6)
    x, u, _ = ctrl(g["x_init"].to(DEV), QuadCost(g["C"].to(DEV), g["c"].to(DEV)), net)
    u.pow(2).sum().backward()
    gw = net.fcs[0].weight.grad
    assert gw is not None and bool(torch.isfinite(gw).all()) and float(gw.abs().max()) > 0


def _nn_grad_setup(name):
    from mpc.dynamics import NNDynamics
    g = load_golden(name)
    nl = int(g["n_layers"])
    net = NNDynamics(2, 2, hidden_sizes=[g[f"W{i}"].shape[0] for i in range(nl - 1)], activation="sigmoid").double()
    with torch.no_grad():
        for i, fc in enumerate(net.fcs):
            fc.weight.copy_(g[f"W{i}"])
            fc.bias.copy_(g[f"b{i}"])
    return g, net.to(DEV)


def _nn_solve(g, net, c, slew, lqr_iter=40):
    from mpc.pytorch_b200 import MPC, QuadCost, GradMethods
    T = g["C"].shape[0]
    ctrl = MPC(2, 2, T, u_lower=-1.0, u_upper=1.0, lqr_iter=lqr_iter, verbose=-1, exit_unconverged=False,
               max_linesearch_iter=1, slew_rate_penalty=slew, grad_method=GradMethods.ANALYTIC)
    return ctrl(g["x_init"].to(DEV), QuadCost(g["C"].to(DEV), c), net)


@pytest.mark.parametrize("name,slew", [("nn_grad_f64", None), ("nn_grad_slew_f64", 1.0)])
def test_nn_dynamics_solution_gradients_match_reference_autograd(name, slew):
    """The reference's test_lqr_backward_cost_nn_dynamics_module_constrained[_slew] (tests/test_mpc.py:560-744):
    d u* / d c and d u* / d (first-layer bias) of a partially active iLQR solution through a learned model.
    Compared with the reference's own autograd Jacobians (fixture) and with central differences of this solver."""
    g, net = _nn_grad_setup(name)
    c = g["c"].to(DEV).requires_grad_(True)
    x, u, _ = _nn_solve(g, net, c, slew)
    assert maxdiff(u, g["u"]) < 2e-4 and maxdiff(x, g["x"]) < 2e-4 * max(1.0, float(g["x"].abs().max()))
    uf = u.reshape(-1)
    on = uf.abs() == 1.0
    assert torch.equal(on.cpu(), g["u"].reshape(-1).abs() == 1.0) and bool(on.any()) and bool((~on).any())
    rows_c, rows_b = [], []
    for i in range(uf.numel()):
        gc, gb = torch.autograd.grad(uf[i], [c, net.fcs[0].bias], retain_graph=True)
        rows_c.append(gc.reshape(-1))
        rows_b.append(gb.reshape(-1))
    Jc, Jb = torch.stack(rows_c), torch.stack(rows_b)
    sc_c, sc_b = float(g["du_dc"].abs().max()), float(g["du_db0"].abs().max())
    assert maxdiff(Jc, g["du_dc"]) < 2e-3 * sc_c, (maxdiff(Jc, g["du_dc"]), sc_c)
    assert maxdiff(Jb, g["du_db0"]) < 2e-3 * sc_b, (maxdiff(Jb, g["du_db0"]), sc_b)
    # central differences of the solver itself on a few coordinates (the reference uses numdifftools, atol 1e-3).
    # The box QPs inside stop at |dx| < 1e-4, so u* carries ~1e-6..1e-5 of solver noise: the step must be large
    # enough for that noise / 2h to stay below the tolerance (h = 1e-4 gave 1.8e-2 of pure noise on one entry).
    h = 1e-2
    with torch.no_grad():
        for j in (0, 5, 11):
            e = torch.zeros_like(c).reshape(-1)
            e[j] = h
            e = e.reshape(c.shape)
            up = _nn_solve(g, net, c.detach() + e, slew)[1].reshape(-1)
            um = _nn_solve(g, net, c.detach() - e, slew)[1].reshape(-1)
            assert float(((up - um) / (2 * h) - Jc[:, j]).abs().max()) < 2e-3
        b0 = net.fcs[0].bias
        for j in (0, 7):
            keep = b0[j].item()
            b0[j] = keep + h
            up = _nn_solve(g, net, c.detach(), slew)[1].reshape(-1)
            b0[j] = keep - h
            um = _nn_solve(g, net, c.detach(), slew)[1].reshape(-1)
            b0[j] = keep
            assert float(((up - um) / (2 * h) - Jb[:, j]).abs().max()) < 2e-3
