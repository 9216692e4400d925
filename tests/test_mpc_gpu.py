"""GPU: the MPC module (outer iLQR loop, reference mpc/mpc.py:184-337) on top of the CUDA step."""
import contextlib
import io

import pytest
import torch

from tests.helpers import condensed_box_lqr_scipy, gen_problem, load_golden, maxdiff

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def test_tvlqr_notebook_example_reproduces_recorded_trace():
    """examples/Time Varying Linear-Quadratic Control.ipynb:26-36 - printed mean(cost) per iteration."""
    from mpc import mpc
    g = load_golden("tvlqr_notebook_f32")
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        x, u, costs = mpc.MPC(n_state=3, n_ctrl=4, T=5, u_lower=g["u_lower"].to(DEV),
                              u_upper=g["u_upper"].to(DEV), lqr_iter=20, verbose=1, backprop=False,
                              exit_unconverged=False)(
            g["x_init"].to(DEV), mpc.QuadCost(g["C"].to(DEV), g["c"].to(DEV)), mpc.LinDx(g["F"].to(DEV)))
    rows = [l for l in buf.getvalue().splitlines() if l.startswith("|") and "iter" not in l]
    mean_costs = [float(r.split("|")[2]) for r in rows]
    for got, want in zip(mean_costs, g["notebook_mean_costs"].tolist()):
        assert abs(got - want) < 5e-4
    assert "Initial mean(cost): 3.9041e+01" in buf.getvalue()
    assert maxdiff(x, g["x"]) < 5e-4 and maxdiff(u, g["u"]) < 5e-4 and maxdiff(costs, g["costs"]) < 5e-4
    # ||full_du||_max column is the reference's batch-mixing norm: first row 1.94e+00 in the notebook
    assert abs(float(rows[0].split("|")[3]) - 1.94) < 0.02


def test_shape_expansion_and_unbounded_lti():
    """2-D C / 1-D c expansion (reference mpc.py:205-226) and agreement with explicit tensors."""
    from mpc import mpc
    B, T, n, m = 5, 6, 4, 2
    C, c, F, f, x0 = [t.to(DEV) for t in gen_problem(60, B, T, n, m, torch.float64)]
    C2, c1 = C[0, 0].clone(), c[0, 0].clone()
    kw = dict(lqr_iter=3, verbose=-1, exit_unconverged=False, n_batch=B)
    a = mpc.MPC(n, m, T, **kw)(x0, mpc.QuadCost(C2, c1), mpc.LinDx(F, f))
    Cf = C2.expand(T, B, n + m, n + m).contiguous()
    cf = c1.expand(T, B, n + m).contiguous()
    b = mpc.MPC(n, m, T, **kw)(x0, mpc.QuadCost(Cf, cf), mpc.LinDx(F, f))
    for s, t in zip(a, b):
        assert maxdiff(s, t) < 1e-12
    with pytest.raises(SystemExit):
        mpc.MPC(n, m, T, verbose=-1)(x0, mpc.QuadCost(C2, c1), mpc.LinDx(F, f))   # batch not inferable


def test_delta_u_trust_region():
    """reference tests/test_mpc.py:197-240: one iteration with delta_u keeps |u| <= delta_u."""
    from mpc import mpc
    B, T, n, m = 2, 5, 3, 4
    C, c, F, f, x0 = [t.to(DEV) for t in gen_problem(61, B, T, n, m, torch.float64, True)]
    ul = -torch.rand(T, B, m, dtype=torch.float64, device=DEV)
    uu = torch.rand(T, B, m, dtype=torch.float64, device=DEV)
    x, u, _ = mpc.MPC(n, m, T, u_lower=ul, u_upper=uu, lqr_iter=1, delta_u=0.1, verbose=-1,
                      exit_unconverged=False)(x0, mpc.QuadCost(C, c), mpc.LinDx(F, f))
    assert float(u.abs().max()) <= 0.1 + 1e-12


def test_unconverged_handling():
    from mpc import mpc
    B, T, n, m = 3, 5, 3, 2
    C, c, F, f, x0 = [t.to(DEV) for t in gen_problem(62, B, T, n, m, torch.float64)]
    with pytest.raises(AssertionError):                       # exit_unconverged default (mpc.py:322-324)
        mpc.MPC(n, m, T, u_lower=-0.01, u_upper=0.01, lqr_iter=1, eps=1e-30, verbose=-1)(
            x0, mpc.QuadCost(C, c), mpc.LinDx(F, f))
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        x, u, _ = mpc.MPC(n, m, T, u_lower=-0.01, u_upper=0.01, lqr_iter=1, eps=1e-30, verbose=0,
                          exit_unconverged=False)(x0.requires_grad_(True), mpc.QuadCost(C, c), mpc.LinDx(F, f))
    assert "did not converge" in buf.getvalue()
    assert not u.requires_grad or float(torch.autograd.grad(u.sum(), x0, allow_unused=True)[0].abs().max()) == 0


def test_slew_rate_penalty():
    """reference tests/test_mpc.py:802-861: tiny penalty recovers the plain solution, large one smooths u."""
    from mpc import mpc
    B, T, n, m = 2, 8, 3, 2
    C, c, F, f, x0 = [t.to(DEV) for t in gen_problem(63, B, T, n, m, torch.float32)]
    kw = dict(u_lower=-1.0, u_upper=1.0, lqr_iter=20, verbose=-1, exit_unconverged=False)
    x0_, u0_, _ = mpc.MPC(n, m, T, **kw)(x0, mpc.QuadCost(C, c), mpc.LinDx(F, f))
    x1_, u1_, _ = mpc.MPC(n, m, T, slew_rate_penalty=1e-6, **kw)(x0, mpc.QuadCost(C, c), mpc.LinDx(F, f))
    x2_, u2_, _ = mpc.MPC(n, m, T, slew_rate_penalty=1.0, **kw)(x0, mpc.QuadCost(C, c), mpc.LinDx(F, f))
    assert maxdiff(u0_, u1_) < 1e-3 and maxdiff(x0_, x1_) < 1e-3
    rough = lambda u: float((u[1:] - u[:-1]).pow(2).sum())
    assert rough(u2_) < rough(u0_)


@pytest.mark.parametrize("name", ["slew_box_f64", "slew_unb_f64"])
def test_slew_rate_matches_reference_fixture(name):
    """The slew-rate augmentation (state = [u_{t-1}; x], reference mpc/mpc.py:362-445) against trajectories the
    unmodified reference produced for the same inputs (oracle/make_golden.py), float64."""
    from mpc import mpc
    g = load_golden(name)
    T, B, p = g["C"].shape[0], g["C"].shape[1], g["C"].shape[2]
    n = g["x_init"].shape[1]
    m = p - n
    bound = g.get("bound")
    kw = {} if bound is None else dict(u_lower=-float(bound), u_upper=float(bound))
    prev = g["prev_ctrl"].to(DEV) if "prev_ctrl" in g else None
    A, Bm = g["A"].to(DEV), g["Bm"].to(DEV)

    class AffineDx(torch.nn.Module):        # the reference's slew branch needs Module dynamics (mpc/mpc.py:411-414)
        def forward(self, xx, uu):
            return xx @ A.t() + uu @ Bm.t()

    x, u, costs = mpc.MPC(n, m, T, lqr_iter=15, verbose=-1, exit_unconverged=False, detach_unconverged=False,
                          slew_rate_penalty=float(g["penalty"]), prev_ctrl=prev, eps=1e-9,
                          grad_method=mpc.GradMethods.AUTO_DIFF, **kw)(
        g["x_init"].to(DEV), mpc.QuadCost(g["C"].to(DEV), g["c"].to(DEV)), AffineDx())
    tol = 2e-4 if bound is not None else 1e-8          # bounded: pnqp step tolerance (batch-coupled reference)
    assert maxdiff(u, g["u"]) < tol and maxdiff(x, g["x"]) < tol
    assert maxdiff(costs, g["costs"]) < 10 * tol * max(1.0, float(g["costs"].abs().max()))


def test_cartpole_ilqr_matches_reference_fixture():
    """BASELINE config 2 recipe (small): nonlinear Module dynamics, AUTO_DIFF linearisation, bounds +-100,
    decay .5, 2 line-search iterations, eps 1e-2 - against the reference's stored trajectory."""
    from mpc import mpc
    from tests.cartpole import Cartpole
    g = load_golden("cartpole_auto_diff_f32")
    T, B = g["Q"].shape[0], g["Q"].shape[1]
    dx = Cartpole()
    x, u, costs = mpc.MPC(5, 1, T, u_lower=-100.0, u_upper=100.0, lqr_iter=8, verbose=-1,
                          exit_unconverged=False, detach_unconverged=False, linesearch_decay=0.5,
                          max_linesearch_iter=2, grad_method=mpc.GradMethods.AUTO_DIFF, eps=1e-2)(
        g["x_init"].to(DEV), mpc.QuadCost(g["Q"].to(DEV), g["p"].to(DEV)), dx)
    # fp32 iLQR over 8 nonlinear iterations: compare costs tightly, trajectories loosely
    rel = (costs.cpu() - g["costs"]).abs() / g["costs"].abs().clamp_min(1.0)
    assert float(rel.max()) < 2e-3
    assert maxdiff(x, g["x"]) < 5e-2 * max(1.0, float(g["x"].abs().max()))


def test_analytic_and_finite_diff_linearisation_agree():
    """reference tests/test_mpc.py:747-799 (atol 1e-4 between linearisation methods), float64."""
    from mpc import mpc
    from tests.cartpole import Cartpole, initial_states

    class CartpoleAnalytic(Cartpole):
        def grad_input(self, x, u):
            xg, ug = x.detach().requires_grad_(True), u.detach().requires_grad_(True)
            with torch.enable_grad():
                y = self.forward(xg, ug)
                rows = [torch.autograd.grad(y[:, j].sum(), [xg, ug], retain_graph=True) for j in range(5)]
            return torch.stack([r[0] for r in rows], 1), torch.stack([r[1] for r in rows], 1)

    T, B = 6, 4
    x0 = initial_states(B, 3, torch.float64).to(DEV)
    u = 0.5 * torch.randn(T, B, 1, dtype=torch.float64, device=DEV)
    from mpc.pytorch_b200.solver import get_traj
    dx = CartpoleAnalytic()
    x = get_traj(T, u, x0, dx)
    outs = []
    for gm in (mpc.GradMethods.ANALYTIC, mpc.GradMethods.AUTO_DIFF, mpc.GradMethods.FINITE_DIFF):
        outs.append(mpc.MPC(5, 1, T, grad_method=gm).linearize_dynamics(x, u, dx, diff=False))
    for F2, f2 in outs[1:]:
        assert maxdiff(F2, outs[0][0]) < 1e-4 and maxdiff(f2, outs[0][1]) < 1e-4


@pytest.mark.parametrize("shape", [(9, 7, 8, 2, torch.float32, True), (5, 6, 3, 4, torch.float64, False),
                                   (4, 5, 6, 1, torch.float64, True), (3, 1, 4, 2, torch.float32, True)])
def test_rollout_kernel_matches_reference_get_traj(shape):
    """mpcb200_rollout (get_traj for LinDx, reference mpc/util.py:102-126) vs the torch recurrence."""
    from mpc.pytorch_b200.step import rollout_raw
    B, T, n, m, dtype, with_f = shape
    C, c, F, f, x0 = [v.to(DEV) if v is not None else None for v in gen_problem(70, B, T, n, m, dtype, True, with_f)]
    u = torch.randn(T, B, m, dtype=dtype, device=DEV)
    if T == 1:
        F = torch.zeros(0, B, n, n + m, dtype=dtype, device=DEV)
        f = None
    got = rollout_raw(n, m, T, x0, u, F, f)
    xs = [x0]
    for k in range(T - 1):
        nx = torch.einsum("bij,bj->bi", F[k], torch.cat((xs[k], u[k]), 1))
        xs.append(nx + f[k] if f is not None else nx)
    want = torch.stack(xs)
    assert got.shape == want.shape
    assert maxdiff(got, want) <= (1e-12 if dtype == torch.float64 else 2e-5) * max(1.0, float(want.abs().max()))


@pytest.mark.parametrize("bound", [None, 0.35])
def test_mpc_solution_is_the_box_qp_optimum(bound):
    """reference tests/test_mpc.py:91-194: the iLQR fixed point computed on the GPU equals the optimum of the
    box-constrained problem found by an independent solver (scipy L-BFGS-B on the condensed problem)."""
    from mpc import mpc
    B, T, n, m = 2, 5, 3, 2
    C, c, F, f, x0 = gen_problem(41, B, T, n, m, torch.float64, time_varying=True)
    lo, hi = (-1e4, 1e4) if bound is None else (-bound, bound)
    kw = {} if bound is None else dict(u_lower=lo, u_upper=hi)
    x, u, _ = mpc.MPC(n, m, T, lqr_iter=30, eps=1e-10, verbose=-1, exit_unconverged=False, **kw)(
        x0.to(DEV), mpc.QuadCost(C.to(DEV), c.to(DEV)), mpc.LinDx(F.to(DEV), f.to(DEV)))
    for b in range(B):
        xs, us = condensed_box_lqr_scipy(C[:, b], c[:, b], F[:, b], f[:, b], x0[b], lo, hi)
        assert maxdiff(u[:, b], us) < 2e-4 and maxdiff(x[:, b], xs) < 2e-4


def test_module_cost_equal_to_a_quadratic_reproduces_quadcost():
    """A cost given as an nn.Module (reference mpc/mpc.py:258-262 `approximate_cost`, lqr_step.py:233-234 true_cost in
    the line search) that happens to be the quadratic 1/2 tau' C tau + c' tau must give the QuadCost solution: the
    second-order expansion is exact and the split-mode rollout evaluates the same numbers (float64)."""
    from mpc.pytorch_b200 import MPC, QuadCost, LinDx
    B, T, n, m = 6, 7, 4, 2
    dt = torch.float64
    Ct, ct, F, f, x0 = gen_problem(77, B, T, n, m, dt, False, True)
    C0, c0 = Ct[0, 0].to(DEV), ct[0, 0].to(DEV)                  # one (C, c) for every t and problem

    class Quad(torch.nn.Module):
        def forward(self, tau):
            return 0.5 * (tau * (tau @ C0.t())).sum(-1) + tau @ c0

    C = C0.expand(T, B, n + m, n + m).contiguous()
    c = c0.expand(T, B, n + m).contiguous()
    kw = dict(u_lower=-0.3, u_upper=0.3, lqr_iter=6, verbose=-1, exit_unconverged=False, detach_unconverged=False)
    dx = LinDx(F.to(DEV), f.to(DEV))
    xa, ua, ca = MPC(n, m, T, **kw)(x0.to(DEV), QuadCost(C, c), dx)
    xb, ub, cb = MPC(n, m, T, n_batch=B, **kw)(x0.to(DEV), Quad(), dx)   # batch size cannot be inferred from a Module (reference :198-199)
    assert maxdiff(ua, ub) < 1e-8 and maxdiff(xa, xb) < 1e-8 * max(1.0, float(xa.abs().max()))
    assert maxdiff(ca, cb) < 1e-9 * max(1.0, float(ca.abs().max()))
