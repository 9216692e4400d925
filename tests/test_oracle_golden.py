"""CPU: the oracle (oracle/lqr_oracle.py) against the fixtures generated from the REAL reference
(oracle/make_golden.py).  These pin the oracle; the GPU tests then compare CUDA with the oracle."""
import glob
import os

import pytest
import torch

from oracle import lqr_oracle as orc
from tests.helpers import GOLD, condensed_box_lqr_scipy, gen_problem, load_golden, maxdiff, nominal_controls


def _names(prefix):
    return sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLD, prefix + "*.npz")))


@pytest.mark.parametrize("name", _names("pnqp_"))
def test_pnqp_matches_reference(name):
    g = load_golden(name)
    x, _, If, it = orc.pnqp(g["H"], g["q"], g["lower"], g["upper"], x_init=g.get("x_init"),
                            n_iter=20, coupled=True)
    tol = 1e-12 if g["H"].dtype == torch.float64 else 1e-6
    assert maxdiff(x, g["x"]) <= tol
    assert torch.equal(If.bool(), g["If"].bool())          # active set: bit exact
    assert int(it.max()) == int(g["n_iter"])


@pytest.mark.parametrize("name", _names("pnqp_f64"))
def test_pnqp_solves_the_box_qp(name):
    """KKT check in float64 (stands in for the reference's cvxpy oracle, tests/test_mpc.py:65-88)."""
    g = load_golden(name)
    H, q, lo, hi = g["H"], g["q"], g["lower"], g["upper"]
    x, _, _, _ = orc.pnqp(H, q, lo, hi, x_init=g.get("x_init"), n_iter=20, coupled=False)
    grad = torch.einsum("bij,bj->bi", H, x) + q
    assert bool(((x >= lo - 1e-12) & (x <= hi + 1e-12)).all())
    interior = (x > lo + 1e-9) & (x < hi - 1e-9)
    assert float(grad[interior].abs().max()) < 2e-3        # pnqp stops at |dx| < 1e-4
    assert bool((grad[x <= lo + 1e-12] > -2e-3).all())
    assert bool((grad[x >= hi - 1e-12] < 2e-3).all())


def _bounds(g):
    ul, uu = g.get("u_lower"), g.get("u_upper")
    return ul, uu


@pytest.mark.parametrize("name", _names("step_"))
def test_step_forward_matches_reference(name):
    g = load_golden(name)
    T, B, p = g["C"].shape[0], g["C"].shape[1], g["C"].shape[2]
    n = g["x_init"].shape[1]
    m = p - n
    ul, uu = _bounds(g)
    o = orc.lqr_step_forward(n, m, T, g["x_init"], g["C"], g["c"], g["F"], g.get("f"), g["cur_x"],
                             g["cur_u"], u_lower=ul, u_upper=uu, delta_u=g.get("delta_u"), coupled=True)
    f64 = g["C"].dtype == torch.float64
    tol = 1e-10 if f64 else 2e-5
    assert maxdiff(o.new_x, g["new_x"]) <= tol
    assert maxdiff(o.new_u, g["new_u"]) <= tol
    assert maxdiff(o.costs, g["costs"]) <= 50 * tol
    assert maxdiff(o.full_du_norm, g["full_du_norm"]) <= 10 * tol
    assert maxdiff(o.mean_alphas, g["mean_alphas"]) <= 1e-12
    if f64:
        assert float(o.n_total_qp_iter) == float(g["n_total_qp_iter"])
    if ul is not None:                                       # clamp masks: exact
        lo = ul if torch.is_tensor(ul) else torch.full_like(o.new_u, ul)
        assert torch.equal(o.new_u == lo.to(o.new_u.dtype), g["new_u"] == lo.to(o.new_u.dtype))


@pytest.mark.parametrize("name", _names("grad_"))
def test_adjoint_matches_reference_autograd(name):
    g = load_golden(name)
    T, B, p = g["C"].shape[0], g["C"].shape[1], g["C"].shape[2]
    n = g["x_init"].shape[1]
    m = p - n
    b = g.get("bound")
    ul, uu = (None, None) if b is None else (-b, b)
    x, u, costs, _ = orc.mpc_forward_lin(n, m, T, g["x_init"], g["C"], g["c"], g["F"], g["f"],
                                         u_lower=ul, u_upper=uu, lqr_iter=int(g["lqr_iter"]),
                                         eps=1e-9, coupled=True)
    assert maxdiff(x, g["x"]) <= 1e-9 and maxdiff(u, g["u"]) <= 1e-9
    out = orc.lqr_step_backward(n, m, T, g["x_init"], g["C"], g["c"], g["F"], g["f"], g["x"], g["u"],
                                g["wx"], g["wu"], u_lower=ul, u_upper=uu, coupled=True)
    for got, key in zip(out[:5], ("dx_init", "dC", "dc", "dF", "df")):
        assert maxdiff(got, g[key]) <= 1e-9, key


def test_tvlqr_notebook_trace():
    """examples/Time Varying Linear-Quadratic Control.ipynb:26-36 (the reference's only recorded output)."""
    g = load_golden("tvlqr_notebook_f32")
    trace = []
    x, u, costs, _ = orc.mpc_forward_lin(3, 4, 5, g["x_init"], g["C"], g["c"], g["F"], None,
                                         u_lower=g["u_lower"], u_upper=g["u_upper"], lqr_iter=20,
                                         coupled=True, trace=trace)
    for got, want in zip([t["mean_cost"] for t in trace], g["notebook_mean_costs"].tolist()):
        assert abs(got - want) < 5e-4
    assert maxdiff(x, g["x"]) < 5e-4 and maxdiff(u, g["u"]) < 5e-4


@pytest.mark.parametrize("bounds", [0.25, "tensor"])
def test_uncoupled_pnqp_is_the_single_problem_reference(bounds):
    """coupled=False must equal running the (reference-pinned) coupled code one problem at a time."""
    B, T, n, m = 6, 7, 4, 2
    C, c, F, f, x0 = gen_problem(31, B, T, n, m, torch.float64)
    u, ul, uu = nominal_controls(31, B, T, m, torch.float64, bounds)
    x = orc.get_traj(T, u, x0, F, f)
    o = orc.lqr_step_forward(n, m, T, x0, C, c, F, f, x, u, u_lower=ul, u_upper=uu, coupled=False)
    for b in range(B):
        sl = lambda t: t[:, b:b + 1].contiguous()
        lb = ul if not torch.is_tensor(ul) else sl(ul)
        ub = uu if not torch.is_tensor(uu) else sl(uu)
        ob = orc.lqr_step_forward(n, m, T, x0[b:b + 1], sl(C), sl(c), sl(F), sl(f), sl(x), sl(u),
                                  u_lower=lb, u_upper=ub, coupled=True)
        assert maxdiff(o.new_u[:, b], ob.new_u[:, 0]) < 1e-12
        assert torch.equal(o.free_masks[:, b], ob.free_masks[:, 0])
        assert torch.equal(o.qp_iters[:, b], ob.qp_iters[:, 0])


def test_unbounded_lqr_solves_the_kkt_system():
    """Dense KKT solve in float64 (stands in for cvxpy lqr_cp, reference tests/test_mpc.py:35-62)."""
    B, T, n, m = 2, 5, 3, 2
    p = n + m
    C, c, F, f, x0 = gen_problem(5, B, T, n, m, torch.float64, time_varying=True)
    u = torch.zeros(T, B, m, dtype=torch.float64)
    x = orc.get_traj(T, u, x0, F, f)
    o = orc.lqr_step_forward(n, m, T, x0, C, c, F, f, x, u)
    for b in range(B):
        # variables tau_0..tau_{T-1}; constraints x_0 = x_init, x_{t+1} = F_t tau_t + f_t
        nv, nc = T * p, T * n
        Hm = torch.zeros(nv, nv, dtype=torch.float64)
        g = torch.zeros(nv, dtype=torch.float64)
        A = torch.zeros(nc, nv, dtype=torch.float64)
        rhs = torch.zeros(nc, dtype=torch.float64)
        for t in range(T):
            Hm[t * p:(t + 1) * p, t * p:(t + 1) * p] = C[t, b]
            g[t * p:(t + 1) * p] = c[t, b]
        A[:n, :n] = torch.eye(n, dtype=torch.float64)
        rhs[:n] = x0[b]
        for t in range(T - 1):
            r0 = (t + 1) * n
            A[r0:r0 + n, (t + 1) * p:(t + 1) * p + n] = torch.eye(n, dtype=torch.float64)
            A[r0:r0 + n, t * p:(t + 1) * p] = -F[t, b]
            rhs[r0:r0 + n] = f[t, b]
        KKT = torch.cat((torch.cat((Hm, A.T), 1), torch.cat((A, torch.zeros(nc, nc, dtype=torch.float64)), 1)), 0)
        sol = torch.linalg.solve(KKT, torch.cat((-g, rhs)))
        tau = sol[:nv].view(T, p)
        assert maxdiff(tau[:, :n], o.new_x[:, b]) < 1e-9
        assert maxdiff(tau[:, n:], o.new_u[:, b]) < 1e-9


@pytest.mark.parametrize("bound", [None, 0.35])
def test_ilqr_fixed_point_is_the_box_qp_optimum(bound):
    """reference tests/test_mpc.py:91-194 (LQR / box-LQR vs an independent convex solver, rtol 1e-3)."""
    B, T, n, m = 2, 5, 3, 2
    C, c, F, f, x0 = gen_problem(41, B, T, n, m, torch.float64, time_varying=True)
    lo, hi = (-1e4, 1e4) if bound is None else (-bound, bound)
    x, u, costs, fdn = orc.mpc_forward_lin(n, m, T, x0, C, c, F, f, u_lower=None if bound is None else lo,
                                           u_upper=None if bound is None else hi, lqr_iter=30, eps=1e-10)
    for b in range(B):
        xs, us = condensed_box_lqr_scipy(C[:, b], c[:, b], F[:, b], f[:, b], x0[b], lo, hi)
        assert maxdiff(u[:, b], us) < 2e-4 and maxdiff(x[:, b], xs) < 2e-4
    if bound is not None:
        assert 0.05 < float(((u.abs() - bound).abs() < 1e-9).double().mean()) < 0.95
