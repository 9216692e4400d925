"""GPU parity at the BASELINE.json configuration sizes (every problem compared, nothing masked out).

  config 3  B=4096, T=20, n=8, m=2  fp32, unbounded and +-0.25            vs the per-problem oracle
  config 4  B=1024, T=20, n=8, m=2  fp32, scalar AND tensor bounds        vs the per-problem oracle
  config 5  B=4096 (the 8-GPU shard of 32768), T=50, n=16, m=4 fp32        properties on all + sampled oracle
  adjoint   config-3 size, LQRStepFn.backward                               vs orc.lqr_step_backward
  config 2  cartpole iLQR, B=128, T=25 (float64 and float32)              vs fixtures of the reference

Tolerances (SURVEY.md section 8c): fp32 unbounded 4e-5 x scale on x,u; fp32 bounded 2e-4 (pnqp stops at
|dx| < 1e-4); pnqp free sets `If`, clamp masks and iteration counts bit exact - including the handful of fp32
QPs that never satisfy |dx| < 1e-4 (the reference prints "Did not converge" for them too).
"""
import pytest
import torch

from oracle import lqr_oracle as orc
from tests.gpu_harness import DEV, run_step, to_dev
from tests.helpers import gen_problem, load_golden, maxdiff

pytestmark = pytest.mark.gpu


def _check_all(r, o, u, ul, uu, tol, bounded):
    scale = max(1.0, float(o.new_x.abs().max()))
    assert maxdiff(r["new_x"], o.new_x) <= tol * scale
    assert maxdiff(r["new_u"], o.new_u) <= tol * scale
    assert maxdiff(r["costs"], o.costs) <= 3e-4 * max(1.0, float(o.costs.abs().max()))
    assert maxdiff(r["alphas"], o.alphas) == 0.0
    if bounded:
        # every problem, every time step: free set, iteration count and which controls sit on a bound
        assert torch.equal(r["free_mask"].bool(), o.free_masks)
        # iteration counts: identical except where the stopping test |dx| < 1e-4 is decided by fp32 round-off
        # (LDL^T on the GPU, LU in the oracle); those must stay a vanishing fraction and the iterates they
        # return are still compared above / below at the 2e-4 tolerance
        dq = r["qp_iters"].long() - o.qp_iters
        nbad = int((dq != 0).sum())
        assert nbad <= 2e-3 * dq.numel(), (nbad, dq.numel(), int(dq.abs().max()))
        lo = ul if torch.is_tensor(ul) else torch.full_like(u, ul)
        hi = uu if torch.is_tensor(uu) else torch.full_like(u, uu)
        assert torch.equal(r["new_u"] == lo, o.new_u == lo)
        assert torch.equal(r["new_u"] == hi, o.new_u == hi)
        assert bool(((r["new_u"] >= lo) & (r["new_u"] <= hi)).all())
        # the status word flags only problems with a QP at the iteration cap, and only problems the reference
        # itself leaves at the cap on the same inputs (it prints "pnqp warning: Did not converge" for them), up
        # to the iteration counts that fp32 round-off decides differently (nbad above)
        capped = (r["qp_iters"] == 19).any(0)
        flagged = (r["status"] & 1) != 0
        ref_capped = (o.qp_iters == 19).any(0)
        assert bool((flagged <= capped).all())
        assert int((flagged & ~ref_capped).sum()) <= nbad, (int(flagged.sum()), int(ref_capped.sum()), nbad)
    assert int((r["status"] & ~1).max()) == 0


@pytest.mark.parametrize("bounds", [None, 0.25], ids=["unbounded", "box"])
def test_config3_all_problems_vs_oracle(bounds):
    B, T, n, m = 4096, 20, 8, 2
    C, c, F, f, x0 = gen_problem(3000, B, T, n, m, torch.float32)
    u = torch.zeros(T, B, m)
    x = orc.get_traj(T, u, x0, F, f)
    kw = {} if bounds is None else dict(u_lower=-bounds, u_upper=bounds)
    o = orc.lqr_step_forward(n, m, T, x0, C, c, F, f, x, u, coupled=False, **kw)
    r, _ = run_step(n, m, T, dict(x0=x0, C=C, c=c, F=F, f=f, x=x, u=u), kw, want_gains=False)
    _check_all(r, o, u, kw.get("u_lower"), kw.get("u_upper"), 2e-4 if bounds else 4e-5, bounds is not None)
    if bounds is not None:
        assert 0.5 < float((r["new_u"].abs() == bounds).float().mean()) < 0.95


@pytest.mark.parametrize("kind", ["scalar", "tensor"])
def test_config4_all_problems_vs_oracle(kind):
    B, T, n, m = 1024, 20, 8, 2
    C, c, F, f, x0 = gen_problem(4000, B, T, n, m, torch.float32)
    if kind == "scalar":
        u, ul, uu = torch.zeros(T, B, m), -0.25, 0.25
    else:
        g = torch.Generator().manual_seed(4001)
        ul = -0.5 * torch.rand(T, B, m, generator=g)
        uu = 0.5 * torch.rand(T, B, m, generator=g)
        u = torch.zeros(T, B, m)
    x = orc.get_traj(T, u, x0, F, f)
    o = orc.lqr_step_forward(n, m, T, x0, C, c, F, f, x, u, u_lower=ul, u_upper=uu, coupled=False)
    r, _ = run_step(n, m, T, dict(x0=x0, C=C, c=c, F=F, f=f, x=x, u=u), dict(u_lower=ul, u_upper=uu),
                    want_gains=False)
    _check_all(r, o, u, ul, uu, 2e-4, True)


def test_config5_shard_properties_and_sampled_oracle():
    """B=4096 is the per-GPU shard of BASELINE config 5 at 8 GPUs (32768 / 8)."""
    from mpc.pytorch_b200.step import lqr_step_raw
    B, T, n, m = 4096, 50, 16, 4
    C, c, F, f, x0 = [to_dev(t) for t in gen_problem(5000, B, T, n, m, torch.float32)]
    u = torch.zeros(T, B, m, device=DEV)
    from mpc.pytorch_b200.solver import get_traj, LinDx
    x = get_traj(T, u, x0, LinDx(F, f))
    o = lqr_step_raw(n, m, T, x0, C, c, F, f, x, u)
    nx, nu = o["new_x"], o["new_u"]
    assert int(o["status"].max()) == 0 and bool(torch.isfinite(o["costs"]).all())
    tau = torch.cat((nx, nu), 2)
    pred = torch.einsum("tbij,tbj->tbi", F, tau[:-1]) + f
    assert float((pred - nx[1:]).abs().max()) < 4e-5 * max(1.0, float(nx.abs().max()))
    assert torch.equal(nx[0], x0)
    cost = (0.5 * (tau * torch.einsum("tbij,tbj->tbi", C, tau)).sum(-1) + (tau * c).sum(-1)).sum(0)
    assert float(((cost - o["costs"]).abs() / cost.abs().clamp_min(1)).max()) < 2e-4
    o2 = lqr_step_raw(n, m, T, x0, C, c, F, f, nx, nu)           # one unconstrained LQR step is exact
    assert float(o2["full_du_norm"].max()) < 1e-3
    idx = torch.arange(0, B, 64)
    sl = lambda t: t[:, idx].cpu().contiguous()
    ob = orc.lqr_step_forward(n, m, T, x0[idx].cpu(), sl(C), sl(c), sl(F), sl(f), sl(x), sl(u), coupled=False)
    scale = max(1.0, float(ob.new_x.abs().max()))
    assert maxdiff(nx[:, idx], ob.new_x) < 1e-4 * scale and maxdiff(nu[:, idx], ob.new_u) < 1e-4 * scale
    assert maxdiff(o["costs"][idx], ob.costs) < 3e-4 * float(ob.costs.abs().max())


@pytest.mark.parametrize("bounds", [None, 0.25], ids=["unbounded", "box"])
def test_adjoint_config3_size_vs_oracle(bounds):
    """LQRStepFn.backward (KKT adjoint) at B=4096, T=20, n=8, m=2, fp32 vs the oracle's adjoint on CPU."""
    from mpc.pytorch_b200 import LQRStep, QuadCost, LinDx
    B, T, n, m = 4096, 20, 8, 2
    C, c, F, f, x0 = gen_problem(3100, B, T, n, m, torch.float32)
    u = torch.zeros(T, B, m)
    x = orc.get_traj(T, u, x0, F, f)
    kw = {} if bounds is None else dict(u_lower=-bounds, u_upper=bounds)
    # the solution the adjoint is taken at: a few oracle steps (converged enough for a meaningful active set)
    for _ in range(3):
        o = orc.lqr_step_forward(n, m, T, x0, C, c, F, f, x, u, coupled=False, **kw)
        x, u = o.new_x, o.new_u
    g = torch.Generator().manual_seed(9)
    wx, wu = torch.randn(T, B, n, generator=g), torch.randn(T, B, m, generator=g)
    ref = orc.lqr_step_backward(n, m, T, x0, C, c, F, f, x, u, wx, wu, coupled=False, **kw)
    lv = [t.to(DEV).requires_grad_(True) for t in (x0, C, c, F, f)]
    fn = LQRStep(n, m, T, true_cost=QuadCost(lv[1], lv[2]), true_dynamics=LinDx(lv[3], lv[4]),
                 current_x=x.to(DEV), current_u=u.to(DEV), no_op_forward=True, **kw)
    xo, uo = fn(*lv)
    grads = torch.autograd.grad((xo * wx.to(DEV)).sum() + (uo * wu.to(DEV)).sum(), lv)
    for gname, a, b in zip(("dx_init", "dC", "dc", "dF", "df"), grads, ref[:5]):
        sc = max(1.0, float(b.abs().max()))
        assert maxdiff(a, b) <= 3e-4 * sc, (gname, maxdiff(a, b), sc)


@pytest.mark.parametrize("name,tol_u,tol_cost", [("cartpole_full_f64", 1e-5, 1e-7), ("cartpole_full_f32", 5e-3, 2e-4)])
def test_config2_cartpole_full_size_vs_reference(name, tol_u, tol_cost):
    """BASELINE config 2: cartpole iLQR MPC, B=128, T=25, bounds +-100, AUTO_DIFF, vs the reference's stored
    trajectories (oracle/make_golden.py).  float64: every problem to 1e-5; float32: costs to 2e-4 relative and
    controls to 5e-3 (fp32 round-off through the nonlinear iterations), compared on ALL problems."""
    from mpc.pytorch_b200 import MPC, QuadCost, GradMethods
    from mpc.env_dx.cartpole import CartpoleDx            # known system: rollout / Jacobians / line search in kernels
    g = load_golden(name)
    dtype = g["x_init"].dtype
    T, B = g["x"].shape[0], g["x"].shape[1]
    assert (B, T) == (128, 25)
    Q = g["Q"].expand(T, B, 6, 6).contiguous()             # the fixture stores one (t, b) slice: Q, p are constant
    p = g["p"].expand(T, B, 6).contiguous()
    dx = CartpoleDx(params=torch.tensor((9.8, 1.0, 0.1, 0.5), dtype=dtype))
    ctrl = MPC(5, 1, T, u_lower=-100.0, u_upper=100.0, lqr_iter=int(g["lqr_iter"]), verbose=-1,
               exit_unconverged=False, detach_unconverged=False, linesearch_decay=0.5, max_linesearch_iter=2,
               grad_method=GradMethods.AUTO_DIFF, eps=1e-2)
    x, u, costs = ctrl(g["x_init"].to(DEV), QuadCost(Q.to(DEV), p.to(DEV)), dx)
    assert x.dtype == dtype
    rel = ((costs.cpu() - g["costs"]).abs() / g["costs"].abs().clamp_min(1.0))
    assert float(rel.max()) <= tol_cost, float(rel.max())
    assert maxdiff(u, g["u"]) <= tol_u * max(1.0, float(g["u"].abs().max()))
    assert maxdiff(x, g["x"]) <= 10 * tol_u * max(1.0, float(g["x"].abs().max()))
