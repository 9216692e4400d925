"""GPU parity: the CUDA LQR step (through the C ABI) against the CPU oracle and the reference
fixtures.  Tolerances (stated per SURVEY.md section 8c):
  float64            : 1e-9 absolute on x,u (identical algorithm, different summation order)
  float32 unbounded  : 2e-5 abs + 1e-4 rel on x,u, 1e-4 rel on costs
  float32 bounded    : 2e-4 abs (pnqp stops at |dx| < 1e-4), active sets bit exact
"""
import glob
import os

import pytest
import torch

from oracle import lqr_oracle as orc
from tests.gpu_harness import DEV, check_step_fixed, run_step, to_dev, tol_for
from tests.helpers import GOLD, gen_problem, load_golden, maxdiff, nominal_controls

pytestmark = pytest.mark.gpu


def raw(n, m, T, x0, C, c, F, f, x, u, **kw):
    """The step with gains and du_first, on the CPU."""
    return run_step(n, m, T, dict(x0=x0, C=C, c=c, F=F, f=f, x=x, u=u), kw, want_du_first=True)[0]


CASES = [
    # name, seed, B, T, n, m, dtype, bounds, delta_u, time_varying, with_f
    ("cfg1_f32", 1, 1, 5, 3, 1, torch.float32, None, None, True, True),
    ("unb_f64_n4m2", 2, 4, 6, 4, 2, torch.float64, None, None, False, True),
    ("unb_f32_n8m2_B37_unaligned", 3, 37, 20, 8, 2, torch.float32, None, None, False, True),
    ("unb_f32_n8m2_B48_bulk", 3, 48, 20, 8, 2, torch.float32, None, None, False, True),
    ("unb_f32_n8m2_B49_tail", 3, 49, 20, 8, 2, torch.float32, None, None, False, True),
    ("box_f64_n4m2", 4, 8, 8, 4, 2, torch.float64, 0.25, None, False, True),
    ("box_f32_n8m2_B96", 5, 96, 20, 8, 2, torch.float32, 0.25, None, False, True),
    ("boxT_f64_n3m4", 6, 6, 6, 3, 4, torch.float64, "tensor", None, True, True),
    ("boxT_f32_n8m2", 16, 24, 12, 8, 2, torch.float32, "tensor", None, False, True),
    ("delta_f64_n3m2", 7, 4, 6, 3, 2, torch.float64, 0.5, 0.1, False, True),
    ("box_f64_n5m1_nof", 8, 6, 9, 5, 1, torch.float64, 0.3, None, False, False),
    ("box_f64_n16m4", 9, 5, 12, 16, 4, torch.float64, 0.25, None, False, True),
    ("unb_f32_n16m4_T50", 13, 6, 50, 16, 4, torch.float32, None, None, False, True),
    ("pad_f64_n3m3", 11, 5, 6, 3, 3, torch.float64, 0.3, None, False, True),
    ("pad_f32_n6m1", 14, 9, 8, 6, 1, torch.float32, None, None, False, True),
    ("unb_f64_n6m2_T60", 12, 7, 60, 6, 2, torch.float64, None, None, False, True),
    ("unb_f64_T1", 15, 3, 1, 4, 2, torch.float64, None, None, False, True),
    ("box_f64_T2", 17, 3, 2, 4, 2, torch.float64, 0.2, None, False, True),
    # shapes / batch sizes that take the column-pair kernel (even n, m; 16-byte aligned spans), every mode
    ("pair_delta_f64_n4m2", 18, 8, 6, 4, 2, torch.float64, 0.5, 0.1, False, True),
    ("pair_boxT_f32_n4m2_tail", 19, 44, 9, 4, 2, torch.float32, "tensor", None, True, True),
    ("pair_boxT_f64_n4m2_tail", 19, 44, 9, 4, 2, torch.float64, "tensor", None, True, True),
    ("pair_delta_f32_n16m4", 20, 8, 7, 16, 4, torch.float32, 0.4, 0.15, False, True),
    ("pair_unb_f32_n2m2", 21, 20, 5, 2, 2, torch.float32, None, None, True, False),
    ("pair_box_f64_n8m4", 22, 12, 6, 8, 4, torch.float64, 0.3, None, False, True),
    ("pair_unb_f64_T1", 23, 4, 1, 4, 2, torch.float64, None, None, False, True),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_step_matches_oracle(case):
    name, seed, B, T, n, m, dtype, bounds, delta_u, tv, wf = case
    C, c, F, f, x0 = gen_problem(seed, B, T, n, m, dtype, tv, wf)
    if T == 1:
        F = torch.zeros(0, B, n, n + m, dtype=dtype)
        f = None
    u, ul, uu = nominal_controls(seed, B, T, m, dtype, bounds)
    x = orc.get_traj(T, u, x0, F, f)
    o = orc.lqr_step_forward(n, m, T, x0, C, c, F, f, x, u, u_lower=ul, u_upper=uu, delta_u=delta_u,
                             coupled=False)
    kw = dict(u_lower=ul, u_upper=uu, delta_u=delta_u)
    r = raw(n, m, T, x0, C, c, F, f, x, u, **kw)
    check_step_fixed(name, r, o, kw, dtype)
    # per-problem ||u_bar - u_1||_2 (the ABI value) and the reference's batch-mixing variant
    tol = tol_for(dtype, bounds is not None)
    scale = max(1.0, float(o.new_x.abs().max()))
    true_fdn = (u - o.new_u).pow(2).sum((0, 2)).sqrt() if float(o.alphas.min()) == 1.0 else None
    if true_fdn is not None:
        assert maxdiff(r["full_du_norm"], true_fdn) <= 10 * tol["xu"] * scale
    from mpc.pytorch_b200.step import reference_full_du_norm
    assert maxdiff(reference_full_du_norm(r["du_first"]), o.full_du_norm) <= 10 * tol["xu"] * scale


@pytest.mark.parametrize("name", sorted(os.path.basename(p)[:-4] for p in
                                        glob.glob(os.path.join(GOLD, "step_*.npz"))))
def test_step_matches_reference_fixture(name):
    """CUDA vs the REAL reference's stored outputs (batch-coupled pnqp): bounded cases agree to the
    pnqp step tolerance, unbounded ones to round-off; clamp masks exactly."""
    g = load_golden(name)
    T, B, p = g["C"].shape[0], g["C"].shape[1], g["C"].shape[2]
    n = g["x_init"].shape[1]
    m = p - n
    ul, uu = g.get("u_lower"), g.get("u_upper")
    r = raw(n, m, T, g["x_init"], g["C"], g["c"], g["F"], g.get("f"), g["cur_x"], g["cur_u"],
            u_lower=ul, u_upper=uu, delta_u=g.get("delta_u"))
    f64 = g["C"].dtype == torch.float64
    tol = (2e-4 if ul is not None else 1e-9) if f64 else (2e-4 if ul is not None else 4e-5)
    assert maxdiff(r["new_x"], g["new_x"]) <= tol
    assert maxdiff(r["new_u"], g["new_u"]) <= tol
    assert maxdiff(r["costs"], g["costs"]) <= 10 * tol * max(1.0, float(g["costs"].abs().max()))
    assert abs(float(r["alphas"].mean()) - float(g["mean_alphas"])) < 1e-6
    if ul is not None and g.get("delta_u") is None:
        lo = ul if torch.is_tensor(ul) else torch.full_like(g["new_u"], ul)
        assert torch.equal(r["new_u"] == lo.to(r["new_u"].dtype), g["new_u"] == lo.to(r["new_u"].dtype))
        n_qp = float((1 + r["qp_iters"].max(dim=1).values).sum())
        assert abs(n_qp - float(g["n_total_qp_iter"])) <= 2          # +-1 noise (SURVEY section 6)


@pytest.mark.parametrize("B", [9, 16])          # 16: aligned spans -> the column-pair kernel also in float32
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_masked_adjoint_mode_matches_oracle(dtype, B):
    """u_zero_I branch (reference lqr_step.py:100-127,197-198) - the mode the backward pass uses."""
    T, n, m = 7, 4, 2
    C, c, F, f, x0 = gen_problem(10, B, T, n, m, dtype)
    g = torch.Generator().manual_seed(3)
    zI = torch.rand(T, B, m, generator=g) < 0.35
    zx = torch.zeros(T, B, n, dtype=dtype)
    zu = torch.zeros(T, B, m, dtype=dtype)
    o = orc.lqr_step_forward(n, m, T, torch.zeros_like(x0), C, c, F, None, zx, zu, u_zero_I=zI, coupled=False)
    r = raw(n, m, T, torch.zeros_like(x0), C, c, F, None, zx, zu, u_zero_I=zI)
    tol = 1e-9 if dtype == torch.float64 else 4e-5
    assert maxdiff(r["new_x"], o.new_x) <= tol and maxdiff(r["new_u"], o.new_u) <= tol
    assert torch.equal(r["free_mask"].bool(), ~zI)
    assert bool((r["new_u"][zI] == 0).all())                             # masked controls exactly zero
    assert bool((r["Ks"][zI] == 0).all())


def test_line_search_alphas_on_notebook_problem():
    """Walk the reference notebook problem (bounded, open-loop unstable): the line search backtracks
    at some iterations (golden mean(alphas) 0.6 / 0.52); CUDA must take the same alphas."""
    g = load_golden("tvlqr_notebook_f32")
    n, m, T = 3, 4, 5
    C, c, F, x0 = (g[k].double() for k in ("C", "c", "F", "x_init"))
    ul, uu = g["u_lower"].double(), g["u_upper"].double()
    u = torch.zeros(T, 2, m, dtype=torch.float64)
    seen_backtrack = False
    for it in range(9):
        x = orc.get_traj(T, u, x0, F, None)
        o = orc.lqr_step_forward(n, m, T, x0, C, c, F, None, x, u, u_lower=ul, u_upper=uu, coupled=False)
        r = raw(n, m, T, x0, C, c, F, None, x, u, u_lower=ul, u_upper=uu)
        # at the fixed point `cost > old_cost` is decided by round-off (the reference's own
        # notebook trace shows alphas 0.52/0.6 there): compare alphas only while still moving
        moving = (u - o.new_u).pow(2).sum((0, 2)).sqrt() > 1e-5      # true per-problem step norm
        assert maxdiff(r["alphas"][moving], o.alphas[moving]) < 1e-12, it
        assert maxdiff(r["new_u"][:, moving], o.new_u[:, moving]) < 1e-7
        assert maxdiff(r["costs"], o.costs) < 1e-7
        seen_backtrack |= float(o.alphas[moving].min()) < 1.0 if bool(moving.any()) else False
        u = o.new_u
    assert seen_backtrack


def test_riccati_only_and_split_rollout_equal_fused():
    """do_rollout=0 exports the gains; LQRStep with a Module as true dynamics (split mode) must
    reproduce the fused kernel when the Module is the same affine map."""
    from mpc.pytorch_b200 import LQRStep, QuadCost, LinDx
    B, T, n, m = 12, 9, 5, 1
    C, c, F, f, x0 = [to_dev(t) for t in gen_problem(50, B, T, n, m, torch.float64, time_varying=False)]
    u = to_dev(nominal_controls(50, B, T, m, torch.float64, 0.3)[0])
    from mpc.pytorch_b200.solver import get_traj
    x = get_traj(T, u, x0, LinDx(F, f))

    class Affine(torch.nn.Module):                      # time-invariant: F[0], f varies -> use f[0] too
        def forward(self, xx, uu):
            return torch.einsum("bij,bj->bi", F[0], torch.cat((xx, uu), 1)) + f0

    f0 = f[0]
    f_ti = f0.unsqueeze(0).repeat(T - 1, 1, 1).contiguous()
    x = get_traj(T, u, x0, LinDx(F, f_ti))
    kw = dict(u_lower=-0.3, u_upper=0.3, current_x=x, current_u=u)
    fused = LQRStep(n, m, T, true_cost=QuadCost(C, c), true_dynamics=LinDx(F, f_ti), **kw)(x0, C, c, F, f_ti)
    split = LQRStep(n, m, T, true_cost=QuadCost(C, c), true_dynamics=Affine(), **kw)(x0, C, c, F, f_ti)
    for a, b in zip(fused, split):
        assert maxdiff(a, b) < 1e-10


def test_config3_full_size_properties():
    """BASELINE config 3 (B=4096,T=20,n=8,m=2) fp32: size-independent properties + a sampled oracle check."""
    from mpc.pytorch_b200.step import lqr_step_raw
    from mpc.pytorch_b200.solver import get_traj, LinDx
    B, T, n, m = 4096, 20, 8, 2
    C, c, F, f, x0 = [to_dev(t) for t in gen_problem(3000, B, T, n, m, torch.float32)]
    u = torch.zeros(T, B, m, device=DEV)
    x = get_traj(T, u, x0, LinDx(F, f))
    for bounds in (None, 0.25):
        kw = {} if bounds is None else dict(u_lower=-bounds, u_upper=bounds)
        o = lqr_step_raw(n, m, T, x0, C, c, F, f, x, u, **kw)
        nx, nu = o["new_x"], o["new_u"]
        # fp32 pnqp: a handful of (t,b) QPs cycle at round-off level and hit the 20-iteration cap - the
        # reference prints "pnqp warning: Did not converge" for the same inputs (oracle: 11 of 81920)
        st = o["status"]
        assert int((st & ~1).max()) == 0 and float((st != 0).float().mean()) < 5e-3
        assert bool(torch.isfinite(o["costs"]).all())
        # (1) dynamics feasibility of the returned trajectory
        tau = torch.cat((nx, nu), 2)
        pred = torch.einsum("tbij,tbj->tbi", F, tau[:-1]) + f
        assert float((pred - nx[1:]).abs().max()) < 2e-5 * max(1.0, float(nx.abs().max()))
        assert torch.equal(nx[0], x0)
        # (2) reported cost is the cost of the returned trajectory and not worse than the nominal one
        cost = (0.5 * (tau * torch.einsum("tbij,tbj->tbi", C, tau)).sum(-1) + (tau * c).sum(-1)).sum(0)
        assert float(((cost - o["costs"]).abs() / cost.abs().clamp_min(1)).max()) < 1e-4
        tb = torch.cat((x, u), 2)
        old = (0.5 * (tb * torch.einsum("tbij,tbj->tbi", C, tb)).sum(-1) + (tb * c).sum(-1)).sum(0)
        assert bool((o["costs"] <= old + 1e-3 * old.abs()).all())
        # (3) bounds hold exactly; (4) idempotence: a second step from the solution does not move
        if bounds is not None:
            assert float(nu.abs().max()) <= bounds
            assert 0.5 < float((nu.abs() == bounds).float().mean()) < 0.95
        o2 = lqr_step_raw(n, m, T, x0, C, c, F, f, nx, nu, **kw)
        if bounds is None:      # one unconstrained LQR step is exact: the solution is a fixed point
            assert float(o2["full_du_norm"].max()) < 2e-4
            assert float((o2["costs"] - o["costs"]).abs().max()) < 1e-3 * float(o["costs"].abs().max())
        else:                   # box-constrained iLQR needs several steps; each one must not increase the cost
            assert bool((o2["costs"] <= o["costs"] + 1e-3 * o["costs"].abs()).all())
        # (5) sampled oracle check
        idx = torch.arange(0, B, 64)
        sl = lambda t: t[:, idx].cpu().contiguous()
        ob = orc.lqr_step_forward(n, m, T, x0[idx].cpu(), sl(C), sl(c), sl(F), sl(f), sl(x), sl(u),
                                  coupled=False, **kw)
        tol = 2e-4 if bounds else 4e-5
        okp = (st[idx].cpu() == 0) & (ob.qp_iters.max(0).values < 19)     # both converged
        assert float(okp.float().mean()) > 0.9
        assert maxdiff(nu[:, idx][:, okp], ob.new_u[:, okp]) < tol
        assert maxdiff(nx[:, idx][:, okp], ob.new_x[:, okp]) < tol
        if bounds is not None:
            assert torch.equal(o["free_mask"][:, idx].cpu().bool()[:, okp], ob.free_masks[:, okp])


@pytest.mark.parametrize("name", ["pnqp_f64_cold", "pnqp_f64_warm", "pnqp_f32_cold", "pnqp_f64_n1"])
def test_standalone_pnqp_matches_reference_fixture(name):
    """mpc.pnqp.pnqp on the GPU vs the reference's stored outputs and the per-problem oracle."""
    from mpc.pnqp import pnqp
    g = load_golden(name)
    H, q, lo, hi = (g[k].to(DEV) for k in ("H", "q", "lower", "upper"))
    x0 = g["x_init"].to(DEV) if "x_init" in g else None
    x, Hf, If, it = pnqp(H, q, lo, hi, x_init=x0, n_iter=20)
    xo, Ho, Ifo, ito = orc.pnqp(g["H"], g["q"], g["lower"], g["upper"], x_init=g.get("x_init"), n_iter=20,
                                coupled=False)
    f64 = g["H"].dtype == torch.float64
    assert maxdiff(x, xo) <= (1e-10 if f64 else 2e-6)
    assert torch.equal(If.cpu().bool(), Ifo.bool()) and it == int(ito.max())
    assert maxdiff(Hf, Ho) <= (1e-12 if f64 else 1e-6)
    assert maxdiff(x, g["x"]) <= 2e-4                      # reference (batch-coupled) result
    assert torch.equal(If.cpu().bool(), g["If"].bool())    # active set: bit exact


def test_bounds_together_with_zero_mask():
    """u_zero_I given AND box bounds (allowed by the reference: pnqp ignores the mask, the rollout zeroes the
    masked controls and then clamps them, mpc/lqr_step.py:129-148,197-213)."""
    B, T, n, m = 7, 6, 4, 2
    C, c, F, f, x0 = gen_problem(81, B, T, n, m, torch.float64)
    u, ul, uu = nominal_controls(81, B, T, m, torch.float64, "tensor")
    g = torch.Generator().manual_seed(4)
    zI = torch.rand(T, B, m, generator=g) < 0.3
    x = orc.get_traj(T, u, x0, F, f)
    o = orc.lqr_step_forward(n, m, T, x0, C, c, F, f, x, u, u_lower=ul, u_upper=uu, u_zero_I=zI, coupled=False)
    r = raw(n, m, T, x0, C, c, F, f, x, u, u_lower=ul, u_upper=uu, u_zero_I=zI)
    assert maxdiff(r["new_x"], o.new_x) < 1e-9 and maxdiff(r["new_u"], o.new_u) < 1e-9
    assert maxdiff(r["costs"], o.costs) < 1e-9 and maxdiff(r["alphas"], o.alphas) == 0.0
    assert torch.equal(r["free_mask"].bool(), o.free_masks)


def test_tensor_bounds_with_delta_u_and_full_length_F():
    """tensor bounds + trust region, and F carrying T time slices (only F[:T-1] is read, reference
    mpc/lqr_step.py:66,217-220; dF[T-1] is zero, :387-395)."""
    from mpc.pytorch_b200 import LQRStep, QuadCost, LinDx
    B, T, n, m = 5, 6, 3, 2
    C, c, F, f, x0 = gen_problem(82, B, T, n, m, torch.float64, time_varying=True)
    FT = torch.cat((F, torch.randn(1, B, n, n + m, dtype=torch.float64)), 0)       # T slices, last one unused
    u, ul, uu = nominal_controls(82, B, T, m, torch.float64, "tensor")
    x = orc.get_traj(T, u, x0, F, f)
    o = orc.lqr_step_forward(n, m, T, x0, C, c, F, f, x, u, u_lower=ul, u_upper=uu, delta_u=0.07, coupled=False)
    r = raw(n, m, T, x0, C, c, FT, f, x, u, u_lower=ul, u_upper=uu, delta_u=0.07)
    assert maxdiff(r["new_x"], o.new_x) < 1e-9 and maxdiff(r["new_u"], o.new_u) < 1e-9
    assert float((r["new_u"] - u).abs().max()) <= 0.07 + 1e-12
    # gradients with the full-length F: slice T-1 of dF must be exactly zero
    lv = [t.to(DEV).requires_grad_(True) for t in (x0, C, c, FT, f)]
    fn = LQRStep(n, m, T, u_lower=to_dev(ul), u_upper=to_dev(uu), true_cost=QuadCost(lv[1], lv[2]),
                 true_dynamics=LinDx(lv[3], lv[4]), current_x=o.new_x.to(DEV), current_u=o.new_u.to(DEV),
                 no_op_forward=True)
    xo, uo = fn(*lv)
    grads = torch.autograd.grad(xo.sum() + (uo * uo).sum(), lv)
    assert grads[3].shape == FT.shape and float(grads[3][T - 1].abs().max()) == 0.0
    ref = orc.lqr_step_backward(n, m, T, x0, C, c, F, f, o.new_x, o.new_u, torch.ones_like(o.new_x), 2 * o.new_u,
                                u_lower=ul, u_upper=uu, coupled=False)
    assert maxdiff(grads[3][:T - 1], ref[3]) < 1e-9 and maxdiff(grads[0], ref[0]) < 1e-9
