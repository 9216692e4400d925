"""CPU: oracle/known_oracle.py, the float64 iLQR loop and episode of a known system, pinned to the reference's own
fixtures (coupled pnqp, as the reference runs a batch); its reductions; and the case builders of
tests/test_known_oracle_gpu.py, which must reach what they claim without a device.

Fixture tolerances, relative to max(1, max|want|): each is what the oracle holds, measured, rounded up to a power
of ten.  The oracle's Jacobians come from autograd over every (t, b) at once where the reference takes them one time
step at a time, and its pnqp is a restatement: where a fixture is reproduced bit for bit the tolerance is 0."""
import os

import numpy as np
import pytest
import torch

from oracle import known_oracle as ko
from oracle import mlp_oracle as mo
from tests.gpu_harness import episode_known_step, pool_size
from tests.helpers import maxdiff

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
F64 = torch.float64


def load(name, prefix=None):
    z = np.load(os.path.join(GOLD, name + ".npz"))
    if prefix is None:
        return {k: torch.from_numpy(z[k]) for k in z.files}
    pre = prefix + "_"
    others = [c + "_" for c in ("pendulum_slew", "linear_plant") if c != prefix and c.startswith(prefix)]
    return {k[len(pre):]: torch.from_numpy(z[k]) for k in z.files
            if k.startswith(pre) and not any(k.startswith(o) for o in others)}


def module(name, params, dt=None, clamp=None):
    """(module, theta row) of a known system with float64 `params`, `dt` and control clamp (None: the module's)."""
    from mpc.pytorch_b200.dynamics import CartpoleDx, PendulumDx
    p = torch.as_tensor(params, dtype=F64)
    if name == "cartpole":
        mod = CartpoleDx(params=p)
    else:
        mod = PendulumDx(params=p, simple=name != "pendulum_full")
    if dt is not None:
        mod.dt = float(dt)
    if clamp is not None:
        setattr(mod, "force_mag" if name == "cartpole" else "max_torque", float(clamp))
    return mod, p


def rel(a, b):
    return maxdiff(a, b) / max(1.0, float(b.abs().max()))


def check(tag, got, want, tol):
    for k, (a, b) in enumerate(zip(got, want)):
        err = rel(a, b)
        assert err <= tol, f"{tag}: output {k} differs by {err:.3e} > {tol:.0e}"


# ------------------------------------------------------------------------------------------------------------------
# the loop against the reference's MPC.forward
# ------------------------------------------------------------------------------------------------------------------
def test_pendulum_ilqr_fixture_bitwise():
    """The pendulum swing-up (B = 16, T = 20, 15 iterations, stop test on): x, u and costs bit for bit."""
    g = load("pendulum_ilqr_f64")
    B, T = g["x_init"].shape[0], g["x"].shape[0]
    mod, p = module("pendulum", (10.0, 1.0, 1.0))
    C = torch.diag(g["q"]).expand(T, B, 4, 4)
    c = g["p"].expand(T, B, 4)
    x, u, costs, it = ko.ilqr(3, 1, T, g["x_init"], C, c, episode_known_step(mod), p.expand(B, -1),
                              lqr_iter=int(g["lqr_iter"]), eps=mod.mpc_eps, u_lower=-2.0, u_upper=2.0,
                              linesearch_decay=0.2, max_linesearch_iter=5, coupled=True)
    check("pendulum", (x, u, costs), (g["x"], g["u"], g["costs"]), 0.0)


def test_cartpole_config2_fixture():
    """BASELINE config 2: cartpole, B = 128, T = 25, bounds +-100, decay 0.5, 2 passes, eps 1e-2, 20 iterations.
    x and u within 1e-8 (largest absolute differences 3.3e-8 and 2.0e-7, 5.1e-9 and 4.6e-9 relative), costs within
    1e-15 (1.9e-16)."""
    g = load("cartpole_full_f64")
    B, T = g["x_init"].shape[0], g["x"].shape[0]
    mod, p = module("cartpole", (9.8, 1.0, 0.1, 0.5))
    x, u, costs, it = ko.ilqr(5, 1, T, g["x_init"], g["Q"].expand(T, B, 6, 6), g["p"].expand(T, B, 6),
                              episode_known_step(mod), p.expand(B, -1), lqr_iter=int(g["lqr_iter"]), eps=1e-2,
                              u_lower=-100.0, u_upper=100.0, linesearch_decay=0.5, max_linesearch_iter=2,
                              coupled=True)
    check("cartpole x, u", (x, u), (g["x"], g["u"]), 1e-8)
    check("cartpole costs", (costs,), (g["costs"],), 1e-15)


@pytest.mark.parametrize("tag", ["unb", "box"])
def test_pendulum_full_ilqr_fixture(tag):
    """The five-parameter pendulum at non-default physics, without bounds (controls pass the clamp) and with a box
    inside it: bit for bit."""
    g = load("pendulum_full_ilqr_f64")
    B, T = g["x_init"].shape[0], g["C"].shape[0]
    mod, p = module("pendulum_full", g["params"], g["dt"], g["clamp"])
    kw = {} if tag == "unb" else dict(u_lower=-float(g["bound_box"]), u_upper=float(g["bound_box"]))
    x, u, costs, _ = ko.ilqr(3, 1, T, g["x_init"], g["C"], g["c"], episode_known_step(mod), p.expand(B, -1),
                             lqr_iter=int(g["lqr_iter"]), eps=1e-9, linesearch_decay=float(g["decay"]),
                             max_linesearch_iter=int(g["ls_iter"]), coupled=True, **kw)
    check(f"pendulum_full {tag}", (x, u, costs), (g["x_" + tag], g["u_" + tag], g["costs_" + tag]), 0.0)


# (x, u) tolerance of each slew fixture; the rest are bit for bit.  Costs within 1e-15 (largest 2.9e-16)
SLEW_TOL = {("cartpole", "in"): 1e-8}          # 7.9e-9 in u, 8.8e-10 in x


@pytest.mark.parametrize("tag", ["in", "wide"])
@pytest.mark.parametrize("name", ["cartpole", "pendulum", "pendulum_full"])
def test_known_slew_fixture(name, tag):
    """MPC(slew_rate_penalty, prev_ctrl) with the system as dynamics: the passthrough loop (n_prev = m) on
    slew_problem's cost.  Bounds inside the clamp ("in") and twice it ("wide", where plans pass the clamp).  x and u
    bit for bit but for cartpole "in" (SLEW_TOL)."""
    g = load(f"known_slew_{name}_f64")
    B, T = g["x_init"].shape[0], g["C"].shape[0]
    n = g["x_init"].shape[1]
    mod, p = module(name, g["params"], g["dt"], g["clamp"])
    b = float(g["bound_" + tag])
    x0, C2, c2 = ko.slew_problem(n, 1, float(g["penalty"]), g["C"], g["c"], g["x_init"], g["prev_ctrl"])
    x, u, costs, _ = ko.ilqr(n + 1, 1, T, x0, C2, c2, episode_known_step(mod), p.expand(B, -1),
                             lqr_iter=int(g["lqr_iter"]), eps=1e-9, u_lower=-b, u_upper=b,
                             linesearch_decay=float(g["decay"]), max_linesearch_iter=int(g["ls_iter"]), n_prev=1,
                             coupled=True)
    assert torch.equal(x[1:, :, :1], u[:-1]) and torch.equal(x[0, :, :1], g["prev_ctrl"])
    if tag == "wide":
        assert bool((u.abs() > float(g["clamp"])).any()), "the wide bounds must let controls pass the clamp"
    check(f"slew {name} {tag}", (x[..., 1:], u), (g["x_" + tag], g["u_" + tag]), SLEW_TOL.get((name, tag), 0.0))
    check(f"slew {name} {tag} costs", (costs,), (g["costs_" + tag],), 1e-15)


# ------------------------------------------------------------------------------------------------------------------
# the episode against the reference's notebook loop
# ------------------------------------------------------------------------------------------------------------------
# case: (system, fixture key of the slew-rate penalty, x / u / costs tolerance; largest errors 1.6e-9, 1.6e-7,
# 3.3e-8 and 9.7e-9, in u: the 15 solves each stop at eps = 1e-2, so the plans carry the loops' differences)
RECEDING = {"cartpole": ("cartpole", None, 1e-8), "pendulum": ("pendulum", None, 1e-6),
            "pendulum_full": ("pendulum_full", None, 1e-7), "pendulum_slew": ("pendulum", "penalty", 1e-8)}


@pytest.mark.parametrize("case", list(RECEDING))
def test_receding_fixture(case):
    """The notebooks' loop (15 control steps, the module's default dt and clamp, lqr_iter 50, eps 1e-2): x, u, costs
    and each solve's iteration count."""
    g = load(f"receding_{case}_f64")
    name, pen, tol = RECEDING[case]
    mod, p = module(name, g["params"])
    B, T = g["x_init"].shape[0], int(g["T"])
    n = g["x_init"].shape[1]
    clamp = float(mod.force_mag if name == "cartpole" else mod.max_torque)
    ep = ko.episode(n, 1, T, int(g["n_steps"]), g["x_init"], g["C"], g["c"], episode_known_step(mod),
                    p.expand(B, -1), u_lower=-clamp, u_upper=clamp, lqr_iter=int(g["lqr_iter"]),
                    eps=float(g["eps"]), linesearch_decay=float(g["decay"]), max_linesearch_iter=int(g["ls_iter"]),
                    slew_rate_penalty=float(g[pen]) if pen else None, coupled=True)
    assert ep.iters == g["iters"].tolist(), (ep.iters, g["iters"].tolist())
    check(f"receding {case}", (ep.x, ep.u, ep.costs), (g["x"], g["u"], g["costs"]), tol)


# x, u and plans: pendulum bit for bit, cartpole 3.8e-8 (its plans), pendulum_slew 2.1e-14
TV_TOL = {"pendulum": 0.0, "cartpole": 1e-7, "pendulum_slew": 1e-13}


@pytest.mark.parametrize("case", ["pendulum", "cartpole", "pendulum_slew"])
def test_receding_tv_fixture(case):
    """The reference's windowed loop with a known model: C, c sliced per control step, eps 1e-4: x, u, the plans and
    the iteration counts."""
    t = load("receding_tv_f64", case)
    name = case.split("_")[0]
    mod, p = module(name, t["params"], clamp=t["clamp"])
    B, T, n = t["x_init"].shape[0], int(t["T"]), t["x_init"].shape[1]
    cl = float(t["clamp"])
    ep = ko.episode(n, 1, T, int(t["n_steps"]), t["x_init"], t["C"], t["c"], episode_known_step(mod),
                    p.expand(B, -1), u_lower=-cl, u_upper=cl, lqr_iter=int(t["lqr_iter"]), eps=float(t["eps"]),
                    linesearch_decay=float(t["ls_decay"]), max_linesearch_iter=int(t["ls_iter"]),
                    slew_rate_penalty=float(t["slew"]) if "slew" in t else None, window=True, coupled=True)
    assert ep.iters == t["iters"].tolist(), (ep.iters, t["iters"].tolist())
    plan_x = ep.plan_x[..., 1:] if "slew" in t else ep.plan_x
    check(f"tv {case}", (ep.x, ep.u, plan_x, ep.plan_u), (t["x"], t["u"], t["plan_x"], t["plan_u"]), TV_TOL[case])


# ------------------------------------------------------------------------------------------------------------------
# reductions
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("slew", [None, 0.5])
def test_one_step_episode_is_one_solve(slew):
    """An episode of one control step is one ilqr call from x_init (under a penalty, from [prev; x_init] on
    slew_problem's cost), bit for bit, and its next state the model's step of the applied control."""
    mod, p = module("cartpole", (9.81, 1.3, 0.25, 0.8), 0.05, 7.5)
    B, T, n = 5, 7, 5
    g = torch.Generator().manual_seed(3)
    q, pp = mod.get_true_obj()
    C = torch.diag(q.double()).expand(T, B, 6, 6)
    c = pp.double().expand(T, B, 6)
    x0 = torch.randn(B, n, generator=g, dtype=F64) * 0.3
    prev = torch.randn(B, 1, generator=g, dtype=F64)
    st, th = episode_known_step(mod), p.expand(B, -1)
    kw = dict(u_lower=-6.0, u_upper=6.0, lqr_iter=4, eps=0.0, not_improved_lim=10, coupled=False)
    ep = ko.episode(n, 1, T, 1, x0, C, c, st, th, slew_rate_penalty=slew, prev_ctrl=prev, **kw)
    if slew is None:
        x, u, costs, it = ko.ilqr(n, 1, T, x0, C, c, st, th, u_init=torch.zeros(T, B, 1, dtype=F64), **kw)
    else:
        xa, Ca, ca = ko.slew_problem(n, 1, slew, C, c, x0, prev)
        x, u, costs, it = ko.ilqr(n + 1, 1, T, xa, Ca, ca, st, th, u_init=torch.zeros(T, B, 1, dtype=F64), n_prev=1,
                                  **kw)
    assert torch.equal(ep.plan_x[0], x) and torch.equal(ep.plan_u[0], u) and torch.equal(ep.costs[0], costs)
    assert ep.iters == [it] and torch.equal(ep.u[0], u[0]) and torch.equal(ep.x[1], st(x0, u[0], th))


# the network cases of tests/golden/mlp_ilqr_loop_f64.npz: (n, m, T, B, bounds, n_prev, passthrough, activation,
# hidden widths, lqr_iter, eps), each run with coupled and per-problem pnqp, linesearch_decay 0.5
MLP_CASES = [(3, 2, 10, 16, "box", 0, False, "sigmoid", (16,), 3, 0.0),
             (5, 2, 6, 12, "tensor", 2, False, "sigmoid", (16,), 3, 0.0),
             (4, 2, 8, 8, "mask", 0, True, "relu", (12, 12), 4, 1e-7),
             (3, 1, 5, 9, "boxD", 0, True, "elu", (8,), 5, 1e-3)]


@pytest.mark.parametrize("i", range(len(MLP_CASES)))
def test_network_loop_unchanged_by_the_shared_loop(i):
    """mlp_oracle.ilqr runs lqr_oracle.ilqr_loop, the loop known_oracle.ilqr runs: x, u, costs and the iteration
    count bit for bit those mlp_oracle.ilqr gave with its own copy of the loop (the fixture), every bound form,
    passthrough, activation and both stop tests, with coupled and per-problem pnqp."""
    n, m, T, B, mode, n_prev, pt, act, hidden, it, eps = MLP_CASES[i]
    z = load("mlp_ilqr_loop_f64")
    g = torch.Generator().manual_seed(i)
    sizes = [n - n_prev + m, *hidden, n - n_prev]
    layers = [(0.5 * torch.randn(o, k, generator=g, dtype=F64), 0.5 * torch.randn(o, generator=g, dtype=F64))
              for k, o in zip(sizes[:-1], sizes[1:])]
    Lc = torch.randn(T, B, n + m, n + m, generator=g, dtype=F64) / (n + m) ** 0.5
    C = Lc @ Lc.transpose(-1, -2) + 0.5 * torch.eye(n + m, dtype=F64)
    c = torch.randn(T, B, n + m, generator=g, dtype=F64)
    x0 = torch.randn(B, n, generator=g, dtype=F64)
    kw = {}
    if mode == "box":
        kw = dict(u_lower=-0.5, u_upper=0.5)
    if mode in ("tensor", "boxD"):
        kw = dict(u_lower=-0.2 - 0.6 * torch.rand(T, B, m, generator=g, dtype=F64),
                  u_upper=0.2 + 0.6 * torch.rand(T, B, m, generator=g, dtype=F64))
        if mode == "boxD":
            kw["delta_u"] = 0.3
    if mode == "mask":
        kw["u_zero_I"] = torch.rand(T, B, m, generator=g) < 0.3
    for coupled in (False, True):
        x, u, costs, its = mo.ilqr(n, m, T, x0, C, c, layers, act, pt, lqr_iter=it, eps=eps, n_prev=n_prev,
                                   coupled=coupled, linesearch_decay=0.5, **kw)
        k = f"c{i}_{int(coupled)}_"
        assert torch.equal(x, z[k + "x"]) and torch.equal(u, z[k + "u"]) and torch.equal(costs, z[k + "costs"])
        assert its == int(z[k + "iters"])


def test_damped_pendulum_is_round_off_sensitive_at_its_switch_horizon():
    """Why test_plans_at_switch leaves out the five-parameter pendulum's damping: with it, over T = 433 steps (just
    below the float64 switch) the float64 oracle's own plans reach |theta| within 1e-3 of pi, where d atan2(sin, cos)
    jumps, and a 1e-15 relative change of x_init moves most problems' plans by more than 1."""
    kg = _gpu_cases()
    T = 433
    case = kg.loop_case("pendulum_full", 0, 8, T, F64, "in", 200, calm=True)
    _, N, P, kw, opts, _, o64 = case[:7]
    mod, p, _ = kg.module("pendulum_full")
    assert float(mod.params[3]) > 0
    x = o64[0]
    assert float(torch.atan2(x[..., 1], x[..., 0]).abs().max()) > torch.pi - 1e-3
    o = ko.ilqr(N, 1, T, P["x0"] * (1 + 1e-15), P["C"], P["c"], episode_known_step(mod), p.expand(8, -1),
                u_init=torch.zeros(T, 8, 1, dtype=F64), coupled=False, **kw, **opts)
    moved = torch.maximum((o[0] - x).abs().amax((0, 2)), (o[1] - o64[1]).abs().amax((0, 2))) > 1.0
    assert int(moved.sum()) > 4, moved


# ------------------------------------------------------------------------------------------------------------------
# the GPU module's case builders reach what they claim
# ------------------------------------------------------------------------------------------------------------------
def _gpu_cases():
    from tests import test_known_oracle_gpu as kg
    return kg


@pytest.mark.parametrize("dtype", [F64, torch.float32], ids=["f64", "f32"])
def test_line_search_cases_decay_and_first_passes_are_worse(dtype):
    """Every case of test_line_search, built with the arguments the GPU module passes, has line-search passes worse
    than their nominal over its loop (the oracle's ls_trace): with more than one pass allowed, their alpha decays;
    with one, the step ends worse and alpha is restored."""
    kg = _gpu_cases()
    for j, name in enumerate(("cartpole", "pendulum")):
        for max_ls, decay in kg.LS:
            physics, bounds = kg.ls_args(j, max_ls, decay, dtype)
            _, N, P, kw, opts = kg.loop_case(name, 0, 16, 15, dtype, bounds, 500 + max_ls, lqr_iter=4,
                                             physics=physics, decay=decay, max_ls=max_ls)[:5]
            mod, p, _ = kg.module(name, physics)
            trace = []
            ko.ilqr(N, 1, 15, P["x0"], P["C"], P["c"], episode_known_step(mod), p.expand(16, -1),
                    u_init=torch.zeros(15, 16, 1, dtype=F64), coupled=False, ls_trace=trace, **kw, **opts)
            worse = sum(int((t > 0).sum()) for t in trace)
            assert worse > 0, (name, max_ls, decay, physics)


@pytest.mark.parametrize("name", ["cartpole", "pendulum", "pendulum_full"])
def test_wide_bounds_pass_the_clamp(name):
    kg = _gpu_cases()
    case = kg.loop_case(name, 0, 12, 10, F64, "wide", 403)
    assert bool((case[6][1].abs() > kg.module(name)[2]).any())


def test_layouts_reach_partial_warps_and_ctas():
    """The step kernel's layout (StepCfg): W = 10 (f64) / 20 (f32) problems per CTA at (5, 1), 8 at (3, 1); the
    layout batches end in partial warps and CTAs at odd and even B; the pool batch's track kernel takes two grid
    passes and its pool copies sit at every position of a warp and a CTA."""
    kg = _gpu_cases()
    assert kg.layout_of("cartpole", 0, F64) == (5, 10) and kg.layout_of("cartpole", 0, torch.float32) == (5, 20)
    assert kg.layout_of("pendulum", 0, F64)[1] == 8 and kg.layout_of("pendulum", 0, torch.float32)[1] == 8
    for name, slew in (("cartpole", 0), ("pendulum", 0), ("pendulum_full", 1)):
        for dtype in (F64, torch.float32):
            ppw, W = kg.layout_of(name, slew, dtype)
            Bs = kg.layout_Bs(name, slew, dtype)
            assert any(b % W and b % 2 for b in Bs) and any(b % W and b % 2 == 0 for b in Bs)
            assert any(b % ppw for b in Bs) and any(b > W and b % W for b in Bs)
    ppw, W = kg.layout_of("pendulum", 0, F64)
    K = pool_size(ppw, W, 128, 256)
    T, N = 10, 3
    B = kg.GRID_CAP // (T * N) + 2 * W + 1
    assert kg.GRID_CAP < T * B * N < 2 * kg.GRID_CAP
    for span in (ppw, W, 128):
        pos = {(b % span, b % K) for b in range(B)}
        assert len(pos) == span * K, span
