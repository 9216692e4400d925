"""CPU: the oracle of receding-horizon episodes (orc.receding_horizon_lin, orc.receding_horizon_backward) pinned to the
reference's own notebook loop (oracle/make_golden_receding_grad.py, oracle/make_golden_receding.py), and the episode
case builders of tests/gpu_harness.py that tests/test_receding_oracle_gpu.py uses, without a device.

  * Fed the reference's stored plans, states and controls, the oracle's reverse sweep gives the reference's gradients
    to 1e-10 relative: LinDx unbounded and bounded (x_init, C, c, F, f), and cartpole, pendulum and the five-parameter
    pendulum (x_init, C, c, params), where the reference's linearisation holds its Jacobians constant
    (full_linearisation=False; INTEGRATION.md section 2).
  * With the reference's batch-coupled pnqp (coupled=True), the oracle's episode gives the reference's x, u, plans and
    iteration counts."""
import os

import numpy as np
import pytest
import torch

from oracle import lqr_oracle as orc
from tests.gpu_harness import (episode_known_inputs, episode_known_module, episode_known_step, episode_linear_inputs,
                               epgrad_launches)

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
F64 = torch.float64


def fixture(name, case):
    z = np.load(os.path.join(GOLD, name + ".npz"))
    pre = case + "_" if case else ""
    return {k[len(pre):]: torch.from_numpy(z[k]) for k in z.files
            if k.startswith(pre) and not (case == "pendulum" and k.startswith("pendulum_full_"))}


def rel(a, b):
    return float((a - b).abs().max()) / max(1e-300, float(b.abs().max()))


@pytest.mark.parametrize("case", ["unbounded", "bounded"])
def test_linear_sweep_against_reference(case):
    t = fixture("receding_grad_linear_f64", case)
    T, n = int(t["T"]), t["F"].shape[2]
    m = t["F"].shape[3] - n
    kw = dict(u_lower=-float(t["bound"]), u_upper=float(t["bound"])) if "bound" in t else {}
    g = orc.receding_horizon_backward(n, m, T, t["C"], t["c"], t["F"], t["f"], t["x"], t["u"], t["plan_x"],
                                      t["plan_u"], t["wx"], t["wu"], **kw)
    for got, ref in (("dx_init", "g_x_init"), ("dC", "g_C"), ("dc", "g_c"), ("dF", "g_F"), ("df", "g_f")):
        assert rel(g[got], t[ref]) <= 1e-10, (case, got, rel(g[got], t[ref]))


@pytest.mark.parametrize("case", ["cartpole", "pendulum", "pendulum_full"])
def test_known_sweep_against_reference(case):
    t = fixture("receding_grad_known_f64", case)
    T, clamp = int(t["T"]), float(t["clamp"])
    mod, _ = episode_known_module(case)
    assert torch.equal(mod.params, t["params"])
    if case == "cartpole":
        mod.force_mag = clamp
    else:
        mod.max_torque = clamp
    B, n = t["x"].shape[1], t["x"].shape[2]
    args = (n, 1, T, t["C"], t["c"], None, None, t["x"], t["u"], t["plan_x"], t["plan_u"], t["wx"], t["wu"])
    kw = dict(u_lower=-clamp, u_upper=clamp, step=episode_known_step(mod), theta=t["params"].expand(B, -1))
    g = orc.receding_horizon_backward(*args, full_linearisation=False, **kw)
    for got, ref in (("dx_init", "g_x_init"), ("dC", "g_C"), ("dc", "g_c")):
        assert rel(g[got], t[ref]) <= 1e-10, (case, got, rel(g[got], t[ref]))
    assert rel(g["dtheta"].sum(0), t["g_params"]) <= 1e-10, (case, rel(g["dtheta"].sum(0), t["g_params"]))
    assert bool((t["plan_u"].abs() == clamp).any()) and not bool((t["plan_u"].abs() == clamp).all())
    assert float(t["g_C"].abs().max()) > 0          # the solves' adjoint reaches the cost
    # the project's convention adds the Jacobians' derivative: the same sweep otherwise
    full = orc.receding_horizon_backward(*args, **kw)
    for k in ("dx_init", "dC", "dc"):
        assert torch.equal(full[k], g[k]), k


@pytest.mark.parametrize("name,case", [("receding_grad_linear_f64", "unbounded"),
                                       ("receding_grad_linear_f64", "bounded"), ("receding_linear_f64", "")])
def test_episode_against_reference(name, case):
    """The reference's batched pnqp couples its problems (coupled=True): x, u and the iterations of every solve."""
    t = fixture(name, case)
    T, n_steps, n = int(t["T"]), int(t["n_steps"]), t["F"].shape[2]
    m = t["F"].shape[3] - n
    kw = dict(u_lower=-float(t["bound"]), u_upper=float(t["bound"])) if "bound" in t else {}
    ep = orc.receding_horizon_lin(n, m, T, n_steps, t["x_init"], t["C"], t["c"], t["F"], t["f"],
                                  lqr_iter=int(t["lqr_iter"]), eps=float(t["eps"]), coupled=True, **kw)
    assert ep.iters == t["iters"].tolist()
    assert rel(ep.x, t["x"]) <= 1e-10 and rel(ep.u, t["u"]) <= 1e-10, (rel(ep.x, t["x"]), rel(ep.u, t["u"]))
    if "plan_x" in t:
        assert rel(ep.plan_x, t["plan_x"]) <= 1e-10 and rel(ep.plan_u, t["plan_u"]) <= 1e-10
    assert torch.equal(ep.u_next[:-2], ep.plan_u[-1][1:-1]) and torch.equal(ep.u_next[-2], ep.u_next[-3])


def test_linear_inputs_forms():
    """The episode input forms hold what they name.  A time-invariant input is dense here (the oracle's input) with
    every slice equal to slice 0, and named in P["time_invariant"]; its stride-0 view over time is made on the device
    (gpu_harness.episode_device_inputs), where the GPU module asserts the staged time stride."""
    T, B, n, m = 8, 5, 4, 2
    P, _ = episode_linear_inputs(1, B, T, n, m, F64, "plain", F_T=T)
    assert P["F"].shape[0] == T and P["f"].shape[0] == T - 1 and P["time_invariant"] == ()
    P, _ = episode_linear_inputs(1, B, T, n, m, F64, "plain", f_T="T")
    assert P["f"].shape[0] == T
    assert episode_linear_inputs(1, B, T, n, m, F64, "plain", f_T="none")[0]["f"] is None
    for names, F_T in ((("F",), T), (("F",), None), (("C", "c"), None)):
        P, _ = episode_linear_inputs(1, B, T, n, m, F64, "plain", F_T=F_T, time_invariant=names)
        assert P["time_invariant"] == names
        for k in names:
            assert P[k].is_contiguous() and bool((P[k] == P[k][:1]).all()), k
        assert P["F"].shape[0] == (T if F_T == T else T - 1)
    P, kw = episode_linear_inputs(1, B, T, n, m, torch.float32, "boxT")
    assert P["C"].dtype == F64 and torch.equal(P["C"], P["C"].float().double())
    assert kw["delta_u"] == 0.125 and bool((kw["u_lower"] < 0).all() and (kw["u_upper"] > 0).all())
    _, kw = episode_linear_inputs(1, B, T, n, m, F64, "mask")
    assert kw["u_zero_I"].dtype == torch.bool and 0 < int(kw["u_zero_I"].sum()) < kw["u_zero_I"].numel()


def test_epgrad_launches():
    """epgrad_record: init, stage, accumulate; a known system's linearisation and VJP; the adjoint's route."""
    assert epgrad_launches("fused", False) == 5
    assert epgrad_launches("three_gains", False) == 8
    assert epgrad_launches("three_shape", True) == 10


@pytest.mark.parametrize("case", ["cartpole", "pendulum", "pendulum_full"])
def test_known_inputs_reach_the_clamp_scale(case):
    """The known cases' problem: the module's own cost, states on the unit circle, and a bound at the clamp."""
    mod, n, m, P, kw, dyn, theta = episode_known_inputs(case, 7, 10, F64, 3)
    assert P["C"].shape == (10, 7, n + m, n + m) and kw["u_upper"] == -kw["u_lower"] > 0
    ic = 2 if case == "cartpole" else 0
    assert torch.allclose(P["x0"][:, ic] ** 2 + P["x0"][:, ic + 1] ** 2, torch.ones(7, dtype=F64))
    assert dyn[0] == mod.mpcb200_kind and tuple(theta.tolist()) == tuple(dyn[1][:theta.numel()])
