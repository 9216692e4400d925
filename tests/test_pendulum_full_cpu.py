"""CPU: the five-parameter pendulum, PendulumDx(simple=False) (kind DYN_PENDULUM_FULL).  Its parameter check, the
kind tables and the dynamics-only step instance it runs on, the status codes and shape checks of its kernel calls
(raised before any launch), MPC.forward's route decisions on tensor metadata alone (FakeTensor CUDA tensors), and the
torch module and the oracle's nonlinear line-search rollout against fixtures of the reference
(oracle/make_golden_pendulum_full.py: damping and gravity bias non-zero, dt and the torque clamp changed)."""
import ctypes
import os
import re

import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode

from mpc.pytorch_b200 import _lib, solver
from mpc.pytorch_b200._lib import Dims, IlqrOpts, MpcB200Error, Params
from mpc.pytorch_b200.dynamics import (DYN_CTRL_PASSTHROUGH, DYN_DIMS, DYN_LINEAR, DYN_NPARAMS, DYN_OWN_INSTANCE,
                                       DYN_PENDULUM, DYN_PENDULUM_FULL, PendulumDx, dyn_linearize_raw,
                                       dyn_linearize_vjp_raw, dyn_rollout_raw, known_kind)
from mpc.pytorch_b200.solver import MPC, CtrlPassthroughDynamics, GradMethods, QuadCost
from oracle import lqr_oracle as orc
from tests.helpers import load_golden, maxdiff

PF, PFP = DYN_PENDULUM_FULL, DYN_PENDULUM_FULL | DYN_CTRL_PASSTHROUGH
F64 = torch.float64
FAKE = 1 << 20          # a non-NULL, 256-byte aligned address that is never dereferenced: every call below fails first
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "mpc", "pytorch_b200", "csrc")


def _module(g, params=None):
    dx = PendulumDx(params=g["params"].clone() if params is None else params, simple=False)
    dx.dt = float(g["dt"])
    dx.max_torque = float(g["clamp"])
    return dx


def _jacobians(module, xs, us):
    xs = xs.clone().requires_grad_(True)
    us = us.clone().requires_grad_(True)
    nx = module(xs, us)
    rows = [torch.autograd.grad(nx[:, j].sum(), [xs, us], retain_graph=True) for j in range(nx.shape[1])]
    return nx.detach(), torch.stack([r[0] for r in rows], 1), torch.stack([r[1] for r in rows], 1)


# ------------------------------------------------------------------------------------------------------------------
# the module and the kind tables
# ------------------------------------------------------------------------------------------------------------------
def test_parameter_count_is_checked():
    for bad in ((10.0, 1.0, 1.0), (10.0, 1.0, 1.0, 0.0), (10.0, 1.0, 1.0, 0.0, 0.0, 0.0)):
        with pytest.raises(ValueError, match="5 params"):
            PendulumDx(params=torch.tensor(bad), simple=False)
    dx = PendulumDx(simple=False)
    assert dx.params.tolist() == [10.0, 1.0, 1.0, 0.0, 0.0] and dx.mpcb200_kind == PF and not dx.simple
    assert (dx.max_torque, dx.dt, dx.lower, dx.upper) == (2.0, 0.05, -2.0, 2.0)
    assert (dx.mpc_eps, dx.linesearch_decay, dx.max_linesearch_iter, dx.ctrl_penalty) == (1e-3, 0.2, 5, 0.001)
    simple = PendulumDx()                               # the simple form is unchanged
    assert simple.mpcb200_kind == DYN_PENDULUM and simple.params.tolist() == [10.0, 1.0, 1.0]


def test_kernel_parameters_layout():
    """(g, m, l, d, b, max_torque, dt, 0): the learnable entries first, where the VJP kernel seeds them."""
    dx = PendulumDx(params=torch.tensor((9.0, 1.5, 0.7, 0.3, -0.2), dtype=F64), simple=False)
    dx.max_torque, dx.dt = 1.25, 0.08
    assert dx.mpcb200_params() == (9.0, 1.5, 0.7, 0.3, -0.2, 1.25, 0.08, 0.0)
    assert CtrlPassthroughDynamics(dx).mpcb200_params() == dx.mpcb200_params()


def test_kind_tables():
    assert DYN_DIMS[PF] == (3, 1) and DYN_DIMS[PFP] == (4, 1)
    assert DYN_NPARAMS[PF] == 5 and PFP not in DYN_NPARAMS
    assert PF & DYN_CTRL_PASSTHROUGH == 0 and PF not in (DYN_LINEAR, DYN_PENDULUM)
    # the dynamics-only instances compiled into the library are exactly the kinds that run on their own instance
    with open(os.path.join(CSRC, "dyn_instances.def")) as fh:
        compiled = {int(k): (int(n), int(m)) for k, n, m in
                    re.findall(r"^MPCB200_DYN_INST\((\d+),\s*(\d+),\s*(\d+)\)", fh.read(), re.M)}
    assert set(compiled) == set(DYN_OWN_INSTANCE)
    assert all(DYN_DIMS[k] == nm for k, nm in compiled.items())
    wrapped = CtrlPassthroughDynamics(PendulumDx(simple=False))
    assert wrapped.mpcb200_kind == PFP and (wrapped.n_state, wrapped.n_ctrl) == (4, 1)
    with FakeTensorMode(allow_non_fake_inputs=True):
        t = torch.zeros(3, 4, dtype=F64, device="cuda")
    assert known_kind(wrapped, 4, 1, t)[0] == PFP
    assert known_kind(PendulumDx(simple=False), 3, 1, t[:, :3])[0] == PF


def test_simple_form_is_the_full_form_with_no_damping_and_no_bias():
    """With d = b = 0 the two forms agree on the unit circle up to rounding (the full form takes sin(atan2(s, c)),
    the simple one s), and differ off it."""
    g = torch.Generator().manual_seed(3)
    th = (torch.rand(50, generator=g, dtype=F64) * 2 - 1) * 3.1
    x = torch.stack((th.cos(), th.sin(), torch.randn(50, generator=g, dtype=F64)), 1)
    u = torch.randn(50, 1, generator=g, dtype=F64)
    full = PendulumDx(params=torch.tensor((9.0, 1.2, 0.8, 0.0, 0.0), dtype=F64), simple=False)
    simple = PendulumDx(params=torch.tensor((9.0, 1.2, 0.8), dtype=F64))
    assert maxdiff(full(x, u), simple(x, u)) <= 1e-13
    assert maxdiff(full(3 * x, u), simple(3 * x, u)) > 1e-3


# ------------------------------------------------------------------------------------------------------------------
# the C ABI and the instance choice
# ------------------------------------------------------------------------------------------------------------------
def _dims(B=4, T=5, n=3, m=1, **kw):
    return Dims(B=B, T=T, n=n, m=m, F_T=T - 1, has_f=0, bounds_kind=0, has_zero_mask=0, has_delta_u=0,
                max_ls_iter=10, pnqp_max_iter=20, do_rollout=1, **kw)


def test_step_picks_the_dynamics_instance_of_the_kind(monkeypatch):
    """A (3, 1) call of DYN_PENDULUM_FULL runs its own instance, not the (3, 1) LinDx instance (whose line search
    would run the simple pendulum); its passthrough runs the (4, 1) one; no other shape has an instance."""
    from mpc.pytorch_b200.step import _pick_instance
    assert _pick_instance(3, 1, 8, PF) == (3, 1) and _pick_instance(3, 1, 4, PF) == (3, 1)
    assert _pick_instance(4, 1, 8, PFP) == (4, 1) and _pick_instance(4, 1, 4, PFP) == (4, 1)
    for n, kind in ((4, PF), (2, PF), (3, PFP), (5, PFP)):
        with pytest.raises(MpcB200Error):
            _pick_instance(n, 1, 8, kind)
    L = _lib.lib()
    # the gain store: the instance's own answer.  Under MPCB200_KERNEL=3 an (n, m) call runs the large-shape kernels,
    # which keep their gains in Ks/ks; a kind with its own instance does not.
    for kind, n in ((PF, 3), (PFP, 4)):
        for esz in (4, 8):
            assert L.mpcb200_step_smem_bytes(ctypes.byref(_dims(T=20, n=n, dynamics_kind=kind)), esz) > 0
            assert L.mpcb200_step_prefers_workspace(ctypes.byref(_dims(T=20, n=n, dynamics_kind=kind)), esz) == 0
            assert L.mpcb200_step_prefers_workspace(ctypes.byref(_dims(T=4096, n=n, dynamics_kind=kind)), esz) == 1
    monkeypatch.setenv("MPCB200_KERNEL", "3")
    assert L.mpcb200_step_prefers_workspace(ctypes.byref(_dims(T=20, dynamics_kind=DYN_PENDULUM)), 8) == 1
    assert L.mpcb200_step_prefers_workspace(ctypes.byref(_dims(T=20, dynamics_kind=PF)), 8) == 0


def test_argument_errors_are_status_codes():
    L = _lib.lib()
    p = Params(u_lo=0, u_hi=0, delta_u=0, ls_decay=0.2)
    # a shape the kind has no instance at
    for n, kind in ((4, PF), (3, PFP)):
        assert L.mpcb200_lqr_step_f64(ctypes.byref(_dims(n=n, dynamics_kind=kind)), ctypes.byref(p),
                                      *([FAKE] * 21), None) == 3          # MPCB200_ERR_UNSUPPORTED_DIMS
        o = IlqrOpts(lqr_iter=10, not_improved_lim=5, m_ref=1, eps=1e-7, best_cost_eps=1e-4)
        assert L.mpcb200_ilqr_f64(ctypes.byref(_dims(n=n, dynamics_kind=kind)), ctypes.byref(p), ctypes.byref(o),
                                  *([FAKE] * 15), 0, None) == 2            # MPCB200_ERR_BAD_DIMS
    dyn = (ctypes.c_double * 8)(*([1.0] * 8))
    # the VJP takes the system, not its passthrough; a bad batch is a dimension error
    assert L.mpcb200_dyn_linearize_vjp_f64(PFP, dyn, 4, 5, *([FAKE] * 6), None) == 2
    assert L.mpcb200_dyn_linearize_vjp_f64(PF, dyn, 0, 5, *([FAKE] * 6), None) == 2
    for fn in ("mpcb200_dyn_rollout_f64", "mpcb200_dyn_linearize_f64"):
        for kind in (PF, PFP):
            assert getattr(L, fn)(kind, dyn, 0, 5, *([FAKE] * (3 if "rollout" in fn else 4)), None) == 2


BAD_SHAPES = [(PF, (6, 5), (4, 6, 1), "x_init"), (PF, (6, 3), (4, 6, 2), "u"), (PF, (6, 3), (3, 6, 1), "u"),
              (PFP, (6, 3), (4, 6, 1), "x_init"), (PFP, (6, 4), (4, 5, 1), "u")]


@pytest.mark.parametrize("kind,xs,us,what", BAD_SHAPES, ids=[f"{c[0]}-{c[3]}-{i}" for i, c in enumerate(BAD_SHAPES)])
def test_dyn_calls_check_shapes_before_launch(kind, xs, us, what):
    T, prm = 4, (1.0,) * 8
    with pytest.raises(MpcB200Error, match=what):
        dyn_rollout_raw(kind, prm, T, torch.zeros(xs, dtype=F64), torch.zeros(us, dtype=F64))
    with pytest.raises(MpcB200Error, match="x" if what == "x_init" else what):
        dyn_linearize_raw(kind, prm, T, torch.zeros((T,) + xs, dtype=F64), torch.zeros(us, dtype=F64))


@pytest.mark.parametrize("kind", [PF, PFP])
def test_dyn_calls_refuse_cpu_tensors(kind):
    n, _ = DYN_DIMS[kind]
    B, T = 3, 5
    x0, x, u = torch.zeros(B, n, dtype=F64), torch.zeros(T, B, n, dtype=F64), torch.zeros(T, B, 1, dtype=F64)
    with pytest.raises(MpcB200Error, match="CUDA tensors only"):
        dyn_rollout_raw(kind, (1.0,) * 8, T, x0, u)
    with pytest.raises(MpcB200Error, match="CUDA tensors only"):
        dyn_linearize_raw(kind, (1.0,) * 8, T, x, u)
    dF, df = torch.zeros(T - 1, B, n, n + 1, dtype=F64), torch.zeros(T - 1, B, n, dtype=F64)
    if kind == PF:
        with pytest.raises(MpcB200Error, match="CUDA tensors only"):
            dyn_linearize_vjp_raw(kind, (1.0,) * 8, T, x, u, dF, df)
        with pytest.raises(MpcB200Error, match="dF: expected shape"):
            dyn_linearize_vjp_raw(kind, (1.0,) * 8, T, x, u, dF[..., :3], df)
    else:
        with pytest.raises(MpcB200Error, match="passthrough"):
            dyn_linearize_vjp_raw(kind, (1.0,) * 8, T, x, u, dF, df)


# ------------------------------------------------------------------------------------------------------------------
# MPC.forward's routes
# ------------------------------------------------------------------------------------------------------------------
def test_mpc_routes_take_the_kernels(monkeypatch):
    """The device loop, the slew-rate device loop and the differentiable tail's kernel linearisation take the
    five-parameter pendulum, on float32 and float64 CUDA tensors, under ANALYTIC and AUTO_DIFF."""
    T, B = 6, 3
    dx = PendulumDx(params=torch.tensor((9.0, 1.2, 0.8, 0.3, 0.2)), simple=False)
    for dtype in (torch.float32, F64):
        with FakeTensorMode(allow_non_fake_inputs=True):
            C = torch.zeros(T, B, 4, 4, dtype=dtype, device="cuda")
            c = torch.zeros(T, B, 4, dtype=dtype, device="cuda")
            x0 = torch.zeros(B, 3, dtype=dtype, device="cuda")
            u = torch.zeros(T, B, 1, dtype=dtype, device="cuda")
            x = torch.zeros(T, B, 3, dtype=dtype, device="cuda")
            xa = torch.zeros(T, B, 4, dtype=dtype, device="cuda")
            prev = torch.zeros(B, 1, dtype=dtype, device="cuda")
            for gm in (GradMethods.ANALYTIC, GradMethods.AUTO_DIFF):
                ctrl = MPC(3, 1, T, grad_method=gm, u_lower=-1.0, u_upper=1.0)
                assert solver._use_device_loop(ctrl, x0, QuadCost(C, c), dx, u)
                slew = MPC(3, 1, T, grad_method=gm, slew_rate_penalty=0.1, prev_ctrl=prev)
                assert solver._use_slew_device_loop(slew, x0, QuadCost(C, c), dx, u)
            assert not solver._use_device_loop(MPC(3, 1, T, grad_method=GradMethods.FINITE_DIFF), x0,
                                               QuadCost(C, c), dx, u)
        # the linearisation reads the parameters back to the host: outside the fake mode, on fake CUDA tensors
        for gm in (GradMethods.ANALYTIC, GradMethods.AUTO_DIFF):
            for diff in (False, True):
                assert MPC(3, 1, T, grad_method=gm)._kernel_linearization(dx, x, diff)[0] == PF
            # the augmented system of a slew solve: its linearisation in the kernels, the differentiable tail on
            # the system itself
            wrapped = CtrlPassthroughDynamics(dx)
            assert MPC(4, 1, T, grad_method=gm)._kernel_linearization(wrapped, xa, False)[0] == PFP
            assert MPC(4, 1, T, grad_method=gm)._kernel_linearization(wrapped, xa, True)[0] == DYN_LINEAR


# ------------------------------------------------------------------------------------------------------------------
# the module and the oracle against the reference
# ------------------------------------------------------------------------------------------------------------------
def test_module_step_and_jacobians_match_reference():
    g = load_golden("known_step_pendulum_full_f64")
    nx, R, S = _jacobians(_module(g), g["step_x"], g["step_u"])
    assert maxdiff(nx, g["step_next"]) <= 1e-13
    assert maxdiff(R, g["R"]) <= 1e-12
    assert maxdiff(S, g["S"]) <= 1e-12
    clamp = float(g["clamp"])
    on = g["step_u"][:, 0].abs() <= clamp
    assert bool((S[~on] == 0).all()) and bool((S[on].abs().sum((1, 2)) > 0).all())
    # all five parameters act: damping and bias are not zero, and each moves the next state
    assert all(float(v) != 0 for v in g["params"])


def test_module_rollout_and_linearisation_match_reference():
    """The rollout and the reference's own AUTO_DIFF linearize_dynamics (F, f) along it."""
    g = load_golden("known_step_pendulum_full_f64")
    dx = _module(g)
    x = [g["roll_x_init"]]
    for t in range(g["roll_u"].shape[0] - 1):
        x.append(dx(x[t], g["roll_u"][t]).detach())
    x = torch.stack(x)
    assert maxdiff(x, g["roll_x"]) <= 1e-12
    T, B, n = x.shape
    nx, R, S = _jacobians(dx, x[:-1].reshape(-1, n), g["roll_u"][:-1].reshape(-1, 1))
    F = torch.cat((R, S), 2).view(T - 1, B, n, n + 1)
    f = (nx - torch.einsum("bij,bj->bi", R, x[:-1].reshape(-1, n))
         - torch.einsum("bij,bj->bi", S, g["roll_u"][:-1].reshape(-1, 1))).view(T - 1, B, n)
    assert maxdiff(F, g["roll_F"]) <= 1e-12 and maxdiff(f, g["roll_f"]) <= 1e-12
    assert bool((g["roll_u"].abs() > float(g["clamp"])).any())


@pytest.mark.parametrize("bounds", ["in", "wide"])
def test_oracle_nonlinear_rollout_matches_reference(bounds):
    g = load_golden("known_step_pendulum_full_f64")
    dx = _module(g)
    n, T = g["x"].shape[2], g["x"].shape[0]
    b = float(g[f"bound_{bounds}"])
    o = orc.lqr_step_forward(n, 1, T, g["x_init"], g["C"], g["c"], g["F"], g["f"], g["x"], g["u"],
                             u_lower=-b, u_upper=b, linesearch_decay=float(g["decay"]),
                             max_linesearch_iter=int(g["ls_iter"]), coupled=True, dynamics=dx)
    for k, got in (("new_x", o.new_x), ("new_u", o.new_u), ("costs", o.costs), ("full_du_norm", o.full_du_norm),
                   ("mean_alpha", o.mean_alphas)):
        want = torch.as_tensor(g[f"{k}_{bounds}"], dtype=F64)
        assert maxdiff(got, want) <= 1e-10 * max(1.0, float(want.abs().max())), k
    assert float(o.n_total_qp_iter) == float(g[f"n_qp_{bounds}"])
    if bounds == "wide":
        assert bool((g["new_u_wide"].abs() > float(g["clamp"])).any())
    assert float(g[f"mean_alpha_{bounds}"]) < 1.0


def test_reference_gradient_has_five_nonzero_entries():
    """The reference's params.grad of the fixture's loss: damping and bias are identifiable."""
    g = load_golden("paramgrad_pendulum_full_f64")
    for regime in ("unb", "box"):
        assert g[f"grad_{regime}"].shape == (5,) and bool((g[f"grad_{regime}"] != 0).all())
