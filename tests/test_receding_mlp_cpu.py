"""CPU: receding-horizon episodes planned with a learned model (mpcb200_episode_mlp_*,
mpcb200_episode_backward_mlp_*): the float64 oracle (oracle/receding_mlp_oracle.py) against the reference's fixture
(tests/golden/receding_nn_f64.npz, oracle/make_golden_receding_nn.py), the routing predicate mlp.episode_on_device on
each case it takes and each it leaves to the host path, the workspace formulas and the status codes, without a
device."""
import ctypes
import os

import numpy as np
import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode

from mpc.pytorch_b200 import _lib, control, mlp
from mpc.pytorch_b200._lib import Dims, IlqrOpts, Params, Plant
from mpc.pytorch_b200.dynamics import PendulumDx
from mpc.pytorch_b200.models import NNDynamics
from mpc.pytorch_b200.solver import MPC, GradMethods, LinDx, QuadCost
from oracle import lqr_oracle as lo
from oracle import mlp_oracle as mo
from oracle import receding_mlp_oracle as rmo
from tests.gpu_harness import episode_known_step

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def fixture(case):
    z = np.load(os.path.join(GOLD, "receding_nn_f64.npz"))
    pre = case + "_"
    return {k[len(pre):]: torch.from_numpy(z[k]) for k in z.files if k.startswith(pre)}


def rel(a, b):
    return float((a - b).abs().max()) / max(1.0, float(b.abs().max()))


@pytest.mark.parametrize("case", ["net", "pendulum"])
def test_oracle_matches_the_reference_fixture(case):
    """The oracle, fed the reference's plans, reproduces the fixture's x, u and every gradient to 1e-10; its own solves
    reproduce the reference's plans with the same iteration counts, to the reference's batched pnqp stopping rule
    (|dx| < 1e-4) where the bounds bind."""
    z = fixture(case)
    nl = int(z["n_layers"])
    layers = [(z[f"W{i}"], z[f"b{i}"]) for i in range(nl)]
    B, n = z["x_init"].shape
    m = z["u"].shape[2]
    T, steps, bound = int(z["T"]), int(z["n_steps"]), float(z["bound"])
    step = theta = None
    if case == "pendulum":
        mod = PendulumDx(simple=True)
        mod.max_torque = bound
        step = episode_known_step(mod)
        theta = z["params"].expand(B, -1)
    xs, us, px, pu, its = [], [], [], [], []
    for k in range(steps):           # one control step at a time from the reference's state and warm start
        u_init = None if k == 0 else lo.shift_warm_start(z["plan_u"][k - 1])
        x1, u1, p_x, p_u, it = rmo.episode(
            n, m, T, 1, z["x"][k], z["C"], z["c"], layers, "sigmoid", True,
            plant=None if step is None else (lambda x, u: step(x, u, theta)), w=z["w"][k:k + 1], u_init=u_init,
            u_lower=-bound, u_upper=bound, lqr_iter=int(z["lqr_iter"]), eps=float(z["eps"]))
        its += it
        px.append(p_x[0])
        pu.append(p_u[0])
        nxt = mo.step(layers, "sigmoid", True, z["x"][k], z["plan_u"][k][0]) if step is None else \
            step(z["x"][k], z["plan_u"][k][0], theta)
        xs.append(nxt + z["w"][k])
        us.append(z["plan_u"][k][0])
    assert its == z["iters"].tolist()
    assert rel(torch.stack(xs), z["x"][1:]) < 1e-10 and rel(torch.stack(us), z["u"]) < 1e-10
    assert rel(torch.stack(pu), z["plan_u"]) < 2e-4 and rel(torch.stack(px), z["plan_x"]) < 2e-4
    out = rmo.backward(n, m, T, z["C"], z["c"], layers, "sigmoid", True, z["x"], z["u"], z["plan_x"], z["plan_u"],
                       z["wx"], z["wu"], u_lower=-bound, u_upper=bound, plant=step, theta=theta)
    pairs = [(out["dx_init"], "x_init"), (out["dC"], "C"), (out["dc"], "c"), (out["dw"], "w")]
    pairs += [(out["dlayers"][i][j], f"{'Wb'[j]}{i}") for i in range(nl) for j in (0, 1)]
    if case == "pendulum":
        pairs.append((out["dtheta_plant"].sum(0), "params"))
    for got, name in pairs:
        assert rel(got, z["g_" + name]) < 1e-10, (name, rel(got, z["g_" + name]))


# ------------------------------------------------------------------------------------------------------------------
# routing, on FakeTensor CUDA tensors (metadata only)
T, B = 6, 3
PEND_PARAMS = torch.tensor((10.0, 1.0, 1.0))


@pytest.fixture
def fake():
    with FakeTensorMode(allow_non_fake_inputs=True) as mode:
        yield mode


def _net(n=3, m=2, hidden=(12,), dtype=torch.float32, cls=NNDynamics, **kw):
    net = cls(n, m, hidden_sizes=hidden, **kw)
    for fc in net.fcs:
        fc.weight = torch.nn.Parameter(torch.zeros(fc.weight.shape, dtype=dtype, device="cuda"))
        fc.bias = torch.nn.Parameter(torch.zeros(fc.bias.shape, dtype=dtype, device="cuda"))
    return net


def _args(n=3, m=2, dtype=torch.float32):
    C = torch.zeros(T, B, n + m, n + m, dtype=dtype, device="cuda")
    c = torch.zeros(T, B, n + m, dtype=dtype, device="cuda")
    x0 = torch.zeros(B, n, dtype=dtype, device="cuda")
    u = torch.zeros(T, B, m, dtype=dtype, device="cuda")
    return QuadCost(C, c), x0, u


def test_episode_on_device_takes_each_in_case(fake):
    for dtype in (torch.float32, torch.float64):
        cost, x0, u = _args(dtype=dtype)
        net = _net(dtype=dtype)
        for gm in (GradMethods.ANALYTIC, GradMethods.AUTO_DIFF):
            ctrl = MPC(3, 2, T, grad_method=gm)
            for diff in (False, True):
                assert mlp.episode_on_device(ctrl, x0, cost, net, u, None, differentiable=diff)
                assert mlp.episode_on_device(ctrl, x0, cost, net, u, net, differentiable=diff)     # w, no plant
                F = torch.zeros(1, B, 3, 5, dtype=dtype, device="cuda")
                assert mlp.episode_on_device(ctrl, x0, cost, net, u, LinDx(F, None), differentiable=diff)
        cost1, x1, u1 = _args(3, 1, dtype)
        pend = PendulumDx(params=PEND_PARAMS)
        pend.mpcb200_params = lambda: (10.0, 1.0, 1.0)     # metadata only: no read of a FakeTensor's values
        assert mlp.episode_on_device(MPC(3, 1, T), x1, cost1, _net(3, 1, dtype=dtype), u1, pend, differentiable=True)


def test_episode_on_device_leaves_each_out_case(fake):
    cost, x0, u = _args()
    net = _net()
    assert not mlp.episode_on_device(MPC(3, 2, T, slew_rate_penalty=0.1), x0, cost, net, u)
    assert not mlp.episode_on_device(MPC(3, 2, T), x0, cost, net, u, time_varying=True)
    assert not mlp.episode_on_device(MPC(3, 2, T), x0, cost, net, u, _net())                   # a network plant

    class Sub(NNDynamics):
        pass
    assert not mlp.episode_on_device(MPC(3, 2, T), x0, cost, _net(cls=Sub), u)                   # a subclass
    assert not mlp.episode_on_device(MPC(3, 2, T), x0, cost, net, u, _net(cls=Sub))
    assert not mlp.episode_on_device(MPC(3, 2, T, grad_method=GradMethods.FINITE_DIFF), x0, cost, net, u)
    assert not mlp.episode_on_device(MPC(3, 2, T, verbose=1), x0, cost, net, u)
    module_cost = torch.nn.Linear(5, 1)
    assert not mlp.episode_on_device(MPC(3, 2, T), x0, module_cost, net, u)
    cost_b, x_b, u_b = _args(3, 80)
    big = _net(3, 80, hidden=(256,))
    ctrl_b = MPC(3, 80, T)
    assert mlp.episode_on_device(ctrl_b, x_b, cost_b, big, u_b) == mlp.fits(big, 0, 4)          # forward only
    assert mlp.fits(big, 0, 4) and not mlp.episode_on_device(ctrl_b, x_b, cost_b, big, u_b, differentiable=True)
    # the existing episode graph keeps its meaning: a network never takes it
    assert not control._takes_device_path(MPC(3, 2, T), x0, cost, net, u)


# ------------------------------------------------------------------------------------------------------------------
# workspace formulas and status codes (no device)
def _dims(n=3, m=2, B=4, T=8):
    return Dims(B=B, T=T, n=n, m=m, F_T=T - 1, has_f=0, bounds_kind=0, has_zero_mask=0, has_delta_u=0, max_ls_iter=10,
                pnqp_max_iter=20, do_rollout=1, dynamics_kind=0)


def _rec(n=3, m=2, hidden=(12, 10)):
    return mlp._record(NNDynamics(n, m, hidden_sizes=hidden), 0, 256)


def _up(v):
    return (v + 255) // 256 * 256


@pytest.mark.parametrize("esz", [4, 8])
def test_workspace_formulas(esz):
    L = _lib.lib()
    d, opts, rec = _dims(), IlqrOpts(lqr_iter=10, not_improved_lim=5, m_ref=2, eps=1e-7, best_cost_eps=1e-4), _rec()
    # forward: the episode's buffers after the network's iLQR workspace instead of the LinDx one
    fwd = L.mpcb200_episode_mlp_workspace_bytes(ctypes.byref(d), ctypes.byref(opts), ctypes.byref(rec), esz)
    assert fwd > 0
    assert fwd - L.mpcb200_episode_workspace_bytes(ctypes.byref(d), ctypes.byref(opts), esz) == \
        L.mpcb200_ilqr_mlp_workspace_bytes(ctypes.byref(d), ctypes.byref(opts), esz) - \
        L.mpcb200_ilqr_workspace_bytes(ctypes.byref(d), ctypes.byref(opts), esz)
    # backward: the LinDx sweep's at the linearisation's dims, then F_k, f_k, dtheta_k and the VJP's workspace
    dn = _dims()
    dn.has_f = 1
    base = L.mpcb200_episode_backward_workspace_bytes(ctypes.byref(dn), esz)
    n, P, T1B = 3, 5, 7 * 4
    n_params = 12 * 5 + 12 + 10 * 12 + 10 + 3 * 10 + 3
    want = base + _up(T1B * n * P * esz) + _up(T1B * n * esz) + _up(n_params * esz) + \
        L.mpcb200_mlp_linearize_vjp_workspace_bytes(ctypes.byref(rec), 4, 8, esz)
    assert L.mpcb200_episode_backward_mlp_workspace_bytes(ctypes.byref(d), ctypes.byref(rec), None, esz) == want
    # a LinDx plant adds nothing; a known plant its per-problem parameter part
    lin = Plant(kind=0, has_f=1)
    assert L.mpcb200_episode_backward_mlp_workspace_bytes(ctypes.byref(d), ctypes.byref(rec), ctypes.byref(lin),
                                                          esz) == want
    # 0 for what the entries do not take: T < 3, a network whose VJP (or which) does not fit, the slew-rate state
    d2 = _dims(T=2)
    assert L.mpcb200_episode_mlp_workspace_bytes(ctypes.byref(d2), ctypes.byref(opts), ctypes.byref(rec), esz) == 0
    assert L.mpcb200_episode_backward_mlp_workspace_bytes(ctypes.byref(d2), ctypes.byref(rec), None, esz) == 0
    vjp_big = mlp._record(NNDynamics(3, 80, hidden_sizes=(256,)), 0, 256)
    d80 = _dims(3, 80)
    assert L.mpcb200_episode_mlp_workspace_bytes(ctypes.byref(d80), ctypes.byref(opts), ctypes.byref(vjp_big), 4) > 0
    assert L.mpcb200_episode_backward_mlp_workspace_bytes(ctypes.byref(d80), ctypes.byref(vjp_big), None, 4) == 0
    huge = mlp._record(NNDynamics(3, 2, hidden_sizes=(256, 256)), 0, 256)
    assert L.mpcb200_episode_mlp_workspace_bytes(ctypes.byref(d), ctypes.byref(opts), ctypes.byref(huge), 8) == 0
    slew = mlp._record(NNDynamics(3, 2, hidden_sizes=(12,)), 2, 256)
    d5 = _dims(5, 2)
    assert L.mpcb200_episode_mlp_workspace_bytes(ctypes.byref(d5), ctypes.byref(opts), ctypes.byref(slew), esz) == 0
    assert L.mpcb200_episode_backward_mlp_workspace_bytes(ctypes.byref(d5), ctypes.byref(slew), None, esz) == 0


FAKE = 1 << 20          # an address the checks never dereference: every error is reported before a launch


def _fwd(d, rec, n_steps=3, nbytes=1 << 30, plant=None, **null):
    opts = IlqrOpts(lqr_iter=10, not_improved_lim=5, m_ref=2, eps=1e-7, best_cost_eps=1e-4)
    names = ["C", "c", "F_plant", "f_plant", "w", "x_init", "u_init", "u_lower", "u_upper", "u_zero_I", "xs", "us",
             "costs", "info", "u_next", "plan_x", "plan_u", "workspace"]
    optional = {"F_plant", "f_plant", "w", "u_lower", "u_upper", "u_zero_I", "plan_x", "plan_u"}
    ptrs = [None if (k in optional and k not in null) or null.get(k) == 0 else ctypes.c_void_p(FAKE) for k in names]
    return _lib.lib().mpcb200_episode_mlp_f32(ctypes.byref(d), ctypes.byref(Params()), ctypes.byref(opts),
                                              ctypes.byref(rec) if rec is not None else None,
                                              ctypes.byref(plant) if plant is not None else None, n_steps, *ptrs,
                                              nbytes, None)


def _bwd(d, rec, n_steps=3, nbytes=1 << 30, plant=None, **null):
    names = ["C", "c", "F_plant", "u_lower", "u_upper", "xs", "us", "plan_x", "plan_u", "dl_dxs", "dl_dus",
             "dx_init", "dC", "dc", "dtheta", "dF_plant", "df_plant", "dtheta_plant", "dw", "workspace"]
    optional = {"F_plant", "u_lower", "u_upper", "dF_plant", "df_plant", "dtheta_plant", "dw"}
    ptrs = [None if (k in optional and k not in null) or null.get(k) == 0 else ctypes.c_void_p(FAKE) for k in names]
    return _lib.lib().mpcb200_episode_backward_mlp_f32(ctypes.byref(d), ctypes.byref(Params()),
                                                       ctypes.byref(rec) if rec is not None else None,
                                                       ctypes.byref(plant) if plant is not None else None, n_steps,
                                                       *ptrs, nbytes, None)


NULL, BAD, SMEM, NO_DEVICE = 1, 2, 4, 6      # a well-formed call gets as far as looking for a device


def test_forward_status_codes():
    d, rec = _dims(), _rec()
    assert _fwd(d, rec) == NO_DEVICE
    assert _fwd(d, None) == NULL
    for k in ("C", "c", "x_init", "xs", "us", "costs", "info", "u_next", "workspace"):
        assert _fwd(d, rec, **{k: 0}) == NULL, k
    assert _fwd(d, rec, plan_x=1) == NULL                                  # plan_x without plan_u
    assert _fwd(_dims(T=2), rec) == BAD and _fwd(d, rec, n_steps=0) == BAD
    assert _fwd(d, rec, nbytes=0) == BAD                                   # a workspace too small
    assert _fwd(d, mlp._record(NNDynamics(3, 2, hidden_sizes=(256, 256)), 0, 256)) == SMEM
    assert _fwd(_dims(5, 2), mlp._record(NNDynamics(3, 2, hidden_sizes=(12,)), 2, 256)) == BAD      # n_prev
    assert _fwd(d, rec, plant=Plant(kind=2)) == BAD                        # a pendulum steps (3, 1), not (3, 2)
    assert _fwd(d, rec, plant=Plant(kind=0)) == NULL                       # a LinDx plant needs F_plant


def test_backward_status_codes():
    d, rec = _dims(), _rec()
    assert _bwd(d, rec) == NO_DEVICE
    assert _bwd(d, None) == NULL
    for k in ("C", "c", "xs", "us", "plan_x", "plan_u", "dl_dxs", "dl_dus", "dx_init", "dC", "dc", "dtheta",
              "workspace"):
        assert _bwd(d, rec, **{k: 0}) == NULL, k
    assert _bwd(_dims(T=2), rec) == BAD and _bwd(d, rec, n_steps=0) == BAD
    assert _bwd(d, rec, nbytes=0) == BAD
    assert _bwd(_dims(3, 80), mlp._record(NNDynamics(3, 80, hidden_sizes=(256,)), 0, 256)) == SMEM   # the VJP
    assert _bwd(d, mlp._record(NNDynamics(3, 2, hidden_sizes=(256, 256)), 0, 256)) == SMEM
    assert _bwd(d, rec, plant=Plant(kind=0, has_f=1), F_plant=1) == NULL   # dF_plant missing
    assert _bwd(d, rec, plant=Plant(kind=2)) == BAD
