"""CPU: the learned model's oracle (oracle/mlp_oracle.py) against the reference's NNDynamics fixtures; the network
entries (mpcb200_mlp_*, mpcb200_ilqr_mlp_*) refuse malformed arguments with status codes before they touch a device,
size their workspaces and answer mpcb200_mlp_fits without one; and which networks MPC.forward runs in the kernels,
decided on tensor metadata alone (FakeTensor CUDA tensors: no device, no kernel)."""
import ctypes

import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode

from mpc.pytorch_b200 import _lib, control, solver
from mpc.pytorch_b200._lib import Dims, IlqrOpts, Mlp, Params
from mpc.pytorch_b200.models import NNDynamics
from mpc.pytorch_b200.solver import MPC, CtrlPassthroughDynamics, GradMethods, QuadCost
from oracle import mlp_oracle as mo
from tests.helpers import build_net, load_golden, maxdiff


# ------------------------------------------------------------------------------------------------------------------
# the oracle against the reference's fixtures
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("act", ["sigmoid", "relu"])
def test_oracle_step_and_jacobian_match_the_reference(act):
    g = load_golden(f"nn_dynamics_{act}_f64")
    layers = mo.layers_of(build_net(g, act))
    nxt = mo.step(layers, act, True, g["step_x"], g["step_u"])
    R, S = mo.jacobian(layers, act, True, g["step_x"], g["step_u"])
    assert maxdiff(nxt, g["step_next"]) < 1e-13
    assert maxdiff(R, g["R"]) < 1e-13 and maxdiff(S, g["S"]) < 1e-13


@pytest.mark.parametrize("act", ["sigmoid", "relu"])
@pytest.mark.parametrize("bounded", [False, True])
def test_oracle_ilqr_matches_the_reference_trajectories(act, bounded):
    g = load_golden(f"nn_dynamics_{act}_f64")
    layers = mo.layers_of(build_net(g, act))
    kw = dict(u_lower=-0.6, u_upper=0.6) if bounded else {}
    x, u, costs, _ = mo.ilqr(3, 2, 8, g["x_init"], g["C"], g["c"], layers, act, True, lqr_iter=12, eps=1e-6, **kw)
    sfx = "" if bounded else "_free"
    tol = 2e-4 if bounded else 1e-7                    # bounded: the reference's batched pnqp stops at |dx| < 1e-4
    sc = max(1.0, float(g["x" + sfx].abs().max()))
    assert maxdiff(u, g["u" + sfx]) < tol * sc and maxdiff(x, g["x" + sfx]) < tol * sc
    cs = max(1.0, float(g["costs" + sfx].abs().max()))
    assert maxdiff(costs, g["costs" + sfx]) < (1e-5 if bounded else 1e-9) * cs


@pytest.mark.parametrize("name,slew", [("nn_grad_f64", None), ("nn_grad_slew_f64", 1.0)])
def test_oracle_ilqr_matches_the_gradient_fixtures(name, slew):
    """The reference's constrained solves of test_lqr_backward_cost_nn_dynamics_module_constrained[_slew], with the
    slew-rate penalty's augmented problem over [u_{t-1}; x] (n_prev = m)."""
    g = load_golden(name)
    nl = int(g["n_layers"])
    layers = [(g[f"W{i}"], g[f"b{i}"]) for i in range(nl)]
    T, n, m = g["C"].shape[0], 2, 2
    C, c, x0, n_prev = g["C"], g["c"], g["x_init"], 0
    if slew is not None:
        ctrl = MPC(n, m, T, slew_rate_penalty=slew)
        _, C, c, _, _, _, x0 = ctrl._slew_augment(x0, C, c, None, None)
        n_prev = m
    x, u, _, _ = mo.ilqr(n + n_prev, m, T, x0, C, c, layers, "sigmoid", True, u_lower=-1.0, u_upper=1.0, lqr_iter=40,
                         max_linesearch_iter=1, n_prev=n_prev)
    assert maxdiff(u, g["u"]) < 2e-4 and maxdiff(x[:, :, n_prev:], g["x"]) < 2e-4 * max(1.0, float(g["x"].abs().max()))


def test_oracle_linearisation_under_a_slew_rate_penalty_is_the_augmented_one():
    g = load_golden("nn_dynamics_sigmoid_f64")
    layers = mo.layers_of(build_net(g, "sigmoid"))
    x, u = g["x"], g["u"]
    F, f = mo.linearize(layers, "sigmoid", True, x, u)
    prev = torch.cat((torch.zeros(1, 4, 2, dtype=torch.float64), u[:-1]))
    F2, f2 = mo.linearize(layers, "sigmoid", True, torch.cat((prev, x), 2), u, n_prev=2)
    assert torch.equal(F2[:, :, 2:, 2:5], F[:, :, :, :3]) and torch.equal(F2[:, :, 2:, 5:], F[:, :, :, 3:])
    assert torch.equal(F2[:, :, :2, 5:], torch.eye(2, dtype=torch.float64).expand(7, 4, 2, 2))
    assert not F2[:, :, :2, :5].any() and not F2[:, :, 2:, :2].any()
    assert torch.equal(f2[:, :, 2:], f) and not f2[:, :, :2].any()


# ------------------------------------------------------------------------------------------------------------------
# status codes, workspaces and the fit, without a device
# ------------------------------------------------------------------------------------------------------------------
FAKE = 1 << 20          # a non-NULL, 256-byte aligned address that is never dereferenced: every call below fails first


def _rec(widths=(5, 100, 3), act=0, n_prev=0, params=FAKE):
    r = Mlp(n_layers=len(widths) - 1, activation=act, passthrough=1, n_prev=n_prev, params=params)
    o = 0
    for i, w in enumerate(widths):
        r.width[i] = w
    for i in range(len(widths) - 1):
        r.W_off[i] = o
        o += widths[i + 1] * widths[i]
        r.b_off[i] = o
        o += widths[i + 1]
    return r


def _nparams(widths):
    return sum(widths[i + 1] * (widths[i] + 1) for i in range(len(widths) - 1))


def _fits(widths, esz, **kw):
    return _lib.lib().mpcb200_mlp_fits(ctypes.byref(_rec(widths, **kw)), esz)


def _smem(widths, esz, n_prev=0):
    """The fit's formula: an mbarrier, the parameters, and one warp's buffers (the larger of the linearisation's
    forward pass and two Jacobian blocks, and the line search's two activation buffers and staged problem)."""
    L, ns, maxw = len(widths) - 1, widths[-1], max(widths)
    lin = widths[0] + sum(widths[1:-1]) + ns + (2 * ns * maxw if L > 1 else 0)
    ls = 2 * maxw + n_prev + widths[0] + 16
    per_warp = (max(lin, ls) + 3) // 4 * 4
    return 16 + (_nparams(widths) * esz + 15) // 16 * 16 + per_warp * esz


LIMIT = 227 * 1024


@pytest.mark.parametrize("esz", [4, 8])
def test_fits_is_the_shared_memory_formula_at_its_edge(esz):
    assert _fits((5, 100, 3), esz) == 1 and _fits((6, 256, 5), esz) == 1
    # a square hidden layer of width h: find the widest that fits, check the formula on both sides of the edge
    widths = lambda h: (6, h, h, 5)                    # noqa: E731
    fitting = [h for h in range(1, 257) if _smem(widths(h), esz) <= LIMIT]
    h = max(fitting)
    assert h < 256
    assert _fits(widths(h), esz) == 1 and _fits(widths(h + 1), esz) == 0
    assert _fits((6, 256, 256, 5), 4) == 0
    for w in [(6, 12, 12, 12, 5), (6, 100, 5), (4, 3)]:
        assert _fits(w, esz) == int(_smem(w, esz) <= LIMIT)


def test_fits_refuses_malformed_records():
    assert _fits((5, 100, 3), 2) == 0                           # element size
    assert _fits((5, 100, 3), 4, act=3) == 0                    # activation
    assert _fits((5, 100, 3), 4, n_prev=1) == 0                 # n_prev must be 0 or m
    assert _fits((5, 100, 3), 4, n_prev=2) == 1
    assert _fits((5, 257, 3), 4) == 0                           # width
    five = _rec((5, 4, 4, 4, 3))
    five.n_layers = 5                                           # five layers
    assert _lib.lib().mpcb200_mlp_fits(ctypes.byref(five), 4) == 0
    assert _fits((3, 3, 3), 4) == 0                             # no control (width[0] = n)
    assert _fits((5, 100, 3), 4, params=None) == 0
    assert _lib.lib().mpcb200_mlp_fits(None, 4) == 0


def _dims(B=4, T=5, n=3, m=2, **kw):
    f = dict(F_T=T - 1, has_f=1, bounds_kind=0, has_zero_mask=0, has_delta_u=0, max_ls_iter=10, pnqp_max_iter=20,
             do_rollout=0)
    f.update(kw)
    return Dims(B=B, T=T, n=n, m=m, **f)


def _up256(v):
    return (v + 255) // 256 * 256


def test_rollout_and_linearize_status_codes():
    L, r = _lib.lib(), _rec()
    for sfx in ("f32", "f64"):
        ro, li = getattr(L, "mpcb200_mlp_rollout_" + sfx), getattr(L, "mpcb200_mlp_linearize_" + sfx)
        assert ro(None, 4, 5, 3, 2, FAKE, FAKE, FAKE, None) == 1
        assert ro(ctypes.byref(r), 4, 5, 3, 2, None, FAKE, FAKE, None) == 1
        assert ro(ctypes.byref(r), 4, 5, 3, 2, FAKE, FAKE, None, None) == 1
        assert ro(ctypes.byref(r), 0, 5, 3, 2, FAKE, FAKE, FAKE, None) == 2
        assert ro(ctypes.byref(r), 4, 5, 2, 2, FAKE, FAKE, FAKE, None) == 2      # N below the network's n
        assert ro(ctypes.byref(r), 4, 5, 3, 1, FAKE, FAKE, FAKE, None) == 2      # M below its m
        assert ro(ctypes.byref(r), 4, 5, 3 + 17, 2, FAKE, FAKE, FAKE, None) == 2  # padding past the slack
        assert li(ctypes.byref(r), 4, 5, 3, 2, FAKE, FAKE, None, FAKE, None) == 1
        assert li(ctypes.byref(r), 4, 5, 3, 2, FAKE, None, FAKE, FAKE, None) == 1
        assert li(ctypes.byref(r), 4, 1, 3, 2, FAKE, FAKE, None, None, None) == 0   # T = 1: nothing to do
        assert li(ctypes.byref(_rec(act=7)), 4, 5, 3, 2, FAKE, FAKE, FAKE, FAKE, None) == 2


def _step(dims, ptrs=None, rec=None, ws_bytes=1 << 30, sfx="f32"):
    p = Params(u_lo=0, u_hi=0, delta_u=0, ls_decay=0.2)
    r = _rec() if rec is None else rec
    if ptrs is None:
        ptrs = [FAKE] * 19
    return getattr(_lib.lib(), "mpcb200_mlp_step_" + sfx)(ctypes.byref(dims), ctypes.byref(p), ctypes.byref(r), *ptrs,
                                                          ws_bytes, None)


def test_step_status_codes_and_workspace():
    L, d = _lib.lib(), _dims()
    for k in (0, 1, 2, 3, 4, 5, 6, 10, 11, 12, 13, 18):       # C c F f x_init cur_x cur_u new_x new_u costs alphas ws
        ptrs = [FAKE] * 19
        ptrs[k] = None
        assert _step(d, ptrs) == 1, k
    assert _step(_dims(bounds_kind=2), [FAKE] * 7 + [None] + [FAKE] * 11) == 1
    assert _step(_dims(has_delta_u=1)) == 2
    assert _step(_dims(dynamics_kind=1)) == 2
    assert _step(_dims(max_ls_iter=0)) == 2
    assert _step(_dims(n=2)) == 2
    need = L.mpcb200_mlp_step_workspace_bytes(ctypes.byref(d), 4)
    assert need == _up256(5 * 4 * 2 * 3 * 4) + _up256(5 * 4 * 2 * 4)
    assert L.mpcb200_mlp_step_workspace_bytes(ctypes.byref(d), 8) == _up256(5 * 4 * 2 * 3 * 8) + _up256(5 * 4 * 2 * 8)
    assert L.mpcb200_mlp_step_workspace_bytes(ctypes.byref(d), 3) == 0
    assert _step(d, ws_bytes=need - 1) == 2
    assert _step(d, [FAKE] * 18 + [FAKE + 16], ws_bytes=need) == 2
    assert _step(d, rec=_rec((6, 256, 256, 5))) == 2                         # (n, m) of the network is (5, 1)
    assert _step(_dims(n=5, m=1), rec=_rec((6, 256, 256, 5))) == 4          # does not fit


def _ilqr(dims, opts, ptrs=None, ws_bytes=1 << 30, rec=None, sfx="f32"):
    p = Params(u_lo=0, u_hi=0, delta_u=0, ls_decay=0.2)
    r = _rec() if rec is None else rec
    if ptrs is None:
        ptrs = [FAKE] * 13
    return getattr(_lib.lib(), "mpcb200_ilqr_mlp_" + sfx)(ctypes.byref(dims), ctypes.byref(p),
                                                          ctypes.byref(opts) if opts is not None else None,
                                                          ctypes.byref(r), *ptrs, ws_bytes, None)


def test_ilqr_status_codes_and_workspace():
    L = _lib.lib()
    d, o = _dims(do_rollout=1, has_f=0), IlqrOpts(lqr_iter=10, not_improved_lim=5, m_ref=2, eps=1e-7,
                                                  best_cost_eps=1e-4)
    assert _ilqr(d, None) == 1
    for k in (0, 1, 2, 7, 8, 9, 10, 11, 12):                   # C c x_init best_x best_u costs fdn info workspace
        ptrs = [FAKE] * 13
        ptrs[k] = None
        assert _ilqr(d, o, ptrs) == 1, k
    assert _ilqr(_dims(T=1), o) == 2
    assert _ilqr(_dims(dynamics_kind=2), o) == 2
    assert _ilqr(d, IlqrOpts(lqr_iter=0, m_ref=2)) == 2
    plain = L.mpcb200_ilqr_workspace_bytes(ctypes.byref(d), ctypes.byref(o), 4)
    need = L.mpcb200_ilqr_mlp_workspace_bytes(ctypes.byref(d), ctypes.byref(o), 4)
    B, T, n, m = 4, 5, 3, 2
    lin = _up256((T - 1) * B * n * (n + m) * 4) + _up256((T - 1) * B * n * 4)
    gains = _up256(T * B * m * n * 4) + _up256(T * B * m * 4)
    assert need in (plain + lin, plain + lin + gains)
    assert L.mpcb200_ilqr_mlp_workspace_bytes(ctypes.byref(_dims(T=1)), ctypes.byref(o), 4) == 0
    assert _ilqr(d, o, ws_bytes=need - 1) == 2
    assert _ilqr(d, o, [FAKE] * 12 + [FAKE + 16], ws_bytes=need) == 2


# ------------------------------------------------------------------------------------------------------------------
# routing
# ------------------------------------------------------------------------------------------------------------------
T, B = 6, 3


@pytest.fixture
def fake():
    with FakeTensorMode(allow_non_fake_inputs=True) as mode:
        yield mode


def _on(net, dtype=torch.float32, device="cuda"):
    for fc in net.fcs:          # fresh parameters (FakeTensor CUDA ones inside `fake`)
        fc.weight = torch.nn.Parameter(torch.zeros(fc.weight.shape, dtype=dtype, device=device))
        fc.bias = torch.nn.Parameter(torch.zeros(fc.bias.shape, dtype=dtype, device=device))
    return net


def _net(n=3, m=2, hidden=(12,), dtype=torch.float32, device="cuda", **kw):
    return _on(NNDynamics(n, m, hidden_sizes=hidden, **kw), dtype, device)


def _problem(n=3, m=2, dtype=torch.float32, device="cuda"):
    C = torch.zeros(T, B, n + m, n + m, dtype=dtype, device=device)
    c = torch.zeros(T, B, n + m, dtype=dtype, device=device)
    x0 = torch.zeros(B, n, dtype=dtype, device=device)
    u = torch.zeros(T, B, m, dtype=dtype, device=device)
    return QuadCost(C, c), x0, u


def _loop(ctrl, cost, dx, x0, u):
    return solver._use_device_loop(ctrl, x0, cost, dx, u) or solver._use_slew_device_loop(ctrl, x0, cost, dx, u)


def test_a_network_takes_the_kernels(fake):
    cost, x0, u = _problem()
    for dtype in (torch.float32, torch.float64):
        c2, x2, u2 = _problem(dtype=dtype)
        for act in ("sigmoid", "relu", "elu"):
            net = _net(dtype=dtype, activation=act)
            assert _loop(MPC(3, 2, T), c2, net, x2, u2)
            assert _loop(MPC(3, 2, T, grad_method=GradMethods.AUTO_DIFF, u_lower=-1.0, u_upper=1.0), c2, net, x2, u2)
            assert _loop(MPC(3, 2, T, slew_rate_penalty=0.1), c2, net, x2, u2)
            assert MPC(3, 2, T)._mlp_on_device(net, x2)
    assert _loop(MPC(3, 2, T), cost, _net(hidden=()), x0, u)
    assert _loop(MPC(3, 2, T), cost, _net(hidden=(100, 100, 12), passthrough=False), x0, u)
    assert _loop(MPC(5, 1, T), _problem(5, 1)[0], _net(5, 1, hidden=(256,)), *_problem(5, 1)[1:])


def test_each_disqualifier_keeps_the_module_path(fake):
    cost, x0, u = _problem()

    class Sub(NNDynamics):
        def forward(self, x, u):
            return super().forward(x, u)
    sub = _on(Sub(3, 2, hidden_sizes=(12,)))
    assert not _loop(MPC(3, 2, T), cost, sub, x0, u)                                   # a subclass
    assert not _loop(MPC(3, 2, T), cost, _net(device="cpu"), x0, u)                    # CPU weights
    mixed = _net()
    mixed.fcs[0].bias = torch.nn.Parameter(torch.zeros(12, dtype=torch.float64, device="cuda"))
    assert not _loop(MPC(3, 2, T), cost, mixed, x0, u)                                 # mixed dtypes
    assert not _loop(MPC(3, 2, T), cost, _net(dtype=torch.float64), x0, u)             # not x's dtype
    assert not _loop(MPC(5, 1, T), _problem(5, 1)[0], _net(5, 1, hidden=(256, 256)), *_problem(5, 1)[1:])  # too big
    assert not _loop(MPC(3, 2, T, grad_method=GradMethods.FINITE_DIFF), cost, _net(), x0, u)
    assert not MPC(3, 2, T, grad_method=GradMethods.FINITE_DIFF)._mlp_on_device(_net(), x0)
    assert not _loop(MPC(2, 2, T), _problem(2, 2)[0], _net(), *_problem(2, 2)[1:])     # another (n, m)
    from mpc.pytorch_b200.mlp import on_device
    assert on_device(CtrlPassthroughDynamics(_net()), 5, 2, x0)
    assert not on_device(CtrlPassthroughDynamics(sub), 5, 2, x0)


def test_the_fit_counts_the_previous_control_of_a_slew_rate_penalty(fake):
    """A network at the shared-memory edge: it fits on its own, but not with the m previous-control states a slew-rate
    penalty adds to the staged problem, so the penalised solve keeps the Module path instead of failing in a kernel."""
    w0, h = 253, 224                                   # (n, m) = (1, 252), one hidden layer of 224, float32
    assert _smem((w0, h, 1), 4) <= LIMIT < _smem((w0, h, 1), 4, n_prev=w0 - 1)
    assert _fits((w0, h, 1), 4) == 1 and _fits((w0, h, 1), 4, n_prev=w0 - 1) == 0
    from mpc.pytorch_b200.mlp import on_device
    net = _net(1, w0 - 1, hidden=(h,))
    x = torch.zeros(B, 1, device="cuda")
    assert on_device(net, 1, w0 - 1, x)
    assert not on_device(CtrlPassthroughDynamics(net), w0, w0 - 1, x)


def test_episodes_with_a_network_keep_the_host_path(fake):
    """The episode graph steps its model and plant itself and has no network step: an NNDynamics model or plant keeps
    receding_horizon's host loop, whose solves take MPC.forward's device loop."""
    cost, x0, u = _problem()
    net = _net()
    assert solver._use_device_loop(MPC(3, 2, T), x0, cost, net, u)
    assert not control._takes_device_path(MPC(3, 2, T), x0, cost, net, u)
    assert not control._takes_device_path(MPC(3, 2, T, slew_rate_penalty=0.1), x0, cost, net, u)
    from mpc.pytorch_b200.solver import LinDx
    F = torch.zeros(T - 1, B, 3, 5, device="cuda")
    assert control._takes_device_path(MPC(3, 2, T), x0, cost, LinDx(F, None), u)
    assert not control._takes_device_path(MPC(3, 2, T), x0, cost, LinDx(F, None), u, plant=net)
