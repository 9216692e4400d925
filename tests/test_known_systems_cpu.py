"""CPU: the plain-torch known systems (CartpoleDx, PendulumDx) and the oracle's nonlinear line-search rollout against
fixtures of the reference at non-default physics, the host-side parameter read, and the shape checks of the
known-system kernel calls (which raise before any launch, so they need no GPU).

Fixtures: oracle/make_golden_nn.py (known_step_cases) - the reference's env modules with non-default parameters,
dt and control clamp; one step on states at radii 0.3 / 1 / 3, theta at +-pi (both signs of sin = 0) and near 0,
controls at, one ulp inside and one ulp outside the clamp; one LQRStep with the module as true dynamics, once with
bounds inside the clamp and once with bounds twice as wide."""
import pytest
import torch

from oracle import lqr_oracle as orc
from tests.helpers import EDIT_ROUTES, load_golden, maxdiff

SYSTEMS = ("cartpole", "pendulum")


def _module(name, g, params=None):
    from mpc.pytorch_b200.dynamics import CartpoleDx, PendulumDx
    cls = CartpoleDx if name == "cartpole" else PendulumDx
    dx = cls(params=g["params"].clone() if params is None else params)
    dx.dt = float(g["dt"])
    if name == "cartpole":
        dx.force_mag = float(g["clamp"])
    else:
        dx.max_torque = float(g["clamp"])
    return dx


def _jacobians(module, xs, us):
    xs = xs.clone().requires_grad_(True)
    us = us.clone().requires_grad_(True)
    nx = module(xs, us)
    rows = [torch.autograd.grad(nx[:, j].sum(), [xs, us], retain_graph=True) for j in range(nx.shape[1])]
    return nx.detach(), torch.stack([r[0] for r in rows], 1), torch.stack([r[1] for r in rows], 1)


@pytest.mark.parametrize("name", SYSTEMS)
def test_module_step_and_jacobians_match_reference(name):
    g = load_golden(f"known_step_{name}_f64")
    nx, R, S = _jacobians(_module(name, g), g["step_x"], g["step_u"])
    assert maxdiff(nx, g["step_next"]) <= 1e-13
    assert maxdiff(R, g["R"]) <= 1e-12
    assert maxdiff(S, g["S"]) <= 1e-12
    # at the clamp (and one ulp inside) the derivative is torch.clamp's, 1; one ulp outside it is exactly 0
    clamp = float(g["clamp"])
    on = g["step_u"][:, 0].abs() <= clamp
    assert bool((S[~on] == 0).all()) and bool((S[on].abs().sum((1, 2)) > 0).all())


@pytest.mark.parametrize("bounds", ["in", "wide"])
@pytest.mark.parametrize("name", SYSTEMS)
def test_oracle_nonlinear_rollout_matches_reference(name, bounds):
    g = load_golden(f"known_step_{name}_f64")
    dx = _module(name, g)
    n, T = g["x"].shape[2], g["x"].shape[0]
    b = float(g[f"bound_{bounds}"])
    o = orc.lqr_step_forward(n, 1, T, g["x_init"], g["C"], g["c"], g["F"], g["f"], g["x"], g["u"],
                             u_lower=-b, u_upper=b, linesearch_decay=float(g["decay"]),
                             max_linesearch_iter=int(g["ls_iter"]), coupled=True, dynamics=dx)
    for k, got in (("new_x", o.new_x), ("new_u", o.new_u), ("costs", o.costs), ("full_du_norm", o.full_du_norm),
                   ("mean_alpha", o.mean_alphas)):
        want = torch.as_tensor(g[f"{k}_{bounds}"], dtype=torch.float64)      # scalars load as Python floats
        assert maxdiff(got, want) <= 1e-10 * max(1.0, float(want.abs().max())), k
    assert float(o.n_total_qp_iter) == float(g[f"n_qp_{bounds}"])
    for side in (-b, b):
        assert torch.equal(o.new_u == side, g[f"new_u_{bounds}"] == side)
    if bounds == "wide":       # the fixture exercises the clamp inside the dynamics
        assert bool((g["new_u_wide"].abs() > float(g["clamp"])).any())
    assert float(g[f"mean_alpha_{bounds}"]) < 1.0      # ... and a line search of several passes
    # the same step with the linearisation as true dynamics is a different step: the rollout is really nonlinear
    lin = orc.lqr_step_forward(n, 1, T, g["x_init"], g["C"], g["c"], g["F"], g["f"], g["x"], g["u"],
                               u_lower=-b, u_upper=b, linesearch_decay=float(g["decay"]),
                               max_linesearch_iter=int(g["ls_iter"]), coupled=True)
    assert maxdiff(lin.new_x, o.new_x) > 1e-6


# ----------------------------------------------------------------------------------------------------------------
# parameters the kernels see: what forward would use at that moment
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("route", [r[0] for r in EDIT_ROUTES])
@pytest.mark.parametrize("name", SYSTEMS)
def test_kernel_parameters_follow_in_place_edits(name, route):
    """mpcb200_params() - the values handed to the kernels - equals what forward uses after every kind of edit,
    inside and outside an MPC solve's parameter scope."""
    from mpc.pytorch_b200.dynamics import params_scope
    edit = dict(EDIT_ROUTES)[route]
    g = load_golden(f"known_step_{name}_f64")
    dx = _module(name, g, params=g["params"].clone().requires_grad_(True))
    npar = len(g["params"])
    for k in range(3):
        assert dx.mpcb200_params()[:npar] == tuple(float(v) for v in dx.params.detach())
        new = g["params"] * (1.0 + 0.1 * (k + 1)) + 0.05
        with params_scope():
            dx.mpcb200_params()
            edit(dx, new)
            got = dx.mpcb200_params()[:npar]
        now = tuple(float(v) for v in dx.params.detach())
        assert maxdiff(torch.tensor(now, dtype=torch.float64), new) <= 1e-12, route       # the edit took effect
        assert got == now, (route, got, now)
        assert dx.mpcb200_params()[:npar] == now
    # forward agrees: the module's own step with the read-back values
    clone = _module(name, g, params=torch.tensor(dx.mpcb200_params()[:npar], dtype=torch.float64))
    assert torch.equal(clone(g["step_x"], g["step_u"]), dx(g["step_x"], g["step_u"]).detach())


def test_parameter_scopes_of_two_threads_never_share_an_epoch():
    """The read-back cache lives on the module, so concurrent solves on two threads must not see each other's
    scope as their own."""
    import threading
    from mpc.pytorch_b200 import dynamics
    seen, go = [], threading.Barrier(2)

    def solve():
        with dynamics.params_scope():
            go.wait()
            seen.append(dynamics._scope.epoch)
            go.wait()

    threads = [threading.Thread(target=solve) for _ in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert len(seen) == 2 and seen[0] != seen[1]


# ----------------------------------------------------------------------------------------------------------------
# shape checks of the known-system kernel calls: raised before the CUDA check, so no launch is ever attempted
# ----------------------------------------------------------------------------------------------------------------
BAD_SHAPES = [
    # (kind, T, rollout x_init shape | linearize x shape, u shape, what the message names)
    ("cartpole", 4, (6, 3), (4, 6, 1), "x_init"),           # pendulum-sized state for the cartpole
    ("pendulum", 4, (6, 5), (4, 6, 1), "x_init"),
    ("pendulum", 4, (6, 3), (4, 6, 2), "u"),                # two controls
    ("cartpole", 4, (6, 5), (3, 6, 1), "u"),                # wrong horizon
    ("cartpole", 4, (6, 5), (4, 5, 1), "u"),                # wrong batch
    ("pendulum", 4, (3,), (4, 1, 1), "x_init"),             # no batch dimension
]


@pytest.mark.parametrize("kind,T,xs,us,what", BAD_SHAPES, ids=[f"{c[0]}-{c[4]}-{i}" for i, c in enumerate(BAD_SHAPES)])
def test_dyn_calls_check_shapes_before_launch(kind, T, xs, us, what):
    from mpc.pytorch_b200 import _lib
    from mpc.pytorch_b200.dynamics import DYN_CARTPOLE, DYN_PENDULUM, dyn_linearize_raw, dyn_rollout_raw
    k = DYN_CARTPOLE if kind == "cartpole" else DYN_PENDULUM
    prm = (1.0,) * 8
    with pytest.raises(_lib.MpcB200Error, match=what):
        dyn_rollout_raw(k, prm, T, torch.zeros(xs, dtype=torch.float64), torch.zeros(us, dtype=torch.float64))
    xl = (T,) + tuple(xs)
    with pytest.raises(_lib.MpcB200Error, match="x" if what == "x_init" else what):
        dyn_linearize_raw(k, prm, T, torch.zeros(xl, dtype=torch.float64), torch.zeros(us, dtype=torch.float64))


@pytest.mark.parametrize("kind", ["cartpole", "pendulum"])
def test_dyn_calls_refuse_cpu_tensors_and_unknown_kinds(kind):
    from mpc.pytorch_b200 import _lib
    from mpc.pytorch_b200.dynamics import DYN_DIMS, DYN_CARTPOLE, DYN_PENDULUM, dyn_linearize_raw, dyn_rollout_raw
    k = DYN_CARTPOLE if kind == "cartpole" else DYN_PENDULUM
    n, _ = DYN_DIMS[k]
    B, T = 3, 5
    x0, x = torch.zeros(B, n, dtype=torch.float64), torch.zeros(T, B, n, dtype=torch.float64)
    u = torch.zeros(T, B, 1, dtype=torch.float64)
    with pytest.raises(_lib.MpcB200Error, match="CUDA tensors only"):
        dyn_rollout_raw(k, (1.0,) * 8, T, x0, u)
    with pytest.raises(_lib.MpcB200Error, match="CUDA tensors only"):
        dyn_linearize_raw(k, (1.0,) * 8, T, x, u)
    with pytest.raises(_lib.MpcB200Error, match="unknown dynamics kind"):
        dyn_rollout_raw(0, (1.0,) * 8, T, x0, u)
    with pytest.raises(_lib.MpcB200Error, match="dtype"):
        dyn_rollout_raw(k, (1.0,) * 8, T, x0.half(), u)
