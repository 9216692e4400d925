"""CPU: every entry point that hands tensors to libmpcb200.so refuses a malformed argument with an MpcB200Error
naming that argument (or the dtype), on tensor metadata alone and before the "CUDA tensors only" check.  So a
malformed call never reaches a kernel, and the whole table runs on CPU tensors.  Table driven: entry point x
malformed argument."""
import pytest
import torch

from mpc.pytorch_b200 import LQRStep, LinDx, QuadCost
from mpc.pytorch_b200._lib import MpcB200Error
from mpc.pytorch_b200.boxqp import pnqp
from mpc.pytorch_b200.dynamics import DYN_CARTPOLE, dyn_linearize_raw, dyn_rollout_raw
from mpc.pytorch_b200.step import lqr_adjoint_raw, lqr_grad_raw, lqr_step_raw, rollout_raw

N, M, T, B = 3, 1, 4, 2
P = N + M
STEP_SHAPES = {"C": (T, B, P, P), "c": (T, B, P), "F": (T - 1, B, N, P), "f": (T - 1, B, N), "x_init": (B, N),
               "current_x": (T, B, N), "current_u": (T, B, M), "u": (T, B, M), "new_x": (T, B, N),
               "new_u": (T, B, M), "dx": (T, B, N), "du": (T, B, M), "dl_dx": (T, B, N), "dl_du": (T, B, M),
               "u_lower": (T, B, M), "u_upper": (T, B, M), "u_zero_I": (T, B, M)}
Q = 4                                    # pnqp variables
NX = 5                                   # cartpole state


def _step_shapes(*names):
    return {k: STEP_SHAPES[k] for k in names}


def _lqr_step(a, no_op_forward):
    fn = LQRStep(N, M, T, u_lower=a["u_lower"], u_upper=a["u_upper"], u_zero_I=a.get("u_zero_I"),
                 true_cost=QuadCost(a["C"], a["c"]), true_dynamics=LinDx(a["F"], a["f"]),
                 current_x=a["current_x"], current_u=a["current_u"], no_op_forward=no_op_forward)
    return fn(a["x_init"], a["C"], a["c"], a["F"], a["f"])


# entry point -> (call on a dict of arguments, shape of each tensor argument; the first one leads: the others
# must share its device)
ENTRIES = {
    "lqr_step_raw": (
        lambda a: lqr_step_raw(N, M, T, a["x_init"], a["C"], a["c"], a["F"], a["f"], a["current_x"], a["current_u"],
                               u_lower=a["u_lower"], u_upper=a["u_upper"], u_zero_I=a["u_zero_I"]),
        _step_shapes("C", "c", "F", "f", "x_init", "current_x", "current_u", "u_lower", "u_upper", "u_zero_I")),
    "lqr_grad_raw": (
        lambda a: lqr_grad_raw(N, M, T, a["C"], a["c"], a["F"], a["new_x"], a["new_u"], a["dx"], a["du"],
                               a["dl_dx"], True),
        _step_shapes("C", "c", "F", "new_x", "new_u", "dx", "du", "dl_dx")),
    "lqr_adjoint_raw": (
        lambda a: lqr_adjoint_raw(N, M, T, a["C"], a["c"], a["F"], a["new_x"], a["new_u"], a["dl_dx"], a["dl_du"],
                                  a["u_lower"], a["u_upper"], True, validated=False),
        _step_shapes("C", "c", "F", "new_x", "new_u", "dl_dx", "dl_du", "u_lower", "u_upper")),
    "rollout_raw": (
        lambda a: rollout_raw(N, M, T, a["x_init"], a["u"], a["F"], a["f"]),
        _step_shapes("x_init", "u", "F", "f")),
    "LQRStep": (
        lambda a: _lqr_step(a, no_op_forward=False),
        _step_shapes("C", "c", "F", "f", "x_init", "current_x", "current_u", "u_lower", "u_upper", "u_zero_I")),
    "LQRStep_no_op_forward": (
        lambda a: _lqr_step(a, no_op_forward=True),
        _step_shapes("C", "c", "F", "f", "x_init", "current_x", "current_u", "u_lower", "u_upper")),
    "pnqp": (
        lambda a: pnqp(a["H"], a["q"], a["lower"], a["upper"], x_init=a["x_init"]),
        {"H": (B, Q, Q), "q": (B, Q), "lower": (B, Q), "upper": (B, Q), "x_init": (B, Q)}),
    "dyn_rollout_raw": (
        lambda a: dyn_rollout_raw(DYN_CARTPOLE, (1.0,) * 8, T, a["x_init"], a["u"]),
        {"x_init": (B, NX), "u": (T, B, 1)}),
    "dyn_linearize_raw": (
        lambda a: dyn_linearize_raw(DYN_CARTPOLE, (1.0,) * 8, T, a["x"], a["u"]),
        {"x": (T, B, NX), "u": (T, B, 1)}),
}


def _cases():
    """(entry point, malformed argument, argument the message must name or "dtype")."""
    for entry, (_, shapes) in ENTRIES.items():
        names = list(shapes)
        for nm in names:
            yield entry, ("shape", nm), nm
            yield entry, ("ndim", nm), nm
        for nm in ("F", "f"):
            if nm in names:
                yield entry, ("time_slices", nm), nm
        if "F" in names:
            yield entry, ("missing", "F"), "F"
        for nm in names[1:]:
            yield entry, ("meta", nm), nm
        yield entry, ("dtype", torch.float16), "dtype"
        yield entry, ("dtype", torch.bfloat16), "dtype"


CASES = list(_cases())


def _args(shapes):
    a = {nm: torch.rand(sh, dtype=torch.float64) for nm, sh in shapes.items()}
    if "u_zero_I" in a:
        a["u_zero_I"] = torch.zeros(shapes["u_zero_I"], dtype=torch.bool)
    return a


def _malform(a, how, nm):
    t = a[nm] if nm in a else None
    if how == "shape":                   # one more element in the last dimension
        a[nm] = torch.zeros(*t.shape[:-1], t.shape[-1] + 1, dtype=t.dtype)
    elif how == "ndim":
        a[nm] = t.unsqueeze(0)
    elif how == "time_slices":           # neither T-1 nor T
        a[nm] = torch.zeros(T + 1, *t.shape[1:], dtype=t.dtype)
    elif how == "missing":
        a[nm] = None
    elif how == "meta":
        a[nm] = torch.empty(t.shape, dtype=t.dtype, device="meta")
    elif how == "dtype":
        for k, v in a.items():
            if v.is_floating_point():
                a[k] = v.to(nm)


@pytest.mark.parametrize("entry,bad,name", CASES,
                         ids=[f"{e}-{b[0]}-{str(b[1]).replace('torch.', '')}" for e, b, _ in CASES])
def test_malformed_argument_is_refused_before_the_cuda_check(entry, bad, name):
    call, shapes = ENTRIES[entry]
    a = _args(shapes)
    _malform(a, *bad)
    with pytest.raises(MpcB200Error) as err:
        call(a)
    msg = str(err.value)
    if name == "dtype":
        assert "unsupported dtype" in msg and str(bad[1]) in msg, msg
    else:
        assert msg.startswith((f"{name}:", f"{name} ")), msg


@pytest.mark.parametrize("entry", list(ENTRIES))
def test_well_formed_cpu_arguments_reach_the_cuda_check(entry):
    """The table's arguments are well formed: unchanged, they fail only because they are not on a GPU."""
    call, shapes = ENTRIES[entry]
    a = _args(shapes)
    with pytest.raises(MpcB200Error, match="CUDA tensors only"):
        call(a)
