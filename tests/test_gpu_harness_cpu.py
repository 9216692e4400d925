"""The shared step checks of the GPU suites are not vacuous: the float64 oracle's own step, posed as kernel output,
passes the trajectory, pnqp and clamp checks, and each single perturbation of it fails the check that covers it."""
import pytest
import torch

from tests.gpu_harness import F64, check_clamps, check_pnqp, check_trajectory, linear_step_case


def _case():
    return linear_step_case(5, 6, 8, 4, 2, F64, "box")


def _as_kernel_output(case):
    """What run_step returns for a bounded step with gains and du_first, made from the oracle's step."""
    P, kw, o, _ = case
    du = P["u"] - o.new_u
    return dict(new_x=o.new_x.clone(), new_u=o.new_u.clone(), costs=o.costs.clone(), alphas=o.alphas.clone(),
                Ks=o.Ks.clone(), ks=o.ks.clone(), du_first=du, full_du_norm=du.pow(2).sum((0, 2)).sqrt(),
                qp_iters=o.qp_iters.int(), free_mask=o.free_masks.to(torch.uint8),
                status=torch.zeros(o.costs.shape[0], dtype=torch.int32))


def _check(r, case):
    P, kw, o64, o32 = case
    check_trajectory("harness", r, P["u"], o64, o32, F64)
    check_pnqp("harness", r, o64, kw)
    check_clamps("harness", r, o64, kw)


def test_the_oracle_step_passes():
    case = _case()
    _check(_as_kernel_output(case), case)


def _perturb(r, case, what):
    _, kw, o, _ = case
    if what == "new_u":                 # 10x the float64 bound, 1e-9 x scale
        sc = max(1.0, float(o.new_x.abs().max()), float(o.new_u.abs().max()))
        r["new_u"][0, 0, 0] += 10 * 1e-9 * sc
    elif what == "free_set":
        r["free_mask"][0, 0, 0] ^= 1
    elif what == "qp_iters":
        r["qp_iters"][0, 0] += 1
    elif what == "clamped_control":     # off its bound, by far less than the trajectory tolerance
        t, b, j = (o.new_u.abs() == kw["u_upper"]).nonzero()[0].tolist()
        r["new_u"][t, b, j] -= 1e-12 * torch.sign(o.new_u[t, b, j])


PERTURBATIONS = [("new_u", "new_u"), ("free_set", "free sets"), ("qp_iters", "pnqp iterations"),
                 ("clamped_control", "clamp mask")]


@pytest.mark.parametrize("what,caught_by", PERTURBATIONS, ids=[w for w, _ in PERTURBATIONS])
def test_each_perturbation_fails(what, caught_by):
    case = _case()
    r = _as_kernel_output(case)
    _perturb(r, case, what)
    with pytest.raises(AssertionError, match=caught_by):
        _check(r, case)
