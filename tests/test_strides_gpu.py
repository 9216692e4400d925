"""GPU: time-strided inputs are honoured without materialising them (reference mpc/mpc.py:205-226 hands over
`expand()`ed cost terms; an LTI system is an `F` with time stride 0).  Results must equal the dense call bit for
bit - the kernels read the same values, only from fewer bytes."""
import pytest
import torch

from tests.helpers import gen_problem, maxdiff, nominal_controls

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


@pytest.mark.parametrize("n,m,B,T", [(8, 2, 48, 12), (16, 4, 24, 9), (4, 2, 40, 7), (5, 1, 18, 8)])
@pytest.mark.parametrize("bounds", [None, 0.3])
def test_time_invariant_and_strided_inputs_equal_dense(n, m, B, T, bounds):
    from mpc.pytorch_b200.step import lqr_grad_raw, lqr_step_raw, rollout_raw, _time_strided
    C, c, F, f, x0 = [t.to(DEV) for t in gen_problem(60 + n, B, T, n, m, torch.float32)]
    u, ul, uu = nominal_controls(60, B, T, m, torch.float32, bounds)
    u = u.to(DEV)
    # LTI dynamics and a time-invariant cost as stride-0 views; c with an explicit (2x dense) time stride
    F_lti = F[:1].expand(T - 1, B, n, n + m)
    C_ti = C[:1].expand(T, B, n + m, n + m)
    c_big = torch.randn(2 * T, B, n + m, device=DEV)
    c_str = c_big[::2]
    assert _time_strided(F_lti, torch.float32)[1] == -1 and _time_strided(c_str, torch.float32)[1] == 2 * B * (n + m)
    x = rollout_raw(n, m, T, x0, u, F_lti, f)
    assert torch.equal(x, rollout_raw(n, m, T, x0, u, F_lti.contiguous(), f))
    kw = dict(u_lower=ul, u_upper=uu, want_gains=False)
    a = lqr_step_raw(n, m, T, x0, C_ti, c_str, F_lti, f, x, u, **kw)
    b = lqr_step_raw(n, m, T, x0, C_ti.contiguous(), c_str.contiguous(), F_lti.contiguous(), f, x, u, **kw)
    torch.cuda.synchronize()
    for k in ("new_x", "new_u", "costs", "alphas", "full_du_norm", "status", "free_mask"):
        assert torch.equal(a[k], b[k]), k
    assert int((a["status"] & ~1).max()) == 0        # (bit 0: an fp32 pnqp instance at the iteration cap, same in both)
    # the gradient kernels read the same strided inputs
    dx, du = a["new_x"] - x, a["new_u"] - u
    ga = lqr_grad_raw(n, m, T, C_ti, c_str, F_lti, a["new_x"], a["new_u"], dx, du, x, True)
    gb = lqr_grad_raw(n, m, T, C_ti.contiguous(), c_str.contiguous(), F_lti.contiguous(), a["new_x"], a["new_u"],
                      dx, du, x, True)
    torch.cuda.synchronize()
    for k, name in enumerate(("dx_init", "dC", "dc", "dF", "df")):
        assert torch.equal(ga[k], gb[k]), name


def test_gradient_of_an_lti_system_sums_over_time():
    """dF of an `expand()`ed F: autograd reduces the kernel's dense [T-1,B,n,p] gradient over the time axis."""
    from mpc.pytorch_b200 import LQRStep, QuadCost, LinDx
    B, T, n, m = 10, 8, 8, 2
    C, c, F, f, x0 = [t.to(DEV) for t in gen_problem(77, B, T, n, m, torch.float64)]
    F0 = F[:1].clone().requires_grad_(True)
    Fd = F[:1].expand(T - 1, B, n, n + m).contiguous().requires_grad_(True)
    u = torch.zeros(T, B, m, dtype=torch.float64, device=DEV)
    from mpc.pytorch_b200.step import rollout_raw
    x = rollout_raw(n, m, T, x0, u, Fd.detach(), f)
    grads = []
    for Fin in (F0.expand(T - 1, B, n, n + m), Fd):
        fn = LQRStep(n, m, T, u_lower=-0.4, u_upper=0.4, true_cost=QuadCost(C, c), true_dynamics=LinDx(Fin, f),
                     current_x=x, current_u=u, no_op_forward=True)
        xo, uo = fn(x0, C, c, Fin, f)
        grads.append(torch.autograd.grad((xo * xo).sum() + uo.sum(), F0 if Fin is not Fd else Fd)[0])
    assert maxdiff(grads[0][0], grads[1].sum(0)) < 1e-9 * max(1.0, float(grads[1].abs().max()))
