"""The large-shape kernels (csrc/lqr_large.cu) against the oracle: (n_state, n_ctrl) pairs that no compiled instance
covers run one thread block per problem with runtime sizes.

Tolerances (`within` in tests/gpu_harness.py): float64 1e-9 x scale with free sets and pnqp iteration counts bit exact;
float32 within 4x the error of the oracle itself run in float32 (same float32-rounded inputs) plus 1e-6 x scale.
MPCB200_KERNEL=3 runs the same kernels on instance shapes, which is how they are checked against the instance
kernels at full batch size."""
import ctypes

import pytest
import torch

from oracle import lqr_oracle as orc
from tests.gpu_harness import (DEV, F32, F64, abi_adjoint, check_alphas, check_clamps, check_pnqp, check_trajectory,
                               linear_step_case, oracle_steps, round_through, run_step, to_dev, within)
from tests.helpers import gen_problem, load_golden, maxdiff, nominal_controls

pytestmark = pytest.mark.gpu
SHAPES = [(17, 1), (20, 4), (14, 7), (24, 8), (32, 32), (48, 16)]


def _L():
    from mpc.pytorch_b200 import _lib
    return _lib


def _largest(dtype, m=4):
    from mpc.pytorch_b200.step import large_limit
    return large_limit(m, 4 if dtype == F32 else 8), m


def _comparable(case):
    """Problems compared: every one in float64; in float32 those whose float32 oracle takes the float64 oracle's pnqp
    path (iteration counts and free sets), which leaves out threshold cases of the |dx| >= 1e-4 test."""
    P, kw, o64, o32 = case
    B = o64.new_u.shape[1]
    if o32 is None:
        return torch.ones(B, dtype=torch.bool)
    same = (o32.qp_iters == o64.qp_iters).all(0) & (o32.free_masks == o64.free_masks).all(2).all(0)
    return same & (o64.qp_iters < 19).all(0)


def check_step(tag, r, case, dtype):
    P, kw, o64, o32 = case
    keep = _comparable(case)
    if dtype == F32 and "u_lower" in kw:    # and the kernel's float32 pnqp takes that path too
        same = (r["qp_iters"].long() == o64.qp_iters).all(0) & (r["free_mask"].bool() == o64.free_masks).all(2).all(0)
        # where the float32 oracle follows the float64 one, the kernel may leave that path only at a threshold case:
        # at most one problem in four
        left = int((keep & ~same).sum())
        assert left <= max(1, int(keep.sum()) // 4), f"{tag}: kernel left the pnqp path in {left} of {int(keep.sum())}"
        keep &= same
    assert bool(keep.any()) and (dtype == F32 or bool(keep.all())), f"{tag}: no comparable problem"
    if "alphas" in r:
        check_alphas(tag, r, o64, o32, keep)
    check_trajectory(tag, r, P["u"], o64, o32, dtype, keep)
    check_pnqp(tag, r, o64, kw, keep)
    if dtype == F64:        # in float32 the kernel and the float64 oracle leave different controls on the bounds
        check_clamps(tag, r, o64, kw)


# ------------------------------------------------------------------------------------------------------------------
# the step against the oracle
# ------------------------------------------------------------------------------------------------------------------
def _shapes(dtype):
    return SHAPES + [_largest(dtype)]


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("mode", ["plain", "box", "boxT", "boxD", "mask"])
@pytest.mark.parametrize("shape", range(len(SHAPES) + 1))
def test_step_matches_oracle(shape, mode, dtype):
    n, m = _shapes(dtype)[shape]
    B, T = (5, 20) if n + m <= 64 else (2, 6)
    case = linear_step_case(11 + shape, B, T, n, m, dtype, mode)
    r, plan = run_step(n, m, T, *case[:2], dtype, want_du_first=True)
    assert plan == _L().PLAN_LARGE
    check_step(f"({n},{m}) {mode}", r, case, dtype)


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("B,T", [(1, 1), (1, 2), (64, 2), (5, 1)])
@pytest.mark.parametrize("mode", ["plain", "boxT"])
def test_step_batch_and_horizon_edges(B, T, mode, dtype):
    n, m = 20, 4
    case = linear_step_case(3, B, T, n, m, dtype, mode)
    r, plan = run_step(n, m, T, *case[:2], dtype, want_du_first=True)
    assert plan == _L().PLAN_LARGE
    check_step(f"B={B} T={T} {mode}", r, case, dtype)


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("variant", ["invariant", "F_T=T", "no_f", "gains_only"])
def test_step_input_variants(variant, dtype):
    n, m, B, T = 14, 7, 5, 20
    case = linear_step_case(5, B, T, n, m, dtype, "box", with_f=variant != "no_f",
                            F_T=T if variant == "F_T=T" else None)
    P = case[0]
    dev = P
    if variant == "invariant":           # the oracle sees the same slice at every t
        P = dict(P, C=P["C"][:1].expand_as(P["C"]).contiguous(), F=P["F"][:1].expand_as(P["F"]).contiguous())
        P["x"] = round_through(orc.get_traj(T, P["u"], P["x0"], P["F"], P["f"]), dtype)
        case = (P, case[1]) + oracle_steps(n, m, T, P, case[1], dtype)
        # the kernel gets a stride-0 time dimension: MPCB200_TIME_INVARIANT
        C, F = to_dev(P["C"], dtype), to_dev(P["F"], dtype)
        dev = dict(P, C=C[:1].expand_as(C), F=F[:1].expand_as(F))
    rollout = variant != "gains_only"
    r, plan = run_step(n, m, T, dev, case[1], dtype, do_rollout=rollout, want_du_first=True)
    assert plan == _L().PLAN_LARGE
    check_step(variant, r, case, dtype)


def test_step_long_horizon_f32():
    n, m, B, T = 20, 4, 4, 200
    for mode in ("plain", "box"):
        case = linear_step_case(9, B, T, n, m, F32, mode)
        r, _ = run_step(n, m, T, *case[:2], F32, want_du_first=True)
        check_step(f"T=200 {mode}", r, case, F32)


def test_batch_independence():
    """A problem's outputs are bitwise equal alone and at another position in a batch of 257."""
    n, m, T = 24, 8, 10
    for dtype in (F32, F64):
        C, c, F, f, x0 = gen_problem(21, 257, T, n, m, dtype)
        u, ul, uu = nominal_controls(21, 257, T, m, dtype, "tensor")
        x = orc.get_traj(T, u.double(), x0.double(), F.double(), f.double()).to(dtype)
        full = dict(x0=x0, C=C, c=c, F=F, f=f, x=x, u=u)
        kw = dict(u_lower=ul, u_upper=uu)
        r_all, _ = run_step(n, m, T, full, kw, dtype, want_du_first=True)
        for i in (0, 131, 256):
            one = {k: v[:, i:i + 1] if v.dim() > 2 or k in ("x", "u") else v[i:i + 1] for k, v in full.items()}
            one["x0"] = x0[i:i + 1]
            r1, _ = run_step(n, m, T, one, dict(u_lower=ul[:, i:i + 1], u_upper=uu[:, i:i + 1]), dtype,
                             want_du_first=True)
            for k in ("new_x", "new_u", "Ks", "ks", "free_mask"):
                assert torch.equal(r1[k], r_all[k][:, i:i + 1]), f"{dtype} b={i}: {k}"
            for k in ("costs", "alphas", "status", "full_du_norm"):
                assert torch.equal(r1[k], r_all[k][i:i + 1]), f"{dtype} b={i}: {k}"


# ------------------------------------------------------------------------------------------------------------------
# the large kernel against the instance kernels at full batch size (MPCB200_KERNEL=3)
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [F32, F64], ids=["f32", "f64"])
@pytest.mark.parametrize("n,m,T,bound", [(8, 2, 20, 0.25), (16, 4, 50, None)])
def test_cross_kernel(n, m, T, bound, dtype):
    B = 4096
    C, c, F, f, x0 = gen_problem(31, B, T, n, m, F64)
    F = F * 0.9
    u, ul, uu = nominal_controls(31, B, T, m, F64, bound)
    x = orc.get_traj(T, u, x0, F, f)
    P = {k: round_through(v, dtype) for k, v in dict(x0=x0, C=C, c=c, F=F, f=f, x=x, u=u).items()}
    kw = {} if bound is None else dict(u_lower=ul, u_upper=uu)
    a, pa = run_step(n, m, T, P, kw, dtype, want_du_first=True)
    b, pb = run_step(n, m, T, P, kw, dtype, impl=3, want_du_first=True)
    assert pb == _L().PLAN_LARGE and pa != pb
    agree = torch.ones(B, dtype=torch.bool)
    if bound is not None:
        agree = (a["qp_iters"] == b["qp_iters"]).all(0) & (a["free_mask"] == b["free_mask"]).all(2).all(0)
        assert int((~agree).sum()) <= (0 if dtype == F64 else B // 100), f"pnqp paths differ in {int((~agree).sum())}"
    for k in ("new_x", "new_u", "costs", "Ks", "ks"):
        x, y = (a[k][agree], b[k][agree]) if a[k].dim() == 1 else (a[k][:, agree], b[k][:, agree])
        sc = max(1.0, float(x.abs().max()))
        assert maxdiff(x, y) <= (1e-9 if dtype == F64 else 2e-5) * sc, k


# ------------------------------------------------------------------------------------------------------------------
# adjoint, rollout
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("mode", ["plain", "boxT"])
def test_adjoint_matches_oracle(mode, dtype):
    from mpc.pytorch_b200 import LQRStep, QuadCost, LinDx
    n, m, B, T = 20, 4, 5, 10
    P, kw, o64, o32 = linear_step_case(41, B, T, n, m, dtype, mode)
    g = torch.Generator().manual_seed(4)
    dl_dx = round_through(torch.randn(T, B, n, generator=g, dtype=F64), dtype)
    dl_du = round_through(torch.randn(T, B, m, generator=g, dtype=F64), dtype)
    bw = dict(u_lower=kw.get("u_lower"), u_upper=kw.get("u_upper"))
    want = orc.lqr_step_backward(n, m, T, P["x0"], P["C"], P["c"], P["F"], P["f"], o64.new_x, o64.new_u, dl_dx,
                                 dl_du, coupled=False, **bw)
    want32 = None
    if dtype == F32:
        lo = lambda t: t.float() if torch.is_tensor(t) else t
        want32 = orc.lqr_step_backward(n, m, T, *(lo(P[k]) for k in ("x0", "C", "c", "F", "f")), lo(o64.new_x),
                                       lo(o64.new_u), lo(dl_dx), lo(dl_du), coupled=False,
                                       **{k: lo(v) for k, v in bw.items()})
    d = lambda t: to_dev(t, dtype)  # noqa: E731
    got, _ = abi_adjoint(n, m, T, d(P["C"]), d(P["c"]), d(P["F"]), d(o64.new_x), d(o64.new_u), d(dl_dx), d(dl_du),
                         d(kw.get("u_lower")), d(kw.get("u_upper")))
    assert _L().last_step_plan() == _L().PLAN_LARGE
    names = ("dx_init", "dC", "dc", "dF", "df")
    for i, k in enumerate(names):
        within(f"abi {mode}", k, got[i], want[i], want32[i] if want32 else None, dtype)
    # through autograd: LQRStepFn.backward is the same library call (prep, masked large step, 2 gradient kernels)
    leaves = [to_dev(P[k], dtype).requires_grad_(True) for k in ("x0", "C", "c", "F", "f")]
    dk = {k: to_dev(v, dtype) for k, v in kw.items()}
    step = LQRStep(n, m, T, current_x=to_dev(P["x"], dtype), current_u=to_dev(P["u"], dtype),
                   true_cost=QuadCost(leaves[1], leaves[2]), true_dynamics=LinDx(leaves[3], leaves[4]), **dk)
    nx, nu = step(*leaves)[:2]
    before = _L().launch_count()
    torch.autograd.backward((nx, nu), (to_dev(dl_dx, dtype), to_dev(dl_du, dtype)))
    torch.cuda.synchronize()
    assert _L().launch_count() - before == 4
    for i, k in enumerate(names):
        if dtype == F64:      # the forward solution is the kernel's, the same as the oracle's to 1e-9
            within(f"autograd {mode}", k, leaves[i].grad.cpu(), want[i], None, dtype,
                   scale=1e3 * max(1.0, float(want[i].abs().max())))
        else:
            assert bool(torch.isfinite(leaves[i].grad).all())


def test_adjoint_finite_differences_f64():
    """d(loss)/d(x_init, c) by central differences through the forward kernel, at (18, 3), B = 2, unbounded."""
    from mpc.pytorch_b200 import LQRStep, QuadCost, LinDx
    n, m, B, T = 18, 3, 2, 5
    C, c, F, f, x0 = (t.to(DEV) for t in gen_problem(51, B, T, n, m, F64))
    u = torch.zeros(T, B, m, dtype=F64, device=DEV)
    w = torch.randn(T, B, m, generator=torch.Generator().manual_seed(2), dtype=F64).to(DEV)

    def loss(x0_, c_):
        x = orc.get_traj(T, u.cpu(), x0_.detach().cpu(), F.cpu(), f.cpu()).to(DEV)
        step = LQRStep(n, m, T, current_x=x, current_u=u, true_cost=QuadCost(C, c_), true_dynamics=LinDx(F, f))
        return (step(x0_, C, c_, F, f)[1] * w).sum()

    x0g, cg = x0.clone().requires_grad_(True), c.clone().requires_grad_(True)
    loss(x0g, cg).backward()
    eps = 1e-6
    for leaf, grad, idx in ((x0, x0g.grad, [(0, 3), (1, 17)]), (c, cg.grad, [(0, 0, 2), (3, 1, 19), (4, 0, 20)])):
        for i in idx:
            hi, lo = leaf.clone(), leaf.clone()
            hi[i] += eps
            lo[i] -= eps
            args = (hi, c) if leaf is x0 else (x0, hi)
            argl = (lo, c) if leaf is x0 else (x0, lo)
            fd = (float(loss(*args)) - float(loss(*argl))) / (2 * eps)
            assert abs(fd - float(grad[i])) <= 1e-4, f"{i}: fd {fd} vs adjoint {float(grad[i])}"


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("n,m", [(20, 4), (48, 16)])
def test_rollout_matches_oracle(n, m, dtype):
    from mpc.pytorch_b200.step import rollout_raw
    B, T = 7, 15
    C, c, F, f, x0 = gen_problem(61, B, T, n, m, F64)
    F = F * 0.9
    u = torch.randn(T, B, m, generator=torch.Generator().manual_seed(3), dtype=F64)
    F, f, x0, u = (round_through(t, dtype) for t in (F, f, x0, u))
    want = orc.get_traj(T, u, x0, F, f)
    got = rollout_raw(n, m, T, to_dev(x0, dtype), to_dev(u, dtype), to_dev(F, dtype), to_dev(f, dtype)).cpu()
    tol = 1e-12 if dtype == F64 else 1e-5 * max(1.0, float(want.abs().max()))
    assert maxdiff(got, want) <= tol


# ------------------------------------------------------------------------------------------------------------------
# MPC.forward
# ------------------------------------------------------------------------------------------------------------------
def _mpc_traced(n, m, T, x0, C, c, F, f, iters):
    """MPC.forward (box +-0.3) and its per-iteration total_qp_iters (the reference's printed table)."""
    import contextlib
    import io
    from mpc.pytorch_b200 import MPC, QuadCost, LinDx
    from mpc.pytorch_b200 import solver
    buf = io.StringIO()
    solver._seen_tables.clear()
    with contextlib.redirect_stdout(buf):
        out = MPC(n, m, T, u_lower=-0.3, u_upper=0.3, lqr_iter=iters, verbose=1, exit_unconverged=False,
                  backprop=False)(x0.to(DEV), QuadCost(C.to(DEV), c.to(DEV)), LinDx(F.to(DEV), f.to(DEV)))
    rows = [l.strip("| \n").split(" | ") for l in buf.getvalue().splitlines() if l.startswith("| ")]
    return out, [float(r[4].strip("tensor([])")) for r in rows if r[0] != "iter"]


def test_mpc_forward_matches_oracle_bounded():
    """MPC.forward at (24, 8) with box bounds.  While the per-iteration pnqp work (total_qp_iters) equals the
    per-problem oracle's - the first three iLQR iterations here - the solution agrees to 1e-9 x scale.  The fourth
    iteration takes one pnqp iteration more at one time step than the oracle, so the ten-iteration solve is held to
    the pnqp step tolerance (1e-4) only."""
    n, m, B, T = 24, 8, 4, 8
    C, c, F, f, x0 = gen_problem(71, B, T, n, m, F64)
    F = F * 0.9
    for iters, tol in ((3, 1e-9), (10, 2e-4)):
        trace = []
        want = orc.mpc_forward_lin(n, m, T, x0, C, c, F, f, u_lower=-0.3, u_upper=0.3, lqr_iter=iters,
                                   coupled=False, trace=trace)
        (x, u, costs), got_qp = _mpc_traced(n, m, T, x0, C, c, F, f, iters)
        want_qp = [t["total_qp_iters"] for t in trace]
        if iters == 3:
            assert got_qp == want_qp, (got_qp, want_qp)
        sc = max(1.0, float(want[0].abs().max()))
        assert maxdiff(x, want[0]) <= tol * sc and maxdiff(u, want[1]) <= tol * sc, (iters, maxdiff(u, want[1]))
        assert maxdiff(costs, want[2]) <= tol * max(1.0, float(want[2].abs().max()))


def test_mpc_split_mode_affine_matches_lindx():
    from mpc.pytorch_b200 import MPC, QuadCost, LinDx, AffineDynamics
    n, m, B, T = 20, 4, 3, 8
    g = torch.Generator().manual_seed(81)
    A = (0.9 * torch.eye(n, dtype=F64) + 0.05 * torch.randn(n, n, generator=g, dtype=F64)).to(DEV)
    Bm = (0.3 * torch.randn(n, m, generator=g, dtype=F64)).to(DEV)
    cc = (0.1 * torch.randn(n, generator=g, dtype=F64)).to(DEV)
    C, c, _, _, x0 = (t.to(DEV) if t is not None else None for t in gen_problem(81, B, T, n, m, F64))
    kw = dict(u_lower=-0.5, u_upper=0.5, lqr_iter=8, verbose=-1, exit_unconverged=False, backprop=False)
    a = MPC(n, m, T, **kw)(x0, QuadCost(C, c), AffineDynamics(A, Bm, cc))
    F = torch.cat((A, Bm), 1).expand(T - 1, B, n, n + m)
    b = MPC(n, m, T, **kw)(x0, QuadCost(C, c), LinDx(F, cc.expand(T - 1, B, n)))
    assert maxdiff(a[0], b[0]) <= 1e-6 and maxdiff(a[1], b[1]) <= 1e-6


def test_mpc_slew_rate_at_config5_shape():
    """MPC(16, 4, slew_rate_penalty=...) solves a (20, 4) LQR step: it runs, and the penalty smooths the controls."""
    from mpc.pytorch_b200 import MPC, QuadCost, LinDx
    n, m, B, T = 16, 4, 4, 10
    C, c, F, f, x0 = (t.to(DEV) for t in gen_problem(91, B, T, n, m, F64))
    kw = dict(u_lower=-1.0, u_upper=1.0, lqr_iter=10, verbose=-1, exit_unconverged=False, backprop=False)
    x0_, u0_, _ = MPC(n, m, T, **kw)(x0, QuadCost(C, c), LinDx(F, f))
    x1_, u1_, _ = MPC(n, m, T, slew_rate_penalty=1.0, **kw)(x0, QuadCost(C, c), LinDx(F, f))
    assert _L().last_step_plan() == _L().PLAN_LARGE
    rough = lambda u: float((u[1:] - u[:-1]).pow(2).sum())
    assert rough(u1_) < rough(u0_)


# ------------------------------------------------------------------------------------------------------------------
# limits and routing
# ------------------------------------------------------------------------------------------------------------------
def _abi_step(n, m, T, B, dtype, with_gains=True):
    from mpc.pytorch_b200._lib import Dims, Params, entry, ptr
    p = n + m
    z = lambda *s: torch.zeros(*s, dtype=dtype, device=DEV)
    C = torch.eye(p, dtype=dtype, device=DEV).expand(T, B, p, p).contiguous()
    ins = [C, z(T, B, p), z(T - 1, B, n, p), None, z(B, n), z(T, B, n), z(T, B, m), None, None, None]
    outs = [z(T, B, n), z(T, B, m), z(B), z(B), z(B), None, None, None, None]
    gains = [z(T, B, m, n), z(T, B, m)] if with_gains else [None, None]
    dims = Dims(B=B, T=T, n=n, m=m, F_T=T - 1, max_ls_iter=1, pnqp_max_iter=20, do_rollout=1)
    return entry("mpcb200_lqr_step", dtype)(ctypes.byref(dims), ctypes.byref(Params(ls_decay=0.2)),
                                           *[ptr(t) for t in ins + outs + gains], None)


@pytest.mark.parametrize("dtype", [F32, F64], ids=["f32", "f64"])
def test_limits(dtype):
    from mpc.pytorch_b200 import LQRStep
    nmax, m = _largest(dtype)
    assert _abi_step(nmax, m, 2, 2, dtype) == 0
    assert _abi_step(nmax + 1, m, 2, 2, dtype) == 4                  # MPCB200_ERR_SMEM
    assert _abi_step(20, 4, 2, 2, dtype, with_gains=False) == 4
    from mpc.pytorch_b200 import QuadCost, LinDx
    T, B, n = 2, 1, nmax + 1
    p = n + m
    C = torch.eye(p, dtype=dtype, device=DEV).expand(T, B, p, p)
    c = torch.zeros(T, B, p, dtype=dtype, device=DEV)
    F = torch.zeros(T - 1, B, n, p, dtype=dtype, device=DEV)
    with pytest.raises(_L().MpcB200Error, match=rf"n_state <= {nmax} for n_ctrl={m}"):
        LQRStep(n, m, T, current_x=torch.zeros(T, B, n, dtype=dtype, device=DEV),
                current_u=torch.zeros(T, B, m, dtype=dtype, device=DEV), true_cost=QuadCost(C, c),
                true_dynamics=LinDx(F))(torch.zeros(B, n, dtype=dtype, device=DEV), C, c, F)


@pytest.mark.parametrize("n,m", [(16, 4), (13, 3), (8, 2), (5, 1)])
def test_instance_and_padded_shapes_keep_their_plan(n, m):
    case = linear_step_case(7, 8, 5, n, m, F64, "box")
    _, plan = run_step(n, m, 5, *case[:2], F64, want_du_first=True)
    assert plan & (_L().PLAN_GENERIC | _L().PLAN_PAIR) and not plan & _L().PLAN_LARGE


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
def test_grad_two_kernels_match_oracle(dtype):
    """mpcb200_lqr_grad_* at a shape without an instance: the costate kernel writes the costates to the workspace,
    the outer-product kernel reads them (2 launches); against the oracle within the policy."""
    from mpc.pytorch_b200._lib import Dims, check, entry, ptr
    n, m, B, T = 20, 4, 5, 10
    P, kw, o64, o32 = linear_step_case(41, B, T, n, m, dtype, "plain")
    g = torch.Generator().manual_seed(4)
    dl_dx = round_through(torch.randn(T, B, n, generator=g, dtype=F64), dtype)
    dl_du = round_through(torch.randn(T, B, m, generator=g, dtype=F64), dtype)
    want = orc.lqr_step_backward(n, m, T, P["x0"], P["C"], P["c"], P["F"], P["f"], o64.new_x, o64.new_u, dl_dx,
                                 dl_du, coupled=False)
    want32 = None
    if dtype == F32:
        lo = lambda t: t.float() if torch.is_tensor(t) else t
        want32 = orc.lqr_step_backward(n, m, T, *(lo(P[k]) for k in ("x0", "C", "c", "F", "f")), lo(o64.new_x),
                                       lo(o64.new_u), lo(dl_dx), lo(dl_du), coupled=False)
    ins = [to_dev(t, dtype).contiguous() for t in (P["C"], P["c"], P["F"], o64.new_x, o64.new_u, want[5], want[6],
                                                  dl_dx)]
    p = n + m
    dims = Dims(B=B, T=T, n=n, m=m, F_T=T - 1, has_f=1)
    ws = torch.empty(2 * T * B * n, dtype=dtype, device=DEV)
    out = [torch.empty(*s, dtype=dtype, device=DEV) for s in ((B, n), (T, B, p, p), (T, B, p), (T - 1, B, n, p),
                                                              (T - 1, B, n))]
    before = _L().launch_count()
    check(entry("mpcb200_lqr_grad", dtype)(ctypes.byref(dims), *[ptr(t) for t in ins + out], ptr(ws), None), "grad")
    torch.cuda.synchronize()
    assert _L().launch_count() - before == 2
    for i, k in enumerate(("dx_init", "dC", "dc", "dF", "df")):
        within("grad", k, out[i].cpu(), want[i], want32[i] if want32 else None, dtype)


# ------------------------------------------------------------------------------------------------------------------
# the reference's own outputs at shapes without an instance (oracle/make_golden_large.py, float64)
# ------------------------------------------------------------------------------------------------------------------
def test_slew_rate_config5_shape_matches_reference_fixture():
    """MPC(16, 4, slew_rate_penalty=1.0) with box bounds - a (20, 4) LQR step - and d u* / d c against the reference.
    The reference couples pnqp's termination over the batch and the kernels do not, so the solution is held to the
    per-problem oracle at 1e-9 and to the reference within the oracle's own per-problem vs batch-coupled difference."""
    from mpc.pytorch_b200 import MPC, QuadCost, LinDx
    from oracle.make_golden_large import slew_augment
    g = load_golden("large_slew_f64")
    T, B, p = g["C"].shape[:3]
    n = g["x_init"].shape[1]
    m = p - n
    b, pen, iters = float(g["bound"]), float(g["penalty"]), int(g["lqr_iter"])
    F = torch.cat((g["A"], g["Bm"]), 1).expand(T - 1, B, n, p).contiguous()
    C2, c2, F2, x02 = slew_augment(g["C"], g["c"], F, g["x_init"], g["prev_ctrl"], pen, n, m)
    ox, ou, _, _ = orc.mpc_forward_lin(n + m, m, T, x02, C2, c2, F2, None, u_lower=-b, u_upper=b, lqr_iter=iters,
                                       eps=1e-9, coupled=False)
    cl = g["c"].to(DEV).requires_grad_(True)
    x, u, costs = MPC(n, m, T, u_lower=-b, u_upper=b, lqr_iter=iters, verbose=-1, exit_unconverged=False,
                      detach_unconverged=False, slew_rate_penalty=pen, prev_ctrl=g["prev_ctrl"].to(DEV), eps=1e-9)(
        g["x_init"].to(DEV), QuadCost(g["C"].to(DEV), cl), LinDx(F.to(DEV)))
    assert _L().last_step_plan() == _L().PLAN_LARGE
    # 20 iLQR iterations of a problem whose slew block [[gI, -gI], [-gI, gI]] is singular: round-off differences
    # of the single step (1e-9 x scale) are carried through the outer loop, so the loop is held to 1e-7 x scale
    sc = max(1.0, float(ou.abs().max()), float(ox.abs().max()))
    assert maxdiff(u, ou) <= 1e-7 * sc and maxdiff(x, ox[:, :, m:]) <= 1e-7 * sc
    assert maxdiff(u, g["u"]) <= maxdiff(ou, g["u"]) + 1e-7 * sc
    assert maxdiff(x, g["x"]) <= maxdiff(ox[:, :, m:], g["x"]) + 1e-7 * sc
    rows = torch.zeros(T, B, m, T, B, p, dtype=F64)          # d u* / d c, all problems at once per (t, control)
    for t in range(T):
        for j in range(m):
            gc, = torch.autograd.grad(u[t, :, j].sum(), cl, retain_graph=True)
            for bb in range(B):
                rows[t, bb, j, :, bb] = gc[:, bb].cpu()
    want = g["du_dc"]
    assert maxdiff(rows.reshape(T * B * m, -1), want) <= 1e-8 * max(1.0, float(want.abs().max()))


def test_unbounded_step_n14m7_matches_reference_fixture():
    from mpc.pytorch_b200 import LQRStep, QuadCost, LinDx
    g = load_golden("large_step_n14m7_f64")
    T, B, p = g["C"].shape[:3]
    n = g["x_init"].shape[1]
    m = p - n
    leaves = [g[k].to(DEV).requires_grad_(True) for k in ("x_init", "C", "c", "F", "f")]
    step = LQRStep(n, m, T, current_x=g["cur_x"].to(DEV), current_u=g["cur_u"].to(DEV),
                   true_cost=QuadCost(leaves[1], leaves[2]), true_dynamics=LinDx(leaves[3], leaves[4]))
    nx, nu = step(*leaves)[:2]
    assert _L().last_step_plan() == _L().PLAN_LARGE
    sc = max(1.0, float(g["new_x"].abs().max()), float(g["new_u"].abs().max()))
    assert maxdiff(nx, g["new_x"]) <= 1e-9 * sc and maxdiff(nu, g["new_u"]) <= 1e-9 * sc
    torch.autograd.backward((nx, nu), (g["wx"].to(DEV), g["wu"].to(DEV)))
    for leaf, k in zip(leaves, ("dx_init", "dC", "dc", "dF", "df")):
        assert maxdiff(leaf.grad, g[k]) <= 1e-9 * max(1.0, float(g[k].abs().max())), k


def test_bounded_step_n24m8_matches_reference_fixture():
    """Tensor bounds at (24, 8); the fixture was made one problem at a time (per-problem pnqp semantics)."""
    g = load_golden("large_step_n24m8_f64")
    T, B, p = g["C"].shape[:3]
    n = g["x_init"].shape[1]
    m = p - n
    P = dict(x0=g["x_init"], C=g["C"], c=g["c"], F=g["F"], f=g["f"], x=g["cur_x"], u=g["cur_u"])
    r, plan = run_step(n, m, T, P, dict(u_lower=g["u_lower"], u_upper=g["u_upper"]), F64, want_du_first=True)
    assert plan == _L().PLAN_LARGE
    sc = max(1.0, float(g["new_x"].abs().max()), float(g["new_u"].abs().max()))
    assert maxdiff(r["new_x"], g["new_x"]) <= 1e-9 * sc and maxdiff(r["new_u"], g["new_u"]) <= 1e-9 * sc
    assert maxdiff(r["costs"], g["costs"]) <= 1e-9 * max(1.0, float(g["costs"].abs().max()))
    assert (1 + r["qp_iters"].long()).sum(0).tolist() == g["n_total_qp_iter"].long().tolist()
