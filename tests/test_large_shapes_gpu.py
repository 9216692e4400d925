"""The large-shape kernels (csrc/lqr_large.cu) against the oracle: (n_state, n_ctrl) pairs that no compiled instance
covers run one thread block per problem with runtime sizes.

Tolerances as in test_horizon_paths_gpu.py: float64 1e-9 x scale with free sets and pnqp iteration counts bit exact;
float32 within 4x the error of the oracle itself run in float32 (same float32-rounded inputs) plus 1e-6 x scale.
MPCB200_KERNEL=3 runs the same kernels on instance shapes, which is how they are checked against the instance
kernels at full batch size."""
import contextlib
import ctypes
import functools
import os

import pytest
import torch

from oracle import lqr_oracle as orc
from tests.helpers import gen_problem, maxdiff, nominal_controls

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
F32, F64 = torch.float32, torch.float64
SHAPES = [(17, 1), (20, 4), (14, 7), (24, 8), (32, 32), (48, 16)]


def _L():
    from mpc.pytorch_b200 import _lib
    return _lib


@contextlib.contextmanager
def _kernel(impl):
    old = os.environ.pop("MPCB200_KERNEL", None)
    if impl is not None:
        os.environ["MPCB200_KERNEL"] = str(impl)
    try:
        yield
    finally:
        os.environ.pop("MPCB200_KERNEL", None)
        if old is not None:
            os.environ["MPCB200_KERNEL"] = old


def _largest(dtype, m=4):
    from mpc.pytorch_b200.step import large_limit
    return large_limit(m, 4 if dtype == F32 else 8), m


def _round(t, dtype):
    return t.to(dtype).double() if torch.is_tensor(t) and t.is_floating_point() and dtype == F32 else t


@functools.lru_cache(maxsize=8)
def step_case(seed, B, T, n, m, dtype, mode, with_f=True, F_T=None):
    """Inputs (float64, rounded through dtype) and the oracle: (P, kw, o64, o32|None).
    mode: plain | mask (u_zero_I) | box (scalar bounds) | boxT (tensor bounds) | boxD (tensor bounds + delta_u)."""
    C, c, F, f, x0 = gen_problem(seed, B, T, n, m, F64, with_f=with_f)
    F = F * 0.9
    if F_T == T:
        F = torch.cat((F, F[-1:]), 0) if T > 1 else gen_problem(seed, B, 2, n, m, F64)[2] * 0.9
    u, ul, uu = nominal_controls(seed, B, T, m, F64, {"box": 0.25, "boxT": "tensor", "boxD": "tensor"}.get(mode))
    kw = {}
    if mode.startswith("box"):
        kw = dict(u_lower=_round(ul, dtype), u_upper=_round(uu, dtype))
    if mode == "boxD":
        kw["delta_u"] = 0.125
    if mode == "mask":
        kw["u_zero_I"] = torch.rand(T, B, m, generator=torch.Generator().manual_seed(seed)) < 0.3
    C, c, F, f, x0, u = (_round(t, dtype) for t in (C, c, F, f, x0, u))
    x = _round(orc.get_traj(T, u, x0, F, f), dtype)
    P = dict(C=C, c=c, F=F, f=f, x0=x0, x=x, u=u)
    o64 = orc.lqr_step_forward(n, m, T, x0, C, c, F, f, x, u, coupled=False, **kw)
    o32 = None
    if dtype == F32:
        lo = lambda t: t.float() if torch.is_tensor(t) and t.is_floating_point() else t
        o32 = orc.lqr_step_forward(n, m, T, lo(x0), lo(C), lo(c), lo(F), lo(f), lo(x), lo(u), coupled=False,
                                   **{k: lo(v) for k, v in kw.items()})
    return P, kw, o64, o32


def _dev(t, dtype):
    return t.to(device=DEV, dtype=dtype if t.is_floating_point() else t.dtype) if torch.is_tensor(t) else t


def _step(n, m, T, P, kw, dtype, impl=None, want_gains=True, do_rollout=True, invariant=False):
    from mpc.pytorch_b200.step import lqr_step_raw
    d = lambda t: _dev(t, dtype)
    C, F = d(P["C"]), d(P["F"])
    if invariant:                              # stride-0 time dimension: MPCB200_TIME_INVARIANT
        C, F = C[:1].expand_as(C), F[:1].expand_as(F)
    with _kernel(impl):
        o = lqr_step_raw(n, m, T, d(P["x0"]), C, d(P["c"]), F, d(P["f"]), d(P["x"]), d(P["u"]),
                         do_rollout=do_rollout, want_gains=want_gains, want_du_first=do_rollout,
                         **{k: d(v) for k, v in kw.items()})
        plan = _L().last_step_plan()
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in o.items() if v is not None}, plan


def _close(tag, what, got, w64, w32, dtype, scale=None):
    if scale is None:
        scale = max(1.0, float(w64.abs().max()))
    err = maxdiff(got, w64)
    bound = 1e-9 * scale if dtype == F64 else 4 * maxdiff(w32, w64) + 1e-6 * scale
    assert err <= bound, f"{tag}: {what} |kernel - oracle| = {err:.3e} > {bound:.3e}"


def _comparable(case):
    """Problems compared: every one in float64; in float32 those whose float32 oracle takes the float64 oracle's pnqp
    path (iteration counts and free sets), which leaves out threshold cases of the |dx| >= 1e-4 test."""
    P, kw, o64, o32 = case
    B = o64.new_u.shape[1]
    if o32 is None:
        return torch.ones(B, dtype=torch.bool)
    same = (o32.qp_iters == o64.qp_iters).all(0) & (o32.free_masks == o64.free_masks).all(2).all(0)
    return same & (o64.qp_iters < 19).all(0)


def _sub(o, keep):
    if o is None:
        return None
    from types import SimpleNamespace
    return SimpleNamespace(**{k: (v[:, keep] if torch.is_tensor(v) and v.dim() >= 2 else v[keep] if torch.is_tensor(v)
                                  and v.dim() == 1 and v.shape[0] == keep.shape[0] else v) for k, v in o._asdict().items()})


def check_step(tag, r, case, dtype, rollout=True):
    keep = _comparable(case)
    if dtype == F32 and "u_lower" in case[1]:    # and the kernel's float32 pnqp takes that path too
        o64 = case[2]
        same = (r["qp_iters"].long() == o64.qp_iters).all(0) & (r["free_mask"].bool() == o64.free_masks).all(2).all(0)
        # where the float32 oracle follows the float64 one, the kernel may leave that path only at a threshold case:
        # at most one problem in four
        left = int((keep & ~same).sum())
        assert left <= max(1, int(keep.sum()) // 4), f"{tag}: kernel left the pnqp path in {left} of {int(keep.sum())}"
        keep &= same
    assert bool(keep.any()) and (dtype == F32 or bool(keep.all())), f"{tag}: no comparable problem"
    P, kw, o64, o32 = case
    P = {k: (v[:, keep] if torch.is_tensor(v) and v.dim() >= 3 else v[keep] if torch.is_tensor(v) else v)
         for k, v in P.items()}
    kw = {k: (v[:, keep] if torch.is_tensor(v) else v) for k, v in kw.items()}
    o64, o32 = _sub(o64, keep), _sub(o32, keep)
    r = {k: (v[:, keep] if v.dim() >= 2 else v[keep]) for k, v in r.items()}
    g = lambda o, k: getattr(o, k) if o is not None else None
    if rollout:
        sc = max(1.0, float(o64.new_x.abs().max()), float(o64.new_u.abs().max()))
        for k in ("new_x", "new_u"):
            _close(tag, k, r[k], g(o64, k), g(o32, k), dtype, sc)
        _close(tag, "costs", r["costs"], o64.costs, g(o32, "costs"), dtype)
        if o32 is None:
            assert torch.equal(r["alphas"], o64.alphas), f"{tag}: alphas"
        else:
            same = (o32.alphas.double() - o64.alphas).abs() <= 1e-6
            assert torch.equal(r["alphas"][same], o32.alphas[same]), f"{tag}: alphas"
        _close(tag, "du_first", r["du_first"], P["u"] - o64.new_u, None if o32 is None else P["u"] - o32.new_u, dtype,
               sc)
        du = (P["u"] - o64.new_u).pow(2).sum((0, 2)).sqrt()
        du32 = None if o32 is None else (P["u"] - o32.new_u).pow(2).sum((0, 2)).sqrt()
        _close(tag, "full_du_norm", r["full_du_norm"], du, du32, dtype, sc)
    _close(tag, "Ks", r["Ks"], o64.Ks, g(o32, "Ks"), dtype)
    _close(tag, "ks", r["ks"], o64.ks, g(o32, "ks"), dtype)
    assert int((r["status"] & ~1).max()) == 0, f"{tag}: status {r['status'].tolist()}"
    if "u_lower" in kw:      # pnqp hit its iteration cap exactly where the oracle's count says so
        assert torch.equal((r["status"] & 1).bool(), (o64.qp_iters == 19).any(0) & (r["status"] & 1).bool()), tag
    assert torch.equal(r["free_mask"].bool(), o64.free_masks), f"{tag}: free sets"
    if "u_lower" in kw:
        assert torch.equal(r["qp_iters"].long(), o64.qp_iters), f"{tag}: pnqp iterations"
    if rollout and "u_zero_I" in kw:
        assert bool((r["new_u"][kw["u_zero_I"]] == 0).all()), f"{tag}: masked controls"


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
    case = step_case(11 + shape, B, T, n, m, dtype, mode)
    r, plan = _step(n, m, T, case[0], case[1], dtype)
    assert plan == _L().PLAN_LARGE
    check_step(f"({n},{m}) {mode}", r, case, dtype)


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("B,T", [(1, 1), (1, 2), (64, 2), (5, 1)])
@pytest.mark.parametrize("mode", ["plain", "boxT"])
def test_step_batch_and_horizon_edges(B, T, mode, dtype):
    n, m = 20, 4
    case = step_case(3, B, T, n, m, dtype, mode)
    r, plan = _step(n, m, T, case[0], case[1], dtype)
    assert plan == _L().PLAN_LARGE
    check_step(f"B={B} T={T} {mode}", r, case, dtype)


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("variant", ["invariant", "F_T=T", "no_f", "gains_only"])
def test_step_input_variants(variant, dtype):
    n, m, B, T = 14, 7, 5, 20
    case = step_case(5, B, T, n, m, dtype, "box", with_f=variant != "no_f", F_T=T if variant == "F_T=T" else None)
    P = case[0]
    if variant == "invariant":           # the oracle sees the same slice at every t
        P = dict(P, C=P["C"][:1].expand_as(P["C"]).contiguous(), F=P["F"][:1].expand_as(P["F"]).contiguous())
        P["x"] = _round(orc.get_traj(T, P["u"], P["x0"], P["F"], P["f"]), dtype)
        o64 = orc.lqr_step_forward(n, m, T, P["x0"], P["C"], P["c"], P["F"], P["f"], P["x"], P["u"], coupled=False,
                                   **case[1])
        lo = lambda t: t.float() if torch.is_tensor(t) and t.is_floating_point() else t
        o32 = None if dtype == F64 else orc.lqr_step_forward(
            n, m, T, *(lo(P[k]) for k in ("x0", "C", "c", "F", "f", "x", "u")), coupled=False,
            **{k: lo(v) for k, v in case[1].items()})
        case = (P, case[1], o64, o32)
    rollout = variant != "gains_only"
    r, plan = _step(n, m, T, P, case[1], dtype, do_rollout=rollout, invariant=variant == "invariant")
    assert plan == _L().PLAN_LARGE
    check_step(variant, r, case, dtype, rollout=rollout)


def test_step_long_horizon_f32():
    n, m, B, T = 20, 4, 4, 200
    for mode in ("plain", "box"):
        case = step_case(9, B, T, n, m, F32, mode)
        r, _ = _step(n, m, T, case[0], case[1], F32)
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
        r_all, _ = _step(n, m, T, full, kw, dtype)
        for i in (0, 131, 256):
            one = {k: v[:, i:i + 1] if v.dim() > 2 or k in ("x", "u") else v[i:i + 1] for k, v in full.items()}
            one["x0"] = x0[i:i + 1]
            r1, _ = _step(n, m, T, one, dict(u_lower=ul[:, i:i + 1], u_upper=uu[:, i:i + 1]), dtype)
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
    P = {k: _round(v, dtype) for k, v in dict(x0=x0, C=C, c=c, F=F, f=f, x=x, u=u).items()}
    kw = {} if bound is None else dict(u_lower=ul, u_upper=uu)
    a, pa = _step(n, m, T, P, kw, dtype)
    b, pb = _step(n, m, T, P, kw, dtype, impl=3)
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
def _abi_adjoint(n, m, T, P, new_x, new_u, dl_dx, dl_du, kw, dtype):
    from mpc.pytorch_b200._lib import Dims, Params, check, entry, lib, ptr
    L = lib()
    d = lambda t: _dev(t, dtype).contiguous() if torch.is_tensor(t) else t
    B = P["C"].shape[1]
    bounded = "u_lower" in kw
    dims = Dims(B=B, T=T, n=n, m=m, F_T=T - 1, has_f=1, bounds_kind=2 if bounded else 0, max_ls_iter=10,
                pnqp_max_iter=20, do_rollout=1)
    nbytes = L.mpcb200_adjoint_workspace_bytes(ctypes.byref(dims), 4 if dtype == F32 else 8)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    p = n + m
    out = [torch.empty(*s, dtype=dtype, device=DEV) for s in ((B, n), (T, B, p, p), (T, B, p), (T - 1, B, n, p),
                                                              (T - 1, B, n))]
    lo, hi = (d(kw["u_lower"]), d(kw["u_upper"])) if bounded else (None, None)
    ins = [d(t) for t in (P["C"], P["c"], P["F"], new_x, new_u, dl_dx, dl_du)] + [lo, hi]   # alive until the sync
    rc = entry("mpcb200_lqr_adjoint", dtype)(
        ctypes.byref(dims), ctypes.byref(Params(ls_decay=0.2)), *[ptr(t) for t in ins + out], ptr(ws), nbytes, None)
    check(rc, "adjoint")
    torch.cuda.synchronize()
    return [o.cpu() for o in out]


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("mode", ["plain", "boxT"])
def test_adjoint_matches_oracle(mode, dtype):
    from mpc.pytorch_b200 import LQRStep, QuadCost, LinDx
    n, m, B, T = 20, 4, 5, 10
    P, kw, o64, o32 = step_case(41, B, T, n, m, dtype, mode)
    g = torch.Generator().manual_seed(4)
    dl_dx = _round(torch.randn(T, B, n, generator=g, dtype=F64), dtype)
    dl_du = _round(torch.randn(T, B, m, generator=g, dtype=F64), dtype)
    bw = dict(u_lower=kw.get("u_lower"), u_upper=kw.get("u_upper"))
    want = orc.lqr_step_backward(n, m, T, P["x0"], P["C"], P["c"], P["F"], P["f"], o64.new_x, o64.new_u, dl_dx,
                                 dl_du, coupled=False, **bw)
    want32 = None
    if dtype == F32:
        lo = lambda t: t.float() if torch.is_tensor(t) else t
        want32 = orc.lqr_step_backward(n, m, T, *(lo(P[k]) for k in ("x0", "C", "c", "F", "f")), lo(o64.new_x),
                                       lo(o64.new_u), lo(dl_dx), lo(dl_du), coupled=False,
                                       **{k: lo(v) for k, v in bw.items()})
    got = _abi_adjoint(n, m, T, P, o64.new_x, o64.new_u, dl_dx, dl_du, kw, dtype)
    assert _L().last_step_plan() == _L().PLAN_LARGE
    names = ("dx_init", "dC", "dc", "dF", "df")
    for i, k in enumerate(names):
        _close(f"abi {mode}", k, got[i], want[i], want32[i] if want32 else None, dtype)
    # through autograd: LQRStepFn.backward takes the multi-call route for these shapes
    leaves = [_dev(P[k], dtype).requires_grad_(True) for k in ("x0", "C", "c", "F", "f")]
    dk = {k: _dev(v, dtype) for k, v in kw.items()}
    step = LQRStep(n, m, T, current_x=_dev(P["x"], dtype), current_u=_dev(P["u"], dtype),
                   true_cost=QuadCost(leaves[1], leaves[2]), true_dynamics=LinDx(leaves[3], leaves[4]), **dk)
    nx, nu = step(*leaves)[:2]
    torch.autograd.backward((nx, nu), (_dev(dl_dx, dtype), _dev(dl_du, dtype)))
    for i, k in enumerate(names):
        if dtype == F64:      # the forward solution is the kernel's, the same as the oracle's to 1e-9
            _close(f"autograd {mode}", k, leaves[i].grad.cpu(), want[i], None, dtype,
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
    F, f, x0, u = (_round(t, dtype) for t in (F, f, x0, u))
    want = orc.get_traj(T, u, x0, F, f)
    got = rollout_raw(n, m, T, _dev(x0, dtype), _dev(u, dtype), _dev(F, dtype), _dev(f, dtype)).cpu()
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
    case = step_case(7, 8, 5, n, m, F64, "box")
    _, plan = _step(n, m, 5, case[0], case[1], F64)
    assert plan & (_L().PLAN_GENERIC | _L().PLAN_PAIR) and not plan & _L().PLAN_LARGE


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
def test_grad_without_workspace(dtype):
    """mpcb200_lqr_grad_* with workspace = NULL: the costate kernel writes the outer products itself.  It equals the
    two-kernel path bit for bit and the oracle within the policy."""
    from mpc.pytorch_b200._lib import Dims, check, entry, ptr
    n, m, B, T = 20, 4, 5, 10
    P, kw, o64, o32 = step_case(41, B, T, n, m, dtype, "plain")
    g = torch.Generator().manual_seed(4)
    dl_dx = _round(torch.randn(T, B, n, generator=g, dtype=F64), dtype)
    dl_du = _round(torch.randn(T, B, m, generator=g, dtype=F64), dtype)
    want = orc.lqr_step_backward(n, m, T, P["x0"], P["C"], P["c"], P["F"], P["f"], o64.new_x, o64.new_u, dl_dx,
                                 dl_du, coupled=False)
    want32 = None
    if dtype == F32:
        lo = lambda t: t.float() if torch.is_tensor(t) else t
        want32 = orc.lqr_step_backward(n, m, T, *(lo(P[k]) for k in ("x0", "C", "c", "F", "f")), lo(o64.new_x),
                                       lo(o64.new_u), lo(dl_dx), lo(dl_du), coupled=False)
    ins = [_dev(t, dtype).contiguous() for t in (P["C"], P["c"], P["F"], o64.new_x, o64.new_u, want[5], want[6],
                                                  dl_dx)]
    p = n + m
    dims = Dims(B=B, T=T, n=n, m=m, F_T=T - 1, has_f=1)
    res = []
    for ws in (torch.empty(2 * T * B * n, dtype=dtype, device=DEV), None):
        out = [torch.empty(*s, dtype=dtype, device=DEV) for s in ((B, n), (T, B, p, p), (T, B, p), (T - 1, B, n, p),
                                                                  (T - 1, B, n))]
        check(entry("mpcb200_lqr_grad", dtype)(ctypes.byref(dims), *[ptr(t) for t in ins + out], ptr(ws), None), "grad")
        torch.cuda.synchronize()
        res.append([o.cpu() for o in out])
    for i, k in enumerate(("dx_init", "dC", "dc", "dF", "df")):
        assert torch.equal(res[0][i], res[1][i]), k
        _close("grad", k, res[1][i], want[i], want32[i] if want32 else None, dtype)


# ------------------------------------------------------------------------------------------------------------------
# the reference's own outputs at shapes without an instance (oracle/make_golden_large.py, float64)
# ------------------------------------------------------------------------------------------------------------------
def test_slew_rate_config5_shape_matches_reference_fixture():
    """MPC(16, 4, slew_rate_penalty=1.0) with box bounds - a (20, 4) LQR step - and d u* / d c against the reference.
    The reference couples pnqp's termination over the batch and the kernels do not, so the solution is held to the
    per-problem oracle at 1e-9 and to the reference within the oracle's own per-problem vs batch-coupled difference."""
    from mpc.pytorch_b200 import MPC, QuadCost, LinDx
    from oracle.make_golden_large import slew_augment
    from tests.helpers import load_golden
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
    from tests.helpers import load_golden
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
    from tests.helpers import load_golden
    g = load_golden("large_step_n24m8_f64")
    T, B, p = g["C"].shape[:3]
    n = g["x_init"].shape[1]
    m = p - n
    P = dict(x0=g["x_init"], C=g["C"], c=g["c"], F=g["F"], f=g["f"], x=g["cur_x"], u=g["cur_u"])
    r, plan = _step(n, m, T, P, dict(u_lower=g["u_lower"], u_upper=g["u_upper"]), F64)
    assert plan == _L().PLAN_LARGE
    sc = max(1.0, float(g["new_x"].abs().max()), float(g["new_u"].abs().max()))
    assert maxdiff(r["new_x"], g["new_x"]) <= 1e-9 * sc and maxdiff(r["new_u"], g["new_u"]) <= 1e-9 * sc
    assert maxdiff(r["costs"], g["costs"]) <= 1e-9 * max(1.0, float(g["costs"].abs().max()))
    assert (1 + r["qp_iters"].long()).sum(0).tolist() == g["n_total_qp_iter"].long().tolist()
