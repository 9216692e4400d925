"""The generic step kernel's lane layout at (n, m) = (8, 2): a problem's results do not depend on where it sits.

In fp32 the kernel gives a problem 8 lanes, 4 problems to a warp and 2 warps to a CTA: lane j owns state column j,
and lanes 0 and 1 also own control columns 8 and 9 in a second slot.  fp64 keeps one column per lane (3 problems per
warp, 2 warps per CTA).  A seeded pool of problems is solved one at a time, then in batches of
B in {1, 3, 4, 5, 7, 9, 4093, 4096} where batch element b is pool problem b % 5.  Since 5 is coprime to the warp
and CTA sizes, every pool problem lands at every position of a warp and of a CTA, in full CTAs and in the tail CTA.  Every output of every batch
element must equal, bit for bit, the output of the same problem solved alone: new_x, new_u, costs, alphas,
full_du_norm, Ks/ks, free_mask, qp_iters, status."""
import pytest
import torch

from tests.helpers import gen_problem, nominal_controls

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
N, M, T = 8, 2, 6
POOL = 5
BATCHES = [1, 3, 4, 5, 7, 9, 4093, 4096]
MODES = ["plain", "box", "boxT", "mask"]
BITS = {torch.float32: torch.int32, torch.float64: torch.int64}


def _pool(dtype, mode):
    """POOL problems as [T, POOL, ...] tensors (time major) and the keyword arguments of the mode."""
    C, c, F, f, x0 = gen_problem(71, POOL, T, N, M, torch.float64)
    u, lo, hi = nominal_controls(71, POOL, T, M, torch.float64, {"box": 0.25, "boxT": "tensor"}.get(mode))
    x = [x0]
    for t in range(T - 1):
        x.append(torch.einsum("bij,bj->bi", F[t], torch.cat((x[t], u[t]), 1)) + f[t])
    P = dict(C=C, c=c, F=F, f=f, x0=x0, x=torch.stack(x), u=u)
    P = {k: v.to(dtype) for k, v in P.items()}
    kw = {}
    if mode == "box":
        kw = dict(u_lower=lo, u_upper=hi)
    elif mode == "boxT":
        kw = dict(u_lower=lo.to(dtype), u_upper=hi.to(dtype))
    elif mode == "mask":
        kw = dict(u_zero_I=torch.rand(T, POOL, M, generator=torch.Generator().manual_seed(71)) < 0.3)
    return P, kw


def _solve(P, kw, idx):
    from mpc.pytorch_b200 import _lib
    from mpc.pytorch_b200.step import lqr_step_raw
    d = lambda t: t.index_select(1, idx).contiguous().to(DEV) if torch.is_tensor(t) else t   # [T, B, ...]
    x0 = P["x0"].index_select(0, idx).to(DEV)
    o = lqr_step_raw(N, M, T, x0, d(P["C"]), d(P["c"]), d(P["F"]), d(P["f"]), d(P["x"]), d(P["u"]),
                     want_gains=True, **{k: d(v) for k, v in kw.items()})
    plan = _lib.last_step_plan()
    torch.cuda.synchronize()
    assert plan & _lib.PLAN_GENERIC, f"expected the generic kernel, plan {plan}"
    return {k: v.cpu() for k, v in o.items() if v is not None}


def _bits(v):
    return v.view(BITS[v.dtype]) if v.is_floating_point() else v


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
def test_results_do_not_depend_on_the_batch_position(dtype, mode):
    P, kw = _pool(dtype, mode)
    alone = [_solve(P, kw, torch.tensor([k])) for k in range(POOL)]
    keys = sorted(alone[0])
    assert {"new_x", "new_u", "costs", "alphas", "full_du_norm", "Ks", "ks", "free_mask", "status"} <= set(keys)
    if mode in ("box", "boxT"):
        assert "qp_iters" in keys
        assert any(int(a["qp_iters"].max()) > 0 for a in alone), "the box cases must run pnqp iterations"
        assert any(bool((a["free_mask"] == 0).any()) for a in alone), "the box cases must clamp some controls"
    if mode == "mask":
        assert any(bool((a["free_mask"] == 0).any()) for a in alone)
    for B in BATCHES:
        idx = torch.arange(B) % POOL
        got = _solve(P, kw, idx)
        for k in keys:
            v = got[k]
            bdim = 0 if v.dim() == 1 else 1
            for p in range(min(B, POOL)):
                sel = (idx == p).nonzero().flatten()
                want = alone[p][k].index_select(bdim, torch.tensor([0]))
                have = v.index_select(bdim, sel)
                same = _bits(have) == _bits(want.expand_as(have))
                if not bool(same.all()):
                    bad = sel[(~same).movedim(bdim, 0).reshape(len(sel), -1).any(1)]
                    pytest.fail(f"{mode} B={B}: {k} of pool problem {p} differs at batch positions "
                                f"{bad[:8].tolist()} from the problem solved alone")
