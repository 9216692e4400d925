"""GPU: gradients through the standalone pnqp (mpc.pnqp.pnqp with inputs that require grad, mpcb200_pnqp_backward_*)
against the float64 implicit-gradient oracle (oracle/pnqp_grad_oracle.py), central differences of the float64 forward
kernel, torch.autograd.gradcheck and the reference's unrolled autograd (fixture boxqp_grad_f64).

Tolerances: float64 within 1e-10 x max|grad| of the oracle evaluated at the kernel's own x and free set; float32 by
tests/gpu_harness.within (4 x the error of the oracle run in float32 on the same float32 x and inputs, plus 1e-6 x
max|grad|); the reference fixture within 1e-8 x max|grad|; central differences within 1e-5 x (1 + |derivative|).
The formula is the derivative of pnqp itself only on settled problems (oracle.pnqp_grad_oracle.settled: converged,
strictly complementary, last step a full Newton step on the final free set), so the difference checks run on those.
"""
import numpy as np
import pytest
import torch

from oracle.pnqp_grad_oracle import pnqp_grad, settled
from tests.gpu_harness import DEV, F32, F64, PNQP_ITER, gen_qp, pnqp_raw, to_dev, within
from tests.helpers import GOLD

pytestmark = pytest.mark.gpu
NAMES = ("H", "q", "lower", "upper")
WARNING = "pnqp warning"


def max_n(dtype):
    from mpc.pytorch_b200 import _lib
    with _lib._on_device(DEV):
        return _lib.lib().mpcb200_pnqp_max_n(torch.empty(0, dtype=dtype).element_size())


def entry_grads(H, q, lo, hi, x0, w, n_iter=PNQP_ITER):
    """mpc.pnqp.pnqp on the device with every tensor among (H, q, lower, upper) requiring grad, then backward of
    sum(w * x).  Returns (x, If, {name: grad}) on the CPU."""
    from mpc.pnqp import pnqp
    args = [to_dev(t).requires_grad_(True) if torch.is_tensor(t) else t for t in (H, q, lo, hi)]
    x, _, If, _ = pnqp(*args, x_init=to_dev(x0), n_iter=n_iter)
    assert x.grad_fn is not None
    (to_dev(w) * x).sum().backward()
    return x.detach().cpu(), If.cpu(), {k: a.grad.cpu() for k, a in zip(NAMES, args) if torch.is_tensor(a)}


def oracle_grads(H, q, lo, hi, x, If, w):
    """The oracle at (x, If), each gradient summed to the shape of its input (floats get none)."""
    full = dict(zip(NAMES, pnqp_grad(H, x, If, lo, hi, w)))
    return {k: full[k].sum_to_size(t.shape) for k, t in zip(NAMES, (H, q, lo, hi)) if torch.is_tensor(t)}


def check_f64(tag, got, want, tol=1e-10):
    scale = max(max(float(t.abs().max()) for t in want.values()), 1e-300)
    assert got.keys() == want.keys(), tag
    for k in want:
        err = float((got[k] - want[k]).abs().max())
        assert err <= tol * scale, f"{tag}: d{k} |kernel - oracle| = {err:.3e} > {tol:.0e} x {scale:.3e}"


def check_case(tag, dtype, H, q, lo, hi, x0, w):
    """The entry's gradients against the oracle at the kernel's x and free set: float64 to 1e-10, float32 by within."""
    cast = lambda t: t.to(dtype) if torch.is_tensor(t) else t  # noqa: E731
    H, q, lo, hi, x0, w = (cast(t) for t in (H, q, lo, hi, x0, w))
    x, If, got = entry_grads(H, q, lo, hi, x0, w)
    if dtype == F64:
        check_f64(tag, got, oracle_grads(H, q, lo, hi, x, If, w))
        return
    d = lambda t: t.double() if torch.is_tensor(t) else t  # noqa: E731
    w64 = oracle_grads(*(d(t) for t in (H, q, lo, hi, x, If, w)))
    w32 = oracle_grads(H, q, lo, hi, x, If, w)
    scale = max(float(t.abs().max()) for t in w64.values())
    for k in w64:
        within(tag, f"d{k}", got[k].double(), w64[k], w32[k].double(), F32, scale=scale)


# ------------------------------------------------------------------------------------------------------------------
# 1. against the oracle: every size of the thread-per-QP kernel, the thread-block kernel up to max_n, both dtypes
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [F32, F64], ids=["f32", "f64"])
@pytest.mark.parametrize("start", ["cold", "warm"])
@pytest.mark.parametrize("B", [1, 129, 300])
@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 6, 7, 8])
def test_small_matches_oracle(n, B, start, dtype):
    H, q, lo, hi, x0 = gen_qp(31 * n + B, B, n)
    check_case(f"n={n} B={B} {start}", dtype, H, q, lo, hi, x0 if start == "warm" else None,
               torch.randn(B, n, generator=torch.Generator().manual_seed(n), dtype=F64))


@pytest.mark.parametrize("dtype", [F32, F64], ids=["f32", "f64"])
@pytest.mark.parametrize("start", ["cold", "warm"])
@pytest.mark.parametrize("n", [9, 16, 33, 64, 100, "max"])
def test_large_matches_oracle(n, start, dtype):
    n = max_n(dtype) if n == "max" else n
    B = 5
    H, q, lo, hi, x0 = gen_qp(17 * n, B, n)
    check_case(f"n={n} {start}", dtype, H, q, lo, hi, x0 if start == "warm" else None,
               torch.randn(B, n, generator=torch.Generator().manual_seed(n), dtype=F64))


# ------------------------------------------------------------------------------------------------------------------
# 2. every broadcast form of q, lower and upper: [B, n], [n], [1, n], and a float for the bounds
# ------------------------------------------------------------------------------------------------------------------
def forms(t, allow_float):
    out = {"batch": t, "row": t[0].clone(), "row1": t[:1].clone()}
    if allow_float:
        out["float"] = float(t[0, 0])
    return out


@pytest.mark.parametrize("n", [3, 12])
def test_every_broadcast_form(n):
    B = 129
    H, q, lo, hi, x0 = gen_qp(400 + n, B, n)
    lo, hi = lo.clamp(max=-0.3), hi.clamp(min=0.3)
    w = torch.randn(B, n, generator=torch.Generator().manual_seed(n), dtype=F64)
    for qf, qv in forms(q, False).items():
        for lf, lv in forms(lo, True).items():
            for hf, hv in forms(hi, True).items():
                check_case(f"n={n} q {qf} lower {lf} upper {hf}", F64, H, qv, lv, hv, None, w)


# ------------------------------------------------------------------------------------------------------------------
# 3. special problems: free, lower- and upper-clamped and weakly active coordinates; all free; all clamped
# ------------------------------------------------------------------------------------------------------------------
def mixed_problems(B, n, seed):
    """Diagonal H with power-of-two entries and dyadic q and bounds, so every quantity pnqp computes is exact, plus a
    coupled block on the first two variables: the unconstrained minimiser lies inside the box, outside it below or
    above, or exactly on a bound (g == 0 there: weakly active, which pnqp keeps free)."""
    g = torch.Generator().manual_seed(seed)
    h = 2.0 ** torch.randint(-1, 3, (B, n), generator=g).double()
    xs = torch.randint(-16, 17, (B, n), generator=g).double() / 8
    step = torch.randint(1, 9, (B, n), generator=g).double() / 8
    kind = torch.randint(0, 5, (B, n), generator=g)
    kind[:, 0] = torch.arange(B) % 5
    lo = torch.where(kind == 0, xs, xs - step)                                # 0: on lower, weakly active
    hi = torch.where(kind == 1, xs, xs + step)                                # 1: on upper, weakly active
    lo, hi = torch.where(kind == 2, xs + step, lo), torch.where(kind == 2, xs + 2 * step, hi)   # 2: below lower
    lo, hi = torch.where(kind == 3, xs - 2 * step, lo), torch.where(kind == 3, xs - step, hi)   # 3: above upper
    H = torch.diag_embed(h)                                                   # 4: inside
    if n > 1:
        H[:, 0, 1] = H[:, 1, 0] = 0.25 * torch.minimum(h[:, 0], h[:, 1])
    return H, -h * xs, lo, hi


@pytest.mark.parametrize("dtype", [F32, F64], ids=["f32", "f64"])
@pytest.mark.parametrize("n", [1, 2, 5, 8, 9, 40])
def test_special_problems(n, dtype):
    B = 150
    w = torch.randn(B, n, generator=torch.Generator().manual_seed(7 * n), dtype=F64)
    H, q, lo, hi = mixed_problems(B, n, 50 + n)
    check_case(f"mixed n={n}", dtype, H, q, lo, hi, None, w)
    H, q, lo, hi, x0 = gen_qp(60 + n, B, n)
    wide = torch.full((B, n), 1e3, dtype=F64)
    check_case(f"all free n={n}", dtype, H, q, -wide, wide, x0, w)
    qc = 1e4 * (1.0 + torch.rand(B, n, generator=torch.Generator().manual_seed(n), dtype=F64))
    x, If, got = entry_grads(H.to(dtype), qc.to(dtype), lo.to(dtype), hi.to(dtype), None, w.to(dtype))
    assert not bool(If.bool().any()) and torch.equal(x, lo.to(dtype))
    assert torch.equal(got["lower"], w.to(dtype)), "all clamped at lower: dL/dx passes to lower unchanged"
    for k in ("H", "q", "upper"):
        assert not bool(got[k].any()), f"all clamped: d{k} must be 0"


# ------------------------------------------------------------------------------------------------------------------
# 4. the derivative of the forward kernel itself: central differences and gradcheck on settled problems
# ------------------------------------------------------------------------------------------------------------------
def settled_problems(seed, B, n):
    H, q, lo, hi, x0 = gen_qp(seed, B, n)
    x, _, If, _, status = pnqp_raw(H, q, lo, hi)
    keep = settled(H, q, lo, hi, x, If) & (status == 0)
    assert int(keep.sum()) >= B // 2, f"only {int(keep.sum())} of {B} problems settled"
    return tuple(t[keep] for t in (H, q, lo, hi))


@pytest.mark.parametrize("n", [1, 2, 5, 8, 12, 40])
def test_central_differences(n):
    H, q, lo, hi = settled_problems(800 + n, 48, n)
    B = H.shape[0]
    g = torch.Generator().manual_seed(n)
    w = torch.randn(B, n, generator=g, dtype=F64)
    _, _, got = entry_grads(H, q, lo, hi, None, w)
    eps = 1e-5     # pnqp's 1e-11 regularisation leaves x within ~1e-11 of the free-set minimiser: ~1e-6 of a difference
    for k in range(3):
        S = torch.randn(B, n, n, generator=g, dtype=F64)
        dirs = [0.5 * (S + S.transpose(1, 2))] + [torch.randn(B, n, generator=g, dtype=F64) for _ in range(3)]
        f = lambda s: (w * pnqp_raw(*(t + s * eps * d for t, d in zip((H, q, lo, hi), dirs)))[0]).sum(1)  # noqa
        fd = (f(1.0) - f(-1.0)) / (2 * eps)
        an = sum((got[nm] * d).flatten(1).sum(1) for nm, d in zip(NAMES, dirs))
        err = (fd - an).abs() / (1.0 + an.abs())
        assert float(err.max()) <= 1e-5, f"n={n} direction {k}: central difference off by {float(err.max()):.3g}"


@pytest.mark.parametrize("n,B", [(3, 2), (10, 1)])
def test_gradcheck(n, B):
    """gradcheck in float64 through a symmetric H = (A + A^T) / 2: pnqp reads H as symmetric, so a perturbation of one
    entry alone is not a problem it solves."""
    from mpc.pnqp import pnqp
    H, q, lo, hi = (t[:B].to(DEV).requires_grad_(True) for t in settled_problems(900 + n, 8 * B, n))
    fn = lambda A, q_, l_, h_: pnqp(0.5 * (A + A.transpose(1, 2)), q_, l_, h_, n_iter=PNQP_ITER)[0]  # noqa: E731
    assert torch.autograd.gradcheck(fn, (H, q, lo, hi))


# ------------------------------------------------------------------------------------------------------------------
# 5. the reference's unrolled autograd
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag", [f"n{n}_{s}" for n in (1, 2, 5, 8, 12, 40) for s in ("cold", "warm")])
def test_reference_fixture(tag):
    z = np.load(f"{GOLD}/boxqp_grad_f64.npz")
    g = {k[len(tag) + 1:]: torch.from_numpy(z[k]) for k in z.files if k.startswith(tag + "_")}
    x, If, got = entry_grads(g["H"], g["q"], g["lower"], g["upper"], g.get("x_init"), g["w"])
    assert float((x - g["x"]).abs().max()) <= 1e-9 and torch.equal(If.bool(), g["If"].bool()), tag
    check_f64(f"{tag} vs the reference", got, {k: g["d" + k] for k in NAMES}, tol=1e-8)


# ------------------------------------------------------------------------------------------------------------------
# 6. repeatability, the path without grad, in-place edits, the bad-pivot warning
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [F32, F64], ids=["f32", "f64"])
@pytest.mark.parametrize("n,B", [(5, 300), (40, 64)])
def test_gradients_repeat_bit_for_bit(n, B, dtype):
    H, q, lo, hi, x0 = (t.to(dtype) for t in gen_qp(70 + n, B, n))
    w = torch.randn(B, n, generator=torch.Generator().manual_seed(n), dtype=dtype)
    first = entry_grads(H, q, lo, hi, x0, w)[2]
    for _ in range(2):
        again = entry_grads(H, q, lo, hi, x0, w)[2]
        for k in first:
            assert torch.equal(first[k], again[k]), f"d{k} changed between calls"


@pytest.mark.parametrize("n", [4, 20])
def test_without_grad_nothing_changes(n):
    """No input requiring grad, or grad mode off: the raw forward's outputs bit for bit, no library launch counted
    beyond the raw call's, and an x without grad_fn.  With grad, the forward's outputs are the same bits too."""
    from mpc.pnqp import pnqp
    from mpc.pytorch_b200 import _lib
    B = 129
    H, q, lo, hi, x0 = gen_qp(5 + n, B, n)
    before = _lib.launch_count()
    raw = pnqp_raw(H, q, lo, hi, x0)
    raw_launches = _lib.launch_count() - before
    dev = [t.to(DEV) for t in (H, q, lo, hi, x0)]
    for how in ("plain", "no_grad", "grad"):
        args = [t.clone().requires_grad_(how != "plain") for t in dev[:4]]
        before = _lib.launch_count()
        if how == "no_grad":
            with torch.no_grad():
                x, Hf, If, it = pnqp(*args, x_init=dev[4], n_iter=PNQP_ITER)
        else:
            x, Hf, If, it = pnqp(*args, x_init=dev[4], n_iter=PNQP_ITER)
        assert _lib.launch_count() - before == raw_launches, how
        assert (x.grad_fn is None) == (how != "grad"), how
        assert torch.equal(x.detach().cpu(), raw[0]) and torch.equal(Hf.cpu(), raw[1]), how
        assert torch.equal(If.cpu(), raw[2].to(F64)) and it == int(raw[3].max()), how
        assert not Hf.requires_grad and not If.requires_grad


@pytest.mark.parametrize("n", [4, 20])
def test_in_place_edit_before_backward_raises(n):
    from mpc.pnqp import pnqp
    B = 3
    H, q, lo, hi, _ = gen_qp(9 + n, B, n)
    for edited in ("H", "lower", "upper", "x"):
        args = [t.to(DEV).requires_grad_(True) for t in (H, q, lo[0], hi)]   # lower as an [n] row
        x, _, _, _ = pnqp(*args, n_iter=PNQP_ITER)
        target = x if edited == "x" else args[NAMES.index(edited)]
        with torch.no_grad():
            target.mul_(1.0)
        with pytest.raises(RuntimeError, match="modified by an inplace operation"):
            x.sum().backward()


@pytest.mark.parametrize("n", [5, 40])
def test_bad_pivot_warns(n, capsys):
    """An indefinite H whose free block keeps a negative pivot: the backward's status bit 4, printed as a warning."""
    from mpc.pnqp import pnqp
    B = 3
    g = torch.Generator().manual_seed(3)
    Q, _ = torch.linalg.qr(torch.randn(B, n, n, generator=g, dtype=F64))
    H = Q @ torch.diag_embed(torch.linspace(-1.0, 5.0, n, dtype=F64).expand(B, n)) @ Q.transpose(1, 2)
    H = (0.5 * (H + H.transpose(1, 2))).to(DEV).requires_grad_(True)
    q = torch.randn(B, n, generator=g, dtype=F64).to(DEV)
    x, _, If, _ = pnqp(H, q, -1e3, 1e3, n_iter=PNQP_ITER)
    assert bool(If.bool().all())
    capsys.readouterr()
    x.sum().backward()
    assert "bad pivot" in capsys.readouterr().out
    capsys.readouterr()
    good = torch.eye(n, dtype=F64, device=DEV).expand(B, n, n).clone().requires_grad_(True)
    pnqp(good, q, -1e3, 1e3, n_iter=PNQP_ITER)[0].sum().backward()
    assert WARNING not in capsys.readouterr().out
