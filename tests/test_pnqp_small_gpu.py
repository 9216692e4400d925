"""GPU: the standalone pnqp for n <= 8 (csrc/pnqp.cu: one thread per QP, on the pnqp_lane / Ldl code the step kernels
inline) against the per-problem CPU oracle (``orc.pnqp(coupled=False)``) and the reference's per-problem fixtures
(``pnqp1_*``, oracle/make_golden_pnqp.py).  The step kernels only instantiate that code at m in {1, 2, 4}; here every
size 1..8 runs, in batches that reach past the first 128-thread block.

Tolerances (those of the n > 8 suite, tests/test_pnqp_large_gpu.py): float64 x within 1e-9 * max(1, |x|_inf), H_free
within 1e-12, free sets, iteration counts and status exact.  float32 (inputs rounded to float32, compared with the
float64 oracle on the rounded inputs): free sets exact and x within 2e-4 (pnqp stops at |dx| < 1e-4) on every problem
that neither the kernel nor the oracle run in float32 leaves at the iteration cap; at most 5 % of the problems are
left out that way.
"""
import glob
import os

import pytest
import torch

from oracle import lqr_oracle as orc
from tests.gpu_harness import DEV, F32, F64, PNQP_ITER, check_qp_f64, gen_qp, pnqp_raw
from tests.helpers import GOLD, load_golden, maxdiff

pytestmark = pytest.mark.gpu
SIZES = [1, 2, 3, 4, 5, 6, 7, 8]
FIXTURES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLD, "pnqp1_*.npz")))
WARNING = "pnqp warning: Did not converge"


def oracle(H, q, lo, hi, x0=None, n_iter=PNQP_ITER):
    return orc.pnqp(H, q, lo, hi, x_init=x0, n_iter=n_iter, coupled=False)


def entry(H, q, lo, hi, x0=None, n_iter=PNQP_ITER):
    """mpc.pnqp.pnqp on the device; tensor arguments are moved there, floats passed as they are."""
    from mpc.pnqp import pnqp
    d = lambda t: t.to(DEV) if torch.is_tensor(t) else t  # noqa: E731
    x, Hf, If, i = pnqp(d(H), d(q), d(lo), d(hi), x_init=d(x0), n_iter=n_iter)
    torch.cuda.synchronize()
    return x.cpu(), Hf.cpu(), If.cpu(), i


def same_as_raw(e, got, tag):
    """The Python entry's (x, H_free, If, i) bit for bit against the raw call's per-problem outputs."""
    x, Hf, If, i = e
    assert torch.equal(x, got[0]) and torch.equal(Hf, got[1]), f"{tag}: entry x / H_free"
    assert If.dtype == x.dtype and torch.equal(If, got[2].to(x.dtype)), f"{tag}: entry If"
    assert i == int(got[3].max()), f"{tag}: entry i"


def check_f32(got, H, q, lo, hi, x0, tag, it32=None, also=None):
    """The float32 rule against the float64 oracle on the (float32) inputs; it32 is the float32 oracle's iteration
    count per problem (computed when not given); `also` is a further float32 solution (x, If) held to the same rule.
    Returns (problems, problems left out)."""
    x, _, If, iters, status = got
    d = lambda t: t.double() if t is not None else None  # noqa: E731
    x64, _, If64, _ = oracle(d(H), d(q), d(lo), d(hi), d(x0))
    if it32 is None:
        it32 = oracle(H, q, lo, hi, x0)[3]
    capped = (status & 1).bool()
    assert torch.equal(iters[capped], torch.full_like(iters[capped], PNQP_ITER - 1)), f"{tag}: capped iterations"
    assert int((status & ~1).abs().max()) == 0, f"{tag}: status {status.tolist()}"
    ok = ~capped & (it32 < PNQP_ITER - 1)
    for xs, Ifs, what in [(x64, If64, "float64 oracle")] + ([also + ("reference",)] if also else []):
        assert torch.equal(If.bool()[ok], Ifs.bool()[ok]), f"{tag}: free set vs the {what}"
        assert maxdiff(x[ok], xs[ok]) <= 2e-4, f"{tag}: x differs from the {what} by {maxdiff(x[ok], xs[ok]):.3g}"
    return len(x), int((~ok).sum())


def warns_iff_capped(capsys, got, H, q, lo, hi, x0, tag):
    """The Python entry on the same problem: the raw call's outputs, and the pnqp warning printed exactly when some
    problem stopped at the iteration cap.  Returns the entry's outputs."""
    capsys.readouterr()
    e = entry(H, q, lo, hi, x0)
    assert (WARNING in capsys.readouterr().out) == bool((got[4] & 1).any()), f"{tag}: warning"
    same_as_raw(e, got, tag)
    return e


# ------------------------------------------------------------------------------------------------------------------
# 1. the reference, run one problem at a time
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", FIXTURES)
def test_reference_fixture(name, capsys):
    g = load_golden(name)
    H, q, lo, hi, x0 = g["H"], g["q"], g["lower"], g["upper"], g.get("x_init")
    got = pnqp_raw(H, q, lo, hi, x0)
    if H.dtype == F64:
        assert maxdiff(got[0], g["x"]) <= 1e-10, f"x differs by {maxdiff(got[0], g['x']):.3g}"
        assert torch.equal(got[2].bool(), g["If"].bool())
        assert torch.equal(got[3], g["iters"].long()), (got[3].tolist(), g["iters"].tolist())
        check_qp_f64(got, oracle(H, q, lo, hi, x0), name)
        assert int(got[4].abs().max()) == 0
    else:
        total, left = check_f32(got, H, q, lo, hi, x0, name, it32=g["iters"].long(), also=(g["x"], g["If"]))
        assert left <= 0.05 * total
    assert warns_iff_capped(capsys, got, H, q, lo, hi, x0, name)[3] == int(g["iters"].max())


def test_every_fixture_present():
    assert len(FIXTURES) == 8, FIXTURES


# ------------------------------------------------------------------------------------------------------------------
# 2. float64 sweep against the oracle: every size, batches past one 128-thread block, three ways to give the bounds
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bounds", ["batch", "shared", "scalar"])
@pytest.mark.parametrize("start", ["cold", "warm"])
@pytest.mark.parametrize("B", [1, 129, 1000])
@pytest.mark.parametrize("n", SIZES)
def test_f64_sweep_matches_oracle(n, B, start, bounds):
    H, q, lo, hi, x0 = gen_qp(700 * n + B, B, n)
    x0 = x0 if start == "warm" else None
    if bounds == "shared":              # (n,): one box for the whole batch
        lo, hi = lo[0].clone(), hi[0].clone()
    elif bounds == "scalar":            # plain floats
        lo, hi = -0.5, 0.5
    dlo, dhi = (torch.full((B, n), v, dtype=F64) if not torch.is_tensor(v) else v for v in (lo, hi))
    got = pnqp_raw(H, q, dlo, dhi, x0)
    tag = f"n={n} B={B} {start} {bounds}"
    check_qp_f64(got, oracle(H, q, dlo, dhi, x0), tag)
    assert int(got[4].abs().max()) == 0, f"{tag}: status"
    same_as_raw(entry(H, q, lo, hi, x0), got, tag)


# ------------------------------------------------------------------------------------------------------------------
# 3. float32 against the float64 oracle
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("start", ["cold", "warm"])
@pytest.mark.parametrize("n", SIZES)
def test_f32_against_f64_oracle(n, start, capsys):
    B = 256
    H, q, lo, hi, x0 = (t.float() for t in gen_qp(5000 + n, B, n))
    x0 = x0 if start == "warm" else None
    got = pnqp_raw(H, q, lo, hi, x0)
    tag = f"n={n} {start}"
    total, left = check_f32(got, H, q, lo, hi, x0, tag)
    assert left <= 0.05 * total, f"{tag}: {left} of {total} problems at the iteration cap"
    warns_iff_capped(capsys, got, H, q, lo, hi, x0, tag)


# ------------------------------------------------------------------------------------------------------------------
# 4. special boxes
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", SIZES)
def test_special_boxes(n):
    B = 6
    H, q, lo, hi, x0 = gen_qp(70 * n, B, n)
    # bounds too wide to clamp anything: the Newton point; a warm start reaches it in one full step
    wlo, whi = torch.full((B, n), -1e3, dtype=F64), torch.full((B, n), 1e3, dtype=F64)
    newton = -torch.linalg.solve(H, q)
    for init, its in ((None, 0), (x0, 1)):
        got = pnqp_raw(H, q, wlo, whi, init)
        check_qp_f64(got, oracle(H, q, wlo, whi, init), f"wide n={n}")
        assert got[3].tolist() == [its] * B and bool(got[2].bool().all())
        assert maxdiff(got[0], newton) <= 1e-9 * max(1.0, float(newton.abs().max()))
    # a linear term that pushes every variable onto its lower bound: nothing stays free
    qc = 1e4 * (1.0 + torch.rand(B, n, generator=torch.Generator().manual_seed(n), dtype=F64))
    got = pnqp_raw(H, qc, lo, hi)
    check_qp_f64(got, oracle(H, qc, lo, hi), f"all clamped n={n}")
    assert torch.equal(got[0], lo) and not bool(got[2].bool().any())
    assert torch.equal(got[1], 1e-11 * torch.eye(n, dtype=F64).expand(B, n, n))
    # some variables fixed by lower == upper (the first variable of the first problem always)
    fixed = torch.rand(B, n, generator=torch.Generator().manual_seed(n + 1), dtype=F64) < 0.25
    fixed[0, 0] = True
    flo, fhi = lo.clone(), torch.where(fixed, lo, hi)
    for init in (None, x0):
        got = pnqp_raw(H, q, flo, fhi, init)
        check_qp_f64(got, oracle(H, q, flo, fhi, init), f"lo == hi n={n}")
        assert torch.equal(got[0][fixed], lo[fixed]) and not bool(got[2].bool()[fixed].any())
        assert int(got[4].abs().max()) == 0
    # a warm start outside the box (every other variable) is clamped onto it first
    far = torch.where(torch.arange(n) % 2 == 0, 4.0 * x0.sign() + x0, x0)
    got = pnqp_raw(H, q, lo, hi, far)
    check_qp_f64(got, oracle(H, q, lo, hi, far), f"x_init outside n={n}")
    assert int(got[4].abs().max()) == 0
    # a warm start at the oracle's own solution is already converged: no iteration, x returned as given
    xo = oracle(H, q, lo, hi)[0]
    got = pnqp_raw(H, q, lo, hi, xo)
    check_qp_f64(got, oracle(H, q, lo, hi, xo), f"warm at the solution n={n}")
    assert got[3].tolist() == [0] * B and torch.equal(got[0], xo)


# ------------------------------------------------------------------------------------------------------------------
# 5. exact ties: the (x == lo) & (g > 0) decision where g is exactly zero
# ------------------------------------------------------------------------------------------------------------------
def tie_problems(B, n, dtype, seed):
    """Diagonal H with power-of-two entries, dyadic q and bounds: every quantity pnqp computes is exact, so the
    unconstrained minimiser x* = -q / h lies exactly on a bound (g == 0 there: free), exactly on a variable with
    lo == hi (free too), strictly outside the box (clamped, g != 0) or inside it."""
    g = torch.Generator().manual_seed(seed)
    h = 2.0 ** torch.randint(-1, 3, (B, n), generator=g).double()
    xs = torch.randint(-16, 17, (B, n), generator=g).double() / 8       # x* in [-2, 2], multiples of 1/8
    step = torch.randint(1, 9, (B, n), generator=g).double() / 8
    kind = torch.randint(0, 6, (B, n), generator=g)
    kind[:, 0] = torch.arange(B) % 6                                   # every kind in every size
    lo = torch.where(kind == 0, xs, xs - step)                         # 0: x* on lo
    hi = torch.where(kind == 1, xs, xs + step)                         # 1: x* on hi
    hi = torch.where(kind == 2, xs, hi)                                # 2: lo == hi == x*
    lo = torch.where(kind == 2, xs, lo)
    lo, hi = torch.where(kind == 3, xs + step, lo), torch.where(kind == 3, xs + 2 * step, hi)   # 3: x* below lo
    lo, hi = torch.where(kind == 4, xs - 2 * step, lo), torch.where(kind == 4, xs - step, hi)  # 4: x* above hi
    H = torch.diag_embed(h)                                            # 5: x* inside
    q = -h * xs
    return [t.to(dtype) for t in (H, q, lo, hi)], kind


@pytest.mark.parametrize("dtype", [F32, F64], ids=["f32", "f64"])
@pytest.mark.parametrize("n", [2, 5, 8])
def test_exact_ties_bit_for_bit(n, dtype):
    B = 150
    (H, q, lo, hi), kind = tie_problems(B, n, dtype, 40 + n)
    got = pnqp_raw(H, q, lo, hi)
    xo, Ho, Ifo, ito = oracle(H, q, lo, hi)
    assert torch.equal(got[0], xo), f"x differs by {maxdiff(got[0], xo):.3g}"
    assert torch.equal(got[1], Ho), "H_free"
    assert torch.equal(got[2].bool(), Ifo.bool()), "free set"
    assert torch.equal(got[3], ito) and int(got[4].abs().max()) == 0
    assert torch.equal(got[2].bool(), (kind <= 2) | (kind == 5)), "ties must stay free, the strictly outside clamped"


# ------------------------------------------------------------------------------------------------------------------
# 6. batch independence: the thread of problem b reads and writes problem b only
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [F32, F64], ids=["f32", "f64"])
@pytest.mark.parametrize("n", [3, 8])
def test_results_do_not_depend_on_the_batch(n, dtype):
    B = 300
    H, q, lo, hi, x0 = (t.to(dtype) for t in gen_qp(77 + n, B, n))
    for init in (None, x0):
        a = pnqp_raw(H, q, lo, hi, init)
        b = pnqp_raw(H, q, lo, hi, init)
        for u, v in zip(a, b):
            assert torch.equal(u, v)
        for i in (0, 127, 128, 255, 256, 299):
            s = slice(i, i + 1)
            one = pnqp_raw(H[s], q[s], lo[s], hi[s], init[s] if init is not None else None)
            for u, v in zip(a, one):
                assert torch.equal(u[s], v), f"problem {i}"


# ------------------------------------------------------------------------------------------------------------------
# 7. the 8 -> 9 boundary between the one-thread kernel and the thread-block kernel
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("start", ["cold", "warm"])
def test_n8_equals_n9_with_a_decoupled_variable(start):
    """QPs at n = 8 and the same QPs with a ninth variable (H = 1, q = 0, box [-1, 1], no coupling), which sits at 0
    and stays free: the two kernels agree on the first eight coordinates."""
    B = 200
    H, q, lo, hi, x0 = gen_qp(98, B, 8)
    x0 = x0 if start == "warm" else None
    H9 = torch.zeros(B, 9, 9, dtype=F64)
    H9[:, :8, :8] = H
    H9[:, 8, 8] = 1.0
    pad = lambda t, v: torch.cat((t, torch.full((B, 1), v, dtype=F64)), 1)  # noqa: E731
    got8 = pnqp_raw(H, q, lo, hi, x0)
    got9 = pnqp_raw(H9, pad(q, 0.0), pad(lo, -1.0), pad(hi, 1.0), pad(x0, 0.0) if x0 is not None else None)
    assert torch.equal(got9[0][:, 8], torch.zeros(B, dtype=F64)) and bool(got9[2][:, 8].bool().all())
    scale = max(1.0, float(got8[0].abs().max()))
    assert maxdiff(got8[0], got9[0][:, :8]) <= 1e-12 * scale, f"x differs by {maxdiff(got8[0], got9[0][:, :8]):.3g}"
    assert torch.equal(got8[2], got9[2][:, :8]), "free set"
    assert torch.equal(got8[3], got9[3]), "iterations"
    assert torch.equal(got8[4], got9[4]), "status"


# ------------------------------------------------------------------------------------------------------------------
# 8. status bits
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", SIZES[1:])
def test_status_bits(n):
    B = 8
    g = torch.Generator().manual_seed(3 + n)
    Q, _ = torch.linalg.qr(torch.randn(B, n, n, generator=g, dtype=F64))
    lam = torch.linspace(-1.0, 5.0, n, dtype=F64)
    Hi = Q @ torch.diag_embed(lam.expand(B, n)) @ Q.transpose(1, 2)
    Hi = 0.5 * (Hi + Hi.transpose(1, 2))
    qi = torch.randn(B, n, generator=g, dtype=F64)
    status = pnqp_raw(Hi, qi, -torch.ones(B, n, dtype=F64), torch.ones(B, n, dtype=F64))[4]
    assert bool((status & 4).bool().all()), f"indefinite H: status {status.tolist()}"
    # one iteration allowed, from a start that is not converged: every problem stops at the cap after one step
    H, q, lo, hi, x0 = gen_qp(900 + n, B, n)
    got = pnqp_raw(H, q, lo, hi, x0, n_iter=1)
    check_qp_f64(got, oracle(H, q, lo, hi, x0, n_iter=1), f"n_iter=1 n={n}")
    assert got[3].tolist() == [0] * B and got[4].tolist() == [1] * B


def fixed_point_problems(B, n, seed):
    """float32 QPs that pnqp cannot leave: the free variables start 1e-3 from their optimum (|dx| > 1e-4), and a
    decoupled last variable fixed at 1e4 adds 5e7 to the objective, whose float32 spacing (4) swallows any decrease
    of the others; every Armijo trial fails (ratio 0), and the last one, x + 1e-9 dx, rounds back to x."""
    H, q, _, _, _ = gen_qp(seed, B, n)
    H[:, -1, :] = 0.0
    H[:, :, -1] = 0.0
    H[:, -1, -1] = 1.0
    q[:, -1] = 0.0
    lo, hi = torch.full((B, n), -100.0, dtype=F64), torch.full((B, n), 100.0, dtype=F64)
    lo[:, -1] = hi[:, -1] = 1e4
    d = torch.randn(B, n - 1, generator=torch.Generator().manual_seed(seed + 1), dtype=F64)
    xs = -torch.linalg.solve(H[:, :-1, :-1], q[:, :-1])
    x0 = torch.cat((xs + 1e-3 * d / d.norm(dim=1, keepdim=True), lo[:, -1:]), 1)
    return [t.float() for t in (H, q, lo, hi, x0)]


@pytest.mark.parametrize("n", SIZES[1:])
def test_f32_fixed_point_reports_the_cap(n, capsys):
    """At a float32 round-off fixed point every later iteration repeats the last one, so the kernel's early return must
    give what the reference's remaining iterations give: x unchanged, iterations n_iter - 1, the cap flag and the
    warning.  In float64 the same QPs converge."""
    B = 160
    H, q, lo, hi, x0 = fixed_point_problems(B, n, 300 + n)
    xo, Ho, Ifo, ito = oracle(H, q, lo, hi, x0)
    assert torch.equal(xo, x0) and ito.tolist() == [PNQP_ITER - 1] * B, "the float32 oracle must be stuck too"
    assert int(oracle(*(t.double() for t in (H, q, lo, hi, x0)))[3].max()) < PNQP_ITER - 1
    for n_iter in (PNQP_ITER, 5):
        got = pnqp_raw(H, q, lo, hi, x0, n_iter=n_iter)
        assert torch.equal(got[0], x0), f"n_iter={n_iter}: x moved"
        assert got[3].tolist() == [n_iter - 1] * B and got[4].tolist() == [1] * B, f"n_iter={n_iter}: iterations"
    got = pnqp_raw(H, q, lo, hi, x0)
    assert torch.equal(got[1], Ho) and torch.equal(got[2].bool(), Ifo.bool())
    warns_iff_capped(capsys, got, H, q, lo, hi, x0, f"fixed point n={n}")


# ------------------------------------------------------------------------------------------------------------------
# 9. the Python entry's argument forms
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [F32, F64], ids=["f32", "f64"])
def test_entry_argument_forms(dtype):
    B, n = 129, 5
    H, q, _, _, x0 = (t.to(dtype) for t in gen_qp(55, B, n))
    forms = [(-0.5, 0.5), (torch.full((n,), -0.5, dtype=dtype), torch.full((n,), 0.5, dtype=dtype)),
             (torch.full((1, n), -0.5, dtype=dtype), torch.full((1, n), 0.5, dtype=dtype)),
             (torch.full((B, n), -0.5, dtype=dtype), torch.full((B, n), 0.5, dtype=dtype))]
    for init in (None, x0[0], x0[:1].expand(B, n).contiguous()):
        outs = [entry(H, q, lo, hi, init) for lo, hi in forms]
        for k, o in enumerate(outs):
            assert o[2].dtype == dtype
            for u, v in zip(o[:3], outs[0][:3]):
                assert torch.equal(u, v), f"bounds form {k}"
            assert o[3] == outs[0][3]
    # x_init as (n,) is the same as that row for every problem
    a = entry(H, q, -0.5, 0.5, x0[0])
    b = entry(H, q, -0.5, 0.5, x0[:1].expand(B, n).contiguous())
    for u, v in zip(a[:3], b[:3]):
        assert torch.equal(u, v)
    assert a[3] == b[3]
