"""GPU: the standalone pnqp for n > 8 (one thread block per QP) against the per-problem CPU oracle
(``orc.pnqp(coupled=False)``) and the reference's n = 100 fixture.

Tolerances: float64 x within 1e-9 * max(1, |x|_inf), H_free within 1e-12, free sets, iteration counts and status
exact.  float32 (inputs rounded to float32, compared with the float64 oracle on the rounded inputs): free sets exact
and x within 2e-4 (pnqp stops at |dx| < 1e-4) on every problem that neither the kernel nor the oracle run in float32
leaves at the iteration cap; in float32 a few problems reach a round-off fixed point above the step tolerance.
"""
import pytest
import torch

from oracle import lqr_oracle as orc
from tests.gpu_harness import DEV, F64, PNQP_ITER as N_ITER, check_qp_f64 as check_f64, gen_qp, pnqp_raw as raw
from tests.helpers import load_golden, maxdiff

pytestmark = pytest.mark.gpu


def max_n(dtype):
    from mpc.pytorch_b200 import _lib
    with _lib._on_device(DEV):
        return _lib.lib().mpcb200_pnqp_max_n(torch.empty(0, dtype=dtype).element_size())


def test_reference_fixture_n100():
    """The reference's test_lqr_qp shape (two QPs, n = 100) through the drop-in mpc.pnqp.pnqp."""
    from mpc.pnqp import pnqp
    g = load_golden("pnqp_f64_n100")
    H, q, lo, hi = (g[k] for k in ("H", "q", "lower", "upper"))
    x, Hf, If, it = pnqp(H.to(DEV), q.to(DEV), lo.to(DEV), hi.to(DEV), n_iter=N_ITER)
    xo, Ho, Ifo, ito = orc.pnqp(H, q, lo, hi, n_iter=N_ITER, coupled=False)
    assert maxdiff(x, g["x"]) <= 1e-9 and maxdiff(x, xo) <= 1e-9
    assert torch.equal(If.cpu().bool(), g["If"].bool())
    assert it == 5 == g["n_iter"] == int(ito.max())
    assert maxdiff(Hf, Ho) <= 1e-12


SIZES = [9, 16, 31, 32, 33, 63, 64, 65, 100, 127, 128, "max"]    # one warp per QP up to 32, four warps above


@pytest.mark.parametrize("bounds", ["batch", "shared", "scalar"])
@pytest.mark.parametrize("start", ["cold", "warm"])
@pytest.mark.parametrize("B", [1, 3, 64])
@pytest.mark.parametrize("n", SIZES)
def test_f64_sweep_matches_oracle(n, B, start, bounds):
    from mpc.pnqp import pnqp
    n = max_n(F64) if n == "max" else n
    H, q, lo, hi, x0 = gen_qp(1000 * n + B, B, n)
    if bounds == "shared":              # (n,): one box for the whole batch
        lo, hi = lo[0].clone(), hi[0].clone()
    elif bounds == "scalar":            # a scalar box given as (1, n)
        lo, hi = torch.full((1, n), -0.5, dtype=F64), torch.full((1, n), 0.5, dtype=F64)
    x0 = x0 if start == "warm" else None
    got = raw(H, q, lo, hi, x0)
    check_f64(got, orc.pnqp(H, q, lo, hi, x_init=x0, n_iter=N_ITER, coupled=False), f"n={n} B={B}")
    assert int(got[4].abs().max()) == 0, "status"
    # the Python entry point broadcasts the same bounds and launches the same kernel
    x, Hf, If, it = pnqp(H.to(DEV), q.to(DEV), lo.to(DEV), hi.to(DEV),
                         x_init=x0.to(DEV) if x0 is not None else None, n_iter=N_ITER)
    assert torch.equal(x.cpu(), got[0]) and torch.equal(Hf.cpu(), got[1])
    assert torch.equal(If.cpu(), got[2].to(F64)) and it == int(got[3].max())


@pytest.mark.parametrize("n", [9, 32, 33, 100, "max"])
def test_special_boxes(n):
    n = max_n(F64) if n == "max" else n
    B = 5
    H, q, lo, hi, x0 = gen_qp(7 * n, B, n)
    # bounds too wide to clamp anything: the Newton point; a warm start reaches it in one full step
    wlo, whi = torch.full((B, n), -1e3, dtype=F64), torch.full((B, n), 1e3, dtype=F64)
    newton = -torch.linalg.solve(H, q)
    for init, its in ((None, 0), (x0, 1)):
        got = raw(H, q, wlo, whi, init)
        check_f64(got, orc.pnqp(H, q, wlo, whi, x_init=init, n_iter=N_ITER, coupled=False), f"wide n={n}")
        assert got[3].tolist() == [its] * B and bool(got[2].bool().all())
        assert maxdiff(got[0], newton) <= 1e-9 * max(1.0, float(newton.abs().max()))
    # a linear term that pushes every variable onto its lower bound: nothing stays free
    qc = 1e4 * (1.0 + torch.rand(B, n, generator=torch.Generator().manual_seed(n), dtype=F64))
    got = raw(H, qc, lo, hi)
    check_f64(got, orc.pnqp(H, qc, lo, hi, n_iter=N_ITER, coupled=False), f"all clamped n={n}")
    assert torch.equal(got[0], lo) and not bool(got[2].bool().any())
    assert torch.equal(got[1], 1e-11 * torch.eye(n, dtype=F64).expand(B, n, n))
    # some variables fixed by lower == upper
    fixed = torch.rand(B, n, generator=torch.Generator().manual_seed(n + 1), dtype=F64) < 0.2
    flo, fhi = lo.clone(), torch.where(fixed, lo, hi)
    for init in (None, x0):
        got = raw(H, q, flo, fhi, init)
        check_f64(got, orc.pnqp(H, q, flo, fhi, x_init=init, n_iter=N_ITER, coupled=False), f"lo == hi n={n}")
        assert torch.equal(got[0][fixed], lo[fixed]) and not bool(got[2].bool()[fixed].any())
        assert int(got[4].abs().max()) == 0


def test_f32_against_f64_oracle(capsys):
    """Inputs rounded to float32; the float64 oracle on the rounded inputs is the yardstick."""
    from mpc.pnqp import pnqp
    B, total, excluded = 64, 0, 0
    for n in [9, 32, 33, 64, 100, 128, max_n(torch.float32)]:
        H, q, lo, hi, x0 = (t.float() for t in gen_qp(5000 + n, B, n))
        for init in (None, x0):
            x, _, If, iters, status = raw(H, q, lo, hi, init)
            x64, _, If64, _ = orc.pnqp(H.double(), q.double(), lo.double(), hi.double(),
                                       x_init=init.double() if init is not None else None, n_iter=N_ITER,
                                       coupled=False)
            _, _, _, it32 = orc.pnqp(H, q, lo, hi, x_init=init, n_iter=N_ITER, coupled=False)
            capped = (status & 1).bool()
            assert torch.equal(iters[capped], torch.full_like(iters[capped], N_ITER - 1))
            assert int((status & ~1).abs().max()) == 0
            ok = ~capped & (it32 < N_ITER - 1)
            total += B
            excluded += int((~ok).sum())
            tag = f"n={n} {'warm' if init is not None else 'cold'}"
            assert torch.equal(If.bool()[ok], If64.bool()[ok]), f"{tag}: free set"
            assert maxdiff(x[ok], x64[ok]) <= 2e-4, f"{tag}: x differs by {maxdiff(x[ok], x64[ok]):.3g}"
            capsys.readouterr()
            pnqp(H.to(DEV), q.to(DEV), lo.to(DEV), hi.to(DEV), x_init=init.to(DEV) if init is not None else None,
                 n_iter=N_ITER)
            warned = "pnqp warning: Did not converge" in capsys.readouterr().out
            assert warned == bool(capped.any()), tag
    assert excluded <= 0.05 * total, f"{excluded} of {total} problems at the iteration cap"


@pytest.mark.parametrize("n,dtype", [(20, torch.float32), (100, F64)])
def test_results_do_not_depend_on_the_batch(n, dtype):
    H, q, lo, hi, x0 = (t.to(dtype) for t in gen_qp(77 + n, 64, n))
    for init in (None, x0):
        a = raw(H, q, lo, hi, init)
        b = raw(H, q, lo, hi, init)
        for u, v in zip(a, b):
            assert torch.equal(u, v)
        for i in range(64):
            one = raw(H[i:i + 1], q[i:i + 1], lo[i:i + 1], hi[i:i + 1], init[i:i + 1] if init is not None else None)
            for u, v in zip(a, one):
                assert torch.equal(u[i:i + 1], v), f"problem {i}"


def test_indefinite_H_sets_bad_pivot():
    n, B = 40, 3
    g = torch.Generator().manual_seed(3)
    Q, _ = torch.linalg.qr(torch.randn(B, n, n, generator=g, dtype=F64))
    lam = torch.linspace(-1.0, 5.0, n, dtype=F64)
    H = Q @ torch.diag_embed(lam.expand(B, n)) @ Q.transpose(1, 2)
    H = 0.5 * (H + H.transpose(1, 2))
    q = torch.randn(B, n, generator=g, dtype=F64)
    status = raw(H, q, -torch.ones(B, n, dtype=F64), torch.ones(B, n, dtype=F64))[4]
    assert bool((status & 4).bool().all()), status.tolist()


def test_iteration_cap_of_one():
    g = load_golden("pnqp_f64_n100")
    H, q, lo, hi = (g[k] for k in ("H", "q", "lower", "upper"))
    got = raw(H, q, lo, hi, n_iter=1)
    check_f64(got, orc.pnqp(H, q, lo, hi, n_iter=1, coupled=False), "n_iter=1")
    assert got[3].tolist() == [0, 0] and got[4].tolist() == [1, 1]


def test_above_max_n_is_refused():
    from mpc.pnqp import pnqp
    from mpc.pytorch_b200 import _lib
    from mpc.pytorch_b200._lib import MpcB200Error
    for dtype in (torch.float32, F64):
        n = max_n(dtype) + 1
        H = torch.eye(n, dtype=dtype, device=DEV).unsqueeze(0)
        q = torch.zeros(1, n, dtype=dtype, device=DEV)
        with pytest.raises(MpcB200Error, match=rf"n <= {n - 1}\b"):
            pnqp(H, q, -1.0, 1.0)
        out = [torch.empty(1, n, dtype=dtype, device=DEV), torch.empty(1, n, n, dtype=dtype, device=DEV),
               torch.empty(1, n, dtype=torch.uint8, device=DEV), torch.empty(1, dtype=torch.int32, device=DEV),
               torch.empty(1, dtype=torch.int32, device=DEV)]
        fn = _lib.entry("mpcb200_pnqp", dtype)
        with _lib._on_device(DEV):
            rc = fn(1, n, _lib.ptr(H), _lib.ptr(q), _lib.ptr(q), _lib.ptr(q), None, N_ITER,
                    *[_lib.ptr(t) for t in out], _lib.stream_handle(DEV))
        assert rc == 4   # MPCB200_ERR_SMEM
