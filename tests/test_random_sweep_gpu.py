"""Seeded random sweep of the step entry point against the per-problem oracle: shapes (compiled instances and padded
ones), horizons, batch sizes incl. tail warps, dtype, scalar / tensor bounds, delta_u, time-varying F, missing f,
u_zero_I - each case under the default dispatch and under both kernels forced (MPCB200_KERNEL=1 generic, =2
column-pair; shapes the pair mapping does not take are skipped for that leg).

float64 cases: x, u, gains to 1e-9, pnqp free sets / iteration counts / clamp masks bit exact.
float32 cases: SURVEY.md section 8(c) tolerances; a QP whose stopping test is decided by round-off must be flagged
(tests/test_step_gpu.py explains) and is excluded from the bit-exact comparisons."""
import random

import pytest
import torch

from oracle import lqr_oracle as orc
from tests.gpu_harness import check_step_fixed, run_step
from tests.helpers import gen_problem, nominal_controls

pytestmark = pytest.mark.gpu
SHAPES = [(1, 1), (2, 1), (2, 2), (3, 1), (3, 2), (3, 4), (4, 1), (4, 2), (4, 4), (5, 1), (6, 2), (7, 4), (8, 1), (8, 2),
          (8, 4), (12, 4), (16, 4), (3, 3), (6, 1), (5, 2), (10, 2)]          # the last four run zero-padded


def make_cases(count=42, seed=2024):
    rng = random.Random(seed)
    cases = []
    for i in range(count):
        n, m = rng.choice(SHAPES)
        T = rng.choice([1, 2, 3, 5, 8, 12])
        B = rng.choice([1, 2, 5, 9, 16, 31, 37, 48, 64])
        dtype = torch.float32 if i % 3 == 2 else torch.float64
        bounds = rng.choice([None, None, 0.2, 0.4, "tensor"])
        delta = rng.choice([None, 0.15]) if bounds is not None else None
        tv, wf = rng.random() < 0.5, rng.random() < 0.7
        mask = bounds is None and rng.random() < 0.3
        cases.append((f"r{i}_n{n}m{m}_T{T}_B{B}_{'f32' if dtype == torch.float32 else 'f64'}_"
                      f"{'unb' if bounds is None else 'boxT' if bounds == 'tensor' else 'box'}"
                      f"{'_du' if delta else ''}{'_mask' if mask else ''}{'_tv' if tv else ''}{'' if wf else '_nof'}",
                      1000 + i, B, T, n, m, dtype, bounds, delta, tv, wf, mask))
    return cases


CASES = make_cases()


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_random_case_matches_oracle_under_every_kernel(case):
    from mpc.pytorch_b200._lib import MpcB200Error
    name, seed, B, T, n, m, dtype, bounds, delta, tv, wf, mask = case
    C, c, F, f, x0 = gen_problem(seed, B, T, n, m, dtype, tv, wf)
    if T == 1:
        F, f = torch.zeros(0, B, n, n + m, dtype=dtype), None
    u, ul, uu = nominal_controls(seed, B, T, m, dtype, bounds)
    x = orc.get_traj(T, u, x0, F, f)
    kw = dict(u_lower=ul, u_upper=uu, delta_u=delta)
    if mask:
        g = torch.Generator().manual_seed(seed)
        kw["u_zero_I"] = torch.rand(T, B, m, generator=g) < 0.3
    o = orc.lqr_step_forward(n, m, T, x0, C, c, F, f, x, u, coupled=False, **kw)
    P = dict(x0=x0, C=C, c=c, F=F, f=f, x=x, u=u)
    ran = 0
    for impl in (None, "1", "2"):
        try:
            r, _ = run_step(n, m, T, P, kw, impl=impl)
        except MpcB200Error as e:
            if impl == "2" and "[3]" in str(e):
                continue                      # the column-pair mapping does not take this shape / alignment
            raise
        ran += 1
        check_step_fixed(f"{name} impl={impl}", r, o, kw, dtype)
    assert ran >= 2
