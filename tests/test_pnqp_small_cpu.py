"""CPU: the per-problem oracle (``orc.pnqp(coupled=False)``) against the reference's pnqp run one problem at a time
(oracle/make_golden_pnqp.py, fixtures ``pnqp1_*``), for the small QPs (n <= 8) of the one-thread-per-QP kernel."""
import glob
import os

import pytest
import torch

from oracle import lqr_oracle as orc
from tests.helpers import GOLD, load_golden, maxdiff

NAMES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLD, "pnqp1_*.npz")))


def test_fixtures_present():
    assert len(NAMES) == 8, NAMES


@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_single_problem_reference(name):
    g = load_golden(name)
    H, q, lo, hi = g["H"], g["q"], g["lower"], g["upper"]
    x, _, If, it = orc.pnqp(H, q, lo, hi, x_init=g.get("x_init"), n_iter=20, coupled=False)
    f64 = H.dtype == torch.float64
    assert maxdiff(x, g["x"]) <= (1e-12 if f64 else 1e-6)
    assert torch.equal(If.bool(), g["If"].bool())
    assert torch.equal(it, g["iters"].long()), (it.tolist(), g["iters"].tolist())
    if f64:
        # KKT check (as test_oracle_golden.test_pnqp_solves_the_box_qp): pnqp stops at |dx| < 1e-4
        grad = torch.einsum("bij,bj->bi", H, x) + q
        assert bool(((x >= lo - 1e-12) & (x <= hi + 1e-12)).all())
        interior = (x > lo + 1e-9) & (x < hi - 1e-9)
        assert float(grad[interior].abs().max()) < 2e-3
        assert bool((grad[x <= lo + 1e-12] > -2e-3).all())
        assert bool((grad[x >= hi - 1e-12] < 2e-3).all())
