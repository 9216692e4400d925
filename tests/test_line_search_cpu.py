"""CPU: the line-search cases of tests/test_line_search_gpu.py are not vacuous, and the oracle matches the reference's
line search on the ls_* fixtures (oracle/make_golden_linesearch.py: the reference's LQRStep one problem at a time)."""
import glob
import os

import pytest
import torch

from oracle import lqr_oracle as orc
from tests.gpu_harness import (LS_MARGIN, MAX, MID, ONE, decays, ls_classes, rollout_passes, step_layout)
from tests.helpers import GOLD, load_golden, maxdiff
from tests.test_line_search_gpu import (ALONE_CASES, INSTANCE_OF, LOOP_CASES, LS_CASES, SHIFT_CASES, build_case,
                                        case_id, loop_case)

# (case, nominal from a shifted initial state)
CASES = [(c, False) for c in LS_CASES + ALONE_CASES] + [(c, True) for c in SHIFT_CASES]


@pytest.mark.parametrize("c,shifted", CASES, ids=[case_id(c) + ("_shifted" if s else "") for c, s in CASES])
def test_case_mixes_line_search_classes_in_a_warp_and_a_cta(c, shifted):
    kernel, n, m, dtype, T, B, mode, max_ls, decay, _ = c
    case = build_case(*c[:9], shifted=shifted)
    cls = case.classes
    ppw, W = step_layout(kernel, *INSTANCE_OF.get((n, m), (n, m)), dtype)
    # every comparison of every problem clears the margin, and a problem worse on every pass moved after pass 0
    old = case.o64.costs - case.trace[-1]
    p = rollout_passes(case.trace)
    counted = torch.arange(case.trace.shape[0]).view(-1, 1) < p.view(1, -1)
    assert bool(((case.trace.abs() >= LS_MARGIN * old.abs().clamp_min(1.0)) | ~counted).all())
    if max_ls > 1:
        assert bool(((case.first64 - case.o64.new_u).abs().amax((0, 2))[cls == MAX] > 0).all())
    assert torch.equal(decays(case.o64.alphas, decay), p - 1)
    groups = [range(w, min(w + ppw, B)) for w in range(0, B, ppw)] if ppw >= 3 else [range(B)]
    assert any({ONE, MAX} <= {int(cls[b]) for b in g} for g in groups), f"no warp holds one pass and max_ls: {cls}"
    ctas = [range(w, min(w + W, B)) for w in range(0, B, W)] if W >= 3 else [range(B)]
    assert any({ONE, MAX} <= {int(cls[b]) for b in g} for g in ctas), f"no CTA holds one pass and max_ls: {cls}"
    back = cls != ONE
    tail = (B - 1) // W * W
    assert bool(back[tail:].any()), f"the tail CTA [{tail}, {B}) has no problem that backtracks: {cls}"
    if ppw > 1:
        # a warp whose first problem takes one pass holds one that backtracks (a vote of lane 0 alone would stop it)
        assert any(cls[w] == ONE and bool(back[w + 1:w + ppw].any()) for w in range(0, B, ppw))
    if W > ppw:
        # an even CTA whose warp 0 takes one pass everywhere has a later warp that backtracks
        assert any(not bool(back[w:w + ppw].any()) and bool(back[w + ppw:w + W].any()) for w in range(0, B, 2 * W))


def test_every_kernel_meets_an_intermediate_pass_count():
    """Problems that backtrack and then improve with 1 < passes < max_ls: at every mapping, and at decay 0.9."""
    seen = set()
    for c, shifted in CASES:
        kernel, n, m, dtype, T, B, mode, max_ls, decay, _ = c
        case = build_case(*c[:9], shifted=shifted)
        p = rollout_passes(case.trace)
        if bool(((case.classes == MID) & (p < max_ls)).any()):
            seen.add(kernel)
            assert max_ls >= 3
    assert seen == {"generic", "pair", "large"}, seen


def test_step_feeds_back_the_initial_state_offset():
    """The oracle's (and the kernels') convention where current_x[0] != x_init: the first control of the full step is
    u_bar_0 + K_0 (x_init - x_bar_0) + k_0.  The reference starts its rollout from dx = 0 (lqr_step.py:181-182) and
    would give u_bar_0 + k_0; DESIGN.md section 4 records the difference."""
    n, m, T, B = 4, 2, 5, 6
    case = build_case("generic", n, m, torch.float64, T, B, "plain", 10, 0.5, shifted=True)
    P, o = case.P, case.o64
    off = P["x0"] - P["x"][0]
    assert float(off.abs().max()) > 0.1
    fb = P["u"][0] + torch.einsum("bij,bj->bi", o.Ks[0], off) + o.ks[0]
    assert maxdiff(case.first64[0], fb) <= 1e-12
    assert maxdiff(case.first64[0], P["u"][0] + o.ks[0]) > 1e-3


@pytest.mark.parametrize("c", LOOP_CASES, ids=[f"n{c[0]}m{c[1]}_{c[4]}" for c in LOOP_CASES])
def test_loop_cases_backtrack(c):
    o = loop_case(*c)[3]
    assert o["iters"] >= 2 and any(t["mean_alphas"] < 1 for t in o["trace"]), o["trace"]


NAMES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLD, "ls_*.npz")))


def test_fixtures_cover_the_settings():
    assert len(NAMES) == 4, NAMES
    gs = [load_golden(nm) for nm in NAMES]
    assert {int(g["max_linesearch_iter"]) for g in gs} >= {1, 3, 40}
    assert {float(g["linesearch_decay"]) for g in gs} >= {0.5, 0.9}
    assert any(bool((g["classes"] == MAX).any()) for g in gs)
    assert any(bool((g["classes"] == MID).any()) for g in gs)
    assert any("delta_u" in g and torch.is_tensor(g.get("u_lower")) for g in gs)
    assert any("u_zero_I" in g and "u_lower" in g for g in gs)


@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_reference_line_search(name):
    g = load_golden(name)
    T, B, p = g["C"].shape[:3]
    n = g["x_init"].shape[1]
    trace, first = [], []
    o = orc.lqr_step_forward(n, p - n, T, g["x_init"], g["C"], g["c"], g["F"], g["f"], g["cur_x"], g["cur_u"],
                             u_lower=g.get("u_lower"), u_upper=g.get("u_upper"), u_zero_I=g.get("u_zero_I"),
                             delta_u=g.get("delta_u"), linesearch_decay=g["linesearch_decay"],
                             max_linesearch_iter=int(g["max_linesearch_iter"]), coupled=False, ls_trace=trace,
                             first_u=first)
    assert maxdiff(o.new_x, g["new_x"]) <= 1e-10 and maxdiff(o.new_u, g["new_u"]) <= 1e-10
    assert maxdiff(o.costs, g["costs"]) <= 1e-9 * max(1.0, float(g["costs"].abs().max()))
    fdn = (g["cur_u"] - first[0]).pow(2).sum((0, 2)).sqrt()        # each problem's own full_du_norm
    assert maxdiff(fdn, g["full_du_norm"]) <= 1e-9 * max(1.0, float(g["full_du_norm"].abs().max()))
    assert torch.equal(o.alphas, g["alphas"])
    assert torch.equal(ls_classes(torch.stack(trace)), g["classes"].long())
