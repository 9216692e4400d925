"""CPU: the case builders of tests/test_receding_window_oracle_gpu.py reach what they are meant to reach, without a
device, and window_oracle's whole-input option (the forms of an episode whose window record leaves an input's bit
clear) is the windowed oracle on an input constant along the axis.  The grid cap and the block size are read from
csrc/episode_grad.cu (epgrad_grid, the window kernels' launches)."""
import math
import os
import re

import pytest
import torch

from mpc.pytorch_b200 import step as S
from oracle import window_oracle as wo
from tests import test_receding_window_oracle_gpu as M
from tests.gpu_harness import F64, INSTANCES, SWITCH_PLANS
from tests.helpers import maxdiff

SRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "mpc", "pytorch_b200", "csrc",
                   "episode_grad.cu")


def _cap():
    src = open(SRC).read()
    cap = re.search(r"static unsigned epgrad_grid\(size_t items\) \{.*?g > (\d+) \? (\d+) : g", src, re.S)
    assert cap and cap.group(1) == cap.group(2)
    blocks = {int(b) for b in re.findall(r"(?:window_stage_kernel|epgrad_\w*window_kernel)<[^>]*><<<[^,]+, (\d+),",
                                         src)}
    assert blocks == {256}, blocks
    return int(cap.group(1)) * 256


def test_grid_cap_read_from_the_source():
    assert M.GRID_CAP == _cap() == 1 << 20


@pytest.mark.parametrize("name", list(M.GRID))
def test_grid_cases_take_two_passes(name):
    """Every window loop a grid case targets runs on a capped grid and needs at least two passes of it: the window
    copy, the init's full-length zeroing (L B P^2), the accumulate and the windowed LinDx stage (B P) of the model or
    the plant."""
    cap = _cap()
    loops = M.grid_loops(name)
    stage = "plant stage" if M.GRID[name]["plant"] != "none" else "model stage"
    assert {"window copy", "init zeroing", "accumulate", stage} == set(loops)
    for loop, (items, capped) in loops.items():
        assert capped, f"{name}: the grid of the {loop} loop is not capped"
        assert items > cap, f"{name}: the {loop} loop has {items} items, one pass"
    assert {g["plant"] for g in M.GRID.values()} == {"none", "lin"}


@pytest.mark.parametrize("name", list(M.GRID))
def test_pool_layout_reaches_every_position(name):
    """Element b is pool problem b mod K, K coprime to the block, N and P: every pool problem has copies in the second
    pass of every targeted loop."""
    K, idx = M.grid_pool(name)
    g = M.GRID[name]
    N, P, B = g["n"], g["n"] + g["m"], g["B"]
    assert math.gcd(K, 256) == 1 and math.gcd(K, N) == 1 and math.gcd(K, P) == 1 and K >= 3
    for loop, (items, _) in M.grid_loops(name).items():
        per_problem = items // B
        first_b = -(-M.GRID_CAP // per_problem)
        assert B - first_b >= K, f"{name}: the {loop} loop's second pass holds fewer than K problems"
        assert set(idx[first_b:first_b + K].tolist()) == set(range(K))


def test_shapes_cover_every_instance():
    """Every compiled instance, a padded shape and one without an instance; the slew systems reach every instance
    with n > m as the augmented (n + m, m)."""
    assert set(INSTANCES) <= set(M.SHAPES)
    assert (6, 1) in M.SHAPES and (5, 2) in M.SHAPES and (20, 4) in M.SHAPES
    aug = {(n + m, m) for n, m in M.SLEW_SYSTEMS}
    assert {s for s in INSTANCES if s[0] > s[1]} <= aug


@pytest.mark.parametrize("group", list(SWITCH_PLANS))
def test_switch_cases_take_both_sides(group):
    """switch_cases puts runs just below and at T* under every dispatch of the pick, both with the model stepping and
    under a slew-rate window, and poisons one run at T*."""
    pick = (8, 2, 40, (None, 1, 2))
    cases = M.switch_cases(pick, list(SWITCH_PLANS).index(group))
    assert {(T, impl) for T, impl, _, _, _ in cases} == {(T, i) for T in (39, 40) for i in pick[3]}
    assert {slew for _, _, slew, _, _ in cases} == {False, True}
    assert [(T, impl) for T, impl, _, _, poison in cases if poison] == [(40, None)]


@pytest.mark.parametrize("form", list(M.FORMS))
def test_window_forms_stage_their_strides(form):
    """Each form's inputs as the device call hands them over (window_inputs, here on the CPU), and the time stride
    the staging records for each at an exact instance (step._time_strided, what _Pad.stage calls): dense 0, a
    stride-0 view over the axis -1 (not copied dense), a strided view its own stride of two slices."""
    mode, kw = M.FORMS[form]
    kw = dict(kw)
    if kw.get("F_T") == "T":
        kw["F_T"] = 6
    for dtype in (torch.float64, torch.float32):
        c = M.Case(4, 2, 6, 12, dtype, 3, mode, seed=1, **kw)
        ins, plant, _ = M.window_inputs(c, "cpu")
        B, N, P = c.B, 4, 6
        slice_ = dict(C=B * P * P, c=B * P, F=B * N * P, f=B * N)
        for k, t in zip(("C", "c", "F", "f"), ins[1:]):
            if t is None:
                continue
            want = -1 if k in c.P["time_invariant"] else 2 * slice_[k] if k in c.strided else 0
            assert S._time_strided(t, dtype)[1] == want, (form, k)
        if c.lin_plant:
            want = -1 if c.plant == "lin_ti" else 0
            assert S._time_strided(plant[1], dtype)[1] == want
            assert plant[1].shape[0] == (c.L if kw.get("Fp_T") == "L" else c.L - 1)
    if form == "strided":
        assert set(c.strided) == {"C", "c", "F", "f"}


def test_every_form_is_needed():
    assert set(M.FORMS) <= M.NEEDED_FORMS


# ------------------------------------------------------------------------------------------------------------------
# window_oracle(whole=...): an input handed whole to every step
# ------------------------------------------------------------------------------------------------------------------
def _const_case(seed, plant):
    """A (4, 2) episode of 3 steps at T = 5 whose model F, f (or LinDx plant) is constant along the axis."""
    from tests.helpers import gen_problem
    n, m, T, n_steps, B = 4, 2, 5, 3, 3
    L = n_steps + T - 1
    C, c, F, f, x0 = gen_problem(seed, B, L, n, m, F64, time_varying=True)
    F, f = 0.9 * F, f
    if plant:
        pl = ("lin", F[:1].expand(L - 1, *F.shape[1:]) * 1.03, f[:1].expand(L - 1, *f.shape[1:]) + 0.01)
    else:
        F, f = F[:1].expand(L - 1, *F.shape[1:]).contiguous(), f[:1].expand(L - 1, *f.shape[1:]).contiguous()
        pl = None
    g = torch.Generator().manual_seed(seed + 1)
    lo = -0.5 * torch.rand(L, B, m, generator=g, dtype=F64) - 0.05
    return n, m, T, n_steps, x0, C, c, F, f, pl, dict(u_lower=lo, u_upper=-lo)


@pytest.mark.parametrize("what", ["F", "plant"])
def test_whole_input_is_the_constant_window(what):
    """An input constant along the axis: handed whole (F [T-1] or the plant's one slice), the episode is bitwise the
    windowed one, and the sweep's gradients of that input are the windowed ones summed over the axis (each solve's
    and each step's part lands at offset 0 instead of k); every other gradient bitwise."""
    n, m, T, n_steps, x0, C, c, F, f, pl, kw = _const_case(7, what == "plant")
    w = 0.02 * torch.randn(n_steps, x0.shape[0], n, generator=torch.Generator().manual_seed(3), dtype=F64)
    opts = dict(lqr_iter=3, eps=0.0, not_improved_lim=10 ** 6, coupled=False)
    if what == "F":
        Fw, fw, plw = F[:T - 1].clone(), f[:T - 1].clone(), pl
    else:
        Fw, fw, plw = F, f, ("lin", pl[1][:1].clone(), pl[2][:1].clone())
    win = wo.receding_horizon_tv(n, m, T, n_steps, x0, C, c, F, f, plant=pl, w=w, **kw, **opts)
    whl = wo.receding_horizon_tv(n, m, T, n_steps, x0, C, c, Fw, fw, plant=plw, w=w, whole=(what,), **kw, **opts)
    for k in ("x", "u", "costs", "plan_x", "plan_u", "u_next"):
        assert torch.equal(getattr(win, k), getattr(whl, k)), k
    g = torch.Generator().manual_seed(5)
    wx = torch.randn(win.x.shape, generator=g, dtype=F64)
    wu = torch.randn(win.u.shape, generator=g, dtype=F64)
    bw = dict(u_lower=kw["u_lower"], u_upper=kw["u_upper"])
    gw = wo.receding_horizon_backward_tv(n, m, T, C, c, F, f, win.x, win.u, win.plan_x, win.plan_u, wx, wu, plant=pl,
                                         **bw)
    gh = wo.receding_horizon_backward_tv(n, m, T, C, c, Fw, fw, win.x, win.u, win.plan_x, win.plan_u, wx, wu,
                                         plant=plw, whole=(what,), **bw)
    summed = ("dF", "df") if what == "F" else ("dF_p", "df_p")
    for k, v in gw.items():
        if v is None:
            assert gh[k] is None, k
        elif k in summed:
            assert gh[k].shape[0] == (T - 1 if what == "F" else 1), k
            assert maxdiff(gh[k].sum(0), v.sum(0)) <= 1e-12 * max(1.0, float(v.abs().max())), k
        else:
            assert torch.equal(gh[k], v), k
