"""CPU: the case builders of tests/test_receding_plant_oracle_gpu.py reach what they are meant to reach, without a
device.  The item counts and the grid cap are restated from the launchers:
  * episode_grad.cu epgrad_grid / ilqr.cu ilqr_grid: ceil(items / 256) blocks of 256 threads, at most 4096, so a
    grid-stride loop takes a second pass once its range exceeds 4096 x 256 = 1 048 576 items of a capped grid;
  * the init and accumulate kernels size their grid by T B P^2 (epgrad_items) and loop over B N (g, dw), B N P (a
    LinDx plant's dF) and B NP (a known plant's dtheta); the stage kernel sizes it by T B max(N, M) and a known
    system's stage loops over the B problems, one thread each;
  * api.cu epgrad_layout: the workspace slot of the stage's parameter part holds up256(B NP_step sz) bytes, NP_step
    the plant's parameter count, and dxk follows it."""
import math

import pytest
import torch

from tests.gpu_harness import INSTANCES
from tests import test_receding_plant_oracle_gpu as M

CAP = 4096 * 256


def up256(v):
    return (v + 255) // 256 * 256


def test_grid_cap_restated():
    assert M.GRID_CAP == CAP == 1 << 20


@pytest.mark.parametrize("name", list(M.GRID))
def test_grid_cases_take_two_passes(name):
    """Every loop a grid case targets runs on a capped grid and exceeds one pass; the detach case's N does not
    divide 2^20, so a mask taken from the first pass's index would land on other columns in the second."""
    g = M.GRID[name]
    N, loops = M.grid_loops(name)
    want = {"slew_detach": {"g"}, "plant_lin_w": {"g", "dw", "plant dF"},
            "plant_pendulum": {"g", "dw", "plant dtheta", "stage"}}[name]
    assert want <= set(loops)
    for loop in want:
        items, capped = loops[loop]
        assert capped, f"{name}: the grid of the {loop} loop is not capped"
        assert items > CAP, f"{name}: the {loop} loop has {items} items, one pass"
    if g["slew"]:
        assert CAP % N != 0, f"{name}: N = {N} divides 2^20"
    P = N + g["m"]
    assert g["T"] * g["B"] * P * P > 4096 * 256     # epgrad_items: the init / accumulate grid is the cap


def test_slew_shapes_cover_every_augmented_instance():
    """The slew systems (n, m) reach every compiled (N, M) with N > M as (n + m, m), a padded shape (n_prev < M) and
    one without an instance."""
    aug = {(n + m, m) for n, m in M.SLEW_SYSTEMS}
    assert {s for s in INSTANCES if s[0] > s[1]} <= aug
    assert (6, 1) in aug and (6, 1) not in INSTANCES and (6, 2) in INSTANCES
    assert any(s not in INSTANCES and s != (6, 1) for s in aug)
    assert set(INSTANCES) <= set(M.PLANT_SHAPES)


def test_known_on_known_overflows_a_model_sized_theta_slot():
    """Pendulum (NP 3) on the five-parameter pendulum (NP 5), float64: a slot sized by the model's NP still holds the
    plant's part at B = 6 (the plant tests' batch) and no longer from B = 7, the batch this module runs."""
    sz, np_model, np_plant = 8, M.KNOWN_NP["pendulum"], M.KNOWN_NP["pendulum_full"]
    assert up256(6 * np_model * sz) >= 6 * np_plant * sz
    pair_batches = {B for a, b, B in M.KNOWN_PAIRS if (a, b) == ("pendulum", "pendulum_full")}
    assert {1, 7, 300} <= pair_batches
    for B in (7, 300):
        assert up256(B * np_model * sz) < B * np_plant * sz


@pytest.mark.parametrize("name", list(M.GRID))
def test_pool_layout_reaches_every_position(name):
    """Element b is pool problem b mod K, K coprime to the 256-thread block and to N: every pool problem sits at every
    thread position of a block, and every pool problem has copies in the second pass of every targeted loop."""
    K, idx = M.grid_pool(name)
    g = M.GRID[name]
    N, loops = M.grid_loops(name)
    assert math.gcd(K, 256) == 1 and math.gcd(K, N) == 1 and K >= 3
    B = g["B"]
    assert B >= K * 256
    pairs = {(int(b) % K, int(b) % 256) for b in range(K * 256)}
    assert len(pairs) == K * 256
    assert bool((idx[:K] == torch.arange(K)).all())
    for loop, (items, _) in loops.items():
        per_problem = items // B
        first_b = -(-CAP // per_problem)          # first problem with an item in the second pass
        assert B - first_b >= K, f"{name}: the {loop} loop's second pass holds fewer than K problems"
        assert set(idx[first_b:first_b + K].tolist()) == set(range(K))
