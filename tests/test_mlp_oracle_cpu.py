"""CPU: the cases of tests/test_mlp_oracle_gpu.py exercise what they claim, checked without a device against the
constants of csrc/mlp.cu and mlp.cuh (the 1024-CTA grid cap, 8 warps per CTA, the VJP's slot constants), the fit
formula and mpcb200_mlp_fits, at the H100's 227 KB of opt-in shared memory:

  * the grid-stride batches take a second pass at the warps per CTA each launch shape runs;
  * the edge network is the widest (n+m, h, h, n) that mpcb200_mlp_fits accepts, and one wider is refused;
  * the padded cases sit exactly at p_max, and one more staged element is MPCB200_ERR_BAD_DIMS;
  * the episode case deals its linearisation items to G > 1 VJP slots, with slots taking two items;
  * each line-search pool holds every pass class in the float64 oracle."""
import ctypes
import os
import re

import pytest
import torch

from mpc.pytorch_b200 import _lib
from tests import test_mlp_oracle_gpu as g
from tests.gpu_harness import MAX, MID, ONE
from tests.test_mlp_cpu import _smem

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "mpc", "pytorch_b200", "csrc")
H100_OPTIN = 227 * 1024


def _read(name):
    with open(os.path.join(SRC, name)) as fh:
        return fh.read()


def _const(name):
    m = re.search(rf"constexpr (?:long long|int) {name} = (\d+)(?:ll << (\d+))?;", _read("mlp.cuh"))
    return int(m.group(1)) << int(m.group(2) or 0)


def test_launch_constants_are_the_launchers():
    src = _read("mlp.cu")
    assert re.search(r"int w = (\d+);", src).group(1) == str(g.MAX_WARPS)                 # mlp_warps
    assert f"grid = (int)(g < {g.MAX_CTAS} ? g : {g.MAX_CTAS});" in src                   # mlp_prepare
    hdr = open(os.path.join(SRC, "..", "..", "..", "include", "mpcb200.h")).read()
    assert int(re.search(r"#define MPCB200_MLP_PAD_SLACK (\d+)", hdr).group(1)) == g.SLACK


@pytest.mark.parametrize("esz", [4, 8])
@pytest.mark.parametrize("n_prev", [0, 2])
def test_the_fit_formula_is_the_library_and_test_mlp_cpu_one(esz, n_prev):
    for widths in [(6, 32, 4), (6, 32, 12, 4), (6, 256, 64, 4), (35, 256, 33), (2, 1), (6, 230, 230, 4)]:
        assert g.smem_bytes(widths, esz, n_prev) == _smem(widths, esz, n_prev)
        if n_prev in (0, widths[0] - widths[-1]):                        # n_prev is 0 or the network's m
            assert g.fits(widths, esz, n_prev) == (g.smem_bytes(widths, esz, n_prev) <= H100_OPTIN)


@pytest.mark.parametrize("esz", [4, 8])
@pytest.mark.parametrize("n_prev", [0, 2])
def test_edge_network_is_the_widest_that_fits(esz, n_prev):
    n, m = g.EDGE_NM
    h = g.edge_hidden(esz, n_prev)
    assert g.fits(g.widths_of(n, m, (h, h)), esz, n_prev) and not g.fits(g.widths_of(n, m, (h + 1, h + 1)), esz, n_prev)
    assert g.launch_warps(g.widths_of(n, m, (h, h)), esz, n_prev, 1 << 30, H100_OPTIN) == 1
    hl = g.edge_hidden(esz, 0, (g.LS_N, g.LS_M))
    assert g.fits(g.widths_of(g.LS_N, g.LS_M, (hl, hl)), esz) and not g.fits(g.widths_of(g.LS_N, g.LS_M,
                                                                                          (hl + 1, hl + 1)), esz)


@pytest.mark.parametrize("esz", [4, 8])
def test_odd_shape_runs_an_odd_warp_count(esz):
    h = g.odd_hidden(esz, H100_OPTIN)
    assert g.launch_warps(g.widths_of(*g.EDGE_NM, (h, h)), esz, 0, 1 << 30, H100_OPTIN) in (3, 5, 7)


@pytest.mark.parametrize("esz", [4, 8])
@pytest.mark.parametrize("shape", g.SHAPES, ids=[s[0] for s in g.SHAPES])
def test_grid_stride_batches_take_a_second_pass(shape, esz):
    name, n, m, hidden, _, _, n_prev = shape
    if hidden is None:
        h = g.odd_hidden(esz, H100_OPTIN) if name == "odd" else g.edge_hidden(esz, n_prev)
        hidden = (h, h)
    W = g.launch_warps(g.widths_of(n, m, hidden), esz, n_prev, 1 << 30, H100_OPTIN)
    K, batches = g.grid_batches(W)
    big = batches[-1]
    assert big > g.MAX_CTAS * W and g.grid_passes(big, W) == 2
    assert (g.GRID_T - 1) * big > g.MAX_CTAS * W
    assert all(g.grid_passes(B, W) == 1 for B in batches[:-1])
    assert all(K % p for p in range(2, W + 1) if W % p == 0)             # K coprime to W
    # the line search's grid batches and the loop's full-size batch
    assert g.grid_passes(g.FULL_B, g.MAX_WARPS) == 2
    assert g.full_samples(g.FULL_B)[-1] == g.FULL_B - 1 and g.MAX_CTAS * g.MAX_WARPS in g.full_samples(g.FULL_B)


def _rec(widths, n_prev):
    return g.record_of(widths, n_prev=n_prev)


@pytest.mark.parametrize("shape", g.SHAPES, ids=[s[0] for s in g.SHAPES])
def test_padded_cases_sit_at_p_max(shape):
    """N + M = n_prev + width[0] + 16 is taken; one more element is MPCB200_ERR_BAD_DIMS before any device use."""
    name, n, m, hidden, _, _, n_prev = shape
    hidden = hidden or (12, 12)
    widths = g.widths_of(n, m, hidden)
    N, M = n_prev + n + g.PAD[0], m + g.PAD[1]
    assert N + M == g.p_max(widths, n_prev)
    L = _lib.lib()
    FAKE = 1 << 20
    r = _rec(widths, n_prev)
    # a NULL output passes the dimension check first: 1 (NULL) means the dims were accepted, 2 that they were not
    assert L.mpcb200_mlp_rollout_f32(ctypes.byref(r), 4, 3, N, M, FAKE, FAKE, None, None) == 1
    assert L.mpcb200_mlp_rollout_f32(ctypes.byref(r), 4, 3, N + 1, M, FAKE, FAKE, None, None) == 2
    assert L.mpcb200_mlp_rollout_f64(ctypes.byref(r), 4, 3, N, M + 1, FAKE, FAKE, None, None) == 2
    assert L.mpcb200_mlp_linearize_f64(ctypes.byref(r), 4, 3, N, M, FAKE, None, FAKE, FAKE, None) == 1
    assert L.mpcb200_mlp_linearize_f64(ctypes.byref(r), 4, 3, N, M + 1, FAKE, None, FAKE, FAKE, None) == 2


def test_staging_cases_take_each_copy_path():
    for (n, m, hidden), tail in zip(g.STAGING, ({4: 0, 8: 0}, {4: 12, 8: 8}, {4: 12, 8: 8})):
        nbytes = {e: g.n_params(g.widths_of(n, m, hidden)) * e for e in (4, 8)}
        assert {e: b % 16 for e, b in nbytes.items()} == tail
    assert g.n_params(g.widths_of(1, 1, ())) * 4 < 16                  # f32: no bulk copy at all


def test_episode_vjp_slots_take_two_items():
    items = (g.EP_T - 1) * g.EP_B
    nparams = g.n_params(g.widths_of(g.EP_N, g.EP_M, g.EP_HIDDEN))
    G = max(1, min(items, _const("kMlpVjpMaxSlots"), max(1, _const("kMlpVjpSlotElems") // nparams)))
    assert G == g._vjp_slots(items, nparams)
    assert 1 < G < items <= 2 * G                                      # every slot one or two items, some two
    assert g.EP_B > g.MAX_WARPS * 2                                    # the episode's kernels span several CTAs


def test_line_search_matrix_gives_each_dtype_every_option():
    values = dict(act=set(g.LS_ACTS), hidden=set(g.LS_HIDDEN), n_prev={0, g.LS_M}, mode=set(g.LS_MODES),
                  decay={0.5, 0.3}, max_ls={1, 3, 10})
    for dtype in (g.F64, g.F32):
        cases = [c for c in g.LS_CASES if c["dtype"] == dtype]
        for k, want in values.items():
            assert {c[k] for c in cases} == want, (dtype, k)


@pytest.mark.parametrize("case", g.LS_CASES, ids=[g.ls_case_id(c) for c in g.LS_CASES])
def test_line_search_pool_holds_every_pass_class(case):
    cls = g.ls_pool(*g._ls_args(case))[-1]
    need = {ONE, MAX} if case["max_ls"] == 1 else {ONE, MID, MAX}
    for c in need:
        assert int((cls == c).sum()) >= 2, (c, {k: int((cls == k).sum()) for k in (ONE, MID, MAX)})
    idx = g.ls_select(cls, g.ls_batch_layout(g.LS_B))
    assert set(cls[idx].tolist()) == need
    layout = g.ls_batch_layout(g.LS_B)
    # neighbouring warps, CTAs' first warps and grid-stride partners differ in pass class
    assert all(layout[b] != layout[b + 1] for b in range(g.LS_B - 2))
    big = g.ls_batch_layout(g.MAX_CTAS * g.MAX_WARPS + 9)
    assert all(big[b] != big[b + g.MAX_CTAS * g.MAX_WARPS] for b in range(8))


def test_grid_line_search_pools_hold_every_pass_class():
    for dt, hidden, K in ((g.F64, (12,), g.LS_POOL), (g.F32, (12,), g.LS_POOL)):
        cls = g.ls_pool(dt, "sigmoid", hidden, 0, "free", 0.5, 10, 480, K=K)[-1]
        assert {ONE, MID, MAX} <= set(cls.tolist())
    h = g.edge_hidden(8, 0, (g.LS_N, g.LS_M))
    cls = g.ls_pool(g.F64, "sigmoid", (h, h), 0, "free", 0.5, 10, 480, K=96)[-1]
    assert {ONE, MID, MAX} <= set(cls.tolist())
    assert torch.is_tensor(cls)
