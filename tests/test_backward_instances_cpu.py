"""The case builders of tests/test_backward_instances_gpu.py do what they claim, without a device: the batch lists put
problems at every warp and CTA position of each kernel's layout, the misaligned views reach the kernels unchanged,
the strided views keep their time strides, and each misalignment case leaves exactly one tensor failing the
16-byte test the library applies (restated here from api.cu)."""
import math

import pytest
import torch

from tests.gpu_harness import (DT, F32, F64, INSTANCES, PAIR_SHAPES, grad_layout, layout_batches, linear_step_case,
                               misaligned, pool_size, rollout_layout, step_layout)
from tests.test_backward_instances_gpu import (LARGE_MISALIGN, LARGE_TENSORS, STEP_TENSORS, misaligned_step_inputs,
                                               step_misalign_B)

LB = ("C", "F", "c", "f", "x", "u", "BOX")        # the large-shape kernel's per-tensor bulk bits (lqr_large.cu)


def _layouts(n, m):
    """(kernel, ppw, W, K | None) of every layout the GPU module derives batch sizes from at (n, m)."""
    out = [("grad", *grad_layout(n, m), pool_size(*grad_layout(n, m))), ("rollout", *rollout_layout(n), None)]
    if (n, m) in PAIR_SHAPES:
        pair = step_layout("pair", n, m, F64)
        out.append(("pair", *pair, pool_size(*pair, *grad_layout(n, m))))
    return out


@pytest.mark.parametrize("n,m", INSTANCES, ids=[f"n{n}m{m}" for n, m in INSTANCES])
def test_batch_lists_reach_every_position(n, m):
    """Every position of a CTA holds a problem in a full CTA and, but for the last one, in a partial tail CTA; every
    position of a warp but the last in a partial warp; with a pool, every pool problem sits at every position of a
    full CTA, and problems one warp or one CTA apart differ."""
    for kernel, ppw, W, K in _layouts(n, m):
        tag = f"n{n}m{m} {kernel}"
        full, tail, part_warp, pool_pos = set(), set(), set(), set()
        for B in layout_batches(ppw, W, K):
            for b in range(B):
                q = b % W
                (full if b < B - B % W else tail).add(q)
                if b >= B - B % ppw:
                    part_warp.add(b % ppw)
                if K is not None and b < B - B % W:
                    pool_pos.add((b % K, q))
        assert full == set(range(W)), f"{tag}: full CTAs miss {set(range(W)) - full}"
        assert tail >= set(range(W - 1)), f"{tag}: tail CTAs miss {set(range(W - 1)) - tail}"
        assert part_warp >= set(range(ppw - 1)), f"{tag}: partial warps miss {set(range(ppw - 1)) - part_warp}"
        if K is not None:
            assert K >= 3 and math.gcd(K, W) == 1, f"{tag}: pool of {K}"
            assert pool_pos == {(k, q) for k in range(K) for q in range(W)}, f"{tag}: pool positions"


@pytest.mark.parametrize("dtype", [F32, F64], ids=["f32", "f64"])
def test_misaligned_views_reach_the_kernels_unchanged(dtype):
    from mpc.pytorch_b200.step import _dense, _time_strided
    t = torch.randn(5, 8, 6, dtype=torch.float64).to(dtype)
    v = misaligned(t)
    assert v.is_contiguous() and v.data_ptr() % 16 != 0 and torch.equal(v, t)
    staged, code = _time_strided(v, dtype)
    assert code == 0 and staged.data_ptr() == v.data_ptr()
    assert _dense(v, dtype).data_ptr() == v.data_ptr()


@pytest.mark.parametrize("dtype", [F32, F64], ids=["f32", "f64"])
def test_strided_views_keep_their_time_strides(dtype):
    """The (c) cases: stride-0 C and F map to the time-invariant code, c with a 2x time stride to that stride."""
    from mpc.pytorch_b200.step import _time_strided
    T, B, n, m = 5, 12, 4, 2
    p = n + m
    C = torch.randn(T, B, p, p, dtype=dtype)
    F = torch.randn(T - 1, B, n, p, dtype=dtype)
    c2 = torch.zeros(2 * T, B, p, dtype=dtype)
    assert _time_strided(C[:1].expand(T, B, p, p), dtype)[1] == -1
    assert _time_strided(F[:1].expand(T - 1, B, n, p), dtype)[1] == -1
    staged, code = _time_strided(c2[::2], dtype)
    assert code == 2 * B * p and staged.data_ptr() == c2.data_ptr()
    # so the GPU module expands after moving to the device and casting: a copy of an expanded tensor (to another
    # device or dtype) is dense and would reach the kernels with the dense time stride
    other = F64 if dtype == F32 else F32
    assert _time_strided(F[:1].expand(T - 1, B, n, p).to(other), other)[1] == 0
    assert _time_strided(F.to(other)[:1].expand(T - 1, B, n, p), other)[1] == -1


def _al16(t):
    return t is None or t.data_ptr() % 16 == 0


def _span16(elems, dtype):
    return elems * dtype.itemsize % 16 == 0


def _tile_aligned(n, m, B, D, kw, dtype):
    """api.cu step_impl: per tensor, base and time stride 16-byte aligned (the instance kernels' bulk_ok needs all,
    and x_init's base)."""
    p = n + m
    lo, hi = kw.get("u_lower"), kw.get("u_upper")
    return dict(C=_al16(D["C"]) and _span16(B * p * p, dtype), c=_al16(D["c"]) and _span16(B * p, dtype),
                F=_al16(D["F"]) and _span16(B * n * p, dtype), f=_al16(D["f"]) and _span16(B * n, dtype),
                cur_x=_al16(D["x"]) and _span16(B * n, dtype), cur_u=_al16(D["u"]) and _span16(B * m, dtype),
                x_init=_al16(D["x0"]),
                u_lower=_al16(lo) and _al16(hi) and _span16(B * m, dtype))


def _large_bits(n, m, al, dtype):
    """api.cu step_impl, large-shape branch: the tensors the large kernel copies in bulk (per-problem spans too)."""
    p = n + m
    bits = dict(C=al["C"] and _span16(p * p, dtype), F=al["F"] and _span16(n * p, dtype),
                c=al["c"] and _span16(p, dtype), f=al["f"] and _span16(n, dtype), x=al["cur_x"] and _span16(n, dtype),
                u=al["cur_u"] and _span16(m, dtype), BOX=al["u_lower"] and _span16(m, dtype))
    return {k for k in LB if bits[k]}


def _on_cpu(P, kw, dtype):
    return {k: v.to(dtype) if torch.is_tensor(v) else v for k, v in P.items()}, \
        {k: v.to(dtype) for k, v in kw.items()}


STEP_PARAMS = [(n, m, d) for n, m in INSTANCES for d in (F64, F32)]


@pytest.mark.parametrize("n,m,dtype", STEP_PARAMS, ids=[f"n{n}m{m}_{DT[d]}" for n, m, d in STEP_PARAMS])
def test_step_misalignment_fails_one_tensor(n, m, dtype):
    """At the batch size of the instance sweep every tensor of the aligned case passes the 16-byte test, and each
    case fails it for its one misaligned tensor only."""
    T, B = 4, step_misalign_B(n, m, dtype)
    assert B % 4 == 0
    P, kw = linear_step_case(1900 + 10 * n + m, B, T, n, m, dtype, "boxT")[:2]
    D, kw = _on_cpu(P, kw, dtype)
    assert all(_tile_aligned(n, m, B, D, kw, dtype).values())
    for which in STEP_TENSORS:
        al = _tile_aligned(n, m, B, *misaligned_step_inputs(D, kw, which), dtype)
        assert {k for k, ok in al.items() if not ok} == {which}, which


@pytest.mark.parametrize("n,m,dtype", LARGE_MISALIGN, ids=[f"n{n}m{m}_{DT[d]}" for n, m, d in LARGE_MISALIGN])
def test_large_misalignment_flips_one_bulk_bit(n, m, dtype):
    T, B = 4, 5
    P, kw = linear_step_case(2000 + n + m, B, T, n, m, dtype, "boxT")[:2]
    D, kw = _on_cpu(P, kw, dtype)
    assert _large_bits(n, m, _tile_aligned(n, m, B, D, kw, dtype), dtype) == set(LB)
    expect = dict(C="C", c="c", F="F", f="f", cur_x="x", cur_u="u", u_lower="BOX")
    for which in LARGE_TENSORS:
        bits = _large_bits(n, m, _tile_aligned(n, m, B, *misaligned_step_inputs(D, kw, which), dtype), dtype)
        assert set(LB) - bits == {expect[which]}, which
