"""CPU: the implicit-gradient oracle of the standalone pnqp (oracle/pnqp_grad_oracle.py) against the reference's
unrolled autograd (fixture boxqp_grad_f64, oracle/make_golden_pnqp_grad.py), and the argument checks of
mpcb200_pnqp_backward_*, which answer before any device is needed."""
import ctypes

import numpy as np
import pytest
import torch

from oracle.pnqp_grad_oracle import pnqp_grad
from tests.helpers import GOLD

CASES = [f"n{n}_{s}" for n in (1, 2, 5, 8, 12, 40) for s in ("cold", "warm")]


def fixture(tag):
    z = np.load(f"{GOLD}/boxqp_grad_f64.npz")
    return {k[len(tag) + 1:]: torch.from_numpy(z[k]) for k in z.files if k.startswith(tag + "_")}


@pytest.mark.parametrize("tag", CASES)
def test_oracle_matches_reference_autograd(tag):
    g = fixture(tag)
    assert ("x_init" in g) == tag.endswith("warm")
    want = pnqp_grad(g["H"], g["x"], g["If"], g["lower"], g["upper"], g["w"])
    scale = max(float(t.abs().max()) for t in want)
    for k, o in zip(("dH", "dq", "dlower", "dupper"), want):
        err = float((o - g[k]).abs().max())
        assert err <= 1e-10 * scale, f"{tag}.{k}: {err:.3g} (max|grad| {scale:.3g})"


def test_fixture_mixes_free_and_both_bounds():
    free = lower = upper = 0
    for tag in CASES:
        g = fixture(tag)
        F = g["If"].bool()
        at_lo = ~F & (g["x"] == g["lower"])
        free, lower, upper = free + int(F.sum()), lower + int(at_lo.sum()), upper + int((~F & ~at_lo).sum())
    assert min(free, lower, upper) > 0, (free, lower, upper)


def test_backward_symbols_exported():
    from mpc.pytorch_b200 import _lib
    for name in ("mpcb200_pnqp_backward_f32", "mpcb200_pnqp_backward_f64"):
        assert name in _lib.EXPORTED_SYMBOLS
        assert getattr(_lib.lib(), name).restype is ctypes.c_int


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
def test_malformed_calls_are_refused(dtype):
    """BAD_DIMS (2) for B or n <= 0, NULL_POINTER (1) for a missing required pointer, SMEM (4) for n above
    mpcb200_pnqp_max_n: every check runs before the library looks for a device, so non-null dummies are safe."""
    from mpc.pytorch_b200 import _lib
    fn = _lib.entry("mpcb200_pnqp_backward", dtype)
    max_n = _lib.lib().mpcb200_pnqp_max_n(torch.empty(0, dtype=dtype).element_size())
    dummy = ctypes.c_void_p(256)
    args = lambda nulls=(): [None if k in nulls else dummy for k in range(11)]  # noqa: E731  H..status
    assert fn(0, 4, *args(), None) == 2
    assert fn(-1, 4, *args(), None) == 2
    assert fn(3, 0, *args(), None) == 2
    for k in range(10):                                    # status (k = 10) is optional
        assert fn(3, 4, *args((k,)), None) == 1, f"null argument {k}"
    assert fn(3, max_n + 1, *args(), None) == 4
    assert fn(3, max_n + 1, *args((10,)), None) == 4
