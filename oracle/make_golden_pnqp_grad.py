#!/usr/bin/env python3
"""Gradient fixture of the standalone pnqp, from the REAL reference.

Run with a checkout of locuslab/mpc.pytorch:   MPC_REFERENCE=<checkout> python oracle/make_golden_pnqp_grad.py
Differentiates the unmodified reference's pnqp (mpc/pnqp.py:5-82) with autograd, one problem at a time (a batch of
one, the control flow every problem follows in the kernels), for the loss sum(w * x) with a random w.  Problems come
from the pnqp recipe of oracle/make_golden.py (H = LL' + I/2, q ~ 2N(0,1), bounds in (-1, 0) and (0, 1), x_init ~
0.3N(0,1)) and are kept only when they are
  * converged (the reference returns from inside its loop),
  * settled (oracle/pnqp_grad_oracle.settled): strictly complementary with a margin of 1e-3, and x_F the minimiser
    over the free set with x_A fixed, which is what the last accepted Newton step gives when it was a full step with
    the final free set.
On such problems the reference's unrolled gradient is the implicit one of oracle/pnqp_grad_oracle.py, up to the 1e-11
regularisation.  Before the file is written the oracle, at the reference's own x and free set, must match the
reference's dH, dq, dlower and dupper within 1e-10 of max|grad|.  Stores, for n in N_SIZES and a cold and a warm
start, H, q, lower, upper, x_init (warm), w, x, If and the reference's dH, dq, dlower, dupper under the prefix
n<n>_<cold|warm>_ in tests/golden/boxqp_grad_f64.npz.  Only numbers are stored.
"""
import contextlib
import io
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from make_golden import GOLD, load_reference   # noqa: E402
from oracle.pnqp_grad_oracle import pnqp_grad, settled   # noqa: E402

F64 = torch.float64
B, N_ITER = 4, 20
N_SIZES = (1, 2, 5, 8, 12, 40)
FIELDS = ("H", "q", "lower", "upper", "x_init", "w", "x", "If", "dH", "dq", "dlower", "dupper")


def candidate(g, n, warm):
    L = torch.randn(1, n, n, generator=g, dtype=F64)
    H = L @ L.transpose(1, 2) + 0.5 * torch.eye(n, dtype=F64)
    q = 2.0 * torch.randn(1, n, generator=g, dtype=F64)
    lo = -torch.rand(1, n, generator=g, dtype=F64)
    hi = torch.rand(1, n, generator=g, dtype=F64)
    x0 = 0.3 * torch.randn(1, n, generator=g, dtype=F64) if warm else None
    w = torch.randn(1, n, generator=g, dtype=F64)
    return H, q, lo, hi, x0, w


def reference_grad(rpnqp, H, q, lo, hi, x0, w):
    leaves = [t.clone().requires_grad_(True) for t in (H, q, lo, hi)]
    out = io.StringIO()
    with contextlib.redirect_stdout(out):
        x, _, If, it = rpnqp.pnqp(*leaves, x_init=x0, n_iter=N_ITER)
    converged = "Did not converge" not in out.getvalue()
    grads = torch.autograd.grad((w * x).sum(), leaves, allow_unused=True)
    grads = [torch.zeros_like(t) if d is None else d for d, t in zip(grads, leaves)]
    return x.detach(), If.to(F64), converged, grads


def main():
    _, _, rpnqp, _ = load_reference()
    arrays = {}
    for n in N_SIZES:
        for warm in (False, True):
            tag = f"n{n}_{'warm' if warm else 'cold'}"
            g = torch.Generator().manual_seed(9000 + 10 * n + warm)
            rows, tried = [], 0
            while len(rows) < B:
                tried += 1
                H, q, lo, hi, x0, w = candidate(g, n, warm)
                x, If, converged, grads = reference_grad(rpnqp, H, q, lo, hi, x0, w)
                if converged and bool(settled(H, q, lo, hi, x, If)):
                    rows.append((H, q, lo, hi, x0, w, x, If, *grads))
            cols = [torch.cat(c) if c[0] is not None else None for c in zip(*rows)]
            got = dict(zip(FIELDS, cols))
            want = pnqp_grad(got["H"], got["x"], got["If"], got["lower"], got["upper"], got["w"])
            scale = max(float(t.abs().max()) for t in want)
            for k, o in zip(("dH", "dq", "dlower", "dupper"), want):
                err = float((o - got[k]).abs().max())
                assert err <= 1e-10 * scale, f"oracle != reference for {tag}.{k}: {err:.3g} (max|grad| {scale:.3g})"
            F = got["If"].bool()
            at_lo = ~F & (got["x"] == got["lower"])
            print(f"  {tag}: {tried} candidates for {B}; free {int(F.sum())}, at lower {int(at_lo.sum())}, "
                  f"at upper {int((~F & ~at_lo).sum())}")
            arrays.update({f"{tag}_{k}": v.numpy() for k, v in got.items() if v is not None})
    np.savez_compressed(os.path.join(GOLD, "boxqp_grad_f64.npz"), **arrays)
    print("wrote boxqp_grad_f64", len(arrays), "arrays")


if __name__ == "__main__":
    main()
