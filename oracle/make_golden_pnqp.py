#!/usr/bin/env python3
"""Per-problem pnqp fixtures for small QPs (n <= 8, the one-thread-per-QP kernel of csrc/pnqp.cu), from the REAL
reference.

Run with a checkout of locuslab/mpc.pytorch:   MPC_REFERENCE=<checkout> python oracle/make_golden_pnqp.py
Calls the unmodified reference's pnqp (mpc/pnqp.py:5-82) one problem at a time (a batch of one), which is the control
flow every problem follows in the kernels, and stacks the results.  Inputs come from the pnqp recipe of
oracle/make_golden.py (H = LL' + I/2, q ~ 2N(0,1), bounds in (-1, 0) and (0, 1), x_init ~ 0.3N(0,1)) with seeds of
their own.  Before a file is written, oracle/lqr_oracle.py's pnqp(coupled=False) must reproduce the reference: x to
1e-12 (float64) or 1e-6 (float32), the free sets and every problem's iteration count exactly.  Stores H, q, lower,
upper, x_init (warm cases), x, If and iters [B] as tests/golden/pnqp1_<dtype>_n<n>_<cold|warm>.npz (the ``pnqp1_``
prefix keeps them apart from the batch-coupled ``pnqp_`` fixtures).  Only numbers are stored.
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
from make_golden import close, load_reference, npz   # noqa: E402
import lqr_oracle as orc                            # noqa: E402

F64, F32 = torch.float64, torch.float32
B, N_ITER = 16, 20
# (dtype, n, warm, seed)
CASES = [(F64, 2, False, 8102), (F64, 3, False, 8103), (F64, 6, False, 8106), (F64, 7, False, 8107),
         (F64, 8, False, 8108), (F64, 6, True, 8206), (F64, 8, True, 8208), (F32, 8, False, 8308)]


def gen_qp(seed, n, dtype, warm):
    g = torch.Generator().manual_seed(seed)
    L = torch.randn(B, n, n, generator=g, dtype=F64)
    H = (L @ L.transpose(1, 2) + 0.5 * torch.eye(n, dtype=F64)).to(dtype)
    q = (2.0 * torch.randn(B, n, generator=g, dtype=F64)).to(dtype)
    lo = (-torch.rand(B, n, generator=g, dtype=F64)).to(dtype)
    hi = torch.rand(B, n, generator=g, dtype=F64).to(dtype)
    x0 = (0.3 * torch.randn(B, n, generator=g, dtype=F64)).to(dtype) if warm else None
    return H, q, lo, hi, x0


def main():
    _, _, rpnqp, _ = load_reference()
    for dtype, n, warm, seed in CASES:
        name = f"pnqp1_{'f64' if dtype == F64 else 'f32'}_n{n}_{'warm' if warm else 'cold'}"
        H, q, lo, hi, x0 = gen_qp(seed, n, dtype, warm)
        xs, Ifs, its = [], [], []
        for b in range(B):
            s = slice(b, b + 1)
            with contextlib.redirect_stdout(io.StringIO()):
                x, _, If, it = rpnqp.pnqp(H[s], q[s], lo[s], hi[s], x_init=x0[s] if warm else None, n_iter=N_ITER)
            xs.append(x)
            Ifs.append(If.to(dtype))
            its.append(int(it))
        x, If, iters = torch.cat(xs), torch.cat(Ifs), torch.tensor(its, dtype=torch.int64)
        xo, _, Ifo, ito = orc.pnqp(H, q, lo, hi, x_init=x0, n_iter=N_ITER, coupled=False)
        close(xo, x, 1e-12 if dtype == F64 else 1e-6, name + ".x")
        assert torch.equal(Ifo.bool(), If.bool()), name + ".If"
        assert torch.equal(ito, iters), (name, ito.tolist(), iters.tolist())
        free = float(If.mean())
        print(f"  {name}: free fraction {free:.2f}, iterations {iters.tolist()}")
        npz(name, H=H, q=q, lower=lo, upper=hi, x_init=x0, x=x, If=If, iters=iters)


if __name__ == "__main__":
    main()
