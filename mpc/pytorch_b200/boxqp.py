"""pnqp: batched projected-Newton box QP on the GPU (drop-in for reference mpc/pnqp.py:5).

Same signature and return tuple as the reference: ``(x, H_free, If, i)``.  ``H_free`` is the masked
matrix ``H_`` of the returning iteration (the reference returns its LU factorisation, or ``H_`` itself
for n == 1); ``If`` is a 0/1 tensor of H's dtype; ``i`` is the iteration count of the slowest problem
(the reference's batch-coupled loop returns when the slowest element converges).  Control flow is per
problem (what the reference computes for n_batch == 1).

QPs with n <= 8 run one per thread; larger ones run one per thread block, with the QP in shared memory, up to
``mpcb200_pnqp_max_n`` (at least 128 in float32 and float64 on an H100); larger n raises ``MpcB200Error``.
``H`` must be symmetric: the Newton systems are solved by an LDL^T factorisation of its lower triangle (the
reference uses an LU, which also accepts a non-symmetric ``H``).
"""

import torch

from . import _lib
from ._lib import MpcB200Error, _on_device, check, ptr, stream_handle


def pnqp(H, q, lower, upper, x_init=None, n_iter=20):
    fn = _lib.entry("mpcb200_pnqp", H.dtype)
    if H.dim() != 3 or H.shape[1] != H.shape[2]:
        raise MpcB200Error(f"H: expected [B,n,n], got {tuple(H.shape)}")
    B, n, _ = H.size()
    for nm, t_ in (("q", q), ("lower", lower), ("upper", upper), ("x_init", x_init)):
        if torch.is_tensor(t_):
            if t_.device != H.device:
                raise MpcB200Error(f"{nm}: expected a tensor on {H.device}, got {t_.device}")
            if tuple(t_.shape) not in ((B, n), (n,), (1, n)):
                raise MpcB200Error(f"{nm}: expected shape {(B, n)}, got {tuple(t_.shape)}")
    if not H.is_cuda:
        raise MpcB200Error("mpc.pytorch_b200 runs on CUDA tensors only (no CPU fallback)")
    dtype, dev = H.dtype, H.device
    with _on_device(dev):
        max_n = _lib.lib().mpcb200_pnqp_max_n(H.element_size())
    if n > max_n:
        raise MpcB200Error(f"pnqp solves QPs with n <= {max_n} in {dtype} on {dev} (got n = {n}): the QP of one "
                           "thread block must fit its shared memory")
    d = lambda t: t.detach().to(dtype).expand(B, n).contiguous() if torch.is_tensor(t) else \
        torch.full((B, n), float(t), dtype=dtype, device=dev)
    Hc, qc, lo, hi = H.detach().contiguous(), d(q), d(lower), d(upper)
    x0 = d(x_init) if x_init is not None else None
    x = torch.empty(B, n, dtype=dtype, device=dev)
    Hf = torch.empty(B, n, n, dtype=dtype, device=dev)
    If = torch.empty(B, n, dtype=torch.uint8, device=dev)
    iters = torch.empty(B, dtype=torch.int32, device=dev)
    status = torch.empty(B, dtype=torch.int32, device=dev)
    with _on_device(dev):
        rc = fn(B, n, ptr(Hc), ptr(qc), ptr(lo), ptr(hi), ptr(x0), int(n_iter), ptr(x), ptr(Hf), ptr(If),
                ptr(iters), ptr(status), stream_handle(dev))
    check(rc, "mpcb200_pnqp")
    if bool((status & 1).any()):
        print("[WARNING] pnqp warning: Did not converge")          # reference mpc/pnqp.py:81
    return x, Hf, If.to(dtype), int(iters.max())
