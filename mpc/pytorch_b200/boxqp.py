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

Gradients: when grad mode is on and one of ``H``, ``q``, ``lower``, ``upper`` is a tensor that requires grad, ``x``
carries the implicit gradient of the solution (``mpcb200_pnqp_backward_*``, include/mpcb200.h), first order only.
With F the returned free set and v = (H_FF + 1e-11 I)^{-1} dL/dx_F: dq = -v on F; row i of dH is -v_i x^T for i in F
(unsymmetrised, as autograd of the reference's g = Hx + q: a caller who builds a symmetric H from other tensors gets
the full derivative through that graph); a clamped coordinate passes dL/dx_i - (H_FA^T v)_i to the bound it sits on.
This is the reference's unrolled autograd when the last accepted Newton step was a full step with the final free set
(a converged, strictly complementary problem); on a problem that stopped at the iteration cap it is the same formula
at the returned point, not the derivative of the iterations.  ``x_init``, ``H_free``, ``If`` and ``i`` carry no
gradient.  Otherwise pnqp runs without autograd bookkeeping and ``x`` has no ``grad_fn``.
"""

import torch

from . import _lib
from ._lib import MpcB200Error, _on_device, check, ptr, stream_handle


def _batch(t, B, n, dtype, dev):
    """A [B, n], [n] or [1, n] tensor, or a float, as a dense [B, n] tensor of the QP's dtype."""
    if torch.is_tensor(t):
        return t.detach().to(dtype).expand(B, n).contiguous()
    return torch.full((B, n), float(t), dtype=dtype, device=dev)


def _solve(H, q, lower, upper, x_init, n_iter):
    """One mpcb200_pnqp_* call: (x, H_free, If as uint8, iters as int32 [B])."""
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
    Hc, qc, lo, hi = H.detach().contiguous(), *(_batch(t, B, n, dtype, dev) for t in (q, lower, upper))
    x0 = _batch(x_init, B, n, dtype, dev) if x_init is not None else None
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
    return x, Hf, If, iters


class _PnqpFn(torch.autograd.Function):
    """pnqp with the implicit gradient of x: one mpcb200_pnqp_backward_* call."""

    @staticmethod
    def forward(ctx, H, q, lower, upper, x_init, n_iter):
        x, Hf, If, iters = _solve(H, q, lower, upper, x_init, n_iter)
        # the inputs the backward reads, so that an in-place edit of one of them before backward raises
        ctx.save_for_backward(H, x, If, *(t if torch.is_tensor(t) else None for t in (lower, upper)))
        ctx.float_bounds = tuple(None if torch.is_tensor(t) else t for t in (lower, upper))
        ctx.q_shape = q.shape if torch.is_tensor(q) else None
        Ifd = If.to(H.dtype)
        ctx.mark_non_differentiable(Hf, Ifd, iters)
        return x, Hf, Ifd, iters

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, dl_dx, *_):
        H, x, If, lower, upper = ctx.saved_tensors
        B, n, _ = H.shape
        dtype, dev = H.dtype, H.device
        lo, hi = (_batch(t if t is not None else f, B, n, dtype, dev)
                  for t, f in zip((lower, upper), ctx.float_bounds))
        Hc = H.detach().contiguous()
        dH = torch.empty_like(Hc)
        dq, dlo, dhi = (torch.empty(B, n, dtype=dtype, device=dev) for _ in range(3))
        status = torch.empty(B, dtype=torch.int32, device=dev)
        with _on_device(dev):
            rc = _lib.entry("mpcb200_pnqp_backward", dtype)(
                B, n, ptr(Hc), ptr(x), ptr(If), ptr(lo), ptr(hi), ptr(dl_dx.contiguous()), ptr(dH),
                ptr(dq), ptr(dlo), ptr(dhi), ptr(status), stream_handle(dev))
        check(rc, "mpcb200_pnqp_backward")
        if bool((status & 4).any()):
            print("[WARNING] pnqp warning: bad pivot in the free block of the backward")
        need = ctx.needs_input_grad
        to_input = lambda g, shape, k: g.sum_to_size(shape) if need[k] and shape is not None else None  # noqa: E731
        return (dH if need[0] else None, to_input(dq, ctx.q_shape, 1),
                to_input(dlo, lower.shape if lower is not None else None, 2),
                to_input(dhi, upper.shape if upper is not None else None, 3), None, None)


def pnqp(H, q, lower, upper, x_init=None, n_iter=20):
    if torch.is_grad_enabled() and any(torch.is_tensor(t) and t.requires_grad for t in (H, q, lower, upper)):
        x, Hf, If, iters = _PnqpFn.apply(H, q, lower, upper, x_init, n_iter)
        return x, Hf, If, int(iters.max())
    x, Hf, If, iters = _solve(H, q, lower, upper, x_init, n_iter)
    return x, Hf, If.to(H.dtype), int(iters.max())
