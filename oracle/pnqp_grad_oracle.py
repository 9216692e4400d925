"""Float64 oracle of the implicit gradient of a pnqp solution (TEST INFRASTRUCTURE ONLY), the companion of
lqr_oracle.pnqp: torch on the CPU, the formula of mpcb200_pnqp_backward_* (include/mpcb200.h) written out directly.

Given the solution x and free set If that pnqp returned for (H, q, lower, upper) and g = dL/dx, with F the free set and
A the rest, v solves (H_FF + 1e-11 I) v = g_F (the regularised block pnqp's Newton systems factor, mpc/pnqp.py:46-48),
and
  dq = -v on F, 0 on A;   dH[i, :] = -v_i x^T for i in F, 0 on the rows of A;
  dlower_i / dupper_i = g_i - (H_FA^T v)_i for i in A, to the bound x_i sits on (lower when x_i == lower_i);
every other entry is 0.  This is the reference's unrolled autograd on a problem whose last accepted Newton step was a
full step with the final free set (oracle/make_golden_pnqp_grad.py pins it against the reference).
"""
import torch

from .lqr_oracle import PNQP_EPS_DIAG


def pnqp_grad(H, x, If, lower, upper, dl_dx):
    """(dH [B,n,n], dq, dlower, dupper [B,n]) in the dtype of H; lower and upper are [B,n], [n], [1,n] or floats."""
    B, n, _ = H.shape
    F = If.bool()
    zero = torch.zeros((), dtype=H.dtype)
    lower = torch.as_tensor(lower, dtype=H.dtype).expand(B, n)
    ff = F.unsqueeze(2) & F.unsqueeze(1)
    H_ = torch.where(ff, H, zero) + PNQP_EPS_DIAG * torch.eye(n, dtype=H.dtype)
    v = torch.linalg.solve(H_, torch.where(F, dl_dx, zero).unsqueeze(-1)).squeeze(-1)
    v = torch.where(F, v, zero)                           # exactly 0 off F, as the decoupled rows of H_ give
    dq = -v
    dH = torch.where(F.unsqueeze(2), -v.unsqueeze(2) * x.unsqueeze(1), zero)
    r = torch.where(F, zero, dl_dx - (H * v.unsqueeze(2)).sum(1))   # (H^T v)_i = sum_{k in F} H_ki v_k
    at_lower = ~F & (x == lower)
    return dH, dq, torch.where(at_lower, r, zero), torch.where(~F & ~at_lower, r, zero)


def settled(H, q, lower, upper, x, If, margin=1e-3):
    """[B] bool: the problems on which the formula is the derivative of pnqp itself.  Strictly complementary (every
    free coordinate at least `margin` inside its box; every clamped one on a bound, with |g_i| >= margin pushing
    outwards, g = Hx + q), and x_F the minimiser over the free set with x_A fixed to 1e-12 relative, which is what
    the last accepted Newton step gives when it was a full step with the final free set.  Such a problem keeps its
    free set under small perturbations, and its solution is a smooth function of (H, q, lower, upper) there."""
    B, n, _ = H.shape
    F = If.bool()
    lower = torch.as_tensor(lower, dtype=H.dtype).expand(B, n)
    upper = torch.as_tensor(upper, dtype=H.dtype).expand(B, n)
    g = (H @ x.unsqueeze(-1)).squeeze(-1) + q
    at_lo, at_hi = x == lower, x == upper
    free_ok = torch.where(F, torch.minimum(x - lower, upper - x) >= margin, True).all(1)
    clamped_ok = torch.where(F, True, (at_lo | at_hi) & (torch.where(at_lo, g, -g) >= margin)).all(1)
    # [H_FF 0; 0 I] [x_F; x_A] = [-(q_F + H_FA x_A); x_A]
    zero = torch.zeros((), dtype=H.dtype)
    xa = torch.where(F, zero, x)
    M = torch.where(F.unsqueeze(2) & F.unsqueeze(1), H, zero) + torch.diag_embed((~F).to(H.dtype))
    rhs = torch.where(F, -(q + (H @ xa.unsqueeze(-1)).squeeze(-1)), x)
    xs = torch.linalg.solve(M, rhs.unsqueeze(-1)).squeeze(-1)
    scale = xs.abs().amax(1).clamp(min=1.0)
    return free_ok & clamped_ok & ((xs - x).abs().amax(1) <= 1e-12 * scale)
