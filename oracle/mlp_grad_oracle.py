"""Float64 oracle of the gradient of a learned model's linearisation in its weights: the vector-Jacobian product of
mlp_oracle.linearize with respect to every layer's W and b, by autograd through that function (the reference's
NNDynamics.grad_input differentiated under create_graph, mpc/dynamics.py:81-131).

A network is mlp_oracle's list of (W [out, in], b [out]) float64 CPU tensors, an activation name and the passthrough
flag.  The result is the list of (dW, db) in the same order: the gradient of sum(dF * F) + sum(df * f).
"""
import torch

from . import mlp_oracle as mo


def linearize_vjp(layers, act, passthrough, x, u, dF, df, n_prev=0):
    """[(dW_i, db_i)] of <dF, F> + <df, f> for (F, f) = mlp_oracle.linearize(layers, act, passthrough, x, u, n_prev);
    dF [T-1, B, N, N+m], df [T-1, B, N] (N = n_prev + n).  The linearisation point (x, u) is a constant."""
    lg = [(W.detach().clone().requires_grad_(True), b.detach().clone().requires_grad_(True)) for W, b in layers]
    with torch.enable_grad():
        F, f = mo.linearize(lg, act, passthrough, x.detach(), u.detach(), n_prev)
        flat = [t for wb in lg for t in wb]
        g = torch.autograd.grad((F * dF).sum() + (f * df).sum(), flat, allow_unused=True)
    g = [torch.zeros_like(t) if gi is None else gi for gi, t in zip(g, flat)]
    return [(g[2 * i], g[2 * i + 1]) for i in range(len(layers))]
