#!/usr/bin/env python3
"""Fixtures for a slew-rate penalty on the known systems, from the REAL reference.

Run with a checkout of locuslab/mpc.pytorch:   MPC_REFERENCE=<checkout> python oracle/make_golden_slew.py
Solves MPC(n, 1, T, slew_rate_penalty=..., prev_ctrl=...) of the unmodified reference (mpc/mpc.py:362-445, its
CtrlPassthroughDynamics, mpc/dynamics.py:133-156) with its own CartpoleDx and PendulumDx (mpc/env_dx/) at the
non-default physics of oracle/make_golden_nn.py (KNOWN_SYSTEMS), float64, AUTO_DIFF, box bounds.  Two bound regimes:
inside the system's control clamp, and twice as wide, so that the controls the passthrough copies into the next
state go beyond the clamp the dynamics apply.  prev_ctrl [B, 1] holds values at, inside and beyond the clamp.  Stores
the inputs, x, u, costs and d u* / d c (the reference's own autograd through the solve) as
tests/golden/known_slew_{cartpole,pendulum}_f64.npz.  Only numbers are stored.
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
from make_golden import load_reference, npz                    # noqa: E402
from make_golden_nn import KNOWN_SYSTEMS, _known_states, load_ref_env    # noqa: E402

PENALTY = 0.5
B, T, LQR_ITER = 6, 10, 12


def main():
    rmpc, _, _, _ = load_reference()
    torch.set_default_dtype(torch.float64)
    for name, spec in KNOWN_SYSTEMS.items():
        renv = load_ref_env(name)
        dx = (renv.CartpoleDx if name == "cartpole" else renv.PendulumDx)(params=torch.tensor(spec["params"]))
        dx.dt = spec["dt"]
        setattr(dx, spec["clamp"][0], spec["clamp"][1])
        clamp = spec["clamp"][1]
        n = dx.n_state
        g = torch.Generator().manual_seed(41 if name == "cartpole" else 42)
        x0 = _known_states(name, B, g)
        prev = torch.tensor((clamp, -clamp, np.nextafter(clamp, np.inf), -1.7 * clamp, 0.4 * clamp, 0.0))[:B]
        prev = prev.view(B, 1)
        q, p = dx.get_true_obj()
        Q = torch.diag(q.double()).repeat(T, B, 1, 1)
        pp = p.double().repeat(T, B, 1)
        pp[..., n:] = 0.3 * clamp * (torch.rand(T, B, 1, generator=g) - 0.5)     # some push on the controls
        out = dict(params=torch.tensor(spec["params"]), dt=np.float64(spec["dt"]), clamp=np.float64(clamp),
                   decay=np.float64(spec["decay"]), ls_iter=np.int64(spec["ls_iter"]), penalty=np.float64(PENALTY),
                   lqr_iter=np.int64(LQR_ITER), x_init=x0, prev_ctrl=prev, C=Q, c=pp)
        for tag, bound in (("in", 0.8 * clamp), ("wide", 2.0 * clamp)):
            c = pp.clone().requires_grad_(True)
            with contextlib.redirect_stdout(io.StringIO()):
                x, u, costs = rmpc.MPC(n, 1, T, u_lower=-bound, u_upper=bound, lqr_iter=LQR_ITER, verbose=-1,
                                       exit_unconverged=False, detach_unconverged=False,
                                       linesearch_decay=spec["decay"], max_linesearch_iter=spec["ls_iter"],
                                       grad_method=rmpc.GradMethods.AUTO_DIFF, eps=1e-9, slew_rate_penalty=PENALTY,
                                       prev_ctrl=prev)(x0, rmpc.QuadCost(Q, c), dx)
            uf = u.reshape(-1)
            rows = [torch.autograd.grad(uf[i], c, retain_graph=True)[0].reshape(-1) for i in range(uf.numel())]
            on = u.abs() == bound
            beyond = u.abs() > clamp
            print(f"{name} bounds {tag}: on the bounds {int(on.sum())} of {u.numel()}, beyond the clamp "
                  f"{int(beyond.sum())}, mean cost {float(costs.mean()):.4e}, max|du/dc| "
                  f"{float(torch.stack(rows).abs().max()):.3e}")
            if tag == "wide":
                assert bool(beyond.any()), "the copied controls must go beyond the system's clamp"
            out.update({f"bound_{tag}": np.float64(bound), f"x_{tag}": x, f"u_{tag}": u, f"costs_{tag}": costs,
                        f"du_dc_{tag}": torch.stack(rows)})
        npz(f"known_slew_{name}_f64", **out)


if __name__ == "__main__":
    main()
