#!/usr/bin/env python3
"""Line-search fixtures: LQR steps whose rollout backtracks, from the REAL reference.

Run with a checkout of locuslab/mpc.pytorch:   MPC_REFERENCE=<checkout> python oracle/make_golden_linesearch.py
Each case is a float64 batch from tests/gpu_harness.line_search_case (nominal trajectories that are not rollouts of
the dynamics from x_init, or unstable dynamics under a tight box) with problems that take one pass, backtrack and
then improve, and stay worse on every pass.  The unmodified reference's LQRStep runs one problem at a time (the
control flow every problem follows in the kernels), and oracle/lqr_oracle.py's lqr_step_forward(coupled=False) must
reproduce it on the whole batch: x, u to 1e-10, costs and the per-problem norm of the first pass's du (full_du_norm
of the problem alone) to 1e-9 relative, every problem's alpha exactly.  Stores the inputs, the options and the reference's new_x, new_u, costs, full_du_norm,
alphas and n_qp [B] (the pnqp iteration total of each problem alone) as tests/golden/ls_<name>.npz.  Only numbers are stored.
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
from tests.gpu_harness import MAX, MID, ONE, line_search_case   # noqa: E402

F64 = torch.float64
LAYOUT = (ONE, MID, MAX, ONE, MAX, MID, ONE, MAX)
# (name, seed, T, n, m, mode, max_ls, decay)
CASES = [("ls_max1_box", 61, 5, 4, 2, "box", 1, 0.2),
         ("ls_max3_boxD", 62, 5, 4, 2, "boxD", 3, 0.5),
         ("ls_max40_boxM", 63, 4, 3, 2, "boxM", 40, 0.9),
         ("ls_max10_plain", 64, 5, 3, 1, "plain", 10, 0.5)]


def main():
    rmpc, rstep, _, _ = load_reference()
    for name, seed, T, n, m, mode, max_ls, decay in CASES:
        case = line_search_case(seed, T, n, m, F64, mode, max_ls, decay, LAYOUT, 64)
        P, kw = case.P, case.kw
        B = P["x0"].shape[0]
        outs = []
        for b in range(B):
            s = lambda v: v[:, b:b + 1].contiguous() if torch.is_tensor(v) else v  # noqa: E731
            opts = {k: s(v) for k, v in kw.items()}
            step = rstep.LQRStep(n, m, T, true_cost=rmpc.QuadCost(s(P["C"]), s(P["c"])),
                                 true_dynamics=rmpc.LinDx(s(P["F"]), s(P["f"])), current_x=s(P["x"]),
                                 current_u=s(P["u"]), **opts)
            with contextlib.redirect_stdout(io.StringIO()):
                outs.append(step(P["x0"][b:b + 1], s(P["C"]), s(P["c"]), s(P["F"]), s(P["f"])))
        nx, nu = torch.cat([o[0] for o in outs], 1), torch.cat([o[1] for o in outs], 1)
        nqp = torch.tensor([float(o[2]) for o in outs], dtype=F64)
        costs, fdn = torch.cat([o[3] for o in outs]), torch.cat([o[4] for o in outs])
        alphas = torch.stack([o[5] for o in outs]).to(F64)
        o = case.o64
        close(o.new_x, nx, 1e-10, name + ".x")
        close(o.new_u, nu, 1e-10, name + ".u")
        close(o.costs, costs, 1e-9 * max(1.0, float(costs.abs().max())), name + ".costs")
        # per problem (the oracle's full_du_norm mixes the batch as the reference's does): from the first pass
        close((P["u"] - case.first64).pow(2).sum((0, 2)).sqrt(), fdn, 1e-9 * max(1.0, float(fdn.abs().max())),
              name + ".fdn")
        assert torch.equal(o.alphas, alphas), (name, o.alphas.tolist(), alphas.tolist())
        print(f"  {name}: classes {case.classes.tolist()}, alphas {alphas.tolist()}")
        npz(name, C=P["C"], c=P["c"], F=P["F"], f=P["f"], x_init=P["x0"], cur_x=P["x"], cur_u=P["u"],
            u_lower=kw.get("u_lower"), u_upper=kw.get("u_upper"), u_zero_I=kw.get("u_zero_I"),
            delta_u=kw.get("delta_u"), linesearch_decay=decay, max_linesearch_iter=np.int64(max_ls),
            new_x=nx, new_u=nu, costs=costs, full_du_norm=fdn, alphas=alphas, n_qp=nqp, classes=case.classes)


if __name__ == "__main__":
    main()
