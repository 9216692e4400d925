"""CPU oracle for the box-constrained LQR step (TEST INFRASTRUCTURE ONLY).

This file is a from-scratch CPU restatement (torch CPU tensors, dtype generic)
of the reference algorithm in locuslab/mpc.pytorch for ONE path:
``LQRStep`` = ``lqr_backward`` + ``pnqp`` + ``lqr_forward`` + KKT adjoint.
Citations are relative to the root of a locuslab/mpc.pytorch checkout.

It is the *checker* for the CUDA path.  Only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline / ``--impl
reference`` legs may import it.  Nothing under ``mpc/`` may: the product path
fails loudly when the CUDA library is missing, it never routes here.

Parity pin: ``oracle/make_golden.py`` runs the real reference (imported from
the checkout named by $MPC_REFERENCE) and this oracle on identical seeded
inputs, asserts agreement, and stores the reference's outputs under
``tests/golden/``; ``tests/test_oracle_golden.py`` replays those fixtures
anywhere, without the reference.

Two pnqp semantics are provided (see SURVEY.md section 8(a) row P):

* ``coupled=True``  - the reference's batch-coupled control flow
  (mpc/pnqp.py:56-59, 65, 73-75): the whole batch keeps iterating until the
  slowest element converges, and the Armijo loop stops as soon as ANY element
  accepts.  This is what the reference computes for a batched call.
* ``coupled=False`` - every batch element follows the control flow the
  reference would take if it were solved alone (n_batch=1).  This is the
  semantics the CUDA kernels implement (one problem per lane group).
"""
from __future__ import annotations

from collections import namedtuple

import torch

StepOut = namedtuple(
    "StepOut",
    "new_x new_u n_total_qp_iter costs full_du_norm mean_alphas "
    "alphas Ks ks free_masks qp_iters",
)

PNQP_GAMMA = 0.1        # mpc/pnqp.py:6
PNQP_EPS_DIAG = 1e-11   # mpc/pnqp.py:8
PNQP_STEP_TOL = 1e-4    # mpc/pnqp.py:56
MASK_EPS_DIAG = 1e-8    # mpc/lqr_step.py:116


# ----------------------------------------------------------------------------
# small batched helpers (mpc/util.py:40-53)
# ----------------------------------------------------------------------------
def _mv(A, x):
    return torch.matmul(A, x.unsqueeze(-1)).squeeze(-1)


def _dot(x, y):
    return (x * y).sum(-1)


def _quad(x, A):
    return _dot(x, _mv(A, x))


def _clamp_assign(x, lo, hi):
    """eclamp (mpc/util.py:56-70): assign the bound where violated.  Out of place."""
    lo_t = torch.as_tensor(lo, dtype=x.dtype).expand_as(x)
    hi_t = torch.as_tensor(hi, dtype=x.dtype).expand_as(x)
    x = torch.where(x < lo_t, lo_t, x)
    x = torch.where(x > hi_t, hi_t, x)
    return x


def _solve(A, b):
    """LU solve with partial pivoting (the reference's Tensor.lu()/lu_solve)."""
    if b.dim() == A.dim() - 1:
        return torch.linalg.solve(A, b.unsqueeze(-1)).squeeze(-1)
    return torch.linalg.solve(A, b)


# ----------------------------------------------------------------------------
# pnqp  (mpc/pnqp.py:5-82)
# ----------------------------------------------------------------------------
def pnqp(H, q, lower, upper, x_init=None, n_iter=20, coupled=True):
    """Projected-Newton box QP  min 0.5 x'Hx + q'x,  lower <= x <= upper.

    Returns (x, H_masked, If, iters) where ``H_masked`` is the free-block
    matrix of the returning iteration (the reference returns its LU,
    mpc/pnqp.py:59,82), ``If`` the 0/1 free mask and ``iters`` an int64 [B]
    tensor (coupled: every entry equals the reference's scalar ``i``).
    """
    B, n, _ = H.shape
    eye = torch.eye(n, dtype=H.dtype)
    lower = torch.as_tensor(lower, dtype=H.dtype).expand(B, n)
    upper = torch.as_tensor(upper, dtype=H.dtype).expand(B, n)

    def obj(z):                                      # mpc/pnqp.py:11-12
        return 0.5 * _quad(z, H) + _dot(q, z)

    if x_init is None:                               # mpc/pnqp.py:14-19
        if n == 1:
            x = -(1.0 / H.squeeze(2)) * q
        else:
            x = -_solve(H, q)
    else:
        x = x_init.clone()                           # mpc/pnqp.py:21
    x = _clamp_assign(x, lower, upper)               # mpc/pnqp.py:23

    def direction(xc):
        g = _mv(H, xc) + q                           # mpc/pnqp.py:29
        Ic = ((xc == lower) & (g > 0)) | ((xc == upper) & (g < 0))   # :32
        If = ~Ic
        ff = If.unsqueeze(2) & If.unsqueeze(1)
        H_ = torch.where(ff, H, torch.zeros_like(H)) + PNQP_EPS_DIAG * eye  # :46-48
        g_ = torch.where(Ic, torch.zeros_like(g), g)                  # :44-45
        if n == 1:
            dx = -(1.0 / H_.squeeze(2)) * g_
        else:
            dx = -_solve(H_, g_)                     # :53-54
        return g, If, H_, dx

    if coupled:
        for i in range(n_iter):
            g, If, H_, dx = direction(x)
            J = torch.norm(dx, 2, 1) >= PNQP_STEP_TOL                 # :56
            if int(J.sum()) == 0:                                     # :57-59
                return x, H_, If.to(H.dtype), torch.full((B,), i, dtype=torch.int64)
            alpha = torch.ones(B, dtype=H.dtype)
            max_armijo = PNQP_GAMMA
            count = 0
            while max_armijo <= PNQP_GAMMA and count < 10:            # :65
                maybe_x = _clamp_assign(x + alpha.unsqueeze(1) * dx, lower, upper)
                armijos = torch.full((B,), PNQP_GAMMA + 1e-6, dtype=H.dtype)
                ratio = (obj(x) - obj(maybe_x)) / _dot(g, x - maybe_x)
                armijos = torch.where(J, ratio, armijos)              # :71-72
                fail = armijos <= PNQP_GAMMA
                alpha = torch.where(fail, alpha * 0.1, alpha)
                max_armijo = float(torch.max(armijos))                # NaN -> exits, like :65
                count += 1
            x = maybe_x                                               # :78
        return x, H_, If.to(H.dtype), torch.full((B,), n_iter - 1, dtype=torch.int64)

    # ---- per-element control flow (what n_batch=1 would do for each b) ----
    active = torch.ones(B, dtype=torch.bool)
    x_out = x.clone()
    H_out = torch.zeros_like(H)
    If_out = torch.ones(B, n, dtype=torch.bool)
    it_out = torch.full((B,), n_iter - 1, dtype=torch.int64)
    for i in range(n_iter):
        g, If, H_, dx = direction(x)
        small = torch.norm(dx, 2, 1) < PNQP_STEP_TOL
        done_now = active & small
        x_out = torch.where(done_now.unsqueeze(1), x, x_out)
        H_out = torch.where(done_now.view(B, 1, 1), H_, H_out)
        If_out = torch.where(done_now.unsqueeze(1), If, If_out)
        it_out = torch.where(done_now, torch.full_like(it_out, i), it_out)
        active = active & ~small
        if not bool(active.any()):
            break
        alpha = torch.ones(B, dtype=H.dtype)
        need = active.clone()
        x_new = x.clone()
        count = 0
        while bool(need.any()) and count < 10:
            maybe_x = _clamp_assign(x + alpha.unsqueeze(1) * dx, lower, upper)
            ratio = (obj(x) - obj(maybe_x)) / _dot(g, x - maybe_x)
            fail = need & (ratio <= PNQP_GAMMA)
            x_new = torch.where(need.unsqueeze(1), maybe_x, x_new)
            alpha = torch.where(fail, alpha * 0.1, alpha)
            need = fail
            count += 1
        x = torch.where(active.unsqueeze(1), x_new, x)
        if i == n_iter - 1:           # fell out of the loop: mpc/pnqp.py:80-82
            x_out = torch.where(active.unsqueeze(1), x, x_out)
            H_out = torch.where(active.view(B, 1, 1), H_, H_out)
            If_out = torch.where(active.unsqueeze(1), If, If_out)
    return x_out, H_out, If_out.to(H.dtype), it_out


# ----------------------------------------------------------------------------
# trajectory helpers (mpc/util.py:102-153) for LinDx / QuadCost
# ----------------------------------------------------------------------------
def get_traj(T, u, x_init, F, f=None):
    x = [x_init]
    for t in range(T - 1):
        xut = torch.cat((x[t], u[t]), 1)
        nx = _mv(F[t], xut)
        if f is not None and f.nelement() > 0:
            nx = nx + f[t]
        x.append(nx)
    return torch.stack(x, 0)


def get_cost(T, u, C, c, x):
    tot = 0
    for t in range(T):
        xut = torch.cat((x[t], u[t]), 1)
        tot = tot + 0.5 * _quad(xut, C[t]) + _dot(xut, c[t])
    return tot


def _bound(v, t):
    """get_bound (mpc/lqr_step.py:264-272)."""
    return v if isinstance(v, float) else v[t]


# ----------------------------------------------------------------------------
# LQRStepFn.forward  (mpc/lqr_step.py:277-309)
# ----------------------------------------------------------------------------
def lqr_step_forward(n_state, n_ctrl, T, x_init, C, c, F, f, current_x, current_u,
                     u_lower=None, u_upper=None, u_zero_I=None, delta_u=None,
                     linesearch_decay=0.2, max_linesearch_iter=10,
                     coupled=True, exact_pinv=True, dynamics=None, ls_trace=None, first_u=None):
    """One box-constrained LQR step in delta space (true cost = QuadCost).

    ``exact_pinv``: use the SVD pseudo-inverse for the unbounded m>1 branch like
    the reference (mpc/lqr_step.py:88-94); False uses an LU solve.
    ``dynamics``: the true dynamics of the line-search rollout, a callable
    ``x_{t+1} = dynamics(x_t, u_t)`` on [B, n] / [B, m] (mpc/lqr_step.py:224-225);
    None rolls out ``F[t] [x; u] + f[t]`` (LinDx, :217-222).  The Riccati sweep
    uses F (and delta space, so not f) either way.
    ``ls_trace``: a list that receives ``current_cost - old_cost`` [B] of every
    line-search pass, the comparison that decides each alpha (:247).
    ``first_u``: a list that receives new_u [T, B, m] of the first line-search pass, the full step (alpha = 1) that
    full_du_norm measures (:243-245), also when later passes backtrack.
    """
    n, m = n_state, n_ctrl
    B = C.shape[1]
    dt = C.dtype
    x, u = current_x, current_u
    has_f = f is not None and f.nelement() > 0
    assert (u_lower is None) == (u_upper is None)
    assert not (delta_u is not None and u_lower is None)   # lqr_step.py:195

    # ---- delta-space linear term (lqr_step.py:289-295)
    tau_bar = torch.cat((x, u), 2)
    c_back = _mv(C, tau_bar) + c

    # ---- backward sweep (lqr_step.py:61-158)
    Ks = [None] * T
    ks = [None] * T
    free_masks = torch.ones(T, B, m, dtype=torch.bool)
    qp_iters = torch.zeros(T, B, dtype=torch.int64)
    n_total_qp_iter = 0
    V = v = None
    prev_k = None
    for t in range(T - 1, -1, -1):
        if t == T - 1:
            Q = C[t]
            qv = c_back[t]
        else:
            Ft = F[t]
            FtT = Ft.transpose(1, 2)
            Q = C[t] + FtT.bmm(V).bmm(Ft)
            qv = c_back[t] + _mv(FtT, v)          # f_back is None in delta space (:296)
        Qxx, Qxu = Q[:, :n, :n], Q[:, :n, n:]
        Qux, Quu = Q[:, n:, :n], Q[:, n:, n:]
        qx, qu = qv[:, :n], qv[:, n:]

        if u_lower is None:
            if m == 1 and u_zero_I is None:                         # :84-86
                K = -(1.0 / Quu) * Qux
                k = -(1.0 / Quu.squeeze(2)) * qu
            elif u_zero_I is None:                                  # :88-94
                if exact_pinv:
                    Quu_inv = torch.linalg.pinv(Quu)
                    K = -Quu_inv.bmm(Qux)
                    k = -_mv(Quu_inv, qu)
                else:
                    K = -_solve(Quu, Qux)
                    k = -_solve(Quu, qu)
            else:                                                   # :100-127
                Z = u_zero_I[t].bool()
                free = ~Z
                qu_ = torch.where(Z, torch.zeros_like(qu), qu)
                ff = free.unsqueeze(2) & free.unsqueeze(1)
                Quu_ = torch.where(ff, Quu, torch.zeros_like(Quu))
                Quu_ = Quu_ + MASK_EPS_DIAG * torch.diag_embed(Z.to(dt))
                Qux_ = torch.where(Z.unsqueeze(2), torch.zeros_like(Qux), Qux)
                if m == 1:
                    K = -(1.0 / Quu_) * Qux_
                    k = -(1.0 / Quu.squeeze(2)) * qu_
                else:
                    K = -_solve(Quu_, Qux_)
                    k = -_solve(Quu_, qu_)
                free_masks[t] = free
        else:                                                       # :129-148
            lb = _bound(u_lower, t) - u[t]
            ub = _bound(u_upper, t) - u[t]
            if delta_u is not None:
                lb = torch.clamp(lb, min=-delta_u)
                ub = torch.clamp(ub, max=delta_u)
            k, H_, If, it = pnqp(Quu, qu, lb, ub, x_init=prev_k, n_iter=20, coupled=coupled)
            n_total_qp_iter += 1 + int(it.max())
            qp_iters[t] = it
            prev_k = k
            Qux_ = torch.where(If.unsqueeze(2) > 0, Qux, torch.zeros_like(Qux))
            if m == 1:
                K = -((1.0 / H_) * Qux_)
            else:
                K = -_solve(H_, Qux_)
            free_masks[t] = If > 0
        KT = K.transpose(1, 2)
        Ks[t], ks[t] = K, k
        V = Qxx + Qxu.bmm(K) + KT.bmm(Qux) + KT.bmm(Quu).bmm(K)      # :155
        v = qx + _mv(Qxu, k) + _mv(KT, qu) + _mv(KT.bmm(Quu), k)     # :156-158

    # ---- rollout with backtracking line search (lqr_step.py:164-261)
    old_cost = get_cost(T, u, C, c, x)
    alphas = torch.ones(B, dtype=dt)
    full_du_norm = None
    current_cost = None
    i = 0
    while (current_cost is None or bool(torch.any(current_cost > old_cost))) \
            and i < max_linesearch_iter:
        new_u, new_x, objs = [], [x_init], []
        for t in range(T):
            dxt = new_x[t] - x[t]
            nu = _mv(Ks[t], dxt) + u[t] + alphas.unsqueeze(1) * ks[t]   # :192
            if u_zero_I is not None:
                nu = torch.where(u_zero_I[t].bool(), torch.zeros_like(nu), nu)
            if u_lower is not None:
                lb = _bound(u_lower, t)
                ub = _bound(u_upper, t)
                if delta_u is not None:                               # :204-211
                    lb = torch.maximum(u[t] - delta_u, torch.as_tensor(lb, dtype=dt).expand_as(u[t]))
                    ub = torch.minimum(u[t] + delta_u, torch.as_tensor(ub, dtype=dt).expand_as(u[t]))
                nu = _clamp_assign(nu, lb, ub)
            new_u.append(nu)
            xut = torch.cat((new_x[t], nu), 1)
            if t < T - 1 and dynamics is not None:
                new_x.append(dynamics(new_x[t], nu))
            elif t < T - 1:
                nx = _mv(F[t], xut)
                if has_f:
                    nx = nx + f[t]
                new_x.append(nx)
            objs.append(0.5 * _quad(xut, C[t]) + _dot(xut, c[t]))     # :232
        current_cost = torch.stack(objs).sum(0)
        new_u = torch.stack(new_u)
        new_x = torch.stack(new_x)
        if full_du_norm is None:                                      # :243-245
            full_du_norm = (u - new_u).transpose(1, 2).reshape(B, -1).norm(2, 1)
            if first_u is not None:
                first_u.append(new_u)
        worse = current_cost > old_cost
        if ls_trace is not None:
            ls_trace.append(current_cost - old_cost)
        alphas = torch.where(worse, alphas * linesearch_decay, alphas)
        i += 1
    worse = current_cost > old_cost
    alphas = torch.where(worse, alphas / linesearch_decay, alphas)    # :252

    return StepOut(new_x, new_u, torch.tensor([float(n_total_qp_iter)]), current_cost,
                   full_du_norm, alphas.mean(), alphas,
                   torch.stack(Ks), torch.stack(ks), free_masks, qp_iters)


# ----------------------------------------------------------------------------
# LQRStepFn.backward  (mpc/lqr_step.py:312-407)
# ----------------------------------------------------------------------------
def lqr_step_backward(n_state, n_ctrl, T, x_init, C, c, F, f, new_x, new_u, dl_dx, dl_du,
                      u_lower=None, u_upper=None, coupled=True):
    """KKT adjoint: returns (dx_init, dC, dc, dF, df) and the adjoint (dx, du)."""
    n, m = n_state, n_ctrl
    B = C.shape[1]
    r = torch.cat((dl_dx, dl_du), 2)                                   # :316-320
    if u_lower is None:
        I = None
    else:                                                             # :325-326
        I = (torch.abs(new_u - u_lower) <= 1e-8) | (torch.abs(new_u - u_upper) <= 1e-8)
    zx = torch.zeros(T, B, n, dtype=C.dtype)
    zu = torch.zeros(T, B, m, dtype=C.dtype)
    # nested MPC(lqr_iter=1, u_zero_I=I)(0, QuadCost(C,-r), LinDx(F,None))  (:328-340):
    # iteration 0 starts from u=0, x=get_traj(0)=0; the best iterate is that one step.
    out = lqr_step_forward(n, m, T, torch.zeros_like(x_init), C, -r, F, None, zx, zu,
                           u_zero_I=I, coupled=coupled)
    dx, du = out.new_x, out.new_u
    dxu = torch.cat((dx, du), 2)
    xu = torch.cat((new_x, new_u), 2)
    dC = -0.5 * (dxu.unsqueeze(-1) * xu.unsqueeze(-2) + xu.unsqueeze(-1) * dxu.unsqueeze(-2))
    dc = -dxu                                                         # :353
    lams = [None] * T
    dlams = [None] * T
    for t in range(T - 1, -1, -1):                                    # :355-385
        Cxx, Cxu = C[t, :, :n, :n], C[t, :, :n, n:]
        lam = _mv(Cxx, new_x[t]) + _mv(Cxu, new_u[t]) + c[t, :, :n]
        dlam = _mv(Cxx, dx[t]) + _mv(Cxu, du[t]) - r[t, :, :n]
        if t < T - 1:
            FxT = F[t, :, :, :n].transpose(1, 2)
            lam = lam + _mv(FxT, lams[t + 1])
            dlam = dlam + _mv(FxT, dlams[t + 1])
        lams[t], dlams[t] = lam, dlam
    dlams_s = torch.stack(dlams)
    dF = torch.zeros_like(F)
    for t in range(T - 1):                                            # :387-395
        dF[t] = -(dlams[t + 1].unsqueeze(-1) * xu[t].unsqueeze(-2)
                  + lams[t + 1].unsqueeze(-1) * dxu[t].unsqueeze(-2))
    if f is not None and f.nelement() > 0:
        df = -dlams_s[1:]
    else:
        df = torch.Tensor()
    dx_init = -dlams_s[0]
    return dx_init, dC, dc, dF, df, dx, du


# ----------------------------------------------------------------------------
# MPC.forward for QuadCost + LinDx  (mpc/mpc.py:184-337, first branch of :339-361)
# ----------------------------------------------------------------------------
def mpc_forward_lin(n_state, n_ctrl, T, x_init, C, c, F, f, u_lower=None, u_upper=None,
                    u_init=None, lqr_iter=10, delta_u=None, eps=1e-7,
                    linesearch_decay=0.2, max_linesearch_iter=10,
                    not_improved_lim=5, best_cost_eps=1e-4, coupled=True, trace=None,
                    u_zero_I=None):
    B = C.shape[1]
    dt = C.dtype
    u = torch.zeros(T, B, n_ctrl, dtype=dt) if u_init is None else u_init.clone()
    best = None
    n_not_improved = 0
    for i in range(lqr_iter):
        x = get_traj(T, u, x_init, F, f)
        out = lqr_step_forward(n_state, n_ctrl, T, x_init, C, c, F, f, x, u,
                               u_lower=u_lower, u_upper=u_upper, u_zero_I=u_zero_I, delta_u=delta_u,
                               linesearch_decay=linesearch_decay,
                               max_linesearch_iter=max_linesearch_iter, coupled=coupled)
        x, u = out.new_x, out.new_u
        n_not_improved += 1
        if best is None:
            best = dict(x=x.clone(), u=u.clone(), costs=out.costs.clone(),
                        full_du_norm=out.full_du_norm.clone())
        else:                                                         # mpc.py:279-285
            better = out.costs <= best["costs"] + best_cost_eps
            if bool(better.any()):
                n_not_improved = 0
            best["x"] = torch.where(better.view(1, B, 1), x, best["x"])
            best["u"] = torch.where(better.view(1, B, 1), u, best["u"])
            best["costs"] = torch.where(better, out.costs, best["costs"])
            best["full_du_norm"] = torch.where(better, out.full_du_norm, best["full_du_norm"])
        if trace is not None:
            trace.append(dict(iter=i, mean_cost=float(best["costs"].mean()),
                              full_du_max=float(out.full_du_norm.max()),
                              mean_alphas=float(out.mean_alphas),
                              total_qp_iters=float(out.n_total_qp_iter)))
        if float(out.full_du_norm.max()) < eps or n_not_improved > not_improved_lim:
            break
    return best["x"], best["u"], best["costs"], best["full_du_norm"]


def ilqr_loop(n_state, n_ctrl, T, x_init, C, c, rollout, linearize, dynamics, u_init=None, lqr_iter=10, eps=1e-7,
              not_improved_lim=5, best_cost_eps=1e-4, **step_kw):
    """MPC.forward's iterations (mpc/mpc.py:244-301) with QuadCost(C, c) and nonlinear dynamics given as callables:
    x = rollout(u) [T, B, n] from x_init, (F, f) = linearize(x, u), and x_{t+1} = dynamics(x_t, u_t), the line search's
    true dynamics in lqr_step_forward.  Best-iterate tracking and the stop test as mpc_forward_lin's.  n_state is the
    (augmented) state count; step_kw: lqr_step_forward's options.  Returns (x, u, costs, iterations)."""
    B = x_init.shape[0]
    u = torch.zeros(T, B, n_ctrl, dtype=torch.float64) if u_init is None else u_init.clone()
    best, n_not_improved, it = None, 0, 0
    for it in range(1, lqr_iter + 1):
        x = rollout(u)
        F, f = linearize(x, u)
        o = lqr_step_forward(n_state, n_ctrl, T, x_init, C, c, F, f, x, u, dynamics=dynamics, **step_kw)
        x, u = o.new_x, o.new_u
        n_not_improved += 1
        if best is None:
            best = {"x": x, "u": u, "costs": o.costs, "fdn": o.full_du_norm}
            any_better = False
        else:
            better = o.costs <= best["costs"] + best_cost_eps
            sel = better.view(1, -1, 1)
            best = {"x": torch.where(sel, x, best["x"]), "u": torch.where(sel, u, best["u"]),
                    "costs": torch.where(better, o.costs, best["costs"]),
                    "fdn": torch.where(better, o.full_du_norm, best["fdn"])}
            any_better = bool(better.any())
        if any_better:
            n_not_improved = 0
        if float(o.full_du_norm.max()) < eps or n_not_improved > not_improved_lim:
            break
    return best["x"], best["u"], best["costs"], it


# ----------------------------------------------------------------------------
# receding-horizon episodes (the notebooks' loop, examples/*.ipynb) and their reverse sweep
# ----------------------------------------------------------------------------
Episode = namedtuple("Episode", "x u costs iters plan_x plan_u u_next")


def shift_warm_start(plan_u):
    """The next solve's u_init: cat(plan_u[1:], 0), then w[-2] = w[-3] (the notebooks' rule)."""
    w = torch.cat((plan_u[1:], torch.zeros_like(plan_u[:1])), 0)
    w[-2] = w[-3]
    return w


def lindx_step(F, f, x, u):
    """The LinDx plant of an episode: F[0] [x; u] + f[0] (no f: None or empty)."""
    nx = _mv(F[0], torch.cat((x, u), 1))
    return nx + f[0] if f is not None and f.nelement() > 0 else nx


def receding_horizon_lin(n_state, n_ctrl, T, n_steps, x_init, C, c, F, f, u_init=None, **kw):
    """n_steps control steps of the notebooks' loop on mpc_forward_lin: solve from x_k with u_init = w_k, apply
    u_k = plan_u[0], step the plant F[0] [x_k; u_k] + f[0], w_{k+1} = shift_warm_start(plan_u).  kw: mpc_forward_lin's
    options (bounds, delta_u, u_zero_I, lqr_iter, eps, coupled, ...).  Returns an Episode: x [n_steps+1, B, n],
    u [n_steps, B, m], costs [n_steps, B], iters [n_steps] (each solve's iterations), each solve's best iterate
    plan_x [n_steps, T, B, n], plan_u [n_steps, T, B, m], and u_next = w_{n_steps}."""
    B = C.shape[1]
    w = torch.zeros(T, B, n_ctrl, dtype=C.dtype) if u_init is None else u_init
    x = x_init
    xs, us, costs, iters, plan_x, plan_u = [x_init], [], [], [], [], []
    for _ in range(n_steps):
        trace = []
        bx, bu, bc, _ = mpc_forward_lin(n_state, n_ctrl, T, x, C, c, F, f, u_init=w, trace=trace, **kw)
        x = lindx_step(F, f, x, bu[0])
        w = shift_warm_start(bu)
        xs.append(x)
        us.append(bu[0])
        costs.append(bc)
        iters.append(len(trace))
        plan_x.append(bx)
        plan_u.append(bu)
    return Episode(torch.stack(xs), torch.stack(us), torch.stack(costs), iters, torch.stack(plan_x),
                   torch.stack(plan_u), w)


def known_linearisation(step, theta, x, u, full=True):
    """F = [R S] [T-1, B, n, n+m] and f = x' - R x - S u of x' = step(x_t, u_t, theta) at the detached points
    (x[:-1], u[:-1]), by autograd; theta [B, NP] (one row per problem) requires grad.  full: F keeps its graph in
    theta (create_graph, this project's convention, INTEGRATION.md section 2); False: F is a constant, as in the
    reference's AUTO_DIFF linearisation (mpc/mpc.py:538-592), so f differentiates as x' alone."""
    T, B, n = x.shape
    m = u.shape[2]
    rows = []
    for t in range(T - 1):
        xt, ut = x[t].detach().requires_grad_(True), u[t].detach().requires_grad_(True)
        nx = step(xt, ut, theta)
        J = [torch.cat(torch.autograd.grad(nx[:, r].sum(), (xt, ut), retain_graph=True,
                                                 create_graph=full), 1) for r in range(n)]
        J = torch.stack(J, 1)
        if not full:
            J = J.detach()
        rows.append((J, nx - _mv(J, torch.cat((xt, ut), 1).detach())))
    return torch.stack([r[0] for r in rows]), torch.stack([r[1] for r in rows])


def receding_horizon_backward(n_state, n_ctrl, T, C, c, F, f, xs, us, plan_x, plan_u, dl_dxs, dl_dus,
                              u_lower=None, u_upper=None, step=None, theta=None, full_linearisation=True,
                              coupled=False):
    """The reverse sweep of an episode from GIVEN plans plan_x [n_steps, T, B, n], plan_u [n_steps, T, B, m], states
    xs [n_steps+1, B, n] and controls us [n_steps, B, m]: autograd's gradient of sum(dl_dxs * xs) + sum(dl_dus * us)
    for the loop `for k: plan = ctrl'(x_k); x_{k+1} = step(x_k, plan_u[k][0])`, each solve contributing MPC.forward's
    differentiable tail (lqr_step_backward at its plan with the step's bounds), the warm starts held constant.

    g = dl_dxs[n]; for k = n-1 .. 0: the model step's VJP at (x_k, u_k) splits g into an x_k part and a u_k part (LinDx:
    F[0]^T g, dF[0] += g z^T, df[0] += g); the solve's adjoint takes dl_du[0] = dl_dus[k] + (u_k part); then
    g = dl_dxs[k] + (x_k part) + dx_init_k, and dC, dc (dF, df) accumulate.

    LinDx: step None, F [T-1|T, B, n, n+m], f [T-1|T, B, n] or None / empty.  A known system: step(x, u, theta) its
    one-step model (a CPU torch forward) with per-problem parameters theta [B, NP], F = f = None; each solve
    linearises it along its plan (known_linearisation, `full_linearisation` as `full` there) and the model step
    contributes only the direct derivative of x' in theta.  Returns a dict of dx_init, dC, dc, and dF, df (LinDx; df
    None without f) or dtheta [B, NP] (one row per problem)."""
    n, m = n_state, n_ctrl
    n_steps = us.shape[0]
    known = step is not None
    dt = C.dtype
    has_f = f is not None and f.nelement() > 0
    if known:
        theta = theta.detach().clone().requires_grad_(True)
    dC, dc = torch.zeros_like(C), torch.zeros_like(c)
    dF = None if known else torch.zeros_like(F)
    df = torch.zeros_like(f) if has_f and not known else None
    dtheta = torch.zeros_like(theta) if known else None
    g = dl_dxs[n_steps].clone()
    B = g.shape[0]
    for k in range(n_steps - 1, -1, -1):
        xk, uk = xs[k], us[k]
        if known:
            xl, ul = xk.detach().requires_grad_(True), uk.detach().requires_grad_(True)
            gx, gu, gth = torch.autograd.grad((step(xl, ul, theta) * g).sum(), (xl, ul, theta))
            dtheta += gth
            Fk, fk = known_linearisation(step, theta, plan_x[k], plan_u[k], full_linearisation)
        else:
            z = torch.cat((xk, uk), 1)
            gz = _mv(F[0].transpose(1, 2), g)
            gx, gu = gz[:, :n], gz[:, n:]
            dF[0] += g.unsqueeze(2) * z.unsqueeze(1)
            if has_f:
                df[0] += g
            Fk, fk = F, f
        dl_dx = torch.zeros(T, B, n, dtype=dt)
        dl_du = torch.zeros(T, B, m, dtype=dt)
        dl_du[0] = dl_dus[k] + gu
        dxk, dCk, dck, dFk, dfk, _, _ = lqr_step_backward(
            n, m, T, plan_x[k][0], C, c, Fk.detach(), fk.detach() if fk is not None else None, plan_x[k], plan_u[k],
            dl_dx, dl_du, u_lower=u_lower, u_upper=u_upper, coupled=coupled)
        dC += dCk
        dc += dck
        if known:
            dtheta += torch.autograd.grad((Fk * dFk).sum() + (fk * dfk).sum(), theta)[0]
        else:
            dF += dFk
            if has_f:
                df[:T - 1] += dfk
        g = dl_dxs[k] + gx + dxk
    out = dict(dx_init=g, dC=dC, dc=dc)
    if known:
        out["dtheta"] = dtheta
    else:
        out.update(dF=dF, df=df)
    return out
