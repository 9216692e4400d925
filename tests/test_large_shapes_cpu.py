"""Shapes without a compiled instance, without a device: which kernel shape the host picks, the error past the
large-shape kernel's shared-memory limit, mpcb200_step_large_fits and the adjoint workspace sizes."""
import ctypes

import pytest

ENVELOPE = [(n, m) for m in range(1, 33) for n in range(1, 65 - m)]


def _lib():
    from mpc.pytorch_b200 import _lib
    return _lib


def _dims(n, m, B=3, T=5):
    return _lib().Dims(B=B, T=T, n=n, m=m, F_T=T - 1, has_f=1, max_ls_iter=10, pnqp_max_iter=20, do_rollout=1)


def _fits(n, m, es):
    return _lib().lib().mpcb200_step_large_fits(ctypes.byref(_dims(n, m)), es)


def test_large_fits_covers_the_envelope():
    """Every (n, m) with n + m <= 64 and m <= 32 runs in float32 and float64."""
    for es in (4, 8):
        assert all(_fits(n, m, es) for n, m in ENVELOPE)


def test_large_fits_is_monotone_and_rejects_bad_input():
    from mpc.pytorch_b200.step import large_limit
    for es in (4, 8):
        for m in (1, 4, 16, 32):
            nmax = large_limit(m, es)
            assert nmax >= 64 - m and _fits(nmax, m, es) and not _fits(nmax + 1, m, es)
    assert large_limit(4, 8) < large_limit(4, 4)
    L = _lib().lib()
    assert L.mpcb200_step_large_fits(None, 4) == 0
    assert L.mpcb200_step_large_fits(ctypes.byref(_dims(20, 4)), 2) == 0
    assert L.mpcb200_step_large_fits(ctypes.byref(_dims(0, 4)), 4) == 0


def test_routing():
    from mpc.pytorch_b200.step import _pick_instance, _pick_instance_uncached
    assert _pick_instance(16, 4) == (16, 4)                   # exact instance
    assert _pick_instance(13, 3) == (16, 4)                   # padded as before
    assert _pick_instance(9, 1) == (12, 4)
    for n, m in ((17, 1), (20, 4), (14, 7), (24, 8), (32, 32), (48, 16), (1, 5)):
        for es in (4, 8):
            assert _pick_instance_uncached(n, m, es) == (n, m)  # no instance covers it: unpadded, large kernel


@pytest.mark.parametrize("es,name", [(4, "float32"), (8, "float64")])
def test_error_past_the_limit_names_it(es, name):
    from mpc.pytorch_b200.step import _pick_instance_uncached, large_limit
    nmax = large_limit(8, es)
    with pytest.raises(_lib().MpcB200Error, match=rf"{name} \(n_state <= {nmax} for n_ctrl=8"):
        _pick_instance_uncached(nmax + 1, 8, es)


def test_step_prefers_workspace_for_large_shapes():
    L = _lib().lib()
    for n, m in ((17, 1), (48, 16)):
        assert L.mpcb200_step_prefers_workspace(ctypes.byref(_dims(n, m)), 4) == 1
    assert L.mpcb200_step_smem_bytes(ctypes.byref(_dims(20, 4)), 4) == 0       # instances only
    assert L.mpcb200_supported(20, 4) == 0


def _adj_bytes_without_gains(B, T, n, m, es):
    """The adjoint workspace of an instance shape (include/mpcb200.h): each piece rounded up to 256 bytes."""
    up = lambda v: (v + 255) // 256 * 256
    TB = T * B
    return (up(TB * (n + m) * es) + up((TB * (n + m) + B * n) * es) + up(TB * n * es) + up(TB * m * es)
            + up(2 * TB * n * es) + up(3 * B * es) + up(TB * m) + up(TB * m * es))


@pytest.mark.parametrize("es", [4, 8])
def test_adjoint_workspace_sizes(es):
    L = _lib().lib()
    size = lambda n, m, B, T: L.mpcb200_adjoint_workspace_bytes(ctypes.byref(_dims(n, m, B, T)), es)
    up = lambda v: (v + 255) // 256 * 256
    prefers = lambda n, m, T: L.mpcb200_step_prefers_workspace(ctypes.byref(_dims(n, m, 7, T)), es)
    gains = lambda n, m, B, T: up(T * B * m * n * es) + up(T * B * m * es)
    for n, m in ((8, 2), (16, 4), (5, 1), (12, 4)):                           # instance shapes, short horizon
        assert not prefers(n, m, 9) and size(n, m, 7, 9) == _adj_bytes_without_gains(7, 9, n, m, es)
    # (16, 4) past the horizon where its step keeps the gains in Ks/ks (KREDUCE): + the nested step's gains
    assert prefers(16, 4, 50) and size(16, 4, 7, 50) == _adj_bytes_without_gains(7, 50, 16, 4, es) + gains(16, 4, 7, 50)
    for n, m in ((20, 4), (14, 7)):                                          # large shapes: + the nested gains
        B, T = 7, 9
        assert size(n, m, B, T) == _adj_bytes_without_gains(B, T, n, m, es) + gains(n, m, B, T)


# ------------------------------------------------------------------------------------------------------------------
# the oracle reproduces the reference's fixtures at shapes without an instance (oracle/make_golden_large.py)
# ------------------------------------------------------------------------------------------------------------------
def test_oracle_reproduces_slew_fixture():
    import torch
    from oracle import lqr_oracle as orc
    from oracle.make_golden_large import slew_augment
    from tests.helpers import load_golden, maxdiff
    g = load_golden("large_slew_f64")
    T, B, p = g["C"].shape[:3]
    n = g["x_init"].shape[1]
    m = p - n
    b = float(g["bound"])
    F = torch.cat((g["A"], g["Bm"]), 1).expand(T - 1, B, n, p)
    C2, c2, F2, x02 = slew_augment(g["C"], g["c"], F, g["x_init"], g["prev_ctrl"], float(g["penalty"]), n, m)
    x, u, _, _ = orc.mpc_forward_lin(n + m, m, T, x02, C2, c2, F2, None, u_lower=-b, u_upper=b,
                                     lqr_iter=int(g["lqr_iter"]), eps=1e-9, coupled=True)
    assert maxdiff(u, g["u"]) <= 1e-10 and maxdiff(x[:, :, m:], g["x"]) <= 1e-10
    # d u* / d c: the KKT adjoint of the returned solution, one unit upstream gradient per (t, control), all
    # problems at once (problems are independent)
    rows = torch.zeros(T, B, m, T, B, p, dtype=torch.float64)
    for t in range(T):
        for j in range(m):
            du = torch.zeros(T, B, m, dtype=torch.float64)
            du[t, :, j] = 1.0
            out = orc.lqr_step_backward(n + m, m, T, x02, C2, c2, F2, None, x, u, torch.zeros(T, B, n + m,
                                        dtype=torch.float64), du, u_lower=-b, u_upper=b, coupled=True)
            dc = out[2][..., m:]
            for bb in range(B):
                rows[t, bb, j, :, bb] = dc[:, bb]
    assert maxdiff(rows.reshape(T * B * m, -1), g["du_dc"]) <= 1e-10


def test_oracle_reproduces_unbounded_step_fixture():
    from oracle import lqr_oracle as orc
    from tests.helpers import load_golden, maxdiff
    g = load_golden("large_step_n14m7_f64")
    T, B, p = g["C"].shape[:3]
    n = g["x_init"].shape[1]
    m = p - n
    o = orc.lqr_step_forward(n, m, T, g["x_init"], g["C"], g["c"], g["F"], g["f"], g["cur_x"], g["cur_u"],
                             coupled=True)
    assert maxdiff(o.new_x, g["new_x"]) <= 1e-10 and maxdiff(o.new_u, g["new_u"]) <= 1e-10
    b = orc.lqr_step_backward(n, m, T, g["x_init"], g["C"], g["c"], g["F"], g["f"], g["new_x"], g["new_u"],
                              g["wx"], g["wu"], coupled=True)
    for got, key in zip(b[:5], ("dx_init", "dC", "dc", "dF", "df")):
        assert maxdiff(got, g[key]) <= 1e-10, key


def test_oracle_reproduces_bounded_step_fixture():
    from oracle import lqr_oracle as orc
    from tests.helpers import load_golden, maxdiff
    g = load_golden("large_step_n24m8_f64")
    T, B, p = g["C"].shape[:3]
    n = g["x_init"].shape[1]
    m = p - n
    o = orc.lqr_step_forward(n, m, T, g["x_init"], g["C"], g["c"], g["F"], g["f"], g["cur_x"], g["cur_u"],
                             u_lower=g["u_lower"], u_upper=g["u_upper"], coupled=False)
    assert maxdiff(o.new_x, g["new_x"]) <= 1e-10 and maxdiff(o.new_u, g["new_u"]) <= 1e-10
    assert maxdiff(o.costs, g["costs"]) <= 1e-9
    assert (1 + o.qp_iters).sum(0).tolist() == g["n_total_qp_iter"].tolist()
