"""CPU: the C-ABI library loads, exports every symbol include/mpcb200.h declares, and the host
side refuses to compute without CUDA (no CPU fallback).  No kernel is launched here."""
import ctypes
import os
import re

import pytest
import torch

from tests.conftest import ROOT


def _header_symbols():
    src = open(os.path.join(ROOT, "include", "mpcb200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(mpcb200_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from mpc.pytorch_b200 import _lib
    L = _lib.lib()
    syms = _header_symbols()
    assert len(syms) >= 10
    for s in syms:
        assert hasattr(L, s), f"{s} declared in include/mpcb200.h but not exported"
    assert set(syms) == set(_lib.EXPORTED_SYMBOLS)
    assert L.mpcb200_version() == 2          # v2: dynamics_kind in mpcb200_dims, dyn[8] in mpcb200_params, mpcb200_dyn_*
    assert L.mpcb200_strerror(0) == b"ok"
    assert b"NULL" in L.mpcb200_strerror(1)


def test_supported_instances_cover_baseline_configs():
    from mpc.pytorch_b200 import _lib
    pairs = _lib.supported_pairs()
    for cfg in [(3, 1), (5, 1), (8, 2), (16, 4), (3, 4), (2, 2)]:
        assert cfg in pairs
        assert _lib.lib().mpcb200_supported(*cfg) == 1
    assert _lib.lib().mpcb200_supported(31, 9) == 0


def test_argument_errors_are_status_codes_not_crashes():
    from mpc.pytorch_b200 import _lib
    from mpc.pytorch_b200._lib import Dims, Params
    L = _lib.lib()
    d = Dims(B=4, T=5, n=8, m=2, F_T=4, has_f=0, bounds_kind=0, has_zero_mask=0, has_delta_u=0,
             max_ls_iter=10, pnqp_max_iter=20, do_rollout=1)
    p = Params(u_lo=0, u_hi=0, delta_u=0, ls_decay=0.2)
    nul = [None] * 22
    assert L.mpcb200_lqr_step_f32(ctypes.byref(d), ctypes.byref(p), *nul) == 1      # NULL pointer
    assert L.mpcb200_lqr_step_f32(None, ctypes.byref(p), *nul) == 1
    d.F_T = 2
    assert L.mpcb200_lqr_step_f32(ctypes.byref(d), ctypes.byref(p), *nul) == 2      # bad dims
    d.F_T, d.B = 4, 0
    assert L.mpcb200_lqr_step_f64(ctypes.byref(d), ctypes.byref(p), *nul) == 2
    assert L.mpcb200_lqr_grad_f32(ctypes.byref(d), *([None] * 15)) == 2
    d.B, d.n, d.m = 4, 8, 2
    fake = [ctypes.c_void_p(1 << 20)] * 13          # never dereferenced: the call fails on the missing workspace first
    assert L.mpcb200_lqr_grad_f32(ctypes.byref(d), *fake, None, None) == 1       # the costate workspace is required
    assert L.mpcb200_lqr_grad_f64(ctypes.byref(d), *fake, None, None) == 1
    assert L.mpcb200_step_smem_bytes(ctypes.byref(d), 4) > 0
    d.n = 31
    assert L.mpcb200_step_smem_bytes(ctypes.byref(d), 4) == 0


def test_last_step_plan_is_per_thread_and_starts_empty():
    import threading
    from mpc.pytorch_b200 import _lib
    seen = []
    th = threading.Thread(target=lambda: seen.append(_lib.last_step_plan()))
    th.start()
    th.join()
    assert seen == [0]
    assert (_lib.PLAN_GENERIC, _lib.PLAN_PAIR, _lib.PLAN_GAINS_SMEM, _lib.PLAN_KREDUCE) == (1, 2, 4, 8)
    hdr = open(os.path.join(ROOT, "include", "mpcb200.h")).read()
    for name, v in (("GENERIC", 1), ("PAIR", 2), ("GAINS_SMEM", 4), ("KREDUCE", 8)):
        assert re.search(rf"#define MPCB200_PLAN_{name} {v}u\b", hdr), name


def test_cpu_tensors_are_rejected_loudly():
    from mpc.pytorch_b200 import LQRStep, QuadCost, LinDx
    from mpc.pytorch_b200._lib import MpcB200Error
    from tests.helpers import gen_problem
    C, c, F, f, x0 = gen_problem(0, 2, 4, 3, 1, torch.float32)
    u = torch.zeros(4, 2, 1)
    x = torch.zeros(4, 2, 3)
    step = LQRStep(3, 1, 4, true_cost=QuadCost(C, c), true_dynamics=LinDx(F, f), current_x=x, current_u=u)
    with pytest.raises(MpcB200Error):
        step(x0, C, c, F, f)


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    from mpc.pytorch_b200 import _lib
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(_lib.MpcB200Error):
        _lib.lib()


def test_drop_in_import_paths():
    from mpc import mpc as m
    from mpc.lqr_step import LQRStep  # noqa: F401
    from mpc.pnqp import pnqp  # noqa: F401
    from mpc import util
    assert all(hasattr(util, k) for k in ("bger", "bmv", "bquad", "bdot", "bdiag", "eclamp", "get_traj", "get_cost",
                                           "table_log", "detach_maybe", "data_maybe", "jacobian", "expandParam"))
    import inspect
    sig = inspect.signature(m.MPC.__init__)
    assert list(sig.parameters)[1:] == [
        "n_state", "n_ctrl", "T", "u_lower", "u_upper", "u_zero_I", "u_init", "lqr_iter", "grad_method",
        "delta_u", "verbose", "eps", "back_eps", "n_batch", "linesearch_decay", "max_linesearch_iter",
        "exit_unconverged", "detach_unconverged", "backprop", "slew_rate_penalty", "prev_ctrl",
        "not_improved_lim", "best_cost_eps"]
    assert sig.parameters["lqr_iter"].default == 10 and sig.parameters["eps"].default == 1e-7
    assert sig.parameters["linesearch_decay"].default == 0.2
    s2 = inspect.signature(LQRStep)
    assert list(s2.parameters) == [
        "n_state", "n_ctrl", "T", "u_lower", "u_upper", "u_zero_I", "delta_u", "linesearch_decay",
        "max_linesearch_iter", "true_cost", "true_dynamics", "delta_space", "current_x", "current_u",
        "verbose", "back_eps", "no_op_forward"]
    assert s2.parameters["back_eps"].default == 1e-3
    assert m.QuadCost()._fields == ("C", "c") and m.QuadCost().C is None
    assert m.LinDx(1).f is None
    assert [g.name for g in m.GradMethods] == ["AUTO_DIFF", "FINITE_DIFF", "ANALYTIC", "ANALYTIC_CHECK"]
