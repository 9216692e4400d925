"""ctypes binding of libmpcb200.so (the C ABI in include/mpcb200.h).

The product path has NO CPU fallback: if the library is missing, or a tensor is
not a CUDA tensor, the calls here raise.  torch is used only for device memory
and the current stream.
"""
import contextlib
import ctypes
import functools
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmpcb200.so")


class Dims(ctypes.Structure):
    _fields_ = [(k, ctypes.c_int32) for k in (
        "B", "T", "n", "m", "F_T", "has_f", "bounds_kind", "has_zero_mask",
        "has_delta_u", "max_ls_iter", "pnqp_max_iter", "do_rollout", "dynamics_kind", "reserved0")] + \
        [(k, ctypes.c_int64) for k in ("C_tstride", "c_tstride", "F_tstride", "f_tstride")]



class Params(ctypes.Structure):
    _fields_ = [(k, ctypes.c_double) for k in ("u_lo", "u_hi", "delta_u", "ls_decay")] + [("dyn", ctypes.c_double * 8)]


class IlqrOpts(ctypes.Structure):
    _fields_ = [(k, ctypes.c_int32) for k in ("lqr_iter", "not_improved_lim", "m_ref", "reserved0")] + \
        [(k, ctypes.c_double) for k in ("eps", "best_cost_eps")]


class Plant(ctypes.Structure):
    _fields_ = [("kind", ctypes.c_int32), ("has_f", ctypes.c_int32), ("dyn", ctypes.c_double * 8)]


# mpcb200_window.on bits (include/mpcb200.h): which inputs of a time-varying episode lie on its time axis
WIN_COST, WIN_DYN, WIN_BOUNDS, WIN_PLANT = 1, 2, 4, 8


class Window(ctypes.Structure):
    _fields_ = [("L", ctypes.c_int32), ("on", ctypes.c_int32)] + \
        [(k, ctypes.c_int64) for k in ("C_tstride", "c_tstride", "F_tstride", "f_tstride", "lo_tstride", "hi_tstride",
                                       "Fp_tstride", "fp_tstride")]


# mpcb200_mlp.activation (include/mpcb200.h)
ACT = {"sigmoid": 0, "relu": 1, "elu": 2}


class Mlp(ctypes.Structure):
    _fields_ = [("n_layers", ctypes.c_int32), ("width", ctypes.c_int32 * 5), ("activation", ctypes.c_int32),
                ("passthrough", ctypes.c_int32), ("n_prev", ctypes.c_int32), ("reserved0", ctypes.c_int32),
                ("params", ctypes.c_void_p), ("W_off", ctypes.c_int64 * 4), ("b_off", ctypes.c_int64 * 4)]


class MpcB200Error(RuntimeError):
    pass


ERR_NO_GRAPH_COND = 7   # MPCB200_ERR_NO_GRAPH_COND: the driver has no conditional graph nodes (before CUDA 12.3)


_lib = None

# every symbol include/mpcb200.h declares
EXPORTED_SYMBOLS = (
    "mpcb200_lqr_step_f32", "mpcb200_lqr_step_f64", "mpcb200_lqr_grad_f32", "mpcb200_lqr_grad_f64",
    "mpcb200_rollout_f32", "mpcb200_rollout_f64", "mpcb200_pnqp_f32", "mpcb200_pnqp_f64", "mpcb200_pnqp_max_n",
    "mpcb200_pnqp_backward_f32", "mpcb200_pnqp_backward_f64",
    "mpcb200_lqr_adjoint_f32", "mpcb200_lqr_adjoint_f64", "mpcb200_adjoint_workspace_bytes",
    "mpcb200_dyn_rollout_f32", "mpcb200_dyn_rollout_f64", "mpcb200_dyn_linearize_f32", "mpcb200_dyn_linearize_f64",
    "mpcb200_dyn_linearize_vjp_f32", "mpcb200_dyn_linearize_vjp_f64",
    "mpcb200_supported", "mpcb200_supported_list", "mpcb200_launch_count",
    "mpcb200_step_smem_bytes", "mpcb200_step_prefers_workspace", "mpcb200_last_step_plan", "mpcb200_version",
    "mpcb200_strerror", "mpcb200_step_large_fits", "mpcb200_ilqr_f32", "mpcb200_ilqr_f64",
    "mpcb200_ilqr_workspace_bytes", "mpcb200_episode_f32", "mpcb200_episode_f64", "mpcb200_episode_workspace_bytes",
    "mpcb200_episode_plans_f32", "mpcb200_episode_plans_f64", "mpcb200_episode_backward_f32",
    "mpcb200_episode_backward_f64", "mpcb200_episode_backward_workspace_bytes",
    "mpcb200_episode_backward_slew_f32", "mpcb200_episode_backward_slew_f64",
    "mpcb200_episode_backward_slew_workspace_bytes", "mpcb200_episode_plant_f32", "mpcb200_episode_plant_f64",
    "mpcb200_episode_backward_plant_f32", "mpcb200_episode_backward_plant_f64",
    "mpcb200_episode_backward_plant_workspace_bytes", "mpcb200_episode_window_f32", "mpcb200_episode_window_f64",
    "mpcb200_episode_window_workspace_bytes", "mpcb200_episode_backward_window_f32",
    "mpcb200_episode_backward_window_f64", "mpcb200_episode_backward_window_workspace_bytes",
    "mpcb200_mlp_fits", "mpcb200_mlp_rollout_f32", "mpcb200_mlp_rollout_f64", "mpcb200_mlp_linearize_f32",
    "mpcb200_mlp_linearize_f64", "mpcb200_mlp_step_f32", "mpcb200_mlp_step_f64", "mpcb200_mlp_step_workspace_bytes",
    "mpcb200_ilqr_mlp_f32", "mpcb200_ilqr_mlp_f64", "mpcb200_ilqr_mlp_workspace_bytes",
    "mpcb200_mlp_linearize_vjp_f32", "mpcb200_mlp_linearize_vjp_f64", "mpcb200_mlp_linearize_vjp_workspace_bytes",
    "mpcb200_episode_mlp_f32", "mpcb200_episode_mlp_f64", "mpcb200_episode_mlp_workspace_bytes",
    "mpcb200_episode_backward_mlp_f32", "mpcb200_episode_backward_mlp_f64",
    "mpcb200_episode_backward_mlp_workspace_bytes",
)

# mpcb200_last_step_plan() bits (include/mpcb200.h)
PLAN_GENERIC, PLAN_PAIR, PLAN_GAINS_SMEM, PLAN_KREDUCE, PLAN_LARGE = 1, 2, 4, 8, 16


def lib():
    """Load (once) and return the shared library; raise loudly if it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise MpcB200Error(
            f"{LIB_PATH} is not built. Run `python -c 'import __graft_entry__ as g; g.build()'` "
            "(or `make -C mpc/pytorch_b200/csrc`). There is no CPU fallback.")
    L = ctypes.CDLL(LIB_PATH)
    vp = ctypes.c_void_p
    step_args = [ctypes.POINTER(Dims), ctypes.POINTER(Params)] + [vp] * 22
    for name in ("mpcb200_lqr_step_f32", "mpcb200_lqr_step_f64"):
        fn = getattr(L, name)
        fn.argtypes = step_args
        fn.restype = ctypes.c_int
    grad_args = [ctypes.POINTER(Dims)] + [vp] * 15
    for name in ("mpcb200_lqr_grad_f32", "mpcb200_lqr_grad_f64"):
        fn = getattr(L, name)
        fn.argtypes = grad_args
        fn.restype = ctypes.c_int
    for name in ("mpcb200_rollout_f32", "mpcb200_rollout_f64"):
        fn = getattr(L, name)
        fn.argtypes = [ctypes.POINTER(Dims)] + [vp] * 6
        fn.restype = ctypes.c_int
    for name in ("mpcb200_pnqp_f32", "mpcb200_pnqp_f64"):
        fn = getattr(L, name)
        fn.argtypes = [ctypes.c_int32, ctypes.c_int32] + [vp] * 5 + [ctypes.c_int32] + [vp] * 6
        fn.restype = ctypes.c_int
    for name in ("mpcb200_pnqp_backward_f32", "mpcb200_pnqp_backward_f64"):
        fn = getattr(L, name)
        fn.argtypes = [ctypes.c_int32, ctypes.c_int32] + [vp] * 12
        fn.restype = ctypes.c_int
    L.mpcb200_pnqp_max_n.argtypes = [ctypes.c_int32]
    L.mpcb200_pnqp_max_n.restype = ctypes.c_int32
    for name in ("mpcb200_lqr_adjoint_f32", "mpcb200_lqr_adjoint_f64"):
        fn = getattr(L, name)
        fn.argtypes = [ctypes.POINTER(Dims), ctypes.POINTER(Params)] + [vp] * 15 + [ctypes.c_size_t, vp]
        fn.restype = ctypes.c_int
    L.mpcb200_adjoint_workspace_bytes.argtypes = [ctypes.POINTER(Dims), ctypes.c_int32]
    L.mpcb200_adjoint_workspace_bytes.restype = ctypes.c_size_t
    for name in ("mpcb200_dyn_rollout_f32", "mpcb200_dyn_rollout_f64"):
        fn = getattr(L, name)
        fn.argtypes = [ctypes.c_int32, ctypes.POINTER(ctypes.c_double), ctypes.c_int32, ctypes.c_int32] + [vp] * 4
        fn.restype = ctypes.c_int
    for name in ("mpcb200_dyn_linearize_f32", "mpcb200_dyn_linearize_f64"):
        fn = getattr(L, name)
        fn.argtypes = [ctypes.c_int32, ctypes.POINTER(ctypes.c_double), ctypes.c_int32, ctypes.c_int32] + [vp] * 5
        fn.restype = ctypes.c_int
    for name in ("mpcb200_dyn_linearize_vjp_f32", "mpcb200_dyn_linearize_vjp_f64"):
        fn = getattr(L, name)
        fn.argtypes = [ctypes.c_int32, ctypes.POINTER(ctypes.c_double), ctypes.c_int32, ctypes.c_int32] + [vp] * 7
        fn.restype = ctypes.c_int
    for name in ("mpcb200_ilqr_f32", "mpcb200_ilqr_f64"):
        fn = getattr(L, name)
        fn.argtypes = [ctypes.POINTER(Dims), ctypes.POINTER(Params), ctypes.POINTER(IlqrOpts)] + [vp] * 15 + \
            [ctypes.c_size_t, vp]
        fn.restype = ctypes.c_int
    L.mpcb200_ilqr_workspace_bytes.argtypes = [ctypes.POINTER(Dims), ctypes.POINTER(IlqrOpts), ctypes.c_int32]
    L.mpcb200_ilqr_workspace_bytes.restype = ctypes.c_size_t
    for name in ("mpcb200_episode_f32", "mpcb200_episode_f64"):
        fn = getattr(L, name)
        fn.argtypes = [ctypes.POINTER(Dims), ctypes.POINTER(Params), ctypes.POINTER(IlqrOpts), ctypes.c_int32] + \
            [vp] * 15 + [ctypes.c_size_t, vp]
        fn.restype = ctypes.c_int
    L.mpcb200_episode_workspace_bytes.argtypes = [ctypes.POINTER(Dims), ctypes.POINTER(IlqrOpts), ctypes.c_int32]
    L.mpcb200_episode_workspace_bytes.restype = ctypes.c_size_t
    for name in ("mpcb200_episode_plans_f32", "mpcb200_episode_plans_f64"):
        fn = getattr(L, name)
        fn.argtypes = [ctypes.POINTER(Dims), ctypes.POINTER(Params), ctypes.POINTER(IlqrOpts), ctypes.c_int32] + \
            [vp] * 17 + [ctypes.c_size_t, vp]
        fn.restype = ctypes.c_int
    for name in ("mpcb200_episode_backward_f32", "mpcb200_episode_backward_f64"):
        fn = getattr(L, name)
        fn.argtypes = [ctypes.POINTER(Dims), ctypes.POINTER(Params), ctypes.c_int32] + [vp] * 18 + \
            [ctypes.c_size_t, vp]
        fn.restype = ctypes.c_int
    L.mpcb200_episode_backward_workspace_bytes.argtypes = [ctypes.POINTER(Dims), ctypes.c_int32]
    L.mpcb200_episode_backward_workspace_bytes.restype = ctypes.c_size_t
    for name in ("mpcb200_episode_backward_slew_f32", "mpcb200_episode_backward_slew_f64"):
        fn = getattr(L, name)
        fn.argtypes = [ctypes.POINTER(Dims), ctypes.POINTER(Params), ctypes.c_int32, ctypes.c_int32] + [vp] * 18 + \
            [ctypes.c_size_t, vp]
        fn.restype = ctypes.c_int
    L.mpcb200_episode_backward_slew_workspace_bytes.argtypes = [ctypes.POINTER(Dims), ctypes.c_int32, ctypes.c_int32]
    L.mpcb200_episode_backward_slew_workspace_bytes.restype = ctypes.c_size_t
    for name in ("mpcb200_episode_plant_f32", "mpcb200_episode_plant_f64"):
        fn = getattr(L, name)
        fn.argtypes = [ctypes.POINTER(Dims), ctypes.POINTER(Params), ctypes.POINTER(IlqrOpts), ctypes.POINTER(Plant),
                       ctypes.c_int32] + [vp] * 20 + [ctypes.c_size_t, vp]
        fn.restype = ctypes.c_int
    for name in ("mpcb200_episode_backward_plant_f32", "mpcb200_episode_backward_plant_f64"):
        fn = getattr(L, name)
        fn.argtypes = [ctypes.POINTER(Dims), ctypes.POINTER(Params), ctypes.POINTER(Plant), ctypes.c_int32,
                       ctypes.c_int32] + [vp] * 23 + [ctypes.c_size_t, vp]
        fn.restype = ctypes.c_int
    L.mpcb200_episode_backward_plant_workspace_bytes.argtypes = [ctypes.POINTER(Dims), ctypes.c_int32,
                                                                 ctypes.POINTER(Plant), ctypes.c_int32]
    L.mpcb200_episode_backward_plant_workspace_bytes.restype = ctypes.c_size_t
    for name in ("mpcb200_episode_window_f32", "mpcb200_episode_window_f64"):
        fn = getattr(L, name)
        fn.argtypes = [ctypes.POINTER(Dims), ctypes.POINTER(Params), ctypes.POINTER(IlqrOpts), ctypes.POINTER(Window),
                       ctypes.POINTER(Plant), ctypes.c_int32] + [vp] * 20 + [ctypes.c_size_t, vp]
        fn.restype = ctypes.c_int
    L.mpcb200_episode_window_workspace_bytes.argtypes = [ctypes.POINTER(Dims), ctypes.POINTER(IlqrOpts),
                                                         ctypes.POINTER(Window), ctypes.c_int32]
    L.mpcb200_episode_window_workspace_bytes.restype = ctypes.c_size_t
    for name in ("mpcb200_episode_backward_window_f32", "mpcb200_episode_backward_window_f64"):
        fn = getattr(L, name)
        fn.argtypes = [ctypes.POINTER(Dims), ctypes.POINTER(Params), ctypes.POINTER(Window), ctypes.POINTER(Plant),
                       ctypes.c_int32, ctypes.c_int32] + [vp] * 23 + [ctypes.c_size_t, vp]
        fn.restype = ctypes.c_int
    L.mpcb200_episode_backward_window_workspace_bytes.argtypes = [ctypes.POINTER(Dims), ctypes.c_int32,
                                                                  ctypes.POINTER(Window), ctypes.POINTER(Plant),
                                                                  ctypes.c_int32]
    L.mpcb200_episode_backward_window_workspace_bytes.restype = ctypes.c_size_t
    mlp = ctypes.POINTER(Mlp)
    L.mpcb200_mlp_fits.argtypes = [mlp, ctypes.c_int32]
    L.mpcb200_mlp_fits.restype = ctypes.c_int
    for name in ("mpcb200_mlp_rollout_f32", "mpcb200_mlp_rollout_f64"):
        fn = getattr(L, name)
        fn.argtypes = [mlp] + [ctypes.c_int32] * 4 + [vp] * 4
        fn.restype = ctypes.c_int
    for name in ("mpcb200_mlp_linearize_f32", "mpcb200_mlp_linearize_f64"):
        fn = getattr(L, name)
        fn.argtypes = [mlp] + [ctypes.c_int32] * 4 + [vp] * 5
        fn.restype = ctypes.c_int
    for name in ("mpcb200_mlp_linearize_vjp_f32", "mpcb200_mlp_linearize_vjp_f64"):
        fn = getattr(L, name)
        fn.argtypes = [mlp] + [ctypes.c_int32] * 4 + [vp] * 6 + [ctypes.c_size_t, vp]
        fn.restype = ctypes.c_int
    L.mpcb200_mlp_linearize_vjp_workspace_bytes.argtypes = [mlp] + [ctypes.c_int32] * 3
    L.mpcb200_mlp_linearize_vjp_workspace_bytes.restype = ctypes.c_size_t
    for name in ("mpcb200_mlp_step_f32", "mpcb200_mlp_step_f64"):
        fn = getattr(L, name)
        fn.argtypes = [ctypes.POINTER(Dims), ctypes.POINTER(Params), mlp] + [vp] * 19 + [ctypes.c_size_t, vp]
        fn.restype = ctypes.c_int
    L.mpcb200_mlp_step_workspace_bytes.argtypes = [ctypes.POINTER(Dims), ctypes.c_int32]
    L.mpcb200_mlp_step_workspace_bytes.restype = ctypes.c_size_t
    for name in ("mpcb200_ilqr_mlp_f32", "mpcb200_ilqr_mlp_f64"):
        fn = getattr(L, name)
        fn.argtypes = [ctypes.POINTER(Dims), ctypes.POINTER(Params), ctypes.POINTER(IlqrOpts), mlp] + [vp] * 13 + \
            [ctypes.c_size_t, vp]
        fn.restype = ctypes.c_int
    L.mpcb200_ilqr_mlp_workspace_bytes.argtypes = [ctypes.POINTER(Dims), ctypes.POINTER(IlqrOpts), ctypes.c_int32]
    L.mpcb200_ilqr_mlp_workspace_bytes.restype = ctypes.c_size_t
    for name in ("mpcb200_episode_mlp_f32", "mpcb200_episode_mlp_f64"):
        fn = getattr(L, name)
        fn.argtypes = [ctypes.POINTER(Dims), ctypes.POINTER(Params), ctypes.POINTER(IlqrOpts), mlp,
                       ctypes.POINTER(Plant), ctypes.c_int32] + [vp] * 18 + [ctypes.c_size_t, vp]
        fn.restype = ctypes.c_int
    L.mpcb200_episode_mlp_workspace_bytes.argtypes = [ctypes.POINTER(Dims), ctypes.POINTER(IlqrOpts), mlp,
                                                      ctypes.c_int32]
    L.mpcb200_episode_mlp_workspace_bytes.restype = ctypes.c_size_t
    for name in ("mpcb200_episode_backward_mlp_f32", "mpcb200_episode_backward_mlp_f64"):
        fn = getattr(L, name)
        fn.argtypes = [ctypes.POINTER(Dims), ctypes.POINTER(Params), mlp, ctypes.POINTER(Plant), ctypes.c_int32] + \
            [vp] * 20 + [ctypes.c_size_t, vp]
        fn.restype = ctypes.c_int
    L.mpcb200_episode_backward_mlp_workspace_bytes.argtypes = [ctypes.POINTER(Dims), mlp, ctypes.POINTER(Plant),
                                                               ctypes.c_int32]
    L.mpcb200_episode_backward_mlp_workspace_bytes.restype = ctypes.c_size_t
    L.mpcb200_supported.argtypes = [ctypes.c_int32, ctypes.c_int32]
    L.mpcb200_supported.restype = ctypes.c_int
    L.mpcb200_supported_list.argtypes = [ctypes.POINTER(ctypes.c_int32), ctypes.c_int32]
    L.mpcb200_supported_list.restype = ctypes.c_int
    L.mpcb200_launch_count.argtypes = []
    L.mpcb200_launch_count.restype = ctypes.c_uint64
    L.mpcb200_step_smem_bytes.argtypes = [ctypes.POINTER(Dims), ctypes.c_int32]
    L.mpcb200_step_smem_bytes.restype = ctypes.c_size_t
    L.mpcb200_step_prefers_workspace.argtypes = [ctypes.POINTER(Dims), ctypes.c_int32]
    L.mpcb200_step_prefers_workspace.restype = ctypes.c_int
    L.mpcb200_step_large_fits.argtypes = [ctypes.POINTER(Dims), ctypes.c_int32]
    L.mpcb200_step_large_fits.restype = ctypes.c_int
    L.mpcb200_last_step_plan.argtypes = []
    L.mpcb200_last_step_plan.restype = ctypes.c_int32
    L.mpcb200_version.argtypes = []
    L.mpcb200_version.restype = ctypes.c_int
    L.mpcb200_strerror.argtypes = [ctypes.c_int]
    L.mpcb200_strerror.restype = ctypes.c_char_p
    _lib = L
    return L


_DTYPE_SUFFIX = {torch.float32: "_f32", torch.float64: "_f64"}


@functools.cache                # the library is loaded once per process: a symbol never changes
def entry(name, dtype):
    """The `name`_f32 or `name`_f64 symbol for tensors of `dtype`.  The outputs are allocated in the inputs' dtype, so
    any other dtype would hand a kernel buffers of the wrong element size: refuse it."""
    suffix = _DTYPE_SUFFIX.get(dtype)
    if suffix is None:
        raise MpcB200Error(f"unsupported dtype {dtype}")
    return getattr(lib(), name + suffix)


def check(rc, what):
    if rc != 0:
        raise MpcB200Error(f"{what} failed: [{rc}] {lib().mpcb200_strerror(rc).decode()}")


def supported_pairs():
    L = lib()
    n = L.mpcb200_supported_list(None, 0)
    buf = (ctypes.c_int32 * (2 * n))()
    L.mpcb200_supported_list(buf, n)
    return [(buf[2 * i], buf[2 * i + 1]) for i in range(n)]


def launch_count():
    return int(lib().mpcb200_launch_count())


def last_step_plan():
    """PLAN_* bits of the step kernel this thread launched last (0: its last step call launched none)."""
    return int(lib().mpcb200_last_step_plan())


def ptr(t):
    """Device pointer of a dense CUDA tensor (None -> NULL)."""
    if t is None:
        return None
    if not t.is_cuda:
        raise MpcB200Error("mpc.pytorch_b200 runs on CUDA tensors only (no CPU fallback)")
    if not t.is_contiguous():
        raise MpcB200Error("internal error: non-contiguous tensor reached the C ABI")
    return ctypes.c_void_p(t.data_ptr())


def ptr_view(t):
    """Device pointer of the first element of a CUDA tensor whose layout the caller has already validated
    (time-strided [T, B, ...] inputs: contiguous [B, ...] slices, any time stride)."""
    if t is None:
        return None
    if not t.is_cuda:
        raise MpcB200Error("mpc.pytorch_b200 runs on CUDA tensors only (no CPU fallback)")
    return ctypes.c_void_p(t.data_ptr())


def stream_handle(device):
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _on_device(dev):
    """`torch.cuda.device(dev)` only when `dev` is not already current (the guard costs microseconds)."""
    if dev.index is None or dev.index == torch.cuda.current_device():
        return contextlib.nullcontext()
    return torch.cuda.device(dev)
