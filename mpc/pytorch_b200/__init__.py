"""mpc.pytorch_b200 - H100-native (sm_90a) batched box-constrained LQR step.

Host-side mirror of the reference's operator interface for ONE path
(LQRStep / MPC with QuadCost + LinDx, reference mpc/lqr_step.py, mpc/mpc.py),
on top of the C ABI in include/mpcb200.h (csrc/, built in-tree as
libmpcb200.so).  CUDA only; there is no CPU fallback.
"""
from .solver import MPC, QuadCost, LinDx, GradMethods  # noqa: F401
from .control import receding_horizon, Episode  # noqa: F401
from .step import LQRStep, lqr_step_raw, lqr_grad_raw  # noqa: F401
from .boxqp import pnqp  # noqa: F401
from .models import NNDynamics, AffineDynamics  # noqa: F401
from . import _lib  # noqa: F401
