"""Drop-in package name of the reference (``from mpc import mpc``); the implementation lives
in :mod:`mpc.pytorch_b200` (H100-native CUDA behind the C ABI of include/mpcb200.h)."""
