"""CPU: the size limit of the standalone pnqp can be queried without a device (no kernel is launched)."""


def test_pnqp_max_n_covers_n128_in_both_precisions():
    from mpc.pytorch_b200 import _lib
    L = _lib.lib()
    assert L.mpcb200_pnqp_max_n(4) >= 128
    assert L.mpcb200_pnqp_max_n(8) >= 128
    assert L.mpcb200_pnqp_max_n(4) >= L.mpcb200_pnqp_max_n(8)
    for bad in (2, 0, -8, 16):
        assert L.mpcb200_pnqp_max_n(bad) == 0
