"""The wgmma conv diagnostic entry points take split-fp16 operands only: rqb200_dbg_conv_tc and rqb200_dbg_conv_tc_gn refuse a null
lo half, or the bf16 operand bit, with RQB200_EINVAL before any CUDA call (no GPU here)."""
import ctypes as C

import pytest

from rqvae import _native as N

# a shape conv_tc_supported accepts, so a refusal can only come from the operand checks
B, H, W, CIN, COUT, KS = 1, 16, 16, 128, 128, 3
BF16_BIT = 2


def call(name, x_lo, w_lo, flags):
    buf = C.create_string_buffer(64)            # stands in for every device pointer; never dereferenced
    L = N.lib()
    if name == "rqb200_dbg_conv_tc":
        return L.rqb200_dbg_conv_tc(buf, buf, x_lo, w_lo, buf, None, buf, B, H, W, CIN, COUT, KS, flags, None)
    return L.rqb200_dbg_conv_tc_gn(buf, buf, x_lo, w_lo, buf, None, buf, buf, B, H, W, CIN, COUT, KS, flags, None)


@pytest.mark.parametrize("name", ["rqb200_dbg_conv_tc", "rqb200_dbg_conv_tc_gn"])
def test_conv_tc_refuses_missing_lo_halves_and_bf16(name):
    assert N.lib().rqb200_version() >= 114
    lo = C.create_string_buffer(64)
    for x_lo, w_lo, flags, why in ((None, lo, 0, "lo halves"), (lo, None, 0, "lo halves"), (lo, lo, BF16_BIT, "bf16")):
        rc = call(name, x_lo, w_lo, flags)
        assert rc == N.EINVAL, (name, why, rc)
        assert why in N.lib().rqb200_last_error().decode(), (name, why)
