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


@pytest.mark.parametrize("name", ["rqb200_dbg_conv_tc", "rqb200_dbg_conv_tc_gn"])
def test_conv_tc_refuses_narrow_nhwc_output_and_nchw_residual(name):
    """the NHWC epilogue reads the bias and stores 16 channels per access, so Cout = 3 (accepted as NCHW conv_out) would write past the
    output; the NCHW epilogue adds no residual.  Both are refused before any CUDA call."""
    assert N.lib().rqb200_version() >= 115
    buf = C.create_string_buffer(64)
    L = N.lib()
    for cout, nchw, resid in ((3, 0, None), (3, 0, buf), (3, 1, buf), (128, 1, buf)):
        if name == "rqb200_dbg_conv_tc":
            rc = L.rqb200_dbg_conv_tc(buf, buf, buf, buf, buf, resid, buf, B, H, W, CIN, cout, KS, nchw, None)
        else:
            rc = L.rqb200_dbg_conv_tc_gn(buf, buf, buf, buf, buf, resid, buf, None, B, H, W, CIN, cout, KS, nchw, None)
        assert rc == N.EINVAL, (name, cout, nchw, rc)


def test_gemm_tc_epi_refuses_bad_modes():
    """rqb200_dbg_gemm_tc_epi: a mode outside 0..3, or a partial buffer without mode 3 (or mode 3 without one), before any CUDA call"""
    buf = C.create_string_buffer(64)
    L = N.lib()
    for mode, part in ((4, None), (-1, None), (3, None), (0, buf)):
        rc = L.rqb200_dbg_gemm_tc_epi(buf, None, buf, mode, None, 1.0, None, 0, 0, None, 0, buf, part, 128, 64, 16, 1, 0, None)
        assert rc == N.EINVAL, (mode, rc)
