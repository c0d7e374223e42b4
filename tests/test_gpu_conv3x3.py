"""The 3x3 stride-1 convs (csrc/conv_tc.cu) on every 3x3 shape the ImageNet / FFHQ (f16) and f8 decoders run, against an fp64 conv
of the very operands the kernel multiplies (hi + lo: the split-fp16 products).  Cout % 128 == 0 -- every shape here but Cout = 3 and
64 -- runs conv3x3_wreg_kernel; conv_out (Cout = 3) and Cout = 64 run the input-stationary conv3x3_tc_kernel."""
import pytest
import torch

from rqvae import _native as N

pytestmark = pytest.mark.gpu
DEV = "cuda"

# (B, H, W, Cin, Cout): conv_in, the res blocks (Cin != Cout: the first block of a level), the upsample convs into each level
DECODER_SHAPES = [
    (2, 8, 8, 256, 512), (3, 8, 8, 512, 512), (2, 16, 16, 512, 512), (2, 32, 32, 512, 256), (1, 32, 32, 256, 256),
    (1, 32, 32, 256, 512), (1, 64, 64, 256, 256), (1, 64, 64, 512, 256), (1, 128, 128, 256, 256), (1, 128, 128, 256, 128),
    (1, 128, 128, 128, 128), (1, 256, 256, 128, 128), (1, 256, 256, 256, 128),
]
# maps smaller than the 8 x 16 tile and the 64-channel output tile
EDGE_SHAPES = [(3, 4, 4, 256, 256), (2, 2, 8, 128, 128), (2, 16, 16, 64, 64)]
# fp32 accumulation of the exact products, minus the dropped lo*lo term (2^-22 relative)
TOL = 2e-4


def operands(B, H, W, Cin, Cout, seed):
    """fp16 NHWC / OHWI operands (hi, lo) and the fp64 NCHW / OIHW tensors they represent exactly"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, H, W, Cin, generator=g)
    w = torch.randn(Cout, 3, 3, Cin, generator=g) / (Cin * 9) ** 0.5
    x_hi, w_hi = x.half(), w.half()
    x_lo, w_lo = (x - x_hi.float()).half(), (w - w_hi.float()).half()
    xr = x_hi.double() + x_lo.double()
    wr = w_hi.double() + w_lo.double()
    dev = [t.to(DEV) for t in (x_hi, w_hi, x_lo, w_lo)]
    return dev, xr.permute(0, 3, 1, 2).to(DEV), wr.permute(0, 3, 1, 2).to(DEV)


def run(ops, bias, resid, B, H, W, Cin, Cout, nchw=False):
    x_hi, w_hi, x_lo, w_lo = ops
    out = torch.full((B, Cout, H, W) if nchw else (B, H, W, Cout), float("nan"), device=DEV)
    N.check(N.lib().rqb200_dbg_conv_tc(N.ptr(x_hi), N.ptr(w_hi), N.ptr(x_lo), N.ptr(w_lo), N.ptr(bias), N.ptr(resid), N.ptr(out),
                                       B, H, W, Cin, Cout, 3, int(nchw), N.stream_ptr()), "dbg_conv_tc")
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("B,H,W,Cin,Cout", DECODER_SHAPES + EDGE_SHAPES)
def test_conv3x3_matches_fp64_conv(B, H, W, Cin, Cout):
    ops, xr, wr = operands(B, H, W, Cin, Cout, B * 7919 + H * 31 + Cin + Cout)
    g = torch.Generator().manual_seed(H + Cout)
    bias = torch.randn(Cout, generator=g).to(DEV)
    R = torch.randn(B, H, W, Cout, generator=g).to(DEV)
    ref = torch.nn.functional.conv2d(xr, wr, bias.double(), padding=1).permute(0, 2, 3, 1)
    got = run(ops, bias, None, B, H, W, Cin, Cout)
    torch.testing.assert_close(got.double(), ref, rtol=TOL, atol=TOL)
    got = run(ops, bias, R, B, H, W, Cin, Cout)
    torch.testing.assert_close(got.double(), ref + R.double(), rtol=TOL, atol=TOL)


@pytest.mark.parametrize("B,H", [(1, 256), (2, 16), (3, 8)])
def test_conv3x3_conv_out_nchw(B, H):
    """the decoder's conv_out: Cout = 3 through a 16-channel tile, NCHW fp32 pixels"""
    ops, xr, wr = operands(B, H, H, 128, 3, 100 + B + H)
    bias = torch.randn(3, generator=torch.Generator().manual_seed(H)).to(DEV)
    ref = torch.nn.functional.conv2d(xr, wr, bias.double(), padding=1)
    got = run(ops, bias, None, B, H, H, 128, 3, nchw=True)
    torch.testing.assert_close(got.double(), ref, rtol=TOL, atol=TOL)


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(2, 8, 8, 256, 512), (3, 8, 8, 512, 512), (2, 16, 16, 128, 128),
                                             (1, 32, 32, 512, 256), (1, 256, 256, 128, 128), (2, 64, 32, 256, 256)])
def test_conv3x3_groupnorm_statistics(B, H, W, Cin, Cout):
    """the epilogue's GroupNorm(32) partial statistics: per (image, group) they add up to the sum and the sum of squares of the
    output the same launch stored (bias and residual included)"""
    ops, _, _ = operands(B, H, W, Cin, Cout, 7 + H + Cout)
    g = torch.Generator().manual_seed(Cin)
    bias = torch.randn(Cout, generator=g).to(DEV)
    R = torch.randn(B, H, W, Cout, generator=g).to(DEV)
    chunks = H * W // 32
    part = torch.full((B * chunks * 32 * 2,), float("nan"), dtype=torch.float64, device=DEV)
    out = torch.full((B, H, W, Cout), float("nan"), device=DEV)
    x_hi, w_hi, x_lo, w_lo = ops
    N.check(N.lib().rqb200_dbg_conv_tc_gn(N.ptr(x_hi), N.ptr(w_hi), N.ptr(x_lo), N.ptr(w_lo), N.ptr(bias), N.ptr(R), N.ptr(out),
                                          N.ptr(part), B, H, W, Cin, Cout, 3, 0, N.stream_ptr()), "dbg_conv_tc_gn")
    torch.cuda.synchronize()
    assert not torch.isnan(part).any()
    got = part.view(B, chunks, 32, 2).sum(1)
    y = out.double().reshape(B, H * W, 32, Cout // 32)
    n = H * W * Cout // 32
    torch.testing.assert_close(got[..., 0], y.sum((1, 3)), rtol=1e-5, atol=1e-5 * n)
    torch.testing.assert_close(got[..., 1], (y * y).sum((1, 3)), rtol=1e-5, atol=1e-5 * n)
