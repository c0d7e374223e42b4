"""The input-stationary 3x3 stride-1 conv (conv3x3_tc_kernel, csrc/conv_tc.cu) on every 3x3 shape the ImageNet / FFHQ (f16) and f8
decoders run, against an fp64 conv of the very operands the kernel multiplies (hi, or hi + lo for the split products)."""
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
FORMATS = {"fp16": (torch.float16, 0), "bf16": (torch.bfloat16, 2)}       # dtype, rqb200_dbg_conv_tc flag bit


def operands(B, H, W, Cin, Cout, split, dt, seed):
    """16-bit NHWC / OHWI operands (hi, lo or None) and the fp64 NCHW / OIHW tensors they represent exactly"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, H, W, Cin, generator=g)
    w = torch.randn(Cout, 3, 3, Cin, generator=g) / (Cin * 9) ** 0.5
    x_hi, w_hi = x.to(dt), w.to(dt)
    x_lo = (x - x_hi.float()).to(dt) if split else None
    w_lo = (w - w_hi.float()).to(dt) if split else None
    xr = x_hi.double() + (x_lo.double() if split else 0)
    wr = w_hi.double() + (w_lo.double() if split else 0)
    dev = [t.to(DEV) if t is not None else None for t in (x_hi, w_hi, x_lo, w_lo)]
    return dev, xr.permute(0, 3, 1, 2).to(DEV), wr.permute(0, 3, 1, 2).to(DEV)


def tolerance(split, fmt):
    # fp32 accumulation of the exact products; split: minus the dropped lo*lo term (2^-22 relative in fp16, 2^-16 in bf16)
    return 1e-3 if (split and fmt == "bf16") else 2e-4


def run(ops, bias, resid, B, H, W, Cin, Cout, flags, nchw=False):
    x_hi, w_hi, x_lo, w_lo = ops
    out = torch.full((B, Cout, H, W) if nchw else (B, H, W, Cout), float("nan"), device=DEV)
    N.check(N.lib().rqb200_dbg_conv_tc(N.ptr(x_hi), N.ptr(w_hi), N.ptr(x_lo), N.ptr(w_lo), N.ptr(bias), N.ptr(resid), N.ptr(out),
                                       B, H, W, Cin, Cout, 3, flags | int(nchw), N.stream_ptr()), "dbg_conv_tc")
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("B,H,W,Cin,Cout", DECODER_SHAPES + EDGE_SHAPES)
@pytest.mark.parametrize("split", [0, 1])
@pytest.mark.parametrize("fmt", ["fp16", "bf16"])
def test_conv3x3_matches_fp64_conv(B, H, W, Cin, Cout, split, fmt):
    dt, flag = FORMATS[fmt]
    ops, xr, wr = operands(B, H, W, Cin, Cout, split, dt, B * 7919 + H * 31 + Cin + Cout)
    g = torch.Generator().manual_seed(H + Cout)
    bias = torch.randn(Cout, generator=g).to(DEV)
    R = torch.randn(B, H, W, Cout, generator=g).to(DEV)
    ref = torch.nn.functional.conv2d(xr, wr, bias.double(), padding=1).permute(0, 2, 3, 1)
    tol = tolerance(split, fmt)
    got = run(ops, bias, None, B, H, W, Cin, Cout, flag)
    torch.testing.assert_close(got.double(), ref, rtol=tol, atol=tol)
    got = run(ops, bias, R, B, H, W, Cin, Cout, flag)
    torch.testing.assert_close(got.double(), ref + R.double(), rtol=tol, atol=tol)


@pytest.mark.parametrize("B,H", [(1, 256), (2, 16), (3, 8)])
@pytest.mark.parametrize("split", [0, 1])
@pytest.mark.parametrize("fmt", ["fp16", "bf16"])
def test_conv3x3_conv_out_nchw(B, H, split, fmt):
    """the decoder's conv_out: Cout = 3 through a 16-channel tile, NCHW fp32 pixels"""
    dt, flag = FORMATS[fmt]
    ops, xr, wr = operands(B, H, H, 128, 3, split, dt, 100 + B + H)
    bias = torch.randn(3, generator=torch.Generator().manual_seed(H)).to(DEV)
    ref = torch.nn.functional.conv2d(xr, wr, bias.double(), padding=1)
    got = run(ops, bias, None, B, H, H, 128, 3, flag, nchw=True)
    tol = tolerance(split, fmt)
    torch.testing.assert_close(got.double(), ref, rtol=tol, atol=tol)


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(2, 8, 8, 256, 512), (3, 8, 8, 512, 512), (2, 16, 16, 128, 128),
                                             (1, 32, 32, 512, 256), (1, 256, 256, 128, 128), (2, 64, 32, 256, 256)])
@pytest.mark.parametrize("split", [0, 1])
def test_conv3x3_groupnorm_statistics(B, H, W, Cin, Cout, split):
    """the epilogue's GroupNorm(32) partial statistics: per (image, group) they add up to the sum and the sum of squares of the
    output the same launch stored (bias and residual included)"""
    ops, _, _ = operands(B, H, W, Cin, Cout, split, torch.float16, 7 + H + Cout)
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
