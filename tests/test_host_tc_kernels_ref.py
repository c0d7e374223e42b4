"""The float64 references of tests/test_gpu_tc_kernels.py (tests/tc_kernels_ref.py), pinned on the CPU against an independent
formulation: matmul of the dequantised operands (quantize_fp8_rows' q * s for E4M3), F.conv2d with F.pad on hi + lo, and a per-pixel
walk of the conv epilogues' GroupNorm chunks.  Every named mistake is visible on its needle inputs: its reference lies more than
both bounds away from the correct one somewhere."""
import pytest
import torch
import torch.nn.functional as F

from rqvae import _native as N
from tests import tc_kernels_ref as R


def separated(ref, tol, mut, mtol):
    return float(((ref - mut).abs() - tol - mtol).max()) > 0


@pytest.mark.parametrize("e4m3", [False, True])
@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_gemm_reference_is_matmul(e4m3, mode):
    g = torch.Generator().manual_seed(mode)
    Nn, K, B, splits = 256, 640, 37, (3 if mode == 3 else 1)
    w = torch.randn(Nn, K, generator=g) / K ** 0.5
    X = torch.randn(B, K, generator=g).half()
    if e4m3:
        W, s = N.quantize_fp8_rows(w)
        wd = W.double() * s.double()[:, None]
    else:
        W, s = w.half(), None
        wd = W.double()
    bias = torch.randn(Nn, generator=g)
    res = torch.randn(B // 4 + 3, 2 * Nn, generator=g)
    kw = dict(bias=bias, bias_scale=3.0, residual=res, ld_res=2 * Nn, res_div=4, res_row0=2, res_row_stride=Nn) if mode != 3 else {}
    ref, slack = R.gemm_ref(W, X, mode, scale=s, splits=splits, **kw)
    acc = X.double() @ wd.t()
    if mode == 3:
        torch.testing.assert_close(ref.sum(0), acc, rtol=1e-12, atol=1e-12)
        k = R.split_range(K // 64, splits, 1)
        torch.testing.assert_close(ref[1], X.double()[:, 64 * k[0]:64 * k[1]] @ wd[:, 64 * k[0]:64 * k[1]].t(), rtol=1e-12, atol=1e-12)
    else:
        want = acc + 3.0 * bias.double()
        if mode == 0:
            want = want + res.double().reshape(-1)[2 * Nn + (torch.arange(B) // 4)[:, None] * 2 * Nn + torch.arange(Nn)]
        if mode == 2:
            want = F.gelu(want)
        torch.testing.assert_close(ref, want, rtol=1e-12, atol=1e-12)
    # the accumulator bound: STEP (K / 16 steps) of sum |x w|, then at most a few u and (16-bit) an ulp
    mag = X.double().abs() @ wd.abs().t()
    assert bool((slack > 0).all())
    if mode == 0:
        assert float((slack / (mag + 10)).max()) < R.STEP * K / 16 + 1e-5


@pytest.mark.parametrize("B,H,W,Cin,Cout,ks,stride,out_nchw", [
    (2, 8, 8, 64, 128, 3, 1, 0), (1, 4, 4, 128, 3, 3, 1, 1), (3, 4, 4, 64, 128, 3, 2, 0), (2, 2, 2, 64, 64, 1, 1, 0),
    (1, 1, 1, 64, 256, 3, 2, 0), (2, 16, 8, 64, 64, 3, 1, 0)])
def test_conv_reference_is_conv2d(B, H, W, Cin, Cout, ks, stride, out_nchw):
    x_hi, x_lo, w_hi, w_lo, bias, res = R.conv_operands(B, H, W, Cin, Cout, ks, stride, seed=H + Cout, resid=not out_nchw)
    ref, slack = R.conv_ref(x_hi, x_lo, w_hi, w_lo, bias, res, B, H, W, Cin, Cout, ks, stride, out_nchw)
    x = (x_hi.double() + x_lo.double()).permute(0, 3, 1, 2)
    w = (w_hi.double() + w_lo.double()).permute(0, 3, 1, 2)
    if stride == 2:
        want = F.conv2d(F.pad(x, (0, 1, 0, 1)), w, bias.double(), stride=2)                # layers.py:50-57
    else:
        want = F.conv2d(x, w, bias.double(), padding=ks // 2)
    if res is not None:
        want = want + res.double().permute(0, 3, 1, 2)
    torch.testing.assert_close(ref if out_nchw else ref.permute(0, 3, 1, 2), want, rtol=1e-12, atol=1e-12)
    # dense operands: n = 3 ks^2 Cin / 16 steps; the split residue lo lo is ~2^-22 of the products
    assert bool((slack > 0).all()) and float((slack / (3 * ks * ks * Cin / 16 + 3)).max()) < 1e-4


def test_tile_rules_name_every_instantiation():
    k = R.conv_kernel
    assert k(32, 32, 512, 3, 1) == "conv3x3_wreg_kernel<32, 1, 1>" and k(16, 16, 512, 3, 1) == "conv3x3_wreg_kernel<16, 1, 3>"
    assert k(8, 8, 512, 3, 1) == "conv3x3_wreg_kernel<8, 2, 3>" and k(256, 256, 3, 3, 1) == "conv3x3_tc_kernel<16, 8>"
    assert k(16, 16, 64, 3, 1) == "conv3x3_tc_kernel<64, 4>" and k(8, 8, 512, 1, 1) == "conv_tc_kernel<256, 2, 3>"
    assert k(8, 8, 384, 1, 1) == "conv_tc_kernel<128, 3, 3>" and k(4, 4, 64, 3, 2) == "conv_tc_kernel<64, 4, 3>"
    assert R.conv_tile(2, 2, 128, 3, 2) == (2, 2, 32) and R.conv_tile(64, 64, 128, 3, 2) == (16, 8, 1)
    assert [R.chunk_rows(b, False) for b in (16, 17, 32, 33, 64, 65, 128, 129, 256)] == [16, 32, 32, 64, 64, 128, 128, 256, 256]
    assert R.chunk_rows(129, True) == 128
    # the AR engine's uneven splits: proj / fc2 at E = 1536 (12 tiles, 24 / 96 k blocks) and E = 1280 (10 tiles, 20 / 80)
    assert R.pick_split(12, 24) == 11 and R.pick_split(12, 96) == 11 and R.pick_split(10, 20) == 13 and R.pick_split(10, 80) == 13


@pytest.mark.parametrize("TW,TH,H,W", [(8, 32, 64, 16), (8, 16, 16, 16), (8, 8, 8, 8), (16, 8, 16, 32), (4, 8, 4, 4)])
def test_gn_partials_follow_the_epilogue_chunks(TW, TH, H, W):
    """each chunk is 32 pixels of one tile in its row-major order; the chunks of an (image, group) add up to the group's totals"""
    g = torch.Generator().manual_seed(TW + H)
    H, W = max(H, TH), max(W, TW)
    out = torch.randn(2, H, W, 128, generator=g)
    ref, mag = R.gn_partials_ref(out, TW, TH)
    v = out.double().reshape(2, H * W, 32, 4)
    torch.testing.assert_close(ref[..., 0].sum(1), v.sum((1, 3)), rtol=1e-12, atol=1e-9)
    torch.testing.assert_close(ref[..., 1].sum(1), (v * v).sum((1, 3)), rtol=1e-12, atol=1e-9)
    tiles_x = W // TW
    for y, x in ((0, 0), (H - 1, W - 1), (TH - 1, TW - 1), (H // 2, 1)):
        r = (y % TH) * TW + x % TW
        c = ((y // TH) * tiles_x + x // TW) * (TW * TH // 32) + r // 32
        ys, xs = [], []
        for yy in range(H):
            for xx in range(W):
                rr = (yy % TH) * TW + xx % TW
                if ((yy // TH) * tiles_x + xx // TW) * (TW * TH // 32) + rr // 32 == c:
                    ys.append(yy)
                    xs.append(xx)
        assert len(ys) == 32
        want = out.double()[1, ys, xs, 8:12].sum()
        assert abs(float(ref[1, c, 2, 0] - want)) < 1e-9
    assert bool((mag[..., 0] >= ref[..., 0].abs()).all())


@pytest.mark.parametrize("mutation", R.GEMM_MUTATIONS)
def test_gemm_mutations_are_visible(mutation):
    case = R.GEMM_MUTATION_CASES[mutation]
    W, s, X, bias, res = R.gemm_case_operands(case, seed=11)
    kw = dict(scale=s, bias=bias, bias_scale=case.get("bias_scale", 1.0), residual=res, ld_res=case["N"], res_div=case.get("res_div", 0),
              splits=case["splits"])
    ref, slack = R.gemm_ref(W, X, case["mode"], **kw)
    mut, mslack = R.gemm_ref(W, X, case["mode"], mutation=mutation, **kw)
    assert separated(ref, slack, mut, mslack)


@pytest.mark.parametrize("mutation", R.CONV_MUTATIONS)
def test_conv_mutations_are_visible(mutation):
    B, H, W, Cin, Cout, ks, stride = R.CONV_MUTATION_CASES[mutation]
    x_hi, x_lo, w_hi, w_lo, bias = R.conv_needles(B, H, W, Cin, Cout, ks, stride, seed=4)
    ref, slack = R.conv_ref(x_hi, x_lo, w_hi, w_lo, bias, None, B, H, W, Cin, Cout, ks, stride, 0)
    mut, mslack = R.conv_ref(x_hi, x_lo, w_hi, w_lo, bias, None, B, H, W, Cin, Cout, ks, stride, 0, mutation=mutation)
    assert separated(ref, slack, mut, mslack)


@pytest.mark.parametrize("mutation", R.GN_MUTATIONS)
def test_gn_mutations_are_visible(mutation):
    B, H, W, Cin, Cout, ks, stride = R.GN_MUTATION_CASES[mutation]
    x_hi, x_lo, w_hi, w_lo, _, _ = R.conv_operands(B, H, W, Cin, Cout, ks, stride, seed=6)
    bias = R.gn_needles_bias(Cout, 6)
    out = R.conv_ref(x_hi, x_lo, w_hi, w_lo, bias, None, B, H, W, Cin, Cout, ks, stride, 0)[0].float()
    TW, TH, _ = R.conv_tile(H, W, Cout, ks, stride)
    kern = "wreg" if ks == 3 and stride == 1 and Cout % 128 == 0 else "tc"
    ref, mag = R.gn_partials_ref(out, TW, TH)
    mut, mmag = R.gn_partials_ref(out, TW, TH, mutation)
    d = R.gn_depth(kern, Cout) * R.U32
    assert separated(ref, d * mag, mut, d * mmag)
