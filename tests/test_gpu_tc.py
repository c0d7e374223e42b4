"""wgmma tier, kernel level: the weight-streaming GEMM against an fp32 matmul of the same 16-bit-rounded operands."""
import pytest
import torch

from rqvae import _native as N

pytestmark = pytest.mark.gpu
DEV = "cuda"
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False


def gelu(x):
    return torch.nn.functional.gelu(x)


DT = {"fp16": (torch.float16, 0), "bf16": (torch.bfloat16, 1)}


@pytest.mark.parametrize("N_out,K,B,splits", [(128, 64, 16, 1), (256, 128, 1, 1), (384, 128, 3, 1), (1536, 1536, 64, 1),
                                               (4608, 1536, 64, 1), (1536, 6144, 64, 6), (1536, 1536, 8, 4),
                                               (16384, 1536, 64, 1), (6144, 1536, 200, 1), (1536, 1536, 33, 24),
                                               (2048, 1024, 128, 2)])
@pytest.mark.parametrize("fmt", ["fp16", "bf16"])
def test_gemm_tc_matches_fp32_matmul(N_out, K, B, splits, fmt):
    dt, code = DT[fmt]
    g = torch.Generator().manual_seed(N_out + K + B)
    W = (torch.randn(N_out, K, generator=g) / K ** 0.5).to(dt).to(DEV)
    X = torch.randn(B, K, generator=g).to(dt).to(DEV)
    bias = torch.randn(N_out, generator=g).to(DEV)
    R = torch.randn(B, N_out, generator=g).to(DEV)
    ref = X.float() @ W.float().t()
    L = N.lib()
    st = N.stream_ptr()
    if splits == 1:
        out = torch.empty(B, N_out, device=DEV)
        N.check(L.rqb200_dbg_gemm_tc(N.ptr(W), N.ptr(X), N.ptr(bias), N.ptr(R), N.ptr(out), 0, 0, None, N_out, K, B, 1, code, st))
        torch.cuda.synchronize()
        # fp32 accumulate of exact 16-bit products: only the summation order differs
        torch.testing.assert_close(out, ref + bias + R, rtol=1e-4, atol=1e-4)
        outb = torch.empty(B, N_out, device=DEV, dtype=dt)
        N.check(L.rqb200_dbg_gemm_tc(N.ptr(W), N.ptr(X), N.ptr(bias), None, N.ptr(outb), 1, 1, None, N_out, K, B, 1, code, st))
        torch.cuda.synchronize()
        torch.testing.assert_close(outb.float(), gelu(ref + bias).to(dt).float(), rtol=2e-2, atol=2e-2)
    else:
        part = torch.full((splits, B, N_out), float("nan"), device=DEV)
        N.check(L.rqb200_dbg_gemm_tc(N.ptr(W), N.ptr(X), None, None, None, 0, 0, N.ptr(part), N_out, K, B, splits, code, st))
        torch.cuda.synchronize()
        torch.testing.assert_close(part.sum(0), ref, rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("N_out,K,M", [(1536, 1536, 257), (4608, 1536, 2048), (1280, 5120, 1000), (256, 256, 4096)])
def test_gemm_tc_large_m_row_chunks(N_out, K, M):
    """more activation rows than one wgmma N (batched prefill / teacher-forced forward): gridDim.y chunks of 256 rows"""
    g = torch.Generator().manual_seed(N_out + K + M)
    W = (torch.randn(N_out, K, generator=g) / K ** 0.5).half().to(DEV)
    X = torch.randn(M, K, generator=g).half().to(DEV)
    bias = torch.randn(N_out, generator=g).to(DEV)
    R = torch.randn(M, N_out, generator=g).to(DEV)
    ref = X.float() @ W.float().t() + bias
    L = N.lib()
    out = R.clone()                                              # in place: out == residual (the prefill's x += ...)
    N.check(L.rqb200_dbg_gemm_tc(N.ptr(W), N.ptr(X), N.ptr(bias), N.ptr(out), N.ptr(out), 0, 0, None, N_out, K, M, 1, 0, N.stream_ptr()))
    torch.cuda.synchronize()
    torch.testing.assert_close(out, ref + R, rtol=1e-4, atol=1e-4)
    outh = torch.empty(M, N_out, device=DEV, dtype=torch.float16)
    N.check(L.rqb200_dbg_gemm_tc(N.ptr(W), N.ptr(X), N.ptr(bias), None, N.ptr(outh), 1, 0, None, N_out, K, M, 1, 0, N.stream_ptr()))
    torch.cuda.synchronize()
    torch.testing.assert_close(outh.float(), ref.half().float(), rtol=2e-3, atol=2e-3)


@pytest.mark.parametrize("B,H,W,Cin,Cout,ks,nchw,res", [
    (2, 8, 8, 256, 512, 3, 0, 0), (3, 16, 16, 512, 512, 1, 0, 1), (1, 64, 64, 256, 256, 3, 0, 1),
    (2, 256, 256, 128, 128, 3, 0, 1), (2, 256, 256, 128, 3, 3, 1, 0), (5, 8, 8, 512, 1536, 1, 0, 0),
    (1, 32, 32, 512, 256, 3, 0, 0), (2, 128, 128, 256, 128, 1, 0, 0)])
def test_conv_tc_matches_fp32_conv(B, H, W, Cin, Cout, ks, nchw, res):
    g = torch.Generator().manual_seed(B * 1000 + H + Cin + Cout)
    x = torch.randn(B, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, ks, ks, generator=g) / (Cin * ks * ks) ** 0.5
    bias = torch.randn(Cout, generator=g)
    R = torch.randn(B, Cout, H, W, generator=g)
    ref = torch.nn.functional.conv2d(x.double().to(DEV), w.double().to(DEV), bias.double().to(DEV), padding=ks // 2).float()
    if res:
        ref = ref + R.to(DEV)
    x_nhwc = x.permute(0, 2, 3, 1).contiguous().to(DEV)
    w_ohwi = w.permute(0, 2, 3, 1).contiguous().to(DEV)
    x_hi, w_hi = x_nhwc.half(), w_ohwi.half()
    x_lo, w_lo = (x_nhwc - x_hi.float()).half(), (w_ohwi - w_hi.float()).half()
    r_nhwc = R.permute(0, 2, 3, 1).contiguous().to(DEV) if res else None
    out = torch.full((B, Cout, H, W) if nchw else (B, H, W, Cout), float("nan"), device=DEV)
    L = N.lib()
    N.check(L.rqb200_dbg_conv_tc(N.ptr(x_hi), N.ptr(w_hi), N.ptr(x_lo), N.ptr(w_lo), N.ptr(bias.to(DEV)), N.ptr(r_nhwc), N.ptr(out),
                                 B, H, W, Cin, Cout, ks, nchw, N.stream_ptr()))
    torch.cuda.synchronize()
    got = out if nchw else out.permute(0, 3, 1, 2)
    # fp32 accumulate of fp32-class (split-fp16) products: summation order only
    torch.testing.assert_close(got, ref, rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("B,Ho,Cin,Cout", [(2, 128, 128, 128), (3, 8, 512, 512), (1, 32, 256, 256), (2, 16, 64, 128)])
def test_conv_tc_stride2_downsample(B, Ho, Cin, Cout):
    """layers.py:50-57: F.pad(x, (0,1,0,1)) + 3x3 stride-2 conv, as the same implicit GEMM through an element-strided tensor map"""
    g = torch.Generator().manual_seed(B * 100 + Ho + Cin)
    Hi = 2 * Ho
    x = torch.randn(B, Cin, Hi, Hi, generator=g)
    w = torch.randn(Cout, Cin, 3, 3, generator=g) / (Cin * 9) ** 0.5
    bias = torch.randn(Cout, generator=g)
    ref = torch.nn.functional.conv2d(torch.nn.functional.pad(x.double().to(DEV), (0, 1, 0, 1)), w.double().to(DEV), bias.double().to(DEV),
                                     stride=2).float()
    x_nhwc = x.permute(0, 2, 3, 1).contiguous().to(DEV)
    w_ohwi = w.permute(0, 2, 3, 1).contiguous().to(DEV)
    x_hi, w_hi = x_nhwc.half(), w_ohwi.half()
    x_lo, w_lo = (x_nhwc - x_hi.float()).half(), (w_ohwi - w_hi.float()).half()
    out = torch.full((B, Ho, Ho, Cout), float("nan"), device=DEV)
    N.check(N.lib().rqb200_dbg_conv_tc(N.ptr(x_hi), N.ptr(w_hi), N.ptr(x_lo), N.ptr(w_lo), N.ptr(bias.to(DEV)), None, N.ptr(out),
                                       B, Ho, Ho, Cin, Cout, 3, 2 << 8, N.stream_ptr()))
    torch.cuda.synchronize()
    torch.testing.assert_close(out.permute(0, 3, 1, 2), ref, rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("M,N_out,K", [(257, 1536, 1536), (2048, 4608, 1536), (1000, 1280, 5120), (4096, 256, 256), (130, 128, 64), (700, 512, 512),
                                       (6080, 6144, 1536)])
@pytest.mark.parametrize("fmt", ["fp16", "bf16"])
def test_rows_gemm_persistent_kernel(M, N_out, K, fmt):
    """the large-M GEMM of the batched prefill / forward passes (persistent 128 x BN tiles through conv_tc_kernel)"""
    dt, code = DT[fmt]
    g = torch.Generator().manual_seed(M + N_out + K)
    Mp = -(-M // 128) * 128
    W = (torch.randn(N_out, K, generator=g) / K ** 0.5).to(dt).to(DEV)
    X = torch.zeros(Mp, K, dtype=dt, device=DEV)
    X[:M] = torch.randn(M, K, generator=g).to(dt).to(DEV)
    bias = torch.randn(N_out, generator=g).to(DEV)
    R = torch.randn(M, N_out, generator=g).to(DEV)
    ref = X[:M].float() @ W.float().t() + bias
    L = N.lib()
    out = torch.cat([R, torch.full((3, N_out), 7.0, device=DEV)])                    # in place + guard rows that must stay untouched
    N.check(L.rqb200_dbg_rows_gemm(N.ptr(X), N.ptr(W), N.ptr(bias), N.ptr(out), N.ptr(out), None, 0, code, M, N_out, K, N.stream_ptr()))
    torch.cuda.synchronize()
    torch.testing.assert_close(out[:M], ref + R, rtol=1e-4, atol=1e-4)
    assert bool((out[M:] == 7.0).all())
    o16 = torch.full((M + 3, N_out), 7.0, dtype=dt, device=DEV)
    N.check(L.rqb200_dbg_rows_gemm(N.ptr(X), N.ptr(W), N.ptr(bias), None, None, N.ptr(o16), 1, code, M, N_out, K, N.stream_ptr()))
    torch.cuda.synchronize()
    torch.testing.assert_close(o16[:M].float(), gelu(ref).to(dt).float(), rtol=2e-2, atol=2e-2)
    assert bool((o16[M:] == 7.0).all())
