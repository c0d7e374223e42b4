"""FP8 (E4M3) weights, kernel level: the fp8 weight streamer against an fp32 matmul of the dequantised weights q * s and the same
fp16 activations.  Every E4M3 x fp16 product is exact in the fp32 accumulator, so only the summation order (and where the row
scale is applied) differs: the fp16 streamer's tolerances apply."""
import ctypes

import pytest
import torch

from rqvae import _native as N

pytestmark = pytest.mark.gpu
DEV = "cuda"
torch.backends.cuda.matmul.allow_tf32 = False


def _operands(N_out, K, B, seed):
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(N_out, K, generator=g) / K ** 0.5
    w[::7] *= 4.0                                                   # rows of different scales
    q, s = N.quantize_fp8_rows(w.to(DEV))
    X = torch.randn(B, K, generator=g).half().to(DEV)
    bias = torch.randn(N_out, generator=g).to(DEV)
    R = torch.randn(B, N_out, generator=g).to(DEV)
    ref = X.float() @ (q.float() * s[:, None]).t()
    return N.pack_fp8_tiles(q), s, X, bias, R, ref


def _gemm(W8, s, X, bias, R, out, out_is_16, gelu, part, N_out, K, B, splits):
    return N.lib().rqb200_dbg_gemm_tc_fp8(N.ptr(W8), N.ptr(s), N.ptr(X), N.ptr(bias), N.ptr(R), N.ptr(out), out_is_16, gelu,
                                          N.ptr(part), N_out, K, B, splits, N.stream_ptr())


@pytest.mark.parametrize("N_out,K,B,splits", [(128, 64, 16, 1), (256, 128, 1, 1), (384, 128, 3, 1), (1536, 1536, 64, 1),
                                               (4608, 1536, 64, 1), (1536, 6144, 64, 6), (1536, 1536, 8, 4),
                                               (16384, 1536, 64, 1), (6144, 1536, 200, 1), (1536, 1536, 33, 24),
                                               (2048, 1024, 128, 2)])
def test_gemm_tc_fp8_matches_fp32_matmul(N_out, K, B, splits):
    W8, s, X, bias, R, ref = _operands(N_out, K, B, N_out + K + B)
    if splits == 1:
        out = torch.empty(B, N_out, device=DEV)
        N.check(_gemm(W8, s, X, bias, R, out, 0, 0, None, N_out, K, B, 1))
        torch.cuda.synchronize()
        torch.testing.assert_close(out, ref + bias + R, rtol=1e-4, atol=1e-4)
        outh = torch.empty(B, N_out, device=DEV, dtype=torch.float16)
        N.check(_gemm(W8, s, X, bias, None, outh, 1, 0, None, N_out, K, B, 1))
        torch.cuda.synchronize()
        torch.testing.assert_close(outh.float(), (ref + bias).half().float(), rtol=2e-3, atol=2e-3)
        N.check(_gemm(W8, s, X, bias, None, outh, 1, 1, None, N_out, K, B, 1))
        torch.cuda.synchronize()
        torch.testing.assert_close(outh.float(), torch.nn.functional.gelu(ref + bias).half().float(), rtol=2e-2, atol=2e-2)
    else:
        part = torch.full((splits, B, N_out), float("nan"), device=DEV)
        N.check(_gemm(W8, s, X, None, None, None, 0, 0, part, N_out, K, B, splits))
        torch.cuda.synchronize()
        torch.testing.assert_close(part.sum(0), ref, rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("N_out,K,M", [(1536, 1536, 257), (4608, 1536, 2048), (1280, 5120, 1000), (256, 256, 4096), (512, 512, 129)])
def test_gemm_tc_fp8_large_m_row_chunks(N_out, K, M):
    """more activation rows than one chunk (batched prefill / teacher-forced forward): gridDim.y chunks of 128 rows"""
    W8, s, X, bias, R, ref = _operands(N_out, K, M, N_out + K + M)
    out = R.clone()                                                  # in place: out == residual
    N.check(_gemm(W8, s, X, bias, out, out, 0, 0, None, N_out, K, M, 1))
    torch.cuda.synchronize()
    torch.testing.assert_close(out, ref + bias + R, rtol=1e-4, atol=1e-4)
    outh = torch.empty(M, N_out, device=DEV, dtype=torch.float16)
    N.check(_gemm(W8, s, X, bias, None, outh, 1, 0, None, N_out, K, M, 1))
    torch.cuda.synchronize()
    torch.testing.assert_close(outh.float(), (ref + bias).half().float(), rtol=2e-3, atol=2e-3)


def test_gemm_tc_fp8_is_deterministic():
    W8, s, X, bias, R, _ = _operands(1536, 6144, 64, 5)
    outs = []
    for _ in range(2):
        part = torch.empty(6, 64, 1536, device=DEV)
        N.check(_gemm(W8, s, X, None, None, None, 0, 0, part, 1536, 6144, 64, 6))
        outs.append(part)
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1])


def test_quantiser_gives_the_same_bits_on_the_gpu_and_the_cpu():
    g = torch.Generator().manual_seed(9)
    w = torch.randn(512, 1536, generator=g) / 40
    w[3] = 0.0
    q_c, s_c = N.quantize_fp8_rows(w)
    q_g, s_g = N.quantize_fp8_rows(w.to(DEV))
    assert torch.equal(s_g.cpu(), s_c)
    assert torch.equal(q_g.cpu().view(torch.uint8), q_c.view(torch.uint8))
    assert torch.equal(N.pack_fp8_tiles(q_g).cpu(), N.pack_fp8_tiles(q_c))


def test_gemm_tc_fp8_refuses_bad_arguments():
    W8, s, X, bias, R, _ = _operands(256, 128, 16, 3)
    out = torch.empty(16, 256, device=DEV)
    L = N.lib()
    odd = ctypes.c_void_p(W8.data_ptr() + 1)                         # the bulk copies need 16-byte aligned tiles
    assert L.rqb200_dbg_gemm_tc_fp8(odd, N.ptr(s), N.ptr(X), None, None, N.ptr(out), 0, 0, None, 256, 128, 16, 1,
                                    N.stream_ptr()) == N.EINVAL
    assert L.rqb200_dbg_gemm_tc_fp8(N.ptr(W8), None, N.ptr(X), None, None, N.ptr(out), 0, 0, None, 256, 128, 16, 1,
                                    N.stream_ptr()) == N.EINVAL
    assert _gemm(W8, s, X, None, None, out, 0, 0, None, 192, 128, 16, 1) == N.EINVAL          # N_out % 128
    assert _gemm(W8, s, X, None, None, out, 0, 0, None, 256, 96, 16, 1) == N.EINVAL           # K % 64
    part = torch.empty(3, 16, 256, device=DEV)
    assert _gemm(W8, s, X, None, None, None, 0, 0, part, 256, 128, 16, 3) == N.EINVAL         # splits > K / 64
