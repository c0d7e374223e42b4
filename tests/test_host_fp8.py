"""FP8 (E4M3) weight format, host side: per-row quantiser and the fragment-order tile packing of the fp8 weight streamer."""
import pytest
import torch

from rqvae import _native as N


def _weights(N_out, K, seed):
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(N_out, K, generator=g) / K ** 0.5
    w[1] *= 300.0                                   # an outlier row
    w[2] *= 1e-3                                    # a small row (its values land in the E4M3 subnormal range too)
    w[3] = 0.0                                      # an all-zero row (the padded rows of the cond classifier)
    w[4, 5] = 40.0                                  # one outlier element
    return w


def test_quantised_values_fill_the_e4m3_range():
    w = _weights(256, 192, 1)
    q, s = N.quantize_fp8_rows(w)
    assert q.dtype == torch.float8_e4m3fn and s.dtype == torch.float32 and q.shape == w.shape and s.shape == (256,)
    qf = q.float()
    assert bool(torch.isfinite(qf).all())
    assert float(qf.abs().max()) <= N.FP8_MAX
    nz = w.abs().amax(1) > 0
    assert bool((qf.abs().amax(1)[nz] == N.FP8_MAX).all())          # every non-zero row's largest element maps to +-448


def test_dequantisation_error_bound():
    """w / s rounded to E4M3: 3 mantissa bits (relative error <= 2^-4) above 2^-6, absolute error <= 2^-10 below it (subnormals)"""
    w = _weights(384, 256, 2)
    q, s = N.quantize_fp8_rows(w)
    err = (q.float() * s[:, None] - w).abs()
    bound = torch.maximum(w.abs() * 2.0 ** -4, s[:, None] * 2.0 ** -10) * (1 + 2.0 ** -20)
    assert bool((err <= bound).all()), float((err / bound).max())


def test_zero_rows_get_unit_scale():
    w = torch.zeros(128, 64)
    w[7, 3] = -2.5
    q, s = N.quantize_fp8_rows(w)
    assert float(s[0]) == 1.0 and bool((q[0].float() == 0).all())
    assert float(s[7]) == float(torch.tensor(2.5) / 448) and float(q[7, 3].float()) == -448.0


def test_every_e4m3_value_is_an_fp16_value():
    """the kernel widens the weights with cvt.rn.f16x2.e4m3x2: that conversion must be exact for every finite code"""
    codes = torch.arange(256, dtype=torch.int32).to(torch.uint8)
    v = codes.view(torch.float8_e4m3fn).float()
    fin = torch.isfinite(v)
    assert int(fin.sum()) == 254                                     # 0x7f / 0xff are the NaNs
    assert torch.equal(v[fin].half().float(), v[fin])


def test_tile_order_is_a_permutation_in_fragment_order():
    idx = N.fp8_tile_order()
    assert torch.equal(idx.sort().values, torch.arange(8192))
    # thread 0 of warpgroup 0, k16 step 0: rows 0 / 8, k 0,1 and 8,9 (the A fragment's four f16x2 registers, lower half first)
    assert idx[:8].tolist() == [0, 1, 8 * 64, 8 * 64 + 1, 8, 9, 8 * 64 + 8, 8 * 64 + 9]
    assert idx[8:10].tolist() == [16, 17]                            # k16 step 1 follows in the same 16 bytes
    assert idx[2048:2050].tolist() == [32, 33]                       # the second 16-byte load: k16 step 2
    assert idx[16:18].tolist() == [2, 3]                             # thread 1: next k pair
    assert idx[4 * 16:4 * 16 + 2].tolist() == [64, 65]               # thread 4: next row
    assert idx[4096:4098].tolist() == [64 * 64, 64 * 64 + 1]         # warpgroup 1: rows 64..127


@pytest.mark.parametrize("N_out,K", [(128, 64), (256, 192), (384, 1536)])
def test_pack_then_unpack_is_the_identity(N_out, K):
    q, _ = N.quantize_fp8_rows(_weights(N_out, K, N_out + K))
    packed = N.pack_fp8_tiles(q)
    assert packed.dtype == torch.uint8 and packed.numel() == N_out * K
    assert torch.equal(N.unpack_fp8_tiles(packed, N_out, K).view(torch.uint8), q.view(torch.uint8))
    # tile (T, kb) is contiguous: its bytes are exactly the bytes of rows [128 T, +128) x k [64 kb, +64)
    T, kb = N_out // 128 - 1, K // 64 - 1
    tile = packed[(T * (K // 64) + kb) * 8192:][:8192]
    want = q.view(torch.uint8)[128 * T:128 * T + 128, 64 * kb:64 * kb + 64].reshape(-1)[N.fp8_tile_order()]
    assert torch.equal(tile, want)


def test_packing_refuses_ragged_shapes():
    q, _ = N.quantize_fp8_rows(torch.randn(130, 64))
    with pytest.raises(ValueError):
        N.pack_fp8_tiles(q)
    q, _ = N.quantize_fp8_rows(torch.randn(128, 96))
    with pytest.raises(ValueError):
        N.pack_fp8_tiles(q)
