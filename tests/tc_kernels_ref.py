"""float64 references of the tensor-core kernels (csrc/gemm_tc.cu: the weight streamer gemm_tc_kernel<BN, WF>; csrc/conv_tc.cu:
conv_tc_kernel<BN, STAGES, PASSES> -- 1x1 and stride-2 convs and the rows GEMM --, conv3x3_tc_kernel<BN, STAGES> and
conv3x3_wreg_kernel<TH, NB, STAGES>), the error bounds the tests hold them to, and the named mistakes the bounds must reject.

Every reference starts from exactly the operands the kernel reads, converted to float64 exactly: the 16-bit X and W of the streamer
and the rows GEMM; the E4M3 q with its fp32 row scale s (the kernel widens q to fp16, exactly); the fp16 hi and lo halves of both
conv operands.  u = 2^-24 is the fp32 unit roundoff.

The accumulator model -- an ASSUMPTION.  Published studies of earlier tensor cores (Volta, Turing, Ampere) describe the fp32
accumulation of one MMA instruction as: the products are exact, they and the accumulator are aligned to the largest exponent among
them, the bits below the accumulator's precision are truncated (not rounded), and the aligned sum is normalised once per instruction.
Nobody has measured this for H100 wgmma here.  The bound below uses a conservative form of that model: one k16 step (one wgmma of
K = 16, on both the descriptor and the register-A forms) of a dot product adds 16 exact products p_j to the accumulator c with
    |error| <= 17 ulp of the largest addend <= STEP (|c| + sum_j |p_j|),   STEP = 17 * 2^-23 = 34 u,
(each of the 16 addends below the largest loses less than one ulp of it to the alignment, the normalisation one more), and a step
whose products are all zero returns the accumulator unchanged.  The E4M3 path widens q to fp16 and runs f16-kind wgmma, so the same
model applies.  Summing over the steps, |c| <= sum |p| at every step, so the accumulator after n nonzero steps is off by at most
    acc = STEP * n * sum_k |a_k w_k|.
n counts the k16 steps of one output whose weights are not all zero (an upper bound on its nonzero steps): K / 16 for the streamer
and the rows GEMM; for the split-fp16 convs, per output channel, the nonzero W_hi steps twice (W_hi X_lo and W_hi X_hi) plus the
nonzero W_lo steps (W_lo X_hi), at most 3 ks^2 Cin / 16.  Split-K: each partial is its own dot product over its k blocks.

Split-fp16.  The convs multiply (W_hi + W_lo)(X_hi + X_lo) as W_hi X_lo + W_lo X_hi + W_hi X_hi: the dropped W_lo X_lo term (at most
2^-22 of |W X| for true hi / lo splits) enters the bound as max |x_lo| sum |w_lo| per output channel, which is at least
sum |w_lo x_lo|.

Epilogues (fp32, one rounding per operation):
  E4M3 row scale: x = s acc, + u |s acc| (and s times the accumulator bound).
  bias (x bias_scale): b bs is rounded (u |b bs|), the sum is rounded (u |x + b bs|); residual: one more rounding.  All are covered by
    3 u (|x| + |b bs| + |r|) beside the accumulator bound.
  gelu_erf: 1.13 times the input's bound (|gelu'| <= 1.13) plus (4 |x| + 2 |gelu(x)|) u (tests/ar_kernels_ref.py).
  16-bit output: tol16 -- an ulp of the 16-bit format at |ref| + slack, plus slack.
GroupNorm partial sums (the conv epilogues' statistics of their own fp32 output v, so the reference is formed from the values the
kernel stored): a sum of m terms formed to addition depth d is off by at most d u sum |v| (sums) or d u sum v^2 (sums of squares,
one more level for fmaf's product folded in).  conv_tc_kernel's gn_chunk_stats<CG>: cg sequential terms per lane, then 5 shuffle
levels: d = cg + 6.  conv3x3_wreg_kernel: per lane 4 rows of (x + y) + (z + w) (and fmaf(x, x, y y) + fmaf(z, z, w w)): 7 levels,
log2(Cout / 128) lane shuffles, then the 8 warps summed in order: d = 16 + log2(Cout / 128).  The fp64 store is exact.
"""
import math

import torch
import torch.nn.functional as F

from tests.ar_kernels_ref import DT, excess, gelu64, gelu_slack, r16, tol16, ulp16  # noqa: F401  (shared tolerance helpers)

U32 = 2.0 ** -24
STEP = 17 * 2.0 ** -23            # per k16 step, relative to |acc| + sum |products| (the model above)
GELU_LIP = 1.13                   # max |gelu'(x)|


# ---------------------------------------------------------------------------------------------------------------- tile rules
def chunk_rows(B, e4m3):
    """gemm_tc_chunk_rows: the streamer's BN for B activation rows (csrc/kernels.h)"""
    return 16 if B <= 16 else 32 if B <= 32 else 64 if B <= 64 else 128 if (B <= 128 or e4m3) else 256


def stages(bn, e4m3):
    """the streamer's ring depth (GtFormat<WF>::stages)"""
    if e4m3:
        return 16 if bn <= 32 else 12 if bn == 64 else 8
    return 8 if bn <= 64 else 6 if bn == 128 else 4


def split_range(nkb, splits, s):
    """k blocks [kb0, kb1) of split s (gemm_tc_kernel)"""
    return nkb * s // splits, nkb * (s + 1) // splits


def pick_split(n_tiles, nkb, n_sm=132):
    """the AR engine's split count for a weight of n_tiles 128-row tiles and nkb k blocks (ar_fast.cu pick_split)"""
    return max(1, min(n_sm // n_tiles, nkb))


def conv_tile(H, W, Cout, ks, stride):
    """(TW, TH, NB) of launch_conv_tc's conv_tile: H, W the output extent"""
    if ks == 3 and stride == 1:
        TH = 32 if (Cout % 128 == 0 and H >= 32) else (16 if H > 8 else 8)
        return 8, TH, 2 if TH == 8 else 1
    TW = min(W, 16)
    TH = min(128 // TW, H)
    return TW, TH, 128 // (TW * TH)


def conv_kernel(H, W, Cout, ks, stride):
    """the instantiation launch_conv_tc runs, by name"""
    TW, TH, NB = conv_tile(H, W, Cout, ks, stride)
    if ks == 3 and stride == 1:
        if Cout % 128 == 0:
            return "conv3x3_wreg_kernel<%d, %d, %d>" % (TH, NB, 1 if TH == 32 else 3)
        return "conv3x3_tc_kernel<16, 8>" if Cout <= 16 else "conv3x3_tc_kernel<64, 4>"
    bn = 16 if Cout <= 16 else 256 if Cout % 256 == 0 else 128 if Cout % 128 == 0 else 64
    return "conv_tc_kernel<%d, %d, 3>" % (bn, {16: 5, 64: 4, 128: 3, 256: 2}[bn])


# ---------------------------------------------------------------------------------------------------------------- streamer
GEMM_MUTATIONS = ("last_kblock_dropped", "last_kblock_twice", "neighbour_row_scale", "neighbour_row_chunk", "tanh_gelu",
                  "bias_scale_ignored", "residual_row_m")


def _row_scale(s, N, mutation):
    if s is None:
        return None
    s = s.double()
    return s.view(-1, 2).flip(1).reshape(N) if mutation == "neighbour_row_scale" else s


def gemm_ref(W, X, mode, scale=None, bias=None, bias_scale=1.0, residual=None, ld_res=None, res_div=0, res_row0=0, res_row_stride=0,
             splits=1, fmt=0, mutation=None):
    """(ref, slack) float64 of one streamer launch.  W [N, K] 16-bit, or E4M3 q [N, K] (float8_e4m3fn) with scale [N]; X [B, K] 16-bit.
    mode 0: fp32 out [B, N] = s acc + bias * bias_scale + residual[res_row0 * res_row_stride + (m / res_div or m) * ld_res + n]
    (residual a flat fp32 tensor); 1: the same without residual, rounded to 16 bits; 2: through gelu_erf first; 3: the fp32 partials
    [splits, B, N] = s * the k blocks of each split."""
    N, K = W.shape
    B = X.shape[0]
    e4m3 = scale is not None
    Wd, Xd = W.double(), X.double()
    if mutation == "neighbour_row_chunk":
        bn = chunk_rows(B, e4m3)
        Xd = Xd[(torch.arange(B, device=X.device) + bn) % B]
    s = _row_scale(scale, N, mutation)
    nkb = K // 64
    nz = Wd.reshape(N, K // 16, 16).ne(0).any(-1)                        # [N, K/16]: k16 steps with a nonzero weight

    def dot(kb0, kb1):
        k0, k1 = 64 * kb0, 64 * kb1
        if mutation == "last_kblock_dropped":
            k1 -= 64
        acc = Xd[:, k0:k1] @ Wd[:, k0:k1].t()
        if mutation == "last_kblock_twice":
            acc = acc + Xd[:, k1 - 64:k1] @ Wd[:, k1 - 64:k1].t()
        mag = Xd[:, 64 * kb0:64 * kb1].abs() @ Wd[:, 64 * kb0:64 * kb1].abs().t()
        n = nz[:, 4 * kb0:4 * kb1].sum(-1).double()
        slack = STEP * n * mag
        if e4m3:
            acc, slack = acc * s, slack * s.abs() + U32 * (acc * s).abs()
        return acc, slack

    if mode == 3:
        parts = [dot(*split_range(nkb, splits, i)) for i in range(splits)]
        return torch.stack([p[0] for p in parts]), torch.stack([p[1] for p in parts])
    acc, slack = dot(0, nkb)
    x, side = acc, acc.abs()
    if bias is not None:
        bb = bias.double() * (1.0 if mutation == "bias_scale_ignored" else bias_scale)
        x = x + bb
        side = side + (bias.double() * bias_scale).abs()
    if mode == 0 and residual is not None:
        rows = torch.arange(B, device=X.device)
        if res_div > 1 and mutation != "residual_row_m":
            rows = rows // res_div
        idx = res_row0 * res_row_stride + rows[:, None] * ld_res + torch.arange(N, device=X.device)[None, :]
        r = residual.double().reshape(-1)[idx]
        x = x + r
        side = side + r.abs()
    slack = slack + 3 * U32 * side
    if mode == 0:
        return x, slack
    if mode == 2:
        y = gelu64(x, "tanh_gelu" if mutation == "tanh_gelu" else None)
        slack = GELU_LIP * slack + gelu_slack(x, y)
        x = y
    return x, tol16(x, slack, fmt)


def gemm_needles(N, K, B, fmt, seed, e4m3=False, device="cpu"):
    """(W or q, scale or None, X) whose every output is a short sum: row n of W is nonzero only in the first and the last k block of
    each of the 11 and 13 splits the tests use (sparse, so the worst-case bound stays tiny), rows of neighbouring pairs differ in
    scale by 2^4 (E4M3), and the activation rows are independent."""
    g = torch.Generator().manual_seed(seed)
    nkb = K // 64
    keep = torch.zeros(K, dtype=torch.bool)
    for splits in (1, 11, 13):
        for i in range(min(splits, nkb)):
            kb0, kb1 = split_range(nkb, min(splits, nkb), i)
            if kb1 > kb0:
                keep[64 * kb0 + 5] = keep[64 * kb1 - 3] = True
    w = torch.randn(N, K, generator=g) * keep
    X = r16(torch.randn(B, K, generator=g), fmt)
    if e4m3:
        w = w * torch.where(torch.arange(N) % 2 == 0, 1.0, 16.0)[:, None]
        from rqvae import _native as N_
        q, s = N_.quantize_fp8_rows(w)
        return q.to(device), s.to(device), X.to(device)
    return r16(w, fmt).to(device), None, X.to(device)


# ---------------------------------------------------------------------------------------------------------------- convs
CONV_MUTATIONS = ("drop_w_hi_x_lo", "drop_w_lo_x_hi", "transposed_taps", "halo_shifted", "stride2_pad_left_top")


def conv_ref(x_hi, x_lo, w_hi, w_lo, bias, res, B, H, W, Cin, Cout, ks, stride, out_nchw, mutation=None):
    """(ref, slack) float64 of rqb200_dbg_conv_tc, laid out as its output (NHWC [B, H, W, Cout] or NCHW).  x_*: NHWC fp16 [B, H stride,
    W stride, Cin]; w_*: OHWI fp16 [Cout, ks, ks, Cin]; H, W the output extent.  3x3 stride 1: "same" zero padding; stride 2: one zero
    row / column on the bottom / right (layers.py:50-57); 1x1: none."""
    nchw = lambda t: t.double().permute(0, 3, 1, 2)
    oihw = lambda t: t.double().permute(0, 3, 1, 2)
    xh, xl, wh, wl = nchw(x_hi), nchw(x_lo), oihw(w_hi), oihw(w_lo)
    if mutation == "transposed_taps":
        wh, wl = wh.transpose(2, 3), wl.transpose(2, 3)
    if mutation == "halo_shifted":                           # every tap reads the pixel one to the right
        sh = lambda t: F.pad(t[..., 1:], (0, 1))
        xh, xl = sh(xh), sh(xl)

    def conv(x, w):
        if stride == 2:
            x = F.pad(x, (1, 0, 1, 0) if mutation == "stride2_pad_left_top" else (0, 1, 0, 1))
            return F.conv2d(x, w, stride=2)
        return F.conv2d(x, w, padding=ks // 2)

    ref = conv(xh + xl, wh + wl)
    if mutation == "drop_w_hi_x_lo":
        ref = ref - conv(xl, wh)
    elif mutation == "drop_w_lo_x_hi":
        ref = ref - conv(xh, wl)
    mag = conv((xh + xl).abs(), (wh + wl).abs())
    lolo = xl.abs().max() * wl.abs().sum((1, 2, 3)).view(1, Cout, 1, 1)      # >= sum |x_lo w_lo| of every output
    nzh = w_hi.reshape(Cout, -1, 16).ne(0).any(-1).sum(-1).double()
    nzl = w_lo.reshape(Cout, -1, 16).ne(0).any(-1).sum(-1).double()
    n = (2 * nzh + nzl).view(1, Cout, 1, 1)
    side = ref.abs()
    if bias is not None:
        ref = ref + bias.double().view(1, Cout, 1, 1)
        side = side + bias.double().abs().view(1, Cout, 1, 1)
    if res is not None:
        r = res.double().permute(0, 3, 1, 2)
        ref, side = ref + r, side + r.abs()
    slack = STEP * n * mag + lolo + 3 * U32 * side
    if out_nchw:
        return ref, slack
    return ref.permute(0, 2, 3, 1), slack.permute(0, 2, 3, 1)


def split16(x):
    """fp32 / fp64 x -> its fp16 (hi, lo) pair: hi = fp16(x), lo = fp16(x - hi)"""
    hi = x.half()
    return hi, (x.float() - hi.float()).half()


def conv_operands(B, H, W, Cin, Cout, ks, stride, seed, device="cpu", resid=False, nchw_out=False):
    """random split-fp16 operands of a conv with output extent H x W: (x_hi, x_lo, w_hi, w_lo, bias, res)"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, H * stride, W * stride, Cin, generator=g)
    w = torch.randn(Cout, ks, ks, Cin, generator=g) / math.sqrt(ks * ks * Cin)
    bias = torch.randn(Cout, generator=g)
    res = torch.randn(B, H, W, Cout, generator=g) if resid else None
    ops = split16(x) + split16(w)
    return tuple(t.to(device) for t in ops) + (bias.to(device), res.to(device) if res is not None else None)


def conv_needles(B, H, W, Cin, Cout, ks, stride, seed, device="cpu"):
    """sparse split-fp16 operands on which every conv mutation is far outside the bound: output channel c has ONE nonzero weight, at
    tap (c % ks^2) and input channel (c * 7) % Cin, whose hi and lo are both large (lo = hi 2^-12 (1 + U[0, 1))); every activation has
    a lo of the same relative size; bias 0.  So each output is one product (three for the split terms), the bound is ~10^-5 of it,
    and each mistake moves it by at least 2^-12 of it (a dropped split term) or by a whole other product."""
    g = torch.Generator().manual_seed(seed)
    lo_of = lambda hi: (hi.float() * 2.0 ** -12 * (1 + torch.rand(hi.shape, generator=g))).half()
    x_hi = (torch.randn(B, H * stride, W * stride, Cin, generator=g) + 3.0 * torch.sign(torch.randn(1, generator=g))).half()
    x_lo = lo_of(x_hi)
    w_hi = torch.zeros(Cout, ks * ks, Cin, dtype=torch.float16)
    c = torch.arange(Cout)
    w_hi[c, c % (ks * ks), (c * 7) % Cin] = (torch.rand(Cout, generator=g) + 0.5).half()
    w_hi = w_hi.view(Cout, ks, ks, Cin)
    w_lo = lo_of(w_hi)
    bias = torch.zeros(Cout)
    return tuple(t.to(device) for t in (x_hi, x_lo, w_hi, w_lo, bias))


# ---------------------------------------------------------------------------------------------------------------- GroupNorm partials
GN_MUTATIONS = ("neighbour_group", "chunk_last_row_dropped")


def gn_depth(kernel, Cout):
    if kernel == "wreg":
        return 16 + int(math.log2(Cout // 128))
    return Cout // 32 + 6


def gn_partials_ref(out, TW, TH, mutation=None):
    """the per-chunk GroupNorm(32) partial statistics of the stored NHWC output out [B, H, W, C] (f32) in the conv epilogues' layout:
    (sums [B, H W / 32, 32, 2] float64, Sabs [same]: sum |v| and sum v^2, for the bound).  Chunk of pixel (y, x): tile (y / TH, x / TW)
    (row-major over the map's tiles), then its 32-pixel run (r / 32, r = (y % TH) TW + x % TW) within the tile."""
    B, H, W, C = out.shape
    cg = C // 32
    dev = out.device
    y, x = torch.meshgrid(torch.arange(H, device=dev), torch.arange(W, device=dev), indexing="ij")
    tiles_x = -(-W // TW)
    r = (y % TH) * TW + x % TW
    chunk = ((y // TH) * tiles_x + x // TW) * (TW * TH // 32) + r // 32
    keep = torch.ones_like(r, dtype=torch.bool)
    if mutation == "chunk_last_row_dropped":
        keep = r % 32 < 32 - TW
    v = out.double().reshape(B, H, W, 32, cg)
    if mutation == "neighbour_group":
        v = v.roll(1, 3)                                              # group g's values credited to group g + 1
    s1 = (v.sum(-1) * keep[..., None]).reshape(B, H * W, 32)
    s2 = ((v * v).sum(-1) * keep[..., None]).reshape(B, H * W, 32)
    a1 = (v.abs().sum(-1) * keep[..., None]).reshape(B, H * W, 32)
    nch = H * W // 32
    idx = chunk.reshape(-1)
    ref = torch.zeros(B, nch, 32, 2, dtype=torch.float64, device=dev)
    mag = torch.zeros_like(ref)
    ref[..., 0].index_add_(1, idx, s1)
    ref[..., 1].index_add_(1, idx, s2)
    mag[..., 0].index_add_(1, idx, a1)
    mag[..., 1].index_add_(1, idx, s2)
    return ref, mag


def gn_needles_bias(Cout, seed, device="cpu"):
    """a bias that makes each output group distinct: group g's channels at 4 (g + 1) (the conv's own output is O(1))"""
    g = torch.Generator().manual_seed(seed)
    return ((torch.arange(Cout) // (Cout // 32) + 1) * 4.0 + 0.1 * torch.randn(Cout, generator=g)).to(device)


# ---------------------------------------------------------------------------------------------------------------- mutation cases
# the launch each named mistake is shown on (shared by the CPU pinning and the GPU tests): streamer (fmt, e4m3, N, K, B, mode, splits,
# epilogue options); convs (B, H, W, Cin, Cout, ks, stride) on conv_needles
GEMM_MUTATION_CASES = {
    "last_kblock_dropped": dict(e4m3=False, N=256, K=1536, B=17, mode=3, splits=11),
    "last_kblock_twice": dict(e4m3=True, N=256, K=1280, B=33, mode=3, splits=13),
    "neighbour_row_scale": dict(e4m3=True, N=256, K=256, B=8, mode=0, splits=1),
    "neighbour_row_chunk": dict(e4m3=False, N=128, K=128, B=300, mode=1, splits=1),
    "tanh_gelu": dict(e4m3=False, N=256, K=128, B=16, mode=2, splits=1, bias=-3.0),
    "bias_scale_ignored": dict(e4m3=False, N=128, K=128, B=16, mode=0, splits=1, bias_scale=4.0),
    "residual_row_m": dict(e4m3=True, N=128, K=128, B=64, mode=0, splits=1, res_div=4),
}
CONV_MUTATION_CASES = {
    "drop_w_hi_x_lo": (2, 16, 16, 64, 128, 3, 1),
    "drop_w_lo_x_hi": (2, 16, 16, 64, 64, 3, 1),
    "transposed_taps": (2, 16, 16, 64, 128, 3, 1),
    "halo_shifted": (1, 8, 8, 64, 64, 3, 1),
    "stride2_pad_left_top": (3, 4, 4, 64, 128, 3, 2),
}
GN_MUTATION_CASES = {"neighbour_group": (2, 16, 16, 64, 128, 3, 1), "chunk_last_row_dropped": (3, 8, 8, 64, 256, 1, 1)}


def gemm_case_operands(case, seed, device="cpu"):
    """(W, scale, X, bias, residual) of a GEMM_MUTATION_CASES entry on gemm_needles"""
    fmt = 0
    W, s, X = gemm_needles(case["N"], case["K"], case["B"], fmt, seed, case["e4m3"], device)
    g = torch.Generator().manual_seed(seed + 1)
    bias = None
    if case["mode"] != 3:
        bias = (torch.full((case["N"],), case["bias"]) if "bias" in case else torch.randn(case["N"], generator=g)).to(device)
    res = torch.randn(case["B"], case["N"], generator=g).to(device) if case["mode"] == 0 else None
    return W, s, X, bias, res
