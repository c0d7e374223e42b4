"""The VAE engine's kernels between its convs, and the exact tier's conv, one launch each through the engine's own launchers
(rqb200_dbg_vae_conv, rqb200_dbg_groupnorm, rqb200_dbg_cast_f16, rqb200_dbg_vae_attn), against the float64 references of
tests/vae_kernels_ref.py: every conv geometry of the tiny / FFHQ / ImageNet layer plans and the edges where the kernels change path,
GroupNorm on both tiers and both statistics paths, the fp16 operand casts, and the spatial attention.  Every output starts as NaN
with a guard region behind it: outputs within the derived tolerance (vae_kernels_ref's docstring; casts bit for bit), the guards keep
their bits, a second launch gives the same bits, and for each family a set of named mistakes that the tolerance rejects."""
import math

import pytest
import torch

from oracle.zoo import VAE_ZOO, vae_ddconfig
from rqvae import _native as N
from tests import vae_kernels_ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda"
GUARD = 512                     # elements behind every output buffer that no launch may touch
WDT = {N.F32: torch.float32, N.F16: torch.float16, N.BF16: torch.bfloat16}
_INT = {2: torch.int16, 4: torch.int32, 8: torch.int64}


def bits(x):
    return x.view(_INT[x.element_size()])


def nan_guarded(shape, dtype):
    """an all-NaN tensor of `shape` at the front of a device buffer with GUARD sentinel elements behind it -> (buffer, view)"""
    n = math.prod(shape)
    full = torch.full((n + GUARD,), float("nan"), dtype=dtype, device=DEV)
    bits(full)[n:] = 0x5A5A
    return full, full[:n].view(shape)


def guard_intact(full, n):
    return bool((bits(full)[n:] == 0x5A5A).all())


def twice(launch, *shapes):
    """launch(*views) on fresh NaN-filled guarded buffers, twice: the guards intact and the two results bit-identical -> views"""
    res = []
    for _ in range(2):
        bufs = [nan_guarded(s, d) if s is not None else (None, None) for s, d in shapes]
        N.check(launch(*[v for _, v in bufs]))
        torch.cuda.synchronize()
        for full, v in bufs:
            assert full is None or guard_intact(full, v.numel()), "guard overwritten"
        res.append([v for _, v in bufs])
    for a, b in zip(*res):
        assert a is None or torch.equal(bits(a), bits(b)), "second launch not bit-identical"
    return res[0]


def within(got, ref, tol, what):
    e = R.excess(got, ref, tol)
    assert e <= 0, "%s: %.3g beyond tolerance" % (what, e)


# ---------------------------------------------------------------------------------------------------------------- conv
def conv_inputs(geo, wcode, resid, seed):
    B, H, W, Cin, Cout, ks, stride, up, in_nchw, out_nchw = geo
    g = torch.Generator(DEV).manual_seed(seed)
    x = torch.randn(B, Cin, H, W, generator=g, device=DEV) if in_nchw else torch.randn(B, H, W, Cin, generator=g, device=DEV)
    w = (torch.randn(Cout, ks, ks, Cin, generator=g, device=DEV) / (ks * ks * Cin) ** 0.5).to(WDT[wcode])
    bias = torch.randn(Cout, generator=g, device=DEV)
    Ho, Wo, _ = R.conv_geom(H, W, ks, stride, up)
    res = torch.randn(B, Ho, Wo, Cout, generator=g, device=DEV) if resid else None
    return x, w, bias, res


def run_conv(geo, x, w, wcode, bias, res):
    B, H, W, Cin, Cout, ks, stride, up, in_nchw, out_nchw = geo
    Ho, Wo, _ = R.conv_geom(H, W, ks, stride, up)
    shape = (B, Cout, Ho, Wo) if out_nchw else (B, Ho, Wo, Cout)
    (out,) = twice(lambda o: N.lib().rqb200_dbg_vae_conv(N.ptr(x), N.ptr(w), wcode, N.ptr(bias), N.ptr(res), N.ptr(o), B, H, W, Cin,
                                                         Cout, ks, stride, up, in_nchw, out_nchw, N.stream_ptr()),
                   (shape, torch.float32))
    return out


def plan_geometries():
    geos = set()
    for name in ("tiny", "ffhq", "imagenet"):
        geos |= R.conv_plan(vae_ddconfig(**VAE_ZOO[name]))["conv"]
    return sorted(geos)


def plan_cases():
    """each geometry once: B = 1 from 64 x 64 up, else 2 or 3; the weight format and the residual cycle"""
    cases = []
    for i, (H, W, Cin, Cout, ks, stride, up, in_nchw, out_nchw) in enumerate(plan_geometries()):
        B = 1 if H >= 64 else 2 + i % 2
        cases.append(((B, H, W, Cin, Cout, ks, stride, up, in_nchw, out_nchw), (N.F32, N.F16, N.BF16)[i % 3],
                      not out_nchw and i % 2 == 0))
    return cases


# (B, H, W, Cin, Cout, ks, stride, upsample, in_nchw, out_nchw)
EDGE_GEOS = [
    (3, 1, 1, 64, 64, 3, 1, 0, 0, 0),       # 1 x 1 map, M = 3
    (3, 7, 7, 32, 96, 3, 1, 0, 0, 0),       # M = 147, Cout % 64 != 0
    (1, 7, 7, 6, 70, 3, 1, 0, 0, 0),        # Cin % 4 != 0 in NHWC: the scalar load path
    (2, 5, 3, 3, 40, 1, 1, 0, 0, 0),        # 1 x 1, Cin = 3 NHWC
    (3, 2, 2, 64, 64, 3, 2, 0, 0, 0),       # Downsample 2 -> 1
    (1, 3, 3, 32, 32, 3, 2, 0, 0, 0),       # odd extent under stride 2
    (3, 3, 5, 8, 24, 3, 1, 1, 0, 0),        # upsample of a non-square map
    (1, 9, 9, 3, 64, 3, 1, 0, 1, 0),        # NCHW conv_in, K = 27
    (3, 6, 6, 128, 3, 3, 1, 0, 0, 1),       # NCHW conv_out, Cout = 3
]


@pytest.mark.parametrize("geo,wcode,resid", plan_cases())
def test_conv_layer_plans(geo, wcode, resid):
    x, w, bias, res = conv_inputs(geo, wcode, resid, seed=sum(geo) * 7 + wcode)
    out = run_conv(geo, x, w, wcode, bias, res)
    ref, slack = R.conv_ref(x, w, bias, res, *geo)
    within(out, ref, slack, "conv %s w %d" % (geo, wcode))


@pytest.mark.parametrize("geo", EDGE_GEOS)
@pytest.mark.parametrize("wcode", [N.F32, N.F16, N.BF16])
@pytest.mark.parametrize("resid", [False, True])
def test_conv_edges(geo, wcode, resid):
    if resid and geo[-1]:
        pytest.skip("the NCHW output takes no residual")
    x, w, bias, res = conv_inputs(geo, wcode, resid, seed=sum(geo) + wcode)
    out = run_conv(geo, x, w, wcode, bias, res)
    ref, slack = R.conv_ref(x, w, bias, res, *geo)
    within(out, ref, slack, "conv %s w %d" % (geo, wcode))


def test_conv_rejects_mutations():
    geos = {"flipped_taps": (2, 5, 5, 8, 8, 3, 1, 0, 0, 0), "pad_wrong_side": (2, 8, 8, 4, 4, 3, 2, 0, 0, 0),
            "upsample_round_up": (2, 4, 5, 4, 4, 3, 1, 1, 0, 0), "bias_dropped": (2, 5, 5, 8, 8, 3, 1, 0, 0, 0),
            "nhwc_as_nchw": (1, 6, 6, 3, 8, 3, 1, 0, 1, 0)}
    for mutation in R.CONV_MUTATIONS:
        geo = geos[mutation]
        x, w, bias, res = conv_inputs(geo, N.F32, True, seed=3)
        out = run_conv(geo, x, w, N.F32, bias, res)
        ref, slack = R.conv_ref(x, w, bias, res, *geo)
        within(out, ref, slack, mutation + " needles")
        mut, mslack = R.conv_ref(x, w, bias, res, *geo, mutation=mutation)
        assert R.excess(out, mut, mslack) > 0, mutation


def test_conv_geometry_rule_refusals():
    x = torch.zeros(64, device=DEV)
    for args in ((1, 4, 4, 4, 4, 2, 1, 0, 0, 0), (1, 4, 4, 4, 4, 3, 3, 0, 0, 0), (1, 4, 4, 4, 4, 3, 2, 1, 0, 0)):
        B, H, W, Cin, Cout, ks, stride, up, i_n, o_n = args
        assert N.lib().rqb200_dbg_vae_conv(N.ptr(x), N.ptr(x), N.F32, None, None, N.ptr(x), B, H, W, Cin, Cout, ks, stride, up, i_n, o_n,
                                           N.stream_ptr()) == N.EINVAL


# ---------------------------------------------------------------------------------------------------------------- GroupNorm
def ws_doubles(B, HW):
    return B * -(-HW // 32) * 64 + B * 64


def run_gn(form, x, gamma, beta, silu, with_lo=True, ws=None):
    """(y f32 | hi, lo fp16): two launches; the statistics workspace (NaN, or `ws` = (buffer, view) a conv's epilogue filled for
    form 2) keeps its guard"""
    B, HW, C = x.shape
    n = ws_doubles(B, HW)
    wsfull, wsv = ws if ws is not None else nan_guarded((n,), torch.float64)

    def launch(y, hi, lo):
        return N.lib().rqb200_dbg_groupnorm(form, N.ptr(x), N.ptr(gamma), N.ptr(beta), N.ptr(y), N.ptr(hi), N.ptr(lo), N.ptr(wsv), n, B,
                                            HW, C, silu, N.stream_ptr())

    shp = (B, HW, C)
    outs = twice(launch, (shp if form == 0 else None, torch.float32), (shp if form else None, torch.float16),
                 (shp if form and with_lo else None, torch.float16))
    assert guard_intact(wsfull, n), "statistics workspace guard"
    return outs


def check_gn(form, x, gamma, beta, silu, outs, what, cancel=True):
    ref = R.gn_ref(x, gamma, beta, silu)
    slack = R.gn_slack(x, gamma, beta, silu, ref, form == 2, form > 0, cancel)
    y, hi, lo = outs
    if form == 0:
        within(y, ref["y"], slack, what)
        return ref
    within(hi, ref["y"], R.tol16(ref["y"], slack, 0), what + ": hi")
    if lo is not None:
        within(hi.double() + lo.double(), ref["y"], slack + R.ulp16(lo.double(), 0) / 2, what + ": hi + lo")
        assert R.split_ok(hi, lo), what + ": hi is not a nearest fp16 of hi + lo"
    return ref


HWS = [1, 16, 31, 64, 255, 256, 257, 1024, 4096, 65536]


def gn_cases():
    cases, i = [], 0
    for HW in HWS:
        for C in (32, 64, 96, 128, 256, 512):
            B = 1 if (i // 2) % 2 == 0 or HW * C > 4096 * 512 else 3
            cases.append((0, B, HW, C, i % 2))
            if C % 128 == 0:
                cases.append((1, 4 - B if HW * C <= 4096 * 512 else 1, HW, C, (i + 1) % 2))
            i += 1
    return cases


@pytest.mark.parametrize("form,B,HW,C,silu", gn_cases())
def test_groupnorm(form, B, HW, C, silu):
    x, gamma, beta = R.gn_inputs(B, HW, C, seed=HW * 7 + C + B, device=DEV)
    outs = run_gn(form, x, gamma, beta, silu, with_lo=(HW + C) % 2 == 0 or HW == 1)
    check_gn(form, x, gamma, beta, silu, outs, "form %d B %d HW %d C %d silu %d" % (form, B, HW, C, silu))
    if form and not silu:                                            # the constant group: x - mean = 0, so hi = fp16(beta)
        hi0 = outs[1][0, :, :C // 32]
        assert torch.equal(hi0, beta[:C // 32].half().expand_as(hi0))


def conv_gn_inputs(B, H, W, Cin, Cout, seed, r=None, needles=False):
    """the fp16 operands of a conv whose output feeds a GroupNorm: x, w, bias, residual.  Output group 0 has zero weights and bias
    0.75 (a constant group); the other groups' bias is +-r (r given; the conv output's std is about 1) or N(0, 2^2) plus N(0, 0.1^2)
    per channel.  needles: group 1's weights scaled by 1e-3 (var ~ 1e-6), and a residual of +40 on the last pixel in groups 2..31."""
    g = torch.Generator().manual_seed(seed)
    cg = Cout // 32
    x = torch.randn(B, H, W, Cin, generator=g).half()
    w = torch.randn(Cout, 3, 3, Cin, generator=g) / (9 * Cin) ** 0.5
    if r is None:
        gb = torch.randn(32, generator=g) * 2
    else:
        gb = r * (torch.randint(0, 2, (32,), generator=g) * 2 - 1).float()
    bias = gb.repeat_interleave(cg) + (0.1 * torch.randn(Cout, generator=g) if r is None else 0)
    w[:cg] = 0
    bias[:cg] = 0.75
    res = None
    if needles:
        w[cg:2 * cg] *= 1e-3
        bias[cg:2 * cg] = 0.3
        res = torch.zeros(B, H, W, Cout)
        res[:, -1, -1, 2 * cg:] = 40.0
    return x.to(DEV), w.half().to(DEV), bias.to(DEV), res.to(DEV) if res is not None else None


def fused_stats(x, w, bias, res, B, H, W, Cin, Cout):
    """one conv through rqb200_dbg_conv_tc_gn: (its output, the guarded workspace (buffer, view) holding its partial statistics).
    x and w are fp16 values, so their split-fp16 lo halves are zero."""
    ws = nan_guarded((ws_doubles(B, H * W),), torch.float64)
    ofull, out = nan_guarded((B, H, W, Cout), torch.float32)
    x_lo, w_lo = torch.zeros_like(x), torch.zeros_like(w)
    N.check(N.lib().rqb200_dbg_conv_tc_gn(N.ptr(x), N.ptr(w), N.ptr(x_lo), N.ptr(w_lo), N.ptr(bias), N.ptr(res), N.ptr(out), N.ptr(ws[1]), B, H, W,
                                          Cin, Cout, 3, 0, N.stream_ptr()), "dbg_conv_tc_gn")
    torch.cuda.synchronize()
    assert guard_intact(ofull, out.numel()) and guard_intact(ws[0], ws[1].numel())
    return out, ws


def gn_affine(C, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(C, generator=g) + 0.5).to(DEV), torch.randn(C, generator=g).to(DEV)


# the decoder shapes of tests/test_gpu_conv3x3.py's GroupNorm statistics test
FUSED_SHAPES = [(2, 8, 8, 256, 512), (3, 8, 8, 512, 512), (2, 16, 16, 128, 128), (1, 32, 32, 512, 256), (1, 256, 256, 128, 128),
                (2, 64, 32, 256, 256)]


@pytest.mark.parametrize("B,H,W,Cin,Cout", FUSED_SHAPES)
@pytest.mark.parametrize("silu", [0, 1])
def test_groupnorm_fused_pipeline(B, H, W, Cin, Cout, silu):
    """form 2: the conv epilogue's partials -> gn_finalize -> gn_apply_f16, against fp64 GroupNorm of the output the conv stored"""
    x, w, bias, _ = conv_gn_inputs(B, H, W, Cin, Cout, seed=H + Cout + silu)
    out, ws = fused_stats(x, w, bias, None, B, H, W, Cin, Cout)
    gamma, beta = gn_affine(Cout, H + silu)
    y = out.view(B, H * W, Cout)
    outs = run_gn(2, y, gamma, beta, silu, with_lo=silu == 1 or H == 8, ws=ws)
    check_gn(2, y, gamma, beta, silu, outs, "fused B %d %dx%d C %d silu %d" % (B, H, W, Cout, silu))


R_SWEEP = [0, 4, 16, 64, 256]


@pytest.mark.parametrize("r", R_SWEEP)
@pytest.mark.parametrize("form", [0, 1, 2])
def test_groupnorm_mean_offset_sweep(form, r):
    """groups whose mean is r standard deviations off zero: the variance's E[x^2] - mean^2 loses ~ r^2 of its relative accuracy, which
    the derived bound carries (scripts/gn_variance_sweep.py records the measured error next to torch's fp32 group_norm)"""
    if form == 2:
        B, H, W, C = 2, 16, 16, 128
        x, w, bias, _ = conv_gn_inputs(B, H, W, C, C, seed=r + 1, r=r)
        out, ws = fused_stats(x, w, bias, None, B, H, W, C, C)
        y, ws = out.view(B, H * W, C), ws
    else:
        y, _, _ = R.gn_inputs(2, 1024, 128, seed=r + 1, r=r, device=DEV)
        ws = None
    gamma, beta = gn_affine(y.shape[2], r)
    outs = run_gn(form, y, gamma, beta, 1, ws=ws)
    check_gn(form, y, gamma, beta, 1, outs, "form %d r %d" % (form, r))


@pytest.mark.parametrize("form", [0, 1, 2])
def test_groupnorm_rejects_mutations(form):
    """needle inputs (vae_kernels_ref.gn_needles; for form 2 the conv-made equivalent): the fp32 output, or hi + lo, is within the bound
    of the reference and outside it for each mistake.  HW = 16, and HW = 257 (64 for the fused 32-pixel chunks) for the dropped chunk."""
    for mutation in R.GN_MUTATIONS:
        last = mutation == "last_chunk_dropped"
        if form == 2:
            B, H, W, C = 2, 8, 8, 128
            x, w, bias, res = conv_gn_inputs(B, H, W, C, C, seed=5, needles=True)
            out, ws = fused_stats(x, w, bias, res, B, H, W, C, C)
            y = out.view(B, H * W, C)
        else:
            y, ws = R.gn_needles(2, 257 if last else 16, 64 if form == 0 else 128, seed=5, device=DEV)[0], None
        gamma, beta = gn_affine(y.shape[2], 9)
        outs = run_gn(form, y, gamma, beta, 1, ws=ws)
        check_gn(form, y, gamma, beta, 1, outs, mutation + " needles")
        got = outs[0] if form == 0 else outs[1].double() + outs[2].double()
        chunk = R.FUSED_PIX if form == 2 else R.GN_PIX
        mut = R.gn_ref(y, gamma, beta, 1, mutation=mutation, chunk=chunk)
        tol = R.gn_slack(y, gamma, beta, 1, mut, form == 2, form > 0) + (R.ulp16(outs[2].double(), 0) / 2 if form else 0)
        assert R.excess(got, mut["y"], tol) > 0, mutation


def test_groupnorm_workspace_check():
    x = torch.zeros(2, 64, 128, device=DEV)
    g = torch.ones(128, device=DEV)
    ws = torch.zeros(ws_doubles(2, 64), dtype=torch.float64, device=DEV)
    y = torch.empty_like(x)
    for form in (0, 1, 2):
        rc = N.lib().rqb200_dbg_groupnorm(form, N.ptr(x), N.ptr(g), N.ptr(g), N.ptr(y), N.ptr(y), None, N.ptr(ws), ws.numel() - 1, 2, 64,
                                          128, 1, N.stream_ptr())
        assert rc == N.EWORKSPACE
    assert N.lib().rqb200_dbg_groupnorm(1, N.ptr(x), N.ptr(g), N.ptr(g), None, N.ptr(y), None, N.ptr(ws), ws.numel(), 2, 64, 96, 1,
                                        N.stream_ptr()) == N.EINVAL


# ---------------------------------------------------------------------------------------------------------------- cast
CAST_CASES = [(2, 8, 8, 512, 1), (1, 16, 16, 512, 1), (1, 32, 32, 256, 1), (1, 64, 64, 256, 1), (1, 128, 128, 128, 1),
              (3, 8, 8, 256, 0), (2, 16, 16, 512, 0), (1, 256, 256, 128, 0), (1, 5, 7, 4, 1), (3, 3, 5, 12, 1), (2, 6, 10, 4, 0)]


def run_cast(x, up, with_lo):
    B, H, W, C = x.shape
    shp = (B, 2 * H, 2 * W, C) if up else (B, H, W, C)
    return twice(lambda hi, lo: N.lib().rqb200_dbg_cast_f16(N.ptr(x), N.ptr(hi), N.ptr(lo), B, H, W, C, up, N.stream_ptr()),
                 (shp, torch.float16), (shp if with_lo else None, torch.float16))


@pytest.mark.parametrize("B,H,W,C,up", CAST_CASES)
@pytest.mark.parametrize("with_lo", [False, True])
def test_cast_f16(B, H, W, C, up, with_lo):
    """bit for bit: hi = x.half(), lo = (x - hi).half(), upsampled by repeat_interleave.  |x| spans about 2^-32 .. 2^13: subnormal hi
    and lo, and lo at every scale"""
    g = torch.Generator(DEV).manual_seed(B * H * W + C)
    x = torch.randn(B, H, W, C, generator=g, device=DEV) * torch.pow(2.0, torch.randint(-30, 12, (B, H, W, C), generator=g, device=DEV))
    hi, lo = run_cast(x, up, with_lo)
    want_hi, want_lo = R.cast_ref(x, up, with_lo)
    assert torch.equal(bits(hi), bits(want_hi))
    if with_lo:
        assert torch.equal(bits(lo), bits(want_lo))


def test_cast_rejects_mutations():
    x = torch.randn(2, 5, 7, 8, generator=torch.Generator(DEV).manual_seed(2), device=DEV)
    for up in (0, 1):
        hi, lo = run_cast(x, up, True)
        for mutation in R.CAST_MUTATIONS:
            mh, ml = R.cast_ref(x, up, True, mutation=mutation)
            assert not (torch.equal(bits(hi), bits(mh)) and torch.equal(bits(lo), bits(ml))), mutation


# ---------------------------------------------------------------------------------------------------------------- attention
def run_attn(qkv, B, HW, C):
    (out,) = twice(lambda o: N.lib().rqb200_dbg_vae_attn(N.ptr(qkv), N.ptr(o), B, HW, C, N.stream_ptr()), ((B, HW, C), torch.float32))
    return out


ATTN_CASES = [(2, 16, 128, False), (1, 64, 512, False), (2, 256, 512, False),            # the engine's shapes
              (3, 1, 128, False), (2, 7, 96, True), (1, 300, 128, True), (1, 1024, 512, False), (2, 64, 96, False),
              (1, 300, 768, True), (2, 256, 512, True), (1, 11800, 128, False)]          # last: near the 48 KB shared-memory limit


@pytest.mark.parametrize("B,HW,C,needles", ATTN_CASES)
def test_vae_attention(B, HW, C, needles):
    qkv = R.attn_inputs(B, HW, C, seed=HW + C, needles=needles, device=DEV)
    out = run_attn(qkv, B, HW, C)
    ref, slack = R.attn_ref(qkv, B, HW, C)
    within(out, ref, slack, "attn B %d HW %d C %d" % (B, HW, C))


def test_vae_attention_rejects_mutations():
    B, HW, C = 2, 300, 128
    qkv = R.attn_inputs(B, HW, C, seed=2, needles=True, device=DEV)
    out = run_attn(qkv, B, HW, C)
    ref, slack = R.attn_ref(qkv, B, HW, C)
    within(out, ref, slack, "needles")
    for mutation in R.ATTN_MUTATIONS:
        mut, mslack = R.attn_ref(qkv, B, HW, C, mutation=mutation)
        assert R.excess(out, mut, mslack) > 0, mutation


@pytest.mark.parametrize("HW", [12127, 12160, 12161])
def test_vae_attention_refuses_past_shared_memory(HW):
    """C + HW floats beside the kernel's static shared memory over 48 KB: RQB200_EINVAL and nothing written.  HW = 12160 and 12127 fit
    48 KB without the static shared memory; the launcher once let them through to a launch that failed with a CUDA error"""
    B, C = 1, 128
    qkv = torch.zeros(B, HW, 3 * C, device=DEV)
    full, out = nan_guarded((B, HW, C), torch.float32)
    assert N.lib().rqb200_dbg_vae_attn(N.ptr(qkv), N.ptr(out), B, HW, C, N.stream_ptr()) == N.EINVAL
    torch.cuda.synchronize()
    assert bool(torch.isnan(out).all()) and guard_intact(full, out.numel())
