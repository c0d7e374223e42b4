"""The float64 references of tests/test_gpu_vae_kernels.py (tests/vae_kernels_ref.py), pinned on the CPU against an independent
formulation: F.conv2d with F.pad / F.interpolate, F.group_norm, AttnBlock's reshape / bmm / softmax (layers.py:158-182) and the
project's CPU oracle (oracle/rq_oracle.py _gn, attn_block).  Every named mistake is visible on its needle inputs: its reference lies
more than both tolerances away from the correct one somewhere."""
import pytest
import torch
import torch.nn.functional as F

from oracle import rq_oracle as O
from oracle.zoo import VAE_ZOO, vae_ddconfig
from tests import vae_kernels_ref as R


def separated(ref, tol, mut, mtol):
    return float(((ref - mut).abs() - tol - mtol).max()) > 0


def conv_case(B, H, W, Cin, Cout, ks, stride, up, in_nchw, out_nchw, seed, wdt=torch.float32, resid=True):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, Cin, H, W, generator=g) if in_nchw else torch.randn(B, H, W, Cin, generator=g)
    w = (torch.randn(Cout, ks, ks, Cin, generator=g) / (ks * ks * Cin) ** 0.5).to(wdt)
    bias = torch.randn(Cout, generator=g)
    Ho, Wo, _ = R.conv_geom(H, W, ks, stride, up)
    res = torch.randn(B, Ho, Wo, Cout, generator=g) if (resid and not out_nchw) else None
    return x, w, bias, res


@pytest.mark.parametrize("B,H,W,Cin,Cout,ks,stride,up,in_nchw,out_nchw", [
    (2, 5, 7, 6, 5, 3, 1, 0, 0, 0), (1, 4, 4, 8, 3, 3, 1, 0, 0, 1), (3, 6, 5, 4, 7, 3, 1, 1, 0, 0), (2, 8, 6, 4, 4, 3, 2, 0, 0, 0),
    (1, 7, 7, 5, 4, 3, 2, 0, 0, 0), (2, 6, 6, 3, 8, 3, 1, 0, 1, 0), (2, 5, 3, 4, 9, 1, 1, 0, 0, 0), (1, 2, 2, 4, 4, 3, 2, 0, 0, 0)])
@pytest.mark.parametrize("wdt", [torch.float32, torch.float16, torch.bfloat16])
def test_conv_reference_is_torch_conv2d(B, H, W, Cin, Cout, ks, stride, up, in_nchw, out_nchw, wdt):
    x, w, bias, res = conv_case(B, H, W, Cin, Cout, ks, stride, up, in_nchw, out_nchw, H * 100 + Cin, wdt)
    ref, slack = R.conv_ref(x, w, bias, res, B, H, W, Cin, Cout, ks, stride, up, in_nchw, out_nchw)
    xn = (x if in_nchw else x.permute(0, 3, 1, 2)).double()
    if up:
        xn = F.interpolate(xn, scale_factor=2.0, mode="nearest")                     # layers.py:31-35
    if stride == 2:
        xn = F.pad(xn, (0, 1, 0, 1))                                                  # layers.py:50-54
    want = F.conv2d(xn, w.double().permute(0, 3, 1, 2), bias.double(), stride=stride, padding=ks // 2 if stride == 1 else 0)
    if res is not None:
        want = want + res.double().permute(0, 3, 1, 2)
    got = ref if out_nchw else ref.permute(0, 3, 1, 2)
    torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)
    assert bool((slack > 0).all()) and float((slack / (ks * ks * Cin + 2)).max()) < 1e-5


@pytest.mark.parametrize("mutation", R.CONV_MUTATIONS)
def test_conv_mutations_are_visible(mutation):
    geo = {"pad_wrong_side": (2, 8, 8, 4, 4, 3, 2, 0, 0, 0), "upsample_round_up": (2, 4, 5, 4, 4, 3, 1, 1, 0, 0),
           "nhwc_as_nchw": (1, 6, 6, 3, 8, 3, 1, 0, 1, 0)}.get(mutation, (2, 5, 5, 8, 8, 3, 1, 0, 0, 0))
    x, w, bias, res = conv_case(*geo, seed=3)
    ref, slack = R.conv_ref(x, w, bias, res, *geo)
    mut, mslack = R.conv_ref(x, w, bias, res, *geo, mutation=mutation)
    assert separated(ref, slack, mut, mslack)


@pytest.mark.parametrize("B,HW,C", [(2, 1, 32), (3, 16, 64), (2, 257, 96), (1, 31, 128)])
@pytest.mark.parametrize("silu", [0, 1])
def test_groupnorm_reference_is_torch_group_norm(B, HW, C, silu):
    x, gamma, beta = R.gn_inputs(B, HW, C, seed=HW + C)
    ref = R.gn_ref(x, gamma, beta, silu)
    xn = x.double().permute(0, 2, 1)                                                  # [B, C, HW]
    want = F.group_norm(xn, 32, gamma.double(), beta.double(), R.GN_EPS)
    sd = {"n.weight": gamma.double(), "n.bias": beta.double()}
    torch.testing.assert_close(O._gn(sd, "n", xn), want, rtol=0, atol=0)            # the oracle's GroupNorm (layers.py:16-17)
    if silu:
        want = F.silu(want)
    torch.testing.assert_close(ref["y"], want.permute(0, 2, 1), rtol=1e-10, atol=1e-10)
    assert float(ref["rstd"][0, 0, 0, 0]) == pytest.approx(1000.0, rel=1e-12)       # the constant group
    for fused, fast in ((False, False), (False, True), (True, True)):
        s = R.gn_slack(x, gamma, beta, silu, ref, fused, fast)
        assert bool((s > 0).all()) and float(s.max()) < 1e-2


def test_groupnorm_cancellation_term_grows_with_r_squared():
    """the bound's variance term with and without the cancellation factor: equal shape at r = 0, r^2 apart at large r"""
    ratios = []
    for r in (0, 16, 256):
        x, gamma, beta = R.gn_inputs(2, 256, 128, seed=1, r=r)
        ref = R.gn_ref(x, gamma, beta, 0)
        s1 = R.gn_slack(x, gamma, beta, 0, ref, True, True)
        s0 = R.gn_slack(x, gamma, beta, 0, ref, True, True, cancel=False)
        ratios.append(float((s1 / s0).max()))
    assert ratios[0] < 3 and ratios[1] > 10 and ratios[2] > 1000


@pytest.mark.parametrize("mutation", R.GN_MUTATIONS)
@pytest.mark.parametrize("path", ["exact", "stats_f16", "fused_f16"])
def test_groupnorm_mutations_are_visible(mutation, path):
    """on gn_needles at HW = 16 (HW = 257, or 64 for the fused chunks of 32 pixels, for last_chunk_dropped): the fp32 outputs differ
    beyond both slacks; the fp16 forms are compared on hi + lo, which carries the fp32 bound plus half an ulp of lo"""
    fused, fast = path == "fused_f16", path != "exact"
    C = 64 if path == "exact" else 128
    HW = (64 if fused else 257) if mutation == "last_chunk_dropped" else 16
    chunk = R.FUSED_PIX if fused else R.GN_PIX
    x, gamma, beta = R.gn_needles(2, HW, C, seed=5)
    ref = R.gn_ref(x, gamma, beta, 1, chunk=chunk)
    mut = R.gn_ref(x, gamma, beta, 1, mutation=mutation, chunk=chunk)
    s = R.gn_slack(x, gamma, beta, 1, ref, fused, fast)
    extra = (lambda y: R.ulp16(y - y.half().double(), 0) / 2) if fast else (lambda y: 0)
    assert separated(ref["y"], s + extra(ref["y"]), mut["y"], R.gn_slack(x, gamma, beta, 1, mut, fused, fast) + extra(mut["y"]))


def test_split_check():
    x = torch.randn(100000, generator=torch.Generator().manual_seed(0)) * torch.logspace(-6, 4, 100000)
    hi = x.half()
    lo = (x - hi.float()).half()
    assert R.split_ok(hi, lo)
    rne = (hi.float() + lo.float()).half() == hi                                       # fp16-RNE of the sum is hi but at exact ties
    assert bool((rne | (lo.double().abs() == R.half_gap(hi, lo))).all())
    bad = (lo.float() + 4 * R.half_gap(hi, lo).float()).half()                         # lo pushed past the neighbour's midpoint
    assert not R.split_ok(hi, bad)


@pytest.mark.parametrize("up", [0, 1])
def test_cast_reference_is_interpolate(up):
    x = torch.randn(2, 3, 5, 8, generator=torch.Generator().manual_seed(1)) * 100
    hi, lo = R.cast_ref(x, up, True)
    xn = x.permute(0, 3, 1, 2)
    if up:
        xn = F.interpolate(xn, scale_factor=2.0, mode="nearest")
    assert torch.equal(hi, xn.permute(0, 2, 3, 1).half())
    assert R.split_ok(hi, lo)
    for m in R.CAST_MUTATIONS:
        mh, _ = R.cast_ref(x, up, True, mutation=m)
        assert not torch.equal(mh, hi), m


def attnblock_core(qkv, B, HW, C):
    """AttnBlock.forward's core as layers.py:158-182 writes it, on NCHW q, k, v"""
    x = qkv.reshape(B, HW, 3, C).double()
    q, k, v = (x[:, :, i].permute(0, 2, 1) for i in range(3))           # [B, C, HW]
    w_ = torch.bmm(q.permute(0, 2, 1), k) * (int(C) ** (-0.5))
    w_ = F.softmax(w_, dim=2)
    return torch.bmm(v, w_.permute(0, 2, 1)).permute(0, 2, 1)            # [B, HW, C]


@pytest.mark.parametrize("B,HW,C", [(1, 1, 32), (2, 7, 96), (1, 300, 64), (2, 16, 128)])
def test_attention_reference_is_attnblock(B, HW, C):
    qkv = R.attn_inputs(B, HW, C, seed=HW, needles=HW > 5)
    ref, slack = R.attn_ref(qkv, B, HW, C, rows=128)
    # the kernel's scale is float(C^-0.5), the layer's the double: the same to 2^-24 relative, well inside the check's 1e-6
    torch.testing.assert_close(ref, attnblock_core(qkv, B, HW, C), rtol=1e-6, atol=1e-6)
    assert bool((slack > 0).all()) and float((slack / (HW + 64)).max()) < 1e-4


def test_attention_block_matches_oracle():
    """GroupNorm -> fused q|k|v 1x1 conv -> attention core -> proj_out 1x1 conv + x, composed from this module's references in the
    engine's layout, equals the oracle's attn_block"""
    B, Hs, C = 2, 4, 64
    g = torch.Generator().manual_seed(4)
    x = torch.randn(B, C, Hs, Hs, generator=g, dtype=torch.float64)
    sd = {"a.norm.weight": torch.rand(C, generator=g, dtype=torch.float64) + 0.5,
          "a.norm.bias": torch.randn(C, generator=g, dtype=torch.float64)}
    for n in ("q", "k", "v", "proj_out"):
        sd["a.%s.weight" % n] = torch.randn(C, C, 1, 1, generator=g, dtype=torch.float64) / C ** 0.5
        sd["a.%s.bias" % n] = torch.randn(C, generator=g, dtype=torch.float64)
    want = O.attn_block(sd, "a", x)
    xh = x.permute(0, 2, 3, 1).reshape(B, Hs * Hs, C)
    h = R.gn_ref(xh, sd["a.norm.weight"], sd["a.norm.bias"], 0)["y"]
    wqkv = torch.cat([sd["a.%s.weight" % n] for n in "qkv"]).permute(0, 2, 3, 1)
    bqkv = torch.cat([sd["a.%s.bias" % n] for n in "qkv"])
    qkv, _ = R.conv_ref(h, wqkv, bqkv, None, B, Hs, Hs, C, 3 * C, 1, 1, 0, 0, 0)
    att, _ = R.attn_ref(qkv, B, Hs * Hs, C)
    out, _ = R.conv_ref(att, sd["a.proj_out.weight"].permute(0, 2, 3, 1), sd["a.proj_out.bias"], xh, B, Hs, Hs, C, C, 1, 1, 0, 0, 0)
    torch.testing.assert_close(out.permute(0, 3, 1, 2), want, rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("mutation", R.ATTN_MUTATIONS)
def test_attention_mutations_are_visible(mutation):
    B, HW, C = 2, 50, 128
    qkv = R.attn_inputs(B, HW, C, seed=2, needles=True)
    ref, slack = R.attn_ref(qkv, B, HW, C)
    mut, mslack = R.attn_ref(qkv, B, HW, C, mutation=mutation)
    assert separated(ref, slack, mut, mslack)


def test_layer_plans():
    """the walked layer plans hold the shapes the kernel tests are built around"""
    tiny = R.conv_plan(vae_ddconfig(**VAE_ZOO["tiny"]))
    big = R.conv_plan(vae_ddconfig(**VAE_ZOO["ffhq"]))
    assert (16, 16, 3, 32, 3, 1, 0, 1, 0) in tiny["conv"] and (16, 16, 32, 3, 3, 1, 0, 0, 1) in tiny["conv"]
    assert (8, 8, 64, 64, 3, 2, 0, 0, 0) in tiny["conv"] and (16, 16, 8192, 4) not in tiny["cast"]
    assert (128, 128, 128, 128, 3, 1, 1, 0, 0) in big["conv"] and (128, 128, 128, 1) in big["cast"]
    assert (256, 512) in big["attn"] and (64, 512) in big["attn"]
    assert (65536, 128) in big["gn"]
