"""The native ResNet-101 on the GPU: both tiers against the torchvision fixture (tests/golden/resnet.pt) and the float64 restatement
(tests/resnet_oracle.py), batch independence across the 2 GiB chunk boundary, the residual epilogues of both conv kernels and the padded
stride-2 convs against float64 at their edges, the input kernel against torch bit for bit, and rejection sampling on zoo models."""
import pytest
import torch
import torch.nn.functional as F

from oracle import synth
from rqvae import _native as N
from rqvae.metrics import inception as INC
from rqvae.metrics import resnet as RN
from rqvae.metrics.resnet import ResNet101
from tests import resnet_oracle as RO

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
# rel-L2 bounds of the logits and of class_log_prob against float64, per tier.  On an H100 the fixture's cases and the restatement's
# shapes measured at most 1.0e-6 (logits) and 4.9e-6 (class log-prob) on the exact tier (fp32 FFMA through 104 convs and 33 residual
# adds), and 1.4e-5 and 2.7e-5 on the fast tier (split-fp16 operands, which drop the lo x lo product)
EXACT_BOUND = 1e-5
FAST_BOUND = 1e-4


def rel(a, b):
    return float((a.double().cpu() - b.double().cpu()).norm() / b.double().cpu().norm())


@pytest.fixture(scope="module")
def fixture(golden):
    return golden("resnet")


@pytest.fixture(scope="module")
def weights(fixture):
    return RO.synth_weights(fixture["seed"])


def make(weights, precision):
    m = ResNet101()
    m.load_state_dict(weights)
    m = m.to(DEV)
    m.precision = precision
    return m


@pytest.fixture(scope="module")
def exact(weights):
    return make(weights, "exact")


@pytest.fixture(scope="module")
def fast(weights):
    return make(weights, "fast")


@pytest.fixture(scope="module")
def sd64(weights):
    return RO.sd_as(weights, torch.float64, DEV)


def check_against(m, tier, x, ref, what):
    """logits and class_log_prob of x against the float64 logits ref; the top-1 class wherever ref's top-2 margin exceeds the bound"""
    b = EXACT_BOUND if tier == "exact" else FAST_BOUND
    crop = what[1]
    with torch.no_grad():
        lg = m(x, center_crop=crop)
        labels = torch.stack([ref.argmax(1).cpu(), torch.full((x.shape[0],), 7)], 0)
        lps = [m.class_log_prob(x, lb.to(DEV), center_crop=crop) for lb in labels]
    ref_lp = torch.log_softmax(ref.double().cpu(), 1)
    e_lg = rel(lg, ref)
    e_lp = max(rel(lp, ref_lp.gather(1, lb[:, None])[:, 0]) for lp, lb in zip(lps, labels))
    print("ResNet-101 %s %s: logits rel-L2 %.3g, class log-prob rel-L2 %.3g" % (tier, what[0], e_lg, e_lp))
    assert e_lg <= b and e_lp <= b, (e_lg, e_lp, b)
    top2 = ref.double().cpu().topk(2, 1).values
    for i in range(x.shape[0]):
        if float(top2[i, 0] - top2[i, 1]) > 2 * b * float(ref[i].double().norm()):
            assert int(lg[i].argmax()) == int(ref[i].argmax()), i


@pytest.mark.parametrize("tier", ["exact", "fast"])
@pytest.mark.parametrize("idx", range(5))
def test_matches_torchvision_fixture(exact, fast, fixture, tier, idx):
    case = fixture["cases"][idx]
    x = RO.case_inputs(case).to(DEV)
    check_against(exact if tier == "exact" else fast, tier, x, case["logits"], (case["name"], case["crop"]))


@pytest.mark.parametrize("tier", ["exact", "fast"])
@pytest.mark.parametrize("B,H,W,crop", [(3, 64, 96, None), (2, 225, 227, 224), (1, 33, 47, None), (2, 300, 260, 256)])
def test_matches_restatement(exact, fast, sd64, tier, B, H, W, crop):
    g = torch.Generator().manual_seed(B * 1000 + H)
    x = torch.rand(B, 3, H, W, generator=g).to(DEV)
    with torch.no_grad():
        ref = RO.logits(sd64, x.double(), crop)
    check_against(exact if tier == "exact" else fast, tier, x, ref, ("%dx%dx%d" % (B, H, W), crop))


def test_features_and_launches(exact, sd64):
    x = torch.rand(2, 3, 64, 64, generator=torch.Generator().manual_seed(5)).to(DEV)
    with torch.no_grad():
        lg, feat = exact._run(x, None, features=True)
        ref = RO.features(sd64, RO.preprocess(x.double(), None))
    assert torch.equal(lg, exact(x, center_crop=None))
    assert rel(feat, ref) <= EXACT_BOUND
    assert exact.last_launches >= 1 + 104 + 1 + 1 + 1          # input, convs, max pool, average pool, fc


@pytest.mark.parametrize("tier", ["exact", "fast"])
def test_rows_do_not_depend_on_the_batch_or_the_chunking(exact, fast, tier):
    """26 images of 512^2 pass the 2 GiB chunk (24 images per chunk on the exact tier, 13 on the fast)"""
    m = exact if tier == "exact" else fast
    x = torch.rand(26, 3, 512, 512, generator=torch.Generator().manual_seed(6)).to(DEV)
    with torch.no_grad():
        full = m(x, center_crop=None)
        for a, b in ((0, 5), (12, 14), (20, 26), (23, 25), (25, 26)):
            assert torch.equal(m(x[a:b], center_crop=None), full[a:b]), (a, b)
        crop = m(x[:3], center_crop=224)
        assert torch.equal(m(x[1:2], center_crop=224), crop[1:2])


def test_engine_rebuilds_after_load_state_dict(weights):
    m = make(weights, "exact")
    x = torch.rand(1, 3, 40, 40, generator=torch.Generator().manual_seed(7)).to(DEV)
    with torch.no_grad():
        before = m(x, center_crop=None).clone()
        sd = {k: v.clone() for k, v in weights.items()}
        sd["fc.bias"] = sd["fc.bias"] + 1.0
        m.load_state_dict(sd)
        after = m(x, center_crop=None)
        m.fc.bias.data.sub_(1.0)
        again = m(x, center_crop=None)
    assert torch.allclose(after, before + 1.0, atol=1e-5)
    assert torch.allclose(again, before, atol=1e-5)


# ------------------------------------------------------------------------------------------------ the residual conv epilogues
# (Cin, Cout, H, W, k, pad, stride, B): bottleneck conv3 at Cout 64 / 256 / 2048, the downsample 1x1/2 and the 3x3/2 pad 1 at odd and
# even extents down to 7 x 7 and 1 x 1 outputs, and batches that end inside a tile (7 x 7 maps are tiled 8 x 8 x 2 images, 1 x 1 maps 128
# images per tile)
GEOMS = [(64, 64, 14, 14, 1, 0, 1, 3), (64, 256, 56, 56, 1, 0, 1, 1), (512, 2048, 7, 7, 1, 0, 1, 3), (128, 512, 9, 11, 1, 0, 1, 2),
         (256, 512, 56, 56, 1, 0, 2, 1), (256, 512, 15, 15, 1, 0, 2, 2), (1024, 2048, 14, 14, 1, 0, 2, 3), (1024, 2048, 13, 13, 1, 0, 2, 1),
         (1024, 2048, 2, 2, 1, 0, 2, 5), (1024, 2048, 1, 1, 1, 0, 2, 5),
         (128, 128, 56, 56, 3, 1, 2, 1), (128, 128, 13, 13, 3, 1, 2, 3), (256, 256, 14, 14, 3, 1, 2, 3), (256, 256, 15, 14, 3, 1, 2, 1),
         (512, 512, 2, 2, 3, 1, 2, 5), (512, 512, 1, 1, 3, 1, 2, 3), (512, 512, 3, 3, 3, 1, 2, 1), (64, 64, 7, 7, 3, 1, 1, 3)]


def conv_case(g, seed):
    ci, co, H, W, k, pad, s, B = g
    x = synth.randn_seeded((B, ci, H, W), seed).abs()
    w = synth.randn_seeded((co, ci, k, k), seed + 1, (2.0 / (k * k * ci)) ** 0.5)
    b = synth.randn_seeded((co,), seed + 2, 0.1)
    Ho, Wo = (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1
    r = synth.randn_seeded((B, Ho, Wo, co), seed + 3)
    return x.to(DEV), w.to(DEV), b.to(DEV), r.to(DEV), Ho, Wo


def ref_conv(x, w, b, r, pad, s, relu):
    y = F.conv2d(x.double(), w.double(), b.double(), stride=s, padding=pad).permute(0, 2, 3, 1)
    if r is not None:
        y = y + r.double()
    return F.relu(y) if relu else y


@pytest.mark.parametrize("g", GEOMS, ids=lambda g: "%dto%d_%dx%d_k%dp%ds%d_B%d" % g)
@pytest.mark.parametrize("form", ["res_relu", "res_id", "id"])
def test_residual_epilogues(g, form):
    ci, co, H, W, k, pad, s, B = g
    x, w, b, r, Ho, Wo = conv_case(g, 31)
    relu = form == "res_relu"
    res = None if form == "id" else r
    L = RN._lib()
    xn, wn = x.permute(0, 2, 3, 1).contiguous(), w.permute(0, 2, 3, 1).contiguous()
    ref = ref_conv(x, w, b, res, pad, s, relu)
    out = torch.full((B, Ho, Wo, co), 7.0, device=DEV)
    N.check(L.rqb200_dbg_resnet_conv(N.ptr(xn), N.ptr(wn), N.ptr(b), N.ptr(res), N.ptr(out), B, H, W, ci, co, k, pad, s, co, 0, int(relu),
                                     N.stream_ptr()), "dbg_resnet_conv")
    assert float((out.double() - ref).abs().max()) <= 1e-5 * float(ref.abs().max()) + 1e-6
    xh, xl = xn.half(), (xn - xn.half().float()).half()
    wh, wl = wn.half(), (wn - wn.half().float()).half()
    ref16 = ref_conv((xh.double() + xl.double()).permute(0, 3, 1, 2), (wh.double() + wl.double()).permute(0, 3, 1, 2), b, res, pad, s, relu)
    out = torch.full((B, Ho, Wo, co), 7.0, device=DEV)
    oh = torch.full((B, Ho, Wo, co), 7.0, device=DEV, dtype=torch.half)
    ol = torch.full((B, Ho, Wo, co), 7.0, device=DEV, dtype=torch.half)
    N.check(L.rqb200_dbg_resnet_conv_tc(N.ptr(xh), N.ptr(xl), N.ptr(wh), N.ptr(wl), N.ptr(b), N.ptr(res), N.ptr(out), N.ptr(oh), N.ptr(ol),
                                        B, H, W, ci, co, k, pad, s, co, 0, int(relu), N.stream_ptr()), "dbg_resnet_conv_tc")
    assert float((out.double() - ref16).abs().max()) <= 2e-5 * float(ref16.abs().max()) + 1e-6
    assert torch.equal(oh, out.half()) and torch.equal(ol, (out - out.half().float()).half())


@pytest.mark.parametrize("g", [g for g in GEOMS if g[6] == 2], ids=lambda g: "%dto%d_%dx%d_k%dp%ds%d_B%d" % g)
def test_padded_stride2_on_the_relu_form(g):
    """the bottleneck conv2 (3x3/2 pad 1) and the 1x1/2 on inc_conv_tc_kernel's plain ReLU form: the box of output column / row 0 starts
    at -1 with element stride 2, and TMA's zero fill must stand for the padding"""
    ci, co, H, W, k, pad, s, B = g
    x, w, b, _, Ho, Wo = conv_case(g, 41)
    xn, wn = x.permute(0, 2, 3, 1).contiguous(), w.permute(0, 2, 3, 1).contiguous()
    xh, xl = xn.half(), (xn - xn.half().float()).half()
    wh, wl = wn.half(), (wn - wn.half().float()).half()
    ref16 = ref_conv((xh.double() + xl.double()).permute(0, 3, 1, 2), (wh.double() + wl.double()).permute(0, 3, 1, 2), b, None, pad, s, True)
    out = torch.full((B, Ho, Wo, co), 7.0, device=DEV)
    N.check(INC._lib().rqb200_dbg_inception_conv_tc(N.ptr(xh), N.ptr(xl), N.ptr(wh), N.ptr(wl), N.ptr(b), N.ptr(out), None, None, B, H, W,
                                                    ci, co, k, k, pad, pad, s, co, 0, N.stream_ptr()), "dbg_inception_conv_tc")
    assert float((out.double() - ref16).abs().max()) <= 2e-5 * float(ref16.abs().max()) + 1e-6


def test_residual_reads_the_output_slice():
    """ldy / yoff place the output and the residual read alike"""
    ci, co, H, W, B, ldy, yoff = 64, 64, 5, 6, 2, 192, 64
    x, w, b, _, Ho, Wo = conv_case((ci, co, H, W, 1, 0, 1, B), 51)
    r = synth.randn_seeded((B, H, W, ldy), 55).to(DEV)
    xn, wn = x.permute(0, 2, 3, 1).contiguous(), w.permute(0, 2, 3, 1).contiguous()
    ref = ref_conv(x, w, b, r[..., yoff:yoff + co], 0, 1, True)
    xh, xl = xn.half(), (xn - xn.half().float()).half()
    wh, wl = wn.half(), (wn - wn.half().float()).half()
    for tc in (False, True):
        out = r.clone()
        if tc:
            N.check(RN._lib().rqb200_dbg_resnet_conv_tc(N.ptr(xh), N.ptr(xl), N.ptr(wh), N.ptr(wl), N.ptr(b), N.ptr(r), N.ptr(out), None, None,
                                                        B, H, W, ci, co, 1, 0, 1, ldy, yoff, 1, N.stream_ptr()), "dbg_resnet_conv_tc")
        else:
            N.check(RN._lib().rqb200_dbg_resnet_conv(N.ptr(xn), N.ptr(wn), N.ptr(b), N.ptr(r), N.ptr(out), B, H, W, ci, co, 1, 0, 1, ldy, yoff, 1,
                                                     N.stream_ptr()), "dbg_resnet_conv")
        assert torch.equal(out[..., :yoff], r[..., :yoff]) and torch.equal(out[..., yoff + co:], r[..., yoff + co:])
        assert float((out[..., yoff:yoff + co].double() - ref).abs().max()) <= 2e-3 * float(ref.abs().max())


# ------------------------------------------------------------------------------------------------ the input kernel
@pytest.mark.parametrize("B,H,W,crop", [(2, 256, 256, 224), (1, 97, 131, 0), (1, 225, 227, 224), (2, 33, 40, 32), (1, 226, 300, 224)])
def test_input_kernel_is_torch_bit_for_bit(B, H, W, crop):
    x = torch.rand(B, 3, H, W, generator=torch.Generator().manual_seed(H * W)).to(DEV)
    c = crop or None
    y = torch.empty(B, c or H, c or W, 3, device=DEV)
    N.check(RN._lib().rqb200_dbg_resnet_input(N.ptr(x), N.ptr(y), B, H, W, crop, N.stream_ptr()), "dbg_resnet_input")
    try:
        from torchvision import transforms
        xc = transforms.CenterCrop(c)(x) if c else x
        ref = transforms.Normalize(RO.MEAN, RO.STD)(xc)
    except ImportError:
        ref = RO.preprocess(x, c)
    assert torch.equal(y, ref.permute(0, 2, 3, 1))


# ------------------------------------------------------------------------------------------------ rejection sampling
@pytest.fixture(scope="module")
def zoo(layouts):
    from tests.helpers import build_ar, build_vae
    ar, _ = build_ar("tiny", layouts, 61, DEV)
    vae, _ = build_vae("tiny_attn_mid", layouts, 62, DEV)
    ar.precision = "exact"
    vae.precision = "exact"
    clf = make(RO.synth_weights(63), "exact")
    return ar, vae, clf


def test_rejection_sample_is_the_hand_written_loop(zoo):
    from rqvae.models.rqtransformer import rejection_sample
    ar, vae, clf = zoo
    labels = torch.tensor([3, 0, 9], device=DEV)
    kw = dict(temperature=1.0, top_k=64, top_p=0.95)
    torch.manual_seed(123)
    codes, pixels, scores = rejection_sample(ar, vae, clf, labels, candidates=4, batch_size=2, center_crop=None, **kw)
    torch.manual_seed(123)
    cands = []
    with torch.no_grad():
        for c in range(4):
            for s, e in ((0, 2), (2, 3)):
                cd = ar.sample(torch.zeros(e - s, 4, 4, 4, dtype=torch.long, device=DEV), model_aux=vae, cond=labels[s:e, None], **kw)
                px = torch.clamp(vae.decode_code(cd) * 0.5 + 0.5, 0, 1)
                cands.append((c, s, e, cd, px, clf.class_log_prob(px, labels[s:e], center_crop=None)))
    all_sc = torch.full((4, 3), float("nan"), device=DEV)
    for c, s, e, cd, px, sc in cands:
        all_sc[c, s:e] = sc
    best = [int(torch.nonzero(all_sc[:, i] == all_sc[:, i].max())[0]) for i in range(3)]       # the first of the maxima
    assert pixels.shape == (3, 3, 32, 32) and codes.shape == (3, 4, 4, 4) and scores.dtype == torch.float32
    for i in range(3):
        c, s, e, cd, px, sc = next(t for t in cands if t[0] == best[i] and t[1] <= i < t[2])
        assert torch.equal(codes[i], cd[i - s]) and torch.equal(pixels[i], px[i - s]) and torch.equal(scores[i], sc[i - s])
    assert float(pixels.min()) >= 0.0 and float(pixels.max()) <= 1.0


def test_one_candidate_is_sample(zoo):
    from rqvae.models.rqtransformer import rejection_sample
    ar, vae, clf = zoo
    labels = torch.tensor([1, 4], device=DEV)
    torch.manual_seed(7)
    codes, _, scores = rejection_sample(ar, vae, clf, labels, candidates=1, center_crop=None, top_k=32)
    torch.manual_seed(7)
    ref = ar.sample(torch.zeros(2, 4, 4, 4, dtype=torch.long, device=DEV), model_aux=vae, cond=labels[:, None], top_k=32)
    assert torch.equal(codes, ref) and bool(torch.isfinite(scores).all())
